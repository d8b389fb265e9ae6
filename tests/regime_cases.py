"""Cases of the launch regimes that only full-size layers reach, and the size rules that decide them, mirrored from the C++
so that a CPU test can check which case tables reach which regime (tests/test_full_size_regimes_cpu.py):
- conv_swap_kernel in a training plan (model.cu, conv_kernel: swap_cases.selects_swap), writing ReLU planes that the next
  layer's data-gradient mask and native weight gradient read, or the raw z of a BatchNormalization layer;
- bn_stats_kernel / bn_bwd_reduce_kernel with more than one element per thread (bn.cu, bn_grid: the grid is capped at
  8 * SMs blocks, and each thread then strides over the pixels with its channel group), also on an odd group count;
- wgrad_direct3x3_kernel / wgrad_direct_kernel with more than one output row per block (train.cu: rows_per_block =
  ceil(B * H / (8 * SMs))), including a last block that holds fewer rows;
- conv_direct_kernel writing the z of a BatchNormalization layer at SSD7's notebook size (B x 300 x 480, 5x5, 3 -> 32).

Each case is a tests/test_gpu_backward_kernels.py case (bcase) sized just past its threshold, plus
  'fwd': {layer: ssdk_model_layer_plan kernel} the training plan must choose,
  'regimes': the regimes (names below) it must reach on the device it runs on.
"""
from conv_cases import SM_COUNT_H100
from oracle import opexact
from swap_cases import selects_swap
import test_gpu_train_step_kernels as ts
from test_gpu_backward_kernels import D, bcase, conv, head

SWAP_RELU = 'swap_relu_train'              # conv_swap_kernel writes ReLU planes in a training plan
SWAP_BN = 'swap_bn_train'                  # conv_swap_kernel writes the z of a BatchNormalization layer
BN_STRIDED = 'bn_strided'                  # BatchNormalization reductions with >= 2 elements per thread
BN_STRIDED_ODD = 'bn_strided_cut_grid'     # ... on a grid cut to a multiple of a group count that does not divide 256
WGRAD_ROWS = 'direct_wgrad_multirow'       # a direct weight gradient with >= 2 output rows per block
DIRECT_BN = 'direct_bn_strided'            # conv_direct_kernel into the z of a strided BatchNormalization
REGIMES = (SWAP_RELU, SWAP_BN, BN_STRIDED, BN_STRIDED_ODD, WGRAD_ROWS, DIRECT_BN)


# ------------------------------------------------------------------------------------------------------------------------------
# the size rules
# ------------------------------------------------------------------------------------------------------------------------------
def bn_grid(B, H, W, C, sm_count=SM_COUNT_H100):
    """bn.cu, bn_grid (mirrored in test_gpu_train_step_kernels) -> (blocks, elements per thread of the longest thread, whether
    the grid was cut below min(elements / 256, 8 * SMs) to a multiple of the group count).  An element is 8 channels of a pixel."""
    total = B * H * W * ((C + 7) // 8)
    blocks = ts.bn_grid(B, H, W, C, sm_count)[0]
    return blocks, -(-total // (blocks * 256)), blocks < min(-(-total // 256), 8 * sm_count)


def direct_wgrad_rows(B, Ho, sm_count=SM_COUNT_H100):
    """train.cu, the direct weight-gradient launch -> (rows_per_block, grid, rows of the last block) (oracle/opexact.py)."""
    return opexact.direct_wgrad_rows(B, Ho, sm_count)


def selects_direct(cin, cout, k, stride):
    """model.cu, conv_kernel: the image-facing conv_direct_kernel (a training plan keeps it; 1 ... 4 input channels)."""
    return 1 <= cin <= 4 and stride == 1 and cout % 16 == 0 and k * k * cin * cout * 4 <= 96 * 1024


def direct_fast(k, dil, cin, cout):
    """train.cu, direct_fast3: wgrad_direct3x3_kernel (the border condition holds for every 'same' 3x3 layer)."""
    return k == 3 and dil == 1 and cin == 3 and cout % 2 == 0 and cout <= 512


def layer_shapes(case):
    """{layer: dict(spec, cin, H, W (its input), Ho, Wo)} of a bcase's conv / head / pool / l2 layers (the geometry of _build)."""
    chans, shapes, out = {0: case['cin']}, {0: (case['H'], case['W'])}, {}
    for i, spec in enumerate(case['layers'], start=1):
        inp = i - 1 if spec['input'] is None else spec['input']
        cin, (H, W) = chans[inp], shapes[inp]
        if spec['op'] in ('conv', 'head', 'pool'):
            k, stride, dil = spec.get('k', 3), spec.get('stride', 1), spec.get('dil', 1)
            if spec['op'] == 'pool':
                pads = tuple(spec['pads'])
            elif spec['op'] == 'head' or spec['pads'] == 'same':
                q = dil * (k - 1) // 2
                pads = (q, q, q, q)
            else:
                pads = (0, 0, 0, 0) if spec['pads'] == 'valid' else tuple(spec['pads'])
            Ho = (H + pads[0] + pads[2] - dil * (k - 1) - 1) // stride + 1
            Wo = (W + pads[1] + pads[3] - dil * (k - 1) - 1) // stride + 1
        else:
            Ho, Wo = H, W
        cout = {'conv': spec.get('cout'), 'head': spec.get('nb', 0) * (case['C'] + 4)}.get(spec['op'], cin)
        chans[i], shapes[i] = cout, (Ho, Wo)
        out[i] = dict(spec=spec, input=inp, cin=cin, H=H, W=W, Ho=Ho, Wo=Wo, cout=cout)
    return out


def reach(case, sm_count=SM_COUNT_H100, training=True):
    """What each conv layer of a bcase launches -> {layer: dict(fwd=kernel, regimes=set, bn=bn_grid(...) or None,
    wgrad=(rows_per_block, grid, last rows, fast) or None)}."""
    out = {}
    for i, s in layer_shapes(case).items():
        spec = s['spec']
        if spec['op'] != 'conv':
            continue
        B, cin, cout, k, stride = case['B'], s['cin'], s['cout'], spec['k'], spec['stride']
        pixels = B * s['Ho'] * s['Wo']
        direct = s['input'] == 0 and selects_direct(cin, cout, k, stride)
        swap = not direct and selects_swap(cin, cout, stride, pixels, sm_count=sm_count)
        bn = spec['bn'] and training
        r = dict(fwd='direct' if direct else 'gemm_swap' if swap else 'other', regimes=set(), bn=None, wgrad=None)
        if bn:
            r['bn'] = bn_grid(B, s['Ho'], s['Wo'], cout, sm_count)
            if r['bn'][1] >= 2:
                r['regimes'].add(BN_STRIDED)
                if r['bn'][2]:
                    r['regimes'].add(BN_STRIDED_ODD)
        if training and swap:
            r['regimes'].add(SWAP_BN if bn else SWAP_RELU if spec['act'] == 'relu' else 'swap_train')
        if training and direct:
            r['wgrad'] = direct_wgrad_rows(B, s['Ho'], sm_count) + (direct_fast(k, spec['dil'], cin, cout),)
            if r['wgrad'][0] >= 2:
                r['regimes'].add(WGRAD_ROWS)
            if BN_STRIDED in r['regimes']:
                r['regimes'].add(DIRECT_BN)
        out[i] = r
    return out


def regimes(case, sm_count=SM_COUNT_H100, training=True):
    return set().union(*[r['regimes'] for r in reach(case, sm_count, training).values()])


# ------------------------------------------------------------------------------------------------------------------------------
# the cases
# ------------------------------------------------------------------------------------------------------------------------------
def rcase(name, B, H, W, cin, layers, fwd, regimes_, expect=None, prec='bf16x3', input_layer=None):
    c = bcase(name, B, H, W, cin, layers, expect or {}, prec=prec, input_layer=input_layer)
    c.update(fwd=fwd, regimes=set(regimes_))
    return c


SWAP2 = {1: 'gemm_swap', 2: 'gemm_swap'}
# the head's and layer 2's data gradients mask with the swap-written ReLU planes; layer 2's native weight gradient reads them
SWAP_RELU_EXPECT = {3: D(64, 1, 0), 2: dict(D(64, 1, 0), wgrad='native'), 1: dict(wgrad='native')}
MEAN_STD = dict(mean=(127.5, 127.5, 127.5), stddev=(127.5, 127.5, 127.5))

REGIME_CASES = [
    # --- conv_swap_kernel in training plans: 2 x 160 x 160 = 51200 output pixels >= 2 * 132 * 192 ---
    rcase('swap_train_relu', 2, 160, 160, 64, [conv(64, 3), conv(64, 3), head(1)], SWAP2, [SWAP_RELU], SWAP_RELU_EXPECT),
    rcase('bf16_swap_train_relu', 2, 160, 160, 64, [conv(64, 3), conv(64, 3), head(1)], SWAP2, [SWAP_RELU], SWAP_RELU_EXPECT,
          prec='bf16'),
    # ... into BatchNormalization (64 and 40 channels: a partial channel group), 8 and 5 groups at 2 elements per thread
    rcase('swap_train_bn_elu64_relu40', 2, 160, 160, 64, [conv(64, 3, act='elu', bn=True), conv(40, 3, bn=True), head(1)], SWAP2,
          [SWAP_BN, BN_STRIDED]),
    rcase('bf16_swap_train_bn_relu64_elu40', 2, 160, 160, 64, [conv(64, 3, bn=True), conv(40, 3, act='elu', bn=True), head(1)],
          SWAP2, [SWAP_BN, BN_STRIDED], prec='bf16'),
    # --- BatchNormalization over a strided grid ---
    # SSD7's conv1 at its notebook size: preprocessed image -> conv_direct_kernel 5x5, 3 -> 32, into z; 4 groups, 5 per thread
    rcase('ssd7_conv1_300x480', 2, 300, 480, 3, [conv(32, 5, act='elu', bn=True), head(1)], {1: 'direct'}, [BN_STRIDED, DIRECT_BN],
          {1: dict(wgrad='direct', direct_fast=0)}, input_layer=MEAN_STD),
    # 6 groups, 7 per thread
    rcase('bf16_bn_c48_300x480', 2, 300, 480, 8, [conv(48, 3, bn=True), head(1)], {}, [BN_STRIDED], prec='bf16'),
    # 17 groups: 1054 blocks (a multiple of 17), 5 per thread
    rcase('bn_c136_cut_grid_150x240', 2, 150, 240, 16, [conv(136, 3, act=None, bn=True), head(1)], {}, [BN_STRIDED, BN_STRIDED_ODD]),
    # --- direct weight gradients with several rows per block (narrow maps keep the references cheap) ---
    # 1101 rows: 2 per block, the last block holds one
    rcase('direct3x3_rows2_last1', 3, 367, 16, 3, [conv(64, 3), head(1)], {1: 'direct'}, [WGRAD_ROWS],
          {1: dict(wgrad='direct', direct_fast=1)}),
    # SSD7 conv1's kernel (generic): 2200 rows, 3 per block
    rcase('direct5x5_rows3', 2, 1100, 16, 3, [conv(32, 5), head(1)], {1: 'direct'}, [WGRAD_ROWS],
          {1: dict(wgrad='direct', direct_fast=0)}),
    rcase('bf16_direct3x3_dil2_cin4_rows2', 1, 1200, 20, 4, [conv(48, 3, dil=2), head(1)], {1: 'direct'}, [WGRAD_ROWS],
          {1: dict(wgrad='direct', direct_fast=0)}, prec='bf16'),
    # 4400 rows: 5 per block
    rcase('bf16_direct3x3_rows5', 4, 1100, 16, 3, [conv(64, 3), head(1)], {1: 'direct'}, [WGRAD_ROWS],
          {1: dict(wgrad='direct', direct_fast=1)}, prec='bf16'),
]
