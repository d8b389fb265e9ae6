"""The benchmark's inference plans, as bench.py builds them, and the size rules that decide which launch regime each of their
layers reaches, mirrored from the C++ so that a CPU test can check which regimes the configurations reach
(tests/test_bench_plan_regimes_cpu.py) and the GPU test can assert the device's plans against them
(tests/test_gpu_bench_plans.py).

The per-launch case tables (tests/conv_cases.py, tests/test_gpu_train_step_kernels.py) run graphs of a few hundred pixels
and a few dozen channels.  These regimes only full-size inference plans reach:
- l2norm8_kernel above 256 channels: the second register half (conv4_3_norm, C = 512);
- head_finalize_kernel with three lane passes per row (SSD512's unfused 81-class heads);
- the fused head epilogue at a non-zero prior offset (every head after the first);
- long K loops: 64 and more k-blocks on one accumulator (3x3 convolutions over 512 channels, conv6_2's im2col GEMM);
- full 256-wide tiles picked by the wave rule of plan_conv_gemm (single-pass bf16, cout % 128 == 0);
- persistent grids whose CTAs run several tiles (at least two waves);
- the folded BatchNormalization scale / shift and ELU in the epilogues of the image-facing and GEMM convolutions (SSD7).
"""
import numpy as np

from conv_cases import SM_COUNT_H100
from swap_cases import selects_swap

SC300 = [0.1, 0.2, 0.37, 0.54, 0.71, 0.88, 1.05]
SC512 = [0.04, 0.1, 0.26, 0.42, 0.58, 0.74, 0.9, 1.06]
SC7 = [0.08, 0.16, 0.32, 0.64, 0.96]
STDDEV = [127.5, 127.5, 127.5]          # bench.py's divide_by_stddev
SWAP_BM = 192                           # conv_swap_bm(): pixels per conv_swap_kernel tile

L2_UPPER = 'l2norm8_upper_half'         # l2norm8_kernel over more than 256 channels
HEAD_UNFUSED_WIDE = 'head_finalize_c_gt_64'   # the unfused head path with more than 64 classes (three lane passes)
HEAD_FUSED_OFFSET = 'head_fused_prior_offset'  # the fused head epilogue writing y_pred rows from a non-zero prior offset
LONG_K = 'gemm_kblocks_ge_64'           # a GEMM tile with at least 64 k-blocks on its accumulator
WIDE_256 = 'gemm_bn256_wave_rule'       # a 256-wide tile the wave rule kept (cout % 128 == 0)
MULTI_WAVE = 'gemm_multi_wave'          # a persistent grid with at least two tiles per CTA
BN_EPILOGUE = 'folded_bn_elu'           # folded BatchNormalization + ELU in a convolution's epilogue
REGIMES = (L2_UPPER, HEAD_UNFUSED_WIDE, HEAD_FUSED_OFFSET, LONG_K, WIDE_256, MULTI_WAVE, BN_EPILOGUE)


def config(name, family, B, n_classes, mode, prec, judged, size, **pre):
    return dict(name=name, family=family, B=B, n_classes=n_classes, mode=mode, prec=prec, judged=tuple(judged), size=size, pre=pre)


# judged images: the first, one in the middle and the last (which holds the final partial m-tile); the m-tiles of the implicit
# GEMMs straddle image boundaries at a different position in each image
CONFIGS = [
    config('ssd300_b32_bf16x3', 'ssd300', 32, 20, 'inference', 'bf16x3', (0, 16, 31), 300, divide_by_stddev=STDDEV),
    config('ssd300_b32_bf16', 'ssd300', 32, 20, 'inference', 'bf16', (0, 16, 31), 300, divide_by_stddev=STDDEV),
    config('ssd512_b16_bf16x3', 'ssd512', 16, 80, 'inference_fast', 'bf16x3', (0, 15), 512, divide_by_stddev=STDDEV),
    # BASELINE config 0 on normalised pixels: raw 0..255 pixels drive the logits into the hundreds, where fp32 exp underflows
    # and a relative probability bound cannot hold
    config('ssd7_b1_bf16x3', 'ssd7', 1, 5, 'inference', 'bf16x3', (0,), 300, subtract_mean=127.5, divide_by_stddev=127.5),
]

# the regimes each configuration must reach on an H100 SXM (132 SMs)
EXPECTED = {
    'ssd300_b32_bf16x3': {L2_UPPER, HEAD_FUSED_OFFSET, LONG_K, MULTI_WAVE},
    'ssd300_b32_bf16': {L2_UPPER, HEAD_FUSED_OFFSET, LONG_K, MULTI_WAVE, WIDE_256},
    'ssd512_b16_bf16x3': {L2_UPPER, HEAD_UNFUSED_WIDE, LONG_K, MULTI_WAVE},
    'ssd7_b1_bf16x3': {HEAD_FUSED_OFFSET, BN_EPILOGUE},
}


def build(cfg):
    """The model of a configuration, through the public builder as bench.py calls it."""
    if cfg['family'] == 'ssd300':
        from ssd_keras_b200.models.keras_ssd300 import ssd_300
        return ssd_300((300, 300, 3), cfg['n_classes'], mode=cfg['mode'], scales=SC300, precision=cfg['prec'], **cfg['pre'])
    if cfg['family'] == 'ssd512':
        from ssd_keras_b200.models.keras_ssd512 import ssd_512
        return ssd_512((512, 512, 3), cfg['n_classes'], mode=cfg['mode'], scales=SC512, precision=cfg['prec'], **cfg['pre'])
    from ssd_keras_b200.models.keras_ssd7 import build_model
    return build_model((300, 300, 3), cfg['n_classes'], mode=cfg['mode'], scales=SC7, normalize_coords=True,
                       precision=cfg['prec'], **cfg['pre'])


def weights(cfg, seed=7):
    """synth weights with non-zero biases; the L2Normalization gamma drawn per channel from U(5, 30); SSD7's BatchNormalization
    layers with random gamma, beta and moving statistics."""
    from oracle import synth
    from oracle.model import ssd7_weight_shapes, vgg_weight_shapes
    rng = np.random.default_rng(seed + 100)
    if cfg['family'] == 'ssd7':
        w = synth.synth_weights(seed, ssd7_weight_shapes(cfg['n_classes']), bias_scale=0.05)
        for i in range(1, 8):
            c = w['conv%d/bias' % i].shape[0]
            w['bn%d/gamma' % i] = rng.uniform(0.8, 1.2, c).astype(np.float32)
            w['bn%d/beta' % i] = (rng.standard_normal(c) * 0.1).astype(np.float32)
            w['bn%d/moving_mean' % i] = (rng.standard_normal(c) * 0.1).astype(np.float32)
            w['bn%d/moving_variance' % i] = rng.uniform(0.5, 1.5, c).astype(np.float32)
        return w
    w = synth.synth_weights(seed, vgg_weight_shapes(cfg['size'], cfg['n_classes']), bias_scale=0.05)
    w['conv4_3_norm/gamma'] = rng.uniform(5.0, 30.0, 512).astype(np.float32)
    return w


def folded_bn(w, bn):
    """The float32 scale and shift the model hands the plan for a folded BatchNormalization(eps=1e-3) (models/_graph.py)."""
    g, b = w[bn + '/gamma'], w[bn + '/beta']
    mu, var = w[bn + '/moving_mean'], w[bn + '/moving_variance']
    scale = g.astype(np.float64) / np.sqrt(var.astype(np.float64) + 1e-3)
    return scale.astype(np.float32), (b - mu * scale).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------------------------
# the size rules of an inference plan
# ------------------------------------------------------------------------------------------------------------------------------
def first_tc_supported(taps, cin, cout):
    """conv.cu, first_tc_supported."""
    return cin <= 4 and taps * 4 <= 128 and cout % 8 == 0 and cout <= 128


def conv_kernel(head, cin, cout, k, stride, dil, pixels, sm_count=SM_COUNT_H100):
    """model.cu, conv_kernel, for an inference plan."""
    taps = k * k
    if not head and 1 <= cin <= 4 and stride == 1 and cout % 16 == 0 and taps * cin * cout * 4 <= 96 * 1024:
        return 'first_tc' if first_tc_supported(taps, cin, cout) and dil >= 1 else 'direct'
    if stride != 1 or cin < 8:
        return 'im2col_gemm'
    if selects_swap(cin, cout, stride, pixels, head=head, sm_count=sm_count):
        return 'gemm_swap'
    return 'gemm'


def gemm_bn(cout, split, n_valid, sm_count=SM_COUNT_H100):
    """model.cu, plan_conv_gemm: the tile width.  bf16x3 tiles carry the cross-term accumulator (at most 160 columns); a
    single-pass cout % 128 == 0 layer keeps 256-wide tiles unless 128-wide ones need fewer tile-columns per SM over all waves."""
    bn = 64 if cout <= 64 else 128 if cout <= 128 else 256
    if split and bn == 256:
        return 160 if cout <= 160 else 128
    if bn == 256 and cout % 128 == 0:
        u256, u128 = n_valid * -(-cout // 256), n_valid * -(-cout // 128)
        if -(-u128 // sm_count) * 128 < -(-u256 // sm_count) * 256:
            return 128
    return bn


def valid_tiles(B, Hp, Wp, Ho, Wo, bm):
    """model.cu, plan_conv_gemm: the bm-row tiles of the stored (B, Hp, Wp) grid that hold at least one valid output pixel (an
    output (y, x) is row y * Wp + x of its image)."""
    rows = np.arange(B * Hp * Wp) % (Hp * Wp)
    ok = (rows // Wp < Ho) & (rows % Wp < Wo)
    tiles = np.zeros(-(-ok.size // bm), bool)
    np.logical_or.at(tiles, np.arange(ok.size) // bm, ok)
    return int(tiles.sum())


def l2norm_kernel_of(C):
    """conv.cu, launch_l2norm: l2norm8_kernel when the channels fill whole 8-channel groups up to 512 (the planes store
    ceil(C / 8) * 8 channels; gamma is a 16-byte aligned device array)."""
    return 'l2norm8' if C % 8 == 0 and C <= 512 else 'l2norm'


def pool_kernel_of(H, W, k, stride, pads):
    """conv.cu, launch_maxpool."""
    Ho, Wo = (H + pads[0] + pads[2] - k) // stride + 1, (W + pads[1] + pads[3] - k) // stride + 1
    fast = k == 2 and stride == 2 and pads[0] == 0 and pads[1] == 0 and 2 * (Ho - 1) < H and 2 * (Wo - 1) < W
    return 'maxpool2x2' if fast else 'maxpool'


def layers(model, B, sm_count=SM_COUNT_H100):
    """The inference plan of a model at batch B, mirrored: [dict(name, op, input, H, W, C (output), ...)] in plan order, with
    for every conv / head its kernel and, for the GEMMs, kblocks, bn, bm, n_tiles_m, n_tiles_n, head_fused, prior_off; for
    every pool and L2Normalization its kernel; and the stored planes' border (pad, Hp, Wp) of every layer with planes."""
    from ssd_keras_b200 import _ffi
    split = model.precision == 'bf16x3'
    out = []
    for i, s in enumerate(model.specs):
        H, W, C = model._shapes[i]
        L = dict(name=s.name, op={_ffi.OP_INPUT: 'input', _ffi.OP_CONV: 'conv', _ffi.OP_HEAD: 'head', _ffi.OP_MAXPOOL: 'pool',
                                  _ffi.OP_L2NORM: 'l2'}[s.op], input=model.index[s.inp] if s.inp is not None else None,
                 H=H, W=W, C=C, k=s.kh, stride=s.stride, dil=s.dilation, pads=tuple(s.pad), n_boxes=s.n_boxes, bn_layer=s.bn,
                 act={_ffi.ACT_NONE: None, _ffi.ACT_RELU: 'relu', _ffi.ACT_ELU: 'elu'}[s.act], pad=0)
        if L['op'] in ('conv', 'head'):
            cin = model._shapes[L['input']][2]
            L['cin'] = cin
            L['kernel'] = conv_kernel(L['op'] == 'head', cin, C, s.kh, s.stride, s.dilation, B * H * W, sm_count)
        out.append(L)
    # pass 2 of ssdk_model_create: the border each consumer reads from its input's planes
    for L in out:
        if L['op'] not in ('conv', 'head'):
            continue
        src = out[L['input']]
        pt, pl, pb, pr = L['pads']
        if L['kernel'] in ('gemm', 'gemm_swap'):
            src['pad'] = max(src['pad'], pt, pl, pb, pr)
        elif L['kernel'] == 'first_tc':
            src['pad'] = max(src['pad'], pt, pl, (L['k'] - 1) * L['dil'] - pt, (L['k'] - 1) * L['dil'] - pl)
    for L in out:
        L['Hp'], L['Wp'] = L['H'] + 2 * L['pad'], L['W'] + L['pad']           # inference plans share the left / right border
    prior_off = 0
    for L in out:
        src = out[L['input']] if L['input'] is not None else None
        if L['op'] == 'pool':
            L['kernel'] = pool_kernel_of(src['H'], src['W'], L['k'], L['stride'], L['pads'])
        elif L['op'] == 'l2':
            L['kernel'] = l2norm_kernel_of(L['C'])
        elif L['op'] in ('conv', 'head'):
            if L['op'] == 'head':
                L['prior_off'] = prior_off
                prior_off += L['H'] * L['W'] * L['n_boxes']
            taps, cin = L['k'] ** 2, L['cin']
            if L['kernel'] == 'first_tc':
                L.update(bn=64 if L['C'] <= 64 else 128, kblocks=-(-taps * 4 // 64), split=int(split), kblocks_per_tile=-(-taps * 4 // 64),
                         n_tiles_m=-(-B * L['H'] * L['W'] // 128), n_tiles_n=1)
                continue
            if L['kernel'] == 'im2col_gemm':
                kb = -(-(-(-taps * cin // 8) * 8) // 64)
                L['n_tiles_m'] = -(-B * L['H'] * L['W'] // 128)
                L['kblocks_per_tile'] = kb
            else:
                kb = -(-(-(-cin // 8) * 8) // 64)
                L['n_tiles_m'] = valid_tiles(B, src['Hp'], src['Wp'], L['H'], L['W'], SWAP_BM if L['kernel'] == 'gemm_swap' else 128)
                L['kblocks_per_tile'] = taps * kb
            L['kblocks'] = kb
            L['bm'] = SWAP_BM if L['kernel'] == 'gemm_swap' else 128
            L['bn'] = gemm_bn(L['C'], split, L['n_tiles_m'], sm_count)
            L['n_tiles_n'] = -(-L['C'] // L['bn'])
            L['split'] = int(split)
            L['grid'] = max(1, min(L['n_tiles_m'] * L['n_tiles_n'], sm_count))
            if L['op'] == 'head':
                L['head_fused'] = int(L['n_tiles_n'] == 1)
    return out


def regimes_of(L, n_classes_total, sm_count=SM_COUNT_H100):
    """The regimes one mirrored layer reaches."""
    r = set()
    if L['op'] == 'l2' and L['kernel'] == 'l2norm8' and L['C'] > 256:
        r.add(L2_UPPER)
    if L['op'] == 'head' and not L['head_fused'] and n_classes_total > 64:
        r.add(HEAD_UNFUSED_WIDE)
    if L['op'] == 'head' and L['head_fused'] and L['prior_off'] > 0:
        r.add(HEAD_FUSED_OFFSET)
    if L.get('kernel') in ('gemm', 'gemm_swap', 'im2col_gemm'):
        if L['kblocks_per_tile'] >= 64:
            r.add(LONG_K)
        if L['bn'] == 256 and L['C'] % 128 == 0 and L['n_tiles_n'] * 256 == L['C'] and not L['split']:
            r.add(WIDE_256)
        if L['n_tiles_m'] * L['n_tiles_n'] >= 2 * sm_count:
            r.add(MULTI_WAVE)
    if L['op'] == 'conv' and L['bn_layer'] and L['act'] == 'elu':
        r.add(BN_EPILOGUE)
    return r


def regimes(model, B, sm_count=SM_COUNT_H100):
    return set().union(*[regimes_of(L, model.n_classes, sm_count) for L in layers(model, B, sm_count)])
