"""Case tables and the GPU harness of the convolution tests (tests/test_gpu_ops.py, tests/test_gpu_conv_heads.py,
tests/test_gpu_backward_kernels.py, tests/test_gpu_train_step_kernels.py).

Every case is a small graph described to ssdk_model_create directly: a float32 tensor input (any channel count) and the layer
under test.  The tables are plain data, so that a CPU test can check that together they reach every kernel variant the plan
builder can choose.  ``expect`` is the part of ssdk_model_layer_plan each case asserts on the device.
"""
import ctypes as C
import json
import os

import numpy as np

from oracle import opexact

SM_COUNT_H100 = 132


def conv_case(name, B, H, W, cin, cout, k, expect, stride=1, dil=1, pads='same', act='relu', bias=True, bn=False,
              prec='bf16x3', env=None, persistent=None):
    """persistent: None, or 'nk<stages' / 'nk%stages' -- the launch must give every CTA at least 3 tiles, with a K loop shorter
    than the TMA ring or one that does not divide it."""
    if pads == 'same':
        p = dil * (k - 1) // 2
        pads = (p, p, p, p)
    elif pads == 'valid':
        pads = (0, 0, 0, 0)
    return dict(name=name, B=B, H=H, W=W, cin=cin, cout=cout, k=k, stride=stride, dil=dil, pads=tuple(pads), act=act, bias=bias,
                bn=bn, prec=prec, env=env or {}, persistent=persistent, expect=expect)


def G(bn, **kw):
    return dict(kernel='gemm', bn=bn, **kw)


def F(bn, kblocks, split):
    return dict(kernel='first_tc', bn=bn, kblocks=kblocks, split=split)


FORWARD_CASES = [
    # --- conv_wgmma_kernel, bf16x3 (BN 64 / 128 / 160) ---
    conv_case('vgg_bn128_bias_relu', 2, 19, 23, 64, 128, 3, G(128, split=1, epilogue='split')),
    conv_case('bn64_1x1_linear_nobias', 1, 10, 12, 16, 32, 1, G(64, split=1), pads='valid', act=None, bias=False),
    conv_case('bn64_cin24_linear', 1, 9, 9, 24, 40, 3, G(64, split=1), act=None),
    conv_case('bn64_cin8_elu', 2, 11, 13, 8, 48, 3, G(64, split=1), act='elu'),
    conv_case('bn128_fc6_dil6', 1, 19, 19, 64, 256, 3, G(128, split=1, n_tiles_n=2), dil=6),
    conv_case('bn128_valid3x3_elu', 1, 7, 7, 128, 256, 3, G(128, split=1, n_tiles_n=2), pads='valid', act='elu'),
    conv_case('bn128_partial_264', 1, 8, 9, 64, 264, 3, G(128, split=1, n_tiles_n=3)),
    conv_case('bn160_cin72_partial_136', 2, 12, 14, 72, 136, 3, G(160, split=1, n_tiles_n=1)),
    conv_case('bn160_cin136_linear', 1, 10, 11, 136, 144, 3, G(160, split=1, kblocks=3), act=None),
    conv_case('bn64_valid4x4', 2, 9, 9, 64, 64, 4, G(64, split=1), pads='valid'),
    conv_case('bn64_pad_0022_shared', 2, 10, 10, 64, 64, 3, G(64, split=1), pads=(0, 0, 2, 2)),
    conv_case('bn64_pad_2200_shared', 2, 10, 10, 64, 64, 3, G(64, split=1), pads=(2, 2, 0, 0)),
    conv_case('bn64_pad_0022_unshared', 2, 10, 10, 64, 64, 3, G(64, split=1), pads=(0, 0, 2, 2), env={'SSDK_SHARED_BORDER': '0'}),
    conv_case('bn64_pad_2200_unshared', 2, 10, 10, 64, 64, 3, G(64, split=1), pads=(2, 2, 0, 0), env={'SSDK_SHARED_BORDER': '0'}),
    conv_case('bn64_folded_batchnorm', 2, 10, 10, 32, 64, 3, G(64, split=1), bn=True),
    conv_case('bn160_folded_batchnorm_elu', 1, 9, 10, 64, 152, 3, G(160, split=1), bn=True, act='elu'),
    conv_case('persistent_1x1_nk_lt_stages', 8, 80, 80, 32, 64, 1, G(64, split=1), pads='valid', persistent='nk<stages'),
    conv_case('persistent_3x3_nk_mod_stages', 8, 80, 80, 8, 64, 3, G(64, split=1), persistent='nk%stages'),
    # --- im2col + conv_wgmma_kernel ---
    conv_case('stride2_im2col8', 2, 19, 19, 32, 64, 3, dict(kernel='im2col_gemm', bn=64, im2col_vec8=1), stride=2, pads=(1, 1, 1, 1)),
    conv_case('cin3_im2col_generic', 2, 14, 13, 3, 40, 3, dict(kernel='im2col_gemm', bn=64, im2col_vec8=0)),
    # --- conv_wgmma_kernel, single-pass bf16 (BN 64 / 128 / 256) ---
    conv_case('bf16_bn64', 2, 12, 12, 64, 64, 3, G(64, split=0), prec='bf16'),
    conv_case('bf16_bn128_dil2', 1, 14, 15, 72, 128, 3, G(128, split=0), dil=2, prec='bf16'),
    conv_case('bf16_bn256_partial_264', 1, 9, 8, 64, 264, 3, G(256, split=0, n_tiles_n=2), prec='bf16', act=None),
    conv_case('bf16_persistent_3x3', 8, 80, 80, 8, 64, 3, G(64, split=0), prec='bf16', persistent='nk%stages'),
    # --- conv_first_kernel: {BN 64, 128} x {1, 2 k-blocks} x {split, single}, 1 ... 4 input channels ---
    conv_case('first_bn64_kb1_split_cin3', 2, 20, 20, 3, 64, 3, F(64, 1, 1)),
    conv_case('first_bn64_kb1_single_cin1_dil2', 2, 17, 18, 1, 64, 3, F(64, 1, 0), dil=2, prec='bf16'),
    conv_case('first_bn64_kb2_split_cin4', 2, 16, 15, 4, 64, 5, F(64, 2, 1)),
    conv_case('first_bn64_kb2_single_cin3', 1, 18, 16, 3, 32, 5, F(64, 2, 0), prec='bf16', act=None),
    conv_case('first_bn128_kb1_split_cin4', 2, 15, 17, 4, 80, 3, F(128, 1, 1), act='elu'),
    conv_case('first_bn128_kb1_single_cin2', 1, 16, 16, 2, 128, 3, F(128, 1, 0), prec='bf16'),
    conv_case('first_bn128_kb2_split_cin3', 2, 14, 14, 3, 96, 5, F(128, 2, 1)),
    conv_case('first_bn128_kb2_single_cin2_dil2', 1, 19, 17, 2, 112, 5, F(128, 2, 0), dil=2, prec='bf16'),
    # --- conv_direct_kernel: an image-facing layer wider than conv_first_kernel's 128 columns ---
    conv_case('direct_cin3_cout144', 2, 13, 15, 3, 144, 3, dict(kernel='direct')),
]


def head_case(name, B, H, W, cin, nb, C, expect, prec='bf16x3', env=None):
    return dict(name=name, B=B, H=H, W=W, cin=cin, nb=nb, C=C, prec=prec, env=env or {}, expect=expect)


def HF(bn, split, fused=1, **kw):
    return dict(kernel='gemm', bn=bn, split=split, epilogue='head' if fused else 'f32', head_fused=fused, **kw)


HEAD_CASES = [
    # fused epilogue, compile-time 25-column boxes (Pascal VOC: 21 classes + 4 offsets), epi_head_fixed<25>
    head_case('fixed25_4boxes_bn128', 2, 10, 9, 64, 4, 21, HF(128, 1)),
    head_case('fixed25_6boxes_bn160', 2, 8, 11, 72, 6, 21, HF(160, 1)),
    head_case('fixed25_8boxes_bn256_bf16', 2, 9, 9, 64, 8, 21, HF(256, 0), prec='bf16'),
    # fused epilogue, run-time box width
    head_case('generic_6classes', 2, 10, 10, 64, 3, 6, HF(64, 1)),
    head_case('generic_81classes_bf16', 1, 7, 8, 64, 3, 81, HF(256, 0), prec='bf16'),
    # unfused: fp32 logits, then head_finalize_kernel
    head_case('unfused_no_head_fusion', 2, 10, 9, 64, 4, 21, HF(128, 1, fused=0), env={'SSDK_NO_HEAD_FUSION': '1'}),
    head_case('unfused_8boxes_bf16x3', 2, 6, 7, 136, 8, 21, HF(128, 1, fused=0, n_tiles_n=2)),
]


# ------------------------------------------------------------------------------------------------------------------------------
# the GPU harness
# ------------------------------------------------------------------------------------------------------------------------------
ACTS = {None: 0, 'relu': 1, 'elu': 2}


def log_ratio(record):
    """Append one JSON line to the file named by SSDK_KERNEL_ERRORS_LOG, if set: the measured |err| / bound of a case and of
    each perturbed reference.  For example
        SSDK_KERNEL_ERRORS_LOG=/tmp/kernel_errors.jsonl python -m pytest -m gpu tests/test_gpu_ops.py tests/test_gpu_conv_heads.py
    (a plain run writes nothing into the tree)."""
    path = os.environ.get('SSDK_KERNEL_ERRORS_LOG')
    if path:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, 'a') as f:
            f.write(json.dumps(record) + '\n')


class Graph:
    """A tensor input plus conv / head layers, planned by ssdk_model_create (inference plan)."""

    def __init__(self, B, H, W, cin, layers, prec='bf16x3', n_classes=0, anchors=None, variances=(0.1, 0.1, 0.2, 0.2),
                 training=False, input_layer=None):
        """input_layer: None (a float32 tensor input), or dict(mean=, stddev=, swap=) of a model input layer (preprocess_kernel;
        each entry may be None)."""
        from ssd_keras_b200 import _ffi
        self.B, self.H, self.W, self.cin = B, H, W, cin
        self._keep = []
        n = 1 + len(layers)
        descs = (_ffi.LayerDesc * n)()
        descs[0].op, descs[0].input = _ffi.OP_TENSOR, -1

        def fptr(a):
            a = np.ascontiguousarray(a, dtype=np.float32)
            self._keep.append(a)
            return _ffi.np_ptr(a, C.c_float)

        if input_layer is not None:
            descs[0].op = _ffi.OP_INPUT
            if input_layer.get('mean') is not None:
                descs[0].mean = fptr(input_layer['mean'])
            if input_layer.get('stddev') is not None:
                descs[0].stddev = fptr(input_layer['stddev'])
            if input_layer.get('swap') is not None:
                sw = np.ascontiguousarray(input_layer['swap'], dtype=np.int32)
                self._keep.append(sw)
                descs[0].swap = _ffi.np_ptr(sw, C.c_int)

        for i, L in enumerate(layers, start=1):
            d = descs[i]
            d.op = L.get('op', _ffi.OP_CONV)
            d.input = L.get('input', i - 1)
            d.cout, d.kh, d.kw = L.get('cout', 0), L.get('k', 0), L.get('k', 0)
            d.stride, d.dilation = L.get('stride', 1), L.get('dil', 1)
            d.pad_t, d.pad_l, d.pad_b, d.pad_r = L.get('pads', (0, 0, 0, 0))
            d.act, d.n_boxes = ACTS[L.get('act')], L.get('n_boxes', 0)
            if L.get('kernel') is not None:                   # conv / head kernel, or an L2Normalization's gamma
                d.kernel = fptr(L['kernel'])
            if L.get('bias') is not None:
                d.bias = fptr(L['bias'])
            if L.get('kernel2') is not None:
                d.kernel2, d.bias2 = fptr(L['kernel2']), fptr(L['bias2'])
            if L.get('bn_scale') is not None:
                d.bn_scale, d.bn_shift = fptr(L['bn_scale']), fptr(L['bn_shift'])
            if L.get('bn_gamma') is not None:                 # raw BatchNormalization parameters (training plans: bn_train)
                d.bn_gamma, d.bn_beta = fptr(L['bn_gamma']), fptr(L['bn_beta'])
                d.bn_mean, d.bn_var = fptr(L['bn_mean']), fptr(L['bn_var'])
                d.bn_eps, d.bn_momentum = L.get('bn_eps', 1e-3), L.get('bn_momentum', 0.99)
        anc = fptr(anchors if anchors is not None else np.zeros(4, np.float32))
        md = _ffi.ModelDesc(B, H, W, cin, n_classes, n, descs, 0 if prec == 'bf16x3' else 1, anc,
                            (C.c_float * 4)(*[float(v) for v in variances]), 1 if training else 0)
        self.h = C.c_void_p()
        self.t = None
        _ffi.check(_ffi.lib().ssdk_model_create(_ffi.context(), C.byref(md), C.byref(self.h)))
        self.split = prec == 'bf16x3'
        self.grad_layers = list(range(1, n))                   # every layer but the tensor input has gradient planes
        P = C.c_int()
        _ffi.check(_ffi.lib().ssdk_model_num_priors(self.h, C.byref(P)))
        self.P = P.value

    def plan(self, layer):
        from ssd_keras_b200 import _ffi
        return _ffi.model_layer_plan(self.h, layer)

    def backward_plan(self, layer):
        """The trainer's backward plan of a layer (training graphs; the trainer is created on first use)."""
        from ssd_keras_b200 import _ffi
        self.trainer()
        return _ffi.trainer_layer_plan(self.t, layer)

    def trainer(self):
        """The trainer of a training graph, created on first use over a flat gradient buffer the test owns (self.grad)."""
        from ssd_keras_b200 import _ffi
        if self.t is None:
            import torch
            L = _ffi.lib()
            t, n = C.c_void_p(), C.c_longlong()                # a first trainer sizes the flat gradient buffer the test owns
            _ffi.check(L.ssdk_trainer_create(self.h, None, C.byref(t)))
            _ffi.check(L.ssdk_trainer_num_params(t, C.byref(n)))
            L.ssdk_trainer_destroy(t)
            self.grad = torch.zeros(n.value, dtype=torch.float32, device='cuda')
            self.t = C.c_void_p()
            _ffi.check(L.ssdk_trainer_create(self.h, _ffi.dptr(self.grad), C.byref(self.t)))
        return self.t

    def apply(self, optimizer, lr, l2=0.0, scale=1.0, momentum=0.9, beta1=0.9, beta2=0.999, eps=1e-8, step=1):
        """One optimiser update from the flat gradient buffer (ssdk_train_apply / ssdk_train_apply_adam)."""
        import torch
        from ssd_keras_b200 import _ffi
        torch.cuda.synchronize()
        if optimizer == 'adam':
            _ffi.check(_ffi.lib().ssdk_train_apply_adam(self.trainer(), lr, beta1, beta2, eps, l2, scale, step, _ffi.stream_ptr()))
        else:
            _ffi.check(_ffi.lib().ssdk_train_apply(self.trainer(), lr, momentum, l2, scale, _ffi.stream_ptr()))
        torch.cuda.synchronize()

    def _flat(self, fn, *args):
        import torch
        from ssd_keras_b200 import _ffi
        out = torch.full_like(self.grad, float('nan'))
        _ffi.check(fn(self.trainer(), *args, _ffi.dptr(out), _ffi.stream_ptr()))
        torch.cuda.synchronize()
        return out.cpu().numpy()

    def params(self):
        """The float32 master parameters in the gradient's layout (ssdk_trainer_read_params)."""
        from ssd_keras_b200 import _ffi
        return self._flat(_ffi.lib().ssdk_trainer_read_params)

    def opt_state(self, slot):
        """One slot of the optimiser state in the gradient's layout (ssdk_trainer_read_opt_state): 0 = SGD velocity / Adam m,
        1 = Adam v."""
        from ssd_keras_b200 import _ffi
        return self._flat(_ffi.lib().ssdk_trainer_read_opt_state, int(slot))

    def bn_stats(self, layer, C_):
        """(moving mean, moving variance) of a BatchNormalization layer (ssdk_trainer_read_bn_stats)."""
        import torch
        from ssd_keras_b200 import _ffi
        mu = torch.empty((C_,), dtype=torch.float32, device='cuda')
        var = torch.empty_like(mu)
        _ffi.check(_ffi.lib().ssdk_trainer_read_bn_stats(self.trainer(), layer, _ffi.dptr(mu), _ffi.dptr(var), _ffi.stream_ptr()))
        torch.cuda.synchronize()
        return mu.cpu().numpy(), var.cpu().numpy()

    def planes(self, layer):
        """The raw forward activation planes of a layer -> (hi, lo, pad), uint16 (B, Hp, Wp, Cs), lo None in bf16 mode."""
        import torch
        from ssd_keras_b200 import _ffi
        hp, wp, cs, pad = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        _ffi.check(_ffi.lib().ssdk_model_layer_planes_shape(self.h, layer, C.byref(hp), C.byref(wp), C.byref(cs), C.byref(pad)))
        shape = (self.B, hp.value, wp.value, cs.value)
        hi = torch.empty(shape, dtype=torch.int16, device='cuda')
        lo = torch.empty(shape, dtype=torch.int16, device='cuda') if self.split else None
        _ffi.check(_ffi.lib().ssdk_model_read_layer_planes(self.h, layer, _ffi.dptr(hi), _ffi.dptr(lo), _ffi.stream_ptr()))
        torch.cuda.synchronize()
        return hi.cpu().numpy().view(np.uint16), (None if lo is None else lo.cpu().numpy().view(np.uint16)), pad.value

    def grad_planes(self, layer):
        """The raw gradient planes of a layer -> (hi, lo) uint16 arrays (B, Hp, Wp, Cs), lo None in bf16 mode, and the pad."""
        import torch
        from ssd_keras_b200 import _ffi
        hp, wp, cs, pad = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        _ffi.check(_ffi.lib().ssdk_trainer_grad_shape(self.t, layer, C.byref(hp), C.byref(wp), C.byref(cs), C.byref(pad)))
        shape = (self.B, hp.value, wp.value, cs.value)
        hi = torch.empty(shape, dtype=torch.int16, device='cuda')
        lo = torch.empty(shape, dtype=torch.int16, device='cuda') if self.split else None
        _ffi.check(_ffi.lib().ssdk_trainer_read_grad_planes(self.t, layer, _ffi.dptr(hi), _ffi.dptr(lo), _ffi.stream_ptr()))
        torch.cuda.synchronize()
        return hi.cpu().numpy().view(np.uint16), (None if lo is None else lo.cpu().numpy().view(np.uint16)), pad.value

    def read_grad(self, layer):
        """hi + lo of a layer's gradient as float32 (B,H,W,C) (ssdk_trainer_read_grad)."""
        import torch
        from ssd_keras_b200 import _ffi
        h, w, c = C.c_int(), C.c_int(), C.c_int()
        _ffi.check(_ffi.lib().ssdk_model_layer_shape(self.h, layer, C.byref(h), C.byref(w), C.byref(c)))
        out = torch.empty((self.B, h.value, w.value, c.value), dtype=torch.float32, device='cuda')
        _ffi.check(_ffi.lib().ssdk_trainer_read_grad(self.t, layer, _ffi.dptr(out), _ffi.stream_ptr()))
        torch.cuda.synchronize()
        return out.cpu().numpy()

    def read_bn_input(self, layer):
        """The raw convolution output z a BatchNormalization layer normalised (ssdk_trainer_read_bn_input)."""
        import torch
        from ssd_keras_b200 import _ffi
        h, w, c = C.c_int(), C.c_int(), C.c_int()
        _ffi.check(_ffi.lib().ssdk_model_layer_shape(self.h, layer, C.byref(h), C.byref(w), C.byref(c)))
        out = torch.empty((self.B, h.value, w.value, c.value), dtype=torch.float32, device='cuda')
        _ffi.check(_ffi.lib().ssdk_trainer_read_bn_input(self.t, layer, _ffi.dptr(out), _ffi.stream_ptr()))
        torch.cuda.synchronize()
        return out.cpu().numpy()

    def snapshot(self):
        """Every gradient buffer (raw planes) and the flat parameter gradient."""
        import torch
        torch.cuda.synchronize()
        planes = {i: self.grad_planes(i) for i in self.grad_layers}
        return planes, self.grad.cpu().numpy().copy()

    def step(self, layer, dy):
        """Run the backward launches of one layer (ssdk_train_backward_layers(t, dy, layer, layer)) -> (before, after) snapshots.
        A pass must start at the top layer and go down one layer per call."""
        import torch
        from ssd_keras_b200 import _ffi
        before = self.snapshot()
        _ffi.check(_ffi.lib().ssdk_train_backward_layers(self.t, _ffi.dptr(dy), layer, layer, _ffi.stream_ptr()))
        torch.cuda.synchronize()
        return before, self.snapshot()

    def forward(self, x, width=0):
        """x float32 (B,H,W,cin) -> y_pred (B,P,width) or None."""
        import torch
        from ssd_keras_b200 import _ffi
        xt = torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
        y = torch.zeros((self.B, max(self.P, 1), max(width, 1)), dtype=torch.float32, device='cuda')
        _ffi.check(_ffi.lib().ssdk_model_forward(self.h, _ffi.dptr(xt), _ffi.dptr(y) if self.P else None, _ffi.stream_ptr()))
        torch.cuda.synchronize()
        return y.cpu().numpy() if self.P else None

    def read(self, layer):
        import torch
        from ssd_keras_b200 import _ffi
        h, w, c = C.c_int(), C.c_int(), C.c_int()
        _ffi.check(_ffi.lib().ssdk_model_layer_shape(self.h, layer, C.byref(h), C.byref(w), C.byref(c)))
        out = torch.empty((self.B, h.value, w.value, c.value), dtype=torch.float32, device='cuda')
        _ffi.check(_ffi.lib().ssdk_model_read_layer(self.h, layer, _ffi.dptr(out), _ffi.stream_ptr()))
        torch.cuda.synchronize()
        return out.cpu().numpy()

    def close(self):
        from ssd_keras_b200 import _ffi
        if self.t:
            _ffi.lib().ssdk_trainer_destroy(self.t)
            self.t = None
        if self.h:
            _ffi.lib().ssdk_model_destroy(self.h)
            self.h = None


def case_data(case, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((case['B'], case['H'], case['W'], case['cin'])).astype(np.float32)
    k = case['k']
    w = (rng.standard_normal((k, k, case['cin'], case['cout'])) * np.sqrt(2.0 / (k * k * case['cin']))).astype(np.float32)
    b = (rng.standard_normal(case['cout']) * 0.1).astype(np.float32) if case['bias'] else None
    scale = shift = None
    if case['bn']:
        scale = rng.uniform(0.5, 1.5, case['cout']).astype(np.float32)
        shift = (rng.standard_normal(case['cout']) * 0.1).astype(np.float32)
    return x, w, b, scale, shift


def n_steps_of(plan, taps, cin):
    if plan['kernel'] in ('gemm', 'im2col_gemm'):
        return opexact.n_steps_gemm(taps if plan['kernel'] == 'gemm' else 1, plan['kblocks'])
    if plan['kernel'] == 'first_tc':
        return opexact.n_steps_first(plan['kblocks'], plan['split'])
    return opexact.n_steps_direct(taps, cin)


def perturbations(plan, taps, cin, split_products, bias):
    """The perturbed references every comparison must reject: a dropped cross term, the middle tap, the last of the kernel's
    own 64-column K blocks (of the middle tap for the implicit GEMM; of the im2col row; 16 taps x 4 channels for
    conv_first_kernel, where a single block is the whole K and is left out), and the largest bias."""
    out = [('cross',)] if split_products else []
    out.append(('tap', taps // 2))
    if plan['kernel'] == 'first_tc':
        if plan['kblocks'] > 1:
            out.append(('taps', 16 * (plan['kblocks'] - 1), 16 * plan['kblocks']))
    elif plan['kernel'] == 'im2col_gemm':
        k_last = 64 * ((taps * cin - 1) // 64)
        out.append(('kcols', k_last, k_last + 64))
    else:
        out.append(('kblock', taps // 2, (cin - 1) // 64))
    if bias is not None:
        out.append(('bias', int(np.argmax(np.abs(bias)))))
    return out


def assert_plan(plan, expect, name):
    for key, v in expect.items():
        assert plan[key] == v, '%s: plan %s = %r, expected %r (full plan %r)' % (name, key, plan[key], v, plan)


def plane_values(planes):
    """(hi, lo, pad) raw planes -> (hi, lo) float32 arrays of the whole padded grid (lo None stays None)."""
    hi, lo, _ = planes
    return opexact.bf16_bits_to_f32(hi), (None if lo is None else opexact.bf16_bits_to_f32(lo))


def interior(planes, H, W, C_):
    """The (B,H,W,C) values of raw planes -> (hi, lo) float32, lo None in bf16 mode."""
    hi, lo = plane_values(planes)
    pad = planes[2]
    cut = (slice(None), slice(pad, pad + H), slice(pad, pad + W), slice(0, C_))
    return hi[cut], (None if lo is None else lo[cut])


def outside(planes, H, W, C_):
    """The stored values outside the (B,H,W,C) interior: zero border and padding channels, both planes."""
    pad = planes[2]
    keep = np.ones(planes[0].shape, bool)
    keep[:, pad:pad + H, pad:pad + W, :C_] = False
    return [p[keep] for p in planes[:2] if p is not None]
