"""GPU tests of the benchmark's inference plans (tests/bench_plan_cases.py), layer by layer, against the operand-exact float64
references of oracle/opexact.py.

Each configuration runs one forward_device on its full batch -- the call bench.py times, with the two-stream schedule on.
Every conv / head plan (ssdk_model_layer_plan) must be the one the mirrored size rules give for the device's SM count.  The
plan query has no entry for the max-pools and L2Normalization, so their kernel choice (maxpool2x2_kernel or maxpool_kernel,
l2norm8_kernel or l2norm_kernel) is mirrored but not read back from the device: the CPU test holds the mirrors to the
per-launch tables, and here only the outputs are judged (the two max-pool kernels are bit-identical by construction).  Then
every layer is judged on the selected images, from the planes the launch actually read (ssdk_model_read_layer_planes):
- the input preprocessing bit-exact (preprocess_ref); max-pools bit-exact on both planes (pool_fwd_ref);
- convolutions against conv_ref with the plan's own k-step count (image-facing: n_steps_first; GEMMs: n_steps_gemm of the
  plan's k-blocks), SSD7's with the folded BatchNormalization scale / shift and ELU;
- conv4_3_norm against l2norm_fwd_ref with its per-channel gamma;
- fused heads: that head's rows of y_pred, probabilities with softmax_ref's bound, offsets with the conv bound, anchors and
  variances bit-exact; unfused heads: the stored fp32 logits with the conv bound, then head_finalize_kernel's rows from
  those logits with the softmax bound;
- the zero border and the padding channels of every output plane.
Perturbed references must fail: per conv a dropped cross term (bf16x3), the middle tap, the middle tap's last k-block, the
largest bias of a channel the ReLU does not zero on every judged pixel; per L2Normalization no gamma and a gamma taken from
the next channel at channels 256 and 511; per head the rows shifted by one prior and two classes swapped.  The middle tap is
the kernel's centre tap (kh, kw) = (k // 2, k // 2): SSD512's 4x4 conv10_2 sees only padding through tap 8 = (2, 0).  For
SSD300 at batch 32 the decoded (32, 200, 6) output must equal oracle.decoder.decode_layer of the same y_pred.  Ratios go to
SSDK_KERNEL_ERRORS_LOG (conv_cases.log_ratio)."""
import os
import time

import numpy as np
import pytest

import bench_plan_cases as bp
import conv_cases as cc
from oracle import opexact

pytestmark = pytest.mark.gpu

PLAN_KEYS = {'first_tc': ('bn', 'kblocks', 'split', 'n_tiles_m', 'n_tiles_n'),
             'gemm': ('bn', 'bm', 'kblocks', 'split', 'n_tiles_m', 'n_tiles_n', 'grid'),
             'im2col_gemm': ('bn', 'bm', 'kblocks', 'split', 'n_tiles_m', 'n_tiles_n', 'grid')}
PLAN_KEYS['gemm_swap'] = PLAN_KEYS['gemm']


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


class _Planes:
    """Reads a layer's stored planes, or a head's fp32 output, of the selected images of a model plan."""

    def __init__(self, handle, B, split, sel):
        import torch
        self.h, self.B, self.split = handle, B, split
        self.sel = torch.tensor(list(sel), device='cuda')

    def planes(self, layer):
        import ctypes as C
        import torch
        from ssd_keras_b200 import _ffi
        hp, wp, cs, pad = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        _ffi.check(_ffi.lib().ssdk_model_layer_planes_shape(self.h, layer, C.byref(hp), C.byref(wp), C.byref(cs), C.byref(pad)))
        shape = (self.B, hp.value, wp.value, cs.value)
        hi = torch.empty(shape, dtype=torch.int16, device='cuda')
        lo = torch.empty(shape, dtype=torch.int16, device='cuda') if self.split else None
        _ffi.check(_ffi.lib().ssdk_model_read_layer_planes(self.h, layer, _ffi.dptr(hi), _ffi.dptr(lo), _ffi.stream_ptr()))
        torch.cuda.synchronize()
        out = (hi[self.sel].cpu().numpy().view(np.uint16), None if lo is None else lo[self.sel].cpu().numpy().view(np.uint16), pad.value)
        del hi, lo
        return out

    def head_f32(self, layer, shape):
        import torch
        from ssd_keras_b200 import _ffi
        out = torch.empty((self.B,) + tuple(shape), dtype=torch.float32, device='cuda')
        _ffi.check(_ffi.lib().ssdk_model_read_layer(self.h, layer, _ffi.dptr(out), _ffi.stream_ptr()))
        torch.cuda.synchronize()
        return out[self.sel].cpu().numpy()


class _Judge:
    """Collects every ratio of a configuration, logs it, and lists the failures (all layers are judged before asserting)."""

    def __init__(self, cfg):
        self.cfg, self.fail, self.worst, self.margin = cfg, [], {}, {}

    def __call__(self, layer, kind, ratio, perturbed, **extra):
        cc.log_ratio(dict(test='bench_plan', case=self.cfg['name'], layer=layer, kind=kind, prec=self.cfg['prec'], ratio=ratio,
                          perturbed={str(k): v for k, v in perturbed.items()}, **extra))
        self.worst[kind] = max(self.worst.get(kind, 0.0), ratio)
        if not ratio <= 1.0:
            self.fail.append('%s (%s): ratio %.4g' % (layer, kind, ratio))
        for k, v in perturbed.items():
            self.margin[(layer, k)] = v
            if not v > 1.0:
                self.fail.append('%s (%s): perturbation %s passes the bound (ratio %.4g)' % (layer, kind, k, v))

    def zero_outside(self, layer, planes, H, W, C_):
        for o in cc.outside(planes, H, W, C_):
            if np.any(o):
                self.fail.append('%s: border / padding channels of the planes not zero' % layer)


def _value(hi_lo):
    hi, lo = hi_lo
    return hi.astype(np.float64) + (0.0 if lo is None else lo)


def _softmax_perturbed(p, l, C_):
    """Rows shifted by one prior, and the last two classes swapped."""
    sw = p.copy()
    sw[..., [C_ - 2, C_ - 1]] = p[..., [C_ - 1, C_ - 2]]
    return {'prior_shift': (np.roll(p, 1, axis=1), np.roll(l, 1, axis=1)), 'class_swap': (sw, l)}


def _perturbations(plan, k, cin, split, bias):
    """conv_cases.perturbations with the centre tap of an even kernel and the bias of a live channel."""
    centre = (k // 2) * k + k // 2
    out = []
    for p in cc.perturbations(plan, k * k, cin, split, bias):
        if p[0] in ('tap', 'kblock'):
            p = (p[0], centre) + p[2:]
        out.append(('bias_live',) if p[0] == 'bias' else p)
    return out


def _judge_plan(model, cfg, B, sm):
    """The device's plan of every conv / head layer against the mirror -> the mirrored layers."""
    mirror = bp.layers(model, B, sm)
    for i, L in enumerate(mirror):
        if L['op'] not in ('conv', 'head'):
            continue
        plan = model.layer_plan(B, L['name'])
        assert plan['kernel'] == L['kernel'], (cfg['name'], L['name'], plan, L)
        for k in PLAN_KEYS[L['kernel']]:
            assert plan[k] == L[k], (cfg['name'], L['name'], k, plan, L)
        if L['op'] == 'head':
            assert plan['head_fused'] == L['head_fused'], (cfg['name'], L['name'], plan)
    reached = bp.regimes(model, B, sm)
    assert bp.EXPECTED[cfg['name']] <= reached, (cfg['name'], sm, sorted(reached))
    return mirror


def _conv(judge, rd, model, w, L, src_planes, src, split, prec):
    plan = model.layer_plan(rd.B, L['name'])
    xin = cc.interior(src_planes, src['H'], src['W'], src['C'])
    taps = L['k'] ** 2
    scale = shift = None
    if L['bn_layer']:
        scale, shift = bp.folded_bn(w, L['bn_layer'])
    b = w[L['name'] + '/bias']
    perts = _perturbations(plan, L['k'], L['cin'], split, b)
    ref, A, pv = opexact.conv_ref(xin, w[L['name'] + '/kernel'], b, stride=L['stride'], dil=L['dil'], pads=L['pads'], mode=prec,
                                  act=L['act'], bn_scale=scale, bn_shift=shift, perturb=perts)
    bnd = opexact.bound(ref, A, cc.n_steps_of(plan, taps, L['cin']), 'split' if split else 'bf16')
    planes = rd.planes(L['index'])
    got = _value(cc.interior(planes, L['H'], L['W'], L['C']))
    judge(L['name'], plan['kernel'], opexact.err_ratio(got, ref, bnd), {p[0]: opexact.err_ratio(got, v, bnd) for p, v in pv.items()},
          bn=plan['bn'], kblocks=plan['kblocks'])
    judge.zero_outside(L['name'], planes, L['H'], L['W'], L['C'])
    return planes


def _head(judge, rd, model, w, L, src_planes, src, y, split, prec):
    plan = model.layer_plan(rd.B, L['name'])
    s = model.specs[L['index']]
    C_, nb, n = model.n_classes, L['n_boxes'], L['H'] * L['W'] * L['n_boxes']
    S = len(rd.sel)
    xin = cc.interior(src_planes, src['H'], src['W'], src['C'])
    kc, bc = w[s.params['conf_name'] + '/kernel'], w[s.params['conf_name'] + '/bias']
    kl, bl = w[s.params['loc_name'] + '/kernel'], w[s.params['loc_name'] + '/bias']
    perts = _perturbations(plan, 3, L['cin'], split, bc)
    geo = dict(pads=L['pads'], mode=prec)
    zc, Ac, pc = opexact.conv_ref(xin, kc, bc, perturb=perts, **geo)
    zl, Al, pl = opexact.conv_ref(xin, kl, bl, perturb=[p for p in perts if p[0] != 'bias_live'], **geo)
    zc, Ac, zl, Al = zc.reshape(S, n, C_), Ac.reshape(S, n, C_), zl.reshape(S, n, 4), Al.reshape(S, n, 4)
    steps = cc.n_steps_of(plan, 9, L['cin'])
    rows = y[:, L['prior_off']:L['prior_off'] + n]
    anchors = model.anchors_f32[L['prior_off']:L['prior_off'] + n]
    if not (np.array_equal(rows[..., C_ + 4:C_ + 8], np.broadcast_to(anchors, (S, n, 4)))
            and np.array_equal(rows[..., C_ + 8:], np.broadcast_to(model.variances, (S, n, 4)))):
        judge.fail.append('%s: anchors / variances of its y_pred rows differ' % L['name'])
    if plan['head_fused']:
        # the epilogue's probabilities and offsets against the logits of the planes it read
        p_ref, p_bnd = opexact.softmax_ref(zc, Ac, steps, C_)
        l_bnd = opexact.bound(zl, Al, steps, 'f32')

        def ratio(p, l):
            return max(opexact.err_ratio(rows[..., :C_], p, p_bnd), opexact.err_ratio(rows[..., C_:C_ + 4], l, l_bnd))
        perturbed = {}
        for d in perts:
            pp, _ = opexact.softmax_ref(pc[d].reshape(S, n, C_), np.zeros((S, n, C_)), steps, C_)
            perturbed[d[0]] = ratio(pp, pl.get(d, zl.reshape(S, n, 4)).reshape(S, n, 4))
        for k, (pp, ll) in _softmax_perturbed(p_ref, zl, C_).items():
            perturbed[k] = ratio(pp, ll)
        judge(L['name'], 'head_fused', ratio(p_ref, zl), perturbed, prior_off=L['prior_off'], C=C_)
        return
    # unfused: the GEMM's fp32 logits, then head_finalize_kernel from those stored logits
    logits = rd.head_f32(L['index'], (L['H'], L['W'], L['C'])).reshape(S, n, C_ + 4)
    got = logits.astype(np.float64)
    bc_ = opexact.bound(zc, Ac, steps, 'f32')
    bl_ = opexact.bound(zl, Al, steps, 'f32')

    def lratio(c, l):
        return max(opexact.err_ratio(got[..., :C_], c, bc_), opexact.err_ratio(got[..., C_:], l, bl_))
    judge(L['name'], 'head_logits', lratio(zc, zl),
          {d[0]: lratio(pc[d].reshape(S, n, C_), pl.get(d, zl).reshape(S, n, 4)) for d in perts}, C=C_)
    p_ref, p_bnd = opexact.softmax_ref(got[..., :C_], np.zeros((S, n, C_)), 0, C_)
    p_bnd = np.maximum(p_bnd, np.finfo(np.float64).tiny)
    off_ok = np.array_equal(rows[..., C_:C_ + 4], logits[..., C_:])

    def fratio(p, l):
        return max(opexact.err_ratio(rows[..., :C_], p, p_bnd), 0.0 if np.array_equal(rows[..., C_:C_ + 4], l) else np.inf)
    judge(L['name'], 'head_finalize', fratio(p_ref, logits[..., C_:]) if off_ok else np.inf,
          {k: fratio(pp, ll) for k, (pp, ll) in _softmax_perturbed(p_ref, logits[..., C_:], C_).items()},
          prior_off=L['prior_off'], C=C_)


@pytest.mark.parametrize('cfg', bp.CONFIGS, ids=[c['name'] for c in bp.CONFIGS])
def test_bench_plan_layers_within_operand_exact_bounds(cfg):
    import torch
    from oracle import synth
    t0 = time.time()
    sm = _sm_count()
    B, split, prec = cfg['B'], cfg['prec'] == 'bf16x3', cfg['prec']
    model = bp.build(cfg)
    w = bp.weights(cfg)
    model.set_weights(w)
    threads = torch.get_num_threads()
    try:
        mirror = _judge_plan(model, cfg, B, sm)
        img = synth.synth_images(11, B, cfg['size'], cfg['size'])
        x_dev = torch.from_numpy(img).cuda()
        y_dev = model.forward_device(x_dev)                                  # the call bench.py times (two-stream schedule)
        torch.cuda.synchronize()
        sel = list(cfg['judged'])
        y = y_dev[sel].cpu().numpy()
        rd = _Planes(model._plan(B)['handle'], B, split, sel)
        judge = _Judge(cfg)
        torch.set_num_threads(min(32, os.cpu_count() or 1))
        planes = {}
        for i, L in enumerate(mirror):
            L['index'] = i
            src = mirror[L['input']] if L['input'] is not None else None
            if L['op'] == 'input':
                p = model.specs[0].params
                mean = None if p.get('mean') is None else np.broadcast_to(np.asarray(p['mean'], np.float32).reshape(-1), (3,))
                std = None if p.get('stddev') is None else np.broadcast_to(np.asarray(p['stddev'], np.float32).reshape(-1), (3,))
                planes[i] = rd.planes(i)
                hi, lo = cc.interior(planes[i], L['H'], L['W'], 3)
                rh, rl = opexact.preprocess_ref(img[sel], mean, std, p.get('swap'))
                same = np.array_equal(hi, rh) and (lo is None or np.array_equal(lo, rl))
                judge(L['name'], 'preprocess', 0.0 if same else np.inf, {})
                judge.zero_outside(L['name'], planes[i], L['H'], L['W'], 3)
            elif L['op'] == 'conv':
                planes[i] = _conv(judge, rd, model, w, L, planes[L['input']], src, split, prec)
            elif L['op'] == 'pool':
                xin = cc.interior(planes[L['input']], src['H'], src['W'], src['C'])
                rh, rl, _ = opexact.pool_fwd_ref(xin[0], xin[1], L['k'], L['k'], L['stride'], L['pads'][0], L['pads'][1], L['H'], L['W'])
                planes[i] = rd.planes(i)
                hi, lo = cc.interior(planes[i], L['H'], L['W'], L['C'])
                same = np.array_equal(hi, rh) and (lo is None or np.array_equal(lo, rl))
                judge(L['name'], L['kernel'], 0.0 if same else np.inf, {})
                judge.zero_outside(L['name'], planes[i], L['H'], L['W'], L['C'])
            elif L['op'] == 'l2':
                gamma = w[L['name'] + '/gamma']
                xv = _value(cc.interior(planes[L['input']], src['H'], src['W'], src['C']))
                perts = [('no_gamma',)] + [('gamma_at', c) for c in (256, 511) if c < L['C']]
                ref, err, pv = opexact.l2norm_fwd_ref(xv, gamma, perturb=perts)
                bnd = np.maximum(err + opexact.UNIT['split' if split else 'bf16'] * np.abs(ref), np.finfo(np.float64).tiny)
                planes[i] = rd.planes(i)
                got = _value(cc.interior(planes[i], L['H'], L['W'], L['C']))
                judge(L['name'], L['kernel'], opexact.err_ratio(got, ref, bnd), {'_'.join(map(str, p)): opexact.err_ratio(got, v, bnd) for p, v in pv.items()})
                judge.zero_outside(L['name'], planes[i], L['H'], L['W'], L['C'])
            elif L['op'] == 'head':
                _head(judge, rd, model, w, L, planes[L['input']], src, y, split, prec)
            # planes no later layer reads are dropped
            last_use = {L2['input'] for L2 in mirror[i + 1:] if L2['input'] is not None}
            for k in [k for k in planes if k not in last_use]:
                del planes[k]
        if cfg['name'] == 'ssd300_b32_bf16x3':
            from oracle import decoder as odec
            out = model.decoder(y_dev).cpu().numpy()
            ref = odec.decode_layer(y_dev.cpu().numpy(), 0.01, 0.45, 200, 400, True, 300, 300, nms=odec.tf_nms_c)
            assert out.shape == (B, 200, 6)
            np.testing.assert_array_equal(out[:, :, :2], ref[:, :, :2])
            np.testing.assert_allclose(out[:, :, 2:], ref[:, :, 2:], rtol=1e-6, atol=1e-4)
        wall = time.time() - t0
        cc.log_ratio(dict(test='bench_plan_summary', case=cfg['name'], wall_s=wall, worst=judge.worst,
                          min_margin=min(judge.margin.values()) if judge.margin else None,
                          min_margin_at=str(min(judge.margin, key=judge.margin.get)) if judge.margin else None, sm_count=sm))
        assert not judge.fail, '%s: %d failures:\n%s' % (cfg['name'], len(judge.fail), '\n'.join(judge.fail))
    finally:
        torch.set_num_threads(threads)
        model._release()
