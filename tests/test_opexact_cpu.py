"""CPU tests of the operand-exact convolution reference (oracle/opexact.py) and of the convolution case tables
(tests/conv_cases.py): the split is bit-exact round-to-nearest-even, the bound accepts an fp32 convolution of the split
operands and rejects every perturbation the GPU tests use, and the tables reach every kernel variant."""
import struct

import numpy as np
import pytest
import torch

import conv_cases as cc
from oracle import opexact


def _rne_bits(f):
    """Bit-level float32 -> bfloat16 round to nearest even, one value at a time."""
    u = struct.unpack('<I', struct.pack('<f', float(f)))[0]
    upper, lower = u >> 16, u & 0xffff
    if (u & 0x7fffffff) > 0x7f800000:
        return struct.unpack('<f', struct.pack('<I', ((upper | 0x40) << 16)))[0]
    if lower > 0x8000 or (lower == 0x8000 and upper & 1):
        upper += 1
    return struct.unpack('<f', struct.pack('<I', (upper << 16) & 0xffffffff))[0]


def test_bf16_rne_matches_bit_level_rounding_including_ties():
    rng = np.random.default_rng(0)
    base = rng.integers(0, 2 ** 32, 4000, dtype=np.uint64).astype(np.uint32)
    ties = (base & 0xffff0000) | 0x8000                                  # exactly halfway: even and odd upper halves
    near = np.concatenate([(base & 0xffff0000) | 0x7fff, (base & 0xffff0000) | 0x8001])
    special = np.array([0x7f7fffff, 0x7f7f8000, 0xff7f8000, 0x00008000, 0x00018000, 0x80008000, 0x7f800000, 0xff800000,
                        0x00000000, 0x80000000], dtype=np.uint32)
    bits = np.concatenate([base, ties, near, special])
    bits = bits[(bits & 0x7f800000) != 0x7f800000]                       # NaN payloads are covered below
    x = bits.view(np.float32)
    got = opexact.bf16_rne(x)
    want = np.array([_rne_bits(v) for v in x], dtype=np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(got.view(np.uint32), torch.from_numpy(x).to(torch.bfloat16).float().numpy().view(np.uint32))
    nan = np.array([0x7fc00000, 0x7f800001], dtype=np.uint32).view(np.float32)
    assert np.isnan(opexact.bf16_rne(nan)).all()


def test_split_is_hi_plus_lo_with_sixteen_bits():
    rng = np.random.default_rng(1)
    x = (rng.standard_normal(20000) * np.exp(rng.uniform(-20, 20, 20000))).astype(np.float32)
    hi, lo = opexact.split(x)
    assert np.array_equal(hi, opexact.bf16_rne(x))
    assert np.array_equal(lo, opexact.bf16_rne(x - hi))
    assert np.array_equal(opexact.bf16_rne(hi), hi) and np.array_equal(opexact.bf16_rne(lo), lo)
    rel = np.abs((hi.astype(np.float64) + lo) - x) / np.abs(x)
    assert rel.max() <= 2.0 ** -16
    # splitting the stored value hi + lo again gives the same planes, except where lo is exactly half an ulp of hi: the tie
    # then goes to the even neighbour (same value, the planes trade half an ulp).  The GPU tests therefore split the
    # float32 tensors they feed in, not the activations they read back.
    h2, l2 = opexact.split(hi + lo)
    assert np.array_equal(h2 + l2, hi + lo)
    moved = (h2 != hi) | (l2 != lo)
    assert moved.mean() < 0.01 and np.all(np.abs(lo[moved]) == np.abs(hi[moved] - h2[moved]) / 2)


def _f32_split_conv(x, w, b, pads, mode, act):
    """A float32 CPU convolution of the split operands, stored like EPI_SPLIT / a bf16 plan."""
    xh, xl = opexact.split(x)
    wh, wl = opexact.split(w)
    terms = [(xh, wh)] + ([(xh, wl), (xl, wh)] if mode == 'bf16x3' else [])
    pt, pl, pb, pr = pads
    y = 0
    for a, k in terms:
        at = torch.nn.functional.pad(torch.from_numpy(a).permute(0, 3, 1, 2), (pl, pr, pt, pb))
        y = y + torch.nn.functional.conv2d(at, torch.from_numpy(k).permute(3, 2, 0, 1))
    y = (y + torch.from_numpy(b).view(1, -1, 1, 1)).permute(0, 2, 3, 1).numpy()
    if act == 'relu':
        y = np.maximum(y, 0)
    hi, lo = opexact.split(y)
    return hi if mode == 'bf16' else hi + lo


@pytest.mark.parametrize('mode', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('cin,k', [(24, 3), (136, 3), (64, 1)])
def test_bound_accepts_fp32_conv_and_rejects_perturbations(mode, cin, k):
    rng = np.random.default_rng(cin + k)
    x = rng.standard_normal((2, 9, 10, cin)).astype(np.float32)
    w = (rng.standard_normal((k, k, cin, 64)) * np.sqrt(2.0 / (k * k * cin))).astype(np.float32)
    b = (rng.standard_normal(64) * 0.1).astype(np.float32)
    p = (k - 1) // 2
    pads = (p, p, p, p)
    if mode == 'bf16':
        x = opexact.bf16_rne(x)                                           # a bf16 plan stores its activations as hi only
    y = _f32_split_conv(x, w, b, pads, mode, 'relu')
    plan = dict(kernel='gemm', kblocks=(cin + 63) // 64)
    perturb = cc.perturbations(plan, k * k, cin, mode == 'bf16x3', b)
    y_ref, A, pert = opexact.conv_ref(x, w, b, pads=pads, mode=mode, act='relu', perturb=perturb)
    n_steps = opexact.n_steps_gemm(k * k, plan['kblocks'])
    bnd = opexact.bound(y_ref, A, n_steps, 'bf16' if mode == 'bf16' else 'split')
    assert opexact.err_ratio(y, y_ref, bnd) <= 1.0
    for d, yp in pert.items():
        assert opexact.err_ratio(y, yp, bnd) > 1.0, d


def test_perturbed_references_equal_recomputed_ones():
    """Each perturbed reference (the dropped products subtracted) equals a reference recomputed without those products."""
    rng = np.random.default_rng(9)
    x = rng.standard_normal((2, 7, 6, 72)).astype(np.float32)
    w = rng.standard_normal((3, 3, 72, 16)).astype(np.float32)
    b = rng.standard_normal(16).astype(np.float32)
    geo = dict(stride=2, dil=1, pads=(1, 0, 1, 2), mode='bf16x3', act='elu')
    perturb = [('tap', 4), ('taps', 2, 5), ('kblock', 7, 1), ('kcols', 100, 300), ('bias', 3)]
    _, _, pert = opexact.conv_ref(x, w, b, perturb=perturb, **geo)
    k = np.arange(9 * 72).reshape(3, 3, 72)
    dropped = {('tap', 4): k // 72 == 4, ('taps', 2, 5): (k // 72 >= 2) & (k // 72 < 5),
               ('kblock', 7, 1): (k // 72 == 7) & (k % 72 >= 64), ('kcols', 100, 300): (k >= 100) & (k < 300)}
    for p, mask in dropped.items():
        w2 = np.where(mask[..., None], 0, w).astype(np.float32)    # zero weights split to zero planes: the same products drop
        want, _, _ = opexact.conv_ref(x, w2, b, **geo)
        assert np.allclose(pert[p], want, rtol=1e-12, atol=1e-12), p
    b2 = b.copy()
    b2[3] = 0
    want, _, _ = opexact.conv_ref(x, w, b2, **geo)
    assert np.allclose(pert[('bias', 3)], want, rtol=1e-12, atol=1e-12)


def test_softmax_bound_accepts_fp32_softmax_and_rejects_a_shifted_logit():
    rng = np.random.default_rng(5)
    z = rng.standard_normal((3, 50, 21)) * 4
    A = np.abs(z) * 30
    p_ref, bnd = opexact.softmax_ref(z, A, 36, 21)
    p32 = torch.softmax(torch.from_numpy(z.astype(np.float32)), -1).numpy()
    assert opexact.err_ratio(p32, p_ref, bnd) <= 1.0
    z2 = z.copy()
    z2[1, 7, 3] += 1e-2
    p2, _ = opexact.softmax_ref(z2, A, 36, 21)
    assert opexact.err_ratio(p32, p2, bnd) > 1.0


def _variants(cases):
    return [(c, c['expect']) for c in cases]


def test_forward_case_table_reaches_every_variant():
    fw = _variants(cc.FORWARD_CASES)
    gemm = {(e['bn'], e['split']) for c, e in fw if e['kernel'] == 'gemm'}
    assert gemm >= {(64, 1), (128, 1), (160, 1), (64, 0), (128, 0), (256, 0)}
    partial = {(e['bn'], c['cout']) for c, e in fw if e['kernel'] == 'gemm' and c['cout'] % e['bn']}
    assert (160, 136) in partial and {(128, 264), (256, 264)} <= partial
    g = [c for c, e in fw if e['kernel'] == 'gemm']
    assert {8, 24, 72, 136} <= {c['cin'] for c in g}
    assert {1, 3, 4} <= {c['k'] for c in g} and 6 in {c['dil'] for c in g}
    assert any(c['k'] == 4 and c['pads'] == (0, 0, 0, 0) for c in g)
    for pads in ((0, 0, 2, 2), (2, 2, 0, 0)):
        envs = {c['env'].get('SSDK_SHARED_BORDER', '1') for c in g if c['pads'] == pads}
        assert envs == {'0', '1'}, pads
    assert any(c['act'] == 'relu' and c['bias'] and not c['bn'] for c in g)      # the bias + ReLU fast path
    assert any(c['act'] is None and c['bias'] for c in g)
    assert any(c['act'] == 'elu' for c in g) and any(not c['bias'] for c in g) and any(c['bn'] for c in g)
    assert {c['persistent'] for c in g} >= {'nk<stages', 'nk%stages'}
    assert any(c['persistent'] and c['prec'] == 'bf16' for c in g)
    first = {(e['bn'], e['kblocks'], e['split']) for c, e in fw if e['kernel'] == 'first_tc'}
    assert first == {(bn, kb, s) for bn in (64, 128) for kb in (1, 2) for s in (0, 1)}
    f = [c for c, e in fw if e['kernel'] == 'first_tc']
    assert {c['cin'] for c in f} == {1, 2, 3, 4} and any(c['dil'] == 2 for c in f)
    assert any(e['kernel'] == 'direct' for c, e in fw)
    assert {e.get('im2col_vec8') for c, e in fw if e['kernel'] == 'im2col_gemm'} == {0, 1}


def test_head_case_table_reaches_every_variant():
    hv = _variants(cc.HEAD_CASES)
    fixed = {(c['nb'], e['bn']) for c, e in hv if e['head_fused'] and c['C'] + 4 == 25}
    assert fixed >= {(4, 128), (6, 160), (8, 256)}
    generic = {(c['C'], c['prec']) for c, e in hv if e['head_fused'] and c['C'] + 4 != 25}
    assert (6, 'bf16x3') in generic and (81, 'bf16') in generic
    assert any(c['nb'] * (c['C'] + 4) == 255 for c, e in hv if e['head_fused'])
    unfused = [(c, e) for c, e in hv if not e['head_fused']]
    assert any(c['env'].get('SSDK_NO_HEAD_FUSION') == '1' for c, e in unfused)
    assert any(c['nb'] * (c['C'] + 4) == 200 and c['prec'] == 'bf16x3' and not c['env'] for c, e in unfused)


# ------------------------------------------------------------------------------------------------------------------------------
# backward references
# ------------------------------------------------------------------------------------------------------------------------------
def _conv_t(x, w, stride, dil, pads):
    pt, pl, pb, pr = pads
    xt = torch.nn.functional.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb))
    return torch.nn.functional.conv2d(xt, w.permute(3, 2, 0, 1), stride=stride, dilation=dil).permute(0, 2, 3, 1)


@pytest.mark.parametrize('k,stride,dil,pads', [(3, 1, 1, (1, 1, 1, 1)), (3, 1, 1, (0, 0, 2, 2)), (4, 1, 1, (0, 0, 0, 0)),
                                               (3, 1, 3, (3, 3, 3, 3)), (3, 2, 1, (1, 1, 1, 1)), (3, 2, 1, (0, 0, 0, 0)),
                                               (5, 1, 1, (2, 2, 2, 2))])
def test_backward_references_equal_float64_autograd(k, stride, dil, pads):
    rng = np.random.default_rng(k * 10 + stride + dil)
    B, H, W, cin, cout = 2, 9, 8, 16, 24
    x = rng.standard_normal((B, H, W, cin)).astype(np.float32)
    w = rng.standard_normal((k, k, cin, cout)).astype(np.float32)
    xt = torch.from_numpy(x.astype(np.float64)).requires_grad_()
    wh, wl = opexact.split(w)
    wt = torch.from_numpy(wh.astype(np.float64) + wl).requires_grad_()
    y = _conv_t(xt, wt, stride, dil, pads)
    dz = opexact.split(rng.standard_normal(y.shape).astype(np.float32))
    # bf16x3 drops dZ_lo * W_lo: autograd of the graph on dZ_hi (with W_hi + W_lo) plus dZ_lo (with W_hi)
    gx_hi = torch.autograd.grad(y, xt, torch.from_numpy(dz[0].astype(np.float64)), retain_graph=True)[0].numpy()
    wt_hi = torch.from_numpy(wh.astype(np.float64))
    xl = torch.from_numpy(x.astype(np.float64)).requires_grad_()
    gx_lo = torch.autograd.grad(_conv_t(xl, wt_hi, stride, dil, pads), xl, torch.from_numpy(dz[1].astype(np.float64)))[0].numpy()
    mask = rng.standard_normal((B, H, W, cin)).astype(np.float32)
    old = rng.standard_normal((B, H, W, cin))
    ref, A, _ = opexact.dgrad_ref(dz, w, (H, W), stride=stride, dil=dil, pads=pads, mask=mask, old=old)
    np.testing.assert_allclose(ref, (gx_hi + gx_lo) * (mask > 0) + old, rtol=1e-12, atol=1e-12)
    # weight gradient on the split operands: X_hi dZ_hi + X_hi dZ_lo + X_lo dZ_hi
    xh, xlo = opexact.split(x)
    want = 0
    for a, d in [(xh, dz[0]), (xh, dz[1]), (xlo, dz[0])]:
        wv = torch.from_numpy(w.astype(np.float64)).requires_grad_()
        want = want + torch.autograd.grad(_conv_t(torch.from_numpy(a.astype(np.float64)), wv, stride, dil, pads), wv,
                                          torch.from_numpy(d.astype(np.float64)))[0].numpy()
    ref, A, _ = opexact.wgrad_ref(x, dz, k, k, stride=stride, dil=dil, pads=pads)
    np.testing.assert_allclose(ref, want.transpose(3, 0, 1, 2), rtol=1e-12, atol=1e-12)


def test_dgrad_and_wgrad_bounds_accept_fp32_and_reject_perturbations():
    rng = np.random.default_rng(3)
    B, H, W, cin, cout, k = 2, 10, 9, 16, 80, 3
    pads = (1, 1, 1, 1)
    x = rng.standard_normal((B, H, W, cin)).astype(np.float32)
    w = (rng.standard_normal((k, k, cin, cout)) * 0.2).astype(np.float32)
    dz = opexact.split(rng.standard_normal((B, H, W, cout)).astype(np.float32))
    mask = rng.standard_normal((B, H, W, cin)).astype(np.float32)
    old = opexact.bf16_rne(rng.standard_normal((B, H, W, cin)).astype(np.float32)).astype(np.float64)
    pert = [('cross',), ('tap', 4), ('kblock', 4, 1), ('mask',), ('old',)]
    ref, A, perts = opexact.dgrad_ref(dz, w, (H, W), pads=pads, mask=mask, old=old, perturb=pert)
    # fp32 emulation: the same products, summed in float32 (torch float32 autograd), then mask, accumulation and the split store
    wh, wl = opexact.split(w)
    got = 0
    for d, kk in [(dz[0], wh), (dz[0], wl), (dz[1], wh)]:
        xt = torch.zeros((B, H, W, cin), dtype=torch.float32, requires_grad=True)
        got = got + torch.autograd.grad(_conv_t(xt, torch.from_numpy(kk), 1, 1, pads), xt, torch.from_numpy(d))[0]
    got = (got.numpy() * (mask > 0) + old.astype(np.float32)).astype(np.float32)
    got = np.sum(opexact.split(got), axis=0, dtype=np.float64)
    bnd = opexact.bound(ref, A, opexact.n_steps_gemm(9, 2) + 1, 'split')
    assert opexact.err_ratio(got, ref, bnd) <= 1.0
    for p, r in perts.items():
        assert opexact.err_ratio(got, r, bnd) > 1.0, p
    plan = dict(wgrad='transposed', kv=B * (H + 2) * 16, k_split=1)
    ref, A, perts = opexact.wgrad_ref(x, dz, k, k, pads=pads, perturb=[('cross',), ('tap', 4), ('kblock', 0), ('pixels', 0, 0, 0, 8, 8)])
    xh, xlo = opexact.split(x)
    got = 0
    for a, d in [(xh, dz[0]), (xh, dz[1]), (xlo, dz[0])]:
        wv = torch.zeros((k, k, cin, cout), dtype=torch.float32, requires_grad=True)
        got = got + torch.autograd.grad(_conv_t(torch.from_numpy(a), wv, 1, 1, pads), wv, torch.from_numpy(d))[0]
    got = got.numpy().transpose(3, 0, 1, 2)
    bnd = opexact.bound(ref, A, opexact.n_steps_wgrad(plan, 3), 'f32')
    assert opexact.err_ratio(got, ref, bnd) <= 1.0
    for p, r in perts.items():
        assert opexact.err_ratio(got, r, bnd) > 1.0, p


def test_perturbed_backward_references_equal_recomputed_ones():
    rng = np.random.default_rng(4)
    B, H, W, cin, cout, k = 1, 7, 6, 8, 72, 3
    pads = (1, 1, 1, 1)
    w = rng.standard_normal((k, k, cin, cout)).astype(np.float32)
    dz = opexact.split(rng.standard_normal((B, H, W, cout)).astype(np.float32))
    _, _, perts = opexact.dgrad_ref(dz, w, (H, W), pads=pads, perturb=[('tap', 4), ('kblock', 4, 1)])
    w_tap = w.copy()
    w_tap[1, 1] = 0
    np.testing.assert_allclose(perts[('tap', 4)], opexact.dgrad_ref(dz, w_tap, (H, W), pads=pads)[0], rtol=1e-12, atol=1e-12)
    d_blk = [d.copy() for d in dz]
    full = opexact.dgrad_ref(dz, w, (H, W), pads=pads)[0]
    for d in d_blk:
        d[..., 64:] = 0
    w_t = np.zeros_like(w)
    w_t[1, 1] = w[1, 1]
    only_blk = opexact.dgrad_ref(dz, w_t, (H, W), pads=pads)[0] - opexact.dgrad_ref(d_blk, w_t, (H, W), pads=pads)[0]
    np.testing.assert_allclose(perts[('kblock', 4, 1)], full - only_blk, rtol=1e-12, atol=1e-12)


def _pool_loop(x, g, KH, KW, s, pt, pl, last=False):
    B, H, W, Cc = x.shape
    out = np.zeros(x.shape)
    for b in range(B):
        for c in range(Cc):
            for yo in range(g.shape[1]):
                for xo in range(g.shape[2]):
                    best, at = None, None
                    for ky in range(KH):
                        for kx in range(KW):
                            y, xx = yo * s - pt + ky, xo * s - pl + kx
                            if 0 <= y < H and 0 <= xx < W:
                                v = x[b, y, xx, c]
                                if best is None or v > best or (last and v == best):
                                    best, at = v, (y, xx)
                    out[b, at[0], at[1], c] += g[b, yo, xo, c]
    return out


@pytest.mark.parametrize('KH,s,pads', [(2, 2, (0, 0, 0, 0)), (2, 2, (0, 0, 1, 1)), (3, 1, (1, 1, 1, 1))])
def test_pool_route_matches_a_literal_loop_on_ties(KH, s, pads):
    rng = np.random.default_rng(KH + s)
    x = rng.integers(-2, 3, (2, 7, 9, 3)).astype(np.float32)
    Ho, Wo = (7 + pads[0] + pads[2] - KH) // s + 1, (9 + pads[1] + pads[3] - KH) // s + 1
    g = rng.standard_normal((2, Ho, Wo, 3))
    r, _, _ = opexact.pool_route(x, g, KH, KH, s, pads[0], pads[1])
    np.testing.assert_allclose(r, _pool_loop(x, g, KH, KH, s, pads[0], pads[1]), rtol=1e-12, atol=1e-12)
    rl, _, _ = opexact.pool_route(x, g, KH, KH, s, pads[0], pads[1], last=True)
    np.testing.assert_allclose(rl, _pool_loop(x, g, KH, KH, s, pads[0], pads[1], last=True), rtol=1e-12, atol=1e-12)
    assert not np.allclose(r, rl), 'the inputs must contain tied maxima'
    old = rng.standard_normal(x.shape)
    ref, A, steps, perts = opexact.pool_bwd_ref(x, g, KH, KH, s, pads[0], pads[1], relu_mask=True, old=old,
                                                perturb=[('last',), ('mask',), ('old',)])
    np.testing.assert_allclose(ref, r * (x > 0) + old, rtol=1e-12, atol=1e-12)
    bnd = opexact.bound(ref, A, steps, 'split')
    got = np.sum(opexact.split((r * (x > 0)).astype(np.float32) + old.astype(np.float32)), axis=0, dtype=np.float64)
    assert opexact.err_ratio(got, ref, np.maximum(bnd, 1e-300)) <= 1.0
    for p, v in perts.items():
        assert opexact.err_ratio(got, v, np.maximum(bnd, 1e-300)) > 1.0, p


def test_l2norm_and_head_backward_references_equal_autograd():
    rng = np.random.default_rng(5)
    x = rng.standard_normal((2, 4, 5, 12))
    x[0, 1, 1] = 0.0                                                     # the clamped branch
    gy = rng.standard_normal(x.shape)
    gamma = rng.uniform(0.5, 20, 12)
    xt, gt = torch.from_numpy(x).requires_grad_(), torch.from_numpy(gamma).requires_grad_()
    y = gt * xt * torch.rsqrt(torch.clamp((xt * xt).sum(-1, keepdim=True), min=1e-12))
    gx, gg = torch.autograd.grad(y, (xt, gt), torch.from_numpy(gy))
    ref, A, kap, gref, gA, gsteps, perts = opexact.l2norm_bwd_ref(x, gy, gamma, perturb=[('proj',)])
    np.testing.assert_allclose(ref, gx.numpy(), rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(gref, gg.numpy(), rtol=1e-10, atol=1e-10)
    # fp32 emulation of the kernel passes, dropping the projection does not
    x32, d32, g32 = x.astype(np.float32), gy.astype(np.float32), gamma.astype(np.float32)
    ss = (x32 * x32).sum(-1, keepdims=True, dtype=np.float32)
    s = (1 / np.sqrt(np.maximum(ss, np.float32(1e-12)))).astype(np.float32)
    dot = (g32 * d32 * x32).sum(-1, keepdims=True, dtype=np.float32)
    got = s * g32 * d32 - np.where(ss > 1e-12, x32 * s * s * s * dot, 0)
    bnd = kap * A + opexact.UNIT['f32'] * np.abs(ref)
    assert opexact.err_ratio(got, ref, np.maximum(bnd, 1e-300)) <= 1.0
    assert opexact.err_ratio(got, perts[('proj',)], np.maximum(bnd, 1e-300)) > 1.0
    # head: softmax backward on the class columns, pass-through on the offsets
    nb, Cc = 3, 21
    z = rng.standard_normal((2, 3, 4, nb * (Cc + 4))) * 4
    dy = rng.standard_normal((2, 3, 4, nb, Cc + 12))
    zt = torch.from_numpy(z.reshape(2, 3, 4, nb, Cc + 4)).requires_grad_()
    out = torch.cat([torch.softmax(zt[..., :Cc], -1), zt[..., Cc:]], -1)
    want = torch.autograd.grad(out, zt, torch.from_numpy(dy[..., :Cc + 4]))[0].numpy().reshape(z.shape)
    ref, A, kap, perts = opexact.head_bwd_ref(z, dy, nb, Cc, perturb=[('dot',)])
    np.testing.assert_allclose(ref, want, rtol=1e-10, atol=1e-12)
    z32 = z.reshape(2, 3, 4, nb, Cc + 4).astype(np.float32)
    e = np.exp(z32[..., :Cc] - z32[..., :Cc].max(-1, keepdims=True))
    p = e / e.sum(-1, keepdims=True, dtype=np.float32)
    d32 = dy.astype(np.float32)
    cls = p * (d32[..., :Cc] - (p * d32[..., :Cc]).sum(-1, keepdims=True, dtype=np.float32))
    got = np.concatenate([cls, d32[..., Cc:Cc + 4]], -1).reshape(z.shape)
    bnd = np.maximum(kap * A + opexact.UNIT['f32'] * np.abs(ref), 1e-300)
    assert opexact.err_ratio(got, ref, bnd) <= 1.0
    assert opexact.err_ratio(got, perts[('dot',)], bnd) > 1.0


def test_backward_case_table_reaches_every_variant():
    import test_gpu_backward_kernels as tb
    seen = {}
    for c in tb.BACKWARD_CASES:
        for i, e in c['expect'].items():
            seen.setdefault(c['prec'], []).append(e)
    allp = [e for v in seen.values() for e in v]

    def has(prec=None, **kv):
        pool_ = allp if prec is None else seen.get(prec, [])
        return any(all(e.get(k) == v for k, v in kv.items()) for e in pool_)
    for bn in (64, 128, 160):
        assert has('bf16x3', dgrad='gemm', dgrad_bn=bn), bn
    for bn in (64, 128, 256):
        assert has('bf16', dgrad='gemm', dgrad_bn=bn), bn
    for m in (0, 1):
        for a in (0, 1):
            assert has(dgrad='strided', dgrad_mask=m, dgrad_accumulate=a), ('strided', m, a)
            assert has(dgrad='gemm', dgrad_mask=m, dgrad_accumulate=a), ('gemm', m, a)
    assert has('bf16', dgrad='strided') and has('bf16x3', dgrad='strided')
    assert has(wgrad='native', k_split=1) and has(wgrad='native', min_k_split=2)
    assert has(wgrad='transposed', k_split=1) and has(wgrad='transposed', min_k_split=2)
    assert has(wgrad='direct', direct_fast=1) and has(wgrad='direct', direct_fast=0)
    for bw in (16, 32, 64):
        assert has(wgrad='native', bw=bw), bw
    assert has(wgrad='native', wgrad_bn=64) and has(wgrad='native', wgrad_bn=128) and has('bf16', wgrad='native')
    assert has(wgrad='native', a_boxes=1) and has(wgrad='native', a_boxes=2) and has(wgrad='native', co_tiles=2)
    assert has(wgrad='native', ci_tiles=2)
    assert has('bf16x3', wgrad='transposed') and has('bf16', wgrad='transposed') and has(wgrad='transposed', n_gemms=16)
    assert has(wgrad='im2col')
    im2col = [(c, L) for c in tb.BACKWARD_CASES for i, e in c['expect'].items() if e.get('wgrad') == 'im2col'
              for L in [c['layers'][i - 1]]]
    assert any(L['stride'] == 2 for c, L in im2col)
    assert any(L['stride'] == 1 and c['cin'] == 3 and L['input'] in (None, 0) and L['cout'] == 40 for c, L in im2col)
    # BatchNormalization backward: ELU, ReLU and no activation, C = 24 and 136, both precisions
    bn = [(c['prec'], L['act'], L['cout']) for c in tb.BACKWARD_CASES for L in c['layers'] if L.get('bn')]
    assert {a for _, a, _ in bn} == {'elu', 'relu', None} and {24, 136} <= {co for _, _, co in bn}
    assert {p for p, _, _ in bn} == {'bf16x3', 'bf16'}
    names = {c['name'] for c in tb.BACKWARD_CASES}
    for n in ('native_unaligned_dw_span', 'direct3x3_cin3_cout480_51840B', 'direct5x5_cin3_cout176_52800B', 'direct_cin1',
              'direct3x3_dil2_cin4', 'im2col_cin3_cout40', 'l2norm_linear_zero_pixel', 'l2norm_mask_acc', 'heads_voc25_two',
              'pool2x2_even_mask', 'pool2x2_odd_endpad_linear_acc', 'pool3x3_s1_p1_mask_acc'):
        assert n in names, n
    assert any(c['env'].get('SSDK_WGRAD_TRANSPOSED') == '1' for c in tb.BACKWARD_CASES)
    # the odd head in front of the unaligned case makes the next span start at an odd float offset
    c = next(c for c in tb.BACKWARD_CASES if c['name'] == 'native_unaligned_dw_span')
    assert (c['layers'][0]['nb'] * (c['C'] + 4) * (9 * c['cin'] + 1)) % 2 == 1



def test_bn_backward_reference_equals_autograd_and_its_bound_rejects_perturbations():
    rng = np.random.default_rng(6)
    B, H, W, Cc = 2, 5, 6, 24
    z = (rng.standard_normal((B, H, W, Cc)) * 2 + 0.5).astype(np.float32)
    gamma = rng.uniform(0.5, 1.5, Cc).astype(np.float32)
    beta = (rng.standard_normal(Cc) * 0.2).astype(np.float32)
    da = rng.standard_normal((B, H, W, Cc)).astype(np.float32)
    eps = 1e-3
    for act in ('elu', 'relu', None):
        zt = torch.from_numpy(z.astype(np.float64)).requires_grad_()
        gt = torch.from_numpy(gamma.astype(np.float64)).requires_grad_()
        bt = torch.from_numpy(beta.astype(np.float64)).requires_grad_()
        mean, var = zt.mean((0, 1, 2)), zt.var((0, 1, 2), unbiased=False)
        y = gt * (zt - mean) / torch.sqrt(var + float(np.float32(eps))) + bt
        a = torch.nn.functional.elu(y) if act == 'elu' else torch.relu(y) if act == 'relu' else y
        gz, gg, gb = torch.autograd.grad(a, (zt, gt, bt), torch.from_numpy(da.astype(np.float64)))
        a64 = a.detach().numpy()
        pert = [('m1',), ('m2',)] + ([('elu1',)] if act == 'elu' else [])
        ref, A, kap, dgam, dbet, Ag, Ab, kp, perts = opexact.bn_bwd_ref(z, a64, da, gamma, act=act, eps=eps, perturb=pert)
        np.testing.assert_allclose(ref, gz.numpy(), rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(dgam, gg.numpy(), rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(dbet, gb.numpy(), rtol=1e-9, atol=1e-12)
        # fp32 emulation of bn_bwd_reduce_kernel + bn_bwd_apply_kernel (fp32 mean / rstd, float64 sums)
        mean32 = z.astype(np.float64).mean((0, 1, 2)).astype(np.float32)
        rstd32 = (1.0 / np.sqrt(z.astype(np.float64).var((0, 1, 2)) + np.float32(eps))).astype(np.float32)
        a32 = a64.astype(np.float32)
        d = np.where(a32 > 0, np.float32(1), a32 + np.float32(1)) if act == 'elu' else (a32 > 0).astype(np.float32) if act == 'relu' \
            else np.ones_like(a32)
        dy = (da * d).astype(np.float32)
        xh = ((z - mean32) * rstd32).astype(np.float32)
        m1 = dy.astype(np.float64).mean((0, 1, 2)).astype(np.float32)
        m2 = (dy * xh).astype(np.float64).mean((0, 1, 2)).astype(np.float32)
        got = (gamma * rstd32 * (dy - m1 - xh * m2)).astype(np.float32)
        bnd = kap * A + opexact.UNIT['split'] * np.abs(ref)
        assert opexact.err_ratio(got, ref, bnd) <= 1.0, act
        for p, r in perts.items():
            assert opexact.err_ratio(got, r, bnd) > 1.0, (act, p)
        g32 = (dy * xh).astype(np.float64).sum((0, 1, 2)).astype(np.float32)
        assert opexact.err_ratio(g32, dgam, kp * Ag) <= 1.0
        # each perturbed reference equals one recomputed without the dropped part
        if act == 'elu':
            np.testing.assert_allclose(perts[('elu1',)], opexact.bn_bwd_ref(z, a64, da, gamma, act=None, eps=eps)[0], rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------------------------------------
# optimiser updates and the training-phase forward launches (sections 6 - 10 of oracle/opexact.py)
# ------------------------------------------------------------------------------------------------------------------------------
def _fma(a, b, c, contract):
    """a * b + c in fp32: one rounding (an FMA, emulated exactly enough in float64) or two."""
    a, b, c = np.float32(a), np.float32(b), np.float32(c)
    if contract:
        return (a.astype(np.float64) * b + c).astype(np.float32)
    return (a * b).astype(np.float32) + c


def _opt_operands(rng, n):
    g = (rng.choice([-1.0, 1.0], n) * 10.0 ** rng.uniform(-9, 2, n)).astype(np.float32)
    g[rng.random(n) < 0.1] = 0
    w = (rng.standard_normal(n) * 0.1).astype(np.float32)
    return w, g


KSHAPE = (5, 3, 3, 4)                                                 # OHWI: distinct cout, taps and cin


def _grad32(w, g, l2, s, ks, contract):
    if ks is not None:                                                # the kernel reads g at the OHWI index of HWIO element i
        g = g.reshape(ks)
    return _fma(np.float32(2 * np.float32(l2)), w, (g.reshape(w.shape) * np.float32(s)).astype(np.float32), contract)


@pytest.mark.parametrize('contract', [False, True])
@pytest.mark.parametrize('kernel', [True, False])
def test_sgd_reference_loop_emulation_and_perturbations(contract, kernel):
    rng = np.random.default_rng(31 + contract)
    n = int(np.prod(KSHAPE))
    ks = KSHAPE if kernel else None
    w, _ = _opt_operands(rng, n)
    v = np.zeros(n, np.float32)
    for t, (lr, s, l2) in enumerate([(1e-2, 1.0, 5e-4), (5e-3, 0.5, 5e-4), (2e-3, 0.5, 0.0)], start=1):
        _, g = _opt_operands(rng, n)
        perts = [('hwio',), ('no_l2',)] if kernel else [('l2_all',)]
        perts = [p for p in perts if l2 or p not in (('no_l2',), ('l2_all',))] + ([('no_scale',)] if s != 1 else []) + \
            ([('no_momentum',)] if t > 1 else [])
        ref, bnd, pv = opexact.sgd_ref(w, v, g, lr, 0.9, l2=l2, scale=s, kernel_shape=ks, perturb=perts)
        # a literal float64 loop over the HWIO master, gradient read at the OHWI index
        want_w, want_v = np.zeros(n), np.zeros(n)
        for co in range(KSHAPE[0]):
            for kh in range(3):
                for kw in range(3):
                    for ci in range(KSHAPE[3]):
                        i = ((co * 3 + kh) * 3 + kw) * KSHAPE[3] + ci
                        gr = float(g[i]) * float(np.float32(s)) + (2 * float(np.float32(l2)) * float(w[i]) if kernel else 0.0)
                        want_v[i] = float(np.float32(0.9)) * float(v[i]) - float(np.float32(lr)) * gr
                        want_w[i] = float(w[i]) + want_v[i]
        np.testing.assert_allclose(ref['v'], want_v, rtol=1e-13, atol=1e-300)
        np.testing.assert_allclose(ref['w'], want_w, rtol=1e-13, atol=1e-300)
        # fp32 emulation of sgd_kernel<true> / sgd_kernel<false>
        gr = _grad32(w, g, l2, s, ks, contract) if kernel else (g * np.float32(s)).astype(np.float32)
        nv = _fma(np.float32(0.9), v, -(np.float32(lr) * gr).astype(np.float32), contract)
        got = {'w': (w + nv).astype(np.float32), 'v': nv}
        assert opexact.state_ratio(got, ref, bnd) <= 1.0, t
        for p, r in pv.items():
            assert opexact.state_ratio(got, r, bnd) > 1.0, (t, p)
        w, v = got['w'], got['v']


@pytest.mark.parametrize('contract', [False, True])
def test_adam_reference_loop_emulation_and_perturbations(contract):
    rng = np.random.default_rng(41 + contract)
    n = int(np.prod(KSHAPE))
    w, _ = _opt_operands(rng, n)
    w[:40] = 0                                                       # no l2 term at the first step: grad = g s exactly
    m = np.zeros(n, np.float32)
    v = np.zeros(n, np.float32)
    b1, b2, eps = np.float32(0.9), np.float32(0.999), np.float32(1e-8)
    for t, (lr, s, l2) in enumerate([(1e-3, 1.0, 5e-4), (2e-3, 0.5, 5e-4), (1e-3, 1.0, 0.0), (5e-4, 0.5, 0.0), (1e-3, 1.0, 5e-4)], 1):
        _, g = _opt_operands(rng, n)
        perts = [('t+1',), ('eps_in_root',)] + ([('t-1',), ('no_m',), ('no_v',)] if t > 1 else [])
        ref, bnd, pv = opexact.adam_ref(w, m, v, g, lr, b1, b2, eps, t, l2=l2, scale=s, kernel_shape=KSHAPE, perturb=perts)
        # literal float64 loop, Keras' formulas
        lr_t = float(np.float32(lr)) * np.sqrt(1 - float(b2) ** t) / (1 - float(b1) ** t)
        for i in range(n):
            gr = float(g[i]) * float(np.float32(s)) + 2 * float(np.float32(l2)) * float(w[i])
            mi = float(b1) * float(m[i]) + (1 - float(b1)) * gr
            vi = float(b2) * float(v[i]) + (1 - float(b2)) * gr * gr
            assert abs(ref['m'][i] - mi) <= 1e-13 * abs(mi) and abs(ref['v'][i] - vi) <= 1e-13 * abs(vi)
            wi = float(w[i]) - lr_t * mi / (np.sqrt(vi) + float(eps))
            assert abs(ref['w'][i] - wi) <= 1e-13 * abs(wi)
        # fp32 emulation of adam_kernel<true>
        lr_t32 = np.float32(np.float32(np.sqrt(1.0 - float(b2) ** t) / (1.0 - float(b1) ** t)) * np.float32(lr))
        gr = _grad32(w, g, l2, s, KSHAPE, contract)
        a = _fma(b1, m, ((np.float32(1) - b1) * gr).astype(np.float32), contract)
        b = _fma(b2, v, ((np.float32(1) - b2) * gr * gr).astype(np.float32), contract)
        den = (np.sqrt(b) + eps).astype(np.float32)
        w = (w - ((lr_t32 * a).astype(np.float32) / den).astype(np.float32)).astype(np.float32)
        got = {'w': w, 'm': a, 'v': b}
        assert opexact.state_ratio(got, ref, bnd) <= 1.0, t
        for p, r in pv.items():
            assert opexact.state_ratio(got, r, bnd) > 1.0, (t, p)
        if t == 1:
            assert np.any(np.sqrt(b) < eps) and np.any(np.sqrt(b) > 1e3 * eps), 'eps must matter for some elements and not for others'
        m, v = a, b


@pytest.mark.parametrize('act', ['elu', 'relu', None])
def test_bn_forward_reference_emulation_and_perturbations(act):
    rng = np.random.default_rng(7)
    B, H, W, Cc = 2, 5, 6, 24
    gamma = rng.uniform(0.5, 1.5, Cc).astype(np.float32)
    beta = (rng.standard_normal(Cc) * 0.2).astype(np.float32)
    mm, mv = np.zeros(Cc, np.float32), np.ones(Cc, np.float32)
    z_prev = None
    for p in range(3):
        z = np.sum(opexact.split((rng.standard_normal((B, H, W, Cc)) * 0.1 + 0.05 * p).astype(np.float32)), axis=0, dtype=np.float32)
        perts = [('biased',), ('no_eps',)] + ([('acc',)] if z_prev is not None else [])
        ref, A, kap, st, sb, pv = opexact.bn_fwd_ref(z, gamma, beta, mm, mv, act=act, z_prev=z_prev, perturb=perts)
        # float64 autograd-free check: torch's batch_norm in training mode on float64
        zt = torch.from_numpy(z.astype(np.float64)).permute(0, 3, 1, 2)
        rm, rv = torch.from_numpy(mm.astype(np.float64)), torch.from_numpy(mv.astype(np.float64))
        y = torch.nn.functional.batch_norm(zt, rm, rv, torch.from_numpy(gamma.astype(np.float64)), torch.from_numpy(beta.astype(np.float64)),
                                           training=True, momentum=1 - float(np.float32(0.99)), eps=float(np.float32(1e-3)))
        y = torch.nn.functional.elu(y) if act == 'elu' else torch.relu(y) if act == 'relu' else y
        np.testing.assert_allclose(ref, y.permute(0, 2, 3, 1).numpy(), rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(st['mean'], rm.numpy(), rtol=1e-10, atol=1e-14)
        np.testing.assert_allclose(st['var'], rv.numpy(), rtol=1e-10, atol=1e-14)
        # fp32 emulation of bn_finalize_kernel + bn_apply_kernel, stored as hi + lo
        z64 = z.astype(np.float64)
        mean, var = z64.mean((0, 1, 2)), np.maximum((z64 * z64).mean((0, 1, 2)) - z64.mean((0, 1, 2)) ** 2, 0)
        bm, br = mean.astype(np.float32), (1 / np.sqrt(var + float(np.float32(1e-3)))).astype(np.float32)
        yy = (gamma * ((z - bm).astype(np.float32) * br).astype(np.float32)).astype(np.float32) + beta
        a32 = np.maximum(yy, 0) if act == 'relu' else np.where(yy > 0, yy, np.expm1(np.minimum(yy, 0)).astype(np.float32)) if act == 'elu' else yy
        got = np.sum(opexact.split(a32.astype(np.float32)), axis=0, dtype=np.float64)
        N = B * H * W
        mom = np.float32(0.99)
        gst = {'mean': (mom * mm + (np.float32(1) - mom) * bm).astype(np.float32),
               'var': (mom * mv + (np.float32(1) - mom) * (var * N / (N - 1)).astype(np.float32)).astype(np.float32)}
        bnd = kap * A + opexact.UNIT['split'] * np.abs(ref)
        assert opexact.err_ratio(got, ref, bnd) <= 1.0 and opexact.state_ratio(gst, st, sb) <= 1.0, (act, p)
        for k, (ap, sp) in pv.items():
            assert max(opexact.err_ratio(got, ap, bnd), opexact.state_ratio(gst, sp, sb)) > 1.0, (act, p, k)
        mm, mv, z_prev = gst['mean'], gst['var'], z


@pytest.mark.parametrize('Cc', [32, 20, 520])
def test_l2norm_forward_reference_emulation_and_perturbations(Cc):
    rng = np.random.default_rng(Cc)
    x = rng.standard_normal((2, 3, 4, Cc)).astype(np.float32)
    x[0, 1, 1] = 0
    x[1, 2, 3] = (rng.standard_normal(Cc) * 1e-8).astype(np.float32)
    gamma = rng.uniform(0.5, 20, Cc).astype(np.float32)
    ref, err, pv = opexact.l2norm_fwd_ref(x, gamma, perturb=[('no_gamma',), ('gamma_shift',)])
    xt = torch.from_numpy(x.astype(np.float64))
    want = xt * torch.rsqrt(torch.clamp((xt * xt).sum(-1, keepdim=True), min=float(np.float32(1e-12)))) * torch.from_numpy(gamma.astype(np.float64))
    np.testing.assert_allclose(ref, want.numpy(), rtol=1e-12, atol=0)
    bnd = np.maximum(err + opexact.UNIT['split'] * np.abs(ref), 1e-300)
    for order in (1, -1):                                              # two summation orders, as l2norm_kernel and l2norm8_kernel
        ss = np.zeros(x.shape[:-1], np.float32)
        for c in range(Cc)[::order]:
            ss = _fma(x[..., c], x[..., c], ss, order > 0)
        inv = (1 / np.sqrt(np.maximum(ss, np.float32(1e-12)).astype(np.float64)) * (1 + 2 ** -22)).astype(np.float32)   # rsqrtf, 1 ulp off
        got = np.sum(opexact.split((x * inv[..., None]).astype(np.float32) * gamma), axis=0, dtype=np.float64)
        assert opexact.err_ratio(got, ref, bnd) <= 1.0, order
        for p, r in pv.items():
            assert opexact.err_ratio(got, r, bnd) > 1.0, (order, p)
    assert not np.any(ref[0, 1, 1]) and np.all(ref[1, 2, 3] != 0)


@pytest.mark.parametrize('k,s,pads', [(2, 2, (0, 0, 0, 0)), (2, 2, (0, 0, 1, 1)), (3, 1, (1, 1, 1, 1)), (3, 2, (0, 0, 0, 0))])
def test_pool_forward_reference_matches_a_literal_loop(k, s, pads):
    import test_gpu_train_step_kernels as ts
    rng = np.random.default_rng(k + s)
    H, W = 7, 9
    x = ts._tie_input(rng, (2, H, W, 3))
    hi, lo = opexact.split(x)
    Ho, Wo = (H + pads[0] + pads[2] - k) // s + 1, (W + pads[1] + pads[3] - k) // s + 1
    rh, rl, pv = opexact.pool_fwd_ref(hi, lo, k, k, s, pads[0], pads[1], Ho, Wo, perturb=[('hi_only',), ('lo_tie',)])
    for b in range(2):
        for c in range(3):
            for yo in range(Ho):
                for xo in range(Wo):
                    best, at = -np.inf, None
                    for ky in range(k):
                        for kx in range(k):
                            y, xx = yo * s - pads[0] + ky, xo * s - pads[1] + kx
                            if 0 <= y < H and 0 <= xx < W and float(hi[b, y, xx, c]) + float(lo[b, y, xx, c]) > best:
                                best, at = float(hi[b, y, xx, c]) + float(lo[b, y, xx, c]), (y, xx)
                    assert rh[b, yo, xo, c] == hi[b, at[0], at[1], c] and rl[b, yo, xo, c] == lo[b, at[0], at[1], c]
    for p, (ph, pl) in pv.items():
        assert not (np.array_equal(ph, rh) and np.array_equal(pl, rl)), p


def test_preprocess_reference_matches_a_literal_loop():
    rng = np.random.default_rng(2)
    img = rng.uniform(0, 255, (2, 3, 4, 3)).astype(np.float32)
    mean, std, swap = (123.68, 116.779, 103.939), (58.393, 57.12, 57.375), (2, 1, 0)
    for m_, s_, w_ in ((mean, None, None), (mean, std, None), (mean, std, swap)):
        hi, lo = opexact.preprocess_ref(img, m_, s_, w_)
        sw = w_ or (0, 1, 2)
        for idx in np.ndindex(img.shape[:3]):
            for c in range(3):
                t = np.float32(img[idx + (sw[c],)]) - np.float32(m_[sw[c]])
                if s_ is not None:
                    t = np.float32(t / np.float32(s_[sw[c]]))
                h = opexact.bf16_rne(np.array([t], np.float32))[0]
                assert hi[idx + (c,)] == h and lo[idx + (c,)] == opexact.bf16_rne(np.array([t - h], np.float32))[0]


def test_train_step_case_tables_reach_every_variant():
    import test_gpu_train_step_kernels as ts
    # optimiser: both optimisers x both precisions over a graph holding every parameter kind; every kernel span is
    # a conv or head kernel with distinct cout, taps and cin (a transposed index lands on another element)
    assert {(c['optimizer'], c['prec']) for c in ts.OPT_CASES} == {(o, p) for o in ('sgd', 'adam') for p in ('bf16x3', 'bf16')}
    L = ts.OPT_LAYERS
    assert L[0]['op'] == 'conv' and L[0]['input'] is None                 # image-facing: the direct kernel (3 input channels)
    assert any(x['op'] == 'conv' and x['k'] == 3 and x['stride'] == 1 and not x['bn'] and x['cout'] not in (9, 24) for x in L[1:])
    assert any(x['op'] == 'conv' and x['bn'] and x['act'] == 'elu' for x in L)
    assert any(x['op'] == 'l2' for x in L) and any(x['op'] == 'head' for x in L) and any(x.get('stride') == 2 for x in L)
    assert len(ts.SGD_STEPS) >= 3 and len(ts.ADAM_STEPS) >= 5
    for steps in (ts.SGD_STEPS, ts.ADAM_STEPS):
        assert {s for _, s, _ in steps} == {1.0, 0.5} and {l for _, _, l in steps} == {0.0, 5e-4}
        assert len({lr for lr, _, _ in steps}) > 1
    # re-pack: every WeightLayout, the direct kernel's master and the head interleave
    fwd = {ts.REPACK_LAYOUTS[e['fwd']] for e in ts.REPACK_EXPECT.values()}
    dgr = {ts.DGRAD_LAYOUTS[e['dgrad']] for e in ts.REPACK_EXPECT.values() if e['dgrad']}
    assert fwd == {'master', 'PACK_FWD', 'PACK_FWD_IM2COL'} and dgr == {'PACK_DGRAD', 'PACK_DGRAD_COL'}
    assert ts.REPACK_LAYERS[-1]['op'] == 'head'
    # max-pool and L2Normalization: both kernels each
    assert {ts.pool_kernel_of(c['H'], c['W'], c['k'], c['stride'], c['pads']) for c in ts.POOL_CASES} == {'maxpool2x2', 'maxpool'}
    assert any(c['H'] == 75 and c['pads'] == (0, 0, 1, 1) for c in ts.POOL_CASES)
    ks = {ts.l2norm_kernel_of(c['C'], -(-c['C'] // 8) * 8): c['C'] for c in ts.L2_CASES}
    assert set(ks) == {'l2norm8', 'l2norm'} and {20, 520} <= {c['C'] for c in ts.L2_CASES}
    # BatchNormalization: ELU / ReLU / none, C = 24 and 136, both precisions, both branches of bn_grid
    bn = [(c, x) for c in ts.BN_CASES for x in c['layers'] if x['bn']]
    assert {x['act'] for _, x in bn} == {'elu', 'relu', None} and {24, 136} <= {x['cout'] for _, x in bn}
    assert {c['prec'] for c in ts.BN_CASES} == {'bf16x3', 'bf16'}
    branches = {ts.bn_grid(c['B'], c['H'], c['W'], x['cout'])[1] for c, x in bn}
    assert branches == {1, 2}
    assert ts.bn_grid(1, 10, 10, 136) == (17, 2)
    # preprocessing: mean only, mean + std, and the BGR swap
    assert [(c['stddev'] is not None, c['swap'] is not None) for c in ts.PRE_CASES] == [(False, False), (True, False), (True, True)]
