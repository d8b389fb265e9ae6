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
