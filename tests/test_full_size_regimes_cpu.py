"""The full-size regime cases (tests/regime_cases.py) against the mirrored size rules: every regime is reached by a new case,
with the shapes its kernels have to handle, and by no case of the per-launch tables, whose graphs are too small for it."""
import numpy as np
import pytest

import conv_cases as cc
import regime_cases as rc
import swap_cases as sc
import test_gpu_backward_kernels as tb
import test_gpu_train_step_kernels as ts
from oracle import opexact


def _conv_case_as_bcase(c):
    """A one-layer inference case of conv_cases / swap_cases in the bcase form regime_cases.reach reads."""
    layer = tb.conv(c['cout'], c['k'], stride=c['stride'], dil=c['dil'], pads=c['pads'], act=c['act'], bn=c['bn'])
    return tb.bcase(c['name'], c['B'], c['H'], c['W'], c['cin'], [layer], {})


def test_every_case_reaches_its_regimes():
    for c in rc.REGIME_CASES:
        got = rc.reach(c)
        assert c['regimes'] <= rc.regimes(c), (c['name'], rc.regimes(c))
        for i, kernel in c['fwd'].items():
            assert got[i]['fwd'] == kernel, (c['name'], i, got[i])
    assert set().union(*[c['regimes'] for c in rc.REGIME_CASES]) == set(rc.REGIMES)


def test_the_cases_cover_each_regime_in_its_variants():
    by = {c['name']: rc.reach(c) for c in rc.REGIME_CASES}
    cases = {c['name']: c for c in rc.REGIME_CASES}
    layers = [(cases[n], i, r) for n, rr in by.items() for i, r in rr.items()]
    # swap in training: ReLU planes read by the next layer's masked data gradient and native weight gradient, in both precisions
    relu = [c for c, i, r in layers if rc.SWAP_RELU in r['regimes'] and i == 1 and by[c['name']].get(2, {}).get('fwd') == 'gemm_swap']
    assert {c['prec'] for c in relu} == {'bf16x3', 'bf16'}
    for c in relu:
        assert c['expect'][2]['dgrad_mask'] == 1 and c['expect'][2]['wgrad'] == 'native', c['name']
    # swap into BatchNormalization: ELU and ReLU, 64 and < 64 channels, both precisions
    bn = [(c, c['layers'][i - 1]) for c, i, r in layers if rc.SWAP_BN in r['regimes']]
    assert {L['act'] for _, L in bn} == {'elu', 'relu'} and {L['cout'] for _, L in bn} == {64, 40}
    assert {c['prec'] for c, _ in bn} == {'bf16x3', 'bf16'}
    # BatchNormalization over a strided grid: >= 4 elements per thread at C = 32, 48 and 136; the cut grid of 17 groups
    strided = {c['layers'][i - 1]['cout']: r['bn'] for c, i, r in layers if r['bn'] and r['bn'][1] >= 4}
    assert {32, 48, 136} <= set(strided), strided
    assert strided[136] == (1054, 5, True)
    assert {c['prec'] for c, i, r in layers if rc.BN_STRIDED in r['regimes']} == {'bf16x3', 'bf16'}
    # the direct weight gradient: both kernels with >= 2 rows per block, a last block of one row, a dilated generic case,
    # >= 5 rows per block
    rows = [(c, c['layers'][i - 1], r['wgrad']) for c, i, r in layers if rc.WGRAD_ROWS in r['regimes']]
    assert {w[3] for _, _, w in rows} == {True, False}
    assert any(w[3] and w[0] == 2 and w[2] == 1 for _, _, w in rows)
    assert any(not w[3] and L['k'] == 5 and w[0] >= 3 for _, L, w in rows)
    assert any(not w[3] and L['dil'] > 1 for _, L, w in rows)
    assert any(w[0] >= 5 for _, _, w in rows)
    for c, _, _ in rows:
        assert c['expect'][1]['direct_fast'] == int(rc.reach(c)[1]['wgrad'][3]), c['name']
    # SSD7's conv1 at its notebook size: a preprocessed image, the 5x5 direct kernel into BatchNormalization + ELU
    c = cases['ssd7_conv1_300x480']
    L = c['layers'][0]
    assert (c['H'], c['W'], c['cin'], L['cout'], L['k'], L['act'], L['bn']) == (300, 480, 3, 32, 5, 'elu', True)
    assert c['input_layer']['stddev'] is not None and rc.DIRECT_BN in rc.regimes(c)


def test_the_per_launch_tables_reach_none_of_the_regimes():
    tables = {'conv_cases.FORWARD_CASES': [(_conv_case_as_bcase(c), False) for c in cc.FORWARD_CASES],
              'swap_cases.SWAP_CASES': [(_conv_case_as_bcase(c), False) for c in sc.SWAP_CASES],
              'BACKWARD_CASES': [(c, True) for c in tb.BACKWARD_CASES],
              'BN_CASES': [(tb.bcase(c['name'], c['B'], c['H'], c['W'], 16, c['layers'], {}), True) for c in ts.BN_CASES],
              'OPT_LAYERS': [(tb.bcase('opt', 1, 10, 10, 3, ts.OPT_LAYERS, {}), True)],
              'REPACK_LAYERS': [(tb.bcase('repack', 2, 12, 12, 3, ts.REPACK_LAYERS, {}), True)]}
    for name, cases in tables.items():
        for c, training in cases:
            assert not rc.regimes(c, training=training), (name, c['name'], rc.regimes(c, training=training))
    # the swap cases are inference plans: at their size a training plan would take the variant too
    assert all(rc.reach(c)[1]['fwd'] == 'gemm_swap' for c, _ in tables['swap_cases.SWAP_CASES'])


def test_the_rules_take_the_real_training_steps():
    # conv1_2 of SSD300 at B = 2 and SSD7's conv4 (64 -> 64 at 37 x 60) at B = 32 take the swap kernel
    assert sc.selects_swap(64, 64, 1, 2 * 300 * 300) and sc.selects_swap(64, 64, 1, 32 * 37 * 60)
    # SSD7's conv1 at its notebook batch: 16 x 300 x 480, 32 channels -> many elements per thread; rows_per_block 5
    assert rc.bn_grid(16, 300, 480, 32)[1] >= 30
    assert rc.direct_wgrad_rows(16, 300)[0] == 5
    # SSD300's conv1_1 at B = 32: rows_per_block 10; the SSD300 B = 2 and SSD512 B = 1 steps keep one row per block
    assert rc.direct_wgrad_rows(32, 300)[0] == 10
    assert rc.direct_wgrad_rows(2, 300)[0] == 1 and rc.direct_wgrad_rows(1, 512)[0] == 1
    # the SSD7 B = 4 96 x 128 step launches 768 blocks, one element per thread
    assert rc.bn_grid(4, 96, 128, 32)[:2] == (768, 1)


def _direct_wgrad_f32(x, g, KH, KW, dil, pads, fast, sm_count):
    """float32 emulation of wgrad_direct3x3_kernel (fast) / wgrad_direct_kernel in their summation order: per thread over the
    block's rows (the fast kernel: every PL-th pixel of a row, PL = 256 / (cout / 2) pixel lanes meeting in shared memory), then
    one fp32 add per block into the result.  x: (B, H, W, cin), g: (B, Ho, Wo, cout) float32 values -> (Cout, KH, KW, Cin)."""
    B, Ho, Wo, cout = g.shape
    cin = x.shape[-1]
    pt, pl, pb, pr = pads
    xp = np.pad(x, ((0, 0), (pt, pb + KH * dil), (pl, pr + KW * dil), (0, 0)))
    win = np.concatenate([xp[:, kh * dil:kh * dil + Ho, kw * dil:kw * dil + Wo] for kh in range(KH) for kw in range(KW)], -1)
    rpb, grid, _ = opexact.direct_wgrad_rows(B, Ho, sm_count)
    K = KH * KW * cin
    XR = np.zeros((grid * rpb, Wo, K), np.float32)
    GR = np.zeros((grid * rpb, Wo, cout), np.float32)
    XR[:B * Ho], GR[:B * Ho] = win.reshape(B * Ho, Wo, K), g.reshape(B * Ho, Wo, cout)
    XR, GR = XR.reshape(grid, rpb, Wo, K), GR.reshape(grid, rpb, Wo, cout)
    lanes = 256 // (cout // 2) if fast else 1
    acc = np.zeros((grid, lanes, K, cout), np.float32)
    for j in range(rpb):
        for t in range(-(-Wo // lanes) if fast else Wo):
            xo = np.arange(lanes) + t * lanes if fast else np.array([t])
            ok = xo < Wo
            xv = np.where(ok[None, :, None], XR[:, j, np.minimum(xo, Wo - 1)], 0).astype(np.float32)
            gv = np.where(ok[None, :, None], GR[:, j, np.minimum(xo, Wo - 1)], 0).astype(np.float32)
            acc = acc + xv[..., :, None] * gv[..., None, :]
    blk = np.zeros((grid, K, cout), np.float32)
    for lane in range(lanes):
        blk = blk + acc[:, lane]
    out = np.zeros((K, cout), np.float32)
    for b in range(grid - 1, -1, -1):
        out = out + blk[b]
    return out.T.reshape(cout, KH, KW, cin)


@pytest.mark.parametrize('case', [c for c in rc.REGIME_CASES if rc.WGRAD_ROWS in c['regimes']],
                         ids=[c['name'] for c in rc.REGIME_CASES if rc.WGRAD_ROWS in c['regimes']])
def test_direct_wgrad_step_count_holds_the_kernels_order_and_rejects_perturbations(case):
    """The step count of opexact.n_steps_wgrad_direct bounds an fp32 emulation of the kernel's own summation order, and the
    bound rejects a dropped middle tap, a dropped last block and a dropped first block of rows, as the GPU test asserts."""
    rng = np.random.default_rng(3)
    L = case['layers'][0]
    s = rc.layer_shapes(case)[1]
    k, dil = L['k'], L['dil']
    q = dil * (k - 1) // 2
    pads = (q, q, q, q)
    xs = opexact.split(rng.standard_normal((case['B'], case['H'], case['W'], case['cin'])).astype(np.float32))
    gs = opexact.split(rng.standard_normal((case['B'], s['Ho'], s['Wo'], L['cout'])).astype(np.float32))
    fast = rc.direct_fast(k, dil, case['cin'], L['cout'])
    got = _direct_wgrad_f32(xs[0] + xs[1], gs[0] + gs[1], k, k, dil, pads, fast, cc.SM_COUNT_H100)
    pert = [('tap', k * k // 2)] + tb.direct_block_perturbations(case['B'], s['Ho'], s['Wo'], cc.SM_COUNT_H100)
    ref, A, pv = opexact.wgrad_ref(xs, gs, k, k, dil=dil, pads=pads, mode='fp32', perturb=pert)
    steps = opexact.n_steps_wgrad_direct(case['B'], s['Ho'], s['Wo'], L['cout'], fast, cc.SM_COUNT_H100)
    assert steps < case['B'] * s['Ho'] * s['Wo'] // 8
    bnd = opexact.bound(ref, A, steps, 'f32')
    assert opexact.err_ratio(got, ref, bnd) <= 1.0
    assert {p[0] for p in pv} == {'tap', 'pixels'} and len(pv) == 3, pv
    for p, v in pv.items():
        assert opexact.err_ratio(got, v, bnd) > 1.0, (case['name'], p, opexact.err_ratio(got, v, bnd))
