"""GPU tests of the SSD loss kernel (ssd_loss_kernel, ssd_loss_phase_kernel in csrc/loss.cu) against the operand-exact float64
reference of oracle/opexact.py (section 11), launch by launch:
- every case asserts its launch plan (ssdk_ssd_loss_plan), runs ssdk_ssd_loss with the loss outputs (fwd), the gradient (bwd)
  and both (fwd_bwd), reads the per-box losses back after each (ssdk_ssd_loss_read_box_losses; they must be identical), holds
  n_pos / nnz / k / want exactly and the per-box losses, the loss and the gradient to their bounds, and requires every listed
  perturbation of the reference to fail;
- the hard-negative mask is checked through the gradient: a kept negative has w_cls = scale, an unkept one 0, a kept positive
  2 scale;
- a sweep of k over every rank of a small batch, refused calls between exact ones, and the phase-wise (multi-GPU) launches with
  1, 2 and 4 emulated ranks, whose histograms must equal np.bincount of the per-box keys and whose loss and gradient must be
  bit-identical to the fused launch.
Ratios go to SSDK_KERNEL_ERRORS_LOG (conv_cases.log_ratio).
"""
import numpy as np
import pytest

import conv_cases as cc
from oracle import opexact

pytestmark = pytest.mark.gpu

K_ROWS, K_COARSE, K_FINE, K_CACHE = 128, 2048, 65536, 2048
SMEM_OPTIN_H100 = 232448            # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
SMEM_PER_SM_H100 = 233472           # shared memory per SM; every resident CTA also takes 1 KB of it for the system
STATIC_SMEM = 2304                  # static shared memory of ssd_loss_kernel / ssd_loss_phase_kernel (ptxas -v)


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


# ------------------------------------------------------------------------------------------------------------------------------
# the launch shape, restated from plan_launch (tests/test_opexact_cpu.py checks the tables below with it)
# ------------------------------------------------------------------------------------------------------------------------------
def smem_bytes(W, stages, grad):
    tile = K_ROWS * W * 4
    pa = stages * 2 * tile + K_COARSE * 4 + K_CACHE * 8
    return max(pa, 3 * tile if grad else 0) + 128


def plan_of(P, C, grad, aligned=True):
    """(stages, bulk_ok) of a call, or None if it is refused."""
    W = C + 12
    stages = 1 if smem_bytes(W, 2, grad) > 100 * 1024 else 2
    if smem_bytes(W, stages, grad) > SMEM_OPTIN_H100 - STATIC_SMEM:
        return None
    return stages, int(P * W % 4 == 0 and aligned)


def grid_of(B, P, C, grad, sm_count):
    """The grid of a call: at most 4 CTAs per SM, as many as the SM's shared memory holds, at most one per tile."""
    stages, _ = plan_of(P, C, grad)
    per_sm = min(4, SMEM_PER_SM_H100 // (smem_bytes(C + 12, stages, grad) + STATIC_SMEM + 1024))
    return max(1, min(B * -(-P // K_ROWS), per_sm * sm_count))


def largest_c(grad):
    return max(c for c in range(2, 400) if plan_of(128, c, grad) is not None)


C_MAX_GRAD, C_MAX_FWD = 137, 188


# ------------------------------------------------------------------------------------------------------------------------------
# the case table (plain data)
# ------------------------------------------------------------------------------------------------------------------------------
LEVELS = (0.5, 0.25, 0.125, 0.0625)          # dyadic p0: every box with the same p0 has exactly the same loss
# p0 whose losses -log p0 fall in fine bins that share a cache slot (bin & 2047) in pairs: 0xbf80 / 0xb780 (slot 0x780) and
# 0xbf81 / 0xb781 (slot 0x781).  With the threshold in a 0x..81 bin, the 0x..80 bin below it in the same coarse bin is populated:
# a fallback count that is lost or lands elsewhere moves the selection into it.
P_2M16 = (1.0 - 256 * 2.0 ** -24, 1.0 - 257 * 2.0 ** -24)   # -log p0 just above 2**-16: fine bin 0xb780
P_2M16B = (1.0 - 258 * 2.0 ** -24, 1.0 - 259 * 2.0 ** -24)  # 2**-16 (1 + 2/256 ..): fine bin 0xb781
P_1 = (float(np.float32(np.exp(-1.003))), float(np.float32(np.exp(-1.005))))   # -log p0 just above 1.0: fine bin 0xbf80
P_1B = (float(np.float32(np.exp(-1.010))), float(np.float32(np.exp(-1.012))))  # 1 + 2/256 ..: fine bin 0xbf81
ALL = ('fwd', 'bwd', 'fwd_bwd')


def case(name, B, P, C, seed, modes=ALL, ratio=3, n_neg_min=0, alpha=1.0, upstream=None, offset=False, grad_offset=False,
         perturb=('drop_last', 'add_next'), **gen):
    return dict(name=name, B=B, P=P, C=C, seed=seed, modes=modes, ratio=ratio, n_neg_min=n_neg_min, alpha=alpha, upstream=upstream,
                offset=offset, grad_offset=grad_offset, perturb=perturb, gen=gen)


LOSS_CASES = [
    case('ssd300_b32_c21', 32, 8732, 21, 1, pos=0.02, neutral=0.05, perturb=('drop_last', 'add_next', 'per_image', 'loc_by_yt0')),
    case('coco_c81', 4, 8732, 81, 2, pos=0.02, neutral=0.05, alpha=0.5, perturb=('drop_last', 'add_next', 'no_alpha')),
    case('c25_two_stages', 3, 700, 25, 3, pos=0.05),
    case('c26_one_stage', 3, 700, 26, 4, pos=0.05),
    case('largest_c_grad', 2, 300, C_MAX_GRAD, 5, pos=0.05),
    case('largest_c_fwd', 2, 300, C_MAX_FWD, 6, modes=('fwd',), pos=0.05),
    case('odd_p_odd_w', 3, 301, 5, 7, pos=0.05),
    case('offset4_inputs', 2, 256, 20, 8, offset=True, pos=0.05),
    case('offset4_grad', 2, 384, 20, 9, grad_offset=True, pos=0.05),
    case('p1_b1', 1, 1, 4, 10, n_neg_min=1, pos=0.0, neutral=0.0, perturb=('drop_last',)),
    case('p127', 3, 127, 4, 11, pos=0.05),
    case('p128', 3, 128, 4, 12, pos=0.05),
    case('p129', 3, 129, 4, 13, pos=0.05),
    # the threshold in each of two fine bins that share a cache slot: whichever of them lost the slot counts through the
    # global-atomic fallback, and a lost or misplaced count there moves the threshold
    case('collision_t_near_1', 2, 400, 6, 14, pos=0.03, collide=True, cut_p0=P_1B[0], perturb=('drop_last', 'add_next', 'tie_reverse')),
    case('collision_t_near_2m16', 2, 400, 6, 26, pos=0.03, collide=True, cut_p0=P_2M16B[0],
         perturb=('drop_last', 'add_next', 'tie_reverse')),
    case('partial_ties_mid_warp', 4, 500, 6, 15, pos=0.0, levels=LEVELS, cut=(2, 300 + 17), perturb=('drop_last', 'add_next', 'tie_reverse')),
    case('partial_ties_tile_edge', 4, 500, 6, 16, pos=0.0, levels=LEVELS, cut=(1, 256), perturb=('drop_last', 'add_next', 'tie_reverse')),
    case('ties_all_kept', 3, 400, 6, 25, pos=0.0, levels=LEVELS, cut=(1, 100), cut_all=True,
         perturb=('drop_last', 'add_next')),
    case('ties_with_positives', 4, 500, 6, 17, pos=0.04, levels=LEVELS, ratio=5, perturb=('drop_last', 'add_next', 'per_image')),
    case('zero_bin', 3, 600, 6, 18, pos=0.05, neutral=0.0, over1=0.15, p0_one=0.2, n_neg_min=10 ** 6,
         perturb=('drop_last', 'add_next', 'signed_zero', 'tie_reverse')),
    case('zero_bin_positive_taken', 3, 600, 6, 19, pos=0.15, neutral=0.0, over1=0.1, n_neg_min=10 ** 6,
         perturb=('drop_last', 'add_next', 'tie_reverse')),
    case('clamp', 2, 300, 6, 20, pos=0.1, clamp=True),
    case('upstream_alpha', 4, 300, 6, 21, pos=0.05, alpha=0.25, upstream=(0.5, 0.0, -1.25, 2.0),
         perturb=('drop_last', 'add_next', 'no_alpha', 'no_upstream')),
    case('n_neg_min_above_nnz', 2, 300, 6, 22, pos=0.05, neutral=0.2, n_neg_min=10 ** 6, perturb=('drop_last', 'k_no_cap')),
    case('no_positives_none', 2, 300, 6, 23, pos=0.0, perturb=('add_next', 'no_max1')),
    case('no_positives_n_neg_min', 2, 300, 6, 24, pos=0.0, n_neg_min=40, perturb=('drop_last', 'add_next', 'no_max1')),
]

SWEEP = dict(B=3, P=300, C=4, seed=30)
PHASE_CASES = [case('phase_ssd300_collisions', 8, 1000, 21, 40, pos=0.03, neutral=0.05, collide=True, cut_p0=P_1B[0]),
               case('phase_ties', 4, 500, 6, 41, pos=0.0, levels=LEVELS, cut=(2, 37)),
               case('phase_ties_pos', 4, 500, 6, 42, pos=0.02, levels=LEVELS, ratio=7)]


def make_case(c):
    """-> (y_true, y_pred, upstream or None, n_neg_min) as float32 NumPy arrays, from the case's seed."""
    g = c['gen']
    rng = np.random.default_rng(c['seed'])
    B, P, C = c['B'], c['P'], c['C']
    W = C + 12
    pos, neu = g.get('pos', 0.05), g.get('neutral', 0.05)
    kind = rng.choice(3, size=(B, P), p=[1 - pos - neu, pos, neu])           # 0 negative, 1 positive, 2 neutral
    yt = np.zeros((B, P, W), np.float32)
    yt[..., 0] = kind == 0
    bi, pi = np.nonzero(kind == 1)
    ci = rng.integers(1, C, bi.size)
    yt[bi, pi, ci] = 1
    yt[..., C:C + 4] = rng.normal(0, 1, (B, P, 4))
    yt[..., C + 4:] = rng.uniform(0.05, 1, (B, P, 8))
    z = rng.normal(0, 2, (B, P, C))
    e = np.exp(z - z.max(-1, keepdims=True))
    yp = np.zeros_like(yt)
    yp[..., :C] = e / e.sum(-1, keepdims=True)
    yp[..., C:C + 4] = yt[..., C:C + 4] + rng.normal(0, 1.0, (B, P, 4))      # |d| on both sides of 1
    yp[..., C + 4:] = rng.uniform(0.05, 1, (B, P, 8))
    neg = kind == 0
    p0 = yp[..., 0]
    if 'levels' in g:                          # ties, interleaved with boxes above and below them
        s = neg & (rng.random((B, P)) < 0.7)
        p0[s] = rng.choice(g['levels'], int(s.sum()))
    if g.get('over1'):                         # class scores > 1: negative losses (negatives) and cls < 0 (positives)
        s = neg & (rng.random((B, P)) < g['over1'])
        p0[s] = rng.uniform(1.0, 4.0, int(s.sum()))
        yp[bi[: bi.size // 2], pi[: bi.size // 2], ci[: bi.size // 2]] = 1.5
    if g.get('p0_one'):                        # p0 = 1: cls = -0, negl = -0
        s = neg & (rng.random((B, P)) < g['p0_one'])
        p0[s] = 1.0
    if g.get('collide'):                       # one tile: fine bins that collide in the cache, in pairs; negative losses too
        rows = np.flatnonzero(neg[0, :K_ROWS])
        vals = list(P_1) + list(P_2M16) + list(P_1B) + list(P_2M16B) + [1.25, 2.5, 3.0]
        p0[0, rows] = [vals[i % len(vals)] for i in range(rows.size)]
    if g.get('clamp'):                         # p = 0 / below 1e-15 where tv != 0: clamped log, zero gradient
        s = rng.random(bi.size) < 0.5
        yp[bi[s], pi[s], ci[s]] = rng.choice([0.0, 1e-20, 1e-16], int(s.sum()))
        yp[np.nonzero(neg)[0][:5], np.nonzero(neg)[1][:5], 0] = 0.0
    n_neg_min = c['n_neg_min']
    if 'cut' in g or 'cut_p0' in g:   # k: every box above the tie level of the cut box, and the ties before it (all: cut_all)
        negl = box_losses_f32(yt, yp)[1].reshape(-1)
        if 'cut' in g:
            at = g['cut'][0] * P + g['cut'][1]
        else:                         # the middle one of the negatives whose p0 is cut_p0
            at = np.flatnonzero(neg.reshape(-1) & (p0.reshape(-1) == np.float32(g['cut_p0'])))
            at = int(at[at.size // 2])
        while negl[at] == 0 or np.sum(negl == negl[at]) < 2:
            at += 1
        v = negl[at]
        n_neg_min = int(np.sum(negl > v) + (np.sum(negl == v) if g.get('cut_all') else np.sum(np.flatnonzero(negl == v) < at)))
    up = None if c['upstream'] is None else np.asarray(c['upstream'], np.float32)
    return yt, yp.astype(np.float32), up, n_neg_min


def box_losses_f32(yt, yp, log_ulp=0):
    """float32 emulation of phase A's per-box losses -> (cls, negl, l): the class loop in order, logf as the correctly rounded
    log moved by log_ulp ulps."""
    B, P, W = yt.shape
    C = W - 12
    acc = np.zeros((B, P), np.float32)
    for c in range(C):
        tv = yt[..., c]
        L = np.log(np.maximum(yp[..., c], np.float32(1e-15)).astype(np.float64)).astype(np.float32)
        for _ in range(abs(log_ulp)):                                    # logf(1) = 0 exactly
            L = np.where(L != 0, np.nextafter(L, np.float32(np.inf if log_ulp > 0 else -np.inf)), L).astype(np.float32)
        acc = np.where(tv != 0, (acc + (tv * L).astype(np.float32)).astype(np.float32), acc)
    cls = (-acc).astype(np.float32)
    negl = (cls * yt[..., 0]).astype(np.float32)
    l = np.zeros((B, P), np.float32)
    for j in range(4):
        d = (yt[..., C + j] - yp[..., C + j]).astype(np.float32)
        ad = np.abs(d)
        l = (l + np.where(ad < 1, (np.float32(0.5) * d * d).astype(np.float32), (ad - np.float32(0.5)).astype(np.float32))).astype(np.float32)
    return cls, negl, l


# ------------------------------------------------------------------------------------------------------------------------------
# running the kernel
# ------------------------------------------------------------------------------------------------------------------------------
def _dev(a, offset=False):
    """A device copy of a, at a 4-byte offset from a 16-byte aligned allocation if asked."""
    import torch
    a = np.ascontiguousarray(a, np.float32)
    buf = torch.zeros(a.size + 4, dtype=torch.float32, device='cuda')
    v = buf[int(offset): int(offset) + a.size]
    v.copy_(torch.from_numpy(a.reshape(-1)))
    return v.view(a.shape)


def run_loss(mode, yt_d, yp_d, C, ratio, n_neg_min, alpha, up_d=None, grad_offset=False):
    """One fused call -> (loss, stats, grad, cls, negl) as NumPy (None where the mode writes nothing)."""
    import torch
    from ssd_keras_b200 import _ffi
    B, P, W = yp_d.shape
    lib, ctx, st, d = _ffi.lib(), _ffi.context(), _ffi.stream_ptr(), _ffi.dptr
    loss = torch.full((B,), np.nan, dtype=torch.float32, device='cuda') if mode != 'bwd' else None
    stats = torch.full((4,), -7, dtype=torch.int32, device='cuda') if mode != 'bwd' else None
    grad = _dev(np.full(yp_d.shape, np.nan, np.float32), grad_offset) if mode != 'fwd' else None
    up = up_d if mode != 'fwd' else None
    _ffi.check(lib.ssdk_ssd_loss(ctx, d(yt_d), d(yp_d), B, P, C, ratio, n_neg_min, alpha, d(up), d(loss), d(stats), d(grad), st))
    cls, negl = _ffi.loss_box_losses(B, P)
    torch.cuda.synchronize()
    f = lambda t: None if t is None else t.cpu().numpy()
    return f(loss), f(stats), f(grad), cls.cpu().numpy(), negl.cpu().numpy()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def judge(name, yt, yp, outs, ratio, n_neg_min, alpha, up, perturb, log=True, **kw):
    """Holds the outputs of one call or of several calls on the same data to the reference -> the ratios."""
    cls, negl = outs[0][3], outs[0][4]
    for o in outs[1:]:
        assert np.array_equal(_bits(o[3]), _bits(cls)) and np.array_equal(_bits(o[4]), _bits(negl)), name
    assert np.array_equal(_bits(negl), _bits((cls * yt[..., 0]).astype(np.float32))), name
    ref, bnd, pv = opexact.loss_ref(yt, yp, cls, negl, ratio, n_neg_min, alpha, up, perturb=perturb, **kw)
    r = {'cls': opexact.loss_ratio(cls, ref['cls'], bnd['cls']), 'loss': 0.0, 'grad': 0.0}
    for loss, stats, grad, _, _ in outs:
        if stats is not None:
            assert list(stats) == ref['stats'], (name, list(stats), ref['stats'])
            r['loss'] = max(r['loss'], opexact.loss_ratio(loss, ref['loss'], bnd['loss']))
        if grad is not None:
            r['grad'] = max(r['grad'], opexact.loss_ratio(grad, ref['grad'], bnd['grad']))
    assert max(r.values()) <= 1.0, (name, r)
    pert, pert_loss = {}, {}
    for p, rp in pv.items():
        worst = on_loss = 0.0
        for loss, stats, grad, _, _ in outs:
            if stats is not None:
                on_loss = max(on_loss, opexact.loss_ratio(loss, rp['loss'], bnd['loss']))
                worst = max(worst, np.inf if list(stats) != rp['stats'] else on_loss)
            if grad is not None:
                worst = max(worst, opexact.loss_ratio(grad, rp['grad'], bnd['grad']))
        pert[p], pert_loss[p] = worst, on_loss
        assert worst > 1.0, (name, p)
    if log:                                    # the perturbed ratios on everything, and on the loss alone
        cc.log_ratio({'kernel': 'ssd_loss', 'case': name, **r, 'perturbed': {p: min(v, 1e300) for p, v in pert.items()},
                      'perturbed_loss': {p: min(v, 1e300) for p, v in pert_loss.items()}})
    return ref, r


# ------------------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('c', LOSS_CASES, ids=[c['name'] for c in LOSS_CASES])
def test_ssd_loss_case(c):
    from ssd_keras_b200 import _ffi
    yt, yp, up, n_neg_min = make_case(c)
    B, P, C = c['B'], c['P'], c['C']
    yt_d, yp_d = _dev(yt, c['offset']), _dev(yp, c['offset'])
    up_d = None if up is None else _dev(up)
    for grad in (False, True):
        want = plan_of(P, C, grad, aligned=not c['offset'])
        if want is None:
            with pytest.raises(ValueError):
                _ffi.loss_plan(yt_d, yp_d, C, grad)
            continue
        p = _ffi.loss_plan(yt_d, yp_d, C, grad)
        assert (p['stages'], p['bulk_ok']) == want, (c['name'], grad, p)
        assert p['smem_bytes'] == smem_bytes(C + 12, want[0], grad), (c['name'], grad, p)
        assert p['grid'] == grid_of(B, P, C, grad, _sm_count()), (c['name'], grad, p)
    outs = [run_loss(m, yt_d, yp_d, C, c['ratio'], n_neg_min, c['alpha'], up_d, c['grad_offset']) for m in c['modes']]
    judge(c['name'], yt, yp, outs, c['ratio'], n_neg_min, c['alpha'], up, c['perturb'])


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def test_ssd_loss_largest_classes_and_one_more():
    """C_MAX_GRAD / C_MAX_FWD launch; one class more is refused with ValueError before any launch, by the plan and by the call."""
    import torch
    from ssd_keras_b200 import _ffi
    assert (largest_c(True), largest_c(False)) == (C_MAX_GRAD, C_MAX_FWD)
    B, P = 1, 200
    for C, modes in ((C_MAX_GRAD, ()), (C_MAX_GRAD + 1, ('bwd', 'fwd_bwd')), (C_MAX_FWD, ()), (C_MAX_FWD + 1, ALL)):
        yt = _dev(np.zeros((B, P, C + 12), np.float32))
        yp = _dev(np.full((B, P, C + 12), 0.5, np.float32))
        for grad in (False, True):
            if plan_of(P, C, grad) is None:
                with pytest.raises(ValueError):
                    _ffi.loss_plan(yt, yp, C, grad)
            else:
                assert _ffi.loss_plan(yt, yp, C, grad)['stages'] == 1
        assert (plan_of(P, C, True) is None) == (C > C_MAX_GRAD) and (plan_of(P, C, False) is None) == (C > C_MAX_FWD)
        for m in modes:
            n0 = _ffi.launch_count()
            with pytest.raises(ValueError):
                run_loss(m, yt, yp, C, 3, 0, 1.0)
            assert _ffi.launch_count() == n0
        torch.cuda.synchronize()


def test_ssd_loss_k_sweep_every_rank():
    """No positives: k = min(n_neg_min, nnz).  n_neg_min from 0 to nnz + 1 puts the threshold at every rank of the batch, so at
    every coarse and fine bin boundary it has; then neg_pos_ratio from 0 to 12 with positives."""
    rng = np.random.default_rng(SWEEP['seed'])
    B, P, C = SWEEP['B'], SWEEP['P'], SWEEP['C']
    c0 = case('sweep', B, P, C, SWEEP['seed'], pos=0.0, neutral=0.05, levels=LEVELS)
    yt, yp, _, _ = make_case(c0)
    p0 = yp[..., 0]
    s = rng.random((B, P)) < 0.5
    p0[s] = np.exp(-10.0 ** rng.uniform(-7, 1.5, int(s.sum())))              # losses over many coarse bins
    yp = yp.astype(np.float32)
    yt_d, yp_d = _dev(yt), _dev(yp)
    nnz = None
    m = 0
    while nnz is None or m <= nnz + 1:
        out = run_loss('fwd_bwd', yt_d, yp_d, C, 3, m, 1.0)
        ref, _ = judge('sweep_n_neg_min', yt, yp, [out], 3, m, 1.0, None, ('drop_last', 'add_next') if 0 < m <= 80 else (),
                       log=m % 50 == 0)
        nnz = ref['stats'][1]
        m += 1
    c1 = case('sweep_ratio', B, P, C, SWEEP['seed'] + 1, pos=0.03, neutral=0.05, levels=LEVELS)
    yt, yp, _, _ = make_case(c1)
    yt_d, yp_d = _dev(yt), _dev(yp)
    for ratio in range(13):
        out = run_loss('fwd_bwd', yt_d, yp_d, C, ratio, 0, 1.0)
        judge('sweep_ratio', yt, yp, [out], ratio, 0, 1.0, None, ('drop_last', 'add_next') if ratio else ())


def test_refused_ssd_loss_call_leaves_the_next_call_exact():
    """A bwd refused at the same (B, P) (too many classes for the gradient's shared memory) between two identical calls; a call
    that asks for neither the loss nor the gradient, refused; three consecutive same-shape calls on different data; two shapes
    alternating.  Every call must be exact."""
    import torch
    from ssd_keras_b200 import _ffi
    B, P = 2, 300
    data = [make_case(case('refused_%d' % i, B, P, 21, 50 + i, pos=0.05, levels=LEVELS)) for i in range(3)]
    other = make_case(case('other_shape', 3, 257, 21, 60, pos=0.05))
    big = C_MAX_GRAD + 1
    yt_big, yp_big = _dev(np.zeros((B, P, big + 12), np.float32)), _dev(np.full((B, P, big + 12), 0.5, np.float32))

    def exact(d, mode='fwd'):
        yt, yp, _, m = d
        out = run_loss(mode, _dev(yt), _dev(yp), 21, 3, m, 1.0)
        judge('refused_sequence', yt, yp, [out], 3, m, 1.0, None, ('drop_last', 'add_next'))
        return out
    first = exact(data[0])
    for C in (big, 150):                       # one refused call at a time: two would flip a wrongly flipped parity back
        n0 = _ffi.launch_count()
        with pytest.raises(ValueError):
            run_loss('bwd', yt_big, yp_big, C, 3, 0, 1.0)
        assert _ffi.launch_count() == n0
        again = exact(data[0])
        assert np.array_equal(_bits(first[0]), _bits(again[0])) and np.array_equal(first[1], again[1])
    n0 = _ffi.launch_count()
    with pytest.raises(ValueError, match='out_loss and out_grad are both NULL'):
        _ffi.check(_ffi.lib().ssdk_ssd_loss(_ffi.context(), _ffi.dptr(yt_big), _ffi.dptr(yp_big), B, P, big, 3, 0, 1.0, None, None,
                                            None, None, _ffi.stream_ptr()))
    assert _ffi.launch_count() == n0
    for d in data:
        exact(d, 'fwd_bwd')
    for _ in range(2):
        exact(other, 'fwd_bwd')
        exact(data[1], 'fwd_bwd')
    torch.cuda.synchronize()


def _phase_run(yt, yp, shards, ratio, n_neg_min, alpha):
    """The phase-wise loss of `shards` emulated ranks on one GPU (the all-reduces and the all-gather replaced by sums), checking
    each rank's histograms after phases 0 and 1 against np.bincount of its own keys."""
    import torch
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.distributed import GlobalLossRun
    B, P, W = yt.shape
    C = W - 12
    per = B // shards
    runs = [GlobalLossRun(torch.from_numpy(yt[r * per:(r + 1) * per]).cuda(), torch.from_numpy(yp[r * per:(r + 1) * per]).cuda(),
                          ratio, n_neg_min, alpha, shards, r, True) for r in range(shards)]
    for r in runs:
        r.phase(0)
    torch.cuda.synchronize()
    keys = []
    for i, r in enumerate(runs):
        _, negl = _ffi.loss_box_losses(per, P, ws=r.ws)
        negl = negl.cpu().numpy().reshape(-1)
        k = opexact.okey(negl[negl != 0]).astype(np.int64)
        keys.append(k)
        h = r.hist1.cpu().numpy().astype(np.int64)
        assert np.array_equal(h[:K_COARSE], np.bincount(k >> 21, minlength=K_COARSE)), i
        assert np.array_equal(h[K_COARSE:], np.bincount(k >> 16, minlength=K_FINE)), i
        pmax = yt[i * per:(i + 1) * per, :, 1:C].max(-1).astype(np.float64)
        cnt = r.counts.cpu().numpy()
        assert cnt[1] == k.size and cnt[0] == int(np.sum(np.rint(pmax * 2.0 ** 32))), i
    for name in ('counts', 'hist1'):
        tot = sum(getattr(r, name).clone() for r in runs)
        for r in runs:
            getattr(r, name).copy_(tot)
    for r in runs:
        r.phase(1)
    torch.cuda.synchronize()
    return runs, keys


@pytest.mark.parametrize('shards', [1, 2, 4])
@pytest.mark.parametrize('c', PHASE_CASES, ids=[c['name'] for c in PHASE_CASES])
def test_phases_match_ssd_loss_bit_for_bit(c, shards):
    import torch
    yt, yp, _, n_neg_min = make_case(c)
    B, P, C = c['B'], c['P'], c['C']
    ratio, alpha = c['ratio'], c['alpha']
    fused = run_loss('fwd_bwd', _dev(yt), _dev(yp), C, ratio, n_neg_min, alpha)
    ref, _ = judge(c['name'], yt, yp, [fused], ratio, n_neg_min, alpha, None, c['perturb'])
    runs, keys = _phase_run(yt, yp, shards, ratio, n_neg_min, alpha)
    # hist2: the low key bits of the boxes in the level-1 bin of the k-th largest loss
    negl = fused[4].reshape(-1)
    k = ref['stats'][2]
    b1 = int(opexact.okey(negl[opexact._order(negl)[k - 1]])[0]) >> 16 if k > 0 else None
    for i, r in enumerate(runs):
        h = r.hist2.cpu().numpy().astype(np.int64)
        kk = keys[i][(keys[i] >> 16) == b1] if b1 is not None else keys[i][:0]
        assert np.array_equal(h[K_COARSE:], np.bincount(kk & 0xffff, minlength=K_FINE)), i
        assert np.array_equal(h[:K_COARSE], np.bincount((kk >> 5) & 0x7ff, minlength=K_COARSE)), i
    tot = sum(r.hist2.clone() for r in runs)
    for r in runs:
        r.hist2.copy_(tot)
    for r in runs:
        r.phase(2); r.phase(3)
    ties = torch.cat([r.ties.clone() for r in runs])
    if shards > 1 and 'cut' in c['gen']:     # the kept ties straddle a rank boundary: one rank keeps some of its ties, not all
        t = ties.cpu().numpy().astype(np.int64)
        before = np.concatenate([[0], np.cumsum(t)[:-1]])
        kept = np.clip(ref['stats'][3] - before, 0, t)
        assert np.any((kept > 0) & (kept < t)), (t, kept)
        if shards == 4:                       # and the others keep all of theirs or none
            assert np.any((kept == t) & (t > 0)) and np.any((kept == 0) & (t > 0)), (t, kept)
    for r in runs:
        r.ties_all.copy_(ties); r.phase(4)
    loss = np.concatenate([r.loss.cpu().numpy() for r in runs])
    grad = np.concatenate([r.grad.cpu().numpy() for r in runs])
    assert list(runs[0].stats.cpu().numpy()) == ref['stats']
    assert np.array_equal(_bits(loss), _bits(fused[0])) and np.array_equal(_bits(grad), _bits(fused[2])), (c['name'], shards)
    if shards > 1:                                                          # a rank's own B in the normalisation must fail
        per = B // shards
        _, bnd, pv = opexact.loss_ref(yt, yp, fused[3], fused[4], ratio, n_neg_min, alpha, global_B=B, local_B=per,
                                      perturb=('local_B',))
        assert opexact.loss_ratio(loss, pv['local_B']['loss'], bnd['loss']) > 1.0
