"""GPU tests of the launches a training step makes besides the convolutions and the backward pass, one launch at a time,
against the operand-exact float64 references of oracle/opexact.py (sections 6 - 10 there):
- the optimiser (sgd_kernel<true / false>, adam_kernel<true / false>) over several steps, each update judged on the parameters and the
  optimiser state read just before it (ssdk_trainer_read_params / ssdk_trainer_read_opt_state);
- the re-pack after an update: the forward planes and the data-gradient planes must hold the new master;
- the training-phase forward launches that are not convolutions: BatchNormalization (three consecutive passes, with the moving
  statistics), max-pooling (bit-exact on both planes), L2Normalization, the input preprocessing (bit-exact);
- the re-attach of an SSDTrainer after set_weights: its next Adam step is a fresh trainer's first step.
Every listed perturbation of a reference must fail its bound; borders and padding channels stay zero.  Ratios go to
SSDK_KERNEL_ERRORS_LOG (conv_cases.log_ratio).
"""
import numpy as np
import pytest

import conv_cases as cc
import test_gpu_backward_kernels as tb
from oracle import opexact

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


# ------------------------------------------------------------------------------------------------------------------------------
# the case tables (plain data: tests/test_opexact_cpu.py checks what they reach)
# ------------------------------------------------------------------------------------------------------------------------------
conv, head, l2 = tb.conv, tb.head, tb.l2

# every parameter kind: the direct image-facing kernel, a 3x3 conv with distinct taps / cin / cout, conv + BatchNormalization
# + ELU (gamma, beta), an L2Normalization gamma, a stride-2 conv and a fused head
OPT_LAYERS = [conv(16, 3), conv(24, 3, act='elu', bn=True), conv(40, 3), l2(), conv(48, 3, stride=2, pads=(1, 1, 1, 1)), head(2)]
# (lr, grad_scale, l2) per update: lr changes every step like LearningRateScheduler
SGD_STEPS = [(1e-2, 1.0, 5e-4), (5e-3, 0.5, 5e-4), (2e-3, 1.0, 0.0), (1e-3, 0.5, 0.0)]
ADAM_STEPS = [(1e-3, 1.0, 5e-4), (2e-3, 0.5, 5e-4), (1e-3, 1.0, 0.0), (5e-4, 0.5, 0.0), (1e-3, 1.0, 5e-4)]
OPT_CASES = [dict(name='%s_%s' % (o, p), optimizer=o, prec=p) for o in ('sgd', 'adam') for p in ('bf16x3', 'bf16')]
KIND_OF = {0: 'kernel', 1: 'bias', 2: 'l2_gamma', 3: 'bn_gamma', 4: 'bn_beta'}

# forward planes: direct (reads the master), PACK_FWD, PACK_FWD_IM2COL, the head's conf / loc interleave; data-gradient planes:
# PACK_DGRAD (layer 2 into 1, head into 3), PACK_DGRAD_COL (the stride-2 layer 3 into 2)
REPACK_LAYERS = [conv(16, 3), conv(32, 3), conv(64, 3, stride=2, pads=(1, 1, 1, 1)), head(2)]
REPACK_EXPECT = {1: dict(fwd='direct', dgrad=None), 2: dict(fwd='gemm', dgrad='gemm'), 3: dict(fwd='im2col_gemm', dgrad='strided'),
                 4: dict(fwd='gemm', dgrad='gemm')}
REPACK_LAYOUTS = {'direct': 'master', 'gemm': 'PACK_FWD', 'im2col_gemm': 'PACK_FWD_IM2COL'}
DGRAD_LAYOUTS = {'gemm': 'PACK_DGRAD', 'strided': 'PACK_DGRAD_COL'}

# BatchNormalization: C = 24 / 136 / 64 with ELU / ReLU / none; 100 pixels put 136 channels (17 groups of 8) on bn_grid's
# `blocks = groups` branch, 240 pixels give 24 channels a grid that divides
BN_CASES = [
    dict(name='bn_elu24_relu136_none64_100px', B=1, H=10, W=10, prec='bf16x3',
         layers=[conv(24, 3, act='elu', bn=True), conv(136, 3, bn=True), conv(64, 1, pads='valid', act=None, bn=True)]),
    dict(name='bf16_bn_relu24_elu136_240px', B=2, H=12, W=10, prec='bf16',
         layers=[conv(24, 3, bn=True), conv(136, 3, act='elu', bn=True), conv(24, 1, pads='valid', act=None, bn=True)]),
]

# max-pool: (k, stride, pads) on an H x W input; maxpool2x2_kernel: 2x2/2 without top-left padding; maxpool_kernel: the rest
POOL_CASES = [
    dict(name='pool2x2_even', H=12, W=12, k=2, stride=2, pads=(0, 0, 0, 0), kernel='maxpool2x2'),
    dict(name='pool2x2_same_odd_75', H=75, W=75, k=2, stride=2, pads=(0, 0, 1, 1), kernel='maxpool2x2'),
    dict(name='pool3x3_s1_same', H=11, W=13, k=3, stride=1, pads=(1, 1, 1, 1), kernel='maxpool'),
    dict(name='pool3x3_s2_valid', H=12, W=11, k=3, stride=2, pads=(0, 0, 0, 0), kernel='maxpool'),
]

# L2Normalization: l2norm8_kernel needs C % 8 == 0, C <= 512 and no padding channels; the other two take l2norm_kernel
L2_CASES = [dict(name='l2norm8_c32', C=32, kernel='l2norm8'), dict(name='l2norm_c20_padded', C=20, kernel='l2norm'),
            dict(name='l2norm_c520_wide', C=520, kernel='l2norm')]

PRE_CASES = [dict(name='mean_only', mean=(123.0, 117.0, 104.0), stddev=None, swap=None),
             dict(name='mean_std', mean=(127.5, 110.25, 99.0), stddev=(127.5, 63.0, 58.395), swap=None),
             dict(name='mean_std_bgr', mean=(123.68, 116.779, 103.939), stddev=(58.393, 57.12, 57.375), swap=(2, 1, 0))]


def l2norm_kernel_of(C_, Cs):
    """The kernel launch_l2norm picks for C channels stored in Cs (gamma is a 16-byte aligned device array)."""
    return 'l2norm8' if C_ % 8 == 0 and C_ <= 512 and Cs == C_ else 'l2norm'


def pool_kernel_of(H, W, k, stride, pads):
    """The kernel launch_maxpool picks."""
    Ho, Wo = (H + pads[0] + pads[2] - k) // stride + 1, (W + pads[1] + pads[3] - k) // stride + 1
    fast = k == 2 and stride == 2 and pads[0] == 0 and pads[1] == 0 and 2 * (Ho - 1) < H and 2 * (Wo - 1) < W
    return 'maxpool2x2' if fast else 'maxpool'


def bn_grid(B, H, W, C_, sm_count=cc.SM_COUNT_H100):
    """bn_grid of bn.cu -> (blocks, branch): 1 when a grid of at most (pixels * groups) / 256 blocks keeps every thread on one
    channel group, 2 when it falls back to blocks = groups."""
    groups = (C_ + 7) // 8
    total = B * H * W * groups
    blocks = min((total + 255) // 256, sm_count * 8)
    while blocks > 1 and (blocks * 256) % groups:
        blocks -= 1
    if (blocks * 256) % groups:
        return groups, 2
    return max(blocks, 1), 1


# ------------------------------------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------------------------------------
def _spans(g, n):
    """{(layer, which): (offset, end)} of every parameter span."""
    out = {}
    for i in range(n):
        for which in KIND_OF:
            s = tb._span(g, i, which)
            if s:
                out[(i, which)] = s
    return out


def _seeded_grad(rng, n, prev):
    """A flat gradient with exact zeros, magnitudes from 1e-9 to 1e2 and, where the previous one was non-zero, sign flips."""
    g = rng.choice([-1.0, 1.0], n) * 10.0 ** rng.uniform(-9, 2, n)
    g[rng.random(n) < 0.1] = 0.0
    if prev is not None:
        flip = (rng.random(n) < 0.3) & (prev != 0)
        g[flip] = -prev[flip] * rng.uniform(0.5, 2.0, int(flip.sum()))
    return g.astype(np.float32)


def _judge(record, ratio, perturbed):
    cc.log_ratio(dict(record, ratio=ratio, perturbed={str(k): v for k, v in perturbed.items()}))
    assert ratio <= 1.0, (record, ratio)
    for k, v in perturbed.items():
        assert v > 1.0, (record, 'perturbation %s passes the bound' % (k,), v)


def _hwio(flat, kernel_shape):
    """A kernel span in the gradient's OHWI layout -> the HWIO master."""
    return flat.reshape(kernel_shape).transpose(1, 2, 3, 0)


# ------------------------------------------------------------------------------------------------------------------------------
# the optimiser across steps
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', OPT_CASES, ids=[c['name'] for c in OPT_CASES])
def test_optimizer_updates_across_steps(case):
    import torch
    bc = tb.bcase(case['name'], 1, 10, 10, 3, OPT_LAYERS, {}, prec=case['prec'])
    g, info, _, _ = tb._build(bc)
    try:
        g.trainer()
        n = len(OPT_LAYERS) + 1
        assert g.plan(1)['kernel'] == 'direct'
        spans = _spans(g, n)
        kinds = {KIND_OF[w] for _, w in spans}
        assert kinds == set(KIND_OF.values()), kinds
        shapes = {}
        for (i, w) in spans:
            if w == 0:
                k = info[i]['k']
                shapes[(i, w)] = (info[i]['C'], k, k, info[info[i]['input']]['C'] if info[i]['input'] else bc['cin'])
        # asking for a slot that does not exist is an error; Adam's second moment exists from its first update on
        for bad in (2, -1) + ((1,) if case['optimizer'] == 'adam' else ()):
            with pytest.raises(ValueError, match='slot'):
                g.opt_state(bad)
        rng = np.random.default_rng(11)
        adam = case['optimizer'] == 'adam'
        steps = ADAM_STEPS if adam else SGD_STEPS
        prev = None
        for t, (lr, scale, l2r) in enumerate(steps, start=1):
            gvec = _seeded_grad(rng, g.grad.numel(), prev)
            prev = gvec
            g.grad.copy_(torch.from_numpy(gvec))
            w0, s0 = g.params(), g.opt_state(0)
            s1 = g.opt_state(1) if adam and t > 1 else np.zeros_like(s0)
            g.apply(case['optimizer'], lr, l2=l2r, scale=scale, step=t)
            w1, m1 = g.params(), g.opt_state(0)
            v1 = g.opt_state(1) if adam else None
            assert np.array_equal(g.grad.cpu().numpy(), gvec), 'the update wrote into the gradient buffer'
            if adam:
                perts = [('t+1',), ('eps_in_root',)] + ([('t-1',), ('no_m',), ('no_v',)] if t > 1 else [])
            else:
                perts = [('hwio',)] + ([('no_l2',), ('l2_all',)] if l2r else []) + ([('no_scale',)] if scale != 1 else []) + \
                        ([('no_momentum',)] if t > 1 else [])
            ratio, pr = 0.0, {p: 0.0 for p in perts}
            for key, (o, e) in spans.items():
                ks = shapes.get(key)
                mine = [p for p in perts if not (p in (('hwio',), ('no_l2',)) and ks is None) and not (p == ('l2_all',) and ks)]
                common = dict(l2=l2r, scale=scale, kernel_shape=ks, perturb=mine)
                if adam:
                    ref, bnd, pv = opexact.adam_ref(w0[o:e], s0[o:e], s1[o:e], gvec[o:e], lr, 0.9, 0.999, 1e-8, t, **common)
                    got = {'w': w1[o:e], 'm': m1[o:e], 'v': v1[o:e]}
                else:
                    ref, bnd, pv = opexact.sgd_ref(w0[o:e], s0[o:e], gvec[o:e], lr, 0.9, **common)
                    got = {'w': w1[o:e], 'v': m1[o:e]}
                r = opexact.state_ratio(got, ref, bnd)
                assert r <= 1.0, (case['name'], t, key, KIND_OF[key[1]], r)
                ratio = max(ratio, r)
                for p, rp in pv.items():
                    pr[p] = max(pr[p], opexact.state_ratio(got, rp, bnd))
            _judge(dict(test='optimizer', case=case['name'], step=t, lr=lr, scale=scale, l2=l2r), ratio, pr)
    finally:
        g.close()


# ------------------------------------------------------------------------------------------------------------------------------
# the re-packed planes hold the new master
# ------------------------------------------------------------------------------------------------------------------------------
def _head_split(w, b, nb, C_):
    """A fused head master (HWIO, n_boxes x [C logits | 4 offsets]) -> (conf kernel, conf bias, loc kernel, loc bias)."""
    kh, kw, cin, _ = w.shape
    w5, b2 = w.reshape(kh, kw, cin, nb, C_ + 4), b.reshape(nb, C_ + 4)
    return (w5[..., :C_].reshape(kh, kw, cin, -1), b2[:, :C_].reshape(-1), w5[..., C_:].reshape(kh, kw, cin, -1), b2[:, C_:].reshape(-1))


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
def test_repacked_planes_hold_the_updated_master(prec):
    import torch
    bc = tb.bcase('repack_' + prec, 2, 12, 12, 3, REPACK_LAYERS, {}, prec=prec)
    g, info, x, P = tb._build(bc)
    try:
        n = len(REPACK_LAYERS) + 1
        C_ = bc['C']
        g.trainer()
        for i, e in REPACK_EXPECT.items():
            assert g.plan(i)['kernel'] == e['fwd'], (i, g.plan(i))
            assert g.backward_plan(i)['dgrad'] == e['dgrad'], (i, g.backward_plan(i))
        spans = _spans(g, n)
        w0 = g.params()
        # one SGD step with lr 1 and no momentum moves every parameter by 30 % of its layer's spread
        rng = np.random.default_rng(5)
        gvec = np.zeros_like(w0)
        for (o, e_) in spans.values():
            gvec[o:e_] = rng.standard_normal(e_ - o) * 0.3 * max(float(np.std(w0[o:e_])), 0.05)
        g.grad.copy_(torch.from_numpy(gvec))
        g.apply('sgd', 1.0, momentum=0.0)
        w1 = g.params()
        assert np.array_equal(w1, (w0 - gvec).astype(np.float32))

        def master(flat, i):
            o, e_ = spans[(i, 0)]
            k, cin = info[i]['k'], info[info[i]['input']]['C'] if info[i]['input'] else bc['cin']
            ob, eb = spans[(i, 1)]
            return _hwio(flat[o:e_], (info[i]['C'], k, k, cin)), flat[ob:eb]
        y = g.forward(x, width=C_ + 12)
        fwd = {i: g.read(i) for i in range(n)}
        # the stored planes each layer read (conv_ref multiplies them as they are, without a re-split of hi + lo)
        shape0 = dict(H=bc['H'], W=bc['W'], C=bc['cin'])
        xin = {i: tb._vals(g.planes(i), info[i] if i else shape0) for i in range(n) if i == 0 or info[i]['op'] != 'head'}
        store = 'split' if prec == 'bf16x3' else 'bf16'
        for i in range(1, n):
            inf, plan = info[i], g.plan(i)
            cin = inf['input'] and info[inf['input']]['C'] or bc['cin']
            steps = cc.n_steps_of(plan, inf['k'] ** 2, cin)
            mode = 'fp32' if plan['kernel'] == 'direct' else prec
            geo = dict(stride=inf['stride'], dil=inf['dil'], pads=inf['pads'], mode=mode)
            ratios = {}
            for tag, flat in (('new', w1), ('old', w0)):
                w, b = master(flat, i)
                if inf['op'] == 'head':
                    kc, bcf, kl, bl = _head_split(w, b, inf['nb'], C_)
                    zc, Ac, _ = opexact.conv_ref(xin[inf['input']], kc, bcf, **geo)
                    zl, Al, _ = opexact.conv_ref(xin[inf['input']], kl, bl, **geo)
                    p_ref, p_bnd = opexact.softmax_ref(zc.reshape(bc['B'], P, C_), Ac.reshape(bc['B'], P, C_), steps, C_)
                    l_bnd = opexact.bound(zl.reshape(bc['B'], P, 4), Al.reshape(bc['B'], P, 4), steps, 'f32')
                    ratios[tag] = max(opexact.err_ratio(y[:, :, :C_], p_ref, p_bnd),
                                      opexact.err_ratio(y[:, :, C_:C_ + 4], zl.reshape(bc['B'], P, 4), l_bnd))
                else:
                    yr, A, _ = opexact.conv_ref(xin[inf['input']], w, b, act=inf['act'], **geo)
                    ratios[tag] = opexact.err_ratio(fwd[i], yr, opexact.bound(yr, A, steps, store))
            _judge(dict(test='repack_forward', case=bc['name'], layer=i, layout=REPACK_LAYOUTS[plan['kernel']] + ('+head' if inf['op'] == 'head' else '')),
                   ratios['new'], {('old_master',): ratios['old']})
            assert ratios['old'] > 10.0, (i, 'the pre-update master is within 10x of the bound', ratios)
        # one backward step per layer: the data gradient must use the re-packed data-gradient planes of the new master
        dy = torch.from_numpy(np.random.default_rng(7).standard_normal((bc['B'], P, C_ + 12)).astype(np.float32)).cuda()
        reached = set()
        for i in range(n - 1, 0, -1):
            inf = info[i]
            (pb, _), (pa, _) = g.step(i, dy)
            plan = g.backward_plan(i)
            if plan['dgrad'] is None:
                continue
            pi, pinf = inf['input'], info[inf['input']]
            dz = tb._vals(pa[i], inf)
            taps = inf['k'] ** 2
            kb = -(-pa[i][0].shape[-1] // 64)
            mask = fwd[pi] if plan['dgrad_mask'] else None
            assert not plan['dgrad_accumulate']
            steps = opexact.n_steps_dgrad(plan, taps, kb)
            got = tb._fval(pa[pi], pinf)
            ratios = {}
            for tag, flat in (('new', w1), ('old', w0)):
                w, _ = master(flat, i)
                ref, A, _ = opexact.dgrad_ref(dz, w, (pinf['H'], pinf['W']), stride=inf['stride'], dil=inf['dil'], pads=inf['pads'],
                                              mode=prec, mask=mask)
                ratios[tag] = opexact.err_ratio(got, ref, np.maximum(opexact.bound(ref, A, steps, store), np.finfo(np.float64).tiny))
            _judge(dict(test='repack_dgrad', case=bc['name'], layer=i, layout=DGRAD_LAYOUTS[plan['dgrad']]), ratios['new'],
                   {('old_master',): ratios['old']})
            assert ratios['old'] > 10.0, (i, 'the pre-update master is within 10x of the data-gradient bound', ratios)
            reached.add(DGRAD_LAYOUTS[plan['dgrad']])
            for o in cc.outside(pa[pi], pinf['H'], pinf['W'], pinf['C']):
                assert not np.any(o), (i, 'border / padding channels of the data gradient not zero')
        assert reached == {'PACK_DGRAD', 'PACK_DGRAD_COL'}, reached
    finally:
        g.close()


# ------------------------------------------------------------------------------------------------------------------------------
# training-phase forward launches
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', BN_CASES, ids=[c['name'] for c in BN_CASES])
def test_batchnorm_forward_and_moving_statistics_over_three_passes(case):
    bc = tb.bcase(case['name'], case['B'], case['H'], case['W'], 16, case['layers'], {}, prec=case['prec'])
    g, info, _, _ = tb._build(bc)
    try:
        g.trainer()
        n = len(case['layers']) + 1
        bn_layers = [i for i in range(1, n) if info[i].get('bn_gamma') is not None]
        store = 'split' if case['prec'] == 'bf16x3' else 'bf16'
        rng = np.random.default_rng(21)
        z_prev = {}
        for p in range(3):
            # different inputs each pass; a small spread keeps layer 1's variance near eps, so that dropping eps shows in bf16
            x = (rng.standard_normal((case['B'], case['H'], case['W'], 16)) * (0.1, 0.06, 0.15)[p] + 0.05 * p).astype(np.float32)
            before = {i: g.bn_stats(i, info[i]['C']) for i in bn_layers}
            g.forward(x)
            ratio, pr = 0.0, {}
            for i in bn_layers:
                inf = info[i]
                z = g.read_bn_input(i)
                planes = g.planes(i)
                a = tb._fval(planes, inf)
                mm, mv = g.bn_stats(i, inf['C'])
                perts = [('biased',), ('no_eps',)] + ([('acc',)] if i in z_prev else [])
                ref, A, kap, st, sb, pv = opexact.bn_fwd_ref(z, inf['bn_gamma'], inf['bn_beta'], before[i][0], before[i][1], act=inf['act'],
                                                             z_prev=z_prev.get(i), perturb=perts)
                bnd = kap * A + opexact.UNIT[store] * np.abs(ref)
                got_st = {'mean': mm, 'var': mv}
                r = max(opexact.err_ratio(a, ref, bnd), opexact.state_ratio(got_st, st, sb))
                assert r <= 1.0, (case['name'], p, i, r)
                ratio = max(ratio, r)
                for k, (ap, sp) in pv.items():
                    pr[k] = max(pr.get(k, 0.0), opexact.err_ratio(a, ap, bnd), opexact.state_ratio(got_st, sp, sb))
                for o in cc.outside(planes, inf['H'], inf['W'], inf['C']):
                    assert not np.any(o), (case['name'], p, i, 'border / padding channels not zero')
                z_prev[i] = z
            _judge(dict(test='bn_forward', case=case['name'], pass_=p), ratio, pr)
    finally:
        g.close()


def _tie_input(rng, shape):
    """Values whose hi parts tie within windows while their lo parts differ, both signs: +-h (1 + k 2**-10), h in {1, 2}, k in 0..3
    (hi = +-h exactly); a fifth of them plain normals."""
    h = rng.choice([-2.0, -1.0, 1.0, 2.0], shape)
    x = h * (1.0 + rng.integers(0, 4, shape) * 2.0 ** -10)
    plain = rng.random(shape) < 0.2
    x[plain] = rng.standard_normal(int(plain.sum()))
    return x.astype(np.float32)


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('case', POOL_CASES, ids=[c['name'] for c in POOL_CASES])
def test_maxpool_forward_is_bit_exact(case, prec):
    from ssd_keras_b200 import _ffi
    B, Cc = 2, 16
    assert pool_kernel_of(case['H'], case['W'], case['k'], case['stride'], case['pads']) == case['kernel']
    g = cc.Graph(B, case['H'], case['W'], Cc, [dict(op=_ffi.OP_MAXPOOL, k=case['k'], stride=case['stride'], pads=case['pads'])], prec=prec)
    try:
        x = _tie_input(np.random.default_rng(case['H'] + case['k']), (B, case['H'], case['W'], Cc))
        g.forward(x)
        xin = cc.interior(g.planes(0), case['H'], case['W'], Cc)
        out = g.planes(1)
        Ho, Wo = g.read(1).shape[1:3]
        hi, lo = cc.interior(out, Ho, Wo, Cc)
        pt, pl = case['pads'][:2]
        perts = [('hi_only',), ('lo_tie',)] if prec == 'bf16x3' else []
        rh, rl, pv = opexact.pool_fwd_ref(xin[0], xin[1], case['k'], case['k'], case['stride'], pt, pl, Ho, Wo, perturb=perts)
        same = np.array_equal(hi, rh) and (lo is None or np.array_equal(lo, rl))
        cc.log_ratio(dict(test='pool_forward', case=case['name'], prec=prec, kernel=case['kernel'], bit_exact=same))
        assert same, (case['name'], prec, 'planes differ from the first maximum of hi + lo')
        for p, (ph, pl_) in pv.items():
            assert not (np.array_equal(ph, rh) and np.array_equal(pl_, rl)), (case['name'], p, 'the input has no window the perturbation changes')
        for o in cc.outside(out, Ho, Wo, Cc):
            assert not np.any(o), (case['name'], 'border / padding channels not zero')
    finally:
        g.close()


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('case', L2_CASES, ids=[c['name'] for c in L2_CASES])
def test_l2norm_forward_within_bound(case, prec):
    from ssd_keras_b200 import _ffi
    B, H, W, Cc = 2, 5, 6, case['C']
    rng = np.random.default_rng(Cc)
    gamma = rng.uniform(0.5, 20.0, Cc).astype(np.float32)
    g = cc.Graph(B, H, W, Cc, [dict(op=_ffi.OP_L2NORM, kernel=gamma)], prec=prec)
    try:
        x = rng.standard_normal((B, H, W, Cc)).astype(np.float32)
        x[0, 1, 1] = 0.0                                              # all-zero pixel: the clamp
        x[1, 2, 3] = (rng.standard_normal(Cc) * 1e-8).astype(np.float32)   # sum x^2 < 1e-12: the clamp with a non-zero input
        g.forward(x)
        xin = cc.interior(g.planes(0), H, W, Cc)
        xv = xin[0].astype(np.float64) + (0.0 if xin[1] is None else xin[1])
        assert (xv[1, 2, 3] ** 2).sum() < 1e-12 and np.any(xv[1, 2, 3])
        out = g.planes(1)
        assert l2norm_kernel_of(Cc, g.planes(0)[0].shape[-1]) == case['kernel'] and out[0].shape[-1] == g.planes(0)[0].shape[-1]
        got = tb._fval(out, dict(H=H, W=W, C=Cc))
        ref, err, pv = opexact.l2norm_fwd_ref(xv, gamma, perturb=[('no_gamma',), ('gamma_shift',)])
        store = 'split' if prec == 'bf16x3' else 'bf16'
        bnd = np.maximum(err + opexact.UNIT[store] * np.abs(ref), np.finfo(np.float64).tiny)
        _judge(dict(test='l2norm_forward', case=case['name'], prec=prec, kernel=case['kernel']), opexact.err_ratio(got, ref, bnd),
               {p: opexact.err_ratio(got, v, bnd) for p, v in pv.items()})
        assert not np.any(got[0, 1, 1]) and np.all(np.abs(got[1, 2, 3]) > 0)
        for o in cc.outside(out, H, W, Cc):
            assert not np.any(o), (case['name'], 'border / padding channels not zero')
    finally:
        g.close()


@pytest.mark.parametrize('prec', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('case', PRE_CASES, ids=[c['name'] for c in PRE_CASES])
def test_preprocess_is_bit_exact(case, prec):
    from ssd_keras_b200 import _ffi
    B, H, W = 2, 9, 11
    inp = {k: case[k] for k in ('mean', 'stddev', 'swap')}
    g = cc.Graph(B, H, W, 3, [dict(op=_ffi.OP_MAXPOOL, k=2, stride=2, pads=(0, 0, 0, 0))], prec=prec, input_layer=inp)
    try:
        img = np.random.default_rng(3).uniform(0, 255, (B, H, W, 3)).astype(np.float32)
        img[0, 0, 0] = (123.0, 117.0, 104.0)
        g.forward(img)
        planes = g.planes(0)
        hi, lo = cc.interior(planes, H, W, 3)
        rh, rl = opexact.preprocess_ref(img, case['mean'], case['stddev'], case['swap'])
        same = np.array_equal(hi, rh) and (lo is None or np.array_equal(lo, rl))
        cc.log_ratio(dict(test='preprocess', case=case['name'], prec=prec, bit_exact=same))
        assert same, (case['name'], prec)
        if case['swap'] is not None:
            assert not np.array_equal(hi, opexact.preprocess_ref(img, case['mean'], case['stddev'])[0])
        for o in cc.outside(planes, H, W, 3):
            assert not np.any(o), (case['name'], 'border / padding channels not zero')
    finally:
        g.close()


# ------------------------------------------------------------------------------------------------------------------------------
# an SSDTrainer re-attached after set_weights starts Adam afresh
# ------------------------------------------------------------------------------------------------------------------------------
def test_reattached_adam_trainer_takes_a_fresh_first_step():
    import torch
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.models.keras_ssd7 import build_model
    from ssd_keras_b200.training import SSDTrainer
    sc = [0.08, 0.16, 0.32, 0.64, 0.96]

    def model():
        return build_model((96, 128, 3), 5, mode='training', l2_regularization=5e-4, scales=sc, normalize_coords=True, weights_seed=2,
                           subtract_mean=127.5, divide_by_stddev=127.5)

    def params(tr):
        out = torch.empty_like(tr.grad)
        _ffi.check(_ffi.lib().ssdk_trainer_read_params(tr.handle, _ffi.dptr(out), _ffi.stream_ptr()))
        torch.cuda.synchronize()
        return out.cpu().numpy()
    m = model()
    w0 = m.get_weights()
    tr = SSDTrainer(m, 2, lr=1e-3, optimizer='adam')
    rng = np.random.default_rng(1)
    gvec = torch.from_numpy((rng.standard_normal(tr.n_params) * 0.1).astype(np.float32)).cuda()
    for _ in range(2):
        tr.grad.copy_(gvec)
        tr.apply()
    m.set_weights(w0)
    tr.grad.copy_(gvec)
    tr.apply()
    again = params(tr)
    m2 = model()
    m2.set_weights(w0)
    fresh = SSDTrainer(m2, 2, lr=1e-3, optimizer='adam')
    fresh.grad.copy_(gvec)
    fresh.apply()
    want = params(fresh)
    assert np.array_equal(again, want), ('the re-attached trainer did not take a first step', float(np.abs(again - want).max()))
