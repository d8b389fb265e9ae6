"""Data-parallel training on one GPU: real ranks, real collectives, judged against the single-process kernels and float64.

The ranks are spawned processes on the same H100 under the gloo backend with CUDA tensors (NCCL refuses two ranks on one
device); tests/data_parallel_cases.py holds the models, the cases and the rank worker.  World 2 runs every case of
PAIR_CASES through ``SSDTrainer.train_on_batch`` (the replica and the global loss, SSDLoss and SSDFocalLoss, SGD and Adam,
the single exchange after the backward pass and the bucketed one under it), the global SSDLoss with the k-th hard-negative
value tied across the rank boundary, and the inference gathers.  World 4 runs two data-parallel jobs side by side on the
subgroups {0, 1} and {2, 3}.  Each case is judged in layers, strictest first:
1. each rank's losses and dy equal one single-process launch on the concatenation of the ranks' own y_pred (global), or one
   launch per shard (replica), bit for bit;
2. the reduced gradient equals the sum of the shards' gradients from single-process trainers at the per-rank batch
   (forward bit-identical to the rank's, backward from the rank's dy), bit for bit wherever each gradient element is written
   once; the spans whose kernels add with fp32 atomics (bias gradients, the direct and the split-K weight gradients, the
   L2Normalization and BatchNormalization parameter gradients) are held to the per-launch bounds of oracle/opexact.py;
3. float64 autograd of the oracle graph, at the bars of tests/test_gpu_train.py: the sum of shard means (replica) or the
   whole-batch mean (global); the whole-batch mean must fail replica mode, a normaliser from rank 0's positives global mode;
4. the update: SGD / Adam on the device's reduced gradient times the mode's scale, every rank bit-identical, and each rank's
   BatchNormalization moving statistics following its own shard's batch statistics;
5. all_gather_detections / all_gather_ragged equal the concatenated per-rank outputs.
Ratios go to SSDK_KERNEL_ERRORS_LOG (conv_cases.log_ratio).
"""
import os
import socket
import subprocess
import time

import numpy as np
import pytest

import conv_cases as cc
import data_parallel_cases as dpc
from oracle import opexact

pytestmark = pytest.mark.gpu

SPAWN_TIMEOUT = 900                            # seconds for one spawn's workers, all cases
U32 = opexact.UNIT['f32']


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


_PROCS = []


def _spawn(out_dir, world, which):
    """Runs the workers of one spawn to the end; whatever is still alive after the timeout is terminated, then killed."""
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    port = _free_port()
    procs = [ctx.Process(target=dpc.worker, args=(r, world, port, out_dir, which)) for r in range(world)]
    _PROCS.extend(procs)
    t0 = time.time()
    try:
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=max(1.0, SPAWN_TIMEOUT - (time.time() - t0)))
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(10)
            if p.is_alive():
                p.kill()
                p.join(10)
    print('spawn %s (world %d): %.1f s, exit codes %s' % (which, world, time.time() - t0, [p.exitcode for p in procs]))
    return [p.exitcode for p in procs]


def _tie_inputs():
    import test_gpu_loss_kernel as tlk
    c = tlk.PHASE_CASES[1]                      # phase_ties: dyadic p0 levels, the cut inside image 2 = rank 1's first image
    assert c['name'] == 'phase_ties' and c['B'] == 2 * dpc.PER_RANK
    yt, yp, _, n_neg_min = tlk.make_case(c)
    return yt, yp, n_neg_min


@pytest.fixture(scope='module')
def pairs(tmp_path_factory):
    d = str(tmp_path_factory.mktemp('dp_world2'))
    inp = {}
    # tools/train_check.py's generators and seeds for this graph (images 11, boxes 5): inputs whose float64 comparison holds the
    # 2e-3 bar (elsewhere a pre-activation within rounding of 0 can flip a ReLU and move c2/kernel's gradient by ~2e-3 of its max)
    inp['two_heads_x'], inp['two_heads_y'] = dpc.make_data('two_heads', 2 * dpc.PER_RANK + 1, 11, gt_seed=5)
    inp['ssd7_x'], inp['ssd7_y'] = dpc.make_data('ssd7', 2 * dpc.PER_RANK, 7)
    inp['tie_yt'], inp['tie_yp'], inp['tie_n_neg_min'] = _tie_inputs()
    np.savez(os.path.join(d, 'inputs.npz'), **inp)
    codes = _spawn(d, 2, 'pairs')
    return d, np.load(os.path.join(d, 'inputs.npz')), codes


@pytest.fixture(scope='module')
def groups(tmp_path_factory):
    d = str(tmp_path_factory.mktemp('dp_world4'))
    x, y = dpc.make_data('two_heads', 4 * dpc.PER_RANK, 31)
    np.savez(os.path.join(d, 'inputs.npz'), groups_x=x, groups_y=y)
    codes = _spawn(d, 4, 'groups')
    return d, np.load(os.path.join(d, 'inputs.npz')), codes


def _load(d, name, ranks):
    out = []
    for r in ranks:
        err = os.path.join(d, '%s.r%d.err' % (name, r))
        if os.path.exists(err):
            pytest.fail('rank %d, %s:\n%s' % (r, name, open(err).read()))
        path = os.path.join(d, '%s.r%d.npz' % (name, r))
        if not os.path.exists(path):
            pytest.fail('rank %d wrote nothing for %s (the worker died or timed out)' % (r, name))
        out.append(np.load(path))
    return out


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _n_pos(y):
    return float(np.asarray(y)[..., 1:-12].max(-1).sum())


# ------------------------------------------------------------------------------------------------------------------------------
# 1. loss and dy against one single-process launch
# ------------------------------------------------------------------------------------------------------------------------------
def _launch(kind, yt, yp):
    import torch
    yt_d, yp_d = torch.from_numpy(np.ascontiguousarray(yt)).cuda(), torch.from_numpy(np.ascontiguousarray(yp)).cuda()
    dy = torch.empty_like(yp_d)
    loss = dpc.make_loss(kind).loss_and_grad(yt_d, yp_d, dy, 'replica')
    torch.cuda.synchronize()
    return loss.cpu().numpy(), dy.cpu().numpy()


def judge_loss_and_dy(c, res, ys, other=None):
    """res / ys: the job's ranks' outputs and y_true shards.  other: (results, y_true shards) of every rank of the process
    group, named in the message when the losses equal a launch over them instead of over the job's batch."""
    B = dpc.PER_RANK
    if c['mode'] == 'global':
        L, D = _launch(c['loss'], np.concatenate(ys), np.concatenate([f['y_pred'] for f in res]))
        want = [(L[i * B:(i + 1) * B], D[i * B:(i + 1) * B]) for i in range(len(res))]
    else:
        want = [_launch(c['loss'], y, f['y_pred']) for f, y in zip(res, ys)]
    for i, (f, (l, d)) in enumerate(zip(res, want)):
        if np.array_equal(_bits(f['loss']), _bits(l)) and np.array_equal(_bits(f['dy']), _bits(d)):
            continue
        msg = '%s, rank %d of the job: losses %s, expected %s from one launch over the job\'s %d images (n_positive %g)' % (
            c['name'], i, f['loss'], l, B * len(res), _n_pos(ys) if c['mode'] == 'global' else _n_pos(ys[i]))
        if other is not None:
            ores, oys = other
            Lw, _ = _launch(c['loss'], np.concatenate(oys), np.concatenate([g['y_pred'] for g in ores]))
            k = [j for j, g in enumerate(ores) if g is f][0]
            if np.array_equal(_bits(f['loss']), _bits(Lw[k * B:(k + 1) * B])):
                msg += '; they equal the launch over all %d ranks\' %d images instead: the normaliser counted n_positive %g ' \
                       'and a batch of %d over the whole default group' % (len(ores), B * len(ores), _n_pos(oys), B * len(ores))
        pytest.fail(msg)


# ------------------------------------------------------------------------------------------------------------------------------
# 2. the reduced gradient against single-process trainers at the per-rank batch
# ------------------------------------------------------------------------------------------------------------------------------
class _Probe(cc.Graph):
    """conv_cases.Graph's readers over an SSDTrainer's training plan and native trainer."""

    def __init__(self, tr):
        self.h, self.t, self.B = tr.plan['handle'], tr.handle, tr.batch
        self.split = tr.model.precision == 'bf16x3'
        self.grad = tr.grad


def _fval(planes, shape):
    hi, lo = cc.interior(planes, *shape)
    return hi.astype(np.float64) + (0.0 if lo is None else lo)


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def shard_reference(c, x, yp_worker, dy):
    """One single-process trainer at the per-rank batch: its forward on the shard (bit-identical to the rank's), then the
    backward pass from the rank's dy one layer per call.  -> (flat gradient, {span: (float64 reference, bound)} of the spans
    written with fp32 atomics, the trainer)."""
    import torch
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.training import SSDTrainer
    m, w, _, _ = dpc.build(c['model'])
    tr = SSDTrainer(m, dpc.PER_RANK, lr=dpc.LR, momentum=dpc.MOMENTUM, l2_regularization=dpc.L2, optimizer=c['opt'])
    tr._attach()
    yp = m.forward_device(torch.from_numpy(x).cuda(), training=True)
    torch.cuda.synchronize()
    assert np.array_equal(_bits(yp.cpu().numpy()), _bits(yp_worker)), (c['name'], 'forward of the shard differs from the rank\'s')
    g = _Probe(tr)
    specs = m.specs
    acts = {_ffi.ACT_NONE: None, _ffi.ACT_RELU: 'relu', _ffi.ACT_ELU: 'elu'}

    def shape(i):
        H, W, C_ = m._shapes[i]
        return (H, W, specs[i].n_boxes * (m.n_classes + 4)) if specs[i].op == _ffi.OP_HEAD else (H, W, C_)
    xpl, fwd, bn_z = {}, {}, {}
    for i, s in enumerate(specs):
        if s.op in (_ffi.OP_CONV, _ffi.OP_HEAD):
            pi = m.index[s.inp]
            xpl[pi] = cc.interior(g.planes(pi), *shape(pi))
        if s.op == _ffi.OP_L2NORM:
            fwd[m.index[s.inp]] = g.read(m.index[s.inp])
        if s.op == _ffi.OP_CONV and s.bn:
            bn_z[i], fwd[i] = g.read_bn_input(i), g.read(i)
    dyt = torch.from_numpy(dy).cuda()
    refs = {}
    sm = _sm_count()
    mode = m.precision
    for i in range(len(specs) - 1, 0, -1):
        s = specs[i]
        bn = s.op == _ffi.OP_CONV and bool(s.bn)
        before = _fval(g.grad_planes(i), shape(i)) if bn or s.op == _ffi.OP_L2NORM else None
        tr._backward_layers(dyt, i, i)
        torch.cuda.synchronize()
        if bn:
            _, _, _, dgam, dbet, Ag, Ab, kp, _ = opexact.bn_bwd_ref(bn_z[i], fwd[i], before, w[s.bn + '/gamma'], act=acts[s.act])
            refs[(s.name, 'bn_gamma')] = (dgam, kp * Ag + U32 * np.abs(dgam))
            refs[(s.name, 'bn_beta')] = (dbet, kp * Ab + U32 * np.abs(dbet))
        if s.op in (_ffi.OP_CONV, _ffi.OP_HEAD):
            plan = g.backward_plan(i)
            pi = m.index[s.inp]
            dz = cc.interior(g.grad_planes(i), *shape(i))
            H, W, C_ = shape(i)
            geo = dict(stride=s.stride, dil=s.dilation, pads=tuple(s.pad))
            if plan['wgrad'] == 'direct':
                steps = opexact.n_steps_wgrad_direct(dpc.PER_RANK, H, W, C_, plan['direct_fast'], sm)
                ref, A, _ = opexact.wgrad_ref(xpl[pi], dz, s.kh, s.kw, mode='fp32', **geo)
                refs[(s.name, 'kernel')] = (ref.reshape(-1), opexact.bound(ref, A, steps, 'f32').reshape(-1))
            elif not (plan['wgrad'] == 'native' and plan['k_split'] == 1):       # several CTAs add into one element
                ref, A, _ = opexact.wgrad_ref(xpl[pi], dz, s.kh, s.kw, mode=mode, **geo)
                steps = opexact.n_steps_wgrad(plan, 3 if mode == 'bf16x3' else 1)
                refs[(s.name, 'kernel')] = (ref.reshape(-1), opexact.bound(ref, A, steps, 'f32').reshape(-1))
            ref, A, nb_, _ = opexact.bias_grad_ref(dz)                            # per-block partials, fp32 atomics
            refs[(s.name, 'bias')] = (ref, opexact.bound(ref, A, nb_ + 1, 'f32'))
        if s.op == _ffi.OP_L2NORM:
            pi = m.index[s.inp]
            relu = specs[pi].op == _ffi.OP_CONV and specs[pi].act == _ffi.ACT_RELU
            _, _, _, gref, gA, gsteps, _ = opexact.l2norm_bwd_ref(fwd[pi], before, w[s.name + '/gamma'], relu_mask=relu)
            refs[(s.name, 'gamma')] = (gref, opexact.bound(gref, gA, gsteps, 'f32'))
    torch.cuda.synchronize()
    return tr.grad.cpu().numpy(), refs, tr


def judge_reduced_gradient(c, res, xs):
    """-> (the reduced gradient, a reference trainer, the span table, the atomic spans).  Every rank of the job holds the same
    bits; spans written once equal the float32 sum of the shards' gradients bit for bit, atomic spans are within the sum of
    the shards' bounds plus the rounding of the sum."""
    for f in res[1:]:
        assert np.array_equal(_bits(f['grad']), _bits(res[0]['grad'])), (c['name'], 'ranks disagree on the reduced gradient')
    shards = [shard_reference(c, x, f['y_pred'], f['dy']) for x, f in zip(xs, res)]
    tr = shards[0][2]
    spans = tr.spans()
    acc = shards[0][0].copy()
    for gr, _, _ in shards[1:]:
        acc = (acc + gr).astype(np.float32)                  # gloo's sum: a + b, the one float32 addition of 2 ranks
    got = res[0]['grad']
    atomic = set(shards[0][1])
    worst = 0.0
    for key, (o, n) in spans.items():
        if key in atomic:
            ref = sum(s[1][key][0] for s in shards)
            bnd = sum(s[1][key][1] for s in shards)
            bnd = np.maximum(bnd + U32 * (np.abs(ref) + bnd), np.finfo(np.float64).tiny)
            r = opexact.err_ratio(got[o:o + n].astype(np.float64), np.asarray(ref, np.float64).reshape(-1), np.asarray(bnd).reshape(-1))
            worst = max(worst, r)
            assert r <= 1.0, (c['name'], key, 'reduced atomic span outside the sum of the per-launch bounds', r)
        else:
            bad = np.flatnonzero(_bits(got[o:o + n]) != _bits(acc[o:o + n]))
            assert bad.size == 0, (c['name'], key, '%d of %d elements differ from the sum of the shards\' gradients, first at %d: %r vs %r'
                                   % (bad.size, n, bad[0], got[o + bad[0]], acc[o + bad[0]]))
    cc.log_ratio({'test': 'data_parallel', 'case': c['name'], 'what': 'reduced_gradient_atomic_spans', 'ratio': worst,
                  'n_atomic_spans': len(atomic), 'n_exact_spans': len(spans) - len(atomic)})
    return got, tr, spans, atomic


# ------------------------------------------------------------------------------------------------------------------------------
# 3. float64 autograd
# ------------------------------------------------------------------------------------------------------------------------------
def autograd(c, xs, ys, objective):
    """-> (per-image losses of each shard, {weight: gradient}, [BatchNormalization batch statistics of each shard]) of the
    objective 'replica' (the sum of the shard means) or 'global' (the mean over the whole batch), float64.  Every shard runs
    the forward on its own (BatchNormalization normalises with its own shard's statistics, as each rank does)."""
    import torch
    import focal_reference as fr
    from oracle import graph as og
    m, w, _, var = dpc.build(c['model'])
    params = og.make_params(m.specs, w, dtype=torch.float64)
    fw = [og.forward(m.specs, params, x, m.n_classes, m.anchors, var, dtype=torch.float64, bn_training=c['model'] == 'ssd7') for x in xs]
    yps = [f[0] for f in fw]
    if c['loss'] == 'ssd':
        if objective == 'replica':
            lv = [og.ssd_loss_torch(y, yp) for y, yp in zip(ys, yps)]
            sum(l.mean() for l in lv).backward()
            losses = [l.detach().numpy() for l in lv]
        else:
            lv = og.ssd_loss_torch(np.concatenate(ys), torch.cat(yps))
            lv.mean().backward()
            losses = np.split(lv.detach().numpy(), len(ys))
    else:
        if objective == 'replica':
            losses = [fr.focal_loss(y, yp.detach().numpy()) for y, yp in zip(ys, yps)]
            torch.autograd.backward(yps, [torch.from_numpy(fr.focal_loss_grad(y, yp.detach().numpy())) for y, yp in zip(ys, yps)])
        else:
            yp_all = torch.cat(yps)
            y_all = np.concatenate(ys)
            losses = np.split(fr.focal_loss(y_all, yp_all.detach().numpy()), len(ys))
            yp_all.backward(torch.from_numpy(fr.focal_loss_grad(y_all, yp_all.detach().numpy())))
    grads = {k: p.grad.numpy() for k, p in params.items() if p.grad is not None}
    return losses, grads, [f[1] for f in fw], m, w


def _grad_ratios(dev, ref, skip):
    """{tensor: max |dev - ref| / (2e-3 max |ref|)}."""
    return {k: float(np.abs(dev[k] - v).max() / (2e-3 * (np.abs(v).max() + 1e-30))) for k, v in ref.items() if k not in skip}


def _grad_ratio(dev, ref, skip):
    return max(_grad_ratios(dev, ref, skip).values())


# ------------------------------------------------------------------------------------------------------------------------------
# the cases
# ------------------------------------------------------------------------------------------------------------------------------
def test_gloo_takes_every_collective_on_cuda_tensors(pairs):
    d, _, _ = pairs
    for r, f in enumerate(_load(d, 'probe', (0, 1))):
        bad = {k: str(f[k]) for k in f.files if str(f[k]) != 'ok'}
        assert not bad, ('rank %d' % r, bad)


@pytest.mark.parametrize('c', dpc.PAIR_CASES, ids=[c['name'] for c in dpc.PAIR_CASES])
def test_data_parallel_step(pairs, c):
    d, inp, _ = pairs
    res = _load(d, c['name'], (0, 1))
    B = dpc.PER_RANK
    xs = [inp[c['model'] + '_x'][r * B:(r + 1) * B] for r in range(2)]
    ys = [inp[c['model'] + '_y'][r * B:(r + 1) * B] for r in range(2)]
    if c['overlap']:
        assert all(int(f['n_buckets']) >= 3 for f in res), (c['name'], [int(f['n_buckets']) for f in res])
    # 1.
    judge_loss_and_dy(c, res, ys)
    # 2.
    got, tr, spans, atomic = judge_reduced_gradient(c, res, xs)
    # 3.
    losses, ref_g, bn_stats, m, w = autograd(c, xs, ys, c['mode'])
    for f, l in zip(res, losses):
        assert np.abs(f['loss'] - l).max() <= 1e-4 * np.abs(np.concatenate(losses)).max(), (c['name'], f['loss'], l)
    dev_g = tr._unflatten(got)
    assert set(dev_g) == set(ref_g), (c['name'], set(dev_g) ^ set(ref_g))
    # a bias in front of a BatchNormalization has an exactly zero gradient; float64 leaves rounding noise there (layer 2 holds it)
    skip = {s.name + '/bias' for s in m.specs if getattr(s, 'bn', None)}
    rs_ = _grad_ratios(dev_g, ref_g, skip)
    r = max(rs_.values())
    assert r <= 1.0, (c['name'], 'reduced gradient against float64 autograd', {k: v for k, v in rs_.items() if v > 0.5})
    if c['mode'] == 'replica':
        _, pert_g, _, _, _ = autograd(c, xs, ys, 'global')
        pert = {'whole_batch_mean': _grad_ratio(dev_g, pert_g, skip)}
    else:
        f0 = max(1.0, _n_pos(np.concatenate(ys))) / max(1.0, _n_pos(ys[0]))
        pert = {'rank0_positives': _grad_ratio(dev_g, {k: v * f0 for k, v in ref_g.items()}, skip)}
    # 4. the update, on the device's reduced gradient times the mode's scale
    scale = 1.0 / len(res) if c['mode'] == 'replica' else 1.0
    trainable = {k: v for k, v in w.items() if not k.endswith(('/moving_mean', '/moving_variance'))}
    new_w = [dpc.unnamed(f, 'w:') for f in res]
    slots = [[dpc.unnamed(f, 's%d:' % i) for i in range(int(f['n_slots']))] for f in res]
    for f in res[1:]:
        assert np.array_equal(_bits(f['params']), _bits(res[0]['params'])), (c['name'], 'ranks disagree on the weights')
    from oracle import graph as og

    def update_ratio(sc):
        g = {k: dev_g[k].astype(np.float64) * sc for k in trainable}
        if c['opt'] == 'sgd':
            ref_w, ref_v = og.sgd_step(trainable, g, {}, dpc.LR, dpc.MOMENTUM, dpc.L2)
            ref_s = [ref_v]
        else:
            f32 = lambda v: float(np.float32(v))           # the hyper-parameters as the device holds them
            ref_w, ref_m, ref_v = og.adam_step(trainable, g, {}, {}, 1, lr=f32(dpc.LR), beta_1=f32(0.9), beta_2=f32(0.999),
                                               epsilon=f32(1e-8), l2_reg=f32(dpc.L2))
            ref_s = [ref_m, ref_v]
        rw = max(float(np.abs(new_w[0][k] - ref_w[k]).max() / (2e-6 * np.abs(ref_w[k]).max() + 1e-9)) for k in trainable)
        rs = max(float(np.abs(slots[0][i][k] - ref[k]).max() / (2e-6 * np.abs(ref[k]).max() + 1e-30))
                 for i, ref in enumerate(ref_s) for k in trainable)
        return rw, rs
    rw, rs = update_ratio(scale)
    assert rw <= 1.0 and rs <= 1.0, (c['name'], 'update', rw, rs)
    pw, ps = update_ratio(1.0 / len(res) if scale == 1.0 else 1.0)
    pert['wrong_scale'] = max(pw, ps)
    cc.log_ratio({'test': 'data_parallel', 'case': c['name'], 'what': 'autograd_and_update', 'ratio': max(r, rw, rs),
                  'perturbed': pert})
    for p, v in pert.items():
        assert v > 1.0, (c['name'], 'perturbation %s passes' % p, v)
    # BatchNormalization: each rank's moving statistics follow the recurrence of its own shard's batch statistics
    for s in m.specs:
        if getattr(s, 'bn', None):
            H, W_, _ = m._shapes[m.index[s.name]]
            n = float(B * H * W_)
            for rank, (nw, outs) in enumerate(zip(new_w, bn_stats)):
                mu, var = outs[s.bn + '/batch_mean'].numpy(), outs[s.bn + '/batch_var'].numpy()
                np.testing.assert_allclose(nw[s.bn + '/moving_mean'], 0.99 * w[s.bn + '/moving_mean'] + 0.01 * mu, rtol=1e-4, atol=1e-5)
                np.testing.assert_allclose(nw[s.bn + '/moving_variance'], 0.99 * w[s.bn + '/moving_variance'] + 0.01 * var * n / (n - 1.0),
                                           rtol=1e-4, atol=1e-5)
            assert not np.array_equal(new_w[0][s.bn + '/moving_mean'], new_w[1][s.bn + '/moving_mean']), s.bn


def test_global_loss_ties_across_the_rank_boundary(pairs):
    """The k-th largest negative loss is a value several boxes share, and the boxes kept at it are some of rank 1's, all of
    rank 0's: the tie gather must hand each rank its place in the global order."""
    import test_gpu_loss_kernel as tlk
    d, inp, _ = pairs
    res = _load(d, 'ties', (0, 1))
    yt, yp, n_neg_min = inp['tie_yt'], inp['tie_yp'], int(inp['tie_n_neg_min'])
    B = dpc.PER_RANK
    negl = tlk.box_losses_f32(yt, yp)[1]
    flat = negl.reshape(-1)
    v = np.sort(flat)[::-1][n_neg_min - 1]
    ties = [int(np.sum(negl[r * B:(r + 1) * B] == v)) for r in range(2)]
    kept_at_v = n_neg_min - int(np.sum(flat > v))
    assert kept_at_v - ties[0] > 0 and kept_at_v - ties[0] < ties[1], (ties, kept_at_v)
    import torch
    yt_d, yp_d = torch.from_numpy(yt).cuda(), torch.from_numpy(yp).cuda()
    dy = torch.empty_like(yp_d)
    L = dpc.make_loss('ssd', n_neg_min).loss_and_grad(yt_d, yp_d, dy, 'replica').cpu().numpy()
    D = dy.cpu().numpy()
    for r, f in enumerate(res):
        assert np.array_equal(_bits(f['y_pred']), _bits(yp[r * B:(r + 1) * B]))
        assert np.array_equal(_bits(f['loss']), _bits(L[r * B:(r + 1) * B])), (r, f['loss'], L)
        assert np.array_equal(_bits(f['dy']), _bits(D[r * B:(r + 1) * B])), r


def test_inference_gathers(pairs):
    d, _, _ = pairs
    res = _load(d, 'gather', (0, 1))
    full = np.concatenate([f['local'] for f in res])
    ragged = np.concatenate([f['ragged_local'] for f in res])
    assert [f['ragged_local'].shape[0] for f in res] == [3, 2]
    for f in res:
        assert np.array_equal(_bits(f['gathered']), _bits(full))
        assert np.array_equal(_bits(f['ragged']), _bits(ragged))


@pytest.mark.parametrize('c', dpc.GROUP_CASES, ids=[c['name'] for c in dpc.GROUP_CASES])
def test_two_jobs_on_subgroups(groups, c):
    """Two data-parallel jobs of 2 ranks in one world of 4: each job's loss, dy and reduced gradient are those of its own
    batch alone, and the replica update is scaled by 1 / (the job's 2 ranks)."""
    d, inp, _ = groups
    res = _load(d, c['name'], range(4))
    B = dpc.PER_RANK
    xs = [inp['groups_x'][r * B:(r + 1) * B] for r in range(4)]
    ys = [inp['groups_y'][r * B:(r + 1) * B] for r in range(4)]
    for members in dpc.GROUPS:
        job = [res[r] for r in members]
        judge_loss_and_dy(c, job, [ys[r] for r in members], other=(res, ys))
        got, tr, _, _ = judge_reduced_gradient(c, job, [xs[r] for r in members])
        if c['mode'] == 'replica':
            from oracle import graph as og
            _, w, _, _ = dpc.build(c['model'])
            dev_g = tr._unflatten(got)
            trainable = {k: v for k, v in w.items() if not k.endswith(('/moving_mean', '/moving_variance'))}
            new_w = dpc.unnamed(job[0], 'w:')

            def ratio(sc):
                ref_w, _ = og.sgd_step(trainable, {k: dev_g[k] * sc for k in trainable}, {}, dpc.LR, dpc.MOMENTUM, dpc.L2)
                return max(float(np.abs(new_w[k] - ref_w[k]).max() / (2e-6 * np.abs(ref_w[k]).max() + 1e-9)) for k in trainable)
            r_half, r_quarter = ratio(0.5), ratio(0.25)
            cc.log_ratio({'test': 'data_parallel', 'case': c['name'], 'what': 'update_scale', 'ratio': r_half,
                          'perturbed': {'scale_1/4': r_quarter}})
            assert r_half <= 1.0 < r_quarter, (c['name'], members, r_half, r_quarter)


def test_no_worker_outlives_the_module(pairs, groups):
    """Last: every spawned rank has exited cleanly, and no process spawned by this one is left."""
    assert _PROCS and not any(p.is_alive() for p in _PROCS)
    assert pairs[2] == [0, 0] and groups[2] == [0, 0, 0, 0], (pairs[2], groups[2])
    try:
        r = subprocess.run(['pgrep', '-P', str(os.getpid()), '-f', 'spawn_main'], capture_output=True, text=True)
        left = r.stdout.split()
    except FileNotFoundError:                   # no pgrep: the parent pids of /proc
        left = []
        for pid in filter(str.isdigit, os.listdir('/proc')):
            try:
                stat = open('/proc/%s/stat' % pid).read()
                cmd = open('/proc/%s/cmdline' % pid).read()
            except OSError:
                continue
            if int(stat.rsplit(')', 1)[1].split()[1]) == os.getpid() and 'spawn_main' in cmd:
                left.append(pid)
    assert not left, 'worker processes still running: %s' % left
