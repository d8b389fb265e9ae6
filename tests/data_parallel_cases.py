"""The models, data and rank workers of tests/test_gpu_data_parallel.py: real multi-process data parallelism on ONE GPU.

NCCL refuses two ranks on one device, so the ranks run the gloo backend on CUDA tensors.  A worker runs every case of its
spawn on its own shard and writes what it produced (losses, y_pred, dy, the reduced flat gradient, the updated weights, the
optimiser state, the BatchNormalization moving statistics) to ``<out>/<case>.r<rank>.npz``, or the error it met to
``<out>/<case>.r<rank>.err``; the parent process judges.  The inputs come from ``<out>/inputs.npz``, written by the parent.
"""
import importlib.util
import os
import traceback

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
PER_RANK = 2                                   # images per rank
LR, MOMENTUM, L2 = 1e-3, 0.9, 5e-4


def case(name, model, loss, mode, opt, overlap):
    return dict(name=name, model=model, loss=loss, mode=mode, opt=opt, overlap=overlap)


# world 2: (model, loss, loss_mode, optimizer, exchange); overlap False = one all-reduce after the backward pass, True = buckets
PAIR_CASES = [case('%s_%s_%s_%s' % (m, l, mo, 'bucketed' if ov else 'single'), m, l, mo, o, ov)
              for m, l, o, modes, ovs in (('two_heads', 'ssd', 'sgd', ('replica', 'global'), (False, True)),
                                          ('two_heads', 'focal', 'sgd', ('replica', 'global'), (True,)),
                                          ('ssd7', 'ssd', 'adam', ('replica', 'global'), (False, True)))
              for mo in modes for ov in ovs]
# world 4, two data-parallel jobs of 2 ranks each on the subgroups {0, 1} and {2, 3}
GROUP_CASES = [case('groups_two_heads_ssd_global', 'two_heads', 'ssd', 'global', 'sgd', None),
               case('groups_two_heads_focal_global', 'two_heads', 'focal', 'global', 'sgd', None),
               case('groups_two_heads_ssd_replica', 'two_heads', 'ssd', 'replica', 'sgd', None)]
GROUPS = ([0, 1], [2, 3])


def _train_check():
    spec = importlib.util.spec_from_file_location('train_check', os.path.join(ROOT, 'tools', 'train_check.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def build(model):
    """-> (model, initial weights, number of classes incl. background, variances).  two_heads: tools/train_check.py's
    ``two_heads_l2norm`` (conv, L2Normalization, two heads, a pool); ssd7: SSD7 at 96x128 (conv + BatchNormalization + ELU)."""
    if model == 'two_heads':
        tc = _train_check()
        m, w, n_cls = tc.build(tc.CASES[2])
        return m, w, n_cls, [0.1, 0.1, 0.2, 0.2]
    from ssd_keras_b200.models.keras_ssd7 import build_model
    sc = [0.08, 0.16, 0.32, 0.64, 0.96]
    m = build_model((96, 128, 3), 5, mode='training', l2_regularization=L2, scales=sc, normalize_coords=True, weights_seed=4,
                    subtract_mean=127.5, divide_by_stddev=127.5)
    w = m.get_weights()
    rng = np.random.default_rng(3)
    for k in w:
        if k.endswith('/bias'):
            w[k] = (rng.standard_normal(w[k].shape) * 0.05).astype(np.float32)
        elif k.endswith('/gamma'):
            w[k] = rng.uniform(0.8, 1.2, w[k].shape).astype(np.float32)
        elif k.endswith('/beta'):
            w[k] = (rng.standard_normal(w[k].shape) * 0.1).astype(np.float32)
        elif k.endswith('/moving_mean'):
            w[k] = (rng.standard_normal(w[k].shape) * 0.1).astype(np.float32)
    m.set_weights(w)
    return m, w, 6, [1.0] * 4


def make_data(model, n_images, seed, gt_seed=None):
    """-> (images, y_true) float32 for ``n_images`` images of the model's input size; the ground truth from ``gt_seed``
    (default ``seed + 1``)."""
    from oracle import synth
    from oracle.encoder import OracleEncoder
    m, _, n_cls, _ = build(model)
    gt_seed = seed + 1 if gt_seed is None else gt_seed
    if model == 'two_heads':
        tc = _train_check()
        hw = tc.CASES[2][1]
        rng = np.random.default_rng(seed)
        x = rng.integers(0, 256, size=(n_images, hw, hw, 3)).astype(np.float32)
        enc = OracleEncoder(hw, hw, n_cls - 1, m.predictor_sizes, scales=m.anchor_cfg['scales'],
                            aspect_ratios_per_layer=m.anchor_cfg['aspect_ratios_per_layer'], variances=[0.1, 0.1, 0.2, 0.2],
                            pos_iou_threshold=0.3, neg_iou_limit=0.2)
        y = enc(tc.small_gt(gt_seed, n_images, 3, hw, n_cls - 1))
    else:
        H, W = 96, 128
        enc = OracleEncoder(H, W, n_cls - 1, m.predictor_sizes, scales=m.anchor_cfg['scales'], aspect_ratios_global=[0.5, 1.0, 2.0],
                            variances=[1.0] * 4, pos_iou_threshold=0.4, neg_iou_limit=0.3, normalize_coords=True)
        x = synth.synth_images(seed, n_images, H, W)
        y = enc(synth.synth_gt(gt_seed, n_images, 3, W, H, n_cls - 1))
    assert np.array_equal(enc.anchors, m.anchors)
    return x.astype(np.float32), y.astype(np.float32)


def make_loss(kind, n_neg_min=0):
    from ssd_keras_b200.keras_loss_function.keras_ssd_focal_loss import SSDFocalLoss
    from ssd_keras_b200.keras_loss_function.keras_ssd_loss import SSDLoss
    return SSDLoss(n_neg_min=n_neg_min) if kind == 'ssd' else SSDFocalLoss()


def _flat_params(tr, fn, *args):
    import torch
    from ssd_keras_b200 import _ffi
    out = torch.empty_like(tr.grad)
    _ffi.check(fn(tr.handle, *args, _ffi.dptr(out), _ffi.stream_ptr()))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _named(prefix, d):
    return {prefix + k.replace('/', '|'): np.asarray(v) for k, v in d.items()}


def unnamed(f, prefix):
    """The Keras-named arrays an npz holds under ``prefix`` (the inverse of ``_named``)."""
    return {k[len(prefix):].replace('|', '/'): f[k] for k in f.files if k.startswith(prefix)}


def run_train_case(c, x, y, group, out_path):
    """One training step of case ``c`` on this rank's shard ``x`` / ``y`` through ``SSDTrainer.train_on_batch(group=group)``."""
    import torch
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.training import SSDTrainer
    m, _, _, _ = build(c['model'])
    tr = SSDTrainer(m, PER_RANK, lr=LR, momentum=MOMENTUM, l2_regularization=L2, loss_mode=c['mode'], optimizer=c['opt'],
                    loss=make_loss(c['loss']))
    n_buckets = 0
    if c['overlap']:
        tr.bucket_bytes = 4                    # every layer with parameters closes its own bucket
        n_buckets = len([b for b in tr.buckets() if b[3]])
    seen = {}
    inner = tr.loss.loss_and_grad

    def spy(y_true, y_pred, grad_out, loss_mode='replica', group=None):
        seen['y_pred'] = y_pred.clone()        # the y_pred the step's loss read
        return inner(y_true, y_pred, grad_out, loss_mode, group=group)
    tr.loss.loss_and_grad = spy
    loss = tr.train_on_batch(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), group=group, overlap=c['overlap'])
    torch.cuda.synchronize()
    st = tr.get_optimizer_state()
    out = dict(loss=loss.cpu().numpy(), y_pred=seen['y_pred'].cpu().numpy(), dy=tr._dy.cpu().numpy(), grad=tr.grad.cpu().numpy(),
               params=_flat_params(tr, _ffi.lib().ssdk_trainer_read_params), n_buckets=np.int64(n_buckets),
               n_slots=np.int64(len(st['slots'])))
    out.update(_named('w:', tr.get_weights()))
    for i, slot in enumerate(st['slots']):
        out.update(_named('s%d:' % i, slot))
    np.savez(out_path, **out)


def run_tie_case(inp, rank, out_path):
    """SSDLoss.loss_and_grad(..., 'global') on y_pred given directly: the k-th hard-negative value ties across the ranks."""
    import torch
    yt = torch.from_numpy(inp['tie_yt'][rank * PER_RANK:(rank + 1) * PER_RANK]).cuda()
    yp = torch.from_numpy(inp['tie_yp'][rank * PER_RANK:(rank + 1) * PER_RANK]).cuda()
    dy = torch.empty_like(yp)
    loss = make_loss('ssd', int(inp['tie_n_neg_min'])).loss_and_grad(yt, yp, dy, 'global')
    torch.cuda.synchronize()
    np.savez(out_path, loss=loss.cpu().numpy(), dy=dy.cpu().numpy(), y_pred=yp.cpu().numpy())


def run_probe(rank, world, out_path):
    """Every collective the library issues, on CUDA tensors under gloo: sync and async all_reduce (float32, int32, int64),
    all_gather_into_tensor (int32) and the list all_gather (int64) -> 'ok' or the error, per call."""
    import torch
    import torch.distributed as dist
    res = {}
    for dt in (torch.float32, torch.int32, torch.int64):
        for async_op in (False, True):
            key = 'all_reduce_%s_%s' % (str(dt).split('.')[-1], 'async' if async_op else 'sync')
            try:
                t = torch.arange(5, device='cuda').to(dt) * (rank + 1)
                w = dist.all_reduce(t, async_op=async_op)
                if async_op:
                    w.wait()
                want = torch.arange(5, device='cuda').to(dt) * sum(range(1, world + 1))
                res[key] = 'ok' if t.is_cuda and torch.equal(t, want) else 'wrong result %s' % t.cpu().tolist()
            except Exception as e:                     # the parent reports which collective gloo refused
                res[key] = 'error: %r' % (e,)
    try:
        t = torch.tensor([rank + 7], dtype=torch.int32, device='cuda')
        o = torch.zeros((world,), dtype=torch.int32, device='cuda')
        dist.all_gather_into_tensor(o, t)
        res['all_gather_into_tensor_int32'] = 'ok' if o.cpu().tolist() == [r + 7 for r in range(world)] else 'wrong result %s' % o.cpu().tolist()
    except Exception as e:
        res['all_gather_into_tensor_int32'] = 'error: %r' % (e,)
    try:
        t = torch.tensor([rank + 3], dtype=torch.int64, device='cuda')
        lst = [torch.zeros_like(t) for _ in range(world)]
        dist.all_gather(lst, t)
        res['all_gather_list_int64'] = 'ok' if [int(v.item()) for v in lst] == [r + 3 for r in range(world)] else 'wrong result'
    except Exception as e:
        res['all_gather_list_int64'] = 'error: %r' % (e,)
    np.savez(out_path, **{k: np.array(v) for k, v in res.items()})


def run_gather(inp, rank, out_path):
    """Inference gather: all_gather_detections of predict_device on equal shards, all_gather_ragged on a 3 / 2 split."""
    import torch
    from ssd_keras_b200.distributed import all_gather_detections, all_gather_ragged
    m, _, _, _ = build('two_heads')
    x = inp['two_heads_x']
    local = m.predict_device(torch.from_numpy(x[rank * PER_RANK:(rank + 1) * PER_RANK]).cuda())
    got = all_gather_detections(local)
    lo, hi = ((0, 3), (3, 5))[rank]
    ragged_local = m.predict_device(torch.from_numpy(x[lo:hi]).cuda())
    ragged = all_gather_ragged(ragged_local)
    torch.cuda.synchronize()
    np.savez(out_path, local=local.cpu().numpy(), gathered=got.cpu().numpy(), ragged_local=ragged_local.cpu().numpy(),
             ragged=ragged.cpu().numpy())


def _attempt(out_dir, name, rank, fn, *args):
    try:
        fn(*args, os.path.join(out_dir, '%s.r%d.npz' % (name, rank)))
    except Exception:
        with open(os.path.join(out_dir, '%s.r%d.err' % (name, rank)), 'w') as f:
            f.write(traceback.format_exc())


def worker(rank, world, port, out_dir, which):
    """The body of one spawned rank.  which: 'pairs' (world 2: the probe, PAIR_CASES, the tie case, the gathers) or 'groups'
    (world 4: GROUP_CASES on two subgroups)."""
    from datetime import timedelta
    import sys
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(0)
    dist.init_process_group('gloo', rank=rank, world_size=world, timeout=timedelta(seconds=120))
    try:
        inp = np.load(os.path.join(out_dir, 'inputs.npz'))
        if which == 'pairs':
            _attempt(out_dir, 'probe', rank, run_probe, rank, world)
            for c in PAIR_CASES:
                sl = slice(rank * PER_RANK, (rank + 1) * PER_RANK)
                _attempt(out_dir, c['name'], rank, run_train_case, c, inp[c['model'] + '_x'][sl], inp[c['model'] + '_y'][sl], None)
                dist.barrier()
            _attempt(out_dir, 'ties', rank, run_tie_case, inp, rank)
            dist.barrier()
            _attempt(out_dir, 'gather', rank, run_gather, inp, rank)
        else:
            groups = [dist.new_group(g) for g in GROUPS]
            mine = groups[rank // 2]
            for c in GROUP_CASES:
                sl = slice(rank * PER_RANK, (rank + 1) * PER_RANK)
                _attempt(out_dir, c['name'], rank, run_train_case, c, inp['groups_x'][sl], inp['groups_y'][sl], mine)
                dist.barrier()
        dist.barrier()
    finally:
        dist.destroy_process_group()
