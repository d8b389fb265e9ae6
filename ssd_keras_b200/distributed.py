"""Multi-GPU plumbing for the one place the path shards: by image (SURVEY.md section 8e).

One process per GPU under torchrun / torch.distributed.  The forward pass, the encoder and the decoders are independent per
image, so ranks exchange nothing on the data path; the only collective in inference is an all-gather of the fixed-size
``(B_local, top_k, 6)`` decoded boxes (plus counts) so that every rank (or rank 0) sees the whole batch.
Works with the 'nccl' backend on CUDA tensors and with 'gloo' on CPU tensors (used by the CPU tests).
"""


def shard_bounds(n_items, rank, world):
    """Contiguous, balanced split of ``n_items`` images: the first ``n_items % world`` ranks get one extra."""
    base, rem = divmod(int(n_items), int(world))
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def init_from_env(device_index=None):
    """Initialise torch.distributed from RANK / WORLD_SIZE / MASTER_* (torchrun).  Returns (rank, world)."""
    import os
    import torch
    import torch.distributed as dist
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    if world > 1 and not dist.is_initialized():
        if torch.cuda.is_available():
            dev = torch.device('cuda', device_index if device_index is not None else int(os.environ.get('LOCAL_RANK', '0')))
            dist.init_process_group('nccl', device_id=dev)
        else:
            dist.init_process_group('gloo')
    return rank, world


def all_gather_detections(local, group=None):
    """``local``: (B_local, top_k, 6) tensor, the same shape on every rank -> (world * B_local, top_k, 6), rank-major
    (= global image order when the batch was split with ``shard_bounds`` into equal shards)."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local
    world = dist.get_world_size(group)
    out = torch.empty((world * local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, local.contiguous(), group=group)
    return out


def all_gather_ragged(local_rows, group=None):
    """All-gather for unequal shards: pads to the largest B_local, gathers, and strips the padding."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local_rows
    world = dist.get_world_size(group)
    n = torch.tensor([local_rows.shape[0]], dtype=torch.int64, device=local_rows.device)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n, group=group)
    sizes = [int(s.item()) for s in sizes]
    mx = max(sizes)
    pad = torch.zeros((mx,) + tuple(local_rows.shape[1:]), dtype=local_rows.dtype, device=local_rows.device)
    pad[:local_rows.shape[0]] = local_rows
    out = torch.empty((world * mx,) + tuple(pad.shape[1:]), dtype=pad.dtype, device=pad.device)
    dist.all_gather_into_tensor(out, pad, group=group)
    return torch.cat([out[r * mx:r * mx + sizes[r]] for r in range(world)], dim=0)


def all_reduce_gradients_(flat_grad, group=None):
    """Data-parallel gradient exchange of the training step (SURVEY section 8e(i)): ONE all-reduce (sum) over the flat fp32
    gradient buffer, in place.  Returns the factor the optimiser must scale the summed gradient with (1 / world size), so that
    the update equals the mean of the replicas' gradients -- what Keras multi-GPU replicas of the reference's loss compute."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return 1.0
    dist.all_reduce(flat_grad, group=group)
    return 1.0 / dist.get_world_size(group)


def plan_buckets(first, size, bucket_bytes):
    """Layer ranges for an overlapped gradient exchange, top of the graph first.

    ``first[i]`` / ``size[i]``: offset (in floats; None if the layer has no parameters) and number of parameters of graph
    layer ``i`` inside the flat gradient buffer, which holds the layers in graph order.  Walking the layers top down, a bucket
    is closed once it holds ``bucket_bytes`` of float32 gradients.  Returns ``[(hi, lo, offset, count), ...]``: the layers
    ``hi .. lo`` own the contiguous span ``[offset, offset + count)``; every layer belongs to exactly one bucket."""
    n = len(size)
    out, hi, acc, lo_off = [], n - 1, 0, None
    for i in range(n - 1, -1, -1):
        if size[i]:
            acc += size[i]
            lo_off = first[i] if lo_off is None else min(lo_off, first[i])
        if acc * 4 >= bucket_bytes or i == 0:
            out.append((hi, i, lo_off if lo_off is not None else 0, acc))
            hi, acc, lo_off = i - 1, 0, None
    return out


def all_reduce_buckets_(flat_grad, buckets, produce, group=None):
    """``for hi, lo, off, cnt in buckets: produce(hi, lo)`` (which enqueues the kernels that finish the gradients of the layers
    ``hi .. lo``) followed at once by an asynchronous all-reduce (sum) of that bucket's span: the collective of bucket k runs
    on the communication stream while ``produce`` of bucket k+1 already runs on the compute stream.  Returns after making the
    current stream (CUDA) / the host (CPU tensors) wait for all of them."""
    import torch.distributed as dist
    on = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
    works = []
    for hi, lo, off, cnt in buckets:
        produce(hi, lo)
        if on and cnt:
            works.append(dist.all_reduce(flat_grad[off:off + cnt], group=group, async_op=True))
    for w in works:
        w.wait()
    return len(works)


class GlobalLossRun:
    """One rank's side of the phase-wise loss (``ssdk_ssd_loss_phase``): owns the workspace and exposes the tensors that have
    to be reduced between the phases.  ``ssd_loss_global`` drives it with torch.distributed; the single-GPU tests drive several
    instances and add the tensors by hand.  With ``return_grad`` the gradient goes to ``grad_out`` when given."""

    def __init__(self, y_true, y_pred, neg_pos_ratio, n_neg_min, alpha, world, rank, return_grad, grad_out=None):
        import ctypes as C
        import torch
        from . import _ffi
        self.yt = y_true.to(device='cuda', dtype=torch.float32).contiguous()
        self.yp = y_pred.to(device='cuda', dtype=torch.float32).contiguous()
        self.B, self.P, self.W = self.yp.shape
        self.cfg = (int(neg_pos_ratio), int(n_neg_min), float(alpha))
        self.world, self.rank = int(world), int(rank)
        lay = _ffi.LossWsLayout()
        _ffi.check(_ffi.lib().ssdk_ssd_loss_ws_layout(self.B, self.P, C.byref(lay)))
        dev = self.yp.device
        self.ws = torch.zeros((lay.bytes,), dtype=torch.uint8, device=dev)
        self.counts = self.ws[lay.counts_offset:lay.counts_offset + 8 * lay.counts_n].view(torch.int64)
        self.hist1 = self.ws[lay.hist1_offset:lay.hist1_offset + 4 * lay.hist_n].view(torch.int32)
        self.hist2 = self.ws[lay.hist2_offset:lay.hist2_offset + 4 * lay.hist_n].view(torch.int32)
        self.ties = self.ws[lay.ties_offset:lay.ties_offset + 4].view(torch.int32)
        self.ties_all = torch.zeros((self.world,), dtype=torch.int32, device=dev)
        self.loss = torch.empty((self.B,), dtype=torch.float32, device=dev)
        self.stats = torch.zeros((4,), dtype=torch.int32, device=dev)
        self.grad = None
        if return_grad:
            self.grad = torch.empty_like(self.yp) if grad_out is None else grad_out
            assert self.grad.shape == self.yp.shape and self.grad.dtype == torch.float32 and self.grad.is_contiguous()

    def phase(self, i):
        from . import _ffi
        final = i == 4
        r, m, a = self.cfg
        _ffi.check(_ffi.lib().ssdk_ssd_loss_phase(_ffi.context(self.yp.device.index), i, _ffi.dptr(self.yt), _ffi.dptr(self.yp), self.B,
                                                  self.P, self.W - 12, r, m, a, _ffi.dptr(self.ws), self.world * self.B,
                                                  _ffi.dptr(self.ties_all), self.rank, _ffi.dptr(None),
                                                  _ffi.dptr(self.loss if final else None), _ffi.dptr(self.stats if final else None),
                                                  _ffi.dptr(self.grad if final else None), _ffi.stream_ptr()))


def ssd_loss_global(y_true, y_pred, neg_pos_ratio=3, n_neg_min=0, alpha=1.0, group=None, return_grad=False, grad_out=None):
    """Global-batch-exact ``SSDLoss.compute_loss`` for a batch that is sharded over the ranks of ``group`` (SURVEY section 8e(ii)).

    The reference's ``n_positive`` (keras_ssd_loss.py:143) and its hard-negative top-k (:179-183) run over the WHOLE batch.
    Every rank holds ``(B_local, P, C+12)`` shards (equal ``B_local``, rank order = image order); the loss kernel's phases run
    one by one and the integer counts / histograms in its workspace are summed with all-reduces in between (2 x int64, then
    two histograms of 67 584 int32), ties at the k-th value are resolved by GLOBAL flat index via an all-gather of one int per
    rank.  Returns the ``(B_local,)`` losses of this rank's images -- exactly the entries the single-process reference
    computes for them -- and, with ``return_grad``, ``(loss, d(mean over the global batch)/d y_pred of this shard, stats)``,
    the gradient written into ``grad_out`` when given.  Without an initialised process group this is the single-rank result
    (phases run back to back)."""
    import torch.distributed as dist
    on = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
    world = dist.get_world_size(group) if on else 1
    rank = dist.get_rank(group) if on else 0
    run = GlobalLossRun(y_true, y_pred, neg_pos_ratio, n_neg_min, alpha, world, rank, return_grad, grad_out)
    run.phase(0)
    if on:
        dist.all_reduce(run.counts, group=group)
        dist.all_reduce(run.hist1, group=group)
    run.phase(1)
    if on:
        dist.all_reduce(run.hist2, group=group)
    run.phase(2)
    run.phase(3)
    if on:
        dist.all_gather_into_tensor(run.ties_all, run.ties, group=group)
    else:
        run.ties_all.copy_(run.ties)
    run.phase(4)
    return (run.loss, run.grad, run.stats) if return_grad else run.loss


def focal_loss_global(y_true, y_pred, gamma=2.0, focal_alpha=0.25, alpha=1.0, group=None, return_grad=False, grad_out=None):
    """``SSDFocalLoss.compute_loss`` for a batch that is sharded over the ranks of ``group``: its normaliser, the number of
    positives, runs over the WHOLE batch.  Every rank holds ``(B_local, P, C+12)`` shards (equal ``B_local``, rank order = image
    order): ``ssdk_focal_loss_phase`` phase 0 counts this rank's positives into one int64 (32.32 fixed point), one all-reduce
    sums it, phase 1 writes the losses and / or the gradient.  Returns the ``(B_local,)`` losses of this rank's images, bit for
    bit the entries one process computes for them on the whole batch, and with ``return_grad`` ``(loss, d(mean over the global
    batch)/d y_pred of this shard)``, written into ``grad_out`` when given.  Without an initialised process group this is the
    single-rank result."""
    import torch
    import torch.distributed as dist
    from . import _ffi
    on = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
    world = dist.get_world_size(group) if on else 1
    yt = y_true.to(device='cuda', dtype=torch.float32).contiguous()
    yp = y_pred.to(device='cuda', dtype=torch.float32).contiguous()
    B, P, W = yp.shape
    dev = yp.device
    count = torch.zeros((1,), dtype=torch.int64, device=dev)
    loss = torch.empty((B,), dtype=torch.float32, device=dev)
    grad = None
    if return_grad:
        grad = torch.empty_like(yp) if grad_out is None else grad_out
        assert grad.shape == yp.shape and grad.dtype == torch.float32 and grad.is_contiguous()
    lib, ctx = _ffi.lib(), _ffi.context(dev.index)
    cfg = (float(gamma), float(focal_alpha), float(alpha))

    def phase(i):
        _ffi.check(lib.ssdk_focal_loss_phase(ctx, i, _ffi.dptr(yt), _ffi.dptr(yp), B, P, W - 12, *cfg, _ffi.dptr(count), world * B,
                                             _ffi.dptr(None), _ffi.dptr(loss), _ffi.dptr(grad), _ffi.stream_ptr()))
    phase(0)
    if on:
        dist.all_reduce(count, group=group)
    phase(1)
    return (loss, grad) if return_grad else loss
