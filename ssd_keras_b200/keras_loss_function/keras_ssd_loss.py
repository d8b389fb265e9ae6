"""``SSDLoss`` on H100 (reference ``keras_loss_function/keras_ssd_loss.py:22-211``), computed by
``csrc/loss.cu``.  ``compute_loss`` takes / returns torch CUDA tensors (NumPy arrays are accepted and
copied) and is differentiable with respect to ``y_pred`` through a ``torch.autograd.Function`` whose
backward is the same hand-written kernel (``ssdk_ssd_loss`` with a gradient output).  ``KernelLoss`` is what ``SSDLoss`` and
``SSDFocalLoss`` share: that autograd Function, the training step's ``loss_and_grad`` and the ``model.save`` configuration.
"""
import numpy as np

from .. import _ffi


def _as_cuda(t):
    import torch
    if isinstance(t, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(t, dtype=np.float32)).pin_memory().cuda(non_blocking=True)
    if not torch.is_tensor(t):
        raise ValueError('expected a NumPy array or a torch tensor, got %s' % type(t).__name__)
    return t.to(device='cuda', dtype=torch.float32).contiguous()


def _make_fn():
    import torch

    class _LossFn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, lossobj, y_true, y_pred):
            out = torch.empty((y_pred.shape[0],), dtype=torch.float32, device=y_pred.device)
            lossobj._launch(y_true, y_pred, None, out, None)
            ctx.save_for_backward(y_true, y_pred)
            ctx.lossobj = lossobj
            return out

        @staticmethod
        def backward(ctx, grad_out):
            y_true, y_pred = ctx.saved_tensors
            g = torch.empty_like(y_pred)
            ctx.lossobj._launch(y_true, y_pred, grad_out.to(dtype=torch.float32).contiguous(), None, g)
            return None, None, g

    return _LossFn


_FN = None


def _check_pair(yt, yp):
    if yt.shape != yp.shape or yt.dim() != 3 or yt.shape[-1] < 14:
        raise ValueError("y_true and y_pred must both have shape (batch, #boxes, #classes + 12) with at least two classes, "
                         "got %s and %s" % (tuple(yt.shape), tuple(yp.shape)))
    if yt.device != yp.device:
        raise ValueError("y_true and y_pred must live on the same device")


class KernelLoss:
    """A loss on ``(batch, #boxes, #classes + 12)`` tensors whose value and gradient come from one hand-written kernel.  A
    subclass gives its parameters and
    - ``config()``: the constructor's arguments, which ``model.save`` stores under ``config_key`` in ``training_config``;
    - ``_launch(y_true, y_pred, upstream, out_loss, out_grad)``: one launch on CUDA float32 tensors, the per-image losses into
      ``out_loss`` and / or d(sum_b upstream[b] loss[b]) / d y_pred into ``out_grad`` (``upstream`` None: 1 / batch each);
    - ``_global(y_true, y_pred, grad_out, group)``: its driver in ``distributed.py``, the losses of this rank's images and the
      gradient of the mean over the batch sharded over the ranks of ``group`` into ``grad_out``."""
    config_key = None

    def compute_loss(self, y_true, y_pred):
        """(B,P,C+12) x2 -> (B,) float32 CUDA tensor, differentiable with respect to ``y_pred``."""
        global _FN
        if _FN is None:
            _FN = _make_fn()
        yt, yp = _as_cuda(y_true), _as_cuda(y_pred)
        _check_pair(yt, yp)
        return _FN.apply(self, yt, yp)

    def loss_and_grad(self, y_true, y_pred, grad_out, loss_mode='replica', group=None):
        """(B,P,C+12) x2 -> the per-image losses (B,), with d(mean loss) / d y_pred written into ``grad_out`` (a contiguous
        float32 tensor of ``y_pred``'s shape on its device).  ``loss_mode``: 'replica' -- the mean over this batch, one launch;
        'global' -- the mean over the batch sharded over the ranks of ``group``."""
        import torch
        yt, yp = _as_cuda(y_true), _as_cuda(y_pred)
        _check_pair(yt, yp)
        if (grad_out.shape != yp.shape or grad_out.dtype != torch.float32 or grad_out.device != yp.device
                or not grad_out.is_contiguous()):
            raise ValueError("grad_out must be a contiguous float32 tensor of y_pred's shape on its device")
        if loss_mode not in ('replica', 'global'):
            raise ValueError("loss_mode must be 'replica' or 'global'")
        if loss_mode == 'global':
            return self._global(yt, yp, grad_out, group)
        loss = torch.empty((yp.shape[0],), dtype=torch.float32, device=yp.device)
        self._launch(yt, yp, None, loss, grad_out)
        return loss


class SSDLoss(KernelLoss):
    """The SSD loss, see https://arxiv.org/abs/1512.02325 (same arguments as the reference, :27-30)."""
    config_key = 'ssd_loss'

    def __init__(self, neg_pos_ratio=3, n_neg_min=0, alpha=1.0):
        self.neg_pos_ratio = neg_pos_ratio
        self.n_neg_min = n_neg_min
        self.alpha = alpha

    def config(self):
        return {'neg_pos_ratio': self.neg_pos_ratio, 'n_neg_min': self.n_neg_min, 'alpha': self.alpha}

    def _launch(self, y_true, y_pred, upstream, out_loss, out_grad, out_stats=None):
        B, P, W = y_pred.shape
        _ffi.check(_ffi.lib().ssdk_ssd_loss(_ffi.context(y_pred.device.index), _ffi.dptr(y_true), _ffi.dptr(y_pred), B, P, W - 12,
                                            int(self.neg_pos_ratio), int(self.n_neg_min), float(self.alpha), _ffi.dptr(upstream),
                                            _ffi.dptr(out_loss), _ffi.dptr(out_stats), _ffi.dptr(out_grad), _ffi.stream_ptr()))

    def _global(self, y_true, y_pred, grad_out, group):
        from ..distributed import ssd_loss_global
        loss, _, _ = ssd_loss_global(y_true, y_pred, self.neg_pos_ratio, self.n_neg_min, self.alpha, group=group, return_grad=True,
                                     grad_out=grad_out)
        return loss

    @staticmethod
    def _smooth_l1_t(y_true, y_pred):
        import torch
        absolute_loss = torch.abs(y_true - y_pred)
        square_loss = 0.5 * (y_true - y_pred) ** 2
        return torch.sum(torch.where(absolute_loss < 1.0, square_loss, absolute_loss - 0.5), dim=-1)

    @staticmethod
    def _log_loss_t(y_true, y_pred):
        import torch
        return -torch.sum(y_true * torch.log(torch.clamp(y_pred, min=1e-15)), dim=-1)

    def smooth_L1_loss(self, y_true, y_pred):
        """Reference :53-75, (B,P,4) x2 -> (B,P) float32 CUDA tensor.  Stand-alone helper (a few tensor operations on the
        device); ``compute_loss`` computes the same quantity inside ``ssdk_ssd_loss``."""
        return self._smooth_l1_t(_as_cuda(y_true), _as_cuda(y_pred))

    def log_loss(self, y_true, y_pred):
        """Reference :77-96, (B,P,C) x2 -> (B,P) float32 CUDA tensor (see ``smooth_L1_loss``)."""
        return self._log_loss_t(_as_cuda(y_true), _as_cuda(y_pred))

    def loss_and_stats(self, y_true, y_pred):
        """-> (loss (B,), stats int32[4] = n_positive, n_neg_losses, k, ties_taken)."""
        import torch
        yt, yp = _as_cuda(y_true), _as_cuda(y_pred)
        out = torch.empty((yp.shape[0],), dtype=torch.float32, device=yp.device)
        stats = torch.zeros((4,), dtype=torch.int32, device=yp.device)
        self._launch(yt, yp, None, out, None, stats)
        return out, stats
