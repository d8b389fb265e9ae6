"""``SSDLoss`` on H100 (reference ``keras_loss_function/keras_ssd_loss.py:22-211``), computed by
``csrc/loss.cu``.  ``compute_loss`` takes / returns torch CUDA tensors (NumPy arrays are accepted and
copied) and is differentiable with respect to ``y_pred`` through a ``torch.autograd.Function`` whose
backward is the hand-written ``ssdk_ssd_loss_bwd`` kernel.
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

    class _SSDLossFn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, y_true, y_pred, neg_pos_ratio, n_neg_min, alpha):
            B, P, W = y_pred.shape
            out = torch.empty((B,), dtype=torch.float32, device=y_pred.device)
            stats = torch.zeros((4,), dtype=torch.int32, device=y_pred.device)
            _ffi.check(_ffi.lib().ssdk_ssd_loss_fwd(_ffi.context(y_pred.device.index), _ffi.dptr(y_true), _ffi.dptr(y_pred), B, P,
                                                    W - 12, int(neg_pos_ratio), int(n_neg_min), float(alpha), _ffi.dptr(out),
                                                    _ffi.dptr(stats), _ffi.stream_ptr()))
            ctx.save_for_backward(y_true, y_pred)
            ctx.cfg = (int(neg_pos_ratio), int(n_neg_min), float(alpha))
            ctx.stats = stats
            return out

        @staticmethod
        def backward(ctx, grad_out):
            y_true, y_pred = ctx.saved_tensors
            B, P, W = y_pred.shape
            r, m, a = ctx.cfg
            g = torch.empty_like(y_pred)
            up = grad_out.to(dtype=torch.float32).contiguous()
            _ffi.check(_ffi.lib().ssdk_ssd_loss_bwd(_ffi.context(y_pred.device.index), _ffi.dptr(y_true), _ffi.dptr(y_pred), B, P,
                                                    W - 12, r, m, a, _ffi.dptr(up), _ffi.dptr(g), _ffi.stream_ptr()))
            return None, g, None, None, None

    return _SSDLossFn


_FN = None


class SSDLoss:
    """The SSD loss, see https://arxiv.org/abs/1512.02325 (same arguments as the reference, :27-30)."""

    def __init__(self, neg_pos_ratio=3, n_neg_min=0, alpha=1.0):
        self.neg_pos_ratio = neg_pos_ratio
        self.n_neg_min = n_neg_min
        self.alpha = alpha

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
        device); ``compute_loss`` computes the same quantity inside ``ssdk_ssd_loss_fwd``."""
        return self._smooth_l1_t(_as_cuda(y_true), _as_cuda(y_pred))

    def log_loss(self, y_true, y_pred):
        """Reference :77-96, (B,P,C) x2 -> (B,P) float32 CUDA tensor (see ``smooth_L1_loss``)."""
        return self._log_loss_t(_as_cuda(y_true), _as_cuda(y_pred))

    def compute_loss(self, y_true, y_pred):
        """(B,P,C+12) x2 -> (B,) float32 CUDA tensor (reference :98-211)."""
        global _FN
        if _FN is None:
            _FN = _make_fn()
        yt, yp = _as_cuda(y_true), _as_cuda(y_pred)
        if yt.shape != yp.shape or yt.dim() != 3 or yt.shape[-1] < 14:
            raise ValueError("y_true and y_pred must both have shape (batch, #boxes, #classes + 12) with at least two classes, "
                             "got %s and %s" % (tuple(yt.shape), tuple(yp.shape)))
        if yt.device != yp.device:
            raise ValueError("y_true and y_pred must live on the same device")
        return _FN.apply(yt, yp, self.neg_pos_ratio, self.n_neg_min, self.alpha)

    def loss_and_stats(self, y_true, y_pred):
        """-> (loss (B,), stats int32[4] = n_positive, n_neg_losses, k, ties_taken)."""
        import torch
        yt, yp = _as_cuda(y_true), _as_cuda(y_pred)
        B, P, W = yp.shape
        out = torch.empty((B,), dtype=torch.float32, device=yp.device)
        stats = torch.zeros((4,), dtype=torch.int32, device=yp.device)
        _ffi.check(_ffi.lib().ssdk_ssd_loss_fwd(_ffi.context(yp.device.index), _ffi.dptr(yt), _ffi.dptr(yp), B, P, W - 12,
                                                int(self.neg_pos_ratio), int(self.n_neg_min), float(self.alpha), _ffi.dptr(out),
                                                _ffi.dptr(stats), _ffi.stream_ptr()))
        return out, stats
