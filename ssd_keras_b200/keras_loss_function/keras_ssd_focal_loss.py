"""``SSDFocalLoss``: the softmax focal loss (Lin et al., https://arxiv.org/abs/1708.02002) in place of ``SSDLoss``'s 3:1
hard-negative mining, on the same ``(batch, #boxes, #classes + 12)`` tensors, computed by ``csrc/focal_loss.cu``.

Every box contributes ``sum_c y_true[c] w_c (1 - q_c)^gamma (-log max(q_c, 1e-15))`` with ``w_0 = 1 - focal_alpha`` for the
background and ``w_c = focal_alpha`` for the object classes: confident, easy boxes are down-weighted instead of left out, so
no batch-global top-k is needed.  The localisation term, the positives and the normalisation are ``SSDLoss``'s: per image
``B * (sum cls + alpha * sum pos * smooth_L1) / max(1, n_positive)``.  ``compute_loss`` is differentiable with respect to
``y_pred`` through a ``torch.autograd.Function`` whose backward is the same kernel (``ssdk_focal_loss`` with a gradient output).
"""
import math

from .. import _ffi
from .keras_ssd_loss import _as_cuda


def _make_fn():
    import torch

    class _SSDFocalLossFn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, y_true, y_pred, gamma, focal_alpha, alpha):
            B, P, W = y_pred.shape
            out = torch.empty((B,), dtype=torch.float32, device=y_pred.device)
            _ffi.check(_ffi.lib().ssdk_focal_loss(_ffi.context(y_pred.device.index), _ffi.dptr(y_true), _ffi.dptr(y_pred), B, P,
                                                  W - 12, gamma, focal_alpha, alpha, _ffi.dptr(None), _ffi.dptr(out),
                                                  _ffi.dptr(None), _ffi.stream_ptr()))
            ctx.save_for_backward(y_true, y_pred)
            ctx.cfg = (gamma, focal_alpha, alpha)
            return out

        @staticmethod
        def backward(ctx, grad_out):
            y_true, y_pred = ctx.saved_tensors
            B, P, W = y_pred.shape
            g = torch.empty_like(y_pred)
            up = grad_out.to(dtype=torch.float32).contiguous()
            _ffi.check(_ffi.lib().ssdk_focal_loss(_ffi.context(y_pred.device.index), _ffi.dptr(y_true), _ffi.dptr(y_pred), B, P,
                                                  W - 12, *ctx.cfg, _ffi.dptr(up), _ffi.dptr(None), _ffi.dptr(g),
                                                  _ffi.stream_ptr()))
            return None, g, None, None, None

    return _SSDFocalLossFn


_FN = None


class SSDFocalLoss:
    """``gamma``: the focusing exponent (0 gives the weighted log-loss); ``focal_alpha``: the weight of the object classes, the
    background's being ``1 - focal_alpha``; ``alpha``: the weight of the localisation term, as in ``SSDLoss``."""

    def __init__(self, gamma=2.0, focal_alpha=0.25, alpha=1.0):
        if not (float(gamma) >= 0 and math.isfinite(float(gamma))):
            raise ValueError('gamma must be a finite number >= 0, got %r' % (gamma,))
        if not 0 <= float(focal_alpha) <= 1:
            raise ValueError('focal_alpha must lie in [0, 1], got %r' % (focal_alpha,))
        self.gamma = float(gamma)
        self.focal_alpha = float(focal_alpha)
        self.alpha = float(alpha)

    def config(self):
        """The constructor's arguments, as ``model.save`` stores them."""
        return {'gamma': self.gamma, 'focal_alpha': self.focal_alpha, 'alpha': self.alpha}

    def compute_loss(self, y_true, y_pred):
        """(B,P,C+12) x2 -> (B,) float32 CUDA tensor."""
        global _FN
        if _FN is None:
            _FN = _make_fn()
        yt, yp = _as_cuda(y_true), _as_cuda(y_pred)
        if yt.shape != yp.shape or yt.dim() != 3 or yt.shape[-1] < 14:
            raise ValueError("y_true and y_pred must both have shape (batch, #boxes, #classes + 12) with at least two classes, "
                             "got %s and %s" % (tuple(yt.shape), tuple(yp.shape)))
        if yt.device != yp.device:
            raise ValueError("y_true and y_pred must live on the same device")
        return _FN.apply(yt, yp, self.gamma, self.focal_alpha, self.alpha)
