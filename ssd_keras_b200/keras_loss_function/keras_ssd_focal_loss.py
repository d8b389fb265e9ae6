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
from .keras_ssd_loss import KernelLoss


class SSDFocalLoss(KernelLoss):
    """``gamma``: the focusing exponent (0 gives the weighted log-loss); ``focal_alpha``: the weight of the object classes, the
    background's being ``1 - focal_alpha``; ``alpha``: the weight of the localisation term, as in ``SSDLoss``."""
    config_key = 'ssd_focal_loss'

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

    def _launch(self, y_true, y_pred, upstream, out_loss, out_grad):
        B, P, W = y_pred.shape
        _ffi.check(_ffi.lib().ssdk_focal_loss(_ffi.context(y_pred.device.index), _ffi.dptr(y_true), _ffi.dptr(y_pred), B, P, W - 12,
                                              self.gamma, self.focal_alpha, self.alpha, _ffi.dptr(upstream), _ffi.dptr(out_loss),
                                              _ffi.dptr(out_grad), _ffi.stream_ptr()))

    def _global(self, y_true, y_pred, grad_out, group):
        from ..distributed import focal_loss_global
        loss, _ = focal_loss_global(y_true, y_pred, self.gamma, self.focal_alpha, self.alpha, group=group, return_grad=True,
                                    grad_out=grad_out)
        return loss
