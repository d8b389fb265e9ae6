"""``L2Normalization`` on H100 (reference ``keras_layers/keras_layer_L2Normalization.py:25-70``):
``x * rsqrt(max(sum_c x^2, 1e-12)) * gamma_c`` over the channel axis of an NHWC tensor, computed by
``ssdk_l2_normalize`` (``l2norm_f32_kernel`` in ``csrc/conv.cu``).  Inside ``ssd_300`` / ``ssd_512`` the same
arithmetic runs on the split-bf16 activation planes (``l2norm_kernel``)."""
import numpy as np

from .. import _ffi


class L2Normalization:
    def __init__(self, gamma_init=20, **kwargs):
        self.axis = 3
        self.gamma_init = gamma_init
        self.gamma = None
        self.name = kwargs.get('name', 'l2_normalization')

    def build(self, input_shape):
        self.gamma = self.gamma_init * np.ones((input_shape[self.axis],), dtype=np.float32)

    def call(self, x, mask=None):
        """x: float32 (B,H,W,C) CUDA tensor or ndarray -> same type."""
        import torch
        is_np = isinstance(x, np.ndarray)
        xt = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda() if is_np else x.float().contiguous()
        if self.gamma is None:
            self.build(xt.shape)
        g = torch.from_numpy(np.ascontiguousarray(self.gamma, dtype=np.float32)).to(xt.device)
        out = torch.empty_like(xt)
        Cc = xt.shape[-1]
        _ffi.check(_ffi.lib().ssdk_l2_normalize(_ffi.context(xt.device.index), _ffi.dptr(xt), xt.numel() // Cc, Cc,
                                                _ffi.dptr(g), _ffi.dptr(out), _ffi.stream_ptr()))
        return out.cpu().numpy() if is_np else out

    __call__ = call

    def get_config(self):
        return {'gamma_init': self.gamma_init}
