"""Training step on H100: what ``model.compile(optimizer=SGD(lr, momentum), loss=SSDLoss().compute_loss)`` +
``train_on_batch`` do in the reference (``ssd300_training.ipynb:169-173``), through ``ssdk_train_backward`` /
``ssdk_train_apply`` (``csrc/train.cu``).  Data-parallel: every rank runs the same step on its shard and the flat
gradient buffer is summed with ONE NCCL all-reduce before the update (replica-local loss, SURVEY.md section 8e(i)).
"""
import ctypes as C
import weakref

import numpy as np

from . import _ffi


class SSDTrainer:
    def __init__(self, model, batch_size, lr=1e-3, momentum=0.9, l2_regularization=None, neg_pos_ratio=3, n_neg_min=0,
                 alpha=1.0, loss_mode='replica', optimizer='sgd', beta_1=0.9, beta_2=0.999, epsilon=1e-8):
        """``loss_mode``: 'replica' -- every rank applies the reference loss to its own shard (what Keras data-parallel replicas
        compute, SURVEY 8e(i)); 'global' -- n_positive and the hard-negative top-k run over the whole sharded batch, so that N
        ranks reproduce the single-process reference on the full batch (8e(ii), ``distributed.ssd_loss_global``)."""
        if loss_mode not in ('replica', 'global'):
            raise ValueError("loss_mode must be 'replica' or 'global'")
        if optimizer not in ('sgd', 'adam'):
            raise ValueError("optimizer must be 'sgd' (SGD(lr, momentum), ssd300_training.ipynb:169) or 'adam' (ssd7_training.ipynb:153)")
        self.loss_mode = loss_mode
        self.optimizer, self.beta_1, self.beta_2, self.epsilon = optimizer, float(beta_1), float(beta_2), float(epsilon)
        self.iterations = 0                      # optimiser steps taken (Adam's bias correction)
        import torch
        self.model = model
        self.batch = int(batch_size)
        self.lr, self.momentum = float(lr), float(momentum)
        self.l2 = float(model.l2_regularization if l2_regularization is None else l2_regularization)
        self.neg_pos_ratio, self.n_neg_min, self.alpha = int(neg_pos_ratio), int(n_neg_min), float(alpha)
        # the flat gradient buffer is a torch tensor so that torch.distributed can all-reduce it in place
        self.n_params = self._count_trainable(model)
        self.grad = torch.zeros((self.n_params,), dtype=torch.float32, device='cuda')
        self.handle = None
        self.plan = None
        self._spans = None
        self._dirty = False                      # device master weights are ahead of model.weights
        self._buckets = None
        self.bucket_bytes = 24 << 20
        model._trainers.append(weakref.ref(self))
        self._attach()

    @staticmethod
    def _count_trainable(model):
        n = 0
        for k, shp in model.weight_shapes().items():
            if k.endswith(('/moving_mean', '/moving_variance')):
                continue
            n += int(np.prod(shp))
        return n

    def _attach(self):
        """(Re-)create the training plan from the model's current weights and the native trainer on top of it."""
        if self.handle is not None:
            return
        self.plan = self.model._plan(self.batch, training=True)
        h = C.c_void_p()
        _ffi.check(_ffi.lib().ssdk_trainer_create(self.plan['handle'], _ffi.dptr(self.grad), C.byref(h)))
        self.handle = h
        n = C.c_longlong()
        _ffi.check(_ffi.lib().ssdk_trainer_num_params(self.handle, C.byref(n)))
        assert int(n.value) == self.n_params, (n.value, self.n_params)
        self._spans = None

    def _detach(self):
        """Called by the model before it destroys its plans (``set_weights`` / ``load_weights``): the native trainer points
        into the training plan.  Optimiser state (momentum, Adam's moments and its step count) does not survive; the next step
        starts from the new weights as a fresh trainer's first step would."""
        if self.handle is not None:
            _ffi.lib().ssdk_trainer_destroy(self.handle)
        self.handle = None
        self.plan = None
        self._dirty = False
        self.iterations = 0

    def __del__(self):
        try:
            if getattr(self, 'handle', None):
                _ffi.lib().ssdk_trainer_destroy(self.handle)
        except Exception:
            pass

    # -- one step ------------------------------------------------------------------------------
    def _check_batch(self, images, y_true):
        P, W = self.model.n_boxes_total, self.model.n_classes + 12
        if images.shape[0] != self.batch or tuple(y_true.shape) != (self.batch, P, W):
            raise ValueError('this trainer was built for batches of %d images: images %s / y_true %s do not match (%d, H, W, 3) / %s; '
                             'build another SSDTrainer for a different batch size (e.g. the last, smaller batch of an epoch)'
                             % (self.batch, tuple(images.shape), tuple(y_true.shape), self.batch, (self.batch, P, W)))
        if not (images.is_cuda and y_true.is_cuda):
            raise ValueError('images and y_true must be CUDA tensors')

    def _loss_and_dy(self, images, y_true):
        """forward + loss; leaves d loss / d y_pred ready for the layer-wise backward.  Returns (loss, y_pred, dy or None)."""
        import torch
        self._attach()
        self._check_batch(images, y_true)
        y_pred = self.model.forward_device(images, training=True)
        y_true = y_true.to(dtype=torch.float32).contiguous()
        if self.loss_mode == 'global':
            from .distributed import ssd_loss_global
            loss, dy, _ = ssd_loss_global(y_true, y_pred, self.neg_pos_ratio, self.n_neg_min, self.alpha, return_grad=True)
            return loss, y_pred, dy
        loss = torch.empty((self.batch,), dtype=torch.float32, device=images.device)
        _ffi.check(_ffi.lib().ssdk_train_backward_begin(self.handle, _ffi.dptr(y_true), _ffi.dptr(y_pred), self.neg_pos_ratio,
                                                        self.n_neg_min, self.alpha, _ffi.dptr(loss), _ffi.stream_ptr()))
        return loss, y_pred, None

    def _backward_layers(self, dy, hi, lo):
        _ffi.check(_ffi.lib().ssdk_train_backward_layers(self.handle, _ffi.dptr(dy), int(hi), int(lo), _ffi.stream_ptr()))

    def forward_backward(self, images, y_true):
        """images (B,H,W,3), y_true (B,P,C+12): float32 CUDA tensors.  Returns (loss (B,), y_pred); gradients in self.grad."""
        loss, y_pred, dy = self._loss_and_dy(images, y_true)
        self._backward_layers(dy, len(self.model.specs) - 1, 0)
        return loss, y_pred

    def apply(self, grad_scale=1.0):
        self._attach()
        self._dirty = True
        self.iterations += 1
        if self.optimizer == 'adam':
            _ffi.check(_ffi.lib().ssdk_train_apply_adam(self.handle, self.lr, self.beta_1, self.beta_2, self.epsilon, self.l2, float(grad_scale),
                                                        int(self.iterations), _ffi.stream_ptr()))
        else:
            _ffi.check(_ffi.lib().ssdk_train_apply(self.handle, self.lr, self.momentum, self.l2, float(grad_scale), _ffi.stream_ptr()))

    def buckets(self, bucket_bytes=None):
        """Layer ranges for the overlapped gradient exchange, top of the graph first: [(hi, lo, offset, count), ...].  The
        parameters lie in the flat buffer in graph order, so the layers hi..lo own one contiguous span of it; a bucket is closed
        once it holds ``bucket_bytes`` of gradients (default 24 MB -- large enough that NCCL runs at NVLink bandwidth, small enough
        that the first exchange starts after ~1/5 of the backward pass of SSD300)."""
        from .distributed import plan_buckets
        bucket_bytes = int(self.bucket_bytes if bucket_bytes is None else bucket_bytes)
        if self._buckets is not None and self._buckets[0] == bucket_bytes:
            return self._buckets[1]
        n = len(self.model.specs)
        first = [None] * n                                       # lowest offset / total count of each layer's parameters
        size = [0] * n
        for (name, _), (o, c) in self.spans().items():
            i = self.model.index[name]
            first[i] = o if first[i] is None else min(first[i], o)
            size[i] += c
        out = plan_buckets(first, size, bucket_bytes)
        self._buckets = (bucket_bytes, out)
        return out

    def train_on_batch(self, images, y_true, group=None, overlap=None):
        """forward + loss + backward + gradient exchange + SGD update.  Returns the per-image loss tensor (B,).
        With several ranks the flat gradient buffer is all-reduced either in buckets, from the top of the network down, each as
        soon as its layers have been differentiated (NCCL on its own stream under the weight / data gradient kernels of the lower
        layers), or in one call after the backward pass.  ``overlap=None`` picks: at 2 ranks the whole exchange is short while
        NCCL's kernels share the SMs with the persistent (one CTA per SM) conv launches when they run side by side, so the
        bucketed exchange is used from 4 ranks on (SSDK_GRAD_OVERLAP=0/1 overrides; SSDK_OVERLAP is the two-stream schedule of inference plans)."""
        import os
        import torch.distributed as dist
        on = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
        loss, _, dy = self._loss_and_dy(images, y_true)
        if not on:
            self._backward_layers(dy, len(self.model.specs) - 1, 0)
            self.apply(1.0)
            return loss
        if overlap is None:
            env = os.environ.get('SSDK_GRAD_OVERLAP')
            overlap = (env == '1') if env in ('0', '1') else dist.get_world_size(group) > 2
        from .distributed import all_reduce_buckets_
        if overlap:
            all_reduce_buckets_(self.grad, self.buckets(), lambda hi, lo: self._backward_layers(dy, hi, lo), group=group)
        else:
            self._backward_layers(dy, len(self.model.specs) - 1, 0)
            dist.all_reduce(self.grad, group=group)
        # 'replica': the mean of the replicas' gradients; 'global': the shards' gradients of the GLOBAL batch mean add up
        self.apply(1.0 if self.loss_mode == 'global' else 1.0 / dist.get_world_size(group))
        return loss

    # -- introspection (tests) -------------------------------------------------------------------
    def spans(self):
        if self._spans is None:
            out = {}
            for i, s in enumerate(self.model.specs):
                for which, tag in ((0, 'kernel'), (1, 'bias'), (2, 'gamma'), (3, 'bn_gamma'), (4, 'bn_beta')):
                    o, c = C.c_longlong(), C.c_longlong()
                    _ffi.check(_ffi.lib().ssdk_trainer_param_span(self.handle, i, which, C.byref(o), C.byref(c)))
                    if c.value > 0:
                        out[(s.name, tag)] = (int(o.value), int(c.value))
            self._spans = out
        return self._spans

    def _unflatten(self, flat):
        """flat float32 ndarray -> dict with Keras names / layouts (kernels HWIO, head kernels split into conf / loc)."""
        m = self.model
        res = {}
        Ct = m.n_classes
        for s in m.specs:
            if s.op == _ffi.OP_CONV:
                cin = m._shapes[m.index[s.inp]][2]
                o, c = self.spans()[(s.name, 'kernel')]
                res[s.name + '/kernel'] = flat[o:o + c].reshape(s.cout, s.kh, s.kw, cin).transpose(1, 2, 3, 0).copy()
                o, c = self.spans()[(s.name, 'bias')]
                res[s.name + '/bias'] = flat[o:o + c].copy()
                if s.bn and (s.name, 'bn_gamma') in self.spans():
                    o, c = self.spans()[(s.name, 'bn_gamma')]
                    res[s.bn + '/gamma'] = flat[o:o + c].copy()
                    o, c = self.spans()[(s.name, 'bn_beta')]
                    res[s.bn + '/beta'] = flat[o:o + c].copy()
            elif s.op == _ffi.OP_HEAD:
                cin = m._shapes[m.index[s.inp]][2]
                nb = s.n_boxes
                o, c = self.spans()[(s.name, 'kernel')]
                w = flat[o:o + c].reshape(nb, Ct + 4, 3, 3, cin)            # fused per box: [C logits | 4 offsets]
                res[s.params['conf_name'] + '/kernel'] = w[:, :Ct].reshape(nb * Ct, 3, 3, cin).transpose(1, 2, 3, 0).copy()
                res[s.params['loc_name'] + '/kernel'] = w[:, Ct:].reshape(nb * 4, 3, 3, cin).transpose(1, 2, 3, 0).copy()
                o, c = self.spans()[(s.name, 'bias')]
                b = flat[o:o + c].reshape(nb, Ct + 4)
                res[s.params['conf_name'] + '/bias'] = b[:, :Ct].reshape(-1).copy()
                res[s.params['loc_name'] + '/bias'] = b[:, Ct:].reshape(-1).copy()
            elif s.op == _ffi.OP_L2NORM:
                o, c = self.spans()[(s.name, 'gamma')]
                res[s.name + '/gamma'] = flat[o:o + c].copy()
        return res

    def gradients(self):
        return self._unflatten(self.grad.cpu().numpy())

    def get_weights(self):
        import torch
        self._attach()
        out = torch.empty_like(self.grad)
        _ffi.check(_ffi.lib().ssdk_trainer_read_params(self.handle, _ffi.dptr(out), _ffi.stream_ptr()))
        res = self._unflatten(out.cpu().numpy())
        for i, s in enumerate(self.model.specs):              # moving statistics of the BatchNormalization layers
            if s.op == _ffi.OP_CONV and s.bn:
                mu = torch.empty((s.cout,), dtype=torch.float32, device='cuda'); var = torch.empty_like(mu)
                _ffi.check(_ffi.lib().ssdk_trainer_read_bn_stats(self.handle, i, _ffi.dptr(mu), _ffi.dptr(var), _ffi.stream_ptr()))
                res[s.bn + '/moving_mean'], res[s.bn + '/moving_variance'] = mu.cpu().numpy(), var.cpu().numpy()
        return res
