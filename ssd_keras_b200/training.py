"""Training step on H100: what ``model.compile(optimizer=SGD(lr, momentum), loss=SSDLoss().compute_loss)`` +
``train_on_batch`` do in the reference (``ssd300_training.ipynb:169-173``): the loss writes d loss / d y_pred into a buffer of
the trainer's (``KernelLoss.loss_and_grad``), then ``ssdk_train_backward_layers`` / ``ssdk_train_apply`` (``csrc/train.cu``).
Data-parallel: every rank runs the same step on its shard and the flat gradient buffer is summed with ONE NCCL all-reduce
before the update (replica-local loss, SURVEY.md section 8e(i)).
"""
import ctypes as C
import weakref

import numpy as np

from . import _ffi


def check_optimizer_state(model, optimizer, state):
    """Raise ``ValueError`` unless ``state`` (``{'iterations': int, 'slots': [dict, ...]}``, see
    ``SSDTrainer.get_optimizer_state``) fits ``model`` and ``optimizer`` ('sgd' / 'adam'): SGD has one slot, Adam two once it
    has taken a step (one before), and every slot holds exactly the model's trainable weights with their shapes."""
    it = state.get('iterations') if isinstance(state, dict) else None
    if not isinstance(it, (int, np.integer)) or isinstance(it, bool) or it < 0:
        raise ValueError('optimizer state: iterations must be a non-negative integer, got %r' % (it,))
    slots = state['slots']
    want = (1,) if optimizer == 'sgd' else (2,) if it > 0 else (1, 2)
    if len(slots) not in want:
        raise ValueError('optimizer state: %d slot(s) after %d iterations, but %s keeps %s' % (len(slots), it, optimizer, ' or '.join(map(str, want))))
    shapes = {k: tuple(v) for k, v in model.weight_shapes().items() if not k.endswith(('/moving_mean', '/moving_variance'))}
    for i, named in enumerate(slots):
        for k, shp in shapes.items():
            if k not in named:
                raise ValueError('optimizer state: slot %d has no entry for weight %s' % (i, k))
            if tuple(np.shape(named[k])) != shp:
                raise ValueError('optimizer state: slot %d, weight %s has shape %s, expected %s' % (i, k, tuple(np.shape(named[k])), shp))
        for k in named:
            if k not in shapes:
                raise ValueError('optimizer state: slot %d has an entry for %s, which is not a trainable weight of this model' % (i, k))


class SSDTrainer:
    def __init__(self, model, batch_size, lr=1e-3, momentum=0.9, l2_regularization=None, loss_mode='replica', optimizer='sgd',
                 beta_1=0.9, beta_2=0.999, epsilon=1e-8, loss=None):
        """``loss``: an ``SSDLoss`` or an ``SSDFocalLoss`` (any ``KernelLoss``); None is ``SSDLoss()``.  Each step it writes
        d loss / d y_pred into a buffer of the trainer's, from which the backward pass starts.
        ``loss_mode``: 'replica' -- every rank applies the loss to its own shard (what Keras data-parallel replicas compute,
        SURVEY 8e(i)); 'global' -- the loss's batch-global quantities (SSDLoss: n_positive and the hard-negative top-k; the
        focal loss: n_positive) run over the whole sharded batch, so that N ranks reproduce the single-process loss on the full
        batch (8e(ii), ``distributed.ssd_loss_global`` / ``focal_loss_global``)."""
        import torch
        from .keras_loss_function.keras_ssd_loss import KernelLoss, SSDLoss
        if loss is None:
            loss = SSDLoss()
        if not isinstance(loss, KernelLoss):
            raise ValueError('loss must be an SSDLoss or an SSDFocalLoss, got %r' % (loss,))
        self.loss = loss
        if loss_mode not in ('replica', 'global'):
            raise ValueError("loss_mode must be 'replica' or 'global'")
        if optimizer not in ('sgd', 'adam'):
            raise ValueError("optimizer must be 'sgd' (SGD(lr, momentum), ssd300_training.ipynb:169) or 'adam' (ssd7_training.ipynb:153)")
        self.loss_mode = loss_mode
        self.optimizer, self.beta_1, self.beta_2, self.epsilon = optimizer, float(beta_1), float(beta_2), float(epsilon)
        self.iterations = 0                      # optimiser steps taken (Adam's bias correction)
        self._n_slots = 1                        # optimiser state slots on the device: Adam's v is made by its first update
        self.model = model
        self.batch = int(batch_size)
        self.lr, self.momentum = float(lr), float(momentum)
        self.l2 = float(model.l2_regularization if l2_regularization is None else l2_regularization)
        self._dy = torch.empty((self.batch, model.n_boxes_total, model.n_classes + 12), dtype=torch.float32, device='cuda')
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
        self._n_slots = 1

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

    def _loss_and_dy(self, images, y_true, group=None):
        """forward + loss; leaves d loss / d y_pred in ``self._dy`` for the layer-wise backward.  Returns (loss, y_pred, dy).
        ``group``: the process group a 'global' loss reduces its batch-global quantities over (None: the default group)."""
        import torch
        self._attach()
        self._check_batch(images, y_true)
        y_pred = self.model.forward_device(images, training=True)
        y_true = y_true.to(dtype=torch.float32).contiguous()
        return self.loss.loss_and_grad(y_true, y_pred, self._dy, self.loss_mode, group=group), y_pred, self._dy

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
            self._n_slots = 2
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
        bucketed exchange is used from 4 ranks on."""
        import torch.distributed as dist
        on = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
        loss, _, dy = self._loss_and_dy(images, y_true, group)
        if not on:
            self._backward_layers(dy, len(self.model.specs) - 1, 0)
            self.apply(1.0)
            return loss
        if overlap is None:
            overlap = dist.get_world_size(group) > 2
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

    def _flatten(self, named):
        """The inverse of ``_unflatten``: dict with Keras names / layouts -> flat float32 ndarray in the gradient's layout."""
        m = self.model
        flat = np.empty((self.n_params,), np.float32)
        sp = self.spans()

        def put(key, a):
            o, c = sp[key]
            flat[o:o + c] = np.asarray(a, np.float32).reshape(-1)

        def ohwi(k):
            return np.asarray(k, np.float32).transpose(3, 0, 1, 2)
        for s in m.specs:
            if s.op == _ffi.OP_CONV:
                put((s.name, 'kernel'), ohwi(named[s.name + '/kernel']))
                put((s.name, 'bias'), named[s.name + '/bias'])
                if s.bn and (s.name, 'bn_gamma') in sp:
                    put((s.name, 'bn_gamma'), named[s.bn + '/gamma'])
                    put((s.name, 'bn_beta'), named[s.bn + '/beta'])
            elif s.op == _ffi.OP_HEAD:
                nb, cn, ln = s.n_boxes, s.params['conf_name'], s.params['loc_name']
                conf, loc = ohwi(named[cn + '/kernel']), ohwi(named[ln + '/kernel'])
                put((s.name, 'kernel'), np.concatenate([conf.reshape(nb, -1), loc.reshape(nb, -1)], axis=1))
                put((s.name, 'bias'), np.concatenate([np.reshape(named[cn + '/bias'], (nb, -1)), np.reshape(named[ln + '/bias'], (nb, -1))], axis=1))
            elif s.op == _ffi.OP_L2NORM:
                put((s.name, 'gamma'), named[s.name + '/gamma'])
        return flat

    # -- optimiser state (resuming a run from a full-model checkpoint) ---------------------------------
    def get_optimizer_state(self):
        """``{'iterations': int, 'slots': [dict, ...]}``: the step count and every optimiser slot that exists (SGD: the velocity;
        Adam: m, then v once an update has made it), each with Keras' weight names and layouts like :meth:`get_weights`."""
        import torch
        self._attach()
        out = torch.empty_like(self.grad)
        slots = []
        for slot in range(self._n_slots):
            _ffi.check(_ffi.lib().ssdk_trainer_read_opt_state(self.handle, slot, _ffi.dptr(out), _ffi.stream_ptr()))
            slots.append(self._unflatten(out.cpu().numpy()))
        return {'iterations': int(self.iterations), 'slots': slots}

    def set_optimizer_state(self, state):
        """Overwrite the optimiser state with ``state`` as :meth:`get_optimizer_state` returns it (checked first by
        :func:`check_optimizer_state`); the next update continues from it, bit for bit.  The state does not depend on the batch
        size, so it may come from a trainer built for another one."""
        import torch
        check_optimizer_state(self.model, self.optimizer, state)
        self._attach()
        slots = list(state['slots'])
        if len(slots) < self._n_slots:               # an Adam state from before its first update: v is zero again
            slots.append({k: np.zeros_like(v) for k, v in slots[0].items()})
        for slot, named in enumerate(slots):
            src = torch.from_numpy(self._flatten(named)).cuda()
            _ffi.check(_ffi.lib().ssdk_trainer_write_opt_state(self.handle, slot, _ffi.dptr(src), _ffi.stream_ptr()))
        self._n_slots = len(slots)
        self.iterations = int(state['iterations'])

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
