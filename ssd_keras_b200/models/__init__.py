"""Model builders (``ssd_300`` / ``ssd_512`` / ``build_model``) and ``load_model`` for the files ``SSDModel.save`` writes."""


def _json_attr(raw):
    import json
    if hasattr(raw, 'tobytes'):
        raw = raw.tobytes()
    if isinstance(raw, bytes):
        raw = raw.rstrip(b'\x00').decode()
    return json.loads(raw)


def load_model(filepath, custom_objects=None, compile=True):
    """``keras.models.load_model(filepath, custom_objects={...})`` for files written by :meth:`SSDModel.save`: rebuilds the model
    with the builder call stored in the file's ``model_config`` attribute and loads the weights.  The layers the reference passes
    in ``custom_objects`` (``AnchorBoxes`` / ``L2Normalization`` / ``DecodeDetections``, ``ssd300_inference.ipynb``) are built in.

    A file saved from a compiled model carries a ``training_config``; with ``compile=True`` the model comes back compiled with
    the stored optimizer and learning rate, and with the loss ``custom_objects['compute_loss']`` when that is an
    ``SSDLoss(...).compute_loss`` (the training notebooks' resume call), else an ``SSDLoss`` with the stored parameters.  A stored
    optimizer state is checked against the model and taken up by the first training step, at any batch size, so that
    ``fit_generator(..., initial_epoch=...)`` continues the saved run; ``compile``, ``set_weights`` and ``load_weights`` drop it.

    A full-model file saved by Keras itself describes an arbitrary Keras graph, which this package does not interpret: build the
    model with ``ssd_300(...)`` and ``load_weights(filepath, by_name=True)`` instead (the weights of such files are read)."""
    from ..misc_utils.hdf5_lite import read_attributes, read_optimizer_weights
    from . import keras_ssd300, keras_ssd512, keras_ssd7
    attrs = read_attributes(str(filepath))
    raw = attrs.get('model_config')
    if raw is None:
        raise ValueError('%s has no model_config attribute: it is a weights file; build the model and call load_weights()' % filepath)
    cfg = _json_attr(raw)
    if cfg.get('class_name') != 'SSDModel':
        raise ValueError('%s was saved by Keras (class_name %r): rebuild the architecture with ssd_300 / ssd_512 / build_model and '
                         'use load_weights(path, by_name=True)' % (filepath, cfg.get('class_name')))
    builders = {'ssd_300': keras_ssd300.ssd_300, 'ssd_512': keras_ssd512.ssd_512, 'build_model': keras_ssd7.build_model}
    b = cfg['config']['builder']
    if b not in builders:
        raise ValueError('unknown builder %r in %s' % (b, filepath))
    model = builders[b](**cfg['config']['kwargs'])
    model.load_weights(str(filepath), by_name=True)
    if compile and attrs.get('training_config') is not None:
        model._restore_training(_json_attr(attrs['training_config']), read_optimizer_weights(str(filepath)), custom_objects)
    return model
