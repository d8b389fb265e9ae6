"""Class transfer for a trained SSD: re-shape the classifier heads of a weights file to another class set (the reference's
``misc_utils/tensor_sampling_utils.py`` and the loop of ``weight_sampling_tutorial.ipynb``).

``sample_tensors`` sub- and up-samples the axes of a group of tensors consistently.  It draws from the global ``np.random``
in the reference's order, so that under the same seed it returns the same arrays and leaves the generator in the same state;
its argument checks raise the reference's exceptions with the reference's messages.

``subsample_classifier_weights`` runs the tutorial's loop over the six ``*_mbox_conf`` heads of a Keras weights file and
writes a new file with only those twelve datasets replaced (``hdf5_lite.write_keras_file``: layer order, ``weight_names`` and
attributes as in the source).  ``subsample_classifier_arrays`` does the same on a ``{name: array}`` dict such as
``model.get_weights()`` returns.  All of this is host work on a few MB of weights, done once."""
import numpy as np

from . import hdf5_lite

SSD300_CLASSIFIER_NAMES = ['conv4_3_norm_mbox_conf', 'fc7_mbox_conf', 'conv6_2_mbox_conf', 'conv7_2_mbox_conf', 'conv8_2_mbox_conf',
                           'conv9_2_mbox_conf']


def _index_zero_and_random(n, k):
    """Index 0, then ``k - 1`` distinct indices of ``1..n-1`` drawn from ``np.random`` and sorted."""
    rest = np.sort(np.random.choice(np.arange(1, n), k - 1, replace=False))
    return np.concatenate([np.array([0]), rest])


def _init_kind(init, j):
    kind = 'gaussian' if init is None else init[j]
    if kind == 'gaussian' or kind == 'zeros':
        return kind
    raise ValueError("Valid initializations are 'gaussian' and 'zeros', but received '{}'.".format(kind))


def _filled(kind, shape, mean, stddev):
    """A float64 tensor of ``shape`` holding the values new elements start from."""
    if kind == 'gaussian':
        return np.random.normal(loc=mean, scale=stddev, size=shape)
    return np.zeros(shape)


def sample_tensors(weights_list, sampling_instructions, axes=None, init=None, mean=0.0, stddev=0.005):
    """Sub-sample and / or up-sample the axes of the tensors in ``weights_list``, the same elements of an axis for every tensor.

    ``weights_list``: NumPy arrays, the one with the most axes first (a kernel, then its bias).  ``sampling_instructions``: one
    entry per axis of the first tensor, either a list / tuple of indices to keep (in that order, duplicates allowed) or a Python
    ``int``: the axis' own length keeps it, a smaller number keeps index 0 and that many minus one random other indices
    (sorted), a larger number keeps every element and inserts new ones at random positions (index 0 stays in place).
    ``axes``: for each tensor after the first, the axes of the first tensor its axes correspond to (``[[3]]`` for a bias).
    ``init``: per tensor, how inserted elements start: ``'gaussian'`` (``normal(mean, stddev)``, the default) or ``'zeros'``.

    Returns the list of new tensors.  Up-sampled tensors are float64 (the fill is drawn as float64); sub-sampled ones keep
    their dtype."""
    first = weights_list[0]
    if not isinstance(sampling_instructions, (list, tuple)) or len(sampling_instructions) != first.ndim:
        raise ValueError("The sampling instructions must be a list whose length is the number of dimensions of the first tensor "
                         "in `weights_list`.")
    if init is not None and len(init) != len(weights_list):
        raise ValueError("`init` must either be `None` or a list of strings that has the same length as `weights_list`.")

    keep, out_shape, grown = [], [], []
    for axis, inst in enumerate(sampling_instructions):
        n = first.shape[axis]
        if isinstance(inst, (list, tuple)):
            largest = np.amax(np.array(inst))
            if largest >= n:
                raise ValueError("The sample instructions for dimension {} contain index {}, which is greater than the length of "
                                 "that dimension.".format(axis, largest))
            keep.append(np.array(inst))
            out_shape.append(len(inst))
        elif isinstance(inst, int):
            out_shape.append(inst)
            if inst == n:
                keep.append(np.arange(inst))
            elif inst < n:
                keep.append(_index_zero_and_random(n, inst))
            else:
                keep.append(np.arange(n))
                grown.append(axis)
        else:
            raise ValueError("Each element of the sampling instructions must be either an integer or a list/tuple of integers, "
                             "but received `{}`".format(type(inst)))

    kept = [np.copy(first[np.ix_(*keep)])]
    for j in range(1, len(weights_list)):
        kept.append(np.copy(weights_list[j][np.ix_(*[keep[a] for a in axes[j - 1]])]))
    if not grown:
        return kept

    out_shape = np.array(out_shape)
    out = [_filled(_init_kind(init, 0), out_shape, mean, stddev)]
    places = [np.arange(k) for k in kept[0].shape]
    for axis in grown:
        places[axis] = _index_zero_and_random(out[0].shape[axis], kept[0].shape[axis])
    out[0][np.ix_(*places)] = kept[0]
    for j in range(1, len(weights_list)):
        t = _filled(_init_kind(init, j), out_shape[axes[j - 1]], mean, stddev)
        t[np.ix_(*[places[a] for a in axes[j - 1]])] = kept[j]
        out.append(t)
    return out


def classifier_indices(out_channels, n_classes_source, classes_of_interest):
    """The sampling instruction of a classifier head's output axis, as ``weight_sampling_tutorial.ipynb`` computes it: a list
    of classes is repeated for every box of the head (class ``c`` of box ``i`` is column ``c + i * n_classes_source``); an
    integer asks for that many classes per box, ``int(classes_of_interest * (out_channels / n_classes_source))`` random columns
    in all (``sample_tensors`` draws them over the whole axis, so they need not be the same classes for every box)."""
    if isinstance(classes_of_interest, (list, tuple)):
        per_box = [np.array(classes_of_interest) + i * n_classes_source for i in range(int(out_channels / n_classes_source))]
        return list(np.concatenate(per_box))
    if isinstance(classes_of_interest, int):
        return int(classes_of_interest * (out_channels / n_classes_source))
    raise ValueError("`classes_of_interest` must be either an integer or a list/tuple.")


def subsample_classifier_arrays(weights, classifier_names, n_classes_source, classes_of_interest, init=('gaussian', 'zeros'),
                                mean=0.0, stddev=0.005):
    """The tutorial's loop on a ``{'<layer>/kernel': array, '<layer>/bias': array, ...}`` dict (``model.get_weights()``,
    ``hdf5_lite.read_keras_weights``): for each head in ``classifier_names``, in that order, one ``sample_tensors`` call on its
    kernel and bias over the output axis.  Returns a new dict, in the order of ``weights``, with the heads replaced; the other
    arrays are the same objects.  ``ssd_300(..., n_classes=k).set_weights(result)`` takes it directly."""
    out = dict(weights)
    for name in classifier_names:
        kernel, bias = weights[name + '/kernel'], weights[name + '/bias']
        height, width, in_channels, out_channels = kernel.shape
        new_kernel, new_bias = sample_tensors(weights_list=[kernel, bias],
                                              sampling_instructions=[height, width, in_channels,
                                                                     classifier_indices(out_channels, n_classes_source, classes_of_interest)],
                                              axes=[[3]], init=init, mean=mean, stddev=stddev)
        out[name + '/kernel'], out[name + '/bias'] = new_kernel, new_bias
    return out


def subsample_classifier_weights(source_path, destination_path, classifier_names, n_classes_source, classes_of_interest,
                                 init=('gaussian', 'zeros'), mean=0.0, stddev=0.005):
    """``weight_sampling_tutorial.ipynb`` sections 1-4 without h5py: read the Keras HDF5 file at ``source_path`` (weights file or
    full-model file), sample the kernel and bias of every head in ``classifier_names`` as ``subsample_classifier_arrays`` does,
    and write ``destination_path`` with the same layers, ``weight_names`` and attributes and only those datasets replaced.  A
    replaced dataset is stored in the dtype ``sample_tensors`` returned (float32 after sub-sampling a float32 file, float64 after
    up-sampling), as h5py's ``create_dataset(data=...)`` does.  A full-model file loses its ``training_config`` and
    ``/optimizer_weights``: they belong to the old heads.  Then ``ssd_300(..., n_classes=k).load_weights(destination_path,
    by_name=True)``."""
    source = hdf5_lite.read_keras_file(source_path)
    weights = source.weights()
    new = subsample_classifier_arrays(weights, classifier_names, n_classes_source, classes_of_interest, init, mean, stddev)
    replaced = {k: v for k, v in new.items() if v is not weights[k]}
    hdf5_lite.write_keras_file(destination_path, source, replace=replaced)
