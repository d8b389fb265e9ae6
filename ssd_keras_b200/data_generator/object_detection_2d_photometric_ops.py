"""The photometric ops as planners for ``DataGenerator.generate`` (the reference's object_detection_2d_photometric_ops.py):
``ConvertColor`` (RGB <-> HSV), ``ConvertDataType``, ``ConvertTo3Channels``, ``Brightness``, ``Contrast``, ``Saturation``,
``Hue``, ``ChannelSwap``, ``HistogramEqualization`` and their random forms.  The device runs them as a prefix of each image's
op list: they must come before every op that changes the image geometry, which ``generate()`` checks when it plans a batch.
Like the reference classes, ``Brightness`` / ``Contrast`` / ``Saturation`` / ``Hue`` expect a float32 image
(``ConvertDataType('float32')`` first, HSV for the last two), and the colour conversions and ``HistogramEqualization`` a uint8
one; the list must end in uint8.  Not covered: conversion to GRAY (``NotImplementedError`` when planned) and ``Gamma`` /
``RandomGamma``, whose ``__call__`` fails in the reference.

``ConvertTo3Channels``: the device converts every image to 3 channels first (gray is replicated, RGBA drops alpha), so it adds
no op.

``RandomBrightness``, ``RandomContrast``, ``RandomSaturation`` and ``RandomHue`` draw ``uniform(0, 1)`` against ``prob``, then
their parameter only when they apply, as the reference does.  ``draw()`` makes those draws and returns the parameter (``None``
when the op does not apply); ``plan()`` returns the op record alone.  Like the reference classes, the records expect the float32
image (HSV for saturation and hue) that the chains' conversions give: the chains put them into ``batch_assembly.photometric_ops``,
which adds those conversions."""
import numpy as np

from . import batch_assembly as ba
from .object_detection_2d_geometric_ops import DevicePlanner


class ConvertTo3Channels(DevicePlanner):
    def plan(self, img_height, img_width, labels):
        return [], img_height, img_width, labels


class ConvertColor(DevicePlanner):
    """``ConvertColor(current, to)``: uint8 ``cv2.cvtColor`` between RGB and HSV; ``current == to`` leaves the image alone."""

    def __init__(self, current='RGB', to='HSV', keep_3ch=True):
        if not ((current in {'RGB', 'HSV'}) and (to in {'RGB', 'HSV', 'GRAY'})):
            raise NotImplementedError
        self.current = current
        self.to = to
        self.keep_3ch = keep_3ch

    def plan(self, img_height, img_width, labels):
        if self.to == 'GRAY':
            raise NotImplementedError('ConvertColor to GRAY is not supported on the device')
        return ([] if self.current == self.to else [ba.convert_color(self.current, self.to)]), img_height, img_width, labels


class ConvertDataType(DevicePlanner):
    """``ConvertDataType(to)``: ``astype(float32)``, or ``np.round`` and ``astype(uint8)``."""

    def __init__(self, to='uint8'):
        if not (to == 'uint8' or to == 'float32'):
            raise ValueError("`to` can be either of 'uint8' or 'float32'.")
        self.to = to

    def plan(self, img_height, img_width, labels):
        return [ba.convert_dtype(self.to)], img_height, img_width, labels


class _Photometric(DevicePlanner):
    """A deterministic op: ``op(value)``, the value in the attribute ``value_name``."""

    def plan(self, img_height, img_width, labels):
        return [self.op(getattr(self, self.value_name))], img_height, img_width, labels


class Brightness(_Photometric):
    """``Brightness(delta)``: ``np.clip(image + delta, 0, 255)`` on an RGB float32 image."""
    op, value_name = staticmethod(ba.brightness), 'delta'

    def __init__(self, delta):
        self.delta = delta


class Contrast(_Photometric):
    """``Contrast(factor)``: ``np.clip(127.5 + factor * (image - 127.5), 0, 255)`` on an RGB float32 image."""
    op, value_name = staticmethod(ba.contrast), 'factor'

    def __init__(self, factor):
        if factor <= 0.0:
            raise ValueError("It must be `factor > 0`.")
        self.factor = factor


class Saturation(_Photometric):
    """``Saturation(factor)``: the S channel of an HSV float32 image times ``factor``, clipped."""
    op, value_name = staticmethod(ba.saturation), 'factor'

    def __init__(self, factor):
        if factor <= 0.0:
            raise ValueError("It must be `factor > 0`.")
        self.factor = factor


class Hue(_Photometric):
    """``Hue(delta)``: ``(H + delta) % 180`` on the H channel of an HSV float32 image."""
    op, value_name = staticmethod(ba.hue), 'delta'

    def __init__(self, delta):
        if not (-180 <= delta <= 180):
            raise ValueError("`delta` must be in the closed interval `[-180, 180]`.")
        self.delta = delta


class ChannelSwap(_Photometric):
    """``ChannelSwap(order)``: ``image[:, :, order]``."""
    op, value_name = staticmethod(ba.channel_swap), 'order'

    def __init__(self, order):
        self.order = order


class HistogramEqualization(DevicePlanner):
    """``HistogramEqualization()``: ``cv2.equalizeHist`` of channel 2 (V of an HSV image) on a uint8 image.  The reference's
    writes into its input, so with images held in memory a 3-channel dataset image it receives directly is changed for later
    epochs; the device leaves the dataset alone."""

    def plan(self, img_height, img_width, labels):
        return [ba.equalize_hist()], img_height, img_width, labels


class RandomHistogramEqualization(DevicePlanner):
    """``HistogramEqualization`` when ``np.random.uniform(0, 1) >= 1 - prob``."""

    def __init__(self, prob=0.5):
        self.prob = prob
        self.equalize = HistogramEqualization()

    def plan(self, img_height, img_width, labels):
        if np.random.uniform(0, 1) >= (1.0 - self.prob):
            return self.equalize.plan(img_height, img_width, labels)
        return [], img_height, img_width, labels


class RandomChannelSwap(DevicePlanner):
    """With ``np.random.uniform(0, 1) >= 1 - prob``, ``ChannelSwap`` to one of the five other orders, ``np.random.randint(5)``."""

    def __init__(self, prob=0.5):
        self.prob = prob
        self.permutations = ((0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0))
        self.swap_channels = ChannelSwap(order=(0, 1, 2))

    def plan(self, img_height, img_width, labels):
        if np.random.uniform(0, 1) >= (1.0 - self.prob):
            self.swap_channels.order = self.permutations[np.random.randint(5)]
            return self.swap_channels.plan(img_height, img_width, labels)
        return [], img_height, img_width, labels


class _RandomPhotometric(DevicePlanner):
    """``uniform(0, 1) >= 1 - prob``, then ``uniform(lower, upper)``."""

    def draw(self):
        if np.random.uniform(0, 1) >= (1.0 - self.prob):
            return np.random.uniform(self.lower, self.upper)
        return None

    def plan(self, img_height, img_width, labels):
        value = self.draw()
        return ([] if value is None else [self.op(value)]), img_height, img_width, labels


class RandomBrightness(_RandomPhotometric):
    """Adds a delta drawn from ``[lower, upper]`` to an RGB float32 image."""
    op = staticmethod(ba.brightness)

    def __init__(self, lower=-84, upper=84, prob=0.5):
        if lower >= upper:
            raise ValueError("`upper` must be greater than `lower`.")
        self.lower = float(lower)
        self.upper = float(upper)
        self.prob = prob


class RandomContrast(_RandomPhotometric):
    """Scales an RGB float32 image about 127.5 by a factor drawn from ``[lower, upper]``."""
    op = staticmethod(ba.contrast)

    def __init__(self, lower=0.5, upper=1.5, prob=0.5):
        if lower >= upper:
            raise ValueError("`upper` must be greater than `lower`.")
        self.lower = lower
        self.upper = upper
        self.prob = prob


class RandomSaturation(_RandomPhotometric):
    """Scales the S channel of an HSV float32 image by a factor drawn from ``[lower, upper]``."""
    op = staticmethod(ba.saturation)

    def __init__(self, lower=0.3, upper=2.0, prob=0.5):
        if lower >= upper:
            raise ValueError("`upper` must be greater than `lower`.")
        self.lower = lower
        self.upper = upper
        self.prob = prob


class RandomHue(_RandomPhotometric):
    """Adds a delta drawn from ``[-max_delta, max_delta]`` to the H channel of an HSV float32 image."""
    op = staticmethod(ba.hue)

    def __init__(self, max_delta=18, prob=0.5):
        if not (0 <= max_delta <= 180):
            raise ValueError("`max_delta` must be in the closed interval `[0, 180]`.")
        self.max_delta = max_delta
        self.prob = prob

    @property
    def lower(self):
        return -self.max_delta

    @property
    def upper(self):
        return self.max_delta


def photometric_draws(brightness, contrast, saturation, hue, sequence):
    """The photometric part of a chain's sequence 1 (brightness, contrast, saturation, hue) or 2 (brightness, saturation, hue,
    contrast), drawn in that order -> ``batch_assembly.photometric_ops`` with the conversions around them."""
    b = brightness.draw()
    c = contrast.draw() if sequence == 1 else None
    s = saturation.draw()
    h = hue.draw()
    if sequence == 2:
        c = contrast.draw()
    return ba.photometric_ops(sequence, brightness=b, contrast=c, saturation=s, hue=h)
