"""The photometric ops of the training chains as planners for ``DataGenerator.generate`` (the reference's
object_detection_2d_photometric_ops.py).

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
