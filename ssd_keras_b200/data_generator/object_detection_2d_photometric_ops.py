"""``ConvertTo3Channels`` as a planner for ``DataGenerator.generate`` (the reference's object_detection_2d_photometric_ops.py):
the device converts every image to 3 channels first (gray is replicated, RGBA drops alpha), so it adds no op."""
from .object_detection_2d_geometric_ops import DevicePlanner


class ConvertTo3Channels(DevicePlanner):
    def plan(self, img_height, img_width, labels):
        return [], img_height, img_width, labels
