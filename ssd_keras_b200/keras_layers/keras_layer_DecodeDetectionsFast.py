"""``DecodeDetectionsFast`` on H100 (reference ``keras_layers/keras_layer_DecodeDetectionsFast.py:29-266``):
class = argmax over all classes, background dropped, one global NMS, top-k / zero padding."""
from ..ssd_encoder_decoder.ssd_output_decoder import FAST
from .keras_layer_DecodeDetections import DecodeDetections


class DecodeDetectionsFast(DecodeDetections):
    _MODE = FAST
