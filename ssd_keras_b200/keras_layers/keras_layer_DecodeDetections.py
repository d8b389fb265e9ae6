"""``DecodeDetections`` on H100 (reference ``keras_layers/keras_layer_DecodeDetections.py:27-283``):
a callable with the reference layer's constructor arguments; ``layer(y_pred)`` maps a float32 CUDA
tensor ``(B, P, C+12)`` to ``(B, top_k, 6)`` rows ``[class_id, confidence, xmin, ymin, xmax, ymax]``,
sorted by confidence and zero padded, through ``ssdk_decode`` (``csrc/decode.cu``)."""
from ..ssd_encoder_decoder.ssd_output_decoder import PER_CLASS, decode_device


class DecodeDetections:
    _MODE = PER_CLASS

    def __init__(self, confidence_thresh=0.01, iou_threshold=0.45, top_k=200, nms_max_output_size=400,
                 coords='centroids', normalize_coords=True, img_height=None, img_width=None, **kwargs):
        if normalize_coords and ((img_height is None) or (img_width is None)):
            raise ValueError("If relative box coordinates are supposed to be converted to absolute coordinates, the decoder needs "
                             "the image size in order to decode the predictions, but `img_height == {}` and `img_width == {}`"
                             .format(img_height, img_width))
        if coords != 'centroids':
            raise ValueError("The DetectionOutput layer currently only supports the 'centroids' coordinate format.")
        self.confidence_thresh = confidence_thresh
        self.iou_threshold = iou_threshold
        self.top_k = top_k
        self.normalize_coords = normalize_coords
        self.img_height = img_height
        self.img_width = img_width
        self.coords = coords
        self.nms_max_output_size = nms_max_output_size
        self.name = kwargs.get('name', 'decoded_predictions')

    def call(self, y_pred, mask=None, return_index=False):
        res = decode_device(y_pred, self._MODE, True, self.confidence_thresh, self.iou_threshold, self.top_k,
                            self.nms_max_output_size, self.coords, self.normalize_coords, self.img_height, self.img_width,
                            return_index=return_index)
        return (res[0], res[2]) if return_index else res[0]

    __call__ = call

    def build(self, input_shape):
        """Keras calls this before the first ``call``; nothing is allocated here (reference ``build`` only records the input spec)."""
        self.input_shape = tuple(input_shape)

    def compute_output_shape(self, input_shape):
        return (input_shape[0], self.top_k, 6)

    def get_config(self):
        return {'confidence_thresh': self.confidence_thresh, 'iou_threshold': self.iou_threshold, 'top_k': self.top_k,
                'nms_max_output_size': self.nms_max_output_size, 'coords': self.coords,
                'normalize_coords': self.normalize_coords, 'img_height': self.img_height, 'img_width': self.img_width}
