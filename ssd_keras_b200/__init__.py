"""ssd_keras_b200 -- the SSD detection hot path of pierluigiferrari/ssd_keras on NVIDIA H100 (sm_90a).

The sub-packages mirror the reference's module layout, so ``from ssd_keras_b200.models.keras_ssd300 import ssd_300``
replaces ``from models.keras_ssd300 import ssd_300`` and so on.  The hot path -- model forward / backward, encoder, decoders,
loss, optimiser -- runs in hand-written CUDA kernels inside ``_lib/libssdk.so`` (C-ABI in ``include/ssdk.h``); there is no CPU
fallback and no PyTorch fallback for it.  A few stand-alone helpers kept for API completeness (``matching_utils``,
``intersection_area``, ``SSDLoss.smooth_L1_loss`` / ``log_loss``) are short tensor expressions on the device; the fused kernels
compute the same quantities on the hot path.  ``training.SSDTrainer`` is what ``model.compile`` + ``train_on_batch`` are in the
reference's notebooks.
"""
__version__ = '0.1.0'


def _exports():
    from .models.keras_ssd300 import ssd_300
    from .models.keras_ssd512 import ssd_512
    from .models.keras_ssd7 import build_model, ssd_7
    from .keras_layers.keras_layer_AnchorBoxes import AnchorBoxes
    from .keras_layers.keras_layer_L2Normalization import L2Normalization
    from .keras_layers.keras_layer_DecodeDetections import DecodeDetections
    from .keras_layers.keras_layer_DecodeDetectionsFast import DecodeDetectionsFast
    from .keras_loss_function.keras_ssd_loss import SSDLoss
    from .ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder, DegenerateBoxError
    from .ssd_encoder_decoder.ssd_output_decoder import decode_detections, decode_detections_fast
    from .bounding_box_utils.bounding_box_utils import iou, convert_coordinates, intersection_area
    from .ssd_encoder_decoder.matching_utils import match_bipartite_greedy, match_multi
    from .training import SSDTrainer
    return locals()


_NAMES = ('ssd_300', 'ssd_512', 'build_model', 'ssd_7', 'AnchorBoxes', 'L2Normalization', 'DecodeDetections',
          'DecodeDetectionsFast', 'SSDLoss', 'SSDInputEncoder', 'DegenerateBoxError', 'decode_detections',
          'decode_detections_fast', 'iou', 'convert_coordinates', 'intersection_area', 'match_bipartite_greedy', 'match_multi',
          'SSDTrainer')


def __getattr__(name):
    if name in _NAMES:
        return _exports()[name]
    raise AttributeError(name)
