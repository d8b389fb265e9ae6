"""Regenerates tests/golden/ref_fuzz_golden.npz: the reference's own results on the seeded random inputs of
tests/test_oracle_vs_reference_fuzz_cpu.py (NumPy half) and tests/test_oracle_vs_reference_tf_fuzz_cpu.py (loss / decode layers
over tf_shim.py).  Needs a checkout of the reference:  python tests/golden/make_fuzz_golden.py /path/to/ssd_keras"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def main(ref_root):
    sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), HERE, ref_root]
    np.float = float    # noqa  the reference targets NumPy < 1.24 (caller-side aliases, SURVEY.md section 8c)
    np.int = int        # noqa
    import test_oracle_vs_reference_fuzz_cpu as fz
    import test_oracle_vs_reference_tf_fuzz_cpu as tfz
    from bounding_box_utils.bounding_box_utils import convert_coordinates, convert_coordinates2, iou
    from ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    from ssd_encoder_decoder.ssd_output_decoder import decode_detections, decode_detections_fast
    import tf_shim
    tf_shim.install()
    from keras_layers.keras_layer_DecodeDetections import DecodeDetections
    from keras_layers.keras_layer_DecodeDetectionsFast import DecodeDetectionsFast
    from keras_loss_function.keras_ssd_loss import SSDLoss
    ref = dict(convert_coordinates=convert_coordinates, convert_coordinates2=convert_coordinates2, iou=iou, SSDInputEncoder=SSDInputEncoder,
               decode_detections=decode_detections, decode_detections_fast=decode_detections_fast,
               DecodeDetections=DecodeDetections, DecodeDetectionsFast=DecodeDetectionsFast, SSDLoss=SSDLoss)
    out = {}

    def put(prefix, arrays):
        out[prefix + '/n'] = np.array(len(arrays))
        for i, a in enumerate(arrays):
            out['%s/%d' % (prefix, i)] = np.asarray(a)
    with np.errstate(all='ignore'):
        for seed in range(40):
            put('encoder/%d' % seed, fz.reference_encoder(ref, seed))
        for seed in range(25):
            put('decoders/%d' % seed, fz.reference_decoders(ref, seed))
        for seed in range(10):
            put('box_math/%d' % seed, fz.reference_box_math(ref, seed))
        for seed in range(20):
            out['loss/%d' % seed] = tfz.reference_loss(ref, seed)
            for i, a in enumerate(tfz.reference_decode_layers(ref, seed)):
                out['decode_layers/%d/%d' % (seed, i)] = a
    np.savez_compressed(os.path.join(HERE, 'ref_fuzz_golden.npz'), **out)


if __name__ == '__main__':
    main(sys.argv[1])
