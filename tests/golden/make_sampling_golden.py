#!/usr/bin/env python
"""Golden vectors for the class transfer of weight_sampling_tutorial.ipynb, from the REAL reference:

- misc_utils/tensor_sampling_utils.sample_tensors on seeded inputs: for every case and seed (``np.random.seed(s)`` before the
  call) the returned arrays (or, for the tutorial-sized kernels, their SHA-256 with shape and dtype) and the global generator's
  state afterwards; for every error case the exception's type and message;
- the tutorial's sample chain ConvertTo3Channels -> RandomMaxCropFixedAR -> Resize on seeded uint8 images of random sizes with
  three boxes each: the patch CropPad was given, the generator's next draw afterwards, the resized image and the boxes.

Writes tests/golden/ref_sampling_golden.npz.  Build container only (needs the reference tree and cv2)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get('SSD_REFERENCE_ROOT', '/root/reference')
sys.path.insert(0, REF_ROOT)
sys.path.insert(0, os.path.join(HERE, '..'))

from misc_utils.tensor_sampling_utils import sample_tensors                                 # noqa: E402
from data_generator.object_detection_2d_photometric_ops import ConvertTo3Channels              # noqa: E402
from data_generator.object_detection_2d_geometric_ops import Resize                            # noqa: E402
import data_generator.object_detection_2d_patch_sampling_ops as pso                            # noqa: E402
from sampling_cases import (CASES, DIGEST_ABOVE, ERRORS, SEEDS, crop_cases, crop_images, crop_labels, sha,  # noqa: E402
                            tensors)

def state_arrays(prefix):
    kind, keys, pos, has_gauss, cached = np.random.get_state()
    return {prefix + '/state_keys_sha': np.array(sha(keys)), prefix + '/state_pos': np.array(pos),
            prefix + '/state_has_gauss': np.array(has_gauss), prefix + '/state_cached_gaussian': np.array(cached)}


def sampling_arrays():
    out = {}
    for name, (seed, shapes, dtype, inst, kw) in CASES.items():
        for s in SEEDS:
            w = tensors(seed, shapes, np.dtype(dtype))
            np.random.seed(s)
            res = sample_tensors(w, inst, **kw)
            p = 'case/%s/%d' % (name, s)
            out[p + '/n'] = np.array(len(res))
            for i, r in enumerate(res):
                if r.size > DIGEST_ABOVE:
                    out['%s/%d/sha' % (p, i)] = np.array(sha(r))
                    out['%s/%d/shape' % (p, i)] = np.array(r.shape)
                    out['%s/%d/dtype' % (p, i)] = np.array(r.dtype.str)
                else:
                    out['%s/%d' % (p, i)] = r
            out.update(state_arrays(p))
        print('case', name, [r.shape for r in res], [r.dtype for r in res])
    for name, (seed, shapes, dtype, inst, kw) in ERRORS.items():
        w = tensors(seed, shapes, np.dtype(dtype))
        np.random.seed(0)
        try:
            sample_tensors(w, inst, **kw)
        except Exception as e:                                   # noqa: BLE001 -- the reference's own exception is the datum
            out['error/%s/type' % name] = np.array(type(e).__name__)
            out['error/%s/msg' % name] = np.array(str(e))
            out.update(state_arrays('error/' + name))
            print('error', name, type(e).__name__, str(e)[:80])
        else:
            raise AssertionError('the reference was expected to raise on ' + name)
    return out


def crop_arrays():
    out = {}
    patches, nxt, outs, labs = [], [], [], []
    orig = pso.CropPad.__call__

    def record(this, image, labels=None, return_inverter=False):
        patches.append((this.patch_ymin, this.patch_xmin, this.patch_height, this.patch_width))
        return orig(this, image, labels, return_inverter)
    pso.CropPad.__call__ = record
    try:
        for k, ((shape, ar, oh, ow), img, lab) in enumerate(zip(crop_cases(), crop_images(), crop_labels())):
            chain = [ConvertTo3Channels(), pso.RandomMaxCropFixedAR(patch_aspect_ratio=ar), Resize(height=oh, width=ow)]
            np.random.seed(100 + k)
            x, y = img, lab.copy()
            for t in chain:
                x, y = t(x, y)
            nxt.append(np.random.randint(0, 2 ** 31 - 1))
            outs.append(x)
            labs.append(np.asarray(y, np.float64).reshape(-1, 5))
    finally:
        pso.CropPad.__call__ = orig
    out['crop/n'] = np.array(len(outs))
    out['crop/image_sha'] = np.array([sha(im) for im in crop_images()])
    out['crop/patches'] = np.array(patches, np.int64)
    out['crop/next_draw'] = np.array(nxt, np.int64)
    for k, (x, y) in enumerate(zip(outs, labs)):
        out['crop/out/%d' % k] = x
        out['crop/labels/%d' % k] = y
    shapes = np.array([im.shape[:2] for im in crop_images()])
    ars = np.array([c[1] for c in crop_cases()])
    wide = shapes[:, 1] / shapes[:, 0] < ars
    assert wide.any() and (~wide).any(), 'both aspect-ratio branches'
    p = out['crop/patches']
    assert (p[:, 0] > 0).any() and (p[:, 1] > 0).any(), 'both offsets drawn non-zero somewhere'
    return out


def main():
    arrays = sampling_arrays()
    arrays.update(crop_arrays())
    np.savez_compressed(os.path.join(HERE, 'ref_sampling_golden.npz'), **arrays)
    print('wrote ref_sampling_golden.npz', len(arrays), 'arrays')


if __name__ == '__main__':
    main()
