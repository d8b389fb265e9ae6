"""Record uint8 cv2.resize with INTER_CUBIC, INTER_AREA and INTER_LANCZOS4 (OpenCV's own code: IPP off) on a fixed set of
images and size pairs -> ref_resize_interp_golden.npz.  Run from the repository root with OpenCV 4.13 installed."""
import os

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SIZES = [(27, 33, 44, 47), (61, 73, 40, 41), (60, 60, 20, 30), (60, 60, 24, 15), (1, 9, 5, 1), (9, 1, 1, 5),
         (17, 23, 16, 22), (90, 135, 45, 45), (64, 64, 21, 32), (5, 7, 41, 39)]


def main():
    cv2.ipp.setUseIPP(False)
    rng = np.random.default_rng(2026)
    out = {}
    n = 0
    for mode in (cv2.INTER_CUBIC, cv2.INTER_AREA, cv2.INTER_LANCZOS4):
        for h, w, oh, ow in SIZES:
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            out['img%d' % n], out['mode%d' % n], out['oh%d' % n], out['ow%d' % n] = img, mode, oh, ow
            out['out%d' % n] = cv2.resize(img, (ow, oh), interpolation=mode)
            n += 1
    out['n'] = n
    np.savez_compressed(os.path.join(HERE, 'ref_resize_interp_golden.npz'), **out)


if __name__ == '__main__':
    main()
