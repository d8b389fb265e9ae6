"""The small dataset of tests/golden/make_ssd_augmentation_golden.py, made from a seed with NumPy alone so that the golden file
holds the reference's outputs but not its inputs: nine images (gray, RGB and RGBA; smaller than the 90 x 120 output and larger,
two of them larger than 300) and label sets that are empty, hold one box, many boxes or boxes at the edges.  ``digest`` lets a
test check that the images are the ones the golden was recorded from."""
import hashlib

import numpy as np

SEED = 20261018
SHAPES = [(160, 210, 3), (97, 61), (310, 330, 4), (75, 110, 3), (120, 120, 3), (128, 96, 1), (305, 240, 3), (64, 64, 3), (140, 90, 4)]
COUNTS = [2, 1, 0, 6, 12, 1, 3, 0, 2]


def _image(rng, shape):
    """16 x 16 blocks of random colour, a diagonal ramp and 2 bits of noise: edges and gradients for every interpolation mode."""
    h, w = shape[:2]
    c = shape[2] if len(shape) == 3 else 1
    base = rng.integers(0, 200, (h // 16 + 1, w // 16 + 1, c), dtype=np.int64)
    img = np.repeat(np.repeat(base, 16, 0), 16, 1)[:h, :w]
    img = img + ((np.arange(h)[:, None] + np.arange(w)[None, :]) * 48 // (h + w))[:, :, None]
    img = (img + rng.integers(0, 4, img.shape)).astype(np.uint8)
    return img[:, :, 0] if len(shape) == 2 else img


def _boxes(rng, h, w, n, edge):
    out = []
    for _ in range(n):
        x0, y0 = int(rng.integers(0, w - 8)), int(rng.integers(0, h - 8))
        x1, y1 = int(rng.integers(x0 + 4, w + 1)), int(rng.integers(y0 + 4, h + 1))
        if edge:
            x0, x1 = (0, x1) if rng.integers(2) else (x0, w)
        out.append([int(rng.integers(1, 21)), x0, y0, x1, y1])
    return np.array(out, dtype=np.int64).reshape(-1, 5)


def dataset():
    """-> (images, labels): uint8 arrays and int64 (k, 5) label arrays [class_id, xmin, ymin, xmax, ymax]."""
    rng = np.random.default_rng(SEED)
    images = [_image(rng, s) for s in SHAPES]
    labels = [_boxes(rng, s[0], s[1], n, i % 3 == 0) for i, (s, n) in enumerate(zip(SHAPES, COUNTS))]
    return images, labels


def digest(images):
    h = hashlib.sha256()
    for im in images:
        h.update(str(im.shape).encode())
        h.update(np.ascontiguousarray(im).tobytes())
    return h.hexdigest()
