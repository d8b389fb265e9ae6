"""The inputs of tests/golden/make_augmentation_chains_golden.py, made from a seed with NumPy alone so that the golden file holds
the reference's outputs but not its inputs, and the CSV of its ``parse_csv`` case.

- ``ssd7_dataset``: ten constant-size 60 x 96 images (gray, gray with one channel, RGB, RGBA) for the SSD7 chain;
- ``variable_dataset``: ten images of different sizes, none of them square, for the variable-input-size and satellite chains.

Label sets are empty, hold boxes at the image edges, boxes under 16 px^2 (the box filters drop them and the validators use up
their trials) and ordinary boxes; ``dtype=float`` adds half-pixel offsets to some coordinates.  ``digest`` lets a test check
that the images are the ones the golden was recorded from."""
import hashlib

import numpy as np

SEED = 20261019
SSD7_HW = (60, 96)
SSD7_CHANNELS = [3, 0, 4, 3, 1, 3, 3, 4, 0, 3]             # 0: a 2-D gray image
SSD7_COUNTS = [2, 0, 3, 1, 5, 0, 2, 4, 1, 3]
VARIABLE_SHAPES = [(70, 110, 3), (97, 61), (50, 90, 4), (64, 80, 3), (120, 75, 3), (45, 100, 1), (88, 66, 3), (59, 73, 3), (100, 140, 4),
                   (81, 57, 3)]
VARIABLE_COUNTS = [3, 1, 2, 4, 2, 1, 0, 6, 2, 3]


def _image(rng, shape):
    """8 x 8 blocks of random colour, a diagonal ramp and 2 bits of noise."""
    h, w = shape[:2]
    c = shape[2] if len(shape) == 3 else 1
    base = rng.integers(0, 200, (h // 8 + 1, w // 8 + 1, c), dtype=np.int64)
    img = np.repeat(np.repeat(base, 8, 0), 8, 1)[:h, :w]
    img = img + ((np.arange(h)[:, None] + np.arange(w)[None, :]) * 48 // (h + w))[:, :, None]
    img = (img + rng.integers(0, 4, img.shape)).astype(np.uint8)
    return img[:, :, 0] if len(shape) == 2 else img


def _boxes(rng, h, w, n, dtype):
    """n boxes: every third one tiny (2-3 px sides), every fourth one touching an image edge."""
    out = []
    for k in range(n):
        if k % 3 == 2:
            x0, y0 = int(rng.integers(0, w - 4)), int(rng.integers(0, h - 4))
            x1, y1 = x0 + int(rng.integers(2, 4)), y0 + int(rng.integers(2, 4))
        else:
            x0, y0 = int(rng.integers(0, w - 12)), int(rng.integers(0, h - 12))
            x1, y1 = int(rng.integers(x0 + 6, w + 1)), int(rng.integers(y0 + 6, h + 1))
        if k % 4 == 3:
            x0, x1 = (0, x1) if rng.integers(2) else (x0, w)
        out.append([int(rng.integers(1, 6)), x0, y0, x1, y1])
    labels = np.array(out, dtype=np.int64).reshape(-1, 5)
    if dtype == 'float':
        labels = labels.astype(np.float64)
        labels[:, 1:] += 0.5 * rng.integers(0, 2, labels[:, 1:].shape)
    return labels


def ssd7_dataset(dtype='int'):
    """-> (images, labels): uint8 arrays, (k, 5) label arrays [class_id, xmin, ymin, xmax, ymax], int64 or float64."""
    rng = np.random.default_rng(SEED)
    h, w = SSD7_HW
    images = [_image(rng, (h, w) if c == 0 else (h, w, c)) for c in SSD7_CHANNELS]
    labels = [_boxes(rng, h, w, n, dtype) for n in SSD7_COUNTS]
    return images, labels


def variable_dataset(dtype='int'):
    rng = np.random.default_rng(SEED + 1)
    images = [_image(rng, s) for s in VARIABLE_SHAPES]
    labels = [_boxes(rng, s[0], s[1], n, dtype) for s, n in zip(VARIABLE_SHAPES, VARIABLE_COUNTS)]
    return images, labels


def digest(images, labels):
    h = hashlib.sha256()
    for im, lab in zip(images, labels):
        h.update(str(im.shape).encode())
        h.update(np.ascontiguousarray(im).tobytes())
        h.update(str(lab.dtype).encode())
        h.update(np.ascontiguousarray(lab).tobytes())
    return h.hexdigest()


# parse_csv: columns in a permuted order with an extra column, cells padded with spaces, rows out of order, a file name with
# two dots, and classes outside ``CSV_INCLUDE``.
CSV_INPUT_FORMAT = ['ymax', 'image_name', 'xmin', 'class_id', 'xmax', 'ymin']
CSV_INCLUDE = [1, 2, 4]
CSV_SAMPLE = 0.6


def csv_text():
    rng = np.random.default_rng(SEED + 2)
    names = ['img_%02d.png' % i for i in range(14)] + ['frame.v2.jpg', 'b.png', 'a10.png', 'a9.png']
    rows = []
    for name in names:
        for _ in range(int(rng.integers(1, 4))):
            x0, y0 = int(rng.integers(0, 200)), int(rng.integers(0, 150))
            cells = {'image_name': name, 'class_id': int(rng.integers(1, 6)), 'xmin': x0, 'ymin': y0,
                     'xmax': x0 + int(rng.integers(1, 80)), 'ymax': y0 + int(rng.integers(1, 60))}
            rows.append([(' %s ' % cells[k]) if rng.integers(2) else str(cells[k]) for k in CSV_INPUT_FORMAT] + ['extra'])
    order = rng.permutation(len(rows))
    lines = [','.join(CSV_INPUT_FORMAT + ['note'])] + [','.join(rows[i]) for i in order]
    return '\n'.join(lines) + '\n'
