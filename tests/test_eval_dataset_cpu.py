"""CPU checks of the dataset half of the evaluation against the REAL reference (tests/golden/ref_eval_dataset_golden.npz, made
by tests/golden/make_eval_dataset_golden.py): the 'pad' patches, the inverse-transformed rows, the per-class lists, the VOC
txt texts and the COCO JSON text restated by oracle/evalops.py, and the package's own patch draws."""
import hashlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)
from oracle import evalops  # noqa: E402

GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'ref_eval_dataset_golden.npz')
RUNS = {'resize_inf': ('resize', 'inference', False, (300, 300), 8, 0),
        'pad_inf_r4': ('pad', 'inference', 4, (300, 300), 8, 1),
        'pad_inf_r3_wide': ('pad', 'inference', 3, (300, 480), 6, 2),
        'resize_train_wide': ('resize', 'training', False, (300, 480), 8, 0),
        'pad_train_r4': ('pad', 'training', 4, (300, 300), 7, 3)}
N_CLASSES = 3


@pytest.fixture(scope='module')
def g():
    return dict(np.load(GOLDEN, allow_pickle=False))


SHAPES = [(375, 500, 3), (500, 375, 3), (300, 300, 3), (7, 5), (9, 13, 1), (60, 40, 4), (150, 600, 3), (600, 150, 3), (320, 400, 3),
          (330, 450, 3), (200, 200, 1), (1, 1, 3), (2, 3), (480, 300, 3), (240, 384, 3), (123, 77, 3), (256, 256, 4), (333, 500, 3),
          (450, 300), (100, 700, 3)]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def images(g):
    """The golden's dataset, regenerated from its seed (make_eval_dataset_golden.make_images) and checked against its digests."""
    rng = np.random.default_rng(7)
    imgs = [rng.integers(0, 256, s, dtype=np.uint8) for s in SHAPES]
    assert [sha(im) for im in imgs] == list(g['image_sha'])
    return imgs


def decoded_per_image(g, name):
    """The rows the reference decoded per image: the stand-in's rows (inference) or decode_detections' (training)."""
    if name + '/dec_counts' in g:
        counts = g[name + '/dec_counts']
        offs = np.concatenate([[0], np.cumsum(counts)])
        return [g[name + '/dec_rows'][offs[i]:offs[i + 1]] for i in range(len(counts))]
    return list(g[name + '/y'])


def oracle_run(g, name, dtype=None):
    mode, mm, rc, (H, W), bs, seed = RUNS[name]
    shapes = [im.shape[:2] for im in images(g)]
    patches = evalops.pad_draws(shapes, H, W, seed) if mode == 'pad' else None
    rows = decoded_per_image(g, name)
    per_image = [(rows[i], shapes[i] if patches is None else patches[i][2:], (H, W), None if patches is None else patches[i][:2])
                 for i in range(len(shapes))]
    batches = [per_image[lo:lo + bs] for lo in range(0, len(per_image), bs)]
    return patches, evalops.collect(batches, dtype or (np.float32 if mm == 'inference' else np.float64), rc)


@pytest.mark.parametrize('name', [n for n in RUNS if RUNS[n][0] == 'pad'])
def test_pad_patches_equal_reference(g, name):
    patches, _ = oracle_run(g, name)
    np.testing.assert_array_equal(np.array(patches), g[name + '/patches'])


@pytest.mark.parametrize('name', [n for n in RUNS if RUNS[n][0] == 'pad'])
def test_package_pad_draws_equal_reference(g, name):
    from ssd_keras_b200.eval_utils.dataset_predict import pad_patch
    mode, mm, rc, (H, W), bs, seed = RUNS[name]
    rs = np.random.RandomState(seed)
    got = [pad_patch(im.shape[0], im.shape[1], H, W, rs) for im in images(g)]
    np.testing.assert_array_equal(np.array(got), g[name + '/patches'])


def test_wide_target_crops_some_images(g):
    """SSD7's 300x480: images with an aspect ratio between 1 and 1.6 get a positive y range and are cropped."""
    p = g['pad_inf_r3_wide/patches']
    shapes = np.array([im.shape[:2] for im in images(g)])
    assert np.any(p[:, 2] < shapes[:, 0])


@pytest.mark.parametrize('name', list(RUNS))
def test_oracle_rows_and_per_class_lists_equal_reference(g, name):
    _, (img, cls, conf, box) = oracle_run(g, name)
    ids = [int(v) for v in g['ids']]
    res = evalops.per_class(img, cls, conf, box, ids, N_CLASSES)
    flat = [(c, p) for c in range(1, N_CLASSES + 1) for p in res[c]]
    np.testing.assert_array_equal(np.array([c for c, _ in flat]), g[name + '/cls'])
    np.testing.assert_array_equal(np.array([p[0] for _, p in flat]), g[name + '/id'])
    vals = np.array([p[1:] for _, p in flat]).reshape(-1, 5)
    assert vals.dtype == g[name + '/vals'].dtype
    np.testing.assert_array_equal(vals, g[name + '/vals'])
    assert np.array_equal(np.signbit(vals), np.signbit(g[name + '/vals']))      # -0.0 stays -0.0, +0 after a pad offset
    for c in range(1, N_CLASSES + 1):
        assert evalops.txt_texts(res, N_CLASSES)[c - 1] == str(g[name + '/txt_%d' % c])


def test_float64_ratio_would_differ(g):
    """The float32 path is not the float64 path: the special rows tell them apart."""
    _, (_, _, _, b32) = oracle_run(g, 'resize_inf', np.float32)
    _, (_, _, _, b64) = oracle_run(g, 'resize_inf', np.float64)
    assert not np.array_equal(b32.astype(np.float64), b64)


@pytest.mark.parametrize('name,hw', [('coco_resize', (300, 300)), ('coco_resize_wide', (300, 480))])
def test_oracle_json_equals_reference(g, name, hw):
    counts = g[name + '/dec_counts']
    offs = np.concatenate([[0], np.cumsum(counts)])
    rows = [g[name + '/dec_rows'][offs[i]:offs[i + 1]] for i in range(len(counts))]
    shapes = [im.shape[:2] for im in images(g)]
    per_image = [(rows[i], shapes[i], hw, None) for i in range(len(shapes))]
    img, cls, conf, box = evalops.collect([per_image], np.float64)
    ids = [int(v) for v in g['ids']]
    assert evalops.json_text(img, cls, conf, box, ids, {1: 3, 2: 17, 3: 90}) == str(g[name + '/json'])
