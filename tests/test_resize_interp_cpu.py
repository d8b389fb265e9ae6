"""tests/resize_reference.py against the installed OpenCV 4.13 wheel: uint8 ``cv2.resize`` with INTER_CUBIC, INTER_AREA and
INTER_LANCZOS4 on a few hundred size pairs each (up and down, integer and non-integer factors, 1-pixel sides, rows whose
element count falls on both sides of the 8-lane vector blocks), and the goldens of tests/golden/make_resize_interp_golden.py."""
import os

import numpy as np
import pytest

import resize_reference as rr

cv2 = pytest.importorskip('cv2')
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_resize_interp_golden.npz')


def size_pairs(seed, n=300):
    """(h, w, oh, ow): random sizes, integer factors both ways, 1-pixel sides and widths around the vector blocks."""
    rng = np.random.default_rng(seed)
    out = []
    for t in range(n):
        kind = t % 5
        if kind == 0:
            h, w, oh, ow = (int(v) for v in rng.integers(1, 70, 4))
        elif kind == 1:                                    # integer downscale factors, 2x2 included
            oh, ow = (int(v) for v in rng.integers(1, 30, 2))
            fy, fx = (int(v) for v in rng.integers(1, 5, 2))
            h, w = oh * fy, ow * fx
        elif kind == 2:                                    # integer upscale factors
            h, w = (int(v) for v in rng.integers(1, 20, 2))
            oh, ow = h * int(rng.integers(1, 4)), w * int(rng.integers(1, 4))
        elif kind == 3:                                    # a 1-pixel side somewhere
            h, w, oh, ow = (int(v) for v in rng.integers(1, 40, 4))
            which = int(rng.integers(0, 4))
            h, w, oh, ow = [1 if i == which else v for i, v in enumerate((h, w, oh, ow))]
        else:                                              # 3 * ow around multiples of 8 (the vector body's end)
            h, w, oh = (int(v) for v in rng.integers(2, 60, 3))
            ow = 8 * int(rng.integers(1, 12)) // 3 + int(rng.integers(-1, 2))
            ow = max(ow, 1)
        if (h, w) != (oh, ow):
            out.append((h, w, oh, ow))
    return out


def _cv2(img, oh, ow, mode):
    use = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    try:
        return cv2.resize(img, (ow, oh), interpolation=mode)
    finally:
        cv2.ipp.setUseIPP(use)


@pytest.mark.parametrize('mode', [rr.INTER_CUBIC, rr.INTER_AREA, rr.INTER_LANCZOS4])
def test_reference_equals_cv2(mode):
    rng = np.random.default_rng(100 + mode)
    bad = []
    for h, w, oh, ow in size_pairs(mode):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        if not np.array_equal(rr.resize(img, oh, ow, mode), _cv2(img, oh, ow, mode)):
            bad.append((h, w, oh, ow))
    assert not bad, 'mode %d differs from cv2 on %s' % (mode, bad[:10])


@pytest.mark.parametrize('mode', [rr.INTER_AREA, rr.INTER_LANCZOS4])
def test_area_and_lanczos_do_not_depend_on_ipp(mode):
    rng = np.random.default_rng(7)
    for h, w, oh, ow in size_pairs(11, 40):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        assert np.array_equal(cv2.resize(img, (ow, oh), interpolation=mode), _cv2(img, oh, ow, mode)), (h, w, oh, ow)


def test_cubic_vector_body_and_tail_round_differently(monkeypatch):
    """The vertical pass's two roundings both matter: restating every element with either one alone misses cv2 somewhere."""
    rng = np.random.default_rng(3)
    cases = []
    for h, w, oh, ow in size_pairs(5, 120):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        cases.append((img, oh, ow, _cv2(img, oh, ow, rr.INTER_CUBIC)))
    for lanes in (1, 10 ** 9):                             # every element in the vector body / none
        monkeypatch.setattr(rr, 'VECTOR_LANES', lanes)
        assert any(not np.array_equal(rr.resize(img, oh, ow, rr.INTER_CUBIC), ref) for img, oh, ow, ref in cases), lanes


def test_goldens():
    """cv2's own outputs, recorded by make_resize_interp_golden.py, equal the restatement."""
    g = np.load(GOLDEN)
    n = int(g['n'])
    for i in range(n):
        img, mode, oh, ow = g['img%d' % i], int(g['mode%d' % i]), int(g['oh%d' % i]), int(g['ow%d' % i])
        assert np.array_equal(rr.resize(img, oh, ow, mode), g['out%d' % i]), (i, mode, img.shape, oh, ow)
