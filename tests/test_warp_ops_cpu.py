"""Translate / Scale / Rotate and BoxFilter's overlap test on the host: oracle/warpops.py and oracle/boxops.py against outputs of
the REAL reference's classes (tests/golden/make_warp_golden.py), against cv2.warpAffine itself and the live reference classes
where they are importable, the op-tuple encodings, the per-class op sequences, and the host-side validation of
ssdk_assemble_images for the new ops (it runs before the entry point touches the device)."""
import ctypes as C
import os

import numpy as np
import pytest

import __graft_entry__ as entry
from oracle import boxops as bo
from oracle import warpops as io

HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, 'golden', 'ref_warp_golden.npz'))
REF_ROOT = os.environ.get('SSD_REFERENCE_ROOT', '/root/reference')


def _ops(k):
    return [tuple(r) for r in G['ops%d' % k].tolist()]


def test_golden_images_bit_exact():
    n = int(G['n'])
    assert n >= 100
    for k in range(n):
        got = io.apply_ops(G['in%d' % k], _ops(k))
        ref = G['out%d' % k]
        assert got.shape == ref.shape, (k, got.shape, ref.shape)
        np.testing.assert_array_equal(got, ref, err_msg='case %d (%s)' % (k, G['kind%d' % k]))


def test_golden_boxes_exact():
    for k in range(int(G['n'])):
        got = bo.apply_box_ops(G['lin%d' % k], _ops(k))
        np.testing.assert_array_equal(got, G['lout%d' % k], err_msg='case %d (%s)' % (k, G['kind%d' % k]))


def test_golden_cases_cover_the_ground():
    seen = set()
    for k in range(int(G['n'])):
        img, ops, kind = G['in%d' % k], G['ops%d' % k], str(G['kind%d' % k])
        seen.add(kind)
        seen.add(('c', 1 if img.ndim == 2 else img.shape[2], img.ndim))
        h, w = img.shape[:2]
        if h == 1 or w == 1:
            seen.add('1px' if h == w else '1xN')
        if h % 2 or w % 2:
            seen.add('odd')
        if G['lin%d' % k].shape[0] > G['lout%d' % k].shape[0]:
            seen.add('dropped')
        for o in ops:
            if o[0] == io.OP_SCALE:
                seen.add('zoom ' + ('out' if o[2] < 1 else 'in' if o[2] > 1 else '1'))
            elif o[0] == io.OP_TRANSLATE and (abs(o[2]) >= h or abs(o[3]) >= w):
                seen.add('beyond')
            elif o[0] == io.OP_ROTATE:
                seen.add(('rotate', int(o[2])))
            elif o[0] == io.OP_OVERLAP:
                seen.add(('overlap', int(o[1]) & 3, (int(o[1]) >> 2) & 3))
                if o[2] == 0:
                    seen.add('lower0')
    for need in ('ssd7_seq1', 'ssd7_seq2', 'satellite', 'tie', '1px', '1xN', 'odd', 'dropped', 'zoom out', 'zoom in', 'zoom 1', 'beyond',
                 'lower0', ('rotate', 90), ('rotate', 180), ('rotate', 270), ('c', 1, 2), ('c', 1, 3), ('c', 3, 3), ('c', 4, 3)):
        assert need in seen, need
    for c in range(3):
        for b in range(3):
            assert ('overlap', c, b) in seen, (c, b)


def test_scale_corner_tie_rounds_twice():
    """np.dot(M, corners) rounds m0*x + m1*y and then + m2: the golden tie case is k + 0.5 exactly, and np.round's half-even
    result differs from what a fused f*x + m2 gives."""
    from fractions import Fraction
    h, w, f, x = G['tie'].tolist()
    M = io.rotation_matrix_2d((w / 2, h / 2), 0, f)
    two = (M[0, 0] * x + M[0, 1] * 10.0) + M[0, 2]
    assert two - np.floor(two) == 0.5
    fused = float(Fraction(M[0, 0]) * Fraction(x) + Fraction(M[0, 2]))
    assert np.round(fused) != np.round(two)
    k = [k for k in range(int(G['n'])) if str(G['kind%d' % k]) == 'tie'][0]
    assert G['lout%d' % k][0, 1] == np.round(two)
    np.testing.assert_array_equal(bo.apply_box_ops(G['lin%d' % k], _ops(k)), G['lout%d' % k])


def test_warp_matches_cv2():
    """A few hundred random Scale / Translate / Rotate cases against cv2.warpAffine and cv2.getRotationMatrix2D."""
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(31)
    for t in range(300):
        h, w = int(rng.integers(1, 100)), int(rng.integers(1, 100))
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        bg = tuple(int(v) for v in rng.integers(0, 256, 3))
        if t % 3 == 0:
            f = 1.0 if t % 21 == 0 else float(rng.uniform(0.3, 2.5))
            M = cv2.getRotationMatrix2D((w / 2, h / 2), 0, f)
            np.testing.assert_array_equal(M, io.rotation_matrix_2d((w / 2, h / 2), 0, f))
            ref = cv2.warpAffine(img, M, (w, h), borderMode=cv2.BORDER_CONSTANT, borderValue=bg)
            got = io.scale(img, f, bg)
        elif t % 3 == 1:
            dy, dx = int(rng.integers(-2 * h, 2 * h + 1)), int(rng.integers(-2 * w, 2 * w + 1))
            ref = cv2.warpAffine(img, np.float32([[1, 0, dx], [0, 1, dy]]), (w, h), borderMode=cv2.BORDER_CONSTANT, borderValue=bg)
            got = io.translate(img, dy, dx, bg)
        else:
            a = (90, 180, 270)[t % 9 // 3]
            M = cv2.getRotationMatrix2D((w / 2, h / 2), a, 1)
            np.testing.assert_array_equal(M, io.rotation_matrix_2d((w / 2, h / 2), a, 1))
            Mr, hn, wn = io.rotate_geometry(h, w, a)
            got = io.rotate(img, a)
            ref = cv2.warpAffine(img, Mr, (wn, hn))
        assert got.shape == ref.shape, t
        np.testing.assert_array_equal(got, ref, err_msg='case %d' % t)
    M = rng.uniform(-2, 2, (2, 3))
    np.testing.assert_array_equal(io.invert_affine(M), cv2.invertAffineTransform(M))


def _reference(monkeypatch):
    if not os.path.isdir(os.path.join(REF_ROOT, 'data_generator')):
        pytest.skip('reference checkout not available')
    pytest.importorskip('cv2')
    monkeypatch.setattr(np, 'float', float, raising=False)           # the reference's NumPy 1.x aliases
    monkeypatch.setattr(np, 'int', int, raising=False)
    monkeypatch.syspath_prepend(REF_ROOT)
    from data_generator import object_detection_2d_geometric_ops as geo
    from data_generator import object_detection_2d_image_boxes_validation_utils as val
    return geo, val


def test_live_reference_random(monkeypatch):
    """The op sequences of batch_assembly's per-class helpers, through the oracle, against the live reference classes."""
    geo, val = _reference(monkeypatch)
    from ssd_keras_b200.data_generator import batch_assembly as ba
    rng = np.random.default_rng(77)
    crits, bps = ('center_point', 'area', 'iou'), ('half', 'include', 'exclude')
    for t in range(150):
        h, w = int(rng.integers(1, 60)), int(rng.integers(1, 60))
        img = io.to3(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        n = int(rng.integers(0, 10))
        x0, y0 = rng.integers(-w // 3 - 1, w + 3, n), rng.integers(-h // 3 - 1, h + 3, n)
        lab = np.stack([rng.integers(1, 9, n), x0, y0, x0 + rng.integers(0, w + 1, n), y0 + rng.integers(0, h + 1, n)], 1).astype(np.float64)
        lab[:, 1:] += rng.integers(0, 2, (n, 4)) * 0.5 * (t % 2)
        kw = dict(check_overlap=bool(t % 5), check_min_area=bool(t % 3), check_degenerate=bool(t % 4), overlap_criterion=crits[t % 3],
                  overlap_bounds=((0.0, 0.7), (0.3, 1.0), (0.5, 1.0))[t % 3 - (t // 3) % 2], border_pixels=bps[(t // 3) % 3],
                  min_area=int(rng.integers(0, 20)))
        bf = val.BoxFilter(**kw)
        clipb, bg = bool(t % 7), tuple(int(v) for v in rng.integers(0, 256, 3))
        kind = t % 3
        if kind == 0:
            dy, dx = float(rng.uniform(-1.2, 1.2)), float(rng.uniform(-1.2, 1.2))
            ref_img, ref_lab = geo.Translate(dy, dx, clip_boxes=clipb, box_filter=bf, background=bg)(img, lab)
            ops = ba.translate_ops(h, w, dy, dx, box_filter=bf, clip_boxes=clipb, background=bg)
        elif kind == 1:
            f = float(rng.uniform(0.4, 2.2))
            ref_img, ref_lab = geo.Scale(f, clip_boxes=clipb, box_filter=bf, background=bg)(img, lab)
            ops = ba.scale_ops(h, w, f, box_filter=kw, clip_boxes=clipb, background=bg)
        else:
            a = (90, 180, 270)[t % 9 // 3]
            ref_img, ref_lab = geo.Rotate(a)(img, lab)
            ops = ba.rotate_ops(h, w, a)
        np.testing.assert_array_equal(io.apply_ops(img, ops), ref_img, err_msg='case %d' % t)
        np.testing.assert_array_equal(bo.apply_box_ops(lab, ops), np.asarray(ref_lab, np.float64).reshape(-1, 5), err_msg='case %d' % t)


def test_op_tuples():
    from ssd_keras_b200.data_generator import batch_assembly as ba
    assert ba.translate(100, 200, 0.125, -0.3) == (6, 0, 12.0, -60.0, 100.0, 200.0)
    assert ba.translate(10, 10, 0.25, 0.35)[2:4] == (2.0, 4.0)                     # int(round(h*dy)): half to even, as Translate
    t = ba.translate(10, 10, 0, 0, background=(123, 117, 104))
    assert io.background_of(t[1]) == (123, 117, 104) and -(1 << 31) <= t[1] < (1 << 31)
    assert ba.scale(30, 40, 1.5) == (7, 0, 1.5, 30.0, 40.0, 0.0)
    assert io.background_of(ba.scale(1, 1, 0.5, background=(255, 254, 253))[1]) == (255, 254, 253)
    assert ba.rotate(30, 40, 270) == (8, 0, 270.0, 30.0, 40.0, 0.0)
    assert ba.overlap_filter(30, 40) == (9, 0, 0.3, 1.0, 30.0, 40.0)
    assert ba.overlap_filter(30, 40, 'area', (0.0, 0.5), 'include') == (9, 1 | 4, 0.0, 0.5, 30.0, 40.0)
    assert ba.overlap_filter(30, 40, 'iou', (0.1, 0.9), 'exclude') == (9, 2 | 8, 0.1, 0.9, 30.0, 40.0)
    assert ba.clip(30, 40) == (10, 0, 30.0, 40.0, 0.0, 0.0)
    ssd7 = dict(check_overlap=True, check_min_area=True, check_degenerate=True, overlap_criterion='area', overlap_bounds=(0.3, 1.0),
                min_area=16)
    assert ba.translate_ops(300, 480, 0.1, 0.2, box_filter=ssd7, clip_boxes=True) == [
        ba.translate(300, 480, 0.1, 0.2), (5, 3, 16.0, 0.0, 0.0, 0.0), (9, 1, 0.3, 1.0, 300.0, 480.0), (10, 0, 300.0, 480.0, 0.0, 0.0)]
    assert ba.scale_ops(300, 480, 0.7, clip_boxes=False) == [ba.scale(300, 480, 0.7)]
    assert ba.box_filter_ops(dict(check_overlap=False, check_min_area=False, check_degenerate=True), 5, 5) == [(5, 1, 0.0, 0.0, 0.0, 0.0)]
    assert ba.box_filter_ops(None, 5, 5) == [] and ba.rotate_ops(3, 4, 90) == [ba.rotate(3, 4, 90)]
    assert ba.crop_pad_ops(1, 2, 10, 12, box_filter=dict(check_min_area=False, check_degenerate=False, overlap_criterion='area')) == [
        ba.crop_pad(1, 2, 10, 12, clip_boxes=False), (9, 1, 0.3, 1.0, 10.0, 12.0), (10, 0, 10.0, 12.0, 0.0, 0.0)]
    assert ba.resize_ops(10, 12, 30, 30, box_filter=dict(check_overlap=False, min_area=16)) == [
        ba.resize(10, 12, 30, 30, drop_degenerate=False), (5, 3, 16.0, 0.0, 0.0, 0.0)]
    for bad in (lambda: ba.rotate(3, 3, 45), lambda: ba.scale(3, 3, 0), lambda: ba.overlap_filter(3, 3, 'centre'),
                lambda: ba.overlap_filter(3, 3, border_pixels='all'), lambda: ba.overlap_filter(3, 3, overlap_bounds=(0.5, 0.2)),
                lambda: ba.translate(3, 3, 0, 0, background=(0, 0, 300)), lambda: ba.box_filter_ops(dict(min_areas=3), 3, 3)):
        with pytest.raises(ValueError):
            bad()


@pytest.fixture(scope='module')
def lib():
    entry.build()
    from ssd_keras_b200 import _ffi
    return _ffi.lib()


def _call(lib, shapes, ops_per_image, out_h, out_w):
    """ssdk_assemble_images with placeholder device pointers: every case here must fail in host validation."""
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.data_generator.batch_assembly import _pack_ops
    hwc = np.asarray(shapes, np.int32).reshape(-1, 3)
    offs = np.concatenate([[0], np.cumsum([int(np.prod(s)) for s in hwc])]).astype(np.int64)
    arr, max_ops = _pack_ops(ops_per_image, len(shapes))
    dummy = C.c_void_p(16)
    rc = lib.ssdk_assemble_images(dummy, dummy, _ffi.np_ptr(offs, C.c_longlong), _ffi.np_ptr(hwc, C.c_int), len(shapes), arr, max_ops,
                                  out_h, out_w, dummy, None)
    return rc, lib.ssdk_last_error().decode()


def test_host_validation_errors(lib):
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.data_generator import batch_assembly as ba
    S = [(10, 12, 3)]
    cases = [
        ([[ba.translate(10, 11, 0.1, 0.1)]], 10, 12, 'TRANSLATE of a 10x11 image, but the canvas is 10x12'),
        ([[(6, 0, 0.5, 1.0, 10.0, 12.0)]], 10, 12, 'TRANSLATE needs integer shifts'),
        ([[(6, 0, float(1 << 21), 1.0, 10.0, 12.0)]], 10, 12, 'TRANSLATE needs integer shifts'),
        ([[ba.scale(12, 10, 1.5)]], 10, 12, 'SCALE of a 12x10 image, but the canvas is 10x12'),
        ([[(7, 0, 0.0, 10.0, 12.0, 0.0)]], 10, 12, 'SCALE factor 0 is not positive'),
        ([[(7, 0, -1.0, 10.0, 12.0, 0.0)]], 10, 12, 'is not positive'),
        ([[(7, 0, 1e-7, 10.0, 12.0, 0.0)]], 10, 12, 'overflows'),
        ([[ba.rotate(12, 10, 90)]], 12, 10, 'ROTATE of a 12x10 image, but the canvas is 10x12'),
        ([[(8, 0, 45.0, 10.0, 12.0, 0.0)]], 10, 12, 'ROTATE angle 45 is not 90, 180 or 270'),
        ([[ba.scale(10, 12, 1.5), ba.scale(10, 12, 1.5)]], 10, 12, 'at most one resampling step'),
        ([[ba.scale(10, 12, 1.5), ba.resize(10, 12, 5, 5)]], 5, 5, 'at most one resampling step'),
        ([[ba.resize(10, 12, 5, 5), ba.scale(5, 5, 1.5)]], 5, 5, 'last op'),
        ([[ba.resize(10, 12, 5, 5), ba.translate(5, 5, 0.2, 0)]], 5, 5, 'last op'),
        ([[ba.resize(10, 12, 12, 10), ba.rotate(12, 10, 90)]], 10, 12, 'last op'),
        ([[ba.translate(10, 12, 0.2, 0, background=(1, 2, 3)), ba.scale(10, 12, 1.5, background=(1, 2, 4))]], 10, 12, 'background'),
        ([[ba.scale(10, 12, 0.5, background=(9, 9, 9)), ba.translate(10, 12, 0.2, 0, background=(0, 0, 0))]], 10, 12, 'background'),
        ([[ba.crop_pad(-1, 0, 12, 12, background=(5, 5, 5)), ba.rotate(12, 12, 90)]], 12, 13, 'background'),
        ([[ba.scale(10, 12, 1.5), ba.translate(10, 12, 0.3, 0.1), ba.flip(12)]], 10, 11, 'ends as 10x12'),
        ([[ba.rotate(10, 12, 90)]], 10, 12, 'ends as 12x10'),
        ([[(11, 0, 0.0, 0.0, 0.0, 0.0)]], 10, 12, 'unknown op code 11'),
    ]
    for ops, oh, ow, msg in cases:
        rc, err = _call(lib, S, ops, oh, ow)
        assert rc == _ffi.SSDK_ERR_INVALID, (ops, rc, err)
        assert msg in err, (msg, err)
    big = [(32767, 2, 1)]
    for ops, msg in (([[ba.scale(32767, 2, 1.5)]], 'SCALE of a 32767x2 canvas'), ([[ba.rotate(32767, 2, 180)]], 'ROTATE of a 32767x2 canvas')):
        rc, err = _call(lib, big, ops, 32767, 2)
        assert rc == _ffi.SSDK_ERR_INVALID and msg in err, (msg, err)
