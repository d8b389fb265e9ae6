"""The image half of the geometric ops on the host: oracle/imageops.py against outputs of the REAL reference's
ConvertTo3Channels / CropPad / Flip / Resize / SSDExpand (tests/golden/make_image_ops_golden.py), a seeded fuzz against cv2
itself where cv2 is importable, the op-tuple encoding of the new flag bits, and the host-side validation of
ssdk_assemble_images (it runs before the entry point touches the device)."""
import ctypes as C
import os

import numpy as np
import pytest

import __graft_entry__ as entry
from oracle import imageops as io

HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, 'golden', 'ref_image_ops_golden.npz'))


def test_golden_cases_bit_exact():
    n = int(G['n'])
    assert n >= 60
    for k in range(n):
        got = io.apply_ops(G['in%d' % k], G['ops%d' % k].tolist())
        ref = G['out%d' % k]
        assert got.shape == ref.shape, (k, got.shape, ref.shape)
        np.testing.assert_array_equal(got, ref, err_msg='case %d' % k)


def test_golden_cases_cover_the_ground():
    """Every path the goldens are meant to cover is present: both modes, up / down / 2x / identity / one axis, 1-pixel inputs,
    every channel layout, pads and crops on every side, flips, mean-colour expansion."""
    seen = set()
    for k in range(int(G['n'])):
        img, ops = G['in%d' % k], G['ops%d' % k]
        seen.add(('c', 1 if img.ndim == 2 else img.shape[2], img.ndim))
        h, w = img.shape[:2]
        if h == 1 or w == 1:
            seen.add('1px')
        for o in ops:
            if o[0] == io.OP_RESIZE:
                ih, iw, oh, ow = (int(v) for v in o[2:])
                mode = io.interpolation_of(o[1])
                seen.add(('mode', mode))
                if (ih, iw) == (oh, ow):
                    seen.add('identity')
                elif ih == 2 * oh and iw == 2 * ow:
                    seen.add('2x')
                elif ih == oh or iw == ow:
                    seen.add('one-axis')
                elif oh > ih and ow > iw:
                    seen.add('up')
                elif oh < ih and ow < iw:
                    seen.add('down')
            elif o[0] == io.OP_CROP_PAD:
                py, px, ph, pw = (int(v) for v in o[2:])
                if py < 0 and px < 0 and py + ph > h and px + pw > w:
                    seen.add('pad-all')
                if py > 0 and px > 0 and py + ph < h and px + pw < w:
                    seen.add('crop-all')
                if io.background_of(o[1]) == (123, 117, 104):
                    seen.add('mean')
            elif o[0] in (io.OP_FLIP_H, io.OP_FLIP_V):
                seen.add(('flip', int(o[0])))
    for need in ('1px', 'identity', '2x', 'one-axis', 'up', 'down', 'pad-all', 'crop-all', 'mean', ('mode', 0), ('mode', 1),
                 ('c', 1, 2), ('c', 1, 3), ('c', 3, 3), ('c', 4, 3), ('flip', io.OP_FLIP_H), ('flip', io.OP_FLIP_V)):
        assert need in seen, need


def _random_chain(rng):
    """A random op list in the encoding of batch_assembly: optional mean-colour expand, optional crop / pad, flips, a resize."""
    h, w = int(rng.integers(1, 90)), int(rng.integers(1, 90))
    c = int(rng.choice([0, 1, 3, 4]))
    img = rng.integers(0, 256, (h, w) if c == 0 else (h, w, c), dtype=np.uint8)
    ops, ch, cw = [], h, w
    bg = (int(rng.integers(256)), int(rng.integers(256)), int(rng.integers(256)))
    flags = (2 | (bg[0] << 8) | (bg[1] << 16) | (bg[2] << 24))
    flags = flags - (1 << 32) if flags >= 1 << 31 else flags
    if rng.random() < 0.5:
        ph, pw = int(ch * rng.uniform(1, 3)), int(cw * rng.uniform(1, 3))
        ops.append((io.OP_CROP_PAD, flags, -int(rng.integers(0, ph - ch + 1)), -int(rng.integers(0, pw - cw + 1)), ph, pw))
        ch, cw = ph, pw
    if rng.random() < 0.6:
        ph, pw = int(rng.integers(1, ch + 20)), int(rng.integers(1, cw + 20))
        ops.append((io.OP_CROP_PAD, flags, int(rng.integers(-10, ch + 1)), int(rng.integers(-10, cw + 1)), ph, pw))
        ch, cw = ph, pw
    if rng.random() < 0.5:
        ops.append((io.OP_FLIP_H, 0, cw, 0, 0, 0))
    if rng.random() < 0.3:
        ops.append((io.OP_FLIP_V, 0, ch, 0, 0, 0))
    r = rng.random()
    oh, ow = (ch // 2, cw // 2) if r < 0.15 and ch > 1 and cw > 1 else (int(rng.integers(1, 120)), int(rng.integers(1, 120)))
    if r > 0.9:
        oh = ch
    ops.append((io.OP_RESIZE, 1 | (int(rng.integers(0, 2)) << 8), ch, cw, oh, ow))
    return img, ops


def test_fuzz_against_cv2():
    """About 200 seeded chains: the oracle's whole-chain result against the same chain with cv2.resize doing the resize."""
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(99)
    for t in range(200):
        img, ops = _random_chain(rng)
        x = io.to3(img)
        for o in ops:
            if o[0] == io.OP_CROP_PAD:
                x = io.crop_pad(x, o[2], o[3], o[4], o[5], io.background_of(o[1]))
            elif o[0] == io.OP_FLIP_H:
                x = x[:, ::-1]
            elif o[0] == io.OP_FLIP_V:
                x = x[::-1]
            else:
                x = cv2.resize(np.ascontiguousarray(x), (o[5], o[4]), interpolation=io.interpolation_of(o[1]))
        np.testing.assert_array_equal(io.apply_ops(img, ops), x, err_msg='chain %d: %r' % (t, ops))


def test_resize_matches_cv2_on_size_pairs():
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(7)
    for t in range(120):
        h, w, oh, ow = (int(v) for v in rng.integers(1, 200, 4))
        if t % 6 == 0:
            oh = h
        if t % 6 == 1:
            h, w = 2 * oh, 2 * ow
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        for mode in (0, 1):
            np.testing.assert_array_equal(io.resize(img, oh, ow, mode), cv2.resize(img, (ow, oh), interpolation=mode),
                                          err_msg='%dx%d -> %dx%d mode %d' % (h, w, oh, ow, mode))


def test_op_tuples_keep_their_box_fields():
    from ssd_keras_b200.data_generator import batch_assembly as ba
    assert ba.crop_pad(-3, -4, 10, 12) == (1, 2, -3.0, -4.0, 10.0, 12.0)
    assert ba.crop_pad(1, 2, 3, 4, center_point_filter=True, clip_boxes=False) == (1, 1, 1.0, 2.0, 3.0, 4.0)
    t = ba.crop_pad(-3, -4, 10, 12, background=(123, 117, 104))
    assert t[0] == 1 and t[2:] == (-3.0, -4.0, 10.0, 12.0) and t[1] & 3 == 2
    assert io.background_of(t[1]) == (123, 117, 104) and -(1 << 31) <= t[1] < (1 << 31)
    assert io.background_of(ba.crop_pad(0, 0, 1, 1, background=(255, 255, 255))[1]) == (255, 255, 255)
    assert ba.resize(100, 200, 300, 300) == (4, 1 | (1 << 8), 100.0, 200.0, 300.0, 300.0)             # Resize's INTER_LINEAR
    assert ba.resize(100, 200, 300, 300, drop_degenerate=False, interpolation_mode=0) == (4, 0, 100.0, 200.0, 300.0, 300.0)
    assert io.interpolation_of(ba.resize(1, 1, 1, 1, interpolation_mode=3)[1]) == 3
    assert ba.flip(77) == (2, 0, 77.0, 0.0, 0.0, 0.0) and ba.flip(5, 'vertical') == (3, 0, 5.0, 0.0, 0.0, 0.0)
    assert ba.box_filter(min_area=4) == (5, 3, 4.0, 0.0, 0.0, 0.0)
    with pytest.raises(ValueError):
        ba.crop_pad(0, 0, 1, 1, background=(0, 0, 256))
    with pytest.raises(ValueError):
        ba.resize(1, 1, 1, 1, interpolation_mode=-1)


@pytest.fixture(scope='module')
def lib():
    entry.build()
    from ssd_keras_b200 import _ffi
    return _ffi.lib()


def _call(lib, shapes, ops_per_image, out_h, out_w, B=None):
    """ssdk_assemble_images with placeholder device pointers: every case here must fail in host validation."""
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.data_generator.batch_assembly import _pack_ops
    B = len(shapes) if B is None else B
    hwc = np.asarray(shapes, np.int32).reshape(-1, 3)
    offs = np.concatenate([[0], np.cumsum([int(np.prod(s)) for s in hwc])]).astype(np.int64)
    arr, max_ops = _pack_ops(ops_per_image, len(shapes))
    dummy = C.c_void_p(16)
    rc = lib.ssdk_assemble_images(dummy, dummy, _ffi.np_ptr(offs, C.c_longlong), _ffi.np_ptr(hwc, C.c_int), B, arr, max_ops,
                                  out_h, out_w, dummy, None)
    return rc, lib.ssdk_last_error().decode()


def test_host_validation_errors(lib):
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.data_generator import batch_assembly as ba
    cases = [
        ([(10, 10, 2)], [[ba.resize(10, 10, 5, 5)]], 5, 5, 'channels'),
        ([(0, 10, 3)], [[]], 5, 5, 'size'),
        ([(10, 10, 3)], [[ba.crop_pad(11, 0, 5, 5)]], 5, 5, "The given patch doesn't overlap with the input image."),
        ([(10, 10, 3)], [[ba.crop_pad(0, 11, 5, 5)]], 5, 5, "The given patch doesn't overlap with the input image."),
        ([(10, 10, 3)], [[ba.crop_pad(0.5, 0, 5, 5)]], 5, 5, 'integer patch'),
        ([(10, 10, 3)], [[ba.resize(10, 12, 5, 5)]], 5, 5, 'canvas'),
        ([(10, 10, 3)], [[ba.crop_pad(0, 0, 8, 8), ba.resize(10, 10, 5, 5)]], 5, 5, 'canvas'),
        ([(10, 10, 3)], [[ba.resize(10, 10, 5, 5), ba.resize(5, 5, 5, 5)]], 5, 5, 'last op'),
        ([(10, 10, 3)], [[ba.resize(10, 10, 5, 5), ba.flip(5)]], 5, 5, 'last op'),
        ([(10, 10, 3)], [[ba.resize(10, 10, 5, 5), ba.crop_pad(0, 0, 5, 5)]], 5, 5, 'last op'),
        ([(10, 10, 3)], [[ba.resize(10, 10, 5, 5)]], 5, 6, 'output'),
        ([(10, 10, 3)], [[]], 5, 5, 'output'),
        ([(10, 10, 3)], [[ba.resize(10, 10, 5, 5, interpolation_mode=2)]], 5, 5, 'interpolation mode 2'),
        ([(10, 10, 3)], [[ba.resize(10, 10, 5, 5, interpolation_mode=3)]], 5, 5, 'interpolation mode 3'),
        ([(10, 10, 3)], [[ba.flip(9)]], 10, 10, 'FLIP_H'),
        ([(10, 10, 3)], [[ba.flip(10, 'vertical'), ba.flip(11, 'vertical')]], 10, 10, 'FLIP_V'),
        ([(10, 10, 3)], [[ba.crop_pad(-2, -2, 14, 14, background=(1, 2, 3)), ba.crop_pad(-1, -1, 16, 16, background=(1, 2, 4))]], 16, 16,
         'background'),
        ([(10, 10, 3), (10, 10, 1)], [[ba.resize(10, 10, 5, 5)], [ba.resize(10, 10, 4, 5)]], 5, 5, 'image 1'),
    ]
    for shapes, ops, oh, ow, msg in cases:
        rc, err = _call(lib, shapes, ops, oh, ow)
        assert rc == _ffi.SSDK_ERR_INVALID, (shapes, ops, rc, err)
        assert msg in err, (msg, err)
    rc, err = _call(lib, [(10, 10, 3)], [[]], 10, 10, B=0)
    assert rc == _ffi.SSDK_ERR_INVALID
