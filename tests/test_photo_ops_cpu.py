"""oracle/photoops.py against the reference's photometric classes (tests/golden/ref_photo_golden.npz, written by
make_photo_golden.py) and, where cv2 imports, against cv2 itself: both uint8 colour conversions on all 256^3 inputs (HSV -> RGB
at a width with and a width without a scalar row tail) and whole sequences built from cv2 + NumPy directly.  Also the op
constructors of batch_assembly and the new codes of ssdk.h / _ffi.py."""
import os
import re

import numpy as np
import pytest

from oracle import photoops as po

HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, 'golden', 'ref_photo_golden.npz'))


def _cube():
    a = np.arange(256, dtype=np.uint8)
    return np.stack(np.meshgrid(a, a, a, indexing='ij'), -1).reshape(-1, 3)


def test_golden_cases_equal():
    assert int(G['n']) > 100
    for k in range(int(G['n'])):
        x = po.to_3_channels(G['in%d' % k])
        for o in G['ops%d' % k].tolist():
            x = po.apply_op(x, o)
        ref = G['out%d' % k]
        assert x.dtype == ref.dtype and np.array_equal(x, ref), k


def test_fma32_is_a_single_rounding():
    rng = np.random.default_rng(5)
    a, b, c = (rng.standard_normal(200000).astype(np.float32) for _ in range(3))
    c[::2] = -(a[::2] * b[::2])                                   # cancellation: the product's low bits decide
    from fractions import Fraction
    got = po.fma32(a, b, c)
    for i in range(0, 200000, 997):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo, hi = np.nextafter(got[i], np.float32(-np.inf)), np.nextafter(got[i], np.float32(np.inf))
        assert abs(exact - Fraction(float(got[i]))) <= min(abs(exact - Fraction(float(lo))), abs(exact - Fraction(float(hi))))


def test_division_tables_have_no_ties():
    """The kernel fills the tables with (2N + i) / (2i) in integers; that is rint(N / i) because no quotient ends in .5."""
    i = np.arange(1, 256)
    assert np.array_equal(po.SDIV[1:], (2 * (255 << 12) + i) // (2 * i))
    assert np.array_equal(po.HDIV[1:], (2 * ((180 << 12) // 6) + i) // (2 * i))


def test_rgb2hsv_equals_cv2_on_every_input():
    cv2 = pytest.importorskip('cv2')
    cube = _cube()
    for w in (4096, 1):
        img = cube.reshape(-1, w, 3)
        assert np.array_equal(po.rgb2hsv(img), cv2.cvtColor(img, cv2.COLOR_RGB2HSV)), w


def test_hsv2rgb_equals_cv2_on_every_input():
    """Width 4096: every pixel in cv2's vector loop; width 16: every pixel in its scalar loop; width 50: 32 + 18."""
    cv2 = pytest.importorskip('cv2')
    cube = _cube()
    for w in (4096, 16, 50):
        img = cube[:len(cube) // w * w].reshape(-1, w, 3)
        assert np.array_equal(po.hsv2rgb(img), cv2.cvtColor(img, cv2.COLOR_HSV2RGB)), w
    last = cube[-64:].reshape(1, 64, 3)                           # the 16 triples width 50 left out
    assert np.array_equal(po.hsv2rgb(last), cv2.cvtColor(last, cv2.COLOR_HSV2RGB))


def _cv2_sequence(cv2, img, which, p):
    """SSDPhotometricDistortions' sequences written out with cv2 + NumPy, as the reference classes compute them."""
    x = po.to_3_channels(img).astype(np.float32)
    if p['brightness'] is not None:
        x = np.clip(x + p['brightness'], 0, 255)
    if which == 1 and p['contrast'] is not None:
        x = np.clip(127.5 + p['contrast'] * (x - 127.5), 0, 255)
    x = cv2.cvtColor(np.round(x, decimals=0).astype(np.uint8), cv2.COLOR_RGB2HSV).astype(np.float32)
    if p['saturation'] is not None:
        x[:, :, 1] = np.clip(x[:, :, 1] * p['saturation'], 0, 255)
    if p['hue'] is not None:
        x[:, :, 0] = (x[:, :, 0] + p['hue']) % 180.0
    x = cv2.cvtColor(np.round(x, decimals=0).astype(np.uint8), cv2.COLOR_HSV2RGB)
    if which == 2 and p['contrast'] is not None:
        x = np.round(np.clip(127.5 + p['contrast'] * (x.astype(np.float32) - 127.5), 0, 255), decimals=0).astype(np.uint8)
    elif which == 2:
        x = np.round(x.astype(np.float32), decimals=0).astype(np.uint8)
    return x if p['channel_swap'] is None else x[:, :, list(p['channel_swap'])]


def test_random_sequences_equal_cv2():
    cv2 = pytest.importorskip('cv2')
    from ssd_keras_b200.data_generator import batch_assembly as ba
    rng = np.random.default_rng(77)
    perms = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]
    for i in range(200):
        draw = lambda lo, hi: float(rng.uniform(lo, hi)) if rng.random() < 0.6 else None      # noqa: E731
        p = dict(brightness=draw(-84, 84), contrast=draw(0.5, 1.5), saturation=draw(0.3, 2.0), hue=draw(-18, 18),
                 channel_swap=perms[int(rng.integers(6))] if rng.random() < 0.3 else None)
        c = (0, 1, 3, 4)[i % 4]
        h, w = int(rng.integers(1, 40)), int(rng.integers(1, 120))
        img = rng.integers(0, 256, (h, w) if c == 0 else (h, w, c), dtype=np.uint8)
        which = 1 + i % 2
        assert np.array_equal(po.apply_ops(img, ba.photometric_ops(which, **p)), _cv2_sequence(cv2, img, which, p)), (i, p)


def test_photometric_ops_are_the_reference_sequences():
    from ssd_keras_b200.data_generator import batch_assembly as ba
    T, U, B, C, S, H, R2H, H2R, SW = range(16, 25)
    full = dict(brightness=1.0, contrast=1.1, saturation=1.2, hue=3.0, channel_swap=(2, 1, 0))
    assert [o[0] for o in ba.photometric_ops(1, **full)] == [T, B, C, U, R2H, T, S, H, U, H2R, SW]
    assert [o[0] for o in ba.photometric_ops(2, **full)] == [T, B, U, R2H, T, S, H, U, H2R, T, C, U, SW]
    assert [o[0] for o in ba.photometric_ops(1)] == [T, U, R2H, T, U, H2R]
    assert [o[0] for o in ba.photometric_ops(2)] == [T, U, R2H, T, U, H2R, T, U]
    assert ba.photometric_ops(2, **full)[-1][2:5] == (2.0, 1.0, 0.0) and ba.photometric_ops(1, hue=-7.5)[4] == ba.hue(-7.5)
    with pytest.raises(ValueError):
        ba.photometric_ops(3)


def test_constructors_raise_what_the_reference_raises():
    from ssd_keras_b200.data_generator import batch_assembly as ba
    for bad in (lambda: ba.contrast(0.0), lambda: ba.saturation(-1.0), lambda: ba.hue(180.5), lambda: ba.hue(-181),
                lambda: ba.convert_dtype('float64'), lambda: ba.channel_swap((0, 0, 1)), lambda: ba.channel_swap((0, 1))):
        with pytest.raises(ValueError):
            bad()
    with pytest.raises(NotImplementedError):
        ba.convert_color('RGB', 'GRAY')


def test_codes_agree_between_header_ffi_and_oracle():
    from ssd_keras_b200 import _ffi
    header = open(os.path.join(HERE, '..', 'include', 'ssdk.h')).read()
    codes = {m.group(1): int(m.group(2)) for m in re.finditer(r'SSDK_BOXOP_(\w+) = (\d+)', header)}
    assert sorted(codes.values()) == list(range(11)) + list(range(16, 25))
    for name, value in codes.items():
        assert getattr(_ffi, 'BOXOP_' + name) == value, name
    for name in ('TO_FLOAT32', 'TO_UINT8', 'BRIGHTNESS', 'CONTRAST', 'SATURATION', 'HUE', 'RGB2HSV', 'HSV2RGB', 'CHANNEL_SWAP'):
        assert getattr(po, name) == codes[name], name
