"""NumPy restatement of uint8 ``cv2.resize`` with ``INTER_CUBIC``, ``INTER_AREA`` and ``INTER_LANCZOS4``, in the scheme of
OpenCV 4.13's own code (``modules/imgproc/src/resize.cpp``), and the op lists' ``RESIZE_INTERP`` record on top of the oracle.

  - cubic / Lanczos4 (resizeGeneric_): ``fx = float32((dx+0.5)*scale - 0.5)``, ``sx = floor(fx)``, ``fx -= sx``; the float32
    coefficients of interpolateCubic (A = -0.75, every step rounded) or interpolateLanczos4 (float64 sin / cos, normalised by
    their float32 sum) scaled by 2048 and rounded to short; 4 or 8 taps per axis from ``sx - 1`` or ``sx - 3`` on, clamped to
    the image in both axes with the fraction kept.  Horizontal pass in int.  Vertical pass: Lanczos4 ``(sum + 2^21) >> 22``;
    cubic the same in the scalar tail of a row, but the elements (column * 3 + channel) below the last whole 8-lane block go
    through VResizeCubicVec_32s8u: float32 ``S3*b3``, then ``S2*b2 + that``, ... each step rounded, rounded half to even.
  - area, downscale by integer factors (both to within DBL_EPSILON of ``1 / (out / in)``): 2 x 2 is the vector rule
    ``(a+b+c+d+2) >> 2`` (``oracle/imageops.py``); other factors ``rint(float32(sum) * float32(1 / area))``.
  - area, other downscales (resizeArea_): computeResizeAreaTab's float64 spans and float32 weights; per source row
    ``buf = sum S * alpha`` in column order, ``sum = beta0 * buf0``, ``sum += beta * buf``, float32, rounded half to even.
  - area when either axis upscales: the linear path with ``sx = floor(dx * scale)``, ``fx = float32((dx+1) - (sx+1) / scale)``,
    ``fx <= 0 ? 0 : fx - floor(fx)``, in both axes.

cv2 wheels built with Intel IPP run ``INTER_CUBIC`` through IPP by default; IPP's result differs from OpenCV's own code in the
last bit at a few pixels in 10^5 and is not the same on every CPU, so the comparisons for cubic turn IPP off
(``cv2.ipp.setUseIPP(False)``).  Area and Lanczos4 are OpenCV's own code either way."""
import math

import numpy as np

from oracle import boxops as bo
from oracle import imageops as io
from oracle import photoops as po
from oracle import warpops as wo

f32 = np.float32
OP_RESIZE_INTERP = 25
INTER_NEAREST, INTER_LINEAR, INTER_CUBIC, INTER_AREA, INTER_LANCZOS4 = range(5)
VECTOR_LANES = 8                     # int16 lanes of OpenCV's baseline (SSE) vector registers


def _short(c):
    return np.clip(np.rint(np.asarray(c, f32) * f32(2048)), -32768, 32767).astype(np.int64)


def cubic_coefs(x):
    x = np.asarray(x, f32)
    A, one = f32(-0.75), f32(1)
    x1, mx = x + one, one - x
    c0 = ((A * x1 - f32(5) * A) * x1 + f32(8) * A) * x1 - f32(4) * A
    c1 = ((A + f32(2)) * x - (A + f32(3))) * x * x + one
    c2 = ((A + f32(2)) * mx - (A + f32(3))) * mx * mx + one
    c3 = one - c0 - c1 - c2
    return np.stack([c0, c1, c2, c3], -1).astype(f32)


_S45 = 0.70710678118654752440084436210485
_CS = ((1, 0), (-_S45, -_S45), (0, 1), (_S45, -_S45), (-1, 0), (_S45, _S45), (0, -1), (-_S45, _S45))


def lanczos4_coefs(x):
    out = np.zeros(np.shape(x) + (8,), f32)
    for n, xv in enumerate(np.asarray(x, f32)):
        if xv < np.finfo(f32).eps:
            out[n, 3] = 1
            continue
        x3 = xv + f32(3)
        y0 = -float(x3) * math.pi * 0.25
        s0, c0 = math.sin(y0), math.cos(y0)
        total = f32(0)
        for i in range(8):
            y = -float(x3 - f32(i)) * math.pi * 0.25
            out[n, i] = f32((_CS[i][0] * s0 + _CS[i][1] * c0) / (y * y))
            total = f32(total + out[n, i])
        out[n] = out[n] * (f32(1) / total)
    return out


def _linear_coords(n_in, n_out):
    scale = 1.0 / (np.float64(n_out) / np.float64(n_in))
    f = ((np.arange(n_out, dtype=np.float64) + 0.5) * scale - 0.5).astype(f32)
    s = np.floor(f).astype(np.int64)
    return s, (f - s.astype(f32)).astype(f32)


def _kernel_resize(img, oh, ow, taps):
    h, w = img.shape[:2]
    coefs = cubic_coefs if taps == 4 else lanczos4_coefs
    sx, fx = _linear_coords(w, ow)
    sy, fy = _linear_coords(h, oh)
    a, b = _short(coefs(fx)), _short(coefs(fy))
    k = np.arange(taps) - taps // 2 + 1
    xt = np.clip(sx[:, None] + k[None], 0, w - 1)
    yt = np.clip(sy[:, None] + k[None], 0, h - 1)
    D = (img.astype(np.int64)[:, xt] * a[None, :, :, None]).sum(2)       # (h, ow, 3), horizontal pass
    rows = D[yt]                                                         # (oh, taps, ow, 3)
    v = ((rows * b[:, :, None, None]).sum(1) + (1 << 21)) >> 22
    if taps == 4:
        bf = (b.astype(f32) * f32(1.0 / (1 << 22))).astype(f32)
        rf = rows.astype(f32)
        t = rf[:, 3] * bf[:, 3, None, None]
        for j in (2, 1, 0):
            t = (rf[:, j] * bf[:, j, None, None]).astype(f32) + t
        vec = np.arange(ow * 3).reshape(ow, 3) < (ow * 3) // VECTOR_LANES * VECTOR_LANES
        v = np.where(vec[None], np.rint(t).astype(np.int64), v)
    return np.clip(v, 0, 255).astype(np.uint8)


def _area_table(n_in, n_out, scale):
    """computeResizeAreaTab -> (indices, float32 weights), (n_out, taps), padded with weight 0 (adding +0 changes no sum)."""
    rows = []
    for d in range(n_out):
        f1 = d * scale
        f2 = f1 + scale
        cell = min(scale, n_in - f1)
        s2 = min(math.floor(f2), n_in - 1)
        s1 = min(math.ceil(f1), s2)
        t = []
        if s1 - f1 > 1e-3:
            t.append((s1 - 1, f32((s1 - f1) / cell)))
        t += [(s, f32(1.0 / cell)) for s in range(s1, s2)]
        if f2 - s2 > 1e-3:
            t.append((s2, f32(min(min(f2 - s2, 1.0), cell) / cell)))
        rows.append(t)
    n = max(len(t) for t in rows)
    idx = np.zeros((n_out, n), np.int64)
    wt = np.zeros((n_out, n), f32)
    for d, t in enumerate(rows):
        for j, (s, a) in enumerate(t):
            idx[d, j], wt[d, j] = s, a
    return idx, wt


def _area_coords(n_in, n_out):
    inv = np.float64(n_out) / np.float64(n_in)
    s = np.floor(np.arange(n_out) * (1.0 / inv)).astype(np.int64)
    f = ((np.arange(n_out) + 1) - (s + 1) * inv).astype(f32)
    return s, np.where(f <= 0, f32(0), f - np.floor(f)).astype(f32)


def _area_resize(img, oh, ow):
    h, w = img.shape[:2]
    sx, sy = 1.0 / (np.float64(ow) / np.float64(w)), 1.0 / (np.float64(oh) / np.float64(h))
    if sx >= 1 and sy >= 1:
        ix, iy = round(sx), round(sy)
        eps = np.finfo(np.float64).eps
        if abs(sx - ix) < eps and abs(sy - iy) < eps:
            if ix == 2 and iy == 2:
                return io.resize(img, oh, ow, INTER_LINEAR)           # the same 2x2 fast path
            total = img.astype(np.int64)[:oh * iy, :ow * ix].reshape(oh, iy, ow, ix, 3).sum((1, 3))
            return np.clip(np.rint(total.astype(f32) * (f32(1) / f32(ix * iy))), 0, 255).astype(np.uint8)
        xi, xa = _area_table(w, ow, sx)
        yi, ya = _area_table(h, oh, sy)
        S = img.astype(f32)
        buf = np.zeros((h, ow, 3), f32)
        for j in range(xi.shape[1]):
            buf = buf + S[:, xi[:, j]] * xa[None, :, j, None]
        acc = ya[:, 0, None, None] * buf[yi[:, 0]]
        for j in range(1, yi.shape[1]):
            acc = acc + ya[:, j, None, None] * buf[yi[:, j]]
        return np.clip(np.rint(acc), 0, 255).astype(np.uint8)
    # an axis upscales: cv2's linear resize with area coordinates in both axes
    xs, xf = _area_coords(w, ow)
    ys, yf = _area_coords(h, oh)
    edge = xs >= w - 1
    xs, xf = np.where(edge, w - 1, xs), np.where(edge, f32(0), xf).astype(f32)
    x0, x1 = xs, np.minimum(xs + 1, w - 1)
    y0, y1 = np.clip(ys, 0, h - 1), np.clip(ys + 1, 0, h - 1)
    a0, a1 = io._coef(xf)
    b0, b1 = io._coef(yf)
    S = img.astype(np.int64)
    D = S[:, x0] * a0[None, :, None] + S[:, x1] * a1[None, :, None]
    v = (((b0[:, None, None] * (D[y0] >> 4)) >> 16) + ((b1[:, None, None] * (D[y1] >> 4)) >> 16) + 2) >> 2
    return np.clip(v, 0, 255).astype(np.uint8)


def resize(img, out_h, out_w, interpolation):
    """uint8 ``cv2.resize(img, (out_w, out_h), interpolation=...)`` of an (h, w, 3) image, any of the codes 0-4."""
    h, w = img.shape[:2]
    if (h, w) == (out_h, out_w):
        return img.copy()
    if interpolation in (INTER_NEAREST, INTER_LINEAR):
        return io.resize(img, out_h, out_w, interpolation)
    if interpolation == INTER_CUBIC:
        return _kernel_resize(img, out_h, out_w, 4)
    if interpolation == INTER_LANCZOS4:
        return _kernel_resize(img, out_h, out_w, 8)
    if interpolation == INTER_AREA:
        return _area_resize(img, out_h, out_w)
    raise ValueError('unsupported interpolation mode %r' % (interpolation,))


def apply_ops(img, ops):
    """An op list's image half with ``RESIZE_INTERP`` too: photometric prefix, the oracle's integer ops and warps, then the
    resampling step -> (h, w, 3) uint8."""
    x = po.apply_ops(img, ops)
    rest = po.split_ops(ops)[1]
    for i, o in enumerate(rest):
        if int(o[0]) == OP_RESIZE_INTERP:
            x = wo.apply_ops(x, rest[:i])
            return resize(x, int(o[4]), int(o[5]), (int(o[1]) >> 8) & 255)
    return wo.apply_ops(x, rest)


def apply_box_ops(labels, ops):
    """The box half: ``RESIZE_INTERP`` is ``RESIZE``'s arithmetic."""
    return bo.apply_box_ops(labels, [(io.OP_RESIZE,) + tuple(o[1:]) if int(o[0]) == OP_RESIZE_INTERP else o for o in ops])
