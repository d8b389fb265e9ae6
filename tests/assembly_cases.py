"""Case table of the batch-assembly tests (tests/test_gpu_assembly_paths.py) and a restatement, in Python, of the decisions
csrc/batch.cu makes for each case (tests/test_assembly_paths_cpu.py checks that together the cases reach every path).

Boxes (``ssdk_assemble_batch``): ``box_ops_kernel`` runs ``kBoxThreads`` threads per image and compacts the survivors in chunks
of that many boxes, carrying the count of the earlier chunks (``s_base``); ``box_offsets_kernel`` is one CTA of 1024 threads,
each of which scans ``per = ceil(B / 1024)`` images.  Images (``ssdk_assemble_images``): ``compose_image`` gives every image
one resampling mode (``kImgCopy`` / ``kImgNearest`` / ``kImgLinear`` / ``kImgArea2`` / ``kImgWarp``); a linear row or column
whose taps fall outside the canvas is clamped; a warp's source coordinate saturates to int16; a batch with a SCALE runs the
``image_assemble_kernel<true>`` instantiation.  The photometric prefix runs on a grid of ``gx`` CTA columns; cv2's HSV -> RGB
rounds in the columns ``>= w & ~31`` (the tail) and truncates in the others.

Every case is plain data plus a seeded generator, so the GPU test and the CPU model see the same inputs."""
import math
import os
import re

import numpy as np

from oracle import warpops as wo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BATCH_CU = os.path.join(ROOT, 'ssd_keras_b200', 'csrc', 'batch.cu')
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'ref_assembly_edges_golden.npz')

CROP_PAD, FLIP_H, FLIP_V, RESIZE, FILTER, TRANSLATE, SCALE, ROTATE, OVERLAP, CLIP = range(1, 11)
PHOTO = range(16, 25)


def kernel_constants():
    """The constants, mode rules and launch shapes of csrc/batch.cu, read from the source so that this model cannot drift."""
    with open(BATCH_CU) as f:
        src = f.read()
    k = {n: int(v) for n, v in re.findall(r'constexpr int (k\w+) = (\d+);', src)}
    for n in ('kBoxThreads', 'kImgThreads', 'kPhotoThreads', 'kPhotoGroupsPerThread', 'kPhotoMaxStages'):
        assert n in k, n
    m = re.search(r'enum \{ (kImg\w+ = \d+(?:, kImg\w+ = \d+)*) \};', src)
    assert m, 'the kImg* mode enum'
    k['modes'] = {n: int(v) for n, v in re.findall(r'(kImg\w+) = (\d+)', m.group(1))}
    assert set(k['modes']) == {'kImgCopy', 'kImgNearest', 'kImgLinear', 'kImgArea2', 'kImgWarp'}, k['modes']
    for rule in ('if (resized && rh == ch && rw == cw) mode = kImgCopy;',
                 'else if (mode == kImgLinear && ch == 2 * rh && cw == 2 * rw) mode = kImgArea2;',
                 'mode = interp == 0 ? kImgNearest : kImgLinear;',
                 'warped = true; mode = kImgWarp;',
                 'const bool warp = std::any_of(descs.begin(), descs.end(), [](const ImgDesc& d) { return d.mode == kImgWarp; });',
                 'launch(ctx, warp ? image_assemble_kernel<true> : image_assemble_kernel<false>, dim3(out_h, B), kImgThreads, 0, stream,',
                 'launch(ctx, box_ops_kernel, B, kBoxThreads, 0, stream,',
                 'launch(ctx, box_offsets_kernel, 1, 1024, 0, stream,',
                 'launch(ctx, box_pack_kernel, B, kBoxThreads, 0, stream,',
                 'const int per = (B + 1023) / 1024;',
                 'for (int base = 0; base < G; base += kBoxThreads) {',
                 'const int gx = std::max(1, std::min(ceil_div(photo_groups, kPhotoThreads * kPhotoGroupsPerThread), 65535));',
                 'launch(ctx, photometric_kernel, dim3(gx, (unsigned)photo.size()), kPhotoThreads, 0, stream,',
                 'const int tail_from = w & ~31;',
                 'SSDK_REQUIRE(B > 0 && B <= 65535,',
                 'const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767)',
                 'if (s >= d.cw - 1) { s = d.cw - 1; f = 0.f; }',
                 'r0 = min(max(s, 0), d.ch - 1); r1 = min(max(s + 1, 0), d.ch - 1);',
                 'if (!(worst < (double)(1 << 30))) return false;'):
        assert rule in src, rule
    return k


K = kernel_constants()
BOX_THREADS, IMG_THREADS, PHOTO_THREADS = K['kBoxThreads'], K['kImgThreads'], K['kPhotoThreads']
PHOTO_GROUPS, PHOTO_MAX_STAGES, MODES = K['kPhotoGroupsPerThread'], K['kPhotoMaxStages'], K['modes']
MODE_NAMES = {v: n for n, v in MODES.items()}
MAX_B = 65535


def assert_f32_bits(got, ref64, msg=''):
    """Device float32 rows equal to the float64 reference rows cast to float32, bit for bit (so -0.0 differs from +0.0); any NaN
    equals any NaN (a device NaN is 0x7fffffff, a NumPy one 0x7fc00000)."""
    got = np.ascontiguousarray(np.asarray(got, np.float32))
    ref = np.ascontiguousarray(np.asarray(ref64, np.float64).astype(np.float32))
    assert got.shape == ref.shape, (msg, got.shape, ref.shape)
    gn, rn = np.isnan(got), np.isnan(ref)
    bad = (gn != rn) | (~gn & ~rn & (got.view(np.uint32) != ref.view(np.uint32)))
    assert not bad.any(), (msg, np.argwhere(bad)[:5].tolist(), got[bad.any(-1)][:3].tolist(), ref[bad.any(-1)][:3].tolist())


# ------------------------------------------------------------------------------------------------
# boxes
# ------------------------------------------------------------------------------------------------
def box_plan(G, keep):
    """One image of G boxes, of which the indices in ``keep`` survive -> (chunks, warps that hold a box, warps that hold a
    survivor, whether a later chunk starts from a non-zero carry)."""
    chunks = -(-G // BOX_THREADS)
    warps = {(g % BOX_THREADS) // 32 for g in range(G)}
    kept = sorted(keep)
    kwarps = {(g % BOX_THREADS) // 32 for g in kept}
    carry = any(g >= BOX_THREADS for g in kept) and any(g < BOX_THREADS for g in kept)
    return dict(chunks=chunks, warps=warps, kept_warps=kwarps, carry=carry)


def offsets_per(B):
    return -(-B // 1024)


G_COUNTS = (0, 1, 31, 32, 33, 127, 128, 129, 300, 1000)
BATCH_SIZES = (1, 1023, 1024, 1025, 3000)


def scattered_labels(rng, G, h=60, w=80):
    """G boxes of which about half have their centre inside an h x w patch at (10, 10): CROP_PAD's filter drops the rest."""
    cy = rng.uniform(-h / 2, 1.5 * h, G) + 10
    cx = rng.uniform(-w / 2, 1.5 * w, G) + 10
    bh, bw = rng.uniform(1, 20, G), rng.uniform(1, 20, G)
    lab = np.stack([rng.integers(1, 9, G), cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1).astype(np.float64)
    return np.round(lab * 4) / 4


def scattered_ops(h=60, w=80):
    return [(CROP_PAD, 1 | 2, 10.0, 10.0, float(h), float(w)), (RESIZE, 1 | (1 << 8), float(h), float(w), 90.0, 70.0)]


# ------------------------------------------------------------------------------------------------
# images
# ------------------------------------------------------------------------------------------------
def _f32(x):
    return float(np.float32(x))


def _linear_s(n_out, scale):
    """cv2's INTER_LINEAR source index of every output index: floor((float)((d + 0.5) * scale - 0.5))."""
    return [math.floor(_f32((d + 0.5) * scale - 0.5)) for d in range(n_out)]


def _fixed_point_fits(m, nh, nw):
    for r in (m[0:3], m[3:6]):
        worst = 0.0
        for y in (0, nh - 1):
            for x in (0, nw - 1):
                worst = max(worst, abs((r[1] * y + r[2]) * 1024.0) + abs(r[0] * x * 1024.0))
        if not worst < float(1 << 30):
            return False
    return True


def scale_inverse(h, w, f):
    return wo.invert_affine(wo.rotation_matrix_2d((w / 2, h / 2), 0, f)).reshape(-1)


def scale_accepted(h, w, f):
    """compose_image's refusal of a SCALE whose fixed-point coordinates overflow int32."""
    return _fixed_point_fits(scale_inverse(h, w, f), h, w)


def _saturates(m, nh, nw):
    y, x = np.arange(nh, dtype=np.float64)[:, None], np.arange(nw, dtype=np.float64)[None, :]
    X0 = np.rint((m[1] * y + m[2]) * 1024.0).astype(np.int64) + 16
    Y0 = np.rint((m[4] * y + m[5]) * 1024.0).astype(np.int64) + 16
    X = (X0 + np.rint(m[0] * x * 1024.0).astype(np.int64)) >> 5
    Y = (Y0 + np.rint(m[3] * x * 1024.0).astype(np.int64)) >> 5
    return bool(((X >> 5) < -32768).any() or ((X >> 5) > 32767).any() or ((Y >> 5) < -32768).any() or ((Y >> 5) > 32767).any())


def image_plan(shape, ops, out_h, out_w):
    """compose_image's decisions for one image: mode, whether a linear row / column tap is clamped or a nearest column is
    capped, whether the warp saturates its int16 source coordinate."""
    ch, cw = shape[0], shape[1]
    mode, rh, rw, warp = 'kImgCopy', None, None, None
    for o in ops:
        op = int(o[0])
        if op == 0:
            break
        if op in (FILTER, OVERLAP, CLIP) or op in PHOTO:
            continue
        if warp is not None:                       # integer ops after the SCALE map its output
            continue
        if op == CROP_PAD:
            ch, cw = int(o[4]), int(o[5])
        elif op == ROTATE and o[2] in (90.0, 270.0):
            ch, cw = cw, ch
        elif op == RESIZE:
            rh, rw = int(o[4]), int(o[5])
            mode = 'kImgNearest' if ((int(o[1]) >> 8) & 255) == 0 else 'kImgLinear'
        elif op == SCALE:
            mode, warp = 'kImgWarp', (ch, cw, float(o[2]))
    plan = dict(mode=mode, row_clamp=False, col_clamp=False, saturates=False, canvas=(ch, cw))
    if rh is not None and rh == ch and rw == cw:
        plan['mode'] = 'kImgCopy'
    elif mode == 'kImgLinear' and ch == 2 * rh and cw == 2 * rw:
        plan['mode'] = 'kImgArea2'
    if plan['mode'] == 'kImgLinear':
        sy, sx = _linear_s(rh, 1.0 / (rh / ch)), _linear_s(rw, 1.0 / (rw / cw))
        plan['row_clamp'] = any(s < 0 or s + 1 > ch - 1 for s in sy)
        plan['col_clamp'] = any(s < 0 or s >= cw - 1 for s in sx)
    elif plan['mode'] == 'kImgNearest':
        plan['col_clamp'] = any(math.floor(d * (1.0 / (rw / cw))) > cw - 1 for d in range(rw))
        plan['row_clamp'] = any(math.floor(d * (1.0 / (rh / ch))) > ch - 1 for d in range(rh))
    elif plan['mode'] == 'kImgWarp':
        h, w, f = warp
        plan['saturates'] = _saturates(scale_inverse(h, w, f), h, w)
    return plan


def instantiation(plans):
    return 'image_assemble_kernel<true>' if any(p['mode'] == 'kImgWarp' for p in plans) else 'image_assemble_kernel<false>'


def photo_grid(shapes):
    """The photometric launch for images of these (h, w) shapes -> (gx, per image: the number of tail columns)."""
    groups = max(-(-(h * w) // 4) for h, w in shapes)
    gx = max(1, min(-(-groups // (PHOTO_THREADS * PHOTO_GROUPS)), 65535))
    return gx, [w - (w & ~31) for h, w in shapes]


def _resize(ih, iw, oh, ow, mode):
    return (RESIZE, (mode << 8), float(ih), float(iw), float(oh), float(ow))


def image_edge_cases():
    """(name, (h, w, c), ops, out_h, out_w): every resampling mode at its edges."""
    cases = []
    for mode in (0, 1):
        m = 'near' if mode == 0 else 'lin'
        cases += [('1x1->300x300 ' + m, (1, 1, 3), [_resize(1, 1, 300, 300, mode)], 300, 300),
                  ('1x7->5x300 ' + m, (1, 7, 1), [_resize(1, 7, 5, 300, mode)], 5, 300),
                  ('7x1->300x5 ' + m, (7, 1, 4), [_resize(7, 1, 300, 5, mode)], 300, 5),
                  ('1000->3 ' + m, (1000, 1000, 3), [_resize(1000, 1000, 3, 3, mode)], 3, 3),
                  ('1x1->1x1 via pad ' + m, (1, 1, 3), [(CROP_PAD, 0, 0.0, 0.0, 1.0, 2.0), _resize(1, 2, 1, 1, mode)], 1, 1),
                  ('2x on rows only ' + m, (40, 60, 3), [_resize(40, 60, 20, 60, mode)], 20, 60),
                  ('2x on columns only ' + m, (40, 60, 3), [_resize(40, 60, 40, 30, mode)], 40, 30),
                  ('2x both ' + m, (40, 60, 3), [_resize(40, 60, 20, 30, mode)], 20, 30),
                  ('2x both after a pad ' + m, (37, 55, 1), [(CROP_PAD, 0, -3.0, -5.0, 40.0, 60.0), _resize(40, 60, 20, 30, mode)], 20, 30),
                  ('identity after crops ' + m, (50, 70, 3), [(CROP_PAD, 0, 5.0, 6.0, 40.0, 60.0), (FLIP_H, 0, 60.0, 0, 0, 0),
                                                             _resize(40, 60, 40, 60, mode)], 40, 60)]
        for (a, b) in ((7, 3), (3, 7), (299, 300), (300, 299)):
            cases.append(('%d->%d %s' % (a, b, m), (a, a + 1, 3), [_resize(a, a + 1, b, b + 1, mode)], b, b + 1))
    for ow in (1, 127, 128, 129, 300, 1000):
        cases.append(('out_w %d' % ow, (9, 61, 3), [_resize(9, 61, 3, ow, 1)], 3, ow))
    cases.append(('out_h 2000', (50, 3, 3), [_resize(50, 3, 2000, 5, 1)], 2000, 5))
    cases.append(('crops only', (20, 30, 3), [(CROP_PAD, 0, -2.0, 3.0, 25.0, 17.0), (FLIP_V, 0, 25.0, 0, 0, 0)], 25, 17))
    return cases


def scale_bound(h, w):
    """The smallest factor compose_image accepts for an h x w SCALE, to float64 resolution (bisection on scale_accepted)."""
    lo, hi = 1e-9, 1.0
    assert not scale_accepted(h, w, lo) and scale_accepted(h, w, hi)
    for _ in range(200):
        mid = (lo + hi) / 2
        if mid in (lo, hi):
            break
        if scale_accepted(h, w, mid):
            hi = mid
        else:
            lo = mid
    return lo, hi


def warp_cases():
    """(name, (h, w, c), factor): zoom 8x, ordinary zooms and factors just above the refusal, which saturate the int16 source
    coordinate."""
    lo, hi = scale_bound(100, 120)
    return [('zoom 8x', (40, 50, 3), 8.0), ('zoom 0.5', (40, 50, 3), 0.5), ('zoom 1.3', (33, 17, 1), 1.3),
            ('tiny factor', (100, 120, 3), hi), ('tiny factor x1.5', (100, 120, 3), hi * 1.5), ('factor 1e-3', (100, 120, 4), 1e-3)], (lo, hi)


PHOTO_WIDTHS = (1, 31, 32, 33)
