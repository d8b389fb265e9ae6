"""Every path of the batch assembly on the device against the oracle (oracle/boxops.py, oracle/warpops.py, oracle/photoops.py),
with the cases of tests/assembly_cases.py.  Boxes are compared as float32 bit patterns, any NaN equal to any NaN (a device NaN is
0x7fffffff, a NumPy one 0x7fc00000), so -0.0 and +0.0 differ; offsets and stats exactly; images with torch.equal.

Boxes: the reference's own outputs on the edge golden (NaN through the clips, -0.0 after Resize, +0 after Scale / Rotate); box
counts across every warp and chunk of box_ops_kernel; batch sizes on both sides of box_offsets_kernel's 1024 threads; the raw
entry point (no boxes, no stats, float32 input, lists without END, skipped codes, a growing and shrinking workspace, rows past
the output left alone); the encoder fed from the device.  Images: every resampling mode at its edges, warps that saturate cv2's
int16 coordinate and the refusal next to them, both kernel instantiations, the grid limit, the photometric prefix at odd widths
and byte offsets, a source past 2^31 bytes, and ten calls in flight."""
import ctypes as C

import numpy as np
import pytest

import assembly_cases as ac
from oracle import boxops as bo
from oracle import photoops as po
from oracle import warpops as wo

pytestmark = pytest.mark.gpu
G = np.load(ac.GOLDEN)


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()


@pytest.fixture(scope='module')
def ba():
    from ssd_keras_b200.data_generator import batch_assembly
    return batch_assembly


assert_f32_bits = ac.assert_f32_bits


def _check_batch(labels, ops, f64=True):
    """assemble_batch_device against the oracle, image by image, plus offsets and stats."""
    from ssd_keras_b200.data_generator.batch_assembly import assemble_batch_device
    gt, offs, stats, _, _ = assemble_batch_device(labels, ops)
    gt, offs, stats = gt.cpu().numpy(), offs.cpu().numpy(), stats.cpu().numpy()
    refs = [bo.apply_box_ops(l, o) for l, o in zip(labels, ops)]
    counts = [r.shape[0] for r in refs]
    np.testing.assert_array_equal(offs, np.cumsum([0] + counts))
    assert stats.tolist() == [sum(counts), max(counts + [0])]
    assert_f32_bits(gt[:offs[-1]], np.concatenate(refs) if refs else np.zeros((0, 5)))
    return refs


# ------------------------------------------------------------------------------------------------
# boxes
# ------------------------------------------------------------------------------------------------
def test_edge_golden_on_device():
    """The reference's outputs on every edge case, in one batch: NaN through CROP_PAD's clip and CLIP, -0.0 after Resize,
    +0 after Scale / Rotate, bounds met with equality, empty and fully dropped images."""
    from ssd_keras_b200.data_generator.batch_assembly import assemble_batch_device
    n = int(G['n'])
    labels = [G['lin%d' % k] for k in range(n)]
    ops = [[(int(r[0]), int(r[1]), *r[2:]) for r in G['ops%d' % k].tolist()] for k in range(n)]
    gt, offs, stats, _, _ = assemble_batch_device(labels, ops)
    gt, offs, stats = gt.cpu().numpy(), offs.cpu().numpy(), stats.cpu().numpy()
    counts = [G['lout%d' % k].shape[0] for k in range(n)]
    np.testing.assert_array_equal(offs, np.cumsum([0] + counts))
    assert stats.tolist() == [sum(counts), max(counts)]
    for k in range(n):
        assert_f32_bits(gt[offs[k]:offs[k + 1]], G['lout%d' % k], 'case %d (%s)' % (k, G['kind%d' % k]))


def test_box_counts_across_warps_and_chunks():
    """G in {0, 1, 31, ..., 1000} per image in one batch, survivors scattered over every warp and chunk."""
    rng = np.random.default_rng(11)
    order = list(ac.G_COUNTS) + list(ac.G_COUNTS[::-1])
    labels = [ac.scattered_labels(rng, g) for g in order]
    ops = [ac.scattered_ops() for _ in order]
    refs = _check_batch(labels, ops)
    for g, lab, ref in zip(order, labels, refs):
        kept = [i for i in range(g) if bo.apply_box_ops(lab[i:i + 1], ac.scattered_ops()).shape[0]]
        assert len(kept) == ref.shape[0]
        p = ac.box_plan(g, kept)
        if g >= 300:
            assert p['carry'] and p['kept_warps'] == {0, 1, 2, 3}, g


def _random_chain(rng, ba, h, w):
    ops = []
    if rng.random() < 0.5:
        ops.append(ba.flip(w))
    if rng.random() < 0.4:
        ops += ba.translate_ops(h, w, float(rng.uniform(-0.3, 0.3)), float(rng.uniform(-0.3, 0.3)),
                                box_filter=dict(overlap_criterion=('center_point', 'area', 'iou')[int(rng.integers(3))]))
    elif rng.random() < 0.5:
        ops += ba.scale_ops(h, w, float(rng.uniform(0.5, 2.0)), box_filter=dict(check_overlap=False, min_area=4))
    ph, pw = int(rng.integers(h // 2, h + 1)), int(rng.integers(w // 2, w + 1))
    ops.append(ba.crop_pad(int(rng.integers(0, h - ph + 1)), int(rng.integers(0, w - pw + 1)), ph, pw, center_point_filter=bool(rng.random() < 0.5)))
    ops.append(ba.resize(ph, pw, 300, 300))
    return ops


@pytest.mark.parametrize('B', ac.BATCH_SIZES)
def test_batch_sizes(ba, B):
    """box_offsets_kernel with per = 1, 2 and 3 images per thread."""
    rng = np.random.default_rng(B)
    h, w = 60, 80
    labels = []
    for b in range(B):
        n = int(rng.integers(0, 7))
        x0, y0 = rng.uniform(-10, w, n), rng.uniform(-10, h, n)
        labels.append(np.stack([rng.integers(1, 21, n), x0, y0, x0 + rng.uniform(0, 40, n), y0 + rng.uniform(0, 40, n)], 1).reshape(-1, 5))
    ops = [_random_chain(rng, ba, h, w) for _ in range(B)]
    assert ac.offsets_per(B) == -(-B // 1024)
    _check_batch(labels, ops)


def _pack(ops_lists, B, max_ops=None):
    import torch
    from ssd_keras_b200 import _ffi
    max_ops = max_ops or max([len(o) for o in ops_lists] + [1])
    arr = (_ffi.BoxOp * (B * max_ops))()
    for b, lst in enumerate(ops_lists):
        for i, o in enumerate(lst):
            e = arr[b * max_ops + i]
            e.op, e.flags, e.a0, e.a1, e.a2, e.a3 = o
    return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).cuda(), max_ops


def _raw(gt_in, f64, counts, ops_lists, gt_out, stats=True, max_ops=None):
    """ssdk_assemble_batch called directly -> (offsets, stats or None) on the host."""
    import torch
    from ssd_keras_b200 import _ffi
    B = len(counts)
    offs_in = torch.tensor(np.cumsum([0] + list(counts)), dtype=torch.int32, device='cuda')
    ops_dev, m = _pack(ops_lists, B, max_ops) if ops_lists else (None, 0)
    offs_out = torch.full((B + 1,), -5, dtype=torch.int32, device='cuda')
    st = torch.full((2,), -5, dtype=torch.int32, device='cuda') if stats else None
    _ffi.check(_ffi.lib().ssdk_assemble_batch(_ffi.context(), _ffi.dptr(gt_in), int(f64), _ffi.dptr(offs_in), B, int(sum(counts)),
                                              _ffi.dptr(ops_dev), int(m), _ffi.dptr(gt_out), _ffi.dptr(offs_out), _ffi.dptr(st),
                                              _ffi.stream_ptr()))
    return offs_out.cpu().numpy(), (st.cpu().numpy() if stats else None)


def test_raw_entry_point_edges(ba):
    import torch
    rng = np.random.default_rng(3)
    SENT = -12345.5
    # no boxes at all (gt_in NULL) and no stats
    out = torch.full((4, 5), SENT, device='cuda')
    offs, _ = _raw(None, 1, [0, 0, 0], [[ba.flip(10)], [], [ba.resize(4, 4, 8, 8)]], out, stats=False)
    assert offs.tolist() == [0, 0, 0, 0] and bool((out == SENT).all())
    # float32 input: the float32 values widened to float64, then the float64 chain
    labels = [ac.scattered_labels(rng, g) + rng.uniform(0, 0.01, (g, 5)) * [0, 1, 1, 1, 1] for g in (40, 0, 200)]
    labels[2][5, 1] = np.nan
    labels[2][6, 3] = -np.inf
    f32 = [l.astype(np.float32) for l in labels]
    ops = [ac.scattered_ops(), [ba.flip(80)], ac.scattered_ops() + [ba.clip(90, 70)]]
    flat = torch.from_numpy(np.concatenate(f32)).cuda()
    out = torch.full((250, 5), SENT, device='cuda')
    offs, st = _raw(flat, 0, [40, 0, 200], ops, out)
    refs = [bo.apply_box_ops(l.astype(np.float64), o) for l, o in zip(f32, ops)]
    assert offs.tolist() == np.cumsum([0] + [r.shape[0] for r in refs]).tolist() and st[0] == offs[-1]
    assert_f32_bits(out[:offs[-1]].cpu().numpy(), np.concatenate(refs), 'float32 input')
    assert bool((out[offs[-1]:] == SENT).all()), 'rows past the output were written'
    # lists of exactly max_ops entries (no END), codes 11-24 and ROTATE by 0 / 45 skipped, a list cut short by END
    lab = [np.array([[1, 2.5, 3.5, 9.5, 12.5], [2, -0.4, -0.3, 5, 6]])] * 4
    full = [[ba.flip(20), (11, 0, 1, 2, 3, 4), (15, 7, 0, 0, 0, 0), ba.rotate(20, 30, 90)],
            [(8, 0, 0.0, 20.0, 30.0, 0.0), (8, 0, 45.0, 20.0, 30.0, 0.0), ba.brightness(10.0), ba.channel_swap((2, 1, 0))],
            [(24, 0, 2.0, 1.0, 0.0, 0.0), (16, 0, 0, 0, 0, 0), (23, 0, 0, 0, 0, 0), ba.scale(20, 30, 1.5)],
            [ba.flip(30), (0, 0, 0, 0, 0, 0), ba.flip(30), ba.flip(30)]]
    flat = torch.from_numpy(np.concatenate(lab)).cuda()
    out = torch.full((8, 5), SENT, device='cuda')
    offs, st = _raw(flat, 1, [2] * 4, full, out)
    refs = [bo.apply_box_ops(l, o) for l, o in zip(lab, full)]
    assert_f32_bits(out.cpu().numpy(), np.concatenate(refs), 'max_ops lists')
    assert_f32_bits(out[2:4].cpu().numpy(), lab[1], 'skipped codes leave the boxes alone')
    # the workspace grows, shrinks and grows again; each result checked
    for g in (5, 5000, 3, 20000, 7):
        lab = [ac.scattered_labels(rng, g)]
        flat = torch.from_numpy(lab[0]).cuda()
        out = torch.full((g + 3, 5), SENT, device='cuda')
        offs, st = _raw(flat, 1, [g], [ac.scattered_ops()], out)
        ref = bo.apply_box_ops(lab[0], ac.scattered_ops())
        assert offs.tolist() == [0, ref.shape[0]] and st.tolist() == [ref.shape[0], ref.shape[0]]
        assert_f32_bits(out[:offs[-1]].cpu().numpy(), ref, 'G = %d' % g)
        assert bool((out[offs[-1]:] == SENT).all())


def test_edge_case_feeds_the_encoder(configs):
    from ssd_keras_b200.data_generator.batch_assembly import encode_batch_device
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    rng = np.random.default_rng(21)
    labels = [ac.scattered_labels(rng, g) for g in (3, 150, 0, 40)]
    labels[1][:, 0] = rng.integers(1, 21, 150)
    ops = [ac.scattered_ops() for _ in labels]
    enc = SSDInputEncoder(**configs['ssd300'])
    y = encode_batch_device(enc, labels, ops).cpu().numpy()
    y_ref = enc([bo.apply_box_ops(l, o) for l, o in zip(labels, ops)])
    np.testing.assert_array_equal(y, y_ref.astype(np.float32))


# ------------------------------------------------------------------------------------------------
# images
# ------------------------------------------------------------------------------------------------
def _image(rng, shape):
    h, w, c = shape
    return rng.integers(0, 256, (h, w) if c == 1 and rng.random() < 0.5 else (h, w, c), dtype=np.uint8)


def _expected(images, ops):
    import torch
    return torch.from_numpy(np.stack([wo.apply_ops(po.apply_ops(im, o), po.split_ops(o)[1]) for im, o in zip(images, ops)]).astype(np.float32))


def _assemble(images, ops, oh, ow, out=None):
    from ssd_keras_b200.data_generator.batch_assembly import assemble_images_device
    return assemble_images_device(images, ops, oh, ow, out=out)


def test_every_mode_at_its_edges():
    import torch
    rng = np.random.default_rng(7)
    for name, shape, ops, oh, ow in ac.image_edge_cases():
        img = _image(rng, shape)
        x = _assemble([img, img], [ops, ops], oh, ow).cpu()
        ref = _expected([img], [ops])[0]
        assert torch.equal(x[0], ref) and torch.equal(x[1], ref), (name, ac.image_plan(shape, ops, oh, ow))


def test_warps_that_saturate_and_the_refusal(ba):
    import torch
    rng = np.random.default_rng(8)
    cases, (lo, hi) = ac.warp_cases()
    for name, (h, w, c), f in cases:
        img = _image(rng, (h, w, c))
        ops = [ba.scale(h, w, f, background=(9, 200, 31))]
        assert torch.equal(_assemble([img], [ops], h, w).cpu()[0], _expected([img], [ops])[0]), (name, f)
    img = _image(rng, (100, 120, 3))
    with pytest.raises(ValueError):
        _assemble([img], [[ba.scale(100, 120, lo)]], 100, 120)


def test_same_bytes_with_and_without_the_warp_instantiation(ba):
    import torch
    rng = np.random.default_rng(9)
    cases = [c for c in ac.image_edge_cases() if c[3:] == (20, 30)]
    imgs = [_image(rng, c[1]) for c in cases]
    ops = [c[2] for c in cases]
    assert ac.instantiation([ac.image_plan(c[1], c[2], 20, 30) for c in cases]) == 'image_assemble_kernel<false>'
    plain = _assemble(imgs, ops, 20, 30).cpu()
    warp_img = _image(rng, (20, 30, 3))
    mixed = _assemble(imgs + [warp_img], ops + [[ba.scale(20, 30, 1.7)]], 20, 30).cpu()
    assert torch.equal(plain, mixed[:-1]) and torch.equal(plain, _expected(imgs, ops))
    assert torch.equal(mixed[-1], _expected([warp_img], [[ba.scale(20, 30, 1.7)]])[0])


def test_grid_limit():
    import torch
    rng = np.random.default_rng(10)
    px = rng.integers(0, 256, (ac.MAX_B, 1, 1, 3), dtype=np.uint8)
    x = _assemble(list(px), None, 1, 1)
    assert torch.equal(x.cpu(), torch.from_numpy(px.astype(np.float32)))
    with pytest.raises(ValueError):
        _assemble(list(px) + [px[0]], None, 1, 1)


def test_photometric_widths_and_byte_offsets(ba):
    import torch
    rng = np.random.default_rng(12)
    seq = ba.photometric_ops(1, brightness=17.5, contrast=1.3, saturation=0.7, hue=-9.0, channel_swap=(2, 0, 1))
    imgs, ops = [], []
    for w in ac.PHOTO_WIDTHS:
        for c in (1, 3, 4):
            imgs.append(np.zeros((1, 1, 1), np.uint8) + 77)                    # one byte: the next image starts at an odd offset
            ops.append([])
            imgs.append(rng.integers(0, 256, (3, w, c), dtype=np.uint8))
            ops.append(seq)
    gx, tails = ac.photo_grid([im.shape[:2] for im, o in zip(imgs, ops) if o])
    assert gx == 1 and set(tails) == {0, 1, 31}
    H, W = 4, 4
    geo = [[ba.resize(im.shape[0], im.shape[1], H, W, interpolation_mode=0)] for im in imgs]
    full = [o + g for o, g in zip(ops, geo)]
    x = _assemble(imgs, full, H, W).cpu()
    assert torch.equal(x, _expected(imgs, full))
    img = rng.integers(0, 256, (5, 33, 3), dtype=np.uint8)
    f32, u8 = ba.convert_dtype('float32'), ba.convert_dtype('uint8')
    ok = [f32] + [ba.brightness(3.0 - k) for k in range(ac.PHOTO_MAX_STAGES - 2)] + [u8]
    assert len(ok) == ac.PHOTO_MAX_STAGES
    assert torch.equal(_assemble([img], [ok], 5, 33).cpu(), _expected([img], [ok]))
    with pytest.raises(ValueError):
        _assemble([img], [[f32, ba.brightness(1.0)] + ok[1:]], 5, 33)


def test_source_past_two_gigabytes(ba):
    """Both images and the photometric prefix read from byte offsets above 2^31 of the packed buffer."""
    import torch
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.data_generator.batch_assembly import _pack_ops
    rng = np.random.default_rng(13)
    a, b = rng.integers(0, 256, (17, 23, 3), dtype=np.uint8), rng.integers(0, 256, (9, 40, 4), dtype=np.uint8)
    base = (1 << 31) + 5
    offs = np.array([base, base + a.size, base + a.size + b.size], np.int64)
    src = torch.zeros((int(offs[-1]) + 16,), dtype=torch.uint8, device='cuda')
    src[offs[0]:offs[1]] = torch.from_numpy(a.reshape(-1)).cuda()
    src[offs[1]:offs[2]] = torch.from_numpy(b.reshape(-1)).cuda()
    hwc = np.array([[17, 23, 3], [9, 40, 4]], np.int32)
    ops = [[ba.crop_pad(-2, 3, 20, 18), ba.resize(20, 18, 12, 14)],
           ba.photometric_ops(2, brightness=-20.0, contrast=0.8) + [ba.resize(9, 40, 12, 14, interpolation_mode=0)]]
    arr, max_ops = _pack_ops(ops, 2)
    x = torch.full((2, 12, 14, 3), -1.0, device='cuda')
    _ffi.check(_ffi.lib().ssdk_assemble_images(_ffi.context(), _ffi.dptr(src), _ffi.np_ptr(offs, C.c_longlong), _ffi.np_ptr(hwc, C.c_int),
                                               2, arr, int(max_ops), 12, 14, _ffi.dptr(x), _ffi.stream_ptr()))
    got = x.cpu()
    del src
    torch.cuda.empty_cache()
    assert torch.equal(got, _expected([a, b], ops))


def test_ten_calls_in_flight(ba):
    """More calls than the descriptor ring has slots, with different lists and no synchronisation between them."""
    import torch
    rng = np.random.default_rng(14)
    H, W = 24, 32
    calls = []
    for t in range(10):
        warp = t % 3 == 0                                            # these calls run the <true> instantiation
        imgs = [_image(rng, (H, W, 3) if warp else (int(rng.integers(5, 50)), int(rng.integers(5, 50)), (1, 3, 4)[t % 3]))
                for _ in range(3 + t)]
        ops = []
        for im in imgs:
            h, w = im.shape[:2]
            lst = ba.scale_ops(H, W, float(rng.uniform(0.5, 2.0)), clip_boxes=False) if warp else [
                ba.resize(h, w, H, W, interpolation_mode=int(rng.integers(2)))]
            if t % 2:
                lst = ba.photometric_ops(1, brightness=float(rng.uniform(-30, 30))) + lst
            ops.append(lst)
        calls.append((imgs, ops, torch.full((len(imgs), H, W, 3), -3.0, device='cuda')))
    torch.cuda._sleep(50_000_000)
    for imgs, ops, out in calls:
        _assemble(imgs, ops, H, W, out=out)
    torch.cuda.synchronize()
    for t, (imgs, ops, out) in enumerate(calls):
        assert torch.equal(out.cpu(), _expected(imgs, ops)), t
