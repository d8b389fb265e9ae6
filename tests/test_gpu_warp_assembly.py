"""Translate / Scale / Rotate and BoxFilter's overlap test on the device: ssdk_assemble_images bit-identical to
oracle/warpops.py and ssdk_assemble_batch to oracle/boxops.py (both pinned to the reference's classes and to cv2 by
tests/test_warp_ops_cpu.py) on the golden cases and on random batches that mix both SSD7 sequences, the satellite list and
the original SSD chain; an SSD7 training batch whose y_true equals the host encoder of the oracle's boxes; no host
synchronisation; refused calls that leave ``out`` untouched."""
import os

import numpy as np
import pytest

from oracle import boxops as bo
from oracle import warpops as io

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, 'golden', 'ref_warp_golden.npz'))
MEAN = (123, 117, 104)
SSD7_FILTER = dict(check_overlap=True, check_min_area=True, check_degenerate=True, overlap_criterion='area', overlap_bounds=(0.3, 1.0),
                   min_area=16)
PATCH_FILTER = dict(check_overlap=True, check_min_area=False, check_degenerate=False, overlap_criterion='area', overlap_bounds=(0.3, 1.0))
RESIZE_FILTER = dict(check_overlap=False, check_min_area=True, check_degenerate=True, min_area=16)


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()


def _expected_images(images, ops):
    import torch
    return torch.from_numpy(np.stack([io.apply_ops(im, o) for im, o in zip(images, ops)]).astype(np.float32))


def _check_boxes(labels, ops, golden=None):
    from ssd_keras_b200.data_generator.batch_assembly import assemble_batch_device
    gt, offs, stats, _, _ = assemble_batch_device(labels, ops)
    gt, offs, stats = gt.cpu().numpy(), offs.cpu().numpy(), stats.cpu().numpy()
    for b in range(len(labels)):
        ref = bo.apply_box_ops(labels[b], ops[b])
        if golden is not None:
            np.testing.assert_array_equal(ref, golden[b])
        got = gt[offs[b]:offs[b + 1]]
        assert got.shape == ref.shape, (b, got.shape, ref.shape, ops[b])
        np.testing.assert_array_equal(got, ref.astype(np.float32), err_msg='image %d: %r' % (b, ops[b]))
    assert stats[0] == offs[-1]


def test_golden_cases_bit_identical():
    import torch
    from ssd_keras_b200.data_generator.batch_assembly import assemble_images_device
    n = int(G['n'])
    ops = [[(int(r[0]), int(r[1]), *r[2:]) for r in G['ops%d' % k].tolist()] for k in range(n)]
    groups = {}
    for k in range(n):
        groups.setdefault(G['out%d' % k].shape[:2], []).append(k)
    for (oh, ow), ks in groups.items():
        x = assemble_images_device([G['in%d' % k] for k in ks], [ops[k] for k in ks], oh, ow).cpu()
        ref = torch.from_numpy(np.stack([G['out%d' % k] for k in ks]).astype(np.float32))
        assert torch.equal(x, ref), [(k, str(G['kind%d' % k])) for i, k in enumerate(ks) if not torch.equal(x[i], ref[i])]
    _check_boxes([G['lin%d' % k] for k in range(n)], ops, [G['lout%d' % k] for k in range(n)])


def _labels(rng, h, w):
    n = int(rng.integers(0, 8))
    x0, y0 = rng.integers(-w // 4, w, n), rng.integers(-h // 4, h, n)
    return np.stack([rng.integers(1, 6, n), x0, y0, x0 + rng.integers(1, max(2, w // 2), n), y0 + rng.integers(1, max(2, h // 2), n)],
                    axis=1).astype(np.float64).reshape(-1, 5)


def _ssd7_chain(rng, H, W, seq, bg):
    """The geometric half of one DataAugmentationConstantInputSize sequence, with decided parameters."""
    from ssd_keras_b200.data_generator import batch_assembly as ba
    ops = []

    def translate():
        if rng.random() < 0.7:
            dy, dx = rng.uniform(0.03, 0.5) * rng.choice([-1, 1]), rng.uniform(0.03, 0.5) * rng.choice([-1, 1])
            ops.extend(ba.translate_ops(H, W, dy, dx, box_filter=SSD7_FILTER, clip_boxes=True, background=bg))

    def zoom(lo, hi):
        if rng.random() < 0.6:
            ops.extend(ba.scale_ops(H, W, rng.uniform(lo, hi), box_filter=SSD7_FILTER, clip_boxes=True, background=bg))
    if seq == 1:
        translate()
        zoom(1.0, 2.0)
    else:
        zoom(0.5, 1.0)
        translate()
    if rng.random() < 0.5:
        ops.append(ba.flip(W))
    return ops


def _satellite_chain(rng, h, w, H, W):
    """The geometric half of DataAugmentationSatellite: flips -> rotate -> patch ('area' filter, clip) -> resize."""
    from ssd_keras_b200.data_generator import batch_assembly as ba
    ops = []
    if rng.random() < 0.5:
        ops.append(ba.flip(w))
    if rng.random() < 0.5:
        ops.append(ba.flip(h, 'vertical'))
    if rng.random() < 0.5:
        a = int(rng.choice([90, 180, 270]))
        ops.extend(ba.rotate_ops(h, w, a))
        if a != 180:
            h, w = w, h
    ph, pw = max(1, int(h * rng.uniform(0.3, 1.5))), max(1, int(w * rng.uniform(0.3, 1.5)))
    py, px = int(rng.integers(min(0, h - ph), max(0, h - ph) + 1)), int(rng.integers(min(0, w - pw), max(0, w - pw) + 1))
    ops.extend(ba.crop_pad_ops(py, px, ph, pw, box_filter=PATCH_FILTER, clip_boxes=True))
    ops.extend(ba.resize_ops(ph, pw, H, W, box_filter=RESIZE_FILTER))
    return ops


def _ssd_chain(rng, h, w, H, W):
    """The original SSD chain's geometric half: expand (mean colour) -> crop -> flip -> resize."""
    from ssd_keras_b200.data_generator import batch_assembly as ba
    ops, ch, cw = [], h, w
    if rng.random() < 0.6:
        r = rng.uniform(1, 3)
        ph, pw = int(ch * r), int(cw * r)
        ops.append(ba.crop_pad(-int(rng.integers(0, ph - ch + 1)), -int(rng.integers(0, pw - cw + 1)), ph, pw, clip_boxes=False, background=MEAN))
        ch, cw = ph, pw
    if rng.random() < 0.5:
        ops.append(ba.flip(cw))
    ops.append(ba.resize(ch, cw, H, W, interpolation_mode=int(rng.integers(2))))
    return ops


def _mixed_batch(rng, B, H, W):
    images, labels, ops = [], [], []
    for b in range(B):
        kind = b % 4
        if kind < 2:
            h, w = H, W
            bg = (0, 0, 0) if rng.random() < 0.5 else tuple(int(v) for v in rng.integers(0, 256, 3))
        else:
            h, w = int(rng.integers(1, 2 * H)), int(rng.integers(1, 2 * W))
        c = (3, 0, 4, 1)[int(rng.integers(4))]
        images.append(rng.integers(0, 256, (h, w) if c == 0 else (h, w, c), dtype=np.uint8))
        labels.append(_labels(rng, h, w))
        if kind < 2:
            ops.append(_ssd7_chain(rng, H, W, 1 + kind, bg))
        elif kind == 2:
            ops.append(_satellite_chain(rng, h, w, H, W))
        else:
            ops.append(_ssd_chain(rng, h, w, H, W))
    return images, labels, ops


def test_random_mixed_batches_bit_identical():
    """200 random chains in batches of 32: both SSD7 sequences, the satellite list and the original SSD chain."""
    import torch
    from ssd_keras_b200.data_generator.batch_assembly import assemble_images_device
    rng = np.random.default_rng(2718)
    n = 0
    for H, W in ((60, 96), (37, 23), (60, 96), (45, 45), (60, 96), (31, 70), (60, 96)):
        B = 32 if n + 32 <= 200 else 200 - n
        images, labels, ops = _mixed_batch(rng, B, H, W)
        x = assemble_images_device(images, ops, H, W)
        ref = _expected_images(images, ops)
        bad = [b for b in range(B) if not torch.equal(x[b].cpu(), ref[b])]
        assert not bad, [(b, ops[b]) for b in bad[:3]]
        _check_boxes(labels, ops)
        n += B
    assert n == 200


def test_integer_ops_after_scale_and_rotate_between():
    """Flips, translations, pads and a rotation after the SCALE map its output; rotations compose before a RESIZE."""
    import torch
    from ssd_keras_b200.data_generator import batch_assembly as ba
    from ssd_keras_b200.data_generator.batch_assembly import assemble_images_device
    rng = np.random.default_rng(9)
    img = rng.integers(0, 256, (21, 34, 3), dtype=np.uint8)
    lists = [[ba.scale(21, 34, 1.3), ba.rotate(21, 34, 90), ba.flip(21), ba.translate(34, 21, 0.2, -0.1), ba.crop_pad(2, -3, 34, 21)],
             [ba.rotate(21, 34, 270), ba.crop_pad(-2, -2, 38, 25), ba.scale(38, 25, 0.6), ba.flip(38, 'vertical'), ba.crop_pad(4, 2, 34, 21)],
             [ba.rotate(21, 34, 180), ba.rotate(21, 34, 90), ba.resize(34, 21, 34, 21)],
             [ba.translate(21, 34, 3.0, 0.0), ba.rotate(21, 34, 90), ba.resize(34, 21, 34, 21, interpolation_mode=0)]]
    x = assemble_images_device([img] * 4, lists, 34, 21)
    assert torch.equal(x.cpu(), _expected_images([img] * 4, lists))


def _ssd7_model(H, W, ncls):
    from ssd_keras_b200.models.keras_ssd7 import build_model
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    sc = [0.08, 0.16, 0.32, 0.64, 0.96]
    m = build_model((H, W, 3), ncls, mode='training', l2_regularization=5e-4, scales=sc, normalize_coords=True, weights_seed=4,
                    subtract_mean=127.5, divide_by_stddev=127.5)
    enc = SSDInputEncoder(img_height=H, img_width=W, n_classes=ncls, predictor_sizes=m.predictor_sizes, scales=sc,
                          aspect_ratios_global=[0.5, 1.0, 2.0], variances=[1.0] * 4, pos_iou_threshold=0.5, neg_iou_limit=0.3,
                          normalize_coords=True)
    return m, enc


def _ssd7_batch(rng, B, H, W, ncls):
    images, labels, ops = [], [], []
    for b in range(B):
        images.append(rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        n = int(rng.integers(1, 6))
        x0, y0 = rng.integers(0, W - 30, n), rng.integers(0, H - 30, n)
        labels.append(np.stack([rng.integers(1, ncls + 1, n), x0, y0, x0 + rng.integers(12, 60, n), y0 + rng.integers(12, 60, n)],
                               axis=1).astype(np.float64))
        ops.append(_ssd7_chain(rng, H, W, 1 + b % 2, (0, 0, 0)))
    return images, labels, ops


def test_ssd7_training_batch():
    import torch
    from ssd_keras_b200.data_generator.batch_assembly import assemble_training_batch
    B, H, W, ncls = 8, 120, 192, 5
    _, enc = _ssd7_model(H, W, ncls)
    rng = np.random.default_rng(17)
    images, labels, ops = _ssd7_batch(rng, B, H, W, ncls)
    x, y = assemble_training_batch(enc, images, labels, ops, H, W)
    assert torch.equal(x.cpu(), _expected_images(images, ops))
    y_ref = enc([bo.apply_box_ops(l, o) for l, o in zip(labels, ops)])
    np.testing.assert_array_equal(y.cpu().numpy(), y_ref.astype(np.float32))


def test_ssd7_training_batch_does_not_synchronise():
    import torch
    from ssd_keras_b200.data_generator.batch_assembly import assemble_training_batch
    B, H, W, ncls = 8, 120, 192, 5
    _, enc = _ssd7_model(H, W, ncls)
    rng = np.random.default_rng(18)
    images, labels, ops = _ssd7_batch(rng, B, H, W, ncls)
    x_out = torch.empty((B, H, W, 3), device='cuda')
    y_out = torch.empty((B, enc.anchors.shape[0], ncls + 1 + 12), device='cuda')
    assemble_training_batch(enc, images, labels, ops, H, W, x_out=x_out, y_out=y_out)        # warm: encoder, pinned pools
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode('error')
    try:
        torch.cuda._sleep(200_000_000)                            # keeps the stream busy while the host enqueues
        x, y = assemble_training_batch(enc, images, labels, ops, H, W, x_out=x_out, y_out=y_out)
        busy = not torch.cuda.current_stream().query()
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    assert busy, 'assemble_training_batch waited for the device'
    torch.cuda.synchronize()
    assert x is x_out and y is y_out
    assert torch.equal(x.cpu(), _expected_images(images, ops))


def test_errors_leave_out_untouched():
    import torch
    from ssd_keras_b200.data_generator import batch_assembly as ba
    from ssd_keras_b200.data_generator.batch_assembly import assemble_images_device
    rng = np.random.default_rng(4)
    img = rng.integers(0, 256, (10, 12, 3), dtype=np.uint8)
    out = torch.full((2, 10, 12, 3), -7.0, device='cuda')
    bad = [[ba.scale(10, 12, 1.5), ba.scale(10, 12, 0.7)],
           [ba.scale(12, 10, 1.5)],
           [ba.translate(10, 12, 0.2, 0.0, background=(1, 2, 3)), ba.scale(10, 12, 1.5)],
           [(8, 0, 45.0, 10.0, 12.0, 0.0)],
           [ba.rotate(10, 12, 90)],
           [ba.resize(10, 12, 10, 12), ba.translate(10, 12, 0.2, 0.0)]]
    for lst in bad:
        with pytest.raises(ValueError):
            assemble_images_device([img, img], [[ba.scale(10, 12, 1.2)], lst], 10, 12, out=out)
        torch.cuda.synchronize()
        assert bool((out == -7.0).all()), lst
