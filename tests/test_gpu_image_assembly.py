"""ssdk_assemble_images on the device: bit-identical to oracle/imageops.py (itself pinned to the reference's CropPad / Flip /
Resize / SSDExpand and to cv2 by tests/test_image_ops_cpu.py) on every golden case and on seeded ragged batches, the one op
list driving both halves of a training batch, errors that leave ``out`` untouched, box results unchanged by the new flag bits,
one launch per call and no host synchronisation."""
import os

import numpy as np
import pytest

from oracle import imageops as io

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, 'golden', 'ref_image_ops_golden.npz'))
MEAN = (123, 117, 104)


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()


def _assemble(images, ops, oh, ow, out=None):
    from ssd_keras_b200.data_generator.batch_assembly import assemble_images_device
    return assemble_images_device(images, ops, oh, ow, out=out)


def _expected(images, ops):
    import torch
    return torch.from_numpy(np.stack([io.apply_ops(im, o) for im, o in zip(images, ops)]).astype(np.float32))


def test_golden_cases_bit_identical():
    import torch
    groups = {}
    for k in range(int(G['n'])):
        groups.setdefault(G['out%d' % k].shape[:2], []).append(k)
    for (oh, ow), ks in groups.items():
        images = [G['in%d' % k] for k in ks]
        ops = [[tuple(r) for r in G['ops%d' % k].tolist()] for k in ks]
        x = _assemble(images, ops, oh, ow).cpu()
        ref = torch.from_numpy(np.stack([G['out%d' % k] for k in ks]).astype(np.float32))
        assert torch.equal(x, ref), [k for i, k in enumerate(ks) if not torch.equal(x[i], ref[i])]


def _ssd_chain(rng, h, w, oh, ow, mode):
    """The geometric part of the original SSD chain with decided parameters: expand (mean colour) -> crop -> flip -> resize."""
    from ssd_keras_b200.data_generator import batch_assembly as ba
    ops, ch, cw = [], h, w
    if rng.random() < 0.7:
        r = rng.uniform(1, 4)
        ph, pw = int(ch * r), int(cw * r)
        ops.append(ba.crop_pad(-int(rng.integers(0, ph - ch + 1)), -int(rng.integers(0, pw - cw + 1)), ph, pw,
                               center_point_filter=False, clip_boxes=False, background=MEAN))
        ch, cw = ph, pw
    if rng.random() < 0.7:
        ph, pw = max(1, int(ch * rng.uniform(0.3, 1))), max(1, int(cw * rng.uniform(0.3, 1)))
        ops.append(ba.crop_pad(int(rng.integers(0, ch - ph + 1)), int(rng.integers(0, cw - pw + 1)), ph, pw,
                               center_point_filter=True, clip_boxes=True))
        ch, cw = ph, pw
    if rng.random() < 0.5:
        ops.append(ba.flip(cw, 'horizontal'))
    if rng.random() < 0.2:
        ops.append(ba.flip(ch, 'vertical'))
    ops.append(ba.resize(ch, cw, oh, ow, interpolation_mode=mode))
    ops.append(ba.box_filter(check_degenerate=True))
    return ops


def _ragged(rng, B, oh, ow):
    images, ops = [], []
    for b in range(B):
        h, w = int(rng.integers(1, 160)), int(rng.integers(1, 160))
        c = (0, 1, 3, 4)[int(rng.integers(4))]
        images.append(rng.integers(0, 256, (h, w) if c == 0 else (h, w, c), dtype=np.uint8))
        if b % 9 == 8:
            ops.append(_to_2x(oh, ow))
        else:
            ops.append(_ssd_chain(rng, h, w, oh, ow, b % 2))
    return images, ops


def _to_2x(oh, ow):
    """Crop / pad to (2*oh, 2*ow), then an exact 2x linear downscale (cv2's INTER_AREA fast path)."""
    from ssd_keras_b200.data_generator import batch_assembly as ba
    return [ba.crop_pad(-3, 0, 2 * oh, 2 * ow, background=(9, 8, 7)), ba.flip(2 * ow), ba.resize(2 * oh, 2 * ow, oh, ow)]


@pytest.mark.parametrize('B', [1, 7, 64])
def test_random_ragged_batches_bit_identical(B):
    import torch
    rng = np.random.default_rng(100 + B)
    for oh, ow in ((300, 300), (37, 91)):
        images, ops = _ragged(rng, B, oh, ow)
        x = _assemble(images, ops, oh, ow)
        assert x.shape == (B, oh, ow, 3) and x.dtype == torch.float32
        ref = _expected(images, ops)
        bad = [b for b in range(B) if not torch.equal(x[b].cpu(), ref[b])]
        assert not bad, (bad, [ops[b] for b in bad[:3]])
        # `out` is reused
        out = torch.full((B, oh, ow, 3), -1.0, device='cuda')
        assert _assemble(images, ops, oh, ow, out=out) is out
        assert torch.equal(out.cpu(), ref)


def test_no_resize_and_accepted_background_rules():
    import torch
    from ssd_keras_b200.data_generator import batch_assembly as ba
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (10, 12, 3), dtype=np.uint8)
    lists = [[ba.crop_pad(-2, -2, 14, 16, background=(1, 2, 3)), ba.crop_pad(-1, -1, 16, 18, background=(1, 2, 3)),
              ba.crop_pad(0, 0, 16, 18, background=(200, 0, 0))],                                    # the last patch stays inside
             [ba.crop_pad(-40, -40, 16, 18, background=(5, 6, 7))],                                   # nothing of the image left
             [ba.flip(12), ba.crop_pad(3, 4, 16, 18, background=(4, 4, 4)), ba.flip(16, 'vertical')]]
    x = _assemble([img] * 3, lists, 16, 18)
    assert torch.equal(x.cpu(), _expected([img] * 3, lists))


def _ssd7(B, H, W, ncls):
    from ssd_keras_b200.models.keras_ssd7 import build_model
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    sc = [0.08, 0.16, 0.32, 0.64, 0.96]
    m = build_model((H, W, 3), ncls, mode='training', l2_regularization=5e-4, scales=sc, normalize_coords=True, weights_seed=4,
                    subtract_mean=127.5, divide_by_stddev=127.5)
    enc = SSDInputEncoder(img_height=H, img_width=W, n_classes=ncls, predictor_sizes=m.predictor_sizes, scales=sc,
                          aspect_ratios_global=[0.5, 1.0, 2.0], variances=[1.0] * 4, pos_iou_threshold=0.4, neg_iou_limit=0.3,
                          normalize_coords=True)
    return m, enc


def _batch(rng, B, H, W, ncls):
    images, labels, ops = [], [], []
    for b in range(B):
        h, w = int(rng.integers(60, 220)), int(rng.integers(60, 220))
        c = (3, 3, 1, 4)[b % 4]
        images.append(rng.integers(0, 256, (h, w, c), dtype=np.uint8))
        n = int(rng.integers(1, 6))
        x0, y0 = rng.integers(0, w - 20, n), rng.integers(0, h - 20, n)
        labels.append(np.stack([rng.integers(1, ncls + 1, n), x0, y0, np.minimum(x0 + rng.integers(8, w // 2, n), w - 1),
                                np.minimum(y0 + rng.integers(8, h // 2, n), h - 1)], axis=1).astype(np.int64))
        ops.append(_ssd_chain(rng, h, w, H, W, b % 2))
    return images, labels, ops


def test_training_batch_drives_both_halves():
    import torch
    from ssd_keras_b200 import _ffi
    from ssd_keras_b200.data_generator.batch_assembly import assemble_training_batch, encode_batch_device
    from ssd_keras_b200.training import SSDTrainer
    B, H, W, ncls = 4, 96, 128, 5
    m, enc = _ssd7(B, H, W, ncls)
    rng = np.random.default_rng(11)
    images, labels, ops = _batch(rng, B, H, W, ncls)
    x, y = assemble_training_batch(enc, images, labels, ops, H, W)
    x_ref = _expected(images, ops)
    assert torch.equal(x.cpu(), x_ref)
    y_ref = encode_batch_device(enc, labels, ops)
    assert torch.equal(y, y_ref)
    # launches: the image kernel plus exactly what the box + encoder path already launches
    n0 = _ffi.launch_count()
    encode_batch_device(enc, labels, ops)
    n1 = _ffi.launch_count()
    assemble_training_batch(enc, images, labels, ops, H, W)
    n2 = _ffi.launch_count()
    _assemble(images, ops, H, W)
    n3 = _ffi.launch_count()
    assert n3 - n2 == 1 and n2 - n1 == (n1 - n0) + 1
    # the training step sees the same input bits whichever way the batch was built (asserted above), so it computes the same
    # loss bits; the weight gradients are summed with float atomics, so two runs on identical inputs may differ in the last
    # bits: the device-built batch is held to the spread of two host-built runs
    tr = SSDTrainer(m, B, lr=1e-3, l2_regularization=5e-4, optimizer='adam')
    loss_dev, _ = tr.forward_backward(x, y)
    g_dev = tr.grad.clone()
    loss_host, _ = tr.forward_backward(x_ref.cuda(), y_ref.clone())
    g_host = tr.grad.clone()
    loss_host2, _ = tr.forward_backward(x_ref.cuda(), y_ref.clone())
    g_host2 = tr.grad.clone()
    assert torch.equal(loss_dev, loss_host) and torch.equal(loss_host, loss_host2)
    spread = float((g_host - g_host2).abs().max())
    scale = float(g_host.abs().max())
    assert float((g_dev - g_host).abs().max()) <= max(4 * spread, 1e-6 * scale), (float((g_dev - g_host).abs().max()), spread, scale)
    assert torch.isfinite(loss_dev).all() and scale > 0


def test_training_batch_does_not_synchronise():
    import torch
    from ssd_keras_b200.data_generator.batch_assembly import assemble_training_batch
    B, H, W, ncls = 8, 96, 128, 5
    _, enc = _ssd7(B, H, W, ncls)
    rng = np.random.default_rng(12)
    images, labels, ops = _batch(rng, B, H, W, ncls)
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
    assert torch.equal(x.cpu(), _expected(images, ops))


def test_errors_leave_out_untouched():
    import torch
    from ssd_keras_b200.data_generator import batch_assembly as ba
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (10, 10, 3), dtype=np.uint8)
    out = torch.full((2, 5, 5, 3), -7.0, device='cuda')
    bad = [[ba.resize(10, 10, 5, 5, interpolation_mode=2)],
           [ba.crop_pad(11, 0, 5, 5), ba.resize(5, 5, 5, 5)],
           [ba.resize(10, 12, 5, 5)],
           [ba.resize(10, 10, 5, 5), ba.flip(5)],
           [ba.resize(10, 10, 6, 5)],
           [ba.crop_pad(-1, -1, 12, 12, background=(1, 1, 1)), ba.crop_pad(-1, -1, 14, 14), ba.resize(14, 14, 5, 5)]]
    for lst in bad:
        with pytest.raises(ValueError):
            _assemble([img, img], [[ba.resize(10, 10, 5, 5)], lst], 5, 5, out=out)
        torch.cuda.synchronize()
        assert bool((out == -7.0).all()), lst
    with pytest.raises(ValueError):
        _assemble([img, np.zeros((4, 4, 2), np.uint8)], [[ba.resize(10, 10, 5, 5)], [ba.resize(4, 4, 5, 5)]], 5, 5, out=out)
    with pytest.raises(ValueError):
        _assemble([img, img.astype(np.float32)], [[ba.resize(10, 10, 5, 5)]] * 2, 5, 5, out=out)
    torch.cuda.synchronize()
    assert bool((out == -7.0).all())


def test_box_results_ignore_the_image_flag_bits():
    import torch
    from ssd_keras_b200.data_generator.batch_assembly import assemble_batch_device
    rng = np.random.default_rng(21)
    B, H, W, ncls = 16, 96, 128, 5
    images, labels, ops = _batch(rng, B, H, W, ncls)
    plain = [[(o[0], o[1] & 3, *o[2:]) for o in lst] for lst in ops]
    assert any(o[1] != p[1] for lst, pl in zip(ops, plain) for o, p in zip(lst, pl))
    a = assemble_batch_device(labels, ops)
    b = assemble_batch_device(labels, plain)
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]) and a[3:] == b[3:]
    n = int(a[1][-1])                                     # rows past the survivors are not written
    assert n > 0 and torch.equal(a[0][:n], b[0][:n])
