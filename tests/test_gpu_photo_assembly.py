"""The photometric prefix of the op lists on the device (photometric_kernel in front of image_assemble_kernel): equal to
oracle/photoops.py (itself pinned to the reference's classes and to cv2 by tests/test_photo_ops_cpu.py) on EVERY uint8 pixel
value -- each op alone and both sequences of SSDPhotometricDistortions -- and through whole chains with the geometric ops;
mixed batches, batches without photometric ops unchanged and without the extra launch, the box half unchanged by the new codes,
rejected lists that leave ``out`` untouched, and one training step from photometric + geometric op lists."""
import os

import numpy as np
import pytest

from oracle import imageops as io
from oracle import photoops as po
from oracle import warpops as wo

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
MEAN = (123, 117, 104)
EDGE_PARAMS = [dict(brightness=32.0, contrast=1.5, saturation=1.5, hue=18.0),
               dict(brightness=-32.0, contrast=0.5, saturation=0.5, hue=-18.0),
               dict(brightness=84.5, saturation=2.0, hue=-1e-6, channel_swap=(2, 0, 1)),      # a delta of k + 0.5: ties; H = 180
               dict(brightness=-84.0, contrast=1.2345678, saturation=0.3, hue=179.99999),
               dict()]


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()


@pytest.fixture(scope='module')
def ba():
    from ssd_keras_b200.data_generator import batch_assembly
    return batch_assembly


def _assemble(images, ops, oh, ow, out=None):
    from ssd_keras_b200.data_generator.batch_assembly import assemble_images_device
    return assemble_images_device(images, ops, oh, ow, out=out)


def _device_u8(image, ops):
    """One image through ops that keep its size -> uint8 (h, w, 3) on the host."""
    h, w = image.shape[:2]
    x = _assemble([image], [ops], h, w)[0]
    return x.to(dtype=__import__('torch').uint8).cpu().numpy(), x


def _all_triples(width):
    a = np.arange(256, dtype=np.uint8)
    cube = np.stack(np.meshgrid(a, a, a, indexing='ij'), -1).reshape(-1, 3)
    rows = -(-len(cube) // width)
    return np.concatenate([cube, cube[:rows * width - len(cube)]]).reshape(rows, width, 3)


def _check_exhaustive(image, ops):
    import torch
    got, x = _device_u8(image, ops)
    assert bool((x == x.round()).all()) and float(x.min()) >= 0 and float(x.max()) <= 255
    del x
    torch.cuda.empty_cache()
    ref = po.apply_ops(image, ops)
    bad = np.argwhere((got != ref).any(-1))
    assert len(bad) == 0, (len(bad), bad[:5].tolist(), ops)


def test_every_rgb_triple_through_each_op(ba):
    img = _all_triples(4096)
    f32, u8 = ba.convert_dtype('float32'), ba.convert_dtype('uint8')
    singles = [[ba.convert_color('RGB', 'HSV')], [f32, u8]]
    singles += [[f32, ba.brightness(d), u8] for d in (32.0, -32.0, 84.0, -84.0, 0.5, -17.5)]
    singles += [[f32, ba.contrast(f), u8] for f in (0.5, 1.5, 0.7310585786300049)]
    singles += [[f32, ba.saturation(f), u8] for f in (0.3, 0.5, 1.5, 2.0)]
    singles += [[f32, ba.hue(d), u8] for d in (18.0, -18.0, 179.99999, -1e-6, 180.0, -180.0)]
    singles += [[ba.channel_swap(o)] for o in ((0, 2, 1), (1, 2, 0), (2, 1, 0))]
    for ops in singles:
        _check_exhaustive(img, ops)


@pytest.mark.parametrize('width', [4096, 50, 16])
def test_every_hsv_triple_through_hsv2rgb(ba, width):
    """4096: every pixel truncates (cv2's vector loop); 16: every pixel rounds (its scalar loop); 50: 32 + 18 per row."""
    _check_exhaustive(_all_triples(width), [ba.convert_color('HSV', 'RGB')])


@pytest.mark.parametrize('sequence', [1, 2])
@pytest.mark.parametrize('params', range(len(EDGE_PARAMS)))
def test_every_rgb_triple_through_the_sequences(ba, sequence, params):
    _check_exhaustive(_all_triples(4096 if params % 2 == 0 else 4000), ba.photometric_ops(sequence, **EDGE_PARAMS[params]))


def _image(rng, h, w, c):
    return rng.integers(0, 256, (h, w) if c == 0 else (h, w, c), dtype=np.uint8)


def _photo(rng, ba):
    draw = lambda lo, hi: float(rng.uniform(lo, hi)) if rng.random() < 0.5 else None          # noqa: E731
    return ba.photometric_ops(1 + int(rng.integers(2)), brightness=draw(-32, 32), contrast=draw(0.5, 1.5), saturation=draw(0.5, 1.5),
                              hue=draw(-18, 18), channel_swap=(1, 2, 0) if rng.random() < 0.1 else None)


def _ssd_geometry(rng, ba, h, w, oh, ow, mode):
    ops, ch, cw = [], h, w
    if rng.random() < 0.5:
        r = rng.uniform(1, 4)
        ph, pw = int(ch * r), int(cw * r)
        ops.append(ba.crop_pad(-int(rng.integers(0, ph - ch + 1)), -int(rng.integers(0, pw - cw + 1)), ph, pw, clip_boxes=False, background=MEAN))
        ch, cw = ph, pw
    if rng.random() < 0.7:
        ph, pw = max(1, int(ch * rng.uniform(0.3, 1))), max(1, int(cw * rng.uniform(0.3, 1)))
        ops.append(ba.crop_pad(int(rng.integers(0, ch - ph + 1)), int(rng.integers(0, cw - pw + 1)), ph, pw, center_point_filter=True))
        ch, cw = ph, pw
    if rng.random() < 0.5:
        ops.append(ba.flip(cw))
    return ops + [ba.resize(ch, cw, oh, ow, interpolation_mode=mode), ba.box_filter()]


def _ssd7_geometry(rng, ba, H, W):
    ops = []
    if rng.random() < 0.6:
        ops += ba.translate_ops(H, W, float(rng.uniform(-0.3, 0.3)), float(rng.uniform(-0.3, 0.3)))
    if rng.random() < 0.6:
        ops += ba.scale_ops(H, W, float(rng.uniform(0.5, 2.0)))
    if rng.random() < 0.5:
        ops.append(ba.flip(W))
    return ops


def _expected(images, ops, geometry):
    import torch
    return torch.from_numpy(np.stack([geometry.apply_ops(po.apply_ops(im, o), po.split_ops(o)[1]) for im, o in zip(images, ops)]).astype(np.float32))


def test_ssd_chains_bit_identical(ba):
    """photometric -> expand -> crop -> flip -> resize, VOC-like sizes, gray / RGBA inputs; ragged sizes put the images at odd
    byte offsets of the packed upload."""
    import torch
    rng = np.random.default_rng(300)
    for _ in range(4):
        images, ops = [], []
        for b in range(25):
            h, w = int(rng.integers(120, 376)), int(rng.integers(161, 501))
            images.append(_image(rng, h, w, (3, 3, 0, 4, 1)[b % 5]))
            ops.append(_photo(rng, ba) + _ssd_geometry(rng, ba, h, w, 150, 150, b % 2))
        assert len({sum(im.size for im in images[:b]) % 4 for b in range(25)}) > 1
        assert torch.equal(_assemble(images, ops, 150, 150).cpu(), _expected(images, ops, io))


def test_ssd7_chains_bit_identical(ba):
    """photometric -> translate -> scale -> flip at a constant input size."""
    import torch
    rng = np.random.default_rng(7)
    H, W = 150, 241
    for _ in range(4):
        images = [_image(rng, H, W, (3, 0, 4, 1)[b % 4]) for b in range(25)]
        ops = [_photo(rng, ba) + _ssd7_geometry(rng, ba, H, W) for _ in range(25)]
        assert torch.equal(_assemble(images, ops, H, W).cpu(), _expected(images, ops, wo))


def test_mixed_batch_equals_one_by_one(ba):
    import torch
    from ssd_keras_b200 import _ffi
    rng = np.random.default_rng(41)
    images, ops = [], []
    for b in range(12):
        h, w = int(rng.integers(5, 90)), int(rng.integers(1, 130))
        images.append(_image(rng, h, w, (3, 0, 4)[b % 3]))
        photo = [[], ba.photometric_ops(1 + b % 2), _photo(rng, ba)][b % 3 if b else 2]
        ops.append(photo + [ba.flip(w), ba.resize(h, w, 40, 40)])
    assert any(not po.split_ops(o)[0] for o in ops)
    n0 = _ffi.launch_count()
    x = _assemble(images, ops, 40, 40)
    assert _ffi.launch_count() - n0 == 2                          # one pre-pass for all of them, one assembly
    for b in range(12):
        assert torch.equal(x[b], _assemble([images[b]], [ops[b]], 40, 40)[0]), b
    assert torch.equal(x.cpu(), _expected(images, ops, io))


def test_batches_without_photometric_ops_are_unchanged(ba):
    """The goldens of the geometric ops, assembled after a photometric call has grown the scratch buffer: the same bits, one
    launch, so neither the pre-pass nor its scratch is touched."""
    import torch
    from ssd_keras_b200 import _ffi
    rng = np.random.default_rng(2)
    _assemble([_image(rng, 30, 30, 3)], [ba.photometric_ops(1, hue=3.0)], 30, 30)
    for name in ('ref_image_ops_golden.npz', 'ref_warp_golden.npz'):
        G = np.load(os.path.join(HERE, 'golden', name))
        keys = [k for k in range(int(G['n'])) if 'in%d' % k in G.files and 'out%d' % k in G.files]
        assert keys
        for k in keys:
            ref = G['out%d' % k]
            lst = [(int(r[0]), int(r[1]), *r[2:]) for r in G['ops%d' % k].tolist()]
            n0 = _ffi.launch_count()
            x = _assemble([G['in%d' % k]], [lst], ref.shape[0], ref.shape[1])
            assert _ffi.launch_count() - n0 == 1
            assert torch.equal(x[0].cpu(), torch.from_numpy(ref.astype(np.float32))), (name, k)


def test_box_half_ignores_the_photometric_codes(ba):
    import torch
    from ssd_keras_b200.data_generator.batch_assembly import assemble_batch_device
    rng = np.random.default_rng(9)
    H, W = 96, 128
    labels, with_photo, without = [], [], []
    for b in range(16):
        n = int(rng.integers(0, 6))
        x0, y0 = rng.integers(0, W - 20, n), rng.integers(0, H - 20, n)
        labels.append(np.stack([rng.integers(1, 5, n), x0, y0, x0 + rng.integers(4, 20, n), y0 + rng.integers(4, 20, n)], axis=1).astype(np.int64))
        geo = _ssd7_geometry(rng, ba, H, W) + [ba.box_filter()]
        without.append(geo)
        with_photo.append(_photo(rng, ba) + geo)
    a, b = assemble_batch_device(labels, with_photo), assemble_batch_device(labels, without)
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]) and a[3:] == b[3:]
    n = int(a[1][-1])
    assert n > 0 and torch.equal(a[0][:n], b[0][:n])


def test_rejected_lists_leave_out_untouched(ba):
    import torch
    rng = np.random.default_rng(3)
    img = _image(rng, 10, 10, 3)
    f32, u8 = ba.convert_dtype('float32'), ba.convert_dtype('uint8')
    out = torch.full((2, 10, 10, 3), -7.0, device='cuda')
    raw = lambda code, a0: (code, 0, a0, 0.0, 0.0, 0.0)           # noqa: E731  (past the constructors' own checks)
    bad = [[ba.flip(10), f32, ba.brightness(1.0), u8],            # photometric after geometric
           [ba.brightness(1.0)],                                  # float op in the uint8 state
           [f32, ba.convert_color('RGB', 'HSV'), u8],             # colour conversion in the float state
           [f32, ba.brightness(1.0)],                             # the prefix ends in the float state
           [f32, raw(po.CONTRAST, 0.0), u8], [f32, raw(po.SATURATION, -1.0), u8],     # factors
           [f32, raw(po.HUE, 180.5), u8], [f32, raw(po.BRIGHTNESS, float('nan')), u8],
           [(po.CHANNEL_SWAP, 0, 0.0, 0.0, 1.0, 0.0)], [(po.CHANNEL_SWAP, 0, 0.0, 1.0, 3.0, 0.0)],
           [f32, u8] * 8 + [ba.channel_swap((0, 1, 2))]]          # 17 stages
    for lst in bad:
        with pytest.raises(ValueError):
            _assemble([img, img], [ba.photometric_ops(1, hue=5.0), lst], 10, 10, out=out)
        torch.cuda.synchronize()
        assert bool((out == -7.0).all()), lst
    ok = [f32, u8] * 8                                            # 16 stages
    x = _assemble([img, img], [ok, ba.photometric_ops(2, contrast=1.3, hue=-5.0)], 10, 10, out=out)
    assert torch.equal(x.cpu(), _expected([img, img], [ok, ba.photometric_ops(2, contrast=1.3, hue=-5.0)], io))


def test_training_step_from_photometric_and_geometric_ops(ba):
    import torch
    from ssd_keras_b200.models.keras_ssd7 import build_model
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    from ssd_keras_b200.training import SSDTrainer
    B, H, W, ncls = 4, 96, 128, 5
    sc = [0.08, 0.16, 0.32, 0.64, 0.96]
    m = build_model((H, W, 3), ncls, mode='training', l2_regularization=5e-4, scales=sc, normalize_coords=True, weights_seed=4,
                    subtract_mean=127.5, divide_by_stddev=127.5)
    enc = SSDInputEncoder(img_height=H, img_width=W, n_classes=ncls, predictor_sizes=m.predictor_sizes, scales=sc,
                          aspect_ratios_global=[0.5, 1.0, 2.0], variances=[1.0] * 4, pos_iou_threshold=0.4, neg_iou_limit=0.3,
                          normalize_coords=True)
    rng = np.random.default_rng(15)
    images, labels, ops = [], [], []
    for b in range(B):
        h, w = int(rng.integers(100, 200)), int(rng.integers(130, 260))
        images.append(_image(rng, h, w, 3))
        labels.append(np.array([[1 + b % ncls, 10, 10, 60, 70], [2, 40, 30, 120, 90]], np.int64))
        ops.append(ba.photometric_ops(1 + b % 2, brightness=10.0 * b - 15.0, saturation=0.8 + 0.2 * b, hue=4.0 * b - 6.0)
                   + ba.crop_pad_ops(0, 0, 96, 128, box_filter=dict(min_area=4)) + [ba.flip(128)])
    x, y = ba.assemble_training_batch(enc, images, labels, ops, H, W)
    assert torch.equal(x.cpu(), _expected(images, ops, io))
    tr = SSDTrainer(m, B, lr=1e-3, l2_regularization=5e-4, optimizer='adam')
    loss = tr.train_on_batch(x, y)
    assert loss.shape == (B,) and bool(torch.isfinite(loss).all())
