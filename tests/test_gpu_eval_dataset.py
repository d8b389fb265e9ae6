"""Predictions over a dataset of mixed-size images on the GPU (eval_utils/dataset_predict.py, ssdk_eval_collect) against the
REAL reference's Evaluator.predict_on_dataset / write_predictions_to_txt / coco_utils.predict_all_to_json
(tests/golden/ref_eval_dataset_golden.npz), with the golden's stand-in model re-implemented on the device; real SSD7 models
against oracle/evalops.py applied to their own decoder output; the kernel alone; the device-results match path against the
list path."""
import hashlib
import os
import sys
import types

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)
from oracle import evalops  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'ref_eval_dataset_golden.npz')
RUNS = {'resize_inf': ('resize', 'inference', False, (300, 300), 8, 0),
        'pad_inf_r4': ('pad', 'inference', 4, (300, 300), 8, 1),
        'pad_inf_r3_wide': ('pad', 'inference', 3, (300, 480), 6, 2),
        'resize_train_wide': ('resize', 'training', False, (300, 480), 8, 0),
        'pad_train_r4': ('pad', 'training', 4, (300, 300), 7, 3)}
DECODE = dict(decoding_pred_coords='corners', decoding_normalize_coords=True, decoding_confidence_thresh=0.3, decoding_top_k=200)
N_CLASSES, K, P = 3, 12, 8


@pytest.fixture(scope='module')
def g():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    import __graft_entry__ as entry
    entry.build()
    return dict(np.load(GOLDEN, allow_pickle=False))


SHAPES = [(375, 500, 3), (500, 375, 3), (300, 300, 3), (7, 5), (9, 13, 1), (60, 40, 4), (150, 600, 3), (600, 150, 3), (320, 400, 3),
          (330, 450, 3), (200, 200, 1), (1, 1, 3), (2, 3), (480, 300, 3), (240, 384, 3), (123, 77, 3), (256, 256, 4), (333, 500, 3),
          (450, 300), (100, 700, 3)]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def images(g):
    """The golden's dataset, regenerated from its seed (make_eval_dataset_golden.make_images) and checked against its digests."""
    rng = np.random.default_rng(7)
    imgs = [rng.integers(0, 256, s, dtype=np.uint8) for s in SHAPES]
    assert [sha(im) for im in imgs] == list(g['image_sha'])
    return imgs


class DeviceStandIn:
    """The golden's stand-in model (make_eval_dataset_golden.py: standin_rows / standin_raw) as torch ops on the device; it
    records every batch it receives."""

    def __init__(self, special, training):
        self.special, self.training, self.batches = special, training, []

    def predict_device(self, x):
        import torch
        self.batches.append(x.cpu().numpy())
        X = x.to(torch.int64)
        B, H, W = X.shape[:3]
        s = X[:, :4, :4, :].sum(dim=(1, 2, 3))
        if self.training:
            y = torch.zeros((B, P, N_CLASSES + 13), dtype=torch.float32, device=x.device)
            for p in range(P):
                for c in range(1, N_CLASSES + 1):
                    y[:, p, c] = ((s + 31 * p + 7 * c) % 97).float() / 128.0
                y[:, p, 0] = 1.0 / 64
                for k in range(4):
                    y[:, p, -12 + k] = (((s + 5 * p + 3 * k) % 33) - 16).float() / 64.0
                ax, ay = (p % 4) * 0.25, (p // 4) * 0.5
                y[:, p, -8:-4] = torch.tensor([ax, ay, ax + 0.25, ay + 0.5], device=x.device)
                y[:, p, -4:] = torch.tensor([0.5, 0.5, 1.0, 1.0], device=x.device)
            return y
        t = X[:, H // 2, W // 2, :].sum(dim=-1)
        out = torch.zeros((B, K, 6), dtype=torch.float64, device=x.device)
        for j in range(K):
            if j in (3, 8):
                continue
            x0 = ((s + 37 * j) % W - 5).double() + (j % 4) * 0.25
            y0 = ((t + 11 * j) % H - 3).double() + (j % 2) * 0.5
            out[:, j, 0] = (1 + (s + j) % N_CLASSES).double()
            out[:, j, 1] = ((s * 7 + t + 13 * j) % 1021 + 1).double() / 1024.0
            out[:, j, 2] = x0; out[:, j, 3] = y0
            out[:, j, 4] = x0 + 8 + ((s + j) % 50).double(); out[:, j, 5] = y0 + 6 + ((t + j) % 40).double()
        sp = torch.from_numpy(self.special).to(x.device).expand(B, -1, -1)
        return torch.cat([out.float(), sp], dim=1)


def dataset(imgs, ids, filenames=None):
    return types.SimpleNamespace(images=None if filenames else list(imgs), filenames=filenames, image_ids=list(ids),
                                 labels=[np.zeros((0, 5)) for _ in imgs], eval_neutral=None)


def run_evaluator(g, name, dg=None):
    from ssd_keras_b200.eval_utils.average_precision_evaluator import Evaluator
    mode, mm, rc, (H, W), bs, seed = RUNS[name]
    model = DeviceStandIn(g['special_rows'], mm == 'training')
    ev = Evaluator(model, N_CLASSES, dg or dataset(images(g), [int(v) for v in g['ids']]), model_mode=mm)
    np.random.seed(seed)
    ev.predict_on_dataset(H, W, bs, data_generator_mode=mode, round_confidences=rc, verbose=False, **DECODE)
    return ev, model


def assert_results_equal_golden(g, name, res):
    mm = RUNS[name][1]
    dtype = np.float32 if mm == 'inference' else np.float64
    flat = [(c, p) for c in range(1, N_CLASSES + 1) for p in res[c]]
    assert all(type(p[1]) is dtype and all(type(v) is dtype for v in p[2:]) for _, p in flat)
    np.testing.assert_array_equal(np.array([c for c, _ in flat]), g[name + '/cls'])
    np.testing.assert_array_equal(np.array([p[0] for _, p in flat]), g[name + '/id'])
    vals = np.array([p[1:] for _, p in flat], dtype=dtype).reshape(-1, 5)
    np.testing.assert_array_equal(vals, g[name + '/vals'])
    assert np.array_equal(np.signbit(vals), np.signbit(g[name + '/vals']))


@pytest.mark.parametrize('name', list(RUNS))
def test_evaluator_equals_reference(g, name, tmp_path):
    ev, model = run_evaluator(g, name)
    X = np.concatenate(model.batches, axis=0)
    assert np.array_equal(X, np.round(X)) and X.min() >= 0 and X.max() <= 255
    assert [sha(x) for x in X.astype(np.uint8)] == list(g[name + '/batch_X_sha'])
    assert_results_equal_golden(g, name, ev.prediction_results)
    ev.write_predictions_to_txt(out_file_prefix=str(tmp_path / 'det_'), verbose=False)
    for c in range(1, N_CLASSES + 1):
        assert (tmp_path / ('det_%04d.txt' % c)).read_text() == str(g[name + '/txt_%d' % c])


@pytest.mark.parametrize('name', ['resize_inf', 'pad_inf_r3_wide'])
def test_evaluator_from_png_files(g, name, tmp_path):
    Image = pytest.importorskip('PIL.Image')
    files = []
    for i, im in enumerate(images(g)):
        a = im[:, :, 0] if im.ndim == 3 and im.shape[2] == 1 else im
        f = str(tmp_path / ('%02d.png' % i))
        Image.fromarray(a).save(f)
        files.append(f)
    from ssd_keras_b200.eval_utils.dataset_predict import load_image
    for f, im in zip(files, images(g)):
        np.testing.assert_array_equal(load_image(f).reshape(-1), im.reshape(-1))
    ev, _ = run_evaluator(g, name, dataset(images(g), [int(v) for v in g['ids']], filenames=files))
    assert_results_equal_golden(g, name, ev.prediction_results)


@pytest.mark.parametrize('name,hw,bs', [('coco_resize', (300, 300), 8), ('coco_resize_wide', (300, 480), 5)])
def test_predict_all_to_json_equals_reference(g, name, hw, bs, tmp_path):
    from ssd_keras_b200.eval_utils.coco_utils import predict_all_to_json
    model = DeviceStandIn(g['special_rows'], True)
    f = str(tmp_path / 'r.json')
    predict_all_to_json(f, model, hw[0], hw[1], {1: 3, 2: 17, 3: 90}, dataset(images(g), [int(v) for v in g['ids']]), bs,
                        confidence_thresh=0.3, pred_coords='corners')
    assert open(f).read() == str(g[name + '/json'])


def labels_for(n_images, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_images):
        k = int(rng.integers(0, 6))
        x0 = rng.integers(-10, 400, k); y0 = rng.integers(-10, 300, k)
        out.append(np.stack([rng.integers(1, N_CLASSES + 1, k), x0, y0, x0 + rng.integers(5, 200, k), y0 + rng.integers(5, 200, k)],
                            axis=1).reshape(-1, 5).astype(np.float64))
    return out


@pytest.mark.parametrize('name', ['pad_inf_r4', 'resize_train_wide'])
def test_device_and_list_matching_agree(g, name):
    """match_predictions on the device results and on the materialised lists: identical tp / fp and AP in both modes."""
    ev, _ = run_evaluator(g, name)
    ev.data_generator.labels = labels_for(len(g['ids']), 5)
    ev.get_num_gt_per_class(ret=False)

    def evaluate():
        tpfp = ev.match_predictions(verbose=False, ret=True)
        ev.compute_precision_recall(verbose=False)
        return tpfp, [ev.compute_average_precisions(mode=m, verbose=False, ret=True) for m in ('sample', 'integrate')]
    got, got_ap = evaluate()
    ev.prediction_results = ev.prediction_results   # assigning replaces the device results: the list path
    assert ev._detections is None
    want, want_ap = evaluate()
    assert sum(len(v) for v in want[0]) > 0
    for a, b in zip(got, want):
        for c in range(1, N_CLASSES + 1):
            np.testing.assert_array_equal(a[c], b[c])
    np.testing.assert_array_equal(np.array(got_ap), np.array(want_ap))


def test_same_size_dataset_keeps_list_path(g):
    """Images that all have the input size are predicted as before: no inverse transform, tuples of Python floats."""
    from ssd_keras_b200.eval_utils.average_precision_evaluator import Evaluator
    imgs = [np.random.default_rng(i).integers(0, 256, (300, 300, 3), dtype=np.uint8) for i in range(4)]

    class HostStandIn:
        def predict(self, x):
            import torch
            return DeviceStandIn(g['special_rows'], False).predict_device(torch.from_numpy(np.asarray(x, np.float32)).cuda()).cpu().numpy()
    ev = Evaluator(HostStandIn(), N_CLASSES, dataset(imgs, [1, 2, 3, 4]))
    ev.predict_on_dataset(300, 300, 2, verbose=False)
    assert ev._detections is None
    assert all(type(p[2]) is float for c in range(1, N_CLASSES + 1) for p in ev.prediction_results[c])


# -- the kernel alone ---------------------------------------------------------------------------------
def collect_device(rows, counts, inv, pad, f64, decimals, image_base=0, capacity=None, state=None):
    import ctypes as C
    import torch
    from ssd_keras_b200 import _ffi
    B, M = rows.shape[:2]
    cap = B * M if capacity is None else capacity
    if state is None:
        state = [torch.zeros((1,), dtype=torch.int32, device='cuda'), torch.full((max(cap, 1),), -7, dtype=torch.int32, device='cuda'),
                 torch.zeros((max(cap, 1),), dtype=torch.int32, device='cuda'), torch.zeros((max(cap, 1),), dtype=torch.float64, device='cuda'),
                 torch.zeros((max(cap, 1), 4), dtype=torch.float64, device='cuda')]
    cols = np.array([0, 1, 2, 3, 4, 5, 3, 5, 2, 4], np.int32)
    d_rows = torch.from_numpy(np.ascontiguousarray(rows, np.float32)).cuda()
    d_counts = None if counts is None else torch.from_numpy(np.asarray(counts, np.int32)).cuda()
    d_inv = torch.from_numpy(np.ascontiguousarray(inv, np.float64)).cuda()
    _ffi.check(_ffi.lib().ssdk_eval_collect(_ffi.context(), _ffi.dptr(d_rows), B, M, _ffi.dptr(d_counts), _ffi.dptr(d_inv),
                                            _ffi.np_ptr(cols, C.c_int), f64, pad, decimals, image_base, cap, _ffi.dptr(state[0]),
                                            *(_ffi.dptr(t) for t in state[1:]), _ffi.stream_ptr()))
    return state


def oracle_collect(rows, counts, shapes, patches, out_hw, dtype, decimals):
    per_image = []
    for b in range(rows.shape[0]):
        r = rows[b] if counts is None else rows[b, :counts[b]]
        canvas = shapes[b] if patches is None else patches[b][2:]
        per_image.append((r, canvas, out_hw, None if patches is None else patches[b][:2]))
    return evalops.collect([per_image], dtype, decimals)


@pytest.mark.parametrize('B,M,n_classes,f64,pad,decimals,with_counts', [
    (1, 200, 2, 0, 0, 0, False), (64, 200, 81, 0, 1, 4, False), (64, 400, 81, 1, 0, 3, True), (7, 400, 2, 1, 1, 4, True),
    (64, 100, 21, 0, 1, 3, False)])
def test_collect_kernel_equals_oracle(g, B, M, n_classes, f64, pad, decimals, with_counts):
    rng = np.random.default_rng(B * 1000 + M + n_classes)
    rows = np.zeros((B, M, 6), np.float32)
    for b in range(B):
        n = 0 if b % 5 == 1 else int(rng.integers(0, M + 1))       # some images with only padding rows
        rows[b, :n, 0] = rng.integers(0, n_classes, n)               # class 0 rows between real ones
        rows[b, :n, 1] = rng.uniform(0, 1, n)
        xy = rng.uniform(-20, 320, (n, 2)).astype(np.float32)
        rows[b, :n, 2:4] = np.round(xy * 4) / 4                     # quarter pixels: products on .5
        rows[b, :n, 4:6] = rows[b, :n, 2:4] + rng.uniform(0, 200, (n, 2))
        if n > 3:
            rows[b, 2, 4] = np.inf; rows[b, 3, 3] = -np.inf
    counts = rng.integers(0, M + 1, B) if with_counts else None
    shapes = [(int(rng.integers(1, 900)), int(rng.integers(1, 900))) for _ in range(B)]
    H, W = 300, 480
    patches = evalops.pad_draws(shapes, H, W, B) if pad else None
    inv = np.array([[(shapes[b] if not pad else patches[b][2:])[0] / H, (shapes[b] if not pad else patches[b][2:])[1] / W,
                     0 if not pad else patches[b][0], 0 if not pad else patches[b][1]] for b in range(B)], np.float64)
    st = collect_device(rows, counts, inv, pad, f64, decimals)
    dtype = np.float64 if f64 else np.float32
    img, cls, conf, box = oracle_collect(rows, counts, shapes, patches, (H, W), dtype, decimals)
    n = int(st[0].item())
    assert n == len(img)
    np.testing.assert_array_equal(st[1][:n].cpu().numpy(), img)
    np.testing.assert_array_equal(st[2][:n].cpu().numpy(), cls)
    got_conf = st[3][:n].cpu().numpy().astype(dtype)
    got_box = st[4][:n].cpu().numpy().astype(dtype)
    np.testing.assert_array_equal(got_conf, conf)
    np.testing.assert_array_equal(got_box, box)
    assert np.array_equal(np.signbit(got_box), np.signbit(box))


def test_collect_kernel_chains_batches_and_counts_overflow(g):
    rows = np.zeros((2, 5, 6), np.float32)
    rows[:, :, 0] = 1
    inv = np.tile([1.0, 1.0, 0.0, 0.0], (2, 1))
    st = collect_device(rows, None, inv, 0, 0, 0, capacity=12)
    st = collect_device(rows, [0, 1], inv, 0, 0, 0, image_base=2, capacity=12, state=st)
    assert int(st[0].item()) == 11
    np.testing.assert_array_equal(st[1][:11].cpu().numpy(), [0] * 5 + [1] * 5 + [3])
    st = collect_device(rows, None, inv, 0, 0, 0, image_base=4, capacity=12, state=st)
    assert int(st[0].item()) == 21                                    # counted past the capacity, nothing written there
    np.testing.assert_array_equal(st[1][11:12].cpu().numpy(), [4])


# -- a real SSD7 ---------------------------------------------------------------------------------------
class Recording:
    def __init__(self, model):
        self.model, self.outputs = model, []

    def predict_device(self, x):
        y = self.model.predict_device(x)
        self.outputs.append(y.cpu().numpy())
        return y


def ssd7(mode, H=300, W=480):
    from oracle import synth
    from oracle.model import ssd7_weight_shapes
    from ssd_keras_b200.models.keras_ssd7 import build_model
    pre = dict(subtract_mean=[127.5] * 3, divide_by_stddev=[127.5] * 3)
    model = build_model((H, W, 3), 5, mode=mode, scales=[0.08, 0.16, 0.32, 0.64, 0.96], normalize_coords=True,
                        **({'confidence_thresh': 0.2} if mode == 'inference' else {}), **pre)
    w = synth.synth_weights(1, ssd7_weight_shapes(5), bias_scale=0.05)
    for i in range(1, 8):
        c = w['conv%d/bias' % i].shape[0]
        w['bn%d/gamma' % i] = np.ones(c, np.float32); w['bn%d/beta' % i] = np.zeros(c, np.float32)
        w['bn%d/moving_mean' % i] = np.zeros(c, np.float32); w['bn%d/moving_variance' % i] = np.ones(c, np.float32)
    model.set_weights(w)
    return model


@pytest.mark.parametrize('mode,model_mode', [('resize', 'inference'), ('pad', 'inference'), ('pad', 'training')])
def test_real_ssd7_equals_oracle_on_its_own_decoder_output(g, mode, model_mode):
    import torch
    from ssd_keras_b200.eval_utils.average_precision_evaluator import Evaluator
    from ssd_keras_b200.ssd_encoder_decoder.ssd_output_decoder import decode_device, PER_CLASS
    rng = np.random.default_rng(3)
    imgs = [rng.integers(0, 256, (int(rng.integers(40, 500)), int(rng.integers(40, 500)), 3), dtype=np.uint8) for _ in range(40)]
    model = Recording(ssd7(model_mode))
    ev = Evaluator(model, 5, dataset(imgs, list(range(40))), model_mode=model_mode)
    np.random.seed(9)
    ev.predict_on_dataset(300, 480, 16, data_generator_mode=mode, round_confidences=4, verbose=False, decoding_confidence_thresh=0.2)
    res = ev.prediction_results
    shapes = [im.shape[:2] for im in imgs]
    patches = evalops.pad_draws(shapes, 300, 480, 9) if mode == 'pad' else None
    per_image = []
    for bi, y in enumerate(model.outputs):
        if model_mode == 'training':
            out, counts = decode_device(torch.from_numpy(y).cuda(), PER_CLASS, False, 0.2, 0.45, 200, 0, 'centroids', True, 300, 480, 'include')
            out, counts = out.cpu().numpy(), counts.cpu().numpy()
            y = [out[k, :counts[k]] for k in range(out.shape[0])]
        for k, r in enumerate(y):
            i = bi * 16 + k
            per_image.append((r, shapes[i] if patches is None else patches[i][2:], (300, 480), None if patches is None else patches[i][:2]))
    dtype = np.float32 if model_mode == 'inference' else np.float64
    want = evalops.per_class(*evalops.collect([per_image], dtype, 4), list(range(40)), 5)
    assert sum(len(v) for v in want) > 0
    for c in range(1, 6):
        assert len(res[c]) == len(want[c])
        for a, b in zip(res[c], want[c]):
            assert a[0] == b[0] and type(a[1]) is dtype
            np.testing.assert_array_equal(np.array(a[1:], dtype), np.array(b[1:], dtype))
