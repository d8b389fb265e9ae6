"""CPU half of the decoder path tests: the Python restatement of csrc/decode.cu's launch decisions (tests/decode_cases.py)
must find every path of the decoder reached by the GPU case table, the exact reference must agree with the reference's own
outputs where they are pinned, and the oracle's semantics at the confidence threshold and for NaN scores must be the
reference's (tests/golden/ref_decode_edges_golden.npz, written by tests/golden/make_decode_edges_golden.py)."""
import os
import re

import numpy as np
import pytest

import decode_cases as dc
from oracle import decoder as odec

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def test_kernel_constants_are_read_from_the_source():
    assert (dc.NMS_CAP, dc.KEPT_SM, dc.MASK_N, dc.TOP_CAP) == (2048, 512, 256, 16384)
    with open(dc.DECODE_CU) as f:
        src = f.read()
    # the stage-1 band rule restated by decode_cases.stage1_band
    assert re.search(r'int want = 4 \* top_k / \(S > 0 \? S : 1\), b = 256;\s*while \(b < want && b < kNmsCap\) b <<= 1;', src)
    assert 'bool two_stage = top_k > 0 && n > band1 && band1 < kNmsCap;' in src
    assert 'if (st.first && cnt <= kMaskN && prm.cap >= 1)' in src
    assert [dc.stage1_band(20, 200), dc.stage1_band(1, 200), dc.stage1_band(2, 3000), dc.stage1_band(20, 16384)] == [256, 1024, 2048, 2048]


@pytest.fixture(scope='module')
def reached():
    out = {}
    for c in dc.CASES:
        _, r, _ = dc.paths(c, dc.inputs(c['name']))
        out[c['name']] = r
    return out


@pytest.mark.parametrize('path', sorted(dc.REQUIRED))
def test_case_table_reaches_path(reached, path):
    """Each path of the decoder, and the case that reaches it."""
    assert path in reached[dc.REQUIRED[path]], (path, dc.REQUIRED[path], sorted(reached[dc.REQUIRED[path]]))


def test_rescan_mixed_batch_model():
    c = dc.BY_NAME['rescan_mixed']
    L, r, redo = dc.paths(c, dc.inputs('rescan_mixed'))
    assert L['two_stage'] and L['band1'] == dc.MASK_N and L['cap'] == 200
    assert redo == [True, False, True]


def test_exp_cr_is_float64_exp_rounded_once():
    x = np.random.default_rng(0).uniform(-20, 20, 100000).astype(np.float32)
    got = odec.exp_cr(x)
    assert got.dtype == np.float32
    np.testing.assert_array_equal(got, np.exp(x.astype(np.float64)).astype(np.float32))
    assert np.isinf(odec.exp_cr(np.float32(100.0))) and odec.exp_cr(np.float32(-200.0)) == 0


def _survivors(rows):
    r = np.asarray(rows, np.float64).reshape(-1, 6)
    return r[np.lexsort((r[:, 0], -r[:, 1]))][:, :2]


def test_fuzz_survivors_do_not_depend_on_exp():
    """tests/test_gpu_decode_paths.py holds the kernels to the reference's fuzz outputs with classes, confidences and counts
    exact: on every seed, the survivors must not depend on which float32 exp decodes the boxes."""
    import test_oracle_vs_reference_fuzz_cpu as fz
    import test_oracle_vs_reference_tf_fuzz_cpu as tfz
    same = []
    for seed in range(25):
        y, kw = fz._decoder_case(seed)
        ok = True
        for fn in (odec.decode_detections, odec.decode_detections_fast):
            ok &= all(np.array_equal(_survivors(a), _survivors(b)) for a, b in zip(fn(y, **kw), fn(y, exp=odec.exp_cr, **kw)))
        if ok:
            same.append(seed)
    assert same == list(range(25))
    same = []
    for seed in range(20):
        y, kw = tfz._decode_case(seed)
        args = (y, kw['confidence_thresh'], kw['iou_threshold'], kw['top_k'], kw['nms_max_output_size'], kw['normalize_coords'],
                120, 160)
        if all(np.array_equal(fn(*args)[..., :2], fn(*args, exp=odec.exp_cr)[..., :2])
               for fn in (odec.decode_layer, odec.decode_layer_fast)):
            same.append(seed)
    assert same == list(range(20))


@pytest.mark.parametrize('name', [c['name'] for c in dc.CASES if c['api'] == 'numpy' and c['top_k'] != 'all'])
def test_numpy_topk_choice_is_one_of_the_reference_sets(name):
    """The exact reference takes the kernel's documented top-k choice (confidence descending, ties class-major) from the full
    survivor list; that must be a valid outcome of the reference's unordered argpartition: the same confidences."""
    c = dc.BY_NAME[name]
    y = dc.inputs(name)
    out, _, counts = dc.reference(c, y)
    fn = odec.decode_detections_fast if c['fast'] else odec.decode_detections
    with np.errstate(all='ignore'):
        ref = fn(y, c['conf'], c['iou'], c['top_k'], c['coords'], c['norm'], c['H'], c['W'], c['border'], exp=odec.exp_cr)
    for b, r in enumerate(ref):
        r = np.asarray(r, np.float64).reshape(-1, 6)
        np.testing.assert_array_equal(np.sort(out[b, :counts[b], 1]), np.sort(r[:, 1].astype(np.float32)))


@pytest.mark.parametrize('coords', ['centroids', 'corners'])
def test_nms_off_keeps_nonfinite_boxes(coords):
    """decode_detections_fast with iou_threshold 0 runs no NMS: rows with NaN or infinite boxes stay, and so do the rows an
    NMS with a threshold no finite IoU exceeds would drop (a NaN IoU never passes `<=`)."""
    name = 'nonfinite_iou0_numpy_%s_fast' % coords
    c = dc.BY_NAME[name]
    y = dc.inputs(name)
    out, _, counts = dc.reference(c, y)
    rows = out[0, :counts[0]]
    assert (~np.isfinite(rows[:, 2:])).any(axis=1).any()
    with np.errstate(all='ignore'):
        nms_inf = odec.decode_detections_fast(y, c['conf'], np.inf, 'all', coords, False, None, None, exp=odec.exp_cr)[0]
    assert nms_inf.shape[0] < counts[0]


def test_ssd300_anchors_are_the_encoders():
    from oracle.encoder import OracleEncoder
    from conftest import golden_configs
    np.testing.assert_array_equal(dc.ssd300_anchors(), OracleEncoder(**golden_configs()['ssd300']).anchors.astype(np.float32))


def test_return_index_leaves_the_rows_alone():
    y = dc.inputs('small_topk_class_major')
    for fn in (odec.decode_detections, odec.decode_detections_fast):
        for coords in ('centroids', 'corners'):
            plain = fn(y, 0.05, 0.45, 200, coords, True, 300, 300)
            rows, idx = fn(y, 0.05, 0.45, 200, coords, True, 300, 300, return_index=True)
            for p, r, i in zip(plain, rows, idx):
                np.testing.assert_array_equal(p, r)
                assert p.dtype == r.dtype and len(i) == np.asarray(r).reshape(-1, 6).shape[0]


# ------------------------------------------------------------------------------------------------
# thresholds and NaN scores: the oracle against the reference's own outputs
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def edges():
    with np.load(os.path.join(GOLD, 'ref_decode_edges_golden.npz')) as z:
        return {k: z[k] for k in z.files}


def _edge_inputs():
    import sys
    sys.path.insert(0, GOLD)
    from make_decode_edges_golden import edge_inputs
    return edge_inputs()


@pytest.mark.parametrize('key', [k for k, _, _ in _edge_inputs()])
def test_oracle_threshold_and_nan_semantics_vs_reference(edges, key):
    (y, kw), = [(y, kw) for k, y, kw in _edge_inputs() if k == key]
    for name, fn in (('per_class', odec.decode_detections), ('fast', odec.decode_detections_fast)):
        with np.errstate(all='ignore'):
            got = np.asarray(fn(y, **kw)[0], np.float64).reshape(-1, 6)
        np.testing.assert_array_equal(got, edges['%s/%s' % (key, name)])


def test_reference_threshold_dtype_per_coords(edges):
    """What the fixture pins: corners compares float32 scores in float32, centroids and minmax in float64, and the first NaN of
    a class vector wins the arg-max in the fast decoder."""
    t3 = np.float32(0.3)
    assert (edges['thr0.3/centroids/per_class'][:, 1] == t3).sum() == 4
    assert (edges['thr0.3/corners/per_class'][:, 1] == t3).sum() == 0
    t1 = np.float32(0.01)
    assert (edges['thr0.01/corners/fast'][:, 1] == t1).sum() == 4
    assert (edges['thr0.01/centroids/fast'][:, 1] == t1).sum() == 0
    for coords in ('centroids', 'corners', 'minmax'):
        np.testing.assert_array_equal(edges['nan/%s/fast' % coords][:, :2], [[1.0, np.float32(0.8)]])
