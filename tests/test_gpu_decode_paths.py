"""Every path of the decoder (csrc/decode.cu, ``ssdk_decode``) against an exact reference, bit for bit.

Each case of tests/decode_cases.py runs with the default two-stage NMS and with ``SSDK_NMS_TWO_STAGE=0`` (always the full
multi-band scan).  The reference is the oracle with the kernel's correctly rounded float32 ``exp``, so class ids, confidences,
prior indices, counts, zero padding and boxes must all be identical; the NumPy API writes float32 rows, so its float64 boxes are
compared after one rounding to float32.  tests/test_decode_paths_cpu.py checks that the cases reach every path."""
import numpy as np
import pytest

import decode_cases as dc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


def run_kernel(c, y):
    import torch
    from ssd_keras_b200.ssd_encoder_decoder.ssd_output_decoder import FAST, PER_CLASS, decode_device
    out, counts, index = decode_device(torch.from_numpy(np.ascontiguousarray(y)).cuda(), FAST if c['fast'] else PER_CLASS,
                                       c['api'] == 'layer', c['conf'], c['iou'], c['top_k'], c['cap'], c['coords'], c['norm'],
                                       c['H'], c['W'], c['border'], return_index=True)
    return out.cpu().numpy(), index.cpu().numpy().astype(np.int64), counts.cpu().numpy().astype(np.int64)


def assert_exact(got, want):
    out, idx, cnt = got
    r_out, r_idx, r_cnt = want
    assert out.shape == r_out.shape, (out.shape, r_out.shape)
    np.testing.assert_array_equal(cnt, r_cnt)
    np.testing.assert_array_equal(idx, r_idx)                      # prior indices, -1 on padding rows
    np.testing.assert_array_equal(out[..., :2], r_out[..., :2])    # class ids and confidences, row by row
    np.testing.assert_array_equal(out[..., 2:], r_out[..., 2:])    # boxes (NaN == NaN), zero padding


@pytest.mark.parametrize('two_stage', ['default', '0'])
@pytest.mark.parametrize('name', [c['name'] for c in dc.CASES])
def test_decode_path_exact(name, two_stage, monkeypatch):
    if two_stage == '0':
        monkeypatch.setenv('SSDK_NMS_TWO_STAGE', '0')
    else:
        monkeypatch.delenv('SSDK_NMS_TWO_STAGE', raising=False)
    c = dc.BY_NAME[name]
    y = dc.inputs(name)
    assert_exact(run_kernel(c, y), dc.reference(c, y))


def test_rescan_is_forced_in_a_mixed_batch(monkeypatch):
    """rescan_mixed: stage 1 must re-scan images 0 and 2 and not image 1; the result equals the full scan bit for bit."""
    c = dc.BY_NAME['rescan_mixed']
    y = dc.inputs('rescan_mixed')
    L, reached, redo = dc.paths(c, y)
    assert L['two_stage'] and redo == [True, False, True]
    monkeypatch.delenv('SSDK_NMS_TWO_STAGE', raising=False)
    two = run_kernel(c, y)
    monkeypatch.setenv('SSDK_NMS_TWO_STAGE', '0')
    one = run_kernel(c, y)
    for a, b in zip(two, one):
        np.testing.assert_array_equal(a, b)
    # without the re-scan, image 0 would report only stage 1's single class-1 survivor among its 1100 coincident boxes
    want = dc.reference(c, y)
    assert (want[0][0, :, 0] == 1).sum() > 1


# ------------------------------------------------------------------------------------------------
# the reference's own fuzz outputs, straight through the kernels
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def fuzz():
    import os
    with np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_fuzz_golden.npz')) as z:
        return {k: z[k] for k in z.files}


def _box_tol(want):
    """NumPy's float32 exp differs from the kernel's by up to 2 ulp, which moves a corner by up to 1 ulp of w / h; the roundings
    of cx - w / 2 and of the scaling to pixels then move it by up to an ulp of the coordinate each, at the scale before and after
    the scaling.  The bound is 2 ulp of the width / height plus 2 ulp of the coordinate -- looser than 2 ulp of w / h alone,
    which the corner's own roundings exceed.  The largest difference on these fixtures is 0.89 of it.  Classes, confidences,
    counts and row order are exact, and the kernels' boxes are held bit for bit to the oracle with the kernel's exp."""
    w = np.abs(want[..., [2, 3, 2, 3]] - want[..., [0, 1, 0, 1]]).astype(np.float32)
    return 2 * (np.spacing(w) + np.spacing(np.abs(want).astype(np.float32)))


@pytest.mark.parametrize('seed', range(25))
def test_numpy_decoders_vs_reference_fuzz(fuzz, seed):
    import test_oracle_vs_reference_fuzz_cpu as fz
    y, kw = fz._decoder_case(seed)
    want = [fuzz['decoders/%d/%d' % (seed, i)] for i in range(int(fuzz['decoders/%d/n' % seed]))]
    B = y.shape[0]
    for k, fast in enumerate((False, True)):
        c = dc.case('fuzz', 'numpy', fast, None, kw['confidence_thresh'], kw['iou_threshold'], kw['top_k'],
                    norm=kw['normalize_coords'], H=kw['img_height'], W=kw['img_width'], border=kw['border_pixels'])
        got = run_kernel(c, y.astype(np.float32))
        assert_exact(got, dc.reference(c, y.astype(np.float32)))
        for b in range(B):
            ref = want[k * B + b]
            n = int(got[2][b])
            rows = got[0][b, :n].astype(np.float64)
            assert n == ref.shape[0]
            # the reference's top-k set is unordered: both sides sorted by (confidence desc, class, reference row order)
            ka = np.lexsort((rows[:, 0], -rows[:, 1])); kb = np.lexsort((ref[:, 0], -ref[:, 1]))
            a, r = rows[ka], ref[kb]
            np.testing.assert_array_equal(a[:, :2], r[:, :2])
            assert (np.abs(a[:, 2:] - r[:, 2:]) <= _box_tol(r[:, 2:])).all()


@pytest.mark.parametrize('seed', range(20))
def test_decode_layers_vs_reference_fuzz(fuzz, seed):
    import test_oracle_vs_reference_tf_fuzz_cpu as tfz
    y, kw = tfz._decode_case(seed)
    y = y.astype(np.float32)
    for i, fast in enumerate((False, True)):
        c = dc.case('fuzz', 'layer', fast, None, kw['confidence_thresh'], kw['iou_threshold'], kw['top_k'],
                    cap=kw['nms_max_output_size'], norm=kw['normalize_coords'], H=kw['img_height'], W=kw['img_width'])
        got = run_kernel(c, y)
        assert_exact(got, dc.reference(c, y))
        want = fuzz['decode_layers/%d/%d' % (seed, i)]
        assert got[0].shape == want.shape
        np.testing.assert_array_equal(got[0][..., :2], want[..., :2])
        assert (np.abs(got[0][..., 2:] - want[..., 2:]) <= _box_tol(want[..., 2:])).all()
