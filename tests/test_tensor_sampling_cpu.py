"""``misc_utils.tensor_sampling_utils.sample_tensors`` against the REAL reference: bit-identical arrays and the same global
``np.random`` state afterwards, under the same seed, for every case of tests/sampling_cases.py (the reference's results are
in tests/golden/ref_sampling_golden.npz, written by tests/golden/make_sampling_golden.py); the reference's exception type and
message for every error case; and, where the reference tree is present, a seeded fuzz over random shapes and instructions."""
import importlib.util
import os

import numpy as np
import pytest

from sampling_cases import CASES, ERRORS, SEEDS, sha, tensors
from ssd_keras_b200.misc_utils.tensor_sampling_utils import classifier_indices, sample_tensors

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get('SSD_REFERENCE_ROOT', '/root/reference')


@pytest.fixture(scope='module')
def g():
    with np.load(os.path.join(HERE, 'golden', 'ref_sampling_golden.npz')) as z:
        return {k: z[k] for k in z.files}


def _state_equals(g, prefix):
    _, keys, pos, has_gauss, cached = np.random.get_state()
    assert sha(keys) == str(g[prefix + '/state_keys_sha']), prefix
    assert (pos, has_gauss) == (int(g[prefix + '/state_pos']), int(g[prefix + '/state_has_gauss'])), prefix
    assert cached == float(g[prefix + '/state_cached_gaussian']), prefix


@pytest.mark.parametrize('name', list(CASES))
def test_outputs_and_generator_state_equal_reference(g, name):
    seed, shapes, dtype, inst, kw = CASES[name]
    for s in SEEDS:
        w = tensors(seed, shapes, np.dtype(dtype))
        np.random.seed(s)
        got = sample_tensors(w, inst, **kw)
        p = 'case/%s/%d' % (name, s)
        assert len(got) == int(g[p + '/n'])
        for i, r in enumerate(got):
            if p + '/%d/sha' % i in g:
                assert r.dtype.str == str(g[p + '/%d/dtype' % i]) and r.shape == tuple(g[p + '/%d/shape' % i]), (p, i)
                assert sha(r) == str(g[p + '/%d/sha' % i]), (p, i)
            else:
                ref = g[p + '/%d' % i]
                assert r.dtype == ref.dtype and r.shape == ref.shape, (p, i, r.dtype, ref.dtype, r.shape, ref.shape)
                assert r.tobytes() == ref.tobytes(), (p, i)
        _state_equals(g, p)


@pytest.mark.parametrize('name', list(ERRORS))
def test_errors_equal_reference(g, name):
    seed, shapes, dtype, inst, kw = ERRORS[name]
    w = tensors(seed, shapes, np.dtype(dtype))
    np.random.seed(0)
    with pytest.raises(Exception) as e:
        sample_tensors(w, inst, **kw)
    assert type(e.value).__name__ == str(g['error/%s/type' % name])
    assert str(e.value) == str(g['error/%s/msg' % name])
    _state_equals(g, 'error/' + name)


def test_dtypes_follow_the_branch():
    """Sub-sampling keeps the dtype and copies; up-sampling makes float64 whatever came in."""
    for dt in (np.float16, np.float32, np.float64):
        k, b = tensors(3, [(3, 3, 4, 10), (10,)], dt)
        np.random.seed(0)
        sk, sb = sample_tensors([k, b], [3, 3, 4, [0, 2, 5]], axes=[[3]])
        assert sk.dtype == dt and sb.dtype == dt
        assert not np.shares_memory(sk, k) and not np.shares_memory(sb, b)
        uk, ub = sample_tensors([k, b], [3, 3, 4, 12], axes=[[3]], init=['gaussian', 'zeros'])
        assert uk.dtype == np.float64 and ub.dtype == np.float64


def test_upsampling_keeps_every_element_and_index_zero():
    k, b = tensors(4, [(1, 1, 2, 5), (5,)])
    np.random.seed(3)
    uk, ub = sample_tensors([k, b], [1, 1, 2, 9], axes=[[3]], init=['zeros', 'zeros'])
    kept = np.flatnonzero(ub)
    assert kept[0] == 0 and len(kept) == 5
    np.testing.assert_array_equal(ub[kept], b.astype(np.float64))
    np.testing.assert_array_equal(uk[..., kept], k.astype(np.float64))


def test_classifier_indices_as_the_tutorial_computes_them():
    idx = classifier_indices(324, 81, [0, 3, 8, 1, 2, 10, 4, 6, 12])
    assert idx[:9] == [0, 3, 8, 1, 2, 10, 4, 6, 12] and idx[9:12] == [81, 84, 89] and len(idx) == 36
    assert classifier_indices(486, 81, 9) == 54 and type(classifier_indices(486, 81, 9)) is int
    with pytest.raises(ValueError, match='`classes_of_interest` must be either an integer or a list/tuple.'):
        classifier_indices(324, 81, np.int64(9))


def _reference_sample_tensors():
    path = os.path.join(REF_ROOT, 'misc_utils', 'tensor_sampling_utils.py')
    if not os.path.isfile(path):
        pytest.skip('the reference tree is not present')
    spec = importlib.util.spec_from_file_location('reference_tensor_sampling_utils', path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.sample_tensors


def _random_call(rng):
    """A random sample_tensors call: 1-4 axes, each kept / sub-sampled (indices or a count) / up-sampled, with 1-3 tensors."""
    nd = int(rng.integers(1, 5))
    shape = [int(v) for v in rng.integers(1, 9, nd)]
    inst = []
    for n in shape:
        kind = int(rng.integers(0, 4))
        if kind == 0:
            inst.append(n)
        elif kind == 1 and n > 1:
            inst.append(int(rng.integers(1, n)))
        elif kind == 2:
            inst.append([int(v) for v in rng.integers(-n, n, int(rng.integers(1, 2 * n + 1)))])
        else:
            inst.append(n + int(rng.integers(1, 6)))
    dtype = [np.float16, np.float32, np.float64][int(rng.integers(0, 3))]
    ws = [rng.standard_normal(shape).astype(dtype)]
    axes = []
    for _ in range(int(rng.integers(0, 3))):
        ax = sorted(rng.choice(nd, int(rng.integers(1, nd + 1)), replace=False).tolist())
        axes.append(ax)
        ws.append(rng.standard_normal([shape[a] for a in ax]).astype(dtype))
    init = None if rng.integers(0, 3) == 0 else [['gaussian', 'zeros'][int(rng.integers(0, 2))] for _ in ws]
    return ws, inst, dict(axes=axes or None, init=init, mean=float(rng.uniform(-1, 1)), stddev=float(rng.uniform(0.001, 1)))


def test_fuzz_against_reference():
    ref = _reference_sample_tensors()
    rng = np.random.default_rng(2024)
    for t in range(60):
        ws, inst, kw = _random_call(rng)
        results = []
        for fn in (ref, sample_tensors):
            np.random.seed(t)
            out = fn([w.copy() for w in ws], inst, **kw)
            results.append((out, np.random.get_state()))
        (a, sa), (b, sb) = results
        assert len(a) == len(b), t
        for x, y in zip(a, b):
            assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), (t, inst)
        assert sa[2:] == sb[2:] and np.array_equal(sa[1], sb[1]), t
