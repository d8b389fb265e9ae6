"""GPU half of the evaluator path tests: Evaluator.match_predictions (eval_match_kernel, eval_cumsum_kernel) against
oracle/evalops.py, bit for bit, on the large generated cases of tests/eval_cases.py: 100+ boxes per image (several lane
passes, ties across lanes), 3000 images x 20 classes (thousands of CTAs), classes of 1023 / 1024 / 1025 / 5000 predictions
and an empty one (1 to 5 cumsum chunks), float32 and float64 images in one call, 16000 predictions bisected onto the
threshold in both arithmetic types, the one-prediction regression case of the float32 predicted area, and overlaps below -1
with a threshold below them (the arg-max must still name a box)."""
import numpy as np
import pytest

import eval_cases as xc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()


@pytest.mark.parametrize('name', xc.CASES)
def test_eval_path_exact(name):
    c = xc.build(name)
    xc.assert_same(xc.device(c), xc.oracle(c), c['n_classes'], name)


def test_regression_float32_predicted_area():
    """IoU 0.5000000034554928 with the float32 predicted area the reference computes: a true positive."""
    tp, fp = xc.device(xc.regression_example())['tp'][1], xc.device(xc.regression_example())['fp'][1]
    assert tp.tolist() == [1] and fp.tolist() == [0]


def test_repeated_calls_and_empty_inputs():
    """The matched flags start from zero on every call; a call without predictions or without labels returns empty arrays."""
    c = xc.build('crowded')
    first, second = xc.device(c), xc.device(c)
    xc.assert_same(second, first, c['n_classes'], 'second call')
    e = dict(c, preds=[[] for _ in range(c['n_classes'] + 1)])
    got = xc.device(e)
    assert all(len(got['tp'][k]) == 0 and len(got['ctp'][k]) == 0 for k in range(1, c['n_classes'] + 1))
    z = dict(c, labels=[np.zeros((0, 5), np.float32) for _ in c['labels']])
    got, want = xc.device(z), xc.oracle(z)
    xc.assert_same(got, want, c['n_classes'], 'no labels')
    assert all(np.all(want['fp'][k] == 1) for k in range(1, c['n_classes'] + 1))
