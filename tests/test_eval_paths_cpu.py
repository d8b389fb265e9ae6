"""CPU half of the evaluator path tests: oracle/evalops.py must equal the reference's own Evaluator bit for bit on every edge
case of tests/eval_cases.py (tests/golden/ref_eval_edges_golden.npz, written by tests/golden/make_eval_edges_golden.py), the
case table must reach every path of eval_match_kernel / eval_cumsum_kernel the GPU tests rely on, and each subtly wrong
variant of the oracle (one step of the arithmetic, the arg-max or the scan changed) must disagree with the goldens, which is
what lets the same cases catch a subtly wrong kernel."""
import os
import sys

import numpy as np
import pytest

import eval_cases as xc
from oracle import evalops as eo

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
G = np.load(os.path.join(GOLD, 'ref_eval_edges_golden.npz'))


def _digest(c):
    sys.path.insert(0, GOLD)
    try:
        from make_eval_edges_golden import digest
    finally:
        sys.path.remove(GOLD)
    return digest(c)


def test_kernel_constants_are_read_from_the_source():
    assert (xc.LANES, xc.WARPS_PER_CTA, xc.CHUNK) == (32, 8, 1024)
    with open(xc.EVALUATE_CU) as f:
        src = f.read()
    # the path model and the oracle's rules follow these lines of the source
    assert 'if (r[0] != (double)cls) continue;' in src
    assert 'double best = -INFINITY; int best_g = INT_MAX;' in src
    assert 'if (is_nan || best_g == INT_MAX || (double)v > best)' in src
    assert 'const double thr = (double)(T)a.thr;' in src
    assert 'if (a.gt_f32[img]) match_segment<float>' in src
    # the launch shape the file's header documents is the one it launches
    assert 'eval_match_kernel<<<ceil_div(n_seg, %d), %d, 0, stream>>>' % (xc.WARPS_PER_CTA, 32 * xc.WARPS_PER_CTA) in src


@pytest.mark.parametrize('name', xc.EDGES)
def test_oracle_equals_reference(name):
    c = xc.edge(name)
    assert str(G[name + '/digest']) == _digest(c), 'the case generator changed; regenerate the golden file'
    xc.assert_same(xc.oracle(c), xc.golden(G, name, c['n_classes']), c['n_classes'], name)


_CACHE = {}


def _reached(name):
    if name not in _CACHE:
        c = xc.edge(name) if name in xc.EDGE_BUILDERS and name not in xc.CASE_BUILDERS else xc.build(name)
        _CACHE[name] = xc.paths(c)[0]
    return _CACHE[name]


@pytest.mark.parametrize('path', sorted(xc.REQUIRED))
def test_case_table_reaches_path(path):
    """Each path of the two kernels, and the case that reaches it."""
    name = xc.REQUIRED[path]
    assert path in _reached(name), (path, name, sorted(_reached(name)))


def test_edge_cases_reach_the_threshold_and_lane_paths():
    """The golden cases themselves (which the GPU suite also runs) reach what the issue of this arithmetic is about."""
    reached = {}
    for name in ('near_i64_include', 'near_f32_include', 'near_f32_half_045', 'lanes_nan_tie_half', 'below_minus_one', 'misc'):
        reached[name] = xc.paths(xc.edge(name))
    assert reached['near_i64_include'][1]['f64'] > 0 and reached['near_f32_include'][1]['f32'] > 0
    assert 'on_float32_threshold' in reached['near_f32_half_045'][0]
    assert {'nan_across_lanes', 'tie_across_lanes', 'lane_passes_gt_1'} <= reached['lanes_nan_tie_half'][0]
    assert 'overlap_below_minus_one' in reached['below_minus_one'][0]
    assert {'empty_class', 'both_types_one_call'} <= reached['misc'][0]


def _f64_pred_area(b, d):
    b = b.astype(np.float64)
    return (b[:, 2] - b[:, 0] + d) * (b[:, 3] - b[:, 1] + d)


MUTANTS = {
    'float64_pred_area': ('pred_area', _f64_pred_area),
    'float64_threshold': ('below', lambda ov, thr: bool(float(ov) < thr)),
    'last_index_tie': ('best_index', lambda ov: len(ov) - 1 - int(np.argmax(ov[::-1]))),
    'nan_ignored': ('best_index', lambda ov: int(np.argmax(np.where(np.isnan(ov), -np.inf, ov)))),
    'truncated_class': ('class_mask', lambda classes, c: classes.astype(np.int64) == c),
    'exclusive_cumsum': ('cumulative', lambda f: np.cumsum(f) - f),
}


@pytest.mark.parametrize('mutant', sorted(MUTANTS))
def test_mutant_disagrees_with_reference(monkeypatch, mutant):
    """A kernel that made this one mistake would fail at least one golden case on at least one prediction."""
    attr, fn = MUTANTS[mutant]
    monkeypatch.setattr(eo, attr, fn)
    for name in xc.EDGES:
        c = xc.edge(name)
        try:
            xc.assert_same(xc.oracle(c), xc.golden(G, name, c['n_classes']), c['n_classes'], name)
        except AssertionError:
            return
    pytest.fail('the %s mutant agrees with every golden case' % mutant)
