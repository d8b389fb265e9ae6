"""The box half of the op lists on the host: oracle/boxops.py bit for bit against the REAL reference's classes on the edge cases
of tests/golden/make_assembly_edges_golden.py (NaN equal to any NaN, -0.0 apart from +0.0), oracle mutants that the golden must
catch, the case table of tests/test_gpu_assembly_paths.py against the model of csrc/batch.cu's decisions (tests/
assembly_cases.py), and the live reference classes on the golden's inputs where the reference checkout is present."""
import importlib.util
import inspect
import os
import sys

import numpy as np
import pytest

import assembly_cases as ac
from oracle import boxops as bo

G = np.load(ac.GOLDEN)
N = int(G['n'])
REF_ROOT = os.environ.get('SSD_REFERENCE_ROOT', '/root/reference')


def _ops(k):
    return [tuple(r) for r in G['ops%d' % k].tolist()]


def same_bits(a, b):
    """Equal float64 bit patterns, any NaN equal to any NaN."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool((na == nb).all() and (a[~na].view(np.uint64) == b[~nb].view(np.uint64)).all())


def _disagreements(apply):
    return [k for k in range(N) if not same_bits(apply(G['lin%d' % k], _ops(k)), G['lout%d' % k])]


def test_oracle_matches_golden_bitwise():
    bad = _disagreements(bo.apply_box_ops)
    assert not bad, [(k, str(G['kind%d' % k])) for k in bad]


def test_golden_covers_the_edges():
    kinds = {str(G['kind%d' % k]) for k in range(N)}
    assert {'resize_tie', 'center', 'area_lower0', 'area_lower', 'area_upper', 'iou_bound', 'min_area', 'negzero', 'nonfinite', 'empty',
            'drop_all', 'class_ids'} <= kinds
    seen = set()
    for k in range(N):
        lin, lout, ops = G['lin%d' % k], G['lout%d' % k], G['ops%d' % k]
        codes = {int(o[0]) for o in ops}
        for j in range(1, 5):
            for name, m in (('nan', np.isnan), ('+inf', np.isposinf), ('-inf', np.isneginf)):
                if m(lin[:, j]).any():
                    seen |= {(name, j, c) for c in codes}
        if (np.signbit(lout[:, 1:]) & (lout[:, 1:] == 0)).any():
            seen.add('-0 out')
        if ac.SCALE in codes or ac.ROTATE in codes:
            pre = np.isnan(lin).any()
            assert not pre, 'NaN through Scale / Rotate is platform-defined'
        if lin.shape[0] == 0:
            seen.add('empty')
        elif lout.shape[0] == 0:
            seen.add('all dropped')
        if (lin[:, 0] != np.round(lin[:, 0])).any() and (lin[:, 0] < 0).any():
            seen.add('class ids')
        for o in ops:
            if int(o[0]) == ac.OVERLAP:
                seen.add(('overlap', int(o[1]) & 3, (int(o[1]) >> 2) & 3))
    for j in range(1, 5):
        for name in ('nan', '+inf', '-inf'):
            for c in (ac.CROP_PAD, ac.FLIP_H, ac.FLIP_V, ac.RESIZE, ac.FILTER, ac.TRANSLATE, ac.OVERLAP, ac.CLIP):
                assert (name, j, c) in seen, (name, j, c)
    for need in ('-0 out', 'empty', 'all dropped', 'class ids'):
        assert need in seen, need
    assert ('overlap', 0, 0) in seen                               # border_pixels plays no part in 'center_point'
    for c in (1, 2):
        for b in range(3):
            assert ('overlap', c, b) in seen, (c, b)


def _mutant(replacements, extra=None):
    """apply_box_ops with text replaced in oracle/boxops.py's functions (each replacement must hit)."""
    ns = dict(bo.__dict__)
    ns.update(extra or {})
    for fn in (bo._corners, bo.overlap_mask, bo.apply_box_ops):
        src = inspect.getsource(fn)
        for old, new in replacements:
            src = src.replace(old, new)
        exec(compile(src, bo.__file__, 'exec'), ns)
    for old, _ in replacements:
        assert any(old in inspect.getsource(fn) for fn in (bo._corners, bo.overlap_mask, bo.apply_box_ops)), old
    return ns['apply_box_ops']


def _iou_with_border(w, h, lab, d):
    iw = np.maximum(0, np.minimum(w, lab[:, 3]) - np.maximum(0, lab[:, 1]) + d)
    ih = np.maximum(0, np.minimum(h, lab[:, 4]) - np.maximum(0, lab[:, 2]) + d)
    inter = iw * ih
    return inter / ((w + d) * (h + d) + (lab[:, 3] - lab[:, 1] + d) * (lab[:, 4] - lab[:, 2] + d) - inter)


@pytest.mark.parametrize('name,replacements,extra,kind', [
    ('clip drops NaN', [('np.clip(', '_fclip(')], {'_fclip': lambda x, lo, hi: np.fmin(np.fmax(x, lo), hi)}, 'nonfinite'),
    ('Scale keeps -0.0', [(' + 0.0', '')], None, 'negzero'),
    ('>= at lower == 0', [('lo = inter > lower * area if', 'lo = inter >= lower * area if')], None, 'area_lower0'),
    ('iou intersection with border_pixels',
     [("v = _boxes.iou(np.array([0, 0, w, h]), lab[:, 1:5], coords='corners', mode='element-wise', border_pixels=border_pixels)",
       'v = _iou_with_border(w, h, lab, d)')], {'_iou_with_border': _iou_with_border}, 'iou_bound'),
])
def test_oracle_mutants_disagree_with_golden(name, replacements, extra, kind):
    bad = _disagreements(_mutant(replacements, extra))
    assert [k for k in bad if str(G['kind%d' % k]) == kind], name


def test_scale_and_rotate_store_plus_zero():
    """Scale / Rotate corners that round to -0 are +0 in the reference (astype(int)); Resize's are -0."""
    for k in range(N):
        if str(G['kind%d' % k]) != 'negzero':
            continue
        codes = [int(o[0]) for o in G['ops%d' % k]]
        z = G['lout%d' % k][:, 1:]
        neg = bool((np.signbit(z) & (z == 0)).any())
        if codes[0] in (ac.SCALE, ac.ROTATE):
            assert not neg, k
    keep = _mutant([(' + 0.0', '')])
    assert any(not same_bits(keep(G['lin%d' % k], _ops(k)), G['lout%d' % k]) for k in range(N)
               if int(G['ops%d' % k][0, 0]) == ac.ROTATE)


def test_case_table_reaches_every_path():
    rng = np.random.default_rng(5)
    plans = []
    for G_ in ac.G_COUNTS:
        lab = ac.scattered_labels(rng, G_)
        kept = [g for g in range(G_) if bo.apply_box_ops(lab[g:g + 1], ac.scattered_ops()).shape[0]]
        plans.append((ac.box_plan(G_, kept), len(kept)))
    assert max(p['chunks'] for p, _ in plans) >= 8
    assert any(p['carry'] for p, _ in plans)
    assert any(p['kept_warps'] == {0, 1, 2, 3} for p, _ in plans)
    assert all(0 < n < G_ for (p, n), G_ in zip(plans, ac.G_COUNTS) if G_ >= 31), [n for _, n in plans]
    assert {ac.offsets_per(B) for B in ac.BATCH_SIZES} == {1, 2, 3}
    modes, clamps = set(), set()
    for name, shape, ops, oh, ow in ac.image_edge_cases():
        p = ac.image_plan(shape, ops, oh, ow)
        modes.add(p['mode'])
        clamps |= {(p['mode'], 'row')} if p['row_clamp'] else set()
        clamps |= {(p['mode'], 'col')} if p['col_clamp'] else set()
        if 'identity' in name or 'crops only' in name:
            assert p['mode'] == 'kImgCopy', name
        if 'only' in name and 'crops' not in name:
            assert p['mode'] != 'kImgArea2', name
        if name.startswith('2x both') and name.endswith('lin'):
            assert p['mode'] == 'kImgArea2', name
    warp, (lo, hi) = ac.warp_cases()
    wplans = [ac.image_plan(s, [(ac.SCALE, 0, f, float(s[0]), float(s[1]), 0.0)], s[0], s[1]) for _, s, f in warp]
    assert not ac.scale_accepted(100, 120, lo) and ac.scale_accepted(100, 120, hi)
    assert any(p['saturates'] for p in wplans) and not all(p['saturates'] for p in wplans)
    modes |= {p['mode'] for p in wplans}
    assert modes == set(ac.MODES), modes
    assert {('kImgLinear', 'row'), ('kImgLinear', 'col')} <= clamps
    assert ac.instantiation(wplans) == 'image_assemble_kernel<true>'
    assert ac.instantiation([ac.image_plan(c[1], c[2], c[3], c[4]) for c in ac.image_edge_cases()]) == 'image_assemble_kernel<false>'
    widths = {ow for _, _, _, _, ow in ac.image_edge_cases()}
    assert {ac.IMG_THREADS - 1, ac.IMG_THREADS, ac.IMG_THREADS + 1} <= widths
    gx, tails = ac.photo_grid([(1, w) for w in ac.PHOTO_WIDTHS])
    assert gx == 1 and tails == [1, 31, 0, 1]
    gx, _ = ac.photo_grid([(1000, 1000)])
    assert gx > 1


def test_image_oracle_matches_cv2_on_the_edge_cases():
    """The image cases of the GPU test through oracle/warpops.py against cv2.resize / cv2.warpAffine themselves."""
    cv2 = pytest.importorskip('cv2')
    from oracle import warpops as wo
    rng = np.random.default_rng(7)
    for name, (h, w, c), ops, oh, ow in ac.image_edge_cases():
        img = wo.to3(rng.integers(0, 256, (h, w, c), dtype=np.uint8))
        if int(ops[-1][0]) != ac.RESIZE:
            continue
        canvas = wo.apply_ops(img, ops[:-1])
        interp = (int(ops[-1][1]) >> 8) & 255
        np.testing.assert_array_equal(wo.apply_ops(img, ops), cv2.resize(canvas, (ow, oh), interpolation=interp), err_msg=name)
    warp, _ = ac.warp_cases()
    for name, (h, w, c), f in warp:
        img = wo.to3(rng.integers(0, 256, (h, w, c), dtype=np.uint8))
        ref = cv2.warpAffine(img, cv2.getRotationMatrix2D((w / 2, h / 2), 0, f), (w, h), borderMode=cv2.BORDER_CONSTANT, borderValue=(9, 200, 31))
        np.testing.assert_array_equal(wo.scale(img, f, (9, 200, 31)), ref, err_msg=name)


def _load_generator(monkeypatch):
    if not os.path.isdir(os.path.join(REF_ROOT, 'data_generator')):
        pytest.skip('reference checkout not available')
    pytest.importorskip('cv2')
    monkeypatch.setattr(sys, 'path', list(sys.path))
    monkeypatch.setenv('SSD_REFERENCE_ROOT', REF_ROOT)
    path = os.path.join(os.path.dirname(ac.GOLDEN), 'make_assembly_edges_golden.py')
    spec = importlib.util.spec_from_file_location('_make_assembly_edges_golden', path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_live_reference_reproduces_golden(monkeypatch):
    gen = _load_generator(monkeypatch)
    for k in range(N):
        calls, h, w = eval(str(G['calls%d' % k]), {'np': np, 'nan': float('nan'), 'inf': float('inf')})
        with np.errstate(invalid='ignore'):
            ref, rows = gen.run(calls, G['lin%d' % k], h, w)
        assert same_bits(ref, G['lout%d' % k]), k
        np.testing.assert_array_equal(rows, G['ops%d' % k])
