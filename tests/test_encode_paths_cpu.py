"""CPU half of the encoder path tests: the Python restatement of csrc/encode.cu's decisions (tests/encode_cases.py) must find
every path of the encoder reached by the GPU case table, the restated tile sets must keep the invariants ``tiles_cover``
enforces, and the oracle must equal the reference's own encoder bit for bit on the threshold, conflict, zero-row and
thr <= 0 cases (tests/golden/ref_encode_edges_golden.npz, written by tests/golden/make_encode_edges_golden.py)."""
import os
import re
import sys

import numpy as np
import pytest

import encode_cases as ec

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def test_kernel_constants_are_read_from_the_source():
    assert (ec.TILE, ec.MAX_RUNS, ec.INLINE_B) == (256, 16, 1024)
    assert (ec.SPATIAL_MIN, ec.LB_MIN, ec.TPC_LADDER, ec.SMEM_MAX) == (24, 17, (16, 48, 96), 227 * 1024)
    with open(ec.ENCODE_CU) as f:
        src = f.read()
    # the restatements below follow these lines of the source
    assert 'while (tpc > 1 && (long long)ceil_div(ts.n_tiles, tpc) * B < 8ll * e->ctx->sm_count) tpc >>= 1;' in src
    assert 'const bool use_spatial = e->spatial.dev.n_tiles > 0 && max_g >= spatial_min;' in src
    assert 'const bool use_lb = max_g >= lb_min && total_g > 0;' in src
    assert 'const bool inline_offs = offs_host != nullptr && B <= kInlineB;' in src
    assert re.search(r'if \(!\(nv < \(double\)lbg\)\) continue;', src)                      # C2
    assert 'if (tid == 0 && s_nrem < G) matches[0] = 0;' in src                               # zero-row quirk in the loop
    assert 'const int nparts = G < kTile ? (kTile / G < kTile / 32 ? kTile / G : kTile / 32) : 1;' in src


@pytest.fixture(scope='module')
def reached():
    out = {}
    for c in ec.CASES + [ec.RING]:
        _, r, _ = ec.paths(c, ec.inputs(c['name']))
        out[c['name']] = r
    return out


@pytest.mark.parametrize('path', sorted(ec.REQUIRED))
def test_case_table_reaches_path(reached, path):
    """Each path of the encoder, and the case that reaches it."""
    assert path in reached[ec.REQUIRED[path]], (path, ec.REQUIRED[path], sorted(reached[ec.REQUIRED[path]]))


def test_conflict_cases_model():
    """The numbers the kernel's SSDK_ENC_COUNTERS=1 counters are held to, and the C1 claim that does not rest on a float32 bound."""
    ev = ec.paths(ec.BY_NAME['chain4'], ec.inputs('chain4'))[2][0]
    assert (ev['iterations'], ev['victims'], ev['c2']) == (4, [3, 2, 1], 0)
    ev = ec.paths(ec.BY_NAME['chain4_lb'], ec.inputs('chain4_lb'))[2][0]
    assert (ev['iterations'], ev['victims'], ev['c2']) == (4, [3, 2, 1], 6)
    ev = ec.paths(ec.BY_NAME['tozero'], ec.inputs('tozero'))[2][0]
    assert (ev['iterations'], ev['victims'], ev['to_zero'], ev['quirk_loop']) == (3, [2, 1], 1, True)
    ev = ec.paths(ec.BY_NAME['c1_other_tile'], ec.inputs('c1_other_tile'))[2][0]
    assert ev['c1_other'] == ['yes'] and ev['iterations'] == 2
    for c in ec.CASES:
        if c['counters']:
            for e in ec.paths(c, ec.inputs(c['name']))[2]:
                assert 'undetermined' not in e['c1_other'], c['name']


def test_threshold_cases_sit_on_the_thresholds():
    """IoU exactly 0.5 / 0.3 in every coordinate format; the 'below' cases raise the thresholds by one float64 ulp."""
    for name in ('thr_at_centroids', 'thr_at_corners', 'thr_at_minmax', 'thr_at_corners_f64', 'thr_below_centroids_f64'):
        c = ec.BY_NAME[name]
        cfg = ec.config(c)
        sim, _ = ec.exact_sim(cfg, ec.inputs(name)[0])
        assert (sim == 0.5).sum() == 2 and (sim == 0.3).sum() == 1, name
    for name in ('thr_below_centroids', 'thr_below_corners', 'thr_below_minmax', 'thr_below_centroids_f64'):
        cfg = ec.config(ec.BY_NAME[name])
        assert cfg['pos_iou_threshold'] == np.nextafter(0.5, 1) and cfg['neg_iou_limit'] == np.nextafter(0.3, 1)
    g = ec.inputs('thr_at_corners_f64')[0]
    assert g.dtype == np.float64 and (g.astype(np.float32).astype(np.float64) != g).any()


def test_oracle_matches_reference_edge_golden():
    if GOLD not in sys.path:
        sys.path.insert(0, GOLD)
    import make_encode_edges_golden as mk
    with np.load(os.path.join(GOLD, 'ref_encode_edges_golden.npz')) as z:
        assert sorted(z.files) == sorted(mk.EDGE_CASES)
        for name in mk.EDGE_CASES:
            c = ec.BY_NAME[name]
            got = ec.oracle_encoder(ec.config(c))(ec.inputs(name))
            np.testing.assert_array_equal(got, z[name], err_msg=name)


def test_golden_cases_differ_at_the_thresholds():
    """One ulp of threshold changes the reference's targets: the 'at' and 'below' fixtures are not the same tensors."""
    with np.load(os.path.join(GOLD, 'ref_encode_edges_golden.npz')) as z:
        for co in ('centroids', 'corners', 'minmax'):
            a, b = z['thr_at_%s' % co], z['thr_below_%s' % co]
            C = 3
            assert (a[..., :C] != b[..., :C]).any(), co


@pytest.mark.parametrize('cfg_name', ['ssd300', 'ssd512', 'ssd7', 'tiny', 'tiny_clip_abs', 'micro', 'dyadic'])
def test_tile_sets_cover_every_prior(cfg_name):
    cfg = dict(ec.DYADIC) if cfg_name == 'dyadic' else ec.golden_configs()[cfg_name]
    P = ec.oracle_encoder(cfg).anchors.shape[0]
    fh, fw, nb = ec.layer_geometry(cfg)
    assert sum(h * w * n for h, w, n in zip(fh, fw, nb)) == P
    for tiles in (ec.linear_tiles(P), ec.spatial_tiles(fh, fw, nb)):
        assert ec.tiles_cover(tiles, P)
        assert len(ec.linear_tiles(P)) == -(-P // ec.TILE)
    # the check itself rejects a prior listed twice
    bad = ec.linear_tiles(P)
    bad[0]['map'][1] = bad[0]['map'][0]
    assert not ec.tiles_cover(bad, P)


def test_spatial_ssd300_has_both_store_routes():
    cfg = ec.golden_configs()['ssd300']
    P = ec.oracle_encoder(cfg).anchors.shape[0]
    al = ec.tile_aligned(ec.spatial_tiles(*ec.layer_geometry(cfg)), P, 33, False)
    assert any(al) and not all(al)


def test_sm_count_clamp():
    c = ec.BY_NAME['tpc8']
    gts = ec.inputs('tpc8')
    assert ec.host_decisions(c, gts, 132)['tpc'] == 8
    assert ec.host_decisions(c, gts, 1000)['tpc'] < 8
