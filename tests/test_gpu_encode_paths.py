"""Every path of the encoder (csrc/encode.cu, ``SSDInputEncoder`` on the device) against the exact reference.

Each case of tests/encode_cases.py runs through the entry points it names.  Class vectors and match / neutral assignments must
be identical to the float64 oracle; every float column must be the oracle's value rounded once to float32, except that the two
centroid ``log`` columns may hold the other neighbouring float32 where the oracle's value lies within 4 float64 ulps of a float32
rounding midpoint (neither CUDA's double ``log`` nor NumPy's is correctly rounded).  tests/test_encode_paths_cpu.py checks
that the cases reach every path; here the kernel's own counters of the conflict loop must equal that model's numbers."""
import re

import numpy as np
import pytest

import encode_cases as ec

pytestmark = pytest.mark.gpu

ENV_KEYS = ('SSDK_ENC_SPATIAL_MIN', 'SSDK_ENC_LB_MIN', 'SSDK_ENC_TPC', 'SSDK_ENC_COUNTERS')


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    import torch
    assert torch.cuda.is_available()


@pytest.fixture
def env(monkeypatch):
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    return monkeypatch


def device_encoder(cfg):
    from ssd_keras_b200.ssd_encoder_decoder.ssd_input_encoder import SSDInputEncoder
    return SSDInputEncoder(**cfg)


def flat(gts, dtype):
    import torch
    rows = [np.asarray(g, np.float64).reshape(-1, 5) for g in gts]
    offs = np.cumsum([0] + [r.shape[0] for r in rows]).astype(np.int32)
    if not offs[-1]:
        return None, offs
    return torch.from_numpy(np.concatenate(rows).astype(dtype)).cuda(), offs


def assert_exact(c, y, match, ref):
    """y (B, P, W) float32 numpy from the kernel, match (B, P) or None; ref = the oracle's (y, match, neutral) of the distinct
    images."""
    y_ref, m_ref, n_ref = ref
    n = y_ref.shape[0]
    cfg = ec.config(c)
    C = cfg['n_classes'] + 1
    assert y.shape[1:] == y_ref.shape[1:] and y.shape[0] % n == 0
    for b0 in range(0, y.shape[0], n):
        yb = y[b0:b0 + n]
        np.testing.assert_array_equal(yb[..., :C], y_ref[..., :C].astype(np.float32))
        ec.assert_float_columns(yb[..., C:], y_ref[..., C:], C, cfg.get('coords', 'centroids'))
        if match is not None:
            np.testing.assert_array_equal(match[b0:b0 + n], np.where(m_ref >= 0, m_ref, np.where(n_ref, -2, -1)))


def run(c, gts, dtype=np.float32):
    """-> (y float32 numpy, match or None) through the case's entry point."""
    import torch
    enc = device_encoder(ec.config(c))
    gd, offs = flat(gts, dtype)
    P, W = enc.anchors.shape[0], enc.n_classes + 12
    B = len(gts)
    if c['entry'] in ('device', 'device_ub'):
        tot, mg = (ec.upper_bounds(c, gts) if c['entry'] == 'device_ub' else (int(offs[-1]), int(np.diff(offs).max())))
        y = enc.encode_device_offsets(gd, torch.from_numpy(offs).cuda(), tot, mg)
        assert int(enc.last_status.item()) == 0
        return y.cpu().numpy(), None
    out = None
    if c['out_offset']:
        buf = torch.empty((B * P * W + 1,), dtype=torch.float32, device='cuda')
        out = buf[1:].view(B, P, W)                                # every image base 4 bytes past a 16-byte boundary
        assert out.data_ptr() % 16 == 4
    y, match = enc.encode_device(gd, offs, return_matches=True, out=out)
    if out is not None:
        assert y is out
    assert int(enc.last_status.item()) == 0
    return y.cpu().numpy(), match.cpu().numpy()


@pytest.mark.parametrize('name', [c['name'] for c in ec.CASES])
def test_encode_path_exact(name, env):
    c = ec.BY_NAME[name]
    for k, v in c['env'].items():
        env.setenv(k, v)
    gts = ec.inputs(name)
    ref = ec.reference(c, gts)
    dtypes = [np.float64] if c['gt64'] else [np.float32, np.float64]
    if c['entry'] != 'host':
        dtypes = dtypes[:1]
    for dt in dtypes:
        y, match = run(c, gts, dt)
        assert_exact(c, y, match, ref)


def test_encode_call_api_exact(env):
    """SSDInputEncoder.__call__ (float64 labels, ssdk_encode with gt_f64 = 1) on the threshold and thr_adj = 0 cases."""
    for name in ('thr_at_centroids', 'thr_below_minmax', 'thr0_neg0', 'thr0_negative', 'tozero', 'c1_other_tile'):
        c = ec.BY_NAME[name]
        gts = ec.inputs(name)
        y = device_encoder(ec.config(c))(gts)
        assert_exact(c, y.astype(np.float32), None, ec.reference(c, gts))


_COUNTERS = re.compile(r'iterations ([\d.]+) victims ([\d.]+) below-bound searches ([\d.]+) \(images (\d+)\)')


@pytest.mark.parametrize('name', [c['name'] for c in ec.CASES if c['counters']])
def test_conflict_loop_counters_enc_counters(name, env, capfd):
    """SSDK_ENC_COUNTERS=1 prints the matching stage's event counts; one image per launch, so they are integers."""
    c = ec.BY_NAME[name]
    for k, v in c['env'].items():
        env.setenv(k, v)
    env.setenv('SSDK_ENC_COUNTERS', '1')
    for b, g in enumerate(ec.inputs(name)):
        _, _, events = ec.paths(c, [g])
        ev = events[0]
        capfd.readouterr()
        y, match = run(c, [g])
        err = capfd.readouterr().err
        m = _COUNTERS.search(err)
        assert m, err
        it, vi, c2, n = float(m.group(1)), float(m.group(2)), float(m.group(3)), int(m.group(4))
        assert n == 1
        assert (it, vi, c2) == (ev['iterations'], sum(ev['victims']), ev['c2']), (name, b, err, ev)
        assert_exact(c, y, match, ec.oracle_encoder(ec.config(c))([g], return_matches=True))


def test_settings_give_the_same_bits(env):
    """Tile set, lower bounds and tiles per CTA change the work, never the result."""
    c = ec.BY_NAME['ssd300_spatial']
    gts = ec.inputs('ssd300_spatial')
    base, bm = run(c, gts)
    for s in (dict(SSDK_ENC_SPATIAL_MIN='0'), dict(SSDK_ENC_SPATIAL_MIN='1000000'), dict(SSDK_ENC_LB_MIN='0'),
              dict(SSDK_ENC_LB_MIN='1000000'), dict(SSDK_ENC_TPC='2', SSDK_ENC_SPATIAL_MIN='0'),
              dict(SSDK_ENC_TPC='8', SSDK_ENC_LB_MIN='1000000')):
        for k in ENV_KEYS:
            env.delenv(k, raising=False)
        for k, v in s.items():
            env.setenv(k, v)
        y, m = run(c, gts)
        np.testing.assert_array_equal(y.view(np.uint32), base.view(np.uint32))
        np.testing.assert_array_equal(m, bm)


def test_pinned_offset_ring_reuse(env):
    """B = 1100 > kInlineB: the offsets go through the 8-slot pinned ring; ten launches with different boxes reuse its slots."""
    c = ec.RING
    cfg = ec.config(c)
    enc = device_encoder(cfg)
    ys = []
    for seed in ec.RING_SEEDS:
        gts = ec.gen_random(seed, 1100, 2, cfg)
        gd, offs = flat(gts, np.float32)
        ys.append((gts, enc.encode_device(gd, offs, return_matches=True)))
    assert ec.host_decisions(c, gts)['route'] == 'ring'
    for gts, (y, m) in ys:
        assert_exact(c, y.cpu().numpy(), m.cpu().numpy(), ec.oracle_encoder(cfg)(gts, return_matches=True))


def test_alternating_grid_widths(env):
    """One encoder, launches whose grids differ (linear tiles, one per CTA / spatial tiles): the per-image tickets reset."""
    cfg = ec.golden_configs()['ssd300']
    enc = device_encoder(cfg)
    a = ec.gen_random(60, 3, 3, cfg)
    b = ec.gen_random(61, 3, 30, cfg)
    ca, cb = ec.case('a', 'ssd300', None), ec.case('b', 'ssd300', None)
    assert len(ec.host_decisions(ca, a)['tiles']) != len(ec.host_decisions(cb, b)['tiles'])
    ra, rb = (ec.oracle_encoder(cfg)(g, return_matches=True) for g in (a, b))
    for gts, ref, c in ((a, ra, ca), (b, rb, cb), (a, ra, ca), (b, rb, cb), (a, ra, ca)):
        gd, offs = flat(gts, np.float32)
        y, m = enc.encode_device(gd, offs, return_matches=True)
        assert_exact(c, y.cpu().numpy(), m.cpu().numpy(), ref)


def test_shared_memory_refusal_before_any_launch(env):
    """About 600 boxes in one image at n_classes = 80 need more than 227 KB of shared memory: refused on the host."""
    from ssd_keras_b200 import _ffi
    cfg = ec.golden_configs()['ssd512']
    enc = device_encoder(cfg)
    enc._encoder()
    gts = ec.gen_random(62, 1, 600, cfg)
    W = cfg['n_classes'] + 13
    assert ec.smem_layout(W, 600) > ec.SMEM_MAX >= ec.smem_layout(W, 500)
    gd, offs = flat(gts, np.float32)
    import torch
    torch.cuda.synchronize()
    n0 = _ffi.launch_count()
    with pytest.raises(ValueError, match='ssdk_encode: n_classes'):
        enc.encode_device(gd, offs)
    assert _ffi.launch_count() == n0


@pytest.mark.parametrize('coords', ['centroids', 'corners', 'minmax'])
@pytest.mark.parametrize('border', ['half', 'include', 'exclude'])
def test_iou_matrix_exact(coords, border):
    import torch
    from ssd_keras_b200 import _ffi
    for base, seed in (('tiny', 70), ('dyadic', 71)):
        cfg = dict(ec.DYADIC) if base == 'dyadic' else dict(ec.golden_configs()[base])
        cfg.update(coords=coords, border_pixels=border)
        enc = device_encoder(cfg)
        g = ec.gen_random(seed, 1, 9, cfg)[0]
        if base == 'dyadic':
            g = np.concatenate([g, ec.gen_threshold(np.float32)[0]])
        G, P = g.shape[0], enc.anchors.shape[0]
        out = torch.empty((G, P), dtype=torch.float64, device='cuda')
        _ffi.check(_ffi.lib().ssdk_iou_matrix(enc._encoder(), _ffi.dptr(torch.from_numpy(g).cuda()), G, _ffi.dptr(out),
                                              _ffi.stream_ptr()))
        want, _ = ec.exact_sim(cfg, g)
        np.testing.assert_array_equal(out.cpu().numpy(), want)
