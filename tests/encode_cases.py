"""Case table of the encoder tests (tests/test_gpu_encode_paths.py) and a restatement, in Python, of the decisions
csrc/encode.cu makes for each case (tests/test_encode_paths_cpu.py checks that together the cases reach every path).

``encode_launch`` picks, from the largest box count of the batch (``max_g``): the linear or the spatial tile set, whether
``enc_lb_kernel`` computes lower bounds of the row maxima, the tiles per CTA (``tpc``, halved while the grid would not fill
the GPU), the route of the ground-truth offsets (kernel argument, pinned ring, or already on the device) and the dynamic
shared memory.  Per tile, rows leave by bulk copy when every run of the tile and the image's base address are 16-byte
aligned, by plain stores otherwise.  The last CTA of an image runs ``match_bipartite_greedy``: without two rows that want the
same prior the rounds commute; otherwise the conflict loop settles rows up to the first one with a later duplicate (stage A /
B), lets the rows that lost their prior re-scan that prior's tile (C1, again in the tile of any taken prior that then wins) and
searches every slice for a row that fell below its lower bound (C2).  ``bipartite_events`` replays that loop on the oracle's
exact float64 IoU matrix.

Every case is plain data plus a seeded generator, so the GPU test and the CPU model see the same inputs."""
import functools
import math
import os
import re

import numpy as np

from oracle import synth
from oracle.boxes import convert_coordinates, iou
from oracle.encoder import OracleEncoder

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENCODE_CU = os.path.join(ROOT, 'ssd_keras_b200', 'csrc', 'encode.cu')
COMMON_CUH = os.path.join(ROOT, 'ssd_keras_b200', 'csrc', 'common.cuh')
GOLDEN_DIR = os.path.join(ROOT, 'tests', 'golden')


def kernel_constants():
    """The constants and host thresholds of csrc/encode.cu, read from the source so that this model cannot drift from it."""
    with open(ENCODE_CU) as f:
        src = f.read()
    k = {n: int(v) for n, v in re.findall(r'constexpr int (k\w+) = (\d+);', src)}
    m = re.search(r'int spatial_min = (\d+), lb_min = (\d+);', src)
    k['spatial_min'], k['lb_min'] = int(m.group(1)), int(m.group(2))
    m = re.search(r'int tpc = max_g <= (\d+) \? 1 : \(max_g <= (\d+) \? 2 : \(max_g < (\d+) \? 4 : 8\)\);', src)
    k['tpc_ladder'] = tuple(int(v) for v in m.groups())
    # each default is what its switch (ssdk::env_int) falls back to; SSDK_ENC_TPC is clamped to >= 1 as in paths() below
    for name, var in (('SSDK_ENC_SPATIAL_MIN', 'spatial_min'), ('SSDK_ENC_LB_MIN', 'lb_min'), ('SSDK_ENC_TPC', 'tpc')):
        assert 'env_int("%s", %s, &%s)' % (name, var, var) in src, name
    assert 'tpc = std::max(1, tpc);' in src, 'tiles per CTA clamped to >= 1'
    # enc_tiles_kernel gets L.total bytes of dynamic shared memory through ssdk::launch, which opts in above 48 KB
    m = re.search(r'launch\(e->ctx, inline_offs \? enc_tiles_kernel<true> : enc_tiles_kernel<false>, grid, kTile, L\.total,', src)
    assert m, 'dynamic shared memory of enc_tiles_kernel'
    with open(COMMON_CUH) as f:
        assert 'if (bytes <= 48 * 1024) return SSDK_OK;' in f.read(), 'dynamic shared-memory opt-in'
    m = re.search(r'SSDK_REQUIRE\(L.total <= (\d+) \* 1024', src)
    k['smem_max'] = int(m.group(1)) * 1024
    return k


_K = kernel_constants()
TILE, MAX_RUNS, INLINE_B = _K['kTile'], _K['kMaxRuns'], _K['kInlineB']
SPATIAL_MIN, LB_MIN, TPC_LADDER, SMEM_MAX = _K['spatial_min'], _K['lb_min'], _K['tpc_ladder'], _K['smem_max']


# ------------------------------------------------------------------------------------------------
# configurations
# ------------------------------------------------------------------------------------------------
def golden_configs():
    import conftest
    return conftest.golden_configs()


# 64 x 64 pixels, not normalised: 16 anchors of 16 x 16 on a 16-pixel grid plus one of 64 x 64; every corner is dyadic, so
# IoUs such as 256 / 512 and 96 / 320 come out as the float64 nearest to 0.5 and 0.3.  P * W = 17 * 15 is odd.
DYADIC = dict(img_height=64, img_width=64, n_classes=2, predictor_sizes=[(4, 4), (1, 1)], scales=[0.25, 1.0, 1.0],
              aspect_ratios_global=[1.0], two_boxes_for_ar1=False, steps=None, offsets=None, clip_boxes=False,
              variances=[0.1, 0.1, 0.2, 0.2], matching_type='multi', pos_iou_threshold=0.5, neg_iou_limit=0.3,
              coords='corners', normalize_coords=False)


def config(c):
    base = c['cfg']
    cfg = dict(DYADIC) if base == 'dyadic' else dict(golden_configs()[base])
    cfg.update(c.get('over', {}))
    return cfg


@functools.lru_cache(maxsize=None)
def _oracle(key):
    import json
    return OracleEncoder(**json.loads(key))


def oracle_encoder(cfg):
    import json
    return _oracle(json.dumps(cfg, sort_keys=True))


# ------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------
def _rows(cls, boxes, dtype=np.float32):
    b = np.asarray(boxes, np.float64).reshape(-1, 4)
    return np.concatenate([np.asarray(cls, np.float64).reshape(-1, 1), b], 1).astype(dtype)


def _anchor_corners(cfg):
    a = oracle_encoder(cfg).anchors
    if cfg.get('coords', 'centroids') == 'centroids':
        return convert_coordinates(a, 0, 'centroids2corners')
    if cfg['coords'] == 'minmax':
        return a[:, [0, 2, 1, 3]]
    return a


def _shrunk(box, f):
    cx, cy, w, h = (box[0] + box[2]) / 2, (box[1] + box[3]) / 2, box[2] - box[0], box[3] - box[1]
    return [cx - f * w / 2, cy - f * h / 2, cx + f * w / 2, cy + f * h / 2]


def gen_threshold(dtype):
    """Dyadic pairs: [0,0,16,32] has IoU 0.5 with two anchors, [10,32,20,48] IoU 96/320 = 0.3 with one, and a few more."""
    rows = [[1, 0, 0, 16, 32], [2, 10, 32, 20, 48], [1, 40, 8, 56, 24], [2, 34, 40, 62, 62]]
    r = np.asarray(rows, np.float64)
    if dtype == np.float64:
        r[3, 1:] += 1e-9                                            # a coordinate float32 cannot hold
    return [r.astype(dtype)]


def gen_thr0(cfg_bg):
    """Boxes of every class including the background class."""
    out = []
    for i, s in enumerate((3, 4)):
        g = synth.synth_gt(s, 1, 5, 160, 120, 3)[0]
        g[:, 0] = np.arange(5) % 4
        out.append(g)
    out[0][0, 0] = cfg_bg
    return out


def gen_chain(n_same):
    """SSD300: n_same identical boxes (each loses the prior the one before it took: one iteration per box) and two others."""
    b = [[1, 100, 80, 160, 150]] * n_same + [[2, 20, 20, 60, 90], [3, 200, 200, 290, 280]]
    return [_rows([r[0] for r in b], [r[1:] for r in b])]


def gen_tozero():
    """Dyadic config: three copies of a small box that overlaps exactly two anchors: the third copy's row falls to zero."""
    b = [[1, 2, 2, 6, 6]] * 3 + [[2, 36, 36, 60, 60]]
    return [_rows([r[0] for r in b], [r[1:] for r in b])]


def gen_c1(cfg):
    """Three boxes around two neighbouring priors a* and r of different linear tiles (SSD300 layer 0, cells 63 and 64):
    P1 = r shrunk (settled first, takes r), Q = a* shrunk (takes a*), V between them, whose maximum is a* and runner-up r.
    V loses a* to Q; the best other tile's recorded pair for V is r, already taken: C1 re-scans r's tile too."""
    anc = _anchor_corners(cfg)
    H, W = cfg['img_height'], cfg['img_width']
    a_star, r = 63 * 4, 64 * 4                                      # first box shape of cells 63 and 64
    A = anc[a_star] * [W, H, W, H]
    R = anc[r] * [W, H, W, H]
    p1 = _shrunk(R, 0.98)
    q = _shrunk(A, 0.95)
    v = [A[0] + 0.3 * (R[0] - A[0]), A[1], A[2] + 0.3 * (R[2] - A[2]), A[3]]
    return [_rows([1, 2, 3], [p1, q, v])]


def gen_random(seed, B, G, cfg, ncls=None):
    n = ncls if ncls is not None else cfg['n_classes']
    return synth.synth_gt(seed, B, G, cfg['img_width'], cfg['img_height'], n)


def case(name, cfg, gen, entry='host', env=None, over=None, B=None, out_offset=False, gt64=False, counters=False):
    return dict(name=name, cfg=cfg, gen=gen, entry=entry, env=dict(env or {}), over=dict(over or {}), B=B,
                out_offset=out_offset, gt64=gt64, counters=counters)


NEXT_05 = float(np.nextafter(0.5, 1.0))
NEXT_03 = float(np.nextafter(0.3, 1.0))

CASES = []
for _co in ('centroids', 'corners', 'minmax'):
    CASES.append(case('thr_at_%s' % _co, 'dyadic', ('threshold', 'f32'), over=dict(coords=_co)))
    CASES.append(case('thr_below_%s' % _co, 'dyadic', ('threshold', 'f32'),
                      over=dict(coords=_co, pos_iou_threshold=NEXT_05, neg_iou_limit=NEXT_03)))
CASES += [
    case('thr_at_corners_f64', 'dyadic', ('threshold', 'f64'), gt64=True),
    case('thr_below_centroids_f64', 'dyadic', ('threshold', 'f64'), gt64=True,
         over=dict(coords='centroids', pos_iou_threshold=NEXT_05, neg_iou_limit=NEXT_03)),
    case('thr0_neg0', 'tiny', ('thr0', 2), over=dict(neg_iou_limit=0.0, background_id=2)),
    case('thr0_negative', 'tiny', ('thr0', 3), over=dict(neg_iou_limit=-0.1, background_id=3, coords='corners')),
    case('no_multi_pos', 'tiny', ('random', 31, 3, 6), over=dict(pos_iou_threshold=1.5)),
    case('bipartite_only', 'ssd7', ('random', 32, 2, 10), over=dict(matching_type='bipartite')),
    case('g1', 'ssd300', ('random', 33, 2, 1)),
    case('chain4', 'ssd300', ('chain', 4), counters=True),
    case('chain4_lb', 'ssd300', ('chain', 4), env=dict(SSDK_ENC_LB_MIN='0'), counters=True),
    case('tozero', 'dyadic', ('tozero',), counters=True),
    case('tozero_lb', 'dyadic', ('tozero',), env=dict(SSDK_ENC_LB_MIN='0'), counters=True),
    case('c1_other_tile', 'ssd300', ('c1',), counters=True),
    case('g150', 'ssd300', ('random', 34, 1, 150)),
    case('g300', 'ssd300', ('random', 35, 1, 300), counters=True),
    case('out_offset', 'ssd300', ('random', 36, 3, 8), out_offset=True),
    case('odd_image_stride', 'dyadic', ('random', 37, 5, 3), env=dict(SSDK_ENC_SPATIAL_MIN='0')),
    case('ssd300_spatial', 'ssd300', ('random', 38, 3, 30)),
    case('forced_linear_lb', 'ssd300', ('random', 38, 3, 30), env=dict(SSDK_ENC_SPATIAL_MIN='1000000', SSDK_ENC_LB_MIN='0')),
    case('forced_spatial_nolb', 'ssd300', ('random', 38, 3, 30), env=dict(SSDK_ENC_SPATIAL_MIN='0', SSDK_ENC_LB_MIN='1000000')),
    case('forced_tpc1', 'ssd300', ('random', 38, 3, 30), env=dict(SSDK_ENC_TPC='1')),
    case('forced_tpc4', 'ssd300', ('replicate', 38, 3, 30, 32), env=dict(SSDK_ENC_TPC='4', SSDK_ENC_LB_MIN='0')),
    case('zero_rows', 'tiny', ('fixed_zero',)),
    case('tpc2', 'ssd300', ('replicate', 39, 4, 40, 16)),
    case('tpc8', 'ssd300', ('replicate', 40, 4, 2, 45), env=dict(SSDK_ENC_TPC='8', SSDK_ENC_SPATIAL_MIN='0')),
    case('device_upper_bounds', 'ssd300', ('random', 41, 4, 5), entry='device_ub'),
    case('c80_inline', 'ssd512', ('random', 42, 2, 20)),
    case('c80_device', 'ssd512', ('random', 42, 2, 20), entry='device'),
]
BY_NAME = {c['name']: c for c in CASES}


@functools.lru_cache(maxsize=None)
def _inputs(name):
    c = BY_NAME[name]
    cfg = config(c)
    kind = c['gen'][0]
    if kind == 'threshold':
        return gen_threshold(np.float64 if c['gen'][1] == 'f64' else np.float32)
    if kind == 'thr0':
        return gen_thr0(c['gen'][1])
    if kind == 'chain':
        return gen_chain(c['gen'][1])
    if kind == 'tozero':
        return gen_tozero()
    if kind == 'fixed_zero':                                        # boxes outside the image: rows whose IoUs are all zero
        return [_rows([1, 2, 3], [[20, 20, 60, 70], [170, 130, 180, 140], [200, 10, 230, 40]]), gen_random(43, 1, 4, cfg)[0]]
    if kind == 'c1':
        return gen_c1(cfg)
    if kind == 'replicate':                                         # distinct images repeated to fill a large grid
        _, seed, n, G, reps = c['gen']
        return gen_random(seed, n, G, cfg) * reps
    _, seed, B, G = c['gen']
    return gen_random(seed, B, G, cfg)


def inputs(name):
    return [g.copy() for g in _inputs(name)]


def distinct(c, gts):
    """The distinct images of a batch: a replicated batch repeats its first n images."""
    return gts[:c['gen'][2]] if c['gen'][0] == 'replicate' else gts


def reference(c, gts):
    """(y float64, match index, neutral flag) of the oracle, for the distinct images (image b of the batch is b % n)."""
    return oracle_encoder(config(c))(distinct(c, gts), return_matches=True)


# ------------------------------------------------------------------------------------------------
# the bar
# ------------------------------------------------------------------------------------------------
def assert_float_columns(got, want, C, coords):
    """got: the float32 kernel columns from C on, want: the float64 oracle columns of the same rows.  Every column must be the
    oracle rounded once to float32; a centroid log column may hold the other neighbour of a value within 4 float64 ulps of a
    float32 rounding midpoint."""
    w32 = want.astype(np.float32)
    logc = [2, 3] if coords == 'centroids' else []
    keep = [k for k in range(want.shape[-1]) if k not in logc]
    np.testing.assert_array_equal(got[..., keep], w32[..., keep])
    for k in logc:
        g, x, f = got[..., k], want[..., k], w32[..., k]
        bad = g != f
        if not bad.any():
            continue
        x, f, g = x[bad], f[bad].astype(np.float64), g[bad].astype(np.float64)
        other = np.where(x > f, np.nextafter(f.astype(np.float32), np.float32(np.inf)),
                         np.nextafter(f.astype(np.float32), np.float32(-np.inf))).astype(np.float64)
        mid = (f + other) / 2
        ok = (g == other) & (np.abs(x - mid) <= 4 * np.spacing(np.abs(x)))
        assert ok.all(), ('log column', k, x[~ok][:5], f[~ok][:5], g[~ok][:5])


# ------------------------------------------------------------------------------------------------
# host decisions (encode_launch)
# ------------------------------------------------------------------------------------------------
def layer_geometry(cfg):
    enc = oracle_encoder(cfg)
    ps = np.asarray(enc.predictor_sizes).reshape(-1, 2)
    return [int(v) for v in ps[:, 0]], [int(v) for v in ps[:, 1]], [int(v) for v in enc.n_boxes]


def linear_tiles(P):
    """linear_layer_tiles over all priors: tile t = priors [256 t, 256 t + 256), one run."""
    return [dict(runs=[(o, min(TILE, P - o))], map=[(o + s, s) for s in range(min(TILE, P - o))]) for o in range(0, P, TILE)]


def spatial_tiles(fh, fw, nbx):
    """spatial_tiles: per layer, blocks of whole rows or of bw x bh cells; map = [(prior, staging slot)] by thread."""
    tiles, off = [], 0

    def begin():
        return dict(runs=[], map={}, fill=0)

    def add_run(t, start, cells, nb, cell0, ncells):
        t['runs'].append((start, cells * nb))
        for cc in range(cells):
            for bx in range(nb):
                t['map'][bx * ncells + cell0 + cc] = (start + cc * nb + bx, t['fill'] + cc * nb + bx)
        t['fill'] += cells * nb

    def lin(first, count):
        for o in range(0, count, TILE):
            t = begin(); n = min(TILE, count - o)
            add_run(t, first + o, n, 1, 0, n); tiles.append(t)

    for H, Wd, nb in zip(fh, fw, nbx):
        count = H * Wd * nb
        if nb > TILE or nb <= 0:
            lin(off, count); off += count
            continue
        cells_max = TILE // nb
        bw = max(1, int(math.floor(math.sqrt(cells_max))))
        if bw >= Wd:
            bh = max(1, min(H, cells_max // Wd))
            for y0 in range(0, H, bh):
                rws = min(bh, H - y0)
                t = begin(); add_run(t, off + y0 * Wd * nb, rws * Wd, nb, 0, rws * Wd); tiles.append(t)
        else:
            bh = max(1, min(H, cells_max // bw, MAX_RUNS))
            for y0 in range(0, H, bh):
                for x0 in range(0, Wd, bw):
                    cw, ch = min(bw, Wd - x0), min(bh, H - y0)
                    t = begin()
                    for y in range(ch):
                        add_run(t, off + ((y0 + y) * Wd + x0) * nb, cw, nb, y * cw, cw * ch)
                    tiles.append(t)
        off += count
    for t in tiles:
        t['map'] = [t['map'].get(s, (-1, 0)) for s in range(TILE)]
        t['map'] = [m for m in t['map'] if m[0] >= 0]
    return tiles


def tiles_cover(tiles, P):
    """The invariants tiles_cover enforces: every prior exactly once, at most 256 slots and kMaxRuns runs per tile, and each
    prior's staging slot is its place in run order."""
    seen = np.zeros(P, bool)
    for t in tiles:
        fill = sum(n for _, n in t['runs'])
        if fill > TILE or len(t['runs']) > MAX_RUNS or len(t['map']) > TILE:
            return False
        slots = set()
        for a, ps in t['map']:
            if a >= P or seen[a] or ps < 0 or ps >= fill or ps in slots:
                return False
            seen[a] = True; slots.add(ps)
            base, want = 0, -1
            for s, n in t['runs']:
                if s <= a < s + n:
                    want = base + a - s
                    break
                base += n
            if want != ps:
                return False
    return bool(seen.all())


def tile_aligned(tiles, P, W, linear):
    """Per tile: its runs leave by bulk copy when the image base is 16-byte aligned (upload_tiles' aligned_mask; the linear
    set tests the single run inline)."""
    out = []
    for t in tiles:
        if linear:
            (s, n), = t['runs']
            out.append((s * W * 4) % 16 == 0 and (n * W * 4) % 16 == 0)
            continue
        ok = (P * W) % 4 == 0
        slot0 = 0
        for s, n in t['runs']:
            ok = ok and (s * W * 4) % 16 == 0 and (n * W * 4) % 16 == 0 and (slot0 * W * 4) % 16 == 0
            slot0 += n
        out.append(ok)
    return out


def smem_layout(W, G):
    """enc_smem_layout(W, G).total."""
    gs = max(G, 1)
    up16 = lambda v: (v + 15) & ~15                                       # noqa: E731
    rows = up16(TILE * W * 4)
    rows = max(rows, up16(gs * 24))
    gf = up16(rows + gs * 40)
    gq = up16(gf + gs * 16)
    wV = up16(gq + gs * 16)
    wU = up16(wV + gs * 64)
    wI = up16(wU + gs * 32)
    items = up16(wI + gs * 32)
    return up16(items + gs * 32 + 16) + 16


def counts_of(c, gts):
    g = [int(np.asarray(x).reshape(-1, 5).shape[0]) for x in gts]
    return g, sum(g), max(g) if g else 0


def upper_bounds(c, gts):
    """The (total_g, max_g) a device_ub case passes: upper bounds that turn the lower bounds and the spatial tiles on."""
    _, tot, mg = counts_of(c, gts)
    return tot + 50, max(mg, 40)


def host_decisions(c, gts, sm_count=132):
    cfg = config(c)
    enc = oracle_encoder(cfg)
    P, W = enc.anchors.shape[0], enc.n_classes + 12
    B = len(gts)
    _, total_g, max_g = counts_of(c, gts)
    if c['entry'] == 'device_ub':
        total_g, max_g = upper_bounds(c, gts)
    env = c['env']
    smin = int(env.get('SSDK_ENC_SPATIAL_MIN', SPATIAL_MIN))
    lmin = int(env.get('SSDK_ENC_LB_MIN', LB_MIN))
    spatial = max_g >= smin                                        # every configuration here has layer geometry
    tiles = spatial_tiles(*layer_geometry(cfg)) if spatial else linear_tiles(P)
    lb = max_g >= lmin and total_g > 0
    l1, l2, l4 = TPC_LADDER
    tpc = 1 if max_g <= l1 else (2 if max_g <= l2 else (4 if max_g < l4 else 8))
    if 'SSDK_ENC_TPC' in env:
        tpc = max(1, int(env['SSDK_ENC_TPC']))
    while tpc > 1 and -(-len(tiles) // tpc) * B < 8 * sm_count:
        tpc >>= 1
    if c['entry'] in ('device', 'device_ub'):
        route = 'device'
    else:
        route = 'inline' if B <= INLINE_B else 'ring'
    smem = smem_layout(W, max_g)
    aligned = tile_aligned(tiles, P, W, not spatial)
    off = 4 if c['out_offset'] else 0
    base_ok = [((off + b * P * W * 4) % 16) == 0 for b in range(B)]
    return dict(P=P, W=W, B=B, total_g=total_g, max_g=max_g, spatial=spatial, tiles=tiles, lb=lb, tpc=tpc, route=route,
                smem=smem, aligned=aligned, base_ok=base_ok,
                bulk=any(base_ok) and any(aligned), fallback=(not all(base_ok)) or (not all(aligned)),
                misaligned_base=not all(base_ok))


# ------------------------------------------------------------------------------------------------
# bipartite events
# ------------------------------------------------------------------------------------------------
def rd_f32(x):
    """__double2float_rd."""
    f = np.float32(x)
    if float(f) > x:
        f = np.nextafter(f, np.float32(-np.inf))
    return float(f)


def exact_sim(cfg, g):
    """The oracle's float64 IoU matrix of one image (G x P) and its ground-truth corner boxes."""
    enc = oracle_encoder(cfg)
    lab = np.asarray(g, np.float64).reshape(-1, 5).copy()
    if cfg.get('normalize_coords', True):
        lab[:, [2, 4]] /= cfg['img_height']
        lab[:, [1, 3]] /= cfg['img_width']
    co = cfg.get('coords', 'centroids')
    bp = cfg.get('border_pixels', 'half')
    if co == 'centroids':
        lab = convert_coordinates(lab, 1, 'corners2centroids', border_pixels=bp)
    elif co == 'minmax':
        lab = convert_coordinates(lab, 1, 'corners2minmax')
    with np.errstate(all='ignore'):
        sim = iou(lab[:, 1:5], enc.anchors, coords=co, mode='outer_product', border_pixels=bp)
    if co == 'centroids':
        gc = convert_coordinates(lab[:, 1:5], 0, 'centroids2corners')
    elif co == 'minmax':
        gc = lab[:, [1, 3, 2, 4]]
    else:
        gc = lab[:, 1:5]
    return sim, gc


def lower_bounds(cfg, tiles, sim, gc):
    """enc_lb_kernel: rd_f32 of the best exact IoU over the anchors of the tiles whose bounding box holds the box centre."""
    anc = _anchor_corners(cfg)
    out = []
    for g in range(sim.shape[0]):
        cx, cy = 0.5 * (gc[g, 0] + gc[g, 2]), 0.5 * (gc[g, 1] + gc[g, 3])
        best = 0.0
        for t in tiles:
            idx = np.array([a for a, _ in t['map']])
            a = anc[idx]
            if a[:, 0].min() <= cx <= a[:, 2].max() and a[:, 1].min() <= cy <= a[:, 3].max():
                v = sim[g, idx]
                v = v[v > 0]
                if v.size:
                    best = max(best, float(v.max()))
        out.append(rd_f32(best))
    return out


def _row_best(row, removed):
    v = np.where(row > 0, row, 0.0).copy()
    if removed:
        v[list(removed)] = 0.0
    a = int(np.argmax(v))
    return (float(v[a]), a) if v[a] > 0 else (0.0, 0)


def bipartite_events(cfg, g, tiles, lb_on):
    """Replays finish_image on the exact IoU matrix of one image.  Returns the events of the matching stage: conflict or not,
    loop iterations (as count(8, ...) counts them, final pass included), victims per iteration, rows that fell to zero, C2
    searches, C1 re-scans of another tile ('yes' / 'no' / 'undetermined' per victim) and the matches[0] quirk."""
    sim, gc = exact_sim(cfg, g)
    G = sim.shape[0]
    ev = dict(G=G, conflict=False, iterations=0, victims=[], to_zero=0, c2=0, c1_other=[], quirk_noconflict=False,
              quirk_loop=False)
    if G == 0:
        return ev
    tile_of = {}
    for t_i, t in enumerate(tiles):
        for a, _ in t['map']:
            tile_of[a] = t_i
    lbs = lower_bounds(cfg, tiles, sim, gc) if lb_on else [0.0] * G
    rv, ra = [], []
    for gg in range(G):
        v, a = _row_best(sim[gg], ())
        rv.append(v); ra.append(a)
    dup = any(rv[gg] > 0 and any(rv[g2] > 0 and ra[g2] == ra[gg] for g2 in range(gg)) for gg in range(G))
    if not dup:
        ev['quirk_noconflict'] = any(not (v > 0) for v in rv)
        return ev
    ev['conflict'] = True
    removed = []
    while True:
        ev['iterations'] += 1
        f, key_f = -1, None
        for gg in range(G):
            if not rv[gg] > 0:
                continue
            has = any(g2 != gg and rv[g2] > 0 and ra[g2] == ra[gg] and (rv[g2] < rv[gg] or (rv[g2] == rv[gg] and g2 > gg))
                      for g2 in range(G))
            if has and (key_f is None or (-rv[gg], gg) < key_f):
                f, key_f = gg, (-rv[gg], gg)
        fv = rv[f] if f >= 0 else 0.0
        a_star = ra[f] if f >= 0 else -1
        for gg in range(G):
            if rv[gg] > 0 and (f < 0 or gg == f or rv[gg] > fv or (rv[gg] == fv and gg < f)):
                removed.append(ra[gg]); rv[gg] = 0.0; ra[gg] = 0
        if f < 0:
            break
        vict = [gg for gg in range(G) if rv[gg] > 0 and ra[gg] == a_star]
        ev['victims'].append(len(vict))
        rem = set(removed)
        for gg in vict:
            T, ta = _row_best(sim[gg], rem)
            # C1 again: a taken prior outside a*'s tile beats every prior left, and its tile certainly recorded it
            st = tile_of[a_star]
            beats = [r for r in rem if tile_of[r] != st and sim[gg, r] > 0 and (sim[gg, r] > T or (sim[gg, r] == T and r < ta))]
            if not beats:
                ev['c1_other'].append('no')
            elif all(sim[gg, r] >= lbs[gg] for r in beats) or not lb_on:
                ev['c1_other'].append('yes')
            else:
                ev['c1_other'].append('undetermined')
            if T < lbs[gg]:
                ev['c2'] += 1
            if not T > 0:
                ev['to_zero'] += 1
            rv[gg], ra[gg] = T, ta
    ev['quirk_loop'] = len(removed) < G
    return ev


def paths(c, gts, sm_count=132):
    """(host decisions, set of reached path names, per-image bipartite events)."""
    L = host_decisions(c, gts, sm_count)
    cfg = config(c)
    reached = {'spatial' if L['spatial'] else 'linear', 'lb' if L['lb'] else 'no_lb', 'tpc%d' % L['tpc'], 'route_' + L['route']}
    if L['bulk']:
        reached.add('store_bulk')
    if L['fallback']:
        reached.add('store_fallback')
    if L['misaligned_base']:
        reached.add('base_misaligned')
    if all(L['base_ok']):
        reached.add('base_aligned')
    if L['smem'] > 48 * 1024:
        reached.add('smem_over_48k_' + ('inline' if L['route'] == 'inline' else 'offsets_dev'))
    enc = oracle_encoder(cfg)
    thr = min(enc.pos_iou_threshold, enc.neg_iou_limit) if enc.matching_type == 'multi' else enc.neg_iou_limit
    if not (thr > 0):
        reached.add('thr_adj_0')
    if cfg.get('matching_type', 'multi') == 'multi' and cfg['pos_iou_threshold'] > 1:
        reached.add('no_multi_matches')
    if cfg.get('matching_type', 'multi') == 'bipartite':
        reached.add('bipartite_type')
    if c['gt64']:
        reached.add('labels_f64')
    events = []
    for g in distinct(c, gts):
        ev = bipartite_events(cfg, g, L['tiles'], L['lb'])
        events.append(ev)
        if ev['G'] == 0:
            continue
        if ev['G'] == 1:
            reached.add('g1')
        if 129 <= ev['G'] <= 255:
            reached.add('g_nparts1')
        if ev['G'] > TILE:
            reached.add('g_over_256')
        reached.add('conflict' if ev['conflict'] else 'no_conflict')
        if ev['iterations'] >= 4:
            reached.add('conflict_chain')
        if 'yes' in ev['c1_other']:
            reached.add('c1_other_tile')
        if ev['c2']:
            reached.add('c2_search')
        if ev['to_zero']:
            reached.add('victim_to_zero')
        if ev['quirk_noconflict']:
            reached.add('zero_row_quirk_no_conflict')
        if ev['quirk_loop']:
            reached.add('zero_row_quirk_loop')
    return L, reached, events


# path -> the case that reaches it
REQUIRED = {
    'linear': 'g1', 'spatial': 'ssd300_spatial', 'lb': 'forced_linear_lb', 'no_lb': 'forced_spatial_nolb',
    'tpc1': 'g1', 'tpc2': 'tpc2', 'tpc4': 'forced_tpc4', 'tpc8': 'tpc8',
    'route_inline': 'g1', 'route_ring': 'ring', 'route_device': 'device_upper_bounds',
    'store_bulk': 'g1', 'store_fallback': 'ssd300_spatial', 'base_aligned': 'g1', 'base_misaligned': 'out_offset',
    'smem_over_48k_inline': 'c80_inline', 'smem_over_48k_offsets_dev': 'c80_device',
    'no_conflict': 'g1', 'conflict': 'chain4', 'conflict_chain': 'chain4', 'c1_other_tile': 'c1_other_tile',
    'c2_search': 'chain4_lb', 'victim_to_zero': 'tozero', 'zero_row_quirk_no_conflict': 'zero_rows',
    'zero_row_quirk_loop': 'tozero', 'g1': 'g1', 'g_nparts1': 'g150', 'g_over_256': 'g300', 'thr_adj_0': 'thr0_neg0',
    'no_multi_matches': 'no_multi_pos', 'bipartite_type': 'bipartite_only', 'labels_f64': 'thr_at_corners_f64',
}

# the pinned-ring route: B = 1100 on the tiny configuration, ten launches with different boxes
RING = case('ring', 'tiny', ('random', 50, 1100, 2))
RING_SEEDS = tuple(range(50, 60))
BY_NAME['ring'] = RING
