// SSDInputEncoder hot path on sm_90a: pairwise IoU, greedy bipartite + multi matching, neutral boxes and offset
// encoding.  Reference: ssd_encoder_decoder/ssd_input_encoder.py:277-418,
// bounding_box_utils/bounding_box_utils.py:283-383, ssd_encoder_decoder/matching_utils.py:22-116.
//
// enc_tiles_kernel   ONE launch per batch, grid (tile groups, images).  A tile is <= 256 anchors: 256 consecutive priors
//                    ("linear" tile set) or a compact block of feature-map cells ("spatial" tile set: fewer ground-truth
//                    boxes touch a tile; threads are ordered box-shape-major so that the anchors of one shape share warps).
//   1. per image: ground-truth boxes -> template coordinates / corner boxes in float64 (shared memory, once per CTA).
//   2. per tile: ordered list of the boxes whose extent can touch the tile's bounding box.
//   3. per (anchor, candidate): a RIGOROUS float32 upper bound U of the float64 IoU (directed rounding on
//      outward-rounded corners, MUFU reciprocal with a safety factor).  The reference's float64 arithmetic is evaluated
//      -- operation for operation, non-contracting intrinsics -- only where a decision can depend on it:
//        * U reaches min(pos_iou_threshold, neg_iou_limit): the pair may matter for the anchor's own row;
//        * U reaches a lower bound LB[g] of the best IoU ground-truth box g has with ANY anchor: the pair may be the
//          row maximum match_bipartite_greedy looks for.  (Anchors that lie inside a large box all have IoU
//          area_anchor / area_box up to rounding noise, and np.argmax picks the first maximum of that noise: those few
//          hundred pairs per box must be exact, the other ~99.5 % need not.)
//      Exact per-(box, tile) bests (value, first prior index) and the per-(box, tile) maximum of U go to global memory.
//   4. the (C+12)-float target rows are staged in shared memory and leave with cp.async.bulk (one bulk store per
//      contiguous run of priors; plain coalesced stores when a run is not 16-byte aligned).
//   5. the LAST CTA of an image (atomic ticket) runs match_bipartite_greedy for that image: one thread per box reduces the
//      tile bests to the exact row maxima; the G greedy rounds commute when no two boxes compete for the same anchor
//      (the common case); otherwise the reference's sequential rounds run, incl. its zeroed-row quirk, re-evaluating only
//      the tile of a taken anchor (and, if a row falls below its LB, the tiles in descending-U order); then the <= G
//      rows whose bipartite match overrides the multi-match row are rewritten.
// enc_lb_kernel      (only for images with many boxes) LB[g] = best exact IoU of box g among the anchors of the tiles whose
//                    bounding box contains the box centre.  Any exact IoU is a valid lower bound: the choice of tiles
//                    affects speed, never the result.  With few boxes per image LB = 0 (every overlapping pair is exact).
// Exactness: every decision is taken on float64 values computed with the reference's operation order; float32 is only
// used for bounds that can skip work, never for a comparison the result depends on.
#include "common.cuh"
#include "tc.cuh"
#include <climits>
#include <cmath>
#include <vector>

using namespace ssdk;

namespace {

constexpr int kTile = 256;      // anchor slots per tile == threads per CTA
constexpr int kMaxRuns = 16;    // contiguous prior runs per tile
constexpr int kRunRec = 1 + 2 * kMaxRuns;
constexpr int kInlineB = 1024;  // batch sizes up to this pass the ground-truth offsets as a kernel argument (no H2D copy)
// the matching stage's event counters (SSDK_ENC_COUNTERS): conflict-loop iterations, victims, below-bound searches, images
enum { EV_ITERATIONS, EV_VICTIMS, EV_BELOW_BOUND, EV_IMAGES, kEvents };

struct EncParams {
  const double* anchors;        // [P*4] template coords (format = coords)
  int P, C, bg, coords, multi, d, normalize;
  double pos_thr, neg_lim, img_w, img_h;
  double var[4];
  float thr_adj;                // pairs whose IoU bound is below this cannot change an anchor's row
};

struct EncScratch {             // per call, global memory; TG = total number of ground-truth boxes in the batch
  double* tV;                   // [n_tiles*TG] best EXACT IoU among the evaluated pairs (0: none)
  int* tI;                      // [n_tiles*TG] its prior index (lowest on ties)
  const float* lb;              // [TG] lower bound of each box's row maximum, or NULL (= 0)
  int* counters;                // [B] tickets
  int TG;
  unsigned long long* events;   // SSDK_ENC_COUNTERS=1: [kEvents] counts of the matching stage, summed over images, else NULL
};

struct TileSetDev {
  int n_tiles;
  int linear;                   // 1: tile t holds priors [256 t, 256 t + 256), thread == staging slot, one run: nothing to load
  const int2* map;              // [n_tiles*kTile] (prior index of a thread or -1, its staging slot)
  const int* runs;              // [n_tiles*kRunRec]: n_runs, then (first prior, length) pairs; staging slots follow run order
  const int* tile_of;           // [P] tile of a prior
  const unsigned* aligned_mask; // [ceil(n_tiles/32)] bit t: every run of tile t starts and ends on a 16-byte boundary of an image's rows
  const double* bbox;           // [n_tiles*4] corner bounding box of the tile's anchors
  const float4* cls;            // [n_tiles*8*2] per 32-thread slice of a tile: (min x0, min y0, max x1, max y1) rounded outwards |
                                //               (max width, max height) rounded up, min area rounded down, -
};

struct OffsArg { int v[kInlineB + 1]; };

struct Box { double x0, y0, x1, y1, area; };

__device__ __forceinline__ Box corners_from_template(const double t[4], int coords, int d) {
  Box b;
  if (coords == SSDK_COORDS_CENTROIDS) {            // convert_coordinates 'centroids2corners' (:76-80)
    double hw = __ddiv_rn(t[2], 2.0), hh = __ddiv_rn(t[3], 2.0);
    b.x0 = __dsub_rn(t[0], hw); b.y0 = __dsub_rn(t[1], hh);
    b.x1 = __dadd_rn(t[0], hw); b.y1 = __dadd_rn(t[1], hh);
  } else if (coords == SSDK_COORDS_MINMAX) {
    b.x0 = t[0]; b.x1 = t[1]; b.y0 = t[2]; b.y1 = t[3];
  } else {
    b.x0 = t[0]; b.y0 = t[1]; b.x1 = t[2]; b.y1 = t[3];
  }
  // area uses d, the intersection never does (reference quirk, bounding_box_utils.py:345,373-374)
  b.area = __dmul_rn(__dadd_rn(__dsub_rn(b.x1, b.x0), (double)d), __dadd_rn(__dsub_rn(b.y1, b.y0), (double)d));
  return b;
}

// Ground-truth row (class,xmin,ymin,xmax,ymax), float32 or float64 pixels.
__device__ __forceinline__ void load_gt(const void* gt, int f64, size_t row, double r[5]) {
  if (f64) {
    const double* q = reinterpret_cast<const double*>(gt) + row * 5;
#pragma unroll
    for (int k = 0; k < 5; ++k) r[k] = q[k];
  } else {
    const float* q = reinterpret_cast<const float*>(gt) + row * 5;
#pragma unroll
    for (int k = 0; k < 5; ++k) r[k] = (double)q[k];
  }
}

// -> template coords in `coords` format (ssd_input_encoder.py:330-347).  Returns false for a degenerate box (:333).
__device__ __forceinline__ bool gt_template(const double r[5], const EncParams& p, double t[4], int& cls) {
  double xmin = r[1], ymin = r[2], xmax = r[3], ymax = r[4];
  cls = (int)r[0];
  bool ok = (__dsub_rn(xmax, xmin) > 0.0) && (__dsub_rn(ymax, ymin) > 0.0);
  if (p.normalize) {
    ymin = __ddiv_rn(ymin, p.img_h); ymax = __ddiv_rn(ymax, p.img_h);
    xmin = __ddiv_rn(xmin, p.img_w); xmax = __ddiv_rn(xmax, p.img_w);
  }
  if (p.coords == SSDK_COORDS_CENTROIDS) {          // 'corners2centroids' with border_pixels (:71-75)
    t[0] = __ddiv_rn(__dadd_rn(xmin, xmax), 2.0);
    t[1] = __ddiv_rn(__dadd_rn(ymin, ymax), 2.0);
    t[2] = __dadd_rn(__dsub_rn(xmax, xmin), (double)p.d);
    t[3] = __dadd_rn(__dsub_rn(ymax, ymin), (double)p.d);
  } else if (p.coords == SSDK_COORDS_MINMAX) {
    t[0] = xmin; t[1] = xmax; t[2] = ymin; t[3] = ymax;
  } else {
    t[0] = xmin; t[1] = ymin; t[2] = xmax; t[3] = ymax;
  }
  return ok;
}

__device__ __forceinline__ double inter_area(const Box& a, const Box& b) {
  double iw = __dsub_rn(fmin(a.x1, b.x1), fmax(a.x0, b.x0));
  double ih = __dsub_rn(fmin(a.y1, b.y1), fmax(a.y0, b.y0));
  if (!(iw > 0.0) || !(ih > 0.0)) return 0.0;
  return __dmul_rn(iw, ih);
}
// union as NumPy forms it: (area_gt + area_anchor) - inter
__device__ __forceinline__ double union_area(const Box& g, const Box& a, double inter) {
  return __dsub_rn(__dadd_rn(g.area, a.area), inter);
}
__device__ __forceinline__ double iou_value(const Box& g, const Box& a, double inter) {
  return __ddiv_rn(inter, union_area(g, a, inter));
}

__device__ __forceinline__ void load_anchor_t(const EncParams& p, int a, double at[4]) {
  const double2* q = reinterpret_cast<const double2*>(p.anchors + (size_t)a * 4);
  double2 u = __ldg(q), v = __ldg(q + 1);
  at[0] = u.x; at[1] = u.y; at[2] = v.x; at[3] = v.y;
}
__device__ __forceinline__ Box load_anchor(const EncParams& p, int a) {
  double t[4];
  load_anchor_t(p, a, t);
  return corners_from_template(t, p.coords, p.d);
}


// ------------------------------------------------------------------------------------------
// IoU matrix (tests / microbench): out[g*P + a], bit-exact float64.
// ------------------------------------------------------------------------------------------
__global__ void iou_matrix_kernel(EncParams p, const float* __restrict__ gt, int G, double* __restrict__ out) {
  int a = blockIdx.x * blockDim.x + threadIdx.x;
  int g = blockIdx.y;
  if (a >= p.P || g >= G) return;
  double r[5], t[4]; int cls;
  load_gt(gt, 0, (size_t)g, r);
  gt_template(r, p, t, cls);
  Box gb = corners_from_template(t, p.coords, p.d);
  Box ab = load_anchor(p, a);
  double inter = inter_area(gb, ab);
  out[(size_t)g * p.P + a] = __ddiv_rn(inter, union_area(gb, ab, inter));
}

__global__ void iou_general_kernel(const double* __restrict__ b1, int m, const double* __restrict__ b2, int n, int coords,
                                   int d, int elementwise, double* __restrict__ out) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = elementwise ? (long long)(m > n ? m : n) : (long long)m * n;
  if (i >= total) return;
  int r1, r2;
  if (elementwise) { r1 = (m == 1) ? 0 : (int)i; r2 = (n == 1) ? 0 : (int)i; }
  else { r1 = (int)(i / n); r2 = (int)(i % n); }
  double t1[4] = {b1[r1 * 4], b1[r1 * 4 + 1], b1[r1 * 4 + 2], b1[r1 * 4 + 3]};
  double t2[4] = {b2[r2 * 4], b2[r2 * 4 + 1], b2[r2 * 4 + 2], b2[r2 * 4 + 3]};
  Box a = corners_from_template(t1, coords, d), b = corners_from_template(t2, coords, d);
  // np.maximum(0, ...) keeps a zero side at exactly 0, so inter is 0 (not negative) for disjoint boxes
  double iw = fmax(0.0, __dsub_rn(fmin(a.x1, b.x1), fmax(a.x0, b.x0)));
  double ih = fmax(0.0, __dsub_rn(fmin(a.y1, b.y1), fmax(a.y0, b.y0)));
  double inter = __dmul_rn(iw, ih);
  out[i] = __ddiv_rn(inter, __dsub_rn(__dadd_rn(a.area, b.area), inter));
}

// ------------------------------------------------------------------------------------------
// target rows
// ------------------------------------------------------------------------------------------
struct RowDecision { int match_g; bool neutral; };

// One target row [one-hot class | 4 offsets | 4 anchor coords | 4 variances] (ssd_input_encoder.py:363,396-410) in compact form:
// the class vector has at most one 1 (index `one`, -1: none).
struct RowCompact { int one; float o4[4]; };
__device__ __forceinline__ RowCompact make_row(const EncParams& p, const void* gt, int gt_f64, int g0, const double at[4],
                                               RowDecision dec) {
  RowCompact r;
  r.one = -1; r.o4[0] = r.o4[1] = r.o4[2] = r.o4[3] = 0.f;
  if (dec.match_g >= 0) {
    double raw[5], gtc[4]; int cls;
    load_gt(gt, gt_f64, (size_t)(g0 + dec.match_g), raw);
    gt_template(raw, p, gtc, cls);
    if (cls >= 0 && cls < p.C) r.one = cls;
    if (p.coords == SSDK_COORDS_CENTROIDS) {                // :396-400
      r.o4[0] = (float)__ddiv_rn(__dsub_rn(gtc[0], at[0]), __dmul_rn(at[2], p.var[0]));
      r.o4[1] = (float)__ddiv_rn(__dsub_rn(gtc[1], at[1]), __dmul_rn(at[3], p.var[1]));
      r.o4[2] = (float)__ddiv_rn(log(__ddiv_rn(gtc[2], at[2])), p.var[2]);
      r.o4[3] = (float)__ddiv_rn(log(__ddiv_rn(gtc[3], at[3])), p.var[3]);
    } else if (p.coords == SSDK_COORDS_CORNERS) {           // :401-405
      double w = __dsub_rn(at[2], at[0]), h = __dsub_rn(at[3], at[1]);
      r.o4[0] = (float)__ddiv_rn(__ddiv_rn(__dsub_rn(gtc[0], at[0]), w), p.var[0]);
      r.o4[1] = (float)__ddiv_rn(__ddiv_rn(__dsub_rn(gtc[1], at[1]), h), p.var[1]);
      r.o4[2] = (float)__ddiv_rn(__ddiv_rn(__dsub_rn(gtc[2], at[2]), w), p.var[2]);
      r.o4[3] = (float)__ddiv_rn(__ddiv_rn(__dsub_rn(gtc[3], at[3]), h), p.var[3]);
    } else {                                                // minmax :406-410
      double w = __dsub_rn(at[1], at[0]), h = __dsub_rn(at[3], at[2]);
      r.o4[0] = (float)__ddiv_rn(__ddiv_rn(__dsub_rn(gtc[0], at[0]), w), p.var[0]);
      r.o4[1] = (float)__ddiv_rn(__ddiv_rn(__dsub_rn(gtc[1], at[1]), w), p.var[1]);
      r.o4[2] = (float)__ddiv_rn(__ddiv_rn(__dsub_rn(gtc[2], at[2]), h), p.var[2]);
      r.o4[3] = (float)__ddiv_rn(__ddiv_rn(__dsub_rn(gtc[3], at[3]), h), p.var[3]);
    }
    if (dec.neutral && r.one == p.bg) r.one = -1;           // neg_iou_limit <= 0 corner case: the background entry is zeroed last
  } else if (!dec.neutral) {
    r.one = p.bg;
  }
  return r;
}
__device__ __forceinline__ void emit_row(const EncParams& p, const void* gt, int gt_f64, int g0, const double at[4],
                                         RowDecision dec, float* dst) {
  const RowCompact r = make_row(p, gt, gt_f64, g0, at, dec);
  for (int c = 0; c < p.C; ++c) dst[c] = (c == r.one) ? 1.f : 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    dst[p.C + k] = r.o4[k];
    dst[p.C + 4 + k] = (float)at[k];
    dst[p.C + 8 + k] = (float)p.var[k];
  }
}

// (value desc, index asc) warp reduction
__device__ __forceinline__ void warp_argmax(double& val, int& idx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double ov = __shfl_xor_sync(0xffffffffu, val, o);
    int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ov > val || (ov == val && oi < idx)) { val = ov; idx = oi; }
  }
}

// ------------------------------------------------------------------------------------------
// tiles
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int tile_anchor(const TileSetDev& ts, int tile, int s, int P, int& pos) {
  if (ts.linear) { const int a = tile * kTile + s; pos = s; return a < P ? a : -1; }
  const int2 m = __ldg(ts.map + (size_t)tile * kTile + s);
  pos = m.y;
  return m.x;
}
__device__ __forceinline__ int tile_of_prior(const TileSetDev& ts, int a) { return ts.linear ? a / kTile : __ldg(ts.tile_of + a); }

__device__ __forceinline__ bool is_removed(const int* removed, int n, int a) {
  bool r = false;
  for (int i = 0; i < n; ++i) r |= (removed[i] == a);
  return r;
}

// Upper bound (can only err upwards) of the float64 IoU between ANY anchor of a 32-thread slice (bounds k0, k1 of
// TileSetDev::cls) and a box given by outward-rounded float32 corners gf and its area rounded down.
__device__ __forceinline__ float slice_iou_bound(const float4 k0, const float4 k1, const float4 gf, float g_area) {
  const float ox = fmaxf(fminf(fminf(k1.x, __fsub_ru(gf.z, gf.x)), fminf(__fsub_ru(k0.z, gf.x), __fsub_ru(gf.z, k0.x))), 0.f);
  const float oy = fmaxf(fminf(fminf(k1.y, __fsub_ru(gf.w, gf.y)), fminf(__fsub_ru(k0.w, gf.y), __fsub_ru(gf.w, k0.y))), 0.f);
  const float inter = __fmul_ru(ox, oy);
  const float un = fmaxf(__fsub_rd(__fadd_rd(k1.z, g_area), inter), 1e-30f);
  return __fmul_ru(__fmul_ru(inter, rcp_approx(un)), 1.0f + 4.76837158203125e-7f);          // (1 + 2^-21): the reciprocal's ulp
}

// One warp: the exact best anchor of `gb` over ALL slices of all tiles, ignoring `removed`, starting from a known candidate
// (out_v, out_i) (0 / INT_MAX for none).  Lanes test 32 slice bounds at a time; a slice is evaluated exactly (one anchor per
// lane) only while its bound reaches the best value found so far.  Used when a row falls below its lower bound after losing
// its prior: pairs under that bound were never evaluated by the tile pass.
__device__ void warp_row_best(const EncParams& p, const TileSetDev& ts, const Box& gb, const int* removed, int n_removed,
                              double& out_v, int& out_i, int part, int nparts) {
  // (this warp takes every nparts-th batch of 32 slices; four batches of bounds are computed before any is acted on, so their
  //  loads overlap)
  const int lane = threadIdx.x & 31;
  const float4 gf = make_float4(__double2float_rd(gb.x0), __double2float_rd(gb.y0), __double2float_ru(gb.x1), __double2float_ru(gb.y1));
  const float g_area = __double2float_rd(gb.area);
  double best = out_v; int bidx = out_i;
  const int n_slices = ts.n_tiles * (kTile / 32);
  for (int base0 = part * 32; base0 < n_slices; base0 += nparts * 32 * 4) {
    float bound[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int sidx = base0 + u * nparts * 32 + lane;
      bound[u] = -1.f;
      if (sidx < n_slices) bound[u] = slice_iou_bound(__ldg(ts.cls + (size_t)sidx * 2), __ldg(ts.cls + (size_t)sidx * 2 + 1), gf, g_area);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int base = base0 + u * nparts * 32;
      unsigned m = __ballot_sync(0xffffffffu, bound[u] > 0.f && (double)bound[u] >= best);
      while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        const int sl = base + src;
        int pos;
        const int a = tile_anchor(ts, sl / (kTile / 32), (sl % (kTile / 32)) * 32 + lane, p.P, pos);
        double v = 0.0; int vi = INT_MAX;
        if (a >= 0) {
          const Box ab = load_anchor(p, a);
          const double inter = inter_area(gb, ab);
          if (inter > 0.0) {
            const double iv = iou_value(gb, ab, inter);
            if (iv > 0.0 && !is_removed(removed, n_removed, a)) { v = iv; vi = a; }
          }
        }
        warp_argmax(v, vi);
        if (v > best || (v == best && v > 0.0 && vi < bidx)) { best = v; bidx = vi; }
        m &= __ballot_sync(0xffffffffu, (double)bound[u] >= best);   // the rest of this batch against the improved best
      }
    }
  }
  out_v = best; out_i = bidx;
}

// ------------------------------------------------------------------------------------------
// enc_lb_kernel: lower bounds of the row maxima (one warp per ground-truth box)
// ------------------------------------------------------------------------------------------
template <bool INLINE_OFFS>
__global__ void __launch_bounds__(kTile) enc_lb_kernel(const __grid_constant__ EncParams p, const __grid_constant__ TileSetDev ts,
                                                       const __grid_constant__ OffsArg offs_arg, const int* __restrict__ offs_dev,
                                                       const void* __restrict__ gt, int gt_f64, float* __restrict__ lb) {
  const int b = blockIdx.y;
  const int g0 = INLINE_OFFS ? offs_arg.v[b] : offs_dev[b];
  const int G = (INLINE_OFFS ? offs_arg.v[b + 1] : offs_dev[b + 1]) - g0;
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * (kTile / 32) + (threadIdx.x >> 5);
  if (g >= G) return;
  double r[5], t[4]; int cls;
  load_gt(gt, gt_f64, (size_t)(g0 + g), r);
  gt_template(r, p, t, cls);
  const Box gb = corners_from_template(t, p.coords, p.d);
  const double cx = 0.5 * (gb.x0 + gb.x1), cy = 0.5 * (gb.y0 + gb.y1);
  const float4 gf = make_float4(__double2float_rd(gb.x0), __double2float_rd(gb.y0), __double2float_ru(gb.x1), __double2float_ru(gb.y1));
  const float g_area = __double2float_rd(gb.area);
  double best = 0.0;
  for (int base = 0; base < ts.n_tiles; base += 32) {
    const int tile = base + lane;
    bool inside = false;
    if (tile < ts.n_tiles) {
      const double* bb = ts.bbox + (size_t)tile * 4;
      inside = bb[0] <= cx && cx <= bb[2] && bb[1] <= cy && cy <= bb[3];
    }
    unsigned m = __ballot_sync(0xffffffffu, inside);
    while (m) {
      const int src = __ffs(m) - 1;
      m &= m - 1;
      // only the slices of that tile whose bound still reaches the best value found so far (lanes 0..7 test one slice each);
      // any evaluated anchor gives a valid lower bound, so skipping slices can only loosen it
      const int t = base + src;
      float bound = -1.f;
      if (lane < kTile / 32)
        bound = slice_iou_bound(__ldg(ts.cls + ((size_t)t * (kTile / 32) + lane) * 2), __ldg(ts.cls + ((size_t)t * (kTile / 32) + lane) * 2 + 1), gf, g_area);
      unsigned ms = __ballot_sync(0xffffffffu, bound > 0.f && (double)bound >= best);
      while (ms) {
        const int w = __ffs(ms) - 1;
        ms &= ms - 1;
        int pos;
        const int a = tile_anchor(ts, t, w * 32 + lane, p.P, pos);
        double v = 0.0;
        if (a >= 0) {
          const Box ab = load_anchor(p, a);
          const double inter = inter_area(gb, ab);
          if (inter > 0.0) { v = iou_value(gb, ab, inter); if (!(v > 0.0)) v = 0.0; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
        best = fmax(best, v);
        ms &= __ballot_sync(0xffffffffu, (double)bound >= best);
      }
    }
  }
  if (lane == 0) lb[g0 + g] = __double2float_rd(best);
}

// ------------------------------------------------------------------------------------------
// match_bipartite_greedy (matching_utils.py:63-77), run by the last CTA of an image
// ------------------------------------------------------------------------------------------
__device__ void finish_image(const EncParams& p, const TileSetDev& ts, const EncScratch& sc, const void* gt, int gt_f64, int g0, int G,
                             int b, const double* s_gbox, unsigned char* scratch, double* pv, int* pi, float* __restrict__ out_y,
                             int* __restrict__ out_match) {
  __shared__ int s_flag[2];
  double* rv = reinterpret_cast<double*>(scratch);           // [G] current row maximum
  int* ra = reinterpret_cast<int*>(rv + G);                   // [G] its (first) prior index
  int* removed = ra + G;                                      // [G] priors taken so far
  int* matches = removed + G;                                 // [G]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int W = p.C + 12, TG = sc.TG;
  auto count = [&](int slot, int n) { if (sc.events && tid == 0 && n) atomicAdd(sc.events + slot, (unsigned long long)n); };
  auto gbox = [&](int g) {
    Box q; q.x0 = s_gbox[g * 5]; q.y0 = s_gbox[g * 5 + 1]; q.x1 = s_gbox[g * 5 + 2]; q.y1 = s_gbox[g * 5 + 3]; q.area = s_gbox[g * 5 + 4];
    return q;
  };
  // exact row maxima over the tile bests: kTile / G threads per box (each scans every nparts-th tile, eight loads in flight),
  // combined through shared memory; consecutive threads read consecutive boxes
  {
    const int nparts = G < kTile ? (kTile / G < kTile / 32 ? kTile / G : kTile / 32) : 1;       // <= 8: pv / pi hold 8 * G entries
    for (int gbase = 0; gbase < G; gbase += kTile) {
      const int g = gbase + (nparts > 1 ? tid % G : tid), part = nparts > 1 ? tid / G : 0;
      double bv = 0.0; int bi = INT_MAX;
      if (g < G && part < nparts) {
        const size_t col = (size_t)(g0 + g);
#pragma unroll 8
        for (int t = part; t < ts.n_tiles; t += nparts) {
          const double v = __ldcg(sc.tV + (size_t)t * TG + col);
          const int i = __ldcg(sc.tI + (size_t)t * TG + col);
          if (v > 0.0 && (v > bv || (v == bv && i < bi))) { bv = v; bi = i; }
        }
        pv[part * G + g] = bv; pi[part * G + g] = bi;
      }
      __syncthreads();
      if (g < G && part == 0) {
        for (int q = 1; q < nparts; ++q) {
          const double v = pv[q * G + g]; const int i = pi[q * G + g];
          if (v > 0.0 && (v > bv || (v == bv && i < bi))) { bv = v; bi = i; }
        }
        rv[g] = bv; ra[g] = (bv > 0.0) ? bi : 0;                  // argmax of an all-zero row is 0
      }
      __syncthreads();
    }
  }
  if (tid == 0) { s_flag[0] = 0; s_flag[1] = 0; }
  __syncthreads();
  for (int g = tid; g < G; g += kTile) {
    if (!(rv[g] > 0.0)) { s_flag[1] = 1; continue; }           // an all-zero row: the zero rounds come last and hit matches[0]
    const int a = ra[g];
    for (int g2 = 0; g2 < g; ++g2)
      if (rv[g2] > 0.0 && ra[g2] == a) { s_flag[0] = 1; break; }
  }
  __syncthreads();
  if (!s_flag[0]) {
    // no two boxes want the same prior: the G rounds commute, every positive row keeps its arg-max; rounds in which
    // all remaining rows are zero select (gt 0, prior 0) (np.argmax of zeros), and rows never selected keep the initial 0
    for (int g = tid; g < G; g += kTile) matches[g] = ra[g];
    __syncthreads();
    if (tid == 0 && s_flag[1]) matches[0] = 0;
  } else {
    // Some boxes want the same prior.  The reference's G rounds take the rows in descending (row maximum, then ascending box
    // index) order; a round only interferes with later ones by removing the prior a LATER row points at.  So instead of G
    // sequential rounds: find the first row (in that order) that has such a later duplicate, settle every row before it at once
    // (none of them can lose its prior), settle that row, let the duplicates recompute their maximum without the taken priors (one
    // warp each; their value can only drop, so they stay behind the settled rows), and repeat.  One iteration per conflict.
    __shared__ double s_cv[kTile / 32], s_sv[kTile / 32];
    __shared__ int s_ci[kTile / 32], s_si[kTile / 32];
    __shared__ int s_first, s_nrem, s_nvict;
    int* victims = matches + G;                               // [G] rows that lost their prior in this iteration
    for (int g = tid; g < G; g += kTile) matches[g] = 0;
    if (tid == 0) s_nrem = 0;
    __syncthreads();
    for (;;) {
      count(EV_ITERATIONS, 1);
      // A. the first row with a later duplicate
      double cv = -1.0; int ci = INT_MAX;
      for (int g = tid; g < G; g += kTile) {
        const double v = rv[g];
        if (!(v > 0.0)) continue;
        const int a = ra[g];
        bool has = false;
        for (int g2 = 0; g2 < G; ++g2) {
          const double v2 = rv[g2];
          has |= (g2 != g) && (v2 > 0.0) && (ra[g2] == a) && (v2 < v || (v2 == v && g2 > g));
        }
        if (has && (v > cv || (v == cv && g < ci))) { cv = v; ci = g; }
      }
      warp_argmax(cv, ci);
      if (lane == 0) { s_cv[warp] = cv; s_ci[warp] = ci; }
      __syncthreads();
      if (tid == 0) {
        double bv = -1.0; int bi = INT_MAX;
        for (int w = 0; w < kTile / 32; ++w)
          if (s_cv[w] > bv || (s_cv[w] == bv && s_ci[w] < bi)) { bv = s_cv[w]; bi = s_ci[w]; }
        s_first = (bv > 0.0) ? bi : -1;
      }
      __syncthreads();
      const int f = s_first;
      const double fv = f >= 0 ? rv[f] : 0.0;
      const int a_star = f >= 0 ? ra[f] : -1;
      __syncthreads();                                           // everyone has read row f before it is settled
      // B. settle every positive row ahead of f (all of them when there is no conflict left), and f itself
      for (int g = tid; g < G; g += kTile) {
        const double v = rv[g];
        if (!(v > 0.0)) continue;
        if (f < 0 || g == f || v > fv || (v == fv && g < f)) {
          const int a = ra[g];
          matches[g] = a;
          removed[atomicAdd(&s_nrem, 1)] = a;
          rv[g] = 0.0; ra[g] = 0;
        }
      }
      __syncthreads();
      if (f < 0) break;
      // C. the rows that pointed at f's prior recompute their maximum (one warp per row)
      const int n_removed = s_nrem;
      if (tid == 0) s_nvict = 0;
      __syncthreads();
      for (int g = tid; g < G; g += kTile)
        if (rv[g] > 0.0 && ra[g] == a_star) victims[atomicAdd(&s_nvict, 1)] = g;
      __syncthreads();
      const int n_vict = s_nvict;
      count(EV_VICTIMS, n_vict);
      // C1. per row, all eight warps together: re-evaluate the tile of the lost prior without the taken priors (one 32-anchor
      // slice per warp) while every thread looks at one or two of the other tiles' recorded bests; repeat while the new best is
      // itself a taken prior recorded by another tile
      for (int vi = 0; vi < n_vict; ++vi) {
        const int gg = victims[vi];
        const size_t col = (size_t)(g0 + gg);
        const Box gb = gbox(gg);
        int stale = a_star;
        for (;;) {                                              // (uniform over the CTA)
          const int st = tile_of_prior(ts, stale);
          // this warp's slice of tile st
          double tv = 0.0; int ti = INT_MAX;
          {
            int pos;
            const int a = tile_anchor(ts, st, warp * 32 + lane, p.P, pos);
            if (a >= 0) {
              const Box ab = load_anchor(p, a);
              const double inter = inter_area(gb, ab);
              if (inter > 0.0) {
                const double v = iou_value(gb, ab, inter);
                if (v > 0.0 && !is_removed(removed, n_removed, a)) { tv = v; ti = a; }
              }
            }
          }
          // this thread's share of the other tiles
          double nv = 0.0; int ni = INT_MAX;
          for (int t = tid; t < ts.n_tiles; t += kTile) {
            if (t == st) continue;
            const double v2 = __ldcg(sc.tV + (size_t)t * TG + col);
            const int i2 = __ldcg(sc.tI + (size_t)t * TG + col);
            if (v2 > 0.0 && (v2 > nv || (v2 == nv && i2 < ni))) { nv = v2; ni = i2; }
          }
          warp_argmax(tv, ti);
          warp_argmax(nv, ni);
          if (lane == 0) { s_cv[warp] = tv; s_ci[warp] = ti; s_sv[warp] = nv; s_si[warp] = ni; }
          __syncthreads();
          if (tid == 0) {
            double bt = 0.0; int it = INT_MAX, io = INT_MAX; double bo = 0.0;
            for (int w = 0; w < kTile / 32; ++w) {
              if (s_cv[w] > bt || (s_cv[w] == bt && s_cv[w] > 0.0 && s_ci[w] < it)) { bt = s_cv[w]; it = s_ci[w]; }
              if (s_sv[w] > bo || (s_sv[w] == bo && s_sv[w] > 0.0 && s_si[w] < io)) { bo = s_sv[w]; io = s_si[w]; }
            }
            if (!(bt > 0.0)) { bt = 0.0; it = INT_MAX; }
            sc.tV[(size_t)st * TG + col] = bt; sc.tI[(size_t)st * TG + col] = it;
            double nb = bt; int nib = it;
            if (bo > nb || (bo == nb && bo > 0.0 && io < nib)) { nb = bo; nib = io; }
            const bool again = (nb > 0.0) && is_removed(removed, n_removed, nib);
            s_first = again ? nib : -1;                          // (s_first is free in this part of the iteration)
            if (!again) { pv[vi] = (nb > 0.0) ? nb : 0.0; pi[vi] = (nb > 0.0) ? nib : INT_MAX; }
          }
          __syncthreads();
          const int nxt = s_first;
          __syncthreads();                                       // everyone has read the verdict before the next round overwrites it
          if (nxt < 0) break;
          stale = nxt;
        }
      }
      __syncthreads();
      // C2. pairs below a row's lower bound were never evaluated by the tile pass: a row whose best that is left fell below it is
      // searched over all slices, by all warps together
      for (int vi = 0; vi < n_vict; ++vi) {
        const int gg = victims[vi];
        const float lbg = sc.lb ? __ldg(sc.lb + g0 + gg) : 0.f;
        double nv = pv[vi]; int ni = pi[vi];
        if (!(nv < (double)lbg)) continue;                       // uniform over the CTA
        count(EV_BELOW_BOUND, 1);
        warp_row_best(p, ts, gbox(gg), removed, n_removed, nv, ni, warp, kTile / 32);
        if (lane == 0) { s_cv[warp] = nv; s_ci[warp] = ni; }
        __syncthreads();
        if (tid == 0) {
          double bv = 0.0; int bi = INT_MAX;
          for (int w = 0; w < kTile / 32; ++w)
            if (s_cv[w] > bv || (s_cv[w] == bv && s_cv[w] > 0.0 && s_ci[w] < bi)) { bv = s_cv[w]; bi = s_ci[w]; }
          pv[vi] = bv; pi[vi] = bi;
        }
        __syncthreads();
      }
      for (int vi = tid; vi < n_vict; vi += kTile) {
        const int gg = victims[vi];
        const double nv = pv[vi];
        rv[gg] = nv; ra[gg] = (nv > 0.0) ? pi[vi] : 0;
      }
      __syncthreads();
    }
    if (tid == 0 && s_nrem < G) matches[0] = 0;                  // rounds with nothing left to match select (box 0, prior 0)
  }
  __syncthreads();
  // y_encoded[i, bipartite_matches, :-8] = labels_one_hot (:363): last writer wins; the matched column is all zero afterwards
  for (int g = tid; g < G; g += kTile) {
    const int a = matches[g];
    bool last = true;
    for (int g2 = g + 1; g2 < G; ++g2) last &= (matches[g2] != a);
    if (!last) continue;
    double at[4];
    load_anchor_t(p, a, at);
    RowDecision dec{g, 0.0 >= p.neg_lim};
    emit_row(p, gt, gt_f64, g0, at, dec, out_y + ((size_t)b * p.P + a) * W);
    if (out_match) out_match[(size_t)b * p.P + a] = g;
  }
  __syncthreads();
  count(EV_IMAGES, 1);
}

// ------------------------------------------------------------------------------------------
// enc_tiles_kernel
// ------------------------------------------------------------------------------------------
struct EncSmem {            // byte offsets inside the dynamic shared memory
  size_t rows, gbox, gf, gq, wU, wV, wI, items, total;
};
__host__ __device__ inline EncSmem enc_smem_layout(int W, int G) {
  EncSmem s;
  const size_t gs = (size_t)(G > 0 ? G : 1);
  size_t rows_bytes = ((size_t)kTile * W * sizeof(float) + 15) & ~(size_t)15;
  const size_t fin = (gs * 24 + 15) & ~(size_t)15;            // finish_image scratch lives in the row staging area
  if (fin > rows_bytes) rows_bytes = fin;
  auto up16 = [](size_t v) { return (v + 15) & ~(size_t)15; };
  s.rows = 0;
  s.gbox = rows_bytes;                                        // [G*5] f64 corner boxes of the ground truth
  s.gf = up16(s.gbox + gs * 40);                              // [G] float4: outward-rounded corners of a box
  s.gq = up16(s.gf + gs * 16);                                // [G] float4: (area rounded down, row-maximum threshold, candidate threshold, -)
  s.wV = up16(s.gq + gs * 16);                                // [8*G] f64: per-slice best exact IoU of a candidate
  s.wU = up16(s.wV + gs * 64);                                // [8*G] u32: per-slice bound of the IoU of a candidate
  s.wI = up16(s.wU + gs * 32);                                // [8*G] i32: per-slice prior index of the best exact IoU
  s.items = up16(s.wI + gs * 32);                             // [8*G] (slice << 16 | box) pairs whose exact per-slice best is needed, + counter
  s.total = up16(s.items + gs * 32 + 16) + 16;
  return s;
}

template <bool INLINE_OFFS>
__global__ void __launch_bounds__(kTile, 3) enc_tiles_kernel(const __grid_constant__ EncParams p, const __grid_constant__ TileSetDev ts,
                                                             const __grid_constant__ OffsArg offs_arg, const int* __restrict__ offs_dev,
                                                             const void* __restrict__ gt, int gt_f64, int tpc,
                                                             const __grid_constant__ EncScratch sc, float* __restrict__ out_y,
                                                             int* __restrict__ out_match, int* __restrict__ status) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ int s_last;
  const int b = blockIdx.y;
  const int g0 = INLINE_OFFS ? offs_arg.v[b] : offs_dev[b];
  const int G = (INLINE_OFFS ? offs_arg.v[b + 1] : offs_dev[b + 1]) - g0;
  const int Gs = G > 0 ? G : 1;
  const int W = p.C + 12, TG = sc.TG;
  const EncSmem L = enc_smem_layout(W, G);
  float* rows = reinterpret_cast<float*>(smem_raw + L.rows);
  double* s_gbox = reinterpret_cast<double*>(smem_raw + L.gbox);
  float4* s_gf = reinterpret_cast<float4*>(smem_raw + L.gf);
  float4* s_gq = reinterpret_cast<float4*>(smem_raw + L.gq);
  double* s_wV = reinterpret_cast<double*>(smem_raw + L.wV);
  unsigned* s_wU = reinterpret_cast<unsigned*>(smem_raw + L.wU);
  int* s_wI = reinterpret_cast<int*>(smem_raw + L.wI);
  int* s_items = reinterpret_cast<int*>(smem_raw + L.items);
  int* s_nitems = s_items + (size_t)(kTile / 32) * Gs;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  const int tile0 = blockIdx.x * tpc;
  const int tile1 = min(ts.n_tiles, tile0 + tpc);
  // the first tile's anchor: issued before anything else so that its latency hides behind the ground-truth set-up
  int pos = 0;
  int a = tile_anchor(ts, tile0, tid, p.P, pos);
  double at[4] = {0, 0, 0, 0};
  if (a >= 0) load_anchor_t(p, a, at);

  // ---- 1. ground truth of this image -> float64 corner boxes ----
  bool bad = false;
  for (int g = tid; g < G; g += kTile) {
    double r[5], t[4]; int cls;
    load_gt(gt, gt_f64, (size_t)(g0 + g), r);
    bad |= !gt_template(r, p, t, cls);
    const Box gb = corners_from_template(t, p.coords, p.d);
    s_gbox[g * 5] = gb.x0; s_gbox[g * 5 + 1] = gb.y0; s_gbox[g * 5 + 2] = gb.x1; s_gbox[g * 5 + 3] = gb.y1; s_gbox[g * 5 + 4] = gb.area;
    // outward-rounded float32 corners, area rounded down: ingredients of IoU bounds that can only err upwards
    s_gf[g] = make_float4(__double2float_rd(gb.x0), __double2float_rd(gb.y0), __double2float_ru(gb.x1), __double2float_ru(gb.y1));
    // a pair needs the exact float64 IoU for the box's row maximum from q_row (the lower bound of that maximum, lowered by more
    // than the bound's own slack; "any overlap at all" when there is none), for the anchor's own row from thr_adj
    float q_row = 1.401298464e-45f;
    if (sc.lb) {
      const float lbg = __ldg(sc.lb + g0 + g);
      if (lbg > 0.f) q_row = fmaxf(q_row, nextafterf(lbg * 0.99999905f, 0.f));
    }
    s_gq[g] = make_float4(__double2float_rd(gb.area), q_row, fminf(q_row, p.thr_adj), 0.f);
  }
  if (tid == 0) *s_nitems = 0;                                  // (warps append right after the barrier below)
  const int any_bad = __syncthreads_or(bad ? 1 : 0);          // also publishes s_gbox
  if (blockIdx.x == 0 && tid == 0 && any_bad && status) atomicMax(status, b + 1);

  bool store_pending = false;
  int prev_one = -1;                                            // staging-row entry this thread set to 1 in the previous tile
  for (int i = tid; i < kTile * W; i += kTile) rows[i] = 0.f;   // (published by the barriers of the first tile)
  for (int tile = tile0; tile < tile1; ++tile) {
    if (tile != tile0) {
      a = tile_anchor(ts, tile, tid, p.P, pos);
      if (a >= 0) load_anchor_t(p, a, at);
    }
    // ---- 2. per 32-anchor slice: which boxes can reach their threshold with ANY anchor of the slice ----
    // Bound of the IoU of a whole slice against a box: the overlap along x is at most min(widest anchor, box width, rightmost anchor
    // edge - box left, box right - leftmost anchor edge), likewise along y; the union is at least smallest anchor area + box area -
    // that intersection.  With the box-shape-major thread order a slice holds one shape at neighbouring positions, so the bound is
    // tight and only the few boxes near the slice survive: the per-anchor loop below runs over ~1 box instead of all that touch the
    // tile, and every warp does the same amount of work here.
    const float4 k0 = __ldg(ts.cls + ((size_t)tile * (kTile / 32) + warp) * 2);
    const float4 k1 = __ldg(ts.cls + ((size_t)tile * (kTile / 32) + warp) * 2 + 1);
    const bool live = a >= 0;
    float fx0 = 0.f, fy0 = 0.f, fx1 = -INFINITY, fy1 = -INFINITY, fa = 0.f;
    Box ab{};
    if (live) {
      ab = corners_from_template(at, p.coords, p.d);
      fx0 = __double2float_rd(ab.x0); fy0 = __double2float_rd(ab.y0);
      fx1 = __double2float_ru(ab.x1); fy1 = __double2float_ru(ab.y1);
      fa = __double2float_rd(ab.area);
    }
    double best = 0.0; int best_g = -1;
    for (int gb0 = 0; gb0 < G; gb0 += 32) {
      const int g = gb0 + lane;
      bool own_f = false;
      if (g < G) {
        const float4 gf = s_gf[g];
        const float4 gq = s_gq[g];
        const float um = slice_iou_bound(k0, k1, gf, gq.x);
        s_wU[warp * Gs + g] = __float_as_uint(um);
        // the slice may hold the box's row maximum: queued for exact evaluation by whichever warp is free (3b); "um >= q_row" is
        // also how the reduction below knows that the slice was evaluated
        if (um >= gq.y) s_items[atomicAdd(s_nitems, 1)] = (warp << 16) | g;
        own_f = um >= p.thr_adj;                                // some anchor of the slice may reach its own-row threshold
      }
      // ---- 3. own rows: rare (a box whose IoU with this slice can reach min(pos_iou_threshold, neg_iou_limit)) ----
      unsigned mo = __ballot_sync(0xffffffffu, own_f);
      while (mo) {                                              // ascending box index: np.argmax keeps the first maximum
        const int g2 = gb0 + __ffs(mo) - 1;
        mo &= mo - 1;
        const float4 gf = s_gf[g2];
        const float ga = s_gq[g2].x;
        // U >= fl64(inter / union): widths and intersection rounded up, union rounded down (directed rounding is monotone)
        const float iw = fmaxf(__fsub_ru(fminf(fx1, gf.z), fmaxf(fx0, gf.x)), 0.f);
        const float ih = fmaxf(__fsub_ru(fminf(fy1, gf.w), fmaxf(fy0, gf.y)), 0.f);
        const float inter = __fmul_ru(iw, ih);
        const float un = fmaxf(__fsub_rd(__fadd_rd(fa, ga), inter), 1e-30f);
        const float U = __fmul_ru(inter, rcp_approx(un));      // within 2^-23 below the bound at worst (thr_adj accounts for it)
        if (live && U >= p.thr_adj) {                           // exact float64 IoU
          Box gb; gb.x0 = s_gbox[g2 * 5]; gb.y0 = s_gbox[g2 * 5 + 1]; gb.x1 = s_gbox[g2 * 5 + 2]; gb.y1 = s_gbox[g2 * 5 + 3]; gb.area = s_gbox[g2 * 5 + 4];
          const double inter64 = inter_area(gb, ab);
          if (inter64 > 0.0) {
            const double val = iou_value(gb, ab, inter64);
            if (val > best) { best = val; best_g = g2; }        // strict '>' keeps the first gt on ties (np.argmax)
          }
        }
      }
    }
    // ---- 3b. exact per-(box, slice) bests, dealt out over all warps ----
    // These evaluations pile up in the slices of the best-fitting anchor shape (every anchor inside a large box ties its row
    // maximum up to rounding): left to their own warps, two of eight would do all of it while six wait at the barrier.
    __syncthreads();
    const int n_items = *s_nitems;
    for (int it = warp; it < n_items; it += kTile / 32) {
      const int w = s_items[it] >> 16, g = s_items[it] & 0xffff;
      int pos2;
      const int a2 = tile_anchor(ts, tile, w * 32 + lane, p.P, pos2);
      double val = 0.0;
      if (a2 >= 0) {
        Box gb; gb.x0 = s_gbox[g * 5]; gb.y0 = s_gbox[g * 5 + 1]; gb.x1 = s_gbox[g * 5 + 2]; gb.y1 = s_gbox[g * 5 + 3]; gb.area = s_gbox[g * 5 + 4];
        const Box ab2 = load_anchor(p, a2);
        const double inter64 = inter_area(gb, ab2);
        if (inter64 > 0.0) { val = iou_value(gb, ab2, inter64); if (!(val > 0.0)) val = 0.0; }
      }
      // best pair of the slice (lowest prior index on ties): REDUX on the two halves of the (non-negative) float64 bit pattern,
      // then on the prior index
      const unsigned hi = (unsigned)__double2hiint(val), lo = (unsigned)__double2loint(val);
      const unsigned mh = __reduce_max_sync(0xffffffffu, hi);
      const unsigned ml = __reduce_max_sync(0xffffffffu, hi == mh ? lo : 0u);
      const bool top = (hi == mh) && (lo == ml) && (val > 0.0);
      const unsigned mi = __reduce_min_sync(0xffffffffu, top ? (unsigned)a2 : 0x7fffffffu);
      if (lane == 0) { s_wV[w * Gs + g] = __hiloint2double((int)mh, (int)ml); s_wI[w * Gs + g] = (int)mi; }
    }
    // the previous tile's bulk store must have finished reading the staging rows before they are rewritten
    if (store_pending && tid == 0) bulk_wait_read<0>();
    __syncthreads();
    if (tid == 0) *s_nitems = 0;                                  // (next appended after the barrier that follows the row stores)
    // ---- per (gt, tile) results -> global (consecutive threads write consecutive boxes) ----
    for (int g = tid; g < G; g += kTile) {
      double bv = 0.0; int bi = INT_MAX;
      const float q_row = s_gq[g].y;
#pragma unroll
      for (int w = 0; w < kTile / 32; ++w) {
        if (__uint_as_float(s_wU[w * Gs + g]) >= q_row) {       // slice w evaluated its pairs with the box exactly ...
          const double v = s_wV[w * Gs + g]; const int i = s_wI[w * Gs + g];
          if (v > bv || (v == bv && v > 0.0 && i < bi)) { bv = v; bi = i; }
        }
      }
      if (!(bv > 0.0)) { bv = 0.0; bi = INT_MAX; }
      const size_t o = (size_t)tile * TG + (size_t)(g0 + g);
      sc.tV[o] = bv; sc.tI[o] = bi;
    }
    // ---- 4. this anchor's row ----
    if (prev_one >= 0) { rows[prev_one] = 0.f; prev_one = -1; }   // (the previous tile's bulk store has finished reading: barrier above)
    // spatial tiles of different shapes map threads to staging slots differently: this thread's previous slot may now be
    // another thread's, whose 1 must not be cleared after it is set
    if (!ts.linear && tile != tile0) __syncthreads();
    if (live) {
      RowDecision dec{-1, false};
      double val = best;
      if (G > 0) {
        const int arg = best_g >= 0 ? best_g : 0;                // np.argmax of an all-zero column is 0
        if (p.multi && val >= p.pos_thr) { dec.match_g = arg; val = 0.0; }   // column zeroed after matching (:381)
        if (val >= p.neg_lim) dec.neutral = true;                            // :388-390
      }
      // the class part of the staging rows is kept all-zero between tiles: set this row's single 1, remember where it went
      const RowCompact r = make_row(p, gt, gt_f64, g0, at, dec);
      float* dst = rows + (size_t)pos * W;
      if (r.one >= 0) { dst[r.one] = 1.f; prev_one = pos * W + r.one; }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        dst[p.C + k] = r.o4[k];
        dst[p.C + 4 + k] = (float)at[k];
        dst[p.C + 8 + k] = (float)p.var[k];
      }
      if (out_match) out_match[(size_t)b * p.P + a] = (dec.match_g >= 0) ? dec.match_g : (dec.neutral ? -2 : -1);
    }
    fence_proxy_async();                                          // generic-proxy writes of the rows -> visible to the bulk copy engine
    __syncthreads();
    // ---- 5. rows leave: one bulk store per contiguous run of priors ----
    // (runs whose byte ranges are not 16-byte aligned fall back to coalesced stores by all threads; whether a tile has any is
    //  known on the host up to the alignment of this image's base address, which is uniform over the CTA)
    const bool base_ok = ((reinterpret_cast<uintptr_t>(out_y + (size_t)b * p.P * W) & 15) == 0);
    const int* rn = ts.linear ? nullptr : ts.runs + (size_t)tile * kRunRec;
    const int lin_len = min(kTile, p.P - tile * kTile);
    const bool fast = base_ok && (ts.linear ? (((size_t)tile * kTile * W * 4) & 15) == 0 && (((size_t)lin_len * W * 4) & 15) == 0
                                            : ((ts.aligned_mask[tile >> 5] >> (tile & 31)) & 1u) != 0);
    bool issued = false;
    if (fast) {
      if (tid == 0) {
        const int nruns = ts.linear ? 1 : rn[0];
        int slot0 = 0;
        for (int r = 0; r < nruns; ++r) {
          const int start = ts.linear ? tile * kTile : rn[1 + 2 * r];
          const int len = ts.linear ? lin_len : rn[2 + 2 * r];
          float* dst = out_y + ((size_t)b * p.P + start) * W;
          bulk_store(dst, smem_u32(rows + (size_t)slot0 * W), (uint32_t)((size_t)len * W * 4));
          slot0 += len;
        }
        bulk_commit();
      }
      issued = true;
    } else {
      const int nruns = ts.linear ? 1 : rn[0];
      int slot0 = 0;
      for (int r = 0; r < nruns; ++r) {
        const int start = ts.linear ? tile * kTile : rn[1 + 2 * r];
        const int len = ts.linear ? lin_len : rn[2 + 2 * r];
        float* dst = out_y + ((size_t)b * p.P + start) * W;
        const float* src = rows + (size_t)slot0 * W;
        const size_t n_f = (size_t)len * W;
        for (size_t i = tid; i < n_f; i += kTile) dst[i] = src[i];
        slot0 += len;
      }
    }
    store_pending = issued;
  }
  // ---- 6. last CTA of the image: bipartite matching ----
  if (tid == 0) bulk_wait<0>();
  if (G <= 0) return;
  __syncthreads();                                              // every thread's global writes happen-before thread 0's fence
  if (tid == 0) {
    __threadfence();
    const int old = atomicAdd(sc.counters + b, 1);
    const int last = (old == (int)gridDim.x - 1);
    if (last) { sc.counters[b] = 0; __threadfence(); }          // ready for the next launch; acquire side of the ticket
    s_last = last;
  }
  __syncthreads();
  if (!s_last) return;
  finish_image(p, ts, sc, gt, gt_f64, g0, G, b, s_gbox, smem_raw + L.rows, s_wV, s_wI, out_y, out_match);
}

__global__ void tile_bbox_kernel(EncParams p, TileSetDev ts, double* __restrict__ bbox, float4* __restrict__ cls) {
  __shared__ double s[4][kTile / 32];
  const int tile = blockIdx.x;
  int pos;
  const int a = tile_anchor(ts, tile, threadIdx.x, p.P, pos);
  double x0 = 1e300, y0 = 1e300, x1 = -1e300, y1 = -1e300;
  if (a >= 0) { Box ab = load_anchor(p, a); x0 = ab.x0; y0 = ab.y0; x1 = ab.x1; y1 = ab.y1; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    x0 = fmin(x0, __shfl_xor_sync(0xffffffffu, x0, o)); y0 = fmin(y0, __shfl_xor_sync(0xffffffffu, y0, o));
    x1 = fmax(x1, __shfl_xor_sync(0xffffffffu, x1, o)); y1 = fmax(y1, __shfl_xor_sync(0xffffffffu, y1, o));
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { s[0][w] = x0; s[1][w] = y0; s[2][w] = x1; s[3][w] = y1; }
  {   // bounds of this 32-thread slice for the IoU bound of a whole slice against a box (enc_tiles_kernel, step 2b)
    double bw = -1e300, bh = -1e300, ar = 1e300;
    if (a >= 0) { Box ab = load_anchor(p, a); bw = __dsub_rn(ab.x1, ab.x0); bh = __dsub_rn(ab.y1, ab.y0); ar = ab.area; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      bw = fmax(bw, __shfl_xor_sync(0xffffffffu, bw, o)); bh = fmax(bh, __shfl_xor_sync(0xffffffffu, bh, o));
      ar = fmin(ar, __shfl_xor_sync(0xffffffffu, ar, o));
    }
    if ((threadIdx.x & 31) == 0) {
      float4 c0, c1;
      if (x0 > x1) {                                            // no anchor in the slice: can never be a candidate
        c0 = make_float4(INFINITY, INFINITY, -INFINITY, -INFINITY); c1 = make_float4(0.f, 0.f, 1.f, 0.f);
      } else {
        c0 = make_float4(__double2float_rd(x0), __double2float_rd(y0), __double2float_ru(x1), __double2float_ru(y1));
        c1 = make_float4(__double2float_ru(bw), __double2float_ru(bh), __double2float_rd(ar), 0.f);
      }
      cls[((size_t)tile * (kTile / 32) + w) * 2] = c0; cls[((size_t)tile * (kTile / 32) + w) * 2 + 1] = c1;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < kTile / 32; ++i) { x0 = fmin(x0, s[0][i]); y0 = fmin(y0, s[1][i]); x1 = fmax(x1, s[2][i]); y1 = fmax(y1, s[3][i]); }
    bbox[tile * 4 + 0] = x0; bbox[tile * 4 + 1] = y0; bbox[tile * 4 + 2] = x1; bbox[tile * 4 + 3] = y1;
  }
}

// ------------------------------------------------------------------------------------------
// host side: tile sets
// ------------------------------------------------------------------------------------------
struct TileSetHost {
  std::vector<int> map, pos, runs;      // map/pos per thread slot
  int n_tiles = 0;
  int fill = 0;
  void begin_tile() { runs.resize((size_t)(n_tiles + 1) * kRunRec, 0); map.resize((size_t)(n_tiles + 1) * kTile, -1); pos.resize(map.size(), 0); fill = 0; }
  // a run of `cells` feature-map cells x nb boxes starting at prior `start`; `cell0` = cells already in this tile, `ncells` = cells
  // the finished tile will hold: thread = box * ncells + cell (box-shape-major), staging slot = run order
  void add_run(int start, int cells, int nb, int cell0, int ncells) {
    int* r = runs.data() + (size_t)n_tiles * kRunRec;
    r[1 + 2 * r[0]] = start; r[2 + 2 * r[0]] = cells * nb; ++r[0];
    for (int c = 0; c < cells; ++c)
      for (int bx = 0; bx < nb; ++bx) {
        const int thread = bx * ncells + cell0 + c;
        map[(size_t)n_tiles * kTile + thread] = start + c * nb + bx;
        pos[(size_t)n_tiles * kTile + thread] = fill + c * nb + bx;
      }
    fill += cells * nb;
  }
  void end_tile() { ++n_tiles; }
};

void linear_layer_tiles(TileSetHost& t, int first, int count) {
  for (int o = 0; o < count; o += kTile) {
    t.begin_tile();
    const int n = std::min(kTile, count - o);
    t.add_run(first + o, n, 1, 0, n);
    t.end_tile();
  }
}

// Compact blocks of feature-map cells per predictor layer (prior index = off + (y*W + x)*nb + box).
void spatial_tiles(TileSetHost& t, int n_layers, const int* fh, const int* fw, const int* nbx) {
  int off = 0;
  for (int l = 0; l < n_layers; ++l) {
    const int H = fh[l], Wd = fw[l], nb = nbx[l];
    const int count = H * Wd * nb;
    if (nb > kTile || nb <= 0) { linear_layer_tiles(t, off, count); off += count; continue; }
    const int cells_max = kTile / nb;
    int bw = (int)std::floor(std::sqrt((double)cells_max));
    if (bw < 1) bw = 1;
    if (bw >= Wd) {                                            // whole rows fit: a tile is bh full rows = one contiguous run
      const int bh = std::max(1, std::min(H, cells_max / Wd));
      for (int y0 = 0; y0 < H; y0 += bh) {
        const int rws = std::min(bh, H - y0);
        t.begin_tile();
        t.add_run(off + y0 * Wd * nb, rws * Wd, nb, 0, rws * Wd);
        t.end_tile();
      }
    } else {
      const int bh = std::max(1, std::min(std::min(H, cells_max / bw), kMaxRuns));
      for (int y0 = 0; y0 < H; y0 += bh)
        for (int x0 = 0; x0 < Wd; x0 += bw) {
          const int cw = std::min(bw, Wd - x0), ch = std::min(bh, H - y0);
          t.begin_tile();
          for (int y = 0; y < ch; ++y) t.add_run(off + ((y0 + y) * Wd + x0) * nb, cw, nb, y * cw, cw * ch);
          t.end_tile();
        }
    }
    off += count;
  }
}

struct TileSetOwned {
  TileSetDev dev{};
  int2* d_map = nullptr; int* d_runs = nullptr; int* d_tile_of = nullptr; double* d_bbox = nullptr; unsigned* d_mask = nullptr; float4* d_cls = nullptr;
  void release() {
    cudaFree(d_map); cudaFree(d_runs); cudaFree(d_tile_of); cudaFree(d_bbox); cudaFree(d_mask); cudaFree(d_cls); d_cls = nullptr;
    d_map = nullptr; d_runs = d_tile_of = nullptr; d_bbox = nullptr; d_mask = nullptr; dev = TileSetDev{};
  }
};

}  // namespace

struct ssdk_encoder {
  ssdk_ctx* ctx = nullptr;
  ssdk_encode_cfg cfg{};
  EncParams p{};
  double* d_anchors = nullptr;
  TileSetOwned linear, spatial;     // spatial.dev.n_tiles == 0: no layer geometry was given
  Scratch tiles;                    // per-(gt, tile) bounds and exact bests, per-gt lower bounds
  Scratch counters;                 // per-image tickets (self-resetting)
  size_t counters_n = 0;
  Scratch events;                   // the matching stage's event counts, allocated by the first call with SSDK_ENC_COUNTERS=1
  Scratch offsets;                  // device copy of the offsets for batches larger than kInlineB
  HostRing<8> offsets_ring;         // pinned staging of those offsets
  OffsArg offs_arg{};               // ground-truth offsets passed by value with the launch (B <= kInlineB)
};

namespace {

int upload_tiles(ssdk_encoder* e, const TileSetHost* h, int n_linear_tiles, TileSetOwned& o) {
  const int n_tiles = h ? h->n_tiles : n_linear_tiles;
  SSDK_CHECK_CUDA(cudaMalloc(&o.d_bbox, (size_t)n_tiles * 4 * sizeof(double)));
  SSDK_CHECK_CUDA(cudaMalloc(&o.d_cls, (size_t)n_tiles * (kTile / 32) * 2 * sizeof(float4)));
  o.dev.n_tiles = n_tiles; o.dev.linear = h ? 0 : 1;
  if (h) {
    std::vector<int2> m(h->map.size());
    std::vector<int> tile_of((size_t)e->p.P, 0);
    for (size_t i = 0; i < m.size(); ++i) {
      m[i] = make_int2(h->map[i], h->pos[i]);
      if (h->map[i] >= 0) tile_of[h->map[i]] = (int)(i / kTile);
    }
    SSDK_CHECK_CUDA(cudaMalloc(&o.d_map, m.size() * sizeof(int2)));
    SSDK_CHECK_CUDA(cudaMalloc(&o.d_runs, h->runs.size() * sizeof(int)));
    SSDK_CHECK_CUDA(cudaMalloc(&o.d_tile_of, tile_of.size() * sizeof(int)));
    SSDK_CHECK_CUDA(cudaMemcpy(o.d_map, m.data(), m.size() * sizeof(int2), cudaMemcpyHostToDevice));
    SSDK_CHECK_CUDA(cudaMemcpy(o.d_runs, h->runs.data(), h->runs.size() * sizeof(int), cudaMemcpyHostToDevice));
    SSDK_CHECK_CUDA(cudaMemcpy(o.d_tile_of, tile_of.data(), tile_of.size() * sizeof(int), cudaMemcpyHostToDevice));
    // a tile's rows can leave by bulk copies iff every run's byte range (relative to the image's first row) is 16-byte aligned
    const int W = e->p.C + 12;
    std::vector<unsigned> mask((h->n_tiles + 31) / 32, 0u);
    for (int t = 0; t < h->n_tiles; ++t) {
      const int* r = h->runs.data() + (size_t)t * kRunRec;
      bool ok = ((size_t)e->p.P * W) % 4 == 0;                 // image stride
      int slot0 = 0;
      for (int i = 0; i < r[0] && ok; ++i) {
        ok = (((size_t)r[1 + 2 * i] * W * 4) % 16 == 0) && (((size_t)r[2 + 2 * i] * W * 4) % 16 == 0) && (((size_t)slot0 * W * 4) % 16 == 0);
        slot0 += r[2 + 2 * i];
      }
      if (ok) mask[t >> 5] |= 1u << (t & 31);
    }
    SSDK_CHECK_CUDA(cudaMalloc(&o.d_mask, mask.size() * sizeof(unsigned)));
    SSDK_CHECK_CUDA(cudaMemcpy(o.d_mask, mask.data(), mask.size() * sizeof(unsigned), cudaMemcpyHostToDevice));
    o.dev.map = o.d_map; o.dev.runs = o.d_runs; o.dev.tile_of = o.d_tile_of; o.dev.aligned_mask = o.d_mask;
  }
  o.dev.bbox = o.d_bbox;
  o.dev.cls = o.d_cls;
  return launch(e->ctx, tile_bbox_kernel, n_tiles, kTile, 0, nullptr, e->p, o.dev, o.d_bbox, o.d_cls);
}

// every prior exactly once, every thread's staging slot inside its tile's runs exactly once
bool tiles_cover(const TileSetHost& h, int P) {
  std::vector<char> seen((size_t)P, 0);
  for (int t = 0; t < h.n_tiles; ++t) {
    std::vector<char> slot(kTile, 0);
    int fill = 0;
    const int* r = h.runs.data() + (size_t)t * kRunRec;
    for (int i = 0; i < r[0]; ++i) fill += r[2 + 2 * i];
    if (fill > kTile || r[0] > kMaxRuns) return false;
    for (int s = 0; s < kTile; ++s) {
      const int a = h.map[(size_t)t * kTile + s];
      if (a < 0) continue;
      const int ps = h.pos[(size_t)t * kTile + s];
      if (a >= P || seen[a] || ps < 0 || ps >= fill || slot[ps]) return false;
      seen[a] = 1; slot[ps] = 1;
      // the staging slot must be the prior's place in run order
      int base = 0, want = -1;
      for (int i = 0; i < r[0]; ++i) {
        if (a >= r[1 + 2 * i] && a < r[1 + 2 * i] + r[2 + 2 * i]) { want = base + (a - r[1 + 2 * i]); break; }
        base += r[2 + 2 * i];
      }
      if (want != ps) return false;
    }
  }
  for (char c : seen) if (!c) return false;
  return true;
}

}  // namespace

extern "C" int ssdk_encoder_create(ssdk_ctx* ctx, const ssdk_encode_cfg* cfg, const double* anchors_host, ssdk_encoder** out) {
  SSDK_REQUIRE(ctx && cfg && anchors_host && out, "ssdk_encoder_create: NULL argument");
  SSDK_REQUIRE(cfg->P > 0 && cfg->n_classes_total > 1, "ssdk_encoder_create: bad P / n_classes");
  SSDK_REQUIRE(cfg->coords >= 0 && cfg->coords <= 2, "Unexpected value for `coords`. Supported values are 'minmax', 'corners' and 'centroids'.");
  SSDK_REQUIRE(cfg->background_id >= 0 && cfg->background_id < cfg->n_classes_total, "background_id out of range");
  for (int i = 0; i < 4; ++i) SSDK_REQUIRE(cfg->variances[i] > 0, "All variances must be >0");
  SSDK_CHECK_CUDA(cudaSetDevice(ctx->device));
  ssdk_encoder* e = new ssdk_encoder();
  e->ctx = ctx; e->cfg = *cfg;
  e->cfg.fm_height = e->cfg.fm_width = e->cfg.n_boxes = nullptr;     // the caller's arrays are only read here
  EncParams& p = e->p;
  p.P = cfg->P; p.C = cfg->n_classes_total; p.bg = cfg->background_id;
  p.coords = cfg->coords; p.multi = cfg->matching_multi; p.d = cfg->border_d; p.normalize = cfg->normalize_coords;
  p.pos_thr = cfg->pos_iou_threshold; p.neg_lim = cfg->neg_iou_limit;
  p.img_w = (double)cfg->img_width; p.img_h = (double)cfg->img_height;
  for (int i = 0; i < 4; ++i) p.var[i] = cfg->variances[i];
  {
    // a pair can change an anchor's row only if its IoU reaches the smaller of the thresholds that are tested (:375,389);
    // the float32 bound is compared against a value safely below it (the bound may be 2^-23 short of the true maximum)
    double thr = p.multi ? std::min(p.pos_thr, p.neg_lim) : p.neg_lim;
    float t = 0.f;
    if (thr > 0.0 && std::isfinite(thr)) {
      t = (float)(thr * (1.0 - 9.5367431640625e-7));           // 1 - 2^-20
      t = std::nextafterf(t, 0.f);
      if (!(t > 0.f)) t = 0.f;
    }
    p.thr_adj = t;                                             // 0: every pair is evaluated exactly
  }
  auto fail = [&](int code) { ssdk_encoder_destroy(e); return code; };
  if (cudaMalloc(&e->d_anchors, (size_t)p.P * 4 * sizeof(double)) != cudaSuccess) { set_error("ssdk_encoder_create: cudaMalloc failed"); return fail(SSDK_ERR_NOMEM); }
  if (cudaMemcpy(e->d_anchors, anchors_host, (size_t)p.P * 4 * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess) {
    set_error("ssdk_encoder_create: anchor upload failed"); return fail(SSDK_ERR_CUDA);
  }
  p.anchors = e->d_anchors;
  int rc = upload_tiles(e, nullptr, ceil_div(p.P, kTile), e->linear);
  if (rc) return fail(rc);
  if (cfg->n_layers > 0 && cfg->fm_height && cfg->fm_width && cfg->n_boxes) {
    long long tot = 0;
    for (int l = 0; l < cfg->n_layers; ++l) tot += (long long)cfg->fm_height[l] * cfg->fm_width[l] * cfg->n_boxes[l];
    if (tot != p.P) { set_error("ssdk_encoder_create: layer geometry describes %lld priors, P is %d", tot, p.P); return fail(SSDK_ERR_INVALID); }
    TileSetHost h;
    spatial_tiles(h, cfg->n_layers, cfg->fm_height, cfg->fm_width, cfg->n_boxes);
    if (!tiles_cover(h, p.P)) { set_error("internal: spatial tiles do not cover the priors exactly once"); return fail(SSDK_ERR_INVALID); }
    rc = upload_tiles(e, &h, 0, e->spatial); if (rc) return fail(rc);
  }
  if (cudaDeviceSynchronize() != cudaSuccess) { set_error("ssdk_encoder_create: tile setup failed"); return fail(SSDK_ERR_CUDA); }
  *out = e;
  return SSDK_OK;
}

extern "C" int ssdk_encoder_destroy(ssdk_encoder* e) {
  if (!e) return SSDK_OK;
  cudaFree(e->d_anchors);
  e->linear.release(); e->spatial.release();
  e->tiles.release(); e->counters.release(); e->events.release(); e->offsets.release();
  e->offsets_ring.release();
  delete e;
  return SSDK_OK;
}

extern "C" int ssdk_iou_matrix(ssdk_encoder* e, const float* gt_boxes_dev, int G, double* out_dev, void* stream) {
  SSDK_REQUIRE(e && gt_boxes_dev && out_dev && G > 0, "ssdk_iou_matrix: bad argument");
  return launch(e->ctx, iou_matrix_kernel, dim3(ceil_div(e->p.P, 256), G), 256, 0, (cudaStream_t)stream, e->p, gt_boxes_dev, G, out_dev);
}

extern "C" int ssdk_iou(ssdk_ctx* ctx, const double* boxes1_dev, int m, const double* boxes2_dev, int n, int coords, int border_d,
                        int elementwise, double* out_dev, void* stream) {
  SSDK_REQUIRE(ctx && boxes1_dev && boxes2_dev && out_dev && m > 0 && n > 0, "ssdk_iou: bad argument");
  SSDK_REQUIRE(coords >= 0 && coords <= 2, "Unexpected value for `coords`. Supported values are 'minmax', 'corners' and 'centroids'.");
  SSDK_REQUIRE(!elementwise || m == n || m == 1 || n == 1, "ssdk_iou: element-wise mode needs broadcast-compatible box counts");
  long long total = elementwise ? (long long)(m > n ? m : n) : (long long)m * n;
  return launch(ctx, iou_general_kernel, (unsigned)ceil_div_ll(total, 256), 256, 0, (cudaStream_t)stream, boxes1_dev, m, boxes2_dev, n,
                coords, border_d, elementwise, out_dev);
}

namespace {

int scan_offsets(const int* offs, int B, int* total_g, int* max_g) {
  SSDK_REQUIRE(offs[0] == 0 && offs[B] >= 0, "ssdk_encode: gt_offsets must start at 0 and be non-decreasing");
  int mg = 0;
  for (int b = 0; b < B; ++b) {
    const int g = offs[b + 1] - offs[b];
    SSDK_REQUIRE(g >= 0, "ssdk_encode: gt_offsets must be non-decreasing");
    mg = g > mg ? g : mg;
  }
  *total_g = offs[B]; *max_g = mg;
  return SSDK_OK;
}

}  // namespace

// Exactly one of offs_host / offs_dev (B+1 ints).  Host offsets are scanned for total_g / max_g; with device offsets the caller
// gives them, and the rows must be float32 (float64 rows with device offsets have no caller).
extern "C" int ssdk_encode(ssdk_encoder* e, const void* gt_dev, int gt_f64, const int* offs_host, const int* offs_dev, int B,
                           int total_g, int max_g, float* out_y_dev, int* out_match_dev, int* status_dev, void* stream_) {
  SSDK_REQUIRE(e && (offs_host != nullptr) != (offs_dev != nullptr) && out_y_dev && B > 0, "ssdk_encode: bad argument");
  if (offs_host) {
    const int rc = scan_offsets(offs_host, B, &total_g, &max_g);
    if (rc) return rc;
  } else {
    SSDK_REQUIRE(total_g >= 0 && max_g >= 0, "ssdk_encode: bad argument");
    SSDK_REQUIRE(!gt_f64, "ssdk_encode: float64 rows need host offsets");
  }
  cudaStream_t stream = (cudaStream_t)stream_;
  const EncParams& p = e->p;
  const int W = p.C + 12;
  SSDK_REQUIRE(total_g == 0 || gt_dev, "ssdk_encode: gt_boxes_dev is NULL");
  SSDK_REQUIRE((reinterpret_cast<uintptr_t>(out_y_dev) & 3) == 0, "ssdk_encode: out_y_dev is not float aligned");
  // tile set: compact cell blocks pay off once many boxes compete per tile; consecutive priors give full tiles, one aligned
  // run each and nothing to look up, which is what matters when the kernel is purely store / latency bound
  int spatial_min = 24, lb_min = 17;
  if (int rc = env_int("SSDK_ENC_SPATIAL_MIN", spatial_min, &spatial_min)) return rc;
  if (int rc = env_int("SSDK_ENC_LB_MIN", lb_min, &lb_min)) return rc;
  const bool use_spatial = e->spatial.dev.n_tiles > 0 && max_g >= spatial_min;
  const TileSetDev& ts = use_spatial ? e->spatial.dev : e->linear.dev;
  const bool use_lb = max_g >= lb_min && total_g > 0;
  int tpc = max_g <= 16 ? 1 : (max_g <= 48 ? 2 : (max_g < 96 ? 4 : 8));   // tiles per CTA: amortises the per-CTA box set-up (measured)
  if (int rc = env_int("SSDK_ENC_TPC", tpc, &tpc)) return rc;
  tpc = std::max(1, tpc);
  int counters;
  if (int rc = env_int("SSDK_ENC_COUNTERS", 0, &counters)) return rc;
  while (tpc > 1 && (long long)ceil_div(ts.n_tiles, tpc) * B < 8ll * e->ctx->sm_count) tpc >>= 1;
  // scratch: tV (f64) | tI (i32) each [n_tiles * TG], lb [TG]
  const size_t TG = (size_t)(total_g > 0 ? total_g : 1);
  const size_t nt = TG * (size_t)ts.n_tiles;
  int rc = e->tiles.ensure(nt * 12 + TG * 4 + 64);
  if (rc) return rc;
  EncScratch sc{};
  sc.tV = reinterpret_cast<double*>(e->tiles.ptr);
  sc.tI = reinterpret_cast<int*>(sc.tV + nt);
  float* lb = reinterpret_cast<float*>(sc.tI + nt);
  sc.lb = use_lb ? lb : nullptr;
  sc.TG = (int)TG;
  if (counters) {
    rc = e->events.ensure(kEvents * sizeof(unsigned long long));
    if (rc) return rc;
    sc.events = reinterpret_cast<unsigned long long*>(e->events.ptr);
    SSDK_CHECK_CUDA(cudaMemsetAsync(sc.events, 0, kEvents * sizeof(unsigned long long), stream));
  }
  if (e->counters_n < (size_t)B) {
    SSDK_CHECK_CUDA(cudaStreamSynchronize(stream));
    rc = e->counters.ensure((size_t)B * sizeof(int));
    if (rc) return rc;
    SSDK_CHECK_CUDA(cudaMemset(e->counters.ptr, 0, e->counters.bytes));
    e->counters_n = e->counters.bytes / sizeof(int);
  }
  sc.counters = reinterpret_cast<int*>(e->counters.ptr);
  const EncSmem L = enc_smem_layout(W, max_g);
  SSDK_REQUIRE(L.total <= 227 * 1024, "ssdk_encode: n_classes (%d) / gt count (%d) need %zu bytes of shared memory", p.C, max_g, L.total);
  // enc_tiles_kernel takes all of it as dynamic shared memory: if (L.total > 48 * 1024), ssdk::launch raises the kernel's limit first
  dim3 grid(ceil_div(ts.n_tiles, tpc), B);
  dim3 grid_lb(ceil_div(max_g, kTile / 32), B);
  const bool inline_offs = offs_host != nullptr && B <= kInlineB;
  const int* d_offs = nullptr;
  if (inline_offs) {
    memcpy(e->offs_arg.v, offs_host, (size_t)(B + 1) * sizeof(int));
  } else if (offs_dev) {
    d_offs = offs_dev;
  } else {                                                 // large batch with host offsets: pinned ring + async copy
    rc = e->offsets.ensure((size_t)(B + 1) * sizeof(int));
    if (rc) return rc;
    rc = e->offsets_ring.upload(e->offsets.ptr, stream, {{offs_host, (size_t)(B + 1) * sizeof(int)}});
    if (rc) return rc;
    d_offs = reinterpret_cast<const int*>(e->offsets.ptr);
  }
  if (use_lb) {
    rc = launch(e->ctx, inline_offs ? enc_lb_kernel<true> : enc_lb_kernel<false>, grid_lb, kTile, 0, stream,
                p, ts, e->offs_arg, d_offs, gt_dev, gt_f64, lb);
    if (rc) return rc;
  }
  rc = launch(e->ctx, inline_offs ? enc_tiles_kernel<true> : enc_tiles_kernel<false>, grid, kTile, L.total, stream,
              p, ts, e->offs_arg, d_offs, gt_dev, gt_f64, tpc, sc, out_y_dev, out_match_dev, status_dev);
  if (rc) return rc;
  if (sc.events) {                                              // synchronises
    unsigned long long h[kEvents];
    SSDK_CHECK_CUDA(cudaMemcpyAsync(h, sc.events, sizeof(h), cudaMemcpyDeviceToHost, stream));
    SSDK_CHECK_CUDA(cudaStreamSynchronize(stream));
    const double n = h[EV_IMAGES] ? (double)h[EV_IMAGES] : 1.0;
    fprintf(stderr, "enc matching stage, per image: iterations %.1f victims %.1f below-bound searches %.1f (images %llu)\n",
            h[EV_ITERATIONS] / n, h[EV_VICTIMS] / n, h[EV_BELOW_BOUND] / n, h[EV_IMAGES]);
  }
  return SSDK_OK;
}
