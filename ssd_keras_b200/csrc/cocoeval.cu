// pycocotools' COCOeval for iouType 'bbox' on the device: evaluateImg's greedy matching (cocoapi PythonAPI/pycocotools/
// cocoeval.py, the IoU of common/maskApi.c bbIou) and accumulate's precision / recall / score tables.
//
//   coco_match_kernel       one 64-thread CTA per (image, category) segment that has ground truths or detections.  The
//                           segment's detection x ground-truth IoUs go into a shared float64 tile when they fit (IOU_TILE), else
//                           each scan recomputes them (the same operations, so the same values).  Each (area range, threshold)
//                           pair is one thread's greedy scan over the detections in score order, with its own matched flags.
//                           The area range only moves its ignored ground truths behind the others (evaluateImg's stable sort), so
//                           a scan walks the non-ignored ones, then the ignored ones, in input order.
//   coco_accumulate_kernel  one CTA per (threshold, category, area range, maxDet) of the output.  It walks the category's
//                           detections in accumulate's order (score desc, image, rank in the image), the rank < maxDet
//                           subsequence of one order made for the largest maxDet: a pass for the totals, then the chunks from the
//                           last one back, so that tp / fp cumulative counts come from suffix sums and the right-to-left running
//                           maximum of the precision is a scan in the same direction.  A detection at which the recall rises
//                           claims the recall thresholds in (previous recall, its recall]: that is searchsorted(rc, thr, 'left').
//
// Every value is taken in float64 with the rn intrinsics, as the reference computes it (the C of bbIou is assumed to be the usual
// x86-64 build, which has no FMA to contract into).
#include "common.cuh"
#include "rn.cuh"
#include <cfloat>
#include <cmath>

using namespace ssdk;

namespace {

constexpr int MATCH_THREADS = 64;
constexpr int IOU_TILE = 2048;               // doubles of the shared IoU tile: 16 KB
constexpr int ACC_THREADS = 256;
constexpr int ACC_WARPS = ACC_THREADS / 32;

// bbIou for one (detection, ground truth) pair of [x, y, w, h] boxes.  fmin / fmax ignore a NaN operand, as C's do.
__device__ __forceinline__ double bb_iou(const double* d, const double* g, bool crowd) {
  const double w = sub_rn(fmin(add_rn(d[2], d[0]), add_rn(g[2], g[0])), fmax(d[0], g[0]));
  if (w <= 0) return 0.0;
  const double h = sub_rn(fmin(add_rn(d[3], d[1]), add_rn(g[3], g[1])), fmax(d[1], g[1]));
  if (h <= 0) return 0.0;
  const double i = mul_rn(w, h), da = mul_rn(d[2], d[3]);
  const double u = crowd ? da : sub_rn(add_rn(da, mul_rn(g[2], g[3])), i);
  return div_rn(i, u);
}

// evaluateImg's ignore flag of a ground truth for the range [lo, hi]: crowd, or an area outside it (both bounds inclusive)
__device__ __forceinline__ bool gt_ignored(unsigned char flags, double area, double lo, double hi) {
  return (flags & 1) || area < lo || area > hi;
}

__global__ void __launch_bounds__(MATCH_THREADS) coco_match_kernel(ssdk_coco_match a) {
  extern __shared__ double s_iou[];
  const int s = blockIdx.x;
  const int g0 = a.seg_gt[s], G = a.seg_gt[s + 1] - g0;
  const int d0 = a.seg_det[s], D = a.seg_det[s + 1] - d0;
  const unsigned char* gfl = a.gt_flags + g0;
  const double* garea = a.gt_area + g0;
  for (int r = threadIdx.x; r < a.n_area; r += MATCH_THREADS) {
    const double lo = a.area_rng[2 * r], hi = a.area_rng[2 * r + 1];
    int n = 0;
    for (int g = 0; g < G; ++g) n += gt_ignored(gfl[g], garea[g], lo, hi) ? 0 : 1;
    a.seg_npig[(size_t)s * a.n_area + r] = n;
    if (n) atomicAdd(&a.npig[a.seg_cat[s] * a.n_area + r], n);
  }
  const bool tiled = (long long)D * G <= IOU_TILE;
  if (tiled)
    for (int x = threadIdx.x; x < D * G; x += MATCH_THREADS) {
      const int dd = x / G, g = x - dd * G;
      s_iou[x] = bb_iou(a.det_box + (size_t)(d0 + dd) * 4, a.gt_box + (size_t)(g0 + g) * 4, gfl[g] & 1);
    }
  __syncthreads();
  const int AT = a.n_area * a.n_thr;
  for (int at = threadIdx.x; at < AT; at += MATCH_THREADS) {
    const int r = at / a.n_thr, t = at - r * a.n_thr;
    const double lo = a.area_rng[2 * r], hi = a.area_rng[2 * r + 1];
    const double cap = 1.0 - 1e-10, thr0 = a.iou_thrs[t];
    const double thr = cap < thr0 ? cap : thr0;                 // min([t, 1 - 1e-10])
    unsigned char* matched = a.gt_matched + (size_t)at * a.n_gt + g0;
    const size_t out = (size_t)at * a.n_det + d0;
    for (int dd = 0; dd < D; ++dd) {
      double best = thr;
      int m = -1;
      // pass 0: the non-ignored ground truths; pass 1, the ignored tail, is reached only without a match in pass 0 (a match
      // there is non-ignored, and the reference breaks at the first ignored ground truth it does not skip)
      for (int pass = 0; pass < 2 && (pass == 0 || m < 0); ++pass)
        for (int g = 0; g < G; ++g) {
          const unsigned char f = gfl[g];
          if ((int)gt_ignored(f, garea[g], lo, hi) != pass) continue;
          if (matched[g] && !(f & 1)) continue;                // already matched and not a crowd box
          const double v = tiled ? s_iou[dd * G + g] : bb_iou(a.det_box + (size_t)(d0 + dd) * 4, a.gt_box + (size_t)(g0 + g) * 4, f & 1);
          if (v < best) continue;                               // so the last of several equal IoUs wins
          best = v;
          m = g;
        }
      bool nonzero = false, ignored = false;                    // dtm != 0 (a ground truth with id 0 reads as unmatched), dtIg
      if (m >= 0) {
        matched[m] = 1;
        nonzero = !(gfl[m] & 2);
        ignored = gt_ignored(gfl[m], garea[m], lo, hi);
      }
      const double da = a.det_area[d0 + dd];
      if (!nonzero && (da < lo || da > hi)) ignored = true;
      a.det_flags[out + dd] = (unsigned char)((nonzero ? 1 : 0) | (ignored ? 2 : 0));
      a.det_match[out + dd] = m >= 0 ? g0 + m : -1;
    }
  }
}

// Inclusive scan of v over the CTA's threads in thread order; *total is the whole CTA's.  op is commutative here.
template <typename T, typename Op>
__device__ __forceinline__ T block_scan(T v, Op op, T* s_warp, T* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v = op(v, u);
  }
  if (lane == 31) s_warp[warp] = v;
  __syncthreads();
  T all = s_warp[0];
  for (int w = 1; w < ACC_WARPS; ++w) {
    if (w == warp) v = op(v, all);                              // all = warps 0 .. warp-1 here
    all = op(all, s_warp[w]);
  }
  *total = all;
  __syncthreads();                                              // s_warp is free again
  return v;
}

// number of entries of the ascending sorted[0..n) that are <= x (NaN entries, sorted last, never are)
__device__ __forceinline__ int count_le(const double* sorted, int n, double x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (sorted[mid] <= x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// counts of one detection packed for one scan: kept | tp << 21 | fp << 42 (a chunk holds at most ACC_THREADS of each)
__device__ __forceinline__ unsigned long long pack3(int k, int t, int f) {
  return (unsigned long long)k | ((unsigned long long)t << 21) | ((unsigned long long)f << 42);
}
__device__ __forceinline__ int unpack(unsigned long long v, int i) { return (int)((v >> (21 * i)) & 0x1fffffu); }

__global__ void __launch_bounds__(ACC_THREADS, 2) coco_accumulate_kernel(ssdk_coco_accumulate a) {
  extern __shared__ double s_qs[];                              // [2 * n_rec]: precision, then scores, of this row
  __shared__ unsigned long long s_u[ACC_WARPS];
  __shared__ double s_d[ACC_WARPS];
  __shared__ int s_tot[3], s_stop;
  int b = blockIdx.x;
  const int m = b % a.n_m; b /= a.n_m;
  const int ar = b % a.n_a; b /= a.n_a;
  const int k = b % a.n_k;
  const int t = b / a.n_k;
  const int k0 = a.sel_cat[k], a0 = a.sel_area[ar], max_det = a.sel_max_det[m];
  const int npig = a.npig[k0 * a.n_area + a0];
  if (npig == 0) return;                                        // no ground truth to recall: the row keeps its -1
  const int lo = a.cat_off[k0], hi = a.cat_off[k0 + 1];
  const unsigned char* flags = a.det_flags + ((size_t)a0 * a.n_thr + t) * a.n_det;
  double* s_q = s_qs;
  double* s_ss = s_qs + a.n_rec;
  for (int r = threadIdx.x; r < a.n_rec; r += ACC_THREADS) { s_q[r] = 0.0; s_ss[r] = 0.0; }

  // pass 1: nd, and the tp / fp totals
  int nk = 0, nt = 0, nf = 0;
  for (int i = lo + threadIdx.x; i < hi; i += ACC_THREADS) {
    if (a.ord_rank[i] >= max_det) continue;
    const unsigned char f = flags[a.ord_det[i]];
    ++nk;
    if (!(f & 2)) { if (f & 1) ++nt; else ++nf; }
  }
  nk = warp_sum(nk); nt = warp_sum(nt); nf = warp_sum(nf);
  if (threadIdx.x == 0) { s_tot[0] = 0; s_tot[1] = 0; s_tot[2] = 0; }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) { atomicAdd(&s_tot[0], nk); atomicAdd(&s_tot[1], nt); atomicAdd(&s_tot[2], nf); }
  __syncthreads();
  const int nd = s_tot[0], ntp = s_tot[1], nfp = s_tot[2];
  const double rc_last = div_rn((double)ntp, (double)npig);
  if (threadIdx.x == 0) {                                       // the fill ends at the first threshold the recall never reaches
    int r = 0;
    while (r < a.n_rec && a.rec_thrs[r] <= rc_last) ++r;
    s_stop = nd ? r : 0;
  }
  __syncthreads();
  const int stop = s_stop;

  // pass 2: chunks from the end; thread x holds i = base - x, so a scan in thread order is a suffix scan of the detections
  int after_k = 0, after_t = 0, after_f = 0;                    // kept / tp / fp counts behind the chunk
  double after_max = -1.0;                                      // running maximum of the precision behind the chunk
  for (int base = hi - 1; base >= lo; base -= ACC_THREADS) {
    const int i = base - (int)threadIdx.x;
    int kt = 0, tt = 0, ft = 0;
    if (i >= lo && a.ord_rank[i] < max_det) {
      const unsigned char f = flags[a.ord_det[i]];
      kt = 1;
      if (!(f & 2)) { if (f & 1) tt = 1; else ft = 1; }
    }
    unsigned long long tot;
    const unsigned long long inc = block_scan(pack3(kt, tt, ft), [](unsigned long long x, unsigned long long y) { return x + y; }, s_u, &tot);
    const int p = nd - 1 - (after_k + unpack(inc, 0) - kt);     // position in the rank < maxDet subsequence
    const int tp = ntp - (after_t + unpack(inc, 1) - tt);       // cumulative counts up to and including p
    const int fp = nfp - (after_f + unpack(inc, 2) - ft);
    const double pr = kt ? div_rn((double)tp, add_rn(add_rn((double)fp, (double)tp), DBL_EPSILON)) : -1.0;
    double mtot;
    double mx = block_scan(pr, [](double x, double y) { return x > y ? x : y; }, s_d, &mtot);
    mx = mx > after_max ? mx : after_max;
    if (kt && (tt || p == 0)) {
      const int r0 = p == 0 ? 0 : count_le(a.rec_sorted, a.n_rec, div_rn((double)(tp - tt), (double)npig));
      const int r1 = count_le(a.rec_sorted, a.n_rec, div_rn((double)tp, (double)npig));
      for (int x = r0; x < r1; ++x) {
        const int r = a.rec_perm[x];
        if (r < stop) { s_q[r] = mx; s_ss[r] = a.ord_score[i]; }
      }
    }
    after_k += unpack(tot, 0); after_t += unpack(tot, 1); after_f += unpack(tot, 2);
    after_max = mtot > after_max ? mtot : after_max;
  }
  __syncthreads();
  const size_t K = a.out_k, A = a.out_a, M = a.out_m;
  for (int r = threadIdx.x; r < a.n_rec; r += ACC_THREADS) {
    const size_t o = ((((size_t)t * a.n_rec + r) * K + k) * A + ar) * M + m;
    a.precision[o] = s_q[r];
    a.scores[o] = s_ss[r];
  }
  if (threadIdx.x == 0) a.recall[(((size_t)t * K + k) * A + ar) * M + m] = nd ? rc_last : 0.0;
}

}  // namespace

extern "C" int ssdk_cocoeval_match(ssdk_ctx* ctx, const ssdk_coco_match* args, void* stream_) {
  SSDK_REQUIRE(ctx && args, "ssdk_cocoeval_match: NULL argument");
  const ssdk_coco_match& a = *args;
  SSDK_REQUIRE(a.n_seg >= 0 && a.n_gt >= 0 && a.n_det >= 0 && a.n_area >= 0 && a.n_thr >= 0, "ssdk_cocoeval_match: bad argument");
  if (a.n_seg == 0) return SSDK_OK;
  SSDK_REQUIRE(a.seg_gt && a.seg_det && a.seg_cat && a.seg_npig && a.npig && (a.n_area == 0 || a.area_rng) && (a.n_thr == 0 || a.iou_thrs),
               "ssdk_cocoeval_match: NULL argument");
  SSDK_REQUIRE(a.n_gt == 0 || (a.gt_box && a.gt_area && a.gt_flags && a.gt_matched), "ssdk_cocoeval_match: NULL ground-truth array");
  SSDK_REQUIRE(a.n_det == 0 || (a.det_box && a.det_area && a.det_flags && a.det_match), "ssdk_cocoeval_match: NULL detection array");
  return launch(ctx, coco_match_kernel, a.n_seg, MATCH_THREADS, IOU_TILE * sizeof(double), (cudaStream_t)stream_, a);
}

extern "C" int ssdk_cocoeval_accumulate(ssdk_ctx* ctx, const ssdk_coco_accumulate* args, void* stream_) {
  SSDK_REQUIRE(ctx && args, "ssdk_cocoeval_accumulate: NULL argument");
  const ssdk_coco_accumulate& a = *args;
  SSDK_REQUIRE(a.n_thr >= 0 && a.n_area >= 0 && a.n_det >= 0 && a.n_rec >= 0 && a.n_k >= 0 && a.n_a >= 0 && a.n_m >= 0 &&
               a.out_k >= a.n_k && a.out_a >= a.n_a && a.out_m >= a.n_m, "ssdk_cocoeval_accumulate: bad argument");
  SSDK_REQUIRE((size_t)2 * a.n_rec * sizeof(double) <= 96 * 1024, "ssdk_cocoeval_accumulate: %d recall thresholds, at most %d", a.n_rec,
               (int)(96 * 1024 / (2 * sizeof(double))));
  const long long grid = (long long)a.n_thr * a.n_k * a.n_a * a.n_m;
  if (grid == 0) return SSDK_OK;
  SSDK_REQUIRE(grid <= INT_MAX, "ssdk_cocoeval_accumulate: %lld output rows", grid);
  SSDK_REQUIRE(a.cat_off && a.npig && a.sel_cat && a.sel_area && a.sel_max_det && a.precision && a.scores && a.recall &&
               (a.n_rec == 0 || (a.rec_thrs && a.rec_sorted && a.rec_perm)), "ssdk_cocoeval_accumulate: NULL argument");
  SSDK_REQUIRE(a.n_det == 0 || (a.ord_det && a.ord_rank && a.ord_score && a.det_flags), "ssdk_cocoeval_accumulate: NULL detection array");
  return launch(ctx, coco_accumulate_kernel, (int)grid, ACC_THREADS, (size_t)2 * a.n_rec * sizeof(double), (cudaStream_t)stream_, a);
}
