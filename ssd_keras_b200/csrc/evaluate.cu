// Evaluator.match_predictions on the device (reference eval_utils/average_precision_evaluator.py:538-736) and the cumulative
// true / false positive counts that compute_precision_recall starts from (:724-729).
//
// The reference walks the predictions of one class in descending confidence; each prediction is compared (element-wise iou,
// :679) with the ground-truth boxes of its image that have the same class, matched to the best one if the overlap reaches the
// threshold and that box is still free, else counted as a false positive (neutral boxes: neither).  The only sequential
// dependency is the "still free" state of a ground-truth box, which is private to one (class, image) pair -- so:
//   eval_match_kernel   one warp per (class, image) segment of the predictions (sorted by class, image, confidence desc), eight
//                       per CTA (eval_match_kernel<<<ceil_div(n_seg, 8), 256, 0, stream>>>): lanes share the image's boxes of
//                       that class, the IoU in the types NumPy uses (below), warp arg-max with np.argmax's rules (first
//                       maximum; the first NaN wins), flags written at the prediction's position in (class, confidence) order.
//   eval_cumsum_kernel  one CTA per class: inclusive scans of the two flag arrays (np.cumsum, :726-727).
// Sorting (two stable key sorts) is done by the caller; precision / recall / AP are a few vector operations on the cumulative
// counts (host, same NumPy expressions as the reference).
//
// The reference's types: the predicted box is a float32 array (the structured array's 'f4' fields), the ground truth keeps the
// labels' dtype.  So the predicted area is float32 arithmetic, the ground-truth area is the labels' dtype (the caller computes
// it with the reference's expression, int16 wrap included, and passes it as column 5), and the intersection, union and quotient
// run in result_type(labels, float32): float32 or float64, one flag per image.  On the float32 path the threshold is rounded to
// float32 before the comparison (a Python float against a float32 scalar).  Minimum and maximum propagate NaN (np.minimum /
// np.maximum), and NaN < thr is False, so a NaN overlap goes on to matching.
#include "common.cuh"
#include "rn.cuh"
#include <climits>
#include <cmath>

using namespace ssdk;

namespace {

struct EvalArgs {
  const int* seg_offsets;      // [n_seg+1] into the (class, image, confidence desc) order
  const int* pred_image;       // [n]
  const int* pred_class;       // [n]
  const float* pred_box;       // [n*4] corners
  const int* pred_rank;        // [n] position in (class, confidence desc) order
  const double* gt_rows;       // [sum G * 6] class, xmin, ymin, xmax, ymax, area (in the labels' dtype, held exactly)
  const int* gt_offsets;       // [n_images+1]
  const unsigned char* gt_f32; // [n_images] 1: the image's overlaps are float32 arithmetic, 0: float64
  const unsigned char* gt_neutral;   // [sum G] or NULL
  unsigned char* gt_matched;   // [sum G], zero on entry
  double thr; int d;
  int* tp; int* fp;            // [n], zero on entry
};

// np.maximum / np.minimum: a NaN in either operand is the result
template <typename T> __device__ __forceinline__ T np_max(T a, T b) { return (a >= b || a != a) ? a : b; }
template <typename T> __device__ __forceinline__ T np_min(T a, T b) { return (a <= b || a != a) ? a : b; }

// One (class, image) segment, overlaps in T (float or double).  best / best_g start from "no candidate" (-inf, INT_MAX); a lane
// takes its first candidate whatever its value, so an arg-max always names a box of the class.
template <typename T>
__device__ __forceinline__ void match_segment(const EvalArgs& a, int p0, int p1, int g0, int g1, int cls, int lane) {
  const double thr = (double)(T)a.thr;
  const float d = (float)a.d;
  for (int p = p0; p < p1; ++p) {                       // descending confidence inside the segment
    const float fx0 = a.pred_box[p * 4], fy0 = a.pred_box[p * 4 + 1], fx1 = a.pred_box[p * 4 + 2], fy1 = a.pred_box[p * 4 + 3];
    const T parea = (T)__fmul_rn(__fadd_rn(__fsub_rn(fx1, fx0), d), __fadd_rn(__fsub_rn(fy1, fy0), d));
    const T px0 = (T)fx0, py0 = (T)fy0, px1 = (T)fx1, py1 = (T)fy1;
    double best = -INFINITY; int best_g = INT_MAX; int best_nan = 0, any = 0;
    for (int g = g0 + lane; g < g1; g += 32) {
      const double* r = a.gt_rows + (size_t)g * 6;
      if (r[0] != (double)cls) continue;                  // gt[:, class_id] == class_id
      any = 1;
      const T iw = np_max((T)0, sub_rn(np_min((T)r[3], px1), np_max((T)r[1], px0)));
      const T ih = np_max((T)0, sub_rn(np_min((T)r[4], py1), np_max((T)r[2], py0)));
      const T inter = mul_rn(iw, ih);
      const T v = div_rn(inter, sub_rn(add_rn((T)r[5], parea), inter));
      if (best_nan) continue;                             // an earlier NaN of this lane already wins
      const int is_nan = (v != v) ? 1 : 0;
      if (is_nan || best_g == INT_MAX || (double)v > best) { best = (double)v; best_g = g; best_nan = is_nan; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int og = __shfl_xor_sync(0xffffffffu, best_g, o);
      const int on = __shfl_xor_sync(0xffffffffu, best_nan, o);
      any |= __shfl_xor_sync(0xffffffffu, any, o);
      bool take;
      if (on != best_nan) take = on > best_nan;           // NaN beats every number
      else if (on) take = og < best_g;                    // two NaNs: the first one
      else take = (ov > best) || (ov == best && og < best_g);   // equal values (or a lane without candidates): the first index
      if (take) { best = ov; best_g = og; best_nan = on; }
    }
    if (lane == 0) {
      const int r = a.pred_rank[p];
      if (!any) a.fp[r] = 1;                              // no box of this class in the image (:672-675)
      else if (best < thr) a.fp[r] = 1;                   // (NaN < thr is False, as in the reference)
      else if (!(a.gt_neutral && a.gt_neutral[best_g])) {
        if (!a.gt_matched[best_g]) { a.tp[r] = 1; a.gt_matched[best_g] = 1; }
        else a.fp[r] = 1;                                 // the box was matched by a more confident prediction
      }
    }
    __syncwarp();                                         // lane 0's gt_matched write is only ever read by lane 0
  }
}

__global__ void __launch_bounds__(256) eval_match_kernel(EvalArgs a, int n_seg) {
  const int seg = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (seg >= n_seg) return;
  const int p0 = a.seg_offsets[seg], p1 = a.seg_offsets[seg + 1];
  if (p1 <= p0) return;
  const int img = a.pred_image[p0], cls = a.pred_class[p0];
  const int g0 = a.gt_offsets[img], g1 = a.gt_offsets[img + 1];
  if (a.gt_f32[img]) match_segment<float>(a, p0, p1, g0, g1, cls, lane);
  else match_segment<double>(a, p0, p1, g0, g1, cls, lane);
}

__global__ void __launch_bounds__(1024) eval_cumsum_kernel(const int* __restrict__ tp, const int* __restrict__ fp, const int* __restrict__ class_offsets,
                                                           int* __restrict__ ctp, int* __restrict__ cfp) {
  __shared__ int s_t[32], s_f[32];
  __shared__ int s_base[2];
  const int c = blockIdx.x;
  const int lo = class_offsets[c], hi = class_offsets[c + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) { s_base[0] = 0; s_base[1] = 0; }
  __syncthreads();
  for (int base = lo; base < hi; base += 1024) {
    const int i = base + threadIdx.x;
    int t = i < hi ? tp[i] : 0, f = i < hi ? fp[i] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int vt = __shfl_up_sync(0xffffffffu, t, o), vf = __shfl_up_sync(0xffffffffu, f, o);
      if (lane >= o) { t += vt; f += vf; }
    }
    if (lane == 31) { s_t[warp] = t; s_f[warp] = f; }
    __syncthreads();
    int bt = s_base[0], bf = s_base[1];
    for (int w = 0; w < warp; ++w) { bt += s_t[w]; bf += s_f[w]; }
    if (i < hi) { ctp[i] = bt + t; cfp[i] = bf + f; }
    __syncthreads();
    if (threadIdx.x == 1023) { s_base[0] = bt + t; s_base[1] = bf + f; }
    __syncthreads();
  }
}

// eval_collect_kernel: ONE CTA per batch walks the rows in (image, row) order, 1024 at a time; a block-wide exclusive scan of
// the keep flags gives every kept row its slot, so the output keeps the reference's order without atomics.
struct CollectCols { int c[10]; };   // class, conf, xmin, ymin, xmax, ymax, inverter ymin, ymax, xmin, xmax

// round(numpy_scalar, n) for n > 0: multiply by 10^n in the scalar's type, rint, divide
template <typename T> __device__ __forceinline__ T round_decimals(T v, T f) { return div_rn(rint_rn(mul_rn(v, f)), f); }

template <typename T>
__device__ __forceinline__ void collect_row(const float* __restrict__ r, const double* __restrict__ inv, const CollectCols& cc, int pad, int decimals,
                                            int& cls, double& conf, double* box) {
  T v[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) v[k] = (T)r[k];
  const T ry = (T)inv[0], rx = (T)inv[1];                      // the Python float ratio as NumPy rounds it for this path
  v[cc.c[6]] = rint_rn(mul_rn(v[cc.c[6]], ry)); v[cc.c[7]] = rint_rn(mul_rn(v[cc.c[7]], ry));
  v[cc.c[8]] = rint_rn(mul_rn(v[cc.c[8]], rx)); v[cc.c[9]] = rint_rn(mul_rn(v[cc.c[9]], rx));
  if (pad) {                                                   // CropPad's inverter: even + 0 matters, it turns -0.0 into 0.0
    const T oy = (T)inv[2], ox = (T)inv[3];
    v[cc.c[6]] = add_rn(v[cc.c[6]], oy); v[cc.c[7]] = add_rn(v[cc.c[7]], oy);
    v[cc.c[8]] = add_rn(v[cc.c[8]], ox); v[cc.c[9]] = add_rn(v[cc.c[9]], ox);
  }
  const T c = v[cc.c[0]];
  cls = (sizeof(T) == 4) ? __float2int_rz((float)c) : __double2int_rz((double)c);
  T p = v[cc.c[1]];
  if (decimals > 0) {
    T f = (T)1;
    for (int i = 0; i < decimals; ++i) f = mul_rn(f, (T)10);   // 10^n is exact in both types for the n a caller uses
    p = round_decimals(p, f);
  }
  conf = (double)p;
#pragma unroll
  for (int k = 0; k < 4; ++k) box[k] = (double)round_decimals(v[cc.c[2 + k]], (T)10);
}

__global__ void __launch_bounds__(1024) eval_collect_kernel(const float* __restrict__ rows, int B, int max_out, const int* __restrict__ counts,
                                                            const double* __restrict__ inv, CollectCols cc, int f64, int pad, int decimals, int image_base,
                                                            int capacity, int* __restrict__ count, int* __restrict__ o_img,
                                                            int* __restrict__ o_cls, double* __restrict__ o_conf, double* __restrict__ o_box) {
  __shared__ int s_warp[32];
  __shared__ int s_base;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_base = *count;
  __syncthreads();
  const long long total = (long long)B * max_out;
  for (long long base = 0; base < total; base += 1024) {
    const long long i = base + threadIdx.x;
    int b = 0, j = 0, keep = 0;
    if (i < total) {
      b = (int)(i / max_out); j = (int)(i - (long long)b * max_out);
      keep = rows[i * 6] != 0.0f && (counts == nullptr || j < counts[b]);
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    int before = s_base, chunk = 0;
    for (int w = 0; w < 32; ++w) { const int n = s_warp[w]; if (w < warp) before += n; chunk += n; }
    before += __popc(ballot & ((1u << lane) - 1u));
    if (keep && before < capacity) {
      int cls; double conf, box[4];
      if (f64) collect_row<double>(rows + i * 6, inv + 4 * b, cc, pad, decimals, cls, conf, box);
      else collect_row<float>(rows + i * 6, inv + 4 * b, cc, pad, decimals, cls, conf, box);
      o_img[before] = image_base + b; o_cls[before] = cls; o_conf[before] = conf;
#pragma unroll
      for (int k = 0; k < 4; ++k) o_box[(size_t)before * 4 + k] = box[k];
    }
    __syncthreads();                                           // every thread has read s_warp and s_base
    if (threadIdx.x == 0) s_base += chunk;
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = s_base;
}

}  // namespace

extern "C" int ssdk_eval_collect(ssdk_ctx* ctx, const float* rows_dev, int B, int max_out, const int* counts_dev, const double* inv_dev,
                                 const int* cols_host, int f64, int pad, int conf_decimals, int image_base, int capacity, int* count_dev,
                                 int* out_image_dev, int* out_class_dev, double* out_conf_dev, double* out_box_dev, void* stream_) {
  SSDK_REQUIRE(ctx && B >= 0 && max_out >= 0 && capacity >= 0 && image_base >= 0 && conf_decimals >= 0 && conf_decimals <= 15,
               "ssdk_eval_collect: bad argument");
  SSDK_REQUIRE(cols_host && count_dev, "ssdk_eval_collect: NULL argument");
  CollectCols cc;
  for (int k = 0; k < 10; ++k) {
    SSDK_REQUIRE(cols_host[k] >= 0 && cols_host[k] < 6, "ssdk_eval_collect: column %d is %d, the decoded rows have 6 columns", k, cols_host[k]);
    cc.c[k] = cols_host[k];
  }
  if (B == 0 || max_out == 0) return SSDK_OK;
  SSDK_REQUIRE(rows_dev && inv_dev && (capacity == 0 || (out_image_dev && out_class_dev && out_conf_dev && out_box_dev)),
               "ssdk_eval_collect: NULL argument");
  return launch(ctx, eval_collect_kernel, 1, 1024, 0, (cudaStream_t)stream_, rows_dev, B, max_out, counts_dev, inv_dev, cc, f64 ? 1 : 0,
                pad ? 1 : 0, conf_decimals, image_base, capacity, count_dev, out_image_dev, out_class_dev, out_conf_dev, out_box_dev);
}

extern "C" int ssdk_eval_match(ssdk_ctx* ctx, int n_pred, const int* seg_offsets_dev, int n_seg, const int* pred_image_dev,
                               const int* pred_class_dev, const float* pred_box_dev, const int* pred_rank_dev, const double* gt_rows_dev,
                               const int* gt_offsets_dev, const unsigned char* gt_f32_dev, const unsigned char* gt_neutral_dev,
                               unsigned char* gt_matched_dev,
                               double matching_iou_threshold, int border_d, int* tp_dev, int* fp_dev, void* stream_) {
  SSDK_REQUIRE(ctx && n_pred >= 0 && n_seg >= 0, "ssdk_eval_match: bad argument");
  if (n_pred == 0 || n_seg == 0) return SSDK_OK;
  SSDK_REQUIRE(seg_offsets_dev && pred_image_dev && pred_class_dev && pred_box_dev && pred_rank_dev && gt_rows_dev && gt_offsets_dev &&
               gt_f32_dev && gt_matched_dev && tp_dev && fp_dev, "ssdk_eval_match: NULL argument");
  EvalArgs a{seg_offsets_dev, pred_image_dev, pred_class_dev, pred_box_dev, pred_rank_dev, gt_rows_dev, gt_offsets_dev, gt_f32_dev,
             gt_neutral_dev, gt_matched_dev, matching_iou_threshold, border_d, tp_dev, fp_dev};
  return launch(ctx, eval_match_kernel, ceil_div(n_seg, 8), 256, 0, (cudaStream_t)stream_, a, n_seg);
}

extern "C" int ssdk_eval_cumsum(ssdk_ctx* ctx, const int* tp_dev, const int* fp_dev, const int* class_offsets_dev, int n_segments,
                                int* ctp_dev, int* cfp_dev, void* stream_) {
  SSDK_REQUIRE(ctx && tp_dev && fp_dev && class_offsets_dev && ctp_dev && cfp_dev && n_segments > 0, "ssdk_eval_cumsum: bad argument");
  return launch(ctx, eval_cumsum_kernel, n_segments, 1024, 0, (cudaStream_t)stream_, tp_dev, fp_dev, class_offsets_dev, ctp_dev, cfp_dev);
}
