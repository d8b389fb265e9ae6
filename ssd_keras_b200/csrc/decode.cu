// Decode path on sm_90a: offset decode, confidence threshold, greedy IoU-NMS and top-k.
// Reference: keras_layers/keras_layer_DecodeDetections.py:109-265, keras_layer_DecodeDetectionsFast.py:111-248,
// ssd_encoder_decoder/ssd_output_decoder.py:77-333.
//
// Three stages, all HBM/latency-bound (no tensor cores):
//   dec_prepare_kernel  rows of y_pred staged through shared memory -> decoded corner boxes and
//                       class-major score planes (coalesced for the per-class NMS CTAs).
//   nms_kernel          one CTA per (class, image) segment.  Candidates are consumed in descending
//                       (score, then ascending index) order in BANDS of at most kNmsCap entries: a
//                       4-pass radix select over the float bits finds the band boundary (ties at the
//                       boundary are taken in index order), the band is compacted into shared memory,
//                       bitonic-sorted there and run through the sequential greedy scan (each thread
//                       tests one candidate against the kept list; warps resolve intra-chunk order with
//                       ballot/shuffle).  With the layer's cap of 400 survivors one band is normally enough.
//   topk_kernel         one CTA per image: concatenates the per-class survivors (class-major, NMS order),
//                       selects top_k with the same radix select, sorts and writes (class,conf,box) rows.
// Only top_k detections per image leave the decoder, so (i) no class ever needs more than top_k survivors, and (ii) a
// candidate whose score is below the top_k-th best SURVIVOR of the image cannot matter.  The NMS therefore runs in two
// stages: stage 1 looks at the best few hundred candidates of every class only (one small band) and records the score
// where it stopped; the top-k stage then checks that every class that was cut short stopped strictly below the score of
// the top_k-th detection -- if so the result is exactly that of the full scan (the remaining candidates could only have
// produced lower-scoring detections).  Classes that fail the check (few survivors, heavy suppression) are redone with
// the full multi-band scan in a third launch whose other CTAs exit at once, and the image's top-k is recomputed.
// Arithmetic follows the reference operation order with non-contracting intrinsics.
#include "common.cuh"
#include <cmath>

using namespace ssdk;

namespace {

constexpr int kNmsThreads = 128;  // NMS: small CTAs, many segments resident per SM (the scan is latency bound)
constexpr int kNmsCap = 2048;     // NMS band capacity (64-bit keys in shared memory)
constexpr int kKeptSm = 512;      // kept (prepared) boxes cached in shared memory
constexpr int kMaskN = 256;       // first-band candidates resolved through a pairwise suppression bit matrix
constexpr int kTopThreads = 512;  // top-k stage
constexpr int kTopCap = 16384;    // largest supported top_k

typedef unsigned long long u64;

__device__ __forceinline__ uint32_t okey(float f) {
  uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

struct SegView {
  const float* scores;   // [n]
  const int* labels;     // [n] or NULL; label 0 (background) never passes
  int n;
  int strict;            // 1: score > thr ; 0: score >= thr
  int use64;             // compare in float64 (NumPy API) or float32 (layer)
  float thr32;
  double thr64;
  int no_thresh;         // top-k stage: everything passes
};

__device__ __forceinline__ bool seg_pass(const SegView& s, int i, float sc) {
  if (s.no_thresh) return true;
  if (s.labels && s.labels[i] == 0) return false;
  if (s.use64) { double v = (double)sc; return s.strict ? (v > s.thr64) : (v >= s.thr64); }
  return s.strict ? (sc > s.thr32) : (sc >= s.thr32);
}

struct BandState { uint32_t hi_key; int hi_idx; int first; };

__device__ __forceinline__ bool remaining(const SegView& s, const BandState& st, int i, float sc, uint32_t& k) {
  if (!seg_pass(s, i, sc)) return false;
  k = okey(sc);
  return st.first || k < st.hi_key || (k == st.hi_key && i > st.hi_idx);
}

template <int NT>
__device__ int block_sum_int(int v, int* s_w) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
  __syncthreads();
  int t = 0;
  for (int w = 0; w < NT / 32; ++w) t += s_w[w];
  __syncthreads();
  return t;
}

// Fill keys[0..count) with the `cap` largest remaining (score desc, index asc) candidates of the segment
// (unsorted).  key = (~okey(score)) << 32 | index, so an ascending sort gives the wanted order.
template <int NT>
__device__ int band_select(const SegView& s, const BandState& st, int cap, u64* keys, int* s_hist, int* s_misc,
                           int* s_w, bool& more) {
  const int tid = threadIdx.x;
  // Radix select over the order-preserving keys, 8 bits per pass.  The first pass doubles as the count of remaining candidates
  // (its histogram total); four scores are loaded before any is used so that their latencies overlap.
  uint32_t prefix = 0, mask = 0;
  int want = cap, R = 0, ties_total = 0;
  bool take_all = false;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += NT) s_hist[i] = 0;
    __syncthreads();
    for (int i0 = tid; i0 < s.n; i0 += 4 * NT) {
      float sc[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) { const int i = i0 + u * NT; sc[u] = i < s.n ? s.scores[i] : 0.f; }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * NT;
        uint32_t k;
        if (i < s.n && remaining(s, st, i, sc[u], k) && ((k & mask) == prefix)) atomicAdd(&s_hist[(k >> shift) & 255u], 1);
      }
    }
    __syncthreads();
    if (tid < 32) {                      // warp 0: suffix scan over the 256 bins, 8 bins per lane
      int loc[8], sum = 0;
#pragma unroll
      for (int e = 0; e < 8; ++e) { loc[e] = s_hist[255 - (tid * 8 + e)]; sum += loc[e]; }
      int incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, o); if (tid >= o) incl += v; }
      if (tid == 31) s_misc[4] = incl;   // candidates that match the prefix so far (first pass: all remaining ones)
      int acc = incl - sum;              // candidates in bins above this lane's 8 bins
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if (acc < want && acc + loc[e] >= want) { s_misc[0] = 255 - (tid * 8 + e); s_misc[1] = want - acc; s_misc[5] = loc[e]; }
        acc += loc[e];
      }
    }
    __syncthreads();
    if (shift == 24) {
      R = s_misc[4];
      if (R == 0) { __syncthreads(); more = false; return 0; }
      if (R <= cap) { take_all = true; __syncthreads(); break; }
    }
    prefix |= ((uint32_t)s_misc[0]) << shift;
    mask |= 0xFFu << shift;
    want = s_misc[1];
    ties_total = s_misc[5];
    __syncthreads();
  }
  const uint32_t T = prefix;
  const int m_ties = want;
  // every candidate equal to the boundary key is kept: their order does not matter, no ranking needed
  const bool all_ties = take_all || (m_ties >= ties_total);
  if (tid == 0) { s_misc[2] = 0; s_misc[3] = 0; }
  __syncthreads();
  const int lane = tid & 31, warp = tid >> 5;
  if (all_ties) {
    for (int i0 = tid; i0 < s.n; i0 += 4 * NT) {
      float sc[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) { const int i = i0 + u * NT; sc[u] = i < s.n ? s.scores[i] : 0.f; }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * NT;
        uint32_t k = 0;
        if (i < s.n && remaining(s, st, i, sc[u], k) && (take_all || k >= T)) {
          const int slot = atomicAdd(&s_misc[2], 1);
          keys[slot] = ((u64)(~k) << 32) | (uint32_t)i;
        }
      }
    }
  } else {
    for (int base = 0; base < s.n; base += NT) {
      const int i = base + tid;
      bool take = false, tie = false;
      uint32_t k = 0;
      if (i < s.n && remaining(s, st, i, s.scores[i], k)) {
        if (k > T) take = true;
        else if (k == T) tie = true;
      }
      // ties at the boundary are taken in ascending index order
      unsigned bal = __ballot_sync(0xffffffffu, tie);
      int wrank = __popc(bal & ((1u << lane) - 1));
      if (lane == 0) s_w[warp] = __popc(bal);
      __syncthreads();
      int wbase = 0, total = 0;
      for (int w = 0; w < NT / 32; ++w) { int c = s_w[w]; if (w < warp) wbase += c; total += c; }
      int tie_rank = s_misc[3] + wbase + wrank;
      if (tie && tie_rank < m_ties) take = true;
      __syncthreads();
      if (tid == 0) s_misc[3] += total;
      if (take) {
        int slot = atomicAdd(&s_misc[2], 1);
        keys[slot] = ((u64)(~k) << 32) | (uint32_t)i;
      }
    }
  }
  __syncthreads();
  more = !take_all;
  return s_misc[2];
}

template <int NT>
__device__ void bitonic_sort(u64* keys, int count) {
  int n = 1;
  while (n < count) n <<= 1;
  for (int i = count + threadIdx.x; i < n; i += NT) keys[i] = ~0ull;
  __syncthreads();
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < (n >> 1); t += NT) {
        int i = ((t / j) * (j << 1)) + (t % j);   // lower index of the pair
        int p = i + j;
        bool up = ((i & k) == 0);
        u64 a = keys[i], b = keys[p];
        if ((a > b) == up) { keys[i] = b; keys[p] = a; }
      }
      __syncthreads();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// IoU suppression rules on "prepared" boxes (coordinates + area computed once per box)
// ---------------------------------------------------------------------------------------------
template <typename T> struct PBox { T x0, y0, x1, y1, a; };

__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }

// std::min / std::max exactly as the TF kernel uses them: NaN handling depends on the argument order.
__device__ __forceinline__ float tf_min(float a, float b) { return (b < a) ? b : a; }
__device__ __forceinline__ float tf_max(float a, float b) { return (a < b) ? b : a; }
template <typename T> __device__ __forceinline__ T np_min(T a, T b) { return (a != a) ? a : ((b != b) ? b : (a < b ? a : b)); }   // NaN propagates
template <typename T> __device__ __forceinline__ T np_max(T a, T b) { return (a != a) ? a : ((b != b) ? b : (a > b ? a : b)); }

template <typename T, bool LAYER>
__device__ __forceinline__ PBox<T> prepare_box(const T* q, T d) {
  PBox<T> b;
  if constexpr (LAYER) {    // tf.image.non_max_suppression normalises each box with min/max first
    b.x0 = tf_min((float)q[0], (float)q[2]); b.x1 = tf_max((float)q[0], (float)q[2]);
    b.y0 = tf_min((float)q[1], (float)q[3]); b.y1 = tf_max((float)q[1], (float)q[3]);
    b.a = mul_rn(sub_rn(b.y1, b.y0), sub_rn(b.x1, b.x0));
  } else {        // iou(): areas use d, the intersection does not (bounding_box_utils.py:345,373-374)
    b.x0 = q[0]; b.y0 = q[1]; b.x1 = q[2]; b.y1 = q[3];
    b.a = mul_rn(add_rn(sub_rn(b.x1, b.x0), d), add_rn(sub_rn(b.y1, b.y0), d));
  }
  return b;
}

// candidate c against selected m.  LAYER: suppress iff IoU > thr, non-positive areas give IoU 0.
// NumPy API (_greedy_nms, ssd_output_decoder.py:90-91): keep iff iou <= thr, i.e. NaN is dropped.
template <typename T, bool LAYER>
__device__ __forceinline__ bool suppressed(const PBox<T>& c, const PBox<T>& m, T thr) {
  if constexpr (LAYER) {
    // disjoint boxes (the vast majority of candidate x kept pairs): the intersection below is 0 (or NaN), which never
    // suppresses for thr >= 0 -- four compares instead of the full IoU
    if (thr >= (T)0 && (c.x1 <= m.x0 || m.x1 <= c.x0 || c.y1 <= m.y0 || m.y1 <= c.y0)) return false;
    if (c.a <= (T)0 || m.a <= (T)0) return false;
    T ih = tf_max((float)sub_rn(tf_min((float)c.y1, (float)m.y1), tf_max((float)c.y0, (float)m.y0)), 0.f);
    T iw = tf_max((float)sub_rn(tf_min((float)c.x1, (float)m.x1), tf_max((float)c.x0, (float)m.x0)), 0.f);
    T inter = mul_rn(ih, iw);
    if (inter == (T)0 && thr >= (T)0) return false;          // IoU is 0 (or NaN): never > thr
    T iou = div_rn(inter, sub_rn(add_rn(c.a, m.a), inter));
    return iou > thr;
  } else {
    T iw = np_max((T)0, sub_rn(np_min(c.x1, m.x1), np_max(c.x0, m.x0)));
    T ih = np_max((T)0, sub_rn(np_min(c.y1, m.y1), np_max(c.y0, m.y0)));
    T inter = mul_rn(iw, ih);
    T uni = sub_rn(add_rn(c.a, m.a), inter);
    if (inter == (T)0 && uni == uni && uni != (T)0) return !((T)0 <= thr);   // IoU is exactly +-0
    T iou = div_rn(inter, uni);
    return !(iou <= thr);
  }
}

struct NmsParams {
  const float* scores;     // [B*S*n]
  const int* labels;       // [B*n] or NULL
  const void* boxes;       // [B*n*4] of T
  int* kept_idx;           // [B*S*kmax]
  int* kept_cnt;           // [B*S]
  int n, S, kmax, cap;     // cap: stop after this many survivors (layer) ; kmax >= cap
  int strict, use64;
  float thr32; double thr64;
  double iou_thr; int d;
  int band_cap;            // candidates per band (<= kNmsCap)
  int max_bands;           // > 0: stop after this many bands even if candidates remain (stage 1)
  uint32_t* cut_key;       // [B*S] out (stage 1): order key of the last candidate looked at when the scan was cut short, else 0
  const int* redo;         // [B*S] in (stage 3): only segments with a non-zero flag are (re)done
};

template <typename T, bool LAYER>
__global__ void __launch_bounds__(kNmsThreads) nms_kernel(NmsParams prm) {
  constexpr int NT = kNmsThreads, NW = NT / 32;
  __shared__ __align__(16) u64 keys[kNmsCap];
  __shared__ __align__(16) T kbox[kKeptSm * 5];
  __shared__ int s_hist[256];
  __shared__ int s_misc[8];
  __shared__ int s_w[NW];
  __shared__ int s_K;

  const int sidx = blockIdx.x, b = blockIdx.y;
  const int seg = b * prm.S + sidx;
  if (prm.redo && !prm.redo[seg]) return;
  SegView sv;
  sv.scores = prm.scores + (size_t)seg * prm.n;
  sv.labels = prm.labels ? prm.labels + (size_t)b * prm.n : nullptr;
  sv.n = prm.n; sv.strict = prm.strict; sv.use64 = prm.use64; sv.thr32 = prm.thr32; sv.thr64 = prm.thr64; sv.no_thresh = 0;
  const T* boxes = reinterpret_cast<const T*>(prm.boxes) + (size_t)b * prm.n * 4;
  int* kept = prm.kept_idx + (size_t)seg * prm.kmax;
  const T thr = (T)prm.iou_thr;
  const T dd = (T)prm.d;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  auto kept_box = [&](int t) {
    PBox<T> m;
    if (t < kKeptSm) { m.x0 = kbox[t * 5]; m.y0 = kbox[t * 5 + 1]; m.x1 = kbox[t * 5 + 2]; m.y1 = kbox[t * 5 + 3]; m.a = kbox[t * 5 + 4]; }
    else m = prepare_box<T, LAYER>(boxes + (size_t)kept[t] * 4, dd);
    return m;
  };

  if (threadIdx.x == 0) s_K = 0;
  BandState st{0u, -1, 1};
  __syncthreads();
  bool done = false;
  int bands = 0;
  uint32_t cut = 0;
  while (!done) {
    bool more = false;
    const int cnt = band_select<NT>(sv, st, prm.band_cap, keys, s_hist, s_misc, s_w, more);
    if (cnt == 0) break;
    bitonic_sort<NT>(keys, cnt);
    if (st.first && cnt <= kMaskN && prm.cap >= 1) {
      // First band, at most 256 candidates (stage 1 of the two-stage scheme): the greedy scan without its serial chain.  All
      // pairwise suppression bits (candidate j against every earlier candidate i) are computed in parallel, then one warp walks
      // the candidates 32 at a time: a candidate survives iff none of the survivors so far suppresses it -- bit operations only.
      PBox<T>* cb = reinterpret_cast<PBox<T>*>(kbox);          // candidate boxes (kept boxes are compacted into the same array)
      uint32_t* msk = reinterpret_cast<uint32_t*>(keys + kMaskN);   // [kMaskN][kMaskN / 32], behind the sorted keys
      for (int j = threadIdx.x; j < cnt; j += NT)
        cb[j] = prepare_box<T, LAYER>(boxes + (size_t)(uint32_t)(keys[j] & 0xffffffffull) * 4, dd);
      __syncthreads();
      for (int r = 0; r < 2; ++r) {                            // rows t and 255 - t: the same number of tests for every thread
        const int j = r == 0 ? (int)threadIdx.x : kMaskN - 1 - (int)threadIdx.x;
        if (j >= cnt || (r == 1 && j < NT)) continue;
        const PBox<T> c = cb[j];
        for (int w = 0; w <= (j >> 5); ++w) {
          uint32_t bits = 0;
          const int i1 = min(j, w * 32 + 32);
          for (int i = w * 32; i < i1; ++i) bits |= (suppressed<T, LAYER>(c, cb[i], thr) ? 1u : 0u) << (i & 31);
          msk[j * (kMaskN / 32) + w] = bits;
        }
      }
      __syncthreads();
      if (warp == 0) {
        uint32_t kw = 0;                                        // lane w (< 8): survivors among candidates 32 w .. 32 w + 31
        int count = 0;
        const int n_chunks = (cnt + 31) >> 5;
        for (int c = 0; c < n_chunks && count < prm.cap; ++c) {
          const int j = c * 32 + lane;
          const bool valid = j < cnt;
          uint32_t early = 0;
          for (int w = 0; w < c; ++w) {
            const uint32_t k_w = __shfl_sync(0xffffffffu, kw, w);
            if (valid) early |= msk[j * (kMaskN / 32) + w] & k_w;
          }
          const uint32_t intra = valid ? msk[j * (kMaskN / 32) + c] : 0u;
          const uint32_t alive = __ballot_sync(0xffffffffu, valid && early == 0u);
          uint32_t kc = 0;
          for (int b = 0; b < 32; ++b) {                        // (uniform: every lane runs the same 32 steps)
            const uint32_t ib = __shfl_sync(0xffffffffu, intra, b);
            if (((alive >> b) & 1u) && !(ib & kc) && count < prm.cap) { kc |= 1u << b; ++count; }
          }
          if (lane == c) kw = kc;
          // survivors of this chunk -> kept list and kept boxes, in order
          const bool mine = (kc >> lane) & 1u;
          const int pos = (count - __popc(kc)) + __popc(kc & ((1u << lane) - 1));
          PBox<T> bx{};
          if (mine) bx = cb[j];
          __syncwarp();
          if (mine) {
            kept[pos] = (int)(uint32_t)(keys[j] & 0xffffffffull);
            if (pos < kKeptSm) { kbox[pos * 5] = bx.x0; kbox[pos * 5 + 1] = bx.y0; kbox[pos * 5 + 2] = bx.x1; kbox[pos * 5 + 3] = bx.y1; kbox[pos * 5 + 4] = bx.a; }
          }
          __syncwarp();
        }
        if (lane == 0) s_K = count;
      }
      __syncthreads();
      if (s_K >= prm.cap) done = true;
    } else
    for (int c0 = 0; c0 < cnt && !done; c0 += NT) {
      const int j = c0 + threadIdx.x;
      bool alive = j < cnt;
      int idx = 0;
      PBox<T> bx{};
      if (alive) {
        idx = (int)(uint32_t)(keys[j] & 0xffffffffull);
        bx = prepare_box<T, LAYER>(boxes + (size_t)idx * 4, dd);
      }
      const int k_start = s_K;
      // four kept boxes per iteration: the tests are independent, so their shared-memory loads and min/max chains overlap
      for (int t = 0; t < k_start && alive; t += 4) {
        bool sup = false;
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (t + u < k_start) sup |= suppressed<T, LAYER>(bx, kept_box(t + u), thr);
        if (sup) alive = false;
      }
      __syncthreads();
      // warps take turns (ascending candidate order) to settle intra-chunk suppression
      for (int w = 0; w < NW; ++w) {
        if (warp == w) {
          const int k_cur = *((volatile int*)&s_K);
          for (int t = k_start; t < k_cur && alive; ++t)          // survivors added by earlier warps of this chunk
            if (suppressed<T, LAYER>(bx, kept_box(t), thr)) alive = false;
          unsigned am = __ballot_sync(0xffffffffu, alive);
          int nk = 0, my_rank = -1;
          while (am) {
            const int i = __ffs(am) - 1;
            PBox<T> m;
            m.x0 = __shfl_sync(0xffffffffu, bx.x0, i); m.y0 = __shfl_sync(0xffffffffu, bx.y0, i);
            m.x1 = __shfl_sync(0xffffffffu, bx.x1, i); m.y1 = __shfl_sync(0xffffffffu, bx.y1, i);
            m.a = __shfl_sync(0xffffffffu, bx.a, i);
            if (lane == i) my_rank = nk;
            ++nk;
            if (k_cur + nk >= prm.cap) break;                      // cap reached: later candidates are never looked at
            if (alive && lane > i && suppressed<T, LAYER>(bx, m, thr)) alive = false;
            am = __ballot_sync(0xffffffffu, alive && lane > i);
          }
          if (my_rank >= 0 && k_cur + my_rank < prm.cap) {
            const int pos = k_cur + my_rank;
            kept[pos] = idx;
            if (pos < kKeptSm) { kbox[pos * 5] = bx.x0; kbox[pos * 5 + 1] = bx.y0; kbox[pos * 5 + 2] = bx.x1; kbox[pos * 5 + 3] = bx.y1; kbox[pos * 5 + 4] = bx.a; }
          }
          __syncwarp();
          if (lane == 0) { const int nkk = k_cur + nk; s_K = nkk < prm.cap ? nkk : prm.cap; }
          __threadfence_block();
        }
        __syncthreads();
      }
      if (s_K >= prm.cap) done = true;
    }
    if (!more || done) break;
    // next band starts strictly below the last (smallest) candidate of this band
    const u64 last = keys[cnt - 1];
    st.hi_key = ~(uint32_t)(last >> 32);
    st.hi_idx = (int)(uint32_t)(last & 0xffffffffull);
    st.first = 0;
    if (prm.max_bands > 0 && ++bands >= prm.max_bands) { cut = st.hi_key ? st.hi_key : 1u; break; }   // cut short: candidates remain
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    prm.kept_cnt[seg] = s_K;
    if (prm.cut_key) prm.cut_key[seg] = cut;
  }
}

// ---------------------------------------------------------------------------------------------
// prepare: decode boxes + transpose scores
// ---------------------------------------------------------------------------------------------
struct PrepParams {
  const float* y;        // [B*P*W]
  int P, C, W;
  int mode;              // ssdk_decode_mode
  int layer;
  int coords, normalize;
  float img_w, img_h;
  void* boxes;           // [B*P*4] float (layer / numpy corners) or double (numpy centroids/minmax)
  float* scores;         // per-class: [B*(C-1)*P]; fast: [B*P]
  int* labels;           // fast: [B*P]
  int box_f64;
};

__device__ __forceinline__ float exp_cr(float x) { return (float)exp((double)x); }   // correctly rounded float32 exp

__global__ void __launch_bounds__(256) dec_prepare_kernel(PrepParams p) {
  extern __shared__ float s_rows[];                            // [256*W]
  const int b = blockIdx.y;
  const int p0 = blockIdx.x * 256;
  const int nrows = min(256, p.P - p0);
  const float* src = p.y + ((size_t)b * p.P + p0) * p.W;
  for (int i = threadIdx.x; i < nrows * p.W; i += 256) s_rows[i] = src[i];
  __syncthreads();
  if (threadIdx.x >= nrows) return;
  const float* r = s_rows + (size_t)threadIdx.x * p.W;
  const int pi = p0 + threadIdx.x;
  const int C = p.C;
  if (p.mode == SSDK_DECODE_PER_CLASS) {
    for (int c = 1; c < C; ++c) p.scores[((size_t)b * (C - 1) + (c - 1)) * p.P + pi] = r[c];
  } else {
    float best = r[0]; int bi = 0;
    for (int c = 1; c < C; ++c) if (r[c] > best) { best = r[c]; bi = c; }   // first index on ties
    p.scores[(size_t)b * p.P + pi] = best;
    p.labels[(size_t)b * p.P + pi] = bi;
  }
  const float* o = r + C;         // 4 offsets
  const float* a = r + C + 4;     // 4 anchor coords
  const float* v = r + C + 8;     // 4 variances
  const size_t bo = ((size_t)b * p.P + pi) * 4;
  if (p.layer) {
    // keras_layer_DecodeDetections.py:124-146 (float32, left-associative products)
    float cx = __fadd_rn(__fmul_rn(__fmul_rn(o[0], v[0]), a[2]), a[0]);
    float cy = __fadd_rn(__fmul_rn(__fmul_rn(o[1], v[1]), a[3]), a[1]);
    float w = __fmul_rn(exp_cr(__fmul_rn(o[2], v[2])), a[2]);
    float h = __fmul_rn(exp_cr(__fmul_rn(o[3], v[3])), a[3]);
    float x0 = __fsub_rn(cx, __fmul_rn(0.5f, w)), y0 = __fsub_rn(cy, __fmul_rn(0.5f, h));
    float x1 = __fadd_rn(cx, __fmul_rn(0.5f, w)), y1 = __fadd_rn(cy, __fmul_rn(0.5f, h));
    if (p.normalize) { x0 = __fmul_rn(x0, p.img_w); x1 = __fmul_rn(x1, p.img_w); y0 = __fmul_rn(y0, p.img_h); y1 = __fmul_rn(y1, p.img_h); }
    float* bx = reinterpret_cast<float*>(p.boxes) + bo;
    bx[0] = x0; bx[1] = y0; bx[2] = x1; bx[3] = y1;
    return;
  }
  // NumPy API, ssd_output_decoder.py:174-198
  if (p.coords == SSDK_COORDS_CENTROIDS) {
    float w = __fmul_rn(exp_cr(__fmul_rn(o[2], v[2])), a[2]);
    float h = __fmul_rn(exp_cr(__fmul_rn(o[3], v[3])), a[3]);
    float cx = __fadd_rn(__fmul_rn(o[0], __fmul_rn(v[0], a[2])), a[0]);
    float cy = __fadd_rn(__fmul_rn(o[1], __fmul_rn(v[1], a[3])), a[1]);
    float x0 = __fsub_rn(cx, __fdiv_rn(w, 2.0f)), y0 = __fsub_rn(cy, __fdiv_rn(h, 2.0f));
    float x1 = __fadd_rn(cx, __fdiv_rn(w, 2.0f)), y1 = __fadd_rn(cy, __fdiv_rn(h, 2.0f));
    double* bx = reinterpret_cast<double*>(p.boxes) + bo;      // float64 container from here on (:179)
    double X0 = x0, Y0 = y0, X1 = x1, Y1 = y1;
    if (p.normalize) { X0 = __dmul_rn(X0, (double)p.img_w); X1 = __dmul_rn(X1, (double)p.img_w); Y0 = __dmul_rn(Y0, (double)p.img_h); Y1 = __dmul_rn(Y1, (double)p.img_h); }
    bx[0] = X0; bx[1] = Y0; bx[2] = X1; bx[3] = Y1;
  } else if (p.coords == SSDK_COORDS_MINMAX) {
    float wa = __fsub_rn(a[1], a[0]), ha = __fsub_rn(a[3], a[2]);
    float xmin = __fadd_rn(__fmul_rn(__fmul_rn(o[0], v[0]), wa), a[0]);
    float xmax = __fadd_rn(__fmul_rn(__fmul_rn(o[1], v[1]), wa), a[1]);
    float ymin = __fadd_rn(__fmul_rn(__fmul_rn(o[2], v[2]), ha), a[2]);
    float ymax = __fadd_rn(__fmul_rn(__fmul_rn(o[3], v[3]), ha), a[3]);
    double* bx = reinterpret_cast<double*>(p.boxes) + bo;
    double X0 = xmin, Y0 = ymin, X1 = xmax, Y1 = ymax;
    if (p.normalize) { X0 = __dmul_rn(X0, (double)p.img_w); X1 = __dmul_rn(X1, (double)p.img_w); Y0 = __dmul_rn(Y0, (double)p.img_h); Y1 = __dmul_rn(Y1, (double)p.img_h); }
    bx[0] = X0; bx[1] = Y0; bx[2] = X1; bx[3] = Y1;
  } else {   // corners: the array stays float32 all the way (no convert_coordinates call, :186-190)
    float wa = __fsub_rn(a[2], a[0]), ha = __fsub_rn(a[3], a[1]);
    float x0 = __fadd_rn(__fmul_rn(__fmul_rn(o[0], v[0]), wa), a[0]);
    float y0 = __fadd_rn(__fmul_rn(__fmul_rn(o[1], v[1]), ha), a[1]);
    float x1 = __fadd_rn(__fmul_rn(__fmul_rn(o[2], v[2]), wa), a[2]);
    float y1 = __fadd_rn(__fmul_rn(__fmul_rn(o[3], v[3]), ha), a[3]);
    if (p.normalize) { x0 = __fmul_rn(x0, p.img_w); x1 = __fmul_rn(x1, p.img_w); y0 = __fmul_rn(y0, p.img_h); y1 = __fmul_rn(y1, p.img_h); }
    float* bx = reinterpret_cast<float*>(p.boxes) + bo;
    bx[0] = x0; bx[1] = y0; bx[2] = x1; bx[3] = y1;
  }
}

// ---------------------------------------------------------------------------------------------
// top-k / output assembly
// ---------------------------------------------------------------------------------------------
struct TopkParams {
  const float* scores;   // [B*S*n]
  const int* labels;     // fast: [B*n]
  const void* boxes; int box_f64;
  const int* kept_idx; const int* kept_cnt;
  int n, S, kmax;
  int top_k, max_out, layer;
  float* cat_score;      // scratch [B*S*kmax]
  int* cat_src;          // scratch [B*S*kmax*2] (s, prior idx)
  float* out; int* out_counts; int* out_index;
  const uint32_t* cut_key; // stage-1 verification (NULL: none): see the file header
  int* redo;             // [B*S] out
  int* any_redo;         // [B] out
  const int* only_if;    // [B] in (second top-k pass): images without a flag keep their output
};

__device__ void emit_row(const TopkParams& p, int b, int row_out, int s, int idx, float score) {
  float* o = p.out + ((size_t)b * p.max_out + row_out) * 6;
  o[0] = p.labels ? (float)p.labels[(size_t)b * p.n + idx] : (float)(s + 1);
  o[1] = score;
  if (p.box_f64) {
    const double* q = reinterpret_cast<const double*>(p.boxes) + ((size_t)b * p.n + idx) * 4;
    o[2] = (float)q[0]; o[3] = (float)q[1]; o[4] = (float)q[2]; o[5] = (float)q[3];
  } else {
    const float* q = reinterpret_cast<const float*>(p.boxes) + ((size_t)b * p.n + idx) * 4;
    o[2] = q[0]; o[3] = q[1]; o[4] = q[2]; o[5] = q[3];
  }
  if (p.out_index) p.out_index[(size_t)b * p.max_out + row_out] = idx;
}

__global__ void __launch_bounds__(kTopThreads) topk_kernel(TopkParams p) {
  constexpr int kThreads = kTopThreads;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  u64* keys = reinterpret_cast<u64*>(smem_raw);
  __shared__ int s_hist[256];
  __shared__ int s_misc[8];
  __shared__ int s_w[kTopThreads / 32];
  __shared__ int s_off[1025];
  const int b = blockIdx.x;
  const int S = p.S;
  if (p.only_if && !p.only_if[b]) return;
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int s = 0; s < S; ++s) { s_off[s] = acc; acc += p.kept_cnt[b * S + s]; }
    s_off[S] = acc;
  }
  __syncthreads();
  const int M = s_off[S];
  float* cs = p.cat_score + (size_t)b * S * p.kmax;
  int* csrc = p.cat_src + (size_t)b * S * p.kmax * 2;
  for (int s = 0; s < S; ++s) {
    const int c = s_off[s + 1] - s_off[s];
    const int* kp = p.kept_idx + ((size_t)b * S + s) * p.kmax;
    const float* sc = p.scores + ((size_t)b * S + s) * p.n;
    for (int j = threadIdx.x; j < c; j += kThreads) {
      int idx = kp[j];
      int r = s_off[s] + j;
      cs[r] = sc[idx]; csrc[2 * r] = s; csrc[2 * r + 1] = idx;
    }
  }
  __syncthreads();
  // zero-fill the output block of this image
  for (int i = threadIdx.x; i < p.max_out * 6; i += kThreads) p.out[(size_t)b * p.max_out * 6 + i] = 0.f;
  if (p.out_index) for (int i = threadIdx.x; i < p.max_out; i += kThreads) p.out_index[(size_t)b * p.max_out + i] = -1;
  __syncthreads();
  int n_out;
  uint32_t sigma = 0;      // order key of the top_k-th detection (0: fewer than top_k detections so far)
  if (p.top_k <= 0 || (!p.layer && M <= p.top_k)) {
    // NumPy API without top-k filtering: class-major / NMS order, as the reference concatenates them
    n_out = M < p.max_out ? M : p.max_out;
    for (int r = threadIdx.x; r < n_out; r += kThreads) emit_row(p, b, r, csrc[2 * r], csrc[2 * r + 1], cs[r]);
  } else {
    SegView sv;
    sv.scores = cs; sv.labels = nullptr; sv.n = M; sv.strict = 0; sv.use64 = 0; sv.thr32 = 0.f; sv.thr64 = 0.0; sv.no_thresh = 1;
    BandState st{0u, -1, 1};
    bool more;
    int want = p.top_k < M ? p.top_k : M;
    int cnt = (M > 0) ? band_select<kTopThreads>(sv, st, want, keys, s_hist, s_misc, s_w, more) : 0;
    if (cnt > 0) bitonic_sort<kTopThreads>(keys, cnt);
    if (cnt > 0 && cnt == p.top_k) sigma = ~(uint32_t)(keys[cnt - 1] >> 32);
    n_out = cnt < p.max_out ? cnt : p.max_out;
    for (int j = threadIdx.x; j < n_out; j += kThreads) {
      int r = (int)(uint32_t)(keys[j] & 0xffffffffull);
      emit_row(p, b, j, csrc[2 * r], csrc[2 * r + 1], cs[r]);
    }
  }
  if (threadIdx.x == 0) p.out_counts[b] = n_out;
  if (p.cut_key) {
    // a class whose scan was cut short is exact iff it stopped strictly below the top_k-th detection of the image
    int flag = 0;
    for (int s = threadIdx.x; s < S; s += kThreads) {
      const uint32_t ck = p.cut_key[b * S + s];
      const int r = (ck != 0u && !(ck < sigma)) ? 1 : 0;
      p.redo[b * S + s] = r;
      flag |= r;
    }
    flag = __syncthreads_or(flag);
    if (threadIdx.x == 0) p.any_redo[b] = flag;
  }
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

template <typename T, bool LAYER>
int launch_nms(ssdk_ctx* ctx, const NmsParams& np, int B, cudaStream_t stream) {
  dim3 grid(np.S, B);
  nms_kernel<T, LAYER><<<grid, kNmsThreads, 0, stream>>>(np);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

int stage1_band(int S, int top_k) {
  int want = 4 * top_k / (S > 0 ? S : 1), b = 256;
  while (b < want && b < kNmsCap) b <<= 1;
  return b;
}

int run_nms_topk(ssdk_ctx* ctx, int B, int n, int S, int layer, int box_f64, int np_f32, const float* scores,
                 const int* labels, const void* boxes, int strict, double conf_thr, double iou_thr, int d, int cap,
                 int top_k, int max_out, unsigned char* scratch, float* out, int* out_counts, int* out_index,
                 cudaStream_t stream) {
  // only top_k rows leave: no class needs more than top_k survivors (rows beyond the top_k-th of one class never reach
  // the global top_k: equal scores are ordered class-major / NMS order, so a class's own earlier survivors come first)
  if (top_k > 0 && top_k < cap) cap = top_k;
  const int kmax = cap;
  size_t o = 0;
  int* kept_idx = reinterpret_cast<int*>(scratch + o); o += align_up((size_t)B * S * kmax * 4, 256);
  int* kept_cnt = reinterpret_cast<int*>(scratch + o); o += align_up((size_t)B * S * 4, 256);
  float* cat_score = reinterpret_cast<float*>(scratch + o); o += align_up((size_t)B * S * kmax * 4, 256);
  int* cat_src = reinterpret_cast<int*>(scratch + o); o += align_up((size_t)B * S * kmax * 8, 256);
  uint32_t* cut_key = reinterpret_cast<uint32_t*>(scratch + o); o += align_up((size_t)B * S * 4, 256);
  int* redo = reinterpret_cast<int*>(scratch + o); o += align_up((size_t)B * S * 4, 256);
  int* any_redo = reinterpret_cast<int*>(scratch + o); o += align_up((size_t)B * 4, 256);
  const int band1 = stage1_band(S, top_k);
  bool two_stage = top_k > 0 && n > band1 && band1 < kNmsCap;
  if (const char* e = getenv("SSDK_NMS_TWO_STAGE")) two_stage = two_stage && atoi(e) != 0;
  NmsParams np{};
  np.scores = scores; np.labels = labels; np.boxes = boxes; np.kept_idx = kept_idx; np.kept_cnt = kept_cnt;
  np.n = n; np.S = S; np.kmax = kmax; np.cap = cap; np.strict = strict; np.use64 = layer ? 0 : 1;
  np.thr32 = (float)conf_thr; np.thr64 = conf_thr; np.iou_thr = iou_thr; np.d = d;
  np.band_cap = two_stage ? band1 : kNmsCap; np.max_bands = two_stage ? 1 : 0; np.cut_key = two_stage ? cut_key : nullptr; np.redo = nullptr;
  auto nms = [&](const NmsParams& q) {
    if (layer) return launch_nms<float, true>(ctx, q, B, stream);
    if (np_f32) return launch_nms<float, false>(ctx, q, B, stream);
    return launch_nms<double, false>(ctx, q, B, stream);
  };
  int rc = nms(np);
  if (rc) return rc;
  TopkParams tp{};
  tp.scores = scores; tp.labels = labels; tp.boxes = boxes; tp.box_f64 = box_f64; tp.kept_idx = kept_idx; tp.kept_cnt = kept_cnt;
  tp.n = n; tp.S = S; tp.kmax = kmax; tp.top_k = top_k; tp.max_out = max_out; tp.layer = layer;
  tp.cat_score = cat_score; tp.cat_src = cat_src; tp.out = out; tp.out_counts = out_counts; tp.out_index = out_index;
  if (two_stage) { tp.cut_key = cut_key; tp.redo = redo; tp.any_redo = any_redo; }
  size_t sm = (size_t)kTopCap * sizeof(u64);
  static bool attr_set = false;
  if (!attr_set) { SSDK_CHECK_CUDA(cudaFuncSetAttribute(topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm)); attr_set = true; }
  topk_kernel<<<B, kTopThreads, sm, stream>>>(tp);
  SSDK_COUNT_LAUNCH(ctx);
  if (two_stage) {
    // classes that failed the check: full scan (the other CTAs exit at once), then the top-k of the affected images again
    np.band_cap = kNmsCap; np.max_bands = 0; np.cut_key = nullptr; np.redo = redo;
    rc = nms(np);
    if (rc) return rc;
    tp.cut_key = nullptr; tp.redo = nullptr; tp.any_redo = nullptr; tp.only_if = any_redo;
    topk_kernel<<<B, kTopThreads, sm, stream>>>(tp);
    SSDK_COUNT_LAUNCH(ctx);
  }
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

size_t nms_scratch_bytes(int B, int S, int kmax) {
  return align_up((size_t)B * S * kmax * 4, 256) * 2 + align_up((size_t)B * S * 4, 256) * 3 + align_up((size_t)B * S * kmax * 8, 256) +
         align_up((size_t)B * 4, 256);
}

}  // namespace

extern "C" int ssdk_decode(ssdk_ctx* ctx, const ssdk_decode_cfg* cfg, const float* y_pred_dev, int B,
                           float* out_dev, int* out_counts_dev, int* out_index_dev, void* stream_) {
  SSDK_REQUIRE(ctx && cfg && y_pred_dev && out_dev && out_counts_dev && B > 0, "ssdk_decode: bad argument");
  SSDK_REQUIRE(cfg->P > 0 && cfg->n_classes_total > 1, "ssdk_decode: bad P / n_classes");
  SSDK_REQUIRE(cfg->coords >= 0 && cfg->coords <= 2, "Unexpected value for `input_coords`. Supported input coordinate formats are 'minmax', 'corners' and 'centroids'.");
  SSDK_REQUIRE(!cfg->layer_semantics || cfg->coords == SSDK_COORDS_CENTROIDS,
               "The DetectionOutput layer currently only supports the 'centroids' coordinate format.");
  SSDK_REQUIRE(!cfg->normalize_coords || (cfg->img_height > 0 && cfg->img_width > 0),
               "If relative box coordinates are supposed to be converted to absolute coordinates, the decoder needs the image size");
  SSDK_REQUIRE(cfg->max_out > 0, "ssdk_decode: max_out must be > 0");
  SSDK_REQUIRE(cfg->top_k <= kTopCap, "ssdk_decode: top_k > %d is not supported", kTopCap);
  SSDK_REQUIRE(cfg->n_classes_total - 1 <= 1024, "ssdk_decode: more than 1024 classes are not supported");
  cudaStream_t stream = (cudaStream_t)stream_;
  const int P = cfg->P, C = cfg->n_classes_total, W = C + 12;
  const int S = (cfg->mode == SSDK_DECODE_PER_CLASS) ? (C - 1) : 1;
  const int layer = cfg->layer_semantics ? 1 : 0;
  const int np_f32 = (!layer && cfg->coords == SSDK_COORDS_CORNERS) ? 1 : 0;
  const int box_f64 = (!layer && !np_f32) ? 1 : 0;
  const int cap = layer ? cfg->nms_max_output : P;
  SSDK_REQUIRE(cap > 0, "ssdk_decode: nms_max_output_size must be > 0");
  size_t b_boxes = align_up((size_t)B * P * 4 * (box_f64 ? 8 : 4), 256);
  size_t b_scores = align_up((size_t)B * S * P * 4, 256);
  size_t b_labels = align_up((size_t)B * P * 4, 256);
  size_t total = b_boxes + b_scores + b_labels + nms_scratch_bytes(B, S, cap);
  int rc = ctx->ws[0].ensure(total);
  if (rc) return rc;
  unsigned char* base = reinterpret_cast<unsigned char*>(ctx->ws[0].ptr);
  void* boxes = base;
  float* scores = reinterpret_cast<float*>(base + b_boxes);
  int* labels = reinterpret_cast<int*>(base + b_boxes + b_scores);
  unsigned char* scratch = base + b_boxes + b_scores + b_labels;

  PrepParams pp{};
  pp.y = y_pred_dev; pp.P = P; pp.C = C; pp.W = W; pp.mode = cfg->mode; pp.layer = layer; pp.coords = cfg->coords;
  pp.normalize = cfg->normalize_coords; pp.img_w = (float)cfg->img_width; pp.img_h = (float)cfg->img_height;
  pp.boxes = boxes; pp.scores = scores; pp.labels = labels; pp.box_f64 = box_f64;
  size_t sm = (size_t)256 * W * sizeof(float);
  SSDK_REQUIRE(sm <= 227 * 1024, "ssdk_decode: too many classes (%d) for the staging buffer", C);
  if (sm > 48 * 1024) SSDK_CHECK_CUDA(cudaFuncSetAttribute(dec_prepare_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  dim3 grid(ceil_div(P, 256), B);
  dec_prepare_kernel<<<grid, 256, sm, stream>>>(pp);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());

  int strict = 1;
  if (!layer && cfg->mode == SSDK_DECODE_FAST) strict = 0;      // decode_detections_fast uses >= (:325)
  double iou_thr = cfg->iou_threshold;
  if (!layer && cfg->mode == SSDK_DECODE_FAST && !(cfg->iou_threshold > 0.0)) iou_thr = INFINITY;   // "if iou_threshold:" (:326)
  return run_nms_topk(ctx, B, P, S, layer, box_f64, np_f32, scores, cfg->mode == SSDK_DECODE_FAST ? labels : nullptr, boxes,
                      strict, cfg->confidence_thresh, iou_thr, cfg->border_d, cap, cfg->top_k, cfg->max_out, scratch,
                      out_dev, out_counts_dev, out_index_dev, stream);
}

extern "C" int ssdk_nms(ssdk_ctx* ctx, const float* boxes_dev, const float* scores_dev, int B, int n,
                        double confidence_thresh, double iou_threshold, int nms_max_output, int top_k,
                        float* out_dev, int* out_counts_dev, int* out_index_dev, void* stream_) {
  SSDK_REQUIRE(ctx && boxes_dev && scores_dev && out_dev && out_counts_dev && B > 0 && n > 0, "ssdk_nms: bad argument");
  SSDK_REQUIRE(nms_max_output > 0 && top_k > 0 && top_k <= kTopCap, "ssdk_nms: bad nms_max_output / top_k");
  size_t total = nms_scratch_bytes(B, 1, nms_max_output);
  int rc = ctx->ws[1].ensure(total);
  if (rc) return rc;
  return run_nms_topk(ctx, B, n, 1, 1, 0, 0, scores_dev, nullptr, boxes_dev, 1, confidence_thresh, iou_threshold, 0,
                      nms_max_output, top_k, top_k, reinterpret_cast<unsigned char*>(ctx->ws[1].ptr), out_dev,
                      out_counts_dev, out_index_dev, (cudaStream_t)stream_);
}
