// SSDLoss on sm_90a as ONE kernel (forward, backward, or both).  Reference: keras_loss_function/keras_ssd_loss.py:53-211.
//
// ssd_loss_kernel is a persistent cooperative kernel (all CTAs co-resident, grid-wide barriers between phases):
//   phase A  tiles of 128 prediction rows stream through shared memory with cp.async.bulk + mbarrier (two stages), one thread
//            per row: log-loss (:93-95), smooth-L1 (:72-75), positives / negatives (:139-140); per-tile partial sums in a
//            fixed order; the per-box negative losses (B*P floats, L2 resident) and a two-level histogram of their order
//            keys (65536 fine bins by global atomics, 2048 coarse bins = sums of 32 fine bins).
//   phase B  every CTA derives k (:166) and the fine bin that holds the k-th largest negative loss from the (small) coarse
//            histogram; second histogram over the low 16 key bits of the boxes in that bin.
//   phase C  threshold key T; only if fewer boxes than those equal to T are wanted, the tf.nn.top_k tie rule (lower flat
//            index first, :179-183) is resolved with per-tile tie counts and one scan.
//   phase D  masked negative sums per tile, and/or the gradient rows (mask held constant) staged in shared memory and
//            written with cp.async.bulk; the last CTA to finish (atomic ticket) reduces the tile partials per image:
//            (pos + neg + alpha*loc) / max(1, n_pos) * B (:204-209).
// All sums that reach the result are reduced in a fixed order (per tile, then per image), histograms and counts are
// integers: the output is deterministic.  The same phases run as separate launches (ssdk_ssd_loss_phase) when the batch is
// spread over several GPUs and the reference's batch-global quantities (n_positive :143, the top-k :179-183) must be
// global too: the histograms and counts in the caller-provided workspace are summed with NCCL between the phases.
#include "common.cuh"
#include "tc.cuh"
#include <cooperative_groups.h>
#include <cmath>

namespace cg = cooperative_groups;
using namespace ssdk;

namespace {

constexpr int kRows = 128;             // rows per tile == threads per CTA
constexpr int kCoarse = 2048;          // coarse bins: key >> 21 (level 1), (key >> 5) & 2047 (level 2)
constexpr int kFine = 65536;           // fine bins:   key >> 16 (level 1), key & 65535 (level 2)
constexpr int kCache = 2048;           // per-CTA direct-mapped cache of level-1 fine bins (slot = bin & 2047, tag = bin >> 11)
constexpr unsigned kZeroKey = 0x80000000u;

// order-preserving key: larger float -> larger unsigned.  -0 and +0 share kZeroKey: the histograms count both as the zero bin,
// and tf.nn.top_k, which the selection restates, does not tell them apart (the lower flat index wins between them).
__device__ __forceinline__ unsigned okey(float f) {
  if (f == 0.f) return kZeroKey;
  unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

struct LossArgs {
  const float* y_true; const float* y_pred;
  int B, P, C;
  int tiles_per_img, n_tiles;
  long long n_total;                   // boxes the selection runs over (B*P, or the global count in multi-GPU mode)
  int global_B;                        // batch size in the normalisation (:209)
  int ratio, n_neg_min;
  float alpha;
  // workspace
  float* cls; float* negl;             // [B*P]
  double* part;                        // [n_tiles*2] sum cls*pos, sum loc*pos
  double* negpart;                     // [n_tiles]
  int* tile_ties;                      // [n_tiles + 1]
  unsigned long long* counts;          // [0] sum of positives in 32.32 fixed point, [1] non-zero negative losses
  unsigned* hist1;                     // [kCoarse + kFine]
  unsigned* hist2;                     // [kCoarse + kFine]
  unsigned* hist_next;                 // the other parity's 2*(kCoarse+kFine) ints, cleared for the next call (or NULL)
  int* ticket;
  const int* ties_all; int rank;       // multi-GPU: boxes equal to T on every rank (all-gathered), this rank's index
  int* ties_local;                     // multi-GPU: out, boxes equal to T on this rank
  // outputs
  float* out_loss; int* out_stats; const float* upstream; float* out_grad;
  int stages;                          // shared-memory stages of phase A / D tile loads (1 or 2)
  int bulk_ok;                         // rows of a tile start 16-byte aligned: cp.async.bulk is usable
};

struct Sel {                           // what phases C / D know about the hard-negative selection
  int none;                            // no negatives are kept
  int k, n_pos, nnz;
  float inv_norm;
  unsigned T;                          // threshold key
  long long want;                      // boxes equal to T that are kept, in flat-index order
  long long ties_total;
};

// ---- shared-memory tile loads ----------------------------------------------------------------------------------
// Loads rows [row0, row0+rows) of y_true and y_pred (W floats each) into the stage buffers.  Bulk path: one elected thread
// issues two copies that complete on the stage's mbarrier; fallback: all threads copy and the caller's __syncthreads publishes.
__device__ __forceinline__ void tile_load(const LossArgs& a, size_t flat_row0, int rows, float* s_t, float* s_p, uint32_t bar) {
  const int W = a.C + 12;
  const float* gt = a.y_true + flat_row0 * W;
  const float* gp = a.y_pred + flat_row0 * W;
  const uint32_t bytes = (uint32_t)rows * W * 4u;
  if (a.bulk_ok) {
    if (threadIdx.x == 0) {
      mbar_expect_tx(bar, 2u * bytes);
      bulk_load(smem_u32(s_t), gt, bytes, bar);
      bulk_load(smem_u32(s_p), gp, bytes, bar);
    }
  } else {
    for (int i = threadIdx.x; i < rows * W; i += kRows) { s_t[i] = gt[i]; s_p[i] = gp[i]; }
  }
}

template <typename T>
__device__ __forceinline__ T block_sum(T v, T* s_red) {       // fixed-order block reduction (4 warps), result in every thread
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  return s_red[0] + s_red[1] + s_red[2] + s_red[3];
}

// ---- selection: which bin holds the `want`-th largest key -----------------------------------------------------------
// hist = [coarse (kCoarse) | fine (kFine)], fine bin f belongs to coarse bin f >> 5.  `zero_fine` (or -1) is a fine bin that
// additionally holds `n_zero` boxes that were never added atomically (the boxes whose negative loss is exactly 0).
// Returns the fine bin; `want` becomes the rank inside it, `in_bin` its population.  All threads get the same answer.
__device__ void select_bin(const unsigned* hist, int zero_fine, long long n_zero, long long& want, long long& in_bin, int& bin,
                           long long* s_scan) {
  // Every global load below is issued by many threads at once (a serial scan by one thread would pay the L2 latency per bin).
  const int t = threadIdx.x;
  __shared__ long long s_misc[4];
  // coarse: 2048 bins / 128 threads = 16 each, thread t owns bins c_hi .. c_hi - 15 (scanned from the top)
  const int c_hi = kCoarse - 1 - t * 16;
  unsigned cv[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) cv[i] = __ldcg(hist + c_hi - i);
  long long mine = 0;
#pragma unroll
  for (int i = 0; i < 16; ++i) mine += (long long)cv[i] + ((zero_fine >= 0 && (zero_fine >> 5) == c_hi - i) ? n_zero : 0);
  __syncthreads();
  s_scan[t] = mine;
  __syncthreads();
  if (t == 0) {
    long long acc = 0; int owner = kRows - 1;
    for (int i = 0; i < kRows; ++i) { if (acc + s_scan[i] >= want) { owner = i; break; } acc += s_scan[i]; }
    s_misc[0] = owner; s_misc[1] = acc;
  }
  __syncthreads();
  if (t == (int)s_misc[0]) {                           // the owner scans its 16 bins (already in registers)
    long long acc = s_misc[1];
    int csel = c_hi - 15;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const long long v = (long long)cv[i] + ((zero_fine >= 0 && (zero_fine >> 5) == c_hi - i) ? n_zero : 0);
      if (acc + v >= want) { csel = c_hi - i; break; }
      acc += v;
    }
    s_misc[2] = csel; s_misc[3] = acc;
  }
  __syncthreads();
  const int csel = (int)s_misc[2];
  if (t < 32) {                                         // the 32 fine bins of that coarse bin, one per lane, top first
    const int f = csel * 32 + 31 - t;
    s_scan[t] = (long long)__ldcg(hist + kCoarse + f) + ((f == zero_fine) ? n_zero : 0);
  }
  __syncthreads();
  if (t == 0) {
    long long acc = s_misc[3];
    int fsel = csel * 32; long long pop = 0;
    for (int i = 0; i < 32; ++i) {
      const long long v = s_scan[i];
      if (acc + v >= want) { fsel = csel * 32 + 31 - i; pop = v; break; }
      acc += v;
    }
    s_misc[0] = fsel; s_misc[1] = want - acc; s_misc[2] = pop;
  }
  __syncthreads();
  bin = (int)s_misc[0]; want = s_misc[1]; in_bin = s_misc[2];
  __syncthreads();
}

__device__ void read_counts(const LossArgs& a, Sel& s) {
  const unsigned long long pos_fx = __ldcg(a.counts), nnz = __ldcg(a.counts + 1);
  const float n_pos_f = (float)((double)pos_fx / 4294967296.0);         // tf.reduce_sum(positives) (:143)
  s.n_pos = (int)n_pos_f;                                                // tf.to_int32
  s.nnz = (int)nnz;
  long long k = (long long)a.ratio * s.n_pos;
  k = k > a.n_neg_min ? k : a.n_neg_min;
  k = k < (long long)nnz ? k : (long long)nnz;                           // :166
  s.k = (int)k;
  s.inv_norm = 1.0f / fmaxf(1.0f, n_pos_f);
  s.none = (k <= 0 || nnz == 0) ? 1 : 0;
}

// level 1: returns the high 16 key bits of the k-th largest negative loss and the rank wanted inside that bin
__device__ void level1(const LossArgs& a, const Sel& s, int& b1, long long& want, long long* s_scan) {
  long long in_bin;
  want = s.k;
  select_bin(a.hist1, (int)(kZeroKey >> 16), a.n_total - s.nnz, want, in_bin, b1, s_scan);
}

__device__ __forceinline__ bool taken(const Sel& s, unsigned key, long long tie_rank) {
  if (s.none) return false;
  return key > s.T || (key == s.T && tie_rank < s.want);
}

// ---- phase A -----------------------------------------------------------------------------------------------------------
__device__ void phase_a(const LossArgs& a, unsigned char* smem, uint32_t bar0) {
  const int W = a.C + 12, C = a.C;
  const int tid = threadIdx.x;
  const size_t stage_floats = (size_t)kRows * W;
  float* s_buf = reinterpret_cast<float*>(smem);                        // [stages][2][kRows*W]
  unsigned* s_coarse = reinterpret_cast<unsigned*>(smem + (size_t)a.stages * 2 * stage_floats * 4);   // [kCoarse]
  // The negative losses of one batch crowd into a few hundred fine bins (same exponent, neighbouring mantissas): one global
  // atomic per box serialises on those addresses in L2.  Each CTA counts in a direct-mapped shared-memory cache instead and adds
  // its totals once at the end; a box whose slot is held by another bin falls back to the global atomic.
  int* s_ftag = reinterpret_cast<int*>(s_coarse + kCoarse);             // [kCache] bin >> 11 of the slot's owner, -1 = free
  unsigned* s_fcnt = reinterpret_cast<unsigned*>(s_ftag + kCache);      // [kCache]
  __shared__ double s_red[4];
  __shared__ unsigned long long s_redu[4];
  for (int i = tid; i < kCoarse; i += kRows) s_coarse[i] = 0;
  for (int i = tid; i < kCache; i += kRows) { s_ftag[i] = -1; s_fcnt[i] = 0; }
  if (a.hist_next)                                                       // clear the other parity's histograms for the next call
    for (size_t i = (size_t)blockIdx.x * kRows + tid; i < 2ull * (kCoarse + kFine); i += (size_t)gridDim.x * kRows) a.hist_next[i] = 0;
  __syncthreads();
  int it = 0;
  // prologue: first tile(s) in flight
  for (int st = 0; st < a.stages; ++st) {
    const int t = blockIdx.x + st * gridDim.x;
    if (t < a.n_tiles) {
      const int b = t / a.tiles_per_img, blk = t - b * a.tiles_per_img;
      const int rows = min(kRows, a.P - blk * kRows);
      tile_load(a, (size_t)b * a.P + (size_t)blk * kRows, rows, s_buf + (size_t)st * 2 * stage_floats, s_buf + (size_t)st * 2 * stage_floats + stage_floats,
                bar0 + 8u * st);
    }
  }
  for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x, ++it) {
    const int st = it % a.stages;
    const uint32_t parity = (uint32_t)(it / a.stages) & 1u;
    const int b = t / a.tiles_per_img, blk = t - b * a.tiles_per_img;
    const int rows = min(kRows, a.P - blk * kRows);
    const float* s_t = s_buf + (size_t)st * 2 * stage_floats;
    const float* s_p = s_t + stage_floats;
    if (a.bulk_ok) mbar_wait(bar0 + 8u * st, parity); else __syncthreads();
    double pc = 0, loc = 0; unsigned long long pos_fx = 0, nz = 0;
    if (tid < rows) {
      const float* yt = s_t + (size_t)tid * W;
      const float* yp = s_p + (size_t)tid * W;
      float acc = 0.f, pmax = -INFINITY;
      for (int c = 0; c < C; ++c) {
        const float tv = yt[c];
        if (tv != 0.f) acc += tv * logf(fmaxf(yp[c], 1e-15f));          // :93-95
        if (c >= 1) pmax = fmaxf(pmax, tv);                              // :140
      }
      float l = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float d = yt[C + j] - yp[C + j];
        const float ad = fabsf(d);
        l += (ad < 1.0f) ? 0.5f * d * d : ad - 0.5f;                     // :72-74
      }
      const float cls = -acc;
      const float nl = cls * yt[0];                                      // :139,151
      const size_t flat = (size_t)b * a.P + (size_t)blk * kRows + tid;
      a.cls[flat] = cls;
      a.negl[flat] = nl;
      pc = (double)(cls * pmax); loc = (double)(l * pmax);
      pos_fx = (unsigned long long)llrint((double)pmax * 4294967296.0);
      if (nl != 0.f) {
        nz = 1;
        const unsigned key = okey(nl);
        const int fine = (int)(key >> 16), slot = fine & (kCache - 1), tag = fine >> 11;
        int cur = *reinterpret_cast<volatile int*>(s_ftag + slot);
        if (cur < 0) { const int old = atomicCAS(s_ftag + slot, -1, tag); cur = old < 0 ? tag : old; }
        if (cur == tag) atomicAdd(s_fcnt + slot, 1u); else atomicAdd(a.hist1 + kCoarse + fine, 1u);
        atomicAdd(s_coarse + (key >> 21), 1u);
      }
    }
    // the stage is free again once every thread has read its row: refill it with the tile `stages` iterations ahead
    const int tn = t + a.stages * gridDim.x;
    pc = block_sum(pc, s_red);
    loc = block_sum(loc, s_red);
    {
      unsigned long long v = pos_fx;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      unsigned long long w = nz;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) w += __shfl_xor_sync(0xffffffffu, w, o);
      __syncthreads();
      if ((tid & 31) == 0) { s_redu[tid >> 5] = v; s_red[tid >> 5] = (double)w; }
      __syncthreads();
      if (tid == 0) {
        a.part[(size_t)t * 2] = pc; a.part[(size_t)t * 2 + 1] = loc;
        const unsigned long long pv = s_redu[0] + s_redu[1] + s_redu[2] + s_redu[3];
        const unsigned long long nv = (unsigned long long)(s_red[0] + s_red[1] + s_red[2] + s_red[3]);
        if (pv) atomicAdd(a.counts, pv);
        if (nv) atomicAdd(a.counts + 1, nv);
      }
    }
    if (tn < a.n_tiles) {                                                // (the block_sum barriers above ordered all row reads before this)
      const int b2 = tn / a.tiles_per_img, blk2 = tn - b2 * a.tiles_per_img;
      const int rows2 = min(kRows, a.P - blk2 * kRows);
      tile_load(a, (size_t)b2 * a.P + (size_t)blk2 * kRows, rows2, s_buf + (size_t)st * 2 * stage_floats,
                s_buf + (size_t)st * 2 * stage_floats + stage_floats, bar0 + 8u * st);
    }
  }
  __syncthreads();
  for (int i = tid; i < kCoarse; i += kRows) { const unsigned v = s_coarse[i]; if (v) atomicAdd(a.hist1 + i, v); }
  for (int i = tid; i < kCache; i += kRows) { const unsigned v = s_fcnt[i]; if (v) atomicAdd(a.hist1 + kCoarse + ((s_ftag[i] << 11) | i), v); }
}

// ---- phase B: histogram of the low key bits inside the level-1 bin ---------------------------------------------------
__device__ void phase_b(const LossArgs& a, const Sel& s, int b1) {
  if (s.none) return;
  const long long n_local = (long long)a.B * a.P;
  for (long long i = (long long)blockIdx.x * kRows + threadIdx.x; i < n_local; i += (long long)gridDim.x * kRows) {
    const float nl = __ldcg(a.negl + i);
    if (nl == 0.f) continue;
    const unsigned key = okey(nl);
    if ((int)(key >> 16) != b1) continue;
    atomicAdd(a.hist2 + kCoarse + (key & 0xffffu), 1u);
    atomicAdd(a.hist2 + ((key >> 5) & 0x7ffu), 1u);
  }
}

// threshold key and tie bookkeeping from the two histograms (every CTA computes the same)
__device__ void finish_select(const LossArgs& a, Sel& s, int b1, long long want1, long long* s_scan) {
  s.T = 0; s.want = 0; s.ties_total = 0;
  if (s.none) return;
  long long want = want1, in_bin; int lo;
  const bool zero_bin = (b1 == (int)(kZeroKey >> 16));
  select_bin(a.hist2, zero_bin ? 0 : -1, zero_bin ? (a.n_total - s.nnz) : 0, want, in_bin, lo, s_scan);
  s.T = ((unsigned)b1 << 16) | (unsigned)lo;
  s.want = want; s.ties_total = in_bin;
}

// per-tile number of boxes whose key equals T (flat order == tile order)
__device__ void phase_ties(const LossArgs& a, const Sel& s) {
  __shared__ int s_cnt[4];
  for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x) {
    const int b = t / a.tiles_per_img, blk = t - b * a.tiles_per_img;
    const int rows = min(kRows, a.P - blk * kRows);
    bool tie = false;
    if ((int)threadIdx.x < rows) tie = okey(__ldcg(a.negl + (size_t)b * a.P + (size_t)blk * kRows + threadIdx.x)) == s.T;
    const unsigned m = __ballot_sync(0xffffffffu, tie);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_cnt[threadIdx.x >> 5] = __popc(m);
    __syncthreads();
    if (threadIdx.x == 0) a.tile_ties[t] = s_cnt[0] + s_cnt[1] + s_cnt[2] + s_cnt[3];
  }
}

// exclusive prefix of tile_ties in place (one CTA); tile_ties[n_tiles] = total
__device__ void scan_ties(const LossArgs& a) {
  __shared__ long long s_part[kRows];
  const int per = (a.n_tiles + kRows - 1) / kRows;
  const int lo = threadIdx.x * per, hi = min(a.n_tiles, lo + per);
  long long sum = 0;
  for (int i = lo; i < hi; ++i) sum += a.tile_ties[i];
  s_part[threadIdx.x] = sum;
  __syncthreads();
  long long base = 0;
  for (int i = 0; i < (int)threadIdx.x; ++i) base += s_part[i];
  for (int i = lo; i < hi; ++i) { const int v = a.tile_ties[i]; a.tile_ties[i] = (int)base; base += v; }
  if (threadIdx.x == kRows - 1) a.tile_ties[a.n_tiles] = (int)base;
}

// ---- phase D: masked negative sums and/or the gradient, then the per-image totals ----------------------------------------
__device__ void phase_d(const LossArgs& a, const Sel& s, bool ordered_ties, long long tie_base, unsigned char* smem, uint32_t bar0) {
  const int W = a.C + 12, C = a.C;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  __shared__ double s_red[4];
  __shared__ int s_cnt[4];
  __shared__ int s_is_last;
  const size_t stage_floats = (size_t)kRows * W;
  float* s_t = reinterpret_cast<float*>(smem);
  float* s_p = s_t + stage_floats;
  float* s_g = s_p + stage_floats;                                       // gradient rows (only with out_grad)
  uint32_t parity = 0;
  bool store_pending = false;
  for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x) {
    const int b = t / a.tiles_per_img, blk = t - b * a.tiles_per_img;
    const int rows = min(kRows, a.P - blk * kRows);
    const size_t flat0 = (size_t)b * a.P + (size_t)blk * kRows;
    if (a.out_grad) tile_load(a, flat0, rows, s_t, s_p, bar0);           // overlaps the mask computation below
    float nl = 0.f, cls = 0.f; unsigned key = 0; bool tie = false;
    if (tid < rows) { nl = __ldcg(a.negl + flat0 + tid); cls = __ldcg(a.cls + flat0 + tid); key = okey(nl); tie = (key == s.T); }
    long long tie_rank = 0;
    if (ordered_ties) {                                                  // rank of this box among the boxes equal to T, flat order
      const unsigned m = __ballot_sync(0xffffffffu, tie);
      __syncthreads();
      if (lane == 0) s_cnt[warp] = __popc(m);
      __syncthreads();
      int before = 0;
      for (int w = 0; w < warp; ++w) before += s_cnt[w];
      tie_rank = tie_base + a.tile_ties[t] + before + __popc(m & ((1u << lane) - 1));
    }
    const bool take = (tid < rows) && taken(s, key, tie_rank);
    if (a.out_loss) {
      const double v = block_sum(take ? (double)cls : 0.0, s_red);
      if (tid == 0) a.negpart[t] = v;
    }
    if (a.out_grad) {
      if (store_pending) { if (tid == 0) bulk_wait_read<0>(); }
      if (a.bulk_ok) mbar_wait(bar0, parity);
      __syncthreads();
      parity ^= 1u;
      if (tid < rows) {
        const float* yt = s_t + (size_t)tid * W;
        const float* yp = s_p + (size_t)tid * W;
        float* g = s_g + (size_t)tid * W;
        float pmax = -INFINITY;
        for (int c = 1; c < C; ++c) pmax = fmaxf(pmax, yt[c]);
        const float up = a.upstream ? a.upstream[b] : (1.0f / (float)a.global_B);
        const float scale = up * (float)a.global_B * s.inv_norm;
        const float w_cls = (pmax + (take ? 1.f : 0.f)) * scale;
        const float w_loc = pmax * scale * a.alpha;
        for (int c = 0; c < C; ++c) {
          const float tv = yt[c];
          float gv = 0.f;
          if (tv != 0.f) { const float q = yp[c]; gv = (q >= 1e-15f) ? (-tv / q) * w_cls : 0.f; }
          g[c] = gv;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float d = yp[C + j] - yt[C + j];
          g[C + j] = ((fabsf(d) < 1.0f) ? d : (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f))) * w_loc;
        }
#pragma unroll
        for (int j = 4; j < 12; ++j) g[C + j] = 0.f;
      }
      fence_proxy_async();
      __syncthreads();
      float* dst = a.out_grad + flat0 * W;
      const size_t n_f = (size_t)rows * W;
      if (a.bulk_ok && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) && (((n_f * 4) & 15) == 0)) {
        if (tid == 0) { bulk_store(dst, smem_u32(s_g), (uint32_t)(n_f * 4)); bulk_commit(); }
        store_pending = true;
      } else {
        for (size_t i = tid; i < n_f; i += kRows) dst[i] = s_g[i];
      }
    }
  }
  if (tid == 0) bulk_wait<0>();
  if (!a.out_loss) return;
  // last CTA: per-image totals in a fixed order
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    const int old = atomicAdd(a.ticket, 1);
    s_is_last = (old == (int)gridDim.x - 1);
    if (s_is_last) *a.ticket = 0;
    __threadfence();
  }
  __syncthreads();
  if (!s_is_last) return;
  for (int b = warp; b < a.B; b += kRows / 32) {               // one warp per image: lanes stride over the tiles, fixed-order tree
    double pc = 0, loc = 0, ng = 0;
    for (int i = lane; i < a.tiles_per_img; i += 32) {
      const size_t t = (size_t)b * a.tiles_per_img + i;
      pc += __ldcg(a.part + t * 2); loc += __ldcg(a.part + t * 2 + 1); ng += __ldcg(a.negpart + t);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      pc += __shfl_xor_sync(0xffffffffu, pc, o); loc += __shfl_xor_sync(0xffffffffu, loc, o); ng += __shfl_xor_sync(0xffffffffu, ng, o);
    }
    const double total = (pc + ng + (double)a.alpha * loc) * (double)s.inv_norm;    // :204
    if (lane == 0) a.out_loss[b] = (float)(total * (double)a.global_B);             // :209
  }
  if (tid == 0 && a.out_stats) {
    a.out_stats[0] = s.n_pos; a.out_stats[1] = s.nnz; a.out_stats[2] = s.none ? 0 : s.k; a.out_stats[3] = s.none ? 0 : (int)s.want;
  }
}

// shared-memory layout (dynamic): phase A: stages * 2 tiles | coarse histogram;  phase D: y_true tile | y_pred tile | grad tile
__host__ __device__ inline size_t loss_smem_bytes(int W, int stages, bool grad) {
  const size_t tile = (size_t)kRows * W * 4;
  const size_t pa = (size_t)stages * 2 * tile + kCoarse * 4 + kCache * 8;
  const size_t pd = grad ? 3 * tile : 0;
  return (pa > pd ? pa : pd) + 128;
}

__device__ __forceinline__ uint32_t setup_barriers(uint64_t* bars) {
  const uint32_t bar0 = smem_u32(bars);
  if (threadIdx.x == 0) {
    mbar_init(bar0, 1); mbar_init(bar0 + 8, 1); mbar_init(bar0 + 16, 1);
    mbar_init_fence();
  }
  __syncthreads();
  return bar0;
}

// The fused kernel.  Cooperative launch: grid-wide barriers separate the phases.
__global__ void __launch_bounds__(kRows) ssd_loss_kernel(const __grid_constant__ LossArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ uint64_t s_bars[3];
  __shared__ long long s_scan[kRows];
  cg::grid_group grid = cg::this_grid();
  const uint32_t bar0 = setup_barriers(s_bars);
  phase_a(a, smem, bar0);
  grid.sync();
  Sel s;
  read_counts(a, s);
  int b1 = 0; long long want1 = 0;
  if (!s.none) level1(a, s, b1, want1, s_scan);
  phase_b(a, s, b1);
  grid.sync();
  finish_select(a, s, b1, want1, s_scan);
  const bool ordered = !s.none && s.want < s.ties_total;                 // uniform over the grid
  if (ordered) {
    phase_ties(a, s);
    grid.sync();
    if (blockIdx.x == 0) scan_ties(a);
    grid.sync();
  } else {
    s.want = s.ties_total;                                               // every box equal to T is kept: no order needed
  }
  phase_d(a, s, ordered, 0, smem, bar0 + 16);
}

// The same phases as separate launches (multi-GPU, global-batch-exact): 0 = A, 1 = B, 2 = threshold + local ties, 3 = scan, 4 = D
__global__ void __launch_bounds__(kRows) ssd_loss_phase_kernel(const __grid_constant__ LossArgs a, int phase) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ uint64_t s_bars[3];
  __shared__ long long s_scan[kRows];
  const uint32_t bar0 = setup_barriers(s_bars);
  if (phase == 0) { phase_a(a, smem, bar0); return; }
  if (phase == 3) { if (blockIdx.x == 0) scan_ties(a); return; }
  Sel s;
  read_counts(a, s);
  int b1 = 0; long long want1 = 0;
  if (!s.none) level1(a, s, b1, want1, s_scan);
  if (phase == 1) { phase_b(a, s, b1); return; }
  finish_select(a, s, b1, want1, s_scan);
  if (phase == 2) {
    if (!s.none) phase_ties(a, s); else for (int t = blockIdx.x * kRows + threadIdx.x; t <= a.n_tiles; t += gridDim.x * kRows) a.tile_ties[t] = 0;
    return;
  }
  // phase 4: the boxes equal to T are taken in global flat order: lower ranks first
  long long before = 0;
  for (int r = 0; r < a.rank; ++r) before += a.ties_all[r];
  // ranks hold disjoint index ranges in rank order, so this rank's ties rank from `before`; tile_ties was scanned by phase 3
  s.want = s.none ? 0 : s.want;
  Sel s2 = s;
  s2.want = s.want - before;                                             // may be <= 0 (none of ours) or >= our tie count (all of ours)
  phase_d(a, s2, !s.none, 0, smem, bar0 + 16);
}

struct LossWs {
  float* cls; float* negl; double* part; double* negpart; int* tile_ties; unsigned long long* counts; unsigned* hist; int* ticket;
};

size_t al256(size_t v) { return (v + 255) / 256 * 256; }

// Workspace layout (bytes, 256-aligned sections): counts | hist A (2*(coarse+fine)) | hist B | ticket | cls | negl | part | negpart | tile_ties
struct WsLayout { size_t counts, histA, histB, ticket, cls, negl, part, negpart, ties, total; };
WsLayout ws_layout(int B, int P) {
  const size_t N = (size_t)B * P, nt = (size_t)B * ((P + kRows - 1) / kRows);
  WsLayout L;
  size_t o = 0;
  L.counts = o; o += 256;
  L.histA = o; o += al256(2ull * (kCoarse + kFine) * 4);
  L.histB = o; o += al256(2ull * (kCoarse + kFine) * 4);
  L.ticket = o; o += 256;
  L.cls = o; o += al256(N * 4);
  L.negl = o; o += al256(N * 4);
  L.part = o; o += al256(nt * 16);
  L.negpart = o; o += al256(nt * 8);
  L.ties = o; o += al256((nt + 1) * 4);
  L.total = o;
  return L;
}

int check_args(ssdk_ctx* ctx, const float* yt, const float* yp, int B, int P, int C) {
  SSDK_REQUIRE(ctx && yt && yp, "ssd_loss: NULL argument");
  SSDK_REQUIRE(B > 0 && P > 0 && C > 1, "ssd_loss: bad shape");
  SSDK_REQUIRE((long long)B * P < (1ll << 31), "ssd_loss: B*P too large");
  return SSDK_OK;
}

struct LossPlan { int grid; size_t smem; int stages; int bulk_ok; };

// The launch shape of one call (stages, bulk loads, dynamic shared memory, grid) and whether it can run at all.  The launches and
// ssdk_ssd_loss_plan both come here, so a plan is refused exactly when the launch would be; nothing here touches a workspace or
// the histogram parity.
int plan_launch(ssdk_ctx* ctx, const float* y_true, const float* y_pred, int B, int P, int C, bool grad, bool cooperative,
                LossPlan& plan) {
  const int W = C + 12;
  // cp.async.bulk needs 16-byte aligned tile starts: image stride P*W*4 and tile stride 128*W*4 (always a multiple of 16)
  plan.bulk_ok = (((size_t)P * W) % 4 == 0) && ((reinterpret_cast<uintptr_t>(y_true) & 15) == 0) && ((reinterpret_cast<uintptr_t>(y_pred) & 15) == 0) ? 1 : 0;
  plan.stages = loss_smem_bytes(W, 2, grad) > 100 * 1024 ? 1 : 2;
  plan.smem = loss_smem_bytes(W, plan.stages, grad);
  // the dynamic shared memory a CTA may opt into is what the device allows per block less the kernels' static arrays
  static size_t static_smem = 0;
  if (!static_smem) {
    cudaFuncAttributes fa, fb;
    SSDK_CHECK_CUDA(cudaFuncGetAttributes(&fa, ssd_loss_kernel));
    SSDK_CHECK_CUDA(cudaFuncGetAttributes(&fb, ssd_loss_phase_kernel));
    static_smem = std::max(fa.sharedSizeBytes, fb.sharedSizeBytes);
  }
  const size_t limit = ctx->prop.sharedMemPerBlockOptin - static_smem;
  SSDK_REQUIRE(plan.smem <= limit, "ssd_loss: %d classes need %zu bytes of shared memory per CTA%s, at most %zu fit", C, plan.smem,
               grad ? " with the gradient" : "", limit);
  const void* kernel = cooperative ? (const void*)ssd_loss_kernel : (const void*)ssd_loss_phase_kernel;
  const int rc = allow_smem(ctx, kernel, plan.smem);             // the occupancy query needs the raised limit
  if (rc) return rc;
  int per_sm = 0;
  SSDK_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kRows, plan.smem));
  SSDK_REQUIRE(per_sm > 0, "ssd_loss: the kernel does not fit on an SM (%zu bytes of shared memory)", plan.smem);
  if (per_sm > 4) per_sm = 4;
  const int n_tiles = B * ((P + kRows - 1) / kRows);
  plan.grid = std::max(1, std::min(n_tiles, per_sm * ctx->sm_count));
  return SSDK_OK;
}

// fills everything of LossArgs that depends on the shapes and the workspace; hist parity chosen by the caller
int fill_args(ssdk_ctx* ctx, LossArgs& a, const float* y_true, const float* y_pred, int B, int P, int C, int ratio, int n_neg_min,
              float alpha, unsigned char* ws, int parity, bool grad, LossPlan& plan, bool cooperative) {
  const int rc = plan_launch(ctx, y_true, y_pred, B, P, C, grad, cooperative, plan);
  if (rc) return rc;
  const WsLayout L = ws_layout(B, P);
  memset(&a, 0, sizeof(a));
  a.y_true = y_true; a.y_pred = y_pred; a.B = B; a.P = P; a.C = C;
  a.tiles_per_img = (P + kRows - 1) / kRows; a.n_tiles = B * a.tiles_per_img;
  a.n_total = (long long)B * P; a.global_B = B;
  a.ratio = ratio; a.n_neg_min = n_neg_min; a.alpha = alpha;
  a.cls = reinterpret_cast<float*>(ws + L.cls); a.negl = reinterpret_cast<float*>(ws + L.negl);
  a.part = reinterpret_cast<double*>(ws + L.part); a.negpart = reinterpret_cast<double*>(ws + L.negpart);
  a.tile_ties = reinterpret_cast<int*>(ws + L.ties);
  a.counts = reinterpret_cast<unsigned long long*>(ws + L.counts);
  unsigned* hA = reinterpret_cast<unsigned*>(ws + L.histA); unsigned* hB = reinterpret_cast<unsigned*>(ws + L.histB);
  unsigned* cur = parity ? hB : hA;
  a.hist1 = cur; a.hist2 = cur + (kCoarse + kFine);
  a.hist_next = parity ? hA : hB;
  a.ticket = reinterpret_cast<int*>(ws + L.ticket);
  a.bulk_ok = plan.bulk_ok; a.stages = plan.stages;
  return SSDK_OK;
}

long long ws_key(int B, int P) { return (long long)B << 32 | (unsigned)P; }

// context-owned workspace: zeroed when (re)allocated; the caller flips the histogram parity once its launch is enqueued (a call
// refused before the launch must not flip it: the set it would have cleared is the one the next call counts in)
int own_ws(ssdk_ctx* ctx, int B, int P, unsigned char** ws, int* parity, cudaStream_t stream) {
  const WsLayout L = ws_layout(B, P);
  const size_t before = ctx->loss_ws.bytes;
  int rc = ctx->loss_ws.ensure(L.total);
  if (rc) return rc;
  if (ctx->loss_ws.bytes != before || ctx->loss_ws_shape != ws_key(B, P)) {
    SSDK_CHECK_CUDA(cudaMemsetAsync(ctx->loss_ws.ptr, 0, ctx->loss_ws.bytes, stream));   // layout moved: start from clean histograms
    ctx->loss_ws_shape = ws_key(B, P);
    ctx->loss_parity = 0;
  }
  *ws = reinterpret_cast<unsigned char*>(ctx->loss_ws.ptr);
  *parity = ctx->loss_parity;
  return SSDK_OK;
}

int launch_fused(ssdk_ctx* ctx, LossArgs& a, const LossPlan& plan, cudaStream_t stream) {
  // the counts are cleared per call (16 bytes); histograms are self-cleaning (parity), the ticket resets itself
  SSDK_CHECK_CUDA(cudaMemsetAsync(a.counts, 0, 16, stream));
  return launch_cooperative(ctx, ssd_loss_kernel, plan.grid, kRows, plan.smem, stream, a);
}

}  // namespace

extern "C" int ssdk_ssd_loss(ssdk_ctx* ctx, const float* y_true, const float* y_pred, int B, int P, int C, int neg_pos_ratio,
                             int n_neg_min, float alpha, const float* upstream, float* out_loss, int* out_stats, float* out_grad,
                             void* stream_) {
  SSDK_REQUIRE(out_loss != nullptr || out_grad != nullptr, "ssdk_ssd_loss: out_loss and out_grad are both NULL");
  int rc = check_args(ctx, y_true, y_pred, B, P, C);
  if (rc) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  unsigned char* ws; int parity;
  rc = own_ws(ctx, B, P, &ws, &parity, stream);
  if (rc) return rc;
  LossArgs a; LossPlan plan;
  rc = fill_args(ctx, a, y_true, y_pred, B, P, C, neg_pos_ratio, n_neg_min, alpha, ws, parity, out_grad != nullptr, plan, true);
  if (rc) return rc;
  a.out_loss = out_loss; a.out_stats = out_stats; a.upstream = upstream; a.out_grad = out_grad;
  rc = launch_fused(ctx, a, plan, stream);
  if (rc == SSDK_OK) ctx->loss_parity ^= 1;                           // this launch clears the other set for the next call
  return rc;
}

extern "C" int ssdk_ssd_loss_ws_layout(int B, int P, ssdk_loss_ws_layout* out) {
  SSDK_REQUIRE(out && B > 0 && P > 0, "ssdk_ssd_loss_ws_layout: bad argument");
  const WsLayout L = ws_layout(B, P);
  out->bytes = (long long)L.total;
  out->counts_offset = (long long)L.counts; out->counts_n = 2;
  out->hist1_offset = (long long)L.histA; out->hist_n = kCoarse + kFine;
  out->hist2_offset = (long long)(L.histA + (size_t)(kCoarse + kFine) * 4);
  out->ties_offset = (long long)(L.ties + (size_t)B * ((P + kRows - 1) / kRows) * 4);
  return SSDK_OK;
}

extern "C" int ssdk_ssd_loss_plan(ssdk_ctx* ctx, const float* y_true, const float* y_pred, int B, int P, int C, int want_grad,
                                  int cooperative, ssdk_loss_plan* out) {
  SSDK_REQUIRE(out != nullptr, "ssdk_ssd_loss_plan: out is NULL");
  int rc = check_args(ctx, y_true, y_pred, B, P, C);
  if (rc) return rc;
  LossPlan plan;
  rc = plan_launch(ctx, y_true, y_pred, B, P, C, want_grad != 0, cooperative != 0, plan);
  if (rc) return rc;
  out->stages = plan.stages; out->bulk_ok = plan.bulk_ok; out->grid = plan.grid; out->smem_bytes = (long long)plan.smem;
  return SSDK_OK;
}

extern "C" int ssdk_ssd_loss_read_box_losses(ssdk_ctx* ctx, const void* ws_dev, int B, int P, float* cls_dev, float* negl_dev,
                                             void* stream_) {
  SSDK_REQUIRE(ctx && B > 0 && P > 0 && (cls_dev || negl_dev), "ssdk_ssd_loss_read_box_losses: bad argument");
  const unsigned char* ws = reinterpret_cast<const unsigned char*>(ws_dev);
  if (!ws) {
    SSDK_REQUIRE(ctx->loss_ws.ptr && ctx->loss_ws_shape == ws_key(B, P),
                 "ssdk_ssd_loss_read_box_losses: the context's loss workspace does not hold a (%d, %d) batch", B, P);
    ws = reinterpret_cast<const unsigned char*>(ctx->loss_ws.ptr);
  }
  const WsLayout L = ws_layout(B, P);
  const size_t bytes = (size_t)B * P * 4;
  cudaStream_t stream = (cudaStream_t)stream_;
  if (cls_dev) SSDK_CHECK_CUDA(cudaMemcpyAsync(cls_dev, ws + L.cls, bytes, cudaMemcpyDeviceToDevice, stream));
  if (negl_dev) SSDK_CHECK_CUDA(cudaMemcpyAsync(negl_dev, ws + L.negl, bytes, cudaMemcpyDeviceToDevice, stream));
  return SSDK_OK;
}

extern "C" int ssdk_ssd_loss_phase(ssdk_ctx* ctx, int phase, const float* y_true, const float* y_pred, int B, int P, int C,
                                   int neg_pos_ratio, int n_neg_min, float alpha, void* ws_dev, int global_B, const int* ties_all_dev,
                                   int rank, const float* upstream, float* out_loss, int* out_stats, float* out_grad, void* stream_) {
  int rc = check_args(ctx, y_true, y_pred, B, P, C);
  if (rc) return rc;
  SSDK_REQUIRE(ws_dev && phase >= 0 && phase <= 4 && global_B >= B && rank >= 0, "ssdk_ssd_loss_phase: bad argument");
  SSDK_REQUIRE(phase != 4 || ties_all_dev, "ssdk_ssd_loss_phase: phase 4 needs the all-gathered tie counts");
  cudaStream_t stream = (cudaStream_t)stream_;
  LossArgs a; LossPlan plan;
  rc = fill_args(ctx, a, y_true, y_pred, B, P, C, neg_pos_ratio, n_neg_min, alpha, reinterpret_cast<unsigned char*>(ws_dev), 0,
                 out_grad != nullptr && phase == 4, plan, false);
  if (rc) return rc;
  a.hist_next = nullptr;                                              // the caller zeroes the workspace before phase 0
  a.global_B = global_B; a.n_total = (long long)global_B * P;
  a.ties_all = ties_all_dev; a.rank = rank;
  if (phase == 4) { a.out_loss = out_loss; a.out_stats = out_stats; a.upstream = upstream; a.out_grad = out_grad; }
  return launch(ctx, ssd_loss_phase_kernel, phase == 3 ? 1 : plan.grid, kRows, plan.smem, stream, a, phase);
}
