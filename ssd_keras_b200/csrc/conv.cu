// wgmma implicit-GEMM convolution for sm_90a plus the small data-movement kernels around it.
// Reference ops: Conv2D / MaxPooling2D / Lambda preprocessing / L2Normalization / Reshape+softmax+Concat in
// models/keras_ssd300.py:263-419, keras_layers/keras_layer_L2Normalization.py:61-63.
//
// conv_wgmma_kernel -- persistent, 384 threads = a TMA producer warpgroup + two wgmma consumer warpgroups (DESIGN.md section "conv"):
//   GEMM view   D[M = output pixels, N = Cout] = sum over (tap, cin-block) A_tap[M, 64] * W_tap[N, 64]^T.
//   "im2col in the TMA descriptor": the activation tensor is a zero-bordered NHWC buffer viewed as a 2-D
//   matrix [B*Hp*Wp, C]; the A tile of filter tap (kh, kw) for output rows [m0, m0+128) is simply rows
//   [m0 + shift(kh,kw), ...) of that matrix, so each tap is ONE 2-D TMA box load with a row offset, and
//   padding / dilation come for free (the border is zero, rows past the end are TMA zero-filled).
//   Outputs are computed for every position of the padded grid ("virtual rows"); the epilogue stores the
//   valid ones, and m-tiles without any valid row are not scheduled.
//   One producer thread keeps a ring of `stages` {A_hi, A_lo, W_hi, W_lo} 128B-swizzled K-major tiles (full / empty mbarriers)
//   filled across tile boundaries; each consumer warpgroup runs wgmma m64nBNk16 on its 64 rows with fp32 accumulators in
//   registers.  Activation outputs are stored from the registers; head / fp32 / atomic outputs go through a shared-memory tile.
//   Precision: operands are bf16 "hi + lo" pairs; three MMAs per k-step (hi*hi, hi*lo, lo*hi) accumulate
//   in fp32, which reproduces an fp32 convolution to ~1e-5 relative (split=0 issues hi*hi only).
#include "conv.cuh"
#include "tc.cuh"
#include <cudaTypedefs.h>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <vector>

namespace ssdk {

// ------------------------------------------------------------------------------------------------
// TMA descriptor creation (driver entry point resolved at run time)
// ------------------------------------------------------------------------------------------------
static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;

int tma_init() {
  if (g_encode) return SSDK_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  SSDK_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (qres != cudaDriverEntryPointSuccess || !fn) { set_error("cuTensorMapEncodeTiled is not available in this driver"); return SSDK_ERR_CUDA; }
  g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  return SSDK_OK;
}

int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t rows, uint64_t row_stride_bytes,
                 uint32_t box_inner, uint32_t box_rows) {
  int rc = tma_init();
  if (rc) return rc;
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): inner=%llu rows=%llu stride=%llu box=%ux%u base=%p", (int)r,
              (unsigned long long)inner, (unsigned long long)rows, (unsigned long long)row_stride_bytes, box_inner, box_rows, base);
    return SSDK_ERR_CUDA;
  }
  return SSDK_OK;
}

int make_tmap_4d(CUtensorMap* out, const void* base, const uint64_t dims_[4], const uint32_t box_[4]) {
  int rc = tma_init();
  if (rc) return rc;
  cuuint64_t dims[4] = {dims_[0], dims_[1], dims_[2], dims_[3]};
  cuuint64_t strides[3] = {dims_[0] * 2, dims_[0] * dims_[1] * 2, dims_[0] * dims_[1] * dims_[2] * 2};
  cuuint32_t box[4] = {box_[0], box_[1], box_[2], box_[3]};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(4d) failed (%d): dims=%llu,%llu,%llu,%llu box=%u,%u,%u,%u base=%p", (int)r,
              (unsigned long long)dims_[0], (unsigned long long)dims_[1], (unsigned long long)dims_[2], (unsigned long long)dims_[3],
              box_[0], box_[1], box_[2], box_[3], base);
    return SSDK_ERR_CUDA;
  }
  return SSDK_OK;
}

static constexpr int kBM = 128;          // output rows per tile: two warpgroups of 64
static constexpr int kBK = 64;           // channels per k-block = one 128-byte swizzle atom of bf16
static constexpr int kATile = kBM * kBK * 2;   // 16 KB
static constexpr int kAccPad = 4;        // the fp32 accumulator tile in shared memory has rows of BN + 4 floats (conflict-free reads)
static constexpr int kParBytes = 3 * 256 * (int)sizeof(float);   // bias | bn scale | bn shift of one n-tile

static size_t stage_bytes(const ConvArgs& a) { return ((size_t)kATile + (size_t)a.BN * kBK * 2) * (a.split ? 2 : 1); }
// (+32 floats: the 32-column chunk reads of the epilogue may run past the end of a row whose width is not a multiple of 64)
static size_t acc_tile_bytes(int BN) { return ((size_t)kBM * (BN + kAccPad) + 32) * sizeof(float); }
static size_t ring_bytes(const ConvArgs& a) { return std::max(stage_bytes(a) * a.stages, acc_tile_bytes(a.BN)); }
size_t conv_smem_bytes(const ConvArgs& a) { return 1024 + ring_bytes(a) + 256 + kParBytes; }
// As many ring stages ({A_hi, A_lo, W_hi, W_lo} per k-iteration) as shared memory holds, 2 ... 6.
void conv_pick_stages(ConvArgs& a) {
  a.stages = 2;
  while (a.stages < 6) {
    ++a.stages;
    if (conv_smem_bytes(a) > 227 * 1024) { --a.stages; break; }
  }
}

// 32 accumulator columns of this thread's row of the shared-memory accumulator tile
__device__ __forceinline__ void ld_acc32(const float* p, float (&v)[32]) {
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 t = reinterpret_cast<const float4*>(p)[q];
    v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
  }
}

// Accumulator fragment of one warpgroup (64 rows x BN) -> rows [64 * wg, +64) of the shared-memory tile (row pitch BN + kAccPad)
template <int BN>
__device__ __forceinline__ void store_acc_tile(const float (&acc)[BN / 2], float* s_acc, int wg, int warp, int lane) {
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    *reinterpret_cast<float2*>(s_acc + (size_t)r0 * (BN + kAccPad) + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2*>(s_acc + (size_t)(r0 + 8) * (BN + kAccPad) + 8 * j + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
}

// Predictor-head epilogue for a compile-time row width CP4 = n_classes + 4 (25: Pascal VOC, the benchmark configuration): one thread =
// one pixel = n_boxes prior rows.  With CP4 known the accumulator columns of a box are compile-time register indices, so each box
// costs one sweep: <= 2 loads of 32 columns, C bias adds, C exponentials (kept in registers), one reciprocal, C+12 stores.
template <int CP4>
__device__ __forceinline__ void epi_head_fixed(const ConvArgs& args, const float* arow, int n, int pix, const float* s_bias) {
  constexpr int C = CP4 - 4, RW = C + 12;
#pragma unroll
  for (int bx = 0; bx < 8; ++bx) {
    if (bx >= args.head_nb) break;                               // uniform
    constexpr int kMaxCol = 256;
    const int c_lo = bx * CP4;                                   // compile-time after unrolling
    const int k_lo = c_lo >> 5, k_hi = (c_lo + CP4 - 1) >> 5;
    if (c_lo + CP4 > kMaxCol) break;
    float v0[32], v1[32];
    ld_acc32(arow + k_lo * 32, v0);
    if (k_hi != k_lo) ld_acc32(arow + k_hi * 32, v1);
    float e[CP4];
#pragma unroll
    for (int r = 0; r < CP4; ++r) {
      const int col = c_lo + r;
      e[r] = (((col >> 5) == k_lo) ? v0[col & 31] : v1[col & 31]) + s_bias[col];
    }
    float mx = e[0];
#pragma unroll
    for (int r = 1; r < C; ++r) mx = fmaxf(mx, e[r]);
    float sum = 0.f;
#pragma unroll
    for (int r = 0; r < C; ++r) { e[r] = expf(e[r] - mx); sum += e[r]; }
    const float inv = 1.0f / sum;
    const int prior = args.head_prior_off + pix * args.head_nb + bx;
    float* dst = args.out_f32 + ((size_t)n * args.head_P + prior) * RW;
    const float4 an = __ldg(reinterpret_cast<const float4*>(args.head_anchors) + prior);
#pragma unroll
    for (int r = 0; r < C; ++r) dst[r] = e[r] * inv;
#pragma unroll
    for (int r = C; r < CP4; ++r) dst[r] = e[r];
    dst[C + 4] = an.x; dst[C + 5] = an.y; dst[C + 6] = an.z; dst[C + 7] = an.w;
    dst[C + 8] = args.head_var[0]; dst[C + 9] = args.head_var[1]; dst[C + 10] = args.head_var[2]; dst[C + 11] = args.head_var[3];
  }
}

// One group of 8 output channels of the activation-producing epilogues: bias / folded BatchNorm / activation -> bf16 hi+lo planes,
// one 16-byte store per plane.  `v`, `sb`, `ss`, `sh` hold the group's accumulators and parameters, `o` is the output element of
// its first column.  BWD adds what the data-gradient launches need: ReLU'(forward value) mask and accumulation into the output.
template <bool BWD>
__device__ __forceinline__ void epi_split8(const ConvArgs& args, const float (&v)[8], size_t o, const float (&sb)[8], const float (&ss)[8],
                                           const float (&sh)[8]) {
  float mk[8], old[8], f[8];
  if (BWD) {
    unpack8(args.mask_hi ? *reinterpret_cast<const uint4*>(args.mask_hi + o) : make_uint4(0x3f803f80u, 0x3f803f80u, 0x3f803f80u, 0x3f803f80u), mk);
    if (args.accumulate) split_load8(args.out_hi, args.out_lo, o, old);
    else {
#pragma unroll
      for (int e = 0; e < 8; ++e) old[e] = 0.f;
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) f[e] = v[e] + sb[e];
  if (args.bn_scale) {
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = f[e] * ss[e] + sh[e];
  }
  apply_act8(f, args.act);
  if (BWD) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      if (!(mk[e] > 0.f)) f[e] = 0.f;                                     // ReLU'(forward value)
      f[e] += old[e];
    }
  }
  split_store8(args.out_hi, args.out_lo, o, f);
}

// 8 consecutive floats of shared memory (16-byte aligned)
__device__ __forceinline__ void ld_f8(const float* p, float (&v)[8]) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

// ------------------------------------------------------------------------------------------------
// The convolution kernel
// ------------------------------------------------------------------------------------------------
// MODE (ConvArgs::split / acc_split as a compile-time constant, so that every wgmma of the K loop is issued on a uniform path):
//   kSingle  one bf16 product per k-step;
//   kSplitXS bf16x3, the cross terms (hi*lo, lo*hi) accumulate in their own registers and are added to the hi*hi sum after the
//            K loop: the large accumulator takes one rounding add per k-step instead of three (deep-K layers: fc6, fc7,
//            conv6_2 ... stay within 1e-4 of an fp32 convolution).
enum { kSingle = 0, kSplitXS = 2 };
static constexpr int kConvThreads = 384;   // warpgroup 0: TMA producer; warpgroups 1, 2: wgmma consumers of rows [0, 64) / [64, 128)

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }   // the two consumer warpgroups

// The 8 accumulator columns [8j, 8j + 8) of a quad's rows, j = jp + (q & 1), row half h = q >> 1, gathered into lane q (= lane % 4)
// of the quad: a 4 x 4 transpose of float2 pairs.  Lane p holds columns 8j + 2p + {0, 1} of rows r and r + 8 (d[4j + 2h + e]).
template <int N>
__device__ __forceinline__ void quad_gather8(const float (&acc)[N], int jp, int q, float (&v)[8]) {
  const float2 c00 = make_float2(acc[4 * jp], acc[4 * jp + 1]), c01 = make_float2(acc[4 * jp + 2], acc[4 * jp + 3]);
  const float2 c10 = make_float2(acc[4 * jp + 4], acc[4 * jp + 5]), c11 = make_float2(acc[4 * jp + 6], acc[4 * jp + 7]);
  float2 rcv[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int u = q ^ r;                                                   // the unit 2h + jj that lane q ^ r gathers
    const float2 s = (u & 1) ? ((u & 2) ? c11 : c10) : ((u & 2) ? c01 : c00);
    rcv[r].x = __shfl_xor_sync(0xffffffffu, s.x, r);
    rcv[r].y = __shfl_xor_sync(0xffffffffu, s.y, r);
  }
#pragma unroll
  for (int p = 0; p < 4; ++p) {                                            // columns 2p, 2p + 1 came from lane p = q ^ r
    const int r = q ^ p;
    const float2 t = r == 0 ? rcv[0] : (r == 1 ? rcv[1] : (r == 2 ? rcv[2] : rcv[3]));
    v[2 * p] = t.x; v[2 * p + 1] = t.y;
  }
}

template <int BN, int MODE>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_wgmma_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                  const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo,
                  const __grid_constant__ ConvArgs args) {
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  unsigned char* smem_al = smem_dyn + (smem_base - smem_u32(smem_dyn));
  const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31;
  constexpr bool split = MODE == kSplitXS;
  const int S = args.stages;
  constexpr uint32_t kBTile = (uint32_t)BN * kBK * 2;
  const uint32_t b_off = (uint32_t)kATile * (split ? 2u : 1u);            // stage: A_hi | A_lo | W_hi | W_lo
  const uint32_t stage = b_off + kBTile * (split ? 2u : 1u);
  const uint32_t ring = max(stage * (uint32_t)S, ((uint32_t)kBM * (BN + kAccPad) + 32u) * 4u);
  const uint32_t bar_base = smem_base + ring;
  auto full = [&](uint32_t s) { return bar_base + 8u * s; };
  auto empty = [&](uint32_t s) { return bar_base + 8u * ((uint32_t)S + s); };
  const uint32_t staged_free = bar_base + 16u * (uint32_t)S;              // staged epilogues: the tile over the ring has been read
  float* s_acc = reinterpret_cast<float*>(smem_al);                       // staged epilogues, after a tile's K loop: [128][BN + kAccPad]
  float* s_bias = reinterpret_cast<float*>(smem_al + ring + 256);
  float* s_scale = s_bias + BN;
  float* s_shift = s_scale + BN;
  // EPI_SPLIT stores from the accumulator registers; the other epilogues go through a shared-memory tile over the ring, so the
  // producer holds the next tile's loads until that tile has been read
  const bool staged = args.epi != EPI_SPLIT;

  if (tid == 0) {
    prefetch_tmap(&tm_a_hi); prefetch_tmap(&tm_b_hi);
    if (split) { prefetch_tmap(&tm_a_lo); prefetch_tmap(&tm_b_lo); }
    for (int s = 0; s < S; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), 8); }   // empty: one arrival per consumer warp
    mbar_init(staged_free, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int KS = args.k_split > 1 ? args.k_split : 1;
  const int total_tiles = args.n_tiles_m * args.n_tiles_n * KS;
  // work unit t -> output rows [m0, m0 + 128), columns [n0, n0 + BN), k-blocks [kb0, kb0 + nkb), nk = taps * nkb k-iterations
  auto unit = [&](int t, int& m0, int& n0, int& kb0, int& nkb) {
    const int tt = t / KS, ks = t - tt * KS;
    m0 = args.tile_list[tt / args.n_tiles_n] * kBM;
    n0 = (tt % args.n_tiles_n) * BN;
    kb0 = KS > 1 ? ks * args.kb_per : 0;
    const int kb1 = KS > 1 ? min(args.kblocks, kb0 + args.kb_per) : args.kblocks;
    nkb = kb1 - kb0;
  };

  if (wg == 0) {
    // ===================== producer: one thread walks the tile schedule and keeps the ring full across tile boundaries =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (tid != 0) return;
    uint32_t g = 0;                                                        // ring uses so far (slot = g % S, phase = g / S)
    uint32_t lt = 0;                                                       // tiles of this CTA so far
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x, ++lt) {
      int m0, n0, kb0, nkb;
      unit(t, m0, n0, kb0, nkb);
      const int nk = args.KH * args.KW * nkb;
      if (staged && lt > 0) mbar_wait(staged_free, (lt - 1) & 1u);
      // k-iteration i = (tap, k-block): the A tile of tap (kh, kw) is rows [m0 + shift(kh, kw), +128) of the activation matrix
      for (int i = 0; i < nk; ++i) {
        const uint32_t gi = g + (uint32_t)i, s = gi % (uint32_t)S;
        mbar_wait(empty(s), ((gi / (uint32_t)S) & 1u) ^ 1u);
        const int tap = i / nkb, kb = kb0 + (i - tap * nkb), kh = tap / args.KW, kw = tap - kh * args.KW;
        const int row = m0 + args.row_shift[kh] + kw * args.kw_rows;
        const int kcol = (tap * args.kblocks + kb) * kBK + args.b_k_offset;
        const uint32_t dst = smem_base + stage * s;
        mbar_expect_tx(full(s), stage);
        tma_load_2d(dst, &tm_a_hi, kb * kBK, row, full(s));
        tma_load_2d(dst + b_off, &tm_b_hi, kcol, n0, full(s));
        if (split) {
          tma_load_2d(dst + kATile, &tm_a_lo, kb * kBK, row, full(s));
          tma_load_2d(dst + b_off + kBTile, &tm_b_lo, kcol, n0, full(s));
        }
      }
      g += (uint32_t)nk;
    }
    return;
  }

  // ===================== consumers: warpgroup cw computes rows [64 cw, +64) of every tile =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int cw = wg - 1, ctid = tid - 128, cwarp = (tid >> 5) & 3;
  uint32_t g = 0;
  float acc[BN / 2], accx[split ? BN / 2 : 1];
  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    int m0, n0, kb0, nkb;
    unit(t, m0, n0, kb0, nkb);
    const int nk = args.KH * args.KW * nkb;
    if (staged)
      for (int i = ctid; i < BN; i += 256) {
        const int col = n0 + i;
        s_bias[i] = (args.bias && col < args.cout) ? args.bias[col] : 0.f;
        if (args.bn_scale) { s_scale[i] = col < args.cout ? args.bn_scale[col] : 0.f; s_shift[i] = col < args.cout ? args.bn_shift[col] : 0.f; }
      }
    // k-iteration j's MMAs are done: its stage goes back to the producer
    auto release = [&](int j) {
      __syncwarp();
      if (lane == 0) mbar_arrive(empty((g + (uint32_t)j) % (uint32_t)S));
    };
    // (the first k-step overwrites the accumulators; zeroing them here only ends their live range at the previous epilogue)
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
#pragma unroll
    for (int j = 0; j < (split ? BN / 2 : 1); ++j) accx[j] = 0.f;
    wgmma_fence_acc(acc);
    wgmma_fence_acc(accx);
    // Every k-iteration issues all 4 k-steps of its 64-channel block: past the last real channel the A tile is TMA zero fill (or
    // the zeros of a padded operand), so the loop body has no data-dependent branch around the wgmma.  One group stays in flight:
    // the MMAs of iteration i are issued before the stage of iteration i-1 is released.
    for (int i = 0; i < nk; ++i) {
      const uint32_t gi = g + (uint32_t)i, s = gi % (uint32_t)S;
      mbar_wait(full(s), (gi / (uint32_t)S) & 1u);
      const uint32_t a_hi = smem_base + stage * s + (uint32_t)cw * (kATile / 2), b_hi = smem_base + stage * s + b_off;
      constexpr uint64_t kDesc = wgmma_desc_hi(16);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t sc = (i | k) ? 1u : 0u;
        const uint64_t da = wgmma_desc(kDesc, a_hi + 32u * k), db = wgmma_desc(kDesc, b_hi + 32u * k);
        Wgmma<BN, 0, 0>::mma(acc, da, db, sc);
        if constexpr (split) {
          Wgmma<BN, 0, 0>::mma(accx, da, wgmma_desc(kDesc, b_hi + kBTile + 32u * k), sc);
          Wgmma<BN, 0, 0>::mma(accx, wgmma_desc(kDesc, a_hi + kATile + 32u * k), db, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (i > 0) release(i - 1);
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    wgmma_fence_acc(accx);
    if (nk > 0) release(nk - 1);
    g += (uint32_t)nk;
    if constexpr (split) {
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) acc[j] += accx[j];
    }
    const int ncols = min(BN, args.cout - n0);

    if (!staged) {
      // ===================== EPI_SPLIT from the registers: a quad exchange gives each lane 8 consecutive columns of one row ====
      const int q = lane & 3;
      const int v = m0 + cw * 64 + cwarp * 16 + (lane >> 2) + 8 * (q >> 1);   // virtual row of this lane's stores
      bool valid = v < args.M_total;
      int n = 0, y = 0, x = 0;
      if (valid) {
        n = v / args.rows_per_img;
        const int rr = v - n * args.rows_per_img;
        y = rr / args.in_Wp;
        x = rr - y * args.in_Wp;
        valid = (y < args.Ho) && (x < args.Wo);
      }
      const size_t o_row = (((size_t)n * args.out_Hp + (y + args.out_pad)) * args.out_Wp + (x + args.out_pad)) * args.out_Cs + n0;
      const bool bwd = args.mask_hi || args.accumulate;
#pragma unroll
      for (int jp = 0; jp < BN / 8; jp += 2) {
        float vr[8];
        quad_gather8(acc, jp, q, vr);
        const int c0 = 8 * (jp + (q & 1));
        if (valid && c0 < ncols) {
          float sb[8], ss[8], sh[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const int col = n0 + c0 + e;
            const bool in = col < args.cout;
            sb[e] = (args.bias && in) ? __ldg(args.bias + col) : 0.f;
            ss[e] = (args.bn_scale && in) ? __ldg(args.bn_scale + col) : 0.f;
            sh[e] = (args.bn_scale && in) ? __ldg(args.bn_shift + col) : 0.f;
          }
          if (bwd) epi_split8<true>(args, vr, o_row + c0, sb, ss, sh);
          else epi_split8<false>(args, vr, o_row + c0, sb, ss, sh);
        }
      }
      continue;
    }

    // ===================== staged epilogues: registers -> shared-memory tile -> one thread per row (and half of the columns) ==
    consumer_sync();                                                       // both warpgroups are done with the ring
    store_acc_tile<BN>(acc, s_acc, cw, cwarp, lane);
    consumer_sync();
    const int r = ctid & (kBM - 1), half = ctid >> 7;
    const int v = m0 + r;                                                  // virtual row of this thread
    bool valid = v < args.M_total;
    int n = 0, y = 0, x = 0;
    if (valid) {
      n = v / args.rows_per_img;
      const int rr = v - n * args.rows_per_img;
      y = rr / args.in_Wp;
      x = rr - y * args.in_Wp;
      valid = (y < args.Ho) && (x < args.Wo);
    }
    const float* arow = s_acc + (size_t)r * (BN + kAccPad);
    const int h0 = half * (BN / 2), nh = min(BN / 2, ncols - h0);       // this thread's columns: [h0, h0 + nh)
    if (valid && args.epi == EPI_HEAD) {
      if (half == 0) {
        const int C = args.head_C, CP4 = C + 4, RW = C + 12;
        const int pix = y * args.Wo + x;
        if (CP4 == 25 && args.head_nb <= 8) {
          epi_head_fixed<25>(args, arow, n, pix, s_bias);
        } else {
          for (int bx = 0; bx < args.head_nb; ++bx) {
            const int c_lo = bx * CP4;
            float mx = -INFINITY;
            for (int c = c_lo; c < c_lo + C; ++c) mx = fmaxf(mx, arow[c] + s_bias[c]);
            float sum = 0.f;
            for (int c = c_lo; c < c_lo + C; ++c) sum += expf(arow[c] + s_bias[c] - mx);
            const int prior = args.head_prior_off + pix * args.head_nb + bx;
            float* dst = args.out_f32 + ((size_t)n * args.head_P + prior) * RW;
            for (int rc = 0; rc < CP4; ++rc) {
              const float val = arow[c_lo + rc] + s_bias[c_lo + rc];
              dst[rc] = rc < C ? expf(val - mx) / sum : val;
            }
            const float4 an = __ldg(reinterpret_cast<const float4*>(args.head_anchors) + prior);
            dst[C + 4] = an.x; dst[C + 5] = an.y; dst[C + 6] = an.z; dst[C + 7] = an.w;
            dst[C + 8] = args.head_var[0]; dst[C + 9] = args.head_var[1]; dst[C + 10] = args.head_var[2]; dst[C + 11] = args.head_var[3];
          }
        }
      }
    } else if (valid && nh > 0) {
      if (args.epi == EPI_ATOMIC) {
        float* dstp = args.out_f32 + (size_t)v * args.out_ld + args.out_col_off + n0 + h0;
        for (int j = 0; j < nh; ++j) atomicAdd(dstp + j, arow[h0 + j]);
      } else {
        const size_t o = (((size_t)n * args.Ho + y) * args.Wo + x) * (size_t)args.cout + n0 + h0;
        for (int j = 0; j < nh; ++j) args.out_f32[o + j] = apply_act(arow[h0 + j] + s_bias[h0 + j], args.act);
      }
    }
    fence_proxy_async();                                                   // the next tile's TMA writes over s_acc
    consumer_sync();
    if (ctid == 0) mbar_arrive(staged_free);
  }
}

template <int BN, int MODE>
static int launch_conv_bn(const ConvLaunch& L, int grid, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    SSDK_CHECK_CUDA(cudaFuncSetAttribute(conv_wgmma_kernel<BN, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  conv_wgmma_kernel<BN, MODE><<<grid, kConvThreads, L.smem, stream>>>(L.a_hi, L.a_lo, L.b_hi, L.b_lo, L.args);
  return SSDK_OK;
}

int launch_conv(ssdk_ctx* ctx, const ConvLaunch& L, cudaStream_t stream, int grid_cap) {
  // the kernel is persistent with a static stride over its work units: any grid size computes the same result
  const int grid = grid_cap > 0 ? std::max(1, std::min(L.grid, grid_cap)) : L.grid;
  const bool split = L.args.split != 0;
  SSDK_REQUIRE(!split || L.args.acc_split, "internal: bf16x3 conv plans carry the cross-term accumulator");
  SSDK_REQUIRE(split || L.args.BN != 160, "internal: 160-wide conv tiles are for bf16x3 predictor heads");
  int rc;
  switch (L.args.BN) {
    case 64: rc = split ? launch_conv_bn<64, kSplitXS>(L, grid, stream) : launch_conv_bn<64, kSingle>(L, grid, stream); break;
    case 128: rc = split ? launch_conv_bn<128, kSplitXS>(L, grid, stream) : launch_conv_bn<128, kSingle>(L, grid, stream); break;
    case 160: rc = launch_conv_bn<160, kSplitXS>(L, grid, stream); break;
    case 256:
      SSDK_REQUIRE(!split, "internal: 256-wide conv tiles have no cross-term accumulator");
      rc = launch_conv_bn<256, kSingle>(L, grid, stream);
      break;
    default: set_error("internal: conv tile width %d", L.args.BN); return SSDK_ERR_INVALID;
  }
  if (rc) return rc;
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

// (x - mean) / std, channel swap (models/keras_ssd300.py:247-272) -> split bf16 planes
__global__ void preprocess_kernel(const float* __restrict__ img, int B, int H, int W, int Cimg, float3 mean, float3 inv_std,
                                  int has_std, int3 swap, ActBuf out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)B * H * W;
  if (i >= total) return;
  const int x = (int)(i % W); const int y = (int)((i / W) % H); const int n = (int)(i / ((size_t)W * H));
  const float* p = img + i * Cimg;
  float v[3];
  const float m[3] = {mean.x, mean.y, mean.z};
  const float s[3] = {inv_std.x, inv_std.y, inv_std.z};
  for (int c = 0; c < Cimg && c < 3; ++c) {
    float t = p[c] - m[c];
    if (has_std) t = t / s[c];          // inv_std holds the divisor itself when has_std
    v[c] = t;
  }
  const int sw[3] = {swap.x, swap.y, swap.z};
  const size_t o = act_index(out, n, y, x);
  if (out.Cs == 8 && Cimg == 3) {               // one 16-byte word per plane and pixel (channels 3..7 are zero)
    const float w[8] = {v[sw[0]], v[sw[1]], v[sw[2]], 0.f, 0.f, 0.f, 0.f, 0.f};
    split_store8(out.hi, out.lo, o, w);
    return;
  }
  for (int c = 0; c < Cimg && c < 3; ++c) split_store(out.hi, out.lo, o + c, v[sw[c]]);
}

int launch_preprocess(ssdk_ctx* ctx, const float* images, int B, int H, int W, int Cimg, const float* mean, const float* stddev,
                      const int* swap, const ActBuf& out, cudaStream_t stream) {
  SSDK_REQUIRE(Cimg == 3, "only 3-channel images are supported (got %d)", Cimg);
  float3 m = mean ? make_float3(mean[0], mean[1], mean[2]) : make_float3(0, 0, 0);
  float3 s = stddev ? make_float3(stddev[0], stddev[1], stddev[2]) : make_float3(1, 1, 1);
  int3 sw = swap ? make_int3(swap[0], swap[1], swap[2]) : make_int3(0, 1, 2);
  const size_t total = (size_t)B * H * W;
  preprocess_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(images, B, H, W, Cimg, m, s, stddev ? 1 : 0, sw, out);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

// Explicit im2col for the few layers the descriptor trick does not cover (3-channel input, strided convs):
// out[row = (n, yo, xo)][k = (kh*KW + kw)*Cin + c], zero padded to Kpad columns.
__global__ void im2col_kernel(ActBuf in, __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo, int Ho, int Wo,
                              int KH, int KW, int stride, int dil, int pad_t, int pad_l, int Kpad) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)in.B * Ho * Wo * Kpad;
  if (i >= total) return;
  const int k = (int)(i % Kpad);
  const size_t row = i / Kpad;
  const int xo = (int)(row % Wo); const int yo = (int)((row / Wo) % Ho); const int n = (int)(row / ((size_t)Wo * Ho));
  __nv_bfloat16 h = __float2bfloat16_rn(0.f), l = h;
  if (k < KH * KW * in.C) {
    const int c = k % in.C; const int tap = k / in.C; const int kw = tap % KW; const int kh = tap / KW;
    const int y = yo * stride + kh * dil - pad_t, x = xo * stride + kw * dil - pad_l;
    if (y >= 0 && y < in.H && x >= 0 && x < in.W) {
      const size_t s = act_index(in, n, y, x) + c;
      h = in.hi[s];
      if (in.lo) l = in.lo[s];
    }
  }
  out_hi[i] = h;
  if (out_lo) out_lo[i] = l;
}

// The same with eight channels (one 16-byte word of a plane) per thread: whenever the input has a multiple of 8 channels, eight
// consecutive K indices are eight consecutive channels of one tap.
__global__ void im2col8_kernel(ActBuf in, __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo, int Ho, int Wo,
                               int KH, int KW, int stride, int dil, int pad_t, int pad_l, int Kpad) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int K8 = Kpad / 8;
  const size_t total = (size_t)in.B * Ho * Wo * K8;
  if (i >= total) return;
  const int k = (int)(i % K8) * 8;
  const size_t row = i / K8;
  const int xo = (int)(row % Wo); const int yo = (int)((row / Wo) % Ho); const int n = (int)(row / ((size_t)Wo * Ho));
  uint4 h = make_uint4(0, 0, 0, 0), l = h;
  if (k < KH * KW * in.C) {
    const int c = k % in.C; const int tap = k / in.C; const int kw = tap % KW; const int kh = tap / KW;
    const int y = yo * stride + kh * dil - pad_t, x = xo * stride + kw * dil - pad_l;
    if (y >= 0 && y < in.H && x >= 0 && x < in.W) {
      const size_t s = act_index(in, n, y, x) + c;
      h = *reinterpret_cast<const uint4*>(in.hi + s);
      if (in.lo) l = *reinterpret_cast<const uint4*>(in.lo + s);
    }
  }
  *reinterpret_cast<uint4*>(out_hi + row * Kpad + k) = h;
  if (out_lo) *reinterpret_cast<uint4*>(out_lo + row * Kpad + k) = l;
}

bool im2col_vec8_ok(const ActBuf& in, int Kpad, const void* out_hi, const void* out_lo) {
  return in.C % 8 == 0 && in.Cs == in.C && Kpad % 8 == 0 && (reinterpret_cast<uintptr_t>(out_hi) & 15) == 0 &&
         (!out_lo || (reinterpret_cast<uintptr_t>(out_lo) & 15) == 0);
}

int launch_im2col(ssdk_ctx* ctx, const ActBuf& in, __nv_bfloat16* out_hi, __nv_bfloat16* out_lo, int Ho, int Wo, int kh, int kw,
                  int stride, int dil, int pad_t, int pad_l, int Kpad, bool vec8, cudaStream_t stream) {
  if (vec8) {
    const size_t total8 = (size_t)in.B * Ho * Wo * (Kpad / 8);
    im2col8_kernel<<<(unsigned)((total8 + 255) / 256), 256, 0, stream>>>(in, out_hi, out_lo, Ho, Wo, kh, kw, stride, dil, pad_t, pad_l, Kpad);
    SSDK_COUNT_LAUNCH(ctx);
    SSDK_CHECK_CUDA(cudaGetLastError());
    return SSDK_OK;
  }
  const size_t total = (size_t)in.B * Ho * Wo * Kpad;
  im2col_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(in, out_hi, out_lo, Ho, Wo, kh, kw, stride, dil, pad_t, pad_l, Kpad);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

// Direct fp32 convolution for the image-facing layer (Cin < 8, e.g. conv1_1 3x3x3 or SSD7's conv1 5x5x3): K = kh*kw*cin is
// far too thin for a tensor-core tile, so each thread computes FOUR horizontally adjacent output pixels x 16 output channels
// with plain FMAs (one shared-memory weight fetch feeds 4 pixels); bias / BN / activation / hi-lo split are fused.
// HWIO weights are used as they are ([K][Cout]).
constexpr int kDirectPx = 4;
template <int CIN, int KHW>     // CIN > 0 / KHW > 0: compile-time input channels / square kernel size (full unrolling); 0: run-time
__global__ void __launch_bounds__(256) conv_direct_kernel(ActBuf in, ActBuf out, const float* __restrict__ w, const float* __restrict__ bias,
                                                          const float* __restrict__ bn_scale, const float* __restrict__ bn_shift, int act,
                                                          int KH_, int KW_, int dil, int pad_t, int pad_l) {
  extern __shared__ float s_w[];                 // [K][Cout]
  const int KH = KHW > 0 ? KHW : KH_, KW = KHW > 0 ? KHW : KW_, Cin = CIN > 0 ? CIN : in.C;
  const int K = KH * KW * Cin, Cout = out.C;
  for (int i = threadIdx.x; i < K * Cout; i += blockDim.x) s_w[i] = w[i];
  __syncthreads();
  const int groups = Cout / 16;
  const int wq = (out.W + kDirectPx - 1) / kDirectPx;
  const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)out.B * out.H * wq * groups;
  if (gid >= total) return;
  const int g = (int)(gid % groups);
  const size_t q = gid / groups;
  const int xo0 = (int)(q % wq) * kDirectPx; const int yo = (int)((q / wq) % out.H); const int n = (int)(q / ((size_t)wq * out.H));
  float acc[kDirectPx][16];
#pragma unroll
  for (int p = 0; p < kDirectPx; ++p)
#pragma unroll
    for (int e = 0; e < 16; ++e) acc[p][e] = 0.f;
#pragma unroll
  for (int kh = 0; kh < KH; ++kh) {
    const int y = yo + kh * dil - pad_t;
    if (y < 0 || y >= in.H) continue;
#pragma unroll
    for (int kw = 0; kw < KW; ++kw) {
      float v[kDirectPx][4];
#pragma unroll
      for (int p = 0; p < kDirectPx; ++p) {
        const int x = xo0 + p + kw * dil - pad_l;
        uint2 h2 = make_uint2(0, 0), l2 = make_uint2(0, 0);
        if (x >= 0 && x < in.W) {
          const size_t s = act_index(in, n, y, x);
          h2 = *reinterpret_cast<const uint2*>(in.hi + s);                    // channels 0..3 (Cin <= 4 used)
          if (in.lo) l2 = *reinterpret_cast<const uint2*>(in.lo + s);
        }
        v[p][0] = __uint_as_float(h2.x << 16) + __uint_as_float(l2.x << 16);
        v[p][1] = __uint_as_float(h2.x & 0xffff0000u) + __uint_as_float(l2.x & 0xffff0000u);
        v[p][2] = __uint_as_float(h2.y << 16) + __uint_as_float(l2.y << 16);
        v[p][3] = __uint_as_float(h2.y & 0xffff0000u) + __uint_as_float(l2.y & 0xffff0000u);
      }
#pragma unroll
      for (int c = 0; c < Cin; ++c) {
        const float4* wr = reinterpret_cast<const float4*>(s_w + (size_t)((kh * KW + kw) * Cin + c) * Cout + g * 16);
        const float4 w0 = wr[0], w1 = wr[1], w2 = wr[2], w3 = wr[3];
        const float wv[16] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w, w2.x, w2.y, w2.z, w2.w, w3.x, w3.y, w3.z, w3.w};
#pragma unroll
        for (int p = 0; p < kDirectPx; ++p) {
          const float vv = c == 0 ? v[p][0] : (c == 1 ? v[p][1] : (c == 2 ? v[p][2] : v[p][3]));
#pragma unroll
          for (int e = 0; e < 16; ++e) acc[p][e] = fmaf(vv, wv[e], acc[p][e]);
        }
      }
    }
  }
#pragma unroll
  for (int p = 0; p < kDirectPx; ++p) {
    const int xo = xo0 + p;
    if (xo >= out.W) break;
    const size_t o = act_index(out, n, yo, xo) + (size_t)g * 16;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int col = g * 16 + h * 8 + e;
        float xv = acc[p][h * 8 + e] + __ldg(bias + col);
        if (bn_scale) xv = xv * __ldg(bn_scale + col) + __ldg(bn_shift + col);
        f[e] = apply_act(xv, act);
      }
      split_store8(out.hi, out.lo, o + h * 8, f);
    }
  }
}

int launch_conv_direct(ssdk_ctx* ctx, const ActBuf& in, const ActBuf& out, const float* w, const float* bias, const float* bn_scale,
                       const float* bn_shift, int act, int kh, int kw, int dil, int pad_t, int pad_l, cudaStream_t stream) {
  const size_t smem = (size_t)kh * kw * in.C * out.C * sizeof(float);
  static bool attr_set = false;
  if (!attr_set) {
    SSDK_CHECK_CUDA(cudaFuncSetAttribute(conv_direct_kernel<0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    attr_set = true;
  }
  const size_t total = (size_t)out.B * out.H * ((out.W + kDirectPx - 1) / kDirectPx) * (out.C / 16);
  const unsigned blocks = (unsigned)((total + 255) / 256);
  conv_direct_kernel<0, 0><<<blocks, 256, smem, stream>>>(in, out, w, bias, bn_scale, bn_shift, act, kh, kw, dil, pad_t, pad_l);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

// ------------------------------------------------------------------------------------------------
// conv_first_kernel: the image-facing layer (Cin <= 4: conv1_1 3x3x3 of models/keras_ssd300.py:263, conv1 5x5x3 of
// models/keras_ssd7.py:277) on the tensor cores.  K = taps * 4 (channels padded to 4) is far too thin for the TMA ring of
// conv_wgmma_kernel -- an explicit im2col would write and re-read ten times the layer's input -- so the A tile is GATHERED.
// Per 128-pixel tile: 256 threads gather (thread = one output pixel and one plane: the taps' 8-byte (4-channel) hi or lo words
// from the zero-bordered input planes, L1/L2 hits since every word is used by taps of neighbouring pixels) into the K-major
// 128B-swizzled A tile; two warpgroups issue wgmma on 64 rows each; the accumulators go through shared memory to the epilogue
// of the other activation-producing launches.  The weights (K-major, swizzled image prepared on the host) stay in shared memory
// for the whole launch.  The layer is bound by writing its output (B*H*W*Cout*4 bytes of hi+lo planes).
// ------------------------------------------------------------------------------------------------
struct FirstArgs {
  ActBuf in;
  const __nv_bfloat16* w_hi; const __nv_bfloat16* w_lo;   // [kblocks][BN][64] swizzled images
  int KH, KW, dil, pad_t, pad_l;
  int tap_off[32];            // element offset of tap t's 4-channel word relative to the output pixel's own word in the input planes
                              // (the planes' zero border covers every tap: checked on the host)
  int kblocks;                // 64-wide blocks that cover taps * 4 (1 or 2; a template parameter of the kernel, as is split)
  int split;
  long long M;                // B * Ho * Wo output pixels
  int n_tiles, Ho, Wo;
  ConvArgs epi;               // bias / bn / act / output planes as the shared epilogue expects them
};

int first_bn(int cout) { return cout <= 64 ? 64 : 128; }
FirstPlan first_plan(const ActBuf& out, int kh, int kw, int sm_count) {
  FirstPlan fp;
  fp.BN = first_bn(out.C);
  fp.kblocks = (kh * kw * 4 + 63) / 64;
  fp.n_tiles = (int)(((long long)out.B * out.H * out.W + kBM - 1) / kBM);
  fp.grid = std::min(fp.n_tiles, sm_count);
  return fp;
}
static size_t first_smem_bytes(int kblocks, int BN, int split) {
  return 1024 + ((size_t)kblocks * kATile + (size_t)kblocks * BN * 128) * (split ? 2 : 1) + acc_tile_bytes(BN) + (size_t)3 * BN * sizeof(float);
}

template <int BN, int KB, bool SPLIT>
__global__ void __launch_bounds__(256, 1) conv_first_kernel(const __grid_constant__ FirstArgs fa) {
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  unsigned char* smem_al = smem_dyn + (smem_base - smem_u32(smem_dyn));
  const int tid = threadIdx.x, wg = tid >> 7, warp = tid >> 5, lane = tid & 31;
  constexpr bool split = SPLIT;
  const uint32_t a_plane = (uint32_t)KB * kATile;                      // A tile: hi plane | lo plane
  const uint32_t b_block = (uint32_t)BN * 128u;                        // one k-block of the weight tile
  const uint32_t b_plane = b_block * KB;
  const uint32_t a_base = smem_base, b_base = a_base + a_plane * (split ? 2 : 1);
  float* s_acc = reinterpret_cast<float*>(smem_al + (b_base + b_plane * (split ? 2 : 1) - smem_base));
  float* s_bias = s_acc + (size_t)kBM * (BN + kAccPad) + 32;
  float* s_scale = s_bias + BN;
  float* s_shift = s_scale + BN;
  for (int i = tid; i < BN; i += blockDim.x) {
    const bool in = i < fa.epi.cout;
    s_bias[i] = (in && fa.epi.bias) ? fa.epi.bias[i] : 0.f;
    if (fa.epi.bn_scale) { s_scale[i] = in ? fa.epi.bn_scale[i] : 0.f; s_shift[i] = in ? fa.epi.bn_shift[i] : 0.f; }
  }
  {   // resident weights: straight copy of the swizzled images
    const uint4* src_h = reinterpret_cast<const uint4*>(fa.w_hi);
    const uint4* src_l = reinterpret_cast<const uint4*>(fa.w_lo);
    uint4* dst = reinterpret_cast<uint4*>(smem_al + (b_base - smem_base));
    const int n16 = (int)(b_plane >> 4);
    for (int i = tid; i < n16; i += blockDim.x) { dst[i] = src_h[i]; if (split) dst[n16 + i] = src_l[i]; }
  }
  const int taps = fa.KH * fa.KW;
  constexpr int slots = KB * 16;                                       // 8-byte (4-channel) K slots; slots >= taps hold zeros
  const int r = tid & (kBM - 1), plane = tid >> 7;                     // gather / epilogue row; gather plane (0 hi, 1 lo)
  const __nv_bfloat16* src_plane = plane ? fa.in.lo : fa.in.hi;
  unsigned char* a_dst = smem_al + (a_base - smem_base) + plane * a_plane;
  float acc[BN / 2];
  for (int t = blockIdx.x; t < fa.n_tiles; t += gridDim.x) {
    // ===================== gather =====================
    const long long v = (long long)t * kBM + r;
    const bool valid = v < fa.M;
    int n = 0, y = 0, x = 0;
    if (valid) {
      n = (int)(v / ((long long)fa.Ho * fa.Wo));
      const int rem = (int)(v - (long long)n * fa.Ho * fa.Wo);
      y = rem / fa.Wo; x = rem - y * fa.Wo;
    }
    if (plane == 0 || split) {
      const size_t src0 = valid ? act_index(fa.in, n, y, x) : 0;
      // all loads of a round are issued before the first store (twelve taps = the whole 3x3 kernel in one round trip)
      constexpr int kRound = 12;
      uint2 w[kRound];
      for (int s0 = 0; s0 < slots; s0 += kRound) {
#pragma unroll
        for (int j = 0; j < kRound; ++j) {
          const int tap = s0 + j;
          w[j] = make_uint2(0, 0);
          if (valid && tap < taps) w[j] = __ldg(reinterpret_cast<const uint2*>(src_plane + (long long)src0 + fa.tap_off[tap]));
        }
#pragma unroll
        for (int j = 0; j < kRound; ++j) {
          const int tap = s0 + j;
          if (tap < slots) {
            const uint32_t off = (uint32_t)(tap >> 4) * kATile + (uint32_t)r * 128u + ((uint32_t)(((tap >> 1) & 7) ^ (r & 7)) << 4) + (uint32_t)(tap & 1) * 8u;
            *reinterpret_cast<uint2*>(a_dst + off) = w[j];
          }
        }
      }
    }
    fence_proxy_async();                                               // generic-proxy stores -> visible to wgmma (async proxy)
    __syncthreads();
    // ===================== MMA: warpgroup wg computes rows [64 wg, +64) =====================
    {
      constexpr uint64_t kDesc = wgmma_desc_hi(16);
      wgmma_fence_acc(acc);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < KB * 4; ++ks) {                             // every k-step of the k-blocks: uniform issue
        const int kb = ks >> 2, k = ks & 3;
        const uint32_t ah = a_base + (uint32_t)kb * kATile + (uint32_t)wg * (kATile / 2) + 32u * k;
        const uint32_t bh = b_base + (uint32_t)kb * b_block + 32u * k;
        const uint64_t da = wgmma_desc(kDesc, ah), db = wgmma_desc(kDesc, bh);
        Wgmma<BN, 0, 0>::mma(acc, da, db, ks ? 1u : 0u);
        if constexpr (split) {
          Wgmma<BN, 0, 0>::mma(acc, da, wgmma_desc(kDesc, bh + b_plane), 1u);
          Wgmma<BN, 0, 0>::mma(acc, wgmma_desc(kDesc, ah + a_plane), db, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
    }
    store_acc_tile<BN>(acc, s_acc, wg, warp, lane);
    __syncthreads();
    // ===================== epilogue: thread = (row, half of the columns) =====================
    const int h0 = plane * (BN / 2), nh = min(BN / 2, fa.epi.cout - h0);
    if (valid && nh > 0) {
      const size_t o = (((size_t)n * fa.epi.out_Hp + (y + fa.epi.out_pad)) * fa.epi.out_Wp + (x + fa.epi.out_pad)) * fa.epi.out_Cs + h0;
      const float* arow = s_acc + (size_t)r * (BN + kAccPad) + h0;
#pragma unroll 4
      for (int c0 = 0; c0 < nh; c0 += 8) {
        float v[8], sb[8], ss[8], sh[8];
        ld_f8(arow + c0, v);
        ld_f8(s_bias + h0 + c0, sb);
        if (fa.epi.bn_scale) { ld_f8(s_scale + h0 + c0, ss); ld_f8(s_shift + h0 + c0, sh); }
        epi_split8<false>(fa.epi, v, o + c0, sb, ss, sh);
      }
    }
    __syncthreads();                                                   // the A tile and s_acc are rewritten by the next tile
  }
}

// K-major, 128B-swizzled shared-memory image of the image-facing layer's weights: row = output channel (padded to BN), element
// k = tap * 4 + c.  HWIO kernel in.
void first_weight_image(const float* hwio, int taps, int cin, int cout, int BN, int kblocks, std::vector<uint16_t>& hi, std::vector<uint16_t>& lo) {
  hi.assign((size_t)kblocks * BN * 64, 0); lo.assign((size_t)kblocks * BN * 64, 0);
  for (int o = 0; o < cout; ++o)
    for (int t = 0; t < taps; ++t)
      for (int c = 0; c < cin; ++c) {
        const int k = t * 4 + c, kb = k >> 6, kk = k & 63;
        const size_t byte = (size_t)kb * BN * 128 + (size_t)o * 128 + ((size_t)((kk >> 3) ^ (o & 7)) << 4) + (size_t)(kk & 7) * 2;
        const float w = hwio[((size_t)t * cin + c) * cout + o];
        const uint16_t h = f2bf(w);
        hi[byte / 2] = h; lo[byte / 2] = f2bf(w - bf2f(h));
      }
}

bool first_border_ok(const ActBuf& in, int kh, int kw, int dil, int pad_t, int pad_l) {
  return in.pad >= pad_t && in.pad >= pad_l && in.pad >= (kh - 1) * dil - pad_t && in.pad >= (kw - 1) * dil - pad_l;
}
int first_tc_supported(int taps, int cin, int cout) { return cin <= 4 && taps * 4 <= 128 && cout % 8 == 0 && cout <= 128; }

template <int BN, int KB, bool SPLIT>
static int launch_first_bn(const FirstArgs& fa, int grid, size_t smem, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    SSDK_CHECK_CUDA(cudaFuncSetAttribute(conv_first_kernel<BN, KB, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  conv_first_kernel<BN, KB, SPLIT><<<grid, 256, smem, stream>>>(fa);
  return SSDK_OK;
}
template <int BN>
static int launch_first_kb(const FirstArgs& fa, int grid, size_t smem, cudaStream_t stream) {
  if (fa.kblocks == 1) return fa.split ? launch_first_bn<BN, 1, true>(fa, grid, smem, stream) : launch_first_bn<BN, 1, false>(fa, grid, smem, stream);
  return fa.split ? launch_first_bn<BN, 2, true>(fa, grid, smem, stream) : launch_first_bn<BN, 2, false>(fa, grid, smem, stream);
}

int launch_conv_first(ssdk_ctx* ctx, const FirstPlan& fp, const ActBuf& in, const ActBuf& out, const __nv_bfloat16* w_hi, const __nv_bfloat16* w_lo,
                      const float* bias, const float* bn_scale, const float* bn_shift, int act, int kh, int kw, int dil, int pad_t,
                      int pad_l, cudaStream_t stream) {
  FirstArgs fa;
  memset(&fa, 0, sizeof(fa));
  fa.in = in; fa.w_hi = w_hi; fa.w_lo = w_lo;
  fa.KH = kh; fa.KW = kw; fa.dil = dil; fa.pad_t = pad_t; fa.pad_l = pad_l;
  SSDK_REQUIRE(first_border_ok(in, kh, kw, dil, pad_t, pad_l), "image-facing convolution: the input planes' zero border is too small");
  for (int t = 0; t < kh * kw; ++t) {
    const int dy = (t / kw) * dil - pad_t, dx = (t % kw) * dil - pad_l;
    fa.tap_off[t] = (dy * in.Wp() + dx) * in.Cs;
  }
  fa.kblocks = fp.kblocks;
  SSDK_REQUIRE(fa.kblocks <= 2, "image-facing convolution: more than 128 K columns");
  const int BN = fp.BN;
  fa.split = (in.lo && w_lo) ? 1 : 0;
  fa.M = (long long)out.B * out.H * out.W; fa.Ho = out.H; fa.Wo = out.W;
  fa.n_tiles = fp.n_tiles;
  fa.epi.cout = out.C; fa.epi.bias = bias; fa.epi.bn_scale = bn_scale; fa.epi.bn_shift = bn_shift; fa.epi.act = act;
  fa.epi.out_hi = out.hi; fa.epi.out_lo = out.lo; fa.epi.out_Hp = out.Hp(); fa.epi.out_Wp = out.Wp(); fa.epi.out_pad = out.pad; fa.epi.out_Cs = out.Cs;
  const size_t smem = first_smem_bytes(fa.kblocks, BN, fa.split);
  SSDK_REQUIRE(smem <= 227 * 1024, "image-facing convolution: %zu bytes of shared memory", smem);
  const int grid = fp.grid;
  const int rc = BN == 64 ? launch_first_kb<64>(fa, grid, smem, stream) : launch_first_kb<128>(fa, grid, smem, stream);
  if (rc) return rc;
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

// Max pooling; out-of-range window positions are ignored (TF 'same' pooling pads with -inf).
// One thread per (pixel, group of 8 channels); the max is taken on the reconstructed value hi + lo.
__global__ void maxpool_kernel(ActBuf in, ActBuf out, int KH, int KW, int stride, int pad_t, int pad_l) {
  const int groups = in.Cs / 8;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)out.B * out.H * out.W * groups;
  if (i >= total) return;
  const int g = (int)(i % groups);
  const size_t pix = i / groups;
  const int xo = (int)(pix % out.W); const int yo = (int)((pix / out.W) % out.H); const int n = (int)(pix / ((size_t)out.W * out.H));
  float best[8];
  uint32_t bh[8], bl[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; bh[e] = 0; bl[e] = 0; }
  for (int ky = 0; ky < KH; ++ky) {
    const int y = yo * stride + ky - pad_t;
    if (y < 0 || y >= in.H) continue;
    for (int kx = 0; kx < KW; ++kx) {
      const int x = xo * stride + kx - pad_l;
      if (x < 0 || x >= in.W) continue;
      const size_t s = act_index(in, n, y, x) + (size_t)g * 8;
      const uint4 h4 = *reinterpret_cast<const uint4*>(in.hi + s);
      uint4 l4 = make_uint4(0, 0, 0, 0);
      if (in.lo) l4 = *reinterpret_cast<const uint4*>(in.lo + s);
      const uint32_t hw[4] = {h4.x, h4.y, h4.z, h4.w}, lw[4] = {l4.x, l4.y, l4.z, l4.w};
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const uint32_t hb = (hw[e >> 1] >> ((e & 1) * 16)) & 0xffffu, lb = (lw[e >> 1] >> ((e & 1) * 16)) & 0xffffu;
        const float v = __uint_as_float(hb << 16) + __uint_as_float(lb << 16);
        if (v > best[e]) { best[e] = v; bh[e] = hb; bl[e] = lb; }
      }
    }
  }
  const size_t o = act_index(out, n, yo, xo) + (size_t)g * 8;
  uint4 oh, ol;
  oh.x = bh[0] | (bh[1] << 16); oh.y = bh[2] | (bh[3] << 16); oh.z = bh[4] | (bh[5] << 16); oh.w = bh[6] | (bh[7] << 16);
  ol.x = bl[0] | (bl[1] << 16); ol.y = bl[2] | (bl[3] << 16); ol.z = bl[4] | (bl[5] << 16); ol.w = bl[6] | (bl[7] << 16);
  *reinterpret_cast<uint4*>(out.hi + o) = oh;
  if (out.lo) *reinterpret_cast<uint4*>(out.lo + o) = ol;
}

// 2x2 / stride 2 without top-left padding (every pool of the VGG trunk but pool5): the four taps are loaded up front (eight
// independent 16-byte loads per thread); a tap that falls off the bottom / right edge ('same' pooling of an odd extent) is
// clamped onto its in-range neighbour, which cannot change a first-maximum scan.
__global__ void __launch_bounds__(256) maxpool2x2_kernel(ActBuf in, ActBuf out) {
  const int groups = in.Cs / 8;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)out.B * out.H * out.W * groups;
  if (i >= total) return;
  const int g = (int)(i % groups);
  const size_t pix = i / groups;
  const int xo = (int)(pix % out.W); const int yo = (int)((pix / out.W) % out.H); const int n = (int)(pix / ((size_t)out.W * out.H));
  const int y0 = 2 * yo, x0 = 2 * xo, y1 = min(y0 + 1, in.H - 1), x1 = min(x0 + 1, in.W - 1);
  const size_t s00 = act_index(in, n, y0, x0) + (size_t)g * 8, s01 = act_index(in, n, y0, x1) + (size_t)g * 8;
  const size_t s10 = act_index(in, n, y1, x0) + (size_t)g * 8, s11 = act_index(in, n, y1, x1) + (size_t)g * 8;
  uint4 h[4], l[4];
  h[0] = __ldcs(reinterpret_cast<const uint4*>(in.hi + s00)); h[1] = __ldcs(reinterpret_cast<const uint4*>(in.hi + s01));
  h[2] = __ldcs(reinterpret_cast<const uint4*>(in.hi + s10)); h[3] = __ldcs(reinterpret_cast<const uint4*>(in.hi + s11));
  if (in.lo) {
    l[0] = __ldcs(reinterpret_cast<const uint4*>(in.lo + s00)); l[1] = __ldcs(reinterpret_cast<const uint4*>(in.lo + s01));
    l[2] = __ldcs(reinterpret_cast<const uint4*>(in.lo + s10)); l[3] = __ldcs(reinterpret_cast<const uint4*>(in.lo + s11));
  } else {
    l[0] = l[1] = l[2] = l[3] = make_uint4(0, 0, 0, 0);
  }
  float best[8];
  uint32_t bh[8], bl[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; bh[e] = 0; bl[e] = 0; }
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const uint32_t hw[4] = {h[t].x, h[t].y, h[t].z, h[t].w}, lw[4] = {l[t].x, l[t].y, l[t].z, l[t].w};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const uint32_t hb = (hw[e >> 1] >> ((e & 1) * 16)) & 0xffffu, lb = (lw[e >> 1] >> ((e & 1) * 16)) & 0xffffu;
      const float v = __uint_as_float(hb << 16) + __uint_as_float(lb << 16);
      if (v > best[e]) { best[e] = v; bh[e] = hb; bl[e] = lb; }
    }
  }
  const size_t o = act_index(out, n, yo, xo) + (size_t)g * 8;
  uint4 oh, ol;
  oh.x = bh[0] | (bh[1] << 16); oh.y = bh[2] | (bh[3] << 16); oh.z = bh[4] | (bh[5] << 16); oh.w = bh[6] | (bh[7] << 16);
  ol.x = bl[0] | (bl[1] << 16); ol.y = bl[2] | (bl[3] << 16); ol.z = bl[4] | (bl[5] << 16); ol.w = bl[6] | (bl[7] << 16);
  *reinterpret_cast<uint4*>(out.hi + o) = oh;
  if (out.lo) *reinterpret_cast<uint4*>(out.lo + o) = ol;
}

int launch_maxpool(ssdk_ctx* ctx, const ActBuf& in, const ActBuf& out, int kh, int kw, int stride, int pad_t, int pad_l,
                   cudaStream_t stream) {
  const size_t total = (size_t)out.B * out.H * out.W * (in.Cs / 8);
  if (kh == 2 && kw == 2 && stride == 2 && pad_t == 0 && pad_l == 0 && 2 * (out.H - 1) < in.H && 2 * (out.W - 1) < in.W) {
    maxpool2x2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(in, out);
    SSDK_COUNT_LAUNCH(ctx);
    SSDK_CHECK_CUDA(cudaGetLastError());
    return SSDK_OK;
  }
  maxpool_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(in, out, kh, kw, stride, pad_t, pad_l);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

// L2Normalization (keras_layer_L2Normalization.py:61-63): x * rsqrt(max(sum_c x^2, 1e-12)) * gamma_c, one warp per pixel.
__global__ void l2norm_kernel(ActBuf in, ActBuf out, const float* __restrict__ gamma) {
  const size_t pix = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const size_t total = (size_t)in.B * in.H * in.W;
  if (pix >= total) return;
  const int x = (int)(pix % in.W); const int y = (int)((pix / in.W) % in.H); const int n = (int)(pix / ((size_t)in.W * in.H));
  const size_t s = act_index(in, n, y, x), o = act_index(out, n, y, x);
  float ss = 0.f;
  for (int c = lane; c < in.C; c += 32) { float v = split_load(in.hi, in.lo, s + c); ss += v * v; }
  ss = warp_sum(ss);
  const float inv = rsqrtf(fmaxf(ss, 1e-12f));
  for (int c = lane; c < in.C; c += 32) split_store(out.hi, out.lo, o + c, split_load(in.hi, in.lo, s + c) * inv * __ldg(gamma + c));
}

// The same with eight channels (16 bytes of each plane) per lane and step: up to 512 channels stay in registers between the two
// passes.  The sum of squares is formed in a different order than above (per-lane partial sums of 8, then the warp tree).
__global__ void __launch_bounds__(256) l2norm8_kernel(ActBuf in, ActBuf out, const float* __restrict__ gamma) {
  const size_t pix = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const size_t total = (size_t)in.B * in.H * in.W;
  if (pix >= total) return;
  const int x = (int)(pix % in.W); const int y = (int)((pix / in.W) % in.H); const int n = (int)(pix / ((size_t)in.W * in.H));
  const size_t s = act_index(in, n, y, x), o = act_index(out, n, y, x);
  float v[2][8];
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int c = (k * 32 + lane) * 8;
#pragma unroll
    for (int e = 0; e < 8; ++e) v[k][e] = 0.f;
    if (c < in.C) {
      split_load8(in.hi, in.lo, s + c, v[k]);
#pragma unroll
      for (int e = 0; e < 8; ++e) ss += v[k][e] * v[k][e];
    }
  }
  ss = warp_sum(ss);
  const float inv = rsqrtf(fmaxf(ss, 1e-12f));
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int c = (k * 32 + lane) * 8;
    if (c < in.C) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c + 4));
      const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = v[k][e] * inv * gm[e];
      split_store8(out.hi, out.lo, o + c, f);
    }
  }
}

int launch_l2norm(ssdk_ctx* ctx, const ActBuf& in, const ActBuf& out, const float* gamma, cudaStream_t stream) {
  const size_t total = (size_t)in.B * in.H * in.W;
  if (in.C % 8 == 0 && in.C <= 512 && in.Cs == in.C && out.Cs == out.C && (reinterpret_cast<uintptr_t>(gamma) & 15) == 0) {
    l2norm8_kernel<<<(unsigned)((total + 7) / 8), 256, 0, stream>>>(in, out, gamma);
    SSDK_COUNT_LAUNCH(ctx);
    SSDK_CHECK_CUDA(cudaGetLastError());
    return SSDK_OK;
  }
  l2norm_kernel<<<(unsigned)((total + 7) / 8), 256, 0, stream>>>(in, out, gamma);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

// Reshape / softmax / Concat (models/keras_ssd300.py:363-419): one warp per prior.
// head row layout per pixel: n_boxes x [C class logits | 4 box offsets].
__global__ void head_finalize_kernel(const float* __restrict__ head, int B, int HW, int n_boxes, int C, int P, int prior_off,
                                     const float* __restrict__ anchors, float4 var, float* __restrict__ y_pred) {
  const size_t wid = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const size_t total = (size_t)B * HW * n_boxes;
  if (wid >= total) return;
  const int b = (int)(wid % n_boxes); const size_t pix = wid / n_boxes;
  const int n = (int)(pix / HW); const int p_local = (int)(pix % HW) * n_boxes + b;
  const float* src = head + pix * (size_t)n_boxes * (C + 4) + (size_t)b * (C + 4);
  float* dst = y_pred + ((size_t)n * P + prior_off + p_local) * (C + 12);
  float mx = -INFINITY;
  for (int c = lane; c < C; c += 32) mx = fmaxf(mx, src[c]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int c = lane; c < C; c += 32) sum += expf(src[c] - mx);
  sum = warp_sum(sum);
  for (int c = lane; c < C; c += 32) dst[c] = expf(src[c] - mx) / sum;
  if (lane < 4) {
    dst[C + lane] = src[C + lane];
    dst[C + 4 + lane] = anchors[(size_t)(prior_off + p_local) * 4 + lane];
    const float v[4] = {var.x, var.y, var.z, var.w};
    dst[C + 8 + lane] = v[lane];
  }
}

int launch_head_finalize(ssdk_ctx* ctx, const float* head, int B, int HW, int n_boxes, int C, int P, int prior_off,
                         const float* anchors, const float* variances, float* y_pred, cudaStream_t stream) {
  const size_t total = (size_t)B * HW * n_boxes;
  head_finalize_kernel<<<(unsigned)((total + 7) / 8), 256, 0, stream>>>(head, B, HW, n_boxes, C, P, prior_off, anchors,
                                                                        make_float4(variances[0], variances[1], variances[2], variances[3]), y_pred);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

__global__ void l2norm_f32_kernel(const float* __restrict__ x, long long rows, int C, const float* __restrict__ gamma,
                                  float* __restrict__ out) {
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* p = x + r * C;
  float ss = 0.f;
  for (int c = lane; c < C; c += 32) { float v = p[c]; ss += v * v; }
  ss = warp_sum(ss);
  const float inv = rsqrtf(fmaxf(ss, 1e-12f));
  for (int c = lane; c < C; c += 32) out[r * C + c] = p[c] * inv * __ldg(gamma + c);
}

__global__ void unpack_kernel(ActBuf in, float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)in.B * in.H * in.W * in.C;
  if (i >= total) return;
  const int c = (int)(i % in.C); const size_t pix = i / in.C;
  const int x = (int)(pix % in.W); const int y = (int)((pix / in.W) % in.H); const int n = (int)(pix / ((size_t)in.W * in.H));
  out[i] = split_load(in.hi, in.lo, act_index(in, n, y, x) + c);
}

// float32 NHWC tensor -> split bf16 planes of an activation buffer (SSDK_OP_TENSOR); channels beyond C stay zero
__global__ void pack_kernel(const float* __restrict__ in, ActBuf out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)out.B * out.H * out.W * out.C;
  if (i >= total) return;
  const int c = (int)(i % out.C); const size_t pix = i / out.C;
  const int x = (int)(pix % out.W); const int y = (int)((pix / out.W) % out.H); const int n = (int)(pix / ((size_t)out.W * out.H));
  split_store(out.hi, out.lo, act_index(out, n, y, x) + c, in[i]);
}

int launch_pack(ssdk_ctx* ctx, const float* in, const ActBuf& out, cudaStream_t stream) {
  const size_t total = (size_t)out.B * out.H * out.W * out.C;
  pack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(in, out);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

int launch_unpack(ssdk_ctx* ctx, const ActBuf& in, float* out, cudaStream_t stream) {
  const size_t total = (size_t)in.B * in.H * in.W * in.C;
  unpack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(in, out);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

}  // namespace ssdk

extern "C" int ssdk_l2_normalize(ssdk_ctx* ctx, const float* x_dev, long long rows, int C, const float* gamma_dev, float* out_dev,
                                 void* stream) {
  using namespace ssdk;
  SSDK_REQUIRE(ctx && x_dev && gamma_dev && out_dev && rows > 0 && C > 0, "ssdk_l2_normalize: bad argument");
  l2norm_f32_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(x_dev, rows, C, gamma_dev, out_dev);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}
