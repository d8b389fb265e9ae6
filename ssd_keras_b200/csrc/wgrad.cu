// Weight gradient of a stride-1 convolution on wgmma, straight from the NHWC activation / gradient tensors (no transposes):
//   dW[co][kh][kw][ci] = sum over output pixels p of dZ[p][co] * X[p + (kh, kw)*dilation - pad][ci]
// (the cuDNN wgrad the reference gets through TensorFlow's autodiff of models/keras_ssd300.py:274-361).
//
// GEMM view: M = co (128 per tile, 64 per warpgroup), N = ci (BNc per tile), K = output pixels.  Both operands are "MN-major": a
// K row (one pixel) holds 64 contiguous channels = one 128-byte line, which is exactly how NHWC tensors lie in HBM, so a K-block
// of 64 pixels is ONE 4-D TMA box {64 channels, bw, bh, 1 image} (bw * bh = 64) per 64-channel group; the X box of tap (kh, kw)
// is the same patch shifted by (kw, kh) * dilation.  Borders are physical zeros, everything further out is TMA zero fill, and
// dZ is zero outside the valid outputs, so no masking is needed.  The pixel axis is split across CTAs (split-K); partial sums
// are reduced into the fp32 gradient buffer with vector atomics (red.global.add.v2.f32) straight from the accumulator registers.
// Work unit = (co tile, ci tile, tap, k-split); persistent CTAs; one thread issues the TMA ring, two warpgroups issue wgmma.
// Precision as in conv.cu: bf16 hi+lo operands, hi*hi + hi*lo + lo*hi into fp32 accumulators.
#include "wgrad.cuh"
#include "tc.cuh"
#include <cudaTypedefs.h>

namespace ssdk {


namespace {

constexpr int kBoxA = 64 * 128;            // one {64 channels x 64 pixels} box: 8 KB

__device__ __forceinline__ void red_add_v2(float* p, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

template <int BNc, bool SPLIT>
__global__ void __launch_bounds__(256, 1)
wgrad_wgmma_kernel(const __grid_constant__ CUtensorMap tm_g_hi, const __grid_constant__ CUtensorMap tm_g_lo,
                   const __grid_constant__ CUtensorMap tm_x_hi, const __grid_constant__ CUtensorMap tm_x_lo,
                   const __grid_constant__ WgradArgs args) {
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  const int tid = threadIdx.x, wg = tid >> 7, warp = tid >> 5, lane = tid & 31;
  constexpr bool split = SPLIT;
  const int S = args.stages, KW = args.KW;
  constexpr int nB = BNc / 64;
  const int nA = args.a_boxes;
  // stage: dZ_hi (2 boxes) | dZ_lo | X_hi (nB boxes) | X_lo
  const uint32_t a_plane = 2u * kBoxA, b_plane = (uint32_t)nB * kBoxA;
  const uint32_t b_off = a_plane * (split ? 2u : 1u);
  const uint32_t stage = (a_plane + b_plane) * (split ? 2u : 1u);
  const uint32_t bar_base = smem_base + stage * S;
  auto full = [&](uint32_t s) { return bar_base + 8u * s; };
  auto empty = [&](uint32_t s) { return bar_base + 8u * ((uint32_t)S + s); };

  if (tid == 0) {
    prefetch_tmap(&tm_g_hi); prefetch_tmap(&tm_x_hi);
    for (int s = 0; s < S; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int taps = args.KH * KW;
  const int total_units = args.co_tiles * args.ci_tiles * taps * args.k_split;
  const int patches_per_img = args.px_tiles * args.py_tiles;
  // with cout <= 64 there is one dZ box: the second warpgroup multiplies it again (a uniform wgmma path) and stores nothing
  const bool active = wg < nA;
  const uint32_t a_box = active ? (uint32_t)wg * kBoxA : 0u;
  uint32_t g = 0;
  float acc[BNc / 2];
  for (int u = blockIdx.x; u < total_units; u += gridDim.x) {
    const int ks = u % args.k_split; int r = u / args.k_split;
    const int tap = r % taps; r /= taps;
    const int kh = tap / KW, kw = tap - kh * KW;
    const int ci0 = (r % args.ci_tiles) * BNc, co0 = (r / args.ci_tiles) * 128;
    const int p0 = ks * args.patches_per_split, p1 = min(args.total_patches, p0 + args.patches_per_split);
    const int nk = p1 - p0;
    auto issue = [&](int i) {
      const uint32_t gi = g + (uint32_t)i, s = gi % (uint32_t)S;
      mbar_wait(empty(s), ((gi / (uint32_t)S) & 1u) ^ 1u);
      const int p = p0 + i;
      const int n = p / patches_per_img; const int q = p - n * patches_per_img;
      const int py = q / args.px_tiles, px = q - py * args.px_tiles;
      const int x0 = px * args.bw, y0 = py * args.bh;
      const uint32_t dst = smem_base + stage * s;
      mbar_expect_tx(full(s), args.tx_bytes);
      for (int pl = 0; pl < (split ? 2 : 1); ++pl) {
        const CUtensorMap* tg = pl ? &tm_g_lo : &tm_g_hi;
        const CUtensorMap* tx = pl ? &tm_x_lo : &tm_x_hi;
        const uint32_t da = dst + pl * a_plane, db = dst + b_off + pl * b_plane;
        for (int a = 0; a < nA; ++a) tma_load_4d(da + a * kBoxA, tg, co0 + 64 * a, x0 + args.g_pad, y0 + args.g_pad, n, full(s));
        for (int j = 0; j < nB; ++j)
          tma_load_4d(db + j * kBoxA, tx, ci0 + 64 * j, x0 + kw * args.dil + args.x_off, y0 + kh * args.dil + args.y_off, n, full(s));
      }
    };
    auto release = [&](int j) {                                  // patch j's MMAs are done: refill its stage with patch j + S
      __syncwarp();
      if (lane == 0) mbar_arrive(empty((g + (uint32_t)j) % (uint32_t)S));
      if (tid == 0 && j + S < nk) issue(j + S);
    };
    if (tid == 0)
      for (int i = 0; i < min(S, nk); ++i) issue(i);
    wgmma_fence_acc(acc);
    for (int i = 0; i < nk; ++i) {                                 // one wgmma group stays in flight
      const uint32_t gi = g + (uint32_t)i, s = gi % (uint32_t)S;
      mbar_wait(full(s), (gi / (uint32_t)S) & 1u);
      constexpr uint64_t kDescA = wgmma_desc_hi(kBoxA), kDescB = wgmma_desc_hi(kBoxA);
      const uint32_t a_hi = smem_base + stage * s + a_box, b_hi = smem_base + stage * s + b_off;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {                                 // 4 k-steps of 16 pixels = 2048 bytes of each box
        const uint64_t dah = wgmma_desc(kDescA, a_hi + 2048u * k), dbh = wgmma_desc(kDescB, b_hi + 2048u * k);
        Wgmma<BNc, 1, 1>::mma(acc, dah, dbh, (i | k) ? 1u : 0u);
        if constexpr (split) {
          Wgmma<BNc, 1, 1>::mma(acc, dah, wgmma_desc(kDescB, b_hi + b_plane + 2048u * k), 1u);
          Wgmma<BNc, 1, 1>::mma(acc, wgmma_desc(kDescA, a_hi + a_plane + 2048u * k), dbh, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (i > 0) release(i - 1);
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    if (nk > 0) release(nk - 1);
    g += (uint32_t)nk;
    // ===================== epilogue: accumulator registers -> atomics into dW[co][tap][ci] =====================
    if (active && nk > 0) {
      const int co_a = co0 + wg * 64 + (warp & 3) * 16 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int co = co_a + 8 * h;
        if (co < args.cout) {
          float* dst = args.dw + ((size_t)co * taps + tap) * args.cin + ci0 + c;
          // the parameter spans of the flat gradient buffer are only 4-byte aligned in general (head biases of 6*25 floats)
          const bool al8 = (reinterpret_cast<uintptr_t>(dst) & 7u) == 0;
#pragma unroll
          for (int j = 0; j < BNc / 8; ++j) {
            const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
            if (al8) red_add_v2(dst + 8 * j, v0, v1);
            else { atomicAdd(dst + 8 * j, v0); atomicAdd(dst + 8 * j + 1, v1); }
          }
        }
      }
    }
  }
}

// bias gradient: gb[c] += sum over all rows of the zero-bordered gradient tensor (borders contribute 0)
__global__ void __launch_bounds__(256) bias_grad_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo, int Cs, int C,
                                                        long long rows, long long rows_per_block, float* __restrict__ gb) {
  extern __shared__ float s_part[];                          // [row lanes][Cs]
  const int CG = Cs >> 3;
  const int rl = threadIdx.x / CG, RL = 256 / CG;
  const int c = (threadIdx.x - rl * CG) * 8;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (rl < RL) {
    const long long r0 = (long long)blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
    for (long long r = r0 + rl; r < r1; r += RL) {
      float v[8];
      unpack8(*reinterpret_cast<const uint4*>(hi + r * Cs + c), v);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += v[e];
      if (lo) {
        unpack8(*reinterpret_cast<const uint4*>(lo + r * Cs + c), v);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] += v[e];
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) s_part[rl * Cs + c + e] = acc[e];
  }
  __syncthreads();
  for (int ch = threadIdx.x; ch < C; ch += 256) {
    float t = 0.f;
    for (int l = 0; l < RL; ++l) t += s_part[l * Cs + ch];
    atomicAdd(gb + ch, t);
  }
}

}  // namespace

bool wgrad_supported(const ActBuf& X, const ActBuf& G, int kh, int kw, int stride, int dil) {
  return stride == 1 && X.C % 64 == 0 && X.Cs == X.C && kw <= 3 && kh <= 8 && G.Cs % 8 == 0 && (kw - 1) * dil <= 16;
}

int plan_wgrad(ssdk_ctx* ctx, WgradLaunch& L, const ActBuf& X, const ActBuf& G, int Ho, int Wo, int KH, int KW, int dil, int pad_t, int pad_l,
               int split, float* dw) {
  WgradArgs& a = L.args;
  a = WgradArgs{};
  a.KH = KH; a.KW = KW; a.dil = dil; a.split = split ? 1 : 0;
  a.cin = X.C; a.cout = G.C; a.taps = KH * KW;
  a.BNc = (X.C % 128 == 0) ? 128 : 64;
  a.ci_tiles = X.C / a.BNc;
  a.co_tiles = (G.C + 127) / 128;
  a.a_boxes = G.C <= 64 ? 1 : 2;
  // pixel patches: bw x bh = 64, bw a multiple of 16 (one wgmma k-step never straddles a patch line)
  int best_bw = 16; double best = 1e30;
  for (int bw : {64, 32, 16}) {
    const int bh = 64 / bw;
    const double cost = (double)((Wo + bw - 1) / bw * bw) * ((Ho + bh - 1) / bh * bh);
    if (cost < best) { best = cost; best_bw = bw; }
  }
  a.bw = best_bw; a.bh = 64 / best_bw;
  a.px_tiles = (Wo + a.bw - 1) / a.bw; a.py_tiles = (Ho + a.bh - 1) / a.bh;
  a.total_patches = G.B * a.px_tiles * a.py_tiles;
  a.g_pad = G.pad;
  a.x_off = X.pad - pad_l; a.y_off = X.pad - pad_t;
  const size_t stage = ((size_t)2 * kBoxA + (size_t)(a.BNc / 64) * kBoxA) * (a.split ? 2 : 1);
  a.tx_bytes = (uint32_t)(((size_t)a.a_boxes * kBoxA + (size_t)(a.BNc / 64) * kBoxA) * (a.split ? 2 : 1));
  a.stages = (int)std::min<size_t>(6, (220 * 1024) / stage);
  if (a.stages < 2) { set_error("wgrad: stage of %zu bytes does not fit twice in shared memory", stage); return SSDK_ERR_UNSUPPORTED; }
  L.smem = 1024 + stage * a.stages + 256;
  const int base_units = a.co_tiles * a.ci_tiles * KH * KW;
  int ks = std::max(1, (2 * ctx->sm_count + base_units - 1) / base_units);
  ks = std::min(ks, std::max(1, a.total_patches / 4));
  a.patches_per_split = (a.total_patches + ks - 1) / ks;
  a.k_split = (a.total_patches + a.patches_per_split - 1) / a.patches_per_split;
  L.grid = std::min(base_units * a.k_split, ctx->sm_count);
  a.dw = dw;
  const uint64_t gd[4] = {(uint64_t)G.Cs, (uint64_t)G.Wp(), (uint64_t)G.Hp(), (uint64_t)G.B};
  const uint64_t xd[4] = {(uint64_t)X.Cs, (uint64_t)X.Wp(), (uint64_t)X.Hp(), (uint64_t)X.B};
  const uint32_t gb[4] = {64, (uint32_t)a.bw, (uint32_t)a.bh, 1};
  const uint32_t xb[4] = {64, (uint32_t)a.bw, (uint32_t)a.bh, 1};
  int rc = make_tmap_4d(&L.g_hi, G.hi, gd, gb); if (rc) return rc;
  rc = make_tmap_4d(&L.x_hi, X.hi, xd, xb); if (rc) return rc;
  if (a.split) {
    rc = make_tmap_4d(&L.g_lo, G.lo, gd, gb); if (rc) return rc;
    rc = make_tmap_4d(&L.x_lo, X.lo, xd, xb); if (rc) return rc;
  } else { L.g_lo = L.g_hi; L.x_lo = L.x_hi; }
  L.flops = 2.0 * a.cout * a.taps * a.cin * (double)G.B * Ho * Wo;
  return SSDK_OK;
}

template <int BNc, bool SPLIT>
static int launch_wgrad_bn(const WgradLaunch& L, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    SSDK_CHECK_CUDA(cudaFuncSetAttribute(wgrad_wgmma_kernel<BNc, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  wgrad_wgmma_kernel<BNc, SPLIT><<<L.grid, 256, L.smem, stream>>>(L.g_hi, L.g_lo, L.x_hi, L.x_lo, L.args);
  return SSDK_OK;
}

int launch_wgrad(ssdk_ctx* ctx, const WgradLaunch& L, cudaStream_t stream) {
  const bool sp = L.args.split != 0;
  const int rc = L.args.BNc == 128 ? (sp ? launch_wgrad_bn<128, true>(L, stream) : launch_wgrad_bn<128, false>(L, stream))
                                   : (sp ? launch_wgrad_bn<64, true>(L, stream) : launch_wgrad_bn<64, false>(L, stream));
  if (rc) return rc;
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

int launch_bias_grad(ssdk_ctx* ctx, const ActBuf& G, float* gb, cudaStream_t stream) {
  if (G.Cs > 2048) { set_error("bias gradient: more than 2048 channels"); return SSDK_ERR_UNSUPPORTED; }
  const long long rows = (long long)G.rows();
  const int blocks = (int)std::min<long long>(4LL * ctx->sm_count, std::max<long long>(1, rows / 64));
  const long long rpb = (rows + blocks - 1) / blocks;
  const int RL = 256 / (G.Cs / 8);
  bias_grad_kernel<<<blocks, 256, (size_t)std::max(1, RL) * G.Cs * sizeof(float), stream>>>(G.hi, G.lo, G.Cs, G.C, rows, rpb, gb);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

}  // namespace ssdk
