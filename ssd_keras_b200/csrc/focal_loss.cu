// The softmax focal loss (Lin et al., arXiv:1708.02002) on SSDLoss's input layout, as two launches:
//
//   focal_count_kernel  phase 0: N = sum over the rows of pos = max_{c=1..C-1} y_true[c] (SSDLoss's positives, fractional values
//                       included), added to a caller-visible int64 in 32.32 fixed point, so the sum does not depend on the order
//                       the CTAs arrive in (nor on how the batch is split over ranks, whose counts are all-reduced in between).
//   focal_loss_kernel   phase 1, one pass over the rows: per box cls = sum_c y_true[c] w_c (1 - q_c)^gamma (-log max(q_c, 1e-15))
//                       and pos * smooth-L1 of the offsets; per-tile double partials, reduced per image by the last CTA to finish;
//                       and / or the gradient rows.
//
// One CTA per tile of 128 rows of one image.  The tile is a contiguous run of 128 * (C + 12) floats; the threads stream it element
// by element (4 consecutive elements per thread and step, float4 loads and stores when the tiles start 16-byte aligned, plain
// loads otherwise, with the same element-to-thread mapping), so no shared-memory buffer grows with the number of classes and
// both load paths give the same bits.  Only pos needs a whole row; it is computed first, each warp for 16 rows, into shared memory.
// No float atomics: the output is bit-reproducible and a sharded batch gives the single launch's per-image losses and gradient
// rows bit for bit.
#include "common.cuh"
#include <cmath>

using namespace ssdk;

namespace {

constexpr int kRows = 128;             // rows per tile
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr float kEps = 1e-15f;         // the log's clamp, as SSDLoss (keras_ssd_loss.py:93)

struct FocalArgs {
  const float* y_true; const float* y_pred;
  int B, P, C, W;
  int tiles_per_img;
  float gamma, w_bg, w_fg, alpha;      // w_bg = 1 - focal_alpha (class 0), w_fg = focal_alpha (classes >= 1)
  int global_B;                        // batch size of the normalisation
  long long* count;                    // sum of llrint(pos * 2^32) over the (global) batch
  double* part;                        // [n_tiles * 2] sum of cls terms, sum of pos * smooth-L1 terms
  int* ticket;
  const float* upstream; float* out_loss; float* out_grad;
  int vec;                             // tiles start 16-byte aligned in every tensor: float4 loads / stores
};

__device__ __forceinline__ void tile_of(const FocalArgs& a, int& b, int& rows, size_t& row0) {
  b = blockIdx.x / a.tiles_per_img;
  const int blk = blockIdx.x - b * a.tiles_per_img;
  rows = min(kRows, a.P - blk * kRows);
  row0 = (size_t)b * a.P + (size_t)blk * kRows;
}

// pos of the rows warp, warp + kWarps, ... of a tile (lane 0 gets them): the max over the class columns 1 .. C-1 of y_true.  The
// loads of all the warp's rows are issued before any of them is reduced; fmaxf does not depend on the order.
constexpr int kRowsPerWarp = kRows / kWarps;
__device__ __forceinline__ void tile_pos(const FocalArgs& a, size_t row0, int rows, int warp, int lane, float (&m)[kRowsPerWarp]) {
#pragma unroll
  for (int i = 0; i < kRowsPerWarp; ++i) m[i] = -INFINITY;
  const float* yt = a.y_true + row0 * a.W;
  for (int c = 1 + lane; c < a.C; c += 32) {
#pragma unroll
    for (int i = 0; i < kRowsPerWarp; ++i) {
      const int r = warp + i * kWarps;
      if (r < rows) m[i] = fmaxf(m[i], __ldg(yt + (size_t)r * a.W + c));
    }
  }
#pragma unroll
  for (int i = 0; i < kRowsPerWarp; ++i)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m[i] = fmaxf(m[i], __shfl_xor_sync(0xffffffffu, m[i], o));
}

template <typename T>
__device__ __forceinline__ T block_sum(T v, T* s_red) {        // fixed-order block reduction, result in thread 0
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  T s = s_red[0];
#pragma unroll
  for (int w = 1; w < kWarps; ++w) s += s_red[w];
  __syncthreads();
  return s;
}

// ---- phase 0 -------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) focal_count_kernel(const __grid_constant__ FocalArgs a) {
  __shared__ long long s_red[kWarps];
  int b, rows; size_t row0;
  tile_of(a, b, rows, row0);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float m[kRowsPerWarp];
  tile_pos(a, row0, rows, warp, lane, m);
  long long acc = 0;
#pragma unroll
  for (int i = 0; i < kRowsPerWarp; ++i)
    if (lane == 0 && warp + i * kWarps < rows) acc += llrint((double)m[i] * 4294967296.0);
  const long long s = block_sum(acc, s_red);
  if (threadIdx.x == 0 && s) atomicAdd(reinterpret_cast<unsigned long long*>(a.count), (unsigned long long)s);
}

// ---- phase 1 -------------------------------------------------------------------------------------------------------------
// One element of a row: its loss terms (into the thread's double sums) and its gradient.
template <bool kGrad>
__device__ __forceinline__ float focal_elem(const FocalArgs& a, float tv, float q, int col, float pos, float scale, double& acc_c,
                                            double& acc_l) {
  float g = 0.f;
  if (col < a.C) {
    if (tv != 0.f) {                                                     // neutral rows and the zero entries carry nothing
      const float w = (col == 0 ? a.w_bg : a.w_fg) * tv;
      const float omq = 1.0f - q;
      const float lg = logf(fmaxf(q, kEps));
      const float pw = powf(omq, a.gamma);
      acc_c += (double)((w * pw) * -lg);
      if (kGrad) {
        // d/dq (1-q)^gamma (-log max(q, eps)) = gamma (1-q)^(gamma-1) log max(q, eps) - [q >= eps] (1-q)^gamma / q; the first
        // term is 0 where log q = 0 (q = 1, its limit) or gamma = 0
        const float d1 = (a.gamma != 0.f && lg != 0.f) ? (a.gamma * powf(omq, a.gamma - 1.0f)) * lg : 0.f;
        const float d2 = (q >= kEps) ? pw / q : 0.f;
        g = ((d1 - d2) * w) * scale;
      }
    }
  } else if (col < a.C + 4) {
    const float d = tv - q;
    const float ad = fabsf(d);
    acc_l += (double)(((ad < 1.0f) ? 0.5f * d * d : ad - 0.5f) * pos);  // SSDLoss's smooth-L1 (keras_ssd_loss.py:72-74)
    if (kGrad) {
      const float e = q - tv;
      g = ((fabsf(e) < 1.0f) ? e : (e > 0.f ? 1.f : (e < 0.f ? -1.f : 0.f))) * ((pos * scale) * a.alpha);
    }
  }
  return g;
}

template <bool kGrad>
__global__ void __launch_bounds__(kThreads) focal_loss_kernel(const __grid_constant__ FocalArgs a) {
  __shared__ float s_pos[kRows];
  __shared__ double s_red[kWarps];
  __shared__ int s_is_last;
  int b, rows; size_t row0;
  tile_of(a, b, rows, row0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  {
    float m[kRowsPerWarp];
    tile_pos(a, row0, rows, warp, lane, m);
#pragma unroll
    for (int i = 0; i < kRowsPerWarp; ++i)
      if (lane == 0 && warp + i * kWarps < rows) s_pos[warp + i * kWarps] = m[i];
  }
  __syncthreads();
  const double n_pos = (double)__ldcg(a.count) / 4294967296.0;
  const double norm = fmax(1.0, n_pos);
  float scale = 0.f;                                                     // d L_b / d (per-box loss) times u_b
  if (kGrad) {
    const double up = a.upstream ? (double)a.upstream[b] : 1.0 / (double)a.global_B;
    scale = (float)(up * (double)a.global_B / norm);
  }
  const int W = a.W, n = rows * W;
  const float* yt = a.y_true + row0 * W;
  const float* yp = a.y_pred + row0 * W;
  float* gr = kGrad ? a.out_grad + row0 * W : nullptr;
  double acc_c = 0.0, acc_l = 0.0;
  for (int e = 4 * tid; e < n; e += 4 * kThreads) {
    const int m = min(4, n - e);
    float tv[4] = {0.f, 0.f, 0.f, 0.f}, qv[4] = {0.f, 0.f, 0.f, 0.f}, gv[4];
    if (a.vec && m == 4) {
      const float4 t4 = __ldcs(reinterpret_cast<const float4*>(yt + e));
      const float4 q4 = __ldcs(reinterpret_cast<const float4*>(yp + e));
      tv[0] = t4.x; tv[1] = t4.y; tv[2] = t4.z; tv[3] = t4.w;
      qv[0] = q4.x; qv[1] = q4.y; qv[2] = q4.z; qv[3] = q4.w;
    } else {
      for (int j = 0; j < m; ++j) { tv[j] = __ldcs(yt + e + j); qv[j] = __ldcs(yp + e + j); }
    }
    int row = e / W, col = e - row * W;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      gv[j] = 0.f;
      if (j < m) {
        gv[j] = focal_elem<kGrad>(a, tv[j], qv[j], col, s_pos[row], scale, acc_c, acc_l);
        if (++col == W) { col = 0; ++row; }
      }
    }
    if (kGrad) {
      if (a.vec && m == 4) __stcs(reinterpret_cast<float4*>(gr + e), make_float4(gv[0], gv[1], gv[2], gv[3]));
      else for (int j = 0; j < m; ++j) __stcs(gr + e + j, gv[j]);
    }
  }
  if (!a.out_loss) return;
  acc_c = block_sum(acc_c, s_red);
  acc_l = block_sum(acc_l, s_red);
  if (tid == 0) {
    a.part[(size_t)blockIdx.x * 2] = acc_c;
    a.part[(size_t)blockIdx.x * 2 + 1] = acc_l;
    __threadfence();
    const int old = atomicAdd(a.ticket, 1);
    s_is_last = (old == (int)gridDim.x - 1);
    if (s_is_last) *a.ticket = 0;
    __threadfence();
  }
  __syncthreads();
  if (!s_is_last) return;
  // the last CTA: per-image totals, one warp per image, lanes over the image's tiles in a fixed order
  for (int img = warp; img < a.B; img += kWarps) {
    double c = 0.0, l = 0.0;
    for (int i = lane; i < a.tiles_per_img; i += 32) {
      const size_t t = (size_t)img * a.tiles_per_img + i;
      c += __ldcg(a.part + t * 2); l += __ldcg(a.part + t * 2 + 1);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { c += __shfl_xor_sync(0xffffffffu, c, o); l += __shfl_xor_sync(0xffffffffu, l, o); }
    if (lane == 0) a.out_loss[img] = (float)((c + (double)a.alpha * l) / norm * (double)a.global_B);
  }
}

int check_args(ssdk_ctx* ctx, const char* fn, const float* yt, const float* yp, int B, int P, int C, float gamma, float focal_alpha,
               bool has_output) {
  SSDK_REQUIRE(ctx && yt && yp, "%s: NULL argument", fn);
  SSDK_REQUIRE(B > 0 && P > 0 && C > 1, "%s: bad shape (B=%d, P=%d, n_classes_total=%d)", fn, B, P, C);
  SSDK_REQUIRE((long long)B * P < (1ll << 31) && (long long)kRows * (C + 12) < (1ll << 31), "%s: B*P or n_classes_total too large", fn);
  SSDK_REQUIRE(gamma >= 0.f, "%s: gamma must be >= 0, got %g", fn, (double)gamma);
  SSDK_REQUIRE(focal_alpha >= 0.f && focal_alpha <= 1.f, "%s: focal_alpha must lie in [0, 1], got %g", fn, (double)focal_alpha);
  SSDK_REQUIRE(has_output, "%s: out_loss and out_grad are both NULL", fn);
  return SSDK_OK;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

void fill_args(FocalArgs& a, const float* yt, const float* yp, int B, int P, int C, float gamma, float focal_alpha, float alpha,
               int global_B, const float* upstream, float* out_loss, float* out_grad) {
  memset(&a, 0, sizeof(a));
  a.y_true = yt; a.y_pred = yp; a.B = B; a.P = P; a.C = C; a.W = C + 12;
  a.tiles_per_img = (P + kRows - 1) / kRows;
  a.gamma = gamma; a.w_bg = (float)(1.0 - (double)focal_alpha); a.w_fg = focal_alpha; a.alpha = alpha;
  a.global_B = global_B;
  a.upstream = upstream; a.out_loss = out_loss; a.out_grad = out_grad;
  a.vec = ((size_t)P * a.W % 4 == 0) && aligned16(yt) && aligned16(yp) && (!out_grad || aligned16(out_grad)) ? 1 : 0;
}

// the context's workspace: the ticket and the tile partials of phase 1, and the count of the single-process call
int own_ws(ssdk_ctx* ctx, FocalArgs& a, cudaStream_t stream) {
  const size_t n_tiles = (size_t)a.B * a.tiles_per_img;
  const size_t before = ctx->focal_ws.bytes;
  int rc = ctx->focal_ws.ensure(256 + n_tiles * 16);
  if (rc) return rc;
  unsigned char* ws = reinterpret_cast<unsigned char*>(ctx->focal_ws.ptr);
  if (ctx->focal_ws.bytes != before) SSDK_CHECK_CUDA(cudaMemsetAsync(ws, 0, 256, stream));   // the ticket starts at 0 and resets itself
  a.ticket = reinterpret_cast<int*>(ws + 8);
  a.part = reinterpret_cast<double*>(ws + 256);
  return SSDK_OK;
}

int run_phase(ssdk_ctx* ctx, int phase, FocalArgs& a, cudaStream_t stream) {
  const dim3 grid((unsigned)(a.B * a.tiles_per_img));
  if (phase == 0) return launch(ctx, focal_count_kernel, grid, kThreads, 0, stream, a);
  if (a.out_grad) return launch(ctx, focal_loss_kernel<true>, grid, kThreads, 0, stream, a);
  return launch(ctx, focal_loss_kernel<false>, grid, kThreads, 0, stream, a);
}

}  // namespace

extern "C" int ssdk_focal_loss(ssdk_ctx* ctx, const float* y_true, const float* y_pred, int B, int P, int C, float gamma,
                               float focal_alpha, float alpha, const float* upstream, float* out_loss, float* out_grad, void* stream_) {
  int rc = check_args(ctx, "ssdk_focal_loss", y_true, y_pred, B, P, C, gamma, focal_alpha, out_loss || out_grad);
  if (rc) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  FocalArgs a;
  fill_args(a, y_true, y_pred, B, P, C, gamma, focal_alpha, alpha, B, upstream, out_loss, out_grad);
  rc = own_ws(ctx, a, stream);
  if (rc) return rc;
  a.count = reinterpret_cast<long long*>(ctx->focal_ws.ptr);
  SSDK_CHECK_CUDA(cudaMemsetAsync(a.count, 0, 8, stream));
  rc = run_phase(ctx, 0, a, stream);
  if (rc) return rc;
  return run_phase(ctx, 1, a, stream);
}

extern "C" int ssdk_focal_loss_phase(ssdk_ctx* ctx, int phase, const float* y_true, const float* y_pred, int B, int P, int C,
                                     float gamma, float focal_alpha, float alpha, long long* count_dev, int global_B,
                                     const float* upstream, float* out_loss, float* out_grad, void* stream_) {
  SSDK_REQUIRE(phase == 0 || phase == 1, "ssdk_focal_loss_phase: phase must be 0 or 1, got %d", phase);
  int rc = check_args(ctx, "ssdk_focal_loss_phase", y_true, y_pred, B, P, C, gamma, focal_alpha,
                      phase == 0 || out_loss || out_grad);
  if (rc) return rc;
  SSDK_REQUIRE(count_dev && global_B >= B, "ssdk_focal_loss_phase: count_dev is NULL or global_B (%d) < B (%d)", global_B, B);
  cudaStream_t stream = (cudaStream_t)stream_;
  FocalArgs a;
  fill_args(a, y_true, y_pred, B, P, C, gamma, focal_alpha, alpha, global_B, upstream, out_loss, out_grad);
  a.count = count_dev;
  if (phase == 1) {
    rc = own_ws(ctx, a, stream);
    if (rc) return rc;
  }
  return run_phase(ctx, phase, a, stream);
}
