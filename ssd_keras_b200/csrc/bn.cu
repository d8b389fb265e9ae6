// BatchNormalization in Keras' training phase + activation, forward and backward, for the conv + BN + ELU stages of SSD7
// (reference models/keras_ssd7.py:277-309: Conv2D -> BatchNormalization(axis=3, momentum=0.99) -> ELU; the arithmetic itself is
// TensorFlow's: batch mean / biased variance over (B,H,W), epsilon 1e-3 (Keras default), moving averages updated with the
// unbiased variance like tf.nn.fused_batch_norm).  HBM-bound elementwise / reduction kernels on the bf16 hi+lo activation planes.
//   forward   bn_stats_kernel (per-channel sum, sum of squares in float64) -> bn_finalize_kernel (mean, rstd, moving averages)
//             -> bn_apply_kernel (a = act(gamma * (z - mean) * rstd + beta), written into the zero-bordered output planes)
//   backward  bn_bwd_reduce_kernel (sum dy, sum dy * xhat with dy = da * act'(a)) -> bn_bwd_apply_kernel
//             (dz = gamma * rstd * (dy - mean(dy) - xhat * mean(dy * xhat)), in place on the gradient planes; dgamma, dbeta)
#include "model.cuh"

namespace ssdk {

namespace {

__device__ __forceinline__ float act_bwd(float a, int act) {      // derivative expressed through the activation's OUTPUT a
  if (act == SSDK_ACT_RELU) return a > 0.f ? 1.f : 0.f;
  if (act == SSDK_ACT_ELU) return a > 0.f ? 1.f : a + 1.f;       // d/dy (e^y - 1) = e^y = a + 1
  return 1.f;
}

// element e -> (pixel, channel group of 8); pixels are the valid (unpadded) positions
struct Elem { int n, y, x, g; bool ok; };
__device__ __forceinline__ Elem elem_of(const ActBuf& a, size_t e, int groups) {
  Elem r;
  r.g = (int)(e % groups);
  const size_t pix = e / groups;
  r.x = (int)(pix % a.W); r.y = (int)((pix / a.W) % a.H); r.n = (int)(pix / ((size_t)a.W * a.H));
  r.ok = r.n < a.B;
  return r;
}

__global__ void __launch_bounds__(256) bn_stats_kernel(ActBuf z, double* __restrict__ acc /* [2*C] */) {
  extern __shared__ double s_acc[];                 // [2*Cs]
  const int groups = z.Cs / 8;
  for (int i = threadIdx.x; i < 2 * z.Cs; i += 256) s_acc[i] = 0.0;
  __syncthreads();
  const size_t total = (size_t)z.B * z.H * z.W * groups;
  // a thread keeps one channel group while it strides over the pixels: gridDim.x * 256 is a multiple of `groups`
  double s[8], q[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { s[e] = 0.0; q[e] = 0.0; }
  int g = -1;
  for (size_t e = (size_t)blockIdx.x * 256 + threadIdx.x; e < total; e += (size_t)gridDim.x * 256) {
    const Elem el = elem_of(z, e, groups);
    g = el.g;
    float v[8];
    split_load8(z.hi, z.lo, act_index(z, el.n, el.y, el.x) + (size_t)el.g * 8, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) { s[k] += (double)v[k]; q[k] += (double)v[k] * (double)v[k]; }
  }
  if (g >= 0) {
#pragma unroll
    for (int k = 0; k < 8; ++k) { atomicAdd(&s_acc[g * 8 + k], s[k]); atomicAdd(&s_acc[z.Cs + g * 8 + k], q[k]); }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < z.C; i += 256) { atomicAdd(acc + i, s_acc[i]); atomicAdd(acc + z.C + i, s_acc[z.Cs + i]); }
}

__global__ void bn_finalize_kernel(double* __restrict__ acc, int C, double N, float eps, float momentum, float* __restrict__ bmean,
                                   float* __restrict__ brstd, float* __restrict__ mmean, float* __restrict__ mvar) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double mean = acc[c] / N;
  double var = acc[C + c] / N - mean * mean;
  if (var < 0.0) var = 0.0;
  bmean[c] = (float)mean;
  brstd[c] = (float)(1.0 / sqrt(var + (double)eps));
  const double unbiased = N > 1.0 ? var * N / (N - 1.0) : var;
  mmean[c] = momentum * mmean[c] + (1.f - momentum) * (float)mean;
  mvar[c] = momentum * mvar[c] + (1.f - momentum) * (float)unbiased;
  acc[c] = 0.0; acc[C + c] = 0.0;                    // ready for the next reduction
}

__global__ void __launch_bounds__(256) bn_apply_kernel(ActBuf z, ActBuf out, const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       const float* __restrict__ bmean, const float* __restrict__ brstd, int act) {
  const int groups = z.Cs / 8;
  const size_t total = (size_t)z.B * z.H * z.W * groups;
  const size_t e = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (e >= total) return;
  const Elem el = elem_of(z, e, groups);
  float v[8], o[8];
  split_load8(z.hi, z.lo, act_index(z, el.n, el.y, el.x) + (size_t)el.g * 8, v);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int c = el.g * 8 + k;
    o[k] = 0.f;
    if (c < z.C) o[k] = apply_act(gamma[c] * ((v[k] - bmean[c]) * brstd[c]) + beta[c], act);
  }
  split_store8(out.hi, out.lo, act_index(out, el.n, el.y, el.x) + (size_t)el.g * 8, o);
}

__global__ void __launch_bounds__(256) bn_bwd_reduce_kernel(ActBuf z, ActBuf a, ActBuf g, const float* __restrict__ bmean, const float* __restrict__ brstd,
                                                            int act, double* __restrict__ acc) {
  extern __shared__ double s_acc[];
  const int groups = z.Cs / 8;
  for (int i = threadIdx.x; i < 2 * z.Cs; i += 256) s_acc[i] = 0.0;
  __syncthreads();
  const size_t total = (size_t)z.B * z.H * z.W * groups;
  double s[8], q[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { s[e] = 0.0; q[e] = 0.0; }
  int gg = -1;
  for (size_t e = (size_t)blockIdx.x * 256 + threadIdx.x; e < total; e += (size_t)gridDim.x * 256) {
    const Elem el = elem_of(z, e, groups);
    gg = el.g;
    float zv[8], av[8], dv[8];
    split_load8(z.hi, z.lo, act_index(z, el.n, el.y, el.x) + (size_t)el.g * 8, zv);
    split_load8(a.hi, a.lo, act_index(a, el.n, el.y, el.x) + (size_t)el.g * 8, av);
    split_load8(g.hi, g.lo, act_index(g, el.n, el.y, el.x) + (size_t)el.g * 8, dv);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = el.g * 8 + k;
      if (c < z.C) {
        const float dy = dv[k] * act_bwd(av[k], act);
        const float xh = (zv[k] - bmean[c]) * brstd[c];
        s[k] += (double)dy; q[k] += (double)dy * (double)xh;
      }
    }
  }
  if (gg >= 0) {
#pragma unroll
    for (int k = 0; k < 8; ++k) { atomicAdd(&s_acc[gg * 8 + k], s[k]); atomicAdd(&s_acc[z.Cs + gg * 8 + k], q[k]); }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < z.C; i += 256) { atomicAdd(acc + i, s_acc[i]); atomicAdd(acc + z.C + i, s_acc[z.Cs + i]); }
}

__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(ActBuf z, ActBuf a, ActBuf g, const float* __restrict__ gamma, const float* __restrict__ bmean,
                                                           const float* __restrict__ brstd, int act, const double* __restrict__ acc, double N,
                                                           float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const int groups = z.Cs / 8;
  const size_t total = (size_t)z.B * z.H * z.W * groups;
  const size_t e = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (e < (size_t)z.C) { dbeta[e] = (float)acc[e]; dgamma[e] = (float)acc[z.C + e]; }
  if (e >= total) return;
  const Elem el = elem_of(z, e, groups);
  float zv[8], av[8], dv[8], o[8];
  const size_t iz = act_index(z, el.n, el.y, el.x) + (size_t)el.g * 8, ig = act_index(g, el.n, el.y, el.x) + (size_t)el.g * 8;
  split_load8(z.hi, z.lo, iz, zv);
  split_load8(a.hi, a.lo, act_index(a, el.n, el.y, el.x) + (size_t)el.g * 8, av);
  split_load8(g.hi, g.lo, ig, dv);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int c = el.g * 8 + k;
    o[k] = 0.f;
    if (c < z.C) {
      const float dy = dv[k] * act_bwd(av[k], act);
      const float xh = (zv[k] - bmean[c]) * brstd[c];
      const float m1 = (float)(acc[c] / N), m2 = (float)(acc[z.C + c] / N);
      o[k] = gamma[c] * brstd[c] * (dy - m1 - xh * m2);
    }
  }
  split_store8(g.hi, g.lo, ig, o);
}

__global__ void zero_acc_kernel(double* acc, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) acc[i] = 0.0;
}

int bn_grid(const ActBuf& z, int sm_count) {
  const int groups = z.Cs / 8;
  const size_t total = (size_t)z.B * z.H * z.W * groups;
  int blocks = (int)std::min<size_t>((total + 255) / 256, (size_t)sm_count * 8);
  // gridDim * 256 must be a multiple of `groups` so that a thread keeps its channel group while striding
  while (blocks > 1 && ((size_t)blocks * 256) % groups != 0) --blocks;
  if (((size_t)blocks * 256) % groups != 0) blocks = groups;       // 256 * groups is always a multiple
  return std::max(blocks, 1);
}

}  // namespace

int launch_bn_forward(ssdk_ctx* ctx, LayerPlan& L, int act, cudaStream_t s) {
  const ActBuf& z = L.z;
  const int groups = z.Cs / 8;
  const size_t total = (size_t)z.B * z.H * z.W * groups;
  const double N = (double)z.B * z.H * z.W;
  if (int rc = launch(ctx, bn_stats_kernel, bn_grid(z, ctx->sm_count), 256, (size_t)2 * z.Cs * sizeof(double), s, z, L.bn_acc)) return rc;
  if (int rc = launch(ctx, bn_finalize_kernel, (z.C + 127) / 128, 128, 0, s,
                      L.bn_acc, z.C, N, L.bn_eps, L.bn_momentum, L.bn_bmean, L.bn_brstd, L.bn_mmean, L.bn_mvar)) return rc;
  return launch(ctx, bn_apply_kernel, (unsigned)((total + 255) / 256), 256, 0, s, z, L.out, L.bn_gamma, L.bn_beta, L.bn_bmean, L.bn_brstd, act);
}

int launch_bn_backward(ssdk_ctx* ctx, LayerPlan& L, int act, const ActBuf& g, float* dgamma, float* dbeta, cudaStream_t s) {
  const ActBuf& z = L.z;
  const int groups = z.Cs / 8;
  const size_t total = (size_t)z.B * z.H * z.W * groups;
  const double N = (double)z.B * z.H * z.W;
  if (int rc = launch(ctx, bn_bwd_reduce_kernel, bn_grid(z, ctx->sm_count), 256, (size_t)2 * z.Cs * sizeof(double), s,
                      z, L.out, g, L.bn_bmean, L.bn_brstd, act, L.bn_acc)) return rc;
  if (int rc = launch(ctx, bn_bwd_apply_kernel, (unsigned)((std::max(total, (size_t)z.C) + 255) / 256), 256, 0, s,
                      z, L.out, g, L.bn_gamma, L.bn_bmean, L.bn_brstd, act, L.bn_acc, N, dgamma, dbeta)) return rc;
  return launch(ctx, zero_acc_kernel, (2 * z.C + 127) / 128, 128, 0, s, L.bn_acc, 2 * z.C);
}

}  // namespace ssdk
