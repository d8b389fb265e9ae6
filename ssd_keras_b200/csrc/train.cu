// Training step for the SSD graphs on sm_90a: backward pass + SGD.  Replaces what TensorFlow/Keras do for the reference
// in fit_generator (autodiff of models/keras_ssd300.py:263-419 and keras_loss_function/keras_ssd_loss.py:98-211, the
// l2 kernel regulariser models/keras_ssd300.py:274 and SGD(lr, momentum) ssd300_training.ipynb:169).
//
// Every convolution gradient runs on the SAME wgmma implicit-GEMM kernel as the forward pass (conv.cu):
//   data gradient    dX = conv(dZ, W rotated by 180 degrees with in/out channels swapped), padding dilation*(k-1)-pad;
//                    the epilogue multiplies by ReLU'(forward value) and accumulates when a tensor has several consumers.
//   weight gradient  dW[co][tap][ci] = sum_v dZT[co][v] * XT[ci][v + shift(tap)]: both operands are transposed once into
//                    [channels][pixels] matrices (K = pixels contiguous), each tap is one GEMM whose weight-side operand
//                    is read at a K offset, the pixel axis is split across CTAs (split-K) and reduced with fp32 atomics.
// Operands stay bf16 hi+lo (three MMAs per product) like the forward pass.  Small pieces (max-pool routing, L2Normalization,
// softmax/concat head, bias sums, image-facing 3-channel conv, SGD, re-packing of the bf16 planes) are plain CUDA kernels.
#include "model.cuh"
#include "wgrad.cuh"
#include <climits>

using namespace ssdk;

namespace {

// dst[c][v] = src[row(v)][c] (or 0), v in [0, Kv): K-major operands for the weight-gradient GEMMs.
struct TMap {
  int identity;             // row(v) = v
  int rows_per_img, Wp;     // the X grid the GEMM iterates over
  int Ho, Wo;               // valid extent on that grid
  int src_Hp, src_Wp, src_pad;
};
__global__ void __launch_bounds__(256) transpose_kernel(const __nv_bfloat16* __restrict__ src_hi, const __nv_bfloat16* __restrict__ src_lo,
                                                        int src_ld, long long src_rows, TMap mp, long long row_off, long long Kv, int C,
                                                        __nv_bfloat16* __restrict__ dst_hi, __nv_bfloat16* __restrict__ dst_lo, long long ldT) {
  __shared__ uint16_t th[64][72], tl[64][72];
  const long long v0 = (long long)blockIdx.x * 64;
  const int c0 = blockIdx.y * 64;
  for (int i = threadIdx.x; i < 64 * 8; i += 256) {          // 64 rows x 8 chunks of 8 channels
    const int r = i >> 3, ch = (i & 7) * 8;
    const long long v = v0 + r;
    long long row = -1;
    if (v < Kv) {
      if (mp.identity) row = v + row_off;
      else {
        const long long vs = v + row_off;
        const int n = (int)(vs / mp.rows_per_img); const int rr = (int)(vs - (long long)n * mp.rows_per_img);
        const int y = rr / mp.Wp, x = rr - y * mp.Wp;
        if (y < mp.Ho && x < mp.Wo) row = ((long long)n * mp.src_Hp + (y + mp.src_pad)) * mp.src_Wp + (x + mp.src_pad);
      }
    }
    uint4 h = make_uint4(0, 0, 0, 0), l = h;
    if (row >= 0 && row < src_rows && c0 + ch < src_ld) {
      h = *reinterpret_cast<const uint4*>(src_hi + row * src_ld + c0 + ch);
      if (src_lo) l = *reinterpret_cast<const uint4*>(src_lo + row * src_ld + c0 + ch);
    }
    const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      th[ch + e][r] = (uint16_t)((hw[e >> 1] >> ((e & 1) * 16)) & 0xffffu);
      tl[ch + e][r] = (uint16_t)((lw[e >> 1] >> ((e & 1) * 16)) & 0xffffu);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 64 * 8; i += 256) {          // 64 channels x 8 chunks of 8 pixels
    const int c = i >> 3, vv = (i & 7) * 8;
    if (c0 + c >= C) continue;
    if (v0 + vv >= ldT) continue;
    uint4 h, l;
    h.x = th[c][vv] | ((uint32_t)th[c][vv + 1] << 16); h.y = th[c][vv + 2] | ((uint32_t)th[c][vv + 3] << 16);
    h.z = th[c][vv + 4] | ((uint32_t)th[c][vv + 5] << 16); h.w = th[c][vv + 6] | ((uint32_t)th[c][vv + 7] << 16);
    l.x = tl[c][vv] | ((uint32_t)tl[c][vv + 1] << 16); l.y = tl[c][vv + 2] | ((uint32_t)tl[c][vv + 3] << 16);
    l.z = tl[c][vv + 4] | ((uint32_t)tl[c][vv + 5] << 16); l.w = tl[c][vv + 6] | ((uint32_t)tl[c][vv + 7] << 16);
    *reinterpret_cast<uint4*>(dst_hi + (long long)(c0 + c) * ldT + v0 + vv) = h;
    if (dst_lo) *reinterpret_cast<uint4*>(dst_lo + (long long)(c0 + c) * ldT + v0 + vv) = l;
  }
}

// bias gradient: gb[c] += sum_v dZT[c][v]
__global__ void __launch_bounds__(256) rowsum_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo, long long ldT,
                                                     long long Kv, float* __restrict__ gb) {
  __shared__ float s[8];
  const int c = blockIdx.y;
  const long long chunk = (Kv + gridDim.x - 1) / gridDim.x;
  const long long v0 = (long long)blockIdx.x * chunk, v1 = min(Kv, v0 + chunk);
  float acc = 0.f;
  for (long long v = v0 + threadIdx.x; v < v1; v += 256) {
    acc += __bfloat162float(hi[(long long)c * ldT + v]);
    if (lo) acc += __bfloat162float(lo[(long long)c * ldT + v]);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += s[w];
    atomicAdd(gb + c, t);
  }
}

// Backward of Reshape/softmax/Concat (models/keras_ssd300.py:363-419): dY_pred rows -> gradient of the fused head conv output.
__global__ void head_bwd_kernel(const float* __restrict__ head, const float* __restrict__ dy, int B, int H, int W, int n_boxes, int C,
                                int P, int prior_off, ActBuf g) {
  const size_t wid = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const size_t total = (size_t)B * H * W * n_boxes;
  if (wid >= total) return;
  const int b = (int)(wid % n_boxes); const size_t pix = wid / n_boxes;
  const int hw = H * W;
  const int n = (int)(pix / hw); const int pl = (int)(pix % hw);
  const int y = pl / W, x = pl % W;
  const float* src = head + pix * (size_t)n_boxes * (C + 4) + (size_t)b * (C + 4);
  const float* d = dy + ((size_t)n * P + prior_off + (size_t)pl * n_boxes + b) * (C + 12);
  float mx = -INFINITY;
  for (int c = lane; c < C; c += 32) mx = fmaxf(mx, src[c]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int c = lane; c < C; c += 32) sum += expf(src[c] - mx);
  sum = warp_sum(sum);
  float dot = 0.f;
  for (int c = lane; c < C; c += 32) dot += (expf(src[c] - mx) / sum) * d[c];
  dot = warp_sum(dot);
  const size_t o = act_index(g, n, y, x) + (size_t)b * (C + 4);
  for (int c = lane; c < C; c += 32) { const float p = expf(src[c] - mx) / sum; split_store(g.hi, g.lo, o + c, p * (d[c] - dot)); }
  if (lane < 4) split_store(g.hi, g.lo, o + C + lane, d[C + lane]);
}

// Max-pool backward (gather form): gin(n,y,x,c) (+)= sum over windows whose FIRST maximum is (y,x) of gout; optional ReLU' mask.
// One thread per (input pixel, 8 channels): 16-byte loads of the hi / lo planes.
__global__ void __launch_bounds__(256) pool_bwd_kernel(ActBuf in, ActBuf gout, ActBuf gin, int Hout, int Wout, int KH, int KW, int stride,
                                                       int pad_t, int pad_l, int relu_mask, int accumulate) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int CG = in.C >> 3;
  const size_t total = (size_t)in.B * in.H * in.W * CG;
  if (i >= total) return;
  const int c = (int)(i % CG) * 8; const size_t pix = i / CG;
  const int x = (int)(pix % in.W); const int y = (int)((pix / in.W) % in.H); const int n = (int)(pix / ((size_t)in.W * in.H));
  float v[8], acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  split_load8(in.hi, in.lo, act_index(in, n, y, x) + c, v);
  const int yo_lo = max(0, (y + pad_t - KH + stride) / stride), yo_hi = min(Hout - 1, (y + pad_t) / stride);
  const int xo_lo = max(0, (x + pad_l - KW + stride) / stride), xo_hi = min(Wout - 1, (x + pad_l) / stride);
  for (int yo = yo_lo; yo <= yo_hi; ++yo) {
    const int y0 = yo * stride - pad_t;
    if (y < y0 || y >= y0 + KH) continue;
    for (int xo = xo_lo; xo <= xo_hi; ++xo) {
      const int x0 = xo * stride - pad_l;
      if (x < x0 || x >= x0 + KW) continue;
      // per channel: is (y, x) the first maximum of this window (row-major scan, strict '>')?
      unsigned first = 0xffu;
      for (int ky = 0; ky < KH && first; ++ky) {
        const int yy = y0 + ky;
        if (yy < 0 || yy >= in.H) continue;
        for (int kx = 0; kx < KW; ++kx) {
          const int xx = x0 + kx;
          if (xx < 0 || xx >= in.W || (yy == y && xx == x)) continue;
          float u[8];
          split_load8(in.hi, in.lo, act_index(in, n, yy, xx) + c, u);
          const bool before = (yy < y) || (yy == y && xx < x);
#pragma unroll
          for (int e = 0; e < 8; ++e) if (u[e] > v[e] || (u[e] == v[e] && before)) first &= ~(1u << e);
        }
      }
      if (first) {
        float g[8];
        split_load8(gout.hi, gout.lo, act_index(gout, n, yo, xo) + c, g);
#pragma unroll
        for (int e = 0; e < 8; ++e) if (first & (1u << e)) acc[e] += g[e];
      }
    }
  }
  const size_t o = act_index(gin, n, y, x) + c;
  if (relu_mask) {
#pragma unroll
    for (int e = 0; e < 8; ++e) if (!(v[e] > 0.f)) acc[e] = 0.f;
  }
  if (accumulate) {
    float old[8];
    split_load8(gin.hi, gin.lo, o, old);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] += old[e];
  }
  split_store8(gin.hi, gin.lo, o, acc);
}

// L2Normalization backward (y_c = gamma_c * x_c * s, s = rsqrt(max(sum x^2, 1e-12))): one warp per pixel.
__global__ void l2norm_bwd_kernel(ActBuf x, ActBuf gy, ActBuf gx, const float* __restrict__ gamma, float* __restrict__ ggamma,
                                  int relu_mask, int accumulate) {
  const size_t pix = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const size_t total = (size_t)x.B * x.H * x.W;
  if (pix >= total) return;
  const int xx = (int)(pix % x.W); const int yy = (int)((pix / x.W) % x.H); const int n = (int)(pix / ((size_t)x.W * x.H));
  const size_t sx = act_index(x, n, yy, xx), sg = act_index(gy, n, yy, xx), so = act_index(gx, n, yy, xx);
  float ss = 0.f, dot = 0.f;
  for (int c = lane; c < x.C; c += 32) {
    const float v = split_load(x.hi, x.lo, sx + c);
    ss += v * v;
    dot += gamma[c] * split_load(gy.hi, gy.lo, sg + c) * v;
  }
  ss = warp_sum(ss); dot = warp_sum(dot);
  const bool clamped = !(ss > 1e-12f);
  const float s = rsqrtf(fmaxf(ss, 1e-12f));
  for (int c = lane; c < x.C; c += 32) {
    const float v = split_load(x.hi, x.lo, sx + c), d = split_load(gy.hi, gy.lo, sg + c);
    float g = s * gamma[c] * d;
    if (!clamped) g -= v * s * s * s * dot;
    atomicAdd(ggamma + c, d * v * s);
    if (relu_mask && !(v > 0.f)) g = 0.f;
    if (accumulate) g += split_load(gx.hi, gx.lo, so + c);
    split_store(gx.hi, gx.lo, so + c, g);
  }
}

// Data gradient of a strided convolution: dX = col2im(dCol), dCol = dZ * W^T computed by the GEMM kernel (one tap).
__global__ void col2im_kernel(const float* __restrict__ dcol, int Ho, int Wo, int KH, int KW, int stride, int dil, int pad_t, int pad_l,
                              int ld, ActBuf fwd, ActBuf gin, int relu_mask, int accumulate) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)gin.B * gin.H * gin.W * gin.C;
  if (i >= total) return;
  const int c = (int)(i % gin.C); const size_t pix = i / gin.C;
  const int x = (int)(pix % gin.W); const int y = (int)((pix / gin.W) % gin.H); const int n = (int)(pix / ((size_t)gin.W * gin.H));
  float acc = 0.f;
  for (int kh = 0; kh < KH; ++kh) {
    const int yy = y + pad_t - kh * dil;
    if (yy < 0 || yy % stride) continue;
    const int yo = yy / stride;
    if (yo >= Ho) continue;
    for (int kw = 0; kw < KW; ++kw) {
      const int xx = x + pad_l - kw * dil;
      if (xx < 0 || xx % stride) continue;
      const int xo = xx / stride;
      if (xo >= Wo) continue;
      acc += dcol[(((size_t)n * Ho + yo) * Wo + xo) * ld + (size_t)(kh * KW + kw) * gin.C + c];
    }
  }
  const size_t o = act_index(gin, n, y, x) + c;
  if (relu_mask && !(split_load(fwd.hi, fwd.lo, act_index(fwd, n, y, x) + c) > 0.f)) acc = 0.f;
  if (accumulate) acc += split_load(gin.hi, gin.lo, o);
  split_store(gin.hi, gin.lo, o, acc);
}

// Weight gradient of the image-facing conv (Cin <= 4): gw[co][tap][ci] += sum_pix dZ[pix][co] * X[pix + tap][ci].
// A block owns `rows_per_block` output rows; thread -> (k = tap*cin + ci, 8 output channels), 16-byte loads of dZ.
__global__ void __launch_bounds__(256) wgrad_direct_kernel(ActBuf in, ActBuf g, float* __restrict__ gw, int KH, int KW, int dil,
                                                           int pad_t, int pad_l, int rows_per_block) {
  extern __shared__ float s_acc[];               // [K][Cout]
  const int K = KH * KW * in.C, Cout = g.C;
  for (int i = threadIdx.x; i < K * Cout; i += 256) s_acc[i] = 0.f;
  __syncthreads();
  const int total_rows = g.B * g.H;
  const int r0 = blockIdx.x * rows_per_block, r1 = min(total_rows, r0 + rows_per_block);
  for (int idx = threadIdx.x; idx < K * (Cout / 8); idx += 256) {
    const int k = idx / (Cout / 8), cg = (idx % (Cout / 8)) * 8;
    const int c = k % in.C, tap = k / in.C, kw = tap % KW, kh = tap / KW;
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int r = r0; r < r1; ++r) {
      const int n = r / g.H, yo = r - n * g.H;
      const int y = yo + kh * dil - pad_t;
      if (y < 0 || y >= in.H) continue;
      const int xo_lo = max(0, pad_l - kw * dil), xo_hi = min(g.W, in.W + pad_l - kw * dil);
      size_t xi = act_index(in, n, y, xo_lo + kw * dil - pad_l) + c;
      size_t go = act_index(g, n, yo, xo_lo) + cg;
      for (int xo = xo_lo; xo < xo_hi; ++xo, xi += in.Cs, go += g.Cs) {
        const float xv = split_load(in.hi, in.lo, xi);
        float gv[8];
        split_load8(g.hi, g.lo, go, gv);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] += xv * gv[e];
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) s_acc[k * Cout + cg + e] += acc[e];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < K * Cout; i += 256) {
    const int k = i / Cout, co = i % Cout;
    atomicAdd(gw + (size_t)co * K + k, s_acc[i]);     // OHWI: [co][tap][ci], k = tap*cin + ci
  }
}

// Fast path of the above for the 3x3x3 image-facing kernel (conv1_1): thread -> (2 output channels, pixel lane), all 27
// accumulators per channel in registers; the 3-channel input is read through 8-byte broadcast loads, dZ through coalesced
// 4-byte loads.
__global__ void __launch_bounds__(256) wgrad_direct3x3_kernel(ActBuf in, ActBuf g, float* __restrict__ gw, int pad_t, int pad_l,
                                                              int rows_per_block) {
  extern __shared__ float s_acc[];               // [27][Cout]
  const int Cout = g.C, CG = Cout >> 1, PL = 256 / CG;
  for (int i = threadIdx.x; i < 27 * Cout; i += 256) s_acc[i] = 0.f;
  __syncthreads();
  const int cq = threadIdx.x % CG, pl = threadIdx.x / CG;
  if (pl < PL) {
    float acc[27][2];
#pragma unroll
    for (int k = 0; k < 27; ++k) { acc[k][0] = 0.f; acc[k][1] = 0.f; }
    const int total_rows = g.B * g.H;
    const int r0 = blockIdx.x * rows_per_block, r1 = min(total_rows, r0 + rows_per_block);
    for (int r = r0; r < r1; ++r) {
      const int n = r / g.H, yo = r - n * g.H;
      for (int xo = pl; xo < g.W; xo += PL) {
        const size_t go = act_index(g, n, yo, xo) + 2 * cq;
        const uint32_t gh = *reinterpret_cast<const uint32_t*>(g.hi + go);
        float g0 = __uint_as_float(gh << 16), g1 = __uint_as_float(gh & 0xffff0000u);
        if (g.lo) {
          const uint32_t gl = *reinterpret_cast<const uint32_t*>(g.lo + go);
          g0 += __uint_as_float(gl << 16); g1 += __uint_as_float(gl & 0xffff0000u);
        }
        if (g0 == 0.f && g1 == 0.f) continue;
        // window origin; the buffer's zero border (>= 2 - pad) makes every tap a constant offset from it
        const size_t x00 = (((size_t)n * in.Hp() + (yo - pad_t + in.pad)) * in.Wp() + (xo - pad_l + in.pad)) * in.Cs;
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
#pragma unroll
          for (int kw = 0; kw < 3; ++kw) {
            const size_t xi = x00 + (size_t)(kh * in.Wp() + kw) * in.Cs;
            const uint2 xh = *reinterpret_cast<const uint2*>(in.hi + xi);
            float x0 = __uint_as_float(xh.x << 16), x1 = __uint_as_float(xh.x & 0xffff0000u), x2 = __uint_as_float(xh.y << 16);
            if (in.lo) {
              const uint2 xl = *reinterpret_cast<const uint2*>(in.lo + xi);
              x0 += __uint_as_float(xl.x << 16); x1 += __uint_as_float(xl.x & 0xffff0000u); x2 += __uint_as_float(xl.y << 16);
            }
            const int k = (kh * 3 + kw) * 3;
            acc[k][0] += x0 * g0; acc[k][1] += x0 * g1;
            acc[k + 1][0] += x1 * g0; acc[k + 1][1] += x1 * g1;
            acc[k + 2][0] += x2 * g0; acc[k + 2][1] += x2 * g1;
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 27; ++k) {
      atomicAdd(&s_acc[k * Cout + 2 * cq], acc[k][0]);
      atomicAdd(&s_acc[k * Cout + 2 * cq + 1], acc[k][1]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 27 * Cout; i += 256) {
    const int k = i / Cout, co = i % Cout;
    atomicAdd(gw + (size_t)co * 27 + k, s_acc[i]);
  }
}

// The optimiser kernels update one parameter span.  KERNEL: a conv / head kernel, whose value and state are HWIO
// [taps][cin][cout] while its gradient is OHWI [cout][taps][cin], and which alone gets the l2 regulariser's gradient 2*l2*w.
// Vector spans (bias, gammas, beta) index all three alike.
__device__ __forceinline__ size_t ohwi_index(size_t i, int taps, int cin, int cout) {
  const int co = (int)(i % cout); const size_t r = i / cout; const int ci = (int)(r % cin); const int t = (int)(r / cin);
  return ((size_t)co * taps + t) * cin + ci;
}

// SGD with momentum (Keras: v = m*v - lr*g; w += v)
template <bool KERNEL>
__global__ void sgd_kernel(float* __restrict__ w, float* __restrict__ v, const float* __restrict__ g, size_t n, int taps, int cin, int cout,
                           float lr, float mom, float l2, float scale) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float nv;
  if constexpr (KERNEL) {
    const float grad = g[ohwi_index(i, taps, cin, cout)] * scale + 2.f * l2 * w[i];
    nv = mom * v[i] - lr * grad;
  } else {
    nv = mom * v[i] - lr * g[i] * scale;
  }
  v[i] = nv;
  w[i] += nv;
}

// Adam (Keras: m = b1*m + (1-b1)*g; v = b2*v + (1-b2)*g^2; w -= lr_t*m / (sqrt(v) + eps))
template <bool KERNEL>
__global__ void adam_kernel(float* __restrict__ w, float* __restrict__ m1, float* __restrict__ m2, const float* __restrict__ g, size_t n, int taps,
                            int cin, int cout, float lr_t, float b1, float b2, float eps, float l2, float scale) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float grad;
  if constexpr (KERNEL) grad = g[ohwi_index(i, taps, cin, cout)] * scale + 2.f * l2 * w[i];
  else grad = g[i] * scale;
  const float a = b1 * m1[i] + (1.f - b1) * grad;
  const float b = b2 * m2[i] + (1.f - b2) * grad * grad;
  m1[i] = a; m2[i] = b;
  w[i] -= lr_t * a / (sqrtf(b) + eps);
}

__global__ void hwio_to_ohwi_kernel(const float* __restrict__ w, int taps, int cin, int cout, float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)taps * cin * cout;
  if (i >= total) return;
  const int ci = (int)(i % cin); const size_t r = i / cin; const int t = (int)(r % taps); const int co = (int)(r / taps);
  out[i] = w[((size_t)t * cin + ci) * cout + co];
}

// ---------------------------------------------------------------------------------------------
// plan
// ---------------------------------------------------------------------------------------------
struct TLayer {
  int cin = 0, cout = 0, taps = 0;          // conv / head kernel shape
  ActBuf g;                                 // gradient of this layer's output (pre-activation); same geometry as the output
  bool has_g = false;
  // data gradient
  bool has_dgrad = false;
  ConvLaunch dgrad{};
  __nv_bfloat16 *w2_hi = nullptr, *w2_lo = nullptr; size_t w2_krow = 0; int w2_kblocks = 0;
  int* dgrad_tiles = nullptr;
  bool dgrad_strided = false;               // stride != 1: col-gradient GEMM (dZ * W^T) + col2im
  int dgrad_relu_mask = 0;                  // col2im zeroes the gradient where the ReLU producer's output is <= 0
  int dgrad_col2im_accumulate = 0;          // col2im adds to a gradient another consumer of the producer already wrote
  float* dcol = nullptr; int dcol_ld = 0;
  // weight gradient
  bool wg_native = false;                   // stride-1 layers: wgrad.cu reads dZ / X in place (no transposed copies)
  WgradLaunch wg;
  std::vector<ConvLaunch> wgrad;            // fallback: one GEMM per tap (or one for the im2col path) on transposed operands
  int Wq = 0;                               // row pitch of the transposed operands' pixel grid
  std::vector<int> wgrad_res;               // tap shift mod 8: TMA needs 16-byte aligned K offsets, so XT is built once per residue
  long long Kv = 0, ldT = 0;
  TMap dy_map{}, x_map{};
};

// One parameter span of the flat gradient buffer.  `which` is ssdk_trainer_param_span's code: 0 conv / head kernel, 1 bias,
// 2 L2Normalization gamma, 3 / 4 BatchNormalization gamma / beta.  `value` is the fp32 parameter the layer plan reads
// (L.w_f32, L.bias, L.gamma, L.bn_gamma, L.bn_beta).
struct ParamSpan {
  int layer = 0, which = 0;
  long long off = 0, count = 0;
  float* value = nullptr;
  int taps = 0, cin = 0, cout = 0;          // kernel spans: the HWIO value is read and written as OHWI; 0: a vector span
};

// wgrad_direct3x3_kernel's conditions: 3x3 undilated taps over 3 input channels, an even cout that fits its shared accumulators, and a
// zero border wide enough that every tap is a constant offset from the window origin
bool direct_fast3(const ssdk_layer_desc& d, const ActBuf& X, int cin, int cout) {
  return d.kh == 3 && d.kw == 3 && d.dilation == 1 && cin == 3 && X.Cs >= 4 && cout % 2 == 0 && cout <= 512 && X.pad >= d.pad_t &&
         X.pad >= d.pad_l && X.pad >= 2 - d.pad_t && X.pad >= 2 - d.pad_l;
}

}  // namespace

struct ssdk_trainer {
  ssdk_model* m = nullptr;
  std::vector<TLayer> tl;
  std::vector<ParamSpan> params;            // the spans of the flat gradient buffer, in its order
  float* grad = nullptr;
  long long n_params = 0;
  // optimiser state in the flat buffer's spans, a kernel's HWIO like its value: [0] SGD velocity / Adam first moment, made with
  // the trainer; [1] Adam second moment, made by the first Adam update
  float* state[2] = {nullptr, nullptr};
  __nv_bfloat16 *xT_hi = nullptr, *xT_lo = nullptr, *dyT_hi = nullptr, *dyT_lo = nullptr;   // scratch, sized for the largest layer
  float* dypred = nullptr;                  // [B*P*(C+12)]
  std::vector<char> written;                // backward pass state: which activations already hold a partial gradient
  std::vector<void*> allocs;
};

namespace {

bool is_conv(int op) { return op == SSDK_OP_CONV || op == SSDK_OP_HEAD; }
// graph sources (preprocessed images, or a caller tensor): no producer, no parameters, no gradient
bool is_source(int op) { return op == SSDK_OP_INPUT || op == SSDK_OP_TENSOR; }

const ParamSpan* find_span(const ssdk_trainer* t, int layer, int which) {
  for (const ParamSpan& p : t->params)
    if (p.layer == layer && p.which == which) return &p;
  return nullptr;
}
// the gradient of a span the layer has
float* span_grad(ssdk_trainer* t, int layer, int which) { return t->grad + find_span(t, layer, which)->off; }

// The bf16 planes of conv layer i from its fp32 master: the forward planes (the image-facing direct kernel reads the master
// itself) and the data-gradient planes
int repack_layer(ssdk_trainer* t, int i, cudaStream_t s) {
  ssdk_model* m = t->m;
  const TLayer& T = t->tl[i];
  const LayerPlan& L = m->layers[i];
  int rc;
  if (!L.direct) {
    rc = launch_repack(m->ctx, L.w_f32, T.taps, T.cin, T.cout, L.im2col ? PACK_FWD_IM2COL : PACK_FWD, L.kblocks, L.w_krow, L.w_hi, L.w_lo, s);
    if (rc) return rc;
  }
  if (T.has_dgrad) {
    rc = launch_repack(m->ctx, L.w_f32, T.taps, T.cin, T.cout, T.dgrad_strided ? PACK_DGRAD_COL : PACK_DGRAD, T.w2_kblocks, T.w2_krow, T.w2_hi,
                       T.w2_lo, s);
    if (rc) return rc;
  }
  return SSDK_OK;
}

// The parameter table in flat-buffer order (per layer: a conv / head's kernel, bias and BatchNormalization gamma / beta, or an
// L2Normalization's gamma), the flat gradient buffer (the caller's, or the trainer's own) and optimiser slot 0.
int plan_params(ssdk_trainer* t, float* flat_grad_dev) {
  ssdk_model* m = t->m;
  long long off = 0;
  auto add = [&](int i, int which, long long count, float* value, int taps = 0, int cin = 0, int cout = 0) {
    t->params.push_back(ParamSpan{i, which, off, count, value, taps, cin, cout});
    off += count;
  };
  for (int i = 0; i < (int)m->layers.size(); ++i) {
    LayerPlan& L = m->layers[i];
    TLayer& T = t->tl[i];
    if (is_conv(L.d.op)) {
      if ((L.d.act == SSDK_ACT_ELU || L.bn_scale) && !L.bn_train) {
        set_error("training: layer %d has an ELU / folded BatchNormalization without the raw BatchNormalization parameters (bn_gamma, ...)", i);
        return SSDK_ERR_UNSUPPORTED;
      }
      T.cin = m->layers[L.d.input].C; T.cout = L.C; T.taps = L.d.kh * L.d.kw;
      add(i, 0, (long long)T.cout * T.taps * T.cin, L.w_f32, T.taps, T.cin, T.cout);
      add(i, 1, T.cout, L.bias);
      if (L.bn_train) { add(i, 3, T.cout, L.bn_gamma); add(i, 4, T.cout, L.bn_beta); }
    } else if (L.d.op == SSDK_OP_L2NORM) {
      add(i, 2, L.C, L.gamma);
    }
  }
  t->n_params = off;
  if (flat_grad_dev) t->grad = flat_grad_dev;
  else { int rc = dev_alloc(t->allocs, &t->grad, (size_t)off, true); if (rc) return rc; }
  return dev_alloc(t->allocs, &t->state[0], (size_t)off, true);
}

// Gradient planes of every layer but the sources, in the geometry of its forward output
int alloc_grad_planes(ssdk_trainer* t) {
  ssdk_model* m = t->m;
  for (int i = 0; i < (int)m->layers.size(); ++i) {
    LayerPlan& L = m->layers[i];
    TLayer& T = t->tl[i];
    if (is_source(L.d.op)) continue;
    ActBuf& g = T.g;
    if (L.d.op == SSDK_OP_HEAD) { g.B = m->B; g.H = L.H; g.W = L.W; g.C = L.C; g.Cs = (L.C + 7) / 8 * 8; g.pad = 1; }
    else { g = L.out; g.hi = nullptr; g.lo = nullptr; }
    const size_t ne = g.elems() + 64 * 8;
    int rc = dev_alloc(t->allocs, &g.hi, ne, true); if (rc) return rc;
    if (m->split) { rc = dev_alloc(t->allocs, &g.lo, ne, true); if (rc) return rc; }
    T.has_g = true;
  }
  return SSDK_OK;
}

// Data-gradient plan of conv layer i into its producer's gradient planes.  written[pi]: the backward pass has already written
// a contribution of another consumer into them when it reaches layer i.
int plan_dgrad(ssdk_trainer* t, int i, std::vector<char>& written) {
  ssdk_model* m = t->m;
  const LayerPlan& L = m->layers[i];
  TLayer& T = t->tl[i];
  const ssdk_layer_desc& d = L.d;
  const int pi = d.input;
  const LayerPlan& PL = m->layers[pi];
  const TLayer& PT = t->tl[pi];
  if (is_source(PL.d.op)) return SSDK_OK;
  if (T.cin % 8 != 0) { set_error("training: input channels must be a multiple of 8 (layer %d)", i); return SSDK_ERR_UNSUPPORTED; }
  const int relu_mask = (PL.d.op == SSDK_OP_CONV && PL.d.act == SSDK_ACT_RELU) ? 1 : 0;
  T.has_dgrad = true;
  T.dgrad_strided = d.stride != 1;
  T.w2_kblocks = (T.g.Cs + 63) / 64;
  ConvGeom gg;
  gg.in = &T.g; gg.B = m->B;
  int rows, rc;                               // rows of the packed planes
  if (T.dgrad_strided) {
    // dCol[M][taps*cin] = dZ[M][cout] * W^T, then col2im
    rows = T.dcol_ld = T.taps * T.cin;
    T.w2_krow = (size_t)T.w2_kblocks * 64;
    rc = dev_alloc(t->allocs, &T.dcol, (size_t)m->B * L.H * L.W * T.dcol_ld, true); if (rc) return rc;
    gg.Ho = L.H; gg.Wo = L.W; gg.cout = T.dcol_ld;
  } else {
    rows = T.cin;
    T.w2_krow = (size_t)T.taps * T.w2_kblocks * 64;
    gg.kh = d.kh; gg.kw = d.kw; gg.dilation = d.dilation;
    gg.pad_t = d.dilation * (d.kh - 1) - d.pad_t; gg.pad_l = d.dilation * (d.kw - 1) - d.pad_l;
    gg.Ho = PL.H; gg.Wo = PL.W; gg.cout = T.cin;
  }
  rc = dev_alloc(t->allocs, &T.w2_hi, (size_t)rows * T.w2_krow, true); if (rc) return rc;
  if (m->split) { rc = dev_alloc(t->allocs, &T.w2_lo, (size_t)rows * T.w2_krow, true); if (rc) return rc; }
  rc = plan_conv_gemm(m, T.dgrad, gg, T.w2_hi, T.w2_lo, T.w2_krow, T.w2_kblocks, &T.dgrad_tiles);
  if (rc) return rc;
  ConvArgs& a = T.dgrad.args;
  a.bias = nullptr; a.act = SSDK_ACT_NONE;
  if (T.dgrad_strided) {
    a.epi = EPI_F32; a.out_f32 = T.dcol;
    T.dgrad_relu_mask = relu_mask;
    T.dgrad_col2im_accumulate = written[pi];
  } else {
    a.epi = EPI_SPLIT;
    a.out_hi = PT.g.hi; a.out_lo = PT.g.lo; a.out_Hp = PT.g.Hp(); a.out_Wp = PT.g.Wp(); a.out_pad = PT.g.pad; a.out_Cs = PT.g.Cs;
    a.mask_hi = relu_mask ? PL.out.hi : nullptr;
    a.accumulate = written[pi];
  }
  written[pi] = 1;
  return SSDK_OK;
}

// Weight-gradient plan of conv layer i: wgrad.cu's GEMM on dZ / X in place, or the geometry of the transposed operands (their
// GEMMs are planned by plan_transposed_gemms once the shared scratch is sized).  Direct layers need none.
int plan_wgrad_layer(ssdk_trainer* t, int i, long long& max_xT, long long& max_dyT) {
  ssdk_model* m = t->m;
  const LayerPlan& L = m->layers[i];
  TLayer& T = t->tl[i];
  const ssdk_layer_desc& d = L.d;
  if (L.direct) return SSDK_OK;               // handled by wgrad_direct_kernel
  const ActBuf& X = m->layers[d.input].out;
  if (!L.im2col && !getenv("SSDK_WGRAD_TRANSPOSED") && wgrad_supported(X, T.g, d.kh, d.kw, d.stride, d.dilation)) {
    T.wg_native = true;
    return plan_wgrad(m->ctx, T.wg, X, T.g, L.H, L.W, d.kh, d.kw, d.dilation, d.pad_t, d.pad_l, m->split, span_grad(t, i, 0));
  }
  if (L.im2col) {
    T.Kv = (long long)m->B * L.H * L.W;
    T.ldT = (T.Kv + 7) / 8 * 8 + 64;
    T.dy_map = TMap{0, L.H * L.W, L.W, L.H, L.W, T.g.Hp(), T.g.Wp(), T.g.pad};
    T.x_map = TMap{1, 0, 0, 0, 0, 0, 0, 0};
    max_xT = std::max(max_xT, (long long)L.Kpad * T.ldT);
  } else {
    // the GEMM's pixel axis runs over X's padded grid with the row pitch rounded up to 8 elements: tap shifts are then
    // kh*Wq + kw (+ const) and only the kw part can break TMA's 16-byte alignment -> one XT copy per distinct kw residue
    const int Wq = (X.Wp() + 7) / 8 * 8;
    T.Wq = Wq;
    T.Kv = (long long)m->B * X.Hp() * Wq;
    T.ldT = (T.Kv + 7) / 8 * 8 + 64;
    T.dy_map = TMap{0, X.Hp() * Wq, Wq, L.H, L.W, T.g.Hp(), T.g.Wp(), T.g.pad};
    T.x_map = TMap{0, X.Hp() * Wq, Wq, X.Hp(), X.Wp(), X.Hp(), X.Wp(), 0};
    max_xT = std::max(max_xT, (long long)X.Cs * T.ldT);
  }
  max_dyT = std::max(max_dyT, (long long)T.g.Cs * T.ldT);
  return SSDK_OK;
}

// The weight-gradient GEMMs of the transposed path (one per tap, or one for an im2col layer) on the shared scratch
int plan_transposed_gemms(ssdk_trainer* t) {
  ssdk_model* m = t->m;
  for (int i = 0; i < (int)m->layers.size(); ++i) {
    const LayerPlan& L = m->layers[i];
    TLayer& T = t->tl[i];
    if (!is_conv(L.d.op) || L.direct || T.wg_native) continue;
    const ssdk_layer_desc& d = L.d;
    const ActBuf& X = m->layers[d.input].out;
    const int n_gemm = L.im2col ? 1 : T.taps;
    const int ncols = L.im2col ? L.Kpad : T.cin;            // N of the GEMM
    const int kblocks = (int)((T.Kv + 63) / 64);
    T.wgrad.resize(n_gemm); T.wgrad_res.assign(n_gemm, 0);
    for (int tp = 0; tp < n_gemm; ++tp) {
      ConvGeom wg;
      wg.a_hi = t->dyT_hi; wg.a_lo = t->dyT_lo; wg.a_inner = (uint64_t)T.ldT; wg.a_ld = (uint64_t)T.ldT; wg.a_rows = (uint64_t)T.cout;
      wg.Ho = T.cout; wg.Wo = 1; wg.B = 1; wg.cout = ncols;
      ConvLaunch& cl = T.wgrad[tp];
      // the transposed operands are [channels][ldT] with zeros in [Kv, ldT)
      int rc = plan_conv_gemm(m, cl, wg, t->xT_hi, t->xT_lo, (size_t)T.ldT, kblocks, nullptr);
      if (rc) return rc;
      ConvArgs& a = cl.args;
      a.epi = EPI_ATOMIC; a.bias = nullptr; a.act = SSDK_ACT_NONE;
      a.out_f32 = span_grad(t, i, 0);
      if (L.im2col) { a.out_ld = T.taps * T.cin; a.out_col_off = 0; a.b_k_offset = 0; a.cout = T.taps * T.cin; a.n_tiles_n = (a.cout + a.BN - 1) / a.BN; }
      else {
        const int kh = tp / d.kw, kw = tp % d.kw;
        a.out_ld = T.taps * T.cin; a.out_col_off = tp * T.cin;
        const int shift = (kh * d.dilation - d.pad_t + X.pad) * T.Wq + (kw * d.dilation - d.pad_l + X.pad);
        T.wgrad_res[tp] = shift & 7;                 // XT_r[c][v] = X[v + r][c], read at the aligned offset shift - r
        a.b_k_offset = shift - (shift & 7);
      }
      const int units = a.n_tiles_m * a.n_tiles_n;
      int ks = std::max(1, (4 * m->ctx->sm_count + units - 1) / units);
      ks = std::min(ks, kblocks);
      a.kb_per = (kblocks + ks - 1) / ks;
      a.k_split = (kblocks + a.kb_per - 1) / a.kb_per;
      cl.grid = std::max(1, std::min(units * a.k_split, m->ctx->sm_count));
    }
  }
  return SSDK_OK;
}

// Everything ssdk_trainer_create makes; on failure the caller destroys the partly made trainer
int plan_trainer(ssdk_trainer* t, float* flat_grad_dev) {
  ssdk_model* m = t->m;
  const int n = (int)m->layers.size();
  t->tl.resize(n);
  int rc = plan_params(t, flat_grad_dev); if (rc) return rc;
  rc = dev_alloc(t->allocs, &t->dypred, (size_t)m->B * m->P * (m->Ctot + 12), true); if (rc) return rc;
  rc = alloc_grad_planes(t); if (rc) return rc;
  // in the backward pass's order: does the producer's gradient buffer already hold a contribution?
  std::vector<char> written(n, 0);
  long long max_xT = 0, max_dyT = 0;
  for (int i = n - 1; i >= 0; --i) {
    const ssdk_layer_desc& d = m->layers[i].d;
    if (is_source(d.op)) continue;
    if (!is_conv(d.op)) { if (!is_source(m->layers[d.input].d.op)) written[d.input] = 1; continue; }
    rc = plan_dgrad(t, i, written); if (rc) return rc;
    rc = plan_wgrad_layer(t, i, max_xT, max_dyT); if (rc) return rc;
  }
  rc = dev_alloc(t->allocs, &t->xT_hi, (size_t)max_xT + 4096, true); if (rc) return rc;
  rc = dev_alloc(t->allocs, &t->dyT_hi, (size_t)max_dyT + 4096, true); if (rc) return rc;
  if (m->split) {
    rc = dev_alloc(t->allocs, &t->xT_lo, (size_t)max_xT + 4096, true); if (rc) return rc;
    rc = dev_alloc(t->allocs, &t->dyT_lo, (size_t)max_dyT + 4096, true); if (rc) return rc;
  }
  rc = plan_transposed_gemms(t); if (rc) return rc;
  for (int i = 0; i < n; ++i)
    if (is_conv(m->layers[i].d.op)) { rc = repack_layer(t, i, 0); if (rc) return rc; }
  SSDK_CHECK_CUDA(cudaDeviceSynchronize());
  return SSDK_OK;
}

}  // namespace

extern "C" int ssdk_trainer_create(ssdk_model* m, float* flat_grad_dev, ssdk_trainer** out) {
  SSDK_REQUIRE(m && out, "ssdk_trainer_create: NULL argument");
  SSDK_REQUIRE(m->training, "ssdk_trainer_create: the model plan was not created with training=1");
  SSDK_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  ssdk_trainer* t = new ssdk_trainer();
  t->m = m;
  const int rc = plan_trainer(t, flat_grad_dev);
  if (rc) { ssdk_trainer_destroy(t); return rc; }
  *out = t;
  return SSDK_OK;
}

extern "C" int ssdk_trainer_destroy(ssdk_trainer* t) {
  if (!t) return SSDK_OK;
  for (void* p : t->allocs) cudaFree(p);
  delete t;
  return SSDK_OK;
}

extern "C" int ssdk_trainer_num_params(const ssdk_trainer* t, long long* out_n) {
  SSDK_REQUIRE(t && out_n, "ssdk_trainer_num_params: NULL argument");
  *out_n = t->n_params;
  return SSDK_OK;
}

extern "C" int ssdk_trainer_param_span(const ssdk_trainer* t, int layer, int which, long long* out_offset, long long* out_count) {
  SSDK_REQUIRE(t && out_offset && out_count && layer >= 0 && layer < (int)t->tl.size(), "ssdk_trainer_param_span: bad argument");
  const ParamSpan* p = find_span(t, layer, which);
  *out_offset = p ? p->off : -1; *out_count = p ? p->count : 0;
  return SSDK_OK;
}

extern "C" float* ssdk_trainer_grad_buffer(ssdk_trainer* t) { return t ? t->grad : nullptr; }

extern "C" int ssdk_trainer_grad_shape(const ssdk_trainer* t, int layer, int* out_hp, int* out_wp, int* out_cs, int* out_pad) {
  SSDK_REQUIRE(t && out_hp && out_wp && out_cs && out_pad && layer >= 0 && layer < (int)t->tl.size(), "ssdk_trainer_grad_shape: bad argument");
  const TLayer& T = t->tl[layer];
  SSDK_REQUIRE(T.has_g, "ssdk_trainer_grad_shape: layer %d has no gradient planes", layer);
  *out_hp = T.g.Hp(); *out_wp = T.g.Wp(); *out_cs = T.g.Cs; *out_pad = T.g.pad;
  return SSDK_OK;
}

extern "C" int ssdk_trainer_read_grad(ssdk_trainer* t, int layer, float* out_dev, void* stream) {
  SSDK_REQUIRE(t && out_dev && layer >= 0 && layer < (int)t->tl.size(), "ssdk_trainer_read_grad: bad argument");
  const TLayer& T = t->tl[layer];
  SSDK_REQUIRE(T.has_g, "ssdk_trainer_read_grad: layer %d has no gradient planes", layer);
  return launch_unpack(t->m->ctx, T.g, out_dev, (cudaStream_t)stream);
}

extern "C" int ssdk_trainer_read_grad_planes(ssdk_trainer* t, int layer, uint16_t* hi_dev, uint16_t* lo_dev, void* stream) {
  SSDK_REQUIRE(t && hi_dev && layer >= 0 && layer < (int)t->tl.size(), "ssdk_trainer_read_grad_planes: bad argument");
  const TLayer& T = t->tl[layer];
  SSDK_REQUIRE(T.has_g, "ssdk_trainer_read_grad_planes: layer %d has no gradient planes", layer);
  const size_t bytes = T.g.elems() * sizeof(uint16_t);
  cudaStream_t s = (cudaStream_t)stream;
  SSDK_CHECK_CUDA(cudaMemcpyAsync(hi_dev, T.g.hi, bytes, cudaMemcpyDeviceToDevice, s));
  if (lo_dev && T.g.lo) SSDK_CHECK_CUDA(cudaMemcpyAsync(lo_dev, T.g.lo, bytes, cudaMemcpyDeviceToDevice, s));
  return SSDK_OK;
}

extern "C" int ssdk_trainer_layer_plan(const ssdk_trainer* t, int layer, ssdk_backward_plan* out) {
  SSDK_REQUIRE(t && out && layer >= 0 && layer < (int)t->tl.size(), "ssdk_trainer_layer_plan: bad argument");
  memset(out, 0, sizeof(*out));
  const TLayer& T = t->tl[layer];
  const LayerPlan& L = t->m->layers[layer];
  if (!is_conv(L.d.op)) return SSDK_OK;
  if (T.has_dgrad) {
    const ConvArgs& a = T.dgrad.args;
    out->dgrad = T.dgrad_strided ? SSDK_DGRAD_STRIDED : SSDK_DGRAD_GEMM;
    out->dgrad_bn = a.BN;
    out->dgrad_mask = T.dgrad_strided ? T.dgrad_relu_mask : (a.mask_hi != nullptr);
    out->dgrad_accumulate = T.dgrad_strided ? T.dgrad_col2im_accumulate : a.accumulate;
    out->dgrad_n_tiles_m = a.n_tiles_m; out->dgrad_n_tiles_n = a.n_tiles_n; out->dgrad_grid = T.dgrad.grid;
  }
  if (L.direct) {
    out->wgrad = SSDK_WGRAD_DIRECT;
    out->direct_fast = direct_fast3(L.d, t->m->layers[L.d.input].out, T.cin, T.cout) ? 1 : 0;
    return SSDK_OK;
  }
  if (T.wg_native) {
    const WgradArgs& w = T.wg.args;
    out->wgrad = SSDK_WGRAD_NATIVE;
    out->wgrad_bn = w.BNc; out->a_boxes = w.a_boxes; out->bw = w.bw; out->bh = w.bh;
    out->co_tiles = w.co_tiles; out->ci_tiles = w.ci_tiles; out->k_split = w.k_split > 1 ? w.k_split : 1;
    out->stages = w.stages; out->grid = T.wg.grid; out->kv = w.total_patches;
    return SSDK_OK;
  }
  if (T.wgrad.empty()) return SSDK_OK;
  const ConvLaunch& c = T.wgrad[0];
  out->wgrad = L.im2col ? SSDK_WGRAD_IM2COL : SSDK_WGRAD_TRANSPOSED;
  out->wgrad_bn = c.args.BN; out->k_split = c.args.k_split > 1 ? c.args.k_split : 1;
  out->n_gemms = (int)T.wgrad.size(); out->stages = c.args.stages; out->grid = c.grid; out->kv = (int)T.Kv;
  return SSDK_OK;
}

namespace {

int do_transpose(ssdk_trainer* t, const __nv_bfloat16* hi, const __nv_bfloat16* lo, int src_ld, long long src_rows, const TMap& mp,
                 long long Kv, int C, __nv_bfloat16* dhi, __nv_bfloat16* dlo, long long ldT, cudaStream_t s, long long row_off = 0) {
  dim3 grid((unsigned)((ldT + 63) / 64), (unsigned)((C + 63) / 64));
  transpose_kernel<<<grid, 256, 0, s>>>(hi, lo, src_ld, src_rows, mp, row_off, Kv, C, dhi, dlo, ldT);
  SSDK_COUNT_LAUNCH(t->m->ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

}  // namespace

namespace {
int backward_layers(ssdk_trainer* t, const float* dypred, int hi, int lo, cudaStream_t s);
}

// Loss (optional) and d loss / d y_pred from one launch of the fused loss kernel; clears the gradient buffer.
extern "C" int ssdk_train_backward_begin(ssdk_trainer* t, const float* y_true, const float* y_pred, int neg_pos_ratio, int n_neg_min,
                                         float alpha, float* out_loss, void* stream_) {
  SSDK_REQUIRE(t && y_true && y_pred, "ssdk_train_backward_begin: NULL argument");
  ssdk_model* m = t->m;
  ssdk_ctx* ctx = m->ctx;
  int rc;
  SSDK_CHECK_CUDA(cudaMemsetAsync(t->grad, 0, (size_t)t->n_params * sizeof(float), (cudaStream_t)stream_));
  if (out_loss) rc = ssdk_ssd_loss_fwd_bwd(ctx, y_true, y_pred, m->B, m->P, m->Ctot, neg_pos_ratio, n_neg_min, alpha, nullptr, out_loss, nullptr, t->dypred, stream_);
  else rc = ssdk_ssd_loss_bwd(ctx, y_true, y_pred, m->B, m->P, m->Ctot, neg_pos_ratio, n_neg_min, alpha, nullptr, t->dypred, stream_);
  return rc;
}

// The backward pass of layers hi, hi-1, ..., lo (graph indices; a full pass is n_layers-1 .. 0 in one or several calls, top
// down).  When it returns (stream order), the parameter gradients of exactly these layers are final -- their span of the
// flat buffer can be all-reduced while the lower layers are still being differentiated.  dypred_dev NULL: the gradient
// ssdk_train_backward_begin left in the trainer; otherwise d loss / d y_pred provided by the caller (the buffer is cleared
// when the pass starts at the top layer).
extern "C" int ssdk_train_backward_layers(ssdk_trainer* t, const float* dypred_dev, int hi, int lo, void* stream_) {
  SSDK_REQUIRE(t, "ssdk_train_backward_layers: NULL trainer");
  const int n = (int)t->m->layers.size();
  SSDK_REQUIRE(hi < n && lo >= 0 && lo <= hi, "ssdk_train_backward_layers: bad layer range [%d, %d] of %d layers", lo, hi, n);
  if (dypred_dev && hi == n - 1) SSDK_CHECK_CUDA(cudaMemsetAsync(t->grad, 0, (size_t)t->n_params * sizeof(float), (cudaStream_t)stream_));
  return backward_layers(t, dypred_dev ? dypred_dev : t->dypred, hi, lo, (cudaStream_t)stream_);
}

extern "C" int ssdk_train_backward(ssdk_trainer* t, const float* y_true, const float* y_pred, int neg_pos_ratio, int n_neg_min,
                                   float alpha, float* out_loss, void* stream_) {
  int rc = ssdk_train_backward_begin(t, y_true, y_pred, neg_pos_ratio, n_neg_min, alpha, out_loss, stream_);
  if (rc) return rc;
  return backward_layers(t, t->dypred, (int)t->m->layers.size() - 1, 0, (cudaStream_t)stream_);
}

extern "C" int ssdk_train_backward_dy(ssdk_trainer* t, const float* dypred_dev, void* stream_) {
  SSDK_REQUIRE(t && dypred_dev, "ssdk_train_backward_dy: NULL argument");
  return ssdk_train_backward_layers(t, dypred_dev, (int)t->m->layers.size() - 1, 0, stream_);
}

namespace {

// parameter gradients of layers hi .. lo from d loss / d y_pred (B,P,C+12), walking the layers in reverse
int backward_layers(ssdk_trainer* t, const float* dypred, int hi, int lo, cudaStream_t s) {
  ssdk_model* m = t->m;
  ssdk_ctx* ctx = m->ctx;
  int rc;
  const int n = (int)m->layers.size();
  if (hi == n - 1) t->written.assign(n, 0);
  SSDK_REQUIRE((int)t->written.size() == n, "ssdk_train_backward_layers: a pass must start at the top layer");
  std::vector<char>& written = t->written;
  for (int i = hi; i >= lo; --i) {
    LayerPlan& L = m->layers[i];
    TLayer& T = t->tl[i];
    const ssdk_layer_desc& d = L.d;
    if (is_source(d.op)) continue;
    const int pi = d.input;
    LayerPlan& PL = m->layers[pi];
    TLayer& PT = t->tl[pi];
    const bool prod_needs_grad = !is_source(PL.d.op);
    const int relu_mask = (PL.d.op == SSDK_OP_CONV && PL.d.act == SSDK_ACT_RELU) ? 1 : 0;
    if (d.op == SSDK_OP_HEAD) {
      const size_t total = (size_t)m->B * L.H * L.W * d.n_boxes;
      head_bwd_kernel<<<(unsigned)((total + 7) / 8), 256, 0, s>>>(L.head_f32, dypred, m->B, L.H, L.W, d.n_boxes, m->Ctot, m->P, L.prior_off, T.g);
      SSDK_COUNT_LAUNCH(ctx);
    }
    if (d.op == SSDK_OP_MAXPOOL) {
      if (prod_needs_grad) {
        if (PL.out.C % 8) { set_error("training: max-pool channels must be a multiple of 8"); return SSDK_ERR_UNSUPPORTED; }
        const size_t total = (size_t)PL.out.B * PL.out.H * PL.out.W * (PL.out.C / 8);
        pool_bwd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(PL.out, T.g, PT.g, L.H, L.W, d.kh, d.kw, d.stride, d.pad_t, d.pad_l,
                                                                         relu_mask, written[pi] ? 1 : 0);
        SSDK_COUNT_LAUNCH(ctx);
        written[pi] = 1;
      }
      continue;
    }
    if (d.op == SSDK_OP_L2NORM) {
      if (prod_needs_grad) {
        const size_t total = (size_t)PL.out.B * PL.out.H * PL.out.W;
        l2norm_bwd_kernel<<<(unsigned)((total + 7) / 8), 256, 0, s>>>(PL.out, T.g, PT.g, L.gamma, span_grad(t, i, 2), relu_mask, written[pi] ? 1 : 0);
        SSDK_COUNT_LAUNCH(ctx);
        written[pi] = 1;
      }
      continue;
    }
    // ---- conv + BatchNormalization + activation: the gradient planes hold d loss / d activation; turn them into the gradient of
    //      the raw conv output (and produce dgamma / dbeta) before the conv's own gradients are formed
    if (L.bn_train) { rc = launch_bn_backward(ctx, L, d.act, T.g, span_grad(t, i, 3), span_grad(t, i, 4), s); if (rc) return rc; }
    // ---- convolution / head: weight + bias gradients
    if (L.direct) {
      const int K = T.taps * T.cin;
      const size_t smem = (size_t)K * T.cout * sizeof(float);
      // the plan admits direct layers whose fp32 [K][Cout] accumulator needs up to 96 KB (model.cu, as conv_direct_kernel)
      static bool attr_set = false;
      if (!attr_set) {
        SSDK_CHECK_CUDA(cudaFuncSetAttribute(wgrad_direct_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        SSDK_CHECK_CUDA(cudaFuncSetAttribute(wgrad_direct3x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        attr_set = true;
      }
      const int total_rows = T.g.B * T.g.H;
      const int rpb = std::max(1, (total_rows + 8 * ctx->sm_count - 1) / (8 * ctx->sm_count));
      const bool fast3 = direct_fast3(d, PL.out, T.cin, T.cout);
      if (fast3) wgrad_direct3x3_kernel<<<(unsigned)((total_rows + rpb - 1) / rpb), 256, smem, s>>>(PL.out, T.g, span_grad(t, i, 0), d.pad_t, d.pad_l, rpb);
      else wgrad_direct_kernel<<<(unsigned)((total_rows + rpb - 1) / rpb), 256, smem, s>>>(PL.out, T.g, span_grad(t, i, 0), d.kh, d.kw, d.dilation, d.pad_t, d.pad_l, rpb);
      SSDK_COUNT_LAUNCH(ctx);
      rc = launch_bias_grad(ctx, T.g, span_grad(t, i, 1), s); if (rc) return rc;
    } else if (T.wg_native) {
      rc = launch_wgrad(ctx, T.wg, s); if (rc) return rc;
      rc = launch_bias_grad(ctx, T.g, span_grad(t, i, 1), s); if (rc) return rc;
    } else {
      // transposed operands
      rc = do_transpose(t, T.g.hi, T.g.lo, T.g.Cs, (long long)T.g.rows(), T.dy_map, T.Kv, T.cout, t->dyT_hi, t->dyT_lo, T.ldT, s); if (rc) return rc;
      if (L.im2col) {
        rc = do_transpose(t, L.col_hi, L.col_lo, L.Kpad, T.Kv, T.x_map, T.Kv, L.Kpad, t->xT_hi, t->xT_lo, T.ldT, s); if (rc) return rc;
        rc = launch_conv(ctx, T.wgrad[0], s); if (rc) return rc;
      } else {
        for (int r = 0; r < 8; ++r) {
          bool any = false;
          for (size_t tp = 0; tp < T.wgrad.size(); ++tp) any |= (T.wgrad_res[tp] == r);
          if (!any) continue;
          rc = do_transpose(t, PL.out.hi, PL.out.lo, PL.out.Cs, (long long)PL.out.rows(), T.x_map, T.Kv, T.cin, t->xT_hi, t->xT_lo, T.ldT, s, r);
          if (rc) return rc;
          for (size_t tp = 0; tp < T.wgrad.size(); ++tp)
            if (T.wgrad_res[tp] == r) { rc = launch_conv(ctx, T.wgrad[tp], s); if (rc) return rc; }
        }
      }
      dim3 gr(64, T.cout);
      rowsum_kernel<<<gr, 256, 0, s>>>(t->dyT_hi, t->dyT_lo, T.ldT, T.Kv, span_grad(t, i, 1));
      SSDK_COUNT_LAUNCH(ctx);
    }
    // ---- data gradient
    if (T.has_dgrad && T.dgrad_strided) {
      rc = launch_conv(ctx, T.dgrad, s); if (rc) return rc;
      const size_t total = (size_t)PT.g.B * PT.g.H * PT.g.W * PT.g.C;
      col2im_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(T.dcol, L.H, L.W, d.kh, d.kw, d.stride, d.dilation, d.pad_t, d.pad_l, T.dcol_ld,
                                                                     PL.out, PT.g, T.dgrad_relu_mask, written[pi] ? 1 : 0);
      SSDK_COUNT_LAUNCH(ctx);
      written[pi] = 1;
    } else if (T.has_dgrad) {
      T.dgrad.args.accumulate = written[pi] ? 1 : 0;
      rc = launch_conv(ctx, T.dgrad, s); if (rc) return rc;
      written[pi] = 1;
    }
  }
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

// the spans of a conv / head layer end at span k: its bf16 planes can be re-packed from the updated master
bool ends_conv_layer(const ssdk_trainer* t, size_t k) {
  const int li = t->params[k].layer;
  return is_conv(t->m->layers[li].d.op) && (k + 1 == t->params.size() || t->params[k + 1].layer != li);
}

// span p of `src` (its value, or its optimiser state) into out_dev, in the gradient's layout
int read_span(ssdk_trainer* t, const ParamSpan& p, const float* src, float* out_dev, cudaStream_t s) {
  if (p.taps) {
    hwio_to_ohwi_kernel<<<(unsigned)((p.count + 255) / 256), 256, 0, s>>>(src, p.taps, p.cin, p.cout, out_dev + p.off);
    SSDK_COUNT_LAUNCH(t->m->ctx);
  } else {
    SSDK_CHECK_CUDA(cudaMemcpyAsync(out_dev + p.off, src, (size_t)p.count * sizeof(float), cudaMemcpyDeviceToDevice, s));
  }
  return SSDK_OK;
}

}  // namespace

extern "C" int ssdk_train_apply(ssdk_trainer* t, float lr, float momentum, float l2_reg, float grad_scale, void* stream_) {
  SSDK_REQUIRE(t, "ssdk_train_apply: NULL trainer");
  cudaStream_t s = (cudaStream_t)stream_;
  for (size_t k = 0; k < t->params.size(); ++k) {
    const ParamSpan& p = t->params[k];
    const auto sgd = p.taps ? sgd_kernel<true> : sgd_kernel<false>;
    sgd<<<(unsigned)((p.count + 255) / 256), 256, 0, s>>>(p.value, t->state[0] + p.off, t->grad + p.off, (size_t)p.count, p.taps, p.cin, p.cout,
                                                           lr, momentum, l2_reg, grad_scale);
    SSDK_COUNT_LAUNCH(t->m->ctx);
    if (ends_conv_layer(t, k)) { const int rc = repack_layer(t, p.layer, s); if (rc) return rc; }
  }
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

extern "C" int ssdk_train_apply_adam(ssdk_trainer* t, float lr, float beta1, float beta2, float eps, float l2_reg, float grad_scale, int step,
                                     void* stream_) {
  SSDK_REQUIRE(t && step >= 1, "ssdk_train_apply_adam: bad argument");
  cudaStream_t s = (cudaStream_t)stream_;
  // Keras: lr_t = lr * sqrt(1 - beta_2^t) / (1 - beta_1^t)
  const float lr_t = lr * (float)(std::sqrt(1.0 - std::pow((double)beta2, (double)step)) / (1.0 - std::pow((double)beta1, (double)step)));
  if (!t->state[1]) { const int rc = dev_alloc(t->allocs, &t->state[1], (size_t)t->n_params, true); if (rc) return rc; }
  for (size_t k = 0; k < t->params.size(); ++k) {
    const ParamSpan& p = t->params[k];
    const auto adam = p.taps ? adam_kernel<true> : adam_kernel<false>;
    adam<<<(unsigned)((p.count + 255) / 256), 256, 0, s>>>(p.value, t->state[0] + p.off, t->state[1] + p.off, t->grad + p.off, (size_t)p.count,
                                                            p.taps, p.cin, p.cout, lr_t, beta1, beta2, eps, l2_reg, grad_scale);
    SSDK_COUNT_LAUNCH(t->m->ctx);
    if (ends_conv_layer(t, k)) { const int rc = repack_layer(t, p.layer, s); if (rc) return rc; }
  }
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

extern "C" int ssdk_trainer_read_opt_state(ssdk_trainer* t, int slot, float* out_dev, void* stream_) {
  SSDK_REQUIRE(t && out_dev, "ssdk_trainer_read_opt_state: NULL argument");
  SSDK_REQUIRE((slot == 0 || slot == 1) && t->state[slot],
               "ssdk_trainer_read_opt_state: slot %d does not exist (0: SGD velocity / Adam first moment, 1: Adam second moment, "
               "after an Adam update)", slot);
  for (const ParamSpan& p : t->params) {
    const int rc = read_span(t, p, t->state[slot] + p.off, out_dev, (cudaStream_t)stream_);
    if (rc) return rc;
  }
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

extern "C" int ssdk_trainer_read_bn_stats(ssdk_trainer* t, int layer, float* mean_dev, float* var_dev, void* stream_) {
  SSDK_REQUIRE(t && mean_dev && var_dev && layer >= 0 && layer < (int)t->tl.size(), "ssdk_trainer_read_bn_stats: bad argument");
  LayerPlan& L = t->m->layers[layer];
  SSDK_REQUIRE(L.bn_train, "ssdk_trainer_read_bn_stats: layer %d has no BatchNormalization", layer);
  SSDK_CHECK_CUDA(cudaMemcpyAsync(mean_dev, L.bn_mmean, (size_t)L.C * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream_));
  SSDK_CHECK_CUDA(cudaMemcpyAsync(var_dev, L.bn_mvar, (size_t)L.C * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream_));
  return SSDK_OK;
}

extern "C" int ssdk_trainer_read_bn_input(ssdk_trainer* t, int layer, float* out_dev, void* stream_) {
  SSDK_REQUIRE(t && out_dev && layer >= 0 && layer < (int)t->tl.size(), "ssdk_trainer_read_bn_input: bad argument");
  LayerPlan& L = t->m->layers[layer];
  SSDK_REQUIRE(L.bn_train, "ssdk_trainer_read_bn_input: layer %d has no BatchNormalization", layer);
  return launch_unpack(t->m->ctx, L.z, out_dev, (cudaStream_t)stream_);
}

extern "C" int ssdk_trainer_read_params(ssdk_trainer* t, float* out_dev, void* stream_) {
  SSDK_REQUIRE(t && out_dev, "ssdk_trainer_read_params: NULL argument");
  for (const ParamSpan& p : t->params) {
    const int rc = read_span(t, p, p.value, out_dev, (cudaStream_t)stream_);
    if (rc) return rc;
  }
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}
