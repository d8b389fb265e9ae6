// Internal interface between model.cu (plan building) and conv.cu (kernels).
#pragma once
#include "common.cuh"
#include <cuda.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <vector>

namespace ssdk {

// An activation tensor: NHWC, channel-padded to a multiple of 8, spatially padded with a zero border
// of `pad` pixels, stored as TWO bf16 planes: value = hi + lo (lo is absent in single-pass bf16 mode).
// hi + lo carries 16 significant bits, which keeps the tensor-core path within ~1e-5 of an fp32 conv.
struct ActBuf {
  __nv_bfloat16* hi = nullptr;
  __nv_bfloat16* lo = nullptr;
  int B = 0, H = 0, W = 0, C = 0;   // logical shape
  int Cs = 0;                        // stored channels (multiple of 8)
  int pad = 0;
  // shared = 1 (inference plans): the row pitch is W + pad, not W + 2*pad -- the right border of a row IS the left border of the
  // next one (the same zeros).  Every index stays ((n*Hp + y + pad)*Wp + x + pad)*Cs; a tap that runs off the right edge lands
  // in the next row's left border.  The implicit GEMM computes every position of the stored grid, so this cuts its padding rows:
  // fc6 (19 wide, border 6) goes from 61 % to 76 % valid rows, the 19-wide conv5_x from 90 % to 95 %.
  int shared = 0;
  __host__ __device__ int Hp() const { return H + 2 * pad; }
  __host__ __device__ int Wp() const { return W + (shared ? pad : 2 * pad); }
  size_t rows() const { return (size_t)B * Hp() * Wp(); }
  size_t elems() const { return rows() * Cs; }
};

// The hi + lo plane format of activations, gradients and packed weights: hi = bf16(v), lo = bf16(v - hi), both rounded to nearest
// even; lo is a null plane in single-pass bf16 mode.  The helpers below are the only code that rounds values into the format or
// reads them back (max-pooling, transposes and gathers move raw 16-bit halves).  They contain no multiply-add, so the per-file
// --fmad settings cannot change their results.
inline uint16_t f2bf(float f) {                  // host: round-to-nearest-even float -> bf16; a NaN stays a (quiet) NaN
  uint32_t u; memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
inline float bf2f(uint16_t h) { uint32_t u = (uint32_t)h << 16; float f; memcpy(&f, &u, 4); return f; }

#ifdef __CUDACC__
// element index of channel 0 of pixel (n, y, x) in a zero-bordered NHWC plane
__device__ __forceinline__ size_t act_index(const ActBuf& a, int n, int y, int x) {
  return (((size_t)n * a.Hp() + (y + a.pad)) * a.Wp() + (x + a.pad)) * a.Cs;
}
// one element: hi, plus lo when that plane exists
__device__ __forceinline__ float split_load(const __nv_bfloat16* hi, const __nv_bfloat16* lo, size_t i) {
  float v = __bfloat162float(hi[i]);
  if (lo) v += __bfloat162float(lo[i]);
  return v;
}
__device__ __forceinline__ void split_store(__nv_bfloat16* hi, __nv_bfloat16* lo, size_t i, float v) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[i] = h;
  if (lo) lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
}
// 8 channels = one 16-byte word per plane: a word of one plane -> 8 values, and 8 values -> the hi and lo words
__device__ __forceinline__ void unpack8(uint4 w, float (&v)[8]) {
  const uint32_t u[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) { v[2 * j] = __uint_as_float(u[j] << 16); v[2 * j + 1] = __uint_as_float(u[j] & 0xffff0000u); }
}
__device__ __forceinline__ void pack8(const float (&v)[8], uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const __nv_bfloat162 hh = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
    h[j] = *reinterpret_cast<const uint32_t*>(&hh);
    const __nv_bfloat162 ll = __floats2bfloat162_rn(v[2 * j] - __uint_as_float(h[j] << 16), v[2 * j + 1] - __uint_as_float(h[j] & 0xffff0000u));
    l[j] = *reinterpret_cast<const uint32_t*>(&ll);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}
// v = hi + lo of 8 channels (a missing lo plane reads as a zero word); `i` is a multiple of 8
__device__ __forceinline__ void split_load8(const __nv_bfloat16* hi, const __nv_bfloat16* lo, size_t i, float (&v)[8]) {
  float l[8];
  unpack8(*reinterpret_cast<const uint4*>(hi + i), v);
  if (lo) unpack8(*reinterpret_cast<const uint4*>(lo + i), l);
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] += lo ? l[e] : 0.f;
}
__device__ __forceinline__ void split_store8(__nv_bfloat16* hi, __nv_bfloat16* lo, size_t i, const float (&v)[8]) {
  uint4 h, l;
  pack8(v, h, l);
  *reinterpret_cast<uint4*>(hi + i) = h;
  if (lo) *reinterpret_cast<uint4*>(lo + i) = l;
}
__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == SSDK_ACT_RELU) return fmaxf(x, 0.f);
  if (act == SSDK_ACT_ELU) return x > 0.f ? x : expm1f(x);
  return x;
}
// the same on 8 values with one branch on `act`, not one per value
__device__ __forceinline__ void apply_act8(float (&v)[8], int act) {
  if (act == SSDK_ACT_RELU) {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = apply_act(v[e], SSDK_ACT_RELU);
  } else if (act == SSDK_ACT_ELU) {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = apply_act(v[e], SSDK_ACT_ELU);
  }
}
#endif

enum { EPI_SPLIT = 0, EPI_F32 = 1, EPI_ATOMIC = 2, EPI_HEAD = 3 };

constexpr int kMaxTaps = 25;

struct ConvArgs {
  // GEMM view
  int M_total;          // virtual rows (B * rows_per_img)
  int rows_per_img;     // rows of the virtual grid per image
  int in_Wp;            // virtual row pitch
  int Ho, Wo, B;        // valid extent: virtual (y, x) is a real output iff y < Ho && x < Wo
  int KH, KW, kblocks;  // K loop = KH * KW taps x kblocks channel blocks of 64
  int row_shift[8];     // row offset of tap (kh, kw=0)
  int kw_rows;          // rows between consecutive kw taps (= dilation)
  int stages;           // TMA ring depth
  int n_tiles_m;        // number of entries in tile_list
  int n_tiles_n;
  const int* tile_list; // m-tile indices that contain at least one valid row
  int BN;               // accumulator tile width (64/128/160/256: the wgmma N); TMA box rows of the weight tile
  int cout;
  int split;            // 1: bf16x3 (hi*hi + hi*lo + lo*hi), 0: single bf16 pass
  int acc_split;        // 1 (always with split): the cross terms accumulate apart from hi*hi and are added after the K loop
  // epilogue
  int epi;
  const float* bias; const float* bn_scale; const float* bn_shift;
  int act;
  __nv_bfloat16* out_hi; __nv_bfloat16* out_lo;
  int out_Hp, out_Wp, out_pad, out_Cs;
  float* out_f32;       // EPI_F32: compact [B*Ho*Wo][cout]; EPI_ATOMIC: atomicAdd into out_f32[row*out_ld + out_col_off + col]
  // --- extensions used by the backward pass ---
  int k_split;          // >1: the K loop (KH == KW == 1 only) is cut into k_split ranges, one work unit each (EPI_ATOMIC)
  int kb_per;           // k-blocks per range
  int b_k_offset;       // added to the K coordinate of the weight-side operand (row-shifted taps of a transposed tensor)
  int out_ld, out_col_off;
  const __nv_bfloat16* mask_hi;   // EPI_SPLIT: zero the result where this plane (same geometry as the output) is <= 0 (ReLU')
  int accumulate;       // EPI_SPLIT: add to the value already stored in the output planes
  // --- EPI_HEAD: Reshape / softmax / Concat of models/keras_ssd300.py:363-419 in the predictor conv's epilogue.  The tile's columns
  //     are n_boxes x [C class logits | 4 offsets]; every (pixel, box) becomes one row of y_pred (out_f32):
  //     [softmax(C) | 4 offsets | 4 anchor coordinates | 4 variances] at prior head_prior_off + pixel * n_boxes + box.
  int head_nb, head_C, head_P, head_prior_off;
  const float* head_anchors;      // [P*4]
  float head_var[4];
};

struct ConvLaunch {
  CUtensorMap a_hi, a_lo, b_hi, b_lo;
  ConvArgs args;
  int grid;
  size_t smem;
  double flops_algo, flops_issued;
};

int tma_init();   // resolves cuTensorMapEncodeTiled through the runtime (no link-time libcuda dependency)
int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t rows, uint64_t row_stride_bytes,
                 uint32_t box_inner, uint32_t box_rows);
// 4-D map over a bf16 NHWC tensor, dims / box innermost first (channels, x, y, image); 128B swizzle, zero fill
int make_tmap_4d(CUtensorMap* out, const void* base, const uint64_t dims[4], const uint32_t box[4]);
size_t conv_smem_bytes(const ConvArgs& a);
void conv_pick_stages(ConvArgs& a);
int launch_conv(ssdk_ctx* ctx, const ConvLaunch& L, cudaStream_t stream, int grid_cap = 0);   // grid_cap > 0: at most that many CTAs

// elementwise / data movement kernels
int launch_preprocess(ssdk_ctx* ctx, const float* images, int B, int H, int W, int Cimg, const float* mean, const float* stddev,
                      const int* swap, const ActBuf& out, cudaStream_t stream);
// im2col8_kernel (8 channels per thread) applies when the input holds a multiple of 8 channels unpadded and the column planes are
// 16-byte aligned; decided once when the plan is built, launch_im2col runs the recorded choice
bool im2col_vec8_ok(const ActBuf& in, int Kpad, const void* out_hi, const void* out_lo);
int launch_im2col(ssdk_ctx* ctx, const ActBuf& in, __nv_bfloat16* out_hi, __nv_bfloat16* out_lo, int Ho, int Wo, int kh, int kw,
                  int stride, int dil, int pad_t, int pad_l, int Kpad, bool vec8, cudaStream_t stream);
int launch_conv_direct(ssdk_ctx* ctx, const ActBuf& in, const ActBuf& out, const float* w, const float* bias, const float* bn_scale,
                       const float* bn_shift, int act, int kh, int kw, int dil, int pad_t, int pad_l, cudaStream_t stream);
// image-facing layer on the tensor cores (gathered A tile, weights resident in shared memory as a swizzled image)
int first_tc_supported(int taps, int cin, int cout);
int first_bn(int cout);     // weight-image rows (wgmma N) of the image-facing layer
// launch shape of conv_first_kernel, chosen when the plan is built
struct FirstPlan { int BN = 0, kblocks = 0, n_tiles = 0, grid = 0; };
FirstPlan first_plan(const ActBuf& out, int kh, int kw, int sm_count);
bool first_border_ok(const ActBuf& in, int kh, int kw, int dil, int pad_t, int pad_l);
void first_weight_image(const float* hwio, int taps, int cin, int cout, int BN, int kblocks, std::vector<uint16_t>& hi, std::vector<uint16_t>& lo);
int launch_conv_first(ssdk_ctx* ctx, const FirstPlan& fp, const ActBuf& in, const ActBuf& out, const __nv_bfloat16* w_hi, const __nv_bfloat16* w_lo,
                      const float* bias, const float* bn_scale, const float* bn_shift, int act, int kh, int kw, int dil, int pad_t,
                      int pad_l, cudaStream_t stream);
int launch_maxpool(ssdk_ctx* ctx, const ActBuf& in, const ActBuf& out, int kh, int kw, int stride, int pad_t, int pad_l,
                   cudaStream_t stream);
int launch_l2norm(ssdk_ctx* ctx, const ActBuf& in, const ActBuf& out, const float* gamma, cudaStream_t stream);
int launch_head_finalize(ssdk_ctx* ctx, const float* head, int B, int HW, int n_boxes, int C, int P, int prior_off,
                         const float* anchors, const float* variances, float* y_pred, cudaStream_t stream);
int launch_unpack(ssdk_ctx* ctx, const ActBuf& in, float* out, cudaStream_t stream);
int launch_pack(ssdk_ctx* ctx, const float* in, const ActBuf& out, cudaStream_t stream);      // float32 NHWC -> hi/lo planes (interior only)

}  // namespace ssdk
