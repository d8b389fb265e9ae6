// Structures shared by model.cu (forward plan) and train.cu (backward plan / optimiser).
#pragma once
#include "conv.cuh"
#include <vector>
#include <algorithm>
#include <cmath>
#include <cstdlib>

namespace ssdk {

struct LayerPlan {
  ssdk_layer_desc d{};
  int H = 0, W = 0, C = 0;            // logical output shape
  int in_H = 0, in_W = 0, in_C = 0;
  ActBuf out;                         // INPUT / CONV / MAXPOOL / L2NORM
  bool im2col = false;
  bool direct = false;                // fp32 SIMT path for the image-facing conv (Cin < 8)
  bool first_tc = false;           // direct layer of an inference plan on the tensor cores (conv_first_kernel)
  FirstPlan first;                    // its launch shape (first_tc)
  bool im2col_vec8 = false;           // im2col path: im2col8_kernel rather than im2col_kernel
  float* w_f32 = nullptr;
  int Kpad = 0;
  __nv_bfloat16* col_hi = nullptr; __nv_bfloat16* col_lo = nullptr;
  __nv_bfloat16* w_hi = nullptr; __nv_bfloat16* w_lo = nullptr;
  size_t w_krow = 0;                  // elements per output-channel row of the packed weights
  int kblocks = 0;
  float* bias = nullptr; float* bn_scale = nullptr; float* bn_shift = nullptr; float* gamma = nullptr;
  int* tile_list = nullptr;
  ConvLaunch launch{};
  float* head_f32 = nullptr;
  bool head_fused = false;            // softmax / concat / anchors done in the conv epilogue (inference plans)
  int prior_off = 0;
  int need_pad = 0;                   // border required by the consumers of this layer's output
  float mean[3] = {0, 0, 0}, stddev[3] = {1, 1, 1}; int swap[3] = {0, 1, 2};
  bool has_mean = false, has_std = false, has_swap = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  // BatchNormalization in Keras' training phase (training plans of conv + BN graphs)
  bool bn_train = false;
  ActBuf z;                           // conv output before the normalisation (bias added)
  float *bn_gamma = nullptr, *bn_beta = nullptr, *bn_mmean = nullptr, *bn_mvar = nullptr;   // [C] parameters and moving statistics
  float *bn_bmean = nullptr, *bn_brstd = nullptr;                                           // [C] batch statistics of the last forward
  double* bn_acc = nullptr;           // [2*C] reduction scratch
  float bn_eps = 1e-3f, bn_momentum = 0.99f;
};

}  // namespace ssdk

struct ssdk_model {
  ssdk_ctx* ctx = nullptr;
  int B = 0, H = 0, W = 0, Cimg = 0, Ctot = 0, P = 0, split = 1;
  int training = 0;                   // activation borders sized for the backward pass, fp32 master kernels kept on the device
  std::vector<ssdk::LayerPlan> layers;
  float* d_anchors = nullptr;
  float var[4] = {0, 0, 0, 0};
  double flops_algo = 0, flops_issued = 0;
  int timing = 0;
  std::vector<void*> allocs;
  // two-stream schedule of inference plans (model.cu, plan_overlap): the narrow tail of the trunk and the narrow predictor
  // heads run on `side` while the wide predictor heads run on the caller's stream with a capped grid
  cudaStream_t side = nullptr;
  std::vector<uint8_t> on_side;       // per layer: 1 = issued on `side`
  std::vector<cudaEvent_t> dep_ev;    // cross-stream dependencies (one per layer is enough) + join
  int grid_cap = 0;                   // grid limit of the conv launches that stay on the caller's stream while `side` is busy
  int overlap_from = -1;              // first layer issued on `side` (-1: single-stream plan)
  std::vector<int> issue_pos;         // scratch of ssdk_model_forward: issue position of every layer on its stream
};

namespace ssdk {

// Device memory owned by a model or a trainer: `allocs` is its owner's list, freed when the owner is destroyed.
template <typename T>
inline int dev_alloc(std::vector<void*>& allocs, T** out, size_t count, bool zero) {
  void* p = nullptr;
  size_t bytes = count * sizeof(T);
  if (bytes == 0) bytes = 16;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e)); return SSDK_ERR_NOMEM; }
  allocs.push_back(p);
  if (zero) { e = cudaMemset(p, 0, bytes); if (e != cudaSuccess) { set_error("cudaMemset failed: %s", cudaGetErrorString(e)); return SSDK_ERR_CUDA; } }
  *out = reinterpret_cast<T*>(p);
  return SSDK_OK;
}

inline int upload_f32(ssdk_model* m, float** out, const float* host, size_t n) {
  int rc = dev_alloc(m->allocs, out, n, false);
  if (rc) return rc;
  SSDK_CHECK_CUDA(cudaMemcpy(*out, host, n * sizeof(float), cudaMemcpyHostToDevice));
  return SSDK_OK;
}

inline int alloc_act(ssdk_model* m, ActBuf& a, int B, int H, int W, int C, int pad) {
  a.B = B; a.H = H; a.W = W; a.C = C; a.Cs = (C + 7) / 8 * 8; a.pad = pad;
  a.shared = 0;
  if (!m->training && pad > 0) { const char* e = getenv("SSDK_SHARED_BORDER"); a.shared = e ? (atoi(e) ? 1 : 0) : 1; }
  // slack: TMA boxes may start on the last rows; with a shared border the last row's right border lies behind the last image
  size_t n = a.elems() + std::max<size_t>(64 * 8, (size_t)(pad + 1) * a.Cs);
  int rc = dev_alloc(m->allocs, &a.hi, n, true);
  if (rc) return rc;
  if (m->split) { rc = dev_alloc(m->allocs, &a.lo, n, true); if (rc) return rc; }
  return SSDK_OK;
}

// Conv GEMM plan shared by the forward and backward builders (defined in model.cu).
struct ConvGeom {
  const ActBuf* in = nullptr;           // virtual path: the zero-bordered input tensor
  const __nv_bfloat16* a_hi = nullptr;  // explicit-matrix path: A [rows][a_inner]
  const __nv_bfloat16* a_lo = nullptr;
  uint64_t a_inner = 0, a_rows = 0;
  uint64_t a_ld = 0;                    // row stride in elements (0: a_inner)
  int kh = 1, kw = 1, dilation = 1, pad_t = 0, pad_l = 0;
  int Ho = 0, Wo = 0, B = 0;
  int cout = 0;
};
// BatchNormalization (training phase) + activation: z -> out with batch statistics; and its backward on the gradient planes
int launch_bn_forward(ssdk_ctx* ctx, LayerPlan& L, int act, cudaStream_t s);
int launch_bn_backward(ssdk_ctx* ctx, LayerPlan& L, int act, const ActBuf& g, float* dgamma, float* dbeta, cudaStream_t s);

int plan_conv_gemm(ssdk_model* m, ConvLaunch& cl, const ConvGeom& g, const __nv_bfloat16* w_hi, const __nv_bfloat16* w_lo,
                   size_t krow, int kblocks, int** tile_list_out);

// Layouts of the packed K-major bf16 hi / lo weight planes, all made on the device from the fp32 HWIO master [taps][cin][cout]
// (defined in model.cu).  Every row is zero-padded to `krow` elements.
enum WeightLayout {
  PACK_FWD,          // forward, implicit GEMM: [cout][tap][kblocks * 64 over cin]
  PACK_FWD_IM2COL,   // forward, im2col GEMM: [cout][k = tap * cin + c]
  PACK_DGRAD,        // data gradient: the kernel rotated by 180 degrees, in / out swapped: [cin][taps - 1 - tap][kblocks * 64 over cout]
  PACK_DGRAD_COL,    // col-gradient GEMM of a strided convolution, W^T: [k = tap * cin + c][cout]
};
int launch_repack(ssdk_ctx* ctx, const float* w, int taps, int cin, int cout, WeightLayout layout, int kblocks, size_t krow,
                  __nv_bfloat16* hi, __nv_bfloat16* lo, cudaStream_t s);

}  // namespace ssdk
