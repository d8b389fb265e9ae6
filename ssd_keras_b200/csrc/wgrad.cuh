// Interface of the wgmma weight-gradient kernel (wgrad.cu) used by train.cu.
#pragma once
#include "conv.cuh"

namespace ssdk {

struct WgradArgs {
  int KH, KW, dil, split;
  int cin, cout, taps;
  int BNc;                 // input channels per tile (64 or 128: the wgmma N)
  int ci_tiles, co_tiles, a_boxes;
  int bw, bh;              // pixel patch of one K-block (bw * bh = 64)
  int px_tiles, py_tiles, total_patches;
  int g_pad, x_off, y_off; // TMA coordinates: dZ box at (x0 + g_pad, y0 + g_pad), X box at (x0 + kw*dil + x_off, y0 + kh*dil + y_off)
  uint32_t tx_bytes;       // bytes one stage's TMA loads deliver
  int stages;
  int k_split, patches_per_split;
  float* dw;               // [cout][taps][cin] fp32, accumulated with atomics
};

struct WgradLaunch {
  CUtensorMap g_hi, g_lo, x_hi, x_lo;
  WgradArgs args;
  int grid = 0;
  size_t smem = 0;
  double flops = 0;
};

bool wgrad_supported(const ActBuf& X, const ActBuf& G, int kh, int kw, int stride, int dil);
int plan_wgrad(ssdk_ctx* ctx, WgradLaunch& L, const ActBuf& X, const ActBuf& G, int Ho, int Wo, int KH, int KW, int dil, int pad_t, int pad_l,
               int split, float* dw);
int launch_wgrad(ssdk_ctx* ctx, const WgradLaunch& L, cudaStream_t stream);
int launch_bias_grad(ssdk_ctx* ctx, const ActBuf& G, float* gb, cudaStream_t stream);

}  // namespace ssdk
