// Shared host/device helpers for libssdk.so (H100 / sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include <cstring>
#include <atomic>
#include <vector>
#include <string>
#include "../../include/ssdk.h"

namespace ssdk {

void set_error(const char* fmt, ...);

#define SSDK_CHECK_CUDA(expr)                                                                   \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) {                                                                    \
      ::ssdk::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return SSDK_ERR_CUDA;                                                                     \
    }                                                                                           \
  } while (0)

#define SSDK_REQUIRE(cond, ...)                                                                 \
  do {                                                                                          \
    if (!(cond)) {                                                                              \
      ::ssdk::set_error(__VA_ARGS__);                                                           \
      return SSDK_ERR_INVALID;                                                                  \
    }                                                                                           \
  } while (0)

// A grow-only device scratch buffer.
struct Scratch {
  void* ptr = nullptr;
  size_t bytes = 0;
  int ensure(size_t need) {
    if (need <= bytes) return SSDK_OK;
    if (ptr) cudaFree(ptr);
    ptr = nullptr; bytes = 0;
    size_t want = need + need / 4 + 256;
    cudaError_t e = cudaMalloc(&ptr, want);
    if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e)); return SSDK_ERR_NOMEM; }
    bytes = want;
    return SSDK_OK;
  }
  void release() { if (ptr) cudaFree(ptr); ptr = nullptr; bytes = 0; }
};

}  // namespace ssdk

struct ssdk_ctx {
  int device = 0;
  int sm_count = 132;
  int64_t launches = 0;
  ssdk::Scratch ws[5];          // decode / loss / nms / box assembly / image descriptor workspaces
  long long loss_ws_shape = -1; // (B, P) the loss workspace is laid out for
  int loss_parity = 0;          // which of its two histogram sets the next loss call uses (the other one is being cleared)
  cudaDeviceProp prop{};
  // Pinned staging for the per-image descriptors of ssdk_assemble_images: a ring of buffers, each with an event recorded after
  // its upload, so that the host can run up to kImgStages calls ahead of the device before a buffer has to be waited for.
  static constexpr int kImgStages = 4;
  struct HostStage { void* ptr = nullptr; size_t bytes = 0; cudaEvent_t done = nullptr; } img_stage[kImgStages];
  int img_stage_next = 0;
};

#define SSDK_COUNT_LAUNCH(ctx) do { (ctx)->launches++; } while (0)

namespace ssdk {

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline long long ceil_div_ll(long long a, long long b) { return (a + b - 1) / b; }

#ifdef __CUDACC__
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
#endif

}  // namespace ssdk
