// Shared host/device helpers for libssdk.so (H100 / sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cctype>
#include <cerrno>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <atomic>
#include <initializer_list>
#include <map>
#include <mutex>
#include <utility>
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

// Pinned staging for host -> device uploads that must not wait for the stream: N buffers used in turn, each with an event
// recorded after the copy issued from it, so the host runs up to N uploads ahead of the device before it waits for a buffer.
template <int N>
struct HostRing {
  struct Slot { void* ptr = nullptr; size_t bytes = 0; cudaEvent_t done = nullptr; } slot[N];
  int next = 0;

  // Copies the concatenation of `parts` (host pointer, bytes) to dst_dev on `stream`.
  int upload(void* dst_dev, cudaStream_t stream, std::initializer_list<std::pair<const void*, size_t>> parts) {
    size_t bytes = 0;
    for (const auto& p : parts) bytes += p.second;
    Slot& s = slot[next];
    if (!s.done) SSDK_CHECK_CUDA(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
    else SSDK_CHECK_CUDA(cudaEventSynchronize(s.done));
    if (s.bytes < bytes) {
      if (s.ptr) cudaFreeHost(s.ptr);
      s.ptr = nullptr; s.bytes = 0;
      const size_t want = std::max(bytes, (size_t)16384);
      SSDK_CHECK_CUDA(cudaHostAlloc(&s.ptr, want, cudaHostAllocDefault));
      s.bytes = want;
    }
    unsigned char* h = static_cast<unsigned char*>(s.ptr);
    for (const auto& p : parts) { if (p.second) std::memcpy(h, p.first, p.second); h += p.second; }
    SSDK_CHECK_CUDA(cudaMemcpyAsync(dst_dev, s.ptr, bytes, cudaMemcpyHostToDevice, stream));
    SSDK_CHECK_CUDA(cudaEventRecord(s.done, stream));
    next = (next + 1) % N;
    return SSDK_OK;
  }

  void release() {
    for (Slot& s : slot) {
      if (s.done) { cudaEventSynchronize(s.done); cudaEventDestroy(s.done); }
      if (s.ptr) cudaFreeHost(s.ptr);
      s = Slot{};
    }
  }
};

}  // namespace ssdk

struct ssdk_ctx {
  int device = 0;
  int sm_count = 132;
  int64_t launches = 0;         // kernels launched through ssdk::launch
  // grow-only device workspaces, one per user
  ssdk::Scratch decode_ws;      // ssdk_decode: decoded boxes, scores, labels and its NMS scratch
  ssdk::Scratch nms_ws;         // ssdk_nms
  ssdk::Scratch loss_ws;        // the SSD loss
  long long loss_ws_shape = -1; // (B, P) the loss workspace is laid out for
  int loss_parity = 0;          // which of its two histogram sets the next loss call uses (the other one is being cleared)
  ssdk::Scratch focal_ws;       // the focal loss: its count, ticket and tile partials
  ssdk::Scratch box_ws;         // ssdk_assemble_batch: transformed boxes and per-image counts
  cudaEvent_t box_ws_done = nullptr;  // recorded after the last ssdk_assemble_batch: box_ws is free once it has completed
  ssdk::Scratch img_desc_ws;    // ssdk_assemble_images: per-image and photometric descriptors
  ssdk::Scratch photo_ws;       // ssdk_assemble_images: images after the photometric pre-pass
  cudaDeviceProp prop{};
  ssdk::HostRing<4> img_desc_ring;   // pinned staging of img_desc_ws
};

namespace ssdk {

// Raises `kernel`'s dynamic shared-memory limit on ctx->device to at least `bytes`; up to 48 KB every kernel may use without it.
// The limit belongs to the kernel in one device's context, so the level set is kept per (kernel, device), behind a lock since
// contexts are per (device, thread).
inline int allow_smem(const ssdk_ctx* ctx, const void* kernel, size_t bytes) {
  if (bytes <= 48 * 1024) return SSDK_OK;
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, size_t> limit;
  std::lock_guard<std::mutex> lock(mu);
  size_t& have = limit[{kernel, ctx->device}];
  if (bytes <= have) return SSDK_OK;
  SSDK_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  have = bytes;
  return SSDK_OK;
}

// Environment switches.  These are the only environment variables the library reads, and env_int is the only place that reads
// them.  They let the tests reach on small inputs the paths the defaults take only on large ones (each selects between paths
// that the tests hold to the same reference), or report what the encoder's matching stage did; none is needed in normal use.
//
//   switch                 default             read at                 selects
//   SSDK_ENC_SPATIAL_MIN   24                  each ssdk_encode        the spatial tile set once the batch's largest image has
//                                                                      this many boxes
//   SSDK_ENC_LB_MIN        17                  each ssdk_encode        enc_lb_kernel's lower bounds from the same count on
//   SSDK_ENC_TPC           1 ... 8 by boxes    each ssdk_encode        tiles per CTA (at least 1; halved while the grid has
//                                                                      fewer than 8 CTAs per SM)
//   SSDK_ENC_COUNTERS      0                   each ssdk_encode        1: print the conflict loop's event counts to stderr
//                                                                      (synchronises the stream)
//   SSDK_NMS_TWO_STAGE     1                   each ssdk_decode / nms  0: always the full multi-band NMS scan
//   SSDK_SHARED_BORDER     1                   model plan creation     0: inference activations keep one border per image
//   SSDK_NO_HEAD_FUSION    0                   model plan creation     1: inference heads write fp32 logits, head_finalize_kernel
//                                                                      finishes them
//   SSDK_OVERLAP           1                   model plan creation     0: inference plans run on one stream
//   SSDK_OVERLAP_R         sm_count / 3 + 1    model plan creation     the grid up to which a launch counts as narrow
//   SSDK_WGRAD_TRANSPOSED  0                   trainer creation        1: weight gradients on transposed copies, never in place
//
// *out = the switch's value: `def` when it is unset or empty, the value of a whole decimal integer, and anything else is refused
// as SSDK_ERR_INVALID under the variable's name.
inline int env_int(const char* name, int def, int* out) {
  const char* s = getenv(name);
  *out = def;
  if (!s || !*s) return SSDK_OK;
  char* end = nullptr;
  errno = 0;
  const long v = strtol(s, &end, 10);
  SSDK_REQUIRE((isdigit((unsigned char)s[0]) || s[0] == '-' || s[0] == '+') && *end == '\0' && errno == 0 && v >= INT_MIN &&
               v <= INT_MAX, "%s=\"%s\" is not an integer", name, s);
  *out = (int)v;
  return SSDK_OK;
}

// Counts a launch in ctx->launches and reports its error (`e`, else the thread's last CUDA error) by the kernel's name.
inline int launched(ssdk_ctx* ctx, const void* kernel, cudaError_t e) {
  const cudaError_t last = cudaGetLastError();   // also clears the error a failed launch leaves behind
  if (e == cudaSuccess) e = last;
  ctx->launches++;
  if (e == cudaSuccess) return SSDK_OK;
  const char* name = nullptr;
  if (cudaFuncGetName(&name, kernel) != cudaSuccess || !name) name = "<unknown kernel>";
  set_error("launch of %s failed: %s", name, cudaGetErrorString(e));
  return SSDK_ERR_CUDA;
}

// Every kernel of the library is launched here: kernel<<<grid, block, smem, stream>>>(args...), with the shared-memory limit
// raised as far as smem needs, the launch counted and its error returned as SSDK_ERR_CUDA.
template <typename... Ps, typename... As>
int launch(ssdk_ctx* ctx, void (*kernel)(Ps...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, As&&... args) {
  if (int rc = allow_smem(ctx, (const void*)kernel, smem)) return rc;
  kernel<<<grid, block, smem, stream>>>(std::forward<As>(args)...);
  return launched(ctx, (const void*)kernel, cudaSuccess);
}

// The same as one cooperative grid: all blocks resident at once, so the kernel may synchronise the whole grid.
template <typename... Ps, typename... As>
int launch_cooperative(ssdk_ctx* ctx, void (*kernel)(Ps...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, As&&... args) {
  if (int rc = allow_smem(ctx, (const void*)kernel, smem)) return rc;
  cudaLaunchAttribute coop{};
  coop.id = cudaLaunchAttributeCooperative;
  coop.val.cooperative = 1;
  const cudaLaunchConfig_t cfg = {grid, block, smem, stream, &coop, 1};
  return launched(ctx, (const void*)kernel, cudaLaunchKernelEx(&cfg, kernel, std::forward<As>(args)...));
}

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
