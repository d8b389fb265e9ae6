// Correctly rounded arithmetic by type, for the code that restates the reference's float32 / float64 expressions operation by
// operation.  These are intrinsics: they never contract into an FMA, whatever --fmad the including file is compiled with.
#pragma once
#include <cuda_runtime.h>

namespace ssdk {

__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float rint_rn(float v) { return rintf(v); }     // to the nearest integer, half to even (np.round)
__device__ __forceinline__ double rint_rn(double v) { return rint(v); }

}  // namespace ssdk
