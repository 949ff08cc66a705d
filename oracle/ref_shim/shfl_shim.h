// oracle/ref_shim/shfl_shim.h -- force-included when compiling the reference's reduce.cu for
// sm_90a: the file predates __shfl_*_sync (reduce.cu:96-130,193-206,719-720 call __shfl_down).
// TEST INFRASTRUCTURE ONLY.
#pragma once
#if defined(__CUDACC__) && defined(__CUDA_ARCH__) && __CUDA_ARCH__ >= 700
__device__ __forceinline__ float __shfl_down(float v, int d, int w = 32) { return __shfl_down_sync(0xffffffffu, v, d, w); }
__device__ __forceinline__ int __shfl_down(int v, int d, int w = 32) { return __shfl_down_sync(0xffffffffu, v, d, w); }
#endif
