// common.cuh -- shared helpers for libetb200 (sm_90a).  Compiled with --fmad=false: every fused
// multiply-add in this library is an explicit fmaf()/__fmaf_rn so the bit-exact kernels (EMA, assigner,
// NMS) reproduce the two-rounding arithmetic of the reference's CPU fp32 path.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include "../../include/etb200.h"

void etb_set_error(const char* fmt, ...);
void etb_count_launch();   // every ETB_CHECK_LAUNCH() follows exactly one kernel launch of this library

#define ETB_CHECK_ARG(cond)                                                   \
  do {                                                                        \
    if (!(cond)) {                                                            \
      etb_set_error("%s:%d: invalid argument: %s", __FILE__, __LINE__, #cond); \
      return ETB_ERR_INVALID;                                                 \
    }                                                                         \
  } while (0)

#define ETB_CHECK_LAUNCH()                                                               \
  do {                                                                                   \
    cudaError_t e__ = cudaGetLastError();                                                \
    if (e__ != cudaSuccess) {                                                            \
      etb_set_error("%s:%d: CUDA launch failed: %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
      return ETB_ERR_CUDA;                                                               \
    }                                                                                    \
    etb_count_launch();                                                                  \
  } while (0)

#define ETB_CHECK_CUDA(call)                                                             \
  do {                                                                                   \
    cudaError_t e__ = (call);                                                            \
    if (e__ != cudaSuccess) {                                                            \
      etb_set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
      return ETB_ERR_CUDA;                                                               \
    }                                                                                    \
  } while (0)

// The library's one launch helper: arguments are converted to the kernel's parameter types, as a <<<>>> launch would.
template <typename... KP, typename... A>
static inline void etb_launch(void (*kernel)(KP...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cfg.numAttrs = 0;
  (void)cudaLaunchKernelEx(&cfg, kernel, static_cast<KP>(args)...);    // the caller checks cudaGetLastError() (ETB_CHECK_LAUNCH)
}

static inline int etb_num_sms() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
      sms = 132;   // H100 SXM
  }
  return sms;
}

// `act` codes of the BatchNorm kernels (bn.cu) and of the folded-BN conv epilogue (conv_wgmma.cu): 0 none, 1 SiLU,
// 2 ReLU, 4 Hardswish.  3 is not used: older documentation of etb_conv_dgrad gave it the meaning "accumulate into dx".

// nn.Hardswish, as torch computes it on the CPU: z * min(max(z + 3, 0), 6) / 6
__device__ __forceinline__ float hswish_f(float z) { return z * fminf(fmaxf(z + 3.0f, 0.0f), 6.0f) / 6.0f; }
// its derivative as torch's hardswish_backward takes it: 0 for z <= -3, z/3 + 1/2 strictly between -3 and 3, 1 for z >= 3
__device__ __forceinline__ float dhswish_f(float z) { return z <= -3.0f ? 0.0f : (z < 3.0f ? z / 3.0f + 0.5f : 1.0f); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide exclusive scan of one int per thread (blockDim.x <= 1024, multiple of 32).
// Returns the exclusive prefix; *total receives the block sum.  smem: int[33].
__device__ __forceinline__ int block_excl_scan(int v, int* smem, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  __syncthreads();  // protect smem reuse across calls
  if (lane == 31) smem[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    int w = lane < nw ? smem[lane] : 0;
    int winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    smem[lane] = winc - w;  // exclusive warp offsets
    if (lane == 31) smem[32] = winc;
  }
  __syncthreads();
  *total = smem[32];
  return smem[wid] + inc - v;
}
