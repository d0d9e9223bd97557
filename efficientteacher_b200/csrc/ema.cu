// ema.cu -- fused multi-tensor EMA (K15).  Replaces the 518x2 tiny ATen launches per update of
// ModelEMA.update / SemiSupModelEMA.update / CosineEMA.update (reference utils/torch_utils.py:328-338,
// 364-375, 405-416).  HBM-bound streaming kernel: algorithmic bytes = 12 B/element (single EMA) or
// 20 B/element (fused EMA + EMA-of-EMA: read v,m,s ; write v,s).
#include "common.cuh"

// v <- fl(fl(v*d) + fl(omd*m)) : the torch CPU path does `v *= d` then `v += (1-d)*m`, each op rounding once
// in fp32 with the python scalars rounded to fp32 first (SURVEY.md D9, probed bit-exact).
__device__ __forceinline__ float ema1(float v, float m, float d, float omd) {
  return __fadd_rn(__fmul_rn(v, d), __fmul_rn(omd, m));
}

// one block per EtbChunk {v, m, s or NULL, unused}; hyper = {d, 1-d, d2, 1-d2} in device memory, so a captured CUDA
// graph replays with the decays the host wrote there last
__global__ void __launch_bounds__(256) ema_kernel(const EtbChunk* __restrict__ tab, const float* __restrict__ hyper) {
  const float d = hyper[0], omd = hyper[1], d2 = hyper[2], omd2 = hyper[3];
  const EtbChunk c = tab[blockIdx.x];
  float* __restrict__ v = c.t[0];
  const float* __restrict__ m = c.t[1];
  float* __restrict__ s = c.t[2];
  const int n = c.n;
  const bool vec = ((((uintptr_t)v) | ((uintptr_t)m) | ((uintptr_t)s)) & 15u) == 0;
  if (vec) {
    const int n4 = n >> 2;
    float4* v4 = reinterpret_cast<float4*>(v);
    const float4* m4 = reinterpret_cast<const float4*>(m);
    float4* s4 = reinterpret_cast<float4*>(s);
    // ETB_CHUNK/4 = 1024 float4 per chunk, 256 threads -> 4 independent 16 B loads per stream in flight
    float4 a[4], b[4], e[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      int i = threadIdx.x + k * 256;
      if (i < n4) {
        a[k] = v4[i];
        b[k] = __ldg(m4 + i);
        if (s) e[k] = s4[i];
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      int i = threadIdx.x + k * 256;
      if (i < n4) {
        float4 r;
        r.x = ema1(a[k].x, b[k].x, d, omd);
        r.y = ema1(a[k].y, b[k].y, d, omd);
        r.z = ema1(a[k].z, b[k].z, d, omd);
        r.w = ema1(a[k].w, b[k].w, d, omd);
        v4[i] = r;
        if (s) {
          float4 q;
          q.x = ema1(e[k].x, r.x, d2, omd2);
          q.y = ema1(e[k].y, r.y, d2, omd2);
          q.z = ema1(e[k].z, r.z, d2, omd2);
          q.w = ema1(e[k].w, r.w, d2, omd2);
          s4[i] = q;
        }
      }
    }
    for (int i = (n4 << 2) + threadIdx.x; i < n; i += 256) {
      float r = ema1(v[i], m[i], d, omd);
      v[i] = r;
      if (s) s[i] = ema1(s[i], r, d2, omd2);
    }
  } else {
    for (int i = threadIdx.x; i < n; i += 256) {
      float r = ema1(v[i], m[i], d, omd);
      v[i] = r;
      if (s) s[i] = ema1(s[i], r, d2, omd2);
    }
  }
}

extern "C" int etb_ema_update(const EtbChunk* table_dev, int64_t n_chunks, const float* hyper_dev, void* stream) {
  ETB_CHECK_ARG(table_dev && hyper_dev && n_chunks >= 0 && n_chunks < (1ll << 31));
  if (n_chunks == 0) return ETB_OK;
  etb_launch(ema_kernel, dim3((unsigned)n_chunks), dim3(256), 0, (cudaStream_t)stream, table_dev, hyper_dev);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
