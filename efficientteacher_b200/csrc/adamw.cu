// adamw.cu -- fused multi-tensor AdamW step: replaces torch.optim.AdamW's foreach kernels and the separate gradient zeroing
// behind `scaler.step(optimizer); optimizer.zero_grad()` when the config sets `adam: True` (reference
// trainer/trainer.py:211-217: AdamW(g_b, lr=lr0, betas=(momentum, 0.999)) + the conv-weight and BN-weight groups).
// Per element, with the per-group fp32 scalars that the host computes in float64 and rounds once (optim.FusedAdamW):
//   p = p * (1 - lr*wd) ; m = lerp(m, g, 1 - b1) ; v = v*b2 ; v = fma(1 - b2, g*g, v)
//   p = fma(-lr/bc1, m / (sqrt(v) / sqrt(bc2) + eps), p) ; g = 0
// which is torch's _multi_tensor_adam (non-capturable, decoupled weight decay) op for op and rounding for rounding: each
// foreach op rounds to fp32 once, addcmul / addcdiv are explicit fmas in ATen, and lerp's `self + w*(end - self)` is
// contracted to an fma by torch's build.  This library builds with --fmad=false, so every fma below is written out.
// One launch for all parameters, one block per EtbChunk {p, g, m, v}; hyper_dev[8*group + k] lives in device memory, so a
// captured CUDA graph of the step follows the schedule and the bias corrections of later steps.
// HBM-bound: read p, g, m, v; write p, m, v and the zeroed g = 32 B/parameter.
#include "common.cuh"

__global__ void __launch_bounds__(256) adamw_kernel(const EtbChunk* __restrict__ tab, const float* __restrict__ hyper,
                                                    int zero_grad) {
  const EtbChunk c = tab[blockIdx.x];
  const float* h = hyper + 8 * c.group;
  const float decay = h[0], w1 = h[1], b2 = h[2], omb2 = h[3], step = h[4], sbc2 = h[5], eps = h[6];
  const bool small = fabsf(w1) < 0.5f;     // at::native::lerp's branch (is_lerp_weight_small)
  const float omw1 = __fsub_rn(1.f, w1);
  float* __restrict__ p = c.t[0];
  float* __restrict__ g = c.t[1];
  float* __restrict__ m = c.t[2];
  float* __restrict__ v = c.t[3];
  const int n = c.n;
  const bool vec = ((((uintptr_t)p) | ((uintptr_t)g) | ((uintptr_t)m) | ((uintptr_t)v)) & 15u) == 0;
  auto upd = [&](float& pv, float& gv, float& mv, float& vv) {
    pv = __fmul_rn(pv, decay);
    const float d = __fsub_rn(gv, mv);
    mv = small ? fmaf(w1, d, mv) : fmaf(-d, omw1, gv);
    vv = fmaf(omb2, __fmul_rn(gv, gv), __fmul_rn(vv, b2));
    const float den = __fadd_rn(__fdiv_rn(__fsqrt_rn(vv), sbc2), eps);
    pv = fmaf(step, __fdiv_rn(mv, den), pv);
    if (zero_grad) gv = 0.f;
  };
  if (vec) {
    const int n4 = n >> 2;
    float4* p4 = reinterpret_cast<float4*>(p);
    float4* g4 = reinterpret_cast<float4*>(g);
    float4* m4 = reinterpret_cast<float4*>(m);
    float4* v4 = reinterpret_cast<float4*>(v);
    for (int i = threadIdx.x; i < n4; i += 256) {
      float4 pv = p4[i], gv = g4[i], mv = m4[i], vv = v4[i];
      upd(pv.x, gv.x, mv.x, vv.x); upd(pv.y, gv.y, mv.y, vv.y); upd(pv.z, gv.z, mv.z, vv.z); upd(pv.w, gv.w, mv.w, vv.w);
      p4[i] = pv; m4[i] = mv; v4[i] = vv;
      if (zero_grad) g4[i] = gv;
    }
    for (int i = (n4 << 2) + threadIdx.x; i < n; i += 256) upd(p[i], g[i], m[i], v[i]);
  } else {
    for (int i = threadIdx.x; i < n; i += 256) upd(p[i], g[i], m[i], v[i]);
  }
}

extern "C" int etb_adamw_step(const EtbChunk* table_dev, int64_t n_chunks, const float* hyper_dev, int32_t zero_grad,
                              void* stream) {
  ETB_CHECK_ARG(table_dev && hyper_dev && n_chunks >= 0 && n_chunks < (1ll << 31));
  if (n_chunks == 0) return ETB_OK;
  etb_launch(adamw_kernel, dim3((unsigned)n_chunks), dim3(256), 0, (cudaStream_t)stream, table_dev, hyper_dev, zero_grad);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
