// sgd.cu -- fused multi-tensor SGD-Nesterov step (K16; SURVEY.md 8f #1): replaces torch.optim.SGD's foreach kernels and the
// separate gradient zeroing behind `scaler.step(optimizer); optimizer.zero_grad()` (reference trainer/ssod_trainer.py:481-484,
// optimizer built in trainer/trainer.py:193-217: 3 param groups, Nesterov momentum, weight decay on conv weights only).
//   g' = g + wd*p ; buf = momentum*buf + g' ; p -= lr*(g' + momentum*buf) ; g = 0
// One launch for all parameters, one block per EtbChunk {p, g, buf, unused}; the per-group hyper-parameters {lr, momentum, wd}
// are read from device memory, so a captured CUDA graph of the step keeps working when the scheduler changes the learning rate.
// HBM-bound: 5 streams x 4 B per parameter (read p, g, buf; write p, buf) + the grad zero write = 24 B/parameter.
#include "common.cuh"

__global__ void __launch_bounds__(256) sgd_kernel(const EtbChunk* __restrict__ tab, const float* __restrict__ hyper, int zero_grad) {
  const EtbChunk c = tab[blockIdx.x];
  const float lr = hyper[4 * c.group + 0], mom = hyper[4 * c.group + 1], wd = hyper[4 * c.group + 2];
  float* __restrict__ p = c.t[0];
  float* __restrict__ g = c.t[1];
  float* __restrict__ b = c.t[2];
  const int n = c.n;
  const bool vec = ((((uintptr_t)p) | ((uintptr_t)g) | ((uintptr_t)b)) & 15u) == 0;
  auto upd = [&](float& pv, float& gv, float& bv) {
    const float g1 = fmaf(wd, pv, gv);
    bv = fmaf(mom, bv, g1);
    pv = fmaf(-lr, fmaf(mom, bv, g1), pv);
    if (zero_grad) gv = 0.f;
  };
  if (vec) {
    const int n4 = n >> 2;
    float4* p4 = reinterpret_cast<float4*>(p);
    float4* g4 = reinterpret_cast<float4*>(g);
    float4* b4 = reinterpret_cast<float4*>(b);
    for (int i = threadIdx.x; i < n4; i += 256) {
      float4 pv = p4[i], gv = g4[i], bv = b4[i];
      upd(pv.x, gv.x, bv.x); upd(pv.y, gv.y, bv.y); upd(pv.z, gv.z, bv.z); upd(pv.w, gv.w, bv.w);
      p4[i] = pv; b4[i] = bv;
      if (zero_grad) g4[i] = gv;
    }
    for (int i = (n4 << 2) + threadIdx.x; i < n; i += 256) upd(p[i], g[i], b[i]);
  } else {
    for (int i = threadIdx.x; i < n; i += 256) upd(p[i], g[i], b[i]);
  }
}

extern "C" int etb_sgd_step(const EtbChunk* table_dev, int64_t n_chunks, const float* hyper_dev, int32_t zero_grad, void* stream) {
  ETB_CHECK_ARG(table_dev && hyper_dev && n_chunks >= 0 && n_chunks < (1ll << 31));
  if (n_chunks == 0) return ETB_OK;
  etb_launch(sgd_kernel, dim3((unsigned)n_chunks), dim3(256), 0, (cudaStream_t)stream, table_dev, hyper_dev, zero_grad);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
