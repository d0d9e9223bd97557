// assign.cu -- Pseudo-Label-Assigner routing (K10) and anchor assignment (K11).
//   etb_select_targets : ComputeStudentMatchLoss.select_targets  (reference models/loss/ssod/ssod_loss.py:130-192)
//   etb_build_targets  : YOLOAnchorAssigner.build_targets / build_uc_targets_aug
//                        (reference models/assigner/yolo_anchor_assigner.py:319-372, 640-697)
// Both are order-preserving stream compactions (block prefix sums), integer-exact with the CPU oracle.
// Latency-bound: <= 15*nt candidate slots per level; no roofline claim.
#include "common.cuh"

// ---------------------------------------------------------------------------------------------------
// select_targets.  One CTA.  Per row t (float64, as the reference compares numpy float64 values):
//   t[6] >= high[int(t[1])]                       -> reliable   <- t[0:7]
//   else t[6] >= low[int(t[1])]                   -> uncertain  <- t[0:6] || t[7]   (with_obj) / t[0:7]
//        and with_obj && t[7] >= 0.99             -> uncertain_obj (same row)
//        and with_obj && t[8] >= 0.99             -> uncertain_cls (same row)
// Outputs cast to fp32 (np.float32 in the reference), order preserved.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) select_targets_kernel(const double* __restrict__ rows, const int32_t* __restrict__ n_dev,
                                                              int32_t n_host, int32_t cap, const double* __restrict__ thr_high,
                                                              const double* __restrict__ thr_low, int32_t nc, int32_t with_obj,
                                                              float* __restrict__ out, int32_t* __restrict__ out_cnt) {
  __shared__ int sscan[33];
  int n = n_dev ? *n_dev : n_host;
  if (n > cap) n = cap;
  int base[4] = {0, 0, 0, 0};
  for (int r0 = 0; r0 < n; r0 += blockDim.x) {
    const int r = r0 + threadIdx.x;
    int f[4] = {0, 0, 0, 0};
    double t[9];
    if (r < n) {
#pragma unroll
      for (int k = 0; k < 9; ++k) t[k] = rows[(size_t)r * 9 + k];
      int c = (int)t[1];
      c = c < 0 ? 0 : (c >= nc ? nc - 1 : c);
      if (t[6] >= thr_high[c]) {
        f[0] = 1;
      } else if (t[6] >= thr_low[c]) {
        f[1] = 1;
        if (with_obj) {
          f[2] = t[7] >= 0.99;
          f[3] = t[8] >= 0.99;
        }
      }
    }
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      int tot;
      int pos = block_excl_scan(f[s], sscan, &tot);
      if (f[s]) {
        float* o = out + ((size_t)s * cap + base[s] + pos) * 7;
#pragma unroll
        for (int k = 0; k < 6; ++k) o[k] = (float)t[k];
        o[6] = (float)((s == 0 || !with_obj) ? t[6] : t[7]);
      }
      base[s] += tot;
    }
  }
  if (threadIdx.x < 4) out_cnt[threadIdx.x] = base[threadIdx.x];
}

extern "C" int etb_select_targets(const double* rows, const int32_t* n_dev, int32_t n_host, int32_t cap,
                                  const double* thr_high, const double* thr_low, int32_t nc, int32_t with_obj,
                                  float* out, int32_t* out_cnt, void* stream) {
  ETB_CHECK_ARG(rows && thr_high && thr_low && out && out_cnt && cap > 0 && nc > 0);
  etb_launch(select_targets_kernel, dim3(1), dim3(1024), 0, (cudaStream_t)stream, rows, n_dev, n_host, cap, thr_high, thr_low, nc, with_obj, out, out_cnt);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// ---------------------------------------------------------------------------------------------------
// build_targets.  grid.x = level.  Candidate slot index q = (o*na + a)*nt + k   (offset-major, anchor-major,
// target order -- the order `t.repeat((5,1,1))[j]` produces in the reference).  A slot survives iff
//   max(w'/Aw, Aw/w', h'/Ah, Ah/h') < anchor_t          (anchor ratio test, :342-345)
//   and offset o is enabled: o=0 always; 1: gx%1<.5 & gx>1; 2: gy%1<.5 & gy>1; 3: (nx-gx)%1<.5 & (nx-gx)>1; 4: same for y.
// All arithmetic is fp32 with single roundings (library is built with --fmad=false).
// ---------------------------------------------------------------------------------------------------
// torch `x % 1.` (remainder: result takes the sign of the divisor), aten/src/ATen/native/cpu/BinaryOpsKernel.cpp
__device__ __forceinline__ float py_mod1(float x) {
  float m = fmodf(x, 1.0f);
  if (m != 0.f && m < 0.f) m = __fadd_rn(m, 1.0f);
  return m;
}

struct AssignArgs {
  const float* targets;
  const int32_t* nt_dev;
  int32_t nt_host, tstride;
  EtbAssignLevels lv;
  EtbAssignOut out;
};

__global__ void __launch_bounds__(1024) build_targets_kernel(const AssignArgs A) {
  __shared__ int sscan[33];
  const int l = blockIdx.x;
  const int nx = A.lv.nx[l], ny = A.lv.ny[l];
  const float fnx = (float)nx, fny = (float)ny;
  int nt = A.nt_dev ? *A.nt_dev : A.nt_host;
  if (nt * 15 > A.out.cap) nt = A.out.cap / 15;
  const int total = 15 * nt;
  int32_t* __restrict__ oidx = A.out.idx[l];
  float* __restrict__ otbox = A.out.tbox[l];
  float* __restrict__ oanch = A.out.anch[l];
  int32_t* __restrict__ otcls = A.out.tcls[l];
  float* __restrict__ otsc = A.out.tscore[l];
  const int ts = A.tstride;
  int base = 0;
  for (int q0 = 0; q0 < total; q0 += blockDim.x) {
    const int q = q0 + threadIdx.x;
    int flag = 0;
    int o = 0, a = 0;
    float img = 0.f, cls = 0.f, gx = 0.f, gy = 0.f, gw = 0.f, gh = 0.f, sc = 0.f, aw = 0.f, ah = 0.f;
    if (q < total) {
      o = q / (3 * nt);
      const int rem = q - o * 3 * nt;
      a = rem / nt;
      const int k = rem - a * nt;
      const float* t = A.targets + (size_t)k * ts;
      img = t[0];
      cls = t[1];
      gx = __fmul_rn(t[2], fnx);
      gy = __fmul_rn(t[3], fny);
      gw = __fmul_rn(t[4], fnx);
      gh = __fmul_rn(t[5], fny);
      if (ts > 6) sc = t[6];
      aw = A.lv.anchors[l][2 * a];
      ah = A.lv.anchors[l][2 * a + 1];
      const float rw = __fdiv_rn(gw, aw), rh = __fdiv_rn(gh, ah);
      const float mw = fmaxf(rw, __fdiv_rn(1.0f, rw)), mh = fmaxf(rh, __fdiv_rn(1.0f, rh));
      const bool match = fmaxf(mw, mh) < A.lv.anchor_t;
      bool en = true;
      if (o == 1) en = (py_mod1(gx) < 0.5f) && (gx > 1.0f);
      else if (o == 2) en = (py_mod1(gy) < 0.5f) && (gy > 1.0f);
      else if (o == 3) { const float ix = __fsub_rn(fnx, gx); en = (py_mod1(ix) < 0.5f) && (ix > 1.0f); }
      else if (o == 4) { const float iy = __fsub_rn(fny, gy); en = (py_mod1(iy) < 0.5f) && (iy > 1.0f); }
      flag = (match && en) ? 1 : 0;
    }
    int tot;
    const int pos = block_excl_scan(flag, sscan, &tot);
    if (flag) {
      const int r = base + pos;
      const float offx = (o == 1) ? 0.5f : ((o == 3) ? -0.5f : 0.f);
      const float offy = (o == 2) ? 0.5f : ((o == 4) ? -0.5f : 0.f);
      // gij = (gxy - offsets).long(): truncation toward zero of the fp32 difference
      const long long gi0 = (long long)__fsub_rn(gx, offx);
      const long long gj0 = (long long)__fsub_rn(gy, offy);
      long long gi = gi0 < 0 ? 0 : (gi0 > nx - 1 ? nx - 1 : gi0);
      long long gj = gj0 < 0 ? 0 : (gj0 > ny - 1 ? ny - 1 : gj0);
      oidx[4 * r + 0] = (int32_t)(long long)img;
      oidx[4 * r + 1] = a;
      oidx[4 * r + 2] = (int32_t)gj;
      oidx[4 * r + 3] = (int32_t)gi;
      otbox[4 * r + 0] = __fsub_rn(gx, (float)gi0);  // uses the UNclamped gij (:369)
      otbox[4 * r + 1] = __fsub_rn(gy, (float)gj0);
      otbox[4 * r + 2] = gw;
      otbox[4 * r + 3] = gh;
      oanch[2 * r + 0] = aw;
      oanch[2 * r + 1] = ah;
      otcls[r] = (int32_t)(long long)cls;
      if (otsc) otsc[r] = sc;
    }
    base += tot;
  }
  if (threadIdx.x == 0) A.out.cnt[l] = base;
}

extern "C" int etb_build_targets(const float* targets, const int32_t* nt_dev, int32_t nt_host, int32_t tstride,
                                 const EtbAssignLevels* lv, const EtbAssignOut* out, void* stream) {
  ETB_CHECK_ARG(lv && out && lv->nl >= 1 && lv->nl <= ETB_MAX_LEVELS);
  ETB_CHECK_ARG(tstride == 6 || tstride == 7);
  ETB_CHECK_ARG(out->cnt && out->cap >= 0);
  ETB_CHECK_ARG(targets != nullptr || (nt_dev == nullptr && nt_host == 0));
  AssignArgs A;
  A.targets = targets;
  A.nt_dev = nt_dev;
  A.nt_host = nt_host;
  A.tstride = tstride;
  A.lv = *lv;
  A.out = *out;
  for (int l = 0; l < lv->nl; ++l) ETB_CHECK_ARG(out->cap == 0 || (out->idx[l] && out->tbox[l] && out->anch[l] && out->tcls[l]));
  etb_launch(build_targets_kernel, dim3(lv->nl), dim3(1024), 0, (cudaStream_t)stream, A);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// ---------------------------------------------------------------------------------------------------
// label_class_hist.  LabelMatch.update's `cls_tmp[int(l[1:2])] += 1` over the labeled rows (reference
// utils/labelmatch.py:126-134), accumulated into hist[nc+1] on the device.  n = *n_dev (or n_host), clamped to cap;
// rows at or past n are never read.  int() truncates toward zero, so (-1, nc) is a valid class; anything else
// (NaN included) is counted in hist[nc].  Integer atomics: the result does not depend on the order.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) label_class_hist_kernel(const float* __restrict__ targets, const int32_t* __restrict__ n_dev,
                                                               int32_t n_host, int32_t cap, int32_t tstride, int32_t nc,
                                                               int32_t* __restrict__ hist) {
  int n = n_dev ? *n_dev : n_host;
  if (n > cap) n = cap;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
    const float v = targets[(size_t)r * tstride + 1];
    const int c = (v > -1.0f && v < (float)nc) ? (int)v : nc;
    atomicAdd(hist + c, 1);
  }
}

extern "C" int etb_label_class_hist(const float* targets, const int32_t* n_dev, int32_t n_host, int32_t cap, int32_t tstride,
                                    int32_t nc, int32_t* hist, void* stream) {
  ETB_CHECK_ARG(hist && nc > 0 && tstride >= 2 && cap >= 0 && n_host >= 0 && n_host <= cap);
  ETB_CHECK_ARG(targets != nullptr || cap == 0);
  if (cap == 0) return ETB_OK;
  // grid sized by the capacity (the count may only be known on the device): one launch shape per buffer, so it can be captured
  const int blocks = (cap + 255) / 256 < 32 ? (cap + 255) / 256 : 32;
  etb_launch(label_class_hist_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, targets, n_dev, n_host, cap, tstride, nc,
             hist);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
