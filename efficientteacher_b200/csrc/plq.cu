// plq.cu -- pseudo-label quality statistics of the SSOD step and the device-resident training meter.
//
// Reference utils/self_supervised_utils.py:481-587 check_pseudo_label_with_gt (restated):
//   1. :456-479 select_targets keeps the UNCERTAIN rows, thr_low[int(cls)] <= conf < thr_high[int(cls)] compared in float64,
//      cast to fp32 (:474).  No thresholds: every row, kept in its own dtype (float64 here).
//   2. pse_num = n_uc / batch_size, gt_num = M / batch_size (float64).
//   3. :521-524 both box sets are normalised xywh: * 640, xywh2xyxy (utils/general.py:630-637, fp32: x - w / 2, x + w / 2),
//      + img_index * 640 on all four coordinates; then box_iou(gt, pseudo) (utils/metrics.py:252-273).  With float64 rows
//      (no thresholds) the pseudo side stays float64, so inter, area2 and the IoU are float64 and only area1 (gt) is fp32.
//   4. :535-570 per IoU threshold t, all in the same image:  tp: iou >= t and same class;  fp_cls: iou >= t and another class;
//      fp_loc: iou < t and iou > float32(0.01), any class.  Each set goes through val.py's de-duplication (sort by IoU
//      descending, np.unique on the detection, then on the label).  As csrc/val.cu restates it, that keeps per label the
//      lowest-index detection among those whose best candidate label it is (IoU ties between labels: the later label, the
//      order of a stable sort; numpy's argsort is not stable on every CPU, so there the reference's choice is machine-dependent),
//      so the COUNT of a set is the number of distinct best labels among the detections that have a candidate.  tp's and
//      fp_cls's best label does not depend on t (the best IoU reaches t whenever any does); fp_loc's does (iou < t).
//   5. :571-578 rate = count / n_uc in float64, or 0 when n_uc == 0.
// Reference :589-606 check_pseudo_label (SSOD.ssod_hyp.with_gt False): reliable = r / bs, uncertain = u / bs (float64);
//   (reliable / (reliable + uncertain) or 0, (reliable + uncertain) * bs / N or 0, reliable + uncertain, reliable), which
//   trainer/ssod_trainer.py:666-670 logs as tp, fp_loc, pse_num, gt_num with fp_cls = 0.
// A step without pseudo labels (n == 0) logs zeros for all five (ssod_trainer.py:658-660).
//
// Images are independent: PLQ_GRID blocks walk the images (block b takes images b, b + PLQ_GRID, ...), each image's labels in
// shared memory (at most PLQ_MAX_LABELS; more sets the overflow flag and the rest are ignored).  Rows per image are not
// limited: every thread tests its rows against the image's labels and marks the best labels in per-label bit masks; the
// first marker of a (label, set, t) bit counts it.  Integer counts, so the order of the atomics does not matter.  A second
// one-block kernel adds the blocks' partial counts and writes the float64 values; no host sync, no allocation.
#include "common.cuh"

#define PLQ_THREADS 256
#define PLQ_GRID 32
#define PLQ_MAX_LABELS 1024
#define PLQ_MAX_T 16
#define PLQ_PART (3 + 3 * PLQ_MAX_T)     // per block: n_reliable, n_uc, overflow, tp[T], fp_cls[T], fp_loc[T]

__device__ __forceinline__ int plq_count(const int32_t* dev, int32_t host) { return dev ? max(0, min(*dev, host)) : host; }

// 0 reliable, 1 uncertain, -1 neither, -2 class index outside [0, nc)
__device__ __forceinline__ int plq_kind(const double* r, const double* thr_high, const double* thr_low, int nc) {
  if (!thr_high) return 1;
  const int c = (int)r[1];
  if (c < 0 || c >= nc) return -2;
  if (r[6] >= thr_high[c]) return 0;
  return r[6] >= thr_low[c] ? 1 : -1;
}

// IoU of the image's label l with a pseudo box, in R (float: the fp32 path; double: float64 rows without thresholds)
template <typename R>
__device__ __forceinline__ R plq_iou(const float* lab, float area1, R x1, R y1, R x2, R y2, R area2);
template <>
__device__ __forceinline__ float plq_iou<float>(const float* lab, float area1, float x1, float y1, float x2, float y2, float area2) {
  const float w = fmaxf(__fsub_rn(fminf(lab[3], x2), fmaxf(lab[1], x1)), 0.f);
  const float h = fmaxf(__fsub_rn(fminf(lab[4], y2), fmaxf(lab[2], y1)), 0.f);
  const float inter = __fmul_rn(w, h);
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area1, area2), inter));
}
template <>
__device__ __forceinline__ double plq_iou<double>(const float* lab, float area1, double x1, double y1, double x2, double y2, double area2) {
  const double w = fmax(__dsub_rn(fmin((double)lab[3], x2), fmax((double)lab[1], x1)), 0.0);
  const double h = fmax(__dsub_rn(fmin((double)lab[4], y2), fmax((double)lab[2], y1)), 0.0);
  const double inter = __dmul_rn(w, h);
  return __ddiv_rn(inter, __dsub_rn(__dadd_rn((double)area1, area2), inter));
}

// pseudo box of row r: xywh * 640 -> xyxy -> + img * 640 (self_supervised_utils.py:522,524)
__device__ __forceinline__ void plq_box(const double* r, float* b) {
  const float x = __fmul_rn(__double2float_rn(r[2]), 640.f), y = __fmul_rn(__double2float_rn(r[3]), 640.f);
  const float w = __fmul_rn(__double2float_rn(r[4]), 640.f), h = __fmul_rn(__double2float_rn(r[5]), 640.f);
  const float off = __fmul_rn(__double2float_rn(r[0]), 640.f);
  b[0] = __fadd_rn(__fsub_rn(x, __fdiv_rn(w, 2.f)), off);
  b[1] = __fadd_rn(__fsub_rn(y, __fdiv_rn(h, 2.f)), off);
  b[2] = __fadd_rn(__fadd_rn(x, __fdiv_rn(w, 2.f)), off);
  b[3] = __fadd_rn(__fadd_rn(y, __fdiv_rn(h, 2.f)), off);
}
__device__ __forceinline__ void plq_box(const double* r, double* b) {
  const double x = __dmul_rn(r[2], 640.0), y = __dmul_rn(r[3], 640.0), w = __dmul_rn(r[4], 640.0), h = __dmul_rn(r[5], 640.0);
  const double off = __dmul_rn(r[0], 640.0);
  b[0] = __dadd_rn(__dsub_rn(x, __ddiv_rn(w, 2.0)), off);
  b[1] = __dadd_rn(__dsub_rn(y, __ddiv_rn(h, 2.0)), off);
  b[2] = __dadd_rn(__dadd_rn(x, __ddiv_rn(w, 2.0)), off);
  b[3] = __dadd_rn(__dadd_rn(y, __ddiv_rn(h, 2.0)), off);
}

__device__ __forceinline__ float plq_area(const float* b) { return __fmul_rn(__fsub_rn(b[2], b[0]), __fsub_rn(b[3], b[1])); }
__device__ __forceinline__ double plq_area(const double* b) { return __dmul_rn(__dsub_rn(b[2], b[0]), __dsub_rn(b[3], b[1])); }

__device__ __forceinline__ void plq_mark(unsigned* mask, unsigned bit, int* counter) {
  if (!(atomicOr(mask, bit) & bit)) atomicAdd(counter, 1);
}

template <typename R>
__global__ void __launch_bounds__(PLQ_THREADS) plq_image_kernel(const double* __restrict__ rows, const int32_t* n_dev, int n_host,
                                                                const double* __restrict__ thr_high, const double* __restrict__ thr_low, int nc,
                                                                const float* __restrict__ gt, const int32_t* m_dev, int m_host,
                                                                const double* __restrict__ iouv, int T, int with_gt, int* __restrict__ partial) {
  __shared__ float lab[PLQ_MAX_LABELS][5];     // cls, x1, y1, x2, y2 (offset by img * 640)
  __shared__ float area1[PLQ_MAX_LABELS];
  __shared__ unsigned hit[PLQ_MAX_LABELS];     // bit t: tp at iouv[t]; bit 16 + t: fp_cls
  __shared__ unsigned loc[PLQ_MAX_LABELS];     // bit t: fp_loc
  __shared__ int cnt[PLQ_PART];
  __shared__ int s_nlab, s_maximg;
  const int n = plq_count(n_dev, n_host), m = with_gt ? plq_count(m_dev, m_host) : 0;
  for (int i = threadIdx.x; i < PLQ_PART; i += PLQ_THREADS) cnt[i] = 0;
  if (threadIdx.x == 0) s_maximg = -1;
  __syncthreads();
  int maximg = -1;
  for (int r = blockIdx.x * PLQ_THREADS + threadIdx.x; r < n; r += PLQ_GRID * PLQ_THREADS) {   // the counts: every row once
    const int k = plq_kind(rows + (size_t)r * 9, thr_high, thr_low, nc);
    if (k >= 0) atomicAdd(&cnt[k], 1);
    else if (k == -2) atomicOr(&cnt[2], 1);
  }
  if (with_gt) {
    for (int r = threadIdx.x; r < n; r += PLQ_THREADS) maximg = max(maximg, (int)floor(rows[(size_t)r * 9]));
    for (int l = threadIdx.x; l < m; l += PLQ_THREADS) maximg = max(maximg, (int)floorf(gt[l * 6]));
    atomicMax(&s_maximg, maximg);
  }
  __syncthreads();
  R thr_r[PLQ_MAX_T];              // torch compares in the IoU's dtype: fp32(iouv) on the fp32 path
#pragma unroll
  for (int i = 0; i < PLQ_MAX_T; ++i) thr_r[i] = i < T ? (sizeof(R) == 4 ? (R)__double2float_rn(iouv[i]) : (R)iouv[i]) : (R)0;
  const R loc_lo = (R)0.01f;
  const int lane = threadIdx.x & 31;
  for (int b = blockIdx.x; b <= s_maximg; b += PLQ_GRID) {
    const float fb = (float)b;
    if (threadIdx.x < 32) {       // the image's labels, in label order (ballot compaction)
      int k = 0;
      for (int base = 0; base < m; base += 32) {
        const int l = base + lane;
        const bool in = l < m && gt[l * 6] == fb;
        const unsigned bal = __ballot_sync(0xffffffffu, in);
        const int pos = k + __popc(bal & ((1u << lane) - 1u));
        if (in && pos < PLQ_MAX_LABELS) {
          const float* g = gt + l * 6;
          const float x = __fmul_rn(g[2], 640.f), y = __fmul_rn(g[3], 640.f), w = __fmul_rn(g[4], 640.f), h = __fmul_rn(g[5], 640.f);
          const float off = __fmul_rn(g[0], 640.f);
          float* L = lab[pos];
          L[0] = g[1];
          L[1] = __fadd_rn(__fsub_rn(x, __fdiv_rn(w, 2.f)), off);
          L[2] = __fadd_rn(__fsub_rn(y, __fdiv_rn(h, 2.f)), off);
          L[3] = __fadd_rn(__fadd_rn(x, __fdiv_rn(w, 2.f)), off);
          L[4] = __fadd_rn(__fadd_rn(y, __fdiv_rn(h, 2.f)), off);
          area1[pos] = __fmul_rn(__fsub_rn(L[3], L[1]), __fsub_rn(L[4], L[2]));
          hit[pos] = 0u;
          loc[pos] = 0u;
        }
        k += __popc(bal);
      }
      if (lane == 0) {
        if (k > PLQ_MAX_LABELS) { atomicOr(&cnt[2], 1); k = PLQ_MAX_LABELS; }
        s_nlab = k;
      }
    }
    __syncthreads();
    const int nlab = s_nlab;
    if (nlab > 0) {
      for (int r = threadIdx.x; r < n; r += PLQ_THREADS) {
        const double* rp = rows + (size_t)r * 9;
        if (sizeof(R) == 4 ? __double2float_rn(rp[0]) != fb : rp[0] != (double)fb) continue;
        if (plq_kind(rp, thr_high, thr_low, nc) != 1) continue;
        R bx[4];
        plq_box(rp, bx);
        const R area2 = plq_area(bx);
        const float c = __double2float_rn(rp[1]);
        R best_same = (R)-1, best_diff = (R)-1;
        int l_same = -1, l_diff = -1;
        R best_loc[PLQ_MAX_T];
        int l_loc[PLQ_MAX_T];
#pragma unroll
        for (int i = 0; i < PLQ_MAX_T; ++i) { best_loc[i] = (R)-1; l_loc[i] = -1; }
        for (int l = 0; l < nlab; ++l) {
          const R iou = plq_iou<R>(lab[l], area1[l], bx[0], bx[1], bx[2], bx[3], area2);
          if (lab[l][0] == c) {
            if (iou >= best_same) { best_same = iou; l_same = l; }     // IoU ties: the later label
          } else if (iou >= best_diff) { best_diff = iou; l_diff = l; }
          if (iou > loc_lo) {
#pragma unroll
            for (int i = 0; i < PLQ_MAX_T; ++i)
              if (i < T && iou < thr_r[i] && iou >= best_loc[i]) { best_loc[i] = iou; l_loc[i] = l; }
          }
        }
#pragma unroll
        for (int i = 0; i < PLQ_MAX_T; ++i) {
          if (i >= T) break;
          if (l_same >= 0 && best_same >= thr_r[i]) plq_mark(&hit[l_same], 1u << i, &cnt[3 + i]);
          if (l_diff >= 0 && best_diff >= thr_r[i]) plq_mark(&hit[l_diff], 1u << (16 + i), &cnt[3 + PLQ_MAX_T + i]);
          if (l_loc[i] >= 0) plq_mark(&loc[l_loc[i]], 1u << i, &cnt[3 + 2 * PLQ_MAX_T + i]);
        }
      }
    }
    __syncthreads();              // the next image reuses the label arrays
  }
  __syncthreads();
  for (int i = threadIdx.x; i < PLQ_PART; i += PLQ_THREADS) partial[blockIdx.x * PLQ_PART + i] = cnt[i];
}

__global__ void plq_finalize_kernel(const int* __restrict__ partial, const int32_t* n_dev, int n_host, const int32_t* m_dev, int m_host,
                                    int T, int bs, int with_gt, double* __restrict__ vals, int32_t* __restrict__ out_cnt) {
  __shared__ int tot[PLQ_PART];
  for (int i = threadIdx.x; i < PLQ_PART; i += blockDim.x) {
    int s = 0;
    for (int b = 0; b < PLQ_GRID; ++b) s = i == 2 ? (s | partial[b * PLQ_PART + i]) : s + partial[b * PLQ_PART + i];
    tot[i] = s;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const int n = plq_count(n_dev, n_host), m = plq_count(m_dev, m_host), n_uc = tot[1], n_rel = tot[0];
  out_cnt[0] = n;
  out_cnt[1] = n_uc;
  out_cnt[2] = n_rel;
  out_cnt[3] = m;
  out_cnt[4] = tot[2];
  for (int i = 0; i < T; ++i)
    for (int s = 0; s < 3; ++s) out_cnt[5 + s * T + i] = tot[3 + s * PLQ_MAX_T + i];
  const double dbs = (double)bs;
  for (int i = 0; i < T; ++i) {
    double v[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
    if (n > 0 && with_gt) {
      for (int s = 0; s < 3; ++s) v[s] = n_uc ? __ddiv_rn((double)tot[3 + s * PLQ_MAX_T + i], (double)n_uc) : 0.0;
      v[3] = __ddiv_rn((double)n_uc, dbs);
      v[4] = __ddiv_rn((double)m, dbs);
    } else if (n > 0) {
      const double rel = __ddiv_rn((double)n_rel, dbs), unc = __ddiv_rn((double)n_uc, dbs), den = __dadd_rn(rel, unc);
      v[0] = den == 0.0 ? 0.0 : __ddiv_rn(rel, den);
      v[2] = __ddiv_rn(__dmul_rn(den, dbs), (double)n);
      v[3] = den;
      v[4] = rel;
    }
    for (int s = 0; s < 5; ++s) vals[s * T + i] = v[s];
  }
}

extern "C" size_t etb_pl_quality_workspace_bytes(void) { return sizeof(int) * PLQ_GRID * PLQ_PART; }

extern "C" int etb_pl_quality(const double* rows, const int32_t* n_dev, int32_t n_host, const double* thr_high, const double* thr_low,
                              int32_t nc, const float* gt, const int32_t* m_dev, int32_t m_host, const double* iouv, int32_t T,
                              int32_t batch_size, int32_t with_gt, int32_t iou64, double* vals, int32_t* cnt, void* workspace,
                              size_t workspace_bytes, void* stream) {
  ETB_CHECK_ARG(vals && cnt && iouv && workspace && workspace_bytes >= etb_pl_quality_workspace_bytes());
  ETB_CHECK_ARG(n_host >= 0 && (rows || n_host == 0) && m_host >= 0 && (gt || m_host == 0 || !with_gt) && batch_size > 0);
  ETB_CHECK_ARG(T > 0 && T <= PLQ_MAX_T && ((thr_high && thr_low && nc > 0) || (!thr_high && !thr_low && with_gt)));
  ETB_CHECK_ARG(!iou64 || !thr_high);
  const cudaStream_t st = (cudaStream_t)stream;
  int* part = (int*)workspace;
  if (iou64)
    etb_launch(plq_image_kernel<double>, dim3(PLQ_GRID), dim3(PLQ_THREADS), 0, st, rows, n_dev, n_host, thr_high, thr_low, nc, gt, m_dev,
               m_host, iouv, T, with_gt, part);
  else
    etb_launch(plq_image_kernel<float>, dim3(PLQ_GRID), dim3(PLQ_THREADS), 0, st, rows, n_dev, n_host, thr_high, thr_low, nc, gt, m_dev,
               m_host, iouv, T, with_gt, part);
  ETB_CHECK_LAUNCH();
  etb_launch(plq_finalize_kernel, dim3(1), dim3(64), 0, st, part, n_dev, n_host, m_dev, m_host, T, batch_size, with_gt, vals, cnt);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// ---- MetricMeter / AverageMeter (utils/metrics.py:352-414) on the device -----------------------------------------------
// state [3][cap] float64: sum, count, val.  AverageMeter.update(val, n=1): val; sum += val * 1; count += 1 -- in float64, one
// entry per key, so the sums agree bit for bit with the reference's Python floats added in the same order.
struct EtbMeterSrc {
  const void* p[ETB_METER_MAX_SRC];
  int32_t slot[ETB_METER_MAX_SRC];
  int32_t f64[ETB_METER_MAX_SRC];
};

__global__ void meter_update_kernel(double* __restrict__ state, int cap, EtbMeterSrc src, int n) {
  const int i = threadIdx.x;
  if (i >= n) return;
  const double v = src.f64[i] ? *(const double*)src.p[i] : (double)*(const float*)src.p[i];
  const int k = src.slot[i];
  state[k] = __dadd_rn(state[k], v);
  state[cap + k] = __dadd_rn(state[cap + k], 1.0);
  state[2 * cap + k] = v;
}

extern "C" int etb_meter_update(double* state, int32_t cap, const void* const* src, const int32_t* slot, const int32_t* f64, int32_t n,
                                void* stream) {
  ETB_CHECK_ARG(state && src && slot && f64 && n > 0 && n <= ETB_METER_MAX_SRC && cap > 0);
  EtbMeterSrc s = {};
  for (int i = 0; i < n; ++i) {
    ETB_CHECK_ARG(src[i] && slot[i] >= 0 && slot[i] < cap);
    for (int j = 0; j < i; ++j) ETB_CHECK_ARG(slot[j] != slot[i]);
    s.p[i] = src[i];
    s.slot[i] = slot[i];
    s.f64[i] = f64[i];
  }
  etb_launch(meter_update_kernel, dim3(1), dim3(32), 0, (cudaStream_t)stream, state, cap, s, n);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
