// metrics.cu -- the validation epoch on the device (reference val.py:275-400 and utils/metrics.py:22-126).
//
// Per batch (etb_val_epoch_append, no host sync, no allocation):
//   the NMS rows of every image are rescaled to its native image space (utils/general.py scale_coords with the loader's
//   ratio_pad), the normalised xywh targets become native-space xyxy labels, etb_val_process_batch matches them, and each
//   detection's (conf, class, correct bits) is appended to an epoch arena at a running offset kept in device memory.
//   The label classes go into an int32 histogram (etb_label_class_hist).  etb_val_epoch_append_confusion also adds the
//   rescaled rows and labels into a confusion matrix (etb_confusion_matrix, csrc/val.cu).
// Epoch end (etb_ap_per_class): the numeric core of ap_per_class -- sort by (class, conf descending), segmented cumulative
//   TP / FP counts, precision / recall in float64, the precision envelope, numpy.interp at the 101 COCO recall points of
//   compute_ap and at the 1000 confidence points of the P and R curves.  The O(nc * 1000) tail (trapz, F1, argmax, means)
//   stays with the host, in numpy, so its summation order is numpy's.
#include <cub/cub.cuh>

#include "common.cuh"

#define VAL_MAX_T 16

// ---- per batch -----------------------------------------------------------------------------------------------------------

// scale_coords(img1_shape, coords, img0_shape, ratio_pad) with ratio_pad = ((gain, _), (padw, padh)) as torch runs it on fp32
// CUDA tensors: coords[:, [0, 2]] -= padw (fp32 subtraction of the scalar rounded to fp32), coords[:, :4] /= gain (torch
// divides by a host scalar as a multiplication by its reciprocal, 1 / gain taken in float64 and rounded to fp32: the caller
// passes that value), then clamp_(0, w0) / clamp_(0, h0).
__device__ __forceinline__ float rescale_x(float v, float pad, float inv, float hi) {
  const float s = __fmul_rn(__fsub_rn(v, pad), inv);
  return fminf(fmaxf(s, 0.f), hi);
}

// meta[b] = (h0, w0, inv_gain, padw, padh).  det rows [b][d][det_ld] (x1,y1,x2,y2,conf,cls) -> det_native [b][d][6];
// targets [nt][6] (img, cls, x, y, w, h normalised) -> labels [nt][6] (img, cls, x1, y1, x2, y2) in native space.
__global__ void __launch_bounds__(256) val_rescale_kernel(const float* __restrict__ det, const int32_t* __restrict__ det_cnt, int B,
                                                          int max_det, int det_ld, const float* __restrict__ meta,
                                                          const float* __restrict__ targets, int nt, float fH, float fW, int single_cls,
                                                          float* __restrict__ det_native, float* __restrict__ labels) {
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B * max_det; i += stride) {
    const int b = i / max_det, d = i - b * max_det;
    if (d >= det_cnt[b]) continue;
    const float* m = meta + b * 5;
    const float inv = m[2];
    const float* r = det + (size_t)i * det_ld;
    float* o = det_native + (size_t)i * 6;
    o[0] = rescale_x(r[0], m[3], inv, m[1]);
    o[1] = rescale_x(r[1], m[4], inv, m[0]);
    o[2] = rescale_x(r[2], m[3], inv, m[1]);
    o[3] = rescale_x(r[3], m[4], inv, m[0]);
    o[4] = r[4];
    o[5] = single_cls ? 0.f : r[5];
  }
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < nt; t += stride) {
    const float* g = targets + (size_t)t * 6;
    float* o = labels + (size_t)t * 6;
    const int b = (int)g[0];
    o[0] = g[0];
    o[1] = g[1];
    if (b < 0 || b >= B) {                      // a target of no image in this batch: never matched (process_batch skips it)
      o[2] = o[3] = o[4] = o[5] = 0.f;
      continue;
    }
    const float* m = meta + b * 5;
    const float inv = m[2];
    const float x = __fmul_rn(g[2], fW), y = __fmul_rn(g[3], fH);           // targets[:, 2:6] *= [W, H, W, H]
    const float hw = __fmul_rn(__fmul_rn(g[4], fW), 0.5f), hh = __fmul_rn(__fmul_rn(g[5], fH), 0.5f);   // xywh2xyxy: w / 2
    o[2] = rescale_x(__fsub_rn(x, hw), m[3], inv, m[1]);
    o[3] = rescale_x(__fsub_rn(y, hh), m[4], inv, m[0]);
    o[4] = rescale_x(__fadd_rn(x, hw), m[3], inv, m[1]);
    o[5] = rescale_x(__fadd_rn(y, hh), m[4], inv, m[0]);
  }
}

// detect.py:240, det[:, :4] = scale_coords(img.shape[2:], det[:, :4], im0.shape).round(): the rescale above, then torch.round
// (half to even).  meta[b] = (h0, w0, inv_gain, padw, padh); out [b][d][6].
__global__ void __launch_bounds__(256) detect_rescale_kernel(const float* __restrict__ det, const int32_t* __restrict__ det_cnt, int B,
                                                             int max_det, int det_ld, const float* __restrict__ meta, float* __restrict__ out) {
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B * max_det; i += stride) {
    const int b = i / max_det, d = i - b * max_det;
    if (d >= det_cnt[b]) continue;
    const float* m = meta + b * 5;
    const float* r = det + (size_t)i * det_ld;
    float* o = out + (size_t)i * 6;
    o[0] = rintf(rescale_x(r[0], m[3], m[2], m[1]));
    o[1] = rintf(rescale_x(r[1], m[4], m[2], m[0]));
    o[2] = rintf(rescale_x(r[2], m[3], m[2], m[1]));
    o[3] = rintf(rescale_x(r[3], m[4], m[2], m[0]));
    o[4] = r[4];
    o[5] = r[5];
  }
}

extern "C" int etb_detect_rescale(const float* det, const int32_t* det_cnt, int32_t B, int32_t max_det, int32_t det_ld, const float* meta,
                                  float* out, void* stream) {
  ETB_CHECK_ARG(det && det_cnt && meta && out && B > 0 && max_det > 0 && det_ld >= 6);
  const int64_t work = (int64_t)B * max_det;
  ETB_CHECK_ARG(work < (1ll << 31));
  const int blocks = (int)((work + 255) / 256 < 1024 ? (work + 255) / 256 : 1024);
  etb_launch(detect_rescale_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, det, det_cnt, B, max_det, det_ld, meta, out);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// One block per image: its detections go to arena rows [*arena_n + sum(det_cnt[:b]), ...).  flags[0] |= any TP bit,
// flags[1] = 1 if the arena would overflow (those rows are dropped).
__global__ void __launch_bounds__(256) val_append_kernel(const float* __restrict__ det_native, const int32_t* __restrict__ det_cnt,
                                                         int max_det, const uint8_t* __restrict__ correct, int T,
                                                         float* __restrict__ a_conf, float* __restrict__ a_cls, uint16_t* __restrict__ a_tp,
                                                         int64_t cap, const int64_t* __restrict__ arena_n, int32_t* __restrict__ flags) {
  __shared__ int64_t s_base;
  const int b = blockIdx.x;
  if (threadIdx.x == 0) {
    int64_t base = *arena_n;
    for (int e = 0; e < b; ++e) base += det_cnt[e];
    s_base = base;
  }
  __syncthreads();
  const int n = det_cnt[b];
  int any = 0;
  for (int d = threadIdx.x; d < n; d += blockDim.x) {
    const int64_t row = s_base + d;
    if (row >= cap) { flags[1] = 1; break; }
    const float* r = det_native + ((size_t)b * max_det + d) * 6;
    const uint8_t* c = correct + ((size_t)b * max_det + d) * T;
    unsigned bits = 0;
    for (int i = 0; i < T; ++i) bits |= (unsigned)(c[i] != 0) << i;
    a_conf[row] = r[4];
    a_cls[row] = r[5];
    a_tp[row] = (uint16_t)bits;
    any |= bits != 0;
  }
  if (__syncthreads_or(any) && threadIdx.x == 0) flags[0] = 1;
}

__global__ void val_advance_kernel(const int32_t* __restrict__ det_cnt, int B, int64_t* __restrict__ arena_n) {
  int64_t s = 0;
  for (int b = 0; b < B; ++b) s += det_cnt[b];
  *arena_n += s;
}

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

extern "C" size_t etb_val_epoch_append_workspace_bytes(int32_t B, int32_t max_det, int32_t nt, int32_t T) {
  return align256((size_t)B * max_det * 6 * sizeof(float)) + align256((size_t)(nt > 0 ? nt : 1) * 6 * sizeof(float)) +
         align256((size_t)B * max_det * T);
}

// The confusion matrix a batch is also added into (etb_val_epoch_append_confusion); NULL: none.
struct ConfusionArgs {
  int32_t nc;
  float conf_thres, iou_thres;
  int64_t* matrix;
  int32_t* flags;
};

static int val_epoch_append(const float* det, const int32_t* det_cnt, int32_t B, int32_t max_det, int32_t det_ld, const float* img_meta,
                            const float* targets, int32_t nt, int32_t H, int32_t W, int32_t single_cls, const float* iouv, int32_t T,
                            int32_t nc, float* arena_conf, float* arena_cls, uint16_t* arena_tp, int64_t arena_cap, int64_t* arena_n,
                            int32_t* hist, int32_t* flags, const ConfusionArgs* cm, void* workspace, size_t workspace_bytes,
                            void* stream) {
  ETB_CHECK_ARG(det && det_cnt && img_meta && iouv && arena_conf && arena_cls && arena_tp && arena_n && hist && flags && workspace);
  ETB_CHECK_ARG(B > 0 && max_det > 0 && det_ld >= 6 && nt >= 0 && (targets || nt == 0) && H > 0 && W > 0 && nc > 0);
  ETB_CHECK_ARG(T > 0 && T <= VAL_MAX_T && arena_cap >= 0);
  ETB_CHECK_ARG(workspace_bytes >= etb_val_epoch_append_workspace_bytes(B, max_det, nt, T));
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  float* det_native = (float*)ws;
  ws += align256((size_t)B * max_det * 6 * sizeof(float));
  float* labels = (float*)ws;
  ws += align256((size_t)(nt > 0 ? nt : 1) * 6 * sizeof(float));
  uint8_t* correct = (uint8_t*)ws;
  const int work = B * max_det > nt ? B * max_det : nt;
  const int blocks = (work + 255) / 256 < 1024 ? (work + 255) / 256 : 1024;
  etb_launch(val_rescale_kernel, dim3(blocks), dim3(256), 0, st, det, det_cnt, B, max_det, det_ld, img_meta, targets, nt, (float)H,
             (float)W, single_cls, det_native, labels);
  ETB_CHECK_LAUNCH();
  int rc = etb_val_process_batch(det_native, det_cnt, B, max_det, 6, labels, nt, iouv, T, correct, flags + 1, stream);
  if (rc != ETB_OK) return rc;
  if (cm) {                                    // the rescaled rows and labels above: predn and labelsn of val.py:373
    rc = etb_confusion_matrix(det_native, det_cnt, B, max_det, 6, labels, nt, cm->nc, cm->conf_thres, cm->iou_thres, cm->matrix, cm->flags,
                              stream);
    if (rc != ETB_OK) return rc;
  }
  etb_launch(val_append_kernel, dim3(B), dim3(256), 0, st, det_native, det_cnt, max_det, correct, T, arena_conf, arena_cls, arena_tp,
             arena_cap, arena_n, flags);
  ETB_CHECK_LAUNCH();
  etb_launch(val_advance_kernel, dim3(1), dim3(1), 0, st, det_cnt, B, arena_n);
  ETB_CHECK_LAUNCH();
  if (nt > 0) {
    rc = etb_label_class_hist(targets, nullptr, nt, nt, 6, nc, hist, stream);
    if (rc != ETB_OK) return rc;
  }
  return ETB_OK;
}

extern "C" int etb_val_epoch_append(const float* det, const int32_t* det_cnt, int32_t B, int32_t max_det, int32_t det_ld,
                                    const float* img_meta, const float* targets, int32_t nt, int32_t H, int32_t W, int32_t single_cls,
                                    const float* iouv, int32_t T, int32_t nc, float* arena_conf, float* arena_cls, uint16_t* arena_tp,
                                    int64_t arena_cap, int64_t* arena_n, int32_t* hist, int32_t* flags, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  return val_epoch_append(det, det_cnt, B, max_det, det_ld, img_meta, targets, nt, H, W, single_cls, iouv, T, nc, arena_conf, arena_cls,
                          arena_tp, arena_cap, arena_n, hist, flags, nullptr, workspace, workspace_bytes, stream);
}

extern "C" int etb_val_epoch_append_confusion(const float* det, const int32_t* det_cnt, int32_t B, int32_t max_det, int32_t det_ld,
                                              const float* img_meta, const float* targets, int32_t nt, int32_t H, int32_t W,
                                              int32_t single_cls, const float* iouv, int32_t T, int32_t nc, float* arena_conf,
                                              float* arena_cls, uint16_t* arena_tp, int64_t arena_cap, int64_t* arena_n, int32_t* hist,
                                              int32_t* flags, int32_t cm_nc, float cm_conf, float cm_iou, int64_t* cm_matrix,
                                              int32_t* cm_flags, void* workspace, size_t workspace_bytes, void* stream) {
  ETB_CHECK_ARG(cm_matrix && cm_flags && cm_nc > 0);
  const ConfusionArgs cm = {cm_nc, cm_conf, cm_iou, cm_matrix, cm_flags};
  return val_epoch_append(det, det_cnt, B, max_det, det_ld, img_meta, targets, nt, H, W, single_cls, iouv, T, nc, arena_conf, arena_cls,
                          arena_tp, arena_cap, arena_n, hist, flags, &cm, workspace, workspace_bytes, stream);
}

// ---- epoch end: ap_per_class ---------------------------------------------------------------------------------------------

// Sort key: class slot in the high 32 bits (rows of a class without labels get slot nu and sort last), confidence descending
// in the low 32 bits.  The radix sort is stable, so equal confidences keep their row order (the stable rule of the oracle;
// numpy's argsort(-conf) leaves their order unspecified).  -0.0 sorts with +0.0; NaN sorts after every number.
__device__ __forceinline__ uint32_t conf_desc_bits(float c) {
  if (isnan(c)) return 0xffffffffu;
  if (c == 0.f) c = 0.f;                                      // -0.0 -> +0.0
  uint32_t u = __float_as_uint(c);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);             // unsigned order == float order
  return ~u;                                                  // descending
}

__global__ void ap_keys_kernel(const float* __restrict__ conf, const float* __restrict__ pcls, int n, const int32_t* __restrict__ cls_slot,
                               int ncls_table, int nu, uint64_t* __restrict__ keys, int32_t* __restrict__ vals) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float c = pcls[i];
    int slot = nu;
    if (c >= 0.f && c < (float)ncls_table && c == truncf(c)) {
      const int s = cls_slot[(int)c];
      if (s >= 0) slot = s;
    }
    keys[i] = ((uint64_t)slot << 32) | conf_desc_bits(conf[i]);
    vals[i] = i;
  }
}

// seg[s] = first sorted row of slot s (s = 0..nu; seg[nu] = end of the labelled classes' rows); gathers conf and tp.
__global__ void ap_segments_kernel(const uint64_t* __restrict__ keys, const int32_t* __restrict__ perm, const float* __restrict__ conf,
                                   const uint16_t* __restrict__ tp, int n, int nu, int32_t* __restrict__ seg, float* __restrict__ sconf,
                                   uint16_t* __restrict__ stp) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int s = (int)(keys[i] >> 32);
    const int sp = i == 0 ? -1 : (int)(keys[i - 1] >> 32);
    for (int q = sp + 1; q <= s && q <= nu; ++q) seg[q] = i;
    if (i == n - 1)
      for (int q = s + 1; q <= nu; ++q) seg[q] = n;
    const int j = perm[i];
    sconf[i] = conf[j];
    stp[i] = tp[j];
  }
}

// numpy.interp between (x0, f0) and (x1, f1) for x0 < x < x1 (numpy/_core/src/multiarray/compiled_base.c): slope * (x - x0)
// + f0, then the two NaN fall-backs.
__device__ __forceinline__ double interp_between(double x, double x0, double f0, double x1, double f1) {
  const double slope = __ddiv_rn(__dsub_rn(f1, f0), __dsub_rn(x1, x0));
  double r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, x0)), f0);
  if (isnan(r)) {
    r = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, x1)), f1);
    if (isnan(r) && f0 == f1) r = f0;
  }
  return r;
}

// first q in [0, n) with a[q] >= v (n if none)
__device__ __forceinline__ int lower_bound_d(const double* a, int n, double v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}
// first q in [0, n) with a[q] > v (n if none)
__device__ __forceinline__ int upper_bound_d(const double* a, int n, double v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] <= v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

#define AP_THREADS 512
#define AP_NX 101
#define AP_NPX 1000

struct ApCarry { int cnt; double env; };

// One block per (class slot, IoU column t).  The class's rows are walked from the last to the first in chunks of
// AP_THREADS; a block-wide scan in that reversed order gives, for every row k, the TP count after it (hence tpc[k] =
// total - after) and the suffix maximum of the precision (the envelope of compute_ap).  numpy.interp picks, for a query x,
// the largest j with xp[j] <= x, so each row k "owns" the queries x in [xp[k], xp[k+1]) and evaluates exactly those.
//   compute_ap: xp = mrec = [0, recall, 1], fp = envelope of [1, precision, 0], queries xs (101, ascending).
//   P / R curves (t == 0): xp = -conf (ascending), fp = precision / recall, queries -px (px: 1000, ascending),
//   left = 1 (P) / 0 (R), right = fp[-1].
__global__ void __launch_bounds__(AP_THREADS) ap_curves_kernel(const float* __restrict__ sconf, const uint16_t* __restrict__ stp,
                                                               const int32_t* __restrict__ seg, const int32_t* __restrict__ n_l_arr,
                                                               int T, const double* __restrict__ px_g, const double* __restrict__ xs_g,
                                                               double* __restrict__ ap_points, double* __restrict__ p_curve,
                                                               double* __restrict__ r_curve, int32_t* __restrict__ n_p_out) {
  typedef cub::BlockScan<int, AP_THREADS> ScanI;
  typedef cub::BlockScan<double, AP_THREADS> ScanD;
  typedef cub::BlockReduce<int, AP_THREADS> RedI;
  __shared__ union {
    typename ScanI::TempStorage si;
    typename ScanD::TempStorage sd;
    typename RedI::TempStorage ri;
  } tmp;
  __shared__ double xs[AP_NX];
  __shared__ double px[AP_NPX];
  __shared__ double s_rec[AP_THREADS], s_env[AP_THREADS], s_p[AP_THREADS], s_xp[AP_THREADS];
  __shared__ int s_total;
  __shared__ ApCarry s_carry;

  const int slot = blockIdx.x, t = blockIdx.y, tid = threadIdx.x;
  const int start = seg[slot], end = seg[slot + 1], n_p = end - start;
  const bool curves = (t == 0);
  double* apo = ap_points + ((size_t)slot * T + t) * AP_NX;
  if (curves && tid == 0) n_p_out[slot] = n_p;
  if (n_p == 0) {
    for (int q = tid; q < AP_NX; q += AP_THREADS) apo[q] = 0.0;
    if (curves)
      for (int q = tid; q < AP_NPX; q += AP_THREADS) p_curve[(size_t)slot * AP_NPX + q] = r_curve[(size_t)slot * AP_NPX + q] = 0.0;
    return;
  }
  for (int q = tid; q < AP_NX; q += AP_THREADS) xs[q] = xs_g[q];
  if (curves)
    for (int q = tid; q < AP_NPX; q += AP_THREADS) px[q] = px_g[q];
  // total TP of column t in the class
  int c = 0;
  for (int k = start + tid; k < end; k += AP_THREADS) c += (stp[k] >> t) & 1;
  c = RedI(tmp.ri).Sum(c);
  if (tid == 0) {
    s_total = c;
    s_carry.cnt = 0;
    s_carry.env = 0.0;                                   // envelope of the trailing sentinel precision 0
  }
  __syncthreads();
  const int total = s_total;
  const double nl = (double)n_l_arr[slot];               // n_l + 1e-16 == n_l in float64 for n_l >= 1
  double next_rec = 1.0, next_env = 0.0;                 // the trailing sentinel of mrec / mpre
  double next_p = 0.0, next_xp = 0.0;                    // P curve / -conf of row k + 1 (unused for the last row)
  for (int hi = end; hi > start; hi -= AP_THREADS) {
    const int k = hi - 1 - tid;
    const bool act = k >= start;
    const int bit = act ? (stp[k] >> t) & 1 : 0;
    int incl;
    ScanI(tmp.si).InclusiveSum(bit, incl);
    __syncthreads();
    const int after = s_carry.cnt + incl - bit;          // TP strictly after row k
    const int tpc = total - after;
    const double prec = __ddiv_rn((double)tpc, (double)(k - start + 1));
    const double rec = __ddiv_rn((double)tpc, nl);
    double env;
    ScanD(tmp.sd).InclusiveScan(act ? prec : -1.0, env, cub::Max());
    env = fmax(env, s_carry.env);
    const double xp = -(double)(act ? sconf[k] : 0.f);
    s_rec[tid] = rec;
    s_env[tid] = env;
    s_p[tid] = prec;
    s_xp[tid] = xp;
    __syncthreads();
    if (act) {
      // right neighbour (row k + 1): the previous thread of this chunk, or the last chunk's first row / the sentinel
      double r1, e1;
      if (tid > 0) { r1 = s_rec[tid - 1]; e1 = s_env[tid - 1]; }
      else { r1 = next_rec; e1 = next_env; }
      // compute_ap: this row owns xs in [rec, r1)
      for (int q = lower_bound_d(xs, AP_NX, rec); q < AP_NX && xs[q] < r1; ++q)
        apo[q] = xs[q] == rec ? env : interp_between(xs[q], rec, env, r1, e1);
      if (k == start) {
        // the leading sentinel (mrec 0, envelope 1: precision never exceeds 1) owns xs in [0, rec)
        for (int q = 0; q < AP_NX && xs[q] < rec; ++q) apo[q] = xs[q] == 0.0 ? 1.0 : interp_between(xs[q], 0.0, 1.0, rec, env);
      }
      if (k == end - 1) {
        // the trailing sentinel owns xs >= 1 (j == len(xp) - 1 -> fp[-1] = 0)
        for (int q = lower_bound_d(xs, AP_NX, 1.0); q < AP_NX; ++q) apo[q] = 0.0;
      }
      if (curves) {
        double* pc = p_curve + (size_t)slot * AP_NPX;
        double* rc = r_curve + (size_t)slot * AP_NPX;
        const double c_k = -xp;
        if (k == end - 1) {
          // x = -px >= xp[-1] (px <= conf[-1]): fp[-1] (numpy's right value is fp[-1] too)
          for (int q = 0, qe = upper_bound_d(px, AP_NPX, c_k); q < qe; ++q) { pc[q] = prec; rc[q] = rec; }
        } else {
          double p1, rr1, x1;
          if (tid > 0) { p1 = s_p[tid - 1]; rr1 = s_rec[tid - 1]; x1 = s_xp[tid - 1]; }
          else { p1 = next_p; rr1 = next_rec; x1 = next_xp; }
          // owns -px in [xp, x1): px in (conf[k + 1], conf[k]]
          for (int q = upper_bound_d(px, AP_NPX, -x1), qe = upper_bound_d(px, AP_NPX, c_k); q < qe; ++q) {
            const double x = -px[q];
            if (x == xp) { pc[q] = prec; rc[q] = rec; }
            else { pc[q] = interp_between(x, xp, prec, x1, p1); rc[q] = interp_between(x, xp, rec, x1, rr1); }
          }
        }
        if (k == start) {
          // x < xp[0] (px > conf[0]): the left values
          for (int q = upper_bound_d(px, AP_NPX, c_k); q < AP_NPX; ++q) { pc[q] = 1.0; rc[q] = 0.0; }
        }
      }
    }
    // carry to the next (earlier) chunk: the values of this chunk's first row hi - AP_THREADS (thread AP_THREADS - 1)
    const int last = hi - start < AP_THREADS ? hi - start - 1 : AP_THREADS - 1;
    next_rec = s_rec[last];
    next_env = s_env[last];
    next_p = s_p[last];
    next_xp = s_xp[last];
    __syncthreads();
    if (tid == last) {
      s_carry.cnt = after + bit;
      s_carry.env = env;
    }
    __syncthreads();
  }
}

static size_t ap_sort_bytes(int n) {
  size_t b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr, (int32_t*)nullptr, n,
                                  0, 64);
  return b;
}

extern "C" size_t etb_ap_per_class_workspace_bytes(int64_t n, int32_t nu) {
  if (n < 1) n = 1;
  return 2 * align256(n * sizeof(uint64_t)) + 2 * align256(n * sizeof(int32_t)) + align256(n * sizeof(float)) +
         align256(n * sizeof(uint16_t)) + align256((size_t)(nu + 1) * sizeof(int32_t)) + align256(ap_sort_bytes((int)n));
}

extern "C" int etb_ap_per_class(const float* conf, const float* pred_cls, const uint16_t* tp, int64_t n, int32_t T, const int32_t* cls_slot,
                                int32_t ncls_table, int32_t nu, const int32_t* n_l, const double* px, const double* xs, double* ap_points,
                                double* p_curve, double* r_curve, int32_t* n_p, void* workspace, size_t workspace_bytes, void* stream) {
  ETB_CHECK_ARG(n >= 0 && n < (int64_t)1 << 31 && T > 0 && T <= VAL_MAX_T && nu >= 0 && ncls_table >= 0);
  ETB_CHECK_ARG(n == 0 || (conf && pred_cls && tp));
  ETB_CHECK_ARG(ncls_table == 0 || cls_slot);
  ETB_CHECK_ARG(nu == 0 || (n_l && px && xs && ap_points && p_curve && r_curve && n_p));
  ETB_CHECK_ARG(workspace && workspace_bytes >= etb_ap_per_class_workspace_bytes(n, nu));
  if (nu == 0) return ETB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int ni = (int)n;
  char* ws = (char*)workspace;
  const size_t nn = ni > 0 ? ni : 1;
  uint64_t* k_in = (uint64_t*)ws;   ws += align256(nn * sizeof(uint64_t));
  uint64_t* k_out = (uint64_t*)ws;  ws += align256(nn * sizeof(uint64_t));
  int32_t* v_in = (int32_t*)ws;     ws += align256(nn * sizeof(int32_t));
  int32_t* v_out = (int32_t*)ws;    ws += align256(nn * sizeof(int32_t));
  float* sconf = (float*)ws;        ws += align256(nn * sizeof(float));
  uint16_t* stp = (uint16_t*)ws;    ws += align256(nn * sizeof(uint16_t));
  int32_t* seg = (int32_t*)ws;      ws += align256((size_t)(nu + 1) * sizeof(int32_t));
  if (ni == 0) {
    ETB_CHECK_CUDA(cudaMemsetAsync(seg, 0, (size_t)(nu + 1) * sizeof(int32_t), st));
  } else {
    const int blocks = (ni + 255) / 256 < 4 * etb_num_sms() ? (ni + 255) / 256 : 4 * etb_num_sms();
    etb_launch(ap_keys_kernel, dim3(blocks), dim3(256), 0, st, conf, pred_cls, ni, cls_slot, ncls_table, nu, k_in, v_in);
    ETB_CHECK_LAUNCH();
    int hi_bits = 0;
    while ((1 << hi_bits) <= nu) ++hi_bits;            // slots 0..nu
    size_t sort_bytes = ap_sort_bytes(ni);
    ETB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs((void*)ws, sort_bytes, k_in, k_out, v_in, v_out, ni, 0, 32 + hi_bits, st));
    etb_count_launch();
    etb_launch(ap_segments_kernel, dim3(blocks), dim3(256), 0, st, k_out, v_out, conf, tp, ni, nu, seg, sconf, stp);
    ETB_CHECK_LAUNCH();
  }
  etb_launch(ap_curves_kernel, dim3(nu, T), dim3(AP_THREADS), 0, st, sconf, stp, seg, n_l, T, px, xs, ap_points, p_curve, r_curve, n_p);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
