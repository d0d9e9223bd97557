// val.cu -- the matching step of the validation pass (8f rank 2): reference val.py:123-145 process_batch, batched on the device.
//   correct[d][i] = detection d is a true positive at IoU threshold iouv[i]
// Reference algorithm per threshold i (restated):  candidates = {(l, d): iou(l, d) >= iouv[i] and cls(l) == cls(d)};
//   sort by IoU descending; np.unique over the detection column keeps, per detection, its highest-IoU label l*(d); the result
//   is then ordered by detection index, so np.unique over the label column keeps, per label, the LOWEST-INDEX detection (=
//   the most confident one: NMS emits detections by descending confidence) among those whose best label it is.
// Hence l*(d) does not depend on the threshold, and
//   correct[d][i] = iou*(d) >= iouv[i]  and  no d' < d with l*(d') == l*(d) and iou*(d') >= iouv[i].
// IoU = inter / (area1 + area2 - inter) in fp32 exactly like utils/metrics.py:252-273 (box_iou).
// Ties in IoU between labels of one detection: the later label wins (stable ascending argsort, reversed).
// One block per image; labels of the image and (l*, iou*) of its detections live in shared memory.  Latency-bound.
#include "common.cuh"

#define VAL_THREADS 256
#define VAL_MAX_LABELS 1024
#define VAL_MAX_DET 1024
#define VAL_MAX_T 16

// The labels of image b (rows of labels [nt][6] whose first column is b), in the order of the targets tensor (val.py:344),
// into lab[k] = (cls, x1, y1, x2, y2).  Run by one thread; returns the count, at most VAL_MAX_LABELS (*overflow = 1 beyond).
__device__ __forceinline__ int load_image_labels(const float* __restrict__ labels, int nt, int b, float (*lab)[5], int* overflow) {
  int k = 0;
  for (int t = 0; t < nt; ++t)
    if ((int)labels[t * 6] == b) {
      if (k < VAL_MAX_LABELS) {
        for (int j = 0; j < 5; ++j) lab[k][j] = labels[t * 6 + 1 + j];
      }
      ++k;
    }
  if (k > VAL_MAX_LABELS) { atomicExch(overflow, 1); k = VAL_MAX_LABELS; }
  return k;
}

// box_iou(labels, detections) of utils/metrics.py:252-273 for one pair: l = the label's (x1, y1, x2, y2), area2 = the
// detection's area; inter / (area1 + area2 - inter) with area1 the label's, every step rounded in fp32 as torch does it.
__device__ __forceinline__ float label_det_iou(const float* l, float x1, float y1, float x2, float y2, float area2) {
  const float w = fmaxf(__fsub_rn(fminf(l[2], x2), fmaxf(l[0], x1)), 0.f);
  const float h = fmaxf(__fsub_rn(fminf(l[3], y2), fmaxf(l[1], y1)), 0.f);
  const float inter = __fmul_rn(w, h);
  const float area1 = __fmul_rn(__fsub_rn(l[2], l[0]), __fsub_rn(l[3], l[1]));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area1, area2), inter));
}

__global__ void __launch_bounds__(VAL_THREADS) val_process_batch_kernel(const float* __restrict__ det, const int* __restrict__ det_cnt, int max_det, int det_ld,
                                                                        const float* __restrict__ labels, int nt, const float* __restrict__ iouv, int T,
                                                                        unsigned char* __restrict__ correct, int* __restrict__ overflow) {
  __shared__ float lab[VAL_MAX_LABELS][5];     // cls, x1, y1, x2, y2
  __shared__ int nlab;
  __shared__ float biou[VAL_MAX_DET];
  __shared__ int blab[VAL_MAX_DET];
  const int b = blockIdx.x;
  const int n = min(det_cnt ? det_cnt[b] : max_det, max_det);
  if (threadIdx.x == 0) nlab = load_image_labels(labels, nt, b, lab, overflow);
  __syncthreads();
  const float* dp = det + (size_t)b * max_det * det_ld;
  for (int d = threadIdx.x; d < n; d += VAL_THREADS) {
    const float x1 = dp[d * det_ld], y1 = dp[d * det_ld + 1], x2 = dp[d * det_ld + 2], y2 = dp[d * det_ld + 3], c = dp[d * det_ld + 5];
    const float area2 = __fmul_rn(__fsub_rn(x2, x1), __fsub_rn(y2, y1));
    float best = -1.f;
    int bl = -1;
    for (int l = 0; l < nlab; ++l) {
      if (lab[l][0] != c) continue;
      const float iou = label_det_iou(lab[l] + 1, x1, y1, x2, y2, area2);
      if (iou >= best) { best = iou; bl = l; }          // ties: the later label
    }
    biou[d] = best;
    blab[d] = bl;
  }
  __syncthreads();
  unsigned char* cp = correct + (size_t)b * max_det * T;
  for (int d = threadIdx.x; d < max_det; d += VAL_THREADS) {
    for (int i = 0; i < T; ++i) {
      unsigned char ok = 0;
      if (d < n && blab[d] >= 0 && biou[d] >= iouv[i]) {
        ok = 1;
        for (int e = 0; e < d; ++e)
          if (blab[e] == blab[d] && biou[e] >= iouv[i]) { ok = 0; break; }
      }
      cp[d * T + i] = ok;
    }
  }
}

// det [B][max_det][det_ld >= 6] fp32 rows (x1,y1,x2,y2,conf,cls) in the labels' coordinate space; det_cnt [B] (NULL: all
// max_det rows valid); labels [nt][6] fp32 (img, cls, x1, y1, x2, y2); iouv [T]; correct [B][max_det][T] uint8 (fully
// written).  *overflow_dev is set to 1 if an image has more than 1024 labels (the rest are ignored).
extern "C" int etb_val_process_batch(const float* det, const int32_t* det_cnt, int32_t B, int32_t max_det, int32_t det_ld, const float* labels,
                                     int32_t nt, const float* iouv, int32_t T, uint8_t* correct, int32_t* overflow_dev, void* stream) {
  ETB_CHECK_ARG(det && iouv && correct && overflow_dev && B > 0 && max_det > 0 && max_det <= VAL_MAX_DET && det_ld >= 6 && nt >= 0 && (labels || nt == 0));
  ETB_CHECK_ARG(T > 0 && T <= VAL_MAX_T);
  etb_launch(val_process_batch_kernel, dim3(B), dim3(VAL_THREADS), 0, (cudaStream_t)stream, det, det_cnt, max_det, det_ld, labels, nt, iouv, T, correct,
             overflow_dev);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// ---- the detection confusion matrix (utils/metrics.py:129-186 ConfusionMatrix.process_batch, called at val.py:372-373) ------
// Reference algorithm per image (restated): keep the detections with conf > conf_thres (fp32 compare); candidates =
//   {(l, d): iou(l, d) > iou_thres}, class-agnostic; sort by IoU descending and keep each detection's first pair (its best
//   label l*(d)); sort the survivors by IoU descending again and keep each label's first pair (its best detection m(l) among
//   those whose best label it is).  numpy's argsort()[::-1] puts equal IoUs in reverse of their original (label-major, then
//   detection) order, so on ties the later label, then the later detection wins.
//   Every label l adds one to matrix[cls(m(l))][cls(l)], or to matrix[nc][cls(l)] without m(l).  Only if the image had a
//   candidate pair, every kept detection that is no label's m(l) adds one to matrix[cls(d)][nc].
// val.py:347-373 passes only images with at least one NMS row and at least one label; so does this kernel (det_cnt[b] == 0
// or no label: nothing is added).  Classes truncate toward zero like Tensor.int(); one outside [0, nc) sets flags[1] and is
// not counted (numpy's indexing of the reference would raise, or land in the background row / wrap).
// One block per image; the labels, l*(d) and its IoU live in shared memory.  The int64 counts are added with atomics, so
// their order does not matter and the float64 of the totals is the reference's sum of += 1.
#define CM_THREADS 256

__device__ __forceinline__ int cm_class(float c, int nc) { return c > -1.f && c < (float)nc ? (int)c : -1; }

__device__ __forceinline__ void cm_add(unsigned long long* matrix, int nc, int row, int col, int* flags) {
  if (row < 0 || col < 0) { flags[1] = 1; return; }
  atomicAdd(matrix + (size_t)row * (nc + 1) + col, 1ull);
}

__global__ void __launch_bounds__(CM_THREADS) confusion_matrix_kernel(const float* __restrict__ det, const int* __restrict__ det_cnt,
                                                                      int max_det, int det_ld, const float* __restrict__ labels, int nt,
                                                                      int nc, float conf_thres, float iou_thres,
                                                                      unsigned long long* __restrict__ matrix, int* __restrict__ flags) {
  __shared__ float lab[VAL_MAX_LABELS][5];     // cls, x1, y1, x2, y2
  __shared__ int nlab;
  __shared__ float biou[VAL_MAX_DET];
  __shared__ int blab[VAL_MAX_DET];            // l*(d); -1: no candidate pair, or conf <= conf_thres
  __shared__ unsigned char taken[VAL_MAX_DET]; // d is some label's m(l)
  const int b = blockIdx.x;
  const int n = min(det_cnt ? det_cnt[b] : max_det, max_det);
  if (n <= 0) return;
  if (threadIdx.x == 0) nlab = load_image_labels(labels, nt, b, lab, flags);
  __syncthreads();
  if (nlab == 0) return;
  const float* dp = det + (size_t)b * max_det * det_ld;
  int any = 0;
  for (int d = threadIdx.x; d < n; d += CM_THREADS) {
    const float* r = dp + (size_t)d * det_ld;
    float best = 0.f;
    int bl = -1;
    if (r[4] > conf_thres) {
      const float area2 = __fmul_rn(__fsub_rn(r[2], r[0]), __fsub_rn(r[3], r[1]));
      for (int l = 0; l < nlab; ++l) {
        const float iou = label_det_iou(lab[l] + 1, r[0], r[1], r[2], r[3], area2);
        if (iou > iou_thres && (bl < 0 || iou >= best)) { best = iou; bl = l; }     // ties: the later label
      }
    }
    biou[d] = best;
    blab[d] = bl;
    taken[d] = 0;
    any |= bl >= 0;
  }
  any = __syncthreads_or(any);
  for (int l = threadIdx.x; l < nlab; l += CM_THREADS) {
    float best = 0.f;
    int m = -1;
    for (int d = 0; d < n; ++d)
      if (blab[d] == l && (m < 0 || biou[d] >= best)) { best = biou[d]; m = d; }   // ties: the later detection
    int row = nc;
    if (m >= 0) {
      taken[m] = 1;                             // m(l) differs between labels: l*(m) == l
      row = cm_class(dp[(size_t)m * det_ld + 5], nc);
    }
    cm_add(matrix, nc, row, cm_class(lab[l][0], nc), flags);
  }
  __syncthreads();
  if (!any) return;
  for (int d = threadIdx.x; d < n; d += CM_THREADS) {
    const float* r = dp + (size_t)d * det_ld;
    if (r[4] > conf_thres && !taken[d]) cm_add(matrix, nc, cm_class(r[5], nc), nc, flags);
  }
}

// det [B][max_det][det_ld >= 6] fp32 rows (x1,y1,x2,y2,conf,cls) in the labels' coordinate space; det_cnt [B] (NULL: all
// max_det rows); labels [nt][6] fp32 (img, cls, x1, y1, x2, y2); matrix [(nc+1)^2] int64, counts ADDED.  flags[0] = 1 if an
// image has more than 1024 labels (the rest are ignored), flags[1] = 1 if a class to be counted is outside [0, nc).
extern "C" int etb_confusion_matrix(const float* det, const int32_t* det_cnt, int32_t B, int32_t max_det, int32_t det_ld, const float* labels,
                                    int32_t nt, int32_t nc, float conf_thres, float iou_thres, int64_t* matrix, int32_t* flags,
                                    void* stream) {
  ETB_CHECK_ARG(det && matrix && flags && B > 0 && max_det > 0 && max_det <= VAL_MAX_DET && det_ld >= 6 && nt >= 0 && (labels || nt == 0));
  ETB_CHECK_ARG(nc > 0);
  etb_launch(confusion_matrix_kernel, dim3(B), dim3(CM_THREADS), 0, (cudaStream_t)stream, det, det_cnt, max_det, det_ld, labels, nt, nc,
             conf_thres, iou_thres, (unsigned long long*)matrix, flags);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// ---- class-agnostic merge NMS of detection lists (extra-teachers path) ----------------------------------------------------
// reference utils/self_supervised_utils.py:256-274: for every extra teacher, per image: x = cat(current detections, that
// teacher's detections (class indices remapped)); index = torchvision.ops.nms(x[:, :4] + 0, x[:, 4], iou_thres); out = x[index].
// torchvision semantics (oracle/port.greedy_nms): stable descending score order, IoU = inter / (a + b - inter), suppress
// iff IoU > thr, kept rows in that order.  One block per image, n <= 1024 rows of `ld` floats; O(n^2) rank + greedy sweep.
#define MERGE_MAXN 1024
__global__ void __launch_bounds__(256) nms_boxes_kernel(const float* __restrict__ rows, const int* __restrict__ cnt, int nmax, int ld, float thr,
                                                        float* __restrict__ out, int* __restrict__ out_cnt) {
  __shared__ int order[MERGE_MAXN];
  __shared__ unsigned char sup[MERGE_MAXN];
  __shared__ int s_keep;
  const int b = blockIdx.x;
  const int n = min(cnt[b], nmax);
  const float* r = rows + (size_t)b * nmax * ld;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float s = r[i * ld + 4];
    int rank = 0;
    for (int j = 0; j < n; ++j) {
      const float t = r[j * ld + 4];
      rank += (t > s) || (t == s && j < i);           // stable descending
    }
    order[rank] = i;
    sup[i] = 0;
  }
  if (threadIdx.x == 0) s_keep = 0;
  __syncthreads();
  for (int a = 0; a < n; ++a) {
    const int i = order[a];
    if (sup[i]) continue;                              // uniform: shared memory, read after the barrier below
    const float x1 = r[i * ld], y1 = r[i * ld + 1], x2 = r[i * ld + 2], y2 = r[i * ld + 3];
    const float ai = __fmul_rn(__fsub_rn(x2, x1), __fsub_rn(y2, y1));
    for (int q = a + 1 + threadIdx.x; q < n; q += blockDim.x) {
      const int j = order[q];
      if (sup[j]) continue;
      const float u1 = r[j * ld], v1 = r[j * ld + 1], u2 = r[j * ld + 2], v2 = r[j * ld + 3];
      const float w = fmaxf(__fsub_rn(fminf(x2, u2), fmaxf(x1, u1)), 0.f), h = fmaxf(__fsub_rn(fminf(y2, v2), fmaxf(y1, v1)), 0.f);
      const float inter = __fmul_rn(w, h);
      const float aj = __fmul_rn(__fsub_rn(u2, u1), __fsub_rn(v2, v1));
      if (__fdiv_rn(inter, __fsub_rn(__fadd_rn(ai, aj), inter)) > thr) sup[j] = 1;
    }
    if (threadIdx.x == 0) {
      const int k = s_keep++;
      for (int c = 0; c < ld; ++c) out[((size_t)b * nmax + k) * ld + c] = r[i * ld + c];
    }
    __syncthreads();
  }
  __syncthreads();
  if (threadIdx.x == 0) out_cnt[b] = s_keep;
}

// rows [B][nmax][ld] fp32 (x1,y1,x2,y2,score,...), cnt [B] valid rows; out [B][nmax][ld] kept rows in descending-score order,
// out_cnt [B].  nmax <= 1024.
extern "C" int etb_nms_boxes(const float* rows, const int32_t* cnt, int32_t B, int32_t nmax, int32_t ld, float iou_thres, float* out,
                             int32_t* out_cnt, void* stream) {
  ETB_CHECK_ARG(rows && cnt && out && out_cnt && B > 0 && nmax > 0 && nmax <= MERGE_MAXN && ld >= 5 && iou_thres >= 0.f);
  etb_launch(nms_boxes_kernel, dim3(B), dim3(256), 0, (cudaStream_t)stream, rows, cnt, nmax, ld, iou_thres, out, out_cnt);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
