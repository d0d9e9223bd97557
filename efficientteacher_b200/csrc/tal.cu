// tal.cu -- the anchor-free (YOLOv8) pieces the reference ships in importable form (SURVEY.md section 8f row 5, config #4):
//   etb_tal_assign : TaskAlignedAssigner.forward        (reference models/assigner/tal_assigner.py:29-80 with the helpers of
//                                                        models/module/nanodet_utils.py:184-248)
//   etb_v8_decode  : DFL softmax-expectation + dist2bbox (reference models/head/yolov8_head.py:169-220 eval branch;
//                                                        models/loss/tal_loss.py:88-95,150-156 for the training-side boxes)
// The reference defines no end-to-end step for this head (tal_loss.py is unimportable, SSODTrainer rejects it), so these two are
// standalone operators with the reference's call contracts; nothing in the YOLOv5 SSOD step uses them.
//
// Bounds: etb_tal_assign is latency / L2 bound (B*M CTAs, each 13 block-wide arg-max rounds over A shared-memory floats) plus one
// HBM pass that writes target_scores (B*A*nc*4 B: 86 MB at 32 x 8400 x 80); etb_v8_decode is one HBM pass over the logits
// (B*A*(4*(reg_max+1)+nc)*4 B in, B*A*(5+nc)*4 B out).  Integer outputs (labels, foreground mask, chosen gt) are exact; the
// alignment metric uses a correctly rounded pow (via double) where torch's CPU path uses a <= 1 ULP one, so scores agree to ~1e-6.
// torch.topk leaves the order among equal values unspecified: this kernel takes the LOWEST index (as oracle/port_v8.py does).
#include "common.cuh"

#define TAL_THREADS 256
#define TAL_WARPS (TAL_THREADS / 32)
// iou_calculator / select_candidates_in_gts are called with their own default eps = 1e-9 (nanodet_utils.py:184,206);
// the assigner's `eps` argument (self.eps) only enters the normalisation (tal_assigner.py:72).
#define TAL_HELPER_EPS 1e-9f

struct TalArgs {
  const float* pd_scores;   // [B,A,nc]
  const float* pd_bboxes;   // [B,A,4] xyxy
  const float* anc;         // [A,2]
  const float* gt_labels;   // [B,M]
  const float* gt_bboxes;   // [B,M,4] xyxy
  const float* mask_gt;     // [B,M]
  int32_t B, A, M, nc, topk;
  float alpha, beta, eps;
  long long* t_labels;      // [B,A]
  float* t_bboxes;          // [B,A,4]
  float* t_scores;          // [B,A,nc]
  uint8_t* fg;              // [B,A]
  int32_t* cnt;             // [B,A]  number of gts whose top-k holds this anchor (and whose box contains its centre)
  int32_t* selm;            // [B,A]  the gt index when cnt == 1
  int32_t* tidx;            // [B,A]  target_gt_idx
  float* tmet;              // [B,A]  align_metric[b, target_gt_idx, a] on foreground anchors
  float* pos_align;         // [B,M]  max over the gt's final positives of the metric
  float* pos_ov;            // [B,M]  max over the gt's final positives of the IoU
};

// iou_calculator (nanodet_utils.py:184-204), box1 = gt, box2 = prediction; same operation order, single roundings
// (the library is compiled with --fmad=false).
__device__ __forceinline__ float tal_iou(float gx1, float gy1, float gx2, float gy2, float px1, float py1, float px2, float py2, float eps) {
  const float ix1 = fmaxf(gx1, px1), iy1 = fmaxf(gy1, py1), ix2 = fminf(gx2, px2), iy2 = fminf(gy2, py2);
  const float overlap = fmaxf(ix2 - ix1, 0.f) * fmaxf(iy2 - iy1, 0.f);
  const float area1 = fmaxf(gx2 - gx1, 0.f) * fmaxf(gy2 - gy1, 0.f);
  const float area2 = fmaxf(px2 - px1, 0.f) * fmaxf(py2 - py1, 0.f);
  const float uni = ((area1 + area2) - overlap) + eps;
  return overlap / uni;
}

// bbox_scores.pow(alpha) * overlaps.pow(beta)   (tal_assigner.py:113).  torch returns x itself for an exponent of 1.
__device__ __forceinline__ float tal_pow(float x, float e) {
  if (e == 1.f) return x;
  return (float)pow((double)x, (double)e);
}
__device__ __forceinline__ float tal_metric(float score, float iou, float alpha, float beta) { return tal_pow(score, alpha) * tal_pow(iou, beta); }

// select_candidates_in_gts (nanodet_utils.py:206-225): min(ax-x1, ay-y1, x2-ax, y2-ay) > eps
__device__ __forceinline__ bool tal_in_gt(float ax, float ay, float gx1, float gy1, float gx2, float gy2, float eps) {
  return fminf(fminf(ax - gx1, ay - gy1), fminf(gx2 - ax, gy2 - ay)) > eps;
}

// gt_labels.to(torch.long) used as an index (tal_assigner.py:106-110): negative labels (the -1 of padded rows) wrap like a torch
// index; labels >= nc would raise in torch -- clamped here (a device kernel cannot raise).
__device__ __forceinline__ int tal_label_index(float lab, int nc) {
  int l = (int)lab;
  if (l < 0) l += nc;
  return l < 0 ? 0 : (l >= nc ? nc - 1 : l);
}

// ---------------------------------------------------------------------------------------------------------------------
// K1: one CTA per (gt m, image b).  Shared memory holds align_metric * mask_in_gts for all A anchors; topk rounds of a
// block-wide arg-max (ties -> lowest index) reproduce select_topk_candidates (tal_assigner.py:117-134); the selected anchors
// that lie inside the gt box (mask_topk * mask_in_gts * mask_gt, :97) are counted per anchor.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(TAL_THREADS) tal_topk_kernel(const TalArgs a) {
  extern __shared__ float smet[];
  __shared__ float s_v[TAL_WARPS];
  __shared__ int s_i[TAL_WARPS];
  __shared__ int s_sel;
  const int m = blockIdx.x, b = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (a.mask_gt[(size_t)b * a.M + m] == 0.f) return;      // padded gt: its thirteen picks all collapse onto index 0 and are dropped (:129-134)
  const float* g = a.gt_bboxes + ((size_t)b * a.M + m) * 4;
  const float gx1 = g[0], gy1 = g[1], gx2 = g[2], gy2 = g[3];
  const int label = tal_label_index(a.gt_labels[(size_t)b * a.M + m], a.nc);
  for (int i = tid; i < a.A; i += TAL_THREADS) {
    const float ax = a.anc[2 * i], ay = a.anc[2 * i + 1];
    float v = 0.f;
    if (tal_in_gt(ax, ay, gx1, gy1, gx2, gy2, TAL_HELPER_EPS)) {
      const float4 p = *reinterpret_cast<const float4*>(a.pd_bboxes + ((size_t)b * a.A + i) * 4);
      const float iou = tal_iou(gx1, gy1, gx2, gy2, p.x, p.y, p.z, p.w, TAL_HELPER_EPS);
      v = tal_metric(a.pd_scores[((size_t)b * a.A + i) * a.nc + label], iou, a.alpha, a.beta);
    }
    smet[i] = v;
  }
  __syncthreads();
  for (int r = 0; r < a.topk; ++r) {
    float bv = -2.f;
    int bi = 0x7fffffff;
    for (int i = tid; i < a.A; i += TAL_THREADS) {
      const float v = smet[i];
      if (v > bv) {          // ascending i per thread: the first (lowest) index of equal values stays
        bv = v;
        bi = i;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) {
        bv = ov;
        bi = oi;
      }
    }
    if (lane == 0) {
      s_v[wid] = bv;
      s_i[wid] = bi;
    }
    __syncthreads();
    if (wid == 0) {
      bv = lane < TAL_WARPS ? s_v[lane] : -2.f;
      bi = lane < TAL_WARPS ? s_i[lane] : 0x7fffffff;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) {
          bv = ov;
          bi = oi;
        }
      }
      if (lane == 0) s_sel = bi;
    }
    __syncthreads();
    if (tid == 0) {
      const int sel = s_sel;
      if (sel >= 0 && sel < a.A) {
        if (tal_in_gt(a.anc[2 * sel], a.anc[2 * sel + 1], gx1, gy1, gx2, gy2, TAL_HELPER_EPS)) {
          atomicAdd(a.cnt + (size_t)b * a.A + sel, 1);
          atomicMax(a.selm + (size_t)b * a.A + sel, m);
        }
        smet[sel] = -1.f;      // metrics are >= 0: never picked again
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// K2: one thread per (image, anchor): select_highest_overlaps (nanodet_utils.py:227-248) + get_targets (tal_assigner.py:136-158).
// An anchor claimed by several gts goes to the gt with the highest IoU among ALL gts (first maximum); target_gt_idx = 0 for
// background anchors, so their label / box are those of gt 0 (label clamped at 0), exactly as the reference returns them.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) tal_resolve_kernel(const TalArgs a) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)a.B * a.A) return;
  const int b = (int)(i / a.A);
  const int c = a.cnt[i];
  const float4 p = *reinterpret_cast<const float4*>(a.pd_bboxes + i * 4);
  const float* gts = a.gt_bboxes + (size_t)b * a.M * 4;
  int idx = 0;
  if (c == 1) {
    idx = a.selm[i];
  } else if (c > 1) {
    float best = -1.f;
    for (int m = 0; m < a.M; ++m) {
      const float o = tal_iou(gts[4 * m], gts[4 * m + 1], gts[4 * m + 2], gts[4 * m + 3], p.x, p.y, p.z, p.w, TAL_HELPER_EPS);
      if (o > best) {
        best = o;
        idx = m;
      }
    }
  }
  const float lab_f = a.gt_labels[(size_t)b * a.M + idx];
  long long lab = (long long)lab_f;
  if (lab < 0) lab = 0;                                     // tal_assigner.py:150
  a.t_labels[i] = lab;
  const float gx1 = gts[4 * idx], gy1 = gts[4 * idx + 1], gx2 = gts[4 * idx + 2], gy2 = gts[4 * idx + 3];
  *reinterpret_cast<float4*>(a.t_bboxes + i * 4) = make_float4(gx1, gy1, gx2, gy2);
  a.fg[i] = c > 0 ? 1 : 0;
  a.tidx[i] = idx;
  float met = 0.f;
  if (c > 0) {
    const float o = tal_iou(gx1, gy1, gx2, gy2, p.x, p.y, p.z, p.w, TAL_HELPER_EPS);
    met = tal_metric(a.pd_scores[i * a.nc + tal_label_index(lab_f, a.nc)], o, a.alpha, a.beta);
    // max over the gt's final positives (tal_assigner.py:69-71); non-negative floats order like their bit patterns
    atomicMax(reinterpret_cast<int*>(a.pos_align + (size_t)b * a.M + idx), __float_as_int(met));
    atomicMax(reinterpret_cast<int*>(a.pos_ov + (size_t)b * a.M + idx), __float_as_int(o));
  }
  a.tmet[i] = met;
}

// ---------------------------------------------------------------------------------------------------------------------
// K3: target_scores = one_hot(target_labels) * fg * norm_align_metric  (tal_assigner.py:152-156,68-73), one pass over [B,A,nc].
// With at most one gt per anchor, norm_align_metric[b,a] = metric[b,idx,a] * pos_ov[b,idx] / (pos_align[b,idx] + eps).
// ---------------------------------------------------------------------------------------------------------------------
template <int VEC>
__global__ void __launch_bounds__(256) tal_scores_kernel(const TalArgs a) {
  const int per = a.nc / VEC;                                // vectors per anchor
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)a.B * a.A * per) return;
  const long long i = e / per;
  const int c0 = (int)(e - i * per) * VEC;
  float v[VEC];
#pragma unroll
  for (int k = 0; k < VEC; ++k) v[k] = 0.f;
  if (a.fg[i]) {
    const int lab = (int)a.t_labels[i];
    if (lab >= c0 && lab < c0 + VEC) {
      const int b = (int)(i / a.A);
      const size_t gm = (size_t)b * a.M + a.tidx[i];
      v[lab - c0] = (a.tmet[i] * a.pos_ov[gm]) / (a.pos_align[gm] + a.eps);
    }
  }
  if constexpr (VEC == 4) {
    *reinterpret_cast<float4*>(a.t_scores + i * a.nc + c0) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    a.t_scores[i * a.nc + c0] = v[0];
  }
}

static inline size_t tal_align(size_t x) { return (x + 255) & ~(size_t)255; }

extern "C" size_t etb_tal_workspace_bytes(int32_t B, int32_t A, int32_t M) {
  if (B <= 0 || A <= 0 || M <= 0) return 0;
  const size_t ba = tal_align((size_t)B * A * 4), bm = tal_align((size_t)B * M * 4);
  return 4 * ba + 2 * bm;
}

extern "C" int etb_tal_assign(const float* pd_scores, const float* pd_bboxes, const float* anc_points, const float* gt_labels,
                              const float* gt_bboxes, const float* mask_gt, int32_t B, int32_t A, int32_t M, int32_t nc, int32_t topk,
                              float alpha, float beta, float eps, int64_t* target_labels, float* target_bboxes, float* target_scores,
                              uint8_t* fg_mask, void* workspace, size_t workspace_bytes, void* stream) {
  ETB_CHECK_ARG(pd_scores && pd_bboxes && anc_points && gt_labels && gt_bboxes && mask_gt);
  ETB_CHECK_ARG(target_labels && target_bboxes && target_scores && fg_mask && workspace);
  ETB_CHECK_ARG(B > 0 && A > 0 && M > 0 && nc > 0 && topk > 0 && topk <= A && M <= 65535 && B <= 65535);
  ETB_CHECK_ARG((((uintptr_t)pd_bboxes) & 15) == 0 && (((uintptr_t)target_bboxes) & 15) == 0 && (((uintptr_t)target_scores) & 15) == 0);
  ETB_CHECK_ARG((((uintptr_t)workspace) & 15) == 0 && workspace_bytes >= etb_tal_workspace_bytes(B, A, M));
  const size_t smem = (size_t)A * sizeof(float);
  ETB_CHECK_ARG(smem <= 200 * 1024);                         // A <= 51200 anchors (a 1560 x 1560 image)
  cudaStream_t st = (cudaStream_t)stream;
  const size_t ba = tal_align((size_t)B * A * 4), bm = tal_align((size_t)B * M * 4);
  char* w = (char*)workspace;
  TalArgs a;
  a.pd_scores = pd_scores; a.pd_bboxes = pd_bboxes; a.anc = anc_points; a.gt_labels = gt_labels; a.gt_bboxes = gt_bboxes; a.mask_gt = mask_gt;
  a.B = B; a.A = A; a.M = M; a.nc = nc; a.topk = topk; a.alpha = alpha; a.beta = beta; a.eps = eps;
  a.t_labels = (long long*)target_labels; a.t_bboxes = target_bboxes; a.t_scores = target_scores; a.fg = fg_mask;
  a.cnt = (int32_t*)w; a.selm = (int32_t*)(w + ba); a.tidx = (int32_t*)(w + 2 * ba); a.tmet = (float*)(w + 3 * ba);
  a.pos_align = (float*)(w + 4 * ba); a.pos_ov = (float*)(w + 4 * ba + bm);
  ETB_CHECK_CUDA(cudaMemsetAsync(w, 0, 2 * ba, st));                       // cnt, selm
  ETB_CHECK_CUDA(cudaMemsetAsync(w + 4 * ba, 0, 2 * bm, st));              // pos_align, pos_ov
  if (smem > 48 * 1024) ETB_CHECK_CUDA(cudaFuncSetAttribute(tal_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  etb_launch(tal_topk_kernel, dim3(M, B), dim3(TAL_THREADS), smem, st, a);
  ETB_CHECK_LAUNCH();
  const long long nba = (long long)B * A;
  etb_launch(tal_resolve_kernel, dim3((unsigned)((nba + 255) / 256)), dim3(256), 0, st, a);
  ETB_CHECK_LAUNCH();
  if (nc % 4 == 0) {
    const long long n = nba * (nc / 4);
    etb_launch(tal_scores_kernel<4>, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, a);
  } else {
    const long long n = nba * nc;
    etb_launch(tal_scores_kernel<1>, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, a);
  }
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// etb_v8_decode.  Anchor a of level l (levels concatenated in order, row-major inside a level) sits at grid point
// (x + offset, y + offset) (generate_anchors, nanodet_utils.py:135-182).  Per side: d = sum_k softmax(reg[side])_k * k
// (yolov8_head.py:196-198 / tal_loss.py:151-155).  Outputs, each optional:
//   pred       [B,A,5+nc] : (cx, cy, w, h) * stride, 1, sigmoid(cls)     -- the eval branch's first return value (:211-220)
//   boxes_grid [B,A,4]    : xyxy in grid units   = bbox_decode(anchor_points / stride, pred_distri)      (tal_loss.py:88-89)
//   boxes_pix  [B,A,4]    : boxes_grid * stride  = the assigner's pd_bboxes                               (tal_loss.py:93)
//   scores     [B,A,nc]   : sigmoid(cls)         = the assigner's pd_scores                               (tal_loss.py:92)
// One thread per (anchor, side); the four sides of an anchor are four adjacent lanes.
// ---------------------------------------------------------------------------------------------------------------------
struct V8Args {
  const float* cls;
  const float* reg;
  EtbV8Levels lv;
  int32_t B, A, nc, R;       // R = reg_max + 1 bins
  float offset;
  float* pred;
  float* boxes_grid;
  float* boxes_pix;
  float* scores;
};

__global__ void __launch_bounds__(256) v8_box_kernel(const V8Args a) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // grid is padded to a multiple of 4 threads per anchor
  const long long total = (long long)a.B * a.A * 4;
  const bool live = t < total;
  const long long i = live ? t >> 2 : 0;                                      // (image, anchor)
  const int side = (int)(t & 3);
  float d = 0.f;
  if (live) {
    const float* x = a.reg + (i * 4 + side) * a.R;
    float mx = x[0];
    for (int k = 1; k < a.R; ++k) mx = fmaxf(mx, x[k]);
    float sum = 0.f;
    for (int k = 0; k < a.R; ++k) sum += expf(x[k] - mx);
    for (int k = 0; k < a.R; ++k) d += (expf(x[k] - mx) / sum) * (float)k;
  }
  const int base = (threadIdx.x & 31) & ~3;
  const float l = __shfl_sync(0xffffffffu, d, base), tp = __shfl_sync(0xffffffffu, d, base + 1);
  const float r = __shfl_sync(0xffffffffu, d, base + 2), bt = __shfl_sync(0xffffffffu, d, base + 3);
  if (!live) return;
  int an = (int)(i % a.A), lvl = 0;
  while (lvl + 1 < a.lv.nl && an >= a.lv.h[lvl] * a.lv.w[lvl]) {
    an -= a.lv.h[lvl] * a.lv.w[lvl];
    ++lvl;
  }
  const int gy = an / a.lv.w[lvl], gx = an - gy * a.lv.w[lvl];
  const float s = a.lv.stride[lvl];
  const float px = (float)gx + a.offset, py = (float)gy + a.offset;
  const float x1 = px - l, y1 = py - tp, x2 = px + r, y2 = py + bt;
  const float xyxy = side == 0 ? x1 : (side == 1 ? y1 : (side == 2 ? x2 : y2));
  if (a.boxes_grid) a.boxes_grid[i * 4 + side] = xyxy;
  if (a.boxes_pix) a.boxes_pix[i * 4 + side] = xyxy * s;
  if (a.pred) {
    const float v = side == 0 ? (x1 + x2) / 2.f : (side == 1 ? (y1 + y2) / 2.f : (side == 2 ? x2 - x1 : y2 - y1));   // dist2bbox 'xywh'
    a.pred[i * (5 + a.nc) + side] = v * s;
  }
}

__global__ void __launch_bounds__(256) v8_cls_kernel(const V8Args a) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int per = a.nc + 1;
  if (e >= (long long)a.B * a.A * per) return;
  const long long i = e / per;
  const int c = (int)(e - i * per);
  if (c == 0) {
    if (a.pred) a.pred[i * (5 + a.nc) + 4] = 1.f;
    return;
  }
  const float v = 1.f / (1.f + expf(-a.cls[i * a.nc + (c - 1)]));
  if (a.pred) a.pred[i * (5 + a.nc) + 4 + c] = v;
  if (a.scores) a.scores[i * a.nc + (c - 1)] = v;
}

extern "C" int etb_v8_decode(const float* cls, const float* reg, const EtbV8Levels* levels, int32_t B, int32_t nc, int32_t reg_max,
                             float grid_cell_offset, float* pred, float* boxes_grid, float* boxes_pix, float* scores, void* stream) {
  ETB_CHECK_ARG(reg && levels && B > 0 && nc > 0 && reg_max >= 1 && reg_max <= 63);
  ETB_CHECK_ARG(levels->nl >= 1 && levels->nl <= ETB_MAX_LEVELS);
  ETB_CHECK_ARG(pred || boxes_grid || boxes_pix || scores);
  ETB_CHECK_ARG(cls || !(pred || scores));
  long long A = 0;
  for (int l = 0; l < levels->nl; ++l) {
    ETB_CHECK_ARG(levels->h[l] > 0 && levels->w[l] > 0 && levels->stride[l] > 0.f);
    A += (long long)levels->h[l] * levels->w[l];
  }
  ETB_CHECK_ARG(A * B < (1ll << 31));
  V8Args a;
  a.cls = cls; a.reg = reg; a.lv = *levels; a.B = B; a.A = (int32_t)A; a.nc = nc; a.R = reg_max + 1; a.offset = grid_cell_offset;
  a.pred = pred; a.boxes_grid = boxes_grid; a.boxes_pix = boxes_pix; a.scores = scores;
  cudaStream_t st = (cudaStream_t)stream;
  if (pred || boxes_grid || boxes_pix) {
    const long long n = (long long)B * A * 4;
    etb_launch(v8_box_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, a);
    ETB_CHECK_LAUNCH();
  }
  if (pred || scores) {
    const long long n = (long long)B * A * (nc + 1);
    etb_launch(v8_cls_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, a);
    ETB_CHECK_LAUNCH();
  }
  return ETB_OK;
}
