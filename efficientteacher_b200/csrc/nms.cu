// nms.cu -- teacher post-processing: candidate filter (K7), batched greedy NMS (K8), pseudo-label box
// transform (K9).  Replaces, for all images of the batch in five launches and without a host sync:
//   non_max_suppression_ssod / non_max_suppression   reference utils/general.py:887-992, 994-1098
//   torchvision.ops.nms (call site utils/general.py:976): stable score sort, IoU = inter/(a+b-inter), suppress iff > thr
//   output_to_target_ssod                             reference utils/plots.py:485-491
//   FairPseudoLabel.create_pseudo_label_online_with_gt box warp / filter / normalise / flip
//                                                     reference utils/self_supervised_utils.py:207-232, 414-454, 316-321
// Integer outputs (keep-sets, row order) are bit-exact with the CPU oracle; arithmetic is literal fp32
// (fp64 for the pseudo-label rows, as numpy does) with no FMA contraction (--fmad=false).
//
// Launch sequence (grid sizes are multiples of the SM count or one CTA per image):
//   A1 cand_count : per 1024-row chunk, count rows with obj > conf_thres                 (HBM: 32 B sector / row)
//   A2 cand_write : order-preserving compaction of candidate row indices (chunk prefix)   (same traffic)
//   B  cand_record: one warp per candidate: 85-float row -> [x1,y1,x2,y2,conf,cls,obj,cls_score] + pass flag
//   C1 rank       : stable descending rank by counting (all SMs; O(n^2/SMs))
//   C2 nms_image  : one CTA per image: 64-wide tiles against the kept list (<= max_det) in shared memory,
//                   early exit at max_det; then the float64 pseudo-label transform of the kept rows
//   C3 gather     : image-major concatenation of the pseudo-label rows + total count
#include "common.cuh"

#define NMS_CHUNK 1024
#define NMS_MAXK 1024

struct NmsWs {
  int32_t* chunk_cnt;  // [B, nchunks]
  int32_t* n1;         // [B] candidates after the obj filter
  int32_t* n2;         // [B] candidates after the conf filter
  int32_t* cand_idx;   // [B, P]
  float* rec;          // [B, P, 8]
  float* key;          // [B, P] conf if it passes conf>thr else -inf
  int32_t* sorted;     // [B, P] rank -> candidate slot
  double* pl_seg;      // [B, max_det, 9]
  int32_t* pl_seg_cnt; // [B]
  int32_t nchunks;
};

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

static size_t nms_layout(const EtbNmsParams* p, char* base, NmsWs* ws) {
  const size_t B = p->B, P = p->P;
  const int nchunks = (p->P + NMS_CHUNK - 1) / NMS_CHUNK;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off = align_up(off + bytes, 256);
    return base ? base + o : (char*)nullptr;
  };
  // counters first so one memset clears them
  char* c0 = take(B * sizeof(int32_t));
  char* c1 = take(B * sizeof(int32_t));
  char* c2 = take(B * sizeof(int32_t));
  char* c3 = take(B * nchunks * sizeof(int32_t));
  char* c4 = take(B * P * sizeof(int32_t));
  char* c5 = take(B * P * 8 * sizeof(float));
  char* c6 = take(B * P * sizeof(float));
  char* c7 = take(B * P * sizeof(int32_t));
  char* c8 = take(B * (size_t)p->max_det * 9 * sizeof(double));
  if (ws) {
    ws->n1 = (int32_t*)c0;
    ws->n2 = (int32_t*)c1;
    ws->pl_seg_cnt = (int32_t*)c2;
    ws->chunk_cnt = (int32_t*)c3;
    ws->cand_idx = (int32_t*)c4;
    ws->rec = (float*)c5;
    ws->key = (float*)c6;
    ws->sorted = (int32_t*)c7;
    ws->pl_seg = (double*)c8;
    ws->nchunks = nchunks;
  }
  return off;
}

extern "C" size_t etb_nms_workspace_bytes(const EtbNmsParams* p) {
  if (!p || p->B <= 0 || p->P <= 0) return 0;
  return nms_layout(p, nullptr, nullptr);
}

// ---- A1 / A2 ---------------------------------------------------------------------------------------
__device__ __forceinline__ bool is_candidate(const float* __restrict__ row, int no, float thr, int need_cls) {
  if (!(row[4] > thr)) return false;
  if (need_cls) {  // non_max_suppression: `prediction[..., 5:].max(-1) > conf_thres` too (general.py:1005)
    float m = row[5];
    for (int c = 6; c < no; ++c) m = fmaxf(m, row[c]);
    return m > thr;
  }
  return true;
}

__global__ void __launch_bounds__(256) cand_count_kernel(const float* __restrict__ pred, EtbNmsParams p, NmsWs ws) {
  const int b = blockIdx.y, chunk = blockIdx.x;
  const float* base = pred + (size_t)b * p.P * p.no;
  int cnt = 0;
#pragma unroll
  for (int k = 0; k < NMS_CHUNK / 256; ++k) {
    const int r = chunk * NMS_CHUNK + k * 256 + threadIdx.x;
    if (r < p.P) cnt += is_candidate(base + (size_t)r * p.no, p.no, p.conf_thres, p.need_cls_conf) ? 1 : 0;
  }
  cnt = warp_sum_i(cnt);
  __shared__ int sw[8];
  if ((threadIdx.x & 31) == 0) sw[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += sw[w];
    ws.chunk_cnt[b * ws.nchunks + chunk] = t;
  }
}

__global__ void __launch_bounds__(256) cand_write_kernel(const float* __restrict__ pred, EtbNmsParams p, NmsWs ws) {
  __shared__ int sscan[33];
  __shared__ int sbase;
  const int b = blockIdx.y, chunk = blockIdx.x;
  // prefix of the preceding chunks of this image (<= ~100 values)
  if (threadIdx.x < 32) {
    int s = 0;
    for (int c = threadIdx.x; c < chunk; c += 32) s += ws.chunk_cnt[b * ws.nchunks + c];
    s = warp_sum_i(s);
    if (threadIdx.x == 0) sbase = s;
  }
  __syncthreads();
  int base = sbase;
  const float* pb = pred + (size_t)b * p.P * p.no;
  // rows are visited in order: sub-tile k covers rows [chunk*1024 + k*256, +256)
  for (int k = 0; k < NMS_CHUNK / 256; ++k) {
    const int r = chunk * NMS_CHUNK + k * 256 + threadIdx.x;
    const int f = (r < p.P && is_candidate(pb + (size_t)r * p.no, p.no, p.conf_thres, p.need_cls_conf)) ? 1 : 0;
    int tot;
    const int pos = block_excl_scan(f, sscan, &tot);
    if (f) ws.cand_idx[(size_t)b * p.P + base + pos] = r;
    base += tot;
  }
  if (chunk == ws.nchunks - 1 && threadIdx.x == 0) ws.n1[b] = base;
}

// ---- B ---------------------------------------------------------------------------------------------
// One warp per candidate (grid-stride).  Literal order of operations of general.py:936-953:
//   cls_score = max_c cls_c ; cls_c *= obj ; box = xywh2xyxy ; conf, j = max_c (first maximal index on ties)
__global__ void __launch_bounds__(256) cand_record_kernel(const float* __restrict__ pred, EtbNmsParams p, NmsWs ws) {
  const int lane = threadIdx.x & 31;
  const int warps_per_grid = gridDim.x * (blockDim.x >> 5);
  const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int nc = p.no - 5;
  for (int b = 0; b < p.B; ++b) {
    const int n1 = ws.n1[b];
    for (int i = gw; i < n1; i += warps_per_grid) {
      const int r = ws.cand_idx[(size_t)b * p.P + i];
      const float* row = pred + ((size_t)b * p.P + r) * p.no;
      const float obj = row[4];
      float best = -INFINITY, cmax = -INFINITY;
      int bj = 0x7fffffff;
      for (int c = lane; c < nc; c += 32) {
        const float cv = row[5 + c];
        cmax = fmaxf(cmax, cv);
        const float pv = __fmul_rn(cv, obj);
        if (pv > best) { best = pv; bj = c; }  // ascending c within a lane keeps the first maximum
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
        const float oc = __shfl_xor_sync(0xffffffffu, cmax, o);
        cmax = fmaxf(cmax, oc);
        if (ob > best || (ob == best && oj < bj)) { best = ob; bj = oj; }
      }
      if (lane == 0) {
        const float cx = row[0], cy = row[1], w = row[2], h = row[3];
        const float hw = __fdiv_rn(w, 2.0f), hh = __fdiv_rn(h, 2.0f);
        float* o = ws.rec + ((size_t)b * p.P + i) * 8;
        o[0] = __fsub_rn(cx, hw);
        o[1] = __fsub_rn(cy, hh);
        o[2] = __fadd_rn(cx, hw);
        o[3] = __fadd_rn(cy, hh);
        o[4] = best;
        o[5] = (float)bj;
        o[6] = obj;
        o[7] = cmax;
        const bool pass = best > p.conf_thres;
        ws.key[(size_t)b * p.P + i] = pass ? best : -INFINITY;
        if (pass) atomicAdd(&ws.n2[b], 1);
      }
    }
  }
}

// ---- C1 --------------------------------------------------------------------------------------------
// rank_i = #{ j : key_j > key_i  or (key_j == key_i and j < i) }  == position in a stable descending sort.
__global__ void __launch_bounds__(256) rank_kernel(EtbNmsParams p, NmsWs ws) {
  __shared__ float sk[256];
  const int b = blockIdx.y;
  const int n1 = ws.n1[b];
  const int i0 = blockIdx.x * 256;
  if (i0 >= n1) return;
  const float* key = ws.key + (size_t)b * p.P;
  const int i = i0 + threadIdx.x;
  const float ki = i < n1 ? key[i] : -INFINITY;
  int rank = 0;
  for (int j0 = 0; j0 < n1; j0 += 256) {
    __syncthreads();
    sk[threadIdx.x] = (j0 + threadIdx.x < n1) ? key[j0 + threadIdx.x] : -INFINITY;
    __syncthreads();
    const int lim = min(256, n1 - j0);
    if (j0 + 255 < i0) {  // every j in this tile precedes every i of the block: ties count
      for (int jj = 0; jj < lim; ++jj) rank += (sk[jj] >= ki) ? 1 : 0;
    } else if (j0 > i0 + 255) {  // every j follows: ties do not count
      for (int jj = 0; jj < lim; ++jj) rank += (sk[jj] > ki) ? 1 : 0;
    } else {
      for (int jj = 0; jj < lim; ++jj) {
        const float kj = sk[jj];
        rank += (kj > ki || (kj == ki && (j0 + jj) < i)) ? 1 : 0;
      }
    }
  }
  if (i < n1 && ki > -INFINITY) ws.sorted[(size_t)b * p.P + rank] = i;
}

// ---- C2 --------------------------------------------------------------------------------------------
__device__ __forceinline__ bool iou_gt(float ax1, float ay1, float ax2, float ay2, float aarea, float bx1, float by1,
                                       float bx2, float by2, float barea, float thr) {
  const float xx1 = fmaxf(ax1, bx1), yy1 = fmaxf(ay1, by1);
  const float xx2 = fminf(ax2, bx2), yy2 = fminf(ay2, by2);
  const float w = fmaxf(0.f, __fsub_rn(xx2, xx1)), h = fmaxf(0.f, __fsub_rn(yy2, yy1));
  const float inter = __fmul_rn(w, h);
  const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(aarea, barea), inter));
  return ovr > thr;
}

__global__ void __launch_bounds__(1024) nms_image_kernel(EtbNmsParams p, NmsWs ws, float* __restrict__ det,
                                                         int32_t* __restrict__ det_cnt, const double* __restrict__ Ms) {
  __shared__ float kx1[NMS_MAXK], ky1[NMS_MAXK], kx2[NMS_MAXK], ky2[NMS_MAXK], karea[NMS_MAXK];
  __shared__ int kslot[NMS_MAXK];
  __shared__ float tx1[64], ty1[64], tx2[64], ty2[64], tarea[64];
  __shared__ int tslot[64];
  __shared__ unsigned long long tmask[64];
  __shared__ unsigned long long tsup;
  __shared__ int s_kept;
  __shared__ int sscan[33];
  const int b = blockIdx.x;
  const int tid = threadIdx.x;
  int n = ws.n2[b];
  if (n > p.max_nms) n = p.max_nms;  // general.py:968-969 (argsort-truncate == prefix of the stable sort absent ties)
  const float* rec = ws.rec + (size_t)b * p.P * 8;
  const int32_t* sorted = ws.sorted + (size_t)b * p.P;
  if (tid == 0) s_kept = 0;
  __syncthreads();
  for (int t0 = 0; t0 < n; t0 += 64) {
    const int m = min(64, n - t0);
    if (tid < 64) {
      tmask[tid] = 0ull;
      if (tid < m) {
        const int slot = sorted[t0 + tid];
        const float* r = rec + (size_t)slot * 8;
        const float c = __fmul_rn(r[5], p.max_wh);  // class offset added in fp32 before IoU (general.py:972-973)
        const float x1 = __fadd_rn(r[0], c), y1 = __fadd_rn(r[1], c), x2 = __fadd_rn(r[2], c), y2 = __fadd_rn(r[3], c);
        tx1[tid] = x1; ty1[tid] = y1; tx2[tid] = x2; ty2[tid] = y2;
        tarea[tid] = __fmul_rn(__fsub_rn(x2, x1), __fsub_rn(y2, y1));
        tslot[tid] = slot;
      }
    }
    if (tid == 0) tsup = 0ull;
    __syncthreads();
    const int kept = s_kept;
    const int c = tid & 63, part = tid >> 6;  // 64 candidates x 16 parts
    if (c < m) {
      const float x1 = tx1[c], y1 = ty1[c], x2 = tx2[c], y2 = ty2[c], ar = tarea[c];
      // phase 1: against the boxes kept so far (kept box is the higher-scored `i` of the reference loop)
      bool sup = false;
      for (int k = part; k < kept && !sup; k += 16)
        sup = iou_gt(kx1[k], ky1[k], kx2[k], ky2[k], karea[k], x1, y1, x2, y2, ar, p.iou_thres);
      if (sup) atomicOr(&tsup, 1ull << c);
      // phase 2: intra-tile suppression mask, row c suppresses later j
      unsigned long long mk = 0ull;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = part * 4 + jj;
        if (j > c && j < m && iou_gt(x1, y1, x2, y2, ar, tx1[j], ty1[j], tx2[j], ty2[j], tarea[j], p.iou_thres)) mk |= 1ull << j;
      }
      if (mk) atomicOr(&tmask[c], mk);
    }
    __syncthreads();
    if (tid == 0) {  // phase 3: sequential resolve inside the tile
      unsigned long long removed = tsup;
      int kk = kept;
      for (int q = 0; q < m && kk < p.max_det; ++q) {
        if (!((removed >> q) & 1ull)) {
          kx1[kk] = tx1[q]; ky1[kk] = ty1[q]; kx2[kk] = tx2[q]; ky2[kk] = ty2[q]; karea[kk] = tarea[q];
          kslot[kk] = tslot[q];
          ++kk;
          removed |= tmask[q];
        }
      }
      s_kept = kk;
    }
    __syncthreads();
    if (s_kept >= p.max_det) break;  // general.py:977-978: only the first max_det survivors are used
  }
  const int K = s_kept;
  if (tid == 0) det_cnt[b] = K;
  // detections [x1,y1,x2,y2,conf,cls,obj,cls_score] (un-offset boxes) in score order
  for (int e = tid; e < K * 8; e += blockDim.x) det[((size_t)b * p.max_det) * 8 + e] = rec[(size_t)kslot[e >> 3] * 8 + (e & 7)];
  if (!Ms) return;

  // ---- pseudo-label rows, float64 like numpy (self_supervised_utils.py:207-232) ----
  int valid = 0;
  double row[9];
  if (tid < K) {
    const float* r = rec + (size_t)kslot[tid] * 8;
    // output_to_target_ssod: xyxy2xywh on a float32 array (plots.py:488-490), then widened to float64
    const float fcx = __fdiv_rn(__fadd_rn(r[0], r[2]), 2.0f), fcy = __fdiv_rn(__fadd_rn(r[1], r[3]), 2.0f);
    const float fw = __fsub_rn(r[2], r[0]), fh = __fsub_rn(r[3], r[1]);
    const double cx = fcx, cy = fcy, w = fw, h = fh;
    // xywh2xyxy in float64 (self_supervised_utils.py:213)
    const double x1 = cx - w / 2, y1 = cy - h / 2, x2 = cx + w / 2, y2 = cy + h / 2;
    // M_select = M_s[M_s[:,0] == i][0]
    int mr = -1;
    for (int q = 0; q < p.B; ++q)
      if (Ms[q * 13] == (double)b) { mr = q; break; }
    if (mr >= 0) {
      const double* M = Ms + mr * 13 + 1;
      const double s = Ms[mr * 13 + 10];
      const int ud = (int)Ms[mr * 13 + 11], lr = (int)Ms[mr * 13 + 12];
      // corners x1y1, x2y2, x1y2, x2y1 -> xy @ M.T (affine part)
      const double px[4] = {x1, x2, x1, x2}, py[4] = {y1, y2, y2, y1};
      double mnx = INFINITY, mny = INFINITY, mxx = -INFINITY, mxy = -INFINITY;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const double ox = px[q] * M[0] + py[q] * M[1] + M[2];
        const double oy = px[q] * M[3] + py[q] * M[4] + M[5];
        mnx = fmin(mnx, ox); mxx = fmax(mxx, ox);
        mny = fmin(mny, oy); mxy = fmax(mxy, oy);
      }
      const double W = (double)p.img_w, H = (double)p.img_h;
      const double nx1 = fmin(fmax(mnx, 0.0), W), nx2 = fmin(fmax(mxx, 0.0), W);
      const double ny1 = fmin(fmax(mny, 0.0), H), ny2 = fmin(fmax(mxy, 0.0), H);
      // box_candidates(box1 = xyxy*s, box2 = new, wh_thr=2, ar_thr=20, area_thr=0.1, eps=1e-16)
      const double w1 = x2 * s - x1 * s, h1 = y2 * s - y1 * s;
      const double w2 = nx2 - nx1, h2 = ny2 - ny1;
      const double ar = fmax(w2 / (h2 + 1e-16), h2 / (w2 + 1e-16));
      valid = (w2 > 2.0) && (h2 > 2.0) && (w2 * h2 / (w1 * h1 + 1e-16) > 0.10) && (ar < 20.0);
      double ocx = (nx1 + nx2) / 2, ocy = (ny1 + ny2) / 2, ow = nx2 - nx1, oh = ny2 - ny1;
      ocx /= W; ow /= W; ocy /= H; oh /= H;
      if (ud == 1) ocy = 1 - ocy;
      if (lr == 1) ocx = 1 - ocx;
      row[0] = (double)b; row[1] = (double)r[5];
      row[2] = ocx; row[3] = ocy; row[4] = ow; row[5] = oh;
      row[6] = (double)r[4]; row[7] = (double)r[6]; row[8] = (double)r[7];
    }
  }
  int tot;
  const int pos = block_excl_scan(valid, sscan, &tot);
  if (valid) {
    double* o = ws.pl_seg + ((size_t)b * p.max_det + pos) * 9;
#pragma unroll
    for (int q = 0; q < 9; ++q) o[q] = row[q];
  }
  if (tid == 0) ws.pl_seg_cnt[b] = tot;
}

// ---- C3 --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) pl_gather_kernel(EtbNmsParams p, NmsWs ws, double* __restrict__ pl_rows, int32_t* __restrict__ pl_cnt) {
  int base = 0;
  for (int b = 0; b < p.B; ++b) {
    const int c = ws.pl_seg_cnt[b];
    const double* src = ws.pl_seg + (size_t)b * p.max_det * 9;
    for (int e = threadIdx.x; e < c * 9; e += blockDim.x) pl_rows[(size_t)base * 9 + e] = src[e];
    base += c;
  }
  if (threadIdx.x == 0) *pl_cnt = base;
}

extern "C" int etb_nms_ssod(const float* pred, const EtbNmsParams* p, float* det, int32_t* det_cnt, const double* Ms,
                            double* pl_rows, int32_t* pl_cnt, void* workspace, size_t workspace_bytes, void* stream) {
  ETB_CHECK_ARG(pred && p && det && det_cnt && workspace);
  ETB_CHECK_ARG(p->B > 0 && p->P > 0 && p->no > 5 && p->max_det > 0 && p->max_det <= NMS_MAXK && p->max_nms > 0);
  ETB_CHECK_ARG(Ms == nullptr || (pl_rows && pl_cnt && p->img_h > 0 && p->img_w > 0));
  NmsWs ws;
  const size_t need = nms_layout(p, (char*)workspace, &ws);
  if (need > workspace_bytes) {
    etb_set_error("etb_nms_ssod: workspace too small (%zu < %zu)", workspace_bytes, need);
    return ETB_ERR_NOMEM;
  }
  cudaStream_t st = (cudaStream_t)stream;
  // n1, n2, pl_seg_cnt are contiguous (256 B aligned slots) at the head of the workspace
  ETB_CHECK_CUDA(cudaMemsetAsync(ws.n1, 0, (char*)ws.chunk_cnt - (char*)ws.n1, st));
  dim3 gA(ws.nchunks, p->B);
  etb_launch(cand_count_kernel, dim3(gA), dim3(256), 0, st, pred, *p, ws);
  ETB_CHECK_LAUNCH();
  etb_launch(cand_write_kernel, dim3(gA), dim3(256), 0, st, pred, *p, ws);
  ETB_CHECK_LAUNCH();
  etb_launch(cand_record_kernel, dim3(etb_num_sms() * 4), dim3(256), 0, st, pred, *p, ws);
  ETB_CHECK_LAUNCH();
  dim3 gR((p->P + 255) / 256, p->B);
  etb_launch(rank_kernel, dim3(gR), dim3(256), 0, st, *p, ws);
  ETB_CHECK_LAUNCH();
  etb_launch(nms_image_kernel, dim3(p->B), dim3(1024), 0, st, *p, ws, det, det_cnt, Ms);
  ETB_CHECK_LAUNCH();
  if (Ms) {
    etb_launch(pl_gather_kernel, dim3(1), dim3(1024), 0, st, *p, ws, pl_rows, pl_cnt);
    ETB_CHECK_LAUNCH();
  }
  return ETB_OK;
}

// =====================================================================================================================
// val.py NMS: non_max_suppression(multi_label=True) (reference utils/general.py:994-1098; val.py:149-465 calls it with
// conf_thres 0.001) -- SURVEY.md 8f rank 2.  Every (row, class) PAIR with obj*cls > conf of a candidate row is a detection
// (row-major order of torch.nonzero, general.py:1052); if an image has more than max_nms (30 000) of them only the max_nms
// best by confidence survive (general.py:1071-1072; ties at the cut: the earlier pair, i.e. a stable descending sort).
// Front end (this section) = exact top-max_nms selection without sorting the up to P*nc pairs:
//   V1 ml_hist   x3 : 12+12+8-bit radix histograms of the pair keys (key = fp32 bits of conf: monotonic for conf > 0)
//   V2 ml_select x3 : one block per image walks the histogram from the top: fixes the next digits of the max_nms-th key
//   V3 ml_count     : per 64-row chunk, pairs with key > T and with key == T
//   V4 ml_write     : order-preserving compaction of {key > T} U {first need_eq pairs with key == T} into the record
//                     layout of the SSOD path ([x1,y1,x2,y2,conf,cls,0,0], key = conf)
// then the SAME rank_kernel / nms_image_kernel as the SSOD path run on the <= max_nms survivors.
// Algorithmic bytes: the prediction tensor is read 5 times (340 B/row each); everything else is O(max_nms).
// =====================================================================================================================
#define ML_ROWS 64          // rows per block (8 warps x 8 rows)
#define ML_BINS 4096

struct MlWs {
  uint32_t* hist;       // [B][ML_BINS]
  uint32_t* state;      // [B][8]: 0 prefix (known high bits), 1 k_rem, 2 greater, 3 all (take everything), 4 total pairs
  int32_t* chunk_gt;    // [B][nchunks]
  int32_t* chunk_eq;    // [B][nchunks]
  int32_t nchunks;
};

__device__ __forceinline__ uint32_t ml_key(float obj, float cls, float thr) {
  const float conf = __fmul_rn(cls, obj);
  return conf > thr ? __float_as_uint(conf) : 0u;      // conf > thr >= 0: positive floats order like their bit patterns
}
// is `row` a candidate of general.py:1005 (obj > thr and max cls > thr)?  One warp; all lanes get the answer.
__device__ __forceinline__ bool ml_row_candidate(const float* __restrict__ row, int nc, float thr, int lane) {
  const float obj = row[4];
  if (!(obj > thr)) return false;
  float m = -INFINITY;
  for (int c = lane; c < nc; c += 32) m = fmaxf(m, row[5 + c]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  return m > thr;
}

// level 0: bins = key >> 20 (all valid keys); level 1: (key >> 8) & 0xFFF of keys whose top 12 bits == prefix >> 20;
// level 2: key & 0xFF of keys whose top 24 bits == prefix >> 8.
__global__ void __launch_bounds__(256) ml_hist_kernel(const float* __restrict__ pred, EtbNmsParams p, MlWs ws, int level) {
  __shared__ uint32_t sh[ML_BINS];
  const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nc = p.no - 5;
  if (level > 0 && ws.state[b * 8 + 3]) return;      // everything is taken: no selection needed
  for (int i = threadIdx.x; i < ML_BINS; i += 256) sh[i] = 0;
  __syncthreads();
  const uint32_t prefix = ws.state[b * 8 + 0];
  for (int rr = warp; rr < ML_ROWS; rr += 8) {
    const int r = blockIdx.x * ML_ROWS + rr;
    if (r >= p.P) break;
    const float* row = pred + ((size_t)b * p.P + r) * p.no;
    if (!ml_row_candidate(row, nc, p.conf_thres, lane)) continue;
    const float obj = row[4];
    for (int c = lane; c < nc; c += 32) {
      const uint32_t k = ml_key(obj, row[5 + c], p.conf_thres);
      if (!k) continue;
      if (level == 0) atomicAdd(&sh[k >> 20], 1u);
      else if (level == 1) { if ((k >> 20) == (prefix >> 20)) atomicAdd(&sh[(k >> 8) & 0xFFFu], 1u); }
      else { if ((k >> 8) == (prefix >> 8)) atomicAdd(&sh[k & 0xFFu], 1u); }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < ML_BINS; i += 256)
    if (sh[i]) atomicAdd(&ws.hist[(size_t)b * ML_BINS + i], sh[i]);
}

// One block (256 threads) per image.  Finds, walking the bins from the top, the bin that holds the k_rem-th largest key
// among the keys that match the digits fixed so far; updates prefix / k_rem / greater; clears the histogram for the next level.
__global__ void __launch_bounds__(256) ml_select_kernel(EtbNmsParams p, MlWs ws, int level) {
  __shared__ uint32_t part[256];
  __shared__ int found_bin;
  const int b = blockIdx.x;
  uint32_t* hist = ws.hist + (size_t)b * ML_BINS;
  uint32_t* st = ws.state + b * 8;
  if (level > 0 && st[3]) return;
  const int nb = level == 2 ? 256 : ML_BINS;
  const int per = nb / 256;                           // bins per thread, thread t owns the descending range [nb-1-t*per, ...]
  uint32_t s = 0;
  for (int j = 0; j < per; ++j) s += hist[nb - 1 - (threadIdx.x * per + j)];
  part[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t total = 0;
    for (int t = 0; t < 256; ++t) total += part[t];
    if (level == 0) {
      st[4] = total;
      st[2] = 0;
      st[0] = 0;
      if (total <= (uint32_t)p.max_nms) { st[3] = 1; st[1] = 0; found_bin = -1; }
      else { st[3] = 0; st[1] = (uint32_t)p.max_nms; found_bin = 0; }
    } else {
      found_bin = 0;
    }
    if (found_bin == 0) {
      uint32_t k_rem = st[1], above = 0;
      int bin = -1;
      for (int t = 0; t < 256 && bin < 0; ++t) {
        if (above + part[t] >= k_rem) {
          for (int j = 0; j < per; ++j) {
            const int bb = nb - 1 - (t * per + j);
            const uint32_t h = hist[bb];
            if (above + h >= k_rem) { bin = bb; break; }
            above += h;
          }
        } else {
          above += part[t];
        }
      }
      // bin >= 0 always: total of the matching keys >= k_rem by construction
      st[2] += above;                                  // keys strictly greater than everything in `bin`
      st[1] = k_rem - above;                           // rank of the wanted key inside `bin`
      if (level == 0) st[0] = (uint32_t)bin << 20;
      else if (level == 1) st[0] |= (uint32_t)bin << 8;
      else st[0] |= (uint32_t)bin;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < ML_BINS; i += 256) hist[i] = 0;
}

// selection predicate pieces for one key: gt = key > T (or everything valid when `all`), eq = key == T
__device__ __forceinline__ void ml_class(uint32_t k, uint32_t T, bool all, int* gt, int* eq) {
  *gt = (k != 0u) && (all || k > T);
  *eq = (k != 0u) && !all && k == T;
}

template <bool WRITE>
__global__ void __launch_bounds__(256) ml_pairs_kernel(const float* __restrict__ pred, EtbNmsParams p, MlWs ws, NmsWs nw, int cap) {
  __shared__ int row_gt[ML_ROWS], row_eq[ML_ROWS];
  __shared__ int sbase_gt, sbase_eq;
  const int b = blockIdx.y, chunk = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nc = p.no - 5;
  const uint32_t T = ws.state[b * 8 + 0];
  const bool all = ws.state[b * 8 + 3] != 0;
  const int need_eq = all ? 0 : (int)ws.state[b * 8 + 1];     // after level 2: how many keys == T are taken (the first ones)
  // pass 1: per-row counts
  for (int rr = warp; rr < ML_ROWS; rr += 8) {
    const int r = chunk * ML_ROWS + rr;
    int g = 0, e = 0;
    if (r < p.P) {
      const float* row = pred + ((size_t)b * p.P + r) * p.no;
      if (ml_row_candidate(row, nc, p.conf_thres, lane)) {
        const float obj = row[4];
        for (int c = lane; c < nc; c += 32) {
          int gt, eq;
          ml_class(ml_key(obj, row[5 + c], p.conf_thres), T, all, &gt, &eq);
          g += gt; e += eq;
        }
      }
    }
    g = warp_sum_i(g); e = warp_sum_i(e);
    if (lane == 0) { row_gt[rr] = g; row_eq[rr] = e; }
  }
  __syncthreads();
  if (!WRITE) {
    if (threadIdx.x == 0) {
      int g = 0, e = 0;
      for (int i = 0; i < ML_ROWS; ++i) { g += row_gt[i]; e += row_eq[i]; }
      ws.chunk_gt[b * ws.nchunks + chunk] = g;
      ws.chunk_eq[b * ws.nchunks + chunk] = e;
    }
    return;
  }
  // pass 2 (WRITE): prefix of the preceding chunks, then of the preceding rows, then the ordered write
  if (threadIdx.x < 32) {
    int g = 0, e = 0;
    for (int c = threadIdx.x; c < chunk; c += 32) { g += ws.chunk_gt[b * ws.nchunks + c]; e += ws.chunk_eq[b * ws.nchunks + c]; }
    g = warp_sum_i(g); e = warp_sum_i(e);
    if (threadIdx.x == 0) {
      sbase_gt = g; sbase_eq = e;
      int pg = g, pe = e;                                 // exclusive prefix over the rows of the chunk (64 values: serial is fine)
      for (int i = 0; i < ML_ROWS; ++i) {
        const int tg = row_gt[i], te = row_eq[i];
        row_gt[i] = pg; row_eq[i] = pe;
        pg += tg; pe += te;
      }
      if (chunk == ws.nchunks - 1) {                      // totals of the image
        const int n = pg + (pe < need_eq ? pe : need_eq);
        nw.n1[b] = n;
        nw.n2[b] = n;
      }
    }
  }
  __syncthreads();
  for (int rr = warp; rr < ML_ROWS; rr += 8) {
    const int r = chunk * ML_ROWS + rr;
    if (r >= p.P) break;
    const float* row = pred + ((size_t)b * p.P + r) * p.no;
    if (!ml_row_candidate(row, nc, p.conf_thres, lane)) continue;
    const float obj = row[4];
    int g_before = row_gt[rr], e_before = row_eq[rr];
    const float cx = row[0], cy = row[1], w = row[2], h = row[3];
    const float hw = __fdiv_rn(w, 2.0f), hh = __fdiv_rn(h, 2.0f);
    for (int c0 = 0; c0 < nc; c0 += 32) {                 // classes in ascending order: 32 at a time, ballot prefix inside
      const int c = c0 + lane;
      uint32_t k = 0;
      float conf = 0.f;
      if (c < nc) { conf = __fmul_rn(row[5 + c], obj); k = conf > p.conf_thres ? __float_as_uint(conf) : 0u; }
      int gt, eq;
      ml_class(k, T, all, &gt, &eq);
      const unsigned mg = __ballot_sync(0xffffffffu, gt), me = __ballot_sync(0xffffffffu, eq);
      const unsigned lower = (1u << lane) - 1u;
      const int g_here = g_before + __popc(mg & lower), e_here = e_before + __popc(me & lower);
      int pos = -1;
      if (gt) pos = g_here + (e_here < need_eq ? e_here : need_eq);
      else if (eq && e_here < need_eq) pos = g_here + e_here;
      if (pos >= 0 && pos < cap) {
        float* o = nw.rec + ((size_t)b * cap + pos) * 8;
        o[0] = __fsub_rn(cx, hw);
        o[1] = __fsub_rn(cy, hh);
        o[2] = __fadd_rn(cx, hw);
        o[3] = __fadd_rn(cy, hh);
        o[4] = conf;
        o[5] = (float)c;
        o[6] = obj;
        o[7] = row[5 + c];
        nw.key[(size_t)b * cap + pos] = conf;
      }
      g_before += __popc(mg);
      e_before += __popc(me);
    }
  }
}

static size_t nms_val_layout(const EtbNmsParams* p, int cap, char* base, NmsWs* nw, MlWs* ml) {
  const size_t B = p->B;
  const int nchunks = (p->P + ML_ROWS - 1) / ML_ROWS;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off = align_up(off + bytes, 256);
    return base ? base + o : (char*)nullptr;
  };
  char* c0 = take(B * sizeof(int32_t));                    // n1
  char* c1 = take(B * sizeof(int32_t));                    // n2
  char* c2 = take(B * sizeof(int32_t));                    // pl_seg_cnt (unused here, kept so the kernels see valid pointers)
  char* h0 = take(B * ML_BINS * sizeof(uint32_t));         // hist   } zeroed together with the counters
  char* s0 = take(B * 8 * sizeof(uint32_t));               // state  }
  char* g0 = take(B * (size_t)nchunks * sizeof(int32_t));
  char* e0 = take(B * (size_t)nchunks * sizeof(int32_t));
  char* r0 = take(B * (size_t)cap * 8 * sizeof(float));
  char* k0 = take(B * (size_t)cap * sizeof(float));
  char* o0 = take(B * (size_t)cap * sizeof(int32_t));
  char* p0 = take(B * (size_t)p->max_det * 9 * sizeof(double));
  if (nw && ml) {
    nw->n1 = (int32_t*)c0; nw->n2 = (int32_t*)c1; nw->pl_seg_cnt = (int32_t*)c2;
    nw->chunk_cnt = (int32_t*)g0; nw->cand_idx = nullptr;
    nw->rec = (float*)r0; nw->key = (float*)k0; nw->sorted = (int32_t*)o0; nw->pl_seg = (double*)p0;
    nw->nchunks = nchunks;
    ml->hist = (uint32_t*)h0; ml->state = (uint32_t*)s0; ml->chunk_gt = (int32_t*)g0; ml->chunk_eq = (int32_t*)e0;
    ml->nchunks = nchunks;
  }
  return off;
}
static int nms_val_cap(const EtbNmsParams* p) {
  const long pairs = (long)p->P * (p->no - 5);
  return (int)(pairs < p->max_nms ? pairs : p->max_nms);
}

extern "C" size_t etb_nms_val_workspace_bytes(const EtbNmsParams* p) {
  if (!p || p->B <= 0 || p->P <= 0 || p->no <= 5 || p->max_nms <= 0) return 0;
  return nms_val_layout(p, nms_val_cap(p), nullptr, nullptr, nullptr);
}

// det [B,max_det,8] rows [x1,y1,x2,y2,conf,cls,obj,cls_score] (the caller keeps columns 0..5), det_cnt [B].
extern "C" int etb_nms_val(const float* pred, const EtbNmsParams* p, float* det, int32_t* det_cnt, void* workspace,
                           size_t workspace_bytes, void* stream) {
  ETB_CHECK_ARG(pred && p && det && det_cnt && workspace);
  ETB_CHECK_ARG(p->B > 0 && p->P > 0 && p->no > 6 && p->max_det > 0 && p->max_det <= NMS_MAXK && p->max_nms > 0 && p->conf_thres >= 0.f);
  const int cap = nms_val_cap(p);
  NmsWs nw;
  MlWs ml;
  const size_t need = nms_val_layout(p, cap, (char*)workspace, &nw, &ml);
  if (need > workspace_bytes) {
    etb_set_error("etb_nms_val: workspace too small (%zu < %zu)", workspace_bytes, need);
    return ETB_ERR_NOMEM;
  }
  cudaStream_t st = (cudaStream_t)stream;
  ETB_CHECK_CUDA(cudaMemsetAsync(nw.n1, 0, (char*)ml.chunk_gt - (char*)nw.n1, st));      // counters, histogram, state
  dim3 gC(ml.nchunks, p->B);
  for (int level = 0; level < 3; ++level) {
    etb_launch(ml_hist_kernel, dim3(gC), dim3(256), 0, st, pred, *p, ml, level);
    ETB_CHECK_LAUNCH();
    etb_launch(ml_select_kernel, dim3(p->B), dim3(256), 0, st, *p, ml, level);
    ETB_CHECK_LAUNCH();
  }
  etb_launch(ml_pairs_kernel<false>, dim3(gC), dim3(256), 0, st, pred, *p, ml, nw, cap);
  ETB_CHECK_LAUNCH();
  etb_launch(ml_pairs_kernel<true>, dim3(gC), dim3(256), 0, st, pred, *p, ml, nw, cap);
  ETB_CHECK_LAUNCH();
  EtbNmsParams q = *p;
  q.P = cap;                                               // the survivors live in [B][cap] record / key / sorted arrays
  dim3 gR((cap + 255) / 256, p->B);
  etb_launch(rank_kernel, dim3(gR), dim3(256), 0, st, q, nw);
  ETB_CHECK_LAUNCH();
  etb_launch(nms_image_kernel, dim3(p->B), dim3(1024), 0, st, q, nw, det, det_cnt, nullptr);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
