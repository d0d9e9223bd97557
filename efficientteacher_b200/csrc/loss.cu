// loss.cu -- fused detection losses, forward + hand-written backward (K12/K13).
//   ComputeLoss.default_loss               reference models/loss/loss.py:138-208
//   ComputeStudentMatchLoss.default_loss   reference models/loss/ssod/ssod_loss.py:194-288
//   bbox_iou (CIoU)                        reference utils/metrics.py:207-249
// Replaces ~150-200 ATen launches per call (advanced-index gather, sigmoid, pow, ~25 elementwise CIoU ops,
// index_put_, one-hot fill, 2x BCEWithLogits per level) by 4 launches forward / 2 backward, with the target
// counts read from device memory (no host sync between the assigner and the loss).
//
// Duplicate (b,a,gj,gi) cells in `tobj[b,a,gj,gi] = iou` resolve to the HIGHEST ROW INDEX, which is what the
// reference's CPU index_put_ does (SURVEY.md Appendix C #8); uncertain soft labels override certain ones
// because the reference writes them later (ssod_loss.py:242-248).
//
// Loss options (cfg.Loss.cls_pw / obj_pw / fl_gamma, loss.py:106-116) change only the per-element criterion
// (etb_det_bce in loss_math.h); autobalance (loss.py:191-197) keeps its double balance state on the device and
// advances it in loss_finalize_kernel, so no call reads anything back to the host.
//
// HBM traffic (algorithmic): forward reads one objectness logit per cell (32 B sector each, B*P*32 B) plus
// 85 floats per matched row; backward writes the dense gradient once (B*P*no*4 B).
#include "common.cuh"
#include "loss_math.h"

struct LossSets {
  const int32_t* idx[4][ETB_MAX_LEVELS];
  const float* tbox[4][ETB_MAX_LEVELS];
  const float* anch[4][ETB_MAX_LEVELS];
  const int32_t* tcls[4][ETB_MAX_LEVELS];
  const float* tscore[4][ETB_MAX_LEVELS];
  const int32_t* cnt[4];
  int32_t cap[4];
};

struct LossWs {
  double* acc;        // [nl][8]
  int32_t* winner_c;  // [cells_total]
  int32_t* winner_u;  // [cells_total]
  float* iou0;        // [nl][cap0]
  float* bal_used;    // [nl] autobalance: the float32 balance this call's forward used, for its backward
  int64_t cell_off[ETB_MAX_LEVELS + 1];
  int32_t cap0;
};

struct LossPtrs {
  const float* p[ETB_MAX_LEVELS];
  float* g[ETB_MAX_LEVELS];
};

static size_t lalign(size_t x) { return (x + 255) / 256 * 256; }

static size_t loss_layout(const EtbLossParams* lp, int32_t cap, char* base, LossWs* ws) {
  int64_t cells = 0;
  int64_t off[ETB_MAX_LEVELS + 1];
  for (int l = 0; l < lp->nl; ++l) {
    off[l] = cells;
    cells += (int64_t)lp->B * lp->na * lp->ny[l] * lp->nx[l];
  }
  off[lp->nl] = cells;
  size_t o = 0;
  size_t o_acc = o; o = lalign(o + sizeof(double) * 8 * ETB_MAX_LEVELS);
  size_t o_wc = o;  o = lalign(o + sizeof(int32_t) * cells);
  size_t o_wu = o;  o = lalign(o + sizeof(int32_t) * cells);
  size_t o_iou = o; o = lalign(o + sizeof(float) * (size_t)cap * lp->nl);
  size_t o_bal = o; o = lalign(o + sizeof(float) * lp->nl);
  if (ws) {
    ws->acc = (double*)(base + o_acc);
    ws->winner_c = (int32_t*)(base + o_wc);
    ws->winner_u = (int32_t*)(base + o_wu);
    ws->iou0 = (float*)(base + o_iou);
    ws->bal_used = (float*)(base + o_bal);
    for (int l = 0; l <= lp->nl; ++l) ws->cell_off[l] = off[l];
    ws->cap0 = cap;
  }
  return o;
}

extern "C" size_t etb_loss_workspace_bytes(const EtbLossParams* lp, int32_t cap) {
  if (!lp || lp->nl < 1 || lp->nl > ETB_MAX_LEVELS || cap < 0) return 0;
  return loss_layout(lp, cap, nullptr, nullptr);
}

static int pack_sets(const EtbLossParams* lp, const EtbAssignOut* sets, LossSets* S) {
  memset(S, 0, sizeof(*S));
  for (int s = 0; s < lp->nsets; ++s) {
    for (int l = 0; l < lp->nl; ++l) {
      S->idx[s][l] = sets[s].idx[l];
      S->tbox[s][l] = sets[s].tbox[l];
      S->anch[s][l] = sets[s].anch[l];
      S->tcls[s][l] = sets[s].tcls[l];
      S->tscore[s][l] = sets[s].tscore[l];
    }
    S->cnt[s] = sets[s].cnt;
    S->cap[s] = sets[s].cap;
    if (!sets[s].cnt) return -1;
  }
  return 0;
}

__device__ __forceinline__ int64_t cell_index(const EtbLossParams& lp, int l, const int32_t* idx4) {
  // ((b*na + a)*ny + gj)*nx + gi
  return (((int64_t)idx4[0] * lp.na + idx4[1]) * lp.ny[l] + idx4[2]) * lp.nx[l] + idx4[3];
}

// -------------------------------------------------------------------------------------------------
// rows kernel (forward when BWD=false, backward when BWD=true): one warp per matched row, grid-stride.
// -------------------------------------------------------------------------------------------------
template <bool BWD>
__global__ void __launch_bounds__(256) loss_rows_kernel(LossPtrs P, EtbLossParams lp, LossSets S, LossWs ws, const float* __restrict__ gscale_dev) {
  const int lane = threadIdx.x & 31;
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  const int gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int nc = lp.no - 5;
  float gs = 1.0f;
  if (BWD) gs = gscale_dev ? *gscale_dev : 1.0f;
  for (int s = 0; s < lp.nsets; ++s) {
    if (s == 2 && !lp.with_bbox) continue;
    if (s == 3 && !lp.with_cls) continue;
    if (BWD && s == 1) continue;
    const bool do_box = (s == 0 || s == 2), do_cls = (s == 0 || s == 3) && nc > 1;
    for (int l = 0; l < lp.nl; ++l) {
      int n = S.cnt[s][l];
      if (n > S.cap[s]) n = S.cap[s];
      const float* __restrict__ p = P.p[l];
      for (int r = gw; r < n; r += nwarps) {
        const int32_t* id = S.idx[s][l] + 4 * (size_t)r;
        const int64_t cell = cell_index(lp, l, id);
        if (s == 1) {  // uncertain: only claims the cell for the soft objectness label
          if (lane == 0) atomicMax(&ws.winner_u[ws.cell_off[l] + cell], r);
          continue;
        }
        const float* ps = p + cell * lp.no;
        float box_g[4] = {0.f, 0.f, 0.f, 0.f};
        float ciou = 0.f;
        if (do_box) {
          float lg[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) lg[k] = ps[k];
          const float* tb = S.tbox[s][l] + 4 * (size_t)r;
          const float tbv[4] = {tb[0], tb[1], tb[2], tb[3]};
          const float aw = S.anch[s][l][2 * (size_t)r], ah = S.anch[s][l][2 * (size_t)r + 1];
          ciou = etb_row_ciou(lg, aw, ah, tbv, BWD ? box_g : nullptr);
        }
        if (!BWD) {
          float csum = 0.f;
          if (do_cls) {
            const int tc = S.tcls[s][l][r];
            for (int c = lane; c < nc; c += 32) csum += etb_det_bce(ps[5 + c], c == tc ? lp.cp : lp.cn, lp.cls_pw, lp.fl_gamma);
            csum = warp_sum(csum);
          }
          if (lane == 0) {
            if (do_box) atomicAdd(&ws.acc[l * 8 + (s == 0 ? 0 : 2)], (double)(1.0f - ciou));
            if (do_cls) atomicAdd(&ws.acc[l * 8 + (s == 0 ? 1 : 3)], (double)csum);
            if (s == 0) {
              ws.iou0[(size_t)l * ws.cap0 + r] = ciou;
              atomicMax(&ws.winner_c[ws.cell_off[l] + cell], r);
            }
          }
        } else {
          float* g = P.g[l] + cell * lp.no;
          const float bs = (float)lp.B;
          if (do_box && lane < 4) {
            // L = box_w * B * mean_r(1 - ciou)  =>  dL/dl = -box_w*B/n * dciou/dl
            const float k = -lp.box_w * bs / (float)n * gs;
            atomicAdd(g + lane, k * box_g[lane]);
          }
          if (do_cls) {
            const int tc = S.tcls[s][l][r];
            const float k = lp.cls_w * bs / ((float)n * (float)nc) * gs;
            for (int c = lane; c < nc; c += 32) {
              const float x = ps[5 + c];
              atomicAdd(g + 5 + c, k * etb_det_bce_grad(x, c == tc ? lp.cp : lp.cn, lp.cls_pw, lp.fl_gamma));
            }
          }
        }
      }
    }
  }
}

// target objectness of a cell: uncertain soft label (or ignore = -1) overrides clamp(iou,0) overrides 0
__device__ __forceinline__ float cell_tobj(const EtbLossParams& lp, const LossSets& S, const LossWs& ws, int l, int64_t cell) {
  if (lp.nsets > 1) {
    const int wu = ws.winner_u[ws.cell_off[l] + cell];
    if (wu >= 0) return lp.ignore_obj ? -1.0f : S.tscore[1][l][wu];
  }
  const int wc = ws.winner_c[ws.cell_off[l] + cell];
  if (wc >= 0) return fmaxf(ws.iou0[(size_t)l * ws.cap0 + wc], 0.0f);  // iou.detach().clamp(0)
  return 0.0f;
}

__global__ void __launch_bounds__(256) loss_obj_fwd_kernel(LossPtrs P, EtbLossParams lp, LossSets S, LossWs ws) {
  __shared__ float ssum[8];
  __shared__ float scnt[8];
  const int l = blockIdx.y;
  const int64_t ncell = ws.cell_off[l + 1] - ws.cell_off[l];
  const float* __restrict__ p = P.p[l];
  float sum = 0.f, cnt = 0.f;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < ncell; c += (int64_t)gridDim.x * blockDim.x) {
    const float t = cell_tobj(lp, S, ws, l, c);
    if (t >= 0.0f) {
      sum += etb_det_bce(p[c * lp.no + 4], t, lp.obj_pw, lp.fl_gamma);
      cnt += 1.0f;
    }
  }
  sum = warp_sum(sum);
  cnt = warp_sum(cnt);
  if ((threadIdx.x & 31) == 0) { ssum[threadIdx.x >> 5] = sum; scnt[threadIdx.x >> 5] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, b = 0.0;
    for (int w = 0; w < 8; ++w) { a += ssum[w]; b += scnt[w]; }
    atomicAdd(&ws.acc[l * 8 + 4], a);
    atomicAdd(&ws.acc[l * 8 + 5], b);
  }
}

__global__ void loss_finalize_kernel(EtbLossParams lp, LossSets S, LossWs ws, float* __restrict__ out4) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int nc = lp.no - 5;
  // fp32 accumulation in the reference's order: lbox += mean ; lobj += mean*balance ; then the weights
  float lbox = 0.f, lobj = 0.f, lcls = 0.f;
  for (int l = 0; l < lp.nl; ++l) {
    const int n0 = min(S.cnt[0][l], S.cap[0]);
    if (n0 > 0) {
      lbox += (float)(ws.acc[l * 8 + 0] / (double)n0);
      if (nc > 1) lcls += (float)(ws.acc[l * 8 + 1] / ((double)n0 * nc));
    }
    if (lp.nsets > 1) {
      if (lp.with_bbox) {
        const int n2 = min(S.cnt[2][l], S.cap[2]);
        if (n2 > 0) lbox += (float)(ws.acc[l * 8 + 2] / (double)n2);
      }
      if (lp.with_cls && nc > 1) {
        const int n3 = min(S.cnt[3][l], S.cap[3]);
        if (n3 > 0) lcls += (float)(ws.acc[l * 8 + 3] / ((double)n3 * nc));
      }
    }
    const float obji = (float)(ws.acc[l * 8 + 4] / ws.acc[l * 8 + 5]);
    float bal = lp.balance[l];
    if (lp.balance_state) {
      // autobalance (loss.py:191-193): lobj uses the balance from before the update, as a float32 scalar; the
      // update runs in double, unfused, as Python evaluates it: b = b*0.9999 + 0.0001/obji
      bal = (float)lp.balance_state[l];
      ws.bal_used[l] = bal;
      lp.balance_state[l] = __dadd_rn(__dmul_rn(lp.balance_state[l], 0.9999), __ddiv_rn(0.0001, (double)obji));
    }
    lobj += obji * bal;
  }
  if (lp.balance_state) {  // loss.py:195-196: every entry divided by the stride-16 level's
    const double d = lp.balance_state[lp.ssi];
    for (int l = 0; l < lp.nl; ++l) lp.balance_state[l] = __ddiv_rn(lp.balance_state[l], d);
  }
  lbox *= lp.box_w;
  lobj *= lp.obj_w;
  lcls *= lp.cls_w;
  out4[0] = lbox;
  out4[1] = lobj;
  out4[2] = lcls;
  out4[3] = (lbox + lobj + lcls) * (float)lp.B;
}

// backward of the objectness term + dense zero-fill of every other element: one thread per element,
// fully coalesced stores.  dL/dx4 = obj_w * B * balance_l / n_valid_l * d crit(x, tobj)/dx for valid cells
// (crit = etb_det_bce: sigmoid(x) - tobj with the default options).
__global__ void __launch_bounds__(256) loss_obj_bwd_kernel(LossPtrs P, EtbLossParams lp, LossSets S, LossWs ws, const float* __restrict__ gscale_dev) {
  const int l = blockIdx.y;
  const int64_t ncell = ws.cell_off[l + 1] - ws.cell_off[l];
  const int64_t nel = ncell * lp.no;
  const float* __restrict__ p = P.p[l];
  float* __restrict__ g = P.g[l];
  const float gs = gscale_dev ? *gscale_dev : 1.0f;
  const float bal = lp.balance_state ? ws.bal_used[l] : lp.balance[l];
  const float k = lp.obj_w * (float)lp.B * bal / (float)ws.acc[l * 8 + 5] * gs;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nel; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t c = e / lp.no;
    const int ch = (int)(e - c * lp.no);
    float v = 0.f;
    if (ch == 4) {
      const float t = cell_tobj(lp, S, ws, l, c);
      if (t >= 0.0f) v = k * etb_det_bce_grad(p[e], t, lp.obj_pw, lp.fl_gamma);
    }
    g[e] = v;
  }
}

static int loss_common(const float* const* p, const EtbLossParams* lp, const EtbAssignOut* sets, void* workspace,
                       size_t workspace_bytes, LossPtrs* P, LossSets* S, LossWs* ws) {
  ETB_CHECK_ARG(p && lp && sets && workspace);
  ETB_CHECK_ARG(lp->nl >= 1 && lp->nl <= ETB_MAX_LEVELS && lp->B > 0 && lp->na > 0 && lp->no > 5);
  ETB_CHECK_ARG(lp->nsets == 1 || lp->nsets == 4);
  ETB_CHECK_ARG(lp->fl_gamma >= 0.0f && lp->ssi >= 0 && lp->ssi < lp->nl);
  ETB_CHECK_ARG(pack_sets(lp, sets, S) == 0);
  const size_t need = loss_layout(lp, sets[0].cap, (char*)workspace, ws);
  if (need > workspace_bytes) {
    etb_set_error("etb_loss: workspace too small (%zu < %zu)", workspace_bytes, need);
    return ETB_ERR_NOMEM;
  }
  for (int l = 0; l < lp->nl; ++l) {
    ETB_CHECK_ARG(p[l] != nullptr);
    P->p[l] = p[l];
    P->g[l] = nullptr;
  }
  return ETB_OK;
}

extern "C" int etb_loss_forward(const float* const* p, const EtbLossParams* lp, const EtbAssignOut* sets, float* out4,
                                void* workspace, size_t workspace_bytes, void* stream) {
  LossPtrs P;
  LossSets S;
  LossWs ws;
  int rc = loss_common(p, lp, sets, workspace, workspace_bytes, &P, &S, &ws);
  if (rc != ETB_OK) return rc;
  ETB_CHECK_ARG(out4 != nullptr);
  cudaStream_t st = (cudaStream_t)stream;
  ETB_CHECK_CUDA(cudaMemsetAsync(ws.acc, 0, sizeof(double) * 8 * ETB_MAX_LEVELS, st));
  // winner_c and winner_u are adjacent: one memset to -1 (0xFF bytes)
  ETB_CHECK_CUDA(cudaMemsetAsync(ws.winner_c, 0xFF, (char*)ws.iou0 - (char*)ws.winner_c, st));
  const int sms = etb_num_sms();
  etb_launch(loss_rows_kernel<false>, dim3(sms * 2), dim3(256), 0, st, P, *lp, S, ws, nullptr);
  ETB_CHECK_LAUNCH();
  dim3 go(sms * 2, lp->nl);
  etb_launch(loss_obj_fwd_kernel, dim3(go), dim3(256), 0, st, P, *lp, S, ws);
  ETB_CHECK_LAUNCH();
  etb_launch(loss_finalize_kernel, dim3(1), dim3(32), 0, st, *lp, S, ws, out4);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// Must follow etb_loss_forward on the same workspace (it reuses the winners, iou rows and valid-cell counts).
extern "C" int etb_loss_backward(const float* const* p, float* const* grad_p, const EtbLossParams* lp,
                                 const EtbAssignOut* sets, const float* gscale_dev, void* workspace, size_t workspace_bytes,
                                 void* stream) {
  LossPtrs P;
  LossSets S;
  LossWs ws;
  int rc = loss_common(p, lp, sets, workspace, workspace_bytes, &P, &S, &ws);
  if (rc != ETB_OK) return rc;
  ETB_CHECK_ARG(grad_p != nullptr);
  for (int l = 0; l < lp->nl; ++l) {
    ETB_CHECK_ARG(grad_p[l] != nullptr);
    P.g[l] = grad_p[l];
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int sms = etb_num_sms();
  dim3 go(sms * 8, lp->nl);
  etb_launch(loss_obj_bwd_kernel, dim3(go), dim3(256), 0, st, P, *lp, S, ws, gscale_dev);
  ETB_CHECK_LAUNCH();
  etb_launch(loss_rows_kernel<true>, dim3(sms * 2), dim3(256), 0, st, P, *lp, S, ws, gscale_dev);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// ---- standalone bbox_iou (CIoU, xywh, 1-to-1): reference utils/metrics.py:207-249 ----
__global__ void bbox_ciou_kernel(const float* __restrict__ b1, const float* __restrict__ b2, int n, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 a = reinterpret_cast<const float4*>(b1)[i], b = reinterpret_cast<const float4*>(b2)[i];
  out[i] = etb_ciou(a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, nullptr);
}

extern "C" int etb_bbox_ciou(const float* box1, const float* box2, int32_t n, float* out, void* stream) {
  ETB_CHECK_ARG(n >= 0);
  if (n == 0) return ETB_OK;
  ETB_CHECK_ARG(box1 && box2 && out);
  etb_launch(bbox_ciou_kernel, dim3((n + 255) / 256), dim3(256), 0, (cudaStream_t)stream, box1, box2, n, out);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
