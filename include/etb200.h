/*
 * etb200.h -- C ABI of libetb200.so, the H100 (sm_90a) kernels behind the EfficientTeacher SSOD step.
 *
 * The reference (AlibabaResearch/efficientteacher) is pure Python and has no FFI of its own
 * (SURVEY.md section 2.1), so every entry point below replaces a *library call made from Python*;
 * the reference call site each one stands in for is cited as file:line relative to the reference root.
 * INTEGRATION.md shows the ctypes binding a maintainer would add on the reference side.
 *
 * Conventions
 *  - plain C types only: raw device pointers, sizes, scalars, `void* stream` (a cudaStream_t).
 *  - the caller owns every buffer (allocated as torch tensors or cudaMalloc); the library never
 *    allocates or frees user-visible memory.  Scratch comes in through explicit workspace pointers
 *    whose size is returned by the matching *_workspace_bytes() query.
 *  - every launch goes to the stream passed in; nothing synchronises the device.
 *  - return value: 0 on success, negative errno-style code otherwise; etb_last_error() gives text.
 *    Errors are never thrown across the ABI.
 *  - there is NO CPU fallback: every compute entry point returns ETB_ERR_CUDA if no sm_90 device
 *    kernel image can run.
 */
#ifndef ETB200_H_
#define ETB200_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ETB_OK 0
#define ETB_ERR_INVALID (-22) /* EINVAL  */
#define ETB_ERR_CUDA (-5)     /* EIO: a CUDA runtime call / launch failed */
#define ETB_ERR_NOMEM (-12)   /* workspace too small */

#define ETB_MAX_LEVELS 3
#define ETB_NA 3 /* anchors per level */

int etb_version(void);
const char* etb_last_error(void);
/* kernels launched by this library in this process so far (bench.py: gpu_launches = delta per timed region) */
long long etb_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * Multi-tensor updates: the EMA, SGD and AdamW below each update every tensor of a list in ONE launch.
 * The host splits each tensor into chunks of at most ETB_CHUNK floats and uploads one EtbChunk per chunk;
 * the kernel runs one 256-thread block per chunk, with float4 accesses when every stream it uses is 16 B
 * aligned.  t[] holds up to four streams, in the order each entry point documents; each block reads its
 * per-group fp32 scalars from device memory at hyper_dev[W*group], so a captured CUDA graph replays with
 * whatever the host wrote there last (schedule, warm-up, decays, bias corrections).
 * ------------------------------------------------------------------------------------------- */
typedef struct EtbChunk {
  float* t[4];    /* the chunk's slice of each stream, NULL for an unused one */
  int32_t n;      /* elements in this chunk (<= ETB_CHUNK) */
  int32_t group;  /* index of the chunk's scalars in hyper_dev */
} EtbChunk;
#define ETB_CHUNK 4096

/* EMA  (replaces the per-tensor Python loop of ModelEMA / SemiSupModelEMA / CosineEMA .update,
 *       utils/torch_utils.py:328-338, 364-375, 405-416; called from trainer/ssod_trainer.py:485-487)
 * streams {v, m, s or NULL, unused}; hyper_dev[0..3] = {d, 1-d, d2, 1-d2} (W = 4, group 0):
 *   v <- fl32(fl32(v*d) + fl32(fl32(1-d)*m))            (two roundings, no FMA: bit-exact with torch CPU)
 * and, when the chunk has a second EMA `s` (the SSOD "semi" EMA of the EMA),
 *   s <- fl32(fl32(s*d2) + fl32(fl32(1-d2)*v_new))      in the same pass (5 HBM streams instead of 6). */
int etb_ema_update(const EtbChunk* table_dev, int64_t n_chunks, const float* hyper_dev, void* stream);

/* Fused SGD-Nesterov step over all parameters (replaces torch.optim.SGD.step + zero_grad behind
 * trainer/ssod_trainer.py:481-484; groups/hyper-parameters as built in trainer/trainer.py:193-217):
 *   g' = g + wd*p ; buf = momentum*buf + g' ; p -= lr*(g' + momentum*buf) ; (g = 0)
 * streams {p, g, buf, unused}; hyper_dev[4*group + {0,1,2}] = {lr, momentum, wd} (W = 4). */
int etb_sgd_step(const EtbChunk* table_dev, int64_t n_chunks, const float* hyper_dev, int32_t zero_grad, void* stream);

/* Fused AdamW step over all parameters for `adam: True` (replaces torch.optim.AdamW.step + zero_grad; optimizer built in
 * trainer/trainer.py:211-217: AdamW(g_b, lr=lr0, betas=(momentum, 0.999)) + conv-weight and BN-weight groups), the same
 * arithmetic as torch's foreach AdamW (decoupled weight decay):
 *   p *= 1-lr*wd ; m = lerp(m, g, 1-b1) ; v = v*b2 + (1-b2)*g*g ; p += (-lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps) ; (g = 0)
 * streams {p, g, m = exp_avg, v = exp_avg_sq}; hyper_dev[8*group + 0..6] = {1-lr*wd, 1-b1, b2, 1-b2, -lr/bc1, sqrt(bc2),
 * eps} (W = 8), computed on the host in float64 and rounded once to fp32. */
int etb_adamw_step(const EtbChunk* table_dev, int64_t n_chunks, const float* hyper_dev, int32_t zero_grad, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Detect eval-mode decode (models/head/yolov5_head.py:66-78): logits [B,na,ny,nx,no] of one level ->
 * rows of pred[B,P,no] at row offset `row0`:  sigmoid; xy=(2s-0.5+grid)*stride; wh=(2s)^2*anchor*stride.
 * ------------------------------------------------------------------------------------------- */
int etb_detect_decode(const float* logits, float* pred, int32_t B, int32_t na, int32_t ny, int32_t nx,
                      int32_t no, int32_t P_total, int32_t row0, const float* anchors_grid /*[na*2] host*/,
                      float stride, void* stream);

/* ---------------------------------------------------------------------------------------------
 * non_max_suppression_ssod + output_to_target_ssod + FairPseudoLabel box transform
 * (utils/general.py:887-992; utils/plots.py:485-491; utils/self_supervised_utils.py:194-245,414-454,316-321)
 *
 * pred [B,P,no] fp32 (decoded), multi_label=False path.  All images in one batch of launches, no host sync.
 *   det      [B,max_det,8] fp32  rows [x1,y1,x2,y2,conf,cls,obj,cls_score] in NMS score order
 *   det_cnt  [B] int32
 *   When Ms != NULL (B x 13 doubles: [img, M(9 row-major), s, ud, lr], utils/datasets_ssod.py:989) the
 *   pseudo-label rows [img,cls,cx,cy,w,h,conf,obj,cls_score] (float64, normalised, strong-aug frame) are
 *   written image-major to pl_rows[B*max_det,9] and their number to pl_cnt[1].
 * ------------------------------------------------------------------------------------------- */
typedef struct EtbNmsParams {
  int32_t B, P, no;         /* batch, predictions per image, 5+nc */
  float conf_thres, iou_thres;
  int32_t max_nms;          /* 30000 (general.py:911) */
  int32_t max_det;          /* 300   (general.py:888) */
  float max_wh;             /* 7680  (general.py:910): class offset; 0 => agnostic */
  int32_t need_cls_conf;    /* 0: non_max_suppression_ssod candidate test (obj only, general.py:900);
                               1: non_max_suppression (general.py:1005) candidate needs max cls > thr too */
  int32_t img_h, img_w;     /* for the pseudo-label normalisation */
} EtbNmsParams;

size_t etb_nms_workspace_bytes(const EtbNmsParams* p);
int etb_nms_ssod(const float* pred, const EtbNmsParams* p, float* det, int32_t* det_cnt, const double* Ms,
                 double* pl_rows, int32_t* pl_cnt, void* workspace, size_t workspace_bytes, void* stream);

/* val.py NMS: non_max_suppression(multi_label=True) (utils/general.py:994-1098, SURVEY.md 8f rank 2).  Every (row, class)
 * pair of a candidate row with obj*cls > conf_thres is a detection; more than max_nms per image: the max_nms best (exact
 * radix select, ties -> earlier pair); then the same rank + greedy NMS kernels as etb_nms_ssod.  Needs nc > 1 (the
 * reference disables multi_label for nc == 1: use etb_nms_ssod with need_cls_conf = 1).  det [B,max_det,8] (columns 0..5
 * are the reference's [xyxy, conf, cls]), det_cnt [B].  No pseudo-label transform on this path. */
size_t etb_nms_val_workspace_bytes(const EtbNmsParams* p);
int etb_nms_val(const float* pred, const EtbNmsParams* p, float* det, int32_t* det_cnt, void* workspace,
                size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Pseudo-Label-Assigner routing: ComputeStudentMatchLoss.select_targets
 * (models/loss/ssod/ssod_loss.py:130-192).  rows [N,9] float64 (N read from n_dev if non-NULL, else n_host);
 * thr_high/thr_low [nc] float64 on device.  Outputs 4 x [cap,7] fp32 (reliable, uncertain, uncertain_obj,
 * uncertain_cls) and out_cnt[4] int32, order preserved.
 * ------------------------------------------------------------------------------------------- */
int etb_select_targets(const double* rows, const int32_t* n_dev, int32_t n_host, int32_t cap,
                       const double* thr_high, const double* thr_low, int32_t nc, int32_t with_obj,
                       float* out /*[4][cap][7]*/, int32_t* out_cnt /*[4]*/, void* stream);

/* ---------------------------------------------------------------------------------------------
 * YOLOAnchorAssigner.build_targets / build_uc_targets_aug
 * (models/assigner/yolo_anchor_assigner.py:319-372, 640-697).
 * targets [nt,tstride] fp32 (tstride 6: img,cls,x,y,w,h ; 7: +score).  nt read from nt_dev if non-NULL.
 * Per level l (capacity cap rows, 15*nt suffices):
 *   idx  [cap,4] int32 = (b, a, gj, gi)      tbox [cap,4] f32 = (gx-gi', gy-gj', gw, gh)
 *   anch [cap,2] f32                        tcls [cap] int32      tscore [cap] f32 (tstride 7 only)
 *   cnt[l] int32.  Row order: offset-major, anchor-major, target order (bit-exact with the reference).
 * ------------------------------------------------------------------------------------------- */
typedef struct EtbAssignLevels {
  int32_t nl;
  int32_t nx[ETB_MAX_LEVELS], ny[ETB_MAX_LEVELS];
  float anchors[ETB_MAX_LEVELS][ETB_NA * 2]; /* grid units (anchors / stride) */
  float anchor_t;                            /* 4.0 */
} EtbAssignLevels;

typedef struct EtbAssignOut {
  int32_t* idx[ETB_MAX_LEVELS];
  float* tbox[ETB_MAX_LEVELS];
  float* anch[ETB_MAX_LEVELS];
  int32_t* tcls[ETB_MAX_LEVELS];
  float* tscore[ETB_MAX_LEVELS]; /* may be NULL when tstride==6 */
  int32_t* cnt;                  /* [nl] */
  int32_t cap;
} EtbAssignOut;

int etb_build_targets(const float* targets, const int32_t* nt_dev, int32_t nt_host, int32_t tstride,
                      const EtbAssignLevels* lv, const EtbAssignOut* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * LabelMatch.update's class histogram of the labeled rows, `cls_tmp[int(l[1:2])] += 1`
 * (utils/labelmatch.py:126-134).  targets [cap,tstride] fp32, class in column 1; the row count is *n_dev if
 * n_dev is non-NULL, else n_host (<= cap); rows past it are never read.  ADDS into hist[nc+1] int32: class =
 * the float truncated toward zero; a class outside [0,nc) (or NaN) is counted in hist[nc].  No host sync, no
 * allocation, order-independent (integer atomics): capturable in a CUDA graph.
 * ------------------------------------------------------------------------------------------- */
int etb_label_class_hist(const float* targets, const int32_t* n_dev, int32_t n_host, int32_t cap, int32_t tstride,
                         int32_t nc, int32_t* hist, void* stream);

/* ---------------------------------------------------------------------------------------------
 * bbox_iou, CIoU branch, xywh 1-to-1 (utils/metrics.py:207-249).  box1,box2 [n,4] fp32 -> out [n].
 * ------------------------------------------------------------------------------------------- */
int etb_bbox_ciou(const float* box1, const float* box2, int32_t n, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * ComputeLoss.default_loss (models/loss/loss.py:138-208) and ComputeStudentMatchLoss.default_loss
 * (models/loss/ssod/ssod_loss.py:194-288), forward and backward, fused:
 *   gather ps -> decode -> CIoU -> (1-iou) mean ; cls BCE ; tobj scatter (highest row index wins, = CPU
 *   oracle) ; uncertain soft-label override ; obj BCE over cells with tobj>=0 ; weights ; x batch.
 * p[l] [B,na,ny,nx,no] fp32.  Target sets come from etb_build_targets (device counts, no host sync).
 *   set 0: certain (box+cls+tobj=iou)    set 1: uncertain (tobj=score or -1)   [SSOD only]
 *   set 2: uncertain_obj (extra box term) set 3: uncertain_cls (extra cls term) [SSOD only]
 * out[4] fp32 = {lbox, lobj, lcls, loss*B} (already weighted like the reference's loss dict).
 * Backward writes dense grad_p[l] (every element written; no pre-zeroing needed), scaled by *gscale_dev.
 * ------------------------------------------------------------------------------------------- */
typedef struct EtbLossParams {
  int32_t nl, B, na, no;
  int32_t nx[ETB_MAX_LEVELS], ny[ETB_MAX_LEVELS];
  float balance[ETB_MAX_LEVELS];
  float box_w, obj_w, cls_w;
  float cp, cn;            /* smoothed BCE targets */
  int32_t nsets;           /* 1 supervised, 4 SSOD */
  int32_t ignore_obj;      /* SSOD.ignore_obj: uncertain cells -> tobj=-1 */
  int32_t with_bbox;       /* SSOD.pseudo_label_with_bbox */
  int32_t with_cls;        /* SSOD.pseudo_label_with_cls  */
  float cls_pw, obj_pw;    /* BCEWithLogitsLoss(pos_weight=) of the class and objectness terms (1: none) */
  float fl_gamma;          /* > 0: FocalLoss(gamma=fl_gamma, alpha=0.25) around both criteria */
  int32_t ssi;             /* autobalance: index of the stride-16 level the balance is normalised by */
  /* autobalance (loss.py:191-197): double[nl] balance state on the device, or NULL to use balance[] above.  When set,
   * the forward reads it, keeps the float32 values it used for the backward, and advances it in place. */
  double* balance_state;
} EtbLossParams;

size_t etb_loss_workspace_bytes(const EtbLossParams* lp, int32_t cap);
int etb_loss_forward(const float* const* p /*[nl]*/, const EtbLossParams* lp, const EtbAssignOut* sets /*[nsets]*/,
                     float* out4, void* workspace, size_t workspace_bytes, void* stream);
int etb_loss_backward(const float* const* p, float* const* grad_p, const EtbLossParams* lp,
                      const EtbAssignOut* sets, const float* gscale_dev, void* workspace, size_t workspace_bytes,
                      void* stream);

/* ---------------------------------------------------------------------------------------------
 * Conv trunk (models/backbone/common.py:471-484 Conv = conv2d(bias=False)+BN+SiLU; Bottleneck :534-544;
 * models/head/yolov5_head.py:55 Detect 1x1).  wgmma implicit GEMM, NHWC bf16 operands, fp32 accumulate
 * in registers, TMA-fed.  x [N,H,W,Cin] bf16 (channel stride x_cstride >= Cin so a concat slice can be read in
 * place), w [Cout, kh*kw*Cin] bf16 (K-major), y [N,Ho,Wo,*] bf16 written at channel offset into a buffer
 * with y_cstride channels (so concat is free).
 *   epilogue: v = acc*scale[c] + bias[c]  (folded eval-mode BN, or conv bias with scale=NULL)
 *             act 0: none, 1: SiLU, 2: ReLU, 4: Hardswish (3 is not a code) ;  optional residual add (Bottleneck
 *             shortcut) after act.
 *   y_f32 != NULL: write fp32 in the Detect train layout [N,na,Ho,Wo,det_no] instead (channel c = a*det_no+o).
 * ------------------------------------------------------------------------------------------- */
typedef struct EtbConvParams {
  int32_t N, H, W, Cin, Cout;
  int32_t kh, kw, stride, pad;
  int32_t x_cstride, y_cstride, y_coffset; /* channel strides of the NHWC buffers, output channel offset */
  int32_t res_cstride, res_coffset;        /* residual buffer geometry (if residual != NULL) */
  int32_t act;                             /* 0 none, 1 SiLU, 2 ReLU, 4 Hardswish; etb_conv_dgrad/wgrad ignore it */
  int32_t det_no;                          /* y_f32 path: outputs per anchor (85); Cout = na*det_no */
} EtbConvParams;

int etb_conv_fwd(const void* x_bf16, const void* w_bf16, const float* scale, const float* bias,
                 const void* residual_bf16, void* y_bf16, float* y_f32, const EtbConvParams* cp, void* stream);

/* data gradient of the same convolution (autograd of Conv.forward, SURVEY.md K2): dx = conv_transpose(dy, W), run as
 * implicit GEMMs on the same wgmma kernel -- one launch per output-parity class (1 for stride 1, 4 for stride 2).
 * `cp` describes the FORWARD conv; cp->x_cstride is the channel stride of dy, cp->y_cstride / y_coffset place dx.
 * wd = the etb_pack_multi mode 1 (or 3) blocks of every parity class, concatenated: Cin*k*k*ceil64(Cout) bf16 elements.
 * accumulate != 0: dx += result. */
int etb_conv_dgrad(const void* dy_bf16, const void* wd_bf16, void* dx_bf16, const EtbConvParams* cp, int32_t accumulate,
                   void* stream);

/* weight gradient (SURVEY.md K2): dW[co][tap][ci] = sum_pixels dy * x(shifted): wgmma GEMM with the pixels as the
 * reduction dimension (MN-major operands straight from the NHWC tensors via TMA).  Two-stage split-K: every CTA stores its
 * partial tile into its slice of `workspace`, then a reduce kernel sums the slices, converts to the parameter layout
 * [Cout,Cin,kh,kw] and writes (flags bit1: adds into) dw_f32 -- which may be the gradient-arena slice of the parameter.
 * `cp` describes the FORWARD conv; cp->x_cstride is x's channel stride, cp->y_cstride dy's.
 * flags bit0: stem (cp = the K=128 pointwise GEMM over the etb_stem_im2col_into buffer; dw_f32 is [Cout,3,6,6]). */
size_t etb_conv_wgrad_workspace_bytes(const EtbConvParams* cp);
int etb_conv_wgrad(const void* x_bf16, const void* dy_bf16, float* dw_f32, const EtbConvParams* cp, int32_t flags,
                   void* workspace, size_t workspace_bytes, void* stream);

/* training-mode BatchNorm2d (eps, momentum, batch statistics, running-stat update with the unbiased variance) + activation
 * around the convolutions (models/backbone/common.py:480-481; utils/torch_utils.py:162-171), forward and backward.
 * y / da / dy / out are NHWC bf16 [M][cstride] with M = N*H*W; per-channel vectors are fp32.
 * act: 0 none, 1 SiLU, 2 ReLU (derivative 0 at 0), 4 Hardswish z*min(max(z+3,0),6)/6 (derivative 0 for z <= -3, z/3+1/2
 * for -3 < z < 3, 1 for z >= 3: torch's hardswish_backward); any other value is ETB_ERR_INVALID.
 *   forward : etb_bn_stats (per-block partial rows [rows][2][C] = sum y, sum y^2; rows = etb_bn_partial_rows(M,C,0))
 *             -> etb_bn_finalize (fixed-order sum of the rows -> scale, shift, mean, invstd, running stats)
 *             -> etb_bn_act_apply_res (a = act(y*scale+shift) [+ res])
 *   backward: etb_bn_act_bwd_reduce (partial rows of sum dz, sum dz*xhat; dz = da*act'(z); rows = etb_bn_partial_rows(M,C,1))
 *             -> etb_bn_act_bwd_finalize (sums[2C]; dbeta, dgamma written or accumulated into the parameters' .grad)
 *             -> etb_bn_act_bwd_apply (dy = gamma*invstd*(dz - sum_dz/M - xhat*sum_dz_xhat/M))
 * No atomics and no memsets: the statistics are bit-reproducible run to run. */
int32_t etb_bn_partial_rows(int64_t M, int32_t C, int32_t which /* 0 forward stats, 1 backward reduce */);
int etb_bn_stats(const void* y_bf16, int64_t M, int32_t C, int32_t y_cstride, float* partials, int32_t rows, void* stream);
int etb_bn_finalize(const float* partials, int32_t rows, int64_t M, int32_t C, const float* gamma, const float* beta, float eps,
                    float momentum, float* running_mean, float* running_var, float* scale, float* shift, float* mean,
                    float* invstd, void* stream);
/* out = act(y*scale+shift), + res when res != NULL: the Bottleneck shortcut (models/backbone/common.py:499
 * `x + cv2(cv1(x))`); res is NHWC bf16 with its own channel stride */
int etb_bn_act_apply_res(const void* y_bf16, const float* scale, const float* shift, const void* res_bf16, void* out_bf16,
                         int64_t M, int32_t C, int32_t y_cstride, int32_t res_cstride, int32_t out_cstride, int32_t act,
                         void* stream);
int etb_bn_act_bwd_reduce(const void* da_bf16, const void* y_bf16, const float* scale, const float* shift, const float* mean,
                          const float* invstd, int64_t M, int32_t C, int32_t da_cstride, int32_t y_cstride, int32_t act,
                          float* partials, int32_t rows, void* stream);
int etb_bn_act_bwd_finalize(const float* partials, int32_t rows, int32_t C, float* sums, float* dgamma, float* dbeta,
                            int32_t accumulate, void* stream);
int etb_bn_act_bwd_apply(const void* da_bf16, const void* y_bf16, const float* scale, const float* shift, const float* mean,
                         const float* invstd, const float* sums, int64_t M, int32_t C, int32_t da_cstride, int32_t y_cstride,
                         int32_t dy_cstride, int32_t act, void* dy_bf16, void* stream);
/* SyncBatchNorm (torch.nn.SyncBatchNorm: statistics of the global batch across ranks).
 *   forward : etb_bn_stats_sums (this rank's sums [2C+1] fp64 = sum y, sum y^2, M; the rows of etb_bn_stats summed in
 *             etb_bn_finalize's fixed order; M == 0 gives zeros) -> SUM all-reduce of sums across the ranks
 *             -> etb_bn_finalize_global (scale, shift, mean, invstd as etb_bn_finalize lays them out; running stats with the
 *             global count: momentum, unbiased var*M/(M-1)) -> etb_bn_act_apply_res
 *   backward: etb_bn_act_bwd_reduce -> etb_bn_act_bwd_finalize (local dgamma / dbeta, as torch's SyncBN returns them)
 *             -> SUM all-reduce of sums[2C] -> etb_bn_act_bwd_apply_global (etb_bn_act_bwd_apply over this rank's M rows,
 *             dividing by the global count fwd_sums[2C] of the forward's all-reduced vector, read on the device). */
int etb_bn_stats_sums(const void* y_bf16, int64_t M, int32_t C, int32_t y_cstride, float* partials, int32_t rows, double* sums,
                      void* stream);
int etb_bn_finalize_global(const double* sums, int32_t C, const float* gamma, const float* beta, float eps, float momentum,
                           float* running_mean, float* running_var, float* scale, float* shift, float* mean, float* invstd,
                           void* stream);
int etb_bn_act_bwd_apply_global(const void* da_bf16, const void* y_bf16, const float* scale, const float* shift, const float* mean,
                                const float* invstd, const float* sums, const double* fwd_sums, int64_t M, int32_t C,
                                int32_t da_cstride, int32_t y_cstride, int32_t dy_cstride, int32_t act, void* dy_bf16, void* stream);

/* small layout / elementwise helpers of the trunk (all HBM-bound, coalesced 16 B vectors) */

/* NCHW fp32 <-> NHWC bf16 (channel stride / offset on the NHWC side) */
int etb_nchw_f32_to_nhwc_bf16(const float* x, void* y, int32_t N, int32_t C, int32_t H, int32_t W,
                              int32_t y_cstride, int32_t y_coffset, float mul, void* stream);
int etb_nhwc_bf16_to_nchw_f32(const void* x, float* y, int32_t N, int32_t C, int32_t H, int32_t W,
                              int32_t x_cstride, int32_t x_coffset, void* stream);
/* SPPF (models/backbone/common.py:702-708): buf [N,H,W,cstride>=4C] holds x in channels [0,C); writes
 * maxpool5(x), maxpool5^2(x)=maxpool9(x), maxpool5^3(x)=maxpool13(x) into [C,2C),[2C,3C),[3C,4C) (the concat). */
int etb_sppf_pool(void* buf_bf16, int32_t N, int32_t H, int32_t W, int32_t C, int32_t cstride, void* stream);
/* nn.Upsample(scale_factor=2, nearest) written into a channel slice of the concat buffer (yolov5_neck.py:92,97) */
int etb_upsample2x_nhwc(const void* x_bf16, void* y_bf16, int32_t N, int32_t H, int32_t W, int32_t C,
                        int32_t x_cstride, int32_t x_coffset, int32_t y_cstride, int32_t y_coffset, void* stream);

/* training-side glue between the student's convolutions (forward AND backward), all on channel slices of NHWC bf16
 * buffers so torch.cat / nn.MaxPool2d / nn.Upsample and their autograd kernels drop out of the step:
 *   etb_maxpool5_fwd : y = maxpool 5x5 s1 p2 (x), idx[N,H,W,C] u8 = argmax position (dy+2)*5+(dx+2), first max wins
 *                      (SPPF, models/backbone/common.py:702-708)
 *   etb_maxpool5_bwd : out = add + scatter of src through idx, in gather form (add may be NULL)
 *   etb_upsample2x_bwd: dx[n,h,w,:] = sum of the 2x2 block of dy (models/neck/yolov5_neck.py:38,46 backward)
 *   etb_copy_slice_nhwc: y[m,0:C] = x[m,0:C] (torch.cat of a tensor that was not produced in place) */
int etb_maxpool5_fwd(const void* x_bf16, void* y_bf16, uint8_t* idx, int32_t N, int32_t H, int32_t W, int32_t C,
                     int32_t x_cstride, int32_t y_cstride, void* stream);
int etb_maxpool5_bwd(const void* src_bf16, const uint8_t* idx, const void* add_bf16, void* out_bf16, int32_t N, int32_t H,
                     int32_t W, int32_t C, int32_t src_cstride, int32_t add_cstride, int32_t out_cstride, void* stream);
int etb_upsample2x_bwd(const void* dy_bf16, void* dx_bf16, int32_t N, int32_t H, int32_t W, int32_t C, int32_t dy_cstride,
                       int32_t dx_cstride, void* stream);
int etb_copy_slice_nhwc(const void* x_bf16, void* y_bf16, int64_t M, int32_t C, int32_t x_cstride, int32_t y_cstride,
                        void* stream);
/* element type of a packing / folding source (model.half() and model.bfloat16() state is read as stored; every value is
 * converted to fp32 first, which is exact, so a half model packs to what its fp32 copy holding the same values packs to) */
#define ETB_DT_F32 0
#define ETB_DT_F16 1
#define ETB_DT_BF16 2
/* conv weight packing: one launch packs every conv weight of the model, or a single one (descs and the chunk list live in
 * device memory; chunk = {desc index, chunk index} covering ETB_PACK_CHUNK destination elements).  w [Cout,Cin,k,k] of
 * element type dtype -> bf16 K-major GEMM operands, written only at real elements (the caller zeroes the pads):
 *   mode 0: forward operand [Cout][kh][kw][out_ld], out_ld = Cin or ceil64(Cin) (every tap padded to the 64-channel K block);
 *   mode 1: one dgrad parity class [Cin][ntaps][out_ld >= Cout] (tap t = (kh[t],kw[t]));
 *   mode 2: stem [Cout][128] in the etb_stem_im2col_into K order (c*6+kh)*6+kw = the OIHW row, zero above 108;
 *   mode 3: mode 1 with the sign flipped (dgrad operand of a conv behind GradReverse, models/detector/yolo_ssod.py:158-172);
 *   mode 4: out[e] = w[e] as fp32 for e < elems (the fp32 conv bias the epilogue reads, from a half-precision model). */
#define ETB_PACK_CHUNK 4096
typedef struct EtbPackDesc {
  const void* w;    /* [Cout,Cin,k,k] of element type dtype */
  void* out;        /* bf16 destination (mode 4: fp32) */
  int64_t elems;    /* destination elements to produce */
  int32_t Cout, Cin, k, mode, ntaps, out_ld;
  int32_t dtype;    /* ETB_DT_* of w */
  int8_t kh[12], kw[12];
} EtbPackDesc;
int etb_pack_multi(const EtbPackDesc* descs_dev, const void* chunks_dev /* int32 pairs */, int32_t n_chunks, void* stream);
typedef struct EtbFoldDesc {
  const void *gamma, *beta, *mean, *var;   /* [C] of element type dtype */
  float *scale, *bias;
  int32_t C;
  float eps;
  int32_t dtype;                           /* ETB_DT_* of gamma, beta, mean and var */
} EtbFoldDesc;
/* eval-mode BatchNorm folded to per-channel scale/bias: scale = g/sqrt(var+eps), bias = b - mean*scale (in fp32) */
int etb_fold_bn_multi(const EtbFoldDesc* descs_dev, int32_t n, void* stream);

/* ---- the last library ops of the student's step (csrc/tail.cu) ----------------------------------------------------------
 * Detect backward layout: the fused loss hands back d(loss)/d(logits) as fp32 [N,na,H,W,no] (the train layout of
 * models/head/yolov5_head.py:66).  etb_detect_dy_pack rewrites it as the bf16 NHWC operand dy [N,H,W,Cpad] (channel =
 * a*no + o, pad channels zeroed) of the wgmma dgrad / wgrad and emits per-block column sums; etb_column_sum reduces them
 * to the conv-bias gradient (yolov5_head.py:55: nn.Conv2d(..., bias=True)) -- replaces autograd's permute/contiguous/sum.
 * Any no >= 1 and any Cpad >= na*no with Cpad % 8 == 0 (DetectConvFn passes ceil64(na*no)); every pad channel of dy is
 * written (zero), so dy needs no initialisation.  partials: [etb_detect_dy_rows(N,H,W)][na*no] floats. */
int64_t etb_detect_dy_rows(int32_t N, int32_t H, int32_t W);
int etb_detect_dy_pack(const float* g, void* dy_bf16, float* partials, int32_t N, int32_t na, int32_t H, int32_t W,
                       int32_t no, int32_t Cpad, void* stream);
/* out[c] (+)= sum_r partials[r][c], fixed-order tree (deterministic); accumulate != 0 adds into out (gradient arena) */
int etb_column_sum(const float* partials, int64_t rows, int32_t C, float* out, int32_t accumulate, void* stream);
/* netD tail (models/detector/yolo_ssod.py:224-238): o[m][0:2] = conv2(h)[m] for h = relu(conv1(x)) [M][h_cstride] bf16,
 * w2 [2][C] fp32; backward: dh[m][c] = (h>0) * (do[m][0] w2[0][c] + do[m][1] w2[1][c]) as bf16 [M][C], and per-block
 * partials [etb_netd_tail_rows(M)][2][C] of dW2 (reduce with etb_column_sum(partials, rows, 2*C, dw2, ...)). */
int32_t etb_netd_tail_rows(int64_t M);
int etb_netd_tail_fwd(const void* h_bf16, int64_t M, int32_t C, int32_t h_cstride, const float* w2, float* o, void* stream);
int etb_netd_tail_bwd(const float* dout, const void* h_bf16, int64_t M, int32_t C, int32_t h_cstride, const float* w2,
                      void* dh_bf16, float* partials, int32_t rows, void* stream);
/* DomainLoss / TargetLoss (models/loss/loss.py:312-421): out[0] = 0.5 * mean_i( -(1-p_i)^2 log p_i ), p_i =
 * softmax(x_i)[label], over all positions of the nl netD maps x[l] ([M[l]][2] fp32, contiguous).  Backward writes
 * dx[l] = gout[0] * d(out)/d(x[l]) (gout: device scalar).  workspace: etb_domain_focal_workspace_bytes(). */
typedef struct EtbFocalParams {
  const float* x[ETB_MAX_LEVELS];
  float* dx[ETB_MAX_LEVELS];
  int64_t M[ETB_MAX_LEVELS];
  int32_t nl, label;
} EtbFocalParams;
int64_t etb_domain_focal_workspace_bytes(void);
int etb_domain_focal_fwd(const EtbFocalParams* fp, float* out, void* workspace, int64_t workspace_bytes, void* stream);
int etb_domain_focal_bwd(const EtbFocalParams* fp, const float* gout, void* stream);
/* stem im2col straight from the loaders' batch (trainer/ssod_trainer.py:694-696 `imgs.to(device).float() / 255` fused with
 * the 6x6 s2 p2 stem patch gather of models/backbone/yolov5_backbone.py:56): x is [N,3,H,W] of element type src, one of
 * ETB_STEM_SRC_* (uint8 with div 255; fp32 or fp16 with div 1 for already scaled input); value = float(x) / div (IEEE
 * division) rounded to bf16 at K index (c*6+kh)*6+kw (the OIHW weight row order) for K < 108, zeros above; the N images go
 * to image slots [img_offset, img_offset+N) of the im2col buffer y [*,H/2,W/2,128] -- torch.cat((imgs, unlabeled_imgs))
 * without the copy.  An fp16 batch gives what its .float() copy gives, bit for bit. */
#define ETB_STEM_SRC_F32 0
#define ETB_STEM_SRC_U8 1
#define ETB_STEM_SRC_F16 2
int etb_stem_im2col_into(const void* x, int32_t src, void* y_bf16, int32_t N, int32_t H, int32_t W, int32_t img_offset,
                         float div, void* stream);

/* validation matching (val.py:123-145 process_batch), all images of a batch in one launch: correct[b][d][i] = detection d of
 * image b is a true positive at IoU threshold iouv[i].  det [B][max_det][det_ld>=6] fp32 rows (x1,y1,x2,y2,conf,cls) in the
 * labels' coordinate space, det_cnt [B] valid rows per image (NULL: max_det); labels [nt][6] fp32 (img,cls,x1,y1,x2,y2);
 * correct [B][max_det][T] uint8, fully written; *overflow_dev = 1 if an image carries more than 1024 labels. */
int etb_val_process_batch(const float* det, const int32_t* det_cnt, int32_t B, int32_t max_det, int32_t det_ld,
                          const float* labels, int32_t nt, const float* iouv, int32_t T, uint8_t* correct,
                          int32_t* overflow_dev, void* stream);

/* one validation batch into the epoch's statistics (val.py:340-376), no host sync: det [B][max_det][det_ld>=6] etb_nms_val rows
 * (x1,y1,x2,y2,conf,cls in the letterboxed H x W image), det_cnt [B]; img_meta [B][5] fp32 (h0, w0, inv_gain, padw, padh
 * from the loader's shapes[b] = ((h0, w0), ((gain, _), (padw, padh))), inv_gain = fp32(1 / gain) with the division in
 * float64); targets [nt][6] fp32 (img, cls, x, y, w, h normalised).  Rows are rescaled to native space as torch does it on
 * fp32 CUDA tensors (x - pad, times inv_gain -- torch divides by a host scalar that way --, clamp to the native image),
 * class 0 if single_cls; labels become native xyxy; etb_val_process_batch matches them (iouv [T], T <= 16).  Each detection's conf, class and correct bits (bit i = IoU threshold i) are appended to arena_conf / arena_cls /
 * arena_tp at rows [*arena_n, ...) and *arena_n advances; label classes are ADDED into hist[nc+1] (etb_label_class_hist).
 * flags[0] |= 1 if any appended bit is set; flags[1] = 1 on overflow (an image with more than 1024 labels, or rows past
 * arena_cap, which are dropped).  workspace: etb_val_epoch_append_workspace_bytes(B, max_det, nt, T). */
size_t etb_val_epoch_append_workspace_bytes(int32_t B, int32_t max_det, int32_t nt, int32_t T);
int etb_val_epoch_append(const float* det, const int32_t* det_cnt, int32_t B, int32_t max_det, int32_t det_ld,
                         const float* img_meta, const float* targets, int32_t nt, int32_t H, int32_t W, int32_t single_cls,
                         const float* iouv, int32_t T, int32_t nc, float* arena_conf, float* arena_cls, uint16_t* arena_tp,
                         int64_t arena_cap, int64_t* arena_n, int32_t* hist, int32_t* flags, void* workspace,
                         size_t workspace_bytes, void* stream);
/* etb_val_epoch_append, and the same batch also added into the confusion matrix cm_matrix [(cm_nc+1)^2] int64 from the rows
 * and labels it rescaled (etb_confusion_matrix with conf cm_conf, IoU cm_iou; its flags go to cm_flags[2]).  One rescale;
 * one launch more than etb_val_epoch_append. */
int etb_val_epoch_append_confusion(const float* det, const int32_t* det_cnt, int32_t B, int32_t max_det, int32_t det_ld,
                                   const float* img_meta, const float* targets, int32_t nt, int32_t H, int32_t W, int32_t single_cls,
                                   const float* iouv, int32_t T, int32_t nc, float* arena_conf, float* arena_cls, uint16_t* arena_tp,
                                   int64_t arena_cap, int64_t* arena_n, int32_t* hist, int32_t* flags, int32_t cm_nc, float cm_conf,
                                   float cm_iou, int64_t* cm_matrix, int32_t* cm_flags, void* workspace, size_t workspace_bytes,
                                   void* stream);

/* the detection confusion matrix (utils/metrics.py:129-186 ConfusionMatrix.process_batch), all images of a batch in one
 * launch: det [B][max_det][det_ld>=6] fp32 rows (x1,y1,x2,y2,conf,cls) in the labels' coordinate space, det_cnt [B] (NULL:
 * max_det rows per image); labels [nt][6] fp32 (img,cls,x1,y1,x2,y2).  Rows with conf > conf_thres are matched to labels
 * class-agnostically at IoU > iou_thres, one label per detection and one detection per label by descending IoU (ties: the
 * later label, then the later detection), and the counts are ADDED into matrix [(nc+1)^2] int64, row = predicted class,
 * column = true class, nc = background.  As val.py calls it, an image with no row or no label adds nothing.  flags[0] = 1 if
 * an image carries more than 1024 labels; flags[1] = 1 if a class to be counted (truncated like Tensor.int()) is outside
 * [0, nc): it is not counted. */
int etb_confusion_matrix(const float* det, const int32_t* det_cnt, int32_t B, int32_t max_det, int32_t det_ld, const float* labels,
                         int32_t nt, int32_t nc, float conf_thres, float iou_thres, int64_t* matrix, int32_t* flags, void* stream);

/* numeric core of ap_per_class (utils/metrics.py:22-126) over n rows conf [n] fp32, pred_cls [n] fp32, tp [n] uint16 (bit t =
 * true positive at IoU column t, T <= 16).  cls_slot [ncls_table]: the slot (0..nu-1, in ascending class order) of every
 * class that has labels, -1 otherwise; a row whose class is not an integer in [0, ncls_table) with a slot is ignored.
 * n_l [nu] labels per slot.  Rows are sorted by (slot, conf descending) with a stable radix sort (equal confidences keep their
 * row order).  px [1000] = numpy.linspace(0, 1, 1000), xs [101] = numpy.linspace(0, 1, 101).  Outputs (float64):
 * ap_points [nu][T][101] = numpy.interp(xs, mrec, envelope(mpre)) of compute_ap, p_curve / r_curve [nu][1000] = the P and R
 * curves at column 0 (numpy.interp(-px, -conf, ., left=1 / 0)), zero for a slot without predictions; n_p [nu] int32.
 * Recall must not decrease along a class (at most n_l true positives per column).
 * workspace: etb_ap_per_class_workspace_bytes(n, nu). */
size_t etb_ap_per_class_workspace_bytes(int64_t n, int32_t nu);
int etb_ap_per_class(const float* conf, const float* pred_cls, const uint16_t* tp, int64_t n, int32_t T, const int32_t* cls_slot,
                     int32_t ncls_table, int32_t nu, const int32_t* n_l, const double* px, const double* xs, double* ap_points,
                     double* p_curve, double* r_curve, int32_t* n_p, void* workspace, size_t workspace_bytes, void* stream);

/* class-agnostic greedy NMS over ready-made detection rows (extra-teachers merge, utils/self_supervised_utils.py:256-274,
 * torchvision.ops.nms semantics): rows [B][nmax<=1024][ld>=5] fp32 (x1,y1,x2,y2,score,...), cnt [B]; kept rows are written
 * to out [B][nmax][ld] in descending-score (stable) order, out_cnt [B]. */
int etb_nms_boxes(const float* rows, const int32_t* cnt, int32_t B, int32_t nmax, int32_t ld, float iou_thres, float* out,
                  int32_t* out_cnt, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Anchor-free (YOLOv8) pieces -- SURVEY.md section 8f row 5.  The reference defines no end-to-end step for this head
 * (models/loss/tal_loss.py cannot be imported, trainer/ssod_trainer.py:598-606 rejects it): these are the importable
 * operators, with the reference's call contracts.
 *
 * etb_tal_assign = TaskAlignedAssigner.forward (models/assigner/tal_assigner.py:29-80; helpers
 * models/module/nanodet_utils.py:184-248) for n_max_boxes = M > 0, all tensors fp32 contiguous on the device:
 *   pd_scores [B,A,nc] (already sigmoid), pd_bboxes [B,A,4] xyxy, anc_points [A,2], gt_labels [B,M] (the reference's
 *   [B,M,1]), gt_bboxes [B,M,4] xyxy, mask_gt [B,M]
 *   -> target_labels [B,A] int64, target_bboxes [B,A,4], target_scores [B,A,nc], fg_mask [B,A] uint8 (torch.bool).
 * Ties inside the top-k go to the lowest anchor index (torch.topk promises no order).  A <= 51200, topk <= A.
 * workspace: etb_tal_workspace_bytes(B, A, M), 16-byte aligned, contents irrelevant on entry.
 * ------------------------------------------------------------------------------------------- */
size_t etb_tal_workspace_bytes(int32_t B, int32_t A, int32_t M);
int etb_tal_assign(const float* pd_scores, const float* pd_bboxes, const float* anc_points, const float* gt_labels,
                   const float* gt_bboxes, const float* mask_gt, int32_t B, int32_t A, int32_t M, int32_t nc, int32_t topk,
                   float alpha, float beta, float eps, int64_t* target_labels, float* target_bboxes, float* target_scores,
                   uint8_t* fg_mask, void* workspace, size_t workspace_bytes, void* stream);

/* etb_v8_decode = the DFL decode of YoloV8Detect's eval branch (models/head/yolov8_head.py:169-220) and of
 * ComputeTalLoss.bbox_decode (models/loss/tal_loss.py:88-95,150-156) from the head's train-layout outputs
 * cls [B,A,nc] / reg [B,A,4*(reg_max+1)] fp32 (levels concatenated along A, row-major inside a level; anchor points
 * (x + grid_cell_offset, y + grid_cell_offset) as models/module/nanodet_utils.py:135-182 generates them).  Each output is
 * optional (NULL):  pred [B,A,5+nc] = (cx,cy,w,h)*stride, 1, sigmoid(cls);  boxes_grid [B,A,4] xyxy in grid units;
 * boxes_pix [B,A,4] = boxes_grid * stride (the assigner's pd_bboxes);  scores [B,A,nc] = sigmoid(cls) (its pd_scores). */
typedef struct EtbV8Levels {
  int32_t nl;
  int32_t h[ETB_MAX_LEVELS], w[ETB_MAX_LEVELS];
  float stride[ETB_MAX_LEVELS];
} EtbV8Levels;
int etb_v8_decode(const float* cls, const float* reg, const EtbV8Levels* levels, int32_t B, int32_t nc, int32_t reg_max,
                  float grid_cell_offset, float* pred, float* boxes_grid, float* boxes_pix, float* scores, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Pseudo-label quality statistics of the SSOD step: utils/self_supervised_utils.py:481-587 check_pseudo_label_with_gt
 * (with_gt = 1) and :589-606 check_pseudo_label (with_gt = 0), including their select_targets (:456-479) -- the host
 * loops (one .cpu() per row, numpy matching) that trainer/ssod_trainer.py:661-670 runs every iteration.  Restated in
 * csrc/plq.cu.  rows [cap,9] float64 pseudo labels, n from n_dev if non-NULL (capped at n_host), else n_host;
 * thr_high / thr_low [nc] float64 (the ones etb_select_targets reads; both NULL: every row, with_gt only); gt [capG,6]
 * fp32 (img, cls, x, y, w, h normalised), m from m_dev / m_host; iouv [T] float64 (T <= 16); batch_size > 0.
 * iou64 = 1 (no thresholds, float64 rows): the IoU in float64 as torch promotes it.
 * vals [5][T] float64: tp, fp_cls, fp_loc per threshold, then pse_num, gt_num (repeated over T), in the trainer's meaning
 * (with_gt = 0: precision, 0, recall, reliable + uncertain, reliable); n == 0 gives all zeros (the invalid step).
 * cnt [5 + 3T] int32: n, n_uncertain, n_reliable, m, overflow (1: an image with more than 1024 GT boxes, whose rest is
 * ignored, a class index outside [0, nc) or a negative image index), then the tp, fp_cls and fp_loc counts [T] each.
 * Two launches, no host sync; workspace: etb_pl_quality_workspace_bytes(), contents irrelevant on entry.
 * ------------------------------------------------------------------------------------------- */
size_t etb_pl_quality_workspace_bytes(void);
int etb_pl_quality(const double* rows, const int32_t* n_dev, int32_t n_host, const double* thr_high, const double* thr_low,
                   int32_t nc, const float* gt, const int32_t* m_dev, int32_t m_host, const double* iouv, int32_t T,
                   int32_t batch_size, int32_t with_gt, int32_t iou64, double* vals, int32_t* cnt, void* workspace,
                   size_t workspace_bytes, void* stream);

/* MetricMeter / AverageMeter.update (utils/metrics.py:352-414) on the device: state [3][cap] float64 (sum, count, val);
 * for each i < n (n <= ETB_METER_MAX_SRC, distinct slots): v = *src[i] (float64 if f64[i], else fp32 widened);
 * sum[slot] += v; count[slot] += 1; val[slot] = v.  src / slot / f64 are host arrays.  One launch. */
#define ETB_METER_MAX_SRC 16
int etb_meter_update(double* state, int32_t cap, const void* const* src, const int32_t* slot, const int32_t* f64, int32_t n,
                     void* stream);

/* ---------------------------------------------------------------------------------------------
 * Batched inference (detect.py): letterbox on the device and rescale of the NMS rows to each frame.
 *
 * etb_letterbox_u8: frames[B] (device table) of uint8 BGR HWC source frames, each (h0, w0), resized to (new_h, new_w) and
 * placed at (top, left) of out [B][3][H][W] uint8 RGB (the stem's uint8 input); every other pixel is 114.  The resize is
 * cv2.resize(INTER_LINEAR) on 8UC3 bit for bit: 11-bit fixed-point coefficients, an exact integer row pass, the column pass
 * ((((S0 >> 4) * b0) >> 16) + (((S1 >> 4) * b1) >> 16) + 2) >> 2, source columns clamped (coefficient 0) at the edges,
 * source rows clamped without touching the coefficients, and a 2x2 box average (sum + 2) >> 2 when the frame is downscaled
 * by exactly 2 on both axes (OpenCV's switch to INTER_AREA).  (new_h, new_w) == (h0, w0) copies.  H % 32 == W % 32 == 0 is
 * not required, but W % 4 == 0 is.  One launch.
 *
 * etb_detect_rescale: det [B][max_det][det_ld>=6] fp32 NMS rows (x1,y1,x2,y2,conf,cls), det_cnt [B]; meta [B][5] fp32
 * (h0, w0, inv_gain, padw, padh) as etb_val_epoch_append takes it -> out [B][max_det][6]: the first det_cnt[b] rows of image
 * b in its frame's pixel space, scale_coords(...).round() as torch computes it on fp32 CUDA tensors (x - pad, times
 * inv_gain, clamp to the frame, round half to even); other rows are not written.  One launch.
 * ------------------------------------------------------------------------------------------- */
typedef struct EtbLetterboxFrame {
  const uint8_t* src;
  int32_t h0, w0, new_h, new_w, top, left;
} EtbLetterboxFrame;
int etb_letterbox_u8(const EtbLetterboxFrame* frames, int32_t B, int32_t H, int32_t W, uint8_t* out, void* stream);
int etb_detect_rescale(const float* det, const int32_t* det_cnt, int32_t B, int32_t max_det, int32_t det_ld, const float* meta,
                       float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ETB200_H_ */
