// tail.cu -- the last library ops of the student's step, as native kernels (all HBM / latency bound, no tensor-core work):
//   * Detect backward layout + bias gradient   reference models/head/yolov5_head.py:55,66 (the autograd of view/permute/
//     contiguous + conv bias): fp32 loss gradient [N,na,H,W,no] -> bf16 NHWC dy [N,H,W,Cpad] (channel = a*no + o) for
//     the wgmma dgrad / wgrad, and db[c] = sum over pixels in the same pass (two-stage, deterministic)
//   * netD tail                                 reference models/detector/yolo_ssod.py:224-238: conv2 (C -> 2, 1x1, no bias)
//     on relu(conv1(x)) forward and backward (dh with the ReLU mask folded in, dW2 two-stage)
//   * Domain / Target focal loss                reference models/loss/loss.py:312-421: 0.5 * mean(-(1-p)^2 log p),
//     p = softmax(logits)[label], over all positions of the three netD maps; forward + backward
//   * stem im2col straight from the loaders' uint8 NCHW batch (x/255 exactly as `.float() / 255`)
//     reference trainer/ssod_trainer.py:694-696
#include "common.cuh"

// ------------------------------------------------------------------------------------------------ Detect backward
#define DET_PIX 64
// grid (chunks, na, N), 128 threads: thread o < no walks DET_PIX pixels of (image n, anchor a): coalesced 340 B rows in,
// 170 B runs out; per-channel partial sums of the bias gradient in registers -> partials[(n*chunks + chunk)][C].
__global__ void __launch_bounds__(128) detect_dy_pack_kernel(const float* __restrict__ g, __nv_bfloat16* __restrict__ dy, float* __restrict__ partials,
                                                             int na, int HW, int no, int Cpad) {
  const int chunk = blockIdx.x, a = blockIdx.y, n = blockIdx.z;
  const int o = threadIdx.x;
  const int C = na * no;
  const int p0 = chunk * DET_PIX, p1 = min(p0 + DET_PIX, HW);
  const float* gp = g + ((size_t)(n * na + a) * HW) * no;
  __nv_bfloat16* dp = dy + (size_t)n * HW * Cpad + a * no;
  float acc = 0.f;
  if (o < no) {
#pragma unroll 4
    for (int p = p0; p < p1; ++p) {
      const float v = __ldg(gp + (size_t)p * no + o);
      acc += v;
      dp[(size_t)p * Cpad + o] = __float2bfloat16(v);
    }
    partials[((size_t)n * gridDim.x + chunk) * C + a * no + o] = acc;
  } else if (a == na - 1 && o - no < Cpad - C) {       // zero the pad channels [C, Cpad) (K padding of the dgrad GEMM)
    __nv_bfloat16* zp = dy + (size_t)n * HW * Cpad + C + (o - no);
    for (int p = p0; p < p1; ++p) zp[(size_t)p * Cpad] = __float2bfloat16(0.f);
  }
}

// out[c] (+)= sum over rows of partials[row][c]; block (32 channels x 32 row lanes), fixed-shape tree: deterministic
__global__ void __launch_bounds__(1024) column_sum_kernel(const float* __restrict__ partials, int rows, int C, float* __restrict__ out, int accumulate) {
  __shared__ float red[32][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float a = 0.f;
  if (c < C)
    for (int r = threadIdx.y; r < rows; r += 32) a += __ldg(partials + (size_t)r * C + c);
  red[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) {
    if ((int)threadIdx.y < s) red[threadIdx.y][threadIdx.x] += red[threadIdx.y + s][threadIdx.x];
    __syncthreads();
  }
  if (threadIdx.y == 0 && c < C) out[c] = accumulate ? out[c] + red[0][threadIdx.x] : red[0][threadIdx.x];
}

extern "C" int64_t etb_detect_dy_rows(int32_t N, int32_t H, int32_t W) { return (int64_t)N * (((int64_t)H * W + DET_PIX - 1) / DET_PIX); }

extern "C" int etb_detect_dy_pack(const float* g, void* dy_bf16, float* partials, int32_t N, int32_t na, int32_t H, int32_t W, int32_t no,
                                  int32_t Cpad, void* stream) {
  ETB_CHECK_ARG(g && dy_bf16 && partials && N > 0 && na > 0 && H > 0 && W > 0 && no > 0 && no <= 128);
  ETB_CHECK_ARG(Cpad >= na * no && Cpad % 8 == 0 && no + (Cpad - na * no) <= 128 && na < 65536 && N < 65536);
  const int HW = H * W;
  dim3 grid((HW + DET_PIX - 1) / DET_PIX, na, N);
  etb_launch(detect_dy_pack_kernel, dim3(grid), dim3(128), 0, (cudaStream_t)stream, g, (__nv_bfloat16*)dy_bf16, partials, na, HW, no, Cpad);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

extern "C" int etb_column_sum(const float* partials, int64_t rows, int32_t C, float* out, int32_t accumulate, void* stream) {
  ETB_CHECK_ARG(partials && out && rows > 0 && rows < (1ll << 31) && C > 0);
  etb_launch(column_sum_kernel, dim3((C + 31) / 32), dim3(dim3(32, 32)), 0, (cudaStream_t)stream, partials, (int)rows, C, out, accumulate);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// ------------------------------------------------------------------------------------------------ netD tail (C -> 2)
#define NETD_THREADS 256
// MAXG channel groups of 8 per lane: C <= 32*8*MAXG.  MAXG 4 (C <= 1024) serves YOLOv5n-l; MAXG 5 (C <= 1280) is a
// second instance for YOLOv5x's det_32, so the narrower layers keep the smaller register allocation.
#define NETD_MAXG_MAX 5
__device__ __forceinline__ void bf8_to_f(const uint4 v, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 t = __bfloat1622float2(h[j]);
    f[2 * j] = t.x;
    f[2 * j + 1] = t.y;
  }
}

// one warp per pixel row: o[m][j] = sum_c h[m][c] * w2[j][c]
__global__ void __launch_bounds__(NETD_THREADS) netd_tail_fwd_kernel(const __nv_bfloat16* __restrict__ h, long M, int C, int hcs,
                                                                     const float* __restrict__ w2, float* __restrict__ o) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = NETD_THREADS / 32;
  const int G = C >> 3;
  for (long m = (long)blockIdx.x * nw + wid; m < M; m += (long)gridDim.x * nw) {
    float a0 = 0.f, a1 = 0.f;
    for (int g = lane; g < G; g += 32) {
      float f[8];
      bf8_to_f(*reinterpret_cast<const uint4*>(h + m * hcs + g * 8), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        a0 = fmaf(f[j], __ldg(w2 + g * 8 + j), a0);
        a1 = fmaf(f[j], __ldg(w2 + C + g * 8 + j), a1);
      }
    }
    a0 = warp_sum(a0);
    a1 = warp_sum(a1);
    if (lane == 0) *reinterpret_cast<float2*>(o + 2 * m) = make_float2(a0, a1);
  }
}

// dh[m][c] = (h[m][c] > 0) * (do[m][0]*w2[0][c] + do[m][1]*w2[1][c])   (ReLU mask of relu(conv1) folded in)
// partial dW2[j][c] = sum over this block's rows of do[m][j] * h[m][c]  -> partials[blockIdx][2][C]
template <int NETD_MAXG>
__global__ void __launch_bounds__(NETD_THREADS) netd_tail_bwd_kernel(const float* __restrict__ dout, const __nv_bfloat16* __restrict__ h, long M, int C,
                                                                     int hcs, const float* __restrict__ w2, __nv_bfloat16* __restrict__ dh,
                                                                     float* __restrict__ partials) {
  extern __shared__ float sm[];      // [nw][2][C]
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = NETD_THREADS / 32;
  const int G = C >> 3;
  float acc[NETD_MAXG][2][8];
  float w0[NETD_MAXG][8], w1[NETD_MAXG][8];
#pragma unroll
  for (int q = 0; q < NETD_MAXG; ++q) {
    const int g = lane + 32 * q;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      acc[q][0][j] = acc[q][1][j] = 0.f;
      w0[q][j] = g < G ? __ldg(w2 + g * 8 + j) : 0.f;
      w1[q][j] = g < G ? __ldg(w2 + C + g * 8 + j) : 0.f;
    }
  }
  for (long m = (long)blockIdx.x * nw + wid; m < M; m += (long)gridDim.x * nw) {
    const float2 d = *reinterpret_cast<const float2*>(dout + 2 * m);
#pragma unroll
    for (int q = 0; q < NETD_MAXG; ++q) {
      const int g = lane + 32 * q;
      if (g < G) {
        float f[8], r[8];
        bf8_to_f(*reinterpret_cast<const uint4*>(h + m * hcs + g * 8), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          r[j] = f[j] > 0.f ? fmaf(d.x, w0[q][j], d.y * w1[q][j]) : 0.f;
          acc[q][0][j] = fmaf(d.x, f[j], acc[q][0][j]);
          acc[q][1][j] = fmaf(d.y, f[j], acc[q][1][j]);
        }
        uint4 ov;
        __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(&ov);
#pragma unroll
        for (int j = 0; j < 4; ++j) o2[j] = __floats2bfloat162_rn(r[2 * j], r[2 * j + 1]);
        *reinterpret_cast<uint4*>(dh + m * C + g * 8) = ov;
      }
    }
  }
#pragma unroll
  for (int q = 0; q < NETD_MAXG; ++q) {
    const int g = lane + 32 * q;
    if (g < G)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        sm[(wid * 2 + 0) * C + g * 8 + j] = acc[q][0][j];
        sm[(wid * 2 + 1) * C + g * 8 + j] = acc[q][1][j];
      }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * C; i += NETD_THREADS) {
    float s = 0.f;
    for (int w = 0; w < nw; ++w) s += sm[w * 2 * C + i];      // fixed order
    partials[(size_t)blockIdx.x * 2 * C + i] = s;
  }
}

static inline int netd_blocks(int64_t M) {
  const int64_t need = (M + NETD_THREADS / 32 - 1) / (NETD_THREADS / 32);
  const int64_t cap = (int64_t)etb_num_sms() * 4;
  return (int)(need < cap ? (need < 1 ? 1 : need) : cap);
}
extern "C" int32_t etb_netd_tail_rows(int64_t M) { return M > 0 ? netd_blocks(M) : 0; }

extern "C" int etb_netd_tail_fwd(const void* h_bf16, int64_t M, int32_t C, int32_t h_cstride, const float* w2, float* o, void* stream) {
  ETB_CHECK_ARG(h_bf16 && w2 && o && M > 0 && C >= 8 && C % 8 == 0 && h_cstride >= C && h_cstride % 8 == 0);
  etb_launch(netd_tail_fwd_kernel, dim3(netd_blocks(M)), dim3(NETD_THREADS), 0, (cudaStream_t)stream, (const __nv_bfloat16*)h_bf16, (long)M, C, h_cstride, w2, o);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

template <int MAXG>
static int launch_netd_tail_bwd(const float* dout, const void* h_bf16, int64_t M, int32_t C, int32_t h_cstride, const float* w2, void* dh_bf16,
                                float* partials, int32_t rows, cudaStream_t st) {
  const size_t smem = (size_t)(NETD_THREADS / 32) * 2 * C * sizeof(float);
  static bool attr_done = false;
  if (!attr_done) {
    ETB_CHECK_CUDA(cudaFuncSetAttribute(netd_tail_bwd_kernel<MAXG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (NETD_THREADS / 32) * 2 * 256 * MAXG * 4));
    attr_done = true;
  }
  etb_launch(netd_tail_bwd_kernel<MAXG>, dim3(rows), dim3(NETD_THREADS), smem, st, dout, (const __nv_bfloat16*)h_bf16, (long)M, C, h_cstride, w2,
             (__nv_bfloat16*)dh_bf16, partials);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// partials: [etb_netd_tail_rows(M)][2][C] floats (fully overwritten); dW2 = etb_column_sum(partials, rows, 2*C, ...)
extern "C" int etb_netd_tail_bwd(const float* dout, const void* h_bf16, int64_t M, int32_t C, int32_t h_cstride, const float* w2, void* dh_bf16,
                                 float* partials, int32_t rows, void* stream) {
  ETB_CHECK_ARG(dout && h_bf16 && w2 && dh_bf16 && partials && M > 0 && C >= 8 && C % 8 == 0 && C <= 256 * NETD_MAXG_MAX);
  ETB_CHECK_ARG(h_cstride >= C && h_cstride % 8 == 0 && rows == netd_blocks(M));
  if (C > 1024) return launch_netd_tail_bwd<5>(dout, h_bf16, M, C, h_cstride, w2, dh_bf16, partials, rows, (cudaStream_t)stream);
  return launch_netd_tail_bwd<4>(dout, h_bf16, M, C, h_cstride, w2, dh_bf16, partials, rows, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------ domain focal loss
// L_i = -(1 - p)^2 log p,  p = softmax(x_i)[label] = sigmoid(d),  d = x_i[label] - x_i[1 - label]
//   log p = -softplus(-d);  dL/dd = (1 - p)^2 (2 p log p - (1 - p))
#define FOCAL_THREADS 256
#define FOCAL_BLOCKS 128
__device__ __forceinline__ void focal_terms(float d, float* logp, float* p) {
  const float sp = fmaxf(-d, 0.f) + log1pf(__expf(-fabsf(d)));     // softplus(-d)
  *logp = -sp;
  *p = __expf(-sp);
}

__global__ void __launch_bounds__(FOCAL_THREADS) focal_fwd_kernel(EtbFocalParams fp, float* __restrict__ partials) {
  __shared__ float red[FOCAL_THREADS / 32];
  float acc = 0.f;
  for (int l = 0; l < fp.nl; ++l) {
    const float2* x = reinterpret_cast<const float2*>(fp.x[l]);
    for (long m = (long)blockIdx.x * FOCAL_THREADS + threadIdx.x; m < fp.M[l]; m += (long)FOCAL_BLOCKS * FOCAL_THREADS) {
      const float2 v = x[m];
      const float d = fp.label ? v.y - v.x : v.x - v.y;
      float logp, p;
      focal_terms(d, &logp, &p);
      const float q = 1.f - p;
      acc = fmaf(-q * q, logp, acc);
    }
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < FOCAL_THREADS / 32; ++w) s += red[w];
    partials[blockIdx.x] = s;
  }
}
__global__ void focal_finalize_kernel(const float* __restrict__ partials, float scale, float* __restrict__ out) {
  float s = 0.f;
  for (int b = 0; b < FOCAL_BLOCKS; ++b) s += partials[b];      // fixed order
  out[0] = s * scale;
}
__global__ void __launch_bounds__(FOCAL_THREADS) focal_bwd_kernel(EtbFocalParams fp, const float* __restrict__ gout, float scale) {
  const float gs = gout[0] * scale;
  for (int l = 0; l < fp.nl; ++l) {
    const float2* x = reinterpret_cast<const float2*>(fp.x[l]);
    float2* dx = reinterpret_cast<float2*>(fp.dx[l]);
    for (long m = (long)blockIdx.x * FOCAL_THREADS + threadIdx.x; m < fp.M[l]; m += (long)gridDim.x * FOCAL_THREADS) {
      const float2 v = x[m];
      const float d = fp.label ? v.y - v.x : v.x - v.y;
      float logp, p;
      focal_terms(d, &logp, &p);
      const float q = 1.f - p;
      const float gd = gs * q * q * (2.f * p * logp - q);
      dx[m] = fp.label ? make_float2(-gd, gd) : make_float2(gd, -gd);
    }
  }
}

static inline int64_t focal_total(const EtbFocalParams* fp) {
  int64_t t = 0;
  for (int l = 0; l < fp->nl; ++l) t += fp->M[l];
  return t;
}
extern "C" int64_t etb_domain_focal_workspace_bytes() { return FOCAL_BLOCKS * sizeof(float); }

// out[0] = 0.5 * mean_i L_i over all positions of the nl maps (x[l]: [M[l]][2] fp32 logits, contiguous)
extern "C" int etb_domain_focal_fwd(const EtbFocalParams* fp, float* out, void* workspace, int64_t workspace_bytes, void* stream) {
  ETB_CHECK_ARG(fp && out && workspace && workspace_bytes >= etb_domain_focal_workspace_bytes() && fp->nl >= 1 && fp->nl <= ETB_MAX_LEVELS);
  ETB_CHECK_ARG(fp->label == 0 || fp->label == 1);
  const int64_t tot = focal_total(fp);
  ETB_CHECK_ARG(tot > 0);
  for (int l = 0; l < fp->nl; ++l) ETB_CHECK_ARG(fp->x[l] && fp->M[l] >= 0 && (((uintptr_t)fp->x[l]) & 7) == 0);
  etb_launch(focal_fwd_kernel, dim3(FOCAL_BLOCKS), dim3(FOCAL_THREADS), 0, (cudaStream_t)stream, *fp, (float*)workspace);
  ETB_CHECK_LAUNCH();
  etb_launch(focal_finalize_kernel, dim3(1), dim3(1), 0, (cudaStream_t)stream, (const float*)workspace, 0.5f / (float)tot, out);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
// dx[l][m][:] = gout[0] * d(out)/d(x[l][m][:])   (gout: device scalar)
extern "C" int etb_domain_focal_bwd(const EtbFocalParams* fp, const float* gout, void* stream) {
  ETB_CHECK_ARG(fp && gout && fp->nl >= 1 && fp->nl <= ETB_MAX_LEVELS && (fp->label == 0 || fp->label == 1));
  const int64_t tot = focal_total(fp);
  ETB_CHECK_ARG(tot > 0);
  for (int l = 0; l < fp->nl; ++l) ETB_CHECK_ARG(fp->x[l] && fp->dx[l] && (((uintptr_t)fp->dx[l]) & 7) == 0);
  int64_t blocks = (tot + FOCAL_THREADS - 1) / FOCAL_THREADS;
  const int64_t cap = (int64_t)etb_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  etb_launch(focal_bwd_kernel, dim3((unsigned)blocks), dim3(FOCAL_THREADS), 0, (cudaStream_t)stream, *fp, gout, 0.5f / (float)tot);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// ------------------------------------------------------------------------------------------------ stem im2col from uint8
// Same tiling as stem_im2col_kernel (trunk.cu): K order (c,kh,kw), 64 output pixels of one output row per block.  The input
// is the loaders' uint8 NCHW batch; value = float(u8) / 255 (IEEE division: bit-identical to `.float() / 255`), rounded
// to bf16 once.  Several source batches (labeled, strong-aug) are written into one im2col buffer at an image offset, which
// is the student's torch.cat((imgs, unlabeled_imgs), 0) (ssod_trainer.py:620) without the copy.
#define STEM_TP 64
#define STEM_PITCH 133
template <typename T>
__global__ void __launch_bounds__(256) stem_im2col_any_kernel(const T* __restrict__ x, __nv_bfloat16* __restrict__ y, int N, int H, int W, float div) {
  __shared__ float sm[18 * STEM_PITCH];
  const int Ho = H / 2, Wo = W / 2;
  const int tiles_w = (Wo + STEM_TP - 1) / STEM_TP;
  const int tw = blockIdx.x % tiles_w;
  const int oh = (blockIdx.x / tiles_w) % Ho;
  const int n = blockIdx.x / (tiles_w * Ho);
  const int ow0 = tw * STEM_TP;
  const int iw0 = 2 * ow0 - 2, ih0 = 2 * oh - 2;
  for (int i = threadIdx.x; i < 18 * 132; i += 256) {
    const int row = i / 132, col = i - row * 132;
    const int c = row / 6, kh = row - c * 6;
    const int ih = ih0 + kh, iw = iw0 + col;
    float v = 0.f;
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) v = __fdiv_rn((float)x[(((int64_t)n * 3 + c) * H + ih) * W + iw], div);
    sm[row * STEM_PITCH + col] = v;
  }
  __syncthreads();
  const int g = threadIdx.x & 15;
  int off[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int k = g * 8 + j;
    off[j] = k < 108 ? (k / 6) * STEM_PITCH + (k % 6) : -1;
  }
  uint4* yo = reinterpret_cast<uint4*>(y) + (((int64_t)n * Ho + oh) * Wo + ow0) * 16;
#pragma unroll
  for (int q = threadIdx.x; q < STEM_TP * 16; q += 256) {
    const int pp = q >> 4;
    if (ow0 + pp >= Wo) break;
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = off[j] >= 0 ? sm[off[j] + 2 * pp] : 0.f;
    uint4 ov;
    __nv_bfloat162* o = reinterpret_cast<__nv_bfloat162*>(&ov);
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);
    yo[q] = ov;
  }
}

// x: [N,3,H,W] uint8 (is_u8 = 1) or fp32 (is_u8 = 0), contiguous; y: the im2col buffer [*,H/2,W/2,128] bf16 of the whole
// (concatenated) batch; the N images of x are written starting at image index img_offset.  div: 255 for raw uint8 pixels.
extern "C" int etb_stem_im2col_into(const void* x, int32_t is_u8, void* y_bf16, int32_t N, int32_t H, int32_t W, int32_t img_offset, float div,
                                    void* stream) {
  ETB_CHECK_ARG(x && y_bf16 && N > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && img_offset >= 0 && div > 0.f);
  const int64_t blocks = (int64_t)N * (H / 2) * ((W / 2 + STEM_TP - 1) / STEM_TP);
  ETB_CHECK_ARG(blocks < (1ll << 31));
  __nv_bfloat16* y = (__nv_bfloat16*)y_bf16 + (size_t)img_offset * (H / 2) * (W / 2) * 128;
  if (is_u8)
    etb_launch(stem_im2col_any_kernel<uint8_t>, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (const uint8_t*)x, y, N, H, W, div);
  else
    etb_launch(stem_im2col_any_kernel<float>, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (const float*)x, y, N, H, W, div);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
