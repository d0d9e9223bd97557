// trunk.cu -- layout / pooling / folding helpers around the wgmma convolutions (K3, K4, K18).
//   SPPF max pools + concat reference models/backbone/common.py:702-708
//   nearest 2x upsample     reference models/neck/yolov5_neck.py:92,97 (+ Concat common.py:796-797, free by slicing)
//   eval BN folding         reference utils/torch_utils.py:199-219 (fuse_conv_and_bn algebra), bn eps 1e-3
// All elementwise / gather kernels: HBM-bound, 16 B vector accesses along the channel (fastest) dimension.
#include "common.cuh"

static inline unsigned grid_for(int64_t n, int threads) {
  int64_t b = (n + threads - 1) / threads;
  const int64_t cap = (int64_t)etb_num_sms() * 32;
  return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}

// ---- NCHW fp32 <-> NHWC bf16 (simple gather; used at the edges of the trunk and by the tests) ----
__global__ void __launch_bounds__(256) nchw2nhwc_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, int N, int C, int H, int W,
                                                        int cs, int co, float mul) {
  const int64_t total = (int64_t)N * H * W * C;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(e % C);
    const int64_t pix = e / C;
    const int w = (int)(pix % W), h = (int)((pix / W) % H), n = (int)(pix / ((int64_t)W * H));
    y[pix * cs + co + c] = __float2bfloat16(__fmul_rn(x[(((int64_t)n * C + c) * H + h) * W + w], mul));
  }
}
__global__ void __launch_bounds__(256) nhwc2nchw_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ y, int N, int C, int H, int W, int cs, int co) {
  const int64_t total = (int64_t)N * H * W * C;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int w = (int)(e % W), h = (int)((e / W) % H), c = (int)((e / ((int64_t)W * H)) % C), n = (int)(e / ((int64_t)W * H * C));
    y[e] = __bfloat162float(x[(((int64_t)n * H + h) * W + w) * cs + co + c]);
  }
}
extern "C" int etb_nchw_f32_to_nhwc_bf16(const float* x, void* y, int32_t N, int32_t C, int32_t H, int32_t W, int32_t y_cstride,
                                         int32_t y_coffset, float mul, void* stream) {
  ETB_CHECK_ARG(x && y && N > 0 && C > 0 && H > 0 && W > 0 && y_cstride >= y_coffset + C);
  etb_launch(nchw2nhwc_kernel, dim3(grid_for((int64_t)N * C * H * W, 256)), dim3(256), 0, (cudaStream_t)stream, x, (__nv_bfloat16*)y, N, C, H, W, y_cstride, y_coffset, mul);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
extern "C" int etb_nhwc_bf16_to_nchw_f32(const void* x, float* y, int32_t N, int32_t C, int32_t H, int32_t W, int32_t x_cstride,
                                         int32_t x_coffset, void* stream) {
  ETB_CHECK_ARG(x && y && N > 0 && C > 0 && H > 0 && W > 0 && x_cstride >= x_coffset + C);
  etb_launch(nhwc2nchw_kernel, dim3(grid_for((int64_t)N * C * H * W, 256)), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16*)x, y, N, C, H, W, x_cstride, x_coffset);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// ---- SPPF: three cascaded 5x5 s1 p2 max pools == 5x5, 9x9, 13x13 windows of x (max is idempotent/associative) ----
__device__ __forceinline__ void bf8_max(uint4& acc, const uint4& v) {
  __nv_bfloat162* a = reinterpret_cast<__nv_bfloat162*>(&acc);
  const __nv_bfloat162* b = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) a[j] = __hmax2(a[j], b[j]);
}
__global__ void __launch_bounds__(256) sppf_pool_kernel(__nv_bfloat16* __restrict__ buf, int N, int H, int W, int C, int cs) {
  const int cg = C / 8;
  const int64_t total = (int64_t)N * H * W * cg;
  const uint32_t ninf2 = 0xFF80FF80u;  // bf16 -inf pair (max-pool padding value)
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(e % cg);
    const int64_t pix = e / cg;
    const int w = (int)(pix % W), h = (int)((pix / W) % H), n = (int)(pix / ((int64_t)W * H));
    uint4 m5 = make_uint4(ninf2, ninf2, ninf2, ninf2), m9 = m5, m13 = m5;
    for (int dy = -6; dy <= 6; ++dy) {
      const int ih = h + dy;
      if (ih < 0 || ih >= H) continue;
      for (int dx = -6; dx <= 6; ++dx) {
        const int iw = w + dx;
        if (iw < 0 || iw >= W) continue;
        const uint4 v = *reinterpret_cast<const uint4*>(buf + (((int64_t)n * H + ih) * W + iw) * cs + g * 8);
        bf8_max(m13, v);
        if (dy >= -4 && dy <= 4 && dx >= -4 && dx <= 4) bf8_max(m9, v);
        if (dy >= -2 && dy <= 2 && dx >= -2 && dx <= 2) bf8_max(m5, v);
      }
    }
    __nv_bfloat16* o = buf + pix * cs + g * 8;
    *reinterpret_cast<uint4*>(o + C) = m5;
    *reinterpret_cast<uint4*>(o + 2 * C) = m9;
    *reinterpret_cast<uint4*>(o + 3 * C) = m13;
  }
}
extern "C" int etb_sppf_pool(void* buf_bf16, int32_t N, int32_t H, int32_t W, int32_t C, int32_t cstride, void* stream) {
  ETB_CHECK_ARG(buf_bf16 && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && cstride >= 4 * C && cstride % 8 == 0);
  etb_launch(sppf_pool_kernel, dim3(grid_for((int64_t)N * H * W * (C / 8), 256)), dim3(256), 0, (cudaStream_t)stream, (__nv_bfloat16*)buf_bf16, N, H, W, C, cstride);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// ---- nearest 2x upsample into a channel slice ----
__global__ void __launch_bounds__(256) upsample2x_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int N, int H, int W, int C,
                                                         int xcs, int xco, int ycs, int yco) {
  const int cg = C / 8;
  const int Ho = 2 * H, Wo = 2 * W;
  const int64_t total = (int64_t)N * Ho * Wo * cg;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(e % cg);
    const int64_t pix = e / cg;
    const int w = (int)(pix % Wo), h = (int)((pix / Wo) % Ho), n = (int)(pix / ((int64_t)Wo * Ho));
    const uint4 v = *reinterpret_cast<const uint4*>(x + (((int64_t)n * H + (h >> 1)) * W + (w >> 1)) * xcs + xco + g * 8);
    *reinterpret_cast<uint4*>(y + pix * ycs + yco + g * 8) = v;
  }
}
extern "C" int etb_upsample2x_nhwc(const void* x_bf16, void* y_bf16, int32_t N, int32_t H, int32_t W, int32_t C, int32_t x_cstride,
                                   int32_t x_coffset, int32_t y_cstride, int32_t y_coffset, void* stream) {
  ETB_CHECK_ARG(x_bf16 && y_bf16 && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0);
  ETB_CHECK_ARG(x_cstride % 8 == 0 && x_coffset % 8 == 0 && y_cstride % 8 == 0 && y_coffset % 8 == 0);
  etb_launch(upsample2x_kernel, dim3(grid_for((int64_t)N * 4 * H * W * (C / 8), 256)), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16*)x_bf16, (__nv_bfloat16*)y_bf16, N, H, W, C, x_cstride, x_coffset, y_cstride, y_coffset);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// ---- weight packing / BN folding: ONE launch for all ~104 convs of the trunk (also the packer of a single weight) ----
// mode 0: fwd  [Cout][kh][kw][Cin or out_ld]   <- w[co][ci][kh][kw]        (dst index e: ci fastest; out_ld > Cin pads every tap)
// mode 1: dgrad class  [Cin][ntaps][out_ld>=Cout] <- w[co][ci][kh_t][kw_t]   (dst: co fastest; row pitch out_ld per tap)
// mode 2: stem [Cout][128] in the etb_stem_im2col_into K order (c,kh,kw) = the OIHW row, zero above 108
// mode 3: mode 1 negated (dgrad operand of a conv that sits behind a GradReverse)
// mode 4: fp32 copy of a 1-D tensor (a conv bias of a half-precision model)
// The source is fp32, fp16 or bf16 (d.dtype, uniform per block): every value is widened to fp32 (exact) before the same
// fp32 -> bf16 rounding, so a .half() model packs to what its fp32 copy holding the fp16 values packs to.
__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T>
__device__ __forceinline__ void pack_chunk(const EtbPackDesc& d, int64_t base) {
  const T* __restrict__ w = (const T*)d.w;
  __nv_bfloat16* __restrict__ o = (__nv_bfloat16*)d.out;
  const int kk = d.k * d.k;
#pragma unroll 4
  for (int i = threadIdx.x; i < ETB_PACK_CHUNK; i += 256) {
    const int64_t e = base + i;
    if (e >= d.elems) break;
    float v;
    int64_t dst = e;
    if (d.mode == 0) {
      const int ci = (int)(e % d.Cin);
      const int64_t t2 = e / d.Cin;
      const int t = (int)(t2 % kk), co = (int)(t2 / kk);
      v = to_f32(w[((int64_t)co * d.Cin + ci) * kk + t]);
      if (d.out_ld > d.Cin) dst = ((int64_t)co * kk + t) * d.out_ld + ci;   // every tap padded to out_ld = ceil64(Cin) (pad stays zero)
    } else if (d.mode == 1 || d.mode == 3) {
      const int co = (int)(e % d.Cout);
      const int64_t t2 = e / d.Cout;
      const int t = (int)(t2 % d.ntaps), ci = (int)(t2 / d.ntaps);
      v = to_f32(w[(((int64_t)co * d.Cin + ci) * d.k + d.kh[t]) * d.k + d.kw[t]]);
      if (d.mode == 3) v = -v;            // GradReverse in front of the conv: dx = -(W^T dy)
      dst = ((int64_t)ci * d.ntaps + t) * d.out_ld + co;
    } else if (d.mode == 2) {
      const int k = (int)(e & 127), oc = (int)(e >> 7);
      v = 0.f;
      if (k < 108) v = to_f32(w[oc * 108 + k]);
    } else {
      ((float*)d.out)[e] = to_f32(w[e]);
      continue;
    }
    o[dst] = __float2bfloat16(v);
  }
}

__global__ void __launch_bounds__(256) pack_multi_kernel(const EtbPackDesc* __restrict__ descs, const int2* __restrict__ chunks) {
  const int2 ch = chunks[blockIdx.x];
  const EtbPackDesc d = descs[ch.x];
  const int64_t base = (int64_t)ch.y * ETB_PACK_CHUNK;
  if (d.dtype == ETB_DT_F16) pack_chunk<__half>(d, base);
  else if (d.dtype == ETB_DT_BF16) pack_chunk<__nv_bfloat16>(d, base);
  else if (d.dtype == ETB_DT_F32) pack_chunk<float>(d, base);   // any other code: nothing is read (the host refuses it)
}

extern "C" int etb_pack_multi(const EtbPackDesc* descs_dev, const void* chunks_dev, int32_t n_chunks, void* stream) {
  ETB_CHECK_ARG(descs_dev && chunks_dev && n_chunks >= 0);
  if (n_chunks == 0) return ETB_OK;
  etb_launch(pack_multi_kernel, dim3(n_chunks), dim3(256), 0, (cudaStream_t)stream, descs_dev, (const int2*)chunks_dev);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

template <typename T>
__device__ __forceinline__ void fold_one(const EtbFoldDesc& d) {
  const T *gamma = (const T*)d.gamma, *beta = (const T*)d.beta, *mean = (const T*)d.mean, *var = (const T*)d.var;
  for (int c = threadIdx.x; c < d.C; c += 256) {
    const float s = to_f32(gamma[c]) / sqrtf(to_f32(var[c]) + d.eps);
    d.scale[c] = s;
    d.bias[c] = to_f32(beta[c]) - to_f32(mean[c]) * s;
  }
}
__global__ void __launch_bounds__(256) fold_multi_kernel(const EtbFoldDesc* __restrict__ descs) {
  const EtbFoldDesc d = descs[blockIdx.x];
  if (d.dtype == ETB_DT_F16) fold_one<__half>(d);
  else if (d.dtype == ETB_DT_BF16) fold_one<__nv_bfloat16>(d);
  else if (d.dtype == ETB_DT_F32) fold_one<float>(d);
}
extern "C" int etb_fold_bn_multi(const EtbFoldDesc* descs_dev, int32_t n, void* stream) {
  ETB_CHECK_ARG(descs_dev && n >= 0);
  if (n == 0) return ETB_OK;
  etb_launch(fold_multi_kernel, dim3(n), dim3(256), 0, (cudaStream_t)stream, descs_dev);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
