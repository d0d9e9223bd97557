// glue.cu -- the data-movement ops BETWEEN the student's convolutions in training mode, forward and backward:
//   SPPF's cascaded 5x5 s1 p2 max pools     reference models/backbone/common.py:702-708 (nn.MaxPool2d + its autograd)
//   the neck's nearest 2x upsample backward reference models/neck/yolov5_neck.py:38,46 (nn.Upsample + its autograd)
//   concat-by-offset slice copy             reference models/neck/yolov5_neck.py:91-104 (torch.cat)
// All operate on NHWC bf16 with a channel stride (so they read / write channel slices of a concat buffer in place), one
// thread per 16 B vector of 8 channels, HBM/L2-bound: algorithmic bytes = 2 B/element per tensor touched (+1 B index).
#include "common.cuh"

static inline unsigned glue_grid(int64_t work) {
  int64_t b = (work + 255) / 256;
  const int64_t cap = (int64_t)etb_num_sms() * 16;
  return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}
__device__ __forceinline__ void g_unpack8(const uint4 v, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 t = __bfloat1622float2(h[j]);
    f[2 * j] = t.x;
    f[2 * j + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 g_pack8(const float* f) {
  uint4 v;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) h[j] = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);
  return v;
}

// ---- max pool 5x5 s1 p2 with argmax (window position (dy+2)*5+(dx+2), first maximum in scan order wins like ATen) ----
__global__ void __launch_bounds__(256) maxpool5_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                           uint8_t* __restrict__ idx, int N, int H, int W, int C, int xcs, int ycs) {
  const int cg = C >> 3;
  const int64_t total = (int64_t)N * H * W * cg;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(e % cg);
    const int64_t pix = e / cg;
    const int w = (int)(pix % W), h = (int)((pix / W) % H), n = (int)(pix / ((int64_t)W * H));
    float best[8];
    int bi[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { best[j] = -INFINITY; bi[j] = 12; }
#pragma unroll
    for (int dy = -2; dy <= 2; ++dy) {
      const int ih = h + dy;
      if (ih < 0 || ih >= H) continue;
#pragma unroll
      for (int dx = -2; dx <= 2; ++dx) {
        const int iw = w + dx;
        if (iw < 0 || iw >= W) continue;
        float f[8];
        g_unpack8(*reinterpret_cast<const uint4*>(x + (((int64_t)n * H + ih) * W + iw) * xcs + g * 8), f);
        const int p = (dy + 2) * 5 + dx + 2;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (f[j] > best[j] || f[j] != f[j]) { best[j] = f[j]; bi[j] = p; }
      }
    }
    *reinterpret_cast<uint4*>(y + pix * ycs + g * 8) = g_pack8(best);
    uint2 iv;
    iv.x = (uint32_t)bi[0] | ((uint32_t)bi[1] << 8) | ((uint32_t)bi[2] << 16) | ((uint32_t)bi[3] << 24);
    iv.y = (uint32_t)bi[4] | ((uint32_t)bi[5] << 8) | ((uint32_t)bi[6] << 16) | ((uint32_t)bi[7] << 24);
    *reinterpret_cast<uint2*>(idx + pix * C + g * 8) = iv;
  }
}

// out[i] = add[i] + sum over the <=25 windows o that contain i of (argmax(o) == i ? src[o] : 0)   (gather form: no atomics)
__global__ void __launch_bounds__(256) maxpool5_bwd_kernel(const __nv_bfloat16* __restrict__ src, const uint8_t* __restrict__ idx,
                                                           const __nv_bfloat16* __restrict__ add, __nv_bfloat16* __restrict__ out, int N, int H,
                                                           int W, int C, int scs, int acs, int ocs) {
  const int cg = C >> 3;
  const int64_t total = (int64_t)N * H * W * cg;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(e % cg);
    const int64_t pix = e / cg;
    const int w = (int)(pix % W), h = (int)((pix / W) % H), n = (int)(pix / ((int64_t)W * H));
    float acc[8];
    if (add) {
      g_unpack8(*reinterpret_cast<const uint4*>(add + pix * acs + g * 8), acc);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    }
#pragma unroll
    for (int dy = -2; dy <= 2; ++dy) {
      const int oh = h + dy;
      if (oh < 0 || oh >= H) continue;
#pragma unroll
      for (int dx = -2; dx <= 2; ++dx) {
        const int ow = w + dx;
        if (ow < 0 || ow >= W) continue;
        const int64_t op = ((int64_t)n * H + oh) * W + ow;
        const uint2 iv = *reinterpret_cast<const uint2*>(idx + op * C + g * 8);
        const uint32_t want = (uint32_t)((2 - dy) * 5 + (2 - dx));      // position of i inside o's window
        const uint32_t w4 = want * 0x01010101u;
        const uint32_t m0 = iv.x ^ w4, m1 = iv.y ^ w4;                   // a zero byte marks a hit
        if ((((m0 - 0x01010101u) & ~m0) | ((m1 - 0x01010101u) & ~m1)) & 0x80808080u) {
          float f[8];
          g_unpack8(*reinterpret_cast<const uint4*>(src + op * scs + g * 8), f);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (((m0 >> (8 * j)) & 0xFFu) == 0) acc[j] += f[j];
            if (((m1 >> (8 * j)) & 0xFFu) == 0) acc[4 + j] += f[4 + j];
          }
        }
      }
    }
    *reinterpret_cast<uint4*>(out + pix * ocs + g * 8) = g_pack8(acc);
  }
}

extern "C" int etb_maxpool5_fwd(const void* x_bf16, void* y_bf16, uint8_t* idx, int32_t N, int32_t H, int32_t W, int32_t C,
                                int32_t x_cstride, int32_t y_cstride, void* stream) {
  ETB_CHECK_ARG(x_bf16 && y_bf16 && idx && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && x_cstride % 8 == 0 && y_cstride % 8 == 0);
  ETB_CHECK_ARG(x_cstride >= C && y_cstride >= C);
  etb_launch(maxpool5_fwd_kernel, dim3(glue_grid((int64_t)N * H * W * (C / 8))), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16*)x_bf16, (__nv_bfloat16*)y_bf16, idx, N, H, W, C, x_cstride, y_cstride);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
extern "C" int etb_maxpool5_bwd(const void* src_bf16, const uint8_t* idx, const void* add_bf16, void* out_bf16, int32_t N, int32_t H,
                                int32_t W, int32_t C, int32_t src_cstride, int32_t add_cstride, int32_t out_cstride, void* stream) {
  ETB_CHECK_ARG(src_bf16 && idx && out_bf16 && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0);
  ETB_CHECK_ARG(src_cstride % 8 == 0 && add_cstride % 8 == 0 && out_cstride % 8 == 0 && src_cstride >= C && out_cstride >= C);
  etb_launch(maxpool5_bwd_kernel, dim3(glue_grid((int64_t)N * H * W * (C / 8))), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16*)src_bf16, idx, (const __nv_bfloat16*)add_bf16, (__nv_bfloat16*)out_bf16, N, H, W, C, src_cstride, add_cstride,
      out_cstride);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// ---- nearest 2x upsample backward: dx[n,h,w,:] = sum of the 2x2 block of dy (fp32 accumulate) ----
__global__ void __launch_bounds__(256) upsample2x_bwd_kernel(const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dx, int N, int H, int W,
                                                             int C, int dycs, int dxcs) {
  const int cg = C >> 3;
  const int64_t total = (int64_t)N * H * W * cg;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(e % cg);
    const int64_t pix = e / cg;
    const int w = (int)(pix % W), h = (int)((pix / W) % H), n = (int)(pix / ((int64_t)W * H));
    const __nv_bfloat16* p = dy + (((int64_t)n * 2 * H + 2 * h) * 2 * W + 2 * w) * dycs + g * 8;
    float a[8], b[8];
    g_unpack8(*reinterpret_cast<const uint4*>(p), a);
    g_unpack8(*reinterpret_cast<const uint4*>(p + dycs), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += b[j];
    g_unpack8(*reinterpret_cast<const uint4*>(p + (int64_t)2 * W * dycs), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += b[j];
    g_unpack8(*reinterpret_cast<const uint4*>(p + (int64_t)2 * W * dycs + dycs), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += b[j];
    *reinterpret_cast<uint4*>(dx + pix * dxcs + g * 8) = g_pack8(a);
  }
}
extern "C" int etb_upsample2x_bwd(const void* dy_bf16, void* dx_bf16, int32_t N, int32_t H, int32_t W, int32_t C, int32_t dy_cstride,
                                  int32_t dx_cstride, void* stream) {
  ETB_CHECK_ARG(dy_bf16 && dx_bf16 && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && dy_cstride % 8 == 0 && dx_cstride % 8 == 0);
  ETB_CHECK_ARG(dy_cstride >= C && dx_cstride >= C);
  etb_launch(upsample2x_bwd_kernel, dim3(glue_grid((int64_t)N * H * W * (C / 8))), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16*)dy_bf16, (__nv_bfloat16*)dx_bf16, N, H, W, C, dy_cstride, dx_cstride);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// ---- channel-slice copy: y[m, 0:C] = x[m, 0:C] for M pixels, both sides with a channel stride ----
__global__ void __launch_bounds__(256) copy_slice_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int64_t M, int C, int xcs,
                                                         int ycs) {
  const int cg = C >> 3;
  const int64_t total = M * cg;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(e % cg);
    const int64_t pix = e / cg;
    *reinterpret_cast<uint4*>(y + pix * ycs + g * 8) = *reinterpret_cast<const uint4*>(x + pix * xcs + g * 8);
  }
}
extern "C" int etb_copy_slice_nhwc(const void* x_bf16, void* y_bf16, int64_t M, int32_t C, int32_t x_cstride, int32_t y_cstride, void* stream) {
  ETB_CHECK_ARG(x_bf16 && y_bf16 && M > 0 && C > 0 && C % 8 == 0 && x_cstride % 8 == 0 && y_cstride % 8 == 0 && x_cstride >= C && y_cstride >= C);
  etb_launch(copy_slice_kernel, dim3(glue_grid(M * (C / 8))), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16*)x_bf16, (__nv_bfloat16*)y_bf16, M, C, x_cstride,
                                                                             y_cstride);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
