// letterbox.cu -- detect.py's pre-processing on the device: letterbox(auto=True) of a batch of raw uint8 BGR frames of any
// sizes (utils/datasets.py LoadImages: cv2.resize INTER_LINEAR + copyMakeBorder(114), then BGR -> RGB, HWC -> CHW), written
// as the [B,3,H,W] uint8 batch the stem's im2col reads.
//
// The resize restates OpenCV's 8UC3 INTER_LINEAR integer path as the x86 build computes it (checked byte for byte against
// cv2 by tests/test_letterbox_host.py):
//   coefficients: f = float((d + 0.5) * (1 / (dst / src)) - 0.5) (double arithmetic), s = floor(f), f -= s (float);
//     a0 = rint((1 - f) * 2048), a1 = rint(f * 2048).  Columns: s < 0 -> (s, f) = (0, 0); s >= w0 - 1 -> (w0 - 1, 0).
//     Rows keep f; only the row indices s and s + 1 are clamped to [0, h0 - 1].
//   row pass: S = p[s] * a0 + p[s + 1] * a1 (exact int32);
//   column pass (the SIMD one: v_mul_hi on S >> 4, then a rounding shift by 2): ((S0>>4)*b0 >> 16) + ((S1>>4)*b1 >> 16) + 2 >> 2.
//   An exact 2x downscale on both axes is INTER_AREA in OpenCV: (a + b + c + d + 2) >> 2.
// One thread writes 4 consecutive output pixels of one row (a 4-byte store per channel plane).
#include "common.cuh"

#define LB_THREADS 256

__device__ __forceinline__ void lb_coef(int d, int dst, int src, bool clamp, int& s0, int& s1, int& c0, int& c1) {
  const double scale = 1.0 / ((double)dst / (double)src);
  float f = __double2float_rn(((double)d + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  if (clamp) {
    if (s < 0) s = 0, f = 0.f;
    if (s >= src - 1) s = src - 1, f = 0.f;
  }
  c0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  c1 = __float2int_rn(__fmul_rn(f, 2048.f));
  s0 = min(max(s, 0), src - 1);
  s1 = min(max(s + 1, 0), src - 1);
}

__device__ __forceinline__ void lb_pixel(const EtbLetterboxFrame& f, int y, int x, int v[3]) {
  y -= f.top;
  x -= f.left;
  if (y < 0 || y >= f.new_h || x < 0 || x >= f.new_w) {
    v[0] = v[1] = v[2] = 114;
    return;
  }
  const uint8_t* p = f.src;
  const int rs = f.w0 * 3;
  if (f.new_h == f.h0 && f.new_w == f.w0) {
    const uint8_t* q = p + (size_t)y * rs + x * 3;
    v[0] = q[0], v[1] = q[1], v[2] = q[2];
    return;
  }
  if (2 * f.new_h == f.h0 && 2 * f.new_w == f.w0) {
    const uint8_t* q = p + (size_t)(2 * y) * rs + 6 * x;
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = (q[c] + q[c + 3] + q[rs + c] + q[rs + c + 3] + 2) >> 2;
    return;
  }
  int x0, x1, a0, a1, y0, y1, b0, b1;
  lb_coef(x, f.new_w, f.w0, true, x0, x1, a0, a1);
  lb_coef(y, f.new_h, f.h0, false, y0, y1, b0, b1);
  const uint8_t* r0 = p + (size_t)y0 * rs;
  const uint8_t* r1 = p + (size_t)y1 * rs;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int S0 = r0[3 * x0 + c] * a0 + r0[3 * x1 + c] * a1;
    const int S1 = r1[3 * x0 + c] * a0 + r1[3 * x1 + c] * a1;
    const int o = ((((S0 >> 4) * b0) >> 16) + (((S1 >> 4) * b1) >> 16) + 2) >> 2;
    v[c] = min(max(o, 0), 255);
  }
}

__global__ void __launch_bounds__(LB_THREADS) letterbox_u8_kernel(const EtbLetterboxFrame* __restrict__ frames, int H, int W,
                                                                 uint8_t* __restrict__ out) {
  const int b = blockIdx.y;
  const int q = blockIdx.x * LB_THREADS + threadIdx.x;
  const int W4 = W >> 2;
  if (q >= H * W4) return;
  const EtbLetterboxFrame f = frames[b];
  const int y = q / W4, x0 = (q - y * W4) * 4;
  uint32_t w[3] = {0u, 0u, 0u};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int v[3];
    lb_pixel(f, y, x0 + i, v);
#pragma unroll
    for (int c = 0; c < 3; ++c) w[2 - c] |= (uint32_t)v[c] << (8 * i);     // BGR -> RGB planes
  }
  const size_t plane = (size_t)H * W;
  uint32_t* o = reinterpret_cast<uint32_t*>(out + (size_t)b * 3 * plane + (size_t)y * W + x0);
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c * (plane >> 2)] = w[c];
}

extern "C" int etb_letterbox_u8(const EtbLetterboxFrame* frames, int32_t B, int32_t H, int32_t W, uint8_t* out, void* stream) {
  ETB_CHECK_ARG(frames && out && B > 0 && B < 65536 && H > 0 && W > 0 && W % 4 == 0 && (((uintptr_t)out) & 3) == 0);
  const int64_t work = (int64_t)H * (W / 4);
  ETB_CHECK_ARG(work < (1ll << 31) - LB_THREADS);
  etb_launch(letterbox_u8_kernel, dim3((unsigned)((work + LB_THREADS - 1) / LB_THREADS), (unsigned)B), dim3(LB_THREADS), 0,
             (cudaStream_t)stream, frames, H, W, out);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
