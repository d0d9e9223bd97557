// decode.cu -- Detect eval-mode decode (K6): reference models/head/yolov5_head.py:66-78.
//   y = sigmoid(x) for all `no` channels; xy = (2y-0.5+grid)*stride; wh = (2y)^2 * (anchor*stride)
// Input logits [B,na,ny,nx,no] (the layout Detect.forward produces with view/permute/contiguous), output rows
// [row0 + (a*ny+gy)*nx+gx] of pred[B,P_total,no]: level-major, anchor, gy, gx (SURVEY.md D2).
// Elementwise and HBM-bound: 8 B/element algorithmic (read logit, write prediction), fully coalesced.
#include "common.cuh"
#include "loss_math.h"

struct DecodeArgs {
  const float* logits;
  float* pred;
  int B, na, ny, nx, no, P_total, row0;
  float aw[ETB_NA], ah[ETB_NA];  // anchor_grid = anchors(grid units) * stride
  float stride;
};

__global__ void __launch_bounds__(256) detect_decode_kernel(const DecodeArgs A) {
  const int64_t per_img = (int64_t)A.na * A.ny * A.nx * A.no;
  const int64_t total = per_img * A.B;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = e / per_img;
    const int64_t r = e - b * per_img;
    const int64_t cell = r / A.no;
    const int ch = (int)(r - cell * A.no);
    const float y = etb_sigmoid(A.logits[e]);
    float v = y;
    if (ch < 4) {
      const int gx = (int)(cell % A.nx);
      const int gy = (int)((cell / A.nx) % A.ny);
      const int a = (int)(cell / ((int64_t)A.nx * A.ny));
      if (ch == 0) v = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(y, 2.0f), 0.5f), (float)gx), A.stride);
      else if (ch == 1) v = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(y, 2.0f), 0.5f), (float)gy), A.stride);
      else {
        const float q = __fmul_rn(y, 2.0f);
        v = __fmul_rn(__fmul_rn(q, q), ch == 2 ? A.aw[a] : A.ah[a]);
      }
    }
    A.pred[((int64_t)b * A.P_total + A.row0) * A.no + r] = v;
  }
}

extern "C" int etb_detect_decode(const float* logits, float* pred, int32_t B, int32_t na, int32_t ny, int32_t nx,
                                 int32_t no, int32_t P_total, int32_t row0, const float* anchors_grid, float stride,
                                 void* stream) {
  ETB_CHECK_ARG(logits && pred && anchors_grid);
  ETB_CHECK_ARG(B > 0 && na > 0 && na <= ETB_NA && ny > 0 && nx > 0 && no > 4 && row0 >= 0 && row0 + na * ny * nx <= P_total);
  DecodeArgs A;
  A.logits = logits; A.pred = pred;
  A.B = B; A.na = na; A.ny = ny; A.nx = nx; A.no = no; A.P_total = P_total; A.row0 = row0;
  for (int a = 0; a < na; ++a) {
    A.aw[a] = anchors_grid[2 * a] * stride;
    A.ah[a] = anchors_grid[2 * a + 1] * stride;
  }
  A.stride = stride;
  const int64_t total = (int64_t)B * na * ny * nx * no;
  int64_t blocks = (total + 255) / 256;
  const int64_t maxb = (int64_t)etb_num_sms() * 16;
  if (blocks > maxb) blocks = maxb;
  etb_launch(detect_decode_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, A);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
