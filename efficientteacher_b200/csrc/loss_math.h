// loss_math.h -- scalar math of the fused loss kernels, shared between device code (loss.cu) and a host
// build used only by the CPU unit tests (tests/hostmath) to check the hand-written backward against
// torch autograd without a GPU.  fp32 throughout, like the reference's CPU path.
//   CIoU            reference utils/metrics.py:207-249 (x1y1x2y2=False, CIoU=True, eps=1e-7)
//   box decode      reference models/loss/loss.py:162-165   pxy = 2*sigmoid-0.5 ; pwh = (2*sigmoid)^2*anchor
//   BCEWithLogits   torch.nn.BCEWithLogitsLoss(pos_weight=1): max(x,0) - x*z + log1p(exp(-|x|))
//   pos_weight + FocalLoss   reference models/loss/loss.py:37-64,106-116 (etb_det_bce / etb_det_bce_grad)
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define ETB_HD __host__ __device__ __forceinline__
#else
#define ETB_HD inline
#endif

#define ETB_CIOU_EPS 1e-7f

ETB_HD float etb_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

ETB_HD float etb_bce_logits(float x, float z) { return fmaxf(x, 0.0f) - x * z + log1pf(expf(-fabsf(x))); }

// softplus(-x) = -log(sigmoid(x))
ETB_HD float etb_softplus_neg(float x) { return fmaxf(-x, 0.0f) + log1pf(expf(-fabsf(x))); }

#define ETB_FOCAL_ALPHA 0.25f

// One element of the reference's detection criterion (models/loss/loss.py:37-64, :106-116):
//   BCEWithLogitsLoss(pos_weight=pw):  (1-z)*x + (1+(pw-1)*z)*softplus(-x)  = bce(x,z) + (pw-1)*z*softplus(-x)
//   FocalLoss(., gamma, alpha=0.25) when gamma > 0: that times alpha_t * (1-p_t)^gamma,
//     p_t = z*s + (1-z)*(1-s), alpha_t = z*alpha + (1-z)*(1-alpha), s = sigmoid(x).
// The positive-weight term adds exactly +0 when pw == 1, so the defaults give etb_bce_logits bit for bit.
ETB_HD float etb_det_bce(float x, float z, float pw, float gamma) {
  const float b = etb_bce_logits(x, z) + (pw - 1.0f) * z * etb_softplus_neg(x);
  if (gamma > 0.0f) {
    const float s = etb_sigmoid(x);
    const float pt = z * s + (1.0f - z) * (1.0f - s);
    const float at = z * ETB_FOCAL_ALPHA + (1.0f - z) * (1.0f - ETB_FOCAL_ALPHA);
    return b * (at * powf(1.0f - pt, gamma));
  }
  return b;
}

// d etb_det_bce / dx.  Weighted BCE: (1+(pw-1)z)*s - pw*z, written as (s - z) + (pw-1)*z*(s-1) (+0 when pw == 1).
// Focal: alpha_t * (b' * m + b * gamma*(1-p_t)^(gamma-1) * (-(2z-1)*s*(1-s))), m = (1-p_t)^gamma.
ETB_HD float etb_det_bce_grad(float x, float z, float pw, float gamma) {
  const float s = etb_sigmoid(x);
  const float db = (s - z) + (pw - 1.0f) * z * (s - 1.0f);
  if (gamma > 0.0f) {
    const float b = etb_bce_logits(x, z) + (pw - 1.0f) * z * etb_softplus_neg(x);
    const float pt = z * s + (1.0f - z) * (1.0f - s);
    const float at = z * ETB_FOCAL_ALPHA + (1.0f - z) * (1.0f - ETB_FOCAL_ALPHA);
    const float q = 1.0f - pt;
    const float m = powf(q, gamma);
    const float dm = gamma * powf(q, gamma - 1.0f) * (-(2.0f * z - 1.0f) * s * (1.0f - s));
    return at * (db * m + b * dm);
  }
  return db;
}

// CIoU of predicted box (px,py,pw,ph) vs target (tx,ty,tw,th), both centre/size.
// If g != nullptr also returns d(ciou)/d(px,py,pw,ph) in g[0..3] (alpha treated as a constant, metrics.py:242-243).
ETB_HD float etb_ciou(float px, float py, float pw, float ph, float tx, float ty, float tw, float th, float* g) {
  const float eps = ETB_CIOU_EPS;
  const float b1x1 = px - pw / 2, b1x2 = px + pw / 2, b1y1 = py - ph / 2, b1y2 = py + ph / 2;
  const float b2x1 = tx - tw / 2, b2x2 = tx + tw / 2, b2y1 = ty - th / 2, b2y2 = ty + th / 2;
  const float iw_raw = fminf(b1x2, b2x2) - fmaxf(b1x1, b2x1);
  const float ih_raw = fminf(b1y2, b2y2) - fmaxf(b1y1, b2y1);
  const float iw = fmaxf(iw_raw, 0.0f), ih = fmaxf(ih_raw, 0.0f);
  const float inter = iw * ih;
  const float w1 = b1x2 - b1x1, h1 = b1y2 - b1y1 + eps;
  const float w2 = b2x2 - b2x1, h2 = b2y2 - b2y1 + eps;
  const float uni = w1 * h1 + w2 * h2 - inter + eps;
  const float iou = inter / uni;
  const float cw = fmaxf(b1x2, b2x2) - fminf(b1x1, b2x1);
  const float ch = fmaxf(b1y2, b2y2) - fminf(b1y1, b2y1);
  const float c2 = cw * cw + ch * ch + eps;
  const float dx = b2x1 + b2x2 - b1x1 - b1x2, dy = b2y1 + b2y2 - b1y1 - b1y2;
  const float rho2 = (dx * dx + dy * dy) / 4;
  const float kv = 4.0f / (3.14159265358979323846f * 3.14159265358979323846f);
  const float u1 = w1 / h1;
  const float dat = atanf(w2 / h2) - atanf(u1);
  const float v = kv * dat * dat;
  const float alpha = v / (v - iou + (1.0f + eps));
  const float ciou = iou - (rho2 / c2 + v * alpha);
  if (g) {
    // reverse mode with d(ciou)=1
    const float g_iou = 1.0f, g_rho2 = -1.0f / c2, g_c2 = rho2 / (c2 * c2), g_v = -alpha;
    float g_inter = g_iou / uni;
    const float g_uni = -g_iou * inter / (uni * uni);
    float g_w1 = g_uni * h1, g_h1 = g_uni * w1;
    g_inter += -g_uni;
    const float g_at1 = -g_v * kv * 2.0f * dat;  // d v / d atan(w1/h1)
    const float dat1 = 1.0f / (1.0f + u1 * u1);
    g_w1 += g_at1 * dat1 / h1;
    g_h1 += g_at1 * dat1 * (-w1 / (h1 * h1));
    const float g_cw = g_c2 * 2.0f * cw, g_ch = g_c2 * 2.0f * ch;
    float gx1 = 0.f, gx2 = 0.f, gy1 = 0.f, gy2 = 0.f;  // grads of b1x1,b1x2,b1y1,b1y2
    if (b1x2 > b2x2) gx2 += g_cw; else if (b1x2 == b2x2) gx2 += 0.5f * g_cw;
    if (b1x1 < b2x1) gx1 -= g_cw; else if (b1x1 == b2x1) gx1 -= 0.5f * g_cw;
    if (b1y2 > b2y2) gy2 += g_ch; else if (b1y2 == b2y2) gy2 += 0.5f * g_ch;
    if (b1y1 < b2y1) gy1 -= g_ch; else if (b1y1 == b2y1) gy1 -= 0.5f * g_ch;
    const float g_dx = g_rho2 * dx / 2.0f, g_dy = g_rho2 * dy / 2.0f;
    gx1 -= g_dx; gx2 -= g_dx; gy1 -= g_dy; gy2 -= g_dy;
    const float g_iw = (iw_raw >= 0.0f) ? g_inter * ih : 0.0f;
    const float g_ih = (ih_raw >= 0.0f) ? g_inter * iw : 0.0f;
    if (b1x2 < b2x2) gx2 += g_iw; else if (b1x2 == b2x2) gx2 += 0.5f * g_iw;
    if (b1x1 > b2x1) gx1 -= g_iw; else if (b1x1 == b2x1) gx1 -= 0.5f * g_iw;
    if (b1y2 < b2y2) gy2 += g_ih; else if (b1y2 == b2y2) gy2 += 0.5f * g_ih;
    if (b1y1 > b2y1) gy1 -= g_ih; else if (b1y1 == b2y1) gy1 -= 0.5f * g_ih;
    gx2 += g_w1; gx1 -= g_w1; gy2 += g_h1; gy1 -= g_h1;
    g[0] = gx1 + gx2;
    g[1] = gy1 + gy2;
    g[2] = (gx2 - gx1) / 2.0f;
    g[3] = (gy2 - gy1) / 2.0f;
  }
  return ciou;
}

// Box branch of one matched row: logits l[0..3], anchor (aw,ah), target tbox (tx,ty,tw,th).
// Returns ciou; if gl != nullptr, gl[0..3] = d(ciou)/d(l[0..3]).
ETB_HD float etb_row_ciou(const float* l, float aw, float ah, const float* tb, float* gl) {
  const float s0 = etb_sigmoid(l[0]), s1 = etb_sigmoid(l[1]), s2 = etb_sigmoid(l[2]), s3 = etb_sigmoid(l[3]);
  const float px = s0 * 2.0f - 0.5f, py = s1 * 2.0f - 0.5f;
  const float q2 = s2 * 2.0f, q3 = s3 * 2.0f;
  const float pw = q2 * q2 * aw, ph = q3 * q3 * ah;
  float g[4];
  const float c = etb_ciou(px, py, pw, ph, tb[0], tb[1], tb[2], tb[3], gl ? g : nullptr);
  if (gl) {
    gl[0] = g[0] * 2.0f * s0 * (1.0f - s0);
    gl[1] = g[1] * 2.0f * s1 * (1.0f - s1);
    gl[2] = g[2] * 2.0f * q2 * aw * 2.0f * s2 * (1.0f - s2);
    gl[3] = g[3] * 2.0f * q3 * ah * 2.0f * s3 * (1.0f - s3);
  }
  return c;
}
