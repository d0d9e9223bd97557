// bn.cu -- training-mode BatchNorm2d + SiLU / ReLU / Hardswish around the wgmma convolutions, forward and backward (K1/K2 tails).
//   Conv.forward = act(bn(conv(x)))           reference models/backbone/common.py:480-481
//   BN settings eps=1e-3, momentum=0.03       reference utils/torch_utils.py:162-171 (initialize_weights)
// Replaces, per Conv, ATen's batch_norm_collect_statistics + batch_norm_transform_input + SiLU (5 passes over the
// activation) by stats (1 read) + apply (1 read, 1 write), and in backward SiLU' + batch_norm_backward_reduce +
// batch_norm_backward_elemt (8 passes) by reduce (2 reads) + apply (2 reads, 1 write).
// Layout: y[M][cstride] bf16 (NHWC, M = N*H*W pixels), C % 8 == 0; one thread = one 16 B vector of 8 channels.
// All HBM-bound: algorithmic bytes = 2 B/element per pass listed above.
#include "common.cuh"

#define BN_THREADS 256

__device__ __forceinline__ void unpack8(const uint4 v, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 t = __bfloat1622float2(h[j]);
    f[2 * j] = t.x;
    f[2 * j + 1] = t.y;
  }
}
struct Vec2 { uint4 a, b; };
// streaming 16 B load; volatile so the UNROLL loads of a batch are issued back to back before the first use
__device__ __forceinline__ uint4 ldg_stream(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ void load8(const __nv_bfloat16* p, float* f) {
  const uint4 v = *reinterpret_cast<const uint4*>(p);
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 t = __bfloat1622float2(h[j]);
    f[2 * j] = t.x;
    f[2 * j + 1] = t.y;
  }
}
__device__ __forceinline__ void ldf8(const float* p, float* f) {   // 8 consecutive per-channel parameters
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float* f) {
  uint4 v;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) h[j] = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);
  *reinterpret_cast<uint4*>(p) = v;
}

// Per-channel reduction of up to two quantities.  Thread t owns channel group g = t % G (G = C/8 <= 256) and pixel lane
// t / G; rows advance by PL*gridDim.x with PL = floor(256/G), so g never changes.  When G does not divide 256 (YOLOv5m/x
// widths) the last 256 - PL*G threads own no lane and stay idle.  Block partials are combined through shared memory and
// written to out[blockIdx.x][NQ][C]: no atomics, no memset, and the second stage (reduce_partials) sums the rows in a
// fixed order, so the statistics are bit-reproducible run to run.
template <int NQ, int UNROLL, typename D, typename L, typename F>
__device__ __forceinline__ void channel_reduce(int M, int C, L&& load_row, F&& per_row, float* __restrict__ out /*[NQ][C]*/) {
  __shared__ float sh[NQ][BN_THREADS][8 + 1];
  const int G = C >> 3;
  const int g = threadIdx.x % G, pl = threadIdx.x / G, PL = BN_THREADS / G;
  float acc[NQ][8];
#pragma unroll
  for (int q = 0; q < NQ; ++q)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[q][j] = 0.f;
  const int step = (int)gridDim.x * PL;
  int r = pl < PL ? (int)blockIdx.x * PL + pl : M;
  for (; r + (UNROLL - 1) * step < M; r += UNROLL * step) {      // UNROLL independent rows in flight per thread
    D d[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) d[u] = load_row(r + u * step, g);
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) per_row(d[u], acc);
  }
  for (; r < M; r += step) per_row(load_row(r, g), acc);
#pragma unroll
  for (int q = 0; q < NQ; ++q)
#pragma unroll
    for (int j = 0; j < 8; ++j) sh[q][threadIdx.x][j] = acc[q][j];
  __syncthreads();
  // thread t < C*NQ... : channel c = t % C handled by threads [0, C) for each quantity
  for (int idx = threadIdx.x; idx < NQ * C; idx += BN_THREADS) {
    const int q = idx / C, c = idx - q * C;
    const int cg = c >> 3, cj = c & 7;
    float s = 0.f;
    for (int p = 0; p < PL; ++p) s += sh[q][p * G + cg][cj];
    out[(size_t)blockIdx.x * NQ * C + idx] = s;
  }
}

// Second stage: block (32 channels x 32 row groups); v[q] = sum over the nb partial rows of channel c, fixed order.
// Returns the totals to the threads with threadIdx.y == 0.
// CH x GR = 1024 threads: 32 x 32 for wide layers, 8 x 128 for C <= 256 (more blocks, shorter serial chains).
template <int BNR_CH, int BNR_GR>
__device__ __forceinline__ void reduce_partials(const float* __restrict__ partials, int nb, int C, int c, float* v0, float* v1) {
  __shared__ float red[2][BNR_GR][BNR_CH + 1];
  float a0 = 0.f, a1 = 0.f;
  if (c < C) {
    int b = threadIdx.y;
    for (; b + 3 * BNR_GR < nb; b += 4 * BNR_GR) {
      const float* p = partials + (size_t)b * 2 * C + c;
      const size_t st = (size_t)BNR_GR * 2 * C;
      const float x0 = __ldg(p), x1 = __ldg(p + st), x2 = __ldg(p + 2 * st), x3 = __ldg(p + 3 * st);
      const float y0 = __ldg(p + C), y1 = __ldg(p + st + C), y2 = __ldg(p + 2 * st + C), y3 = __ldg(p + 3 * st + C);
      a0 += (x0 + x1) + (x2 + x3);
      a1 += (y0 + y1) + (y2 + y3);
    }
    for (; b < nb; b += BNR_GR) {
      a0 += __ldg(partials + (size_t)b * 2 * C + c);
      a1 += __ldg(partials + (size_t)b * 2 * C + C + c);
    }
  }
  red[0][threadIdx.y][threadIdx.x] = a0;
  red[1][threadIdx.y][threadIdx.x] = a1;
  __syncthreads();
#pragma unroll
  for (int s = BNR_GR / 2; s >= 8; s >>= 1) {     // fixed-shape tree: deterministic
    if ((int)threadIdx.y < s) {
      red[0][threadIdx.y][threadIdx.x] += red[0][threadIdx.y + s][threadIdx.x];
      red[1][threadIdx.y][threadIdx.x] += red[1][threadIdx.y + s][threadIdx.x];
    }
    __syncthreads();
  }
  if (threadIdx.y == 0) {
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int g = 0; g < 8; ++g) { s0 += red[0][g][threadIdx.x]; s1 += red[1][g][threadIdx.x]; }
    *v0 = s0;
    *v1 = s1;
  }
}

// ---- forward statistics: sums[0][c] = sum y, sums[1][c] = sum y^2 ----
__global__ void __launch_bounds__(BN_THREADS) bn_stats_kernel(const __nv_bfloat16* __restrict__ y, int M, int C, int cs, float* __restrict__ sums) {
  channel_reduce<2, 8, uint4>(M, C, [&](int r, int g) { return ldg_stream(y + (size_t)r * cs + g * 8); },
                              [&](const uint4 v, float (*acc)[8]) {
    float f[8];
    unpack8(v, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { acc[0][j] += f[j]; acc[1][j] = fmaf(f[j], f[j], acc[1][j]); }
  }, sums);
}

// ---- finalize: batch mean / biased var -> scale, shift; running stats with the unbiased variance (torch semantics) ----
template <int BNR_CH, int BNR_GR>
__global__ void __launch_bounds__(BNR_CH * BNR_GR) bn_finalize_kernel(const float* __restrict__ partials, int nb, int M, int C,
                                                                       const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                                       float momentum, float* __restrict__ running_mean,
                                                                       float* __restrict__ running_var, float* __restrict__ scale,
                                                                       float* __restrict__ shift, float* __restrict__ mean_out,
                                                                       float* __restrict__ invstd_out) {
  const int c = blockIdx.x * BNR_CH + threadIdx.x;
  float sum = 0.f, sumsq = 0.f;
  reduce_partials<BNR_CH, BNR_GR>(partials, nb, C, c, &sum, &sumsq);
  if (c >= C || threadIdx.y != 0) return;
  const float inv = 1.0f / (float)M;
  const float mean = sum * inv;
  float var = fmaf(-mean, mean, sumsq * inv);
  var = fmaxf(var, 0.0f);
  const float invstd = rsqrtf(var + eps);
  const float sc = gamma[c] * invstd;
  scale[c] = sc;
  shift[c] = fmaf(-mean, sc, beta[c]);
  mean_out[c] = mean;
  invstd_out[c] = invstd;
  if (running_mean) {
    const float unbiased = M > 1 ? var * ((float)M / (float)(M - 1)) : var;
    running_mean[c] = fmaf(momentum, mean - running_mean[c], running_mean[c]);
    running_var[c] = fmaf(momentum, unbiased - running_var[c], running_var[c]);
  }
}

// sigmoid through ONE MUFU op: s = 0.5*tanh(0.5 z) + 0.5 (tanh.approx.f32, rel. error ~2^-11: below bf16 resolution)
__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float silu_f(float z) {          // z*sigmoid(z) = h + h*tanh(h), h = z/2
  const float h = 0.5f * z;
  return fmaf(h, tanh_approx(h), h);
}
// d silu(z)/dz = s*(1 + z*(1-s)),  s = sigmoid(z)
__device__ __forceinline__ float dsilu_f(float z) {
  const float s = fmaf(0.5f, tanh_approx(0.5f * z), 0.5f);
  return s * fmaf(z, 1.0f - s, 1.0f);
}

// act(z) / act'(z).  HSWISH selects the Hardswish instance of each kernel (act 4); the other instance reads act 0 / 1 / 2 at
// run time.  Hardswish as a third run-time case would cost the SiLU kernels registers (bn_act_bwd_apply 114 -> 128).
template <bool HSWISH>
__device__ __forceinline__ float bn_act(float z, int act) {
  return HSWISH ? hswish_f(z) : (act == 1 ? silu_f(z) : (act == 2 ? fmaxf(z, 0.f) : z));
}
template <bool HSWISH>
__device__ __forceinline__ float bn_dact(float z, int act) {   // ReLU'(0) = 0, as threshold_backward takes it
  return HSWISH ? dhswish_f(z) : (act == 1 ? dsilu_f(z) : (act == 2 ? (z > 0.f ? 1.f : 0.f) : 1.f));
}

// Index space of the apply kernels, in which every thread keeps one channel group g for its whole life.
//   POW2 (G = C/8 a power of two): e counts 16 B vectors, row = e >> lg; the grid stride (gridDim.x*256 vectors) is a
//     multiple of G, so g = e & (G-1) never changes.
//   otherwise (YOLOv5m/x widths): thread t owns g = t % G and row lane t / G < PL = floor(256/G), as in channel_reduce;
//     e counts rows (lg = 0) and advances by PL*gridDim.x.  The 256 - PL*G tail threads of a block return at once.
// Either way the loop body needs no division.  Returns false for an idle thread.
template <bool POW2>
__device__ __forceinline__ bool bn_apply_index(long M, int C, int* g, int* lg, long* e, long* stride, long* total) {
  const int G = C >> 3;
  if (POW2) {
    *lg = 31 - __clz(G);
    *total = M * G;
    *stride = (long)gridDim.x * blockDim.x;
    *e = (long)blockIdx.x * blockDim.x + threadIdx.x;
    *g = (int)(*e & (G - 1));
    return true;
  }
  const int PL = BN_THREADS / G, pl = threadIdx.x / G;
  *lg = 0;
  *total = M;
  *stride = (long)gridDim.x * PL;
  *e = (long)blockIdx.x * PL + pl;
  *g = threadIdx.x - pl * G;
  return pl < PL;
}

// ---- forward apply: a = act(y*scale + shift) ----
// A thread's channel group never changes (bn_apply_index): its scale/shift live in registers for the whole kernel and the
// loop body is 2 independent 16 B loads, 8 FMAs + SiLU, 2 stores.
template <bool HSWISH, bool POW2>
__global__ void __launch_bounds__(BN_THREADS) bn_act_apply_kernel(const __nv_bfloat16* __restrict__ y, const float* __restrict__ scale,
                                                                  const float* __restrict__ shift, __nv_bfloat16* __restrict__ out, long M, int C,
                                                                  int ycs, int ocs, int act, const __nv_bfloat16* __restrict__ res, int rcs) {
  int g, lg;
  long e, stride, total;
  if (!bn_apply_index<POW2>(M, C, &g, &lg, &e, &stride, &total)) return;
  float sc[8], sh[8];
  ldf8(scale + g * 8, sc); ldf8(shift + g * 8, sh);
  y += g * 8;
  out += g * 8;
  if (res) res += g * 8;
  auto body = [&](float* f, long r) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float z = fmaf(f[j], sc[j], sh[j]);
      f[j] = bn_act<HSWISH>(z, act);
    }
    if (res) {      // Bottleneck shortcut (common.py:499): x + cv2(cv1(x)); the sum is rounded once, from fp32
      float q[8];
      load8(res + r * rcs, q);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] += q[j];
    }
  };
  // 4 rows (4 x 16 B loads) in flight per thread: the loop is latency-bound, not bandwidth-bound, on the mid-size layers
  for (; e + 3 * stride < total; e += 4 * stride) {
    long r[4];
    uint4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      r[u] = (e + u * stride) >> lg;
      v[u] = *reinterpret_cast<const uint4*>(y + r[u] * ycs);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      float f[8];
      unpack8(v[u], f);
      body(f, r[u]);
      store8(out + r[u] * ocs, f);
    }
  }
  for (; e < total; e += stride) {
    const long r0 = e >> lg;
    float f0[8];
    load8(y + r0 * ycs, f0);
    body(f0, r0);
    store8(out + r0 * ocs, f0);
  }
}

// ---- backward reduce: sums[0][c] = sum dz, sums[1][c] = sum dz*xhat,  dz = da * act'(z) ----
template <bool HSWISH>
__global__ void __launch_bounds__(BN_THREADS) bn_act_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ da, const __nv_bfloat16* __restrict__ y,
                                                                       const float* __restrict__ scale, const float* __restrict__ shift,
                                                                       const float* __restrict__ mean, const float* __restrict__ invstd, int M,
                                                                       int C, int dacs, int ycs, int act, float* __restrict__ sums) {
  // per-thread channel group is fixed: hoist its parameters out of the row loop
  float sc[8], sh[8], mu[8], is[8];
  {
    const int g0 = threadIdx.x % (C >> 3);
    ldf8(scale + g0 * 8, sc); ldf8(shift + g0 * 8, sh); ldf8(mean + g0 * 8, mu); ldf8(invstd + g0 * 8, is);
#pragma unroll
    for (int j = 0; j < 8; ++j) mu[j] = -mu[j] * is[j];     // xhat = y*invstd + (-mean*invstd): one FMA per element
  }
  channel_reduce<2, 4, Vec2>(M, C, [&](int r, int g) {
    Vec2 v;
    v.a = ldg_stream(y + (size_t)r * ycs + g * 8);
    v.b = ldg_stream(da + (size_t)r * dacs + g * 8);
    return v;
  }, [&](const Vec2 v, float (*acc)[8]) {
    float fy[8], fd[8];
    unpack8(v.a, fy);
    unpack8(v.b, fd);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float z = fmaf(fy[j], sc[j], sh[j]);
      const float dz = fd[j] * bn_dact<HSWISH>(z, act);
      const float xh = fmaf(fy[j], is[j], mu[j]);
      acc[0][j] += dz;
      acc[1][j] = fmaf(dz, xh, acc[1][j]);
    }
  }, sums);
}

// ---- backward finalize: sums[2C] = totals of the partial rows; dbeta / dgamma written or accumulated (gradient arena) ----
template <int BNR_CH, int BNR_GR>
__global__ void __launch_bounds__(BNR_CH * BNR_GR) bn_bwd_finalize_kernel(const float* __restrict__ partials, int nb, int C, float* __restrict__ sums,
                                                                           float* __restrict__ dgamma, float* __restrict__ dbeta, int accumulate) {
  const int c = blockIdx.x * BNR_CH + threadIdx.x;
  float s0 = 0.f, s1 = 0.f;
  reduce_partials<BNR_CH, BNR_GR>(partials, nb, C, c, &s0, &s1);
  if (c >= C || threadIdx.y != 0) return;
  sums[c] = s0;
  sums[C + c] = s1;
  if (accumulate) {
    dbeta[c] += s0;
    dgamma[c] += s1;
  } else {
    dbeta[c] = s0;
    dgamma[c] = s1;
  }
}

// ---- backward apply: dy = gamma*invstd * (dz - sum_dz/M - xhat*sum_dz_xhat/M) ----
// Same fixed-channel-group structure as the forward apply: the six per-channel vectors are folded into five register
// arrays once per thread.
template <bool HSWISH, bool POW2>
__global__ void __launch_bounds__(BN_THREADS, 2) bn_act_bwd_apply_kernel(const __nv_bfloat16* __restrict__ da, const __nv_bfloat16* __restrict__ y,
                                                                      const float* __restrict__ scale, const float* __restrict__ shift,
                                                                      const float* __restrict__ mean, const float* __restrict__ invstd,
                                                                      const float* __restrict__ sums, long M, int C, int dacs, int ycs, int ocs,
                                                                      int act, __nv_bfloat16* __restrict__ dy) {
  const float invM = 1.0f / (float)M;
  int g, lg;
  long e, stride, total;
  if (!bn_apply_index<POW2>(M, C, &g, &lg, &e, &stride, &total)) return;
  // dy = sc*(dz - k0 - xhat*k1), xhat = y*invstd - mean*invstd  ==>  dy = sc*dz + y*P + Q with
  // P = -sc*invstd*k1, Q = -sc*(k0 - mean*invstd*k1): four register arrays per thread instead of six
  float sc[8], sh[8], P[8], Q[8];
  {
    float a1[8], mu[8], k0[8], k1[8];
    ldf8(scale + g * 8, sc); ldf8(shift + g * 8, sh); ldf8(invstd + g * 8, a1); ldf8(mean + g * 8, mu);
    ldf8(sums + g * 8, k0); ldf8(sums + C + g * 8, k1);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float k1m = k1[j] * invM * a1[j];
      P[j] = -sc[j] * k1m;
      Q[j] = -sc[j] * fmaf(-mu[j], k1m, k0[j] * invM);
    }
  }
  y += g * 8;
  da += g * 8;
  dy += g * 8;
  auto body = [&](const float* fy, float* fd) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float z = fmaf(fy[j], sc[j], sh[j]);
      const float dz = fd[j] * bn_dact<HSWISH>(z, act);
      fd[j] = fmaf(sc[j], dz, fmaf(fy[j], P[j], Q[j]));   // sc = gamma*invstd
    }
  };
  // 4 rows (8 x 16 B loads) in flight per thread
  for (; e + 3 * stride < total; e += 4 * stride) {
    long r[4];
    uint4 vy[4], vd[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      r[u] = (e + u * stride) >> lg;
      vy[u] = *reinterpret_cast<const uint4*>(y + r[u] * ycs);
      vd[u] = *reinterpret_cast<const uint4*>(da + r[u] * dacs);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      float fy[8], fd[8];
      unpack8(vy[u], fy);
      unpack8(vd[u], fd);
      body(fy, fd);
      store8(dy + r[u] * ocs, fd);
    }
  }
  for (; e < total; e += stride) {
    const long r0 = e >> lg;
    float y0[8], d0[8];
    load8(y + r0 * ycs, y0);
    load8(da + r0 * dacs, d0);
    body(y0, d0);
    store8(dy + r0 * ocs, d0);
  }
}

// One full wave: grid = min(needed, SMs x resident blocks of THIS kernel) so a grid-stride loop never runs a partial
// second wave (the reduce kernels hold 3-5 blocks per SM; a fixed 8-per-SM grid left the last wave 60% empty).
template <typename K>
static inline long bn_wave(K kernel) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, BN_THREADS, 0) != cudaSuccess || per_sm < 1) per_sm = 2;
  return (long)etb_num_sms() * per_sm;
}
#define BN_WAVE(kernel)                           \
  ([]() -> long {                                 \
    static long w = 0;                            \
    if (!w) w = bn_wave(kernel);                  \
    return w;                                     \
  }())
static inline unsigned bn_grid(long work_threads, long cap) {
  long b = (work_threads + BN_THREADS - 1) / BN_THREADS;
  return (unsigned)(b > cap ? cap : (b < 1 ? 1 : b));
}
static inline bool bn_act_ok(int act) { return act == 0 || act == 1 || act == 2 || act == 4; }
static inline bool bn_c_ok(int C) { return C >= 8 && C % 8 == 0 && (C / 8) <= BN_THREADS; }
static inline bool bn_pow2(int C) { return ((C / 8) & (C / 8 - 1)) == 0; }
// vectors (POW2) or rows (otherwise) of work threads of an apply kernel: both give ceil(M / PL) blocks
static inline long bn_apply_threads(long M, int C) {
  const int PL = BN_THREADS / (C / 8);
  return bn_pow2(C) ? M * (C / 8) : (M + PL - 1) / PL * BN_THREADS;
}
// the four instances of an apply kernel: the Hardswish one (act 4) or the run-time SiLU / ReLU / none one, each with the
// power-of-two or the general channel mapping
#define BN_APPLY_LAUNCH(kernel, M, C, act, stream, ...)                                                                   \
  do {                                                                                                                    \
    const long wt_ = bn_apply_threads((M), (C));                                                                          \
    if ((act) == 4 && bn_pow2(C))                                                                                         \
      etb_launch(kernel<true, true>, dim3(bn_grid(wt_, BN_WAVE((kernel<true, true>)))), dim3(BN_THREADS), 0, (stream), __VA_ARGS__);     \
    else if ((act) == 4)                                                                                                  \
      etb_launch(kernel<true, false>, dim3(bn_grid(wt_, BN_WAVE((kernel<true, false>)))), dim3(BN_THREADS), 0, (stream), __VA_ARGS__);   \
    else if (bn_pow2(C))                                                                                                  \
      etb_launch(kernel<false, true>, dim3(bn_grid(wt_, BN_WAVE((kernel<false, true>)))), dim3(BN_THREADS), 0, (stream), __VA_ARGS__);   \
    else                                                                                                                  \
      etb_launch(kernel<false, false>, dim3(bn_grid(wt_, BN_WAVE((kernel<false, false>)))), dim3(BN_THREADS), 0, (stream), __VA_ARGS__); \
  } while (0)

static inline long bn_reduce_blocks(long M, int C, long wave) {
  const int PL = BN_THREADS / (C / 8);
  long blocks = (M + PL - 1) / PL;
  // at least ~64 KB of activation per block so the partial-row count stays small for the second stage
  const long by_bytes = (M * C * 2 + 65535) / 65536;
  if (blocks > by_bytes) blocks = by_bytes;
  if (blocks > wave) blocks = wave;
  return blocks < 1 ? 1 : blocks;
}

// rows of the partial-sum buffer ([rows][2][C] floats) the reduction kernels need: which = 0 forward stats, 1 backward reduce
extern "C" int32_t etb_bn_partial_rows(int64_t M, int32_t C, int32_t which) {
  if (M <= 0 || !bn_c_ok(C)) return 0;
  return (int32_t)bn_reduce_blocks((long)M, C, which ? BN_WAVE(bn_act_bwd_reduce_kernel<false>) : BN_WAVE(bn_stats_kernel));
}

// partials: [rows = etb_bn_partial_rows(M,C,0)][2][C] floats, fully overwritten.  y [M][y_cstride] bf16.
extern "C" int etb_bn_stats(const void* y_bf16, int64_t M, int32_t C, int32_t y_cstride, float* partials, int32_t rows, void* stream) {
  ETB_CHECK_ARG(y_bf16 && partials && M > 0 && M < (1ll << 31) && bn_c_ok(C) && y_cstride % 8 == 0 && y_cstride >= C);
  ETB_CHECK_ARG(rows == etb_bn_partial_rows(M, C, 0));
  etb_launch(bn_stats_kernel, dim3((unsigned)rows), dim3(BN_THREADS), 0, (cudaStream_t)stream, (const __nv_bfloat16*)y_bf16, (int)M, C, y_cstride, partials);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

extern "C" int etb_bn_finalize(const float* partials, int32_t rows, int64_t M, int32_t C, const float* gamma, const float* beta, float eps,
                               float momentum, float* running_mean, float* running_var, float* scale, float* shift, float* mean, float* invstd,
                               void* stream) {
  ETB_CHECK_ARG(partials && rows > 0 && gamma && beta && scale && shift && mean && invstd && M > 0 && C > 0);
  if (C <= 256)
    etb_launch(bn_finalize_kernel<8, 128>, dim3((C + 7) / 8), dim3(dim3(8, 128)), 0, (cudaStream_t)stream, partials, rows, (int)M, C, gamma, beta, eps, momentum, running_mean,
                                                                                      running_var, scale, shift, mean, invstd);
  else
    etb_launch(bn_finalize_kernel<32, 32>, dim3((C + 31) / 32), dim3(dim3(32, 32)), 0, (cudaStream_t)stream, partials, rows, (int)M, C, gamma, beta, eps, momentum, running_mean,
                                                                                        running_var, scale, shift, mean, invstd);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

extern "C" int etb_bn_act_apply_res(const void* y_bf16, const float* scale, const float* shift, const void* res_bf16, void* out_bf16,
                                    int64_t M, int32_t C, int32_t y_cstride, int32_t res_cstride, int32_t out_cstride, int32_t act,
                                    void* stream) {
  ETB_CHECK_ARG(y_bf16 && scale && shift && out_bf16 && M > 0 && bn_c_ok(C) && y_cstride % 8 == 0 && out_cstride % 8 == 0);
  ETB_CHECK_ARG(!res_bf16 || (res_cstride % 8 == 0 && res_cstride >= C));
  ETB_CHECK_ARG(bn_act_ok(act));
  BN_APPLY_LAUNCH(bn_act_apply_kernel, M, C, act, (cudaStream_t)stream, (const __nv_bfloat16*)y_bf16, scale, shift, (__nv_bfloat16*)out_bf16,
                  (long)M, C, y_cstride, out_cstride, act, (const __nv_bfloat16*)res_bf16, res_cstride);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
extern "C" int etb_bn_act_apply(const void* y_bf16, const float* scale, const float* shift, void* out_bf16, int64_t M, int32_t C,
                                int32_t y_cstride, int32_t out_cstride, int32_t act, void* stream) {
  return etb_bn_act_apply_res(y_bf16, scale, shift, nullptr, out_bf16, M, C, y_cstride, 0, out_cstride, act, stream);
}

// partials: [rows = etb_bn_partial_rows(M,C,1)][2][C] floats: per-block [sum dz][sum dz*xhat], fully overwritten
extern "C" int etb_bn_act_bwd_reduce(const void* da_bf16, const void* y_bf16, const float* scale, const float* shift, const float* mean,
                                     const float* invstd, int64_t M, int32_t C, int32_t da_cstride, int32_t y_cstride, int32_t act,
                                     float* partials, int32_t rows, void* stream) {
  ETB_CHECK_ARG(da_bf16 && y_bf16 && scale && shift && mean && invstd && partials && M > 0 && M < (1ll << 31) && bn_c_ok(C));
  ETB_CHECK_ARG(da_cstride % 8 == 0 && y_cstride % 8 == 0 && rows == etb_bn_partial_rows(M, C, 1) && bn_act_ok(act));
  etb_launch(act == 4 ? bn_act_bwd_reduce_kernel<true> : bn_act_bwd_reduce_kernel<false>, dim3((unsigned)rows), dim3(BN_THREADS), 0, (cudaStream_t)stream, (const __nv_bfloat16*)da_bf16, (const __nv_bfloat16*)y_bf16, scale, shift, mean, invstd, (int)M, C, da_cstride, y_cstride, act, partials);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

// sums[2C] = column totals of partials; dbeta = sum dz, dgamma = sum dz*xhat, written (accumulate = 0) or added in place
// (accumulate = 1: dgamma / dbeta are the parameters' .grad in the gradient arena)
extern "C" int etb_bn_act_bwd_finalize(const float* partials, int32_t rows, int32_t C, float* sums, float* dgamma, float* dbeta,
                                       int32_t accumulate, void* stream) {
  ETB_CHECK_ARG(partials && rows > 0 && C > 0 && sums && dgamma && dbeta);
  if (C <= 256)
    etb_launch(bn_bwd_finalize_kernel<8, 128>, dim3((C + 7) / 8), dim3(dim3(8, 128)), 0, (cudaStream_t)stream, partials, rows, C, sums, dgamma, dbeta, accumulate);
  else
    etb_launch(bn_bwd_finalize_kernel<32, 32>, dim3((C + 31) / 32), dim3(dim3(32, 32)), 0, (cudaStream_t)stream, partials, rows, C, sums, dgamma, dbeta, accumulate);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

extern "C" int etb_bn_act_bwd_apply(const void* da_bf16, const void* y_bf16, const float* scale, const float* shift, const float* mean,
                                    const float* invstd, const float* sums, int64_t M, int32_t C, int32_t da_cstride, int32_t y_cstride,
                                    int32_t dy_cstride, int32_t act, void* dy_bf16, void* stream) {
  ETB_CHECK_ARG(da_bf16 && y_bf16 && scale && shift && mean && invstd && sums && dy_bf16 && M > 0 && bn_c_ok(C));
  ETB_CHECK_ARG(da_cstride % 8 == 0 && y_cstride % 8 == 0 && dy_cstride % 8 == 0 && bn_act_ok(act));
  BN_APPLY_LAUNCH(bn_act_bwd_apply_kernel, M, C, act, (cudaStream_t)stream, (const __nv_bfloat16*)da_bf16, (const __nv_bfloat16*)y_bf16, scale,
                  shift, mean, invstd, sums, (long)M, C, da_cstride, y_cstride, dy_cstride, act, (__nv_bfloat16*)dy_bf16);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
