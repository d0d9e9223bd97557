// conv_wgmma.cu -- implicit-GEMM convolution on the Hopper tensor cores (wgmma), fed by TMA (K1/K2/K5).
//
// Replaces cuDNN conv + BN(eval) + SiLU (+ residual add / Detect bias + permute copy) behind
//   Conv.forward        reference models/backbone/common.py:471-484
//   Bottleneck.forward  reference models/backbone/common.py:534-544   (residual add fused in the epilogue)
//   Detect.forward      reference models/head/yolov5_head.py:55,66     (1x1 conv + bias, scattered to [B,3,ny,nx,85])
// and the data / weight gradients of the training convolutions.
//
// GEMM view per CTA:  D[128 pixels, BN couts] += A[128 pixels, 64 ch] * B[BN couts, 64 ch]^T  over taps x channel blocks.
//   * A (activations, NHWC bf16) comes straight from global memory through a 4-D TMA tile
//     {64 ch, TW, TH, 1 image}; the tap shift (kh,kw) is a coordinate offset and the zero padding is TMA's
//     out-of-bounds fill, so no im2col buffer exists.  Stride-2 convs use the tensor map's element strides.
//   * B (weights, [Cout][kh*kw*Cin] bf16, K-major) is a 2-D TMA tile {64, BN}.
//   * both land in 128B-swizzled shared memory = the canonical K-major wgmma layout.
//   * warpgroup roles: warpgroup 0 is the TMA producer (one elected lane of its first warp issues), warpgroups 1 and 2
//     each own 64 of the 128 pixel rows and issue wgmma.m64nBNk16 x4 per stage; the fp32 accumulator lives in their
//     registers, and the epilogue (folded BN scale/bias -> SiLU -> +residual -> bf16 NHWC store at a channel offset of a
//     wider buffer, so torch.cat is free) runs straight from those registers.
//   * every mbarrier wait is bounded (trap after ~2 s) so a descriptor bug cannot hang the GPU.
#include "common.cuh"
#include <cuda.h>

#define CONV_BLOCK_M 128
#define CONV_BLOCK_K 64
#define CONV_THREADS 384     // warpgroup 0: TMA producer; warpgroups 1-2: wgmma consumers (64 rows each)
#define CONV_SMEM_STAGES_BYTES (192 * 1024)   // operand ring per CTA (H100: up to 227 KB of shared memory per block)

// ------------------------------------------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// bounded wait: a wrong descriptor / byte count must fail loudly, never hang the box.  No printf here: a function call
// inside the consumers' K loop would make ptxas serialize every wgmma.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000ll) __trap();
  }
}
// One lane of a CONVERGED warp (elect.sync): the producer warp runs its loop with all 32 lanes (warp-uniform control flow)
// and wraps only the TMA instructions in `if (elect_one())`.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_4d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)map) : "memory");
}

// wgmma shared-memory matrix descriptor, 128B swizzle: [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [62,64) 1 = SW128.
//   K-major operand:  LBO unused (1), SBO = 1024 B (8 rows x 128 B); a K=16 step is +32 B inside the swizzle atom.
//   MN-major operand: LBO = byte distance between 64-element MN groups, SBO = 1024 B (8 K rows); a K=16 step is +2048 B.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) | ((uint64_t)(1024 >> 4) << 32) |
         ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
template <int R>
__device__ __forceinline__ void acc_fence(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, bf16 operands from shared memory, fp32 accumulator in registers.
// TA / TB = 1: the operand is MN-major (transposed) instead of K-major.  Fragment of thread t of the warpgroup:
// d[j*4 + i*2 + e] = D[16*(t/32) + (t%32)/4 + 8*i][8*j + 2*(t%4) + e].
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_tile(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  if (BN == 128) wgmma_m64n128k16<TA, TB>(d, adesc, bdesc, scale_d);
  else wgmma_m64n64k16<TA, TB>(d, adesc, bdesc, scale_d);
}

// ------------------------------------------------------------------------------------------------- kernel
struct ConvKArgs {
  int ntaps;              // filter taps visited (kh*kw forward; 1/2/4 per parity class of a stride-2 dgrad)
  signed char tap_dh[12], tap_dw[12];   // input coordinate = tile origin * stride + tap offset (zero padding = TMA OOB fill)
  int kblocks;            // K channels / 64 per tap
  int stride;
  int out_os, out_ph, out_pw;           // output pixel (oh,ow) is stored at (oh*out_os+out_ph, ow*out_os+out_pw) ...
  int out_H, out_W;                     // ... of an out_H x out_W plane (dgrad of stride-2 convs fills one parity lattice)
  int accumulate;         // out_mode 0: y += result (gradient accumulation for tensors with several consumers)
  int TW, TH;             // output tile (TW*TH <= 128 rows)
  int tiles_w, tiles_h;   // per image
  int nimg;               // images (1 in the flat pointwise tiling)
  int Ho, Wo, Cout;
  int y_cstride, y_coffset;
  int res_cstride, res_coffset;
  int act;                // 0 none, 1 SiLU, 2 ReLU (EPI 1), 4 Hardswish (EPI 3)
  int out_mode;           // 0: bf16 NHWC ; 1: fp32 Detect layout [N, na, Ho, Wo, no] with c = a*no + o
  int det_no, det_hw;     // outputs per anchor, pixels per image (Detect layout)
  const float* scale;     // [Cout] or null (=1)
  const float* bias;      // [Cout] or null (=0)
  const __nv_bfloat16* residual;
  __nv_bfloat16* y;
  float* y_f32;
};

template <int BN>
struct ConvSmem {
  static constexpr int A_BYTES = CONV_BLOCK_M * 128;
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = CONV_SMEM_STAGES_BYTES / STAGE_BYTES;   // 6 (BN = 128) or 8 (BN = 64)
  static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
  static constexpr int TOTAL = BAR_OFF + 256 + 1024;        // + barriers + slack for the 1024 B alignment
};

__device__ __forceinline__ float conv_act(float x, int act) {
  if (act == 1) { const float h = 0.5f * x; float th; asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(h)); x = fmaf(h, th, h); }   // SiLU with one MUFU op
  else if (act == 2) x = fmaxf(x, 0.0f);
  return x;
}

// Epilogue of one consumer warpgroup's 64 x BN accumulator, straight from the wgmma fragment (see wgmma_m64n*k16): this
// thread owns pixel rows r0 and r0+8 and, per 8-column block j, the channel pair 8j + 2*(lane%4) + {0,1}.  EPI selects the
// fused tail at compile time so every register array is statically indexed:
//   EPI 0: raw bf16 store (+= existing when a.accumulate)       -- dgrad, training forward
//   EPI 1: v*scale+bias (folded BN) -> SiLU/ReLU -> (+residual) -- teacher forward
//   EPI 2: +bias, fp32 scatter into the Detect layout           -- head
//   EPI 3: EPI 1 with Hardswish                                 -- teacher forward of Hardswish layers
// (Hardswish as a third run-time case of EPI 1 would raise the SiLU instances from 122 / 89 to 132 / 98 registers.)
template <int BN, int EPI>
__device__ __forceinline__ void conv_epilogue(const ConvKArgs& a, const float* d, int n0, const bool* row_ok, const size_t* pix, int lane) {
  const size_t hw = (size_t)a.det_hw;
  const int na = EPI == 2 ? a.Cout / a.det_no : 1;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int gc = n0 + 8 * j + 2 * (lane & 3);
    if (gc >= a.Cout) continue;
    const bool pair = gc + 1 < a.Cout;
    float sc0 = 1.f, sc1 = 1.f, bi0 = 0.f, bi1 = 0.f;
    if ((EPI == 1 || EPI == 3) && a.scale) { sc0 = __ldg(a.scale + gc); sc1 = pair ? __ldg(a.scale + gc + 1) : 1.f; }
    if (EPI != 0 && a.bias) { bi0 = __ldg(a.bias + gc); bi1 = pair ? __ldg(a.bias + gc + 1) : 0.f; }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (!row_ok[i]) continue;
      float v0 = d[j * 4 + i * 2], v1 = d[j * 4 + i * 2 + 1];
      if (EPI == 2) {
        // Detect train layout: y[img][anchor][oh][ow][o], channel c = anchor*no + o  (yolov5_head.py:66)
        const size_t img_r = pix[i] / hw, pin = pix[i] - img_r * hw;   // pix is the global pixel index in both tilings
        const int an0 = gc / a.det_no, o0 = gc - an0 * a.det_no;
        a.y_f32[((img_r * na + an0) * hw + pin) * a.det_no + o0] = v0 + bi0;
        if (pair) {
          const int an1 = (gc + 1) / a.det_no, o1 = gc + 1 - an1 * a.det_no;
          a.y_f32[((img_r * na + an1) * hw + pin) * a.det_no + o1] = v1 + bi1;
        }
        continue;
      }
      __nv_bfloat16* yp = a.y + pix[i] * a.y_cstride + a.y_coffset + gc;
      if (EPI == 1 || EPI == 3) {
        v0 = EPI == 3 ? hswish_f(fmaf(v0, sc0, bi0)) : conv_act(fmaf(v0, sc0, bi0), a.act);
        v1 = EPI == 3 ? hswish_f(fmaf(v1, sc1, bi1)) : conv_act(fmaf(v1, sc1, bi1), a.act);
        if (a.residual) {     // Cout % 8 == 0 whenever a shortcut is fused: the pair is whole
          const float2 rf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(a.residual + pix[i] * a.res_cstride + a.res_coffset + gc));
          v0 += rf.x;
          v1 += rf.y;
        }
      }
      if (pair) {
        if (EPI == 0 && a.accumulate) {
          const float2 pf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(yp));
          v0 += pf.x;
          v1 += pf.y;
        }
        *reinterpret_cast<__nv_bfloat162*>(yp) = __floats2bfloat162_rn(v0, v1);
      } else {
        if (EPI == 0 && a.accumulate) v0 += __bfloat162float(*yp);
        *yp = __float2bfloat16(v0);
      }
    }
  }
}

// Persistent: gridDim.x CTAs walk the tile list (tile = blockIdx.x + i*gridDim.x; N tile fastest so the CTAs running
// concurrently share A tiles in L2).  The smem ring runs across tile boundaries, so the producer streams the operands of
// tile i+1 while the consumers run the epilogue of tile i.
template <int BN, int EPI>
__global__ void __launch_bounds__(CONV_THREADS, 1)
conv_fwd_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const ConvKArgs a) {
  using L = ConvSmem<BN>;
  constexpr int STAGES = L::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full = (uint64_t*)(smem + L::BAR_OFF);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int n_tiles = (a.Cout + BN - 1) / BN;
  const int m_tiles = a.tiles_w * a.tiles_h * a.nimg;
  const int total_tiles = n_tiles * m_tiles;
  const int kiters = a.ntaps * a.kblocks;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapA);
    tma_prefetch_desc(&mapB);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }   // 8 consumer warps release a stage
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (warp != 0) return;
    // ===== TMA producer: the whole warp runs the loop (uniform), one elected lane issues =====
    const uint32_t a_bytes = (uint32_t)(a.TW * a.TH * 128);
    int s = 0;                     // stage / phase advance incrementally: no divisions inside the K loop
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int n0 = (tile % n_tiles) * BN;
      int t = tile / n_tiles;
      const int tw_i = t % a.tiles_w; t /= a.tiles_w;
      const int th_i = t % a.tiles_h; t /= a.tiles_h;
      const int img = t;
      const int w0 = tw_i * a.TW * a.stride, h0 = th_i * a.TH * a.stride;
      int bk = 0;                  // K coordinate of the weight tile
      for (int tp = 0; tp < a.ntaps; ++tp) {
        const int wc = w0 + a.tap_dw[tp], hc = h0 + a.tap_dh[tp];
        for (int kb = 0; kb < a.kblocks; ++kb, bk += CONV_BLOCK_K) {
          mbar_wait(&empty[s], ph ^ 1u);
          uint8_t* sa = smem + s * L::STAGE_BYTES;
          uint8_t* sb = sa + L::A_BYTES;
          if (elect_one()) {
            mbar_expect_tx(&full[s], a_bytes + (uint32_t)L::B_BYTES);
            tma_load_4d(&mapA, &full[s], sa, kb * CONV_BLOCK_K, wc, hc, img);
            tma_load_2d(&mapB, &full[s], sb, bk, n0);
          }
          __syncwarp();
          if (++s == STAGES) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }
  // ===== consumers: warpgroup wg owns pixel rows 64*(wg-1) .. +63 of every tile =====
  const int cw = wg - 1;
  const int rbase = 64 * cw + 16 * (warp & 3) + (lane >> 2);
  const uint32_t a_off = (uint32_t)(cw * 64 * 128);
  float d[BN / 2];
  int s = 0;
  uint32_t ph = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    int prev = -1;
    for (int ki = 0; ki < kiters; ++ki) {
      mbar_wait(&full[s], ph);
      const uint32_t sa = smem_u32(smem + s * L::STAGE_BYTES);
      const uint64_t adesc = gmma_desc(sa + a_off, 16), bdesc = gmma_desc(sa + L::A_BYTES, 16);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < CONV_BLOCK_K / 16; ++k)   // +32 B per K=16 step inside the 128 B swizzle atom
        wgmma_tile<BN, 0, 0>(d, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (ki | k) != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();             // the previous stage's MMAs are done: hand it back to the producer
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
      prev = s;
      if (++s == STAGES) { s = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();
    acc_fence<BN / 2>(d);
    if (lane == 0) mbar_arrive(&empty[prev]);
    const int n0 = (tile % n_tiles) * BN;
    int t = tile / n_tiles;
    const int tw_i = t % a.tiles_w; t /= a.tiles_w;
    const int th_i = t % a.tiles_h; t /= a.tiles_h;
    const int img = t;
    bool row_ok[2];
    size_t pix[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = rbase + 8 * i;
      const int th = row / a.TW, tw = row - th * a.TW;
      const int oh = th_i * a.TH + th, ow = tw_i * a.TW + tw;
      row_ok[i] = (row < a.TW * a.TH) && (oh < a.Ho) && (ow < a.Wo);
      pix[i] = ((size_t)img * a.out_H + (size_t)(oh * a.out_os + a.out_ph)) * a.out_W + (size_t)(ow * a.out_os + a.out_pw);
    }
    conv_epilogue<BN, EPI>(a, d, n0, row_ok, pix, lane);
  }
}

// ------------------------------------------------------------------------------------------------- host side
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                        const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                        CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled get_encode() {
  static PFN_tmapEncodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (PFN_tmapEncodeTiled)p;
  }
  return fn;
}

static void pick_tile(int Wo, int Ho, int* TW, int* TH) {
  // maximise useful rows of the 128-row MMA tile: TW*TH <= 128, TW <= 128 (stride-2 boxes need 2*TW <= 256)
  double best = -1.0;
  for (int tw = 1; tw <= 128; ++tw) {
    if (tw > Wo && tw != 1) break;
    int th = 128 / tw;
    if (th > Ho) th = Ho;
    if (th < 1) continue;
    const long tiles = (long)((Wo + tw - 1) / tw) * ((Ho + th - 1) / th);
    const double eff = (double)Wo * Ho / ((double)tiles * 128.0);
    if (eff > best + 1e-9) { best = eff; *TW = tw; *TH = th; }
  }
}

template <int BN, int EPI>
static int launch_conv_e(const CUtensorMap& mA, const CUtensorMap& mB, const ConvKArgs& ka, dim3 grid, cudaStream_t st) {
  using L = ConvSmem<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    ETB_CHECK_CUDA(cudaFuncSetAttribute(conv_fwd_kernel<BN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
    attr_set = true;
  }
  etb_launch(conv_fwd_kernel<BN, EPI>, dim3(grid), dim3(CONV_THREADS), L::TOTAL, st, mA, mB, ka);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
template <int BN>
static int launch_conv(const CUtensorMap& mA, const CUtensorMap& mB, const ConvKArgs& ka, dim3 grid, cudaStream_t st) {
  if (ka.out_mode == 1) return launch_conv_e<BN, 2>(mA, mB, ka, grid, st);
  if (ka.act == 4) return launch_conv_e<BN, 3>(mA, mB, ka, grid, st);
  if (ka.scale || ka.bias || ka.act || ka.residual) return launch_conv_e<BN, 1>(mA, mB, ka, grid, st);
  return launch_conv_e<BN, 0>(mA, mB, ka, grid, st);
}

// One implicit-GEMM launch: D[pixels, rows_B] = sum_taps A(shifted) * B^T.  `ka` carries the epilogue.
struct GemmGeom {
  const void* a_ptr;          // NHWC bf16 tensor the A tiles come from
  int aN, aH, aW, aC, a_cstride;
  const void* b_ptr;          // [b_rows][ntaps*aC] bf16, K-major
  int b_rows;
  int tile_H, tile_W;         // per-image extent of the output-tile index space
  bool flat;                  // pointwise stride-1: all N*H*W pixels as one row-major [pixels, C] matrix
};

static int launch_gemm(const GemmGeom& g, ConvKArgs ka, cudaStream_t st) {
  PFN_tmapEncodeTiled enc = get_encode();
  if (!enc) {
    etb_set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return ETB_ERR_CUDA;
  }
  // aC need not be a multiple of the 64-channel K block: the A box is clipped by TMA (zero fill beyond aC) and the B operand is
  // packed with every tap padded to aCp = ceil64(aC) zero columns (etb_pack_weight Cin_pad / dgrad out_ld)
  ETB_CHECK_ARG(g.aC % 8 == 0 && g.aC > 0 && g.a_cstride >= g.aC && g.a_cstride % 8 == 0);
  const int aCp = (g.aC + CONV_BLOCK_K - 1) / CONV_BLOCK_K * CONV_BLOCK_K;
  ETB_CHECK_ARG((((uintptr_t)g.a_ptr) & 15) == 0 && (((uintptr_t)g.b_ptr) & 15) == 0);
  ETB_CHECK_ARG(ka.ntaps >= 1 && ka.ntaps <= 12);
  cuuint64_t gdim[4], gstr[3];
  cuuint32_t box[4], estr[4];
  int nimg;
  if (g.flat) {
    const long npix = (long)g.aN * g.aH * g.aW;
    ETB_CHECK_ARG(npix < (1l << 31));
    ka.TW = 128; ka.TH = 1;
    ka.Ho = 1; ka.Wo = (int)npix;
    ka.tiles_w = (int)((npix + 127) / 128); ka.tiles_h = 1;
    ka.out_os = 1; ka.out_ph = ka.out_pw = 0; ka.out_H = 1; ka.out_W = (int)npix;
    nimg = 1;
    gdim[0] = g.aC; gdim[1] = (cuuint64_t)npix; gdim[2] = 1; gdim[3] = 1;
    gstr[0] = (cuuint64_t)g.a_cstride * 2; gstr[1] = gstr[0] * (cuuint64_t)npix; gstr[2] = gstr[1];
    box[0] = 64; box[1] = 128; box[2] = 1; box[3] = 1;
    estr[0] = estr[1] = estr[2] = estr[3] = 1;
  } else {
    pick_tile(g.tile_W, g.tile_H, &ka.TW, &ka.TH);
    ka.Ho = g.tile_H; ka.Wo = g.tile_W;
    ka.tiles_w = (g.tile_W + ka.TW - 1) / ka.TW; ka.tiles_h = (g.tile_H + ka.TH - 1) / ka.TH;
    nimg = g.aN;
    gdim[0] = g.aC; gdim[1] = g.aW; gdim[2] = g.aH; gdim[3] = g.aN;
    gstr[0] = (cuuint64_t)g.a_cstride * 2; gstr[1] = gstr[0] * g.aW; gstr[2] = gstr[1] * g.aH;
    // with element strides the box is measured in input elements: ceil(box/stride) elements are loaded
    box[0] = 64; box[1] = (cuuint32_t)(ka.TW * ka.stride); box[2] = (cuuint32_t)(ka.TH * ka.stride); box[3] = 1;
    estr[0] = 1; estr[1] = (cuuint32_t)ka.stride; estr[2] = (cuuint32_t)ka.stride; estr[3] = 1;
    ETB_CHECK_ARG(box[1] <= 256 && box[2] <= 256);
  }
  CUtensorMap mA, mB;
  CUresult r = enc(&mA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(g.a_ptr), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    etb_set_error("cuTensorMapEncodeTiled(A) failed: %d", (int)r);
    return ETB_ERR_CUDA;
  }
  const long Ktot = (long)ka.ntaps * aCp;
  // the accumulator is held in the consumers' registers: 64 (BN = 128) or 32 (BN = 64) fp32 per thread
  const int BN = g.b_rows > 64 ? 128 : 64;
  cuuint64_t wdim[2] = {(cuuint64_t)Ktot, (cuuint64_t)g.b_rows};
  cuuint64_t wstr[1] = {(cuuint64_t)Ktot * 2};
  cuuint32_t wbox[2] = {64, (cuuint32_t)BN};
  cuuint32_t westr[2] = {1, 1};
  r = enc(&mB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(g.b_ptr), wdim, wstr, wbox, westr, CU_TENSOR_MAP_INTERLEAVE_NONE,
          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    etb_set_error("cuTensorMapEncodeTiled(B) failed: %d", (int)r);
    return ETB_ERR_CUDA;
  }
  ka.kblocks = aCp / CONV_BLOCK_K;
  ka.Cout = g.b_rows;
  ka.nimg = nimg;
  const long total_tiles = (long)ka.tiles_w * ka.tiles_h * nimg * ((g.b_rows + BN - 1) / BN);
  const long resident = (long)etb_num_sms();   // persistent: one CTA per SM (the operand ring takes 192 KB of shared memory)
  dim3 grid((unsigned)(total_tiles < resident ? total_tiles : resident), 1);
  return BN == 128 ? launch_conv<128>(mA, mB, ka, grid, st) : launch_conv<64>(mA, mB, ka, grid, st);
}

extern "C" size_t etb_conv_workspace_bytes(const EtbConvParams* cp) { (void)cp; return 0; }

extern "C" int etb_conv_fwd(const void* x_bf16, const void* w_bf16, const float* scale, const float* bias,
                            const void* residual_bf16, void* y_bf16, float* y_f32, const EtbConvParams* cp, void* workspace,
                            size_t workspace_bytes, void* stream) {
  (void)workspace; (void)workspace_bytes;
  ETB_CHECK_ARG(x_bf16 && w_bf16 && cp && (y_bf16 || y_f32));
  ETB_CHECK_ARG(cp->N > 0 && cp->H > 0 && cp->W > 0 && cp->Cin > 0 && cp->Cout > 0);
  ETB_CHECK_ARG(cp->act == 0 || cp->act == 1 || cp->act == 2 || cp->act == 4);
  ETB_CHECK_ARG(cp->kh >= 1 && cp->kw >= 1 && cp->kh * cp->kw <= 12 && (cp->stride == 1 || cp->stride == 2) && cp->pad >= 0);
  const int Ho = (cp->H + 2 * cp->pad - cp->kh) / cp->stride + 1;
  const int Wo = (cp->W + 2 * cp->pad - cp->kw) / cp->stride + 1;
  ETB_CHECK_ARG(Ho > 0 && Wo > 0);
  const bool det = (y_f32 != nullptr);
  if (!det) ETB_CHECK_ARG(cp->y_cstride % 8 == 0 && cp->y_coffset % 8 == 0 && cp->y_cstride >= cp->y_coffset + cp->Cout && (((uintptr_t)y_bf16) & 15) == 0);
  if (residual_bf16) ETB_CHECK_ARG(!det && cp->res_cstride % 8 == 0 && cp->res_coffset % 8 == 0 && cp->Cout % 8 == 0);
  if (det) ETB_CHECK_ARG(cp->det_no > 0 && cp->Cout % cp->det_no == 0);
  ConvKArgs ka;
  memset(&ka, 0, sizeof(ka));
  GemmGeom g;
  g.a_ptr = x_bf16; g.aN = cp->N; g.aH = cp->H; g.aW = cp->W; g.aC = cp->Cin; g.a_cstride = cp->x_cstride;
  g.b_ptr = w_bf16; g.b_rows = cp->Cout;
  g.tile_H = Ho; g.tile_W = Wo;
  g.flat = (cp->kh == 1 && cp->kw == 1 && cp->stride == 1 && cp->pad == 0);
  ka.ntaps = cp->kh * cp->kw;
  for (int kh = 0; kh < cp->kh; ++kh)
    for (int kw = 0; kw < cp->kw; ++kw) {
      ka.tap_dh[kh * cp->kw + kw] = (signed char)(kh - cp->pad);
      ka.tap_dw[kh * cp->kw + kw] = (signed char)(kw - cp->pad);
    }
  ka.stride = cp->stride;
  ka.out_os = 1; ka.out_ph = ka.out_pw = 0; ka.out_H = Ho; ka.out_W = Wo;
  ka.y_cstride = cp->y_cstride; ka.y_coffset = cp->y_coffset;
  ka.res_cstride = cp->res_cstride; ka.res_coffset = cp->res_coffset;
  ka.act = cp->act;
  ka.out_mode = det ? 1 : 0;
  ka.det_no = cp->det_no;
  ka.det_hw = Ho * Wo;
  ka.scale = scale; ka.bias = bias;
  ka.residual = (const __nv_bfloat16*)residual_bf16;
  ka.y = (__nv_bfloat16*)y_bf16;
  ka.y_f32 = y_f32;
  return launch_gemm(g, ka, (cudaStream_t)stream);
}

// ---- data gradient (K2): dx = conv_transpose(dy, W) as implicit GEMMs on the same kernel ------------------------------
// For each output-parity class (ph,pw) of dx (one class when stride==1):  dx[n, s*i+ph, s*j+pw, :] =
//   sum over the taps (kh,kw) with (ph+pad-kh) % s == 0, (pw+pad-kw) % s == 0 of  dy[n, i+dh, j+dw, :] * W[:, :, kh, kw]
//   with dh = (ph+pad-kh)/s, dw = (pw+pad-kw)/s.   B operand: etb_pack_weight_dgrad (same tap order).
static int dgrad_taps(int k, int s, int pad, int ph, int pw, signed char* kh_l, signed char* kw_l, signed char* dh, signed char* dw) {
  int n = 0;
  for (int kh = 0; kh < k; ++kh) {
    if ((ph + pad - kh) % s != 0) continue;
    for (int kw = 0; kw < k; ++kw) {
      if ((pw + pad - kw) % s != 0) continue;
      kh_l[n] = (signed char)kh; kw_l[n] = (signed char)kw;
      // floor division is exact here (remainder checked); C division of negatives truncates toward zero, also exact
      dh[n] = (signed char)((ph + pad - kh) / s); dw[n] = (signed char)((pw + pad - kw) / s);
      ++n;
    }
  }
  return n;
}

extern "C" int64_t etb_dgrad_weight_elems(int32_t Cout, int32_t Cin, int32_t k, int32_t stride) {
  (void)stride;
  const int64_t Coutp = (Cout + CONV_BLOCK_K - 1) / CONV_BLOCK_K * CONV_BLOCK_K;   // every tap padded to the 64-channel K block
  return (int64_t)Cin * k * k * Coutp;   // all parity classes together visit every tap exactly once
}

struct TapTable { signed char v[24]; };
__global__ void __launch_bounds__(256) pack_weight_dgrad_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ o, int Cout, int Coutp, int Cin, int k, int ntaps, TapTable tt) {
  const int64_t total = (int64_t)Cin * ntaps * Coutp;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int co = (int)(e % Coutp);
    const int t = (int)((e / Coutp) % ntaps);
    const int ci = (int)(e / ((int64_t)Coutp * ntaps));
    o[e] = __float2bfloat16(co < Cout ? w[(((int64_t)co * Cin + ci) * k + tt.v[t]) * k + tt.v[12 + t]] : 0.f);
  }
}

// w [Cout,Cin,k,k] fp32 -> for each parity class c (row-major ph,pw) a [Cin][ntaps_c*ceil64(Cout)] bf16 block (zero padded), blocks concatenated
extern "C" int etb_pack_weight_dgrad(const float* w_oihw, void* out_bf16, int32_t Cout, int32_t Cin, int32_t k, int32_t stride,
                                     int32_t pad, void* stream) {
  ETB_CHECK_ARG(w_oihw && out_bf16 && Cout > 0 && Cin > 0 && k >= 1 && k * k <= 12 && (stride == 1 || stride == 2));
  __nv_bfloat16* o = (__nv_bfloat16*)out_bf16;
  for (int ph = 0; ph < stride; ++ph)
    for (int pw = 0; pw < stride; ++pw) {
      TapTable tt;
      signed char dh[12], dw[12];
      const int nt = dgrad_taps(k, stride, pad, ph, pw, tt.v, tt.v + 12, dh, dw);
      if (nt == 0) continue;
      const int Coutp = (Cout + CONV_BLOCK_K - 1) / CONV_BLOCK_K * CONV_BLOCK_K;
      const int64_t total = (int64_t)Cin * nt * Coutp;
      int64_t blocks = (total + 255) / 256;
      if (blocks > etb_num_sms() * 16) blocks = etb_num_sms() * 16;
      etb_launch(pack_weight_dgrad_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, w_oihw, o, Cout, Coutp, Cin, k, nt, tt);
      ETB_CHECK_LAUNCH();
      o += total;
    }
  return ETB_OK;
}

// dy [N,Ho,Wo,*] bf16 (channels [dy_coffset.. +Cout) of stride dy_cstride) -> dx [N,H,W,*] bf16 at channel offset.
// cp describes the FORWARD conv (N,H,W,Cin,Cout,k,stride,pad); x_cstride/ y_* name the dy / dx buffers:
//   cp->x_cstride = channel stride of dy, cp->y_cstride/y_coffset = geometry of dx; cp->act is not read.
//   accumulate != 0 -> dx += result.
extern "C" int etb_conv_dgrad(const void* dy_bf16, const void* wd_bf16, void* dx_bf16, const EtbConvParams* cp, int32_t accumulate,
                              void* stream) {
  ETB_CHECK_ARG(dy_bf16 && wd_bf16 && dx_bf16 && cp);
  ETB_CHECK_ARG(cp->kh == cp->kw && cp->kh * cp->kw <= 12 && (cp->stride == 1 || cp->stride == 2));
  ETB_CHECK_ARG(cp->Cout % 8 == 0 && cp->y_cstride % 8 == 0 && cp->y_coffset % 8 == 0 && cp->y_cstride >= cp->y_coffset + cp->Cin);
  const int Coutp = (cp->Cout + CONV_BLOCK_K - 1) / CONV_BLOCK_K * CONV_BLOCK_K;   // row pitch of one tap in the packed operand
  const int k = cp->kh, s = cp->stride, pad = cp->pad;
  const int Ho = (cp->H + 2 * pad - k) / s + 1, Wo = (cp->W + 2 * pad - k) / s + 1;
  const __nv_bfloat16* wd = (const __nv_bfloat16*)wd_bf16;
  for (int ph = 0; ph < s; ++ph)
    for (int pw = 0; pw < s; ++pw) {
      ConvKArgs ka;
      memset(&ka, 0, sizeof(ka));
      signed char kh_l[12], kw_l[12];
      const int nt = dgrad_taps(k, s, pad, ph, pw, kh_l, kw_l, ka.tap_dh, ka.tap_dw);
      // etb_pack_weight_dgrad packs a block for every class with taps, also for classes with no pixels (H or W == 1):
      // step past it before skipping the class, or the next class would run on this one's weights
      const __nv_bfloat16* wcls = wd;
      wd += (size_t)cp->Cin * nt * Coutp;
      const int subH = (cp->H - ph + s - 1) / s, subW = (cp->W - pw + s - 1) / s;
      if (subH <= 0 || subW <= 0) continue;
      ETB_CHECK_ARG(nt > 0);   // k >= stride for every conv of the trunk, so every parity class is reached
      GemmGeom g;
      g.a_ptr = dy_bf16; g.aN = cp->N; g.aH = Ho; g.aW = Wo; g.aC = cp->Cout; g.a_cstride = cp->x_cstride;
      g.b_ptr = wcls; g.b_rows = cp->Cin;
      g.tile_H = subH; g.tile_W = subW;
      g.flat = (k == 1 && s == 1 && pad == 0);
      ka.ntaps = nt;
      ka.stride = 1;
      ka.out_os = s; ka.out_ph = ph; ka.out_pw = pw; ka.out_H = cp->H; ka.out_W = cp->W;
      ka.y_cstride = cp->y_cstride; ka.y_coffset = cp->y_coffset;
      ka.act = 0; ka.out_mode = 0; ka.accumulate = accumulate;
      ka.y = (__nv_bfloat16*)dx_bf16;
      int rc = launch_gemm(g, ka, (cudaStream_t)stream);
      if (rc != ETB_OK) return rc;
    }
  return ETB_OK;
}

// =====================================================================================================================
// weight gradient (K2):  dW[co][tap][ci] = sum over pixels  dy[n,oh,ow,co] * x[n, oh*s+kh-p, ow*s+kw-p, ci]
//
// GEMM with the PIXELS as the reduction (K) dimension: D[128 co, BN ci] += A[128 co, kpix]*B[BN ci, kpix]^T where both
// operands are MN-major (the channel index is the contiguous one in NHWC).  Each K block is one spatial tile of one
// image, fetched for both operands by 4-D TMA boxes {64 ch, TW, TH, 1} (x with the tap shift / element strides, zero
// padding = OOB fill) into 128B-swizzled smem = the canonical MN-major wgmma layout:
//   64-channel group = kpix rows x 128 B;  8-row K atoms 1024 B apart (SBO);  channel groups one region apart (LBO).
// Consumer warpgroup cw multiplies dy channel group cw (64 co) with the BN-wide x tile (wgmma with both operands
// transposed).  One CTA owns one (co tile, ci tile, tap) and a contiguous slice of the K blocks (split-K across
// gridDim.y); every CTA stores its partial tile into its own slice of the workspace (plain stores, no atomics, no
// memset) and a second kernel (wgrad_reduce_kernel / wgrad_reduce_taps_kernel) sums the slices in a fixed order into
// the parameter layout.
// =====================================================================================================================
struct WgradArgs {
  int ntaps;
  int kw, pad;              // tap t reads x at (oh*s + t/kw - pad, ow*s + t%kw - pad): no runtime-indexed table (local memory)
  int stride;
  int TW, TH, tiles_w, tiles_h, nimg;
  int kpix;                 // TW*TH, multiple of 16, <= WGRAD_KP = 128
  int co_tiles, ci_tiles;
  int Cout, Cin;
  float* dw;                // split-K partials: slice `blockIdx.y` of [splitk][Cout][ntaps][Cin] fp32
  long dw_split_stride;     // elements per slice
};

#define WGRAD_KP 128         // pixel rows per K block

template <int BN>
struct WgradSmem {
  static constexpr int GROUP_BYTES = WGRAD_KP * 128;      // one 64-channel group, up to WGRAD_KP K rows
  static constexpr int A_BYTES = 2 * GROUP_BYTES;         // 128 co
  static constexpr int B_BYTES = (BN / 64) * GROUP_BYTES;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = CONV_SMEM_STAGES_BYTES / STAGE_BYTES;   // 3 (BN = 128) or 4 (BN = 64)
  static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
  static constexpr int TOTAL = BAR_OFF + 256 + 1024;
};

// One K block of the weight gradient: KS straight-line K=16 steps (16 K rows = two 1024 B atoms each).  A runtime trip
// count, or a guard around each wgmma, makes ptxas insert a warpgroup.arrive before every wgmma.
template <int BN, int KS>
__device__ __forceinline__ void wgrad_issue(float* d, uint64_t adesc, uint64_t bdesc) {
  wgmma_fence();            // fence and commit inside the branch: outside it, ptxas adds its own warpgroup.arrive
#pragma unroll
  for (int k = 0; k < KS; ++k) wgmma_tile<BN, 1, 1>(d, adesc + (uint64_t)(k * (2048 >> 4)), bdesc + (uint64_t)(k * (2048 >> 4)), 1u);
  wgmma_commit();
}

template <int BN>
__global__ void __launch_bounds__(CONV_THREADS, 1)
wgrad_kernel(const __grid_constant__ CUtensorMap mapDy, const __grid_constant__ CUtensorMap mapX, const WgradArgs a) {
  using L = WgradSmem<BN>;
  constexpr int STAGES = L::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full = (uint64_t*)(smem + L::BAR_OFF);
  uint64_t* empty = full + STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;

  int t = blockIdx.x;
  const int tap = t % a.ntaps; t /= a.ntaps;
  const int ci_t = t % a.ci_tiles; t /= a.ci_tiles;
  const int co_t = t;
  const int co0 = co_t * 128, ci0 = ci_t * BN;
  const int total_kb = a.nimg * a.tiles_h * a.tiles_w;
  const int chunk = (total_kb + gridDim.y - 1) / gridDim.y;
  const int kb0 = blockIdx.y * chunk;
  const int kb1 = min(total_kb, kb0 + chunk);
  if (kb0 >= kb1) return;   // uniform for the CTA, before any barrier (the host plan never leaves a slice empty)
  const int kiters = kb1 - kb0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapDy);
    tma_prefetch_desc(&mapX);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  const uint32_t box_bytes = (uint32_t)a.kpix * 128u;   // bytes one TMA box writes (all rows, OOB rows zero-filled)

  if (wg == 0) {
    if (warp != 0) return;
    // warp-uniform loop, one elected lane issues; K-block coordinates, stage and phase advance incrementally
    int tw_i = kb0 % a.tiles_w, th_i = (kb0 / a.tiles_w) % a.tiles_h, img = kb0 / (a.tiles_w * a.tiles_h);
    const int xdh = tap / a.kw - a.pad, xdw = tap % a.kw - a.pad;
    int s = 0;
    uint32_t ph = 0;
    for (int it = 0; it < kiters; ++it) {
      const int w0 = tw_i * a.TW, h0 = th_i * a.TH;
      mbar_wait(&empty[s], ph ^ 1u);
      uint8_t* sa = smem + s * L::STAGE_BYTES;
      uint8_t* sb = sa + L::A_BYTES;
      if (elect_one()) {
        mbar_expect_tx(&full[s], box_bytes * (2u + BN / 64));
#pragma unroll
        for (int g = 0; g < 2; ++g) tma_load_4d(&mapDy, &full[s], sa + g * L::GROUP_BYTES, co0 + 64 * g, w0, h0, img);
#pragma unroll
        for (int g = 0; g < BN / 64; ++g)
          tma_load_4d(&mapX, &full[s], sb + g * L::GROUP_BYTES, ci0 + 64 * g, w0 * a.stride + xdw, h0 * a.stride + xdh, img);
      }
      __syncwarp();
      if (++tw_i == a.tiles_w) { tw_i = 0; if (++th_i == a.tiles_h) { th_i = 0; ++img; } }
      if (++s == STAGES) { s = 0; ph ^= 1u; }
    }
    return;
  }
  const int cw = wg - 1;
  const int ksteps = a.kpix / 16;
  float d[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) d[i] = 0.0f;
  int s = 0, prev = -1;
  uint32_t ph = 0;
  for (int it = 0; it < kiters; ++it) {
    mbar_wait(&full[s], ph);
    const uint32_t sa = smem_u32(smem + s * L::STAGE_BYTES);
    const uint64_t adesc = gmma_desc(sa + cw * L::GROUP_BYTES, L::GROUP_BYTES);
    const uint64_t bdesc = gmma_desc(sa + L::A_BYTES, L::GROUP_BYTES);
    switch (ksteps) {   // warpgroup-uniform
      case 1: wgrad_issue<BN, 1>(d, adesc, bdesc); break;
      case 2: wgrad_issue<BN, 2>(d, adesc, bdesc); break;
      case 3: wgrad_issue<BN, 3>(d, adesc, bdesc); break;
      case 4: wgrad_issue<BN, 4>(d, adesc, bdesc); break;
      case 5: wgrad_issue<BN, 5>(d, adesc, bdesc); break;
      case 6: wgrad_issue<BN, 6>(d, adesc, bdesc); break;
      case 7: wgrad_issue<BN, 7>(d, adesc, bdesc); break;
      default: wgrad_issue<BN, 8>(d, adesc, bdesc); break;
    }
    wgmma_wait<1>();
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
    prev = s;
    if (++s == STAGES) { s = 0; ph ^= 1u; }
  }
  wgmma_wait<0>();
  acc_fence<BN / 2>(d);
  // two-stage split-K: every CTA writes its partial tile into its own slice; wgrad_reduce_kernel sums the slices
  const int r0 = co0 + 64 * cw + 16 * (warp & 3) + (lane >> 2);
  float* slice = a.dw + (size_t)blockIdx.y * a.dw_split_stride;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int co = r0 + 8 * i;
    if (co >= a.Cout) continue;
    float* row = slice + ((size_t)co * a.ntaps + tap) * a.Cin;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int ci = ci0 + 8 * j + 2 * (lane & 3);
      if (ci < a.Cin) *reinterpret_cast<float2*>(row + ci) = make_float2(d[j * 4 + i * 2], d[j * 4 + i * 2 + 1]);   // Cin % 8 == 0
    }
  }
}

template <int BN>
static int launch_wgrad(const CUtensorMap& mDy, const CUtensorMap& mX, const WgradArgs& wa, dim3 grid, cudaStream_t st) {
  using L = WgradSmem<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    ETB_CHECK_CUDA(cudaFuncSetAttribute(wgrad_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
    attr_set = true;
  }
  etb_launch(wgrad_kernel<BN>, dim3(grid), dim3(CONV_THREADS), L::TOTAL, st, mDy, mX, wa);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}

static void pick_tile16(int Wo, int Ho, int maxrows, int* TW, int* TH) {
  // K tiles must be a whole number of K=16 wgmma steps: TW*TH % 16 == 0, <= maxrows; out-of-image rows are zero-filled by TMA
  double best = -1.0;
  for (int tw = 1; tw <= maxrows; ++tw)
    for (int th = 1; th * tw <= maxrows; ++th) {
      if ((tw * th) % 16) continue;
      if (tw > 2 * Wo || th > 2 * Ho) continue;
      const long tiles = (long)((Wo + tw - 1) / tw) * ((Ho + th - 1) / th);
      const double eff = (double)Wo * Ho / ((double)tiles * tw * th) * (tw * th >= maxrows / 2 ? 1.0 : 0.8);
      if (eff > best + 1e-9) { best = eff; *TW = tw; *TH = th; }
    }
  if (best >= 0.0) return;
  // maps of at most 3 pixels (1x1, 1x2, 1x3, 2x1, 3x1): no box stays within twice the map, so take the smallest box that
  // covers it in one tile.  Its extra rows are out of the image for both operands (zero-filled): wasted, never wrong.
  int best_rows = maxrows + 1;
  for (int tw = Wo; tw <= maxrows; ++tw)
    for (int th = Ho; th * tw <= maxrows; ++th)
      if ((tw * th) % 16 == 0 && tw * th < best_rows) { best_rows = tw * th; *TW = tw; *TH = th; }
}

// ---- second stage of the split-K: sum the slices, emit the parameter layout, optionally accumulate ----
// block = 32 lanes (each 4 consecutive ci of one (co, tap): coalesced float4 reads of every slice) x SG slice groups;
// group g sums slices g, g+SG, ... (4 independent loads in flight), the groups are combined through shared memory in a
// fixed order (deterministic).  SG grows with the split count so a split across every SM for a small layer is not one serial chain.
template <int SG>
__global__ void __launch_bounds__(32 * SG) wgrad_reduce_kernel(const float* __restrict__ ws, long slice, int splitk, float* __restrict__ out, int Cout,
                                                               int Cin, int kk, int flags) {
  __shared__ float4 red[SG][32];
  const long n4 = (long)Cout * kk * Cin / 4;
  const int lane = threadIdx.x, sg = threadIdx.y;
  for (long e4 = (long)blockIdx.x * 32 + lane; e4 - lane < n4; e4 += (long)gridDim.x * 32) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (e4 < n4) {
      const float4* p = reinterpret_cast<const float4*>(ws) + e4;
      const size_t st4 = (size_t)slice / 4;
      int sidx = sg;
      for (; sidx + 3 * SG < splitk; sidx += 4 * SG) {
        const float4 v0 = __ldg(p + (size_t)sidx * st4), v1 = __ldg(p + (size_t)(sidx + SG) * st4);
        const float4 v2 = __ldg(p + (size_t)(sidx + 2 * SG) * st4), v3 = __ldg(p + (size_t)(sidx + 3 * SG) * st4);
        acc.x += (v0.x + v1.x) + (v2.x + v3.x); acc.y += (v0.y + v1.y) + (v2.y + v3.y);
        acc.z += (v0.z + v1.z) + (v2.z + v3.z); acc.w += (v0.w + v1.w) + (v2.w + v3.w);
      }
      for (; sidx < splitk; sidx += SG) {
        const float4 v = __ldg(p + (size_t)sidx * st4);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    }
    if (SG > 1) {
      red[sg][lane] = acc;
      __syncthreads();
      if (sg == 0) {
#pragma unroll
        for (int g = 1; g < SG; ++g) {
          const float4 v = red[g][lane];
          acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
      }
    }
    if (sg == 0 && e4 < n4) {
      const long e = e4 * 4;
      const int ci = (int)(e % Cin);
      const long t2 = e / Cin;
      const int t = (int)(t2 % kk), co = (int)(t2 / kk);
      const float vals[4] = {acc.x, acc.y, acc.z, acc.w};
      if (kk == 1 && !(flags & 1) && (reinterpret_cast<uintptr_t>(out) & 15) == 0) {   // pointwise: the GEMM layout IS the parameter layout
        float4* o = reinterpret_cast<float4*>(out + e);
        if (flags & 2) { const float4 q = *o; acc.x += q.x; acc.y += q.y; acc.z += q.z; acc.w += q.w; }
        *o = acc;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          long dst;
          if (flags & 1) {                       // stem: [Cout][128 slots, k = (c*6+kh)*6+kw] -> [Cout,3,6,6] (same order)
            const int k = ci + j;
            if (k >= 108) continue;
            dst = (long)co * 108 + k;
          } else {
            dst = ((long)co * Cin + ci + j) * kk + t;
          }
          out[dst] = (flags & 2) ? out[dst] + vals[j] : vals[j];
        }
      }
    }
    if (SG > 1) __syncthreads();
  }
}

// kk > 1 (3x3 ...): the GEMM layout [co][tap][ci] has to become the parameter layout [co][ci][tap].  One block = one co
// and 64 consecutive ci: unit (tap, lane) sums its float4 over the slices (coalesced along ci), the [64][kk] patch is
// transposed through shared memory and written (or accumulated) as ONE contiguous run of 64*kk floats -- the naive
// scatter cost 8x sector amplification on both the read-modify-write and the store (60 us per 3x3 layer).
// When Cin % 64 != 0 (YOLOv5m: 96, YOLOv5x: 80, 160, ...) the last chunk of a co holds the remaining Cin % 64 channels.
__global__ void __launch_bounds__(256) wgrad_reduce_taps_kernel(const float* __restrict__ ws, long slice, int splitk, float* __restrict__ out, int Cin,
                                                                int kk, int flags) {
  __shared__ float sm[64 * 12];
  const int chunks = (Cin + 63) >> 6;
  const int co = blockIdx.x / chunks, ci0 = (blockIdx.x - co * chunks) * 64;
  const int CW = min(Cin - ci0, 64);             // channels of this block, a multiple of 8
  const int L4 = CW >> 2;                        // float4 lanes per tap
  const size_t st4 = (size_t)slice / 4;
  for (int u = threadIdx.x; u < kk * L4; u += 256) {
    const int t = u / L4, lane = u - t * L4;
    const float4* p = reinterpret_cast<const float4*>(ws + ((size_t)co * kk + t) * Cin + ci0) + lane;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int sidx = 0;
    for (; sidx + 3 < splitk; sidx += 4) {
      const float4 v0 = __ldg(p + (size_t)sidx * st4), v1 = __ldg(p + (size_t)(sidx + 1) * st4);
      const float4 v2 = __ldg(p + (size_t)(sidx + 2) * st4), v3 = __ldg(p + (size_t)(sidx + 3) * st4);
      acc.x += (v0.x + v1.x) + (v2.x + v3.x); acc.y += (v0.y + v1.y) + (v2.y + v3.y);
      acc.z += (v0.z + v1.z) + (v2.z + v3.z); acc.w += (v0.w + v1.w) + (v2.w + v3.w);
    }
    for (; sidx < splitk; ++sidx) {
      const float4 v = __ldg(p + (size_t)sidx * st4);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    sm[(4 * lane + 0) * kk + t] = acc.x;
    sm[(4 * lane + 1) * kk + t] = acc.y;
    sm[(4 * lane + 2) * kk + t] = acc.z;
    sm[(4 * lane + 3) * kk + t] = acc.w;
  }
  __syncthreads();
  float* o = out + ((size_t)co * Cin + ci0) * kk;
  for (int i = threadIdx.x; i < CW * kk; i += 256) o[i] = (flags & 2) ? o[i] + sm[i] : sm[i];
}

static int wgrad_plan(const EtbConvParams* cp, int* BN_, int* TW, int* TH, int* tiles_w, int* tiles_h, int* nimg, int* out_tiles, int* splitk) {
  const int Ho = (cp->H + 2 * cp->pad - cp->kh) / cp->stride + 1;
  const int Wo = (cp->W + 2 * cp->pad - cp->kw) / cp->stride + 1;
  ETB_CHECK_ARG(Ho > 0 && Wo > 0);
  const int BN = cp->Cin >= 128 ? 128 : 64;
  const bool flat = (cp->kh == 1 && cp->kw == 1 && cp->stride == 1 && cp->pad == 0);
  *TW = *TH = 0;
  if (flat) {
    const long npix = (long)cp->N * cp->H * cp->W;
    *TW = WGRAD_KP; *TH = 1; *tiles_w = (int)((npix + WGRAD_KP - 1) / WGRAD_KP); *tiles_h = 1; *nimg = 1;
  } else {
    pick_tile16(Wo, Ho, WGRAD_KP, TW, TH);
    // a K tile is a positive whole number of K=16 steps and fits the stage: anything else is a hole in the plan
    ETB_CHECK_ARG(*TW > 0 && *TH > 0 && (*TW * *TH) % 16 == 0 && *TW * *TH <= WGRAD_KP);
    *tiles_w = (Wo + *TW - 1) / *TW; *tiles_h = (Ho + *TH - 1) / *TH; *nimg = cp->N;
  }
  const int ntaps = cp->kh * cp->kw;
  *out_tiles = ((cp->Cout + 127) / 128) * ((cp->Cin + BN - 1) / BN) * ntaps;
  const int total_kb = *nimg * *tiles_h * *tiles_w;
  // split-K: minimise  rounds(out_tiles*sk) * (K blocks per CTA * t_kb + t_fixed)  -- whole waves of CTAs (one per SM) matter
  // more than raw parallelism.  t_kb ~ the MMA time of one 128-pixel block of a 128x128 tile, t_fixed ~ launch + pipeline
  // fill + the partial-tile stores of one CTA (both in us).
  const int sms = etb_num_sms();
  const double t_kb = 0.6 * (double)(*TW * *TH) / 128.0, t_fixed = 6.0;
  int sk = 1;
  double best = 1e30;
  const int sk_max = total_kb < 512 ? total_kb : 512;
  for (int c = 1; c <= sk_max; ++c) {
    const long ctas = (long)*out_tiles * c;
    if (ctas > 8L * sms) break;
    const long rounds = (ctas + sms - 1) / sms;
    const int per = (total_kb + c - 1) / c;
    if ((long)(c - 1) * per >= total_kb) continue;          // would leave an empty slice
    const double cost = (double)rounds * (per * t_kb + t_fixed) + 0.002 * c;   // tiny bias towards fewer partials to reduce
    if (cost < best) { best = cost; sk = c; }
  }
  *splitk = sk; *BN_ = BN;
  return ETB_OK;
}

extern "C" size_t etb_conv_wgrad_workspace_bytes(const EtbConvParams* cp) {
  if (!cp || cp->N <= 0 || cp->H <= 0 || cp->W <= 0 || cp->Cin <= 0 || cp->Cout <= 0 || cp->stride <= 0) return 0;
  int BN, TW, TH, tw, th, ni, ot, sk;
  if (wgrad_plan(cp, &BN, &TW, &TH, &tw, &th, &ni, &ot, &sk) != ETB_OK) return 0;
  return (size_t)sk * cp->Cout * cp->kh * cp->kw * cp->Cin * sizeof(float);
}

// x [N,H,W,*] bf16 (cp->x_cstride), dy [N,Ho,Wo,*] bf16 (channel stride cp->y_cstride) -> dw [Cout,Cin,kh,kw] fp32 (the
// nn.Parameter layout).  flags bit0: stem (cp describes the K=128 pointwise GEMM over the im2col buffer, dw is [Cout,3,6,6]);
// bit1: dw += result (dw may be the gradient-arena slice).  workspace: etb_conv_wgrad_workspace_bytes(cp).
extern "C" int etb_conv_wgrad(const void* x_bf16, const void* dy_bf16, float* dw_f32, const EtbConvParams* cp, int32_t flags, void* workspace,
                              size_t workspace_bytes, void* stream) {
  ETB_CHECK_ARG(x_bf16 && dy_bf16 && dw_f32 && cp && workspace);
  ETB_CHECK_ARG(cp->N > 0 && cp->H > 0 && cp->W > 0 && cp->Cin > 0 && cp->Cout > 0 && cp->Cin % 8 == 0);
  ETB_CHECK_ARG(cp->kh * cp->kw <= 12 && (cp->stride == 1 || cp->stride == 2));
  ETB_CHECK_ARG(cp->x_cstride % 8 == 0 && cp->y_cstride % 8 == 0 && (((uintptr_t)x_bf16) & 15) == 0 && (((uintptr_t)dy_bf16) & 15) == 0);
  ETB_CHECK_ARG((((uintptr_t)workspace) & 15) == 0);
  PFN_tmapEncodeTiled enc = get_encode();
  if (!enc) {
    etb_set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return ETB_ERR_CUDA;
  }
  const int Ho = (cp->H + 2 * cp->pad - cp->kh) / cp->stride + 1;
  const int Wo = (cp->W + 2 * cp->pad - cp->kw) / cp->stride + 1;
  WgradArgs wa;
  memset(&wa, 0, sizeof(wa));
  int BN, out_tiles, splitk;
  const int prc = wgrad_plan(cp, &BN, &wa.TW, &wa.TH, &wa.tiles_w, &wa.tiles_h, &wa.nimg, &out_tiles, &splitk);
  if (prc != ETB_OK) return prc;
  wa.kpix = wa.TW * wa.TH;
  wa.ntaps = cp->kh * cp->kw;
  wa.kw = cp->kw; wa.pad = cp->pad;
  wa.stride = cp->stride;
  wa.Cout = cp->Cout; wa.Cin = cp->Cin;
  const size_t dw_elems = (size_t)cp->Cout * wa.ntaps * cp->Cin;
  if (workspace_bytes < (size_t)splitk * dw_elems * sizeof(float)) {
    etb_set_error("etb_conv_wgrad: workspace too small (%zu < %zu)", workspace_bytes, (size_t)splitk * dw_elems * sizeof(float));
    return ETB_ERR_NOMEM;
  }
  wa.dw = (float*)workspace;
  wa.dw_split_stride = (long)dw_elems;
  const bool flat = (cp->kh == 1 && cp->kw == 1 && cp->stride == 1 && cp->pad == 0);
  cuuint64_t ddim[4], dstr[3], xdim[4], xstr[3];
  cuuint32_t dbox[4], xbox[4], one[4] = {1, 1, 1, 1}, xes[4];
  if (flat) {
    const long npix = (long)cp->N * cp->H * cp->W;
    ETB_CHECK_ARG(npix < (1l << 31));
    ddim[0] = cp->Cout; ddim[1] = (cuuint64_t)npix; ddim[2] = 1; ddim[3] = 1;
    dstr[0] = (cuuint64_t)cp->y_cstride * 2; dstr[1] = dstr[0] * (cuuint64_t)npix; dstr[2] = dstr[1];
    xdim[0] = cp->Cin; xdim[1] = (cuuint64_t)npix; xdim[2] = 1; xdim[3] = 1;
    xstr[0] = (cuuint64_t)cp->x_cstride * 2; xstr[1] = xstr[0] * (cuuint64_t)npix; xstr[2] = xstr[1];
    dbox[0] = 64; dbox[1] = WGRAD_KP; dbox[2] = 1; dbox[3] = 1;
    xbox[0] = 64; xbox[1] = WGRAD_KP; xbox[2] = 1; xbox[3] = 1;
    xes[0] = xes[1] = xes[2] = xes[3] = 1;
  } else {
    ddim[0] = cp->Cout; ddim[1] = Wo; ddim[2] = Ho; ddim[3] = cp->N;
    dstr[0] = (cuuint64_t)cp->y_cstride * 2; dstr[1] = dstr[0] * Wo; dstr[2] = dstr[1] * Ho;
    xdim[0] = cp->Cin; xdim[1] = cp->W; xdim[2] = cp->H; xdim[3] = cp->N;
    xstr[0] = (cuuint64_t)cp->x_cstride * 2; xstr[1] = xstr[0] * cp->W; xstr[2] = xstr[1] * cp->H;
    dbox[0] = 64; dbox[1] = wa.TW; dbox[2] = wa.TH; dbox[3] = 1;
    xbox[0] = 64; xbox[1] = wa.TW * cp->stride; xbox[2] = wa.TH * cp->stride; xbox[3] = 1;
    xes[0] = 1; xes[1] = cp->stride; xes[2] = cp->stride; xes[3] = 1;
    ETB_CHECK_ARG(xbox[1] <= 256 && xbox[2] <= 256);
  }
  CUtensorMap mDy, mX;
  CUresult r = enc(&mDy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(dy_bf16), ddim, dstr, dbox, one, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { etb_set_error("cuTensorMapEncodeTiled(dy) failed: %d", (int)r); return ETB_ERR_CUDA; }
  r = enc(&mX, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(x_bf16), xdim, xstr, xbox, xes, CU_TENSOR_MAP_INTERLEAVE_NONE,
          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { etb_set_error("cuTensorMapEncodeTiled(x) failed: %d", (int)r); return ETB_ERR_CUDA; }
  wa.co_tiles = (cp->Cout + 127) / 128;
  wa.ci_tiles = (cp->Cin + BN - 1) / BN;
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid((unsigned)out_tiles, (unsigned)splitk);
  const int rc = BN == 128 ? launch_wgrad<128>(mDy, mX, wa, grid, st) : launch_wgrad<64>(mDy, mX, wa, grid, st);
  if (rc != ETB_OK) return rc;
  // rows co >= Cout of the last tile are never written: the reduce only reads [Cout] rows
  const long n4 = (long)dw_elems / 4;
  long blocks = (n4 + 31) / 32;
  const long cap = (long)etb_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  if (wa.ntaps > 1 && !(flags & 1))
    etb_launch(wgrad_reduce_taps_kernel, dim3((unsigned)(cp->Cout * ((cp->Cin + 63) >> 6))), dim3(256), 0, st, (const float*)workspace, (long)dw_elems, splitk, dw_f32, cp->Cin, wa.ntaps,
                                                                                  flags);
  else if (splitk >= 32)
    etb_launch(wgrad_reduce_kernel<16>, dim3((unsigned)blocks), dim3(dim3(32, 16)), 0, st, (const float*)workspace, (long)dw_elems, splitk, dw_f32, cp->Cout, cp->Cin, wa.ntaps, flags);
  else if (splitk >= 6)
    etb_launch(wgrad_reduce_kernel<4>, dim3((unsigned)blocks), dim3(dim3(32, 4)), 0, st, (const float*)workspace, (long)dw_elems, splitk, dw_f32, cp->Cout, cp->Cin, wa.ntaps, flags);
  else
    etb_launch(wgrad_reduce_kernel<1>, dim3((unsigned)blocks), dim3(dim3(32, 1)), 0, st, (const float*)workspace, (long)dw_elems, splitk, dw_f32, cp->Cout, cp->Cin, wa.ntaps, flags);
  ETB_CHECK_LAUNCH();
  return ETB_OK;
}
