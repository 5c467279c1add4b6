// Kernels of DfM's LIGAResNet-34 image backbone (mmdet3d/models/backbones/liga_resnet.py with the
// shipped KITTI `backbone` block: strides (1, 2, 1, 1), dilations (1, 1, 2, 4), channel factors
// (1, 2, 2, 2), no max-pool, no ReLU after the residual add).  Activations are channels-last
// [N][h][w][C] over all images of a call.
//
// resnet_conv_tc_kernel<C>: the 3x3 stride-1 convs (C -> C, C = 64 / 128, dilation 1 / 2 / 4,
// padding = dilation) as a 2-D implicit GEMM on wgmma:
//   * M = a tile of 8 (w) x 16 (h) output pixels, N = all C output channels in one MMA, K = 16
//     input channels x 9 taps per pipeline stage.  Two consumer warpgroups own 64 pixels each
//     (C / 2 fp32 accumulators per thread).
//   * Operands are the project's 3-term bf16 split (x_hi w_hi + x_lo w_hi + x_hi w_lo, fp32
//     accumulation) in the K-major no-swizzle layout of conv_tc_neck.cuh: a stage holds the input
//     brick of the tile with a halo of d pixels on every side, (8 + 2d) x (16 + 2d) rows of
//     16 bytes per 8-channel chunk, and a tap (ky, kx) is the same brick addressed d * ky brick
//     rows and d * kx pixels further on -- dilation costs nothing but a wider halo (at most
//     384 rows, d = 4), so no polyphase split is needed.
//   * Weights cannot stay resident (a 128 -> 128 hi + lo image is 590 KB): each stage carries
//     its 16-input-channel slice of all 9 taps (73.7 KB hi + lo for C = 128), copied with
//     cp.async next to the loader's transpose of the brick.  Every tile re-reads the whole
//     image from L2 once.
//   * Input goes through a dfm::Term (identity, or the consumer-side BatchNorm + ReLU of the
//     previous conv's raw output).
//   * Epilogue: the raw conv output is always written; with `bscale` the block output
//     bn2(raw) + identity (the identity a dfm::Term: the previous block's output, the stem's
//     bn1 + ReLU, or the downsample's BatchNorm) is written as well, in fp32.
//
// resnet_conv_simt_kernel<CIN, COUT, K>: every layer on fp32 CUDA cores (conv_impl = simt, and
// the stride-2 3x3 conv and 1x1 downsample of layer2.0 under every impl), with runtime stride,
// padding and dilation and the same epilogue.
//
// resnet_stem_kernel: conv1 7x7 stride 2 pad 3, 3 -> 64, reading the NCHW image directly.
#pragma once
#include "conv_tc.cuh"

namespace dfm {

constexpr int RN_BX = 8, RN_BY = 16;        // tile: 8 pixels along w (core-matrix rows) x 16 along h
constexpr int RN_KC = 16;                   // input channels per stage
constexpr int RN_MAX_DIL = 4;
constexpr int RN_ROWS = (RN_BX + 2 * RN_MAX_DIL) * (RN_BY + 2 * RN_MAX_DIL);  // 384 brick rows
constexpr uint32_t RN_A_LBO = RN_ROWS * 16;           // 8-channel chunk pitch (bytes)
constexpr uint32_t RN_A_HL = 2 * RN_A_LBO;            // hi -> lo
constexpr uint32_t RN_A_BYTES = 2 * RN_A_HL;          // 24 KB
constexpr int RN_MMA_THREADS = 256;
constexpr int RN_LOAD_THREADS = 256;                  // 2 groups x 4 warps, alternate stages
constexpr int RN_THREADS = RN_MMA_THREADS + RN_LOAD_THREADS;  // 16 warps: 128 registers/thread

template <int C>
struct RnCfg {
  static constexpr uint32_t B_HL = 9 * 2 * C * 16;    // one stage's weight slice, hi (or lo)
  static constexpr uint32_t STAGE_BYTES = RN_A_BYTES + 2 * B_HL;
  static constexpr int NSTAGE = C == 128 ? 2 : 3;
  static constexpr size_t SMEM = (size_t)NSTAGE * STAGE_BYTES + 2 * NSTAGE * 8;
  static constexpr size_t IMG_BYTES = (size_t)(C / RN_KC) * 2 * B_HL;  // whole weight image
};

struct ResnetConvParams {
  Term in;                 // input [N][Hi][Wi][Cin], fused transform
  const uint8_t* wimg;     // tc: [Cin / 16][hi | lo][9 taps][2 chunks][Cout][8] bf16
  const float* wt;         // simt: [K * K][Cin][Cout] fp32
  float* raw;              // raw conv output [N][Ho][Wo][Cout]
  const float* bscale;     // optional block epilogue: out = raw * bscale + bshift + identity
  const float* bshift;
  Term id;                 // identity [N][Ho][Wo][Cout]
  float* out;
  int N, Hi, Wi, Ho, Wo, Cin, Cout;
  int stride, pad, dil;
  int tiles_x, tiles_y, ntiles;
  int* err;
};

__device__ __forceinline__ float rn_term(const Term& t, long long idx, int c) {
  float v = __ldg(t.x + idx);
  if (t.scale) v = fmaf(v, __ldg(t.scale + c), __ldg(t.shift + c));
  return t.relu ? fmaxf(v, 0.f) : v;
}

// block epilogue of one output element (pixel-major index pix, channel c)
__device__ __forceinline__ float rn_block(const ResnetConvParams& p, long long pix, int c, float v) {
  return fmaf(v, __ldg(p.bscale + c), __ldg(p.bshift + c)) + rn_term(p.id, pix * p.Cout + c, c);
}

__device__ __forceinline__ void cp_async16_rn(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}

template <int C>
__global__ void __launch_bounds__(RN_THREADS, 1)
resnet_conv_tc_kernel(const __grid_constant__ ResnetConvParams p) {
  using Cfg = RnCfg<C>;
  constexpr int NSTAGE = Cfg::NSTAGE;
  constexpr uint32_t STAGE = Cfg::STAGE_BYTES, B_HL = Cfg::B_HL;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + NSTAGE * STAGE);
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const uint32_t bar0 = smem_u32(bars);
  auto full = [&](int s) { return bar0 + 8u * s; };
  auto empty = [&](int s) { return bar0 + 8u * (NSTAGE + s); };
  if (tid == 0) {
    for (int s = 0; s < NSTAGE; ++s) {
      mbar_init(full(s), 4);    // one arrival per loader warp of the group
      mbar_init(empty(s), 8);   // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int nk = p.Cin / RN_KC, d = p.dil;
  const int PX = RN_BX + 2 * d, PY = RN_BY + 2 * d, npos = PX * PY;
  const int tpi = p.tiles_x * p.tiles_y;

  if (warp >= RN_MMA_THREADS / 32) {
    // ================================ loaders ================================
    const int lw = warp - RN_MMA_THREADS / 32, grp = lw >> 2, lt = (lw & 3) * 32 + lane;
    uint32_t ctr = 0;
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
      const int img = tile / tpi, r = tile - img * tpi;
      const int x0 = (r % p.tiles_x) * RN_BX - d, y0 = (r / p.tiles_x) * RN_BY - d;
      const long long ibase = (long long)img * p.Hi * p.Wi;
      for (int kc = 0; kc < nk; ++kc, ++ctr) {
        if ((int)(ctr & 1) != grp) continue;
        const int s = ctr % NSTAGE;
        mbar_wait(empty(s), ((ctr / NSTAGE) & 1) ^ 1, p.err);
        uint8_t* st = smem + s * STAGE;
        // this stage's weight slice (hi and lo images are adjacent in global memory)
        const uint32_t b_dst = smem_u32(st + RN_A_BYTES);
        const uint8_t* b_src = p.wimg + (size_t)kc * 2 * B_HL;
#pragma unroll 1
        for (uint32_t i = lt; i < 2 * B_HL / 16; i += 128) cp_async16_rn(b_dst + 16 * i, b_src + 16 * i);
        // the brick: item = (pixel, 8-channel chunk)
        constexpr int LB = 3;
#pragma unroll 1
        for (int i0 = lt; i0 < 2 * npos; i0 += LB * 128) {
          float4 raw[LB][2];
          int soff[LB], cch[LB];
          bool live[LB], inb[LB];
#pragma unroll
          for (int b = 0; b < LB; ++b) {
            const int i = i0 + b * 128;
            live[b] = i < 2 * npos;
            const int pos = i >> 1, ch = i & 1;
            const int bx = pos % PX, by = pos / PX;
            const int x = x0 + bx, y = y0 + by;
            inb[b] = live[b] && x >= 0 && x < p.Wi && y >= 0 && y < p.Hi;
            soff[b] = ch * RN_A_LBO + pos * 16;
            cch[b] = kc * RN_KC + ch * 8;
            if (inb[b]) {
              const float4* src = reinterpret_cast<const float4*>(
                  p.in.x + (ibase + (long long)y * p.Wi + x) * p.Cin + cch[b]);
              raw[b][0] = __ldg(src);
              raw[b][1] = __ldg(src + 1);
            }
          }
#pragma unroll
          for (int b = 0; b < LB; ++b) {
            if (!live[b]) continue;
            float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (inb[b]) {
              const float u[8] = {raw[b][0].x, raw[b][0].y, raw[b][0].z, raw[b][0].w,
                                  raw[b][1].x, raw[b][1].y, raw[b][1].z, raw[b][1].w};
#pragma unroll
              for (int e = 0; e < 8; ++e) {
                float a = u[e];
                if (p.in.scale) a = fmaf(a, __ldg(p.in.scale + cch[b] + e), __ldg(p.in.shift + cch[b] + e));
                v[e] = p.in.relu ? fmaxf(a, 0.f) : a;
              }
            }
            split_store(v, st + soff[b], st + RN_A_HL + soff[b]);
          }
        }
        asm volatile("cp.async.wait_all;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) mbar_arrive(full(s));
      }
    }
  } else {
    // ===================== consumer warpgroups: MMA, then the epilogue =====================
    const int wg = warp >> 2, wq = warp & 3;
    constexpr uint32_t B_LBO16 = C;                 // 16-byte rows between the two K chunks
    constexpr uint32_t TAP16 = 2 * C;               // one tap of the slice
    const uint32_t a_desc_hi = (uint32_t)PX, b_desc_hi = 128u >> 4;   // SBO (16-byte units)
    float acc[C / 2];
    uint32_t ctr = 0;
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
#pragma unroll
      for (int i = 0; i < C / 2; ++i) acc[i] = 0.f;
      for (int kc = 0; kc < nk; ++kc, ++ctr) {
        const int s = ctr % NSTAGE;
        mbar_wait(full(s), (ctr / NSTAGE) & 1, p.err);
        const uint32_t st16 = (smem_u32(smem + s * STAGE) >> 4) & 0x3FFF;
        // warpgroup wg reads brick rows 8 wg .. 8 wg + 7 (+ the tap's offset)
        const uint32_t a_lo = (st16 + (uint32_t)(8 * wg * PX)) | ((RN_A_LBO >> 4) << 16);
        const uint32_t b_lo = (st16 + (RN_A_BYTES >> 4)) | (B_LBO16 << 16);
        wgmma_fence();
#pragma unroll 1
        for (int ky = 0; ky < 3; ++ky) {
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            const uint32_t ao = (uint32_t)(ky * d * PX + kx * d);
            const uint32_t bo = (uint32_t)(ky * 3 + kx) * TAP16;
            const uint64_t ah = pack64(a_lo + ao, a_desc_hi);
            const uint64_t al = pack64(a_lo + ao + (RN_A_HL >> 4), a_desc_hi);
            const uint64_t bh = pack64(b_lo + bo, b_desc_hi);
            const uint64_t bl = pack64(b_lo + bo + (B_HL >> 4), b_desc_hi);
            wgmma_bf16<C>(acc, ah, bh);
            wgmma_bf16<C>(acc, al, bh);
            wgmma_bf16<C>(acc, ah, bl);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(empty(s));
      }
      // registers (i, i + 1): pixel row 8 wg + 2 wq + ((i / 2) & 1) of the tile, column lane / 4;
      //                       channels 8 (i / 4) + 2 (lane % 4) + {0, 1}
      const int img = tile / tpi, r = tile - img * tpi;
      const int x = (r % p.tiles_x) * RN_BX + (lane >> 2);
      const int yb = (r / p.tiles_x) * RN_BY + 8 * wg + 2 * wq;
      const int n0 = 2 * (lane & 3);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int y = yb + rr;
        if (x >= p.Wo || y >= p.Ho) continue;
        const long long o = (((long long)img * p.Ho + y) * p.Wo + x) * C + n0;
        float2* raw = reinterpret_cast<float2*>(p.raw + o);
#pragma unroll
        for (int j = 0; j < C / 8; ++j)
          raw[4 * j] = make_float2(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1]);
        if (!p.bscale) continue;
        float2* out = reinterpret_cast<float2*>(p.out + o);
        const float2* idp = reinterpret_cast<const float2*>(p.id.x + o);
#pragma unroll
        for (int j = 0; j < C / 8; ++j) {
          const int n = 8 * j + n0;
          const float2 bs = __ldg(reinterpret_cast<const float2*>(p.bscale + n));
          const float2 bh = __ldg(reinterpret_cast<const float2*>(p.bshift + n));
          float2 id = __ldg(idp + 4 * j);
          if (p.id.scale) {
            const float2 is = __ldg(reinterpret_cast<const float2*>(p.id.scale + n));
            const float2 ih = __ldg(reinterpret_cast<const float2*>(p.id.shift + n));
            id = make_float2(fmaf(id.x, is.x, ih.x), fmaf(id.y, is.y, ih.y));
          }
          if (p.id.relu) id = make_float2(fmaxf(id.x, 0.f), fmaxf(id.y, 0.f));
          out[4 * j] = make_float2(fmaf(acc[4 * j + 2 * rr], bs.x, bh.x) + id.x,
                                   fmaf(acc[4 * j + 2 * rr + 1], bs.y, bh.y) + id.y);
        }
      }
    }
  }
}

// One warp owns VOX consecutive output pixels (image-major), lane = output channel (mod 32);
// weights [K * K][CIN][COUT], fp32 FMAs in (tap, input channel) order.
template <int CIN, int COUT, int K>
__global__ void __launch_bounds__(256, 1) resnet_conv_simt_kernel(const ResnetConvParams p) {
  constexpr int VOX = 8;
  constexpr int CI = (CIN + 31) / 32, CO = (COUT + 31) / 32;
  const int lane = threadIdx.x & 31;
  const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nout = (long long)p.N * p.Ho * p.Wo;
  const long long v0 = warp_id * VOX;
  if (v0 >= nout) return;
  int im[VOX], yo[VOX], xo[VOX];
  bool vv[VOX];
#pragma unroll
  for (int v = 0; v < VOX; ++v) {
    const long long idx = v0 + v;
    vv[v] = idx < nout;
    const long long i2 = vv[v] ? idx : 0;
    xo[v] = (int)(i2 % p.Wo);
    yo[v] = (int)((i2 / p.Wo) % p.Ho);
    im[v] = (int)(i2 / ((long long)p.Wo * p.Ho));
  }
  float acc[CO][VOX];
#pragma unroll
  for (int j = 0; j < CO; ++j)
#pragma unroll
    for (int v = 0; v < VOX; ++v) acc[j][v] = 0.f;
  for (int tap = 0; tap < K * K; ++tap) {
    const int ky = tap / K, kx = tap % K;
    float xin[CI][VOX];
    bool any = false;
#pragma unroll
    for (int v = 0; v < VOX; ++v) {
      const int yi = yo[v] * p.stride - p.pad + ky * p.dil;
      const int xi = xo[v] * p.stride - p.pad + kx * p.dil;
      const bool ok = vv[v] && yi >= 0 && yi < p.Hi && xi >= 0 && xi < p.Wi;
      any |= ok;
      const long long base = (((long long)im[v] * p.Hi + yi) * p.Wi + xi) * CIN;
#pragma unroll
      for (int j = 0; j < CI; ++j) {
        const int c = lane + 32 * j;
        xin[j][v] = (ok && c < CIN) ? rn_term(p.in, base + c, c) : 0.f;
      }
    }
    if (!any) continue;  // warp-uniform
    const float* wt = p.wt + (long long)tap * CIN * COUT;
#pragma unroll
    for (int j = 0; j < CI; ++j) {
#pragma unroll 8
      for (int l = 0; l < 32; ++l) {
        const int ci = j * 32 + l;
        if (ci >= CIN) break;
        float wv[CO];
#pragma unroll
        for (int jo = 0; jo < CO; ++jo) wv[jo] = __ldg(wt + (long long)ci * COUT + lane + 32 * jo);
#pragma unroll
        for (int v = 0; v < VOX; ++v) {
          const float xv = __shfl_sync(0xffffffffu, xin[j][v], l);
#pragma unroll
          for (int jo = 0; jo < CO; ++jo) acc[jo][v] = fmaf(xv, wv[jo], acc[jo][v]);
        }
      }
    }
  }
#pragma unroll
  for (int v = 0; v < VOX; ++v) {
    if (!vv[v]) continue;
    const long long pix = v0 + v;
#pragma unroll
    for (int jo = 0; jo < CO; ++jo) {
      const int co = lane + 32 * jo;
      p.raw[pix * COUT + co] = acc[jo][v];
      if (p.bscale) p.out[pix * COUT + co] = rn_block(p, pix, co, acc[jo][v]);
    }
  }
}

// Stem: conv1 7x7 / 2 / 3, 3 -> 64 from the NCHW image [N][3][H][W]; raw output channels-last.
// 256 threads = 64 output pixels x 4 groups of 16 channels; the 147 x 64 weights sit in shared
// memory ([tap][ci][64]); fp32 FMAs in (ci, ky, kx) order.
constexpr int RN_STEM_PIX = 64;
__global__ void __launch_bounds__(256)
resnet_stem_kernel(const float* __restrict__ img, const float* __restrict__ w, float* __restrict__ out,
                   int N, int H, int W, int Ho, int Wo) {
  __shared__ float ws[147 * 64];
  for (int i = threadIdx.x; i < 147 * 64; i += 256) ws[i] = __ldg(w + i);
  __syncthreads();
  const int cg = threadIdx.x >> 6;
  const long long pix = (long long)blockIdx.x * RN_STEM_PIX + (threadIdx.x & 63);
  if (pix >= (long long)N * Ho * Wo) return;
  const int xo = (int)(pix % Wo), yo = (int)((pix / Wo) % Ho), n = (int)(pix / ((long long)Wo * Ho));
  float acc[16];
#pragma unroll
  for (int o = 0; o < 16; ++o) acc[o] = 0.f;
  for (int ci = 0; ci < 3; ++ci) {
    const float* src = img + ((long long)n * 3 + ci) * H * W;
    for (int ky = 0; ky < 7; ++ky) {
      const int yi = 2 * yo - 3 + ky;
      if (yi < 0 || yi >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        const int xi = 2 * xo - 3 + kx;
        if (xi < 0 || xi >= W) continue;
        const float v = __ldg(src + (long long)yi * W + xi);
        const float* wr = ws + ((ci * 7 + ky) * 7 + kx) * 64 + 16 * cg;
#pragma unroll
        for (int o = 0; o < 16; ++o) acc[o] = fmaf(v, wr[o], acc[o]);
      }
    }
  }
  float4* dst = reinterpret_cast<float4*>(out + pix * 64 + 16 * cg);
#pragma unroll
  for (int o = 0; o < 4; ++o)
    dst[o] = make_float4(acc[4 * o], acc[4 * o + 1], acc[4 * o + 2], acc[4 * o + 3]);
}

}  // namespace dfm
