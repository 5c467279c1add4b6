// 32 -> 1 channel 3x3x3 "logits" conv (build_depth_pred_module's last layer,
// dfm_backbone.py:128) on the tensor cores, third formulation.
//
// With one output channel an implicit-GEMM conv has N = 1.  Here the GEMM is turned around: per
// INPUT position the 27 per-tap dot products q_t = <x, w_t> are ONE small GEMM
//     Q[128 positions x 32 (27 taps)] = X[128 x 32 channels] * W^T[32 channels x 32]
// -- 12 wgmma (2 halves of 64 positions x 2 K steps x 3 bf16 hi/lo terms) per 128 positions
// and plane instead of 864 FMAs per position -- and the 3x3x3 stencil becomes a gather of Q over
// the 27 shifted neighbours, done from shared memory with three running sums per output pixel
// along z.
//   * CTA tile: 16 (x) x 8 (y) input positions = 128 accumulator rows, 14 x 6 outputs;
//     persistent over (tile, z chunk) items, one pipeline stage per input plane.
//   * warps 0-3: one consumer warpgroup (wgmma into registers, Q to shared memory, gather),
//     4-11 loaders (the same fused GroupNorm + ReLU + bf16 split loader as conv_tc.cuh); two
//     CTAs per SM.
#pragma once
#include "conv_tc.cuh"

namespace dfm {

constexpr int LT_PX = 16, LT_PY = 8;                 // input positions of a tile
constexpr int LT_OX = LT_PX - 2, LT_OY = LT_PY - 2;  // outputs of a tile
constexpr int LT_ZC = 16;                            // output planes per item
constexpr int LT_NSTAGE = 4;                        // operand stages
constexpr uint32_t LT_A_LBO = 128 * 16;              // chunk stride (128 rows x 16 B)
constexpr uint32_t LT_A_HL = 4 * LT_A_LBO;           // hi -> lo
constexpr uint32_t LT_STAGE_BYTES = 2 * LT_A_HL;     // 16 KB
constexpr uint32_t LT_B_LBO = 32 * 16;               // weight image: [chunk][32 tap rows][16 B]
constexpr uint32_t LT_B_HL = 4 * LT_B_LBO;
constexpr uint32_t LT_W_BYTES = 2 * LT_B_HL;         // 4 KB
constexpr int LT_THREADS = 128 + 256;              // consumer warpgroup | loaders

struct LogitsTcParams {
  const uint8_t* wimg;   // device, LT_W_BYTES: hi image then lo image
  float* out;            // [D][H][W]
  int D, H, W;
  int tiles_x, tiles_y, zchunks, nitems;
  int* err;
};

// host: [27][32] fp32 -> bf16 hi/lo images, rows 27..31 zero
inline void logits_tc_pack(const float* w, std::vector<uint16_t>& img) {
  img.assign(LT_W_BYTES / 2, 0);
  for (int t = 0; t < 27; ++t)
    for (int c = 0; c < 32; ++c) {
      const float v = w[t * 32 + c];
      const uint16_t hi = bf16_rn_bits(v);
      const uint16_t lo = bf16_rn_bits(v - bf16_bits_to_float(hi));
      const size_t off = ((size_t)(c / 8) * 32 + t) * 8 + (c % 8);
      img[off] = hi;
      img[off + LT_B_HL / 2] = lo;
    }
}

__global__ void __launch_bounds__(LT_THREADS, 2)
logits_tc_kernel(const __grid_constant__ LogitsTcParams p, const SrcLoader8<1> ld) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* w_s = smem;                                     // 4 KB
  uint8_t* a_s = smem + LT_W_BYTES;                        // operand stages, 16 KB each
  float* q_s = reinterpret_cast<float*>(a_s + LT_NSTAGE * LT_STAGE_BYTES);  // [2][27][128]
  uint64_t* bars = reinterpret_cast<uint64_t*>(q_s + 2 * 27 * 128);

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const uint32_t bar0 = smem_u32(bars);
  auto full_a = [&](int s) { return bar0 + 8u * s; };
  auto empty_a = [&](int s) { return bar0 + 8u * (LT_NSTAGE + s); };

  if (tid == 0) {
    for (int s = 0; s < LT_NSTAGE; ++s) {
      mbar_init(full_a(s), 4);    // one arrival per loader warp of the group
      mbar_init(empty_a(s), 4);   // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // the 4 KB weight image (generic-proxy copy, fenced for the tensor core)
  for (int i = tid; i < (int)(LT_W_BYTES / 16); i += LT_THREADS)
    reinterpret_cast<uint4*>(w_s)[i] = __ldg(reinterpret_cast<const uint4*>(p.wimg) + i);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const long long plane = (long long)p.H * p.W;

  auto item_geom = [&](int item, int& x0, int& y0, int& z_lo, int& z_hi) {
    int b = item;
    const int tx = b % p.tiles_x;
    b /= p.tiles_x;
    const int ty = b % p.tiles_y;
    const int zc = b / p.tiles_y;
    x0 = tx * LT_OX;
    y0 = ty * LT_OY;
    z_lo = zc * LT_ZC;
    z_hi = min(p.D, z_lo + LT_ZC);
  };

  if (warp >= 4) {
    // ============================ loaders ============================
    const int lgrp = (warp - 4) & 1;
    const int lt = ((warp - 4) >> 1) * 32 + lane;   // 0..127 inside the group
    const int chunk = lt & 3;
    uint32_t stage_ctr = 0;
    for (int item = blockIdx.x; item < p.nitems; item += gridDim.x) {
      int x0, y0, z_lo, z_hi;
      item_geom(item, x0, y0, z_lo, z_hi);
      int gx[4], gy[4];
      bool inb[4];
      uint32_t soff[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int pos = (lt >> 2) + k * 32;          // 128 positions x 4 chunks, 4 items/thread
        gx[k] = x0 - 1 + (pos % LT_PX);
        gy[k] = y0 - 1 + (pos / LT_PX);
        inb[k] = gx[k] >= 0 && gx[k] < p.W && gy[k] >= 0 && gy[k] < p.H;
        soff[k] = (uint32_t)(chunk * 128 + pos) * 16;
      }
      for (int zi = max(z_lo - 1, 0); zi <= min(z_hi, p.D - 1); ++zi, ++stage_ctr) {
        if ((int)(stage_ctr & 1) != lgrp) continue;
        const int s = stage_ctr % LT_NSTAGE;
        mbar_wait(empty_a(s), ((stage_ctr / LT_NSTAGE) & 1) ^ 1, p.err);
        uint8_t* st = a_s + s * LT_STAGE_BYTES;
        SrcLoader8<1>::Raw raw[4];
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (inb[k]) ld.issue(zi, gy[k], gx[k], chunk * 8, raw[k]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float v[8];
          if (inb[k]) {
            ld.finish(raw[k], chunk * 8, v);
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = 0.f;
          }
          split_store(v, st + soff[k], st + LT_A_HL + soff[k]);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) mbar_arrive(full_a(s));
      }
    }
  } else {
    // ============ consumer warpgroup (warps 0-3): MMA issue, then the stencil gather ============
    // Two m64n32 wgmma chains per plane (positions 0-63 and 64-127); thread m == position in
    // the gather.
    const uint32_t w_base = smem_u32(w_s), a_base = smem_u32(a_s);
    const uint32_t desc_hi = 128u >> 4;   // SBO = 128 B (dense 8-row groups)
    const int m = tid;                    // position of the gather
    const int bx = m % LT_PX, by = m / LT_PX;
    const bool inner = bx >= 1 && bx <= LT_OX && by >= 1 && by <= LT_OY;
    float acc[2][16];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[h][i] = 0.f;
    uint32_t stage_ctr = 0;
    for (int item = blockIdx.x; item < p.nitems; item += gridDim.x) {
      int x0, y0, z_lo, z_hi;
      item_geom(item, x0, y0, z_lo, z_hi);
      const int ox = x0 + bx - 1, oy = y0 + by - 1;
      const bool olive = inner && ox < p.W && oy < p.H;
      float accA = 0.f, accB = 0.f;                  // output planes zi-1 and zi
      for (int zi = max(z_lo - 1, 0); zi <= min(z_hi, p.D - 1); ++zi, ++stage_ctr) {
        const int s = stage_ctr % LT_NSTAGE;
        float* qb = q_s + (stage_ctr & 1) * (27 * 128);
        mbar_wait(full_a(s), (stage_ctr / LT_NSTAGE) & 1, p.err);
        __syncwarp();
        const uint32_t a_lo = (((a_base + s * LT_STAGE_BYTES) >> 4) & 0x3FFF) |
                              ((LT_A_LBO >> 4) << 16);
        const uint32_t b_lo = ((w_base >> 4) & 0x3FFF) | ((LT_B_LBO >> 4) << 16);
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int ks = 0; ks < 2; ++ks) {
            const uint32_t al0 = a_lo + 64u * h + 2 * ks * (LT_A_LBO >> 4);
            const uint64_t ah = pack64(al0, desc_hi);
            const uint64_t al = pack64(al0 + (LT_A_HL >> 4), desc_hi);
            const uint64_t bh = pack64(b_lo + 2 * ks * (LT_B_LBO >> 4), desc_hi);
            const uint64_t bl = pack64(b_lo + 2 * ks * (LT_B_LBO >> 4) + (LT_B_HL >> 4), desc_hi);
            wgmma_bf16<32>(acc[h], ah, bh);
            wgmma_bf16<32>(acc[h], al, bh);
            wgmma_bf16<32>(acc[h], ah, bl);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_a(s));
        // Q of this plane to shared memory: register i holds position 64h + 16*warp + lane/4 +
        // 8*((i/2)&1), tap 8*(i/4) + 2*(lane%4) + (i&1)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int t = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
            const int pos = 64 * h + 16 * warp + (lane >> 2) + 8 * ((i >> 1) & 1);
            if (t < 27) qb[t * 128 + pos] = acc[h][i];
            acc[h][i] = 0.f;
          }
        // all 128 positions of this plane are in shared memory (the other q buffer still
        // belongs to the previous plane's gather, which every thread has left by now)
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (olive) {
          float s0 = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
          for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
              const int pos = (by + ky - 1) * LT_PX + bx + kx - 1;
              s0 += qb[(0 * 9 + ky * 3 + kx) * 128 + pos];
              s1 += qb[(1 * 9 + ky * 3 + kx) * 128 + pos];
              s2 += qb[(2 * 9 + ky * 3 + kx) * 128 + pos];
            }
          const int zo = zi - 1;
          if (zo >= z_lo && zo < z_hi) p.out[(long long)zo * plane + (long long)oy * p.W + ox] = accA + s2;
          accA = accB + s1;
          accB = s0;
        }
      }
      if (z_hi == p.D && olive)
        p.out[(long long)(p.D - 1) * plane + (long long)oy * p.W + ox] = accA;
    }
  }
}

struct LogitsTcWeights {
  uint8_t* dev = nullptr;
  bool ready() const { return dev != nullptr; }
  void release() {
    if (dev) cudaFree(dev);
    dev = nullptr;
  }
  bool build(const float* w /*[27][32]*/) {
    release();
    std::vector<uint16_t> img;
    logits_tc_pack(w, img);
    return cudaMalloc(&dev, LT_W_BYTES) == cudaSuccess &&
           cudaMemcpy(dev, img.data(), LT_W_BYTES, cudaMemcpyHostToDevice) == cudaSuccess;
  }
};

inline bool logits_tc_launch(const Src& s, const LogitsTcWeights& w, float* out, int D, int H,
                             int W, cudaStream_t st) {
  if (s.n != 1 || s.outer_relu || !w.ready()) return false;
  LogitsTcParams p{};
  p.wimg = w.dev;
  p.out = out;
  p.D = D; p.H = H; p.W = W;
  p.tiles_x = (W + LT_OX - 1) / LT_OX;
  p.tiles_y = (H + LT_OY - 1) / LT_OY;
  p.zchunks = (D + LT_ZC - 1) / LT_ZC;
  const long long items = (long long)p.tiles_x * p.tiles_y * p.zchunks;
  if (items > 0x7fffffffLL) return false;
  p.nitems = (int)items;
  p.err = tc_err_flag().get();
  const size_t smem = LT_W_BYTES + LT_NSTAGE * LT_STAGE_BYTES + 2 * 27 * 128 * 4 +
                      2 * LT_NSTAGE * 8;
  bool& attr_done = per_device<bool, 31>();
  if (!attr_done) {
    if (cudaFuncSetAttribute(logits_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)smem) != cudaSuccess)
      return false;
    attr_done = true;
  }
  // two CTAs per SM (96 KB of shared memory each): the loaders are latency bound, a second
  // CTA fills their stalls
  const int grid = (int)std::min<long long>(items, 2LL * tc_sm_count());
  logits_tc_kernel<<<grid, LT_THREADS, smem, st>>>(p, SrcLoader8<1>{s, 32, H, W});
  return cudaGetLastError() == cudaSuccess;
}

}  // namespace dfm
