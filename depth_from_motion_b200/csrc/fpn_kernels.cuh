// Kernels of mmdet's FPN image neck as both MultiViewDfM (Waymo) configs use it
// (in_channels [256, 512, 1024, 2048], out_channels 64, num_outs 4, no extra convs, no norm,
// nearest upsampling): the lateral 1x1 convs with the top-down merge fused into their epilogue
//     merged_l[p][:] = W_l x_l[:, p] + b_l + merged_{l+1}[nearest(p)][:]
// computed coarsest level first.  The 3x3 fpn_convs run on the 2-D layer driver of bev_api.inc.
//
// fpn_lateral_tc_kernel: the wgmma GEMM of head1x1_tc.cuh (same tile of 128 flattened cells,
// same loader transpose into the K-major no-swizzle layout, same 3-term bf16 split with fp32
// accumulation) with two differences:
//   * The weights are streamed.  K = 2048 would need a 512 KB resident hi + lo image, so each
//     64-channel stage carries its 64 x 64 slice of the weight image next to the activations;
//     the loaders copy it with cp.async while they transpose the activations.  The weight
//     image is 16 KB per stage and is read from L2 by every tile.
//   * Input is NCHW for N images in one launch; output is channels-last [N][h][w][64].  The
//     tile index runs over (image, 128-cell tile); tiles never straddle images, and each
//     image's last tile is ragged.  The epilogue stages the accumulators as [cell][64 + 8]
//     (float2 fragment stores hit every bank once per 8-lane phase), then each thread writes
//     whole float4 channel groups of a cell: bias and the upsampled coarser level are added in
//     fp32, and one tile's output is 32 KB of contiguous memory.
//
// fpn_lateral_simt_kernel: the same layer on fp32 CUDA cores (the conv_impl = simt cross-check
// and the fall-back for out_channels without a tensor-core kernel).
#pragma once
#include "head1x1_tc.cuh"

namespace dfm {

constexpr int FPN_N = 64;                               // output channels of the tc kernel
constexpr uint32_t FPN_A_BYTES = H1_STAGE_BYTES;        // activations hi | lo (32 KB)
constexpr uint32_t FPN_B_HL = (H1_KC / 8) * FPN_N * 16;  // weight slice hi -> lo (8 KB)
constexpr uint32_t FPN_STAGE_BYTES = FPN_A_BYTES + 2 * FPN_B_HL;  // 48 KB
constexpr int FPN_OUT_LD = FPN_N + 8;                   // staged row pitch (floats)
constexpr size_t FPN_TC_SMEM =
    (size_t)H1_NSTAGE * FPN_STAGE_BYTES + (size_t)H1_M * FPN_OUT_LD * 4 + 2 * H1_NSTAGE * 8;

struct FpnLateralParams {
  const float* x;        // [N][cin][h][w]
  const uint8_t* wimg;   // tc: hi image then lo image, each [cin_pad / 8][64][8] bf16
  const float* wt;       // simt: [cin][cout] fp32
  const float* bias;     // [cout]
  const float* up;       // merged coarser level [N][hc][wc][cout], or null (coarsest level)
  float* out;            // [N][h][w][cout]
  int cin, cin_pad, h, w, hc, wc, hw, tpi, ntiles, vec4;
  int* err;
};

// PyTorch's legacy nearest index for F.interpolate(size=...): identity for equal sizes,
// dst >> 1 for an exact doubling, else min(floor(dst * (in / out)), in - 1) in fp32
__device__ __forceinline__ int fpn_nearest(int dst, int in, int out) {
  if (in == out) return dst;
  if (out == 2 * in) return dst >> 1;
  const float scale = (float)in / (float)out;
  return min((int)floorf((float)dst * scale), in - 1);
}

// index of the coarser level's cell (image-major) that cell `cell` of image img adds
__device__ __forceinline__ long long fpn_up_row(const FpnLateralParams& p, int img, int cell) {
  const int y = cell / p.w, x = cell - y * p.w;
  const int yc = fpn_nearest(y, p.hc, p.h), xc = fpn_nearest(x, p.wc, p.w);
  return ((long long)img * p.hc * p.wc + (long long)yc * p.wc + xc);
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}

__global__ void __launch_bounds__(H1_THREADS, 1)
fpn_lateral_tc_kernel(const __grid_constant__ FpnLateralParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* st_s = smem;
  float* out_s = reinterpret_cast<float*>(smem + H1_NSTAGE * FPN_STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(out_s + H1_M * FPN_OUT_LD);

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const uint32_t bar0 = smem_u32(bars);
  auto full = [&](int s) { return bar0 + 8u * s; };
  auto empty = [&](int s) { return bar0 + 8u * (H1_NSTAGE + s); };

  if (tid == 0) {
    for (int s = 0; s < H1_NSTAGE; ++s) {
      mbar_init(full(s), 4);    // one arrival per loader warp of the group
      mbar_init(empty(s), 8);   // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int nk = p.cin_pad / H1_KC;

  if (warp >= 8) {
    // ================================ loaders ================================
    const int lw = warp - 8, grp = lw >> 2, wq = lw & 3, lt = wq * 32 + lane;
    const int rot = (lane >> 1) & 3;
    const size_t w_half = (size_t)p.cin_pad * FPN_N * 2;   // bytes of the hi image
    uint32_t ctr = 0;
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
      const int img = tile / p.tpi;
      const int cell = (tile - img * p.tpi) * H1_M + 4 * lane;
      const float* xc = p.x + (long long)img * p.cin * p.hw + cell;
      for (int kc = 0; kc < nk; ++kc, ++ctr) {
        if ((int)(ctr & 1) != grp) continue;
        const int s = ctr % H1_NSTAGE;
        float4 f[2][8];
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
          for (int c = 0; c < 8; ++c)
            f[q][c] = h1_load4(xc, p.hw, p.hw - cell, p.vec4, kc * H1_KC + (2 * wq + q) * 8 + c,
                               p.cin);
        mbar_wait(empty(s), ((ctr / H1_NSTAGE) & 1) ^ 1, p.err);
        uint8_t* st = st_s + s * FPN_STAGE_BYTES;
        // this stage's weight slice: 8 KB of the hi image and 8 KB of the lo image
        const uint32_t b_dst = smem_u32(st + FPN_A_BYTES);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int i = lt + 128 * j, half = i >> 9, off = (i & 511) * 16;
          cp_async16(b_dst + half * FPN_B_HL + off,
                     p.wimg + half * w_half + (size_t)kc * FPN_B_HL + off);
        }
#pragma unroll
        for (int q = 0; q < 2; ++q) {
#pragma unroll
          for (int c = 0; c < 8; ++c) f[q][c] = h1_rot4(f[q][c], rot);
          uint8_t* chunk = st + (2 * wq + q) * H1_A_LBO;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float v[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) v[c] = h1_comp(f[q][c], j);
            const int row = 4 * lane + ((j + rot) & 3);
            split_store(v, chunk + row * 16, chunk + H1_A_HL + row * 16);
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
    const int wg = warp >> 2;
    constexpr uint32_t B_LBO = FPN_N * 16;
    const uint32_t desc_hi = 128u >> 4;                            // SBO: dense 8-row groups
    float acc[FPN_N / 2];
    uint32_t ctr = 0;
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
#pragma unroll
      for (int i = 0; i < FPN_N / 2; ++i) acc[i] = 0.f;
      for (int kc = 0; kc < nk; ++kc, ++ctr) {
        const int s = ctr % H1_NSTAGE;
        mbar_wait(full(s), (ctr / H1_NSTAGE) & 1, p.err);
        const uint32_t st = smem_u32(st_s + s * FPN_STAGE_BYTES);
        const uint32_t a_lo = (((st + wg * 64 * 16) >> 4) & 0x3FFF) | ((H1_A_LBO >> 4) << 16);
        const uint32_t b_lo = (((st + FPN_A_BYTES) >> 4) & 0x3FFF) | ((B_LBO >> 4) << 16);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < H1_KC / 16; ++ks) {
          const uint64_t ah = pack64(a_lo + 2 * ks * (H1_A_LBO >> 4), desc_hi);
          const uint64_t al = pack64(a_lo + 2 * ks * (H1_A_LBO >> 4) + (H1_A_HL >> 4), desc_hi);
          const uint64_t bh = pack64(b_lo + 2 * ks * (B_LBO >> 4), desc_hi);
          const uint64_t bl = pack64(b_lo + 2 * ks * (B_LBO >> 4) + (FPN_B_HL >> 4), desc_hi);
          wgmma_bf16<FPN_N>(acc, ah, bh);
          wgmma_bf16<FPN_N>(acc, al, bh);
          wgmma_bf16<FPN_N>(acc, ah, bl);
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(empty(s));
      }
      // every consumer has finished reading the previous tile's staging rows
      asm volatile("bar.sync 1, 256;" ::: "memory");
      // registers (i, i + 1): cell 64 wg + 16 (warp % 4) + lane / 4 + 8 ((i / 2) & 1),
      //                       channels 8 (i / 4) + 2 (lane % 4) + {0, 1}
#pragma unroll
      for (int i = 0; i < FPN_N / 2; i += 2) {
        const int m = 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * ((i >> 1) & 1);
        const int n = 8 * (i >> 2) + 2 * (lane & 3);
        *reinterpret_cast<float2*>(out_s + m * FPN_OUT_LD + n) = make_float2(acc[i], acc[i + 1]);
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      const int img = tile / p.tpi;
      const int p0 = (tile - img * p.tpi) * H1_M;
      float* out = p.out + ((long long)img * p.hw + p0) * FPN_N;
#pragma unroll 2
      for (int j = 0; j < H1_M * FPN_N / 4 / 256; ++j) {
        const int idx = tid + 256 * j, m = idx >> 4, c4 = (idx & 15) * 4;
        if (p0 + m >= p.hw) break;
        const float4 a = *reinterpret_cast<const float4*>(out_s + m * FPN_OUT_LD + c4);
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + c4));
        float4 v = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
        if (p.up) {
          const float4 u = __ldg(reinterpret_cast<const float4*>(
              p.up + fpn_up_row(p, img, p0 + m) * FPN_N + c4));
          v = make_float4(v.x + u.x, v.y + u.y, v.z + u.z, v.w + u.w);
        }
        *reinterpret_cast<float4*>(out + (long long)m * FPN_N + c4) = v;
      }
    }
  }
}

constexpr int FPN_SIMT_CELLS = 64;   // cells per block
constexpr int FPN_SIMT_KC = 32;      // input channels per shared-memory step

// 256 threads: thread t owns cells 4 (t % 16) .. + 3 of the tile and output channels
// (t / 16) * COUT / 16 .. + COUT / 16 - 1; fp32 FMAs in input-channel order
template <int COUT>
__global__ void __launch_bounds__(256) fpn_lateral_simt_kernel(const FpnLateralParams p) {
  constexpr int CPT = COUT / 16;
  __shared__ float xs[FPN_SIMT_KC][FPN_SIMT_CELLS];
  __shared__ float ws[FPN_SIMT_KC][COUT];
  const int tid = threadIdx.x, cg = tid & 15, og = tid >> 4;
  const int img = blockIdx.x / p.tpi;
  const int p0 = (blockIdx.x - img * p.tpi) * FPN_SIMT_CELLS;
  const float* xi = p.x + (long long)img * p.cin * p.hw;
  float acc[4][CPT];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int o = 0; o < CPT; ++o) acc[j][o] = 0.f;
  for (int k0 = 0; k0 < p.cin; k0 += FPN_SIMT_KC) {
    for (int i = tid; i < FPN_SIMT_KC * FPN_SIMT_CELLS; i += 256) {
      const int kk = i / FPN_SIMT_CELLS, cc = i % FPN_SIMT_CELLS;
      xs[kk][cc] = (k0 + kk < p.cin && p0 + cc < p.hw)
                       ? __ldg(xi + (long long)(k0 + kk) * p.hw + p0 + cc) : 0.f;
    }
    for (int i = tid; i < FPN_SIMT_KC * COUT; i += 256) {
      const int kk = i / COUT, o = i % COUT;
      ws[kk][o] = k0 + kk < p.cin ? __ldg(p.wt + (long long)(k0 + kk) * COUT + o) : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int kk = 0; kk < FPN_SIMT_KC; ++kk) {
      float xv[4], wv[CPT];
#pragma unroll
      for (int j = 0; j < 4; ++j) xv[j] = xs[kk][4 * cg + j];
#pragma unroll
      for (int o = 0; o < CPT; ++o) wv[o] = ws[kk][og * CPT + o];
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int o = 0; o < CPT; ++o) acc[j][o] = fmaf(xv[j], wv[o], acc[j][o]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int cell = p0 + 4 * cg + j;
    if (cell >= p.hw) continue;
    const float* up = p.up ? p.up + fpn_up_row(p, img, cell) * COUT : nullptr;
    float* out = p.out + ((long long)img * p.hw + cell) * COUT;
#pragma unroll
    for (int o = 0; o < CPT; ++o) {
      const int c = og * CPT + o;
      float v = acc[j][o] + __ldg(p.bias + c);
      if (up) v += __ldg(up + c);
      out[c] = v;
    }
  }
}

}  // namespace dfm
