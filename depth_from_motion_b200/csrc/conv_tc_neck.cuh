// wgmma 3x3x3 conv for the BEV necks (DfMNeck / OutdoorImVoxelNeck, SURVEY.md 8a row a7):
// 64..256 channels on a [Nx=220][Ny=300][Nz<=12] voxel grid, strides (1,1,1) / (1,1,2),
// pads (1,1,1) / (1,1,0).
//
// Same operand formulation as conv_tc.cuh (bf16 hi/lo split, K-major no-swizzle bricks, one
// brick serves the 9 in-plane taps, kz folded into N), but the loop nest is K-outer because
// the weights (27*Cin*Cout*4 B, up to 7 MB) cannot stay resident:
//   * a CTA owns a 16 (x) x 8 (y) tile and a window of output planes of the short z axis
//     (as many as NK_ACC_COLS accumulator columns hold; taller volumes are cut into windows
//     whose halo planes are real data); the accumulators live in the registers of the two
//     consumer warpgroups for the whole item;
//   * for each 32-channel input group: copy that group's 110.6 KB weight image to shared
//     memory, then march the input planes through the usual loader -> MMA pipeline;
//   * after the last group the consumers store the planes (raw conv output; BatchNorm/ReLU
//     are applied by the consumer's load, like everywhere else).
// "Windowed" use (neck_tc_conv_dhw): the same kernel runs the 64-channel stride-1 layers of the
// plane-sweep volume [D][H][W][C] -- tile over (H, W), marched axis D cut into windows of output
// planes whose halo planes are real data -- because there the resident-weight kernel
// (conv_tc.cuh) has to split the output channels four ways and issues N = 48 MMAs; here an MMA
// covers 32 output channels x 3 planes (N = 96).
#pragma once
#include "conv_tc.cuh"

namespace dfm {

constexpr int NK_BX = 8, NK_BY = 16;           // tile: 8 along y (brick x), 16 along x (brick y)
constexpr int NK_PX = NK_BX + 2, NK_PY = NK_BY + 2;
constexpr int NK_ROWS = 186;                    // 180 brick rows padded (== 2 mod 8)
// accumulator columns per CTA: 64 registers per consumer thread
constexpr int NK_ACC_COLS = 128;
// Two shapes of the per-CTA weight image (always 110.6 KB = 9 taps x CG x 3*NCTA x hi/lo):
//   CG = 32 input channels per group, NCTA = 32 output channels per CTA (4 planes per window)
//   CG = 16, NCTA = 64: every loaded brick feeds twice the MMA columns (N = 128 / 64 instead of
//   96 / 32) and the output channels are split half as often, i.e. every brick is loaded half as
//   often -- for layers with <= 2 output planes per tile (64 accumulator columns per plane).
template <int CG>
struct NkCfg {
  static constexpr int NCH = CG / 8;             // 16-byte channel chunks per stage
  static constexpr int NCTA = 1024 / CG;         // output channels per CTA
  static constexpr int KS = CG / 16;             // K steps per tap
  static constexpr int NSTAGE = CG == 32 ? 4 : 8;
  static constexpr int ZMAX = NK_ACC_COLS / NCTA;  // (tile, plane) accumulators of an item
  static constexpr uint32_t STAGE_BYTES = 2 * NCH * NK_ROWS * 16;
  static constexpr uint32_t B_LBO16 = 3 * NCTA;  // rows of a group image: [kw block][NCTA]
  static constexpr uint32_t TAP16 = NCH * B_LBO16;   // one in-plane tap, 16-byte units (= 384)
};
constexpr uint32_t NK_TAP16 = 4 * 96;           // == NkCfg<32>::TAP16 == NkCfg<16>::TAP16
constexpr uint32_t NK_WHI_BYTES = 9 * NK_TAP16 * 16;
constexpr uint32_t NK_W_BYTES = 2 * NK_WHI_BYTES;
constexpr int NK_MAX_NCTA = 64;
constexpr int NK_MMA_THREADS = 256;    // two warpgroups: MMA issue + epilogue, 64 rows each
constexpr int NK_LOAD_THREADS = 256;   // 2 groups x 4 warps
constexpr int NK_THREADS = NK_MMA_THREADS + NK_LOAD_THREADS;  // 16 warps: 128 registers/thread

enum { NKZ_S1P1 = 0, NKZ_S2P1 = 1, NKZ_S1P0 = 2 };

inline int nk_zmode(const ConvGeom& g) {
  if (g.transposed || g.sd != 1 || g.sh != 1 || g.pd != 1 || g.ph != 1) return -1;
  if (g.Cin % 32 || g.Cout % 32 || g.Cin < 64 || g.Wo > 16) return -1;
  if (g.sw == 1 && g.pw == 1) return NKZ_S1P1;
  if (g.sw == 2 && g.pw == 1 && g.Wi % 2 == 0) return NKZ_S2P1;
  if (g.sw == 1 && g.pw == 0 && g.Wo == 1 && g.Wi == 3) return NKZ_S1P0;
  return -1;
}

struct NeckTcWeights {
  DevArray<uint8_t> dev;   // [nsplit][ncg][NK_W_BYTES]
  int Cin = 0, Cout = 0, zmode = -1;
  int cg = 32;             // input channels per group (32 -> NCTA 32, 16 -> NCTA 64)
  bool ready() const { return dev.p != nullptr; }
  void release() { dev.release(); }
  // packed: [27][Cin][Cout] fp32, tap = kz*9 + ky*3 + kx with (kz,ky,kx) over (Nz, Ny, Nx)...
  // NOTE the conv dims are (D,H,W) = (Nx, Ny, Nz): the packed tap index is kd*9 + kh*3 + kw,
  // i.e. kd over Nx, kh over Ny, kw over Nz (the short, marched axis).
  // dhw: the volume is [D][H][W][C] with D the marched axis (tile over H (16) x W (8)): the
  // in-plane tap t is kh * 3 + kw and the marched tap is kd
  bool build(const float* packed, int cin, int cout, int zm, std::string* err, bool dhw = false,
             int cgroup = 32) {
    release();
    Cin = cin;
    Cout = cout;
    zmode = zm;
    cg = cgroup;
    const int ncta = 1024 / cg, nch = cg / 8;
    if ((cg != 32 && cg != 16) || cout % ncta || cin % cg) {
      if (err) *err = "NeckTcWeights: channel counts do not fit the group shape";
      return false;
    }
    const int nsplit = cout / ncta, ncg = cin / cg;
    // order of the three marched-axis taps inside an image (see kernel): consecutive row
    // blocks must land in consecutive output planes
    const int order[3][3] = {{2, 1, 0}, {2, 0, 1}, {0, 1, 2}};
    std::vector<uint16_t> img((size_t)nsplit * ncg * NK_W_BYTES / 2);
    for (int s = 0; s < nsplit; ++s)
      for (int g = 0; g < ncg; ++g)
        for (int t = 0; t < 9; ++t) {      // in-plane tap: kd (Nx) * 3 + kh (Ny)
          const int kd = t / 3, kh = t % 3;
          for (int kc = 0; kc < nch; ++kc)
            for (int r = 0; r < 3 * ncta; ++r)
              for (int e = 0; e < 8; ++e) {
                const int kw = order[zm][r / ncta];
                const int co = s * ncta + r % ncta, ci = g * cg + kc * 8 + e;
                const int tap = dhw ? kw * 9 + kd * 3 + kh : kd * 9 + kh * 3 + kw;
                const float w = packed[((size_t)tap * cin + ci) * cout + co];
                const uint16_t hi = bf16_rn_bits(w);
                const uint16_t lo = bf16_rn_bits(w - bf16_bits_to_float(hi));
                const size_t base = ((size_t)s * ncg + g) * (NK_W_BYTES / 2);
                const size_t off = base + (((size_t)t * nch + kc) * (3 * ncta) + r) * 8 + e;
                img[off] = hi;
                img[off + NK_WHI_BYTES / 2] = lo;
              }
        }
    if (dev.upload(reinterpret_cast<const uint8_t*>(img.data()), img.size() * 2) != cudaSuccess) {
      if (err) *err = "NeckTcWeights: device upload failed";
      release();
      return false;
    }
    return true;
  }
};

struct NeckParams {
  const uint8_t* wimg;
  float* out;
  Src src;
  int Nx, Ny, Zi, Zo, Cin, Cout;
  int zmode;
  int tiles_x, tiles_y, nsplit, ncg, n_items;
  int ntiles;   // tiles_x * tiles_y
  int tpi;      // tiles per item: their accumulators (ZC * NCTA columns each) share the
                // NK_ACC_COLS register columns, so one 110 KB weight image serves tpi tiles
  // voxel strides of (tile-y axis "x", tile-x axis "y", marched axis) for the input / output
  long long in_sx, in_sy, in_sz, out_sx, out_sy, out_sz;
  int ZC;       // output planes per item along the marched axis (== Zo unless windowed)
  int nchunk;   // windows along the marched axis (1 unless windowed; not for NKZ_S1P0)
  double* stats;            // optional per-output-channel (sum, sum of squares) of the raw output
  int zw_lo, zw_hi;         // planes [zw_lo, zw_hi) enter the statistics with weight zw
  float zw;
  int* err;
};

// 8 consecutive channels of input voxel (ix, iy, iz), with the fused input transform
template <int NT>
struct NeckLoader {
  struct Raw {
    float4 a[NT][2];
  };
  static __device__ __forceinline__ void issue(const NeckParams& p, long long vox, int c0, Raw& r) {
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const float* px = p.src.t[t].x + vox * p.Cin + c0;
      r.a[t][0] = __ldg(reinterpret_cast<const float4*>(px));
      r.a[t][1] = __ldg(reinterpret_cast<const float4*>(px) + 1);
    }
  }
  static __device__ __forceinline__ void finish(const NeckParams& p, const Raw& r, int c0,
                                                float v[8]) {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = 0.f;
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      float u[8] = {r.a[t][0].x, r.a[t][0].y, r.a[t][0].z, r.a[t][0].w,
                    r.a[t][1].x, r.a[t][1].y, r.a[t][1].z, r.a[t][1].w};
      const Term& tm = p.src.t[t];
      if (tm.scale) {
        const float4 s0 = __ldg(reinterpret_cast<const float4*>(tm.scale + c0));
        const float4 s1 = __ldg(reinterpret_cast<const float4*>(tm.scale + c0) + 1);
        const float4 h0 = __ldg(reinterpret_cast<const float4*>(tm.shift + c0));
        const float4 h1 = __ldg(reinterpret_cast<const float4*>(tm.shift + c0) + 1);
        const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
        const float sh[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) u[i] = fmaf(u[i], sc[i], sh[i]);
      }
      if (tm.relu) {
#pragma unroll
        for (int i = 0; i < 8; ++i) u[i] = fmaxf(u[i], 0.f);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] += u[i];
    }
    if (p.src.outer_relu) {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = fmaxf(v[i], 0.f);
    }
  }
};

// which weight rows / output planes input plane iz feeds: rows [n0, n0+n) -> planes zo0...
// (iz: absolute input plane; the item owns output planes [zo_lo, zo_hi); zo0 is relative to zo_lo)
// n0 is in weight-row BLOCKS (multiply by NCTA)
__device__ __forceinline__ void nk_plane_map(int zmode, int iz, int zo_lo, int zo_hi, int& n0,
                                             int& nblk, int& zo0) {
  if (zmode == NKZ_S1P1) {        // rows [kw=2|1|0] -> planes iz-1, iz, iz+1
    const int first = max(iz - 1, zo_lo), last = min(iz + 1, zo_hi - 1);
    n0 = first - (iz - 1);
    nblk = last - first + 1;
    zo0 = first - zo_lo;
  } else if (zmode == NKZ_S2P1) { // rows [kw=2|0|1]; iz = 2q+1 -> planes q, q+1; iz = 2q -> q
    const int q = iz >> 1;
    if (iz & 1) {
      const int first = max(q, zo_lo), last = min(q + 1, zo_hi - 1);
      n0 = first - q;
      nblk = last - first + 1;
      zo0 = first - zo_lo;
    } else {
      n0 = 2;
      nblk = 1;
      zo0 = q - zo_lo;
    }
  } else {                        // pad 0, single output plane: kw = iz
    n0 = iz;
    nblk = 1;
    zo0 = 0;
  }
}

// item -> (first tile, tiles, marched-axis window and the input planes it reads)
struct NkItem {
  int tile0, nt, zo_lo, zo_hi, iz_lo, nzi;
};
__device__ __forceinline__ NkItem nk_item(const NeckParams& p, int item) {
  NkItem it;
  const int unit = item / p.nsplit;
  const int chunk = unit % p.nchunk;
  it.tile0 = (unit / p.nchunk) * p.tpi;
  it.nt = min(p.tpi, p.ntiles - it.tile0);
  it.zo_lo = chunk * p.ZC;
  it.zo_hi = min(it.zo_lo + p.ZC, p.Zo);
  // halo planes of a window are real data where they exist
  int iz_hi;
  if (p.zmode == NKZ_S1P1) {
    it.iz_lo = max(it.zo_lo - 1, 0);
    iz_hi = min(it.zo_hi + 1, p.Zi);
  } else if (p.zmode == NKZ_S2P1) {
    it.iz_lo = max(2 * it.zo_lo - 1, 0);
    iz_hi = min(2 * it.zo_hi, p.Zi);
  } else {
    it.iz_lo = 0;
    iz_hi = p.Zi;
  }
  it.nzi = iz_hi - it.iz_lo;
  return it;
}

// calls f(Q, NB) with compile-time Q == q, NB == nb (Q + NB <= ZMAX)
template <int Q, int ZMAX, class F>
__device__ __forceinline__ void nk_dispatch(int q, int nb, F&& f) {
  if constexpr (Q < ZMAX) {
    if (q == Q) {
      if (nb == 1) f(std::integral_constant<int, Q>(), std::integral_constant<int, 1>());
      if constexpr (Q + 2 <= ZMAX)
        if (nb == 2) f(std::integral_constant<int, Q>(), std::integral_constant<int, 2>());
      if constexpr (Q + 3 <= ZMAX)
        if (nb == 3) f(std::integral_constant<int, Q>(), std::integral_constant<int, 3>());
    } else {
      nk_dispatch<Q + 1, ZMAX>(q, nb, f);
    }
  }
}

template <int NT, int CG>
__global__ void __launch_bounds__(NK_THREADS, 1)
neck_conv_kernel(const __grid_constant__ NeckParams p) {
  using Cfg = NkCfg<CG>;
  constexpr int NCH = Cfg::NCH, NK_NCTA = Cfg::NCTA, KS = Cfg::KS, NK_NSTAGE = Cfg::NSTAGE;
  constexpr int ZMAX = Cfg::ZMAX;
  constexpr uint32_t NK_STAGE_BYTES = Cfg::STAGE_BYTES;
  constexpr uint32_t A_LBO = NK_ROWS * 16, A_SBO = NK_PX * 16, A_HL = NCH * NK_ROWS * 16;
  constexpr uint32_t A_LBO16 = A_LBO >> 4, A_HL16 = A_HL >> 4, B_LBO16 = Cfg::B_LBO16;
  constexpr int NPOS = NK_PX * NK_PY, LG_THREADS = NK_LOAD_THREADS / 2;
  constexpr int NITEM = (NPOS * NCH + LG_THREADS - 1) / LG_THREADS;
  constexpr int LB = NITEM < 6 / NT ? NITEM : 6 / NT;
  constexpr int NACC = ZMAX * NK_NCTA / 2;
  constexpr int LOAD_WARP0 = NK_MMA_THREADS / 32;

  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* w_s = smem;
  uint8_t* a_s = smem + NK_W_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(a_s + NK_NSTAGE * NK_STAGE_BYTES);
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const uint32_t bar0 = smem_u32(bars);
  auto full_a = [&](int s) { return bar0 + 8u * s; };
  auto empty_a = [&](int s) { return bar0 + 8u * (NK_NSTAGE + s); };
  const uint32_t w_full = bar0 + 8u * (2 * NK_NSTAGE), w_empty = w_full + 8;

  if (tid == 0) {
    for (int s = 0; s < NK_NSTAGE; ++s) {
      mbar_init(full_a(s), LG_THREADS / 32);
      mbar_init(empty_a(s), NK_MMA_THREADS / 32);
    }
    mbar_init(w_full, NK_LOAD_THREADS / 32);
    mbar_init(w_empty, NK_MMA_THREADS / 32);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int split = blockIdx.x % p.nsplit;

  if (warp >= LOAD_WARP0) {
    // ============================ loaders ============================
    const int lw = warp - LOAD_WARP0, lgrp = lw & 1;
    const int lt = (lw >> 1) * 32 + lane, lall = lw * 32 + lane;
    const int chunk = lt % NCH;
    uint32_t stage_ctr = 0, w_ctr = 0;
    for (int item = blockIdx.x; item < p.n_items; item += gridDim.x) {
      const NkItem it = nk_item(p, item);
      const int tile0 = it.tile0, nt = it.nt;
      for (int cg = 0; cg < p.ncg; ++cg, ++w_ctr) {
        // this group's weight image (all loader threads), once the previous group's MMAs retired
        mbar_wait(w_empty, (w_ctr & 1) ^ 1, p.err);
        {
          const uint4* src = reinterpret_cast<const uint4*>(
              p.wimg + ((size_t)split * p.ncg + cg) * NK_W_BYTES);
          uint4* dst = reinterpret_cast<uint4*>(w_s);
          for (uint32_t i = lall; i < NK_W_BYTES / 16; i += NK_LOAD_THREADS) dst[i] = __ldg(src + i);
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          __syncwarp();
          if (lane == 0) mbar_arrive(w_full);
        }
        for (int t = 0; t < nt; ++t) {
          const int tile = tile0 + t;
          const int y0 = (tile % p.tiles_x) * NK_BX, x0 = (tile / p.tiles_x) * NK_BY;
          for (int izl = 0; izl < it.nzi; ++izl, ++stage_ctr) {
            if ((int)(stage_ctr & 1) != lgrp) continue;
            const int iz = it.iz_lo + izl;
            const int s = stage_ctr % NK_NSTAGE;
            mbar_wait(empty_a(s), ((stage_ctr / NK_NSTAGE) & 1) ^ 1, p.err);
            uint8_t* st = a_s + s * NK_STAGE_BYTES;
            const int c0 = cg * CG + chunk * 8;
#pragma unroll
            for (int k0 = 0; k0 < NITEM; k0 += LB) {
              typename NeckLoader<NT>::Raw raw[LB];
              bool inb[LB], live[LB];
              int soff[LB];
#pragma unroll
              for (int b = 0; b < LB; ++b) {
                const int i = lt + (k0 + b) * LG_THREADS;
                live[b] = (k0 + b) < NITEM && i < NPOS * NCH;
                const int pos = i / NCH;
                const int bx = pos % NK_PX, by = pos / NK_PX;
                const int gy = y0 - 1 + bx, gx = x0 - 1 + by;
                inb[b] = live[b] && gx >= 0 && gx < p.Nx && gy >= 0 && gy < p.Ny;
                soff[b] = (chunk * NK_ROWS + pos) * 16;
                if (inb[b])
                  NeckLoader<NT>::issue(p, gx * p.in_sx + gy * p.in_sy + iz * p.in_sz, c0, raw[b]);
              }
#pragma unroll
              for (int b = 0; b < LB; ++b) {
                if (live[b]) {
                  float v[8];
                  if (inb[b]) {
                    NeckLoader<NT>::finish(p, raw[b], c0, v);
                  } else {
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] = 0.f;
                  }
                  split_store(v, st + soff[b], st + A_HL + soff[b]);
                }
              }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(full_a(s));
          }
        }
      }
    }
  } else {
    // ================= consumers: two MMA + epilogue warpgroups (64 rows each) =================
    // The accumulators of all (tile, plane) pairs of an item stay in registers across the
    // input-channel groups; plane P = t * ZC + (zo - zo_lo) owns registers [P, P+1) * NCTA / 2.
    const int wg = warp >> 2, wq = warp & 3;
    const int xr = lane >> 2, cq = lane & 3;
    const uint32_t w_base = smem_u32(w_s), a_base = smem_u32(a_s);
    const uint32_t a_desc_hi = A_SBO >> 4, b_desc_hi = 128u >> 4;
    const uint32_t w_hi16 = NK_WHI_BYTES >> 4;
    const uint32_t a_wg16 = (uint32_t)wg * 8u * (A_SBO >> 4);
    float acc[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    constexpr int NST = NK_NCTA / 4;
    float ssum[NST], ssq[NST];   // GroupNorm sums of this item (p.stats), fp32
#pragma unroll
    for (int i = 0; i < NST; ++i) ssum[i] = ssq[i] = 0.f;
    uint32_t stage_ctr = 0, w_ctr = 0;
    for (int item = blockIdx.x; item < p.n_items; item += gridDim.x) {
      const NkItem it = nk_item(p, item);
      const int nt = it.nt;
      for (int cg = 0; cg < p.ncg; ++cg, ++w_ctr) {
        mbar_wait(w_full, w_ctr & 1, p.err);
        for (int t = 0; t < nt; ++t) {
          for (int izl = 0; izl < it.nzi; ++izl, ++stage_ctr) {
            const int s = stage_ctr % NK_NSTAGE;
            mbar_wait(full_a(s), (stage_ctr / NK_NSTAGE) & 1, p.err);
            __syncwarp();
            int n0, nblk, zo0;
            nk_plane_map(p.zmode, it.iz_lo + izl, it.zo_lo, it.zo_hi, n0, nblk, zo0);
            const uint32_t a_lo_stage =
                ((((a_base + s * NK_STAGE_BYTES) >> 4) & 0x3FFF) + a_wg16) | (A_LBO16 << 16);
            const uint32_t b_lo0 = ((w_base >> 4) & 0x3FFF) + (uint32_t)n0 * NK_NCTA + (B_LBO16 << 16);
            wgmma_fence();
            nk_dispatch<0, ZMAX>(t * p.ZC + zo0, nblk, [&](auto qc, auto nbc) {
              constexpr int Q = decltype(qc)::value, NB = decltype(nbc)::value;
              float* d = acc + Q * (NK_NCTA / 2);
              uint64_t da[KS][2], db[KS][2];
#pragma unroll
              for (int ks = 0; ks < KS; ++ks) {
                da[ks][0] = pack64(a_lo_stage + 2 * ks * A_LBO16, a_desc_hi);
                da[ks][1] = pack64(a_lo_stage + 2 * ks * A_LBO16 + A_HL16, a_desc_hi);
                db[ks][0] = pack64(b_lo0 + 2 * ks * B_LBO16, b_desc_hi);
                db[ks][1] = pack64(b_lo0 + 2 * ks * B_LBO16 + w_hi16, b_desc_hi);
              }
#pragma unroll 1
              for (int tap = 0; tap < 9; ++tap) {
#pragma unroll
                for (int ks = 0; ks < KS; ++ks) {
                  wgmma_bf16<NB * NK_NCTA>(d, da[ks][0], db[ks][0]);
                  wgmma_bf16<NB * NK_NCTA>(d, da[ks][1], db[ks][0]);
                  wgmma_bf16<NB * NK_NCTA>(d, da[ks][0], db[ks][1]);
                }
                const uint32_t ainc = (tap == 2 || tap == 5) ? (uint32_t)(NK_PX - 2) : 1u;
#pragma unroll
                for (int ks = 0; ks < KS; ++ks) {
                  desc_add(da[ks][0], ainc);
                  desc_add(da[ks][1], ainc);
                  desc_add(db[ks][0], NK_TAP16);
                  desc_add(db[ks][1], NK_TAP16);
                }
              }
            });
            wgmma_commit();
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_a(s));
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(w_empty);  // weights may be replaced: their MMAs retired
      }
      // ---- epilogue: raw conv output of every (tile, plane) of the item ----
      const int zc = it.zo_hi - it.zo_lo;
#pragma unroll
      for (int P = 0; P < ZMAX; ++P) {
        const int t = P / p.ZC, zo = it.zo_lo + P % p.ZC;
        if (t < nt && P % p.ZC < zc) {
          const int tile = it.tile0 + t;
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const int y = (tile % p.tiles_x) * NK_BX + xr;
            const int x = (tile / p.tiles_x) * NK_BY + 8 * wg + 2 * wq + rr;
            if (x >= p.Nx || y >= p.Ny) continue;
            float* dst = p.out + (x * p.out_sx + y * p.out_sy + zo * p.out_sz) * p.Cout +
                         split * NK_NCTA + 2 * cq;
            const float wz = (zo >= p.zw_lo && zo < p.zw_hi) ? p.zw : 1.f;
#pragma unroll
            for (int j = 0; j < NK_NCTA / 8; ++j) {
              const float v0 = acc[P * (NK_NCTA / 2) + 4 * j + 2 * rr];
              const float v1 = acc[P * (NK_NCTA / 2) + 4 * j + 2 * rr + 1];
              *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(v0, v1);
              if (p.stats) {
                ssum[2 * j] = fmaf(wz, v0, ssum[2 * j]);
                ssq[2 * j] = fmaf(wz * v0, v0, ssq[2 * j]);
                ssum[2 * j + 1] = fmaf(wz, v1, ssum[2 * j + 1]);
                ssq[2 * j + 1] = fmaf(wz * v1, v1, ssq[2 * j + 1]);
              }
            }
          }
        }
      }
#pragma unroll
      for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
      if (p.stats) {  // one flush per item keeps the fp32 partial sums short
#pragma unroll
        for (int k = 0; k < NST; ++k) {
          double a = ssum[k], b = ssq[k];
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, o);
            b += __shfl_xor_sync(0xffffffffu, b, o);
          }
          if (lane < 4) {
            const int ch = split * NK_NCTA + 8 * (k >> 1) + 2 * lane + (k & 1);
            atomicAdd(p.stats + 2 * ch, a);
            atomicAdd(p.stats + 2 * ch + 1, b);
          }
          ssum[k] = ssq[k] = 0.f;
        }
      }
    }
  }
}

inline bool neck_launch(NeckParams& p, int nterms, int cg, cudaStream_t st, std::string* err) {
  const size_t stages = cg == 32 ? (size_t)NkCfg<32>::NSTAGE * NkCfg<32>::STAGE_BYTES
                                 : (size_t)NkCfg<16>::NSTAGE * NkCfg<16>::STAGE_BYTES;
  const int nstage = cg == 32 ? NkCfg<32>::NSTAGE : NkCfg<16>::NSTAGE;
  const size_t smem = NK_W_BYTES + stages + (2 * nstage + 2) * 8;
  p.err = tc_err_flag().get();
  const int sms = tc_sm_count();
  int grid = std::max(p.nsplit, sms / p.nsplit * p.nsplit);
  grid = std::min(grid, p.n_items);
  grid = std::max(p.nsplit, grid / p.nsplit * p.nsplit);
  auto launch = [&](auto kern) -> bool {
    // (the instantiations share one function-pointer type, so no static "done" flag here)
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
        cudaSuccess) {
      if (err) *err = "neck_tc_conv: cannot reserve shared memory";
      return false;
    }
    kern<<<grid, NK_THREADS, smem, st>>>(p);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      if (err) *err = std::string("neck_tc_conv launch: ") + cudaGetErrorString(e);
      return false;
    }
    return true;
  };
  if (cg == 32 && nterms == 1) return launch(neck_conv_kernel<1, 32>);
  if (cg == 32 && nterms == 2) return launch(neck_conv_kernel<2, 32>);
  if (cg == 16 && nterms == 1) return launch(neck_conv_kernel<1, 16>);
  if (cg == 16 && nterms == 2) return launch(neck_conv_kernel<2, 16>);
  if (err) *err = "neck_tc_conv: at most two input terms";
  return false;
}

// group shape of a layer with `planes` output planes per tile: 16 / 64 when the accumulators fit
// (windowed = true: the layer is stride 1 / pad 1 along the short axis, so a taller volume can be
// cut into windows that fit -- DFM_NECK_WIN=1, A/B)
inline int neck_group_for(int cin, int cout, int planes, bool windowed = false) {
  static const bool off = getenv("DFM_NECK_CG32") != nullptr;   // A/B runs
  static const bool win = getenv("DFM_NECK_WIN") != nullptr;
  const bool fits = planes * 64 <= NK_ACC_COLS || (windowed && win);
  return (!off && fits && cout % 64 == 0 && cin % 16 == 0) ? 16 : 32;
}

// BEV-neck orientation: volume [Nx][Ny][Nz][C], the short Nz axis is marched whole
inline bool neck_tc_conv(const Src& s, const NeckTcWeights& w, float* out, const ConvGeom& g,
                         cudaStream_t st, std::string* err) {
  NeckParams p{};
  p.wimg = w.dev.p;
  p.out = out;
  p.src = s;
  p.Nx = g.Di; p.Ny = g.Hi; p.Zi = g.Wi; p.Zo = g.Wo;
  p.Cin = g.Cin; p.Cout = g.Cout;
  p.zmode = w.zmode;
  p.tiles_x = (g.Hi + NK_BX - 1) / NK_BX;   // along Ny
  p.tiles_y = (g.Di + NK_BY - 1) / NK_BY;   // along Nx
  const int ncta = 1024 / w.cg;
  // more planes than the accumulators hold in this group shape: windows along the short axis
  // (pad 1 only; their halo planes are real data)
  const int zmax = NK_ACC_COLS / ncta;
  int zc = g.Wo, nchunk = 1;
  if (g.Wo > zmax) {
    if (w.zmode == NKZ_S1P0) {
      if (err) *err = "neck_tc_conv: the weight image's group shape does not fit this plane count";
      return false;
    }
    nchunk = (g.Wo + zmax - 1) / zmax;
    zc = (g.Wo + nchunk - 1) / nchunk;
    nchunk = (g.Wo + zc - 1) / zc;
  }
  p.nsplit = g.Cout / ncta;
  p.ncg = g.Cin / w.cg;
  p.ntiles = p.tiles_x * p.tiles_y;
  p.in_sx = (long long)g.Hi * g.Wi; p.in_sy = g.Wi; p.in_sz = 1;
  p.out_sx = (long long)g.Ho * g.Wo; p.out_sy = g.Wo; p.out_sz = 1;
  p.ZC = zc;
  p.nchunk = nchunk;
  p.stats = nullptr;
  // tiles per item: as many as the accumulators hold (zc * NCTA columns per tile), but not so
  // many that the persistent grid runs short of items
  const int tpi_env = getenv("DFM_NECK_TPI") ? atoi(getenv("DFM_NECK_TPI")) : 0;  // tests / A-B runs
  {
    const int cap = std::max(1, zmax / zc);
    const int sms0 = tc_sm_count();
    int tpi = std::min(cap, std::max(1, p.ntiles * nchunk * p.nsplit / (2 * sms0)));
    if (tpi_env > 0) tpi = std::min(cap, tpi_env);
    p.tpi = std::max(1, tpi);
  }
  p.n_items = (p.ntiles + p.tpi - 1) / p.tpi * nchunk * p.nsplit;
  return neck_launch(p, s.n, w.cg, st, err);
}

// Plane-sweep-volume orientation: [D][H][W][C], stride 1, pad 1; tiles over (H: 16, W: 8), the
// D axis cut into windows of `zc` output planes (<= NK_ACC_COLS / NCTA).  `w` must have
// been built with dhw = true.  stats: optional GroupNorm sums of the raw output (zeroed by the
// caller), planes [zw_lo, zw_hi) weighted by zw.
inline bool neck_dhw_supported(const ConvGeom& g) {
  return !g.transposed && g.sd == 1 && g.sh == 1 && g.sw == 1 && g.pd == 1 && g.ph == 1 &&
         g.pw == 1 && g.Cin % 32 == 0 && g.Cout % 32 == 0 && g.Cin >= 64;
}
// Window length / tiles per item of the windowed launch: static round-robin over equal items, so
// pick the pair that minimises rounds x item cost (item cost ~ tpi * (zc + 2 halo planes) + the
// weight-image reload, ~1.5 plane-equivalents per 32-channel input group).
struct NeckDhwPlan {
  int zc, tpi, items;
};
inline NeckDhwPlan neck_dhw_plan(const ConvGeom& g, int ncta = 32) {
  const int sms = tc_sm_count();
  const int ntiles = ((g.Wi + NK_BX - 1) / NK_BX) * ((g.Hi + NK_BY - 1) / NK_BY);
  const int nsplit = g.Cout / ncta;
  const int zmax = std::min(g.Do, NK_ACC_COLS / ncta);
  NeckDhwPlan best{zmax, 1, 0};
  double best_cost = 1e30;
  for (int zc = zmax; zc >= std::min(g.Do, 4); --zc) {
    const int nchunk = (g.Do + zc - 1) / zc;
    for (int tpi = 1; tpi <= NK_ACC_COLS / (zc * ncta); ++tpi) {
      const int items = (ntiles + tpi - 1) / tpi * nchunk * nsplit;
      const int rounds = (items + sms - 1) / sms;
      const double cost = rounds * (tpi * (zc + 2.0) + 1.5);
      if (cost < best_cost - 1e-9) {
        best_cost = cost;
        best = NeckDhwPlan{zc, tpi, items};
      }
    }
  }
  return best;
}
// worth it only when the items fill the machine (the resident-weight kernel cuts its work
// stream-K style and keeps every SM busy on small volumes)
inline bool neck_dhw_profitable(const ConvGeom& g, int ncta = 32) {
  return neck_dhw_supported(g) && neck_dhw_plan(g, ncta).items >= tc_sm_count();
}
inline bool neck_tc_conv_dhw(const Src& s, const NeckTcWeights& w, float* out, const ConvGeom& g,
                             double* stats, int zw_lo, int zw_hi, float zw, cudaStream_t st,
                             std::string* err) {
  NeckParams p{};
  p.wimg = w.dev.p;
  p.out = out;
  p.src = s;
  p.Nx = g.Hi; p.Ny = g.Wi; p.Zi = g.Di; p.Zo = g.Do;
  p.Cin = g.Cin; p.Cout = g.Cout;
  p.zmode = NKZ_S1P1;
  p.tiles_x = (g.Wi + NK_BX - 1) / NK_BX;   // along W
  p.tiles_y = (g.Hi + NK_BY - 1) / NK_BY;   // along H
  const int ncta = 1024 / w.cg;
  p.nsplit = g.Cout / ncta;
  p.ncg = g.Cin / w.cg;
  p.ntiles = p.tiles_x * p.tiles_y;
  p.in_sx = g.Wi; p.in_sy = 1; p.in_sz = (long long)g.Hi * g.Wi;
  p.out_sx = g.Wo; p.out_sy = 1; p.out_sz = (long long)g.Ho * g.Wo;
  const NeckDhwPlan plan = neck_dhw_plan(g, ncta);
  // tests / A-B runs (read per call, like DFM_NECK_TPI)
  const int zc_env = getenv("DFM_NECK_ZC") ? atoi(getenv("DFM_NECK_ZC")) : 0;
  const int tpi_env = getenv("DFM_NECK_ZTPI") ? atoi(getenv("DFM_NECK_ZTPI")) : 0;
  p.ZC = std::min(zc_env > 0 ? std::min(zc_env, NK_ACC_COLS / ncta) : plan.zc, g.Do);
  p.nchunk = (g.Do + p.ZC - 1) / p.ZC;
  // (the window logic of nk_item serves nchunk == 1 too: iz_lo = 0, nzi = Zi)
  p.tpi = std::max(1, std::min(NK_ACC_COLS / (p.ZC * ncta), tpi_env > 0 ? tpi_env : plan.tpi));
  p.n_items = (p.ntiles + p.tpi - 1) / p.tpi * p.nchunk * p.nsplit;
  p.stats = stats;
  p.zw_lo = zw_lo; p.zw_hi = zw_hi; p.zw = zw;
  return neck_launch(p, s.n, w.cg, st, err);
}

}  // namespace dfm
