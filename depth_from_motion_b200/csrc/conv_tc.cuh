// wgmma tensor-core implicit-GEMM 3x3x3 convolution (stride 1, pad 1) for sm_90a.
//
// Formulation (see DESIGN.md "conv_tc"):
//   * activations are channels-last fp32 in HBM; a persistent CTA owns an 8x16 (x,y)
//     output tile and marches along z.  For every input plane the loader warps
//     gather a 10x18 halo brick, apply the fused input transform (GroupNorm /
//     BatchNorm affine, ReLU, residual add -- or the plane-sweep warp for the first
//     layer), split every value into bf16 hi + bf16 lo and store both in shared
//     memory in the K-major *no-swizzle* core-matrix layout
//     [chunk of 8 channels][brick row][16 B].  In that layout a 3x3 in-plane tap is
//     just a 16-byte-granular shift of the descriptor start address and the 8-row
//     group stride (SBO) is the brick row pitch, so ONE brick serves all 9 taps.
//   * the three dz taps are folded into the N dimension: one MMA of input plane z
//     against the weight image rows [kz=2 | kz=1 | kz=0] accumulates into the three
//     accumulator blocks of output planes z-1, z, z+1 at once (N = 3*NCTA), so each
//     input plane is read from HBM/L2 once per tile.
//   * fp32 parity: x*w is evaluated as x_hi*w_hi + x_lo*w_hi + x_hi*w_lo on the bf16
//     tensor pipe with fp32 accumulation (~2^-17 relative), because a single
//     TF32/bf16 pass does not hold the 1e-3 end-to-end tolerance through 22 layers.
//   * weights (hi+lo images of all 27 taps, <= 110.6 KB) stay resident in shared
//     memory for the life of the CTA; layers with Cin*Cout > 1024 are split over
//     output-channel groups of NCTA = 1024/Cin handled by different CTAs.
//   * warp roles: warps 0-7 are two consumer warpgroups (64 accumulator rows each) that issue
//     wgmma.mma_async into register accumulators and store the finished planes (GroupNorm sums
//     on the way); warps 8-15 are loaders (two groups filling alternate stages).  Shared-memory
//     stages are handed over with mbarriers.
//   * modes: stride 1 (TC_S1), stride 2 (TC_S2, x/y parity sub-bricks) and the stride-2
//     transposed conv (TC_T, 4 (px,py) parity classes per output plane); the work of a launch
//     is cut "stream-K" style into equal contiguous (tile column, plane) ranges per CTA.
//   * diagnosis: DFM_TC_ROLE_CYCLES=1 prints per-role busy / wait cycles of every launch,
//     DFM_TC_DEBUG=<bits> disables loader work (1 everything, 8 proxy fence, 16 the
//     loaders' global loads, 32 the loaders' shared-memory stores).
#pragma once
#include <cuda_bf16.h>

#include <algorithm>
#include <cstdlib>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "simt_kernels.cuh"
#include "wgmma.cuh"

namespace dfm {

// ----------------------------------------------------------------------------------
// host side: weight images
// ----------------------------------------------------------------------------------
inline uint16_t bf16_rn_bits(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7F800000u) == 0x7F800000u) return (uint16_t)(u >> 16);
  u += 0x7FFFu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
inline float bf16_bits_to_float(uint16_t b) {
  uint32_t u = (uint32_t)b << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

inline int tc_sm_count() {
  int& cached = per_device<int, 1>();
  if (!cached) cudaDeviceGetAttribute(&cached, cudaDevAttrMultiProcessorCount, cur_device());
  return cached;
}

// ----------------------------------------------------------------------------------
// modes and compile-time geometry
// ----------------------------------------------------------------------------------
enum { TC_S1 = 0, TC_S2 = 1, TC_T = 2 };
constexpr int TC_BX = 8, TC_BY = 16;  // M tile: 8 (x) * 16 (y) = 128 accumulator rows
constexpr int TC_MMA_THREADS = 256;   // two warpgroups: MMA issue + epilogue, 64 rows each
constexpr int TC_LOAD_THREADS = 256;  // 2 groups x 4 warps
constexpr int TC_THREADS = TC_MMA_THREADS + TC_LOAD_THREADS;  // 16 warps: 128 registers/thread
constexpr int TC_MAXOPS = 9, TC_MAXBLK = 48;
constexpr int TC_ZERO_TAP = 255;  // TcBlk::tap of an all-zero padding block

template <int MODE>
struct TcMode;
template <>
struct TcMode<TC_S1> {  // out(x,y,z) <- in(x+dx-1, y+dy-1, z+dz-1)
  static constexpr int PXB = 10, PYB = 18, PITCH = 10, ROWS = 186, CG = 32, NSTAGE = 4;
  static constexpr int SLOT_BLOCKS = 1;
  __host__ __device__ static int zo_of(int zi, int dz) { return zi + dz; }
  __host__ __device__ static int zi_first(int zo) { return zo - 1; }
  __host__ __device__ static int zi_last(int zo) { return zo + 1; }
  __host__ __device__ static int ptype(int) { return 0; }
};
template <>
struct TcMode<TC_S2> {  // out(x,y,z) <- in(2x+dx-1, 2y+dy-1, 2z+dz-1); x/y parity arrays
  static constexpr int PXB = 17, PYB = 33, PITCH = 9, ROWS = 620, CG = 16, NSTAGE = 3;
  static constexpr int SLOT_BLOCKS = 1;
  __host__ __device__ static int zo_of(int zi, int dz) { return (zi >> 1) + dz; }
  __host__ __device__ static int zi_first(int zo) { return 2 * zo - 1; }
  __host__ __device__ static int zi_last(int zo) { return 2 * zo + 1; }
  __host__ __device__ static int ptype(int zi) { return zi & 1; }
};
template <>
struct TcMode<TC_T> {  // ConvTranspose3d(k3,s2,p1,op1): out(2m+p) <- in(m + s), 8 parity classes
  static constexpr int PXB = 9, PYB = 17, PITCH = 9, ROWS = 154, CG = 32, NSTAGE = 4;
  static constexpr int SLOT_BLOCKS = 4;  // 4 (px,py) classes per output plane
  __host__ __device__ static int zo_of(int zi, int dz) { return 2 * zi + dz; }
  __host__ __device__ static int zi_first(int zo) { return zo >> 1; }
  __host__ __device__ static int zi_last(int zo) { return (zo + 1) >> 1; }
  __host__ __device__ static int ptype(int) { return 0; }
};

inline int tc_mode_of(const ConvGeom& g) {
  if (g.transposed) return TC_T;
  if (g.sd == 1 && g.sh == 1 && g.sw == 1 && g.pd == 1 && g.ph == 1 && g.pw == 1) return TC_S1;
  if (g.sd == 2 && g.sh == 2 && g.sw == 2 && g.pd == 1 && g.ph == 1 && g.pw == 1 &&
      g.Di % 2 == 0 && g.Hi % 2 == 0 && g.Wi % 2 == 0)
    return TC_S2;
  return -1;
}
inline bool tc_supported(int Cin, int Cout, int /*transposed*/) {
  if (Cin != 32 && Cin != 64) return false;
  const int ncta = 1024 / Cin;
  return Cout % ncta == 0 && Cout <= 64;
}
inline bool tc_geom_supported(const ConvGeom& g) { return tc_mode_of(g) >= 0; }

// One MMA "op" = one A view (tap shift of the brick) against a weight image whose
// NCTA-row blocks land in consecutive accumulator column blocks.  The host lays the weight
// images out from this op list; the kernel issues the same sequence from compile-time constants.
struct TcOp {
  uint32_t a_off;   // byte offset of the A view inside a stage (hi array)
  uint32_t b_off;   // byte offset of this op's weight image (hi half) in smem
  uint32_t b_lbo;   // bytes between 8-channel chunks of the weight image
  uint16_t blk0, blk1;
  // static decomposition into MMAs when every output plane is live:
  // run = nblk | first block << 4 | lin0 << 10, lin = (dz+1) * SLOT_BLOCKS + colblk of the
  // first block; a run is a range of consecutive lin values (split at issue time only where
  // the accumulator slot ring wraps between two planes)
  uint32_t nruns;
  uint32_t runs[3];
};
struct TcBlk {
  int8_t dz;        // output plane relative to zo_of(zi, 0)
  uint8_t colblk;   // column block inside the accumulator slot
  uint8_t tap;      // 27-tap index (kz*9 + ky*3 + kx) of the weights in this block
  uint8_t pad;
};
struct TcProgram {
  int nops;
  uint32_t need;    // mask of (dz+1) values this plane type writes
  TcOp ops[TC_MAXOPS];
  TcBlk blks[TC_MAXBLK];
};

// host: the op list of one input-plane type
template <int MODE>
inline void tc_build_program(int ptype, int Cin, int ncta, uint32_t* w_cursor, TcProgram* pr) {
  using M = TcMode<MODE>;
  pr->nops = 0;
  pr->need = 0;
  int nb = 0;
  auto add_op = [&](int a_rows, std::vector<TcBlk> blks) {
    TcOp& op = pr->ops[pr->nops++];
    op.a_off = (uint32_t)a_rows * 16;
    op.b_off = *w_cursor;
    op.b_lbo = (uint32_t)blks.size() * ncta * 16;
    op.blk0 = (uint16_t)nb;
    for (TcBlk b : blks) pr->blks[nb++] = b;
    op.blk1 = (uint16_t)nb;
    *w_cursor += (uint32_t)(Cin / 8) * op.b_lbo;
    // static runs: maximal groups of blocks that are consecutive in (plane, colblk) order
    op.nruns = 0;
    size_t i = 0;
    while (i < blks.size()) {
      size_t e = i + 1;
      auto lin = [&](const TcBlk& b) { return (b.dz + 1) * M::SLOT_BLOCKS + b.colblk; };
      while (e < blks.size() && lin(blks[e]) == lin(blks[i]) + (int)(e - i)) ++e;
      const int nblk = (int)(e - i);
      op.runs[op.nruns++] = (uint32_t)nblk | ((uint32_t)i << 4) | ((uint32_t)lin(blks[i]) << 10);
      for (size_t k = i; k < e; ++k) pr->need |= 1u << (blks[k].dz + 1);
      i = e;
    }
  };
  if (MODE == TC_S1) {
    for (int t = 0; t < 9; ++t) {
      const int dy = t / 3, dx = t % 3;
      // planes z-1, z, z+1 receive kz = 2, 1, 0
      add_op(dy * M::PITCH + dx, {TcBlk{-1, 0, (uint8_t)(18 + t), 0}, TcBlk{0, 0, (uint8_t)(9 + t), 0},
                                  TcBlk{1, 0, (uint8_t)t, 0}});
    }
  } else if (MODE == TC_S2) {
    for (int t = 0; t < 9; ++t) {
      const int dy = t / 3, dx = t % 3;
      const int a_rows = (((dx & 1) * 2 + (dy & 1)) * 17 + (dy >> 1)) * M::PITCH + (dx >> 1);
      if (ptype == 0)  // zi = 2q: kz = 1 -> zo = q
        add_op(a_rows, {TcBlk{0, 0, (uint8_t)(9 + t), 0}});
      else             // zi = 2q+1: kz = 2 -> zo = q, kz = 0 -> zo = q+1
        add_op(a_rows, {TcBlk{0, 0, (uint8_t)(18 + t), 0}, TcBlk{1, 0, (uint8_t)t, 0}});
    }
  } else {
    // class order inside a slot: (px,py) = (0,0), (1,0), (1,1), (0,1) so that every
    // shift's class set is a contiguous column range
    const int cls_px[4] = {0, 1, 1, 0}, cls_py[4] = {0, 0, 1, 1};
    for (int sh = 0; sh < 4; ++sh) {
      const int sx = sh & 1, sy = sh >> 1;
      std::vector<TcBlk> blks;
      for (int dz = -1; dz <= 1; ++dz) {
        // out plane 2zi+dz: dz=-1 uses kz=0 (this plane is its m+1 input), 0 -> kz=1, +1 -> kz=2
        const int kz = dz + 1;
        for (int c = 0; c < 4; ++c) {
          const int px = cls_px[c], py = cls_py[c];
          // o = 2i - 1 + k: p=0 -> k=1,s=0 ; p=1 -> (k=2,s=0) or (k=0,s=1)
          int kx = -1, ky = -1;
          if (px == 0) { if (!sx) kx = 1; } else kx = sx ? 0 : 2;
          if (py == 0) { if (!sy) ky = 1; } else ky = sy ? 0 : 2;
          const bool real = kx >= 0 && ky >= 0;
          blks.push_back(TcBlk{(int8_t)dz, (uint8_t)c,
                               (uint8_t)(real ? kz * 9 + ky * 3 + kx : TC_ZERO_TAP), 0});
        }
      }
      // The x-only and y-only shifts touch two classes per plane: instead of three small
      // N = 2*NCTA MMAs keep the all-zero blocks between the first and the last real one, so that
      // one N = 10*NCTA MMA spans the three planes (the kernel's MMA sequence stays static).  The
      // diagonal shift touches one class per plane; padding it would not fit in shared memory
      // next to four stages, so it stays three small MMAs.
      if (sh == 3) {
        std::vector<TcBlk> real;
        for (const TcBlk& b : blks)
          if (b.tap != TC_ZERO_TAP) real.push_back(b);
        blks = real;
      } else {
        while (!blks.empty() && blks.front().tap == TC_ZERO_TAP) blks.erase(blks.begin());
        while (!blks.empty() && blks.back().tap == TC_ZERO_TAP) blks.pop_back();
      }
      add_op(sy * M::PITCH + sx, blks);
    }
  }
}

struct TcWeights {
  DevArray<uint8_t> dev;  // [nsplit][image bytes]
  int Cin = 0, Cout = 0, ncta = 0, nsplit = 0, mode = -1, kslice = 0;
  int cluster = 1;  // > 1: the nsplit output-channel groups share bricks as one cluster (32 -> 64)
  uint32_t image_bytes = 0, hi_bytes = 0;
  TcProgram prog[2];

  bool ready() const { return dev.p != nullptr; }
  void release() { dev.release(); }
  // packed: [27][Cin][Cout] fp32 (tap = kz*9 + ky*3 + kx; transposed weights are
  // already in "o = 2i - 1 + k" orientation)
  // ks (stride 2 only): the CTA groups split the *input* channels (16 per group) and each covers
  // all output channels; partial sums meet in global memory (see conv_tc_kernel, KSLICE).
  template <int MODE>
  bool build_mode(const float* packed, int cin, int cout, std::string* err, bool ks = false) {
    release();
    mode = MODE;
    Cin = cin;
    Cout = cout;
    kslice = ks ? 1 : 0;
    cluster = 1;
    const int cin_img = ks ? 16 : cin;  // input channels of one weight image
    ncta = ks ? cout : 1024 / cin;
    nsplit = ks ? cin / 16 : cout / ncta;
    uint32_t cursor = 0;
    const int ntypes = MODE == TC_S2 ? 2 : 1;
    for (int t = 0; t < ntypes; ++t) tc_build_program<MODE>(t, cin_img, ncta, &cursor, &prog[t]);
    hi_bytes = cursor;
    image_bytes = 2 * hi_bytes;
    std::vector<uint16_t> img((size_t)nsplit * image_bytes / 2);
    const int kch = cin_img / 8;
    for (int s = 0; s < nsplit; ++s)
      for (int t = 0; t < ntypes; ++t)
        for (int o = 0; o < prog[t].nops; ++o) {
          const TcOp& op = prog[t].ops[o];
          const int nblk = op.blk1 - op.blk0;
          for (int kc = 0; kc < kch; ++kc)
            for (int b = 0; b < nblk; ++b)
              for (int j = 0; j < ncta; ++j)
                for (int e = 0; e < 8; ++e) {
                  const int tap = prog[t].blks[op.blk0 + b].tap;
                  if (tap == TC_ZERO_TAP) continue;  // img is zero-initialised
                  const int ci = kc * 8 + e + (ks ? s * 16 : 0), co = ks ? j : s * ncta + j;
                  const float w = packed[((size_t)tap * cin + ci) * cout + co];
                  const uint16_t hi = bf16_rn_bits(w);
                  const uint16_t lo = bf16_rn_bits(w - bf16_bits_to_float(hi));
                  const size_t off = (size_t)s * image_bytes / 2 + op.b_off / 2 +
                                     ((size_t)kc * nblk * ncta + (size_t)b * ncta + j) * 8 + e;
                  img[off] = hi;
                  img[off + hi_bytes / 2] = lo;
                }
        }
    if (dev.upload(reinterpret_cast<const uint8_t*>(img.data()), img.size() * 2) != cudaSuccess) {
      if (err) *err = "TcWeights: device upload failed";
      release();
      return false;
    }
    return true;
  }
  bool build(const float* packed, int cin, int cout, int m, std::string* err) {
    if (m == TC_S1) return build_mode<TC_S1>(packed, cin, cout, err);
    if (m == TC_S2) {
      // stride-2 layers are loader-bound: with independent output-channel groups every group
      // re-loads and re-transforms the whole input (2x for 32->64, 4x for 64->64).
      // 32 -> 64: the two groups run as one thread-block cluster and share every brick
      // (conv_tc_kernel, CL), so the input is read once and no partial sums exist.
      // 64 -> 64: input-channel slices with partial outputs in global memory and a reduce pass.
      // Four clustered groups of 16 outputs issue N = 16 / 32 MMAs that each re-read the whole
      // 64-channel brick from shared memory: H100 SXM, KITTI D = 112 stereo conv3, 0.570 ms
      // clustered vs 0.220 ms sliced.
      // Other shapes keep independent output-channel groups.
      const bool ks = cin == 64 && cout == 64;
      if (!build_mode<TC_S2>(packed, cin, cout, err, ks)) return false;
      if (cin == 32 && cout == 64) cluster = nsplit;  // 2
      return true;
    }
    return build_mode<TC_T>(packed, cin, cout, err);
  }
};

// ----------------------------------------------------------------------------------
// device helpers
// ----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// bounded wait: a protocol bug must not hang the GPU; on timeout flag the error.
// CL: the phase is completed by arrivals of other CTAs of the cluster (acquire at cluster scope)
template <bool CL = false>
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int* err) {
  for (int it = 0; it < (1 << 26); ++it) {
    uint32_t ok;
    if constexpr (CL)
      asm volatile(
          "{\n\t.reg .pred q;\n\t"
          "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 q, [%1], %2;\n\t"
          "selp.u32 %0, 1, 0, q;\n\t}\n"
          : "=r"(ok)
          : "r"(bar), "r"(parity)
          : "memory");
    else
      asm volatile(
          "{\n\t.reg .pred q;\n\t"
          "mbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2;\n\t"
          "selp.u32 %0, 1, 0, q;\n\t}\n"
          : "=r"(ok)
          : "r"(bar), "r"(parity)
          : "memory");
    if (ok) return;
  }
  // err is mapped host memory (TcErrFlag)
  *reinterpret_cast<volatile int*>(err) = 1;
  __threadfence_system();
}
template <bool CL = false>
__device__ __forceinline__ void mbar_wait_timed(uint32_t bar, uint32_t parity, int* err,
                                                unsigned long long& acc, bool timed) {
  if (!timed) {
    mbar_wait<CL>(bar, parity, err);
    return;
  }
  const long long t0 = clock64();
  mbar_wait<CL>(bar, parity, err);
  acc += (unsigned long long)(clock64() - t0);
}
// distributed shared memory: the address of the same shared-memory location in CTA `rank` of
// the cluster, a release-arrive on an mbarrier there, a 16-byte store there
__device__ __forceinline__ uint32_t mapa_u32(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_bar) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_bar)
               : "memory");
}
__device__ __forceinline__ void st_cluster_v4(uint32_t addr, uint4 v) {
  asm volatile("st.shared::cluster.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;"
               ::: "memory");
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}
// bump the 14-bit start-address field of a descriptor (low word only: no carry into the
// LBO field as long as the operand stays inside the 256 KB shared window)
__device__ __forceinline__ void desc_add(uint64_t& d, uint32_t inc16) {
  asm("{\n\t.reg .b32 lo, hi;\n\tmov.b64 {lo, hi}, %0;\n\tadd.u32 lo, lo, %1;\n\t"
      "mov.b64 %0, {lo, hi};\n\t}\n"
      : "+l"(d)
      : "r"(inc16));
}
__device__ __forceinline__ uint64_t pack64(uint32_t lo, uint32_t hi) {
  return ((uint64_t)hi << 32) | lo;
}
__device__ __forceinline__ void split8(const float v[8], uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __nv_bfloat162 hh = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    const float2 hf = __bfloat1622float2(hh);
    const __nv_bfloat162 ll = __floats2bfloat162_rn(v[2 * i] - hf.x, v[2 * i + 1] - hf.y);
    h[i] = *reinterpret_cast<const uint32_t*>(&hh);
    l[i] = *reinterpret_cast<const uint32_t*>(&ll);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}
__device__ __forceinline__ void split_store(const float v[8], uint8_t* hi_dst, uint8_t* lo_dst) {
  uint4 h, l;
  split8(v, h, l);
  *reinterpret_cast<uint4*>(hi_dst) = h;
  *reinterpret_cast<uint4*>(lo_dst) = l;
}

// ----------------------------------------------------------------------------------
// loaders: 8 consecutive channels [c0, c0+8) of input voxel (z, y, x), in bounds.
// issue() only starts the global loads (so several items are in flight per thread),
// finish() applies the fused transform.
// ----------------------------------------------------------------------------------
// 16-byte activation load of the loader warps (experiment hook: DFM_LD_VARIANT)
#ifndef DFM_LD_VARIANT
#define DFM_LD_VARIANT 0
#endif
__device__ __forceinline__ float4 ld_act(const float4* p) {
#if DFM_LD_VARIANT == 1
  return __ldcg(p);
#elif DFM_LD_VARIANT == 2
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::256B.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
#elif DFM_LD_VARIANT == 3
  return __ldcs(p);
#elif DFM_LD_VARIANT == 4
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
#else
  return __ldg(p);
#endif
}

template <int NT>  // number of input terms (compile-time: sizes the in-flight registers)
struct SrcLoader8 {
  Src s;
  int C, H, W;
  // items of a thread in flight at once: at most 12 float4 (48 registers) of raw loads
  static constexpr int BATCH = 6 / NT;
  struct Raw {
    float4 a[NT][2];
  };
  __device__ __forceinline__ void issue(int z, int y, int x, int c0, Raw& r) const {
    const long long inpl = ((long long)y * W + x) * C + c0, plane = (long long)H * W * C;
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const float* px = s.t[t].x + term_plane(s.t[t], z) * plane + inpl;
      r.a[t][0] = ld_act(reinterpret_cast<const float4*>(px));
      r.a[t][1] = ld_act(reinterpret_cast<const float4*>(px) + 1);
    }
  }
  __device__ __forceinline__ void finish(const Raw& r, int c0, float v[8]) const {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = 0.f;
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      {
        float u[8] = {r.a[t][0].x, r.a[t][0].y, r.a[t][0].z, r.a[t][0].w,
                      r.a[t][1].x, r.a[t][1].y, r.a[t][1].z, r.a[t][1].w};
        if (s.t[t].scale) {
          const float4 s0 = __ldg(reinterpret_cast<const float4*>(s.t[t].scale + c0));
          const float4 s1 = __ldg(reinterpret_cast<const float4*>(s.t[t].scale + c0) + 1);
          const float4 h0 = __ldg(reinterpret_cast<const float4*>(s.t[t].shift + c0));
          const float4 h1 = __ldg(reinterpret_cast<const float4*>(s.t[t].shift + c0) + 1);
          const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
          const float sh[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
#pragma unroll
          for (int i = 0; i < 8; ++i) u[i] = fmaf(u[i], sc[i], sh[i]);
        }
        if (s.t[t].relu) {
#pragma unroll
          for (int i = 0; i < 8; ++i) u[i] = fmaxf(u[i], 0.f);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] += u[i];
      }
    }
    if (s.outer_relu) {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = fmaxf(v[i], 0.f);
    }
  }
};

struct WarpLoader8 {
  WarpLoader w;
  static constexpr int BATCH = 1;
  struct Raw {
    float4 t[4][2];
    float wt[4];
  };
  __device__ __forceinline__ void issue(int z, int y, int x, int c0, Raw& r) const {
    c0 += w.first;
    if (c0 < w.C) {  // cur half: exact stride-lattice fetch, single tap of weight 1
      const float* p = w.cur + ((long long)(y * w.g.step) * w.g.Wf + x * w.g.step) * w.C + c0;
      r.t[0][0] = __ldg(reinterpret_cast<const float4*>(p));
      r.t[0][1] = __ldg(reinterpret_cast<const float4*>(p) + 1);
      r.wt[0] = 1.f;
      r.wt[1] = r.wt[2] = r.wt[3] = 0.f;
      return;
    }
    c0 -= w.C;
    float fx, fy;
    warp_coord(w.g, x, y, __ldg(w.depths + z), fx, fy);
    const Taps t = bilinear_taps(fx, fy, w.g.Hf, w.g.Wf);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      r.wt[k] = t.w[k];
      if (t.w[k] != 0.f) {
        const float* p = w.prev + (long long)t.off[k] * w.C + c0;
        r.t[k][0] = __ldg(reinterpret_cast<const float4*>(p));
        r.t[k][1] = __ldg(reinterpret_cast<const float4*>(p) + 1);
      }
    }
  }
  __device__ __forceinline__ void finish(const Raw& r, int, float v[8]) const {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (r.wt[k] != 0.f) {
        v[0] = fmaf(r.wt[k], r.t[k][0].x, v[0]); v[1] = fmaf(r.wt[k], r.t[k][0].y, v[1]);
        v[2] = fmaf(r.wt[k], r.t[k][0].z, v[2]); v[3] = fmaf(r.wt[k], r.t[k][0].w, v[3]);
        v[4] = fmaf(r.wt[k], r.t[k][1].x, v[4]); v[5] = fmaf(r.wt[k], r.t[k][1].y, v[5]);
        v[6] = fmaf(r.wt[k], r.t[k][1].z, v[6]); v[7] = fmaf(r.wt[k], r.t[k][1].w, v[7]);
      }
    }
  }
};

struct TcParams {
  const uint8_t* wimg;
  float* out;
  double* stats;        // [Cout][2] sum / sum of squares of the raw conv output, or null
  int Di, Hi, Wi;       // input volume
  int Do, Ho, Wo, Cout; // output volume
  int Mx, My;           // extent of the M grid (output grid; input grid for transposed)
  int tiles_x, tiles_y, nsplit;
  int z_unit;  // granularity of a z cut in output planes (2 for the transposed conv)
  uint32_t w_bytes, w_hi_bytes;
  int* err;
  unsigned long long* role_cycles;  // optional [grid][8] role wait/busy cycle counters
  const float* addend;  // optional [3][Ho][Wo][Cout] added to the output by z class (0, interior,
                        // Do-1): the z-invariant cur-frame contribution of the first layer
  // statistics weight of output planes [zw_lo, zw_hi): the planes that stand for the
  // (longer) z-invariant interior of a shortened volume
  int zw_lo, zw_hi;
  float zw;
  long long slice_stride;  // K-slice variant: elements between the slices' partial outputs
  int store1;  // epilogue stores only output channel 0, densely ([V] floats): the Cout=1 conv
  int dbg;  // diagnosis only (DFM_TC_DEBUG): 1 loaders skip work, 8 loaders skip the proxy
            // fence, 16 / 32 loaders skip their global loads / shared-memory stores
};

struct TcItem {
  int x0, y0, split, z_lo, z_hi;
};
// Work partition ("stream-K" over z): the (tile column, output plane) space of one
// output-channel split is linearised column-major and cut into gridDim.x / nsplit equal
// contiguous ranges, one per CTA; a CTA walks its range as pieces that end at column
// boundaries.  Every CTA gets the same number of planes (+-1 unit), the only overhead is
// the halo input planes at the 2-3 piece ends.  All roles of a CTA derive the same piece
// list from blockIdx alone.
struct TcWalk {
  long long cur, end;  // in units of `unit` output planes
  int split;
};
__device__ __forceinline__ TcWalk tc_walk_begin(const TcParams& p) {
  TcWalk w;
  const int per_split = gridDim.x / p.nsplit;
  w.split = blockIdx.x % p.nsplit;
  const int r = blockIdx.x / p.nsplit;
  const long long units_col = p.Do / p.z_unit;
  const long long total = (long long)p.tiles_x * p.tiles_y * units_col;
  w.cur = total * r / per_split;
  w.end = total * (r + 1) / per_split;
  return w;
}
__device__ __forceinline__ bool tc_walk_next(const TcParams& p, TcWalk& w, TcItem& it) {
  if (w.cur >= w.end) return false;
  const long long units_col = p.Do / p.z_unit;
  const int col = (int)(w.cur / units_col);
  const long long u0 = w.cur % units_col;
  const long long u1 = min(units_col, u0 + (w.end - w.cur));
  it.split = w.split;
  it.x0 = (col % p.tiles_x) * TC_BX;
  it.y0 = (col / p.tiles_x) * TC_BY;
  it.z_lo = (int)u0 * p.z_unit;
  it.z_hi = (int)u1 * p.z_unit;
  w.cur += u1 - u0;
  return true;
}

// Accumulator window of the consumer warpgroups: the output planes that the current input plane
// zi feeds, kept in registers.  Plane j of the window is output plane base(zi) + j; every block of
// NCTA columns of a plane is one (px,py) class of the transposed conv (one block otherwise).
template <int MODE>
struct TcWin;
template <>
struct TcWin<TC_S1> {  // zi feeds zi-1 (kz=2), zi (kz=1), zi+1 (kz=0)
  static constexpr int NPL = 3;
  __device__ static int base(int zi) { return zi - 1; }
};
template <>
struct TcWin<TC_S2> {  // zi = 2q feeds q (kz=1); zi = 2q+1 feeds q (kz=2), q+1 (kz=0)
  static constexpr int NPL = 2;
  __device__ static int base(int zi) { return zi >> 1; }
};
template <>
struct TcWin<TC_T> {  // zi feeds 2zi-1 (kz=0), 2zi (kz=1), 2zi+1 (kz=2)
  static constexpr int NPL = 3;
  __device__ static int base(int zi) { return 2 * zi - 1; }
};

// ----------------------------------------------------------------------------------
// the kernel
// ----------------------------------------------------------------------------------
// CL > 1: cluster-shared bricks.  The CL output-channel groups of one work range run as one
// thread-block cluster (group = cluster rank); the loaders of each CTA gather and transform brick
// rows rank, rank + CL, ... and store them into the stage of EVERY CTA of the cluster (distributed
// shared memory), so each input value is read from HBM and transformed once, and every CTA's
// accumulators still hold complete sums for its own output channels.  A stage is full when the
// loader warps of all CL CTAs have arrived on it, and free when the consumer warps of all CL CTAs
// have released it (remote mbarrier arrivals in both directions).
template <int MODE, int CIN, int NCTA, class Loader, int CL = 1>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_kernel(const __grid_constant__ TcParams p,
                                                                 const __grid_constant__ Loader ld) {
  using M = TcMode<MODE>;
  using Win = TcWin<MODE>;
  constexpr bool CLU = CL > 1;
  static_assert(!CLU || (MODE == TC_S2 && CIN != 16),
                "cluster-shared bricks serve the stride-2 output-channel split");
  constexpr int CG = M::CG < CIN ? M::CG : CIN;  // channels per stage
  constexpr int NCH = CG / 8;                    // 16-byte channel chunks per stage
  constexpr int NCG = CIN / CG;                  // pipeline stages per input plane
  // stage layout: [hi|lo][chunk][ROWS rows] with the four x/y parity classes of a stride-2
  // brick inside a chunk's rows
  constexpr uint32_t S2_CLS16 = 17 * M::PITCH;  // stride-2 class stride, 16-byte rows
  constexpr uint32_t A_LBO = M::ROWS * 16;
  constexpr uint32_t A_SBO = M::PITCH * 16;
  constexpr uint32_t A_HL = NCH * M::ROWS * 16;  // hi -> lo offset
  constexpr uint32_t STAGE_BYTES = 2 * A_HL;
  constexpr uint32_t B_SBO = 128;
  // K-slice variant (stride 2, instantiated with CIN = 16 = the channels this CTA group loads,
  // NCTA = all output channels): every slice stores its partial sums; kslice_reduce_kernel adds
  // them in slice order (deterministic) and takes the GroupNorm statistics on the way
  constexpr bool KSLICE = CIN == 16;
  // brick rows this CTA loads (every CL-th, from its cluster rank)
  constexpr int ROWS_CTA = (M::PYB + CL - 1) / CL;
  // two loader groups (even / odd loader warps) fill alternate stages: while one group
  // waits for its global loads the other transforms and stores -> two stages in flight
  constexpr int LGROUPS = 2;
  constexpr int LG_THREADS = TC_LOAD_THREADS / LGROUPS;
  constexpr int NITEM = (ROWS_CTA * M::PXB * NCH + LG_THREADS - 1) / LG_THREADS;
  constexpr int PCOLS = M::SLOT_BLOCKS * NCTA;        // accumulator columns per output plane
  constexpr int NACC = Win::NPL * PCOLS / 2;          // accumulator registers per thread

  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* w_s = smem;
  uint8_t* a_s = smem + p.w_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(a_s + M::NSTAGE * STAGE_BYTES);

  const int tid = threadIdx.x, lane = tid & 31;
  // shfl broadcast: tells the compiler the warp index is warp-uniform, so the role
  // branches below are convergent
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const uint32_t bar0 = smem_u32(bars);
  auto full_a = [&](int s) { return bar0 + 8u * s; };
  auto empty_a = [&](int s) { return bar0 + 8u * (M::NSTAGE + s); };
  const uint32_t w_bar = bar0 + 8u * (2 * M::NSTAGE);
  constexpr int LOAD_WARP0 = TC_MMA_THREADS / 32;
  // cluster rank (a 1-D grid launched with cluster dimension (CL, 1, 1)) = output-channel group
  const int rank = CLU ? (int)(blockIdx.x % CL) : 0;

  if (tid == 0) {
    for (int s = 0; s < M::NSTAGE; ++s) {
      // one arrival per loader warp of the group (of every CTA of the cluster)
      mbar_init(full_a(s), CL * LG_THREADS / 32);
      mbar_init(empty_a(s), CL * TC_MMA_THREADS / 32);  // one arrival per consumer warp
    }
    mbar_init(w_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    // Resident weights of this CTA's output-channel group: bulk async copies (TMA engine)
    // that land while the loaders fill the first stages; only the consumers wait for them.
    // (A thread-copy loop here cost every launch ~10 us of serialised load latency.)
    const int split = blockIdx.x % p.nsplit;
    const uint8_t* src = p.wimg + (size_t)split * p.w_bytes;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(w_bar),
                 "r"(p.w_bytes)
                 : "memory");
    constexpr uint32_t CHUNK = 32768;
    for (uint32_t off = 0; off < p.w_bytes; off += CHUNK) {
      const uint32_t n = min(CHUNK, p.w_bytes - off);
      asm volatile(
          "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
          ::"r"(smem_u32(w_s + off)), "l"(src + off), "r"(n), "r"(w_bar)
          : "memory");
    }
  }
  // (cluster: no peer may arrive on or store into this CTA's shared memory before its barriers
  // are initialised)
  if constexpr (CLU) cluster_sync_all();
  else __syncthreads();

  if (warp >= LOAD_WARP0) {
    // ============================ loaders ============================
    const int lw = warp - LOAD_WARP0;
    const int lgrp = lw & (LGROUPS - 1);
    const int lt = (lw / LGROUPS) * 32 + lane;  // thread index inside the group
    const int chunk = lt % NCH;
    uint32_t stage_ctr = 0;
    const bool timed = p.role_cycles != nullptr && lw == 0 && lane == 0;
    unsigned long long t_wait_e = 0;
    const long long t_begin = clock64();
    // stage base of every CTA of the cluster, in the cluster's shared window
    uint32_t peer_a[CL];
#pragma unroll
    for (int q = 0; q < CL; ++q) peer_a[q] = CLU ? mapa_u32(smem_u32(a_s), q) : 0u;
    const int nitems = (M::PYB - rank + CL - 1) / CL * M::PXB * NCH;
    TcWalk walk = tc_walk_begin(p);
    TcItem it;
    while (tc_walk_next(p, walk, it)) {
      int soff[NITEM], gx[NITEM], gy[NITEM];
      bool inb[NITEM], live[NITEM];
#pragma unroll
      for (int k = 0; k < NITEM; ++k) {
        const int i = lt + k * LG_THREADS;
        live[k] = i < nitems;
        const int pos = i / NCH;
        const int bx = pos % M::PXB, by = pos / M::PXB * CL + rank;
        int row;
        if (MODE == TC_S1) {
          gx[k] = it.x0 - 1 + bx;
          gy[k] = it.y0 - 1 + by;
          row = by * M::PITCH + bx;
        } else if (MODE == TC_S2) {
          gx[k] = 2 * it.x0 - 1 + bx;
          gy[k] = 2 * it.y0 - 1 + by;
          row = (((bx & 1) * 2 + (by & 1)) * 17 + (by >> 1)) * M::PITCH + (bx >> 1);
        } else {
          gx[k] = it.x0 + bx;
          gy[k] = it.y0 + by;
          row = by * M::PITCH + bx;
        }
        inb[k] = live[k] && gx[k] >= 0 && gx[k] < p.Wi && gy[k] >= 0 && gy[k] < p.Hi;
        soff[k] = (chunk * M::ROWS + row) * 16;
      }
      const int zi0 = max(M::zi_first(it.z_lo), 0);
      const int zi1 = min(M::zi_last(it.z_hi - 1), p.Di - 1);
      for (int zi = zi0; zi <= zi1; ++zi) {
#pragma unroll 1
        for (int cg = 0; cg < NCG; ++cg, ++stage_ctr) {
          if ((int)(stage_ctr & (LGROUPS - 1)) != lgrp) continue;
          const int s = stage_ctr % M::NSTAGE;
          mbar_wait_timed<CLU>(empty_a(s), ((stage_ctr / M::NSTAGE) & 1) ^ 1, p.err, t_wait_e,
                               timed);
          uint8_t* st = a_s + s * STAGE_BYTES;
          const int c0 = cg * CG + chunk * 8 + (KSLICE ? it.split * CIN : 0);
          constexpr int LB = Loader::BATCH < NITEM ? Loader::BATCH : NITEM;
          if (!(p.dbg & 1))
#pragma unroll
          for (int k0 = 0; k0 < NITEM; k0 += LB) {
            typename Loader::Raw raw[LB];
#pragma unroll
            for (int b = 0; b < LB; ++b)
              if (k0 + b < NITEM && inb[k0 + b] && !(p.dbg & 16))
                ld.issue(zi, gy[k0 + b], gx[k0 + b], c0, raw[b]);
#pragma unroll
            for (int b = 0; b < LB; ++b) {
              if (k0 + b < NITEM && live[k0 + b]) {
                float v[8];
                if (inb[k0 + b]) {
                  ld.finish(raw[b], c0, v);
                } else {
#pragma unroll
                  for (int i = 0; i < 8; ++i) v[i] = 0.f;
                }
                if (p.dbg & 32) {
                  if (v[0] + v[1] + v[2] + v[3] + v[4] + v[5] + v[6] + v[7] == 1.2345f) st[0] = 1;
                } else if constexpr (CLU) {
                  uint4 h, l;
                  split8(v, h, l);
                  const uint32_t off = (uint32_t)(s * STAGE_BYTES + soff[k0 + b]);
#pragma unroll
                  for (int q = 0; q < CL; ++q) {
                    st_cluster_v4(peer_a[q] + off, h);
                    st_cluster_v4(peer_a[q] + off + A_HL, l);
                  }
                } else {
                  split_store(v, st + soff[k0 + b], st + A_HL + soff[k0 + b]);
                }
              }
            }
          }
          if (!(p.dbg & 8)) {
            if constexpr (CLU) asm volatile("fence.proxy.async.shared::cluster;" ::: "memory");
            else asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          }
          __syncwarp();
          if (lane == 0) {
            if constexpr (CLU) {
#pragma unroll
              for (int q = 0; q < CL; ++q) mbar_arrive_cluster(mapa_u32(full_a(s), q));
            } else {
              mbar_arrive(full_a(s));
            }
          }
        }
      }
    }
    if (timed) {
      unsigned long long* rc = p.role_cycles + (size_t)blockIdx.x * 8;
      rc[3] = (unsigned long long)(clock64() - t_begin);
      rc[4] = t_wait_e;
    }
  } else {
    // ======================= consumers: two MMA + epilogue warpgroups =======================
    // Warpgroup wg owns accumulator rows [64*wg, 64*wg + 64) of the 128-row tile, i.e. tile
    // rows y = 8*wg .. 8*wg + 7 (8 brick rows further into every A view).  Its accumulators are
    // the window of output planes the current input plane feeds (TcWin): all window planes are
    // computed for every input plane, planes outside the item's range are simply never stored,
    // so the MMA sequence of a plane type is static.  A plane leaves the window (is stored,
    // then its registers are reused) once the last input plane that feeds it is done.
    const int wg = warp >> 2, wq = warp & 3;
    const bool timed = p.role_cycles != nullptr && tid == 0;
    unsigned long long t_wait_a = 0;
    const long long t_begin = clock64();
    mbar_wait(w_bar, 0u, p.err);  // weight image has landed
    const uint32_t w_base = smem_u32(w_s), a_base = smem_u32(a_s);
    constexpr uint32_t A_LBO16 = A_LBO >> 4, A_HL16 = A_HL >> 4;
    const uint32_t a_desc_hi = A_SBO >> 4;
    const uint32_t b_desc_hi = B_SBO >> 4;
    const uint32_t w_hi16 = p.w_hi_bytes >> 4;
    const uint32_t a_wg16 = (uint32_t)wg * 8u * (A_SBO >> 4);  // this warpgroup's first A row

    float acc[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    constexpr int NST = KSLICE ? 1 : NCTA / 4;  // channels of this thread (the K-slice variant keeps no statistics)
    float ssum[NST], ssq[NST];
#pragma unroll
    for (int i = 0; i < NST; ++i) ssum[i] = ssq[i] = 0.f;

    // rows of this thread: tile (x, y) = (lane / 4, 8*wg + 2*wq + r), r = 0, 1
    const int xr = lane >> 2, cq = lane & 3;
    auto flush_stats = [&](int split) {
      if (KSLICE || !p.stats) return;
#pragma unroll
      for (int k = 0; k < NST; ++k) {
        double a = ssum[k], b = ssq[k];
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          a += __shfl_xor_sync(0xffffffffu, a, o);
          b += __shfl_xor_sync(0xffffffffu, b, o);
        }
        if (lane < 4) {
          const int ch = split * NCTA + 8 * (k >> 1) + 2 * lane + (k & 1);
          atomicAdd(p.stats + 2 * ch, a);
          atomicAdd(p.stats + 2 * ch + 1, b);
        }
        ssum[k] = ssq[k] = 0.f;
      }
    };
    // store window plane J (output plane zo) if the item owns it
    auto emit = [&](const TcItem& it, auto jc, int zo) {
      constexpr int J = decltype(jc)::value;
      if (zo < it.z_lo || zo >= it.z_hi) return;
#pragma unroll
      for (int cb = 0; cb < M::SLOT_BLOCKS; ++cb) {
        const float* r = acc + (J * PCOLS + cb * NCTA) / 2;
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int mx = it.x0 + xr, my = it.y0 + 8 * wg + 2 * wq + rr;
          if (mx >= p.Mx || my >= p.My) continue;
          int xo = mx, yo = my;
          if (MODE == TC_T) {  // class order (0,0), (1,0), (1,1), (0,1)
            xo = 2 * mx + ((cb == 1 || cb == 2) ? 1 : 0);
            yo = 2 * my + (cb >= 2 ? 1 : 0);
          }
          const long long vox = ((long long)zo * p.Ho + yo) * p.Wo + xo;
          if (p.store1) {
            if (cq == 0) p.out[vox] = r[2 * rr];
            continue;
          }
          const int ch_base = (KSLICE ? 0 : it.split * NCTA) + 2 * cq;
          const float wz = (zo >= p.zw_lo && zo < p.zw_hi) ? p.zw : 1.f;
#pragma unroll
          for (int j = 0; j < NCTA / 8; ++j) {
            float v0 = r[4 * j + 2 * rr], v1 = r[4 * j + 2 * rr + 1];
            const int ch = ch_base + 8 * j;
            if (p.addend) {
              const int cls = zo == 0 ? 0 : (zo == p.Do - 1 ? 2 : 1);
              const float2 a2 = __ldg(reinterpret_cast<const float2*>(
                  p.addend + (((long long)cls * p.Ho + yo) * p.Wo + xo) * p.Cout + ch));
              v0 += a2.x;
              v1 += a2.y;
            }
            // (K-slice variant: p.out is the scratch, every slice stores its partial sums)
            *reinterpret_cast<float2*>(p.out + (KSLICE ? it.split * p.slice_stride : 0) +
                                       vox * p.Cout + ch) = make_float2(v0, v1);
            if constexpr (!KSLICE) {
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
    };
    // drop the first SH planes of the window, open SH empty ones at its end
    auto shift = [&](auto shc) {
      constexpr int SH = decltype(shc)::value * PCOLS / 2;
#pragma unroll
      for (int i = 0; i < NACC; ++i) acc[i] = i + SH < NACC ? acc[i + SH] : 0.f;
    };

    uint32_t stage_ctr = 0;
    TcWalk walk = tc_walk_begin(p);
    TcItem it;
    while (tc_walk_next(p, walk, it)) {
      const int zi0 = max(M::zi_first(it.z_lo), 0);
      const int zi1 = min(M::zi_last(it.z_hi - 1), p.Di - 1);
      for (int zi = zi0; zi <= zi1; ++zi) {
#pragma unroll 1
        for (int cg = 0; cg < NCG; ++cg, ++stage_ctr) {
          const int s = stage_ctr % M::NSTAGE;
          mbar_wait_timed<CLU>(full_a(s), (stage_ctr / M::NSTAGE) & 1, p.err, t_wait_a, timed);
          __syncwarp();
          const uint32_t a_lo_stage =
              ((((a_base + s * STAGE_BYTES) >> 4) & 0x3FFF) + a_wg16) | (A_LBO16 << 16);
          wgmma_fence();
          if constexpr (MODE == TC_S1) {
            // one N = 3*NCTA MMA per (tap, K step, operand term): weight rows [kz=2|kz=1|kz=0]
            // land in window planes zi-1, zi, zi+1; a 3x3 in-plane tap is a shift of the A view
            constexpr uint32_t B_LBO16 = 3 * NCTA;               // weight image rows
            constexpr uint32_t TAP16 = (CIN / 8) * B_LBO16;      // one tap, 16-byte units
            constexpr int NKS = CG / 16;
            const uint32_t b_lo0 = ((w_base >> 4) & 0x3FFF) + (uint32_t)(cg * NCH) * B_LBO16 +
                                   (B_LBO16 << 16);
            uint64_t da[NKS][2], db[NKS][2];
#pragma unroll
            for (int ks = 0; ks < NKS; ++ks) {
              da[ks][0] = pack64(a_lo_stage + 2 * ks * A_LBO16, a_desc_hi);
              da[ks][1] = pack64(a_lo_stage + 2 * ks * A_LBO16 + A_HL16, a_desc_hi);
              const uint32_t bl = b_lo0 + 2 * ks * B_LBO16;
              db[ks][0] = pack64(bl, b_desc_hi);
              db[ks][1] = pack64(bl + w_hi16, b_desc_hi);
            }
#pragma unroll 1
            for (int tap = 0; tap < 9; ++tap) {
#pragma unroll
              for (int ks = 0; ks < NKS; ++ks) {
                wgmma_bf16<3 * NCTA>(acc, da[ks][0], db[ks][0]);
                wgmma_bf16<3 * NCTA>(acc, da[ks][1], db[ks][0]);
                wgmma_bf16<3 * NCTA>(acc, da[ks][0], db[ks][1]);
              }
              const uint32_t ainc = (tap == 2 || tap == 5) ? (uint32_t)(M::PITCH - 2) : 1u;
#pragma unroll
              for (int ks = 0; ks < NKS; ++ks) {
                desc_add(da[ks][0], ainc);
                desc_add(da[ks][1], ainc);
                desc_add(db[ks][0], TAP16);
                desc_add(db[ks][1], TAP16);
              }
            }
          }
          if constexpr (MODE == TC_S2) {
            // one K step per 16-channel stage.  Even input planes feed window plane 0 (kz = 1);
            // odd planes feed planes 0 and 1 (kz = 2, kz = 0) with one N = 2*NCTA MMA.
            constexpr uint32_t KCH16 = CIN / 8;
            const uint32_t odd = (uint32_t)zi & 1u;
            auto run = [&](auto nbc) {
              constexpr uint32_t NB = decltype(nbc)::value;
              constexpr uint32_t b_lbo16 = NB * NCTA;
              constexpr uint32_t tap16 = KCH16 * b_lbo16;
              const uint32_t b_lo0 = ((w_base >> 4) & 0x3FFF) + (NB == 2 ? 9u * KCH16 * NCTA : 0u) +
                                     (uint32_t)(cg * NCH) * b_lbo16 + (b_lbo16 << 16);
              uint64_t dbh = pack64(b_lo0, b_desc_hi);
              uint64_t dbl = pack64(b_lo0 + w_hi16, b_desc_hi);
#pragma unroll
              for (int tap = 0; tap < 9; ++tap) {
                const int dy = tap / 3, dx = tap % 3;
                const uint32_t a16 = (uint32_t)(((dx & 1) * 2 + (dy & 1)) * S2_CLS16 +
                                                (dy >> 1) * M::PITCH + (dx >> 1));
                const uint64_t dah = pack64(a_lo_stage + a16, a_desc_hi);
                const uint64_t dal = pack64(a_lo_stage + a16 + A_HL16, a_desc_hi);
                wgmma_bf16<NB * NCTA>(acc, dah, dbh);
                wgmma_bf16<NB * NCTA>(acc, dal, dbh);
                wgmma_bf16<NB * NCTA>(acc, dah, dbl);
                desc_add(dbh, tap16);
                desc_add(dbl, tap16);
              }
            };
            if (odd) run(std::integral_constant<uint32_t, 2>());
            else run(std::integral_constant<uint32_t, 1>());
          }
          if constexpr (MODE == TC_T) {
            // the op list of tc_build_program<TC_T>: shift (0,0) one run of 12 class blocks from
            // block 0; x-only / y-only shifts one (zero-padded) run of 10 blocks from block 1 /
            // block 2; diagonal shift single blocks 2, 6, 10
            constexpr uint32_t KCH16 = CIN / 8;
            constexpr uint32_t NB[4] = {12u, 10u, 10u, 3u};      // blocks per weight image
            constexpr uint32_t LIN0[4] = {0u, 1u, 2u, 2u};
            uint32_t b_img16 = (w_base >> 4) & 0x3FFF;  // start of this shift's weight image
#pragma unroll
            for (int sh = 0; sh < 4; ++sh) {
              const uint32_t b_lbo16 = NB[sh] * NCTA;
              const uint32_t a16 = (uint32_t)((sh >> 1) * M::PITCH + (sh & 1));
#pragma unroll
              for (int ks = 0; ks < CG / 16; ++ks) {
                const uint32_t alo = a_lo_stage + a16 + 2 * ks * A_LBO16;
                const uint64_t dah = pack64(alo, a_desc_hi);
                const uint64_t dal = pack64(alo + A_HL16, a_desc_hi);
                const uint32_t blo = b_img16 + (uint32_t)(cg * NCH + 2 * ks) * b_lbo16 +
                                     (b_lbo16 << 16);
                auto mma3 = [&](float* d, uint32_t bl, auto nc) {
                  constexpr int N = decltype(nc)::value;
                  const uint64_t dbh = pack64(bl, b_desc_hi);
                  const uint64_t dbl = pack64(bl + w_hi16, b_desc_hi);
                  wgmma_bf16<N>(d, dah, dbh);
                  wgmma_bf16<N>(d, dal, dbh);
                  wgmma_bf16<N>(d, dah, dbl);
                };
                if (sh == 0) {
                  mma3(acc, blo, std::integral_constant<int, 12 * NCTA>());
                } else if (sh == 1) {
                  mma3(acc + NCTA / 2, blo, std::integral_constant<int, 10 * NCTA>());
                } else if (sh == 2) {
                  mma3(acc + NCTA, blo, std::integral_constant<int, 10 * NCTA>());
                } else {
#pragma unroll
                  for (uint32_t k = 0; k < 3; ++k)
                    mma3(acc + (LIN0[3] + k * 4) * (NCTA / 2), blo + k * NCTA,
                         std::integral_constant<int, NCTA>());
                }
              }
              b_img16 += KCH16 * b_lbo16;
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
          __syncwarp();
          // stage refillable: its MMAs have retired (cluster: tell the loaders of every CTA)
          if (lane == 0) {
            if constexpr (CLU) {
#pragma unroll
              for (int q = 0; q < CL; ++q) mbar_arrive_cluster(mapa_u32(empty_a(s), q));
            } else {
              mbar_arrive(empty_a(s));
            }
          }
        }
        // planes whose last contribution was this input plane leave the window
        if constexpr (MODE == TC_S1) {
          emit(it, std::integral_constant<int, 0>(), zi - 1);
          shift(std::integral_constant<int, 1>());
        } else if constexpr (MODE == TC_S2) {
          if (zi & 1) {
            emit(it, std::integral_constant<int, 0>(), zi >> 1);
            shift(std::integral_constant<int, 1>());
          }
        } else {
          emit(it, std::integral_constant<int, 0>(), 2 * zi - 1);
          emit(it, std::integral_constant<int, 1>(), 2 * zi);
          shift(std::integral_constant<int, 2>());
        }
      }
      // the planes still open after the item's last input plane
      const int zb = Win::base(zi1 + 1);
      emit(it, std::integral_constant<int, 0>(), zb);
      emit(it, std::integral_constant<int, 1>(), zb + 1);
      if constexpr (Win::NPL > 2) emit(it, std::integral_constant<int, 2>(), zb + 2);
#pragma unroll
      for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
      // a CTA keeps one output-channel group, so one flush per item keeps the fp32
      // partial sums short (<= planes-per-item * classes * 2 values per thread)
      flush_stats(it.split);
    }
    if (timed) {
      unsigned long long* rc = p.role_cycles + (size_t)blockIdx.x * 8;
      rc[0] = (unsigned long long)(clock64() - t_begin);
      rc[1] = t_wait_a;
    }
  }
  // no CTA may retire while a peer can still store into its stages or arrive on its barriers
  if constexpr (CLU) cluster_sync_all();
}

// ----------------------------------------------------------------------------------
// host launch
// ----------------------------------------------------------------------------------
// Error flag of the tensor-core kernels: page-locked host memory mapped into every device's
// address space (portable), written by a kernel whose mbarrier wait timed out and read by the
// host without any synchronisation, so every entry point can poll it for free.
struct TcErrFlag {
  int* host = nullptr;
  int* dev = nullptr;
  int* get() {
    if (!host) {
      if (cudaHostAlloc(&host, sizeof(int), cudaHostAllocMapped | cudaHostAllocPortable) !=
          cudaSuccess) {
        host = nullptr;
        cudaGetLastError();
        return nullptr;
      }
      *host = 0;
      cudaHostGetDevicePointer(&dev, host, 0);
    }
    return dev;
  }
};
inline TcErrFlag& tc_err_flag() {
  static TcErrFlag f;
  return f;
}
// returns non-zero if any tensor-core kernel timed out on a barrier since the last call
// (kernels that have completed; callers that need the current stream's state synchronise
// first, dfm_sync_check)
inline int tc_consume_error() {
  TcErrFlag& f = tc_err_flag();
  if (!f.host) return 0;
  const int h = *reinterpret_cast<volatile int*>(f.host);
  if (h) *reinterpret_cast<volatile int*>(f.host) = 0;
  return h;
}

// out[v][c] = sum over slices (in slice order) of part[s][v][c], C = 64; optional per-channel
// sum / sum of squares (planes [zw_lo, zw_hi) weighted by zw, like the conv epilogue does)
__global__ void __launch_bounds__(256)
kslice_reduce_kernel(const float* __restrict__ part, int nsl, long long V, long long HW,
                     float* __restrict__ out, double* __restrict__ stats, int zw_lo, int zw_hi,
                     float zw) {
  __shared__ double sh[2][16][64];
  const int q = threadIdx.x & 15, r = threadIdx.x >> 4;  // channel quad, voxel row
  double s[4] = {0, 0, 0, 0}, ss[4] = {0, 0, 0, 0};
  const long long w0 = (long long)zw_lo * HW, w1 = (long long)zw_hi * HW;
  for (long long v = (long long)blockIdx.x * 16 + r; v < V; v += (long long)gridDim.x * 16) {
    float4 a = __ldg(reinterpret_cast<const float4*>(part + v * 64) + q);
    for (int k = 1; k < nsl; ++k) {
      const float4 b = __ldg(reinterpret_cast<const float4*>(part + ((long long)k * V + v) * 64) + q);
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    reinterpret_cast<float4*>(out + v * 64)[q] = a;
    if (stats) {
      const double wgt = (v >= w0 && v < w1) ? (double)zw : 1.0;
      s[0] += wgt * a.x; ss[0] += wgt * (double)a.x * a.x;
      s[1] += wgt * a.y; ss[1] += wgt * (double)a.y * a.y;
      s[2] += wgt * a.z; ss[2] += wgt * (double)a.z * a.z;
      s[3] += wgt * a.w; ss[3] += wgt * (double)a.w * a.w;
    }
  }
  if (!stats) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    sh[0][r][4 * q + i] = s[i];
    sh[1][r][4 * q + i] = ss[i];
  }
  __syncthreads();
  if (threadIdx.x < 128) {
    const int c = threadIdx.x & 63, which = threadIdx.x >> 6;
    double t = 0.0;
    for (int k = 0; k < 16; ++k) t += sh[which][k][c];
    atomicAdd(stats + 2 * c + which, t);
  }
}
struct TcScratch {
  float* p = nullptr;
  size_t n = 0;
  float* get(size_t count) {  // grow-only, lives as long as the library
    if (n >= count) return p;
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
    if (cudaMalloc(&p, count * sizeof(float)) != cudaSuccess) return nullptr;
    n = count;
    return p;
  }
};
inline TcScratch& tc_kslice_scratch() { return per_device<TcScratch>(); }

struct TcOpts {
  int store1 = 0;
  const float* addend = nullptr;
  int zw_lo = 0, zw_hi = 0;
  float zw = 1.f;
  long long slice_stride = 0;
};
template <int MODE, int CIN, int NCTA, class Loader, int CL = 1>
bool tc_launch(const Loader& ld, const TcWeights& w, float* out, double* stats,
               const ConvGeom& g, cudaStream_t st, std::string* err, TcOpts opt = TcOpts()) {
  using M = TcMode<MODE>;
  constexpr int CG = M::CG < CIN ? M::CG : CIN;
  constexpr size_t STAGE_BYTES = (size_t)2 * (CG / 8) * M::ROWS * 16;
  const size_t smem = w.image_bytes + M::NSTAGE * STAGE_BYTES + (2 * M::NSTAGE + 1) * 8;
  auto kern = conv_tc_kernel<MODE, CIN, NCTA, Loader, CL>;
  if (w.cluster != CL || (CL > 1 && w.nsplit != CL)) {
    if (err) *err = "conv_tc: weight image was built for a different cluster size";
    return false;
  }
  struct AttrTag { size_t v = 0; };
  static AttrTag attr_dev[kMaxDevices];  // per kernel instantiation and device
  size_t& attr_smem = attr_dev[cur_device()].v;
  if (smem > attr_smem) {
    if (smem > 232448 ||
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
            cudaSuccess) {
      if (err) *err = "conv_tc: cannot reserve " + std::to_string(smem) + " B of shared memory";
      return false;
    }
    attr_smem = smem;
  }
  const int sms = tc_sm_count();
  TcParams p{};
  p.wimg = w.dev.p;
  p.out = out;
  p.stats = stats;
  p.store1 = opt.store1;
  p.slice_stride = opt.slice_stride;
  p.addend = opt.addend;
  p.zw_lo = opt.zw_lo;
  p.zw_hi = opt.zw_hi;
  p.zw = opt.zw;
  p.Di = g.Di; p.Hi = g.Hi; p.Wi = g.Wi;
  p.Do = g.Do; p.Ho = g.Ho; p.Wo = g.Wo;
  p.Cout = g.Cout;
  p.Mx = MODE == TC_T ? g.Wi : g.Wo;
  p.My = MODE == TC_T ? g.Hi : g.Ho;
  p.tiles_x = (p.Mx + TC_BX - 1) / TC_BX;
  p.tiles_y = (p.My + TC_BY - 1) / TC_BY;
  p.nsplit = w.nsplit;
  p.w_bytes = w.image_bytes;
  p.w_hi_bytes = w.hi_bytes;
  p.z_unit = MODE == TC_T ? 2 : 1;
  const long long cols = (long long)p.tiles_x * p.tiles_y;
  const long long units = cols * (g.Do / p.z_unit);
  // persistent grid: one CTA per SM, a multiple of the output-channel splits; never more
  // CTAs per split than there are z units.  Clusters: as many as fit at once (a cluster is
  // placed inside one GPC, so SMs that are left over in a GPC stay idle)
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute cl_attr[1];
  int per_split = std::max(1, sms / p.nsplit);
  if constexpr (CL > 1) {
    cfg.gridDim = dim3(CL);
    cfg.blockDim = dim3(TC_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cl_attr[0].id = cudaLaunchAttributeClusterDimension;
    cl_attr[0].val.clusterDim.x = CL;
    cl_attr[0].val.clusterDim.y = 1;
    cl_attr[0].val.clusterDim.z = 1;
    cfg.attrs = cl_attr;
    cfg.numAttrs = 1;
    static int max_clusters[kMaxDevices];  // per kernel instantiation and device
    int& mc = max_clusters[cur_device()];
    if (!mc && (cudaOccupancyMaxActiveClusters(&mc, kern, &cfg) != cudaSuccess || mc < 1)) {
      mc = 0;
      if (err) *err = "conv_tc: no cluster of " + std::to_string(CL) + " CTAs fits on this device";
      return false;
    }
    per_split = mc;
  }
  per_split = (int)std::min<long long>(per_split, units);
  const int grid = per_split * p.nsplit;
  p.err = tc_err_flag().get();
  static const bool role_dbg = getenv("DFM_TC_ROLE_CYCLES") != nullptr;
  static const int dbg_flags = getenv("DFM_TC_DEBUG") ? atoi(getenv("DFM_TC_DEBUG")) : 0;
  p.dbg = dbg_flags;
  static unsigned long long* role_buf = nullptr;
  if (role_dbg) {
    if (!role_buf) cudaMalloc(&role_buf, 1024 * 8 * sizeof(unsigned long long));
    cudaMemsetAsync(role_buf, 0, 1024 * 8 * sizeof(unsigned long long), st);
    p.role_cycles = role_buf;
  }
  if constexpr (CL > 1) {
    cfg.gridDim = dim3(grid);
    const cudaError_t le = cudaLaunchKernelEx(&cfg, kern, p, ld);
    if (le != cudaSuccess) {
      if (err) *err = std::string("conv_tc cluster launch: ") + cudaGetErrorString(le);
      return false;
    }
  } else {
    kern<<<grid, TC_THREADS, smem, st>>>(p, ld);
  }
  if (role_dbg) {  // debugging aid: synchronous, prints mean cycles per role
    cudaStreamSynchronize(st);
    std::vector<unsigned long long> h((size_t)grid * 8);
    cudaMemcpy(h.data(), role_buf, h.size() * 8, cudaMemcpyDeviceToHost);
    double a[8] = {0};
    for (int b = 0; b < grid; ++b)
      for (int k = 0; k < 8; ++k) a[k] += (double)h[(size_t)b * 8 + k] / grid;
    fprintf(stderr,
            "[tc mode=%d cin=%d ncta=%d cluster=%d grid=%d cols=%lld Do=%d] mma+epilogue: total "
            "%.0f wait_full_a %.0f | load: total %.0f wait_empty_a %.0f\n",
            MODE, CIN, NCTA, CL, grid, cols, g.Do, a[0], a[1], a[3], a[4]);
  }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    if (err) *err = std::string("conv_tc launch: ") + cudaGetErrorString(e);
    return false;
  }
  return true;
}

template <class Loader>
bool tc_dispatch(const Loader& ld, const TcWeights& w, float* out, double* stats,
                 const ConvGeom& g, cudaStream_t st, std::string* err, TcOpts opt = TcOpts()) {
  const int mode = tc_mode_of(g);
  if (mode != w.mode) {
    if (err) *err = "conv_tc: weight image was built for a different conv mode";
    return false;
  }
  if (w.kslice) {
    // the input-channel slices store partial outputs into a scratch; a second kernel adds them
    // in slice order into `out` and accumulates the GroupNorm statistics
    if (mode != TC_S2 || g.Cout != 64 || opt.addend || opt.store1) {
      if (err) *err = "conv_tc: K-slice weights are for plain stride-2 convs with 64 outputs";
      return false;
    }
    const long long V = (long long)g.Do * g.Ho * g.Wo;
    float* part = tc_kslice_scratch().get((size_t)w.nsplit * V * 64);
    if (!part) {
      if (err) *err = "conv_tc: cannot allocate the K-slice scratch";
      return false;
    }
    TcOpts o2 = opt;
    o2.slice_stride = V * 64;
    if (!tc_launch<TC_S2, 16, 64, Loader>(ld, w, part, nullptr, g, st, err, o2)) return false;
    const int blocks = (int)std::min<long long>(8LL * tc_sm_count(), (V + 15) / 16);
    kslice_reduce_kernel<<<blocks, 256, 0, st>>>(part, w.nsplit, V, (long long)g.Ho * g.Wo, out,
                                                 stats, opt.zw_lo, opt.zw_hi, opt.zw);
    if (cudaGetLastError() != cudaSuccess) {
      if (err) *err = "conv_tc: kslice_reduce_kernel launch failed";
      return false;
    }
    return true;
  }
  if (mode == TC_S2 && w.cluster > 1) {
    if (g.Cin == 32 && w.cluster == 2)
      return tc_launch<TC_S2, 32, 32, Loader, 2>(ld, w, out, stats, g, st, err, opt);
    if (err) *err = "conv_tc: unsupported (Cin, cluster size)";
    return false;
  }
#define TC_CASE(MD, CI, NC) \
  if (mode == MD && g.Cin == CI) \
    return tc_launch<MD, CI, NC, Loader>(ld, w, out, stats, g, st, err, opt)
  TC_CASE(TC_S1, 32, 32);
  TC_CASE(TC_S1, 64, 16);
  TC_CASE(TC_S2, 32, 32);
  TC_CASE(TC_S2, 64, 16);
  TC_CASE(TC_T, 64, 16);
#undef TC_CASE
  if (err) *err = "conv_tc: unsupported (mode, Cin)";
  return false;
}

inline bool tc_conv_src(const Src& s, const TcWeights& w, float* out, double* stats,
                        const ConvGeom& g, cudaStream_t st, std::string* err,
                        TcOpts opt = TcOpts()) {
  if (s.n == 1) {
    SrcLoader8<1> ld{s, g.Cin, g.Hi, g.Wi};
    return tc_dispatch(ld, w, out, stats, g, st, err, opt);
  }
  if (s.n == 2) {
    SrcLoader8<2> ld{s, g.Cin, g.Hi, g.Wi};
    return tc_dispatch(ld, w, out, stats, g, st, err, opt);
  }
  SrcLoader8<3> ld{s, g.Cin, g.Hi, g.Wi};
  return tc_dispatch(ld, w, out, stats, g, st, err, opt);
}
inline bool tc_conv_warp(const WarpLoader& wl, const TcWeights& w, float* out, double* stats,
                         const ConvGeom& g, cudaStream_t st, std::string* err,
                         TcOpts opt = TcOpts()) {
  if (tc_mode_of(g) != TC_S1) {
    if (err) *err = "conv_tc: the warp loader feeds stride-1 convs only";
    return false;
  }
  WarpLoader8 ld{wl};
  if (g.Cin == 32)
    return tc_launch<TC_S1, 32, 32, WarpLoader8>(ld, w, out, stats, g, st, err, opt);
  if (g.Cin == 64)
    return tc_launch<TC_S1, 64, 16, WarpLoader8>(ld, w, out, stats, g, st, err, opt);
  if (err) *err = "conv_tc: unsupported Cin";
  return false;
}

}  // namespace dfm
