// wgmma tensor-core 1x1 conv with bias for the output layer of Anchor3DHead
// (mmdet3d/models/dense_heads/anchor3d_head.py:139-164): conv_cls, conv_dir_cls and conv_reg
// on the same BEV map, computed as ONE GEMM
//     out[N][P] = W[N][Cin] * x[Cin][P] + b,   N = cls | dir | reg rows,  P = Ny * Nx cells
// so the map (67.6 MB at the Waymo shape) is read from HBM exactly once.
//   * Input and outputs are NCHW fp32, the layout the BEV neck writes and the reference head
//     returns.  A 1x1 conv has no halo: a tile is 128 consecutive cells of the flattened grid
//     (one channel of a tile = 512 contiguous bytes); the last tile is ragged.
//   * Persistent CTAs, one per SM, march over tiles.  Warps 0-7 are two consumer warpgroups
//     (64 accumulator rows = cells each), warps 8-15 two loader groups that fill alternate
//     stages of 64 input channels.  Stages are handed over with mbarriers, as in conv_tc.cuh.
//   * A operand: K-major no-swizzle core matrices [8-channel chunk][128 cells][16 B], the layout
//     of every other tensor-core kernel here, so the wgmma.cuh wrappers are reused unchanged.
//     The loaders do the channel-major -> K-major transpose in registers: a lane loads one
//     float4 (4 cells) of each of 8 channels -- every load instruction of a warp covers one
//     512-byte channel row of the tile -- and stores 16 B (8 channels) per cell.  The order of
//     a lane's four cell stores is rotated by (lane / 2) % 4, which makes each 8-lane store
//     phase hit 8 distinct 16-byte bank groups.  (An MN-major A descriptor would take the rows
//     as loaded, but needs its own descriptor layout and validation; the transpose costs the
//     loaders a few selects per value, and the kernel is HBM-bound.)
//   * B operand: the hi + lo weight image [Cin/8][NP][16 B] (NP = N padded to a supported
//     wgmma width, zero rows) and the bias stay resident in shared memory for the CTA's life.
//   * fp32 parity as everywhere (DESIGN.md section 1): x*w = x_hi w_hi + x_lo w_hi + x_hi w_lo
//     on the bf16 tensor pipe with fp32 accumulation in registers; the bias is added in fp32.
//   * Epilogue: the accumulators go to a shared [NP][128 + 4] staging tile (the pitch makes
//     the fragment scatter conflict-free); each warp then writes whole 128-cell channel rows,
//     bias added, straight into the cls / dir / reg tensors.
#pragma once
#include "conv_tc.cuh"

namespace dfm {

constexpr int H1_M = 128;                          // cells per tile (two warpgroups x 64)
constexpr int H1_KC = 64;                          // input channels per stage
constexpr int H1_NSTAGE = 3;
constexpr uint32_t H1_A_LBO = H1_M * 16;           // between 8-channel chunks of a stage
constexpr uint32_t H1_A_HL = (H1_KC / 8) * H1_A_LBO;  // hi -> lo (16 KB)
constexpr uint32_t H1_STAGE_BYTES = 2 * H1_A_HL;   // 32 KB
constexpr int H1_OUT_LD = H1_M + 4;                // staged output row pitch (floats)
constexpr int H1_THREADS = 256 + 256;              // consumer warpgroups | loader warps
constexpr size_t H1_SMEM_MAX = 227 * 1024;

struct Head1x1Params {
  const float* x;       // [Cin][P]
  const uint8_t* wimg;  // hi image then lo image, each [cin_pad / 8][NP][8] bf16
  const float* bias;    // [NP], zero past N
  float* out[3];        // cls, dir, reg: [rows][P]
  int rows[3];
  int P;                // cells; cin_pad * P < 2^31
  int cin, cin_pad, ntiles, vec4;
  int* err;
};

// padded output width: the wgmma N the kernel is instantiated for
inline int head1x1_np(int n) {
  for (int v : {32, 64, 72, 96, 128})
    if (n <= v) return v;
  return 0;
}
inline int head1x1_cin_pad(int cin) { return (cin + H1_KC - 1) / H1_KC * H1_KC; }
inline size_t head1x1_smem(int cin, int np) {
  return (size_t)4 * head1x1_cin_pad(cin) * np + (size_t)(np * 4 + 127) / 128 * 128 +
         (size_t)H1_NSTAGE * H1_STAGE_BYTES + (size_t)np * H1_OUT_LD * 4 + 2 * H1_NSTAGE * 8;
}
// Shapes the kernel takes: Cin a multiple of 16 (one bf16 K step), N within the widest
// instantiation (the accumulators, N / 2 registers per consumer thread, must fit the
// 128-register budget of a 512-thread CTA) and the resident weight image plus stages and
// staging tile within the 227 KB of shared memory of one CTA.
inline bool head1x1_supported(int cin, int n) {
  const int np = head1x1_np(n);
  return cin > 0 && cin % 16 == 0 && n > 0 && np > 0 && head1x1_smem(cin, np) <= H1_SMEM_MAX;
}

// 4 cells [cell, cell + 4) of channel ch; xc = x + cell, nleft = P - cell (> 0 for a live
// lane).  32-bit channel offsets (the host requires Cin * P < 2^31) keep the 16 loads a lane
// has in flight from holding 16 64-bit addresses.
__device__ __forceinline__ float4 h1_load4(const float* __restrict__ xc, int P, int nleft,
                                           int vec4, int ch, int cin) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (ch >= cin || nleft <= 0) return v;
  const float* r = xc + (unsigned)(ch * P);
  if (vec4) {
    v = __ldg(reinterpret_cast<const float4*>(r));
  } else {
    v.x = __ldg(r);
    if (nleft > 1) v.y = __ldg(r + 1);
    if (nleft > 2) v.z = __ldg(r + 2);
    if (nleft > 3) v.w = __ldg(r + 3);
  }
  return v;
}
__device__ __forceinline__ float h1_comp(const float4& f, int j) {
  return j == 0 ? f.x : j == 1 ? f.y : j == 2 ? f.z : f.w;
}
// g[j] = f[(j + r) & 3]
__device__ __forceinline__ float4 h1_rot4(float4 f, int r) {
  if (r & 1) f = make_float4(f.y, f.z, f.w, f.x);
  if (r & 2) f = make_float4(f.z, f.w, f.x, f.y);
  return f;
}

template <int NP>
__global__ void __launch_bounds__(H1_THREADS, 1)
head1x1_tc_kernel(const __grid_constant__ Head1x1Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t w_bytes = 4u * p.cin_pad * NP;
  uint8_t* w_s = smem;
  float* bias_s = reinterpret_cast<float*>(smem + w_bytes);
  uint8_t* a_s = smem + w_bytes + (NP * 4 + 127) / 128 * 128;
  float* out_s = reinterpret_cast<float*>(a_s + H1_NSTAGE * H1_STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(out_s + NP * H1_OUT_LD);

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
  // resident weight image (generic-proxy copy, fenced for the tensor core) and bias
  for (int i = tid; i < (int)(w_bytes / 16); i += H1_THREADS)
    reinterpret_cast<uint4*>(w_s)[i] = __ldg(reinterpret_cast<const uint4*>(p.wimg) + i);
  for (int i = tid; i < NP; i += H1_THREADS) bias_s[i] = __ldg(p.bias + i);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const int nk = p.cin_pad / H1_KC;

  if (warp >= 8) {
    // ================================ loaders ================================
    const int lw = warp - 8, grp = lw >> 2, wq = lw & 3;
    const int rot = (lane >> 1) & 3;
    uint32_t ctr = 0;
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
      const int cell = tile * H1_M + 4 * lane;
      const float* xc = p.x + cell;
      for (int kc = 0; kc < nk; ++kc, ++ctr) {
        if ((int)(ctr & 1) != grp) continue;
        const int s = ctr % H1_NSTAGE;
        // this warp's two 8-channel chunks of the stage; loads are in flight while the stage
        // may still be in use by the MMAs
        float4 f[2][8];
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
          for (int c = 0; c < 8; ++c)
            f[q][c] = h1_load4(xc, p.P, p.P - cell, p.vec4, kc * H1_KC + (2 * wq + q) * 8 + c,
                               p.cin);
        mbar_wait(empty(s), ((ctr / H1_NSTAGE) & 1) ^ 1, p.err);
        uint8_t* st = a_s + s * H1_STAGE_BYTES;
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
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) mbar_arrive(full(s));
      }
    }
  } else {
    // ===================== consumer warpgroups: MMA, then the epilogue =====================
    const int wg = warp >> 2;
    constexpr uint32_t B_LBO = NP * 16;
    const uint32_t a_base = smem_u32(a_s) + wg * 64 * 16, w_base = smem_u32(w_s);
    const uint32_t w_hl16 = (uint32_t)(2 * p.cin_pad * NP) >> 4;   // hi image -> lo image
    const uint32_t desc_hi = 128u >> 4;                            // SBO: dense 8-row groups
    const int n_rows = p.rows[0] + p.rows[1] + p.rows[2];
    float acc[NP / 2];
    uint32_t ctr = 0;
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
#pragma unroll
      for (int i = 0; i < NP / 2; ++i) acc[i] = 0.f;
      for (int kc = 0; kc < nk; ++kc, ++ctr) {
        const int s = ctr % H1_NSTAGE;
        mbar_wait(full(s), (ctr / H1_NSTAGE) & 1, p.err);
        const uint32_t a_lo = (((a_base + s * H1_STAGE_BYTES) >> 4) & 0x3FFF) |
                              ((H1_A_LBO >> 4) << 16);
        const uint32_t b_lo = (((w_base + kc * (H1_KC / 8) * B_LBO) >> 4) & 0x3FFF) |
                              ((B_LBO >> 4) << 16);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < H1_KC / 16; ++ks) {
          const uint64_t ah = pack64(a_lo + 2 * ks * (H1_A_LBO >> 4), desc_hi);
          const uint64_t al = pack64(a_lo + 2 * ks * (H1_A_LBO >> 4) + (H1_A_HL >> 4), desc_hi);
          const uint64_t bh = pack64(b_lo + 2 * ks * (B_LBO >> 4), desc_hi);
          const uint64_t bl = pack64(b_lo + 2 * ks * (B_LBO >> 4) + w_hl16, desc_hi);
          wgmma_bf16<NP>(acc, ah, bh);
          wgmma_bf16<NP>(acc, al, bh);
          wgmma_bf16<NP>(acc, ah, bl);
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(empty(s));
      }
      // every consumer has finished reading the previous tile's staging rows
      asm volatile("bar.sync 1, 256;" ::: "memory");
      // register i: cell 64 wg + 16 (warp % 4) + lane / 4 + 8 ((i / 2) & 1),
      //             output row 8 (i / 4) + 2 (lane % 4) + (i & 1)
#pragma unroll
      for (int i = 0; i < NP / 2; ++i) {
        const int m = 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * ((i >> 1) & 1);
        const int n = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        out_s[n * H1_OUT_LD + m] = acc[i];
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      const int p0 = tile * H1_M;
      for (int n = warp; n < n_rows; n += 8) {
        int o = 0, r = n;
        while (r >= p.rows[o]) r -= p.rows[o++];
        float* dst = p.out[o] + (long long)r * p.P + p0;
        const float b = bias_s[n];
#pragma unroll
        for (int q = 0; q < H1_M / 32; ++q) {
          const int m = lane + 32 * q;
          if (p0 + m < p.P) dst[m] = out_s[n * H1_OUT_LD + m] + b;
        }
      }
    }
  }
}

// Device images of the combined 1x1 conv: hi + lo bf16 weights and the fp32 bias.
struct Head1x1Weights {
  DevArray<uint8_t> wimg;
  DevArray<float> bias;
  int cin = 0, n = 0, np = 0;
  bool ready() const { return wimg.p != nullptr; }
  // w: [n][cin] rows (cls | dir | reg), b: [n]
  bool build(const float* w, const float* b, int cin_, int n_, std::string* err) {
    wimg.release();
    bias.release();
    cin = cin_;
    n = n_;
    np = head1x1_np(n);
    const int cp = head1x1_cin_pad(cin);
    const size_t half = (size_t)cp * np;   // bf16 elements of one image
    std::vector<uint16_t> img(2 * half, 0);
    for (int co = 0; co < n; ++co)
      for (int ci = 0; ci < cin; ++ci) {
        const float v = w[(size_t)co * cin + ci];
        const uint16_t hi = bf16_rn_bits(v);
        const uint16_t lo = bf16_rn_bits(v - bf16_bits_to_float(hi));
        const size_t off = ((size_t)(ci / 8) * np + co) * 8 + ci % 8;
        img[off] = hi;
        img[off + half] = lo;
      }
    std::vector<float> bp(np, 0.f);
    std::copy(b, b + n, bp.begin());
    if (wimg.upload(reinterpret_cast<const uint8_t*>(img.data()), img.size() * 2) !=
            cudaSuccess ||
        bias.upload(bp.data(), np) != cudaSuccess) {
      cudaGetLastError();
      if (err) *err = "head1x1_tc: weight upload failed";
      wimg.release();
      bias.release();
      return false;
    }
    return true;
  }
};

// x [cin][P] -> out[o] [rows[o]][P] for o = cls, dir, reg (rows summing to w.n)
inline bool head1x1_tc_launch(const Head1x1Weights& w, const float* x, long long P,
                              float* const out[3], const int rows[3], cudaStream_t st,
                              std::string* err) {
  if (!w.ready() || rows[0] + rows[1] + rows[2] != w.n) {
    if (err) *err = "head1x1_tc: weights not built for this layer";
    return false;
  }
  Head1x1Params p{};
  p.x = x;
  p.wimg = w.wimg.p;
  p.bias = w.bias.p;
  for (int o = 0; o < 3; ++o) {
    p.out[o] = out[o];
    p.rows[o] = rows[o];
  }
  p.cin = w.cin;
  p.cin_pad = head1x1_cin_pad(w.cin);
  if ((long long)p.cin_pad * (P + H1_M) > 0x7fffffffLL) {
    if (err) *err = "head1x1_tc: map too large for 32-bit offsets";
    return false;
  }
  p.P = (int)P;
  const long long tiles = (P + H1_M - 1) / H1_M;
  p.ntiles = (int)tiles;
  p.vec4 = P % 4 == 0 && reinterpret_cast<uintptr_t>(x) % 16 == 0;
  p.err = tc_err_flag().get();
  const size_t smem = head1x1_smem(w.cin, w.np);
  const int grid = (int)std::min<long long>(tiles, tc_sm_count());
  auto launch = [&](auto kern, int& attr) -> bool {
    if (attr < (int)smem) {
      if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
          cudaSuccess) {
        cudaGetLastError();
        if (err) *err = "head1x1_tc: cannot reserve shared memory";
        return false;
      }
      attr = (int)smem;
    }
    kern<<<grid, H1_THREADS, smem, st>>>(p);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      if (err) *err = std::string("head1x1_tc launch: ") + cudaGetErrorString(e);
      return false;
    }
    return true;
  };
  switch (w.np) {
    case 32: return launch(head1x1_tc_kernel<32>, per_device<int, 1032>());
    case 64: return launch(head1x1_tc_kernel<64>, per_device<int, 1064>());
    case 72: return launch(head1x1_tc_kernel<72>, per_device<int, 1072>());
    case 96: return launch(head1x1_tc_kernel<96>, per_device<int, 1096>());
    case 128: return launch(head1x1_tc_kernel<128>, per_device<int, 1128>());
  }
  if (err) *err = "head1x1_tc: unsupported output width";
  return false;
}

}  // namespace dfm
