// HBM-bound tail of the KITTI path, second generation (round 2):
//   * logits_conv_kernel  -- the 32 -> 1 channel 3x3x3 conv of build_depth_pred_module
//     (dfm_backbone.py:128) as a CUDA-core kernel.  The op reads V*32 floats and writes V
//     (0.43 GB); on the tensor-core conv it would run as an N = 96 MMA with 1/32 useful
//     columns.  Formulation: per INPUT voxel, the 27
//     per-tap dot products q_t = <x, w_t> (864 FMAs whose weight operands come from the
//     constant bank: the weights are a __grid_constant__ kernel parameter and every index is a
//     compile-time constant), staged in shared memory; per OUTPUT voxel, out(o) = sum_t q_t(o + off_t) is 27 shared-memory reads.
//     A block owns a 26 x 16 (x, y) output tile (28 x 18 halo = 504 positions, two per thread)
//     and marches along z with three running accumulators per output pixel.
//   * depth_head4_kernel  -- DepthHead.forward with four consecutive x pixels per thread so the
//     two [4D,4H,4W] volumes are written with 16-byte stores, 512 contiguous bytes per warp
//     and depth bin.
//   * gate_persistent_kernel -- the mono/stereo gate with the 1x1 conv weights resident in
//     shared memory (transposed), one persistent block per SM.
#pragma once
#include "conv_tc.cuh"
#include "simt_kernels.cuh"

namespace dfm {

constexpr int LC_TX = 26, LC_TY = 16;                 // output tile
constexpr int LC_PX = LC_TX + 2, LC_PY = LC_TY + 2;   // input halo
constexpr int LC_NPOS = LC_PX * LC_PY;                // 504
constexpr int LC_THREADS = 256;
constexpr int LC_ZCHUNK = 8;                          // output planes per block

struct LogitsConvParams {
  float w[27 * 32];   // [tap = kz*9 + ky*3 + kx][channel]
  Term t;             // single input term (GroupNorm affine + ReLU folded into the load)
  int D, H, W;
  int tiles_x, tiles_y, zchunks;
};

// Weights come from the constant bank; one position at a time.
__global__ void __launch_bounds__(LC_THREADS)
logits_conv_kernel(const __grid_constant__ LogitsConvParams p, float* __restrict__ out) {
  extern __shared__ float lc_q[];   // [27][LC_NPOS]
  float (*q)[LC_NPOS] = reinterpret_cast<float (*)[LC_NPOS]>(lc_q);
  const int tid = threadIdx.x;
  int b = blockIdx.x;
  const int tx_i = b % p.tiles_x;
  b /= p.tiles_x;
  const int ty_i = b % p.tiles_y;
  const int zc = b / p.tiles_y;
  const int x0 = tx_i * LC_TX, y0 = ty_i * LC_TY;
  const int z_lo = zc * LC_ZCHUNK, z_hi = min(p.D, z_lo + LC_ZCHUNK);
  const long long plane = (long long)p.H * p.W;

  // per-channel affine of the input term, in registers (32 + 32)
  float sc[32], sh[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) {
    sc[c] = p.t.scale ? __ldg(p.t.scale + c) : 1.f;
    sh[c] = p.t.scale ? __ldg(p.t.shift + c) : 0.f;
  }
  // the (up to) two output pixels of this thread: tile-linear indices tid and tid + 256
  int oy[2], ox[2];
  bool olive[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int i = tid + k * LC_THREADS;
    oy[k] = i / LC_TX;
    ox[k] = i % LC_TX;
    olive[k] = i < LC_TX * LC_TY && y0 + oy[k] < p.H && x0 + ox[k] < p.W;
  }
  float accA[2] = {0.f, 0.f}, accB[2] = {0.f, 0.f};  // output planes zi-1 and zi

  for (int zi = max(z_lo - 1, 0); zi <= min(z_hi, p.D - 1); ++zi) {
    // ---- phase 1: q_t of this input plane's halo positions ----
#pragma unroll 1
    for (int k = 0; k < 2; ++k) {
      const int pos = tid + k * LC_THREADS;
      if (pos >= LC_NPOS) break;
      const int py = pos / LC_PX, px = pos % LC_PX;
      const int gy = y0 - 1 + py, gx = x0 - 1 + px;
      if (gy < 0 || gy >= p.H || gx < 0 || gx >= p.W) {
#pragma unroll
        for (int t = 0; t < 27; ++t) q[t][pos] = 0.f;
        continue;
      }
      const float4* src = reinterpret_cast<const float4*>(
          p.t.x + ((long long)term_plane(p.t, zi) * plane + (long long)gy * p.W + gx) * 32);
      float x[32];
#pragma unroll
      for (int v = 0; v < 8; ++v) {
        const float4 a = __ldg(src + v);
        x[4 * v] = a.x; x[4 * v + 1] = a.y; x[4 * v + 2] = a.z; x[4 * v + 3] = a.w;
      }
#pragma unroll
      for (int c = 0; c < 32; ++c) {
        x[c] = fmaf(x[c], sc[c], sh[c]);
        if (p.t.relu) x[c] = fmaxf(x[c], 0.f);
      }
#pragma unroll
      for (int t = 0; t < 27; ++t) {
        float a0 = 0.f, a1 = 0.f;   // two chains per tap
#pragma unroll
        for (int c = 0; c < 32; c += 2) {
          a0 = fmaf(x[c], p.w[t * 32 + c], a0);
          a1 = fmaf(x[c + 1], p.w[t * 32 + c + 1], a1);
        }
        q[t][pos] = a0 + a1;
      }
    }
    __syncthreads();
    // ---- phase 2: gather.  Input plane zi feeds output planes zi-1 (kz = 2), zi (kz = 1)
    // and zi+1 (kz = 0); out(zi-1) is complete after this plane.
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      if (!olive[k]) continue;
      float s0 = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const int pos = (oy[k] + ky) * LC_PX + ox[k] + kx;
          s0 += q[0 * 9 + ky * 3 + kx][pos];
          s1 += q[1 * 9 + ky * 3 + kx][pos];
          s2 += q[2 * 9 + ky * 3 + kx][pos];
        }
      const int zo = zi - 1;
      if (zo >= z_lo && zo < z_hi)
        out[(long long)zo * plane + (long long)(y0 + oy[k]) * p.W + x0 + ox[k]] = accA[k] + s2;
      accA[k] = accB[k] + s1;
      accB[k] = s0;
    }
    __syncthreads();
  }
  // the last output plane of the chunk when it is the volume's last plane (no input plane
  // z_hi exists to flush it)
  if (z_hi == p.D) {
#pragma unroll
    for (int k = 0; k < 2; ++k)
      if (olive[k])
        out[(long long)(p.D - 1) * plane + (long long)(y0 + oy[k]) * p.W + x0 + ox[k]] = accA[k];
  }
}

inline bool logits_conv_launch(const Src& s, const float* h_w /*[27][32] host*/, float* out,
                               int D, int H, int W, cudaStream_t st) {
  if (s.n != 1 || s.outer_relu) return false;
  LogitsConvParams p;
  memcpy(p.w, h_w, sizeof(p.w));
  p.t = s.t[0];
  p.D = D; p.H = H; p.W = W;
  p.tiles_x = (W + LC_TX - 1) / LC_TX;
  p.tiles_y = (H + LC_TY - 1) / LC_TY;
  p.zchunks = (D + LC_ZCHUNK - 1) / LC_ZCHUNK;
  const long long blocks = (long long)p.tiles_x * p.tiles_y * p.zchunks;
  if (blocks > 0x7fffffffLL) return false;
  constexpr size_t smem = sizeof(float) * 27 * LC_NPOS;
  bool& attr_done = per_device<bool, 7>();
  if (!attr_done) {
    if (cudaFuncSetAttribute(logits_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)smem) != cudaSuccess)
      return false;
    attr_done = true;
  }
  logits_conv_kernel<<<(unsigned)blocks, LC_THREADS, smem, st>>>(p, out);
  return cudaGetLastError() == cudaSuccess;
}

// ---------------------------------------------------------------------------------
// DepthHead.forward, four x pixels per thread (requires (Wo * f) % 4 == 0).
// Structure chosen to cut the instructions per 4-pixel depth bin (the first version was
// issue-bound): the two low-res rows a block interpolates between are blended ONCE
// while staging (R[z][c] = ly0*row0 + ly1*row1), the depth loop walks low-res intervals with
// the carried pair (b0, b1) and an inner loop over the bins of the interval, all per-bin
// constants come from shared-memory tables.
// ---------------------------------------------------------------------------------
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
constexpr int DH4_PX = 128;   // output pixels along x per block
__host__ __device__ inline int dh4_ncols(int f) { return DH4_PX / f + 3; }
constexpr int DH4_ZS = 8;     // depth segments (warps) per block: they share the staged rows
// dynamic shared memory: per-bin table float4[D f] | first-bin table int[D + 2 (+pad)] | rows
__host__ __device__ inline int dh4_k0_ints(int D) { return (D + 2 + 3) / 4 * 4; }
inline size_t dh4_smem_bytes(int D, int f) {
  return (size_t)D * f * sizeof(float4) + (size_t)dh4_k0_ints(D) * sizeof(int) +
         (size_t)D * dh4_ncols(f) * sizeof(float);
}

__global__ void __launch_bounds__(32 * DH4_ZS, 4)
depth_head4_kernel(const float* __restrict__ cost, const float* __restrict__ samples, int D,
                   int Ho, int Wo, int f, float* __restrict__ vol, float* __restrict__ sm,
                   float* __restrict__ preds, float2* __restrict__ norm) {
  constexpr int DH_ZS = DH4_ZS;                      // (shadows the one-pixel kernel's constant)
  extern __shared__ float4 dh4_dyn[];
  const int OW = Wo * f, OH = Ho * f, OD = D * f;
  float4* tab = dh4_dyn;                                          // per bin: (l0, l1, sample, -)
  int* tab_k0 = reinterpret_cast<int*>(tab + OD);                 // first bin of interval z
  float* dh_rows = reinterpret_cast<float*>(tab_k0 + dh4_k0_ints(D));  // [D][nc]: y-blended rows
  __shared__ float red[3][DH_ZS][DH4_PX];
  const int tx = threadIdx.x, seg = threadIdx.y, tid = seg * 32 + tx;
  const float sz = OD > 1 ? (float)(D - 1) / (OD - 1) : 0.f;
  for (int z = tid; z <= D; z += 32 * DH_ZS) tab_k0[z] = OD;
  __syncthreads();
  for (int k = tid; k < OD; k += 32 * DH_ZS) {
    const float fz = sz * k;       // ATen: area_pixel_compute_source_index, align_corners
    const int z0 = min((int)fz, D - 1);
    const float l1 = fz - z0;
    tab[k] = make_float4(1.f - l1, l1, samples ? __ldg(samples + k) : 0.f, 0.f);
    atomicMin(&tab_k0[z0], k);
  }
  const int Xb = blockIdx.x * DH4_PX;
  const int X0 = Xb + 4 * tx;                        // first of this thread's four pixels
  const bool live = X0 < OW;                          // OW % 4 == 0: all four or none
  const int Y = blockIdx.y;
  const float sx = OW > 1 ? (float)(Wo - 1) / (OW - 1) : 0.f;
  const float sy = OH > 1 ? (float)(Ho - 1) / (OH - 1) : 0.f;
  const float fy = sy * Y;
  const int y0 = (int)fy;
  const int y1 = y0 + (y0 < Ho - 1 ? 1 : 0);
  const float ly1 = fy - y0, ly0 = 1.f - ly1;
  const long long plane = (long long)Ho * Wo;
  const long long oplane = (long long)OH * OW;
  const int nc = dh4_ncols(f);
  const int xb = (int)(sx * Xb);                      // first low-res column of the block
  for (int i = tid; i < D * nc; i += 32 * DH_ZS) {
    const int z = i / nc, c = i - z * nc;
    const int xc = min(xb + c, Wo - 1);
    dh_rows[i] = ly0 * __ldg(cost + z * plane + y0 * Wo + xc) +
                 ly1 * __ldg(cost + z * plane + y1 * Wo + xc);
  }
  int c0[4], c1[4];
  float wx0[4], wx1[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int X = min(X0 + j, OW - 1);
    const float fx = sx * X;
    const int x0 = (int)fx;
    const int x1 = x0 + (x0 < Wo - 1 ? 1 : 0);
    wx1[j] = fx - x0;
    wx0[j] = 1.f - wx1[j];
    c0[j] = x0 - xb;
    c1[j] = x1 - xb;
  }
  __syncthreads();
  // an interval without bins (fp32 rounding can leave the last one empty) starts where the
  // next one does
  if (tid == 0)
    for (int z = D - 1; z >= 0; --z) tab_k0[z] = min(tab_k0[z], tab_k0[z + 1]);
  __syncthreads();
  auto col = [&](int z, int j) {
    const float* pz = dh_rows + z * nc;
    return wx0[j] * pz[c0[j]] + wx1[j] * pz[c1[j]];
  };
  // this thread's share of the depth axis: low-res planes [zA, zB) for the maximum, the bins of
  // the intervals [zA, zB) for the sums and the writes
  const int zA = seg * D / DH_ZS, zB = (seg + 1) * D / DH_ZS;
  float m[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float mm = -INFINITY;
    for (int z = zA; z < zB; ++z) mm = fmaxf(mm, col(z, j));
    red[0][seg][4 * tx + j] = mm;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    m[j] = red[0][0][4 * tx + j];
#pragma unroll
    for (int i = 1; i < DH_ZS; ++i) m[j] = fmaxf(m[j], red[0][i][4 * tx + j]);
  }
  float ssum[4] = {0.f, 0.f, 0.f, 0.f}, esum[4] = {0.f, 0.f, 0.f, 0.f};
  float b0[4], b1[4];
  // sum pass in the exp2 domain with the maximum folded into the interval ends:
  // l0 + l1 == 1, so l0 * (b0 - m) + l1 * (b1 - m) == v - m and a bin costs mul, fma, ex2,
  // add, fma per pixel
  constexpr float LOG2E = 1.4426950408889634f;
  float ml2[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    ml2[j] = m[j] * LOG2E;
    b1[j] = fmaf(col(zA, j), LOG2E, -ml2[j]);
  }
  for (int z = zA; z < zB; ++z) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      b0[j] = b1[j];
      b1[j] = z < D - 1 ? fmaf(col(z + 1, j), LOG2E, -ml2[j]) : b0[j];
    }
    const int ke = tab_k0[z + 1];
    for (int k = tab_k0[z]; k < ke; ++k) {
      const float4 tk = tab[k];
      const float l0 = tk.x, l1 = tk.y, s = tk.z;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float e = ex2_approx(fmaf(l1, b1[j], l0 * b0[j]));
        ssum[j] += e;
        esum[j] = fmaf(e, s, esum[j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    red[1][seg][4 * tx + j] = ssum[j];
    red[2][seg][4 * tx + j] = esum[j];
  }
  __syncthreads();
  float inv[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float a = 0.f, e = 0.f;
#pragma unroll
    for (int i = 0; i < DH_ZS; ++i) {
      a += red[1][i][4 * tx + j];
      e += red[2][i][4 * tx + j];
    }
    ssum[j] = a;
    esum[j] = e;
    inv[j] = 1.f / a;
  }
  if (!live) return;
  const long long opix = (long long)Y * OW + X0;
  if (seg == 0) {
    if (preds)
      *reinterpret_cast<float4*>(preds + opix) =
          make_float4(esum[0] / ssum[0], esum[1] / ssum[1], esum[2] / ssum[2], esum[3] / ssum[3]);
    if (norm) {
#pragma unroll
      for (int j = 0; j < 4; ++j) norm[opix + j] = make_float2(m[j], inv[j]);
    }
  }
  if (!sm && !vol) return;
#pragma unroll
  for (int j = 0; j < 4; ++j) b1[j] = col(zA, j);
  // bins are visited in increasing k: running output pointers (null outputs are never stored)
  float* pv = vol + (long long)tab_k0[zA] * oplane + opix;
  float* ps = sm + (long long)tab_k0[zA] * oplane + opix;
  for (int z = zA; z < zB; ++z) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      b0[j] = b1[j];
      b1[j] = z < D - 1 ? col(z + 1, j) : b0[j];
    }
    const int ke = tab_k0[z + 1];
    for (int k = tab_k0[z]; k < ke; ++k) {
      const float2 tk = *reinterpret_cast<const float2*>(&tab[k]);
      const float l0 = tk.x, l1 = tk.y;
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = l0 * b0[j] + l1 * b1[j];
      if (vol) __stcs(reinterpret_cast<float4*>(pv), make_float4(v[0], v[1], v[2], v[3]));
      pv += oplane;
      if (sm)
        __stcs(reinterpret_cast<float4*>(ps),
               make_float4(ex2_approx(fmaf(v[0], LOG2E, -ml2[0])) * inv[0],
                           ex2_approx(fmaf(v[1], LOG2E, -ml2[1])) * inv[1],
                           ex2_approx(fmaf(v[2], LOG2E, -ml2[2])) * inv[2],
                           ex2_approx(fmaf(v[3], LOG2E, -ml2[3])) * inv[3]));
      ps += oplane;
    }
  }
}

// ---------------------------------------------------------------------------------
// mono/stereo gate (dfm_backbone.py:135-141), persistent: the (D x 2D) 1x1-conv weights live
// in shared memory, transposed to [2D][DG*16] so the 16 weights of a thread's plane group for
// one input plane j are four broadcast 16-byte reads.
// ---------------------------------------------------------------------------------
constexpr int GT_PG = 16;   // output planes per thread
__host__ __device__ inline int gate_row_pitch(int D) { return (D + GT_PG - 1) / GT_PG * GT_PG; }
// pixel halves per block: 2 x 32 pixels share the resident weights when the block stays <= 512
// threads (14 instead of 7 warps per SM to hide the shared-memory latency)
__host__ __device__ inline int gate_halves(int D) { return 32 * ((D + GT_PG - 1) / GT_PG) * 2 <= 512 ? 2 : 1; }
inline size_t gate_smem_bytes(int D) {
  return ((size_t)2 * D * gate_row_pitch(D) + (size_t)2 * D * 32 * gate_halves(D)) * sizeof(float);
}
// wT: the 1x1 conv weight transposed and padded on the host, [2D][gate_row_pitch(D)]
__global__ void __launch_bounds__(512)
gate_persistent_kernel(const float* __restrict__ ls, const float* __restrict__ lm,
                       const float* __restrict__ wT_g, float* __restrict__ cost, int D, int HW,
                       ZExpand zm) {
  extern __shared__ float gsm[];
  const int ng = (D + GT_PG - 1) / GT_PG, DP = ng * GT_PG;
  float* wT = gsm;                          // [2D][DP]
  const int NH = gate_halves(D), TP = 32 * NH;   // pixels per tile
  float* cat = gsm + (size_t)2 * D * DP;    // [2D][TP]
  const int nthreads = blockDim.x;          // 32 * ng * NH
  {
    const float4* src = reinterpret_cast<const float4*>(wT_g);
    float4* dst = reinterpret_cast<float4*>(wT);
    for (int i = threadIdx.x; i < 2 * D * DP / 4; i += nthreads) dst[i] = __ldg(src + i);
  }
  const int g = (threadIdx.x >> 5) % ng;
  const int px = (threadIdx.x & 31) + 32 * ((threadIdx.x >> 5) / ng);   // pixel inside the tile
  const int ntiles = (HW + TP - 1) / TP;
  constexpr int MAXJ = 32;                  // planes of the cat column a thread stages (2D / ng)
  const int nj = (2 * D - g + ng - 1) / ng; // j = g, g + ng, ...
  float stage[MAXJ];
  auto fetch = [&](int tile) {
    const int p = tile * TP + px;
#pragma unroll
    for (int q = 0; q < MAXJ; ++q) {
      const int j = g + q * ng;
      float v = 0.f;
      if (q < nj && p < HW)
        v = j < D ? __ldg(ls + (long long)j * HW + p)
                  : __ldg(lm + (long long)zexpand(zm, j - D) * HW + p);
      stage[q] = v;
    }
  };
  int tile = blockIdx.x;
  if (tile < ntiles) fetch(tile);
  for (; tile < ntiles; tile += gridDim.x) {
    const int p = tile * TP + px;
    __syncthreads();   // previous tile's cat fully consumed (and wT written, first time)
#pragma unroll
    for (int q = 0; q < MAXJ; ++q)
      if (q < nj) cat[(g + q * ng) * TP + px] = stage[q];
    __syncthreads();
    // the next tile's column is fetched while this one is being reduced
    if (tile + (int)gridDim.x < ntiles) fetch(tile + gridDim.x);
    float a[GT_PG];
#pragma unroll
    for (int k = 0; k < GT_PG; ++k) a[k] = 0.f;
    const float4* wrow = reinterpret_cast<const float4*>(wT + g * GT_PG);
#pragma unroll 4
    for (int j = 0; j < 2 * D; ++j) {
      const float c = cat[j * TP + px];
      const float4* w4 = wrow + (size_t)j * (DP / 4);
#pragma unroll
      for (int q = 0; q < GT_PG / 4; ++q) {
        const float4 w = w4[q];
        a[4 * q] = fmaf(w.x, c, a[4 * q]);
        a[4 * q + 1] = fmaf(w.y, c, a[4 * q + 1]);
        a[4 * q + 2] = fmaf(w.z, c, a[4 * q + 2]);
        a[4 * q + 3] = fmaf(w.w, c, a[4 * q + 3]);
      }
    }
    if (p < HW) {
#pragma unroll
      for (int k = 0; k < GT_PG; ++k) {
        const int d = g * GT_PG + k;
        if (d < D) {
          const float wgt = 1.f / (1.f + __expf(-a[k]));
          const float sv = cat[d * TP + px], mv = cat[(D + d) * TP + px];
          cost[(long long)d * HW + p] = wgt * sv + (1.f - wgt) * mv;
        }
      }
    }
  }
}

// Register-tiled variant: a thread owns 4 consecutive pixels x 16 output planes, so one broadcast
// 16-byte weight read feeds 16 FMAs instead of 4.  (Measured: the one-pixel kernel is bound by its
// shared-memory reads -- a warp-wide LDS.128 costs four LSU cycles even when every lane reads the
// same address -- and doubling its occupancy changed nothing.)  Tiles of 128 pixels, the cat
// column block [2D][128] staged once per tile; same summation order per output as the other
// gate kernels.  Requires HW % 4 == 0.
constexpr int GT4_TP = 128;
inline size_t gate4_smem_bytes(int D) {
  return ((size_t)2 * D * gate_row_pitch(D) + (size_t)2 * D * GT4_TP) * sizeof(float);
}
__global__ void __launch_bounds__(512)
gate_tile4_kernel(const float* __restrict__ ls, const float* __restrict__ lm,
                  const float* __restrict__ wT_g, float* __restrict__ cost, int D, int HW,
                  ZExpand zm) {
  extern __shared__ float gsm[];
  const int ng = (D + GT_PG - 1) / GT_PG, DP = ng * GT_PG;
  float* wT = gsm;                                   // [2D][DP]
  float4* cat4 = reinterpret_cast<float4*>(gsm + (size_t)2 * D * DP);   // [2D][32] float4
  const int nthreads = blockDim.x;                   // 32 * ng
  {
    const float4* src = reinterpret_cast<const float4*>(wT_g);
    float4* dst = reinterpret_cast<float4*>(wT);
    for (int i = threadIdx.x; i < 2 * D * DP / 4; i += nthreads) dst[i] = __ldg(src + i);
  }
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int ntiles = (HW + GT4_TP - 1) / GT4_TP;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int p0 = tile * GT4_TP;
    __syncthreads();   // previous tile's columns consumed (and wT written, first time)
    for (int i = threadIdx.x; i < 2 * D * 32; i += nthreads) {
      const int j = i >> 5, q = i & 31, p = p0 + 4 * q;
      const float* row = j < D ? ls + (long long)j * HW : lm + (long long)zexpand(zm, j - D) * HW;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (p < HW) v = __ldg(reinterpret_cast<const float4*>(row + p));   // HW % 4 == 0
      cat4[i] = v;
    }
    __syncthreads();
    float a[GT_PG][4];
#pragma unroll
    for (int k = 0; k < GT_PG; ++k) a[k][0] = a[k][1] = a[k][2] = a[k][3] = 0.f;
    const float4* wrow = reinterpret_cast<const float4*>(wT + g * GT_PG);
#pragma unroll 2
    for (int j = 0; j < 2 * D; ++j) {
      const float4 c = cat4[j * 32 + lane];
      const float4* w4 = wrow + (size_t)j * (DP / 4);
#pragma unroll
      for (int q = 0; q < GT_PG / 4; ++q) {
        const float4 w = w4[q];
        const float wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          a[4 * q + r][0] = fmaf(wv[r], c.x, a[4 * q + r][0]);
          a[4 * q + r][1] = fmaf(wv[r], c.y, a[4 * q + r][1]);
          a[4 * q + r][2] = fmaf(wv[r], c.z, a[4 * q + r][2]);
          a[4 * q + r][3] = fmaf(wv[r], c.w, a[4 * q + r][3]);
        }
      }
    }
    const int p = p0 + 4 * lane;
    if (p < HW) {
#pragma unroll
      for (int k = 0; k < GT_PG; ++k) {
        const int d = g * GT_PG + k;
        if (d < D) {
          const float4 sv = cat4[d * 32 + lane], mv = cat4[(D + d) * 32 + lane];
          float4 o;
          float wgt = 1.f / (1.f + __expf(-a[k][0]));
          o.x = wgt * sv.x + (1.f - wgt) * mv.x;
          wgt = 1.f / (1.f + __expf(-a[k][1]));
          o.y = wgt * sv.y + (1.f - wgt) * mv.y;
          wgt = 1.f / (1.f + __expf(-a[k][2]));
          o.z = wgt * sv.z + (1.f - wgt) * mv.z;
          wgt = 1.f / (1.f + __expf(-a[k][3]));
          o.w = wgt * sv.w + (1.f - wgt) * mv.w;
          *reinterpret_cast<float4*>(cost + (long long)d * HW + p) = o;
        }
      }
    }
  }
}

}  // namespace dfm
