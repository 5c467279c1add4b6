// CUDA-core (fp32) kernels of the DfM path: layout changes, the generic 3x3x3
// conv / transposed conv with fused input transform, GroupNorm statistics, the
// residual "materialise" pass, the 32->1 logit conv, the mono/stereo gate, the
// DepthHead, the cost-volume materialiser (parity op) and multi-view lifting.
//
// The fp32 conv here is the bring-up / cross-check implementation (DFM_CONV_SIMT);
// the tensor-core implementation lives in conv_tc.cuh.
#pragma once
#include "common.cuh"

namespace dfm {

// ---------------------------------------------------------------------------------
// NCHW [C][HW] -> NHWC [HW][C]   (stereo features arrive NCHW from the 2-D neck)
// ---------------------------------------------------------------------------------
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out,
                                    int C, long long HW) {
  __shared__ float tile[32][33];
  const long long p0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j;
    const long long p = p0 + tx;
    tile[j][tx] = (c < C && p < HW) ? in[(long long)c * HW + p] : 0.f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const long long p = p0 + j;
    const int c = c0 + tx;
    if (p < HW && c < C) out[p * C + c] = tile[tx][j];
  }
}

// Vectorised variant for C = 32 / 64 and HW % 4 == 0: 16-byte global accesses on both sides
// (512-byte runs along the pixels in, whole channel rows out), a [C][128 + 1] tile whose odd
// pitch keeps both the (4 rows x 8 float4) store pattern and the (4 pixels x 8 channel
// quads) gather pattern free of bank conflicts.  blockIdx.y walks a batch of images.
template <int C>
__device__ __forceinline__ void nchw_to_nhwc_v4_tile(const float* __restrict__ src,
                                                     float* __restrict__ dst, long long HW) {
  constexpr int TP = 128, P = TP + 1;
  __shared__ float tile[C * P];
  const long long p0 = (long long)blockIdx.x * TP;
  const int tid = threadIdx.x;
#pragma unroll
  for (int i = tid; i < C * (TP / 4); i += 256) {
    const int q8 = i & 7, r = (i >> 3) & 3, blk = i >> 5;
    const int colgrp = blk % (TP / 32), rowgrp = blk / (TP / 32);
    const int c = rowgrp * 4 + r, px = (colgrp * 8 + q8) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p0 + px < HW) v = __ldcs(reinterpret_cast<const float4*>(src + (long long)c * HW + p0 + px));
    float* t = tile + c * P + px;
    t[0] = v.x; t[1] = v.y; t[2] = v.z; t[3] = v.w;
  }
  __syncthreads();
#pragma unroll
  for (int i = tid; i < TP * (C / 4); i += 256) {
    const int cq8 = i & 7, px4 = (i >> 3) & 3, blk = i >> 5;
    const int cgrp = blk % (C / 32), pgrp = blk / (C / 32);
    const int c = (cgrp * 8 + cq8) * 4, px = pgrp * 4 + px4;
    if (p0 + px < HW) {
      const float* t = tile + c * P + px;
      *reinterpret_cast<float4*>(dst + (p0 + px) * C + c) = make_float4(t[0], t[P], t[2 * P], t[3 * P]);
    }
  }
}

template <int C>
__global__ void __launch_bounds__(256)
nchw_to_nhwc_v4_kernel(const float* __restrict__ in, float* __restrict__ out, long long HW,
                       long long in_bstride, long long out_bstride) {
  nchw_to_nhwc_v4_tile<C>(in + (long long)blockIdx.y * in_bstride,
                          out + (long long)blockIdx.y * out_bstride, HW);
}

// The same transpose of up to 16 separately allocated images (multi-view lifting's views,
// some of them held by a feature cache): blockIdx.y indexes the pointer table.
struct ViewTable {
  const float* p[16];
};
template <int C>
__global__ void __launch_bounds__(256)
nchw_to_nhwc_v4_views_kernel(ViewTable in, float* __restrict__ out, long long HW,
                             long long out_bstride) {
  nchw_to_nhwc_v4_tile<C>(in.p[blockIdx.y], out + (long long)blockIdx.y * out_bstride, HW);
}

// channels-last [V][C] -> NCDHW [C][V]
__global__ void cl_to_ncdhw_kernel(const float* __restrict__ in, float* __restrict__ out,
                                   int C, long long V) {
  __shared__ float tile[32][33];
  const long long v0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int j = ty; j < 32; j += 8) {
    const long long v = v0 + j;
    const int c = c0 + tx;
    tile[j][tx] = (v < V && c < C) ? in[v * C + c] : 0.f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j;
    const long long v = v0 + tx;
    if (c < C && v < V) out[(long long)c * V + v] = tile[tx][j];
  }
}

// ---------------------------------------------------------------------------------
// Input loaders for the SIMT conv: value of (input voxel, channel) after the fused
// transform.  Bounds are checked by the caller.
// ---------------------------------------------------------------------------------
struct SrcLoader {
  Src s;
  int C, Hi, Wi;
  __device__ __forceinline__ float load(int z, int y, int x, int c) const {
    return load_src(s, z, (long long)y * Wi + x, (long long)Hi * Wi, C, c);
  }
};

// First layer: the plane-sweep volume computed on the fly (never stored).
// channels [0,C) = cur feature at the stride lattice, [C,2C) = prev feature warped
// onto plane z.  `first` selects the channel window start (0, or C for prev only).
struct WarpLoader {
  const float* cur;   // NHWC
  const float* prev;  // NHWC
  const float* depths;
  WarpGeom g;
  int C;      // channels per frame
  int first;  // channel offset into the 2C-channel volume
  __device__ __forceinline__ float load(int z, int y, int x, int c) const {
    c += first;
    if (c < C)
      return __ldg(cur + ((long long)(y * g.step) * g.Wf + x * g.step) * C + c);
    c -= C;
    float fx, fy;
    warp_coord(g, x, y, __ldg(depths + z), fx, fy);
    const Taps t = bilinear_taps(fx, fy, g.Hf, g.Wf);
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (t.w[i] != 0.f) v = fmaf(t.w[i], __ldg(prev + (long long)t.off[i] * C + c), v);
    return v;
  }
};

// ---------------------------------------------------------------------------------
// Generic fp32 3x3x3 conv / stride-2 transposed conv, channels-last in and out.
// One warp owns VOX consecutive output voxels; lane = output channel (mod 32).
// Weights packed [27][Cin][Cout].
// ---------------------------------------------------------------------------------
template <int CIN, int COUT, class Loader>
__global__ void __launch_bounds__(256)
conv3d_simt_kernel(Loader ld, const float* __restrict__ wp, float* __restrict__ out,
                   ConvGeom g) {
  constexpr int VOX = 8;
  constexpr int CI = (CIN + 31) / 32, CO = (COUT + 31) / 32;
  const int lane = threadIdx.x & 31;
  const long long warp_id = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nout = (long long)g.Do * g.Ho * g.Wo;
  const long long v0 = warp_id * VOX;
  if (v0 >= nout) return;

  int zo[VOX], yo[VOX], xo[VOX];
  bool vv[VOX];
#pragma unroll
  for (int v = 0; v < VOX; ++v) {
    const long long idx = v0 + v;
    vv[v] = idx < nout;
    const long long i2 = vv[v] ? idx : 0;
    xo[v] = (int)(i2 % g.Wo);
    yo[v] = (int)((i2 / g.Wo) % g.Ho);
    zo[v] = (int)(i2 / ((long long)g.Wo * g.Ho));
  }
  float acc[CO][VOX];
#pragma unroll
  for (int j = 0; j < CO; ++j)
#pragma unroll
    for (int v = 0; v < VOX; ++v) acc[j][v] = 0.f;

  for (int tap = 0; tap < 27; ++tap) {
    const int kz = tap / 9, ky = (tap / 3) % 3, kx = tap % 3;
    float xin[CI][VOX];
    bool any = false;
#pragma unroll
    for (int v = 0; v < VOX; ++v) {
      int zi, yi, xi;
      bool ok = vv[v];
      if (!g.transposed) {
        zi = zo[v] * g.sd + kz - g.pd;
        yi = yo[v] * g.sh + ky - g.ph;
        xi = xo[v] * g.sw + kx - g.pw;
      } else {  // o = 2 i - 1 + k  =>  i = (o + 1 - k) / 2 when even
        const int tz = zo[v] + 1 - kz, ty = yo[v] + 1 - ky, tx = xo[v] + 1 - kx;
        ok = ok && !((tz | ty | tx) & 1) && tz >= 0 && ty >= 0 && tx >= 0;
        zi = tz >> 1;
        yi = ty >> 1;
        xi = tx >> 1;
      }
      ok = ok && zi >= 0 && zi < g.Di && yi >= 0 && yi < g.Hi && xi >= 0 && xi < g.Wi;
      any |= ok;
#pragma unroll
      for (int j = 0; j < CI; ++j) {
        const int c = lane + 32 * j;
        xin[j][v] = (ok && c < CIN) ? ld.load(zi, yi, xi, c) : 0.f;
      }
    }
    if (!any) continue;  // warp-uniform
    const float* wt = wp + (long long)tap * CIN * COUT;
#pragma unroll
    for (int j = 0; j < CI; ++j) {
#pragma unroll 8
      for (int l = 0; l < 32; ++l) {
        const int ci = j * 32 + l;
        if (ci >= CIN) break;
        float wv[CO];
#pragma unroll
        for (int jo = 0; jo < CO; ++jo) {
          const int co = lane + 32 * jo;
          wv[jo] = co < COUT ? __ldg(wt + (long long)ci * COUT + co) : 0.f;
        }
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
#pragma unroll
    for (int jo = 0; jo < CO; ++jo) {
      const int co = lane + 32 * jo;
      if (co < COUT) out[(v0 + v) * COUT + co] = acc[jo][v];
    }
  }
}

// ---------------------------------------------------------------------------------
// Per-channel sum / sum-of-squares of a channels-last tensor (GroupNorm statistics,
// nn.GroupNorm(32, C): conv_modules.py:42-43).  fp64 accumulation across blocks.
// ---------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(256)
channel_stats_kernel(const float* __restrict__ x, long long V, double* __restrict__ sums) {
  constexpr int ROWS = 256 / C;  // voxels per block-iteration
  __shared__ double sh[2][256];
  const int c = threadIdx.x % C, r = threadIdx.x / C;
  double s = 0.0, ss = 0.0;
  for (long long v = (long long)blockIdx.x * ROWS + r; v < V; v += (long long)gridDim.x * ROWS) {
    const float a = x[v * C + c];
    s += a;
    ss += (double)a * a;
  }
  sh[0][threadIdx.x] = s;
  sh[1][threadIdx.x] = ss;
  __syncthreads();
  if (r == 0) {
    for (int k = 1; k < ROWS; ++k) {
      s += sh[0][k * C + c];
      ss += sh[1][k * C + c];
    }
    atomicAdd(sums + 2 * c, s);
    atomicAdd(sums + 2 * c + 1, ss);
  }
}

// Statistics of a z-class-compressed tensor [3][HW][C] that stands for D planes
// (plane 0 once, plane 1 D-2 times, plane 2 once).
// grid (blocks per plane, 3): blockIdx.y is the class plane, so the weight is a per-block
// constant; fp32 partial sums per thread are short (<= HW / (gridDim.x * ROWS) values), fp64
// across threads.
template <int C>
__global__ void __launch_bounds__(256)
channel_stats_zcls_kernel(const float* __restrict__ x, int HW, int D,
                          double* __restrict__ sums) {
  constexpr int ROWS = 256 / C;
  __shared__ double sh[2][256];
  const int c = threadIdx.x % C, r = threadIdx.x / C;
  const float* xp = x + (long long)blockIdx.y * HW * C;
  float s = 0.f, ss = 0.f;
  for (int v = blockIdx.x * ROWS + r; v < HW; v += gridDim.x * ROWS) {
    const float a = xp[(long long)v * C + c];
    s += a;
    ss = fmaf(a, a, ss);
  }
  const double wgt = blockIdx.y == 1 ? (double)(D - 2) : 1.0;
  sh[0][threadIdx.x] = wgt * s;
  sh[1][threadIdx.x] = wgt * ss;
  __syncthreads();
  if (r == 0) {
    double ds = sh[0][c], dss = sh[1][c];
    for (int k = 1; k < ROWS; ++k) {
      ds += sh[0][k * C + c];
      dss += sh[1][k * C + c];
    }
    atomicAdd(sums + 2 * c, ds);
    atomicAdd(sums + 2 * c + 1, dss);
  }
}

// planes 0, 2, 4 of a 5-plane conv output -> the 3-plane class tensor (grid.y = class plane,
// 16-byte copies; plane_elems % 4 == 0)
__global__ void pick_planes_kernel(const float* __restrict__ in, float* __restrict__ out,
                                   long long plane_elems) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= plane_elems) return;
  const long long pl = blockIdx.y;
  *reinterpret_cast<float4*>(out + pl * plane_elems + i) =
      __ldg(reinterpret_cast<const float4*>(in + 2 * pl * plane_elems + i));
}

// scale/shift of GroupNorm(groups, C) from per-channel sums over `count` voxels:
// y = (x - mean_g) * rstd_g * gamma[c] + beta[c]  ==  x * scale[c] + shift[c]
// The sums are zeroed once consumed, so the next frame's conv epilogues accumulate into clean
// buffers without a memset node per layer in the stream.
__global__ void gn_finalize_kernel(double* __restrict__ sums, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, int C, int groups,
                                   double count, float eps, float* __restrict__ scale,
                                   float* __restrict__ shift) {
  const int c = threadIdx.x;
  const int cpg = C / groups, g = (c < C ? c : 0) / cpg;
  double s = 0.0, ss = 0.0;
  for (int k = 0; k < cpg; ++k) {
    s += sums[2 * (g * cpg + k)];
    ss += sums[2 * (g * cpg + k) + 1];
  }
  __syncthreads();  // every group member has read its group's sums
  if (c >= C) return;
  sums[2 * c] = 0.0;
  sums[2 * c + 1] = 0.0;
  const double n = count * cpg;
  const double mean = s / n;
  double var = ss / n - mean * mean;
  if (var < 0.0) var = 0.0;
  const double rstd = 1.0 / sqrt(var + (double)eps);
  const double sc = (double)gamma[c] * rstd;
  scale[c] = (float)sc;
  shift[c] = (float)((double)beta[c] - mean * sc);
}

// ---------------------------------------------------------------------------------
// Materialise a (<= 3 term) sum as a channels-last tensor and/or NCDHW output:
// cur_cost = cost0 + hourglass(cost0)  (dfm_backbone.py:176-183).
// ---------------------------------------------------------------------------------
// z expansion of a tensor that was computed on a shortened volume.  Away from the two z
// ends the mono tower is invariant under shifts by 4 planes (two stride-2 levels), so a full
// plane z reads source plane z (head), z - shift (tail) or the interior plane of the same
// phase, mid + (z - head) mod 4.
struct ZExpand {
  int head;   // planes [0, head) map to themselves
  int tail0;  // planes [tail0, D) map to z - shift
  int shift;
  int mid;
};
__device__ __forceinline__ int zexpand(const ZExpand& e, int z) {
  return z < e.head ? z : (z >= e.tail0 ? z - e.shift : e.mid + ((z - e.head) & 3));
}

__global__ void __launch_bounds__(256)
materialize_kernel(Src s, int C, long long V, long long HW, ZExpand ze, float* __restrict__ out_cl,
                   float* __restrict__ out_ncdhw) {
  __shared__ float tile[32][33];
  const long long v0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  for (int j = ty; j < 32; j += 8) {
    const long long v = v0 + j;
    const int c = c0 + tx;
    float val = 0.f;
    if (v < V && c < C) {
      val = load_src(s, zexpand(ze, (int)(v / HW)), v % HW, HW, C, c);
      if (out_cl) out_cl[v * C + c] = val;
    }
    tile[j][tx] = val;
  }
  if (!out_ncdhw) return;
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j;
    const long long v = v0 + tx;
    if (c < C && v < V) out_ncdhw[(long long)c * V + v] = tile[tx][j];
  }
}

// Vectorised variant for C == 32: a block walks tiles of 128 voxels.  256 threads = 32 voxels x
// 8 channel quads, four voxel groups per tile (12 independent 16-byte loads in flight per
// thread); the per-channel affine parameters of a thread's quad live in registers, loads and
// channels-last stores are float4.  The NCDHW copy goes through a [32][128 + 1] shared-memory
// transpose (odd pitch: both the quad-wise stores and the voxel-wise reads are conflict-free)
// and leaves as 512-byte runs per channel.
constexpr int MAT_TV = 128;
__global__ void __launch_bounds__(256)
materialize32_kernel(Src s, int V, int HW, ZExpand ze, float* __restrict__ out_cl,
                     float* __restrict__ out_ncdhw) {
  constexpr int C = 32, P = MAT_TV + 1;
  __shared__ float tile[C * P];
  const int q = threadIdx.x & 7, vl = threadIdx.x >> 3;
  float4 sc[3], sh[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    sc[i] = make_float4(1.f, 1.f, 1.f, 1.f);
    sh[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < s.n && s.t[i].scale) {
      sc[i] = __ldg(reinterpret_cast<const float4*>(s.t[i].scale) + q);
      sh[i] = __ldg(reinterpret_cast<const float4*>(s.t[i].shift) + q);
    }
  }
  const int ntiles = (V + MAT_TV - 1) / MAT_TV;
  for (int tile_i = blockIdx.x; tile_i < ntiles; tile_i += gridDim.x) {
    float4 raw[4][3];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const int v = tile_i * MAT_TV + g * 32 + vl;
      if (v < V) {
        const int z = zexpand(ze, v / HW), pos = v % HW;
#pragma unroll
        for (int i = 0; i < 3; ++i)
          if (i < s.n)
            raw[g][i] = __ldg(reinterpret_cast<const float4*>(
                s.t[i].x + ((long long)term_plane(s.t[i], z) * HW + pos) * C + 4 * q));
      }
    }
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const int v = tile_i * MAT_TV + g * 32 + vl;
      float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
      if (v < V) {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          if (i < s.n) {
            float4 a = raw[g][i];
            a.x = fmaf(a.x, sc[i].x, sh[i].x);
            a.y = fmaf(a.y, sc[i].y, sh[i].y);
            a.z = fmaf(a.z, sc[i].z, sh[i].z);
            a.w = fmaf(a.w, sc[i].w, sh[i].w);
            if (s.t[i].relu) {
              a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f);
              a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f);
            }
            val.x += a.x; val.y += a.y; val.z += a.z; val.w += a.w;
          }
        }
        if (s.outer_relu) {
          val.x = fmaxf(val.x, 0.f); val.y = fmaxf(val.y, 0.f);
          val.z = fmaxf(val.z, 0.f); val.w = fmaxf(val.w, 0.f);
        }
        if (out_cl) *reinterpret_cast<float4*>(out_cl + (long long)v * C + 4 * q) = val;
      }
      if (out_ncdhw) {
        float* t = tile + (4 * q) * P + g * 32 + vl;
        t[0] = val.x; t[P] = val.y; t[2 * P] = val.z; t[3 * P] = val.w;
      }
    }
    if (out_ncdhw) {
      __syncthreads();
      const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;   // warp w: channels w, w+8, ...
      const int vbase = tile_i * MAT_TV;
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
        const int c = w + 8 * cc;
        float* dst = out_ncdhw + (long long)c * V + vbase;
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (vbase + k * 32 + lane < V) __stcs(dst + k * 32 + lane, tile[c * P + k * 32 + lane]);
      }
      __syncthreads();
    }
  }
}

// ---------------------------------------------------------------------------------
// 3x3x3 conv C -> 1 (nn.Conv3d(cv, 1, 3, 1, 1, bias=False), dfm_backbone.py:128).
// 8 lanes per output voxel, each lane owns 4 of the 32 input channels.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
conv3d_c32_to_1_kernel(Src s, const float* __restrict__ w /*[27][32]*/, float* __restrict__ out,
                       int D, int H, int W) {
  __shared__ float ws[27 * 32];
  for (int i = threadIdx.x; i < 27 * 32; i += blockDim.x) ws[i] = w[i];
  __syncthreads();
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long vox = gid >> 3;
  const int sub = (int)(gid & 7);
  const long long V = (long long)D * H * W;
  const bool live = vox < V;
  const long long vq = live ? vox : 0;
  const int x = (int)(vq % W), y = (int)((vq / W) % H), z = (int)(vq / ((long long)W * H));
  float acc = 0.f;
  for (int tap = 0; tap < 27; ++tap) {
    const int zi = z + tap / 9 - 1, yi = y + (tap / 3) % 3 - 1, xi = x + tap % 3 - 1;
    if (!live || zi < 0 || zi >= D || yi < 0 || yi >= H || xi < 0 || xi >= W) continue;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = sub * 4 + k;
      acc = fmaf(load_src(s, zi, (long long)yi * W + xi, (long long)H * W, 32, c),
                 ws[tap * 32 + c], acc);
    }
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  acc += __shfl_xor_sync(0xffffffffu, acc, 4);
  if (live && sub == 0) out[vox] = acc;
}

// ---------------------------------------------------------------------------------
// mono/stereo gate (dfm_backbone.py:135-141): cat the two [D] logit columns of a pixel,
// 1x1 conv (2D -> D), sigmoid, blend.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
gate_kernel(const float* __restrict__ ls, const float* __restrict__ lm,
            const float* __restrict__ wagg /*[D][2D]*/, float* __restrict__ cost, int D,
            int HW, ZExpand zm /* z expansion of the mono logits */) {
  extern __shared__ float cat[];  // [2D][32]
  const int p0 = blockIdx.x * 32;
  const int px = threadIdx.x & 31, dg = threadIdx.x >> 5;
  for (int j = dg; j < 2 * D; j += 4) {
    const int p = p0 + px;
    float v = 0.f;
    if (p < HW)
      v = j < D ? ls[(long long)j * HW + p] : lm[(long long)zexpand(zm, j - D) * HW + p];
    cat[j * 32 + px] = v;
  }
  __syncthreads();
  const int p = p0 + px;
  // each warp owns output planes d = dg, dg+4, ...; four of them at a time so the four
  // dot products give independent FMA chains (the weight row reads are warp-uniform)
  for (int d0 = dg; d0 < D; d0 += 16) {
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    const float* wr[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) wr[k] = wagg + (long long)min(d0 + 4 * k, D - 1) * 2 * D;
    for (int j = 0; j < 2 * D; ++j) {
      const float c = cat[j * 32 + px];
#pragma unroll
      for (int k = 0; k < 4; ++k) a[k] = fmaf(__ldg(wr[k] + j), c, a[k]);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int d = d0 + 4 * k;
      if (d < D && p < HW) {
        const float wgt = 1.f / (1.f + __expf(-a[k]));
        const float sv = cat[d * 32 + px], mv = cat[(D + d) * 32 + px];
        cost[(long long)d * HW + p] = wgt * sv + (1.f - wgt) * mv;
      }
    }
  }
}

// ---------------------------------------------------------------------------------
// DepthHead.forward (depth_head.py:190-212): x`f` trilinear upsample with
// align_corners=True, softmax over depth, expectation.  One thread per full-res pixel;
// the (y,x)-interpolated logit column is rebuilt on the fly from the low-res logits
// (L2-resident), the two optional 4-D outputs are written coalesced along x.
// ---------------------------------------------------------------------------------
__device__ __forceinline__ float dh_plane(const float* __restrict__ c, long long zoff,
                                          const int o[4], const float w[4]) {
  // same association as ATen upsample_trilinear3d:
  // h0*(w0*v00 + w1*v01) + h1*(w0*v10 + w1*v11)
  return w[2] * (w[0] * __ldg(c + zoff + o[0]) + w[1] * __ldg(c + zoff + o[1])) +
         w[3] * (w[0] * __ldg(c + zoff + o[2]) + w[1] * __ldg(c + zoff + o[3]));
}

// DH_ZS threads share one pixel: each owns a contiguous range of the depth axis (its share of
// the low-res planes for the maximum, of the upsampled bins for the sums and the writes), so
// the serial per-pixel loops are DH_ZS times shorter and the grid DH_ZS times larger.
constexpr int DH_ZS = 4;
constexpr int DH_MAXBINS = 1024;  // bins (f * D) whose interpolation table fits in shared memory
__host__ __device__ inline int dh_ncols(int f) { return 32 / f + 3; }
inline size_t dh_smem_bytes(int D, int f) { return (size_t)D * 2 * dh_ncols(f) * sizeof(float); }
__global__ void __launch_bounds__(32 * DH_ZS)
depth_head_kernel(const float* __restrict__ cost, const float* __restrict__ samples, int D,
                  int Ho, int Wo, int f, float* __restrict__ vol, float* __restrict__ sm,
                  float* __restrict__ preds, float2* __restrict__ norm = nullptr) {
  // the two low-res rows (y0, y1) x the <= 32/f + 3 low-res columns this block of 32 pixels
  // interpolates between, all D planes: [D][2][nc].  Staged once per block -- every thread
  // fetching its four corners per plane from global memory made the kernel L1-wavefront bound.
  extern __shared__ float dh_cols[];
  __shared__ float red[3][DH_ZS][32];
  // per upsampled bin k: low-res plane z0 = floor(sz * k), weight of plane z0 + 1, and the bin's
  // depth.  Tabulated once per block: the int<->float conversions of computing them per
  // (pixel, bin) run at a quarter of the FMA rate and dominated the reduction pass.
  __shared__ int tab_z0[DH_MAXBINS];
  __shared__ float tab_l1[DH_MAXBINS], tab_s[DH_MAXBINS];
  const int OW = Wo * f, OH = Ho * f, OD = D * f;
  const int tx = threadIdx.x, seg = threadIdx.y;
  const float sz = OD > 1 ? (float)(D - 1) / (OD - 1) : 0.f;
  for (int k = seg * 32 + tx; k < OD; k += 32 * DH_ZS) {
    const float fz = sz * k;
    const int z0 = (int)fz;
    tab_z0[k] = z0;
    tab_l1[k] = fz - z0;
    tab_s[k] = samples ? __ldg(samples + k) : 0.f;
  }
  const int Xr = blockIdx.x * 32 + tx;
  const bool live = Xr < OW;
  const int X = live ? Xr : OW - 1;
  const int Y = blockIdx.y;
  const float sx = OW > 1 ? (float)(Wo - 1) / (OW - 1) : 0.f;
  const float sy = OH > 1 ? (float)(Ho - 1) / (OH - 1) : 0.f;
  const float fx = sx * X, fy = sy * Y;
  const int x0 = (int)fx, y0 = (int)fy;
  const int x1 = x0 + (x0 < Wo - 1 ? 1 : 0), y1 = y0 + (y0 < Ho - 1 ? 1 : 0);
  const float lx1 = fx - x0, ly1 = fy - y0;
  const float w[4] = {1.f - lx1, lx1, 1.f - ly1, ly1};
  const long long plane = (long long)Ho * Wo;
  const long long opix = (long long)Y * OW + X, oplane = (long long)OH * OW;
  const int nc = dh_ncols(f);
  const int xb = (int)(sx * (blockIdx.x * 32));  // first low-res column of the block
  for (int i = seg * 32 + tx; i < D * 2 * nc; i += 32 * DH_ZS) {
    const int z = i / (2 * nc), rc = i - z * 2 * nc;
    const int r = rc >= nc ? 1 : 0, c = rc - r * nc;
    dh_cols[i] = __ldg(cost + z * plane + (r ? y1 : y0) * Wo + min(xb + c, Wo - 1));
  }
  __syncthreads();
  const int c0 = x0 - xb, c1 = x1 - xb;
  // same association as ATen upsample_trilinear3d:
  // h0*(w0*v00 + w1*v01) + h1*(w0*v10 + w1*v11)
  auto col = [&](int z) {
    const float* pz = dh_cols + z * 2 * nc;
    return w[2] * (w[0] * pz[c0] + w[1] * pz[c1]) + w[3] * (w[0] * pz[nc + c0] + w[1] * pz[nc + c1]);
  };

  // The upsampled column is piecewise linear in k between the low-res planes, so its maximum
  // is the maximum of the D (y,x)-interpolated low-res values: no online-softmax rescaling.
  float m = -INFINITY;
  for (int z = seg * D / DH_ZS; z < (seg + 1) * D / DH_ZS; ++z) m = fmaxf(m, col(z));
  red[0][seg][tx] = m;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < DH_ZS; ++i) m = fmaxf(m, red[0][i][tx]);
  // pass 1: sum of exponentials and the expectation over this thread's bins
  const int k_lo = seg * OD / DH_ZS, k_hi = (seg + 1) * OD / DH_ZS;
  float ssum = 0.f, esum = 0.f;
  int zc = -1;
  float b0 = 0.f, b1 = 0.f;
  for (int k = k_lo; k < k_hi; ++k) {
    const int z0 = tab_z0[k];
    const float lz1 = tab_l1[k];
    if (z0 != zc) {
      b0 = (z0 == zc + 1 && zc >= 0) ? b1 : col(z0);
      b1 = z0 < D - 1 ? col(z0 + 1) : b0;
      zc = z0;
    }
    const float v = (1.f - lz1) * b0 + lz1 * b1;
    const float e = __expf(v - m);
    ssum += e;
    esum = fmaf(e, tab_s[k], esum);
  }
  red[1][seg][tx] = ssum;
  red[2][seg][tx] = esum;
  __syncthreads();
  ssum = esum = 0.f;
#pragma unroll
  for (int i = 0; i < DH_ZS; ++i) {
    ssum += red[1][i][tx];
    esum += red[2][i][tx];
  }
  if (!live) return;
  if (seg == 0) {
    if (preds) preds[opix] = esum / ssum;
    // (max, 1 / sum of exponentials) per pixel: lets a consumer evaluate any softmax value
    // from the low-res logits without the full-resolution volume (frustum_kernels.cuh)
    if (norm) norm[opix] = make_float2(m, 1.f / ssum);
  }
  if (!sm && !vol) return;
  // pass 2: the two 4-D outputs
  const float inv = 1.f / ssum;
  zc = -1;
  for (int k = k_lo; k < k_hi; ++k) {
    const int z0 = tab_z0[k];
    const float lz1 = tab_l1[k];
    if (z0 != zc) {
      b0 = (z0 == zc + 1 && zc >= 0) ? b1 : col(z0);
      b1 = z0 < D - 1 ? col(z0 + 1) : b0;
      zc = z0;
    }
    const float v = (1.f - lz1) * b0 + lz1 * b1;
    if (vol) vol[k * oplane + opix] = v;
    if (sm) sm[k * oplane + opix] = __expf(v - m) * inv;
  }
}

// ---------------------------------------------------------------------------------
// build_dfm_cost materialised as the reference's NCDHW volume (parity op only).
// One thread per (voxel, channel); writes are coalesced along x.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
cost_volume_kernel(WarpLoader ld, int D, int Ho, int Wo, float* __restrict__ out) {
  const long long V = (long long)D * Ho * Wo;
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int c = blockIdx.y;
  if (gid >= V) return;
  const int x = (int)(gid % Wo), y = (int)((gid / Wo) % Ho), z = (int)(gid / ((long long)Wo * Ho));
  out[(long long)c * V + gid] = ld.load(z, y, x, c);
}

// ---------------------------------------------------------------------------------
// Multi-view lifting (multiview_dfm.py:139-209 + point_fusion.py:57-106, nearest tap,
// valid mask, per-frame valid-count, temporal mean / concat).  One warp per voxel,
// lane = channel (C = 64 -> 2 per lane).  feats are NHWC per (frame, view); output layout
// [C_out][Nx][Ny][Nz] with C_out index f*C + c for 'concat'.
// ---------------------------------------------------------------------------------
struct LiftParams {
  float proj[16][16];  // up to 16 (frame, view) matrices, row-major 4x4
  int img_w[16];
  int T, Nv, C, Hf, Wf;
  int nx, ny, nz;
  float scale_x, scale_y, crop_x, crop_y;
  int flip, in_h, in_w, concat;
};

// points_cam2img + scale/crop of point_sample (structures/utils.py:199-214,
// point_fusion.py:63-69) with the reference's rounding sequence spelled out: the fp32
// [N,4] x [4,4]^T product accumulates k = 0..3 with one fused multiply-add per step (what
// the CPU GEMM micro-kernel does; checked bit-for-bit against torch.matmul), the perspective
// divide, the scale multiply and the crop subtraction round separately.  Nearest-tap
// sampling is discontinuous, so letting nvcc contract these into different FMAs moves
// voxels that project onto a rounding tie to the neighbouring tap.
__device__ __forceinline__ void lift_project(const float* m, float px, float py, float pz,
                                             float sx, float sy, float crx, float cry,
                                             float& cx, float& cy, float& d) {
  const float a = __fadd_rn(__fmaf_rn(pz, m[2], __fmaf_rn(py, m[1], __fmul_rn(px, m[0]))), m[3]);
  const float b = __fadd_rn(__fmaf_rn(pz, m[6], __fmaf_rn(py, m[5], __fmul_rn(px, m[4]))), m[7]);
  d = __fadd_rn(__fmaf_rn(pz, m[10], __fmaf_rn(py, m[9], __fmul_rn(px, m[8]))), m[11]);
  cx = __fsub_rn(__fmul_rn(__fdiv_rn(a, d), sx), crx);
  cy = __fsub_rn(__fmul_rn(__fdiv_rn(b, d), sy), cry);
}

__device__ __forceinline__ int nearest_index(float coord, int size, float norm_size) {
  // grid_sample(mode='nearest', align_corners=True): unnormalise then nearbyint
  // norm = coord / size * 2 - 1 (point_fusion.py:82-83); ATen unnormalises with
  // ((g + 1) / 2) * (size - 1); the *2 and /2 are exact, the rest rounds once per step
  const float g = __fsub_rn(__fmul_rn(__fdiv_rn(coord, norm_size), 2.f), 1.f);
  const float ix = __fmul_rn(__fmul_rn(__fadd_rn(g, 1.f), 0.5f), (float)(size - 1));
  return (int)nearbyintf(ix);
}

__global__ void __launch_bounds__(256)
lift_kernel(LiftParams p, const float* __restrict__ feats, const float* __restrict__ xs,
            const float* __restrict__ ys, const float* __restrict__ zs, float* __restrict__ out) {
  const long long nvox = (long long)p.nx * p.ny * p.nz;
  const long long vox = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (vox >= nvox) return;
  // anchor order: z-major, then y, then x fastest (reshape [Nz,Ny,Nx] in the caller)
  const int ix = (int)(vox % p.nx), iy = (int)((vox / p.nx) % p.ny),
            iz = (int)(vox / ((long long)p.nx * p.ny));
  const float px = __ldg(xs + ix), py = __ldg(ys + iy), pz = __ldg(zs + iz);
  const int CL = (p.C + 31) / 32;
  const long long fstride = (long long)p.C * p.Hf * p.Wf;
  const long long ovox = ((long long)ix * p.ny + iy) * p.nz + iz;  // [Nx][Ny][Nz]
  float tot[4] = {0.f, 0.f, 0.f, 0.f};
  int tot_n = 0;
  for (int f = 0; f < p.T; ++f) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    int nvalid = 0;
    for (int v = 0; v < p.Nv; ++v) {
      const int s = f * p.Nv + v;
      const float* m = p.proj[s];
      float cx, cy, d;
      lift_project(m, px, py, pz, p.scale_x, p.scale_y, p.crop_x, p.crop_y, cx, cy, d);
      if (p.flip) cx = __fsub_rn((float)p.img_w[s], cx);
      const bool valid = cx < (float)p.in_w && cx > 0.f && cy < (float)p.in_h && cy > 0.f &&
                         d > 0.f;
      if (!valid) continue;
      ++nvalid;
      const int sx = nearest_index(cx, p.Wf, (float)p.in_w);
      const int sy = nearest_index(cy, p.Hf, (float)p.in_h);
      if (sx < 0 || sx >= p.Wf || sy < 0 || sy >= p.Hf) continue;
      const float* fp = feats + s * fstride + ((long long)sy * p.Wf + sx) * p.C;  // NHWC
      for (int j = 0; j < CL; ++j) {
        const int c = lane + 32 * j;
        if (c < p.C) acc[j] += __ldg(fp + c);
      }
    }
    if (p.concat) {
      // sum / clamp(count, 1): a true division like multiview_dfm.py:194-203
      const float den = (float)max(nvalid, 1);
      for (int j = 0; j < CL; ++j) {
        const int c = lane + 32 * j;
        if (c < p.C)
          out[((long long)(f * p.C + c)) * nvox + ovox] = nvalid > 0 ? __fdiv_rn(acc[j], den) : 0.f;
      }
    } else {
      for (int j = 0; j < CL; ++j) tot[j] += nvalid > 0 ? acc[j] : 0.f;
      tot_n += nvalid;
    }
  }
  if (!p.concat) {
    const float den = (float)max(tot_n, 1);
    for (int j = 0; j < CL; ++j) {
      const int c = lane + 32 * j;
      if (c < p.C) out[(long long)c * nvox + ovox] = tot_n > 0 ? __fdiv_rn(tot[j], den) : 0.f;
    }
  }
}

// Thread-per-voxel variant for C <= 64: voxels are taken in OUTPUT order ([Nx][Ny][Nz]
// linear), every thread keeps its C running sums in registers and the final stores are
// coalesced across the warp for every channel (the warp-per-voxel kernel above writes one
// 4-byte element per 4-byte-strided channel plane).
template <int C>
__global__ void __launch_bounds__(128)
lift_voxel_kernel(LiftParams p, const float* __restrict__ feats, const float* __restrict__ xs,
                  const float* __restrict__ ys, const float* __restrict__ zs,
                  float* __restrict__ out) {
  const long long nvox = (long long)p.nx * p.ny * p.nz;
  const long long ovox = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (ovox >= nvox) return;
  const int iz = (int)(ovox % p.nz), iy = (int)((ovox / p.nz) % p.ny),
            ix = (int)(ovox / ((long long)p.nz * p.ny));
  const float px = __ldg(xs + ix), py = __ldg(ys + iy), pz = __ldg(zs + iz);
  const long long fstride = (long long)C * p.Hf * p.Wf;
  float tot[C];
#pragma unroll
  for (int c = 0; c < C; ++c) tot[c] = 0.f;
  int tot_n = 0;
  for (int f = 0; f < p.T; ++f) {
    float acc[C];
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] = 0.f;
    int nvalid = 0;
    for (int v = 0; v < p.Nv; ++v) {
      const int s = f * p.Nv + v;
      const float* m = p.proj[s];
      float cx, cy, d;
      lift_project(m, px, py, pz, p.scale_x, p.scale_y, p.crop_x, p.crop_y, cx, cy, d);
      if (p.flip) cx = __fsub_rn((float)p.img_w[s], cx);
      const bool valid = cx < (float)p.in_w && cx > 0.f && cy < (float)p.in_h && cy > 0.f &&
                         d > 0.f;
      if (!valid) continue;
      ++nvalid;
      const int sx = nearest_index(cx, p.Wf, (float)p.in_w);
      const int sy = nearest_index(cy, p.Hf, (float)p.in_h);
      if (sx < 0 || sx >= p.Wf || sy < 0 || sy >= p.Hf) continue;
      const float4* fp = reinterpret_cast<const float4*>(
          feats + s * fstride + ((long long)sy * p.Wf + sx) * C);
#pragma unroll
      for (int q = 0; q < C / 4; ++q) {
        const float4 t4 = __ldg(fp + q);
        acc[4 * q] += t4.x;
        acc[4 * q + 1] += t4.y;
        acc[4 * q + 2] += t4.z;
        acc[4 * q + 3] += t4.w;
      }
    }
    if (p.concat) {
      const float den = (float)max(nvalid, 1);  // acc is all zero when nvalid == 0
#pragma unroll
      for (int c = 0; c < C; ++c)
        out[((long long)(f * C + c)) * nvox + ovox] = __fdiv_rn(acc[c], den);
    } else {
      if (nvalid > 0) {
#pragma unroll
        for (int c = 0; c < C; ++c) tot[c] += acc[c];
      }
      tot_n += nvalid;
    }
  }
  if (!p.concat) {
    const float den = (float)max(tot_n, 1);  // tot is all zero when tot_n == 0
#pragma unroll
    for (int c = 0; c < C; ++c) out[(long long)c * nvox + ovox] = __fdiv_rn(tot[c], den);
  }
}


// Channels-last variant, one warp per 32 consecutive voxels.  Phase A (lane = voxel) runs the
// reference's projection / validity / nearest-pixel arithmetic exactly as lift_voxel_kernel does;
// phase B (lane = channel pair) gathers the 256-byte feature rows of the valid (voxel, view)
// pairs with one coalesced warp load each and writes every voxel's channels as one contiguous
// 256-byte row of out [nvox][Ctot] -- the layout the neck's conv loaders read, so neither the
// strided channel-plane stores of the NCDHW kernel nor the neck's transpose pass exist on this
// path.  Per-frame sums run over the views in the reference's order (bit-identical results).
// Requires C == 64 and (concat or T == 1).
__global__ void __launch_bounds__(256)
lift_cl_kernel(LiftParams p, const float* __restrict__ feats, const float* __restrict__ xs,
               const float* __restrict__ ys, const float* __restrict__ zs,
               float* __restrict__ out) {
  constexpr int C = 64;
  const unsigned FULL = 0xffffffffu;
  __shared__ int s_off[8][16][32];  // [warp][view][voxel]: float2 index of the sampled row, or -1
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const long long nvox = (long long)p.nx * p.ny * p.nz;
  const long long v0 = ((long long)blockIdx.x * (blockDim.x >> 5) + wib) * 32;
  if (v0 >= nvox) return;
  const bool live = v0 + lane < nvox;
  const long long ovox = min(v0 + lane, nvox - 1);
  const int iz = (int)(ovox % p.nz), iy = (int)((ovox / p.nz) % p.ny),
            ix = (int)(ovox / ((long long)p.nz * p.ny));
  const float px = __ldg(xs + ix), py = __ldg(ys + iy), pz = __ldg(zs + iz);
  const int HW = p.Hf * p.Wf;
  const int ctot = p.concat ? p.T * C : C;
  const int S = p.T * p.Nv;
  // ---- phase A (lane = voxel): all views, independent chains --------------------------------
  unsigned vmask = 0;  // views in which this voxel is valid (counts towards the mean)
#pragma unroll 5
  for (int s = 0; s < S; ++s) {
    float cx, cy, d;
    lift_project(p.proj[s], px, py, pz, p.scale_x, p.scale_y, p.crop_x, p.crop_y, cx, cy, d);
    if (p.flip) cx = __fsub_rn((float)p.img_w[s], cx);
    const bool valid = live && cx < (float)p.in_w && cx > 0.f && cy < (float)p.in_h &&
                       cy > 0.f && d > 0.f;
    const int sx = nearest_index(cx, p.Wf, (float)p.in_w);
    const int sy = nearest_index(cy, p.Hf, (float)p.in_h);
    const bool inside = valid && sx >= 0 && sx < p.Wf && sy >= 0 && sy < p.Hf;
    s_off[wib][s][lane] = inside ? (s * HW + sy * p.Wf + sx) * (C / 2) : -1;
    vmask |= valid ? 1u << s : 0u;
  }
  __syncwarp();
  // ---- phase B (lane = channel pair) ----------------------------------------------------------
  const float2* f2 = reinterpret_cast<const float2*>(feats) + lane;
  for (int f = 0; f < p.T; ++f) {
    float2 acc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = make_float2(0.f, 0.f);
    for (int v = 0; v < p.Nv; ++v) {
      const int s = f * p.Nv + v;
      if (__ballot_sync(FULL, s_off[wib][s][lane] >= 0) == 0u) continue;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int o = s_off[wib][s][j];  // broadcast read
        if (o >= 0) {
          const float2 t = __ldg(f2 + o);
          acc[j].x += t.x;
          acc[j].y += t.y;
        }
      }
    }
    const int nvalid = __popc((vmask >> (f * p.Nv)) & ((1u << p.Nv) - 1u));
    const float den = (float)max(nvalid, 1);  // acc is all zero when nvalid == 0
    float2* o2 = reinterpret_cast<float2*>(out + v0 * ctot + (long long)f * C) + lane;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const float dj = __shfl_sync(FULL, den, j);
      if (v0 + j < nvox) {
        // x / 1 == x: most voxels are seen by one camera (warp-uniform branch)
        const float2 r = dj == 1.f ? acc[j]
                                   : make_float2(__fdiv_rn(acc[j].x, dj), __fdiv_rn(acc[j].y, dj));
        __stcs(o2 + (long long)j * (ctot / 2), r);
      }
    }
  }
}

}  // namespace dfm
