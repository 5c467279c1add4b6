// Non-GEMM kernels of SPPUNetNeck (mmdet3d/models/necks/spp_unet_neck.py, shipped KITTI config):
// the four SPP branches, the 512-channel concat both 512-channel convs read, and the two
// upconv_module merges (models/utils/conv_modules.py:46-70).  The 3x3 convs with >= 64 input
// channels run on the BEV stage's 2-D layer driver (bev_api.inc); these kernels feed them and
// apply the folded BatchNorm / GroupNorm of their raw outputs.  Activations are channels-last.
#pragma once
#include "common.cuh"

namespace dfm {

constexpr int SPP_C = 128;       // channels of f2, f3, f4 (in_channels[2:])
constexpr int SPP_BR = 32;       // spp_channel
constexpr int SPP_CAT = 512;     // concat channels: f2 | f3 | f4 | spp64 | spp32 | spp16 | spp8
constexpr int SPP_MAX_CELLS8 = 8192;   // 8x8 cells of f4 held in shared memory by spp_pool_kernel

struct SppPoolParams {
  const float* f4;       // NCHW [128][H4][W4]
  float* pool[4];        // channels-last [Ph_s][Pw_s][128], s = 64, 32, 16, 8
  int H4, W4;
  int ph[4], pw[4];      // floor(H4 / s), floor(W4 / s)
};

// AvgPool2d(s, stride=s) (floor mode) of f4 for s = 64, 32, 16, 8, one CTA per channel: the
// CTA reads its channel plane once into 8x8 cell sums in shared memory (rows / columns past the
// last whole 8-cell are dropped, like the floor mode of every s), then sums 2x2, 4x4 and 8x8
// blocks of them for the coarser pools (a whole s-cell is exactly (s/8)^2 whole 8-cells).
__global__ void __launch_bounds__(256) spp_pool_kernel(SppPoolParams p) {
  extern __shared__ float s8[];   // [ph8][pw8] sums of 64 values
  const int c = blockIdx.x;
  const int ph8 = p.ph[3], pw8 = p.pw[3];
  const float* plane = p.f4 + (long long)c * p.H4 * p.W4;
  const int cols = pw8 * 8;                       // whole 8-cells only
  const int cols32 = (cols + 31) / 32 * 32;       // lanes 8j..8j+7 of a warp share a cell
  for (int i = 0; i < ph8; ++i)
    for (int x = threadIdx.x; x < cols32; x += blockDim.x) {
      float s = 0.f;
      if (x < cols)
#pragma unroll
        for (int r = 0; r < 8; ++r) s += __ldg(plane + (long long)(8 * i + r) * p.W4 + x);
      s += __shfl_xor_sync(0xffffffffu, s, 4);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      if ((x & 7) == 0 && x < cols) s8[i * pw8 + (x >> 3)] = s;
    }
  __syncthreads();
#pragma unroll
  for (int b = 0; b < 4; ++b) {
    const int r = 8 >> b;          // 8-cells per side of an s-cell: s = 64, 32, 16, 8
    const float inv = 1.f / (float)(64 * r * r);
    const int n = p.ph[b] * p.pw[b];
    for (int k = threadIdx.x; k < n; k += blockDim.x) {
      const int i = k / p.pw[b], j = k % p.pw[b];
      float s = 0.f;
      for (int u = 0; u < r; ++u)
        for (int v = 0; v < r; ++v) s += s8[(i * r + u) * pw8 + j * r + v];
      p.pool[b][(long long)k * SPP_C + c] = s * inv;
    }
  }
}

struct SppBranchParams {
  const float* pool[4];    // [cells][128]
  const float* w[4];       // 1x1 conv [32][128]
  const float* gamma[4];
  const float* beta[4];
  float* out[4];           // [cells][32]: relu(gn(conv)) -- the branch map before upsampling
  int cells[4];
};

// One CTA per branch: 1x1 conv 128 -> 32 (no bias) on every pooled cell, then GroupNorm(32, 32)
// -- per-channel statistics over the cells, in fp64 -- and ReLU.  A warp owns a cell, lane = co.
__global__ void __launch_bounds__(256) spp_branch_kernel(SppBranchParams p) {
  __shared__ float ws[SPP_C][SPP_BR + 1];
  __shared__ double red[2][8][SPP_BR];
  __shared__ float aff[2][SPP_BR];
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < SPP_C * SPP_BR; i += blockDim.x)
    ws[i % SPP_C][i / SPP_C] = __ldg(p.w[b] + i);     // [co][ci] -> [ci][co]
  __syncthreads();
  const int n = p.cells[b];
  const float* in = p.pool[b];
  float* out = p.out[b];
  double s = 0.0, ss = 0.0;
  for (int k = warp; k < n; k += 8) {
    const float* x = in + (long long)k * SPP_C;
    float a0 = 0.f, a1 = 0.f;
#pragma unroll 4
    for (int ci = 0; ci < SPP_C; ci += 2) {
      a0 = fmaf(__ldg(x + ci), ws[ci][lane], a0);
      a1 = fmaf(__ldg(x + ci + 1), ws[ci + 1][lane], a1);
    }
    const float v = a0 + a1;
    out[(long long)k * SPP_BR + lane] = v;
    s += v;
    ss += (double)v * v;
  }
  red[0][warp][lane] = s;
  red[1][warp][lane] = ss;
  __syncthreads();
  if (warp == 0) {
    double t = 0.0, tt = 0.0;
    for (int w = 0; w < 8; ++w) {
      t += red[0][w][lane];
      tt += red[1][w][lane];
    }
    const double mean = t / n, var = fmax(tt / n - mean * mean, 0.0);
    const double sc = (double)__ldg(p.gamma[b] + lane) / sqrt(var + 1e-5);
    aff[0][lane] = (float)sc;
    aff[1][lane] = (float)((double)__ldg(p.beta[b] + lane) - mean * sc);
  }
  __syncthreads();
  for (int k = warp; k < n; k += 8) {
    float* o = out + (long long)k * SPP_BR + lane;
    *o = fmaxf(fmaf(*o, aff[0][lane], aff[1][lane]), 0.f);
  }
}

// F.interpolate(bilinear, align_corners=True) source coordinate of output index `d`
struct LerpAC {
  int i0, i1;
  float l1;
};
__device__ __forceinline__ LerpAC lerp_ac(int d, int in, int out) {
  const float scale = out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f;
  const float src = scale * (float)d;
  LerpAC r;
  r.i0 = min((int)src, in - 1);
  r.i1 = min(r.i0 + 1, in - 1);
  r.l1 = src - (float)r.i0;
  return r;
}
// nn.Upsample(scale_factor=2, bilinear), i.e. align_corners=False: src = (d + 0.5) / 2 - 0.5,
// clamped at 0
__device__ __forceinline__ LerpAC lerp_up2(int d, int in) {
  const float src = fmaxf(((float)d + 0.5f) * 0.5f - 0.5f, 0.f);
  LerpAC r;
  r.i0 = min((int)src, in - 1);
  r.i1 = r.i0 < in - 1 ? r.i0 + 1 : r.i0;
  r.l1 = src - (float)r.i0;
  return r;
}

struct SppConcatParams {
  const float* f[3];       // f2, f3, f4: NCHW [128][H4][W4]
  const float* br[4];      // branch maps [ph][pw][32], s = 64, 32, 16, 8
  int ph[4], pw[4];
  int H4, W4;
  float* out;              // [H4][W4][512]
};

// grid (pixel blocks of 32, 16 channel blocks of 32), block (32, 8).  Channel blocks 0..11
// transpose f2 | f3 | f4 through a shared tile; 12..15 upsample one branch map each.
__global__ void __launch_bounds__(256) spp_concat_kernel(SppConcatParams p) {
  __shared__ float tile[32][33];
  const long long HW = (long long)p.H4 * p.W4;
  const long long p0 = (long long)blockIdx.x * 32;
  const int cb = blockIdx.y, tx = threadIdx.x, ty = threadIdx.y;
  if (cb < 12) {
    const float* f = cb < 4 ? p.f[0] : (cb < 8 ? p.f[1] : p.f[2]);
    const float* src = f + (long long)((cb & 3) * 32) * HW;
    for (int j = ty; j < 32; j += 8)
      tile[j][tx] = p0 + tx < HW ? __ldg(src + (long long)j * HW + p0 + tx) : 0.f;
    __syncthreads();
    for (int j = ty; j < 32; j += 8)
      if (p0 + j < HW) p.out[(p0 + j) * SPP_CAT + cb * 32 + tx] = tile[tx][j];
    return;
  }
  // branch b = cb - 12, selected without indexing the parameter arrays (no local copy)
  const float* m = cb == 12 ? p.br[0] : cb == 13 ? p.br[1] : cb == 14 ? p.br[2] : p.br[3];
  const int ph = cb == 12 ? p.ph[0] : cb == 13 ? p.ph[1] : cb == 14 ? p.ph[2] : p.ph[3];
  const int pw = cb == 12 ? p.pw[0] : cb == 13 ? p.pw[1] : cb == 14 ? p.pw[2] : p.pw[3];
  for (int j = ty; j < 32; j += 8) {
    const long long q = p0 + j;
    if (q >= HW) break;
    const int y = (int)(q / p.W4), x = (int)(q % p.W4);
    const LerpAC ly = lerp_ac(y, ph, p.H4), lx = lerp_ac(x, pw, p.W4);
    const float v00 = __ldg(m + ((long long)ly.i0 * pw + lx.i0) * SPP_BR + tx);
    const float v01 = __ldg(m + ((long long)ly.i0 * pw + lx.i1) * SPP_BR + tx);
    const float v10 = __ldg(m + ((long long)ly.i1 * pw + lx.i0) * SPP_BR + tx);
    const float v11 = __ldg(m + ((long long)ly.i1 * pw + lx.i1) * SPP_BR + tx);
    const float h0 = 1.f - ly.l1, w0 = 1.f - lx.l1;
    p.out[q * SPP_CAT + cb * 32 + tx] =
        h0 * (w0 * v00 + lx.l1 * v01) + ly.l1 * (w0 * v10 + lx.l1 * v11);
  }
}

// upconv_module stage 0: x0 = relu(up2(bn(conv0)) + bn(redir0)), 64 channels at H2 x W2.
// conv0 is the raw [H4][W4][64] output, redir0 the raw [H2][W2][64]; one thread per 4 channels.
__global__ void __launch_bounds__(256)
upconv_merge_kernel(const float* __restrict__ conv0, const float* __restrict__ sc0,
                    const float* __restrict__ sh0, const float* __restrict__ redir0,
                    const float* __restrict__ scr, const float* __restrict__ shr, int H4, int W4,
                    float* __restrict__ x0) {
  const int H2 = 2 * H4, W2 = 2 * W4;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)H2 * W2 * 16) return;
  const int q = (int)(idx & 15);
  const long long pix = idx >> 4;
  const int y = (int)(pix / W2), x = (int)(pix % W2);
  const LerpAC ly = lerp_up2(y, H4), lx = lerp_up2(x, W4);
  const float4* c4 = reinterpret_cast<const float4*>(conv0);
  const float4 v00 = __ldg(c4 + ((long long)ly.i0 * W4 + lx.i0) * 16 + q);
  const float4 v01 = __ldg(c4 + ((long long)ly.i0 * W4 + lx.i1) * 16 + q);
  const float4 v10 = __ldg(c4 + ((long long)ly.i1 * W4 + lx.i0) * 16 + q);
  const float4 v11 = __ldg(c4 + ((long long)ly.i1 * W4 + lx.i1) * 16 + q);
  const float4 r = __ldg(reinterpret_cast<const float4*>(redir0) + pix * 16 + q);
  const float4 a = __ldg(reinterpret_cast<const float4*>(sc0) + q);
  const float4 bb = __ldg(reinterpret_cast<const float4*>(sh0) + q);
  const float4 ar = __ldg(reinterpret_cast<const float4*>(scr) + q);
  const float4 br = __ldg(reinterpret_cast<const float4*>(shr) + q);
  const float h0 = 1.f - ly.l1, w0 = 1.f - lx.l1, h1 = ly.l1, w1 = lx.l1;
#define SPP_UP(k) (h0 * (w0 * fmaf(v00.k, a.k, bb.k) + w1 * fmaf(v01.k, a.k, bb.k)) + \
                   h1 * (w0 * fmaf(v10.k, a.k, bb.k) + w1 * fmaf(v11.k, a.k, bb.k)) + \
                   fmaf(r.k, ar.k, br.k))
  float4 o;
  o.x = fmaxf(SPP_UP(x), 0.f);
  o.y = fmaxf(SPP_UP(y), 0.f);
  o.z = fmaxf(SPP_UP(z), 0.f);
  o.w = fmaxf(SPP_UP(w), 0.f);
#undef SPP_UP
  reinterpret_cast<float4*>(x0)[pix * 16 + q] = o;
}

// upconv_module stage 1: x1 = relu(up2(bn(conv1)) + bn(redir1(img))), 32 channels at H x W,
// channels-last.  redir1 (3 -> 32, 3x3, pad 1, no bias) is computed here from the NCHW image:
// 27 fp32 MACs per output, weights [27][32] in shared memory.  One thread per pixel.
__global__ void __launch_bounds__(256)
upconv_merge_img_kernel(const float* __restrict__ conv1, const float* __restrict__ sc1,
                        const float* __restrict__ sh1, const float* __restrict__ img,
                        const float* __restrict__ wr, const float* __restrict__ scr,
                        const float* __restrict__ shr, int H2, int W2, float* __restrict__ x1) {
  __shared__ float ws[27][32];
  __shared__ float aff[4][32];
  for (int i = threadIdx.x; i < 27 * 32; i += blockDim.x)
    ws[i % 27][i / 27] = __ldg(wr + i);               // (co, ci, ky, kx) -> [ci*9 + ky*3 + kx][co]
  if (threadIdx.x < 128) {
    const int k = threadIdx.x >> 5, c = threadIdx.x & 31;
    aff[k][c] = __ldg((k == 0 ? sc1 : k == 1 ? sh1 : k == 2 ? scr : shr) + c);
  }
  __syncthreads();
  const int H = 2 * H2, W = 2 * W2;
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (long long)H * W) return;
  const int y = (int)(pix / W), x = (int)(pix % W);
  const long long HW = (long long)H * W;
  float xin[27];
#pragma unroll
  for (int ci = 0; ci < 3; ++ci)
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int yy = y + ky - 1, xx = x + kx - 1;
        xin[ci * 9 + ky * 3 + kx] = (yy >= 0 && yy < H && xx >= 0 && xx < W)
                                        ? __ldg(img + ci * HW + (long long)yy * W + xx) : 0.f;
      }
  const LerpAC ly = lerp_up2(y, H2), lx = lerp_up2(x, W2);
  const float h0 = 1.f - ly.l1, w0 = 1.f - lx.l1, h1 = ly.l1, w1 = lx.l1;
  const float4* c4 = reinterpret_cast<const float4*>(conv1);
  const long long o00 = ((long long)ly.i0 * W2 + lx.i0) * 8, o01 = ((long long)ly.i0 * W2 + lx.i1) * 8;
  const long long o10 = ((long long)ly.i1 * W2 + lx.i0) * 8, o11 = ((long long)ly.i1 * W2 + lx.i1) * 8;
  float4* dst = reinterpret_cast<float4*>(x1 + pix * 32);
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 v00 = __ldg(c4 + o00 + q), v01 = __ldg(c4 + o01 + q);
    const float4 v10 = __ldg(c4 + o10 + q), v11 = __ldg(c4 + o11 + q);
    const float a00[4] = {v00.x, v00.y, v00.z, v00.w}, a01[4] = {v01.x, v01.y, v01.z, v01.w};
    const float a10[4] = {v10.x, v10.y, v10.z, v10.w}, a11[4] = {v11.x, v11.y, v11.z, v11.w};
    float o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = 4 * q + k;
      const float a = aff[0][c], b = aff[1][c];
      const float up = h0 * (w0 * fmaf(a00[k], a, b) + w1 * fmaf(a01[k], a, b)) +
                       h1 * (w0 * fmaf(a10[k], a, b) + w1 * fmaf(a11[k], a, b));
      float r = 0.f;
#pragma unroll
      for (int t = 0; t < 27; ++t) r = fmaf(xin[t], ws[t][c], r);
      o[k] = fmaxf(up + fmaf(r, aff[2][c], aff[3][c]), 0.f);
    }
    dst[q] = make_float4(o[0], o[1], o[2], o[3]);
  }
}

}  // namespace dfm
