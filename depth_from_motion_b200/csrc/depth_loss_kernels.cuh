// DepthHead.loss (dense_heads/depth_head.py:75-188) for the ce / balanced_ce / focal /
// balanced_focal types: per pixel w_pix * sum_k p_k * alpha (1 - P_k)^gamma * (-log P_k) over the
// f*D bins of the x-f trilinear (align_corners) upsampling of the low-res cost logits, read
// column by column so the [fD, fH, fW] volume and its gradient never exist.
//   * dl_pixel_kernel  -- one warp per masked full-res pixel: its column from the 2 x 2 low-res
//     columns, the log-softmax, the loss term and the sum of the per-bin coefficients c_k of
//     dL/dz_k = c_k - P_k * sum(c).  A few floats per pixel are kept for the adjoint pass; the
//     dense form writes its gradient column here instead.
//   * dl_finish_kernel -- one CTA: count, loss and gradient scale from the per-block partials.
//   * dl_adjoint_kernel -- one thread per low-res voxel: the transposed interpolation, gathered
//     over the full-res pixels and bins whose interpolation reads the voxel, with z_k recomputed
//     by the same helpers as the pixel pass (bitwise the same value).
// No floating-point atomics: every sum runs in a fixed order.
#pragma once
#include "tail_kernels.cuh"

namespace dfm {

constexpr int DL_WARPS = 8;                 // pixel pass: warps per block
constexpr int DL_PIX = 32 * DL_WARPS;       // pixels per pixel-pass block, 32 per warp
constexpr int DL_ADJ_X = 128;               // adjoint pass: low-res columns per block
constexpr int DL_FIN_THREADS = 256;

struct DepthLossParams {
  int n, D, Ho, Wo, dense;    // dense: vol is [n][D][Ho][Wo] at full resolution, f = 1
  int OD, OH, OW;             // full resolution
  float sz, sy, sx;           // ac_scale of each axis
  float min_d, max_d, alpha, gamma, fg_w, bg_w;
  int balanced;
  const float* vol;
  const float* samples;       // [OD]
  const float* depth;         // [n][OH][OW]
  const unsigned char* fg;    // [n][OH][OW], balanced types only
  float* grad;                // same layout as vol, or null
  // per full-res pixel [n][OH][OW]: weight (0 outside the mask), gt depth, max and log-sum of
  // exp of the column, sum of c_k, weighted loss term
  float *w, *gt, *mx, *lse, *sc, *pix_loss;
  double* part_loss;          // [blocks]
  int* part_cnt;              // [blocks]
  int blocks;
};

// Low-res column z of a full-res pixel: rows blended first, then columns (the order of
// depth_head4_kernel), every product rounded, so both passes get the same bits.
__device__ __forceinline__ float dl_col(const float* __restrict__ c, int z, long long plane,
                                        int Wo, int y0, int y1, float ly0, float ly1, int x0,
                                        int x1, float wx0, float wx1) {
  const float* p = c + z * plane;
  const float r0 = __fmaf_rn(ly1, __ldg(p + y1 * Wo + x0), __fmul_rn(ly0, __ldg(p + y0 * Wo + x0)));
  const float r1 = __fmaf_rn(ly1, __ldg(p + y1 * Wo + x1), __fmul_rn(ly0, __ldg(p + y0 * Wo + x1)));
  return __fmaf_rn(wx1, r1, __fmul_rn(wx0, r0));
}
__device__ __forceinline__ float dl_lerp(float l0, float l1, float a, float b) {
  return __fmaf_rn(l1, b, __fmul_rn(l0, a));
}
// (1 - P)^g; 0, 1 and 2 exactly, as torch.pow does
__device__ __forceinline__ float dl_pow(float x, float g) {
  if (g == 0.f) return 1.f;
  if (g == 1.f) return x;
  if (g == 2.f) return __fmul_rn(x, x);
  return powf(x, g);
}
// the reference's soft target: 1 - min(|s - gt| / interval, 1), a true division
__device__ __forceinline__ float dl_target(float s, float gt, float interval) {
  return __fsub_rn(1.f, fminf(__fdiv_rn(fabsf(__fsub_rn(s, gt)), interval), 1.f));
}
// log P_k of value v in a column with maximum m and log-sum-exp lse = log(sum exp(v - m))
__device__ __forceinline__ float dl_logp(float v, float m, float lse) {
  return __fsub_rn(__fsub_rn(v, m), lse);
}
// Loss term t = -p alpha (1 - P)^g log P of one bin and its derivative c = dt / d log P.
__device__ __forceinline__ void dl_term(float p, float lp, float alpha, float gamma, float& t,
                                        float& c) {
  const float P = expf(lp);
  const float q = __fsub_rn(1.f, P);
  const float F = dl_pow(q, gamma);
  t = -__fmul_rn(p, __fmul_rn(__fmul_rn(alpha, F), lp));
  float d = F;
  if (gamma != 0.f)
    d = __fsub_rn(F, __fmul_rn(__fmul_rn(gamma, dl_pow(q, gamma - 1.f)), __fmul_rn(P, lp)));
  c = -__fmul_rn(__fmul_rn(p, alpha), d);
}
// dL_pix / dz_k = w (c_k - P_k sum(c)) of one bin
__device__ __forceinline__ float dl_grad(float v, float s, float gt, float interval, float m,
                                         float lse, float sc, float w, float alpha, float gamma) {
  const float lp = dl_logp(v, m, lse);
  const float p = dl_target(s, gt, interval);
  float c = 0.f;
  if (p > 0.f) {
    float t;
    dl_term(p, lp, alpha, gamma, t, c);
  }
  return __fmul_rn(w, __fsub_rn(c, __fmul_rn(expf(lp), sc)));
}

__device__ __forceinline__ float dl_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return __shfl_sync(0xffffffffu, v, 0);
}
__device__ __forceinline__ float dl_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return __shfl_sync(0xffffffffu, v, 0);
}

// dynamic shared memory: per-bin float4 (l0, l1, sample, z0) [OD] | per-warp columns [WARPS][D]
inline size_t dl_pixel_smem(int OD, int D) {
  return (size_t)OD * sizeof(float4) + (size_t)DL_WARPS * D * sizeof(float);
}

__global__ void __launch_bounds__(DL_PIX)
dl_pixel_kernel(const DepthLossParams p) {
  extern __shared__ float4 dl_dyn[];
  float4* tab = dl_dyn;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* colz = reinterpret_cast<float*>(tab + p.OD) + warp * p.D;
  __shared__ double s_loss[DL_WARPS];
  __shared__ int s_cnt[DL_WARPS];
  for (int k = threadIdx.x; k < p.OD; k += DL_PIX) {
    int z0 = k;
    float l0 = 1.f, l1 = 0.f;
    if (!p.dense) ac_bin(p.sz, k, p.D, z0, l0, l1);
    tab[k] = make_float4(l0, l1, __ldg(p.samples + k), __int_as_float(z0));
  }
  __syncthreads();
  const float interval = __fsub_rn(__ldg(p.samples + 1), __ldg(p.samples));
  const long long opl = (long long)p.OH * p.OW, npix = (long long)p.n * opl;
  const long long plane = (long long)p.Ho * p.Wo;
  const long long pix = (long long)blockIdx.x * DL_PIX + warp * 32 + lane;
  float wpix = 0.f, gtv = 0.f;
  bool masked = false;   // NaN fails both tests
  if (pix < npix) {
    gtv = __ldg(p.depth + pix);
    masked = gtv > p.min_d && gtv < p.max_d;
    if (masked) wpix = p.balanced ? (__ldg(p.fg + pix) ? p.fg_w : p.bg_w) : 1.f;
    p.w[pix] = wpix;
    if (!masked) p.pix_loss[pix] = 0.f;
  }
  const unsigned live = __ballot_sync(0xffffffffu, masked);
  double wsum = 0.0;
  for (unsigned todo = live; todo; todo &= todo - 1) {
    const int src = __ffs(todo) - 1;
    const long long q = (long long)blockIdx.x * DL_PIX + warp * 32 + src;
    const float gt = __shfl_sync(0xffffffffu, gtv, src);
    const float w = __shfl_sync(0xffffffffu, wpix, src);
    const int ni = (int)(q / opl);
    const int rem = (int)(q - (long long)ni * opl);
    const int Y = rem / p.OW, X = rem - Y * p.OW;
    const float* dv = p.dense ? p.vol + (long long)ni * p.OD * opl + rem : nullptr;
    if (!p.dense) {
      int y0, y1, x0, x1;
      float ly0, ly1, wx0, wx1;
      ac_tap(p.sy, Y, p.Ho, y0, y1, ly0, ly1);
      ac_tap(p.sx, X, p.Wo, x0, x1, wx0, wx1);
      const float* c = p.vol + (long long)ni * p.D * plane;
      for (int z = lane; z < p.D; z += 32)
        colz[z] = dl_col(c, z, plane, p.Wo, y0, y1, ly0, ly1, x0, x1, wx0, wx1);
      __syncwarp();
    }
    auto value = [&](int k, const float4& tk) {
      if (p.dense) return __ldg(dv + k * opl);
      const int z0 = __float_as_int(tk.w);
      return dl_lerp(tk.x, tk.y, colz[z0], colz[min(z0 + 1, p.D - 1)]);
    };
    float m = -INFINITY;
    for (int k = lane; k < p.OD; k += 32) m = fmaxf(m, value(k, tab[k]));
    m = dl_warp_max(m);
    float s = 0.f;
    for (int k = lane; k < p.OD; k += 32) s += expf(__fsub_rn(value(k, tab[k]), m));
    const float lse = logf(dl_warp_sum(s));
    float t = 0.f, sc = 0.f;
    for (int k = lane; k < p.OD; k += 32) {
      const float4 tk = tab[k];
      const float pk = dl_target(tk.z, gt, interval);
      if (pk > 0.f) {
        float tt, cc;
        dl_term(pk, dl_logp(value(k, tk), m, lse), p.alpha, p.gamma, tt, cc);
        t += tt;
        sc += cc;
      }
    }
    t = dl_warp_sum(t);
    sc = dl_warp_sum(sc);
    if (p.dense && p.grad) {
      float* g = p.grad + (long long)ni * p.OD * opl + rem;
      for (int k = lane; k < p.OD; k += 32) {
        const float4 tk = tab[k];
        g[k * opl] = dl_grad(value(k, tk), tk.z, gt, interval, m, lse, sc, w, p.alpha, p.gamma);
      }
    }
    const float wt = __fmul_rn(w, t);
    if (lane == 0) {
      p.gt[q] = gt;
      p.mx[q] = m;
      p.lse[q] = lse;
      p.sc[q] = sc;
      p.pix_loss[q] = wt;
    }
    wsum += (double)wt;
    __syncwarp();   // colz is rewritten by the next pixel
  }
  if (lane == 0) {
    s_loss[warp] = wsum;
    s_cnt[warp] = __popc(live);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    int cnt = 0;
    for (int i = 0; i < DL_WARPS; ++i) {
      a += s_loss[i];
      cnt += s_cnt[i];
    }
    p.part_loss[blockIdx.x] = a;
    p.part_cnt[blockIdx.x] = cnt;
  }
}

// loss = lw2 * sum / count and scale = lw2 / count; with no masked pixel, loss = *empty (the
// reference's depth_preds.mean() * 0.0) and scale = 0
__global__ void __launch_bounds__(DL_FIN_THREADS)
dl_finish_kernel(const double* __restrict__ part_loss, const int* __restrict__ part_cnt,
                 int blocks, double lw2, const float* __restrict__ empty, int* __restrict__ count,
                 float* __restrict__ loss, float* __restrict__ scale) {
  __shared__ double sl[DL_FIN_THREADS];
  __shared__ long long sn[DL_FIN_THREADS];
  double a = 0.0;
  long long c = 0;
  for (int i = threadIdx.x; i < blocks; i += DL_FIN_THREADS) {
    a += part_loss[i];
    c += part_cnt[i];
  }
  sl[threadIdx.x] = a;
  sn[threadIdx.x] = c;
  __syncthreads();
  for (int s = DL_FIN_THREADS / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      sl[threadIdx.x] += sl[threadIdx.x + s];
      sn[threadIdx.x] += sn[threadIdx.x + s];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const long long n = sn[0];
    *count = (int)n;
    *loss = n > 0 ? (float)(lw2 * sl[0] / (double)n) : (empty ? *empty : 0.f);
    *scale = n > 0 ? (float)(lw2 / (double)n) : 0.f;
  }
}

// full-res indices i in [lo, hi] whose taps (ac_tap) may include low-res index t; the caller
// tests each exactly
__device__ __forceinline__ void dl_candidates(float s, int t, int n_out, int& lo, int& hi) {
  if (s > 0.f) {
    lo = max(0, (int)floor((t - 1) / (double)s) - 1);
    hi = min(n_out - 1, (int)ceil((t + 1) / (double)s) + 1);
  } else {
    lo = 0;
    hi = n_out - 1;
  }
}

// dynamic shared memory: per-bin float4 (l0, l1, sample, z0) [OD]
__global__ void __launch_bounds__(DL_ADJ_X)
dl_adjoint_kernel(const DepthLossParams p) {
  extern __shared__ float4 dl_tab[];
  for (int k = threadIdx.x; k < p.OD; k += DL_ADJ_X) {
    int z0;
    float l0, l1;
    ac_bin(p.sz, k, p.D, z0, l0, l1);
    dl_tab[k] = make_float4(l0, l1, __ldg(p.samples + k), __int_as_float(z0));
  }
  __syncthreads();
  const int xq = blockIdx.x * DL_ADJ_X + threadIdx.x;
  const int yq = blockIdx.y;
  const int ni = blockIdx.z / p.D, z = blockIdx.z - ni * p.D;
  if (xq >= p.Wo) return;
  const float interval = __fsub_rn(__ldg(p.samples + 1), __ldg(p.samples));
  const long long plane = (long long)p.Ho * p.Wo, opl = (long long)p.OH * p.OW;
  const float* c = p.vol + (long long)ni * p.D * plane;
  const long long pbase = (long long)ni * opl;
  int ylo, yhi, xlo, xhi, klo, khi;
  dl_candidates(p.sy, yq, p.OH, ylo, yhi);
  dl_candidates(p.sx, xq, p.OW, xlo, xhi);
  dl_candidates(p.sz, z, p.OD, klo, khi);
  double acc = 0.0;
  for (int Y = ylo; Y <= yhi; ++Y) {
    int y0, y1;
    float ly0, ly1;
    ac_tap(p.sy, Y, p.Ho, y0, y1, ly0, ly1);
    const float wy = (y0 == yq ? ly0 : 0.f) + (y1 == yq ? ly1 : 0.f);
    if (y0 != yq && y1 != yq) continue;
    for (int X = xlo; X <= xhi; ++X) {
      int x0, x1;
      float wx0, wx1;
      ac_tap(p.sx, X, p.Wo, x0, x1, wx0, wx1);
      if (x0 != xq && x1 != xq) continue;
      const long long q = pbase + (long long)Y * p.OW + X;
      const float w = p.w[q];
      if (w == 0.f) continue;
      const float wx = (x0 == xq ? wx0 : 0.f) + (x1 == xq ? wx1 : 0.f);
      const float gt = p.gt[q], m = p.mx[q], lse = p.lse[q], sc = p.sc[q];
      // the columns of planes z - 1, z, z + 1 (those a bin reading plane z interpolates between)
      const float cm = z > 0 ? dl_col(c, z - 1, plane, p.Wo, y0, y1, ly0, ly1, x0, x1, wx0, wx1)
                             : 0.f;
      const float cz = dl_col(c, z, plane, p.Wo, y0, y1, ly0, ly1, x0, x1, wx0, wx1);
      const float cp = z < p.D - 1
                           ? dl_col(c, z + 1, plane, p.Wo, y0, y1, ly0, ly1, x0, x1, wx0, wx1)
                           : cz;
      const double wyx = (double)wy * (double)wx;
      for (int k = klo; k <= khi; ++k) {
        const float4 tk = dl_tab[k];
        const int z0 = __float_as_int(tk.w);
        float v, lz;
        if (z0 == z - 1) {
          v = dl_lerp(tk.x, tk.y, cm, cz);
          lz = tk.y;
        } else if (z0 == z) {
          v = dl_lerp(tk.x, tk.y, cz, cp);
          lz = z == p.D - 1 ? tk.x + tk.y : tk.x;
        } else {
          continue;
        }
        const float g = dl_grad(v, tk.z, gt, interval, m, lse, sc, w, p.alpha, p.gamma);
        acc += (double)g * ((double)lz * wyx);
      }
    }
  }
  p.grad[((long long)ni * p.D + z) * plane + (long long)yq * p.Wo + xq] = (float)acc;
}

}  // namespace dfm
