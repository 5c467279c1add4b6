// Device helpers the anchor-head and ATSS losses share (anchor_loss_kernels.cuh,
// atss_loss_kernels.cuh): the focal term of one logit, axis-aligned box areas and IoUs, and fixed-
// order fp64 block sums.
#pragma once
#include <cuda_runtime.h>

#include <cfloat>

namespace dfm {

// mmcv sigmoid_focal_loss forward (l) and backward (g) of one logit x in fp32, as its CUDA
// kernels compute them; is_target: the logit's class is the anchor's label
__device__ __forceinline__ void sigmoid_focal_term(float x, bool is_target, float gamma,
                                                   float alpha, float& l, float& g) {
  const float pr = 1.f / (1.f + expf(-x));
  if (is_target) {
    const float lp = logf(fmaxf(pr, FLT_MIN));
    l = -alpha * powf(1.f - pr, gamma) * lp;
    g = -alpha * powf(1.f - pr, gamma) * (1.f - pr - gamma * pr * lp);
  } else {
    const float lq = logf(fmaxf(1.f - pr, FLT_MIN));
    l = -(1.f - alpha) * powf(pr, gamma) * lq;
    g = -(1.f - alpha) * powf(pr, gamma) * (gamma * (1.f - pr) * lq - pr);
  }
}

// (x2 - x1) * (y2 - y1) of an (x1, y1, x2, y2) box
__device__ __forceinline__ float al_area(const float* o) {
  return __fmul_rn(__fsub_rn(o[2], o[0]), __fsub_rn(o[3], o[1]));
}

// mmdet bbox_overlaps(gt, anchor), mode 'iou', eps 1e-6, of axis-aligned (x1, y1, x2, y2) boxes
// with areas ga and aa; symmetric in its two boxes, as every op it rounds is
__device__ __forceinline__ float al_iou(const float* g, float ga, const float* a, float aa) {
  const float w = fmaxf(__fsub_rn(fminf(g[2], a[2]), fmaxf(g[0], a[0])), 0.f);
  const float h = fmaxf(__fsub_rn(fminf(g[3], a[3]), fmaxf(g[1], a[1])), 0.f);
  const float ov = __fmul_rn(w, h);
  if (ov == 0.f) return 0.f;
  const float un = fmaxf(__fsub_rn(__fadd_rn(ga, aa), ov), 1e-6f);
  return __fdiv_rn(ov, un);
}

// K fp64 sums over a block of NT threads in a fixed tree order; the totals land in red[k][0]
template <int K, int NT>
__device__ __forceinline__ void block_sum_fp64(const double* v, double (*red)[NT]) {
#pragma unroll
  for (int k = 0; k < K; ++k) red[k][threadIdx.x] = v[k];
  __syncthreads();
  for (int h = NT / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) {
#pragma unroll
      for (int k = 0; k < K; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + h];
    }
    __syncthreads();
  }
}

}  // namespace dfm
