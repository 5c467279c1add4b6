// Training loss of DfM's 2-D auxiliary head (LIGAATSSHead.loss_single / centerness_target /
// _get_target_single, dense_heads/liga_atss_head.py:176-270, 380-483, with mmdet 2.x's
// ATSSHead.loss / get_targets) and its target assignment (ATSS3DCenterAssigner.assign,
// core/bbox/assigners/atss_3dcenter_assigner.py:27-168), for a batch of B images over L levels
// of one square anchor per location:
//
//   at_assign_kernel   one block per GT: the topk nearest valid anchors of every level to the
//                      GT's projected 3-D centre, their IoUs, the mean + std threshold and the
//                      in-GT test; each positive candidate is offered to its anchor through an
//                      atomicMax on (IoU bits, GT order), which keeps the highest IoU and, on a
//                      tie, the first GT whatever the thread order
//   at_loss_kernel     per anchor: labels, label weights, DeltaXYWHBBoxCoder targets and the
//                      centerness target; sigmoid focal loss, GIoU of the decoded positives and
//                      the centerness BCE with their gradients, on the NCHW head outputs of every
//                      level; per-block sums in fp64
//   at_norm_kernel     the per-level sums in a fixed order, num_total_pos = sum_b max(pos_b, 1)
//                      and the sum of the centerness targets
//   at_finish_kernel   the 3 x L loss values and the scale each stored gradient takes
//
// Every op that decides a target rounds as the reference's fp32 PyTorch ops do: explicitly
// rounded intrinsics (no FMA contraction) in the same order.
#pragma once
#include <cuda_runtime.h>

#include <cfloat>
#include <cstdint>

#include "anchor_loss_kernels.cuh"

namespace dfm {

constexpr int AT_MAX_LEVELS = 8;
constexpr int AT_MAX_IMAGES = 32;
constexpr int AT_MAX_CLASSES = 16;
constexpr int AT_TOPK = 9;  // ATSS3DCenterAssigner(topk=9)
constexpr int AT_THREADS = 256;

struct AtssLossParams {
  int B, L, C, N;                     // N anchors per image over all levels
  int H[AT_MAX_LEVELS], W[AT_MAX_LEVELS], stride[AT_MAX_LEVELS];
  int off[AT_MAX_LEVELS + 1];         // first anchor of each level
  int blk_off[AT_MAX_LEVELS + 1];     // first loss-kernel block of each level
  float half[AT_MAX_LEVELS];          // half the anchor side, fp32 as AnchorGenerator forms it
  int pad_h[AT_MAX_IMAGES], pad_w[AT_MAX_IMAGES];
  float gamma, alpha;                 // FocalLoss
  float std_xy, std_wh;               // DeltaXYWHBBoxCoder target_stds (means 0)
  float max_ratio;                    // fp32 |log(wh_ratio_clip)|
  float giou_eps;                     // GIoULoss eps
  // per forward
  const float* cls[AT_MAX_LEVELS];    // [B][C][H][W]
  const float* reg[AT_MAX_LEVELS];    // [B][4 * C][H][W], channel k * C + c
  const float* ctr[AT_MAX_LEVELS];    // [B][1][H][W]
  float* g_cls[AT_MAX_LEVELS];        // gradients of the unnormalised sums, or null
  float* g_reg[AT_MAX_LEVELS];
  float* g_ctr[AT_MAX_LEVELS];
  const float* gt;                    // [G][6]: x1, y1, x2, y2, projected 3-D centre x, y
  const int* gt_label;                // [G]
  const int* gt_off;                  // [B + 1]
  int G;
  // workspace
  unsigned long long* best;           // [B][N] (IoU bits << 32) | ~GT index in the image; 0 none
  float* thr;                         // [G] the assigner's IoU threshold of each GT
  int* assigned;                      // [B][N] 0 negative or invalid, g + 1 (GT g of the image)
  int* labels;                        // [B][N]
  float* label_w;                     // [B][N]
  float* targets;                     // [B][N][4]
  float* ctr_t;                       // [B][N]
  int* pos_count;                     // [B]
  int* status;                        // bit 0: a GT label outside 0..C-1
  double* partial;                    // [B][blocks][4]: focal, GIoU, BCE, centerness target
  double* level_sum;                  // [L][4]
  int blocks;                         // loss-kernel blocks per image
};

// valid anchors of level l in image b: AnchorGenerator.valid_flags from the pad shape
__device__ __forceinline__ int at_valid_h(const AtssLossParams& p, int b, int l) {
  const int v = (p.pad_h[b] + p.stride[l] - 1) / p.stride[l];
  return v < p.H[l] ? v : p.H[l];
}
__device__ __forceinline__ int at_valid_w(const AtssLossParams& p, int b, int l) {
  const int v = (p.pad_w[b] + p.stride[l] - 1) / p.stride[l];
  return v < p.W[l] ? v : p.W[l];
}

// anchor (x1, y1, x2, y2) at column x, row y of level l: base anchor (-half, half) plus the shift
__device__ __forceinline__ void at_anchor(const AtssLossParams& p, int l, int x, int y, float* a) {
  const float sx = (float)(x * p.stride[l]), sy = (float)(y * p.stride[l]), h = p.half[l];
  a[0] = __fadd_rn(-h, sx);
  a[1] = __fadd_rn(-h, sy);
  a[2] = __fadd_rn(h, sx);
  a[3] = __fadd_rn(h, sy);
}

// DeltaXYWHBBoxCoder.decode (mmdet delta2bbox, means 0, no max_shape) of 4 deltas; e_out: the
// exp of the clamped size deltas, in_clamp: whether each size delta lies inside the clamp
__device__ __forceinline__ void at_decode(const AtssLossParams& p, const float* a, const float* d,
                                          float* o, float* e_out, bool* in_clamp) {
  const float px = __fmul_rn(__fadd_rn(a[0], a[2]), 0.5f);
  const float py = __fmul_rn(__fadd_rn(a[1], a[3]), 0.5f);
  const float pw = __fsub_rn(a[2], a[0]), ph = __fsub_rn(a[3], a[1]);
  const float dx = __fmul_rn(d[0], p.std_xy), dy = __fmul_rn(d[1], p.std_xy);
  float dw = __fmul_rn(d[2], p.std_wh), dh = __fmul_rn(d[3], p.std_wh);
  if (in_clamp) {
    in_clamp[0] = dw >= -p.max_ratio && dw <= p.max_ratio;
    in_clamp[1] = dh >= -p.max_ratio && dh <= p.max_ratio;
  }
  dw = fminf(fmaxf(dw, -p.max_ratio), p.max_ratio);
  dh = fminf(fmaxf(dh, -p.max_ratio), p.max_ratio);
  const float gx = __fadd_rn(px, __fmul_rn(pw, dx)), gy = __fadd_rn(py, __fmul_rn(ph, dy));
  const float ew = expf(dw), eh = expf(dh);
  const float gw = __fmul_rn(pw, ew), gh = __fmul_rn(ph, eh);
  const float hw = __fmul_rn(gw, 0.5f), hh = __fmul_rn(gh, 0.5f);
  o[0] = __fsub_rn(gx, hw);
  o[1] = __fsub_rn(gy, hh);
  o[2] = __fadd_rn(gx, hw);
  o[3] = __fadd_rn(gy, hh);
  if (e_out) {
    e_out[0] = ew;
    e_out[1] = eh;
  }
}

// DeltaXYWHBBoxCoder.encode (mmdet bbox2delta, means 0) of GT box g against anchor a
__device__ __forceinline__ void at_encode(const AtssLossParams& p, const float* a, const float* g,
                                          float* t) {
  const float px = __fmul_rn(__fadd_rn(a[0], a[2]), 0.5f);
  const float py = __fmul_rn(__fadd_rn(a[1], a[3]), 0.5f);
  const float pw = __fsub_rn(a[2], a[0]), ph = __fsub_rn(a[3], a[1]);
  const float gx = __fmul_rn(__fadd_rn(g[0], g[2]), 0.5f);
  const float gy = __fmul_rn(__fadd_rn(g[1], g[3]), 0.5f);
  const float gw = __fsub_rn(g[2], g[0]), gh = __fsub_rn(g[3], g[1]);
  t[0] = __fdiv_rn(__fdiv_rn(__fsub_rn(gx, px), pw), p.std_xy);
  t[1] = __fdiv_rn(__fdiv_rn(__fsub_rn(gy, py), ph), p.std_xy);
  t[2] = __fdiv_rn(logf(__fdiv_rn(gw, pw)), p.std_wh);
  t[3] = __fdiv_rn(logf(__fdiv_rn(gh, ph)), p.std_wh);
}

// LIGAATSSHead.centerness_target of one positive: the decoded target box against the anchor
// centre
__device__ __forceinline__ float at_centerness(const float* a, const float* g) {
  const float cx = __fmul_rn(__fadd_rn(a[2], a[0]), 0.5f);
  const float cy = __fmul_rn(__fadd_rn(a[3], a[1]), 0.5f);
  const float l = __fsub_rn(cx, g[0]), t = __fsub_rn(cy, g[1]);
  const float r = __fsub_rn(g[2], cx), b = __fsub_rn(g[3], cy);
  const float lr = __fdiv_rn(fminf(l, r), fmaxf(l, r));
  const float tb = __fdiv_rn(fminf(t, b), fmaxf(t, b));
  return __fsqrt_rn(__fmul_rn(lr, tb));
}

// the share of a gradient that torch.maximum (gate_max) / torch.minimum (gate_min) passes to its
// first argument: all of it, half on a tie, none otherwise
__device__ __forceinline__ double gate_max(float a, float b) {
  return a > b ? 1.0 : (a == b ? 0.5 : 0.0);
}
__device__ __forceinline__ double gate_min(float a, float b) {
  return a < b ? 1.0 : (a == b ? 0.5 : 0.0);
}

// mmdet bbox_overlaps(pred, target, mode='giou', is_aligned=True, eps) in fp32, rounded as its
// ops are; gp[4] = d giou / d pred (x1, y1, x2, y2) as PyTorch's autograd forms it, in fp64
// (ties of min / max split the gradient in half, clamp(min=0) passes it at 0)
__device__ __forceinline__ float at_giou(const float* pr, const float* tg, float eps,
                                         double* gp) {
  const float a1 = al_area(pr), a2 = al_area(tg);
  const float wr = __fsub_rn(fminf(pr[2], tg[2]), fmaxf(pr[0], tg[0]));
  const float hr = __fsub_rn(fminf(pr[3], tg[3]), fmaxf(pr[1], tg[1]));
  const float w = fmaxf(wr, 0.f), h = fmaxf(hr, 0.f);
  const float ov = __fmul_rn(w, h);
  const float unr = __fsub_rn(__fadd_rn(a1, a2), ov), un = fmaxf(unr, eps);
  const float iou = __fdiv_rn(ov, un);
  const float ewr = __fsub_rn(fmaxf(pr[2], tg[2]), fminf(pr[0], tg[0]));
  const float ehr = __fsub_rn(fmaxf(pr[3], tg[3]), fminf(pr[1], tg[1]));
  const float ew = fmaxf(ewr, 0.f), eh = fmaxf(ehr, 0.f);
  const float ear = __fmul_rn(ew, eh), ea = fmaxf(ear, eps);
  const float num = __fsub_rn(ea, un);
  const float giou = __fsub_rn(iou, __fdiv_rn(num, ea));
  // backward of giou = ov / un - (ea - un) / ea
  const double dea = ea, dun = un;
  const double g_num = -1.0 / dea;
  const double g_ea = g_num + (double)num / (dea * dea);
  double g_un = -g_num - (double)ov / (dun * dun);
  double g_ov = 1.0 / dun;
  const double g_unr = g_un * gate_max(unr, eps);
  g_ov -= g_unr;
  const double g_ear = g_ea * gate_max(ear, eps);
  const double g_ewr = ewr >= 0.f ? g_ear * eh : 0.0;
  const double g_ehr = ehr >= 0.f ? g_ear * ew : 0.0;
  const double g_wr = wr >= 0.f ? g_ov * h : 0.0;
  const double g_hr = hr >= 0.f ? g_ov * w : 0.0;
  const double ph = __fsub_rn(pr[3], pr[1]), pw = __fsub_rn(pr[2], pr[0]);
  gp[0] = -g_wr * gate_max(pr[0], tg[0]) - g_ewr * gate_min(pr[0], tg[0]) - g_unr * ph;
  gp[1] = -g_hr * gate_max(pr[1], tg[1]) - g_ehr * gate_min(pr[1], tg[1]) - g_unr * pw;
  gp[2] = g_wr * gate_min(pr[2], tg[2]) + g_ewr * gate_max(pr[2], tg[2]) + g_unr * ph;
  gp[3] = g_hr * gate_min(pr[3], tg[3]) + g_ehr * gate_max(pr[3], tg[3]) + g_unr * pw;
  return giou;
}

// ---- assignment ----

__device__ __forceinline__ unsigned long long at_block_min(unsigned long long v,
                                                           unsigned long long* wred) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long u = __shfl_xor_sync(0xffffffffu, v, o);
    v = u < v ? u : v;
  }
  if ((threadIdx.x & 31) == 0) wred[threadIdx.x >> 5] = v;
  __syncthreads();
  v = wred[0];
#pragma unroll
  for (int w = 1; w < AT_THREADS / 32; ++w) v = wred[w] < v ? wred[w] : v;
  __syncthreads();
  return v;
}

__global__ void __launch_bounds__(AT_THREADS) at_assign_kernel(AtssLossParams p) {
  __shared__ unsigned long long wred[AT_THREADS / 32];
  __shared__ int cand[AT_MAX_LEVELS * AT_TOPK];
  __shared__ float cand_iou[AT_MAX_LEVELS * AT_TOPK];
  __shared__ float s_thr;
  const int g = blockIdx.x;
  if (g >= p.G) return;
  int b = 0;
  while (g >= p.gt_off[b + 1]) ++b;
  const float* gb = p.gt + (size_t)g * 6;
  const float gbox[4] = {gb[0], gb[1], gb[2], gb[3]};
  const float gcx = gb[4], gcy = gb[5];
  if (threadIdx.x == 0) {
    const int lab = p.gt_label[g];
    if (lab < 0 || lab >= p.C) atomicOr(p.status, 1);
  }
  // per level, the topk valid anchors nearest to the 3-D centre: the smallest keys (distance bits,
  // index in the level), so equal distances keep the lower anchor index
  int K = 0;
  for (int l = 0; l < p.L; ++l) {
    const int vh = at_valid_h(p, b, l), vw = at_valid_w(p, b, l), n = vh * vw;
    unsigned long long lst[AT_TOPK];
#pragma unroll
    for (int j = 0; j < AT_TOPK; ++j) lst[j] = ~0ull;
    for (int i = threadIdx.x; i < n; i += AT_THREADS) {
      const int y = i / vw, x = i - y * vw;
      float a[4];
      at_anchor(p, l, x, y, a);
      // bboxes_points - gt_points, pow(2), sum over the two coordinates, sqrt
      const float dx = __fsub_rn(__fmul_rn(__fadd_rn(a[0], a[2]), 0.5f), gcx);
      const float dy = __fsub_rn(__fmul_rn(__fadd_rn(a[1], a[3]), 0.5f), gcy);
      const float d = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
      const unsigned long long key =
          ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)(y * p.W[l] + x);
      if (key < lst[AT_TOPK - 1]) {
        lst[AT_TOPK - 1] = key;
#pragma unroll
        for (int j = AT_TOPK - 1; j > 0; --j) {
          if (lst[j] < lst[j - 1]) {
            const unsigned long long t = lst[j];
            lst[j] = lst[j - 1];
            lst[j - 1] = t;
          }
        }
      }
    }
    const int k = n < AT_TOPK ? n : AT_TOPK;
    for (int j = 0; j < k; ++j) {
      const unsigned long long m = at_block_min(lst[0], wred);
      if (lst[0] == m) {  // keys are unique: one thread owns the minimum
#pragma unroll
        for (int q = 0; q < AT_TOPK - 1; ++q) lst[q] = lst[q + 1];
        lst[AT_TOPK - 1] = ~0ull;
      }
      if (threadIdx.x == 0) cand[K + j] = p.off[l] + (int)(unsigned)(m & 0xffffffffu);
    }
    K += k;
  }
  __syncthreads();
  // the candidates' IoUs (mmdet bbox_overlaps, mode 'iou')
  const float ga = al_area(gbox);
  for (int j = threadIdx.x; j < K; j += AT_THREADS) {
    const int n = cand[j];
    int l = 0;
    while (n >= p.off[l + 1]) ++l;
    const int i = n - p.off[l], y = i / p.W[l], x = i - y * p.W[l];
    float a[4];
    at_anchor(p, l, x, y, a);
    cand_iou[j] = al_iou(gbox, ga, a, al_area(a));
  }
  __syncthreads();
  // threshold mean + std (unbiased) of the candidate IoUs: both in fp64 in candidate order
  // (level, then distance), each rounded to fp32, then added in fp32
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int j = 0; j < K; ++j) s = __dadd_rn(s, (double)cand_iou[j]);
    const double mean = __ddiv_rn(s, (double)K);
    double v = 0.0;
    for (int j = 0; j < K; ++j) {
      const double d = __dsub_rn((double)cand_iou[j], mean);
      v = __dadd_rn(v, __dmul_rn(d, d));
    }
    const float sd = __double2float_rn(__dsqrt_rn(__ddiv_rn(v, (double)(K - 1))));
    s_thr = __fadd_rn(__double2float_rn(mean), sd);
    p.thr[g] = s_thr;
  }
  __syncthreads();
  const float thr = s_thr;
  const unsigned gi = (unsigned)(g - p.gt_off[b]);
  for (int j = threadIdx.x; j < K; j += AT_THREADS) {
    const int n = cand[j];
    int l = 0;
    while (n >= p.off[l + 1]) ++l;
    const int i = n - p.off[l], y = i / p.W[l], x = i - y * p.W[l];
    float a[4];
    at_anchor(p, l, x, y, a);
    const float cx = __fmul_rn(__fadd_rn(a[0], a[2]), 0.5f);
    const float cy = __fmul_rn(__fadd_rn(a[1], a[3]), 0.5f);
    const float e = fminf(fminf(__fsub_rn(cx, gbox[0]), __fsub_rn(cy, gbox[1])),
                          fminf(__fsub_rn(gbox[2], cx), __fsub_rn(gbox[3], cy)));
    const float iou = cand_iou[j];
    // 0.01 as PyTorch compares an fp32 tensor with a Python float: in fp32
    if (iou >= thr && e > 0.01f)
      atomicMax(p.best + (size_t)b * p.N + n,
                ((unsigned long long)__float_as_uint(iou) << 32) | (0xffffffffu - gi));
  }
}

// ---- targets, losses and gradients ----

__global__ void __launch_bounds__(AT_THREADS) at_loss_kernel(AtssLossParams p) {
  __shared__ double red[4][AT_THREADS];
  const int b = blockIdx.y;
  int l = 0;
  while ((int)blockIdx.x >= p.blk_off[l + 1]) ++l;
  const int HW = p.H[l] * p.W[l], C = p.C;
  const int j = ((int)blockIdx.x - p.blk_off[l]) * AT_THREADS + threadIdx.x;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  if (j < HW) {
    const int y = j / p.W[l], x = j - y * p.W[l];
    const int n = p.off[l] + j;
    const size_t i = (size_t)b * p.N + n;
    const bool valid = y < at_valid_h(p, b, l) && x < at_valid_w(p, b, l);
    const unsigned long long key = p.best[i];
    int gi = -1, label = C;
    if (valid && key != 0ull) {
      gi = (int)(0xffffffffu - (unsigned)(key & 0xffffffffu));
      const int lab = p.gt_label[p.gt_off[b] + gi];
      if (lab >= 0 && lab < C) label = lab;  // else flagged by the assign kernel
      else gi = -1;
    }
    const bool pos = gi >= 0;
    const float lw = valid ? 1.f : 0.f;
    float a[4];
    at_anchor(p, l, x, y, a);
    float t[4] = {0.f, 0.f, 0.f, 0.f}, ct = 0.f;
    float tbox[4];
    if (pos) {
      at_encode(p, a, p.gt + (size_t)(p.gt_off[b] + gi) * 6, t);
      at_decode(p, a, t, tbox, nullptr, nullptr);
      ct = at_centerness(a, tbox);
      atomicAdd(p.pos_count + b, 1);
    }
    p.assigned[i] = gi + 1;
    p.labels[i] = label;
    p.label_w[i] = lw;
#pragma unroll
    for (int k = 0; k < 4; ++k) p.targets[i * 4 + k] = t[k];
    p.ctr_t[i] = ct;
    // sigmoid focal loss over every anchor, weighted by its label weight
    const float* cl = p.cls[l] + (size_t)b * C * HW + j;
    float* gc = p.g_cls[l] ? p.g_cls[l] + (size_t)b * C * HW + j : nullptr;
    for (int c = 0; c < C; ++c) {
      float lo, g;
      sigmoid_focal_term(__ldg(cl + (size_t)c * HW), label == c, p.gamma, p.alpha, lo, g);
      acc[0] += (double)(lo * lw);
      if (gc) gc[(size_t)c * HW] = g * lw;
    }
    // GIoU of the decoded positive against its decoded target, weighted by the centerness target,
    // and its gradient through the decode into the label's 4 regression channels
    const float* rg = p.reg[l] + (size_t)b * 4 * C * HW + j;
    double gd[4] = {0.0, 0.0, 0.0, 0.0};
    float gcz = 0.f;
    if (pos) {
      float d[4], pb[4], e[2];
      bool inc[2];
#pragma unroll
      for (int k = 0; k < 4; ++k) d[k] = __ldg(rg + (size_t)(k * C + label) * HW);
      at_decode(p, a, d, pb, e, inc);
      double gp[4];
      const float giou = at_giou(pb, tbox, p.giou_eps, gp);
      acc[1] += (double)__fmul_rn(__fsub_rn(1.f, giou), ct);
      // loss = ct * (1 - giou): d / d pred box = -ct * gp; x1 = gx - gw / 2, x2 = gx + gw / 2
      const double pw = __fsub_rn(a[2], a[0]), ph = __fsub_rn(a[3], a[1]);
      const double gx = -(double)ct * (gp[0] + gp[2]), gy = -(double)ct * (gp[1] + gp[3]);
      const double gw = -(double)ct * 0.5 * (gp[2] - gp[0]);
      const double gh = -(double)ct * 0.5 * (gp[3] - gp[1]);
      gd[0] = gx * pw * p.std_xy;
      gd[1] = gy * ph * p.std_xy;
      gd[2] = inc[0] ? gw * pw * e[0] * p.std_wh : 0.0;
      gd[3] = inc[1] ? gh * ph * e[1] * p.std_wh : 0.0;
      // centerness: binary_cross_entropy_with_logits, (1 - t) x - log_sigmoid(x)
      const float z = __ldg(p.ctr[l] + (size_t)b * HW + j);
      const float ls = __fsub_rn(fminf(0.f, z), log1pf(expf(-fabsf(z))));
      acc[2] += (double)__fsub_rn(__fmul_rn(__fsub_rn(1.f, ct), z), ls);
      gcz = __fsub_rn(1.f / (1.f + expf(-z)), ct);
      acc[3] += (double)ct;
    }
    if (p.g_reg[l]) {
      float* gr = p.g_reg[l] + (size_t)b * 4 * C * HW + j;
      for (int k = 0; k < 4; ++k)
        for (int c = 0; c < C; ++c) gr[(size_t)(k * C + c) * HW] = c == label ? (float)gd[k] : 0.f;
    }
    if (p.g_ctr[l]) p.g_ctr[l][(size_t)b * HW + j] = gcz;
  }
  block_sum_fp64<4, AT_THREADS>(acc, red);
  if (threadIdx.x == 0) {
    double* o = p.partial + ((size_t)b * p.blocks + blockIdx.x) * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k] = red[k][0];
  }
}

// norm[0] = sum_b max(pos_b, 1); norm[1] = the centerness targets summed per level in fp64,
// rounded to fp32 per level and added over levels in fp32 (the reference sums fp32 level sums)
__global__ void __launch_bounds__(AT_THREADS) at_norm_kernel(AtssLossParams p, float* norm) {
  __shared__ double red[4][AT_THREADS];
  for (int l = 0; l < p.L; ++l) {
    const int nb = p.blk_off[l + 1] - p.blk_off[l];
    double v[4] = {0.0, 0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < p.B * nb; i += AT_THREADS) {
      const int b = i / nb, r = i - b * nb;
      const double* s = p.partial + ((size_t)b * p.blocks + p.blk_off[l] + r) * 4;
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] += s[k];
    }
    block_sum_fp64<4, AT_THREADS>(v, red);
    if (threadIdx.x < 4) p.level_sum[l * 4 + threadIdx.x] = red[threadIdx.x][0];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    long long s = 0;
    for (int b = 0; b < p.B; ++b) s += p.pos_count[b] > 1 ? p.pos_count[b] : 1;
    float c = 0.f;
    for (int l = 0; l < p.L; ++l) c = __fadd_rn(c, (float)p.level_sum[l * 4 + 3]);
    norm[0] = (float)s;
    norm[1] = c;
  }
}

// losses / scales [3][L]: cls, bbox, centerness per level.  avg[0] num_total_pos and avg[1] the
// centerness sum, each all-reduced to its mean over ranks under torch.distributed.
//   loss_cls   = w0 * focal / (max(avg0, 1) + FLT_EPSILON)
//   loss_bbox  = w1 * (sum ctr (1 - giou)) / (1 + FLT_EPSILON) / max(avg1, 1)
//   loss_ctr   = w2 * bce / (max(avg0, 1) + FLT_EPSILON)
// NaN everywhere when the forward saw a GT label outside 0..C-1.
__global__ void at_finish_kernel(const double* level_sum, int L, const float* avg,
                                 const float* loss_weight, const int* status, float* losses,
                                 float* scales) {
  const int t = threadIdx.x;
  if (t >= 3 * L) return;
  const int kind = t / L, l = t - kind * L;
  const double eps = (double)FLT_EPSILON;
  const double nts = avg[0] > 1.f ? (double)avg[0] : 1.0;
  const double baf = avg[1] > 1.f ? (double)avg[1] : 1.0;
  const double sc = kind == 1 ? (double)loss_weight[1] / ((1.0 + eps) * baf)
                              : (double)loss_weight[kind] / (nts + eps);
  const int src = kind == 0 ? 0 : (kind == 1 ? 1 : 2);
  losses[t] = *status ? __int_as_float(0x7fc00000) : (float)(level_sum[l * 4 + src] * sc);
  scales[t] = (float)sc;
}

}  // namespace dfm
