// Training losses of the anchor heads (Anchor3DHead.loss / loss_single, anchor3d_head.py:199-406,
// LIGAAnchor3DHead.loss_single, liga_anchor3d_head.py:130-226) with the target assignment of
// AnchorTrainMixin (train_mixins.py:102-318), for a batch of B samples of one feature level:
//
//   al_max_kernel      per anchor: nearest-BEV IoU with every GT its assigner sees, max / argmax;
//                      per GT: max over the assigner's anchors (atomicMax on the fp32 bits, which
//                      order non-negative floats; the result does not depend on thread order)
//   al_assign_kernel   MaxIoUAssigner's thresholds and low-quality pass, PseudoSampler, the
//                      DeltaXYZWLHRBBoxCoder targets and the direction targets; positives per sample
//   al_loss_kernel     focal / SmoothL1 / direction CE (and for LIGA the 3-D IoU loss of the
//                      positives) with their gradients, on the NCHW head outputs; per-block sums
//                      in fp64, reduced in a fixed tree order
//   al_count_kernel    num_total_samples = sum_b max(pos_b, 1), on the device
//   al_finish_kernel   the per-block sums in a fixed order, the normalisers, the loss values and
//                      the scale each stored gradient takes in backward
//
// The IoU that decides positives is computed op for op as the reference's fp32 PyTorch ops run on
// CUDA: explicitly rounded intrinsics (no FMA contraction) and a * (1 / s) wherever PyTorch divides
// a CUDA tensor by a Python scalar.
#pragma once
#include <cuda_runtime.h>

#include <cfloat>
#include <cstdint>

#include "box_post_kernels.cuh"

namespace dfm {

constexpr int AL_MAX_GT = 1024;     // GT boxes per sample (kept in shared memory)
constexpr int AL_MAX_SIZES = 8;     // anchor sizes = assigners
constexpr int AL_MAX_CLASSES = 16;  // sigmoid score columns
constexpr int AL_THREADS = 256;

struct AnchorLossParams {
  int B, HW, A, R, S, C, N;      // anchors per cell A = S * R; N = HW * A
  int per_class, sin_diff, use_dir, with_iou;
  float pos_thr[AL_MAX_SIZES], neg_thr[AL_MAX_SIZES], min_pos[AL_MAX_SIZES];
  float pos_weight;              // train_cfg.pos_weight (<= 0: 1)
  float gamma, alpha, beta, inv_beta;
  float dir_offset, dir_limit_offset;
  // fp32 constants as PyTorch forms them from Python floats on CUDA
  float pi_f, inv_pi_f, quarter_pi_f, two_pi_f, inv_two_pi_f, inv_pi_bin_f;
  const float* anchors;          // [N][7]
  const float* anchor_bev;       // [N][4] nearest_bev (x1, y1, x2, y2)
  const float* anchor_area;      // [N]
  // per forward
  const float* cls;              // [B][A * C][HW]
  const float* reg;              // [B][A * 7][HW]
  const float* dir;              // [B][A * 2][HW] (use_dir)
  const float* gt;               // [G][7]
  const int* gt_label;           // [G]
  const int* gt_off;             // [B + 1]
  int G;
  float* g_cls;                  // gradients of the unnormalised sums, or null
  float* g_reg;
  float* g_dir;
  float* g_iou;
  // workspace
  unsigned* gt_max;              // [S][G] fp32 bits
  float* max_iou;                // [B][N]
  int* argmax;                   // [B][N]
  int* assigned;                 // [B][N] -1 ignore, 0 negative, g + 1 (index in the sample)
  int* labels;                   // [B][N]
  float* label_w;                // [B][N]
  float* targets;                // [B][N][7]
  int* dir_t;                    // [B][N]
  int* pos_count;                // [B]
  int* status;                   // bit 0: a GT label outside 0..C-1
  double* partial;               // [B * blocks][4]
  int blocks;                    // blocks per sample of the anchor grid
};

// LiDARInstance3DBoxes.nearest_bev of one box: limit_period(yaw, 0.5, pi), abs, swap dx / dy past
// pi / 4, then (centre - dims / 2, centre + dims / 2)
__device__ __forceinline__ void al_nearest_bev(const AnchorLossParams& p, const float* b,
                                               float* o) {
  const float r = b[6];
  const float f = floorf(__fadd_rn(__fmul_rn(r, p.inv_pi_f), 0.5f));
  const float nr = fabsf(__fsub_rn(r, __fmul_rn(f, p.pi_f)));
  const bool swap = nr > p.quarter_pi_f;
  const float dx = swap ? b[4] : b[3], dy = swap ? b[3] : b[4];
  const float hx = __fmul_rn(dx, 0.5f), hy = __fmul_rn(dy, 0.5f);
  o[0] = __fsub_rn(b[0], hx);
  o[1] = __fsub_rn(b[1], hy);
  o[2] = __fadd_rn(b[0], hx);
  o[3] = __fadd_rn(b[1], hy);
}

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

__global__ void al_anchor_bev_kernel(AnchorLossParams p, float* bev, float* area) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= p.N) return;
  float o[4];
  al_nearest_bev(p, p.anchors + (size_t)n * 7, o);
#pragma unroll
  for (int k = 0; k < 4; ++k) bev[(size_t)n * 4 + k] = o[k];
  area[n] = al_area(o);
}

// the sample's GT in shared memory: nearest-BEV box, area, label
struct AlGtSmem {
  float box[AL_MAX_GT][4];
  float area[AL_MAX_GT];
  int label[AL_MAX_GT];
};

__device__ __forceinline__ int al_load_gt(const AnchorLossParams& p, int b, AlGtSmem& s) {
  const int off = p.gt_off[b], n = p.gt_off[b + 1] - off;
  for (int g = threadIdx.x; g < n; g += blockDim.x) {
    al_nearest_bev(p, p.gt + (size_t)(off + g) * 7, s.box[g]);
    s.area[g] = al_area(s.box[g]);
    s.label[g] = p.gt_label[off + g];
    if (s.label[g] < 0 || s.label[g] >= p.C) atomicOr(p.status, 1);
  }
  __syncthreads();
  return n;
}

__global__ void __launch_bounds__(AL_THREADS) al_max_kernel(AnchorLossParams p) {
  __shared__ AlGtSmem s;
  const int b = blockIdx.y, n = blockIdx.x * blockDim.x + threadIdx.x;
  const int ng = al_load_gt(p, b, s);
  if (n >= p.N) return;
  const int sz = (n % p.A) / p.R, off = p.gt_off[b];
  float ab[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) ab[k] = __ldg(p.anchor_bev + (size_t)n * 4 + k);
  const float aa = __ldg(p.anchor_area + n);
  float best = -1.f;
  int arg = 0;
  for (int g = 0; g < ng; ++g) {
    if (p.per_class && s.label[g] != sz) continue;
    const float iou = al_iou(s.box[g], s.area[g], ab, aa);
    if (iou > best) {  // first maximum wins, as torch.max over the GT axis
      best = iou;
      arg = g;
    }
    if (iou > 0.f) atomicMax(p.gt_max + (size_t)sz * p.G + off + g, __float_as_uint(iou));
  }
  p.max_iou[(size_t)b * p.N + n] = best;
  p.argmax[(size_t)b * p.N + n] = arg;
}

__global__ void __launch_bounds__(AL_THREADS) al_assign_kernel(AnchorLossParams p) {
  __shared__ AlGtSmem s;
  __shared__ int npos;
  const int b = blockIdx.y, n = blockIdx.x * blockDim.x + threadIdx.x;
  if (threadIdx.x == 0) npos = 0;
  const int ng = al_load_gt(p, b, s);
  if (n < p.N) {
    const int sz = (n % p.A) / p.R, off = p.gt_off[b];
    const size_t i = (size_t)b * p.N + n;
    const float best = p.max_iou[i];
    int as = 0;  // no GT for this assigner: every anchor is negative
    if (best >= 0.f) {
      as = best < p.neg_thr[sz] ? 0 : -1;
      if (best >= p.pos_thr[sz]) as = p.argmax[i] + 1;
      float ab[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) ab[k] = __ldg(p.anchor_bev + (size_t)n * 4 + k);
      const float aa = __ldg(p.anchor_area + n);
      // low-quality matches: every anchor at a GT's best IoU, GT in index order, later ones win
      for (int g = 0; g < ng; ++g) {
        if (p.per_class && s.label[g] != sz) continue;
        const float gm = __uint_as_float(p.gt_max[(size_t)sz * p.G + off + g]);
        if (gm >= p.min_pos[sz] && al_iou(s.box[g], s.area[g], ab, aa) == gm) as = g + 1;
      }
    }
    p.assigned[i] = as;
    int label = p.C;
    float lw = as == 0 ? 1.f : 0.f;
    float t[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int dt = 0;
    if (as > 0) {
      const float* an = p.anchors + (size_t)n * 7;
      const float* gb = p.gt + (size_t)(off + as - 1) * 7;
      label = s.label[as - 1];
      lw = p.pos_weight <= 0.f ? 1.f : p.pos_weight;
      // DeltaXYZWLHRBBoxCoder.encode(anchor, gt)
      const float xa = an[0], ya = an[1], wa = an[3], la = an[4], ha = an[5], ra = an[6];
      const float xg = gb[0], yg = gb[1], wg = gb[3], lg = gb[4], hg = gb[5], rg = gb[6];
      const float za = __fadd_rn(an[2], __fmul_rn(ha, 0.5f));
      const float zg = __fadd_rn(gb[2], __fmul_rn(hg, 0.5f));
      const float diag = __fsqrt_rn(__fadd_rn(__fmul_rn(la, la), __fmul_rn(wa, wa)));
      t[0] = __fdiv_rn(__fsub_rn(xg, xa), diag);
      t[1] = __fdiv_rn(__fsub_rn(yg, ya), diag);
      t[2] = __fdiv_rn(__fsub_rn(zg, za), ha);
      t[3] = logf(__fdiv_rn(wg, wa));
      t[4] = logf(__fdiv_rn(lg, la));
      t[5] = logf(__fdiv_rn(hg, ha));
      t[6] = __fsub_rn(rg, ra);
      // get_direction_target
      const float v = __fsub_rn(__fadd_rn(t[6], ra), p.dir_offset);
      const float f = floorf(__fadd_rn(__fmul_rn(v, p.inv_two_pi_f), p.dir_limit_offset));
      const float o = __fsub_rn(v, __fmul_rn(f, p.two_pi_f));
      dt = (int)floorf(__fmul_rn(o, p.inv_pi_bin_f));
      dt = dt < 0 ? 0 : (dt > 1 ? 1 : dt);
      atomicAdd(&npos, 1);
    }
    p.labels[i] = label;
    p.label_w[i] = lw;
#pragma unroll
    for (int k = 0; k < 7; ++k) p.targets[i * 7 + k] = t[k];
    p.dir_t[i] = dt;
  }
  __syncthreads();
  if (threadIdx.x == 0 && npos) atomicAdd(p.pos_count + b, npos);
}

// ---- 1 - IoU3D (mmcv diff_iou_rotated_3d) and its gradient with respect to the first box ----

// a value and its derivatives with respect to the predicted BEV box (x, y, dx, dy, yaw)
struct Dual5 {
  double v, d[5];
};
__device__ __forceinline__ Dual5 dconst(double v) {
  Dual5 r;
  r.v = v;
#pragma unroll
  for (int k = 0; k < 5; ++k) r.d[k] = 0.0;
  return r;
}
__device__ __forceinline__ Dual5 operator+(const Dual5& a, const Dual5& b) {
  Dual5 r;
  r.v = a.v + b.v;
#pragma unroll
  for (int k = 0; k < 5; ++k) r.d[k] = a.d[k] + b.d[k];
  return r;
}
__device__ __forceinline__ Dual5 operator-(const Dual5& a, const Dual5& b) {
  Dual5 r;
  r.v = a.v - b.v;
#pragma unroll
  for (int k = 0; k < 5; ++k) r.d[k] = a.d[k] - b.d[k];
  return r;
}
__device__ __forceinline__ Dual5 operator*(const Dual5& a, const Dual5& b) {
  Dual5 r;
  r.v = a.v * b.v;
#pragma unroll
  for (int k = 0; k < 5; ++k) r.d[k] = a.d[k] * b.v + a.v * b.d[k];
  return r;
}
__device__ __forceinline__ Dual5 operator/(const Dual5& a, const Dual5& b) {
  Dual5 r;
  r.v = a.v / b.v;
#pragma unroll
  for (int k = 0; k < 5; ++k) r.d[k] = (a.d[k] - r.v * b.d[k]) / b.v;
  return r;
}

// Intersection area of the predicted rectangle (duals) and the target rectangle (constants):
// Sutherland-Hodgman clipping of the prediction's corners by the target's edges, then the shoelace
// sum.  Every vertex carries its derivatives: a corner of the prediction through the box
// parameters, a crossing of a prediction edge with a target edge through the edge's end points, a
// target corner with none.  Both rectangles are counter-clockwise (mmcv box2corners order).
__device__ __noinline__ Dual5 al_bev_intersection(const Dual5* px, const Dual5* py,
                                                  const double* qx, const double* qy) {
  // a convex quad clipped by a convex quad has at most 8 vertices; rounding that makes nearly
  // collinear vertices alternate in and out could add more, so every push is bounded
  constexpr int MAXV = 10;
  Dual5 vx[2][MAXV], vy[2][MAXV];
  int n = 4, cur = 0;
  for (int i = 0; i < 4; ++i) {
    vx[0][i] = px[i];
    vy[0][i] = py[i];
  }
  for (int e = 0; e < 4 && n > 0; ++e) {
    const double ax = qx[e], ay = qy[e];
    const double ex = qx[(e + 1) & 3] - ax, ey = qy[(e + 1) & 3] - ay;
    const int nxt = cur ^ 1;
    int m = 0;
    for (int i = 0; i < n; ++i) {
      const int j = i + 1 == n ? 0 : i + 1;
      const Dual5 si = dconst(ex) * (vy[cur][i] - dconst(ay)) - dconst(ey) * (vx[cur][i] - dconst(ax));
      const Dual5 sj = dconst(ex) * (vy[cur][j] - dconst(ay)) - dconst(ey) * (vx[cur][j] - dconst(ax));
      const bool in_i = si.v >= 0.0, in_j = sj.v >= 0.0;
      if (in_i && m < MAXV) {
        vx[nxt][m] = vx[cur][i];
        vy[nxt][m] = vy[cur][i];
        ++m;
      }
      if (in_i != in_j && m < MAXV) {
        const Dual5 t = si / (si - sj);
        vx[nxt][m] = vx[cur][i] + t * (vx[cur][j] - vx[cur][i]);
        vy[nxt][m] = vy[cur][i] + t * (vy[cur][j] - vy[cur][i]);
        ++m;
      }
    }
    n = m;
    cur = nxt;
  }
  Dual5 area = dconst(0.0);
  for (int i = 0; i < n; ++i) {
    const int j = i + 1 == n ? 0 : i + 1;
    area = area + (vx[cur][i] * vy[cur][j] - vy[cur][i] * vx[cur][j]);
  }
  area = area * dconst(0.5);
  if (area.v < 0.0) area = dconst(0.0) - area;
  return area;
}

// 1 - IoU3D(pred, tgt) for decoded boxes (x, y, z, dx, dy, dz, yaw), z read as the centre as mmcv
// does; grad[7] = its derivatives with respect to pred
__device__ __noinline__ double al_iou3d_loss(const float* pred, const float* tgt, double* grad) {
  Dual5 px[4], py[4];
  double qx[4], qy[4];
  const double sx[4] = {0.5, -0.5, -0.5, 0.5}, sy[4] = {0.5, 0.5, -0.5, -0.5};
  Dual5 x = dconst(pred[0]), y = dconst(pred[1]), w = dconst(pred[3]), l = dconst(pred[4]);
  x.d[0] = 1.0;
  y.d[1] = 1.0;
  w.d[2] = 1.0;
  l.d[3] = 1.0;
  double sr, cr;
  sincos((double)pred[6], &sr, &cr);
  Dual5 c = dconst(cr), s = dconst(sr);
  c.d[4] = -sr;
  s.d[4] = cr;
  double st, ct;
  sincos((double)tgt[6], &st, &ct);
  for (int i = 0; i < 4; ++i) {
    const Dual5 ox = dconst(sx[i]) * w, oy = dconst(sy[i]) * l;
    px[i] = ox * c - oy * s + x;
    py[i] = ox * s + oy * c + y;
    const double tx = sx[i] * tgt[3], ty = sy[i] * tgt[4];
    qx[i] = tx * ct - ty * st + tgt[0];
    qy[i] = tx * st + ty * ct + tgt[1];
  }
  const Dual5 a2 = al_bev_intersection(px, py, qx, qy);
  const double z1 = pred[2], h1 = pred[5], z2 = tgt[2], h2 = tgt[5];
  const double zmax1 = z1 + h1 * 0.5, zmin1 = z1 - h1 * 0.5;
  const double zmax2 = z2 + h2 * 0.5, zmin2 = z2 - h2 * 0.5;
  const double top = fmin(zmax1, zmax2), bot = fmax(zmin1, zmin2);
  const double zr = top - bot, zo = zr > 0.0 ? zr : 0.0;
  // torch.minimum / maximum split a tie's gradient in half; clamp(min=0) passes it at 0
  const double gtop = zmax1 < zmax2 ? 1.0 : (zmax1 == zmax2 ? 0.5 : 0.0);
  const double gbot = zmin1 > zmin2 ? 1.0 : (zmin1 == zmin2 ? 0.5 : 0.0);
  const double pass = zr >= 0.0 ? 1.0 : 0.0;
  const double dzo_dz = pass * (gtop - gbot), dzo_dh = pass * 0.5 * (gtop + gbot);
  const double inter = a2.v * zo;
  const double v1 = (double)pred[3] * pred[4] * pred[5];
  const double v2 = (double)tgt[3] * tgt[4] * tgt[5];
  const double uni = v1 + v2 - inter;
  // d(inter / union) = (d inter * union - inter * (d v1 - d inter)) / union^2
  double di[7] = {a2.d[0] * zo, a2.d[1] * zo, a2.v * dzo_dz, a2.d[2] * zo, a2.d[3] * zo,
                  a2.v * dzo_dh, a2.d[4] * zo};
  const double dv[7] = {0.0, 0.0, 0.0, (double)pred[4] * pred[5], (double)pred[3] * pred[5],
                        (double)pred[3] * pred[4], 0.0};
  const double u2 = uni * uni;
#pragma unroll
  for (int k = 0; k < 7; ++k) grad[k] = -(di[k] * uni - inter * (dv[k] - di[k])) / u2;
  return 1.0 - inter / uni;
}

// ---- loss-and-gradient pass ----

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

__device__ __forceinline__ void al_block_sum4(double* v, double (*red)[AL_THREADS]) {
  block_sum_fp64<4, AL_THREADS>(v, red);
}

__global__ void __launch_bounds__(AL_THREADS) al_loss_kernel(AnchorLossParams p) {
  __shared__ double red[4][AL_THREADS];
  const int b = blockIdx.y, n = blockIdx.x * blockDim.x + threadIdx.x;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  if (n < p.N) {
    const int cell = n / p.A, a = n % p.A;
    const size_t i = (size_t)b * p.N + n;
    const int label = p.labels[i];
    const float lw = p.label_w[i];
    // sigmoid focal loss (mmcv sigmoid_focal_loss forward and backward, fp32), weighted per anchor
    const float* cl = p.cls + ((size_t)b * p.A * p.C + (size_t)a * p.C) * p.HW + cell;
    float* gc = p.g_cls ? p.g_cls + ((size_t)b * p.A * p.C + (size_t)a * p.C) * p.HW + cell
                        : nullptr;
    for (int c = 0; c < p.C; ++c) {
      float l, g;
      sigmoid_focal_term(__ldg(cl + (size_t)c * p.HW), label == c, p.gamma, p.alpha, l, g);
      acc[0] += (double)(l * lw);
      if (gc) gc[(size_t)c * p.HW] = g * lw;
    }
    const bool pos = label >= 0 && label < p.C;
    const float* rg = p.reg + ((size_t)b * p.A * 7 + (size_t)a * 7) * p.HW + cell;
    float pr7[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) pr7[k] = pos ? __ldg(rg + (size_t)k * p.HW) : 0.f;
    const float* tg = p.targets + i * 7;
    // SmoothL1 over the positives, channel 6 as sin(p)cos(t) against cos(p)sin(t).  Forward and
    // gradient round as mmdet's smooth_l1_loss and its autograd do in fp32 on CUDA: no FMA
    // contraction (sin(p) cos(t) - cos(p) sin(t) is exactly 0 at p == t), / beta as
    // * (1 / beta)_f, and the sin difference's two gradient paths summed last
    float gr[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      gr[k] = 0.f;
      if (!pos) continue;
      const float t = tg[k];
      const bool sin6 = k == 6 && p.sin_diff;
      float d, sp = 0.f, cp = 0.f, st = 0.f, ct = 0.f;
      if (sin6) {
        sincosf(pr7[6], &sp, &cp);
        sincosf(t, &st, &ct);
        d = __fsub_rn(__fmul_rn(sp, ct), __fmul_rn(cp, st));
      } else {
        d = __fsub_rn(pr7[k], t);
      }
      const float ad = fabsf(d);
      const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
      float g;
      if (ad < p.beta) {
        acc[1] += (double)__fmul_rn(__fmul_rn(__fmul_rn(0.5f, ad), ad), p.inv_beta);
        g = __fmul_rn(ad, p.inv_beta) * sg;
      } else {
        acc[1] += (double)__fsub_rn(ad, __fmul_rn(0.5f, p.beta));
        g = sg;
      }
      gr[k] = sin6 ? __fadd_rn(__fmul_rn(__fmul_rn(g, ct), cp), __fmul_rn(__fmul_rn(g, st), sp))
                   : g;
    }
    if (p.g_reg) {
      float* gp = p.g_reg + ((size_t)b * p.A * 7 + (size_t)a * 7) * p.HW + cell;
#pragma unroll
      for (int k = 0; k < 7; ++k) gp[(size_t)k * p.HW] = gr[k];
    }
    // softmax cross-entropy over the two direction logits of the positives
    if (p.use_dir) {
      const float* dr = p.dir + ((size_t)b * p.A * 2 + (size_t)a * 2) * p.HW + cell;
      float g0 = 0.f, g1 = 0.f;
      if (pos) {
        const float d0 = __ldg(dr), d1 = __ldg(dr + p.HW);
        const float m = fmaxf(d0, d1);
        const float e0 = expf(d0 - m), e1 = expf(d1 - m), se = e0 + e1;
        const int t = p.dir_t[i];
        acc[2] += (double)(logf(se) + m - (t ? d1 : d0));
        g0 = e0 / se - (t == 0 ? 1.f : 0.f);
        g1 = e1 / se - (t == 1 ? 1.f : 0.f);
      }
      if (p.g_dir) {
        float* gd = p.g_dir + ((size_t)b * p.A * 2 + (size_t)a * 2) * p.HW + cell;
        gd[0] = g0;
        gd[p.HW] = g1;
      }
    }
    // 1 - IoU3D of the decoded prediction and target of each positive against its own anchor
    if (p.with_iou) {
      double gi[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      if (pos) {
        const float* an = p.anchors + (size_t)n * 7;
        float bp[7], bt[7];
        bp_decode_box(pr7, an, bp);
        bp_decode_box(tg, an, bt);
        // iou3d_loss's torch.where(isnan(target), pred, target); the gradient flows through the
        // first box only (see dfm_anchor_loss_forward in the header)
#pragma unroll
        for (int k = 0; k < 7; ++k)
          if (isnan(bt[k])) bt[k] = bp[k];
        double gb[7];
        acc[3] += al_iou3d_loss(bp, bt, gb);
        // through the decode: x, y scale by the diagonal, sizes by exp, z by ha and -h / 2
        const float wa = an[3], la = an[4], ha = an[5];
        const double diag = __fsqrt_rn(__fadd_rn(__fmul_rn(la, la), __fmul_rn(wa, wa)));
        gi[0] = gb[0] * diag;
        gi[1] = gb[1] * diag;
        gi[2] = gb[2] * ha;
        gi[3] = gb[3] * bp[3];
        gi[4] = gb[4] * bp[4];
        gi[5] = gb[5] * bp[5] - gb[2] * 0.5 * bp[5];
        gi[6] = gb[6];
      }
      if (p.g_iou) {
        float* gp = p.g_iou + ((size_t)b * p.A * 7 + (size_t)a * 7) * p.HW + cell;
#pragma unroll
        for (int k = 0; k < 7; ++k) gp[(size_t)k * p.HW] = (float)gi[k];
      }
    }
  }
  al_block_sum4(acc, red);
  if (threadIdx.x == 0) {
    double* o = p.partial + ((size_t)b * p.blocks + blockIdx.x) * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k] = red[k][0];
  }
}

__global__ void al_count_kernel(const int* pos_count, int B, float* norm) {
  if (threadIdx.x != 0) return;
  long long s = 0;
  for (int b = 0; b < B; ++b) s += pos_count[b] > 1 ? pos_count[b] : 1;
  *norm = (float)s;
}

// losses[k] = loss_weight[k] * sum_k / denom_k; scales[k] = loss_weight[k] / denom_k.
// NaN when the forward saw a GT label outside 0..C-1.
// Anchor3DHead: denom = num_total_samples + FLT_EPSILON for every term.  LIGA: cls divides by
// (avg + clamp) + FLT_EPSILON, the others by max(avg, clamp) + FLT_EPSILON.
__global__ void __launch_bounds__(AL_THREADS) al_finish_kernel(const double* partial, int nparts,
                                                               const float* avg, int liga,
                                                               float clamp_value,
                                                               const float* loss_weight,
                                                               const int* status,
                                                               float* losses, float* scales) {
  __shared__ double red[4][AL_THREADS];
  double v[4] = {0.0, 0.0, 0.0, 0.0};
  for (int i = threadIdx.x; i < nparts; i += AL_THREADS) {
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] += partial[(size_t)i * 4 + k];
  }
  al_block_sum4(v, red);
  if (threadIdx.x < 4) {
    const int k = threadIdx.x;
    const double a = *avg, eps = (double)FLT_EPSILON;
    double denom;
    if (!liga)
      denom = a + eps;
    else if (k == 0)
      denom = (a + clamp_value) + eps;
    else
      denom = (a > clamp_value ? a : (double)clamp_value) + eps;
    const double sc = (double)loss_weight[k] / denom;
    // an out-of-range GT label (checked on the device, so the host never waits) poisons every
    // loss rather than passing silently
    losses[k] = *status ? __int_as_float(0x7fc00000) : (float)(red[k][0] * sc);
    scales[k] = (float)sc;
  }
}

}  // namespace dfm
