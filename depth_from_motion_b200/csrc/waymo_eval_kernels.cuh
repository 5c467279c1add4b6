// Pair stage of Waymo's camera-only LET-3D-AP (compute_detection_let_metrics_main): the
// longitudinal-error-tolerant alignment of a prediction to a GT, the fp64 3-D rotated IoU of
// the aligned pair, the longitudinal affinity and the heading accuracy.  oracle/waymo_let_oracle.py
// restates every step; the products and sums are rounded one by one (no FMA contraction), so
// the two differ only where libdevice's cos / sin / sqrt differ from the host's.
#pragma once

#include <cuda_runtime.h>

namespace dfm {
namespace we {

// the binary's LET config: sensor location, 10 % longitudinal tolerance, 0.5 m floor
constexpr double SENSOR_X = 1.43, SENSOR_Y = 0.0, SENSOR_Z = 2.18;
constexpr double LON_TOL_PCT = 0.1, LON_TOL_MIN = 0.5;
// a box with a dimension at or below this has LET-IoU 0 with every box
constexpr double MIN_BOX_DIM = 0.01;
constexpr double PI = 3.14159265358979323846;

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }

struct P2 {
  double x, y;
};

// counter-clockwise BEV corners of (x, y, z, length, width, height, heading)
__device__ inline void bev_corners(const double* b, P2* c) {
  const double co = cos(b[6]), si = sin(b[6]);
  const double hl = b[3] / 2.0, hw = b[4] / 2.0;
  const double dx[4] = {hl, -hl, -hl, hl}, dy[4] = {hw, hw, -hw, -hw};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    c[i].x = sub(add(b[0], mul(dx[i], co)), mul(dy[i], si));
    c[i].y = add(add(b[1], mul(dx[i], si)), mul(dy[i], co));
  }
}

__device__ __forceinline__ double side(P2 a, P2 b, P2 p) {
  return sub(mul(sub(b.x, a.x), sub(p.y, a.y)), mul(sub(b.y, a.y), sub(p.x, a.x)));
}

// Sutherland-Hodgman clip of the n-gon `in` to the left of a->b.  Each input edge emits at
// most two vertices, so `out` needs room for 2 n.  (An exactly convex polygon gains at most
// one vertex per clip, but with rounding, a box far from the origin can yield vertex sides
// that alternate in sign.)
constexpr int MAX_POLY = 4 << 4;  // 4 corners, doubled by each of the four clips at worst

__device__ inline int clip(const P2* in, int n, P2 a, P2 b, P2* out) {
  int m = 0;
  for (int i = 0; i < n; ++i) {
    const P2 p = in[i], q = in[(i + 1) % n];
    const double sp = side(a, b, p), sq = side(a, b, q);
    if (sp >= 0) out[m++] = p;
    if ((sp >= 0) != (sq >= 0)) {
      const double t = sp / sub(sp, sq);
      out[m++] = P2{add(p.x, mul(t, sub(q.x, p.x))), add(p.y, mul(t, sub(q.y, p.y)))};
    }
  }
  return m;
}

__device__ inline double area(const P2* p, int n) {
  double s = 0.0;
  for (int i = 0; i < n; ++i) {
    const P2 a = p[i], b = p[(i + 1) % n];
    s = add(s, sub(mul(a.x, b.y), mul(b.x, a.y)));
  }
  return mul(0.5, s);
}

__device__ inline double iou3d(const double* a, const double* b) {
  if (fmin(fmin(fmin(a[3], a[4]), fmin(a[5], b[3])), fmin(b[4], b[5])) <= MIN_BOX_DIM) return 0.0;
  const double va = mul(mul(a[3], a[4]), a[5]);
  const double vb = mul(mul(b[3], b[4]), b[5]);
  const double zo = sub(fmin(add(a[2], a[5] / 2), add(b[2], b[5] / 2)),
                        fmax(sub(a[2], a[5] / 2), sub(b[2], b[5] / 2)));
  if (zo <= 0) return 0.0;
  P2 buf[2][MAX_POLY], cb[4];
  bev_corners(a, buf[0]);
  bev_corners(b, cb);
  int n = 4, cur = 0;
  for (int i = 0; i < 4; ++i) {
    if (n < 3) return 0.0;
    n = clip(buf[cur], n, cb[i], cb[(i + 1) % 4], buf[cur ^ 1]);
    cur ^= 1;
  }
  if (n < 3) return 0.0;
  const double inter = mul(fmax(area(buf[cur], n), 0.0), zo);
  const double u = sub(add(va, vb), inter);
  return u > 0 ? inter / u : 0.0;
}

__device__ __forceinline__ double dot3(double ax, double ay, double az, double bx, double by,
                                       double bz) {
  return add(add(mul(ax, bx), mul(ay, by)), mul(az, bz));
}

// (LET-IoU, affinity, heading accuracy) of prediction pd and GT gt
__device__ inline void let_pair(const double* pd, const double* gt, double* out) {
  // alignment: the point of the sensor -> prediction ray closest to the GT centre
  double al[7];
#pragma unroll
  for (int i = 0; i < 7; ++i) al[i] = pd[i];
  const double vx = sub(pd[0], SENSOR_X), vy = sub(pd[1], SENSOR_Y), vz = sub(pd[2], SENSOR_Z);
  const double gx = sub(gt[0], SENSOR_X), gy = sub(gt[1], SENSOR_Y), gz = sub(gt[2], SENSOR_Z);
  const double n2 = dot3(vx, vy, vz, vx, vy, vz);
  if (n2 > 0.0) {
    const double t = dot3(gx, gy, gz, vx, vy, vz) / n2;
    al[0] = add(SENSOR_X, mul(t, vx));
    al[1] = add(SENSOR_Y, mul(t, vy));
    al[2] = add(SENSOR_Z, mul(t, vz));
  }
  out[0] = iou3d(al, gt);
  // longitudinal affinity
  const double rg = sqrt(dot3(gx, gy, gz, gx, gy, gz));
  const double tol = fmax(mul(LON_TOL_PCT, rg), LON_TOL_MIN);
  double e = 0.0;
  if (rg > 0.0)
    e = dot3(sub(pd[0], gt[0]), sub(pd[1], gt[1]), sub(pd[2], gt[2]), gx, gy, gz) / rg;
  out[1] = sub(1.0, fmin(fabs(e) / tol, 1.0));
  // heading accuracy
  double d = fmod(fabs(sub(pd[6], gt[6])), mul(2.0, PI));
  d = fmin(d, sub(mul(2.0, PI), d));
  out[2] = sub(1.0, d / PI);
}

// out[(i * k + j) * 3 + c]: pair (prediction i, GT j)
__global__ void let_iou_kernel(const double* __restrict__ pd, const double* __restrict__ gt,
                               int n, int k, double* __restrict__ out) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= (long long)n * k) return;
  const int i = (int)(q / k), j = (int)(q % k);
  double p[7], g[7], r[3];
#pragma unroll
  for (int c = 0; c < 7; ++c) {
    p[c] = pd[(size_t)i * 7 + c];
    g[c] = gt[(size_t)j * 7 + c];
  }
  let_pair(p, g, r);
#pragma unroll
  for (int c = 0; c < 3; ++c) out[q * 3 + c] = r[c];
}

}  // namespace we
}  // namespace dfm
