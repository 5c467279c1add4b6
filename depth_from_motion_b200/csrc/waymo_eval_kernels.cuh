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


// ---- WaymoDataset.convert_valid_bboxes + bbox2result_kitti, load_mode 'lidar_frame' ----
// One thread per LiDAR box of the set (CSR: box_off[F + 1]).  float32 throughout, each
// product and sum rounded on its own in the order of the reference's torch / numpy calls:
// limit_yaw(0.5, 2 pi); Box3DMode LIDAR -> CAM with rt = R0_rect @ Tr_velo_to_cam (the
// caller's float32 product); the camera box's corners projected with P0; the min / max of
// the projection clipped to image_shape; alpha = -arctan2(-y, x) + ry_cam.  A box is kept iff
// its centre lies strictly inside the limit range.  The matrix products of the reference run
// through BLAS, whose summation order is not fixed, so the values agree with it to float32
// rounding; the keep mask depends on the input centre alone and is exact.
// out columns: the anno's bbox[4] (clipped) alpha location[3] dimensions[3] rotation_y, then
// convert_valid_bboxes' LiDAR yaw and its unclipped 2-D box[4]
constexpr int KC_W = 17;

__device__ __forceinline__ float fmulr(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float faddr(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsubr(float a, float b) { return __fsub_rn(a, b); }

// limit_period(val, 0.5, 2 pi) of a float32 tensor: the period is rounded to float32
__device__ __forceinline__ float limit_2pi(float v) {
  const float period = (float)(2.0 * PI);
  return fsubr(v, fmulr(floorf(faddr(__fdiv_rn(v, period), 0.5f)), period));
}

// one row of a [K, 4] @ [4, 4]^T product: sum_j a[j] * m[row][j], j ascending
__device__ __forceinline__ float row_dot4(const float* m, float a0, float a1, float a2, float a3) {
  return faddr(faddr(faddr(fmulr(a0, m[0]), fmulr(a1, m[1])), fmulr(a2, m[2])), fmulr(a3, m[3]));
}

__global__ void kitti_convert_kernel(int F, int K, const float* __restrict__ boxes,
                                     const int* __restrict__ box_off,
                                     const float* __restrict__ calib,
                                     const int* __restrict__ image_shape,
                                     const long long* __restrict__ image_idx, float lx0, float ly0,
                                     float lz0, float lx1, float ly1, float lz1,
                                     unsigned char* __restrict__ keep, float* __restrict__ out,
                                     long long* __restrict__ sample_idx) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  int lo = 0, hi = F - 1;   // the last frame with box_off[f] <= k
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (box_off[mid] <= k) lo = mid;
    else hi = mid - 1;
  }
  const int f = lo;
  const float* b = boxes + (size_t)k * 7;
  const float* rt = calib + (size_t)f * 32;   // R0_rect @ Tr_velo_to_cam, [4][4]
  const float* P0 = rt + 16;                  // [4][4]
  const float x = b[0], y = b[1], z = b[2], dx = b[3], dy = b[4], dz = b[5];
  const float yaw = limit_2pi(b[6]);
  keep[k] = (x > lx0 && y > ly0 && z > lz0 && x < lx1 && y < ly1 && z < lz1) ? 1 : 0;
  sample_idx[k] = image_idx[f];
  // Box3DMode.convert: xyz @ rt^T, sizes (dx, dz, dy), yaw -> limit_period(-yaw - pi / 2)
  const float cx = row_dot4(rt, x, y, z, 1.f), cy = row_dot4(rt + 4, x, y, z, 1.f),
              cz = row_dot4(rt + 8, x, y, z, 1.f);
  const float ry = limit_2pi(fsubr(-yaw, (float)(PI / 2)));
  const float dims[3] = {dx, dz, dy};
  // CameraInstance3DBoxes.corners: dims * (unit corner - (0.5, 1, 0.5)), rotated about y
  const float rc = cosf(ry), rs = sinf(ry);
  float u0 = INFINITY, v0 = INFINITY, u1 = -INFINITY, v1 = -INFINITY;
  bool nan = false;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const float n0 = (float)((c >> 2) & 1) - 0.5f, n1 = (float)((c >> 1) & 1) - 1.f,
                n2 = (float)(c & 1) - 0.5f;
    const float c0 = fmulr(dims[0], n0), c1 = fmulr(dims[1], n1), c2 = fmulr(dims[2], n2);
    const float px = faddr(faddr(fmulr(c0, rc), fmulr(c2, rs)), cx);
    const float py = faddr(c1, cy);
    const float pz = faddr(faddr(fmulr(c0, -rs), fmulr(c2, rc)), cz);
    // points_cam2img: (p, 1) @ P0^T, then the first two over the third
    const float w = row_dot4(P0 + 8, px, py, pz, 1.f);
    const float u = __fdiv_rn(row_dot4(P0, px, py, pz, 1.f), w);
    const float v = __fdiv_rn(row_dot4(P0 + 4, px, py, pz, 1.f), w);
    nan |= u != u || v != v;   // torch.min / max propagate NaN
    u0 = fminf(u0, u);
    v0 = fminf(v0, v);
    u1 = fmaxf(u1, u);
    v1 = fmaxf(v1, v);
  }
  if (nan) u0 = v0 = u1 = v1 = NAN;
  // bbox2result_kitti: bbox[2:] = min(bbox[2:], (W, H)), bbox[:2] = max(bbox[:2], 0)
  const float H = (float)image_shape[2 * f], W = (float)image_shape[2 * f + 1];
  float* o = out + (size_t)k * KC_W;
  o[0] = u0 < 0.f ? 0.f : u0;
  o[1] = v0 < 0.f ? 0.f : v0;
  o[2] = u1 > W ? W : u1;
  o[3] = v1 > H ? H : v1;
  o[4] = faddr(-atan2f(-y, x), ry);
  o[5] = cx;
  o[6] = cy;
  o[7] = cz;
  o[8] = dims[0];
  o[9] = dims[1];
  o[10] = dims[2];
  o[11] = ry;
  o[12] = yaw;
  o[13] = u0;
  o[14] = v0;
  o[15] = u1;
  o[16] = v1;
}

}  // namespace we
}  // namespace dfm
