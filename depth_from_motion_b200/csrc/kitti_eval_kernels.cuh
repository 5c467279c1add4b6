// KITTI evaluation (mmdet3d core/evaluation/kitti_utils/eval.py, kitti_eval -> do_eval ->
// eval_class) for one set of N frames, ground truth and detections in CSR form:
//
//   ignore codes per (class, difficulty, frame)                      (clean_data, eval.py:30-82)
//   per part of frames: overlaps per (metric, frame, dt, gt), only within a frame
//                       (calculate_iou_partly), then pass 1: TP scores per (config, frame)
//                       (compute_statistics_jit, compute_fp=False)
//   thresholds per config: bitonic sort of its TP scores + the 41-point pick (get_thresholds)
//   per part of frames: overlaps again, then pass 2: tp / fp / fn / similarity per (config,
//                       threshold, frame)   (compute_fp=True)
//   reduce per (config, threshold): integer counts, similarity summed in frame order
//
// A part is a run of whole frames whose overlaps fit the handle's limit.  Every per-frame
// result (TP scores, counts, similarity term) depends on that frame's overlaps alone, the
// counts are integers and the similarity is summed in frame order afterwards, so the results
// are bitwise the same for any division into parts.
//
// A config is (metric slot, class slot, difficulty, overlap set), indexed in the order
// eval_class walks them.  The rotated IoU restates rotate_iou.py op for op, typed as numba
// types it: float32 arithmetic, float64 where a float64 literal or an integer enters, libdevice
// cosf / sinf, and every product and sum rounded on its own (no FMA contraction).  The 2-D and
// 3-D overlaps follow image_box_overlap / d3_box_overlap_kernel with the dtypes of the caller's
// arrays (float32 detections compute their box areas in float32, as numba does).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace dfm {
namespace ke {

constexpr int MAX_T = 41;          // N_SAMPLE_PTS: thresholds per config
constexpr int MAX_DT_FRAME = 1024; // detections per frame (assigned-detection bit mask)
constexpr int GT_W = 14;           // bbox[4] alpha loc[3] dims[3] rot_y occluded truncated
constexpr int DT_W = 13;           // bbox[4] alpha loc[3] dims[3] rot_y score
constexpr int CODE_DONTCARE = 8;   // gt code bit: the name is exactly "DontCare"
// f32 flags: which input arrays the caller held as float32
constexpr int F_GT_BBOX = 1, F_DT_BBOX = 2, F_GT_3D = 4, F_DT_3D = 8, F_GT_DATA = 16,
              F_DT_DATA = 32;

struct Params {
  int N, G, D, C, M, NC;  // frames, gt boxes, dt boxes, classes, metrics, configs
  int classes[3], metrics[3];
  int compute_aos, f32;
  double min_overlap[3][3][2];
  const double* gt;        // [G][GT_W]
  const double* dt;        // [D][DT_W]
  const int* gt_code;      // [G] class id (0 car 1 pedestrian 2 cyclist 3 van 4 person_sitting
                           //  7 other) | CODE_DONTCARE
  const int* dt_code;      // [D] class id
  const int* gt_off;       // [N + 1]
  const int* dt_off;       // [N + 1]
  const long long* pair_off;  // [N + 1] sum of dt * gt counts of the frames before
  long long P;             // pairs of the whole set
  // the current part: frames [f0, f0 + nf), pairs [q0, q0 + nq) of the set
  int f0, nf;
  long long q0, nq;
  long long OP;            // pairs the overlap buffer holds per metric (the largest part)
  // workspace
  signed char* ign_gt;     // [C * 3][G]
  signed char* ign_dt;     // [C * 3][D]
  int* num_valid;          // [C * 3]
  double* ov;              // [M][OP] [dt][gt] within each frame of the current part
  double* tp_scores;       // [NC][G] at each frame's gt offset
  int* tp_count;           // [NC][N]
  double* sorted;          // [NC][S] S = pow2 >= G
  long long S;
  int* sorted_count;       // [NC]
  double* thresholds;      // [NC][MAX_T]
  int* thr_count;          // [NC]  MAX_T + 1 flags more thresholds than the reference holds
  unsigned long long* cnt; // [NC][MAX_T][3] tp fp fn
  double* sim;             // [NC][MAX_T][N]
  double* pr;              // [NC][MAX_T][4] output
  int* status;             // bit 0: a frame holds more than MAX_DT_FRAME detections
};

// ---- explicitly rounded arithmetic, overloaded for the two numba dtypes ----
__device__ __forceinline__ float rmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double rmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float radd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double radd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float rsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double rsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float rdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double rdiv(double a, double b) { return __ddiv_rn(a, b); }
// Python's min / max of two scalars: the first unless the second is strictly smaller / larger
template <class T>
__device__ __forceinline__ T pmin(T a, T b) { return b < a ? b : a; }
template <class T>
__device__ __forceinline__ T pmax(T a, T b) { return b > a ? b : a; }

// ---- rotate_iou.py, op for op ----
__device__ __forceinline__ void rbbox_to_corners(float* c, const float* r) {
  const float a_cos = cosf(r[4]), a_sin = sinf(r[4]);
  const float hx = r[2] / 2.f, hy = r[3] / 2.f;   // exact halving (float64 in numba, same value)
  const float cx[4] = {-hx, -hx, hx, hx};
  const float cy[4] = {-hy, hy, hy, -hy};
  for (int i = 0; i < 4; ++i) {
    c[2 * i] = __fadd_rn(__fadd_rn(__fmul_rn(a_cos, cx[i]), __fmul_rn(a_sin, cy[i])), r[0]);
    c[2 * i + 1] = __fadd_rn(__fadd_rn(__fmul_rn(-a_sin, cx[i]), __fmul_rn(a_cos, cy[i])), r[1]);
  }
}

__device__ __forceinline__ bool point_in_quadrilateral(float px, float py, const float* c) {
  const float ab0 = __fsub_rn(c[2], c[0]), ab1 = __fsub_rn(c[3], c[1]);
  const float ad0 = __fsub_rn(c[6], c[0]), ad1 = __fsub_rn(c[7], c[1]);
  const float ap0 = __fsub_rn(px, c[0]), ap1 = __fsub_rn(py, c[1]);
  const float abab = __fadd_rn(__fmul_rn(ab0, ab0), __fmul_rn(ab1, ab1));
  const float abap = __fadd_rn(__fmul_rn(ab0, ap0), __fmul_rn(ab1, ap1));
  const float adad = __fadd_rn(__fmul_rn(ad0, ad0), __fmul_rn(ad1, ad1));
  const float adap = __fadd_rn(__fmul_rn(ad0, ap0), __fmul_rn(ad1, ap1));
  return abab >= abap && abap >= 0.f && adad >= adap && adap >= 0.f;
}

__device__ __forceinline__ bool line_segment_intersection(const float* p1, const float* p2, int i,
                                                          int j, float* out) {
  const float A0 = p1[2 * i], A1 = p1[2 * i + 1];
  const float B0 = p1[2 * ((i + 1) % 4)], B1 = p1[2 * ((i + 1) % 4) + 1];
  const float C0 = p2[2 * j], C1 = p2[2 * j + 1];
  const float D0 = p2[2 * ((j + 1) % 4)], D1 = p2[2 * ((j + 1) % 4) + 1];
  const float BA0 = __fsub_rn(B0, A0), BA1 = __fsub_rn(B1, A1);
  const float DA0 = __fsub_rn(D0, A0), CA0 = __fsub_rn(C0, A0);
  const float DA1 = __fsub_rn(D1, A1), CA1 = __fsub_rn(C1, A1);
  const bool acd = __fmul_rn(DA1, CA0) > __fmul_rn(CA1, DA0);
  const bool bcd = __fmul_rn(__fsub_rn(D1, B1), __fsub_rn(C0, B0)) >
                   __fmul_rn(__fsub_rn(C1, B1), __fsub_rn(D0, B0));
  if (acd != bcd) {
    const bool abc = __fmul_rn(CA1, BA0) > __fmul_rn(BA1, CA0);
    const bool abd = __fmul_rn(DA1, BA0) > __fmul_rn(BA1, DA0);
    if (abc != abd) {
      const float DC0 = __fsub_rn(D0, C0), DC1 = __fsub_rn(D1, C1);
      const float ABBA = __fsub_rn(__fmul_rn(A0, B1), __fmul_rn(B0, A1));
      const float CDDC = __fsub_rn(__fmul_rn(C0, D1), __fmul_rn(D0, C1));
      const float DH = __fsub_rn(__fmul_rn(BA1, DC0), __fmul_rn(BA0, DC1));
      const float Dx = __fsub_rn(__fmul_rn(ABBA, DC0), __fmul_rn(BA0, CDDC));
      const float Dy = __fsub_rn(__fmul_rn(ABBA, DC1), __fmul_rn(BA1, CDDC));
      out[0] = __fdiv_rn(Dx, DH);
      out[1] = __fdiv_rn(Dy, DH);
      return true;
    }
  }
  return false;
}

// inter(): intersection polygon, centroid-angle insertion sort, triangle-fan area (float64
// accumulation: trangle_area divides its float32 cross product by the float64 literal 2.0).
// The reference's arrays hold 8 points; boxes that coincide or share edges yield up to 8
// corners plus 16 edge crossings, which it writes past their end.  Here there is room for all
// 24, so such pairs get the polygon of every point found.
__device__ __forceinline__ double rotated_inter(const float* r1, const float* r2) {
  float c1[8], c2[8], pts[48];
  rbbox_to_corners(c1, r1);
  rbbox_to_corners(c2, r2);
  int n = 0;
  for (int i = 0; i < 4; ++i) {
    if (point_in_quadrilateral(c1[2 * i], c1[2 * i + 1], c2)) {
      pts[2 * n] = c1[2 * i];
      pts[2 * n + 1] = c1[2 * i + 1];
      ++n;
    }
    if (point_in_quadrilateral(c2[2 * i], c2[2 * i + 1], c1)) {
      pts[2 * n] = c2[2 * i];
      pts[2 * n + 1] = c2[2 * i + 1];
      ++n;
    }
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      float t[2];
      if (line_segment_intersection(c1, c2, i, j, t)) {
        pts[2 * n] = t[0];
        pts[2 * n + 1] = t[1];
        ++n;
      }
    }
  if (n > 0) {
    float cx = 0.f, cy = 0.f;
    for (int i = 0; i < n; ++i) {
      cx = __fadd_rn(cx, pts[2 * i]);
      cy = __fadd_rn(cy, pts[2 * i + 1]);
    }
    cx = (float)__ddiv_rn((double)cx, (double)n);   // float32 / int64 is float64 in numba
    cy = (float)__ddiv_rn((double)cy, (double)n);
    float vs[24];
    for (int i = 0; i < n; ++i) {
      float v0 = __fsub_rn(pts[2 * i], cx), v1 = __fsub_rn(pts[2 * i + 1], cy);
      const float d = __fsqrt_rn(__fadd_rn(__fmul_rn(v0, v0), __fmul_rn(v1, v1)));
      v0 = __fdiv_rn(v0, d);
      v1 = __fdiv_rn(v1, d);
      if (v1 < 0.f) v0 = (float)__dsub_rn(-2.0, (double)v0);
      vs[i] = v0;
    }
    for (int i = 1; i < n; ++i) {
      if (vs[i - 1] > vs[i]) {
        const float temp = vs[i], tx = pts[2 * i], ty = pts[2 * i + 1];
        int j = i;
        while (j > 0 && vs[j - 1] > temp) {
          vs[j] = vs[j - 1];
          pts[2 * j] = pts[2 * j - 2];
          pts[2 * j + 1] = pts[2 * j - 1];
          --j;
        }
        vs[j] = temp;
        pts[2 * j] = tx;
        pts[2 * j + 1] = ty;
      }
    }
  }
  double area = 0.0;
  for (int i = 0; i < n - 2; ++i) {
    const float* a = pts;
    const float* b = pts + 2 * i + 2;
    const float* c = pts + 2 * i + 4;
    const float cr = __fsub_rn(__fmul_rn(__fsub_rn(a[0], c[0]), __fsub_rn(b[1], c[1])),
                               __fmul_rn(__fsub_rn(a[1], c[1]), __fsub_rn(b[0], c[0])));
    area = __dadd_rn(area, fabs(__ddiv_rn((double)cr, 2.0)));
  }
  return area;
}

// devRotateIoUEval(rbox1, rbox2, criterion), rounded to the float32 its output array holds
__device__ __forceinline__ float rotate_iou_eval(const float* r1, const float* r2, int criterion) {
  const float area1 = __fmul_rn(r1[2], r1[3]);
  const float area2 = __fmul_rn(r2[2], r2[3]);
  const double inter = rotated_inter(r1, r2);
  if (criterion == -1) return (float)__ddiv_rn(inter, __dsub_rn((double)__fadd_rn(area1, area2),
                                                                inter));
  if (criterion == 0) return (float)__ddiv_rn(inter, (double)area1);
  if (criterion == 1) return (float)__ddiv_rn(inter, (double)area2);
  return (float)inter;
}

// image_box_overlap(boxes, query_boxes, criterion) for one pair, in the arrays' dtypes; the
// value is what the output array (dtype of boxes) holds
template <class TB, class TQ>
__device__ __forceinline__ double image_overlap(const double* bd, const double* qd, int criterion) {
  typedef decltype(TB() + TQ()) TP;
  const TB b0 = (TB)bd[0], b1 = (TB)bd[1], b2 = (TB)bd[2], b3 = (TB)bd[3];
  const TQ q0 = (TQ)qd[0], q1 = (TQ)qd[1], q2 = (TQ)qd[2], q3 = (TQ)qd[3];
  const TQ qarea = rmul(rsub(q2, q0), rsub(q3, q1));
  const TP iw = rsub(pmin((TP)b2, (TP)q2), pmax((TP)b0, (TP)q0));
  if (!(iw > 0)) return 0.0;
  const TP ih = rsub(pmin((TP)b3, (TP)q3), pmax((TP)b1, (TP)q1));
  if (!(ih > 0)) return 0.0;
  const TB barea = rmul(rsub(b2, b0), rsub(b3, b1));
  TP ua;
  if (criterion == -1)
    ua = rsub((TP)radd((TP)barea, (TP)qarea), rmul(iw, ih));
  else if (criterion == 0)
    ua = (TP)barea;
  else if (criterion == 1)
    ua = (TP)qarea;
  else
    ua = (TP)1;
  return (double)(TB)rdiv(rmul(iw, ih), ua);
}

// d3_box_overlap_kernel for one pair given rinc (the float32 criterion-2 intersection area)
template <class TB, class TQ>
__device__ __forceinline__ double d3_overlap(const double* bd, const double* qd, float rinc) {
  typedef decltype(TB() + TQ()) TP;
  if (!(rinc > 0.f)) return (double)rinc;
  const TB b1 = (TB)bd[1], b3 = (TB)bd[3], b4 = (TB)bd[4], b5 = (TB)bd[5];
  const TQ q1 = (TQ)qd[1], q3 = (TQ)qd[3], q4 = (TQ)qd[4], q5 = (TQ)qd[5];
  const TP iw = rsub(pmin((TP)b1, (TP)q1), pmax((TP)rsub(b1, b4), (TP)rsub(q1, q4)));
  if (!(iw > 0)) return 0.0;
  const TB area1 = rmul(rmul(b3, b4), b5);
  const TQ area2 = rmul(rmul(q3, q4), q5);
  const TP inc = rmul(iw, (TP)rinc);
  const TP ua = rsub((TP)radd((TP)area1, (TP)area2), inc);
  return (double)(float)rdiv(inc, ua);
}

// ---- kernels ----

// clean_data per (class slot, difficulty, frame)
__global__ void ke_ignore_kernel(Params p) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  const int cd = blockIdx.y, cs = cd / 3, diff = cd % 3;
  if (f >= p.N) return;
  const int MIN_HEIGHT[3] = {40, 25, 25};
  const int MAX_OCCLUSION[3] = {0, 1, 2};
  const double MAX_TRUNCATION[3] = {0.15, 0.3, 0.5};
  const int cls = p.classes[cs];
  int valid = 0;
  for (int i = p.gt_off[f]; i < p.gt_off[f + 1]; ++i) {
    const double* g = p.gt + (size_t)i * GT_W;
    const int name = p.gt_code[i] & 7;
    const double height = (p.f32 & F_GT_BBOX) ? (double)__fsub_rn((float)g[3], (float)g[1])
                                               : __dsub_rn(g[3], g[1]);
    int vc = -1;
    if (name == cls) vc = 1;
    else if (cls == 1 && name == 4) vc = 0;
    else if (cls == 0 && name == 3) vc = 0;
    const bool ignore = g[12] > MAX_OCCLUSION[diff] || g[13] > MAX_TRUNCATION[diff] ||
                        height <= MIN_HEIGHT[diff];
    signed char code;
    if (vc == 1 && !ignore) {
      code = 0;
      ++valid;
    } else if (vc == 0 || (ignore && vc == 1)) {
      code = 1;
    } else {
      code = -1;
    }
    p.ign_gt[(size_t)cd * p.G + i] = code;
  }
  for (int j = p.dt_off[f]; j < p.dt_off[f + 1]; ++j) {
    const double* d = p.dt + (size_t)j * DT_W;
    const double height = (p.f32 & F_DT_BBOX) ? (double)fabsf(__fsub_rn((float)d[3], (float)d[1]))
                                               : fabs(__dsub_rn(d[3], d[1]));
    signed char code;
    if (height < MIN_HEIGHT[diff]) code = 1;
    else if (p.dt_code[j] == cls) code = 0;
    else code = -1;
    p.ign_dt[(size_t)cd * p.D + j] = code;
  }
  if (valid) atomicAdd(p.num_valid + cd, valid);
}

__device__ __forceinline__ int frame_of_pair(const long long* off, int N, long long q) {
  int lo = 0, hi = N - 1;   // last frame with off[f] <= q
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= q) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// calculate_iou_partly(dt_annos, gt_annos, metric): ov[ms][pair - q0] for each (dt, gt) of a
// frame of the current part
__global__ void ke_overlap_kernel(Params p) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int ms = blockIdx.y;
  if (q >= p.nq) return;
  const int f = p.f0 + frame_of_pair(p.pair_off + p.f0, p.nf, p.q0 + q);
  const int ng = p.gt_off[f + 1] - p.gt_off[f];
  const long long local = p.q0 + q - p.pair_off[f];
  const int j = p.dt_off[f] + (int)(local / ng), i = p.gt_off[f] + (int)(local % ng);
  const double* g = p.gt + (size_t)i * GT_W;
  const double* d = p.dt + (size_t)j * DT_W;
  const int metric = p.metrics[ms];
  double v;
  if (metric == 0) {
    const bool fb = p.f32 & F_DT_BBOX, fq = p.f32 & F_GT_BBOX;
    v = fb ? (fq ? image_overlap<float, float>(d, g, -1) : image_overlap<float, double>(d, g, -1))
           : (fq ? image_overlap<double, float>(d, g, -1)
                 : image_overlap<double, double>(d, g, -1));
  } else {
    // BEV box = columns [0, 2, 3, 5, 6] of the (loc, dims, ry) box at column 5, as float32
    const float rg[5] = {(float)g[5], (float)g[7], (float)g[8], (float)g[10], (float)g[11]};
    const float rd[5] = {(float)d[5], (float)d[7], (float)d[8], (float)d[10], (float)d[11]};
    if (metric == 1) {
      v = (double)rotate_iou_eval(rg, rd, -1);
    } else {
      const float rinc = rotate_iou_eval(rg, rd, 2);
      const bool fb = p.f32 & F_DT_3D, fq = p.f32 & F_GT_3D;
      v = fb ? (fq ? d3_overlap<float, float>(d + 5, g + 5, rinc)
                   : d3_overlap<float, double>(d + 5, g + 5, rinc))
             : (fq ? d3_overlap<double, float>(d + 5, g + 5, rinc)
                   : d3_overlap<double, double>(d + 5, g + 5, rinc));
    }
  }
  p.ov[(size_t)ms * p.OP + q] = v;
}

__device__ __forceinline__ void config_parts(const Params& p, int cfg, int& ms, int& cd, int& k) {
  k = cfg & 1;
  const int r = cfg >> 1;   // (ms * C + cs) * 3 + diff
  cd = r % (p.C * 3);
  ms = r / (p.C * 3);
}

// compute_statistics_jit for one (config, frame).  compute_fp == false: TP scores only.
// compute_fp == true: counts at `thresh`; returns the frame's similarity term through *sim_out
struct Stats {
  int tp, fp, fn;
  double sim;   // 0 when the reference's similarity is -1 (not added)
};

__device__ Stats frame_statistics(const Params& p, int cfg, int f, bool compute_fp, double thresh,
                                  double* tp_out) {
  int ms, cd, k;
  config_parts(p, cfg, ms, cd, k);
  const int metric = p.metrics[ms];
  const double min_overlap = p.min_overlap[ms][cd / 3][k];
  const bool compute_aos = compute_fp && p.compute_aos && metric == 0;
  const int g0 = p.gt_off[f], ng = p.gt_off[f + 1] - g0;
  const int d0 = p.dt_off[f], nd = p.dt_off[f + 1] - d0;
  if (nd > MAX_DT_FRAME) {   // the bit masks below hold MAX_DT_FRAME detections
    atomicOr(p.status, 1);
    return Stats{0, 0, 0, 0.0};
  }
  const signed char* ig = p.ign_gt + (size_t)cd * p.G + g0;
  const signed char* id = p.ign_dt + (size_t)cd * p.D + d0;
  const double* ov = p.ov + (size_t)ms * p.OP + (p.pair_off[f] - p.q0);
  unsigned assigned[MAX_DT_FRAME / 32];
  unsigned below[MAX_DT_FRAME / 32];
  for (int w = 0; w < (nd + 31) / 32; ++w) {
    assigned[w] = 0;
    below[w] = 0;
  }
  if (compute_fp)
    for (int j = 0; j < nd; ++j)
      if (p.dt[(size_t)(d0 + j) * DT_W + 12] < thresh) below[j >> 5] |= 1u << (j & 31);
  const double NO_DETECTION = -10000000.0;
  Stats s{0, 0, 0, 0.0};
  double sim = 0.0;
  for (int i = 0; i < ng; ++i) {
    if (ig[i] == -1) continue;
    int det_idx = -1;
    double valid_detection = NO_DETECTION, max_overlap = 0.0;
    bool assigned_ignored_det = false;
    for (int j = 0; j < nd; ++j) {
      if (id[j] == -1) continue;
      if ((assigned[j >> 5] >> (j & 31)) & 1) continue;
      if ((below[j >> 5] >> (j & 31)) & 1) continue;
      const double overlap = ov[(size_t)j * ng + i];
      const double dt_score = p.dt[(size_t)(d0 + j) * DT_W + 12];
      if (!compute_fp && overlap > min_overlap && dt_score > valid_detection) {
        det_idx = j;
        valid_detection = dt_score;
      } else if (compute_fp && overlap > min_overlap &&
                 (overlap > max_overlap || assigned_ignored_det) && id[j] == 0) {
        max_overlap = overlap;
        det_idx = j;
        valid_detection = 1;
        assigned_ignored_det = false;
      } else if (compute_fp && overlap > min_overlap && valid_detection == NO_DETECTION &&
                 id[j] == 1) {
        det_idx = j;
        valid_detection = 1;
        assigned_ignored_det = true;
      }
    }
    if (valid_detection == NO_DETECTION && ig[i] == 0) {
      ++s.fn;
    } else if (valid_detection != NO_DETECTION && (ig[i] == 1 || id[det_idx] == 1)) {
      assigned[det_idx >> 5] |= 1u << (det_idx & 31);
    } else if (valid_detection != NO_DETECTION) {
      if (tp_out) tp_out[s.tp] = p.dt[(size_t)(d0 + det_idx) * DT_W + 12];
      ++s.tp;
      if (compute_aos) {
        const double ga = p.gt[(size_t)(g0 + i) * GT_W + 4];
        const double da = p.dt[(size_t)(d0 + det_idx) * DT_W + 4];
        const double delta = ((p.f32 & F_GT_DATA) && (p.f32 & F_DT_DATA))
                                 ? (double)__fsub_rn((float)ga, (float)da)
                                 : __dsub_rn(ga, da);
        sim = __dadd_rn(sim, __ddiv_rn(__dadd_rn(1.0, cos(delta)), 2.0));
      }
      assigned[det_idx >> 5] |= 1u << (det_idx & 31);
    }
  }
  if (compute_fp) {
    for (int j = 0; j < nd; ++j)
      if (!(((assigned[j >> 5] >> (j & 31)) & 1) || id[j] == -1 || id[j] == 1 ||
            ((below[j >> 5] >> (j & 31)) & 1)))
        ++s.fp;
    int nstuff = 0;
    if (metric == 0) {
      // DontCare boxes of the frame in GT order; dt_datas holds bbox, alpha and score
      const bool fb = p.f32 & F_DT_DATA;
      for (int i = 0; i < ng; ++i) {
        if (!(p.gt_code[g0 + i] & CODE_DONTCARE)) continue;
        const double* dc = p.gt + (size_t)(g0 + i) * GT_W;
        for (int j = 0; j < nd; ++j) {
          if ((assigned[j >> 5] >> (j & 31)) & 1) continue;
          if (id[j] == -1 || id[j] == 1) continue;
          if ((below[j >> 5] >> (j & 31)) & 1) continue;
          const double* db = p.dt + (size_t)(d0 + j) * DT_W;
          const double o = fb ? image_overlap<float, double>(db, dc, 0)
                              : image_overlap<double, double>(db, dc, 0);
          if (o > min_overlap) {
            assigned[j >> 5] |= 1u << (j & 31);
            ++nstuff;
          }
        }
      }
    }
    s.fp -= nstuff;
    if (compute_aos && (s.tp > 0 || s.fp > 0)) s.sim = sim;
  }
  return s;
}

// pass 1: grid (frames of the part, configs)
__global__ void ke_pass1_kernel(Params p) {
  const int fl = blockIdx.x * blockDim.x + threadIdx.x, cfg = blockIdx.y;
  if (fl >= p.nf) return;
  const int f = p.f0 + fl;
  const Stats s = frame_statistics(p, cfg, f, false, 0.0,
                                   p.tp_scores + (size_t)cfg * p.G + p.gt_off[f]);
  p.tp_count[(size_t)cfg * p.N + f] = s.tp;
}

// get_thresholds per config: gather the TP scores in frame order, sort them descending
// (bitonic, in this config's slice of `sorted`), then make the sequential 41-point pick
__global__ void __launch_bounds__(1024) ke_thresholds_kernel(Params p) {
  const int cfg = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  __shared__ int chunk_off[1025];
  const int* cnt = p.tp_count + (size_t)cfg * p.N;
  const int per = (p.N + nt - 1) / nt;
  const int f0 = min(p.N, tid * per), f1 = min(p.N, f0 + per);
  int mine = 0;
  for (int f = f0; f < f1; ++f) mine += cnt[f];
  chunk_off[tid + 1] = mine;
  __syncthreads();
  if (tid == 0) {
    chunk_off[0] = 0;
    for (int t = 1; t <= nt; ++t) chunk_off[t] += chunk_off[t - 1];
  }
  __syncthreads();
  const int L = chunk_off[nt];
  double* s = p.sorted + (size_t)cfg * p.S;
  int o = chunk_off[tid];
  for (int f = f0; f < f1; ++f) {
    const double* src = p.tp_scores + (size_t)cfg * p.G + p.gt_off[f];
    for (int t = 0; t < cnt[f]; ++t) s[o++] = src[t];
  }
  int n2 = 1;
  while (n2 < L) n2 <<= 1;
  for (int i = L + tid; i < n2; i += nt) s[i] = -INFINITY;
  __syncthreads();
  for (int k = 2; k <= n2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < n2; i += nt) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const double a = s[i], b = s[ixj];
          const bool desc = (i & k) == 0;
          if (desc ? a < b : a > b) {
            s[i] = b;
            s[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  if (tid != 0) return;
  int ms, cd, k;
  config_parts(p, cfg, ms, cd, k);
  const double num_gt = (double)p.num_valid[cd];
  double current_recall = 0.0;
  int count = 0;
  for (int i = 0; i < L; ++i) {
    const double l_recall = __ddiv_rn((double)(i + 1), num_gt);
    const double r_recall = i < L - 1 ? __ddiv_rn((double)(i + 2), num_gt) : l_recall;
    if (__dsub_rn(r_recall, current_recall) < __dsub_rn(current_recall, l_recall) && i < L - 1)
      continue;
    if (count < MAX_T) p.thresholds[(size_t)cfg * MAX_T + count] = s[i];
    ++count;
    current_recall = __dadd_rn(current_recall, 1.0 / 40.0);
  }
  p.sorted_count[cfg] = L;
  p.thr_count[cfg] = min(count, MAX_T + 1);
}

// pass 2: grid (frames of the part, thresholds, configs)
__global__ void ke_pass2_kernel(Params p) {
  const int fl = blockIdx.x * blockDim.x + threadIdx.x, t = blockIdx.y, cfg = blockIdx.z;
  if (fl >= p.nf || t >= min(p.thr_count[cfg], MAX_T)) return;
  const int f = p.f0 + fl;
  const Stats s = frame_statistics(p, cfg, f, true, p.thresholds[(size_t)cfg * MAX_T + t],
                                   nullptr);
  unsigned long long* c = p.cnt + ((size_t)cfg * MAX_T + t) * 3;
  if (s.tp) atomicAdd(c, (unsigned long long)s.tp);
  if (s.fp) atomicAdd(c + 1, (unsigned long long)s.fp);
  if (s.fn) atomicAdd(c + 2, (unsigned long long)s.fn);
  p.sim[((size_t)cfg * MAX_T + t) * p.N + f] = s.sim;
}

// pr[cfg][t] = (tp, fp, fn, similarity summed over frames in order); zero past the count
__global__ void ke_reduce_kernel(Params p) {
  const int t = threadIdx.x, cfg = blockIdx.x;
  if (t >= MAX_T) return;
  double* o = p.pr + ((size_t)cfg * MAX_T + t) * 4;
  if (t >= min(p.thr_count[cfg], MAX_T)) {
    o[0] = o[1] = o[2] = o[3] = 0.0;
    return;
  }
  const unsigned long long* c = p.cnt + ((size_t)cfg * MAX_T + t) * 3;
  const double* sim = p.sim + ((size_t)cfg * MAX_T + t) * p.N;
  double acc = 0.0;
  for (int f = 0; f < p.N; ++f) acc = __dadd_rn(acc, sim[f]);
  o[0] = (double)c[0];
  o[1] = (double)(long long)c[1];
  o[2] = (double)c[2];
  o[3] = acc;
}

// dfm_op_eval_rotated_iou: iou[n][k] = devRotateIoUEval(qboxes[k], boxes[n], criterion)
__global__ void ke_rotate_iou_kernel(const float* boxes, const float* qboxes, int N, int K,
                                     int criterion, float* iou) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= (long long)N * K) return;
  const int n = (int)(q / K), k = (int)(q % K);
  iou[q] = rotate_iou_eval(qboxes + (size_t)k * 5, boxes + (size_t)n * 5, criterion);
}

}  // namespace ke
}  // namespace dfm
