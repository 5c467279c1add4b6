// Anchor-head post-processing (Anchor3DHead.get_bboxes_single, anchor3d_head.py:459-547, with
// box3d_multiclass_nms / nms_bev, box3d_nms.py:8-128, 231-268) for a batch of B samples:
//
//   score + key -> radix select of the top nms_pre keys -> block sort       (only if N > nms_pre)
//   decode + round-tripped BEV box + per-class candidate lists -> per-class block sort
//   -> 64 x 64 rotated-IoU tiles (one u64 row mask per box) -> greedy sweep per (sample, class)
//   -> merge (class-major concat, or score sort + cut at max_num) + yaw fix
//
// No host synchronisation: every count stays on the device, grids are sized for the worst case
// and CTAs past a count return.  Arithmetic that decides a bit of the result is written with
// explicitly rounded intrinsics so nvcc cannot contract it into an FMA the reference's
// one-op-at-a-time PyTorch does not perform.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace dfm {

constexpr int BP_MAX_CAND = 4096;   // candidates per (sample, class): row masks of <= 64 words
constexpr int BP_MAX_CLASSES = 16;  // score columns kept in registers per anchor
constexpr int BP_TILE = 64;         // IoU tile edge = bits per mask word
// Corner convention of mmcv's nms_rotated (box_iou_rotated_utils.hpp, mmcv-full 1.6.0, its
// clockwise=True default): corners sit at centre + R(BP_ROT_SIGN * theta) * (+-w/2, +-h/2).
// LiDARInstance3DBoxes.corners rotates by +theta; the IoU NMS uses is that of the mirrored pair.
constexpr float BP_ROT_SIGN = -1.f;

typedef unsigned long long u64;

struct BoxPostParams {
  const float* cls;      // [B][A * ncol][HW]
  const float* reg;      // [B][A * 7][HW]
  const float* dir;      // [B][A * 2][HW]
  const float* anchors;  // [N][7]
  int B, HW, A, C, ncol, sigmoid;
  int N, K, W;           // anchors, selected anchors per sample, mask words per row
  int topk;              // N > nms_pre > 0
  int max_num;
  float score_thr, nms_thr, dir_offset, dir_limit_offset;
  // workspace
  u64* keys;             // [B][N]       top-k keys
  unsigned* hist;        // [B][256]     radix histogram
  u64* prefix;           // [B]          radix prefix
  int* kleft;            // [B]          keys still to take below the prefix
  int* sel_count;        // [B]
  u64* sel;              // [B][K]       selected keys, unordered
  int* topk_index;       // [B][K]       selected anchors, (score desc, anchor asc)
  float* boxes;          // [B][K][7]    decoded boxes
  float* bev;            // [B][K][5]    round-tripped NMS boxes (x, y, w, h, r)
  int* dirlab;           // [B][K]
  int* cand_count;       // [B][C]
  u64* cand_key;         // [B][C][K]    (score bits << 32) | ~anchor, sorted in place
  int* cand_slot;        // [B][C][K]    slot (index into the K selected anchors)
  float* cand_bev;       // [B][C][K][5] NMS boxes in sorted order
  u64* mask;             // [B][C][K][W] suppression row masks (upper triangle)
  int* keep_count;       // [B][C]
  int* keep_rank;        // [B][C][K]    kept candidates, as ranks in the sorted class list
  // outputs
  float* out_boxes;      // [B][max_num][7]
  float* out_scores;     // [B][max_num]
  int* out_labels;       // [B][max_num]
  int* out_count;        // [B]
};

__device__ __forceinline__ u64 bp_key(float score, int anchor) {
  return ((u64)__float_as_uint(score) << 32) | (u64)(0xFFFFFFFFu - (unsigned)anchor);
}
__device__ __forceinline__ int bp_key_anchor(u64 k) {
  return (int)(0xFFFFFFFFu - (unsigned)(k & 0xFFFFFFFFull));
}

// Class scores of anchor j of a cell: sigmoid 1 / (1 + exp(-x)) as torch's CUDA sigmoid computes
// it, or softmax over ncol = C + 1 columns (the last, background, is not returned).
__device__ __forceinline__ void bp_class_scores(const BoxPostParams& p, int b, int cell, int j,
                                                float (&s)[BP_MAX_CLASSES]) {
  const float* x = p.cls + ((size_t)b * p.A * p.ncol + (size_t)j * p.ncol) * p.HW + cell;
  if (p.sigmoid) {
#pragma unroll
    for (int c = 0; c < BP_MAX_CLASSES; ++c)
      s[c] = c < p.C ? 1.f / (1.f + expf(-__ldg(x + (size_t)c * p.HW))) : 0.f;
    return;
  }
  float m = -INFINITY;
  for (int c = 0; c < p.ncol; ++c) m = fmaxf(m, __ldg(x + (size_t)c * p.HW));
  float sum = 0.f;
  for (int c = 0; c < p.ncol; ++c) sum = __fadd_rn(sum, expf(__fsub_rn(__ldg(x + (size_t)c * p.HW), m)));
#pragma unroll
  for (int c = 0; c < BP_MAX_CLASSES; ++c)
    s[c] = c < p.C ? __fdiv_rn(expf(__fsub_rn(__ldg(x + (size_t)c * p.HW), m)), sum) : 0.f;
}

// ---- top-k: 64-bit keys, 8 radix passes of 8 bits from the top, then a gather ----

__global__ void bp_score_key_kernel(BoxPostParams p) {
  const int b = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.N) return;
  float s[BP_MAX_CLASSES];
  bp_class_scores(p, b, i / p.A, i % p.A, s);
  float best = s[0];
#pragma unroll
  for (int c = 1; c < BP_MAX_CLASSES; ++c)
    if (c < p.C && s[c] > best) best = s[c];
  p.keys[(size_t)b * p.N + i] = bp_key(best, i);
}

__global__ void bp_radix_hist_kernel(BoxPostParams p, int shift) {
  __shared__ unsigned h[256];
  const int b = blockIdx.y;
  for (int t = threadIdx.x; t < 256; t += blockDim.x) h[t] = 0;
  __syncthreads();
  const u64 hi = shift >= 56 ? 0ull : (~0ull << (shift + 8));
  const u64 pre = p.prefix[b] & hi;
  const u64* keys = p.keys + (size_t)b * p.N;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < p.N; i += gridDim.x * blockDim.x) {
    const u64 k = keys[i];
    if ((k & hi) == pre) atomicAdd(&h[(unsigned)(k >> shift) & 255u], 1u);
  }
  __syncthreads();
  for (int t = threadIdx.x; t < 256; t += blockDim.x)
    if (h[t]) atomicAdd(&p.hist[b * 256 + t], h[t]);
}

// <<<B, 256>>>: picks the digit holding the kleft-th largest key and clears the histogram
__global__ void bp_radix_select_kernel(BoxPostParams p, int shift, int first) {
  __shared__ unsigned h[256];
  const int b = blockIdx.x, t = threadIdx.x;
  h[t] = p.hist[b * 256 + t];
  p.hist[b * 256 + t] = 0;
  const int k = first ? p.K : p.kleft[b];
  __syncthreads();
  unsigned above = 0;
  for (int d = t + 1; d < 256; ++d) above += h[d];
  __syncthreads();
  if (above < (unsigned)k && above + h[t] >= (unsigned)k) {
    p.kleft[b] = k - (int)above;
    p.prefix[b] = (first ? 0ull : p.prefix[b]) | ((u64)t << shift);
  }
}

__global__ void bp_gather_kernel(BoxPostParams p) {
  const int b = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.N) return;
  const u64 k = p.keys[(size_t)b * p.N + i];
  if (k >= p.prefix[b]) {
    const int pos = atomicAdd(&p.sel_count[b], 1);
    if (pos < p.K) p.sel[(size_t)b * p.K + pos] = k;
  }
}

// Descending bitonic sort of P (a power of two) keys in shared memory, optional 16-bit payload.
__device__ void bp_bitonic_desc(u64* key, unsigned short* val, int P) {
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const int o = i ^ j;
        if (o > i) {
          const u64 a = key[i], c = key[o];
          if (((i & k) == 0) ? (a < c) : (a > c)) {
            key[i] = c;
            key[o] = a;
            if (val) {
              const unsigned short v = val[i];
              val[i] = val[o];
              val[o] = v;
            }
          }
        }
      }
      __syncthreads();
    }
}

__device__ __forceinline__ int bp_pow2(int n) {
  int P = 1;
  while (P < n) P <<= 1;
  return P;
}

// <<<B, 1024>>>: orders the K selected keys (score desc, anchor asc) into topk_index
__global__ void __launch_bounds__(1024) bp_topk_sort_kernel(BoxPostParams p) {
  __shared__ u64 key[BP_MAX_CAND];
  const int b = blockIdx.x;
  const int P = bp_pow2(p.K);
  for (int i = threadIdx.x; i < P; i += blockDim.x)
    key[i] = i < p.K ? p.sel[(size_t)b * p.K + i] : 0ull;
  __syncthreads();
  bp_bitonic_desc(key, nullptr, P);
  for (int i = threadIdx.x; i < p.K; i += blockDim.x)
    p.topk_index[(size_t)b * p.K + i] = bp_key_anchor(key[i]);
}

// ---- decode (DeltaXYZWLHRBBoxCoder.decode, op for op) and per-class candidate lists ----

// box = decode(an, t): both [7] (x, y, z, w, l, h, yaw), z at the bottom centre
__device__ __forceinline__ void bp_decode_box(const float* t, const float* an, float* box) {
  const float xa = an[0], ya = an[1], wa = an[3], la = an[4], ha = an[5], ra = an[6];
  const float za = __fadd_rn(an[2], __fdiv_rn(ha, 2.f));
  const float diag = __fsqrt_rn(__fadd_rn(__fmul_rn(la, la), __fmul_rn(wa, wa)));
  box[0] = __fadd_rn(__fmul_rn(t[0], diag), xa);
  box[1] = __fadd_rn(__fmul_rn(t[1], diag), ya);
  const float zg = __fadd_rn(__fmul_rn(t[2], ha), za);
  box[4] = __fmul_rn(expf(t[4]), la);
  box[3] = __fmul_rn(expf(t[3]), wa);
  box[5] = __fmul_rn(expf(t[5]), ha);
  box[6] = __fadd_rn(t[6], ra);
  box[2] = __fsub_rn(zg, __fdiv_rn(box[5], 2.f));
}

__global__ void bp_decode_kernel(BoxPostParams p) {
  const int b = blockIdx.y;
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= p.K) return;
  const int a = p.topk ? p.topk_index[(size_t)b * p.K + slot] : slot;
  const int cell = a / p.A, j = a % p.A;
  float s[BP_MAX_CLASSES];
  bp_class_scores(p, b, cell, j, s);
  const float* dr = p.dir + ((size_t)b * p.A * 2 + (size_t)j * 2) * p.HW + cell;
  const int dl = __ldg(dr + p.HW) > __ldg(dr) ? 1 : 0;  // argmax, first index on a tie
  const float* rg = p.reg + ((size_t)b * p.A * 7 + (size_t)j * 7) * p.HW + cell;
  float t[7], an[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    t[k] = __ldg(rg + (size_t)k * p.HW);
    an[k] = __ldg(p.anchors + (size_t)a * 7 + k);
  }
  float* box = p.boxes + ((size_t)b * p.K + slot) * 7;
  bp_decode_box(t, an, box);
  const float xg = box[0], yg = box[1], wg = box[3], lg = box[4], rgo = box[6];
  p.dirlab[(size_t)b * p.K + slot] = dl;
  // bev = [x, y, dx, dy, yaw]; xywhr2xyxyr, then nms_bev's way back to xywhr
  const float hw = __fdiv_rn(wg, 2.f), hh = __fdiv_rn(lg, 2.f);
  const float x1 = __fsub_rn(xg, hw), y1 = __fsub_rn(yg, hh);
  const float x2 = __fadd_rn(xg, hw), y2 = __fadd_rn(yg, hh);
  float* bv = p.bev + ((size_t)b * p.K + slot) * 5;
  bv[0] = __fdiv_rn(__fadd_rn(x1, x2), 2.f);
  bv[1] = __fdiv_rn(__fadd_rn(y1, y2), 2.f);
  bv[2] = __fsub_rn(x2, x1);
  bv[3] = __fsub_rn(y2, y1);
  bv[4] = rgo;
#pragma unroll
  for (int c = 0; c < BP_MAX_CLASSES; ++c) {
    if (c < p.C && s[c] > p.score_thr) {
      const size_t bc = (size_t)b * p.C + c;
      const int pos = atomicAdd(&p.cand_count[bc], 1);
      p.cand_key[bc * p.K + pos] = bp_key(s[c], a);
      p.cand_slot[bc * p.K + pos] = slot;
    }
  }
}

// <<<B * C, 1024>>>: sorts a class's candidates (score desc, anchor asc) and lays out their boxes
__global__ void __launch_bounds__(1024) bp_class_sort_kernel(BoxPostParams p) {
  __shared__ u64 key[BP_MAX_CAND];
  __shared__ unsigned short slot[BP_MAX_CAND];
  const int bc = blockIdx.x, b = bc / p.C;
  const int n = p.cand_count[bc];
  if (n == 0) return;
  const int P = bp_pow2(n);
  u64* gk = p.cand_key + (size_t)bc * p.K;
  int* gs = p.cand_slot + (size_t)bc * p.K;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    key[i] = i < n ? gk[i] : 0ull;
    slot[i] = i < n ? (unsigned short)gs[i] : 0;
  }
  __syncthreads();
  bp_bitonic_desc(key, slot, P);
  float* cb = p.cand_bev + (size_t)bc * p.K * 5;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    gk[i] = key[i];
    gs[i] = slot[i];
    const float* src = p.bev + ((size_t)b * p.K + slot[i]) * 5;
#pragma unroll
    for (int k = 0; k < 5; ++k) cb[(size_t)i * 5 + k] = src[k];
  }
}

// ---- rotated IoU (fp32, pair-centred) ----

struct BpRect {
  float x, y, area, radius;
  float ox[4], oy[4];  // corner offsets from the centre, counter-clockwise
};

__device__ __forceinline__ BpRect bp_rect(const float* bv) {
  BpRect r;
  r.x = bv[0];
  r.y = bv[1];
  const float w = bv[2], h = bv[3];
  r.area = __fmul_rn(w, h);
  r.radius = 0.5f * sqrtf(w * w + h * h);
  float sn, cs;
  sincosf(bv[4], &sn, &cs);
  sn *= BP_ROT_SIGN;
  const float us[4] = {0.5f, -0.5f, -0.5f, 0.5f}, vs[4] = {0.5f, 0.5f, -0.5f, -0.5f};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float u = us[k] * w, v = vs[k] * h;
    r.ox[k] = __fsub_rn(__fmul_rn(cs, u), __fmul_rn(sn, v));
    r.oy[k] = __fadd_rn(__fmul_rn(sn, u), __fmul_rn(cs, v));
  }
  return r;
}

__device__ __forceinline__ float bp_cross(float ax, float ay, float bx, float by) {
  return __fsub_rn(__fmul_rn(ax, by), __fmul_rn(ay, bx));
}

// Vertex slots of the intersection polygon.  Clipping an n-gon by one half-plane keeps its i
// inside vertices and adds one per sign change of the side values, of which there are at most
// 2 min(i, n - i): at most floor(3 n / 2) vertices whatever the rounding.  From the 4 corners
// that is 6, 9, 13, then 19 after the fourth line, so no vertex is ever dropped (exactly, a
// convex quadrilateral needs at most 8; rounding adds vertices where several lie within
// rounding of one clip line, as on near-duplicate boxes).  The polygon lives in local memory.
constexpr int BP_POLY = 19;

// One Sutherland-Hodgman step: the polygon (x, y)[0..n) clipped to the closed half-plane left of
// the line through (qx, qy) along (ex, ey).  Each vertex's side is computed once and an edge
// that crosses the line gives one point at t = s0 / (s0 - s1), which lies in [0, 1] however
// the side values round, so the clipped area is continuous in the corners: an edge of P lying
// on one of Q's edge lines is kept or cut by its two end vertices alone, never counted twice.
__device__ __forceinline__ int bp_clip(const float* x, const float* y, int n, float qx, float qy,
                                       float ex, float ey, float* ox, float* oy) {
  if (n == 0) return 0;
  const float sf = bp_cross(ex, ey, __fsub_rn(x[0], qx), __fsub_rn(y[0], qy));
  float s0 = sf;
  int m = 0;
  for (int i = 0; i < n; ++i) {
    const int k = i + 1 == n ? 0 : i + 1;
    const float s1 = k == 0 ? sf : bp_cross(ex, ey, __fsub_rn(x[k], qx), __fsub_rn(y[k], qy));
    const bool in0 = s0 >= 0.f, in1 = s1 >= 0.f;
    if (in0) {
      ox[m] = x[i];
      oy[m] = y[i];
      ++m;
    }
    if (in0 != in1) {
      const float t = __fdiv_rn(s0, __fsub_rn(s0, s1));
      ox[m] = __fadd_rn(x[i], __fmul_rn(t, __fsub_rn(x[k], x[i])));
      oy[m] = __fadd_rn(y[i], __fmul_rn(t, __fsub_rn(y[k], y[i])));
      ++m;
    }
    s0 = s1;
  }
  return m;
}

__device__ __forceinline__ float bp_iou(const BpRect& a, const BpRect& b) {
  const float dx = b.x - a.x, dy = b.y - a.y, rr = a.radius + b.radius;
  if (dx * dx + dy * dy > rr * rr * 1.0001f + 1e-6f) return 0.f;  // bounding circles apart
  const float cx = __fmul_rn(__fadd_rn(a.x, b.x), 0.5f), cy = __fmul_rn(__fadd_rn(a.y, b.y), 0.5f);
  const float ax = __fsub_rn(a.x, cx), ay = __fsub_rn(a.y, cy);
  const float bx = __fsub_rn(b.x, cx), by = __fsub_rn(b.y, cy);
  float px[BP_POLY], py[BP_POLY], tx[BP_POLY], ty[BP_POLY], qx[4], qy[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    px[k] = __fadd_rn(ax, a.ox[k]);
    py[k] = __fadd_rn(ay, a.oy[k]);
    qx[k] = __fadd_rn(bx, b.ox[k]);
    qy[k] = __fadd_rn(by, b.oy[k]);
  }
  // P (box a) clipped by Q's four edge lines in turn, ping-ponging between p and t
  int n = 4;
#pragma unroll
  for (int k = 0; k < 4; k += 2) {
    const float ex0 = __fsub_rn(qx[k + 1], qx[k]), ey0 = __fsub_rn(qy[k + 1], qy[k]);
    const float ex1 = __fsub_rn(qx[(k + 2) & 3], qx[k + 1]);
    const float ey1 = __fsub_rn(qy[(k + 2) & 3], qy[k + 1]);
    n = bp_clip(px, py, n, qx[k], qy[k], ex0, ey0, tx, ty);
    n = bp_clip(tx, ty, n, qx[k + 1], qy[k + 1], ex1, ey1, px, py);
  }
  // shoelace as a fan from vertex 0 (short difference vectors for a small polygon)
  float a2 = 0.f;
  for (int i = 1; i + 1 < n; ++i)
    a2 = __fadd_rn(a2, bp_cross(__fsub_rn(px[i], px[0]), __fsub_rn(py[i], py[0]),
                                __fsub_rn(px[i + 1], px[0]), __fsub_rn(py[i + 1], py[0])));
  float inter = 0.5f * a2;
  inter = fminf(fmaxf(inter, 0.f), fminf(a.area, b.area));
  const float uni = a.area + b.area - inter;
  return uni > 0.f ? inter / uni : 0.f;
}

// grid (W * (W + 1) / 2, B * C), 64 threads: tile (row block rb, column block cb >= rb)
__global__ void __launch_bounds__(BP_TILE) bp_iou_mask_kernel(BoxPostParams p) {
  __shared__ BpRect col[BP_TILE];
  const int bc = blockIdx.y;
  const int n = p.cand_count[bc];
  int rb = 0, rem = blockIdx.x;
  while (rem >= p.W - rb) {
    rem -= p.W - rb;
    ++rb;
  }
  const int cb = rb + rem;
  if (cb * BP_TILE >= n) return;
  const float* cand = p.cand_bev + (size_t)bc * p.K * 5;
  const int t = threadIdx.x;
  if (cb * BP_TILE + t < n) col[t] = bp_rect(cand + (size_t)(cb * BP_TILE + t) * 5);
  __syncthreads();
  const int i = rb * BP_TILE + t;
  if (i >= n) return;
  const BpRect r = bp_rect(cand + (size_t)i * 5);
  const int jn = min(BP_TILE, n - cb * BP_TILE);
  u64 bits = 0;
  for (int jj = rb == cb ? t + 1 : 0; jj < jn; ++jj)
    if (bp_iou(r, col[jj]) > p.nms_thr) bits |= 1ull << jj;
  p.mask[((size_t)bc * p.K + i) * p.W + cb] = bits;
}

// <<<B * C, 512>>>: greedy sweep in score order; `removed` lives in shared memory.  Per block of
// 64 rows one thread resolves the diagonal word, then 8 x 64 threads OR the kept rows' masks.
__global__ void __launch_bounds__(512) bp_nms_reduce_kernel(BoxPostParams p) {
  __shared__ u64 removed[BP_TILE], diag[BP_TILE], part[8][BP_TILE];
  __shared__ u64 kept_s;
  const int bc = blockIdx.x, tid = threadIdx.x;
  const int n = p.cand_count[bc];
  const int nblk = (n + BP_TILE - 1) / BP_TILE;
  const u64* mask = p.mask + (size_t)bc * p.K * p.W;
  int* keep = p.keep_rank + (size_t)bc * p.K;
  if (tid < BP_TILE) removed[tid] = 0ull;
  int nkeep = 0;
  __syncthreads();
  for (int rb = 0; rb < nblk; ++rb) {
    const int rows = min(BP_TILE, n - rb * BP_TILE);
    if (tid < rows) diag[tid] = mask[(size_t)(rb * BP_TILE + tid) * p.W + rb];
    __syncthreads();
    if (tid == 0) {
      u64 cur = removed[rb], kept = 0ull;
      for (int t = 0; t < rows; ++t)
        if (!((cur >> t) & 1ull)) {
          kept |= 1ull << t;
          cur |= diag[t];
        }
      kept_s = kept;
    }
    __syncthreads();
    const u64 kept = kept_s;
    if (tid < rows && ((kept >> tid) & 1ull))
      keep[nkeep + __popcll(kept & ((1ull << tid) - 1ull))] = rb * BP_TILE + tid;
    nkeep += __popcll(kept);
    const int w = tid & (BP_TILE - 1), g = tid >> 6;
    u64 acc = 0ull;
    if (w > rb && w < nblk)
      for (int t = g; t < rows; t += 8)
        if ((kept >> t) & 1ull) acc |= mask[(size_t)(rb * BP_TILE + t) * p.W + w];
    part[g][w] = acc;
    __syncthreads();
    if (tid < BP_TILE && tid > rb && tid < nblk) {
      u64 o = removed[tid];
#pragma unroll
      for (int q = 0; q < 8; ++q) o |= part[q][tid];
      removed[tid] = o;
    }
    __syncthreads();
  }
  if (tid == 0) p.keep_count[bc] = nkeep;
}

// score bits of the r-th kept box of (sample, class) bc
__device__ __forceinline__ unsigned bp_kept_score(const BoxPostParams& p, int bc, int r) {
  const int i = p.keep_rank[(size_t)bc * p.K + r];
  return (unsigned)(p.cand_key[(size_t)bc * p.K + i] >> 32);
}

// number of kept boxes of bc ordered before score s: score > s, or >= s when `ties_first`
__device__ __forceinline__ int bp_count_before(const BoxPostParams& p, int bc, int n, unsigned s,
                                               bool ties_first) {
  int lo = 0, hi = n;  // kept scores are non-increasing
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const unsigned v = bp_kept_score(p, bc, mid);
    if (v > s || (ties_first && v == s)) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// <<<B, 1024>>>: class-major concatenation, or (total > max_num) the first max_num in (score desc,
// class asc, rank asc) order; yaw = limit_period(yaw - off, limit_off, pi) + off + pi * dir_label
__global__ void __launch_bounds__(1024) bp_merge_kernel(BoxPostParams p) {
  __shared__ int cnt[BP_MAX_CLASSES], off[BP_MAX_CLASSES + 1];
  const int b = blockIdx.x;
  if (threadIdx.x < p.C) cnt[threadIdx.x] = p.keep_count[b * p.C + threadIdx.x];
  __syncthreads();
  if (threadIdx.x == 0) {
    off[0] = 0;
    for (int c = 0; c < p.C; ++c) off[c + 1] = off[c] + cnt[c];
    p.out_count[b] = min(off[p.C], p.max_num);
  }
  __syncthreads();
  const int total = off[p.C];
  const float pi = 3.14159265358979323846f;
  for (int c = 0; c < p.C; ++c) {
    const int bc = b * p.C + c;
    for (int r = threadIdx.x; r < cnt[c]; r += blockDim.x) {
      const int i = p.keep_rank[(size_t)bc * p.K + r];
      const u64 key = p.cand_key[(size_t)bc * p.K + i];
      const unsigned sb = (unsigned)(key >> 32);
      int pos = off[c] + r;
      if (total > p.max_num) {
        pos = r;
        for (int c2 = 0; c2 < p.C; ++c2)
          if (c2 != c) pos += bp_count_before(p, b * p.C + c2, cnt[c2], sb, c2 < c);
      }
      if (pos >= p.max_num) continue;
      const int slot = p.cand_slot[(size_t)bc * p.K + i];
      const float* src = p.boxes + ((size_t)b * p.K + slot) * 7;
      float* dst = p.out_boxes + ((size_t)b * p.max_num + pos) * 7;
#pragma unroll
      for (int k = 0; k < 6; ++k) dst[k] = src[k];
      const float val = __fsub_rn(src[6], p.dir_offset);
      const float fl = floorf(__fadd_rn(__fdiv_rn(val, pi), p.dir_limit_offset));
      const float rot = __fsub_rn(val, __fmul_rn(fl, pi));
      const float dl = (float)p.dirlab[(size_t)b * p.K + slot];
      dst[6] = __fadd_rn(__fadd_rn(rot, p.dir_offset), __fmul_rn(pi, dl));
      p.out_scores[(size_t)b * p.max_num + pos] = __uint_as_float(sb);
      p.out_labels[(size_t)b * p.max_num + pos] = c;
    }
  }
}

}  // namespace dfm
