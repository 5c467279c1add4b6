// Shared device/host definitions for the DfM library.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <string>

namespace dfm {

// Scratch / caches that outlive a call are kept per CUDA device (one process may drive
// several GPUs; the library as a whole is still not re-entrant, see include/dfm_b200.h).
constexpr int kMaxDevices = 64;
inline int cur_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev >= 0 && dev < kMaxDevices ? dev : 0;
}
// The slots are never destroyed: freeing device memory during static destruction could run
// after the CUDA runtime has torn down its context.
template <class T, int TAG = 0>
inline T& per_device() {
  static T* slots = new T[kMaxDevices]();  // value-initialised, as a static array would be
  return slots[cur_device()];
}

// Sole owner of one device allocation of n elements: move-only, freed by the destructor.
// alloc is grow-only: it keeps the allocation when that already holds `count` elements.
template <class T>
struct DevArray {
  T* p = nullptr;
  size_t n = 0;

  DevArray() = default;
  DevArray(const DevArray&) = delete;
  DevArray& operator=(const DevArray&) = delete;
  DevArray(DevArray&& o) noexcept : p(o.p), n(o.n) {
    o.p = nullptr;
    o.n = 0;
  }
  DevArray& operator=(DevArray&& o) noexcept {
    if (this != &o) {
      release();
      p = o.p;
      n = o.n;
      o.p = nullptr;
      o.n = 0;
    }
    return *this;
  }
  ~DevArray() { release(); }

  cudaError_t alloc(size_t count) {
    if (p && n >= count) return cudaSuccess;
    release();
    const cudaError_t e = cudaMalloc(&p, count * sizeof(T));
    if (e != cudaSuccess) {
      p = nullptr;
      return e;
    }
    n = count;
    return cudaSuccess;
  }
  // alloc + a synchronous copy of `count` host elements
  cudaError_t upload(const T* h, size_t count) {
    cudaError_t e = alloc(count);
    if (e == cudaSuccess) e = cudaMemcpy(p, h, count * sizeof(T), cudaMemcpyHostToDevice);
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
};

// One additive term of a layer input, read from a channels-last fp32 tensor
// [D][H][W][C]:  term(c) = act(x * scale[c] + shift[c]).  scale == nullptr means the
// identity affine.  This is how GroupNorm / BatchNorm + ReLU + residual adds of the
// reference (dfm_backbone.py:175-183, conv_modules.py:129-149) are folded into the
// *load* side of the consuming kernel instead of being separate passes over HBM.
struct Term {
  const float* x;
  const float* scale;
  const float* shift;
  int relu;
  // > 0: x holds only three planes -- z = 0, any interior z, z = zcls - 1 -- of a tensor
  // that is constant along z except at its two ends (the cur-frame half of the plane-sweep
  // volume and everything computed from it alone); zcls is the logical depth.
  int zcls;
};
__device__ __forceinline__ int term_plane(const Term& t, int z) {
  return t.zcls > 0 ? (z == 0 ? 0 : (z == t.zcls - 1 ? 2 : 1)) : z;
}

// value = outer_act( sum_i term_i )
struct Src {
  Term t[3];
  int n;
  int outer_relu;
};

// Closed-form plane-sweep warp (SURVEY.md section 7; dfm_backbone.py:217-314):
// lattice pixel (x*step, y*step) of the network input -> canonical image (undo crop /
// scale / flip) -> [a,b,c] = z * (A [u,v,1]^T) + t with M = P4 * cur2prev * P4^-1
// (computed in fp64 on the host) -> (a/c, b/c) -> redo flip / scale / crop -> feature px.
struct WarpGeom {
  float A[9];
  float t[3];
  float scale, inv_scale;
  float crop_x, crop_y;
  float org_w;
  float lattice;   // feat_sample_factor * cost_sample_factor (image px per volume cell)
  float inv_fsf;   // 1 / feat_sample_factor
  int step;        // cost_sample_factor (feature px per volume cell)
  int flip;
  int Hf, Wf;      // feature map size
};

struct ConvGeom {
  int Di, Hi, Wi, Cin;
  int Do, Ho, Wo, Cout;
  int sd, sh, sw;
  int pd, ph, pw;
  int transposed;  // ConvTranspose3d(k3, s2, p1, op1)
};

// (z, pos): plane index and in-plane voxel index; HW: voxels per plane
__device__ __forceinline__ float load_src(const Src& s, int z, long long pos, long long HW, int C,
                                          int c) {
  float v = 0.f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (i < s.n) {
      float a = __ldg(s.t[i].x + ((long long)term_plane(s.t[i], z) * HW + pos) * C + c);
      if (s.t[i].scale) a = fmaf(a, __ldg(s.t[i].scale + c), __ldg(s.t[i].shift + c));
      if (s.t[i].relu) a = fmaxf(a, 0.f);
      v += a;
    }
  }
  if (s.outer_relu) v = fmaxf(v, 0.f);
  return v;
}

// prev-frame sample position (feature pixels) for volume cell (x, y) on plane depth z
__device__ __forceinline__ void warp_coord(const WarpGeom& g, int x, int y, float z,
                                           float& fx, float& fy) {
  float u = (x * g.lattice + g.crop_x) * g.inv_scale;
  float v = (y * g.lattice + g.crop_y) * g.inv_scale;
  if (g.flip) u = g.org_w - u;
  const float qa = fmaf(g.A[0], u, fmaf(g.A[1], v, g.A[2]));
  const float qb = fmaf(g.A[3], u, fmaf(g.A[4], v, g.A[5]));
  const float qc = fmaf(g.A[6], u, fmaf(g.A[7], v, g.A[8]));
  const float a = fmaf(z, qa, g.t[0]);
  const float b = fmaf(z, qb, g.t[1]);
  const float c = fmaf(z, qc, g.t[2]);
  float pu = a / c, pv = b / c;
  if (g.flip) pu = g.org_w - pu;
  fx = (pu * g.scale - g.crop_x) * g.inv_fsf;
  fy = (pv * g.scale - g.crop_y) * g.inv_fsf;
}

// bilinear tap setup with grid_sample(padding_mode='zeros', align_corners=True)
// semantics: out-of-range corners contribute zero individually; non-finite
// coordinates contribute nothing.
struct Taps {
  int off[4];
  float w[4];
};
__device__ __forceinline__ Taps bilinear_taps(float fx, float fy, int H, int W) {
  Taps t;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    t.off[i] = 0;
    t.w[i] = 0.f;
  }
  if (!(fabsf(fx) < 1e8f) || !(fabsf(fy) < 1e8f)) return t;
  const float x0f = floorf(fx), y0f = floorf(fy);
  const int x0 = (int)x0f, y0 = (int)y0f;
  const float ax = fx - x0f, ay = fy - y0f;
  const float wx[2] = {1.f - ax, ax}, wy[2] = {1.f - ay, ay};
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int xx = x0 + i, yy = y0 + j;
      const bool ok = xx >= 0 && xx < W && yy >= 0 && yy < H;
      t.off[j * 2 + i] = ok ? yy * W + xx : 0;
      t.w[j * 2 + i] = ok ? wx[i] * wy[j] : 0.f;
    }
  return t;
}

}  // namespace dfm
