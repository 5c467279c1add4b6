// Kernels behind the detectors' per-view image-feature cache (modules.DfM.set_feature_cache):
// a 128-bit content fingerprint of each input view, and a bitwise comparison of view pairs.
//
// Fingerprint.  Word i (the raw 32 bits w of element i) of a view contributes, in each of two
// lanes with keys K_j and odd multipliers M_j,
//     x = ((uint64(w) << 32) ^ uint64(i) ^ K_j) * M_j,   mix = x ^ (x >> 32),
// and a lane is the sum of mix over the view modulo 2^64.  mix is a bijection of w for a given
// i (xor with a constant, odd multiply, xorshift), so any change of one word changes the sum;
// the xorshift after the multiply makes it non-linear, so swapped words change it too.  It
// costs one 64-bit multiply per lane and word.  The sum is order-free, so the 64-bit atomics
// that combine the blocks give the same bits whatever the thread order.  Raw bits: -0.0 and
// +0.0 differ, and so do NaN payloads.  tests/test_view_cache.py restates it in numpy.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace dfm {

constexpr unsigned long long kViewKey0 = 0x9E3779B97F4A7C15ULL;
constexpr unsigned long long kViewKey1 = 0xC2B2AE3D27D4EB4FULL;
constexpr unsigned long long kViewMul0 = 0xBF58476D1CE4E5B9ULL;
constexpr unsigned long long kViewMul1 = 0x94D049BB133111EBULL;

__device__ __forceinline__ unsigned long long view_mix(unsigned w, unsigned long long i,
                                                       unsigned long long key,
                                                       unsigned long long mul) {
  const unsigned long long x = (((unsigned long long)w << 32) ^ i ^ key) * mul;
  return x ^ (x >> 32);
}

__device__ __forceinline__ void view_add(unsigned w, unsigned long long i, unsigned long long& a,
                                         unsigned long long& b) {
  a += view_mix(w, i, kViewKey0, kViewMul0);
  b += view_mix(w, i, kViewKey1, kViewMul1);
}

// grid (blocks per view, num_views), 256 threads; out[v][2] must be zero on entry.  Each view
// is read as a scalar head up to 16-byte alignment, a 16-byte body and a scalar tail.
__global__ void __launch_bounds__(256)
view_fingerprint_kernel(const float* __restrict__ views, long long n,
                        unsigned long long* __restrict__ out) {
  const unsigned* p = reinterpret_cast<const unsigned*>(views + (long long)blockIdx.y * n);
  long long head = (long long)(((16 - (reinterpret_cast<uintptr_t>(p) & 15)) & 15) >> 2);
  if (head > n) head = n;
  const long long nvec = (n - head) >> 2;
  const uint4* q = reinterpret_cast<const uint4*>(p + head);
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nth = (long long)gridDim.x * blockDim.x;
  unsigned long long a = 0, b = 0;
  for (long long k = tid; k < nvec; k += nth) {
    const uint4 w = q[k];
    const unsigned long long i = (unsigned long long)(head + 4 * k);
    view_add(w.x, i, a, b);
    view_add(w.y, i + 1, a, b);
    view_add(w.z, i + 2, a, b);
    view_add(w.w, i + 3, a, b);
  }
  for (long long k = tid; k < head; k += nth) view_add(p[k], (unsigned long long)k, a, b);
  for (long long k = head + 4 * nvec + tid; k < n; k += nth)
    view_add(p[k], (unsigned long long)k, a, b);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  __shared__ unsigned long long red[2][8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    red[0][warp] = a;
    red[1][warp] = b;
  }
  __syncthreads();
  if (threadIdx.x < 2) {
    unsigned long long s = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[threadIdx.x][w];
    atomicAdd(out + 2 * blockIdx.y + threadIdx.x, s);
  }
}

// Up to 64 (a, b) view pairs per launch, passed by value.
constexpr int kViewPairsPerLaunch = 64;
struct ViewPairs {
  const float* a[kViewPairsPerLaunch];
  const float* b[kViewPairsPerLaunch];
};

// grid (blocks per pair, pairs); mismatch[pair] is set to 1 when any 32-bit word differs and is
// left alone otherwise.  vec: every pointer is 16-byte aligned and n % 4 == 0.
__global__ void __launch_bounds__(256)
views_equal_kernel(ViewPairs t, long long n, int vec, int* __restrict__ mismatch) {
  const unsigned* a = reinterpret_cast<const unsigned*>(t.a[blockIdx.y]);
  const unsigned* b = reinterpret_cast<const unsigned*>(t.b[blockIdx.y]);
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nth = (long long)gridDim.x * blockDim.x;
  unsigned diff = 0;
  if (vec) {
    const uint4* a4 = reinterpret_cast<const uint4*>(a);
    const uint4* b4 = reinterpret_cast<const uint4*>(b);
    for (long long k = tid; k < (n >> 2); k += nth) {
      const uint4 x = a4[k], y = b4[k];
      diff |= (x.x ^ y.x) | (x.y ^ y.y) | (x.z ^ y.z) | (x.w ^ y.w);
    }
  } else {
    for (long long k = tid; k < n; k += nth) diff |= a[k] ^ b[k];
  }
  if (__syncthreads_or(diff != 0) && threadIdx.x == 0) mismatch[blockIdx.y] = 1;
}

}  // namespace dfm
