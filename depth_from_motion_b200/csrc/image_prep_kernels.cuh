// Image preparation of the shipped test pipelines: decoded 8-bit BGR HWC views -> the
// detector's fp32 NCHW `img`, normalised and zero-padded, views stacked.
//
//   crop    (KITTI, dfm_r34_1x8_kitti-3d-3class.py:316-338): RandomCrop3D's window
//           img[y1:y1+h, x1:x1+w] (transforms_3d.py:2527-2542), then Normalize, then Pad.
//   rescale (Waymo, multiview-dfm_r101_dcn_*.py test_pipeline): LoadMultiViewImageFromFiles
//           (to_float32, exact for uint8), MultiViewImageResize3D (mmcv.imrescale: cv2.resize
//           INTER_LINEAR on float32), MultiViewImageNormalize, MultiViewImagePad.
//
// Normalisation is mmcv.imnormalize_ with the float32 mean / std the Normalize transforms store
// (transforms_3d.py:2064-2066): optional BGR->RGB swap, then cv2.subtract and cv2.multiply by
// those values widened to float64.  cv2 subtracts in fp32, x - mean, but multiplies in fp64 and
// rounds once: float(double(x - mean) * (1 / double(std))).  Padding is
// impad_to_multiple with pad_val 0, applied after normalising.  Every arithmetic step below
// uses an explicit round-to-nearest intrinsic, so the compiler cannot contract a multiply and an
// add into an FMA: cv2 rounds each operation separately, and the kernel matches it bit for bit
// because of that.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace dfm {

struct ImagePrepParams {
  int mode;            // 0: crop, 1: rescale
  int src_h, src_w;    // decoded view size
  int crop_x, crop_y;  // crop: window origin
  int out_h, out_w;    // crop: window size; rescale: resized size
  int pad_h, pad_w;    // output plane size (out_* rounded up to the pad divisor)
  int to_rgb;
  double scale_x, scale_y;  // rescale: cv2's 1 / (double(dst) / src)
  float mean[3];
  double stdinv[3];
};

// cv2.resize (INTER_LINEAR, float) source index and weight of the second tap for output
// coordinate d: f = float((d + 0.5) * scale - 0.5), s = floor(f), w = f - s.  Columns clamp
// both ends to the edge pixel with weight 0 (resizeGeneric_'s xofs / alpha); rows do not
// clamp the weight, they clip the two row indices (its yofs / beta and srows).
__device__ __forceinline__ void cv_linear_coord(int d, double scale, int& s, float& w) {
  const float f = __double2float_rn(__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5));
  const float fl = floorf(f);
  s = (int)fl;
  w = __fsub_rn(f, fl);
}

// One thread per output pixel (all three channels); blockIdx.z is the view.  Threads of a
// warp hold consecutive x, so each channel plane's stores are coalesced; the pad region is
// written by the same threads.
__global__ void __launch_bounds__(128)
image_prep_kernel(ImagePrepParams p, const uint8_t* __restrict__ src, float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  const int v = blockIdx.z;
  if (x >= p.pad_w) return;
  const size_t plane = (size_t)p.pad_h * p.pad_w;
  float* o = out + (size_t)v * 3 * plane + (size_t)y * p.pad_w + x;
  float val[3] = {0.f, 0.f, 0.f};
  if (x < p.out_w && y < p.out_h) {
    const uint8_t* img = src + (size_t)v * p.src_h * p.src_w * 3;
    float bgr[3];
    if (p.mode == 0) {
      const uint8_t* px = img + ((size_t)(y + p.crop_y) * p.src_w + (x + p.crop_x)) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) bgr[c] = (float)px[c];
    } else {
      int sx, sy;
      float ax, by;
      cv_linear_coord(x, p.scale_x, sx, ax);
      if (sx < 0) {
        sx = 0;
        ax = 0.f;
      }
      if (sx >= p.src_w - 1) {
        sx = p.src_w - 1;
        ax = 0.f;
      }
      const int sx1 = min(sx + 1, p.src_w - 1);
      cv_linear_coord(y, p.scale_y, sy, by);
      const int sy0 = min(max(sy, 0), p.src_h - 1), sy1 = min(max(sy + 1, 0), p.src_h - 1);
      const float a0 = __fsub_rn(1.f, ax), b0 = __fsub_rn(1.f, by);
      const uint8_t* r0 = img + (size_t)sy0 * p.src_w * 3;
      const uint8_t* r1 = img + (size_t)sy1 * p.src_w * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        // horizontal pass per source row, then the vertical blend (HResizeLinear, VResizeLinear)
        const float h0 = __fadd_rn(__fmul_rn((float)r0[sx * 3 + c], a0),
                                   __fmul_rn((float)r0[sx1 * 3 + c], ax));
        const float h1 = __fadd_rn(__fmul_rn((float)r1[sx * 3 + c], a0),
                                   __fmul_rn((float)r1[sx1 * 3 + c], ax));
        bgr[c] = __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, by));
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float s = bgr[p.to_rgb ? 2 - c : c];
      val[c] = __double2float_rn(__dmul_rn((double)__fsub_rn(s, p.mean[c]), p.stdinv[c]));
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) o[(size_t)c * plane] = val[c];
}

}  // namespace dfm
