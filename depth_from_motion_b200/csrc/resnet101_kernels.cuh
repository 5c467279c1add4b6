// Kernels of mmdet's ResNet-101 with DCNv2 in layer3 / layer4, the image backbone of both
// MultiViewDfM (Waymo) configs.  Activations are channels-last [N][h][w][C] over all images of a
// call.  The stem reuses resnet_stem_kernel and the stride-1 3x3 convs of layer1 / layer2 reuse
// resnet_conv_tc_kernel<64 / 128> (resnet_kernels.cuh); everything else runs here.
//
// rn101_gather_tc_kernel<BN>: every other conv as an implicit GEMM on wgmma whose A operand is
// gathered one (output pixel, tap) row at a time:
//   * 1x1 convs (conv1, conv3, downsample; stride 1 or 2): one tap, the input pixel itself;
//   * the plain stride-2 3x3 layer2.0.conv2 and every conv_offset (3x3, stride 1 or 2, C -> 27
//     padded to 32, + bias): nine integer taps, zero outside the map;
//   * the modulated deformable 3x3 (DCNv2) conv2 of layer3 / layer4 (stride 1 or 2): tap k of
//     output (y, x) samples the input bilinearly at (y s - 1 + ky + dy_k, x s - 1 + kx + dx_k),
//     dy_k / dx_k = channels 2k / 2k + 1 of conv_offset, and scales the sample by mask_k =
//     sigmoid(channel 18 + k).  Each of the 4 corners goes through the input dfm::Term (the
//     producer's BatchNorm + ReLU) BEFORE the blend -- the activation is what is sampled -- and a
//     corner outside the map counts as 0.  The corner index and fraction are formed as
//     (integer tap position + floor(d)) and (d - floor(d)), both exact in fp32, so the sampling
//     point carries no rounding of the absolute coordinate.
//   M = 128 output pixels of the flattened [N][Ho][Wo] grid (tiles may straddle images: every row
//   computes its own image index), N = BN output columns of one CTA, K = 32 input channels of one
//   tap per pipeline stage, in (tap, channel) order.  Work items (m tile, n block) are ordered
//   n-block-fastest so that CTAs reading the same A tile run together and share it in L2; the
//   gather is repeated once per n block (BN = 128 keeps 64 fp32 accumulators per consumer thread
//   inside the 128-register budget of a 512-thread CTA).
//   Two loader groups of 4 warps fill alternate stages: loader thread t owns A row t (its sample
//   geometry is formed once per stage) and writes its four 8-channel chunks, hi and lo, in the
//   K-major no-swizzle layout (16-byte rows, row-contiguous: conflict-free), next to a cp.async
//   copy of the stage's contiguous hi + lo weight slice.  Operands are the project's 3-term bf16
//   split (x_hi w_hi + x_lo w_hi + x_hi w_lo, fp32 accumulation).
//   Epilogue (rn101_store2): the raw conv output; with a block BatchNorm also the Bottleneck
//   output relu(bn3(raw) + identity) (identity a dfm::Term); with a bias (conv_offset) raw =
//   conv + bias and out = raw with the sigmoid applied to channels 18..26.
//
// rn101_conv_simt_kernel: the same convs (and, under conv_impl = simt, every conv of the
// backbone but the stem) on fp32 CUDA cores, with the same gather (rn101_tap / rn101_sample8)
// and the same epilogue.
//
// rn101_maxpool_kernel: relu(bn1(stem)) followed by the 3x3 / 2 / 1 max-pool, channels-last.
#pragma once
#include "resnet_kernels.cuh"

namespace dfm {

constexpr int R1_M = 128;                              // output pixels per tile
constexpr int R1_KC = 32;                              // input channels per stage
constexpr int R1_NSTAGE = 4;
constexpr uint32_t R1_A_LBO = R1_M * 16;               // 8-channel chunk pitch (bytes)
constexpr uint32_t R1_A_HL = (R1_KC / 8) * R1_A_LBO;   // hi -> lo (8 KB)
constexpr uint32_t R1_A_BYTES = 2 * R1_A_HL;           // 16 KB
constexpr int R1_THREADS = 256 + 256;                  // consumer warpgroups | loader warps
constexpr int R1_OM = 32;                              // conv_offset channels (27 + zero padding)
constexpr int R1_SIMT_PIX = 32, R1_SIMT_CO = 64;       // simt tile

template <int BN>
struct R1Cfg {
  static constexpr uint32_t B_LBO = BN * 16;             // K chunk pitch of the weight slice
  static constexpr uint32_t B_HL = (R1_KC / 8) * B_LBO;  // one stage's weight slice, hi (or lo)
  static constexpr uint32_t STAGE_BYTES = R1_A_BYTES + 2 * B_HL;
  static constexpr size_t SMEM = (size_t)R1_NSTAGE * STAGE_BYTES + 2 * R1_NSTAGE * 8;
};

struct Rn101Params {
  Term in;                 // input [N][Hi][Wi][Cin], fused transform
  const float* om;         // deformable: [N][Ho][Wo][32] = dy, dx of tap k at 2k, 2k + 1 and
                           // sigmoid masks at 18 + k; null: integer taps
  const uint8_t* wimg;     // tc: [Cout / BN][k * k][Cin / 32][hi | lo][4 chunks][BN][8] bf16
  const float* wt;         // simt: [k * k][Cin][Cout] fp32
  const float* bias;       // conv_offset: [Cout]
  float* raw;              // raw conv output [N][Ho][Wo][Cout]
  const float* bscale;     // optional block epilogue: out = relu(raw * bscale + bshift + id)
  const float* bshift;
  Term id;                 // identity [N][Ho][Wo][Cout]
  float* out;
  int N, Hi, Wi, Ho, Wo, Cin, Cout;
  int k, stride, pad;
  int P;                   // N * Ho * Wo
  int mtiles, nblk, items;
  int* err;
};

// Sample geometry of one (output pixel, tap): element offsets of the 4 corners ((y0, x0),
// (y0, x0 + 1), (y0 + 1, x0), (y0 + 1, x0 + 1); -1 = outside the map or unused), their bilinear
// weights and the modulation mask.
struct R1Tap {
  long long off[4];
  float w[4];
  float m;
};

__device__ __forceinline__ void rn101_tap(const Rn101Params& p, long long pix, int tap, R1Tap& g) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    g.off[c] = -1;
    g.w[c] = 0.f;
  }
  g.m = 1.f;
  if (pix >= p.P) return;
  const int xo = (int)(pix % p.Wo), yo = (int)((pix / p.Wo) % p.Ho);
  const long long img = pix / ((long long)p.Wo * p.Ho);
  const int ky = tap / p.k, kx = tap - ky * p.k;
  const int yi = yo * p.stride - p.pad + ky, xi = xo * p.stride - p.pad + kx;
  const long long ibase = img * p.Hi * p.Wi;
  if (!p.om) {
    if (yi >= 0 && yi < p.Hi && xi >= 0 && xi < p.Wi) {
      g.off[0] = (ibase + (long long)yi * p.Wi + xi) * p.Cin;
      g.w[0] = 1.f;
    }
    return;
  }
  const float* o = p.om + pix * R1_OM;
  const float dy = __ldg(o + 2 * tap), dx = __ldg(o + 2 * tap + 1);
  g.m = __ldg(o + 18 + tap);
  // floor(d) clamped so the int conversion is defined; such a point is off the map anyway
  const float fy = fminf(fmaxf(floorf(dy), -1048576.f), 1048576.f);
  const float fx = fminf(fmaxf(floorf(dx), -1048576.f), 1048576.f);
  const float ly = dy - fy, lx = dx - fx, hy = 1.f - ly, hx = 1.f - lx;
  const int y0 = yi + (int)fy, x0 = xi + (int)fx;
  g.w[0] = hy * hx;
  g.w[1] = hy * lx;
  g.w[2] = ly * hx;
  g.w[3] = ly * lx;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int y = y0 + (c >> 1), x = x0 + (c & 1);
    if (y >= 0 && y < p.Hi && x >= 0 && x < p.Wi) g.off[c] = (ibase + (long long)y * p.Wi + x) * p.Cin;
  }
}

// 8 channels [c0, c0 + 8) of one tap's sample: sum_c w_c * term(corner_c), times the mask
__device__ __forceinline__ void rn101_sample8(const Rn101Params& p, const R1Tap& g, int c0,
                                              float v[8]) {
  float4 r[4][2];
#pragma unroll
  for (int c = 0; c < 4; ++c)
    if (g.off[c] >= 0) {
      const float4* src = reinterpret_cast<const float4*>(p.in.x + g.off[c] + c0);
      r[c][0] = __ldg(src);
      r[c][1] = __ldg(src + 1);
    }
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    float sc = 1.f, sh = 0.f;
    if (p.in.scale) {
      sc = __ldg(p.in.scale + c0 + e);
      sh = __ldg(p.in.shift + c0 + e);
    }
    float acc = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if (g.off[c] < 0) continue;
      const float4 q = r[c][e >> 2];
      float a = (e & 3) == 0 ? q.x : (e & 3) == 1 ? q.y : (e & 3) == 2 ? q.z : q.w;
      if (p.in.scale) a = fmaf(a, sc, sh);
      if (p.in.relu) a = fmaxf(a, 0.f);
      acc = fmaf(g.w[c], a, acc);
    }
    v[e] = acc * g.m;
  }
}

// Epilogue of output channels n, n + 1 (n even) of pixel pix.
__device__ __forceinline__ void rn101_store2(const Rn101Params& p, long long pix, int n, float v0,
                                             float v1) {
  const long long o = pix * p.Cout + n;
  if (p.bias) {
    v0 += __ldg(p.bias + n);
    v1 += __ldg(p.bias + n + 1);
    *reinterpret_cast<float2*>(p.raw + o) = make_float2(v0, v1);
    const float s0 = (n >= 18 && n < 27) ? 1.f / (1.f + expf(-v0)) : v0;
    const float s1 = (n + 1 >= 18 && n + 1 < 27) ? 1.f / (1.f + expf(-v1)) : v1;
    *reinterpret_cast<float2*>(p.out + o) = make_float2(s0, s1);
    return;
  }
  *reinterpret_cast<float2*>(p.raw + o) = make_float2(v0, v1);
  if (!p.bscale) return;
  const float a = fmaf(v0, __ldg(p.bscale + n), __ldg(p.bshift + n)) + rn_term(p.id, o, n);
  const float b = fmaf(v1, __ldg(p.bscale + n + 1), __ldg(p.bshift + n + 1)) +
                  rn_term(p.id, o + 1, n + 1);
  *reinterpret_cast<float2*>(p.out + o) = make_float2(fmaxf(a, 0.f), fmaxf(b, 0.f));
}

template <int BN>
__global__ void __launch_bounds__(R1_THREADS, 1)
rn101_gather_tc_kernel(const __grid_constant__ Rn101Params p) {
  using Cfg = R1Cfg<BN>;
  constexpr uint32_t STAGE = Cfg::STAGE_BYTES, B_HL = Cfg::B_HL, B_LBO = Cfg::B_LBO;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + R1_NSTAGE * STAGE);
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const uint32_t bar0 = smem_u32(bars);
  auto full = [&](int s) { return bar0 + 8u * s; };
  auto empty = [&](int s) { return bar0 + 8u * (R1_NSTAGE + s); };
  if (tid == 0) {
    for (int s = 0; s < R1_NSTAGE; ++s) {
      mbar_init(full(s), 4);    // one arrival per loader warp of the group
      mbar_init(empty(s), 8);   // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int ncc = p.Cin / R1_KC, nks = p.k * p.k * ncc;

  if (warp >= 8) {
    // ================================ loaders ================================
    const int lw = warp - 8, grp = lw >> 2, lt = (lw & 3) * 32 + lane;
    uint32_t ctr = 0;
    for (int item = blockIdx.x; item < p.items; item += gridDim.x) {
      const int mt = item / p.nblk, nb = item - mt * p.nblk;
      const long long pix = (long long)mt * R1_M + lt;
      const uint8_t* wb = p.wimg + (size_t)nb * nks * 2 * B_HL;
      for (int ks = 0; ks < nks; ++ks, ++ctr) {
        if ((int)(ctr & 1) != grp) continue;
        const int s = ctr % R1_NSTAGE;
        const int tap = ks / ncc, kc = ks - tap * ncc;
        R1Tap g;
        rn101_tap(p, pix, tap, g);
        mbar_wait(empty(s), ((ctr / R1_NSTAGE) & 1) ^ 1, p.err);
        uint8_t* st = smem + s * STAGE;
        const uint32_t b_dst = smem_u32(st + R1_A_BYTES);
        const uint8_t* b_src = wb + (size_t)ks * 2 * B_HL;
#pragma unroll 1
        for (uint32_t i = lt; i < 2 * B_HL / 16; i += 128) cp_async16_rn(b_dst + 16 * i, b_src + 16 * i);
#pragma unroll 1
        for (int ch = 0; ch < R1_KC / 8; ++ch) {
          float v[8];
          rn101_sample8(p, g, kc * R1_KC + ch * 8, v);
          split_store(v, st + ch * R1_A_LBO + lt * 16, st + R1_A_HL + ch * R1_A_LBO + lt * 16);
        }
        asm volatile("cp.async.wait_all;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) mbar_arrive(full(s));
      }
    }
  } else {
    // ===================== consumer warpgroups: MMA, then the epilogue =====================
    const int wg = warp >> 2, wq = warp & 3;
    const uint32_t desc_hi = 128u >> 4;                   // SBO: dense 8-row groups
    float acc[BN / 2];
    uint32_t ctr = 0;
    for (int item = blockIdx.x; item < p.items; item += gridDim.x) {
      const int mt = item / p.nblk, nb = item - mt * p.nblk;
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      for (int ks = 0; ks < nks; ++ks, ++ctr) {
        const int s = ctr % R1_NSTAGE;
        mbar_wait(full(s), (ctr / R1_NSTAGE) & 1, p.err);
        const uint32_t st = smem_u32(smem + s * STAGE);
        const uint32_t a_lo = (((st + wg * 64 * 16) >> 4) & 0x3FFF) | ((R1_A_LBO >> 4) << 16);
        const uint32_t b_lo = (((st + R1_A_BYTES) >> 4) & 0x3FFF) | ((B_LBO >> 4) << 16);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < R1_KC / 16; ++kk) {
          const uint64_t ah = pack64(a_lo + 2 * kk * (R1_A_LBO >> 4), desc_hi);
          const uint64_t al = pack64(a_lo + 2 * kk * (R1_A_LBO >> 4) + (R1_A_HL >> 4), desc_hi);
          const uint64_t bh = pack64(b_lo + 2 * kk * (B_LBO >> 4), desc_hi);
          const uint64_t bl = pack64(b_lo + 2 * kk * (B_LBO >> 4) + (B_HL >> 4), desc_hi);
          wgmma_bf16<BN>(acc, ah, bh);
          wgmma_bf16<BN>(acc, al, bh);
          wgmma_bf16<BN>(acc, ah, bl);
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(empty(s));
      }
      // registers (4j + 2rr, 4j + 2rr + 1): tile row 64 wg + 16 wq + lane / 4 + 8 rr,
      //                                     columns 8 j + 2 (lane % 4) + {0, 1}
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const long long pix = (long long)mt * R1_M + 64 * wg + 16 * wq + (lane >> 2) + 8 * rr;
        if (pix >= p.P) continue;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
          rn101_store2(p, pix, nb * BN + 8 * j + 2 * (lane & 3), acc[4 * j + 2 * rr],
                       acc[4 * j + 2 * rr + 1]);
      }
    }
  }
}

// 32 output pixels x 64 output channels per CTA of 256 threads; thread (ty, tx) accumulates
// pixels 2 ty, 2 ty + 1 and channels 4 tx .. 4 tx + 3 in fp32, in (tap, input channel) order.
__global__ void __launch_bounds__(256) rn101_conv_simt_kernel(const Rn101Params p) {
  __shared__ float a_s[R1_KC][R1_SIMT_PIX + 1];
  __shared__ __align__(16) float w_s[R1_KC][R1_SIMT_CO];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const long long pix0 = (long long)blockIdx.x * R1_SIMT_PIX;
  const int co0 = blockIdx.y * R1_SIMT_CO;
  const int gp = tid & 31, gch = tid >> 5;              // gather: pixel, 8-channel chunk
  const int ncc = p.Cin / R1_KC;
  float acc[2][4] = {};
  for (int tap = 0; tap < p.k * p.k; ++tap) {
    R1Tap g;
    if (tid < 128) rn101_tap(p, pix0 + gp, tap, g);
    for (int kc = 0; kc < ncc; ++kc) {
      __syncthreads();
      if (tid < 128) {
        float v[8];
        rn101_sample8(p, g, kc * R1_KC + gch * 8, v);
#pragma unroll
        for (int e = 0; e < 8; ++e) a_s[gch * 8 + e][gp] = v[e];
      }
      for (int i = tid; i < R1_KC * R1_SIMT_CO; i += 256) {
        const int ci = i / R1_SIMT_CO, co = co0 + i % R1_SIMT_CO;
        w_s[ci][i % R1_SIMT_CO] =
            co < p.Cout ? __ldg(p.wt + ((long long)tap * p.Cin + kc * R1_KC + ci) * p.Cout + co) : 0.f;
      }
      __syncthreads();
#pragma unroll 8
      for (int ci = 0; ci < R1_KC; ++ci) {
        const float a0 = a_s[ci][2 * ty], a1 = a_s[ci][2 * ty + 1];
        const float4 w = *reinterpret_cast<const float4*>(&w_s[ci][4 * tx]);
        acc[0][0] = fmaf(a0, w.x, acc[0][0]);
        acc[0][1] = fmaf(a0, w.y, acc[0][1]);
        acc[0][2] = fmaf(a0, w.z, acc[0][2]);
        acc[0][3] = fmaf(a0, w.w, acc[0][3]);
        acc[1][0] = fmaf(a1, w.x, acc[1][0]);
        acc[1][1] = fmaf(a1, w.y, acc[1][1]);
        acc[1][2] = fmaf(a1, w.z, acc[1][2]);
        acc[1][3] = fmaf(a1, w.w, acc[1][3]);
      }
    }
  }
  const int n = co0 + 4 * tx;
  if (n >= p.Cout) return;
#pragma unroll
  for (int v = 0; v < 2; ++v) {
    const long long pix = pix0 + 2 * ty + v;
    if (pix >= p.P) continue;
    rn101_store2(p, pix, n, acc[v][0], acc[v][1]);
    rn101_store2(p, pix, n + 2, acc[v][2], acc[v][3]);
  }
}

// out [N][Ho][Wo][64] = maxpool 3x3 / 2 / 1 of relu(bn1(stem raw)); one thread per 4 channels
__global__ void __launch_bounds__(256)
rn101_maxpool_kernel(const Term in, float* __restrict__ out, int N, int Hi, int Wi, int Ho, int Wo) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * Ho * Wo * 16) return;
  const int c = 4 * (int)(i & 15);
  const long long pix = i >> 4;
  const int xo = (int)(pix % Wo), yo = (int)((pix / Wo) % Ho);
  const long long img = pix / ((long long)Wo * Ho);
  float m[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
  for (int ky = 0; ky < 3; ++ky) {
    const int y = 2 * yo - 1 + ky;
    if (y < 0 || y >= Hi) continue;
    for (int kx = 0; kx < 3; ++kx) {
      const int x = 2 * xo - 1 + kx;
      if (x < 0 || x >= Wi) continue;
      const long long b = ((img * Hi + y) * Wi + x) * 64 + c;
#pragma unroll
      for (int e = 0; e < 4; ++e) m[e] = fmaxf(m[e], rn_term(in, b + e, c + e));
    }
  }
  *reinterpret_cast<float4*>(out + pix * 64 + c) = make_float4(m[0], m[1], m[2], m[3]);
}

}  // namespace dfm
