// DfM's LiDAR imitation loss (DfM.imitation_loss / get_imitation_reg_layer_loss,
// detectors/dfm.py:455-539, with imitation_utils.py's NormalizeLayer('cw_scale') and
// WeightedL2WithSigmaLoss) for a batch of B samples and one or two feature pairs: a stereo
// feature x [B][C][Z][ny][nx] (Z = 1 for the BEV pair), its 1x1 imitation conv (W [C][C], bias
// [C]) and the teacher's feature t of the same shape.  A row is one (b, z, y, x) position; it is
// positive when its BEV cell's anchor centre lies in one of the sample's GT boxes and any channel
// of the teacher row is non-zero (NaN counts as non-zero):
//
//   im_inbox_kernel      one thread per (sample, BEV cell): mmcv's points_in_boxes_part test of
//                        the cell's anchor centre (z = 0) against the sample's GT (z = 0), fp32
//   im_forward_kernel    per pair, a fixed grid striding over chunks of IM_THREADS rows: at the
//                        positives the conv row, sum_c 0.5 (pred_c - t_c / scale_c)^2 with the
//                        old scale (0 at NaN targets), the row count and |t_c|; fixed per-block
//                        partials, fp64
//   im_reduce_kernel     one CTA: the partials in block order, packed per pair as
//                        (count / world, count, sum |t_c|) in fp32 for one all-reduce
//   im_finish_kernel     one warp: the normaliser 1 / max(mean count, clamp), the losses, the
//                        gradient coefficients and, in training mode, the running-scale update
//   im_backward_kernel   per pair, the same grid: grad_x at every position (W^T g at positives,
//                        0 elsewhere) with g = coef * (pred - t), and per-block partials of
//                        sum g x^T and sum g in fp64
//   im_wreduce_kernel    grad_W and grad_b from those partials in block order
//
// No floating-point atomics anywhere, so repeated calls are bitwise equal.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace dfm {

constexpr int IM_THREADS = 256;  // rows per chunk and threads per block
constexpr int IM_MAX_PAIRS = 2;
constexpr int IM_MAX_SAMPLES = 64;

struct ImPair {
  int C, Z;                 // channels, z slices (1 for the BEV pair)
  long long R;              // rows per sample: Z * ny * nx
  float loss_weight;
  const float* x;           // stereo feature [B][C][Z][ny][nx]
  const float* t;           // teacher feature, same layout
  const float* W;           // [C][C] (out, in)
  const float* bias;        // [C]
  float* scale;             // [C] the cw_scale buffer, updated in place by finish in training
  float* old_scale;         // [C] workspace: the buffer as it was at this call's start
  float* gx;                // grad of x, or null
  float* gW;                // grad of W, or null
  float* gb;                // grad of bias, or null
  double* part_loss;        // [blocks]
  int* part_cnt;            // [blocks]
  double* part_abs;         // [blocks][C]
  double* part_gw;          // [blocks][C * C + C]: sum g x^T, then sum g
};

struct ImParams {
  int B, ny, nx, P, blocks;
  float clamp;
  const float* anchor_x;    // [nx] anchor centre x of each BEV column
  const float* anchor_y;    // [ny]
  const float* gt;          // [G][7] (only columns 0, 1, 3, 4, 5, 6 are read: z is taken as 0)
  const int* gt_off;        // [B + 1]
  unsigned char* inbox;     // [B][ny][nx]
  double* loss_sum;         // [P] the unnormalised loss sums of this rank
  int* count;               // [P] positives of this rank
  ImPair pair[IM_MAX_PAIRS];
};

// mmcv 1.x check_pt_in_box3d for a point at z = 0 and a box whose bottom centre z is 0, in fp32
// with every product and sum rounded on its own (no FMA contraction), so it is exact at rz = 0
__device__ __forceinline__ bool im_point_in_box(float x, float y, const float* box) {
  const float cx = box[0], cy = box[1], dx = box[3], dy = box[4], dz = box[5], rz = box[6];
  const float cz = dz * 0.5f;                    // cz (0) += dz / 2.0
  if (fabsf(0.f - cz) > dz * 0.5f) return false;
  const float cosa = cosf(-rz), sina = sinf(-rz);
  const float sx = __fsub_rn(x, cx), sy = __fsub_rn(y, cy);
  const float lx = __fadd_rn(__fmul_rn(sx, cosa), __fmul_rn(sy, -sina));
  const float ly = __fadd_rn(__fmul_rn(sx, sina), __fmul_rn(sy, cosa));
  const float hx = dx * 0.5f, hy = dy * 0.5f;
  return lx > -hx && lx < hx && ly > -hy && ly < hy;
}

__global__ void __launch_bounds__(IM_THREADS) im_inbox_kernel(ImParams p) {
  const int cells = p.ny * p.nx;
  const int i = blockIdx.x * IM_THREADS + threadIdx.x;
  if (i >= p.B * cells) return;
  const int b = i / cells, c = i % cells;
  const float x = p.anchor_x[c % p.nx], y = p.anchor_y[c / p.nx];
  unsigned char in = 0;
  for (int g = p.gt_off[b]; g < p.gt_off[b + 1]; ++g)
    if (im_point_in_box(x, y, p.gt + (size_t)g * 7)) { in = 1; break; }
  p.inbox[i] = in;
}

// positive test of row (b, r): in-box cell and a teacher row with any channel != 0
template <int C>
__device__ __forceinline__ bool im_positive(const ImParams& p, const ImPair& q, int b, long long r,
                                            const float* t) {
  const int cells = p.ny * p.nx;
  if (!p.inbox[(size_t)b * cells + (int)(r % cells)]) return false;
  bool any = false;
#pragma unroll 8
  for (int c = 0; c < C; ++c) any |= !(t[(long long)c * q.R] == 0.f);
  return any;
}

// dynamic shared memory of the forward (the |t| tile) and backward (x and g tiles) kernels
__host__ __device__ constexpr size_t im_forward_smem(int C) {
  return (size_t)IM_THREADS * (C + 1) * sizeof(float);
}
__host__ __device__ constexpr size_t im_backward_smem(int C) {
  return 2 * im_forward_smem(C) +
         (size_t)((C * C + C + IM_THREADS - 1) / IM_THREADS) * IM_THREADS * sizeof(double);
}

// pred_c of a row held in registers, with the weights in shared memory
template <int C>
__device__ __forceinline__ float im_pred(const float* Ws, const float* bs, const float* xr, int c) {
  float acc = bs[c];
#pragma unroll
  for (int k = 0; k < C; ++k) acc = fmaf(Ws[c * C + k], xr[k], acc);
  return acc;
}

// pred_c - target_c with NaN targets replaced by the prediction (WeightedL2WithSigmaLoss)
__device__ __forceinline__ float im_diff(float pred, float tv, float sc) {
  const float tn = __fdiv_rn(tv, sc);
  return __fsub_rn(pred, isnan(tn) ? pred : tn);
}

template <int C>
__device__ __forceinline__ void im_load_weights(const ImPair& q, float* Ws, float* bs, float* ss) {
  for (int i = threadIdx.x; i < C * C; i += IM_THREADS) Ws[i] = q.W[i];
  for (int i = threadIdx.x; i < C; i += IM_THREADS) {
    bs[i] = q.bias[i];
    ss[i] = q.old_scale[i];
  }
  __syncthreads();
}

template <int C>
__global__ void __launch_bounds__(IM_THREADS) im_forward_kernel(ImParams p, int pi) {
  constexpr int PARTS = IM_THREADS / C;  // threads summing one channel of the |t| tile
  __shared__ float Ws[C * C], bs[C], ss[C];
  extern __shared__ float im_dyn[];
  float(*tile)[C + 1] = reinterpret_cast<float(*)[C + 1]>(im_dyn);  // [IM_THREADS][C + 1]
  __shared__ double red[IM_THREADS];
  __shared__ int redc[IM_THREADS];
  const ImPair& q = p.pair[pi];
  im_load_weights<C>(q, Ws, bs, ss);
  const long long rows = (long long)p.B * q.R;
  const long long chunks = (rows + IM_THREADS - 1) / IM_THREADS;
  double loss = 0.0, abs_acc = 0.0;
  int cnt = 0;
  const int ac = threadIdx.x % C, apart = threadIdx.x / C;
  for (long long ch = blockIdx.x; ch < chunks; ch += gridDim.x) {
    const long long g = ch * IM_THREADS + threadIdx.x;
    bool pos = false;
    int b = 0;
    long long r = 0;
    if (g < rows) {
      b = (int)(g / q.R);
      r = g % q.R;
      pos = im_positive<C>(p, q, b, r, q.t + (size_t)b * C * q.R + r);
    }
    if (!__syncthreads_or(pos)) continue;
    if (pos) {
      const float* xp = q.x + (size_t)b * C * q.R + r;
      const float* tp = q.t + (size_t)b * C * q.R + r;
      float xr[C];
#pragma unroll
      for (int k = 0; k < C; ++k) xr[k] = xp[(long long)k * q.R];
      for (int c = 0; c < C; ++c) {
        const float tv = tp[(long long)c * q.R];
        const float d = im_diff(im_pred<C>(Ws, bs, xr, c), tv, ss[c]);
        loss += 0.5 * (double)d * (double)d;
        tile[threadIdx.x][c] = fabsf(tv);
      }
      ++cnt;
    } else {
#pragma unroll 8
      for (int c = 0; c < C; ++c) tile[threadIdx.x][c] = 0.f;
    }
    __syncthreads();
    for (int i = apart; i < IM_THREADS; i += PARTS) abs_acc += (double)tile[i][ac];
    __syncthreads();
  }
  // block partials in a fixed tree order
  red[threadIdx.x] = loss;
  redc[threadIdx.x] = cnt;
  __syncthreads();
  for (int h = IM_THREADS / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) {
      red[threadIdx.x] += red[threadIdx.x + h];
      redc[threadIdx.x] += redc[threadIdx.x + h];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    q.part_loss[blockIdx.x] = red[0];
    q.part_cnt[blockIdx.x] = redc[0];
  }
  __syncthreads();
  red[threadIdx.x] = abs_acc;
  __syncthreads();
  if (threadIdx.x < C) {
    double s = 0.0;
    for (int k = 0; k < PARTS; ++k) s += red[k * C + threadIdx.x];
    q.part_abs[(size_t)blockIdx.x * C + threadIdx.x] = s;
  }
}

// red per pair: [count / world, count, sum |t_c| (C)]
__global__ void __launch_bounds__(IM_THREADS) im_reduce_kernel(ImParams p, int world,
                                                               float* packed) {
  __shared__ double red[IM_THREADS];
  __shared__ long long redc[IM_THREADS];
  int off = 0;
  for (int pi = 0; pi < p.P; ++pi) {
    const ImPair& q = p.pair[pi];
    double s = 0.0;
    long long n = 0;
    for (int i = threadIdx.x; i < p.blocks; i += IM_THREADS) {
      s += q.part_loss[i];
      n += q.part_cnt[i];
    }
    red[threadIdx.x] = s;
    redc[threadIdx.x] = n;
    __syncthreads();
    for (int h = IM_THREADS / 2; h > 0; h >>= 1) {
      if (threadIdx.x < h) {
        red[threadIdx.x] += red[threadIdx.x + h];
        redc[threadIdx.x] += redc[threadIdx.x + h];
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      p.loss_sum[pi] = red[0];
      p.count[pi] = (int)redc[0];
      const float cf = (float)redc[0];
      packed[off] = __fdiv_rn(cf, (float)world);  // dist_reduce_mean's t / world_size
      packed[off + 1] = cf;
    }
    for (int c = threadIdx.x; c < q.C; c += IM_THREADS) {
      double a = 0.0;
      for (int i = 0; i < p.blocks; ++i) a += q.part_abs[(size_t)i * q.C + c];
      packed[off + 2 + c] = (float)a;
    }
    __syncthreads();
    off += 2 + q.C;
  }
}

// packed: the all-reduced buffer; losses [P]; coef [P] the factor that turns pred - t into the
// loss's gradient with respect to pred
__global__ void im_finish_kernel(ImParams p, const float* packed, int training, float* losses,
                                 float* coef) {
  int off = 0;
  for (int pi = 0; pi < p.P; ++pi) {
    const ImPair& q = p.pair[pi];
    const float mean = packed[off], n = packed[off + 1];
    // reg_weights = 1 / clamp(N, min=clamp) in fp32
    const float nc = fmaxf(mean, p.clamp);
    const float w = __fdiv_rn(1.f, isnan(mean) ? mean : nc);
    if (threadIdx.x == 0) {
      losses[pi] = (float)(p.loss_sum[pi] / q.C * (double)w / p.B * (double)q.loss_weight);
      coef[pi] = (float)((double)q.loss_weight * (double)w / ((double)p.B * q.C));
    }
    if (training && n > 10.f) {
      for (int c = threadIdx.x; c < q.C; c += blockDim.x) {
        const float ns = __fdiv_rn(packed[off + 2 + c], n);
        q.scale[c] = __fadd_rn(__fmul_rn(q.scale[c], 0.99f), __fmul_rn(ns, 0.01f));
      }
    }
    off += 2 + q.C;
  }
}

template <int C>
__global__ void __launch_bounds__(IM_THREADS, 1)
    im_backward_kernel(ImParams p, int pi, const float* coef, const float* grad_out) {
  constexpr int E = (C * C + C + IM_THREADS - 1) / IM_THREADS;  // partial entries per thread
  __shared__ float Ws[C * C], bs[C], ss[C];
  extern __shared__ float im_dyn[];
  float(*xs)[C + 1] = reinterpret_cast<float(*)[C + 1]>(im_dyn);  // [IM_THREADS][C + 1] each
  float(*gs)[C + 1] = reinterpret_cast<float(*)[C + 1]>(im_dyn + IM_THREADS * (C + 1));
  const ImPair& q = p.pair[pi];
  im_load_weights<C>(q, Ws, bs, ss);
  const float k0 = grad_out ? __fmul_rn(coef[pi], grad_out[pi]) : coef[pi];
  const bool want_w = q.gW || q.gb;
  const long long rows = (long long)p.B * q.R;
  const long long chunks = (rows + IM_THREADS - 1) / IM_THREADS;
  // this thread's running partials of [W | bias] entries e * IM_THREADS + threadIdx.x
  double* acc = reinterpret_cast<double*>(im_dyn + 2 * IM_THREADS * (C + 1));
  for (int e = 0; e < E; ++e) acc[e * IM_THREADS + threadIdx.x] = 0.0;
  for (long long ch = blockIdx.x; ch < chunks; ch += gridDim.x) {
    const long long g = ch * IM_THREADS + threadIdx.x;
    bool pos = false;
    int b = 0;
    long long r = 0;
    if (g < rows) {
      b = (int)(g / q.R);
      r = g % q.R;
      pos = im_positive<C>(p, q, b, r, q.t + (size_t)b * C * q.R + r);
    }
    const bool any = __syncthreads_or(pos);
    float* gxp = q.gx && g < rows ? q.gx + (size_t)b * C * q.R + r : nullptr;
    if (!pos) {
      if (gxp) {
#pragma unroll 8
        for (int k = 0; k < C; ++k) gxp[(long long)k * q.R] = 0.f;
      }
      if (any && want_w) {
#pragma unroll 8
        for (int c = 0; c < C; ++c) xs[threadIdx.x][c] = gs[threadIdx.x][c] = 0.f;
      }
    } else {
      // the x row is staged in this thread's row of the x tile (which the grad_W partials read
      // too), so only the C grad_x accumulators live in registers
      const float* xp = q.x + (size_t)b * C * q.R + r;
      const float* tp = q.t + (size_t)b * C * q.R + r;
      const float* xr = xs[threadIdx.x];
      float gr[C];
#pragma unroll
      for (int k = 0; k < C; ++k) {
        xs[threadIdx.x][k] = xp[(long long)k * q.R];
        gr[k] = 0.f;
      }
      for (int c = 0; c < C; ++c) {
        const float gc =
            __fmul_rn(k0, im_diff(im_pred<C>(Ws, bs, xr, c), tp[(long long)c * q.R], ss[c]));
#pragma unroll
        for (int k = 0; k < C; ++k) gr[k] = fmaf(Ws[c * C + k], gc, gr[k]);
        gs[threadIdx.x][c] = gc;
      }
      if (gxp) {
#pragma unroll
        for (int k = 0; k < C; ++k) gxp[(long long)k * q.R] = gr[k];
      }
    }
    if (!any || !want_w) continue;
    __syncthreads();
#pragma unroll 1
    for (int e = 0; e < E; ++e) {
      const int idx = e * IM_THREADS + threadIdx.x;
      if (idx < C * C) {
        const int c = idx / C, k = idx % C;
        double s = 0.0;
        for (int i = 0; i < IM_THREADS; ++i) s += (double)gs[i][c] * (double)xs[i][k];
        acc[e * IM_THREADS + threadIdx.x] += s;
      } else if (idx < C * C + C) {
        const int c = idx - C * C;
        double s = 0.0;
        for (int i = 0; i < IM_THREADS; ++i) s += (double)gs[i][c];
        acc[e * IM_THREADS + threadIdx.x] += s;
      }
    }
    __syncthreads();
  }
  if (!want_w) return;
  for (int e = 0; e < E; ++e) {
    const int idx = e * IM_THREADS + threadIdx.x;
    if (idx < C * C + C) q.part_gw[(size_t)blockIdx.x * (C * C + C) + idx] = acc[idx];
  }
}

// one thread per entry of [W | bias] of every pair, summing the blocks' partials in order
__global__ void __launch_bounds__(IM_THREADS) im_wreduce_kernel(ImParams p) {
  int i = blockIdx.x * IM_THREADS + threadIdx.x;
  for (int pi = 0; pi < p.P; ++pi) {
    const ImPair& q = p.pair[pi];
    const int n = q.C * q.C + q.C;
    if (i < n) {
      float* dst = i < q.C * q.C ? q.gW : q.gb;
      if (!dst) return;
      double s = 0.0;
      for (int k = 0; k < p.blocks; ++k) s += q.part_gw[(size_t)k * n + i];
      dst[i < q.C * q.C ? i : i - q.C * q.C] = (float)s;
      return;
    }
    i -= n;
  }
}

}  // namespace dfm
