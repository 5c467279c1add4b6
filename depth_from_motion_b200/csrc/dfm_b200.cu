// C-ABI implementation of include/dfm_b200.h: handles, weight repacking, and the
// per-frame launch sequence of the DfM plane-sweep cost-volume path on one H100.
#include "../../include/dfm_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <climits>
#include <cmath>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

#include "common.cuh"
#include "conv_tc.cuh"
#include "conv_tc_neck.cuh"
#include "simt_kernels.cuh"
#include "frustum_kernels.cuh"
#include "tail_kernels.cuh"
#include "logits_tc.cuh"
#include "head1x1_tc.cuh"
#include "spp_neck_kernels.cuh"
#include "fpn_kernels.cuh"
#include "resnet_kernels.cuh"
#include "resnet101_kernels.cuh"
#include "box_post_kernels.cuh"
#include "anchor_loss_kernels.cuh"
#include "depth_loss_kernels.cuh"
#include "atss_loss_kernels.cuh"
#include "imitation_loss_kernels.cuh"
#include "image_prep_kernels.cuh"
#include "view_cache_kernels.cuh"
#include "kitti_eval_kernels.cuh"
#include "waymo_eval_kernels.cuh"

namespace {

thread_local std::string g_err;
std::atomic<long long> g_launches{0}, g_tc_launches{0};

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

#define CU_TRY(expr)                                                                    \
  do {                                                                                  \
    cudaError_t e__ = (expr);                                                           \
    if (e__ != cudaSuccess)                                                             \
      return fail(DFM_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e__) +   \
                                    " (" __FILE__ ":" + std::to_string(__LINE__) + ")"); \
  } while (0)

#define DFM_TRY(expr)            \
  do {                           \
    int rc__ = (expr);           \
    if (rc__ != DFM_OK) return rc__; \
  } while (0)

#define LAUNCH_CHECK()                       \
  do {                                       \
    g_launches.fetch_add(1);                 \
    CU_TRY(cudaGetLastError());              \
  } while (0)

// ---- optional per-launch device timing (bench.py roofline) ----
struct ProfRec {
  std::string cls;
  cudaEvent_t e0, e1;
  double flops;
};
bool g_prof_on = false;
std::vector<ProfRec> g_prof;
std::vector<cudaEvent_t> g_event_pool;
cudaEvent_t prof_event() {
  if (!g_event_pool.empty()) {
    cudaEvent_t e = g_event_pool.back();
    g_event_pool.pop_back();
    return e;
  }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}
struct ProfScope {
  bool on;
  ProfRec r;
  cudaStream_t st;
  ProfScope(const std::string& cls, double flops, cudaStream_t s) : on(g_prof_on), st(s) {
    if (!on) return;
    r.cls = cls;
    r.flops = flops;
    r.e0 = prof_event();
    r.e1 = prof_event();
    cudaEventRecord(r.e0, st);
  }
  ~ProfScope() {
    if (!on) return;
    cudaEventRecord(r.e1, st);
    g_prof.push_back(r);
  }
};
double conv_flops(const dfm::ConvGeom& g) {
  const double vout = (double)g.Do * g.Ho * g.Wo;
  // a transposed stride-2 conv touches 27/8 taps per output voxel on average
  return 2.0 * vout * g.Cin * g.Cout * (g.transposed ? 27.0 / 8.0 : 27.0);
}
std::string conv_class(const char* kind, const dfm::ConvGeom& g, const char* loader) {
  return std::string(kind) + "<" + std::to_string(g.Cin) + "->" + std::to_string(g.Cout) +
         (g.transposed ? ",T" : (g.sd == 2 || g.sh == 2 || g.sw == 2) ? ",s2" : ",s1") + "," +
         loader + ">@" +
         std::to_string(g.Do) + "x" + std::to_string(g.Ho) + "x" + std::to_string(g.Wo);
}
// launches of the BEV-neck kernel (conv_tc_neck.cuh) also name the short-axis mode (s1, z2 =
// stride (1,1,2), p0 = pad (1,1,0)) and the weight-group shape (g32 / g16 input channels)
std::string neck_class(const char* kind, const dfm::ConvGeom& g, const dfm::NeckTcWeights& w) {
  const char* zm = w.zmode == dfm::NKZ_S2P1 ? "z2" : w.zmode == dfm::NKZ_S1P0 ? "p0" : "s1";
  return std::string(kind) + "<" + std::to_string(g.Cin) + "->" + std::to_string(g.Cout) + "," +
         zm + ",g" + std::to_string(w.cg) + ",src>@" + std::to_string(g.Do) + "x" +
         std::to_string(g.Ho) + "x" + std::to_string(g.Wo);
}

// Grow-only fp32 device buffer of the handles.  Its alloc returns a DFM_* code (a failure is
// DFM_ERR_CUDA with the message set), unlike DevArray::alloc / upload, which return the
// cudaError_t; upload() below is the DFM_* counterpart of DevArray::upload.
struct DevBuf : dfm::DevArray<float> {
  int alloc(size_t count) {
    CU_TRY(DevArray::alloc(count));
    return DFM_OK;
  }
};

// every handle's create: the kernels are built for sm_90a only
int require_sm90() {
  int maj = 0;
  DFM_TRY(dfm_device_info(nullptr, &maj, nullptr, nullptr));
  if (maj != 9) return fail(DFM_ERR_NOGPU, "this library is built for sm_90a only");
  return DFM_OK;
}

// The state_dict of a parameterised handle: its create registers every key once, with the
// key's element count and what to do with the host data, and its set_param is set().
struct ParamTable {
  // key -> (element count, what to do with the host data)
  std::map<std::string, std::pair<long long, std::function<int(const float*)>>> entries;
  std::set<std::string> missing;  // sorted: forward_prologue names the first
  void add(std::string key, long long numel, std::function<int(const float*)> set) {
    missing.insert(key);
    entries[std::move(key)] = {numel, std::move(set)};
  }
  // a setter's error is returned as it is and leaves the key missing
  int set(const char* family, const char* key, const float* h, long long numel) {
    if (!key || !h) return fail(DFM_ERR_INVALID, "null argument");
    const auto it = entries.find(key);
    if (it == entries.end())
      return fail(DFM_ERR_INVALID, std::string("unknown ") + family + " parameter: " + key);
    if (numel != it->second.first)
      return fail(DFM_ERR_INVALID, it->first + ": wrong element count (expected " +
                                       std::to_string(it->second.first) + ", got " +
                                       std::to_string(numel) + ")");
    DFM_TRY(it->second.second(h));
    missing.erase(it->first);
    return DFM_OK;
  }
};

// every handle's forward: refuse to run after a tensor-core kernel timed out, or with
// parameters missing (the message names the first missing key in sorted order)
int forward_prologue(const ParamTable& params) {
  if (dfm::tc_consume_error())
    return fail(DFM_ERR_CUDA, "an earlier tensor-core conv kernel timed out on an mbarrier "
                              "hand-over: its outputs were invalid");
  const std::set<std::string>& missing = params.missing;
  if (!missing.empty())
    return fail(DFM_ERR_STATE, "missing parameter: " + *missing.begin() + " (+" +
                                   std::to_string(missing.size() - 1) + " more)");
  return DFM_OK;
}

// Test hooks of the downstream handles (dfm_neck_debug_tensor, ...): copies the `written`
// floats the last forward left in `b`.  written == 0: that forward did not write the tensor.
int debug_copy(const DevBuf& b, long long written, const std::string& name, float* d_out,
               long long numel, void* stream) {
  if (written <= 0 || !b.p)
    return fail(DFM_ERR_STATE, name + " was not written by the last forward");
  if (numel != written)
    return fail(DFM_ERR_INVALID, name + ": the last forward wrote " + std::to_string(written) +
                                     " elements, not " + std::to_string(numel));
  CU_TRY(cudaMemcpyAsync(d_out, b.p, numel * sizeof(float), cudaMemcpyDeviceToDevice,
                         (cudaStream_t)stream));
  return DFM_OK;
}

// Test hooks of the loss and eval handles, once the name is known and a forward has run: copies
// the `want` elements of `elem_bytes` each at `src` into a tensor of `numel` elements, which must
// be `want` (an empty tensor copies nothing).
int copy_debug(const std::string& k, const void* src, long long want, long long numel,
               size_t elem_bytes, void* d_out, void* stream) {
  if (numel != want)
    return fail(DFM_ERR_INVALID, k + ": the tensor holds " + std::to_string(want) +
                                     " elements, not " + std::to_string(numel));
  if (want > 0)
    CU_TRY(cudaMemcpyAsync(d_out, src, (size_t)want * elem_bytes, cudaMemcpyDeviceToDevice,
                           (cudaStream_t)stream));
  return DFM_OK;
}

// The host GT offsets [B + 1] of a loss forward: they start at 0 and ascend, give each sample at
// most `per_sample` boxes and all samples at most `total`; *G is the total.  Any other offsets
// fail with `msg`.
int check_gt_offsets(const int* h_off, int B, long long per_sample, long long total,
                     const std::string& msg, int* G) {
  long long g = 0;
  for (int b = 0; b < B; ++b) {
    const long long n = (long long)h_off[b + 1] - h_off[b];
    if (h_off[b] != g || n < 0 || n > per_sample || g + n > total)
      return fail(DFM_ERR_INVALID, msg);
    g += n;
  }
  *G = (int)g;
  return DFM_OK;
}

// carves aligned sub-arrays out of one allocation (a first pass with base == nullptr sizes it)
struct BpArena {
  char* base;
  size_t off = 0;
  template <class T>
  T* take(size_t count) {
    off = (off + 255) & ~(size_t)255;
    T* r = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += count * sizeof(T);
    return r;
  }
};

struct Norm {  // GroupNorm (statistics computed per frame) or folded BatchNorm (static)
  int C = 0;
  DevBuf gamma, beta, scale, shift;
  dfm::DevArray<double> sums;
  bool sums_clean = false;  // gn_finalize_kernel left the sums zeroed and nothing touched them since
  // call before launching kernels that accumulate into `sums`
  int begin_stats(cudaStream_t st) {
    if (!sums_clean) CU_TRY(cudaMemsetAsync(sums.p, 0, 2 * C * sizeof(double), st));
    sums_clean = false;
    return DFM_OK;
  }
  int init(int c) {
    C = c;
    DFM_TRY(gamma.alloc(c));
    DFM_TRY(beta.alloc(c));
    DFM_TRY(scale.alloc(c));
    DFM_TRY(shift.alloc(c));
    CU_TRY(sums.alloc(2 * c));
    return DFM_OK;
  }
};

// eval-mode BatchNorm (weight, bias, running_mean, running_var) folded on the host into the
// static scale / shift of `n`, once all four fields have arrived
struct FoldedBn {
  Norm n;
  std::vector<float> v[4];
  bool have[4] = {false, false, false, false};
  int set(int field, const float* h) {
    v[field].assign(h, h + n.C);
    have[field] = true;
    if (!(have[0] && have[1] && have[2] && have[3])) return DFM_OK;
    const int C = n.C;
    std::vector<float> sc(C), sh(C);
    for (int c = 0; c < C; ++c) {
      const double s = (double)v[0][c] / std::sqrt((double)v[3][c] + 1e-5);
      sc[c] = (float)s;
      sh[c] = (float)((double)v[1][c] - (double)v[2][c] * s);
    }
    CU_TRY(cudaMemcpy(n.scale.p, sc.data(), C * 4, cudaMemcpyHostToDevice));
    CU_TRY(cudaMemcpy(n.shift.p, sh.data(), C * 4, cudaMemcpyHostToDevice));
    return DFM_OK;
  }
};

// registration of <prefix>.weight / .bias of a GroupNorm and of the four fields of a BatchNorm;
// both need the norm's channel count (Norm::init) first
void add_norm(ParamTable& t, const std::string& prefix, Norm& n) {
  for (DevBuf* dst : {&n.gamma, &n.beta})
    t.add(prefix + (dst == &n.gamma ? ".weight" : ".bias"), n.C, [dst, &n](const float* h) {
      CU_TRY(cudaMemcpy(dst->p, h, n.C * sizeof(float), cudaMemcpyHostToDevice));
      return DFM_OK;
    });
}

void add_bn(ParamTable& t, const std::string& prefix, FoldedBn& bn) {
  const char* const field[4] = {".weight", ".bias", ".running_mean", ".running_var"};
  for (int f = 0; f < 4; ++f)
    t.add(prefix + field[f], bn.n.C, [&bn, f](const float* h) { return bn.set(f, h); });
}

struct ConvW {
  int Cin = 0, Cout = 0, transposed = 0;
  DevBuf simt;          // [27][Cin][Cout] fp32
  dfm::TcWeights tc;    // bf16 hi/lo images for the tensor-core kernel
  dfm::NeckTcWeights ntc;  // K-outer tensor-core kernel of the BEV necks
  dfm::NeckTcWeights ntk;  // the same kernel on the plane-sweep volume (stride-1 layers with
                           // >= 64 input channels: N = 96 MMAs instead of four N = 48 splits)
};

// (Cout,Cin,3,3,3) or transposed (Cin,Cout,3,3,3)  ->  [tap][ci][co]
std::vector<float> repack_simt(const float* w, int Cin, int Cout, int transposed) {
  std::vector<float> o((size_t)27 * Cin * Cout);
  for (int co = 0; co < Cout; ++co)
    for (int ci = 0; ci < Cin; ++ci)
      for (int t = 0; t < 27; ++t) {
        const size_t src = transposed ? ((size_t)ci * Cout + co) * 27 + t
                                      : ((size_t)co * Cin + ci) * 27 + t;
        o[((size_t)t * Cin + ci) * Cout + co] = w[src];
      }
  return o;
}

int upload(DevBuf& b, const float* h, size_t n) {
  DFM_TRY(b.alloc(n));
  CU_TRY(cudaMemcpy(b.p, h, n * sizeof(float), cudaMemcpyHostToDevice));
  return DFM_OK;
}

// tc_mode: dfm::TC_S1 / TC_S2 / TC_T, or -1 for "no tensor-core kernel for this layer"
int set_conv(ConvW& cw, const float* h, long long numel, int Cin, int Cout, int transposed,
             int tc_mode) {
  if (numel != (long long)27 * Cin * Cout)
    return fail(DFM_ERR_INVALID, "conv weight has wrong element count");
  cw.Cin = Cin;
  cw.Cout = Cout;
  cw.transposed = transposed;
  const std::vector<float> p = repack_simt(h, Cin, Cout, transposed);
  DFM_TRY(upload(cw.simt, p.data(), p.size()));
  cw.tc.release();
  if (tc_mode >= 0 && dfm::tc_supported(Cin, Cout, transposed)) {
    std::string err;
    if (!cw.tc.build(p.data(), Cin, Cout, tc_mode, &err))
      return fail(DFM_ERR_CUDA, err);
  }
  cw.ntk.release();
  if (tc_mode == dfm::TC_S1 && !transposed && Cin >= 64 && Cin % 32 == 0 && Cout % 32 == 0) {
    std::string err;
    // (32-channel groups: the 16 / 64 shape holds only NK_ACC_COLS / 64 = 2 planes per window,
    // so every window would re-load two halo planes for two planes of output)
    if (!cw.ntk.build(p.data(), Cin, Cout, dfm::NKZ_S1P1, &err, /*dhw=*/true, 32))
      return fail(DFM_ERR_CUDA, err);
  }
  return DFM_OK;
}

dfm::Term term(const DevBuf& x, const Norm* nrm, int relu, int zcls = 0) {
  dfm::Term t;
  t.x = x.p;
  t.scale = nrm ? nrm->scale.p : nullptr;
  t.shift = nrm ? nrm->shift.p : nullptr;
  t.relu = relu;
  t.zcls = zcls;
  return t;
}

dfm::Src src1(dfm::Term a, int outer_relu = 0) {
  dfm::Src s{};
  s.t[0] = a;
  s.n = 1;
  s.outer_relu = outer_relu;
  return s;
}
dfm::Src src2(dfm::Term a, dfm::Term b, int outer_relu = 0) {
  dfm::Src s{};
  s.t[0] = a;
  s.t[1] = b;
  s.n = 2;
  s.outer_relu = outer_relu;
  return s;
}
dfm::Src src3(dfm::Term a, dfm::Term b, dfm::Term c) {
  dfm::Src s{};
  s.t[0] = a;
  s.t[1] = b;
  s.t[2] = c;
  s.n = 3;
  s.outer_relu = 0;
  return s;
}

dfm::ConvGeom geom_s(int Di, int Hi, int Wi, int Cin, int Cout, int sd, int sh, int sw, int pd,
                     int ph, int pw) {
  dfm::ConvGeom g{};
  g.Di = Di; g.Hi = Hi; g.Wi = Wi; g.Cin = Cin; g.Cout = Cout;
  g.sd = sd; g.sh = sh; g.sw = sw; g.pd = pd; g.ph = ph; g.pw = pw;
  g.transposed = 0;
  g.Do = (Di + 2 * pd - 3) / sd + 1;
  g.Ho = (Hi + 2 * ph - 3) / sh + 1;
  g.Wo = (Wi + 2 * pw - 3) / sw + 1;
  return g;
}
dfm::ConvGeom geom_t(int Di, int Hi, int Wi, int Cin, int Cout) {
  dfm::ConvGeom g{};
  g.Di = Di; g.Hi = Hi; g.Wi = Wi; g.Cin = Cin; g.Cout = Cout;
  g.sd = g.sh = g.sw = 2; g.pd = g.ph = g.pw = 1;
  g.transposed = 1;
  g.Do = 2 * Di; g.Ho = 2 * Hi; g.Wo = 2 * Wi;
  return g;
}

template <int CIN, int COUT, class L>
int launch_simt(const L& ld, const ConvW& w, float* out, const dfm::ConvGeom& g,
                cudaStream_t st) {
  const long long nout = (long long)g.Do * g.Ho * g.Wo;
  const long long warps = (nout + 7) / 8;
  const long long blocks = (warps + 7) / 8;
  dfm::conv3d_simt_kernel<CIN, COUT, L><<<(unsigned)blocks, 256, 0, st>>>(ld, w.simt.p, out, g);
  LAUNCH_CHECK();
  return DFM_OK;
}

template <class L>
int conv_simt_dispatch(const L& ld, const ConvW& w, float* out, const dfm::ConvGeom& g,
                       cudaStream_t st) {
#define CASE(ci, co) \
  if (g.Cin == ci && g.Cout == co) return launch_simt<ci, co, L>(ld, w, out, g, st)
  CASE(32, 32);
  CASE(64, 32);
  CASE(32, 64);
  CASE(64, 64);
  CASE(160, 64);
  CASE(128, 64);
  CASE(64, 128);
  CASE(128, 128);
  CASE(128, 256);
  CASE(256, 256);
  if constexpr (std::is_same<L, dfm::SrcLoader>::value) {
    // SPPUNetNeck's upconv_module.conv.0, rpnconv.0 and rpnconv.1 (2-D layer driver only)
    CASE(512, 64);
    CASE(512, 128);
    CASE(128, 32);
  }
#undef CASE
  return fail(DFM_ERR_INVALID, "conv3d: unsupported (Cin, Cout) = (" + std::to_string(g.Cin) +
                                   ", " + std::to_string(g.Cout) + ")");
}

int gn_finalize(Norm& n, long long V, int groups, cudaStream_t st) {
  dfm::gn_finalize_kernel<<<1, 256, 0, st>>>(n.sums.p, n.gamma.p, n.beta.p, n.C, groups,
                                           (double)V, 1e-5f, n.scale.p, n.shift.p);
  LAUNCH_CHECK();
  n.sums_clean = true;
  return DFM_OK;
}

int run_gn(const float* raw, long long V, Norm& n, int groups, cudaStream_t st) {
  DFM_TRY(n.begin_stats(st));
  const int blocks = (int)std::min<long long>(8LL * dfm::tc_sm_count(), (V * n.C + 255) / 256);
  if (n.C == 32)
    dfm::channel_stats_kernel<32><<<blocks, 256, 0, st>>>(raw, V, n.sums.p);
  else if (n.C == 64)
    dfm::channel_stats_kernel<64><<<blocks, 256, 0, st>>>(raw, V, n.sums.p);
  else
    return fail(DFM_ERR_INVALID, "GroupNorm: unsupported channel count");
  LAUNCH_CHECK();
  return gn_finalize(n, V, groups, st);
}

// conv + (optionally) the GroupNorm statistics of its raw output.  The tensor-core kernel
// accumulates the per-channel sums in its epilogue; the fp32 SIMT path runs a reduction
// pass afterwards.
// ZW: the statistics weighting of a z-shortened volume (see tower_forward); count_planes is
// the number of output planes the statistics stand for (0: g.Do)
struct ZW {
  int lo = 0, hi = 0;
  float w = 1.f;
  int count_planes = 0;
};
template <class L, class TCFN>
int run_conv_impl(const L& simt_loader, TCFN tc_fn, const char* loader_name, const ConvW& w,
                  float* out, const dfm::ConvGeom& g, int impl, Norm* gn, cudaStream_t st,
                  const ZW& zw = ZW()) {
  const long long V = (long long)(zw.count_planes ? zw.count_planes : g.Do) * g.Ho * g.Wo;
  const bool tc_ok = w.tc.ready() && dfm::tc_mode_of(g) == w.tc.mode;
  if (impl == DFM_CONV_TC && !tc_ok)
    return fail(DFM_ERR_INVALID, "conv3d: no tensor-core kernel for this layer");
  if (impl != DFM_CONV_SIMT && tc_ok) {
    std::string err;
    if (gn) DFM_TRY(gn->begin_stats(st));
    {
      // K-sliced launches carry their own tag (they also run the slice-reduce kernel), and so do
      // cluster launches that share bricks
      ProfScope ps(conv_class(w.tc.kslice ? "conv_tc_ks" : w.tc.cluster > 1 ? "conv_tc_cl" : "conv_tc",
                              g, loader_name),
                   conv_flops(g), st);
      if (!tc_fn(gn ? gn->sums.p : nullptr, &err)) return fail(DFM_ERR_CUDA, err);
    }
    g_launches.fetch_add(w.tc.kslice ? 2 : 1);  // K-slice convs run a slice-reduce kernel too
    g_tc_launches.fetch_add(1);
    return gn ? gn_finalize(*gn, V, 32, st) : DFM_OK;
  }
  {
    ProfScope ps(conv_class("conv_simt", g, loader_name), conv_flops(g), st);
    DFM_TRY(conv_simt_dispatch(simt_loader, w, out, g, st));
  }
  return gn ? run_gn(out, V, *gn, 32, st) : DFM_OK;
}

int run_conv(const dfm::Src& s, const ConvW& w, float* out, const dfm::ConvGeom& g, int impl,
             cudaStream_t st, Norm* gn = nullptr, const ZW& zw = ZW()) {
  dfm::SrcLoader ld{s, g.Cin, g.Hi, g.Wi};
  if (zw.count_planes && (impl == DFM_CONV_SIMT || !w.tc.ready()))
    return fail(DFM_ERR_INVALID, "z-shortened volumes exist only on the tensor-core path");
  // stride-1 layers with >= 64 input channels: K-outer kernel (conv_tc_neck.cuh, windowed along D)
  static const bool no_ntk = getenv("DFM_NO_NTK") != nullptr;
  if (impl != DFM_CONV_SIMT && !no_ntk && w.ntk.ready() &&
      dfm::neck_dhw_profitable(g, 1024 / w.ntk.cg) &&
      s.n <= 2 && s.t[0].zcls == 0 && (s.n < 2 || s.t[1].zcls == 0)) {
    const long long V = (long long)(zw.count_planes ? zw.count_planes : g.Do) * g.Ho * g.Wo;
    if (gn) DFM_TRY(gn->begin_stats(st));
    {
      std::string err;
      ProfScope ps(conv_class("conv_tck", g, "src"), conv_flops(g), st);
      if (!dfm::neck_tc_conv_dhw(s, w.ntk, out, g, gn ? gn->sums.p : nullptr, zw.lo, zw.hi, zw.w,
                                 st, &err))
        return fail(DFM_ERR_CUDA, err);
    }
    g_launches.fetch_add(1);
    g_tc_launches.fetch_add(1);
    return gn ? gn_finalize(*gn, V, 32, st) : DFM_OK;
  }
  return run_conv_impl(
      ld, [&](double* stats, std::string* err) {
        dfm::TcOpts o;
        o.zw_lo = zw.lo;
        o.zw_hi = zw.hi;
        o.zw = zw.w;
        return dfm::tc_conv_src(s, w.tc, out, stats, g, st, err, o);
      }, "src", w, out, g, impl, gn, st, zw);
}

int run_conv_warp(const dfm::WarpLoader& ld, const ConvW& w, float* out, const dfm::ConvGeom& g,
                  int impl, cudaStream_t st, Norm* gn = nullptr, const float* addend = nullptr) {
  if (addend && (impl == DFM_CONV_SIMT || !w.tc.ready()))
    return fail(DFM_ERR_INVALID, "the z-class addend exists only on the tensor-core path");
  return run_conv_impl(
      ld, [&](double* stats, std::string* err) {
        dfm::TcOpts o;
        o.addend = addend;
        return dfm::tc_conv_warp(ld, w.tc, out, stats, g, st, err, o);
      }, "warp", w, out, g, impl, gn, st);
}

// `batch` images of [C][HW], contiguous on both sides
int to_nhwc(const float* in, float* out, int C, long long HW, cudaStream_t st, int batch = 1) {
  const bool aligned = (reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) % 16 == 0;
  if ((C == 32 || C == 64) && HW % 4 == 0 && aligned && batch <= 65535) {
    dim3 grid((unsigned)((HW + 127) / 128), batch);
    if (C == 32)
      dfm::nchw_to_nhwc_v4_kernel<32><<<grid, 256, 0, st>>>(in, out, HW, C * HW, C * HW);
    else
      dfm::nchw_to_nhwc_v4_kernel<64><<<grid, 256, 0, st>>>(in, out, HW, C * HW, C * HW);
    LAUNCH_CHECK();
    return DFM_OK;
  }
  for (int b = 0; b < batch; ++b) {
    dim3 grid((unsigned)((HW + 31) / 32), (C + 31) / 32), block(32, 8);
    dfm::nchw_to_nhwc_kernel<<<grid, block, 0, st>>>(in + (size_t)b * C * HW,
                                                      out + (size_t)b * C * HW, C, HW);
    LAUNCH_CHECK();
  }
  return DFM_OK;
}
int to_ncdhw(const float* in, float* out, int C, long long V, cudaStream_t st) {
  dim3 grid((unsigned)((V + 31) / 32), (C + 31) / 32), block(32, 8);
  dfm::cl_to_ncdhw_kernel<<<grid, block, 0, st>>>(in, out, C, V);
  LAUNCH_CHECK();
  return DFM_OK;
}

void mat4_mul(const double* a, const double* b, double* o) {
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double s = 0;
      for (int k = 0; k < 4; ++k) s += a[i * 4 + k] * b[k * 4 + j];
      o[i * 4 + j] = s;
    }
}
bool mat4_inv(const double* m, double* inv) {
  double a[4][8];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      a[i][j] = m[i * 4 + j];
      a[i][4 + j] = i == j ? 1.0 : 0.0;
    }
  for (int c = 0; c < 4; ++c) {
    int piv = c;
    for (int r = c + 1; r < 4; ++r)
      if (std::fabs(a[r][c]) > std::fabs(a[piv][c])) piv = r;
    if (std::fabs(a[piv][c]) < 1e-300) return false;
    if (piv != c)
      for (int j = 0; j < 8; ++j) std::swap(a[piv][j], a[c][j]);
    const double d = a[c][c];
    for (int j = 0; j < 8; ++j) a[c][j] /= d;
    for (int r = 0; r < 4; ++r)
      if (r != c) {
        const double f = a[r][c];
        for (int j = 0; j < 8; ++j) a[r][j] -= f * a[c][j];
      }
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) inv[i * 4 + j] = a[i][4 + j];
  return true;
}

// M = P4 * T * P4^-1 in fp64; the reference pads cam2img[:3] into an identity 4x4
// (structures/utils.py:239-241) and re-homogenises with ones (dfm_backbone.py:267-271).
int make_warp_geom(const dfm_geometry_t* gm, int Hf, int Wf, int csf, int fsf, dfm::WarpGeom* out) {
  // unproject uses cam2img[:3] padded into an identity 4x4 (structures/utils.py:239-241);
  // the 3-D points are re-homogenised with ones before cur2prev and again before the
  // projection (dfm_backbone.py:267-271, structures/utils.py:206), i.e. the 4th row of
  // cur2prev never contributes.
  double P[16], Pi[16], T[16], tmp[16], M[16];
  for (int i = 0; i < 16; ++i) P[i] = gm->cam2img[i];
  P[12] = P[13] = P[14] = 0.0;
  P[15] = 1.0;
  for (int i = 0; i < 16; ++i) T[i] = gm->cur2prev[i];
  T[12] = T[13] = T[14] = 0.0;
  T[15] = 1.0;
  if (!mat4_inv(P, Pi)) return fail(DFM_ERR_INVALID, "ori_cam2img is singular");
  mat4_mul(T, Pi, tmp);
  mat4_mul(P, tmp, M);
  dfm::WarpGeom g{};
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) g.A[i * 3 + j] = (float)M[i * 4 + j];
    g.t[i] = (float)M[i * 4 + 3];
  }
  g.scale = (float)gm->scale;
  g.inv_scale = (float)(1.0 / gm->scale);
  g.crop_x = (float)gm->crop_x;
  g.crop_y = (float)gm->crop_y;
  g.org_w = (float)gm->org_w;
  g.lattice = (float)(fsf * csf);
  g.inv_fsf = 1.f / (float)fsf;
  g.step = csf;
  g.flip = gm->flip;
  g.Hf = Hf;
  g.Wf = Wf;
  *out = g;
  return DFM_OK;
}

}  // namespace

// =====================================================================================
// backbone handle
// =====================================================================================
struct Tower {
  ConvW dres0, dres1, c1, c2, c3, c4, c5, c6, p0;
  DevBuf p1w;  // [27][32]: conv3d_c32_to_1_kernel (SIMT path)
  dfm::LogitsTcWeights p1q;     // same as a 32 x 32 (27 taps) bf16 hi/lo image: logits_tc_kernel
  // z-invariance of the cur-frame half (SURVEY.md section 7): dres0 split into its cur- and
  // prev-channel halves (stereo); the cur contribution is computed on 5 replicated planes
  // and kept as 3 z-class planes (first / interior / last)
  ConvW d0cur, d0prev;
  DevBuf cls5, cls3;
  Norm g0, g1, gc1, gc2, gc3, gc4, gc5, gc6, gp0;
  DevBuf raw0, raw1, b1, b2, b3, b4, b5, b6, cur, p0b, logit;
  // what the last forward wrote (dfm_backbone_debug_tensor refuses the rest): the z-class
  // path keeps dres0_mono's output in cls3 only, and only that path writes cls3
  bool raw0_written = false, cls3_written = false;
};

struct dfm_backbone {
  dfm_backbone_desc_t d;
  int D, Ho, Wo;
  Tower st, mo;
  DevBuf cur_nhwc, prev_nhwc, depths, wagg, waggT, cost, volume_dbg;
  // NCHW staging of the host-buffer entry point, double-buffered so that the next pair can be
  // copied in (dfm_backbone_prefetch_host) while the current one is being processed
  struct HostStage {
    DevBuf cur, prev, sem;
    const float* h_cur = nullptr;
    const float* h_prev = nullptr;
    const float* h_sem = nullptr;  // staged with the pair by dfm_pipeline_prefetch_host
    bool pending = false;      // holds a prefetched pair that no forward has consumed yet
    cudaEvent_t ready = nullptr;
    cudaEvent_t consumed = nullptr;  // recorded after the last kernel that reads this slot
                                     // (asynchronous pipeline: a later prefetch waits for it)
    unsigned long long tick = 0;
    ~HostStage() {
      if (ready) cudaEventDestroy(ready);
      if (consumed) cudaEventDestroy(consumed);
    }
  } stage[2];
  unsigned long long stage_tick = 0;
  // grow-only device scratch of the host-buffer entry points (no cudaMalloc per call)
  DevBuf out_st, out_mo, pipe_sem, pipe_vox, pipe_preds, pipe_samples;
  std::vector<float> pipe_samples_host;  // what pipe_samples holds (re-uploaded on change only)
  bool depths_set = false;
  ParamTable params;
  struct DebugTensor {
    const DevBuf* buf;
    const bool* written;  // null: every forward writes it
  };
  std::map<std::string, DebugTensor> dbg;
};

namespace {

// cur_cost materialisation: vectorised kernel for the 32-channel case
int launch_materialize(const dfm::Src& src, int C, long long V, long long HW, dfm::ZExpand ze,
                       float* out_cl, float* out_ncdhw, const char* tag, cudaStream_t st) {
  ProfScope ps(tag, 0.0, st);
  if (C == 32 && V < (1LL << 31)) {
    const int ntiles = (int)((V + dfm::MAT_TV - 1) / dfm::MAT_TV);
    dfm::materialize32_kernel<<<std::min(ntiles, dfm::tc_sm_count() * 6), 256, 0, st>>>(
        src, (int)V, (int)HW, ze, out_cl, out_ncdhw);
  } else {
    dim3 block(32, 8), grid((unsigned)((V + 31) / 32), (C + 31) / 32);
    dfm::materialize_kernel<<<grid, block, 0, st>>>(src, C, V, HW, ze, out_cl, out_ncdhw);
  }
  LAUNCH_CHECK();
  return DFM_OK;
}

int tower_alloc(Tower& t, int D, int Ho, int Wo, int cv) {
  const size_t V = (size_t)D * Ho * Wo, V2 = V / 8, V4 = V / 64;
  DFM_TRY(t.raw0.alloc(V * cv));
  DFM_TRY(t.raw1.alloc(V * cv));
  DFM_TRY(t.b1.alloc(V2 * 2 * cv));
  DFM_TRY(t.b2.alloc(V2 * 2 * cv));
  DFM_TRY(t.b3.alloc(V4 * 2 * cv));
  DFM_TRY(t.b4.alloc(V4 * 2 * cv));
  DFM_TRY(t.b5.alloc(V2 * 2 * cv));
  DFM_TRY(t.b6.alloc(V * cv));
  DFM_TRY(t.cur.alloc(V * cv));
  DFM_TRY(t.p0b.alloc(V * cv));
  DFM_TRY(t.logit.alloc(V));
  DFM_TRY(t.cls5.alloc((size_t)5 * Ho * Wo * cv));
  DFM_TRY(t.cls3.alloc((size_t)3 * Ho * Wo * cv));
  DFM_TRY(t.g0.init(cv));
  DFM_TRY(t.g1.init(cv));
  DFM_TRY(t.gc1.init(2 * cv));
  DFM_TRY(t.gc2.init(2 * cv));
  DFM_TRY(t.gc3.init(2 * cv));
  DFM_TRY(t.gc4.init(2 * cv));
  DFM_TRY(t.gc5.init(2 * cv));
  DFM_TRY(t.gc6.init(cv));
  DFM_TRY(t.gp0.init(cv));
  return DFM_OK;
}

bool ends_with(const std::string& s, const std::string& e) {
  return s.size() >= e.size() && s.compare(s.size() - e.size(), e.size(), e) == 0;
}

// one tower's keys: dres0 / dres1, the hourglass and the pred convs (cin0: dres0's input
// channels).  The norms are initialised (tower_alloc).
void tower_add_params(ParamTable& p, Tower& t, bool mono, int cin0, int cv) {
  const std::string sfx = mono ? "_mono" : "";
  const std::string hg = mono ? "hg_mono.0" : "hg_stereo.0";
  const std::string pr = mono ? "pred_mono.0" : "pred_stereo.0";
  const long long n0 = 27LL * cin0 * cv, n1 = 27LL * cv * cv;
  p.add("dres0" + sfx + ".conv.weight", n0, [&t, mono, cin0, cv, n0](const float* h) {
    if (!mono) {  // (cv, 2C, 27): channel halves as two C -> cv convs
      const int C = cin0 / 2;
      std::vector<float> hc((size_t)cv * C * 27), hp((size_t)cv * C * 27);
      for (int co = 0; co < cv; ++co)
        for (int ci = 0; ci < C; ++ci)
          for (int k = 0; k < 27; ++k) {
            hc[((size_t)co * C + ci) * 27 + k] = h[((size_t)co * cin0 + ci) * 27 + k];
            hp[((size_t)co * C + ci) * 27 + k] = h[((size_t)co * cin0 + C + ci) * 27 + k];
          }
      DFM_TRY(set_conv(t.d0cur, hc.data(), (long long)hc.size(), C, cv, 0, dfm::TC_S1));
      DFM_TRY(set_conv(t.d0prev, hp.data(), (long long)hp.size(), C, cv, 0, dfm::TC_S1));
    }
    return set_conv(t.dres0, h, n0, cin0, cv, 0, dfm::TC_S1);
  });
  p.add("dres1" + sfx + ".conv.weight", n1,
        [&t, cv, n1](const float* h) { return set_conv(t.dres1, h, n1, cv, cv, 0, dfm::TC_S1); });
  add_norm(p, "dres0" + sfx + ".gn", t.g0);
  add_norm(p, "dres1" + sfx + ".gn", t.g1);
  struct HG { const char* key; ConvW* w; Norm* n; int ci, co, tr, mode; };
  const HG hgs[] = {{"conv1.0", &t.c1, &t.gc1, cv, 2 * cv, 0, dfm::TC_S2},
                    {"conv2", &t.c2, &t.gc2, 2 * cv, 2 * cv, 0, dfm::TC_S1},
                    {"conv3.0", &t.c3, &t.gc3, 2 * cv, 2 * cv, 0, dfm::TC_S2},
                    {"conv4.0", &t.c4, &t.gc4, 2 * cv, 2 * cv, 0, dfm::TC_S1},
                    {"conv5", &t.c5, &t.gc5, 2 * cv, 2 * cv, 1, dfm::TC_T},
                    {"conv6", &t.c6, &t.gc6, 2 * cv, cv, 1, dfm::TC_T}};
  for (const HG& e : hgs) {
    const std::string base = hg + "." + e.key;
    const long long n = 27LL * e.ci * e.co;
    p.add(base + ".0.weight", n,
          [e, n](const float* h) { return set_conv(*e.w, h, n, e.ci, e.co, e.tr, e.mode); });
    add_norm(p, base + ".1", *e.n);
  }
  p.add(pr + ".0.conv.weight", n1,
        [&t, cv, n1](const float* h) { return set_conv(t.p0, h, n1, cv, cv, 0, dfm::TC_S1); });
  add_norm(p, pr + ".0.gn", t.gp0);
  p.add(pr + ".1.weight", 27LL * cv, [&t, cv](const float* h) {
    std::vector<float> p((size_t)27 * cv);  // (1,cv,3,3,3) -> [tap][c]
    for (int c = 0; c < cv; ++c)
      for (int k = 0; k < 27; ++k) p[(size_t)k * cv + c] = h[(size_t)c * 27 + k];
    if (cv == 32 && !t.p1q.build(p.data())) return fail(DFM_ERR_CUDA, "logits weight upload failed");
    return upload(t.p1w, p.data(), p.size());
  });
}

// one tower of DfMBackbone.forward: dfm_backbone.py:175-183 / 189-197 + pred convs
//
// z-invariance (SURVEY.md section 7, "optional algorithmic shortcut", validated against the
// full computation by tests/test_gpu_parity.py): the cur-frame half of the volume is the
// same on every depth plane, so everything the MONO tower computes is 4-periodic in z (two
// stride-2 levels) on all planes whose receptive field does not reach the two z ends (zero
// padding).  Through dres0/dres1, the hourglass and the pred convs that influence reaches
// 14 planes (measured with the oracle).  The mono tower therefore runs on a shortened
// volume: kZHead head planes, kZMid (two periods) interior planes, kZHead tail planes;
// GroupNorm statistics weigh the interior planes so the sums equal those of the full
// volume, and consumers expand z on read (same phase mod 4).
constexpr int kZHead = 16, kZMid = 8;

int tower_forward(dfm_backbone* bb, Tower& t, bool mono, const dfm::WarpLoader& wl,
                  float* d_feat_out, cudaStream_t st, dfm::ZExpand* zexp_out) {
  const int Dfull = bb->D, Ho = bb->Ho, Wo = bb->Wo, cv = bb->d.cv_channels;
  const int impl = bb->d.conv_impl;
  const int cin0 = mono ? bb->d.in_channels : 2 * bb->d.in_channels;

  dfm::ConvGeom g;
  dfm::Term T0;
  const ConvW& wcur = mono ? t.dres0 : t.d0cur;
  const bool zinv = impl != DFM_CONV_SIMT && wcur.tc.ready() && (mono || t.d0prev.tc.ready());
  const bool shorten = mono && zinv && Dfull >= 2 * kZHead + 2 * kZMid &&
                       getenv("DFM_NO_ZSHORTEN") == nullptr;
  const int D = shorten ? 2 * kZHead + kZMid : Dfull;  // planes actually computed
  const long long V = (long long)D * Ho * Wo;           // computed voxels
  t.raw0_written = !(zinv && mono);
  t.cls3_written = zinv;
  dfm::ZExpand ze{Dfull, Dfull, 0, 0};                  // identity
  if (shorten) ze = dfm::ZExpand{kZHead, Dfull - kZHead, Dfull - D, kZHead};
  if (zexp_out) *zexp_out = ze;
  // statistics weighting per resolution level (scale 1, 2, 4): interior planes
  // [head/s, (head+mid)/s) each stand for (Dfull - 2 head) / mid planes
  auto zw_at = [&](int scale) {
    ZW z;
    if (shorten) {
      z.lo = kZHead / scale;
      z.hi = (kZHead + kZMid) / scale;
      z.w = (float)(Dfull - 2 * kZHead) / (float)kZMid;
      z.count_planes = Dfull / scale;
    }
    return z;
  };

  // ---- first layer: dres0 on the on-the-fly plane-sweep volume --------------------------
  if (zinv) {
    // The cur-frame half of the volume is the same on every plane, so its conv response is
    // too, except on the first and last plane (zero padding in z).  Five replicated planes
    // give the three variants as output planes 0 / 2 / 4.
    const int C = bb->d.in_channels;
    dfm::WarpLoader wc = wl;
    wc.first = 0;
    g = geom_s(5, Ho, Wo, C, cv, 1, 1, 1, 1, 1, 1);
    DFM_TRY(run_conv_warp(wc, wcur, t.cls5.p, g, impl, st));
    const long long pe = (long long)Ho * Wo * cv;
    dfm::pick_planes_kernel<<<dim3((unsigned)((pe / 4 + 255) / 256), 3), 256, 0, st>>>(
        t.cls5.p, t.cls3.p, pe);   // pe = Ho * Wo * 32: a multiple of 4
    LAUNCH_CHECK();
    if (mono) {
      // dres0_mono's whole output is z-class compressed; its GroupNorm statistics weigh the
      // three planes 1 : Dfull-2 : 1
      DFM_TRY(t.g0.begin_stats(st));
      dfm::channel_stats_zcls_kernel<32><<<dim3(296, 3), 256, 0, st>>>(t.cls3.p, Ho * Wo, Dfull,
                                                                    t.g0.sums.p);
      LAUNCH_CHECK();
      DFM_TRY(gn_finalize(t.g0, (long long)Dfull * Ho * Wo, 32, st));
      T0 = term(t.cls3, &t.g0, 1, D);  // first / interior / last plane of the computed volume
    } else {
      // stereo: prev-frame half on the tensor cores, cur-frame response added per z class
      dfm::WarpLoader wp = wl;
      wp.first = C;
      g = geom_s(D, Ho, Wo, C, cv, 1, 1, 1, 1, 1, 1);
      DFM_TRY(run_conv_warp(wp, t.d0prev, t.raw0.p, g, impl, st, &t.g0, t.cls3.p));
      T0 = term(t.raw0, &t.g0, 1);
    }
  } else {
    g = geom_s(D, Ho, Wo, cin0, cv, 1, 1, 1, 1, 1, 1);
    DFM_TRY(run_conv_warp(wl, t.dres0, t.raw0.p, g, impl, st, &t.g0));
    T0 = term(t.raw0, &t.g0, 1);
  }
  // dres1 (GN, no act) on relu(gn(raw0))
  g = geom_s(D, Ho, Wo, cv, cv, 1, 1, 1, 1, 1, 1);
  DFM_TRY(run_conv(src1(T0), t.dres1, t.raw1.p, g, impl, st, &t.g1, zw_at(1)));
  // cost0 = gn1(raw1) + relu(gn0(raw0)) is never stored: consumers re-evaluate it
  const dfm::Term T1 = term(t.raw1, &t.g1, 0);
  // hourglass (conv_modules.py:129-149)
  // conv1 runs as a cluster of two output-channel groups that share every input brick, conv3 as
  // input-channel slices (conv_tc.cuh, TcWeights::build)
  g = geom_s(D, Ho, Wo, cv, 2 * cv, 2, 2, 2, 1, 1, 1);
  DFM_TRY(run_conv(src2(T1, T0), t.c1, t.b1.p, g, impl, st, &t.gc1, zw_at(2)));
  const int D2 = g.Do, H2 = g.Ho, W2 = g.Wo;
  g = geom_s(D2, H2, W2, 2 * cv, 2 * cv, 1, 1, 1, 1, 1, 1);
  DFM_TRY(run_conv(src1(term(t.b1, &t.gc1, 1)), t.c2, t.b2.p, g, impl, st, &t.gc2, zw_at(2)));
  g = geom_s(D2, H2, W2, 2 * cv, 2 * cv, 2, 2, 2, 1, 1, 1);
  DFM_TRY(run_conv(src1(term(t.b2, &t.gc2, 1)), t.c3, t.b3.p, g, impl, st, &t.gc3, zw_at(4)));
  const int D4 = g.Do, H4 = g.Ho, W4 = g.Wo;
  g = geom_s(D4, H4, W4, 2 * cv, 2 * cv, 1, 1, 1, 1, 1, 1);
  DFM_TRY(run_conv(src1(term(t.b3, &t.gc3, 1)), t.c4, t.b4.p, g, impl, st, &t.gc4, zw_at(4)));
  g = geom_t(D4, H4, W4, 2 * cv, 2 * cv);
  DFM_TRY(run_conv(src1(term(t.b4, &t.gc4, 1)), t.c5, t.b5.p, g, impl, st, &t.gc5, zw_at(2)));
  // post = relu(gn5(conv5) + pre),  pre = relu(gn2(conv2))
  g = geom_t(D2, H2, W2, 2 * cv, cv);
  DFM_TRY(run_conv(src2(term(t.b5, &t.gc5, 0), term(t.b2, &t.gc2, 1), 1), t.c6, t.b6.p, g, impl,
                   st, &t.gc6, zw_at(1)));
  // cur_cost = cost0 + gn6(conv6): a channels-last copy feeds the pred conv (a one-term load
  // keeps that conv MMA-bound; the three-term load made it loader-bound), the NCDHW copy
  // (z-expanded for the shortened mono tower) is the output the caller asked for
  const dfm::Src cur_src = src3(T1, T0, term(t.b6, &t.gc6, 0));
  {
    const dfm::ZExpand ident{D, D, 0, 0};
    const bool one_pass = !shorten;  // same iteration space for both copies
    DFM_TRY(launch_materialize(cur_src, cv, V, (long long)Ho * Wo, ident, t.cur.p,
                               one_pass ? d_feat_out : nullptr, "materialize", st));
    // the z-expanded NCDHW copy re-reads every stored plane up to 20 times: read the one-term
    // channels-last copy just written instead of summing the three terms again
    if (!one_pass && d_feat_out)
      DFM_TRY(launch_materialize(src1(term(t.cur, nullptr, 0)), cv, (long long)Dfull * Ho * Wo,
                                 (long long)Ho * Wo, ze, nullptr, d_feat_out,
                                 "materialize_expand", st));
  }
  // depth prediction module (dfm_backbone.py:118-128)
  g = geom_s(D, Ho, Wo, cv, cv, 1, 1, 1, 1, 1, 1);
  DFM_TRY(run_conv(src1(term(t.cur, nullptr, 0)), t.p0, t.p0b.p, g, impl, st, &t.gp0, zw_at(1)));
  // 32 -> 1 logits conv (dfm_backbone.py:128), HBM-bound: logits_tc_kernel (logits_tc.cuh)
  // computes the 27 per-tap dot products of every input position as one small wgmma GEMM and
  // the stencil as a shared-memory gather; the fp32 SIMT path keeps its own kernel.
  const dfm::Src lsrc = src1(term(t.p0b, &t.gp0, 1));
  if (impl != DFM_CONV_SIMT) {
    if (!t.p1q.ready()) return fail(DFM_ERR_STATE, "logits weights not uploaded");
    ProfScope ps(conv_class("cout1_logits_tc", g, "src"), 2.0 * V * cv * 27, st);
    if (!dfm::logits_tc_launch(lsrc, t.p1q, t.logit.p, D, Ho, Wo, st))
      return fail(DFM_ERR_CUDA, "logits_tc_kernel launch failed");
    g_launches.fetch_add(1);
    g_tc_launches.fetch_add(1);
  } else {
    const long long threads = V * 8;
    ProfScope ps(conv_class("conv_simt_cout1", g, "src"), 2.0 * V * cv * 27, st);
    dfm::conv3d_c32_to_1_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(
        lsrc, t.p1w.p, t.logit.p, D, Ho, Wo);
    LAUNCH_CHECK();
  }
  return DFM_OK;
}

}  // namespace

extern "C" {

const char* dfm_last_error(void) { return g_err.c_str(); }
int dfm_version(void) { return 100; }

int dfm_device_info(int* sm_count, int* cc_major, int* cc_minor, long long* l2_bytes) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    return fail(DFM_ERR_NOGPU, "no CUDA device visible");
  }
  int dev = 0;
  CU_TRY(cudaGetDevice(&dev));
  cudaDeviceProp p;
  CU_TRY(cudaGetDeviceProperties(&p, dev));
  if (sm_count) *sm_count = p.multiProcessorCount;
  if (cc_major) *cc_major = p.major;
  if (cc_minor) *cc_minor = p.minor;
  if (l2_bytes) *l2_bytes = p.l2CacheSize;
  return DFM_OK;
}

int dfm_sync_check(void* stream) {
  CU_TRY(cudaStreamSynchronize((cudaStream_t)stream));
  CU_TRY(cudaGetLastError());
  if (dfm::tc_consume_error())
    return fail(DFM_ERR_CUDA, "tensor-core conv kernel: mbarrier hand-over timed out");
  return DFM_OK;
}

int dfm_profile_enable(int on) {
  g_prof_on = on != 0;
  return DFM_OK;
}

int dfm_profile_report(char* buf, int cap) {
  if (!buf || cap < 3) return fail(DFM_ERR_INVALID, "null/short buffer");
  CU_TRY(cudaDeviceSynchronize());
  std::map<std::string, std::pair<long long, std::pair<double, double>>> agg;
  for (ProfRec& r : g_prof) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, r.e0, r.e1);
    auto& a = agg[r.cls];
    a.first += 1;
    a.second.first += ms;
    a.second.second += r.flops;
    g_event_pool.push_back(r.e0);
    g_event_pool.push_back(r.e1);
  }
  g_prof.clear();
  std::string js = "{";
  bool first = true;
  for (auto& kv : agg) {
    char tmp[512];
    snprintf(tmp, sizeof tmp, "%s\"%s\": {\"launches\": %lld, \"ms\": %.6f, \"flops\": %.6e}",
             first ? "" : ", ", kv.first.c_str(), kv.second.first, kv.second.second.first,
             kv.second.second.second);
    js += tmp;
    first = false;
  }
  js += "}";
  strncpy(buf, js.c_str(), cap - 1);
  buf[cap - 1] = 0;
  return DFM_OK;
}

int dfm_launch_counters(long long* launches, long long* tc_launches) {
  if (launches) *launches = g_launches.load();
  if (tc_launches) *tc_launches = g_tc_launches.load();
  return DFM_OK;
}

int dfm_backbone_create(const dfm_backbone_desc_t* desc, dfm_backbone_t** out) {
  if (!desc || !out) return fail(DFM_ERR_INVALID, "null argument");
  if (desc->in_channels != 32 || desc->cv_channels != 32)
    return fail(DFM_ERR_INVALID, "only in_channels == cv_channels == 32 is implemented");
  const int csf = desc->cost_sample_factor, fsf = desc->feat_sample_factor;
  if (csf < 1 || fsf < 1) return fail(DFM_ERR_INVALID, "sample factors must be >= 1");
  // Python's round() (dfm_backbone.py:243-244) rounds halves to even: std::nearbyint in the
  // default rounding mode, not std::lround (half away from zero)
  const int Ho = (int)std::nearbyint((double)desc->feat_h / csf);
  const int Wo = (int)std::nearbyint((double)desc->feat_w / csf);
  const int D = desc->num_planes;
  if (D % 4 || Ho % 4 || Wo % 4 || D < 4 || Ho < 4 || Wo < 4)
    return fail(DFM_ERR_INVALID,
                "D, H/4 and W/4 must be positive multiples of 4 (the reference hourglass "
                "adds conv5 output to conv2 output, conv_modules.py:145)");
  if ((Ho - 1) * csf > desc->feat_h - 1 || (Wo - 1) * csf > desc->feat_w - 1)
    return fail(DFM_ERR_INVALID, "feature size not compatible with cost_sample_factor");
  DFM_TRY(require_sm90());
  std::unique_ptr<dfm_backbone> bb(new dfm_backbone());
  bb->d = *desc;
  bb->D = D;
  bb->Ho = Ho;
  bb->Wo = Wo;
  const size_t HW = (size_t)desc->feat_h * desc->feat_w;
  DFM_TRY(bb->cur_nhwc.alloc(HW * desc->in_channels));
  DFM_TRY(bb->prev_nhwc.alloc(HW * desc->in_channels));
  DFM_TRY(bb->depths.alloc(D));
  DFM_TRY(bb->wagg.alloc((size_t)D * 2 * D));
  DFM_TRY(bb->cost.alloc((size_t)D * Ho * Wo));
  DFM_TRY(tower_alloc(bb->st, D, Ho, Wo, desc->cv_channels));
  DFM_TRY(tower_alloc(bb->mo, D, Ho, Wo, desc->cv_channels));
  tower_add_params(bb->params, bb->st, false, 2 * desc->in_channels, desc->cv_channels);
  tower_add_params(bb->params, bb->mo, true, desc->in_channels, desc->cv_channels);
  dfm_backbone* b = bb.get();
  bb->params.add("aggregate_cost.weight", (long long)D * 2 * D, [b, D](const float* h) {
    CU_TRY(cudaMemcpy(b->wagg.p, h, (size_t)D * 2 * D * sizeof(float), cudaMemcpyHostToDevice));
    // transposed, padded copy [2D][gate_row_pitch(D)] for the persistent gate kernel
    const int pitch = dfm::gate_row_pitch(D);
    std::vector<float> wt((size_t)2 * D * pitch, 0.f);
    for (int d = 0; d < D; ++d)
      for (int j = 0; j < 2 * D; ++j) wt[(size_t)j * pitch + d] = h[(size_t)d * 2 * D + j];
    return upload(b->waggT, wt.data(), wt.size());
  });
  for (int m = 0; m < 2; ++m) {
    Tower& t = m ? bb->mo : bb->st;
    const std::string s = m ? "_mono" : "";
    bb->dbg["raw0" + s] = {&t.raw0, &t.raw0_written};
    bb->dbg["cls3" + s] = {&t.cls3, &t.cls3_written};
    bb->dbg["raw1" + s] = {&t.raw1, nullptr};
    bb->dbg["c1" + s] = {&t.b1, nullptr};
    bb->dbg["c2" + s] = {&t.b2, nullptr};
    bb->dbg["c3" + s] = {&t.b3, nullptr};
    bb->dbg["c4" + s] = {&t.b4, nullptr};
    bb->dbg["c5" + s] = {&t.b5, nullptr};
    bb->dbg["c6" + s] = {&t.b6, nullptr};
    bb->dbg["cur" + s] = {&t.cur, nullptr};
    bb->dbg["p0" + s] = {&t.p0b, nullptr};
    bb->dbg["logit" + s] = {&t.logit, nullptr};
  }
  *out = bb.release();
  return DFM_OK;
}

void pipeline_forget(const dfm_backbone* bb);  // pipeline_api.inc
int dfm_backbone_destroy(dfm_backbone_t* bb) {
  if (!bb) return DFM_OK;
  pipeline_forget(bb);
  delete bb;
  return DFM_OK;
}

int dfm_backbone_set_param(dfm_backbone_t* bb, const char* name, const float* h_data,
                           long long numel) {
  return bb ? bb->params.set("DfMBackbone", name, h_data, numel)
            : fail(DFM_ERR_INVALID, "null argument");
}

int dfm_backbone_set_depths(dfm_backbone_t* bb, const float* h_depths, int n) {
  if (!bb || !h_depths) return fail(DFM_ERR_INVALID, "null argument");
  if (n != bb->D) return fail(DFM_ERR_INVALID, "downsampled_depth must have D entries");
  CU_TRY(cudaMemcpy(bb->depths.p, h_depths, n * sizeof(float), cudaMemcpyHostToDevice));
  bb->depths_set = true;
  return DFM_OK;
}

int dfm_backbone_missing_params(const dfm_backbone_t* bb) {
  return bb ? (int)bb->params.missing.size() : -1;
}

long long dfm_backbone_workspace_bytes(const dfm_backbone_t* bb) {
  if (!bb) return 0;
  long long n = 0;
  for (const Tower* t : {&bb->st, &bb->mo})
    for (const DevBuf* b : {&t->raw0, &t->raw1, &t->b1, &t->b2, &t->b3, &t->b4, &t->b5, &t->b6,
                            &t->cur, &t->p0b, &t->logit})
      n += (long long)b->n * 4;
  n += (long long)(bb->cur_nhwc.n + bb->prev_nhwc.n + bb->cost.n) * 4;
  return n;
}

}  // extern "C"

namespace {
// prev_ready: optional event after which d_prev may be read (host-buffer entry point: the
// prev-frame H2D copy runs on a second stream underneath the mono tower, which needs only
// the cur-frame features)
int backbone_forward_impl(dfm_backbone_t* bb, const float* d_cur, const float* d_prev,
                          const dfm_geometry_t* geom, float* d_cost, float* d_stereo,
                          float* d_mono, void* stream, cudaEvent_t prev_ready,
                          bool channels_last = false) {
  if (!bb || !d_cur || !d_prev || !geom) return fail(DFM_ERR_INVALID, "null argument");
  DFM_TRY(forward_prologue(bb->params));
  if (!bb->depths_set) return fail(DFM_ERR_STATE, "downsampled_depth not set");
  cudaStream_t st = (cudaStream_t)stream;
  ProfScope ps_all("backbone_forward_total", 0.0, st);
  const int C = bb->d.in_channels;
  const long long HW = (long long)bb->d.feat_h * bb->d.feat_w;
  if (!channels_last) {
    ProfScope ps("nchw_to_nhwc_cur", 0.0, st);
    DFM_TRY(to_nhwc(d_cur, bb->cur_nhwc.p, C, HW, st));
  }
  dfm::WarpLoader wl{};
  wl.cur = channels_last ? d_cur : bb->cur_nhwc.p;
  wl.prev = channels_last ? d_prev : bb->prev_nhwc.p;
  wl.depths = bb->depths.p;
  wl.C = C;
  wl.first = 0;
  DFM_TRY(make_warp_geom(geom, bb->d.feat_h, bb->d.feat_w, bb->d.cost_sample_factor,
                         bb->d.feat_sample_factor, &wl.g));
  dfm::ZExpand ze_mono{bb->D, bb->D, 0, 0};
  DFM_TRY(tower_forward(bb, bb->mo, true, wl, d_mono, st, &ze_mono));
  if (prev_ready) CU_TRY(cudaStreamWaitEvent(st, prev_ready, 0));
  if (!channels_last) {
    ProfScope ps("nchw_to_nhwc_prev", 0.0, st);
    DFM_TRY(to_nhwc(d_prev, bb->prev_nhwc.p, C, HW, st));
  }
  DFM_TRY(tower_forward(bb, bb->st, false, wl, d_stereo, st, nullptr));
  // mono/stereo gate (dfm_backbone.py:130-141)
  const int HWo = bb->Ho * bb->Wo;
  const size_t gsm = dfm::gate_smem_bytes(bb->D);
  const size_t gsm4 = dfm::gate4_smem_bytes(bb->D);
  if (bb->D <= 256 && HWo % 4 == 0 && gsm4 <= 220 * 1024) {
    // 4 pixels x 16 planes per thread, weights resident in shared memory, persistent blocks
    size_t& attr_sz = dfm::per_device<size_t, 11>();
    if (attr_sz < gsm4) {
      CU_TRY(cudaFuncSetAttribute(dfm::gate_tile4_kernel,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gsm4));
      attr_sz = gsm4;
    }
    const int ng = (bb->D + dfm::GT_PG - 1) / dfm::GT_PG;
    const int ntiles = (HWo + dfm::GT4_TP - 1) / dfm::GT4_TP;
    // equal rounds per block: e.g. 234 tiles on 132 SMs -> 117 blocks x 2 rather than 132 blocks with 102 doing 2
    const int sms = dfm::tc_sm_count();
    const int rounds = (ntiles + sms - 1) / sms;
    const int grid = (ntiles + rounds - 1) / rounds;
    ProfScope ps("gate_tile4", 0.0, st);
    dfm::gate_tile4_kernel<<<grid, 32 * ng, gsm4, st>>>(bb->st.logit.p, bb->mo.logit.p,
                                                       bb->waggT.p, bb->cost.p, bb->D, HWo,
                                                       ze_mono);
  } else if (bb->D <= 256 && gsm <= 200 * 1024) {
    // weights resident in shared memory, one persistent block per SM
    bool& attr_done = dfm::per_device<bool, 8>();
    size_t& attr_sz = dfm::per_device<size_t, 9>();
    if (!attr_done || attr_sz < gsm) {
      CU_TRY(cudaFuncSetAttribute(dfm::gate_persistent_kernel,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gsm));
      attr_done = true;
      attr_sz = gsm;
    }
    const int ng = (bb->D + dfm::GT_PG - 1) / dfm::GT_PG;
    const int nh = dfm::gate_halves(bb->D);
    const int grid = std::min((HWo + 32 * nh - 1) / (32 * nh), dfm::tc_sm_count());
    ProfScope ps("gate_persistent", 0.0, st);
    dfm::gate_persistent_kernel<<<grid, 32 * ng * nh, gsm, st>>>(bb->st.logit.p, bb->mo.logit.p,
                                                            bb->waggT.p, bb->cost.p, bb->D, HWo,
                                                            ze_mono);
  } else {
    const size_t smem = (size_t)2 * bb->D * 32 * sizeof(float);
    if (smem > 48 * 1024)
      CU_TRY(cudaFuncSetAttribute(dfm::gate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)smem));
    ProfScope ps("gate_v1", 0.0, st);
    dfm::gate_kernel<<<(HWo + 31) / 32, 128, smem, st>>>(bb->st.logit.p, bb->mo.logit.p,
                                                         bb->wagg.p, bb->cost.p, bb->D, HWo, ze_mono);
  }
  LAUNCH_CHECK();
  if (d_cost)
    CU_TRY(cudaMemcpyAsync(d_cost, bb->cost.p, (size_t)bb->D * HWo * sizeof(float),
                           cudaMemcpyDeviceToDevice, st));
  return DFM_OK;
}
}  // namespace

namespace {
// DepthHead.forward kernel selection: four x pixels per thread (16-byte stores) whenever the
// output width allows it, else the one-pixel-per-thread kernel (profiled as tag + "_px1")
int launch_depth_head(const float* d_cost, const float* d_samples, int D, int Ho, int Wo,
                      int factor, float* d_volume, float* d_softmax, float* d_preds,
                      float2* d_norm, const char* tag, cudaStream_t st) {
  const size_t sm4 = dfm::dh4_smem_bytes(D, factor);
  const bool four = (Wo * factor) % 4 == 0 && sm4 <= 160 * 1024;
  ProfScope ps(four ? std::string(tag) : std::string(tag) + "_px1", 0.0, st);
  if (four) {
    size_t& attr_sz = dfm::per_device<size_t, 10>();
    if (attr_sz < sm4) {
      CU_TRY(cudaFuncSetAttribute(dfm::depth_head4_kernel,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm4));
      attr_sz = sm4;
    }
    dim3 grid((Wo * factor + dfm::DH4_PX - 1) / dfm::DH4_PX, Ho * factor), block(32, dfm::DH4_ZS);
    dfm::depth_head4_kernel<<<grid, block, sm4, st>>>(d_cost, d_samples, D, Ho, Wo, factor,
                                                      d_volume, d_softmax, d_preds, d_norm);
  } else {
    if (dfm::dh_smem_bytes(D, factor) > 32768)
      return fail(DFM_ERR_INVALID, "DepthHead: too many depth planes for the staged columns");
    dim3 grid((Wo * factor + 31) / 32, Ho * factor), block(32, dfm::DH_ZS);
    dfm::depth_head_kernel<<<grid, block, dfm::dh_smem_bytes(D, factor), st>>>(
        d_cost, d_samples, D, Ho, Wo, factor, d_volume, d_softmax, d_preds, d_norm);
  }
  LAUNCH_CHECK();
  return DFM_OK;
}
}  // namespace

extern "C" {

int dfm_backbone_forward(dfm_backbone_t* bb, const float* d_cur, const float* d_prev,
                         const dfm_geometry_t* geom, float* d_cost, float* d_stereo,
                         float* d_mono, void* stream) {
  return backbone_forward_impl(bb, d_cur, d_prev, geom, d_cost, d_stereo, d_mono, stream, nullptr);
}

int dfm_backbone_forward_cl(dfm_backbone_t* bb, const float* d_cur_cl, const float* d_prev_cl,
                            const dfm_geometry_t* geom, float* d_cost, float* d_stereo,
                            float* d_mono, void* stream) {
  return backbone_forward_impl(bb, d_cur_cl, d_prev_cl, geom, d_cost, d_stereo, d_mono, stream,
                               nullptr, true);
}

const float* dfm_backbone_cost_device(const dfm_backbone_t* bb) { return bb ? bb->cost.p : nullptr; }
const float* dfm_backbone_stereo_feat_device(const dfm_backbone_t* bb) {
  return bb ? bb->st.cur.p : nullptr;
}

}  // extern "C"

namespace {
// side stream + fork event of the host-buffer entry points (the library is not re-entrant)
struct HostCopyCtx {
  cudaStream_t stream = nullptr;
  cudaEvent_t fork = nullptr, prev_done = nullptr;
};
int host_copy_ctx(HostCopyCtx** out) {
  HostCopyCtx& ctx = dfm::per_device<HostCopyCtx>();
  if (!ctx.stream) {
    CU_TRY(cudaStreamCreateWithFlags(&ctx.stream, cudaStreamNonBlocking));
    CU_TRY(cudaEventCreateWithFlags(&ctx.fork, cudaEventDisableTiming));
    CU_TRY(cudaEventCreateWithFlags(&ctx.prev_done, cudaEventDisableTiming));
  }
  *out = &ctx;
  return DFM_OK;
}
int stage_alloc(dfm_backbone::HostStage& hs, size_t nfeat) {
  DFM_TRY(hs.cur.alloc(nfeat));
  DFM_TRY(hs.prev.alloc(nfeat));
  if (!hs.ready) CU_TRY(cudaEventCreateWithFlags(&hs.ready, cudaEventDisableTiming));
  if (!hs.consumed) CU_TRY(cudaEventCreateWithFlags(&hs.consumed, cudaEventDisableTiming));
  return DFM_OK;
}
}  // namespace

namespace {
// Device copies of a host (cur, prev) pair: the staged copy of a matching
// dfm_backbone_prefetch_host, else a fresh copy whose prev half rides the side stream
// underneath the mono tower (*prev_ready is the event to wait for before reading d_prev).
int stage_host_pair(dfm_backbone_t* bb, const float* h_cur, const float* h_prev, cudaStream_t st,
                    float** d_cur_out, float** d_prev_out, cudaEvent_t* prev_ready,
                    int* slot_out = nullptr) {
  const size_t nfeat = (size_t)bb->d.in_channels * bb->d.feat_h * bb->d.feat_w;
  HostCopyCtx* cx = nullptr;
  DFM_TRY(host_copy_ctx(&cx));
  *prev_ready = nullptr;
  float* d_cur = nullptr;
  float* d_prev = nullptr;
  int hit = -1;
  for (int i = 0; i < 2; ++i)
    if (bb->stage[i].pending && bb->stage[i].h_cur == h_cur && bb->stage[i].h_prev == h_prev)
      hit = i;
  if (hit >= 0) {
    // the pair was prefetched: both maps are (being) copied on the side stream
    dfm_backbone::HostStage& hs = bb->stage[hit];
    hs.pending = false;
    d_cur = hs.cur.p;
    d_prev = hs.prev.p;
    CU_TRY(cudaStreamWaitEvent(st, hs.ready, 0));
    if (slot_out) *slot_out = hit;
  } else {
    const int slot = !bb->stage[0].pending ? 0 : !bb->stage[1].pending ? 1
                     : (bb->stage[0].tick <= bb->stage[1].tick ? 0 : 1);
    dfm_backbone::HostStage& hs = bb->stage[slot];
    hs.pending = false;
    DFM_TRY(stage_alloc(hs, nfeat));
    d_cur = hs.cur.p;
    d_prev = hs.prev.p;
    // the prev-frame copy rides the side stream underneath the mono tower
    CU_TRY(cudaEventRecord(cx->fork, st));  // staging buffers are free once prior work is done
    CU_TRY(cudaStreamWaitEvent(cx->stream, cx->fork, 0));
    CU_TRY(cudaMemcpyAsync(d_cur, h_cur, nfeat * 4, cudaMemcpyHostToDevice, st));
    CU_TRY(cudaMemcpyAsync(d_prev, h_prev, nfeat * 4, cudaMemcpyHostToDevice, cx->stream));
    CU_TRY(cudaEventRecord(cx->prev_done, cx->stream));
    *prev_ready = cx->prev_done;
    if (slot_out) *slot_out = slot;
  }
  *d_cur_out = d_cur;
  *d_prev_out = d_prev;
  return DFM_OK;
}

int prefetch_impl(dfm_backbone_t* bb, const float* h_cur, const float* h_prev, const float* h_sem,
                  size_t nsem) {
  HostCopyCtx* cx = nullptr;
  DFM_TRY(host_copy_ctx(&cx));
  const size_t nfeat = (size_t)bb->d.in_channels * bb->d.feat_h * bb->d.feat_w;
  // a slot that holds no unconsumed pair, else the older of the two (its pair is dropped)
  int slot = !bb->stage[0].pending ? 0 : !bb->stage[1].pending ? 1
             : (bb->stage[0].tick <= bb->stage[1].tick ? 0 : 1);
  dfm_backbone::HostStage& hs = bb->stage[slot];
  DFM_TRY(stage_alloc(hs, nfeat));
  if (h_sem && nsem) DFM_TRY(hs.sem.alloc(nsem));
  // the synchronous entry points return after the device is done with this slot; the
  // asynchronous pipeline records `consumed` after the last kernel that reads it
  CU_TRY(cudaStreamWaitEvent(cx->stream, hs.consumed, 0));
  CU_TRY(cudaMemcpyAsync(hs.cur.p, h_cur, nfeat * 4, cudaMemcpyHostToDevice, cx->stream));
  CU_TRY(cudaMemcpyAsync(hs.prev.p, h_prev, nfeat * 4, cudaMemcpyHostToDevice, cx->stream));
  if (h_sem && nsem)
    CU_TRY(cudaMemcpyAsync(hs.sem.p, h_sem, nsem * 4, cudaMemcpyHostToDevice, cx->stream));
  CU_TRY(cudaEventRecord(hs.ready, cx->stream));
  hs.h_cur = h_cur;
  hs.h_prev = h_prev;
  hs.h_sem = (h_sem && nsem) ? h_sem : nullptr;
  hs.pending = true;
  hs.tick = ++bb->stage_tick;
  return DFM_OK;
}
}  // namespace

extern "C" {

int dfm_backbone_prefetch_host(dfm_backbone_t* bb, const float* h_cur, const float* h_prev) {
  if (!bb || !h_cur || !h_prev) return fail(DFM_ERR_INVALID, "null argument");
  return prefetch_impl(bb, h_cur, h_prev, nullptr, 0);
}

int dfm_backbone_forward_host(dfm_backbone_t* bb, const float* h_cur, const float* h_prev,
                              const dfm_geometry_t* geom, int out_flags, float* h_cost,
                              float* h_stereo, float* h_mono, void* stream) {
  if (!bb || !h_cur || !h_prev) return fail(DFM_ERR_INVALID, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t nfeat = (size_t)bb->d.in_channels * bb->d.feat_h * bb->d.feat_w;
  const size_t V = (size_t)bb->D * bb->Ho * bb->Wo;
  cudaEvent_t prev_ready = nullptr;
  float* d_cur = nullptr;
  float* d_prev = nullptr;
  DFM_TRY(stage_host_pair(bb, h_cur, h_prev, st, &d_cur, &d_prev, &prev_ready));
  float* d_st = nullptr;
  float* d_mo = nullptr;
  if ((out_flags & DFM_OUT_STEREO) && h_stereo) {
    DFM_TRY(bb->out_st.alloc(V * 32));
    d_st = bb->out_st.p;
  }
  if ((out_flags & DFM_OUT_MONO) && h_mono) {
    DFM_TRY(bb->out_mo.alloc(V * 32));
    d_mo = bb->out_mo.p;
  }
  int rc = backbone_forward_impl(bb, d_cur, d_prev, geom, nullptr, d_st, d_mo, stream, prev_ready);
  if (rc == DFM_OK && (out_flags & DFM_OUT_COST) && h_cost)
    if (cudaMemcpyAsync(h_cost, bb->cost.p, V * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess)
      rc = fail(DFM_ERR_CUDA, "D2H copy of cost failed");
  if (rc == DFM_OK && d_st)
    if (cudaMemcpyAsync(h_stereo, d_st, V * 32 * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess)
      rc = fail(DFM_ERR_CUDA, "D2H copy of stereo feature failed");
  if (rc == DFM_OK && d_mo)
    if (cudaMemcpyAsync(h_mono, d_mo, V * 32 * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess)
      rc = fail(DFM_ERR_CUDA, "D2H copy of mono feature failed");
  cudaError_t e = cudaStreamSynchronize(st);
  if (rc == DFM_OK && e != cudaSuccess) rc = fail(DFM_ERR_CUDA, cudaGetErrorString(e));
  if (rc == DFM_OK && dfm::tc_consume_error())
    rc = fail(DFM_ERR_CUDA, "tensor-core conv kernel: mbarrier hand-over timed out");
  return rc;
}

int dfm_backbone_debug_tensor(dfm_backbone_t* bb, const char* name, float* d_out,
                              long long numel, void* stream) {
  if (!bb || !name || !d_out) return fail(DFM_ERR_INVALID, "null argument");
  auto it = bb->dbg.find(name);
  if (it == bb->dbg.end()) return fail(DFM_ERR_INVALID, std::string("unknown tensor ") + name);
  const DevBuf* b = it->second.buf;
  if (it->second.written && !*it->second.written)
    return fail(DFM_ERR_STATE, std::string(name) + " was not written by the last forward");
  if ((size_t)numel > b->n) return fail(DFM_ERR_INVALID, "numel larger than the tensor");
  CU_TRY(cudaMemcpyAsync(d_out, b->p, numel * sizeof(float), cudaMemcpyDeviceToDevice,
                         (cudaStream_t)stream));
  return DFM_OK;
}

// -------------------------------------------------------------------------------------
int dfm_op_build_cost_volume(const float* d_cur, const float* d_prev, int C, int H, int W,
                             const float* h_depths, int D, int cost_sample_factor,
                             int feat_sample_factor, const dfm_geometry_t* geom,
                             float* d_volume, void* stream) {
  if (!d_cur || !d_prev || !h_depths || !geom || !d_volume)
    return fail(DFM_ERR_INVALID, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (cost_sample_factor < 1 || feat_sample_factor < 1 || C < 1 || D < 1 || H < 1 || W < 1)
    return fail(DFM_ERR_INVALID, "bad shape / sample factor");
  const int Ho = (int)std::nearbyint((double)H / cost_sample_factor);  // round-half-even
  const int Wo = (int)std::nearbyint((double)W / cost_sample_factor);
  if (Ho < 1 || Wo < 1 || (long long)(Ho - 1) * cost_sample_factor > H - 1 ||
      (long long)(Wo - 1) * cost_sample_factor > W - 1)
    return fail(DFM_ERR_INVALID, "feature size not compatible with cost_sample_factor");
  DevBuf cur, prev, dep;
  const long long HW = (long long)H * W;
  DFM_TRY(cur.alloc(HW * C));
  DFM_TRY(prev.alloc(HW * C));
  DFM_TRY(dep.alloc(D));
  CU_TRY(cudaMemcpyAsync(dep.p, h_depths, D * sizeof(float), cudaMemcpyHostToDevice, st));
  DFM_TRY(to_nhwc(d_cur, cur.p, C, HW, st));
  DFM_TRY(to_nhwc(d_prev, prev.p, C, HW, st));
  dfm::WarpLoader wl{};
  wl.cur = cur.p;
  wl.prev = prev.p;
  wl.depths = dep.p;
  wl.C = C;
  wl.first = 0;
  DFM_TRY(make_warp_geom(geom, H, W, cost_sample_factor, feat_sample_factor, &wl.g));
  const long long V = (long long)D * Ho * Wo;
  dim3 grid((unsigned)((V + 255) / 256), 2 * C);
  dfm::cost_volume_kernel<<<grid, 256, 0, st>>>(wl, D, Ho, Wo, d_volume);
  LAUNCH_CHECK();
  CU_TRY(cudaStreamSynchronize(st));
  return DFM_OK;
}

int dfm_op_conv3d(const float* d_x, int Cin, int Di, int Hi, int Wi, const float* h_w, int Cout,
                  const int stride[3], const int pad[3], int transposed, int conv_impl,
                  float* d_y, void* stream) {
  if (!d_x || !h_w || !d_y || !stride || !pad) return fail(DFM_ERR_INVALID, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  ConvW w;
  dfm::ConvGeom g = transposed ? geom_t(Di, Hi, Wi, Cin, Cout)
                               : geom_s(Di, Hi, Wi, Cin, Cout, stride[0], stride[1], stride[2],
                                        pad[0], pad[1], pad[2]);
  DFM_TRY(set_conv(w, h_w, (long long)27 * Cin * Cout, Cin, Cout, transposed,
                   dfm::tc_mode_of(g)));
  const long long Vi = (long long)Di * Hi * Wi, Vo = (long long)g.Do * g.Ho * g.Wo;
  DevBuf xin, yout;
  DFM_TRY(xin.alloc(Vi * Cin));
  DFM_TRY(yout.alloc(Vo * Cout));
  DFM_TRY(to_nhwc(d_x, xin.p, Cin, Vi, st));
  int rc = DFM_OK;
  // the K-outer kernel of the BEV necks (conv_tc_neck.cuh) serves the shapes the resident-weight
  // kernel does not: 64..256 channels, a short (<= 16) W axis, strides (1,1,1) / (1,1,2)
  const int zm = dfm::nk_zmode(g);
  const bool want_neck = zm >= 0 && conv_impl != DFM_CONV_SIMT &&
                         (conv_impl == DFM_CONV_TC_NECK || !w.tc.ready());
  if (conv_impl == DFM_CONV_TC_NECK && zm < 0)
    rc = fail(DFM_ERR_INVALID, "conv3d: the BEV-neck tensor-core kernel does not serve this shape");
  if (conv_impl == DFM_CONV_TC_NECK_DHW) {
    // the same kernel in plane-sweep-volume orientation (windowed along D), forced
    if (!dfm::neck_dhw_supported(g)) {
      rc = fail(DFM_ERR_INVALID, "conv3d: the windowed K-outer kernel needs stride 1, pad 1, "
                                 "channels in multiples of 32 and >= 64 input channels");
    } else {
      const std::vector<float> packed = repack_simt(h_w, Cin, Cout, 0);
      std::string err;
      // DFM_NTK_CG16=1: exercise the 16-channel-group / 64-output shape in this orientation too
      if (!w.ntk.build(packed.data(), Cin, Cout, dfm::NKZ_S1P1, &err, true,
                       getenv("DFM_NTK_CG16") ? dfm::neck_group_for(Cin, Cout, 1) : 32) ||
          !dfm::neck_tc_conv_dhw(src1(term(xin, nullptr, 0)), w.ntk, yout.p, g, nullptr, 0, 0, 1.f,
                                 st, &err))
        rc = fail(DFM_ERR_CUDA, err);
      g_launches.fetch_add(1);
      g_tc_launches.fetch_add(1);
    }
  } else if (rc == DFM_OK && want_neck) {
    const std::vector<float> packed = repack_simt(h_w, Cin, Cout, 0);
    std::string err;
    if (!w.ntc.build(packed.data(), Cin, Cout, zm, &err, false,
                     dfm::neck_group_for(Cin, Cout, g.Wo)) ||
        !dfm::neck_tc_conv(src1(term(xin, nullptr, 0)), w.ntc, yout.p, g, st, &err))
      rc = fail(DFM_ERR_CUDA, err);
    g_launches.fetch_add(1);
    g_tc_launches.fetch_add(1);
  } else if (rc == DFM_OK) {
    rc = run_conv(src1(term(xin, nullptr, 0)), w, yout.p, g, conv_impl, st);
  }
  if (rc == DFM_OK) rc = to_ncdhw(yout.p, d_y, Cout, Vo, st);
  cudaError_t e = cudaStreamSynchronize(st);
  if (rc == DFM_OK && e != cudaSuccess) rc = fail(DFM_ERR_CUDA, cudaGetErrorString(e));
  if (rc == DFM_OK && dfm::tc_consume_error())
    rc = fail(DFM_ERR_CUDA, "tensor-core conv kernel: mbarrier hand-over timed out");
  return rc;
}

int dfm_depth_head_forward(const float* d_cost, const float* d_depth_samples, int D, int Ho,
                           int Wo, int factor, float* d_volume, float* d_softmax,
                           float* d_preds, void* stream) {
  if (!d_cost || !d_depth_samples) return fail(DFM_ERR_INVALID, "null argument");
  if (D < 1 || Ho < 1 || Wo < 1 || factor < 1) return fail(DFM_ERR_INVALID, "bad shape");
  if ((long long)D * factor > dfm::DH_MAXBINS)
    return fail(DFM_ERR_INVALID, "DepthHead: more than 1024 depth bins");
  DFM_TRY(launch_depth_head(d_cost, d_depth_samples, D, Ho, Wo, factor, d_volume, d_softmax,
                            d_preds, nullptr, "depth_head", (cudaStream_t)stream));
  return DFM_OK;
}

}  // extern "C"

#include "neck_api.inc"
#include "frustum_api.inc"
#include "pipeline_api.inc"
#include "bev_api.inc"
#include "anchor3d_head_api.inc"
#include "voxel_sample_api.inc"
#include "stereo_tail_api.inc"
#include "spp_neck_api.inc"
#include "fpn_api.inc"
#include "liga_resnet_api.inc"
#include "resnet101_api.inc"
#include "box_post_api.inc"
#include "anchor_loss_api.inc"
#include "depth_loss_api.inc"
#include "atss_loss_api.inc"
#include "imitation_loss_api.inc"
#include "image_prep_api.inc"
#include "view_cache_api.inc"
#include "kitti_eval_api.inc"
#include "waymo_eval_api.inc"
