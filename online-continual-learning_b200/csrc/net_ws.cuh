// net_ws.cuh -- carving of the caller-provided workspaces of the ResNet engine.
#pragma once
#include "wgrad_tc.cuh"
#include "conv.cuh"
#include "net_plan.cuh"

namespace b200ocl {

constexpr int NET_COUNTERS = 8 * NET_MAX_CONV * 2;  // forward: [conv][tile]; backward uses the second half

struct EvalWs {
  float* buf[4];  // NHWC ping-pong activations, N * max_act_per_image floats each
  size_t bytes;
};

inline EvalWs eval_ws(const NetPlan& p, int N, void* base) {
  EvalWs w{};
  unsigned char* b = static_cast<unsigned char*>(base);
  const size_t one = align_up((size_t)N * p.max_act_per_image * sizeof(float), 256);
  for (int i = 0; i < 4; ++i) w.buf[i] = reinterpret_cast<float*>(b + i * one);
  w.bytes = 4 * one;
  return w;
}

// Tiling of the fp32 weight-gradient kernel (wgrad_kernel, net_bwd.cu) over conv layer c.
struct WgradCfg {
  int k_total;    // ks*ks*cin
  int k4_groups;  // k_total / 4
  int kw;         // warps along K per CTA (each covers 32 k4-groups = 128 k)
  int nw;         // warps along Cout per CTA (each covers 20 channels)
  int grid_k;     // CTAs along K
  int grid_n;     // CTAs along Cout
  int splits;     // CTAs along the pixel (reduction) dimension
  int pix_per_split;
};

inline WgradCfg wgrad_cfg(const ConvL& c, int N, int sms) {
  WgradCfg g{};
  g.k_total = c.ks * c.ks * c.cin;
  g.k4_groups = g.k_total / 4;
  const int k_tiles = (g.k4_groups + 31) / 32;
  const int n_groups = c.cout / 20;
  g.kw = k_tiles < 2 ? k_tiles : 2;
  g.nw = n_groups < 2 ? n_groups : 2;
  g.grid_k = (k_tiles + g.kw - 1) / g.kw;
  g.grid_n = (n_groups + g.nw - 1) / g.nw;
  const int M = N * c.hout * c.wout;
  // >= 16 resident warps per SM overall, at least 64 pixels of reduction per CTA (fewer, larger splits
  // measured slower: the kernel needs the parallelism more than the finalize pass needs fewer partials)
  const int warps_per_cta = g.kw * g.nw;
  constexpr int target = 8;   // resident warps per SM the split count aims for
  int splits = (target * sms + warps_per_cta * g.grid_k * g.grid_n - 1) / (warps_per_cta * g.grid_k * g.grid_n);
  const int max_by_pixels = (M + 63) / 64;
  if (splits > max_by_pixels) splits = max_by_pixels;
  if (splits < 1) splits = 1;
  g.pix_per_split = ((M + splits - 1) / splits + 15) / 16 * 16;
  g.splits = (M + g.pix_per_split - 1) / g.pix_per_split;
  return g;
}

constexpr int SW_PX = 128;   // pixels per chunk of the stem weight-gradient kernel (stem_wgrad_kernel, net_bwd.cu)

// Which kernel computes the weight gradient of conv layer ci, with what configuration, and how many partials it writes.
// The workspace sizing (train_ws), the launch and the finalize table of b200ocl_net_backward all read it.
enum WgradKernel { WGRAD_STEM, WGRAD_TC, WGRAD_FP32 };
struct WgradPlan {
  WgradKernel kernel;
  WgradTcCfg tc;      // WGRAD_TC (wgrad_tc.cu)
  WgradCfg fp32;      // WGRAD_FP32 (wgrad_kernel)
  int stem_ppc;       // WGRAD_STEM: pixels per CTA
  int splits;         // partials of [ks*ks*cin][cout] floats the kernel writes; the finalize sums exactly these
};

inline WgradPlan wgrad_plan(const NetPlan& p, int ci, int N, int sms) {
  WgradPlan w{};
  const ConvL& c = p.conv[ci];
  if (ci == 0) {
    // one partial per CTA, at most two CTAs per SM
    w.kernel = WGRAD_STEM;
    const int M = N * p.in_h * p.in_w;
    int ctas = (M + SW_PX - 1) / SW_PX;
    if (ctas > 2 * sms) ctas = 2 * sms;
    w.stem_ppc = ((M + ctas - 1) / ctas + SW_PX - 1) / SW_PX * SW_PX;
    w.splits = (M + w.stem_ppc - 1) / w.stem_ppc;
    return w;
  }
  // 3x3 stride-1 layers on maps the strip holds: wgmma with the activation read in place from a strip
  w.tc = wgrad_tc_cfg(N, c.hin, c.win, c.ks, c.stride, c.pad, c.cin, c.cout, sms);
  if (w.tc.eligible) {
    w.kernel = WGRAD_TC;
    w.splits = w.tc.chains;
    return w;
  }
  w.kernel = WGRAD_FP32;
  w.fp32 = wgrad_cfg(c, N, sms);
  w.splits = w.fp32.splits;
  return w;
}

// Launch geometry of the BN backward over M pixels x C channels (launch_bn_bwd, net_bwd.cu).  With fused_ok (the
// caller has a ready counter) it is the fused kernel when its grid is co-resident (at most one CTA per SM) and its
// rows fit in shared memory; otherwise the two-phase reduce + apply.  The fused rows are split over sms CTAs, the
// two-phase rows over 2 * sms, so the fused rows are never fewer and its grid never larger: the two-phase grid
// bounds the partials either path writes (train_ws).
struct BnBwdGeom {
  bool fused;
  int rows;       // rows per CTA, a multiple of the rows a CTA covers per pass
  int grid;
  size_t smem;    // dynamic shared memory of the fused or the reduce kernel
};

inline BnBwdGeom bn_bwd_geom(int M, int C, int sms, bool fused_ok) {
  const int R = 256 / (C / 4);                     // rows per pass: 256 threads over C / 4 float4 columns
  const int groups = 256 / C > 0 ? 256 / C : 1;    // thread groups of the final reduction
  const size_t sred = (size_t)(R > groups ? R : groups) * C * 2 * sizeof(double);
  auto split = [&](int ctas) {
    int rows = (M + ctas - 1) / ctas;
    if (rows < 4 * R) rows = 4 * R;
    return (rows + R - 1) / R * R;
  };
  BnBwdGeom g{};
  if (fused_ok) {
    g.rows = split(sms);
    g.grid = (M + g.rows - 1) / g.rows;
    g.smem = sred + (size_t)g.rows * C * 2 * sizeof(float);   // all of a CTA's rows stay resident
    g.fused = g.grid <= sms && g.smem <= 200 * 1024;
    if (g.fused) return g;
  }
  constexpr int per_sm = 2;   // CTAs per SM the two-phase row split aims for
  g.rows = split(per_sm * sms);
  g.grid = (M + g.rows - 1) / g.rows;
  g.smem = sred;
  return g;
}
constexpr int NET_COEF_DOUBLES = 512;  // 3 x 160 floats of BN-backward coefficients fit in front of the partials

// The convolution launches of a layer: train-mode forward (batch statistics), eval-mode forward, data gradient.
enum ConvPass { PASS_TRAIN = 0, PASS_EVAL = 1, PASS_DGRAD = 2 };

// conv_plan of layer c's launch in pass `pass` over N images.  Only the presence of the weight images matters to the
// plan, so they are addressed from a null packed arena (their offsets are never 0: the packed weights come first).
inline ConvPlan layer_conv_plan(const ConvL& c, int N, int pass, int sms) {
  ConvArgs a = conv_layer_args(c, N, nullptr, nullptr, nullptr, pass == PASS_DGRAD);
  a.mode = pass == PASS_TRAIN ? CONV_TRAIN : (pass == PASS_EVAL ? CONV_EVAL : CONV_RAW);
  return conv_plan(a, sms);
}

struct TrainWs {
  unsigned int* counters;  // NET_COUNTERS x u32 (8 per conv), zeroed at the start of forward / backward
  double* stat_part;
  float* save;    // batch mean / invstd per BN (BnL::save_off)
  float* run_scratch;  // [2][1024] throw-away running statistics (eval-statistics forward, net_fwd.cu)
  float* run_defer;    // deferred-statistics forward: (batch mean, unbiased batch variance) per BN, laid out like bn_stats
  float* z;       // raw conv outputs, conv i at N * ConvL::act_off
  float* a;       // activated outputs (conv2 slot holds the block output)
  float* feat;    // [N, dim_in]
  float* hid;     // [N, dim_in] mlp hidden (post-ReLU)
  float* proj;    // [N, out_dim] pre-normalisation projection
  float* g0;      // backward scratch: gradient w.r.t. a block output
  float* g1;      // gradient w.r.t. a block input (accumulated)
  float* g2;      // dz of the current conv
  float* g3;      // gradient w.r.t. conv1's activation inside a block
  float* g4;      // second dz buffer: weight gradients run on a side stream while the next dz is produced
  float* dfeat;
  float* dhid;
  float* dproj;
  float* wg_part;  // weight-gradient partials, conv i at wg_off[i]
  size_t wg_off[NET_MAX_CONV];
  size_t stat_bytes;   // size of the stat_part region
  int sms;             // SM count the launch geometries (and so the partial regions) were planned for
  size_t bytes;
};

inline TrainWs train_ws(const NetPlan& p, int N, void* base, int sms) {
  TrainWs w{};
  unsigned char* b = static_cast<unsigned char*>(base);
  size_t off = 0;
  auto take = [&](size_t nbytes) {
    unsigned char* r = b + off;
    off += align_up(nbytes, 256);
    return r;
  };
  w.counters = reinterpret_cast<unsigned int*>(take(NET_COUNTERS * sizeof(unsigned int)));
  // stat_part holds the batch-statistics partials of the train-mode convolution that runs (one per CTA along the
  // pixels of its grid) and, in the backward, the BN-backward coefficients and partials
  size_t stat_max = 0;
  for (int i = 0; i < p.n_conv; ++i) {
    const size_t M = (size_t)N * p.conv[i].hout * p.conv[i].wout;
    const size_t s = conv_stat_bytes(layer_conv_plan(p.conv[i], N, PASS_TRAIN, sms), p.conv[i].cout);
    if (s > stat_max) stat_max = s;
    const int grid = bn_bwd_geom((int)M, p.conv[i].cout, sms, false).grid;
    const size_t sb = ((size_t)grid * p.conv[i].cout * 2 + NET_COEF_DOUBLES) * sizeof(double);
    if (sb > stat_max) stat_max = sb;
  }
  w.stat_part = reinterpret_cast<double*>(take(stat_max));
  w.stat_bytes = stat_max;
  w.sms = sms;
  w.save = reinterpret_cast<float*>(take(2 * p.n_bn_channels * sizeof(float)));
  w.run_scratch = reinterpret_cast<float*>(take(2 * 1024 * sizeof(float)));
  w.run_defer = reinterpret_cast<float*>(take(p.n_stats * sizeof(float)));
  w.z = reinterpret_cast<float*>(take((size_t)N * p.act_per_image * sizeof(float)));
  w.a = reinterpret_cast<float*>(take((size_t)N * p.act_per_image * sizeof(float)));
  w.feat = reinterpret_cast<float*>(take((size_t)N * p.dim_in * sizeof(float)));
  w.hid = reinterpret_cast<float*>(take((size_t)N * p.dim_in * sizeof(float)));
  w.proj = reinterpret_cast<float*>(take((size_t)N * p.out_dim * sizeof(float)));
  const size_t act = (size_t)N * p.max_act_per_image * sizeof(float);
  w.g0 = reinterpret_cast<float*>(take(act));
  w.g1 = reinterpret_cast<float*>(take(act));
  w.g2 = reinterpret_cast<float*>(take(act));
  w.g3 = reinterpret_cast<float*>(take(act));
  w.g4 = reinterpret_cast<float*>(take(act));
  w.dfeat = reinterpret_cast<float*>(take((size_t)N * p.dim_in * sizeof(float)));
  w.dhid = reinterpret_cast<float*>(take((size_t)N * p.dim_in * sizeof(float)));
  w.dproj = reinterpret_cast<float*>(take((size_t)N * p.out_dim * sizeof(float)));
  size_t wg = 0;
  for (int i = 0; i < p.n_conv; ++i) {
    const ConvL& c = p.conv[i];
    w.wg_off[i] = wg;
    wg += (size_t)wgrad_plan(p, i, N, sms).splits * c.ks * c.ks * c.cin * c.cout;
  }
  w.wg_part = reinterpret_cast<float*>(take(wg * sizeof(float)));
  w.bytes = off;
  return w;
}

}  // namespace b200ocl
