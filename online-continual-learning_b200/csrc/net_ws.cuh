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

// Weight-gradient tiling of conv layer c (shared by the workspace sizing and the launcher).
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

// Grid of the BN-backward reduction over M pixels x C channels (shared by sizing and launch).
inline int bn_bwd_rows_per_cta(int M, int C, int sms) {
  const int R = 256 / (C / 4);
  constexpr int per_sm = 2;   // CTAs per SM the row split aims for
  int rows = (M + per_sm * sms - 1) / (per_sm * sms);
  if (rows < 4 * R) rows = 4 * R;
  return (rows + R - 1) / R * R;
}
// bytes of BN-backward partials the workspace holds for a layer (the fused kernel's grid must fit as well)
inline size_t bn_bwd_part_capacity(int M, int C, int sms) {
  const int rows = bn_bwd_rows_per_cta(M, C, sms);
  return (size_t)((M + rows - 1) / rows) * C * 2 * sizeof(double);
}
constexpr int NET_COEF_DOUBLES = 512;  // 3 x 160 floats of BN-backward coefficients fit in front of the partials

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
  size_t stat_max = 0;
  for (int i = 0; i < p.n_conv; ++i) {
    const size_t M = (size_t)N * p.conv[i].hout * p.conv[i].wout;
    const size_t s = (size_t)conv_max_grid_m((int)M) * p.conv[i].cout * 2 * sizeof(double);
    if (s > stat_max) stat_max = s;
    const int rows = bn_bwd_rows_per_cta((int)M, p.conv[i].cout, sms);
    const size_t sb = ((M + rows - 1) / rows * p.conv[i].cout * 2 + NET_COEF_DOUBLES) * sizeof(double);
    if (sb > stat_max) stat_max = sb;
  }
  w.stat_part = reinterpret_cast<double*>(take(stat_max));
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
    w.wg_off[i] = wg;
    if (i == 0) {
      wg += (size_t)(8 * sms) * 27 * 20;  // stem: one partial per CTA
    } else {
      const WgradCfg g = wgrad_cfg(p.conv[i], N, sms);
      const ConvL& c = p.conv[i];
      const WgradTcCfg tg = wgrad_tc_cfg(N, c.hin, c.win, c.ks, c.stride, c.pad, c.cin, c.cout, sms);   // wgrad_tc.cu
      const int splits = (tg.eligible && tg.chains > g.splits) ? tg.chains : g.splits;
      wg += (size_t)splits * g.k_total * p.conv[i].cout;
    }
  }
  w.wg_part = reinterpret_cast<float*>(take(wg * sizeof(float)));
  w.bytes = off;
  return w;
}

}  // namespace b200ocl
