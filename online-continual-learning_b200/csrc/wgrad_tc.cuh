// wgrad_tc.cuh -- weight gradient of a 3x3 stride-1 convolution on wgmma (wgrad_tc.cu): its configuration, which the
// network's weight-gradient plan (wgrad_plan, net_ws.cuh) and the self-test read.
#pragma once
#include <cuda_runtime.h>

namespace b200ocl {

// x rows a wgrad_tc loader thread stages per tile (16 rows per pass): bounds the strip of 128 + 2 * (W + 2) + 2 rows
constexpr int WT_LD_MAX = 13;
// activation channels per CTA: 3 kernel columns x 20 channels fill 60 of a warpgroup's 64 fragment rows
constexpr int WT_SLICE = 20;
// output channels per CTA: the accumulators of the three kernel rows hold 3 x WT_BN_MAX / 2 registers per thread
constexpr int WT_BN_MAX = 40;

struct WgradTcCfg {
  int eligible;        // geometry covered (3x3, stride 1, pad 1, W <= 37, channels % 4 == 0)
  int slices;          // ceil(cin / WT_SLICE): one CTA column per 20-channel slice of the activation
  int cout_blocks;     // ceil(cout / WT_BN_MAX): one CTA layer per block of the output gradient
  int bn;              // MMA N: the block's output channels, the real ones rounded up to a multiple of 8 (<= WT_BN_MAX)
  int tiles;           // 128-position tiles of the zero-padded strip
  int tpc;             // tiles accumulated on the tensor core before the sum is written out as one partial ("chain")
  int chains;          // = partials per (slice, block): ceil(tiles / tpc) -- the `splits` the finalize kernel sums
  int chains_per_cta;
  int ctas_x;
};

inline int wgrad_tc_tiles(int N, int H, int W) {
  const long pp = (long)(H + 2) * (W + 2);
  const long last = (long)(N - 1) * pp + (long)(H - 1) * (W + 2) + (W - 1);
  return (int)(last / 128) + 1;
}

inline WgradTcCfg wgrad_tc_cfg(int N, int H, int W, int ks, int stride, int pad, int cin, int cout, int sms) {
  WgradTcCfg g{};
  g.eligible = (ks == 3 && stride == 1 && pad == 1 && cin % 4 == 0 && cout % 4 == 0 && cin >= 4 && cout >= 4 &&
                128 + 2 * (W + 2) + 2 <= 16 * WT_LD_MAX && (long)N * (H + 2) * (W + 2) < 2000000000L) ? 1 : 0;
  if (!g.eligible) return g;
  g.slices = (cin + WT_SLICE - 1) / WT_SLICE;
  g.cout_blocks = (cout + WT_BN_MAX - 1) / WT_BN_MAX;
  g.bn = ((cout + g.cout_blocks - 1) / g.cout_blocks + 7) / 8 * 8;   // 20 -> 24, 40 / 80 / 160 -> 40, 12 -> 16
  g.tiles = wgrad_tc_tiles(N, H, W);
  g.tpc = 2;   // 256 positions per tensor-core accumulation chain: ~2e-6 relative
  g.chains = (g.tiles + g.tpc - 1) / g.tpc;
  int want = sms / (g.slices * g.cout_blocks);
  if (want < 1) want = 1;
  if (want > g.chains) want = g.chains;
  g.chains_per_cta = (g.chains + want - 1) / want;
  // the CTA's two consumer warpgroups take alternate chains: an even count keeps them equally busy
  if (g.chains_per_cta > 1) g.chains_per_cta += g.chains_per_cta & 1;
  g.ctas_x = (g.chains + g.chains_per_cta - 1) / g.chains_per_cta;
  return g;
}

struct WgradTcArgs {
  const float* x;    // NHWC [N,H,W,Cin]   the convolution's input activation
  const float* dz;   // NHWC [N,H,W,Cout]  gradient of its raw output
  float* part;       // [chains][9 * Cin][Cout] partial sums, k = (kh * 3 + kw) * Cin + ci
  int N, H, W, Cin, Cout;
  int tpc, chains, chains_per_cta;
};

int launch_wgrad_tc(const WgradTcArgs& a, const WgradTcCfg& g, cudaStream_t stream);

}  // namespace b200ocl
