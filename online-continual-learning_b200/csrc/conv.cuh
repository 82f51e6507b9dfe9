// conv.cuh -- argument block and launchers of the implicit-GEMM convolution kernels.
#pragma once
#include "common.cuh"

namespace b200ocl {

enum ConvMode {
  CONV_RAW = 0,    // out = acc
  CONV_EVAL = 1,   // out = relu?((acc - rmean) * gamma/sqrt(rvar+eps) + beta (+ residual))   (folded eval-mode BN)
  CONV_TRAIN = 2,  // out = acc, plus per-channel batch statistics (sum, sum of squares) -> mean/invstd,
                   // running-stat update by the last CTA of each channel tile
  CONV_ACCUM = 3   // out += acc (data-gradient merged into an existing gradient)
};

struct ConvArgs {
  const float* in;   // NHWC [N,Hin,Win,CK]   (stem: NCHW [N,3,Hin,Win])
  const float* w;    // packed [ks*ks][CK][CN]
  float* out;        // NHWC [N,Hout,Wout,CN]
  int N, Hin, Win, CK, Hout, Wout, CN;
  int ks, stride, pad;
  int transposed;    // 0: forward gather (hi = ho*stride - pad + kh); 1: data-gradient gather
                     //    (input pixel (t/stride) with t = ho + pad - kh, only when divisible)
  const float* w_tc; // tensor-core operand image of the same weights (net_plan.cuh), nullable
  int tc_kb, tc_bn;  // its K blocks and real channels per tile
  const float* w_tp; // halo-patch tensor-core image (conv_tcp.cu), nullable
  int tp_bn, tp_slices;
  int tp_ps, tp_bs, tp_tiles;  // set by the launcher: patch stages, weight ring depth, 128-position tiles
  int force_path;    // 0 automatic; 1 CUDA-core kernels only; 2 conv_tc; 3 conv_tcp (selftest: fails if not eligible)
  int parity_order;  // stride-2 data gradient only: pixels enumerated [parity class][n][h/2][w/2] so that a CTA
                     //    sees one class and skips the taps that cannot reach it (9 of 36 tap-pixel pairs are live)
  int flip;          // patch kernel only: use tap (ks*ks-1-tap) of the weights (stride-1 data gradient)
  int th, tw, ti;    // patch kernel only: spatial tile (rows, cols, images), set by the launcher
  int M;             // N*Hout*Wout output pixels
  int mode;
  // CONV_EVAL
  const float* gamma;
  const float* beta;
  const float* rmean;
  const float* rvar;
  const float* residual;  // NHWC like out, nullable
  int relu;
  float eps;
  // CONV_TRAIN
  double* stat_part;       // [gridDim.x][CN][2]
  unsigned int* counter;   // [gridDim.y], zeroed before the forward pass
  float* save_mean;
  float* save_invstd;
  float* run_mean;
  float* run_var;
  float momentum;
};

// running = (1 - m) * running + m * s with one fixed rounding sequence (m * s rounded, then one fused multiply-add),
// so that the train-mode epilogues and the deferred apply (net_fwd.cu) move a running statistic to the same bits.
__device__ __forceinline__ float bn_running_update(float run, float s, float m) {
  return __fmaf_rn(1.f - m, run, __fmul_rn(m, s));
}

// BatchNorm finalize of channel c from its fp64 batch sums S = sum x and Q = sum x^2 over a.M pixels: batch mean,
// 1/sqrt(biased variance + eps), and the running mean / unbiased variance moved by a.momentum.
__device__ __forceinline__ void bn_finalize(const ConvArgs& a, int c, double S, double Q) {
  const double cnt = (double)a.M;
  const double mean = S / cnt;
  double var = Q / cnt - mean * mean;
  if (var < 0.0) var = 0.0;
  a.save_mean[c] = (float)mean;
  a.save_invstd[c] = (float)(1.0 / sqrt(var + (double)a.eps));
  const double unbiased = (a.M > 1) ? var * cnt / (cnt - 1.0) : var;
  a.run_mean[c] = bn_running_update(a.run_mean[c], (float)mean, a.momentum);
  a.run_var[c] = bn_running_update(a.run_var[c], (float)unbiased, a.momentum);
}

// conv_tcp.cu stages 128 + 2 * (W + 1) + 2 strip rows per tile; 16 * TP_LD_MAX is the bound on those rows (its patch
// loaders size their per-thread loads from it).  The bound still counts the 128 + 2 * (W + 2) + 2 rows of the earlier
// two-position halo, so the eligible maps stay those up to W = 37 wide.  The network plan builds halo-strip weight
// images exactly for the maps that fit.
constexpr int TP_LD_MAX = 13;
inline bool tcp_strip_fits(int W) { return 128 + 2 * (W + 2) + 2 <= 16 * TP_LD_MAX; }

// The kernel launch_conv runs for one ConvArgs on a GPU with `sms` SMs.  The numbering is the one
// b200ocl_conv_geom reports (include/b200ocl.h).
enum ConvKernel {
  CONV_K_NONE = -1,   // no kernel covers the launch (ConvPlan::why)
  CONV_K_STEM = 0,    // stem_kernel: 3 -> 20 channels, NCHW input
  CONV_K_TCP = 1,     // conv_tcp_kernel<nt>: wgmma fed from a halo strip (conv_tcp.cu)
  CONV_K_TC = 2,      // conv_tc_kernel<nt>: wgmma with im2col tiles (conv_tc.cu)
  CONV_K_PATCH = 3,   // conv_patch_kernel<bn, pt>
  CONV_K_TILED = 4,   // conv_kernel<bn, pt>
  CONV_K_KSPLIT = 5   // conv_ksplit_kernel<pt, kwarps>
};
struct ConvPlan {
  int kernel;            // ConvKernel
  int nt;                // CONV_K_TCP / CONV_K_TC: padded MMA N
  int bn, pt;            // CONV_K_PATCH / CONV_K_TILED: channels and pixels per thread; CONV_K_KSPLIT: bn = 20, pt
  int kwarps;            // CONV_K_KSPLIT: warps sharing the K loop
  int grid_x, grid_y;    // the grid; a train-mode launch writes grid_x * CN (sum, sum of squares) partials
  int th, tw, ti;        // CONV_K_PATCH: spatial tile (rows, columns, images)
  size_t smem;           // CONV_K_PATCH: dynamic shared memory
  int tp_ps, tp_bs;      // CONV_K_TCP: patch stages and weight ring depth (conv_tcp_pipeline)
  const char* why;       // CONV_K_NONE: the reason
};
// Pure host function: every decision launch_conv takes, for a GPU with `sms` SMs.  CK == 3 is the stem.
ConvPlan conv_plan(const ConvArgs& a, int sms);
// Bytes of statistics partials (stat_part) a train-mode launch with plan `pl` writes.
inline size_t conv_stat_bytes(const ConvPlan& pl, int CN) { return (size_t)pl.grid_x * CN * 2 * sizeof(double); }
int launch_conv(const ConvArgs& a, int sms, cudaStream_t stream);   // runs conv_plan(a, sms)
bool conv_tc_eligible(const ConvArgs& a, int sms);
int launch_conv_tc(const ConvArgs& a, const ConvPlan& pl, cudaStream_t stream);   // conv_tc.cu: wgmma 3xTF32 path
bool conv_tcp_eligible(const ConvArgs& a);
int conv_tcp_grid_x(const ConvArgs& a, int sms);   // persistent CTAs per channel tile of conv_tcp_kernel
// Pure host function: the patch stages and weight ring depth conv_tcp_kernel<nt> runs with (its shared-memory fit).
void conv_tcp_pipeline(const ConvArgs& a, int nt, int* ps, int* bs);
int launch_conv_tcp(const ConvArgs& a, const ConvPlan& pl, cudaStream_t stream);  // conv_tcp.cu: wgmma fed from a halo patch

}  // namespace b200ocl
