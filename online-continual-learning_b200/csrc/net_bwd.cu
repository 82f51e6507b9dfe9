// net_bwd.cu -- backward pass of the Reduced-ResNet18 / SupConResNet engine (sm_90a).
//
// Replaces loss.backward() through reference models/resnet.py:33-36,90-109,159-165
// (autograd over cuDNN conv / batch-norm backward, addmm, normalize), as used at
// agents/exp_replay.py:55,77,86 and agents/scr.py:59.
//
// Per BasicBlock, in reverse:  BN2 backward (reduce + apply, ReLU mask folded in) -> weight
// gradient of conv2 -> data gradient of conv2 -> [shortcut BN/conv backward] -> BN1 backward ->
// weight gradient of conv1 -> data gradient of conv1 accumulated onto the shortcut gradient.
// Data gradients reuse the implicit-GEMM kernel of conv.cu (transposed gather, [tap][cout][cin]
// weights).  Weight gradients are a GEMM over pixels: split over pixel ranges, partials reduced
// in fixed order by one finalize kernel for all layers (deterministic; no float atomics).
#include <float.h>
#include <math.h>
#include <stdlib.h>

#include "net_ws.cuh"

namespace b200ocl {
namespace {

// ----------------------------------------------------------------------------- BN backward
struct BnBwdArgs {
  const float* dA;     // gradient w.r.t. the activated output, NHWC [M][C]
  const float* amask;  // activated output (ReLU mask: > 0), nullable
  const float* z;      // raw conv output
  const float* mean;
  const float* invstd;
  const float* gamma;
  int M, C;
  int rows_per_cta;
  double* part;  // [gridDim.x][C][2]
  unsigned int* counter;
  unsigned int* ready;   // fused kernel: set by the finalizing CTA once coef[] is written
  float* dgamma;
  float* dbeta;
  int accumulate;
  int eval_stats;   // BN in eval mode: the statistics are constants, no mean / covariance terms in dz
  float* coef;  // [3][C]: gamma*invstd, mean(g), mean(g*xhat)
  float* dz;
  float* gout;  // nullable: masked gradient g (identity-shortcut branch)
};

__global__ void __launch_bounds__(256) bn_bwd_reduce_kernel(BnBwdArgs a) {
  extern __shared__ __align__(16) double sred[];  // [R][C][2]
  __shared__ bool is_last;
  const int cols = a.C / 4;
  const int R = 256 / cols;
  const int tid = threadIdx.x;
  const int col = tid % cols, rl = tid / cols;
  const bool active = rl < R;
  float s[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f};
  if (active) {
    const float4 mu = *reinterpret_cast<const float4*>(a.mean + col * 4);
    const float4 is = *reinterpret_cast<const float4*>(a.invstd + col * 4);
    const int r0 = blockIdx.x * a.rows_per_cta;
    const int r1 = min(a.M, r0 + a.rows_per_cta);
    // four rows per trip: all twelve 16-byte loads are issued before the first use
    for (int rb = r0 + rl; rb < r1; rb += 4 * R) {
      float4 g[4], m[4], zz[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int r = rb + u * R;
        const size_t i = (size_t)(r < r1 ? r : rb) * cols + col;
        g[u] = __ldg(reinterpret_cast<const float4*>(a.dA) + i);
        zz[u] = __ldg(reinterpret_cast<const float4*>(a.z) + i);
        m[u] = a.amask ? __ldg(reinterpret_cast<const float4*>(a.amask) + i) : make_float4(1.f, 1.f, 1.f, 1.f);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (rb + u * R >= r1) break;
        const float gx = m[u].x > 0.f ? g[u].x : 0.f;
        const float gy = m[u].y > 0.f ? g[u].y : 0.f;
        const float gz = m[u].z > 0.f ? g[u].z : 0.f;
        const float gw = m[u].w > 0.f ? g[u].w : 0.f;
        s[0] += gx; s[1] += gy; s[2] += gz; s[3] += gw;
        q[0] = fmaf(gx, (zz[u].x - mu.x) * is.x, q[0]);
        q[1] = fmaf(gy, (zz[u].y - mu.y) * is.y, q[1]);
        q[2] = fmaf(gz, (zz[u].z - mu.z) * is.z, q[2]);
        q[3] = fmaf(gw, (zz[u].w - mu.w) * is.w, q[3]);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      sred[((size_t)rl * a.C + col * 4 + j) * 2 + 0] = (double)s[j];
      sred[((size_t)rl * a.C + col * 4 + j) * 2 + 1] = (double)q[j];
    }
  }
  __syncthreads();
  for (int c = tid; c < a.C; c += 256) {
    double S = 0.0, Q = 0.0;
    for (int r = 0; r < R; ++r) {
      S += sred[((size_t)r * a.C + c) * 2 + 0];
      Q += sred[((size_t)r * a.C + c) * 2 + 1];
    }
    a.part[((size_t)blockIdx.x * a.C + c) * 2 + 0] = S;
    a.part[((size_t)blockIdx.x * a.C + c) * 2 + 1] = Q;
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) is_last = (atomicAdd(a.counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  const int groups = 256 / a.C > 0 ? 256 / a.C : 1;
  // channels beyond 256 do not occur (C <= 160)
  const int ch = tid % a.C, grp = tid / a.C;
  double S = 0.0, Q = 0.0;
  if (grp < groups) {
    unsigned int b = grp;
    for (; b + 7u * groups < gridDim.x; b += 8u * groups) {   // eight loads in flight, fixed association
      double2 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u)
        v[u] = __ldcg(reinterpret_cast<const double2*>(a.part + ((size_t)(b + u * groups) * a.C + ch) * 2));
      S += ((v[0].x + v[1].x) + (v[2].x + v[3].x)) + ((v[4].x + v[5].x) + (v[6].x + v[7].x));
      Q += ((v[0].y + v[1].y) + (v[2].y + v[3].y)) + ((v[4].y + v[5].y) + (v[6].y + v[7].y));
    }
    for (; b < gridDim.x; b += groups) {
      const double2 v = __ldcg(reinterpret_cast<const double2*>(a.part + ((size_t)b * a.C + ch) * 2));
      S += v.x;
      Q += v.y;
    }
    sred[((size_t)grp * a.C + ch) * 2 + 0] = S;
    sred[((size_t)grp * a.C + ch) * 2 + 1] = Q;
  }
  __syncthreads();
  if (tid < a.C) {
    double db = 0.0, dg = 0.0;
    for (int g = 0; g < groups; ++g) {
      db += sred[((size_t)g * a.C + tid) * 2 + 0];
      dg += sred[((size_t)g * a.C + tid) * 2 + 1];
    }
    if (a.accumulate) {
      a.dgamma[tid] += (float)dg;
      a.dbeta[tid] += (float)db;
    } else {
      a.dgamma[tid] = (float)dg;
      a.dbeta[tid] = (float)db;
    }
    a.coef[tid] = a.gamma[tid] * a.invstd[tid];
    a.coef[a.C + tid] = a.eval_stats ? 0.f : (float)(db / (double)a.M);
    a.coef[2 * a.C + tid] = a.eval_stats ? 0.f : (float)(dg / (double)a.M);
  }
}

__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(BnBwdArgs a) {
  const size_t n_vec = (size_t)a.M * a.C / 4;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += stride) {
    const int c = (int)((i * 4) % (size_t)a.C);
    float4 g = reinterpret_cast<const float4*>(a.dA)[i];
    if (a.amask) {
      const float4 m = reinterpret_cast<const float4*>(a.amask)[i];
      g.x = m.x > 0.f ? g.x : 0.f;
      g.y = m.y > 0.f ? g.y : 0.f;
      g.z = m.z > 0.f ? g.z : 0.f;
      g.w = m.w > 0.f ? g.w : 0.f;
    }
    const float4 zz = reinterpret_cast<const float4*>(a.z)[i];
    const float4 mu = *reinterpret_cast<const float4*>(a.mean + c);
    const float4 is = *reinterpret_cast<const float4*>(a.invstd + c);
    const float4 k1 = *reinterpret_cast<const float4*>(a.coef + c);
    const float4 mb = *reinterpret_cast<const float4*>(a.coef + a.C + c);
    const float4 mg = *reinterpret_cast<const float4*>(a.coef + 2 * a.C + c);
    float4 d;
    d.x = k1.x * (g.x - mb.x - (zz.x - mu.x) * is.x * mg.x);
    d.y = k1.y * (g.y - mb.y - (zz.y - mu.y) * is.y * mg.y);
    d.z = k1.z * (g.z - mb.z - (zz.z - mu.z) * is.z * mg.z);
    d.w = k1.w * (g.w - mb.w - (zz.w - mu.w) * is.w * mg.w);
    reinterpret_cast<float4*>(a.dz)[i] = d;
    if (a.gout) reinterpret_cast<float4*>(a.gout)[i] = g;
  }
}


// One cooperative launch instead of reduce + apply: every CTA keeps the masked gradient g and the normalised
// activation xhat of its own rows in shared memory between the two phases, so dA / z / mask are read from
// HBM / L2 once instead of twice and a launch disappears.  The per-channel sums still meet in fp64 partials that
// the LAST arriving CTA reduces in CTA order (same association as the two-kernel path); the others spin on a
// ready flag.  Requires the whole grid to be co-resident: grid <= number of SMs, one CTA per SM.
__global__ void __launch_bounds__(256, 1) bn_bwd_fused_kernel(BnBwdArgs a) {
  extern __shared__ __align__(16) double sred[];  // [max(R, groups)][C][2] doubles, then the resident rows
  __shared__ bool is_last;
  const int cols = a.C / 4;
  const int R = 256 / cols;
  const int tid = threadIdx.x;
  const int col = tid % cols, rl = tid / cols;
  const bool active = rl < R;
  const int groups = 256 / a.C > 0 ? 256 / a.C : 1;
  const int srows = R > groups ? R : groups;
  float4* sg = reinterpret_cast<float4*>(sred + (size_t)srows * a.C * 2);      // [rows_per_cta][cols]
  float4* sx = sg + (size_t)a.rows_per_cta * cols;
  const int r0 = blockIdx.x * a.rows_per_cta;
  const int r1 = min(a.M, r0 + a.rows_per_cta);
  float s[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f};
  if (active) {
    const float4 mu = *reinterpret_cast<const float4*>(a.mean + col * 4);
    const float4 is = *reinterpret_cast<const float4*>(a.invstd + col * 4);
    for (int rb = r0 + rl; rb < r1; rb += 4 * R) {
      float4 g[4], m[4], zz[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int r = rb + u * R;
        const size_t i = (size_t)(r < r1 ? r : rb) * cols + col;
        g[u] = __ldg(reinterpret_cast<const float4*>(a.dA) + i);
        zz[u] = __ldg(reinterpret_cast<const float4*>(a.z) + i);
        m[u] = a.amask ? __ldg(reinterpret_cast<const float4*>(a.amask) + i) : make_float4(1.f, 1.f, 1.f, 1.f);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int r = rb + u * R;
        if (r >= r1) break;
        float4 gm, xh;
        gm.x = m[u].x > 0.f ? g[u].x : 0.f;
        gm.y = m[u].y > 0.f ? g[u].y : 0.f;
        gm.z = m[u].z > 0.f ? g[u].z : 0.f;
        gm.w = m[u].w > 0.f ? g[u].w : 0.f;
        xh.x = (zz[u].x - mu.x) * is.x;
        xh.y = (zz[u].y - mu.y) * is.y;
        xh.z = (zz[u].z - mu.z) * is.z;
        xh.w = (zz[u].w - mu.w) * is.w;
        s[0] += gm.x; s[1] += gm.y; s[2] += gm.z; s[3] += gm.w;
        q[0] = fmaf(gm.x, xh.x, q[0]);
        q[1] = fmaf(gm.y, xh.y, q[1]);
        q[2] = fmaf(gm.z, xh.z, q[2]);
        q[3] = fmaf(gm.w, xh.w, q[3]);
        sg[(size_t)(r - r0) * cols + col] = gm;
        sx[(size_t)(r - r0) * cols + col] = xh;
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      sred[((size_t)rl * a.C + col * 4 + j) * 2 + 0] = (double)s[j];
      sred[((size_t)rl * a.C + col * 4 + j) * 2 + 1] = (double)q[j];
    }
  }
  __syncthreads();
  for (int c = tid; c < a.C; c += 256) {
    double S = 0.0, Q = 0.0;
    for (int r = 0; r < R; ++r) {
      S += sred[((size_t)r * a.C + c) * 2 + 0];
      Q += sred[((size_t)r * a.C + c) * 2 + 1];
    }
    a.part[((size_t)blockIdx.x * a.C + c) * 2 + 0] = S;
    a.part[((size_t)blockIdx.x * a.C + c) * 2 + 1] = Q;
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) is_last = (atomicAdd(a.counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (is_last) {
    __threadfence();
    const int ch = tid % a.C, grp = tid / a.C;
    double S = 0.0, Q = 0.0;
    if (grp < groups) {
      unsigned int b = grp;
      for (; b + 7u * groups < gridDim.x; b += 8u * groups) {   // eight loads in flight, fixed association
        double2 v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u)
          v[u] = __ldcg(reinterpret_cast<const double2*>(a.part + ((size_t)(b + u * groups) * a.C + ch) * 2));
        S += ((v[0].x + v[1].x) + (v[2].x + v[3].x)) + ((v[4].x + v[5].x) + (v[6].x + v[7].x));
        Q += ((v[0].y + v[1].y) + (v[2].y + v[3].y)) + ((v[4].y + v[5].y) + (v[6].y + v[7].y));
      }
      for (; b < gridDim.x; b += groups) {
        const double2 v = __ldcg(reinterpret_cast<const double2*>(a.part + ((size_t)b * a.C + ch) * 2));
        S += v.x;
        Q += v.y;
      }
      sred[((size_t)grp * a.C + ch) * 2 + 0] = S;
      sred[((size_t)grp * a.C + ch) * 2 + 1] = Q;
    }
    __syncthreads();
    if (tid < a.C) {
      double db = 0.0, dg = 0.0;
      for (int g = 0; g < groups; ++g) {
        db += sred[((size_t)g * a.C + tid) * 2 + 0];
        dg += sred[((size_t)g * a.C + tid) * 2 + 1];
      }
      if (a.accumulate) {
        a.dgamma[tid] += (float)dg;
        a.dbeta[tid] += (float)db;
      } else {
        a.dgamma[tid] = (float)dg;
        a.dbeta[tid] = (float)db;
      }
      a.coef[tid] = a.gamma[tid] * a.invstd[tid];
      a.coef[a.C + tid] = a.eval_stats ? 0.f : (float)(db / (double)a.M);
      a.coef[2 * a.C + tid] = a.eval_stats ? 0.f : (float)(dg / (double)a.M);
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) atomicExch(a.ready, 1u);
  } else if (tid == 0) {
    unsigned int seen;
    do {
      asm volatile("ld.acquire.gpu.u32 %0, [%1];\n" : "=r"(seen) : "l"(a.ready) : "memory");
    } while (seen == 0u);
  }
  __syncthreads();
  if (!active) return;
  const float4 k1 = __ldcg(reinterpret_cast<const float4*>(a.coef) + col);
  const float4 mb = __ldcg(reinterpret_cast<const float4*>(a.coef + a.C) + col);
  const float4 mg = __ldcg(reinterpret_cast<const float4*>(a.coef + 2 * a.C) + col);
  for (int r = r0 + rl; r < r1; r += R) {
    const float4 g = sg[(size_t)(r - r0) * cols + col];
    const float4 xh = sx[(size_t)(r - r0) * cols + col];
    float4 d;
    d.x = k1.x * (g.x - mb.x - xh.x * mg.x);
    d.y = k1.y * (g.y - mb.y - xh.y * mg.y);
    d.z = k1.z * (g.z - mb.z - xh.z * mg.z);
    d.w = k1.w * (g.w - mb.w - xh.w * mg.w);
    const size_t i = (size_t)r * cols + col;
    reinterpret_cast<float4*>(a.dz)[i] = d;
    if (a.gout) reinterpret_cast<float4*>(a.gout)[i] = g;
  }
}

int launch_bn_bwd(BnBwdArgs a, cudaStream_t stream) {
  const BnBwdGeom g = bn_bwd_geom(a.M, a.C, sm_count(), a.ready != nullptr);
  a.rows_per_cta = g.rows;
  if (g.fused) {
    B200OCL_CUDA(raise_smem_limit<bn_bwd_fused_kernel>(200 * 1024));
    B200OCL_PROF("bn_bwd", (a.amask ? 16.0 : 12.0) * a.M * a.C + (a.gout ? 4.0 * a.M * a.C : 0.0), stream);
    bn_bwd_fused_kernel<<<g.grid, 256, g.smem, stream>>>(a);
    B200OCL_LAUNCHED();
    return B200OCL_OK;
  }
  B200OCL_PROF("bn_bwd", (a.amask ? 12.0 : 8.0) * a.M * a.C, stream);
  bn_bwd_reduce_kernel<<<g.grid, 256, g.smem, stream>>>(a);
  B200OCL_LAUNCHED();
  size_t blocks = ((size_t)a.M * a.C / 4 + 255) / 256;
  const size_t cap = (size_t)16 * sm_count();
  if (blocks > cap) blocks = cap;
  B200OCL_PROF("bn_bwd", (a.amask ? 16.0 : 12.0) * a.M * a.C + (a.gout ? 4.0 * a.M * a.C : 0.0), stream);
  bn_bwd_apply_kernel<<<(unsigned)blocks, 256, 0, stream>>>(a);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

// ----------------------------------------------------------------------------- weight gradient
// part[split][k][co] = sum over the split's pixels of  x[pixel shifted by tap(k)][ci(k)] * dz[pixel][co]
struct WgradArgs {
  const float* x;   // NHWC [N,Hin,Win,Cin]  block input activation
  const float* dz;  // NHWC [N,Hout,Wout,Cout]
  float* part;
  int N, Hin, Win, Cin, Hout, Wout, Cout, ks, stride, pad, M;
  int k_total, k4_groups, kw, nw, pix_per_split;
};

constexpr int WG_MC = 16;   // pixels staged per iteration
constexpr int WG_NST = 3;   // cp.async ring depth

__global__ void __launch_bounds__(128, 3) wgrad_kernel(WgradArgs a) {
  extern __shared__ __align__(16) float smem[];
  const int KS = a.kw * 128;  // floats of K staged per pixel
  const int NS = a.nw * 20;
  const int stage_f = WG_MC * (KS + NS);
  float* sbuf = smem;                                              // [NST][ MC*KS | MC*NS ]
  int* s_info = reinterpret_cast<int*>(sbuf + WG_NST * stage_f);   // [NST+1][3][MC]: base, h0, w0

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nthreads = blockDim.x;
  const int kwi = warp % a.kw, nwi = warp / a.kw;
  const int g4_base = blockIdx.x * a.kw * 32;
  const int co_base = blockIdx.y * NS;
  const int m_begin = blockIdx.z * a.pix_per_split;
  const int m_end = min(a.M, m_begin + a.pix_per_split);
  const int hw_out = a.Hout * a.Wout;
  const int nch = (m_end - m_begin + WG_MC - 1) / WG_MC;

  // Per-thread gather constants: nthreads = 32*kw*nw is a multiple of the staged row length (kw*32
  // k4-groups), so a thread always stages the same k4-group: its tap / channel offset is fixed and the
  // per-pixel work is two compares and one add.
  const int row_len = a.kw * 32;
  const int gl = tid % row_len, pm0 = tid / row_len;   // pm = pm0 + it * nw
  const int g4_mine = g4_base + gl;
  bool k_ok = g4_mine < a.k4_groups;
  int kh = 0, kwd = 0, k_off = 0;
  if (k_ok) {
    const int k = g4_mine * 4;
    const int tap = k / a.Cin, ci = k - tap * a.Cin;
    kh = tap / a.ks;
    kwd = tap - kh * a.ks;
    k_off = (kh * a.Win + kwd) * a.Cin + ci;
  }
  const int nq = NS / 4;                 // float4 per dz row: 5 or 10
  const int dz_iters = (WG_MC * nq + nthreads - 1) / nthreads;

  auto rowinfo = [&](int c) {   // threads < MC
    if (tid < WG_MC) {
      int* inf = s_info + (c % (WG_NST + 1)) * 3 * WG_MC;
      const int m = m_begin + c * WG_MC + tid;
      if (c < nch && m < m_end) {
        const int n = m / hw_out, rem = m - n * hw_out;
        const int ho = rem / a.Wout, wo = rem - ho * a.Wout;
        const int h0 = ho * a.stride - a.pad, w0 = wo * a.stride - a.pad;
        inf[tid] = ((n * a.Hin + h0) * a.Win + w0) * a.Cin;   // element offset of the window origin (may be < 0)
        inf[WG_MC + tid] = h0;
        inf[2 * WG_MC + tid] = w0;
      } else {
        inf[tid] = 0;
        inf[WG_MC + tid] = -(1 << 20);
        inf[2 * WG_MC + tid] = -(1 << 20);
      }
    }
  };
  auto gather = [&](int c) {
    const int* inf = s_info + (c % (WG_NST + 1)) * 3 * WG_MC;
    float* sA = sbuf + (c % WG_NST) * stage_f;
    float* sG = sA + WG_MC * KS;
    const int m0 = m_begin + c * WG_MC;
#pragma unroll 4
    for (int pm = pm0; pm < WG_MC; pm += a.nw) {
      const int hi = inf[WG_MC + pm] + kh, wi = inf[2 * WG_MC + pm] + kwd;
      const bool ok = k_ok && (unsigned)hi < (unsigned)a.Hin && (unsigned)wi < (unsigned)a.Win;
      const float* src = ok ? a.x + (inf[pm] + k_off) : a.x;
      cp_async16(sA + pm * KS + gl * 4, src, ok ? 16 : 0);
    }
    for (int it = 0; it < dz_iters; ++it) {
      const int idx = tid + it * nthreads;
      if (idx < WG_MC * nq) {
        const int pm = idx / nq, q = idx - pm * nq;
        const int m = m0 + pm;
        const bool ok = (m < m_end) && (co_base + q * 4 < a.Cout);
        const float* src = ok ? a.dz + (size_t)m * a.Cout + co_base + q * 4 : a.dz;
        cp_async16(sG + pm * NS + q * 4, src, ok ? 16 : 0);
      }
    }
  };

  float acc[4][20];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int c = 0; c < 20; ++c) acc[i][c] = 0.f;

  for (int c = 0; c < WG_NST; ++c) rowinfo(c);
  __syncthreads();
#pragma unroll
  for (int st = 0; st < WG_NST - 1; ++st) {
    if (st < nch) gather(st);
    cp_async_commit();
  }
  for (int c = 0; c < nch; ++c) {
    cp_async_wait<WG_NST - 2>();
    __syncthreads();
    rowinfo(c + WG_NST);                       // consumed by the gather of the NEXT iteration
    if (c + WG_NST - 1 < nch) gather(c + WG_NST - 1);
    cp_async_commit();
    const float* pA = sbuf + (c % WG_NST) * stage_f + kwi * 128 + lane * 4;
    const float* pG = sbuf + (c % WG_NST) * stage_f + WG_MC * KS + nwi * 20;
#pragma unroll 4
    for (int pm = 0; pm < WG_MC; ++pm) {
      const float4 a4 = *reinterpret_cast<const float4*>(pA + pm * KS);
      float g[20];
#pragma unroll
      for (int j = 0; j < 5; ++j)
        *reinterpret_cast<float4*>(&g[4 * j]) = *reinterpret_cast<const float4*>(pG + pm * NS + 4 * j);
#pragma unroll
      for (int cc = 0; cc < 20; ++cc) {
        acc[0][cc] = fmaf(a4.x, g[cc], acc[0][cc]);
        acc[1][cc] = fmaf(a4.y, g[cc], acc[1][cc]);
        acc[2][cc] = fmaf(a4.z, g[cc], acc[2][cc]);
        acc[3][cc] = fmaf(a4.w, g[cc], acc[3][cc]);
      }
    }
  }
  cp_async_wait<0>();
  const int g4 = g4_base + kwi * 32 + lane;
  const int co = co_base + nwi * 20;
  if (g4 < a.k4_groups && co < a.Cout) {
    float* dst = a.part + ((size_t)blockIdx.z * a.k_total + (size_t)g4 * 4) * a.Cout + co;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 5; ++j)
        *reinterpret_cast<float4*>(dst + (size_t)i * a.Cout + 4 * j) =
            make_float4(acc[i][4 * j], acc[i][4 * j + 1], acc[i][4 * j + 2], acc[i][4 * j + 3]);
  }
}

// Stem weight gradient: dW[co][ci][kh][kw] over NCHW images.  A CTA owns a contiguous pixel range and
// walks it in chunks of 128 pixels: the chunk's im2col values sx[27][128] and gradients sdz[128][20] are
// staged in shared memory (coalesced), then 225 threads = 5 pixel slices x (9 taps x 5 channel quads)
// accumulate 3 ci x 4 co each; the slices meet in shared memory in fixed order and the CTA writes one
// partial [27][20].
constexpr int SW_LD = SW_PX + 4, SW_SLICES = 5;   // SW_PX: net_ws.cuh

__global__ void __launch_bounds__(256) stem_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dz,
                                                         float* __restrict__ part, int N, int H, int W, int M,
                                                         int pix_per_cta) {
  __shared__ __align__(16) float sx[27 * SW_LD];
  __shared__ __align__(16) float sdz[SW_PX * 20];
  const int tid = threadIdx.x;
  const int hw = H * W;
  const int m0 = blockIdx.x * pix_per_cta, m1 = min(M, m0 + pix_per_cta);
  const int slice = tid / 45, j = tid - slice * 45;
  const int tap = j / 5, cq = j - tap * 5;
  const bool worker = slice < SW_SLICES;
  const int pl = tid & (SW_PX - 1), k0 = tid >> 7;   // staging role: pixel pl, k = k0, k0 + 2, ...
  float acc[3][4];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[i][c] = 0.f;

  for (int mc = m0; mc < m1; mc += SW_PX) {
    __syncthreads();   // previous chunk fully consumed
    {
      const int m = mc + pl;
      const bool pok = m < m1;
      int n = 0, ho = 0, wo = 0;
      if (pok) {
        n = m / hw;
        const int rem = m - n * hw;
        ho = rem / W;
        wo = rem - ho * W;
      }
      float v[14];
#pragma unroll
      for (int it = 0; it < 14; ++it) {
        const int k = k0 + 2 * it;
        v[it] = 0.f;
        if (k < 27 && pok) {
          const int tp = k / 3, ci = k - tp * 3;
          const int kh = tp / 3, kw = tp - kh * 3;
          const int hi = ho + kh - 1, wi = wo + kw - 1;
          if ((unsigned)hi < (unsigned)H && (unsigned)wi < (unsigned)W)
            v[it] = __ldg(x + ((size_t)(n * 3 + ci) * H + hi) * W + wi);
        }
      }
#pragma unroll
      for (int it = 0; it < 14; ++it) {
        const int k = k0 + 2 * it;
        if (k < 27) sx[k * SW_LD + pl] = v[it];
      }
      const int nvec = SW_PX * 5;
      for (int idx = tid; idx < nvec; idx += 256) {
        const int pm = idx / 5;
        float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
        if (mc + pm < m1) g = __ldg(reinterpret_cast<const float4*>(dz + (size_t)mc * 20) + idx);
        reinterpret_cast<float4*>(sdz)[idx] = g;
      }
    }
    __syncthreads();
    if (worker) {
      const float* px = sx + tap * 3 * SW_LD;
#pragma unroll 2
      for (int p = slice; p < SW_PX; p += SW_SLICES) {
        const float4 g = *reinterpret_cast<const float4*>(sdz + p * 20 + cq * 4);
        const float x0 = px[p], x1 = px[SW_LD + p], x2 = px[2 * SW_LD + p];
        acc[0][0] = fmaf(x0, g.x, acc[0][0]); acc[0][1] = fmaf(x0, g.y, acc[0][1]);
        acc[0][2] = fmaf(x0, g.z, acc[0][2]); acc[0][3] = fmaf(x0, g.w, acc[0][3]);
        acc[1][0] = fmaf(x1, g.x, acc[1][0]); acc[1][1] = fmaf(x1, g.y, acc[1][1]);
        acc[1][2] = fmaf(x1, g.z, acc[1][2]); acc[1][3] = fmaf(x1, g.w, acc[1][3]);
        acc[2][0] = fmaf(x2, g.x, acc[2][0]); acc[2][1] = fmaf(x2, g.y, acc[2][1]);
        acc[2][2] = fmaf(x2, g.z, acc[2][2]); acc[2][3] = fmaf(x2, g.w, acc[2][3]);
      }
    }
  }
  __syncthreads();
  float* red = sx;   // [SLICES][540] = 2700 floats <= 27 * 132
  if (worker) {
#pragma unroll
    for (int ci = 0; ci < 3; ++ci)
#pragma unroll
      for (int c = 0; c < 4; ++c) red[slice * 540 + (tap * 3 + ci) * 20 + cq * 4 + c] = acc[ci][c];
  }
  __syncthreads();
  for (int e = tid; e < 540; e += 256) {
    float s = 0.f;
#pragma unroll
    for (int sl = 0; sl < SW_SLICES; ++sl) s += red[sl * 540 + e];
    part[(size_t)blockIdx.x * 540 + e] = s;
  }
}

// One launch reduces the partials of every conv layer and writes OIHW gradients.  A CTA owns EPB = 256 / SG
// consecutive gradient elements of one layer; its SG thread groups each sum every SG-th split (eight loads in
// flight, fixed association), the groups meet in shared memory in fixed order.  SG grows with the layer's
// split count so that no thread walks more than a few dozen partials.
struct WgFinalTable {
  int n;
  unsigned int n_blocks;
  struct {
    unsigned long long part_off;
    unsigned int w_off, blk_start;
    int splits, cin, cout, taps, sg_log2;
  } e[NET_MAX_CONV];
};

__global__ void __launch_bounds__(256) wgrad_finalize_kernel(WgFinalTable t, const float* __restrict__ part,
                                                             float* __restrict__ grads, int accumulate) {
  __shared__ float red[256];
  int l = 0;
  while (l + 1 < t.n && blockIdx.x >= t.e[l + 1].blk_start) ++l;
  const auto& L = t.e[l];
  const int SG = 1 << L.sg_log2, EPB = 256 >> L.sg_log2;
  const int el = threadIdx.x & (EPB - 1), sg = threadIdx.x >> (8 - L.sg_log2);
  const int K = L.cin * L.taps;
  const int total = K * L.cout;
  const int e = (int)(blockIdx.x - L.blk_start) * EPB + el;
  float s = 0.f;
  if (e < total) {
    const float* p = part + L.part_off + e;
    int sp = sg;
    for (; sp + 7 * SG < L.splits; sp += 8 * SG) {
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = __ldcs(p + (size_t)(sp + u * SG) * total);
      s += ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
    }
    for (; sp < L.splits; sp += SG) s += __ldcs(p + (size_t)sp * total);
  }
  red[threadIdx.x] = s;   // [sg][el]
  __syncthreads();
  if (sg == 0 && e < total) {
    float tot = 0.f;
    for (int g = 0; g < SG; ++g) tot += red[g * EPB + el];
    const int k = e / L.cout, co = e - k * L.cout;
    const int tap = k / L.cin, ci = k - tap * L.cin;
    float* dst = grads + L.w_off + ((size_t)co * L.cin + ci) * L.taps + tap;
    if (accumulate) *dst += tot; else *dst = tot;
  }
}

// ----------------------------------------------------------------------------- heads
// dpre = (dout - y * <y, dout>) / max(||pre||, eps),  y = pre / max(||pre||, eps)
__global__ void __launch_bounds__(256) l2norm_bwd_kernel(const float* __restrict__ pre, const float* __restrict__ dout,
                                                         float* __restrict__ dpre, int N, int d) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = blockIdx.x * 8 + warp;
  if (n >= N) return;
  const float* x = pre + (size_t)n * d;
  const float* g = dout + (size_t)n * d;
  float ss = 0.f, dot = 0.f;
  for (int i = lane; i < d; i += 32) {
    ss = fmaf(x[i], x[i], ss);
    dot = fmaf(x[i], g[i], dot);
  }
  ss = warp_sum(ss);
  dot = warp_sum(dot);
  const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
  const float ydot = dot * inv;  // <y, dout>
  for (int i = lane; i < d; i += 32) dpre[(size_t)n * d + i] = (g[i] - x[i] * inv * ydot) * inv;
}

// dX[n][i] = sum_o dY[n][o] * W[o][i]   (* 1[mask[n][i] > 0])
__global__ void __launch_bounds__(256) linear_bwd_x_kernel(const float* __restrict__ dY, const float* __restrict__ W,
                                                           const float* __restrict__ mask, float* __restrict__ dX, int N,
                                                           int in, int out) {
  extern __shared__ float sdy[];
  for (int n = blockIdx.x; n < N; n += gridDim.x) {
    __syncthreads();
    for (int o = threadIdx.x; o < out; o += blockDim.x) sdy[o] = dY[(size_t)n * out + o];
    __syncthreads();
    for (int i = threadIdx.x; i < in; i += blockDim.x) {
      float s = 0.f;
      for (int o = 0; o < out; ++o) s = fmaf(sdy[o], W[(size_t)o * in + i], s);
      if (mask && !(mask[(size_t)n * in + i] > 0.f)) s = 0.f;
      dX[(size_t)n * in + i] = s;
    }
  }
}

// dW[o][i] (+)= sum_n dY[n][o] * X[n][i];  db[o] (+)= sum_n dY[n][o]
__global__ void __launch_bounds__(256) linear_bwd_w_kernel(const float* __restrict__ dY, const float* __restrict__ X,
                                                           float* __restrict__ dW, float* __restrict__ db, int N, int in,
                                                           int out, int accumulate) {
  const int total = out * in;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    const int o = e / in, i = e - o * in;
    float s = 0.f;
    for (int n = 0; n < N; ++n) s = fmaf(dY[(size_t)n * out + o], X[(size_t)n * in + i], s);
    if (accumulate) dW[e] += s; else dW[e] = s;
    if (i == 0) {
      float b = 0.f;
      for (int n = 0; n < N; ++n) b += dY[(size_t)n * out + o];
      if (accumulate) db[o] += b; else db[o] = b;
    }
  }
}

// gradient of avg_pool2d(., 4) + NCHW flatten:  dA[n,h,w,c] = dfeat[n][(c*PH + h/4)*PW + w/4] / 16
__global__ void __launch_bounds__(256) pool_bwd_kernel(const float* __restrict__ dfeat, float* __restrict__ dA, int N,
                                                       int H, int W, int C, int PH, int PW) {
  const size_t total = (size_t)N * H * W * C;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    size_t t = i / C;
    const int w = (int)(t % W);
    t /= W;
    const int h = (int)(t % H), n = (int)(t / H);
    float v = 0.f;
    if (h < 4 * PH && w < 4 * PW) v = dfeat[(size_t)n * (C * PH * PW) + (c * PH + h / 4) * PW + w / 4] * 0.0625f;
    dA[i] = v;
  }
}

int linear_backward(const LinL& l, const float* params, float* grads, const float* X, const float* dY, const float* mask,
                    float* dX, int N, int accumulate, cudaStream_t stream) {
  int blocks = (l.in * l.out + 255) / 256;
  if (blocks > 4 * sm_count()) blocks = 4 * sm_count();
  B200OCL_PROF("head", 4.0 * ((double)N * l.in + (double)N * l.out + (double)l.in * l.out), stream);
  linear_bwd_w_kernel<<<blocks, 256, 0, stream>>>(dY, X, grads + l.w_off, grads + l.b_off, N, l.in, l.out, accumulate);
  B200OCL_LAUNCHED();
  if (dX) {
    B200OCL_PROF("head", 4.0 * ((double)N * l.in + (double)N * l.out + (double)l.in * l.out), stream);
    linear_bwd_x_kernel<<<N < 2 * sm_count() ? N : 2 * sm_count(), 256, l.out * sizeof(float), stream>>>(
        dY, params + l.w_off, mask, dX, N, l.in, l.out);
    B200OCL_LAUNCHED();
  }
  return B200OCL_OK;
}

}  // namespace
}  // namespace b200ocl

// Weight gradients leave the critical path: wgrad(i) only feeds the final reduction, while the chain
// BN-backward -> data gradient -> BN-backward ... is strictly serial and made of launches that fill a fraction of the
// GPU (a fraction of a wave).  So wgrad(i) is launched on a side stream, forked after the
// BN-backward that produced its dz and joined before the finalize; dz alternates between two buffers so that the next
// BN-backward does not wait for it.  Fork / join are events, captured as parallel branches when the call is recorded
// into a CUDA graph.  One side stream and four events per caller stream (bwd_async below), created on first use.
namespace b200ocl {
namespace {
struct BwdAsync {
  cudaStream_t side = nullptr;
  cudaStream_t owner = nullptr;   // the caller stream this slot serves
  cudaEvent_t ready[2] = {nullptr, nullptr}, done[2] = {nullptr, nullptr};
  int state = 0;   // 0 = free, 1 = usable, -1 = failed
};
constexpr int BWD_ASYNC_SLOTS = 4;
// One helper stream + four events per CALLER STREAM (up to four caller streams per device): two backward passes that the
// host runs concurrently on different streams (learners: SCR's two views) must not share fork / join events.  A fifth
// caller stream gets no helper (serial weight gradients).  Slots are created on the first eager call from a stream; calls
// recorded into CUDA graphs only need the events while capturing.
BwdAsync* bwd_async(cudaStream_t caller) {
  static BwdAsync per_dev[B200OCL_MAX_DEVICES][BWD_ASYNC_SLOTS];
  static int enabled = -1;
  if (enabled < 0) {
    const char* e = getenv("B200OCL_WG_ASYNC");
    enabled = (e && e[0] == '0') ? 0 : 1;
  }
  if (!enabled) return nullptr;
  BwdAsync* slots = per_dev[device_slot()];
  for (int i = 0; i < BWD_ASYNC_SLOTS; ++i)
    if (slots[i].state == 1 && slots[i].owner == caller) return &slots[i];
  for (int i = 0; i < BWD_ASYNC_SLOTS; ++i) {
    BwdAsync& a = slots[i];
    if (a.state != 0) continue;
    a.state = -1;
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);      // lo = least priority
    bool ok = cudaStreamCreateWithPriority(&a.side, cudaStreamNonBlocking, lo) == cudaSuccess;
    for (int j = 0; ok && j < 2; ++j)
      ok = cudaEventCreateWithFlags(&a.ready[j], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&a.done[j], cudaEventDisableTiming) == cudaSuccess;
    if (!ok) {
      (void)cudaGetLastError();
      return nullptr;
    }
    a.owner = caller;
    a.state = 1;
    return &a;
  }
  return nullptr;
}
}  // namespace
}  // namespace b200ocl

extern "C" int b200ocl_net_backward(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const float* x,
                                    const float* dout, int N, void* workspace, size_t workspace_bytes, int accumulate,
                                    void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(desc && st && st->params && st->grads && st->packed, "null descriptor/state pointer");
  NetPlan p;
  int rc = build_plan(*desc, p);
  if (rc) {
    set_error("b200ocl_net_backward: unsupported network description");
    return rc;
  }
  B200OCL_CHECK_ARG(N >= 1 && dout && x, "need N >= 1, x and dout");
  if ((rc = check_batch("b200ocl_net_backward", p, N))) return rc;
  if ((rc = check_workspace("b200ocl_net_backward", workspace, workspace_bytes,
                            b200ocl_net_train_workspace_bytes(desc, N)))) return rc;
  const int eval_stats = (accumulate >> 1) & 1;   // bit 1 of `accumulate`: backward of b200ocl_net_forward_evalgrad
  const int from_feat = (accumulate >> 2) & 1;    // bit 2: dout is dL/dfeatures [N, dim_in]; the head is skipped
  accumulate &= 1;
  const int sms = sm_count();
  TrainWs w = train_ws(p, N, workspace, sms);
  unsigned int* counters = w.counters + NET_COUNTERS / 2;
  B200OCL_CUDA(cudaMemsetAsync(counters, 0, (NET_COUNTERS / 2) * sizeof(unsigned int), stream));
  float* coef = reinterpret_cast<float*>(w.stat_part);                       // [3][C] at the front
  double* bn_part = w.stat_part + NET_COEF_DOUBLES;                           // partial sums behind the coefficients
  const int C_last = desc->nf * 8;

  // ---- heads: dout -> dfeat
  const float* dfeat = from_feat ? dout : w.dfeat;
  if (from_feat) {
    // the head's gradient entries are left as they are
  } else if (p.head == 0) {
    if ((rc = linear_backward(p.lin[0], st->params, st->grads, w.feat, dout, nullptr, w.dfeat, N, accumulate, stream))) return rc;
  } else {
    const float* pre = (p.head == 3) ? w.feat : w.proj;
    float* dpre = (p.head == 3) ? w.dfeat : w.dproj;
    B200OCL_PROF("head", 12.0 * N * p.out_dim, stream);
    l2norm_bwd_kernel<<<(N + 7) / 8, 256, 0, stream>>>(pre, dout, dpre, N, p.out_dim);
    B200OCL_LAUNCHED();
    if (p.head == 1) {
      if ((rc = linear_backward(p.lin[1], st->params, st->grads, w.feat, w.dproj, nullptr, w.dfeat, N, accumulate, stream))) return rc;
    } else if (p.head == 2) {
      if ((rc = linear_backward(p.lin[2], st->params, st->grads, w.hid, w.dproj, w.hid, w.dhid, N, accumulate, stream))) return rc;
      if ((rc = linear_backward(p.lin[1], st->params, st->grads, w.feat, w.dhid, nullptr, w.dfeat, N, accumulate, stream))) return rc;
    }
  }
  float* g0 = w.g0;
  float* g1 = w.g1;
  {
    const size_t total = (size_t)N * p.final_h * p.final_w * C_last;
    size_t blocks = (total + 255) / 256;
    if (blocks > (size_t)16 * sms) blocks = (size_t)16 * sms;
    B200OCL_PROF("pool", 8.0 * total, stream);
    pool_bwd_kernel<<<(unsigned)blocks, 256, 0, stream>>>(dfeat, g0, N, p.final_h, p.final_w, C_last, p.pooled_h,
                                                          p.pooled_w);
    B200OCL_LAUNCHED();
  }

  auto bn_backward = [&](int ci, const float* dA, const float* amask, float* dz, float* gout) -> int {
    const ConvL& c = p.conv[ci];
    const BnL& b = p.bn[ci];
    BnBwdArgs a{};
    a.dA = dA;
    a.amask = amask;
    a.z = w.z + (size_t)N * c.act_off;
    a.mean = w.save + b.save_off;
    a.invstd = w.save + b.save_off + b.c;
    a.gamma = st->params + b.g_off;
    a.M = N * c.hout * c.wout;
    a.C = c.cout;
    a.part = bn_part;
    a.counter = counters + ci;
    a.ready = counters + 4 * NET_MAX_CONV + ci;
    a.dgamma = st->grads + b.g_off;
    a.dbeta = st->grads + b.b_off;
    a.accumulate = accumulate;
    a.eval_stats = eval_stats;
    a.coef = coef;
    a.dz = dz;
    a.gout = gout;
    return launch_bn_bwd(a, stream);
  };
  auto wgrad_on = [&](int ci, const float* x, const float* dz, cudaStream_t stream) -> int {
    const ConvL& c = p.conv[ci];
    const WgradPlan wp = wgrad_plan(p, ci, N, sms);
    float* part = w.wg_part + w.wg_off[ci];
    if (wp.kernel == WGRAD_STEM) {
      const int M = N * p.in_h * p.in_w;
      B200OCL_PROF("wgrad", 2.0 * M * 540.0, stream);
      stem_wgrad_kernel<<<wp.splits, 256, 0, stream>>>(x, dz, part, N, p.in_h, p.in_w, M, wp.stem_ppc);
      B200OCL_LAUNCHED();
      return B200OCL_OK;
    }
    if (wp.kernel == WGRAD_TC) {
      const WgradTcCfg& tg = wp.tc;
      WgradTcArgs ta{};
      ta.x = x; ta.dz = dz;
      ta.part = part;
      ta.N = N; ta.H = c.hin; ta.W = c.win; ta.Cin = c.cin; ta.Cout = c.cout;
      ta.tpc = tg.tpc; ta.chains = tg.chains; ta.chains_per_cta = tg.chains_per_cta;
      return launch_wgrad_tc(ta, tg, stream);
    }
    const WgradCfg& g = wp.fp32;
    WgradArgs a{};
    a.x = x; a.dz = dz;
    a.part = part;
    a.N = N; a.Hin = c.hin; a.Win = c.win; a.Cin = c.cin;
    a.Hout = c.hout; a.Wout = c.wout; a.Cout = c.cout;
    a.ks = c.ks; a.stride = c.stride; a.pad = c.pad;
    a.M = N * c.hout * c.wout;
    a.k_total = g.k_total; a.k4_groups = g.k4_groups; a.kw = g.kw; a.nw = g.nw;
    a.pix_per_split = g.pix_per_split;
    const size_t smem = (size_t)WG_NST * WG_MC * (g.kw * 128 + g.nw * 20) * sizeof(float) +
                        (size_t)(WG_NST + 1) * 3 * WG_MC * sizeof(int);
    B200OCL_CUDA(raise_smem_limit<wgrad_kernel>(64 * 1024));
    B200OCL_PROF("wgrad", 2.0 * a.M * (double)a.k_total * a.Cout, stream);
    wgrad_kernel<<<dim3(g.grid_k, g.grid_n, g.splits), 32 * g.kw * g.nw, smem, stream>>>(a);
    B200OCL_LAUNCHED();
    return B200OCL_OK;
  };
  auto dgrad = [&](int ci, const float* dz, float* dx, int accum) -> int {
    ConvArgs a = conv_layer_args(p.conv[ci], N, dz, st->packed, dx, true);
    a.mode = accum ? CONV_ACCUM : CONV_RAW;
    return launch_conv(a, sms, stream);
  };

  // dz double buffer + fork / join (see bwd_async above)
  BwdAsync* as = g_prof_on ? nullptr : bwd_async(stream);   // per-launch profiling (bench.py) wants serial launches
  float* dzbuf[2] = {w.g2, w.g4};
  bool pending[2] = {false, false};
  int cur = 0;
  auto next_dz = [&]() -> float* {           // the buffer the next BN-backward writes: its last reader must be done
    if (as && pending[cur]) {
      if (cudaStreamWaitEvent(stream, as->done[cur], 0) != cudaSuccess) return nullptr;
      pending[cur] = false;
    }
    return dzbuf[cur];
  };
  auto wgrad = [&](int ci, const float* xin, const float* dz) -> int {
    if (!as) return wgrad_on(ci, xin, dz, stream);
    B200OCL_CUDA(cudaEventRecord(as->ready[cur], stream));
    B200OCL_CUDA(cudaStreamWaitEvent(as->side, as->ready[cur], 0));
    const int rcw = wgrad_on(ci, xin, dz, as->side);
    if (rcw) return rcw;
    B200OCL_CUDA(cudaEventRecord(as->done[cur], as->side));
    pending[cur] = true;
    cur ^= 1;
    return B200OCL_OK;
  };
  auto join_side = [&]() -> int {
    for (int i = 0; i < 2; ++i)
      if (as && pending[i]) {
        B200OCL_CUDA(cudaStreamWaitEvent(stream, as->done[i], 0));
        pending[i] = false;
      }
    return B200OCL_OK;
  };
  float* dz = nullptr;

  for (int b = 7; b >= 0; --b) {
    const BlockL& B = p.blk[b];
    const int prev = (b == 0) ? 0 : p.blk[b - 1].c2;
    const float* x_in = w.a + (size_t)N * p.conv[prev].act_off;
    const float* out_act = w.a + (size_t)N * p.conv[B.c2].act_off;
    const float* a1 = w.a + (size_t)N * p.conv[B.c1].act_off;
    // main branch, second conv
    if (!(dz = next_dz())) return B200OCL_ECUDA;
    if ((rc = bn_backward(B.c2, g0, out_act, dz, B.sc < 0 ? g1 : nullptr))) return rc;
    if ((rc = wgrad(B.c2, a1, dz))) return rc;
    if ((rc = dgrad(B.c2, dz, w.g3, 0))) return rc;
    // shortcut branch
    if (B.sc >= 0) {
      if (!(dz = next_dz())) return B200OCL_ECUDA;
      if ((rc = bn_backward(B.sc, g0, out_act, dz, nullptr))) return rc;
      if ((rc = wgrad(B.sc, x_in, dz))) return rc;
      if ((rc = dgrad(B.sc, dz, g1, 0))) return rc;
    }
    // main branch, first conv
    if (!(dz = next_dz())) return B200OCL_ECUDA;
    if ((rc = bn_backward(B.c1, w.g3, a1, dz, nullptr))) return rc;
    if ((rc = wgrad(B.c1, x_in, dz))) return rc;
    if ((rc = dgrad(B.c1, dz, g1, 1))) return rc;
    float* t = g0; g0 = g1; g1 = t;
  }
  // stem
  if (!(dz = next_dz())) return B200OCL_ECUDA;
  if ((rc = bn_backward(0, g0, w.a + (size_t)N * p.conv[0].act_off, dz, nullptr))) return rc;
  if ((rc = wgrad_on(0, x, dz, stream))) return rc;   // on the caller stream: nothing is left to overlap it with
  if ((rc = join_side())) return rc;                   // every weight-gradient partial is in place
  WgFinalTable t{};
  t.n = p.n_conv;
  unsigned int blocks = 0;
  for (int i = 0; i < p.n_conv; ++i) {
    auto& e = t.e[i];
    e.part_off = w.wg_off[i];
    e.w_off = (unsigned)p.conv[i].w_off;
    e.cin = p.conv[i].cin;
    e.cout = p.conv[i].cout;
    e.taps = p.conv[i].ks * p.conv[i].ks;
    e.splits = wgrad_plan(p, i, N, sms).splits;
    e.sg_log2 = e.splits >= 256 ? 5 : (e.splits >= 64 ? 4 : (e.splits >= 16 ? 3 : 2));
    e.blk_start = blocks;
    const int epb = 256 >> e.sg_log2;
    blocks += (unsigned)((e.cin * e.taps * e.cout + epb - 1) / epb);
  }
  t.n_blocks = blocks;
  B200OCL_PROF("wgrad_finalize", 8.0 * p.n_packed / 2, stream);
  wgrad_finalize_kernel<<<blocks, 256, 0, stream>>>(t, w.wg_part, st->grads, accumulate);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}
