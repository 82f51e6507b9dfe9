// conv.cu -- fp32 implicit-GEMM convolution for the Reduced-ResNet18 blocks (sm_90a).
//
// One kernel serves the forward 3x3 / 1x1 convolutions (stride 1 or 2), their eval-mode
// variant with BatchNorm folded into the epilogue (+ReLU, +residual), their train-mode variant
// that also produces the batch statistics, and the data-gradient convolutions (transposed
// gather, optional accumulate).  Replaces the cuDNN calls behind nn.Conv2d / nn.BatchNorm2d
// in reference models/resnet.py:11-12,20-36,73-74.
//
// fp32 on the CUDA cores, not TF32 tensor cores, on purpose: ASER ranks buffer samples by
// nearest neighbours in this network's feature space and the parity bar is bit-exact
// retrieved / evicted indices (BASELINE.json north_star); 10-bit-mantissa products move the
// features by ~1e-3 relative and reorder neighbours.  (The tensor-core kernels keep
// fp32 grade with a 3xTF32 split: conv_tc.cu, conv_tcp.cu.)
//
// Tiling: GEMM M = output pixels, N = output channels, K = taps x input channels.
//   CTA = 4 warps; a warp owns 32*PT pixels x 20 channels, a thread PT pixels x 20 channels
//   (lanes = consecutive pixels, so the 20 weights of a k are a broadcast LDS.128 x5 and the
//   activations a conflict-free LDS.128 per 4 k);  BN in {20,40,80} channels per CTA,
//   BM = (80/BN)*32*PT pixels;  K advances one (tap, 20-channel) chunk at a time through a
//   two-stage cp.async pipeline with zero-fill for the padding halo.
#include "conv.cuh"

namespace b200ocl {
namespace {

constexpr int CONV_THREADS = 128;

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL_MASK, v, o);
  return v;
}

// Pixel enumeration.  Default: m = (n, ho, wo) row-major.  With parity_order (stride-2 data gradient, even
// Hout / Wout): m = (class, n, ho/2, wo/2), class = 2*(ho&1) + (wo&1) -- a tile then holds pixels of one parity
// class, for which only the taps with kh = ho + pad (mod 2), kw = wo + pad (mod 2) contribute.
__device__ __forceinline__ void decode_pixel(const ConvArgs& a, int m, int& n, int& ho, int& wo) {
  if (a.parity_order) {
    const int hh = a.Hout >> 1, wh = a.Wout >> 1;
    const int mq = a.N * hh * wh;
    const int cls = m / mq;
    int idx = m - cls * mq;
    n = idx / (hh * wh);
    idx -= n * hh * wh;
    const int y = idx / wh;
    ho = 2 * y + (cls >> 1);
    wo = 2 * (idx - y * wh) + (cls & 1);
  } else {
    const int hw_out = a.Hout * a.Wout;
    n = m / hw_out;
    const int rem = m - n * hw_out;
    ho = rem / a.Wout;
    wo = rem - ho * a.Wout;
  }
}
// Taps a tile of pixels [m0, m0 + bm) can use, as a packed list: nibble i = i-th usable tap, count in `n`.
__device__ __forceinline__ unsigned long long tile_tap_list(const ConvArgs& a, int m0, int bm, int& n) {
  unsigned long long list = 0;
  n = 0;
  if (!a.parity_order) {
    n = a.ks * a.ks;
    return 0x876543210ull;
  }
  const int mq = a.N * (a.Hout >> 1) * (a.Wout >> 1);
  const int c0 = m0 / mq, c1 = min(m0 + bm - 1, a.M - 1) / mq;
  for (int kh = 0; kh < a.ks; ++kh)
    for (int kw = 0; kw < a.ks; ++kw) {
      bool live = false;
      for (int cls = c0; cls <= c1; ++cls)
        live = live || ((((cls >> 1) + a.pad - kh) & 1) == 0 && (((cls & 1) + a.pad - kw) & 1) == 0);
      if (live) list |= (unsigned long long)(kh * a.ks + kw) << (4 * n++);
    }
  return list;
}

// Shared epilogue: thread holds acc[PT][20] for rows r = row_base + 32*p (p < PT) and
// channels n0 + wn*20 .. +19.  `scratch` is >= 4*20*2 doubles of shared memory, free to use.
template <int BN, int PT, int WM = 4 / (BN / 20)>
__device__ __forceinline__ void conv_epilogue(const ConvArgs& a, float (&acc)[PT][20], const int (&mrow)[PT], int n0,
                                              int wm, int wn, int lane, int tid, double* scratch,
                                              bool participates = true) {
  const int cbase = n0 + wn * 20;
  if (a.mode == CONV_EVAL) {
    if (!participates) return;
    float sc[20], mu[20], be[20];
#pragma unroll
    for (int c = 0; c < 20; ++c) {
      const float inv = 1.0f / sqrtf(a.rvar[cbase + c] + a.eps);
      sc[c] = inv * a.gamma[cbase + c];
      mu[c] = a.rmean[cbase + c];
      be[c] = a.beta[cbase + c];
    }
#pragma unroll
    for (int p = 0; p < PT; ++p) {
      const int m = mrow[p];
      if (m < 0) continue;
      float* o = a.out + (size_t)m * a.CN + cbase;
      const float* rs = a.residual ? a.residual + (size_t)m * a.CN + cbase : nullptr;
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        float4 v;
        v.x = (acc[p][4 * j + 0] - mu[4 * j + 0]) * sc[4 * j + 0] + be[4 * j + 0];
        v.y = (acc[p][4 * j + 1] - mu[4 * j + 1]) * sc[4 * j + 1] + be[4 * j + 1];
        v.z = (acc[p][4 * j + 2] - mu[4 * j + 2]) * sc[4 * j + 2] + be[4 * j + 2];
        v.w = (acc[p][4 * j + 3] - mu[4 * j + 3]) * sc[4 * j + 3] + be[4 * j + 3];
        if (rs) {
          const float4 r4 = *reinterpret_cast<const float4*>(rs + 4 * j);
          v.x += r4.x; v.y += r4.y; v.z += r4.z; v.w += r4.w;
        }
        if (a.relu) {
          v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
        }
        *reinterpret_cast<float4*>(o + 4 * j) = v;
      }
    }
    return;
  }
  // RAW / TRAIN / ACCUM: store (or add) the accumulators
#pragma unroll
  for (int p = 0; p < PT; ++p) {
    const int m = mrow[p];
    if (m < 0 || !participates) continue;
    float* o = a.out + (size_t)m * a.CN + cbase;
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      float4 v = make_float4(acc[p][4 * j], acc[p][4 * j + 1], acc[p][4 * j + 2], acc[p][4 * j + 3]);
      if (a.mode == CONV_ACCUM) {
        const float4 old = *reinterpret_cast<const float4*>(o + 4 * j);
        v.x += old.x; v.y += old.y; v.z += old.z; v.w += old.w;
      }
      *reinterpret_cast<float4*>(o + 4 * j) = v;
    }
  }
  if (a.mode != CONV_TRAIN) return;

  // ---- batch statistics: fp64 sums, fixed order (thread -> warp shuffle -> warps -> CTAs)
  double* s_stat = scratch;  // [WM][BN][2]
#pragma unroll
  for (int c = 0; c < 20; ++c) {
    double s = 0.0, q = 0.0;
#pragma unroll
    for (int p = 0; p < PT; ++p) {
      if (mrow[p] >= 0 && participates) {
        const double v = (double)acc[p][c];
        s += v;
        q += v * v;
      }
    }
    s = warp_sum_d(s);
    q = warp_sum_d(q);
    if (lane == 0 && participates) {
      s_stat[((wm * BN) + wn * 20 + c) * 2 + 0] = s;
      s_stat[((wm * BN) + wn * 20 + c) * 2 + 1] = q;
    }
  }
  __syncthreads();
  if (tid < BN) {
    double s = 0.0, q = 0.0;
#pragma unroll
    for (int w = 0; w < WM; ++w) {
      s += s_stat[((w * BN) + tid) * 2 + 0];
      q += s_stat[((w * BN) + tid) * 2 + 1];
    }
    double* dst = a.stat_part + ((size_t)blockIdx.x * a.CN + n0 + tid) * 2;
    dst[0] = s;
    dst[1] = q;
  }
  __threadfence();
  __syncthreads();
  __shared__ bool is_last;
  if (tid == 0) is_last = (atomicAdd(a.counter + blockIdx.y, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // all 128 threads: channel = tid % BN, CTA-partials strided by 128/BN groups, then fixed-order combine
  constexpr int GROUPS = CONV_THREADS / BN;  // 6, 3 or 1
  const int ch = tid % BN, grp = tid / BN;
  double s = 0.0, q = 0.0;
  if (grp < GROUPS) {
    unsigned int b = grp;
    for (; b + 7 * GROUPS < gridDim.x; b += 8 * GROUPS) {      // eight loads in flight, fixed association
      double2 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u)
        v[u] = __ldcg(reinterpret_cast<const double2*>(a.stat_part + ((size_t)(b + u * GROUPS) * a.CN + n0 + ch) * 2));
      s += ((v[0].x + v[1].x) + (v[2].x + v[3].x)) + ((v[4].x + v[5].x) + (v[6].x + v[7].x));
      q += ((v[0].y + v[1].y) + (v[2].y + v[3].y)) + ((v[4].y + v[5].y) + (v[6].y + v[7].y));
    }
    for (; b < gridDim.x; b += GROUPS) {
      const double2 v = __ldcg(reinterpret_cast<const double2*>(a.stat_part + ((size_t)b * a.CN + n0 + ch) * 2));
      s += v.x;
      q += v.y;
    }
  }
  __syncthreads();  // s_stat reuse
  double* s_fin = scratch;  // [GROUPS][BN][2]
  if (grp < GROUPS) {
    s_fin[(grp * BN + ch) * 2 + 0] = s;
    s_fin[(grp * BN + ch) * 2 + 1] = q;
  }
  __syncthreads();
  if (tid < BN) {
    double S = 0.0, Q = 0.0;
    for (int g = 0; g < GROUPS; ++g) {
      S += s_fin[(g * BN + tid) * 2 + 0];
      Q += s_fin[(g * BN + tid) * 2 + 1];
    }
    bn_finalize(a, n0 + tid, S, Q);
  }
}

template <int BN, int PT>
__global__ void __launch_bounds__(CONV_THREADS, (PT <= 2 ? 4 : 3)) conv_kernel(ConvArgs a) {
  constexpr int WN = BN / 20, WM = 4 / WN, BM = WM * 32 * PT;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int NST = 3;
  float* sA = reinterpret_cast<float*>(smem_raw);  // [NST][BM][20]
  float* sB = sA + NST * BM * 20;                  // [NST][20][BN]
  int* s_base = reinterpret_cast<int*>(sB + NST * 20 * BN);
  int* s_h0 = s_base + BM;
  int* s_w0 = s_h0 + BM;
  int* s_m = s_w0 + BM;   // real (row-major) pixel index of each tile row, -1 past the end

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp / WN, wn = warp % WN;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;

  for (int r = tid; r < BM; r += CONV_THREADS) {
    const int m = m0 + r;
    if (m < a.M) {
      int n, ho, wo;
      decode_pixel(a, m, n, ho, wo);
      s_base[r] = n * a.Hin * a.Win;
      s_h0[r] = a.transposed ? ho + a.pad : ho * a.stride - a.pad;
      s_w0[r] = a.transposed ? wo + a.pad : wo * a.stride - a.pad;
      s_m[r] = (n * a.Hout + ho) * a.Wout + wo;
    } else {
      s_base[r] = 0;
      s_h0[r] = -(1 << 20);
      s_w0[r] = -(1 << 20);
      s_m[r] = -1;
    }
  }
  __syncthreads();

  const int cpk = a.CK / 20;
  int ntaps;
  const unsigned long long tap_list = tile_tap_list(a, m0, BM, ntaps);
  const int nchunks = ntaps * cpk;

  auto load_chunk = [&](int c, int buf) {
    const int ti = c / cpk, ci0 = (c - ti * cpk) * 20;
    const int tap = (int)((tap_list >> (4 * ti)) & 15ull);
    const int kh = tap / a.ks, kw = tap - kh * a.ks;
    float* dA = sA + buf * BM * 20;
    for (int r = tid; r < BM; r += CONV_THREADS) {   // one thread stages a whole 80-byte row
      int hi, wi;
      bool ok;
      if (!a.transposed) {
        hi = s_h0[r] + kh;
        wi = s_w0[r] + kw;
        ok = (unsigned)hi < (unsigned)a.Hin && (unsigned)wi < (unsigned)a.Win;
      } else {
        const int th = s_h0[r] - kh, tw = s_w0[r] - kw;
        ok = (th >= 0) && (tw >= 0);
        if (a.stride == 2) {
          ok = ok && (((th | tw) & 1) == 0);
          hi = th >> 1;
          wi = tw >> 1;
        } else {
          hi = th;
          wi = tw;
        }
        ok = ok && hi < a.Hin && wi < a.Win;
      }
      const float* src = ok ? a.in + ((size_t)(s_base[r] + hi * a.Win + wi) * a.CK + ci0) : a.in;
      const int nb = ok ? 16 : 0;
      float* dst = dA + r * 20;
#pragma unroll
      for (int q = 0; q < 5; ++q) cp_async16(dst + q * 4, ok ? src + q * 4 : src, nb);
    }
    float* dB = sB + buf * 20 * BN;
    const float* wsrc = a.w + ((size_t)(a.flip ? a.ks * a.ks - 1 - tap : tap) * a.CK + ci0) * a.CN + n0;
    for (int idx = tid; idx < 20 * (BN / 4); idx += CONV_THREADS) {
      const int kk = idx / (BN / 4), q = idx - kk * (BN / 4);
      cp_async16(dB + kk * BN + q * 4, wsrc + (size_t)kk * a.CN + q * 4, 16);
    }
  };

  float acc[PT][20];
#pragma unroll
  for (int p = 0; p < PT; ++p)
#pragma unroll
    for (int c = 0; c < 20; ++c) acc[p][c] = 0.f;

  const int row_base = wm * 32 * PT + lane;
#pragma unroll
  for (int st = 0; st < NST - 1; ++st) {
    if (st < nchunks) load_chunk(st, st);
    cp_async_commit();
  }
  for (int c = 0; c < nchunks; ++c) {
    const int buf = c % NST;
    cp_async_wait<NST - 2>();
    __syncthreads();
    if (c + NST - 1 < nchunks) load_chunk(c + NST - 1, (c + NST - 1) % NST);
    cp_async_commit();
    const float* pA = sA + buf * BM * 20 + row_base * 20;
    const float* pB = sB + buf * 20 * BN + wn * 20;
#pragma unroll
    for (int k4 = 0; k4 < 5; ++k4) {
      float4 av[PT];
#pragma unroll
      for (int p = 0; p < PT; ++p) av[p] = *reinterpret_cast<const float4*>(pA + p * 32 * 20 + k4 * 4);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        float w[20];
#pragma unroll
        for (int j = 0; j < 5; ++j)
          *reinterpret_cast<float4*>(&w[4 * j]) = *reinterpret_cast<const float4*>(pB + (k4 * 4 + kk) * BN + 4 * j);
#pragma unroll
        for (int p = 0; p < PT; ++p) {
          const float x = kk == 0 ? av[p].x : (kk == 1 ? av[p].y : (kk == 2 ? av[p].z : av[p].w));
#pragma unroll
          for (int cc = 0; cc < 20; ++cc) acc[p][cc] = fmaf(x, w[cc], acc[p][cc]);
        }
      }
    }
  }
  cp_async_wait<0>();
  __syncthreads();
  int mrow[PT];
#pragma unroll
  for (int p = 0; p < PT; ++p) mrow[p] = s_m[row_base + 32 * p];
  __syncthreads();   // s_m read before the epilogue reuses the front of shared memory
  conv_epilogue<BN, PT>(a, acc, mrow, n0, wm, wn, lane, tid, reinterpret_cast<double*>(smem_raw));
}

// Stem: 3 -> 20 channels, 3x3, stride 1, pad 1, NCHW input read directly (no layout pass).
// One thread per output pixel, 27 x 20 weights broadcast from shared memory.
__global__ void __launch_bounds__(CONV_THREADS) stem_kernel(ConvArgs a) {
  __shared__ __align__(16) float sW[27 * 20];
  __shared__ __align__(16) double scratch[4 * 20 * 2 * 2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < 27 * 20; i += CONV_THREADS) sW[i] = a.w[i];
  __syncthreads();
  const int m0 = blockIdx.x * CONV_THREADS;
  const int m = m0 + tid;
  float acc[1][20];
#pragma unroll
  for (int c = 0; c < 20; ++c) acc[0][c] = 0.f;
  if (m < a.M) {
    const int hw = a.Hin * a.Win;
    const int n = m / hw, rem = m - n * hw;
    const int ho = rem / a.Win, wo = rem - ho * a.Win;
    const float* xin = a.in + (size_t)n * 3 * hw;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int hi = ho + kh - 1;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int wi = wo + kw - 1;
        const bool ok = (unsigned)hi < (unsigned)a.Hin && (unsigned)wi < (unsigned)a.Win;
#pragma unroll
        for (int ci = 0; ci < 3; ++ci) {
          const float x = ok ? __ldg(xin + (size_t)ci * hw + hi * a.Win + wi) : 0.f;
          const float* w = sW + ((kh * 3 + kw) * 3 + ci) * 20;
#pragma unroll
          for (int j = 0; j < 5; ++j) {
            const float4 w4 = *reinterpret_cast<const float4*>(w + 4 * j);
            acc[0][4 * j + 0] = fmaf(x, w4.x, acc[0][4 * j + 0]);
            acc[0][4 * j + 1] = fmaf(x, w4.y, acc[0][4 * j + 1]);
            acc[0][4 * j + 2] = fmaf(x, w4.z, acc[0][4 * j + 2]);
            acc[0][4 * j + 3] = fmaf(x, w4.w, acc[0][4 * j + 3]);
          }
        }
      }
    }
  }
  // BN = 20, PT = 1: warp w owns rows 32*w + lane  (WM = 4, WN = 1)
  const int mrow[1] = {m < a.M ? m : -1};
  conv_epilogue<20, 1>(a, acc, mrow, 0, warp, 0, lane, tid, scratch);
}


// Small-M variant: when the pixel count cannot fill the GPU the K loop is the critical path
// (72 chunks for the 160-channel layers).  Here a CTA owns only 32*PT pixels x 20 channels and its
// four warps each take every fourth (tap, 20-channel) chunk; partial sums meet in shared memory in
// warp order (deterministic) and warp 0 runs the epilogue.  4x shorter dependency chain, 4-8x more CTAs.
template <int PT, int KS>
__global__ void __launch_bounds__(32 * KS, (KS == 4 ? 4 : 1)) conv_ksplit_kernel(ConvArgs a) {
  constexpr int BM = 32 * PT, BN = 20, THREADS = 32 * KS;
  constexpr int NST = (PT == 1 && KS == 4) ? 4 : 3;   // cp.async ring depth: the per-iteration math is shorter than one L2 round trip
  constexpr int SLOT = BM * 20 + 20 * BN;  // floats per (stage, k-slot): A chunk then B chunk
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* sbuf = reinterpret_cast<float*>(smem_raw);              // [NST][KS][SLOT]
  int* s_base = reinterpret_cast<int*>(sbuf + NST * KS * SLOT);  // [BM]
  int* s_h0 = s_base + BM;
  int* s_w0 = s_h0 + BM;
  int* s_m = s_w0 + BM;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  for (int r = tid; r < BM; r += THREADS) {
    const int m = m0 + r;
    if (m < a.M) {
      int n, ho, wo;
      decode_pixel(a, m, n, ho, wo);
      s_base[r] = n * a.Hin * a.Win;
      s_h0[r] = a.transposed ? ho + a.pad : ho * a.stride - a.pad;
      s_w0[r] = a.transposed ? wo + a.pad : wo * a.stride - a.pad;
      s_m[r] = (n * a.Hout + ho) * a.Wout + wo;
    } else {
      s_base[r] = 0;
      s_h0[r] = -(1 << 20);
      s_w0[r] = -(1 << 20);
      s_m[r] = -1;
    }
  }
  __syncthreads();
  const int cpk = a.CK / 20;
  int ntaps;
  const unsigned long long tap_list = tile_tap_list(a, m0, BM, ntaps);
  const int nchunks = ntaps * cpk;
  const int niter = (nchunks + KS - 1) / KS;

  // all threads stage the (up to) KS chunks of iteration `it` into stage `buf`: one (chunk, pixel row) pair
  // per thread and trip, so the staging is as wide as the CTA
  auto load_iter = [&](int it, int buf) {
    for (int idx = tid; idx < KS * BM; idx += THREADS) {
      const int slot = idx / BM, r = idx - slot * BM;
      const int c = it * KS + slot;
      if (c >= nchunks) continue;
      const int ti = c / cpk, ci0 = (c - ti * cpk) * 20;
      const int tap = (int)((tap_list >> (4 * ti)) & 15ull);
      const int kh = tap / a.ks, kw = tap - kh * a.ks;
      int hi, wi;
      bool ok;
      if (!a.transposed) {
        hi = s_h0[r] + kh;
        wi = s_w0[r] + kw;
        ok = (unsigned)hi < (unsigned)a.Hin && (unsigned)wi < (unsigned)a.Win;
      } else {
        const int th = s_h0[r] - kh, tw = s_w0[r] - kw;
        ok = (th >= 0) && (tw >= 0);
        if (a.stride == 2) {
          ok = ok && (((th | tw) & 1) == 0);
          hi = th >> 1;
          wi = tw >> 1;
        } else {
          hi = th;
          wi = tw;
        }
        ok = ok && hi < a.Hin && wi < a.Win;
      }
      const float* src = ok ? a.in + ((size_t)(s_base[r] + hi * a.Win + wi) * a.CK + ci0) : a.in;
      const int nb = ok ? 16 : 0;
      float* dst = sbuf + (buf * KS + slot) * SLOT + r * 20;
#pragma unroll
      for (int q = 0; q < 5; ++q) cp_async16(dst + q * 4, ok ? src + q * 4 : src, nb);
    }
    for (int idx = tid; idx < KS * 100; idx += THREADS) {
      const int slot = idx / 100, rem = idx - slot * 100;
      const int c = it * KS + slot;
      if (c >= nchunks) continue;
      const int ti = c / cpk, ci0 = (c - ti * cpk) * 20;
      const int tap = (int)((tap_list >> (4 * ti)) & 15ull);
      const int kk = rem / 5, q = rem - kk * 5;
      const float* wsrc = a.w + ((size_t)(a.flip ? a.ks * a.ks - 1 - tap : tap) * a.CK + ci0) * a.CN + n0;
      cp_async16(sbuf + (buf * KS + slot) * SLOT + BM * 20 + kk * BN + q * 4, wsrc + (size_t)kk * a.CN + q * 4, 16);
    }
  };

  float acc[PT][20];
#pragma unroll
  for (int p = 0; p < PT; ++p)
#pragma unroll
    for (int c = 0; c < 20; ++c) acc[p][c] = 0.f;

#pragma unroll
  for (int st = 0; st < NST - 1; ++st) {
    if (st < niter) load_iter(st, st);
    cp_async_commit();
  }
  for (int it = 0; it < niter; ++it) {
    const int buf = it % NST;
    cp_async_wait<NST - 2>();
    __syncthreads();   // stage `it` has landed; stage (it-1) is free for the prefetch below
    if (it + NST - 1 < niter) load_iter(it + NST - 1, (it + NST - 1) % NST);
    cp_async_commit();
    if (it * KS + warp < nchunks) {
      const float* pA = sbuf + (buf * KS + warp) * SLOT + lane * 20;
      const float* pB = sbuf + (buf * KS + warp) * SLOT + BM * 20;
#pragma unroll
      for (int k4 = 0; k4 < 5; ++k4) {
        float4 av[PT];
#pragma unroll
        for (int p = 0; p < PT; ++p) av[p] = *reinterpret_cast<const float4*>(pA + p * 32 * 20 + k4 * 4);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          float w[20];
#pragma unroll
          for (int j = 0; j < 5; ++j)
            *reinterpret_cast<float4*>(&w[4 * j]) = *reinterpret_cast<const float4*>(pB + (k4 * 4 + kk) * BN + 4 * j);
#pragma unroll
          for (int p = 0; p < PT; ++p) {
            const float x = kk == 0 ? av[p].x : (kk == 1 ? av[p].y : (kk == 2 ? av[p].z : av[p].w));
#pragma unroll
            for (int cc = 0; cc < 20; ++cc) acc[p][cc] = fmaf(x, w[cc], acc[p][cc]);
          }
        }
      }
    }
  }
  cp_async_wait<0>();
  __syncthreads();
  // fixed-order combine of the KS K-partials: warps 1.. publish, warp 0 adds them in warp order
  float* red = sbuf;  // [KS-1][BM][20]  (all staging buffers are free now)
  if (warp > 0) {
#pragma unroll
    for (int p = 0; p < PT; ++p)
#pragma unroll
      for (int j = 0; j < 5; ++j)
        *reinterpret_cast<float4*>(red + ((warp - 1) * BM + lane + 32 * p) * 20 + 4 * j) =
            make_float4(acc[p][4 * j], acc[p][4 * j + 1], acc[p][4 * j + 2], acc[p][4 * j + 3]);
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int w = 0; w < KS - 1; ++w)
#pragma unroll
      for (int p = 0; p < PT; ++p)
#pragma unroll
        for (int j = 0; j < 5; ++j) {
          const float4 v = *reinterpret_cast<const float4*>(red + (w * BM + lane + 32 * p) * 20 + 4 * j);
          acc[p][4 * j] += v.x; acc[p][4 * j + 1] += v.y; acc[p][4 * j + 2] += v.z; acc[p][4 * j + 3] += v.w;
        }
  }
  __syncthreads();
  int mrow[PT];
#pragma unroll
  for (int p = 0; p < PT; ++p) mrow[p] = s_m[lane + 32 * p];
  __syncthreads();
  conv_epilogue<20, PT, 1>(a, acc, mrow, n0, 0, 0, lane, tid, reinterpret_cast<double*>(smem_raw), warp == 0);
}

template <int PT, int KS>
int launch_conv_ksplit(const ConvArgs& a, const ConvPlan& pl, cudaStream_t stream) {
  constexpr int BM = 32 * PT;
  constexpr int NST = (PT == 1 && KS == 4) ? 4 : 3;
  constexpr size_t smem = (size_t)(NST * KS * (BM * 20 + 400)) * sizeof(float) + 4 * BM * sizeof(int);
  B200OCL_CUDA((raise_smem_limit<conv_ksplit_kernel<PT, KS>>(smem)));
  dim3 grid(pl.grid_x, pl.grid_y);
  B200OCL_PROF(a.transposed ? "conv_dgrad" : (a.mode == CONV_EVAL ? "conv_eval" : "conv_train"),
               2.0 * a.M * (double)a.CN * a.CK * a.ks * a.ks, stream);
  conv_ksplit_kernel<PT, KS><<<grid, 32 * KS, smem, stream>>>(a);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}


// Direct ("patch") variant for the forward 3x3 / 1x1 convolutions and the stride-1 data gradients:
// a CTA owns a spatial tile of TI images x TH x TW output pixels and stages, per 20-channel slice of
// the input, the input patch WITH its halo once (zero-filled outside the image) together with the
// weights of all taps; the taps then read the same shared-memory patch at shifted offsets.  Compared
// with the gather kernel above this removes the per-tap re-gather (9x less L2 traffic and address
// arithmetic) and all but two barriers per 20 input channels.  flip = 1 turns it into the stride-1
// data gradient (correlation with the spatially flipped taps of the [tap][cout][cin] weights).
template <int BN, int PT>
__global__ void __launch_bounds__(CONV_THREADS, (PT <= 2 ? 3 : 2)) conv_patch_kernel(ConvArgs a) {
  static_assert(PT == 1 || PT == 2 || PT == 4, "pixels per thread");
  constexpr int WN = BN / 20;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ __align__(16) double scratch[4 * 20 * 2 * 2];
  const int taps = a.ks * a.ks;
  const int PH = (a.th - 1) * a.stride + a.ks, PW = (a.tw - 1) * a.stride + a.ks;
  const int prows = a.ti * PH * PW;
  float* spatch = reinterpret_cast<float*>(smem_raw);   // [prows][20]
  float* sW = spatch + prows * 20;                      // [taps*20][BN]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp / WN, wn = warp % WN;
  const int n0 = blockIdx.y * BN;
  int t = blockIdx.x;
  const int tiles_x = (a.Wout + a.tw - 1) / a.tw, tiles_y = (a.Hout + a.th - 1) / a.th;
  const int tx_i = t % tiles_x;
  t /= tiles_x;
  const int ty_i = t % tiles_y;
  const int img0 = (t / tiles_y) * a.ti;
  const int x0 = tx_i * a.tw, y0 = ty_i * a.th;
  const int iy0 = y0 * a.stride - a.pad, ix0 = x0 * a.stride - a.pad;

  int mrow[PT], prow0[PT];
#pragma unroll
  for (int p = 0; p < PT; ++p) {
    const int r = wm * 32 * PT + lane + 32 * p;   // wm < 4 / WN pixel-warps
    const int img = r / (a.th * a.tw), rem = r - img * (a.th * a.tw);
    const int y = rem / a.tw, x = rem - y * a.tw;
    const bool valid = (img < a.ti) && (img0 + img < a.N) && (y0 + y < a.Hout) && (x0 + x < a.Wout);
    mrow[p] = valid ? ((img0 + img) * a.Hout + y0 + y) * a.Wout + x0 + x : -1;
    prow0[p] = (img < a.ti) ? (img * PH + y * a.stride) * PW + x * a.stride : 0;
  }

  float acc[PT][20];
#pragma unroll
  for (int p = 0; p < PT; ++p)
#pragma unroll
    for (int c = 0; c < 20; ++c) acc[p][c] = 0.f;

  const int nslices = a.CK / 20;
  for (int cc = 0; cc < nslices; ++cc) {
    __syncthreads();  // previous slice fully consumed
    for (int row = tid; row < prows; row += CONV_THREADS) {
      const int img = row / (PH * PW), rr = row - img * (PH * PW);
      const int py = rr / PW, px = rr - py * PW;
      const int iy = iy0 + py, ix = ix0 + px;
      const bool ok = (img0 + img < a.N) && (unsigned)iy < (unsigned)a.Hin && (unsigned)ix < (unsigned)a.Win;
      const float* src = ok ? a.in + ((size_t)((img0 + img) * a.Hin + iy) * a.Win + ix) * a.CK + cc * 20 : a.in;
      const int nb = ok ? 16 : 0;
      float* dst = spatch + row * 20;
#pragma unroll
      for (int q = 0; q < 5; ++q) cp_async16(dst + q * 4, ok ? src + q * 4 : src, nb);
    }
    for (int idx = tid; idx < taps * 20 * (BN / 4); idx += CONV_THREADS) {
      const int row = idx / (BN / 4), q = idx - row * (BN / 4);
      const int tap = row / 20, kk = row - tap * 20;
      const int wt = a.flip ? taps - 1 - tap : tap;
      cp_async16(sW + row * BN + q * 4, a.w + ((size_t)wt * a.CK + cc * 20 + kk) * a.CN + n0 + q * 4, 16);
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    for (int tap = 0; tap < taps; ++tap) {
      const int kh = tap / a.ks, kw = tap - kh * a.ks;
      const float* pA = spatch + (kh * PW + kw) * 20;
      const float* pB = sW + tap * 20 * BN + wn * 20;
#pragma unroll
      for (int k4 = 0; k4 < 5; ++k4) {
        float4 av[PT];
#pragma unroll
        for (int p = 0; p < PT; ++p) av[p] = *reinterpret_cast<const float4*>(pA + prow0[p] * 20 + k4 * 4);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          float w[20];
#pragma unroll
          for (int j = 0; j < 5; ++j)
            *reinterpret_cast<float4*>(&w[4 * j]) = *reinterpret_cast<const float4*>(pB + (k4 * 4 + kk) * BN + 4 * j);
#pragma unroll
          for (int p = 0; p < PT; ++p) {
            const float x = kk == 0 ? av[p].x : (kk == 1 ? av[p].y : (kk == 2 ? av[p].z : av[p].w));
#pragma unroll
            for (int cc2 = 0; cc2 < 20; ++cc2) acc[p][cc2] = fmaf(x, w[cc2], acc[p][cc2]);
          }
        }
      }
    }
  }
  conv_epilogue<BN, PT>(a, acc, mrow, n0, wm, wn, lane, tid, scratch);
}

struct PatchTile {
  int th, tw, ti;
  long ctas;
  size_t smem;
};

// Spatial tile of bm = 32*PT*WM output pixels: widest power-of-two strip of a row (<= 32), then rows,
// then images.
inline PatchTile patch_tile(const ConvArgs& a, int bn, int pt) {
  PatchTile t{};
  const int bm = (80 / bn) * 32 * pt;
  int tw = 1;
  while (tw * 2 <= a.Wout && tw < 32) tw *= 2;
  if (tw > bm) tw = bm;
  int hp = 1;
  while (hp < a.Hout) hp *= 2;
  int th = bm / tw;
  if (th > hp) th = hp;
  t.tw = tw; t.th = th; t.ti = bm / (tw * th);
  const int PH = (th - 1) * a.stride + a.ks, PW = (tw - 1) * a.stride + a.ks;
  const long tiles = (long)((a.N + t.ti - 1) / t.ti) * ((a.Hout + th - 1) / th) * ((a.Wout + tw - 1) / tw);
  t.ctas = tiles * (a.CN / bn);
  t.smem = ((size_t)t.ti * PH * PW * 20 + (size_t)a.ks * a.ks * 20 * bn) * sizeof(float);
  return t;
}

template <int BN, int PT>
int launch_conv_patch(ConvArgs a, const ConvPlan& pl, cudaStream_t stream) {
  a.th = pl.th; a.tw = pl.tw; a.ti = pl.ti;
  B200OCL_CUDA((raise_smem_limit<conv_patch_kernel<BN, PT>>(pl.smem)));
  dim3 grid(pl.grid_x, pl.grid_y);
  B200OCL_PROF(a.flip ? "conv_dgrad" : (a.mode == CONV_EVAL ? "conv_eval" : "conv_train"),
               2.0 * a.M * (double)a.CN * a.CK * a.ks * a.ks, stream);
  conv_patch_kernel<BN, PT><<<grid, CONV_THREADS, pl.smem, stream>>>(a);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

template <int BN, int PT>
int launch_conv_cfg(const ConvArgs& a, const ConvPlan& pl, cudaStream_t stream) {
  constexpr int WN = BN / 20, WM = 4 / WN, BM = WM * 32 * PT;
  constexpr size_t smem = (size_t)(3 * BM * 20 + 3 * 20 * BN) * sizeof(float) + 4 * BM * sizeof(int);
  B200OCL_CUDA((raise_smem_limit<conv_kernel<BN, PT>>(smem)));
  dim3 grid(pl.grid_x, pl.grid_y);
  B200OCL_PROF(a.transposed ? "conv_dgrad" : (a.mode == CONV_EVAL ? "conv_eval" : "conv_train"), 2.0 * a.M * (double)a.CN * a.CK * a.ks * a.ks, stream);
  conv_kernel<BN, PT><<<grid, CONV_THREADS, smem, stream>>>(a);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

int launch_stem(const ConvArgs& a, const ConvPlan& pl, cudaStream_t stream) {
  B200OCL_PROF(a.mode == CONV_EVAL ? "conv_eval" : "conv_train", 2.0 * a.M * 20.0 * 27.0, stream);
  stem_kernel<<<pl.grid_x, CONV_THREADS, 0, stream>>>(a);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

ConvPlan none(const char* why) {
  ConvPlan pl{};
  pl.kernel = CONV_K_NONE;
  pl.why = why;
  return pl;
}

ConvPlan tiled(const ConvArgs& a, int kernel, int bn, int pt, int bm) {
  ConvPlan pl{};
  pl.kernel = kernel;
  pl.bn = bn;
  pl.pt = pt;
  pl.grid_x = (a.M + bm - 1) / bm;
  pl.grid_y = a.CN / bn;
  return pl;
}

}  // namespace

ConvPlan conv_plan(const ConvArgs& a, int sms) {
  if (a.CK == 3) {
    if (a.CN != 20 || a.ks != 3 || a.stride != 1 || a.Hin != a.Hout || a.Win != a.Wout || a.M <= 0 || a.transposed)
      return none("only the 3->20 3x3 stride-1 stem is supported");
    return tiled(a, CONV_K_STEM, 20, 1, CONV_THREADS);
  }
  if (a.CK % 20 != 0 || a.CN % 20 != 0 || a.M <= 0) return none("channel counts must be multiples of 20");
  ConvPlan pl{};
  // 3x3 stride-1 convolutions on 8/16/32-wide maps: tensor cores fed from a halo patch (conv_tcp.cu);
  // other 3x3 stride-1 shapes with enough 128-pixel tiles: tensor cores with an im2col tile (conv_tc.cu).
  bool tcp = false, tc = false;
  if (a.force_path == 3) {
    if (!conv_tcp_eligible(a)) return none("launch not covered by the halo-patch tensor-core kernel (3x3 stride 1, no train mode)");
    tcp = true;
  } else if (a.force_path == 2) {
    if (!(a.w_tc && a.ks == 3 && a.stride == 1 && !a.transposed)) return none("shape not covered by conv_tc");
    tc = true;
  } else if (a.force_path == 0) {
    tcp = conv_tcp_eligible(a);
    tc = !tcp && conv_tc_eligible(a, sms);
  }
  if (tcp) {
    pl.kernel = CONV_K_TCP;
    pl.nt = a.tp_bn <= 20 ? 32 : 48;   // tp_bn <= 40 (conv_tcp_eligible)
    pl.grid_x = conv_tcp_grid_x(a, sms);
    pl.grid_y = a.CN / a.tp_bn;
    conv_tcp_pipeline(a, pl.nt, &pl.tp_ps, &pl.tp_bs);
    return pl;
  }
  if (tc) {
    pl.kernel = CONV_K_TC;
    pl.nt = a.tc_bn <= 20 ? 32 : (a.tc_bn <= 40 ? 48 : 80);
    pl.grid_x = (a.M + 127) / 128;
    pl.grid_y = a.CN / a.tc_bn;
    return pl;
  }
  // Forward convolutions and stride-1 data gradients with enough pixels go to the patch kernel:
  // pick the widest channel tile and 2 pixels per thread that still give >= 3 CTAs per SM.
  if (!a.transposed && a.ks * a.ks * 20 * 80 * sizeof(float) <= 64 * 1024) {
    // The inner loop issues 5 broadcast LDS.128 (20 weights) per k for 20*PT FMAs and a warp-wide
    // LDS.128 occupies the shared-memory pipe for 4 cycles, so PT = 2 is shared-memory bound by ~2x
    // PT = 4 is close to balance.  Take PT = 4 whenever it still fills the SMs.
    const long want3 = 5L * sms / 2;
    const int pbn[3] = {80, 40, 20};
    const int ppt[3] = {4, 2, 1};
    for (int pi = 0; pi < 3; ++pi)
      for (int bi = 0; bi < 3; ++bi) {
        if (a.CN % pbn[bi]) continue;
        const PatchTile t = patch_tile(a, pbn[bi], ppt[pi]);
        const long need = (ppt[pi] == 4) ? 3L * sms / 2 : want3;
        if (t.ctas < need || t.smem > (ppt[pi] == 4 ? 100 : 72) * 1024) continue;
        pl.kernel = CONV_K_PATCH;
        pl.bn = pbn[bi];
        pl.pt = ppt[pi];
        pl.grid_y = a.CN / pl.bn;
        pl.grid_x = (int)(t.ctas / pl.grid_y);
        pl.th = t.th; pl.tw = t.tw; pl.ti = t.ti;
        pl.smem = t.smem;
        return pl;
      }
  }
  // Tiling: the kernels are latency-sensitive (4 warps per CTA, LDS -> FMA chains), so the first goal is
  // >= 4 resident CTAs per SM (16 warps); among tilings that reach it prefer wide channel tiles (the
  // gathered pixel rows are shared by BN/20 warps) and 2-4 pixels per thread (weight loads amortised).
  // When the pixel count cannot provide that many CTAs the K loop is split inside the CTA instead.
  const long want = 4L * sms;
  const int bns[3] = {80, 40, 20};
  auto ctas_reg = [&](int bn, int pt) {
    const int bm = (80 / bn) * 32 * pt;
    return (long)((a.M + bm - 1) / bm) * (a.CN / bn);
  };
  for (int bi = 0; bi < 3; ++bi)
    if (a.CN % bns[bi] == 0 && ctas_reg(bns[bi], 2) >= want) return tiled(a, CONV_K_TILED, bns[bi], 2, (80 / bns[bi]) * 64);
  if (a.ks * a.ks * (a.CK / 20) >= 4) {
    int pt = 1, kwarps = 4;
    const long ctas2 = (long)((a.M + 63) / 64) * (a.CN / 20);
    const long ctas1 = (long)((a.M + 31) / 32) * (a.CN / 20);
    if (ctas2 >= want) pt = 2;
    // fewer than two CTAs per SM and a long K: eight warps share the K loop
    else if (ctas1 < 2L * sms && a.ks * a.ks * (a.CK / 20) >= 16) kwarps = 8;
    pl = tiled(a, CONV_K_KSPLIT, 20, pt, 32 * pt);
    pl.kwarps = kwarps;
    return pl;
  }
  return tiled(a, CONV_K_TILED, 20, 1, 128);   // 1x1 convolutions with a short K: most CTAs
}

int launch_conv(const ConvArgs& a, int sms, cudaStream_t stream) {
  const ConvPlan pl = conv_plan(a, sms);
  switch (pl.kernel) {
    case CONV_K_STEM: return launch_stem(a, pl, stream);
    case CONV_K_TCP: return launch_conv_tcp(a, pl, stream);
    case CONV_K_TC: return launch_conv_tc(a, pl, stream);
    case CONV_K_PATCH:
#define B200OCL_PATCH_CASE(BN_, PT_) \
      if (pl.bn == BN_ && pl.pt == PT_) return launch_conv_patch<BN_, PT_>(a, pl, stream)
      B200OCL_PATCH_CASE(80, 4); B200OCL_PATCH_CASE(40, 4); B200OCL_PATCH_CASE(20, 4);
      B200OCL_PATCH_CASE(80, 2); B200OCL_PATCH_CASE(40, 2); B200OCL_PATCH_CASE(20, 2);
      B200OCL_PATCH_CASE(80, 1); B200OCL_PATCH_CASE(40, 1); B200OCL_PATCH_CASE(20, 1);
#undef B200OCL_PATCH_CASE
      break;
    case CONV_K_TILED:
#define B200OCL_CONV_CASE(BN_, PT_) \
      if (pl.bn == BN_ && pl.pt == PT_) return launch_conv_cfg<BN_, PT_>(a, pl, stream)
      B200OCL_CONV_CASE(80, 4); B200OCL_CONV_CASE(80, 2); B200OCL_CONV_CASE(80, 1);
      B200OCL_CONV_CASE(40, 4); B200OCL_CONV_CASE(40, 2); B200OCL_CONV_CASE(40, 1);
      B200OCL_CONV_CASE(20, 4); B200OCL_CONV_CASE(20, 2); B200OCL_CONV_CASE(20, 1);
#undef B200OCL_CONV_CASE
      break;
    case CONV_K_KSPLIT:
      if (pl.pt == 2) return launch_conv_ksplit<2, 4>(a, pl, stream);
      if (pl.kwarps == 8) return launch_conv_ksplit<1, 8>(a, pl, stream);
      return launch_conv_ksplit<1, 4>(a, pl, stream);
    default:
      set_error("launch_conv: %s (CK=%d CN=%d M=%d)", pl.why, a.CK, a.CN, a.M);
      return B200OCL_EUNSUPPORTED;
  }
  set_error("launch_conv: no kernel instantiated for the planned tiling");
  return B200OCL_EUNSUPPORTED;
}

}  // namespace b200ocl
