// supcon.cu -- fused supervised-contrastive loss, forward + backward (sm_90a).
//
// Replaces SupConLoss.forward and its autograd backward (utils/loss.py:19-96; ~40 ATen
// kernels on [A,A] temporaries, A = V*B anchors).  The [A,A] logit matrix is never materialised.
//
// Main path (d % 4 == 0, d <= 256): ONE launch, supcon_fused_kernel.  Persistent CTAs own blocks of
// TM anchors; contrast rows stream through a double-buffered shared-memory ring filled by TMA 1-D bulk
// copies (cp.async.bulk + mbarrier, one row per copy into a padded pitch); the logit tile is a register-tiled
// fp32 product (RM x RN outputs per thread, 128-bit shared loads along d); row statistics are reduced with
// width-16 warp shuffles.  Phase A: online max / exp-sum / positive sums per anchor -> lse, |P(i)|, loss
// partial.  One grid-wide arrive/wait (all CTAs are co-resident: grid <= SMs x occupancy).  Phase B: logits
// recomputed, w_ij = (G_ij + G_ji)/T written transposed to shared memory, dC_i += W x C_j as a second
// register-tiled product.  The loss is summed in unit order by CTA 0 (no float atomics anywhere).
//
// Fallback for other d (<= 1024): two launches,
//   stats kernel  one warp per anchor i streams all contrast rows through shared memory,
//                 lane j of a 32-row tile owns logit l_ij = c_i.c_j / T; online max /
//                 exp-sum (diagonal in the max, out of the sum: loss.py:71-86), positive
//                 logit sum and count; writes lse_i = max_i + log Z_i, |P(i)|, and the loss
//                 through a fixed-order two-level reduction (last CTA finishes);
//   grad kernel   recomputes l_ij tile by tile and accumulates
//                 dc_i = (1/T) sum_j (G_ij + G_ji) c_j,  G_ij = (exp(l_ij - lse_i) - 1[j in P(i)]/|P(i)|)/A,
//                 using l_ji = l_ij (anchor set == contrast set in 'all' mode, loss.py:60-62).
// Anchors are in view-major order a = v*B + b (loss.py:56); features/grad are [B,V,d].
//
// supcon_plan() below is the one place that picks the launch: the resident fused kernel <1,4,NC,true>, the ring
// kernels <1,2,NC,false> (16-anchor units) and <4,4,NC,false> (64-anchor units), or the two-kernel fallback with
// grad kernel <DCH>.  b200ocl_supcon_plan reports it without launching anything.
//
// An anchor without positives (V = 1 and a class with one sample): its loss term is 0/0, so the loss is NaN, as in
// the reference (loss.py:90).  The gradient stays finite on every launch: G_ij's positive term 1[j in P(i)] / |P(i)|
// is taken as 0 for every j when P(i) is empty, so that anchor contributes its softmax term (the gradient of
// lse_i / A) and nothing else.  Autograd on the reference would make every entry NaN.
#include <float.h>
#include <limits.h>
#include <math.h>

#include "common.cuh"
#include "umma.cuh"

namespace b200ocl {
namespace {

constexpr int SC_THREADS = 256;
constexpr int SC_WARPS = 8;
constexpr int SCF_MAX_D = 256;

struct SupconParams {
  const float* feats;
  const long long* labels;
  int B, V, d, A, pitch;
  float T;
  float* lse;             // [A]
  float* npos;            // [A]
  float* part;            // [gridDim] loss partials
  unsigned int* counter;
  float* loss;
  float* dfeats;
  int n_units;            // fused kernel: anchor blocks
};

__device__ __forceinline__ const float* anchor_row(const SupconParams& p, int a) {
  const int v = a / p.B, b = a - v * p.B;
  return p.feats + ((size_t)b * p.V + v) * p.d;
}

// Cooperative load of contrast rows [j0, j0+32) into sct (pitch floats per row, odd pitch).
__device__ __forceinline__ void load_tile(const SupconParams& p, int j0, float* sct, int tid) {
  for (int idx = tid; idx < 32 * p.d; idx += SC_THREADS) {
    const int r = idx / p.d, dd = idx - r * p.d;
    const int j = j0 + r;
    sct[r * p.pitch + dd] = (j < p.A) ? anchor_row(p, j)[dd] : 0.f;
  }
}

__device__ __forceinline__ float tile_dot(const float* sa_row, const float* sct_row, int d) {
  float acc0 = 0.f, acc1 = 0.f;
  int dd = 0;
  for (; dd + 1 < d; dd += 2) {
    acc0 = fmaf(sa_row[dd], sct_row[dd], acc0);
    acc1 = fmaf(sa_row[dd + 1], sct_row[dd + 1], acc1);
  }
  if (dd < d) acc0 = fmaf(sa_row[dd], sct_row[dd], acc0);
  return acc0 + acc1;
}

__global__ void __launch_bounds__(SC_THREADS) supcon_stats_kernel(SupconParams p) {
  extern __shared__ __align__(16) float smem[];
  float* sa = smem;                          // [8][d]
  float* sct = sa + SC_WARPS * p.d;          // [32][pitch]
  __shared__ float s_loss[SC_WARPS];
  __shared__ bool is_last;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int a0 = blockIdx.x * SC_WARPS;
  const int i = a0 + warp;
  const bool valid = i < p.A;

  for (int idx = tid; idx < SC_WARPS * p.d; idx += SC_THREADS) {
    const int w = idx / p.d, dd = idx - w * p.d;
    sa[idx] = (a0 + w < p.A) ? anchor_row(p, a0 + w)[dd] : 0.f;
  }
  const long long yi = valid ? p.labels[i % p.B] : 0;

  float mx = -FLT_MAX, z = 0.f, ps = 0.f, np = 0.f;
  for (int j0 = 0; j0 < p.A; j0 += 32) {
    __syncthreads();
    load_tile(p, j0, sct, tid);
    __syncthreads();
    const int j = j0 + lane;
    if (valid && j < p.A) {
      const float l = __fdiv_rn(tile_dot(sa + warp * p.d, sct + lane * p.pitch, p.d), p.T);
      if (l > mx) {                  // rescale the running sum to the new max
        z *= expf(mx - l);
        mx = l;
      }
      if (j != i) {
        z += expf(l - mx);
        if (p.labels[j % p.B] == yi) {
          ps += l;
          np += 1.f;
        }
      }
    }
  }
  // combine lanes
  const float M = warp_max(mx);
  const float Z = warp_sum(z * expf(mx - M));   // lanes that saw nothing: z == 0
  const float PS = warp_sum(ps);
  const float NP = warp_sum(np);
  float loss_i = 0.f;
  if (valid) {
    const float lse = M + logf(Z);
    loss_i = -(PS - NP * lse) / NP;             // 0/0 -> NaN like loss.py:90
    if (lane == 0) {
      p.lse[i] = lse;
      p.npos[i] = NP;
    }
  }
  if (lane == 0) s_loss[warp] = loss_i;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < SC_WARPS; ++w) t += s_loss[w];
    p.part[blockIdx.x] = t;
    __threadfence();
    is_last = (atomicAdd(p.counter, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (is_last && tid == 0) {
    __threadfence();
    double t = 0.0;
    for (unsigned int b = 0; b < gridDim.x; ++b) t += (double)__ldcg(p.part + b);
    *p.loss = (float)(t / (double)p.A);
  }
}

template <int DCH>
__global__ void __launch_bounds__(SC_THREADS) supcon_grad_kernel(SupconParams p) {
  extern __shared__ __align__(16) float smem[];
  float* sa = smem;                          // [8][d]
  float* sct = sa + SC_WARPS * p.d;          // [32][pitch]
  float* wbuf = sct + 32 * p.pitch;          // [8][32]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int a0 = blockIdx.x * SC_WARPS;
  const int i = a0 + warp;
  const bool valid = i < p.A;

  for (int idx = tid; idx < SC_WARPS * p.d; idx += SC_THREADS) {
    const int w = idx / p.d, dd = idx - w * p.d;
    sa[idx] = (a0 + w < p.A) ? anchor_row(p, a0 + w)[dd] : 0.f;
  }
  const long long yi = valid ? p.labels[i % p.B] : 0;
  const float lse_i = valid ? p.lse[i] : 0.f;
  const float np_i = valid ? p.npos[i] : 1.f;
  const float invA = 1.f / (float)p.A;

  float acc[DCH];
#pragma unroll
  for (int c = 0; c < DCH; ++c) acc[c] = 0.f;

  for (int j0 = 0; j0 < p.A; j0 += 32) {
    __syncthreads();
    load_tile(p, j0, sct, tid);
    __syncthreads();
    const int j = j0 + lane;
    float w = 0.f;
    if (valid && j < p.A && j != i) {
      const float l = __fdiv_rn(tile_dot(sa + warp * p.d, sct + lane * p.pitch, p.d), p.T);
      // the positive terms only where j in P(i) (then i in P(j)): an anchor without positives has none (see the top)
      const bool pos = p.labels[j % p.B] == yi;
      const float g_ij = expf(l - lse_i) - (pos ? 1.f / np_i : 0.f);
      const float g_ji = expf(l - p.lse[j]) - (pos ? 1.f / p.npos[j] : 0.f);
      w = (g_ij + g_ji) * invA / p.T;
    }
    wbuf[warp * 32 + lane] = w;
    __syncwarp();
    const int jn = min(32, p.A - j0);
    for (int jj = 0; jj < jn; ++jj) {
      const float wj = wbuf[warp * 32 + jj];
      const float* row = sct + jj * p.pitch;
#pragma unroll
      for (int c = 0; c < DCH; ++c) {
        const int dd = lane + 32 * c;
        if (dd < p.d) acc[c] = fmaf(wj, row[dd], acc[c]);
      }
    }
    __syncwarp();
  }
  if (valid) {
    const int v = i / p.B, b = i - v * p.B;
    float* out = p.dfeats + ((size_t)b * p.V + v) * p.d;
#pragma unroll
    for (int c = 0; c < DCH; ++c) {
      const int dd = lane + 32 * c;
      if (dd < p.d) out[dd] = acc[c];
    }
  }
}


// ------------------------------------------------------------------------------------------------
// fused single-launch kernel
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ const float* anchor_row_ptr(const SupconParams& p, int a) {
  const int v = a / p.B, b = a - v * p.B;
  return p.feats + ((size_t)b * p.V + v) * p.d;
}

// warp 0: stage `rows` feature rows starting at anchor a0 into dst (pitch floats per row) with bulk copies
__device__ __forceinline__ void stage_rows(const SupconParams& p, int a0, int rows, float* dst, int pitch, uint64_t* bar,
                                           int lane) {
  const int nvalid = max(0, min(rows, p.A - a0));
  const uint32_t row_bytes = (uint32_t)p.d * 4u;
  if (lane == 0) umma::mbar_expect_tx(bar, row_bytes * (uint32_t)nvalid);
  __syncwarp();
  for (int r = lane; r < nvalid; r += 32) umma::bulk_g2s(dst + (size_t)r * pitch, anchor_row_ptr(p, a0 + r), row_bytes, bar);
}

// every CTA arrives once; valid because the whole grid is co-resident
__device__ __forceinline__ void grid_arrive_wait(unsigned int* counter, unsigned int expected) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    unsigned int seen;
    do {
      asm volatile("ld.acquire.gpu.u32 %0, [%1];\n" : "=r"(seen) : "l"(counter) : "memory");
    } while (seen < expected);
    __threadfence();
  }
  __syncthreads();
}

template <int RM, int RN>
__device__ __forceinline__ void logit_tile(const float* __restrict__ sA, const float* __restrict__ sBt, int P, int d,
                                           int ty, int tx, float inv_T, float (&l)[RM][RN]) {
#pragma unroll
  for (int r = 0; r < RM; ++r)
#pragma unroll
    for (int c = 0; c < RN; ++c) l[r][c] = 0.f;
  const float* ap = sA + (size_t)(ty * RM) * P;
  const float* bp = sBt + (size_t)tx * P;
#pragma unroll 2
  for (int k = 0; k < d; k += 4) {
    float4 a[RM], b[RN];
#pragma unroll
    for (int r = 0; r < RM; ++r) a[r] = *reinterpret_cast<const float4*>(ap + (size_t)r * P + k);
#pragma unroll
    for (int c = 0; c < RN; ++c) b[c] = *reinterpret_cast<const float4*>(bp + (size_t)(16 * c) * P + k);
#pragma unroll
    for (int r = 0; r < RM; ++r)
#pragma unroll
      for (int c = 0; c < RN; ++c) {
        l[r][c] = fmaf(a[r].x, b[c].x, l[r][c]);
        l[r][c] = fmaf(a[r].y, b[c].y, l[r][c]);
        l[r][c] = fmaf(a[r].z, b[c].z, l[r][c]);
        l[r][c] = fmaf(a[r].w, b[c].w, l[r][c]);
      }
  }
#pragma unroll
  for (int r = 0; r < RM; ++r)
#pragma unroll
    for (int c = 0; c < RN; ++c) l[r][c] *= inv_T;   // anchor_dot_contrast / T (loss.py:67-69) as a product with fl(1/T): <= 1 ulp apart
}

// RES: the whole contrast set (all n_tiles x TN rows) is resident in shared memory, staged once with one
// mbarrier -- the shape of the replay path itself (A = 220 anchors, d = 128: 113 KB).  Otherwise rows stream
// through a two-slot ring, tile t+1 in flight while tile t is consumed.
template <int RM, int RN, int NC, bool RES>
__global__ void __launch_bounds__(SC_THREADS, 1) supcon_fused_kernel(SupconParams p) {
  constexpr int TM = 16 * RM, TN = 16 * RN, WP = TM + 4;
  extern __shared__ __align__(128) unsigned char raw[];
  const int P = p.d + 4;
  const int n_tiles = (p.A + TN - 1) / TN;
  const int b_rows = RES ? n_tiles * TN : 2 * TN;             // contrast rows held in shared memory
  uint64_t* bars = reinterpret_cast<uint64_t*>(raw);          // [0] anchors, [1],[2] contrast ring / resident set
  float* sA = reinterpret_cast<float*>(raw + 128);
  float* sB = sA + (size_t)TM * P;                            // [b_rows][P]
  float* sWt = sB + (size_t)b_rows * P;                       // [TN][WP]
  long long* sLab = reinterpret_cast<long long*>(sWt + (size_t)TN * WP);   // [b_rows]
  float* sLse = reinterpret_cast<float*>(sLab + b_rows);      // [b_rows]
  float* sInvNp = sLse + b_rows;                              // [b_rows]  1 / |P(j)|
  float* sRow = sInvNp + b_rows;                              // [TM] per-anchor loss terms

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ty = tid >> 4, tx = tid & 15;
  const float invA = 1.f / (float)p.A;
  const float inv_T = 1.f / p.T;

  // zero the staging buffers once: rows past A are never written by a copy and must stay finite
  for (int idx = tid; idx < (TM + b_rows) * P; idx += SC_THREADS) sA[idx] = 0.f;
  if (tid == 0) {
    umma::mbar_init(&bars[0], 1);
    umma::mbar_init(&bars[1], 1);
    umma::mbar_init(&bars[2], 1);
    umma::fence_mbar_init();
  }
  umma::fence_proxy_async_smem();
  __syncthreads();
  uint32_t a_phase = 0, b_count = 0;      // b_count: contrast tiles consumed so far (ring slot = count & 1)

  if (RES) {
    if (warp == 0) stage_rows(p, 0, p.A, sB, P, &bars[1], lane);        // every contrast row, one barrier
    for (int j = tid; j < b_rows; j += SC_THREADS) sLab[j] = (j < p.A) ? p.labels[j % p.B] : 0;
  }

  for (int phase = 0; phase < 2; ++phase) {
    if (phase == 1) {
      if (!p.dfeats) break;
      grid_arrive_wait(p.counter, gridDim.x);
      if (RES) {
        for (int j = tid; j < b_rows; j += SC_THREADS) {
          sLse[j] = (j < p.A) ? __ldcg(p.lse + j) : 0.f;
          sInvNp[j] = (j < p.A) ? 1.f / __ldcg(p.npos + j) : 1.f;
        }
        __syncthreads();
      }
    }
    for (int unit = blockIdx.x; unit < p.n_units; unit += gridDim.x) {
      const int i0 = unit * TM;
      if (warp == 0) {
        stage_rows(p, i0, TM, sA, P, &bars[0], lane);
        if (!RES) stage_rows(p, 0, TN, sB + (size_t)(b_count & 1) * TN * P, P, &bars[1 + (b_count & 1)], lane);
      }
      long long yi[RM];
      float lse_i[RM], inv_np_i[RM];
      int gi[RM];
#pragma unroll
      for (int r = 0; r < RM; ++r) {
        gi[r] = i0 + ty * RM + r;
        const bool v = gi[r] < p.A;
        yi[r] = v ? p.labels[gi[r] % p.B] : 0;
        lse_i[r] = (phase == 1 && v) ? __ldcg(p.lse + gi[r]) : 0.f;
        inv_np_i[r] = (phase == 1 && v) ? 1.f / __ldcg(p.npos + gi[r]) : 1.f;
      }
      float m[RM], z[RM], ps[RM], np[RM];
      float acc[RM][NC * 4];
#pragma unroll
      for (int r = 0; r < RM; ++r) {
        m[r] = -FLT_MAX; z[r] = 0.f; ps[r] = 0.f; np[r] = 0.f;
#pragma unroll
        for (int q = 0; q < NC * 4; ++q) acc[r][q] = 0.f;
      }
      umma::mbar_wait(&bars[0], a_phase);
      a_phase ^= 1;
      if (RES && phase == 0) {
        umma::mbar_wait(&bars[1], 0);
        __syncthreads();                                     // sLab visible
      }

      for (int t = 0; t < n_tiles; ++t, ++b_count) {
        const int slot = RES ? t : (int)(b_count & 1);
        const int j0 = t * TN;
        const float* sBt = sB + (size_t)slot * TN * P;
        const int ab = slot * TN;                            // base of this tile's per-row arrays
        if (!RES) {
          if (warp == 0 && t + 1 < n_tiles)
            stage_rows(p, j0 + TN, TN, sB + (size_t)(slot ^ 1) * TN * P, P, &bars[1 + (slot ^ 1)], lane);
          if (tid < TN) {
            const int j = j0 + tid;
            const bool v = j < p.A;
            sLab[ab + tid] = v ? p.labels[j % p.B] : 0;
            if (phase == 1) {
              sLse[ab + tid] = v ? __ldcg(p.lse + j) : 0.f;
              sInvNp[ab + tid] = v ? 1.f / __ldcg(p.npos + j) : 1.f;
            }
          }
          umma::mbar_wait(&bars[1 + slot], (b_count >> 1) & 1);
          __syncthreads();
        }

        float l[RM][RN];
        logit_tile<RM, RN>(sA, sBt, P, p.d, ty, tx, inv_T, l);

        if (phase == 0) {
#pragma unroll
          for (int r = 0; r < RM; ++r) {
            float tm = -FLT_MAX;
#pragma unroll
            for (int c = 0; c < RN; ++c)
              if (j0 + tx + 16 * c < p.A) tm = fmaxf(tm, l[r][c]);     // the diagonal takes part in the max (loss.py:71)
            if (tm > m[r]) {
              z[r] *= __expf(m[r] - tm);
              m[r] = tm;
            }
#pragma unroll
            for (int c = 0; c < RN; ++c) {
              const int j = j0 + tx + 16 * c;
              if (j < p.A && j != gi[r]) {
                z[r] += __expf(l[r][c] - m[r]);
                if (sLab[ab + tx + 16 * c] == yi[r]) {
                  ps[r] += l[r][c];
                  np[r] += 1.f;
                }
              }
            }
          }
        } else {
#pragma unroll
          for (int r = 0; r < RM; ++r)
#pragma unroll
            for (int c = 0; c < RN; ++c) {
              const int jl = tx + 16 * c, j = j0 + jl;
              float w = 0.f;
              if (j < p.A && gi[r] < p.A && j != gi[r]) {
                const bool pos = sLab[ab + jl] == yi[r];
                // G_ij + G_ji, G_ij = exp(l_ij - lse_i) - 1[j in P(i)] / |P(i)|   (1 * (1/n) == 1/n exactly)
                float g = __expf(l[r][c] - lse_i[r]) + __expf(l[r][c] - sLse[ab + jl]);
                if (pos) g -= inv_np_i[r] + sInvNp[ab + jl];
                w = g * invA * inv_T;
              }
              sWt[jl * WP + ty * RM + r] = w;
            }
          __syncthreads();
          const int jn = min(TN, p.A - j0);
          const float* wp = sWt + ty * RM;
#pragma unroll 4
          for (int jj = 0; jj < jn; ++jj) {
            float wv[RM];
#pragma unroll
            for (int r = 0; r < RM; ++r) wv[r] = wp[jj * WP + r];
#pragma unroll
            for (int c = 0; c < NC; ++c) {
              const int dd = (tx + 16 * c) * 4;
              if (dd < p.d) {
                const float4 cv = *reinterpret_cast<const float4*>(sBt + (size_t)jj * P + dd);
#pragma unroll
                for (int r = 0; r < RM; ++r) {
                  acc[r][c * 4 + 0] = fmaf(wv[r], cv.x, acc[r][c * 4 + 0]);
                  acc[r][c * 4 + 1] = fmaf(wv[r], cv.y, acc[r][c * 4 + 1]);
                  acc[r][c * 4 + 2] = fmaf(wv[r], cv.z, acc[r][c * 4 + 2]);
                  acc[r][c * 4 + 3] = fmaf(wv[r], cv.w, acc[r][c * 4 + 3]);
                }
              }
            }
          }
        }
        if (!RES || phase == 1) __syncthreads();   // ring slot / sWt / per-tile arrays are free for the next stage
      }

      if (phase == 0) {
        // combine the 16 lanes that share a row (xor 8,4,2,1 stays inside a half-warp)
#pragma unroll
        for (int r = 0; r < RM; ++r) {
          float M = m[r];
#pragma unroll
          for (int o = 8; o > 0; o >>= 1) M = fmaxf(M, __shfl_xor_sync(FULL_MASK, M, o));
          float Z = z[r] * __expf(m[r] - M), PS = ps[r], NP = np[r];
#pragma unroll
          for (int o = 8; o > 0; o >>= 1) {
            Z += __shfl_xor_sync(FULL_MASK, Z, o);
            PS += __shfl_xor_sync(FULL_MASK, PS, o);
            NP += __shfl_xor_sync(FULL_MASK, NP, o);
          }
          if (tx == 0) {
            float li = 0.f;
            if (gi[r] < p.A) {
              const float lse = M + logf(Z);
              li = -(PS - NP * lse) / NP;               // 0/0 -> NaN like loss.py:90
              p.lse[gi[r]] = lse;
              p.npos[gi[r]] = NP;
            }
            sRow[ty * RM + r] = li;
          }
        }
        __syncthreads();
        if (tid == 0) {
          float tsum = 0.f;
          for (int r = 0; r < TM; ++r) tsum += sRow[r];
          p.part[unit] = tsum;
        }
        __syncthreads();
      } else {
#pragma unroll
        for (int r = 0; r < RM; ++r) {
          if (gi[r] >= p.A) continue;
          const int v = gi[r] / p.B, b = gi[r] - v * p.B;
          float* out = p.dfeats + ((size_t)b * p.V + v) * p.d;
#pragma unroll
          for (int c = 0; c < NC; ++c) {
            const int dd = (tx + 16 * c) * 4;
            if (dd < p.d)
              *reinterpret_cast<float4*>(out + dd) = make_float4(acc[r][c * 4], acc[r][c * 4 + 1], acc[r][c * 4 + 2], acc[r][c * 4 + 3]);
          }
        }
      }
    }
    if (phase == 0 && !p.dfeats) grid_arrive_wait(p.counter, gridDim.x);   // loss needs every unit's partial
  }
  // after the grid-wide wait every partial is visible: CTA 0 adds them in unit order
  if (blockIdx.x == 0 && tid == 0) {
    double t = 0.0;
    for (int u = 0; u < p.n_units; ++u) t += (double)__ldcg(p.part + u);
    *p.loss = (float)(t / (double)p.A);
  }
}

template <int RM, int RN, int NC, bool RES>
size_t fused_smem_bytes(int A, int d) {
  constexpr int TM = 16 * RM, TN = 16 * RN, WP = TM + 4;
  const int P = d + 4;
  const int b_rows = RES ? (A + TN - 1) / TN * TN : 2 * TN;
  return 128 + (size_t)(TM + b_rows) * P * 4 + (size_t)TN * WP * 4 + (size_t)b_rows * 16 + (size_t)TM * 4;
}

constexpr size_t SCF_SMEM_LIMIT = 227 * 1024;     // the fused kernels' dynamic shared-memory limit
constexpr size_t SCF_RES_MAX_SMEM = 200 * 1024;   // the resident family is taken up to this much
constexpr size_t SC_SMEM_LIMIT = 200 * 1024;      // the two-kernel fallback's limit (d = 1024 needs 165 KB)

// The one place that decides which SupCon kernels a call launches (b200ocl_supcon launches what this returns;
// b200ocl_supcon_plan reports it).  Host only.
b200ocl_supcon_launch supcon_plan(int B, int V, int d, bool aligned, int sms) {
  b200ocl_supcon_launch L{};
  const int A = B * V;
  L.sms = sms;
  if (d % 4 == 0 && d <= SCF_MAX_D && aligned) {
    L.nc = (d + 63) / 64;
    if (A <= 16 * sms && fused_smem_bytes<1, 4, 4, true>(A, d) <= SCF_RES_MAX_SMEM) {
      L.family = B200OCL_SUPCON_RESIDENT;
      L.rm = 1; L.rn = 4;
    } else if (A <= 16 * sms) {
      L.family = B200OCL_SUPCON_RING16;
      L.rm = 1; L.rn = 2;
    } else {
      // large anchor sets: 64-anchor blocks, one CTA per SM.  Shared memory, not occupancy, bounds the inner loop, so
      // the 4 x 4 register tile with the least shared-memory traffic per FMA is used.
      L.family = B200OCL_SUPCON_RING64;
      L.rm = 4; L.rn = 4;
    }
    const int TM = 16 * L.rm, TN = 16 * L.rn;
    const bool res = L.family == B200OCL_SUPCON_RESIDENT;
    // fused_smem_bytes does not depend on NC
    L.smem_bytes = res ? fused_smem_bytes<1, 4, 4, true>(A, d)
                       : (L.rm == 1 ? fused_smem_bytes<1, 2, 4, false>(A, d) : fused_smem_bytes<4, 4, 4, false>(A, d));
    L.smem_limit = SCF_SMEM_LIMIT;
    L.n_units = (A + TM - 1) / TM;
    L.grid = L.n_units < sms ? L.n_units : sms;          // the grid-wide wait needs every CTA resident: one per SM
    L.units_per_cta = (L.n_units + L.grid - 1) / L.grid;
    const int staged = res ? A : (TM > TN ? TM : TN);    // rows behind one mbarrier expect_tx
    L.tx_bytes = (size_t)staged * (size_t)d * 4;
  } else {
    L.family = B200OCL_SUPCON_FALLBACK;
    L.dch = d <= 128 ? 4 : d <= 256 ? 8 : d <= 512 ? 16 : 32;
    L.n_units = (A + SC_WARPS - 1) / SC_WARPS;
    L.grid = L.n_units;
    L.units_per_cta = 1;
    const int pitch = (d % 2 == 0) ? d + 1 : d;
    L.smem_bytes = (size_t)(SC_WARPS * d + 32 * pitch) * sizeof(float) + SC_WARPS * 32 * sizeof(float);   // grad kernel
    L.smem_limit = SC_SMEM_LIMIT;
  }
  return L;
}

template <int RM, int RN, int NC, bool RES>
int launch_fused(SupconParams p, const b200ocl_supcon_launch& L, cudaStream_t stream) {
  B200OCL_CUDA((raise_smem_limit<supcon_fused_kernel<RM, RN, NC, RES>>(SCF_SMEM_LIMIT)));
  p.n_units = L.n_units;
  // the grid-wide wait needs every CTA resident: one CTA per SM
  int per_sm = 0;
  B200OCL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, supcon_fused_kernel<RM, RN, NC, RES>, SC_THREADS,
                                                             L.smem_bytes));
  if (per_sm < 1) {
    set_error("b200ocl_supcon: fused kernel does not fit on an SM (%zu bytes of shared memory)", L.smem_bytes);
    return B200OCL_EUNSUPPORTED;
  }
  B200OCL_PROF("supcon", 2.0 * 4.0 * p.A * p.d + 8.0 * p.B, stream);
  supcon_fused_kernel<RM, RN, NC, RES><<<L.grid, SC_THREADS, L.smem_bytes, stream>>>(p);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

template <int RM, int RN, bool RES>
int launch_fused_nc(const SupconParams& p, const b200ocl_supcon_launch& L, cudaStream_t stream) {
  switch (L.nc) {
    case 1: return launch_fused<RM, RN, 1, RES>(p, L, stream);
    case 2: return launch_fused<RM, RN, 2, RES>(p, L, stream);
    case 3: return launch_fused<RM, RN, 3, RES>(p, L, stream);
    default: return launch_fused<RM, RN, 4, RES>(p, L, stream);
  }
}

}  // namespace
}  // namespace b200ocl

extern "C" {

size_t b200ocl_supcon_workspace_bytes(int B, int V, int d) {
  (void)d;
  const size_t A = (size_t)(B > 0 ? B : 0) * (size_t)(V > 0 ? V : 0);
  const size_t blocks = (A + b200ocl::SC_WARPS - 1) / b200ocl::SC_WARPS;
  return 256 + b200ocl::align_up((2 * A + blocks) * sizeof(float), 256);
}

int b200ocl_supcon(const float* feats, const int64_t* labels, int B, int V, int d, float temperature, float* loss,
                   float* dfeats, void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(feats && labels && loss, "null pointer");
  B200OCL_CHECK_ARG(B >= 1 && V >= 1 && d >= 1, "need B,V,d >= 1");
  B200OCL_CHECK_ARG(temperature > 0.f, "temperature must be positive");
  if (d > 1024) {
    set_error("b200ocl_supcon: d=%d exceeds the kernel's limit of 1024", d);
    return B200OCL_EUNSUPPORTED;
  }
  const int rc = check_workspace("b200ocl_supcon", workspace, workspace_bytes, b200ocl_supcon_workspace_bytes(B, V, d));
  if (rc) return rc;
  SupconParams p{};
  p.feats = feats;
  p.labels = reinterpret_cast<const long long*>(labels);
  p.B = B; p.V = V; p.d = d; p.A = B * V;
  p.pitch = (d % 2 == 0) ? d + 1 : d;
  p.T = temperature;
  p.counter = static_cast<unsigned int*>(workspace);
  float* ws = reinterpret_cast<float*>(static_cast<unsigned char*>(workspace) + 256);
  p.lse = ws;
  p.npos = ws + p.A;
  p.part = ws + 2 * (size_t)p.A;
  p.loss = loss;
  p.dfeats = dfeats;
  const bool aligned = (reinterpret_cast<uintptr_t>(feats) & 15) == 0 &&
                       (!dfeats || (reinterpret_cast<uintptr_t>(dfeats) & 15) == 0);
  const b200ocl_supcon_launch L = supcon_plan(B, V, d, aligned, sm_count());

  B200OCL_CUDA(cudaMemsetAsync(p.counter, 0, sizeof(unsigned int), stream));
  switch (L.family) {
    case B200OCL_SUPCON_RESIDENT: return launch_fused_nc<1, 4, true>(p, L, stream);
    case B200OCL_SUPCON_RING16: return launch_fused_nc<1, 2, false>(p, L, stream);
    case B200OCL_SUPCON_RING64: return launch_fused_nc<4, 4, false>(p, L, stream);
    default: break;
  }
  // static smem takes a little of the 227 KB
  const size_t smem_stats = L.smem_bytes - SC_WARPS * 32 * sizeof(float);
  B200OCL_CUDA((raise_smem_limit<supcon_stats_kernel, supcon_grad_kernel<4>, supcon_grad_kernel<8>, supcon_grad_kernel<16>,
                                 supcon_grad_kernel<32>>(L.smem_limit)));
  B200OCL_PROF("supcon", 4.0 * p.A * d + 8.0 * B + 8.0 * p.A, stream);
  supcon_stats_kernel<<<L.grid, SC_THREADS, smem_stats, stream>>>(p);
  B200OCL_LAUNCHED();
  if (!dfeats) return B200OCL_OK;
#define B200OCL_SC_GRAD(DCH) supcon_grad_kernel<DCH><<<L.grid, SC_THREADS, L.smem_bytes, stream>>>(p)
  B200OCL_PROF("supcon", 8.0 * p.A * d, stream);
  switch (L.dch) {
    case 4: B200OCL_SC_GRAD(4); break;
    case 8: B200OCL_SC_GRAD(8); break;
    case 16: B200OCL_SC_GRAD(16); break;
    default: B200OCL_SC_GRAD(32); break;
  }
#undef B200OCL_SC_GRAD
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

int b200ocl_supcon_plan(int B, int V, int d, int aligned, int sms, b200ocl_supcon_launch* out) {
  using namespace b200ocl;
  B200OCL_CHECK_ARG(out, "null pointer");
  B200OCL_CHECK_ARG(B >= 1 && V >= 1 && d >= 1, "need B,V,d >= 1");
  B200OCL_CHECK_ARG((long long)B * V <= INT_MAX / 2, "B*V out of range");
  B200OCL_CHECK_ARG(sms >= 0, "sms must be 0 (this device) or an SM count");
  if (d > 1024) {
    set_error("b200ocl_supcon_plan: d=%d exceeds the kernel's limit of 1024", d);
    return B200OCL_EUNSUPPORTED;
  }
  *out = supcon_plan(B, V, d, aligned != 0, sms ? sms : sm_count());
  return B200OCL_OK;
}

}  // extern "C"
