// gem.cu -- GEM's projection (Lopez-Paz & Ranzato, "Gradient Episodic Memory for Continual Learning", NeurIPS 2017) on
// the flat gradient arena: t <= 64 task gradients G [t,n] (rows at a pitch), the stream gradient g [n].
//   P = G G^T, q = G g (fp64); when min_k q_k < 0:
//     v = arg min_v 1/2 v^T (P + eps I) v + q^T v  subject to  v_k >= margin,   out = g + G^T v
//   (the authors' project2cone2 with margin = memory_strength; margin 0 is the dual of the paper's projection).
// Three launches, no host synchronisation, every reduction in a fixed order with no floating-point atomics:
//   gem_gram_kernel  each CTA owns a contiguous slice of n, stages (t+1) x TC tiles of it in shared memory (cp.async,
//                    two stages) and forms every pair from the tile, so each element is read from HBM once; products of
//                    two floats are exact in fp64, sums are fp64 in column order per lane, lanes summed in lane order;
//                    one fp64 partial per pair (packed upper triangle of the (t+1) x (t+1) Gram of [G; g]) per CTA
//   gem_qp_kernel    one CTA: partials summed in CTA order, P symmetrised, the flag min q < 0, and when it is set the
//                    QP solved exactly by a primal active-set method on w = v - margin >= 0 (Cholesky of the free block
//                    at every iteration); the iteration count is bounded by GEM_QP_MAX_ITERS and running out sets
//                    *err_flag
//   gem_project_kernel  out[i] = fl32((double)g[i] + sum_k v_k (double)G_k[i]) in k order, each product and sum
//                    rounded once; returns without reading or
//                    writing anything when the flag is clear, so g stays bit-identical
// gem_plan() is the one place that derives the launch geometry (and the partials' size) from t, n and the SM count.
#include <math.h>

#include "common.cuh"

namespace b200ocl {
namespace {

constexpr int GEM_MAX_T = 64;
constexpr int GEM_THREADS = 256;
constexpr int GEM_RB = 4;                        // rows per register block: a thread forms a 4 x 4 block of pairs
constexpr int GEM_TILE_BYTES = 32 * 1024;        // target bytes of one staged tile (one of two stages)
constexpr int GEM_QP_THREADS = 256;
constexpr int GEM_PROJ_THREADS = 256;
// The active-set method below (Lawson & Hanson's NNLS loop applied to the strictly convex QP) adds one index per outer
// iteration and every inner iteration removes at least one, with the objective strictly decreasing between outer
// iterations, so it terminates; in practice it takes at most about 2t Cholesky solves (the GPU tests record the most
// seen).  The bound is 3 * 64 + 64 = 256 solves, four times what t = 64 needs by that count.
constexpr int GEM_QP_MAX_ITERS = 256;

__host__ __device__ inline int tri_index(int k, int l, int R) {   // k <= l < R, packed upper triangle, row-major
  return k * R - k * (k - 1) / 2 + (l - k);
}

b200ocl_gem_launch gem_plan(int t, size_t n, int sms) {
  b200ocl_gem_launch L = {};
  L.sms = sms;
  L.rows = t + 1;
  L.rows_padded = (L.rows + GEM_RB - 1) / GEM_RB * GEM_RB;
  L.row_blocks = L.rows_padded / GEM_RB;
  L.block_pairs = L.row_blocks * (L.row_blocks + 1) / 2;
  L.lanes = GEM_THREADS / L.block_pairs;
  int tc = 128;
  while (tc < 4096 && (size_t)L.rows_padded * (2 * tc + 4) * sizeof(float) <= (size_t)GEM_TILE_BYTES) tc *= 2;
  L.tile_cols = tc;
  L.tile_stride = tc + 4;
  const size_t stage = (size_t)L.rows_padded * L.tile_stride * sizeof(float);
  const size_t red = (size_t)GEM_THREADS * GEM_RB * GEM_RB * sizeof(double);
  L.smem_bytes = 2 * stage > red ? 2 * stage : red;
  L.pairs = L.rows * (L.rows + 1) / 2;
  if (n == 0) return L;
  // two CTAs per SM; a CTA's slice is at least one tile, and the grid is then cut so that every CTA has columns
  const size_t want = 2 * (size_t)sms;
  const size_t by_tiles = (n + tc - 1) / tc;
  const size_t g0 = want < by_tiles ? want : by_tiles;
  L.chunk = (n + g0 - 1) / g0;
  L.grid = (int)((n + L.chunk - 1) / L.chunk);
  L.tiles_per_cta = (int)((L.chunk + tc - 1) / tc);
  L.part_bytes = (size_t)L.grid * L.pairs * sizeof(double);
  L.workspace_bytes = align_up(L.part_bytes, 256);
  const size_t pg = (n + GEM_PROJ_THREADS - 1) / GEM_PROJ_THREADS;
  L.proj_grid = (int)(pg < 4 * (size_t)sms ? pg : 4 * (size_t)sms);
  return L;
}

__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gmem_src, int src_bytes) {
  const unsigned int s = static_cast<unsigned int>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(s), "l"(gmem_src), "r"(src_bytes));
}

// Stage columns [c0, c0 + TC) of rows 0..R-1 (row R-1 is g) into one tile; columns past `end` and the padding rows
// are zero (cp.async with a zero source size fills zeros).
__device__ __forceinline__ void stage_tile(float* tile, const float* __restrict__ G, size_t pitch, const float* __restrict__ g,
                                           int R, int RP, int TC, int stride, size_t c0, size_t end) {
  for (int r = 0; r < RP; ++r) {
    const float* row = r < R - 1 ? G + (size_t)r * pitch : g;
    for (int c = threadIdx.x; c < TC; c += GEM_THREADS) {
      const size_t col = c0 + c;
      const bool live = r < R && col < end;
      cp_async4(tile + r * stride + c, live ? row + col : g, live ? 4 : 0);
    }
  }
}

__global__ void __launch_bounds__(GEM_THREADS) gem_gram_kernel(const float* __restrict__ G, size_t pitch,
                                                               const float* __restrict__ g, size_t n,
                                                               b200ocl_gem_launch L, double* __restrict__ part) {
  extern __shared__ __align__(16) unsigned char gem_smem[];
  float* tiles = reinterpret_cast<float*>(gem_smem);
  const int R = L.rows, RP = L.rows_padded, TC = L.tile_cols, S = L.tile_stride;
  const size_t stage = (size_t)RP * S;
  const size_t c_begin = (size_t)blockIdx.x * L.chunk;
  const size_t c_end = c_begin + L.chunk < n ? c_begin + L.chunk : n;
  const int ntiles = (int)((c_end - c_begin + TC - 1) / TC);

  const int tid = threadIdx.x;
  const int lanes = L.lanes;
  const int b = tid / lanes, lane = tid % lanes;
  const bool active = b < L.block_pairs;
  int bi = 0, bj = 0;
  if (active) {                                    // block pair b -> (bi, bj), bi <= bj, row-major upper triangle
    int rem = b;
    while (rem >= L.row_blocks - bi) {
      rem -= L.row_blocks - bi;
      ++bi;
    }
    bj = bi + rem;
  }
  double acc[GEM_RB][GEM_RB];
#pragma unroll
  for (int i = 0; i < GEM_RB; ++i)
#pragma unroll
    for (int j = 0; j < GEM_RB; ++j) acc[i][j] = 0.0;

  if (ntiles > 0) stage_tile(tiles, G, pitch, g, R, RP, TC, S, c_begin, c_end);
  cp_async_commit();
  for (int it = 0; it < ntiles; ++it) {
    if (it + 1 < ntiles)
      stage_tile(tiles + ((it + 1) & 1) * stage, G, pitch, g, R, RP, TC, S, c_begin + (size_t)(it + 1) * TC, c_end);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const float* tile = tiles + (it & 1) * stage;
    if (active) {
      const float* A = tile + (bi * GEM_RB) * S;
      const float* B = tile + (bj * GEM_RB) * S;
      for (int c4 = lane; c4 < TC / 4; c4 += lanes) {
        float4 a[GEM_RB], bb[GEM_RB];
#pragma unroll
        for (int i = 0; i < GEM_RB; ++i) {
          a[i] = *reinterpret_cast<const float4*>(A + i * S + 4 * c4);
          bb[i] = *reinterpret_cast<const float4*>(B + i * S + 4 * c4);
        }
#pragma unroll
        for (int i = 0; i < GEM_RB; ++i)
#pragma unroll
          for (int j = 0; j < GEM_RB; ++j) {
            acc[i][j] = fma((double)a[i].x, (double)bb[j].x, acc[i][j]);
            acc[i][j] = fma((double)a[i].y, (double)bb[j].y, acc[i][j]);
            acc[i][j] = fma((double)a[i].z, (double)bb[j].z, acc[i][j]);
            acc[i][j] = fma((double)a[i].w, (double)bb[j].w, acc[i][j]);
          }
      }
    }
    __syncthreads();                               // the tile is overwritten by the stage after next
  }
  cp_async_wait<0>();
  __syncthreads();
  // lanes of one block pair summed in lane order; the tiles' space holds the per-thread blocks
  double* red = reinterpret_cast<double*>(gem_smem);
#pragma unroll
  for (int i = 0; i < GEM_RB; ++i)
#pragma unroll
    for (int j = 0; j < GEM_RB; ++j) red[(size_t)(i * GEM_RB + j) * GEM_THREADS + tid] = acc[i][j];
  __syncthreads();
  double* out = part + (size_t)blockIdx.x * L.pairs;
  for (int e = tid; e < L.block_pairs * GEM_RB * GEM_RB; e += GEM_THREADS) {
    const int bp = e / (GEM_RB * GEM_RB), ij = e % (GEM_RB * GEM_RB);
    int pi = 0, rem = bp;
    while (rem >= L.row_blocks - pi) {
      rem -= L.row_blocks - pi;
      ++pi;
    }
    const int k = pi * GEM_RB + ij / GEM_RB, l = (pi + rem) * GEM_RB + ij % GEM_RB;
    if (k > l || l >= R) continue;
    double s = 0.0;
    for (int ln = 0; ln < lanes; ++ln) s += red[(size_t)ij * GEM_THREADS + bp * lanes + ln];
    out[tri_index(k, l, R)] = s;
  }
}

// Cholesky of the free block H[F,F] (m x m, row stride GEM_MAX_T) into Lc, then Lc Lc^T z = rhs: z overwrites rhs.
// Returns false when a pivot is not positive (cannot happen for P + eps I with eps > 0 in exact arithmetic).
__device__ bool chol_solve(const double* H, const int* F, int m, double* Lc, double* rhs, bool* s_ok) {
  const int tid = threadIdx.x;
  for (int e = tid; e < m * m; e += GEM_QP_THREADS) {
    const int i = e / m, j = e % m;
    Lc[i * GEM_MAX_T + j] = j <= i ? H[F[i] * GEM_MAX_T + F[j]] : 0.0;
  }
  if (tid == 0) *s_ok = true;
  __syncthreads();
  for (int j = 0; j < m; ++j) {
    if (tid == 0) {
      const double d = Lc[j * GEM_MAX_T + j];
      if (!(d > 0.0)) *s_ok = false;
      Lc[j * GEM_MAX_T + j] = d > 0.0 ? sqrt(d) : 1.0;
    }
    __syncthreads();
    const double dj = Lc[j * GEM_MAX_T + j];
    for (int i = j + 1 + tid; i < m; i += GEM_QP_THREADS) Lc[i * GEM_MAX_T + j] /= dj;
    __syncthreads();
    const int rest = m - j - 1;
    for (int e = tid; e < rest * rest; e += GEM_QP_THREADS) {
      const int i = j + 1 + e / rest, k = j + 1 + e % rest;
      if (k <= i) Lc[i * GEM_MAX_T + k] -= Lc[i * GEM_MAX_T + j] * Lc[k * GEM_MAX_T + j];
    }
    __syncthreads();
  }
  if (tid == 0) {                                  // two triangular solves, m <= 64: one thread, fixed order
    for (int i = 0; i < m; ++i) {
      double s = rhs[i];
      for (int k = 0; k < i; ++k) s -= Lc[i * GEM_MAX_T + k] * rhs[k];
      rhs[i] = s / Lc[i * GEM_MAX_T + i];
    }
    for (int i = m - 1; i >= 0; --i) {
      double s = rhs[i];
      for (int k = i + 1; k < m; ++k) s -= Lc[k * GEM_MAX_T + i] * rhs[k];
      rhs[i] = s / Lc[i * GEM_MAX_T + i];
    }
  }
  __syncthreads();
  return *s_ok;
}

struct GemQpSmem {
  double H[GEM_MAX_T * GEM_MAX_T];   // P + eps I
  double Lc[GEM_MAX_T * GEM_MAX_T];  // Cholesky factor of the free block
  double q[GEM_MAX_T], c[GEM_MAX_T], w[GEM_MAX_T], z[GEM_MAX_T], lam[GEM_MAX_T];
  int F[GEM_MAX_T];                  // free indices, ascending
  int in_free[GEM_MAX_T];
  int m, flag, done, add, iters, fail;
  bool ok;
};

__global__ void __launch_bounds__(GEM_QP_THREADS) gem_qp_kernel(const double* __restrict__ part, int n_part, int t,
                                                                double margin, double eps, double* __restrict__ v_out,
                                                                int* __restrict__ flag_out, int* __restrict__ err_flag,
                                                                double* __restrict__ kkt_out) {
  extern __shared__ __align__(16) unsigned char qp_smem[];
  GemQpSmem& s = *reinterpret_cast<GemQpSmem*>(qp_smem);
  const int tid = threadIdx.x;
  const int R = t + 1, pairs = R * (R + 1) / 2;
  // partials summed in CTA order; P symmetrised from its upper triangle
  for (int e = tid; e < pairs; e += GEM_QP_THREADS) {
    double acc = 0.0;
    for (int b = 0; b < n_part; ++b) acc += part[(size_t)b * pairs + e];
    int k = 0, rem = e;
    while (rem >= R - k) {
      rem -= R - k;
      ++k;
    }
    const int l = k + rem;
    if (l < t) {
      s.H[k * GEM_MAX_T + l] = acc + (k == l ? eps : 0.0);
      s.H[l * GEM_MAX_T + k] = acc + (k == l ? eps : 0.0);
    } else if (k < t) {
      s.q[k] = acc;                                // l == t: the row of g
    }
  }
  __syncthreads();
  if (tid == 0) {
    int f = 0;
    for (int k = 0; k < t; ++k) f |= s.q[k] < 0.0;
    s.flag = f;
    *flag_out = f;
    s.iters = 0;
    s.fail = 0;
  }
  __syncthreads();
  if (!s.flag) {
    for (int k = tid; k < t; k += GEM_QP_THREADS) v_out[k] = 0.0;
    if (kkt_out && tid < 4) kkt_out[tid] = 0.0;
    return;
  }
  // w = v - margin >= 0: min 1/2 w^T H w + c^T w with c = q + margin H 1
  for (int k = tid; k < t; k += GEM_QP_THREADS) {
    double hs = 0.0;
    for (int l = 0; l < t; ++l) hs += s.H[k * GEM_MAX_T + l];
    s.c[k] = s.q[k] + margin * hs;
    s.w[k] = 0.0;
    s.in_free[k] = 0;
  }
  if (tid == 0) {
    s.m = 0;
    s.done = 0;
  }
  __syncthreads();
  while (true) {
    // multipliers lam = H w + c; optimal when lam_k >= -tol off the free set
    for (int k = tid; k < t; k += GEM_QP_THREADS) {
      double a = s.c[k];
      for (int l = 0; l < t; ++l) a += s.H[k * GEM_MAX_T + l] * s.w[l];
      s.lam[k] = a;
    }
    __syncthreads();
    if (tid == 0) {
      double cmax = 0.0, hmax = 0.0, wmax = 0.0;
      for (int k = 0; k < t; ++k) {
        cmax = fmax(cmax, fabs(s.c[k]));
        hmax = fmax(hmax, s.H[k * GEM_MAX_T + k]);
        wmax = fmax(wmax, s.w[k]);
      }
      const double tol = 1e-12 * (cmax + hmax * wmax);
      int add = -1;
      double most = -tol;
      for (int k = 0; k < t; ++k)
        if (!s.in_free[k] && s.lam[k] < most) {
          most = s.lam[k];
          add = k;
        }
      s.add = add;
      if (add < 0) s.done = 1;
      else if (s.iters >= GEM_QP_MAX_ITERS) {
        s.done = 1;
        s.fail = 1;
      } else {
        s.in_free[add] = 1;
      }
    }
    __syncthreads();
    if (s.done) break;
    // inner loop: solve on the free set, step back to feasibility while a free w would turn non-positive
    while (true) {
      if (tid == 0) {
        int m = 0;
        for (int k = 0; k < t; ++k)
          if (s.in_free[k]) s.F[m++] = k;
        s.m = m;
        for (int i = 0; i < m; ++i) s.z[i] = -s.c[s.F[i]];
        s.iters++;
      }
      __syncthreads();
      const bool ok = chol_solve(s.H, s.F, s.m, s.Lc, s.z, &s.ok);
      if (tid == 0) {
        const int m = s.m;
        bool positive = ok;
        for (int i = 0; i < m && positive; ++i) positive = s.z[i] > 0.0;
        if (!ok) s.fail = 1;
        if (positive || !ok) {
          for (int k = 0; k < t; ++k) s.w[k] = 0.0;
          if (ok)
            for (int i = 0; i < m; ++i) s.w[s.F[i]] = s.z[i];
          s.done = 2;                              // back to the outer loop
        } else {
          double alpha = 1.0;
          for (int i = 0; i < m; ++i) {
            const int k = s.F[i];
            if (s.z[i] <= 0.0) {
              const double a = s.w[k] / (s.w[k] - s.z[i]);
              if (a < alpha) alpha = a;
            }
          }
          for (int i = 0; i < m; ++i) {
            const int k = s.F[i];
            const double nw = s.w[k] + alpha * (s.z[i] - s.w[k]);
            // the index (or indices) that reach the bound leave the free set at exactly 0
            if (nw <= 0.0 || (s.z[i] <= 0.0 && s.w[k] / (s.w[k] - s.z[i]) <= alpha)) {
              s.w[k] = 0.0;
              s.in_free[k] = 0;
            } else {
              s.w[k] = nw;
            }
          }
          s.done = s.iters >= GEM_QP_MAX_ITERS ? 3 : 0;
        }
      }
      __syncthreads();
      if (s.done) break;
    }
    __syncthreads();
    if (tid == 0) {
      if (s.done == 3) s.fail = 1;
      s.done = (s.fail != 0);
    }
    __syncthreads();
    if (s.done) break;
  }
  if (tid == 0 && s.fail && err_flag) *err_flag = 1;
  for (int k = tid; k < t; k += GEM_QP_THREADS) v_out[k] = s.w[k] + margin;
  if (kkt_out) {
    // residuals of the returned w: primal max(0, -w), dual max(0, -lam) off the free set, complementarity max |w lam|
    __syncthreads();
    for (int k = tid; k < t; k += GEM_QP_THREADS) {
      double a = s.c[k];
      for (int l = 0; l < t; ++l) a += s.H[k * GEM_MAX_T + l] * s.w[l];
      s.lam[k] = a;
    }
    __syncthreads();
    if (tid == 0) {
      double pr = 0.0, du = 0.0, co = 0.0;
      for (int k = 0; k < t; ++k) {
        pr = fmax(pr, -s.w[k]);
        if (s.w[k] == 0.0) du = fmax(du, -s.lam[k]);
        else du = fmax(du, fabs(s.lam[k]));
        co = fmax(co, fabs(s.w[k] * s.lam[k]));
      }
      kkt_out[0] = pr;
      kkt_out[1] = du;
      kkt_out[2] = co;
      kkt_out[3] = (double)s.iters;
    }
  }
}

__global__ void __launch_bounds__(GEM_PROJ_THREADS) gem_project_kernel(const float* __restrict__ G, size_t pitch, int t,
                                                                       const float* g, float* out, size_t n,
                                                                       const double* __restrict__ v,
                                                                       const int* __restrict__ flag) {
  __shared__ double s_v[GEM_MAX_T];
  if (*flag == 0) return;
  for (int k = threadIdx.x; k < t; k += GEM_PROJ_THREADS) s_v[k] = v[k];
  __syncthreads();
  for (size_t i = (size_t)blockIdx.x * GEM_PROJ_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * GEM_PROJ_THREADS) {
    double a = (double)g[i];
    // product and sum rounded separately (no contraction), so that the result is the fp64 formula's, term by term
    for (int k = 0; k < t; ++k) a = __dadd_rn(a, __dmul_rn(s_v[k], (double)G[(size_t)k * pitch + i]));
    out[i] = __double2float_rn(a);
  }
}

}  // namespace
}  // namespace b200ocl

extern "C" {

int b200ocl_gem_plan(int t, size_t n, int sms, b200ocl_gem_launch* out) {
  using namespace b200ocl;
  B200OCL_CHECK_ARG(out, "null pointer");
  B200OCL_CHECK_ARG(t >= 1 && t <= GEM_MAX_T && n >= 1 && sms >= 0, "need 1 <= t <= 64, n >= 1, sms >= 0");
  *out = gem_plan(t, n, sms ? sms : sm_count());
  return B200OCL_OK;
}

size_t b200ocl_gem_project_workspace_bytes(int t, size_t n) {
  using namespace b200ocl;
  if (t < 1 || t > GEM_MAX_T || n < 1) return 0;
  return gem_plan(t, n, sm_count()).workspace_bytes;
}

int b200ocl_gem_project(const float* G, size_t pitch, int t, const float* g, float* out, size_t n, double margin,
                        double eps, double* v_out, int* flag_out, int* err_flag, double* kkt_out, void* workspace,
                        size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(G && g && out && v_out && flag_out, "null pointer");
  B200OCL_CHECK_ARG(t >= 1 && n >= 1 && pitch >= n, "need t >= 1, n >= 1 and pitch >= n");
  B200OCL_CHECK_ARG(isfinite(margin) && margin >= 0.0 && isfinite(eps) && eps > 0.0,
                    "need a finite margin >= 0 and a finite eps > 0");
  if (t > GEM_MAX_T) {
    set_error("b200ocl_gem_project: t=%d exceeds the QP's limit of %d task gradients", t, GEM_MAX_T);
    return B200OCL_EUNSUPPORTED;
  }
  const b200ocl_gem_launch L = gem_plan(t, n, sm_count());
  const int rc = check_workspace("b200ocl_gem_project", workspace, workspace_bytes, L.workspace_bytes);
  if (rc) return rc;
  double* part = static_cast<double*>(workspace);
  B200OCL_CUDA(raise_smem_limit<gem_gram_kernel>(L.smem_bytes));
  B200OCL_PROF("gem", 4.0 * (double)(t + 1) * (double)n, stream);
  gem_gram_kernel<<<L.grid, GEM_THREADS, L.smem_bytes, stream>>>(G, pitch, g, n, L, part);
  B200OCL_LAUNCHED();
  B200OCL_CUDA(raise_smem_limit<gem_qp_kernel>(sizeof(GemQpSmem)));
  B200OCL_PROF("gem", 8.0 * (double)L.grid * L.pairs, stream);
  gem_qp_kernel<<<1, GEM_QP_THREADS, sizeof(GemQpSmem), stream>>>(part, L.grid, t, margin, eps, v_out, flag_out,
                                                                  err_flag, kkt_out);
  B200OCL_LAUNCHED();
  B200OCL_PROF("gem", 4.0 * (double)(t + 2) * (double)n, stream);
  gem_project_kernel<<<L.proj_grid, GEM_PROJ_THREADS, 0, stream>>>(G, pitch, t, g, out, n, v_out, flag_out);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

}  // extern "C"
