// knn_sv.cu -- fused kNN Shapley-value kernel (sm_90a).
//
// Replaces, in one launch, the reference chain
//   sorted_cand_ind -> euclidean_distance -> argsort -> label gather -> indicator diff ->
//   factor -> flip.cumsum.flip -> index_put scatter -> sum/max/min over rows
// (utils/buffer/aser_utils.py:29-59,94-116; utils/utils.py:93-95; aser_retrieve.py:79-86;
// aser_update.py:80), which the reference runs as ~30 ATen kernels and a materialised
// [E*C, d] broadcast.
//
// Work decomposition (persistent CTAs, 8 warps):
//   phase 1  a tile of TE eval rows x all C candidates: squared-L2 distances in
//            direct-difference form, register-tiled (TE/8 rows x up to 8 candidates per
//            thread), operands staged through shared memory in 32-wide feature chunks;
//            the [TE][Cpad] distance tile stays in shared memory (never touches HBM);
//   phase 2  one warp per eval row: (distance, candidate) packed into a 64-bit key
//            (distance bits are order-preserving because d2 >= 0; the low word breaks ties
//            lowest-index-first) and sorted by a register-resident bitonic network, KPL keys
//            per lane, warp shuffles for the cross-lane stages -- no shared-memory traffic;
//   phase 3  label match against the eval label, the Shapley recurrence as a reverse
//            scan (lane-local then a 5-step shuffle scan), scatter back to candidate order,
//            optional coalesced store of the SV row, and per-warp column sum/max/min kept in
//            shared memory across ALL tiles of the CTA;
//   finish   fixed-order combine of the 8 warps, one partial per CTA, and the last CTA to
//            arrive reduces the partials in CTA order: deterministic, no float atomics.
#include <float.h>

#include "common.cuh"

namespace b200ocl {
namespace {

constexpr int KNN_THREADS = 256;
constexpr int KNN_WARPS = 8;
constexpr int KNN_DK = 32;  // feature chunk staged per iteration

struct KnnSvParams {
  const float* eval_f;
  const long long* eval_y;
  const float* cand_f;
  const long long* cand_y;
  int E, C, d, k;
  float* sv;
  float* col_sum;
  float* col_max;
  float* col_min;
  float* part;            // [gridDim][3][C]  (sum, max, min)
  unsigned int* counter;  // zeroed before launch
  int n_tiles;
};

// Shared-memory column swizzle: lane l of the sorting warp reads positions l*KPL+q; the XOR
// spreads those 32 addresses over 32 banks.
template <int KPL>
__device__ __forceinline__ int swz(int p) {
  return p ^ ((p >> 5) & (KPL - 1));
}

template <int KPL>
__device__ __forceinline__ void bitonic_sort_blocked(unsigned long long (&key)[KPL], int lane) {
  constexpr int N = 32 * KPL;
#pragma unroll
  for (int k2 = 2; k2 <= N; k2 <<= 1) {
#pragma unroll
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      if (j < KPL) {
        // both elements of the pair live in this thread
#pragma unroll
        for (int i = 0; i < KPL; ++i) {
          const int partner = i ^ j;
          if (partner > i) {
            const bool up = (k2 < KPL) ? ((i & k2) == 0) : (((lane * KPL) & k2) == 0);
            const unsigned long long a = key[i], b = key[partner];
            const bool sw = up ? (a > b) : (a < b);
            key[i] = sw ? b : a;
            key[partner] = sw ? a : b;
          }
        }
      } else {
        // partner element lives in lane ^ (j / KPL), same register slot
        const int lj = j / KPL;
        const bool up = (((lane * KPL) & k2) == 0);
        const bool lower = ((lane & lj) == 0);
        const bool keep_min = (up == lower);
#pragma unroll
        for (int i = 0; i < KPL; ++i) {
          const unsigned long long a = key[i];
          const unsigned long long o = __shfl_xor_sync(FULL_MASK, a, lj);
          key[i] = keep_min ? (a < o ? a : o) : (a > o ? a : o);
        }
      }
    }
  }
}

template <int KPL, int TE>
__global__ void __launch_bounds__(KNN_THREADS) knn_sv_kernel(KnnSvParams p) {
  constexpr int CPAD = 32 * KPL;
  constexpr int TM = TE / KNN_WARPS;       // eval rows per warp
  constexpr int NJ = KPL < 8 ? KPL : 8;    // candidates per thread per pass
  constexpr int CT = 32 * NJ;              // candidates per distance pass
  constexpr int DK = KNN_DK;

  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* sd = reinterpret_cast<float*>(smem_raw);               // [TE][CPAD] distances, later SV rows
  long long* slab = reinterpret_cast<long long*>(sd + TE * CPAD);  // [CPAD] candidate labels
  float* se = reinterpret_cast<float*>(slab + CPAD);            // [DK][TE+1]
  float* sc = se + DK * (TE + 1);                               // [DK][CT+1]
  float* wred = sc + DK * (CT + 1);                             // [3][8][CPAD] per-warp col sum/max/min

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool want_red = (p.col_sum != nullptr) || (p.col_max != nullptr) || (p.col_min != nullptr);

  for (int c = tid; c < CPAD; c += KNN_THREADS) slab[c] = (c < p.C) ? p.cand_y[c] : 0;
  if (want_red) {
    for (int c = lane; c < CPAD; c += 32) {
      wred[(0 * KNN_WARPS + warp) * CPAD + c] = 0.f;
      wred[(1 * KNN_WARPS + warp) * CPAD + c] = -FLT_MAX;
      wred[(2 * KNN_WARPS + warp) * CPAD + c] = FLT_MAX;
    }
  }

  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    const int row0 = tile * TE;

    // ------------------------------------------------------------------ phase 1: distances
    // Wide variant for 513..1024 candidates (the memory-sweep shape): with TE = 16 the row-per-warp tiling
    // below has only 2 x 8 pairs per thread for 10 shared-memory loads per feature (LSU-bound, far
    // off the FMA bound).  Here warp w owns candidates [128w, 128w+128) for ALL 16 rows: 16 x 4 pairs per
    // thread for five 16-byte loads per feature, operands prefetched into registers one 8-feature chunk ahead.
    // Same per-pair fma order over the features, so the distances are bit-identical to the other tiling.
    bool wide_done = false;
    if constexpr (KPL == 32 && TE == 16) {
      // knn_wide_form (host, below) restates this predicate for the launch plan: keep the two equal.
      if (p.d % 8 == 0 && (reinterpret_cast<uintptr_t>(p.eval_f) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.cand_f) & 15) == 0) {
        constexpr int DKW = 8;
        float* se_w = se;   // [DKW][16]
        float* sc_w = sc;   // [DKW][CPAD]   (8192 floats <= DK * (CT + 1))
        float acc[16][4];
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
        float4 pc[8], pe = make_float4(0.f, 0.f, 0.f, 0.f);
        auto fetch = [&](int k0) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int item = tid + KNN_THREADS * i;          // (candidate, half of the 8-feature chunk)
            const int c = item >> 1, half = item & 1;
            pc[i] = (c < p.C) ? __ldg(reinterpret_cast<const float4*>(p.cand_f + (size_t)c * p.d + k0 + half * 4))
                              : make_float4(0.f, 0.f, 0.f, 0.f);
          }
          if (tid < 32) {
            const int r = tid >> 1, half = tid & 1;
            pe = (row0 + r < p.E) ? __ldg(reinterpret_cast<const float4*>(p.eval_f + (size_t)(row0 + r) * p.d + k0 + half * 4))
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
          }
        };
        fetch(0);
        for (int k0 = 0; k0 < p.d; k0 += DKW) {
          __syncthreads();   // previous chunk (and the previous tile's phase 3) fully consumed
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int item = tid + KNN_THREADS * i;
            const int c = item >> 1, half = item & 1;
            sc_w[(half * 4 + 0) * CPAD + c] = pc[i].x;
            sc_w[(half * 4 + 1) * CPAD + c] = pc[i].y;
            sc_w[(half * 4 + 2) * CPAD + c] = pc[i].z;
            sc_w[(half * 4 + 3) * CPAD + c] = pc[i].w;
          }
          if (tid < 32) {
            const int r = tid >> 1, half = tid & 1;
            se_w[(half * 4 + 0) * 16 + r] = pe.x;
            se_w[(half * 4 + 1) * 16 + r] = pe.y;
            se_w[(half * 4 + 2) * 16 + r] = pe.z;
            se_w[(half * 4 + 3) * 16 + r] = pe.w;
          }
          __syncthreads();
          if (k0 + DKW < p.d) fetch(k0 + DKW);   // in flight during the arithmetic below
#pragma unroll
          for (int kk = 0; kk < DKW; ++kk) {
            float a[16];
#pragma unroll
            for (int i4 = 0; i4 < 4; ++i4)
              *reinterpret_cast<float4*>(&a[4 * i4]) = *reinterpret_cast<const float4*>(se_w + kk * 16 + 4 * i4);
            const float4 b4 = *reinterpret_cast<const float4*>(sc_w + kk * CPAD + warp * 128 + lane * 4);
            const float b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int i = 0; i < 16; ++i)
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const float df = a[i] - b[j];
                acc[i][j] = fmaf(df, df, acc[i][j]);
              }
          }
        }
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) sd[i * CPAD + swz<KPL>(warp * 128 + lane * 4 + j)] = acc[i][j];
        __syncthreads();   // a warp sorts rows whose distances every warp contributed to
        wide_done = true;
      }
    }
    for (int c0 = 0; !wide_done && c0 < CPAD; c0 += CT) {
      float acc[TM][NJ];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) acc[i][j] = 0.f;

      for (int k0 = 0; k0 < p.d; k0 += DK) {
        __syncthreads();  // previous chunk (and previous tile's phase 3) fully consumed
        for (int idx = tid; idx < TE * DK; idx += KNN_THREADS) {
          const int r = idx / DK, kk = idx % DK;
          const int gr = row0 + r, gk = k0 + kk;
          se[kk * (TE + 1) + r] = (gr < p.E && gk < p.d) ? p.eval_f[(size_t)gr * p.d + gk] : 0.f;
        }
        for (int idx = tid; idx < CT * DK; idx += KNN_THREADS) {
          const int c = idx / DK, kk = idx % DK;
          const int gc = c0 + c, gk = k0 + kk;
          sc[kk * (CT + 1) + c] = (gc < p.C && gk < p.d) ? p.cand_f[(size_t)gc * p.d + gk] : 0.f;
        }
        __syncthreads();
#pragma unroll 4
        for (int kk = 0; kk < DK; ++kk) {
          float a[TM], b[NJ];
#pragma unroll
          for (int i = 0; i < TM; ++i) a[i] = se[kk * (TE + 1) + warp * TM + i];
#pragma unroll
          for (int j = 0; j < NJ; ++j) b[j] = sc[kk * (CT + 1) + lane + 32 * j];
#pragma unroll
          for (int i = 0; i < TM; ++i)
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
              const float df = a[i] - b[j];
              acc[i][j] = fmaf(df, df, acc[i][j]);
            }
        }
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const int c = c0 + lane + 32 * j;
          sd[(warp * TM + i) * CPAD + swz<KPL>(c)] = acc[i][j];
        }
    }
    __syncwarp();  // a warp sorts only rows it produced itself

    // ------------------------------------------------------------------ phases 2+3: one warp per row
#pragma unroll 1
    for (int i = 0; i < TM; ++i) {
      const int lr = warp * TM + i;
      const int row = row0 + lr;
      if (row >= p.E) break;  // warp-uniform
      const long long ey = p.eval_y[row];
      float* srow = sd + lr * CPAD;

      unsigned long long key[KPL];
#pragma unroll
      for (int q = 0; q < KPL; ++q) {
        const int pos = lane * KPL + q;
        const unsigned int bits = __float_as_uint(srow[swz<KPL>(pos)]);
        key[q] = (pos < p.C) ? ((static_cast<unsigned long long>(bits) << 32) | static_cast<unsigned int>(pos))
                             : ~0ull;
      }
      bitonic_sort_blocked<KPL>(key, lane);

      // match indicators at sorted positions lane*KPL + q, one bit per register slot
      unsigned int mbits = 0;
#pragma unroll
      for (int q = 0; q < KPL; ++q) {
        const int pos = lane * KPL + q;
        const unsigned int idx = static_cast<unsigned int>(key[q]);
        if (pos < p.C && slab[idx & (CPAD - 1)] == ey) mbits |= (1u << q);
      }
      unsigned int m_next_lane = __shfl_down_sync(FULL_MASK, mbits, 1) & 1u;
      if (lane == 31) m_next_lane = 0u;

      // s_pos = sum_{t >= pos} (m_t - m_{t+1}) * factor_t     (aser_utils.py:38-52)
      float s[KPL];
      float run = 0.f;
#pragma unroll
      for (int q = KPL - 1; q >= 0; --q) {
        const int pos = lane * KPL + q;
        const int mq = (int)((mbits >> q) & 1u);
        const int mn = (q == KPL - 1) ? (int)m_next_lane : (int)((mbits >> (q + 1 < KPL ? q + 1 : q)) & 1u);
        float term = 0.f;
        if (pos < p.C && mq != mn) {
          const int rank = pos + 1;
          const float f = (pos == p.C - 1) ? __fdiv_rn(1.f, (float)p.C)
                                           : __fdiv_rn((float)min(rank, p.k), (float)rank * (float)p.k);
          term = (float)(mq - mn) * f;
        }
        run += term;
        s[q] = run;
      }
      float incl = run;  // inclusive suffix sum over lanes
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const float v = __shfl_down_sync(FULL_MASK, incl, off);
        if (lane + off < 32) incl += v;
      }
      float above = __shfl_down_sync(FULL_MASK, incl, 1);
      if (lane == 31) above = 0.f;

      __syncwarp();  // every lane has consumed its distances; srow becomes the SV row
#pragma unroll
      for (int q = 0; q < KPL; ++q) {
        const int pos = lane * KPL + q;
        if (pos < p.C) {
          const unsigned int idx = static_cast<unsigned int>(key[q]);
          const float v = s[q] + above;
          if (p.sv) srow[idx] = v;
          if (want_red) {
            float* ws = wred + (0 * KNN_WARPS + warp) * CPAD + idx;
            float* wx = wred + (1 * KNN_WARPS + warp) * CPAD + idx;
            float* wn = wred + (2 * KNN_WARPS + warp) * CPAD + idx;
            *ws += v;
            *wx = fmaxf(*wx, v);
            *wn = fminf(*wn, v);
          }
        }
      }
      if (p.sv) {
        __syncwarp();
        for (int c = lane; c < p.C; c += 32) p.sv[(size_t)row * p.C + c] = srow[c];
      }
      __syncwarp();
    }
  }

  if (!want_red) return;
  // ------------------------------------------------------------------ finish: deterministic reduction
  __syncthreads();
  float* my_part = p.part + (size_t)blockIdx.x * 3 * p.C;
  for (int c = tid; c < p.C; c += KNN_THREADS) {
    float sum = 0.f, mx = -FLT_MAX, mn = FLT_MAX;
#pragma unroll
    for (int w = 0; w < KNN_WARPS; ++w) {
      sum += wred[(0 * KNN_WARPS + w) * CPAD + c];
      mx = fmaxf(mx, wred[(1 * KNN_WARPS + w) * CPAD + c]);
      mn = fminf(mn, wred[(2 * KNN_WARPS + w) * CPAD + c]);
    }
    my_part[0 * p.C + c] = sum;
    my_part[1 * p.C + c] = mx;
    my_part[2 * p.C + c] = mn;
  }
  __threadfence();
  __syncthreads();
  __shared__ bool is_last;
  if (tid == 0) is_last = (atomicAdd(p.counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (int c = tid; c < p.C; c += KNN_THREADS) {
    double sum = 0.0;
    float mx = -FLT_MAX, mn = FLT_MAX;
    for (unsigned int b = 0; b < gridDim.x; ++b) {
      const float* q = p.part + (size_t)b * 3 * p.C;
      sum += (double)__ldcg(q + c);
      mx = fmaxf(mx, __ldcg(q + p.C + c));
      mn = fminf(mn, __ldcg(q + 2 * p.C + c));
    }
    if (p.col_sum) p.col_sum[c] = (float)sum;
    if (p.col_max) p.col_max[c] = mx;
    if (p.col_min) p.col_min[c] = mn;
  }
}

constexpr size_t knn_smem_bytes(int kpl, int te) {
  const int cpad = 32 * kpl;
  const int ct = 32 * (kpl < 8 ? kpl : 8);
  return (size_t)(te * cpad + KNN_DK * (te + 1) + KNN_DK * (ct + 1) + 3 * KNN_WARPS * cpad) * sizeof(float) +
         (size_t)cpad * sizeof(long long);
}

// Host copy of the wide phase-1 predicate that knn_sv_kernel evaluates in phase 1 (KPL == 32, TE == 16, d % 8 == 0,
// eval_f and cand_f 16-byte aligned).  The kernel decides on its own; this copy only reports the decision in the
// launch plan, so it must stay equal to the kernel's.
bool knn_wide_form(int kpl, int te, int d, bool aligned) { return kpl == 32 && te == 16 && d % 8 == 0 && aligned; }

size_t knn_fused_workspace_bytes(int C, int sms) {
  return 256 + align_up((size_t)sms * 3 * (size_t)C * sizeof(float), 256);
}

template <int KPL, int TE>
int launch_knn(const KnnSvParams& p0, const b200ocl_knn_launch& L, cudaStream_t stream) {
  KnnSvParams p = p0;
  static_assert(knn_smem_bytes(KPL, TE) <= 227 * 1024, "kNN-SV tile does not fit in shared memory");
  p.n_tiles = L.n_tiles;
  B200OCL_CUDA((raise_smem_limit<knn_sv_kernel<KPL, TE>>(L.smem_limit)));
  B200OCL_PROF("knn_sv", 4.0 * p.d * ((double)p.E + p.C) + 8.0 * ((double)p.E + p.C) + 4.0 * p.C * 3 + (p.sv ? 4.0 * p.E * p.C : 0.0), stream);
  knn_sv_kernel<KPL, TE><<<L.grid, KNN_THREADS, L.smem_bytes, stream>>>(p);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

template <int KPL>
int dispatch_te(const KnnSvParams& p, const b200ocl_knn_launch& L, cudaStream_t stream) {
  if (L.te == 8) return launch_knn<KPL, 8>(p, L, stream);
  if constexpr (KPL == 32) {
    return launch_knn<KPL, 16>(p, L, stream);
  } else {
    return launch_knn<KPL, 32>(p, L, stream);
  }
}

}  // namespace

// knn_sv_large.cu
int knn_large_max_d();
size_t knn_large_workspace_bytes(int C, int sms);
void knn_large_plan(int E, int C, int d, bool want_red, int sms, b200ocl_knn_launch* L);
int launch_knn_large(const float* eval_f, const long long* eval_y, const float* cand_f, const long long* cand_y, int E, int C,
                     int d, int k, float* sv, float* col_sum, float* col_max, float* col_min, void* workspace,
                     size_t workspace_bytes, const b200ocl_knn_launch& L, cudaStream_t stream);

size_t knn_workspace_bytes(int C, int sms) {
  if (C < 0) C = 0;
  return C > B200OCL_KNN_MAX_CAND ? knn_large_workspace_bytes(C, sms) : knn_fused_workspace_bytes(C, sms);
}

// The one place that decides which kNN-SV kernel a call launches (b200ocl_knn_sv launches what this returns;
// b200ocl_knn_sv_plan reports it).  Host only.  E, C >= 1; C <= B200OCL_KNN_MAX_CAND_LARGE, and d <= the large kernel's
// limit when C > B200OCL_KNN_MAX_CAND (the callers check both).
b200ocl_knn_launch knn_plan(int E, int C, int d, bool aligned, bool want_red, int sms) {
  b200ocl_knn_launch L{};
  L.sms = sms;
  L.workspace_bytes = knn_workspace_bytes(C, sms);
  if (C > B200OCL_KNN_MAX_CAND) {   // rows too long for the register-resident sort: scratch-line path
    knn_large_plan(E, C, d, want_red, sms, &L);
    return L;
  }
  L.family = B200OCL_KNN_FUSED;
  L.kpl = C <= 32 ? 1 : C <= 64 ? 2 : C <= 128 ? 4 : C <= 256 ? 8 : C <= 512 ? 16 : 32;
  // Few rows: small tiles so that more SMs take part.  Many rows: 32-row tiles for operand reuse
  // (KPL=32 keeps 16 so that the three reduction arrays still fit).
  L.te = E <= 8 * sms ? 8 : (L.kpl == 32 ? 16 : 32);
  L.wide = knn_wide_form(L.kpl, L.te, d, aligned) ? 1 : 0;
  L.cpad = 32 * L.kpl;
  L.n_tiles = (E + L.te - 1) / L.te;
  L.grid = L.n_tiles < sms ? L.n_tiles : sms;
  if (L.grid < 1) L.grid = 1;
  L.tiles_per_cta = (L.n_tiles + L.grid - 1) / L.grid;
  L.smem_bytes = knn_smem_bytes(L.kpl, L.te);
  L.smem_limit = L.smem_bytes;      // the launcher raises each instantiation to exactly what it uses
  L.part_bytes = want_red ? (size_t)L.grid * 3 * (size_t)C * sizeof(float) : 0;
  return L;
}

}  // namespace b200ocl

extern "C" {

size_t b200ocl_knn_sv_workspace_bytes(int E, int C, int d) {
  (void)E;
  (void)d;
  return b200ocl::knn_workspace_bytes(C, b200ocl::sm_count());
}

int b200ocl_knn_sv(const float* eval_f, const int64_t* eval_y, const float* cand_f, const int64_t* cand_y, int E,
                   int C, int d, int k, float* sv, float* col_sum, float* col_max, float* col_min, void* workspace,
                   size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(E >= 0 && C >= 0 && d >= 1 && k >= 1, "need E,C >= 0, d >= 1, k >= 1");
  if (C > B200OCL_KNN_MAX_CAND_LARGE) {
    set_error("b200ocl_knn_sv: C=%d exceeds the limit of %d candidates", C, B200OCL_KNN_MAX_CAND_LARGE);
    return B200OCL_EUNSUPPORTED;
  }
  if (C == 0) return B200OCL_OK;
  if (E == 0) {
    // sum over zero rows is 0 (torch: sv_matrix.sum(0)); max/min over zero rows are undefined
    if (col_max || col_min) {
      set_error("b200ocl_knn_sv: col_max/col_min over E=0 rows is undefined");
      return B200OCL_EINVAL;
    }
    if (col_sum) B200OCL_CUDA(cudaMemsetAsync(col_sum, 0, (size_t)C * sizeof(float), stream));
    return B200OCL_OK;
  }
  B200OCL_CHECK_ARG(eval_f && eval_y && cand_f && cand_y, "null input pointer");
  if (C > B200OCL_KNN_MAX_CAND && d > knn_large_max_d()) {
    set_error("b200ocl_knn_sv: d=%d exceeds %d on the large-candidate path", d, knn_large_max_d());
    return B200OCL_EUNSUPPORTED;
  }
  const bool want_red = col_sum || col_max || col_min;
  const bool aligned = (reinterpret_cast<uintptr_t>(eval_f) & 15) == 0 && (reinterpret_cast<uintptr_t>(cand_f) & 15) == 0;
  const b200ocl_knn_launch L = knn_plan(E, C, d, aligned, want_red, sm_count());
  if (L.family == B200OCL_KNN_LARGE)
    return launch_knn_large(eval_f, reinterpret_cast<const long long*>(eval_y), cand_f, reinterpret_cast<const long long*>(cand_y),
                            E, C, d, k, sv, col_sum, col_max, col_min, workspace, workspace_bytes, L, stream);
  KnnSvParams p{};
  p.eval_f = eval_f;
  p.eval_y = reinterpret_cast<const long long*>(eval_y);
  p.cand_f = cand_f;
  p.cand_y = reinterpret_cast<const long long*>(cand_y);
  p.E = E; p.C = C; p.d = d; p.k = k;
  p.sv = sv; p.col_sum = col_sum; p.col_max = col_max; p.col_min = col_min;
  if (want_red) {
    const int rc = check_workspace("b200ocl_knn_sv", workspace, workspace_bytes, L.workspace_bytes);
    if (rc) return rc;
    p.counter = static_cast<unsigned int*>(workspace);
    p.part = reinterpret_cast<float*>(static_cast<unsigned char*>(workspace) + 256);
    B200OCL_CUDA(cudaMemsetAsync(p.counter, 0, sizeof(unsigned int), stream));
  }
  switch (L.kpl) {
    case 1: return dispatch_te<1>(p, L, stream);
    case 2: return dispatch_te<2>(p, L, stream);
    case 4: return dispatch_te<4>(p, L, stream);
    case 8: return dispatch_te<8>(p, L, stream);
    case 16: return dispatch_te<16>(p, L, stream);
    default: return dispatch_te<32>(p, L, stream);
  }
}

int b200ocl_knn_sv_plan(int E, int C, int d, int aligned, int want_red, int sms, b200ocl_knn_launch* out) {
  using namespace b200ocl;
  B200OCL_CHECK_ARG(out, "null pointer");
  B200OCL_CHECK_ARG(E >= 1 && C >= 1 && d >= 1, "need E,C,d >= 1 (b200ocl_knn_sv launches nothing otherwise)");
  B200OCL_CHECK_ARG(sms >= 0, "sms must be 0 (this device) or an SM count");
  if (C > B200OCL_KNN_MAX_CAND_LARGE) {
    set_error("b200ocl_knn_sv_plan: C=%d exceeds the limit of %d candidates", C, B200OCL_KNN_MAX_CAND_LARGE);
    return B200OCL_EUNSUPPORTED;
  }
  if (C > B200OCL_KNN_MAX_CAND && d > knn_large_max_d()) {
    set_error("b200ocl_knn_sv_plan: d=%d exceeds %d on the large-candidate path", d, knn_large_max_d());
    return B200OCL_EUNSUPPORTED;
  }
  *out = knn_plan(E, C, d, aligned != 0, want_red != 0, sms ? sms : sm_count());
  return B200OCL_OK;
}

}  // extern "C"
