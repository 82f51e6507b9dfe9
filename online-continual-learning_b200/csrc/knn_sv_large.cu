// knn_sv_large.cu -- kNN Shapley values for candidate sets beyond the fused kernel's 1024 (sm_90a).
//
// Same arithmetic as knn_sv.cu (utils/buffer/aser_utils.py:29-59,94-116): squared-L2 distances in
// direct-difference form, a full ascending sort of (distance, candidate) with ties lowest-index-first, the
// Shapley recurrence as a reverse scan over the sorted order, scatter to candidate order and the callers'
// column sum / max / min over eval rows.  What changes is where a row lives: C keys do not fit in registers,
// so a CTA (1024 threads, persistent over eval rows) keeps the row's 64-bit keys in a global scratch line
// (L2-resident: 512 KB at C = 50 000) and sorts them with a bitonic network whose stages run in 16 384-key
// shared-memory blocks whenever the compare distance allows (all but 3 of the 136 stages at C = 65 536).
// Used for the transposed memory sweep (1 000 eval rows x 50 000 candidates, SURVEY.md section 8d config 5)
// and for ASER configurations with n_smp_cls * num_classes > 1024.
#include <float.h>

#include "common.cuh"

namespace b200ocl {
namespace {

constexpr int KL_THREADS = 1024;
constexpr int KL_WARPS = 32;
constexpr int KL_S = 16384;            // keys per shared-memory block (128 KB)
constexpr int KL_MAX_D = 4096;

struct KnnLargeParams {
  const float* eval_f;
  const long long* eval_y;
  const float* cand_f;
  const long long* cand_y;
  int E, C, Cpad, d, k;
  float* sv;
  float* col_sum;
  float* col_max;
  float* col_min;
  float* part;                  // [gridDim][3][C]
  unsigned long long* keys;     // [gridDim][Cpad]
  unsigned int* counter;
};

__device__ __forceinline__ void cmpx(unsigned long long& a, unsigned long long& b, bool up) {
  const bool sw = up ? (a > b) : (a < b);
  const unsigned long long t = a;
  a = sw ? b : a;
  b = sw ? t : b;
}

// stages j = j_hi, j_hi/2, ..., 1 of merge size k2 on the block [base, base + n) held in shared memory
__device__ __forceinline__ void local_stages(unsigned long long* sk, int n, int base, int k2, int j_hi) {
  for (int j = j_hi; j > 0; j >>= 1) {
    for (int t = threadIdx.x; t < n / 2; t += KL_THREADS) {
      const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));      // insert a 0 bit at position log2(j)
      const bool up = (((base + lo) & k2) == 0);
      unsigned long long a = sk[lo], b = sk[lo + j];
      cmpx(a, b, up);
      sk[lo] = a;
      sk[lo + j] = b;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(KL_THREADS, 1) knn_sv_large_kernel(KnnLargeParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* sk = reinterpret_cast<unsigned long long*>(smem_raw);      // [min(Cpad, KL_S)]
  const int S = p.Cpad < KL_S ? p.Cpad : KL_S;
  float* se = reinterpret_cast<float*>(sk + S);                                  // [d] eval row
  float* sscan = se + p.d;                                                       // [KL_THREADS]
  __shared__ bool is_last;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  unsigned long long* gk = p.keys + (size_t)blockIdx.x * p.Cpad;
  float* my_part = p.part + (size_t)blockIdx.x * 3 * p.C;
  const bool want_red = p.col_sum || p.col_max || p.col_min;
  if (want_red)
    for (int c = tid; c < p.C; c += KL_THREADS) {
      my_part[c] = 0.f;
      my_part[p.C + c] = -FLT_MAX;
      my_part[2 * p.C + c] = FLT_MAX;
    }

  for (int row = blockIdx.x; row < p.E; row += gridDim.x) {
    __syncthreads();
    for (int dd = tid; dd < p.d; dd += KL_THREADS) se[dd] = p.eval_f[(size_t)row * p.d + dd];
    __syncthreads();
    // ---- distances: one warp per candidate, lanes stride the features, fixed shuffle tree
    for (int c = warp; c < p.Cpad; c += KL_WARPS) {
      unsigned long long key = ~0ull;
      if (c < p.C) {
        const float* cf = p.cand_f + (size_t)c * p.d;
        float acc = 0.f;
        for (int dd = lane; dd < p.d; dd += 32) {
          const float df = se[dd] - __ldg(cf + dd);
          acc = fmaf(df, df, acc);
        }
        acc = warp_sum(acc);
        key = (static_cast<unsigned long long>(__float_as_uint(acc)) << 32) | static_cast<unsigned int>(c);
      }
      if (lane == 0) gk[c] = key;
    }
    __syncthreads();
    // ---- bitonic sort, ascending.  Stages with compare distance < S run inside shared-memory blocks.
    for (int base = 0; base < p.Cpad; base += S) {               // every merge size up to S, block by block
      for (int t = tid; t < S; t += KL_THREADS) sk[t] = gk[base + t];
      __syncthreads();
      for (int k2 = 2; k2 <= S; k2 <<= 1) local_stages(sk, S, base, k2, k2 >> 1);
      for (int t = tid; t < S; t += KL_THREADS) gk[base + t] = sk[t];
      __syncthreads();
    }
    for (int k2 = 2 * S; k2 <= p.Cpad; k2 <<= 1) {
      for (int j = k2 >> 1; j >= S; j >>= 1) {                   // far partners: through global memory (L2)
        for (int t = tid; t < p.Cpad / 2; t += KL_THREADS) {
          const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));
          const bool up = ((lo & k2) == 0);
          unsigned long long a = gk[lo], b = gk[lo + j];
          cmpx(a, b, up);
          gk[lo] = a;
          gk[lo + j] = b;
        }
        __syncthreads();
      }
      for (int base = 0; base < p.Cpad; base += S) {
        for (int t = tid; t < S; t += KL_THREADS) sk[t] = gk[base + t];
        __syncthreads();
        local_stages(sk, S, base, k2, S >> 1);
        for (int t = tid; t < S; t += KL_THREADS) gk[base + t] = sk[t];
        __syncthreads();
      }
    }
    // ---- Shapley recurrence over the sorted order: s_pos = sum_{t >= pos} (m_t - m_{t+1}) * factor_t
    const long long ey = p.eval_y[row];
    const int L = p.Cpad / KL_THREADS > 0 ? p.Cpad / KL_THREADS : 1;     // contiguous sorted positions per thread
    const int p0 = tid * L;
    float run = 0.f;
    int m_next = 0;
    {
      const int pn = p0 + L;
      if (pn < p.C) m_next = (p.cand_y[static_cast<unsigned int>(gk[pn])] == ey) ? 1 : 0;
    }
    for (int q = L - 1; q >= 0; --q) {                            // pass 1: the thread's own suffix total
      const int pos = p0 + q;
      if (pos < p.C && pos < p.Cpad) {
        const int mq = (p.cand_y[static_cast<unsigned int>(gk[pos])] == ey) ? 1 : 0;
        if (mq != m_next) {
          const int rank = pos + 1;
          const float f = (pos == p.C - 1) ? __fdiv_rn(1.f, (float)p.C)
                                           : __fdiv_rn((float)min(rank, p.k), (float)rank * (float)p.k);
          run += (float)(mq - m_next) * f;
        }
        m_next = mq;
      }
    }
    if (p0 >= p.Cpad) run = 0.f;
    sscan[tid] = run;
    __syncthreads();
    if (warp == 0) {                                              // suffix scan of the 1024 thread totals
      float carry = 0.f;
      for (int blk = KL_THREADS / 32 - 1; blk >= 0; --blk) {
        float v = sscan[blk * 32 + lane];
        float incl = v;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          const float o = __shfl_down_sync(FULL_MASK, incl, off);
          if (lane + off < 32) incl += o;
        }
        sscan[blk * 32 + lane] = incl - v + carry;               // exclusive: sum of the totals above this thread
        carry += __shfl_sync(FULL_MASK, incl, 0);
      }
    }
    __syncthreads();
    {
      float acc = sscan[tid];
      int mn = 0;
      const int pn = p0 + L;
      if (pn < p.C) mn = (p.cand_y[static_cast<unsigned int>(gk[pn])] == ey) ? 1 : 0;
      for (int q = L - 1; q >= 0; --q) {                          // pass 2: values, scatter, column reductions
        const int pos = p0 + q;
        if (pos < p.C && pos < p.Cpad) {
          const unsigned int idx = static_cast<unsigned int>(gk[pos]);
          const int mq = (p.cand_y[idx] == ey) ? 1 : 0;
          if (mq != mn) {
            const int rank = pos + 1;
            const float f = (pos == p.C - 1) ? __fdiv_rn(1.f, (float)p.C)
                                             : __fdiv_rn((float)min(rank, p.k), (float)rank * (float)p.k);
            acc += (float)(mq - mn) * f;
          }
          mn = mq;
          if (p.sv) p.sv[(size_t)row * p.C + idx] = acc;
          if (want_red) {                                         // idx is unique within a row: no conflicts
            my_part[idx] += acc;
            my_part[p.C + idx] = fmaxf(my_part[p.C + idx], acc);
            my_part[2 * p.C + idx] = fminf(my_part[2 * p.C + idx], acc);
          }
        }
      }
    }
  }
  if (!want_red) return;
  __threadfence();
  __syncthreads();
  if (tid == 0) is_last = (atomicAdd(p.counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (int c = tid; c < p.C; c += KL_THREADS) {                   // partials combined in CTA order
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

}  // namespace

int knn_large_cpad(int C) {
  int cp = 1024;
  while (cp < C) cp <<= 1;
  return cp;
}

int knn_large_max_d() { return KL_MAX_D; }

size_t knn_large_part_region(int C, int sms) { return align_up((size_t)sms * 3 * (size_t)C * sizeof(float), 256); }

size_t knn_large_workspace_bytes(int C, int sms) {
  return 256 + knn_large_part_region(C, sms) + (size_t)sms * (size_t)knn_large_cpad(C) * sizeof(unsigned long long);
}

// The scratch-line part of knn_plan (knn_sv.cu): E >= 1, d <= KL_MAX_D.
void knn_large_plan(int E, int C, int d, bool want_red, int sms, b200ocl_knn_launch* L) {
  L->family = B200OCL_KNN_LARGE;
  L->cpad = knn_large_cpad(C);
  const int S = L->cpad < KL_S ? L->cpad : KL_S;
  L->block_keys = S;
  int far = 0;                                                     // the kernel's far-partner loop, counted
  for (int k2 = 2 * S; k2 <= L->cpad; k2 <<= 1)
    for (int j = k2 >> 1; j >= S; j >>= 1) ++far;
  L->far_stages = far;
  L->grid = E < sms ? E : sms;
  L->n_tiles = E;                                                  // one eval row per CTA iteration
  L->tiles_per_cta = (E + L->grid - 1) / L->grid;
  L->smem_bytes = (size_t)S * sizeof(unsigned long long) + (size_t)(d + KL_THREADS) * sizeof(float);
  L->smem_limit = 200 * 1024;
  L->part_bytes = want_red ? (size_t)L->grid * 3 * (size_t)C * sizeof(float) : 0;
  L->key_offset = 256 + knn_large_part_region(C, sms);
  L->key_bytes = (size_t)L->grid * L->cpad * sizeof(unsigned long long);
}

int launch_knn_large(const float* eval_f, const long long* eval_y, const float* cand_f, const long long* cand_y, int E, int C,
                     int d, int k, float* sv, float* col_sum, float* col_max, float* col_min, void* workspace,
                     size_t workspace_bytes, const b200ocl_knn_launch& L, cudaStream_t stream) {
  const int rc = check_workspace("b200ocl_knn_sv", workspace, workspace_bytes, L.workspace_bytes);
  if (rc) return rc;
  KnnLargeParams p{};
  p.eval_f = eval_f; p.eval_y = eval_y; p.cand_f = cand_f; p.cand_y = cand_y;
  p.E = E; p.C = C; p.Cpad = L.cpad; p.d = d; p.k = k;
  p.sv = sv; p.col_sum = col_sum; p.col_max = col_max; p.col_min = col_min;
  unsigned char* w = static_cast<unsigned char*>(workspace);
  p.counter = reinterpret_cast<unsigned int*>(w);
  p.part = reinterpret_cast<float*>(w + 256);
  p.keys = reinterpret_cast<unsigned long long*>(w + L.key_offset);
  B200OCL_CUDA(cudaMemsetAsync(p.counter, 0, sizeof(unsigned int), stream));
  B200OCL_CUDA(raise_smem_limit<knn_sv_large_kernel>(L.smem_limit));
  B200OCL_PROF("knn_sv", 4.0 * d * ((double)E + C) + 8.0 * ((double)E + C) + 4.0 * C * 3 + (sv ? 4.0 * E * C : 0.0), stream);
  knn_sv_large_kernel<<<L.grid, KL_THREADS, L.smem_bytes, stream>>>(p);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

}  // namespace b200ocl
