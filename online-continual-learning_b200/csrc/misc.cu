// misc.cu -- ranking, buffer row gather/scatter (sm_90a).
#include <float.h>

#include "common.cuh"

namespace b200ocl {
namespace {

// ----------------------------------------------------------------------------- rank_desc
// One CTA, shared-memory bitonic sort of (order-preserving score bits, index) 64-bit keys.
// Descending score, ties lowest index first == ascending sort of (~orderable(score), index).
__device__ __forceinline__ unsigned int orderable(float f) {
  const unsigned int b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__global__ void __launch_bounds__(1024) rank_desc_kernel(const float* __restrict__ a, float sa,
                                                         const float* __restrict__ b, float sb, int n, int npad,
                                                         long long* __restrict__ idx_out, int n_out,
                                                         float* __restrict__ score_out) {
  extern __shared__ __align__(16) unsigned long long keys[];
  const int tid = threadIdx.x;
  for (int i = tid; i < npad; i += blockDim.x) {
    unsigned long long key = ~0ull;
    if (i < n) {
      float s = a[i] * sa;
      if (b) s += b[i] * sb;
      if (s == 0.f) s = 0.f;  // -0 -> +0 so that equal scores compare equal
      if (score_out) score_out[i] = s;
      key = (static_cast<unsigned long long>(~orderable(s)) << 32) | static_cast<unsigned int>(i);
    }
    keys[i] = key;
  }
  __syncthreads();
  for (int k2 = 2; k2 <= npad; k2 <<= 1) {
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < npad / 2; t += blockDim.x) {
        const int lo = ((t / j) * 2 * j) + (t % j);
        const int hi = lo + j;
        const bool up = ((lo & k2) == 0);
        const unsigned long long x = keys[lo], y = keys[hi];
        if (up ? (x > y) : (x < y)) {
          keys[lo] = y;
          keys[hi] = x;
        }
      }
      __syncthreads();
    }
  }
  for (int i = tid; i < n_out; i += blockDim.x) idx_out[i] = (long long)(keys[i] & 0xffffffffull);
}

// ----------------------------------------------------------------------------- rows
// One CTA per row (grid-stride), 16-byte vectors when the row size and all bases allow it.
template <bool SCATTER, typename VecT>
__global__ void __launch_bounds__(256) move_rows_kernel(const unsigned char* __restrict__ src,
                                                        const long long* __restrict__ idx, int n_rows,
                                                        size_t row_bytes, unsigned char* __restrict__ dst) {
  const size_t nvec = row_bytes / sizeof(VecT);
  for (int r = blockIdx.x; r < n_rows; r += gridDim.x) {
    const long long ir = idx[r];
    const VecT* s = reinterpret_cast<const VecT*>(src + (SCATTER ? (size_t)r : (size_t)ir) * row_bytes);
    VecT* d = reinterpret_cast<VecT*>(dst + (SCATTER ? (size_t)ir : (size_t)r) * row_bytes);
    for (size_t v = threadIdx.x; v < nvec; v += blockDim.x) d[v] = s[v];
  }
}

template <bool SCATTER>
int move_rows(const void* src, const int64_t* idx, int n_rows, size_t row_bytes, void* dst, cudaStream_t stream) {
  if (n_rows == 0) return B200OCL_OK;
  const bool vec16 = (row_bytes % 16 == 0) && ((reinterpret_cast<uintptr_t>(src) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(dst) & 15) == 0);
  const int grid = n_rows < 8 * sm_count() ? n_rows : 8 * sm_count();
  B200OCL_PROF("move_rows", 2.0 * n_rows * (double)row_bytes, stream);
  if (vec16)
    move_rows_kernel<SCATTER, uint4><<<grid, 256, 0, stream>>>(static_cast<const unsigned char*>(src),
                                                               reinterpret_cast<const long long*>(idx), n_rows,
                                                               row_bytes, static_cast<unsigned char*>(dst));
  else
    move_rows_kernel<SCATTER, unsigned int><<<grid, 256, 0, stream>>>(static_cast<const unsigned char*>(src),
                                                                      reinterpret_cast<const long long*>(idx), n_rows,
                                                                      row_bytes, static_cast<unsigned char*>(dst));
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

// ----------------------------------------------------------------------------- ASER memory replacement
// Replacement rule of reference utils/buffer/aser_update.py:88-112 taken on the device.  `order` is the
// descending SV ranking over [buffered candidates (n_cand_buf) | current batch (n_cur)].  Current samples
// ranked inside the first n_cand_buf places replace, pairwise in rank order, the buffered candidates
// ranked below them:  buffer[cand_slot[small_j]] <- cur[large_j - n_cand_buf].  CTA j finds the j-th pair
// by a ballot scan of the ranking (one warp, <= 4096 ranks) and moves that row; CTA 0 also publishes
// pairs_out = [count, src_0.., dst_0..] (src/dst padded with -1) for the host mirror, read asynchronously.
__global__ void __launch_bounds__(256) aser_replace_kernel(const long long* __restrict__ order, int n_total,
                                                           int n_cand_buf, const long long* __restrict__ cand_slot,
                                                           const unsigned char* __restrict__ cur_x,
                                                           const long long* __restrict__ cur_y, int n_cur,
                                                           size_t row_bytes, unsigned char* __restrict__ buffer_img,
                                                           long long* __restrict__ buffer_label,
                                                           long long* __restrict__ pairs_out) {
  __shared__ long long s_src, s_dst;
  __shared__ int s_count;
  const int j = blockIdx.x;
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    long long src = -1, dst = -1;
    int seen_cur = 0, seen_buf = 0;
    // top part: the j-th current-batch sample in rank order
    for (int base = 0; base < n_cand_buf; base += 32) {
      const int r = base + lane;
      const long long o = (r < n_cand_buf) ? order[r] : -1;
      const bool f = o >= n_cand_buf;
      const unsigned int m = __ballot_sync(0xffffffffu, f);
      const int before = seen_cur + __popc(m & ((1u << lane) - 1u));
      if (f && before == j) src = o - n_cand_buf;
      seen_cur += __popc(m);
    }
    // bottom part: the j-th buffered candidate in rank order
    for (int base = n_cand_buf; base < n_total; base += 32) {
      const int r = base + lane;
      const long long o = (r < n_total) ? order[r] : (long long)n_cand_buf;
      const bool f = o < n_cand_buf;
      const unsigned int m = __ballot_sync(0xffffffffu, f);
      const int before = seen_buf + __popc(m & ((1u << lane) - 1u));
      if (f && before == j) dst = cand_slot[o];
      seen_buf += __popc(m);
    }
    // exactly one lane (or none) holds each value
    for (int o = 16; o > 0; o >>= 1) {
      src = max(src, __shfl_xor_sync(0xffffffffu, src, o));
      dst = max(dst, __shfl_xor_sync(0xffffffffu, dst, o));
    }
    if (lane == 0) {
      s_src = src;
      s_dst = dst;
      s_count = seen_cur;   // == seen_buf by counting
      if (pairs_out) {
        if (j == 0) pairs_out[0] = seen_cur;
        pairs_out[1 + j] = (j < seen_cur) ? src : -1;
        pairs_out[1 + n_cur + j] = (j < seen_cur) ? dst : -1;
      }
    }
  }
  __syncthreads();
  if (j >= s_count || s_src < 0 || s_dst < 0) return;
  const uint4* s = reinterpret_cast<const uint4*>(cur_x + (size_t)s_src * row_bytes);
  uint4* d = reinterpret_cast<uint4*>(buffer_img + (size_t)s_dst * row_bytes);
  for (size_t v = threadIdx.x; v < row_bytes / 16; v += blockDim.x) d[v] = s[v];
  if (threadIdx.x == 0) buffer_label[s_dst] = cur_y[s_src];
}

// Stream feeder (continuum/data_utils.py:38-54 + ToTensor): image i of the output = source image perm[i],
// uint8 HWC -> fp32 CHW, value / 255 with an IEEE division (bit-identical to torchvision's CPU ToTensor).
// One CTA per image: coalesced word loads of the interleaved bytes into shared memory, planar coalesced stores.
__global__ void __launch_bounds__(256) stream_prepare_kernel(const unsigned char* __restrict__ src,
                                                             const long long* __restrict__ perm, float* __restrict__ dst,
                                                             int hw) {
  extern __shared__ __align__(16) unsigned char s_img[];
  const size_t row = (size_t)hw * 3;
  const unsigned char* in = src + (size_t)(perm ? perm[blockIdx.x] : blockIdx.x) * row;
  const int words = (int)(row / 4);
  for (int i = threadIdx.x; i < words; i += blockDim.x)
    reinterpret_cast<unsigned int*>(s_img)[i] = __ldg(reinterpret_cast<const unsigned int*>(in) + i);
  for (int i = words * 4 + threadIdx.x; i < (int)row; i += blockDim.x) s_img[i] = in[i];
  __syncthreads();
  float* out = dst + (size_t)blockIdx.x * row;
  for (int o = threadIdx.x; o < (int)row; o += blockDim.x) {
    const int c = o / hw, pix = o - c * hw;
    out[o] = u8_unit(s_img[pix * 3 + c]);
  }
}

// float64 -> fp32 as the host CPU's conversion does it (torch's .float(), x86 cvtsd2ss): IEEE round to nearest even with
// subnormal results kept (no .ftz), overflow to inf, and a NaN kept with its sign and the top 22 bits of its payload,
// quiet bit set.  cvt.rn.f32.f64 alone would return the canonical NaN.
__device__ __forceinline__ float f64_to_f32_host(double v) {
  if (v != v) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    return __uint_as_float(((unsigned)(b >> 32) & 0x80000000u) | 0x7fc00000u | ((unsigned)(b >> 29) & 0x3fffffu));
  }
  return __double2float_rn(v);
}

// Stream feeder for the reference's non-stationary tasks (continuum/non_stationary.py:9-124 give float64 HWC images in
// [0,1]; ToTensor on them only transposes, then .float(), continuum/data_utils.py:38-54): image i of the output = source
// image perm[i], float64 HWC -> fp32 CHW.  One CTA per chunk of PREP64_PIX consecutive pixels of one image (any
// number of rows, or part of one): its 3 * PREP64_PIX source doubles are contiguous and read once with 16-byte loads,
// converted and staged as fp32 (12 KB, not a whole image), then written as three contiguous plane segments.
constexpr int PREP64_THREADS = 256;
constexpr int PREP64_PIX = 1024;
constexpr int PREP64_LOADS = 3 * PREP64_PIX / 2 / PREP64_THREADS;   // double2 loads per thread

__global__ void __launch_bounds__(PREP64_THREADS) stream_prepare_f64_kernel(const double* __restrict__ src,
                                                                            const long long* __restrict__ perm,
                                                                            float* __restrict__ dst, long long hw,
                                                                            int chunks) {
  __shared__ float s_val[3 * PREP64_PIX];
  const long long img = blockIdx.x / chunks;
  const long long p0 = (long long)(blockIdx.x - img * chunks) * PREP64_PIX;
  const int pix = (int)min((long long)PREP64_PIX, hw - p0);
  const int cnt = 3 * pix;
  const double* in = src + ((perm ? perm[img] : img) * hw + p0) * 3;
  // a chunk starts 16-byte aligned or one double past it: the odd leading and trailing doubles load alone
  const int lead = (int)((reinterpret_cast<uintptr_t>(in) >> 3) & 1);
  const int pairs = (cnt - lead) >> 1;
  const double2* in2 = reinterpret_cast<const double2*>(in + lead);
  double2 v[PREP64_LOADS];
#pragma unroll
  for (int j = 0; j < PREP64_LOADS; ++j) {
    const int k = threadIdx.x + j * PREP64_THREADS;
    if (k < pairs) v[j] = __ldg(in2 + k);
  }
#pragma unroll
  for (int j = 0; j < PREP64_LOADS; ++j) {
    const int k = threadIdx.x + j * PREP64_THREADS;
    if (k < pairs) {
      s_val[lead + 2 * k] = f64_to_f32_host(v[j].x);
      s_val[lead + 2 * k + 1] = f64_to_f32_host(v[j].y);
    }
  }
  if (threadIdx.x == 0) {
    if (lead) s_val[0] = f64_to_f32_host(__ldg(in));
    if ((cnt - lead) & 1) s_val[cnt - 1] = f64_to_f32_host(__ldg(in + cnt - 1));
  }
  __syncthreads();
  float* out = dst + img * 3 * hw + p0;
  for (int o = threadIdx.x; o < cnt; o += PREP64_THREADS) {
    const int c = o / pix, p = o - c * pix;
    out[c * hw + p] = s_val[p * 3 + c];
  }
}

// A-GEM projection (agents/agem.py:60-80): g <- g - (g.g_ref / g_ref.g_ref) g_ref when g.g_ref < 0, else g.
// Launch 1: per-CTA fp64 partials of the two dot products over the flat gradient arenas; launch 2: every thread
// re-reduces the (<= 296) partials in CTA order -- same value everywhere, deterministic -- and writes the result.
__global__ void __launch_bounds__(256) agem_dots_kernel(const float* __restrict__ g, const float* __restrict__ gref, size_t n,
                                                        double* __restrict__ part) {
  __shared__ double s_a[8], s_b[8];
  double a = 0.0, b = 0.0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const double x = (double)g[i], r = (double)gref[i];
    a += x * r;
    b += r * r;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(FULL_MASK, a, o);
    b += __shfl_xor_sync(FULL_MASK, b, o);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    s_a[warp] = a;
    s_b[warp] = b;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double ta = 0.0, tb = 0.0;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      ta += s_a[w];
      tb += s_b[w];
    }
    part[2 * blockIdx.x] = ta;
    part[2 * blockIdx.x + 1] = tb;
  }
}

__global__ void __launch_bounds__(256) agem_apply_kernel(const float* __restrict__ g, const float* __restrict__ gref, size_t n,
                                                         const double* __restrict__ part, int n_part, float* __restrict__ out,
                                                         float* __restrict__ dots_out) {
  double prod = 0.0, prod_ref = 0.0;
  for (int b = 0; b < n_part; ++b) {
    prod += part[2 * b];
    prod_ref += part[2 * b + 1];
  }
  const bool project = prod < 0.0;
  const float coef = project ? (float)(prod / prod_ref) : 0.f;
  if (dots_out && blockIdx.x == 0 && threadIdx.x == 0) {
    dots_out[0] = (float)prod;
    dots_out[1] = (float)prod_ref;
  }
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = project ? g[i] - coef * gref[i] : g[i];
}

// GSS-greedy scores (utils/buffer/gss_greedy_update.py:84,120; buffer_utils.py:50-55): cosine similarity of a flat gradient g
// with each of K stored gradients, and the maximum.  Launch 1: per-CTA fp64 partials of the K dot products, the K squared
// norms and |g|^2 over the CTA's slice of the 1.1 M parameters; launch 2: partials reduced in CTA order (deterministic).
constexpr int GC_MAX_K = 64;
__global__ void __launch_bounds__(256) grad_cosine_partial_kernel(const float* __restrict__ mem, const float* __restrict__ g, int K,
                                                                  size_t n, double* __restrict__ part) {
  __shared__ double s_red[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* my = part + (size_t)blockIdx.x * (2 * K + 1);
  for (int q = 0; q <= 2 * K; ++q) {
    double acc = 0.0;
    const float* row = (q < K) ? mem + (size_t)q * n : (q < 2 * K ? mem + (size_t)(q - K) * n : g);
    const float* other = (q < K) ? g : row;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
      acc += (double)row[i] * (double)other[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(FULL_MASK, acc, o);
    if (lane == 0) s_red[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += s_red[w];
      my[q] = t;
    }
    __syncthreads();
  }
}

__global__ void grad_cosine_final_kernel(const double* __restrict__ part, int n_part, int K, float eps, float* __restrict__ cos_out,
                                         float* __restrict__ max_out) {
  __shared__ float s_cos[GC_MAX_K];
  const int k = threadIdx.x;
  double ng = 0.0;
  for (int b = 0; b < n_part; ++b) ng += part[(size_t)b * (2 * K + 1) + 2 * K];
  if (k < K) {
    double dot = 0.0, nm = 0.0;
    for (int b = 0; b < n_part; ++b) {
      dot += part[(size_t)b * (2 * K + 1) + k];
      nm += part[(size_t)b * (2 * K + 1) + K + k];
    }
    const float den = fmaxf(sqrtf((float)nm) * sqrtf((float)ng), eps);     // (w1 * w2.t()).clamp(min=eps)
    s_cos[k] = (float)dot / den;
    if (cos_out) cos_out[k] = s_cos[k];
  }
  __syncthreads();
  if (k == 0 && max_out) {
    float m = s_cos[0];
    for (int j = 1; j < K; ++j) m = fmaxf(m, s_cos[j]);
    *max_out = m;
  }
}
}  // namespace
}  // namespace b200ocl

extern "C" {

int b200ocl_rank_desc(const float* a, float sa, const float* b, float sb, int n, int64_t* idx_out, int n_out,
                      float* score_out, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(a && idx_out, "null pointer");
  B200OCL_CHECK_ARG(n >= 0 && n_out >= 0 && n_out <= n, "need 0 <= n_out <= n");
  if (n > 4096) {
    set_error("b200ocl_rank_desc: n=%d exceeds the limit of 4096", n);
    return B200OCL_EUNSUPPORTED;
  }
  if (n == 0) return B200OCL_OK;
  int npad = 2;
  while (npad < n) npad <<= 1;
  const int threads = npad / 2 < 32 ? 32 : (npad / 2 > 1024 ? 1024 : npad / 2);
  B200OCL_PROF("rank_desc", 12.0 * n, stream);
  rank_desc_kernel<<<1, threads, (size_t)npad * sizeof(unsigned long long), stream>>>(
      a, sa, b, sb, n, npad, reinterpret_cast<long long*>(idx_out), n_out, score_out);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

int b200ocl_gather_rows(const void* src, const int64_t* idx, int n_rows, size_t row_bytes, void* dst, void* stream) {
  using namespace b200ocl;
  B200OCL_CHECK_ARG(n_rows >= 0 && row_bytes % 4 == 0, "need n_rows >= 0 and row_bytes % 4 == 0");
  B200OCL_CHECK_ARG(n_rows == 0 || (src && idx && dst), "null pointer");
  return move_rows<false>(src, idx, n_rows, row_bytes, dst, static_cast<cudaStream_t>(stream));
}

int b200ocl_scatter_rows(const void* src, const int64_t* idx, int n_rows, size_t row_bytes, void* dst, void* stream) {
  using namespace b200ocl;
  B200OCL_CHECK_ARG(n_rows >= 0 && row_bytes % 4 == 0, "need n_rows >= 0 and row_bytes % 4 == 0");
  B200OCL_CHECK_ARG(n_rows == 0 || (src && idx && dst), "null pointer");
  return move_rows<true>(src, idx, n_rows, row_bytes, dst, static_cast<cudaStream_t>(stream));
}

int b200ocl_stream_prepare(const uint8_t* src_hwc, const int64_t* perm, int n, int h, int w, float* dst_chw, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(n >= 0 && h > 0 && w > 0, "need n >= 0 and positive h, w");
  if (n == 0) return B200OCL_OK;
  B200OCL_CHECK_ARG(src_hwc && dst_chw, "null pointer");
  const size_t row = (size_t)h * w * 3;
  B200OCL_CHECK_ARG(row % 4 == 0 && (reinterpret_cast<uintptr_t>(src_hwc) & 3) == 0, "image rows must be 4-byte aligned");
  B200OCL_CHECK_ARG(row <= 200 * 1024, "image larger than shared memory");
  B200OCL_CUDA(raise_smem_limit<stream_prepare_kernel>(200 * 1024));
  B200OCL_PROF("stream_prepare", 5.0 * n * (double)row, stream);
  stream_prepare_kernel<<<n, 256, row, stream>>>(src_hwc, reinterpret_cast<const long long*>(perm), dst_chw, h * w);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

int b200ocl_stream_prepare_f64(const double* src_hwc, const int64_t* perm, int n, int h, int w, float* dst_chw,
                               void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(n >= 0 && h > 0 && w > 0, "need n >= 0 and positive h, w");
  if (n == 0) return B200OCL_OK;
  B200OCL_CHECK_ARG(src_hwc && dst_chw, "null pointer");
  B200OCL_CHECK_ARG((reinterpret_cast<uintptr_t>(src_hwc) & 7) == 0, "source must be 8-byte aligned");
  const long long hw = (long long)h * w;
  const long long chunks = (hw + PREP64_PIX - 1) / PREP64_PIX;
  B200OCL_CHECK_ARG(chunks * n <= 0x7fffffffLL, "more than 2^31 - 1 pixel chunks");
  B200OCL_PROF("stream_prepare_f64", 12.0 * n * 3.0 * (double)hw, stream);
  stream_prepare_f64_kernel<<<(unsigned)(chunks * n), PREP64_THREADS, 0, stream>>>(
      src_hwc, reinterpret_cast<const long long*>(perm), dst_chw, hw, (int)chunks);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

size_t b200ocl_agem_project_workspace_bytes(void) { return (size_t)2 * 2 * 148 * sizeof(double) + 256; }

int b200ocl_agem_project(const float* g, const float* g_ref, float* out, size_t n, float* dots_out, void* workspace,
                         size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n == 0) return B200OCL_OK;
  B200OCL_CHECK_ARG(g && g_ref && out, "null pointer");
  const int rc = check_workspace("b200ocl_agem_project", workspace, workspace_bytes, b200ocl_agem_project_workspace_bytes());
  if (rc) return rc;
  int grid = 2 * sm_count();
  if (grid > 296) grid = 296;
  double* part = static_cast<double*>(workspace);
  B200OCL_PROF("misc", 8.0 * n, stream);
  agem_dots_kernel<<<grid, 256, 0, stream>>>(g, g_ref, n, part);
  B200OCL_LAUNCHED();
  B200OCL_PROF("misc", 12.0 * n, stream);
  agem_apply_kernel<<<grid, 256, 0, stream>>>(g, g_ref, n, part, grid, out, dots_out);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

size_t b200ocl_grad_cosine_workspace_bytes(int K) {
  if (K < 0) K = 0;
  return (size_t)296 * (2 * (size_t)K + 1) * sizeof(double) + 256;
}

int b200ocl_grad_cosine(const float* mem_grads, const float* g, int K, size_t n, float* cos_out, float* max_out, void* workspace,
                        size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(K >= 1 && K <= GC_MAX_K && n >= 1, "need 1 <= K <= 64 and n >= 1");
  B200OCL_CHECK_ARG(mem_grads && g && (cos_out || max_out), "null pointer");
  const int rc = check_workspace("b200ocl_grad_cosine", workspace, workspace_bytes, b200ocl_grad_cosine_workspace_bytes(K));
  if (rc) return rc;
  int grid = 2 * sm_count();
  if (grid > 296) grid = 296;
  double* part = static_cast<double*>(workspace);
  B200OCL_PROF("misc", 4.0 * (double)n * (2.0 * K + 1.0), stream);
  grad_cosine_partial_kernel<<<grid, 256, 0, stream>>>(mem_grads, g, K, n, part);
  B200OCL_LAUNCHED();
  B200OCL_PROF("misc", 8.0 * grid * (2.0 * K + 1.0), stream);
  grad_cosine_final_kernel<<<1, GC_MAX_K, 0, stream>>>(part, grid, K, 1e-8f, cos_out, max_out);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

int b200ocl_aser_replace(const int64_t* order, int n_total, int n_cand_buf, const int64_t* cand_slot, const void* cur_x,
                         const int64_t* cur_y, int n_cur, size_t row_bytes, void* buffer_img, int64_t* buffer_label,
                         int64_t* pairs_out, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(n_cur >= 0 && n_cand_buf >= 0 && n_total == n_cand_buf + n_cur, "need n_total == n_cand_buf + n_cur");
  if (n_cur == 0) return B200OCL_OK;
  B200OCL_CHECK_ARG(order && (cand_slot || n_cand_buf == 0) && cur_x && cur_y && buffer_img && buffer_label, "null pointer");
  B200OCL_CHECK_ARG(row_bytes % 16 == 0 && ((reinterpret_cast<uintptr_t>(cur_x) | reinterpret_cast<uintptr_t>(buffer_img)) & 15) == 0,
                    "rows must be 16-byte aligned multiples of 16 bytes");
  B200OCL_PROF("move_rows", 2.0 * n_cur * (double)row_bytes, stream);
  aser_replace_kernel<<<n_cur, 256, 0, stream>>>(reinterpret_cast<const long long*>(order), n_total, n_cand_buf,
                                                 reinterpret_cast<const long long*>(cand_slot),
                                                 static_cast<const unsigned char*>(cur_x),
                                                 reinterpret_cast<const long long*>(cur_y), n_cur, row_bytes,
                                                 static_cast<unsigned char*>(buffer_img),
                                                 reinterpret_cast<long long*>(buffer_label),
                                                 reinterpret_cast<long long*>(pairs_out));
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

}  // extern "C"
