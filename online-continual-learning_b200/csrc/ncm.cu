// ncm.cu -- the evaluate() path of agents/base.py:118-171 on encoder features (sm_90a).
//
// The reference extracts the feature of every buffered exemplar with one model.features() call per image
// (5000 Python iterations), normalises it, averages per class, normalises the mean (base.py:121-141); then for
// every test batch builds a [B, d, C] broadcast, takes squared distances and the arg-min (base.py:155-170).
// Here the buffer features come from the batched eval-feature pass of the engine and three small kernels do the
// rest:
//   ncm_class_means   one CTA per class: samples of that class in slot order, 4 or 16 feature dimensions per thread,
//                     x / ||x|| accumulated in fp32, mean, normalised mean; deterministic (no atomics)
//   ncm_classify      one warp per test sample: normalise, squared distance to every class mean with the
//                     reference's (f - mu)^2 form, first arg-min, label lookup, correct count (integer atomic)
//   linear_argmax     the non-NCM branch (base.py:172-175): arg-max of the classifier logits
#include <float.h>

#include "common.cuh"

namespace b200ocl {
namespace {

// DPT dimensions per thread: d <= 256 * DPT.  DPT = 4 serves d <= 1024 (32x32 and 84x84 networks), NCM_WIDE_DPT the
// wider features up to NET_MAX_DIM (2560 at 128x128); the per-thread sums run in the same order for every DPT.
constexpr int NCM_MAX_DIM = B200OCL_NET_MAX_DIM;
constexpr int NCM_WIDE_DPT = NCM_MAX_DIM / 256;

template <int DPT>
__global__ void __launch_bounds__(256) ncm_class_means_kernel(const float* __restrict__ feats,
                                                              const long long* __restrict__ labels, int n, int d,
                                                              const long long* __restrict__ class_ids, float* __restrict__ means,
                                                              int* __restrict__ counts) {
  __shared__ float s_red[8];
  __shared__ float s_inv;
  const long long cls = class_ids[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float acc[DPT] = {};
  int count = 0;
  for (int i = 0; i < n; ++i) {
    if (labels[i] != cls) continue;                       // uniform across the CTA
    const float* f = feats + (size_t)i * d;
    float v[DPT], ss = 0.f;
#pragma unroll
    for (int q = 0; q < DPT; ++q) {
      const int dd = tid + q * 256;
      v[q] = dd < d ? f[dd] : 0.f;
      ss = fmaf(v[q], v[q], ss);
    }
    ss = warp_sum(ss);
    if (lane == 0) s_red[warp] = ss;
    __syncthreads();
    if (tid == 0) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += s_red[w];
      s_inv = sqrtf(t);
    }
    __syncthreads();
    const float nrm = s_inv;
#pragma unroll
    for (int q = 0; q < DPT; ++q) acc[q] += v[q] / nrm;    // feature / feature.norm() (base.py:131)
    ++count;
    __syncthreads();
  }
  if (tid == 0) counts[blockIdx.x] = count;
  if (count == 0) return;                                  // the caller draws the reference's random mean for empty classes
  float ss = 0.f;
#pragma unroll
  for (int q = 0; q < DPT; ++q) {
    acc[q] /= (float)count;                                // features.mean(0)
    ss = fmaf(acc[q], acc[q], ss);
  }
  ss = warp_sum(ss);
  if (lane == 0) s_red[warp] = ss;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += s_red[w];
    s_inv = sqrtf(t);
  }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < DPT; ++q) {
    const int dd = tid + q * 256;
    if (dd < d) means[(size_t)blockIdx.x * d + dd] = acc[q] / s_inv;   // mu_y / mu_y.norm() (base.py:139)
  }
}

// NCM: score = squared distance, smaller wins.  LINEAR: score = -(f.w + b), so that one arg-min serves both.
template <bool NCM>
__global__ void __launch_bounds__(256) classify_kernel(const float* __restrict__ feats, int B, int d,
                                                       const float* __restrict__ means, const float* __restrict__ bias, int K,
                                                       const long long* __restrict__ class_ids,
                                                       const long long* __restrict__ truth, long long* __restrict__ pred,
                                                       unsigned long long* __restrict__ n_correct) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (b >= B) return;
  const float* f = feats + (size_t)b * d;
  float inv = 1.f;
  if (NCM) {
    float ss = 0.f;
    for (int dd = lane; dd < d; dd += 32) ss = fmaf(f[dd], f[dd], ss);
    inv = sqrtf(warp_sum(ss));
  }
  float best = FLT_MAX;
  int best_k = 0;
  for (int k = 0; k < K; ++k) {
    const float* mu = means + (size_t)k * d;
    float s = 0.f;
    for (int dd = lane; dd < d; dd += 32) {
      if (NCM) {
        const float df = f[dd] / inv - mu[dd];             // normalised feature (base.py:159-160) minus the mean
        s = fmaf(df, df, s);
      } else {
        s = fmaf(f[dd], mu[dd], s);
      }
    }
    s = warp_sum(s);
    if (!NCM) s = -(s + bias[k]);
    if (s < best) {                                        // strict: the first minimum wins
      best = s;
      best_k = k;
    }
  }
  if (lane == 0) {
    const long long label = class_ids ? class_ids[best_k] : (long long)best_k;
    if (pred) pred[b] = label;
    if (truth && n_correct && truth[b] == label) atomicAdd(n_correct, 1ull);
  }
}

}  // namespace
}  // namespace b200ocl

extern "C" {

int b200ocl_ncm_class_means(const float* feats, const int64_t* labels, int n, int d, const int64_t* class_ids, int K,
                            float* means, int* counts, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(n >= 0 && d >= 1 && d <= NCM_MAX_DIM && K >= 0, "need n >= 0, 1 <= d <= 4096, K >= 0");
  if (K == 0) return B200OCL_OK;
  B200OCL_CHECK_ARG(class_ids && means && counts && (n == 0 || (feats && labels)), "null pointer");
  B200OCL_PROF("ncm", 4.0 * n * (double)d + 8.0 * n * (double)K, stream);
  const long long* lab = reinterpret_cast<const long long*>(labels);
  const long long* ids = reinterpret_cast<const long long*>(class_ids);
  if (d <= 256 * 4)
    ncm_class_means_kernel<4><<<K, 256, 0, stream>>>(feats, lab, n, d, ids, means, counts);
  else
    ncm_class_means_kernel<NCM_WIDE_DPT><<<K, 256, 0, stream>>>(feats, lab, n, d, ids, means, counts);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

int b200ocl_ncm_classify(const float* feats, int B, int d, const float* means, int K, const int64_t* class_ids,
                         const int64_t* truth, int64_t* pred, uint64_t* n_correct, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(B >= 0 && d >= 1 && K >= 1, "need B >= 0, d >= 1, K >= 1");
  if (B == 0) return B200OCL_OK;
  B200OCL_CHECK_ARG(feats && means, "null pointer");
  B200OCL_PROF("ncm", 4.0 * B * (double)d + 4.0 * K * (double)d, stream);
  classify_kernel<true><<<(B + 7) / 8, 256, 0, stream>>>(feats, B, d, means, nullptr, K,
                                                         reinterpret_cast<const long long*>(class_ids),
                                                         reinterpret_cast<const long long*>(truth),
                                                         reinterpret_cast<long long*>(pred),
                                                         reinterpret_cast<unsigned long long*>(n_correct));
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

int b200ocl_linear_argmax(const float* feats, int B, int d, const float* weight, const float* bias, int C,
                          const int64_t* truth, int64_t* pred, uint64_t* n_correct, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(B >= 0 && d >= 1 && C >= 1, "need B >= 0, d >= 1, C >= 1");
  if (B == 0) return B200OCL_OK;
  B200OCL_CHECK_ARG(feats && weight && bias, "null pointer");
  B200OCL_PROF("ncm", 4.0 * B * (double)d + 4.0 * C * (double)d, stream);
  classify_kernel<false><<<(B + 7) / 8, 256, 0, stream>>>(feats, B, d, weight, bias, C, nullptr,
                                                          reinterpret_cast<const long long*>(truth),
                                                          reinterpret_cast<long long*>(pred),
                                                          reinterpret_cast<unsigned long long*>(n_correct));
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

}  // extern "C"
