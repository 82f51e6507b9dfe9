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
//   cosine_argmax     PCR's evaluation: arg-max of the cosine between the feature and each classifier row
//   linear_argmax_ea  the same launch with the error analysis of base.py:144-226 (--error_analysis) riding along:
//                     predicted task, per-row fp64 logit sums over the new / old class sets, wrong rows bucketed by
//                     the set they were predicted into; rows_mean the classifier's weight / bias means over a row set
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

// Side outputs of the error-analysis arg-max (EA): every pointer is set when EA is.
struct EaArgs {
  const unsigned char* sets;    // [C] bit 0: class of the last task (new_labels_zombie); bit 1: set(old_labels) - zombie
  const long long* task_of;     // [C] class_task_map, -1 where a class has no entry
  long long* pred_task;         // [B] task of the predicted class
  double* set_sums;             // [B,2] the row's logits summed over the bit-0 / bit-1 classes, in class order, in fp64
  unsigned long long* counts;   // [4] wrong rows predicted into a bit-0 / bit-1 / neither class; rows predicted unmapped
};

// NCM: score = squared distance, smaller wins.  LINEAR: score = -(f.w + b), so that one arg-min serves both.
// EA (LINEAR only) adds the error-analysis outputs; the arg-max and the hit count run the same instructions either way.
// COS (LINEAR only, no bias): score = -<f / (||f|| + eps), w / (||w|| + eps)>, eps = 1e-6.
template <bool NCM, bool EA = false, bool COS = false>
__global__ void __launch_bounds__(256) classify_kernel(const float* __restrict__ feats, int B, int d,
                                                       const float* __restrict__ means, const float* __restrict__ bias, int K,
                                                       const long long* __restrict__ class_ids,
                                                       const long long* __restrict__ truth, long long* __restrict__ pred,
                                                       unsigned long long* __restrict__ n_correct, EaArgs ea = EaArgs()) {
  static_assert(!(NCM && EA), "the error analysis reads logits: linear branch only");
  static_assert(!(COS && (NCM || EA)), "the cosine arg-max is a linear-branch form without the error analysis");
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (b >= B) return;
  const float* f = feats + (size_t)b * d;
  float inv = 1.f;
  if (NCM || COS) {
    float ss = 0.f;
    for (int dd = lane; dd < d; dd += 32) ss = fmaf(f[dd], f[dd], ss);
    inv = sqrtf(warp_sum(ss));
  }
  float best = FLT_MAX;
  int best_k = 0;
  double sum_new = 0.0, sum_old = 0.0;
  for (int k = 0; k < K; ++k) {
    const float* mu = means + (size_t)k * d;
    float s = 0.f, ww = 0.f;
    for (int dd = lane; dd < d; dd += 32) {
      if (NCM) {
        const float df = f[dd] / inv - mu[dd];             // normalised feature (base.py:159-160) minus the mean
        s = fmaf(df, df, s);
      } else {
        s = fmaf(f[dd], mu[dd], s);
        if (COS) ww = fmaf(mu[dd], mu[dd], ww);
      }
    }
    s = warp_sum(s);
    if (COS) s = -((s / (inv + 1e-6f)) / (sqrtf(warp_sum(ww)) + 1e-6f));
    else if (!NCM) s = -(s + bias[k]);
    if (EA) {                                              // -s is the logit f.w + b exactly
      const unsigned m = ea.sets[k];
      if (m & 1u) sum_new += (double)(-s);
      if (m & 2u) sum_old += (double)(-s);
    }
    if (s < best) {                                        // strict: the first minimum wins
      best = s;
      best_k = k;
    }
  }
  if (lane == 0) {
    const long long label = class_ids ? class_ids[best_k] : (long long)best_k;
    if (pred) pred[b] = label;
    if (truth && n_correct && truth[b] == label) atomicAdd(n_correct, 1ull);
    if (EA) {
      const long long t = ea.task_of[best_k];
      ea.pred_task[b] = t;
      ea.set_sums[2 * (size_t)b] = sum_new;
      ea.set_sums[2 * (size_t)b + 1] = sum_old;
      if (t < 0) atomicAdd(&ea.counts[3], 1ull);           // class_task_map[p] raises KeyError in the reference
      if (truth[b] != label) {
        const unsigned m = ea.sets[best_k];
        atomicAdd(&ea.counts[(m & 1u) ? 0 : (m & 2u) ? 1 : 2], 1ull);
      }
    }
  }
}

// One CTA: mean of weight[rows] (n x d elements) and of bias[rows], each summed in fp64 in a fixed order (thread-strided
// partial sums, then a fixed tree) and rounded to fp32 once.  n == 0 gives NaN, as torch's mean of an empty tensor.
__global__ void __launch_bounds__(256) rows_mean_kernel(const float* __restrict__ weight, const float* __restrict__ bias,
                                                        int d, const long long* __restrict__ rows, int n,
                                                        float* __restrict__ out) {
  __shared__ double s_w[256], s_b[256];
  const int tid = threadIdx.x;
  const long long total = (long long)n * d;
  double w = 0.0, bb = 0.0;
  for (long long i = tid; i < total; i += 256) w += (double)weight[(size_t)rows[i / d] * d + i % d];
  for (int i = tid; i < n; i += 256) bb += (double)bias[rows[i]];
  s_w[tid] = w;
  s_b[tid] = bb;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (tid < o) {
      s_w[tid] += s_w[tid + o];
      s_b[tid] += s_b[tid + o];
    }
    __syncthreads();
  }
  if (tid == 0) {
    out[0] = (float)(s_w[0] / (double)total);
    out[1] = (float)(s_b[0] / (double)n);
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

int b200ocl_cosine_argmax(const float* feats, int B, int d, const float* weight, int C, const int64_t* truth,
                          int64_t* pred, uint64_t* n_correct, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(B >= 0 && d >= 1 && C >= 1, "need B >= 0, d >= 1, C >= 1");
  if (B == 0) return B200OCL_OK;
  B200OCL_CHECK_ARG(feats && weight, "null pointer");
  B200OCL_PROF("ncm", 4.0 * B * (double)d + 8.0 * C * (double)d, stream);
  classify_kernel<false, false, true><<<(B + 7) / 8, 256, 0, stream>>>(feats, B, d, weight, nullptr, C, nullptr,
                                                                       reinterpret_cast<const long long*>(truth),
                                                                       reinterpret_cast<long long*>(pred),
                                                                       reinterpret_cast<unsigned long long*>(n_correct));
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

int b200ocl_linear_argmax_ea(const float* feats, int B, int d, const float* weight, const float* bias, int C,
                             const int64_t* truth, const uint8_t* class_sets, const int64_t* class_task, int64_t* pred,
                             uint64_t* n_correct, int64_t* pred_task, double* set_sums, uint64_t* counts, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(B >= 0 && d >= 1 && C >= 1, "need B >= 0, d >= 1, C >= 1");
  if (B == 0) return B200OCL_OK;
  B200OCL_CHECK_ARG(feats && weight && bias && truth && class_sets && class_task && pred_task && set_sums && counts,
                    "null pointer");
  B200OCL_PROF("ncm", 4.0 * B * (double)d + 4.0 * C * (double)d, stream);
  EaArgs ea;
  ea.sets = class_sets;
  ea.task_of = reinterpret_cast<const long long*>(class_task);
  ea.pred_task = reinterpret_cast<long long*>(pred_task);
  ea.set_sums = set_sums;
  ea.counts = reinterpret_cast<unsigned long long*>(counts);
  classify_kernel<false, true><<<(B + 7) / 8, 256, 0, stream>>>(feats, B, d, weight, bias, C, nullptr,
                                                                reinterpret_cast<const long long*>(truth),
                                                                reinterpret_cast<long long*>(pred),
                                                                reinterpret_cast<unsigned long long*>(n_correct), ea);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

int b200ocl_rows_mean(const float* weight, const float* bias, int C, int d, const int64_t* rows, int n, float* out,
                      void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(C >= 1 && d >= 1 && n >= 0, "need C >= 1, d >= 1, n >= 0");
  B200OCL_CHECK_ARG(weight && bias && out && (n == 0 || rows), "null pointer");
  B200OCL_PROF("ncm", 4.0 * n * (double)d, stream);
  rows_mean_kernel<<<1, 256, 0, stream>>>(weight, bias, d, reinterpret_cast<const long long*>(rows), n, out);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

}  // extern "C"
