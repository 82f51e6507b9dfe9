// der.cu -- DER++'s logit-matching loss (Buzzega et al., NeurIPS 2020): alpha * mean((z - L[idx])^2) over the
// memory batch's logits z [n,C] and the logits L [mem_rows,C] the network gave those samples when they were stored.
#include <math.h>

#include "common.cuh"

namespace b200ocl {
namespace {

constexpr int LM_THREADS = 256;

// One CTA.  Thread t owns the elements t, t + 256, ... of the n x C block (a fixed assignment), keeps its sum of squares
// in double, and the 256 partials are added by a fixed shared-memory tree: the same inputs give the same bits on every
// launch, with no atomics.  Each gradient element is formed in double and rounded once.
__global__ void __launch_bounds__(LM_THREADS) logit_mse_kernel(const float* __restrict__ z, const float* __restrict__ mem,
                                                               int mem_rows, const long long* __restrict__ idx, int n,
                                                               int C, double alpha, float* __restrict__ loss,
                                                               float* __restrict__ dz, int* __restrict__ err) {
  __shared__ double s_sum[LM_THREADS];
  const long long total = (long long)n * C;
  const double inv = 1.0 / (double)total;
  const double g = 2.0 * alpha * inv;
  double acc = 0.0;
  for (long long e = threadIdx.x; e < total; e += LM_THREADS) {
    const int row = (int)(e / C);
    const int col = (int)(e - (long long)row * C);
    const long long slot = idx[row];
    if (slot < 0 || slot >= mem_rows) {        // the row adds nothing and gets no gradient
      if (err && col == 0) *err = 1;
      dz[e] = 0.f;
      continue;
    }
    const double d = (double)z[e] - (double)mem[slot * C + col];
    acc += d * d;
    dz[e] = (float)(g * d);
  }
  s_sum[threadIdx.x] = acc;
  __syncthreads();
#pragma unroll
  for (int s = LM_THREADS / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) s_sum[threadIdx.x] += s_sum[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss = (float)(alpha * s_sum[0] * inv);
}

}  // namespace
}  // namespace b200ocl

extern "C" {

int b200ocl_logit_mse(const float* z, const float* mem, int mem_rows, const int64_t* idx, int n, int C, double alpha,
                      float* loss, float* dz, int* err_flag, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(z && mem && idx && loss && dz, "null pointer");
  B200OCL_CHECK_ARG(n >= 1 && C >= 1 && mem_rows >= 1, "need n >= 1, C >= 1 and mem_rows >= 1");
  B200OCL_PROF("misc", 16.0 * (double)n * C, stream);
  logit_mse_kernel<<<1, LM_THREADS, 0, stream>>>(z, mem, mem_rows, reinterpret_cast<const long long*>(idx), n, C, alpha,
                                                 loss, dz, err_flag);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

}  // extern "C"
