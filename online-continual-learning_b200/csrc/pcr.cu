// pcr.cu -- PCR's proxy-contrastive loss (Lin et al., "PCR: Proxy-based Contrastive Replay for Online Class-Incremental
// Continual Learning", CVPR 2023) with both of its gradients, over encoder features F [R,d] and the classifier weight
// W [C,d], whose rows are the class proxies:
//   u_i = F_i / (||F_i|| + eps),  v_c = W_c / (||W_c|| + eps),  g_ic = <u_i, v_c> / tau
//   m_ic = n_c - [c = y_i]  (n_c: rows labelled c; the anchor's own pair is masked, as SupConLoss masks it)
//   Z_i = sum_c m_ic exp(g_ic),  l_i = log Z_i - g_{i,y_i},  L = (1/R) sum_i l_i
// Two launches, both deterministic (fixed reduction orders, no floating-point atomics, nothing depends on the SM count):
//   pcr_rows_kernel     one CTA per row i: ||F_i||, g_i., log Z_i, l_i, the coefficients p_ic - [y_i = c] (kept in the
//                       workspace for the second launch), dL/du_i and dL/dF_i through the normalisation
//   pcr_proxies_kernel  one CTA per class c: dL/dv_c = sum_i coef_ic u_i / (tau R) in row order, dL/dW_c through the
//                       normalisation, the bias gradient 0; one more CTA sums the l_i in double into the loss
#include <math.h>

#include "common.cuh"

namespace b200ocl {
namespace {

constexpr int PCR_THREADS = 256;
constexpr int PCR_WARPS = PCR_THREADS / 32;
constexpr int PCR_MAX_R = 4096;
constexpr int PCR_MAX_D = 2560;
constexpr int PCR_MAX_C = 1024;
constexpr float PCR_EPS = 1e-6f;

struct PcrWs {
  int* counts;       // [C] n_c
  float* den;        // [R] ||F_i|| + eps (1 for a row with a label outside [0, C))
  double* row_loss;  // [R] l_i (0 for a row with a label outside [0, C), NaN for an anchor without positives)
  float* coef;       // [R,C] p_ic - [y_i = c and the anchor has positives]
};

PcrWs pcr_ws(void* base, int R, int C) {
  unsigned char* p = static_cast<unsigned char*>(base);
  PcrWs w;
  w.counts = reinterpret_cast<int*>(p);
  p += align_up((size_t)C * sizeof(int), 256);
  w.den = reinterpret_cast<float*>(p);
  p += align_up((size_t)R * sizeof(float), 256);
  w.row_loss = reinterpret_cast<double*>(p);
  p += align_up((size_t)R * sizeof(double), 256);
  w.coef = reinterpret_cast<float*>(p);
  return w;
}

size_t pcr_ws_bytes(int R, int C) {
  return align_up((size_t)C * sizeof(int), 256) + align_up((size_t)R * sizeof(float), 256) +
         align_up((size_t)R * sizeof(double), 256) + align_up((size_t)R * C * sizeof(float), 256);
}

// ||x||^2 of one row by one warp: lane-strided fmaf partials, then the xor butterfly.  Both kernels take each proxy's
// norm through this one function, so they see the same bits.
__device__ __forceinline__ float warp_sq_norm(const float* __restrict__ x, int d, int lane) {
  float ss = 0.f;
  for (int k = lane; k < d; k += 32) ss = fmaf(x[k], x[k], ss);
  return warp_sum(ss);
}

// Sum of one float per thread over the CTA: warp butterflies, then the eight warp sums in warp order.
__device__ __forceinline__ float block_sum(float v, float* s_red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < PCR_WARPS; ++w) t += s_red[w];
  return t;
}

// Sum of one double per thread over the CTA by a fixed shared-memory tree.
__device__ __forceinline__ double block_sum_d(double v, double* s_red) {
  __syncthreads();
  s_red[threadIdx.x] = v;
  __syncthreads();
#pragma unroll
  for (int s = PCR_THREADS / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) s_red[threadIdx.x] += s_red[threadIdx.x + s];
    __syncthreads();
  }
  return s_red[0];
}

__global__ void __launch_bounds__(PCR_THREADS) pcr_rows_kernel(const float* __restrict__ F,
                                                               const long long* __restrict__ labels, int R, int d,
                                                               const float* __restrict__ W, int C, float tau,
                                                               float* __restrict__ dF, PcrWs ws, int* __restrict__ err) {
  __shared__ float s_f[PCR_MAX_D];
  __shared__ float s_du[PCR_MAX_D];
  __shared__ float s_g[PCR_MAX_C];
  __shared__ float s_vden[PCR_MAX_C];
  __shared__ float s_cv[PCR_MAX_C];      // coef_c / (||W_c|| + eps)
  __shared__ int s_cnt[PCR_MAX_C];
  __shared__ double s_red_d[PCR_THREADS];
  __shared__ float s_red[PCR_WARPS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int i = blockIdx.x;

  for (int c = tid; c < C; c += PCR_THREADS) s_cnt[c] = 0;
  __syncthreads();
  for (int j = tid; j < R; j += PCR_THREADS) {
    const long long y = labels[j];
    if (y >= 0 && y < C) atomicAdd(&s_cnt[y], 1);        // integer counts: the same result in any order
    else if (i == 0 && err) *err = 1;
  }
  __syncthreads();
  if (i == 0)
    for (int c = tid; c < C; c += PCR_THREADS) ws.counts[c] = s_cnt[c];

  const long long yl = labels[i];
  float* dFi = dF + (size_t)i * d;
  float* coef = ws.coef + (size_t)i * C;
  if (yl < 0 || yl >= C) {                                 // a label outside the classifier: nothing from this row
    for (int k = tid; k < d; k += PCR_THREADS) dFi[k] = 0.f;
    for (int c = tid; c < C; c += PCR_THREADS) coef[c] = 0.f;
    if (tid == 0) {
      ws.den[i] = 1.f;
      ws.row_loss[i] = 0.0;
    }
    return;
  }
  const int y = (int)yl;
  const bool pos = s_cnt[y] > 1;                           // the anchor has at least one positive

  const float* Fi = F + (size_t)i * d;
  float ss = 0.f;
  for (int k = tid; k < d; k += PCR_THREADS) {
    const float v = Fi[k];
    s_f[k] = v;
    ss = fmaf(v, v, ss);
  }
  const float nf = sqrtf(block_sum(ss, s_red));           // block_sum's barriers also publish s_f
  const float fden = nf + PCR_EPS;

  for (int c = warp; c < C; c += PCR_WARPS) {
    const float* Wc = W + (size_t)c * d;
    float dot = 0.f;
    for (int k = lane; k < d; k += 32) dot = fmaf(s_f[k], Wc[k], dot);
    dot = warp_sum(dot);
    const float vden = sqrtf(warp_sq_norm(Wc, d, lane)) + PCR_EPS;
    if (lane == 0) {
      s_g[c] = (dot / (fden * vden)) / tau;
      s_vden[c] = vden;
    }
  }
  __syncthreads();

  // log Z_i with the largest contrasted logit taken out; R >= 2 leaves every anchor at least one contrast
  float mx = -INFINITY;
  for (int c = tid; c < C; c += PCR_THREADS)
    if (s_cnt[c] - (c == y) > 0) mx = fmaxf(mx, s_g[c]);
  mx = warp_max(mx);
  __syncthreads();
  if (lane == 0) s_red[warp] = mx;
  __syncthreads();
  mx = s_red[0];
#pragma unroll
  for (int w = 1; w < PCR_WARPS; ++w) mx = fmaxf(mx, s_red[w]);
  double z = 0.0;
  for (int c = tid; c < C; c += PCR_THREADS) {
    const int m = s_cnt[c] - (c == y);
    if (m > 0) z += (double)m * exp((double)s_g[c] - (double)mx);
  }
  z = block_sum_d(z, s_red_d);
  for (int c = tid; c < C; c += PCR_THREADS) {
    const int m = s_cnt[c] - (c == y);
    double p = m > 0 ? (double)m * exp((double)s_g[c] - (double)mx) / z : 0.0;
    if (pos && c == y) p -= 1.0;                           // the positive term; an anchor without positives keeps log Z only
    const float cf = (float)p;
    coef[c] = cf;
    s_cv[c] = cf / s_vden[c];
  }
  if (tid == 0) {
    ws.den[i] = fden;
    ws.row_loss[i] = pos ? (log(z) + (double)mx - (double)s_g[y]) : (double)NAN;   // SupConLoss's 0/0 positive mean
  }
  __syncthreads();

  // dL/du_i = sum_c coef_ic v_c / (tau R), in class order
  const float scale = 1.f / (tau * (float)R);
  float fdu = 0.f;
  for (int k = tid; k < d; k += PCR_THREADS) {
    float acc = 0.f;
    for (int c = 0; c < C; ++c) acc = fmaf(s_cv[c], W[(size_t)c * d + k], acc);
    const float du = acc * scale;
    s_du[k] = du;
    fdu = fmaf(s_f[k], du, fdu);
  }
  fdu = block_sum(fdu, s_red);
  // through u = F / (||F|| + eps): dF = du / (n + eps) - F <F, du> / (n (n + eps)^2), the second term 0 at n = 0
  const float t = nf > 0.f ? fdu / (nf * fden * fden) : 0.f;
  for (int k = tid; k < d; k += PCR_THREADS) dFi[k] = s_du[k] / fden - s_f[k] * t;
}

__global__ void __launch_bounds__(PCR_THREADS) pcr_proxies_kernel(const float* __restrict__ F, int R, int d,
                                                                  const float* __restrict__ W, int C, float tau,
                                                                  float* __restrict__ dW, float* __restrict__ db,
                                                                  float* __restrict__ loss, PcrWs ws) {
  __shared__ float s_a[PCR_MAX_R];
  __shared__ float s_dv[PCR_MAX_D];
  __shared__ double s_red_d[PCR_THREADS];
  __shared__ float s_red[PCR_WARPS];
  __shared__ float s_vden;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int c = blockIdx.x;
  if (c == C) {                                            // the loss: l_i summed in double in row order
    double acc = 0.0;
    for (int i = tid; i < R; i += PCR_THREADS) acc += ws.row_loss[i];
    acc = block_sum_d(acc, s_red_d);
    if (tid == 0) *loss = (float)(acc / (double)R);
    return;
  }
  float* dWc = dW + (size_t)c * d;
  if (tid == 0) db[c] = 0.f;                               // linear.bias never enters the loss
  if (ws.counts[c] == 0) {                                 // no row carries c: every coef_ic is 0, dW_c is exactly 0
    for (int k = tid; k < d; k += PCR_THREADS) dWc[k] = 0.f;
    return;
  }
  for (int i = tid; i < R; i += PCR_THREADS) s_a[i] = ws.coef[(size_t)i * C + c] / ws.den[i];
  const float* Wc = W + (size_t)c * d;
  if (warp == 0) {
    const float vden = sqrtf(warp_sq_norm(Wc, d, lane)) + PCR_EPS;
    if (lane == 0) s_vden = vden;
  }
  __syncthreads();
  const float vden = s_vden;
  const float nw = vden - PCR_EPS;
  const float scale = 1.f / (tau * (float)R);
  float wdv = 0.f;
  for (int k = tid; k < d; k += PCR_THREADS) {
    float acc = 0.f;
    for (int i = 0; i < R; ++i) acc = fmaf(s_a[i], F[(size_t)i * d + k], acc);
    const float dv = acc * scale;
    s_dv[k] = dv;
    wdv = fmaf(Wc[k], dv, wdv);
  }
  wdv = block_sum(wdv, s_red);
  const float t = nw > 0.f ? wdv / (nw * vden * vden) : 0.f;
  for (int k = tid; k < d; k += PCR_THREADS) dWc[k] = s_dv[k] / vden - Wc[k] * t;
}

}  // namespace
}  // namespace b200ocl

extern "C" {

size_t b200ocl_pcr_loss_workspace_bytes(int R, int C) {
  if (R < 1 || C < 1) return 0;
  return b200ocl::pcr_ws_bytes(R, C);
}

int b200ocl_pcr_loss(const float* feats, const int64_t* labels, int R, int d, const float* proxies, int C,
                     float temperature, float* loss, float* dfeats, float* dproxies, float* dbias, int* err_flag,
                     void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(feats && labels && proxies && loss && dfeats && dproxies && dbias, "null pointer");
  B200OCL_CHECK_ARG(R >= 2 && d >= 1 && C >= 1, "need R >= 2, d >= 1, C >= 1");
  B200OCL_CHECK_ARG(isfinite(temperature) && temperature > 0.f, "temperature must be finite and positive");
  if (R > PCR_MAX_R || d > PCR_MAX_D || C > PCR_MAX_C) {
    set_error("b200ocl_pcr_loss: R=%d, d=%d, C=%d exceed the kernel's limits %d, %d, %d", R, d, C, PCR_MAX_R,
              PCR_MAX_D, PCR_MAX_C);
    return B200OCL_EUNSUPPORTED;
  }
  const int rc = check_workspace("b200ocl_pcr_loss", workspace, workspace_bytes, pcr_ws_bytes(R, C));
  if (rc) return rc;
  const PcrWs ws = pcr_ws(workspace, R, C);
  const long long* lab = reinterpret_cast<const long long*>(labels);
  B200OCL_PROF("pcr", 6.0 * (double)R * C * d, stream);
  pcr_rows_kernel<<<R, PCR_THREADS, 0, stream>>>(feats, lab, R, d, proxies, C, temperature, dfeats, ws, err_flag);
  B200OCL_LAUNCHED();
  B200OCL_PROF("pcr", 2.0 * (double)R * C * d, stream);
  pcr_proxies_kernel<<<C + 1, PCR_THREADS, 0, stream>>>(feats, R, d, proxies, C, temperature, dproxies, dbias, loss, ws);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

}  // extern "C"
