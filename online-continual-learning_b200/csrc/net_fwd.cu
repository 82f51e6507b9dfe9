// net_fwd.cu -- Reduced-ResNet18 / SupConResNet forward passes, weight packing, SGD, CE loss.
//
// Replaces model.features / model.forward of reference models/resnet.py:90-109,159-168 in
// eval mode (ASER deep features, utils/utils.py:45-90) and train mode (exp_replay.py:40,62,84;
// scr.py:55; mir_retrieve.py:24-25), torch.optim.SGD.step (setup_elements.py:73-75) and
// F.cross_entropy (agents/base.py:95,113; mir_retrieve.py:26-27).
#include <float.h>
#include <math.h>

#include "net_ws.cuh"
#include "umma.cuh"

namespace b200ocl {
namespace {

// ----------------------------------------------------------------------------- weight packing
struct PackTable {
  int n;
  struct {
    unsigned int w_off, pkf_off, pkd_off;
    int cin, cout, taps;
  } e[NET_MAX_CONV];
};

__global__ void __launch_bounds__(256) pack_kernel(PackTable t, const float* __restrict__ params,
                                                   float* __restrict__ packed) {
  const auto& L = t.e[blockIdx.y];
  const int total = L.cout * L.cin * L.taps;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    const int co = e / (L.cin * L.taps);
    const int rem = e - co * (L.cin * L.taps);
    const int ci = rem / L.taps, tap = rem - ci * L.taps;
    const float v = params[L.w_off + e];                              // OIHW
    packed[L.pkf_off + (tap * L.cin + ci) * L.cout + co] = v;         // [tap][cin][cout]
    packed[L.pkd_off + (tap * L.cout + co) * L.cin + ci] = v;         // [tap][cout][cin]
  }
}


// Tensor-core operand images: B[n][k] tiles, split into TF32 hi / lo, 128-byte swizzled.
//   forward        n = cout, k = tap*cin + ci            value W[co][ci][tap]
//   data gradient  n = cin,  k = tap*cout + co (flipped)  value W[co][ci][8 - tap]
struct TcPackTable {
  int n;
  struct {
    unsigned int w_off, img_off;
    int cin, cout, bn, nt, kb, dgrad;
  } e[2 * NET_MAX_CONV];
};

__global__ void __launch_bounds__(256) tc_pack_kernel(TcPackTable t, const float* __restrict__ params,
                                                      float* __restrict__ packed) {
  const auto& L = t.e[blockIdx.y];
  const int n_ch = L.dgrad ? L.cin : L.cout;      // output channels of this direction
  const int k_ch = L.dgrad ? L.cout : L.cin;      // channels contracted per tap
  const int ktot = 9 * k_ch;
  const int n_tiles = n_ch / L.bn;
  const int total = n_tiles * L.kb * L.nt * 8;    // (tile, kb, row, 16-byte chunk)
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    const int c = e & 7;
    int r = e >> 3;
    const int row = r % L.nt;
    r /= L.nt;
    const int kb = r % L.kb, tile = r / L.kb;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    const int k0 = kb * 32 + c * 4;
    if (row < L.bn && k0 < ktot) {
      const int tap = k0 / k_ch, kc = k0 - tap * k_ch;   // 4 consecutive k share the tap (k_ch % 4 == 0)
      const int nch = tile * L.bn + row;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int co = L.dgrad ? kc + j : nch;
        const int ci = L.dgrad ? nch : kc + j;
        const int wt = L.dgrad ? 8 - tap : tap;
        v[j] = params[L.w_off + ((size_t)co * L.cin + ci) * 9 + wt];
      }
    }
    float4 h, l;
    umma::split_tf32(v[0], h.x, l.x); umma::split_tf32(v[1], h.y, l.y);
    umma::split_tf32(v[2], h.z, l.z); umma::split_tf32(v[3], h.w, l.w);
    float* base = packed + L.img_off + ((size_t)(tile * L.kb + kb) * 2) * L.nt * 32;
    const int off = umma::sw128_offset_f32(row, c);
    *reinterpret_cast<float4*>(base + off) = h;
    *reinterpret_cast<float4*>(base + L.nt * 32 + off) = l;
  }
}

// Halo-patch tensor-core images (conv_tcp.cu): blocks [channel tile][slice][tap][hi | lo][NT x 32], row n =
// output channel of the direction, K slot = channel slice*32 + k of the contracted side, zero padded;
// the data-gradient image stores tap t of the correlation = W[.][.][8 - t].
struct TpPackTable {
  int n;
  struct {
    unsigned int w_off, img_off;
    int cin, cout, bn, nt, slices, dgrad;
  } e[2 * NET_MAX_CONV];
};

__global__ void __launch_bounds__(256) tp_pack_kernel(TpPackTable t, const float* __restrict__ params,
                                                      float* __restrict__ packed) {
  const auto& L = t.e[blockIdx.y];
  const int n_ch = L.dgrad ? L.cin : L.cout;
  const int k_ch = L.dgrad ? L.cout : L.cin;
  const int n_tiles = n_ch / L.bn;
  const int total = n_tiles * L.slices * 9 * L.nt * 8;   // (tile, slice, tap, row, 16-byte chunk)
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    const int c = e & 7;
    int r = e >> 3;
    const int row = r % L.nt;
    r /= L.nt;
    const int tap = r % 9;
    r /= 9;
    const int sl = r % L.slices, tile = r / L.slices;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    const int k0 = sl * 32 + c * 4;
    if (row < L.bn && k0 < k_ch) {
      const int nch = tile * L.bn + row;
      const int wt = L.dgrad ? 8 - tap : tap;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int co = L.dgrad ? k0 + j : nch;
        const int ci = L.dgrad ? nch : k0 + j;
        v[j] = params[L.w_off + ((size_t)co * L.cin + ci) * 9 + wt];
      }
    }
    float4 h, l;
    umma::split_tf32(v[0], h.x, l.x); umma::split_tf32(v[1], h.y, l.y);
    umma::split_tf32(v[2], h.z, l.z); umma::split_tf32(v[3], h.w, l.w);
    float* base = packed + L.img_off + ((size_t)((tile * L.slices + sl) * 9 + tap) * 2) * L.nt * 32;
    const int off = umma::sw128_offset_f32(row, c);
    *reinterpret_cast<float4*>(base + off) = h;
    *reinterpret_cast<float4*>(base + L.nt * 32 + off) = l;
  }
}

int launch_pack(const NetPlan& p, const float* params, float* packed, cudaStream_t stream) {
  PackTable t{};
  t.n = p.n_conv;
  for (int i = 0; i < p.n_conv; ++i) {
    t.e[i].w_off = (unsigned)p.conv[i].w_off;
    t.e[i].pkf_off = (unsigned)p.conv[i].pkf_off;
    t.e[i].pkd_off = (unsigned)p.conv[i].pkd_off;
    t.e[i].cin = p.conv[i].cin;
    t.e[i].cout = p.conv[i].cout;
    t.e[i].taps = p.conv[i].ks * p.conv[i].ks;
  }
  B200OCL_PROF("pack", 12.0 * p.n_packed / 2, stream);
  pack_kernel<<<dim3(16, p.n_conv), 256, 0, stream>>>(t, params, packed);
  B200OCL_LAUNCHED();
  TcPackTable tc{};
  for (int i = 0; i < p.n_conv; ++i) {
    const ConvL& c = p.conv[i];
    if (!c.tc_kb_f) continue;
    for (int d = 0; d < 2; ++d) {
      auto& e = tc.e[tc.n++];
      e.w_off = (unsigned)c.w_off;
      e.img_off = (unsigned)(d ? c.tc_d_off : c.tc_f_off);
      e.cin = c.cin; e.cout = c.cout;
      e.bn = d ? c.tc_bn_d : c.tc_bn_f;
      e.nt = tc_nt(e.bn);
      e.kb = d ? c.tc_kb_d : c.tc_kb_f;
      e.dgrad = d;
    }
  }
  if (tc.n) {
    B200OCL_PROF("pack", 16.0 * p.n_packed / 2, stream);
    tc_pack_kernel<<<dim3(32, tc.n), 256, 0, stream>>>(tc, params, packed);
    B200OCL_LAUNCHED();
  }
  TpPackTable tp{};
  for (int i = 0; i < p.n_conv; ++i) {
    const ConvL& c = p.conv[i];
    for (int d = 0; d < 2; ++d) {
      if (!(d ? c.tp_sl_d : c.tp_sl_f)) continue;
      auto& e = tp.e[tp.n++];
      e.w_off = (unsigned)c.w_off;
      e.img_off = (unsigned)(d ? c.tp_d_off : c.tp_f_off);
      e.cin = c.cin; e.cout = c.cout;
      e.bn = d ? c.tp_bn_d : c.tp_bn_f;
      e.nt = tc_nt(e.bn);
      e.slices = d ? c.tp_sl_d : c.tp_sl_f;
      e.dgrad = d;
    }
  }
  if (tp.n) {
    B200OCL_PROF("pack", 16.0 * p.n_packed / 2, stream);
    tp_pack_kernel<<<dim3(32, tp.n), 256, 0, stream>>>(tp, params, packed);
    B200OCL_LAUNCHED();
  }
  return B200OCL_OK;
}

// ----------------------------------------------------------------------------- SGD over the arena
// CLIP: the gradient is first scaled by the clipping coefficient *coef (grad_norm_kernel) and the scaled value is
// written back to the gradient arena through g_out (== g).  Each element is read and then written by one thread only,
// so the read-only load of g cannot see a stale value.
template <bool CLIP>
__global__ void __launch_bounds__(256) net_sgd_kernel(const float* __restrict__ p, const float* __restrict__ g,
                                                      float* __restrict__ out, size_t n, float lr, float wd,
                                                      size_t skip_lo, size_t skip_hi, const float* coef, float* g_out) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  float c = 1.f;
  if (CLIP) c = *coef;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float w = p[i];
    if (i >= skip_lo && i < skip_hi) {  // tensors that never receive a gradient: torch skips them
      out[i] = w;
      continue;
    }
    float gi = g[i];
    if (CLIP) {
      gi = gi * c;                      // torch._foreach_mul_(grads, clip_coef_clamped)
      g_out[i] = gi;
    }
    if (wd != 0.f) gi = fmaf(wd, w, gi);
    out[i] = w - lr * gi;
  }
}

// L2 norm of the gradient arena outside [skip_lo, skip_hi) and torch's clipping coefficient
// (torch/nn/utils/clip_grad.py, _clip_grads_with_norm_): coef = min(max_norm / (norm + 1e-6), 1) in fp32, with torch's roundings.
// Per-CTA fp64 partial sums of squares in a fixed order; the last CTA to arrive adds them in CTA order.
constexpr int NORM_MAX_GRID = 1024;

// Workspace of the arena reductions (grad_norm_kernel, the EWC++ kernels): one 8-byte partial per CTA (up to
// NORM_MAX_GRID), then, at the next 256-byte boundary, the arrival counter followed by the reduction's fp32 results.
constexpr size_t REDUCE_TAIL_OFF = (NORM_MAX_GRID * sizeof(double) + 255) / 256 * 256;
constexpr size_t REDUCE_WS_BYTES = REDUCE_TAIL_OFF + 256;
inline unsigned int* reduce_counter(void* ws) {
  return reinterpret_cast<unsigned int*>(static_cast<unsigned char*>(ws) + REDUCE_TAIL_OFF);
}
inline float* reduce_scalars(void* ws) { return reinterpret_cast<float*>(reduce_counter(ws) + 1); }

// The tensors that never receive a gradient (the SupCon network's unused classifier): every pass that steps the
// arenas leaves [lo, hi) out.
inline void sgd_skip_range(const NetPlan& p, size_t& lo, size_t& hi) {
  lo = hi = 0;
  if (p.head != 0) {
    lo = p.lin[0].w_off;
    hi = p.lin[0].b_off + p.lin[0].out;
  }
}

// Grid of a grid-stride pass of 256-thread CTAs over the parameter arena: at most per_sm CTAs per SM and `cap`.
inline unsigned arena_grid(const NetPlan& p, int per_sm, size_t cap) {
  size_t blocks = (p.n_params + 255) / 256;
  const size_t sm_cap = (size_t)per_sm * sm_count();
  if (blocks > sm_cap) blocks = sm_cap;
  return (unsigned)(blocks < cap ? blocks : cap);
}

__global__ void __launch_bounds__(256) grad_norm_kernel(const float* __restrict__ g, size_t n, size_t skip_lo,
                                                        size_t skip_hi, float max_norm, double* __restrict__ part,
                                                        unsigned int* counter, float* coef, float* norm_out) {
  __shared__ double s_red[8];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double acc = 0.0;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (i >= skip_lo && i < skip_hi) continue;
    const double v = (double)g[i];
    acc = fma(v, v, acc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(FULL_MASK, acc, o);
  if (lane == 0) s_red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += s_red[w];
    part[blockIdx.x] = t;
    __threadfence();
    is_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (is_last && threadIdx.x == 0) {
    __threadfence();
    double t = 0.0;
    for (unsigned int b = 0; b < gridDim.x; ++b) t += __ldcg(part + b);
    const float norm = (float)sqrt(t);
    // torch forms max_norm / (norm + 1e-6) as Tensor.__rdiv__: (norm + 1e-6).reciprocal() * max_norm, two roundings
    const float q = __fmul_rn(__frcp_rn(norm + 1e-6f), max_norm);
    *coef = q > 1.f ? 1.f : q;          // torch.clamp(max=1.0): a NaN norm stays NaN

    if (norm_out) *norm_out = norm;
  }
}

// ----------------------------------------------------------------------------- EWC++ step and consolidation
// One pass per element in the order of agents/ewc_pp.py: the EMA of update_running_fisher (EMA), the penalty's gradient
// added to the network's (PEN), accum_fisher's tmp += g*g, then the SGD update of net_sgd_kernel.  Every torch op is
// its own rounding, so the products and sums are spelled with __f*_rn: nvcc would contract them to fma.  The SGD
// update is written as net_sgd_kernel writes it, so that it compiles to the same instructions.  With PEN and pen_out,
// sum F*d^2 over the pre-step weights goes to pen_out: per-CTA fp64 partials, added in CTA order by the last CTA.
template <bool EMA, bool PEN>
__global__ void __launch_bounds__(256) net_sgd_ewc_kernel(float* __restrict__ p, float* __restrict__ g,
                                                          float* __restrict__ running, float* __restrict__ tmp,
                                                          const float* __restrict__ fisher,
                                                          const float* __restrict__ prev, size_t n, size_t skip_lo,
                                                          size_t skip_hi, float lr, float wd, float up, float ema_keep,
                                                          float ema_add, double* __restrict__ part,
                                                          unsigned int* counter, float* pen_out) {
  double acc = 0.0;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (i >= skip_lo && i < skip_hi) continue;   // tensors that never receive a gradient: untouched in every arena
    const float w = p[i];
    float gi = g[i];
    float t = tmp[i];
    if (EMA) {
      // (1 - alpha) * running + (1/fua * alpha) * tmp, then tmp = 0 (ewc_pp.py:104-108)
      running[i] = __fadd_rn(__fmul_rn(ema_keep, running[i]), __fmul_rn(ema_add, t));
      t = 0.f;
    }
    if (PEN) {
      // autograd of lambda * (F * (p - prev)**2).sum(): (up * F) * (2 * d), added once to the network's gradient
      const float f = fisher[i];
      const float d = __fsub_rn(w, prev[i]);
      gi = __fadd_rn(gi, __fmul_rn(__fmul_rn(up, f), __fmul_rn(2.f, d)));
      g[i] = gi;
      const double dd = (double)d;
      acc = fma((double)f * dd, dd, acc);
    }
    tmp[i] = __fadd_rn(t, __fmul_rn(gi, gi));   // accum_fisher: tmp += grad ** 2 (pow 2 is grad * grad)
    if (wd != 0.f) gi = fmaf(wd, w, gi);
    p[i] = w - lr * gi;
  }
  if (!PEN || !pen_out) return;
  __shared__ double s_red[8];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(FULL_MASK, acc, o);
  if (lane == 0) s_red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += s_red[k];
    part[blockIdx.x] = s;
    __threadfence();
    is_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (is_last && threadIdx.x == 0) {
    __threadfence();
    double s = 0.0;
    for (unsigned int b = 0; b < gridDim.x; ++b) s += __ldcg(part + b);
    *pen_out = (float)s;
  }
}

// End of an EWC++ call, first half: prev = params, and the global min / max of running (per-CTA partials, combined by
// the last CTA, which stores mn and the denominator (mx - mn) + 1e-32 with torch's fp32 roundings).
__global__ void __launch_bounds__(256) ewc_minmax_kernel(const float* __restrict__ p, const float* __restrict__ running,
                                                         float* __restrict__ prev, size_t n, size_t skip_lo,
                                                         size_t skip_hi, float2* __restrict__ part,
                                                         unsigned int* counter, float* range) {
  __shared__ float s_mn[8], s_mx[8];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float mn = INFINITY, mx = -INFINITY;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (i >= skip_lo && i < skip_hi) continue;
    prev[i] = p[i];
    const float v = running[i];
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(FULL_MASK, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(FULL_MASK, mx, o));
  }
  if (lane == 0) {
    s_mn[warp] = mn;
    s_mx[warp] = mx;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 1; k < 8; ++k) {
      s_mn[0] = fminf(s_mn[0], s_mn[k]);
      s_mx[0] = fmaxf(s_mx[0], s_mx[k]);
    }
    part[blockIdx.x] = make_float2(s_mn[0], s_mx[0]);
    __threadfence();
    is_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (is_last && threadIdx.x == 0) {
    __threadfence();
    float a = INFINITY, b = -INFINITY;
    for (unsigned int k = 0; k < gridDim.x; ++k) {
      const float2 v = __ldcg(part + k);
      a = fminf(a, v.x);
      b = fmaxf(b, v.y);
    }
    range[0] = a;
    range[1] = __fadd_rn(__fsub_rn(b, a), 1e-32f);
  }
}

// Second half: normalized = (running - mn) / ((mx - mn) + 1e-32), an IEEE division.
__global__ void __launch_bounds__(256) ewc_normalize_kernel(const float* __restrict__ running,
                                                            float* __restrict__ normalized, size_t n, size_t skip_lo,
                                                            size_t skip_hi, const float* __restrict__ range) {
  const float mn = range[0], den = range[1];
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (i >= skip_lo && i < skip_hi) continue;
    normalized[i] = __fdiv_rn(__fsub_rn(running[i], mn), den);
  }
}

// ----------------------------------------------------------------------------- train-mode BN apply
struct BnApplyArgs {
  const float* z;
  float* a;
  size_t n_vec;  // float4 count
  int C;
  const float *gamma, *beta, *mean, *invstd;
  const float* res;                            // nullable
  const float *rgamma, *rbeta, *rmean, *rinvstd;  // when res is a raw conv output that needs its own BN
  int relu;
};

__global__ void __launch_bounds__(256) bn_apply_kernel(BnApplyArgs a) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const float4* z4 = reinterpret_cast<const float4*>(a.z);
  const float4* r4 = reinterpret_cast<const float4*>(a.res);
  float4* o4 = reinterpret_cast<float4*>(a.a);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n_vec; i += stride) {
    const int c = (int)((i * 4) % (size_t)a.C);
    const float4 g = *reinterpret_cast<const float4*>(a.gamma + c);
    const float4 b = *reinterpret_cast<const float4*>(a.beta + c);
    const float4 mu = *reinterpret_cast<const float4*>(a.mean + c);
    const float4 is = *reinterpret_cast<const float4*>(a.invstd + c);
    const float4 x = z4[i];
    float4 v;
    v.x = (x.x - mu.x) * is.x * g.x + b.x;
    v.y = (x.y - mu.y) * is.y * g.y + b.y;
    v.z = (x.z - mu.z) * is.z * g.z + b.z;
    v.w = (x.w - mu.w) * is.w * g.w + b.w;
    if (a.res) {
      float4 r = r4[i];
      if (a.rgamma) {
        const float4 rg = *reinterpret_cast<const float4*>(a.rgamma + c);
        const float4 rb = *reinterpret_cast<const float4*>(a.rbeta + c);
        const float4 rm = *reinterpret_cast<const float4*>(a.rmean + c);
        const float4 ri = *reinterpret_cast<const float4*>(a.rinvstd + c);
        r.x = (r.x - rm.x) * ri.x * rg.x + rb.x;
        r.y = (r.y - rm.y) * ri.y * rg.y + rb.y;
        r.z = (r.z - rm.z) * ri.z * rg.z + rb.z;
        r.w = (r.w - rm.w) * ri.w * rg.w + rb.w;
      }
      v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    }
    if (a.relu) {
      v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    }
    o4[i] = v;
  }
}

int launch_bn_apply(const BnApplyArgs& a, cudaStream_t stream) {
  size_t blocks = (a.n_vec + 255) / 256;
  const size_t cap = (size_t)16 * sm_count();
  if (blocks > cap) blocks = cap;
  B200OCL_PROF("bn_apply", (a.res ? 48.0 : 32.0) * a.n_vec, stream);
  bn_apply_kernel<<<(unsigned)blocks, 256, 0, stream>>>(a);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

// ----------------------------------------------------------------------------- avg_pool2d(.,4) + flatten
// in NHWC [N,H,W,C] -> feat[n][c*PH*PW + ph*PW + pw]  (NCHW flatten order, resnet.py:97-98)
__global__ void __launch_bounds__(256) pool_kernel(const float* __restrict__ in, float* __restrict__ feat, int N,
                                                   int H, int W, int C, int PH, int PW) {
  const int total = N * PH * PW * C;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = i % C;
    int t = i / C;
    const int pw = t % PW;
    t /= PW;
    const int ph = t % PH, n = t / PH;
    float s = 0.f;
#pragma unroll
    for (int dy = 0; dy < 4; ++dy)
#pragma unroll
      for (int dx = 0; dx < 4; ++dx) s += in[((size_t)(n * H + ph * 4 + dy) * W + pw * 4 + dx) * C + c];
    feat[(size_t)n * (C * PH * PW) + (c * PH + ph) * PW + pw] = s * 0.0625f;
  }
}

// ----------------------------------------------------------------------------- linear forward
// y[n][o] = b[o] + sum_i x[n][i] * W[o][i]  (+ReLU).  One warp per output feature keeps its weight
// row in registers and walks the batch; in <= 1024.
__global__ void __launch_bounds__(256) linear_fwd_kernel(const float* __restrict__ x, const float* __restrict__ W,
                                                         const float* __restrict__ b, float* __restrict__ y, int N,
                                                         int in, int out, int relu) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int o = blockIdx.x * 8 + warp;
  if (o >= out) return;
  float w[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int i = lane + 32 * j;
    w[j] = (i < in) ? W[(size_t)o * in + i] : 0.f;
  }
  const float bias = b[o];
  for (int n = blockIdx.y; n < N; n += gridDim.y) {
    const float* xr = x + (size_t)n * in;
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int i = lane + 32 * j;
      if (i < in) s = fmaf(xr[i], w[j], s);
    }
    s = warp_sum(s);
    if (lane == 0) {
      s += bias;
      y[(size_t)n * out + o] = relu ? fmaxf(s, 0.f) : s;
    }
  }
}

int launch_linear_fwd(const float* x, const float* W, const float* b, float* y, int N, int in, int out, int relu,
                      cudaStream_t stream) {
  int gy = N < 32 ? N : 32;
  B200OCL_PROF("head", 4.0 * ((double)N * in + (double)in * out + (double)N * out), stream);
  linear_fwd_kernel<<<dim3((out + 7) / 8, gy), 256, 0, stream>>>(x, W, b, y, N, in, out, relu);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

// ----------------------------------------------------------------------------- F.normalize(dim=1)
__global__ void __launch_bounds__(256) l2norm_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int N,
                                                         int d) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = blockIdx.x * 8 + warp;
  if (n >= N) return;
  const float* xr = x + (size_t)n * d;
  float s = 0.f;
  for (int i = lane; i < d; i += 32) s = fmaf(xr[i], xr[i], s);
  s = warp_sum(s);
  const float inv = 1.f / fmaxf(sqrtf(s), 1e-12f);
  for (int i = lane; i < d; i += 32) y[(size_t)n * d + i] = xr[i] * inv;
}

// ----------------------------------------------------------------------------- cross-entropy
// Warp-wide maximum (ties to the lowest index) and log-sum-exp of the K values get(0..K-1) of one row.  Lanes take
// strided elements and reduce through shuffles, so the summation order is the same on every call.
struct RowLse {
  float mx;
  int arg;
  float lse;
};

template <class Get>
__device__ __forceinline__ RowLse row_lse(Get get, int K, int lane) {
  float mx = -FLT_MAX;
  int arg = 0;
  for (int c = lane; c < K; c += 32) {
    const float v = get(c);
    if (v > mx) { mx = v; arg = c; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(FULL_MASK, mx, o);
    const int oa = __shfl_xor_sync(FULL_MASK, arg, o);
    if (om > mx || (om == mx && oa < arg)) { mx = om; arg = oa; }
  }
  float z = 0.f;
  for (int c = lane; c < K; c += 32) z += expf(get(c) - mx);
  z = warp_sum(z);
  return RowLse{mx, arg, mx + logf(z)};
}

__global__ void __launch_bounds__(256) ce_kernel(const float* __restrict__ logits, const long long* __restrict__ labels,
                                                 int N, int C, float* __restrict__ loss, float* __restrict__ per_sample,
                                                 float* __restrict__ dlogits, long long* __restrict__ n_correct) {
  __shared__ float s_loss[8];
  __shared__ int s_corr[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float lsum = 0.f;
  int corr = 0;
  for (int n = warp; n < N; n += 8) {   // fixed assignment of rows to warps: deterministic sum
    const float* lr = logits + (size_t)n * C;
    const RowLse r = row_lse([=](int c) { return __ldg(lr + c); }, C, lane);
    const float lse = r.lse;
    const int arg = r.arg;
    const long long y = labels[n];
    const float l = lse - lr[y];
    if (per_sample && lane == 0) per_sample[n] = l;
    if (dlogits) {
      const float invN = 1.f / (float)N;
      for (int c = lane; c < C; c += 32)
        dlogits[(size_t)n * C + c] = (expf(lr[c] - lse) - (c == y ? 1.f : 0.f)) * invN;
    }
    lsum += l;
    corr += (arg == (int)y) ? 1 : 0;
  }
  if (lane == 0) { s_loss[warp] = lsum; s_corr[warp] = corr; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    int k = 0;
    for (int w = 0; w < 8; ++w) { t += s_loss[w]; k += s_corr[w]; }
    if (loss) *loss = t / (float)N;
    if (n_correct) *n_correct = k;
  }
}

// ----------------------------------------------------------------------------- classification-loss variants
// The criteria of agents/base.py:93-113 besides plain CE and SupCon, with the distillation term of
// utils/kd_manager.py:6-11 mixed in (exp_replay.py:41-47, agem.py:40-46, lwf.py:38-40).  Like ce_kernel: one CTA,
// a fixed assignment of rows to warps and fixed-order sums, so repeated launches give identical bits.
struct ClsLossArgs {
  const float* logits;
  const long long* labels;
  int N, C, mode;
  const long long* cols;     // separated softmax: old_labels ++ new_labels (duplicates allowed)
  int n_cols, n_old;         // ... and the segment boundary
  const long long* pos;      // label -> position in cols (lbl_inv_map), -1 where unmapped
  int n_pos;
  const float* teacher;      // nullable: teacher logits [N,C]
  float w_ce, w_kd;
  float* loss;
  float* dlogits;
  long long* n_correct;
  int* err;
};

constexpr float KD_T = 2.f;  // loss_fn_kd's temperature (kd_manager.py:6)

__global__ void __launch_bounds__(256) cls_loss_kernel(ClsLossArgs a) {
  extern __shared__ int s_on[];          // labels trick: class c occurs in the batch
  __shared__ float s_ce[8], s_kd[8];
  __shared__ int s_corr[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int C = a.C;
  if (a.mode == B200OCL_CLS_LABELS) {
    // the batch's class set labels.unique(): a presence map over the C columns.  CE over the present columns with
    // each label remapped to its rank among them is CE over those columns at the label's own column.
    for (int c = threadIdx.x; c < C; c += blockDim.x) s_on[c] = 0;
    __syncthreads();
    for (int n = threadIdx.x; n < a.N; n += blockDim.x) {
      const long long y = a.labels[n];
      if (y >= 0 && y < C) s_on[y] = 1;
    }
    __syncthreads();
  }
  const float invN = 1.f / (float)a.N;
  float ce_sum = 0.f, kd_sum = 0.f;
  int corr = 0;
  for (int n = warp; n < a.N; n += 8) {
    const float* lr = a.logits + (size_t)n * C;
    const float* tr = a.teacher ? a.teacher + (size_t)n * C : nullptr;
    const long long y = a.labels[n];
    bool bad = y < 0 || y >= C;
    int p = 0, s0 = 0, s1 = 0;           // separated softmax: the target's position and its segment [s0, s1)
    if (a.mode == B200OCL_CLS_SEPARATED) {
      const long long q = (!bad && y < a.n_pos) ? a.pos[y] : -1;
      bad = bad || q < 0 || q >= a.n_cols;
      p = bad ? 0 : (int)q;
      s0 = p < a.n_old ? 0 : a.n_old;
      s1 = p < a.n_old ? a.n_old : a.n_cols;
    }
    if (bad) {                           // the host raises KeyError; the row adds nothing
      if (lane == 0 && a.err) *a.err = 1;
      if (a.dlogits)
        for (int c = lane; c < C; c += 32) a.dlogits[(size_t)n * C + c] = 0.f;
      continue;
    }
    const RowLse all = row_lse([=](int c) { return __ldg(lr + c); }, C, lane);     // arg-max over every column (meters)
    const int arg = all.arg;
    float lse = all.lse, tgt = lr[y];
    if (a.mode == B200OCL_CLS_LABELS) {
      lse = row_lse([=](int c) { return s_on[c] ? __ldg(lr + c) : -INFINITY; }, C, lane).lse;
    } else if (a.mode == B200OCL_CLS_SEPARATED) {
      const long long* cs = a.cols + s0;
      lse = row_lse([=](int k) { return __ldg(lr + __ldg(cs + k)); }, s1 - s0, lane).lse;
      tgt = lr[a.cols[p]];
    }
    ce_sum += lse - tgt;
    corr += (arg == (int)y) ? 1 : 0;
    float lse_s = 0.f, lse_t = 0.f;
    if (tr) {                            // T^2 * sum_c -softmax(t/T)_c * log_softmax(s/T)_c
      lse_s = row_lse([=](int c) { return __ldg(lr + c) / KD_T; }, C, lane).lse;
      lse_t = row_lse([=](int c) { return __ldg(tr + c) / KD_T; }, C, lane).lse;
      float k = 0.f;
      for (int c = lane; c < C; c += 32) k -= expf(tr[c] / KD_T - lse_t) * (lr[c] / KD_T - lse_s);
      kd_sum += warp_sum(k) * (KD_T * KD_T);
    }
    if (a.dlogits) {
      const float sce = a.w_ce * invN, skd = a.w_kd * KD_T * invN;
      for (int c = lane; c < C; c += 32) {
        float g = 0.f;
        if (a.mode == B200OCL_CLS_SEPARATED) {
          // every position of the target's segment that holds column c, in position order
          const float e = expf(lr[c] - lse);
          for (int k = s0; k < s1; ++k)
            if (a.cols[k] == c) g += e - (k == p ? 1.f : 0.f);
        } else if (a.mode == B200OCL_CLS_CE || s_on[c]) {
          g = expf(lr[c] - lse) - (c == (int)y ? 1.f : 0.f);
        }
        float d = g * sce;
        if (tr) d = fmaf(skd, expf(lr[c] / KD_T - lse_s) - expf(tr[c] / KD_T - lse_t), d);
        a.dlogits[(size_t)n * C + c] = d;
      }
    }
  }
  if (lane == 0) { s_ce[warp] = ce_sum; s_kd[warp] = kd_sum; s_corr[warp] = corr; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float ce = 0.f, kd = 0.f;
    int k = 0;
    for (int w = 0; w < 8; ++w) { ce += s_ce[w]; kd += s_kd[w]; k += s_corr[w]; }
    float l = a.w_ce * (ce / (float)a.N);
    if (a.teacher) l += a.w_kd * (kd / (float)a.N);
    if (a.loss) *a.loss = l;
    if (a.n_correct) *a.n_correct = k;
  }
}

// ----------------------------------------------------------------------------- iCaRL's criterion
// F.binary_cross_entropy_with_logits(logits[:, :K], target, reduction='none').sum(1).mean() of agents/icarl.py:42-62
// and its gradient.  The target is one-hot at the label's position for the stream rows and zero for the memory rows,
// with the teacher's sigmoids in the first n_old columns of every row.  Like ce_kernel: one CTA, a fixed assignment of
// rows to warps and fixed-order sums, so repeated launches give identical bits.
struct IcarlLossArgs {
  const float* logits;
  const float* teacher;      // previous model's logits [N,C]; nullable when n_old == 0
  const long long* labels;   // [n_stream]
  const long long* pos;      // label -> position (lbl_inv_map), -1 where unmapped
  int n_pos, N, n_stream, C, K, n_old;
  float* loss;
  float* dlogits;
  int* err;
};

__device__ __forceinline__ float sigmoid_f(float z) { return 1.f / (1.f + expf(-z)); }

__global__ void __launch_bounds__(256) icarl_loss_kernel(IcarlLossArgs a) {
  __shared__ float s_loss[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int C = a.C, K = a.K, n_old = a.n_old;
  const float invN = 1.f / (float)a.N;
  float lsum = 0.f;
  for (int n = warp; n < a.N; n += 8) {
    const float* lr = a.logits + (size_t)n * C;
    const float* tr = a.teacher ? a.teacher + (size_t)n * C : nullptr;
    float* dr = a.dlogits ? a.dlogits + (size_t)n * C : nullptr;
    int p = -1;                          // the one-hot column; memory rows have none
    if (n < a.n_stream) {
      const long long y = a.labels[n];
      const long long q = (y >= 0 && y < a.n_pos) ? a.pos[y] : -1;
      if (q < n_old || q >= K) {         // not a label of this task (icarl.py:44 raises); the row adds nothing
        if (lane == 0 && a.err) *a.err = 1;
        if (dr)
          for (int c = lane; c < C; c += 32) dr[c] = 0.f;
        continue;
      }
      p = (int)q;
    }
    // max(z,0) - z*t + log1p(exp(-|z|)): finite for any finite z
    float s = 0.f;
    for (int c = lane; c < K; c += 32) {
      const float z = __ldg(lr + c);
      const float t = c < n_old ? sigmoid_f(__ldg(tr + c)) : (c == p ? 1.f : 0.f);
      s += fmaxf(z, 0.f) - z * t + log1pf(expf(-fabsf(z)));
      if (dr) dr[c] = (sigmoid_f(z) - t) * invN;
    }
    if (dr)
      for (int c = K + lane; c < C; c += 32) dr[c] = 0.f;
    lsum += warp_sum(s);
  }
  if (lane == 0) s_loss[warp] = lsum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += s_loss[w];
    if (a.loss) *a.loss = t / (float)a.N;
  }
}

// ----------------------------------------------------------------------------- orchestration
int conv_eval(const NetPlan& p, const b200ocl_net_state& st, int ci, int N, const float* in, float* out,
              const float* residual, int relu, cudaStream_t stream) {
  ConvArgs a = conv_layer_args(p.conv[ci], N, in, st.packed, out, false);
  const BnL& b = p.bn[ci];
  a.mode = CONV_EVAL;
  a.eps = NET_BN_EPS;
  a.momentum = NET_BN_MOMENTUM;
  a.gamma = st.params + b.g_off;
  a.beta = st.params + b.b_off;
  a.rmean = st.bn_stats + b.stat_off;
  a.rvar = st.bn_stats + b.stat_off + b.c;
  a.residual = residual;
  a.relu = relu;
  return ci == 0 ? launch_stem(a, stream) : launch_conv(a, stream);
}


// Eval-statistics forward (GSS-greedy differentiates the network in eval mode, gss_greedy_update.py:16): the
// "saved" statistics that bn_apply and the backward use are the RUNNING ones; the batch statistics the train-mode
// convolution computes go to a throw-away buffer and the running statistics are left alone.
__global__ void bn_save_running_kernel(const float* __restrict__ rmean, const float* __restrict__ rvar, float eps, int C,
                                       float* __restrict__ save_mean, float* __restrict__ save_invstd) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) {
    save_mean[c] = rmean[c];
    save_invstd[c] = 1.0f / sqrtf(rvar[c] + eps);
  }
}

// stats: where the BatchNorm statistics of a train-mode convolution go.
//   STATS_RUNNING  the reference's train mode: batch statistics normalise, the running statistics move (momentum 0.1)
//   STATS_EVAL     GSS-greedy's differentiable eval-mode pass: the running statistics normalise, nothing moves
//   STATS_DEFER    batch statistics normalise; the running statistics are NOT touched: the (mean, unbiased variance) pair
//                  of every BN is left in the workspace (momentum 1 into a zeroed buffer: 0 * 0 + 1 * s = s exactly) and
//                  applied later, in the caller's order, by b200ocl_net_apply_running_stats -- so that several train-mode
//                  passes of one step (exp_replay.py:40,62,84; scr.py:55) can run concurrently on different streams
enum { STATS_RUNNING = 0, STATS_EVAL = 1, STATS_DEFER = 2 };

int conv_train(const NetPlan& p, const b200ocl_net_state& st, const TrainWs& w, int ci, int N, const float* in,
               cudaStream_t stream, int stats = STATS_RUNNING) {
  const bool eval_stats = stats == STATS_EVAL;
  const ConvL& c = p.conv[ci];
  ConvArgs a = conv_layer_args(c, N, in, st.packed, w.z + (size_t)N * c.act_off, false);
  const BnL& b = p.bn[ci];
  a.mode = CONV_TRAIN;
  a.eps = NET_BN_EPS;
  a.momentum = NET_BN_MOMENTUM;
  a.stat_part = w.stat_part;
  a.counter = w.counters + 8 * ci;   // up to 8 channel tiles per conv (160 = 8 x 20)
  a.save_mean = w.save + b.save_off;
  a.save_invstd = w.save + b.save_off + b.c;
  a.run_mean = eval_stats ? w.run_scratch : st.bn_stats + b.stat_off;
  a.run_var = eval_stats ? w.run_scratch + 1024 : st.bn_stats + b.stat_off + b.c;
  if (stats == STATS_DEFER) {
    a.run_mean = w.run_defer + b.stat_off;
    a.run_var = w.run_defer + b.stat_off + b.c;
    a.momentum = 1.0f;
  }
  const int rc = ci == 0 ? launch_stem(a, stream) : launch_conv(a, stream);
  if (rc == 0 && eval_stats) {
    bn_save_running_kernel<<<(b.c + 127) / 128, 128, 0, stream>>>(st.bn_stats + b.stat_off, st.bn_stats + b.stat_off + b.c, a.eps,
                                                                   b.c, a.save_mean, a.save_invstd);
    B200OCL_LAUNCHED();
  }
  return rc;
}

int bn_apply_train(const NetPlan& p, const b200ocl_net_state& st, const TrainWs& w, int ci, int N, int res_conv,
                   const float* res_plain, cudaStream_t stream) {
  const ConvL& c = p.conv[ci];
  const BnL& b = p.bn[ci];
  BnApplyArgs a{};
  a.z = w.z + (size_t)N * c.act_off;
  a.a = w.a + (size_t)N * c.act_off;
  a.n_vec = (size_t)N * c.hout * c.wout * c.cout / 4;
  a.C = c.cout;
  a.gamma = st.params + b.g_off;
  a.beta = st.params + b.b_off;
  a.mean = w.save + b.save_off;
  a.invstd = w.save + b.save_off + b.c;
  a.relu = 1;
  if (res_conv >= 0) {
    const BnL& rb = p.bn[res_conv];
    a.res = w.z + (size_t)N * p.conv[res_conv].act_off;
    a.rgamma = st.params + rb.g_off;
    a.rbeta = st.params + rb.b_off;
    a.rmean = w.save + rb.save_off;
    a.rinvstd = w.save + rb.save_off + rb.c;
  } else {
    a.res = res_plain;
  }
  return launch_bn_apply(a, stream);
}

int head_forward(const NetPlan& p, const b200ocl_net_state& st, const float* feat, int N, float* hid, float* proj,
                 float* out, cudaStream_t stream) {
  int rc;
  if (p.head == 0) {
    const LinL& l = p.lin[0];
    return launch_linear_fwd(feat, st.params + l.w_off, st.params + l.b_off, out, N, l.in, l.out, 0, stream);
  }
  const float* pre = feat;
  if (p.head == 1) {
    const LinL& l = p.lin[1];
    if ((rc = launch_linear_fwd(feat, st.params + l.w_off, st.params + l.b_off, proj, N, l.in, l.out, 0, stream))) return rc;
    pre = proj;
  } else if (p.head == 2) {
    const LinL& l1 = p.lin[1];
    const LinL& l2 = p.lin[2];
    if ((rc = launch_linear_fwd(feat, st.params + l1.w_off, st.params + l1.b_off, hid, N, l1.in, l1.out, 1, stream))) return rc;
    if ((rc = launch_linear_fwd(hid, st.params + l2.w_off, st.params + l2.b_off, proj, N, l2.in, l2.out, 0, stream))) return rc;
    pre = proj;
  }
  B200OCL_PROF("head", 8.0 * N * p.out_dim, stream);
  l2norm_fwd_kernel<<<(N + 7) / 8, 256, 0, stream>>>(pre, out, N, p.out_dim);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

// running = (1 - momentum) * running + momentum * s for every BN statistic (bn_running_update, as in the convolution
// epilogues), plus num_batches_tracked += 1: one deferred train-mode pass applied to the running statistics
__global__ void bn_running_apply_kernel(float* __restrict__ run, const float* __restrict__ s, int n, float momentum,
                                        long long* __restrict__ tracked, int n_bn) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) run[i] = bn_running_update(run[i], s[i], momentum);
  if (tracked && i < n_bn) tracked[i] += 1;
}

__global__ void bump_tracked_kernel(long long* t, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) t[i] += 1;
}

int check_state(const b200ocl_net_desc* desc, const b200ocl_net_state* st, NetPlan& p) {
  if (!desc || !st || !st->params || !st->packed || !st->bn_stats) {
    set_error("net: null descriptor/state pointer");
    return B200OCL_EINVAL;
  }
  const int rc = build_plan(*desc, p);
  if (rc) set_error("net: unsupported network description (nf must be 20, head in 0..3, dims <= 1024)");
  return rc;
}

}  // namespace
}  // namespace b200ocl

extern "C" {

int b200ocl_net_query(const b200ocl_net_desc* desc, b200ocl_net_info* info) {
  using namespace b200ocl;
  B200OCL_CHECK_ARG(desc && info, "null pointer");
  NetPlan p;
  const int rc = build_plan(*desc, p);
  if (rc) {
    set_error("b200ocl_net_query: unsupported network description");
    return rc;
  }
  info->n_params = p.n_params;
  info->n_packed = p.n_packed;
  info->n_bn_stats = p.n_stats;
  info->n_bn = p.n_conv;
  info->n_tensors = 3 * p.n_conv + 2 * p.n_lin;
  info->dim_in = p.dim_in;
  info->out_dim = p.out_dim;
  return B200OCL_OK;
}

int b200ocl_net_tensor(const b200ocl_net_desc* desc, int i, size_t* offset, size_t* numel, int* has_grad) {
  using namespace b200ocl;
  B200OCL_CHECK_ARG(desc && offset && numel && has_grad, "null pointer");
  NetPlan p;
  const int rc = build_plan(*desc, p);
  if (rc) return rc;
  const int n_conv_t = 3 * p.n_conv;
  *has_grad = 1;
  if (i < 0 || i >= n_conv_t + 2 * p.n_lin) {
    set_error("b200ocl_net_tensor: index out of range");
    return B200OCL_EINVAL;
  }
  if (i < n_conv_t) {
    const int c = i / 3, k = i % 3;
    if (k == 0) { *offset = p.conv[c].w_off; *numel = (size_t)p.conv[c].cout * p.conv[c].cin * p.conv[c].ks * p.conv[c].ks; }
    else if (k == 1) { *offset = p.bn[c].g_off; *numel = p.bn[c].c; }
    else { *offset = p.bn[c].b_off; *numel = p.bn[c].c; }
    return B200OCL_OK;
  }
  const int l = (i - n_conv_t) / 2, k = (i - n_conv_t) % 2;
  if (k == 0) { *offset = p.lin[l].w_off; *numel = (size_t)p.lin[l].in * p.lin[l].out; }
  else { *offset = p.lin[l].b_off; *numel = p.lin[l].out; }
  if (p.head != 0 && l == 0) *has_grad = 0;
  return B200OCL_OK;
}

int b200ocl_net_pack(const b200ocl_net_desc* desc, const b200ocl_net_state* st, void* stream) {
  using namespace b200ocl;
  NetPlan p;
  int rc = check_state(desc, st, p);
  if (rc) return rc;
  return launch_pack(p, st->params, st->packed, static_cast<cudaStream_t>(stream));
}

static void selftest_layer(b200ocl::ConvL& c, int cin, int cout, int H, int W, int ks, int stride, size_t& pk) {
  c = b200ocl::ConvL{};
  c.cin = cin; c.cout = cout; c.ks = ks; c.stride = stride; c.pad = (ks == 3) ? 1 : 0;
  c.hin = H; c.win = W;
  c.hout = b200ocl::conv_out(H, ks, stride, c.pad);
  c.wout = b200ocl::conv_out(W, ks, stride, c.pad);
  c.w_off = 0;
  pk = 0;
  b200ocl::conv_pack_layout(c, pk);
}

size_t b200ocl_conv_selftest_workspace_bytes(int N, int cin, int cout, int H, int W, int ks, int stride) {
  b200ocl::ConvL c;
  size_t pk = 0;
  selftest_layer(c, cin, cout, H, W, ks, stride, pk);
  const size_t M = (size_t)N * H * W;   // upper bound (stride 1)
  const size_t stat = (size_t)b200ocl::conv_max_grid_m((int)M) * (cin > cout ? cin : cout) * 2 * sizeof(double);
  return b200ocl::align_up(pk * sizeof(float), 256) + b200ocl::align_up(stat, 256) + 256 /* counters */ + 256;
}

int b200ocl_conv_selftest(const float* x, const float* w_oihw, float* out, int N, int H, int W, int cin, int cout,
                          int ks, int stride, int dgrad, int path, int mode, float* stats_out, void* workspace,
                          size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(x && w_oihw && out && workspace, "null pointer");
  B200OCL_CHECK_ARG(N > 0 && H > 0 && W > 0 && cin % 20 == 0 && cout % 20 == 0 && cin > 0 && cout > 0, "bad shape");
  B200OCL_CHECK_ARG(mode >= 0 && mode <= 4 && (mode != 2 || (stats_out && !dgrad)), "mode 2 (train) needs stats_out, forward only");
  B200OCL_CHECK_ARG(mode < 3 || (stats_out && !dgrad && (mode == 3 || cin == cout)),
                    "modes 3 / 4 (eval) need stats_out, forward only; mode 4 needs cin == cout");
  B200OCL_CHECK_ARG((ks == 3 || ks == 1) && (stride == 1 || stride == 2) && (!dgrad || (ks == 3 && stride == 1)),
                    "3x3 or 1x1, stride 1 or 2; data gradient for 3x3 stride 1 only");
  B200OCL_CHECK_ARG(workspace_bytes >= b200ocl_conv_selftest_workspace_bytes(N, cin, cout, H, W, ks, stride), "workspace too small");
  NetPlan p;
  memset(&p, 0, sizeof(p));
  p.n_conv = 1;
  size_t pk = 0;
  selftest_layer(p.conv[0], cin, cout, H, W, ks, stride, pk);
  p.n_packed = pk;
  unsigned char* base = static_cast<unsigned char*>(workspace);
  float* packed = reinterpret_cast<float*>(base);
  double* stat_part = reinterpret_cast<double*>(base + align_up(pk * sizeof(float), 256));
  const size_t M = (size_t)N * H * W;
  const size_t stat = (size_t)conv_max_grid_m((int)M) * (cin > cout ? cin : cout) * 2 * sizeof(double);
  unsigned int* counters = reinterpret_cast<unsigned int*>(reinterpret_cast<unsigned char*>(stat_part) + align_up(stat, 256));
  int rc = launch_pack(p, w_oihw, packed, stream);
  if (rc) return rc;
  ConvArgs a = conv_layer_args(p.conv[0], N, x, packed, out, dgrad);
  a.mode = mode >= 3 ? CONV_EVAL : mode == 2 ? CONV_TRAIN : (mode == 1 ? CONV_ACCUM : CONV_RAW);
  a.force_path = path;
  a.eps = NET_BN_EPS;
  a.momentum = NET_BN_MOMENTUM;
  if (mode == 2) {
    B200OCL_CUDA(cudaMemsetAsync(counters, 0, 64, stream));
    B200OCL_CUDA(cudaMemsetAsync(stats_out, 0, (size_t)4 * cout * sizeof(float), stream));
    a.stat_part = stat_part;
    a.counter = counters;
    a.save_mean = stats_out;
    a.save_invstd = stats_out + cout;
    a.run_mean = stats_out + 2 * cout;
    a.run_var = stats_out + 3 * cout;
  }
  if (mode >= 3) {
    a.rmean = stats_out;
    a.rvar = stats_out + cout;
    a.gamma = stats_out + 2 * cout;
    a.beta = stats_out + 3 * cout;
    a.residual = mode == 4 ? x : nullptr;
    a.relu = mode == 4;
  }
  return launch_conv(a, stream);
}

int b200ocl_net_sgd_step(const b200ocl_net_desc* desc, const b200ocl_net_state* st, float lr, float weight_decay,
                         const b200ocl_net_state* dst, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NetPlan p;
  int rc = check_state(desc, st, p);
  if (rc) return rc;
  B200OCL_CHECK_ARG(st->grads, "state has no gradient arena");
  float* out_params = dst ? dst->params : st->params;
  float* out_packed = dst ? dst->packed : st->packed;
  B200OCL_CHECK_ARG(out_params && out_packed, "destination state incomplete");
  size_t skip_lo, skip_hi;
  sgd_skip_range(p, skip_lo, skip_hi);
  const unsigned blocks = arena_grid(p, 8, (size_t)-1);
  B200OCL_PROF("sgd", 12.0 * p.n_params, stream);
  net_sgd_kernel<false><<<blocks, 256, 0, stream>>>(st->params, st->grads, out_params, p.n_params, lr,
                                                              weight_decay, skip_lo, skip_hi, nullptr, nullptr);
  B200OCL_LAUNCHED();
  return launch_pack(p, out_params, out_packed, stream);
}

// The workspace of the entry points that reduce over the arenas (b200ocl::REDUCE_WS_BYTES); 0 for a bad description.
static size_t reduce_workspace_bytes(const b200ocl_net_desc* desc) {
  using namespace b200ocl;
  NetPlan p;
  if (!desc || build_plan(*desc, p)) return 0;
  return REDUCE_WS_BYTES;
}

size_t b200ocl_net_sgd_step_clipped_workspace_bytes(const b200ocl_net_desc* desc) {
  return reduce_workspace_bytes(desc);   // partials, then counter and coefficient
}

int b200ocl_net_sgd_step_clipped(const b200ocl_net_desc* desc, const b200ocl_net_state* st, float lr,
                                 float weight_decay, float max_norm, float* norm_out, void* workspace,
                                 size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NetPlan p;
  int rc = check_state(desc, st, p);
  if (rc) return rc;
  B200OCL_CHECK_ARG(st->grads, "state has no gradient arena");
  if ((rc = check_workspace("b200ocl_net_sgd_step_clipped", workspace, workspace_bytes,
                            b200ocl_net_sgd_step_clipped_workspace_bytes(desc)))) return rc;
  double* part = static_cast<double*>(workspace);
  unsigned int* counter = reduce_counter(workspace);
  float* coef = reduce_scalars(workspace);
  size_t skip_lo, skip_hi;
  sgd_skip_range(p, skip_lo, skip_hi);
  const unsigned norm_grid = arena_grid(p, 2, NORM_MAX_GRID);
  B200OCL_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int), stream));
  B200OCL_PROF("grad_norm", 4.0 * p.n_params, stream);
  grad_norm_kernel<<<norm_grid, 256, 0, stream>>>(st->grads, p.n_params, skip_lo, skip_hi, max_norm, part, counter, coef,
                                                  norm_out);
  B200OCL_LAUNCHED();
  B200OCL_PROF("sgd", 16.0 * p.n_params, stream);
  net_sgd_kernel<true><<<arena_grid(p, 8, (size_t)-1), 256, 0, stream>>>(st->params, st->grads, st->params, p.n_params, lr,
                                                             weight_decay, skip_lo, skip_hi, coef, st->grads);
  B200OCL_LAUNCHED();
  return launch_pack(p, st->params, st->packed, stream);
}

static int ewc_setup(const char* entry, const b200ocl_net_desc* desc, const b200ocl_net_state* st,
                     const b200ocl_ewc_state* ewc, void* workspace, size_t workspace_bytes, b200ocl::NetPlan& p) {
  using namespace b200ocl;
  int rc = check_state(desc, st, p);
  if (rc) return rc;
  B200OCL_CHECK_ARG(ewc && ewc->running && ewc->tmp && ewc->normalized && ewc->prev, "EWC state incomplete");
  return check_workspace(entry, workspace, workspace_bytes, REDUCE_WS_BYTES);
}

size_t b200ocl_net_sgd_step_ewc_workspace_bytes(const b200ocl_net_desc* desc) { return reduce_workspace_bytes(desc); }

int b200ocl_net_sgd_step_ewc(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const b200ocl_ewc_state* ewc,
                             float lr, float weight_decay, float up, int flags, float ema_keep, float ema_add,
                             float* penalty_out, void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NetPlan p;
  int rc = ewc_setup("b200ocl_net_sgd_step_ewc", desc, st, ewc, workspace, workspace_bytes, p);
  if (rc) return rc;
  size_t skip_lo, skip_hi;
  sgd_skip_range(p, skip_lo, skip_hi);
  const unsigned grid = arena_grid(p, 8, NORM_MAX_GRID);
  unsigned int* counter = reduce_counter(workspace);
  B200OCL_CHECK_ARG(st->grads, "state has no gradient arena");
  B200OCL_CHECK_ARG((flags & ~(B200OCL_EWC_PENALTY | B200OCL_EWC_EMA)) == 0, "unknown EWC flags");
  const bool pen = flags & B200OCL_EWC_PENALTY, ema = flags & B200OCL_EWC_EMA;
  double* part = static_cast<double*>(workspace);
  float* pen_out = pen ? penalty_out : nullptr;
  if (pen_out) B200OCL_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int), stream));
  auto kernel = pen ? (ema ? net_sgd_ewc_kernel<true, true> : net_sgd_ewc_kernel<false, true>)
                    : (ema ? net_sgd_ewc_kernel<true, false> : net_sgd_ewc_kernel<false, false>);
  B200OCL_PROF("sgd_ewc", 4.0 * p.n_params * (5 + (pen ? 3 : 0) + (ema ? 2 : 0)), stream);
  kernel<<<grid, 256, 0, stream>>>(st->params, st->grads, ewc->running, ewc->tmp, ewc->normalized, ewc->prev,
                                   p.n_params, skip_lo, skip_hi, lr, weight_decay, up, ema_keep, ema_add, part, counter,
                                   pen_out);
  B200OCL_LAUNCHED();
  if (penalty_out && !pen) B200OCL_CUDA(cudaMemsetAsync(penalty_out, 0, sizeof(float), stream));
  return launch_pack(p, st->params, st->packed, stream);
}

size_t b200ocl_ewc_consolidate_workspace_bytes(const b200ocl_net_desc* desc) { return reduce_workspace_bytes(desc); }

int b200ocl_ewc_consolidate(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const b200ocl_ewc_state* ewc,
                            void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NetPlan p;
  int rc = ewc_setup("b200ocl_ewc_consolidate", desc, st, ewc, workspace, workspace_bytes, p);
  if (rc) return rc;
  size_t skip_lo, skip_hi;
  sgd_skip_range(p, skip_lo, skip_hi);
  const unsigned grid = arena_grid(p, 8, NORM_MAX_GRID);
  unsigned int* counter = reduce_counter(workspace);
  float* range = reduce_scalars(workspace);
  B200OCL_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int), stream));
  B200OCL_PROF("ewc_consolidate", 12.0 * p.n_params, stream);
  ewc_minmax_kernel<<<grid, 256, 0, stream>>>(st->params, ewc->running, ewc->prev, p.n_params, skip_lo, skip_hi,
                                              static_cast<float2*>(workspace), counter, range);
  B200OCL_LAUNCHED();
  B200OCL_PROF("ewc_consolidate", 8.0 * p.n_params, stream);
  ewc_normalize_kernel<<<grid, 256, 0, stream>>>(ewc->running, ewc->normalized, p.n_params, skip_lo, skip_hi, range);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

size_t b200ocl_net_eval_workspace_bytes(const b200ocl_net_desc* desc, int N) {
  using namespace b200ocl;
  NetPlan p;
  if (!desc || N < 0 || build_plan(*desc, p)) return 0;
  return eval_ws(p, N > 0 ? N : 1, nullptr).bytes;
}

int b200ocl_net_features_eval(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const float* x, int N,
                              float* feat, void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NetPlan p;
  int rc = check_state(desc, st, p);
  if (rc) return rc;
  B200OCL_CHECK_ARG(N >= 0, "negative batch");
  if (N == 0) return B200OCL_OK;
  B200OCL_CHECK_ARG(x && feat, "null pointer");
  if ((rc = check_workspace("b200ocl_net_features_eval", workspace, workspace_bytes,
                            b200ocl_net_eval_workspace_bytes(desc, N)))) return rc;
  EvalWs w = eval_ws(p, N, workspace);
  float* cur = w.buf[0];
  float* t1 = w.buf[1];
  float* t2 = w.buf[2];
  float* nxt = w.buf[3];
  if ((rc = conv_eval(p, *st, 0, N, x, cur, nullptr, 1, stream))) return rc;   // relu(bn1(conv1(x)))
  for (int b = 0; b < 8; ++b) {
    const BlockL& B = p.blk[b];
    if ((rc = conv_eval(p, *st, B.c1, N, cur, t1, nullptr, 1, stream))) return rc;
    const float* res = cur;
    if (B.sc >= 0) {
      if ((rc = conv_eval(p, *st, B.sc, N, cur, t2, nullptr, 0, stream))) return rc;
      res = t2;
    }
    if ((rc = conv_eval(p, *st, B.c2, N, t1, nxt, res, 1, stream))) return rc;
    float* tmp = cur; cur = nxt; nxt = tmp;
  }
  const int total = N * p.pooled_h * p.pooled_w * (desc->nf * 8);
  B200OCL_PROF("pool", 4.0 * 17 * total, stream);
  pool_kernel<<<(total + 255) / 256, 256, 0, stream>>>(cur, feat, N, p.final_h, p.final_w, desc->nf * 8, p.pooled_h,
                                                       p.pooled_w);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

size_t b200ocl_net_train_workspace_bytes(const b200ocl_net_desc* desc, int N) {
  using namespace b200ocl;
  NetPlan p;
  if (!desc || N < 0 || build_plan(*desc, p)) return 0;
  return train_ws(p, N > 0 ? N : 1, nullptr, sm_count()).bytes;
}

int b200ocl_net_train_ws_layout(const b200ocl_net_desc* desc, int N, int layer, b200ocl_net_ws_layout* out) {
  using namespace b200ocl;
  B200OCL_CHECK_ARG(desc && out, "null pointer");
  NetPlan p;
  const int rc = build_plan(*desc, p);
  if (rc) {
    set_error("b200ocl_net_train_ws_layout: unsupported network description");
    return rc;
  }
  B200OCL_CHECK_ARG(N >= 1, "need N >= 1");
  B200OCL_CHECK_ARG(layer >= 0 && layer < p.n_conv, "layer out of range");
  const int sms = sm_count();
  const TrainWs w = train_ws(p, N, nullptr, sms);   // offsets from a null base
  const ConvL& c = p.conv[layer];
  auto off = [](const void* q) { return (size_t)reinterpret_cast<uintptr_t>(q); };
  *out = b200ocl_net_ws_layout{};
  out->bytes = w.bytes;
  out->z = off(w.z + (size_t)N * c.act_off);
  out->a = off(w.a + (size_t)N * c.act_off);
  out->mean = off(w.save + p.bn[layer].save_off);
  out->invstd = off(w.save + p.bn[layer].save_off + p.bn[layer].c);
  out->feat = off(w.feat);
  out->hid = off(w.hid);
  out->proj = off(w.proj);
  out->wg_part = off(w.wg_part);
  out->wg_layer = off(w.wg_part + w.wg_off[layer]);
  out->cin = c.cin; out->cout = c.cout; out->ks = c.ks; out->stride = c.stride; out->hout = c.hout; out->wout = c.wout;
  const BnBwdGeom g = bn_bwd_geom(N * c.hout * c.wout, c.cout, sms, true);   // b200ocl_net_backward always has a ready flag
  out->bn_fused = g.fused ? 1 : 0;
  out->bn_grid = g.grid;
  const WgradPlan wp = wgrad_plan(p, layer, N, sms);
  out->wgrad_kernel = wp.kernel == WGRAD_STEM ? 0 : (wp.kernel == WGRAD_TC ? 1 : 2);
  out->wgrad_splits = wp.splits;
  out->sms = sms;
  return B200OCL_OK;
}

static int net_forward_impl(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const float* x, int N, float* out,
                            void* workspace, size_t workspace_bytes, void* stream_, int ev) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NetPlan p;
  int rc = check_state(desc, st, p);
  if (rc) return rc;
  B200OCL_CHECK_ARG(N >= 1 && x && out, "need N >= 1 and non-null x/out");
  if ((rc = check_workspace("b200ocl_net_forward_train", workspace, workspace_bytes,
                            b200ocl_net_train_workspace_bytes(desc, N)))) return rc;
  TrainWs w = train_ws(p, N, workspace, sm_count());
  B200OCL_CUDA(cudaMemsetAsync(w.counters, 0, NET_COUNTERS * sizeof(unsigned int), stream));
  if (ev == STATS_DEFER) B200OCL_CUDA(cudaMemsetAsync(w.run_defer, 0, p.n_stats * sizeof(float), stream));
  if ((rc = conv_train(p, *st, w, 0, N, x, stream, ev))) return rc;
  if ((rc = bn_apply_train(p, *st, w, 0, N, -1, nullptr, stream))) return rc;
  const float* cur = w.a + (size_t)N * p.conv[0].act_off;
  for (int b = 0; b < 8; ++b) {
    const BlockL& B = p.blk[b];
    if ((rc = conv_train(p, *st, w, B.c1, N, cur, stream, ev))) return rc;
    if ((rc = bn_apply_train(p, *st, w, B.c1, N, -1, nullptr, stream))) return rc;
    const float* a1 = w.a + (size_t)N * p.conv[B.c1].act_off;
    if ((rc = conv_train(p, *st, w, B.c2, N, a1, stream, ev))) return rc;
    if (B.sc >= 0) {
      if ((rc = conv_train(p, *st, w, B.sc, N, cur, stream, ev))) return rc;
      if ((rc = bn_apply_train(p, *st, w, B.c2, N, B.sc, nullptr, stream))) return rc;
    } else {
      if ((rc = bn_apply_train(p, *st, w, B.c2, N, -1, cur, stream))) return rc;
    }
    cur = w.a + (size_t)N * p.conv[B.c2].act_off;
  }
  if (st->bn_tracked && ev == STATS_RUNNING) {
    B200OCL_PROF("misc", 16.0 * p.n_conv, stream);
    bump_tracked_kernel<<<1, 32, 0, stream>>>(reinterpret_cast<long long*>(st->bn_tracked), p.n_conv);
    B200OCL_LAUNCHED();
  }
  const int total = N * p.pooled_h * p.pooled_w * (desc->nf * 8);
  B200OCL_PROF("pool", 4.0 * 17 * total, stream);
  pool_kernel<<<(total + 255) / 256, 256, 0, stream>>>(cur, w.feat, N, p.final_h, p.final_w, desc->nf * 8, p.pooled_h,
                                                       p.pooled_w);
  B200OCL_LAUNCHED();
  return head_forward(p, *st, w.feat, N, w.hid, w.proj, out, stream);
}

int b200ocl_net_forward_train(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const float* x, int N,
                              float* out, void* workspace, size_t workspace_bytes, void* stream_) {
  return net_forward_impl(desc, st, x, N, out, workspace, workspace_bytes, stream_, b200ocl::STATS_RUNNING);
}

int b200ocl_net_forward_evalgrad(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const float* x, int N,
                                 float* out, void* workspace, size_t workspace_bytes, void* stream_) {
  return net_forward_impl(desc, st, x, N, out, workspace, workspace_bytes, stream_, b200ocl::STATS_EVAL);
}

int b200ocl_net_forward_train_deferred(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const float* x, int N,
                                       float* out, void* workspace, size_t workspace_bytes, void* stream_) {
  return net_forward_impl(desc, st, x, N, out, workspace, workspace_bytes, stream_, b200ocl::STATS_DEFER);
}

int b200ocl_net_apply_running_stats(const b200ocl_net_desc* desc, const b200ocl_net_state* st, int N, void* workspace,
                                    size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NetPlan p;
  int rc = check_state(desc, st, p);
  if (rc) return rc;
  B200OCL_CHECK_ARG(N >= 1, "need N >= 1");
  if ((rc = check_workspace("b200ocl_net_apply_running_stats", workspace, workspace_bytes,
                            b200ocl_net_train_workspace_bytes(desc, N)))) return rc;
  TrainWs w = train_ws(p, N, workspace, sm_count());
  const int n = (int)p.n_stats;
  B200OCL_PROF("misc", 12.0 * n, stream);
  bn_running_apply_kernel<<<(n + 255) / 256, 256, 0, stream>>>(st->bn_stats, w.run_defer, n, NET_BN_MOMENTUM,
                                                               reinterpret_cast<long long*>(st->bn_tracked), p.n_conv);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

int b200ocl_ce_loss(const float* logits, const int64_t* labels, int N, int C, float* loss, float* per_sample,
                    float* dlogits, int64_t* n_correct, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(logits && labels && N >= 1 && C >= 1, "need logits, labels, N >= 1, C >= 1");
  B200OCL_PROF("ce_loss", 8.0 * N * C, stream);
  ce_kernel<<<1, 256, 0, stream>>>(logits, reinterpret_cast<const long long*>(labels), N, C, loss, per_sample, dlogits,
                                   reinterpret_cast<long long*>(n_correct));
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

int b200ocl_cls_loss(const float* logits, const int64_t* labels, int N, int C, int mode, const int64_t* cols,
                     int n_cols, int n_old, const int64_t* pos_table, int table_len, const float* teacher, float w_ce,
                     float w_kd, float* loss, float* dlogits, int64_t* n_correct, int* err_flag, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(logits && labels && N >= 1 && C >= 1, "need logits, labels, N >= 1, C >= 1");
  B200OCL_CHECK_ARG(mode == B200OCL_CLS_CE || mode == B200OCL_CLS_LABELS || mode == B200OCL_CLS_SEPARATED, "unknown mode");
  B200OCL_CHECK_ARG(mode != B200OCL_CLS_SEPARATED ||
                    (cols && pos_table && n_cols >= 1 && n_old >= 0 && n_old <= n_cols && table_len >= 0),
                    "separated softmax needs cols [n_cols >= 1], 0 <= n_old <= n_cols and a position table");
  if (mode == B200OCL_CLS_LABELS && C > B200OCL_CLS_MAX_C) {
    set_error("b200ocl_cls_loss: labels trick over C = %d > %d classes", C, B200OCL_CLS_MAX_C);
    return B200OCL_EUNSUPPORTED;
  }
  ClsLossArgs a{logits, reinterpret_cast<const long long*>(labels), N, C, mode,
                reinterpret_cast<const long long*>(cols), n_cols, n_old,
                reinterpret_cast<const long long*>(pos_table), table_len, teacher, w_ce, w_kd, loss, dlogits,
                reinterpret_cast<long long*>(n_correct), err_flag};
  const size_t smem = mode == B200OCL_CLS_LABELS ? (size_t)C * sizeof(int) : 0;
  B200OCL_PROF("cls_loss", (teacher ? 12.0 : 8.0) * N * C, stream);
  cls_loss_kernel<<<1, 256, smem, stream>>>(a);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

int b200ocl_icarl_loss(const float* logits, const float* teacher, const int64_t* labels, const int64_t* pos_table,
                       int pos_len, int N, int n_stream, int C, int K, int n_old, float* loss, float* dlogits,
                       int* err_flag, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(logits && N >= 1 && C >= 1, "need logits, N >= 1, C >= 1");
  B200OCL_CHECK_ARG(n_stream >= 0 && n_stream <= N, "need 0 <= n_stream <= N");
  B200OCL_CHECK_ARG(n_stream == 0 || (labels && pos_table && pos_len >= 0), "stream rows need labels and a position table");
  B200OCL_CHECK_ARG(K >= 1 && K <= C, "need 1 <= K <= C");
  B200OCL_CHECK_ARG(n_old >= 0 && n_old <= K, "need 0 <= n_old <= K");
  B200OCL_CHECK_ARG(teacher || n_old == 0, "n_old > 0 needs the teacher's logits");
  IcarlLossArgs a{logits, teacher, reinterpret_cast<const long long*>(labels),
                  reinterpret_cast<const long long*>(pos_table), pos_len, N, n_stream, C, K, n_old, loss, dlogits,
                  err_flag};
  B200OCL_PROF("icarl_loss", 4.0 * N * (K + n_old) + (dlogits ? 4.0 * N * C : 0.0), stream);
  icarl_loss_kernel<<<1, 256, 0, stream>>>(a);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

}  // extern "C"
