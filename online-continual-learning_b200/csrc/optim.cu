// optim.cu -- the optimizer steps over the parameter arena and over flat buffers: torch.optim.SGD.step
// (setup_elements.py:73-75) and MIR's virtual update (mir_retrieve.py:34-47), GDumb's clip_grad_norm_ + step
// (agents/gdumb.py:82-83), EWC++'s per-step pass and consolidation (agents/ewc_pp.py:40-112) and torch.optim.Adam.step
// (setup_elements.py:76-78).  Every per-element update is one instantiation of arena_step_kernel.
#include <math.h>

#include <type_traits>

#include "net_plan.cuh"

namespace b200ocl {
namespace {

// L2 norm of the gradient arena and the EWC++ penalty: per-CTA fp64 partials, added in CTA order by the last CTA.
constexpr int NORM_MAX_GRID = 1024;

// Workspace of the arena reductions (grad_norm_kernel, the EWC++ kernels): one 8-byte partial per CTA (up to
// NORM_MAX_GRID), then, at the next 256-byte boundary, the arrival counter followed by the reduction's fp32 results.
constexpr size_t REDUCE_TAIL_OFF = (NORM_MAX_GRID * sizeof(double) + 255) / 256 * 256;
constexpr size_t REDUCE_WS_BYTES = REDUCE_TAIL_OFF + 256;
inline unsigned int* reduce_counter(void* ws) {
  return reinterpret_cast<unsigned int*>(static_cast<unsigned char*>(ws) + REDUCE_TAIL_OFF);
}
inline float* reduce_scalars(void* ws) { return reinterpret_cast<float*>(reduce_counter(ws) + 1); }

// Grid of a grid-stride pass of 256-thread CTAs over n elements: at most per_sm CTAs per SM and `cap`.
inline unsigned step_grid(size_t n, int per_sm, size_t cap) {
  size_t blocks = (n + 255) / 256;
  const size_t sm_cap = (size_t)per_sm * sm_count();
  if (blocks > sm_cap) blocks = sm_cap;
  return (unsigned)(blocks < cap ? blocks : cap);
}

// Block sum of acc over the 256 threads, stored as this CTA's partial; returns true in thread 0 of the last CTA to
// arrive, with the partials added in CTA order in `total`: the sum does not depend on the order the CTAs end in.
__device__ __forceinline__ bool last_cta_sum(double acc, double* __restrict__ part, unsigned int* counter,
                                             double& total) {
  __shared__ double s_red[8];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
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
  if (!is_last || threadIdx.x != 0) return false;
  __threadfence();
  double t = 0.0;
  for (unsigned int b = 0; b < gridDim.x; ++b) t += __ldcg(part + b);
  total = t;
  return true;
}

// ----------------------------------------------------------------------------- the update policies
// torch.optim.SGD's update (momentum off) as torch's CUDA kernel contracts it.  Its prescale is GDumb's clipping
// coefficient, which grad_norm_kernel leaves in device memory.
struct Sgd {
  float lr, wd;
  const float* coef;
  __device__ __forceinline__ float prescale() const { return *coef; }
  __device__ __forceinline__ float update(float w, float gi, size_t, float*, float*) const {
    if (wd != 0.f) gi = fmaf(wd, w, gi);
    return w - lr * gi;
  }
};

// torch.optim.Adam's update (amsgrad, maximize and decoupled weight decay off) as torch's CUDA kernels round it, one op
// at a time, so that the step is bit-identical to the optimizer the caller built:
//   g' = fma(wd, p, g)                   grad.add(param, alpha=wd), only when wd != 0 (a temporary: g is not written)
//   m  = lerp(m, g', w1)                 exp_avg.lerp_(grad, 1 - beta1), ATen/native/Lerp.h as nvcc contracts it:
//                                        fma(w1, g' - m, m) for |w1| < 0.5, else fma(-(g' - m), 1 - w1, g')
//   v  = fma(c2, g' * g', v * b2)        exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
//                                        (DeviceAddCmulCdiv.cuh: fma(g', g', v * b2) when the value is 1)
//   d  = sqrt(v) / bc2_sqrt + eps        FOREACH (torch's default on CUDA, _foreach_div_ by a scalar list): an IEEE
//                                        division; otherwise CUDA Tensor / Python float, which multiplies by the fp32
//                                        rounding of the double reciprocal: `bc2` holds that reciprocal
//   p  = fma(step_size, m / d, p)        param.addcdiv_(exp_avg, denom, value=-(lr / bc1))
// Its prescale is the review trick's p.grad.clone() / 10. (also Tensor / Python float: g * fp32(1 / 10.), `gmul`).
struct AdamCoef {
  float wd, w1, w1c, b2, c2, bc2, eps, step, gmul;   // w1c = 1 - w1 in fp32, as Lerp.h forms it on the device
};

template <bool FOREACH>
struct Adam {
  AdamCoef c;
  __device__ __forceinline__ float prescale() const { return c.gmul; }
  __device__ __forceinline__ float update(float w, float gi, size_t i, float* m, float* v) const {
    if (c.wd != 0.f) gi = __fmaf_rn(c.wd, w, gi);
    float mi = m[i];
    const float diff = __fsub_rn(gi, mi);
    mi = fabsf(c.w1) < 0.5f ? __fmaf_rn(c.w1, diff, mi) : __fmaf_rn(-diff, c.w1c, gi);
    const float vb = __fmul_rn(v[i], c.b2);
    const float vi = c.c2 == 1.f ? __fmaf_rn(gi, gi, vb) : __fmaf_rn(c.c2, __fmul_rn(gi, gi), vb);
    const float s = __fsqrt_rn(vi);
    const float d = __fadd_rn(FOREACH ? __fdiv_rn(s, c.bc2) : __fmul_rn(s, c.bc2), c.eps);
    m[i] = mi;
    v[i] = vi;
    return __fmaf_rn(c.step, __fdiv_rn(mi, d), w);
  }
};

// The kernel's coefficients from the caller's scalars; false for unknown flags.
inline bool adam_coef(const b200ocl_adam_scalars& s, int flags, AdamCoef& c) {
  if (flags & ~(B200OCL_ADAM_FOREACH | B200OCL_ADAM_GRAD_SCALE)) return false;
  c.wd = s.weight_decay;
  c.w1 = s.beta1_c;
  c.w1c = 1.f - s.beta1_c;
  c.b2 = s.beta2;
  c.c2 = s.beta2_c;
  c.bc2 = (flags & B200OCL_ADAM_FOREACH) ? s.bc2_sqrt : s.bc2_sqrt_inv;
  c.eps = s.eps;
  c.step = s.step_size;
  c.gmul = (flags & B200OCL_ADAM_GRAD_SCALE) ? s.grad_scale : 1.f;
  return true;
}

// EWC++'s scalars: the penalty's gradient factor and the EMA's weights.
struct EwcScalars {
  float up, ema_keep, ema_add;
};

// ----------------------------------------------------------------------------- one step over the arena
// One pass per element, outside [skip_lo, skip_hi), in the order of the torch ops it replaces:
//   PRESCALE  g *= the update's prescale, one rounding, written back to the gradient arena (torch scales p.grad in
//             place)
//   EWC       EWC++ (ewc_pp.py:58-63, 104-108): the EMA into running (EMA), the penalty's gradient added to the
//             network's and written back (PEN), then accum_fisher's tmp += g*g
//   then      the update, with Adam's m and v, in place; the plain SGD step writes out instead (out == p but for MIR's
//             virtual update)
// Every torch op is its own rounding, so the EWC++ products and sums are spelled with __f*_rn: nvcc would contract them
// to fma.  With PEN and pen_out, sum F*d^2 over the pre-step weights goes to pen_out (last_cta_sum).  Each element is
// read and then written by one thread only, so a read-only load of an arena the step also writes cannot see a stale
// value.
template <class Update, bool PRESCALE, bool EWC, bool EMA, bool PEN>
__global__ void __launch_bounds__(256) arena_step_kernel(float* __restrict__ p, float* __restrict__ g,
                                                         float* __restrict__ out, float* __restrict__ m,
                                                         float* __restrict__ v, float* __restrict__ running,
                                                         float* __restrict__ tmp, const float* __restrict__ fisher,
                                                         const float* __restrict__ prev, size_t n, size_t skip_lo,
                                                         size_t skip_hi, Update u, EwcScalars e,
                                                         double* __restrict__ part, unsigned int* counter,
                                                         float* pen_out) {
  // Only the plain SGD step may write a second arena (MIR's virtual update), which must hold the skipped tensors too;
  // every other step leaves them untouched in every arena.
  constexpr bool COPY_SKIPPED = std::is_same<Update, Sgd>::value && !EWC;
  const float c = PRESCALE ? u.prescale() : 1.f;
  double acc = 0.0;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (i >= skip_lo && i < skip_hi) {   // tensors that never receive a gradient: torch steps nothing there
      if (COPY_SKIPPED) out[i] = p[i];
      continue;
    }
    const float w = p[i];
    float gi = g[i];
    if (PRESCALE) {
      gi = __fmul_rn(gi, c);
      g[i] = gi;
    }
    if (EWC) {
      float t = tmp[i];
      if (EMA) {
        // (1 - alpha) * running + (1/fua * alpha) * tmp, then tmp = 0 (ewc_pp.py:104-108)
        running[i] = __fadd_rn(__fmul_rn(e.ema_keep, running[i]), __fmul_rn(e.ema_add, t));
        t = 0.f;
      }
      if (PEN) {
        // autograd of lambda * (F * (p - prev)**2).sum(): (up * F) * (2 * d), added once to the network's gradient
        const float f = fisher[i];
        const float d = __fsub_rn(w, prev[i]);
        gi = __fadd_rn(gi, __fmul_rn(__fmul_rn(e.up, f), __fmul_rn(2.f, d)));
        g[i] = gi;
        const double dd = (double)d;
        acc = fma((double)f * dd, dd, acc);
      }
      tmp[i] = __fadd_rn(t, __fmul_rn(gi, gi));   // accum_fisher: tmp += grad ** 2 (pow 2 is grad * grad)
    }
    (COPY_SKIPPED ? out : p)[i] = u.update(w, gi, i, m, v);
  }
  double pen;
  if (PEN && pen_out && last_cta_sum(acc, part, counter, pen)) *pen_out = (float)pen;
}

// One step for launch_step: the arenas, n elements of which [skip_lo, skip_hi) are left out, whether the gradient is
// prescaled, and for the EWC++ steps (ewc non-null) their state, flags (B200OCL_EWC_*), scalars, reduction workspace
// and penalty output.
struct ArenaStep {
  float *p, *g;
  float* out;     // the plain SGD step's destination
  float *m, *v;   // Adam's exp_avg and exp_avg_sq
  size_t n, skip_lo, skip_hi;
  bool prescale;
  const b200ocl_ewc_state* ewc;
  int ewc_flags;
  EwcScalars e;
  void* ws;
  float* penalty_out;
};

// The step over a network state's arenas, in place.  It leaves out the tensors that never receive a gradient (the
// SupCon network's unused classifier).
ArenaStep net_step(const NetPlan& p, const b200ocl_net_state& st) {
  ArenaStep a{};
  a.p = a.out = st.params;
  a.g = st.grads;
  a.n = p.n_params;
  if (p.head != 0) {
    a.skip_lo = p.lin[0].w_off;
    a.skip_hi = p.lin[0].b_off + p.lin[0].out;
  }
  return a;
}

// Launches the instantiation of arena_step_kernel that the update and a's flags select, as kernel class `prof` with
// `work` bytes.  The EWC++ steps write a partial per CTA, so their grid stops at NORM_MAX_GRID; with the penalty off,
// penalty_out is set to 0.
template <class Update>
int launch_step(const ArenaStep& a, const Update& u, const char* prof, double work, cudaStream_t stream) {
  const bool ema = a.ewc_flags & B200OCL_EWC_EMA, pen = a.ewc_flags & B200OCL_EWC_PENALTY;
  const auto kernel = !a.ewc ? (a.prescale ? arena_step_kernel<Update, true, false, false, false>
                                           : arena_step_kernel<Update, false, false, false, false>)
                      : ema  ? (pen ? arena_step_kernel<Update, false, true, true, true>
                                    : arena_step_kernel<Update, false, true, true, false>)
                             : (pen ? arena_step_kernel<Update, false, true, false, true>
                                    : arena_step_kernel<Update, false, true, false, false>);
  const unsigned grid = step_grid(a.n, 8, a.ewc ? NORM_MAX_GRID : (size_t)-1);
  const b200ocl_ewc_state e = a.ewc ? *a.ewc : b200ocl_ewc_state{};
  unsigned int* counter = a.ewc ? reduce_counter(a.ws) : nullptr;
  float* pen_out = pen ? a.penalty_out : nullptr;
  if (pen_out) B200OCL_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int), stream));
  B200OCL_PROF(prof, work, stream);
  kernel<<<grid, 256, 0, stream>>>(a.p, a.g, a.out, a.m, a.v, e.running, e.tmp, e.normalized, e.prev, a.n, a.skip_lo,
                                   a.skip_hi, u, a.e, static_cast<double*>(a.ws), counter, pen_out);
  B200OCL_LAUNCHED();
  if (a.penalty_out && !pen) B200OCL_CUDA(cudaMemsetAsync(a.penalty_out, 0, sizeof(float), stream));
  return B200OCL_OK;
}

// Adam's update with the division `foreach` selects.
int launch_adam_step(const ArenaStep& a, const AdamCoef& c, bool foreach, const char* prof, double work,
                     cudaStream_t stream) {
  return foreach ? launch_step(a, Adam<true>{c}, prof, work, stream)
                 : launch_step(a, Adam<false>{c}, prof, work, stream);
}

// torch's clipping coefficient (torch/nn/utils/clip_grad.py, _clip_grads_with_norm_) from the L2 norm of the gradient
// arena outside [skip_lo, skip_hi): coef = min(max_norm / (norm + 1e-6), 1) in fp32, with torch's roundings.
__global__ void __launch_bounds__(256) grad_norm_kernel(const float* __restrict__ g, size_t n, size_t skip_lo,
                                                        size_t skip_hi, float max_norm, double* __restrict__ part,
                                                        unsigned int* counter, float* coef, float* norm_out) {
  double acc = 0.0;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (i >= skip_lo && i < skip_hi) continue;
    const double v = (double)g[i];
    acc = fma(v, v, acc);
  }
  double t;
  if (!last_cta_sum(acc, part, counter, t)) return;
  const float norm = (float)sqrt(t);
  // torch forms max_norm / (norm + 1e-6) as Tensor.__rdiv__: (norm + 1e-6).reciprocal() * max_norm, two roundings
  const float q = __fmul_rn(__frcp_rn(norm + 1e-6f), max_norm);
  *coef = q > 1.f ? 1.f : q;          // torch.clamp(max=1.0): a NaN norm stays NaN
  if (norm_out) *norm_out = norm;
}

// ----------------------------------------------------------------------------- EWC++ consolidation
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

}  // namespace
}  // namespace b200ocl

// The workspace of the entry points that reduce over the arenas (b200ocl::REDUCE_WS_BYTES); 0 for a bad description.
static size_t reduce_workspace_bytes(const b200ocl_net_desc* desc) {
  using namespace b200ocl;
  NetPlan p;
  if (!desc || build_plan(*desc, p)) return 0;
  return REDUCE_WS_BYTES;
}

static int ewc_setup(const char* entry, const b200ocl_net_desc* desc, const b200ocl_net_state* st,
                     const b200ocl_ewc_state* ewc, void* workspace, size_t workspace_bytes, b200ocl::NetPlan& p) {
  using namespace b200ocl;
  int rc = check_state(desc, st, p);
  if (rc) return rc;
  B200OCL_CHECK_ARG(ewc && ewc->running && ewc->tmp && ewc->normalized && ewc->prev, "EWC state incomplete");
  return check_workspace(entry, workspace, workspace_bytes, REDUCE_WS_BYTES);
}

extern "C" {

int b200ocl_sgd_step(const float* p, const float* g, float* out, size_t n, float lr, float wd, void* stream_) {
  using namespace b200ocl;
  B200OCL_CHECK_ARG(n == 0 || (p && g && out), "null pointer");
  if (n == 0) return B200OCL_OK;
  ArenaStep a{};
  a.p = const_cast<float*>(p);   // only read: the plain step writes out
  a.g = const_cast<float*>(g);   // only read: the step has no prescale and no penalty
  a.out = out;
  a.n = n;
  return launch_step(a, Sgd{lr, wd, nullptr}, "sgd", 12.0 * n, static_cast<cudaStream_t>(stream_));
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
  ArenaStep a = net_step(p, *st);
  a.out = out_params;
  if ((rc = launch_step(a, Sgd{lr, weight_decay, nullptr}, "sgd", 12.0 * p.n_params, stream))) return rc;
  return launch_pack(p, out_params, out_packed, stream);
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
  unsigned int* counter = reduce_counter(workspace);
  float* coef = reduce_scalars(workspace);
  ArenaStep a = net_step(p, *st);
  a.prescale = true;
  const unsigned norm_grid = step_grid(p.n_params, 2, NORM_MAX_GRID);
  B200OCL_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int), stream));
  B200OCL_PROF("grad_norm", 4.0 * p.n_params, stream);
  grad_norm_kernel<<<norm_grid, 256, 0, stream>>>(st->grads, p.n_params, a.skip_lo, a.skip_hi, max_norm,
                                                  static_cast<double*>(workspace), counter, coef, norm_out);
  B200OCL_LAUNCHED();
  if ((rc = launch_step(a, Sgd{lr, weight_decay, coef}, "sgd", 16.0 * p.n_params, stream))) return rc;
  return launch_pack(p, st->params, st->packed, stream);
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
  B200OCL_CHECK_ARG(st->grads, "state has no gradient arena");
  B200OCL_CHECK_ARG((flags & ~(B200OCL_EWC_PENALTY | B200OCL_EWC_EMA)) == 0, "unknown EWC flags");
  ArenaStep a = net_step(p, *st);
  a.ewc = ewc;
  a.ewc_flags = flags;
  a.e = EwcScalars{up, ema_keep, ema_add};
  a.ws = workspace;
  a.penalty_out = penalty_out;
  const bool pen = flags & B200OCL_EWC_PENALTY, ema = flags & B200OCL_EWC_EMA;
  if ((rc = launch_step(a, Sgd{lr, weight_decay, nullptr}, "sgd_ewc",
                        4.0 * p.n_params * (5 + (pen ? 3 : 0) + (ema ? 2 : 0)), stream))) return rc;
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
  const ArenaStep a = net_step(p, *st);
  const unsigned grid = step_grid(p.n_params, 8, NORM_MAX_GRID);
  unsigned int* counter = reduce_counter(workspace);
  float* range = reduce_scalars(workspace);
  B200OCL_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int), stream));
  B200OCL_PROF("ewc_consolidate", 12.0 * p.n_params, stream);
  ewc_minmax_kernel<<<grid, 256, 0, stream>>>(st->params, ewc->running, ewc->prev, p.n_params, a.skip_lo, a.skip_hi,
                                              static_cast<float2*>(workspace), counter, range);
  B200OCL_LAUNCHED();
  B200OCL_PROF("ewc_consolidate", 8.0 * p.n_params, stream);
  ewc_normalize_kernel<<<grid, 256, 0, stream>>>(ewc->running, ewc->normalized, p.n_params, a.skip_lo, a.skip_hi,
                                                 range);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

int b200ocl_adam_step(float* p, float* g, float* m, float* v, size_t n, const b200ocl_adam_scalars* s, int flags,
                      void* stream_) {
  using namespace b200ocl;
  B200OCL_CHECK_ARG(s && (n == 0 || (p && g && m && v)), "null pointer");
  AdamCoef c;
  B200OCL_CHECK_ARG(adam_coef(*s, flags, c), "unknown Adam flags");
  if (n == 0) return B200OCL_OK;
  ArenaStep a{};
  a.p = p;
  a.g = g;
  a.m = m;
  a.v = v;
  a.n = n;
  a.prescale = flags & B200OCL_ADAM_GRAD_SCALE;
  return launch_adam_step(a, c, flags & B200OCL_ADAM_FOREACH, "adam", 28.0 * n, static_cast<cudaStream_t>(stream_));
}

int b200ocl_net_adam_step(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const b200ocl_adam_state* adam,
                          const b200ocl_adam_scalars* s, int flags, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NetPlan p;
  int rc = check_state(desc, st, p);
  if (rc) return rc;
  B200OCL_CHECK_ARG(st->grads, "state has no gradient arena");
  B200OCL_CHECK_ARG(adam && adam->exp_avg && adam->exp_avg_sq && s, "Adam state incomplete");
  AdamCoef c;
  B200OCL_CHECK_ARG(adam_coef(*s, flags, c), "unknown Adam flags");
  ArenaStep a = net_step(p, *st);
  a.m = adam->exp_avg;
  a.v = adam->exp_avg_sq;
  a.prescale = flags & B200OCL_ADAM_GRAD_SCALE;
  if ((rc = launch_adam_step(a, c, flags & B200OCL_ADAM_FOREACH, "adam", (a.prescale ? 32.0 : 28.0) * p.n_params,
                             stream))) return rc;
  return launch_pack(p, st->params, st->packed, stream);
}

int b200ocl_net_adam_step_ewc(const b200ocl_net_desc* desc, const b200ocl_net_state* st, const b200ocl_ewc_state* ewc,
                              const b200ocl_adam_state* adam, const b200ocl_adam_scalars* s, int adam_flags, float up,
                              int flags, float ema_keep, float ema_add, float* penalty_out, void* workspace,
                              size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  NetPlan p;
  int rc = ewc_setup("b200ocl_net_adam_step_ewc", desc, st, ewc, workspace, workspace_bytes, p);
  if (rc) return rc;
  B200OCL_CHECK_ARG(st->grads, "state has no gradient arena");
  B200OCL_CHECK_ARG(adam && adam->exp_avg && adam->exp_avg_sq && s, "Adam state incomplete");
  B200OCL_CHECK_ARG((adam_flags & ~B200OCL_ADAM_FOREACH) == 0, "unknown Adam flags for the EWC++ step");
  AdamCoef c;
  B200OCL_CHECK_ARG(adam_coef(*s, adam_flags, c), "unknown Adam flags");
  B200OCL_CHECK_ARG((flags & ~(B200OCL_EWC_PENALTY | B200OCL_EWC_EMA)) == 0, "unknown EWC flags");
  ArenaStep a = net_step(p, *st);
  a.m = adam->exp_avg;
  a.v = adam->exp_avg_sq;
  a.ewc = ewc;
  a.ewc_flags = flags;
  a.e = EwcScalars{up, ema_keep, ema_add};
  a.ws = workspace;
  a.penalty_out = penalty_out;
  const bool pen = flags & B200OCL_EWC_PENALTY, ema = flags & B200OCL_EWC_EMA;
  if ((rc = launch_adam_step(a, c, adam_flags & B200OCL_ADAM_FOREACH, "adam_ewc",
                             4.0 * p.n_params * (10 + (pen ? 3 : 0) + (ema ? 2 : 0)), stream))) return rc;
  return launch_pack(p, st->params, st->packed, stream);
}

}  // extern "C"
