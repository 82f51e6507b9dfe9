// conv_tc.cu -- 3x3 stride-1 convolution on the Hopper tensor cores (wgmma, sm_90a).
//
// Implicit GEMM  D[128 pixels, NT channels] += A[128, 32] * B[NT, 32]^T  per K block of 32 (tap, cin)
// values, tf32 inputs with fp32 accumulators in registers (one warpgroup, the 128-row tile as two
// m64 halves).  fp32 accuracy is kept with the 3xTF32 split (A_hi*B_hi + A_hi*B_lo + A_lo*B_hi, both
// halves exactly representable in TF32) AND by promoting every K block: the tensor core's own
// accumulation truncates, so each K block accumulates its 12 MMAs into a fresh register fragment that
// the threads then add into the fp32 sum with round-to-nearest.  The MMAs of block kb run while the
// operands of block kb+1 are staged into the other of two shared-memory stages.
//
//   A  activations, NHWC fp32 in HBM; thread t owns pixel t of the tile, gathers its 8 x 16-byte
//      chunks of the K block (zero outside the image / beyond K), splits them and writes the two
//      128-byte-swizzled K-major tiles the MMA reads (no im2col in HBM);
//   B  weights, pre-split and pre-swizzled tile images written by tc_pack_kernel (net_fwd.cu):
//      a byte copy with cp.async;
//   D  registers; after the last K block the fragments go through shared memory so that thread t
//      holds pixel row t for the epilogue.
// Epilogues as in conv.cu: folded eval BN (+ReLU, +residual), raw store + deterministic fp64 batch
// statistics for training, raw / accumulate for the flipped stride-1 data gradient.
#include "conv.cuh"
#include "umma.cuh"

namespace b200ocl {
namespace {

constexpr int TC_THREADS = 128;
constexpr int A_TILE = 128 * 32;  // floats

// acc += tmp for one 64-row half of the tile (fragment layout of umma.cuh)
template <int R>
__device__ __forceinline__ void promote(float (&acc)[R], const float (&tmp)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) acc[i] += tmp[i];
}

template <int NT>
__device__ __forceinline__ void issue_kblock(float (&d)[2][NT / 2], const float* sAh, const float* sAl, const float* sB) {
  constexpr int B_TILE = NT * 32;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint64_t dAh = umma::make_smem_desc_sw128(umma::smem_u32(sAh + h * 64 * 32));
    const uint64_t dAl = umma::make_smem_desc_sw128(umma::smem_u32(sAl + h * 64 * 32));
    const uint64_t dBh = umma::make_smem_desc_sw128(umma::smem_u32(sB));
    const uint64_t dBl = umma::make_smem_desc_sw128(umma::smem_u32(sB + B_TILE));
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t adv = (uint64_t)(k * 2);  // 32 bytes per K step, in 16-byte units
      umma::mma_tf32_ss<NT>(d[h], dAh + adv, dBh + adv, k > 0 ? 1u : 0u);
      umma::mma_tf32_ss<NT>(d[h], dAh + adv, dBl + adv, 1u);
      umma::mma_tf32_ss<NT>(d[h], dAl + adv, dBh + adv, 1u);
    }
  }
}

template <int NT>
__global__ void __launch_bounds__(TC_THREADS) conv_tc_kernel(ConvArgs a) {
  constexpr int B_TILE = NT * 32;
  constexpr int STAGE_F = 2 * A_TILE + 2 * B_TILE;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  float* stage0 = reinterpret_cast<float*>(smem_raw);
  __shared__ bool is_last;

  const int tid = threadIdx.x;
  const int bn = a.tc_bn;
  const int n0 = blockIdx.y * bn;
  const int KB = a.tc_kb;
  const int m = blockIdx.x * 128 + tid;
  const bool valid = m < a.M;
  const int hw = a.Hout * a.Wout;
  const int img = valid ? m / hw : 0;
  const int rem = valid ? m - img * hw : 0;
  const int py = rem / a.Wout, px = rem - py * a.Wout;
  const float* wimg = a.w_tc + (size_t)blockIdx.y * KB * 2 * B_TILE;

  float accf[2][NT / 2], tmp[2][NT / 2];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) accf[h][i] = 0.f;

  // running (tap, channel) position of this thread's next 16-byte chunk and the tap's source pointer
  int tap = 0, ci = 0;
  const float* tap_src = nullptr;
  auto set_tap = [&]() {
    const int kh = tap / 3, kw = tap - kh * 3;
    const int iy = py + kh - 1, ix = px + kw - 1;
    const bool ok = valid && tap < 9 && (unsigned)iy < (unsigned)a.Hin && (unsigned)ix < (unsigned)a.Win;
    tap_src = ok ? a.in + ((size_t)(img * a.Hin + iy) * a.Win + ix) * a.CK : nullptr;
  };
  set_tap();

  for (int kb = 0; kb < KB; ++kb) {
    const int s = kb & 1;
    float* sAh = stage0 + s * STAGE_F;
    float* sAl = sAh + A_TILE;
    float* sB = sAl + A_TILE;  // [hi | lo], contiguous like the image
    // ---- B: byte copy of the pre-swizzled hi/lo tiles of this K block
    const float* bsrc = wimg + (size_t)kb * 2 * B_TILE;
#pragma unroll
    for (int i = 0; i < (2 * B_TILE / 4) / TC_THREADS; ++i)
      cp_async16(sB + (tid + i * TC_THREADS) * 4, bsrc + (tid + i * TC_THREADS) * 4);
    cp_async_commit();
    // ---- A: gather this pixel's 8 chunks (all loads first, then split + store)
    float4 v[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      v[c] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (tap_src != nullptr) v[c] = __ldg(reinterpret_cast<const float4*>(tap_src + ci));
      ci += 4;
      if (ci == a.CK) {
        ci = 0;
        ++tap;
        set_tap();
      }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      float4 h, l;
      umma::split_tf32(v[c].x, h.x, l.x); umma::split_tf32(v[c].y, h.y, l.y);
      umma::split_tf32(v[c].z, h.z, l.z); umma::split_tf32(v[c].w, h.w, l.w);
      const int off = umma::sw128_offset_f32(tid, c);
      *reinterpret_cast<float4*>(sAh + off) = h;
      *reinterpret_cast<float4*>(sAl + off) = l;
    }
    cp_async_wait<0>();
    umma::fence_proxy_async_smem();
    __syncthreads();
    // ---- promote the previous K block (its MMAs ran while this block was staged), then issue this one
    if (kb > 0) {
      umma::wait<0>();
      umma::fence_regs(tmp[0]);
      umma::fence_regs(tmp[1]);
      promote(accf[0], tmp[0]);
      promote(accf[1], tmp[1]);
    }
    umma::fence();
    issue_kblock<NT>(tmp, sAh, sAl, sB);
    umma::commit();
  }
  umma::wait<0>();
  umma::fence_regs(tmp[0]);
  umma::fence_regs(tmp[1]);
  promote(accf[0], tmp[0]);
  promote(accf[1], tmp[1]);

  // ---- fragments -> one pixel row per thread through shared memory (the staging buffers are free)
  __syncthreads();
  float* s_acc = stage0;  // [128][NT + 1]
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < NT / 2; ++i)
      s_acc[(64 * h + umma::frag_row(tid, i)) * (NT + 1) + umma::frag_col(tid, i)] = accf[h][i];
  __syncthreads();
  float acc[NT];
#pragma unroll
  for (int c = 0; c < NT; ++c) acc[c] = s_acc[tid * (NT + 1) + c];

  // ------------------------------------------------------------------ epilogue (thread = pixel row)
  if (a.mode == CONV_EVAL) {
    if (valid) {
      float* o = a.out + (size_t)m * a.CN + n0;
      const float* rs = a.residual ? a.residual + (size_t)m * a.CN + n0 : nullptr;
#pragma unroll
      for (int c0 = 0; c0 < NT; c0 += 4) {   // compile-time indices into acc[]; tiles are 20/40/80 wide
        if (c0 >= bn) break;
        float r[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = n0 + c0 + j;
          const float inv = 1.0f / sqrtf(a.rvar[c] + a.eps);
          r[j] = (acc[c0 + j] - a.rmean[c]) * (inv * a.gamma[c]) + a.beta[c];
        }
        if (rs) {
          const float4 r4 = *reinterpret_cast<const float4*>(rs + c0);
          r[0] += r4.x; r[1] += r4.y; r[2] += r4.z; r[3] += r4.w;
        }
        if (a.relu) {
#pragma unroll
          for (int j = 0; j < 4; ++j) r[j] = fmaxf(r[j], 0.f);
        }
        *reinterpret_cast<float4*>(o + c0) = make_float4(r[0], r[1], r[2], r[3]);
      }
    }
  } else {
    if (valid) {
      float* o = a.out + (size_t)m * a.CN + n0;
#pragma unroll
      for (int c0 = 0; c0 < NT; c0 += 4) {
        if (c0 >= bn) break;
        float4 r = make_float4(acc[c0], acc[c0 + 1], acc[c0 + 2], acc[c0 + 3]);
        if (a.mode == CONV_ACCUM) {
          const float4 old = *reinterpret_cast<const float4*>(o + c0);
          r.x += old.x; r.y += old.y; r.z += old.z; r.w += old.w;
        }
        *reinterpret_cast<float4*>(o + c0) = r;
      }
    }
    if (a.mode == CONV_TRAIN) {
      // batch statistics: transpose through shared memory, one thread per channel sums its 128 rows in
      // fp64 in row order (rows beyond M hold exact zeros), then partial per CTA + last-CTA finalize
      __syncthreads();  // staging buffers are free
      float* s_t = stage0;  // [128][bn + 1]
#pragma unroll
      for (int c = 0; c < NT; ++c)
        if (c < bn) s_t[tid * (bn + 1) + c] = acc[c];
      __syncthreads();
      if (tid < bn) {
        double S = 0.0, Q = 0.0;
        for (int r = 0; r < 128; ++r) {
          const double x = (double)s_t[r * (bn + 1) + tid];
          S += x;
          Q += x * x;
        }
        double* dst = a.stat_part + ((size_t)blockIdx.x * a.CN + n0 + tid) * 2;
        dst[0] = S;
        dst[1] = Q;
      }
      __threadfence();
      __syncthreads();
      if (tid == 0) is_last = (atomicAdd(a.counter + blockIdx.y, 1u) == gridDim.x - 1);
      __syncthreads();
      if (is_last) {
        __threadfence();
        const int groups = TC_THREADS / bn;          // 6, 3 or 1 partial-subsets per channel
        const int ch = tid % bn, grp = tid / bn;
        double* s_fin = reinterpret_cast<double*>(stage0);   // [groups][bn][2]
        __syncthreads();
        if (grp < groups) {
          double s4[4] = {0.0, 0.0, 0.0, 0.0}, q4[4] = {0.0, 0.0, 0.0, 0.0};
          unsigned int b = grp;
          for (; b + 3 * groups < gridDim.x; b += 4 * groups) {
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const double2 pv = __ldcg(reinterpret_cast<const double2*>(a.stat_part + ((size_t)(b + u * groups) * a.CN + n0 + ch) * 2));
              s4[u] += pv.x;
              q4[u] += pv.y;
            }
          }
          for (; b < gridDim.x; b += groups) {
            const double2 pv = __ldcg(reinterpret_cast<const double2*>(a.stat_part + ((size_t)b * a.CN + n0 + ch) * 2));
            s4[0] += pv.x;
            q4[0] += pv.y;
          }
          s_fin[(grp * bn + ch) * 2 + 0] = (s4[0] + s4[1]) + (s4[2] + s4[3]);
          s_fin[(grp * bn + ch) * 2 + 1] = (q4[0] + q4[1]) + (q4[2] + q4[3]);
        }
        __syncthreads();
        if (tid < bn) {
          double S = 0.0, Q = 0.0;
          for (int g = 0; g < groups; ++g) {
            S += s_fin[(g * bn + tid) * 2 + 0];
            Q += s_fin[(g * bn + tid) * 2 + 1];
          }
          bn_finalize(a, n0 + tid, S, Q);
        }
      }
    }
  }
}

template <int NT>
int launch_tc(const ConvArgs& a, const ConvPlan& pl, cudaStream_t stream) {
  constexpr size_t smem = (size_t)2 * (2 * A_TILE + 2 * NT * 32) * sizeof(float) + 1024;
  B200OCL_CUDA(raise_smem_limit<conv_tc_kernel<NT>>(smem));
  dim3 grid(pl.grid_x, pl.grid_y);
  B200OCL_PROF(a.flip ? "conv_tc_dgrad" : (a.mode == CONV_EVAL ? "conv_tc_eval" : "conv_tc_train"),
               2.0 * a.M * (double)a.CN * a.CK * 9.0, stream);
  conv_tc_kernel<NT><<<grid, TC_THREADS, smem, stream>>>(a);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

}  // namespace

bool conv_tc_eligible(const ConvArgs& a, int sms) {
  if (!a.w_tc || a.ks != 3 || a.stride != 1 || a.transposed || a.CK % 20 != 0) return false;
  if (a.Hin != a.Hout || a.Win != a.Wout) return false;
  // enough 128-pixel tiles to occupy a good part of the machine; small problems stay on the fp32 kernels
  const long ctas = (long)((a.M + 127) / 128) * (a.CN / a.tc_bn);
  if (ctas < sms / 4) return false;
  // 20 -> 20 channels (layer 1): K = 180 leaves the tensor-core kernel dominated by its per-tile gather, so the
  // fp32 patch kernel takes the layer once there are more than two tiles per SM.
  if (a.CK == 20 && a.CN == 20 && ctas > 2L * sms) return false;
  return true;
}

int launch_conv_tc(const ConvArgs& a, const ConvPlan& pl, cudaStream_t stream) {
  if (pl.nt == 32) return launch_tc<32>(a, pl, stream);
  if (pl.nt == 48) return launch_tc<48>(a, pl, stream);
  return launch_tc<80>(a, pl, stream);
}

}  // namespace b200ocl
