// wgrad_tc.cu -- weight gradient of a 3x3 stride-1 convolution on wgmma, the activation read in place from a strip (sm_90a).
//
//   dW[co][ci][kh][kw] = sum over output pixels p of  dz[p][co] * x[p + (kh-1, kw-1)][ci]
//
// The contraction runs over pixel positions.  With the zero-padded batch as a strip of positions (as in conv_tcp.cu)
//   strip position s = (img*(H+2) + yp)*(W+2) + xp,  x_strip[s] = x[img, yp-1, xp-1] (zero on the halo),
//   dz_strip[s] = dz[img, yp, xp] when yp < H and xp < W, zero otherwise,
// the sum becomes  dW[co][ci][kh][kw] = sum_s dz_strip[s][co] * x_strip[s + kh*(W+2) + kw][ci].
// Per tile of 128 positions and kernel row kh this is one GEMM  D[(kw, ci)][co] += A[(kw, ci)][s] * B[co][s]^T  with
// M = 4 x 32 (kw = 0..2, the fourth block a by-product), N = 32 output channels, K = the 128 positions:
//   A  the x strip, one row of 32 channels per position (padded to 40 floats: conflict-free fragment loads).  Row m of
//      A is the strip shifted by kw = m / 32 positions, so A cannot be a shared-memory descriptor (wgmma's tf32 operands
//      are K-major only); every thread loads its register fragment directly, splits it into TF32 hi / lo and feeds
//      wgmma's register-A form.  Kernel row kh moves the fragment rows by W+2 positions.
//   B  the dz tile of one 32-channel block, transposed by its loaders into K-major 128-byte-swizzled tiles (hi / lo).
// fp32 grade as everywhere else: 3xTF32 (x_hi*dz_hi + x_hi*dz_lo + x_lo*dz_hi); the tensor core's accumulation
// truncates, so a chain is cut after `tpc` tiles (default 2 = 256 positions) and written out as one fp32 partial; the
// existing deterministic finalize kernel sums the partials in fixed order.
//
// CTA = (range of chains, 32-channel slice of x, 32-channel block of dz), 14 warps:
//   warps 0-7   two consumer warpgroups: warpgroup h owns rows 64h .. 64h+63 of D (kw blocks 2h, 2h+1) for the three kh,
//               issues their MMAs and writes rows [k = (kh*3+kw)*Cin + ci][32 co] of the partial
//   warps 8-11  x loaders: coalesced LDG.128 of NHWC pixels with halo, plain fp32 stores
//   warps 12-13 dz loaders: the tile's 128 positions of one channel block, cvt.rna.tf32 split, transposed swizzled
//               stores, zero at halo / by-product positions
// Two staging slots (dz hi / lo + x).
#include "common.cuh"
#include "umma.cuh"
#include "wgrad_tc.cuh"

namespace b200ocl {
namespace {

constexpr int WT_THREADS = 32 * 14;
constexpr int WT_PS = 2;
constexpr int WT_XP = 40;                 // floats per x row in shared memory (32 channels + 8: conflict-free fragments)
constexpr int WT_DZ_BYTES = 128 * 128;    // one dz half (hi or lo) of a tile: 4 K-major [32 co][32 positions] tiles

struct WtGeom {
  int wp, pp, prow, xbytes;
};
__host__ __device__ inline WtGeom wt_geom(int H, int W) {
  WtGeom g;
  g.wp = W + 2;
  g.pp = (H + 2) * (W + 2);
  g.prow = 128 + 2 * g.wp + 2;
  // one row beyond the staged ones: the by-product block (kw = 3) of the last K step reads it
  g.xbytes = ((g.prow + 1) * WT_XP * 4 + 1023) / 1024 * 1024;
  return g;
}

// A fragment of one K step: x rows r and r + 4 (positions q, q + 4 of the step), channels c and c + 8
__device__ __forceinline__ void load_a(const float* xs, int r, int c, uint32_t (&hi)[4], uint32_t (&lo)[4]) {
  const float v[4] = {xs[r * WT_XP + c], xs[r * WT_XP + c + 8], xs[(r + 4) * WT_XP + c], xs[(r + 4) * WT_XP + c + 8]};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float h, l;
    umma::split_tf32(v[i], h, l);
    hi[i] = __float_as_uint(h);
    lo[i] = __float_as_uint(l);
  }
}

__global__ void __launch_bounds__(WT_THREADS, 1) wgrad_tc_kernel(WgradTcArgs a, int tiles_m) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t full[WT_PS], empty[WT_PS];
  __shared__ int s_fail;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const WtGeom G = wt_geom(a.H, a.W);
  const int stage_bytes = 2 * WT_DZ_BYTES + G.xbytes;   // [dz hi | dz lo | x]
  const int sl = blockIdx.y, cb = blockIdx.z;
  const int chain0 = blockIdx.x * a.chains_per_cta;
  const int chain1 = min(a.chains, chain0 + a.chains_per_cta);
  const int k_total = 9 * a.Cin;

  if (tid == 0) {
    for (int i = 0; i < WT_PS; ++i) {
      umma::mbar_init(&full[i], 128 + 64);
      umma::mbar_init(&empty[i], 8);
    }
    umma::fence_mbar_init();
    s_fail = 0;
  }
  __syncthreads();

  if (warp >= 12) {
    // =========================================================== dz loaders (64 threads)
    const int lt = tid - 32 * 12;
    const int ch = lt & 7, r0 = lt >> 3;                         // chunk, first row; rows r0 + 8 i
    const bool ch_real = cb * 32 + ch * 4 < a.Cout;
    const int hp = a.H + 2;
    int pc = 0;
    for (int chain = chain0; chain < chain1; ++chain) {
      const int t1 = min(tiles_m, (chain + 1) * a.tpc);
      for (int tile = chain * a.tpc; tile < t1; ++tile, ++pc) {
        float4 v[16];
        int img, yp, xp;
        {
          const int sp = tile * 128 + r0;
          img = sp / G.pp;
          const int rem = sp - img * G.pp;
          yp = rem / G.wp;
          xp = rem - yp * G.wp;
        }
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ch_real && img < a.N && yp < a.H && xp < a.W)
            v[i] = __ldg(reinterpret_cast<const float4*>(a.dz + ((size_t)(img * a.H + yp) * a.W + xp) * a.Cout + cb * 32) + ch);
          xp += 8;
          while (xp >= G.wp) {
            xp -= G.wp;
            if (++yp == hp) {
              yp = 0;
              ++img;
            }
          }
        }
        const int ps = pc % WT_PS;
        if (!umma::mbar_wait(&empty[ps], (uint32_t)(((pc / WT_PS) & 1) ^ 1))) s_fail = 1;
        float* zh = reinterpret_cast<float*>(smem_raw + (size_t)ps * stage_bytes);
        float* zl = zh + WT_DZ_BYTES / 4;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int pos = r0 + 8 * i;
          const float e[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float h, l;
            umma::split_tf32(e[j], h, l);
            // row = output channel, K = position: tile pos / 32, 16-byte chunk (pos % 32) / 4, element pos % 4
            const int off = (pos >> 5) * 1024 + umma::sw128_offset_f32(ch * 4 + j, (pos & 31) >> 2) + (pos & 3);
            zh[off] = h;
            zl[off] = l;
          }
        }
        umma::fence_proxy_async_smem();
        umma::mbar_arrive(&full[ps]);
      }
    }
  } else if (warp >= 8) {
    // =========================================================== x loaders (128 threads)
    const int lt = tid - 32 * 8;
    const int ch = lt & 7, r0 = lt >> 3;                         // rows r0 + 16 i
    const int ch_valid = min(32, a.Cin - sl * 32);
    const bool ch_real = ch * 4 < ch_valid;
    const int nrow = G.prow;
    const int hp = a.H + 2;
    int pc = 0;
    for (int chain = chain0; chain < chain1; ++chain) {
      const int t1 = min(tiles_m, (chain + 1) * a.tpc);
      for (int tile = chain * a.tpc; tile < t1; ++tile, ++pc) {
        float4 v[WT_LD_MAX];
        int img, yp, xp;
        {
          const int sp = tile * 128 + r0;
          img = sp / G.pp;
          const int rem = sp - img * G.pp;
          yp = rem / G.wp;
          xp = rem - yp * G.wp;
        }
#pragma unroll
        for (int i = 0; i < WT_LD_MAX; ++i) {
          v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
          const int ri = r0 + 16 * i;
          if (ch_real && ri < nrow) {
            const int y = yp - 1, x = xp - 1;
            if (img < a.N && (unsigned)y < (unsigned)a.H && (unsigned)x < (unsigned)a.W)
              v[i] = __ldg(reinterpret_cast<const float4*>(a.x + ((size_t)(img * a.H + y) * a.W + x) * a.Cin + sl * 32) + ch);
          }
          xp += 16;
          while (xp >= G.wp) {
            xp -= G.wp;
            if (++yp == hp) {
              yp = 0;
              ++img;
            }
          }
        }
        const int ps = pc % WT_PS;
        if (!umma::mbar_wait(&empty[ps], (uint32_t)(((pc / WT_PS) & 1) ^ 1))) s_fail = 1;
        float* xs = reinterpret_cast<float*>(smem_raw + (size_t)ps * stage_bytes + 2 * WT_DZ_BYTES);
#pragma unroll
        for (int i = 0; i < WT_LD_MAX; ++i) {
          const int ri = r0 + 16 * i;
          if (ri < nrow) *reinterpret_cast<float4*>(xs + ri * WT_XP + ch * 4) = v[i];   // zeros beyond the channels
        }
        umma::mbar_arrive(&full[ps]);
      }
    }
  } else {
    // =========================================================== consumers: MMA issue + partial rows
    const int h = warp >> 2, wt = tid & 127;
    // fragment rows of this thread: m = 64 h + 16 (warp % 4) + lane / 4 (+ 8) -> kernel column kw, channel c (+ 8)
    const int m0 = 64 * h + 16 * (warp & 3) + (lane >> 2);
    const int kw = m0 >> 5, c = m0 & 31, q = lane & 3;
    const int n_valid = min(32, a.Cout - cb * 32);
    int pc = 0;
    for (int chain = chain0; chain < chain1; ++chain) {
      float acc[3][16];
      const int t0 = chain * a.tpc, t1 = min(tiles_m, (chain + 1) * a.tpc);
      for (int tile = t0; tile < t1; ++tile, ++pc) {
        const int ps = pc % WT_PS;
        if (!umma::mbar_wait(&full[ps], (uint32_t)((pc / WT_PS) & 1))) s_fail = 1;
        const unsigned char* st = smem_raw + (size_t)ps * stage_bytes;
        const float* xs = reinterpret_cast<const float*>(st + 2 * WT_DZ_BYTES);
        const uint64_t dZ0 = umma::make_smem_desc_sw128(umma::smem_u32(st));
        constexpr uint32_t Z_LO = (uint32_t)WT_DZ_BYTES >> 4;
#pragma unroll 1
        for (int ks = 0; ks < 16; ++ks) {
          // B: 4 KB tile ks / 4, 32 bytes per K step inside it (16-byte units)
          const uint64_t dZh = dZ0 + (uint64_t)((ks >> 2) * 256 + (ks & 3) * 2), dZl = dZh + Z_LO;
          uint32_t ah[3][4], al[3][4];
#pragma unroll
          for (int kh = 0; kh < 3; ++kh) load_a(xs, ks * 8 + q + kh * G.wp + kw, c, ah[kh], al[kh]);
          const uint32_t accumulate = (tile == t0 && ks == 0) ? 0u : 1u;
          umma::fence();
#pragma unroll
          for (int kh = 0; kh < 3; ++kh) {
            umma::mma_tf32_rs<32>(acc[kh], ah[kh], dZh, accumulate);
            umma::mma_tf32_rs<32>(acc[kh], ah[kh], dZl, 1u);
            umma::mma_tf32_rs<32>(acc[kh], al[kh], dZh, 1u);
          }
          umma::commit();
          umma::wait<0>();
        }
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) umma::fence_regs(acc[kh]);
        if (lane == 0) umma::mbar_arrive(&empty[ps]);
      }
      // ---- the chain's partial: rows (kh*3 + kw)*Cin + ci, the 32 output channels of this block
#pragma unroll
      for (int i = 0; i < 16; i += 2) {
        const int m = 64 * h + umma::frag_row(wt, i), co = umma::frag_col(wt, i);
        const int kwi = m >> 5, ci = sl * 32 + (m & 31);
        if (kwi < 3 && ci < a.Cin && co < n_valid) {
#pragma unroll
          for (int kh = 0; kh < 3; ++kh) {
            float* dst = a.part + ((size_t)chain * k_total + (size_t)(kh * 3 + kwi) * a.Cin + ci) * a.Cout + cb * 32 + co;
            *reinterpret_cast<float2*>(dst) = make_float2(acc[kh][i], acc[kh][i + 1]);
          }
        }
      }
    }
  }
  __syncthreads();
  // a timed-out barrier (must never happen) poisons the partials instead of hanging the GPU
  if (s_fail && tid == 0) a.part[0] = __int_as_float(0x7fc00000);
}

// selftest helper: dW[co][ci][kh][kw] = sum over chains of part[chain][(kh*3+kw)*Cin + ci][co]
__global__ void wgrad_tc_reduce_kernel(const float* __restrict__ part, int chains, int Cin, int Cout, float* __restrict__ dw) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const int total = 9 * Cin * Cout;
  if (e >= total) return;
  const int k = e / Cout, co = e - k * Cout;
  const int tap = k / Cin, ci = k - tap * Cin;
  double s = 0.0;
  for (int sp = 0; sp < chains; ++sp) s += (double)part[(size_t)sp * total + e];
  dw[((size_t)co * Cin + ci) * 9 + tap] = (float)s;
}

}  // namespace

int launch_wgrad_tc(const WgradTcArgs& a, const WgradTcCfg& g, cudaStream_t stream) {
  const WtGeom G = wt_geom(a.H, a.W);
  const size_t smem = (size_t)WT_PS * (2 * WT_DZ_BYTES + (size_t)G.xbytes) + 1024;
  B200OCL_CUDA(raise_smem_limit<wgrad_tc_kernel>(smem));
  const double M = (double)a.N * a.H * a.W;
  B200OCL_PROF("wgrad_tc", 2.0 * M * 9.0 * a.Cin * a.Cout, stream);
  wgrad_tc_kernel<<<dim3(g.ctas_x, g.slices, g.cout_blocks), WT_THREADS, smem, stream>>>(a, g.tiles);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

}  // namespace b200ocl

extern "C" size_t b200ocl_wgrad_tc_selftest_workspace_bytes(int N, int H, int W, int cin, int cout) {
  using namespace b200ocl;
  if (N < 1 || H < 1 || W < 1 || cin < 1 || cout < 1) return 0;
  const WgradTcCfg g = wgrad_tc_cfg(N, H, W, 3, 1, 1, cin, cout, sm_count());
  if (!g.eligible) return 0;
  return align_up((size_t)g.chains * 9 * cin * cout * sizeof(float), 256);
}

extern "C" int b200ocl_wgrad_tc_selftest(const float* x, const float* dz, float* dw_oihw, int N, int H, int W, int cin, int cout,
                                         void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(x && dz && dw_oihw && N >= 1, "null pointer / empty batch");
  const WgradTcCfg g = wgrad_tc_cfg(N, H, W, 3, 1, 1, cin, cout, sm_count());
  if (!g.eligible) {
    set_error("b200ocl_wgrad_tc_selftest: geometry not covered (3x3 stride 1, W <= 37, channels %% 4 == 0)");
    return B200OCL_EUNSUPPORTED;
  }
  int rc = check_workspace("b200ocl_wgrad_tc_selftest", workspace, workspace_bytes,
                           b200ocl_wgrad_tc_selftest_workspace_bytes(N, H, W, cin, cout));
  if (rc) return rc;
  WgradTcArgs a{};
  a.x = x; a.dz = dz; a.part = static_cast<float*>(workspace);
  a.N = N; a.H = H; a.W = W; a.Cin = cin; a.Cout = cout;
  a.tpc = g.tpc; a.chains = g.chains; a.chains_per_cta = g.chains_per_cta;
  if ((rc = launch_wgrad_tc(a, g, stream))) return rc;
  const int total = 9 * cin * cout;
  wgrad_tc_reduce_kernel<<<(total + 255) / 256, 256, 0, stream>>>(a.part, g.chains, cin, cout, dw_oihw);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}
