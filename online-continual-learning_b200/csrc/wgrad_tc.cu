// wgrad_tc.cu -- weight gradient of a 3x3 stride-1 convolution on wgmma, the activation read in place from a strip (sm_90a).
//
//   dW[co][ci][kh][kw] = sum over output pixels p of  dz[p][co] * x[p + (kh-1, kw-1)][ci]
//
// The contraction runs over pixel positions.  With the zero-padded batch as a strip of positions (as in conv_tcp.cu)
//   strip position s = (img*(H+2) + yp)*(W+2) + xp,  x_strip[s] = x[img, yp-1, xp-1] (zero on the halo),
//   dz_strip[s] = dz[img, yp, xp] when yp < H and xp < W, zero otherwise,
// the sum becomes  dW[co][ci][kh][kw] = sum_s dz_strip[s][co] * x_strip[s + kh*(W+2) + kw][ci].
// Per tile of 128 positions and kernel row kh this is one GEMM  D[(kw, ci)][co] += A[(kw, ci)][s] * B[co][s]^T  with
// M = 3 x 20 (kw = 0..2 times a 20-channel slice: 60 of 64 rows), N = the block's output channels rounded up to a
// multiple of 8 (24 for 20 channels, 40 for 40 / 80 / 160), K = the 128 positions:
//   A  the x strip, one row of 20 channels per position (pitch 24 floats).  Row m of A is channel m % 20 of the strip
//      shifted by kw = m / 20 positions, so A cannot be a shared-memory descriptor (wgmma's tf32 operands are K-major
//      only); every thread loads its register fragment directly, splits it into TF32 hi / lo and feeds wgmma's
//      register-A form.  Kernel row kh moves the fragment rows by W+2 positions.
//   B  the dz block, transposed by its loaders into K-major 128-byte-swizzled tiles (hi / lo).
// fp32 grade as everywhere else: 3xTF32 (x_hi*dz_hi + x_hi*dz_lo + x_lo*dz_hi); the tensor core's accumulation
// truncates, so a chain is cut after `tpc` tiles (default 2 = 256 positions) and written out as one fp32 partial; the
// existing deterministic finalize kernel sums the partials in fixed order.  An accumulator element depends only on its
// row of A and column of B, so neither the row placement nor the N padding changes a bit of a partial.
//
// CTA = (range of chains, 20-channel slice of x, block of dz), 16 warps:
//   warps 0-7   two consumer warpgroups: warpgroup h takes every other chain of the CTA (h, h + 2, ...) whole, issues
//               its MMAs with one K step in flight and writes rows [k = (kh*3+kw)*Cin + ci][co] of the partial
//   warps 8-11  x loaders: LDG.128 of NHWC pixels with halo, plain fp32 stores
//   warps 12-15 dz loaders: one of the tile's 128 positions per thread, cvt.rna.tf32 split, transposed swizzled
//               stores, zero at halo positions and beyond the real output channels
// setmaxnreg moves registers from the loader warpgroups (96) to the consumers (160): at the launch's 128 the three
// accumulators and two fragment sets do not fit, and ptxas serialises the MMAs.
// Staging slots (dz hi / lo + x): 4 where they fit (2 per consumer warpgroup), else 2.
#include "common.cuh"
#include "umma.cuh"
#include "wgrad_tc.cuh"

namespace b200ocl {
namespace {

constexpr int WT_THREADS = 32 * 16;
constexpr int WT_PS_MAX = 4;
constexpr int WT_XP = 24;                 // floats per x row in shared memory (20 channels + 4 zeros)
constexpr size_t WT_SMEM_LIMIT = 227 * 1024 - 1024;   // the barriers are static shared memory on top

// one dz half (hi or lo) of a tile: 4 K-major [bn co][32 positions] tiles of bn 128-byte rows
__host__ __device__ constexpr int wt_dz_bytes(int bn) { return 4 * bn * 128; }

struct WtGeom {
  int wp, pp, prow, xbytes;
};
__host__ __device__ inline WtGeom wt_geom(int H, int W) {
  WtGeom g;
  g.wp = W + 2;
  g.pp = (H + 2) * (W + 2);
  g.prow = 128 + 2 * g.wp + 2;
  g.xbytes = (g.prow * WT_XP * 4 + 1023) / 1024 * 1024;
  return g;
}

__host__ __device__ inline int wt_stage_bytes(const WtGeom& G, int bn) { return 2 * wt_dz_bytes(bn) + G.xbytes; }

// A fragments of one K step for the three kernel rows: fragment rows g (x offset o0) and g + 8 (o1), positions
// p and p + 4, split into TF32 hi / lo
__device__ __forceinline__ void load_a(const float* xs, int p, int wp, int o0, int o1, uint32_t (&hi)[3][4],
                                       uint32_t (&lo)[3][4]) {
#pragma unroll
  for (int kh = 0; kh < 3; ++kh) {
    const float* r = xs + (p + kh * wp) * WT_XP;
    const float v[4] = {r[o0], r[o1], r[4 * WT_XP + o0], r[4 * WT_XP + o1]};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float h, l;
      umma::split_tf32(v[i], h, l);
      hi[kh][i] = __float_as_uint(h);
      lo[kh][i] = __float_as_uint(l);
    }
  }
}

// the nine MMAs of one K step (per kernel row: hi*hi, hi*lo, lo*hi), committed as one group
template <int BN>
__device__ __forceinline__ void issue_step(float (&acc)[3][BN / 2], const uint32_t (&hi)[3][4], const uint32_t (&lo)[3][4],
                                           uint64_t dZh, uint64_t dZl, uint32_t accumulate) {
  umma::fence();
#pragma unroll
  for (int kh = 0; kh < 3; ++kh) {
    umma::mma_tf32_rs<BN>(acc[kh], hi[kh], dZh, accumulate);
    umma::mma_tf32_rs<BN>(acc[kh], hi[kh], dZl, 1u);
    umma::mma_tf32_rs<BN>(acc[kh], lo[kh], dZh, 1u);
  }
  umma::commit();
}

// Row of A held by fragment row m: kernel column kw, channel c of the slice.  Rows 60..63 read the zero columns
// 20..23 of the kw = 2 rows and are never written out.
__device__ __forceinline__ int wt_row_kw(int m) { return min(m / WT_SLICE, 2); }

template <int BN>
__global__ void __launch_bounds__(WT_THREADS, 1) wgrad_tc_kernel(WgradTcArgs a, int tiles_m, int stages) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t full[WT_PS_MAX], empty[WT_PS_MAX];
  __shared__ int s_fail;
  constexpr int DZ_BYTES = wt_dz_bytes(BN);
  constexpr int SUB = BN * 128;             // one K-major [BN][32 positions] tile

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const WtGeom G = wt_geom(a.H, a.W);
  const int stage_bytes = wt_stage_bytes(G, BN);   // [dz hi | dz lo | x]
  const int per = stages >> 1;                     // slots per consumer warpgroup: h, h + 2
  const int sl = blockIdx.y, cb = blockIdx.z;
  const int chain0 = blockIdx.x * a.chains_per_cta;
  const int chain1 = min(a.chains, chain0 + a.chains_per_cta);
  const int k_total = 9 * a.Cin;

  if (tid == 0) {
    for (int i = 0; i < stages; ++i) {
      umma::mbar_init(&full[i], 128 + 128);
      umma::mbar_init(&empty[i], 4);
    }
    umma::fence_mbar_init();
    s_fail = 0;
  }
  __syncthreads();

  if (warp >= 8) {
    // =========================================================== loaders: tiles in the order the two consumer
    // warpgroups take them (chain pair, tile of the chain, warpgroup), each warpgroup's tiles through its own slots
    umma::reg_dealloc<96>();
    const bool dz_loader = warp >= 12;
    int pc0 = 0, pc1 = 0;
    for (int c2 = chain0; c2 < chain1; c2 += 2) {
      for (int tt = 0; tt < a.tpc; ++tt) {
#pragma unroll 1
        for (int h = 0; h < 2; ++h) {
          const int chain = c2 + h, tile = chain * a.tpc + tt;
          if (chain >= chain1 || tile >= tiles_m) continue;
          const int n = h ? pc1++ : pc0++;
          const int ps = h + 2 * (n % per);
          const uint32_t parity = (uint32_t)(((n / per) & 1) ^ 1);
          unsigned char* st = smem_raw + (size_t)ps * stage_bytes;
          if (dz_loader) {
            // ------------------------------------------------- dz: position pos, BN / 4 chunks
            const int pos = tid - 32 * 12;
            constexpr int NC = BN / 4;
            float4 v[NC];
            {
              const int sp = tile * 128 + pos;
              const int img = sp / G.pp, rem = sp - img * G.pp;
              const int yp = rem / G.wp, xp = rem - yp * G.wp;
              const bool pix = img < a.N && yp < a.H && xp < a.W;
              const float* src = a.dz + ((size_t)(img * a.H + yp) * a.W + xp) * a.Cout + cb * BN;
#pragma unroll
              for (int j = 0; j < NC; ++j) {
                v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (pix && cb * BN + 4 * j < a.Cout) v[j] = __ldg(reinterpret_cast<const float4*>(src) + j);
              }
            }
            if (!umma::mbar_wait(&empty[ps], parity)) s_fail = 1;
            float* zh = reinterpret_cast<float*>(st);
            float* zl = zh + DZ_BYTES / 4;
#pragma unroll
            for (int j = 0; j < NC; ++j) {
              const float e[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                float hv, lv;
                umma::split_tf32(e[k], hv, lv);
                // row = output channel, K = position: tile pos / 32, 16-byte chunk (pos % 32) / 4, element pos % 4
                const int off = (pos >> 5) * (SUB / 4) + umma::sw128_offset_f32(4 * j + k, (pos & 31) >> 2) + (pos & 3);
                zh[off] = hv;
                zl[off] = lv;
              }
            }
            umma::fence_proxy_async_smem();
          } else {
            // ------------------------------------------------- x: strip rows r0 + 16 i, 16-byte chunk ch (0..5)
            const int lt = tid - 32 * 8;
            const int ch = lt & 7, r0 = lt >> 3;
            const bool ch_real = ch * 4 < min(WT_SLICE, a.Cin - sl * WT_SLICE);
            const int hp = a.H + 2;
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
              if (ch_real && ri < G.prow) {
                const int y = yp - 1, x = xp - 1;
                if (img < a.N && (unsigned)y < (unsigned)a.H && (unsigned)x < (unsigned)a.W)
                  v[i] = __ldg(reinterpret_cast<const float4*>(a.x + ((size_t)(img * a.H + y) * a.W + x) * a.Cin +
                                                               sl * WT_SLICE + ch * 4));
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
            if (!umma::mbar_wait(&empty[ps], parity)) s_fail = 1;
            float* xs = reinterpret_cast<float*>(st + 2 * DZ_BYTES);
            if (ch < WT_XP / 4) {
#pragma unroll
              for (int i = 0; i < WT_LD_MAX; ++i) {
                const int ri = r0 + 16 * i;
                if (ri < G.prow) *reinterpret_cast<float4*>(xs + ri * WT_XP + ch * 4) = v[i];   // zeros beyond the channels
              }
            }
          }
          umma::mbar_arrive(&full[ps]);
        }
      }
    }
  } else {
    // =========================================================== consumers: MMA issue + partial rows
    umma::reg_alloc<160>();
    const int h = warp >> 2, wt = tid & 127;
    // fragment rows g and g + 8 of this thread -> kernel column kw, channel c -> offset kw * pitch + c in the x rows
    const int g = 16 * (warp & 3) + (lane >> 2), q = lane & 3;
    const int kw0 = wt_row_kw(g), kw1 = wt_row_kw(g + 8);
    const int o0 = kw0 * WT_XP + g - WT_SLICE * kw0, o1 = kw1 * WT_XP + g + 8 - WT_SLICE * kw1;
    const int n_valid = min(BN, a.Cout - cb * BN);
    constexpr uint32_t Z_LO = (uint32_t)DZ_BYTES >> 4;
    int pc = 0;
    for (int chain = chain0 + h; chain < chain1; chain += 2) {
      float acc[3][BN / 2];
      const int t0 = chain * a.tpc, t1 = min(tiles_m, (chain + 1) * a.tpc);
      for (int tile = t0; tile < t1; ++tile, ++pc) {
        const int ps = h + 2 * (pc % per);
        if (!umma::mbar_wait(&full[ps], (uint32_t)((pc / per) & 1))) s_fail = 1;
        const unsigned char* st = smem_raw + (size_t)ps * stage_bytes;
        const float* xs = reinterpret_cast<const float*>(st + 2 * DZ_BYTES);
        const uint64_t dZ0 = umma::make_smem_desc_sw128(umma::smem_u32(st));
        // B of K step ks: tile ks / 4, 32 bytes per K step inside it (16-byte units)
        auto dz_desc = [&](int ks) { return dZ0 + (uint64_t)(((ks >> 2) * SUB + (ks & 3) * 32) >> 4); };
        // Two fragment sets: step ks + 1 is issued while step ks is in flight; wait_group 1 retires the older step
        // before its fragments are reloaded.  The MMAs of every accumulator keep their order (steps 0..15).
        uint32_t ah[2][3][4], al[2][3][4];
        load_a(xs, q, G.wp, o0, o1, ah[0], al[0]);
#pragma unroll 1
        for (int ks = 0; ks < 16; ks += 2) {
          issue_step<BN>(acc, ah[0], al[0], dz_desc(ks), dz_desc(ks) + Z_LO, (tile == t0 && ks == 0) ? 0u : 1u);
          umma::wait<1>();
          load_a(xs, (ks + 1) * 8 + q, G.wp, o0, o1, ah[1], al[1]);
          issue_step<BN>(acc, ah[1], al[1], dz_desc(ks + 1), dz_desc(ks + 1) + Z_LO, 1u);
          umma::wait<1>();
          // the last pass reloads step 15 (unused): keeps the loop free of a branch between the MMA groups
          load_a(xs, min(ks + 2, 15) * 8 + q, G.wp, o0, o1, ah[0], al[0]);
        }
        umma::wait<0>();
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) umma::fence_regs(acc[kh]);
        if (lane == 0) umma::mbar_arrive(&empty[ps]);
      }
      // ---- the chain's partial: rows (kh*3 + kw)*Cin + ci, the real output channels of this block
#pragma unroll
      for (int i = 0; i < BN / 2; i += 2) {
        const int m = umma::frag_row(wt, i), co = umma::frag_col(wt, i);
        const int kwi = wt_row_kw(m), c = m - WT_SLICE * kwi, ci = sl * WT_SLICE + c;
        if (c < WT_SLICE && ci < a.Cin && co < n_valid) {
#pragma unroll
          for (int kh = 0; kh < 3; ++kh) {
            float* dst = a.part + ((size_t)chain * k_total + (size_t)(kh * 3 + kwi) * a.Cin + ci) * a.Cout + cb * BN + co;
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

template <int BN>
int launch_bn(const WgradTcArgs& a, const WgradTcCfg& g, cudaStream_t stream) {
  const WtGeom G = wt_geom(a.H, a.W);
  const size_t stage = (size_t)wt_stage_bytes(G, BN);
  const int stages = 4 * stage + 1024 <= WT_SMEM_LIMIT ? 4 : 2;
  const size_t smem = stages * stage + 1024;
  B200OCL_CUDA(raise_smem_limit<wgrad_tc_kernel<BN>>(smem));
  const double M = (double)a.N * a.H * a.W;
  B200OCL_PROF("wgrad_tc", 2.0 * M * 9.0 * a.Cin * a.Cout, stream);
  wgrad_tc_kernel<BN><<<dim3(g.ctas_x, g.slices, g.cout_blocks), WT_THREADS, smem, stream>>>(a, g.tiles, stages);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

}  // namespace

int launch_wgrad_tc(const WgradTcArgs& a, const WgradTcCfg& g, cudaStream_t stream) {
  switch (g.bn) {
    case 8: return launch_bn<8>(a, g, stream);
    case 16: return launch_bn<16>(a, g, stream);
    case 24: return launch_bn<24>(a, g, stream);
    case 32: return launch_bn<32>(a, g, stream);
    case 40: return launch_bn<40>(a, g, stream);
  }
  set_error("launch_wgrad_tc: no kernel for a %d-channel output block", g.bn);
  return B200OCL_EUNSUPPORTED;
}

}  // namespace b200ocl

extern "C" size_t b200ocl_wgrad_tc_selftest_workspace_bytes(int N, int H, int W, int cin, int cout) {
  using namespace b200ocl;
  if (N < 1 || H < 1 || W < 1 || cin < 1 || cout < 1) return 0;
  const WgradTcCfg g = wgrad_tc_cfg(N, H, W, 3, 1, 1, cin, cout, sm_count());
  if (!g.eligible) return 0;
  return align_up((size_t)g.chains * 9 * cin * cout * sizeof(float), 256);
}

extern "C" int b200ocl_wgrad_tc_selftest_geom(int N, int H, int W, int cin, int cout, int sms, b200ocl_wgrad_tc_geom* out) {
  using namespace b200ocl;
  B200OCL_CHECK_ARG(out && N >= 1 && H >= 1 && W >= 1 && cin >= 1 && cout >= 1 && sms >= 0, "null pointer / bad shape");
  if (sms == 0) sms = sm_count();
  const WgradTcCfg g = wgrad_tc_cfg(N, H, W, 3, 1, 1, cin, cout, sms);
  *out = b200ocl_wgrad_tc_geom{};
  out->eligible = g.eligible;
  out->sms = sms;
  if (!g.eligible) return B200OCL_OK;
  out->slices = g.slices; out->cout_blocks = g.cout_blocks; out->bn = g.bn;
  out->tiles = g.tiles; out->tpc = g.tpc; out->chains = g.chains;
  out->chains_per_cta = g.chains_per_cta; out->ctas_x = g.ctas_x;
  out->sm_share = sms / (g.slices * g.cout_blocks);
  return B200OCL_OK;
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
