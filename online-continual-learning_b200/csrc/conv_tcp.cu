// conv_tcp.cu -- 3x3 stride-1 convolution on wgmma fed IN PLACE from a halo patch (sm_90a).
//
// conv_tc.cu builds an im2col tile per K block: every output pixel re-gathers, re-splits and re-stores
// its input 9 times, and that staging chain -- not the tensor core -- is what a K block costs.  Here the
// input patch of a tile (with its halo) is staged ONCE per 32-channel slice as two 128-byte-swizzled
// arrays (TF32 hi / lo) of one 128-byte row per patch pixel, and the A operand of every tap is that
// same array read through a shifted shared-memory descriptor:
//
//   strip  = the input of the whole batch with a one-position zero halo shared between neighbours, row-major:
//            row length W+1, image size (H+1)*(W+1); pixel (img, y, x) sits at position
//            s = img*(H+1)*(W+1) + (y+1)*(W+1) + (x+1), one 128-byte row (32 channel slots) per position.
//            Strip row 0 and strip column 0 of every image hold zeros: they are the neighbours above pixel row 0
//            and left of pixel column 0; the right neighbour of pixel column W-1 is the next strip row's column 0,
//            and the row below pixel row H-1 is the next image's strip row 0 (or the zero tail past the last image).
//   tile   = 128 consecutive strip positions = the 128 rows of an MMA tile; row i at s_i = img*(H+1)*(W+1) +
//            y*(W+1) + x is the output pixel (img, y, x) when y < H and x < W, a discarded by-product otherwise
//   tap (kh, kw) of row i reads strip position  s_i + kh*(W+1) + kw  -> one descriptor per tap whose start
//            address is the patch base + (kh*(W+1) + kw) * 128 bytes; rows stay consecutive, so the 8-row
//            groups are the standard 1024 bytes apart.
// A stage therefore holds 128 + 2*(W+1) + 2 strip rows.  Any H, W works; the share of useful rows is
// H*W / ((H+1)*(W+1)): 94 % at 32x32, 89 % at 16x16, 79 % at 8x8, 64 % at 4x4 -- tensor-core time is not
// what bounds the kernel, and no im2col or per-shape tiling is needed.
//
// The hardware applies the 128-byte swizzle to absolute address bits, so a window that starts at any
// 128-byte row of a patch stored with "chunk ^= row & 7" reads back exactly (b200ocl_selftest_umma_window).
//
// Per tile and slice the tensor core runs 9 taps x ceil(channels/8) K steps x 3 MMAs (3xTF32:
// hi*hi + hi*lo + lo*hi); each tap accumulates into a fresh register fragment that is added into the fp32
// sum in tap order (a long tensor-core accumulation truncates, see conv_tc.cu).  Two taps are in flight per
// warpgroup: tap t+1 is issued into the other of two fragments before the wait that completes tap t, so the
// tensor core works on t+1 while tap t is added into the sum.  Roles (four warpgroups, registers reallocated
// with setmaxnreg: TP_REG_* below):
//   warps 0-7   two consumer warpgroups: warpgroup g issues the MMAs of tile rows 64g .. 64g+63 and promotes
//               them; a finished tile goes to one of two shared-memory tiles s_acc[2][128][NT + 1]
//   warps 8-11  epilogue, one pixel row per thread: folded eval BN (+ residual, ReLU) / raw / accumulate,
//               streamed in float4 chunks while the consumers run the next tile
//   warp  12    weight loader (one elected lane): cp.async.bulk of pre-split, pre-swizzled [NT x 32] tiles,
//               resident for the whole kernel when all 9 taps fit (cin <= 32), a ring otherwise
//   warps 13-15 patch loaders: coalesced LDG.128 of NHWC pixels, cvt.rna.tf32 split, swizzled stores
// CTAs are persistent over pixel tiles (one CTA per SM).  The kernel serves eval-mode forwards and
// stride-1 data gradients; train-mode forwards, which need batch statistics, run on conv.cu or conv_tc.cu
// (conv_tcp_eligible says why).
#include "conv.cuh"
#include "umma.cuh"

namespace b200ocl {
namespace {

constexpr int TP_THREADS = 32 * 16;
constexpr int TP_EPI_WARP = 8;                      // first epilogue warp
constexpr int TP_WLOAD_WARP = 12;                   // weight loader
constexpr int TP_LOADER_WARP = 13;                  // first patch-loader warp
constexpr int TP_LOADERS = 96;                      // patch-loader threads: nch chunks x 96 / nch rows per pass
constexpr int TP_LD = (16 * TP_LD_MAX + 11) / 12;   // loads per patch-loader thread: the rows tcp_strip_fits allows
                                                    // at 12 rows per pass (a full 32-channel slice)
constexpr int TP_PS_MAX = 3;                        // patch stages: 3 when shared memory allows, else 2
constexpr int TP_BS_MAX = 6;                        // weight ring depth (streaming mode): 6 or 4
constexpr int TP_CONSUMER_WARPS = 8;                // arrivals that release a patch stage or a weight slot
// Registers per thread after setmaxnreg: loaders, consumers (the fp32 sum and two fragments), epilogue.
// 128 * P + 256 * C + 128 * E = 65536, the 128 per thread of the 512-thread launch.  The patch loaders hold 18 float4
// loads across the stage wait and need all 128 (at 120 ptxas spills), so the loader warpgroup keeps its launch count;
// the epilogue, which streams its row, hands 32 to the consumers.
constexpr int TP_REG_LOAD = 128, TP_REG_MMA = 144, TP_REG_EPI = 96;
static_assert(TP_REG_LOAD == 128, "the loader warpgroup runs no setmaxnreg");
static_assert(128 * TP_REG_LOAD + 256 * TP_REG_MMA + 128 * TP_REG_EPI <= 65536, "register file");

using umma::mbar_expect_tx;
using umma::bulk_g2s;

// Timeline build (-DB200OCL_TCP_TRACE, tools/tcp_trace.py; never in the shipped library): one thread per role writes
// %clock64 stamps into the buffer b200ocl_tcp_trace_set installs, laid out [CTA][role][unit][TCP_EV] (unit: the CTA's
// tap, slice or tile counter).  Role TCP_HDR holds %globaltimer / %clock64 at the CTA's start and end and its SM.
// Events per unit --
//   consumer warpgroup 0 / 1, per tap: 0 issue start (pfull wait), 1 bfull wait, 2 MMA issue, 3 committed,
//     4 wait_group, 5 promotion, 6 retired; the tile's last tap: 7 aempty waited, 8 s_acc stored and afull arrived
//   weight loader, per tap: 0 bempty wait, 1 copy issue, 2 issued
//   patch loaders, per slice: 0 loads issued from, 1 pempty wait, 2 split and store, 3 pfull arrived
//   epilogue, per tile: 0 residual loads, 1 afull wait, 2 store, 3 aempty arrived
#ifdef B200OCL_TCP_TRACE
enum { TCP_C0, TCP_C1, TCP_WLOAD, TCP_PLOAD, TCP_EPI, TCP_HDR, TCP_ROLES };
constexpr int TCP_EV = 9;
__device__ unsigned long long* g_tcp_trace;
__device__ int g_tcp_trace_units;
__device__ __forceinline__ unsigned long long tcp_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// tcp_units / tcp_cta are read once per CTA (TCP_TRACE_SETUP), so that a stamp is a clock read and a store
#define TCP_TRACE_SETUP                                                                                          \
  const int tcp_units = g_tcp_trace_units;                                                                      \
  unsigned long long* const tcp_cta =                                                                           \
      g_tcp_trace + ((unsigned long long)blockIdx.y * gridDim.x + blockIdx.x) * TCP_ROLES * tcp_units * TCP_EV
#define TCP_AT(role, unit, ev) tcp_cta[((role) * tcp_units + (unit)) * TCP_EV + (ev)]
#define TCP_STAMP(on, role, unit, ev)                                          \
  do {                                                                         \
    if ((on) && (unit) < tcp_units) TCP_AT(role, unit, ev) = clock64();        \
  } while (0)
#else
#define TCP_STAMP(on, role, unit, ev) do { } while (0)
#endif

struct TileGeom {
  int wp, pp;        // strip row length W + 1, strip image size (H + 1) * (W + 1)
  int tiles_m;       // tiles of 128 strip positions
  int prow;          // strip rows staged per tile: 128 + 2 * wp + 2
  int pbytes;        // bytes of one hi (or lo) patch, 1024-aligned
};
__host__ __device__ inline TileGeom tile_geom(int N, int H, int W) {
  TileGeom g;
  g.wp = W + 1;
  g.pp = (H + 1) * (W + 1);
  // the last useful position is the last real pixel of the last image
  const long last = (long)(N - 1) * g.pp + (long)(H - 1) * g.wp + (W - 1);
  g.tiles_m = (int)(last / 128) + 1;
  g.prow = 128 + 2 * g.wp + 2;
  g.pbytes = (g.prow * 128 + 1023) / 1024 * 1024;
  return g;
}

// One tap of one 32-channel slice into a fresh fragment: KS K steps (8 channels each) x 3 MMAs, committed as one
// group; the caller waits for it.  The commit stays inside each KS variant: committed after the caller's switch
// joins, ptxas closes every variant's chain there itself and adds an empty group at the join, so a tap would be two
// groups and wait_group 1 would leave only the empty one outstanding.
template <int NT, int KS>
__device__ __forceinline__ void issue_tap(float (&d)[NT / 2], uint64_t dAh, uint64_t dAl, uint64_t dBh, uint64_t dBl) {
  umma::fence();
#pragma unroll
  for (int k = 0; k < KS; ++k) {
    const uint64_t adv = (uint64_t)(k * 2);   // 32 bytes per K step, in 16-byte units
    umma::mma_tf32_ss<NT>(d, dAh + adv, dBh + adv, k > 0 ? 1u : 0u);
    umma::mma_tf32_ss<NT>(d, dAh + adv, dBl + adv, 1u);
    umma::mma_tf32_ss<NT>(d, dAl + adv, dBh + adv, 1u);
  }
  umma::commit();
}

template <int NT>
__global__ void __launch_bounds__(TP_THREADS, 1) conv_tcp_kernel(ConvArgs a) {
  constexpr int B_BLOCK = 2 * NT * 32;   // floats: hi tile then lo tile
  constexpr int R = NT / 2;              // accumulator registers per thread (m64 x NT per warpgroup)
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  unsigned char* patch0 = smem_raw;                                          // [PS][hi | lo][PROWS][128 B]
  __shared__ __align__(8) uint64_t pfull[TP_PS_MAX], pempty[TP_PS_MAX], bfull[9], bempty[TP_BS_MAX];
  __shared__ __align__(8) uint64_t afull[2], aempty[2];   // s_acc buffer written by the consumers / read by the epilogue
  __shared__ int s_fail;
  __shared__ float s_coef[3 * 80];   // eval BN: mean, scale, shift per channel of the tile

  const int tid = threadIdx.x, warp = tid >> 5;
  const int bn = a.tp_bn;
  const int n0 = blockIdx.y * bn;
  const int slices = a.tp_slices;
  const TileGeom G = tile_geom(a.N, a.Hin, a.Win);
  const int PS = a.tp_ps, BS = a.tp_bs;            // patch stages, weight ring depth (launcher fits them to smem)
  // the tile loops run to a.tp_tiles (= G.tiles_m): a kernel parameter is not a register live across them
  float* sB = reinterpret_cast<float*>(smem_raw + (size_t)PS * 2 * G.pbytes);   // weight blocks
  const bool resident = (slices == 1 && NT == 32);   // all 9 weight blocks stay in shared memory
  const int b_slots = resident ? 9 : BS;
  constexpr int ACC_TILE = 128 * (NT + 1);
  float* s_acc = sB + (size_t)b_slots * B_BLOCK;   // [2][128][NT + 1] finished tiles, one pixel row per epilogue thread

  if (tid == 0) {
    for (int i = 0; i < TP_PS_MAX; ++i) {
      umma::mbar_init(&pfull[i], TP_LOADERS);
      umma::mbar_init(&pempty[i], TP_CONSUMER_WARPS);
    }
    for (int i = 0; i < 9; ++i) umma::mbar_init(&bfull[i], 1);
    for (int i = 0; i < TP_BS_MAX; ++i) umma::mbar_init(&bempty[i], TP_CONSUMER_WARPS);
    for (int i = 0; i < 2; ++i) {
      umma::mbar_init(&afull[i], 256);    // every consumer thread, after its stores
      umma::mbar_init(&aempty[i], 128);   // every epilogue thread, after its reads
    }
    umma::fence_mbar_init();
    s_fail = 0;
  }
  __syncthreads();
#ifdef B200OCL_TCP_TRACE
  TCP_TRACE_SETUP;
  if (tid == 0) {
    TCP_AT(TCP_HDR, 0, 0) = tcp_globaltimer();
    TCP_AT(TCP_HDR, 0, 1) = clock64();
  }
#endif
  const float* wimg = a.w_tp + (size_t)blockIdx.y * slices * 9 * B_BLOCK;

  if (warp >= TP_LOADER_WARP) {
    // =========================================================== patch loaders (96 threads)
    const int lt = tid - 32 * TP_LOADER_WARP;
    int pc = 0;
    for (int tile = blockIdx.x; tile < a.tp_tiles; tile += gridDim.x) {
      for (int sl = 0; sl < slices; ++sl, ++pc) {
        TCP_STAMP(lt == 0, TCP_PLOAD, pc, 0);
        const int ch_valid = min(32, a.CK - sl * 32);       // real channels in this slice (multiple of 4)
        const int nch = 2 * ((ch_valid + 7) / 8);            // 16-byte chunks the MMAs will read per row
        // thread -> (patch row lt/nch + step*i, chunk lt%nch): every lane loads, so a slice of 8 / 16 / 24 channels
        // takes 1/4 / 1/2 / 3/4 of a full slice's passes (nch = 2, 4, 6 or 8 divides the 96 threads)
        const int step = TP_LOADERS / nch;                   // rows per pass: 48, 24, 16 or 12
        const int ch = lt % nch, r0 = lt / nch;
        const int nrow = G.prow;
        const bool ch_real = ch * 4 < ch_valid;
        float4 v[TP_LD];
        // strip position of this thread's first row, then step rows further per pass (no divisions in the loop)
        int img, yp, xp;
        {
          const int sp = tile * 128 + r0;
          img = sp / G.pp;
          const int rem = sp - img * G.pp;
          yp = rem / G.wp;
          xp = rem - yp * G.wp;
        }
        const int hp = a.Hin + 1;                             // strip rows per image: the zero row, then H pixel rows
#pragma unroll
        for (int i = 0; i < TP_LD; ++i) {
          const int ri = r0 + step * i;
          if (ri >= nrow) break;
          v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ch_real) {
            const int y = yp - 1, x = xp - 1;
            if (img < a.N && (unsigned)y < (unsigned)a.Hin && (unsigned)x < (unsigned)a.Win)
              v[i] = __ldg(reinterpret_cast<const float4*>(a.in + ((size_t)(img * a.Hin + y) * a.Win + x) * a.CK + sl * 32) + ch);
          }
          xp += step;
          while (xp >= G.wp) {
            xp -= G.wp;
            if (++yp == hp) {
              yp = 0;
              ++img;
            }
          }
        }
        const int ps = pc % PS;
        TCP_STAMP(lt == 0, TCP_PLOAD, pc, 1);
        if (!umma::mbar_wait(&pempty[ps], (uint32_t)(((pc / PS) & 1) ^ 1))) s_fail = 1;
        TCP_STAMP(lt == 0, TCP_PLOAD, pc, 2);
        float* ph = reinterpret_cast<float*>(patch0 + (size_t)ps * 2 * G.pbytes);
        float* pl = ph + G.pbytes / 4;
#pragma unroll
        for (int i = 0; i < TP_LD; ++i) {
          const int ri = r0 + step * i;
          if (ri >= nrow) break;
          float4 h, l;
          umma::split_tf32(v[i].x, h.x, l.x); umma::split_tf32(v[i].y, h.y, l.y);
          umma::split_tf32(v[i].z, h.z, l.z); umma::split_tf32(v[i].w, h.w, l.w);
          const int off = umma::sw128_offset_f32(ri, ch);
          *reinterpret_cast<float4*>(ph + off) = h;
          *reinterpret_cast<float4*>(pl + off) = l;
        }
        umma::fence_proxy_async_smem();
        umma::mbar_arrive(&pfull[ps]);
        TCP_STAMP(lt == 0, TCP_PLOAD, pc, 3);
      }
    }
  } else if (warp == TP_WLOAD_WARP) {
    // =========================================================== weight loader (one elected lane)
    const uint32_t bytes = (uint32_t)(B_BLOCK * sizeof(float));
    if (resident) {
      if (umma::elect_one_sync()) {
        for (int b = 0; b < 9; ++b) {
          TCP_STAMP(true, TCP_WLOAD, b, 0);
          TCP_STAMP(true, TCP_WLOAD, b, 1);
          mbar_expect_tx(&bfull[b], bytes);
          bulk_g2s(sB + (size_t)b * B_BLOCK, wimg + (size_t)b * B_BLOCK, bytes, &bfull[b]);
          TCP_STAMP(true, TCP_WLOAD, b, 2);
        }
      }
    } else {
      int q = 0;
      for (int tile = blockIdx.x; tile < a.tp_tiles; tile += gridDim.x)
        for (int sl = 0; sl < slices; ++sl)
          for (int tap = 0; tap < 9; ++tap, ++q) {
            const int bs = q % BS;
            TCP_STAMP((tid & 31) == 0, TCP_WLOAD, q, 0);
            if (!umma::mbar_wait(&bempty[bs], (uint32_t)(((q / BS) & 1) ^ 1))) s_fail = 1;
            TCP_STAMP((tid & 31) == 0, TCP_WLOAD, q, 1);
            if (umma::elect_one_sync()) {
              mbar_expect_tx(&bfull[bs], bytes);
              bulk_g2s(sB + (size_t)bs * B_BLOCK, wimg + (size_t)(sl * 9 + tap) * B_BLOCK, bytes, &bfull[bs]);
            }
            __syncwarp();
            TCP_STAMP((tid & 31) == 0, TCP_WLOAD, q, 2);
          }
    }
  } else if (warp >= TP_EPI_WARP) {
    // =========================================================== epilogue (warps 8-11)
    umma::reg_dealloc<TP_REG_EPI>();
    const int et = tid - 32 * TP_EPI_WARP;               // pixel row of the tile
    if (a.mode == CONV_EVAL) {
      for (int c = et; c < bn; c += 128) {
        const float inv = 1.0f / sqrtf(a.rvar[n0 + c] + a.eps);
        s_coef[c] = a.rmean[n0 + c];
        s_coef[80 + c] = inv * a.gamma[n0 + c];
        s_coef[160 + c] = a.beta[n0 + c];
      }
      asm volatile("bar.sync 1, 128;\n" ::);
    }
    int k = 0;                                           // tiles this CTA has finished
    for (int tile = blockIdx.x; tile < a.tp_tiles; tile += gridDim.x, ++k) {
      const int buf = k & 1;
      TCP_STAMP(et == 0, TCP_EPI, k, 0);
      const int sp = tile * 128 + et;                    // strip position of this MMA row
      const int img = sp / G.pp, rem = sp - img * G.pp;
      const int y = rem / G.wp, x = rem - y * G.wp;
      const bool valid = img < a.N && y < a.Hin && x < a.Win;   // halo positions are by-products
      const size_t m = ((size_t)img * a.Hin + y) * a.Win + x;   // stride 1: output pixel = input pixel
      // src = the residual (eval) or the gradient being accumulated into (data gradient); pre is 0 without one
      const float* src = nullptr;
      if (valid && a.mode == CONV_EVAL && a.residual) src = a.residual + m * a.CN + n0;
      if (valid && a.mode == CONV_ACCUM) src = a.out + m * a.CN + n0;
      // All of the row's loads are issued before the wait, so their latency hides behind the consumers' tile: src
      // may be the output itself (accumulate) or alias it, so a load after a store could not be moved ahead of it.
      float pre[NT];
#pragma unroll
      for (int c = 0; c < NT; ++c) pre[c] = 0.f;
      if (src) {
#pragma unroll
        for (int c0 = 0; c0 < NT; c0 += 4) {
          if (c0 >= bn) break;
          const float4 v = *reinterpret_cast<const float4*>(src + c0);
          pre[c0] = v.x; pre[c0 + 1] = v.y; pre[c0 + 2] = v.z; pre[c0 + 3] = v.w;
        }
      }
      TCP_STAMP(et == 0, TCP_EPI, k, 1);
      if (!umma::mbar_wait(&afull[buf], (uint32_t)((k >> 1) & 1))) s_fail = 1;
      TCP_STAMP(et == 0, TCP_EPI, k, 2);
      const float* row = s_acc + (size_t)buf * ACC_TILE + et * (NT + 1);
      if (valid) {
        float* o = a.out + m * a.CN + n0;
#pragma unroll
        for (int c0 = 0; c0 < NT; c0 += 4) {   // the tile's row streams from s_acc a float4 at a time
          if (c0 >= bn) break;
          float rr[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float acc = row[c0 + j];
            if (a.mode == CONV_EVAL) {
              rr[j] = (acc - s_coef[c0 + j]) * s_coef[80 + c0 + j] + s_coef[160 + c0 + j];
              rr[j] += pre[c0 + j];                       // residual (0 when there is none)
              if (a.relu) rr[j] = fmaxf(rr[j], 0.f);
            } else {
              rr[j] = acc + pre[c0 + j];                  // raw: pre == 0; accumulate: pre = previous contents
            }
          }
          *reinterpret_cast<float4*>(o + c0) = make_float4(rr[0], rr[1], rr[2], rr[3]);
        }
      }
      umma::mbar_arrive(&aempty[buf]);
      TCP_STAMP(et == 0, TCP_EPI, k, 3);
    }
  } else {
    // =========================================================== consumers (warps 0-7)
    umma::reg_alloc<TP_REG_MMA>();
    const int g = warp >> 2, wt = tid & 127;            // warpgroup, thread inside it
    const bool lane0 = (tid & 31) == 0;
    // descriptor templates: only the 14-bit start-address field (16-byte units) changes per stage / tap / K step
    const uint64_t dA0 = umma::make_smem_desc_sw128(umma::smem_u32(patch0) + (uint32_t)(g * 64 * 128));
    const uint64_t dB0 = umma::make_smem_desc_sw128(umma::smem_u32(sB));
    const uint32_t A_LO = (uint32_t)G.pbytes >> 4;            // hi -> lo patch, 16-byte units
    const uint32_t A_STAGE = (uint32_t)(2 * G.pbytes) >> 4;
    constexpr uint32_t B_LO = (NT * 128) >> 4;
    constexpr uint32_t B_SLOT = (B_BLOCK * 4) >> 4;
    const int T = 9 * slices;                // taps per tile
    // Issue side: patch stage and its phase, weight slot and its phase.  Retire side: the stage and slot to release.
    // All run on over the CTA's tiles; counters wrap instead of dividing.
    int ips = 0, ib = 0, rps = 0, rb = 0;
    uint32_t ipph = 0, ibph = 0;
    bool b_ready = false;
#ifdef B200OCL_TCP_TRACE
    const bool tr = wt == 0;
    int tu_i = 0, tu_r = 0;                  // the CTA's taps issued / retired
#endif
    int k = 0;                               // tiles this CTA has finished
    for (int tile = blockIdx.x; tile < a.tp_tiles; tile += gridDim.x, ++k) {
      float accf[R];
#pragma unroll
      for (int i = 0; i < R; ++i) accf[i] = 0.f;
      // The tile's T taps as one stream (slice by slice, tap order within a slice).  Issue position (is, it) runs
      // one tap ahead of the retire position rt; a weight slot or patch stage is released once the wait that
      // completes the last MMA reading it has returned.
      int is = 0, it = 0, rt = 0;
      auto issue = [&](float (&d)[R]) {
        TCP_STAMP(tr, g, tu_i, 0);
        if (it == 0)
          if (!umma::mbar_wait(&pfull[ips], ipph)) s_fail = 1;
        TCP_STAMP(tr, g, tu_i, 1);
        const int b = resident ? it : ib;
        if (!(resident && b_ready))
          if (!umma::mbar_wait(&bfull[b], resident ? 0u : ibph)) s_fail = 1;
        TCP_STAMP(tr, g, tu_i, 2);
        const int kh = it / 3, kw = it - 3 * kh;
        const uint64_t dAh = dA0 + (uint64_t)(ips * A_STAGE) + (uint64_t)((kh * G.wp + kw) * 8);   // + (kh*(W+1) + kw) rows
        const uint64_t dAl = dAh + A_LO;
        const uint64_t dBh = dB0 + (uint64_t)(b * B_SLOT);
        const uint64_t dBl = dBh + B_LO;
        switch ((min(32, a.CK - is * 32) + 7) / 8) {   // straight-line issue sequences: a run-time trip count
          case 1: issue_tap<NT, 1>(d, dAh, dAl, dBh, dBl); break;   // would serialise the MMAs
          case 2: issue_tap<NT, 2>(d, dAh, dAl, dBh, dBl); break;
          case 3: issue_tap<NT, 3>(d, dAh, dAl, dBh, dBl); break;
          default: issue_tap<NT, 4>(d, dAh, dAl, dBh, dBl); break;
        }
#ifdef B200OCL_TCP_TRACE
        TCP_STAMP(tr, g, tu_i, 3);
        ++tu_i;
#endif
        if (!resident && ++ib == BS) {
          ib = 0;
          ibph ^= 1u;
        }
        if (++it == 9) {
          it = 0;
          ++is;
          b_ready = true;
          if (++ips == PS) {
            ips = 0;
            ipph ^= 1u;
          }
        }
      };
      auto retire = [&](float (&d)[R]) {
        TCP_STAMP(tr, g, tu_r, 5);
        umma::fence_regs(d);
#pragma unroll
        for (int i = 0; i < R; ++i) accf[i] += d[i];
        if (!resident) {
          if (lane0) umma::mbar_arrive(&bempty[rb]);
          if (++rb == BS) rb = 0;
        }
        if (rt == 8) {
          if (lane0) umma::mbar_arrive(&pempty[rps]);
          if (++rps == PS) rps = 0;
        }
        if (++rt == 9) rt = 0;
#ifdef B200OCL_TCP_TRACE
        TCP_STAMP(tr, g, tu_r, 6);
        ++tu_r;
#endif
      };
      // Every exit drains with wait<0> in the block that leaves the loop, so that the compiler sees no fragment
      // in flight past it.
      float fa[R], fb[R];
      issue(fa);
#pragma unroll 1
      for (int j = 0;; j += 2) {   // fa holds tap j, fb tap j + 1
        if (j + 1 >= T) {
          TCP_STAMP(tr, g, tu_r, 4);
          umma::wait<0>();
          retire(fa);
          break;
        }
        issue(fb);
        TCP_STAMP(tr, g, tu_r, 4);
        umma::wait<1>();
        retire(fa);
        if (j + 2 >= T) {
          TCP_STAMP(tr, g, tu_r, 4);
          umma::wait<0>();
          retire(fb);
          break;
        }
        issue(fa);
        TCP_STAMP(tr, g, tu_r, 4);
        umma::wait<1>();
        retire(fb);
      }
      // ---- fragments -> pixel rows of s_acc[k % 2], once the epilogue has read that buffer's previous tile
      const int buf = k & 1;
      if (!umma::mbar_wait(&aempty[buf], (uint32_t)(((k >> 1) & 1) ^ 1))) s_fail = 1;
      TCP_STAMP(tr, g, tu_r - 1, 7);
      float* acc_out = s_acc + (size_t)buf * ACC_TILE;
#pragma unroll
      for (int i = 0; i < R; ++i) acc_out[(64 * g + umma::frag_row(wt, i)) * (NT + 1) + umma::frag_col(wt, i)] = accf[i];
      umma::mbar_arrive(&afull[buf]);
      TCP_STAMP(tr, g, tu_r - 1, 8);
    }
  }
  __syncthreads();
#ifdef B200OCL_TCP_TRACE
  if (tid == 0) {
    TCP_AT(TCP_HDR, 0, 2) = tcp_globaltimer();
    TCP_AT(TCP_HDR, 0, 3) = clock64();
    unsigned smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    TCP_AT(TCP_HDR, 0, 4) = smid;
  }
#endif
  // a timed-out barrier (must never happen) poisons the output instead of hanging the GPU
  if (s_fail && tid == 0) a.out[(size_t)n0] = __int_as_float(0x7fc00000);
}

template <int NT>
size_t tcp_smem_bytes(const TileGeom& G, int slices, int ps, int bs) {
  const int b_slots = (slices == 1 && NT == 32) ? 9 : bs;
  return (size_t)ps * 2 * G.pbytes + (size_t)b_slots * 2 * NT * 32 * sizeof(float) +
         (size_t)2 * 128 * (NT + 1) * sizeof(float) + 1024;
}

// Deepest pipeline that fits next to the two s_acc tiles: 3 patch stages + 6 weight slots, 3 + 4, 2 + 6, else 2 + 4
// (two taps in flight hold two slots and two stages at once, so both stay >= 2).  The network's maps: 32x32
// (resident weights) keeps 2 stages, 8x8 and 4x4 keep 3 + 4, 16x16 goes from 3 + 4 (one s_acc tile) to 2 + 6.
template <int NT>
void fit_pipeline(const ConvArgs& a, int* ps, int* bs) {
  const TileGeom G = tile_geom(a.N, a.Hin, a.Win);
  const size_t limit = 227 * 1024 - 4096;      // static shared memory (barriers, coefficients) comes on top
  *ps = 3; *bs = 6;
  if (tcp_smem_bytes<NT>(G, a.tp_slices, *ps, *bs) > limit) *bs = 4;
  if (tcp_smem_bytes<NT>(G, a.tp_slices, *ps, *bs) > limit) { *ps = 2; *bs = 6; }
  if (tcp_smem_bytes<NT>(G, a.tp_slices, *ps, *bs) > limit) *bs = 4;
}

template <int NT>
int launch_tcp(ConvArgs a, const ConvPlan& pl, cudaStream_t stream) {
  const TileGeom G = tile_geom(a.N, a.Hin, a.Win);
  fit_pipeline<NT>(a, &a.tp_ps, &a.tp_bs);
  const size_t smem = tcp_smem_bytes<NT>(G, a.tp_slices, a.tp_ps, a.tp_bs);
  B200OCL_CUDA(raise_smem_limit<conv_tcp_kernel<NT>>(smem));
  a.tp_tiles = G.tiles_m;
  // one kernel, two epilogues (eval / data gradient): profiled as one class
  B200OCL_PROF("conv_tcp",
               2.0 * a.M * (double)a.CN * a.CK * 9.0, stream);
  conv_tcp_kernel<NT><<<dim3(pl.grid_x, pl.grid_y), TP_THREADS, smem, stream>>>(a);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

}  // namespace

void conv_tcp_pipeline(const ConvArgs& a, int nt, int* ps, int* bs) {
  if (nt == 32) fit_pipeline<32>(a, ps, bs);
  else fit_pipeline<48>(a, ps, bs);
}

int conv_tcp_grid_x(const ConvArgs& a, int sms) {
  const TileGeom G = tile_geom(a.N, a.Hin, a.Win);
  int gx = sms / (a.CN / a.tp_bn);
  if (gx < 1) gx = 1;
  if (gx > G.tiles_m) gx = G.tiles_m;
  // even out the tiles per CTA (e.g. 880 tiles on 132 CTAs = 7 rounds -> 126 CTAs of 7, one of 2)
  const int rounds = (G.tiles_m + gx - 1) / gx;
  return (G.tiles_m + rounds - 1) / rounds;
}

bool conv_tcp_eligible(const ConvArgs& a) {
  // Precision policy: no train-mode forwards.  The truncating tensor-core accumulate leaves a small sign-dependent
  // bias that a train-mode forward differentiates through BatchNorm, while eval features and data gradients keep to
  // the fp32 bar of the drop-in comparison (tests/test_gpu_dropin.py).
  if (a.mode == CONV_TRAIN || !a.w_tp || a.transposed || a.CK % 4 != 0) return false;
  if (a.ks != 3 || a.pad != 1 || a.stride != 1 || a.Hout != a.Hin || a.Wout != a.Win) return false;
  if (!tcp_strip_fits(a.Win)) return false;
  if ((long)a.N * (a.Hin + 2) * (a.Win + 2) > 2000000000L) return false;
  if (a.tp_bn <= 0 || a.tp_bn > 40 || a.CN % a.tp_bn != 0) return false;
  return true;
}

int launch_conv_tcp(const ConvArgs& a, const ConvPlan& pl, cudaStream_t stream) {
  if (pl.nt == 32) return launch_tcp<32>(a, pl, stream);
  return launch_tcp<48>(a, pl, stream);
}

}  // namespace b200ocl

#ifdef B200OCL_TCP_TRACE
// Timeline build only: the stamp buffer of the conv_tcp launches that follow, `units` per CTA and role
// ([CTA][role][unit][TCP_EV] uint64).  Declared by the tool that loads that build, not in include/b200ocl.h.
extern "C" int b200ocl_tcp_trace_set(unsigned long long* buf, int units) {
  using namespace b200ocl;
  B200OCL_CUDA(cudaMemcpyToSymbol(g_tcp_trace, &buf, sizeof(buf)));
  B200OCL_CUDA(cudaMemcpyToSymbol(g_tcp_trace_units, &units, sizeof(units)));
  return B200OCL_OK;
}
#endif
