// umma.cuh -- thin inline-PTX layer over the Hopper warpgroup tensor-core path (wgmma.mma_async, sm_90a) used by
// the tensor-core convolutions and the weight gradient.
//
// Operand layout used throughout: K-major tiles with the 128-byte swizzle.  A tile is [rows][32 fp32] = rows x 128 B;
// row r, 16-byte chunk c lives at
//     (r / 8) * 1024 + (r % 8) * 128 + ((c ^ (r % 8)) * 16)
// from a 1024-byte aligned base.  The hardware applies the XOR to address bits 4..6 from bits 7..9 of the absolute
// shared-memory address, so a descriptor may start at any 128-byte row of such an array (the halo-patch convolution
// reads every tap through a shifted window) and consecutive K steps inside the 128-byte row advance the start address
// by 32 bytes.  One wgmma ...k8.f32.tf32.tf32 consumes K = 8 fp32 (32 bytes) per row for M = 64 rows; the 128-row tiles
// of the kernels are two such halves 8 KB apart.
//
// Accumulators live in the registers of the issuing warpgroup (4 warps).  Thread t of the warpgroup holds, for an
// m64nN fp32 accumulator, register i at
//     row = 16 * (t / 32) + (t % 32) / 4 + 8 * ((i % 4) / 2),   col = 8 * (i / 4) + 2 * (t % 4) + (i % 2).
#pragma once
#include <stdint.h>

namespace b200ocl {
namespace umma {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- swizzled K-major tile addressing (in floats from the tile base)
__device__ __forceinline__ int sw128_offset_f32(int row, int chunk16) {
  return (row >> 3) * 256 + (row & 7) * 32 + ((chunk16 ^ (row & 7)) << 2);
}

// ---- accumulator fragment coordinates (see the header comment)
__device__ __forceinline__ int frag_row(int t, int i) { return ((t >> 5) << 4) + ((t & 31) >> 2) + ((i & 2) << 2); }
__device__ __forceinline__ int frag_col(int t, int i) { return ((i >> 2) << 3) + ((t & 3) << 1) + (i & 1); }

// Shared-memory matrix descriptor: K-major, 128-byte swizzle, 8-row groups 1024 B apart, base offset 0.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);          // start address
  d |= (uint64_t)1 << 16;                               // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)((1024 >> 4) & 0x3FFF) << 32;          // stride byte offset: next 8-row group
  d |= (uint64_t)1 << 62;                               // layout type: 128-byte swizzle
  return d;
}

// ---- warpgroup MMA ordering
__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMA window
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// ---- per-warpgroup register reallocation (all four warps of a warpgroup execute it).  The kernel launches with its
// __launch_bounds__ register count; a warpgroup that needs less gives registers back to the pool and one that needs
// more blocks in setmaxnreg.inc until the pool holds them.  N: a multiple of 8 in 24 .. 256.
template <int N>
__device__ __forceinline__ void reg_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void reg_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(N)); }
// generic-proxy shared-memory writes -> visible to the async proxy (tensor core operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;\n" ::); }

// ---- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::); }
// Bounded wait: returns false if the phase did not complete within max_spins polls (a wrong
// descriptor must not hang the GPU).
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity, uint32_t max_spins = (1u << 24)) {
  const uint32_t addr = smem_u32(bar);
#pragma unroll 1
  for (uint32_t i = 0; i < max_spins; ++i) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) return true;
  }
  return false;
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}

// ---- TMA 1-D bulk copy global -> shared (cp.async.bulk); completion counted in bytes on an mbarrier.
// dst / src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
          smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ---- one elected lane of a converged warp
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---- MMA issue (the whole warpgroup): D[64, N] (+)= A[64, 8] * B[N, 8]^T, fp32 accumulate in registers.
// _ss: A and B from shared memory through descriptors; _rs: A from registers, thread t holding
// (row g, k q), (g + 8, q), (g, q + 4), (g + 8, q + 4) with g = 16 * (t / 32) + (t % 32) / 4, q = t % 4.
template <int N>
__device__ __forceinline__ void mma_tf32_ss(float (&d)[N / 2], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate);
template <int N>
__device__ __forceinline__ void mma_tf32_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate);

template <>
__device__ __forceinline__ void mma_tf32_ss<16>(float (&d)[8], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

template <>
__device__ __forceinline__ void mma_tf32_ss<32>(float (&d)[16], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

template <>
__device__ __forceinline__ void mma_tf32_ss<48>(float (&d)[24], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %26, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

template <>
__device__ __forceinline__ void mma_tf32_ss<80>(float (&d)[40], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %42, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n80k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39}, %40, %41, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

template <>
__device__ __forceinline__ void mma_tf32_rs<32>(float (&d)[16], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}

template <>
__device__ __forceinline__ void mma_tf32_rs<8>(float (&d)[4], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %9, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n8k8.f32.tf32.tf32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, %8, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}

template <>
__device__ __forceinline__ void mma_tf32_rs<16>(float (&d)[8], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}

template <>
__device__ __forceinline__ void mma_tf32_rs<24>(float (&d)[12], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %17, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n24k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, %16, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}

template <>
__device__ __forceinline__ void mma_tf32_rs<40>(float (&d)[20], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %25, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n40k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19}, {%20,%21,%22,%23}, %24, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}

// ---- TF32 split: x = hi + lo with hi = x ROUNDED to TF32 (cvt.rna: one instruction) and lo the exact
// fp32 remainder.  Rounding matters: a truncated hi leaves a same-signed remainder whose own truncation
// by the tensor core then accumulates linearly over K.  With a rounded hi the remainder is sign-symmetric,
// so the hardware's truncation of lo to 10 mantissa bits (|error| <= 2^-22 |x|) is unbiased.
__device__ __forceinline__ float round_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = round_tf32(x);
  lo = x - hi;
}

}  // namespace umma
}  // namespace b200ocl
