// tc_selftest.cu -- minimal wgmma (tf32, SS operands, register accumulator) GEMM used to validate the
// descriptor encodings of umma.cuh on the device before the tensor-core convolution relies on them.
//   D[128, N] = A[128, K] * B[N, K]^T     K multiple of 32, N multiple of 16 in [16, 256]
// mode 0: single TF32 pass (inputs truncated by the hardware); mode 1: 3xTF32 split
// (hi*hi + hi*lo + lo*hi), the numerics the convolution uses.  One warpgroup computes the output one
// [64 x 16] block at a time, each block one accumulation over the whole K.
#include "common.cuh"
#include "umma.cuh"

namespace b200ocl {
namespace {

__global__ void __launch_bounds__(128) wgmma_selftest_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                             float* __restrict__ D, int N, int K, int mode) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  // [A_hi | A_lo | B_hi | B_lo], each a swizzled K-major tile of 32 fp32 per row
  float* sAh = reinterpret_cast<float*>(smem_raw);
  float* sAl = sAh + 64 * 32;
  float* sBh = sAl + 64 * 32;
  float* sBl = sBh + 16 * 32;
  const int tid = threadIdx.x;
  for (int h = 0; h < 2; ++h)
    for (int q = 0; q < N / 16; ++q) {
      float d[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) d[i] = 0.f;
      for (int kb = 0; kb < K / 32; ++kb) {
        for (int idx = tid; idx < (64 + 16) * 8; idx += 128) {
          const int r = idx >> 3, c = idx & 7;
          const bool is_a = r < 64;
          const float* src = is_a ? A + (size_t)(64 * h + r) * K : B + (size_t)(16 * q + r - 64) * K;
          const float4 v = *reinterpret_cast<const float4*>(src + kb * 32 + c * 4);
          float4 hi, lo;
          umma::split_tf32(v.x, hi.x, lo.x); umma::split_tf32(v.y, hi.y, lo.y);
          umma::split_tf32(v.z, hi.z, lo.z); umma::split_tf32(v.w, hi.w, lo.w);
          const int off = umma::sw128_offset_f32(is_a ? r : r - 64, c);
          *reinterpret_cast<float4*>((is_a ? sAh : sBh) + off) = (mode == 0) ? v : hi;
          *reinterpret_cast<float4*>((is_a ? sAl : sBl) + off) = lo;
        }
        umma::fence_proxy_async_smem();
        __syncthreads();
        const uint64_t dAh = umma::make_smem_desc_sw128(umma::smem_u32(sAh));
        const uint64_t dAl = umma::make_smem_desc_sw128(umma::smem_u32(sAl));
        const uint64_t dBh = umma::make_smem_desc_sw128(umma::smem_u32(sBh));
        const uint64_t dBl = umma::make_smem_desc_sw128(umma::smem_u32(sBl));
        umma::fence_regs(d);
        umma::fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t adv = (uint64_t)(k * 2);   // 32 bytes per K step, in 16-byte units
          umma::mma_tf32_ss<16>(d, dAh + adv, dBh + adv, (kb > 0 || k > 0) ? 1u : 0u);
          if (mode == 1) {
            umma::mma_tf32_ss<16>(d, dAh + adv, dBl + adv, 1u);
            umma::mma_tf32_ss<16>(d, dAl + adv, dBh + adv, 1u);
          }
        }
        umma::commit();
        umma::wait<0>();
        umma::fence_regs(d);
        __syncthreads();   // the staging buffers are overwritten next
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
        D[(size_t)(64 * h + umma::frag_row(tid, i)) * N + 16 * q + umma::frag_col(tid, i)] = d[i];
    }
}

// Window test: the A operand is NOT a packed tile but a window into a larger swizzled buffer of 128-byte
// rows ("patch"): tile row 8g + r is patch row start_row + g * sbo_rows + r.  The patch is stored with the
// swizzle keyed on the absolute row index (row & 7), the start address is not 1024-byte aligned when
// start_row % 8 != 0, and the descriptor's base-offset field (bits 49..51) is set to start_row & 7 when
// base_off_mode == 1.  This is what lets a convolution feed the tensor core straight from a halo patch.
__global__ void __launch_bounds__(128) wgmma_window_kernel(const float* __restrict__ P, const float* __restrict__ B,
                                                           float* __restrict__ D, int rows, int start_row, int sbo_rows,
                                                           int base_off_mode, int N) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  float* sP = reinterpret_cast<float*>(smem_raw);           // rows x 32 fp32
  float* sB = sP + (size_t)((rows + 7) / 8 * 8) * 32;       // 1024-byte aligned
  const int tid = threadIdx.x;
  for (int idx = tid; idx < rows * 8; idx += 128) {
    const int r = idx >> 3, c = idx & 7;
    *reinterpret_cast<float4*>(sP + umma::sw128_offset_f32(r, c)) = *reinterpret_cast<const float4*>(P + (size_t)r * 32 + c * 4);
  }
  for (int idx = tid; idx < N * 8; idx += 128) {
    const int r = idx >> 3, c = idx & 7;
    *reinterpret_cast<float4*>(sB + umma::sw128_offset_f32(r, c)) = *reinterpret_cast<const float4*>(B + (size_t)r * 32 + c * 4);
  }
  umma::fence_proxy_async_smem();
  __syncthreads();
  for (int h = 0; h < 2; ++h) {
    const int row0 = start_row + 8 * h * sbo_rows;   // the second 64-row half starts 8 row groups further
    uint64_t dA = umma::make_smem_desc_sw128(umma::smem_u32(sP) + (uint32_t)row0 * 128u);
    dA &= ~((uint64_t)0x3FFF << 32);
    dA |= (uint64_t)(((uint32_t)sbo_rows * 128u >> 4) & 0x3FFF) << 32;
    if (base_off_mode == 1) dA |= (uint64_t)(row0 & 7) << 49;
    for (int q = 0; q < N / 16; ++q) {
      const uint64_t dB = umma::make_smem_desc_sw128(umma::smem_u32(sB + q * 16 * 32));
      float d[8];
      umma::fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t adv = (uint64_t)(k * 2);
        umma::mma_tf32_ss<16>(d, dA + adv, dB + adv, k > 0 ? 1u : 0u);
      }
      umma::commit();
      umma::wait<0>();
      umma::fence_regs(d);
#pragma unroll
      for (int i = 0; i < 8; ++i)
        D[(size_t)(64 * h + umma::frag_row(tid, i)) * N + 16 * q + umma::frag_col(tid, i)] = d[i];
    }
  }
}

}  // namespace
}  // namespace b200ocl

extern "C" int b200ocl_selftest_umma_tf32(const float* A, const float* B, float* D, int N, int K, int mode, int* status,
                                          void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(A && B && D && status, "null pointer");
  B200OCL_CHECK_ARG(N >= 16 && N <= 256 && N % 16 == 0 && K >= 32 && K % 32 == 0, "need N in [16,256] %16, K %32");
  const size_t smem = (size_t)(2 * 64 * 32 + 2 * 16 * 32) * sizeof(float) + 1024;
  // wgmma completion is waited for in the kernel (no mbarrier): the status word is always 0
  B200OCL_CUDA(cudaMemsetAsync(status, 0, sizeof(int), stream));
  wgmma_selftest_kernel<<<1, 128, smem, stream>>>(A, B, D, N, K, mode);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

extern "C" int b200ocl_selftest_umma_window(const float* P, const float* B, float* D, int rows, int start_row,
                                            int sbo_rows, int base_off_mode, int N, int* status, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(P && B && D && status, "null pointer");
  B200OCL_CHECK_ARG(N >= 16 && N <= 256 && N % 16 == 0, "need N in [16,256] %16");
  B200OCL_CHECK_ARG(rows > 0 && rows <= 1024 && start_row >= 0 && sbo_rows > 0 &&
                        start_row + 15 * sbo_rows + 8 <= rows,
                    "window exceeds the patch");
  const size_t smem = (size_t)((rows + 7) / 8 * 8 + 256) * 32 * sizeof(float) + 1024;
  B200OCL_CUDA(raise_smem_limit<wgmma_window_kernel>(smem));
  B200OCL_CUDA(cudaMemsetAsync(status, 0, sizeof(int), stream));
  wgmma_window_kernel<<<1, 128, smem, stream>>>(P, B, D, rows, start_row, sbo_rows, base_off_mode, N);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}
