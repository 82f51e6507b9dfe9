// common.cuh -- shared helpers for libb200ocl (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "../../include/b200ocl.h"

namespace b200ocl {

void set_error(const char* fmt, ...);
// Optional per-launch timing (bench.py roofline): when enabled, every launch is bracketed by CUDA
// events on its own stream and accumulated per kernel class.  Off by default (no overhead).
extern bool g_prof_on;
void prof_begin(const char* kernel_class, double work, cudaStream_t stream);
void prof_end();
extern std::atomic<uint64_t> g_launches;
int sm_count();
#define B200OCL_MAX_DEVICES 64
inline int device_slot() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= B200OCL_MAX_DEVICES) dev = 0;
  return dev;
}

// Raises the dynamic shared-memory limit of the kernels Ks to `bytes` on the current device.  Function attributes are
// per device, so each instantiation keeps the limit it set per device and only calls cudaFuncSetAttribute when a
// launch asks for more; a smaller request changes nothing.
template <auto... Ks>
cudaError_t raise_smem_limit(size_t bytes) {
  static size_t set_dev[B200OCL_MAX_DEVICES] = {};
  size_t& set = set_dev[device_slot()];
  if (bytes <= set) return cudaSuccess;
  for (const void* k : {reinterpret_cast<const void*>(Ks)...}) {
    const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return e;
  }
  set = bytes;
  return cudaSuccess;
}

// B200OCL_OK when the caller's workspace is non-null, 256-byte aligned and at least `need` bytes; otherwise records
// which entry point refused it and returns B200OCL_EWORKSPACE.
int check_workspace(const char* entry, const void* ws, size_t ws_bytes, size_t need);

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

#define B200OCL_CHECK_ARG(cond, msg)                      \
  do {                                                    \
    if (!(cond)) {                                        \
      b200ocl::set_error("%s: %s", __func__, msg);        \
      return B200OCL_EINVAL;                              \
    }                                                     \
  } while (0)

#define B200OCL_CUDA(call)                                                                    \
  do {                                                                                        \
    cudaError_t err__ = (call);                                                               \
    if (err__ != cudaSuccess) {                                                               \
      (void)cudaGetLastError(); /* clear the non-sticky error state */                        \
      b200ocl::set_error("%s: %s failed: %s", __func__, #call, cudaGetErrorString(err__));    \
      return B200OCL_ECUDA;                                                                   \
    }                                                                                         \
  } while (0)

// Count the launch and surface launch-configuration errors immediately.
// Declare the kernel class and its algorithmic work (FLOPs or bytes) right before a launch.
#define B200OCL_PROF(kernel_class, work, stream)                                              \
  do {                                                                                        \
    if (b200ocl::g_prof_on) b200ocl::prof_begin(kernel_class, (double)(work), stream);        \
  } while (0)

#define B200OCL_LAUNCHED()                                                                    \
  do {                                                                                        \
    if (b200ocl::g_prof_on) b200ocl::prof_end();                                              \
    b200ocl::g_launches.fetch_add(1, std::memory_order_relaxed);                              \
    cudaError_t err__ = cudaGetLastError();                                                   \
    if (err__ != cudaSuccess) {                                                               \
      b200ocl::set_error("%s: kernel launch failed: %s", __func__, cudaGetErrorString(err__)); \
      return B200OCL_ECUDA;                                                                   \
    }                                                                                         \
  } while (0)

constexpr unsigned FULL_MASK = 0xffffffffu;

// 16-byte global -> shared copies (cp.async.cg).  With src_bytes < 16 the rest of the 16 bytes is zero-filled.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src, int src_bytes) {
  const unsigned int s = static_cast<unsigned int>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem_src), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  const unsigned int s = static_cast<unsigned int>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
// wait until at most N committed groups are still in flight
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

// An 8-bit image value in [0, 1]: u / 255 with an IEEE division (torchvision's ToTensor).  The stream feeder and the
// snapshot encoder / decoder share it, so a stored byte always decodes to the value the stream produced.
__device__ __forceinline__ float u8_unit(unsigned u) { return __fdiv_rn((float)u, 255.f); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL_MASK, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL_MASK, v, o));
  return v;
}

}  // namespace b200ocl
