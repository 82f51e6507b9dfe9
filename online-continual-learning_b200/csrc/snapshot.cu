// snapshot.cu -- a run's task snapshot, staged on the device (checkpoint.py, B200OCL_CHECKPOINT_ASYNC).
//
// pack copies every segment of a snapshot (engine arenas, memory rows and labels, GSS scores, GDumb's pool) into one
// staging arena, so that training can go on while another stream moves the arena to the host.  Replay-memory rows that
// came from 8-bit images are stored as one byte per value; unpack is the inverse, for a restore.
#include "common.cuh"

namespace b200ocl {
namespace {

constexpr int SNAP_THREADS = 256;

// The byte u with u8_unit(u) == v bit for bit, or -1.  The range test keeps NaN out and the conversion defined;
// -0.0, subnormals and every neighbour of an accepted value fail the bitwise comparison.
__device__ __forceinline__ int snap_encode(float v) {
  if (!(v >= 0.f && v <= 1.f)) return -1;
  const unsigned u = (unsigned)__float2int_rn(v * 255.f);
  return __float_as_uint(u8_unit(u)) == __float_as_uint(v) ? (int)u : -1;
}

// Bytes the segment's region holds in its `kind` form (unpack) or at most (pack: the fp32 size).
__device__ __forceinline__ unsigned long long region_bytes(const b200ocl_snapshot_segment& s, bool packed_form) {
  return (packed_form && s.kind == B200OCL_SNAP_U8) ? s.bytes / 4 : s.bytes;
}

__device__ __forceinline__ bool segment_ok(const b200ocl_snapshot_segment& s, unsigned long long staging_bytes,
                                           bool packed_form) {
  if (s.kind != B200OCL_SNAP_COPY && s.kind != B200OCL_SNAP_U8) return false;
  if (s.kind == B200OCL_SNAP_U8 && (s.bytes & 3)) return false;
  if (s.bytes != 0 && s.ptr == 0) return false;
  const unsigned long long r = region_bytes(s, packed_form);
  return r <= staging_bytes && s.offset <= staging_bytes - r;
}

__device__ __forceinline__ void copy_bytes(unsigned char* dst, const unsigned char* src, unsigned long long bytes,
                                           size_t tid, size_t nth) {
  size_t done = 0;
  if (((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src)) & 15) == 0) {
    const size_t n16 = bytes / 16;
    const uint4* s = reinterpret_cast<const uint4*>(src);
    uint4* d = reinterpret_cast<uint4*>(dst);
    for (size_t i = tid; i < n16; i += nth) d[i] = s[i];
    done = n16 * 16;
  }
  for (size_t i = done + tid; i < bytes; i += nth) dst[i] = src[i];
}

// fallback = 0: copy COPY segments, encode U8 segments (a rejected value is written as byte 0 and counted);
// fallback = 1: store the fp32 rows of every U8 segment whose counter the first launch left non-zero.
__global__ void __launch_bounds__(SNAP_THREADS) snapshot_pack_kernel(const b200ocl_snapshot_segment* __restrict__ table,
                                                                     int n, unsigned char* __restrict__ staging,
                                                                     unsigned long long staging_bytes,
                                                                     int* __restrict__ counters, int fallback) {
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (size_t)gridDim.x * blockDim.x;
  for (int si = 0; si < n; ++si) {
    const b200ocl_snapshot_segment seg = table[si];
    if (!segment_ok(seg, staging_bytes, false)) {
      if (!fallback && tid == 0) atomicAdd(counters + n, 1);
      continue;
    }
    const bool u8 = seg.kind == B200OCL_SNAP_U8;
    unsigned char* dst = staging + seg.offset;
    if (fallback) {
      if (u8 && counters[si] != 0) copy_bytes(dst, reinterpret_cast<const unsigned char*>(seg.ptr), seg.bytes, tid, nth);
      continue;
    }
    if (!u8) {
      copy_bytes(dst, reinterpret_cast<const unsigned char*>(seg.ptr), seg.bytes, tid, nth);
      continue;
    }
    const float* src = reinterpret_cast<const float*>(seg.ptr);
    const size_t count = seg.bytes / 4;
    int bad = 0;
    size_t done = 0;
    if (((reinterpret_cast<uintptr_t>(src) & 15) | (reinterpret_cast<uintptr_t>(dst) & 3)) == 0) {
      const size_t n4 = count / 4;
      for (size_t i = tid; i < n4; i += nth) {
        const float4 v = reinterpret_cast<const float4*>(src)[i];
        const int a = snap_encode(v.x), b = snap_encode(v.y), c = snap_encode(v.z), d = snap_encode(v.w);
        bad += (a < 0) + (b < 0) + (c < 0) + (d < 0);
        reinterpret_cast<uchar4*>(dst)[i] = make_uchar4(a < 0 ? 0 : a, b < 0 ? 0 : b, c < 0 ? 0 : c, d < 0 ? 0 : d);
      }
      done = n4 * 4;
    }
    for (size_t i = done + tid; i < count; i += nth) {
      const int a = snap_encode(src[i]);
      bad += a < 0;
      dst[i] = (unsigned char)(a < 0 ? 0 : a);
    }
    if (bad) atomicAdd(counters + si, bad);
  }
}

__global__ void __launch_bounds__(SNAP_THREADS)
    snapshot_unpack_kernel(const b200ocl_snapshot_segment* __restrict__ table, int n,
                           const unsigned char* __restrict__ staging, unsigned long long staging_bytes,
                           int* __restrict__ counters) {
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (size_t)gridDim.x * blockDim.x;
  for (int si = 0; si < n; ++si) {
    const b200ocl_snapshot_segment seg = table[si];
    if (!segment_ok(seg, staging_bytes, true)) {
      if (tid == 0) atomicAdd(counters + n, 1);
      continue;
    }
    const unsigned char* src = staging + seg.offset;
    if (seg.kind == B200OCL_SNAP_COPY) {
      copy_bytes(reinterpret_cast<unsigned char*>(seg.ptr), src, seg.bytes, tid, nth);
      continue;
    }
    float* dst = reinterpret_cast<float*>(seg.ptr);
    const size_t count = seg.bytes / 4;
    size_t done = 0;
    if (((reinterpret_cast<uintptr_t>(dst) & 15) | (reinterpret_cast<uintptr_t>(src) & 3)) == 0) {
      const size_t n4 = count / 4;
      for (size_t i = tid; i < n4; i += nth) {
        const uchar4 u = reinterpret_cast<const uchar4*>(src)[i];
        reinterpret_cast<float4*>(dst)[i] = make_float4(u8_unit(u.x), u8_unit(u.y), u8_unit(u.z), u8_unit(u.w));
      }
      done = n4 * 4;
    }
    for (size_t i = done + tid; i < count; i += nth) dst[i] = u8_unit(src[i]);
  }
}

int snapshot_blocks() { return 4 * sm_count(); }

}  // namespace
}  // namespace b200ocl

size_t b200ocl_snapshot_workspace_bytes(int n_segments) {
  if (n_segments < 0) return 0;
  return b200ocl::align_up(((size_t)n_segments + 1) * sizeof(int), 256);
}

int b200ocl_snapshot_pack(const b200ocl_snapshot_segment* table, int n_segments, void* staging, size_t staging_bytes,
                          void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(n_segments >= 0, "need n_segments >= 0");
  const int rc = check_workspace(__func__, workspace, workspace_bytes, b200ocl_snapshot_workspace_bytes(n_segments));
  if (rc != B200OCL_OK) return rc;
  B200OCL_CUDA(cudaMemsetAsync(workspace, 0, ((size_t)n_segments + 1) * sizeof(int), stream));
  if (n_segments == 0) return B200OCL_OK;
  B200OCL_CHECK_ARG(table && staging, "null pointer");
  int* counters = static_cast<int*>(workspace);
  unsigned char* st = static_cast<unsigned char*>(staging);
  B200OCL_PROF("snapshot_pack", 0, stream);
  snapshot_pack_kernel<<<snapshot_blocks(), SNAP_THREADS, 0, stream>>>(table, n_segments, st, staging_bytes, counters, 0);
  B200OCL_LAUNCHED();
  B200OCL_PROF("snapshot_pack_fallback", 0, stream);
  snapshot_pack_kernel<<<snapshot_blocks(), SNAP_THREADS, 0, stream>>>(table, n_segments, st, staging_bytes, counters, 1);
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}

int b200ocl_snapshot_unpack(const b200ocl_snapshot_segment* table, int n_segments, const void* staging,
                            size_t staging_bytes, void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace b200ocl;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200OCL_CHECK_ARG(n_segments >= 0, "need n_segments >= 0");
  const int rc = check_workspace(__func__, workspace, workspace_bytes, b200ocl_snapshot_workspace_bytes(n_segments));
  if (rc != B200OCL_OK) return rc;
  B200OCL_CUDA(cudaMemsetAsync(workspace, 0, ((size_t)n_segments + 1) * sizeof(int), stream));
  if (n_segments == 0) return B200OCL_OK;
  B200OCL_CHECK_ARG(table && staging, "null pointer");
  B200OCL_PROF("snapshot_unpack", 0, stream);
  snapshot_unpack_kernel<<<snapshot_blocks(), SNAP_THREADS, 0, stream>>>(
      table, n_segments, static_cast<const unsigned char*>(staging), staging_bytes, static_cast<int*>(workspace));
  B200OCL_LAUNCHED();
  return B200OCL_OK;
}
