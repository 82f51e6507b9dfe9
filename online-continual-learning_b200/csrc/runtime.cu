// runtime.cu -- error string, launch counter, device properties.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "common.cuh"

namespace b200ocl {

static thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_workspace(const char* entry, const void* ws, size_t ws_bytes, size_t need) {
  if (ws && !(reinterpret_cast<uintptr_t>(ws) & 255) && ws_bytes >= need) return B200OCL_OK;
  set_error("%s: workspace missing, misaligned or smaller than %zu bytes", entry, need);
  return B200OCL_EWORKSPACE;
}

bool g_prof_on = false;
namespace {
struct ProfRec {
  const char* name;
  double work;
  cudaEvent_t a, b;
  bool open;
};
std::vector<ProfRec> g_recs;
cudaStream_t g_prof_stream = nullptr;
struct ProfAgg {
  std::string name;
  double ms, work;
  int count;
};
std::vector<ProfAgg> g_agg;
}  // namespace

void prof_begin(const char* kernel_class, double work, cudaStream_t stream) {
  ProfRec r{kernel_class, work, nullptr, nullptr, true};
  if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) return;
  cudaEventRecord(r.a, stream);
  g_prof_stream = stream;
  g_recs.push_back(r);
}

void prof_end() {
  if (g_recs.empty() || !g_recs.back().open) return;
  cudaEventRecord(g_recs.back().b, g_prof_stream);
  g_recs.back().open = false;
}

// The SM count every launch geometry, plan and workspace size is derived from.  B200OCL_SM_COUNT=n plans for n SMs
// instead of the device's count (an H100 PCIe's 114, a MIG slice's 16 or 60), read once per device so a process never
// mixes two counts.  It only goes down: bn_bwd_fused_kernel and supcon_fused_kernel wait on each other across their
// CTAs, one per SM, and a grid planned for more SMs than the device has need not be resident at once.  _native.lib()
// refuses a value outside [1, device count] before anything launches; the clamp here is the last line of defence.
static int planned_sms(int device_sms) {
  if (const char* e = getenv("B200OCL_SM_COUNT")) {
    const long v = strtol(e, nullptr, 10);
    if (v >= 1 && v < device_sms) return (int)v;
  }
  return device_sms;
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  // no device (host-only plan queries): plan for 148 SMs, or fewer when asked
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return planned_sms(148);
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 148;
    cached[dev] = planned_sms(n);
  }
  return cached[dev];
}

}  // namespace b200ocl

extern "C" {
const char* b200ocl_last_error(void) { return b200ocl::g_err; }
int b200ocl_version(void) { return 100; }
uint64_t b200ocl_launch_count(void) { return b200ocl::g_launches.load(std::memory_order_relaxed); }
int b200ocl_sm_count(void) { return b200ocl::sm_count(); }

void b200ocl_profile_begin(void) {
  using namespace b200ocl;
  for (auto& r : g_recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  g_recs.clear();
  g_agg.clear();
  g_prof_on = true;
}

int b200ocl_profile_end(void) {
  using namespace b200ocl;
  g_prof_on = false;
  cudaDeviceSynchronize();
  g_agg.clear();
  FILE* dump = nullptr;
  if (const char* path = getenv("B200OCL_PROF_DUMP")) dump = fopen(path, "a");   // one line per launch
  for (size_t i = 0; i < g_recs.size(); ++i) {
    auto& r = g_recs[i];
    float ms = 0.f;
    if (r.open || cudaEventElapsedTime(&ms, r.a, r.b) != cudaSuccess) ms = 0.f;
    if (dump) {
      // 4th column: idle time on the stream between the previous recorded launch and this one
      float gap = 0.f;
      if (i > 0 && !g_recs[i - 1].open && cudaEventElapsedTime(&gap, g_recs[i - 1].b, r.a) != cudaSuccess) gap = 0.f;
      fprintf(dump, "%s,%.1f,%.3f,%.3f\n", r.name, r.work, ms * 1e3, gap * 1e3);
    }
    bool found = false;
    for (auto& a : g_agg)
      if (a.name == r.name) { a.ms += ms; a.work += r.work; a.count += 1; found = true; break; }
    if (!found) g_agg.push_back({r.name, (double)ms, r.work, 1});
  }
  for (auto& r : g_recs) {
    cudaEventDestroy(r.a);
    cudaEventDestroy(r.b);
  }
  if (dump) fclose(dump);
  g_recs.clear();
  (void)cudaGetLastError();
  return (int)g_agg.size();
}

int b200ocl_profile_get(int k, char* name, int name_len, double* ms, int* launches, double* work) {
  using namespace b200ocl;
  if (k < 0 || k >= (int)g_agg.size() || !name || name_len < 1) return B200OCL_EINVAL;
  strncpy(name, g_agg[k].name.c_str(), name_len - 1);
  name[name_len - 1] = 0;
  if (ms) *ms = g_agg[k].ms;
  if (launches) *launches = g_agg[k].count;
  if (work) *work = g_agg[k].work;
  return B200OCL_OK;
}
}
