// Library plumbing: version, error string, launch accounting, device queries.
#include "common.cuh"
#include "../../include/b200asr.h"
#include <stdarg.h>
#include <atomic>

namespace b200asr {

static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

static int query_attr(cudaDeviceAttr attr, int fallback) {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return fallback; }
    if (cudaDeviceGetAttribute(&v, attr, dev) != cudaSuccess) { cudaGetLastError(); return fallback; }
    return v > 0 ? v : fallback;
}
// H100 (SXM) defaults when no device is visible (host-only planning / symbol tests)
int sm_count() { return query_attr(cudaDevAttrMultiProcessorCount, 132); }
int max_optin_smem() { return query_attr(cudaDevAttrMaxSharedMemoryPerBlockOptin, 232448); }

}  // namespace b200asr

extern "C" int b200asr_version(void) { return B200ASR_VERSION; }
extern "C" const char* b200asr_last_error(void) { return b200asr::g_err; }
extern "C" unsigned long long b200asr_launch_count(void) { return b200asr::g_launches.load(); }
extern "C" void b200asr_launch_count_reset(void) { b200asr::g_launches.store(0); }
extern "C" int b200asr_device_sm_count(void) { return b200asr::sm_count(); }
