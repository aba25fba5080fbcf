// coach_b200/csrc/core.cu -- error string, launch counter, device info, tuning knobs for libcoach_b200.so
#include <stdarg.h>
#include <string.h>

#include <atomic>
#include <map>
#include <mutex>
#include <string>

#include "common.cuh"

namespace cb200 {

static thread_local char g_error[512] = "";
static std::atomic<int64_t> g_launches{0};
static std::mutex g_tune_mutex;
static std::map<std::string, int> g_tune;

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

// cb200_last_dispatch: the GEMM entry points store static names here, the string is only assembled when asked for
static thread_local const char* g_dispatch_kernel = "";
static thread_local const char* g_dispatch_fetch = nullptr;
static thread_local const char* g_dispatch_reduce = nullptr;
static thread_local char g_dispatch[128] = "";

void set_dispatch(const char* kernel, const char* fetch) {
    g_dispatch_kernel = kernel;
    g_dispatch_fetch = fetch;
    g_dispatch_reduce = nullptr;
}
void set_dispatch_reduce(const char* reduce) { g_dispatch_reduce = reduce; }

int sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cached[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached[dev] = n;
    }
    return cached[dev];
}

int tune_get(const char* key, int dflt, int lo, int hi) {
    std::lock_guard<std::mutex> g(g_tune_mutex);
    auto it = g_tune.find(key);
    if (it == g_tune.end()) return dflt;
    int v = it->second;
    if (v < lo) v = lo;
    if (v > hi) v = hi;
    return v;
}

}  // namespace cb200

extern "C" {

int cb200_abi_version(void) { return CB200_ABI_VERSION; }
const char* cb200_last_error(void) { return cb200::g_error; }
const char* cb200_last_dispatch(void) {
    snprintf(cb200::g_dispatch, sizeof(cb200::g_dispatch), "%s%s%s%s%s", cb200::g_dispatch_kernel,
             cb200::g_dispatch_fetch ? "/" : "", cb200::g_dispatch_fetch ? cb200::g_dispatch_fetch : "",
             cb200::g_dispatch_reduce ? "+" : "", cb200::g_dispatch_reduce ? cb200::g_dispatch_reduce : "");
    return cb200::g_dispatch;
}
int64_t cb200_launch_count(void) { return cb200::g_launches.load(std::memory_order_relaxed); }

int cb200_tune(const char* key, int value) {
    if (!key) return CB200_ERR_INVALID_ARGUMENT;
    if (strcmp(key, "gemm_persistent") == 0) {
        cb200::set_error("cb200_tune: \"gemm_persistent\" was removed (the persistent tiled-GEMM schedule no longer exists)");
        return CB200_ERR_INVALID_ARGUMENT;
    }
    std::lock_guard<std::mutex> g(cb200::g_tune_mutex);
    cb200::g_tune[key] = value;
    return CB200_OK;
}

int cb200_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0;
    CB200_CUDA(cudaGetDevice(&dev));
    if (sm_count) CB200_CUDA(cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, dev));
    if (cc_major) CB200_CUDA(cudaDeviceGetAttribute(cc_major, cudaDevAttrComputeCapabilityMajor, dev));
    if (cc_minor) CB200_CUDA(cudaDeviceGetAttribute(cc_minor, cudaDevAttrComputeCapabilityMinor, dev));
    return CB200_OK;
}

}  // extern "C"
