// Library-wide C ABI plumbing: version, thread-local error text, device check.
#include "ezr_common.cuh"
#include "../../include/easyrag_b200.h"
#include <stdarg.h>
#include <utility>
#include <vector>

namespace ezr {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

const char* get_error() { return g_err; }

int sm_count() {
    static int cached = 0;
    if (cached) return cached;
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
    cached = n;
    return n;
}

// ------------------------------------------------------------- profiler ----
// Optional CUDA-event timing of individual kernels on the stream they are launched on
// (bench.py's roofline numbers).  Off by default: no events, no overhead.
struct ProfSlot {
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev;
    size_t used = 0;
};
static bool g_prof_on = false;
unsigned long long g_launches = 0;
void count_launch() { __atomic_fetch_add(&g_launches, 1ull, __ATOMIC_RELAXED); }

static ProfSlot g_prof[EZR_PROF_COUNT];

bool prof_begin(int slot, cudaStream_t st) {
    if (!g_prof_on || slot < 0 || slot >= EZR_PROF_COUNT) return false;
    ProfSlot& s = g_prof[slot];
    if (s.used == s.ev.size()) {
        cudaEvent_t a, b;
        if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) return false;
        s.ev.emplace_back(a, b);
    }
    cudaEventRecord(s.ev[s.used].first, st);
    return true;
}

void prof_end(int slot, cudaStream_t st, bool began) {
    if (!began) return;
    ProfSlot& s = g_prof[slot];
    cudaEventRecord(s.ev[s.used].second, st);
    s.used++;
}

}  // namespace ezr

extern "C" {

int ezr_profile_enable(int32_t on) {
    ezr::g_prof_on = on != 0;
    return EZR_OK;
}

long long ezr_launch_count(void) { return (long long)__atomic_load_n(&ezr::g_launches, __ATOMIC_RELAXED); }

int ezr_profile_reset(void) {
    for (auto& s : ezr::g_prof) s.used = 0;
    return EZR_OK;
}

int ezr_profile_read(int32_t slot, double* total_ms, int32_t* launches) {
    EZR_CHECK_ARG(slot >= 0 && slot < EZR_PROF_COUNT, "profile_read: bad slot %d", slot);
    EZR_CHECK_ARG(total_ms && launches, "profile_read: NULL output");
    ezr::ProfSlot& s = ezr::g_prof[slot];
    double sum = 0;
    for (size_t i = 0; i < s.used; ++i) {
        EZR_CUDA(cudaEventSynchronize(s.ev[i].second));
        float ms = 0;
        EZR_CUDA(cudaEventElapsedTime(&ms, s.ev[i].first, s.ev[i].second));
        sum += ms;
    }
    *total_ms = sum;
    *launches = (int32_t)s.used;
    return EZR_OK;
}

int ezr_version(void) { return 100; }   // 0.1.0

const char* ezr_last_error(void) { return ezr::get_error(); }

int ezr_device_check(void) {
    int dev = 0, major = 0, minor = 0;
    EZR_CUDA(cudaGetDevice(&dev));
    EZR_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    EZR_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    if (major != 9 || minor != 0) {
        ezr::set_error("easyrag_b200 is built for sm_90a only; device %d is sm_%d%d", dev, major, minor);
        return EZR_ERR_ARCH;
    }
    return EZR_OK;
}

}  // extern "C"
