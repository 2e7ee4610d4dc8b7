// Library-wide C ABI plumbing: version, thread-local error text, device check; host helpers every kernel file uses.
#include "ezr_common.cuh"
#include "ptx.cuh"
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

// ---------------------------------------------------------- tensor maps ----
// encode_tmap_2d_bf16 (declared in ptx.cuh): the GEMMs, attention, the dense forms and the int8 scan all use it.
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int encode_tmap_2d_bf16(CUtensorMap* map, const void* base, uint64_t cols, uint64_t rows, uint64_t row_stride_elems,
                        uint32_t box_cols, uint32_t box_rows, int swizzle_bytes) {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        EZR_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres));
        if (qres != cudaDriverEntryPointSuccess || !sym) {
            set_error("cuTensorMapEncodeTiled not available from the driver");
            return EZR_ERR_CUDA;
        }
        fn = reinterpret_cast<PFN_encodeTiled>(sym);
    }
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {row_stride_elems * 2};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE,
                    swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d): cols=%llu rows=%llu stride=%llu box=%ux%u", (int)r,
                  (unsigned long long)cols, (unsigned long long)rows, (unsigned long long)row_stride_elems, box_cols,
                  box_rows);
        return EZR_ERR_CUDA;
    }
    return EZR_OK;
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
