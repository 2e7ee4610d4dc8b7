// Common device/host helpers for the easyrag_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/easyrag_b200.h"

namespace ezr {

// ---------------------------------------------------------------- errors ----
// status codes: ezr_status in include/easyrag_b200.h

void set_error(const char* fmt, ...);
const char* get_error();

#define EZR_CHECK_ARG(cond, ...)                         \
    do {                                                 \
        if (!(cond)) {                                   \
            ::ezr::set_error(__VA_ARGS__);               \
            return EZR_ERR_INVALID;               \
        }                                                \
    } while (0)

#define EZR_CUDA(call)                                                                   \
    do {                                                                                 \
        cudaError_t e__ = (call);                                                        \
        if (e__ != cudaSuccess) {                                                        \
            ::ezr::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__),    \
                             __FILE__, __LINE__);                                        \
            return EZR_ERR_CUDA;                                                  \
        }                                                                                \
    } while (0)

// every kernel launch of the library passes through here: the launch counter behind ezr_launch_count()
void count_launch();
#define EZR_LAUNCH_CHECK()              \
    do {                                \
        ::ezr::count_launch();          \
        EZR_CUDA(cudaGetLastError());   \
    } while (0)

inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

int sm_count();

// kernel timing slots (include/easyrag_b200.h: ezr_profile_*)
bool prof_begin(int slot, cudaStream_t st);
void prof_end(int slot, cudaStream_t st, bool began);
struct ProfScope {
    int slot; cudaStream_t st; bool began;
    ProfScope(int slot_, cudaStream_t st_) : slot(slot_), st(st_), began(prof_begin(slot_, st_)) {}
    ~ProfScope() { prof_end(slot, st, began); }
};

// ------------------------------------------------------- score ordering ----
// Canonical rank order used everywhere (SURVEY.md 8(c)): score descending, then
// document id DESCENDING -- identical to numpy ``argsort(kind="stable")[::-1]``.
template <typename S>
__device__ __forceinline__ bool better(S sa, int ia, S sb, int ib) {
    return sa > sb || (sa == sb && ia > ib);
}

template <typename S> struct ScoreTraits;
template <> struct ScoreTraits<float> {
    __device__ static __forceinline__ float lowest() { return -INFINITY; }
};
template <> struct ScoreTraits<double> {
    __device__ static __forceinline__ double lowest() { return -INFINITY; }
};

__device__ __forceinline__ float shfl_idx(float v, int src) { return __shfl_sync(0xffffffffu, v, src); }
__device__ __forceinline__ int shfl_idx(int v, int src) { return __shfl_sync(0xffffffffu, v, src); }
__device__ __forceinline__ double shfl_idx(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }
__device__ __forceinline__ float shfl_up1(float v) { return __shfl_up_sync(0xffffffffu, v, 1); }
__device__ __forceinline__ int shfl_up1(int v) { return __shfl_up_sync(0xffffffffu, v, 1); }
__device__ __forceinline__ double shfl_up1(double v) { return __shfl_up_sync(0xffffffffu, v, 1); }

// ------------------------------------------------------------ WarpTopK ----
// A warp keeps its best K<=32 (score,id) pairs sorted across lanes: lane i holds
// the i-th best.  Candidates are offered 32 at a time (one per lane); a ballot
// finds the few that beat the current K-th, and each of those is inserted with a
// shuffle-shift.  After warm-up almost no candidate passes the ballot, so the
// steady-state cost is one compare + one ballot per 32 candidates.
template <typename S>
struct WarpTopK {
    S s;      // lane i: score of the i-th best
    int id;   // lane i: its id (-1 = empty)
    int k;
    S kth_s;  // broadcast copy of lane k-1
    int kth_id;

    __device__ __forceinline__ void init(int k_) {
        k = k_;
        s = ScoreTraits<S>::lowest();
        id = -1;
        kth_s = s;
        kth_id = -1;
    }

    // every lane calls with its own candidate; ``valid`` = lane has a candidate
    __device__ __forceinline__ void offer(S cs, int cid, bool valid) {
        const int lane = threadIdx.x & 31;
        unsigned m = __ballot_sync(0xffffffffu, valid && better<S>(cs, cid, kth_s, kth_id));
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            const S bs = shfl_idx(cs, src);
            const int bid = shfl_idx(cid, src);
            // the threshold may have risen since the ballot
            if (!better<S>(bs, bid, kth_s, kth_id)) continue;
            const bool mine_better = better<S>(s, id, bs, bid);
            const int pos = __popc(__ballot_sync(0xffffffffu, mine_better));
            const S us = shfl_up1(s);
            const int uid = shfl_up1(id);
            if (lane == pos) { s = bs; id = bid; }
            else if (lane > pos) { s = us; id = uid; }
            kth_s = shfl_idx(s, k - 1);
            kth_id = shfl_idx(id, k - 1);
        }
    }
};

}  // namespace ezr
