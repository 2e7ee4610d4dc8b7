// Dense cosine top-k over an int8 copy of the corpus: a certified int8 candidate pass, then exact rescoring from
// the bf16 rows.  The result is the canonical top-k (score descending, id descending) under
//
//   rescore(q, r) = acc_{dim-1},  acc_0 = q_0 r_0,  acc_i = __fadd_rn(acc_{i-1}, __fmul_rn(q_i, r_i)),
//
// an fp32 dot product of the bf16 query and the bf16 row in increasing coordinate order without FMA contraction
// (`-0.0` is returned as `+0.0`), taken over EVERY row that passes the filter.  Separate float32 multiplies and adds
// in numpy or eager torch reproduce it bit for bit.
//
// Quantization (per row, symmetric): scale = fl(max|x_i| / 127), R_i = clamp(rint(fl(x_i / scale)), -127, 127);
// a zero row has scale 0 and R = 0.  Stored with the row: e_r and n_r, the fp64 values of ||x - scale R||_2 and
// ||scale R||_2 rounded up to fp32.  The fp64 sums may fall short of the real norms by a relative dim 2^-53; the
// (1 + 2^-20) factor of D_q below covers that, so e_r and n_r enter the bound as if they were upper bounds.  The index keeps e_max = max e_r and n_max = max n_r.  Queries are
// quantized the same way on every call, giving a_q, Q, e_q, n_q.
//
// The bound.  Let S = sum Q_i R_i (exact in int32, and exact as a float: |S| <= 1024 * 127^2 < 2^24), and
//   s^ = fl(fl(a_q a_r) * (float)S)                        (what the scan computes per (query, row)),
//   s  = q . x  (the real dot product),  s' = rescore(q, x).
// (1) rescore: dim rounded operations per term, u = 2^-24, gamma_n = n u / (1 - n u), underflow of a product adds at
//     most 2^-150 (subnormal additions are exact):  |s' - s| <= gamma_dim ||q|| ||x|| + dim 2^-149.
//     ||q|| <= n_q + e_q and ||x|| <= n_max + e_max (triangle inequality), so no separate norm is stored.
// (2) quantization, Cauchy-Schwarz on q = a_q Q + dq, x = a_r R + dx:
//     |s - a_q a_r S| <= n_q e_max + e_q n_max + e_q e_max.
// (3) s^: fl(a_q a_r) = a_q a_r (1 + d1) + h1, s^ = fl(a_q a_r) S (1 + d2) + h2 with |d| <= u, |h| <= 2^-150, and
//     |a_q a_r S| <= n_q n_max:  |s^ - a_q a_r S| <= (2u + u^2) n_q n_max + 2^-125.
// D_q = (sum of the three) * (1 + 2^-20): the factor covers the fp64 evaluation of D_q and of the fp64 sums behind
// e and n (relative error <= dim 2^-53 each).  D_q is evaluated in fp64 and 2 D_q is stored rounded up to fp32.
//
// Certified candidates.  Let s^_(k) be the k-th largest s^ among the rows that pass the filter.  The k rows with the
// largest s^ have s' >= s^_(k) - D_q, so the k-th largest s' is >= s^_(k) - D_q and every answer row a has
// s^_a >= s'_a - D_q >= s^_(k) - 2 D_q.  Any T <= s^_(k) therefore admits every answer row through s^ >= T - 2 D_q.
// The scan uses T = max(the thread's own KT-th best s^ over the filtered-in rows it has seen (KT >= k), the
// per-query bound those values raise across work units); both are k-th bests of subsets.  The threshold T - 2 D_q
// is formed with a downward-rounded subtraction, so it never exceeds the real value.
//
// Kernels.
//   dense_s8_prep_kernel    one warp per query: quantize, 2 D_q, reset the per-query state.
//   dense_s8_scan_kernel    the layout of dense_wgmma_kernel's 64-query / 128-row form (dense_tc.cu): a TMA
//                           producer warpgroup, the 64-query int8 block resident in shared memory (128-byte swizzled
//                           64 x 128-byte boxes), a ring of 128-row corpus tiles, wgmma.m64n128k32.s32.s8.s8, and
//                           persistent CTAs over (split, query block) units.  The epilogue appends each row that can
//                           still be an answer to its query's candidate buffer (atomic slot; counting past the
//                           capacity marks an overflow, after which the query emits nothing more: a thread stops at
//                           its first slot past the capacity, the others when they read the count at their next
//                           tile).  Each (query, row) is scored once, so no row is emitted twice.
//   dense_s8_rescore_kernel one CTA per query: rescore the candidates, canonical top-k (select.cuh); queries whose
//                           buffer overflowed take the result of the full scan instead.
// Overflowed queries, and every call with k > 16, are answered by the full scan of dense.cu (score rows with the
// rescore arithmetic + ezr_select_rows) for those queries only.  The capacity never changes a result.
#include "ezr_common.cuh"
#include "ptx.cuh"
#include "select.cuh"
#include "dense_tc.h"
#include "../../include/easyrag_b200.h"

namespace ezr {

constexpr int S8_TN = 128;                           // corpus rows per tile (wgmma N)
constexpr int S8_KC = 128;                           // int8 per k-chunk = one 128-byte swizzle row
constexpr int S8_MAXD = 1024;
constexpr int S8_KMAX = 16;
constexpr int S8_A_BOX_BYTES = 64 * S8_KC;           // 8192: 64 queries x one k-chunk
constexpr int S8_B_STAGE_BYTES = S8_TN * S8_KC;      // 16384
constexpr int S8_MAX_STAGES = 32;
constexpr int S8_SMEM_LIMIT = 232448;
constexpr int S8_DEFAULT_CAP = 4096;                 // candidates per query

static thread_local int g_s8_cap = S8_DEFAULT_CAP;   // ezr_dense_s8_set_capacity (per host thread, like the kernel choice)

// floats <-> ints with the same order (for atomicMax on signed ints); an involution
__device__ __forceinline__ int f2ord(float f) {
    const int b = __float_as_int(f);
    return b >= 0 ? b : b ^ 0x7fffffff;
}
__device__ __forceinline__ float ord2f(int o) { return __int_as_float(o >= 0 ? o : o ^ 0x7fffffff); }

// ---------------------------------------------------------------- quantizer ----
// One warp quantizes one bf16 row of `dim` values.  Returns (in every lane) e = ||x - scale R||, n = ||scale R||
// in fp64.
__device__ __forceinline__ void quant_row_warp(const __nv_bfloat16* __restrict__ x, int dim, int8_t* __restrict__ out,
                                               float& scale_out, double& e2_out, double& n2_out) {
    const int lane = threadIdx.x & 31;
    float m = 0.f;
    for (int i = lane; i < dim; i += 32) m = fmaxf(m, fabsf(__bfloat162float(x[i])));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    const float scale = __fdiv_rn(m, 127.f);
    double e2 = 0.0, n2 = 0.0;
    for (int i = lane; i < dim; i += 32) {
        const float v = __bfloat162float(x[i]);
        float r = 0.f;
        if (scale > 0.f) r = fminf(fmaxf(rintf(__fdiv_rn(v, scale)), -127.f), 127.f);
        out[i] = (int8_t)(int)r;
        const double a = (double)scale * (double)r;          // exact: 24-bit x 8-bit significands
        const double d = (double)v - a;
        e2 += d * d;
        n2 += a * a;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        e2 += __shfl_xor_sync(0xffffffffu, e2, o);
        n2 += __shfl_xor_sync(0xffffffffu, n2, o);
    }
    scale_out = scale;
    e2_out = e2;
    n2_out = n2;
}

// Rows: int8 rows + scale, e_r, n_r; maxima[0] / [1] (e_max / n_max, non-negative floats) raised atomically.
__global__ void dense_s8_quantize_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, int64_t n_rows, int dim,
                                         int8_t* __restrict__ out, int64_t ldo, float* __restrict__ scale,
                                         float* __restrict__ err, float* __restrict__ norm, float* maxima) {
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    float s;
    double e2, n2;
    quant_row_warp(x + row * ldx, dim, out + row * ldo, s, e2, n2);
    if ((threadIdx.x & 31) == 0) {
        const float e = __double2float_ru(sqrt(e2)), n = __double2float_ru(sqrt(n2));
        scale[row] = s;
        err[row] = e;
        norm[row] = n;
        if (maxima) {
            atomicMax(reinterpret_cast<int*>(maxima), __float_as_int(e));     // non-negative floats order as ints
            atomicMax(reinterpret_cast<int*>(maxima) + 1, __float_as_int(n));
        }
    }
}

// Queries: int8 rows (ld = dim) + a_q and the margin 2 D_q; resets the per-query scan state.
__global__ void dense_s8_prep_kernel(const __nv_bfloat16* __restrict__ q, int64_t ldq, int n_q, int dim,
                                     const float* __restrict__ maxima, int8_t* __restrict__ q8,
                                     float* __restrict__ q_scale, float* __restrict__ q_margin,
                                     int32_t* __restrict__ bound, int32_t* __restrict__ cand_cnt) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_q) return;
    float s;
    double e2, n2;
    quant_row_warp(q + (int64_t)row * ldq, dim, q8 + (int64_t)row * dim, s, e2, n2);
    if ((threadIdx.x & 31) == 0) {
        const double u = 0x1p-24;
        const double eq = (double)__double2float_ru(sqrt(e2)), nq = (double)__double2float_ru(sqrt(n2));
        const double emax = (double)maxima[0], nmax = (double)maxima[1];
        const double gam = dim * u / (1.0 - dim * u);
        double D = nq * emax + eq * nmax + eq * emax                 // quantization (Cauchy-Schwarz)
                   + gam * (nq + eq) * (nmax + emax) + dim * 0x1p-149   // rescore rounding and underflow
                   + (2 * u + u * u) * nq * nmax + 0x1p-125;            // rounding of s^
        D *= 1.0 + 0x1p-20;
        q_scale[row] = s;
        q_margin[row] = __double2float_ru(2.0 * D);
        bound[row] = f2ord(-INFINITY);
        cand_cnt[row] = 0;
    }
}

// ---------------------------------------------------------------- scan ----
struct S8Params {
    int64_t n_rows;
    int rows_per_slice;   // multiple of S8_TN
    int n_queries;
    int kchunks;          // dim / 128
    int n_stages;
    int n_slices;
    int n_qblocks;
    int cap;
    const int32_t* doc_group;
    const int32_t* q_group;
    const float* row_scale;
    const float* q_scale;
    const float* q_margin;
    int32_t* bound;       // [n_queries] f2ord of a proven lower bound of s^_(k)
    int32_t* cand_cnt;    // [n_queries] candidates appended (> cap: overflowed)
    int32_t* cand_id;     // [n_queries][cap] local row ids
};

struct S8Barriers {
    uint64_t a_full;
    uint64_t a_empty;
    uint64_t b_full[S8_MAX_STAGES];
    uint64_t b_empty[S8_MAX_STAGES];
};

__device__ __forceinline__ void wgmma_s8_n128(int (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]),
          "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]),
          "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]),
          "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]),
          "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]),
          "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]),
          "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]),
          "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(da), "l"(db), "r"(acc));
}

__device__ __forceinline__ void fence_regs_i(int (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

// One query row of a thread: the KT best s^ it has seen (values only), the threshold, the margin.
template <int KT>
struct S8Row {
    float ts[KT];
    float margin;     // 2 D_q, rounded up
    float shared;     // the per-query bound last read
    float ethr;       // emit threshold: T - 2 D_q rounded down
    int q, want, published;
    bool active, dirty;
    bool over;        // the query's buffer has overflowed: the full scan answers it, so nothing more is emitted
};

template <int KT>
__device__ __forceinline__ void s8_row_start(S8Row<KT>& L, int q, const S8Params& p, bool filter) {
    L.q = q;
    L.active = q < p.n_queries;
#pragma unroll
    for (int j = 0; j < KT; ++j) L.ts[j] = -INFINITY;
    L.want = (filter && L.active) ? p.q_group[q] : -1;
    L.margin = L.active ? p.q_margin[q] : 0.f;
    L.published = f2ord(-INFINITY);
    L.shared = L.active ? ord2f(*reinterpret_cast<const volatile int32_t*>(p.bound + q)) : -INFINITY;
    L.ethr = __fsub_rd(L.shared, L.margin);
    L.dirty = false;
    L.over = L.active && *reinterpret_cast<const volatile int32_t*>(p.cand_cnt + q) > p.cap;
}

template <int KT>
__device__ __forceinline__ void s8_set_thr(S8Row<KT>& L) {
    const float t = fmaxf(L.ts[KT - 1], L.shared);
    L.ethr = __fsub_rd(t, L.margin);          // -inf stays -inf
}

// this thread's 32 s^ of query row H of a 128-row tile (columns 8 j + 2 (lane % 4) + e, increasing document order)
template <bool FILTER, int KT, int H>
__device__ __forceinline__ void s8_scan_row(const int (&acc)[64], const float (&rs)[32], S8Row<KT>& L, float qs,
                                            int64_t doc0, int64_t left, const S8Params& p) {
    if (!L.active || L.over) return;
    float vals[32];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const float v = __fmul_rn(__fmul_rn(qs, rs[2 * j + e]), (float)acc[4 * j + 2 * H + e]);
            vals[2 * j + e] = v;
            if (8 * j + e < left) mx = fmaxf(mx, v);
        }
    }
    if (!(mx >= L.ethr)) return;
    uint32_t mask = 0;
#pragma unroll
    for (int b = 0; b < 32; ++b) mask |= ((8 * (b >> 1) + (b & 1) < left && vals[b] >= L.ethr) ? 1u : 0u) << b;
    while (mask) {
        const int b = __ffs(mask) - 1;
        mask &= mask - 1;
        const float v = vals[b];
        if (!(v >= L.ethr)) continue;                         // the threshold may have risen inside this batch
        const int64_t doc = doc0 + 8 * (b >> 1) + (b & 1);
        if (FILTER && L.want != -1 && __ldg(p.doc_group + doc) != L.want) continue;
        const int slot = atomicAdd(p.cand_cnt + L.q, 1);
        if (slot >= p.cap) {                                  // the count now marks the overflow
            L.over = true;
            return;
        }
        p.cand_id[(int64_t)L.q * p.cap + slot] = (int)doc;
        if (v > L.ts[KT - 1]) {
            float cv = v;
#pragma unroll
            for (int s = 0; s < KT; ++s) {
                const float fs = L.ts[s];
                const bool sw = cv > fs;
                L.ts[s] = sw ? cv : fs;
                cv = sw ? fs : cv;
            }
            L.dirty = true;
            s8_set_thr<KT>(L);
        }
    }
}

// publish this thread's KT-th best (a k-th best of a subset) and take in what other threads published; `cnt` is the
// query's candidate count read at the start of the tile
template <int KT>
__device__ __forceinline__ void s8_row_sync(S8Row<KT>& L, int seen, int cnt, const S8Params& p) {
    if (!L.active || L.over) return;
    if (cnt > p.cap) {
        L.over = true;
        return;
    }
    if (L.dirty && L.ts[KT - 1] > -INFINITY) {
        const int o = f2ord(L.ts[KT - 1]);
        if (o > L.published && o > seen) atomicMax(p.bound + L.q, o);
        L.published = o;
    }
    L.dirty = false;
    const float sh = ord2f(seen);
    if (sh > L.shared) {
        L.shared = sh;
        s8_set_thr<KT>(L);
    }
}

template <bool FILTER, int KT>
__global__ void __launch_bounds__(256, 1)
dense_s8_scan_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_c,
                     const S8Params p) {
    extern __shared__ unsigned char smem_dyn[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    unsigned char* smem_a = smem;                                              // [kchunks] boxes of 8 KB
    unsigned char* smem_b = smem + (size_t)p.kchunks * S8_A_BOX_BYTES;
    S8Barriers* bars = reinterpret_cast<S8Barriers*>(smem_b + (size_t)p.n_stages * S8_B_STAGE_BYTES);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n_units = p.n_slices * p.n_qblocks;

    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&map_c);
        ptx::prefetch_tensormap(&map_q);
        ptx::mbar_init(&bars->a_full, 1);
        ptx::mbar_init(&bars->a_empty, 1);
        for (int i = 0; i < p.n_stages; ++i) {
            ptx::mbar_init(&bars->b_full[i], 1);
            ptx::mbar_init(&bars->b_empty[i], 1);
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        ptx::regs_dealloc<40>();
        if (threadIdx.x == 0) {
            // ---------------- TMA producer: the query block + corpus tiles of every unit of this CTA
            int stage = 0;
            uint32_t phase = 0;
            int ui = 0;
            for (int u = blockIdx.x; u < n_units; u += gridDim.x, ++ui) {
                const int slice = u / p.n_qblocks;
                const int q0 = (u % p.n_qblocks) * 64;
                const int64_t row_begin = (int64_t)slice * p.rows_per_slice;
                const int64_t row_end = min(p.n_rows, row_begin + p.rows_per_slice);
                const int n_tiles = (int)((row_end - row_begin + S8_TN - 1) / S8_TN);
                ptx::mbar_wait(&bars->a_empty, ((uint32_t)ui & 1u) ^ 1u);
                ptx::mbar_expect_tx(&bars->a_full, (uint32_t)(p.kchunks * S8_A_BOX_BYTES));
                // the tensor maps see an int8 row as 16-bit elements: a 128-byte chunk is 64 of them
                for (int kc = 0; kc < p.kchunks; ++kc)
                    ptx::tma_load_2d_hint(smem_a + (size_t)kc * S8_A_BOX_BYTES, &map_q, &bars->a_full, kc * 64, q0,
                                          ptx::kEvictLast);
                for (int t = 0; t < n_tiles; ++t) {
                    const int row0 = (int)(row_begin + (int64_t)t * S8_TN);
                    for (int kc = 0; kc < p.kchunks; ++kc) {
                        ptx::mbar_wait(&bars->b_empty[stage], phase ^ 1);
                        ptx::mbar_expect_tx(&bars->b_full[stage], S8_B_STAGE_BYTES);
                        ptx::tma_load_2d(smem_b + (size_t)stage * S8_B_STAGE_BYTES, &map_c, &bars->b_full[stage],
                                         kc * 64, row0);
                        if (++stage == p.n_stages) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
    } else {
        // ---------------- consumer warpgroup: the 64 query rows of the block
        ptx::regs_alloc<232>();
        const int wq = warp & 3;
        const bool leader = (threadIdx.x & 127) == 0;
        const uint32_t a_base = ptx::smem_u32(smem_a);
        const uint32_t b_base = ptx::smem_u32(smem_b);
        int stage = 0;
        uint32_t phase = 0;
        int ui = 0;
        for (int u = blockIdx.x; u < n_units; u += gridDim.x, ++ui) {
            const int slice = u / p.n_qblocks;
            const int q0 = (u % p.n_qblocks) * 64;
            const int64_t row_begin = (int64_t)slice * p.rows_per_slice;
            const int64_t row_end = min(p.n_rows, row_begin + p.rows_per_slice);
            const int n_tiles = (int)((row_end - row_begin + S8_TN - 1) / S8_TN);
            const int qr = q0 + wq * 16 + (lane >> 2);           // accumulator fragment rows qr and qr + 8
            S8Row<KT> L0, L1;
            s8_row_start<KT>(L0, qr, p, FILTER);
            s8_row_start<KT>(L1, qr + 8, p, FILTER);
            const float qs0 = L0.active ? p.q_scale[qr] : 0.f;
            const float qs1 = L1.active ? p.q_scale[qr + 8] : 0.f;
            ptx::mbar_wait(&bars->a_full, (uint32_t)ui & 1u);

            for (int t = 0; t < n_tiles; ++t) {
                // the shared bounds are read before the MMAs so the load latency hides under them
                const int seen0 = L0.active ? *reinterpret_cast<const volatile int32_t*>(p.bound + L0.q) : 0;
                const int seen1 = L1.active ? *reinterpret_cast<const volatile int32_t*>(p.bound + L1.q) : 0;
                const int cnt0 = L0.active ? *reinterpret_cast<const volatile int32_t*>(p.cand_cnt + L0.q) : 0;
                const int cnt1 = L1.active ? *reinterpret_cast<const volatile int32_t*>(p.cand_cnt + L1.q) : 0;
                const int64_t doc0 = row_begin + (int64_t)t * S8_TN + (lane & 3) * 2;
                const int64_t left = row_end - doc0;
                float rs[32];
#pragma unroll
                for (int j = 0; j < 16; ++j) {
#pragma unroll
                    for (int e = 0; e < 2; ++e)
                        rs[2 * j + e] = (8 * j + e < left) ? __ldg(p.row_scale + doc0 + 8 * j + e) : 0.f;
                }
                int acc[64];
#pragma unroll
                for (int i = 0; i < 64; ++i) acc[i] = 0;
                int prev = -1;
                for (int kc = 0; kc < p.kchunks; ++kc) {
                    ptx::mbar_wait(&bars->b_full[stage], phase);
                    ptx::wgmma_fence();
#pragma unroll
                    for (int k4 = 0; k4 < S8_KC / 32; ++k4) {
                        const uint64_t da = ptx::make_desc_sw128(a_base + (uint32_t)(kc * S8_A_BOX_BYTES + k4 * 32));
                        const uint64_t db = ptx::make_desc_sw128(b_base + (uint32_t)(stage * S8_B_STAGE_BYTES + k4 * 32));
                        wgmma_s8_n128(acc, da, db, (uint32_t)((kc | k4) != 0));
                    }
                    ptx::wgmma_commit();
                    ptx::wgmma_wait<1>();
                    if (prev >= 0 && leader) ptx::mbar_arrive(&bars->b_empty[prev]);
                    prev = stage;
                    if (++stage == p.n_stages) { stage = 0; phase ^= 1; }
                }
                ptx::wgmma_wait<0>();
                fence_regs_i(acc);
                if (leader) {
                    ptx::mbar_arrive(&bars->b_empty[prev]);
                    if (t == n_tiles - 1) ptx::mbar_arrive(&bars->a_empty);
                }
                s8_row_sync<KT>(L0, seen0, cnt0, p);
                s8_row_sync<KT>(L1, seen1, cnt1, p);
                s8_scan_row<FILTER, KT, 0>(acc, rs, L0, qs0, doc0, left, p);
                s8_scan_row<FILTER, KT, 1>(acc, rs, L1, qs1, doc0, left, p);
            }
            // publish what the last tile raised (units of the same query that start later begin from it)
            s8_row_sync<KT>(L0, f2ord(-INFINITY), 0, p);
            s8_row_sync<KT>(L1, f2ord(-INFINITY), 0, p);
        }
    }
}

// ---------------------------------------------------------------- rescore ----
// Overflowed queries: over_pos[q] = their row in the full-scan results, else -1.
__global__ void dense_s8_overflow_kernel(const int32_t* __restrict__ cand_cnt, int n_q, int cap,
                                         int32_t* __restrict__ over_pos, int32_t* __restrict__ over_list,
                                         int32_t* __restrict__ over_n) {
    __shared__ int n;
    if (threadIdx.x == 0) n = 0;
    __syncthreads();
    for (int q = threadIdx.x; q < n_q; q += blockDim.x) {
        int pos = -1;
        if (cand_cnt[q] > cap) {
            pos = atomicAdd(&n, 1);
            over_list[pos] = q;
        }
        over_pos[q] = pos;
    }
    __syncthreads();
    if (threadIdx.x == 0) *over_n = n;
}

// the overflowed queries' rows (and filter classes), packed for the full scan
__global__ void dense_s8_gather_kernel(const __nv_bfloat16* __restrict__ q, int64_t ldq, int dim,
                                       const int32_t* __restrict__ q_group, const int32_t* __restrict__ over_list,
                                       int n_over, __nv_bfloat16* __restrict__ out, int32_t* __restrict__ out_group) {
    const int i = blockIdx.x;
    if (i >= n_over) return;
    const int src = over_list[i];
    for (int c = threadIdx.x; c < dim; c += blockDim.x) out[(int64_t)i * dim + c] = q[(int64_t)src * ldq + c];
    if (threadIdx.x == 0 && q_group) out_group[i] = q_group[src];
}

constexpr int S8_RESCORE_THREADS = 256;

__global__ void __launch_bounds__(S8_RESCORE_THREADS)
dense_s8_rescore_kernel(const __nv_bfloat16* __restrict__ corpus, int64_t ldc, int dim,
                        const __nv_bfloat16* __restrict__ queries, int64_t ldq, int k, int id_base,
                        const int32_t* __restrict__ cand_cnt, const int32_t* __restrict__ cand_id, int cap,
                        const int32_t* __restrict__ over_pos, const float* __restrict__ fb_scores,
                        const int32_t* __restrict__ fb_ids, const int32_t* __restrict__ fb_counts,
                        float* __restrict__ out_scores, int32_t* __restrict__ out_ids, int32_t* __restrict__ out_counts,
                        int32_t* __restrict__ out_cand) {
    extern __shared__ unsigned char smem_dyn[];
    const int q = blockIdx.x;
    const int cnt = cand_cnt[q];
    if (threadIdx.x == 0 && out_cand) out_cand[q] = cnt;
    const int op = over_pos[q];
    if (op >= 0) {
        for (int i = threadIdx.x; i < k; i += blockDim.x) {
            out_scores[(int64_t)q * k + i] = fb_scores[(int64_t)op * k + i];
            out_ids[(int64_t)q * k + i] = fb_ids[(int64_t)op * k + i];
        }
        if (threadIdx.x == 0 && out_counts) out_counts[q] = fb_counts[op];
        return;
    }
    float* qf = reinterpret_cast<float*>(smem_dyn);                            // [dim]
    SelSmem<float> m = sel_carve<float>(smem_dyn + (size_t)S8_MAXD * 4);
    for (int i = threadIdx.x; i < dim; i += blockDim.x) qf[i] = __bfloat162float(queries[(int64_t)q * ldq + i]);
    sel_init<float>(m);                                                        // (its barrier publishes qf)
    const int n = cnt;                                                         // <= cap: not overflowed
    for (int base = 0; base < n; base += S8_RESCORE_THREADS) {
        const int i = base + threadIdx.x;
        if (i < n) {
            const int row = cand_id[(int64_t)q * cap + i];
            const uint4* r = reinterpret_cast<const uint4*>(corpus + (int64_t)row * ldc);
            float acc = 0.f;
            for (int c = 0; c < dim / 8; ++c) {
                const uint4 w = __ldg(r + c);
                const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&w);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = __bfloat1622float2(h[j]);
                    acc = __fadd_rn(acc, __fmul_rn(qf[8 * c + 2 * j], f.x));
                    acc = __fadd_rn(acc, __fmul_rn(qf[8 * c + 2 * j + 1], f.y));
                }
            }
            sel_push<float>(m, acc + 0.0f, row + id_base);                     // -0.0 -> +0.0
        }
        sel_maybe_flush<float>(m, k);
    }
    sel_compact<float>(m, k);
    // sel_compact pads the buffer only up to the next power of two of what it holds: the slots past the count are
    // written here, id -1, as every top-k route leaves them (the sharded merge reads every slot with an id >= 0)
    const int got = *m.cnt;
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        out_scores[(int64_t)q * k + i] = i < got ? m.ks[i] : -INFINITY;
        out_ids[(int64_t)q * k + i] = i < got ? m.kid[i] : -1;
    }
    if (threadIdx.x == 0 && out_counts) out_counts[q] = got;
}

// ------------------------------------------------------------------ host ----
static size_t s8_rescore_smem() { return (size_t)S8_MAXD * 4 + sel_smem_bytes<float>(); }

struct S8Layout {
    size_t q8, q_scale, q_margin, bound, cand_cnt, cand_id, over_pos, over_list, over_n, g_q, g_group, fb_s, fb_i,
        fb_c, full, total;
};

static S8Layout s8_layout(int64_t n_rows, int dim, int n_q, int k, int cap) {
    S8Layout l;
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o += align_up(bytes, 256); return at; };
    l.q8 = take((size_t)n_q * dim);
    l.q_scale = take((size_t)n_q * 4);
    l.q_margin = take((size_t)n_q * 4);
    l.bound = take((size_t)n_q * 4);
    l.cand_cnt = take((size_t)n_q * 4);
    l.cand_id = take((size_t)n_q * cap * 4);
    l.over_pos = take((size_t)n_q * 4);
    l.over_list = take((size_t)n_q * 4);
    l.over_n = take(4);
    l.g_q = take((size_t)n_q * dim * 2);
    l.g_group = take((size_t)n_q * 4);
    l.fb_s = take((size_t)n_q * k * 4);
    l.fb_i = take((size_t)n_q * k * 4);
    l.fb_c = take((size_t)n_q * 4);
    l.full = take(dense_exact_workspace(n_rows, n_q, k));
    l.total = o;
    return l;
}

static bool s8_shape_ok(int dim) { return dim % S8_KC == 0 && dim >= S8_KC && dim <= S8_MAXD; }

}  // namespace ezr

using namespace ezr;

extern "C" {

int ezr_dense_quantize_rows(const void* x_bf16, int64_t ldx, int64_t n_rows, int32_t dim, int8_t* out_s8, int64_t ldo,
                            float* scale, float* err, float* norm, float* maxima, void* stream) {
    EZR_CHECK_ARG(dim >= 1 && ldx >= dim && ldo >= dim, "dense_quantize_rows: bad dim / strides");
    if (n_rows <= 0) return EZR_OK;
    const int wpb = 8;
    dense_s8_quantize_kernel<<<(unsigned)((n_rows + wpb - 1) / wpb), wpb * 32, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x_bf16, ldx, n_rows, dim, out_s8, ldo, scale, err, norm, maxima);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_dense_s8_set_capacity(int32_t cap) {
    EZR_CHECK_ARG(cap >= 0 && cap <= (1 << 20), "dense_s8_set_capacity: 0 (default) or 1..2^20 candidates per query");
    g_s8_cap = cap == 0 ? S8_DEFAULT_CAP : cap;
    return EZR_OK;
}

size_t ezr_dense_s8_topk_workspace(int64_t n_rows, int32_t dim, int32_t n_queries, int32_t k) {
    if (n_rows <= 0 || n_queries <= 0 || k <= 0) return 0;
    if (k > S8_KMAX) return dense_exact_workspace(n_rows, n_queries, k);
    return s8_layout(n_rows, dim, n_queries, k, g_s8_cap).total;
}

int ezr_dense_s8_topk(const void* corpus_bf16, int64_t n_rows, int32_t dim, int64_t ld_corpus,
                      const void* queries_bf16, int32_t n_queries, int64_t ld_queries, int32_t k,
                      const int32_t* doc_group, const int32_t* q_group, int32_t id_base, float* out_scores,
                      int32_t* out_ids, int32_t* out_counts, const int8_t* corpus_s8, int64_t ld_s8,
                      const float* row_scale, const float* maxima, int32_t* out_cand_counts, void* workspace,
                      size_t workspace_bytes, void* stream) {
    EZR_CHECK_ARG(k >= 1 && k <= 1024, "dense_s8_topk: k=%d out of [1,1024]", k);
    EZR_CHECK_ARG(s8_shape_ok(dim), "dense_s8_topk: dim=%d unsupported (multiple of 128, at most 1024)", dim);
    EZR_CHECK_ARG(n_rows >= 0 && n_rows < ((int64_t)1 << 31), "dense_s8_topk: n_rows out of range");
    EZR_CHECK_ARG(ld_corpus >= dim && ld_queries >= dim && ld_s8 >= dim, "dense_s8_topk: row stride smaller than dim");
    EZR_CHECK_ARG(ld_corpus % 8 == 0 && ld_s8 % 16 == 0, "dense_s8_topk: row strides must be 16-byte multiples");
    // an empty shard's doc_group is empty, and an empty tensor has no address: nothing is filtered, so no check
    EZR_CHECK_ARG(q_group == nullptr || doc_group != nullptr || n_rows == 0,
                  "dense_s8_topk: q_group without doc_group");
    EZR_CHECK_ARG(((uintptr_t)corpus_bf16 & 15) == 0 && ((uintptr_t)corpus_s8 & 15) == 0,
                  "dense_s8_topk: corpus rows must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_queries == 0) return EZR_OK;
    if (n_rows == 0) {
        if (out_counts) EZR_CUDA(cudaMemsetAsync(out_counts, 0, (size_t)n_queries * 4, st));
        if (out_cand_counts) EZR_CUDA(cudaMemsetAsync(out_cand_counts, 0, (size_t)n_queries * 4, st));
        EZR_CUDA(cudaMemsetAsync(out_ids, 0xff, (size_t)n_queries * k * 4, st));
        return EZR_OK;
    }
    const __nv_bfloat16* c = reinterpret_cast<const __nv_bfloat16*>(corpus_bf16);
    const __nv_bfloat16* qv = reinterpret_cast<const __nv_bfloat16*>(queries_bf16);
    if (k > S8_KMAX) {
        // the scan keeps k <= 16 values per thread; larger k is the full scan over every query
        if (out_cand_counts) EZR_CUDA(cudaMemsetAsync(out_cand_counts, 0, (size_t)n_queries * 4, st));
        ProfScope prof(EZR_PROF_DENSE_S8_FULL, st);
        return dense_exact_topk(c, n_rows, dim, ld_corpus, qv, n_queries, ld_queries, k, doc_group, q_group, id_base,
                                out_scores, out_ids, out_counts, workspace, workspace_bytes, st);
    }
    const int cap = g_s8_cap;
    const S8Layout l = s8_layout(n_rows, dim, n_queries, k, cap);
    if (!workspace || workspace_bytes < l.total) {
        set_error("dense_s8_topk: workspace %zu < %zu", workspace_bytes, l.total);
        return EZR_ERR_WORKSPACE;
    }
    char* ws = reinterpret_cast<char*>(workspace);
    int8_t* q8 = reinterpret_cast<int8_t*>(ws + l.q8);

    S8Params p;
    p.n_rows = n_rows;
    p.n_queries = n_queries;
    p.kchunks = dim / S8_KC;
    p.n_qblocks = (n_queries + 63) / 64;
    p.cap = cap;
    p.doc_group = doc_group;
    p.q_group = q_group;
    p.row_scale = row_scale;
    p.q_scale = reinterpret_cast<float*>(ws + l.q_scale);
    p.q_margin = reinterpret_cast<float*>(ws + l.q_margin);
    p.bound = reinterpret_cast<int32_t*>(ws + l.bound);
    p.cand_cnt = reinterpret_cast<int32_t*>(ws + l.cand_cnt);
    p.cand_id = reinterpret_cast<int32_t*>(ws + l.cand_id);
    const int sms = sm_count();
    // the cost model's corpus time is in bf16 elements: an int8 row of dim bytes counts as dim / 2
    p.n_slices = ts_choose_splits(p.n_qblocks, n_rows, dim / 2, sms, S8_TN);
    p.rows_per_slice = tc_rows_per_slice(n_rows, p.n_slices, S8_TN);
    p.n_slices = (int)((n_rows + p.rows_per_slice - 1) / p.rows_per_slice);
    const size_t a_bytes = (size_t)p.kchunks * S8_A_BOX_BYTES;
    const size_t fixed = 1024 + sizeof(S8Barriers);
    int stages = (int)((S8_SMEM_LIMIT - fixed - a_bytes) / S8_B_STAGE_BYTES);
    if (stages > S8_MAX_STAGES) stages = S8_MAX_STAGES;
    p.n_stages = stages;
    const size_t smem = fixed + a_bytes + (size_t)stages * S8_B_STAGE_BYTES;

    {
        ProfScope prof(EZR_PROF_DENSE_S8_SCAN, st);
        const int wpb = 8;
        dense_s8_prep_kernel<<<(unsigned)((n_queries + wpb - 1) / wpb), wpb * 32, 0, st>>>(
            qv, ld_queries, n_queries, dim, maxima, q8, const_cast<float*>(p.q_scale), const_cast<float*>(p.q_margin),
            p.bound, p.cand_cnt);
        EZR_LAUNCH_CHECK();
        CUtensorMap map_q, map_c;
        int rc = encode_tmap_2d_bf16(&map_q, q8, (uint64_t)dim / 2, (uint64_t)n_queries, (uint64_t)dim / 2, 64, 64);
        if (rc) return rc;
        rc = encode_tmap_2d_bf16(&map_c, corpus_s8, (uint64_t)dim / 2, (uint64_t)n_rows, (uint64_t)ld_s8 / 2, 64,
                                 S8_TN);
        if (rc) return rc;
        typedef void (*kern_t)(const CUtensorMap, const CUtensorMap, const S8Params);
        static const kern_t table[2][5] = {
            {dense_s8_scan_kernel<false, 1>, dense_s8_scan_kernel<false, 2>, dense_s8_scan_kernel<false, 4>,
             dense_s8_scan_kernel<false, 8>, dense_s8_scan_kernel<false, 16>},
            {dense_s8_scan_kernel<true, 1>, dense_s8_scan_kernel<true, 2>, dense_s8_scan_kernel<true, 4>,
             dense_s8_scan_kernel<true, 8>, dense_s8_scan_kernel<true, 16>}};
        const int fi = q_group != nullptr ? 1 : 0;
        const int kt = k <= 1 ? 0 : k <= 2 ? 1 : k <= 4 ? 2 : k <= 8 ? 3 : 4;
        static bool attr_done[2][5] = {};
        if (!attr_done[fi][kt]) {
            EZR_CUDA(cudaFuncSetAttribute(table[fi][kt], cudaFuncAttributeMaxDynamicSharedMemorySize, S8_SMEM_LIMIT));
            attr_done[fi][kt] = true;
        }
        const int units = p.n_slices * p.n_qblocks;
        table[fi][kt]<<<(unsigned)(units < sms ? units : sms), 256, smem, st>>>(map_q, map_c, p);
        EZR_LAUNCH_CHECK();
    }
    int32_t* over_pos = reinterpret_cast<int32_t*>(ws + l.over_pos);
    int32_t* over_list = reinterpret_cast<int32_t*>(ws + l.over_list);
    int32_t* over_n_d = reinterpret_cast<int32_t*>(ws + l.over_n);
    dense_s8_overflow_kernel<<<1, 1024, 0, st>>>(p.cand_cnt, n_queries, cap, over_pos, over_list, over_n_d);
    EZR_LAUNCH_CHECK();
    // the host learns how many queries overflowed (one small copy + stream sync) to size the full scan
    int32_t n_over = 0;
    EZR_CUDA(cudaMemcpyAsync(&n_over, over_n_d, 4, cudaMemcpyDeviceToHost, st));
    EZR_CUDA(cudaStreamSynchronize(st));
    float* fb_s = reinterpret_cast<float*>(ws + l.fb_s);
    int32_t* fb_i = reinterpret_cast<int32_t*>(ws + l.fb_i);
    int32_t* fb_c = reinterpret_cast<int32_t*>(ws + l.fb_c);
    if (n_over > 0) {
        ProfScope prof(EZR_PROF_DENSE_S8_FULL, st);
        __nv_bfloat16* g_q = reinterpret_cast<__nv_bfloat16*>(ws + l.g_q);
        int32_t* g_group = reinterpret_cast<int32_t*>(ws + l.g_group);
        dense_s8_gather_kernel<<<n_over, 256, 0, st>>>(qv, ld_queries, dim, q_group, over_list, n_over, g_q, g_group);
        EZR_LAUNCH_CHECK();
        const int rc = dense_exact_topk(c, n_rows, dim, ld_corpus, g_q, n_over, dim, k, doc_group,
                                        q_group ? g_group : nullptr, id_base, fb_s, fb_i, fb_c, ws + l.full,
                                        l.total - l.full, st);
        if (rc) return rc;
    }
    {
        ProfScope prof(EZR_PROF_DENSE_S8_RESCORE, st);
        static bool attr_done = false;
        if (!attr_done) {
            EZR_CUDA(cudaFuncSetAttribute(dense_s8_rescore_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)s8_rescore_smem()));
            attr_done = true;
        }
        dense_s8_rescore_kernel<<<n_queries, S8_RESCORE_THREADS, s8_rescore_smem(), st>>>(
            c, ld_corpus, dim, qv, ld_queries, k, id_base, p.cand_cnt, p.cand_id, cap, over_pos, fb_s, fb_i, fb_c,
            out_scores, out_ids, out_counts, out_cand_counts);
        EZR_LAUNCH_CHECK();
    }
    return EZR_OK;
}

}  // extern "C"
