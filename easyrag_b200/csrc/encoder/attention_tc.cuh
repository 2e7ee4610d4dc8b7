// Multi-head attention over PACKED variable-length sequences on wgmma (Hopper warpgroup MMA), bidirectional or causal.
//
// Reference: Qwen2 attention run with is_causal=False (modeling_qwen.py:289-308 eager / :704-712 SDPA, padding
// handled by an additive mask :1037-1040) and BERT self-attention behind SentenceTransformer.encode
// (hf_embeddings.py:118-123).  Sequences are packed, so the mask reduces to "keys beyond this sequence".
// The causal form (CAUSAL = true; Qwen2Model.forward(is_causal=True), mask built at modeling_qwen.py:1043-1051) lets
// query row r of a sequence see keys 0..r: an item walks only the key tiles up to its last row's diagonal, and only
// the last two of them carry the per-element mask.
//
// Work item = 128 query rows of one (sequence, head).  A small plan kernel lists the (sequence, query block) pairs
// that exist; PERSISTENT CTAs walk the items round-robin, query blocks of one (sequence, head) next to each other so
// that concurrently running CTAs share its K / V tiles through L2.
//   warpgroup 0    TMA producer (one thread): Q tile per item, K / V tiles of 64 keys (one packed [tokens, (H + 2 KV) hd] matrix
//                  serves Q, K and V through two tensor maps -- 128-row and 64-row boxes; 128B swizzle; rows past the
//                  matrix are zero-filled), running ahead across items
//   warpgroups 1-2 64 query rows each:  S = Q K^T      wgmma SS m64n64k16 (both operands K-major in shared memory)
//                                       online softmax in registers (a row lives in the four threads of a quad)
//                                       O += P V       wgmma RS m64n{hd}k16: P straight from the S registers as bf16
//                                                      A fragments, V the MN-major B operand from its row-major TMA
//                                                      tile -- no transpose anywhere
//                  at the end of an item O / row sum -> bf16 -> global.
#pragma once
#include "../ezr_common.cuh"
#include "../ptx.cuh"

namespace ezr {

constexpr int AT_M = 128;                 // query rows per work item
constexpr int AT_N = 64;                  // keys per tile
constexpr int AT_THREADS = 384;           // producer warpgroup + two consumer warpgroups (wgmma needs 4-warp-aligned groups)
constexpr int AT_BOX_BYTES = 128 * 64 * 2;   // one Q TMA box: 128 rows x 64 bf16
constexpr int AT_KV_BOX_BYTES = AT_N * 64 * 2;   // one K / V TMA box: 64 rows x 64 bf16
constexpr int AT_STAGES = 2;              // K and V rings (own barriers each)

struct AttnBarriers {
    uint64_t q_full, q_empty;
    uint64_t k_full[AT_STAGES], k_empty[AT_STAGES], v_full[AT_STAGES], v_empty[AT_STAGES];
};

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// plan[i] = {first token of the sequence, its length, first query row of the block, sequence} for every 128-row query
// block that exists (fully resolved: the attention kernel's roles read ONE 16-byte entry per work item, one item
// ahead, instead of a chain of dependent loads at every item start); plan_n[0] = their number.
// One CTA; sequences in order, so the query blocks of a sequence are adjacent.  Causal: query block j reads about
// 2 (j + 1) key tiles, so a sequence's blocks are listed last, first, second-to-last, second, ... -- the costliest
// first, and each adjacent pair (which one CTA runs back to back, see attn_wgmma_kernel) costs about the same.
template <bool CAUSAL>
__global__ void __launch_bounds__(256)
attn_plan_kernel(const int32_t* __restrict__ cu, int n_seq, int4* __restrict__ plan, int32_t* __restrict__ plan_n) {
    __shared__ int s_warp[8];
    __shared__ int s_base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int b0 = 0; b0 < n_seq; b0 += 256) {
        const int b = b0 + tid;
        const int lo_b = b < n_seq ? cu[b] : 0, len_b = b < n_seq ? cu[b + 1] - lo_b : 0;
        const int nqb = (len_b + AT_M - 1) / AT_M;
        int inc = nqb;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
        }
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        int before = s_base;
        for (int w = 0; w < warp; ++w) before += s_warp[w];
        const int first = before + inc - nqb;
        for (int j = 0; j < nqb; ++j)
            plan[first + j] = make_int4(lo_b, len_b, (CAUSAL ? ((j & 1) ? j >> 1 : nqb - 1 - (j >> 1)) : j) * AT_M, b);
        __syncthreads();
        if (tid == 255) s_base = before + inc;
        __syncthreads();
    }
    if (tid == 0) plan_n[0] = s_base;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
}

template <int HD, bool CAUSAL>
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_wgmma_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_kv,
                  const int4* __restrict__ plan, const int32_t* __restrict__ plan_n,
                  int n_heads, int n_kv_heads, float scale_log2, __nv_bfloat16* __restrict__ out, int64_t ldo) {
    constexpr int CH = HD / 64;                          // 64-column TMA boxes per tile
    constexpr int Q_BYTES = CH * AT_BOX_BYTES;           // one Q tile
    constexpr int KV_BYTES = CH * AT_KV_BOX_BYTES;       // one K / V tile
    extern __shared__ unsigned char smem_dyn[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    unsigned char* smem_q = smem;
    unsigned char* smem_k = smem_q + Q_BYTES;
    unsigned char* smem_v = smem_k + AT_STAGES * KV_BYTES;
    AttnBarriers* bars = reinterpret_cast<AttnBarriers*>(smem_v + AT_STAGES * KV_BYTES);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_pairs = plan_n[0];
    const int n_work = n_pairs * n_heads;                // work w: head = w / n_pairs, pair = w % n_pairs
    const int kv_group = n_heads / n_kv_heads;

    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&map_q);
        ptx::prefetch_tensormap(&map_kv);
        ptx::mbar_init(&bars->q_full, 1);
        ptx::mbar_init(&bars->q_empty, 2);
        for (int i = 0; i < AT_STAGES; ++i) {
            ptx::mbar_init(&bars->k_full[i], 1);
            ptx::mbar_init(&bars->k_empty[i], 2);
            ptx::mbar_init(&bars->v_full[i], 1);
            ptx::mbar_init(&bars->v_empty[i], 2);
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    // every role walks the same items w = blockIdx.x, + gridDim.x, ... (causal: the pairs 2 blockIdx.x and
    // 2 blockIdx.x + 1, + 2 gridDim.x, ... -- the plan pairs a long item with a short one); the plan entry of the NEXT
    // item is requested at the top of each iteration, so no role ever waits for it
    auto plan_at = [&](int w) { return w < n_work ? __ldg(plan + w % n_pairs) : make_int4(0, 0, 0, 0); };
    auto first_item = [&]() { return CAUSAL ? 2 * (int)blockIdx.x : (int)blockIdx.x; };
    auto next_item = [&](int w) {
        if constexpr (CAUSAL) return (w & 1) ? w - 1 + 2 * (int)gridDim.x : w + 1;
        else return (int)(w + gridDim.x);
    };

    if (warp < 4) {
        if (threadIdx.x == 0) {
            // ---------------- TMA producer: runs ahead of the consumers, across work items ----------------
            int jt = 0;                                   // K/V tiles issued so far (ring position)
            int it = 0;                                   // items started
            int4 cur = plan_at(first_item());
            for (int w = first_item(); w < n_work; w = next_item(w), ++it) {
                const int4 nxt = plan_at(next_item(w));
                const int h = w / n_pairs;
                const int lo = cur.x, len = cur.y, q0 = cur.z;
                cur = nxt;
                const int kvh = h / kv_group;
                const int col_q = h * HD, col_k = (n_heads + kvh) * HD, col_v = (n_heads + n_kv_heads + kvh) * HD;
                int n_kt = (len + AT_N - 1) / AT_N;
                if constexpr (CAUSAL) n_kt = min(n_kt, (q0 + AT_M) / AT_N);    // tiles above the diagonal are never loaded
                ptx::mbar_wait(&bars->q_empty, ((uint32_t)it & 1u) ^ 1u);   // the QK^T MMAs that read the Q buffer are done
                ptx::mbar_expect_tx(&bars->q_full, Q_BYTES);
                for (int c = 0; c < CH; ++c)
                    ptx::tma_load_2d(smem_q + c * AT_BOX_BYTES, &map_q, &bars->q_full, col_q + c * 64, lo + q0);
                for (int j = 0; j < n_kt; ++j, ++jt) {
                    const int s = jt % AT_STAGES;
                    const uint32_t ph = (uint32_t)(jt / AT_STAGES) & 1u;
                    const int row = lo + j * AT_N;
                    ptx::mbar_wait(&bars->k_empty[s], ph ^ 1);
                    ptx::mbar_expect_tx(&bars->k_full[s], KV_BYTES);
                    for (int c = 0; c < CH; ++c)
                        ptx::tma_load_2d(smem_k + s * KV_BYTES + c * AT_KV_BOX_BYTES, &map_kv, &bars->k_full[s], col_k + c * 64, row);
                    ptx::mbar_wait(&bars->v_empty[s], ph ^ 1);
                    ptx::mbar_expect_tx(&bars->v_full[s], KV_BYTES);
                    for (int c = 0; c < CH; ++c)
                        ptx::tma_load_2d(smem_v + s * KV_BYTES + c * AT_KV_BOX_BYTES, &map_kv, &bars->v_full[s], col_v + c * 64, row);
                }
            }
        }
        return;
    }

    // ---------------- consumers: warpgroup cw owns query rows [64 cw, 64 cw + 64) of the item
    const int cw = (threadIdx.x >> 7) - 1;
    const int wq = warp & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    const int r_in = cw * 64 + wq * 16 + (lane >> 2);    // this thread's rows r_in and r_in + 8 of the item
    const uint32_t q_addr = ptx::smem_u32(smem_q) + (uint32_t)(cw * 64 * 128);
    int jt = 0, it = 0;
    int4 cur = plan_at(first_item());
    for (int w = first_item(); w < n_work; w = next_item(w), ++it) {
        const int4 nxt = plan_at(next_item(w));
        const int h = w / n_pairs;
        const int lo = cur.x, len = cur.y, q0 = cur.z;
        cur = nxt;
        int n_kt = (len + AT_N - 1) / AT_N;
        if constexpr (CAUSAL) n_kt = min(n_kt, (q0 + AT_M) / AT_N);
        float o[HD / 2];
#pragma unroll
        for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
        float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
        ptx::mbar_wait(&bars->q_full, (uint32_t)it & 1u);
        for (int j = 0; j < n_kt; ++j, ++jt) {
            const int s = jt % AT_STAGES;
            const uint32_t ph = (uint32_t)(jt / AT_STAGES) & 1u;
            const int valid = len - j * AT_N;
            if constexpr (CAUSAL) {
                if (j * AT_N > q0 + cw * 64 + 63) {
                    // every key of the tile lies past every row of this warpgroup (warpgroup 0 on the item's last
                    // tile): no MMAs, o / l / m stay as they are.  The slot is still released: k_empty / v_empty count
                    // both consumers, and waiting for the fills first keeps these arrivals on this tile's phase.
                    ptx::mbar_wait(&bars->k_full[s], ph);
                    ptx::mbar_wait(&bars->v_full[s], ph);
                    if (leader) {
                        ptx::mbar_arrive(&bars->k_empty[s]);
                        if (j == n_kt - 1) ptx::mbar_arrive(&bars->q_empty);
                        ptx::mbar_arrive(&bars->v_empty[s]);
                    }
                    continue;
                }
            }
            // ---- S = Q K^T (64 x 64 per warpgroup)
            float sc[32];
            const uint32_t k_addr = ptx::smem_u32(smem_k + s * KV_BYTES);
            ptx::mbar_wait(&bars->k_full[s], ph);
            ptx::wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < HD / 16; ++kk) {
                const uint32_t qoff = (uint32_t)((kk >> 2) * AT_BOX_BYTES + (kk & 3) * 32);
                const uint32_t koff = (uint32_t)((kk >> 2) * AT_KV_BOX_BYTES + (kk & 3) * 32);
                ptx::wgmma_ss_n64(sc, ptx::make_desc_sw128(q_addr + qoff), ptx::make_desc_sw128(k_addr + koff),
                                  (uint32_t)(kk != 0));
            }
            ptx::wgmma_commit();
            ptx::wgmma_wait<0>();
            ptx::fence_regs(sc);
            if (leader) {
                ptx::mbar_arrive(&bars->k_empty[s]);
                if (j == n_kt - 1) ptx::mbar_arrive(&bars->q_empty);       // the Q tile may be overwritten
            }
            // ---- online softmax: keys past the sequence -> -inf; a row is spread over the 4 threads of a quad
            const int c0 = (lane & 3) * 2;
            if constexpr (CAUSAL) {
                // causal: key j*64 + col is visible to sequence row q0 + r_in (+ 8) while col < valid and
                // j*64 + col <= that row; only the tiles that reach past this warpgroup's first row need the test
                if (valid < AT_N || j * AT_N + AT_N - 1 > q0 + cw * 64) {
                    const int d0 = q0 + r_in - j * AT_N + 1;
                    const int lim0 = min(valid, d0), lim1 = min(valid, d0 + 8);
#pragma unroll
                    for (int i = 0; i < 32; ++i) {
                        const int col = (i >> 2) * 8 + c0 + (i & 1);
                        if (col >= ((i & 2) ? lim1 : lim0)) sc[i] = -INFINITY;
                    }
                }
            } else if (valid < AT_N) {
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                    const int col = (i >> 2) * 8 + c0 + (i & 1);
                    if (col >= valid) sc[i] = -INFINITY;
                }
            }
            uint32_t pa[16];                             // P as bf16 A fragments: 4 k16 slices x 4 registers
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                float mx = -INFINITY;
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) mx = fmaxf(mx, fmaxf(sc[4 * jj + 2 * hh], sc[4 * jj + 2 * hh + 1]));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                const float m_new = fmaxf(m_run[hh], mx);         // finite: every tile has >= 1 valid key
                const float alpha = ex2_approx((m_run[hh] - m_new) * scale_log2);     // 0 on the first tile
                m_run[hh] = m_new;
                const float mb = m_new * scale_log2;
                float l = 0.f;
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {
                    const float p0 = ex2_approx(fmaf(sc[4 * jj + 2 * hh], scale_log2, -mb));
                    const float p1 = ex2_approx(fmaf(sc[4 * jj + 2 * hh + 1], scale_log2, -mb));
                    l += p0 + p1;
                    // key columns 8 jj + c0 (+1): slice jj / 2, register (jj % 2) * 2 + hh
                    pa[(jj >> 1) * 4 + (jj & 1) * 2 + hh] = pack_bf16x2(p0, p1);
                }
                l_run[hh] = l_run[hh] * alpha + l;
#pragma unroll
                for (int i = 0; i < HD / 8; ++i) {
                    o[4 * i + 2 * hh] *= alpha;
                    o[4 * i + 2 * hh + 1] *= alpha;
                }
            }
            // ---- O += P V
            const uint32_t v_addr = ptx::smem_u32(smem_v + s * KV_BYTES);
            ptx::mbar_wait(&bars->v_full[s], ph);
            ptx::wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < AT_N / 16; ++kk) {
                const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
                const uint64_t db = ptx::make_desc_sw128_mn(v_addr + (uint32_t)kk * 2048u, AT_KV_BOX_BYTES);
                if constexpr (HD == 64) ptx::wgmma_rs_n64_bmn(*reinterpret_cast<float(*)[32]>(o), a, db, 1u);
                else ptx::wgmma_rs_n128_bmn(*reinterpret_cast<float(*)[64]>(o), a, db, 1u);
            }
            ptx::wgmma_commit();
            ptx::wgmma_wait<0>();
            ptx::fence_regs(o);
            if (leader) ptx::mbar_arrive(&bars->v_empty[s]);
        }
        // ---- epilogue of the item: O / row sum -> bf16 -> global
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            float l = l_run[hh];
            l += __shfl_xor_sync(0xffffffffu, l, 1);
            l += __shfl_xor_sync(0xffffffffu, l, 2);
            const float inv = 1.0f / l;
            const int row = q0 + r_in + 8 * hh;
            if (row >= len) continue;
            __nv_bfloat16* orow = out + (int64_t)(lo + row) * ldo + h * HD + (lane & 3) * 2;
#pragma unroll
            for (int i = 0; i < HD / 8; ++i)
                *reinterpret_cast<uint32_t*>(orow + 8 * i) = pack_bf16x2(o[4 * i + 2 * hh] * inv, o[4 * i + 2 * hh + 1] * inv);
        }
    }
}

// plan + attention kernel on the caller's tensor maps (scale_log2 = softmax scale * log2 e).  The plan of a call is
// its own: drawn from the stream-ordered pool of the launch stream before the plan kernel and released after the
// attention kernel, so calls on different streams never share it, and graph capture records both as memory nodes.
template <int HD, bool CAUSAL>
static int attn_tc_launch(const CUtensorMap& map_q, const CUtensorMap& map_kv, const int32_t* cu, int n_seq, int max_len,
                          int n_heads, int n_kv_heads, float scale_log2, __nv_bfloat16* out, int64_t ldo, cudaStream_t st) {
    const size_t smem = 1024 + (size_t)(HD / 64) * (AT_BOX_BYTES + 2 * AT_STAGES * AT_KV_BOX_BYTES) + sizeof(AttnBarriers);
    static bool attr_done = false;
    if (!attr_done) {
        EZR_CUDA(cudaFuncSetAttribute(attn_wgmma_kernel<HD, CAUSAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done = true;
    }
    const int max_qb = (max_len + AT_M - 1) / AT_M;
    const size_t n_items = (size_t)n_seq * max_qb;              // query blocks at most
    // ints: 4 for the count (keeps the entries 16-byte aligned) + 4 per entry
    int32_t* buf = nullptr;
    EZR_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&buf), (n_items + 1) * 4 * sizeof(int32_t), st));
    int32_t* plan_n = buf;
    int4* plan = reinterpret_cast<int4*>(buf + 4);
    ProfScope prof(EZR_PROF_ENC_ATTN, st);
    attn_plan_kernel<CAUSAL><<<1, 256, 0, st>>>(cu, n_seq, plan, plan_n);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) {
        long long upper = (long long)n_items * n_heads;         // work items at most
        if (CAUSAL) upper = (upper + 1) / 2;                    // causal CTAs take items in pairs
        const int grid = (int)(upper < sm_count() ? upper : sm_count());
        attn_wgmma_kernel<HD, CAUSAL><<<grid, AT_THREADS, smem, st>>>(map_q, map_kv, plan, plan_n, n_heads, n_kv_heads,
                                                                      scale_log2, out, ldo);
        count_launch();
        e = cudaGetLastError();
    }
    const cudaError_t e_free = cudaFreeAsync(buf, st);          // released on every path, after the last reader
    EZR_CUDA(e);
    EZR_CUDA(e_free);
    return EZR_OK;
}

// the causal instances, compiled in a translation unit of their own (attention_tc_causal.cu)
int attn_tc_causal_launch(int head_dim, const CUtensorMap& map_q, const CUtensorMap& map_kv, const int32_t* cu,
                          int n_seq, int max_len, int n_heads, int n_kv_heads, float scale_log2, __nv_bfloat16* out,
                          int64_t ldo, cudaStream_t st);

}  // namespace ezr
