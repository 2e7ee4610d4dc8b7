// Bidirectional (non-causal) multi-head attention over PACKED variable-length sequences on wgmma (Hopper warpgroup MMA).
//
// Reference: Qwen2 attention run with is_causal=False (modeling_qwen.py:289-308 eager / :704-712 SDPA, padding
// handled by an additive mask :1037-1040) and BERT self-attention behind SentenceTransformer.encode
// (hf_embeddings.py:118-123).  Sequences are packed, so the mask reduces to "keys beyond this sequence".
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
// One CTA; sequences in order, so the query blocks of a sequence are adjacent.
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
        for (int j = 0; j < nqb; ++j) plan[first + j] = make_int4(lo_b, len_b, j * AT_M, b);
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

template <int HD>
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
    // every role walks the same items w = blockIdx.x, + gridDim.x, ...; the plan entry of the NEXT item is requested at
    // the top of each iteration, so no role ever waits for it
    auto plan_at = [&](int w) { return w < n_work ? __ldg(plan + w % n_pairs) : make_int4(0, 0, 0, 0); };

    if (warp < 4) {
        if (threadIdx.x == 0) {
            // ---------------- TMA producer: runs ahead of the consumers, across work items ----------------
            int jt = 0;                                   // K/V tiles issued so far (ring position)
            int it = 0;                                   // items started
            int4 cur = plan_at(blockIdx.x);
            for (int w = blockIdx.x; w < n_work; w += gridDim.x, ++it) {
                const int4 nxt = plan_at(w + gridDim.x);
                const int h = w / n_pairs;
                const int lo = cur.x, len = cur.y, q0 = cur.z;
                cur = nxt;
                const int kvh = h / kv_group;
                const int col_q = h * HD, col_k = (n_heads + kvh) * HD, col_v = (n_heads + n_kv_heads + kvh) * HD;
                const int n_kt = (len + AT_N - 1) / AT_N;
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
    int4 cur = plan_at(blockIdx.x);
    for (int w = blockIdx.x; w < n_work; w += gridDim.x, ++it) {
        const int4 nxt = plan_at(w + gridDim.x);
        const int h = w / n_pairs;
        const int lo = cur.x, len = cur.y, q0 = cur.z;
        cur = nxt;
        const int n_kt = (len + AT_N - 1) / AT_N;
        float o[HD / 2];
#pragma unroll
        for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
        float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
        ptx::mbar_wait(&bars->q_full, (uint32_t)it & 1u);
        for (int j = 0; j < n_kt; ++j, ++jt) {
            const int s = jt % AT_STAGES;
            const uint32_t ph = (uint32_t)(jt / AT_STAGES) & 1u;
            const int valid = len - j * AT_N;
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
            if (valid < AT_N) {
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

int attn_bidir_legacy(const void* qkv, int64_t ld, const int32_t* cu_seqlens, int32_t n_seq, int32_t max_len,
                      int32_t n_heads, int32_t n_kv_heads, int32_t head_dim, float softmax_scale, void* out, int64_t ldo,
                      cudaStream_t st);

static int g_attn_kernel = 0;     // ezr_attn_set_kernel: 0 = wgmma (default), 1 = legacy mma.sync kernel (cross-checks)
static thread_local const char* g_attn_last = "none";

// plan buffer (query-block list) of the calling thread's device, grown on demand
static thread_local int32_t* g_plan = nullptr;
static thread_local size_t g_plan_cap = 0;
static thread_local int g_plan_dev = -1;

template <int HD>
static int attn_tc_launch(const CUtensorMap& map_q, const CUtensorMap& map_kv, const int32_t* cu, int n_seq, int max_len,
                          int n_heads, int n_kv_heads, float scale_log2, __nv_bfloat16* out, int64_t ldo, cudaStream_t st) {
    const size_t smem = 1024 + (size_t)(HD / 64) * (AT_BOX_BYTES + 2 * AT_STAGES * AT_KV_BOX_BYTES) + sizeof(AttnBarriers);
    static bool attr_done = false;
    if (!attr_done) {
        EZR_CUDA(cudaFuncSetAttribute(attn_wgmma_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done = true;
    }
    const int max_qb = (max_len + AT_M - 1) / AT_M;
    const size_t need = ((size_t)n_seq * max_qb + 1) * 4;          // ints: 4 for the count (keeps the entries 16-byte aligned) + 4 per entry
    int dev = 0;
    EZR_CUDA(cudaGetDevice(&dev));
    if (need > g_plan_cap || dev != g_plan_dev) {         // first call / larger batch / other device: (re)allocate
        if (g_plan && dev == g_plan_dev) EZR_CUDA(cudaFree(g_plan));
        g_plan_dev = dev;
        g_plan = nullptr;
        g_plan_cap = 0;
        EZR_CUDA(cudaMalloc(&g_plan, need * 2 * sizeof(int32_t)));
        g_plan_cap = need * 2;
    }
    int32_t* plan_n = g_plan;
    int4* plan = reinterpret_cast<int4*>(g_plan + 4);
    ProfScope prof(EZR_PROF_ENC_ATTN, st);
    attn_plan_kernel<<<1, 256, 0, st>>>(cu, n_seq, plan, plan_n);
    EZR_LAUNCH_CHECK();
    const long long upper = (long long)n_seq * max_qb * n_heads;      // work items at most
    const int grid = (int)(upper < sm_count() ? upper : sm_count());
    attn_wgmma_kernel<HD><<<grid, AT_THREADS, smem, st>>>(map_q, map_kv, plan, plan_n, n_heads, n_kv_heads, scale_log2, out, ldo);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

}  // namespace ezr

extern "C" int ezr_attn_set_kernel(int32_t which) {
    EZR_CHECK_ARG(which == 0 || which == 1, "attn_set_kernel: 0 = wgmma, 1 = legacy mma.sync");
    ezr::g_attn_kernel = which;
    return EZR_OK;
}

extern "C" const char* ezr_attn_last_kernel(void) { return ezr::g_attn_last; }

extern "C" int ezr_attn_bidir(const void* qkv, int64_t n_tokens, int64_t ld, const int32_t* cu_seqlens, int32_t n_seq,
                              int32_t max_len, int32_t n_heads, int32_t n_kv_heads, int32_t head_dim, float softmax_scale,
                              void* out, int64_t ldo, void* stream) {
    using namespace ezr;
    EZR_CHECK_ARG(head_dim == 64 || head_dim == 128, "attn: head_dim must be 64 or 128 (got %d)", head_dim);
    EZR_CHECK_ARG(n_kv_heads >= 1 && n_heads % n_kv_heads == 0, "attn: n_heads must be a multiple of n_kv_heads");
    EZR_CHECK_ARG(ld % 8 == 0 && ldo % 8 == 0, "attn: row strides must be multiples of 8 elements");
    EZR_CHECK_ARG(ld >= (int64_t)(n_heads + 2 * n_kv_heads) * head_dim, "attn: qkv rows narrower than (H + 2 KV) * head_dim");
    EZR_CHECK_ARG(((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
                  "attn: qkv / out must be 16-byte aligned");
    EZR_CHECK_ARG(softmax_scale > 0.f, "attn: softmax_scale must be positive");
    if (n_seq == 0 || max_len == 0 || n_tokens == 0) return EZR_OK;
    EZR_CHECK_ARG(n_seq <= 65535 && n_heads <= 65535, "attn: grid too large");
    cudaStream_t st = (cudaStream_t)stream;
    if (g_attn_kernel == 1) {
        g_attn_last = "mma.sync";
        return attn_bidir_legacy(qkv, ld, cu_seqlens, n_seq, max_len, n_heads, n_kv_heads, head_dim, softmax_scale, out,
                                 ldo, st);
    }
    g_attn_last = "wgmma";
    CUtensorMap map_q, map_kv;
    const uint64_t width = (uint64_t)(n_heads + 2 * n_kv_heads) * head_dim;
    int rc = encode_tmap_2d_bf16(&map_q, qkv, width, (uint64_t)n_tokens, (uint64_t)ld, 64, AT_M);
    if (rc) return rc;
    rc = encode_tmap_2d_bf16(&map_kv, qkv, width, (uint64_t)n_tokens, (uint64_t)ld, 64, AT_N);
    if (rc) return rc;
    const float scale_log2 = softmax_scale * 1.4426950408889634f;
    return head_dim == 64 ? attn_tc_launch<64>(map_q, map_kv, cu_seqlens, n_seq, max_len, n_heads, n_kv_heads,
                                               scale_log2, (__nv_bfloat16*)out, ldo, st)
                          : attn_tc_launch<128>(map_q, map_kv, cu_seqlens, n_seq, max_len, n_heads, n_kv_heads,
                                                scale_log2, (__nv_bfloat16*)out, ldo, st);
}
