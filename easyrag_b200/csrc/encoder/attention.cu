// Bidirectional (non-causal) multi-head attention over PACKED variable-length sequences, GQA aware.
//
// Reference: Qwen2 attention run with is_causal=False (modeling_qwen.py:289-308 eager / :704-712 SDPA, padding
// handled by an additive mask :1037-1040) and BERT self-attention behind SentenceTransformer.encode.  With packed
// sequences there are no padding keys, so the mask reduces to "keys beyond this sequence's length".
//
// Flash-style: one CTA = 64 query rows of one (sequence, head); K/V streamed in 64-key tiles through
// XOR-swizzled shared memory; S = QK^T and O += PV on warp-level bf16 MMA (m16n8k16, fp32 accumulate), online
// softmax in fp32 (exp2 with the 1/sqrt(d) scale folded in).  Attention is ~10% of the encoder FLOPs at
// L <= 512 (SURVEY.md 8(d)); the projections around it run on wgmma (gemm_tc.cu).
#include "../ezr_common.cuh"

namespace ezr {

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
    const int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ uint32_t pack2(float a, float b) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
}

template <int HD>
__device__ __forceinline__ uint32_t tile_addr(uint32_t base, int row, int chunk) {
    return base + (uint32_t)(row * (HD * 2) + ((chunk ^ (row & 7)) << 4));
}

// rows [r0, r0+64) of a [len, HD] slab with row stride ld -> swizzled smem tile; rows >= len are zero-filled
template <int HD>
__device__ __forceinline__ void load_tile(uint32_t smem_base, const __nv_bfloat16* src, int64_t ld, int r0, int len) {
    constexpr int CH = HD / 8;               // 16-byte chunks per row
    for (int e = threadIdx.x; e < 64 * CH; e += 128) {
        const int row = e / CH, chunk = e % CH;
        const int gr = r0 + row;
        const bool ok = gr < len;
        const __nv_bfloat16* g = src + (int64_t)(ok ? gr : 0) * ld + chunk * 8;
        cp_async16(tile_addr<HD>(smem_base, row, chunk), g, ok);
    }
}

template <int HD>
__global__ void __launch_bounds__(128)
attn_bidir_kernel(const __nv_bfloat16* __restrict__ qkv, int64_t ld, const int32_t* __restrict__ cu, int n_heads,
                  int n_kv_heads, float scale_log2, __nv_bfloat16* __restrict__ out, int64_t ldo) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    constexpr uint32_t kTile = 64 * HD * 2;
    const uint32_t sQ = static_cast<uint32_t>(__cvta_generic_to_shared(smem_raw));
    const uint32_t sK0 = sQ + kTile;            // K/V tiles are double buffered: [K0 V0 K1 V1]
    const int qb = blockIdx.x, b = blockIdx.y, h = blockIdx.z;
    const int lo = cu[b];
    const int len = cu[b + 1] - lo;
    const int q0 = qb * 64;
    if (q0 >= len) return;
    const int kvh = h / (n_heads / n_kv_heads);
    const __nv_bfloat16* q_ptr = qkv + (int64_t)lo * ld + h * HD;
    const __nv_bfloat16* k_ptr = qkv + (int64_t)lo * ld + (n_heads + kvh) * HD;
    const __nv_bfloat16* v_ptr = qkv + (int64_t)lo * ld + (n_heads + n_kv_heads + kvh) * HD;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    load_tile<HD>(sQ, q_ptr, ld, q0, len);
    load_tile<HD>(sK0, k_ptr, ld, 0, len);
    load_tile<HD>(sK0 + kTile, v_ptr, ld, 0, len);
    cp_async_wait_all();
    __syncthreads();
    uint32_t qf[HD / 16][4];
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks)
        ldsm_x4(qf[ks], tile_addr<HD>(sQ, warp * 16 + (lane & 15), ks * 2 + (lane >> 4)));

    float o[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
    float m_run[2] = {-INFINITY, -INFINITY};
    float l_run[2] = {0.f, 0.f};
    const int mi = lane >> 3, r8 = lane & 7;
    const int n_kt = (len + 63) / 64;

    for (int kt = 0; kt < n_kt; ++kt) {
        const uint32_t sK = sK0 + (uint32_t)(kt & 1) * 2 * kTile;
        const uint32_t sV = sK + kTile;
        if (kt + 1 < n_kt) {                                 // prefetch the next K/V tile into the other buffer
            const uint32_t nK = sK0 + (uint32_t)((kt + 1) & 1) * 2 * kTile;
            load_tile<HD>(nK, k_ptr, ld, (kt + 1) * 64, len);
            load_tile<HD>(nK + kTile, v_ptr, ld, (kt + 1) * 64, len);
            cp_async_commit();
        }

        float s[8][4];
#pragma unroll
        for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
            for (int ks = 0; ks < HD / 16; ++ks) {
                uint32_t bk[4];
                ldsm_x4(bk, tile_addr<HD>(sK, j * 16 + (mi >> 1) * 8 + r8, ks * 2 + (mi & 1)));
                mma_bf16(s[2 * j], qf[ks], bk[0], bk[1]);
                mma_bf16(s[2 * j + 1], qf[ks], bk[2], bk[3]);
            }
        }
        // mask keys beyond the sequence, running max
        const int key0 = kt * 64 + (lane & 3) * 2;
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = key0 + nb * 8 + (e & 1);
                if (key >= len) s[nb][e] = -INFINITY;
                mx[e >> 1] = fmaxf(mx[e >> 1], s[nb][e]);
            }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        }
        float alpha[2], m_new[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            m_new[r] = fmaxf(m_run[r], mx[r]);
            alpha[r] = exp2f((m_run[r] - m_new[r]) * scale_log2);
            m_run[r] = m_new[r];
            l_run[r] *= alpha[r];
        }
#pragma unroll
        for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float pv = exp2f((s[nb][e] - m_new[e >> 1]) * scale_log2);
                s[nb][e] = pv;
                l_run[e >> 1] += pv;
            }
        }
#pragma unroll
        for (int i = 0; i < HD / 8; ++i) {
            o[i][0] *= alpha[0]; o[i][1] *= alpha[0];
            o[i][2] *= alpha[1]; o[i][3] *= alpha[1];
        }
        // O += P V
#pragma unroll
        for (int k2 = 0; k2 < 4; ++k2) {
            uint32_t pa[4];
            pa[0] = pack2(s[2 * k2][0], s[2 * k2][1]);
            pa[1] = pack2(s[2 * k2][2], s[2 * k2][3]);
            pa[2] = pack2(s[2 * k2 + 1][0], s[2 * k2 + 1][1]);
            pa[3] = pack2(s[2 * k2 + 1][2], s[2 * k2 + 1][3]);
#pragma unroll
            for (int jn = 0; jn < HD / 16; ++jn) {
                uint32_t bv[4];
                ldsm_x4_t(bv, tile_addr<HD>(sV, k2 * 16 + (mi & 1) * 8 + r8, jn * 2 + (mi >> 1)));
                mma_bf16(o[2 * jn], pa, bv[0], bv[1]);
                mma_bf16(o[2 * jn + 1], pa, bv[2], bv[3]);
            }
        }
        if (kt + 1 < n_kt) {
            cp_async_wait<0>();                              // next tile has landed (it had the whole tile to do so)
            __syncthreads();                                 // and everyone is done reading the current one
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
    const float inv0 = 1.f / l_run[0], inv1 = 1.f / l_run[1];
    const int row0 = q0 + warp * 16 + (lane >> 2);
    __nv_bfloat16* obase = out + (int64_t)lo * ldo + h * HD + (lane & 3) * 2;
#pragma unroll
    for (int nb = 0; nb < HD / 8; ++nb) {
        if (row0 < len)
            *reinterpret_cast<uint32_t*>(obase + (int64_t)row0 * ldo + nb * 8) = pack2(o[nb][0] * inv0, o[nb][1] * inv0);
        if (row0 + 8 < len)
            *reinterpret_cast<uint32_t*>(obase + (int64_t)(row0 + 8) * ldo + nb * 8) = pack2(o[nb][2] * inv1, o[nb][3] * inv1);
    }
}

}  // namespace ezr

// The first attention kernel of this library (warp-level mma.sync), kept as an independent implementation the
// wgmma kernel (attention_tc.cu) is cross-checked against: ezr_attn_set_kernel(1).
namespace ezr {
int attn_bidir_legacy(const void* qkv, int64_t ld, const int32_t* cu_seqlens, int32_t n_seq, int32_t max_len,
                      int32_t n_heads, int32_t n_kv_heads, int32_t head_dim, float softmax_scale, void* out, int64_t ldo,
                      cudaStream_t st) {
    EZR_CHECK_ARG(head_dim == 64 || head_dim == 128, "attn: head_dim must be 64 or 128 (got %d)", head_dim);
    EZR_CHECK_ARG(n_kv_heads >= 1 && n_heads % n_kv_heads == 0, "attn: n_heads must be a multiple of n_kv_heads");
    EZR_CHECK_ARG(ld % 8 == 0 && ldo % 2 == 0, "attn: qkv row stride must be a multiple of 8 elements");
    EZR_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0, "attn: qkv must be 16-byte aligned");
    if (n_seq == 0 || max_len == 0) return EZR_OK;
    EZR_CHECK_ARG(n_seq <= 65535 && n_heads <= 65535, "attn: grid too large");
    const float scale_log2 = softmax_scale * 1.4426950408889634f;
    dim3 grid((max_len + 63) / 64, n_seq, n_heads);
    const size_t smem = (size_t)5 * 64 * head_dim * 2;      // Q + double-buffered K/V
    ProfScope prof(EZR_PROF_ENC_ATTN, st);
    if (head_dim == 64) {
        attn_bidir_kernel<64><<<grid, 128, smem, st>>>((const __nv_bfloat16*)qkv, ld, cu_seqlens, n_heads, n_kv_heads,
                                                       scale_log2, (__nv_bfloat16*)out, ldo);   // 40 KB: no opt-in needed
    } else {
        static bool attr_done = false;
        if (!attr_done) {
            EZR_CUDA(cudaFuncSetAttribute(attn_bidir_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attr_done = true;
        }
        attn_bidir_kernel<128><<<grid, 128, smem, st>>>((const __nv_bfloat16*)qkv, ld, cu_seqlens, n_heads, n_kv_heads,
                                                        scale_log2, (__nv_bfloat16*)out, ldo);
    }
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}
}  // namespace ezr
