// Memory-bound pieces of the chunk-embedding forward pass (everything that is not a GEMM or attention).
// Sequences are PACKED: token t of the batch lives in row t of every activation matrix, sequence b owns rows
// [cu_seqlens[b], cu_seqlens[b+1]); there are no padding tokens, so no compute is spent on them (the reference
// pads to the longest text of the batch: gte_embeddings.py:63, and masks in attention).
//
// Reference arithmetic mirrored here:
//   Qwen2RMSNorm            modeling_qwen.py:91-96   fp32 statistics, cast to bf16, then weight * x in bf16
//   rotary embedding        modeling_qwen.py:137-169 half-split layout, cos/sin tables cast to bf16, bf16 products
//   last_token_pool + F.normalize(p=2) in bf16       gte_embeddings.py:42-50,70
//   BERT embeddings + LayerNorm, CLS / mean pooling, fp32 normalise   (SentenceTransformer.encode, hf_embeddings.py:118-123)
#include "norm_row.cuh"

namespace ezr {

// block-wide sum for blockDim.x <= 1024 (result broadcast to all threads)
__device__ __forceinline__ float block_sum(float v, float* sh) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    float t = (threadIdx.x < nw) ? sh[threadIdx.x] : 0.f;
    if (warp == 0) t = warp_sum(t);
    if (threadIdx.x == 0) sh[32] = t;
    __syncthreads();
    return sh[32];
}

// ---------------------------------------------------------------- embedding gather (K1)
__global__ void embed_gather_kernel(const int32_t* __restrict__ ids, const __nv_bfloat16* __restrict__ table,
                                    int64_t ldt, int vocab, int dim, __nv_bfloat16* __restrict__ out, int64_t ldo,
                                    int n_tokens) {
    const int t = blockIdx.x;
    if (t >= n_tokens) return;
    int id = ids[t];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    const __nv_bfloat16* src = table + (int64_t)id * ldt;
    __nv_bfloat16* dst = out + (int64_t)t * ldo;
    if ((dim & 7) == 0 && (ldt & 7) == 0 && (ldo & 7) == 0) {
        for (int i = threadIdx.x; i < dim / 8; i += blockDim.x)
            reinterpret_cast<uint4*>(dst)[i] = __ldg(reinterpret_cast<const uint4*>(src) + i);
    } else {
        for (int i = threadIdx.x; i < dim; i += blockDim.x) dst[i] = src[i];
    }
}

// ------------------------------------------------- BERT embeddings: word + position + type, then LayerNorm
// TYPED: token t adds row types[t] of the [n_types, dim] type table; otherwise every token adds row 0 (type_table).
template <bool TYPED>
__global__ void bert_embed_ln_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ positions,
                                     const int32_t* __restrict__ types, const __nv_bfloat16* __restrict__ word,
                                     const __nv_bfloat16* __restrict__ pos, const __nv_bfloat16* __restrict__ type_table,
                                     int n_types, const __nv_bfloat16* __restrict__ gamma,
                                     const __nv_bfloat16* __restrict__ beta, float eps, int vocab, int max_pos, int dim,
                                     __nv_bfloat16* __restrict__ out, int n_tokens) {
    extern __shared__ float sh_x[];          // dim floats + 33 scratch
    float* scratch = sh_x + dim;
    const int t = blockIdx.x;
    if (t >= n_tokens) return;
    int id = ids[t];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    int pp = positions[t];
    pp = pp < 0 ? 0 : (pp >= max_pos ? max_pos - 1 : pp);
    const __nv_bfloat16* trow = type_table;
    if (TYPED) {
        int tt = types[t];
        tt = tt < 0 ? 0 : (tt >= n_types ? n_types - 1 : tt);
        trow += (int64_t)tt * dim;
    }
    float s = 0.f;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) {
        // each addend is a bf16 tensor in a bf16 model: word + type, then + position, each sum rounded (HF BertEmbeddings order)
        float v = __bfloat162float(__float2bfloat16(__bfloat162float(word[(int64_t)id * dim + i]) + __bfloat162float(trow[i])));
        v = __bfloat162float(__float2bfloat16(v + __bfloat162float(pos[(int64_t)pp * dim + i])));
        sh_x[i] = v;
        s += v;
    }
    const float mean = block_sum(s, scratch) / dim;
    float q = 0.f;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) { const float d = sh_x[i] - mean; q += d * d; }
    const float rstd = rsqrtf(block_sum(q, scratch) / dim + eps);
    for (int i = threadIdx.x; i < dim; i += blockDim.x)
        out[(int64_t)t * dim + i] = __float2bfloat16((sh_x[i] - mean) * rstd * __bfloat162float(gamma[i]) + __bfloat162float(beta[i]));
}

// ---------------------------------------------------------------- norms (K2)
// MODE 0: Qwen2RMSNorm.  MODE 1: LayerNorm (gamma, beta).
template <int MODE>
__global__ void norm_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, const __nv_bfloat16* __restrict__ gamma,
                            const __nv_bfloat16* __restrict__ beta, float eps, int dim, __nv_bfloat16* __restrict__ out,
                            int64_t ldo, int n_rows) {
    extern __shared__ float sh_x[];
    float* scratch = sh_x + dim;
    const int r = blockIdx.x;
    if (r >= n_rows) return;
    const __nv_bfloat16* xr = x + (int64_t)r * ldx;
    float s = 0.f, q = 0.f;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) {
        const float v = __bfloat162float(xr[i]);
        sh_x[i] = v;
        s += v;
        q += v * v;
    }
    if (MODE == 0) {
        const float var = block_sum(q, scratch) / dim;
        const float rstd = rsqrtf(var + eps);
        for (int i = threadIdx.x; i < dim; i += blockDim.x) {
            const float y = __bfloat162float(__float2bfloat16(sh_x[i] * rstd));     // .to(input_dtype)
            out[(int64_t)r * ldo + i] = __float2bfloat16(__bfloat162float(gamma[i]) * y);
        }
    } else {
        const float mean = block_sum(s, scratch) / dim;
        float q2 = 0.f;
        for (int i = threadIdx.x; i < dim; i += blockDim.x) { const float d = sh_x[i] - mean; q2 += d * d; }
        const float rstd = rsqrtf(block_sum(q2, scratch) / dim + eps);
        for (int i = threadIdx.x; i < dim; i += blockDim.x)
            out[(int64_t)r * ldo + i] =
                __float2bfloat16((sh_x[i] - mean) * rstd * __bfloat162float(gamma[i]) + __bfloat162float(beta[i]));
    }
}

// Warp-per-row variant for dim % 8 == 0 and dim <= 256 * MAXC (norm_row_warp), 8 rows per 256-thread CTA.
template <int MODE, int MAXC>
__global__ void __launch_bounds__(256)
norm_warp_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, const __nv_bfloat16* __restrict__ gamma,
                 const __nv_bfloat16* __restrict__ beta, float eps, int dim, __nv_bfloat16* __restrict__ out,
                 int64_t ldo, int n_rows) {
    float v[MAXC][8];
    norm_row_warp<MODE, MAXC>(x, ldx, gamma, beta, eps, dim, blockIdx.x * 8 + (threadIdx.x >> 5), n_rows, true, out,
                              ldo, v);
}

template <int MODE>
static bool launch_norm_warp(const void* x, int64_t ldx, const void* gamma, const void* beta, float eps, int n_rows,
                             int dim, void* out, int64_t ldo, cudaStream_t st) {
    const bool aligned = (dim % 8 == 0) && (ldx % 8 == 0) && (ldo % 8 == 0) &&
                         (((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out) |
                            reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta)) & 15) == 0);
    if (!aligned || dim > 4096) return false;
    const int grid = (n_rows + 7) / 8;
    if (dim <= 1024)
        norm_warp_kernel<MODE, 4><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)gamma,
                                                        (const __nv_bfloat16*)beta, eps, dim, (__nv_bfloat16*)out, ldo,
                                                        n_rows);
    else
        norm_warp_kernel<MODE, 16><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)gamma,
                                                         (const __nv_bfloat16*)beta, eps, dim, (__nv_bfloat16*)out, ldo,
                                                         n_rows);
    return true;
}

// ---------------------------------------------------------------- RoPE (K4), in place on packed q|k|v rows
__global__ void rope_kernel(__nv_bfloat16* __restrict__ qkv, int64_t ld, const int32_t* __restrict__ positions,
                            const __nv_bfloat16* __restrict__ cos_t, const __nv_bfloat16* __restrict__ sin_t,
                            int max_pos, int n_heads_qk, int head_dim, int n_tokens) {
    const int t = blockIdx.x;
    if (t >= n_tokens) return;
    const int half = head_dim >> 1;
    int pp = positions[t];
    pp = pp < 0 ? 0 : (pp >= max_pos ? max_pos - 1 : pp);
    const __nv_bfloat16* c = cos_t + (int64_t)pp * half;
    const __nv_bfloat16* s = sin_t + (int64_t)pp * half;
    __nv_bfloat16* row = qkv + (int64_t)t * ld;
    for (int e = threadIdx.x; e < n_heads_qk * half; e += blockDim.x) {
        const int h = e / half, i = e % half;
        __nv_bfloat16* p = row + h * head_dim;
        const float x1 = __bfloat162float(p[i]), x2 = __bfloat162float(p[i + half]);
        const float cf = __bfloat162float(c[i]), sf = __bfloat162float(s[i]);
        // q*cos + rotate_half(q)*sin with every bf16 op rounded, as torch evaluates it on bf16 tensors
        const float a1 = __bfloat162float(__float2bfloat16(x1 * cf));
        const float b1 = __bfloat162float(__float2bfloat16(-x2 * sf));
        const float a2 = __bfloat162float(__float2bfloat16(x2 * cf));
        const float b2 = __bfloat162float(__float2bfloat16(x1 * sf));
        p[i] = __float2bfloat16(a1 + b1);
        p[i + half] = __float2bfloat16(a2 + b2);
    }
}

// 16-byte form (head_dim % 16 == 0, 16-byte aligned rows): a thread rotates 8 (x1, x2) pairs of one head -- two
// 16-byte loads of the row, one of cos, one of sin, two 16-byte stores; same rounding points as rope_kernel.
__global__ void __launch_bounds__(256)
rope_vec_kernel(__nv_bfloat16* __restrict__ qkv, int64_t ld, const int32_t* __restrict__ positions,
                const __nv_bfloat16* __restrict__ cos_t, const __nv_bfloat16* __restrict__ sin_t, int max_pos,
                int n_heads_qk, int head_dim, int n_tokens) {
    const int half = head_dim >> 1, per_head = half >> 3, per_tok = n_heads_qk * per_head;
    const int64_t n_items = (int64_t)n_tokens * per_tok;
    for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < n_items; it += (int64_t)gridDim.x * blockDim.x) {
        const int t = (int)(it / per_tok), e = (int)(it % per_tok);
        const int h = e / per_head, i = (e % per_head) << 3;
        int pp = __ldg(positions + t);
        pp = pp < 0 ? 0 : (pp >= max_pos ? max_pos - 1 : pp);
        __nv_bfloat16* p = qkv + (int64_t)t * ld + h * head_dim + i;
        const uint4 u1 = *reinterpret_cast<const uint4*>(p), u2 = *reinterpret_cast<const uint4*>(p + half);
        const uint4 uc = __ldg(reinterpret_cast<const uint4*>(cos_t + (int64_t)pp * half + i));
        const uint4 us = __ldg(reinterpret_cast<const uint4*>(sin_t + (int64_t)pp * half + i));
        const __nv_bfloat16* x1 = reinterpret_cast<const __nv_bfloat16*>(&u1);
        const __nv_bfloat16* x2 = reinterpret_cast<const __nv_bfloat16*>(&u2);
        const __nv_bfloat16* cc = reinterpret_cast<const __nv_bfloat16*>(&uc);
        const __nv_bfloat16* ss = reinterpret_cast<const __nv_bfloat16*>(&us);
        uint4 o1, o2;
        __nv_bfloat16* y1 = reinterpret_cast<__nv_bfloat16*>(&o1);
        __nv_bfloat16* y2 = reinterpret_cast<__nv_bfloat16*>(&o2);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float a = __bfloat162float(x1[j]), b = __bfloat162float(x2[j]);
            const float cf = __bfloat162float(cc[j]), sf = __bfloat162float(ss[j]);
            const float a1 = __bfloat162float(__float2bfloat16(a * cf));
            const float b1 = __bfloat162float(__float2bfloat16(-b * sf));
            const float a2 = __bfloat162float(__float2bfloat16(b * cf));
            const float b2 = __bfloat162float(__float2bfloat16(a * sf));
            y1[j] = __float2bfloat16(a1 + b1);
            y2[j] = __float2bfloat16(a2 + b2);
        }
        *reinterpret_cast<uint4*>(p) = o1;
        *reinterpret_cast<uint4*>(p + half) = o2;
    }
}

// ---------------------------------------------------------------- pooling + (final norm) + L2 normalise (K9, K10)
// pool: 0 = last token (gte_embeddings.py:42-50), 1 = first token / CLS, 2 = mean over tokens.
// final_norm: 0 none, 1 RMSNorm with `gamma` (Qwen2Model.norm applied only to the pooled row: it is per-token).
// l2: 0 none, 1 bf16 semantics (F.normalize on a bf16 tensor), 2 fp32 semantics (normalize_embeddings=True).
__global__ void pool_normalize_kernel(const __nv_bfloat16* __restrict__ h, int64_t ldh, const int32_t* __restrict__ cu,
                                      int pool, int final_norm, const __nv_bfloat16* __restrict__ gamma, float eps,
                                      int l2, int dim, __nv_bfloat16* __restrict__ out_bf16, float* __restrict__ out_f32,
                                      int n_seq) {
    extern __shared__ float sh_x[];
    float* scratch = sh_x + dim;
    const int b = blockIdx.x;
    if (b >= n_seq) return;
    const int lo = cu[b], hi = cu[b + 1];
    const int len = hi - lo;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) {
        float v = 0.f;
        if (len > 0) {
            if (pool == 0) v = __bfloat162float(h[(int64_t)(hi - 1) * ldh + i]);
            else if (pool == 1) v = __bfloat162float(h[(int64_t)lo * ldh + i]);
            else {
                for (int t = lo; t < hi; ++t) v += __bfloat162float(h[(int64_t)t * ldh + i]);
                v /= (float)len;
            }
        }
        sh_x[i] = v;
    }
    __syncthreads();
    if (final_norm == 1) {
        float q = 0.f;
        for (int i = threadIdx.x; i < dim; i += blockDim.x) q += sh_x[i] * sh_x[i];
        const float rstd = rsqrtf(block_sum(q, scratch) / dim + eps);
        for (int i = threadIdx.x; i < dim; i += blockDim.x) {
            const float y = __bfloat162float(__float2bfloat16(sh_x[i] * rstd));
            sh_x[i] = __bfloat162float(__float2bfloat16(__bfloat162float(gamma[i]) * y));
        }
        __syncthreads();
    }
    float q = 0.f;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) q += sh_x[i] * sh_x[i];
    float nrm = sqrtf(block_sum(q, scratch));
    if (l2 == 1) nrm = __bfloat162float(__float2bfloat16(nrm));      // the norm itself is a bf16 tensor
    nrm = fmaxf(nrm, 1e-12f);
    for (int i = threadIdx.x; i < dim; i += blockDim.x) {
        float v = sh_x[i];
        if (l2 != 0) v = v / nrm;
        const __nv_bfloat16 vb = __float2bfloat16(v);
        out_bf16[(int64_t)b * dim + i] = vb;
        if (out_f32) out_f32[(int64_t)b * dim + i] = (l2 == 2 || l2 == 0) ? v : __bfloat162float(vb);
    }
}

static inline int norm_threads(int dim) { return dim >= 1024 ? 256 : 128; }

}  // namespace ezr

using namespace ezr;

extern "C" {

int ezr_embed_gather(const int32_t* ids, int32_t n_tokens, const void* table, int64_t ldt, int32_t vocab, int32_t dim,
                     void* out, int64_t ldo, void* stream) {
    if (n_tokens == 0) return EZR_OK;
    ProfScope prof(EZR_PROF_ENC_OTHER, (cudaStream_t)stream);
    embed_gather_kernel<<<n_tokens, 128, 0, (cudaStream_t)stream>>>(ids, (const __nv_bfloat16*)table, ldt, vocab, dim,
                                                                   (__nv_bfloat16*)out, ldo, n_tokens);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_bert_embed(const int32_t* ids, const int32_t* positions, int32_t n_tokens, const void* word, const void* pos,
                   const void* type0, const void* gamma, const void* beta, float eps, int32_t vocab, int32_t max_pos,
                   int32_t dim, void* out, void* stream) {
    if (n_tokens == 0) return EZR_OK;
    EZR_CHECK_ARG(dim <= 8192, "bert_embed: dim too large");
    ProfScope prof(EZR_PROF_ENC_OTHER, (cudaStream_t)stream);
    bert_embed_ln_kernel<false><<<n_tokens, norm_threads(dim), (dim + 40) * sizeof(float), (cudaStream_t)stream>>>(
        ids, positions, nullptr, (const __nv_bfloat16*)word, (const __nv_bfloat16*)pos, (const __nv_bfloat16*)type0, 1,
        (const __nv_bfloat16*)gamma, (const __nv_bfloat16*)beta, eps, vocab, max_pos, dim, (__nv_bfloat16*)out, n_tokens);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_bert_embed_typed(const int32_t* ids, const int32_t* positions, const int32_t* types, int32_t n_tokens,
                         const void* word, const void* pos, const void* type_table, int32_t n_types, const void* gamma,
                         const void* beta, float eps, int32_t vocab, int32_t max_pos, int32_t dim, void* out,
                         void* stream) {
    if (n_tokens == 0) return EZR_OK;
    EZR_CHECK_ARG(dim <= 8192, "bert_embed_typed: dim too large");
    EZR_CHECK_ARG(types && type_table && n_types >= 1, "bert_embed_typed: needs types and a type table of >= 1 row");
    ProfScope prof(EZR_PROF_ENC_OTHER, (cudaStream_t)stream);
    bert_embed_ln_kernel<true><<<n_tokens, norm_threads(dim), (dim + 40) * sizeof(float), (cudaStream_t)stream>>>(
        ids, positions, types, (const __nv_bfloat16*)word, (const __nv_bfloat16*)pos, (const __nv_bfloat16*)type_table,
        n_types, (const __nv_bfloat16*)gamma, (const __nv_bfloat16*)beta, eps, vocab, max_pos, dim, (__nv_bfloat16*)out,
        n_tokens);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_rmsnorm(const void* x, int64_t ldx, const void* gamma, float eps, int32_t n_rows, int32_t dim, void* out,
                int64_t ldo, void* stream) {
    if (n_rows == 0) return EZR_OK;
    EZR_CHECK_ARG(dim <= 8192, "rmsnorm: dim too large");
    ProfScope prof(EZR_PROF_ENC_OTHER, (cudaStream_t)stream);
    if (launch_norm_warp<0>(x, ldx, gamma, nullptr, eps, n_rows, dim, out, ldo, (cudaStream_t)stream)) {
        EZR_LAUNCH_CHECK();
        return EZR_OK;
    }
    norm_kernel<0><<<n_rows, norm_threads(dim), (dim + 40) * sizeof(float), (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)gamma, nullptr, eps, dim, (__nv_bfloat16*)out, ldo, n_rows);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_layernorm(const void* x, int64_t ldx, const void* gamma, const void* beta, float eps, int32_t n_rows,
                  int32_t dim, void* out, int64_t ldo, void* stream) {
    if (n_rows == 0) return EZR_OK;
    EZR_CHECK_ARG(dim <= 8192, "layernorm: dim too large");
    ProfScope prof(EZR_PROF_ENC_OTHER, (cudaStream_t)stream);
    if (launch_norm_warp<1>(x, ldx, gamma, beta, eps, n_rows, dim, out, ldo, (cudaStream_t)stream)) {
        EZR_LAUNCH_CHECK();
        return EZR_OK;
    }
    norm_kernel<1><<<n_rows, norm_threads(dim), (dim + 40) * sizeof(float), (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)gamma, (const __nv_bfloat16*)beta, eps, dim,
        (__nv_bfloat16*)out, ldo, n_rows);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_rope(void* qkv, int64_t ld, const int32_t* positions, const void* cos_table, const void* sin_table,
             int32_t max_pos, int32_t n_heads_qk, int32_t head_dim, int32_t n_tokens, void* stream) {
    if (n_tokens == 0) return EZR_OK;
    EZR_CHECK_ARG(head_dim % 2 == 0, "rope: head_dim must be even");
    ProfScope prof(EZR_PROF_ENC_OTHER, (cudaStream_t)stream);
    if (head_dim % 16 == 0 && ld % 8 == 0 && (reinterpret_cast<uintptr_t>(qkv) & 15) == 0 &&
        ((reinterpret_cast<uintptr_t>(cos_table) | reinterpret_cast<uintptr_t>(sin_table)) & 15) == 0) {
        const int64_t n_items = (int64_t)n_tokens * n_heads_qk * (head_dim / 16);
        const int64_t want = (n_items + 255) / 256, cap = (int64_t)sm_count() * 32;
        rope_vec_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, (cudaStream_t)stream>>>(
            (__nv_bfloat16*)qkv, ld, positions, (const __nv_bfloat16*)cos_table, (const __nv_bfloat16*)sin_table, max_pos,
            n_heads_qk, head_dim, n_tokens);
        EZR_LAUNCH_CHECK();
        return EZR_OK;
    }
    rope_kernel<<<n_tokens, 128, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)qkv, ld, positions,
                                                            (const __nv_bfloat16*)cos_table,
                                                            (const __nv_bfloat16*)sin_table, max_pos, n_heads_qk,
                                                            head_dim, n_tokens);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_pool_normalize(const void* hidden, int64_t ldh, const int32_t* cu_seqlens, int32_t n_seq, int32_t pool,
                       int32_t final_norm, const void* gamma, float eps, int32_t l2_mode, int32_t dim, void* out_bf16,
                       float* out_f32, void* stream) {
    if (n_seq == 0) return EZR_OK;
    EZR_CHECK_ARG(pool >= 0 && pool <= 2, "pool_normalize: pool must be 0 (last) 1 (cls) 2 (mean)");
    EZR_CHECK_ARG(final_norm == 0 || gamma != nullptr, "pool_normalize: final norm needs gamma");
    EZR_CHECK_ARG(dim <= 8192, "pool_normalize: dim too large");
    ProfScope prof(EZR_PROF_ENC_OTHER, (cudaStream_t)stream);
    pool_normalize_kernel<<<n_seq, norm_threads(dim), (dim + 40) * sizeof(float), (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)hidden, ldh, cu_seqlens, pool, final_norm, (const __nv_bfloat16*)gamma, eps, l2_mode, dim,
        (__nv_bfloat16*)out_bf16, out_f32, n_seq);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

}  // extern "C"
