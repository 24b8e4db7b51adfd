// CausalSelfAttention over the paged KV cache (core/model/CausalSelfAttention.java:145-385,
// core/tensor/KvBufferCache.java:99-112,299-352).
//
//  rope_kv_append : per position -- copy k,v rows into the KV page (:230-243), RoPE on q (scratch)
//                   and on k *inside the page* with the reference's table-index quirk (:247-311).
//  paged_attention: per (row, head) -- scores over all pages (batchDotProduct :324-330), scale
//                   (:332), softmax (VectorMath.softMax), P.V (batched saxpy :349-354); split
//                   along the context ("flash decoding") when the context is long.
//
// HBM/L2-bound: K/V rows are read with 128-bit coalesced loads (one head row = hs*4 bytes
// contiguous inside a page row of kv_len floats), reductions are warp shuffles.
#include "jl_common.cuh"
#include "jl_attn_task.cuh"
#include "jl_attn_flat.cuh"
#include <algorithm>

#define ATT_THREADS 128

template <int KVDT = -1>
__device__ __forceinline__ const void *kv_row_ptr(const KvLayout &kv, int session, int layer, int pos, int which) {
    const int lp = layer / kv.layers_per_page, rl = layer % kv.layers_per_page;
    const int cp = pos / kv.ctx_per_page, rc = pos % kv.ctx_per_page;
    const char *base = (const char *)kv.page_table[((size_t)session * kv.n_layer_pages + lp) * kv.n_ctx_pages + cp];
    if constexpr (KVDT == JL_I8) return base + kv_rows_bytes<KVDT>(KVDT, kv.kv_len, ((size_t)rl * 2 + which) * kv.ctx_per_page + rc);
    // F32 / BF16: kept in the element-count form their instantiations were register-allocated with
    const size_t elem = (((size_t)rl * 2 + which) * kv.ctx_per_page + rc) * kv.kv_len;
    return base + elem * (kv.kv_dtype == JL_F32 ? 4 : 2);
}

// one CTA per row (position).  KVDT = JL_I8: every warp quantises whole 32-element blocks of the row; -1: F32 or BF16 at run time.
template <int KVDT = -1>
__global__ void rope_kv_append_kernel(const AttnParams p, float *q) {
    const int row = blockIdx.x;
    const int session = p.sessions[row], pos = p.positions[row];
    const int hs = p.head_size, hp = hs / 2;
    const size_t poffset = (size_t)pos * hp;
    // q heads: rf[poffset + kvh*hs + j]  (CausalSelfAttention.java:260-268)
    float *qr = q + (size_t)row * p.q_ld;
    const int group = p.heads / p.kv_heads;
    for (int idx = threadIdx.x; idx < p.heads * hp; idx += blockDim.x) {
        const int h = idx / hp, j = idx % hp;
        const int kvh_global = (p.head0_global + h) / group;
        const float2 f = ((const float2 *)p.rope)[poffset + (size_t)kvh_global * hs + j];
        const int i = h * hs + j;
        const float q0 = qr[i], q1 = qr[i + hp];
        qr[i] = __fsub_rn(__fmul_rn(q0, f.x), __fmul_rn(q1, f.y));
        qr[i + hp] = __fadd_rn(__fmul_rn(q0, f.y), __fmul_rn(q1, f.x));
    }
    // k heads: rf[poffset + i] with i the GLOBAL column of the key row (:279-285); v copied as is
    void *krow = (void *)kv_row_ptr<KVDT>(p.kv, session, p.layer, pos, 0);
    void *vrow = (void *)kv_row_ptr<KVDT>(p.kv, session, p.layer, pos, 1);
    const float *ks = p.k + (size_t)row * p.kv_ld, *vs = p.v + (size_t)row * p.kv_ld;
    if constexpr (KVDT == JL_I8) { // warp w: blocks w, w + warps, ... of the row (a block lies inside one head)
        const int lane = threadIdx.x & 31;
        for (int e0 = (threadIdx.x >> 5) * 32; e0 < p.kv_heads * hs; e0 += blockDim.x) {
            const int h = e0 / hs, j = e0 - h * hs + lane;
            const float r = rope_key_elem(ks + h * hs, (const float2 *)p.rope + poffset + (size_t)(p.kv_head0_global + h) * hs, j, hp);
            kv_q8_append((char *)krow, p.kv.kv_len, e0, r);
            kv_q8_append((char *)vrow, p.kv.kv_len, e0, vs[e0 + lane]);
        }
        return;
    }
    for (int idx = threadIdx.x; idx < p.kv_heads * hp; idx += blockDim.x) {
        const int h = idx / hp, j = idx % hp;
        const int i = h * hs + j;
        const size_t gi = (size_t)(p.kv_head0_global + h) * hs + j;
        const float2 f = ((const float2 *)p.rope)[poffset + gi];
        const float k0 = ks[i], k1 = ks[i + hp];
        const float r0 = __fsub_rn(__fmul_rn(k0, f.x), __fmul_rn(k1, f.y));
        const float r1 = __fadd_rn(__fmul_rn(k0, f.y), __fmul_rn(k1, f.x));
        if (p.kv.kv_dtype == JL_F32) {
            ((float *)krow)[i] = r0;
            ((float *)krow)[i + hp] = r1;
            ((float *)vrow)[i] = vs[i];
            ((float *)vrow)[i + hp] = vs[i + hp];
        } else {
            ((uint16_t *)krow)[i] = f32_to_bf16_rne(r0);
            ((uint16_t *)krow)[i + hp] = f32_to_bf16_rne(r1);
            ((uint16_t *)vrow)[i] = f32_to_bf16_rne(vs[i]);
            ((uint16_t *)vrow)[i + hp] = f32_to_bf16_rne(vs[i + hp]);
        }
    }
}

int jl_launch_rope_kv_append(jl_ctx *ctx, cudaStream_t s, const AttnParams &p, float *q_inplace) {
    if (p.rows <= 0) return JL_OK;
    JL_CUDA_CHECK(ctx, kv_dispatch<false>(p.kv.kv_dtype, [&](auto t) {
                      return jl_launch_kernel(rope_kv_append_kernel<decltype(t)::value>, dim3(p.rows), dim3(256), 0, s, p, q_inplace);
                  }));
    ctx->launches++;
    return JL_OK;
}

// grid = (kv_heads, rows, splits).  One CTA handles the context range [t0,t1) of one query row for
// ALL query heads of one KV head (GQA group), so every K/V row is read from HBM/L2 once per group.
// The range is walked in tiles of ATT_TILE positions staged in shared memory with coalesced
// 128-bit loads (all loads of a tile in flight together), online softmax across tiles.
#define ATT_TILE 64
// KVDT = JL_I8: the I8 page rows, dequantised as they are staged; -1: F32 or BF16 at run time.
template <int HS, int KVDT = -1>
__global__ void __launch_bounds__(ATT_THREADS) paged_attention_kernel(const AttnParams p) {
    constexpr int C4 = HS / 4;          // float4 per head row
    constexpr int G = ATT_THREADS / HS;  // PV thread groups (1 for hs=128)
    extern __shared__ __align__(16) unsigned char att_smem[];
    float4 *Ks = (float4 *)att_smem;                       // [ATT_TILE][C4] swizzled
    float4 *Vs = Ks + ATT_TILE * C4;                        // [ATT_TILE][C4] plain
    float *qs = (float *)(Vs + ATT_TILE * C4);              // [group][HS]
    float *ps = qs + MG_MAX_GROUP * HS;                    // [ATT_TILE][MG_MAX_GROUP]
    float *hm = ps + ATT_TILE * MG_MAX_GROUP;              // [group] running max
    float *hl = hm + MG_MAX_GROUP;                         // [group] running sum
    float *hc = hl + MG_MAX_GROUP;                         // [group] correction of this tile
    float *comb = hc + MG_MAX_GROUP;                       // [G][MG_MAX_GROUP][HS] (G>1 only)

    const int kvh = blockIdx.x, row = blockIdx.y, split = blockIdx.z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int session = p.sessions[row], pos = p.positions[row];
    const int n = pos + 1;
    const int group = p.heads / p.kv_heads;
    const int per = (((n + p.splits - 1) / p.splits) + ATT_TILE - 1) / ATT_TILE * ATT_TILE;
    const int t0 = split * per;
    const int t1 = min(n, t0 + per);
    const int xoff = kvh * HS;
    const int dt = p.kv.kv_dtype;
    const int h0 = kvh * group;

    if (t0 >= t1) { // empty split
        if (p.splits > 1)
            for (int i = tid; i < group * (HS + 2); i += ATT_THREADS) {
                const int h = i / (HS + 2), d = i % (HS + 2);
                float *w = p.ws + (((size_t)row * p.heads + h0 + h) * p.splits + split) * (HS + 2);
                w[d] = d == HS ? -INFINITY : 0.0f;
            }
        return;
    }
    for (int i = tid; i < group * HS; i += ATT_THREADS) qs[i] = p.q[(size_t)row * p.q_ld + h0 * HS + i];
    if (tid < group) hm[tid] = -INFINITY, hl[tid] = 0.0f;
    float acc[MG_MAX_GROUP];
#pragma unroll
    for (int h = 0; h < MG_MAX_GROUP; h++) acc[h] = 0.0f;
    const int g = tid / HS, d = tid % HS;

    for (int tb = t0; tb < t1; tb += ATT_TILE) {
        const int cnt = min(ATT_TILE, t1 - tb);
        __syncthreads(); // previous tile fully consumed
        // ---- stage K and V tiles (coalesced; every thread issues all its loads before using any) ----
        for (int f = tid; f < cnt * C4; f += ATT_THREADS) {
            const int r = f / C4, c4 = f % C4;
            const void *kr = kv_row_ptr<KVDT>(p.kv, session, p.layer, tb + r, 0);
            const void *vr = kv_row_ptr<KVDT>(p.kv, session, p.layer, tb + r, 1);
            float4 k4, v4;
            if constexpr (KVDT == JL_I8) { // 4 int8 values and their block's scale
                const size_t e = (size_t)xoff + c4 * 4, so = kv_q8_scale_off(p.kv.kv_len, e);
                k4 = kv_q8x4(*(const uint32_t *)((const char *)kr + e), *(const float *)((const char *)kr + so));
                v4 = kv_q8x4(*(const uint32_t *)((const char *)vr + e), *(const float *)((const char *)vr + so));
            } else if (dt == JL_F32) {
                k4 = *(const float4 *)((const float *)kr + xoff + c4 * 4);
                v4 = *(const float4 *)((const float *)vr + xoff + c4 * 4);
            } else {
                const uint2 uk = *(const uint2 *)((const uint16_t *)kr + xoff + c4 * 4);
                const uint2 uv = *(const uint2 *)((const uint16_t *)vr + xoff + c4 * 4);
                k4 = make_float4(__uint_as_float(uk.x << 16), __uint_as_float(uk.x & 0xffff0000u),
                                 __uint_as_float(uk.y << 16), __uint_as_float(uk.y & 0xffff0000u));
                v4 = make_float4(__uint_as_float(uv.x << 16), __uint_as_float(uv.x & 0xffff0000u),
                                 __uint_as_float(uv.y << 16), __uint_as_float(uv.y & 0xffff0000u));
            }
            Ks[r * C4 + (c4 ^ (r & 7))] = k4;
            Vs[r * C4 + c4] = v4;
        }
        __syncthreads();
        // ---- scores: thread -> (head, position); K rows read with the XOR swizzle (conflict-free) ----
        for (int idx = tid; idx < group * ATT_TILE; idx += ATT_THREADS) {
            const int h = idx / ATT_TILE, t = idx % ATT_TILE;
            float s = -INFINITY;
            if (t < cnt) {
                float a = 0.0f;
                const float4 *q4 = (const float4 *)(qs + h * HS);
#pragma unroll 8
                for (int c4 = 0; c4 < C4; c4++) {
                    const float4 k4 = Ks[t * C4 + (c4 ^ (t & 7))];
                    const float4 qq = q4[c4];
                    a = fmaf(qq.x, k4.x, a);
                    a = fmaf(qq.y, k4.y, a);
                    a = fmaf(qq.z, k4.z, a);
                    a = fmaf(qq.w, k4.w, a);
                }
                s = __fmul_rn(a, p.scale); // scale(): CausalSelfAttention.java:332
            }
            ps[t * MG_MAX_GROUP + h] = s;
        }
        __syncthreads();
        // ---- online softmax: warp w owns heads w, w+4, ... (ATT_TILE == 64 -> two scores per lane) ----
        for (int h = warp; h < group; h += ATT_THREADS / 32) {
            const float s0 = ps[lane * MG_MAX_GROUP + h], s1 = ps[(lane + 32) * MG_MAX_GROUP + h];
            const float m_old = hm[h];
            const float m_new = fmaxf(m_old, warp_max(fmaxf(s0, s1)));
            const float e0 = s0 == -INFINITY ? 0.0f : (float)exp((double)__fsub_rn(s0, m_new));
            const float e1 = s1 == -INFINITY ? 0.0f : (float)exp((double)__fsub_rn(s1, m_new));
            const float ts = warp_sum(e0 + e1);
            ps[lane * MG_MAX_GROUP + h] = e0;
            ps[(lane + 32) * MG_MAX_GROUP + h] = e1;
            if (lane == 0) {
                const float corr = m_old == -INFINITY ? 0.0f : (float)exp((double)__fsub_rn(m_old, m_new));
                hc[h] = corr;
                hm[h] = m_new;
                hl[h] = fmaf(hl[h], corr, ts);
            }
        }
        __syncthreads();
        // ---- P.V: thread (g,d) accumulates positions t = g, g+G, ... in order (saxpy :349-354) ----
        if (g < G) {
#pragma unroll
            for (int h = 0; h < MG_MAX_GROUP; h++)
                if (h < group) acc[h] *= hc[h];
            for (int t = g; t < cnt; t += G) {
                const float v = ((const float *)Vs)[t * HS + d];
#pragma unroll
                for (int h = 0; h < MG_MAX_GROUP; h++)
                    if (h < group) acc[h] = fmaf(v, ps[t * MG_MAX_GROUP + h], acc[h]);
            }
        }
    }
    if (G > 1) {
        __syncthreads();
        if (g < G)
            for (int h = 0; h < group; h++) comb[(g * MG_MAX_GROUP + h) * HS + d] = acc[h];
        __syncthreads();
        if (g == 0)
            for (int h = 0; h < group; h++)
                for (int gg = 1; gg < G; gg++) acc[h] += comb[(gg * MG_MAX_GROUP + h) * HS + d];
    }
    if (g == 0) {
        for (int h = 0; h < group; h++) {
            if (p.splits == 1) {
                p.out[(size_t)row * p.q_ld + (h0 + h) * HS + d] = __fdiv_rn(acc[h], hl[h]);
            } else {
                float *w = p.ws + (((size_t)row * p.heads + h0 + h) * p.splits + split) * (HS + 2);
                w[d] = acc[h];
                if (d == 0) w[HS] = hm[h], w[HS + 1] = hl[h];
            }
        }
    }
}

// merge the split partials: out = sum_s acc_s*exp(m_s-M) / sum_s l_s*exp(m_s-M)
template <int HS>
__global__ void attention_merge_kernel(const AttnParams p) {
    const int h = blockIdx.x, row = blockIdx.y, d = threadIdx.x;
    const float *w = p.ws + ((size_t)row * p.heads + h) * p.splits * (HS + 2);
    float M = -INFINITY;
    for (int s = 0; s < p.splits; s++) M = fmaxf(M, w[s * (HS + 2) + HS]);
    float num = 0.0f, den = 0.0f;
    for (int s = 0; s < p.splits; s++) {
        const float m = w[s * (HS + 2) + HS];
        if (m == -INFINITY) continue;
        const float f = (float)exp((double)__fsub_rn(m, M));
        num = fmaf(w[s * (HS + 2) + d], f, num);
        den = fmaf(w[s * (HS + 2) + HS + 1], f, den);
    }
    p.out[(size_t)row * p.q_ld + h * HS + d] = __fdiv_rn(num, den);
}

template <int HS>
static size_t att_smem_bytes() {
    constexpr int G = ATT_THREADS / HS;
    return (size_t)2 * ATT_TILE * HS * 4 + (size_t)MG_MAX_GROUP * HS * 4 + (size_t)ATT_TILE * MG_MAX_GROUP * 4 +
           3 * MG_MAX_GROUP * 4 + (G > 1 ? (size_t)G * MG_MAX_GROUP * HS * 4 : 0);
}
template <int HS, int KVDT>
static int launch_att(jl_ctx *ctx, cudaStream_t s, const AttnParams &p) {
    const size_t smem = att_smem_bytes<HS>();
    static size_t configured[JL_MAX_DEVICES] = {};
    JL_CUDA_CHECK(ctx, (jl_ensure_dyn_smem(paged_attention_kernel<HS, KVDT>, ctx->device, smem, configured)));
    JL_CUDA_CHECK(ctx, jl_launch_kernel(paged_attention_kernel<HS, KVDT>, dim3(p.kv_heads, p.rows, p.splits), dim3(ATT_THREADS),
                                        smem, s, p));
    ctx->launches++;
    if (p.splits > 1) {
        JL_CUDA_CHECK(ctx, jl_launch_kernel(attention_merge_kernel<HS>, dim3(p.heads, p.rows), dim3(HS), 0, s, p));
        ctx->launches++;
    }
    return JL_OK;
}

int jl_launch_paged_attention(jl_ctx *ctx, cudaStream_t s, const AttnParams &p) {
    if (p.rows <= 0) return JL_OK;
    if (p.heads % p.kv_heads || p.heads / p.kv_heads > MG_MAX_GROUP)
        return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "attention: head group size %d/%d unsupported", p.heads, p.kv_heads);
    if (p.splits > 1 && !p.ws) return jl_set_error(ctx, JL_ERR_INVALID, "attention: split workspace missing");
    return kv_dispatch<false>(p.kv.kv_dtype, [&](auto t) {
        constexpr int KVDT = decltype(t)::value;
        switch (p.head_size) {
            case 32: return launch_att<32, KVDT>(ctx, s, p);
            case 64: return launch_att<64, KVDT>(ctx, s, p);
            case 128: return launch_att<128, KVDT>(ctx, s, p);
        }
        return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "attention: head_size %d (supported: 32, 64, 128)", p.head_size);
    });
}

// ---- stand-alone decode attention: RoPE + KV append + scores + softmax + P.V in ONE kernel ----------------------------------
// For decode steps every row is a different session, so a (row, kv head, split) task can append the row's own K/V and attend in
// the same kernel (no separate rope_kv_append launch).  grid = (kv_heads, rows, splits).  The last of the `splits` CTAs of a
// (row, kv head) to arrive merges their partials (decode_attention_epilogue).  done_cnt: the arrival counters (zero before the first
// launch, left zero).
template <int HS, int NT>
__device__ __forceinline__ void decode_attention_epilogue(const AttnParams &p, int m, int kvh, unsigned *done_cnt, unsigned long long *trace,
                                                          unsigned char *smem) {
    __shared__ int s_last;
    if (p.splits > 1) {
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            unsigned *c = &done_cnt[m * p.kv_heads + kvh];
            const unsigned old = atomicAdd(c, 1u);
            s_last = (old == (unsigned)p.splits - 1);
            if (s_last) *c = 0; // ready for the next launch
            __threadfence();
        }
        __syncthreads();
        if (s_last) attention_merge<HS, NT>(p, m, kvh, smem);
    }
    if (trace) {
        __syncthreads();
        ktrace_end(trace);
    }
}

// the tiled task (jl_attn_task.cuh)
#define FDA_THREADS 256
template <int HS, int KVDT>
__global__ void __launch_bounds__(FDA_THREADS) fused_decode_attention_kernel(const AttnParams p, unsigned *done_cnt, unsigned long long *trace) {
    ktrace_begin(trace, 0xA00u | (unsigned long long)p.splits << 16);
    ktrace_mid(trace);
    extern __shared__ __align__(16) unsigned char fda_smem[];
    const int kvh = blockIdx.x, m = blockIdx.y, split = blockIdx.z;
    attention_task<HS, FDA_THREADS, KVDT>(p, m, kvh, split, fda_smem);
    decode_attention_epilogue<HS, FDA_THREADS>(p, m, kvh, done_cnt, trace, fda_smem);
}

// The flat decode task (jl_attn_flat.cuh: K/V rows straight into registers, one exponential per (position, head), 4-5 CTA
// barriers whatever the context).  Used for batched decode (several sessions per step -- the persistent kernel covers the
// single-session case) whenever a split holds <= FA_MAX_POS positions and the GQA group is a power of two; the tiled task above
// stays for everything else.
#define FFA_THREADS 512
template <int HS, int KVDT = -1>
__global__ void __launch_bounds__(FFA_THREADS) flat_decode_attention_kernel(const AttnParams p, unsigned *done_cnt, unsigned long long *trace) {
    ktrace_begin(trace, 0xA00u | (unsigned long long)p.splits << 16);
    ktrace_mid(trace);
    extern __shared__ __align__(16) unsigned char ffa_smem[];
    const int kvh = blockIdx.x, m = blockIdx.y, split = blockIdx.z;
    attention_flat<HS, FFA_THREADS, KVDT>(p, m, kvh, split, ffa_smem, [] {});
    decode_attention_epilogue<HS, FFA_THREADS>(p, m, kvh, done_cnt, trace, ffa_smem);
}

template <int HS, int KVDT, bool FLAT>
static int launch_decode_attention(jl_ctx *ctx, cudaStream_t s, const AttnParams &p, unsigned *done_cnt) {
    void (*kernel)(const AttnParams, unsigned *, unsigned long long *);
    size_t smem;
    if constexpr (FLAT) // the merge step borrows the tiled task's layout
        kernel = flat_decode_attention_kernel<HS, KVDT>, smem = std::max(attention_flat_smem<HS, FFA_THREADS>(), attention_task_smem<HS, FFA_THREADS>());
    else
        kernel = fused_decode_attention_kernel<HS, KVDT>, smem = attention_task_smem<HS, FDA_THREADS>();
    static size_t configured[JL_MAX_DEVICES] = {};
    JL_CUDA_CHECK(ctx, jl_ensure_dyn_smem(kernel, ctx->device, smem, configured));
    unsigned long long *trace = jl_ktrace_slot(ctx);
    JL_CUDA_CHECK(ctx, jl_launch_kernel(kernel, dim3(p.kv_heads, p.rows, p.splits), dim3(FLAT ? FFA_THREADS : FDA_THREADS), smem, s, p,
                                        done_cnt, trace));
    ctx->launches++;
    return JL_OK;
}

// max_pos: the largest position among the rows (bounds the positions a split can hold)
static bool flat_decode_ok(const AttnParams &p, int max_pos) {
    if (p.rows < 2) return false;
    const int group = p.heads / p.kv_heads;
    if (group & (group - 1)) return false;
    if (p.head_size != 64 && p.head_size != 128) return false;
    const int splits = p.splits > 0 ? p.splits : 1;
    const int per = (((max_pos + 1 + splits - 1) / splits) + 31) / 32 * 32;
    return per <= FA_MAX_POS;
}

int jl_launch_fused_decode_attention(jl_ctx *ctx, cudaStream_t s, const AttnParams &p, unsigned *done_cnt, int max_pos) {
    if (p.rows <= 0) return JL_OK;
    if (p.heads % p.kv_heads || p.heads / p.kv_heads > MG_MAX_GROUP)
        return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "attention: head group size %d/%d unsupported", p.heads, p.kv_heads);
    if (max_pos >= 0 && flat_decode_ok(p, max_pos))
        return kv_dispatch<false>(p.kv.kv_dtype, [&](auto t) {
            constexpr int KVDT = decltype(t)::value;
            return p.head_size == 64 ? launch_decode_attention<64, KVDT, true>(ctx, s, p, done_cnt) : launch_decode_attention<128, KVDT, true>(ctx, s, p, done_cnt);
        });
    return kv_dispatch<true>(p.kv.kv_dtype, [&](auto t) {
        constexpr int KVDT = decltype(t)::value;
        switch (p.head_size) {
            case 32: return launch_decode_attention<32, KVDT, false>(ctx, s, p, done_cnt);
            case 64: return launch_decode_attention<64, KVDT, false>(ctx, s, p, done_cnt);
            case 128: return launch_decode_attention<128, KVDT, false>(ctx, s, p, done_cnt);
        }
        return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "attention: head_size %d (supported: 32, 64, 128)", p.head_size);
    });
}
