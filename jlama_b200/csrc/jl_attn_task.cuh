// Shared device code of the decode attention tasks: one (row, kv head, context split) per CTA-sized thread group.
// The tiled task is run by the stand-alone fused decode attention kernel (jl_attention.cu); the flat task (jl_attn_flat.cuh) and
// attention_merge also by the persistent decode kernel (jl_pdecode.cu, NT = its threads).  CausalSelfAttention.java:199-356.
#pragma once
#include "jl_common.cuh"

#define MG_ATT_TILE 32
#define MG_MAX_GROUP 8

// softmax exponent exactly as the reference computes it: (float)Math.exp((double)x) (one out-of-line copy: the double exp
// is ~150 instructions and the attention kernel starts with a cold instruction cache every layer)
#ifndef JL_EXP_FN
#define JL_EXP_FN __noinline__
#endif
static __device__ JL_EXP_FN float exp_ref(float x) { return (float)exp((double)x); }
// two independent exponentials in one call: the two double-precision dependency chains interleave, so the pair costs
// about the latency of one (the softmax needs exp(s - m_new) and the running-sum correction exp(m_old - m_new) together)
static __device__ JL_EXP_FN float2 exp_ref2(float a, float b) { return make_float2((float)exp((double)a), (float)exp((double)b)); }

template <int NT>
__device__ __forceinline__ void task_bar() {
    asm volatile("bar.sync 1, %0;" ::"n"(NT) : "memory");
}

// shared memory needed by attention_task<HS, NT>
template <int HS, int NT>
__host__ __device__ constexpr size_t attention_task_smem() {
    return (size_t)2 * MG_ATT_TILE * HS * 4 + (size_t)MG_MAX_GROUP * HS * 4 + (size_t)MG_ATT_TILE * MG_MAX_GROUP * 4 + 256 +
           (size_t)2 * HS * 4 + (size_t)(NT / HS) * MG_MAX_GROUP * HS * 4;
}

// One (row m, kv head, split) task.  smem `u` (sized by uarea_bytes) aliases the
// activation staging area, which is dead between the QKV stages and the o_proj prologue.
// Latency plan: the RoPE inputs, the KV append and the first K/V tile are all requested before the first
// barrier; the next tile is prefetched into registers while the current one is processed; the row of the
// current position is taken from shared memory (never re-read from the page it was just written to).
// KVDT: JL_F32 / JL_BF16 / JL_I8 fix the page element type at compile time (half the fetch / append code); -1 = F32 or BF16 at run
// time.  I8 rows are prefetched raw and dequantised as the tile is staged; the owner's append quantises one 32-element block per warp.
template <int HS, int NT, int KVDT = -1>
__device__ void attention_task(const AttnParams &P, int m, int kvh, int split, unsigned char *u) {
    constexpr int C4 = HS / 4;
    constexpr int PARTS = NT / HS; // P.V position groups
    constexpr int NF = (MG_ATT_TILE * C4 + NT - 1) / NT; // float4 per thread per tile
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int group = P.heads / P.kv_heads;
    float4 *Ks = (float4 *)u;                    // [TILE][C4] swizzled
    float4 *Vs = Ks + MG_ATT_TILE * C4;          // [TILE][C4]
    float *qs = (float *)(Vs + MG_ATT_TILE * C4); // [group][HS] rotated queries
    float *ps = qs + MG_MAX_GROUP * HS;          // [TILE][MAX_GROUP]
    float *hm = ps + MG_ATT_TILE * MG_MAX_GROUP; // running max / sum / correction per head
    float *hl = hm + MG_MAX_GROUP;
    float *hc = hl + MG_MAX_GROUP;
    float *knew = hc + MG_MAX_GROUP + 8;         // [HS] rotated key of the current position
    float *vnew = knew + HS;                     // [HS]
    float *comb = vnew + HS;                     // [PARTS][MAX_GROUP][HS] P.V combine buffer

    const int session = P.sessions[m], pos = P.positions[m];
    const int n = pos + 1;
    const int S = P.splits;
    const int per = (((n + S - 1) / S) + MG_ATT_TILE - 1) / MG_ATT_TILE * MG_ATT_TILE;
    const int t0 = split * per, t1 = min(n, t0 + per);
    const int hp = HS / 2;
    const int h0 = kvh * group, xoff = kvh * HS, dt = KVDT >= 0 ? KVDT : P.kv.kv_dtype;
    const size_t poffset = (size_t)pos * hp;
    const bool owner = pos >= t0 && pos < t1;

    // page addressing (KvBufferCache.java:160-199 geometry): the layer split is fixed for the task, the context split is
    // resolved once per tile (a tile of consecutive positions touches at most two pages when ctx_per_page >= TILE)
    const int lpage = P.layer / P.kv.layers_per_page, rlayer = P.layer - lpage * P.kv.layers_per_page;
    const size_t v_off = kv_rows_bytes<KVDT>(dt, P.kv.kv_len, P.kv.ctx_per_page); // K block -> V block of the same layer
    const size_t layer_off = kv_rows_bytes<KVDT>(dt, P.kv.kv_len, (size_t)rlayer * 2 * P.kv.ctx_per_page);
    char *const *ptab = (char *const *)P.kv.page_table + ((size_t)session * P.kv.n_layer_pages + lpage) * P.kv.n_ctx_pages;
    auto k_row = [&](int position) -> char * { // one division: used for single rows only
        const int cp = position / P.kv.ctx_per_page, rc = position - cp * P.kv.ctx_per_page;
        return ptab[cp] + layer_off + kv_rows_bytes<KVDT>(dt, P.kv.kv_len, rc);
    };
    float4 kreg[NF], vreg[NF];
    auto fetch_tile = [&](int tb) {
        const int cp0 = tb / P.kv.ctx_per_page, rc0 = tb - cp0 * P.kv.ctx_per_page;
#pragma unroll
        for (int i = 0; i < NF; i++) {
            const int f = tid + i * NT;
            const int r = f / C4, c4 = f % C4;
            kreg[i] = make_float4(0.f, 0.f, 0.f, 0.f), vreg[i] = kreg[i];
            if (f < MG_ATT_TILE * C4 && tb + r < t1 && tb + r != pos) {
                int cp = cp0, rc = rc0 + r;
                while (rc >= P.kv.ctx_per_page) rc -= P.kv.ctx_per_page, cp++;
                const char *kr = ptab[cp] + layer_off + kv_rows_bytes<KVDT>(dt, P.kv.kv_len, rc);
                const char *vr = kr + v_off;
                if constexpr (KVDT == JL_I8) {
                    // 4 int8 values (.x) and their block's scale (.y), held raw: dequantised when the tile is staged, so that the
                    // prefetch of the next tile stays in flight while this one is processed
                    const size_t e = (size_t)xoff + c4 * 4, so = kv_q8_scale_off(P.kv.kv_len, e);
                    kreg[i] = make_float4(__uint_as_float(__ldcg((const unsigned *)(kr + e))), __ldcg((const float *)(kr + so)), 0.f, 0.f);
                    vreg[i] = make_float4(__uint_as_float(__ldcg((const unsigned *)(vr + e))), __ldcg((const float *)(vr + so)), 0.f, 0.f);
                } else if (dt == JL_F32) {
                    kreg[i] = __ldcg((const float4 *)((const float *)kr + xoff + c4 * 4));
                    vreg[i] = __ldcg((const float4 *)((const float *)vr + xoff + c4 * 4));
                } else {
                    const uint2 uk = __ldcg((const uint2 *)((const uint16_t *)kr + xoff + c4 * 4));
                    const uint2 uv = __ldcg((const uint2 *)((const uint16_t *)vr + xoff + c4 * 4));
                    kreg[i] = make_float4(__uint_as_float(uk.x << 16), __uint_as_float(uk.x & 0xffff0000u),
                                          __uint_as_float(uk.y << 16), __uint_as_float(uk.y & 0xffff0000u));
                    vreg[i] = make_float4(__uint_as_float(uv.x << 16), __uint_as_float(uv.x & 0xffff0000u),
                                          __uint_as_float(uv.y << 16), __uint_as_float(uv.y & 0xffff0000u));
                }
            }
        }
    };
    if (t0 < t1) fetch_tile(t0);

    // RoPE on this group's queries (CausalSelfAttention.java:260-268: table index poffset + kvh_global*hs + j)
    for (int idx = tid; idx < group * hp; idx += NT) {
        const int h = idx / hp, j = idx % hp;
        const float2 f = __ldg((const float2 *)P.rope + poffset + (size_t)(P.kv_head0_global + kvh) * HS + j);
        const float *qr = P.q + (size_t)m * P.q_ld + (h0 + h) * HS;
        const float q0 = __ldcg(qr + j), q1 = __ldcg(qr + j + hp);
        qs[h * HS + j] = __fsub_rn(__fmul_rn(q0, f.x), __fmul_rn(q1, f.y));
        qs[h * HS + j + hp] = __fadd_rn(__fmul_rn(q0, f.y), __fmul_rn(q1, f.x));
    }
    // the split that contains `pos` rotates the key, appends key and value to the page (:230-243,279-285)
    // and keeps both in shared memory for its own scores
    if constexpr (KVDT == JL_I8) {
        // the last HS / 32 warps (the ones the q loop leaves idle) each quantise one block of the rotated key and the value
        const int blk = NT / 32 - 1 - warp;
        if (owner && blk < HS / 32) {
            const int j = blk * 32 + lane;
            const float r = rope_key_elem(P.k + (size_t)m * P.kv_ld + xoff, (const float2 *)P.rope + poffset + (size_t)(P.kv_head0_global + kvh) * HS, j, hp);
            char *krow = k_row(pos);
            knew[j] = kv_q8_append(krow, P.kv.kv_len, xoff + blk * 32, r);
            vnew[j] = kv_q8_append(krow + v_off, P.kv.kv_len, xoff + blk * 32, __ldcg(P.v + (size_t)m * P.kv_ld + xoff + j));
        }
    } else if (owner) {
        for (int j = NT - 1 - tid; j < hp; j += NT) { // use the warps the q loop leaves idle
            const float2 f = __ldg((const float2 *)P.rope + poffset + (size_t)(P.kv_head0_global + kvh) * HS + j);
            const float *kr = P.k + (size_t)m * P.kv_ld + xoff, *vr = P.v + (size_t)m * P.kv_ld + xoff;
            const float k0 = __ldcg(kr + j), k1 = __ldcg(kr + j + hp);
            const float v0 = __ldcg(vr + j), v1 = __ldcg(vr + j + hp);
            float r0 = __fsub_rn(__fmul_rn(k0, f.x), __fmul_rn(k1, f.y));
            float r1 = __fadd_rn(__fmul_rn(k0, f.y), __fmul_rn(k1, f.x));
            char *krow = k_row(pos);
            char *vrow = krow + v_off;
            if (dt == JL_F32) {
                ((float *)krow)[xoff + j] = r0, ((float *)krow)[xoff + j + hp] = r1;
                ((float *)vrow)[xoff + j] = v0, ((float *)vrow)[xoff + j + hp] = v1;
                knew[j] = r0, knew[j + hp] = r1, vnew[j] = v0, vnew[j + hp] = v1;
            } else { // the scores see the values as stored (bf16-rounded), like a later read of the page would
                const uint16_t b0 = f32_to_bf16_rne(r0), b1 = f32_to_bf16_rne(r1), c0 = f32_to_bf16_rne(v0), c1 = f32_to_bf16_rne(v1);
                ((uint16_t *)krow)[xoff + j] = b0, ((uint16_t *)krow)[xoff + j + hp] = b1;
                ((uint16_t *)vrow)[xoff + j] = c0, ((uint16_t *)vrow)[xoff + j + hp] = c1;
                knew[j] = bf16_bits_to_f32(b0), knew[j + hp] = bf16_bits_to_f32(b1);
                vnew[j] = bf16_bits_to_f32(c0), vnew[j + hp] = bf16_bits_to_f32(c1);
            }
        }
    }
    if (tid < group) hm[tid] = -INFINITY, hl[tid] = 0.0f;
    float acc[MG_MAX_GROUP];
#pragma unroll
    for (int h = 0; h < MG_MAX_GROUP; h++) acc[h] = 0.0f;
    const int part = tid / HS, d = tid % HS;
    task_bar<NT>();

    for (int tb = t0; tb < t1; tb += MG_ATT_TILE) {
        const int cnt = min(MG_ATT_TILE, t1 - tb);
        // registers -> shared (the current position's row comes from knew/vnew)
#pragma unroll
        for (int i = 0; i < NF; i++) {
            const int f = tid + i * NT;
            const int r = f / C4, c4 = f % C4;
            if (f < MG_ATT_TILE * C4 && r < cnt) {
                float4 k4 = kreg[i], v4 = vreg[i];
                if constexpr (KVDT == JL_I8) {
                    k4 = kv_q8x4(__float_as_uint(k4.x), k4.y);
                    v4 = kv_q8x4(__float_as_uint(v4.x), v4.y);
                }
                if (tb + r == pos) {
                    k4 = *(const float4 *)(knew + c4 * 4);
                    v4 = *(const float4 *)(vnew + c4 * 4);
                }
                Ks[r * C4 + (c4 ^ (r & 7))] = k4;
                Vs[r * C4 + c4] = v4;
            }
        }
        if (tb + MG_ATT_TILE < t1) fetch_tile(tb + MG_ATT_TILE); // in flight while this tile is processed
        task_bar<NT>();
        // scores (batchDotProduct :324-330, scale :332): 4 threads per (head, position), 1/4 of the head each
        for (int idx = tid; idx < group * MG_ATT_TILE * 4; idx += NT) {
            const int qd = idx & 3, t = (idx >> 2) % MG_ATT_TILE, h = idx / (4 * MG_ATT_TILE);
            float a = 0.0f;
            if (t < cnt) {
                const float4 *q4 = (const float4 *)(qs + h * HS);
#pragma unroll
                for (int c = 0; c < C4 / 4; c++) {
                    const int c4 = qd * (C4 / 4) + c;
                    const float4 k4 = Ks[t * C4 + (c4 ^ (t & 7))];
                    const float4 qq = q4[c4];
                    a = fmaf(qq.x, k4.x, a);
                    a = fmaf(qq.y, k4.y, a);
                    a = fmaf(qq.z, k4.z, a);
                    a = fmaf(qq.w, k4.w, a);
                }
            }
            a += __shfl_xor_sync(0xffffffffu, a, 1);
            a += __shfl_xor_sync(0xffffffffu, a, 2);
            if (qd == 0) ps[t * MG_MAX_GROUP + h] = t < cnt ? __fmul_rn(a, P.scale) : -INFINITY;
        }
        task_bar<NT>();
        // online softmax: warp h owns head h (TILE == 32: one score per lane)
        if (warp < group) {
            const int h = warp;
            const float s0 = ps[lane * MG_MAX_GROUP + h];
            const float m_old = hm[h];
            const float m_new = fmaxf(m_old, warp_max(s0));
            // exp(s - m_new) for this lane's score and, in the same call, the correction exp(m_old - m_new) of the running
            // sum (every lane computes the same correction; lane 0 uses it)
            const float2 ee = exp_ref2(s0 == -INFINITY ? 0.0f : __fsub_rn(s0, m_new), m_old == -INFINITY ? 0.0f : __fsub_rn(m_old, m_new));
            const float e0 = s0 == -INFINITY ? 0.0f : ee.x;
            const float ts = warp_sum(e0);
            ps[lane * MG_MAX_GROUP + h] = e0;
            if (lane == 0) {
                const float corr = m_old == -INFINITY ? 0.0f : ee.y;
                hc[h] = corr, hm[h] = m_new, hl[h] = fmaf(hl[h], corr, ts);
            }
        }
        task_bar<NT>();
        // P.V: thread (part, d) accumulates positions t = part, part+PARTS, ...
#pragma unroll
        for (int h = 0; h < MG_MAX_GROUP; h++)
            if (h < group) acc[h] *= hc[h];
        for (int t = part; t < cnt; t += PARTS) {
            const float v = ((const float *)Vs)[t * HS + d];
#pragma unroll
            for (int h = 0; h < MG_MAX_GROUP; h++)
                if (h < group) acc[h] = fmaf(v, ps[t * MG_MAX_GROUP + h], acc[h]);
        }
        task_bar<NT>(); // tile fully consumed before the next one overwrites Ks/Vs/ps
    }
    // combine the PARTS partial sums
    for (int h = 0; h < group; h++) comb[((size_t)part * MG_MAX_GROUP + h) * HS + d] = acc[h];
    task_bar<NT>();
    if (part == 0) {
        for (int h = 0; h < group; h++) {
            float a = 0.0f;
            for (int pp = 0; pp < PARTS; pp++) a += comb[((size_t)pp * MG_MAX_GROUP + h) * HS + d];
            if (S == 1) {
                P.out[(size_t)m * P.q_ld + (h0 + h) * HS + d] = t0 < t1 ? __fdiv_rn(a, hl[h]) : 0.0f;
            } else {
                float *w = P.ws + (((size_t)m * P.heads + h0 + h) * S + split) * (HS + 2);
                w[d] = a;
                if (d == 0) w[HS] = hm[h], w[HS + 1] = hl[h];
            }
        }
    }
}

// merge the split partials of one (row, kv head): out = sum_s acc_s*exp(m_s-M) / sum_s l_s*exp(m_s-M)
template <int HS, int NT>
__device__ void attention_merge(const AttnParams &P, int m, int kvh, unsigned char *u) {
    const int group = P.heads / P.kv_heads, S = P.splits;
    // rescaling factors exp(m_s - M), one per (head, split), computed once (one exponential deep) instead of S serial
    // exponentials in every (head, d) thread
    float *fac = (float *)u; // [group][S] in the task's shared-memory area (dead once the task's partials are written)
    for (int idx = threadIdx.x; idx < group * S; idx += NT) {
        const int hl = idx / S, s = idx - hl * S;
        const float *w = P.ws + ((size_t)m * P.heads + kvh * group + hl) * S * (HS + 2);
        float M = -INFINITY;
        for (int t = 0; t < S; t++) M = fmaxf(M, __ldcg(w + t * (HS + 2) + HS));
        const float ms = __ldcg(w + s * (HS + 2) + HS);
        fac[idx] = ms == -INFINITY ? 0.0f : exp_ref(__fsub_rn(ms, M));
    }
    task_bar<NT>(); // all NT task threads call this function (whole CTA in the fused kernel, the consumer warps in the megakernel)
    for (int idx = threadIdx.x; idx < group * HS; idx += NT) {
        const int hl = idx / HS, h = kvh * group + hl, d = idx % HS;
        const float *w = P.ws + ((size_t)m * P.heads + h) * S * (HS + 2);
        float num = 0.0f, den = 0.0f;
        for (int s = 0; s < S; s++) {
            const float f = fac[hl * S + s];
            if (f == 0.0f) continue; // empty split (or a contribution that underflows to nothing)
            num = fmaf(__ldcg(w + s * (HS + 2) + d), f, num);
            den = fmaf(__ldcg(w + s * (HS + 2) + HS + 1), f, den);
        }
        P.out[(size_t)m * P.q_ld + h * HS + d] = __fdiv_rn(num, den);
    }
}
