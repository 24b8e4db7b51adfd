// Decode attention, "flat" form: one (kv head, context split) task on one CTA, every phase one step deep.
// CausalSelfAttention.java:199-356 for ONE new position: RoPE on the group's queries and on the new key (table-index quirk
// :260-268), append of K/V to the page (:230-243), scores q.K^T * scale over positions [t0, t1) (:324-332), softmax
// (VectorMath.softMax: max, (float)exp((double)(x - max)), sum, divide) and P.V (:349-354).
//
// Why another attention task (jl_attn_task.cuh is the tiled online-softmax one): at decode contexts of tens to a few thousand
// positions the kernel is a latency chain, not a bandwidth problem -- the tiled task spends 4 CTA barriers and two serial
// double-precision exponentials per 32-position tile plus a staging round trip through shared memory (9.5 us at 40
// positions stand-alone, 12 us inside the persistent kernel).  Here:
//   * a warp owns 4 consecutive positions per step (8 lanes per position, HS/8 dims per lane): K and V rows go straight from
//     L2/HBM into registers with fully coalesced 128-bit loads (8 lanes x 64 B = one 512 B head row), no staging tile;
//   * the first step's K and V are requested BEFORE the caller-supplied wait (the persistent kernel's QKV barrier): old
//     positions do not depend on this step's projections;
//   * scores of the whole split go to shared memory, then ONE max, ONE exponential per (position, head) spread over all
//     threads (no serial chains, no running-max corrections), ONE sum -- 4 CTA barriers in total whatever the context;
//   * P.V accumulates in registers (group x HS/8 per lane), 2 shuffles fold the 4 positions of a step, warps meet in smem.
// Contexts longer than FA_MAX_POS positions per split are the caller's business (more splits, or the tiled task).
#pragma once
#include "jl_attn_task.cuh"

#define FA_MAX_POS 1024 // positions per (kv head, split) task
#define FA_HPASS 4      // query heads of the group accumulated per P.V pass (register budget)

template <int HS, int NT>
__host__ __device__ constexpr size_t attention_flat_smem() {
    // qs[MAX_GROUP][HS] + knew[HS] + vnew[HS] + S[FA_MAX_POS][MAX_GROUP] + wmax/wsum[NT/32][MAX_GROUP] x2 + comb[NT/32][FA_HPASS][HS]
    return ((size_t)MG_MAX_GROUP * HS + 2 * HS + (size_t)FA_MAX_POS * MG_MAX_GROUP + 2 * (size_t)(NT / 32) * MG_MAX_GROUP +
            (size_t)(NT / 32) * FA_HPASS * HS) * 4 + 64;
}

// wait(): called by all threads once the first K/V requests are in flight; returns when q/k/v of this step are readable.
// KVDT = JL_I8: I8 page rows (a lane's HS / 8 dimensions lie in one block: one int8 load and one scale load per row part), and the
// owner's append quantises one 32-element block per warp; -1: F32 or BF16 at run time.
template <int HS, int NT, int KVDT = -1, typename Wait>
__device__ __forceinline__ void attention_flat(const AttnParams &P, const int m, const int kvh, const int split, unsigned char *u, Wait wait) {
    constexpr int NW = NT / 32;
    constexpr int DPL = HS / 8;  // dims per lane
    constexpr int NF = DPL / 4;  // float4 per lane per row
    constexpr int hp = HS / 2;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int pp = lane >> 3, sg = lane & 7; // position within the step, segment of the head row
    const int group = P.heads / P.kv_heads;
    float *qs = (float *)u;                         // [group][HS] rotated queries
    float *knew = qs + MG_MAX_GROUP * HS;           // [HS] rotated key of the current position
    float *vnew = knew + HS;                        // [HS]
    float *S = vnew + HS;                           // [FA_MAX_POS][group] scores, then probabilities
    float *wmax = S + (size_t)FA_MAX_POS * MG_MAX_GROUP; // [NW][MAX_GROUP]
    float *wsum = wmax + NW * MG_MAX_GROUP;         // [NW][MAX_GROUP]
    float *comb = wsum + NW * MG_MAX_GROUP;         // [NW][FA_HPASS][HS]

    const int session = P.sessions[m], pos = __ldcg(P.positions + m); // the position may have been advanced inside this launch
    const int n = pos + 1, Sp = P.splits;
    const int per = (((n + Sp - 1) / Sp) + 31) / 32 * 32;
    const int t0 = split * per, t1 = min(n, t0 + per);
    const int cnt = max(0, t1 - t0);
    const int nsteps = (cnt + 3) / 4;
    const int h0 = kvh * group, xoff = kvh * HS, dt = KVDT >= 0 ? KVDT : P.kv.kv_dtype;
    const bool owner = pos >= t0 && pos < t1;
    const int lpage = P.layer / P.kv.layers_per_page, rlayer = P.layer - lpage * P.kv.layers_per_page;
    const size_t v_off = kv_rows_bytes<KVDT>(dt, P.kv.kv_len, P.kv.ctx_per_page);
    const size_t layer_off = kv_rows_bytes<KVDT>(dt, P.kv.kv_len, (size_t)rlayer * 2 * P.kv.ctx_per_page);
    char *const *ptab = (char *const *)P.kv.page_table + ((size_t)session * P.kv.n_layer_pages + lpage) * P.kv.n_ctx_pages;
    auto row_ptr = [&](int position) -> const char * { // K row of `position` (V row = + v_off)
        const int cp = position / P.kv.ctx_per_page, rc = position - cp * P.kv.ctx_per_page;
        return ptab[cp] + layer_off + kv_rows_bytes<KVDT>(dt, P.kv.kv_len, rc);
    };
    // this lane's part of a K or V row: NF float4 (dims [DPL*sg, DPL*sg + DPL)); positions == pos come from smem later
    auto load_part = [&](float4 (&r)[NF], const char *row, bool live) {
        if constexpr (KVDT == JL_I8) {
            static_assert(DPL == 8 || DPL == 16, "one load of a lane's int8 values");
            const size_t e = (size_t)xoff + DPL * sg;
            uint4 w = make_uint4(0u, 0u, 0u, 0u);
            float sc = 0.0f;
            if (live) {
                if constexpr (DPL == 16) w = __ldcg((const uint4 *)(row + e));
                else { const uint2 w2 = __ldcg((const uint2 *)(row + e)); w.x = w2.x, w.y = w2.y; }
                sc = __ldcg((const float *)(row + kv_q8_scale_off(P.kv.kv_len, e)));
            }
            const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int i = 0; i < NF; i++) r[i] = kv_q8x4(ws[i], sc);
            return;
        }
#pragma unroll
        for (int i = 0; i < NF; i++) {
            r[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (live) {
                if (dt == JL_F32) {
                    r[i] = __ldcg((const float4 *)((const float *)row + xoff + DPL * sg + 4 * i));
                } else {
                    const uint2 b = __ldcg((const uint2 *)((const uint16_t *)row + xoff + DPL * sg + 4 * i));
                    r[i] = make_float4(__uint_as_float(b.x << 16), __uint_as_float(b.x & 0xffff0000u), __uint_as_float(b.y << 16),
                                       __uint_as_float(b.y & 0xffff0000u));
                }
            }
        }
    };
    // ---- first step's K and V in flight before the dependency wait ----
    float4 kreg[NF], vreg[NF];
    {
        const int p0 = t0 + 4 * warp + pp;
        const bool live = warp < nsteps && p0 < t1 && p0 != pos;
        const char *row = live ? row_ptr(p0) : nullptr;
        load_part(kreg, row, live);
        load_part(vreg, live ? row + v_off : nullptr, live);
    }
    wait();
    // ---- RoPE on the group's queries (table index poffset + kvh_global*hs + j, :260-268), new key / value ----
    const size_t poffset = (size_t)pos * hp;
    for (int idx = tid; idx < group * hp; idx += NT) {
        const int h = idx / hp, j = idx - h * hp;
        const float2 f = __ldg((const float2 *)P.rope + poffset + (size_t)(P.kv_head0_global + kvh) * HS + j);
        const float *qr = P.q + (size_t)m * P.q_ld + (h0 + h) * HS;
        const float q0 = __ldcg(qr + j), q1 = __ldcg(qr + j + hp);
        qs[h * HS + j] = __fsub_rn(__fmul_rn(q0, f.x), __fmul_rn(q1, f.y));
        qs[h * HS + j + hp] = __fadd_rn(__fmul_rn(q0, f.y), __fmul_rn(q1, f.x));
    }
    if constexpr (KVDT == JL_I8) {
        // the last HS / 32 warps (the ones the q loop leaves idle) each quantise one block of the rotated key and the value
        const int blk = NW - 1 - warp;
        if (owner && blk < HS / 32) {
            const int j = blk * 32 + lane;
            const float r = rope_key_elem(P.k + (size_t)m * P.kv_ld + xoff, (const float2 *)P.rope + poffset + (size_t)(P.kv_head0_global + kvh) * HS, j, hp);
            char *krow = (char *)row_ptr(pos);
            knew[j] = kv_q8_append(krow, P.kv.kv_len, xoff + blk * 32, r);
            vnew[j] = kv_q8_append(krow + v_off, P.kv.kv_len, xoff + blk * 32, __ldcg(P.v + (size_t)m * P.kv_ld + xoff + j));
        }
    } else if (owner) {
        for (int j = NT - 1 - tid; j < hp; j += NT) { // the warps the q loop leaves idle
            const float2 f = __ldg((const float2 *)P.rope + poffset + (size_t)(P.kv_head0_global + kvh) * HS + j);
            const float *kr = P.k + (size_t)m * P.kv_ld + xoff, *vr = P.v + (size_t)m * P.kv_ld + xoff;
            const float k0 = __ldcg(kr + j), k1 = __ldcg(kr + j + hp);
            const float v0 = __ldcg(vr + j), v1 = __ldcg(vr + j + hp);
            const float r0 = __fsub_rn(__fmul_rn(k0, f.x), __fmul_rn(k1, f.y));
            const float r1 = __fadd_rn(__fmul_rn(k0, f.y), __fmul_rn(k1, f.x));
            char *krow = (char *)row_ptr(pos);
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
    task_bar<NT>(); // (1) qs / knew / vnew visible

    // ---- scores: S[pos_local][h] = scale * q_h . k_pos ----
    for (int st = warp; st < nsteps; st += NW) {
        const int pl = 4 * st + pp, position = t0 + pl;
        if (st != warp) { // later steps: fetch now (the first step's rows are already here)
            const bool live = position < t1 && position != pos;
            load_part(kreg, live ? row_ptr(position) : nullptr, live);
        }
        if (position == pos) {
#pragma unroll
            for (int i = 0; i < NF; i++) kreg[i] = *(const float4 *)(knew + DPL * sg + 4 * i);
        }
        for (int h = 0; h < group; h++) {
            float a = 0.0f;
#pragma unroll
            for (int i = 0; i < NF; i++) {
                const float4 qq = *(const float4 *)(qs + h * HS + DPL * sg + 4 * i);
                a = fmaf(qq.x, kreg[i].x, a);
                a = fmaf(qq.y, kreg[i].y, a);
                a = fmaf(qq.z, kreg[i].z, a);
                a = fmaf(qq.w, kreg[i].w, a);
            }
            a += __shfl_xor_sync(0xffffffffu, a, 1);
            a += __shfl_xor_sync(0xffffffffu, a, 2);
            a += __shfl_xor_sync(0xffffffffu, a, 4);
            if (sg == 0 && position < t1) S[pl * group + h] = __fmul_rn(a, P.scale);
        }
    }
    task_bar<NT>(); // (2) scores complete

    // ---- softmax over [t0, t1): thread t owns head t % group (NT is a multiple of every supported group size) ----
    const int hh = tid % group, gper = NT / group;
    float mx = -INFINITY;
    for (int pl = tid / group; pl < cnt; pl += gper) mx = fmaxf(mx, S[pl * group + hh]);
    for (int o = group; o < 32; o <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); // lanes with the same lane % group
    if (lane < group) wmax[warp * MG_MAX_GROUP + lane] = mx;
    task_bar<NT>(); // (3) per-warp maxima
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < NW; w++) M = fmaxf(M, wmax[w * MG_MAX_GROUP + hh]);
    float sum = 0.0f;
    for (int pl = tid / group; pl < cnt; pl += gper) {
        const float e = exp_ref(__fsub_rn(S[pl * group + hh], M)); // (float)Math.exp((double)(x - max)), VectorMath.java:81-84
        S[pl * group + hh] = e;
        sum += e;
    }
    for (int o = group; o < 32; o <<= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane < group) wsum[warp * MG_MAX_GROUP + lane] = sum;
    task_bar<NT>(); // (4) probabilities and per-warp sums

    // ---- P.V: FA_HPASS heads per pass, acc[h][DPL] per lane ----
    for (int hb = 0; hb < group; hb += FA_HPASS) {
        float acc[FA_HPASS][DPL];
#pragma unroll
        for (int h = 0; h < FA_HPASS; h++)
#pragma unroll
            for (int i = 0; i < DPL; i++) acc[h][i] = 0.0f;
        for (int st = warp; st < nsteps; st += NW) {
            const int pl = 4 * st + pp, position = t0 + pl;
            if (st != warp || hb != 0) {
                const bool live = position < t1 && position != pos;
                load_part(vreg, live ? row_ptr(position) + v_off : nullptr, live);
            }
            if (position == pos) {
#pragma unroll
                for (int i = 0; i < NF; i++) vreg[i] = *(const float4 *)(vnew + DPL * sg + 4 * i);
            }
            if (position < t1) {
#pragma unroll
                for (int h = 0; h < FA_HPASS; h++) {
                    if (hb + h < group) {
                        const float p = S[pl * group + hb + h];
#pragma unroll
                        for (int i = 0; i < NF; i++) {
                            acc[h][4 * i] = fmaf(p, vreg[i].x, acc[h][4 * i]);
                            acc[h][4 * i + 1] = fmaf(p, vreg[i].y, acc[h][4 * i + 1]);
                            acc[h][4 * i + 2] = fmaf(p, vreg[i].z, acc[h][4 * i + 2]);
                            acc[h][4 * i + 3] = fmaf(p, vreg[i].w, acc[h][4 * i + 3]);
                        }
                    }
                }
            }
        }
        // fold the 4 positions of a step (lanes pp = 0..3 with the same segment), then park the warp's partial
#pragma unroll
        for (int h = 0; h < FA_HPASS; h++)
#pragma unroll
            for (int i = 0; i < DPL; i++) {
                float a = acc[h][i];
                a += __shfl_xor_sync(0xffffffffu, a, 8);
                a += __shfl_xor_sync(0xffffffffu, a, 16);
                acc[h][i] = a;
            }
        if (pp == 0) {
#pragma unroll
            for (int h = 0; h < FA_HPASS; h++)
#pragma unroll
                for (int i = 0; i < NF; i++)
                    *(float4 *)(comb + ((size_t)warp * FA_HPASS + h) * HS + DPL * sg + 4 * i) =
                        make_float4(acc[h][4 * i], acc[h][4 * i + 1], acc[h][4 * i + 2], acc[h][4 * i + 3]);
        }
        task_bar<NT>(); // (5) partials of this pass
        const int nwa = nsteps < NW ? nsteps : NW; // warps that had at least one step
        for (int idx = tid; idx < FA_HPASS * HS; idx += NT) {
            const int h = idx / HS, d = idx - h * HS;
            if (hb + h >= group) continue;
            float a = 0.0f, L = 0.0f;
            for (int w = 0; w < nwa; w++) a += comb[((size_t)w * FA_HPASS + h) * HS + d];
#pragma unroll
            for (int w = 0; w < NW; w++) L += wsum[w * MG_MAX_GROUP + hb + h];
            if (Sp == 1) {
                P.out[(size_t)m * P.q_ld + (h0 + hb + h) * HS + d] = cnt > 0 ? __fdiv_rn(a, L) : 0.0f;
            } else {
                float *wsp = P.ws + (((size_t)m * P.heads + h0 + hb + h) * Sp + split) * (HS + 2);
                wsp[d] = a;
                if (d == 0) {
                    float Mh = -INFINITY;
                    for (int w = 0; w < NW; w++) Mh = fmaxf(Mh, wmax[w * MG_MAX_GROUP + hb + h]);
                    wsp[HS] = Mh, wsp[HS + 1] = L;
                }
            }
        }
        if (hb + FA_HPASS < group) task_bar<NT>(); // comb is reused by the next pass
    }
}
