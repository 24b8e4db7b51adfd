// Prefill attention: a chunk of consecutive query positions of ONE session against the paged KV cache, tiled so that a
// K/V tile is read once per 16 query rows x GQA group instead of once per (row, head).  A pass that holds chunks of several sessions
// (jl_model_batch_forward_multi) runs the same body from a table of CTA row blocks (prefill_attention_table_kernel).
//
// Replaces, for the tensor-core prefill path (jl_model.cu forward_rows_tc), the per-position loop of
// CausalSelfAttention.forward (core/model/CausalSelfAttention.java:199-356: per position scores over all previous keys
// :324-330, scale :332, softmax, P.V :349-354), which at a 2048-token prompt dominated the prefill (VERDICT r1 weak #8).
//
//   * one CTA = one KV head x RB blocks of 16 query rows; warp w owns query head kvh*group + (w % group), rows
//     16 * (w / group): every warp of the CTA consumes the same K/V tile, so GQA sharing is free;
//   * K/V tiles of 64 positions are gathered from the pages (F32, BF16 or I8 cache), rounded to BF16 and staged in shared
//     memory with a 16-byte row pad (ldmatrix is then conflict free); V is consumed through ldmatrix.trans;
//   * S = Q K^T and O += P V on mma.sync.m16n8k16 BF16 -> F32 (the accumulator layout of S is the A-operand layout of
//     the second product, so P never leaves registers); online softmax in F32 with the running max / sum per row;
//   * causal: row r of the chunk (absolute position pos0 + r) sees keys 0 .. pos0 + r; tiles past a warp's last row are
//     skipped, CTAs are issued heaviest first.
//
// Numerics: Q, K, V and P are rounded to BF16, accumulation and softmax are F32 -- the same tolerance class as the BF16
// tensor-core GEMMs around it (1e-2 rel on logits, tests/test_gpu_model.py); the exact path (prefill_tensor_core = 0) keeps
// the per-position F32 kernel of jl_attention.cu.
#include "jl_common.cuh"
#include <cuda_bf16.h>
#include <algorithm>
#include <cstdlib>

#define PA_KT 64 // key positions per tile

__device__ __forceinline__ uint32_t pa_pack(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t *>(&v);
}
__device__ __forceinline__ void pa_ldsm4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void pa_ldsm4t(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(addr));
}

// base of the context page `cp` of (session, layer); K row rc of the layer is at ((rl*2)*ctx_per_page + rc)*kv_len elements,
// the V row `v_off` bytes further (same page, which = 1)
__device__ __forceinline__ const char *pa_page(const KvLayout &kv, int session, int layer, int cp) {
    const int lp = layer / kv.layers_per_page;
    return (const char *)kv.page_table[((size_t)session * kv.n_layer_pages + lp) * kv.n_ctx_pages + cp];
}

// TAB = false: one session, the grid's x covers the chunk in CTA row blocks (heaviest first).  TAB = true: the rows of a pass hold
// chunks of several sessions; CTA x reads its block from `tab` = {session, absolute position of the block's first row, first row of the
// block in the pass, rows in the block (<= 16 * NW / group)}, which the host orders heaviest first.  A block of the table computes what
// the block at the same offset of a single-session launch computes, bit for bit.
template <int HS, int KVDT, int NW, bool TAB>
__device__ __forceinline__ void prefill_attention_body(const AttnParams &p, int session, int pos0, int group, const int4 *tab) {
    constexpr int LDS = HS + 8;  // bf16 elements per staged row
    constexpr int NT = NW * 32;
    constexpr int C4 = HS / 4;   // 4-element groups per row
    constexpr int RPP = NT / C4; // rows staged per pass
    static_assert(NT % C4 == 0 && PA_KT % RPP == 0, "staging shape");
    __shared__ __align__(16) __nv_bfloat16 Ks[PA_KT * LDS];
    __shared__ __align__(16) __nv_bfloat16 Vs[PA_KT * LDS];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int RB = NW / group;
    const int4 e = TAB ? tab[blockIdx.x] : make_int4(0, 0, 0, 0);
    if (TAB) session = e.x, pos0 = e.y;
#define PA_ROWS (TAB ? e.w : p.rows) // (not a local: the single-session kernel re-reads p.rows where it always did)
    const int rbi = TAB ? 0 : gridDim.x - 1 - blockIdx.x; // heaviest (latest rows) first
    const int kvh = blockIdx.y;
    const int head = kvh * group + warp % group;
    const int r0 = (rbi * RB + warp / group) * 16;
    const int cta_r0 = rbi * RB * 16;
    int cta_last = cta_r0 + RB * 16 - 1;
    if (cta_last > PA_ROWS - 1) cta_last = PA_ROWS - 1;
    const int last_key = pos0 + cta_last;                   // last key position any row of this CTA attends to
    const int warp_last_key = pos0 + min(r0 + 15, PA_ROWS - 1);
    const bool warp_live = r0 < PA_ROWS;
    const int ntiles = last_key / PA_KT + 1;
    constexpr int esz = KVDT == JL_F32 ? 4 : (KVDT == JL_BF16 ? 2 : 1); // bytes per stored value (I8: its block scale follows the values)
    // (F32 / BF16 keep the element-count form of these offsets, which is what their instantiations were register-allocated with)
    const size_t v_off = KVDT == JL_I8 ? kv_rows_bytes<KVDT>(KVDT, p.kv.kv_len, p.kv.ctx_per_page) : (size_t)p.kv.ctx_per_page * p.kv.kv_len * esz;

    // Q fragments (rows r0+g and r0+g+8), BF16
    uint32_t qf[HS / 16][4];
    {
        const int ra = r0 + g, rb = r0 + g + 8;
        const float *qa = p.q + ((TAB ? (size_t)e.z : 0) + ra) * p.q_ld + head * HS, *qb = p.q + ((TAB ? (size_t)e.z : 0) + rb) * p.q_ld + head * HS;
#pragma unroll
        for (int ks = 0; ks < HS / 16; ks++) {
            float2 a0 = make_float2(0.f, 0.f), a1 = a0, a2 = a0, a3 = a0;
            if (ra < PA_ROWS) {
                a0 = *(const float2 *)(qa + ks * 16 + 2 * t);
                a2 = *(const float2 *)(qa + ks * 16 + 8 + 2 * t);
            }
            if (rb < PA_ROWS) {
                a1 = *(const float2 *)(qb + ks * 16 + 2 * t);
                a3 = *(const float2 *)(qb + ks * 16 + 8 + 2 * t);
            }
            qf[ks][0] = pa_pack(a0.x, a0.y), qf[ks][1] = pa_pack(a1.x, a1.y);
            qf[ks][2] = pa_pack(a2.x, a2.y), qf[ks][3] = pa_pack(a3.x, a3.y);
        }
    }
    float o[HS / 8][4];
#pragma unroll
    for (int i = 0; i < HS / 8; i++) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f; // rows g and g+8

    const uint32_t ks_base = (uint32_t)__cvta_generic_to_shared(Ks), vs_base = (uint32_t)__cvta_generic_to_shared(Vs);
    const int lm = lane >> 3, lr = lane & 7; // ldmatrix: matrix index and row supplied by this lane
    const int srow = tid / C4, sc4 = tid % C4;

    // A 64-position tile touches at most two context pages; their bases are looked up one tile ahead, so that the row loads of a
    // tile do not wait for a page-table load first.
    const int cpp = p.kv.ctx_per_page;
    const size_t layer_off = (KVDT == JL_I8 ? kv_rows_bytes<KVDT>(KVDT, p.kv.kv_len, ((size_t)(p.layer % p.kv.layers_per_page) * 2) * cpp)
                                            : ((size_t)(p.layer % p.kv.layers_per_page) * 2) * cpp * p.kv.kv_len * esz) +
                             ((size_t)kvh * HS + sc4 * 4) * esz;
    const size_t row_bytes = KVDT == JL_I8 ? kv_rows_bytes<KVDT>(KVDT, p.kv.kv_len, 1) : (size_t)p.kv.kv_len * esz;
    // I8: from this thread's 4 values to their block's scale
    const size_t sc_off = KVDT == JL_I8 ? kv_q8_scale_off(p.kv.kv_len, (size_t)kvh * HS + sc4 * 4) - ((size_t)kvh * HS + sc4 * 4) : 0;
    const char *nb0 = pa_page(p.kv, session, p.layer, 0), *nb1 = nb0;
    {
        const int c1 = min(PA_KT - 1, last_key) / cpp;
        if (c1 != 0) nb1 = pa_page(p.kv, session, p.layer, c1);
    }
    for (int tile = 0; tile < ntiles; tile++) {
        const int t0 = tile * PA_KT;
        const char *b0 = nb0, *b1 = nb1;
        const int cp0 = t0 / cpp;
        if (tile + 1 < ntiles) { // next tile's pages
            const int n0 = (t0 + PA_KT) / cpp, n1 = min(t0 + 2 * PA_KT - 1, last_key) / cpp;
            nb0 = n0 == cp0 ? b0 : pa_page(p.kv, session, p.layer, n0);
            nb1 = n1 == n0 ? nb0 : pa_page(p.kv, session, p.layer, n1);
        }
        __syncthreads(); // the previous tile's fragments have been consumed
        // ---- stage K and V [64][HS] as BF16 ------------------------------------------------------------------
#pragma unroll 8
        for (int r = srow; r < PA_KT; r += RPP) {
            const int pos = t0 + r;
            uint2 kq = make_uint2(0u, 0u), vq = kq;
            if (pos <= last_key) {
                const int cp = pos / cpp;
                // (pages shorter than a tile are looked up per row: the reference solver does not produce them for real models, the
                // I8 geometry does for deep ones, e.g. 80 layers x 45 positions at kv_len 1024)
                const char *pg = cpp >= PA_KT ? (cp == cp0 ? b0 : b1) : pa_page(p.kv, session, p.layer, cp);
                const char *kr = pg + layer_off + (size_t)(pos - cp * cpp) * row_bytes;
                if constexpr (KVDT == JL_I8) { // dequantised to f32, then rounded to BF16 like the F32 pages
                    const float4 kf = kv_q8x4(__ldg((const unsigned *)kr), __ldg((const float *)(kr + sc_off)));
                    const float4 vf = kv_q8x4(__ldg((const unsigned *)(kr + v_off)), __ldg((const float *)(kr + v_off + sc_off)));
                    kq = make_uint2(pa_pack(kf.x, kf.y), pa_pack(kf.z, kf.w));
                    vq = make_uint2(pa_pack(vf.x, vf.y), pa_pack(vf.z, vf.w));
                } else if (KVDT == JL_F32) {
                    const float4 kf = __ldg((const float4 *)kr), vf = __ldg((const float4 *)(kr + v_off));
                    kq = make_uint2(pa_pack(kf.x, kf.y), pa_pack(kf.z, kf.w));
                    vq = make_uint2(pa_pack(vf.x, vf.y), pa_pack(vf.z, vf.w));
                } else {
                    kq = __ldg((const uint2 *)kr), vq = __ldg((const uint2 *)(kr + v_off));
                }
            }
            *(uint2 *)(Ks + r * LDS + sc4 * 4) = kq;
            *(uint2 *)(Vs + r * LDS + sc4 * 4) = vq;
        }
        __syncthreads();
        if (!warp_live || t0 > warp_last_key) continue; // warp-uniform: nothing of this tile is visible to these rows

        // ---- S = Q K^T ----------------------------------------------------------------------------------------
        float s[PA_KT / 8][4];
#pragma unroll
        for (int i = 0; i < PA_KT / 8; i++) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
        for (int ks = 0; ks < HS / 16; ks++) {
#pragma unroll
            for (int nt = 0; nt < PA_KT / 8; nt += 2) {
                uint32_t b[4]; // (nt, k lo) (nt, k hi) (nt+1, k lo) (nt+1, k hi)
                pa_ldsm4(b, ks_base + (uint32_t)((((nt + (lm >> 1)) * 8 + lr) * LDS + ks * 16 + (lm & 1) * 8) * 2));
                mma_bf16(s[nt], qf[ks], b[0], b[1]);
                mma_bf16(s[nt + 1], qf[ks], b[2], b[3]);
            }
        }
        // ---- scale, causal mask, online softmax ---------------------------------------------------------------
        const int lim_a = pos0 + r0 + g, lim_b = lim_a + 8; // last visible key of rows g / g+8
        const bool diag = t0 + PA_KT - 1 > pos0 + r0;        // some element of the tile may be masked
        float mx_a = m_a, mx_b = m_b;
#pragma unroll
        for (int nt = 0; nt < PA_KT / 8; nt++) {
            const int c = t0 + nt * 8 + 2 * t;
            s[nt][0] = (!diag || c <= lim_a) ? s[nt][0] * p.scale : -INFINITY;
            s[nt][1] = (!diag || c + 1 <= lim_a) ? s[nt][1] * p.scale : -INFINITY;
            s[nt][2] = (!diag || c <= lim_b) ? s[nt][2] * p.scale : -INFINITY;
            s[nt][3] = (!diag || c + 1 <= lim_b) ? s[nt][3] * p.scale : -INFINITY;
            mx_a = fmaxf(mx_a, fmaxf(s[nt][0], s[nt][1]));
            mx_b = fmaxf(mx_b, fmaxf(s[nt][2], s[nt][3]));
        }
        mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 1));
        mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 2));
        mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 1));
        mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 2));
        // tile 0 always holds key 0, which every row sees: the running max is finite from the first tile on
        const float al_a = expf(m_a - mx_a), al_b = expf(m_b - mx_b);
        m_a = mx_a, m_b = mx_b;
        float sum_a = 0.f, sum_b = 0.f;
        uint32_t pf[PA_KT / 16][4];
#pragma unroll
        for (int nt = 0; nt < PA_KT / 8; nt++) {
            const float e0 = expf(s[nt][0] - mx_a), e1 = expf(s[nt][1] - mx_a);
            const float e2 = expf(s[nt][2] - mx_b), e3 = expf(s[nt][3] - mx_b);
            sum_a += e0 + e1, sum_b += e2 + e3;
            pf[nt >> 1][(nt & 1) * 2 + 0] = pa_pack(e0, e1);
            pf[nt >> 1][(nt & 1) * 2 + 1] = pa_pack(e2, e3);
        }
        l_a = l_a * al_a + sum_a, l_b = l_b * al_b + sum_b;
#pragma unroll
        for (int i = 0; i < HS / 8; i++) o[i][0] *= al_a, o[i][1] *= al_a, o[i][2] *= al_b, o[i][3] *= al_b;
        // ---- O += P V -----------------------------------------------------------------------------------------
#pragma unroll
        for (int j = 0; j < PA_KT / 16; j++) {
#pragma unroll
            for (int nt = 0; nt < HS / 8; nt += 2) {
                uint32_t b[4]; // (k lo, nt) (k hi, nt) (k lo, nt+1) (k hi, nt+1)
                pa_ldsm4t(b, vs_base + (uint32_t)(((j * 16 + (lm & 1) * 8 + lr) * LDS + (nt + (lm >> 1)) * 8) * 2));
                mma_bf16(o[nt], pf[j], b[0], b[1]);
                mma_bf16(o[nt + 1], pf[j], b[2], b[3]);
            }
        }
    }
    if (!warp_live) return;
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 1);
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 1);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
    const float inv_a = 1.0f / l_a, inv_b = 1.0f / l_b;
    const int ra = r0 + g, rb = ra + 8;
#pragma unroll
    for (int nt = 0; nt < HS / 8; nt++) {
        if (ra < PA_ROWS) *(float2 *)(p.out + ((TAB ? (size_t)e.z : 0) + ra) * p.q_ld + head * HS + nt * 8 + 2 * t) = make_float2(o[nt][0] * inv_a, o[nt][1] * inv_a);
        if (rb < PA_ROWS) *(float2 *)(p.out + ((TAB ? (size_t)e.z : 0) + rb) * p.q_ld + head * HS + nt * 8 + 2 * t) = make_float2(o[nt][2] * inv_b, o[nt][3] * inv_b);
    }
}
#undef PA_ROWS

template <int HS, int KVDT, int NW>
__global__ void __launch_bounds__(NW * 32) prefill_attention_kernel(const AttnParams p, int session, int pos0, int group) {
    prefill_attention_body<HS, KVDT, NW, false>(p, session, pos0, group, nullptr);
}

// (at HS = 64 the table variant is held to the single-session kernel's 128 registers: its table entry would otherwise cost a CTA per SM)
template <int HS, int KVDT, int NW>
__global__ void __launch_bounds__(NW * 32, HS == 64 ? 512 / (NW * 32) : 1) prefill_attention_table_kernel(const AttnParams p, int group, const int4 *tab) {
    prefill_attention_body<HS, KVDT, NW, true>(p, 0, 0, group, tab);
}

bool jl_prefill_attention_supported(const AttnParams &p) {
    if (p.head_size != 64 && p.head_size != 128) return false;
    if (p.kv_heads <= 0 || p.heads % p.kv_heads) return false;
    const int group = p.heads / p.kv_heads;
    if (group != 1 && group != 2 && group != 4 && group != 8) return false;
    if ((p.q_ld % 2) || (p.kv.kv_len % 4)) return false;
    return p.kv.kv_dtype == JL_F32 || p.kv.kv_dtype == JL_BF16 || p.kv.kv_dtype == JL_I8;
}

// 8 warps (32 rows x group 4, or 16 rows x group 8) when there are enough rows to fill the chip: a staged K/V tile then serves twice
// the MMA work, and the staging round trip is what the kernel waits for (ncu: tensor pipe 9 % active).  p.rows = rows of the launch.
static int pa_warps(jl_ctx *ctx, const AttnParams &p) {
    const int group = p.heads / p.kv_heads;
    const char *force = getenv("JL_PA_WARPS"); // tests: "8" / "4" pin the CTA shape regardless of the row count
    const bool big = force ? atoi(force) == 8 : p.rows * p.kv_heads >= 32 * 2 * ctx->sm_count;
    return group == 8 || big ? 8 : 4;
}

template <int HS, int KVDT, bool TAB>
static int launch_pa(jl_ctx *ctx, cudaStream_t s, const AttnParams &p, int session, int pos0, const int4 *tab, int ntab) {
    const int group = p.heads / p.kv_heads;
    const int nw = pa_warps(ctx, p);
    const int rows_per_cta = 16 * (nw / group);
    const dim3 grid(TAB ? ntab : (p.rows + rows_per_cta - 1) / rows_per_cta, p.kv_heads);
    if (TAB && nw == 8) JL_CUDA_CHECK(ctx, jl_launch_kernel(prefill_attention_table_kernel<HS, KVDT, 8>, grid, dim3(256), 0, s, p, group, tab));
    else if (TAB) JL_CUDA_CHECK(ctx, jl_launch_kernel(prefill_attention_table_kernel<HS, KVDT, 4>, grid, dim3(128), 0, s, p, group, tab));
    else if (nw == 8) JL_CUDA_CHECK(ctx, jl_launch_kernel(prefill_attention_kernel<HS, KVDT, 8>, grid, dim3(256), 0, s, p, session, pos0, group));
    else JL_CUDA_CHECK(ctx, jl_launch_kernel(prefill_attention_kernel<HS, KVDT, 4>, grid, dim3(128), 0, s, p, session, pos0, group));
    ctx->launches++;
    return JL_OK;
}

template <bool TAB>
static int launch_pa_any(jl_ctx *ctx, cudaStream_t s, const AttnParams &p, int session, int pos0, const int4 *tab, int ntab) {
    if (!jl_prefill_attention_supported(p)) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "prefill attention: unsupported head shape");
    return kv_dispatch<true>(p.kv.kv_dtype, [&](auto t) {
        constexpr int KVDT = decltype(t)::value;
        return p.head_size == 64 ? launch_pa<64, KVDT, TAB>(ctx, s, p, session, pos0, tab, ntab) : launch_pa<128, KVDT, TAB>(ctx, s, p, session, pos0, tab, ntab);
    });
}

// rows p.rows of one session at positions pos0 .. pos0 + rows - 1; q is post-RoPE, the chunk's own K/V are already in the pages
int jl_launch_prefill_attention(jl_ctx *ctx, cudaStream_t s, const AttnParams &p, int session, int pos0) {
    return launch_pa_any<false>(ctx, s, p, session, pos0, nullptr, 0);
}

// Block table of a pass of several chunks (segs[i] = {session, pos0, first row, rows}): every chunk is cut into the CTA row blocks a
// single-session launch of it would use, and the blocks of all chunks are ordered by the last key they see, heaviest first.
// At most p.rows / 16 + nseg entries.
int jl_prefill_attention_table(jl_ctx *ctx, const AttnParams &p, const int4 *segs, int nseg, int4 *out) {
    const int rpc = 16 * (pa_warps(ctx, p) / (p.heads / p.kv_heads));
    int n = 0;
    for (int i = 0; i < nseg; i++)
        for (int r = 0; r < segs[i].w; r += rpc) out[n++] = make_int4(segs[i].x, segs[i].y + r, segs[i].z + r, min(rpc, segs[i].w - r));
    std::stable_sort(out, out + n, [](const int4 &a, const int4 &b) { return a.y + a.w > b.y + b.w; });
    return n;
}

// the table on the device, built by jl_prefill_attention_table for the same AttnParams shape and row count
int jl_launch_prefill_attention_table(jl_ctx *ctx, cudaStream_t s, const AttnParams &p, const int4 *tab, int ntab) {
    return launch_pa_any<true>(ctx, s, p, 0, 0, tab, ntab);
}
