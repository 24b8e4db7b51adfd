// Many-row decode GEMM: 9..64 activation rows (concurrent sessions) against Q4 / Q8_0 weights that are streamed from HBM ONCE
// per launch for all rows.  gemm8 (jl_gemm8.cu) keeps the Q8 activations of all rows in shared memory and places its 8 sessions on
// the n = 8 of one m16n8k32; at 64 rows and K = 14336 those activations are 918 KB, so this kernel tiles them along K instead.
//
// Arithmetic (the same as gemm8 and the reference's I8 x Q4 / I8 x I8 batchDotProduct, vector_simd.c:384-420):
//   per 32-element block an exact int32 product (u8 nibbles x s8 minus 8 * sum(a) for Q4, s8 x s8 for Q8_0) on the tensor cores
//   (mma.sync.m16n8k32, 16 weight rows x 8 sessions per instruction, NT instructions for 8 * NT sessions), then
//   acc = fmaf(sa * sw, (float)isum, acc) in f32, blocks in K order.  The int32 -> f32 conversion is the exact magic-number form
//   (|isum| <= 32 * 127 * 128 < 2^22): the bit pattern 0x4B400000 + isum is the float 1.5 * 2^23 + isum, so one integer add and
//   one FADD replace the quarter-rate I2F; for Q4 the -8 * sum(a) term is folded into the integer add.
// Prologue (separate launch, gemm64_quant_kernel): RMSNorm (float products summed in double, RMSNorm.java:34-56) and the Q8
//   quantiser (d = max/127, q = (int)(x * (127/max) + 0.5f), PanamaTensorOperations.java:1696-1710) of every row, written once to
//   a global [rows][K] int8 buffer + [K/32][rows] {scale, integer offset} that stays in L2.
// Tiling: a CTA owns 8 strips of 16 weight rows (one per warp, 128 rows) and a range of K.  Every pipeline stage holds one
//   128-byte chunk of each of its 128 weight rows (per-warp cp.async copies, as in gemm8) and the matching K-slice of ALL
//   activation rows (shared by the 8 warps).  When the row groups alone do not cover the SMs (QKV, o_proj, down_proj), K is split
//   over `ks` CTAs; their partial tiles meet in a global workspace and the last CTA to arrive adds them in split order
//   (deterministic: the same inputs give the same bits on every run).
// Epilogues: store, residual add, SiLU(gate) * up -- as gemm8.
// Grouped (mixture of experts, GR): the rows of one launch are the (row, slot) pairs of a step grouped by expert
//   (jl_launch_moe_group); a CTA owns (tile, 128 weight rows of the tile's expert), gathers the tile's quantised rows and their
//   block scales through the pair list, and writes each pair's output row.  No K split: a pair's bits are those of its own row
//   against its expert, whatever the tile it lands in, its place there and the pairs that share the step.
// lm_head (FA): F32 activations, not quantised (AbstractModel.java:444-449); the prologue splits each normalised value exactly into
//   three BF16 planes and the block products run as bf16 x bf16 -> f32 MMAs against the weights as exact BF16 (see fa_chunk).
#include "jl_common.cuh"

#define G64_WARPS 8
#define G64_THREADS (G64_WARPS * 32)
#define G64_MAX_STAGES 6
#define G64_SMEM_LIMIT (227 * 1024)
#define G64_MAGIC 0x4B400000 // float bits of 1.5 * 2^23

// two nibbles (bytes `sel` of x, each 0..15) -> BF16x2 of (nibble - 8), exact: 0x4300 | n is the BF16 128 + n
__device__ __forceinline__ uint32_t g64_nib2bf(uint32_t x, uint32_t sel) {
    const uint32_t v = __byte_perm(x, 0, sel) | 0x43004300u;
    const __nv_bfloat162 r = __hsub2(*(const __nv_bfloat162 *)&v, __floats2bfloat162_rn(136.0f, 136.0f));
    return *(const uint32_t *)&r;
}
// two int8 (bytes 2h, 2h+1 of w) -> BF16x2, exact
__device__ __forceinline__ uint32_t g64_s82bf(uint32_t w, int h) {
    const __nv_bfloat162 r = __floats2bfloat162_rn((float)(int8_t)(w >> (16 * h)), (float)(int8_t)(w >> (16 * h + 8)));
    return *(const uint32_t *)&r;
}

// ---- prologue: (RMSNorm) + Q8 quantisation, one CTA per padded row ----------------------------------------------------------
// Row r < mpad reads source row min(r, M - 1), so the padding rows of the last 8-session tile hold defined values (their outputs
// are never stored).  Layout of `act`: int8 [mpad][K], each 32-byte block permuted so that bytes [8t, 8t + 8) are elements
// 4t..4t+3 and 16+4t..19+4t -- the two B-fragment registers of lane t in one 8-byte load; then uint2 [K/32][mpad] {scale bits,
// G64_MAGIC - 8 * sum(q) for Q4 weights / G64_MAGIC for Q8_0}.
// SPLIT (lm_head, F32 activations): instead of quantising, each (normalised) f32 value a is written as three BF16 planes
// [3][mpad][K] in natural element order, hi = bf16(a), mid = bf16(a - hi), lo = bf16(a - hi - mid): both differences are exact in
// f32 and hi + mid + lo = a exactly (three 8-bit significands cover the 24 of an f32).
template <bool NORM, bool SPLIT>
__global__ void __launch_bounds__(G64_THREADS) gemm64_quant_kernel(const GemvParams p, const int mpad, const int q4) {
    const int r = blockIdx.x, m = r < p.M ? r : p.M - 1;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int K = p.K;
    const float *x = (const float *)p.a + (size_t)m * p.lda + p.a_col_off;
    __shared__ double red_sh[G64_WARPS];
    float rsf = 0.0f;
    if (NORM) {
        double ss = 0.0; // float products summed in double (RMSNorm.java:41-52)
        for (int i = tid * 4; i < K; i += G64_THREADS * 4) {
            const float4 v = *(const float4 *)(x + i);
            ss += (double)__fmul_rn(v.x, v.x) + (double)__fmul_rn(v.y, v.y) + (double)__fmul_rn(v.z, v.z) + (double)__fmul_rn(v.w, v.w);
        }
        ss = warp_sum_d(ss);
        if (lane == 0) red_sh[warp] = ss;
        __syncthreads();
        double tt = 0.0;
        for (int w = 0; w < G64_WARPS; w++) tt += red_sh[w];
        tt = tt / (double)p.norm_E;
        tt += (double)p.norm_eps;
        rsf = (float)(1.0 / sqrt(tt));
    }
    int8_t *aq = (int8_t *)p.wide_act + (size_t)r * K;
    uint2 *ass = (uint2 *)((int8_t *)p.wide_act + (size_t)mpad * K);
    const int nh = K / 16; // half blocks; the two halves of a block sit in adjacent lanes (K / 16 and the stride are even)
    for (int base = 0; base < nh; base += G64_THREADS) {
        const int task = base + tid;
        const bool live = task < nh;
        const int e0 = (live ? task : 0) * 16;
        float v[16];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const float4 f = *(const float4 *)(x + e0 + 4 * i);
            v[4 * i] = f.x, v[4 * i + 1] = f.y, v[4 * i + 2] = f.z, v[4 * i + 3] = f.w;
        }
        if (NORM) {
            float w[16];
            if (p.norm_w_dtype == JL_BF16) {
#pragma unroll
                for (int i = 0; i < 16; i++) w[i] = bf16_bits_to_f32(((const uint16_t *)p.norm_w)[e0 + i]);
            } else {
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const float4 f = __ldg((const float4 *)((const float *)p.norm_w + e0) + i);
                    w[4 * i] = f.x, w[4 * i + 1] = f.y, w[4 * i + 2] = f.z, w[4 * i + 3] = f.w;
                }
            }
#pragma unroll
            for (int i = 0; i < 16; i++) v[i] = __fmul_rn(__fadd_rn(p.norm_adj, w[i]), __fmul_rn(rsf, v[i]));
        }
        if (SPLIT) {
            if (!live) continue;
            uint16_t *pl = (uint16_t *)p.wide_act + (size_t)r * K + e0;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                uint32_t hw[3][4];
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    uint32_t part[3][2];
#pragma unroll
                    for (int k = 0; k < 2; k++) {
                        const float a = v[8 * h + 2 * i + k];
                        const __nv_bfloat16 hi = __float2bfloat16_rn(a);
                        const float r1 = __fsub_rn(a, __bfloat162float(hi));
                        const __nv_bfloat16 mid = __float2bfloat16_rn(r1);
                        const __nv_bfloat16 lo = __float2bfloat16_rn(__fsub_rn(r1, __bfloat162float(mid)));
                        part[0][k] = __bfloat16_as_ushort(hi), part[1][k] = __bfloat16_as_ushort(mid), part[2][k] = __bfloat16_as_ushort(lo);
                    }
#pragma unroll
                    for (int P = 0; P < 3; P++) hw[P][i] = part[P][0] | (part[P][1] << 16);
                }
#pragma unroll
                for (int P = 0; P < 3; P++) *(uint4 *)(pl + (size_t)P * mpad * K + 8 * h) = make_uint4(hw[P][0], hw[P][1], hw[P][2], hw[P][3]);
            }
            continue;
        }
        // PanamaTensorOperations.java:1696-1710: d = max/127, q = (byte)(x*(127/max) + 0.5f), the cast truncates
        float mx = 0.0f;
#pragma unroll
        for (int i = 0; i < 16; i++) mx = fmaxf(mx, fabsf(v[i]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        const float d = __fdiv_rn(mx, 127.0f), id = mx != 0.0f ? __fdiv_rn(127.0f, mx) : 0.0f;
        uint32_t w4[4];
        int sum = 0;
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int q0 = (int)__fadd_rn(__fmul_rn(v[4 * i], id), 0.5f), q1 = (int)__fadd_rn(__fmul_rn(v[4 * i + 1], id), 0.5f);
            const int q2 = (int)__fadd_rn(__fmul_rn(v[4 * i + 2], id), 0.5f), q3 = (int)__fadd_rn(__fmul_rn(v[4 * i + 3], id), 0.5f);
            sum += q0 + q1 + q2 + q3;
            w4[i] = (uint32_t)(q0 & 0xFF) | ((uint32_t)(q1 & 0xFF) << 8) | ((uint32_t)(q2 & 0xFF) << 16) | ((uint32_t)(q3 & 0xFF) << 24);
        }
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        if (!live) continue;
        const int b = e0 >> 5, h = (e0 >> 4) & 1; // half h holds elements 16h + 4t + i: word 2t + h of the permuted block
        uint32_t *dst = (uint32_t *)(aq + (size_t)b * 32);
#pragma unroll
        for (int t = 0; t < 4; t++) dst[2 * t + h] = w4[t];
        if (h == 0) ass[(size_t)b * mpad + r] = make_uint2(__float_as_uint(d), (uint32_t)(G64_MAGIC - (q4 ? 8 * sum : 0)));
    }
}

// ---- main kernel ------------------------------------------------------------------------------------------------------------
// grid = groups * ks: CTA (group, split) computes rows [group * 128, +128) over weight chunks [split * cpk, (split + 1) * cpk).
// FA (lm_head): F32 activations as three BF16 planes (gemm64_quant_kernel<*, true>), read by every warp straight from L2 / L1;
// per block and plane two mma.sync.m16n8k16 (bf16 x bf16 -> f32) with the weights as exact BF16 (nibble - 8 or q), summed into one
// f32 block sum, then acc = fmaf(sw, block sum, acc) in K order.
__device__ __forceinline__ void cp8(uint32_t dst, const void *src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(dst), "l"(src));
}
// GR: grid = tiles * groups, CTA (tile, group); ks == 1
template <int WDT, int EPI, int NT, bool FA, bool GR = false>
__global__ void __launch_bounds__(G64_THREADS, 1) gemm64_kernel(const GemvParams p, const int nst, const int ks) {
    extern __shared__ __align__(16) unsigned char smem[];
    constexpr int NW = EPI == EPI_SILU_MUL ? 2 : 1;
    using S = Strip<WDT>;
    constexpr int BPC = S::BPC, SCS = S::SCS;
    constexpr int KC = BPC * 32;  // K elements per stage
    constexpr int AST = KC + 16;  // staged activation row stride (bytes)
    constexpr int MP = NT * 8; // padded rows
    constexpr int W_BYTES = G64_WARPS * NW * STRIP_STAGE, A_BYTES = FA ? 0 : MP * AST, S_BYTES = FA ? 0 : BPC * MP * 8;
    constexpr int STAGE = W_BYTES + A_BYTES + S_BYTES;
    // gate+up at 48 / 64 rows: 48 / 64 accumulators; a full unroll spills (grouped: from 32 rows, the gather's registers)
    constexpr int UNROLL_U = NW * NT >= (GR ? 8 : 12) ? 1 : BPC;
    __shared__ int last_sh;
    __shared__ int pair_sh[GR ? MP : 1], src_sh[GR ? MP : 1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int K = p.K, nblk = K / 32;
    const int strips = (p.total_rows + 15) / 16;
    int grp = blockIdx.x / ks, split = blockIdx.x - grp * ks, M = p.M, expert = 0;
    if (GR) {
        const int groups = (strips + G64_WARPS - 1) / G64_WARPS, tile = blockIdx.x / groups;
        if (tile >= *p.g_ntiles) return;
        grp = blockIdx.x - tile * groups, split = 0;
        const int4 tl = p.g_tiles[tile];
        expert = tl.x, M = tl.z;
        if (tid < MP) {
            const int pr = p.g_pairs[tl.y + (tid < M ? tid : 0)]; // padding rows repeat the first pair; never stored
            pair_sh[tid] = pr, src_sh[tid] = pr / p.g_div;
        }
        __syncthreads();
    }
    const int strip = grp * G64_WARPS + warp;
    const bool have = strip < strips;
    const int cpk = nblk / BPC / ks; // chunks of this CTA
    const int c0 = split * cpk;
    ktrace_begin(p.trace, 0x200u | (unsigned)EPI | ((unsigned long long)p.M << 8) | ((unsigned long long)p.total_rows << 16) |
                              ((unsigned long long)p.K << 40));

    // this warp's weight tensors: (base pointers, first row) per tensor w; all 16 rows of a strip lie in one tensor
    const void *wb[NW];
    const float *wsb[NW];
    int local0[NW];
#pragma unroll
    for (int w = 0; w < NW; w++) {
        int seg = w, local = (have ? strip : 0) * 16;
        if (NW == 1) {
            seg = 0;
            if (p.nseg > 1 && local >= p.seg[0].rows) {
                local -= p.seg[0].rows, seg = 1;
                if (p.nseg > 2 && local >= p.seg[1].rows) local -= p.seg[1].rows, seg = 2;
            }
        }
        if (GR) wb[w] = p.w_tab[seg][expert], wsb[w] = p.ws_tab[seg][expert];
        else gemv_seg_base(p, seg, wb[w], wsb[w]);
        local0[w] = local;
    }
    const int rows_left = p.total_rows - strip * 16;
    const size_t ldb = (size_t)(p.ldw / 32);
    const unsigned long long pol = l2_evict_first_policy();
    const uint32_t smem_u32 = (uint32_t)__cvta_generic_to_shared(smem);
    const int8_t *act = (const int8_t *)p.wide_act;
    const unsigned char *act_s = (const unsigned char *)p.wide_act + (size_t)(GR ? p.M : MP) * K; // GR: p.M quantised rows

    auto issue = [&](int q) {
        if (q < cpk) {
            const int c = c0 + q;
            const uint32_t st = smem_u32 + (uint32_t)(q % nst) * STAGE;
            if (have) {
                const size_t cb = (size_t)(p.w_col_off / 32) + (size_t)c * BPC;
#pragma unroll
                for (int w = 0; w < NW; w++)
                    strip_stage<WDT>(st + (uint32_t)(warp * NW + w) * STRIP_STAGE, p, wb[w], wsb[w], local0[w], rows_left, ldb, cb, lane, pol);
            }
            if (FA) {
                cp_commit();
                return;
            }
            // activations of every row for this K-slice (L2 hits; default policy keeps them there for the other CTAs)
            const uint32_t as = st + W_BYTES;
            for (int i = tid; i < MP * (KC / 16); i += G64_THREADS) {
                const int r = i / (KC / 16), o = (i - r * (KC / 16)) * 16;
                cp16(as + r * AST + o, act + (size_t)(GR ? src_sh[r] : r) * K + (size_t)c * KC + o);
            }
            const uint32_t ss = as + A_BYTES;
            if (GR) // the {scale, offset} of each gathered row, block by block: [BPC][MP] as the staged layout
                for (int i = tid; i < BPC * MP; i += G64_THREADS) {
                    const int u = i / MP, r = i - u * MP;
                    cp8(ss + i * 8, act_s + ((size_t)(c * BPC + u) * p.M + src_sh[r]) * 8);
                }
            else
                for (int i = tid; i < S_BYTES / 16; i += G64_THREADS) cp16(ss + i * 16, act_s + (size_t)c * S_BYTES + (size_t)i * 16);
        }
        cp_commit();
    };
    for (int i = 0; i < nst - 1; i++) issue(i);

    float acc[NW][NT][4];
#pragma unroll
    for (int w = 0; w < NW; w++)
#pragma unroll
        for (int j = 0; j < NT; j++)
#pragma unroll
            for (int i = 0; i < 4; i++) acc[w][j][i] = 0.0f;

    // FA: one staged weight chunk against the BF16 planes of every row.  The k-slots of a block are permuted consistently on both
    // operands: lane t supplies elements 4t..4t+3 (first MMA) and 16+4t..19+4t (second), k-slots 2t, 2t+1, 2t+8, 2t+9 of each.
    const uint16_t *fa_act = (const uint16_t *)p.wide_act;
    auto fa_chunk = [&](const unsigned char *st, int c) {
        const unsigned char *ws = st + warp * STRIP_STAGE; // NW == 1
#pragma unroll 1
        for (int u = 0; u < BPC; u++) {
            uint32_t A[2][4];
            if (WDT == JL_Q4) {
                const uint32_t w0 = *(const uint32_t *)(ws + g * S::ROWB + u * 16 + 4 * t), w1 = *(const uint32_t *)(ws + (g + 8) * S::ROWB + u * 16 + 4 * t);
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const uint32_t x0 = (w0 >> (4 * h)) & 0x0F0F0F0Fu, x1 = (w1 >> (4 * h)) & 0x0F0F0F0Fu;
                    A[h][0] = g64_nib2bf(x0, 0x4140), A[h][1] = g64_nib2bf(x1, 0x4140), A[h][2] = g64_nib2bf(x0, 0x4342), A[h][3] = g64_nib2bf(x1, 0x4342);
                }
            } else {
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const uint32_t w0 = *(const uint32_t *)(ws + g * S::ROWB + u * 32 + 16 * h + 4 * t);
                    const uint32_t w1 = *(const uint32_t *)(ws + (g + 8) * S::ROWB + u * 32 + 16 * h + 4 * t);
                    A[h][0] = g64_s82bf(w0, 0), A[h][1] = g64_s82bf(w1, 0), A[h][2] = g64_s82bf(w0, 1), A[h][3] = g64_s82bf(w1, 1);
                }
            }
            const float sw0 = *(const float *)(ws + S::SC_OFF + g * SCS + u * 4), sw1 = *(const float *)(ws + S::SC_OFF + (g + 8) * SCS + u * 4);
            const size_t e = (size_t)c * KC + u * 32 + 4 * t;
#pragma unroll
            for (int j = 0; j < NT; j++) {
                const uint16_t *ar = fa_act + (size_t)(8 * j + g) * K + e;
                float cf[4] = {0.0f, 0.0f, 0.0f, 0.0f}; // block sum, the small planes first
#pragma unroll
                for (int P = 2; P >= 0; P--) {
                    const uint16_t *pp = ar + (size_t)P * MP * K;
                    const uint2 b0 = __ldg((const uint2 *)pp), b1 = __ldg((const uint2 *)(pp + 16));
                    mma_bf16(cf, A[0], b0.x, b0.y);
                    mma_bf16(cf, A[1], b1.x, b1.y);
                }
                acc[0][j][0] = fmaf(sw0, cf[0], acc[0][j][0]);
                acc[0][j][1] = fmaf(sw0, cf[1], acc[0][j][1]);
                acc[0][j][2] = fmaf(sw1, cf[2], acc[0][j][2]);
                acc[0][j][3] = fmaf(sw1, cf[3], acc[0][j][3]);
            }
        }
    };

    for (int q = 0; q < cpk; q++) {
        cp_wait(nst - 2); // this thread's copies of stage q have landed ...
        __syncthreads();   // ... and every thread's; all threads are also done with stage q - 1, which the next issue overwrites
        issue(q + nst - 1);
        if (!have) continue;
        const unsigned char *st = smem + (size_t)(q % nst) * STAGE;
        if (FA) {
            fa_chunk(st, c0 + q);
            continue;
        }
        const unsigned char *as = st + W_BYTES, *ss = as + A_BYTES;
#pragma unroll
        for (int w = 0; w < NW; w++) {
            const unsigned char *ws = st + (warp * NW + w) * STRIP_STAGE;
#pragma unroll(UNROLL_U)
            for (int u = 0; u < BPC; u++) {
                uint32_t a0, a1, a2, a3;
                if (WDT == JL_Q4) {
                    // bytes [4t, 4t+4) of a block: low nibbles = elements 4t..4t+3, high nibbles = elements 16+4t..19+4t
                    const uint32_t w0 = *(const uint32_t *)(ws + g * S::ROWB + u * 16 + 4 * t), w1 = *(const uint32_t *)(ws + (g + 8) * S::ROWB + u * 16 + 4 * t);
                    a0 = w0 & 0x0F0F0F0Fu, a1 = w1 & 0x0F0F0F0Fu, a2 = (w0 >> 4) & 0x0F0F0F0Fu, a3 = (w1 >> 4) & 0x0F0F0F0Fu;
                } else {
                    const unsigned char *r0p = ws + g * S::ROWB + u * 32 + 4 * t, *r1p = ws + (g + 8) * S::ROWB + u * 32 + 4 * t;
                    a0 = *(const uint32_t *)r0p, a1 = *(const uint32_t *)r1p, a2 = *(const uint32_t *)(r0p + 16), a3 = *(const uint32_t *)(r1p + 16);
                }
                const float sw0 = *(const float *)(ws + S::SC_OFF + g * SCS + u * 4), sw1 = *(const float *)(ws + S::SC_OFF + (g + 8) * SCS + u * 4);
#pragma unroll
                for (int j = 0; j < NT; j++) {
                    const uint2 bf = *(const uint2 *)(as + (8 * j + g) * AST + u * 32 + 8 * t);
                    int c[4] = {0, 0, 0, 0};
                    if (WDT == JL_Q4) mma_u8s8(c, a0, a1, a2, a3, bf.x, bf.y);
                    else mma_s8s8(c, a0, a1, a2, a3, bf.x, bf.y);
                    // c[0] = (row g, session 8j+2t), c[1] = (row g, 8j+2t+1), c[2] = (row g+8, 8j+2t), c[3] = (row g+8, 8j+2t+1)
                    const uint4 s = *(const uint4 *)(ss + ((size_t)u * MP + 8 * j + 2 * t) * 8);
                    const float sa0 = __uint_as_float(s.x), sa1 = __uint_as_float(s.z);
                    const float f0 = __fsub_rn(__int_as_float(c[0] + (int)s.y), 12582912.0f), f1 = __fsub_rn(__int_as_float(c[1] + (int)s.w), 12582912.0f);
                    const float f2 = __fsub_rn(__int_as_float(c[2] + (int)s.y), 12582912.0f), f3 = __fsub_rn(__int_as_float(c[3] + (int)s.w), 12582912.0f);
                    acc[w][j][0] = fmaf(__fmul_rn(sa0, sw0), f0, acc[w][j][0]); // acc += (sa*sb) * isum   (vector_simd.c:384-420)
                    acc[w][j][1] = fmaf(__fmul_rn(sa1, sw0), f1, acc[w][j][1]);
                    acc[w][j][2] = fmaf(__fmul_rn(sa0, sw1), f2, acc[w][j][2]);
                    acc[w][j][3] = fmaf(__fmul_rn(sa1, sw1), f3, acc[w][j][3]);
                }
            }
        }
    }
    cp_wait(0);

    if (ks > 1) {
        // split-K: publish this CTA's tile; the last CTA of the group adds all tiles in split order
        constexpr int TILE = NW * NT * 4 * G64_THREADS;
        float *part = p.wide_part + (size_t)blockIdx.x * TILE;
#pragma unroll
        for (int w = 0; w < NW; w++)
#pragma unroll
            for (int j = 0; j < NT; j++)
#pragma unroll
                for (int i = 0; i < 4; i++) __stcg(part + ((w * NT + j) * 4 + i) * G64_THREADS + tid, acc[w][j][i]);
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            const unsigned old = atomicAdd(&p.wide_cnt[grp], 1u);
            last_sh = old == (unsigned)(ks - 1);
            if (last_sh) p.wide_cnt[grp] = 0; // every CTA of the group has arrived: reset for the next launch
        }
        __syncthreads();
        if (!last_sh) return;
        __threadfence();
        const float *p0 = p.wide_part + (size_t)grp * ks * TILE;
#pragma unroll
        for (int w = 0; w < NW; w++)
#pragma unroll
            for (int j = 0; j < NT; j++)
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const int idx = ((w * NT + j) * 4 + i) * G64_THREADS + tid;
                    float v = __ldcg(p0 + idx);
                    for (int s2 = 1; s2 < ks; s2++) v = __fadd_rn(v, __ldcg(p0 + (size_t)s2 * TILE + idx));
                    acc[w][j][i] = v;
                }
    }
    if (have) {
        // ---- epilogue: rows strip*16 + g (+8) in the concatenated row space of the launch, sessions 8j + 2t (+1) ----
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int rr = strip * 16 + g + 8 * h;
            if (rr >= p.total_rows) continue;
            int seg = 0, local = rr;
            if (NW == 1 && p.nseg > 1 && local >= p.seg[0].rows) {
                local -= p.seg[0].rows, seg = 1;
                if (p.nseg > 2 && local >= p.seg[1].rows) local -= p.seg[1].rows, seg = 2;
            }
            const GemvSeg &sg = p.seg[seg];
#pragma unroll
            for (int j = 0; j < NT; j++)
#pragma unroll
                for (int jj = 0; jj < 2; jj++) {
                    const int m = 8 * j + 2 * t + jj;
                    if (m >= M) continue;
                    const int o = GR ? pair_sh[m] : m;
                    float v = acc[NW - 1][j][2 * h + jj];
                    if (EPI == EPI_ADD_RESIDUAL) v = __fadd_rn(v, p.residual[(size_t)o * p.res_ld + (p.row0 + local)]);
                    if (EPI == EPI_SILU_MUL) v = __fmul_rn(silu_ref(acc[0][j][2 * h + jj]), v);
                    sg.out[(size_t)o * sg.out_ld + p.row0 + local + sg.out_off] = v;
                }
        }
    }
    if (p.trace) {
        __syncthreads();
        ktrace_end(p.trace);
    }
}

static int g64_nt(int M) { return M <= 16 ? 2 : (M <= 32 ? 4 : (M <= 48 ? 6 : 8)); }
static bool g64_fa(int prologue) { return prologue == PRO_F32 || prologue == PRO_RMSNORM_F32; }
static size_t g64_stage(int wdt, int epi, int nt, bool fa) {
    const int bpc = wdt == JL_Q4 ? 8 : 4, kc = bpc * 32, nw = epi == EPI_SILU_MUL ? 2 : 1;
    return (size_t)G64_WARPS * nw * STRIP_STAGE + (fa ? 0 : (size_t)nt * 8 * (kc + 16) + (size_t)bpc * nt * 8 * 8);
}
static int g64_stages(int wdt, int epi, int nt, bool fa) {
    const int n = (int)((G64_SMEM_LIMIT - 1024) / g64_stage(wdt, epi, nt, fa));
    return n > G64_MAX_STAGES ? G64_MAX_STAGES : n;
}

// the larger of the Q8 layout (int8 rows + {scale, offset} per block) and the three BF16 planes of F32 activations
size_t jl_gemm64_act_bytes(int K) { return (size_t)3 * JL_MAX_DECODE_ROWS * K * 2; }
size_t jl_gemm64_part_floats(int sm_count) { return (size_t)sm_count * 2 * 8 * 4 * G64_THREADS; }

// the weight shape, prologue and epilogue of a launch at NT row tiles: Q4 / Q8_0 weights, whole 128-byte chunks; Q8 activations
// made in the prologue, or F32 activations (store epilogue, one tensor: the lm_head) split into BF16 planes in the prologue
static bool g64_shape_ok(const GemvParams &p, int prologue, int epilogue, int nt) {
    if (p.w_dtype != JL_Q4 && p.w_dtype != JL_I8) return false;
    const bool fa = g64_fa(prologue);
    if (prologue != PRO_F32_QUANT && prologue != PRO_RMSNORM_QUANT && !fa) return false;
    if (fa && (epilogue != EPI_STORE || p.nseg != 1)) return false;
    const int bpc = p.w_dtype == JL_Q4 ? 8 : 4;
    if ((p.K % 32) || ((p.K / 32) % bpc) || (p.a_col_off % 4) || (p.lda % 4)) return false;
    if ((p.ldw % 32) || ((p.ldw / 32) % bpc) || (p.w_col_off % (32 * bpc))) return false; // 16-byte aligned cp.async sources
    const bool norm = prologue == PRO_RMSNORM_QUANT || prologue == PRO_RMSNORM_F32;
    if (norm && p.norm_w_dtype != JL_BF16 && p.norm_w_dtype != JL_F32) return false;
    if (epilogue == EPI_SILU_MUL && p.nseg != 2) return false;
    if (epilogue != EPI_SILU_MUL)
        for (int i = 0; i + 1 < p.nseg; i++)
            if (p.seg[i].rows % 16) return false; // a strip must not straddle two weight tensors
    return g64_stages(p.w_dtype, epilogue, nt, fa) >= 2;
}

// usable for this launch?  9..64 rows
bool jl_gemm64_supported(const GemvParams &p, int prologue, int epilogue) {
    if (p.M <= GEMV_MAX_M || p.M > JL_MAX_DECODE_ROWS || p.sel) return false;
    if (!p.wide_act || !p.wide_part || !p.wide_cnt) return false;
    return g64_shape_ok(p, prologue, epilogue, g64_nt(p.M));
}

// grouped: tiles of R = 16, 32, 48 or 64 rows (NT = R / 8), the smallest that holds every pair of an expert when no expert can
// receive more than max_rows_per_expert (a step's rows: top-k selects distinct experts), 64 past that
int jl_gemm64_group_rows(int max_rows_per_expert) { return 8 * g64_nt(max_rows_per_expert); }
size_t jl_gemm64_q8_bytes(int rows, int K) { return (size_t)rows * K + (size_t)rows * (K / 32) * 8; }
bool jl_gemm64_grouped_supported(const GemvParams &p, int prologue, int epilogue, int R) {
    if (R != 8 * g64_nt(R) || p.M < 1 || p.sel || !p.wide_act || !p.g_tiles || !p.g_ntiles || !p.g_pairs || p.g_div < 1) return false;
    if (!p.w_tab[0] || !p.ws_tab[0] || (epilogue == EPI_SILU_MUL && (!p.w_tab[1] || !p.ws_tab[1]))) return false;
    if (prologue != PRO_F32_QUANT && prologue != PRO_RMSNORM_QUANT) return false;
    if (epilogue == EPI_ADD_RESIDUAL) return false; // a pair's output row is not a residual row
    return g64_shape_ok(p, prologue, epilogue, R / 8);
}

// K splits: the smallest power of two (<= 8, dividing the chunk count) whose CTAs cover the SMs, and no more CTAs than SMs
static int g64_ksplit(const GemvParams &p, int sm_count) {
    const int groups = ((p.total_rows + 15) / 16 + G64_WARPS - 1) / G64_WARPS;
    const int nch = (p.K / 32) / (p.w_dtype == JL_Q4 ? 8 : 4);
    int ks = 1;
    while (ks < 8 && groups * ks * 2 <= sm_count && nch % (ks * 2) == 0) ks *= 2;
    return ks;
}

// tiles > 0: grouped, one CTA per (tile, group) and no K split
template <int WDT, int EPI, int NT, bool FA, bool GR>
static int launch_g64(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int tiles) {
    auto kern = gemm64_kernel<WDT, EPI, NT, FA, GR>;
    const int nst = g64_stages(WDT, EPI, NT, FA);
    const size_t smem = (size_t)nst * g64_stage(WDT, EPI, NT, FA);
    static size_t configured[JL_MAX_DEVICES] = {};
    JL_CUDA_CHECK(ctx, jl_ensure_dyn_smem(kern, ctx->device, smem, configured));
    const int groups = ((p.total_rows + 15) / 16 + G64_WARPS - 1) / G64_WARPS;
    const int ks = GR ? 1 : g64_ksplit(p, ctx->sm_count);
    JL_CUDA_CHECK(ctx, jl_launch_kernel(kern, dim3(groups * (GR ? tiles : ks)), dim3(G64_THREADS), smem, stream, p, nst, ks));
    ctx->launches++;
    return JL_OK;
}
template <int WDT, int EPI, bool FA, bool GR = false>
static int launch_g64_n(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int nt, int tiles = 0) {
    switch (nt) {
        case 2: return launch_g64<WDT, EPI, 2, FA, GR>(ctx, stream, p, tiles);
        case 4: return launch_g64<WDT, EPI, 4, FA, GR>(ctx, stream, p, tiles);
        case 6: return launch_g64<WDT, EPI, 6, FA, GR>(ctx, stream, p, tiles);
        default: return launch_g64<WDT, EPI, 8, FA, GR>(ctx, stream, p, tiles);
    }
}
template <int WDT>
static int launch_g64_e(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue, int epilogue) {
    const int nt = g64_nt(p.M);
    if (g64_fa(prologue)) return launch_g64_n<WDT, EPI_STORE, true>(ctx, stream, p, nt);
    switch (epilogue) {
        case EPI_STORE: return launch_g64_n<WDT, EPI_STORE, false>(ctx, stream, p, nt);
        case EPI_ADD_RESIDUAL: return launch_g64_n<WDT, EPI_ADD_RESIDUAL, false>(ctx, stream, p, nt);
        default: return launch_g64_n<WDT, EPI_SILU_MUL, false>(ctx, stream, p, nt);
    }
}

// the prologue of mpad rows into p.wide_act
static int g64_prologue(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue, int mpad) {
    const int q4 = p.w_dtype == JL_Q4 ? 1 : 0;
    cudaError_t e;
    switch (prologue) {
        case PRO_RMSNORM_QUANT: e = jl_launch_kernel(gemm64_quant_kernel<true, false>, dim3(mpad), dim3(G64_THREADS), 0, stream, p, mpad, q4); break;
        case PRO_F32_QUANT: e = jl_launch_kernel(gemm64_quant_kernel<false, false>, dim3(mpad), dim3(G64_THREADS), 0, stream, p, mpad, q4); break;
        case PRO_RMSNORM_F32: e = jl_launch_kernel(gemm64_quant_kernel<true, true>, dim3(mpad), dim3(G64_THREADS), 0, stream, p, mpad, q4); break;
        default: e = jl_launch_kernel(gemm64_quant_kernel<false, true>, dim3(mpad), dim3(G64_THREADS), 0, stream, p, mpad, q4); break;
    }
    JL_CUDA_CHECK(ctx, e);
    ctx->launches++;
    return JL_OK;
}

int jl_launch_gemm64(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue, int epilogue) {
    const int rc = g64_prologue(ctx, stream, p, prologue, g64_nt(p.M) * 8);
    if (rc != JL_OK) return rc;
    return p.w_dtype == JL_Q4 ? launch_g64_e<JL_Q4>(ctx, stream, p, prologue, epilogue) : launch_g64_e<JL_I8>(ctx, stream, p, prologue, epilogue);
}

template <int WDT>
static int launch_g64_grouped(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int epilogue, int nt, int tiles) {
    if (epilogue == EPI_SILU_MUL) return launch_g64_n<WDT, EPI_SILU_MUL, false, true>(ctx, stream, p, nt, tiles);
    return launch_g64_n<WDT, EPI_STORE, false, true>(ctx, stream, p, nt, tiles);
}

// the p.M rows of p.a quantised once (the prologue of jl_launch_gemm64), then the grouped GEMM over `tiles` tile entries
int jl_launch_gemm64_grouped(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p_in, int prologue, int epilogue, int R, int tiles) {
    if (!jl_gemm64_grouped_supported(p_in, prologue, epilogue, R)) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "gemm64 grouped: launch not supported");
    if (tiles < 1) return JL_OK;
    GemvParams p = p_in;
    p.trace = nullptr, p.norm_inv_E = p.norm_E > 0 ? 1.0 / (double)p.norm_E : 0.0;
    const int rc = g64_prologue(ctx, stream, p, prologue, p.M);
    if (rc != JL_OK) return rc;
    return p.w_dtype == JL_Q4 ? launch_g64_grouped<JL_Q4>(ctx, stream, p, epilogue, R / 8, tiles)
                              : launch_g64_grouped<JL_I8>(ctx, stream, p, epilogue, R / 8, tiles);
}
