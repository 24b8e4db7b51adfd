// Batched-decode GEMM: 2..8 activation rows (concurrent sessions, the reference's "batch": KvBufferCache.java:58-60,
// AbstractModel.java:295-312) against block-quantised weights that are streamed ONCE for all sessions.
//
// The reference arithmetic (I8 x Q4 / I8 x I8 batchDotProduct: PanamaTensorOperations.java:768-1044, vector_simd.c:261-437) is an
// exact int32 dot product per 32-element block, scaled by (sa * sb) and accumulated in f32.  With 8 sessions the dp4a form of
// jl_gemv.cu needs 64 dp4a per weight block per lane and is issue-bound at ~1/4 of the HBM rate; this shape IS a small GEMM,
// so the integer block products go to the tensor cores with mma.sync.m16n8k32 (u8/s8 x s8 -> s32, exact): 16 weight rows x 8
// sessions x one 32-element block per instruction; the per-block scaling stays in f32 registers.  (wgmma would bring nothing at
// N = 8: the kernel is bound by the weight stream, not by the MMA.)
//   Q4: a lane's 32-bit load is bytes [4t, 4t+4) of a block = low nibbles of elements 4t..4t+3 and high nibbles of elements
//       16+4t..19+4t -- exactly the k-slots of that lane's A fragment (a0 / a2), no shuffles; nibbles stay unsigned (u8) and the
//       -8 offset is taken out with the activation block sums, as in the GEMV.
//   I8: a lane's 64-bit load is bytes [8t, 8t+8) of a block; the k index inside a block is permuted consistently on both operands
//       (an int32 sum does not care), so the activation fragment is one 64-bit shared-memory load.
// Prologue (fused): RMSNorm (RMSNorm.java:34-56) and the Q8 activation quantiser (PanamaTensorOperations.java:1684-1723) for all
// rows; epilogues: store, residual add, SiLU(gate) * up.
#include "jl_common.cuh"

#define G8_MAX_WARPS 16
#define G8_PAD 16        // bytes added to a session's activation row in shared memory: makes the fragment loads bank-conflict free
#define G8_MAX_STAGES 6
#define G8_SMEM_LIMIT (227 * 1024)

// first weight/scale block of (strip, sub-tensor w) rows; all 16 rows of a strip lie in one tensor (jl_gemm8_supported)
template <int NW>
__device__ __forceinline__ void g8_strip_base(const GemvParams &p, int strip, int w, const void *&wb, const float *&wsb, int &local0) {
    int seg = w, local = strip * 16;
    if (NW == 1) {
        seg = 0;
        if (p.nseg > 1 && local >= p.seg[0].rows) {
            local -= p.seg[0].rows, seg = 1;
            if (p.nseg > 2 && local >= p.seg[1].rows) local -= p.seg[1].rows, seg = 2;
        }
    }
    gemv_seg_base(p, seg, wb, wsb);
    local0 = local;
}

// The weights reach the tensor cores through per-warp cp.async pipelines: a stage holds a 128-byte chunk of each of the 16 rows of
// a strip (+ their block scales); 16-byte copies, 8 lanes per row chunk (whole 128-byte lines), `nst` stages per warp sized by the
// shared memory left beside the activations -- about 2 KB x (nst - 1) in flight per warp, ~10 MB on the chip, which is what the
// HBM latency x bandwidth product asks for.  A warp walks a flat list of (strip, tensor, chunk) tasks, so its pipeline never drains
// between strips, and the first stages are issued BEFORE the activation prologue so that the prologue hides their latency.
// NWARP = 8 or 16 warps per CTA (one CTA per SM): 16 when the shared memory left beside the activations still gives every warp a
// 3-stage pipeline (K <= 8192) -- the main loop is a chain of shared-memory -> MMA -> FMA steps and 8 warps leave the issue slots
// 60 % idle (ncu: issue active 40 %, occupancy 12.5 %)
template <int WDT, int EPI, int PRO, int NWARP>
__global__ void __launch_bounds__(NWARP * 32, 1) gemm8_kernel(const GemvParams p, const int nst, const int ksplit) {
    constexpr int G8_THREADS = NWARP * 32, G8_WARPS = NWARP;
    extern __shared__ __align__(16) unsigned char smem[];
    constexpr bool NORM = PRO == PRO_RMSNORM_QUANT;
    constexpr int NW = EPI == EPI_SILU_MUL ? 2 : 1;
    using S = Strip<WDT>;
    constexpr int BPC = S::BPC, SCS = S::SCS;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int K = p.K, nblk = K / 32, M = p.M;
    const int astride = K + G8_PAD;                       // bytes per session row
    int8_t *aq = (int8_t *)smem;                          // [8][astride]
    const int sst = nblk + 1;                             // scale / sum row stride (+1: the sessions a lane group reads hit different banks)
    uint2 *ass = (uint2 *)(smem + (size_t)8 * astride);   // [8][sst] {scale bits, block sum}
    unsigned char *stages = (unsigned char *)(ass + (size_t)8 * sst) + (size_t)warp * nst * STRIP_STAGE;
    const uint32_t stages_u32 = (uint32_t)__cvta_generic_to_shared(stages);
    __shared__ double red_sh[G8_WARPS][8];
    __shared__ float rs_sh[8];
    ktrace_begin(p.trace, 0x100u | (unsigned)EPI | ((unsigned long long)PRO << 4) | ((unsigned long long)p.total_rows << 16) | ((unsigned long long)p.K << 40));

    // ---- this warp's task list ----
    // The reduction dimension of a strip is split over `ksplit` warps of the CTA (8 for the Llama shapes): a lone warp walking all
    // of K is a chain of dependent shared-memory -> MMA -> FMA steps (about 7 us at K = 4096) however fast the weights arrive.
    // Round r gives the CTA 8 / ksplit strips; a warp owns chunk range [part * cpp, (part + 1) * cpp) of its strip, the partial
    // sums meet in shared memory and are added in part order by the part-0 warp (deterministic).
    const int strips = (p.total_rows + 15) / 16;
    const int nch = nblk / BPC;
    const int part = warp % ksplit, slot = warp / ksplit, spr = G8_WARPS / ksplit;
    const int cpp = nch / ksplit; // chunks per part
    const int rstride = gridDim.x * spr;
    const int strip0 = blockIdx.x * spr + slot;                                    // strip of round 0
    const int rounds = (strips + rstride - 1) / rstride;                           // the same for every warp of the grid
    const int my_rounds = strip0 < strips ? (strips - 1 - strip0) / rstride + 1 : 0; // rounds in which this warp has a strip
    const int ntask = my_rounds * NW * cpp;
    const unsigned long long pol = l2_evict_first_policy();
    // producer cursor
    int p_q = 0, p_c = 0, p_w = 0, p_strip = strip0;
    auto issue = [&]() {
        if (p_q < ntask) {
            const void *wb;
            const float *wsb;
            int local0;
            g8_strip_base<NW>(p, p_strip, p_w, wb, wsb, local0);
            const uint32_t st = stages_u32 + (uint32_t)(p_q % nst) * STRIP_STAGE;
            const int rows_left = p.total_rows - p_strip * 16; // rows of this strip that exist (>= 1)
            const size_t ldb = (size_t)(p.ldw / 32);
            const size_t cb = (size_t)(p.w_col_off / 32) + (size_t)(part * cpp + p_c) * BPC;
            strip_stage<WDT>(st, p, wb, wsb, local0, rows_left, ldb, cb, lane, pol);
            if (++p_c == cpp) {
                p_c = 0;
                if (++p_w == NW) p_w = 0, p_strip += rstride;
            }
        }
        p_q++;
        cp_commit();
    };
    for (int i = 0; i < nst - 1; i++) issue();

    // ---- prologue: (RMSNorm) + Q8 quantisation of the M rows; rows >= M are zero ----
    if (NORM) {
        // sum of squares: float products summed in double (RMSNorm.java:41-52), all threads on every row
        double ss[8];
#pragma unroll
        for (int m = 0; m < 8; m++) ss[m] = 0.0;
        for (int i = tid * 4; i < K; i += G8_THREADS * 4) {
#pragma unroll
            for (int m = 0; m < 8; m++) {
                if (m < M) {
                    const float4 v = *(const float4 *)((const float *)p.a + (size_t)m * p.lda + p.a_col_off + i);
                    ss[m] += (double)__fmul_rn(v.x, v.x) + (double)__fmul_rn(v.y, v.y) + (double)__fmul_rn(v.z, v.z) + (double)__fmul_rn(v.w, v.w);
                }
            }
        }
#pragma unroll
        for (int m = 0; m < 8; m++) {
            if (m < M) {
                const double r = warp_sum_d(ss[m]);
                if (lane == 0) red_sh[warp][m] = r;
            }
        }
        __syncthreads();
        if (tid < M) {
            double tt = 0.0;
            for (int w = 0; w < G8_WARPS; w++) tt += red_sh[w][tid];
            tt = tt / (double)p.norm_E;
            tt += (double)p.norm_eps;
            rs_sh[tid] = (float)(1.0 / sqrt(tt));
        }
        __syncthreads();
    }
    // rows >= M: zero activations (their columns of the MMA are never stored)
    for (int i = tid; i < (8 - M) * (K / 16); i += G8_THREADS) {
        const int m = M + i / (K / 16), e0 = (i % (K / 16)) * 16;
        *(uint4 *)(aq + (size_t)m * astride + e0) = make_uint4(0u, 0u, 0u, 0u);
        if ((e0 & 16) == 0) ass[m * sst + (e0 >> 5)] = make_uint2(0u, 0u);
    }
    // a task = 16 consecutive elements = half a block; G8_PB tasks per thread are loaded before any is processed (the loop is
    // otherwise a chain of dependent L2 round trips: 8 at K = 4096, 28 at K = 14336)
    constexpr int G8_PB = 4;
    const int ntasks = M * (K / 16);
    for (int base = 0; base < ntasks; base += G8_THREADS * G8_PB) {
        float4 ld[G8_PB][4];
#pragma unroll
        for (int j = 0; j < G8_PB; j++) {
            const int task = base + j * G8_THREADS + tid;
            if (task < ntasks) {
                const int m = task / (K / 16), e0 = (task - m * (K / 16)) * 16;
                const float4 *x = (const float4 *)((const float *)p.a + (size_t)m * p.lda + p.a_col_off + e0);
#pragma unroll
                for (int i = 0; i < 4; i++) ld[j][i] = x[i];
            }
        }
#pragma unroll
        for (int j = 0; j < G8_PB; j++) {
            const int task = base + j * G8_THREADS + tid;
            // the two halves of a block sit in adjacent lanes and K/16 is even, so a lane pair is either both live or both idle
            if (task >= ntasks) continue;
            const int m = task / (K / 16), e0 = (task - m * (K / 16)) * 16;
            float v[16];
#pragma unroll
            for (int i = 0; i < 4; i++) v[4 * i] = ld[j][i].x, v[4 * i + 1] = ld[j][i].y, v[4 * i + 2] = ld[j][i].z, v[4 * i + 3] = ld[j][i].w;
            if (NORM) {
                const float rsf = rs_sh[m];
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
            // PanamaTensorOperations.java:1696-1710: d = max/127, q = (byte)(x*(127/max) + 0.5f), the cast truncates
            float mx = 0.0f;
#pragma unroll
            for (int i = 0; i < 16; i++) mx = fmaxf(mx, fabsf(v[i]));
            const unsigned pair = __activemask();
            mx = fmaxf(mx, __shfl_xor_sync(pair, mx, 1));
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
            sum += __shfl_xor_sync(pair, sum, 1);
            *(uint4 *)(aq + (size_t)m * astride + e0) = make_uint4(w4[0], w4[1], w4[2], w4[3]);
            if ((e0 & 16) == 0) ass[m * sst + (e0 >> 5)] = make_uint2(__float_as_uint(d), (uint32_t)sum);
        }
    }
    __syncthreads();
    ktrace_mid(p.trace);

    // ---- main loop: rounds of (strip, tensor, chunk) tasks ----
    const int8_t *arow = aq + (size_t)g * astride; // this lane's session (B fragment column n = g)
    float *red = (float *)(stages - (size_t)warp * nst * STRIP_STAGE + (size_t)G8_WARPS * nst * STRIP_STAGE); // [2][8 warps][NW][4][32]
    int q = 0;
    for (int r = 0; r < rounds; r++) {
        const int strip = strip0 + r * rstride;
        const bool have = r < my_rounds;
        float acc[NW][4];
#pragma unroll
        for (int w = 0; w < NW; w++)
#pragma unroll
            for (int i = 0; i < 4; i++) acc[w][i] = 0.0f;
        if (have) {
#pragma unroll
            for (int w = 0; w < NW; w++) {
                for (int cc = 0; cc < cpp; cc++, q++) {
                    cp_wait(nst - 2); // task q has landed (for this lane's copies) ...
                    __syncwarp();     // ... and for every lane's; all lanes are also done with task q - 1, whose stage the next issue overwrites
                    issue();
                    const unsigned char *st = stages + (size_t)(q % nst) * STRIP_STAGE;
                    const int cbase = (part * cpp + cc) * BPC;
#pragma unroll
                    for (int u = 0; u < BPC; u++) {
                        const int b = cbase + u;
                        int c[4] = {0, 0, 0, 0};
                        const uint32_t bl = *(const uint32_t *)(arow + b * 32 + 4 * t), bh = *(const uint32_t *)(arow + b * 32 + 16 + 4 * t);
                        if (WDT == JL_Q4) {
                            // bytes [4t, 4t+4) of a block = low nibbles of elements 4t..4t+3 and high nibbles of elements 16+4t..19+4t: the
                            // k-slots of this lane's A fragment registers a0 / a2 (rows g, g+8 -> a0,a2 / a1,a3)
                            const uint32_t w0 = *(const uint32_t *)(st + g * S::ROWB + u * 16 + 4 * t), w1 = *(const uint32_t *)(st + (g + 8) * S::ROWB + u * 16 + 4 * t);
                            mma_u8s8(c, w0 & 0x0F0F0F0Fu, w1 & 0x0F0F0F0Fu, (w0 >> 4) & 0x0F0F0F0Fu, (w1 >> 4) & 0x0F0F0F0Fu, bl, bh);
                        } else {
                            const unsigned char *r0p = st + g * S::ROWB + u * 32 + 4 * t, *r1p = st + (g + 8) * S::ROWB + u * 32 + 4 * t;
                            mma_s8s8(c, *(const uint32_t *)r0p, *(const uint32_t *)r1p, *(const uint32_t *)(r0p + 16), *(const uint32_t *)(r1p + 16), bl, bh);
                        }
                        const float sw0 = *(const float *)(st + S::SC_OFF + g * SCS + u * 4), sw1 = *(const float *)(st + S::SC_OFF + (g + 8) * SCS + u * 4);
                        // c[0] = (row g, session 2t), c[1] = (row g, 2t+1), c[2] = (row g+8, 2t), c[3] = (row g+8, 2t+1)
                        const uint2 s0 = ass[(2 * t) * sst + b], s1 = ass[(2 * t + 1) * sst + b];
                        const float sa0 = __uint_as_float(s0.x), sa1 = __uint_as_float(s1.x);
                        if (WDT == JL_Q4) { // sum a*(nib-8) = sum a*nib - 8*sum a   (exact)
                            const int z0 = 8 * (int)s0.y, z1 = 8 * (int)s1.y;
                            c[0] -= z0, c[1] -= z1, c[2] -= z0, c[3] -= z1;
                        }
                        acc[w][0] = fmaf(__fmul_rn(sa0, sw0), (float)c[0], acc[w][0]); // acc += (sa*sb) * isum   (vector_simd.c:384-420)
                        acc[w][1] = fmaf(__fmul_rn(sa1, sw0), (float)c[1], acc[w][1]);
                        acc[w][2] = fmaf(__fmul_rn(sa0, sw1), (float)c[2], acc[w][2]);
                        acc[w][3] = fmaf(__fmul_rn(sa1, sw1), (float)c[3], acc[w][3]);
                    }
                }
            }
        }
        if (ksplit > 1) {
            float *rb = red + (size_t)(r & 1) * (G8_WARPS * NW * 128);
            if (have && part != 0) {
#pragma unroll
                for (int w = 0; w < NW; w++)
#pragma unroll
                    for (int i = 0; i < 4; i++) rb[((warp * NW + w) * 4 + i) * 32 + lane] = acc[w][i];
            }
            __syncthreads(); // one barrier per round: the buffers alternate, and a reader is done before it arrives at the next one
            if (have && part == 0) {
                for (int pp = 1; pp < ksplit; pp++)
#pragma unroll
                    for (int w = 0; w < NW; w++)
#pragma unroll
                        for (int i = 0; i < 4; i++) acc[w][i] = __fadd_rn(acc[w][i], rb[(((warp + pp) * NW + w) * 4 + i) * 32 + lane]);
            }
        }
        if (!have || part != 0) continue;
        // ---- epilogue of `strip`: rows strip*16 + g and + 8 in the concatenated row space of the launch ----
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
            for (int j = 0; j < 2; j++) {
                const int m = 2 * t + j;
                if (m >= M) continue;
                float v = acc[NW - 1][2 * h + j];
                if (EPI == EPI_ADD_RESIDUAL) v = __fadd_rn(v, p.residual[(size_t)m * p.res_ld + (p.row0 + local)]);
                if (EPI == EPI_SILU_MUL) v = __fmul_rn(silu_ref(acc[0][2 * h + j]), v);
                sg.out[(size_t)m * sg.out_ld + p.row0 + local + sg.out_off] = v;
            }
        }
    }
    cp_wait(0);
    if (p.trace) {
        __syncthreads();
        ktrace_end(p.trace);
    }
}

static size_t g8_act_smem(const GemvParams &p) { return (size_t)8 * (p.K + G8_PAD) + (size_t)8 * (p.K / 32 + 1) * 8; }
static size_t g8_red_bytes(int nwarp) { return (size_t)2 * nwarp * 2 * 128 * 4; } // partial sums of the K split: [2 buffers][warps][2 tensors][4 x 32 lanes] f32
static int g8_stages(const GemvParams &p, int nwarp) {
    const size_t act = g8_act_smem(p) + g8_red_bytes(nwarp);
    if (act + 2048 >= G8_SMEM_LIMIT) return 0;
    int n = (int)((G8_SMEM_LIMIT - 2048 - act) / ((size_t)nwarp * STRIP_STAGE));
    return n > G8_MAX_STAGES ? G8_MAX_STAGES : n;
}
static size_t g8_smem(const GemvParams &p, int nwarp) { return g8_act_smem(p) + g8_red_bytes(nwarp) + (size_t)g8_stages(p, nwarp) * nwarp * STRIP_STAGE; }
// warps per CTA: 16 while every warp still gets a 3-stage pipeline
static int g8_warps(const GemvParams &p) { return g8_stages(p, 16) >= 3 ? 16 : 8; }
// warps of a CTA sharing one strip: the largest of 8, 4, 2, 1 that divides the chunk count of a row
// Measured at the 8B shapes (gpurun_out/r2_gemv_batch.txt): the split pays while a round's strips do not fill the warps of the
// chip (o_proj 18.4 -> 14.4 us, down 53 -> 36 us) and costs a little once they do (lm_head 114 -> 129 us): split only as far as
// needed to give every warp work.
static int g8_ksplit(const GemvParams &p, int sm_count, int nwarp) {
    const int nch = (p.K / 32) / (p.w_dtype == JL_Q4 ? 8 : 4);
    const int strips = (p.total_rows + 15) / 16;
    int want = 1;
    while (want < nwarp && strips * want < sm_count * nwarp) want <<= 1;
    for (int s = want; s > 1; s >>= 1)
        if (nch % s == 0) return s;
    return 1;
}

// usable for this launch?  (2..8 rows, quantised weights with Q8 activations produced in the prologue, whole 128-byte chunks)
bool jl_gemm8_supported(const GemvParams &p, int prologue, int epilogue) {
    if (p.M < 2 || p.M > 8) return false;
    if (p.w_dtype != JL_Q4 && p.w_dtype != JL_I8) return false;
    if (prologue != PRO_F32_QUANT && prologue != PRO_RMSNORM_QUANT) return false;
    const int bpc = p.w_dtype == JL_Q4 ? 8 : 4;
    if ((p.K % 32) || ((p.K / 32) % bpc) || (p.a_col_off % 4) || (p.lda % 4)) return false;
    if ((p.ldw % 32) || ((p.ldw / 32) % bpc) || (p.w_col_off % (32 * bpc))) return false; // 16-byte aligned cp.async sources (weights and scales)
    if (prologue == PRO_RMSNORM_QUANT && p.norm_w_dtype != JL_BF16 && p.norm_w_dtype != JL_F32) return false;
    if (epilogue == EPI_SILU_MUL && p.nseg != 2) return false;
    if (epilogue != EPI_SILU_MUL)
        for (int i = 0; i + 1 < p.nseg; i++)
            if (p.seg[i].rows % 16) return false; // a strip must not straddle two weight tensors
    return g8_stages(p, 8) >= 2;
}

template <int WDT, int EPI, int PRO, int NWARP>
static int launch_g8w(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p) {
    auto kern = gemm8_kernel<WDT, EPI, PRO, NWARP>;
    const size_t smem = g8_smem(p, NWARP);
    const int nst = g8_stages(p, NWARP);
    static size_t configured[JL_MAX_DEVICES] = {};
    JL_CUDA_CHECK(ctx, jl_ensure_dyn_smem(kern, ctx->device, smem, configured));
    const int strips = (p.total_rows + 15) / 16;
    const int ksplit = g8_ksplit(p, ctx->sm_count, NWARP), spr = NWARP / ksplit;
    int grid = ctx->sm_count; // one CTA per SM; a CTA takes NWARP / ksplit strips per round
    if (grid > (strips + spr - 1) / spr) grid = (strips + spr - 1) / spr;
    JL_CUDA_CHECK(ctx, jl_launch_kernel(kern, dim3(grid), dim3(NWARP * 32), smem, stream, p, nst, ksplit));
    ctx->launches++;
    return JL_OK;
}
template <int WDT, int EPI, int PRO>
static int launch_g8(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p) {
    return g8_warps(p) == 16 ? launch_g8w<WDT, EPI, PRO, 16>(ctx, stream, p) : launch_g8w<WDT, EPI, PRO, 8>(ctx, stream, p);
}
template <int WDT, int EPI>
static int launch_g8_p(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue) {
    return prologue == PRO_RMSNORM_QUANT ? launch_g8<WDT, EPI, PRO_RMSNORM_QUANT>(ctx, stream, p) : launch_g8<WDT, EPI, PRO_F32_QUANT>(ctx, stream, p);
}
template <int WDT>
static int launch_g8_e(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue, int epilogue) {
    switch (epilogue) {
        case EPI_STORE: return launch_g8_p<WDT, EPI_STORE>(ctx, stream, p, prologue);
        case EPI_ADD_RESIDUAL: return launch_g8_p<WDT, EPI_ADD_RESIDUAL>(ctx, stream, p, prologue);
        default: return launch_g8_p<WDT, EPI_SILU_MUL>(ctx, stream, p, prologue);
    }
}
int jl_launch_gemm8(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue, int epilogue) {
    return p.w_dtype == JL_Q4 ? launch_g8_e<JL_Q4>(ctx, stream, p, prologue, epilogue) : launch_g8_e<JL_I8>(ctx, stream, p, prologue, epilogue);
}
