// Block-quantised GEMV / small-M GEMM for decode:  out[m, n] = sum_k A[m,k] * W[n,k]
//
// Replaces, for M <= 8, the reference's batchDotProduct back-ends
//   I8 x Q4  : PanamaTensorOperations.java:768-1044 (GemmerI8Q4_512), vector_simd.c:261-437
//   F32 x Q4 : PanamaTensorOperations.java:289-548, vector_simd.c:770-964
// and the WebGPU GEMV native/res/gemm_i8q4_v5.wgsl:57-137, and fuses the scalar Java loops that
// surround them in the decode step: RMSNorm (RMSNorm.java:34-56), the Q8 activation quantiser
// (PanamaTensorOperations.java:1684-1723), the residual add (TransformerBlock.java:185,203) and
// SiLU*up (MLPBlock.java:132-141).
//
// HBM-bound by design: every weight byte is read exactly once with 128-bit coalesced
// ld.global.nc loads straight into registers (one 16-byte Q4 block per lane, 512 B per warp
// request), activations are staged once per CTA in shared memory in a bank-conflict-free
// [half][block][16B] layout, integer dot products use dp4a, the reduction is a warp shuffle.
//
// Decode shape of the kernel (M = 1, Q4 weights, Q8 activations; DESIGN.md "GEMV v3"): ONE 512-thread CTA per SM with
// a three-deep register ring (two 2.5 KB chunks per warp = 80 KB per SM in flight).
// More CTAs per SM only repeat the prologue: with three 256-thread CTAs the RMSNorm + Q8 quantisation runs three times
// per SM and its loads queue behind the weight requests.  Here the
// first warps ("stagers") request the hidden row BEFORE any weight load, every warp then puts its first chunks in
// flight, and the stagers normalise / quantise into shared memory while the weights stream.  The gate+up launch uses
// 640 threads with a two-deep ring instead (more issue slots for the long stream); finished rows are parked one per lane
// and their epilogues run together.
#include "jl_common.cuh"
#include <stdlib.h>

#include "jl_gemv_body.cuh"

// End of an output row.
template <int EPI, int MM>
__device__ __forceinline__ void finish_row_fn(const GemvParams &p, int rr, int wrr, float (&acc)[MM], float (&gate)[MM]) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int m = 0; m < MM; m++) acc[m] = warp_sum(acc[m]);
    if (EPI == EPI_SILU_MUL && wrr == 0) {
#pragma unroll
        for (int m = 0; m < MM; m++) gate[m] = acc[m], acc[m] = 0.0f;
        return;
    }
    if (lane == 0) {
        int seg = 0, local = rr;
        if (EPI != EPI_SILU_MUL) seg_lookup(p, rr, seg, local);
        const GemvSeg &sg = p.seg[seg];
        const int col = p.row0 + local + sg.out_off;
#pragma unroll
        for (int m = 0; m < MM; m++) {
            if (m < p.M) {
                float v = acc[m];
                if (EPI == EPI_ADD_RESIDUAL) v = __fadd_rn(v, p.residual[(size_t)m * p.res_ld + (p.row0 + local)]);
                if (EPI == EPI_SILU_MUL) v = __fmul_rn(silu_ref(gate[m]), v);
                sg.out[(size_t)m * sg.out_ld + col] = v;
            }
        }
    }
#pragma unroll
    for (int m = 0; m < MM; m++) acc[m] = 0.0f;
}

// ---- generic kernel: any M <= 8, any prologue (run time), 256 threads -------------------------------------------
template <int WDT, bool ACTQ8, int EPI, int MM, int CH, int NBUF, int MINB>
__global__ void __launch_bounds__(GEMV_THREADS, MINB) gemv_kernel(const GemvParams p, const int prologue) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nblk = p.K / 32;
    const int nchunks = (nblk + 32 * CH - 1) / (32 * CH);
    constexpr int NW = (EPI == EPI_SILU_MUL) ? 2 : 1; // weight rows per output row
    const int wbytes_per_blk = (WDT == JL_Q4) ? 16 : 32;
    ktrace_begin(p.trace, 0x100u | (unsigned)EPI | ((unsigned long long)prologue << 4) | ((unsigned long long)p.total_rows << 16) |
                              ((unsigned long long)p.K << 40));
    if (gemv_absent<EPI>(p)) return; // expert held by another rank

    // balanced static partition of output rows over all warps of the grid
    const long long gw = (long long)blockIdx.x * GEMV_WARPS + warp;
    const long long tw = (long long)gridDim.x * GEMV_WARPS;
    const int r0 = (int)(((long long)p.total_rows * gw) / tw);
    const int r1 = (int)(((long long)p.total_rows * (gw + 1)) / tw);

    // item iterator: (row r, weight-row wr, chunk c)
    struct It {
        int r, wr, c;
    };
    auto row_ptrs = [&](const It &it, const uint8_t *&wrow, const float *&srow) {
        int seg, local;
        if (EPI == EPI_SILU_MUL) {
            seg = it.wr;
            local = it.r;
        } else {
            seg_lookup(p, it.r, seg, local);
        }
        const void *wb;
        const float *wsb;
        gemv_seg_base(p, seg, wb, wsb);
        const size_t grow = (size_t)(p.row0 + local);
        wrow = (const uint8_t *)wb + (grow * (size_t)(p.ldw / 32) + (size_t)(p.w_col_off / 32)) * wbytes_per_blk;
        srow = wsb + grow * (size_t)(p.ldw / 32) + (size_t)(p.w_col_off / 32);
    };
    auto advance = [&](It &it) {
        if (++it.c == nchunks) {
            it.c = 0;
            if (++it.wr == NW) {
                it.wr = 0;
                ++it.r;
            }
        }
    };

    WBuf<WDT, CH> buf[NBUF];
    const uint8_t *wrow;
    const float *srow;
    const unsigned long long pol = l2_evict_first_policy();
    It cur = {r0, 0, 0}, ld = cur;
    // NBUF-1 chunks per warp go in flight before anything else: the weight stream does not depend on the previous kernel
#pragma unroll
    for (int b = 0; b < NBUF - 1; b++) {
        if (ld.r < r1) {
            row_ptrs(ld, wrow, srow);
            load_chunk<WDT, CH>(buf[b], wrow, srow, ld.c * 32 * CH, nblk, lane, pol);
            advance(ld);
        }
    }
    if (ACTQ8 && (prologue == PRO_F32_QUANT || prologue == PRO_RMSNORM_QUANT))
        stage_q8_pairs<MM>(p, prologue == PRO_RMSNORM_QUANT, smem, nblk);
    else
        stage_activations<ACTQ8, MM>(p, prologue, smem, nblk);
    ktrace_mid(p.trace);

    float acc[MM];
    float gate[MM];
#pragma unroll
    for (int m = 0; m < MM; m++) acc[m] = 0.0f, gate[m] = 0.0f;

    while (cur.r < r1) {
#pragma unroll
        for (int b = 0; b < NBUF; b++) {
            if (cur.r < r1) {
                if (ld.r < r1) {
                    row_ptrs(ld, wrow, srow);
                    load_chunk<WDT, CH>(buf[(b + NBUF - 1) % NBUF], wrow, srow, ld.c * 32 * CH, nblk, lane, pol);
                    advance(ld);
                }
                compute_chunk<WDT, ACTQ8, MM, CH>(buf[b], acc, smem, cur.c * 32 * CH, nblk, lane);
                if (cur.c == nchunks - 1) finish_row_fn<EPI, MM>(p, cur.r, cur.wr, acc, gate);
                advance(cur);
            }
        }
    }
    if (p.trace) {
        __syncthreads();
        ktrace_end(p.trace);
    }
}

// ---- decode kernel: M = 1, Q8 activations, prologue fixed at compile time, one big CTA per SM -----------------------
// The pass is gemv_phase (jl_gemv_body.cuh).  The kernel is kept small on purpose: five different kernels alternate every
// ~50 us, each starts with a cold instruction cache, and every kilobyte on the prologue path showed up in the timeline
// (tools/ktrace.py).

// gemv_phase's view of a launch: segments and MoE pointer tables, the hidden row staged (and normalised) around the ring
// priming, and the epilogue into the segment's output
template <int WDT, int EPI, int PRO, int NT, bool LONG>
struct DecodeGemv {
    static constexpr bool NORM = PRO == PRO_RMSNORM_QUANT, XLONG = LONG && !NORM;
    using Stage = StageRegs<NORM, XLONG>;
    const GemvParams &p;
    // The hidden row, in flight while the ring is primed.  A separate object: its arrays are indexed in loops that are not
    // unrolled yet when the compiler first splits up this struct, which would keep `p` in memory until then as well and
    // move every parameter load of the kernel.
    Stage &sr;
    size_t row_blocks, col_blocks; // weight row stride and column offset in 32-element blocks, set by begin()
    __device__ __forceinline__ DecodeGemv(const GemvParams &p_, Stage &sr_) : p(p_), sr(sr_) {}
    __device__ __forceinline__ int tid() const { return threadIdx.x; }
    __device__ __forceinline__ unsigned cta() const { return blockIdx.x; }
    __device__ __forceinline__ unsigned ncta() const { return gridDim.x; }
    __device__ __forceinline__ int K() const { return p.K; }
    __device__ __forceinline__ int rows() const { return p.total_rows; }
    __device__ __forceinline__ bool begin() {
        ktrace_begin(p.trace, 0x100u | (unsigned)EPI | ((unsigned long long)PRO << 4) | ((unsigned long long)p.total_rows << 16) |
                                  ((unsigned long long)p.K << 40));
        if (gemv_absent<EPI>(p)) return false; // expert held by another rank
        row_blocks = (size_t)(p.ldw / 32), col_blocks = (size_t)(p.w_col_off / 32);
        return true;
    }
    __device__ __forceinline__ void end() const {
        if (p.trace) {
            __syncthreads();
            ktrace_end(p.trace);
        }
    }
    __device__ __forceinline__ void row_ptrs(int row, int wr, int, const uint8_t *&wrow, const float *&srow) const {
        int seg, local;
        if (EPI == EPI_SILU_MUL) {
            seg = wr;
            local = row;
        } else {
            seg_lookup(p, row, seg, local);
        }
        const size_t blk = (size_t)(p.row0 + local) * row_blocks + col_blocks;
        const void *wb;
        const float *wsb;
        gemv_seg_base(p, seg, wb, wsb);
        wrow = (const uint8_t *)wb + blk * (WDT == JL_Q4 ? 16 : 32);
        srow = wsb + blk;
    }
    // the hidden row (and the norm weights) are requested before this SM's ~80 KB of weight requests
    template <class Buf>
    __device__ __forceinline__ void prime_begin(Buf &) {
        stage_q8_issue<NORM, XLONG, NT>(p, sr);
    }
    __device__ __forceinline__ void prime_end(unsigned char *smem, int nblk) {
        stage_q8_finish<NORM, XLONG, NT>(p, sr, smem, nblk);
        ktrace_mid(p.trace);
    }
    __device__ __forceinline__ void cta_bar() const { __syncthreads(); }
    __device__ __forceinline__ void store_row(int row, float v0, float v1) const {
        int seg = 0, local = row;
        if (EPI != EPI_SILU_MUL) seg_lookup(p, row, seg, local);
        const GemvSeg &sg = p.seg[seg];
        float v = EPI == EPI_SILU_MUL ? v1 : v0;
        if (EPI == EPI_ADD_RESIDUAL) v = __fadd_rn(v, p.residual[p.row0 + local]);
        if (EPI == EPI_SILU_MUL) v = __fmul_rn(silu_ref(v0), v);
        sg.out[p.row0 + local + sg.out_off] = v;
    }
};

template <int WDT, int EPI, int PRO, int CH, int NBUF, int NT, bool LONG>
__global__ void __launch_bounds__(NT, 1) gemv_decode_kernel(const GemvParams p, const int) {
    extern __shared__ __align__(16) unsigned char smem[];
    using Ph = DecodeGemv<WDT, EPI, PRO, NT, LONG>;
    typename Ph::Stage sr;
    Ph ph(p, sr);
    gemv_phase<Ph, WDT, EPI, CH, NBUF, NT, LONG>(ph, smem);
}

// ---- dense (F32 / BF16 weights) GEMV: GemmerF32 / GemmerF32BF16 (PanamaTensorOperations.java:1046-1231,1466-1539)
template <int WDT, int EPI, int MM>
__global__ void __launch_bounds__(GEMV_THREADS) gemv_dense_kernel(const GemvParams p, const int prologue) {
    extern __shared__ __align__(16) unsigned char smem[];
    float *af = (float *)smem; // [MM][K]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ double red[GEMV_WARPS];
    __shared__ float rs_sh;
    const int K = p.K;
    for (int m = 0; m < MM; m++) {
        const bool live = m < p.M;
        float rsf = 1.0f;
        const bool norm = (prologue == PRO_RMSNORM_F32);
        const float *x = (const float *)p.a + (size_t)m * p.lda + p.a_col_off;
        if (norm && live) {
            double ss = 0.0;
            for (int i = tid; i < K; i += GEMV_THREADS) {
                float v = x[i];
                ss += (double)__fmul_rn(v, v);
            }
            ss = warp_sum_d(ss);
            if (lane == 0) red[warp] = ss;
            __syncthreads();
            if (tid == 0) {
                double t = 0;
                for (int w = 0; w < GEMV_WARPS; w++) t += red[w];
                t /= (double)p.norm_E;
                t += (double)p.norm_eps;
                rs_sh = (float)(1.0 / sqrt(t));
            }
            __syncthreads();
            rsf = rs_sh;
        }
        for (int i = tid; i < K; i += GEMV_THREADS) {
            float v = 0.0f;
            if (live) {
                if (prologue == PRO_BF16_GLOBAL)
                    v = bf16_bits_to_f32(((const uint16_t *)p.a)[(size_t)m * p.lda + p.a_col_off + i]);
                else
                    v = x[i];
                if (norm) {
                    float w = p.norm_w_dtype == JL_BF16 ? bf16_bits_to_f32(((const uint16_t *)p.norm_w)[i])
                                                        : ((const float *)p.norm_w)[i];
                    v = __fmul_rn(__fadd_rn(p.norm_adj, w), __fmul_rn(rsf, v));
                }
            }
            af[(size_t)m * K + i] = v;
        }
    }
    __syncthreads();
    const long long gw = (long long)blockIdx.x * GEMV_WARPS + warp;
    const long long tw = (long long)gridDim.x * GEMV_WARPS;
    const int r0 = (int)(((long long)p.total_rows * gw) / tw);
    const int r1 = (int)(((long long)p.total_rows * (gw + 1)) / tw);
    for (int r = r0; r < r1; r++) {
        int seg, local;
        seg_lookup(p, r, seg, local);
        const GemvSeg &sg = p.seg[seg];
        const size_t grow = (size_t)(p.row0 + local);
        float acc[MM];
#pragma unroll
        for (int m = 0; m < MM; m++) acc[m] = 0.0f;
        if (WDT == JL_F32) {
            const float *wrow = (const float *)sg.w + grow * (size_t)p.ldw + p.w_col_off;
            for (int i = lane; i < K; i += 32) {
                float w = ldg_nc_f32(wrow + i);
#pragma unroll
                for (int m = 0; m < MM; m++) acc[m] = fmaf(af[(size_t)m * K + i], w, acc[m]);
            }
        } else {
            const uint16_t *wrow = (const uint16_t *)sg.w + grow * (size_t)p.ldw + p.w_col_off;
            for (int i = lane; i < K; i += 32) {
                float w = bf16_bits_to_f32(wrow[i]);
#pragma unroll
                for (int m = 0; m < MM; m++) acc[m] = fmaf(af[(size_t)m * K + i], w, acc[m]);
            }
        }
#pragma unroll
        for (int m = 0; m < MM; m++) acc[m] = warp_sum(acc[m]);
        if (lane == 0) {
            const int col = p.row0 + local + sg.out_off;
#pragma unroll
            for (int m = 0; m < MM; m++)
                if (m < p.M) {
                    float v = acc[m];
                    if (EPI == EPI_ADD_RESIDUAL) v = __fadd_rn(v, p.residual[(size_t)m * p.res_ld + (p.row0 + local)]);
                    sg.out[(size_t)m * sg.out_ld + col] = v;
                }
        }
    }
}

// ---- host launcher ---------------------------------------------------------------------------------
template <typename KERN>
static int launch_kern(jl_ctx *ctx, cudaStream_t stream, KERN kern, const GemvParams &p, int prologue, int grid, int threads,
                       size_t smem, size_t (&configured)[JL_MAX_DEVICES]) {
    JL_CUDA_CHECK(ctx, jl_ensure_dyn_smem(kern, ctx->device, smem, configured));
    JL_CUDA_CHECK(ctx, jl_launch_kernel(kern, dim3(grid), dim3(threads), smem, stream, p, prologue));
    ctx->launches++;
    return JL_OK;
}

// grid for the generic 256-thread kernels: a multiple of the SM count; every warp gets >= 1 row when possible
static int generic_grid(jl_ctx *ctx, int rows, int max_per_sm) {
    int per_sm = rows >= ctx->sm_count * GEMV_WARPS * 4 ? 3 : (rows >= ctx->sm_count * GEMV_WARPS * 2 ? 2 : 1);
    if (per_sm > max_per_sm) per_sm = max_per_sm;
    int grid = ctx->sm_count * per_sm;
    const int max_grid = (rows + GEMV_WARPS - 1) / GEMV_WARPS;
    if (grid > max_grid) grid = max_grid;
    return grid < 1 ? 1 : grid;
}

// decode hot path: one big CTA per SM, prologue fixed at compile time
template <int WDT, int EPI, int PRO, int NT, int NBUF, int CH, bool LONG>
static int launch_decode_k(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int grid, size_t smem) {
    static size_t configured[JL_MAX_DEVICES] = {};
    return launch_kern(ctx, stream, gemv_decode_kernel<WDT, EPI, PRO, CH, NBUF, NT, LONG>, p, 0, grid, NT, smem, configured);
}

template <int WDT, int EPI, int PRO, int NT, int NBUF, int CH>
static int launch_decode(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p) {
    if (PRO == PRO_RMSNORM_QUANT && p.K > 16 * NT)
        return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "gemv: RMSNorm prologue supports rows up to %d", 16 * NT);
    int grid = ctx->sm_count;
    const int max_grid = (p.total_rows + NT / 32 - 1) / (NT / 32);
    if (grid > max_grid) grid = max_grid;
    const int nchunks = (p.K / 32 + 32 * CH - 1) / (32 * CH);
    const bool lng = nchunks > 1;
    size_t smem_d = gemv_parts_offset(p.K / 32);
    if (lng) {
        const int rows_per_cta = (p.total_rows + grid - 1) / grid;
        const int maxsplit = nchunks < NT / 32 ? nchunks : NT / 32;
        smem_d += (size_t)rows_per_cta * (EPI == EPI_SILU_MUL ? 2 : 1) * maxsplit * 4;
    }
    if (smem_d > 200 * 1024) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "gemv: shape exceeds shared memory");
    if (lng) return launch_decode_k<WDT, EPI, PRO, NT, NBUF, CH, true>(ctx, stream, p, grid, smem_d);
    return launch_decode_k<WDT, EPI, PRO, NT, NBUF, CH, false>(ctx, stream, p, grid, smem_d);
}

template <int WDT, bool ACTQ8, int EPI, int MM>
static int launch_q(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue, size_t smem) {
    if constexpr (WDT == JL_Q4 && ACTQ8 && MM == 1) {
        // CTA shape per launch kind, from A/B timelines on the 8B step (tools/ktrace.py; us per launch QKV / o / gate+up / down):
        //   512 threads x 3-deep ring 5.92 / 4.43 / 16.58 / 10.41      640 x 2: 6.28 / 4.53 / 15.38 / 10.53
        //   704 x 2: 5.98 / 4.62 / 15.93 / 11.10    768 x 2: 6.17 / 4.77 / 16.07 / 11.12    384 x 4: 6.32 / 4.75 / 17.01 / 11.42
        // The long gate+up stream wants warps (issue slots), the short launches want the deeper ring.
        constexpr int NT = EPI == EPI_SILU_MUL ? 640 : 512, NB = EPI == EPI_SILU_MUL ? 2 : 3;
        if (prologue == PRO_F32_QUANT) return launch_decode<WDT, EPI, PRO_F32_QUANT, NT, NB, 4>(ctx, stream, p);
        if (prologue == PRO_RMSNORM_QUANT && p.K <= 16 * NT)
            return launch_decode<WDT, EPI, PRO_RMSNORM_QUANT, NT, NB, 4>(ctx, stream, p);
    }
    constexpr int MINB = (MM <= 2) ? 2 : 1;
    static size_t cfg[JL_MAX_DEVICES] = {};
    return launch_kern(ctx, stream, gemv_kernel<WDT, ACTQ8, EPI, MM, 4, 2, MINB>, p, prologue, generic_grid(ctx, p.total_rows, MINB),
                       GEMV_THREADS, smem, cfg);
}

template <int WDT, bool ACTQ8, int EPI>
static int launch_m(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue, size_t smem1) {
    if (p.M <= 1) return launch_q<WDT, ACTQ8, EPI, 1>(ctx, stream, p, prologue, smem1);
    if (p.M <= 2) return launch_q<WDT, ACTQ8, EPI, 2>(ctx, stream, p, prologue, smem1 * 2);
    if (p.M <= 4) return launch_q<WDT, ACTQ8, EPI, 4>(ctx, stream, p, prologue, smem1 * 4);
    return launch_q<WDT, ACTQ8, EPI, 8>(ctx, stream, p, prologue, smem1 * 8);
}

template <int WDT, bool ACTQ8>
static int launch_e(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue, int epi, size_t smem1) {
    switch (epi) {
        case EPI_STORE: return launch_m<WDT, ACTQ8, EPI_STORE>(ctx, stream, p, prologue, smem1);
        case EPI_ADD_RESIDUAL: return launch_m<WDT, ACTQ8, EPI_ADD_RESIDUAL>(ctx, stream, p, prologue, smem1);
        case EPI_SILU_MUL: return launch_m<WDT, ACTQ8, EPI_SILU_MUL>(ctx, stream, p, prologue, smem1);
    }
    return jl_set_error(ctx, JL_ERR_INVALID, "bad epilogue %d", epi);
}

template <int WDT, int EPI, int MM>
static int launch_dense(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue, int grid) {
    auto kern = gemv_dense_kernel<WDT, EPI, MM>;
    size_t smem = (size_t)MM * p.K * 4;
    if (smem > 200 * 1024) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "dense gemv: M*K too large for shared memory");
    static size_t cfg[JL_MAX_DEVICES] = {};
    JL_CUDA_CHECK(ctx, jl_ensure_dyn_smem(kern, ctx->device, smem, cfg));
    JL_CUDA_CHECK(ctx, jl_launch_kernel(kern, dim3(grid), dim3(GEMV_THREADS), smem, stream, p, prologue));
    ctx->launches++;
    return JL_OK;
}

template <int WDT, int EPI>
static int launch_dense_m(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p, int prologue, int grid) {
    if (p.M <= 1) return launch_dense<WDT, EPI, 1>(ctx, stream, p, prologue, grid);
    if (p.M <= 2) return launch_dense<WDT, EPI, 2>(ctx, stream, p, prologue, grid);
    if (p.M <= 4) return launch_dense<WDT, EPI, 4>(ctx, stream, p, prologue, grid);
    return launch_dense<WDT, EPI, 8>(ctx, stream, p, prologue, grid);
}

// Largest activation-row chunk (1, 2, 4 or 8) whose staged activations fit the kernels' shared-memory budget; 0 = even one
// row does not fit.  Callers split M into chunks of this size (the reference's F32 x Q4 GEMM has no such limit,
// PanamaTensorOperations.java:289-548).
int jl_gemv_max_m(int w_dtype, int prologue, int K) {
    const bool quant_w = (w_dtype == JL_Q4 || w_dtype == JL_I8);
    const bool actq8 = quant_w && (prologue == PRO_Q8_GLOBAL || prologue == PRO_F32_QUANT || prologue == PRO_RMSNORM_QUANT);
    const size_t smem1 = actq8 ? (size_t)(K / 32) * 40 : (size_t)K * 4;
    for (int mm = GEMV_MAX_M; mm >= 1; mm >>= 1)
        if (smem1 * mm <= 200 * 1024) return mm;
    return 0;
}

int jl_launch_gemv(jl_ctx *ctx, cudaStream_t stream, const GemvParams &p_in, int prologue, int epilogue) {
    GemvParams p = p_in;
    p.trace = jl_ktrace_slot(ctx);
    p.norm_inv_E = p.norm_E > 0 ? 1.0 / (double)p.norm_E : 0.0;

    if (p.K <= 0 || p.total_rows <= 0) return jl_set_error(ctx, JL_ERR_INVALID, "gemv: empty problem");
    if (p.M > GEMV_MAX_M && jl_gemm64_supported(p, prologue, epilogue)) return jl_launch_gemm64(ctx, stream, p, prologue, epilogue);
    if (p.M < 1 || p.M > GEMV_MAX_M) return jl_set_error(ctx, JL_ERR_INVALID, "gemv: M=%d out of range", p.M);
    const bool quant_w = (p.w_dtype == JL_Q4 || p.w_dtype == JL_I8);
    if (!p.sel && jl_gemm8_supported(p, prologue, epilogue)) return jl_launch_gemm8(ctx, stream, p, prologue, epilogue);
    const int rows = p.total_rows;
    const int grid = generic_grid(ctx, rows, 3);

    if (!quant_w) {
        if (prologue != PRO_F32 && prologue != PRO_RMSNORM_F32 && prologue != PRO_BF16_GLOBAL)
            return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "dense weights need f32/bf16 activations");
        if (epilogue == EPI_SILU_MUL) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "dense silu epilogue");
        if (p.w_dtype == JL_F32)
            return epilogue == EPI_STORE ? launch_dense_m<JL_F32, EPI_STORE>(ctx, stream, p, prologue, grid)
                                         : launch_dense_m<JL_F32, EPI_ADD_RESIDUAL>(ctx, stream, p, prologue, grid);
        return epilogue == EPI_STORE ? launch_dense_m<JL_BF16, EPI_STORE>(ctx, stream, p, prologue, grid)
                                     : launch_dense_m<JL_BF16, EPI_ADD_RESIDUAL>(ctx, stream, p, prologue, grid);
    }
    if ((p.K % 32) || (p.w_col_off % 32) || (p.ldw % 32))
        return jl_set_error(ctx, JL_ERR_INVALID, "quantised gemv needs K, offsets and ld multiples of 32");
    const bool actq8 = (prologue == PRO_Q8_GLOBAL || prologue == PRO_F32_QUANT || prologue == PRO_RMSNORM_QUANT);
    const int nblk = p.K / 32;
    const size_t smem1 = actq8 ? (size_t)nblk * 40 : (size_t)p.K * 4;
    const int mm = p.M <= 1 ? 1 : (p.M <= 2 ? 2 : (p.M <= 4 ? 4 : 8));
    if (smem1 * mm > 200 * 1024)
        return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "gemv: activations (M=%d,K=%d) exceed shared memory", p.M, p.K);
    if (p.w_dtype == JL_Q4)
        return actq8 ? launch_e<JL_Q4, true>(ctx, stream, p, prologue, epilogue, smem1)
                     : launch_e<JL_Q4, false>(ctx, stream, p, prologue, epilogue, smem1);
    return actq8 ? launch_e<JL_I8, true>(ctx, stream, p, prologue, epilogue, smem1)
                 : launch_e<JL_I8, false>(ctx, stream, p, prologue, epilogue, smem1);
}
