// Device code shared by the quantised GEMV kernels (jl_gemv.cu) and the persistent decode kernel (jl_pdecode.cu):
// register chunk buffers, weight loads, activation staging (RMSNorm / Q8 quantiser), the per-chunk dot products and the
// M = 1 decode pass built from them (gemv_phase).
// Everything here is header-only device code; see jl_gemv.cu for the design notes and the reference citations.
#pragma once
#include "jl_common.cuh"

#define GEMV_THREADS 256 // generic kernels
#define GEMV_WARPS 8
// CH = 32-element blocks per lane per chunk (a chunk is CH*32 blocks = CH*1024 weights of one row), NBUF = register
// chunk buffers per warp (NBUF-1 chunks are in flight while one is being consumed)

template <int WDT, int CH>
struct WBuf {
    uint4 q[CH * (WDT == JL_I8 ? 2 : 1)];
    float s[CH];
};

// Which weight row does item-row `row` (index within the launch) map to?
__device__ __forceinline__ void seg_lookup(const GemvParams &p, int row, int &seg, int &local) {
    seg = 0;
    local = row;
#pragma unroll
    for (int i = 0; i < 2; i++) {
        if (seg == i && i + 1 < p.nseg && local >= p.seg[i].rows) {
            local -= p.seg[i].rows;
            seg = i + 1;
        }
    }
}

// Expert-parallel mixture of experts: the expert this launch was routed to lives on another rank (null entry in the pointer
// table).  The launch then contributes nothing: outputs are zero (store, SiLU*up) or the running sum passed through (add).
template <int EPI>
__device__ __forceinline__ bool gemv_absent(const GemvParams &p) {
    if (!p.sel) return false;
    if (p.w_tab[0][__ldg(p.sel)] != nullptr) return false;
    const long long total = (long long)p.M * p.total_rows;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int m = (int)(i / p.total_rows), rr = (int)(i - (long long)m * p.total_rows);
        int seg = 0, local = rr;
        if (EPI != EPI_SILU_MUL) seg_lookup(p, rr, seg, local);
        const GemvSeg &sg = p.seg[seg];
        float v = 0.0f;
        if (EPI == EPI_ADD_RESIDUAL) v = p.residual[(size_t)m * p.res_ld + (p.row0 + local)];
        sg.out[(size_t)m * sg.out_ld + p.row0 + local + sg.out_off] = v;
    }
    return true;
}

template <int WDT, int CH>
__device__ __forceinline__ void load_chunk(WBuf<WDT, CH> &b, const uint8_t *wrow, const float *srow, int blk0, int nblk,
                                           int lane, unsigned long long pol) {
#pragma unroll
    for (int j = 0; j < CH; j++) {
        int bi = blk0 + j * 32 + lane;
        if (bi < nblk) {
            if (WDT == JL_Q4) {
                b.q[j] = ldg_stream_u4(wrow + (size_t)bi * 16, pol);
            } else {
                b.q[2 * j] = ldg_stream_u4(wrow + (size_t)bi * 32, pol);
                b.q[2 * j + 1] = ldg_stream_u4(wrow + (size_t)bi * 32 + 16, pol);
            }
            b.s[j] = ldg_stream_f32(srow + bi, pol);
        }
    }
}

// ---- activation staging -------------------------------------------------------------------------
// Q8 layout in smem:  q[m][half][blk][16] int8, then sc[m][blk] f32, then sum[m][blk] int32
// F32 layout in smem: f[m][c4(8)][blk][4] floats
// gemv_phase (M = 1) keeps the partial sums of its LONG rows behind the Q8 row, from this 16-byte aligned offset
__host__ __device__ __forceinline__ size_t gemv_parts_offset(int nblk) { return ((size_t)nblk * 40 + 15) & ~(size_t)15; }

// One thread owns one 32-element block: 8 independent 128-bit loads, the block max, the Q8 rounding
// and the packing all stay in registers (no shuffles), so the prologue costs about one L2 round trip.
template <bool ACTQ8, int MM>
__device__ void stage_activations(const GemvParams &p, int prologue, unsigned char *smem, int nblk) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ double red[MM][GEMV_WARPS];
    __shared__ float rs_sh[MM];
    int8_t *aq = (int8_t *)smem;
    float *asc = (float *)(smem + (size_t)MM * nblk * 32);
    int *asum = (int *)(smem + (size_t)MM * nblk * 32 + (size_t)MM * nblk * 4);
    float4 *af4 = (float4 *)smem;
    const int K = p.K;
    const bool norm = (prologue == PRO_RMSNORM_QUANT || prologue == PRO_RMSNORM_F32);

    if (norm) {
        // RMSNorm.java:41-52: float products summed in double over [0, E), all rows in one pass
        double ss[MM];
#pragma unroll
        for (int m = 0; m < MM; m++) ss[m] = 0.0;
        for (int i4 = tid; i4 < K / 4; i4 += GEMV_THREADS) {
            float4 v[MM];
#pragma unroll
            for (int m = 0; m < MM; m++)
                v[m] = m < p.M ? *(const float4 *)((const float *)p.a + (size_t)m * p.lda + p.a_col_off + i4 * 4)
                               : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int m = 0; m < MM; m++) {
                ss[m] += (double)__fmul_rn(v[m].x, v[m].x);
                ss[m] += (double)__fmul_rn(v[m].y, v[m].y);
                ss[m] += (double)__fmul_rn(v[m].z, v[m].z);
                ss[m] += (double)__fmul_rn(v[m].w, v[m].w);
            }
        }
#pragma unroll
        for (int m = 0; m < MM; m++) {
            ss[m] = warp_sum_d(ss[m]);
            if (lane == 0) red[m][warp] = ss[m];
        }
        __syncthreads();
        if (tid < MM) {
            double t = 0;
            for (int w = 0; w < GEMV_WARPS; w++) t += red[tid][w];
            t /= (double)p.norm_E;
            t += (double)p.norm_eps;
            rs_sh[tid] = (float)(1.0 / sqrt(t));
        }
        __syncthreads();
    }

    for (int idx = tid; idx < MM * nblk; idx += GEMV_THREADS) {
        const int m = idx / nblk, b = idx - m * nblk;
        const bool live = m < p.M;
        if (prologue == PRO_Q8_GLOBAL) {
            uint4 lo = make_uint4(0, 0, 0, 0), hi = lo;
            float sc = 0.0f;
            if (live) {
                const int8_t *src = (const int8_t *)p.a + (size_t)m * p.lda + p.a_col_off + b * 32;
                lo = *(const uint4 *)src;
                hi = *(const uint4 *)(src + 16);
                sc = p.a_scales[(size_t)m * (p.lda / 32) + p.a_col_off / 32 + b];
            }
            int sum = 0;
            sum = __dp4a((int)lo.x, 0x01010101, sum);
            sum = __dp4a((int)lo.y, 0x01010101, sum);
            sum = __dp4a((int)lo.z, 0x01010101, sum);
            sum = __dp4a((int)lo.w, 0x01010101, sum);
            sum = __dp4a((int)hi.x, 0x01010101, sum);
            sum = __dp4a((int)hi.y, 0x01010101, sum);
            sum = __dp4a((int)hi.z, 0x01010101, sum);
            sum = __dp4a((int)hi.w, 0x01010101, sum);
            *(uint4 *)(aq + (((size_t)m * 2 + 0) * nblk + b) * 16) = lo;
            *(uint4 *)(aq + (((size_t)m * 2 + 1) * nblk + b) * 16) = hi;
            asc[m * nblk + b] = sc;
            asum[m * nblk + b] = sum;
            continue;
        }
        float v[32];
        if (!live) {
#pragma unroll
            for (int i = 0; i < 32; i++) v[i] = 0.0f;
        } else if (prologue == PRO_BF16_GLOBAL) {
            const uint4 *src = (const uint4 *)((const uint16_t *)p.a + (size_t)m * p.lda + p.a_col_off + b * 32);
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const uint4 u = src[i];
                const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
                for (int t = 0; t < 4; t++) {
                    v[i * 8 + t * 2] = __uint_as_float(w[t] << 16);
                    v[i * 8 + t * 2 + 1] = __uint_as_float(w[t] & 0xffff0000u);
                }
            }
        } else {
            const float4 *src = (const float4 *)((const float *)p.a + (size_t)m * p.lda + p.a_col_off + b * 32);
            float4 x4[8];
#pragma unroll
            for (int i = 0; i < 8; i++) x4[i] = src[i];
#pragma unroll
            for (int i = 0; i < 8; i++) v[i * 4] = x4[i].x, v[i * 4 + 1] = x4[i].y, v[i * 4 + 2] = x4[i].z, v[i * 4 + 3] = x4[i].w;
            if (norm) {
                const float rsf = rs_sh[m];
                if (p.norm_w_dtype == JL_BF16) {
                    const uint16_t *wp = (const uint16_t *)p.norm_w + b * 32;
#pragma unroll
                    for (int i = 0; i < 32; i++)
                        v[i] = __fmul_rn(__fadd_rn(p.norm_adj, bf16_bits_to_f32(wp[i])), __fmul_rn(rsf, v[i]));
                } else {
                    const float4 *wp = (const float4 *)((const float *)p.norm_w + b * 32);
#pragma unroll
                    for (int i = 0; i < 8; i++) {
                        const float4 w4 = wp[i];
                        v[i * 4] = __fmul_rn(__fadd_rn(p.norm_adj, w4.x), __fmul_rn(rsf, v[i * 4]));
                        v[i * 4 + 1] = __fmul_rn(__fadd_rn(p.norm_adj, w4.y), __fmul_rn(rsf, v[i * 4 + 1]));
                        v[i * 4 + 2] = __fmul_rn(__fadd_rn(p.norm_adj, w4.z), __fmul_rn(rsf, v[i * 4 + 2]));
                        v[i * 4 + 3] = __fmul_rn(__fadd_rn(p.norm_adj, w4.w), __fmul_rn(rsf, v[i * 4 + 3]));
                    }
                }
            }
        }
        if (ACTQ8) {
            // PanamaTensorOperations.java:1696-1710: d = max/127, q = (byte)(x*(127/max) + 0.5f), F2B truncates
            float mx = 0.0f;
#pragma unroll
            for (int i = 0; i < 32; i++) mx = fmaxf(mx, fabsf(v[i]));
            const float d = __fdiv_rn(mx, 127.0f);
            const float id = mx != 0.0f ? __fdiv_rn(127.0f, mx) : 0.0f;
            uint32_t w[8];
            int sum = 0;
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const int q0 = (int)__fadd_rn(__fmul_rn(v[i * 4], id), 0.5f);
                const int q1 = (int)__fadd_rn(__fmul_rn(v[i * 4 + 1], id), 0.5f);
                const int q2 = (int)__fadd_rn(__fmul_rn(v[i * 4 + 2], id), 0.5f);
                const int q3 = (int)__fadd_rn(__fmul_rn(v[i * 4 + 3], id), 0.5f);
                sum += q0 + q1 + q2 + q3;
                w[i] = (uint32_t)(q0 & 0xFF) | ((uint32_t)(q1 & 0xFF) << 8) | ((uint32_t)(q2 & 0xFF) << 16) |
                       ((uint32_t)(q3 & 0xFF) << 24);
            }
            *(uint4 *)(aq + (((size_t)m * 2 + 0) * nblk + b) * 16) = make_uint4(w[0], w[1], w[2], w[3]);
            *(uint4 *)(aq + (((size_t)m * 2 + 1) * nblk + b) * 16) = make_uint4(w[4], w[5], w[6], w[7]);
            asc[m * nblk + b] = d;
            asum[m * nblk + b] = sum;
        } else {
#pragma unroll
            for (int c4 = 0; c4 < 8; c4++)
                af4[((size_t)m * 8 + c4) * nblk + b] = make_float4(v[c4 * 4], v[c4 * 4 + 1], v[c4 * 4 + 2], v[c4 * 4 + 3]);
        }
    }
    __syncthreads();
}


// ---- fast F32 -> (RMSNorm) -> Q8 staging ------------------------------------------------------------------------
// Thread pair (t, t^1) owns one 32-element Q8 block: thread t holds the 16 contiguous floats that become one 16-byte
// half of the smem layout, so a 4096-element tile is quantised by all 256 threads at once with a single shuffle for the
// block max and one for the block sum.  For the decode case (one row, K <= 4096) the hidden row and the norm weights
// are requested together and stay in registers: the whole prologue costs one L2 round trip instead of three.
__device__ __forceinline__ void quant_half_block(const float (&v)[16], int8_t *aq, float *asc, int *asum, int m, int nblk,
                                                 int blk, int half, bool in) {
    // PanamaTensorOperations.java:1696-1710: d = max/127, q = (byte)(x*(127/max) + 0.5f), F2B truncates
    float mx = 0.0f;
#pragma unroll
    for (int i = 0; i < 16; i++) mx = fmaxf(mx, fabsf(v[i]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    const float d = __fdiv_rn(mx, 127.0f);
    const float id = mx != 0.0f ? __fdiv_rn(127.0f, mx) : 0.0f;
    uint32_t w[4];
    int sum = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int q0 = (int)__fadd_rn(__fmul_rn(v[i * 4], id), 0.5f);
        const int q1 = (int)__fadd_rn(__fmul_rn(v[i * 4 + 1], id), 0.5f);
        const int q2 = (int)__fadd_rn(__fmul_rn(v[i * 4 + 2], id), 0.5f);
        const int q3 = (int)__fadd_rn(__fmul_rn(v[i * 4 + 3], id), 0.5f);
        sum += q0 + q1 + q2 + q3;
        w[i] = (uint32_t)(q0 & 0xFF) | ((uint32_t)(q1 & 0xFF) << 8) | ((uint32_t)(q2 & 0xFF) << 16) | ((uint32_t)(q3 & 0xFF) << 24);
    }
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    if (in) {
        *(uint4 *)(aq + (((size_t)m * 2 + half) * nblk + blk) * 16) = make_uint4(w[0], w[1], w[2], w[3]);
        if (half == 0) {
            asc[m * nblk + blk] = d;
            asum[m * nblk + blk] = sum;
        }
    }
}

__device__ __forceinline__ void load16(float (&v)[16], const float *src, bool in) {
#pragma unroll
    for (int i = 0; i < 4; i++) {
        // through L2 (ld.global.cg): inside the persistent decode kernel the row was written by other CTAs of the same grid
        const float4 t = in ? __ldcg((const float4 *)(src + i * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
        v[i * 4] = t.x, v[i * 4 + 1] = t.y, v[i * 4 + 2] = t.z, v[i * 4 + 3] = t.w;
    }
}
__device__ __forceinline__ void load16_normw(float (&v)[16], const GemvParams &p, int e0, bool in) {
    const unsigned long long pol = l2_evict_last_policy();
    if (p.norm_w_dtype == JL_BF16) {
        const uint4 *src = (const uint4 *)((const uint16_t *)p.norm_w + e0);
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const uint4 u = in ? ldg_keep_u4(src + i, pol) : make_uint4(0, 0, 0, 0);
            const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
            for (int t = 0; t < 4; t++) {
                v[i * 8 + t * 2] = __uint_as_float(w[t] << 16);
                v[i * 8 + t * 2 + 1] = __uint_as_float(w[t] & 0xffff0000u);
            }
        }
    } else {
        const uint4 *src = (const uint4 *)((const float *)p.norm_w + e0);
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const uint4 u = in ? ldg_keep_u4(src + i, pol) : make_uint4(0, 0, 0, 0);
            v[i * 4] = __uint_as_float(u.x), v[i * 4 + 1] = __uint_as_float(u.y);
            v[i * 4 + 2] = __uint_as_float(u.z), v[i * 4 + 3] = __uint_as_float(u.w);
        }
    }
}

// RMSNorm.java:41-52 scale factor from the double sum of float squares.  inv_E = 1.0 / E (exact for the power-of-two
// embedding lengths of every Llama-family model; otherwise within 1 ulp(double) of the division, far below float
// resolution).  rsqrt() is within 1 ulp(double) of 1.0 / sqrt(t); after the cast to float the two agree.
__device__ __forceinline__ float rms_scale(double sumsq, double inv_E, float eps) {
    double t = sumsq * inv_E;
    t += (double)eps;
    return (float)rsqrt(t);
}

// Stagers = the first ceil(K/16/32) warps (at most all of them).  The registers were loaded by stage_q8_issue() before
// the weight loads were queued.  NT = threads per CTA.  LONG (K > 16*NT, no norm): a second register tile and a tail loop.
template <bool NORM, bool LONG>
struct StageRegs {
    float x0[16], x1[LONG ? 16 : 1], w[NORM ? 16 : 1];
};

template <bool NORM, bool LONG, int NT>
__device__ __forceinline__ void stage_q8_issue(const GemvParams &p, StageRegs<NORM, LONG> &r) {
    const int tid = threadIdx.x;
    const float *x0 = (const float *)p.a + p.a_col_off;
    const int e0 = tid * 16;
    load16(r.x0, x0 + e0, e0 < p.K);
    if constexpr (NORM) load16_normw(r.w, p, e0, e0 < p.K);
    if constexpr (LONG) load16(r.x1, x0 + (NT + tid) * 16, (NT + tid) * 16 < p.K);
}

// FULLBAR: 0 = the closing barrier is __syncthreads(); otherwise bar.sync FULLBAR over NT threads (a CTA that carries extra
// non-consumer warps, e.g. the TMA producer warp of the persistent decode kernel)
template <bool NORM, bool LONG, int NT, int FULLBAR = 0>
__device__ __forceinline__ void stage_q8_finish(const GemvParams &p, StageRegs<NORM, LONG> &r, unsigned char *smem, const int nblk) {
    constexpr int NWARP = NT / 32;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ double red[NORM ? NWARP : 1];
    int8_t *aq = (int8_t *)smem;
    float *asc = (float *)(smem + (size_t)nblk * 32);
    int *asum = (int *)(smem + (size_t)nblk * 32 + (size_t)nblk * 4);
    const int K = p.K;
    const int half = tid & 1;
    const int e0 = tid * 16;
    // warps that hold part of the row (whole warps, so the pair shuffles and the named barrier see full warps)
    const int nsw = min(NWARP, (K / 16 + 31) / 32);
    if (warp < nsw) {
        if constexpr (NORM) {
            double ss = 0.0;
#pragma unroll
            for (int i = 0; i < 16; i++) ss += (double)__fmul_rn(r.x0[i], r.x0[i]); // float products, double sum
            ss = warp_sum_d(ss);
            if (lane == 0) red[warp] = ss;
            asm volatile("bar.sync 2, %0;" ::"r"(nsw * 32) : "memory");
            double t = 0.0;
            for (int i = 0; i < nsw; i++) t += red[i];
            const float rsf = rms_scale(t, p.norm_inv_E, p.norm_eps);
#pragma unroll
            for (int i = 0; i < 16; i++) r.x0[i] = __fmul_rn(__fadd_rn(p.norm_adj, r.w[i]), __fmul_rn(rsf, r.x0[i])); // RMSNorm.java:50-52
        }
        quant_half_block(r.x0, aq, asc, asum, 0, nblk, e0 >> 5, half, e0 < K);
    }
    if constexpr (LONG) {
        // second register tile, then the rest of the row tile by tile (uniform trip count: all warps)
        const int e1 = (NT + tid) * 16;
        quant_half_block(r.x1, aq, asc, asum, 0, nblk, e1 >> 5, half, e1 < K);
        const float *x0 = (const float *)p.a + p.a_col_off;
        for (int e = (2 * NT + tid) * 16; e - tid * 16 < K; e += NT * 16) {
            load16(r.x1, x0 + e, e < K);
            quant_half_block(r.x1, aq, asc, asum, 0, nblk, e >> 5, half, e < K);
        }
    }
    if (FULLBAR == 0) __syncthreads();
    else asm volatile("bar.sync %0, %1;" ::"n"(FULLBAR), "n"(NT) : "memory");
}

template <int MM>
__device__ void stage_q8_pairs(const GemvParams &p, const bool norm, unsigned char *smem, const int nblk) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ double red[MM][GEMV_WARPS];
    int8_t *aq = (int8_t *)smem;
    float *asc = (float *)(smem + (size_t)MM * nblk * 32);
    int *asum = (int *)(smem + (size_t)MM * nblk * 32 + (size_t)MM * nblk * 4);
    const int K = p.K;
    const int half = tid & 1;
    const float *x0 = (const float *)p.a + p.a_col_off;

    float rsf[MM];
#pragma unroll
    for (int m = 0; m < MM; m++) rsf[m] = 1.0f;
    if (norm) {
        double ss[MM];
#pragma unroll
        for (int m = 0; m < MM; m++) ss[m] = 0.0;
        for (int e0 = tid * 16; e0 < K; e0 += 16 * GEMV_THREADS) {
#pragma unroll
            for (int m = 0; m < MM; m++) {
                float x[16];
                load16(x, x0 + (size_t)m * p.lda + e0, m < p.M);
#pragma unroll
                for (int i = 0; i < 16; i++) ss[m] += (double)__fmul_rn(x[i], x[i]);
            }
        }
#pragma unroll
        for (int m = 0; m < MM; m++) {
            ss[m] = warp_sum_d(ss[m]);
            if (lane == 0) red[m][warp] = ss[m];
        }
        __syncthreads();
#pragma unroll
        for (int m = 0; m < MM; m++) {
            double t = 0.0;
#pragma unroll
            for (int i = 0; i < GEMV_WARPS; i++) t += red[m][i];
            t /= (double)p.norm_E;
            t += (double)p.norm_eps;
            rsf[m] = (float)(1.0 / sqrt(t));
        }
    }
    // tiles of 16*GEMV_THREADS elements; the trip count is uniform so the pair shuffles see full warps
    const int ntiles = (K + 16 * GEMV_THREADS - 1) / (16 * GEMV_THREADS);
    for (int j = 0; j < ntiles; j++) {
        const int e0 = j * 16 * GEMV_THREADS + tid * 16;
        const bool in = e0 < K;
        float w[16];
        if (norm) load16_normw(w, p, e0, in);
#pragma unroll
        for (int m = 0; m < MM; m++) {
            float x[16];
            load16(x, x0 + (size_t)m * p.lda + e0, in && m < p.M);
            if (norm) {
#pragma unroll
                for (int i = 0; i < 16; i++) x[i] = __fmul_rn(__fadd_rn(p.norm_adj, w[i]), __fmul_rn(rsf[m], x[i]));
            }
            quant_half_block(x, aq, asc, asum, m, nblk, e0 >> 5, half, in);
        }
    }
    __syncthreads();
}

// LONG rows of the decode GEMV (gemv_decode_kernel and the persistent kernel's phases): the warp that owns item i of a CTA's
// `items` when they are dealt to `nwarp` warps in order
__device__ __forceinline__ int item_owner(int i, int items, int nwarp) { return (int)((((long long)(i + 1)) * nwarp - 1) / items); }

// ---- per-chunk math -------------------------------------------------------------------------------
template <int WDT, bool ACTQ8, int MM, int CH>
__device__ __forceinline__ void compute_chunk(const WBuf<WDT, CH> &w, float (&acc)[MM], const unsigned char *smem, int blk0,
                                              int nblk, int lane) {
    const int8_t *aq = (const int8_t *)smem;
    const float *asc = (const float *)(smem + (size_t)MM * nblk * 32);
    const int *asum = (const int *)(smem + (size_t)MM * nblk * 32 + (size_t)MM * nblk * 4);
    const float *af = (const float *)smem;
#pragma unroll
    for (int j = 0; j < CH; j++) {
        int bi = blk0 + j * 32 + lane;
        if (bi >= nblk) continue;
        const float sb = w.s[j];
        if (ACTQ8) {
#pragma unroll
            for (int m = 0; m < MM; m++) {
                const uint4 alo = *(const uint4 *)(aq + (((size_t)m * 2 + 0) * nblk + bi) * 16);
                const uint4 ahi = *(const uint4 *)(aq + (((size_t)m * 2 + 1) * nblk + bi) * 16);
                int s = 0;
                if (WDT == JL_Q4) {
                    const uint4 q = w.q[j];
                    s = __dp4a((int)(q.x & 0x0F0F0F0Fu), (int)alo.x, s);
                    s = __dp4a((int)((q.x >> 4) & 0x0F0F0F0Fu), (int)ahi.x, s);
                    s = __dp4a((int)(q.y & 0x0F0F0F0Fu), (int)alo.y, s);
                    s = __dp4a((int)((q.y >> 4) & 0x0F0F0F0Fu), (int)ahi.y, s);
                    s = __dp4a((int)(q.z & 0x0F0F0F0Fu), (int)alo.z, s);
                    s = __dp4a((int)((q.z >> 4) & 0x0F0F0F0Fu), (int)ahi.z, s);
                    s = __dp4a((int)(q.w & 0x0F0F0F0Fu), (int)alo.w, s);
                    s = __dp4a((int)((q.w >> 4) & 0x0F0F0F0Fu), (int)ahi.w, s);
                    s -= 8 * asum[m * nblk + bi]; // sum a*(nib-8) = sum a*nib - 8*sum a   (exact)
                } else {
                    const uint4 q0 = w.q[2 * j], q1 = w.q[2 * j + 1];
                    s = __dp4a((int)q0.x, (int)alo.x, s);
                    s = __dp4a((int)q0.y, (int)alo.y, s);
                    s = __dp4a((int)q0.z, (int)alo.z, s);
                    s = __dp4a((int)q0.w, (int)alo.w, s);
                    s = __dp4a((int)q1.x, (int)ahi.x, s);
                    s = __dp4a((int)q1.y, (int)ahi.y, s);
                    s = __dp4a((int)q1.z, (int)ahi.z, s);
                    s = __dp4a((int)q1.w, (int)ahi.w, s);
                }
                // acc += (sa*sb) * isum   (vector_simd.c:384-420)
                acc[m] = fmaf(__fmul_rn(asc[m * nblk + bi], sb), (float)s, acc[m]);
            }
        } else {
            // F32 activations: acc += sb * sum_j a_j * (w_j)   with w_j = nib-8 (Q4) or int8 (I8)
            float wf[32];
            if (WDT == JL_Q4) {
                const uint4 q = w.q[j];
                const uint32_t qw[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const uint32_t lo = qw[i] & 0x0F0F0F0Fu, hi = (qw[i] >> 4) & 0x0F0F0F0Fu;
#pragma unroll
                    for (int t = 0; t < 4; t++) {
                        // byte t -> float(2^23 + nib) via PRMT, minus (2^23 + 8)
                        wf[i * 4 + t] = __uint_as_float(__byte_perm(lo, 0x4B000000u, 0x7540 | t)) - 8388616.0f;
                        wf[16 + i * 4 + t] = __uint_as_float(__byte_perm(hi, 0x4B000000u, 0x7540 | t)) - 8388616.0f;
                    }
                }
            } else {
                const uint4 q0 = w.q[2 * j], q1 = w.q[2 * j + 1];
                const uint32_t qw[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
                for (int i = 0; i < 8; i++)
#pragma unroll
                    for (int t = 0; t < 4; t++) wf[i * 4 + t] = (float)(int)(int8_t)((qw[i] >> (8 * t)) & 0xFF);
            }
#pragma unroll
            for (int m = 0; m < MM; m++) {
                float part = 0.0f;
#pragma unroll
                for (int c4 = 0; c4 < 8; c4++) {
                    const float4 a4 = *(const float4 *)(af + (((size_t)m * 8 + c4) * nblk + bi) * 4);
                    part = fmaf(a4.x, wf[c4 * 4 + 0], part);
                    part = fmaf(a4.y, wf[c4 * 4 + 1], part);
                    part = fmaf(a4.z, wf[c4 * 4 + 2], part);
                    part = fmaf(a4.w, wf[c4 * 4 + 3], part);
                }
                acc[m] = fmaf(sb, part, acc[m]);
            }
        }
    }
}

// ---- one M = 1 GEMV pass over quantised weights with Q8 activations -----------------------------------------------
// The body of gemv_decode_kernel (jl_gemv.cu) and of every GEMV phase of the persistent decode kernel (jl_pdecode.cu).
// Work split: output rows are dealt to the CTAs; inside a CTA the (row, weight-row, chunk) items are dealt to the warps.
// LONG = false (a weight row is one chunk, K <= 1024*CH): whole rows go to warps, a warp finishes its rows alone.
// LONG = true (down_proj: K = 14336 = 3.5 chunks): rows are split at chunk granularity, so every warp streams the same
// number of bytes (+-1 chunk) however few rows the CTA has; a warp leaves one partial sum per (row, weight-row) it
// touched in shared memory and, after a barrier, one thread per output row adds the partials in chunk order
// (deterministic).
//
// Ph supplies, as inline methods, what differs between the two kernels:
//   tid(), cta(), ncta()                     thread id, CTA id and grid size (the persistent kernel's are opaque copies)
//   K(), rows()                              reduction length and output rows of the pass
//   begin(), end()                           first and last code of the pass; begin() == false skips the pass and end()
//   row_ptrs(row, wr, nblk, wrow, srow)      weight and scale row of weight-row wr (gate / up) of output row `row`
//   prime_begin(buf), prime_end(smem, nblk)  before and after the ring is primed: activation staging, dependency waits
//   cta_bar()                                the CTA barrier before the LONG partials are combined
//   store_row(row, v0, v1)                   epilogue of one output row (v0 = value or gate, v1 = up)
// Each hook runs where the kernel ran that code before the two passes were merged: moving any of it changes the
// compiled kernels.
template <class Ph, int WDT, int EPI, int CH, int NBUF, int NT, bool LONG>
__device__ __forceinline__ void gemv_phase(Ph &ph, unsigned char *smem) {
    constexpr int NWARP = NT / 32;
    constexpr int NW = (EPI == EPI_SILU_MUL) ? 2 : 1; // weight rows per output row
    const int tid = ph.tid(), lane = tid & 31, warp = tid >> 5;
    const int nblk = ph.K() / 32;
    const int nchunks = LONG ? (nblk + 32 * CH - 1) / (32 * CH) : 1;
    if (!ph.begin()) return;

    // rows of this CTA, items of this warp
    const int R0 = (int)(((long long)ph.rows() * ph.cta()) / ph.ncta());
    const int R1 = (int)(((long long)ph.rows() * (ph.cta() + 1)) / ph.ncta());
    const int nrows = R1 - R0;
    const int per_row = NW * nchunks;
    const int items = nrows * per_row;
    int i0, i1;
    if (LONG) {
        i0 = (int)(((long long)items * warp) / NWARP);
        i1 = (int)(((long long)items * (warp + 1)) / NWARP);
    } else {
        i0 = (int)(((long long)nrows * warp) / NWARP) * per_row;
        i1 = (int)(((long long)nrows * (warp + 1)) / NWARP) * per_row;
    }
    // cursor: (row relative to R0, weight-row, chunk)
    struct It {
        int r, wr, c;
    };
    auto row_ptrs = [&](const It &it, const uint8_t *&wrow, const float *&srow) { ph.row_ptrs(R0 + it.r, it.wr, nblk, wrow, srow); };
    auto advance = [&](It &it) {
        if (!LONG || ++it.c == nchunks) {
            it.c = 0;
            if (++it.wr == NW) {
                it.wr = 0;
                ++it.r;
            }
        }
    };
    It cur, ld;
    {
        cur.r = i0 / per_row;
        const int rem = i0 - cur.r * per_row;
        cur.wr = rem / nchunks;
        cur.c = rem - cur.wr * nchunks;
        ld = cur;
    }

    WBuf<WDT, CH> buf[NBUF];
    // NBUF-1 chunks per warp go in flight before the activations are staged: the weight stream does not depend on them
    ph.prime_begin(buf);
    const uint8_t *wrow;
    const float *srow;
    const unsigned long long pol = l2_evict_first_policy();
    int ci = i0, li = i0;
#pragma unroll
    for (int b = 0; b < NBUF - 1; b++) {
        if (li < i1) {
            row_ptrs(ld, wrow, srow);
            load_chunk<WDT, CH>(buf[b], wrow, srow, ld.c * 32 * CH, nblk, lane, pol);
            advance(ld);
            li++;
        }
    }
    ph.prime_end(smem, nblk);

    float *parts = (float *)(smem + gemv_parts_offset(nblk));
    const int maxsplit = nchunks < NWARP ? nchunks : NWARP;
    float acc[1] = {0.0f};
    // !LONG: finished rows are parked one per lane (lane i holds the i-th finished row of this warp) and the epilogue --
    // residual add or the double-precision SiLU -- runs for all parked rows at once with coalesced stores, instead of
    // lane 0 doing it serially after every row (gate+up: 18.7 vs 19.9 us per launch)
    float park0 = 0.0f, park1 = 0.0f; // value (or gate), up
    int nparked = 0, park_row0 = R0 + cur.r;
    auto flush = [&]() {
        if (lane < nparked) ph.store_row(park_row0 + lane, park0, park1);
        park_row0 += nparked;
        nparked = 0;
    };
    while (ci < i1) {
#pragma unroll
        for (int b = 0; b < NBUF; b++) {
            if (ci < i1) {
                if (li < i1) {
                    row_ptrs(ld, wrow, srow);
                    load_chunk<WDT, CH>(buf[(b + NBUF - 1) % NBUF], wrow, srow, ld.c * 32 * CH, nblk, lane, pol);
                    advance(ld);
                    li++;
                }
                compute_chunk<WDT, true, 1, CH>(buf[b], acc, smem, cur.c * 32 * CH, nblk, lane);
                if (!LONG) {
                    const float v = warp_sum(acc[0]); // every lane has the total
                    acc[0] = 0.0f;
                    if (NW == 2 && cur.wr == 0) {
                        if (lane == nparked) park0 = v;
                    } else {
                        if (lane == nparked) (NW == 2 ? park1 : park0) = v;
                        ++nparked;
                    }
                } else if (cur.c == nchunks - 1 || ci == i1 - 1) {
                    // partial of (row, weight-row) from this warp
                    const float v = warp_sum(acc[0]);
                    const int rw = cur.r * NW + cur.wr;
                    // slot: with at least one item per warp the row's owners are consecutive warps; with fewer items than warps
                    // (a launch of few rows) each warp owns at most one item, so its chunk is its slot (owners are not consecutive)
                    const int slot = items >= NWARP ? warp - item_owner(rw * nchunks, items, NWARP) : cur.c;
                    if (lane == 0) parts[rw * maxsplit + slot] = v;
                    acc[0] = 0.0f;
                }
                advance(cur);
                ci++;
            }
        }
        if (!LONG && nparked > 32 - NBUF) flush(); // checked once per ring revolution: at most NBUF rows arrive in between
    }
    if (!LONG) flush();
    if (LONG) {
        ph.cta_bar();
        for (int o = tid; o < nrows; o += NT) {
            float sums[NW];
#pragma unroll
            for (int wr = 0; wr < NW; wr++) {
                const int rw = o * NW + wr;
                const int wa = items >= NWARP ? item_owner(rw * nchunks, items, NWARP) : 0;
                const int ns = items >= NWARP ? item_owner(rw * nchunks + nchunks - 1, items, NWARP) - wa + 1 : nchunks;
                float t = 0.0f;
                for (int s = 0; s < ns; s++) t = __fadd_rn(t, parts[rw * maxsplit + s]);
                sums[wr] = t;
            }
            ph.store_row(R0 + o, sums[0], sums[NW - 1]);
        }
    }
    ph.end();
}

