// Persistent decode kernel: ONE cooperative launch = one decoded token (M = 1), one 512-thread CTA per SM.
//
// It executes AbstractModel.forward + sample (core/model/AbstractModel.java:314-329,443-473) for one session:
// embedding row, then per layer TransformerBlock.forward (TransformerBlock.java:158-215) = RMSNorm -> Q8 -> QKV
// (CausalSelfAttention.java:161-171) -> RoPE / KV append / attention over the pages (:199-356) -> Q8 -> o_proj + residual
// (:363-378) -> RMSNorm -> Q8 -> gate/up + SiLU*up (MLPBlock.java:117-141) -> Q8 -> down_proj + residual (:144-160), then
// the final norm, the F32 x Q4 lm_head GEMV and the arg-max (strict '>', lowest index).
//
// Why one kernel (DESIGN.md sections 5 and 9.1): in the kernel-per-op graph every GEMV launch paid ~0.85 us of launch
// gap plus ~3 us until its first weights arrived; 128 launches per token = 0.5 ms of a 1.74 ms step.  Here the five ops
// of a layer are PHASES of one resident grid:
//   * the GEMV body is the register-ring body of jl_gemv.cu (128-bit evict-first loads straight into a 3-deep ring of
//     register chunks, dp4a against Q8 activations staged in shared memory, warp-shuffle reduction, fused epilogues);
//   * a phase ends with `bar.sync; red.release.gpu` on a cumulative counter; the next phase's weights do not depend on
//     activations, so every warp puts its first ring chunks in flight BEFORE it polls the counter (ld.acquire.gpu): the
//     weight stream keeps running through the barrier and the ~3 us first-data latency of a fresh kernel is hidden;
//   * activations written by other CTAs are only ever read through L2 (ld.global.cg); residual rows are re-read by the
//     CTA that wrote them (same row partition in o_proj and down_proj);
//   * attention runs as (kv head, context split) tasks on the first CTAs while all others sit at the barrier with
//     their o_proj ring primed;
//   * tensor parallelism (jlama-net model shards, DistributedContext.java:79-98): the o_proj / down_proj partial sums
//     are exchanged INSIDE the kernel over NVLink peer memory with 8-byte self-validating {value, tag} stores (the LL
//     protocol: no fence round trip), reduced in rank order by the CTA that owns the rows, residual added in the same
//     pass -- this replaces JlamaService.combine (jlama-net .../JlamaService.java:300-359) and the round-1
//     ncclAllReduce + copy + accumulate; the lm_head is sharded by vocabulary rows with an exchange of per-rank
//     (max, argmax) candidates.
// Every spin is bounded: a protocol error sets sync[1] and the launch drains instead of hanging the GPU.
#include "jl_pdecode.cuh"
#include "jl_gemv_body.cuh"
#define JL_EXP_FN __forceinline__ // no ABI calls inside the persistent kernel
#include "jl_attn_task.cuh"
#include "jl_attn_flat.cuh"
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

#define PD_NT PD_THREADS
#define PD_NWARP (PD_NT / 32)
#define PD_CH(WDT) ((WDT) == JL_Q4 ? 4 : 2) // 32-block groups per lane per chunk: an int8 block is two 128-bit loads
#define PD_NBUF 3
#define PD_SPIN_LOCAL (1u << 22)
#define PD_SPIN_PEER (1u << 26)
#define EPI_LL 3 // partial sums to every rank's LL receive buffer (tensor parallel o_proj / down_proj)

// ---- model constants ----------------------------------------------------------------------------------------------------
// Everything a phase needs -- dims, buffers, per-layer weight pointers -- lives in __constant__ memory, so the phase bodies use
// constant-bank operands exactly like the stand-alone kernels use their kernel parameters.  (First version: descriptors built
// in registers / local memory and handed to the phase functions by reference cost ~40 local loads per chunk in the hot loop
// and made every phase 2x slower than its stand-alone kernel: 4.5 ms/token.)  The host uploads the block when another model
// takes the device over (jl_launch_pdecode); token-varying values (context splits, flags) are kernel arguments.
#define PD_MAX_LAYERS 128
struct PdConst {
    PdParams P[1];
    PdLayer layers[PD_MAX_LAYERS];
};
__constant__ PdConst c_pd;
#define CP (c_pd.P[0])
// (the helpers below still carry a `pz` argument from an experiment with opaque-indexed constant reads; it is unused)
#define PD_OPAQUE_ZERO(name) const int name = 0

enum { PH_QKV = 0, PH_O, PH_GU, PH_DOWN };

// Every CTA-wide barrier of the kernel is the named barrier 1 over its PD_NT threads.
__device__ __forceinline__ void pd_cta_bar() { asm volatile("bar.sync 1, %0;" ::"n"(PD_NT) : "memory"); }

// ---- cross-CTA ordering ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long pd_ld_acquire(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long pd_ld_volatile(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
// all threads of the CTA call; publishes everything the CTA wrote in this phase
__device__ __forceinline__ void pd_arrive(const int pz, int which) {
    pd_cta_bar();
    if (threadIdx.x == 0) asm volatile("red.release.gpu.global.add.u64 [%0], 1;" ::"l"(CP.sync + which) : "memory");
}
// all threads of the CTA call
__device__ __forceinline__ void pd_wait(const int pz, int which, unsigned long long target) {
    if (threadIdx.x == 0) {
        unsigned long long *sync = CP.sync;
        const unsigned long long *c = sync + which;
        unsigned n = 0;
        while (pd_ld_acquire(c) < target) {
            if ((++n & 0x3ff) == 0) {
                if (pd_ld_volatile(sync + 1) != 0) break; // another CTA gave up: drain
                if (n > PD_SPIN_LOCAL) {
                    sync[1] = (unsigned long long)which;
                    break;
                }
            }
        }
    }
    pd_cta_bar();
}
__device__ __forceinline__ void pd_stamp(const int pz, int idx) {
    if (CP.trace && blockIdx.x == 0 && threadIdx.x == 0) CP.trace[idx] = globaltimer_ns();
}

// ---- LL exchange ----------------------------------------------------------------------------------------------------------
// half-line (8 bytes {value, tag}) of row `row` in the [this rank] block of every rank's receive buffer
template <int PH>
__device__ __forceinline__ void ll_store(const int pz, int row, float v, uint32_t tag) {
    const int world = CP.world;
#pragma unroll 1
    for (int d = 0; d < world; d++) {
        uint32_t *dst = (uint32_t *)(PH == PH_O ? CP.ll_o[d] : CP.ll_d[d]) + ((size_t)CP.rank * CP.E + row) * 2;
        asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(dst), "r"(__float_as_uint(v)), "r"(tag) : "memory");
    }
}
__device__ __forceinline__ float ll_load(const int pz, const uint4 *mine, int src_rank, int row, uint32_t tag) {
    const uint32_t *src = (const uint32_t *)mine + ((size_t)src_rank * CP.E + row) * 2;
    uint32_t v, t;
    unsigned n = 0;
    for (;;) {
        asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(v), "=r"(t) : "l"(src) : "memory");
        if (t == tag) break;
        if ((++n & 0x3ff) == 0) {
            if (pd_ld_volatile(CP.sync + 1) != 0) break;
            if (n > PD_SPIN_PEER) {
                CP.sync[1] = 100 + (unsigned long long)src_rank;
                break;
            }
        }
    }
    return __uint_as_float(v);
}

__device__ __forceinline__ unsigned long long pd_pack_arg(float v, int idx) {
    if (!(v == v)) return 0ull; // NaN never wins (AbstractModel.java:465: 'v > maxv' is false)
    uint32_t b = __float_as_uint(v);
    b = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    return ((unsigned long long)b << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)idx);
}

// ---- phase descriptors straight from constant memory ---------------------------------------------------------------------
template <int PH>
__device__ __forceinline__ int ph_K(const int pz) { return PH == PH_O ? CP.attn_seg : (PH == PH_DOWN ? CP.H : CP.E); }
template <int PH>
__device__ __forceinline__ int ph_rows(const int pz) { return PH == PH_QKV ? CP.attn_seg + 2 * CP.kv_seg : (PH == PH_GU ? CP.H : CP.E); }
// concatenated row -> (segment, row inside the segment); only QKV has more than one segment (gate/up pairs use wr)
template <int PH>
__device__ __forceinline__ void ph_seg(const int pz, int row, int &seg, int &local) {
    seg = 0, local = row;
    if (PH == PH_QKV && local >= CP.attn_seg) {
        local -= CP.attn_seg, seg = 1;
        if (local >= CP.kv_seg) local -= CP.kv_seg, seg = 2;
    }
}
template <int PH>
__device__ __forceinline__ void ph_weights(int L, int seg, const uint8_t *&w, const float *&s) {
    const PdLayer &l = c_pd.layers[L];
    const int slot = PH == PH_QKV ? PW_Q + seg : (PH == PH_O ? PW_O : (PH == PH_GU ? PW_GATE + seg : PW_DOWN));
    w = l.w[slot], s = l.s[slot];
}
template <int PH>
__device__ __forceinline__ float *ph_out(const int pz, int seg) {
    return PH == PH_QKV ? (seg == 0 ? CP.q : (seg == 1 ? CP.k : CP.v)) : (PH == PH_O ? CP.xb : (PH == PH_GU ? CP.h : CP.x));
}

// The ring registers are only ever written under conditions (rows left, block inside the row).  With several phases inlined into
// one kernel a conditionally-defined register is live from the kernel entry to its last use: every phase's ring then overlaps all
// earlier phases and the allocator spills the rings to local memory (LDG -> STL -> LDL, 2x slower phases).  A definite
// definition at the start of the phase ends that.
template <int WDT, int CH, int NBUF>
__device__ __forceinline__ void pd_ring_clear(WBuf<WDT, CH> (&buf)[NBUF]) {
#pragma unroll
    for (int b = 0; b < NBUF; b++) {
#pragma unroll
        for (int j = 0; j < CH * (WDT == JL_I8 ? 2 : 1); j++) buf[b].q[j] = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int j = 0; j < CH; j++) buf[b].s[j] = 0.0f;
    }
}

// ---- one quantised GEMV phase (M = 1, Q8 activations) -------------------------------------------------------------------
// The pass is gemv_phase (jl_gemv_body.cuh).  The ring is primed BEFORE the dependency counter is polled.
// gemv_phase's view of a phase: the layer's weights and activations from constant memory, the dependency wait between ring
// priming and staging, and the epilogue into the phase's output or (EPI_LL) every rank's receive buffer
template <int WDT, int PH, int EPI, bool LONG>
struct PdGemv {
    static constexpr bool NORM = PH == PH_QKV || PH == PH_GU, XLONG = LONG && !NORM;
    int tid_, cta_, ncta_; // opaque copies, see pd_gemv
    int L;
    uint32_t tag;
    int dep_which;
    unsigned long long dep_target;
    int stamp_idx;
    __device__ __forceinline__ int K() const { return ph_K<PH>(0); }
    __device__ __forceinline__ int rows() const { return ph_rows<PH>(0); }
    __device__ __forceinline__ int tid() const { return tid_; }
    __device__ __forceinline__ int cta() const { return cta_; }
    __device__ __forceinline__ int ncta() const { return ncta_; }
    __device__ __forceinline__ bool begin() const { return true; }
    __device__ __forceinline__ void end() const {}
    __device__ __forceinline__ void row_ptrs(int row, int wr, int nblk, const uint8_t *&wrow, const float *&srow) const {
        int seg, local;
        if (EPI == EPI_SILU_MUL) {
            seg = wr;
            local = row;
        } else {
            ph_seg<PH>(0, row, seg, local);
        }
        const uint8_t *w;
        const float *s;
        ph_weights<PH>(L, seg, w, s);
        const size_t blk = (size_t)local * (size_t)nblk;
        wrow = w + blk * (WDT == JL_Q4 ? 16 : 32);
        srow = s + blk;
    }
    template <int CH, int NBUF>
    __device__ __forceinline__ void prime_begin(WBuf<WDT, CH> (&buf)[NBUF]) {
        pd_ring_clear<WDT, CH, NBUF>(buf);
    }
    __device__ __forceinline__ void prime_end(unsigned char *smem, int nblk) {
        PD_OPAQUE_ZERO(pz);
        pd_wait(pz, dep_which, dep_target);
        pd_stamp(pz, stamp_idx);
        GemvParams p; // only the staging fields; dead after the prologue
        p.a = PH == PH_QKV ? CP.x : (PH == PH_O ? CP.att : (PH == PH_GU ? CP.xb : CP.h));
        p.a_col_off = 0, p.K = ph_K<PH>(pz), p.lda = p.K;
        p.norm_w = PH == PH_QKV ? c_pd.layers[L].attn_norm : c_pd.layers[L].ffn_norm;
        p.norm_w_dtype = PH == PH_QKV ? c_pd.layers[L].attn_norm_dt : c_pd.layers[L].ffn_norm_dt;
        p.norm_adj = 0.0f, p.norm_eps = CP.eps, p.norm_E = CP.E, p.norm_inv_E = 1.0 / (double)CP.E;
        StageRegs<NORM, XLONG> sr;
        stage_q8_issue<NORM, XLONG, PD_NT>(p, sr);
        stage_q8_finish<NORM, XLONG, PD_NT, 1>(p, sr, smem, nblk);
    }
    __device__ __forceinline__ void cta_bar() const { pd_cta_bar(); }
    // row = index in the concatenated row space of the phase
    __device__ __forceinline__ void store_row(int row, float v0, float v1) const {
        PD_OPAQUE_ZERO(pz);
        int seg = 0, local = row;
        if (EPI != EPI_SILU_MUL) ph_seg<PH>(pz, row, seg, local);
        float v = EPI == EPI_SILU_MUL ? v1 : v0;
        if (EPI == EPI_ADD_RESIDUAL) v = __fadd_rn(v, __ldcg((PH == PH_O ? CP.x : CP.xb) + local));
        if (EPI == EPI_SILU_MUL) v = __fmul_rn(silu_ref(v0), v);
        if (EPI == EPI_LL) ll_store<PH>(pz, local, v, tag);
        else ph_out<PH>(pz, seg)[local] = v;
    }
};

template <int WDT, int PH, int EPI, bool LONG>
__device__ __forceinline__ void pd_gemv(const int, const int L, const uint32_t tag, const int dep_which, const unsigned long long dep_target,
                                        const int stamp_idx, unsigned char *smem) {
    // The phases are inlined into one loop over the layers and all their index arithmetic (row ranges, item ranges, ...) is
    // loop-invariant: hoisted out of the layer loop it stayed live across every phase (~60 registers) and the weight ring
    // spilled to local memory.  An opaque copy of the thread / CTA ids keeps each phase's bookkeeping inside the phase.
    int tid = threadIdx.x, cta_id = blockIdx.x, ncta = gridDim.x;
    asm volatile("" : "+r"(tid), "+r"(cta_id), "+r"(ncta));
    PdGemv<WDT, PH, EPI, LONG> ph{tid, cta_id, ncta, L, tag, dep_which, dep_target, stamp_idx};
    gemv_phase<decltype(ph), WDT, EPI, PD_CH(WDT), PD_NBUF, PD_NT, LONG>(ph, smem);
}

// ---- lm_head: F32 activations (RMSNorm, not re-quantised: AbstractModel.java:444-449) x quantised rows + running arg-max --
template <int WDT>
__device__ __forceinline__ unsigned long long pd_lm_head(const int, const int dep_which, const unsigned long long dep_target, const int stamp_idx,
                                                     const int want_logits, unsigned char *smem) {
    PD_OPAQUE_ZERO(pz);
    constexpr int NT = PD_NT, NWARP = PD_NWARP, CH = PD_CH(WDT), NBUF = PD_NBUF;
    constexpr int WB = (WDT == JL_Q4) ? 16 : 32;
    __shared__ double red[NWARP];
    __shared__ unsigned long long wbest[NWARP];
    int tid = threadIdx.x, cta_id = blockIdx.x, ncta = gridDim.x;
    asm volatile("" : "+r"(tid), "+r"(cta_id), "+r"(ncta)); // see pd_gemv
    const int lane = tid & 31, warp = tid >> 5;
    const int K = CP.E, nblk = K / 32;
    const int R0 = (int)(((long long)CP.vocab_rows * cta_id) / ncta);
    const int R1 = (int)(((long long)CP.vocab_rows * (cta_id + 1)) / ncta);
    const int nrows = R1 - R0;
    const int r0 = R0 + (int)(((long long)nrows * warp) / NWARP), r1 = R0 + (int)(((long long)nrows * (warp + 1)) / NWARP);
    const int nchunks = (nblk + 32 * CH - 1) / (32 * CH);
    WBuf<WDT, CH> buf[NBUF];
    pd_ring_clear<WDT, CH, NBUF>(buf);
    const unsigned long long pol = l2_evict_first_policy();
    int lr = r0, lc = 0, cr = r0, cc = 0;
    auto issue = [&](WBuf<WDT, CH> &b) {
        const size_t blk = (size_t)lr * nblk;
        load_chunk<WDT, CH>(b, CP.lm_w + blk * WB, CP.lm_s + blk, lc * 32 * CH, nblk, lane, pol);
        if (++lc == nchunks) lc = 0, ++lr;
    };
#pragma unroll
    for (int b = 0; b < NBUF - 1; b++)
        if (lr < r1) issue(buf[b]);
    pd_wait(pz, dep_which, dep_target);
    pd_stamp(pz, stamp_idx);
    // final RMSNorm into the [c4(8)][blk][4] float layout of compute_chunk<.., ACTQ8 = false>
    {
        float4 *af4 = (float4 *)smem;
        double ss = 0.0;
        for (int i4 = tid; i4 < K / 4; i4 += NT) {
            const float4 v = __ldcg((const float4 *)(CP.x + i4 * 4));
            ss += (double)__fmul_rn(v.x, v.x);
            ss += (double)__fmul_rn(v.y, v.y);
            ss += (double)__fmul_rn(v.z, v.z);
            ss += (double)__fmul_rn(v.w, v.w);
        }
        ss = warp_sum_d(ss);
        if (lane == 0) red[warp] = ss;
        pd_cta_bar();
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < NWARP; w++) t += red[w];
        const float rsf = rms_scale(t, 1.0 / (double)CP.E, CP.eps);
        for (int i4 = tid; i4 < K / 4; i4 += NT) {
            const float4 v = __ldcg((const float4 *)(CP.x + i4 * 4));
            float w[4];
            if (CP.out_norm_dt == JL_BF16) {
                const uint2 u = __ldg((const uint2 *)((const uint16_t *)CP.out_norm + i4 * 4));
                w[0] = __uint_as_float(u.x << 16), w[1] = __uint_as_float(u.x & 0xffff0000u);
                w[2] = __uint_as_float(u.y << 16), w[3] = __uint_as_float(u.y & 0xffff0000u);
            } else {
                const float4 f = __ldg((const float4 *)((const float *)CP.out_norm + i4 * 4));
                w[0] = f.x, w[1] = f.y, w[2] = f.z, w[3] = f.w;
            }
            const int b = i4 >> 3, c4 = i4 & 7;
            af4[(size_t)c4 * nblk + b] = make_float4(__fmul_rn(__fadd_rn(0.0f, w[0]), __fmul_rn(rsf, v.x)), __fmul_rn(__fadd_rn(0.0f, w[1]), __fmul_rn(rsf, v.y)),
                                                     __fmul_rn(__fadd_rn(0.0f, w[2]), __fmul_rn(rsf, v.z)), __fmul_rn(__fadd_rn(0.0f, w[3]), __fmul_rn(rsf, v.w)));
        }
        pd_cta_bar();
    }
    float acc[1] = {0.0f};
    float best_v = -INFINITY;
    int best_i = 0x7fffffff;
    while (cr < r1) {
#pragma unroll
        for (int b = 0; b < NBUF; b++) {
            if (cr < r1) {
                if (lr < r1) issue(buf[(b + NBUF - 1) % NBUF]);
                compute_chunk<WDT, false, 1, CH>(buf[b], acc, smem, cc * 32 * CH, nblk, lane);
                if (++cc == nchunks) {
                    const float v = warp_sum(acc[0]);
                    acc[0] = 0.0f;
                    const int grow = CP.vocab0 + cr;
                    if (lane == 0) {
                        CP.logits[grow] = v;
                        if (want_logits)
                            for (int d = 0; d < CP.world; d++)
                                if (d != CP.rank) CP.logits_peer[d][grow] = v;
                    }
                    if (v > best_v) best_v = v, best_i = grow; // rows ascend: strict '>' keeps the lowest index
                    cc = 0, ++cr;
                }
            }
        }
    }
    if (lane == 0) wbest[warp] = best_i == 0x7fffffff ? 0ull : pd_pack_arg(best_v, best_i);
    pd_cta_bar();
    unsigned long long b = 0ull;
    if (tid == 0)
        for (int w = 0; w < NWARP; w++) b = wbest[w] > b ? wbest[w] : b;
    return b; // valid in thread 0
}

__device__ __forceinline__ float pd_embed_value(const int pz, size_t tok, int c) {
    // LlamaModel.java:68-100 (Q4 / I8 rows are read through get(): Q4ByteBufferTensor.java:179-197)
    const int E = CP.E;
    if (CP.embed_dt == JL_F32) return ((const float *)CP.embed_w)[tok * E + c];
    if (CP.embed_dt == JL_BF16) return bf16_bits_to_f32(((const uint16_t *)CP.embed_w)[tok * E + c]);
    if (CP.embed_dt == JL_Q4) {
        const int blk = c / 32, in = c % 32;
        const uint8_t byte = ((const uint8_t *)CP.embed_w)[(tok * E + blk * 32) / 2 + (in & 15)];
        const int nib = in < 16 ? (byte & 0x0F) : (byte >> 4);
        return __fmul_rn((float)(nib - 8), CP.embed_s[tok * (E / 32) + blk]);
    }
    return __fmul_rn((float)((const int8_t *)CP.embed_w)[tok * E + c], CP.embed_s[tok * (E / 32) + c / 32]);
}

// reduce the LL partials of this CTA's rows in rank order, add the residual, store the new hidden rows (local global)
template <int PH>
__device__ __forceinline__ void pd_ll_reduce(const int, uint32_t tag, float *scratch /* smem [rows][world] */) {
    PD_OPAQUE_ZERO(pz);
    const int tid = threadIdx.x;
    const int E = CP.E, W = CP.world;
    const int R0 = (int)(((long long)E * blockIdx.x) / gridDim.x), R1 = (int)(((long long)E * (blockIdx.x + 1)) / gridDim.x);
    const int nrows = R1 - R0;
    const uint4 *mine = PH == PH_O ? CP.ll_o[CP.rank] : CP.ll_d[CP.rank];
    const float *residual = PH == PH_O ? CP.x : CP.xb;
    float *out = PH == PH_O ? CP.xb : CP.x;
    for (int t = tid; t < nrows * W; t += PD_NT) {
        const int r = t / W, src = t - r * W;
        scratch[t] = ll_load(pz, mine, src, R0 + r, tag);
    }
    pd_cta_bar();
    for (int r = tid; r < nrows; r += PD_NT) {
        float s = scratch[r * W];
        for (int src = 1; src < W; src++) s = __fadd_rn(s, scratch[r * W + src]); // rank order: identical on every rank
        out[R0 + r] = __fadd_rn(s, __ldcg(residual + R0 + r));
    }
}

// One attention task.  qkv_target != 0: the QKV barrier is waited for inside (after the first K/V rows have been requested).
template <int HS>
__device__ __forceinline__ void pd_attention(const int, const int layer, const int kvh, const int split, const int splits, const bool merge,
                                         const unsigned long long qkv_target, unsigned char *smem) {
    PD_OPAQUE_ZERO(pz);
    AttnParams at;
    at.kv = CP.kv, at.layer = layer, at.heads = CP.heads, at.kv_heads = CP.kv_heads, at.head_size = CP.head_size;
    at.kv_head0_global = CP.kv_head0_global, at.q = CP.q, at.k = CP.k, at.v = CP.v, at.q_ld = CP.attn_seg, at.kv_ld = CP.kv_seg;
    at.out = CP.att, at.rope = CP.rope, at.sessions = CP.sessions, at.positions = CP.positions, at.scale = CP.attn_scale;
    at.ws = CP.attn_ws, at.splits = splits, at.head0_global = 0, at.rows = 1; // (head0_global: only the per-op append reads it)
    if (merge) {
        attention_merge<HS, PD_NT>(at, 0, kvh, smem);
        return;
    }
    // (the host only selects this kernel for power-of-two head groups and <= FA_MAX_POS positions per split)
    attention_flat<HS, PD_NT>(at, 0, kvh, split, smem, [&]() { pd_wait(pz, PC_QKV, qkv_target); });
}

template <int WDT, int HS>
__global__ void __launch_bounds__(PD_NT, 1) pdecode_kernel(const int splits0, const int resident, const int want_logits, const int ntok,
                                                            const int split_cap) {
    PD_OPAQUE_ZERO(pz);
    extern __shared__ __align__(1024) unsigned char smem[];
    __shared__ int s_last;
    const int tid = threadIdx.x;
    const int G = gridDim.x, cta = blockIdx.x;
    unsigned long long epoch = pd_ld_volatile(CP.sync); // tokens decoded by this model so far
    const unsigned long long fin0 = pd_ld_volatile(CP.sync + PC_FINAL);
    // ntok > 1 (device-resident loop only): several tokens per launch; the token fed back by CTA 0 is published to the
    // grid through one more barrier (PC_FINAL) instead of a kernel boundary
    for (int tk = 0; tk < ntok; tk++) {
    int splits = splits0;
    if (tk > 0) { // context splits of this token: one per 64 positions up to split_cap (the host computes token 0's)
        pd_wait(pz, PC_FINAL, fin0 + (unsigned long long)tk);
        const int pos = *(volatile const int32_t *)CP.positions;
        splits = (pos + 1 + 63) / 64;
        splits = splits > split_cap ? split_cap : (splits < 1 ? 1 : splits);
    }
    const unsigned long long uG = (unsigned long long)G;
    const bool tp = CP.world > 1;
    const int layers = CP.layers;
    // rows longer than one register chunk run in the split-row form
    const bool lng_E = CP.E > 32 * 32 * PD_CH(WDT), lng_A = CP.attn_seg > 32 * 32 * PD_CH(WDT), lng_H = CP.H > 32 * 32 * PD_CH(WDT);
    pd_stamp(pz, 0);

    // ---- embedding row (columns split over the grid) ----
    {
        const int E = CP.E;
        const int c_a = (int)(((long long)E * cta) / G), c_b = (int)(((long long)E * (cta + 1)) / G);
        const size_t tok = (size_t)__ldcg(CP.tokens); // fed back by CTA 0 of this very launch when ntok > 1
        for (int c = c_a + tid; c < c_b; c += PD_NT) CP.x[c] = pd_embed_value(pz, tok, c);
        pd_arrive(pz, PC_EMBED);
    }
    const int ntasks = CP.kv_heads * splits;

    for (int L = 0; L < layers; L++) {
        PD_OPAQUE_ZERO(pz); // per-iteration: see the note at c_pd
        const unsigned long long use = epoch * (unsigned long long)layers + (unsigned long long)L + 1; // 1-based use count
        const uint32_t tag_o = (uint32_t)(use * 2), tag_d = (uint32_t)(use * 2 + 1);
        // ---- QKV: RMSNorm(x) -> Q8 -> q | k | v ----
        {
            const int dw = L == 0 ? PC_EMBED : PC_DOWN;
            const unsigned long long dt = L == 0 ? (epoch + 1) * uG : (use - 1) * uG;
            if (lng_E) pd_gemv<WDT, PH_QKV, EPI_STORE, true>(pz, L, 0u, dw, dt, 1 + L * 8 + 0, smem);
            else pd_gemv<WDT, PH_QKV, EPI_STORE, false>(pz, L, 0u, dw, dt, 1 + L * 8 + 0, smem);
            pd_arrive(pz, PC_QKV);
            pd_stamp(pz, 1 + L * 8 + 1);
        }
        // ---- attention tasks on the first CTAs (RoPE, KV append, scores, softmax, P.V) ----
        if (cta < ntasks) {
            const int split = cta % splits, kvh = cta / splits;
            pd_attention<HS>(pz, L, kvh, split, splits, false, use * uG, smem);
            bool signal = true;
            if (splits > 1) {
                pd_cta_bar();
                if (tid == 0) {
                    __threadfence();
                    unsigned *c = &CP.att_done[kvh];
                    const unsigned old = atomicAdd(c, 1u);
                    s_last = (old == (unsigned)splits - 1);
                    if (s_last) *c = 0;
                    __threadfence();
                }
                pd_cta_bar();
                signal = s_last != 0;
                if (signal) pd_attention<HS>(pz, L, kvh, split, splits, true, 0ull, smem);
            }
            pd_cta_bar();
            if (signal && tid == 0) asm volatile("red.release.gpu.global.add.u64 [%0], 1;" ::"l"(CP.sync + PC_ATT) : "memory");
            pd_stamp(pz, 1 + L * 8 + 2);
        }
        // ---- o_proj: Q8(att) -> x + o (single rank) or LL partials -> rank-ordered reduce + residual (tensor parallel) ----
        {
            const unsigned long long dt = use * (unsigned long long)CP.kv_heads;
            if (tp) {
                if (lng_A) pd_gemv<WDT, PH_O, EPI_LL, true>(pz, L, tag_o, PC_ATT, dt, 1 + L * 8 + 3, smem);
                else pd_gemv<WDT, PH_O, EPI_LL, false>(pz, L, tag_o, PC_ATT, dt, 1 + L * 8 + 3, smem);
                pd_cta_bar();
                pd_ll_reduce<PH_O>(pz, tag_o, (float *)smem);
            } else {
                if (lng_A) pd_gemv<WDT, PH_O, EPI_ADD_RESIDUAL, true>(pz, L, 0u, PC_ATT, dt, 1 + L * 8 + 3, smem);
                else pd_gemv<WDT, PH_O, EPI_ADD_RESIDUAL, false>(pz, L, 0u, PC_ATT, dt, 1 + L * 8 + 3, smem);
            }
            pd_arrive(pz, PC_O);
            pd_stamp(pz, 1 + L * 8 + 4);
        }
        // ---- gate / up: RMSNorm(xb) -> Q8 -> silu(gate) * up ----
        {
            if (lng_E) pd_gemv<WDT, PH_GU, EPI_SILU_MUL, true>(pz, L, 0u, PC_O, use * uG, 1 + L * 8 + 5, smem);
            else pd_gemv<WDT, PH_GU, EPI_SILU_MUL, false>(pz, L, 0u, PC_O, use * uG, 1 + L * 8 + 5, smem);
            pd_arrive(pz, PC_GU);
            pd_stamp(pz, 1 + L * 8 + 6);
        }
        // ---- down_proj: Q8(h) -> xb + down ----
        {
            if (tp) {
                if (lng_H) pd_gemv<WDT, PH_DOWN, EPI_LL, true>(pz, L, tag_d, PC_GU, use * uG, 1 + L * 8 + 7, smem);
                else pd_gemv<WDT, PH_DOWN, EPI_LL, false>(pz, L, tag_d, PC_GU, use * uG, 1 + L * 8 + 7, smem);
                pd_cta_bar();
                pd_ll_reduce<PH_DOWN>(pz, tag_d, (float *)smem);
            } else {
                if (lng_H) pd_gemv<WDT, PH_DOWN, EPI_ADD_RESIDUAL, true>(pz, L, 0u, PC_GU, use * uG, 1 + L * 8 + 7, smem);
                else pd_gemv<WDT, PH_DOWN, EPI_ADD_RESIDUAL, false>(pz, L, 0u, PC_GU, use * uG, 1 + L * 8 + 7, smem);
            }
            pd_arrive(pz, PC_DOWN);
        }
    }
    // ---- final norm + lm_head + arg-max ----
    const unsigned long long cta_best = pd_lm_head<WDT>(pz, PC_DOWN, (epoch + 1) * (unsigned long long)layers * uG, 1 + layers * 8 + 0, want_logits, smem);
    if (tid == 0) CP.argmax_slots[cta] = cta_best;
    pd_arrive(pz, PC_LM);
    if (cta == 0) {
        pd_wait(pz, PC_LM, (epoch + 1) * uG);
        if (tid < 32) {
            unsigned long long b = 0ull;
            for (int i = tid; i < G; i += 32) {
                const unsigned long long c = __ldcg(&CP.argmax_slots[i]);
                b = c > b ? c : b;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const unsigned long long c = __shfl_xor_sync(0xffffffffu, b, o);
                b = c > b ? c : b;
            }
            if (tp) {
                // exchange the per-rank candidates (lm_head is sharded by vocabulary rows): LL line {lo, tag, hi, tag}
                const uint32_t tag = (uint32_t)(epoch + 1);
                const int world = CP.world, rank = CP.rank;
                if (tid < world) {
                    uint4 *dst = CP.ll_a[tid] + rank;
                    asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "r"((uint32_t)b), "r"(tag), "r"((uint32_t)(b >> 32)), "r"(tag)
                                 : "memory");
                }
                unsigned long long c = 0ull;
                if (tid < world) {
                    const uint4 *src = CP.ll_a[rank] + tid;
                    uint4 v;
                    unsigned n = 0;
                    for (;;) {
                        asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src) : "memory");
                        if (v.y == tag && v.w == tag) break;
                        if ((++n & 0x3ff) == 0) {
                            if (pd_ld_volatile(CP.sync + 1) != 0) break;
                            if (n > PD_SPIN_PEER) {
                                CP.sync[1] = 200 + (unsigned long long)tid;
                                break;
                            }
                        }
                    }
                    c = ((unsigned long long)v.z << 32) | v.x;
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const unsigned long long d = __shfl_xor_sync(0xffffffffu, c, o);
                    c = d > c ? d : c;
                }
                b = c;
            }
            if (tid == 0) {
                const int tok = b == 0ull ? 0 : (int)(0xFFFFFFFFu - (uint32_t)(b & 0xFFFFFFFFull));
                CP.next[0] = tok;
                if (resident) {
                    const int cntv = *CP.counter;
                    CP.tokens[0] = tok;
                    CP.positions[0] += 1;
                    if (cntv < CP.hist_cap) CP.hist[cntv] = tok;
                    *CP.counter = cntv + 1;
                }
                CP.sync[0] = epoch + 1;
                pd_stamp(pz, 1 + layers * 8 + 1);
                if (tk + 1 < ntok) {
                    __threadfence();
                    asm volatile("red.release.gpu.global.add.u64 [%0], 1;" ::"l"(CP.sync + PC_FINAL) : "memory");
                }
            }
        }
    }
    epoch++;
    } // tokens of this launch
}

// ---- host side ----------------------------------------------------------------------------------------------------------------
// G: the grid (one CTA per SM); the split-row phases give each CTA ceil(rows / G) rows
static size_t pd_smem_bytes(const PdParams &p, int G) {
    int Kmax = p.E;
    if (p.H > Kmax) Kmax = p.H;
    if (p.attn_seg > Kmax) Kmax = p.attn_seg;
    int Rmax = p.E > p.H ? p.E : p.H; // rows of the largest phase that may run in the split-row (LONG) form; gate+up has two weight rows
    if (p.attn_seg + 2 * p.kv_seg > Rmax) Rmax = p.attn_seg + 2 * p.kv_seg;
    size_t acts = gemv_parts_offset(Kmax / 32) + (size_t)((Rmax + G - 1) / G + 2) * 2 * PD_NWARP * 4 + 64;
    const size_t lm = (size_t)p.E * 4;
    if (lm > acts) acts = lm;
    const int hs = p.head_size;
    size_t att = hs == 32 ? attention_flat_smem<32, PD_NT>() : (hs == 64 ? attention_flat_smem<64, PD_NT>() : attention_flat_smem<128, PD_NT>());
    att += 1024; // merge factors
    size_t m = acts > att ? acts : att;
    const size_t red = (size_t)((p.E + G - 1) / G + 2) * PD_MAX_TP * 4;
    if (red > m) m = red;
    return (m + 1023) & ~(size_t)1023;
}

bool jl_pdecode_supported(const PdParams &p, int w_dtype, int grid) {
    if (w_dtype != JL_Q4 && w_dtype != JL_I8) return false;
    if (p.head_size != 32 && p.head_size != 64 && p.head_size != 128) return false;
    if (p.heads % p.kv_heads || p.heads / p.kv_heads > MG_MAX_GROUP) return false;
    if ((p.E % 32) || (p.H % 32) || (p.attn_seg % 32) || (p.E % 8)) return false;
    if (p.E > 16 * PD_NT) return false;        // RMSNorm prologue keeps the row in registers (16 floats per thread)
    if (p.kv_heads * 1 > grid) return false;
    if (p.world > PD_MAX_TP || p.layers > PD_MAX_LAYERS) return false;
    {
        const int group = p.heads / p.kv_heads;
        if (group & (group - 1)) return false; // flat attention: power-of-two head groups
    }
    return pd_smem_bytes(p, grid) <= 200 * 1024;
}

// The constant block belongs to one model per device at a time: (owner id, version) of the last upload.
static const void *g_pd_owner[JL_MAX_DEVICES] = {};
static std::mutex g_pd_mu;

void jl_pdecode_forget(int device, const void *owner) {
    std::lock_guard<std::mutex> lk(g_pd_mu);
    if (device >= 0 && device < JL_MAX_DEVICES && g_pd_owner[device] == owner) g_pd_owner[device] = nullptr;
}

template <int WDT, int HS>
static int launch_pd(jl_ctx *ctx, cudaStream_t stream, const PdParams &p) {
    auto kern = pdecode_kernel<WDT, HS>;
    const size_t smem = pd_smem_bytes(p, ctx->sm_count);
    static size_t configured[JL_MAX_DEVICES] = {};
    JL_CUDA_CHECK(ctx, jl_ensure_dyn_smem(kern, ctx->device, smem, configured));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(ctx->sm_count);
    cfg.blockDim = dim3(PD_NT);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative; // all CTAs co-resident: the (bounded) spin waits cannot starve each other
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    JL_CUDA_CHECK(ctx, cudaLaunchKernelEx(&cfg, kern, p.splits, p.resident, p.want_logits, p.ntok > 0 ? p.ntok : 1, p.split_cap));
    ctx->launches++;
    return JL_OK;
}

template <int WDT>
static int launch_pd_hs(jl_ctx *ctx, cudaStream_t stream, const PdParams &p) {
    switch (p.head_size) {
        case 32: return launch_pd<WDT, 32>(ctx, stream, p);
        case 64: return launch_pd<WDT, 64>(ctx, stream, p);
        default: return launch_pd<WDT, 128>(ctx, stream, p);
    }
}

// `owner`: identity of the model the constants belong to; `layers_host`: its PdLayer table (host copy).
int jl_launch_pdecode(jl_ctx *ctx, cudaStream_t stream, const PdParams &p, const PdLayer *layers_host, const void *owner, int w_dtype) {
    if (!jl_pdecode_supported(p, w_dtype, ctx->sm_count)) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "persistent decode: unsupported shape");
    {
        std::lock_guard<std::mutex> lk(g_pd_mu);
        const int d = ctx->device >= 0 && ctx->device < JL_MAX_DEVICES ? ctx->device : 0;
        if (g_pd_owner[d] != owner) {
            // another model's launches may still be reading the block: drain the device before replacing it
            JL_CUDA_CHECK(ctx, cudaDeviceSynchronize());
            PdParams hp = p;
            hp.lw = nullptr;
            JL_CUDA_CHECK(ctx, cudaMemcpyToSymbol(c_pd, &hp, sizeof(PdParams), offsetof(PdConst, P)));
            JL_CUDA_CHECK(ctx, cudaMemcpyToSymbol(c_pd, layers_host, sizeof(PdLayer) * p.layers, offsetof(PdConst, layers)));
            g_pd_owner[d] = owner;
        }
    }
    return w_dtype == JL_Q4 ? launch_pd_hs<JL_Q4>(ctx, stream, p) : launch_pd_hs<JL_I8>(ctx, stream, p);
}
