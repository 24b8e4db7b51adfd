// Memory-bound companions of the GEMV: the element-wise TensorOperations methods, the block
// quantisers, RMSNorm, softmax, SiLU*up, the embedding lookup and arg-max sampling.  In the
// reference most of these are scalar Java loops on AbstractTensor.get/set (SURVEY 8a a9-a17).
#include "jl_common.cuh"

// ---- accumulate: a[r, off+i] += b[(r or 0), off+i]  (NaiveTensorOperations.java:34-46) -------------
__global__ void accumulate_kernel(float *a, int a_rows, int lda, int b_dtype, const void *b, const float *b_scales,
                                  int b_rows, int ldb, int offset, int length) {
    const int r = blockIdx.y;
    const int br = b_rows > 1 ? r : 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < length; i += gridDim.x * blockDim.x) {
        const int c = offset + i;
        float bv;
        if (b_dtype == JL_F32) bv = ((const float *)b)[(size_t)br * ldb + c];
        else if (b_dtype == JL_BF16) bv = bf16_bits_to_f32(((const uint16_t *)b)[(size_t)br * ldb + c]);
        else { // JL_Q4: PanamaTensorOperations.java:2297-2325  a += (nib-8)*scale
            const int blk = c / 32, in = c % 32;
            const uint8_t byte = ((const uint8_t *)b)[((size_t)br * ldb + blk * 32) / 2 + (in & 15)];
            const int nib = in < 16 ? (byte & 0x0F) : (byte >> 4);
            bv = __fmul_rn((float)(nib - 8), b_scales[(size_t)br * (ldb / 32) + blk]);
        }
        a[(size_t)r * lda + c] = __fadd_rn(a[(size_t)r * lda + c], bv);
    }
}
int jl_launch_accumulate(jl_ctx *ctx, cudaStream_t s, float *a, int a_rows, int lda, int b_dtype, const void *b,
                         const float *b_scales, int b_rows, int ldb, int offset, int length) {
    if (length <= 0 || a_rows <= 0) return JL_OK;
    dim3 grid((length + 255) / 256 > 1024 ? 1024 : (length + 255) / 256, a_rows);
    accumulate_kernel<<<grid, 256, 0, s>>>(a, a_rows, lda, b_dtype, b, b_scales, b_rows, ldb, offset, length);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- maccumulate: a *= b (NaiveTensorOperations.java:49-61) ------------------------------------------
__global__ void maccumulate_kernel(float *a, int lda, const float *b, int b_rows, int ldb, int offset, int length) {
    const int r = blockIdx.y, br = b_rows > 1 ? r : 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < length; i += gridDim.x * blockDim.x)
        a[(size_t)r * lda + offset + i] = __fmul_rn(a[(size_t)r * lda + offset + i], b[(size_t)br * ldb + offset + i]);
}
int jl_launch_maccumulate(jl_ctx *ctx, cudaStream_t s, float *a, int a_rows, int lda, const float *b, int b_rows, int ldb,
                          int offset, int length) {
    if (length <= 0 || a_rows <= 0) return JL_OK;
    dim3 grid((length + 255) / 256 > 1024 ? 1024 : (length + 255) / 256, a_rows);
    maccumulate_kernel<<<grid, 256, 0, s>>>(a, lda, b, b_rows, ldb, offset, length);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- scale (NaiveTensorOperations.java:113-119) --------------------------------------------------------
__global__ void scale_kernel(float f, float *x, int ldx, int offset, int length) {
    const int r = blockIdx.y;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < length; i += gridDim.x * blockDim.x)
        x[(size_t)r * ldx + offset + i] = __fmul_rn(x[(size_t)r * ldx + offset + i], f);
}
int jl_launch_scale(jl_ctx *ctx, cudaStream_t s, float f, float *x, int rows, int ldx, int offset, int length) {
    if (length <= 0 || rows <= 0) return JL_OK;
    dim3 grid((length + 255) / 256 > 1024 ? 1024 : (length + 255) / 256, rows);
    scale_kernel<<<grid, 256, 0, s>>>(f, x, ldx, offset, length);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- batched saxpy: y[yoff+i] += sum_r alpha[aoff+r] * x[xrow+r, xoff+i]  (rows in order, FMA) -----------
// PanamaTensorOperations.java:2648-2698 (4 rows per pass, r0 = x0*a0 + y; r0 = x1*a1 + r0; ...)
__global__ void saxpy_batch_kernel(const float *alpha, const float *x, int ldx, float *y, int xoffset, int yoffset,
                                   int limit, int a_offset, int x_row_offset, int batch) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < limit; i += gridDim.x * blockDim.x) {
        float acc = y[yoffset + i];
        for (int r = 0; r < batch; r++)
            acc = fmaf(x[(size_t)(x_row_offset + r) * ldx + xoffset + i], alpha[a_offset + r], acc);
        y[yoffset + i] = acc;
    }
}
int jl_launch_saxpy_batch(jl_ctx *ctx, cudaStream_t s, const float *alpha, const float *x, int ldx, float *y, int xoffset,
                          int yoffset, int limit, int a_offset, int x_row_offset, int batch) {
    if (limit <= 0) return JL_OK;
    saxpy_batch_kernel<<<(limit + 127) / 128, 128, 0, s>>>(alpha, x, ldx, y, xoffset, yoffset, limit, a_offset,
                                                           x_row_offset, batch);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- Q8 activation quantiser (PanamaTensorOperations.java:1684-1723): one warp per 32-block ---------------
__global__ void quantize_q8_kernel(const float *x, int rows, int ldx, int offset, int length, int8_t *q, float *scales) {
    const int lane = threadIdx.x & 31;
    const int nblk = length / 32;
    const long long total = (long long)rows * nblk;
    for (long long w = (long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); w < total;
         w += (long long)gridDim.x * (blockDim.x / 32)) {
        const int r = (int)(w / nblk), b = (int)(w % nblk);
        const size_t idx = (size_t)r * ldx + offset + b * 32 + lane;
        const float v = x[idx];
        const float mx = warp_max(fabsf(v));
        const float d = __fdiv_rn(mx, 127.0f);
        const float id = mx != 0.0f ? __fdiv_rn(127.0f, mx) : 0.0f;
        q[idx] = (int8_t)(int)__fadd_rn(__fmul_rn(v, id), 0.5f);
        if (lane == 0) scales[(size_t)r * (ldx / 32) + offset / 32 + b] = d;
    }
}
int jl_launch_quantize_q8(jl_ctx *ctx, cudaStream_t s, const float *x, int rows, int ldx, int offset, int length,
                          int8_t *q, float *scales) {
    if ((length % 32) || (offset % 32) || (ldx % 32))
        return jl_set_error(ctx, JL_ERR_INVALID, "quantize_q8: offset/length/ld must be multiples of 32");
    long long total = (long long)rows * (length / 32);
    if (total <= 0) return JL_OK;
    int blocks = (int)((total + 7) / 8);
    if (blocks > ctx->sm_count * 8) blocks = ctx->sm_count * 8;
    quantize_q8_kernel<<<blocks, 256, 0, s>>>(x, rows, ldx, offset, length, q, scales);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- f32 -> bf16 RNE, NaN preserving (f32_to_bf16_rne, FloatConversions.java:35-61) ---------------------------------
__global__ void quantize_bf16_kernel(const float *x, int ldx, int offset, int length, uint16_t *out) {
    const int r = blockIdx.y;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < length; i += gridDim.x * blockDim.x)
        out[(size_t)r * ldx + offset + i] = f32_to_bf16_rne(x[(size_t)r * ldx + offset + i]);
}
int jl_launch_quantize_bf16(jl_ctx *ctx, cudaStream_t s, const float *x, int rows, int ldx, int offset, int length,
                            uint16_t *out) {
    if (length <= 0 || rows <= 0) return JL_OK;
    dim3 grid((length + 255) / 256 > 1024 ? 1024 : (length + 255) / 256, rows);
    quantize_bf16_kernel<<<grid, 256, 0, s>>>(x, ldx, offset, length, out);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- fused producers of the BF16 activation operand of the tensor-core prefill GEMMs (jl_model.cu forward_rows_tc) ----------
// RMSNorm (RMSNorm.java:34-56, double sum like rmsnorm_kernel) rounded straight to BF16: no f32 round trip through HBM.
__global__ void rmsnorm_bf16_kernel(const float *x, int ldx, int w_dtype, const void *w, float adj, float eps, int E, uint16_t *out, int ldo) {
    const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ double red[8];
    __shared__ float rs_sh;
    const float *xr = x + (size_t)r * ldx;
    double ss = 0.0;
    for (int i = tid; i < E; i += blockDim.x) {
        const float v = xr[i];
        ss += (double)__fmul_rn(v, v);
    }
    ss = warp_sum_d(ss);
    if (lane == 0) red[warp] = ss;
    __syncthreads();
    if (tid == 0) {
        double t = 0;
        for (int i = 0; i < (int)(blockDim.x >> 5); i++) t += red[i];
        t /= (double)E;
        t += (double)eps;
        rs_sh = (float)(1.0 / sqrt(t));
    }
    __syncthreads();
    const float rsf = rs_sh;
    for (int i = tid; i < E; i += blockDim.x) {
        const float wv = w_dtype == JL_BF16 ? bf16_bits_to_f32(((const uint16_t *)w)[i]) : ((const float *)w)[i];
        out[(size_t)r * ldo + i] = f32_to_bf16_rne(__fmul_rn(__fadd_rn(adj, wv), __fmul_rn(rsf, xr[i])));
    }
}
int jl_launch_rmsnorm_bf16(jl_ctx *ctx, cudaStream_t s, const float *x, int rows, int ldx, int w_dtype, const void *w, float adj, float eps,
                           int E, uint16_t *out, int ldo) {
    if (rows <= 0 || E <= 0) return JL_OK;
    rmsnorm_bf16_kernel<<<rows, 256, 0, s>>>(x, ldx, w_dtype, w, adj, eps, E, out, ldo);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}
// silu(gate) * up (MLPBlock.java:117-141) rounded straight to BF16.  The operand is BF16 anyway (tolerance class of the
// tensor-core path), so the sigmoid uses the f32 exponential instead of the reference's double one.
__global__ void silu_mul_bf16_kernel(const float *gate, const float *up, int ld, int length, uint16_t *out, int ldo) {
    const int r = blockIdx.y;
    const float4 *g4 = (const float4 *)(gate + (size_t)r * ld), *u4 = (const float4 *)(up + (size_t)r * ld);
    uint2 *o2 = (uint2 *)(out + (size_t)r * ldo);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < length / 4; i += gridDim.x * blockDim.x) {
        const float4 g = g4[i], u = u4[i];
        float v[4] = {g.x, g.y, g.z, g.w};
        const float w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int k = 0; k < 4; k++) v[k] = __fmul_rn(__fdividef(v[k], 1.0f + __expf(-v[k])), w[k]);
        o2[i] = make_uint2((uint32_t)f32_to_bf16_rne(v[0]) | ((uint32_t)f32_to_bf16_rne(v[1]) << 16),
                           (uint32_t)f32_to_bf16_rne(v[2]) | ((uint32_t)f32_to_bf16_rne(v[3]) << 16));
    }
}
int jl_launch_silu_mul_bf16(jl_ctx *ctx, cudaStream_t s, const float *gate, const float *up, int rows, int ld, int length, uint16_t *out, int ldo) {
    if (length <= 0 || rows <= 0) return JL_OK;
    if ((length % 4) || (ld % 4) || (ldo % 4)) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "silu_mul_bf16: lengths must be multiples of 4");
    dim3 grid((length / 4 + 255) / 256 > 64 ? 64 : (length / 4 + 255) / 256, rows);
    silu_mul_bf16_kernel<<<grid, 256, 0, s>>>(gate, up, ld, length, out, ldo);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- Q4 weight quantiser (Q4ByteBufferTensor.java:66-120): one warp per block, byte-identical output --------
__global__ void quantize_q4w_kernel(const float *x, long long rows, long long cols, uint8_t *q, float *scales) {
    const int lane = threadIdx.x & 31;
    const long long nblk = cols / 32, total = rows * nblk;
    for (long long w = (long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); w < total;
         w += (long long)gridDim.x * (blockDim.x / 32)) {
        const float v = x[w * 32 + lane];
        // first index holding the largest |v| keeps its sign (strict '>' scan, :74-81)
        float av = fabsf(v);
        float best = av;
        int besti = lane;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
            if (ob > best || (ob == best && oi < besti)) best = ob, besti = oi;
        }
        float maxv = __shfl_sync(0xffffffffu, v, besti);
        if (!(best > 1.401298464e-45f)) maxv = 1.401298464e-45f; // Float.MIN_VALUE initial value survives
        const float scale = __fdiv_rn(maxv, -8.0f);
        const float iscale = scale != 0.0f ? __fdiv_rn(1.0f, scale) : 0.0f;
        int qi = (int)__fadd_rn(__fmul_rn(v, iscale), 8.5f);
        qi = (int)(int8_t)qi;
        if (qi > 15) qi = 15;
        const int hi = __shfl_down_sync(0xffffffffu, qi, 16);
        if (lane < 16) q[w * 16 + lane] = (uint8_t)((qi & 0xFF) | (hi << 4));
        if (lane == 0) scales[w] = scale;
    }
}
int jl_launch_quantize_q4w(jl_ctx *ctx, cudaStream_t s, const float *x, int64_t rows, int64_t cols, uint8_t *q,
                           float *scales) {
    if (cols % 32) return jl_set_error(ctx, JL_ERR_INVALID, "quantize_q4: cols must be a multiple of 32");
    long long total = rows * (cols / 32);
    if (total <= 0) return JL_OK;
    long long blocks = (total + 7) / 8;
    if (blocks > ctx->sm_count * 16) blocks = ctx->sm_count * 16;
    quantize_q4w_kernel<<<(int)blocks, 256, 0, s>>>(x, rows, cols, q, scales);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- Q8 weight quantiser (Q8ByteBufferTensor.java:47-90): max from Float.MIN_VALUE, iscale = 127/max, q = (byte)Math.round(x*iscale)
__global__ void quantize_q8w_kernel(const float *x, long long rows, long long cols, int8_t *q, float *scales) {
    const int lane = threadIdx.x & 31;
    const long long nblk = cols / 32, total = rows * nblk;
    for (long long w = (long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); w < total;
         w += (long long)gridDim.x * (blockDim.x / 32)) {
        float scale;
        q[w * 32 + lane] = q8_block_quantize(x[w * 32 + lane], scale);
        if (lane == 0) scales[w] = scale;
    }
}
int jl_launch_quantize_q8w(jl_ctx *ctx, cudaStream_t s, const float *x, int64_t rows, int64_t cols, int8_t *q, float *scales) {
    if (cols % 32) return jl_set_error(ctx, JL_ERR_INVALID, "quantize_q8_weights: cols must be a multiple of 32");
    long long total = rows * (cols / 32);
    if (total <= 0) return JL_OK;
    long long blocks = (total + 7) / 8;
    if (blocks > ctx->sm_count * 16) blocks = ctx->sm_count * 16;
    quantize_q8w_kernel<<<(int)blocks, 256, 0, s>>>(x, rows, cols, q, scales);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- RMSNorm (RMSNorm.java:34-56): one CTA per row -------------------------------------------------------------
__global__ void rmsnorm_kernel(const float *x, int ldx, int w_dtype, const void *w, float adj, float eps, int E,
                               int offset, int length, float *out) {
    const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ double red[8];
    __shared__ float rs_sh;
    const float *xr = x + (size_t)r * ldx;
    double ss = 0.0;
    for (int i = tid; i < length; i += blockDim.x) {
        const float v = xr[offset + i];
        ss += (double)__fmul_rn(v, v);
    }
    ss = warp_sum_d(ss);
    if (lane == 0) red[warp] = ss;
    __syncthreads();
    if (tid == 0) {
        double t = 0;
        for (int i = 0; i < (int)(blockDim.x >> 5); i++) t += red[i];
        t /= (double)E;
        t += (double)eps;
        rs_sh = (float)(1.0 / sqrt(t));
    }
    __syncthreads();
    const float rsf = rs_sh;
    for (int i = tid; i < length; i += blockDim.x) {
        const int c = offset + i;
        const float wv = w_dtype == JL_BF16 ? bf16_bits_to_f32(((const uint16_t *)w)[c]) : ((const float *)w)[c];
        out[(size_t)r * ldx + c] = __fmul_rn(__fadd_rn(adj, wv), __fmul_rn(rsf, xr[c]));
    }
}
int jl_launch_rmsnorm(jl_ctx *ctx, cudaStream_t s, const float *x, int rows, int ldx, int w_dtype, const void *w, float adj,
                      float eps, int E, int offset, int length, float *out) {
    if (rows <= 0 || length <= 0) return JL_OK;
    rmsnorm_kernel<<<rows, 256, 0, s>>>(x, ldx, w_dtype, w, adj, eps, E, offset, length, out);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- LayerNorm (model/LayerNorm.java:41-67, GPT-2 family): mean and E[x^2] over [offset, offset+length) divided by
// embeddingLength, variance = E[x^2] - mean^2, invStddev = 1 / (float)sqrt(variance + eps), out = (x - mean) * invStddev * w + b.
// The reference accumulates sum and sumSq sequentially in float; here the float products are summed in double and rounded to
// float once (closer to the exact sums than either order; 1e-6-level differences, the tests' tolerance says so).
__global__ void layernorm_kernel(const float *x, int ldx, int w_dtype, const void *w, int b_dtype, const void *bias, float eps, int E,
                                 int offset, int length, float *out) {
    const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ double red[2][8];
    __shared__ float stat[2];
    const float *xr = x + (size_t)r * ldx;
    double s = 0.0, ss = 0.0;
    for (int i = tid; i < length; i += blockDim.x) {
        const float v = xr[offset + i];
        s += (double)v;
        ss += (double)__fmul_rn(v, v);
    }
    s = warp_sum_d(s), ss = warp_sum_d(ss);
    if (lane == 0) red[0][warp] = s, red[1][warp] = ss;
    __syncthreads();
    if (tid == 0) {
        double a = 0, b = 0;
        for (int i = 0; i < (int)(blockDim.x >> 5); i++) a += red[0][i], b += red[1][i];
        const float sum = (float)a, sumSq = (float)b;
        const float mean = __fdiv_rn(sum, (float)E);
        const float variance = __fsub_rn(__fdiv_rn(sumSq, (float)E), __fmul_rn(mean, mean));
        stat[0] = mean;
        stat[1] = __fdiv_rn(1.0f, (float)sqrt((double)__fadd_rn(variance, eps)));
    }
    __syncthreads();
    const float mean = stat[0], inv = stat[1];
    for (int i = tid; i < length; i += blockDim.x) {
        const int c = offset + i;
        const float wv = w_dtype == JL_BF16 ? bf16_bits_to_f32(((const uint16_t *)w)[c]) : ((const float *)w)[c];
        const float bv = b_dtype == JL_BF16 ? bf16_bits_to_f32(((const uint16_t *)bias)[c]) : ((const float *)bias)[c];
        out[(size_t)r * ldx + c] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(xr[c], mean), inv), wv), bv);
    }
}
int jl_launch_layernorm(jl_ctx *ctx, cudaStream_t s, const float *x, int rows, int ldx, int w_dtype, const void *w, int b_dtype,
                        const void *bias, float eps, int E, int offset, int length, float *out) {
    if (rows <= 0 || length <= 0) return JL_OK;
    layernorm_kernel<<<rows, 256, 0, s>>>(x, ldx, w_dtype, w, b_dtype, bias, eps, E, offset, length, out);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- ActivationFunction.eval (math/ActivationFunction.java:29-37) in place: 0 SILU, 1 GELU / GELU_PYTORCH_TANH, 2 TANH; double math
__global__ void activation_kernel(int type, float *x, int rows, int ld, int offset, int length) {
    const long long n = (long long)rows * length;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float *p = x + (size_t)(i / length) * ld + offset + (i % length);
        const float v = *p;
        float o;
        if (type == 0) o = silu_ref(v);
        else if (type == 1) o = (float)(0.5 * (double)v * (1.0 + tanh(sqrt(2.0 / 3.14159265358979323846) * ((double)v + 0.044715 * pow((double)v, 3.0)))));
        else o = (float)tanh((double)v);
        *p = o;
    }
}
int jl_launch_activation(jl_ctx *ctx, cudaStream_t s, int type, float *x, int rows, int ld, int offset, int length) {
    if (rows <= 0 || length <= 0) return JL_OK;
    long long n = (long long)rows * length;
    int blocks = (int)((n + 255) / 256);
    if (blocks > ctx->sm_count * 8) blocks = ctx->sm_count * 8;
    activation_kernel<<<blocks, 256, 0, s>>>(type, x, rows, ld, offset, length);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- MoE router (MoEBlock.java:90-92,151-168): one warp per row; at most 64 experts ----------------------------------------
__global__ void moe_route_kernel(float *logits, int n_experts, int k, int32_t *sel) {
    const int row = blockIdx.x, lane = threadIdx.x;
    float *x = logits + (size_t)row * n_experts;
    // VectorMath.softMax (:69-90): max, (float)exp((double)(x - max)), float sum in index order, divide
    float v0 = lane < n_experts ? x[lane] : -INFINITY, v1 = lane + 32 < n_experts ? x[lane + 32] : -INFINITY;
    const float mx = warp_max(fmaxf(v0, v1));
    const float e0 = lane < n_experts ? (float)exp((double)__fsub_rn(v0, mx)) : 0.0f;
    const float e1 = lane + 32 < n_experts ? (float)exp((double)__fsub_rn(v1, mx)) : 0.0f;
    __shared__ float pe[64];
    pe[lane] = e0, pe[lane + 32] = e1;
    __syncwarp();
    if (lane == 0) {
        float sum = 0.0f;
        for (int i = 0; i < n_experts; i++) sum = __fadd_rn(sum, pe[i]);
        for (int i = 0; i < n_experts; i++) pe[i] = __fdiv_rn(pe[i], sum), x[i] = pe[i];
        // topk: the first k experts, then every later expert replaces the current minimum if it is larger (strict)
        int s[64];
        for (int i = 0; i < k; i++) s[i] = i;
        for (int i = k; i < n_experts; i++) {
            int mn = 0;
            for (int j = 1; j < k; j++)
                if (pe[s[j]] < pe[s[mn]]) mn = j;
            if (pe[i] > pe[s[mn]]) s[mn] = i;
        }
        for (int i = 0; i < k; i++) sel[(size_t)row * k + i] = s[i];
    }
}
int jl_launch_moe_route(jl_ctx *ctx, cudaStream_t s, float *logits, int rows, int n_experts, int k, int32_t *sel) {
    if (rows <= 0) return JL_OK;
    if (n_experts < 1 || n_experts > 64 || k < 1 || k > n_experts) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "moe_route: %d experts / top-%d", n_experts, k);
    moe_route_kernel<<<rows, 32, 0, s>>>(logits, n_experts, k, sel);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// HOST-buffer entry point for crafted router rows
extern "C" int jl_moe_route(jl_ctx *ctx, int n, int n_experts, int k, const float *logits, float *probs_out, int32_t *sel_out) {
    if (!ctx) return JL_ERR_INVALID;
    if (n < 1 || n_experts < 1 || n_experts > 64 || k < 1 || k > n_experts || !logits || !probs_out || !sel_out)
        return jl_set_error(ctx, JL_ERR_INVALID, "moe_route: bad arguments (n=%d, experts=%d, k=%d)", n, n_experts, k);
    std::lock_guard<std::mutex> lk(ctx->mu);
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    const size_t lb = (size_t)n * n_experts * 4, sb = (size_t)n * k * 4;
    float *dl = (float *)jl_scratch(ctx, 0, lb);
    int32_t *ds = (int32_t *)jl_scratch(ctx, 1, sb);
    if (!dl || !ds) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dl, logits, lb, cudaMemcpyHostToDevice, ctx->stream));
    const int rc = jl_launch_moe_route(ctx, ctx->stream, dl, n, n_experts, k, ds);
    if (rc != JL_OK) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(probs_out, dl, lb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(sel_out, ds, sb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

// ---- MoE grouping: a stable counting sort of a step's (row, slot) pairs by expert, and the tile table of the grouped expert GEMM --
// One CTA of 1024 threads.  The scatter walks the pairs in chunks of 1024: a pair's place is its expert's running offset, plus the
// pairs of that expert in earlier warps of the chunk, plus those in earlier lanes of its own warp (__match_any_sync), so the order
// within an expert is the pair order whatever the warps' timing.
#define MOE_GROUP_THREADS 1024
__global__ void __launch_bounds__(MOE_GROUP_THREADS) moe_group_kernel(const int32_t *sel, int n, int n_experts, int R, MoeGroups g) {
    __shared__ int cnt[64], run[64], tile0[65];
    __shared__ int wc[MOE_GROUP_THREADS / 32][64];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 64) cnt[tid] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += MOE_GROUP_THREADS) atomicAdd(&cnt[sel[i]], 1);
    __syncthreads();
    if (tid == 0) {
        int o = 0, t = 0;
        for (int e = 0; e < n_experts; e++) {
            run[e] = o, tile0[e] = t;
            o += cnt[e], t += (cnt[e] + R - 1) / R;
        }
        tile0[n_experts] = t;
        *g.ntiles = t;
    }
    __syncthreads();
    if (tid < n_experts) {
        const int e = tid, c = cnt[e], o = run[e];
        g.counts[e] = c, g.offsets[e] = o;
        for (int f = 0, t = tile0[e]; f < c; f += R, t++) g.tiles[t] = make_int4(e, o + f, c - f < R ? c - f : R, 0);
    }
    for (int c0 = 0; c0 < n; c0 += MOE_GROUP_THREADS) {
        const int i = c0 + tid;
        const bool live = i < n;
        const int e = live ? sel[i] : -1;
        for (int j = tid; j < (MOE_GROUP_THREADS / 32) * 64; j += MOE_GROUP_THREADS) wc[j >> 6][j & 63] = 0;
        __syncthreads();
        const unsigned peers = __match_any_sync(0xffffffffu, e);
        const int rank = __popc(peers & ((1u << lane) - 1u));
        if (live && rank == 0) wc[warp][e] = __popc(peers);
        __syncthreads();
        if (tid < n_experts) { // the warps' counts -> their first places, warp by warp
            int s = run[tid];
            for (int w = 0; w < MOE_GROUP_THREADS / 32; w++) {
                const int v = wc[w][tid];
                wc[w][tid] = s, s += v;
            }
            run[tid] = s;
        }
        __syncthreads();
        if (live) g.pairs[wc[warp][e] + rank] = i;
        __syncthreads();
    }
}
int jl_launch_moe_group(jl_ctx *ctx, cudaStream_t s, const int32_t *sel, int rows, int n_experts, int k, int R, const MoeGroups &g) {
    if (rows < 1 || n_experts < 1 || n_experts > 64 || k < 1 || k > 8 || k > n_experts || R < 1)
        return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "moe_group: %d rows, %d experts / top-%d, tiles of %d", rows, n_experts, k, R);
    moe_group_kernel<<<1, MOE_GROUP_THREADS, 0, s>>>(sel, rows * k, n_experts, R, g);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// HOST-buffer entry point for crafted selections
extern "C" int jl_moe_group(jl_ctx *ctx, int n, int n_experts, int k, int R, const int32_t *sel, int32_t *counts_out,
                            int32_t *offsets_out, int32_t *pairs_out, int32_t *tiles_out, int32_t *ntiles_out) {
    if (!ctx) return JL_ERR_INVALID;
    if (n < 1 || n_experts < 1 || n_experts > 64 || k < 1 || k > 8 || k > n_experts || R < 1 || R > 64 || !sel || !counts_out ||
        !offsets_out || !pairs_out || !tiles_out || !ntiles_out)
        return jl_set_error(ctx, JL_ERR_INVALID, "moe_group: bad arguments (n=%d, experts=%d, k=%d, R=%d)", n, n_experts, k, R);
    const size_t np = (size_t)n * k;
    if (np > (size_t)1 << 24) return jl_set_error(ctx, JL_ERR_INVALID, "moe_group: %zu pairs", np);
    for (size_t i = 0; i < np; i++)
        if (sel[i] < 0 || sel[i] >= n_experts) return jl_set_error(ctx, JL_ERR_INVALID, "moe_group: selection %zu is %d", i, sel[i]);
    std::lock_guard<std::mutex> lk(ctx->mu);
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    const int bound = jl_moe_tile_bound((int)np, n_experts, R);
    const size_t sb = np * 4, cb = (size_t)n_experts * 4, tb = (size_t)bound * sizeof(int4);
    int32_t *ds = (int32_t *)jl_scratch(ctx, 0, sb);
    char *dout = (char *)jl_scratch(ctx, 1, 2 * cb + sb + tb + 16);
    if (!ds || !dout) return JL_ERR_OOM;
    MoeGroups g;
    g.tiles = (int4 *)dout, g.pairs = (int32_t *)(dout + tb), g.counts = (int32_t *)(dout + tb + sb);
    g.offsets = g.counts + n_experts, g.ntiles = g.offsets + n_experts;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(ds, sel, sb, cudaMemcpyHostToDevice, ctx->stream));
    const int rc = jl_launch_moe_group(ctx, ctx->stream, ds, n, n_experts, k, R, g);
    if (rc != JL_OK) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(ntiles_out, g.ntiles, 4, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(counts_out, g.counts, cb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(offsets_out, g.offsets, cb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(pairs_out, g.pairs, sb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    const int nt = *ntiles_out < bound ? *ntiles_out : bound;
    JL_CUDA_CHECK(ctx, cudaMemcpy(tiles_out, g.tiles, (size_t)nt * sizeof(int4), cudaMemcpyDeviceToHost));
    return JL_OK;
}

// ---- MoE combine: the expert outputs of each row summed in slot order, then the residual (the per-row loop's add chain) --------
__global__ void moe_combine_kernel(const float4 *d, int rows, int k, int E4, const float4 *xb, float4 *x) {
    const long long n = (long long)rows * E4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / E4, c = i - b * E4;
        float4 t = d[(size_t)b * k * E4 + c];
        for (int s = 1; s < k; s++) {
            const float4 v = d[((size_t)b * k + s) * E4 + c];
            t = make_float4(__fadd_rn(v.x, t.x), __fadd_rn(v.y, t.y), __fadd_rn(v.z, t.z), __fadd_rn(v.w, t.w));
        }
        const float4 r = xb[i];
        x[i] = make_float4(__fadd_rn(t.x, r.x), __fadd_rn(t.y, r.y), __fadd_rn(t.z, r.z), __fadd_rn(t.w, r.w));
    }
}
int jl_launch_moe_combine(jl_ctx *ctx, cudaStream_t s, const float *d, int rows, int k, int E, const float *xb, float *x) {
    if (rows <= 0) return JL_OK;
    if (E % 4) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "moe_combine: E=%d", E);
    const long long n = (long long)rows * (E / 4);
    long long blocks = (n + 255) / 256;
    if (blocks > ctx->sm_count * 8) blocks = ctx->sm_count * 8;
    moe_combine_kernel<<<(int)blocks, 256, 0, s>>>((const float4 *)d, rows, k, E / 4, (const float4 *)xb, (float4 *)x);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- softmax (VectorMath.java:69-90), single row, one CTA ---------------------------------------------------------
__global__ void softmax_kernel(float *x, int offset, int length) {
    __shared__ float red[32];
    __shared__ float bc;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    float mx = -INFINITY;
    for (int i = tid; i < length; i += blockDim.x) mx = fmaxf(mx, x[offset + i]);
    mx = warp_max(mx);
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    if (tid == 0) {
        float t = red[0];
        for (int i = 1; i < nw; i++) t = fmaxf(t, red[i]);
        bc = t;
    }
    __syncthreads();
    mx = bc;
    float sum = 0.0f;
    for (int i = tid; i < length; i += blockDim.x) {
        const float e = (float)exp((double)__fsub_rn(x[offset + i], mx));
        x[offset + i] = e;
        sum += e;
    }
    sum = warp_sum(sum);
    __syncthreads();
    if (lane == 0) red[warp] = sum;
    __syncthreads();
    if (tid == 0) {
        float t = 0;
        for (int i = 0; i < nw; i++) t += red[i];
        bc = t;
    }
    __syncthreads();
    sum = bc;
    // the reference's normalisation loop starts at index 0, not `offset` (:87)
    for (int i = tid; i < offset + length; i += blockDim.x) x[i] = __fdiv_rn(x[i], sum);
}
int jl_launch_softmax(jl_ctx *ctx, cudaStream_t s, float *x, int offset, int length) {
    if (length <= 0) return JL_OK;
    softmax_kernel<<<1, 1024, 0, s>>>(x, offset, length);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- gate = silu(gate) * up  (MLPBlock.java:132-141) -----------------------------------------------------------------
__global__ void silu_mul_kernel(float *gate, const float *up, int ld, int offset, int length) {
    const int r = blockIdx.y;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < length; i += gridDim.x * blockDim.x) {
        const size_t idx = (size_t)r * ld + offset + i;
        gate[idx] = __fmul_rn(silu_ref(gate[idx]), up[idx]);
    }
}
int jl_launch_silu_mul(jl_ctx *ctx, cudaStream_t s, float *gate, const float *up, int rows, int ld, int offset, int length) {
    if (length <= 0 || rows <= 0) return JL_OK;
    dim3 grid((length + 255) / 256 > 2048 ? 2048 : (length + 255) / 256, rows);
    silu_mul_kernel<<<grid, 256, 0, s>>>(gate, up, ld, offset, length);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- learned position embeddings (GPT2Model.java:54-69): x[r, :] = wte row (already there) + wpe[position[r], :] ----------------
__global__ void pos_embed_add_kernel(float *x, int E, int dtype, const void *wpe, const int32_t *positions) {
    const int r = blockIdx.y;
    const size_t pos = (size_t)positions[r];
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < E; c += gridDim.x * blockDim.x) {
        const float v = dtype == JL_BF16 ? bf16_bits_to_f32(((const uint16_t *)wpe)[pos * E + c]) : ((const float *)wpe)[pos * E + c];
        x[(size_t)r * E + c] = __fadd_rn(x[(size_t)r * E + c], v);
    }
}
int jl_launch_pos_embed_add(jl_ctx *ctx, cudaStream_t s, float *x, int rows, int E, const DevTensor &wpe, const int32_t *positions) {
    if (rows <= 0) return JL_OK;
    dim3 grid((E + 255) / 256, rows);
    pos_embed_add_kernel<<<grid, 256, 0, s>>>(x, E, wpe.dtype, wpe.data, positions);
    ctx->launches++;
    JL_CUDA_CHECK(ctx, cudaGetLastError());
    return JL_OK;
}

// ---- embedding rows -> f32 (LlamaModel.java:68-100; Q4 rows are consumed through get(), Q4ByteBufferTensor.java:179-197)
__global__ void embed_kernel(int dtype, const void *w, const float *scales, const int32_t *tokens, float *out, int E) {
    const int r = blockIdx.y;
    const size_t tok = (size_t)tokens[r];
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < E; c += gridDim.x * blockDim.x) {
        float v;
        if (dtype == JL_F32) v = ((const float *)w)[tok * E + c];
        else if (dtype == JL_BF16) v = bf16_bits_to_f32(((const uint16_t *)w)[tok * E + c]);
        else if (dtype == JL_Q4) {
            const int blk = c / 32, in = c % 32;
            const uint8_t byte = ((const uint8_t *)w)[(tok * E + blk * 32) / 2 + (in & 15)];
            const int nib = in < 16 ? (byte & 0x0F) : (byte >> 4);
            v = __fmul_rn((float)(nib - 8), scales[tok * (E / 32) + blk]);
        } else {
            v = __fmul_rn((float)((const int8_t *)w)[tok * E + c], scales[tok * (E / 32) + c / 32]);
        }
        out[(size_t)r * E + c] = v;
    }
}
int jl_launch_embed(jl_ctx *ctx, cudaStream_t s, const DevTensor &wte, const int32_t *tokens, int n, float *out, int E) {
    if (n <= 0) return JL_OK;
    dim3 grid((E + 255) / 256, n);
    JL_CUDA_CHECK(ctx, jl_launch_kernel(embed_kernel, grid, dim3(256), 0, s, wte.dtype, (const void *)wte.data,
                                        (const float *)wte.scales, tokens, out, E));
    ctx->launches++;
    return JL_OK;
}

// ---- arg-max with strict '>' (lowest index wins; AbstractModel.java:455-469) ----------------------------------------------
struct ArgPair {
    float v;
    int i;
};
__device__ __forceinline__ bool arg_better(float v, int i, float bv, int bi) {
    // NaN never wins ('v > maxv' is false), ties keep the lower index
    return (v > bv) || (v == bv && i < bi);
}
#define ARGMAX_BLOCKS 64
__global__ void argmax_stage1(const float *logits, int vocab, int ld, ArgPair *part) {
    const int r = blockIdx.y;
    const float *x = logits + (size_t)r * ld;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < vocab; i += gridDim.x * blockDim.x) {
        const float v = x[i];
        if (arg_better(v, i, bv, bi)) bv = v, bi = i;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (arg_better(ov, oi, bv, bi)) bv = ov, bi = oi;
    }
    __shared__ ArgPair sm[8];
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = {bv, bi};
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); w++)
            if (arg_better(sm[w].v, sm[w].i, bv, bi)) bv = sm[w].v, bi = sm[w].i;
        part[r * ARGMAX_BLOCKS + blockIdx.x] = {bv, bi};
    }
}
__global__ void argmax_stage2(const ArgPair *part, int32_t *out) {
    const int r = blockIdx.x;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < ARGMAX_BLOCKS; i += 32) {
        const ArgPair p = part[r * ARGMAX_BLOCKS + i];
        if (arg_better(p.v, p.i, bv, bi)) bv = p.v, bi = p.i;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (arg_better(ov, oi, bv, bi)) bv = ov, bi = oi;
    }
    // all -inf / NaN logits: the reference returns Integer.MIN_VALUE's initial maxi; we return 0
    if (threadIdx.x == 0) out[r] = bi == 0x7fffffff ? 0 : bi;
}
size_t jl_argmax_scratch_bytes(int rows) { return (size_t)rows * ARGMAX_BLOCKS * sizeof(ArgPair); }
int jl_launch_argmax(jl_ctx *ctx, cudaStream_t s, const float *logits, int rows, int vocab, int ld, int32_t *out_tokens,
                     void *scratch) {
    if (rows <= 0) return JL_OK;
    JL_CUDA_CHECK(ctx, jl_launch_kernel(argmax_stage1, dim3(ARGMAX_BLOCKS, rows), dim3(256), 0, s, logits, vocab, ld,
                                        (ArgPair *)scratch));
    JL_CUDA_CHECK(ctx, jl_launch_kernel(argmax_stage2, dim3(rows), dim3(32), 0, s, (const ArgPair *)scratch, out_tokens));
    ctx->launches += 2;
    return JL_OK;
}
