// Context, tensor registry and the TensorOperations-granular C ABI on HOST buffers
// (the literal drop-in for NativeGPUTensorOperations -> gpu_gemm, vector_gpu.h:7-19).
#include "jl_common.cuh"

#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

// Error text is kept per calling thread (errno style): op-level calls fail under ctx->mu, model-level calls under their model's lock,
// request threads and a scheduler thread may fail at the same time -- one shared std::string would be written concurrently and the
// pointer jl_last_error hands out could be freed under its reader.  The context also keeps the latest message of any thread for a
// caller that asks from a thread which has not failed itself.
static thread_local std::string g_thread_error = "";

int jl_set_error(jl_ctx *ctx, int code, const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_thread_error = buf;
    if (ctx) {
        std::lock_guard<std::mutex> lk(ctx->err_mu);
        ctx->last_error = buf;
    }
    return code;
}

extern "C" const char *jl_version(void) { return "jlama_b200 0.1 (sm_90a)"; }

extern "C" const char *jl_last_error(jl_ctx *ctx) {
    if (g_thread_error.empty() && ctx) {
        std::lock_guard<std::mutex> lk(ctx->err_mu);
        g_thread_error = ctx->last_error; // a copy this thread owns: valid until its next failing call
    }
    return g_thread_error.c_str();
}

extern "C" int jl_init(int device, jl_ctx **out, int64_t *info) {
    if (!out) return JL_ERR_INVALID;
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0)
        return jl_set_error(nullptr, JL_ERR_CUDA, "no CUDA device: %s (there is no CPU fallback)", cudaGetErrorString(e));
    if (device < 0 || device >= count) return jl_set_error(nullptr, JL_ERR_INVALID, "device %d out of range", device);
    cudaDeviceProp prop;
    if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess)
        return jl_set_error(nullptr, JL_ERR_CUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0)
        return jl_set_error(nullptr, JL_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a only", device,
                            prop.major, prop.minor);
    if ((e = cudaSetDevice(device)) != cudaSuccess)
        return jl_set_error(nullptr, JL_ERR_CUDA, "cudaSetDevice: %s", cudaGetErrorString(e));
    jl_ctx *ctx = new jl_ctx();
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    if ((e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess) {
        delete ctx;
        return jl_set_error(nullptr, JL_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e));
    }
    if (info) {
        size_t fr = 0, tot = 0;
        cudaMemGetInfo(&fr, &tot);
        info[0] = (int64_t)fr;
        info[1] = (int64_t)tot;
        info[2] = prop.multiProcessorCount;
        info[3] = prop.major * 10 + prop.minor;
    }
    *out = ctx;
    return JL_OK;
}

extern "C" int jl_comm_destroy(jl_ctx *ctx);

extern "C" int jl_shutdown(jl_ctx *ctx) {
    if (!ctx) return JL_ERR_INVALID;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    while (!ctx->models.empty()) jl_model_free(ctx->models.back()); // models first: their graphs point at the tensors
    jl_comm_destroy(ctx);
    for (auto &kv : ctx->tensors) {
        cudaFree(kv.second.data);
        if (kv.second.scales) cudaFree(kv.second.scales);
    }
    for (int i = 0; i < 4; i++)
        if (ctx->scratch[i]) cudaFree(ctx->scratch[i]);
    cudaStreamDestroy(ctx->stream);
    delete ctx;
    return JL_OK;
}

extern "C" int jl_sync(jl_ctx *ctx) {
    if (!ctx) return JL_ERR_INVALID;
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    JL_CUDA_CHECK(ctx, cudaDeviceSynchronize());
    return JL_OK;
}

extern "C" int64_t jl_kernel_launches(jl_ctx *ctx) { return ctx ? ctx->launches : -1; }

void *jl_scratch(jl_ctx *ctx, int slot, size_t bytes) {
    if (bytes <= ctx->scratch_bytes[slot]) return ctx->scratch[slot];
    if (ctx->scratch[slot]) {
        cudaStreamSynchronize(ctx->stream);
        cudaFree(ctx->scratch[slot]);
        ctx->scratch[slot] = nullptr;
        ctx->scratch_bytes[slot] = 0;
    }
    size_t want = bytes + bytes / 4 + 4096;
    if (cudaMalloc(&ctx->scratch[slot], want) != cudaSuccess) {
        cudaGetLastError();
        jl_set_error(ctx, JL_ERR_OOM, "out of device memory allocating %zu scratch bytes", want);
        return nullptr;
    }
    ctx->scratch_bytes[slot] = want;
    return ctx->scratch[slot];
}

static size_t dtype_row_bytes(int dtype, int64_t cols) {
    switch (dtype) {
        case JL_F32: return (size_t)cols * 4;
        case JL_BF16: return (size_t)cols * 2;
        case JL_Q4: return (size_t)cols / 2;
        case JL_I8: return (size_t)cols;
    }
    return 0;
}

extern "C" int64_t jl_register_tensor(jl_ctx *ctx, int dtype, int64_t rows, int64_t cols, const void *data,
                                      const float *scales) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    cudaSetDevice(ctx->device);
    if (!data || rows <= 0 || cols <= 0 || dtype < JL_F32 || dtype > JL_I8) {
        jl_set_error(ctx, JL_ERR_INVALID, "register_tensor: bad arguments");
        return -1;
    }
    const bool quant = dtype == JL_Q4 || dtype == JL_I8;
    if (quant && (!scales || (cols % 32))) {
        jl_set_error(ctx, JL_ERR_INVALID, "register_tensor: quantised tensors need scales and cols %% 32 == 0");
        return -1;
    }
    DevTensor t;
    t.dtype = dtype;
    t.rows = rows;
    t.cols = cols;
    t.bytes = dtype_row_bytes(dtype, cols) * (size_t)rows;
    // +64 bytes of slack: the GEMV loads whole 16-byte blocks
    if (cudaMalloc(&t.data, t.bytes + 64) != cudaSuccess) {
        cudaGetLastError();
        jl_set_error(ctx, JL_ERR_OOM, "register_tensor: out of device memory (%zu bytes)", t.bytes);
        return -1;
    }
    if (cudaMemcpy(t.data, data, t.bytes, cudaMemcpyHostToDevice) != cudaSuccess) {
        jl_set_error(ctx, JL_ERR_CUDA, "register_tensor: upload failed: %s", cudaGetErrorString(cudaGetLastError()));
        cudaFree(t.data);
        return -1;
    }
    if (quant) {
        size_t sb = (size_t)rows * (cols / 32) * 4;
        if (cudaMalloc((void **)&t.scales, sb + 64) != cudaSuccess) {
            cudaGetLastError();
            cudaFree(t.data);
            jl_set_error(ctx, JL_ERR_OOM, "register_tensor: out of device memory (scales)");
            return -1;
        }
        if (cudaMemcpy(t.scales, scales, sb, cudaMemcpyHostToDevice) != cudaSuccess) {
            jl_set_error(ctx, JL_ERR_CUDA, "register_tensor: scale upload failed");
            cudaFree(t.data);
            cudaFree(t.scales);
            return -1;
        }
        t.bytes += sb;
    }
    int64_t id = ctx->next_id++;
    t.id = id;
    ctx->tensors[id] = t;
    return id;
}

extern "C" int jl_unregister_tensor(jl_ctx *ctx, int64_t id) {
    if (!ctx) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->mu);
    auto it = ctx->tensors.find(id);
    if (it == ctx->tensors.end()) return jl_set_error(ctx, JL_ERR_INVALID, "unknown tensor id %lld", (long long)id);
    if (it->second.refs > 0)
        return jl_set_error(ctx, JL_ERR_INVALID, "tensor %lld is bound to %d live model slot(s); free the model first", (long long)id,
                            it->second.refs);
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize(); // model streams may still be reading it
    cudaFree(it->second.data);
    if (it->second.scales) cudaFree(it->second.scales);
    ctx->tensors.erase(it);
    return JL_OK;
}

// ---- batchDotProduct on host buffers ----------------------------------------------------------------
static int gemm_locked(jl_ctx *ctx, int a_dtype, const void *a, const float *a_scales, int a_col_off, int lda,
                       const DevTensor &B, int b_col_off, float *r, int roffset, int m, int n0, int n, int k, int ldc) {
    if (m <= 0 || n <= 0 || k <= 0) return JL_OK;
    if (!a || !r) return jl_set_error(ctx, JL_ERR_INVALID, "gemm: null buffer");
    if (n0 < 0 || n0 + n > B.rows || b_col_off < 0 || b_col_off + k > B.cols || a_col_off < 0 || a_col_off + k > lda)
        return jl_set_error(ctx, JL_ERR_INVALID, "gemm: slice out of range (n0=%d n=%d k=%d rows=%lld cols=%lld)", n0, n, k,
                            (long long)B.rows, (long long)B.cols);
    const bool bq = B.dtype == JL_Q4 || B.dtype == JL_I8;
    // supported (A,B) pairs mirror PanamaTensorOperations.java:118-143 plus I8 weights
    if (a_dtype == JL_I8 && !bq) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "gemm: I8 activations need Q4/I8 weights");
    if (a_dtype == JL_I8 && !a_scales) return jl_set_error(ctx, JL_ERR_INVALID, "gemm: I8 activations need scales");
    if (a_dtype != JL_F32 && a_dtype != JL_BF16 && a_dtype != JL_I8)
        return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "gemm: activation dtype %d", a_dtype);
    if (bq && ((k % 32) || (b_col_off % 32) || (a_dtype == JL_I8 && (a_col_off % 32))))
        return jl_set_error(ctx, JL_ERR_INVALID, "gemm: quantised operands need 32-aligned offsets/length");
    // an I8 row's scales are its lda / 32 block scales: a row stride that is not whole blocks has no scale layout
    if (a_dtype == JL_I8 && (lda % 32)) return jl_set_error(ctx, JL_ERR_INVALID, "gemm: I8 activations need lda %% 32 == 0 (lda=%d)", lda);
    // the output row slice written by this call: columns [n0-roffset, n0-roffset+n)
    const int c0 = n0 - roffset;
    if (c0 < 0 || c0 + n > ldc) return jl_set_error(ctx, JL_ERR_INVALID, "gemm: result offset out of range");

    // Only the k columns each row uses are uploaded, packed at a row stride of k rounded up to 32 elements: the kernels load
    // activations 16 bytes at a time, so every row must start 16-byte aligned whatever the caller's column offset and row stride.
    const size_t esz = a_dtype == JL_F32 ? 4 : (a_dtype == JL_BF16 ? 2 : 1);
    const int kp = (k + 31) & ~31;
    void *da = jl_scratch(ctx, 0, (size_t)m * kp * esz);
    float *dr = (float *)jl_scratch(ctx, 1, (size_t)m * n * 4);
    float *das = nullptr;
    if (!da || !dr) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpy2DAsync(da, (size_t)kp * esz, (const char *)a + (size_t)a_col_off * esz, (size_t)lda * esz,
                                         (size_t)k * esz, m, cudaMemcpyHostToDevice, ctx->stream));
    if (a_dtype == JL_I8) {
        das = (float *)jl_scratch(ctx, 2, (size_t)m * (kp / 32) * 4);
        if (!das) return JL_ERR_OOM;
        JL_CUDA_CHECK(ctx, cudaMemcpy2DAsync(das, (size_t)(kp / 32) * 4, a_scales + a_col_off / 32, (size_t)(lda / 32) * 4,
                                             (size_t)(k / 32) * 4, m, cudaMemcpyHostToDevice, ctx->stream));
    }
    const int pro = a_dtype == JL_I8 ? PRO_Q8_GLOBAL : (a_dtype == JL_BF16 ? PRO_BF16_GLOBAL : PRO_F32);
    const int chunk = jl_gemv_max_m(B.dtype, pro, k);
    if (chunk < 1) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "gemm: k=%d does not fit shared memory", k);
    for (int m0 = 0; m0 < m; m0 += chunk) {
        const int mc = m - m0 < chunk ? m - m0 : chunk;
        GemvParams p = {};
        p.nseg = 1;
        p.seg[0].w = B.data;
        p.seg[0].ws = B.scales;
        p.seg[0].out = dr + (size_t)m0 * n;
        p.seg[0].rows = n;
        p.seg[0].out_ld = n;
        p.seg[0].out_off = -n0;
        p.w_dtype = B.dtype;
        p.ldw = (int)B.cols;
        p.w_col_off = b_col_off;
        p.K = k;
        p.M = mc;
        p.a = (const char *)da + (size_t)m0 * kp * esz;
        p.a_scales = das ? das + (size_t)m0 * (kp / 32) : nullptr;
        p.lda = kp;
        p.a_col_off = 0;
        p.row0 = n0;
        p.total_rows = n;
        int rc = jl_launch_gemv(ctx, ctx->stream, p, pro, EPI_STORE);
        if (rc != JL_OK) return rc;
    }
    JL_CUDA_CHECK(ctx, cudaMemcpy2DAsync(r + c0, (size_t)ldc * 4, dr, (size_t)n * 4, (size_t)n * 4, m, cudaMemcpyDeviceToHost,
                                        ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

extern "C" int jl_gemm(jl_ctx *ctx, int a_dtype, const void *a, const float *a_scales, int a_col_off, int lda, int64_t b_id,
                       int b_col_off, float *r, int roffset, int m, int n0, int n, int k, int ldc) {
    if (!ctx) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->mu);
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    auto it = ctx->tensors.find(b_id);
    if (it == ctx->tensors.end()) return jl_set_error(ctx, JL_ERR_INVALID, "gemm: unknown tensor id %lld", (long long)b_id);
    return gemm_locked(ctx, a_dtype, a, a_scales, a_col_off, lda, it->second, b_col_off, r, roffset, m, n0, n, k, ldc);
}

extern "C" int jl_gemm_tc(jl_ctx *ctx, int a_dtype, const void *a, int a_col_off, int lda, int64_t b_id, int b_col_off, float *r,
                          int roffset, int m, int n0, int n, int k, int ldc) {
    if (!ctx) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->mu);
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    auto it = ctx->tensors.find(b_id);
    if (it == ctx->tensors.end()) return jl_set_error(ctx, JL_ERR_INVALID, "gemm_tc: unknown tensor id %lld", (long long)b_id);
    const DevTensor &B = it->second;
    if (m <= 0 || n <= 0 || k <= 0) return JL_OK;
    if (!a || !r) return jl_set_error(ctx, JL_ERR_INVALID, "gemm_tc: null buffer");
    if (a_dtype != JL_F32 && a_dtype != JL_BF16) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "gemm_tc: activations must be F32 or BF16");
    if (n0 < 0 || n0 + n > B.rows || b_col_off < 0 || b_col_off + k > B.cols || a_col_off < 0 || a_col_off + k > lda)
        return jl_set_error(ctx, JL_ERR_INVALID, "gemm_tc: slice out of range");
    if ((n0 % 128) || (a_col_off % 8) || (lda % 8)) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "gemm_tc: n0 %% 128, a_col_off %% 8, lda %% 8 required");
    const int c0 = n0 - roffset;
    if (c0 < 0 || c0 + n > ldc) return jl_set_error(ctx, JL_ERR_INVALID, "gemm_tc: result offset out of range");
    const size_t a_elems = (size_t)m * lda;
    uint16_t *dab = (uint16_t *)jl_scratch(ctx, 0, a_elems * 2);
    float *dr = (float *)jl_scratch(ctx, 1, (size_t)m * n * 4);
    if (!dab || !dr) return JL_ERR_OOM;
    if (a_dtype == JL_F32) {
        float *daf = (float *)jl_scratch(ctx, 2, a_elems * 4);
        if (!daf) return JL_ERR_OOM;
        JL_CUDA_CHECK(ctx, cudaMemcpyAsync(daf, a, a_elems * 4, cudaMemcpyHostToDevice, ctx->stream));
        int rc = jl_launch_quantize_bf16(ctx, ctx->stream, daf, m, lda, 0, lda, dab); // FloatConversions.float32ToBFloat16 (RNE)
        if (rc) return rc;
    } else {
        JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dab, a, a_elems * 2, cudaMemcpyHostToDevice, ctx->stream));
    }
    // view of B starting at row n0: the kernel indexes weight rows from 0 (row pitch cols/2 bytes for Q4, cols for Q8_0)
    DevTensor Bv = B;
    Bv.data = (uint8_t *)B.data + (size_t)n0 * dtype_row_bytes(B.dtype, B.cols);
    Bv.scales = B.scales + (size_t)n0 * (B.cols / 32);
    int rc = jl_launch_gemm_tc(ctx, ctx->stream, dab + a_col_off, lda, m, Bv, n, b_col_off, k, dr, n, 0, nullptr, 0);
    if (rc) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpy2DAsync(r + c0, (size_t)ldc * 4, dr, (size_t)n * 4, (size_t)n * 4, m, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

extern "C" int jl_gemm_batch(jl_ctx *ctx, int batch_num, int a_dtype, const void *a, const float *a_scales, int a_col_off,
                             int lda, const int64_t *b_ids, int b_col_off, float *const *r, int roffset, int m, int n0, int n,
                             int k, int ldc) {
    if (!ctx || !b_ids || !r) return JL_ERR_INVALID;
    for (int i = 0; i < batch_num; i++) {
        int rc = jl_gemm(ctx, a_dtype, a, a_scales, a_col_off, lda, b_ids[i], b_col_off, r[i], roffset, m, n0, n, k, ldc);
        if (rc != JL_OK) return rc;
    }
    return JL_OK;
}

extern "C" int jl_gemm_host(jl_ctx *ctx, int a_dtype, const void *a, int a_col_off, int lda, int b_dtype, const void *b,
                            int b_col_off, int ldb, float *r, int roffset, int m, int n0, int n, int k, int ldc) {
    if (!ctx) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->mu);
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    if (b_dtype != JL_F32 && b_dtype != JL_BF16) return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "gemm_host: B must be F32/BF16");
    if (!b || n <= 0) return n <= 0 ? JL_OK : jl_set_error(ctx, JL_ERR_INVALID, "gemm_host: null B");
    if (n0 < 0 || ldb <= 0) return jl_set_error(ctx, JL_ERR_INVALID, "gemm_host: negative row offset / row stride");
    const size_t esz = b_dtype == JL_F32 ? 4 : 2;
    // upload only the rows used
    DevTensor B;
    B.dtype = b_dtype;
    B.rows = n;
    B.cols = ldb;
    B.data = jl_scratch(ctx, 3, (size_t)n * ldb * esz);
    if (!B.data) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(B.data, (const char *)b + (size_t)n0 * ldb * esz, (size_t)n * ldb * esz,
                                       cudaMemcpyHostToDevice, ctx->stream));
    // rows are now [0,n): shift roffset accordingly so the output index stays j - roffset
    return gemm_locked(ctx, a_dtype, a, nullptr, a_col_off, lda, B, b_col_off, r, roffset - n0, m, 0, n, k, ldc);
}

// ---- element-wise ops on host buffers -----------------------------------------------------------------
#define HOST_OP_PROLOGUE()                              \
    if (!ctx) return JL_ERR_INVALID;                    \
    std::lock_guard<std::mutex> lk(ctx->mu);            \
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));

extern "C" int jl_accumulate(jl_ctx *ctx, float *a, int a_rows, int lda, int b_dtype, const void *b, const float *b_scales,
                             int b_rows, int ldb, int offset, int length) {
    HOST_OP_PROLOGUE();
    if (!a || !b || a_rows < 0 || length < 0 || offset < 0 || (int64_t)offset + length > lda || (int64_t)offset + length > ldb)
        return jl_set_error(ctx, JL_ERR_INVALID, "accumulate: bad arguments");
    if (a_rows == 0 || length == 0) return JL_OK;
    if (b_rows != 1 && b_rows != a_rows) return jl_set_error(ctx, JL_ERR_INVALID, "accumulate: b must have 1 or a_rows rows");
    if (b_dtype != JL_F32 && b_dtype != JL_BF16 && b_dtype != JL_Q4)
        return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "accumulate: b dtype %d", b_dtype);
    if (b_dtype == JL_Q4 && (!b_scales || (ldb % 32))) return jl_set_error(ctx, JL_ERR_INVALID, "accumulate: Q4 needs scales");
    const size_t ab = (size_t)a_rows * lda * 4, bb = dtype_row_bytes(b_dtype, ldb) * b_rows;
    float *da = (float *)jl_scratch(ctx, 0, ab);
    void *db = jl_scratch(ctx, 1, bb);
    float *dbs = nullptr;
    if (!da || !db) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(da, a, ab, cudaMemcpyHostToDevice, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(db, b, bb, cudaMemcpyHostToDevice, ctx->stream));
    if (b_dtype == JL_Q4) {
        dbs = (float *)jl_scratch(ctx, 2, (size_t)b_rows * (ldb / 32) * 4);
        if (!dbs) return JL_ERR_OOM;
        JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dbs, b_scales, (size_t)b_rows * (ldb / 32) * 4, cudaMemcpyHostToDevice, ctx->stream));
    }
    int rc = jl_launch_accumulate(ctx, ctx->stream, da, a_rows, lda, b_dtype, db, dbs, b_rows, ldb, offset, length);
    if (rc) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(a, da, ab, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

extern "C" int jl_maccumulate(jl_ctx *ctx, float *a, int a_rows, int lda, const float *b, int b_rows, int ldb, int offset,
                              int length) {
    HOST_OP_PROLOGUE();
    if (!a || !b || a_rows < 0 || length < 0 || offset < 0 || (int64_t)offset + length > lda || (int64_t)offset + length > ldb ||
        (b_rows != 1 && b_rows != a_rows))
        return jl_set_error(ctx, JL_ERR_INVALID, "maccumulate: bad arguments");
    if (a_rows == 0 || length == 0) return JL_OK;
    const size_t ab = (size_t)a_rows * lda * 4, bb = (size_t)b_rows * ldb * 4;
    float *da = (float *)jl_scratch(ctx, 0, ab), *db = (float *)jl_scratch(ctx, 1, bb);
    if (!da || !db) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(da, a, ab, cudaMemcpyHostToDevice, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(db, b, bb, cudaMemcpyHostToDevice, ctx->stream));
    int rc = jl_launch_maccumulate(ctx, ctx->stream, da, a_rows, lda, db, b_rows, ldb, offset, length);
    if (rc) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(a, da, ab, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

extern "C" int jl_scale(jl_ctx *ctx, float factor, float *x, int rows, int ldx, int offset, int length) {
    HOST_OP_PROLOGUE();
    if (!x || rows < 0 || length < 0 || offset < 0 || (int64_t)offset + length > ldx) return jl_set_error(ctx, JL_ERR_INVALID, "scale: bad arguments");
    if (rows == 0 || length == 0) return JL_OK;
    const size_t xb = (size_t)rows * ldx * 4;
    float *dx = (float *)jl_scratch(ctx, 0, xb);
    if (!dx) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dx, x, xb, cudaMemcpyHostToDevice, ctx->stream));
    int rc = jl_launch_scale(ctx, ctx->stream, factor, dx, rows, ldx, offset, length);
    if (rc) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(x, dx, xb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

extern "C" int jl_saxpy_batch(jl_ctx *ctx, const float *alpha, const float *x, int ldx, float *y, int xoffset, int yoffset,
                              int limit, int a_offset, int x_row_offset, int batch) {
    HOST_OP_PROLOGUE();
    if (!alpha || !x || !y || limit < 0 || batch < 0 || xoffset < 0 || yoffset < 0 || a_offset < 0 || x_row_offset < 0 ||
        (int64_t)xoffset + limit > ldx)
        return jl_set_error(ctx, JL_ERR_INVALID, "saxpy: bad arguments");
    if (limit == 0 || batch == 0) return JL_OK;
    float *da = (float *)jl_scratch(ctx, 0, (size_t)batch * 4);
    float *dx = (float *)jl_scratch(ctx, 1, (size_t)batch * ldx * 4);
    float *dy = (float *)jl_scratch(ctx, 2, (size_t)limit * 4);
    if (!da || !dx || !dy) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(da, alpha + a_offset, (size_t)batch * 4, cudaMemcpyHostToDevice, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dx, x + (size_t)x_row_offset * ldx, (size_t)batch * ldx * 4, cudaMemcpyHostToDevice,
                                       ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dy, y + yoffset, (size_t)limit * 4, cudaMemcpyHostToDevice, ctx->stream));
    int rc = jl_launch_saxpy_batch(ctx, ctx->stream, da, dx, ldx, dy, xoffset, 0, limit, 0, 0, batch);
    if (rc) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(y + yoffset, dy, (size_t)limit * 4, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

extern "C" int jl_saxpy(jl_ctx *ctx, float alpha, const float *x, float *y, int xoffset, int yoffset, int limit) {
    if (!x) return JL_ERR_INVALID;
    // one-row batch: y += alpha * x
    return jl_saxpy_batch(ctx, &alpha, x, xoffset + limit, y, xoffset, yoffset, limit, 0, 0, 1);
}

extern "C" int jl_quantize_q8(jl_ctx *ctx, const float *x, int rows, int ldx, int offset, int length, int8_t *q,
                              float *scales) {
    HOST_OP_PROLOGUE();
    if (!x || !q || !scales || rows < 0 || length < 0 || offset < 0 || (int64_t)offset + length > ldx)
        return jl_set_error(ctx, JL_ERR_INVALID, "quantize_q8: bad arguments");
    if (rows == 0) return JL_OK;
    const size_t xb = (size_t)rows * ldx * 4, qb = (size_t)rows * ldx, sb = (size_t)rows * (ldx / 32) * 4;
    float *dx = (float *)jl_scratch(ctx, 0, xb);
    int8_t *dq = (int8_t *)jl_scratch(ctx, 1, qb);
    float *ds = (float *)jl_scratch(ctx, 2, sb);
    if (!dx || !dq || !ds) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dx, x, xb, cudaMemcpyHostToDevice, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemsetAsync(dq, 0, qb, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemsetAsync(ds, 0, sb, ctx->stream));
    int rc = jl_launch_quantize_q8(ctx, ctx->stream, dx, rows, ldx, offset, length, dq, ds);
    if (rc) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(q, dq, qb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(scales, ds, sb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

extern "C" int jl_quantize_bf16(jl_ctx *ctx, const float *x, int rows, int ldx, int offset, int length, uint16_t *out) {
    HOST_OP_PROLOGUE();
    if (!x || !out || rows < 0 || length < 0 || offset < 0 || (int64_t)offset + length > ldx)
        return jl_set_error(ctx, JL_ERR_INVALID, "quantize_bf16: bad arguments");
    if (rows == 0) return JL_OK;
    const size_t xb = (size_t)rows * ldx * 4, ob = (size_t)rows * ldx * 2;
    float *dx = (float *)jl_scratch(ctx, 0, xb);
    uint16_t *dout = (uint16_t *)jl_scratch(ctx, 1, ob);
    if (!dx || !dout) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dx, x, xb, cudaMemcpyHostToDevice, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemsetAsync(dout, 0, ob, ctx->stream));
    int rc = jl_launch_quantize_bf16(ctx, ctx->stream, dx, rows, ldx, offset, length, dout);
    if (rc) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(out, dout, ob, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

extern "C" int jl_quantize_q4_weights(jl_ctx *ctx, const float *x, int64_t rows, int64_t cols, uint8_t *q, float *scales) {
    HOST_OP_PROLOGUE();
    if (!x || !q || !scales || rows <= 0 || cols <= 0 || (cols % 32))
        return jl_set_error(ctx, JL_ERR_INVALID, "quantize_q4: bad arguments (cols must be a multiple of the 32-element block)");
    const size_t xb = (size_t)rows * cols * 4, qb = (size_t)rows * cols / 2, sb = (size_t)rows * (cols / 32) * 4;
    float *dx = (float *)jl_scratch(ctx, 0, xb);
    uint8_t *dq = (uint8_t *)jl_scratch(ctx, 1, qb);
    float *ds = (float *)jl_scratch(ctx, 2, sb);
    if (!dx || !dq || !ds) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dx, x, xb, cudaMemcpyHostToDevice, ctx->stream));
    int rc = jl_launch_quantize_q4w(ctx, ctx->stream, dx, rows, cols, dq, ds);
    if (rc) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(q, dq, qb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(scales, ds, sb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

extern "C" int jl_layernorm(jl_ctx *ctx, const float *x, int rows, int ldx, int w_dtype, const void *w, int b_dtype, const void *bias, float eps,
                            int embedding_length, int offset, int length, float *out) {
    HOST_OP_PROLOGUE();
    if (!x || !w || !bias || !out || rows < 0 || length < 0 || offset < 0 || (int64_t)offset + length > ldx ||
        (w_dtype != JL_F32 && w_dtype != JL_BF16) || (b_dtype != JL_F32 && b_dtype != JL_BF16))
        return jl_set_error(ctx, JL_ERR_INVALID, "layernorm: bad arguments");
    if (rows == 0 || length == 0) return JL_OK;
    const size_t xb = (size_t)rows * ldx * 4, n = (size_t)(offset + length);
    const size_t wb = n * (w_dtype == JL_F32 ? 4 : 2), bb = n * (b_dtype == JL_F32 ? 4 : 2);
    float *dx = (float *)jl_scratch(ctx, 0, xb);
    float *dout = (float *)jl_scratch(ctx, 1, xb);
    char *dw = (char *)jl_scratch(ctx, 2, wb + bb + 32);
    if (!dx || !dout || !dw) return JL_ERR_OOM;
    char *dbias = dw + ((wb + 15) & ~(size_t)15);
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dx, x, xb, cudaMemcpyHostToDevice, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dout, out, xb, cudaMemcpyHostToDevice, ctx->stream)); // columns outside the slice keep their values
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dw, w, wb, cudaMemcpyHostToDevice, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dbias, bias, bb, cudaMemcpyHostToDevice, ctx->stream));
    int rc = jl_launch_layernorm(ctx, ctx->stream, dx, rows, ldx, w_dtype, dw, b_dtype, dbias, eps, embedding_length, offset, length, dout);
    if (rc) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(out, dout, xb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

extern "C" int jl_activation(jl_ctx *ctx, int type, float *x, int rows, int ld, int offset, int length) {
    HOST_OP_PROLOGUE();
    if (!x || type < 0 || type > 2 || rows < 0 || length < 0 || offset < 0 || (int64_t)offset + length > ld)
        return jl_set_error(ctx, JL_ERR_INVALID, "activation: bad arguments");
    if (rows == 0 || length == 0) return JL_OK;
    const size_t xb = (size_t)rows * ld * 4;
    float *dx = (float *)jl_scratch(ctx, 0, xb);
    if (!dx) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dx, x, xb, cudaMemcpyHostToDevice, ctx->stream));
    int rc = jl_launch_activation(ctx, ctx->stream, type, dx, rows, ld, offset, length);
    if (rc) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(x, dx, xb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

extern "C" int jl_quantize_q8_weights(jl_ctx *ctx, const float *x, int64_t rows, int64_t cols, int8_t *q, float *scales) {
    HOST_OP_PROLOGUE();
    if (!x || !q || !scales || rows <= 0 || cols <= 0 || (cols % 32))
        return jl_set_error(ctx, JL_ERR_INVALID, "quantize_q8_weights: bad arguments (cols must be a multiple of the 32-element block)");
    const size_t xb = (size_t)rows * cols * 4, qb = (size_t)rows * cols, sb = (size_t)rows * (cols / 32) * 4;
    float *dx = (float *)jl_scratch(ctx, 0, xb);
    int8_t *dq = (int8_t *)jl_scratch(ctx, 1, qb);
    float *ds = (float *)jl_scratch(ctx, 2, sb);
    if (!dx || !dq || !ds) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dx, x, xb, cudaMemcpyHostToDevice, ctx->stream));
    int rc = jl_launch_quantize_q8w(ctx, ctx->stream, dx, rows, cols, dq, ds);
    if (rc) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(q, dq, qb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(scales, ds, sb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

extern "C" int jl_rmsnorm(jl_ctx *ctx, const float *x, int rows, int ldx, int w_dtype, const void *w, float weight_adjustment,
                          float eps, int embedding_length, int offset, int length, float *out) {
    HOST_OP_PROLOGUE();
    if (!x || !w || !out || rows < 0 || length < 0 || offset < 0 || (int64_t)offset + length > ldx || (w_dtype != JL_F32 && w_dtype != JL_BF16))
        return jl_set_error(ctx, JL_ERR_INVALID, "rmsnorm: bad arguments");
    if (rows == 0) return JL_OK;
    const size_t xb = (size_t)rows * ldx * 4, wb = (size_t)(offset + length) * (w_dtype == JL_F32 ? 4 : 2);
    float *dx = (float *)jl_scratch(ctx, 0, xb);
    void *dw = jl_scratch(ctx, 1, wb);
    float *dout = (float *)jl_scratch(ctx, 2, xb);
    if (!dx || !dw || !dout) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dx, x, xb, cudaMemcpyHostToDevice, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dw, w, wb, cudaMemcpyHostToDevice, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemsetAsync(dout, 0, xb, ctx->stream));
    int rc = jl_launch_rmsnorm(ctx, ctx->stream, dx, rows, ldx, w_dtype, dw, weight_adjustment, eps, embedding_length, offset,
                               length, dout);
    if (rc) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(out, dout, xb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

extern "C" int jl_softmax(jl_ctx *ctx, float *x, int offset, int length) {
    HOST_OP_PROLOGUE();
    if (!x || offset < 0 || length <= 0) return jl_set_error(ctx, JL_ERR_INVALID, "softmax: bad arguments");
    const size_t xb = (size_t)(offset + length) * 4;
    float *dx = (float *)jl_scratch(ctx, 0, xb);
    if (!dx) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dx, x, xb, cudaMemcpyHostToDevice, ctx->stream));
    int rc = jl_launch_softmax(ctx, ctx->stream, dx, offset, length);
    if (rc) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(x, dx, xb, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

extern "C" int jl_silu_mul(jl_ctx *ctx, float *gate, const float *up, int rows, int ld, int offset, int length) {
    HOST_OP_PROLOGUE();
    if (!gate || !up || rows < 0 || length < 0 || offset < 0 || (int64_t)offset + length > ld)
        return jl_set_error(ctx, JL_ERR_INVALID, "silu_mul: bad arguments");
    if (rows == 0 || length == 0) return JL_OK;
    const size_t b = (size_t)rows * ld * 4;
    float *dg = (float *)jl_scratch(ctx, 0, b), *du = (float *)jl_scratch(ctx, 1, b);
    if (!dg || !du) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(dg, gate, b, cudaMemcpyHostToDevice, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(du, up, b, cudaMemcpyHostToDevice, ctx->stream));
    int rc = jl_launch_silu_mul(ctx, ctx->stream, dg, du, rows, ld, offset, length);
    if (rc) return rc;
    JL_CUDA_CHECK(ctx, cudaMemcpyAsync(gate, dg, b, cudaMemcpyDeviceToHost, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    return JL_OK;
}

// ---- pure host logic ---------------------------------------------------------------------------------------
// VectorMath.precomputeFreqsCis (core/math/VectorMath.java:148-165)
extern "C" int jl_precompute_freqs_cis(int dim, int end, double theta, double scaling_factor, float *out) {
    if (dim <= 0 || (dim & 1) || end <= 0 || !out) return JL_ERR_INVALID;
    const int half = dim / 2;
    std::vector<float> freqs(half);
    float step = 0.0f;
    for (int i = 0; i < half; i++, step += 2.0f) freqs[i] = (float)((1.0 / pow(theta, (double)(step / dim))) / scaling_factor);
    for (int64_t p = 0; p < end; p++) {
        const float t = (float)p;
        for (int i = 0; i < half; i++) {
            volatile float ang = t * freqs[i];
            out[(p * half + i) * 2 + 0] = (float)cos((double)ang);
            out[(p * half + i) * 2 + 1] = (float)sin((double)ang);
        }
    }
    return JL_OK;
}

// DistributedContext (core/model/DistributedContext.java:60-98)
extern "C" int jl_dctx_build(int E, int attention_length, int H, int head_size, int head_group_size, int num_layers,
                             int model_shard, int num_model_shards, int layer_shard, int num_layer_shards, jl_dctx *d) {
    if (!d || num_model_shards <= 0 || num_layer_shards <= 0 || model_shard < 0 || model_shard >= num_model_shards ||
        layer_shard < 0 || layer_shard >= num_layer_shards || head_size <= 0 || head_group_size <= 0)
        return JL_ERR_INVALID;
    d->numberOfLayers = num_layers / num_layer_shards;
    d->layerStart = d->numberOfLayers * layer_shard;
    d->layerEnd = d->layerStart + d->numberOfLayers;
    d->embeddingSegmentLength = E / num_model_shards;
    d->embeddingSegmentStart = d->embeddingSegmentLength * model_shard;
    d->attentionSegmentLength = attention_length / num_model_shards;
    d->attentionSegmentStart = d->attentionSegmentLength * model_shard;
    d->hiddenSegmentLength = H / num_model_shards;
    d->hiddenSegmentStart = d->hiddenSegmentLength * model_shard;
    d->kvSegmentStart = d->attentionSegmentStart / head_group_size;
    d->kvSegmentLength = d->attentionSegmentLength / head_group_size;
    const int embEnd = d->embeddingSegmentStart + d->embeddingSegmentLength;
    d->headStart = d->embeddingSegmentStart / head_size;
    d->headEnd = embEnd / head_size;
    d->groupHeadStart = d->kvSegmentStart / head_size;
    d->groupHeadEnd = (d->kvSegmentStart + d->kvSegmentLength) / head_size;
    return JL_OK;
}

// KvBufferCache.computePageSize (core/tensor/KvBufferCache.java:224-280)
extern "C" int jl_kv_page_geometry(int num_layers, int context_length, int kv_segment_length, int dtype_size,
                                   int64_t max_page_bytes, int *layers_per_page, int *ctx_per_page) {
    if (!layers_per_page || !ctx_per_page || num_layers <= 0 || context_length <= 0 || kv_segment_length <= 0 || dtype_size <= 0)
        return JL_ERR_INVALID; // a zero element size would divide by zero below
    const int64_t s = 2LL * dtype_size * kv_segment_length;
    if (max_page_bytes <= s) return JL_ERR_INVALID; // Preconditions.checkArgument(:229)
    int optL = 1, optC = 1;
    int64_t maxProduct = 0;
    for (int x = num_layers; x >= 1; x--) {
        const int64_t y = max_page_bytes / (x * s);
        if (y >= 1 && y <= context_length) {
            const int64_t product = x * y;
            if (product > maxProduct) {
                optL = x;
                optC = (int)y;
                maxProduct = product;
            }
            if (product < maxProduct) break;
        }
    }
    *layers_per_page = optL;
    *ctx_per_page = optC;
    return JL_OK;
}

// ---- diagnostic micro-benchmark of the GEMV kernel ----------------------------------------------------------
extern "C" int jl_debug_gemv_bench(jl_ctx *ctx, int64_t b_id, int n, int m, int mode, int iters, double *avg_us) {
    HOST_OP_PROLOGUE();
    auto it = ctx->tensors.find(b_id);
    if (it == ctx->tensors.end() || !avg_us || iters <= 0 || m < 1 || m > JL_MAX_DECODE_ROWS)
        return jl_set_error(ctx, JL_ERR_INVALID, "gemv_bench: bad arguments");
    const DevTensor &B = it->second;
    if (n <= 0 || n > B.rows) return jl_set_error(ctx, JL_ERR_INVALID, "gemv_bench: n out of range");
    const int k = (int)B.cols;
    float *da = (float *)jl_scratch(ctx, 0, (size_t)m * k * 4);
    float *dr = (float *)jl_scratch(ctx, 1, (size_t)m * B.rows * 4);
    float *dw = (float *)jl_scratch(ctx, 2, (size_t)k * 4);
    if (!da || !dr || !dw) return JL_ERR_OOM;
    // m > GEMV_MAX_M: the many-row decode GEMM, with its workspaces (activations | partial tiles | counters) in one buffer
    const size_t act_b = (jl_gemm64_act_bytes(k) + 255) & ~(size_t)255, part_b = jl_gemm64_part_floats(ctx->sm_count) * 4;
    char *wide = m > GEMV_MAX_M ? (char *)jl_scratch(ctx, 3, act_b + part_b + (size_t)ctx->sm_count * 4) : nullptr;
    if (m > GEMV_MAX_M && !wide) return JL_ERR_OOM;
    if (wide) JL_CUDA_CHECK(ctx, cudaMemset(wide + act_b + part_b, 0, (size_t)ctx->sm_count * 4));
    std::vector<float> ha((size_t)m * k), hw(k, 1.0f);
    for (size_t i = 0; i < ha.size(); i++) ha[i] = (float)((int)(i * 2654435761u % 2001) - 1000) / 500.0f;
    JL_CUDA_CHECK(ctx, cudaMemcpy(da, ha.data(), ha.size() * 4, cudaMemcpyHostToDevice));
    JL_CUDA_CHECK(ctx, cudaMemcpy(dw, hw.data(), hw.size() * 4, cudaMemcpyHostToDevice));
    JL_CUDA_CHECK(ctx, cudaMemset(dr, 0, (size_t)m * B.rows * 4));
    cudaEvent_t e0, e1;
    JL_CUDA_CHECK(ctx, cudaEventCreate(&e0));
    JL_CUDA_CHECK(ctx, cudaEventCreate(&e1));
    const int slots = (int)(B.rows / n);
    for (int pass = 0; pass < 2; pass++) { // pass 0 = warm-up
        if (pass == 1) JL_CUDA_CHECK(ctx, cudaEventRecord(e0, ctx->stream));
        for (int i = 0; i < (pass == 0 ? (iters < 8 ? iters : 8) : iters); i++) {
            GemvParams p = {};
            p.nseg = 1;
            p.seg[0].w = B.data;
            p.seg[0].ws = B.scales;
            p.seg[0].out = dr;
            p.seg[0].rows = n;
            p.seg[0].out_ld = (int)B.rows;
            p.seg[0].out_off = 0;
            p.w_dtype = B.dtype;
            p.ldw = k;
            p.K = k;
            p.M = m;
            p.a = da;
            p.lda = k;
            p.row0 = (i % slots) * n;
            p.total_rows = n;
            p.norm_w = dw;
            p.norm_w_dtype = JL_F32;
            p.norm_eps = 1e-5f;
            p.norm_E = k;
            p.residual = dr;
            p.res_ld = (int)B.rows;
            if (wide) p.wide_act = wide, p.wide_part = (float *)(wide + act_b), p.wide_cnt = (unsigned *)(wide + act_b + part_b);
            const int pro = mode == 1 ? PRO_RMSNORM_QUANT : (mode == 2 ? PRO_F32 : PRO_F32_QUANT);
            if (m > GEMV_MAX_M && !jl_gemm64_supported(p, pro, mode == 3 ? EPI_ADD_RESIDUAL : EPI_STORE))
                return jl_set_error(ctx, JL_ERR_UNSUPPORTED, "gemv_bench: m=%d needs Q4 / Q8_0 weights", m);
            int rc = jl_launch_gemv(ctx, ctx->stream, p, pro, mode == 3 ? EPI_ADD_RESIDUAL : EPI_STORE);
            if (rc) return rc;
        }
    }
    JL_CUDA_CHECK(ctx, cudaEventRecord(e1, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    *avg_us = (double)ms * 1000.0 / iters;
    return JL_OK;
}

extern "C" int jl_debug_gemm_tc_bench(jl_ctx *ctx, int64_t b_id, int t, int iters, double *avg_us) {
    HOST_OP_PROLOGUE();
    auto it = ctx->tensors.find(b_id);
    if (it == ctx->tensors.end() || !avg_us || iters <= 0 || t <= 0) return jl_set_error(ctx, JL_ERR_INVALID, "gemm_tc_bench: bad arguments");
    const DevTensor &B = it->second;
    const int k = (int)B.cols, n = (int)B.rows;
    uint16_t *da = (uint16_t *)jl_scratch(ctx, 0, (size_t)t * k * 2);
    float *dr = (float *)jl_scratch(ctx, 1, (size_t)t * n * 4);
    if (!da || !dr) return JL_ERR_OOM;
    JL_CUDA_CHECK(ctx, cudaMemsetAsync(da, 0x3c, (size_t)t * k * 2, ctx->stream)); // bf16 ~0.0115
    cudaEvent_t e0, e1;
    JL_CUDA_CHECK(ctx, cudaEventCreate(&e0));
    JL_CUDA_CHECK(ctx, cudaEventCreate(&e1));
    for (int pass = 0; pass < 2; pass++) {
        if (pass == 1) JL_CUDA_CHECK(ctx, cudaEventRecord(e0, ctx->stream));
        for (int i = 0; i < (pass == 0 ? 3 : iters); i++) {
            int rc = jl_launch_gemm_tc(ctx, ctx->stream, da, k, t, B, n, 0, k, dr, n, 0, nullptr, 0);
            if (rc) return rc;
        }
    }
    JL_CUDA_CHECK(ctx, cudaEventRecord(e1, ctx->stream));
    JL_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    *avg_us = (double)ms * 1000.0 / iters;
    return JL_OK;
}

// ---- kernel timeline diagnostics ---------------------------------------------------------------------------------------
// capacity > 0: allocate [capacity][4] stamps and hand one slot to every traced launch from now on (graphs captured
// afterwards keep their slots, every replay re-stamps them); capacity == 0: stop tracing.
extern "C" int jl_debug_ktrace(jl_ctx *ctx, int capacity) {
    if (!ctx || capacity < 0) return JL_ERR_INVALID;
    std::lock_guard<std::mutex> lk(ctx->mu);
    JL_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
    JL_CUDA_CHECK(ctx, cudaDeviceSynchronize());
    jl_models_invalidate_graphs(ctx); // captured graphs carry the old slot pointers in their kernel parameters
    if (ctx->ktrace) cudaFree(ctx->ktrace);
    ctx->ktrace = nullptr, ctx->ktrace_cap = 0, ctx->ktrace_n = 0;
    if (capacity == 0) return JL_OK;
    JL_CUDA_CHECK(ctx, cudaMalloc(&ctx->ktrace, (size_t)capacity * KTRACE_WORDS * 8));
    ctx->ktrace_cap = capacity;
    return jl_debug_ktrace_clear(ctx);
}
static __global__ void ktrace_clear_kernel(unsigned long long *t, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        t[(size_t)KTRACE_WORDS * i] = ~0ull;
        for (int j = 1; j < KTRACE_WORDS; j++) t[(size_t)KTRACE_WORDS * i + j] = 0;
    }
}
extern "C" int jl_debug_ktrace_clear(jl_ctx *ctx) {
    if (!ctx || !ctx->ktrace) return JL_ERR_INVALID;
    JL_CUDA_CHECK(ctx, cudaDeviceSynchronize());
    ktrace_clear_kernel<<<(ctx->ktrace_cap + 255) / 256, 256>>>(ctx->ktrace, ctx->ktrace_cap);
    JL_CUDA_CHECK(ctx, cudaDeviceSynchronize());
    return JL_OK;
}
// copies min(slots handed out, max_slots) * 16 words to `out`; returns the number of slots, or < 0
extern "C" int jl_debug_ktrace_read(jl_ctx *ctx, uint64_t *out, int max_slots) {
    if (!ctx || !ctx->ktrace || !out) return JL_ERR_INVALID;
    const int n = ctx->ktrace_n < max_slots ? ctx->ktrace_n : max_slots;
    if (cudaDeviceSynchronize() != cudaSuccess) return JL_ERR_CUDA;
    if (n > 0 && cudaMemcpy(out, ctx->ktrace, (size_t)n * KTRACE_WORDS * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return JL_ERR_CUDA;
    return n;
}
