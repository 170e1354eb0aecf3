// device.cu -- device object, stream, activation pool, buffers, LUT upload.
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include "common.cuh"

static std::string g_create_error;

int cc_fail(cc_device* dev, int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (dev) dev->last_error = buf; else g_create_error = buf;
    return code;
}

// ---- type facts (crabml-core/src/gguf.rs:86-108; block sizes SURVEY Appendix A) ------------------
int cc_block_elems(int t) {
    switch (t) {
    case CC_F32: case CC_F16: return 1;
    case CC_Q4_0: case CC_Q4_1: case CC_Q5_0: case CC_Q5_1: case CC_Q8_0: case CC_Q8_1: return 32;
    case CC_Q2_K: case CC_Q3_K: case CC_Q4_K: case CC_Q5_K: case CC_Q6_K: case CC_Q8_K: return 256;
    }
    return 0;
}
size_t cc_block_bytes(int t) {
    switch (t) {
    case CC_F32: return 4; case CC_F16: return 2;
    case CC_Q4_0: return 18; case CC_Q4_1: return 20; case CC_Q5_0: return 22; case CC_Q5_1: return 24;
    case CC_Q8_0: return 34; case CC_Q8_1: return 36;
    case CC_Q2_K: return 84; case CC_Q3_K: return 110; case CC_Q4_K: return 144; case CC_Q5_K: return 176;
    case CC_Q6_K: return 210; case CC_Q8_K: return 292;
    }
    return 0;
}
int cc_partner_type(int t) {   // buf/api.rs:142-159
    switch (t) {
    case CC_F32: return CC_F32; case CC_F16: return CC_F16;
    case CC_Q8_0: case CC_Q4_0: case CC_Q5_0: return CC_Q8_0;
    case CC_Q8_1: case CC_Q4_1: case CC_Q5_1: return CC_Q8_1;
    case CC_Q2_K: case CC_Q3_K: case CC_Q4_K: case CC_Q5_K: case CC_Q6_K: case CC_Q8_K: return CC_Q8_K;
    }
    return -1;
}
bool cc_is_quant(int t) { return cc_block_elems(t) > 1; }

// ---- LUTs (cpu_device.rs:108-124): computed with the HOST libm, exactly as the reference does ---
static float h2f_host(uint16_t h) { return __half2float(__ushort_as_half(h)); }
static uint16_t f2h_host(float f) { return __half_as_ushort(__float2half_rn(f)); }
static float gelu_single(float x) {   // gelu.rs:17-21
    const float COEF_A = 0.044715f;
    const float SQRT_2_OVER_PI = (float)0.7978845608028654;
    return 0.5f * x * (1.0f + tanhf(SQRT_2_OVER_PI * x * (1.0f + COEF_A * x * x)));
}

extern "C" CC_API int cc_device_create(const cc_device_options* opts, cc_device** out) {
    if (!out) return cc_fail(nullptr, CC_ERR_ARG, "cc_device_create: out is NULL");
    *out = nullptr;
    int ord = opts ? opts->device_ordinal : 0;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0)
        return cc_fail(nullptr, CC_ERR_CUDA, "no CUDA device available (%s); crabml-cuda has no CPU fallback",
                       e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    if (ord < 0 || ord >= count) return cc_fail(nullptr, CC_ERR_ARG, "device ordinal %d out of range (%d devices)", ord, count);
    cc_device* dev = new cc_device();
    dev->ordinal = ord;
    dev->debug_named_tensors = opts && opts->debug_named_tensors;
    dev->lazy = opts && opts->lazy;
    dev->exact = opts && opts->exact_order;
    dev->mega = opts && opts->lazy >= 2;
#define CREATE_CUDA(call)                                                                          \
    do { cudaError_t _e = (call); if (_e != cudaSuccess) { cc_fail(nullptr, CC_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(_e)); delete dev; return CC_ERR_CUDA; } } while (0)
    CREATE_CUDA(cudaSetDevice(ord));
    cudaDeviceProp prop;
    CREATE_CUDA(cudaGetDeviceProperties(&prop, ord));
    dev->sm_count = prop.multiProcessorCount;
    CREATE_CUDA(cudaStreamCreateWithFlags(&dev->stream, cudaStreamNonBlocking));
    std::vector<uint16_t> lut(65536);
    for (uint32_t x = 0; x < 65536; x++) lut[x] = f2h_host(expf(h2f_host((uint16_t)x)));
    CREATE_CUDA(cudaMalloc(&dev->exp_lut, 65536 * 2));
    CREATE_CUDA(cudaMemcpy(dev->exp_lut, lut.data(), 65536 * 2, cudaMemcpyHostToDevice));
    for (uint32_t x = 0; x < 65536; x++) lut[x] = f2h_host(gelu_single(h2f_host((uint16_t)x)));
    CREATE_CUDA(cudaMalloc(&dev->gelu_lut, 65536 * 2));
    CREATE_CUDA(cudaMemcpy(dev->gelu_lut, lut.data(), 65536 * 2, cudaMemcpyHostToDevice));
    CREATE_CUDA(cudaHostAlloc((void**)&dev->err_host, 64, cudaHostAllocMapped));
    *dev->err_host = 0u;
    CREATE_CUDA(cudaMalloc((void**)&dev->err_dev, 256));
    CREATE_CUDA(cudaMemset(dev->err_dev, 0, 256));
#undef CREATE_CUDA
    // scratch buffers are sized once for every realistic row (k up to 1M elements): growing them later means cudaFree, which waits
    // for EVERY kernel of the context -- with several devices of one process on one GPU (in-process ranks) a peer may be spinning
    // on this rank's exchange at that moment
    if (cc_ensure_act_scratch(dev, (size_t)4 << 20) != CC_OK || cc_ensure_dev_idx(dev, (size_t)64 << 10) != CC_OK) {
        delete dev;
        return CC_ERR_CUDA;
    }
    if (dev->lazy && !dev->exact) {
        dev->lz = cc_lazy_create(dev);
        if (!dev->lz) { cc_fail(nullptr, CC_ERR_CUDA, "lazy mode: could not allocate the dynamic-argument buffers"); delete dev; return CC_ERR_CUDA; }
    }
    *out = dev;
    return CC_OK;
}

extern "C" CC_API void cc_device_destroy(cc_device* dev) {
    if (!dev) return;
    cudaSetDevice(dev->ordinal);
    cudaStreamSynchronize(dev->stream);
    cc_lazy_destroy(dev);
    cc_comm_destroy(dev);
    cc_prefill_release(dev);
    for (auto& kv : dev->free_lists)
        for (uintptr_t p : kv.second) cudaFree((void*)p);
    if (dev->act_scratch) cudaFree(dev->act_scratch);
    for (int i = 0; i < 2; i++) { if (dev->up_pinned[i]) cudaFreeHost(dev->up_pinned[i]); if (dev->up_ev[i]) cudaEventDestroy(dev->up_ev[i]); }
    if (dev->err_host) cudaFreeHost(dev->err_host);
    if (dev->err_dev) cudaFree(dev->err_dev);
    if (dev->slots) cudaFree(dev->slots);
    if (dev->history) cudaFree(dev->history);
    if (dev->sample_scratch) cudaFree(dev->sample_scratch);
    if (dev->dev_idx) cudaFree(dev->dev_idx);
    cudaFree(dev->exp_lut);
    cudaFree(dev->gelu_lut);
    cudaStreamDestroy(dev->stream);
    delete dev;
}

extern "C" CC_API const char* cc_last_error(cc_device* dev) { return dev ? dev->last_error.c_str() : g_create_error.c_str(); }
extern "C" CC_API uint64_t cc_device_launch_count(cc_device* dev) { return dev ? dev->launches : 0; }
extern "C" CC_API void* cc_device_stream(cc_device* dev) { return dev ? (void*)dev->stream : nullptr; }

extern "C" CC_API int cc_device_synchronize(cc_device* dev) {
    if (!dev) return CC_ERR_ARG;
    CC_ENTER(dev);
    if (dev->lz) { int rc = cc_lazy_flush(dev); if (rc) return rc; }
    CC_CUDA(dev, cudaStreamSynchronize(dev->stream));
    return cc_check_async_error(dev);
}
// test / co-tenancy hook: persistent kernels of this device use at most `n` SMs (their grid = n CTAs), so that two devices of one
// process can run their megakernels side by side on ONE GPU (tests/test_gpu_sharded.py: world of 2 on a single GPU)
extern "C" CC_API int cc_device_set_sm_limit(cc_device* dev, int32_t n) {
    if (!dev) return CC_ERR_ARG;
    CC_ENTER(dev);
    cudaDeviceProp prop;
    CC_CUDA(dev, cudaGetDeviceProperties(&prop, dev->ordinal));
    CC_REQUIRE(dev, n >= 1 && n <= prop.multiProcessorCount, "sm_limit %d out of range (1..%d)", n, prop.multiProcessorCount);
    if (dev->lz) { int rc = cc_lazy_flush(dev); if (rc) return rc; }
    if (dev->lz && n != dev->sm_count) {         // cached graphs keep the grid they were captured with
        CC_CUDA(dev, cudaStreamSynchronize(dev->stream));
        if (int rc = cc_lazy_invalidate(dev)) return rc;
    }
    dev->sm_count = n;
    return CC_OK;
}
extern "C" CC_API int cc_device_flush(cc_device* dev) {
    if (!dev) return CC_ERR_ARG;
    CC_ENTER(dev);
    return dev->lz ? cc_lazy_flush(dev) : CC_OK;
}

extern "C" CC_API int cc_bench_timer_begin(cc_device* dev) {
    if (!dev) return CC_ERR_ARG;
    CC_ENTER(dev);
    if (!dev->ev_begin) { CC_CUDA(dev, cudaEventCreate(&dev->ev_begin)); CC_CUDA(dev, cudaEventCreate(&dev->ev_end)); }
    if (dev->lz) { int rc = cc_lazy_flush(dev); if (rc) return rc; }
    CC_CUDA(dev, cudaEventRecord(dev->ev_begin, dev->stream));
    return CC_OK;
}
extern "C" CC_API int cc_bench_timer_end(cc_device* dev, float* ms) {
    if (!dev || !ms || !dev->ev_begin) return CC_ERR_ARG;
    CC_ENTER(dev);
    if (dev->lz) { int rc = cc_lazy_flush(dev); if (rc) return rc; }
    CC_CUDA(dev, cudaEventRecord(dev->ev_end, dev->stream));
    CC_CUDA(dev, cudaEventSynchronize(dev->ev_end));
    CC_CUDA(dev, cudaEventElapsedTime(ms, dev->ev_begin, dev->ev_end));
    return cc_check_async_error(dev);
}

// ---- activation pool: power-of-two size classes, stream-ordered reuse (single stream) -------------
static size_t size_class(size_t bytes) {
    size_t c = 512;
    while (c < bytes) c <<= 1;
    return c;
}
int cc_pool_alloc(cc_device* dev, size_t bytes, void** out, size_t* cls) {
    size_t c = size_class(bytes ? bytes : 1);
    *cls = c;
    {
        std::lock_guard<std::mutex> g(dev->mu);
        auto& fl = dev->free_lists[c];
        if (!fl.empty()) {
            // lowest address first: the buffer a call gets depends only on the SET of free buffers, not on the order in
            // which they were released -> identical pointers token after token (lazy.cu hashes them into the graph key)
            *out = (void*)*fl.begin();
            fl.erase(fl.begin());
            return CC_OK;
        }
    }
    CC_CUDA(dev, cudaMalloc(out, c));
    dev->pool_live_bytes += c;
    return CC_OK;
}
void cc_pool_free(cc_device* dev, void* p, size_t cls) {
    std::lock_guard<std::mutex> g(dev->mu);
    dev->free_lists[cls].insert((uintptr_t)p);
}

int cc_new_activation(cc_device* dev, int64_t nelems, int dtype, bool zero, cc_buf** out) {
    size_t esz = dtype == CC_F32 ? 4 : 2;
    void* p = nullptr;
    size_t cls = 0;
    int rc = cc_pool_alloc(dev, (size_t)nelems * esz, &p, &cls);
    if (rc) return rc;
    if (zero && nelems > 0) CC_CUDA(dev, cudaMemsetAsync(p, 0, (size_t)nelems * esz, dev->stream));
    cc_buf* b = new cc_buf();
    b->dev = dev; b->dtype = dtype; b->nelems = nelems; b->base = p; b->bytes = cls; b->pooled = true;
    b->plane[0] = (uint8_t*)p;
    *out = b;
    return CC_OK;
}

int cc_ensure_slots(cc_device* dev) {
    if (dev->slots) return CC_OK;
    CC_CUDA(dev, cudaMalloc((void**)&dev->slots, CC_N_SLOTS * 8));
    CC_CUDA(dev, cudaMemset(dev->slots, 0, CC_N_SLOTS * 8));
    CC_CUDA(dev, cudaMalloc((void**)&dev->history, (size_t)CC_HISTORY_CAP * 8));
    return CC_OK;
}

int cc_ensure_act_scratch(cc_device* dev, size_t bytes) {
    if (bytes <= dev->act_scratch_bytes) return CC_OK;
    if (dev->act_scratch) {
        CC_CUDA(dev, cudaStreamSynchronize(dev->stream));
        if (int rc = cc_lazy_invalidate(dev)) return rc;      // the lazy modes' cached graphs of eager matvec steps hold the old pointer
        CC_CUDA(dev, cudaFree(dev->act_scratch));
    }
    size_t nb = size_class(bytes);
    CC_CUDA(dev, cudaMalloc(&dev->act_scratch, nb));
    dev->act_scratch_bytes = nb;
    return CC_OK;
}
int cc_ensure_dev_idx(cc_device* dev, size_t bytes) {
    if (bytes <= dev->dev_idx_bytes) return CC_OK;
    if (dev->dev_idx) { CC_CUDA(dev, cudaStreamSynchronize(dev->stream)); CC_CUDA(dev, cudaFree(dev->dev_idx)); }
    size_t nb = size_class(bytes);
    CC_CUDA(dev, cudaMalloc(&dev->dev_idx, nb));
    dev->dev_idx_bytes = nb;
    return CC_OK;
}

// ---- buffers -----------------------------------------------------------------------------------------
extern "C" CC_API void cc_tensor_retain(cc_buf* b) { if (b) b->refs.fetch_add(1); }
extern "C" CC_API void cc_tensor_release(cc_buf* b) {
    if (!b) return;
    if (b->refs.fetch_sub(1) != 1) return;
    CC_ENTER(b->dev);
    if (b->pooled) cc_pool_free(b->dev, b->base, b->bytes);
    else if (b->base) cudaFree(b->base);
    if (b->raw) cudaFree(b->raw);
    if (b->f16) cudaFree(b->f16);
    delete b;
}
extern "C" CC_API int32_t cc_tensor_dtype(const cc_buf* b) { return b ? b->dtype : -1; }
extern "C" CC_API int64_t cc_tensor_capacity(const cc_buf* b) { return b ? b->nelems : 0; }

static int64_t prod(const int64_t* shape, int ndim) {
    int64_t n = 1;
    for (int i = 0; i < ndim; i++) n *= shape[i];
    return n;
}

extern "C" CC_API int cc_tensor_alloc(cc_device* dev, const int64_t* shape, int32_t ndim, int32_t t, cc_buf** out) {
    if (!dev || !shape || !out || ndim < 1 || ndim > CC_MAX_DIMS) return cc_fail(dev, CC_ERR_ARG, "cc_tensor_alloc: bad argument");
    CC_ENTER(dev);
    CC_REQUIRE(dev, t == CC_F32 || t == CC_F16, "only f32/f16 is supported");   // cpu_tensor.rs:139-141
    // F32 is zero-filled (vec![0.0; n]); F16 is uninitialised in the reference (buf_f16.rs:23-28), zeroed here
    return cc_new_activation(dev, prod(shape, ndim), t, true, out);
}

// Host bytes -> device through two pinned 16 MB staging buffers (model.rs:462-477 hands over slices of the GGUF mmap: pageable and
// usually not yet resident).  While chunk i is DMA'd, the host copies (= page-faults) chunk i+1 into the other buffer; nothing here
// waits for the GPU except the reuse of a staging buffer, so uploads of consecutive tensors and their repack kernels overlap.
#define CC_UP_CHUNK ((size_t)16 << 20)
static int cc_upload_staged(cc_device* dev, void* dst, const void* src, size_t n) {
    if (n <= ((size_t)1 << 20)) {
        CC_CUDA(dev, cudaMemcpyAsync(dst, src, n, cudaMemcpyHostToDevice, dev->stream));     // small: the driver's own staging is fine
        return CC_OK;
    }
    for (int i = 0; i < 2; i++)
        if (!dev->up_pinned[i]) {
            CC_CUDA(dev, cudaMallocHost(&dev->up_pinned[i], CC_UP_CHUNK));
            CC_CUDA(dev, cudaEventCreateWithFlags(&dev->up_ev[i], cudaEventDisableTiming));
        }
    int i = 0;
    for (size_t off = 0; off < n; off += CC_UP_CHUNK, i ^= 1) {
        const size_t len = n - off < CC_UP_CHUNK ? n - off : CC_UP_CHUNK;
        CC_CUDA(dev, cudaEventSynchronize(dev->up_ev[i]));                      // the copy that last read this buffer is done
        memcpy(dev->up_pinned[i], (const uint8_t*)src + off, len);
        CC_CUDA(dev, cudaMemcpyAsync((uint8_t*)dst + off, dev->up_pinned[i], len, cudaMemcpyHostToDevice, dev->stream));
        CC_CUDA(dev, cudaEventRecord(dev->up_ev[i], dev->stream));
    }
    return CC_OK;
}

extern "C" CC_API int cc_tensor_from_cpu(cc_device* dev, const void* bytes, size_t nbytes, const int64_t* shape,
                                  int32_t ndim, int32_t t, cc_buf** out) {
    if (!dev || !bytes || !shape || !out || ndim < 1 || ndim > CC_MAX_DIMS) return cc_fail(dev, CC_ERR_ARG, "cc_tensor_from_cpu: bad argument");
    CC_ENTER(dev);
    int be = cc_block_elems(t);
    CC_REQUIRE(dev, be > 0, "from_cpu: unsupported ggml type %d", t);
    int64_t n = prod(shape, ndim);
    int64_t cols = shape[ndim - 1], rows = n / (cols ? cols : 1);
    CC_REQUIRE(dev, cols % be == 0, "from_cpu: last dim %lld is not a multiple of the %d-element block", (long long)cols, be);
    size_t need = (size_t)(n / be) * cc_block_bytes(t);   // size from shape, not slice length (B16, gguf.rs:742-747)
    CC_REQUIRE(dev, nbytes >= need, "from_cpu: %zu bytes given, %zu needed for shape", nbytes, need);
    cc_buf* b = new cc_buf();
    b->dev = dev; b->dtype = t; b->nelems = n; b->rows = rows; b->cols = cols;
    if (!cc_is_quant(t)) {
        b->bytes = need;
        cudaError_t e = cudaMalloc(&b->base, need ? need : 1);
        if (e != cudaSuccess) { delete b; return cc_fail(dev, CC_ERR_CUDA, "cudaMalloc(%zu): %s", need, cudaGetErrorString(e)); }
        b->plane[0] = (uint8_t*)b->base;
        int urc = cc_upload_staged(dev, b->base, bytes, need);
        if (urc == CC_OK && need <= ((size_t)1 << 20)) { e = cudaStreamSynchronize(dev->stream); if (e != cudaSuccess) urc = cc_fail(dev, CC_ERR_CUDA, "upload: %s", cudaGetErrorString(e)); }
        if (urc != CC_OK) { cudaFree(b->base); delete b; return urc; }      // (small copies read the caller's buffer asynchronously: wait; staged ones were copied out)
        *out = b;
        return CC_OK;
    }
    // quantized: stage the GGUF bytes on device, repack into planes, drop the staging copy
    b->bytes = cc_device_layout_bytes(t, rows, cols);
    uint8_t* staging = nullptr;
    cudaError_t e = cudaMalloc(&b->base, b->bytes ? b->bytes : 1);
    if (e == cudaSuccess) e = cudaMalloc(&staging, need ? need : 1);
    if (e == cudaSuccess && cc_upload_staged(dev, staging, bytes, need) != CC_OK) e = cudaErrorUnknown;
    if (e != cudaSuccess) {
        if (b->base) cudaFree(b->base);
        if (staging) cudaFree(staging);
        delete b;
        return cc_fail(dev, CC_ERR_CUDA, "from_cpu upload (%zu bytes): %s", need, cudaGetErrorString(e));
    }
    cc_assign_planes(b);
    int rc = cc_launch_repack(dev, staging, b);
    cudaError_t e2 = cudaStreamSynchronize(dev->stream);
    if (dev->exact) b->raw = staging; else cudaFree(staging);     // exact_order keeps the GGUF-layout bytes
    if (rc == CC_OK && e2 != cudaSuccess) rc = cc_fail(dev, CC_ERR_CUDA, "repack: %s", cudaGetErrorString(e2));
    if (rc != CC_OK) { cudaFree(b->base); if (b->raw) cudaFree(b->raw); delete b; return rc; }
    *out = b;
    return CC_OK;
}

extern "C" CC_API int cc_tensor_synth(cc_device* dev, const int64_t* shape, int32_t ndim, int32_t t, uint64_t seed,
                               uint64_t tensor_id, float scale, cc_buf** out) {
    if (!dev || !shape || !out || ndim < 1 || ndim > CC_MAX_DIMS) return cc_fail(dev, CC_ERR_ARG, "cc_tensor_synth: bad argument");
    CC_ENTER(dev);
    int be = cc_block_elems(t);
    CC_REQUIRE(dev, be > 1, "synth: quantized types only, got %d", t);
    int64_t n = prod(shape, ndim);
    int64_t cols = shape[ndim - 1], rows = n / cols;
    CC_REQUIRE(dev, cols % be == 0, "synth: last dim %lld is not a multiple of the block", (long long)cols);
    size_t need = (size_t)(n / be) * cc_block_bytes(t);
    cc_buf* b = new cc_buf();
    b->dev = dev; b->dtype = t; b->nelems = n; b->rows = rows; b->cols = cols;
    b->bytes = cc_device_layout_bytes(t, rows, cols);
    uint8_t* staging = nullptr;
    cudaError_t e = cudaMalloc(&b->base, b->bytes);
    if (e == cudaSuccess) e = cudaMalloc(&staging, need);
    if (e != cudaSuccess) {
        if (b->base) cudaFree(b->base);
        delete b;
        return cc_fail(dev, CC_ERR_CUDA, "synth alloc: %s", cudaGetErrorString(e));
    }
    cc_assign_planes(b);
    int rc = cc_launch_synth(dev, staging, t, n / be, seed, tensor_id, scale);
    if (rc == CC_OK) rc = cc_launch_repack(dev, staging, b);
    cudaError_t e2 = cudaStreamSynchronize(dev->stream);
    if (dev->exact) b->raw = staging; else cudaFree(staging);
    if (rc == CC_OK && e2 != cudaSuccess) rc = cc_fail(dev, CC_ERR_CUDA, "synth: %s", cudaGetErrorString(e2));
    if (rc != CC_OK) { cudaFree(b->base); if (b->raw) cudaFree(b->raw); delete b; return rc; }
    *out = b;
    return CC_OK;
}

// Shard of a synthetic matrix: the full tensor is generated (same counter-based bytes as cc_tensor_synth), then the
// requested rows x block-columns are compacted and repacked.  Rows shard wq/wk/wv/gate/up/classifier, columns shard wo/down.
extern "C" CC_API int cc_tensor_synth_slice(cc_device* dev, const int64_t* shape, int32_t ndim, int32_t t, uint64_t seed, uint64_t tensor_id,
                                            float scale, int64_t row0, int64_t nrows, int64_t col0, int64_t ncols, cc_buf** out) {
    if (!dev || !shape || !out || ndim != 2) return cc_fail(dev, CC_ERR_ARG, "cc_tensor_synth_slice: bad argument (2-d tensors only)");
    CC_ENTER(dev);
    int be = cc_block_elems(t);
    CC_REQUIRE(dev, be > 1, "synth_slice: quantized types only, got %d", t);
    const int64_t rows = shape[0], cols = shape[1];
    CC_REQUIRE(dev, cols % be == 0 && col0 % be == 0 && ncols % be == 0, "synth_slice: columns must be multiples of the %d-element block", be);
    CC_REQUIRE(dev, row0 >= 0 && nrows > 0 && row0 + nrows <= rows && col0 >= 0 && ncols > 0 && col0 + ncols <= cols, "synth_slice: slice out of range");
    const size_t bb = cc_block_bytes(t);
    const size_t full = (size_t)(rows * cols / be) * bb, part = (size_t)(nrows * ncols / be) * bb;
    cc_buf* b = new cc_buf();
    b->dev = dev; b->dtype = t; b->nelems = nrows * ncols; b->rows = nrows; b->cols = ncols;
    b->bytes = cc_device_layout_bytes(t, nrows, ncols);
    uint8_t *staging = nullptr, *compact = nullptr;
    cudaError_t e = cudaMalloc(&b->base, b->bytes);
    if (e == cudaSuccess) e = cudaMalloc(&staging, full);
    if (e == cudaSuccess) e = cudaMalloc(&compact, part);
    if (e != cudaSuccess) {
        if (b->base) cudaFree(b->base);
        if (staging) cudaFree(staging);
        delete b;
        return cc_fail(dev, CC_ERR_CUDA, "synth_slice alloc: %s", cudaGetErrorString(e));
    }
    cc_assign_planes(b);
    int rc = cc_launch_synth(dev, staging, t, rows * cols / be, seed, tensor_id, scale);
    if (rc == CC_OK) {
        const size_t row_bytes = (size_t)(cols / be) * bb, w = (size_t)(ncols / be) * bb;
        e = cudaMemcpy2DAsync(compact, w, staging + (size_t)row0 * row_bytes + (size_t)(col0 / be) * bb, row_bytes, w, (size_t)nrows, cudaMemcpyDeviceToDevice, dev->stream);
        if (e != cudaSuccess) rc = cc_fail(dev, CC_ERR_CUDA, "synth_slice compact: %s", cudaGetErrorString(e));
    }
    if (rc == CC_OK) rc = cc_launch_repack(dev, compact, b);
    cudaError_t e2 = cudaStreamSynchronize(dev->stream);
    cudaFree(staging);
    if (dev->exact) b->raw = compact; else cudaFree(compact);
    if (rc == CC_OK && e2 != cudaSuccess) rc = cc_fail(dev, CC_ERR_CUDA, "synth_slice: %s", cudaGetErrorString(e2));
    if (rc != CC_OK) { cudaFree(b->base); if (b->raw) cudaFree(b->raw); delete b; return rc; }
    *out = b;
    return CC_OK;
}

extern "C" CC_API int cc_test_export_blocks(cc_device* dev, const cc_buf* buf, void* dst, size_t nbytes) {
    if (!dev || !buf || !dst) return cc_fail(dev, CC_ERR_ARG, "cc_test_export_blocks: bad argument");
    CC_ENTER(dev);
    if (dev->lz) { int rc = cc_lazy_flush(dev); if (rc) return rc; }
    CC_REQUIRE(dev, cc_is_quant(buf->dtype), "export_blocks: not a quantized tensor");
    size_t need = (size_t)(buf->nelems / cc_block_elems(buf->dtype)) * cc_block_bytes(buf->dtype);
    CC_REQUIRE(dev, nbytes >= need, "export_blocks: %zu bytes given, %zu needed", nbytes, need);
    uint8_t* staging = nullptr;
    CC_CUDA(dev, cudaMalloc(&staging, need));
    int rc = cc_launch_unrepack(dev, buf, staging);
    if (rc == CC_OK) {
        cudaError_t e = cudaMemcpyAsync(dst, staging, need, cudaMemcpyDeviceToHost, dev->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(dev->stream);
        if (e != cudaSuccess) rc = cc_fail(dev, CC_ERR_CUDA, "export_blocks: %s", cudaGetErrorString(e));
    }
    cudaFree(staging);
    return rc;
}
