// capi.cu -- extern "C" entry points: argument checks mirroring CpuTensor (cpu_tensor.rs:126-446), then one op record (op_record.cuh)
// that eager mode runs at once and lazy mode queues.
#include "op_record.cuh"

static bool view_ok(const cc_view* v) { return v && v->buf && v->ndim >= 1 && v->ndim <= CC_MAX_DIMS; }
// highest element offset the view addresses (-1 for an empty view); negative strides / shapes are rejected by the caller
static int64_t view_max_offset(const cc_view* v) {
    int64_t off = 0;
    for (int i = 0; i < v->ndim; i++) {
        if (v->shape[i] <= 0) return -1;
        off += (v->shape[i] - 1) * v->strides[i];
    }
    return off;
}
static bool view_in_bounds(const cc_view* v) {
    for (int i = 0; i < v->ndim; i++) if (v->shape[i] < 0 || v->strides[i] < 0) return false;
    return view_max_offset(v) < v->buf->nelems;
}

// argument checks shared by every op: a usable view whose highest addressed element lies inside its buffer (the strider lives on
// the host side of the ABI, so a stale or mismatched shape must become a TensorError here, not an out-of-bounds device read)
#define CHECK_VIEW(dev, v, what)                                                         \
    if (!(dev)) return CC_ERR_ARG;                                                       \
    CC_ENTER(dev);                                                                       \
    if (!view_ok(v)) return cc_fail((dev), CC_ERR_ARG, "%s: bad tensor view", what);     \
    if (!view_in_bounds(v)) return cc_fail((dev), CC_ERR_TENSOR, "%s: view addresses element %lld of a buffer of %lld", what, \
                                           (long long)view_max_offset(v), (long long)(v)->buf->nelems)
// a quantized weight matrix is laid out in planes that depend on its row length: the view must be the matrix itself (or a prefix
// of its rows), never a reshape
#define CHECK_QUANT_MATRIX(dev, v, what)                                                                                       \
    if (cc_is_quant((v)->buf->dtype))                                                                                          \
        CC_REQUIRE(dev, (v)->ndim == 2 && (v)->shape[1] == (v)->buf->cols && (v)->shape[0] <= (v)->buf->rows,                  \
                   "%s: view [%lld, %lld] does not match the quantized matrix [%lld, %lld]", what, (long long)(v)->shape[0],   \
                   (long long)((v)->ndim == 2 ? (v)->shape[1] : 0), (long long)(v)->buf->rows, (long long)(v)->buf->cols)
#define LAZY(dev) ((dev)->lz != nullptr && !(dev)->exact)
#define FLUSH(dev)                                  \
    do {                                            \
        if (LAZY(dev)) { int _rc = cc_lazy_flush(dev); if (_rc) return _rc; } \
    } while (0)

#define REQUIRE_F32(dev, v, what) CC_REQUIRE(dev, (v)->buf->dtype == CC_F32, "%s: not f32, but got type %d", what, (v)->buf->dtype)

// ---- one op's launch ----------------------------------------------------------------------------------------------------
// fast-order matmul_vec of b rows of x: x quantised to the weight's partner type, then the streaming kernel (decode), the dense
// tensor-core GEMM (prefill_gemm.cu) or the warp-per-row kernel.  The activation scratch only grows here when it is too small; lazy.cu
// sizes it before any capture.
static int launch_matmul_vec(cc_device* dev, const cc_buf* w, const float* xf, float* out, int64_t m, int64_t k, int64_t b) {
    const int wt = w->dtype, at = cc_partner_type(wt);
    const bool stream = b == 1 && cc_stream_supported(wt, k);
    const bool dense = !stream && cc_prefill_supported(wt, m, k, b);
    int rc = CC_OK;
    if (at != CC_F32 && !(dense && at == CC_Q8_0)) {         // (the dense path quantises Q8_0 partners itself, fused with the f16 conversion)
        rc = cc_ensure_act_scratch(dev, cc_act_bytes(at, b * k));
        if (!rc) rc = cc_launch_quantize(dev, xf, b * k, at, dev->act_scratch);     // matmul_vec.rs:37-40
    }
    if (rc) return rc;
    if (stream) return cc_launch_matvec_stream_plain(dev, w, dev->act_scratch, out, m, k);     // decode hot path
    if (dense) return cc_launch_prefill_matmul(dev, w, dev->act_scratch, at == CC_Q8_0 ? xf : nullptr, out, m, k, b);
    return cc_launch_matvec(dev, w, dev->act_scratch, xf, out, m, k, b);
}

// exact_order: reference-layout activation blocks + scalar-order dot on the GGUF-layout weights
static int launch_matmul_vec_exact(cc_device* dev, const cc_buf* w, const float* xf, float* out, int64_t m, int64_t k, int64_t b) {
    const int wt = w->dtype, at = cc_partner_type(wt);
    int rc = CC_OK;
    if (at != CC_F32) {
        rc = cc_ensure_act_scratch(dev, cc_act_bytes(at, b * k));
        if (!rc) rc = cc_launch_quantize(dev, xf, b * k, at, dev->act_scratch);     // matmul_vec.rs:37-40
    }
    const uint8_t* wraw = cc_is_quant(wt) ? w->raw : w->plane[0];
    if (!rc && !wraw) rc = cc_fail(dev, CC_ERR_TENSOR, "matmul_vec(exact): weight has no GGUF-layout copy");
    void* blocks = nullptr; size_t cls = 0;
    if (!rc && (at == CC_Q8_0 || at == CC_Q8_1 || at == CC_Q8_K)) {
        rc = cc_pool_alloc(dev, (size_t)(b * k / cc_block_elems(at)) * cc_block_bytes(at), &blocks, &cls);
        if (!rc) rc = cc_launch_act_to_blocks(dev, dev->act_scratch, b * k, at, (uint8_t*)blocks);
    }
    const uint8_t* act = blocks ? (const uint8_t*)blocks : at == CC_F32 ? (const uint8_t*)xf : (const uint8_t*)dev->act_scratch;
    if (!rc) rc = cc_launch_matvec_exact(dev, wt, wraw, act, out, m, k, b);
    if (blocks) cc_pool_free(dev, blocks, cls);
    return rc;
}

// The kernels of one checked op: every op of eager mode, and every op of lazy mode that no fused step takes.  An exact_order device
// runs the reference's summation order where it differs from the fast one (exact.cu); lazy mode never runs on such a device.
int cc_run_op(cc_device* d, const LOp& op) {
    const cc_view &a = op.a, &b = op.b;
    float* x = (float*)a.buf->plane[0];
    switch (op.kind) {
    case L_DUP: {
        const int64_t n = view_len(&a);
        if (n) CC_CUDA(d, cudaMemcpyAsync(op.out->base, a.buf->plane[0], (size_t)n * 4, cudaMemcpyDeviceToDevice, d->stream));
        return CC_OK;
    }
    case L_CONTIGUOUS: {
        int64_t dstr[CC_MAX_DIMS];
        int64_t s = 1;
        for (int i = a.ndim - 1; i >= 0; i--) { dstr[i] = s; s *= a.shape[i]; }
        return cc_launch_strided_copy(d, a.buf->plane[0], a.buf->dtype, a.shape, a.strides, op.out->base, a.buf->dtype, dstr, 0, a.ndim);
    }
    case L_CONCAT:
        return cc_launch_strided_copy(d, b.buf->plane[0], b.buf->dtype, b.shape, b.strides, a.buf->plane[0], a.buf->dtype, a.strides,
                                      a.shape[op.i0] * a.strides[op.i0], a.ndim);
    case L_COPY_ROWS: {
        const int64_t cols = a.shape[a.ndim - 1];
        if (op.i2 > 0)      // NOTE: the id in the slot was produced by argmax over this model's logits, i.e. it is < vocab rows by construction
            return cc_launch_dequant_rows(d, cc_deq_planes(b.buf, cols), b.buf->dtype, d->slots + (op.i2 - 1), 1, cols, a.buf->plane[0], a.buf->dtype);
        const size_t n = op.rows.size();
        int rc = cc_ensure_dev_idx(d, n * 8);
        if (rc) return rc;
        CC_CUDA(d, cudaMemcpyAsync(d->dev_idx, op.rows.data(), n * 8, cudaMemcpyHostToDevice, d->stream));
        return cc_launch_dequant_rows(d, cc_deq_planes(b.buf, cols), b.buf->dtype, (const int64_t*)d->dev_idx, (int)n, cols, a.buf->plane[0], a.buf->dtype);
    }
    case L_ROPE:
        // cos/sin are evaluated on the host with the same libm calls as the reference (rope.rs:52-53,74-75) in both
        // modes: bit-exact, and no slow large-argument device sinf/cosf
        return cc_launch_rope_exact(d, x, op.i1, op.i2, a.shape[a.ndim - 1], (int)op.f, op.i0, op.rows[0]);
    case L_RMS_NORM: {
        const int64_t rows = a.ndim == 1 ? 1 : a.shape[0], cols = a.shape[a.ndim - 1];
        return d->exact ? cc_launch_rms_norm_exact(d, x, rows, cols, op.f) : cc_launch_rms_norm(d, x, rows, cols, op.f);
    }
    case L_SOFTMAX: {
        const int64_t cols = a.shape[a.ndim - 1], rows = cols ? view_len(&a) / cols : 0;
        return d->exact ? cc_launch_softmax_exact(d, x, rows, cols) : cc_launch_softmax(d, x, rows, cols);
    }
    case L_SILU: return cc_launch_silu(d, x, view_len(&a));
    case L_GELU: return cc_launch_gelu(d, x, view_len(&a));
    case L_MUL: return cc_launch_binary(d, x, op.i0, (const float*)b.buf->plane[0], op.i1, 1);
    case L_ADD: return cc_launch_binary(d, x, op.i0, (const float*)b.buf->plane[0], op.i1, 0);
    case L_SCALE: return cc_launch_scale(d, x, view_len(&a), op.f);
    case L_ALLREDUCE: return cc_launch_all_reduce(d, x, op.i0, nullptr);
    case L_ALLGATHER: return cc_launch_all_gather(d, (const float*)b.buf->plane[0], op.i0, x);
    case L_ARGMAX: return cc_launch_argmax(d, x, view_len(&a), d->slots + op.i0, d->history, nullptr, op.i1);
    case L_SAMPLE: {
        int rc = cc_ensure_sample_scratch(d, view_len(&a));
        if (rc) return rc;
        const SampleDyn s = cc_sample_dyn(op);
        return cc_launch_sample(d, x, view_len(&a), &s, nullptr, d->slots + op.i0, d->history);
    }
    case L_MATVEC: {
        const float* xf = (const float*)b.buf->plane[0];
        const int64_t rows = b.ndim == 1 ? 1 : b.shape[0];
        if (d->exact) return launch_matmul_vec_exact(d, a.buf, xf, (float*)op.out->base, a.shape[0], a.shape[1], rows);
        return launch_matmul_vec(d, a.buf, xf, (float*)op.out->base, a.shape[0], a.shape[1], rows);
    }
    case L_BMM:
        if (d->exact && b.strides[1] == 1)
            return cc_launch_bmm_kcontig_exact(d, x, b.buf->plane[0], b.buf->dtype, (float*)op.out->base, a.shape[0], b.shape[0], a.shape[1],
                                               a.shape[2], b.shape[2], b.strides[0], b.strides[2]);
        return cc_launch_batch_matmul(d, x, b.buf->plane[0], b.buf->dtype, (float*)op.out->base, a.shape[0], b.shape[0], a.shape[1], a.shape[2],
                                      b.shape[2], b.strides[0], b.strides[1], b.strides[2]);
    }
    return cc_fail(d, CC_ERR_UNSUPPORTED, "unknown op kind %d", op.kind);
}

// lazy mode queues a checked op (lazy.cu), eager mode runs it now.  An op with a result (out != NULL) gets a new activation of out_elems
// elements as op.out: *out receives it on success, and it is released on failure.
static int submit(cc_device* dev, LOp op, cc_buf** out = nullptr, int64_t out_elems = 0, int out_type = CC_F32) {
    if (out) {
        int rc = cc_new_activation(dev, out_elems, out_type, false, &op.out);
        if (rc) return rc;
    }
    cc_buf* result = op.out;
    const int rc = LAZY(dev) ? cc_lazy_record(dev, std::move(op)) : cc_run_op(dev, op);
    if (out) {
        if (rc) cc_tensor_release(result);
        else *out = result;
    }
    return rc;
}

// ---- dup / export / contiguous ----------------------------------------------------------------------------------
extern "C" CC_API int cc_tensor_dup(cc_device* dev, const cc_view* src, cc_buf** out) {     // cpu_tensor.rs:333-337
    CHECK_VIEW(dev, src, "dup");
    if (!out) return cc_fail(dev, CC_ERR_ARG, "dup: out is NULL");
    REQUIRE_F32(dev, src, "dup");
    // the reference copies the WHOLE buffer (iter_f32) and gives it the view's shape
    int64_t n = view_len(src);
    CC_REQUIRE(dev, n == src->buf->nelems || view_contiguous(src), "dup: shape does not cover the buffer");
    return submit(dev, LOp{.kind = L_DUP, .a = *src}, out, n);
}

extern "C" CC_API int cc_tensor_export_f32(cc_device* dev, const cc_view* src, float* dst, size_t n) {   // cpu_tensor.rs:339-349
    CHECK_VIEW(dev, src, "export");
    if (!dst) return cc_fail(dev, CC_ERR_ARG, "export: dst is NULL");
    REQUIRE_F32(dev, src, "export");
    CC_REQUIRE(dev, view_contiguous(src), "export: tensor is not contiguous");
    FLUSH(dev);
    int64_t len = view_len(src);
    size_t cnt = n < (size_t)len ? n : (size_t)len;
    if (cnt) CC_CUDA(dev, cudaMemcpyAsync(dst, src->buf->plane[0], cnt * 4, cudaMemcpyDeviceToHost, dev->stream));
    CC_CUDA(dev, cudaStreamSynchronize(dev->stream));
    return cc_check_async_error(dev);
}

extern "C" CC_API int cc_contiguous(cc_device* dev, const cc_view* src, cc_buf** out) {     // cpu_tensor.rs:294-304
    CHECK_VIEW(dev, src, "contiguous");
    if (!out) return cc_fail(dev, CC_ERR_ARG, "contiguous: out is NULL");
    if (view_contiguous(src)) {                                   // no-op: same storage
        cc_tensor_retain(src->buf);
        *out = src->buf;
        return CC_OK;
    }
    int t = src->buf->dtype;
    CC_REQUIRE(dev, t == CC_F32 || t == CC_F16, "contiguous: only f32/f16");
    CC_REQUIRE(dev, src->ndim == 2 || src->ndim == 3, "contiguous: only 2d/3d tensors");
    return submit(dev, LOp{.kind = L_CONTIGUOUS, .a = *src}, out, view_len(src), t);
}

// ---- concatenate: cpu_tensor.rs:251-292 ------------------------------------------------------------------------------
extern "C" CC_API int cc_concatenate(cc_device* dev, const cc_view* self, const cc_view* rhs, int32_t axis) {
    CHECK_VIEW(dev, self, "concatenate");
    CHECK_VIEW(dev, rhs, "concatenate rhs");
    int t1 = self->buf->dtype, t2 = rhs->buf->dtype;
    CC_REQUIRE(dev, self->buf->pooled, "tensor not owned on concatenate");
    CC_REQUIRE(dev, t1 == CC_F32 || t1 == CC_F16, "only f32/f16 is supported on concatenate");
    CC_REQUIRE(dev, t2 == CC_F32 || t2 == CC_F16, "only f32/f16 is supported on concatenate rhs");
    CC_REQUIRE(dev, !(t1 == CC_F32 && t2 == CC_F16), "can not concatenate F32 and F16");
    CC_REQUIRE(dev, self->ndim == rhs->ndim && axis >= 0 && axis < self->ndim, "concatenate: bad axis/rank");
    for (int i = 0; i < self->ndim; i++)
        if (i != axis) CC_REQUIRE(dev, self->shape[i] == rhs->shape[i], "shape mismatch on concatenate");
    // highest destination element must stay inside the pre-allocated storage
    int64_t hi = 0;
    for (int i = 0; i < self->ndim; i++) {
        int64_t top = (i == axis ? self->shape[i] + rhs->shape[i] : self->shape[i]) - 1;
        if (top >= 0) hi += top * self->strides[i];
    }
    CC_REQUIRE(dev, view_len(rhs) == 0 || hi < self->buf->nelems, "concatenate: exceeds the pre-allocated storage");
    return submit(dev, LOp{.kind = L_CONCAT, .a = *self, .b = *rhs, .i0 = axis});
}

// ---- copy_rows_from: cpu_tensor.rs:306-331 ----------------------------------------------------------------------------
extern "C" CC_API int cc_copy_rows_from(cc_device* dev, const cc_view* dst, const cc_view* src, const int64_t* rows, int32_t n_rows) {
    CHECK_VIEW(dev, dst, "copy_rows_from");
    CHECK_VIEW(dev, src, "copy_rows_from src");
    CC_REQUIRE(dev, dst->buf->pooled, "not owned");
    CC_REQUIRE(dev, view_contiguous(dst), "dst tensor is not contiguous");
    CC_REQUIRE(dev, view_contiguous(src), "src tensor is not contiguous");
    CC_REQUIRE(dev, src->ndim == 1 || src->ndim == 2, "copy_rows_from: src tensor is not 2d or 1d");
    int dt = dst->buf->dtype;
    CC_REQUIRE(dev, dt == CC_F32 || dt == CC_F16, "only f32/f16 can be copied to");
    int64_t cols = dst->shape[dst->ndim - 1];
    int be = cc_block_elems(src->buf->dtype);
    CC_REQUIRE(dev, cols % be == 0, "copy_rows_from: row length %lld is not block aligned", (long long)cols);
    CC_REQUIRE(dev, !cc_is_quant(src->buf->dtype) || cols == src->buf->cols, "copy_rows_from: row length %lld does not match the quantized matrix (%lld columns)",
               (long long)cols, (long long)src->buf->cols);
    CC_REQUIRE(dev, (int64_t)n_rows * cols <= view_len(dst), "copy_rows_from: dst too small");
    int64_t src_len = view_len(src);
    for (int i = 0; i < n_rows; i++)
        CC_REQUIRE(dev, rows[i] >= 0 && (rows[i] + 1) * cols <= src_len, "copy_rows_from: row %lld out of range", (long long)rows[i]);
    if (n_rows == 0) return CC_OK;
    return submit(dev, LOp{.kind = L_COPY_ROWS, .a = *dst, .b = *src, .rows = std::vector<int64_t>(rows, rows + n_rows)});
}

// ---- in-place ops -------------------------------------------------------------------------------------------------------
extern "C" CC_API int cc_rope_inplace(cc_device* dev, const cc_view* x, int32_t mode, int64_t pos, int64_t rope_dims) {   // rope.rs:10-45
    CHECK_VIEW(dev, x, "rope_inplace");
    CC_REQUIRE(dev, x->buf->dtype == CC_F32 && x->buf->pooled, "only support f32 yet");
    CC_REQUIRE(dev, view_contiguous(x), "rope_inplace: not contiguous");
    CC_REQUIRE(dev, x->ndim == 2 || x->ndim == 3, "rope_inplace: only 2d/3d tensors");
    CC_REQUIRE(dev, mode == CC_ROPE_LLAMA || mode == CC_ROPE_NEOX, "rope_inplace: bad mode");
    int64_t n_batch, stride, hd;
    if (x->ndim == 2) { n_batch = 1; stride = view_len(x); hd = x->shape[1]; }
    else { n_batch = x->shape[0]; stride = x->strides[0]; hd = x->shape[2]; }
    CC_REQUIRE(dev, rope_dims >= 0 && rope_dims <= hd && rope_dims % 2 == 0, "rope_inplace: bad rope_dims %lld", (long long)rope_dims);
    return submit(dev, LOp{.kind = L_ROPE, .a = *x, .f = (float)mode, .i0 = pos, .i1 = n_batch, .i2 = stride, .rows = {rope_dims}});
}

extern "C" CC_API int cc_rms_norm_inplace(cc_device* dev, const cc_view* x, float eps) {    // rms_norm.rs:9-30
    CHECK_VIEW(dev, x, "rms_norm_inplace");
    CC_REQUIRE(dev, view_contiguous(x), "rms_norm_inplace: not contiguous");
    CC_REQUIRE(dev, x->ndim == 1 || x->ndim == 2, "rms_norm_inplace: only 1d/2d tensors");
    REQUIRE_F32(dev, x, "rms_norm_inplace");
    int64_t cols = x->shape[x->ndim - 1];
    CC_REQUIRE(dev, cols % 32 == 0, "rms_norm_inplace: length %lld %% 32 != 0", (long long)cols);   // rms_norm.rs:34
    return submit(dev, LOp{.kind = L_RMS_NORM, .a = *x, .f = eps});
}

extern "C" CC_API int cc_softmax_inplace(cc_device* dev, const cc_view* x, int32_t axis) {  // softmax.rs:11-37
    CHECK_VIEW(dev, x, "softmax_inplace");
    CC_REQUIRE(dev, x->ndim == 2 || x->ndim == 3, "softmax_inplace: only 2d/3d tensors");
    CC_REQUIRE(dev, view_contiguous(x), "softmax_inplace: not contiguous");
    REQUIRE_F32(dev, x, "softmax_inplace");
    CC_REQUIRE(dev, axis == x->ndim - 1, "only axis=%d is supported on a %d dimensions tensor", x->ndim - 1, x->ndim);
    return submit(dev, LOp{.kind = L_SOFTMAX, .a = *x});
}

extern "C" CC_API int cc_silu_inplace(cc_device* dev, const cc_view* x) {                   // silu.rs:6-13: whole buffer
    CHECK_VIEW(dev, x, "silu_inplace");
    REQUIRE_F32(dev, x, "silu_inplace");
    return submit(dev, LOp{.kind = L_SILU, .a = *x});
}
extern "C" CC_API int cc_gelu_inplace(cc_device* dev, const cc_view* x) {                   // gelu.rs:10-15
    CHECK_VIEW(dev, x, "gelu_inplace");
    REQUIRE_F32(dev, x, "gelu_inplace");
    return submit(dev, LOp{.kind = L_GELU, .a = *x});
}

static int binary(cc_device* dev, const cc_view* x, const cc_view* rhs, int kind, const char* what) {   // arithmetic.rs:5-68
    CHECK_VIEW(dev, x, what);
    CHECK_VIEW(dev, rhs, what);
    REQUIRE_F32(dev, x, what);
    REQUIRE_F32(dev, rhs, what);
    int64_t n = view_len(x), ny = view_len(rhs);
    CC_REQUIRE(dev, ny > 0 && n % ny == 0, "%s: len %lld is not a multiple of rhs len %lld", what, (long long)n, (long long)ny);
    CC_REQUIRE(dev, x->shape[x->ndim - 1] == rhs->shape[rhs->ndim - 1] || ny == 1, "%s: last dims differ", what);
    CC_REQUIRE(dev, view_contiguous(x) && view_contiguous(rhs), "%s: not contiguous", what);
    if (ny != 1) {             // chunks_exact(4) on both sides: tails are silently skipped in the reference
        n -= n % 4;
        ny -= ny % 4;
        if (ny == 0) return CC_OK;
    }
    return submit(dev, LOp{.kind = kind, .a = *x, .b = *rhs, .i0 = n, .i1 = ny});
}
extern "C" CC_API int cc_mul_inplace(cc_device* dev, const cc_view* x, const cc_view* rhs) { return binary(dev, x, rhs, L_MUL, "mul_inplace"); }
extern "C" CC_API int cc_add_inplace(cc_device* dev, const cc_view* x, const cc_view* rhs) { return binary(dev, x, rhs, L_ADD, "add_inplace"); }
extern "C" CC_API int cc_scale_inplace(cc_device* dev, const cc_view* x, float rhs) {
    CHECK_VIEW(dev, x, "scale_inplace");
    REQUIRE_F32(dev, x, "scale_inplace");
    CC_REQUIRE(dev, view_contiguous(x), "scale_inplace: not contiguous");
    return submit(dev, LOp{.kind = L_SCALE, .a = *x, .f = rhs});
}

// ---- exchange step of the sharded path (comm.cu) ------------------------------------------------------------------------
extern "C" CC_API int cc_all_reduce_sum_inplace(cc_device* dev, const cc_view* x) {
    CHECK_VIEW(dev, x, "all_reduce_sum_inplace");
    REQUIRE_F32(dev, x, "all_reduce_sum_inplace");
    CC_REQUIRE(dev, view_contiguous(x), "all_reduce_sum_inplace: not contiguous");
    CC_REQUIRE(dev, dev->comm, "all_reduce_sum_inplace: no communicator on this device");
    const int64_t n = view_len(x);
    CC_REQUIRE(dev, n % 4 == 0 && n <= CC_COMM_MAX_ELEMS, "all_reduce_sum_inplace: %lld elements unsupported", (long long)n);
    return submit(dev, LOp{.kind = L_ALLREDUCE, .a = *x, .i0 = n});
}
extern "C" CC_API int cc_all_gather(cc_device* dev, const cc_view* dst, const cc_view* src) {
    CHECK_VIEW(dev, dst, "all_gather dst");
    CHECK_VIEW(dev, src, "all_gather src");
    REQUIRE_F32(dev, dst, "all_gather dst");
    REQUIRE_F32(dev, src, "all_gather src");
    CC_REQUIRE(dev, view_contiguous(dst) && view_contiguous(src), "all_gather: not contiguous");
    CC_REQUIRE(dev, dev->comm, "all_gather: no communicator on this device");
    const int64_t n = view_len(src);
    CC_REQUIRE(dev, view_len(dst) == n * cc_comm_world(dev), "all_gather: dst has %lld elements, want %lld x %d", (long long)view_len(dst), (long long)n, cc_comm_world(dev));
    CC_REQUIRE(dev, n % 4 == 0 && n <= CC_COMM_MAX_ELEMS, "all_gather: %lld elements per rank unsupported", (long long)n);
    return submit(dev, LOp{.kind = L_ALLGATHER, .a = *dst, .b = *src, .i0 = n});
}

// ---- greedy decoding without a host round trip per token (extension: not part of the reference's trait) ---------------------------------
// The sampled token id stays on the device: cc_argmax_to_slot writes it to a slot, the next token's embedding lookup reads it from
// there (cc_copy_rows_from_slot), so the host can submit token t+1 before token t has finished.  sampler.rs:109-116 semantics (the
// LAST maximum).  hist_index >= 0 additionally records the id in the device-side history that cc_read_history copies back.
extern "C" CC_API int cc_argmax_to_slot(cc_device* dev, const cc_view* x, int32_t slot, int64_t hist_index) {
    CHECK_VIEW(dev, x, "argmax_to_slot");
    REQUIRE_F32(dev, x, "argmax_to_slot");
    CC_REQUIRE(dev, view_contiguous(x) && view_len(x) > 0, "argmax_to_slot: tensor must be contiguous and non-empty");
    CC_REQUIRE(dev, slot >= 0 && slot < CC_N_SLOTS && hist_index < CC_HISTORY_CAP, "argmax_to_slot: slot %d / history index %lld out of range", slot, (long long)hist_index);
    int rc = cc_ensure_slots(dev);
    if (rc) return rc;
    return submit(dev, LOp{.kind = L_ARGMAX, .a = *x, .i0 = slot, .i1 = hist_index});
}
// Temperature + top-p sampling into a slot (sampler.rs:27-107; sample_dev.cuh).  coin = 24 bits of splitmix64(seed ^
// splitmix64(coin_index)) / 2^24, so one seed reproduces one run in every mode.  temperature 0 is cc_argmax_to_slot (same op, same bits).
// The logits are not modified.
extern "C" CC_API int cc_sample_to_slot(cc_device* dev, const cc_view* x, float temperature, float topp, uint64_t seed, int64_t coin_index,
                                        int32_t slot, int64_t hist_index) {
    CHECK_VIEW(dev, x, "sample_to_slot");
    REQUIRE_F32(dev, x, "sample_to_slot");
    CC_REQUIRE(dev, view_contiguous(x) && view_len(x) > 0, "sample_to_slot: tensor must be contiguous and non-empty");
    CC_REQUIRE(dev, view_len(x) <= INT32_MAX, "sample_to_slot: %lld logits are too many", (long long)view_len(x));
    CC_REQUIRE(dev, slot >= 0 && slot < CC_N_SLOTS && hist_index < CC_HISTORY_CAP, "sample_to_slot: slot %d / history index %lld out of range", slot, (long long)hist_index);
    CC_REQUIRE(dev, temperature >= 0.0f, "sample_to_slot: temperature %g is not a number >= 0", (double)temperature);
    CC_REQUIRE(dev, topp == topp, "sample_to_slot: topp is NaN");
    if (temperature == 0.0f) return cc_argmax_to_slot(dev, x, slot, hist_index);        // sampler.rs:28-30
    int rc = cc_ensure_slots(dev);
    if (rc) return rc;
    uint32_t pb;
    memcpy(&pb, &topp, 4);
    return submit(dev, LOp{.kind = L_SAMPLE, .a = *x, .f = temperature, .i0 = slot, .i1 = hist_index, .i2 = coin_index, .rows = {(int64_t)seed, (int64_t)pb}});
}
// copy_rows_from with ONE row whose index is the content of a device slot
extern "C" CC_API int cc_copy_rows_from_slot(cc_device* dev, const cc_view* dst, const cc_view* src, int32_t slot) {
    CHECK_VIEW(dev, dst, "copy_rows_from_slot");
    CHECK_VIEW(dev, src, "copy_rows_from_slot src");
    CC_REQUIRE(dev, dst->buf->pooled, "not owned");
    CC_REQUIRE(dev, view_contiguous(dst) && view_contiguous(src), "copy_rows_from_slot: tensors must be contiguous");
    CC_REQUIRE(dev, src->ndim == 2, "copy_rows_from_slot: src tensor is not 2d");
    CC_REQUIRE(dev, slot >= 0 && slot < CC_N_SLOTS, "copy_rows_from_slot: slot %d out of range", slot);
    int dt = dst->buf->dtype;
    CC_REQUIRE(dev, dt == CC_F32 || dt == CC_F16, "only f32/f16 can be copied to");
    int64_t cols = dst->shape[dst->ndim - 1];
    CC_REQUIRE(dev, cols == src->shape[1] && cols <= view_len(dst), "copy_rows_from_slot: row length mismatch");
    CC_REQUIRE(dev, !cc_is_quant(src->buf->dtype) || cols == src->buf->cols, "copy_rows_from_slot: row length does not match the quantized matrix");
    int rc = cc_ensure_slots(dev);
    if (rc) return rc;
    return submit(dev, LOp{.kind = L_COPY_ROWS, .a = *dst, .b = *src, .i2 = slot + 1});
}
extern "C" CC_API int cc_slot_set(cc_device* dev, int32_t slot, int64_t value) {
    if (!dev) return CC_ERR_ARG;
    CC_ENTER(dev);
    CC_REQUIRE(dev, slot >= 0 && slot < CC_N_SLOTS, "slot_set: slot %d out of range", slot);
    int rc = cc_ensure_slots(dev);
    if (rc) return rc;
    FLUSH(dev);
    CC_CUDA(dev, cudaMemcpyAsync(dev->slots + slot, &value, 8, cudaMemcpyHostToDevice, dev->stream));
    CC_CUDA(dev, cudaStreamSynchronize(dev->stream));
    return CC_OK;
}
// synchronises, then copies history[first .. first + count) to the host
extern "C" CC_API int cc_read_history(cc_device* dev, int64_t first, int64_t count, int64_t* out) {
    if (!dev || !out) return CC_ERR_ARG;
    CC_ENTER(dev);
    CC_REQUIRE(dev, first >= 0 && count >= 0 && first + count <= CC_HISTORY_CAP, "read_history: range out of bounds");
    int rc = cc_ensure_slots(dev);
    if (rc) return rc;
    FLUSH(dev);
    if (count) CC_CUDA(dev, cudaMemcpyAsync(out, dev->history + first, (size_t)count * 8, cudaMemcpyDeviceToHost, dev->stream));
    CC_CUDA(dev, cudaStreamSynchronize(dev->stream));
    return cc_check_async_error(dev);
}
// export without waiting: the copy is enqueued behind the work queued so far; `dst` must stay valid (and should be pinned: cc_host_alloc)
// until the next synchronising call
extern "C" CC_API int cc_tensor_export_f32_async(cc_device* dev, const cc_view* src, float* dst, size_t n) {
    CHECK_VIEW(dev, src, "export_async");
    if (!dst) return cc_fail(dev, CC_ERR_ARG, "export_async: dst is NULL");
    REQUIRE_F32(dev, src, "export_async");
    CC_REQUIRE(dev, view_contiguous(src), "export_async: tensor is not contiguous");
    FLUSH(dev);
    int64_t len = view_len(src);
    size_t cnt = n < (size_t)len ? n : (size_t)len;
    if (cnt) CC_CUDA(dev, cudaMemcpyAsync(dst, src->buf->plane[0], cnt * 4, cudaMemcpyDeviceToHost, dev->stream));
    return CC_OK;
}
// pinned host memory for staging (async exports, weight uploads)
extern "C" CC_API int cc_host_alloc(cc_device* dev, size_t bytes, void** out) {
    if (!dev || !out) return CC_ERR_ARG;
    CC_ENTER(dev);
    CC_CUDA(dev, cudaMallocHost(out, bytes ? bytes : 1));
    return CC_OK;
}
extern "C" CC_API void cc_host_free(cc_device* dev, void* p) {
    if (!dev || !p) return;
    CC_ENTER(dev);
    cudaFreeHost(p);
}

// ---- matmul_vec: cpu_tensor.rs:371-386 + primitives/matmul_vec.rs:9-78 -------------------------------------------------
extern "C" CC_API int cc_matmul_vec(cc_device* dev, const cc_view* w, const cc_view* x, cc_buf** out) {
    CHECK_VIEW(dev, w, "matmul_vec");
    CHECK_VIEW(dev, x, "matmul_vec x");
    if (!out) return cc_fail(dev, CC_ERR_ARG, "matmul_vec: out is NULL");
    CC_REQUIRE(dev, w->ndim == 2, "matmul_vec: weight must be 2d");
    CHECK_QUANT_MATRIX(dev, w, "matmul_vec");
    CC_REQUIRE(dev, view_contiguous(w) && view_contiguous(x), "matmul_vec: operands must be contiguous");   // matmul_vec.rs:17-18
    CC_REQUIRE(dev, x->ndim == 1 || x->ndim == 2, "matmul_vec: x must be 1d or 2d");
    CC_REQUIRE(dev, w->shape[1] == x->shape[x->ndim - 1], "matmul_vec: last dims differ (%lld vs %lld)",
               (long long)w->shape[1], (long long)x->shape[x->ndim - 1]);                                  // matmul_vec.rs:19
    REQUIRE_F32(dev, x, "matmul_vec x");
    const int64_t m = w->shape[0], k = w->shape[1], b = x->ndim == 1 ? 1 : x->shape[0];
    const int wt = w->buf->dtype, at = cc_partner_type(wt);
    CC_REQUIRE(dev, at >= 0, "matmul_vec: unsupported weight type %d", wt);
    CC_REQUIRE(dev, k % cc_block_elems(at) == 0, "matmul_vec: k=%lld is not a multiple of the %d-element activation block",
               (long long)k, cc_block_elems(at));
    return submit(dev, LOp{.kind = L_MATVEC, .a = *w, .b = *x}, out, b * m);
}

// ---- batch_matmul: cpu_tensor.rs:352-366 + primitives/batch_matmul.rs:15-45 --------------------------------------------
extern "C" CC_API int cc_batch_matmul(cc_device* dev, const cc_view* a, const cc_view* b, cc_buf** out) {
    CHECK_VIEW(dev, a, "batch_matmul");
    CHECK_VIEW(dev, b, "batch_matmul b");
    if (!out) return cc_fail(dev, CC_ERR_ARG, "batch_matmul: out is NULL");
    CC_REQUIRE(dev, a->ndim == 3 && b->ndim == 3, "batch_matmul: both operands must be 3d");
    CC_REQUIRE(dev, view_contiguous(a), "batch_matmul: lhs must be contiguous");
    CC_REQUIRE(dev, b->strides[1] == 1 || b->strides[2] == 1, "batch_matmul: rhs must be contiguous on k or n");
    REQUIRE_F32(dev, a, "batch_matmul lhs");
    int bt = b->buf->dtype;
    CC_REQUIRE(dev, bt == CC_F32 || bt == CC_F16, "batch_matmul: rhs must be f32/f16");
    const int64_t ab = a->shape[0], m = a->shape[1], k = a->shape[2], bb = b->shape[0], n = b->shape[2];
    CC_REQUIRE(dev, b->shape[1] == k, "batch_matmul: inner dims differ");
    CC_REQUIRE(dev, bb > 0 && ab >= bb && ab % bb == 0, "batch_matmul: lhs batch %lld is not a multiple of rhs batch %lld",
               (long long)ab, (long long)bb);
    return submit(dev, LOp{.kind = L_BMM, .a = *a, .b = *b}, out, ab * m * n);
}

// ---- debug tap: cpu_tensor.rs:232-241 -------------------------------------------------------------------------------------
extern "C" CC_API int cc_debug_tensor_tap(cc_device* dev, const char* name, const cc_view* x) {
    CHECK_VIEW(dev, x, "with_name");
    if (!name) return cc_fail(dev, CC_ERR_ARG, "with_name: name is NULL");
    if (!dev->debug_named_tensors) return CC_OK;
    REQUIRE_F32(dev, x, "with_name");
    FLUSH(dev);
    int64_t n = view_len(x);                     // the reference snapshots the whole buffer; callers tap dense tensors
    std::vector<float> host((size_t)n);
    if (n) CC_CUDA(dev, cudaMemcpyAsync(host.data(), x->buf->plane[0], (size_t)n * 4, cudaMemcpyDeviceToHost, dev->stream));
    CC_CUDA(dev, cudaStreamSynchronize(dev->stream));
    { int rc = cc_check_async_error(dev); if (rc) return rc; }
    dev->debug_tensors[name] = std::move(host);
    return CC_OK;
}
extern "C" CC_API int cc_dump_debug_tensor(cc_device* dev, const char* name, float* dst, size_t* n) {
    if (!dev || !name || !n) return CC_ERR_ARG;
    auto it = dev->debug_tensors.find(name);
    if (it == dev->debug_tensors.end()) return cc_fail(dev, CC_ERR_TENSOR, "no debug tensor named %s", name);
    size_t cnt = it->second.size();
    if (dst) memcpy(dst, it->second.data(), (cnt < *n ? cnt : *n) * 4);
    *n = cnt;
    return CC_OK;
}

// ---- test hook ----------------------------------------------------------------------------------------------------------------
extern "C" CC_API int cc_test_quantize_activation(cc_device* dev, const cc_view* x, int32_t act_type, void* dst, size_t nbytes) {
    CHECK_VIEW(dev, x, "quantize_activation");
    REQUIRE_F32(dev, x, "quantize_activation");
    CC_REQUIRE(dev, view_contiguous(x), "quantize_activation: not contiguous");
    CC_REQUIRE(dev, act_type == CC_Q8_0 || act_type == CC_Q8_1 || act_type == CC_Q8_K, "quantize_activation: bad type");
    int64_t n = view_len(x);
    int be = cc_block_elems(act_type);
    CC_REQUIRE(dev, n % be == 0, "quantize_activation: length %lld %% %d != 0", (long long)n, be);
    size_t need = (size_t)(n / be) * cc_block_bytes(act_type);
    CC_REQUIRE(dev, nbytes >= need, "quantize_activation: %zu bytes given, %zu needed", nbytes, need);
    FLUSH(dev);
    int rc = cc_ensure_act_scratch(dev, cc_act_bytes(act_type, n));
    if (rc) return rc;
    rc = cc_launch_quantize(dev, (const float*)x->buf->plane[0], n, act_type, dev->act_scratch);
    if (rc) return rc;
    uint8_t* blocks = nullptr;
    CC_CUDA(dev, cudaMalloc(&blocks, need ? need : 1));
    rc = cc_launch_act_to_blocks(dev, dev->act_scratch, n, act_type, blocks);
    if (rc == CC_OK) {
        cudaError_t e = cudaMemcpyAsync(dst, blocks, need, cudaMemcpyDeviceToHost, dev->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(dev->stream);
        if (e != cudaSuccess) rc = cc_fail(dev, CC_ERR_CUDA, "quantize_activation: %s", cudaGetErrorString(e));
    }
    cudaFree(blocks);
    return rc;
}
