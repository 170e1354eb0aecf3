// repack.cu -- GGUF AoS blocks <-> device planes, row dequantisation (copy_rows_from), synthetic weights.
//
// Block field orders follow the reference structs (SURVEY Appendix A):
//   Q8_0 buf_q8_0.rs:8-13 | Q4_0 buf_q4_0.rs:10-15 | Q4_1 buf_q4_1.rs:10-16 | Q5_0 buf_q5_0.rs:13-19
//   Q5_1 buf_q5_1.rs:10-17 | Q2_K buf_q2_k.rs:17-28 | Q3_K buf_q3_k.rs:19-30 | Q4_K buf_q4_k.rs:14-21
//   Q5_K ggml order d,dmin,scales,qh,qs (the reference struct buf_q5_k.rs:15-21 is wrong, B9)
//   Q6_K buf_q6_k.rs:11-18 | Q8_K buf_q8_k.rs:6-12
#include "common.cuh"
#include "dequant.cuh"

struct PlaneSpec { int bytes[CC_MAX_PLANES]; int src_off[CC_MAX_PLANES]; int n; };

// per-block bytes of each plane and the offset of that field inside the GGUF block
static PlaneSpec plane_spec(int t) {
    switch (t) {
    case CC_Q8_0: return {{32, 2, 0, 0}, {2, 0, 0, 0}, 2};
    case CC_Q4_0: return {{16, 2, 0, 0}, {2, 0, 0, 0}, 2};
    case CC_Q4_1: return {{16, 4, 0, 0}, {4, 0, 0, 0}, 2};
    case CC_Q5_0: return {{16, 2, 4, 0}, {6, 0, 2, 0}, 3};
    case CC_Q5_1: return {{16, 4, 4, 0}, {8, 0, 4, 0}, 3};
    case CC_Q2_K: return {{64, 16, 4, 0}, {16, 0, 80, 0}, 3};
    case CC_Q3_K: return {{64, 32, 12, 2}, {32, 0, 96, 108}, 4};
    case CC_Q4_K: return {{144, 0, 0, 0}, {0, 0, 0, 0}, 1};
    case CC_Q5_K: return {{176, 0, 0, 0}, {0, 0, 0, 0}, 1};
    case CC_Q6_K: return {{128, 64, 16, 2}, {0, 128, 192, 208}, 4};
    case CC_Q8_K: return {{256, 4, 0, 0}, {4, 0, 0, 0}, 2};     // bsums are activation-only and dropped
    case CC_Q8_1: return {{32, 4, 0, 0}, {4, 0, 0, 0}, 2};
    }
    return {{0, 0, 0, 0}, {0, 0, 0, 0}, 0};
}

static size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

size_t cc_device_layout_bytes(int t, int64_t rows, int64_t cols) {
    PlaneSpec ps = plane_spec(t);
    int64_t nblk = rows * (cols / cc_block_elems(t));
    size_t total = 0;
    for (int p = 0; p < ps.n; p++)
        total += align256(p == 1 && CC_HAS_PADDED_D(t) ? (size_t)rows * CC_D_STRIDE(cols / 32) * 2 : (size_t)nblk * ps.bytes[p]);
    return total ? total : 256;
}

void cc_assign_planes(cc_buf* b) {
    PlaneSpec ps = plane_spec(b->dtype);
    int64_t nblk = b->nelems / cc_block_elems(b->dtype);
    uint8_t* p = (uint8_t*)b->base;
    for (int i = 0; i < ps.n; i++) {
        b->plane[i] = p;
        p += align256(i == 1 && CC_HAS_PADDED_D(b->dtype) ? (size_t)b->rows * CC_D_STRIDE(b->cols / 32) * 2 : (size_t)nblk * ps.bytes[i]);
    }
}

struct RepackArgs {
    uint8_t* plane[CC_MAX_PLANES];
    int bytes[CC_MAX_PLANES];
    int src_off[CC_MAX_PLANES];
    int n;
    int block_bytes;
    int q8_0_nb;          // > 0: plane 0 is the Q8_0 qs plane with `nb` blocks per row -> half-planar groups
    int d_nb;             // > 0: plane 1 is a padded f16 scale plane (CC_D_STRIDE) with `nb` blocks per row
};

template <bool TO_PLANES>
__global__ void repack_kernel(uint8_t* gguf, RepackArgs a, int64_t nblk, int plane) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int pb = a.bytes[plane];
    if (i >= nblk * pb) return;
    int64_t blk = i / pb;
    int j = (int)(i - blk * pb);
    uint8_t* g = gguf + blk * a.block_bytes + a.src_off[plane] + j;
    uint8_t* p = a.plane[plane] + i;
    if (a.q8_0_nb > 0 && plane == 0) {
        int64_t row = blk / a.q8_0_nb;
        int b = (int)(blk - row * a.q8_0_nb);
        p = a.plane[0] + row * a.q8_0_nb * 32 + q8_0_row_offset(b, j, a.q8_0_nb);
    }
    if (a.d_nb > 0 && plane == 1) {
        int64_t row = blk / a.d_nb;
        p = a.plane[1] + (row * CC_D_STRIDE(a.d_nb) + (blk - row * a.d_nb)) * 2 + j;
    }
    if (TO_PLANES) *p = *g; else *g = *p;
}

static RepackArgs make_args(const cc_buf* b) {
    PlaneSpec ps = plane_spec(b->dtype);
    RepackArgs a;
    a.n = ps.n;
    a.block_bytes = (int)cc_block_bytes(b->dtype);
    a.q8_0_nb = b->dtype == CC_Q8_0 ? (int)(b->cols / 32) : 0;
    a.d_nb = CC_HAS_PADDED_D(b->dtype) ? (int)(b->cols / 32) : 0;
    for (int i = 0; i < CC_MAX_PLANES; i++) { a.plane[i] = b->plane[i]; a.bytes[i] = ps.bytes[i]; a.src_off[i] = ps.src_off[i]; }
    return a;
}

int cc_launch_repack(cc_device* dev, const uint8_t* gguf_dev, cc_buf* dst) {
    RepackArgs a = make_args(dst);
    int64_t nblk = dst->nelems / cc_block_elems(dst->dtype);
    for (int p = 0; p < a.n; p++) {
        int64_t total = nblk * a.bytes[p];
        if (total == 0) continue;
        repack_kernel<true><<<(unsigned)((total + 255) / 256), 256, 0, dev->stream>>>((uint8_t*)gguf_dev, a, nblk, p);
        CC_LAUNCH_CHECK(dev);
    }
    return CC_OK;
}

int cc_launch_unrepack(cc_device* dev, const cc_buf* src, uint8_t* gguf_dev) {
    RepackArgs a = make_args(src);
    int64_t nblk = src->nelems / cc_block_elems(src->dtype);
    CC_CUDA(dev, cudaMemsetAsync(gguf_dev, 0, (size_t)nblk * a.block_bytes, dev->stream));
    for (int p = 0; p < a.n; p++) {
        int64_t total = nblk * a.bytes[p];
        if (total == 0) continue;
        repack_kernel<false><<<(unsigned)((total + 255) / 256), 256, 0, dev->stream>>>(gguf_dev, a, nblk, p);
        CC_LAUNCH_CHECK(dev);
    }
    return CC_OK;
}

__global__ void dequant_rows_kernel(int t, DeqPlanes P, const int64_t* rows, int n_rows, int64_t cols,
                                    float* dst_f32, __half* dst_f16) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)n_rows * cols) return;
    int64_t r = i / cols, c = i - r * cols;
    int64_t e = rows[r] * cols + c;
    float v;
    if (t == CC_F32) v = ((const float*)P.p[0])[e];
    else if (t == CC_F16) v = __half2float(((const __half*)P.p[0])[e]);
    else v = dequant_elem(t, P, e);
    if (dst_f32) dst_f32[i] = v; else dst_f16[i] = __float2half_rn(v);
}

int cc_launch_dequant_rows(cc_device* dev, const DeqPlanes& src, int src_dtype, const int64_t* rows_dev, int n_rows, int64_t cols,
                           void* dst, int dst_dtype) {
    int64_t total = (int64_t)n_rows * cols;
    if (total == 0) return CC_OK;
    dequant_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, dev->stream>>>(
        src_dtype, src, rows_dev, n_rows, cols, dst_dtype == CC_F32 ? (float*)dst : nullptr,
        dst_dtype == CC_F16 ? (__half*)dst : nullptr);
    CC_LAUNCH_CHECK(dev);
    return CC_OK;
}

// ---------------------------------------------------------------------------------------------------
// Synthetic weights (SURVEY §8d config 3/4): counter-based splitmix64 over (seed, tensor, byte index)
// written in GGUF block layout, f16 scale fields overwritten with values uniform in [0.75,1.25)*scale.
// oracle/synth.py holds the identical CPU generator (checked bit for bit in tests/test_gpu_synth.py).
// ---------------------------------------------------------------------------------------------------

struct SynthSpec { int n_f16; int off[2]; int is_min[2]; int d_f32_off; };

static SynthSpec synth_spec(int t) {
    switch (t) {
    case CC_Q8_0: case CC_Q4_0: case CC_Q5_0: return {1, {0, 0}, {0, 0}, -1};
    case CC_Q4_1: case CC_Q5_1: return {2, {0, 2}, {0, 1}, -1};
    case CC_Q2_K: return {2, {80, 82}, {0, 1}, -1};
    case CC_Q3_K: return {1, {108, 0}, {0, 0}, -1};
    case CC_Q4_K: case CC_Q5_K: return {2, {0, 2}, {0, 1}, -1};
    case CC_Q6_K: return {1, {208, 0}, {0, 0}, -1};
    case CC_Q8_K: return {0, {0, 0}, {0, 0}, 0};
    }
    return {0, {0, 0}, {0, 0}, -1};
}

__global__ void synth_kernel(uint8_t* out, int64_t nblocks, int bb, SynthSpec sp, uint64_t key, float scale) {
    int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // one thread per 8 output bytes
    int64_t total = nblocks * bb;
    int64_t base = w * 8;
    if (base >= total) return;
    uint64_t r = cc_splitmix64(key ^ (uint64_t)w);
    for (int j = 0; j < 8 && base + j < total; j++) out[base + j] = (uint8_t)(r >> (8 * j));
}
__global__ void synth_scales_kernel(uint8_t* out, int64_t nblocks, int bb, SynthSpec sp, uint64_t key, float scale) {
    int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    uint64_t r = cc_splitmix64(key ^ 0xD1B54A32D192ED03ull ^ (uint64_t)b);
    for (int f = 0; f < sp.n_f16; f++) {
        // uniform in [0.75, 1.25) * scale: plain f32 mul/add only, so oracle/synth.py reproduces it bit for bit
        float u = (float)((r >> (16 * f)) & 0xFFFF) * (1.0f / 65536.0f);
        float v = scale * (0.75f + 0.5f * u);
        if (sp.is_min[f]) v *= 0.25f;
        // 16-bit store (all f16 fields sit at even offsets of even-sized blocks); see quantize.cu on why
        // f16 bits must not be narrowed bytewise
        *reinterpret_cast<__half*>(out + b * bb + sp.off[f]) = __float2half_rn(v);
    }
    if (sp.d_f32_off >= 0) {
        float u = (float)(r & 0xFFFF) * (1.0f / 65536.0f);
        float v = scale * (0.75f + 0.5f * u);
        uint32_t bits = __float_as_uint(v);
        for (int j = 0; j < 4; j++) out[b * bb + sp.d_f32_off + j] = (uint8_t)(bits >> (8 * j));
    }
}

int cc_launch_synth(cc_device* dev, uint8_t* gguf_dev, int t, int64_t nblocks, uint64_t seed, uint64_t tid, float scale) {
    int bb = (int)cc_block_bytes(t);
    SynthSpec sp = synth_spec(t);
    uint64_t key = cc_splitmix64(seed ^ cc_splitmix64(tid));
    int64_t words = (nblocks * bb + 7) / 8;
    synth_kernel<<<(unsigned)((words + 255) / 256), 256, 0, dev->stream>>>(gguf_dev, nblocks, bb, sp, key, scale);
    CC_LAUNCH_CHECK(dev);
    synth_scales_kernel<<<(unsigned)((nblocks + 255) / 256), 256, 0, dev->stream>>>(gguf_dev, nblocks, bb, sp, key, scale);
    CC_LAUNCH_CHECK(dev);
    return CC_OK;
}
