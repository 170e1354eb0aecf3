// exact.cu -- "exact_order" verification mode.
//
// Why it exists: the reference's numerics are chaotic with respect to f32 summation order.  The
// truncating Q8_0 activation quantizer (buf_q8_0.rs:118-125) and the f16 exp LUT (cpu_device.rs:108-115)
// turn 1e-7 perturbations into 1e-3..1e-2 jumps, which compound through the layers: the reference's OWN
// scalar and AVX2 vec_dot orders (buf_q8_0.rs:275-286 vs :228-272) give logits that differ by 1.6-4.1 %
// of max|logit| on the tinyllamas fixture (tests/test_oracle_order_sensitivity.py).  A warp-parallel
// kernel necessarily sums in yet another order, so "logits within 1e-3" is only meaningful against ONE
// fixed order.  This mode evaluates every reduction in the reference's scalar order -- one thread per
// output, sequential loops, GGUF-layout blocks -- so the whole decode is BIT-IDENTICAL to the scalar
// reference path.  It is a proof tool (slow), selected with cc_device_options.exact_order; the fast
// kernels are checked op-by-op against the same oracle within summation-order noise.
//
// Each function cites the reference loop it follows.  File compiled with -fmad=false.
#include "common.cuh"

#pragma pack(push, 1)
struct xq8_0 { uint16_t d; int8_t qs[32]; };
struct xq4_0 { uint16_t d; uint8_t qs[16]; };
struct xq4_1 { uint16_t d, m; uint8_t qs[16]; };
struct xq5_0 { uint16_t d; uint8_t qh[4]; uint8_t qs[16]; };
struct xq5_1 { uint16_t d, m; uint8_t qh[4]; uint8_t qs[16]; };
struct xq8_1 { uint16_t d, s; int8_t qs[32]; };
struct xq2_k { uint8_t scales[16]; uint8_t qs[64]; uint16_t d, dmin; };
struct xq3_k { uint8_t hmask[32]; uint8_t qs[64]; uint8_t scales[12]; uint16_t d; };
struct xq4_k { uint16_t d, dmin; uint8_t scales[12]; uint8_t qs[128]; };
struct xq5_k { uint16_t d, dmin; uint8_t scales[12]; uint8_t qh[32]; uint8_t qs[128]; };
struct xq6_k { uint8_t ql[128]; uint8_t qh[64]; int8_t scales[16]; uint16_t d; };
struct xq8_k { float d; int8_t qs[256]; int16_t bsums[16]; };
#pragma pack(pop)

__device__ __forceinline__ float xh(uint16_t h) { return __half2float(__ushort_as_half(h)); }
__device__ __forceinline__ float xhmul(uint16_t a, uint16_t b) { return __half2float(__float2half_rn(xh(a) * xh(b))); }
__device__ __forceinline__ uint32_t xrd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

__device__ float x_dot_q8_0(const xq8_0* a, const xq8_0* b, int nb) {           // buf_q8_0.rs:275-286
    float sumf = 0.0f;
    for (int i = 0; i < nb; i++) {
        int sumi = 0;
        for (int j = 0; j < 32; j++) sumi += (int)a[i].qs[j] * (int)b[i].qs[j];
        sumf += (float)sumi * xh(a[i].d) * xh(b[i].d);
    }
    return sumf;
}
__device__ float x_dot_q4_0(const xq4_0* a, const xq8_0* b, int nb) {           // buf_q4_0.rs:240-253
    float sumf = 0.0f;
    for (int i = 0; i < nb; i++) {
        int sumi = 0;
        for (int j = 0; j < 16; j++) {
            int v0 = (a[i].qs[j] & 0x0F) - 8, v1 = (a[i].qs[j] >> 4) - 8;
            sumi += v0 * b[i].qs[j] + v1 * b[i].qs[j + 16];
        }
        sumf += (float)sumi * xh(a[i].d) * xh(b[i].d);
    }
    return sumf;
}
__device__ float x_dot_q4_1(const xq4_1* a, const xq8_1* b, int nb) {           // buf_q4_1.rs:266-280
    float sumf = 0.0f;
    for (int i = 0; i < nb; i++) {
        int sumi = 0;
        for (int j = 0; j < 16; j++) sumi += (a[i].qs[j] & 0x0F) * b[i].qs[j] + ((a[i].qs[j] >> 4) & 0x0F) * b[i].qs[j + 16];
        sumf += xhmul(a[i].d, b[i].d) * (float)sumi + xhmul(a[i].m, b[i].s);
    }
    return sumf;
}
__device__ float x_dot_q5_0(const xq5_0* a, const xq8_0* b, int nb) {           // buf_q5_0.rs:145-163
    float sumf = 0.0f;
    for (int i = 0; i < nb; i++) {
        uint32_t qh = xrd32(a[i].qh);
        int sumi = 0;
        for (int j = 0; j < 16; j++) {
            int x0 = (int)((a[i].qs[j] & 0x0F) | (((qh >> j) & 1) << 4)) - 16;
            int x1 = (int)((a[i].qs[j] >> 4) | (((qh >> (j + 16)) & 1) << 4)) - 16;
            sumi += x0 * b[i].qs[j] + x1 * b[i].qs[j + 16];
        }
        sumf += (float)sumi * xh(a[i].d) * xh(b[i].d);
    }
    return sumf;
}
__device__ float x_dot_q5_1(const xq5_1* a, const xq8_1* b, int nb) {           // buf_q5_1.rs:142-161
    float sumf = 0.0f;
    for (int i = 0; i < nb; i++) {
        uint32_t qh = xrd32(a[i].qh);
        int sumi = 0;
        for (int j = 0; j < 16; j++) {
            int x0 = (int)((a[i].qs[j] & 0xF) | (((qh >> j) & 1) << 4));
            int x1 = (int)((a[i].qs[j] >> 4) | (((qh >> (j + 16)) & 1) << 4));
            sumi += x0 * b[i].qs[j] + x1 * b[i].qs[j + 16];
        }
        sumf += (float)sumi * xhmul(a[i].d, b[i].d) + xhmul(a[i].m, b[i].s);
    }
    return sumf;
}
__device__ float x_dot_q2_k(const xq2_k* a, const xq8_k* b, int nb) {           // buf_q2_k.rs:214-257 (i32 summs, B7)
    float sumf = 0.0f;
    for (int i = 0; i < nb; i++) {
        int summs = 0;
        for (int j = 0; j < 16; j++) summs += (int)b[i].bsums[j] * (int)(a[i].scales[j] >> 4);
        float dall = b[i].d * xh(a[i].d), dmin = b[i].d * xh(a[i].dmin);
        int isum = 0, is = 0, q8 = 0, q2 = 0;
        for (int n = 0; n < 2; n++) {
            int shift = 0;
            for (int j = 0; j < 4; j++) {
                int d = a[i].scales[is++] & 0xF, isuml = 0;
                for (int l = 0; l < 16; l++) isuml += (int)b[i].qs[q8 + l] * (int)((a[i].qs[q2 + l] >> shift) & 3);
                isum += d * isuml;
                d = a[i].scales[is++] & 0xF; isuml = 0;
                for (int l = 16; l < 32; l++) isuml += (int)b[i].qs[q8 + l] * (int)((a[i].qs[q2 + l] >> shift) & 3);
                isum += d * isuml;
                shift += 2;
                q8 += 32;
            }
            q2 += 32;
        }
        sumf += dall * (float)isum - dmin * (float)summs;
    }
    return sumf;
}
__device__ void x_q3k_scales(const uint8_t* s12, int8_t* out) {                   // buf_q3_k.rs:286-296
    const uint32_t K1 = 0x03030303u, K2 = 0x0f0f0f0fu;
    uint32_t a0 = xrd32(s12), a1 = xrd32(s12 + 4), tmp = xrd32(s12 + 8);
    uint32_t aux[4];
    aux[2] = ((a0 >> 4) & K2) | (((tmp >> 4) & K1) << 4);
    aux[3] = ((a1 >> 4) & K2) | (((tmp >> 6) & K1) << 4);
    aux[0] = (a0 & K2) | ((tmp & K1) << 4);
    aux[1] = (a1 & K2) | (((tmp >> 2) & K1) << 4);
    for (int i = 0; i < 16; i++) out[i] = (int8_t)((aux[i >> 2] >> (8 * (i & 3))) & 0xFF);
}
__device__ float x_dot_q3_k(const xq3_k* a, const xq8_k* b, int nb) {           // buf_q3_k.rs:240-328
    float sums[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < nb; i++) {
        int aux32[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        int8_t scales[16];
        x_q3k_scales(a[i].scales, scales);
        for (int e = 0; e < 256; e++) {      // element e: half n, shift group s, byte l (same walk as aux_8)
            int n = e >> 7, s = (e >> 5) & 3, l = e & 31;
            int v = (int)((a[i].qs[32 * n + l] >> (2 * s)) & 3) - ((a[i].hmask[l] & (1 << (4 * n + s))) ? 0 : 4);
            int sc = (int)scales[e >> 4] - 32;
            aux32[e & 7] += sc * (int)(int16_t)((int)b[i].qs[e] * v);
        }
        float d = xh(a[i].d) * b[i].d;
        for (int l = 0; l < 8; l++) sums[l] += d * (float)aux32[l];
    }
    float s = sums[0];
    for (int l = 1; l < 8; l++) s += sums[l];
    return s;
}
__device__ void x_k4_scales_mins(const uint8_t* sc12, uint8_t* scales, uint8_t* mins) {   // buf_q4_k.rs:219-234
    const uint32_t K1 = 0x3f3f3f3fu, K2 = 0x0f0f0f0fu, K3 = 0x03030303u;
    uint32_t u0 = xrd32(sc12), u1 = xrd32(sc12 + 4), u2 = xrd32(sc12 + 8);
    uint32_t u3 = ((u2 >> 4) & K2) | (((u1 >> 6) & K3) << 4);
    uint32_t uaux = u1 & K1;
    u1 = (u2 & K2) | (((u0 >> 6) & K3) << 4);
    u2 = uaux;
    u0 &= K1;
    for (int i = 0; i < 4; i++) {
        scales[i] = (u0 >> (8 * i)) & 0xFF; scales[4 + i] = (u1 >> (8 * i)) & 0xFF;
        mins[i] = (u2 >> (8 * i)) & 0xFF; mins[4 + i] = (u3 >> (8 * i)) & 0xFF;
    }
}
// buf_q4_k.rs:192-277 / buf_q5_k.rs:223-319 (ggml field order): per-lane f32 accumulation over blocks
template <bool FIVE>
__device__ float x_dot_q45_k(const void* av, const xq8_k* b, int nb) {
    float sums[8] = {0, 0, 0, 0, 0, 0, 0, 0}, sumf = 0.0f;
    for (int i = 0; i < nb; i++) {
        const uint8_t *qs, *qh = nullptr, *sc;
        uint16_t hd, hdmin;
        if (FIVE) { const xq5_k* a = (const xq5_k*)av + i; qs = a->qs; qh = a->qh; sc = a->scales; hd = a->d; hdmin = a->dmin; }
        else { const xq4_k* a = (const xq4_k*)av + i; qs = a->qs; sc = a->scales; hd = a->d; hdmin = a->dmin; }
        uint8_t scales[8], mins[8];
        x_k4_scales_mins(sc, scales, mins);
        long long sumi = 0;
        for (int j = 0; j < 16; j++) sumi += (int)b[i].bsums[j] * (int)mins[j / 2];
        float aux32[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int e = 0; e < 256; e++) {
            int c = e >> 6, r = e & 63, l = r & 31, hi = r >> 5;
            int q = hi ? (qs[32 * c + l] >> 4) : (qs[32 * c + l] & 0xF);
            if (FIVE) q += (qh[l] & (1 << (2 * c + hi))) ? 16 : 0;
            float scale = (float)scales[e >> 5];
            aux32[e & 7] += scale * (float)(int16_t)((int)b[i].qs[e] * q);      // order: e ascending within each lane l
        }
        float d = xh(hd) * b[i].d;
        for (int l = 0; l < 8; l++) sums[l] += d * aux32[l];
        float dmin = xh(hdmin) * b[i].d;
        sumf -= dmin * (float)sumi;
    }
    for (int l = 0; l < 8; l++) sumf += sums[l];
    return sumf;
}
__device__ float x_dot_q6_k(const xq6_k* a, const xq8_k* b, int nb) {           // buf_q6_k.rs:183-235
    float sums[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < nb; i++) {
        float aux32[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int e = 0; e < 256; e++) {
            int n = e >> 7, r = e & 127, g = r >> 5, l = r & 31;
            const uint8_t* ql = a[i].ql + 64 * n;
            uint8_t qh = a[i].qh[32 * n + l];
            uint8_t lo = (g & 1) ? ql[l + 32] : ql[l];
            int nib = (g >= 2) ? (lo >> 4) : (lo & 0xF);
            int q = (int)(int8_t)((nib | (((qh >> (2 * g)) & 3) << 4)) - 32);
            float scale = (float)a[i].scales[e >> 4];
            aux32[e & 7] += scale * (float)(int16_t)((int)b[i].qs[e] * q);
        }
        float d = xh(a[i].d) * b[i].d;
        for (int l = 0; l < 8; l++) sums[l] += aux32[l] * d;
    }
    float s = 0.0f;
    for (int l = 0; l < 8; l++) s += sums[l];
    return s;
}
__device__ float x_dot_q8_k(const xq8_k* a, const xq8_k* b, int nb) {           // buf_q8_k.rs:213-224
    float sumf = 0.0f;
    for (int i = 0; i < nb; i++) {
        int sumi = 0;
        for (int j = 0; j < 256; j++) sumi += (int)a[i].qs[j] * (int)b[i].qs[j];
        sumf += (float)sumi * a[i].d * b[i].d;
    }
    return sumf;
}

// one thread per output element (bi, row); act = reference-layout activation blocks / f32 / f16
__global__ void matvec_exact_kernel(int t, const uint8_t* w, const uint8_t* act, float* out, int64_t m, int64_t k, int64_t b,
                                    size_t row_bytes, size_t act_row_bytes) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m * b) return;
    int64_t mi = e % m, bi = e / m;
    const uint8_t* wr = w + mi * row_bytes;
    const uint8_t* ar = act + bi * act_row_bytes;
    float r = 0.0f;
    switch (t) {
    case CC_F32: { const float* a = (const float*)wr; const float* x = (const float*)ar; for (int64_t i = 0; i < k; i++) r += a[i] * x[i]; } break;   // buf_f32.rs:19-27
    case CC_F16: { const __half* a = (const __half*)wr; const __half* x = (const __half*)ar; for (int64_t i = 0; i < k; i++) r += __half2float(a[i]) * __half2float(x[i]); } break;
    case CC_Q8_0: r = x_dot_q8_0((const xq8_0*)wr, (const xq8_0*)ar, (int)(k / 32)); break;
    case CC_Q4_0: r = x_dot_q4_0((const xq4_0*)wr, (const xq8_0*)ar, (int)(k / 32)); break;
    case CC_Q4_1: r = x_dot_q4_1((const xq4_1*)wr, (const xq8_1*)ar, (int)(k / 32)); break;
    case CC_Q5_0: r = x_dot_q5_0((const xq5_0*)wr, (const xq8_0*)ar, (int)(k / 32)); break;
    case CC_Q5_1: r = x_dot_q5_1((const xq5_1*)wr, (const xq8_1*)ar, (int)(k / 32)); break;
    case CC_Q2_K: r = x_dot_q2_k((const xq2_k*)wr, (const xq8_k*)ar, (int)(k / 256)); break;
    case CC_Q3_K: r = x_dot_q3_k((const xq3_k*)wr, (const xq8_k*)ar, (int)(k / 256)); break;
    case CC_Q4_K: r = x_dot_q45_k<false>(wr, (const xq8_k*)ar, (int)(k / 256)); break;
    case CC_Q5_K: r = x_dot_q45_k<true>(wr, (const xq8_k*)ar, (int)(k / 256)); break;
    case CC_Q6_K: r = x_dot_q6_k((const xq6_k*)wr, (const xq8_k*)ar, (int)(k / 256)); break;
    case CC_Q8_K: r = x_dot_q8_k((const xq8_k*)wr, (const xq8_k*)ar, (int)(k / 256)); break;
    }
    out[e] = r;
}

int cc_launch_matvec_exact(cc_device* dev, int t, const uint8_t* w_gguf, const uint8_t* act_blocks, float* out,
                           int64_t m, int64_t k, int64_t b) {
    if (m * b == 0) return CC_OK;
    int at = cc_partner_type(t);
    size_t row_bytes = (size_t)(k / cc_block_elems(t)) * cc_block_bytes(t);
    size_t act_row_bytes = (size_t)(k / cc_block_elems(at)) * cc_block_bytes(at);
    matvec_exact_kernel<<<(unsigned)((m * b + 63) / 64), 64, 0, dev->stream>>>(t, w_gguf, act_blocks, out, m, k, b, row_bytes, act_row_bytes);
    CC_LAUNCH_CHECK(dev);
    return CC_OK;
}

// ---- sequential-order small ops -------------------------------------------------------------------------
// rms_norm.rs:32-47: ordered 32-lane chunk sums added to a running scalar
__global__ void rms_norm_exact_kernel(float* x, int64_t cols, float eps) {
    __shared__ float s_rms;
    float* v = x + (int64_t)blockIdx.x * cols;
    if (threadIdx.x == 0) {
        float sum = 0.0f;
        for (int64_t c = 0; c + 32 <= cols; c += 32) {
            float cs = 0.0f;
            for (int l = 0; l < 32; l++) cs += v[c + l] * v[c + l];
            sum += cs;
        }
        s_rms = sqrtf(sum / (float)cols + eps);
    }
    __syncthreads();
    float rms = s_rms;
    for (int64_t i = threadIdx.x; i < cols; i += blockDim.x) v[i] = v[i] / rms;
}
int cc_launch_rms_norm_exact(cc_device* dev, float* x, int64_t rows, int64_t cols, float eps) {
    if (rows == 0 || cols == 0) return CC_OK;
    rms_norm_exact_kernel<<<(unsigned)rows, 128, 0, dev->stream>>>(x, cols, eps);
    CC_LAUNCH_CHECK(dev);
    return CC_OK;
}

// softmax.rs:39-54: sequential sum of the LUT exps
__global__ void softmax_exact_kernel(float* x, int64_t cols, const uint16_t* __restrict__ lut) {
    __shared__ float s_sum;
    float* v = x + (int64_t)blockIdx.x * cols;
    if (threadIdx.x == 0) {
        float m = -INFINITY;
        for (int64_t i = 0; i < cols; i++) m = fmaxf(v[i], m);
        float s = 0.0f;
        for (int64_t i = 0; i < cols; i++) {
            float e = h2f_bits(lut[f2h_bits(v[i] - m)]);
            v[i] = e;
            s += e;
        }
        s_sum = s;
    }
    __syncthreads();
    float s = s_sum;
    for (int64_t i = threadIdx.x; i < cols; i += blockDim.x) v[i] = v[i] / s;
}
int cc_launch_softmax_exact(cc_device* dev, float* x, int64_t rows, int64_t cols) {
    if (rows == 0 || cols == 0) return CC_OK;
    softmax_exact_kernel<<<(unsigned)rows, 64, 0, dev->stream>>>(x, cols, dev->exp_lut);
    CC_LAUNCH_CHECK(dev);
    return CC_OK;
}

// rope with HOST-evaluated cos/sin (glibc cosf/sinf, exactly what the reference calls): rope.rs:47-80
// The base is 10000 in both modes, whatever a model file says (rope.rs:48,69 hard-code it; a GGUF `rope.freq_base` is not read):
// llama: theta_j = pos * scale^j by the running product (rope.rs:48-53); neox: theta_j = pos / 10000^(2j / head_dim), one powf per j
// (rope.rs:66-79).
void cc_rope_table(int mode, int64_t pos, int64_t head_dim, int pairs, float* cos_out, float* sin_out) {
    const float fpos = (float)pos;
    if (mode == CC_ROPE_LLAMA) {
        float theta_scale = powf(10000.0f, -2.0f / (float)head_dim), theta = fpos;
        for (int j = 0; j < pairs; j++) { cos_out[j] = cosf(theta); sin_out[j] = sinf(theta); theta *= theta_scale; }
    } else {
        for (int j = 0; j < pairs; j++) {
            float timescale = powf(10000.0f, 2.0f * (float)j / (float)head_dim);
            float theta = fpos / timescale;
            cos_out[j] = cosf(theta); sin_out[j] = sinf(theta);
        }
    }
}
struct RopeTable { float c[128], s[128]; };
__global__ void rope_table_kernel(float* row, int64_t heads, int head_dim, int mode, int pairs, RopeTable tb) {
    int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= heads * pairs) return;
    int j = (int)(idx % pairs);
    float* c = row + (idx / pairs) * head_dim;
    int i0 = mode == CC_ROPE_LLAMA ? 2 * j : j, i1 = mode == CC_ROPE_LLAMA ? 2 * j + 1 : j + head_dim / 2;
    float q0 = c[i0], q1 = c[i1];
    c[i0] = q0 * tb.c[j] - q1 * tb.s[j];
    c[i1] = q0 * tb.s[j] + q1 * tb.c[j];
}
int cc_launch_rope_exact(cc_device* dev, float* x, int64_t n_batch, int64_t batch_stride, int64_t head_dim, int mode,
                         int64_t pos, int64_t rope_dim) {
    int pairs = (int)(rope_dim / 2);
    CC_REQUIRE(dev, pairs <= 128, "rope_inplace(exact): rope_dims %lld > 256", (long long)rope_dim);
    if (pairs == 0) return CC_OK;
    int64_t heads = batch_stride / head_dim;
    for (int64_t bi = 0; bi < n_batch; bi++) {
        RopeTable tb;
        cc_rope_table(mode, pos + bi, head_dim, pairs, tb.c, tb.s);
        int64_t total = heads * pairs;
        rope_table_kernel<<<(unsigned)((total + 127) / 128), 128, 0, dev->stream>>>(x + bi * batch_stride, heads, (int)head_dim, mode, pairs, tb);
        CC_LAUNCH_CHECK(dev);
    }
    return CC_OK;
}

// batch_matmul.rs:47-71 / :97-105: k innermost, sequential, one thread per output (B contiguous on k)
template <bool B_F16>
__global__ void bmm_kcontig_exact_kernel(const float* __restrict__ a, const void* __restrict__ b, float* __restrict__ c,
                                         int64_t ab, int64_t bb, int64_t m, int64_t k, int64_t n, int64_t sb0, int64_t sb2) {
    int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= ab * m * n) return;
    int64_t ni = o % n, mi = (o / n) % m, bi = o / (m * n);
    const float* pa = a + bi * (m * k) + mi * k;
    float acc = 0.0f;
    if (B_F16) {
        const __half* pb = (const __half*)b + (bi / (ab / bb)) * sb0 + ni * sb2;
        for (int64_t ki = 0; ki < k; ki++) acc += __half2float(__float2half_rn(pa[ki])) * __half2float(pb[ki]);
    } else {
        const float* pb = (const float*)b + (bi % bb) * sb0 + ni * sb2;
        for (int64_t ki = 0; ki < k; ki++) acc += pa[ki] * pb[ki];
    }
    c[o] = acc;
}
int cc_launch_bmm_kcontig_exact(cc_device* dev, const float* a, const void* b, int b_dtype, float* c, int64_t ab, int64_t bb,
                                int64_t m, int64_t k, int64_t n, int64_t sb0, int64_t sb2) {
    int64_t outs = ab * m * n;
    if (outs == 0) return CC_OK;
    unsigned grid = (unsigned)((outs + 127) / 128);
    if (b_dtype == CC_F16) bmm_kcontig_exact_kernel<true><<<grid, 128, 0, dev->stream>>>(a, b, c, ab, bb, m, k, n, sb0, sb2);
    else bmm_kcontig_exact_kernel<false><<<grid, 128, 0, dev->stream>>>(a, b, c, ab, bb, m, k, n, sb0, sb2);
    CC_LAUNCH_CHECK(dev);
    return CC_OK;
}
