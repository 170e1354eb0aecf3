// quantize.cu -- on-the-fly activation quantisation (SURVEY §8a rows a3-a5).
//   Q8_0: buf_q8_0.rs:87-134   d = max|x|/127 (f32), q = trunc(x / d)   (TRUNCATION, quirk B1)
//   Q8_1: buf_q8_1.rs:90-129   q = trunc(clamp(x/d,-128,127)), s = d * sum(q) stored f16
//   Q8_K: buf_q8_k.rs:84-131   scale = -128/max_signed, q = min(round_half_away(scale*x),127), d = 1/scale
// Compiled with -fmad=false and IEEE division: results are bit-identical to the reference.
#include "common.cuh"
#include "quantize_dev.cuh"

static size_t al16(size_t v) { return (v + 15) & ~(size_t)15; }

size_t cc_act_bytes(int t, int64_t n) {
    switch (t) {
    case CC_Q8_0: return al16(n) + al16(n / 32 * 4) + al16(n / 32 * 4);
    case CC_Q8_1: return al16(n) + al16(n / 32 * 4);
    case CC_Q8_K: return al16(n) + al16(n / 256 * 4) + al16(n / 16 * 2);
    case CC_F16: return al16(n * 2);
    case CC_F32: return 0;
    }
    return 0;
}
ActQ8_0 cc_act_q8_0(void* s, int64_t n) {
    uint8_t* p = (uint8_t*)s;
    ActQ8_0 a;
    a.qs = (int8_t*)p; p += al16(n);
    a.d = (float*)p; p += al16(n / 32 * 4);
    a.isum = (int32_t*)p;
    return a;
}
ActQ8_1 cc_act_q8_1(void* s, int64_t n) {
    uint8_t* p = (uint8_t*)s;
    ActQ8_1 a;
    a.qs = (int8_t*)p; p += al16(n);
    a.ds = (__half2*)p;
    return a;
}
ActQ8_K cc_act_q8_k(void* s, int64_t n) {
    uint8_t* p = (uint8_t*)s;
    ActQ8_K a;
    a.qs = (int8_t*)p; p += al16(n);
    a.d = (float*)p; p += al16(n / 256 * 4);
    a.bsums = (int16_t*)p;
    return a;
}

// one warp per 32-element block, lane = element
__global__ void quantize_q8_0_kernel(const float* __restrict__ x, int64_t nblocks, ActQ8_0 a) {
    int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (b >= nblocks) return;
    float v = x[b * 32 + lane];
    float amax = warp_max(fabsf(v));
    float d = amax / 127.0f;
    int q = __float2int_rz(v / d);          // NaN (0/0) -> 0, like Rust's `as i32`
    a.qs[b * 32 + lane] = (int8_t)q;
    int s = warp_sum_i((int)(int8_t)q);
    if (lane == 0) {
        a.d[b] = __half2float(__float2half_rn(d));
        a.isum[b] = s;
    }
}

__global__ void quantize_q8_1_kernel(const float* __restrict__ x, int64_t nblocks, ActQ8_1 a) {
    int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (b >= nblocks) return;
    float v = x[b * 32 + lane];
    float amax = warp_max(fabsf(v));
    float d = amax / 127.0f;
    float sv = v / d;
    // Rust: scaled.max(-128.0).min(127.0) as i8 ; fmaxf/fminf return the non-NaN operand like f32::max/min
    int q = __float2int_rz(fminf(fmaxf(sv, -128.0f), 127.0f));
    a.qs[b * 32 + lane] = (int8_t)q;
    int s = warp_sum_i(q);                  // |sum| <= 4096: exact in f32 in any order
    if (lane == 0) a.ds[b] = __halves2half2(__float2half_rn(d), __float2half_rn((float)s * d));
}

// one warp per 256-element super-block; lane handles elements lane*8 .. lane*8+7 (cc_quant_q8k_sblock, quantize_dev.cuh)
__global__ void quantize_q8_k_kernel(const float* __restrict__ x, int64_t nsb, ActQ8_K a) {
    int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (b >= nsb) return;
    const float* xb = x + b * 256 + lane * 8;
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = xb[i];
    cc_quant_q8k_sblock(v, lane, a.qs + b * 256, a.d + b, a.bsums + b * 16);
}

__global__ void quantize_f16_kernel(const float* __restrict__ x, int64_t n, __half* out) {   // buf/api.rs:198
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = __float2half_rn(x[i]);
}

int cc_launch_quantize(cc_device* dev, const float* x, int64_t n, int act_type, void* scratch) {
    switch (act_type) {
    case CC_Q8_0: {
        CC_REQUIRE(dev, n % 32 == 0, "quantize q8_0: length %lld %% 32 != 0", (long long)n);
        int64_t nb = n / 32;
        if (nb == 0) return CC_OK;
        quantize_q8_0_kernel<<<(unsigned)((nb + 7) / 8), 256, 0, dev->stream>>>(x, nb, cc_act_q8_0(scratch, n));
        break;
    }
    case CC_Q8_1: {
        CC_REQUIRE(dev, n % 32 == 0, "quantize q8_1: length %lld %% 32 != 0", (long long)n);
        int64_t nb = n / 32;
        if (nb == 0) return CC_OK;
        quantize_q8_1_kernel<<<(unsigned)((nb + 7) / 8), 256, 0, dev->stream>>>(x, nb, cc_act_q8_1(scratch, n));
        break;
    }
    case CC_Q8_K: {
        CC_REQUIRE(dev, n % 256 == 0, "quantize q8_k: length %lld %% 256 != 0", (long long)n);
        int64_t nb = n / 256;
        if (nb == 0) return CC_OK;
        quantize_q8_k_kernel<<<(unsigned)((nb + 7) / 8), 256, 0, dev->stream>>>(x, nb, cc_act_q8_k(scratch, n));
        break;
    }
    case CC_F16:
        if (n == 0) return CC_OK;
        quantize_f16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, dev->stream>>>(x, n, (__half*)scratch);
        break;
    default:
        return cc_fail(dev, CC_ERR_TENSOR, "quantize to type %d is not supported", act_type);
    }
    CC_LAUNCH_CHECK(dev);
    return CC_OK;
}

// reassemble reference-layout blocks (for cc_test_quantize_activation): one thread per block
__global__ void act_to_blocks_kernel(int t, const void* scratch, int64_t n, uint8_t* out,
                                     ActQ8_0 a0, ActQ8_1 a1, ActQ8_K ak) {
    int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t == CC_Q8_0) {
        if (b >= n / 32) return;
        uint8_t* o = out + b * 34;
        // 16-bit store on purpose: ptxas 12.9 folds `cvt.rn.f16.f32` + a truncating byte store into a
        // NUMERIC F2I.U8.F16 (observed with ptxas 12.9 for sm_100a), so never narrow f16 bits with `& 0xFF`.
        *reinterpret_cast<__half*>(o) = __float2half_rn(a0.d[b]);
        for (int i = 0; i < 32; i++) o[2 + i] = (uint8_t)a0.qs[b * 32 + i];
    } else if (t == CC_Q8_1) {
        if (b >= n / 32) return;
        uint8_t* o = out + b * 36;
        *reinterpret_cast<__half2*>(o) = a1.ds[b];
        for (int i = 0; i < 32; i++) o[4 + i] = (uint8_t)a1.qs[b * 32 + i];
    } else {
        if (b >= n / 256) return;
        uint8_t* o = out + b * 292;
        uint32_t bits = __float_as_uint(ak.d[b]);
        for (int j = 0; j < 4; j++) o[j] = (uint8_t)(bits >> (8 * j));
        for (int i = 0; i < 256; i++) o[4 + i] = (uint8_t)ak.qs[b * 256 + i];
        for (int i = 0; i < 16; i++) {
            uint16_t v = (uint16_t)ak.bsums[b * 16 + i];
            o[260 + 2 * i] = v & 0xFF; o[261 + 2 * i] = v >> 8;
        }
    }
}

int cc_launch_act_to_blocks(cc_device* dev, const void* scratch, int64_t n, int t, uint8_t* blocks_dev) {
    int64_t nb = n / (t == CC_Q8_K ? 256 : 32);
    if (nb == 0) return CC_OK;
    act_to_blocks_kernel<<<(unsigned)((nb + 127) / 128), 128, 0, dev->stream>>>(
        t, scratch, n, blocks_dev, cc_act_q8_0((void*)scratch, n), cc_act_q8_1((void*)scratch, n), cc_act_q8_k((void*)scratch, n));
    CC_LAUNCH_CHECK(dev);
    return CC_OK;
}
