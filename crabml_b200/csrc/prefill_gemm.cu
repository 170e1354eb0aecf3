// prefill_gemm.cu -- the dense (prefill) path of matmul_vec: C[b, m] = sum_k W[m, k] * x[b, k] for a BATCH of activation rows
// (Tensor::matmul_vec with a (b, k) rhs: cpu_tensor.rs:368-386, primitives/matmul_vec.rs:26-78; the prompt walk of
// llama2.rs:111-139).  With b >= 32 rows the contraction is genuinely dense, so it runs on the Hopper tensor cores (wgmma):
//
//   1. dequant_w_f16_kernel : GGUF quant blocks (device plane layout, any of the 11 weight types) -> f16 tile source [m][k], ONCE per
//      weight (kept beside the quantised planes: a 7B model's 13-14 GB of f16 fit in 80 GB of HBM next to its quantised weights)
//      (w = f32 dequantised value as BlockQ*::dequantize gives it, rounded once to f16: |q| <= 127 times an f16 scale)
//   2. act_f32_to_q8f16_kernel / act_q8k_to_f16_kernel : the activation is quantised exactly like the decode path, to Q8_0
//      (buf_q8_0.rs:87-134) or, for K-quant weights, to Q8_K (buf_q8_k.rs:84-131), and the quantised value q * d is what enters the
//      GEMM, so the only deviation from the reference is the f16 rounding of the two operands (relative 2^-11 each) and the f32
//      accumulation order.  A row whose largest |q * d| reaches 2^15 would overflow f16 (127 * f16(65504 / 127) rounds to +inf);
//      it enters scaled by a power of two 2^-e (the smallest e that brings it below 2^15), and the epilogue multiplies its outputs
//      by 2^e.  Rows in range have e = 0: the multiply by 1.0f is exact and changes no bit
//   3. wgmma_gemm_kernel    : TMA (cp.async.bulk.tensor.2d, 128-byte swizzle) stages [128 x 64] / [N x 64] f16 tiles into a
//      4-deep shared-memory ring; two consumer warpgroups each own 64 weight rows and issue
//      wgmma.mma_async.m64n64k16.f32.f16.f16 (N / 64 per 16-wide K step) with the f32 accumulator in registers, then store
//      C[b][m] straight from those registers.  Warpgroup roles: 0 TMA producer (one thread), 1-2 MMA + epilogue.
// MMA-M is the WEIGHT row dimension (large: 4096 .. 32000), MMA-N the batch dimension.
// Every mbarrier wait is bounded (trap after ~2 s) so that a descriptor mistake ends in an error, not a hung GPU.
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "dequant.cuh"

#define PG_BLOCK_M 128                    // 2 consumer warpgroups x 64 rows
#define PG_BLOCK_K 64                     // 64 f16 = 128 bytes = one swizzle-128B row
#define PG_STAGES 4
#define PG_THREADS 384                    // 3 warpgroups
#define PG_MMA_K 16

// ---- PTX helpers ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned pg_smem(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void pg_mbar_init(unsigned bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void pg_mbar_expect_tx(unsigned bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void pg_mbar_arrive(unsigned bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void pg_mbar_wait(unsigned bar, unsigned parity) {
    unsigned done = 0;
    for (unsigned it = 0; !done; it++) {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (it > (1u << 26)) __trap();          // bounded: a pipeline bug must not hang the GPU
    }
}
__device__ __forceinline__ void pg_tma_load_2d(unsigned dst, const void* tmap, unsigned bar, int x, int y) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(tmap), "r"(bar), "r"(x), "r"(y) : "memory");
}
// shared-memory matrix descriptor of a K-major tile stored as rows of 128 bytes with the 128-byte swizzle (what the TMA box
// {64 x rows} with CU_TENSOR_MAP_SWIZZLE_128B writes): 8-row groups are 1024 bytes apart (stride byte offset), the leading byte
// offset is unused for swizzled K-major operands, layout type 1 = SWIZZLE_128B (sm_90 encoding).  Tiles start 1024-aligned, so the
// base offset is 0.
__device__ __forceinline__ uint64_t pg_smem_desc(unsigned smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);                  // bits [0, 14): start address >> 4
    d |= (uint64_t)1 << 16;                                       // bits [16, 30): leading byte offset >> 4 (unused)
    d |= (uint64_t)(1024 >> 4) << 32;                             // bits [32, 46): stride byte offset >> 4
    d |= (uint64_t)1 << 62;                                       // bits [62, 64): SWIZZLE_128B
    return d;
}
__device__ __forceinline__ void pg_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void pg_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void pg_wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T, both K-major in shared memory, f16 inputs, f32 accumulator in registers (the warpgroup's
// 128 threads hold 32 values each); issued by the whole warpgroup
__device__ __forceinline__ void pg_wgmma_64x64(float (&d)[32], uint64_t desc_a, uint64_t desc_b, int accumulate) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

struct PgShared {
    unsigned long long full[PG_STAGES], empty[PG_STAGES];
};

// grid: (ceil(m / 128), ceil(b / BLOCK_N)); dynamic smem: 1024-aligned ring of PG_STAGES x (A tile 16 KB + B tile BLOCK_N * 128 B),
// at most 4 x 48 KB.  The accumulator of a consumer warpgroup is BLOCK_N / 2 registers per thread (128 at BLOCK_N = 256).
// row_scale[b]: 2^e of each activation row (the inverse of the scale its f16 operand was taken at; 1.0 for rows in f16 range).
template <int BLOCK_N>
__global__ void __launch_bounds__(PG_THREADS, 1) wgmma_gemm_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                                                                   const float* __restrict__ row_scale, float* __restrict__ C, int m, int b, int k) {
    extern __shared__ __align__(1024) uint8_t pg_smem_raw[];
    __shared__ PgShared sh;
    const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
    constexpr unsigned A_BYTES = PG_BLOCK_M * PG_BLOCK_K * 2, B_BYTES = BLOCK_N * PG_BLOCK_K * 2, STAGE = A_BYTES + B_BYTES;
    constexpr int NJ = BLOCK_N / 64;
    uint8_t* ring = (uint8_t*)(((uintptr_t)pg_smem_raw + 1023) & ~(uintptr_t)1023);
    const int num_kb = k / PG_BLOCK_K;
    const int m0 = blockIdx.x * PG_BLOCK_M, n0 = blockIdx.y * BLOCK_N;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_w) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_x) : "memory");
        for (int s = 0; s < PG_STAGES; s++) { pg_mbar_init(pg_smem(&sh.full[s]), 1); pg_mbar_init(pg_smem(&sh.empty[s]), 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wg == 0) {
        // ===== TMA producer: a single thread =====
        if (t == 0) {
            for (int kb = 0; kb < num_kb; kb++) {
                const int s = kb % PG_STAGES;
                const unsigned ph = (unsigned)(kb / PG_STAGES) & 1u;
                pg_mbar_wait(pg_smem(&sh.empty[s]), ph ^ 1u);           // slot free (passes at once on the first round)
                const unsigned full = pg_smem(&sh.full[s]);
                pg_mbar_expect_tx(full, STAGE);
                uint8_t* st = ring + (size_t)s * STAGE;
                pg_tma_load_2d(pg_smem(st), &tmap_w, full, kb * PG_BLOCK_K, m0);
                pg_tma_load_2d(pg_smem(st + A_BYTES), &tmap_x, full, kb * PG_BLOCK_K, n0);
            }
        }
        return;
    }
    // ===== consumers: warpgroup c = wg - 1 owns weight rows m0 + 64 c .. m0 + 64 c + 63 =====
    const int c = wg - 1;
    float acc[NJ][32];
#pragma unroll
    for (int j = 0; j < NJ; j++)
#pragma unroll
        for (int i = 0; i < 32; i++) acc[j][i] = 0.0f;
    for (int kb = 0; kb < num_kb; kb++) {
        const int s = kb % PG_STAGES;
        const unsigned ph = (unsigned)(kb / PG_STAGES) & 1u;
        pg_mbar_wait(pg_smem(&sh.full[s]), ph);                          // TMA landed this stage
        uint8_t* st = ring + (size_t)s * STAGE;
        const uint64_t da = pg_smem_desc(pg_smem(st + c * 64 * 128));
        const uint64_t db = pg_smem_desc(pg_smem(st + A_BYTES));
        pg_wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < PG_BLOCK_K / PG_MMA_K; kk++) {
            // advancing K inside the 128-byte swizzle atom = advancing the (pre-swizzle) start address by 32 bytes
            const uint64_t adv = (uint64_t)((kk * PG_MMA_K * 2) >> 4);
#pragma unroll
            for (int j = 0; j < NJ; j++) pg_wgmma_64x64(acc[j], da + adv, db + (uint64_t)((j * 64 * 128) >> 4) + adv, 1);
        }
        pg_wgmma_commit();
        pg_wgmma_wait<1>();                                              // the MMAs of stage kb - 1 have read their operands
        if (kb > 0 && t == 0) pg_mbar_arrive(pg_smem(&sh.empty[(kb - 1) % PG_STAGES]));
    }
    pg_wgmma_wait<0>();
    // ===== epilogue: registers -> C[b][m].  wgmma's f32 layout: thread t of the warpgroup holds, for column chunk j and i = 0..31,
    // row 16 (t / 32) + (t % 32) / 4 + 8 ((i / 2) % 2), column 64 j + 8 (i / 4) + 2 (t % 4) + i % 2.
    const int r0 = m0 + c * 64 + 16 * (t >> 5) + ((t & 31) >> 2);
#pragma unroll
    for (int j = 0; j < NJ; j++)
#pragma unroll
        for (int i = 0; i < 32; i++) {
            const int row = r0 + 8 * ((i >> 1) & 1), bi = n0 + 64 * j + 8 * (i >> 2) + 2 * (t & 3) + (i & 1);
            if (row < m && bi < b) C[(size_t)bi * m + row] = acc[j][i] * row_scale[bi];
        }
}

// ---- operand preparation ---------------------------------------------------------------------------------------------------------
// weights: device plane layout -> f16 [m][k]; one thread per 2 elements
__global__ void dequant_w_f16_kernel(int dtype, DeqPlanes planes, int64_t nelems, __half* __restrict__ out) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 2;
    if (i >= nelems) return;
    float a, b2;
    if (dtype == CC_F32) { a = ((const float*)planes.p[0])[i]; b2 = ((const float*)planes.p[0])[i + 1]; }
    else if (dtype == CC_F16) { a = __half2float(((const __half*)planes.p[0])[i]); b2 = __half2float(((const __half*)planes.p[0])[i + 1]); }
    else { a = dequant_elem(dtype, planes, i); b2 = dequant_elem(dtype, planes, i + 1); }
    *(__half2*)(out + i) = __halves2half2(__float2half_rn(a), __float2half_rn(b2));
}
// Activation rows -> f16 GEMM operand, one CTA of PG_ACT_THREADS per batch row.  The row is converted as if in f16 range and its
// largest |q * d| is reduced on the way; only a row at or above 2^15 is converted a second time, at 2^-e (pg_row_exp), so an in-range
// row is read once, as before.  row_scale[row] = 2^e undoes the scale in the GEMM's epilogue.
#define PG_ACT_THREADS 256
// the smallest e >= 0 with amax * 2^-e < 2^15 (amax = f * 2^x, f in [0.5, 1): e = x - 15); 0 for non-finite amax, which no scale helps
__device__ __forceinline__ int pg_row_exp(float amax) {
    int x = 0;
    if (amax >= 32768.0f && amax <= 3.402823466e38f) { frexpf(amax, &x); x -= 15; }
    return x;
}
__device__ __forceinline__ float pg_cta_max(float v) {
    __shared__ float red[PG_ACT_THREADS / 32];
    v = warp_max(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    v = red[0];
#pragma unroll
    for (int i = 1; i < PG_ACT_THREADS / 32; i++) v = fmaxf(v, red[i]);
    return v;
}
__device__ __forceinline__ uint2 pg_pack4_f16(float a0, float a1, float a2, float a3, float s) {
    __half2 h0 = __halves2half2(__float2half_rn(a0 * s), __float2half_rn(a1 * s)), h1 = __halves2half2(__float2half_rn(a2 * s), __float2half_rn(a3 * s));
    return make_uint2(*(unsigned*)&h0, *(unsigned*)&h1);
}

// Q8_0 partners: f32 activation rows -> f16(q * d), quantised on the way (what quantize_q8_0_kernel computes, same arithmetic:
// d = max|x| / 127, q = trunc(x / d), stored scale f32(f16(d)); buf_q8_0.rs:87-134).  A lane takes 4 elements, 8 lanes one 32-element
// block.  k % 64 == 0, so the bound check is uniform across each 8-lane group.
__device__ __forceinline__ void pg_q8_0_4(const float4* __restrict__ xr, int i, bool ok, float (&a)[4]) {
    const float4 v = ok ? xr[i] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    float amax = fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)));
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float d = amax / 127.0f;
    const float d16 = __half2float(__float2half_rn(d));
    const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; j++) a[j] = (float)(int)(int8_t)__float2int_rz(vv[j] / d) * d16;        // NaN (0 / 0) -> 0
}
__global__ void __launch_bounds__(PG_ACT_THREADS) act_f32_to_q8f16_kernel(const float* __restrict__ x, int k, __half* __restrict__ out, float* __restrict__ row_scale) {
    const int n4 = k / 4, lane = threadIdx.x & 31, w0 = (threadIdx.x >> 5) * 32;
    const float4* xr = (const float4*)(x + (size_t)blockIdx.x * k);
    uint2* orow = (uint2*)(out + (size_t)blockIdx.x * k);
    float vmax = 0.0f;
    for (int base = w0; base < n4; base += PG_ACT_THREADS) {
        const int i = base + lane;
        float a[4];
        pg_q8_0_4(xr, i, i < n4, a);
        if (i < n4) orow[i] = pg_pack4_f16(a[0], a[1], a[2], a[3], 1.0f);
        vmax = fmaxf(vmax, fmaxf(fmaxf(fabsf(a[0]), fabsf(a[1])), fmaxf(fabsf(a[2]), fabsf(a[3]))));
    }
    const int e = pg_row_exp(pg_cta_max(vmax));
    if (threadIdx.x == 0) row_scale[blockIdx.x] = ldexpf(1.0f, e);
    if (e == 0) return;
    const float s = ldexpf(1.0f, -e);
    for (int base = w0; base < n4; base += PG_ACT_THREADS) {
        const int i = base + lane;
        float a[4];
        pg_q8_0_4(xr, i, i < n4, a);
        if (i < n4) orow[i] = pg_pack4_f16(a[0], a[1], a[2], a[3], s);
    }
}

// K-quant partners: Q8_K SoA (qs, f32 d per 256; buf_q8_k.rs:84-131) -> f16(q * d); a thread takes 4 quants per step
__global__ void __launch_bounds__(PG_ACT_THREADS) act_q8k_to_f16_kernel(ActQ8_K act, int k, __half* __restrict__ out, float* __restrict__ row_scale) {
    const int n4 = k / 4;
    const char4* qr = (const char4*)(act.qs + (size_t)blockIdx.x * k);
    const float* dr = act.d + (size_t)blockIdx.x * (k / 256);
    uint2* orow = (uint2*)(out + (size_t)blockIdx.x * k);
    float vmax = 0.0f;
    for (int i = threadIdx.x; i < n4; i += PG_ACT_THREADS) {
        const char4 q = qr[i];
        const float d = dr[i >> 6];
        const float a0 = (float)q.x * d, a1 = (float)q.y * d, a2 = (float)q.z * d, a3 = (float)q.w * d;
        orow[i] = pg_pack4_f16(a0, a1, a2, a3, 1.0f);
        vmax = fmaxf(vmax, fmaxf(fmaxf(fabsf(a0), fabsf(a1)), fmaxf(fabsf(a2), fabsf(a3))));
    }
    const int e = pg_row_exp(pg_cta_max(vmax));
    if (threadIdx.x == 0) row_scale[blockIdx.x] = ldexpf(1.0f, e);
    if (e == 0) return;
    const float s = ldexpf(1.0f, -e);
    for (int i = threadIdx.x; i < n4; i += PG_ACT_THREADS) {
        const char4 q = qr[i];
        const float d = dr[i >> 6];
        orow[i] = pg_pack4_f16((float)q.x * d, (float)q.y * d, (float)q.z * d, (float)q.w * d, s);
    }
}

// ---- host side ------------------------------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled pg_encode() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess) fn = (PFN_encodeTiled)p;
    }
    return fn;
}
// f16 matrix [rows][k] (k contiguous), box = 64 columns x box_rows rows, 128-byte swizzle, out-of-bounds rows read as zero
static int pg_make_tmap(cc_device* dev, CUtensorMap* tm, const void* base, int64_t rows, int64_t k, int box_rows) {
    PFN_encodeTiled enc = pg_encode();
    if (!enc) return cc_fail(dev, CC_ERR_CUDA, "prefill: cuTensorMapEncodeTiled is not available from this driver");
    cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)k * 2};
    cuuint32_t box[2] = {PG_BLOCK_K, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return cc_fail(dev, CC_ERR_CUDA, "prefill: cuTensorMapEncodeTiled failed (%d)", (int)r);
    return CC_OK;
}

struct PgScratch { void* w = nullptr; size_t w_bytes = 0; void* x = nullptr; size_t x_bytes = 0; };
static PgScratch* pg_scratch(cc_device* dev) {
    static std::mutex mu;
    static std::map<cc_device*, PgScratch> tab;
    std::lock_guard<std::mutex> g(mu);
    return &tab[dev];
}
static int pg_ensure(cc_device* dev, void** p, size_t* cap, size_t need) {
    if (need <= *cap) return CC_OK;
    if (*p) { CC_CUDA(dev, cudaStreamSynchronize(dev->stream)); CC_CUDA(dev, cudaFree(*p)); *p = nullptr; *cap = 0; }
    size_t c = (need + ((size_t)1 << 20) - 1) & ~(((size_t)1 << 20) - 1);
    CC_CUDA(dev, cudaMalloc(p, c));
    *cap = c;
    return CC_OK;
}
void cc_prefill_release(cc_device* dev) {
    PgScratch* s = pg_scratch(dev);
    if (s->w) cudaFree(s->w);
    if (s->x) cudaFree(s->x);
    s->w = s->x = nullptr; s->w_bytes = s->x_bytes = 0;
}

bool cc_prefill_supported(int wtype, int64_t m, int64_t k, int64_t b) {
    const int at = cc_partner_type(wtype);
    return b >= 32 && k % PG_BLOCK_K == 0 && k >= PG_BLOCK_K && m >= 1 && (at == CC_Q8_0 || at == CC_Q8_K);
}

template <int BLOCK_N>
static int pg_launch(cc_device* dev, const CUtensorMap& tw, const CUtensorMap& tx, const float* row_scale, float* out, int64_t m, int64_t b, int64_t k) {
    const size_t smem = (size_t)PG_STAGES * ((size_t)PG_BLOCK_M * PG_BLOCK_K * 2 + (size_t)BLOCK_N * PG_BLOCK_K * 2) + 1024;
    CC_CUDA(dev, cudaFuncSetAttribute(wgmma_gemm_kernel<BLOCK_N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((unsigned)((m + PG_BLOCK_M - 1) / PG_BLOCK_M), (unsigned)((b + BLOCK_N - 1) / BLOCK_N));
    wgmma_gemm_kernel<BLOCK_N><<<grid, PG_THREADS, smem, dev->stream>>>(tw, tx, row_scale, out, (int)m, (int)b, (int)k);
    CC_LAUNCH_CHECK(dev);
    return CC_OK;
}

// Dequantised weights are kept: with 80 GB of HBM a 7B model's f16 tile source (2 bytes per weight, 13-14 GB) fits beside its
// quantised weights, and dequantising 58 MB per matrix on every call costs as much as the GEMM itself.  CRABML_PREFILL_NOCACHE=1 keeps
// the round-trip through one reusable scratch buffer instead (memory-constrained deployments).
static int pg_weight_f16(cc_device* dev, const cc_buf* w, int64_t m, int64_t k, PgScratch* s, const void** out) {
    static const bool nocache = getenv("CRABML_PREFILL_NOCACHE") != nullptr;
    cc_buf* wb = const_cast<cc_buf*>(w);
    const bool cacheable = !nocache && m == w->rows && k == w->cols;
    if (cacheable && wb->f16) { *out = wb->f16; return CC_OK; }
    void* dst = nullptr;
    if (cacheable) { CC_CUDA(dev, cudaMalloc(&dst, (size_t)m * k * 2)); }
    else { int rc = pg_ensure(dev, &s->w, &s->w_bytes, (size_t)m * k * 2); if (rc) return rc; dst = s->w; }
    const DeqPlanes pl = cc_deq_planes(w, k);
    const int64_t n = m * k;
    dequant_w_f16_kernel<<<(unsigned)((n / 2 + 255) / 256), 256, 0, dev->stream>>>(w->dtype, pl, n, (__half*)dst);
    CC_LAUNCH_CHECK(dev);
    if (cacheable) wb->f16 = dst;
    *out = dst;
    return CC_OK;
}

// act_q8_k: for K-quant weights, the (b, k) activation quantised to Q8_K (quantize.cu layout); x_f32: for Q8_0 partners, the f32
// activation itself, quantised on the way to f16 (the caller skips its own quantise launch); out: f32 [b][m]
int cc_launch_prefill_matmul(cc_device* dev, const cc_buf* w, const void* act_q8_k, const float* x_f32, float* out, int64_t m, int64_t k, int64_t b) {
    const int at = cc_partner_type(w->dtype);
    if (at == CC_Q8_0 && !x_f32) return cc_fail(dev, CC_ERR_ARG, "prefill: a Q8_0-partner weight needs the f32 activation");
    PgScratch* s = pg_scratch(dev);
    const void* wf16 = nullptr;
    int rc = pg_weight_f16(dev, w, m, k, s, &wf16);
    if (rc) return rc;
    // x scratch: the f16 operand [b][k], then the f32 row scales [b] (b * k * 2 is a multiple of 128 bytes)
    rc = pg_ensure(dev, &s->x, &s->x_bytes, (size_t)b * k * 2 + (size_t)b * 4);
    if (rc) return rc;
    float* row_scale = (float*)((uint8_t*)s->x + (size_t)b * k * 2);
    if (at == CC_Q8_K) act_q8k_to_f16_kernel<<<(unsigned)b, PG_ACT_THREADS, 0, dev->stream>>>(cc_act_q8_k((void*)act_q8_k, b * k), (int)k, (__half*)s->x, row_scale);
    else act_f32_to_q8f16_kernel<<<(unsigned)b, PG_ACT_THREADS, 0, dev->stream>>>(x_f32, (int)k, (__half*)s->x, row_scale);
    CC_LAUNCH_CHECK(dev);
    const int block_n = b >= 192 ? 256 : b >= 96 ? 128 : 64;
    CUtensorMap tw, tx;
    rc = pg_make_tmap(dev, &tw, wf16, m, k, PG_BLOCK_M);
    if (rc) return rc;
    rc = pg_make_tmap(dev, &tx, s->x, b, k, block_n);
    if (rc) return rc;
    if (block_n == 256) return pg_launch<256>(dev, tw, tx, row_scale, out, m, b, k);
    if (block_n == 128) return pg_launch<128>(dev, tw, tx, row_scale, out, m, b, k);
    return pg_launch<64>(dev, tw, tx, row_scale, out, m, b, k);
}
