// fused.cu -- kernels of the fused decode path (lazy mode).  They implement exactly the arithmetic of the trait ops
// they replace (cited inline); the lazy recorder (lazy.cu) substitutes them for runs of trait calls it recognises.
// All of them are written for programmatic dependent launch: they call cudaTriggerProgrammaticLaunchCompletion()
// immediately (so the NEXT kernel can be scheduled and start prefetching its weights) and
// cudaGridDependencySynchronize() before they touch anything the previous kernel produced.
#include "common.cuh"

__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------------------------
// normq: [dup] + [rms_norm + mul] + Q8_0 activation quantisation, one CTA.
//   orig (optional)  <- x                                   Tensor::dup            (llama2.rs:227,607)
//   x <- (x / sqrt(sum(x^2)/n + eps)) * w   (optional)      rms_norm_inplace + mul_inplace (rms_norm.rs:32-47, llama2.rs:231-232,611-612)
//   act <- quantize_q8_0(x)                                 buf_q8_0.rs:87-134 (what matmul_vec does first, matmul_vec.rs:37-40)
// ---------------------------------------------------------------------------------------------------------------
#define NQ_THREADS CC_RED_THREADS            // canonical reduction order (common.cuh)
#define NQ_MAX_CTAS 16
// Every CTA recomputes sum(x^2) over the whole row (a few KB from L2, same order in every CTA -> identical rms), then
// normalises / copies / quantises only its own slice of 32-element blocks.
// write_back = 0 (x is dead after its consumers) is REQUIRED for a multi-CTA grid: no CTA may overwrite x while
// another still sums it.
__global__ void __launch_bounds__(NQ_THREADS) normq_kernel(float* x, float* orig, const float* norm_w, float eps, int n, ActQ8_0 act, int write_back) {
    __shared__ float s_red[NQ_THREADS / 32];
    pdl_trigger();
    pdl_wait();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float rms = 1.0f;
    if (norm_w) {
        float ss = 0.0f;
        const float4* x4 = (const float4*)x;
        const int n4 = n >> 2;
        for (int i0 = 0; i0 < n4; i0 += NQ_THREADS * 4) {           // 4 independent 16-byte loads in flight per thread
            float4 v[4];
#pragma unroll
            for (int j = 0; j < 4; j++) { int i = i0 + j * NQ_THREADS + threadIdx.x; v[j] = i < n4 ? x4[i] : make_float4(0, 0, 0, 0); }
#pragma unroll
            for (int j = 0; j < 4; j++) ss += cc_sq4(v[j]);
        }
        rms = sqrtf(cc_block_sum_512(ss, s_red) / (float)n + eps);
    }
    const int nb = n >> 5;
    const int gw = blockIdx.x * (NQ_THREADS / 32) + warp, tw = gridDim.x * (NQ_THREADS / 32);
    for (int b = gw; b < nb; b += tw) {
        float v = x[b * 32 + lane];
        if (orig) orig[b * 32 + lane] = v;
        if (norm_w) { v = (v / rms) * norm_w[b * 32 + lane]; if (write_back) x[b * 32 + lane] = v; }
        float amax = warp_max(fabsf(v));
        float d = amax / 127.0f;
        int q = __float2int_rz(v / d);
        act.qs[b * 32 + lane] = (int8_t)q;
        int s = warp_sum_i(q);
        if (lane == 0) { act.d[b] = __half2float(__float2half_rn(d)); act.isum[b] = s; }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// attn_decode: one CTA per query head, n_batch = 1.  Replaces (llama2.rs:252-256, 541-590):
//   rope_inplace(q), rope_inplace(k)            rope.rs:47-80 (llama or neox pairs), cos/sin table evaluated on the host (cc_rope_table)
//   k_cache.concatenate(k), v_cache.concatenate(v)   concatenate.rs (F32 or F16 cache, f16::from_f32 on append)
//   q.contiguous().scale_inplace(1/sqrt(hd))
//   attn = q.batch_matmul(k_cache^T); softmax_inplace; out = attn.batch_matmul(v_cache)
//   (F32: batch_matmul.rs:47-71, kv head = h % n_kv;  F16: batch_matmul.rs:73-131, kv head = h / (n_heads/n_kv),
//    f32-accumulated f16 dot for QK, f16-accumulated FMA for PV)
// and additionally emits the Q8_0 quantisation of the output row (input of wo.matmul_vec).
// dyn: {pos, kv_len}; rope_tab: cos[pairs] then sin[pairs].
// ---------------------------------------------------------------------------------------------------------------
#define AT_THREADS CC_RED_THREADS            // canonical softmax order (common.cuh); also 16 score warps per head
template <bool KV_F16, bool NEOX>
__global__ void __launch_bounds__(AT_THREADS) attn_decode_kernel(const float* __restrict__ q_in, const float* __restrict__ k_in, const float* __restrict__ v_in,
                                                                 void* kcache, void* vcache, float* __restrict__ out, ActQ8_0 act,
                                                                 const int64_t* __restrict__ dyn, const float* __restrict__ rope_tab,
                                                                 const uint16_t* __restrict__ exp_lut, int n_heads, int n_kv, int hd, int rope_dim,
                                                                 int64_t seq_stride /* elements between kv heads */, float scale) {
    extern __shared__ __align__(16) float sm[];
    pdl_trigger();
    pdl_wait();
    const int h = blockIdx.x;
    const int g = KV_F16 ? h / (n_heads / n_kv) : h % n_kv;
    const int kv_len = (int)dyn[1];                 // cache length BEFORE this token's append
    const int L = kv_len + 1;
    float* s_q = sm;                                // [hd]
    float* s_k = sm + hd;                           // [hd] this token's roped key
    float* s_v = sm + 2 * hd;                       // [hd] this token's value
    float* s_p = sm + 3 * hd;                       // [L] scores
    __shared__ float s_red[AT_THREADS / 32];
    const int pairs = rope_dim >> 1;
    // rope, q additionally scaled AFTER the rotation (scale_inplace, llama2.rs:565); pairs as exact.cu rope_table_kernel (rope.rs:47-80):
    //   llama: (2j, 2j+1) for j < rope_dim/2
    //   neox: (j, j + hd/2) for j < rope_dim/2 -- half the HEAD dim even when rope_dim < hd, the reference's pairing
    const int half = hd >> 1;
    for (int i = threadIdx.x; i < hd; i += AT_THREADS) {
        float qv, kvv;
        const bool second = NEOX ? i >= half : (i & 1);
        const int j = NEOX ? (second ? i - half : i) : i >> 1;
        if (j < pairs) {
            const int lo = NEOX ? j : 2 * j, hi = NEOX ? j + half : 2 * j + 1;
            const float c = rope_tab[j], s = rope_tab[pairs + j];
            const float q0 = q_in[h * hd + lo], q1 = q_in[h * hd + hi];
            const float k0 = k_in[g * hd + lo], k1 = k_in[g * hd + hi];
            qv = second ? q0 * s + q1 * c : q0 * c - q1 * s;
            kvv = second ? k0 * s + k1 * c : k0 * c - k1 * s;
        } else {
            qv = q_in[h * hd + i];
            kvv = k_in[g * hd + i];
        }
        s_q[i] = qv * scale;
        s_k[i] = kvv;
        s_v[i] = v_in[g * hd + i];
    }
    __syncthreads();
    // append to the caches (one CTA per kv head does the write; every CTA uses its local copy for position kv_len)
    const bool owner = KV_F16 ? (h % (n_heads / n_kv) == 0) : (h < n_kv);
    if (owner) {
        for (int i = threadIdx.x; i < hd; i += AT_THREADS) {
            const int64_t off = (int64_t)g * seq_stride + (int64_t)kv_len * hd + i;
            if (KV_F16) { ((__half*)kcache)[off] = __float2half_rn(s_k[i]); ((__half*)vcache)[off] = __float2half_rn(s_v[i]); }
            else { ((float*)kcache)[off] = s_k[i]; ((float*)vcache)[off] = s_v[i]; }
        }
    }
    // scores: one warp per position
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int s = warp; s < L; s += AT_THREADS / 32) {
        float acc = 0.0f;
        if (s < kv_len) {
            if (KV_F16) {
                const __half* kr = (const __half*)kcache + (int64_t)g * seq_stride + (int64_t)s * hd;
                for (int i = lane; i < hd; i += 32) acc += __half2float(__float2half_rn(s_q[i])) * __half2float(kr[i]);
            } else {
                const float* kr = (const float*)kcache + (int64_t)g * seq_stride + (int64_t)s * hd;
                for (int i = lane; i < hd; i += 32) acc += s_q[i] * kr[i];
            }
        } else {
            for (int i = lane; i < hd; i += 32) {
                if (KV_F16) acc += __half2float(__float2half_rn(s_q[i])) * __half2float(__float2half_rn(s_k[i]));
                else acc += s_q[i] * s_k[i];
            }
        }
        acc = warp_sum(acc);
        if (lane == 0) s_p[s] = acc;
    }
    __syncthreads();
    // softmax with the f16 exp LUT (softmax.rs:39-54)
    float m = -INFINITY;
    for (int s = threadIdx.x; s < L; s += AT_THREADS) m = fmaxf(m, s_p[s]);
    m = warp_max(m);
    if (lane == 0) s_red[warp] = m;
    __syncthreads();
    m = s_red[0];
#pragma unroll
    for (int w = 1; w < AT_THREADS / 32; w++) m = fmaxf(m, s_red[w]);
    __syncthreads();
    float sum = 0.0f;
    for (int s = threadIdx.x; s < L; s += AT_THREADS) {
        float e = h2f_bits(exp_lut[f2h_bits(s_p[s] - m)]);
        s_p[s] = e;
        sum += e;
    }
    sum = warp_sum(sum);
    if (lane == 0) s_red[warp] = sum;
    __syncthreads();
    sum = 0.0f;
#pragma unroll
    for (int w = 0; w < AT_THREADS / 32; w++) sum += s_red[w];
    for (int s = threadIdx.x; s < L; s += AT_THREADS) s_p[s] = s_p[s] / sum;
    __syncthreads();
    // out[d] = sum_s p[s] * V[s][d]: one thread per d, sequential over s (the reference's order: batch_matmul.rs:60-68)
    float* s_o = s_k;                                  // reuse: keys no longer needed
    for (int d = threadIdx.x; d < hd; d += AT_THREADS) {
        float o;
        if (KV_F16) {
            const __half* vb = (const __half*)vcache + (int64_t)g * seq_stride + d;
            __half acc = __float2half_rn(0.0f);
            for (int s = 0; s < kv_len; s++) acc = __hadd(acc, __hmul(vb[(int64_t)s * hd], __float2half_rn(s_p[s])));
            acc = __hadd(acc, __hmul(__float2half_rn(s_v[d]), __float2half_rn(s_p[kv_len])));
            o = __half2float(acc);
        } else {
            const float* vb = (const float*)vcache + (int64_t)g * seq_stride + d;
            float acc = 0.0f;
            for (int s = 0; s < kv_len; s++) acc += s_p[s] * vb[(int64_t)s * hd];
            acc += s_p[kv_len] * s_v[d];
            o = acc;
        }
        out[h * hd + d] = o;
        s_o[d] = o;
    }
    __syncthreads();
    // Q8_0 quantisation of this head's hd outputs (hd/32 blocks), input of wo.matmul_vec -- only when blocks do not
    // straddle heads (hd % 32 == 0); otherwise the consumer quantises the f32 row itself
    if (act.qs != nullptr)
    for (int b = warp; b < (hd >> 5); b += AT_THREADS / 32) {
        float v = s_o[b * 32 + lane];
        float amax = warp_max(fabsf(v));
        float d = amax / 127.0f;
        int qq = __float2int_rz(v / d);
        const int gb = h * (hd >> 5) + b;
        act.qs[gb * 32 + lane] = (int8_t)qq;
        int ss = warp_sum_i(qq);
        if (lane == 0) { act.d[gb] = __half2float(__float2half_rn(d)); act.isum[gb] = ss; }
    }
}

int cc_launch_normq(cc_device* dev, float* x, float* orig, const float* norm_w, float eps, int64_t n, ActQ8_0 act, bool write_back) {
    CC_REQUIRE(dev, n % 32 == 0, "normq: length %lld %% 32 != 0", (long long)n);
    CC_REQUIRE(dev, n % 4 == 0, "normq: length %lld %% 4 != 0", (long long)n);
    int ctas = (int)((n / 32 + NQ_THREADS / 32 - 1) / (NQ_THREADS / 32));
    if (ctas > NQ_MAX_CTAS) ctas = NQ_MAX_CTAS;
    if (ctas < 1 || (norm_w && write_back)) ctas = 1;
    cudaError_t e = launch_pdl(normq_kernel, dim3(ctas), dim3(NQ_THREADS), 0, dev->stream, dev->pdl, x, orig, norm_w, eps, (int)n, act, write_back ? 1 : 0);
    if (e != cudaSuccess) return cc_fail(dev, CC_ERR_CUDA, "normq launch: %s", cudaGetErrorString(e));
    dev->launches++;
    return CC_OK;
}

// q, k, v of the head and the whole score row live in shared memory: max_len <= 50 808 positions at head_dim 128
#define AT_SMEM_MAX (200 * 1024)
static size_t attn_decode_smem(int64_t hd, int64_t max_len) { return (size_t)(3 * hd + max_len + 8) * sizeof(float); }
bool cc_attn_decode_fits(int64_t hd, int64_t max_len) { return attn_decode_smem(hd, max_len) <= AT_SMEM_MAX; }

template <bool KV_F16, bool NEOX>
static cudaError_t launch_attn(cc_device* dev, const AttnArgs& a, ActQ8_0 act, const int64_t* dyn, const float* rope_tab, size_t smem) {
    if (smem > 48 * 1024) cudaFuncSetAttribute(attn_decode_kernel<KV_F16, NEOX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    return launch_pdl(attn_decode_kernel<KV_F16, NEOX>, dim3(a.n_heads), dim3(AT_THREADS), smem, dev->stream, dev->pdl, a.q, a.k, a.v, a.kcache, a.vcache, a.out, act,
                      dyn, rope_tab, (const uint16_t*)dev->exp_lut, a.n_heads, a.n_kv, a.hd, a.rope_dim, a.seq_stride, a.scale);
}

int cc_launch_attn_decode(cc_device* dev, const AttnArgs& a, const int64_t* dyn, const float* rope_tab) {
    const size_t smem = attn_decode_smem(a.hd, a.max_len);
    CC_REQUIRE(dev, smem <= AT_SMEM_MAX, "attention: context %d too long for the single-pass kernel", a.max_len);
    ActQ8_0 act = cc_act_q8_0(a.act_scratch, (int64_t)a.n_heads * a.hd);
    if (!a.act_scratch) act.qs = nullptr;
    const cudaError_t e = a.kv_f16 ? (a.rope_neox ? launch_attn<true, true>(dev, a, act, dyn, rope_tab, smem) : launch_attn<true, false>(dev, a, act, dyn, rope_tab, smem))
                                   : (a.rope_neox ? launch_attn<false, true>(dev, a, act, dyn, rope_tab, smem) : launch_attn<false, false>(dev, a, act, dyn, rope_tab, smem));
    if (e != cudaSuccess) return cc_fail(dev, CC_ERR_CUDA, "attention launch: %s", cudaGetErrorString(e));
    dev->launches++;
    return CC_OK;
}
