// sample_dev.cuh -- temperature + top-p sampling on the device (crabml-llama2/src/sampler.rs:27-129), one CTA of 512 threads.
// Included by sample.cu (the standalone kernel of eager mode and the CUDA-graph mode) and by mega.cu / mega_ring.cu (the MK_SAMPLE
// phase): the same routine with the same thread layout, so every fast mode picks the same id by construction.
//
//   1. v = logit / T (IEEE), max = NaN-ignoring fold (sampler.rs:120), e = exp LUT (v - max), p = e / sum(e)
//   2. cutoff = (1 - topp) / (n - 1); keep (p, i) with p >= cutoff, in index order (sampler.rs:76-83)
//   3. stable ascending sort of the pairs (sampler.rs:84): LSD radix sort, 4 passes of 8 bits over the f32 bit patterns (p >= 0, so
//      the bits order like unsigned integers); every pass is stable, ties keep index order
//   4. prefix sums C_j of the sorted probabilities; last = first j with C_j > topp (else n0 - 1); r = coin * C_last;
//      pick = first j <= last with C_j > r (else last) (sampler.rs:86-106)
// Sums (the softmax denominator and the prefix sums) are sequential on exact_order devices -- the reference's order, so the pick
// equals the oracle's for any coin -- and otherwise the canonical 512-thread tree (common.cuh: p has softmax_kernel's bits) and
// one fixed tiled block scan.  Everything else is order-free.
// n0 == 0 (the reference panics: n == 1 with topp <= 1, or topp < 1/n on a near-uniform row) picks the argmax of the logits, the
// LAST maximum, as temperature 0 would.  NaN logits are outside the contract; the routine still ends and returns an index in [0, n).
#pragma once
#include <limits.h>

#include "common.cuh"

struct SampleDyn {                     // per-call values; the lazy modes carry them in the per-token dyn block
    unsigned long long seed;
    long long coin_index, hist_index;
    float temperature, topp;
};
// global scratch of one call: p[n] f32 (exponentials, then prefix sums) | k0[n], k1[n] u64 (probability bits << 32 | index)
struct SampleScratch { float* p; unsigned long long *k0, *k1; };
inline size_t cc_sample_scratch_bytes(int64_t n) { return (((size_t)n * 4 + 15) & ~(size_t)15) + (size_t)n * 16; }
__host__ __device__ inline SampleScratch cc_sample_scratch(void* base, int64_t n) {
    SampleScratch s;
    s.p = (float*)base;
    s.k0 = (unsigned long long*)((uint8_t*)base + (((size_t)n * 4 + 15) & ~(size_t)15));
    s.k1 = s.k0 + n;
    return s;
}
// coin in [0, 1 - 2^-24]: 24 bits of splitmix64(seed ^ splitmix64(coin_index)); one seed reproduces one run in every mode
__host__ __device__ inline float cc_sample_coin(uint64_t seed, int64_t coin_index) {
    return (float)(cc_splitmix64(seed ^ cc_splitmix64((uint64_t)coin_index)) >> 40) * 0x1p-24f;
}

#define SMP_THREADS 512
#define SMP_ITEMS 8
#define SMP_TILE (SMP_THREADS * SMP_ITEMS)
#define SMP_STAGE 2048          // exact_order: entries per staged chunk of the sequential sums (8 KB)
// shared memory: per-warp digit counters u16 [16][256] | digit histograms u32 [4][256] | digit offsets u32 [256] | f32 [16] | int [20] | i64 [16]
#define SMP_SMEM_BYTES 13600

#ifdef __CUDACC__
// a named barrier over the 512 threads: the ring megakernel's producer warps never take part (mega_ring.cu MK_SYNC)
__device__ __forceinline__ void smp_sync() { asm volatile("bar.sync 1, 512;" ::: "memory"); }

// sampler.rs:109-116 via ops.cu argmax_kernel's order: the LAST maximum
__device__ __forceinline__ long long smp_argmax(const float* x, int n, float* s_f, long long* s_ll) {
    float bv = 0.0f; long long bi = -1;
    for (long long i = threadIdx.x; i < n; i += SMP_THREADS) { const float v = __ldcg(x + i); if (bi < 0 || !(v < bv)) { bv = v; bi = i; } }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (oi >= 0 && (bi < 0 || ov > bv || (ov == bv && oi > bi))) { bv = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { s_f[threadIdx.x >> 5] = bv; s_ll[threadIdx.x >> 5] = bi; }
    smp_sync();
    bv = s_f[0]; bi = s_ll[0];
    for (int w = 1; w < 16; w++) { const float ov = s_f[w]; const long long oi = s_ll[w]; if (oi >= 0 && (bi < 0 || ov > bv || (ov == bv && oi > bi))) { bv = ov; bi = oi; } }
    smp_sync();
    return bi < 0 ? 0 : bi;
}

// Returns the sampled index (in every thread).  x: n logits (read through L2: in the megakernel other CTAs wrote them); never modified.
static __device__ __noinline__ long long cc_sample_block(const float* x, int n, const SampleDyn a, bool exact, const SampleScratch S, uint8_t* sm,
                                                         const uint16_t* __restrict__ lut) {
    uint16_t* s_wc = (uint16_t*)sm;
    unsigned* s_hist = (unsigned*)(sm + 8192);
    unsigned* s_off = (unsigned*)(sm + 12288);
    float* s_f = (float*)(sm + 13312);
    int* s_i = (int*)(sm + 13376);
    long long* s_ll = (long long*)(sm + 13472);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const float T = a.temperature, topp = a.topp;
    if (!(T > 0.0f)) return smp_argmax(x, n, s_f, s_ll);

    // ---- 1. softmax of logits / T (sampler.rs:34-38, 119-129) ----
    float m = __int_as_float(0x7fffffff);          // fold from NaN: f32::max ignores NaN
    for (int i = t; i < n; i += SMP_THREADS) m = fmaxf(m, __ldcg(x + i) / T);
    m = warp_max(m);
    if (lane == 0) s_f[warp] = m;
    smp_sync();
    m = s_f[0];
    for (int w = 1; w < 16; w++) m = fmaxf(m, s_f[w]);
    smp_sync();
    float s = 0.0f;
    for (int i = t; i < n; i += SMP_THREADS) {
        const float e = h2f_bits(lut[f2h_bits(__ldcg(x + i) / T - m)]);
        __stcg(S.p + i, e);
        s += e;
    }
    if (exact) {                                   // sequential, the reference's order
        // the CTA stages SMP_STAGE entries at a time into shared memory (the digit counters' area, free until the sort) and thread 0
        // adds them up from there: its chain of dependent adds never waits on L2
        float* s_stage = (float*)s_wc;
        float q = 0.0f;
        for (int base = 0; base < n; base += SMP_STAGE) {
            smp_sync();
            for (int i = t; i < SMP_STAGE && base + i < n; i += SMP_THREADS) s_stage[i] = __ldcg(S.p + base + i);
            smp_sync();
            if (t == 0) { const int m = min(SMP_STAGE, n - base); for (int i = 0; i < m; i++) q += s_stage[i]; }
        }
        if (t == 0) s_f[0] = q;
        smp_sync();
        s = s_f[0];
    } else {                                       // cc_block_sum_512's order: softmax_kernel's bits
        s = warp_sum(s);
        if (lane == 0) s_f[warp] = s;
        smp_sync();
        s = 0.0f;
        for (int w = 0; w < 16; w++) s += s_f[w];
    }
    smp_sync();

    // ---- 2. filter in index order + the four digit histograms ----
    const float cutoff = (1.0f - topp) / (float)(n - 1);
    for (int i = t; i < 4 * 256; i += SMP_THREADS) s_hist[i] = 0u;
    smp_sync();
    int n0 = 0;
    for (int base = 0; base < n; base += SMP_TILE) {
        const int i0 = base + t * SMP_ITEMS;
        unsigned kb[SMP_ITEMS], flags = 0u;
#pragma unroll
        for (int k = 0; k < SMP_ITEMS; k++) {
            float pk = 0.0f;
            if (i0 + k < n) { pk = __ldcg(S.p + i0 + k) / s; if (pk >= cutoff) flags |= 1u << k; }
            kb[k] = __float_as_uint(pk);
        }
        const int cnt = __popc(flags);
        int inc = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
        if (lane == 31) s_i[warp] = inc;
#pragma unroll
        for (int k = 0; k < SMP_ITEMS; k++)
#pragma unroll
            for (int d = 0; d < 4; d++) {
                const unsigned dg = (flags >> k) & 1u ? (kb[k] >> (8 * d)) & 255u : 256u;
                const unsigned peers = __match_any_sync(0xffffffffu, dg);
                if (dg < 256u && (peers & ((1u << lane) - 1u)) == 0u) atomicAdd(&s_hist[d * 256 + dg], (unsigned)__popc(peers));
            }
        smp_sync();
        int woff = 0, tot = 0;
        for (int w = 0; w < 16; w++) { const int v = s_i[w]; woff += w < warp ? v : 0; tot += v; }
        int pos = n0 + woff + inc - cnt;
#pragma unroll
        for (int k = 0; k < SMP_ITEMS; k++)
            if ((flags >> k) & 1u) __stcg(S.k0 + pos++, ((unsigned long long)kb[k] << 32) | (unsigned)(i0 + k));
        n0 += tot;
        smp_sync();
    }
    if (n0 == 0) return smp_argmax(x, n, s_f, s_ll);

    // ---- 3. stable LSD radix sort, ascending ----
    unsigned long long *src = S.k0, *dst = S.k1;
    for (int d = 0; d < 4; d++) {
        if (t == 0) s_i[17] = 0;
        smp_sync();
        unsigned hv = 0u, hinc = 0u;
        if (t < 256) {
            hv = s_hist[d * 256 + t];
            if (hv == (unsigned)n0) s_i[17] = 1;         // every key has this digit: the pass would not move anything
            hinc = hv;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const unsigned y = __shfl_up_sync(0xffffffffu, hinc, o); if (lane >= o) hinc += y; }
            if (lane == 31) s_i[warp] = (int)hinc;
        }
        smp_sync();
        const bool skip = s_i[17] != 0;
        if (t < 256) { unsigned wo = 0u; for (int w = 0; w < warp; w++) wo += (unsigned)s_i[w]; s_off[t] = wo + hinc - hv; }
        smp_sync();
        if (skip) continue;
        const int shift = 32 + 8 * d;
        uint16_t* wc = s_wc + warp * 256;
        for (int base = 0; base < n0; base += SMP_TILE) {
            for (int j = lane; j < 256; j += 32) wc[j] = 0;
            __syncwarp();
            unsigned long long e[SMP_ITEMS];
            unsigned rk[SMP_ITEMS];
#pragma unroll
            for (int k = 0; k < SMP_ITEMS; k++) {            // element order within the tile: (warp, item, lane) = index order
                const int j = base + warp * (32 * SMP_ITEMS) + k * 32 + lane;
                e[k] = j < n0 ? __ldcg(src + j) : 0ull;
                const unsigned dg = j < n0 ? (unsigned)(e[k] >> shift) & 255u : 256u;
                const unsigned peers = __match_any_sync(0xffffffffu, dg);
                const unsigned below = peers & ((1u << lane) - 1u);
                rk[k] = dg < 256u ? wc[dg] + (unsigned)__popc(below) : 0u;
                __syncwarp();
                if (dg < 256u && below == 0u) wc[dg] += (uint16_t)__popc(peers);
                __syncwarp();
            }
            smp_sync();
            unsigned ttot = 0u;
            if (t < 256) {                                   // per digit: exclusive prefix over the warps of this tile
                for (int w = 0; w < 16; w++) { const unsigned c = s_wc[w * 256 + t]; s_wc[w * 256 + t] = (uint16_t)ttot; ttot += c; }
            }
            smp_sync();
#pragma unroll
            for (int k = 0; k < SMP_ITEMS; k++) {
                const int j = base + warp * (32 * SMP_ITEMS) + k * 32 + lane;
                if (j < n0) { const unsigned dg = (unsigned)(e[k] >> shift) & 255u; __stcg(dst + s_off[dg] + wc[dg] + rk[k], e[k]); }
            }
            smp_sync();
            if (t < 256) s_off[t] += ttot;
        }
        unsigned long long* sw = src; src = dst; dst = sw;
        smp_sync();
    }

    // ---- 4. prefix sums, truncation at topp, the pick (sampler.rs:86-106) ----
    float* C = S.p;                                          // the exponentials are no longer needed
    if (t == 0) s_i[18] = INT_MAX;
    smp_sync();
    if (exact) {                                             // sequential, staged like the softmax sum
        float* s_stage = (float*)s_wc;
        float c = 0.0f;
        for (int base = 0; base < n0; base += SMP_STAGE) {
            for (int i = t; i < SMP_STAGE && base + i < n0; i += SMP_THREADS) s_stage[i] = __uint_as_float((unsigned)(__ldcg(src + base + i) >> 32));
            smp_sync();
            if (t == 0) {
                const int m = min(SMP_STAGE, n0 - base);
                for (int i = 0; i < m; i++) {
                    c += s_stage[i];
                    __stcg(C + base + i, c);
                    if (c > topp) { s_i[18] = base + i; break; }
                }
            }
            smp_sync();
            if (s_i[18] != INT_MAX) break;
        }
    } else {
        // tiles of 4096: thread t sums its 8 consecutive entries left to right; C = carry + ((warp offset + lane offset) + local prefix)
        float carry = 0.0f;
        for (int base = 0; base < n0; base += SMP_TILE) {
            const int j0 = base + t * SMP_ITEMS;
            float l[SMP_ITEMS], acc = 0.0f;
#pragma unroll
            for (int k = 0; k < SMP_ITEMS; k++) { acc += j0 + k < n0 ? __uint_as_float((unsigned)(__ldcg(src + j0 + k) >> 32)) : 0.0f; l[k] = acc; }
            float inc = acc;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const float y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
            float ex = __shfl_up_sync(0xffffffffu, inc, 1);
            if (lane == 0) ex = 0.0f;
            if (lane == 31) s_f[warp] = inc;
            smp_sync();
            float woff = 0.0f, tot = 0.0f;
            for (int w = 0; w < 16; w++) { if (w == warp) woff = tot; tot += s_f[w]; }
            const float off = woff + ex;
            int first = INT_MAX;
#pragma unroll
            for (int k = 0; k < SMP_ITEMS; k++) {
                if (j0 + k >= n0) break;
                const float c = carry + (off + l[k]);
                __stcg(C + j0 + k, c);
                if (c > topp && first == INT_MAX) first = j0 + k;
            }
            if (first != INT_MAX) atomicMin(&s_i[18], first);
            carry = carry + tot;
            smp_sync();
            if (s_i[18] != INT_MAX) break;
        }
    }
    const int last = s_i[18] == INT_MAX ? n0 - 1 : s_i[18];
    const float r = cc_sample_coin(a.seed, a.coin_index) * __ldcg(C + last);
    if (t == 0) s_i[19] = INT_MAX;
    smp_sync();
    for (int j = t; j <= last; j += SMP_THREADS) if (__ldcg(C + j) > r) { atomicMin(&s_i[19], j); break; }
    smp_sync();
    const int pick = s_i[19] == INT_MAX ? last : s_i[19];
    const long long id = (long long)(unsigned)(__ldcg(src + pick) & 0xffffffffull);
    smp_sync();                                              // shared memory may be reused by the caller
    return id;
}
#endif
