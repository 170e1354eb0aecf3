// ringbench.cu -- can a TMA-fed shared-memory ring (up to 4 producer warps, 16 consumer warps per SM: the structure of mega_ring.cu) stream
// HBM at full speed, and with which slot size / depth / number of issuing lanes?  Developer tool.
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/build/ringbench tools/ringbench.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

__device__ __forceinline__ void mbar_init(unsigned mbar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(count) : "memory"); }
__device__ __forceinline__ bool try_wait(unsigned bar, unsigned parity) {
    unsigned ok;
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void expect_tx(unsigned bar, unsigned bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void bulk_g2s(unsigned dst, const void* src, unsigned bytes, unsigned bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void st_release(unsigned addr, unsigned v) { asm volatile("st.release.cta.shared::cta.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned ld_acquire(unsigned addr) {
    unsigned v;
    asm volatile("ld.acquire.cta.shared::cta.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}

#define MAX_SLOTS 128
// every CTA streams `n_ent` entries of `ent_bytes` (contiguous region per CTA); copies = 1: one bulk copy per entry, 2: main part + a tail of
// 256 bytes per 4352 (the f16 scale plane of mega_ring.cu); lanes: issuing threads of the producer warps (threads 512 ..)
__global__ void __launch_bounds__(640, 1) k_ring(const uint8_t* __restrict__ in, size_t cta_stride, int n_ent, int ent_bytes, int slot_bytes, int nslots, int copies,
                                                 int lanes, int work, int pattern, int* out) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) unsigned long long s_full[MAX_SLOTS];
    __shared__ unsigned s_done[MAX_SLOTS], s_seq[MAX_SLOTS];
    const unsigned full0 = (unsigned)__cvta_generic_to_shared(s_full), done0 = (unsigned)__cvta_generic_to_shared(s_done);
    const unsigned ring0 = (unsigned)__cvta_generic_to_shared(smem);
    if (threadIdx.x == 0) for (int i = 0; i < nslots; i++) { mbar_init(full0 + 8u * i, 1u); s_done[i] = 0; s_seq[i] = 0; }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const uint8_t* base = in + (size_t)blockIdx.x * cta_stride;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (warp >= 16) {
        const int pt = (int)threadIdx.x - 512;
        if (pt >= lanes) return;
        int j = pt;
        while (j < n_ent) {
            const unsigned e = (unsigned)j, slot = e % (unsigned)nslots, use = e / (unsigned)nslots;
            if (!use || ld_acquire(done0 + 4u * slot) == e - (unsigned)nslots + 1u) {
                const unsigned fb = full0 + 8u * slot, dst = ring0 + slot * (unsigned)slot_bytes;
                const uint8_t* src = base + (size_t)e * ent_bytes;
                expect_tx(fb, (unsigned)ent_bytes);
                if (pattern == 1) {        // mega_ring.cu's addresses: CTA c takes the 4 KB rows c, c + gridDim.x, ... of a matrix; their 256-byte scale rows live in another plane
                    const size_t idx = (size_t)e * gridDim.x + blockIdx.x;
                    bulk_g2s(dst, in + idx * 4096, 4096u, fb);
                    bulk_g2s(dst + 4096, in + ((size_t)5 << 30) + idx * 256, 256u, fb);
                } else if (copies == 2) {
                    const unsigned tail = (unsigned)(ent_bytes / 17) & ~15u;
                    bulk_g2s(dst, src, (unsigned)ent_bytes - tail, fb); bulk_g2s(dst + ent_bytes - tail, src + ent_bytes - tail, tail, fb);
                }
                else bulk_g2s(dst, src, (unsigned)ent_bytes, fb);
                __threadfence_block();
                ((volatile unsigned*)s_seq)[slot] = e + 1u;
                j += lanes;
            }
        }
        return;
    }
    int acc = 0;
    // work 1 / 2: the arithmetic of mega_ring.cu's consumer on every 4352 bytes of an entry (8 weight LDS.128 + 4 scales, 8 activation LDS.128,
    // 32 dp4a, f32 scale-accumulate; an entry of R such rows holds R x 4096 B of quants, then R x 256 B of scales); activation layout
    // 1 = block-major (lane stride 32 B: 2-way bank conflicts), 2 = half-split (conflict-free)
    uint8_t* act = smem + (size_t)nslots * slot_bytes;         // 4096 B quants + 512 B scales
    if (work) { for (int i = threadIdx.x; i < 4608 / 4; i += 512) ((int*)act)[i] = i * 2654435761u; asm volatile("bar.sync 1, 512;" ::: "memory"); }
    float facc = 0.0f;
    for (int j = warp; j < n_ent; j += 16) {
        const unsigned e = (unsigned)j, slot = e % (unsigned)nslots, par = (e / (unsigned)nslots) & 1u;
        while (!(((volatile unsigned*)s_seq)[slot] == e + 1u && try_wait(full0 + 8u * slot, par))) {}
        const int4* sp = (const int4*)(smem + (size_t)slot * slot_bytes);
        if (!work) { for (int i = lane; i < ent_bytes / 16; i += 32) { const int4 v = sp[i]; acc += v.x ^ v.y ^ v.z ^ v.w; } }
        else {
            const int rows = ent_bytes / 4352 > 0 ? ent_bytes / 4352 : 1;
            const float* ad = (const float*)(act + 4096) + lane;
            float part = 0.0f;
            for (int r = 0; r < rows; r++) {
                const uint8_t* q = (const uint8_t*)sp + r * 4096 + lane * 16;
                const uint16_t* d = (const uint16_t*)((const uint8_t*)sp + rows * 4096 + r * 256) + lane;
#pragma unroll
                for (int g = 0; g < 4; g++) {
                    const int4 wa = *(const int4*)(q + g * 1024), wb = *(const int4*)(q + g * 1024 + 512);
                    int4 aa, ab;
                    if (work == 1) { aa = *(const int4*)(act + g * 1024 + lane * 32); ab = *(const int4*)(act + g * 1024 + lane * 32 + 16); }
                    else { aa = *(const int4*)(act + g * 1024 + lane * 16); ab = *(const int4*)(act + g * 1024 + 512 + lane * 16); }
                    int si = __dp4a(wa.x, aa.x, __dp4a(wa.y, aa.y, __dp4a(wa.z, aa.z, __dp4a(wa.w, aa.w, 0)))) + __dp4a(wb.x, ab.x, __dp4a(wb.y, ab.y, __dp4a(wb.z, ab.z, __dp4a(wb.w, ab.w, 0))));
                    part += (float)si * __half2float(__ushort_as_half(d[g * 32])) * ad[g * 32];
                }
            }
            facc += part;
            acc += __float_as_int(part) & 1;
        }
        __syncwarp();
        if (lane == 0) asm volatile("st.release.cta.shared::cta.u32 [%0], %1;" ::"r"(done0 + 4u * slot), "r"(e + 1u), "r"(acc) : "memory");
    }
    if (acc == 0x12345678 || facc == 1.2345f) *out = acc;
}

int main() {
    const size_t total = (size_t)6 << 30;      // 6 GB >> L2 (pattern 1: 5 GB of "quants" + a scale plane behind them)
    uint8_t* in; int* out;
    cudaMalloc(&in, total); cudaMalloc(&out, 4);
    cudaMemset(in, 1, total);
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaFuncSetAttribute(k_ring, cudaFuncAttributeMaxDynamicSharedMemorySize, 225 * 1024);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    // ring_kb: ring bytes in KB (slots = ring_kb * 1024 / slot size); lanes 128 = 4 producer warps (mega_ring.cu), 32 = one
    struct Cfg { int ent, ring_kb, copies, lanes, work, pattern; };
    const Cfg cfgs[] = {
        // the ring kernel today: 4352-byte Q8_0 entries (4096 B quants + 256 B scales, two copies), ~40 slots, 4 producer warps
        {4352, 174, 2, 128, 2, 1}, {4352, 174, 2, 128, 2, 0}, {4352, 174, 2, 128, 0, 0}, {4352, 174, 2, 32, 2, 0},
        // one copy per entry: 4.3, 8.7 and 17 KB, at ~174 KB and ~200 KB of ring
        {4352, 174, 1, 128, 2, 0}, {8704, 174, 1, 128, 2, 0}, {17408, 174, 1, 128, 2, 0},
        {4352, 200, 1, 128, 2, 0}, {8704, 204, 1, 128, 2, 0}, {17408, 204, 1, 128, 2, 0},
        // two copies per entry (quants + scales) at 8.7 / 17 KB: a row pair / quad in one slot
        {8704, 174, 2, 128, 2, 0}, {8704, 204, 2, 128, 2, 0}, {17408, 204, 2, 128, 2, 0}, {8704, 204, 2, 64, 2, 0}, {8704, 204, 2, 32, 2, 0},
        // Q4_0 entries (2048 B quants + 256 B scales per row): 1, 2 and 4 rows per slot, two copies, read only
        {2304, 174, 2, 128, 0, 0}, {4608, 174, 2, 128, 0, 0}, {4608, 204, 2, 128, 0, 0}, {9216, 204, 2, 128, 0, 0},
    };
    for (const Cfg& c : cfgs) {
        const int slot_bytes = (c.ent + 127) & ~127;
        int nslots = c.ring_kb * 1024 / slot_bytes; if (nslots > MAX_SLOTS) nslots = MAX_SLOTS;
        const size_t per_cta = (c.pattern ? ((size_t)5 << 30) : total) / sms / 256 * 256;
        const int n_ent = (int)(per_cta / (c.pattern ? 4096 : c.ent));
        const size_t smem = (size_t)nslots * slot_bytes + 4608;
        float best = 1e30f;
        for (int rep = 0; rep < 3; rep++) {
            cudaEventRecord(e0);
            k_ring<<<sms, 640, smem>>>(in, per_cta, n_ent, c.ent, slot_bytes, nslots, c.copies, c.lanes, c.work, c.pattern, out);
            cudaEventRecord(e1);
            cudaError_t err = cudaEventSynchronize(e1);
            if (err != cudaSuccess) { printf("error: %s\n", cudaGetErrorString(err)); return 1; }
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            if (ms < best) best = ms;
        }
        const double bytes = (double)n_ent * c.ent * sms;
        printf("entry %5d B  slots %3d (%3d KB)  copies %d  lanes %3d  work %d  pattern %d : %8.1f GB/s  (%.3f ms)\n", c.ent, nslots, (int)(smem / 1024), c.copies, c.lanes, c.work, c.pattern, bytes / best / 1e6, best);
        fflush(stdout);
    }
    return 0;
}
