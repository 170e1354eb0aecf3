// membench.cu -- what read bandwidth can a streaming kernel reach on this H100, and with which shape?
// (developer tool; informs matvec_stream.cu).  Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/build/membench tools/membench.cu
#include <cstdio>
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>

__device__ __forceinline__ int4 ld_nc(const int4* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ int4 ld_plain(const int4* p) { return *p; }

// A: grid-stride, U independent loads per thread per iteration
template <int U, bool NC>
__global__ void k_gridstride(const int4* __restrict__ in, size_t n, int* out) {
    size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    int acc = 0;
    for (size_t i = tid; i + (U - 1) * stride < n; i += U * stride) {
        int4 v[U];
#pragma unroll
        for (int j = 0; j < U; j++) v[j] = NC ? ld_nc(in + i + j * stride) : ld_plain(in + i + j * stride);
#pragma unroll
        for (int j = 0; j < U; j++) acc += v[j].x ^ v[j].y ^ v[j].z ^ v[j].w;
    }
    if (acc == 0x12345678) *out = acc;
}
// B: each warp streams contiguous chunks of CH*512 bytes (lane-interleaved int4), chunks dealt round-robin to warps,
//    double-buffered (DB) or not
template <int CH, bool DB>
__global__ void k_warpchunk(const int4* __restrict__ in, size_t n_chunks, int* out) {
    const int lane = threadIdx.x & 31;
    size_t gw = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, tw = ((size_t)gridDim.x * blockDim.x) >> 5;
    int acc = 0;
    int4 a[CH], b[CH];
    if (DB) {
        size_t c = gw;
        if (c < n_chunks) {
#pragma unroll
            for (int j = 0; j < CH; j++) a[j] = ld_nc(in + c * CH * 32 + j * 32 + lane);
        }
        for (; c < n_chunks; c += 2 * tw) {
            size_t c1 = c + tw, c2 = c + 2 * tw;
            if (c1 < n_chunks) {
#pragma unroll
                for (int j = 0; j < CH; j++) b[j] = ld_nc(in + c1 * CH * 32 + j * 32 + lane);
            }
#pragma unroll
            for (int j = 0; j < CH; j++) acc += a[j].x ^ a[j].y ^ a[j].z ^ a[j].w;
            if (c2 < n_chunks) {
#pragma unroll
                for (int j = 0; j < CH; j++) a[j] = ld_nc(in + c2 * CH * 32 + j * 32 + lane);
            }
            if (c1 < n_chunks) {
#pragma unroll
                for (int j = 0; j < CH; j++) acc += b[j].x ^ b[j].y ^ b[j].z ^ b[j].w;
            }
        }
    } else {
        for (size_t c = gw; c < n_chunks; c += tw) {
#pragma unroll
            for (int j = 0; j < CH; j++) a[j] = ld_nc(in + c * CH * 32 + j * 32 + lane);
#pragma unroll
            for (int j = 0; j < CH; j++) acc += a[j].x ^ a[j].y ^ a[j].z ^ a[j].w;
        }
    }
    if (acc == 0x12345678) *out = acc;
}


// C: L2-resident read bandwidth: the same `n` int4 are read `reps` times inside one launch (warp-chunk pattern, double-buffered)
__global__ void k_l2_reread(const int4* __restrict__ in, size_t n, int reps, int* out) {
    size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    int acc = 0;
    for (int r = 0; r < reps; r++)
        for (size_t i = tid; i + 7 * stride < n; i += 8 * stride) {
            int4 v[8];
#pragma unroll
            for (int j = 0; j < 8; j++) v[j] = ld_nc(in + i + j * stride);
#pragma unroll
            for (int j = 0; j < 8; j++) acc += v[j].x ^ v[j].y ^ v[j].z ^ v[j].w;
        }
    if (acc == 0x12345678) *out = acc;
}
// D: cp.async.bulk.prefetch.L2 of a region (each thread one `chunk`-byte piece), optional wait, then read it: does the bulk L2
//    prefetch work, and how fast is the read afterwards?  stamps: [0] start, [1] prefetch issued, [2] read done (CTA 0, ns)
__global__ void k_prefetch_then_read(const int4* __restrict__ in, size_t bytes, unsigned chunk, unsigned wait_ns, int do_pf, int* out, unsigned long long* stamps) {
    size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nthreads = (size_t)gridDim.x * blockDim.x;
    unsigned long long t0;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t0));
    if (do_pf)
        for (size_t off = tid * chunk; off < bytes; off += nthreads * chunk) {
            unsigned sz = (unsigned)(bytes - off < chunk ? bytes - off : chunk);
            asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"((const char*)in + off), "r"(sz) : "memory");
        }
    unsigned long long t1;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t1));
    while (true) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); if (t - t0 >= wait_ns) break; }
    unsigned long long t2;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t2));
    size_t n = bytes / 16;
    int acc = 0;
    for (size_t i = tid; i + 7 * nthreads < n; i += 8 * nthreads) {
        int4 v[8];
#pragma unroll
        for (int j = 0; j < 8; j++) v[j] = ld_nc(in + i + j * nthreads);
#pragma unroll
        for (int j = 0; j < 8; j++) acc += v[j].x ^ v[j].y ^ v[j].z ^ v[j].w;
    }
    __syncthreads();
    unsigned long long t3;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t3));
    if (threadIdx.x == 0) { unsigned long long* s = stamps + blockIdx.x * 4; s[0] = t0; s[1] = t1; s[2] = t2; s[3] = t3; }
    if (acc == 0x12345678) *out = acc;
}

template <class F>
static float timeit(F f, int reps = 5) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    f(); cudaDeviceSynchronize();
    float best = 1e9;
    for (int r = 0; r < reps; r++) {
        cudaEventRecord(e0); f(); cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) best = ms;
    }
    return best;
}

int main(int argc, char** argv) {
    size_t bytes = (argc > 1 ? atol(argv[1]) : 512) * (size_t)1 << 20;
    int4* buf; int* out;
    cudaMalloc(&buf, bytes); cudaMalloc(&out, 4);
    cudaMemset(buf, 1, bytes);
    size_t n = bytes / 16;
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    printf("buffer %zu MB\n", bytes >> 20);
#define RUN_A(U, NC, CPS, T) { float ms = timeit([&] { k_gridstride<U, NC><<<sms * CPS, T>>>(buf, n, out); }); \
    printf("A gridstride U=%2d nc=%d ctas/sm=%d threads=%4d : %7.1f GB/s\n", U, NC, CPS, T, bytes / ms / 1e6); }
    RUN_A(4, true, 8, 256) RUN_A(8, true, 8, 256) RUN_A(8, true, 4, 256) RUN_A(16, true, 4, 256) RUN_A(16, true, 2, 256)
    RUN_A(8, false, 8, 256) RUN_A(8, true, 2, 1024) RUN_A(4, true, 2, 1024) RUN_A(8, true, 1, 1024) RUN_A(16, true, 1, 1024)
#define RUN_B(CH, DB, CPS, T) { size_t nc = n / (CH * 32); float ms = timeit([&] { k_warpchunk<CH, DB><<<sms * CPS, T>>>(buf, nc, out); }); \
    printf("B warpchunk CH=%2d (%4d B) db=%d ctas/sm=%d threads=%4d : %7.1f GB/s\n", CH, CH * 512, DB, CPS, T, nc * CH * 512.0 / ms / 1e6); }
    RUN_B(8, false, 8, 256) RUN_B(8, false, 4, 256) RUN_B(8, true, 2, 256) RUN_B(8, true, 4, 256) RUN_B(8, true, 3, 256)
    RUN_B(4, true, 4, 256) RUN_B(4, true, 8, 256) RUN_B(4, false, 8, 256) RUN_B(2, true, 8, 256) RUN_B(16, false, 4, 256) RUN_B(16, true, 2, 256)
    // small-problem behaviour: a 48 MB read (one 11008x4096 Q8_0 matrix) with different buffers each time
    size_t small = (size_t)48 << 20;
    for (int cps : {2, 4, 8}) {
        int rot = 0;
        float ms = timeit([&] { rot = (rot + 1) % 8; k_warpchunk<8, true><<<sms * cps, 256>>>(buf + rot * (small / 16), small / 16 / 256, out); }, 8);
        printf("B 48MB CH=8 db=1 ctas/sm=%d: %7.2f us  %7.1f GB/s\n", cps, ms * 1e3, small / ms / 1e6);
        ms = timeit([&] { rot = (rot + 1) % 8; k_gridstride<8, true><<<sms * cps, 256>>>(buf + rot * (small / 16), small / 16, out); }, 8);
        printf("A 48MB U=8 ctas/sm=%d: %7.2f us  %7.1f GB/s\n", cps, ms * 1e3, small / ms / 1e6);
    }

    // L2-resident re-read (one launch, `reps` passes)
    for (size_t mb : {16, 32, 64, 96}) {
        size_t nn = (mb << 20) / 16; int reps = 20;
        float ms = timeit([&] { k_l2_reread<<<sms * 2, 512>>>(buf, nn, reps, out); }, 3);
        printf("C L2 reread %3zu MB x %d: %7.1f GB/s\n", mb, reps, (double)(mb << 20) * reps / ms / 1e6);
    }
    // bulk L2 prefetch, wait, read: per-CTA max of (read time); fresh region every run (rotating through the big buffer)
    {
        unsigned long long* st; cudaMalloc(&st, sms * 4 * 8);
        std::vector<unsigned long long> h(sms * 4);
        int rot = 0;
        for (size_t mb : {16, 48, 96})
            for (int pf = 0; pf < 2; pf++)
                for (unsigned chunk : {4096u, 16384u})
                    for (unsigned wait_us : {0u, 20u, 40u}) {
                        if (!pf && chunk != 4096u) continue;
                        size_t bytes_r = mb << 20;
                        rot = (rot + 1) % 4;
                        const int4* base = buf + (size_t)rot * ((size_t)100 << 20) / 16;
                        k_prefetch_then_read<<<sms, 512>>>(base, bytes_r, chunk, wait_us * 1000, pf, out, st);
                        cudaDeviceSynchronize();
                        cudaMemcpy(h.data(), st, h.size() * sizeof(h[0]), cudaMemcpyDeviceToHost);
                        unsigned long long t0 = ~0ull, tpf = 0, t2 = ~0ull, t3 = 0;
                        for (int b = 0; b < sms; b++) { if (h[b*4] < t0) t0 = h[b*4]; if (h[b*4+1] > tpf) tpf = h[b*4+1]; if (h[b*4+2] < t2) t2 = h[b*4+2]; if (h[b*4+3] > t3) t3 = h[b*4+3]; }
                        printf("D %3zu MB pf=%d chunk=%5u wait=%2u us: issue %6.2f us, read %7.2f us = %7.1f GB/s, total %7.2f us\n", mb, pf, chunk, wait_us,
                               (tpf - t0) / 1e3, (t3 - t2) / 1e3, bytes_r / ((t3 - t2) / 1e9) / 1e9, (t3 - t0) / 1e3);
                    }
    }
    return 0;
}
