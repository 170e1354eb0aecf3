// mega.cu -- one persistent kernel per token ("megakernel") for the fused decode path of phase tables WITHOUT a Q8_0 / Q4_0 matvec:
// K-quant weights (the generic MATVEC phase of mega_phases.cuh) and flushes with no matvec at all (a sampler or an attention phase
// alone).  Tables with a streaming Q8_0 / Q4_0 phase run mega_ring.cu (weights through a TMA-fed shared-memory ring: DESIGN.md
// section 4.5).  The phase bodies both kernels share live in mega_phases.cuh; the host side at the bottom of this file serves both.
//
// Why: a kernel boundary costs a few us for a full-GPU streaming kernel (drain, launch latency,
// ramp-up); a fused Llama-2-7B token still has ~260 of them, of the order of the time the weights need at HBM speed.  Here the whole token is ONE launch of one 512-thread CTA per SM that walks a table of
// phases (built by lazy.cu from the recorded trait calls) separated by grid-wide barriers:
//     MATVEC  K-quant matvec over 1-3 matrices + epilogue, with a fused prologue ([dup] + rms_norm * w + Q8_K quantisation of the
//             input row, recomputed by every CTA)
//     NORMQ   normalise + Q8_0 quantise as a phase of its own
//     ATTN    rope + KV append + attention + output quantise    (up to 4 CTAs per head, K/V chunks through a TMA pipeline)
//     ROWS    copy_rows_from (embedding row dequantisation)
//     ARGMAX / SAMPLE   the next token on the device
// The per-phase time breakdown: tools/mega_profile.py.
// Data written by one CTA and read by another in a later phase is always read with ld.global.cg (L2), never through
// the non-coherent L1.  All CTAs execute the same number of barriers.
#define MK_SYNC() __syncthreads()
#include "mega_phases.cuh"

// norm weights of the next MATVEC phase's fused prologue, fetched one word per thread at phase start
struct MkNextNorm { const float* norm_w; int norm_n; };

// SMP: the table ends with its only SAMPLE phase, run after the phase loop.  Only these instantiations carry the call, so the greedy ones keep
// their register allocation.
template <bool SMP>
__global__ void __launch_bounds__(MK_THREADS, MK_CTAS_PER_SM) mega_kernel(const MkPhase* __restrict__ phases, int n_phases, const uint8_t* dyn,
                                                                         unsigned* bar, const uint16_t* exp_lut, unsigned long long* prof, bool test_stall, int wtop_off,
                                                                         unsigned* err_host, float* scores) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ float s_red[MK_WARPS];
    __shared__ MkPhase s_phs[2];             // phase descriptors, double-buffered: p+1 is fetched while p runs
    __shared__ MkNextNorm s_next;            // norm weights of the next MATVEC phase
    __shared__ int s_abort;
    __shared__ __align__(8) unsigned long long s_abar[AT_NBUF];                // attention chunk buffers (TMA completion)
    unsigned apar = 0u;                      // per-buffer wait parity of the attention chunk pipeline
    const unsigned abar0 = (unsigned)__cvta_generic_to_shared(&s_abar[0]);
    if (threadIdx.x == 0) { for (int i = 0; i < AT_NBUF; i++) mbar_init(abar0 + 8u * i, 1u); s_abort = 0; }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const CommDev nocomm = {};               // no exchange phase runs here (lazy.cu builds them for Q8_0 / Q4_0 tables only)
    KSeg S0, S1;                             // weight segments in flight of the generic MATVEC phase (MK_GENERIC_SEGS)
    uint8_t* work = smem;                    // per-phase working area (activation arrays, attention tiles)
    float* s_w = (float*)(smem + wtop_off);  // norm weights of the next fused prologue (top of dynamic shared memory)
    int wstaged = -1;                        // phase index whose norm weights were requested into s_w
    int xstaged = -1;                        // phase index whose f32 input row was requested into its prologue's staging area
    unsigned gen = 0;                        // barriers completed; starts from the value left by the last launch
    if (threadIdx.x == MK_BAR_THREAD) gen = ld_acquire_u32(&bar[32]);
    {
        const int* src = (const int*)phases;
        int* dst = (int*)&s_phs[0];
        for (int i = threadIdx.x; i < (int)(sizeof(MkPhase) / 4); i += MK_THREADS) dst[i] = src[i];
    }
    const int n_loop = SMP ? n_phases - 1 : n_phases;      // SMP: the last phase, the sampler, runs after the loop
    for (int p = 0; p < n_loop; p++) {
        // developer profiling, 4 stamps per phase from CTA 0 / thread 0: start, activation ready (MATVEC), rows done, arrived + norm weights requested
        const bool stamp = prof && blockIdx.x == 0 && threadIdx.x == 0;
        if (stamp) { prof[p * MK_PROF_SLOTS] = globaltimer_ns(); prof[p * MK_PROF_SLOTS + 1] = 0; prof[p * MK_PROF_SLOTS + 4] = 0; prof[p * MK_PROF_SLOTS + 5] = 0; }
        __syncthreads();                     // descriptor p is in shared memory (stored one phase ago)
        const MkPhase& s_ph = s_phs[p & 1];
        // Descriptor p+1 and the norm weights of the next MATVEC phase are LOADED now, into one register each, and STORED to shared
        // memory after the phase body: a load followed directly by its st.shared would block the thread for an L2 round trip
        // (in-order issue) before it could issue the phase's own loads.
        static_assert(sizeof(MkPhase) / 4 <= MK_THREADS, "descriptor does not fit one word per thread");
        const int nx = s_ph.next_matvec;
        const bool look = nx > p && nx < n_phases;
        int desc_w = 0, next_w = 0;
        if (p + 1 < n_phases && threadIdx.x < sizeof(MkPhase) / 4) desc_w = ((const int*)(phases + p + 1))[threadIdx.x];
        // only weights no phase of the table writes (norm_ahead): they are requested before the barrier, i.e. before the phases in
        // between have finished on every CTA
        if (look && threadIdx.x < 3) {
            const MkPhase* ph = phases + nx;
            next_w = threadIdx.x < 2 ? ((const int*)&ph->norm_w)[threadIdx.x] : ph->x && ph->norm_w && ph->norm_ahead ? ph->n : 0;
        }
        switch (s_ph.type) {
        case MK_NORMQ: phase_normq(s_ph, s_red); break;
        case MK_MATVEC: {                    // K-quant weights: the generic phase
            unsigned long long* st1 = stamp ? prof + p * MK_PROF_SLOTS + 1 : nullptr;
            switch (s_ph.wtype) {
            case CC_Q2_K: phase_matvec_generic<TQ2_K>(s_ph, work, s_w, wstaged == p, xstaged == p, exp_lut, st1, S0, S1); break;
            case CC_Q3_K: phase_matvec_generic<TQ3_K>(s_ph, work, s_w, wstaged == p, xstaged == p, exp_lut, st1, S0, S1); break;
            case CC_Q4_K: phase_matvec_generic<TQ45_K<false>>(s_ph, work, s_w, wstaged == p, xstaged == p, exp_lut, st1, S0, S1); break;
            case CC_Q5_K: phase_matvec_generic<TQ45_K<true>>(s_ph, work, s_w, wstaged == p, xstaged == p, exp_lut, st1, S0, S1); break;
            case CC_Q6_K: phase_matvec_generic<TQ6_K>(s_ph, work, s_w, wstaged == p, xstaged == p, exp_lut, st1, S0, S1); break;
            default: phase_matvec_generic<TQ8_K>(s_ph, work, s_w, wstaged == p, xstaged == p, exp_lut, st1, S0, S1); break;
            }
            break;
        }
        case MK_ATTN:
            if (s_ph.at.kv_f16) phase_attn<true, false>(s_ph, (float*)work, s_red, dyn, exp_lut, abar0, apar, AT_CH, bar, err_host, &s_abort, scores);
            else phase_attn<false, false>(s_ph, (float*)work, s_red, dyn, exp_lut, abar0, apar, AT_CH, bar, err_host, &s_abort, scores);
            break;
        case MK_ROWS: phase_rows(s_ph, dyn); break;
        case MK_ARGMAX: phase_argmax(s_ph, dyn, s_red); break;
        }
        if (stamp) prof[p * MK_PROF_SLOTS + 2] = globaltimer_ns();
        if (p + 1 < n_phases && threadIdx.x < sizeof(MkPhase) / 4) ((int*)&s_phs[(p + 1) & 1])[threadIdx.x] = desc_w;
        if (look && threadIdx.x < 3) ((int*)&s_next)[threadIdx.x] = next_w;
        const bool more = p + 1 < n_phases;
        // test hook (tests/test_gpu_robustness.py): one CTA deserts before the third barrier, as if it had never become resident
        if (test_stall && p == 2 && blockIdx.x == gridDim.x - 1) { if (threadIdx.x == 0) s_abort = 1; break; }
        if (more) grid_barrier_arrive(bar, gridDim.x, gen);       // its bar.sync also publishes s_next (written just above)
        // immutable norm weights of the next fused prologue, requested before waiting at the barrier: one L2 trip less after it
        if (look && s_next.norm_n > 0) {
            const unsigned sw = (unsigned)__cvta_generic_to_shared(s_w);
            const float* nw = s_next.norm_w;
            for (int i = threadIdx.x; i < (s_next.norm_n >> 2); i += MK_THREADS)
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sw + i * 16), "l"(nw + i * 4) : "memory");
            asm volatile("cp.async.commit_group;" ::: "memory");
            wstaged = nx;
        }
        if (stamp) prof[p * MK_PROF_SLOTS + 3] = globaltimer_ns();
        if (more) {
            grid_barrier_wait(bar, gridDim.x, gen, nocomm, 0u, &s_abort, err_host);
            gen++;
            if (s_abort) break;              // a barrier timed out (a CTA never became resident): bail out, host reports
            // the barrier is open: the row the next fused prologue normalises is complete -- request it before anything else (descriptor
            // bookkeeping, geometry) so that its L2 round trip overlaps them
            const MkPhase& nph = s_phs[(p + 1) & 1];
            if (nph.type == MK_MATVEC && nph.x) {
                const unsigned sx = (unsigned)__cvta_generic_to_shared(work + mk_generic_sx_offset(nph.mv.k));      // = s_x of the phase's prologue
                const float* xg = nph.x;
                for (int i = threadIdx.x; i < (nph.mv.k >> 2); i += MK_THREADS)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sx + i * 16), "l"(xg + i * 4) : "memory");
                asm volatile("cp.async.commit_group;" ::: "memory");
                xstaged = p + 1;
            }
        }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");      // a launch that gave up may still have norm-weight or x-row copies in flight
    // the SAMPLE phase (lazy.cu: the only one, and the last): called after the loop, so the call saves nothing around itself (the
    // barrier before it was the last iteration's)
    if constexpr (SMP) {
        __syncthreads();
        if (!s_abort) phase_sample(s_phs[(n_phases - 1) & 1], dyn, work, exp_lut);
    }
    if (prof && blockIdx.x == 0 && threadIdx.x == 0) prof[n_phases * MK_PROF_SLOTS] = globaltimer_ns();
}

// working shared memory of one phase (the staging area of the norm weights comes on top: MegaLaunch::wstage); a MATVEC phase here is
// generic (K-quant weights): the streaming ones run mega_ring.cu, whose working areas are cc_mega_ring_smem_for_phase
size_t cc_mega_smem_for_phase(const MkPhase& ph) {
    if (ph.type == MK_MATVEC) return (size_t)(((TKBase::smem_bytes(ph.mv.k) + 15) & ~15) + 256) + (size_t)ph.mv.k * 4;
    if (ph.type == MK_ATTN) return (size_t)(3 * ph.at.hd + ((ph.at.max_len + 8 + 3) & ~3) + AT_NBUF * AT_CH * ph.at.hd) * 4 + 64;
    if (ph.type == MK_SAMPLE) return SMP_SMEM_BYTES;
    return 1024;
}

// developer hook: a table of `n` empty phases -> the pure per-phase floor (descriptor fetch + grid barrier)
extern "C" CC_API int cc_test_mega_barrier_floor(cc_device* dev, int n, float* us_per_phase) {
    if (!dev || n < 2 || !us_per_phase) return CC_ERR_ARG;
    std::vector<MkPhase> tab((size_t)n);
    for (auto& p : tab) { memset(&p, 0, sizeof(p)); p.type = 99; p.next_matvec = -1; }
    MkPhase* d_tab = nullptr; unsigned* d_bar = nullptr;
    CC_CUDA(dev, cudaMalloc(&d_tab, tab.size() * sizeof(MkPhase)));
    CC_CUDA(dev, cudaMalloc(&d_bar, 4096));
    CC_CUDA(dev, cudaMemcpy(d_tab, tab.data(), tab.size() * sizeof(MkPhase), cudaMemcpyHostToDevice));
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    float best = 1e30f;
    for (int rep = 0; rep < 4; rep++) {
        CC_CUDA(dev, cudaMemsetAsync(d_bar, 0, 4096, dev->stream));
        cudaEventRecord(e0, dev->stream);
        MegaLaunch L;
        L.variant = MEGA_REGISTER;
        int rc = cc_launch_mega(dev, d_tab, n, nullptr, d_bar, L, nullptr);
        if (rc) return rc;
        cudaEventRecord(e1, dev->stream);
        CC_CUDA(dev, cudaEventSynchronize(e1));
        float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) best = ms;
    }
    *us_per_phase = best * 1e3f / (float)n;
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(d_tab); cudaFree(d_bar);
    return CC_OK;
}

// CTAs per head of the attention phase (mega_phases.cuh phase_attn) in a grid of `grid` CTAs: the largest of 4, 2, 1 for which every
// CTA owns whole Q8_0 blocks of the head's output (hd % (32 S) == 0) and every CTA serves one head at most (n_heads S <= grid), so no CTA
// waits for a peer that is still busy with another head.  a.split is the most the score scratch allows (1: none); with more heads than
// arrival words, one CTA per head.
int cc_attn_split(const AttnArgs& a, int grid) {
    if (a.split <= 1 || a.n_heads > AT_SPLIT_MAX_HEADS) return 1;
    for (int S = AT_SPLIT_MAX; S > 1; S >>= 1)
        if (a.hd % (32 * S) == 0 && a.n_heads * S <= grid) return S;
    return 1;
}

bool cc_mega_generic_supported(int type, int64_t k) {
    return (type == CC_Q2_K || type == CC_Q3_K || type == CC_Q4_K || type == CC_Q5_K || type == CC_Q6_K || type == CC_Q8_K) && k % 256 == 0 && k <= 32768;
}

// test hook of both persistent kernels: bit 0x80 (MK_F_TESTSTALL) of CRABML_MEGA_FLAGS; the word's other bits have no effect
bool cc_mega_test_stall() {
    static const bool on = getenv("CRABML_MEGA_FLAGS") && (strtol(getenv("CRABML_MEGA_FLAGS"), nullptr, 0) & MK_F_TESTSTALL);
    return on;
}

int cc_launch_mega(cc_device* dev, const MkPhase* phases_dev, int n_phases, const uint8_t* dyn_dev, unsigned* bar_dev, const MegaLaunch& L,
                   unsigned long long* prof) {
    int max_ctas_per_sm = 0;
    const size_t wtop = (L.smem + 15) & ~(size_t)15;
    const size_t smem = wtop + L.wstage;
    CC_REQUIRE(dev, smem <= 227 * 1024, "megakernel: a phase needs %zu bytes of shared memory", smem);
    auto kern = L.sample ? mega_kernel<true> : mega_kernel<false>;
    if (smem > 48 * 1024) CC_CUDA(dev, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CC_CUDA(dev, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&max_ctas_per_sm, kern, MK_THREADS, smem));
    CC_REQUIRE(dev, max_ctas_per_sm >= 1, "megakernel does not fit on an SM");
    int per_sm = max_ctas_per_sm < MK_CTAS_PER_SM ? max_ctas_per_sm : MK_CTAS_PER_SM;
    const uint16_t* lut = dev->exp_lut;
    return mk_launch(dev, kern, dev->sm_count * per_sm, MK_THREADS, smem, phases_dev, n_phases, dyn_dev, bar_dev, lut, prof, cc_mega_test_stall(),
                     (int)wtop, dev->err_host, L.scores);
}
