// mega.cu -- one persistent kernel per token ("megakernel") for the fused decode path: the variant whose weight stream runs through
// REGISTERS (two segments per warp in flight, look-ahead prefetch across the grid barrier).  Since round 2 the default is the variant in
// mega_ring.cu (weights through a TMA-fed shared-memory ring: DESIGN.md section 4.5); this one is the fallback (CRABML_MEGA_FLAGS without
// MK_F_RING, or a phase table whose working area leaves the ring fewer than 12 slots) and the A/B baseline.  The phase bodies both
// kernels share live in mega_phases.cuh; the host side at the bottom of this file serves both.
//
// Why: a kernel boundary costs a few us for a full-GPU streaming kernel (drain, launch latency,
// ramp-up); a fused Llama-2-7B token still has ~260 of them, of the order of the time the weights need at HBM speed.  Here the whole token is ONE launch of one 512-thread CTA per SM that walks a table of
// phases (built by lazy.cu from the recorded trait calls) separated by grid-wide barriers:
//     MATVEC  streaming matvec over 1-3 matrices + epilogue, optionally with a fused prologue ([dup] + rms_norm * w + Q8_0
//             quantisation of the input row, recomputed by every CTA) and, on the sharded path, the exchange with the other GPUs
//     NORMQ   the same normalise + quantise as a phase of its own (only when the f32 row must be materialised)
//     ATTN    rope + KV append + attention + output quantise    (one CTA per head, K/V chunks through a TMA pipeline)
//     ROWS    copy_rows_from (embedding row dequantisation)
//     REDUCE / GATHER   second half of an exchange when it cannot fold into the next MATVEC prologue
// The per-phase time breakdown: tools/mega_profile.py.
// Data written by one CTA and read by another in a later phase is always read with ld.global.cg (L2), never through
// the non-coherent L1.  All CTAs execute the same number of barriers.
#define MK_SYNC() __syncthreads()
#include "mega_phases.cuh"

// Issue the loads of this warp's first two segments of a MATVEC phase (register stages).  Weights are immutable, so this may run
// long before the phase itself -- across barriers and small phases -- keeping HBM busy while the grid synchronises.
template <int TYPE>
__device__ __forceinline__ void matvec_prefetch(const StreamArgs& A, MkPipe& P) {
    const int lane = threadIdx.x & 31;
    const MkGeo g = mk_geo(A);
    int l_i = 0, l_seg = 0;
    MkRowPtr l_ptr = mk_vrow_ptr<TYPE>(A.mats, g, 0, lane);
    auto advance_load = [&]() { if (++l_seg == g.NSEG) { l_seg = 0; l_ptr = mk_vrow_ptr<TYPE>(A.mats, g, ++l_i, lane); } };
    mk_seg_load<TYPE>(P.buf0, l_ptr, l_seg, g.nb, g.GR, g.last_half_off, lane, g.U > 0); advance_load();
    mk_seg_load<TYPE>(P.buf1, l_ptr, l_seg, g.nb, g.GR, g.last_half_off, lane, g.U > 1);
}

// precondition: the pipe holds this warp's segments 0, 1 (matvec_prefetch).  s_w: staging area of the norm weights at the top
// of dynamic shared memory; w_staged: they were already requested there (cp.async, before the barrier) by the look-ahead.
template <int TYPE>
__device__ void phase_matvec(const MkPhase& ph, uint8_t* smem, float* s_w, bool w_staged, bool x_staged, const uint16_t* exp_lut, MkPipe& P,
                             const CommDev& comm, unsigned xseq, unsigned long long* stamp1, const MkNext* early_next, int next_w) {
    const StreamArgs& A = ph.mv;
    const int k = A.k;
    const MkGeo g = mk_geo(A);
    const int nb = g.nb, GR = g.GR, NSEG = g.NSEG, U = g.U, gw = g.gw, TW = g.TW;
    const bool pair = g.pair;
    const int nbp = NSEG * MK_SEG * 32;
    int8_t* s_q = (int8_t*)smem;
    float* s_d = (float*)(smem + (size_t)nbp * 32);
    int* s_s = (int*)(smem + (size_t)nbp * 32 + (size_t)nbp * 4);
    const int lane = threadIdx.x & 31;
    const StreamMats& M = A.mats;
    // load cursor: points at segment 2
    int l_i = 0, l_seg = 0;
    MkRowPtr l_ptr = mk_vrow_ptr<TYPE>(M, g, 0, lane);
    auto advance_load = [&]() { if (++l_seg == NSEG) { l_seg = 0; l_ptr = mk_vrow_ptr<TYPE>(M, g, ++l_i, lane); } };
    if (++l_seg == NSEG) { l_seg = 0; l_ptr = mk_vrow_ptr<TYPE>(M, g, ++l_i, lane); }       // -> segment 1 (already requested)
    if (++l_seg == NSEG) { l_seg = 0; l_ptr = mk_vrow_ptr<TYPE>(M, g, ++l_i, lane); }       // -> segment 2
    MkSeg& buf0 = P.buf0;
    MkSeg& buf1 = P.buf1;
    if (ph.x) {
        // Fused prologue: [rms_norm * w] + Q8_0 quantisation of x, computed by EVERY CTA straight into its shared memory
        // (redundant across SMs) -- cheaper than a separate NORMQ phase, which costs a grid barrier plus its own latency chain.  The weight segments requested by matvec_prefetch are in flight meanwhile.
        const int n = k;
        const int warp = threadIdx.x >> 5;
        float* s_red = (float*)(smem + (size_t)nbp * 40);                // scratch behind the activation arrays (256 B), then the 2 KB exchange stage
        float* s_x = s_red + 64 + 512;                                    // f32 copy of x
        {   // one L2 round trip: every 16-byte chunk of x (and of the norm weights) requested at once
            const int n4 = n >> 2;
            const unsigned sx = (unsigned)__cvta_generic_to_shared(s_x), sw = (unsigned)__cvta_generic_to_shared(s_w);
            if (ph.norm_w && !w_staged)
                for (int i = threadIdx.x; i < n4; i += MK_THREADS)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sw + i * 16), "l"(ph.norm_w + i * 4) : "memory");
            if (ph.red_n) {
                // second half of the exchange that ended the previous phase (comm.cu): x = sum over ranks of the partial rows
                // in rank order (+ residual), rebuilt by every CTA from this GPU's window -- no separate REDUCE phase
                const float* base = comm.data[comm.rank] + (size_t)(xseq & 1u) * CC_COMM_MAX_RANKS * CC_COMM_MAX_ELEMS;
                for (int i = threadIdx.x; i < n4; i += MK_THREADS) {
                    float4 acc4 = __ldcg((const float4*)base + i);
                    for (int p = 1; p < comm.world; p++) {
                        const float4 t4 = __ldcg((const float4*)(base + (size_t)p * CC_COMM_MAX_ELEMS) + i);
                        acc4.x += t4.x; acc4.y += t4.y; acc4.z += t4.z; acc4.w += t4.w;
                    }
                    if (ph.red_res) { const float4 r4 = __ldcg((const float4*)ph.red_res + i); acc4.x += r4.x; acc4.y += r4.y; acc4.z += r4.z; acc4.w += r4.w; }
                    ((float4*)s_x)[i] = acc4;
                }
            } else if (!x_staged) {
                for (int i = threadIdx.x; i < n4; i += MK_THREADS)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sx + i * 16), "l"(ph.x + i * 4) : "memory");
            }
            asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
            __syncthreads();
            if (stamp1) stamp1[3] = globaltimer_ns();          // x (and the norm weights) are in shared memory
        }
        float rms = 1.0f;
        if (ph.norm_w) {
            float ss = 0.0f;
            const float4* x4 = (const float4*)s_x;
            for (int i = threadIdx.x; i < (n >> 2); i += MK_THREADS) { float4 v = x4[i]; ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w; }
            ss = warp_sum(ss);
            if (lane == 0) s_red[warp] = ss;
            __syncthreads();
            float t = 0.0f;
#pragma unroll
            for (int w = 0; w < MK_WARPS; w++) t += s_red[w];
            rms = sqrtf(t / (float)n + ph.eps);
        }
        if (stamp1) stamp1[4] = globaltimer_ns();              // rms known
        if (ph.orig && blockIdx.x == 0)                              // Tensor::dup of the un-normalised row (llama2.rs:227,607)
            for (int i = threadIdx.x; i < (n >> 2); i += MK_THREADS) ((float4*)ph.orig)[i] = ((const float4*)s_x)[i];
        // quantise: 4 consecutive elements per thread, 8 threads per 32-block, 64 blocks per pass (same arithmetic per element as
        // quantize.cu: d = amax / 127, q = trunc(x / d), stored scale = f32(f16(d)))
        const int sub = threadIdx.x & 7;
        for (int b = threadIdx.x >> 3; b < nbp; b += MK_THREADS / 8) {        // nbp % 128 == 0: uniform trip count per warp
            const bool live = b < nb;
            float4 v = live ? ((const float4*)s_x)[b * 8 + sub] : make_float4(0, 0, 0, 0);
            if (ph.norm_w && live) {
                const float4 w4 = ((const float4*)s_w)[b * 8 + sub];
                v.x = (v.x / rms) * w4.x; v.y = (v.y / rms) * w4.y; v.z = (v.z / rms) * w4.z; v.w = (v.w / rms) * w4.w;
            }
            float amax = fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)));
#pragma unroll
            for (int o = 4; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
            const float d = amax / 127.0f;
            const int q0 = live ? __float2int_rz(v.x / d) : 0, q1 = live ? __float2int_rz(v.y / d) : 0;
            const int q2 = live ? __float2int_rz(v.z / d) : 0, q3 = live ? __float2int_rz(v.w / d) : 0;
            ((int*)s_q)[b * 8 + sub] = (q0 & 255) | ((q1 & 255) << 8) | ((q2 & 255) << 16) | (q3 << 24);
            if constexpr (TYPE == CC_Q4_0) {
                int sq = q0 + q1 + q2 + q3;
#pragma unroll
                for (int o = 4; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
                if (sub == 0) s_s[b] = sq;
            }
            if (sub == 0) s_d[b] = live ? __half2float(__float2half_rn(d)) : 0.0f;
        }
    } else {   // stage the quantised activation (written by other CTAs in the previous phase: L2 loads)
        const uint8_t* act = (const uint8_t*)A.act;
        const int4* gq = (const int4*)act;
        int4* sq4 = (int4*)s_q;
        const float* gd = (const float*)(act + ((k + 15) & ~15));
        const int* gs = (const int*)(act + ((k + 15) & ~15) + ((nb * 4 + 15) & ~15));
        if (nbp <= MK_THREADS) {           // every load of the thread is issued before its first store (one L2 round trip, not three)
            const int i0 = threadIdx.x, i1 = threadIdx.x + MK_THREADS;
            const int4 z4 = make_int4(0, 0, 0, 0);
            const int4 qa = i0 < nb * 2 ? __ldcg(gq + i0) : z4, qb = i1 < nb * 2 ? __ldcg(gq + i1) : z4;
            const float dv = i0 < nb ? __ldcg(gd + i0) : 0.0f;
            int sv = 0;
            if constexpr (TYPE == CC_Q4_0) sv = i0 < nb ? __ldcg(gs + i0) : 0;
            if (i0 < nbp * 2) sq4[i0] = qa;
            if (i1 < nbp * 2) sq4[i1] = qb;
            if (i0 < nbp) { s_d[i0] = dv; if constexpr (TYPE == CC_Q4_0) s_s[i0] = sv; }
        } else {
            for (int i = threadIdx.x; i < nbp * 2; i += MK_THREADS) sq4[i] = i < nb * 2 ? __ldcg(gq + i) : make_int4(0, 0, 0, 0);
            for (int i = threadIdx.x; i < nbp; i += MK_THREADS) {
                s_d[i] = i < nb ? __ldcg(gd + i) : 0.0f;
                if constexpr (TYPE == CC_Q4_0) s_s[i] = i < nb ? __ldcg(gs + i) : 0;
            }
        }
    }
    if (early_next && threadIdx.x < 128) {      // look-ahead arguments (loaded at phase start) become visible with the barrier below
        const int slot = threadIdx.x >> 6, t = threadIdx.x & 63;
        if (t < (int)(sizeof(StreamArgs) / 4) + 4) ((int*)&early_next[slot])[t] = next_w;
    }
    __syncthreads();
    if (stamp1) *stamp1 = globaltimer_ns();
    const int4* aq_l = (const int4*)s_q + 2 * lane;
    const float* ad_l = s_d + lane;
    const int* as_l = s_s + lane;
    float* s_part = (float*)(smem + (size_t)nbp * 40 + 256);             // exchange stage: this CTA's block of partial rows (<= MK_XSTAGE_ROWS floats)
    float acc = 0.0f, first = 0.0f;
    int c_i = 0, c_seg = 0;
    // Epilogues that need a value from memory (the residual, or the exp LUT entry of silu) are finished ONE ROW LATER: the load
    // is issued when the row's dot is known and consumed after the next row, so the warp never stalls an L2 round trip with its
    // weight stream idle (in-order issue).  lane 0 only.
    float pend_a = 0.0f, pend_b = 0.0f, pend_res = 0.0f;
    unsigned short pend_lut = 0;
    int pend_row = -1;
    auto flush_pending = [&]() {
        if (lane == 0 && pend_row >= 0) {
            if (pair) M.out[0][pend_row] = (pend_a / (1.0f + h2f_bits(pend_lut))) * pend_b;
            else M.out[0][pend_row] = pend_a + pend_res;
        }
        pend_row = -1;
    };
    auto finish_segment = [&]() {
        if (++c_seg < NSEG) return;
        c_seg = 0;
        float r = warp_sum(acc);
        acc = 0.0f;
        const int i = c_i++;
        if (pair) {
            if ((i & 1) == 0) { first = r; return; }
            flush_pending();
            if (lane == 0) {
                pend_a = first; pend_b = r; pend_row = gw + (i >> 1) * TW;
                pend_lut = exp_lut[f2h_bits(-first)];
            }
            return;
        }
        if (A.epilogue == 1) {                 // single matrix: out = dot + residual (llama2.rs:266,636)
            flush_pending();
            if (lane == 0) { pend_a = r; pend_row = gw + i * TW; pend_res = ldcg_f(A.residual + pend_row); }
            return;
        }
        if (lane == 0) {
            int mat = 0, rr = gw + i * TW;
            if (M.n > 1 && rr >= M.m[0]) { rr -= M.m[0]; mat = 1; if (M.n > 2 && rr >= M.m[1]) { rr -= M.m[1]; mat = 2; } }
            if (A.epilogue == 3) {         // partial row -> this CTA's stage; sent to the peers as one run when the phase body is done
                s_part[rr - (int)blockIdx.x * g.rpc] = r;
                return;
            }
            float* o = mat == 0 ? M.out[0] : mat == 1 ? M.out[1] : M.out[2];
            o[rr] = r;
        }
    };
    for (int u = 0; u < U; u += 2) {          // two segments (8 KB of Q8_0) in flight per warp at all times
        acc += mk_seg_dot<TYPE>(buf0, c_seg, aq_l, ad_l, as_l);
        finish_segment();
        mk_seg_load<TYPE>(buf0, l_ptr, l_seg, nb, GR, g.last_half_off, lane, u + 2 < U);
        advance_load();
        if (u + 1 >= U) break;
        acc += mk_seg_dot<TYPE>(buf1, c_seg, aq_l, ad_l, as_l);
        finish_segment();
        mk_seg_load<TYPE>(buf1, l_ptr, l_seg, nb, GR, g.last_half_off, lane, u + 3 < U);
        advance_load();
    }
    flush_pending();
    if (A.epilogue == 3) {
        // the CTA's block of partial rows -> slot[rank] of every GPU's exchange window: warp p serves peer p with ONE coalesced NVLink
        // store of 16 bytes per lane (28 rows = 112 contiguous bytes at 7B shapes) instead of one 4-byte store per row and peer
        __syncthreads();
        const int warp = threadIdx.x >> 5;
        const int first_row = (int)blockIdx.x * g.rpc;
        const int m_all = M.m[0];
        const int cnt = min(g.rpc, max(0, m_all - first_row));
        if (warp < comm.world) {
            const size_t off = ((size_t)((xseq + 1u) & 1u) * CC_COMM_MAX_RANKS + comm.rank) * CC_COMM_MAX_ELEMS + first_row;
            for (int c4 = lane * 4; c4 < cnt; c4 += 128) *(float4*)(comm.data[warp] + off + c4) = *(const float4*)(s_part + c4);
        }
    }
    // this warp is done: its register stages are free, so it requests its first segments of the next MATVEC phase right away instead
    // of idling until the slowest warp of the CTA reaches the barrier (the tail of a phase becomes prefetch time)
    if (early_next) { if (early_next[0].wtype == CC_Q8_0) matvec_prefetch<CC_Q8_0>(early_next[0].mv, P); else if (early_next[0].wtype == CC_Q4_0) matvec_prefetch<CC_Q4_0>(early_next[0].mv, P); }
}

// GEN: the phase table contains generic (K-quant) MATVEC phases.  The streaming-only instantiation carries none of their code, so
// its register allocation (the weight pipe lives in registers across phases) is not disturbed by them.
// SMP: the table ends with its only SAMPLE phase, run after the phase loop.  Only these instantiations carry the call, so the greedy ones keep
// their register allocation.
template <bool GEN, bool SMP>
__global__ void __launch_bounds__(MK_THREADS, MK_CTAS_PER_SM) mega_kernel(const MkPhase* __restrict__ phases, int n_phases, const uint8_t* dyn,
                                                                         unsigned* bar, const uint16_t* exp_lut, unsigned long long* prof, int flags, int wtop_off,
                                                                         unsigned* err_host, const CommDev comm) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ float s_red[MK_WARPS];
    __shared__ MkPhase s_phs[2];             // phase descriptors, double-buffered: p+1 is fetched while p runs
    __shared__ MkNext s_next[2];             // arguments of the next two MATVEC phases (look-ahead prefetch)
    __shared__ int s_abort;
    __shared__ __align__(8) unsigned long long s_abar[AT_NBUF];                // attention chunk buffers (TMA completion)
    unsigned apar = 0u;                      // per-buffer wait parity of the attention chunk pipeline
    const unsigned abar0 = (unsigned)__cvta_generic_to_shared(&s_abar[0]);
    if (threadIdx.x == 0) { for (int i = 0; i < AT_NBUF; i++) mbar_init(abar0 + 8u * i, 1u); s_abort = 0; }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    MkPipe pipe;                             // weight prefetch registers, live across phases and barriers
    uint8_t* work = smem;                    // per-phase working area (activation arrays, attention tiles)
    float* s_w = (float*)(smem + wtop_off);  // norm weights of the next fused prologue (top of dynamic shared memory)
    int prefetched = -1;                     // phase index whose first segments sit in the pipe
    int wstaged = -1;                        // phase index whose norm weights were requested into s_w
    int xstaged = -1;                        // phase index whose f32 input row was requested into its prologue's staging area
    unsigned gen = 0;                        // barriers completed; starts from the value left by the last launch
    if (threadIdx.x == MK_BAR_THREAD) gen = ld_acquire_u32(&bar[32]);
    unsigned xseq = comm.world > 0 ? *comm.seq : 0u;     // exchanges finished so far on this rank (comm.cu)
    {
        const int* src = (const int*)phases;
        int* dst = (int*)&s_phs[0];
        for (int i = threadIdx.x; i < (int)(sizeof(MkPhase) / 4); i += MK_THREADS) dst[i] = src[i];
    }
    const int n_loop = SMP ? n_phases - 1 : n_phases;      // SMP: the last phase, the sampler, runs after the loop
    for (int p = 0; p < n_loop; p++) {
        // developer profiling, 4 stamps per phase from CTA 0 / thread 0: start, activation ready (MATVEC), rows done, arrived + prefetch issued
        const bool stamp = prof && blockIdx.x == 0 && threadIdx.x == 0;
        if (stamp) { prof[p * MK_PROF_SLOTS] = globaltimer_ns(); prof[p * MK_PROF_SLOTS + 1] = 0; prof[p * MK_PROF_SLOTS + 4] = 0; prof[p * MK_PROF_SLOTS + 5] = 0; }
        __syncthreads();                     // descriptor p is in shared memory (stored one phase ago)
        const MkPhase& s_ph = s_phs[p & 1];
        // Descriptor p+1 and the arguments of the next MATVEC phases (look-ahead prefetch) are LOADED now, into one register each,
        // and STORED to shared memory after the phase body: a load followed directly by its st.shared would block the thread for
        // an L2 round trip (in-order issue) before it could issue the phase's own loads.
        static_assert(sizeof(MkPhase) / 4 <= MK_THREADS, "descriptor does not fit one word per thread");
        const int nx = s_ph.next_matvec, nx2 = s_ph.next_matvec2;
        const bool look = (flags & MK_F_LOOK) && nx > p && nx < n_phases && prefetched != nx && p + 1 < n_phases;     // (the next MATVEC may turn out generic: checked below)
        int desc_w = 0, next_w = 0;
        if (p + 1 < n_phases && threadIdx.x < sizeof(MkPhase) / 4) desc_w = ((const int*)(phases + p + 1))[threadIdx.x];
        if (look && threadIdx.x < 128) {
            const int slot = threadIdx.x >> 6, t = threadIdx.x & 63;
            const int q = slot == 0 ? nx : nx2;
            if (q > p && q < n_phases) {
                const MkPhase* ph = phases + q;
                constexpr int NW = (int)(sizeof(StreamArgs) / 4);
                if (t < NW) next_w = ((const int*)&ph->mv)[t];
                else if (t == NW) next_w = ph->wtype;
                else if (t == NW + 1) next_w = ph->x && ph->norm_w ? ph->n : 0;
                else if (t == NW + 2) next_w = ((const int*)&ph->norm_w)[0];
                else if (t == NW + 3) next_w = ((const int*)&ph->norm_w)[1];
            } else if (t == (int)(sizeof(StreamArgs) / 4)) next_w = -1;     // no such phase
        }
        bool early = false;                  // the MATVEC phase issued the look-ahead itself, warp by warp
        switch (s_ph.type) {
        case MK_NORMQ: phase_normq(s_ph, s_red); break;
        case MK_MATVEC:
            if (GEN && s_ph.act_type == CC_Q8_K) {   // K-quant weights: generic phase, no register look-ahead
                unsigned long long* st1 = stamp ? prof + p * MK_PROF_SLOTS + 1 : nullptr;
                switch (s_ph.wtype) {
                case CC_Q2_K: phase_matvec_generic<TQ2_K>(s_ph, work, s_w, wstaged == p, xstaged == p, exp_lut, MK_GENERIC_PIPE_ARG st1); break;
                case CC_Q3_K: phase_matvec_generic<TQ3_K>(s_ph, work, s_w, wstaged == p, xstaged == p, exp_lut, MK_GENERIC_PIPE_ARG st1); break;
                case CC_Q4_K: phase_matvec_generic<TQ45_K<false>>(s_ph, work, s_w, wstaged == p, xstaged == p, exp_lut, MK_GENERIC_PIPE_ARG st1); break;
                case CC_Q5_K: phase_matvec_generic<TQ45_K<true>>(s_ph, work, s_w, wstaged == p, xstaged == p, exp_lut, MK_GENERIC_PIPE_ARG st1); break;
                case CC_Q6_K: phase_matvec_generic<TQ6_K>(s_ph, work, s_w, wstaged == p, xstaged == p, exp_lut, MK_GENERIC_PIPE_ARG st1); break;
                default: phase_matvec_generic<TQ8_K>(s_ph, work, s_w, wstaged == p, xstaged == p, exp_lut, MK_GENERIC_PIPE_ARG st1); break;
                }
                prefetched = -1;              // the generic phase used the pipe's registers: a pending streaming look-ahead (mixed models) is gone
                break;
            }
            if (prefetched != p) MK_TYPE_CALL(s_ph.wtype, matvec_prefetch<CC_Q8_0>(s_ph.mv, pipe), matvec_prefetch<CC_Q4_0>(s_ph.mv, pipe));
            early = look && (flags & MK_F_EARLY);
            MK_TYPE_CALL(s_ph.wtype,
                         phase_matvec<CC_Q8_0>(s_ph, work, s_w, wstaged == p, xstaged == p, exp_lut, pipe, comm, xseq, stamp ? prof + p * MK_PROF_SLOTS + 1 : nullptr,
                                               early ? s_next : nullptr, next_w),
                         phase_matvec<CC_Q4_0>(s_ph, work, s_w, wstaged == p, xstaged == p, exp_lut, pipe, comm, xseq, stamp ? prof + p * MK_PROF_SLOTS + 1 : nullptr,
                                               early ? s_next : nullptr, next_w));
            break;
        case MK_ATTN:
            if (s_ph.at.kv_f16) phase_attn<true>(s_ph, (float*)work, s_red, dyn, exp_lut, abar0, apar, AT_CH); else phase_attn<false>(s_ph, (float*)work, s_red, dyn, exp_lut, abar0, apar, AT_CH);
            break;
        case MK_ROWS: phase_rows(s_ph, dyn); break;
        case MK_REDUCE: phase_reduce(s_ph, comm, xseq, false); break;
        case MK_GATHER: phase_reduce(s_ph, comm, xseq, true); break;
        case MK_ARGMAX: phase_argmax(s_ph, dyn, s_red); break;
        }
        if (stamp) prof[p * MK_PROF_SLOTS + 2] = globaltimer_ns();
        if (p + 1 < n_phases && threadIdx.x < sizeof(MkPhase) / 4) ((int*)&s_phs[(p + 1) & 1])[threadIdx.x] = desc_w;
        if (look && !early && threadIdx.x < 128) {
            const int slot = threadIdx.x >> 6, t = threadIdx.x & 63;
            if (t < (int)(sizeof(StreamArgs) / 4) + 4) ((int*)&s_next[slot])[t] = next_w;
        }
        // look-ahead: request the first two weight segments of the next MATVEC phase (and, into L2, the rows behind them and the first
        // rows of the phase after it) before waiting at the barrier, so HBM keeps streaming through the barrier, the prologue and any
        // small (NORMQ / ATTN / ROWS) phases in between
        const bool more = p + 1 < n_phases;
        const bool xg = s_ph.xgpu != 0;
        // test hook (tests/test_gpu_robustness.py): one CTA deserts before the third barrier, as if it had never become resident
        if ((flags & MK_F_TESTSTALL) && p == 2 && blockIdx.x == gridDim.x - 1) return;
        if (more) grid_barrier_arrive(bar, gridDim.x, gen, xg, (flags & MK_F_SYSFENCE) != 0);       // its bar.sync also publishes s_next (written just above)
        if (look) {
            const bool next_stream = s_next[0].wtype == CC_Q8_0 || s_next[0].wtype == CC_Q4_0;
            if (!early && next_stream) MK_TYPE_CALL(s_next[0].wtype, matvec_prefetch<CC_Q8_0>(s_next[0].mv, pipe), matvec_prefetch<CC_Q4_0>(s_next[0].mv, pipe));
            if (next_stream) prefetched = nx;
            if ((flags & MK_F_WSTAGE) && s_next[0].norm_n > 0) {     // immutable norm weights of the next fused prologue: one L2 trip less after the barrier
                const unsigned sw = (unsigned)__cvta_generic_to_shared(s_w);
                const float* nw = s_next[0].norm_w;
                for (int i = threadIdx.x; i < (s_next[0].norm_n >> 2); i += MK_THREADS)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sw + i * 16), "l"(nw + i * 4) : "memory");
                asm volatile("cp.async.commit_group;" ::: "memory");
                wstaged = nx;
            }
        }
        if (stamp) prof[p * MK_PROF_SLOTS + 3] = globaltimer_ns();
        if (more) {
            grid_barrier_wait(bar, gridDim.x, gen, comm, xg ? xseq + 1u : 0u, (flags & MK_F_POLLCNT) != 0, &s_abort, err_host);
            gen++; if (xg) xseq++;
            if (s_abort) break;              // a barrier timed out (a CTA never became resident, or a peer GPU died): bail out, host reports
            // the barrier is open: the row the next fused prologue normalises is complete -- request it before anything else (descriptor
            // bookkeeping, geometry, look-ahead loads) so that its L2 round trip overlaps them
            const MkPhase& nph = s_phs[(p + 1) & 1];
            if ((flags & MK_F_XEARLY) && nph.type == MK_MATVEC && nph.x && !nph.red_n) {
                const int nb = nph.mv.k >> 5, nbp = ((((nb + 31) >> 5) + MK_SEG - 1) / MK_SEG) * MK_SEG * 32;
                const size_t xoff = nph.act_type == CC_Q8_K ? (size_t)mk_generic_sx_offset(nph.mv.k) : (size_t)nbp * 40 + 256 + 2048;
                const unsigned sx = (unsigned)__cvta_generic_to_shared(work + xoff);      // = s_x of the phase's prologue
                const float* xg = nph.x;
                for (int i = threadIdx.x; i < (nph.mv.k >> 2); i += MK_THREADS)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sx + i * 16), "l"(xg + i * 4) : "memory");
                asm volatile("cp.async.commit_group;" ::: "memory");
                xstaged = p + 1;
            }
        }
    }
    // the SAMPLE phase (lazy.cu: the only one, and the last): called after the loop, where the weight pipe is dead, so the call saves
    // nothing around itself (the barrier before it was the last iteration's)
    if constexpr (SMP) {
        __syncthreads();
        if (!s_abort) phase_sample(s_phs[(n_phases - 1) & 1], dyn, work, exp_lut);
    }
    if (comm.world > 0 && blockIdx.x == 0 && threadIdx.x == 0) *comm.seq = xseq;
    if (prof && blockIdx.x == 0 && threadIdx.x == 0) prof[n_phases * MK_PROF_SLOTS] = globaltimer_ns();
}

// working shared memory of one phase (the staging area of the norm weights comes on top, see cc_launch_mega)
size_t cc_mega_smem_for_phase(const MkPhase& ph) {
    if (ph.type == MK_MATVEC && ph.act_type == CC_Q8_K) return (size_t)(((TKBase::smem_bytes(ph.mv.k) + 15) & ~15) + 256) + (size_t)ph.mv.k * 4;
    if (ph.type == MK_MATVEC) {
        const size_t k = (size_t)ph.mv.k, nb = k / 32, GR = (nb + 31) / 32, NSEG = (GR + MK_SEG - 1) / MK_SEG, nbp = NSEG * MK_SEG * 32;
        // quants | scales | block sums | prologue: reduction scratch, f32 x
        return nbp * 40 + 256 + 2048 + (ph.x ? k * 4 : 0);
    }
    if (ph.type == MK_ATTN) return (size_t)(3 * ph.at.hd + ((ph.at.max_len + 8 + 3) & ~3) + AT_NBUF * AT_CH * ph.at.hd) * 4 + 64;
    if (ph.type == MK_SAMPLE) return SMP_SMEM_BYTES;
    return 1024;
}

// developer hook: a table of `n` empty phases -> the pure per-phase floor (descriptor fetch + grid barrier)
extern "C" CC_API int cc_test_mega_barrier_floor(cc_device* dev, int n, float* us_per_phase) {
    if (!dev || n < 2 || !us_per_phase) return CC_ERR_ARG;
    std::vector<MkPhase> tab((size_t)n);
    for (auto& p : tab) { memset(&p, 0, sizeof(p)); p.type = 99; p.next_matvec = -1; p.next_matvec2 = -1; }
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
        int rc = cc_launch_mega(dev, d_tab, n, nullptr, d_bar, 1024, 0, nullptr, nullptr, false, false);
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

bool cc_mega_generic_supported(int type, int64_t k) {
    return (type == CC_Q2_K || type == CC_Q3_K || type == CC_Q4_K || type == CC_Q5_K || type == CC_Q6_K || type == CC_Q8_K) && k % 256 == 0 && k <= 32768;
}

// developer A/B switches: CRABML_MEGA_FLAGS replaces the default flag word (see MK_F_* and the L2 budget byte)
#define MK_DEFAULT_FLAGS (MK_F_LOOK | MK_F_WSTAGE | MK_F_POLLCNT | MK_F_XEARLY | MK_F_RING | MK_F_RPAIR)      // ring + pairs: the fastest of the measured flag words
int cc_mega_flags() {
    static const int f = getenv("CRABML_MEGA_FLAGS") ? (int)strtol(getenv("CRABML_MEGA_FLAGS"), nullptr, 0) : MK_DEFAULT_FLAGS;
    return f;
}
bool cc_mega_ring_enabled() { return (cc_mega_flags() & MK_F_RING) != 0; }

int cc_launch_mega(cc_device* dev, const MkPhase* phases_dev, int n_phases, const uint8_t* dyn_dev, unsigned* bar_dev, size_t smem_work, size_t smem_wstage,
                   unsigned long long* prof, const CommDev* comm, bool generic, bool sample) {
    const int flags = cc_mega_flags();
    int max_ctas_per_sm = 0;
    const size_t wtop = (smem_work + 15) & ~(size_t)15;
    const size_t smem = wtop + smem_wstage;
    CC_REQUIRE(dev, smem <= 227 * 1024, "megakernel: a phase needs %zu bytes of shared memory", smem);
    auto kern = generic ? (sample ? mega_kernel<true, true> : mega_kernel<true, false>) : (sample ? mega_kernel<false, true> : mega_kernel<false, false>);
    if (smem > 48 * 1024) CC_CUDA(dev, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CC_CUDA(dev, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&max_ctas_per_sm, kern, MK_THREADS, smem));
    CC_REQUIRE(dev, max_ctas_per_sm >= 1, "megakernel does not fit on an SM");
    int per_sm = max_ctas_per_sm < MK_CTAS_PER_SM ? max_ctas_per_sm : MK_CTAS_PER_SM;
    int grid = dev->sm_count * per_sm;          // all CTAs co-resident: required by the grid barrier
    CommDev cd;
    memset(&cd, 0, sizeof(cd));
    if (comm) cd = *comm;
    // The grid barrier needs every CTA resident at once.  On a GPU this process owns, a plain launch of sm_count CTAs (1 per SM)
    // is co-resident by construction.  With another tenant on the same GPU (a second process, MPS) a partially scheduled grid
    // cannot finish a barrier: every spin in the kernel is bounded (MkSpin) and ends in CC_ERR_CUDA "megakernel barrier timeout"
    // instead of a hang; CRABML_MEGA_COOP=1 adds the cooperative launch attribute (all-or-nothing placement).  That is opt-in
    // because a cooperative kernel node in a CUDA graph is much slower to launch than a plain one.
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(MK_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = dev->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = getenv("CRABML_MEGA_COOP") ? 1 : 0;
    cfg.attrs = attr; cfg.numAttrs = 1;
    const uint16_t* lut = dev->exp_lut;
    CC_CUDA(dev, cudaLaunchKernelEx(&cfg, kern, phases_dev, n_phases, dyn_dev, bar_dev, lut, prof, flags, (int)wtop, dev->err_host, (const CommDev)cd));
    CC_LAUNCH_CHECK(dev);
    return CC_OK;
}
