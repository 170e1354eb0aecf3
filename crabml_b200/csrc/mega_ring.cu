// mega_ring.cu -- the persistent decode kernel with the weight stream decoupled from the compute warps.
//
// Why: when every warp alternates "issue the loads of a segment" and "consume a segment" (weights through registers, as in
// matvec_stream.cu), no warp issues loads at a phase boundary (slowest warp -> grid barrier -> activation prologue), so at most the
// segments a warp requested ahead cover the bubble and HBM idles for the rest.  Weights are immutable, so nothing forces the weight stream to follow the phase order of the compute:
//   * warps 16-19 of every CTA are PRODUCERS: their threads walk the phase table on their own, ahead of the compute warps, and
//     issue cp.async.bulk (TMA) copies of row segments (4 groups of 32 blocks: 4096 B of Q8_0 quants + 256 B of f16 scales) into a
//     ring of shared-memory slots -- as many as fit beside the per-phase working area (~37-47 slots = 160-200 KB per SM, 24-30 MB
//     per GPU in flight or landed).  It never waits for a barrier or an activation: whenever a slot is free the next segment of
//     this CTA's rows -- of this phase or any later one -- is already being fetched.
//   * warps 0-15 are CONSUMERS: same row dealing (row r -> CTA r % gridDim.x, rows of a CTA -> its warps round-robin), same per-lane
//     block order, same arithmetic as matvec_stream.cu (bit-identical results), but a segment is read from the ring with
//     LDS.128 after waiting on the slot's "full" mbarrier, and the slot is handed back through its "empty" mbarrier.  No weight
//     registers live across phases -> no register pipe, no look-ahead bookkeeping, 96 registers are enough.
//   * the inputs of a fused prologue arrive before it needs them: the norm weights go into a stage that lives across phases as soon
//     as the previous fused-norm prologue is done (a phase ahead, while HBM is busy with weights anyway), and the input row is
//     requested into the phase's working area with cp.async the moment the grid barrier opens -- one L2 trip for every width,
//     ffn_down's 11008 included.  Only an exchange prologue (sharded path) sums its `world` partial rows from registers.
// The 512 compute threads synchronise on named barrier 1 (MK_SYNC); the producer warp never joins it.
// 20 warps: five per SM sub-partition, so its 16384 registers allow 96 per thread (what __launch_bounds__(640, 1) yields).
#define MK_SYNC() asm volatile("bar.sync 1, 512;" ::: "memory")
#define MK_GENERIC_NOINLINE 1
#include "mega_phases.cuh"

#define MR_PRODUCER_WARPS 4        // 20 warps: five per SM sub-partition, still 96 registers per thread
#define MR_THREADS (MK_THREADS + 32 * MR_PRODUCER_WARPS)
#define MR_MAX_SLOTS 112
#define MR_Q8_FLIGHT 10            // Q8_0 entries a producer lets be in flight at once (cc_launch_mega_ring)
#define MR_DESC_WORDS ((int)(sizeof(MkPhase) / 4))
#define MR_DESC_PER_LANE ((MR_DESC_WORDS + 31) / 32)

struct MrRing {
    int ring_off;          // byte offset of the ring in dynamic shared memory (16-byte aligned)
    int slot_bytes;        // bytes per slot (multiple of 128): quants of up to 4 groups, then their f16 scales
    int nslots;
    int at_ch;             // ATTN phase: cache rows per TMA chunk
    int flight;            // entry e is issued only once entry e - flight has landed (flight = nslots: no such limit)
};

__device__ __forceinline__ void mr_expect_tx(unsigned bar, unsigned bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
// `pol`: an L2::evict_first policy -- every weight byte is read once per token, so its lines should be the first to leave L2, not the
// rows a token reads again (norm weights, the exp LUT, the KV history)
__device__ __forceinline__ void mr_bulk_g2s(unsigned dst, const void* src, unsigned bytes, unsigned bar, unsigned long long pol) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(pol) : "memory");
}
// cp.async.cg of floats [0, n) to shared memory, thread t the 16-byte chunks t, t + 512, ... -- the chunks it later reads itself (the
// prologue's mapping), so its own cp.async.wait_group makes them visible without a CTA barrier; one commit group per call
__device__ __forceinline__ void mr_stage_f32(float* dst, const float* src, int n) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(dst);
    for (int i = threadIdx.x; i < (n >> 2); i += MK_THREADS) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s + i * 16), "l"(src + i * 4) : "memory");
    asm volatile("cp.async.commit_group;" ::: "memory");
}
// working area of a streaming MATVEC phase: quants [nbp * 32] | f32 scales [nbp] | block sums [nbp] | reduction scratch 256 B |
// exchange stage 2 KB | f32 input row [k] (fused prologues without an exchange)
__host__ __device__ __forceinline__ int mr_nbp(int k) { const int GR = ((k >> 5) + 31) >> 5; return (GR + MK_SEG - 1) / MK_SEG * MK_SEG * 32; }
__host__ __device__ __forceinline__ int mr_x_off(int k) { return mr_nbp(k) * 40 + 256 + 2048; }
__device__ __forceinline__ bool mr_try_wait(unsigned bar, unsigned parity) {
    unsigned ok;
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ bool mr_test_wait(unsigned bar, unsigned parity) {
    unsigned ok;
    asm volatile("{\n.reg .pred p;\nmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// Developer profiling (CTA 0, warp 0, all lanes), as the barrier in front of a phase opens: how many entries from `ent` on (the consumers'
// next entry) the producers have issued into the ring and how many of those have landed, as (landed << 8) | issued -- one look at every
// slot.  A called function: inlined, or taken at more points of a phase, it moves the kernel's spills.
__device__ __noinline__ unsigned mr_ring_fill(const volatile unsigned* s_seq, unsigned full0, int nslots, unsigned ent) {
    unsigned iss = 0, got = 0;
    for (int sl = threadIdx.x & 31; sl < nslots; sl += 32) {
        const unsigned q = s_seq[sl];
        if (q && (int)(q - 1u - ent) >= 0) { iss++; got += mr_test_wait(full0 + 8u * sl, ((q - 1u) / (unsigned)nslots) & 1u) ? 1u : 0u; }
    }
    iss = __reduce_add_sync(0xffffffffu, iss);
    got = __reduce_add_sync(0xffffffffu, got);
    return (got << 8) | iss;
}
// Slot hand-back: the consumer stores (entry number + 1) into the slot's "done" word (release), the producer polls it (acquire) for
// exactly the previous tenant's number -- an mbarrier parity could not tell one lap from two.  `dep` ties the store behind the
// arithmetic that consumed the slot's data.
__device__ __forceinline__ void mr_release(unsigned done_addr, unsigned v, float dep) { asm volatile("st.release.cta.shared::cta.u32 [%0], %1;" ::"r"(done_addr), "r"(v), "f"(dep) : "memory"); }
__device__ __forceinline__ unsigned mr_ld_acquire_shared(unsigned addr) {
    unsigned v;
    asm volatile("ld.acquire.cta.shared::cta.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}

// rows of a streaming MATVEC phase that belong to this CTA, as "units": unit u -> concatenated row first + u * stride, consumed by
// warp u % 16; a unit is V virtual rows (2 for the gate/up pair, else 1) of NSEG segments each.  Producer and consumers derive the
// same entry sequence from this.
struct MrGeo {
    int nb, GR, NSEG, V, E, n_units, first, stride, last_half_off, m_cat;
    bool pair;
};
__device__ __forceinline__ MrGeo mr_geo(const StreamArgs& A) {
    MrGeo g;
    g.nb = A.k >> 5; g.GR = (g.nb + 31) >> 5; g.NSEG = (g.GR + MK_SEG - 1) / MK_SEG;
    g.pair = A.epilogue == 2;
    const StreamMats& M = A.mats;
    g.m_cat = g.pair ? M.m[0] : M.m[0] + (M.n > 1 ? M.m[1] : 0) + (M.n > 2 ? M.m[2] : 0);
    if (A.epilogue == 3) {             // exchange phases: one contiguous block of rows per CTA, so its partial rows go to each peer as one run
        const int rpc = (((g.m_cat + (int)gridDim.x - 1) / (int)gridDim.x) + 3) & ~3;
        g.first = (int)blockIdx.x * rpc; g.stride = 1;
        g.n_units = min(rpc, max(0, g.m_cat - g.first));
    } else {
        g.first = (int)blockIdx.x; g.stride = (int)gridDim.x;
        g.n_units = g.first < g.m_cat ? (g.m_cat - g.first + g.stride - 1) / g.stride : 0;
    }
    g.V = g.pair ? 2 : 1;
    g.E = g.V * g.NSEG;
    g.last_half_off = 16 * (g.nb - 32 * (g.GR - 1));
    return g;
}
__device__ __forceinline__ int mr_locate(const StreamMats& M, const MrGeo& g, int rc, int v, int& mat) {
    mat = 0;
    int r = rc;
    if (g.pair) { mat = v; return r; }
    if (M.n > 1 && r >= M.m[0]) { r -= M.m[0]; mat = 1; if (M.n > 2 && r >= M.m[1]) { r -= M.m[1]; mat = 2; } }
    return r;
}

// entry f has landed: it has been consumed (the slot's done word has reached it; a slot's tenants are consumed in order), or it is the
// slot's tenant and its barrier phase has completed -- exact, since the tenant cannot change before it is consumed
__device__ __forceinline__ bool mr_landed(unsigned f, int nslots, unsigned full0, unsigned done0, volatile unsigned* s_seq) {
    const unsigned sl = f % (unsigned)nslots;
    if ((int)(mr_ld_acquire_shared(done0 + 4u * sl) - 1u - f) >= 0) return true;
    return s_seq[sl] == f + 1u && mr_test_wait(full0 + 8u * sl, (f / (unsigned)nslots) & 1u);
}
// ---- producer warp: runs ahead of everybody ---------------------------------------------------------------------------------------------
// All 32 lanes issue (a single issuing thread manages only ~1 entry per few hundred cycles); lane l owns the entries l, l + 32, ...
// of a phase: it decomposes the entry index into (unit, virtual row, segment), waits until the slot's previous tenant has been consumed, arms the
// slot's "full" barrier with the byte count, issues the two bulk copies (quants, scales) and publishes the entry number in the slot's
// sequence word.  Consumers check that word before they look at the barrier: an mbarrier parity alone cannot tell "this use has not
// landed" from "the previous use has not landed" when a warp gets more than one lap ahead (16 warps x 3 segments > 40 slots).
// (Measured on the earlier target: 4 producer warps were the fastest of 1 / 2 / 4 / 8 -- a warp's probe-and-issue trip takes ~400
// cycles, so the number of polling warps bounds the refill rate, and at 8 the 80-register cap starts to cost.  Sleeping after a failed probe,
// SIMT-wide parameter computation, in-order probe loops and fence-free hand-back words changed nothing.)
__device__ void mr_producer(const MkPhase* __restrict__ phases, int n_phases, const MrRing R, unsigned full0, unsigned done0, unsigned ring0,
                            MkPhase* s_pd, volatile unsigned* s_seq, volatile int* s_abort, int* s_prod_done, unsigned long long* prof_tail) {
    const int lane = threadIdx.x & 31;
    const int pt = (int)threadIdx.x - MK_THREADS;          // producer thread 0 .. 32 * MR_PRODUCER_WARPS - 1: owns the entries pt, pt + 128, ... of every phase
    unsigned long long p_trips = 0, p_cyc = 0, p_iss = 0;       // developer profiling (CTA 0 / lane 0)
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    for (int i = lane; i < MR_DESC_WORDS; i += 32) ((int*)&s_pd[0])[i] = ((const int*)phases)[i];
    __syncwarp();
    unsigned ent = 0;
    bool dead = false;
    for (int p = 0; p < n_phases && !dead; p++) {
        int nw[MR_DESC_PER_LANE];
#pragma unroll
        for (int j = 0; j < MR_DESC_PER_LANE; j++) { const int i = lane + 32 * j; nw[j] = (p + 1 < n_phases && i < MR_DESC_WORDS) ? ((const int*)(phases + p + 1))[i] : 0; }
        const MkPhase& ph = s_pd[p & 1];
        if (ph.type == MK_MATVEC && ph.act_type != CC_Q8_K) {
            const StreamArgs& A = ph.mv;
            const StreamMats& M = A.mats;
            const MrGeo g = mr_geo(A);
            const unsigned BB = ph.wtype == CC_Q8_0 ? 32u : 16u;
            const unsigned doff = MK_SEG * 32u * BB;
            const int N = g.n_units * g.E, twoE = 2 * g.E, Npair = (g.n_units >> 1) * twoE;
            // a flat loop, one probe of the thread's own slot per trip (a load of the slot's "done" word: no suspension): thread t serves the entries
            // t, t + 128, ... at its own pace, so a slot is refilled as soon as it is released, not when the slowest lane of a batch is ready
            int j = pt;
            bool have = false, mydead = false;
            const uint8_t* q0 = nullptr; const uint16_t* d0 = nullptr;
            unsigned nbe = 0, e = 0, slot = 0, use = 0, it = 0;
            const long long pc0 = clock64();
            while (j < N) {
                p_trips++;
                if (!have) {
                    // ring order: the units of a CTA go in PAIRS whose entries alternate (A v0 s0, B v0 s0, A v0 s1, B v0 s1, ...): the consumer warp that
                    // takes a pair always works on two ADJACENT entries and hands them back at once (16 warps x 2 entries < the ring); an odd last unit
                    // follows on its own
                    int u, vs;
                    if (j < Npair) { const int P = j / twoE, w = j - P * twoE; u = 2 * P + (w & 1); vs = w >> 1; }
                    else { u = g.n_units - 1; vs = j - Npair; }
                    const int v = vs / g.NSEG, sg = vs - v * g.NSEG;
                    int mat;
                    const int r = mr_locate(M, g, g.first + u * g.stride, v, mat);
                    q0 = M.qs[mat] + ((size_t)r * g.nb + (size_t)sg * (MK_SEG * 32)) * BB;
                    d0 = M.d[mat] + (size_t)r * CC_D_STRIDE(g.nb) + sg * (MK_SEG * 32);
                    nbe = (unsigned)min(MK_SEG * 32, g.nb - MK_SEG * 32 * sg);
                    e = ent + (unsigned)j; slot = e % (unsigned)R.nslots; use = e / (unsigned)R.nslots;
                    have = true;
                }
                if ((!use || mr_ld_acquire_shared(done0 + 4u * slot) == e - (unsigned)R.nslots + 1u)      // the slot's previous tenant has been consumed
                    && (R.flight >= R.nslots || e < (unsigned)R.flight || mr_landed(e - (unsigned)R.flight, R.nslots, full0, done0, s_seq))) {
                    const unsigned fb = full0 + 8u * slot, dst = ring0 + slot * (unsigned)R.slot_bytes;
                    const unsigned dbytes = (nbe * 2u + 15u) & ~15u;        // the scale rows are padded to 16 bytes (CC_D_STRIDE): a short last segment copies its padding
                    mr_expect_tx(fb, nbe * BB + dbytes);
                    mr_bulk_g2s(dst, q0, nbe * BB, fb, pol);
                    mr_bulk_g2s(dst + doff, d0, dbytes, fb, pol);
                    __threadfence_block();
                    s_seq[slot] = e + 1u;
                    j += 32 * MR_PRODUCER_WARPS; have = false; p_iss++;
                } else if ((++it & 0x3FFu) == 0 && *s_abort) { mydead = true; break; }
            }
            p_cyc += (unsigned long long)(clock64() - pc0);
            dead = __any_sync(0xffffffffu, mydead);
            ent += (unsigned)N;
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < MR_DESC_PER_LANE; j++) { const int i = lane + 32 * j; if (i < MR_DESC_WORDS) ((int*)&s_pd[(p + 1) & 1])[i] = nw[j]; }
        __syncwarp();
    }
    if (lane == 0) { __threadfence_block(); atomicAdd(s_prod_done, 1); }
    if (pt == 0 && prof_tail && blockIdx.x == 0) { prof_tail[1] = p_trips; prof_tail[2] = p_cyc; prof_tail[3] = p_iss; prof_tail[4] = (unsigned)R.nslots; }
}

// ---- consumer side of a streaming MATVEC phase ------------------------------------------------------------------------------------------
struct MrCons { unsigned full0, done0; const uint8_t* ring; int slot_bytes, nslots; unsigned ent_base; int* s_unit; volatile unsigned* s_seq; volatile int* s_dead; unsigned* err_dev; unsigned* err_host; };

// Bounded wait for a slot to fill.  A wait that does not end within 2 s (it takes microseconds) raises the error words (code 4, reported by
// cc_check_async_error) and marks the ring dead for the whole CTA: every later wait returns at once, the launch drains with garbage
// results instead of hanging the GPU.
__device__ __forceinline__ void mr_wait_full(const MrCons& RC, unsigned slot, unsigned e, unsigned parity) {
    const unsigned bar = RC.full0 + 8u * slot;
    volatile unsigned* seq = RC.s_seq + slot;
    if (*seq == e + 1u && mr_try_wait(bar, parity)) return;
    unsigned it = 0;
    unsigned long long t0 = 0;
    for (;;) {
        if (*seq == e + 1u && mr_try_wait(bar, parity)) return;     // entry e has been issued into the slot, and it has landed
        if ((++it & 0xFFFu) != 0) continue;
        if (*RC.s_dead) return;
        const unsigned long long t = cc_globaltimer_ns();
        if (!t0) { t0 = t; continue; }
        if (t - t0 < 2000000000ull) continue;
        *RC.s_dead = 1;
        if (RC.err_dev) atomicExch(RC.err_dev, 4u);
        if (RC.err_host) { *(volatile unsigned*)RC.err_host = 4u; __threadfence_system(); }
        return;
    }
}

// Activation quants in shared memory, per group of 32 blocks: the 16-byte first halves of all 32 blocks, then the second halves (the layout of
// the Q8_0 weight plane) -- lane l reads block 32 g + l with two conflict-free LDS.128 (block-major, 32 bytes apart, is a 2-way bank conflict:
// 64 instead of 32 shared-memory wavefronts per segment, and the ring's throughput is bounded by shared-memory bandwidth)
__device__ __forceinline__ int mr_act_word(int i) {           // i = 4-byte word index in block-major order (block i >> 3, word i & 7)
    const int b = i >> 3, w = i & 7;
    return (b >> 5) * 256 + (w >> 2) * 128 + (b & 31) * 4 + (w & 3);
}
__device__ __forceinline__ int mr_act_int4(int i) {           // i = 16-byte index in block-major order (block i >> 1, half i & 1)
    const int b = i >> 1;
    return (b >> 5) * 64 + (i & 1) * 32 + (b & 31);
}

// One segment (4 groups) of TWO rows against the same activation segment: the activation quants and scales are read once for both rows
// (shared-memory wavefronts per 4352-byte entry: 34 TMA write + 34 weight read + 16 activation, against 64 + for one row at a time).
// Per row the arithmetic is matvec_stream.cu's, term by term (bit-identical).
template <int TYPE>
__device__ __forceinline__ void mr_dot2(const uint8_t* spA, const uint8_t* spB, int seg, int nb, int GR, int last_half_off, int lane,
                                        const int4* aq_l, const float* ad_l, const int* as_l, float& partA, float& partB) {
    constexpr int GB = TYPE == CC_Q8_0 ? 1024 : 512;
    const uint8_t* qA = spA + lane * 16;
    const uint8_t* qB = spB + lane * 16;
    const uint16_t* dA = (const uint16_t*)(spA + MK_SEG * GB) + lane;
    const uint16_t* dB = (const uint16_t*)(spB + MK_SEG * GB) + lane;
    const int4* aq = aq_l + seg * (MK_SEG * 64);
    const float* ad = ad_l + seg * (MK_SEG * 32);
    const int4 z4 = make_int4(0, 0, 0, 0);
    float accA = 0.0f, accB = 0.0f;
#pragma unroll
    for (int g = 0; g < MK_SEG; g++) {
        const int gi = seg * MK_SEG + g;
        const bool on = gi * 32 + lane < nb;
        const int4 alo = aq[g * 64], ahi = aq[g * 64 + 32];
        const float adv = ad[g * 32];
        if constexpr (TYPE == CC_Q8_0) {
            const int hoff = gi == GR - 1 ? last_half_off : 512;
            int4 a0 = z4, a1 = z4, b0 = z4, b1 = z4; uint16_t sA = 0, sB = 0;
            if (on) { a0 = *(const int4*)(qA + g * GB); a1 = *(const int4*)(qA + g * GB + hoff); sA = dA[g * 32];
                      b0 = *(const int4*)(qB + g * GB); b1 = *(const int4*)(qB + g * GB + hoff); sB = dB[g * 32]; }
            const int sumA = mk_dp16(a0, alo) + mk_dp16(a1, ahi);
            const int sumB = mk_dp16(b0, alo) + mk_dp16(b1, ahi);
            accA += (float)sumA * h2f_bits(sA) * adv;
            accB += (float)sumB * h2f_bits(sB) * adv;
        } else {
            int4 wA = z4, wB = z4; uint16_t sA = 0, sB = 0;
            if (on) { wA = *(const int4*)(qA + g * GB); sA = dA[g * 32]; wB = *(const int4*)(qB + g * GB); sB = dB[g * 32]; }
            const int asv = as_l[(seg * MK_SEG + g) * 32];
            const int4 loA = make_int4(wA.x & 0x0F0F0F0F, wA.y & 0x0F0F0F0F, wA.z & 0x0F0F0F0F, wA.w & 0x0F0F0F0F);
            const int4 hiA = make_int4((wA.x >> 4) & 0x0F0F0F0F, (wA.y >> 4) & 0x0F0F0F0F, (wA.z >> 4) & 0x0F0F0F0F, (wA.w >> 4) & 0x0F0F0F0F);
            const int4 loB = make_int4(wB.x & 0x0F0F0F0F, wB.y & 0x0F0F0F0F, wB.z & 0x0F0F0F0F, wB.w & 0x0F0F0F0F);
            const int4 hiB = make_int4((wB.x >> 4) & 0x0F0F0F0F, (wB.y >> 4) & 0x0F0F0F0F, (wB.z >> 4) & 0x0F0F0F0F, (wB.w >> 4) & 0x0F0F0F0F);
            const int sumA = mk_dp16(loA, alo) + mk_dp16(hiA, ahi) - 8 * asv;
            const int sumB = mk_dp16(loB, alo) + mk_dp16(hiB, ahi) - 8 * asv;
            accA += (float)sumA * h2f_bits(sA) * adv;
            accB += (float)sumB * h2f_bits(sB) * adv;
        }
    }
    partA = accA; partB = accB;
}

// smem: the phase's working area (mr_x_off); s_wn: the norm-weight stage, holding the weights `wst` once this thread's cp.async groups
// are complete (requested here when they are not ph.norm_w); x_staged: the input row was requested into the working area as the
// barrier opened
// QW: epilogue 1 adds the vector of the row's matrix (qwen2's q/k/v biases); otherwise it has one matrix (the residual add)
template <int TYPE, bool QW>
__device__ void phase_matvec_ring(const MkPhase& ph, uint8_t* smem, float* s_wn, const float*& wst, bool x_staged, const uint16_t* exp_lut, MrCons& RC,
                                  const CommDev& comm, unsigned xseq, unsigned long long* stamp1) {
    const StreamArgs& A = ph.mv;
    const int k = A.k;
    const MrGeo g = mr_geo(A);
    const int nb = g.nb, GR = g.GR, NSEG = g.NSEG;
    const bool pair = g.pair;
    const int nbp = NSEG * MK_SEG * 32;
    int8_t* s_q = (int8_t*)smem;
    float* s_d = (float*)(smem + (size_t)nbp * 32);
    int* s_s = (int*)(smem + (size_t)nbp * 32 + (size_t)nbp * 4);
    float* s_red = (float*)(smem + (size_t)nbp * 40);
    float* s_part = (float*)(smem + (size_t)nbp * 40 + 256);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const StreamMats& M = A.mats;
    if (threadIdx.x == 0) *RC.s_unit = 0;          // ordered before the row loop by the MK_SYNC that ends the prologue
    if (ph.x) {
        // Fused prologue: [exchange reduction] + [rms_norm * w] + Q8_0 quantisation of x by EVERY CTA: thread t owns the float4 chunks
        // t, t + 512, ... (the canonical reduction order of common.cuh, and 8 consecutive threads = one 32-block).  The norm weights were
        // staged one fused-norm phase ago; the row itself lands in shared memory after one L2 trip, except in an exchange prologue, which
        // sums `world` partial rows from registers.
        const int n4 = k >> 2;
        const int npass = nbp >> 6;                                    // 64 blocks per pass of 512 threads (nbp % 128 == 0)
        const float4 z4 = make_float4(0, 0, 0, 0);
        const float4* s_w4 = (const float4*)s_wn;
        const float4* s_x4 = (const float4*)(smem + mr_x_off(k));
        const float* xbase = ph.red_n ? comm.data[comm.rank] + (size_t)(xseq & 1u) * CC_COMM_MAX_RANKS * CC_COMM_MAX_ELEMS : ph.x;
        auto load_x = [&](int i) -> float4 {                            // chunk i of the input row
            if (i >= n4) return z4;
            if (!ph.red_n) return s_x4[i];
            float4 a4 = __ldcg((const float4*)xbase + i);               // sum over ranks in rank order (+ residual): comm.cu
            for (int p = 1; p < comm.world; p++) {
                const float4 t4 = __ldcg((const float4*)(xbase + (size_t)p * CC_COMM_MAX_ELEMS) + i);
                a4.x += t4.x; a4.y += t4.y; a4.z += t4.z; a4.w += t4.w;
            }
            if (ph.red_res) { const float4 r4 = __ldcg((const float4*)ph.red_res + i); a4.x += r4.x; a4.y += r4.y; a4.z += r4.z; a4.w += r4.w; }
            return a4;
        };
        if (ph.norm_w && ph.norm_w != wst) { mr_stage_f32(s_wn, ph.norm_w, k); wst = ph.norm_w; }     // weights an earlier phase writes
        if (!ph.red_n && !x_staged) mr_stage_f32((float*)s_x4, ph.x, k);
        asm volatile("cp.async.wait_group 1;" ::: "memory");           // groups in flight, oldest first: [norm-weight stage] [x row]
        if (stamp1) stamp1[7] = globaltimer_ns();
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        if (stamp1) stamp1[3] = globaltimer_ns();
        float rms = 1.0f;
        const bool in_regs = ph.red_n && npass <= 4;
        float4 xr[4];
#pragma unroll
        for (int j = 0; j < 4; j++) xr[j] = z4;
        if (in_regs) {
#pragma unroll
            for (int j = 0; j < 4; j++) if (j < npass) xr[j] = load_x(j * MK_THREADS + (int)threadIdx.x);
        }
        if (ph.norm_w) {
            float ss = 0.0f;
            if (in_regs) {
#pragma unroll
                for (int j = 0; j < 4; j++) if (j * MK_THREADS + (int)threadIdx.x < n4) ss += cc_sq4(xr[j]);
            } else {
                for (int i = threadIdx.x; i < n4; i += MK_THREADS) { const float4 v = load_x(i); ss += cc_sq4(v); }
            }
            ss = warp_sum(ss);
            if (lane == 0) s_red[warp] = ss;
            MK_SYNC();
            float t = 0.0f;
#pragma unroll
            for (int w = 0; w < MK_WARPS; w++) t += s_red[w];
            rms = sqrtf(t / (float)k + ph.eps);
        }
        if (stamp1) stamp1[4] = globaltimer_ns();
        const int sub = threadIdx.x & 7;
        int* s_q32 = (int*)s_q;
        auto quant_chunk = [&](int i, float4 v, const float4& w4) {      // i = chunk index (block i >> 3), v = its 4 elements (zeros past the row)
            const bool live = i < n4;
            if (ph.orig && blockIdx.x == 0 && live) ((float4*)ph.orig)[i] = v;      // Tensor::dup of the un-normalised row (llama2.rs:227,607)
            if (ph.norm_w && live) { v.x = (v.x / rms) * w4.x; v.y = (v.y / rms) * w4.y; v.z = (v.z / rms) * w4.z; v.w = (v.w / rms) * w4.w; }
            float amax = fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)));
#pragma unroll
            for (int o = 4; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
            const float d = amax / 127.0f;
            const int q0 = live ? __float2int_rz(v.x / d) : 0, q1 = live ? __float2int_rz(v.y / d) : 0;
            const int q2 = live ? __float2int_rz(v.z / d) : 0, q3 = live ? __float2int_rz(v.w / d) : 0;
            s_q32[mr_act_word(i)] = (q0 & 255) | ((q1 & 255) << 8) | ((q2 & 255) << 16) | (q3 << 24);
            if constexpr (TYPE == CC_Q4_0) {
                int sq = q0 + q1 + q2 + q3;
#pragma unroll
                for (int o = 4; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
                if (sub == 0) s_s[i >> 3] = sq;
            }
            if (sub == 0) s_d[i >> 3] = live ? __half2float(__float2half_rn(d)) : 0.0f;
        };
        auto load_w = [&](int i) -> float4 { return ph.norm_w && i < n4 ? s_w4[i] : z4; };
        if (in_regs) {
#pragma unroll
            for (int j = 0; j < 4; j++) if (j < npass) quant_chunk(j * MK_THREADS + (int)threadIdx.x, xr[j], load_w(j * MK_THREADS + (int)threadIdx.x));
        } else if (!ph.red_n) {
            for (int j = 0; j < npass; j++) { const int i = j * MK_THREADS + (int)threadIdx.x; quant_chunk(i, load_x(i), load_w(i)); }
        } else {
            for (int j0 = 0; j0 < npass; j0 += 4) {                      // four chunks requested before the first is quantised
                float4 v[4];
#pragma unroll
                for (int j = 0; j < 4; j++) v[j] = j0 + j < npass ? load_x((j0 + j) * MK_THREADS + (int)threadIdx.x) : z4;
#pragma unroll
                for (int j = 0; j < 4; j++) if (j0 + j < npass) quant_chunk((j0 + j) * MK_THREADS + (int)threadIdx.x, v[j], load_w((j0 + j) * MK_THREADS + (int)threadIdx.x));
            }
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
            if (i0 < nbp * 2) sq4[mr_act_int4(i0)] = qa;
            if (i1 < nbp * 2) sq4[mr_act_int4(i1)] = qb;
            if (i0 < nbp) { s_d[i0] = dv; if constexpr (TYPE == CC_Q4_0) s_s[i0] = sv; }
        } else {
            for (int i = threadIdx.x; i < nbp * 2; i += MK_THREADS) sq4[mr_act_int4(i)] = i < nb * 2 ? __ldcg(gq + i) : make_int4(0, 0, 0, 0);
            for (int i = threadIdx.x; i < nbp; i += MK_THREADS) {
                s_d[i] = i < nb ? __ldcg(gd + i) : 0.0f;
                if constexpr (TYPE == CC_Q4_0) s_s[i] = i < nb ? __ldcg(gs + i) : 0;
            }
        }
    }
    MK_SYNC();
    if (stamp1) *stamp1 = globaltimer_ns();
    // every thread has read the stage: the next fused-norm phase's weights may go in now, a phase ahead of their use
    if (ph.x && ph.norm_w) { wst = ph.next_norm_w; if (wst) mr_stage_f32(s_wn, wst, ph.next_norm_n); }
    const int4* aq_l = (const int4*)s_q + lane;
    const float* ad_l = s_d + lane;
    const int* as_l = s_s + lane;
    // Epilogues that need a value from memory (the residual, or the exp LUT entry of silu) are finished one round later, so the warp never stalls an L2 round trip; lane 0 only
    float pend_a[2] = {0.0f, 0.0f}, pend_b[2] = {0.0f, 0.0f}, pend_res[2] = {0.0f, 0.0f};
    unsigned short pend_lut[2] = {0, 0};
    int pend_row[2] = {-1, -1};
    auto flush_pending = [&]() {
#pragma unroll
        for (int t = 0; t < 2; t++) {
            if (lane == 0 && pend_row[t] >= 0) {
                if (pair) M.out[0][pend_row[t]] = (pend_a[t] / (1.0f + h2f_bits(pend_lut[t]))) * pend_b[t];
                else if (QW) {
                    int mat;
                    const int rr = mr_locate(M, g, pend_row[t], 0, mat);
                    (mat == 0 ? M.out[0] : mat == 1 ? M.out[1] : M.out[2])[rr] = pend_a[t] + pend_res[t];
                } else M.out[0][pend_row[t]] = pend_a[t] + pend_res[t];
            }
            pend_row[t] = -1;
        }
    };
    long long c_wait = 0, c_all = 0; int c_n = 0;  // developer profiling (CTA 0 / warp 0): cycles waiting for slots, cycles in the row loop, entries
    if (stamp1) c_all = clock64();
    const unsigned NS = (unsigned)RC.nslots;
    // Pairs of units are dealt dynamically in ring order (the CTA's pair counter): no warp idles while another still has rows left, and the
    // two rows of a pair share every activation load.  Which warp computes a row does not change its bits.
    const int npairs = g.n_units >> 1, twoE = 2 * g.E;
    // A CTA with at most one unit claims it alone at entry 0 under either arithmetic below.  The single-unit arm is kept for it on
    // purpose: compiled for pairs only, ptxas allocates this kernel worse (64 -> 72-byte frame, 128 / 208 -> 140-180 / 240-274 bytes of
    // spills) and a sampled Llama-2-7B Q8_0 token got 1 % slower (NVIDIA H100 80GB HBM3, 700 W).
    const bool pairs = g.n_units > 1;
    for (;;) {
        int P = 0;
        if (lane == 0) P = atomicAdd(RC.s_unit, 1);
        P = __shfl_sync(0xffffffffu, P, 0);
        // claim P: units 2P and 2P + 1, or an odd last unit alone
        const bool two = pairs && P < npairs;
        if (pairs ? (!two && !(P == npairs && (g.n_units & 1))) : P >= g.n_units) break;
        const int u0 = !pairs ? P : two ? 2 * P : g.n_units - 1;
        const unsigned step = two ? 2u : 1u;
        unsigned eA = RC.ent_base + (unsigned)(!pairs ? P * g.E : two ? P * twoE : npairs * twoE);
        unsigned slotA = eA % NS, parA = (eA / NS) & 1u;
        float first[2] = {0.0f, 0.0f};
        for (int v = 0; v < g.V; v++) {
            float accA = 0.0f, accB = 0.0f;
            for (int sg = 0; sg < NSEG; sg++) {
                unsigned slotB = slotA + 1u, parB = parA;
                if (slotB == NS) { slotB = 0; parB ^= 1u; }
                long long t0 = 0;
                if (stamp1) t0 = clock64();
                mr_wait_full(RC, slotA, eA, parA);
                if (two) mr_wait_full(RC, slotB, eA + 1u, parB);
                if (stamp1) { c_wait += clock64() - t0; c_n += two ? 2 : 1; }
                const uint8_t* spA = RC.ring + (size_t)slotA * RC.slot_bytes;
                const uint8_t* spB = two ? RC.ring + (size_t)slotB * RC.slot_bytes : spA;
                float partA, partB;
                mr_dot2<TYPE>(spA, spB, sg, nb, GR, g.last_half_off, lane, aq_l, ad_l, as_l, partA, partB);
                accA += partA; accB += partB;
                __syncwarp();
                if (lane == 0) { mr_release(RC.done0 + 4u * slotA, eA + 1u, partA); if (two) mr_release(RC.done0 + 4u * slotB, eA + 2u, partB); }
                eA += step; slotA += step;
                if (slotA >= NS) { slotA -= NS; parA ^= 1u; }
            }
            const float rA = warp_sum(accA), rB = warp_sum(accB);
            if (pair && v == 0) { first[0] = rA; first[1] = rB; continue; }
            if (pair || A.epilogue == 1) flush_pending();
#pragma unroll
            for (int t = 0; t < 2; t++) {
                if (t == 1 && !two) break;
                const float r = t ? rB : rA;
                const int u = u0 + t, rc = g.first + u * g.stride;
                if (lane != 0) continue;
                if (pair) { pend_a[t] = first[t]; pend_b[t] = r; pend_row[t] = rc; pend_lut[t] = exp_lut[f2h_bits(-first[t])]; }      // silu(gate) * up
                else if (A.epilogue == 1 && QW) {                                                                                   // + bias of the row's matrix
                    int mat;
                    const int rr = mr_locate(M, g, rc, 0, mat);
                    pend_a[t] = r; pend_row[t] = rc; pend_res[t] = ldcg_f((mat == 0 ? A.residual[0] : mat == 1 ? A.residual[1] : A.residual[2]) + rr);
                }
                else if (A.epilogue == 1) { pend_a[t] = r; pend_row[t] = rc; pend_res[t] = ldcg_f(A.residual[0] + rc); }           // + residual (llama2.rs:266,636)
                else if (A.epilogue == 3) s_part[u] = r;                                                                            // partial row -> this CTA's exchange stage
                else {
                    int mat;
                    const int rr = mr_locate(M, g, rc, 0, mat);
                    float* o = mat == 0 ? M.out[0] : mat == 1 ? M.out[1] : M.out[2];
                    o[rr] = r;
                }
            }
        }
    }
    flush_pending();
    if (stamp1) { stamp1[5] = (unsigned long long)c_wait; stamp1[6] = ((unsigned long long)(clock64() - c_all) << 20) | (unsigned long long)c_n; }
    RC.ent_base += (unsigned)(g.n_units * g.E);
    if (A.epilogue == 3) {
        // the CTA's block of partial rows -> slot[rank] of every GPU's exchange window: warp p serves peer p with coalesced 16-byte
        // NVLink stores instead of one 4-byte store per row and peer
        MK_SYNC();
        if (warp < comm.world) {
            const size_t off = ((size_t)((xseq + 1u) & 1u) * CC_COMM_MAX_RANKS + comm.rank) * CC_COMM_MAX_ELEMS + g.first;
            for (int c4 = lane * 4; c4 < g.n_units; c4 += 128) *(float4*)(comm.data[warp] + off + c4) = *(const float4*)(s_part + c4);
        }
    }
}

// SMP: the table ends with its only SAMPLE phase (see mega.cu).  QWEN2: the table has qwen2 layers -- Neox RoPE in its attention phases,
// one bias per matrix in its q/k/v phases -- a separate instantiation, so that the llama ones compile exactly as without qwen2
template <bool GEN, bool SMP, bool QWEN2>
__global__ void __launch_bounds__(MR_THREADS, 1) mega_ring_kernel(const MkPhase* __restrict__ phases, int n_phases, const uint8_t* dyn, unsigned* bar,
                                                                  const uint16_t* exp_lut, unsigned long long* prof, bool test_stall, int wtop_off, unsigned* err_host,
                                                                  const CommDev comm, const MrRing R, float* scores) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ float s_red[MK_WARPS];
    __shared__ MkPhase s_phs[2];             // phase descriptors of the compute warps, double-buffered
    __shared__ MkPhase s_pd[MR_PRODUCER_WARPS][2];      // every producer warp keeps its own copies (it runs phases ahead, at its own pace)
    __shared__ int s_abort;
    __shared__ int s_prod_done;
    __shared__ int s_ring_dead;
    __shared__ int s_unit;                   // dynamic dealing of a phase's units to the consumer warps
    __shared__ __align__(8) unsigned long long s_abar[AT_NBUF];
    __shared__ __align__(8) unsigned long long s_full[MR_MAX_SLOTS];
    __shared__ unsigned s_done[MR_MAX_SLOTS];     // entry number + 1 of the slot's last consumed tenant
    __shared__ unsigned s_seq[MR_MAX_SLOTS];      // entry number + 1 of the slot's current tenant
    unsigned apar = 0u;
    const unsigned abar0 = (unsigned)__cvta_generic_to_shared(&s_abar[0]);
    const unsigned full0 = (unsigned)__cvta_generic_to_shared(&s_full[0]);
    const unsigned done0 = (unsigned)__cvta_generic_to_shared(&s_done[0]);
    if (threadIdx.x == 0) {
        for (int i = 0; i < AT_NBUF; i++) mbar_init(abar0 + 8u * i, 1u);
        for (int i = 0; i < R.nslots; i++) { mbar_init(full0 + 8u * i, 1u); s_done[i] = 0u; s_seq[i] = 0u; }
        s_abort = 0; s_prod_done = 0; s_ring_dead = 0;
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();                         // the only barrier all 640 threads share
    if (threadIdx.x >= MK_THREADS) {
        mr_producer(phases, n_phases, R, full0, done0, (unsigned)__cvta_generic_to_shared(smem + R.ring_off), s_pd[(threadIdx.x - MK_THREADS) >> 5], s_seq, &s_abort, &s_prod_done,
                    prof ? prof + (size_t)n_phases * MK_PROF_SLOTS : nullptr);
        return;
    }
    MrCons RC;
    RC.full0 = full0; RC.done0 = done0; RC.ring = smem + R.ring_off; RC.slot_bytes = R.slot_bytes; RC.nslots = R.nslots; RC.ent_base = 0u;
    RC.s_unit = &s_unit; RC.s_seq = s_seq; RC.s_dead = &s_ring_dead; RC.err_dev = &bar[MK_BAR_ERR]; RC.err_host = err_host;
    uint8_t* work = smem;
    // norm-weight stage: the weights of the next fused-norm MATVEC phase, requested when the previous one's prologue is done (the
    // first at kernel start) -- they are read once per token, so from HBM, and would otherwise cost a trip after the barrier
    float* s_wn = (float*)(smem + wtop_off);
    const float* wst = nullptr;              // the norm weights requested into s_wn
    int xstaged = -1;                        // phase whose input row was requested into its working area as the barrier opened
    unsigned gen = 0;
    if (threadIdx.x == MK_BAR_THREAD) gen = ld_acquire_u32(&bar[32]);
    unsigned xseq = comm.world > 0 ? *comm.seq : 0u;
    for (int i = threadIdx.x; i < MR_DESC_WORDS; i += MK_THREADS) ((int*)&s_phs[0])[i] = ((const int*)phases)[i];
    const int n_loop = SMP ? n_phases - 1 : n_phases;      // SMP: the last phase, the sampler, runs after the loop
    for (int p = 0; p < n_loop; p++) {
        const bool stamp = prof && blockIdx.x == 0 && threadIdx.x == 0;
        const bool stampw = prof && blockIdx.x == 0 && threadIdx.x < 32;        // warp 0: ring occupancy (mr_ring_fill)
        if (stamp) {
            prof[p * MK_PROF_SLOTS] = globaltimer_ns(); prof[p * MK_PROF_SLOTS + 1] = 0; prof[p * MK_PROF_SLOTS + 4] = 0; prof[p * MK_PROF_SLOTS + 5] = 0; prof[p * MK_PROF_SLOTS + 8] = 0;
            if (p == 0) prof[9] = 0;            // later phases: stamped as the barrier in front of them opens
        }
        MK_SYNC();                           // descriptor p is in shared memory (stored one phase ago)
        const MkPhase& s_ph = s_phs[p & 1];
        if (p == 0 && !(s_ph.type == MK_MATVEC && s_ph.x && s_ph.norm_w)) { wst = s_ph.next_norm_w; if (wst) mr_stage_f32(s_wn, wst, s_ph.next_norm_n); }
        static_assert(sizeof(MkPhase) / 4 <= MK_THREADS, "descriptor does not fit one word per thread");
        int desc_w = 0;
        if (p + 1 < n_phases && threadIdx.x < sizeof(MkPhase) / 4) desc_w = ((const int*)(phases + p + 1))[threadIdx.x];
        unsigned long long* st1 = stamp ? prof + p * MK_PROF_SLOTS + 1 : nullptr;
        switch (s_ph.type) {
        case MK_NORMQ: phase_normq(s_ph, s_red); break;
        case MK_MATVEC:
            if (GEN && s_ph.act_type == CC_Q8_K) {
                switch (s_ph.wtype) {      // its cp.async.wait_group 0 also completes the norm-weight stage; without one it requests its weights
                case CC_Q2_K: phase_matvec_generic<TQ2_K>(s_ph, work, s_wn, s_ph.norm_w == wst, false, exp_lut, st1); break;
                case CC_Q3_K: phase_matvec_generic<TQ3_K>(s_ph, work, s_wn, s_ph.norm_w == wst, false, exp_lut, st1); break;
                case CC_Q4_K: phase_matvec_generic<TQ45_K<false>>(s_ph, work, s_wn, s_ph.norm_w == wst, false, exp_lut, st1); break;
                case CC_Q5_K: phase_matvec_generic<TQ45_K<true>>(s_ph, work, s_wn, s_ph.norm_w == wst, false, exp_lut, st1); break;
                case CC_Q6_K: phase_matvec_generic<TQ6_K>(s_ph, work, s_wn, s_ph.norm_w == wst, false, exp_lut, st1); break;
                default: phase_matvec_generic<TQ8_K>(s_ph, work, s_wn, s_ph.norm_w == wst, false, exp_lut, st1); break;
                }
                if (s_ph.x && s_ph.norm_w) { wst = s_ph.next_norm_w; if (wst) mr_stage_f32(s_wn, wst, s_ph.next_norm_n); }
                break;
            }
            if (s_ph.wtype == CC_Q8_0) phase_matvec_ring<CC_Q8_0, QWEN2>(s_ph, work, s_wn, wst, xstaged == p, exp_lut, RC, comm, xseq, st1);
            else phase_matvec_ring<CC_Q4_0, QWEN2>(s_ph, work, s_wn, wst, xstaged == p, exp_lut, RC, comm, xseq, st1);
            break;
        case MK_ATTN:
            if (s_ph.at.kv_f16) phase_attn<true, QWEN2>(s_ph, (float*)work, s_red, dyn, exp_lut, abar0, apar, R.at_ch, bar, err_host, &s_abort, scores);
            else phase_attn<false, QWEN2>(s_ph, (float*)work, s_red, dyn, exp_lut, abar0, apar, R.at_ch, bar, err_host, &s_abort, scores);
            break;
        case MK_ROWS: phase_rows(s_ph, dyn); break;
        case MK_REDUCE: phase_reduce(s_ph, comm, xseq, false); break;
        case MK_GATHER: phase_reduce(s_ph, comm, xseq, true); break;
        case MK_ARGMAX: phase_argmax(s_ph, dyn, s_red); break;
        }
        if (stamp) prof[p * MK_PROF_SLOTS + 2] = globaltimer_ns();
        if (p + 1 < n_phases && threadIdx.x < sizeof(MkPhase) / 4) ((int*)&s_phs[(p + 1) & 1])[threadIdx.x] = desc_w;
        const bool more = p + 1 < n_phases;
        const bool xg = s_ph.xgpu != 0;
        if (test_stall && p == 2 && blockIdx.x == gridDim.x - 1) { if (threadIdx.x == 0) s_abort = 1; break; }     // test hook: this CTA deserts
        if (more) grid_barrier_arrive(bar, gridDim.x, gen);
        if (stamp) prof[p * MK_PROF_SLOTS + 3] = globaltimer_ns();
        if (more) {
            grid_barrier_wait(bar, gridDim.x, gen, comm, xg ? xseq + 1u : 0u, &s_abort, err_host);
            gen++; if (xg) xseq++;
            // the occupancy as the barrier opened, or as this CTA gave up on it
            if (stampw) { const unsigned f = mr_ring_fill(s_seq, full0, R.nslots, RC.ent_base); if (stamp) prof[(p + 1) * MK_PROF_SLOTS + 9] = f; }
            if (s_abort) break;              // a barrier timed out: bail out, the host reports it
            // the barrier is open: the row the next fused prologue quantises is complete -- request it before the descriptor bookkeeping
            const MkPhase& nph = s_phs[(p + 1) & 1];
            if (nph.type == MK_MATVEC && nph.act_type != CC_Q8_K && nph.x && !nph.red_n) { mr_stage_f32((float*)(work + mr_x_off(nph.mv.k)), nph.x, nph.mv.k); xstaged = p + 1; }
        }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");      // a launch that gave up may still have stage copies in flight
    if constexpr (SMP) {                     // the SAMPLE phase after the loop, as in mega.cu
        MK_SYNC();
        if (!s_abort) phase_sample(s_phs[(n_phases - 1) & 1], dyn, work, exp_lut);
    }
    if (comm.world > 0 && blockIdx.x == 0 && threadIdx.x == 0) *comm.seq = xseq;
    if (prof && blockIdx.x == 0 && threadIdx.x == 0) prof[n_phases * MK_PROF_SLOTS] = globaltimer_ns();
    // a launch that gave up: the producer stops at its next look at s_abort; bulk copies it has already issued must land before
    // the CTA's shared memory goes away
    MK_SYNC();
    if (s_abort && threadIdx.x == 0) {
        while (*(volatile int*)&s_prod_done < MR_PRODUCER_WARPS) {}
        for (unsigned sl = 0; sl < (unsigned)R.nslots; sl++) {               // every slot's latest tenant has landed
            const unsigned q = *(volatile unsigned*)&s_seq[sl];
            if (q) mbar_wait(full0 + 8u * sl, ((q - 1u) / (unsigned)R.nslots) & 1u);
        }
    }
}

// ---- host side ---------------------------------------------------------------------------------------------------------------------------
// a streaming MATVEC phase can be fed by bulk copies when every segment is a whole number of 16-byte units at a 16-byte aligned address
// (always, since the scale rows are padded: CC_D_STRIDE; the check keeps the pointer alignment honest)
bool cc_mega_ring_phase_ok(const MkPhase& ph) {
    if (ph.type != MK_MATVEC || ph.act_type == CC_Q8_K) return true;
    if (ph.wtype != CC_Q8_0 && ph.wtype != CC_Q4_0) return false;
    if (ph.mv.k % 32) return false;
    for (int t = 0; t < ph.mv.mats.n; t++)
        if (((uintptr_t)ph.mv.mats.qs[t] | (uintptr_t)ph.mv.mats.d[t]) & 15u) return false;
    return true;
}
int cc_mega_ring_at_ch(const MkPhase& ph) {       // 48 KB of cache rows in flight per CTA either way (a V chunk: S times the rows, 1 / S of the columns)
    return ph.at.kv_f16 ? 64 : 32;
}
size_t cc_mega_ring_smem_for_phase(const MkPhase& ph) {
    if (ph.type == MK_MATVEC && ph.act_type == CC_Q8_K) return cc_mega_smem_for_phase(ph);
    if (ph.type == MK_MATVEC) return (size_t)mr_x_off(ph.mv.k) + (ph.x && !ph.red_n ? (size_t)ph.mv.k * 4 : 0);
    if (ph.type == MK_ATTN) return (size_t)(3 * ph.at.hd + ((ph.at.max_len + 8 + 3) & ~3)) * 4 + (size_t)AT_NBUF * cc_mega_ring_at_ch(ph) * ph.at.hd * (ph.at.kv_f16 ? 2 : 4) + 64;
    if (ph.type == MK_SAMPLE) return SMP_SMEM_BYTES;
    return 1024;
}
// Ring layout, for the fit decision (lazy.cu choose_mega) and the launch alike: the ring starts at mr_ring_off, after the working area
// and the norm-weight stage, and takes what is left of the SM's shared memory.  Returns the slot count, or 0 when fewer than
// MR_MIN_SLOTS fit -- e.g. a 32 K-token context, whose attention phase needs 128 KB for the score row alone -- and lazy.cu runs the
// table in the CUDA-graph mode.
// Ring depth, history: a Q8_0 ring (4352-byte slots) was faster SHALLOW -- 24 slots = 104 KB per SM decode a Llama-2-7B token in 3.88 ms
// against 4.04 ms with the ~40 that fit, and 20 / 16 / 12 slots are slower again (NVIDIA H100 80GB HBM3, 400 W).  Retuned with the
// prologue inputs staged early: 16-24 slots within the spread, 28 and 32 are 4-6 % slower (same card, 700 W).  The Q4_0 consumer is
// ALU-bound and keeps every slot that fits: a 55 KB ring (24 of its slots) cost it 2-4 %, 46 KB 9 %.
// Why: more than ~24 Q8_0 entries in flight per SM make the SMs' progress through a phase uneven, and the barrier waits for the
// slowest; but a 24-slot ring is full, and its SM reads no weights, through every prologue and attention phase (tools/mega_profile.py).
// So every ring now takes all the slots that fit, and a Q8_0 producer keeps at most MR_Q8_FLIGHT entries in flight: the in-phase queue
// stays short, and the slots beyond it fill with landed weights while the SM has nothing else to read (DESIGN §10).  The Q4_0 consumer
// is the bound of its phases and keeps no in-flight limit.
#define MR_MIN_SLOTS 12
static size_t mr_ring_off(const MegaLaunch& L) { return ((((L.smem + 15) & ~(size_t)15) + L.wstage) + 127) & ~(size_t)127; }
static auto mr_kernel(const MegaLaunch& L) {
    if (L.qwen2) return L.generic ? (L.sample ? mega_ring_kernel<true, true, true> : mega_ring_kernel<true, false, true>) : (L.sample ? mega_ring_kernel<false, true, true> : mega_ring_kernel<false, false, true>);
    return L.generic ? (L.sample ? mega_ring_kernel<true, true, false> : mega_ring_kernel<true, false, false>) : (L.sample ? mega_ring_kernel<false, true, false> : mega_ring_kernel<false, false, false>);
}
int cc_mega_ring_slots(const MegaLaunch& L) {
    cudaFuncAttributes fa;
    if (cudaFuncGetAttributes(&fa, mr_kernel(L)) != cudaSuccess) { cudaGetLastError(); return 0; }
    const size_t cap = 227 * 1024 - fa.sharedSizeBytes, off = mr_ring_off(L);
    if (L.slot_bytes <= 0 || off >= cap) return 0;
    const int fit = (int)std::min((cap - off) / (size_t)L.slot_bytes, (size_t)MR_MAX_SLOTS);
    if (fit < MR_MIN_SLOTS) return 0;
    return fit;
}

int cc_launch_mega_ring(cc_device* dev, const MkPhase* phases_dev, int n_phases, const uint8_t* dyn_dev, unsigned* bar_dev, const MegaLaunch& L,
                        unsigned long long* prof, const CommDev* comm) {
    auto kern = mr_kernel(L);
    const size_t wtop = (L.smem + 15) & ~(size_t)15;
    const size_t ring_off = mr_ring_off(L);
    const size_t smem = ring_off + (size_t)L.nslots * L.slot_bytes;
    CC_CUDA(dev, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int max_ctas_per_sm = 0;
    CC_CUDA(dev, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&max_ctas_per_sm, kern, MR_THREADS, smem));
    CC_REQUIRE(dev, max_ctas_per_sm >= 1, "megakernel (ring) does not fit on an SM");
    CommDev cd;
    memset(&cd, 0, sizeof(cd));
    if (comm) cd = *comm;
    MrRing R;
    R.ring_off = (int)ring_off; R.slot_bytes = L.slot_bytes; R.nslots = L.nslots; R.at_ch = L.at_ch;
    R.flight = L.slot_bytes >= 4352 ? std::min(L.nslots, MR_Q8_FLIGHT) : L.nslots;
    const uint16_t* lut = dev->exp_lut;
    return mk_launch(dev, kern, dev->sm_count, MR_THREADS, smem, phases_dev, n_phases, dyn_dev, bar_dev, lut, prof, cc_mega_test_stall(), (int)wtop,
                     dev->err_host, (const CommDev)cd, (const MrRing)R, L.scores);
}
