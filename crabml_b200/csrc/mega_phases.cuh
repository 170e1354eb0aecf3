// mega_phases.cuh -- device code shared by the two persistent decode kernels (mega.cu: tables without a Q8_0 / Q4_0 phase,
// mega_ring.cu: Q8_0 / Q4_0 weights through a TMA-fed shared-memory ring): grid barrier, phase bodies other than the streaming MATVEC.
// The including file defines MK_SYNC() -- the barrier of the 512 compute threads of a CTA (mega.cu: the whole CTA; mega_ring.cu:
// named barrier 1, the producer warp stays out of it) -- before including this header.
#pragma once
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "dequant.cuh"
#include "quantize_dev.cuh"
#include "vecdot.cuh"
#include "sample_dev.cuh"

#ifndef MK_SYNC
#error "define MK_SYNC() before including mega_phases.cuh"
#endif

// one CTA of 16 warps per SM: the grid barrier has one participant per SM instead of two (its cost is what bounds a phase)
#define MK_THREADS 512
#define MK_WARPS 16
#define MK_CTAS_PER_SM 1
#define MK_SEG 4
#define MK_XSTAGE_ROWS 512         // exchange phases: rows of one CTA's contiguous block (2 KB stage in shared memory)

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u32(unsigned* p, unsigned v) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

// Split grid barrier (tools/barrier_floor.py times it against a two-level acq_rel-atomic version and relaxed polling + fence):
//   arrive : bar.sync, then ONE thread does a fire-and-forget red.release.gpu.add on a flat monotonic counter
//            (the release publishes the CTA's phase output; that thread never issues prefetch loads);
//   ...      the other warps may already request the next phase's norm weights (mega.cu);
//   wait   : every CTA watches the counter reach (gen+1) * nblocks with ld.acquire (one L2 round trip less than counter -> CTA 0
//            -> generation word); CTA 0 also publishes the generation word, which the next launch starts from and which the other
//            CTAs wait for at an exchange barrier; then bar.sync.
// Layout (u32 words on separate 128-byte lines): [0] arrival counter, [32] generation.  Both are monotonic ACROSS launches (u32
// wrap-around included: only equality is tested): a launch starts from the generation the previous one left, so a graph
// replay needs no reset node in front of the kernel.
__device__ __forceinline__ void red_add_release(unsigned* p, unsigned v) { asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
#define MK_BAR_THREAD (MK_THREADS - 1)
#define MK_BAR_ERR 64                        // bar[64]: non-zero once any spin on this GPU has timed out
__device__ __forceinline__ unsigned long long globaltimer_ns() { return cc_globaltimer_ns(); }
// every spin is bounded (CcSpin, common.cuh): a barrier that cannot complete ends in CC_ERR_CUDA "megakernel barrier timeout"
struct MkSpin {
    CcSpin sp;
    __device__ __forceinline__ bool expired(unsigned* bar, unsigned* err_host, unsigned code) { return sp.expired(&bar[MK_BAR_ERR], err_host, code); }
};
// Exchange phases: the partial rows a CTA stored into the peers' exchange slots are ordered before the peers' reads by the chain
// (CTA i) red.release.gpu -> (CTA 0) ld.acquire.gpu ... st.release.sys -> (peer) ld.acquire.sys (grid_barrier_wait): release/acquire
// patterns of different scopes compose (PTX memory model: causality order is transitive over morally strong synchronisation), so no
// CTA needs a system-scope fence of its own before it arrives.
__device__ __forceinline__ void grid_barrier_arrive(unsigned* bar, unsigned nblocks, unsigned gen) {
    MK_SYNC();
    if (threadIdx.x == MK_BAR_THREAD) red_add_release(&bar[0], 1u);
}
// xseq != 0: the barrier doubles as the handshake of exchange number xseq with the other GPUs (protocol: comm.cu).  CTA 0's
// barrier thread, once every local CTA has arrived (all partial rows are stored in the peers' slots), publishes xseq in each
// peer's flag word, waits for every peer's xseq in its own flag words, and only then opens the local barrier (the generation word).
__device__ __forceinline__ void grid_barrier_wait(unsigned* bar, unsigned nblocks, unsigned gen, const CommDev& comm, unsigned xseq,
                                                  int* s_abort, unsigned* err_host) {
    const int lane = threadIdx.x & 31;
    if ((threadIdx.x >> 5) == MK_WARPS - 1) {              // the warp of MK_BAR_THREAD (its lane 31)
        const unsigned target = (gen + 1u) * nblocks;
        bool ok = true;
        if (blockIdx.x == 0) {
            if (lane == 31) { MkSpin sp; while ((int)(ld_acquire_u32(&bar[0]) - target) < 0) if (sp.expired(bar, err_host, 1u)) { ok = false; break; } }   // (the others may already be arriving at the next barrier)
            if (xseq) {                                     // kernel-uniform: the whole warp takes this branch together
                __syncwarp();                               // every local CTA has arrived: all partial rows are in the peers' slots
                if (lane < comm.world) {                    // one lane per peer: publish and poll in parallel, not rank after rank
                    // st.release.sys orders everything this warp has observed (lane 31's acquire of the arrival counter, handed over
                    // by the __syncwarp above) before the flag: no separate system fence
                    cc_st_release_sys(comm.flag[lane] + comm.rank * 32, xseq);
                    const unsigned* f = comm.flag[comm.rank] + lane * 32;
                    MkSpin sp;
                    while ((int)(cc_ld_acquire_sys(f) - xseq) < 0) if (sp.expired(bar, err_host, 2u)) { ok = false; break; }
                }
                __syncwarp();
            }
            if (lane == 31) st_release_u32(&bar[32], gen + 1u);
        } else if (lane == 31) {
            MkSpin sp;
            if (!xseq) { while ((int)(ld_acquire_u32(&bar[0]) - target) < 0) if (sp.expired(bar, err_host, 1u)) { ok = false; break; } }   // fast CTAs may already have arrived at the NEXT barrier
            else { while (ld_acquire_u32(&bar[32]) != gen + 1u) if (sp.expired(bar, err_host, 1u)) { ok = false; break; } }   // exchange: opened by CTA 0 after the handshake
        }
        if (!ok) *s_abort = 1;
    }
    MK_SYNC();
}

__device__ __forceinline__ float ldcg_f(const float* p) { return __ldcg(p); }
// cc_block_sum_512 (common.cuh) on the CTA's compute barrier
__device__ __forceinline__ float mk_block_sum_512(float v, float* s_red /* [16] */) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    MK_SYNC();
    float t = 0.0f;
#pragma unroll
    for (int w = 0; w < CC_RED_WARPS; w++) t += s_red[w];
    MK_SYNC();
    return t;
}


// ---- NORMQ phase (fused.cu normq_kernel, grid-wide) -----------------------------------------------------------------
static __device__ void phase_normq(const MkPhase& ph, float* s_red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n = ph.n;
    float* x = ph.x;
    float rms = 1.0f;
    // write_back: the normalised row must be materialised in place -> one CTA does the whole row (nobody else may
    // still be summing x while it is overwritten)
    if (ph.write_back && blockIdx.x != 0) return;
    // this warp's blocks are requested first, so their latency overlaps the row pass below (one L2 round trip in total)
    const int nb0 = n >> 5;
    const int gw0 = ph.write_back ? warp : blockIdx.x * MK_WARPS + warp, tw0 = ph.write_back ? MK_WARPS : gridDim.x * MK_WARPS;
    float pre[4];
#pragma unroll
    for (int j = 0; j < 4; j++) { const int b = gw0 + j * tw0; pre[j] = b < nb0 ? ldcg_f(x + b * 32 + lane) : 0.0f; }
    if (ph.norm_w) {
        float ss = 0.0f;
        const float4* x4 = (const float4*)x;
        const int n4 = n >> 2;
        for (int i0 = 0; i0 < n4; i0 += MK_THREADS * 4) {
            float4 v[4];
#pragma unroll
            for (int j = 0; j < 4; j++) { int i = i0 + j * MK_THREADS + threadIdx.x; v[j] = i < n4 ? __ldcg(x4 + i) : make_float4(0, 0, 0, 0); }
#pragma unroll
            for (int j = 0; j < 4; j++) ss += v[j].x * v[j].x + v[j].y * v[j].y + v[j].z * v[j].z + v[j].w * v[j].w;
        }
        ss = warp_sum(ss);
        if (lane == 0) s_red[warp] = ss;
        MK_SYNC();
        float t = 0.0f;
#pragma unroll
        for (int w = 0; w < MK_WARPS; w++) t += s_red[w];
        rms = sqrtf(t / (float)n + ph.eps);
        MK_SYNC();
    }
    ActQ8_0 act = ph.act;
    const int nb = n >> 5;
    const int gw = ph.write_back ? warp : blockIdx.x * MK_WARPS + warp, tw = ph.write_back ? MK_WARPS : gridDim.x * MK_WARPS;
    auto do_block = [&](int b, float v) {
        if (ph.orig) ph.orig[b * 32 + lane] = v;
        if (ph.norm_w) { v = (v / rms) * ph.norm_w[b * 32 + lane]; if (ph.write_back) x[b * 32 + lane] = v; }
        float amax = warp_max(fabsf(v));
        float d = amax / 127.0f;
        int q = __float2int_rz(v / d);
        act.qs[b * 32 + lane] = (int8_t)q;
        int s = warp_sum_i(q);
        if (lane == 0) { act.d[b] = __half2float(__float2half_rn(d)); act.isum[b] = s; }
    };
#pragma unroll
    for (int j = 0; j < 4; j++) { const int b = gw + j * tw; if (b < nb) do_block(b, pre[j]); }
    for (int b = gw + 4 * tw; b < nb; b += tw) do_block(b, ldcg_f(x + b * 32 + lane));
}

// ---- streaming MATVEC phase (mega_ring.cu): the body of matvec_stream_kernel (see matvec_stream.cu for the design notes) ----------
__device__ __forceinline__ int mk_dp16(const int4& w, const int4& a) {
    return __dp4a(w.x, a.x, __dp4a(w.y, a.y, __dp4a(w.z, a.z, __dp4a(w.w, a.w, 0))));
}
__device__ __forceinline__ void mbar_init(unsigned mbar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_wait(unsigned mbar, unsigned parity) {
    asm volatile(
        "{\n.reg .pred p;\nMK_WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@!p bra MK_WAIT_%=;\n}\n" ::"r"(mbar), "r"(parity) : "memory");
}
// (Tried and removed in round 2: an L2 look-ahead of each warp's coming rows -- cp.async.bulk.prefetch.L2 as
// well as per-lane prefetch.global.L2 -- made the token SLOWER: a bulk prefetch request occupies its issuing thread for
// a long time, line prefetches cost issue slots at the phase boundary, and the phase bodies already stream at HBM speed.)

// ---- generic MATVEC phase: K-quant weights (Q2_K .. Q6_K, Q8_K) against the Q8_K-quantised activation ---------------------------
// Same shape as the streaming phase of mega_ring.cu -- fused prologue ([rms_norm * w] + activation quantisation, recomputed by every
// CTA), the same epilogues -- but the row dot is the type's T::row_dot of vecdot.cuh (what the eager matvec_kernel runs, hence the
// same bits) and the weights are loaded by the computing warp itself.
// shared memory: qs [k] | d [k/256] | bsums [k/16] (TKBase) | reduction scratch | f32 x
__device__ __forceinline__ int mk_generic_sx_offset(int k) { return ((TKBase::smem_bytes(k) + 15) & ~15) + 256; }
// __noinline__ in the ring kernel (MK_GENERIC_NOINLINE, mega_ring.cu): the K-quant row dots are register-hungry; as a called function they
// get their own allocation instead of pushing spills into the streaming phases of the same kernel (every phase of the Q4_0 body was slower
// in the instantiation that carries the generic code inline).  mega.cu has no streaming phase: there the phase stays inline, and the two
// weight segments in flight live in the caller's KSeg pair (MK_GENERIC_SEGS), one pair for all six inlined instantiations -- a pair of
// their own each costs mega_kernel a 480-byte stack frame and 848 / 1312-1328 bytes of spills instead of 112 and 208 / 284 (both layouts compiled from the same
// sources, nvcc 12.9 -Xptxas -v).
#ifndef MK_GENERIC_NOINLINE
#define MK_GENERIC_NOINLINE 0
#endif
#if MK_GENERIC_NOINLINE
#define MK_GENERIC_ATTR __noinline__
#define MK_GENERIC_SEGS
#else
#define MK_GENERIC_ATTR
#define MK_GENERIC_SEGS , KSeg& S0, KSeg& S1
#endif
template <class T>
static __device__ MK_GENERIC_ATTR void phase_matvec_generic(const MkPhase& ph, uint8_t* smem, float* s_w, bool w_staged, bool x_staged, const uint16_t* exp_lut, unsigned long long* stamp1 MK_GENERIC_SEGS) {
    const StreamArgs& A = ph.mv;
    const StreamMats& M = A.mats;
    const int k = A.k;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int8_t* s_q = (int8_t*)smem;
    float* s_d = (float*)(smem + al16i(k));
    int16_t* s_bs = (int16_t*)(smem + al16i(k) + al16i(k / 256 * 4));
    float* s_red = (float*)(smem + mk_generic_sx_offset(k) - 256);
    float* s_x = (float*)(smem + mk_generic_sx_offset(k));
    {   // one L2 round trip: the f32 row (unless requested right after the barrier) and the norm weights (unless staged before it)
        const int n4 = k >> 2;
        const unsigned sx = (unsigned)__cvta_generic_to_shared(s_x), sw = (unsigned)__cvta_generic_to_shared(s_w);
        if (ph.norm_w && !w_staged)
            for (int i = threadIdx.x; i < n4; i += MK_THREADS) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sw + i * 16), "l"(ph.norm_w + i * 4) : "memory");
        if (!x_staged)
            for (int i = threadIdx.x; i < n4; i += MK_THREADS) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sx + i * 16), "l"(ph.x + i * 4) : "memory");
        asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
        MK_SYNC();
        if (stamp1) stamp1[3] = globaltimer_ns();
    }
    float rms = 1.0f;
    if (ph.norm_w) {                                                    // canonical order (common.cuh)
        float ss = 0.0f;
        const float4* x4 = (const float4*)s_x;
        for (int i = threadIdx.x; i < (k >> 2); i += MK_THREADS) ss += cc_sq4(x4[i]);
        rms = sqrtf(mk_block_sum_512(ss, s_red) / (float)k + ph.eps);
    }
    if (stamp1) stamp1[4] = globaltimer_ns();
    if (ph.orig && blockIdx.x == 0)                                     // Tensor::dup of the un-normalised row (llama2.rs:227,607)
        for (int i = threadIdx.x; i < (k >> 2); i += MK_THREADS) ((float4*)ph.orig)[i] = ((const float4*)s_x)[i];
    for (int sb = warp; sb < (k >> 8); sb += MK_WARPS) {                // one warp per 256-element super-block (buf_q8_k.rs:84-131)
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            v[i] = s_x[sb * 256 + lane * 8 + i];
            if (ph.norm_w) v[i] = (v[i] / rms) * s_w[sb * 256 + lane * 8 + i];
        }
        cc_quant_q8k_sblock(v, lane, s_q + sb * 256, s_d + sb, s_bs + sb * 16);
    }
    MK_SYNC();
    if (stamp1) *stamp1 = globaltimer_ns();
    // rows dealt warp-major: when rows do not divide by the warp count, every SM gets the same mix of k- and (k+1)-row warps
    // (CTA-major numbering left the last SMs with half the work of the first ones)
    const int gw = warp * gridDim.x + blockIdx.x, TW = gridDim.x * MK_WARPS;
    const bool pair = A.epilogue == 2;
    const int m_cat = pair ? M.m[0] : M.m[0] + (M.n > 1 ? M.m[1] : 0) + (M.n > 2 ? M.m[2] : 0);
    const int n_rows = gw < m_cat ? (m_cat - gw + TW - 1) / TW : 0;
    const int n_vrows = pair ? 2 * n_rows : n_rows;
    float first = 0.0f, pend_a = 0.0f, pend_b = 0.0f, pend_res = 0.0f;
    unsigned short pend_lut = 0;
    int pend_row = -1;
    auto flush_pending = [&]() {
        if (lane == 0 && pend_row >= 0) {
            if (pair) M.out[0][pend_row] = (pend_a / (1.0f + h2f_bits(pend_lut))) * pend_b;
            else M.out[0][pend_row] = pend_a + pend_res;
        }
        pend_row = -1;
    };
    auto locate = [&](int i, int& mat) -> int {                          // i-th virtual row of this warp -> (matrix, row)
        int r;
        mat = 0;
        if (pair) { mat = i & 1; r = gw + (i >> 1) * TW; }
        else {
            r = gw + i * TW;
            if (M.n > 1 && r >= M.m[0]) { r -= M.m[0]; mat = 1; if (M.n > 2 && r >= M.m[1]) { r -= M.m[1]; mat = 2; } }
        }
        return r;
    };
    auto planes = [&](int mat) -> WPlanes {
        WPlanes W;
        W.p[0] = mat == 0 ? M.qs[0] : mat == 1 ? M.qs[1] : M.qs[2];
        W.p[1] = (const uint8_t*)(mat == 0 ? M.d[0] : mat == 1 ? M.d[1] : M.d[2]);
        W.p[2] = mat == 0 ? M.p2[0] : mat == 1 ? M.p2[1] : M.p2[2];
        W.p[3] = mat == 0 ? M.p3[0] : mat == 1 ? M.p3[1] : M.p3[2];
        return W;
    };
    auto emit = [&](int i, float v) {                                    // row i of this warp is reduced: epilogue
        int mat;
        const int r = locate(i, mat);
        if (pair) {
            if ((i & 1) == 0) { first = v; return; }
            flush_pending();
            if (lane == 0) { pend_a = first; pend_b = v; pend_row = r; pend_lut = exp_lut[f2h_bits(-first)]; }
        } else if (A.epilogue == 1) {
            flush_pending();
            if (lane == 0) { pend_a = v; pend_row = r; pend_res = ldcg_f(A.residual[0] + r); }      // one matrix: lazy.cu keeps per-matrix vectors out of this phase
        } else if (lane == 0) {
            float* o = mat == 0 ? M.out[0] : mat == 1 ? M.out[1] : M.out[2];
            o[r] = v;
        }
    };
    if constexpr (T::kSegmented) {
        // rows cut into segments of 16 super-blocks; the loads of segment u + 2 are issued before segment u + 1 is consumed (two
        // segments = 16-24 LDG.128 per lane in flight), across row boundaries
        const int NSEG = ((k >> 8) + 15) >> 4;
        const int U = n_vrows * NSEG;
#if MK_GENERIC_NOINLINE
        KSeg S0, S1;
#endif
        int x0[4] = {0, 0, 0, 0}, x1[4] = {0, 0, 0, 0};
        int l_i = 0, l_seg = 0;
        auto load = [&](KSeg& S, int (&x)[4], bool valid) {
            if (valid) { int mat; const int r = locate(l_i, mat); T::seg_load(S, x, planes(mat), r, k, l_seg, lane); }
            if (++l_seg == NSEG) { l_seg = 0; l_i++; }
        };
        load(S0, x0, U > 0);
        load(S1, x1, U > 1);
        float acc = 0.0f;
        int c_i = 0, c_seg = 0;
        auto finish = [&]() { if (++c_seg < NSEG) return; c_seg = 0; const float v = warp_sum(acc); acc = 0.0f; emit(c_i++, v); };
        for (int u = 0; u < U; u += 2) {
            acc = T::seg_dot(S0, x0, k, c_seg, smem, lane, acc);
            finish();
            load(S0, x0, u + 2 < U);
            if (u + 1 >= U) break;
            acc = T::seg_dot(S1, x1, k, c_seg, smem, lane, acc);
            finish();
            load(S1, x1, u + 3 < U);
        }
    } else {
        for (int i = 0; i < n_vrows; i++) {
            int mat;
            const int r = locate(i, mat);
            emit(i, warp_sum(T::row_dot(planes(mat), r, k, smem, lane)));
        }
    }
    flush_pending();
}

// ---- ATTN phase: arithmetic of fused.cu attn_decode_kernel, each head on S CTAs (phase_attn: S = 1 on a short history, else a.split
// from cc_attn_split).  The K (then V) rows a CTA reads are staged in shared memory in chunks with ALL loads of a chunk in flight at once: at
// decode the cost of this phase is HBM/L2 latency and the one SM a head's history streams through, not bandwidth, so round trips and SMs
// per head are what matter.
#define AT_CH 64
#define AT_NBUF 3
__device__ __forceinline__ unsigned atom_add_release(unsigned* p, unsigned v) {
    unsigned old;
    asm volatile("atom.release.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
    return old;
}
// Each head on S CTAs: S = a.split when SPLIT, else 1.  CTA c of head h scores the positions [c L / S, (c + 1) L / S) (the last range
// holds this token's own position, scored from s_q . s_k).  With SPLIT it publishes them in the head's row of the score scratch; once all
// S CTAs have arrived every CTA reads the whole row and runs the softmax over it in the canonical order, so all of them hold the same p.
// CTA c then accumulates PV for the dimensions [c hd / S, (c + 1) hd / S), sequentially over s, and quantises those hd / (32 S) Q8_0
// blocks of the output.  Each score is an independent dot product and each output element's PV sum keeps its order, so the bits do not
// depend on S.
template <bool KV_F16, bool SPLIT, bool NEOX>
static __device__ void phase_attn_heads(const MkPhase& ph, float* sm, float* s_red, const uint8_t* dyn, const uint16_t* exp_lut, unsigned abar0, unsigned& apar, const int at_ch,
                                        unsigned* bar, unsigned* err_host, int* s_abort, float* scores) {
    const AttnArgs& a = ph.at;
    const int n_heads = a.n_heads, n_kv = a.n_kv, hd = a.hd, rope_dim = a.rope_dim, S = SPLIT ? a.split : 1;
    const int64_t seq_stride = a.seq_stride;
    const int64_t* dynv = (const int64_t*)(dyn + ph.dyn_off);
    const float* rope_tab = (const float*)(dyn + ph.rope_off);
    const int kv_len = (int)dynv[1], L = kv_len + 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* s_q = sm; float* s_k = sm + hd; float* s_v = sm + 2 * hd; float* s_p = sm + 3 * hd;
    // AT_NBUF chunk buffers of at_ch cache rows each (raw bytes: f32 or f16), filled in a K-chunks-then-V-chunks job sequence with
    // AT_NBUF jobs in flight; one mbarrier per buffer.  A K chunk is at_ch contiguous rows of the CTA's range, one TMA bulk copy.  A V
    // chunk is vch = S at_ch rows of the CTA's dw = hd / S columns (the same bytes: the working area does not depend on S): with S = 1
    // contiguous rows again, one bulk copy; with S > 1 a strided slice of every row.
    uint8_t* s_buf = (uint8_t*)(sm + 3 * hd + ((a.max_len + 8 + 3) & ~3));
    const unsigned s_buf_smem = (unsigned)__cvta_generic_to_shared(s_buf);
    constexpr int ELT = KV_F16 ? 2 : 4;
    const unsigned buf_bytes = (unsigned)(at_ch * hd * ELT);
    const int pairs = rope_dim >> 1;
    const int dw = hd / S, vch = at_ch * S;
    const int NCV = (kv_len + vch - 1) / vch;                     // V chunks: every CTA of the head reads all kv_len rows (its columns)
    for (int u = blockIdx.x; u < n_heads * S; u += gridDim.x) {
        const int part = SPLIT ? u / n_heads : 0, h = u - part * n_heads;      // part-major: part 0 of every head on the CTA that has it without the split
        const int g = KV_F16 ? h / (n_heads / n_kv) : h % n_kv;
        const int p_lo = (int)((int64_t)part * L / S), p_hi = (int)((int64_t)(part + 1) * L / S), k_hi = SPLIT ? min(p_hi, kv_len) : kv_len;
        const int NCK = !SPLIT ? NCV : k_hi > p_lo ? (k_hi - p_lo + at_ch - 1) / at_ch : 0;      // K chunks of the cached positions in [p_lo, p_hi)
        const int NJ = NCK + NCV;
        int v_issued = 0;                                            // SPLIT: V chunks requested so far (one cp.async group each)
        const bool issuer = SPLIT || threadIdx.x == 0;               // who requests a job: all threads with cp.async V pieces, else thread 0
        auto issue_job = [&](int j) {                                // the issuers
            const unsigned mb = abar0 + 8u * (unsigned)(j % AT_NBUF), dst = s_buf_smem + (unsigned)(j % AT_NBUF) * buf_bytes;
            if (j < NCK || !SPLIT) {                                 // contiguous rows: one bulk copy
                const bool kj = j < NCK;
                const int p0 = kj ? p_lo + j * at_ch : (j - NCK) * at_ch, cnt = min(at_ch, (kj ? k_hi : kv_len) - p0);
                if (threadIdx.x == 0) {
                    const uint8_t* src = (const uint8_t*)(kj ? a.kcache : a.vcache) + ((int64_t)g * seq_stride + (int64_t)p0 * hd) * ELT;
                    const unsigned bytes = (unsigned)(cnt * hd * ELT);
                    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mb), "r"(bytes) : "memory");
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(mb) : "memory");
                }
            } else {
                // this CTA's dw columns of vch rows: 16-byte cp.async pieces spread over all threads (a bulk copy per 64-128-byte row
                // slice is a TMA request each, and the requests of a long context queue up behind each other)
                const int p0 = (j - NCK) * vch, cnt = min(vch, kv_len - p0), pr = dw * ELT / 16;
                const uint8_t* src = (const uint8_t*)a.vcache + ((int64_t)g * seq_stride + (int64_t)p0 * hd + part * dw) * ELT;
                for (int i = threadIdx.x; i < cnt * pr; i += MK_THREADS) {
                    const int r = i / pr, q = i - r * pr;
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + (unsigned)(r * pr + q) * 16u), "l"(src + (int64_t)r * hd * ELT + q * 16) : "memory");
                }
                asm volatile("cp.async.commit_group;" ::: "memory");
                v_issued++;
            }
        };
        auto wait_job = [&](int j) {                                // all threads, in job order
            if (SPLIT && j >= NCK) {                                 // this thread's pieces of chunk j have landed (later chunks may still be in flight), then everybody's
                const int newer = v_issued - (j - NCK) - 1;
                if (newer >= 2) asm volatile("cp.async.wait_group 2;" ::: "memory");
                else if (newer == 1) asm volatile("cp.async.wait_group 1;" ::: "memory");
                else asm volatile("cp.async.wait_group 0;" ::: "memory");
                MK_SYNC();
                return;
            }
            const int bsel = j % AT_NBUF;
            mbar_wait(abar0 + 8u * (unsigned)bsel, (apar >> bsel) & 1u);
            apar ^= 1u << bsel;
        };
        auto ld_kv = [&](const uint8_t* buf, int idx) -> float { return KV_F16 ? __half2float(((const __half*)buf)[idx]) : ((const float*)buf)[idx]; };
        // the first AT_NBUF jobs are requested up front; every later job is issued as soon as its buffer has been consumed
        if (issuer) for (int j = 0; j < min(AT_NBUF, NJ); j++) issue_job(j);
        for (int i = threadIdx.x; i < hd; i += MK_THREADS) {
            float qv, kvv;
            if (NEOX) {                                              // pairs (j, j + hd/2), j < rope_dim/2 (fused.cu attn_decode_kernel)
                const int half = hd >> 1;
                const bool second = i >= half;
                const int j = second ? i - half : i;
                if (j < pairs) {
                    const float c = rope_tab[j], s = rope_tab[pairs + j];
                    const float q0 = ldcg_f(a.q + h * hd + j), q1 = ldcg_f(a.q + h * hd + j + half);
                    const float k0 = ldcg_f(a.k + g * hd + j), k1 = ldcg_f(a.k + g * hd + j + half);
                    qv = second ? q0 * s + q1 * c : q0 * c - q1 * s;
                    kvv = second ? k0 * s + k1 * c : k0 * c - k1 * s;
                } else {
                    qv = ldcg_f(a.q + h * hd + i);
                    kvv = ldcg_f(a.k + g * hd + i);
                }
            } else if (i < rope_dim) {
                const int j = i >> 1;
                const float c = rope_tab[j], s = rope_tab[pairs + j];
                const float q0 = ldcg_f(a.q + h * hd + 2 * j), q1 = ldcg_f(a.q + h * hd + 2 * j + 1);
                const float k0 = ldcg_f(a.k + g * hd + 2 * j), k1 = ldcg_f(a.k + g * hd + 2 * j + 1);
                qv = (i & 1) ? q0 * s + q1 * c : q0 * c - q1 * s;
                kvv = (i & 1) ? k0 * s + k1 * c : k0 * c - k1 * s;
            } else {
                qv = ldcg_f(a.q + h * hd + i);
                kvv = ldcg_f(a.k + g * hd + i);
            }
            s_q[i] = qv * a.scale;
            s_k[i] = kvv;
            s_v[i] = ldcg_f(a.v + g * hd + i);
        }
        MK_SYNC();
        // one CTA per kv group appends this token's row: no CTA reads cache row kv_len in this phase
        const bool owner = part == 0 && (KV_F16 ? (h % (n_heads / n_kv) == 0) : (h < n_kv));
        if (owner) {
            for (int i = threadIdx.x; i < hd; i += MK_THREADS) {
                const int64_t off = (int64_t)g * seq_stride + (int64_t)kv_len * hd + i;
                if (KV_F16) { ((__half*)a.kcache)[off] = __float2half_rn(s_k[i]); ((__half*)a.vcache)[off] = __float2half_rn(s_v[i]); }
                else { ((float*)a.kcache)[off] = s_k[i]; ((float*)a.vcache)[off] = s_v[i]; }
            }
        }
        float* srow = SPLIT ? scores + (size_t)h * (size_t)(a.max_len + 1) : nullptr;
        // scores, chunk by chunk; per-lane summation order i = lane, lane+32, ... as in fused.cu
        for (int j = 0; j < NCK; j++) {
            const int p0 = p_lo + j * at_ch, cnt = min(at_ch, k_hi - p0);
            const uint8_t* kb = s_buf + (size_t)(j % AT_NBUF) * buf_bytes;
            wait_job(j);
            for (int s = warp; s < cnt; s += MK_WARPS) {
                float acc = 0.0f;
                for (int i = lane; i < hd; i += 32) acc += (KV_F16 ? __half2float(__float2half_rn(s_q[i])) : s_q[i]) * ld_kv(kb, s * hd + i);
                acc = warp_sum(acc);
                if (lane == 0) { s_p[p0 + s] = acc; if (SPLIT) srow[p0 + s] = acc; }
            }
            MK_SYNC();                                       // buffer consumed by every warp -> refill it
            if (issuer && j + AT_NBUF < NJ) issue_job(j + AT_NBUF);
        }
        if (warp == 0 && p_hi == L) {                              // this token's own position (the last range)
            float acc = 0.0f;
            for (int i = lane; i < hd; i += 32) {
                if (KV_F16) acc += __half2float(__float2half_rn(s_q[i])) * __half2float(__float2half_rn(s_k[i]));
                else acc += s_q[i] * s_k[i];
            }
            acc = warp_sum(acc);
            if (lane == 0) { s_p[kv_len] = acc; if (SPLIT) srow[kv_len] = acc; }
        }
        MK_SYNC();
        if (SPLIT) {
            // score exchange: the MK_SYNC above orders the CTA's row stores before the release; the arrival word is monotonic across phases
            // and launches (each phase adds AT_SPLIT_MAX in all), so the value it held before this CTA's add tells which phase this is
            if (threadIdx.x == 0) {
                unsigned* w = bar + AT_ARRIVE_WORD + 8 * h;
                const unsigned old = atom_add_release(w, AT_SPLIT_MAX / S), target = (old & ~(unsigned)(AT_SPLIT_MAX - 1)) + AT_SPLIT_MAX;
                MkSpin sp;
                for (unsigned v = old + AT_SPLIT_MAX / S; (int)(v - target) < 0; v = ld_acquire_u32(w))      // the last to arrive does not poll
                    if (sp.expired(bar, err_host, 1u)) { *s_abort = 1; break; }
            }
            MK_SYNC();
            for (int s = threadIdx.x; s < L; s += MK_THREADS) if (s < p_lo || s >= p_hi) s_p[s] = ldcg_f(srow + s);
            MK_SYNC();
        }
        float m = -INFINITY;
        for (int s = threadIdx.x; s < L; s += MK_THREADS) m = fmaxf(m, s_p[s]);
        m = warp_max(m);
        if (lane == 0) s_red[warp] = m;
        MK_SYNC();
        m = s_red[0];
#pragma unroll
        for (int w = 1; w < MK_WARPS; w++) m = fmaxf(m, s_red[w]);
        MK_SYNC();
        float sum = 0.0f;
        for (int s = threadIdx.x; s < L; s += MK_THREADS) {
            float e = h2f_bits(exp_lut[f2h_bits(s_p[s] - m)]);
            s_p[s] = e;
            sum += e;
        }
        sum = warp_sum(sum);
        if (lane == 0) s_red[warp] = sum;
        MK_SYNC();
        sum = 0.0f;
#pragma unroll
        for (int w = 0; w < MK_WARPS; w++) sum += s_red[w];
        for (int s = threadIdx.x; s < L; s += MK_THREADS) s_p[s] = s_p[s] / sum;
        MK_SYNC();
        // out[d] = sum_s p[s] * V[s][d], sequential over s (batch_matmul.rs:60-68 order); F16: f16 accumulation (buf_f16.rs:152-163)
        float accf = 0.0f;
        __half acch = __float2half_rn(0.0f);
        const int t = threadIdx.x, d = part * dw + t;
        for (int j = NCK; j < NJ; j++) {
            const int p0 = (j - NCK) * vch, cnt = min(vch, kv_len - p0);
            const uint8_t* vb = s_buf + (size_t)(j % AT_NBUF) * buf_bytes;
            wait_job(j);
            if (t < dw) {
                for (int s = 0; s < cnt; s++) {
                    if (KV_F16) acch = __hadd(acch, __hmul(((const __half*)vb)[s * dw + t], __float2half_rn(s_p[p0 + s])));
                    else accf += s_p[p0 + s] * ((const float*)vb)[s * dw + t];
                }
            }
            MK_SYNC();
            if (issuer && j + AT_NBUF < NJ) issue_job(j + AT_NBUF);
        }
        float* s_o = s_k;
        MK_SYNC();
        if (t < dw) {
            float o;
            if (KV_F16) { acch = __hadd(acch, __hmul(__float2half_rn(s_v[d]), __float2half_rn(s_p[kv_len]))); o = __half2float(acch); }
            else { accf += s_p[kv_len] * s_v[d]; o = accf; }
            a.out[h * hd + d] = o;
            s_o[t] = o;
        }
        MK_SYNC();
        if (a.act_scratch) {
            ActQ8_0 act = ph.act;
            for (int b = warp; b < (dw >> 5); b += MK_WARPS) {
                float v = s_o[b * 32 + lane];
                float amax = warp_max(fabsf(v));
                float dd = amax / 127.0f;
                int qq = __float2int_rz(v / dd);
                const int gb = h * (hd >> 5) + part * (dw >> 5) + b;
                act.qs[gb * 32 + lane] = (int8_t)qq;
                int ss = warp_sum_i(qq);
                if (lane == 0) { act.d[gb] = __half2float(__float2half_rn(dd)); act.isum[gb] = ss; }
            }
        }
        MK_SYNC();
    }
}

// SPLIT is a template parameter, and the one-CTA instantiation folds to the code of a one-CTA phase (thread 0 requests every job, K and V
// chunks cover the same kv_len rows) and stays inline: both kernels then compile to the registers, frames, spills and instruction counts
// of separate one-CTA and split functions (nvcc 12.9 -Xptxas -v).  One called function with a run-time S took 12.7 instead of 9.1 us per
// layer at ~60 positions; folding less than this cost the K-quant kernel 4 % (Llama-2-7B; NVIDIA H100 80GB HBM3, 700 W).  The split
// instantiation is a called function in the ring kernel (MK_GENERIC_NOINLINE), as the generic phase: inlined there, it cost the phases
// every token runs (Llama-2-7B Q8_0 at ~32-104 positions decoded 268 instead of 271 tok/s; called, 280: the kernel spills
// less than before the split; NVIDIA H100 80GB HBM3, 700 W).  Inlined in mega.cu, where a call spills more (nvcc 12.9 -Xptxas -v).
#if MK_GENERIC_NOINLINE
#define MK_ATTN_SPLIT_ATTR __noinline__
#else
#define MK_ATTN_SPLIT_ATTR
#endif
template <bool KV_F16, bool NEOX>
static __device__ MK_ATTN_SPLIT_ATTR void phase_attn_split(const MkPhase& ph, float* sm, float* s_red, const uint8_t* dyn, const uint16_t* exp_lut, unsigned abar0, unsigned& apar, const int at_ch,
                                        unsigned* bar, unsigned* err_host, int* s_abort, float* scores) {
    phase_attn_heads<KV_F16, true, NEOX>(ph, sm, s_red, dyn, exp_lut, abar0, apar, at_ch, bar, err_host, s_abort, scores);
}

// below AT_SPLIT_MIN_KV cached positions the score exchange costs more than the split saves (Llama-2-7B, per layer, split against one
// CTA per head: 10.4 / 8.8 us at ~60 positions, 14.3 / 12.9 at ~190, 22.3 / 23.1 at ~440, 70 / 88 at ~2040; NVIDIA H100 80GB HBM3,
// 700 W): one CTA per head
// NEOX: the qwen2 instantiations of the ring kernel (mega_ring.cu QWEN2), whose attention phases pair RoPE elements (j, j + hd/2)
template <bool KV_F16, bool NEOX>
static __device__ __forceinline__ void phase_attn(const MkPhase& ph, float* sm, float* s_red, const uint8_t* dyn, const uint16_t* exp_lut, unsigned abar0, unsigned& apar,
                                                  const int at_ch, unsigned* bar, unsigned* err_host, int* s_abort, float* scores) {
    if (ph.at.split > 1 && ((const int64_t*)(dyn + ph.dyn_off))[1] >= AT_SPLIT_MIN_KV) phase_attn_split<KV_F16, NEOX>(ph, sm, s_red, dyn, exp_lut, abar0, apar, at_ch, bar, err_host, s_abort, scores);
    else phase_attn_heads<KV_F16, false, NEOX>(ph, sm, s_red, dyn, exp_lut, abar0, apar, at_ch, bar, err_host, s_abort, scores);
}

// ---- ROWS phase: copy_rows_from with the row indices in dyn (embedding lookup / row pick) -----------------------------------
static __device__ void phase_rows(const MkPhase& ph, const uint8_t* dyn) {
    const int64_t* rows = ph.rows_dev ? (const int64_t*)ph.rows_dev : (const int64_t*)(dyn + ph.dyn_off);      // a device slot: read through L2 (written by a previous launch)
    const int64_t total = (int64_t)ph.n_rows * ph.cols;
    for (int64_t i = (int64_t)blockIdx.x * MK_THREADS + threadIdx.x; i < total; i += (int64_t)gridDim.x * MK_THREADS) {
        const int64_t r = i / ph.cols, c = i - r * ph.cols;
        const int64_t e = rows[r] * ph.cols + c;
        float v;
        if (ph.src_dtype == CC_F32) v = __ldcg((const float*)ph.planes.p[0] + e);
        else if (ph.src_dtype == CC_F16) v = __half2float(((const __half*)ph.planes.p[0])[e]);
        else v = dequant_elem(ph.src_dtype, ph.planes, e);
        if (ph.dst_dtype == CC_F32) ((float*)ph.dst)[i] = v; else ((__half*)ph.dst)[i] = __float2half_rn(v);
    }
}

// ---- ARGMAX phase: greedy sampling on the device (ops.cu argmax_kernel, the LAST maximum: sampler.rs:109-116); CTA 0 only -----------------
static __device__ void phase_argmax(const MkPhase& ph, const uint8_t* dyn, float* s_red) {
    if (blockIdx.x != 0) return;
    __shared__ long long s_idx[MK_WARPS];
    const float* x = ph.x;
    float bv = 0.0f; long long bi = -1;
    for (long long i = threadIdx.x; i < ph.n; i += MK_THREADS) { const float v = ldcg_f(x + i); if (bi < 0 || !(v < bv)) { bv = v; bi = i; } }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (oi >= 0 && (bi < 0 || ov > bv || (ov == bv && oi > bi))) { bv = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { s_red[threadIdx.x >> 5] = bv; s_idx[threadIdx.x >> 5] = bi; }
    MK_SYNC();
    if (threadIdx.x == 0) {
        for (int w = 1; w < MK_WARPS; w++) { const float ov = s_red[w]; const long long oi = s_idx[w]; if (oi >= 0 && (bi < 0 || ov > bv || (ov == bv && oi > bi))) { bv = ov; bi = oi; } }
        if (bi < 0) bi = 0;
        *ph.slot_dev = bi;
        const long long h = *(const long long*)(dyn + ph.dyn_off);
        if (h >= 0 && h < CC_HISTORY_CAP) ph.hist_dev[h] = bi;
    }
    MK_SYNC();
}

// ---- SAMPLE phase: temperature + top-p sampling (sample_dev.cuh, the kernel of the other modes); CTA 0 only, in the working area ----------
// __noinline__: the sampler's registers are its own; neither persistent kernel's allocation sees them
static __device__ __noinline__ void phase_sample(const MkPhase& ph, const uint8_t* dyn, uint8_t* work, const uint16_t* exp_lut) {
    if (blockIdx.x != 0) return;
    const SampleDyn a = *(const SampleDyn*)(dyn + ph.dyn_off);
    const long long id = cc_sample_block(ph.x, ph.n, a, false, cc_sample_scratch(ph.dst, ph.n), work, exp_lut);
    if (threadIdx.x == 0) {
        *ph.slot_dev = id;
        if (a.hist_index >= 0 && a.hist_index < CC_HISTORY_CAP) ph.hist_dev[a.hist_index] = id;
    }
}

// ---- REDUCE / GATHER phases: second half of an exchange (the first half is epilogue 3 of the MATVEC phase + the handshake
// carried by its barrier).  REDUCE: dst = sum over ranks of the partial rows, rank order, (+ residual)   GATHER: dst = slices
static __device__ void phase_reduce(const MkPhase& ph, const CommDev& comm, unsigned xseq, bool gather) {
    const float* base = comm.data[comm.rank] + (size_t)(xseq & 1u) * CC_COMM_MAX_RANKS * CC_COMM_MAX_ELEMS;
    const int n4 = ph.red_n >> 2;
    if (gather) {
        for (int i = blockIdx.x * MK_THREADS + threadIdx.x; i < n4 * comm.world; i += gridDim.x * MK_THREADS) {
            const int p = i / n4, j = i - p * n4;
            ((float4*)(ph.red_dst + (size_t)p * ph.red_n))[j] = __ldcg((const float4*)(base + (size_t)p * CC_COMM_MAX_ELEMS) + j);
        }
        return;
    }
    for (int i = blockIdx.x * MK_THREADS + threadIdx.x; i < n4; i += gridDim.x * MK_THREADS) {
        float4 a = __ldcg((const float4*)base + i);
        for (int p = 1; p < comm.world; p++) {
            const float4 b = __ldcg((const float4*)(base + (size_t)p * CC_COMM_MAX_ELEMS) + i);
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        if (ph.red_res) { const float4 r = __ldcg((const float4*)ph.red_res + i); a.x += r.x; a.y += r.y; a.z += r.z; a.w += r.w; }
        ((float4*)ph.red_dst)[i] = a;
    }
}


#define MK_F_TESTSTALL 128     // test hook: the last CTA leaves before barrier 2 -> every other CTA must time out, not hang (cc_mega_test_stall)

// Launch of a persistent kernel (mega.cu, mega_ring.cu).  The grid barrier needs every CTA resident at once.  On a GPU this process
// owns, a plain launch of one CTA per SM is co-resident by construction.  With another tenant on the same GPU (a second process, MPS)
// a partially scheduled grid cannot finish a barrier: every spin in the kernel is bounded (MkSpin) and ends in CC_ERR_CUDA "megakernel
// barrier timeout" instead of a hang; CRABML_MEGA_COOP=1 adds the cooperative launch attribute (all-or-nothing placement).  That is
// opt-in because a cooperative kernel node in a CUDA graph is much slower to launch than a plain one.
template <typename... P, typename... A>
static int mk_launch(cc_device* dev, void (*kern)(P...), int grid, int threads, size_t smem, A... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem; cfg.stream = dev->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = getenv("CRABML_MEGA_COOP") ? 1 : 0;
    cfg.attrs = attr; cfg.numAttrs = 1;
    CC_CUDA(dev, cudaLaunchKernelEx(&cfg, kern, args...));
    CC_LAUNCH_CHECK(dev);
    return CC_OK;
}
