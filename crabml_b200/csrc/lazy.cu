// lazy.cu -- lazy mode: record the trait calls of one forward(), fuse, replay as a CUDA graph.
//
// The reference's Tensor API is eager: ~31 calls per layer, ~1000 per token (SURVEY §3.2), each a separate launch in
// eager mode.  Per-launch overhead, not kernel bodies, is what caps decode.  In lazy mode the
// SAME C-ABI calls only append to a queue (after the same argument checks); the queue is executed at the first call that
// needs a result on the host (export / debug tap / synchronize -- the reference synchronises only there too, llama2.rs:209):
//   1. fuse: runs of ops that match the Llama decode layer (llama2.rs:226-269, 527-638) are replaced by fused steps, each described by
//      one phase descriptor (MkPhase) that the persistent kernels run and the CUDA-graph mode launches as a kernel of fused.cu /
//      matvec_stream.cu; anything unrecognised runs in order through cc_run_op (capi.cu), as in eager mode;
//   2. the plan is hashed: each eager op's words and each fused step's descriptor bytes.  Values that change every token
//      (position, KV length, token ids, RoPE table) live in a small device buffer `dyn` that the kernels read;
//   3. first time a hash is seen the launches are stream-captured into a CUDA graph (programmatic-dependent-launch edges
//      included); afterwards a token = one 1-2 KB H2D copy of `dyn` + one cudaGraphLaunch.
// The activation pool hands out the same pointers for the same call sequence (lowest free address first), which is what makes the
// hash stable from token to token.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <chrono>

#include "op_record.cuh"

// one captured token graph.  The cache key is a 64-bit fold of the launch signature; `sig` is the signature itself and is compared
// on every hit (a colliding key must re-capture, never replay another plan's baked pointers); `last_use` drives the LRU bound.
struct GraphEntry { cudaGraphExec_t exec = nullptr; size_t dyn_bytes = 0; uint64_t launches = 0; MkPhase* phases_dev = nullptr;
                    std::vector<uint64_t> sig; uint64_t last_use = 0; MegaVariant mega_variant = MEGA_NONE; };
#define LZ_MAX_GRAPHS 64                             // cached token graphs per device (a decode loop needs 2-4)

struct LazyState {
    std::vector<LOp> q;
    std::unordered_map<cc_buf*, int> qrefs;
#define LZ_DYN_SLOTS 8                               // tokens the host may run ahead of the GPU (absorbs host scheduling hiccups)
    uint8_t* dyn_host[LZ_DYN_SLOTS] = {nullptr};   // pinned, rotated so the host can build tokens t+1.. while t runs
    cudaEvent_t dyn_ev[LZ_DYN_SLOTS] = {nullptr};
    int dyn_slot = 0;
    uint8_t* dyn_dev = nullptr;
    size_t dyn_cap = 1 << 16;
    void* act[2] = {nullptr, nullptr};
    float* scores = nullptr;         // megakernels' attention phase: the score rows the CTAs of a head exchange (cc_attn_split)
    size_t scores_cap = 0;
    unsigned* bar_dev = nullptr;     // megakernel grid barrier {count, generation}, attention arrival words (AT_ARRIVE_WORD)
    unsigned long long* prof_dev = nullptr;   // CRABML_MEGA_PROF=1: per-phase start timestamps of the last megakernel run
    std::vector<int> prof_types;
    size_t act_cap = 0;
    std::unordered_map<uint64_t, GraphEntry> cache;
    uint64_t flushes = 0, graph_hits = 0, captures = 0, uncached = 0, evictions = 0, collisions = 0;
    uint64_t ns_record = 0, ns_fuse = 0, ns_submit = 0, n_ops = 0;      // host-side cost accounting
    MegaVariant mega_variant = MEGA_NONE;     // persistent kernel of the last megakernel flush
};

static void graph_entry_free(GraphEntry& ge) {
    if (ge.exec) cudaGraphExecDestroy(ge.exec);
    if (ge.phases_dev) cudaFree(ge.phases_dev);
    ge.exec = nullptr; ge.phases_dev = nullptr;
}
// drop every cached graph (their baked pointers are stale after the scratch buffers moved); the stream must be idle
static void graph_cache_clear(LazyState* lz) {
    for (auto& kv : lz->cache) graph_entry_free(kv.second);
    lz->cache.clear();
}
// the same, for what a graph bakes in outside the lazy state: the eager matvec steps' dev->act_scratch (cc_ensure_act_scratch) and the
// grid of every persistent or streaming kernel (cc_device_set_sm_limit).  Both change rarely, so the next flush of every plan
// re-captures rather than each signature carrying a scratch generation and the SM count.  The grid barrier restarts from zero too, as
// on a new device: its arrival counter holds (barriers so far) x (grid size), which a launch with another grid cannot continue
// (mega_phases.cuh grid_barrier_wait).  The stream must be idle.
int cc_lazy_invalidate(cc_device* dev) {
    LazyState* lz = dev->lz;
    if (!lz) return CC_OK;
    graph_cache_clear(lz);
    if (cudaMemsetAsync(lz->bar_dev, 0, 4096, dev->stream) != cudaSuccess) return cc_fail(dev, CC_ERR_CUDA, "lazy: barrier reset failed");
    return CC_OK;
}

LazyState* cc_lazy_create(cc_device* dev) {
    LazyState* lz = new LazyState();
    for (int i = 0; i < LZ_DYN_SLOTS; i++)
        if (cudaMallocHost(&lz->dyn_host[i], lz->dyn_cap) != cudaSuccess || cudaEventCreateWithFlags(&lz->dyn_ev[i], cudaEventDisableTiming) != cudaSuccess) { delete lz; return nullptr; }
    if (cudaMalloc(&lz->dyn_dev, lz->dyn_cap) != cudaSuccess) { delete lz; return nullptr; }
    if (getenv("CRABML_MEGA_PROF") && cudaMalloc(&lz->prof_dev, MK_PROF_SLOTS * 8 * 4097) == cudaSuccess) cudaMemset(lz->prof_dev, 0, MK_PROF_SLOTS * 8 * 4097);    // stamps a kernel never takes read 0
    if (cudaMalloc(&lz->bar_dev, 4096) != cudaSuccess || cudaMemset(lz->bar_dev, 0, 4096) != cudaSuccess) { delete lz; return nullptr; }
    lz->scores_cap = (size_t)1 << 20;                // 32 heads x 8K positions before the first regrowth (size_scratch)
    if (cudaMalloc(&lz->scores, lz->scores_cap) != cudaSuccess) { delete lz; return nullptr; }
    return lz;
}
void cc_lazy_destroy(cc_device* dev) {
    LazyState* lz = dev->lz;
    if (!lz) return;
    for (auto& op : lz->q) { if (op.a.buf) cc_tensor_release(op.a.buf); if (op.b.buf) cc_tensor_release(op.b.buf); if (op.out) cc_tensor_release(op.out); }
    for (auto& kv : lz->cache) graph_entry_free(kv.second);
    lz->cache.clear();
    if (lz->bar_dev) cudaFree(lz->bar_dev);
    for (int i = 0; i < LZ_DYN_SLOTS; i++) { if (lz->dyn_host[i]) cudaFreeHost(lz->dyn_host[i]); if (lz->dyn_ev[i]) cudaEventDestroy(lz->dyn_ev[i]); }
    if (lz->dyn_dev) cudaFree(lz->dyn_dev);
    for (int i = 0; i < 2; i++) if (lz->act[i]) cudaFree(lz->act[i]);
    if (lz->scores) cudaFree(lz->scores);
    delete lz;
    dev->lz = nullptr;
}

// ---- recording ---------------------------------------------------------------------------------------------------
static void hold(LazyState* lz, cc_buf* b) { if (b) { cc_tensor_retain(b); lz->qrefs[b]++; } }

int cc_lazy_record(cc_device* dev, LOp op) {
    LazyState* lz = dev->lz;
    auto t0 = std::chrono::steady_clock::now();
    for (cc_view* v : {&op.a, &op.b})      // a caller's view may leave the dims past ndim undefined; the plan signature hashes them all
        for (int k = v->ndim; k < CC_MAX_DIMS; k++) v->shape[k] = v->strides[k] = 0;
    hold(lz, op.a.buf); hold(lz, op.b.buf); hold(lz, op.out);
    lz->q.push_back(std::move(op));
    lz->n_ops++;
    lz->ns_record += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
    return CC_OK;
}

// ---- plan building ---------------------------------------------------------------------------------------------------
// A zero-filled descriptor of one fused step: its bytes, padding included (AttnArgs has 4 at its end), become signature words.
// Fill its fields in place: a struct assigned into it need not carry its own padding over.
static MkPhase new_phase(int type) {
    MkPhase ph;
    memset(&ph, 0, sizeof(ph));
    ph.type = type;
    return ph;
}

struct Plan {
    std::vector<uint64_t> sig;
    std::vector<uint8_t> dyn;
    // the CUDA-graph mode's launches, in order: a fused step (index into `emitted`) or an eager op (index into the queue)
    struct Step { bool eager; uint32_t at; };
    std::vector<Step> steps;
    bool cacheable = true;
    std::vector<MkPhase> emitted;    // the fused steps' descriptors as emitted, before merge_prologue folds any of `phases` together
    std::vector<MkPhase> phases;     // megakernel form of the same plan (valid while mega_ok)
    bool mega_ok = true;
    void S(uint64_t v) { sig.push_back(v); }
    void SP(const void* p) { sig.push_back((uint64_t)(uintptr_t)p); }
    // One fused step.  A captured graph bakes in all of its descriptor: the persistent kernels read the uploaded table, the CUDA-graph
    // mode launches from it (launch_phase).  So the descriptor's bytes are its signature words.  graph_step = false: a phase whose
    // CUDA-graph form is the eager ops the caller emits after it (Fuser::eager).
    void phase(const MkPhase& ph, bool graph_step = true) {
        static_assert(sizeof(MkPhase) % 8 == 0, "a descriptor is whole signature words");
        S(0x2000);
        const size_t at = sig.size();
        sig.resize(at + sizeof(MkPhase) / 8);
        memcpy(&sig[at], &ph, sizeof(MkPhase));
        phases.push_back(ph);
        if (graph_step) { steps.push_back({false, (uint32_t)emitted.size()}); emitted.push_back(ph); }
    }
    size_t dyn_put(const void* p, size_t n) {
        size_t off = (dyn.size() + 15) & ~(size_t)15;
        dyn.resize(off + n);
        memcpy(dyn.data() + off, p, n);
        return off;
    }
};

// Four interleaved lanes, so that the ~15 000 words of a Llama-2-7B token are not one chain of dependent multiplies.  The key only
// has to spread plans apart: a hit compares the whole signature.
static uint64_t hash_sig(const std::vector<uint64_t>& s) {
    const uint64_t prime = 1099511628211ull;
    uint64_t h[4] = {1469598103934665603ull, 1469598103934665603ull ^ 1, 1469598103934665603ull ^ 2, 1469598103934665603ull ^ 3};
    for (size_t i = 0; i < s.size(); i += 4)
        for (size_t l = 0; l < 4 && i + l < s.size(); l++) { h[l] ^= s[i + l]; h[l] *= prime; h[l] ^= h[l] >> 29; }
    return ((h[0] * prime ^ h[1]) * prime ^ h[2]) * prime ^ h[3];
}

// ---- the CUDA-graph mode's launches ---------------------------------------------------------------------------------------------
// one fused step, by its descriptor, as the kernel of fused.cu / matvec_stream.cu / comm.cu that does what its phase does in the
// persistent kernels (a generic K-quant MATVEC phase has none: its graph form is eager ops)
static int launch_phase(cc_device* d, const MkPhase& ph, const uint8_t* dyn_dev) {
    switch (ph.type) {
    case MK_NORMQ: return cc_launch_normq(d, ph.x, ph.orig, ph.norm_w, ph.eps, ph.n, ph.act, ph.write_back);
    case MK_MATVEC: {
        StreamArgs A = ph.mv;
        if (A.epilogue == 3) A.epilogue = 0;      // the exchange's stores into every rank's slot: here the REDUCE / GATHER step's kernel
        return cc_launch_matvec_stream(d, ph.wtype, A);
    }
    case MK_ATTN: return cc_launch_attn_decode(d, ph.at, (const int64_t*)(dyn_dev + ph.dyn_off), (const float*)(dyn_dev + ph.rope_off));
    case MK_ROWS:
        return cc_launch_dequant_rows(d, ph.planes, ph.src_dtype, ph.rows_dev ? (const int64_t*)ph.rows_dev : (const int64_t*)(dyn_dev + ph.dyn_off),
                                      ph.n_rows, ph.cols, ph.dst, ph.dst_dtype);
    case MK_REDUCE: return cc_launch_all_reduce(d, ph.red_dst, ph.red_n, ph.red_res);
    case MK_GATHER: return cc_launch_all_gather(d, ph.x, ph.red_n, ph.red_dst);
    case MK_ARGMAX: return cc_launch_argmax(d, ph.x, ph.n, (int64_t*)ph.slot_dev, (int64_t*)ph.hist_dev, (const int64_t*)(dyn_dev + ph.dyn_off), -1);
    case MK_SAMPLE: return cc_launch_sample(d, ph.x, ph.n, nullptr, (const SampleDyn*)(dyn_dev + ph.dyn_off), (int64_t*)ph.slot_dev, (int64_t*)ph.hist_dev);
    }
    return cc_fail(d, CC_ERR_UNSUPPORTED, "lazy: unknown phase type %d", ph.type);
}

struct Fuser {
    cc_device* dev;
    LazyState* lz;
    std::vector<LOp>& q;
    Plan& P;
    size_t rope_off = (size_t)-1; int64_t rope_pos = -1; int rope_hd = 0, rope_dim = 0, rope_mode = -1;

    bool is(size_t i, int kind) const { return i < q.size() && !q[i].done && q[i].kind == kind; }
    std::unordered_map<cc_buf*, size_t> last_use;      // buffer -> index of the last queued op that touches it (built once per flush)
    void index_uses() {
        last_use.reserve(q.size() * 2);
        for (size_t j = 0; j < q.size(); j++) {
            if (q[j].a.buf) last_use[q[j].a.buf] = j;
            if (q[j].b.buf) last_use[q[j].b.buf] = j;
            if (q[j].out) last_use[q[j].out] = j;
        }
    }
    // may an op of this flush write b?  (`a` is the destination of every in-place op; conservative for the others)
    bool written(const cc_buf* b) const {
        for (const LOp& op : q) if (op.a.buf == b || op.out == b) return true;
        return false;
    }
    // no op at or after `from` touches buf, and nobody outside the queue holds it
    bool dead_after(cc_buf* b, size_t from) const {
        auto lu = last_use.find(b);
        if (lu != last_use.end() && lu->second >= from) return false;
        auto it = lz->qrefs.find(b);
        int held = it == lz->qrefs.end() ? 0 : it->second;
        return b->refs.load() == held;
    }
    // an ADD / MUL that covers all n elements: the recorded counts are those capi.cu's binary() kept after chunks_exact(4), which
    // skips the tail of an rhs longer than 1 (arithmetic.rs:5-68) -- a fused epilogue or norm would apply it to every element
    bool covers(const LOp& op, int64_t n) const { return op.i0 == n && op.i1 == n; }

    // ---- eager steps ----------------------------------------------------------------------------------------------------------
    // op i runs as its eager kernel in the CUDA-graph mode
    void eager(size_t i) {
        const LOp& op = q[i];
        P.S(0x1000 + op.kind); P.SP(op.a.buf ? op.a.buf->plane[0] : nullptr); P.SP(op.b.buf ? op.b.buf->plane[0] : nullptr);
        P.SP(op.out ? op.out->plane[0] : nullptr);
        // the pool hands an f32 and an f16 buffer of one size class the same address, and a weight re-created at a freed address may
        // have another type: the kernels a step launches depend on the types
        P.S(op.a.buf ? op.a.buf->dtype : -1); P.S(op.b.buf ? op.b.buf->dtype : -1); P.S(op.out ? op.out->dtype : -1);
        for (int k = 0; k < CC_MAX_DIMS; k++) { P.S(op.a.shape[k]); P.S(op.a.strides[k]); P.S(op.b.shape[k]); P.S(op.b.strides[k]); }
        P.S(op.i0); P.S(op.i1); P.S(op.i2); uint32_t fb; memcpy(&fb, &op.f, 4); P.S(fb);
        switch (op.kind) {
        case L_ROPE: case L_CONCAT: case L_BMM: case L_SOFTMAX: P.cacheable = false; break;   // position / length dependent
        case L_COPY_ROWS: P.cacheable = false; break;   // (normally taken by try_copy_rows) host row list would be baked into a graph
        case L_MATVEC: if (op.b.ndim > 1 && op.b.shape[0] > 1) P.cacheable = false; break;   // batched (prefill) matmul: its scratch may be (re)allocated, never captured
        default: break;
        }
        for (int64_t r : op.rows) P.S((uint64_t)r);
        P.steps.push_back({true, (uint32_t)i});
        q[i].done = true;
    }
    // op i runs as its eager kernel, and no phase of the persistent kernels covers it: the plan runs in the CUDA-graph mode
    void fallback(size_t i) {
        P.mega_ok = false;
        eager(i);
    }

    // ---- matchers shared by the patterns below -------------------------------------------------------------------------------
    // [DUP] RMS_NORM MUL on one contiguous f32 row x (1 x n) with an f32 weight row: len = ops consumed, 0 = no match
    struct NormMatch { size_t len = 0; cc_buf* orig = nullptr; cc_buf* x = nullptr; cc_buf* w = nullptr; int64_t n = 0; float eps = 0.0f; };
    NormMatch match_norm(size_t i) const {
        NormMatch m;
        size_t j = i;
        if (is(j, L_DUP) && is(j + 1, L_RMS_NORM) && q[j + 1].a.buf == q[j].a.buf) { m.orig = q[j].out; j++; }
        if (!(is(j, L_RMS_NORM) && is(j + 1, L_MUL))) return NormMatch();
        const LOp &rn = q[j], &mu = q[j + 1];
        if (mu.a.buf != rn.a.buf) return NormMatch();
        const int64_t n = view_len(&rn.a);
        if (rn.a.ndim > 2 || (rn.a.ndim == 2 && rn.a.shape[0] != 1) || !view_contiguous(&rn.a)) return NormMatch();
        if (view_len(&mu.b) != n || mu.b.buf->dtype != CC_F32 || !view_contiguous(&mu.b) || !covers(mu, n)) return NormMatch();
        m.len = j + 2 - i; m.x = rn.a.buf; m.w = mu.b.buf; m.n = n; m.eps = rn.f;
        return m;
    }
    // does the streaming kernel take the MATVEC at t on row x?
    bool streams(size_t t, const cc_buf* x) const {
        if (!is(t, L_MATVEC)) return false;
        const LOp& mv = q[t];
        return mv.b.buf == x && cc_stream_supported(mv.a.buf->dtype, mv.a.shape[1]) && view_len(&mv.b) == mv.a.shape[1] && view_contiguous(&mv.b);
    }
    // the MATVEC at j (weight type wt, k columns) and up to two more of the same type and k on row x, with the epilogue that follows:
    // gate/up + silu + mul (llama2.rs:620-630), or one ADD of an f32 vector per matrix, in matrix order: x = matvec + residual
    // (llama2.rs:266,636) and qwen2's q/k/v biases (llama2.rs:315-317).  n matrices, `used` ops consumed.
    struct GroupMatch { size_t n = 1, used = 1; int epilogue = 0; cc_buf* residual[3] = {nullptr, nullptr, nullptr}; };
    // the ADD at `at` adds a whole contiguous f32 vector to the output of the MATVEC at t
    bool adds_vector(size_t at, size_t t) const {
        if (!is(at, L_ADD)) return false;
        const LOp &mv = q[t], &ad = q[at];
        return ad.a.buf == mv.out && view_len(&ad.b) == mv.a.shape[0] && covers(ad, mv.a.shape[0]) && ad.b.buf->dtype == CC_F32 && view_contiguous(&ad.b);
    }
    GroupMatch match_group(size_t j, const cc_buf* x, int wt, int64_t k) const {
        GroupMatch g;
        while (g.n < 3 && is(j + g.n, L_MATVEC) && q[j + g.n].b.buf == x && q[j + g.n].a.buf->dtype == wt && q[j + g.n].a.shape[1] == k &&
               view_len(&q[j + g.n].b) == k) g.n++;
        g.used = g.n;
        const LOp& m0 = q[j];
        bool adds = true;
        for (size_t t = 0; t < g.n; t++) adds = adds && adds_vector(j + g.n + t, j + t);
        if (g.n >= 2 && is(j + 2, L_SILU) && is(j + 3, L_MUL) && q[j + 2].a.buf == m0.out && q[j + 3].a.buf == m0.out && q[j + 3].b.buf == q[j + 1].out &&
            m0.a.shape[0] == q[j + 1].a.shape[0] && view_len(&q[j + 3].b) == m0.a.shape[0] && covers(q[j + 3], m0.a.shape[0]) && dead_after(q[j + 1].out, j + 4)) {
            g.n = 2; g.epilogue = 2; g.used = 4;
        } else if (adds) {
            g.epilogue = 1; g.used = 2 * g.n;
            for (size_t t = 0; t < g.n; t++) g.residual[t] = q[j + g.n + t].b.buf;
        } else if (g.n > 1 && is(j + g.n, L_SILU)) {
            g.n = 1; g.used = 1;                   // do not swallow a gate/up pair we could not fuse as a pair
        }
        return g;
    }

    // ---- pattern: [DUP] RMS_NORM MUL -> normq ; returns number of ops consumed (0 = no match) ---------------------------------
    // On success *xbuf receives the normalised row, whose quantisation is now in scratch act_sel.
    size_t try_normq(size_t i, int act_sel, cc_buf** xbuf) {
        const NormMatch nm = match_norm(i);
        if (!nm.len || nm.n % 32 || nm.n > 65536) return 0;
        // the normalised f32 row only has to be materialised if something other than the following matvecs reads it
        // (only matvecs the streaming kernel will take consume the quantised scratch; any other reader -- a K-quant or batched
        // matvec falling back to its eager kernel -- needs the f32 row)
        size_t end = i + nm.len;
        while (streams(end, nm.x)) end++;
        MkPhase ph = new_phase(MK_NORMQ);
        ph.write_back = !dead_after(nm.x, end);
        ph.x = (float*)nm.x->plane[0]; ph.orig = nm.orig ? (float*)nm.orig->base : nullptr; ph.norm_w = (const float*)nm.w->plane[0];
        ph.eps = nm.eps; ph.n = (int)nm.n; ph.act = cc_act_q8_0(lz->act[act_sel], nm.n); ph.norm_ahead = !written(nm.w);
        P.phase(ph);
        *xbuf = nm.x;
        for (size_t t = i; t < i + nm.len; t++) q[t].done = true;
        return nm.len;
    }

    // ---- pattern: 1-3 MATVECs on the same activation through the streaming kernel (+ optional epilogues) ------------------------------
    // `act_sel` >= 0: scratch already holds quantize(x) ; < 0: emit a plain quantise first.
    size_t try_stream(size_t i, cc_buf* xbuf, int act_sel) {
        if (!streams(i, xbuf)) return 0;
        const LOp& m0 = q[i];
        const int wt = m0.a.buf->dtype; const int64_t k = m0.a.shape[1];
        const GroupMatch g = match_group(i, xbuf, wt, k);
        size_t n = g.n, used = g.used;
        // sharded path: column-split matvec -> allreduce [-> + residual]  /  row-split classifier -> allgather (comm.cu)
        int xchg = 0; float* xdst = nullptr; const float* xres = nullptr;
        if (g.epilogue == 0 && is(i + 1, L_ALLREDUCE) && q[i + 1].a.buf == m0.out && q[i + 1].i0 == m0.a.shape[0]) {
            n = 1; xchg = 1; used = 2; xdst = (float*)m0.out->base;
            if (is(i + 2, L_ADD) && q[i + 2].a.buf == m0.out && view_len(&q[i + 2].b) == m0.a.shape[0] && covers(q[i + 2], m0.a.shape[0]) &&
                q[i + 2].b.buf->dtype == CC_F32 && view_contiguous(&q[i + 2].b)) {
                xres = (const float*)q[i + 2].b.buf->plane[0];
                used = 3;
            }
        } else if (g.epilogue == 0 && is(i + 1, L_ALLGATHER) && q[i + 1].b.buf == m0.out && q[i + 1].i0 == m0.a.shape[0]) {
            n = 1; xchg = 2; used = 2; xdst = (float*)q[i + 1].a.buf->plane[0];
        }
        void* act = lz->act[act_sel >= 0 ? act_sel : 1];
        if (act_sel < 0) {                     // plain quantise of x (matmul_vec.rs:37-40)
            MkPhase qz = new_phase(MK_NORMQ);
            qz.x = (float*)m0.b.buf->plane[0]; qz.n = (int)k; qz.act = cc_act_q8_0(act, k);
            P.phase(qz);
        }
        MkPhase ph = new_phase(MK_MATVEC);
        ph.wtype = wt;
        StreamArgs& A = ph.mv;
        A.k = (int)k; A.epilogue = xchg ? 3 : g.epilogue; A.act = act;
        ph.xgpu = xchg != 0;
        for (int t = 0; t < 3; t++) A.residual[t] = g.residual[t] ? (const float*)g.residual[t]->plane[0] : nullptr;
        A.mats.n = (int)n;
        for (size_t t = 0; t < n; t++) {
            A.mats.qs[t] = q[i + t].a.buf->plane[0];
            A.mats.d[t] = (const uint16_t*)q[i + t].a.buf->plane[1];
            A.mats.out[t] = (float*)q[i + t].out->base;
            A.mats.m[t] = (int)q[i + t].a.shape[0];
        }
        P.phase(ph);
        if (xchg) {
            const int64_t mrows = m0.a.shape[0];
            MkPhase ex = new_phase(xchg == 1 ? MK_REDUCE : MK_GATHER);
            ex.red_n = (int)mrows; ex.red_dst = xdst; ex.red_res = xres;
            if (xchg == 2) ex.x = A.mats.out[0];      // the row to gather, for launch_phase (the persistent kernels read the exchange slots)
            P.phase(ex);
            if (!cc_comm_dev(dev) || cc_comm_is_nccl(dev)) P.mega_ok = false;      // NCCL baseline: graph of kernels + NCCL nodes (lazy mode 1)
            if ((((mrows + dev->sm_count - 1) / dev->sm_count + 3) & ~(int64_t)3) > 512) P.mega_ok = false;   // one CTA's row block must fit the exchange stage (mega_phases.cuh MK_XSTAGE_ROWS)
        }
        for (size_t t = i; t < i + used; t++) q[t].done = true;
        return used;
    }

    // ---- pattern: rope q,k (llama or neox) + kv append + attention (llama2.rs:252-256, 541-590), n_batch == 1 -----------------------------------------------
    size_t try_attention(size_t i, cc_buf** obuf, bool* quantized) {
        if (!(is(i, L_ROPE) && is(i + 1, L_ROPE) && is(i + 2, L_CONCAT) && is(i + 3, L_CONCAT) && is(i + 4, L_CONTIGUOUS) && is(i + 5, L_SCALE) &&
              is(i + 6, L_BMM) && is(i + 7, L_SOFTMAX) && is(i + 8, L_BMM))) return 0;
        const LOp &rq = q[i], &rk = q[i + 1], &ck = q[i + 2], &cv = q[i + 3], &ct = q[i + 4], &sc = q[i + 5], &b1 = q[i + 6], &sm = q[i + 7], &b2 = q[i + 8];
        if (rq.a.ndim != 3 || rk.a.ndim != 3 || rq.a.shape[0] != 1 || rk.a.shape[0] != 1) return 0;
        const int64_t n_heads = rq.a.shape[1], hd = rq.a.shape[2], n_kv = rk.a.shape[1];
        const int mode = (int)rq.f;
        if (rk.a.shape[2] != hd || (mode != CC_ROPE_LLAMA && mode != CC_ROPE_NEOX) || (int)rk.f != mode || rq.i0 != rk.i0 || rq.rows[0] != rk.rows[0]) return 0;
        if (hd > 256 || n_heads % n_kv) return 0;
        *quantized = hd % 32 == 0;
        cc_buf *qb = rq.a.buf, *kb = rk.a.buf, *kc = ck.a.buf, *vc = cv.a.buf, *vb = cv.b.buf;
        if (ck.b.buf != kb || ck.i0 != 1 || cv.i0 != 1 || ck.a.ndim != 3 || cv.a.ndim != 3) return 0;
        if (ck.a.shape[0] != n_kv || ck.a.shape[2] != hd || ck.a.strides[2] != 1 || ck.a.strides[1] != hd) return 0;
        if (cv.a.shape[0] != n_kv || cv.a.shape[2] != hd || cv.a.strides[2] != 1 || cv.a.strides[1] != hd || cv.a.strides[0] != ck.a.strides[0]) return 0;
        if (ck.a.shape[1] != cv.a.shape[1] || kc->dtype != vc->dtype) return 0;
        const int64_t kv_len = ck.a.shape[1], seq_stride = ck.a.strides[0];
        // rhs of the concats: [n_kv, 1, hd] views of the raw k / v rows
        if (ck.b.ndim != 3 || ck.b.shape[0] != n_kv || ck.b.shape[1] != 1 || ck.b.shape[2] != hd || ck.b.strides[0] != hd || ck.b.strides[2] != 1) return 0;
        if (cv.b.ndim != 3 || cv.b.shape[0] != n_kv || cv.b.shape[1] != 1 || cv.b.shape[2] != hd || cv.b.strides[0] != hd || cv.b.strides[2] != 1) return 0;
        if (vb->dtype != CC_F32 || kb->dtype != CC_F32 || qb->dtype != CC_F32) return 0;
        if (ct.a.buf != qb || sc.a.buf != ct.out || b1.a.buf != ct.out || b1.b.buf != kc || sm.a.buf != b1.out || b2.a.buf != b1.out || b2.b.buf != vc) return 0;
        if (b1.b.shape[2] != kv_len + 1 || b1.b.strides[1] != 1 || b2.b.shape[1] != kv_len + 1 || b2.b.strides[2] != 1) return 0;
        if (kv_len + 1 > seq_stride / hd) return 0;
        // a cache longer than the single-pass kernel's score row (50 808 positions at head_dim 128): the ops run as their eager kernels
        if (!cc_attn_decode_fits(hd, seq_stride / hd)) return 0;
        // intermediates must not be observable afterwards
        if (!dead_after(ct.out, i + 9) || !dead_after(b1.out, i + 9) || !dead_after(qb, i + 9) || !dead_after(kb, i + 9) || !dead_after(vb, i + 9)) return 0;
        const int64_t pos = rq.i0, rope_dim = rq.rows[0];
        if (rope_dim > hd || rope_dim % 2) return 0;
        // RoPE table: host libm, identical calls to the reference and the eager kernel (cc_rope_table); shared by all layers of this flush
        if (rope_off == (size_t)-1 || rope_pos != pos || rope_hd != hd || this->rope_dim != rope_dim || rope_mode != mode) {
            std::vector<float> tab((size_t)rope_dim);
            const int pairs = (int)rope_dim / 2;
            cc_rope_table(mode, pos, hd, pairs, tab.data(), tab.data() + pairs);
            rope_off = P.dyn_put(tab.data(), tab.size() * 4);
            rope_pos = pos; rope_hd = (int)hd; this->rope_dim = (int)rope_dim; rope_mode = mode;
        }
        const int64_t dynv[2] = {pos, kv_len};
        MkPhase ph = new_phase(MK_ATTN);
        AttnArgs& A = ph.at;
        A.q = (const float*)qb->plane[0]; A.k = (const float*)kb->plane[0]; A.v = (const float*)vb->plane[0];
        A.kcache = kc->plane[0]; A.vcache = vc->plane[0];
        A.out = (float*)b2.out->base;
        if (*quantized && is(i + 9, L_MATVEC) && !cc_stream_supported(q[i + 9].a.buf->dtype, q[i + 9].a.shape[1])) *quantized = false;   // K-quant wo quantises (Q8_K) itself
        A.act_scratch = *quantized ? lz->act[1] : nullptr;
        A.n_heads = (int)n_heads; A.n_kv = (int)n_kv; A.hd = (int)hd; A.rope_dim = (int)rope_dim;
        A.rope_neox = mode == CC_ROPE_NEOX;
        A.max_len = (int)(seq_stride / hd); A.kv_f16 = kc->dtype == CC_F16;
        A.seq_stride = seq_stride; A.scale = sc.f;
        // the most CTAs per head the score scratch allows; the persistent kernel's split is chosen with its grid (choose_mega)
        A.split = (size_t)n_heads * (size_t)(A.max_len + 1) * 4 <= lz->scores_cap ? AT_SPLIT_MAX : 1;
        ph.dyn_off = P.dyn_put(dynv, sizeof(dynv)); ph.rope_off = rope_off; ph.act = cc_act_q8_0(lz->act[1], n_heads * hd);
        P.phase(ph);
        *obuf = b2.out;
        for (size_t t = i; t < i + 9; t++) q[t].done = true;
        return 9;
    }

    // ---- pattern: embedding / row pick: COPY_ROWS with the row indices in dyn ---------------------------------------------------------------------
    size_t try_copy_rows(size_t i) {
        if (!is(i, L_COPY_ROWS)) return 0;
        const LOp& op = q[i];
        const int64_t cols = op.a.shape[op.a.ndim - 1];
        const int slot = (int)op.i2 - 1;                     // >= 0: the single row index lives in a device slot (cc_copy_rows_from_slot)
        MkPhase ph = new_phase(MK_ROWS);
        ph.planes = cc_deq_planes(op.b.buf, cols); ph.src_dtype = op.b.buf->dtype;
        ph.dst = op.a.buf->plane[0]; ph.dst_dtype = op.a.buf->dtype; ph.n_rows = slot >= 0 ? 1 : (int)op.rows.size(); ph.cols = cols;
        if (slot >= 0) ph.rows_dev = (const long long*)(dev->slots + slot);
        else ph.dyn_off = P.dyn_put(op.rows.data(), op.rows.size() * 8);
        P.phase(ph);
        q[i].done = true;
        return 1;
    }

    // ---- pattern: greedy sampling on the device (cc_argmax_to_slot): the history index travels in dyn ------------------------------------------------
    size_t try_argmax(size_t i) {
        if (!is(i, L_ARGMAX)) return 0;
        const LOp& op = q[i];
        const int64_t hidx = op.i1;
        MkPhase ph = new_phase(MK_ARGMAX);
        ph.x = (float*)op.a.buf->plane[0]; ph.n = (int)view_len(&op.a); ph.dyn_off = P.dyn_put(&hidx, 8);
        ph.slot_dev = (long long*)(dev->slots + op.i0); ph.hist_dev = (long long*)dev->history;
        P.phase(ph);
        q[i].done = true;
        return 1;
    }

    // ---- pattern: temperature + top-p sampling (cc_sample_to_slot): seed, coin index, temperature, topp and the history index travel
    // in dyn, so one graph serves every step and every setting -------------------------------------------------------------------------
    size_t try_sample(size_t i) {
        if (!is(i, L_SAMPLE)) return 0;
        const LOp& op = q[i];
        const SampleDyn a = cc_sample_dyn(op);
        MkPhase ph = new_phase(MK_SAMPLE);
        ph.x = (float*)op.a.buf->plane[0]; ph.n = (int)view_len(&op.a); ph.dyn_off = P.dyn_put(&a, sizeof(a));
        ph.slot_dev = (long long*)(dev->slots + op.i0); ph.hist_dev = (long long*)dev->history;
        ph.dst = dev->sample_scratch;                    // sized for this queue before fusing (cc_lazy_flush)
        P.phase(ph);
        q[i].done = true;
        return 1;
    }

    // ---- pattern: K-quant matvecs (generic MATVEC phase of the megakernel) ----------------------------------------------------------------
    //   [[DUP] RMS_NORM MUL]  MATVEC{1..3, same K-quant type, same f32 row x, b = 1}  [SILU MUL | ADD]
    // In the CUDA-graph mode (lazy = 1) these ops keep running as their eager kernels, in order (eager steps); for the megakernel
    // the whole group is ONE phase: fused prologue (norm + Q8_K quantisation of x) + T::row_dot rows + epilogue -- the same
    // arithmetic as the eager kernels, so the two modes agree bit for bit.
    size_t try_generic(size_t i) {
        const NormMatch nm = match_norm(i);
        const size_t j = i + nm.len;           // a DUP or RMS_NORM that is not a whole norm prefix leaves j on an op that is no MATVEC
        if (!is(j, L_MATVEC)) return 0;
        const LOp& m0 = q[j];
        const int wt = m0.a.buf->dtype; const int64_t k = m0.a.shape[1];
        if (!cc_mega_generic_supported(wt, k)) return 0;
        cc_buf* xb = nm.len ? nm.x : m0.b.buf;
        if (m0.b.buf != xb || xb->dtype != CC_F32 || view_len(&m0.b) != k || !view_contiguous(&m0.b) || (m0.b.ndim == 2 && m0.b.shape[0] != 1) || m0.b.ndim > 2) return 0;
        GroupMatch g = match_group(j, xb, wt, k);
        // the generic phase never writes a normalised row back (below), so a residual that is x itself would read the wrong row;
        // the residual add then runs as its own op, with or without a norm.  Its epilogue adds one vector to one matrix: the bias adds
        // of a q/k/v group run as their own ops too (and keep the table out of the persistent kernels)
        if (g.epilogue == 1 && (g.residual[0] == xb || g.n > 1)) { const size_t n = g.n; g = GroupMatch(); g.n = g.used = n; }
        if (is(j + g.used, L_ALLREDUCE) || is(j + g.used, L_ALLGATHER)) return 0;      // sharded K-quant models run in the CUDA-graph mode
        const size_t end = j + g.used;
        // the normalised row is overwritten in place by the eager ops; the fused prologue never materialises it: nobody else may read it
        if (nm.len && !dead_after(xb, end)) return 0;
        for (size_t t = 0; t < g.n; t++) if (q[j + t].a.buf->cols != k) return 0;
        MkPhase ph = new_phase(MK_MATVEC);
        ph.wtype = wt; ph.act_type = CC_Q8_K;
        StreamArgs& A = ph.mv;
        A.k = (int)k; A.epilogue = g.epilogue; A.residual[0] = g.residual[0] ? (const float*)g.residual[0]->plane[0] : nullptr;
        A.mats.n = (int)g.n;
        for (size_t t = 0; t < g.n; t++) {
            const cc_buf* w = q[j + t].a.buf;
            A.mats.qs[t] = w->plane[0]; A.mats.d[t] = (const uint16_t*)w->plane[1]; A.mats.p2[t] = w->plane[2]; A.mats.p3[t] = w->plane[3];
            A.mats.out[t] = (float*)q[j + t].out->base;
            A.mats.m[t] = (int)q[j + t].a.shape[0];
        }
        ph.x = (float*)xb->plane[0]; ph.orig = nm.orig ? (float*)nm.orig->base : nullptr; ph.eps = nm.eps; ph.n = (int)k;
        ph.norm_w = nm.len ? (const float*)nm.w->plane[0] : nullptr;
        ph.norm_ahead = nm.len && !written(nm.w);
        // the CUDA-graph mode runs the group's ops as their eager kernels, in order; the phase covers them in the persistent kernel
        P.phase(ph, false);
        for (size_t t = i; t < end; t++) eager(t);
        return end - i;
    }

    // megakernel only: phases[at] = NORMQ (not write-back) directly followed by its single MATVEC consumer -> one MATVEC
    // phase with a fused prologue (saves a grid barrier per merge; see mega_ring.cu phase_matvec_ring)
    void merge_prologue(size_t at) {
        // [at] NORMQ, [at + 1] MATVEC, optionally [at + 2] the REDUCE / GATHER half of the matvec's exchange (sharded path)
        const bool tail = at + 3 == P.phases.size() && (P.phases[at + 2].type == MK_REDUCE || P.phases[at + 2].type == MK_GATHER);
        if (at + 2 != P.phases.size() && !tail) return;
        MkPhase& nq = P.phases[at];
        MkPhase& mv = P.phases[at + 1];
        if (nq.type != MK_NORMQ || mv.type != MK_MATVEC || nq.write_back || nq.n != mv.mv.k) return;
        mv.x = nq.x; mv.orig = nq.orig; mv.norm_w = nq.norm_w; mv.eps = nq.eps; mv.n = nq.n; mv.norm_ahead = nq.norm_ahead;
        P.phases.erase(P.phases.begin() + at);
        // sharded path: the REDUCE phase that produced x folds into the same prologue (x itself is dead after this group:
        // !write_back), so an exchange costs no phase of its own
        if (at >= 1 && P.phases[at - 1].type == MK_REDUCE && P.phases[at - 1].red_dst == P.phases[at].x && P.phases[at - 1].red_n == P.phases[at].n) {
            MkPhase& m2 = P.phases[at];
            m2.red_n = P.phases[at - 1].red_n; m2.red_res = P.phases[at - 1].red_res;
            P.phases.erase(P.phases.begin() + (at - 1));
        }
    }

    void run() {
        index_uses();
        size_t i = 0;
        while (i < q.size()) {
            if (q[i].done) { i++; continue; }
            size_t used;
            cc_buf* xb = nullptr;
            if ((used = try_copy_rows(i))) { i += used; continue; }
            if ((used = try_argmax(i))) { i += used; continue; }
            if ((used = try_sample(i))) { i += used; continue; }
            if ((used = try_generic(i))) { i += used; continue; }
            if ((used = try_normq(i, 0, &xb))) {
                i += used;
                // every following group of matvecs on the normalised x reuses scratch 0
                const size_t ph0 = P.phases.size();
                int groups = 0;
                while (size_t u2 = try_stream(i, xb, 0)) { i += u2; groups++; }
                if (groups == 1) merge_prologue(ph0 - 1);
                continue;
            }
            bool quantized = false;
            if ((used = try_attention(i, &xb, &quantized))) {
                i += used;
                if (size_t u2 = try_stream(i, xb, quantized ? 1 : -1)) i += u2;      // wo consumes the (quantised) attention output
                continue;
            }
            if (is(i, L_MATVEC) && q[i].b.buf->dtype == CC_F32 && (q[i].b.ndim == 1 || q[i].b.shape[0] == 1)) {
                const size_t ph0 = P.phases.size();
                if ((used = try_stream(i, q[i].b.buf, -1))) { i += used; merge_prologue(ph0); continue; }
            }
            fallback(i);
            i++;
        }
    }
};

// The persistent kernel that runs a phase table and its launch geometry (MEGA_NONE: the CUDA-graph mode); on success the phases get
// their links to the next MATVEC phase and to the next fused-norm weights the kernel may stage early.  A table with a streaming (Q8_0 /
// Q4_0) MATVEC phase runs mega_ring.cu when every such phase can be fed by bulk copies and the ring gets enough slots beside the working
// area; any other table runs mega.cu when its working area fits.  At head_dim 128 the attention phase's working area (the score row +
// its chunk buffers) decides this at long contexts; past 50 808 positions the fuser leaves attention to the per-op kernels.
static MegaLaunch choose_mega(const cc_device* dev, bool mega_ok, std::vector<MkPhase>& phs) {
    MegaLaunch L;
    if (!dev->mega || !mega_ok || phs.empty()) return L;
    bool stream = false, ring_ok = true;
    int n_sample = 0;
    for (auto& ph : phs) {
        if (ph.type == MK_MATVEC) (ph.act_type == CC_Q8_K ? L.generic : stream) = true;
        if (!cc_mega_ring_phase_ok(ph)) ring_ok = false;
        n_sample += ph.type == MK_SAMPLE;
        if ((ph.type == MK_ATTN && ph.at.rope_neox) || (ph.type == MK_MATVEC && ph.mv.epilogue == 1 && ph.mv.mats.n > 1)) L.qwen2 = true;
    }
    // the megakernel runs ONE SAMPLE phase, after its phase loop (mega.cu): a table with more than one, or with anything queued
    // behind the sampler (several tokens submitted before one flush), runs in the CUDA-graph mode
    L.sample = n_sample > 0;
    if (n_sample > 1 || (n_sample == 1 && phs.back().type != MK_SAMPLE)) return L;
    if (L.qwen2 && !stream) return L;          // qwen2 phases are in the ring kernel only (mega_ring.cu QWEN2)
    for (auto& ph : phs) {
        L.smem = std::max(L.smem, stream ? cc_mega_ring_smem_for_phase(ph) : cc_mega_smem_for_phase(ph));
        if (ph.type == MK_MATVEC && ph.x && ph.norm_w) L.wstage = std::max(L.wstage, (size_t)ph.n * 4);
        if (stream && ph.type == MK_MATVEC && ph.act_type != CC_Q8_K) L.slot_bytes = std::max(L.slot_bytes, ph.wtype == CC_Q8_0 ? 4352 : 2304);
        if (stream && ph.type == MK_ATTN) L.at_ch = cc_mega_ring_at_ch(ph);
    }
    if (stream ? !ring_ok || !(L.nslots = cc_mega_ring_slots(L)) : L.smem + L.wstage + 4096 > 227 * 1024) return L;
    L.variant = stream ? MEGA_RING : MEGA_REGISTER;
    for (auto& ph : phs) if (ph.type == MK_ATTN) ph.at.split = cc_attn_split(ph.at, dev->sm_count);      // both kernels: one CTA per SM
    L.scores = dev->lz->scores;
    int nxt = -1, nxn = -1;
    for (int t = (int)phs.size() - 1; t >= 0; t--) {
        MkPhase& ph = phs[t];
        ph.next_matvec = nxt;
        ph.next_norm_w = nxn >= 0 && phs[nxn].norm_ahead ? phs[nxn].norm_w : nullptr;
        ph.next_norm_n = ph.next_norm_w ? phs[nxn].n : 0;
        if (ph.type == MK_MATVEC) nxt = t;
        if (ph.type == MK_MATVEC && ph.x && ph.norm_w) nxn = t;
    }
    return L;
}

// scratch the queued ops need, at its final size before anything is captured: graphs bake the pointers in
static int size_scratch(cc_device* dev, LazyState* lz) {
    // quantised activations (largest k in the queue)
    int64_t max_k = 0;
    for (auto& op : lz->q) if (op.kind == L_MATVEC) max_k = std::max<int64_t>(max_k, std::max<int64_t>(op.a.shape[1], 0));
    // the fused attention quantises its OUTPUT row (n_heads * head_dim = the PV product's a_batch * n) into act[1]; QK^T products
    // ([heads, 1, kv_len + 1]) are never quantised, so the scratch does not grow with the context
    for (auto& op : lz->q) if (op.kind == L_BMM && op.b.ndim == 3 && op.b.strides[2] == 1) max_k = std::max<int64_t>(max_k, op.a.shape[0] * op.b.shape[2]);
    size_t need = cc_act_bytes(CC_Q8_0, (max_k + 255) / 256 * 256) + 256;
    int rc = CC_OK;
    if (need > lz->act_cap) {
        cudaStreamSynchronize(dev->stream);
        graph_cache_clear(lz);                       // cached graphs hold the old scratch pointers
        for (int i = 0; i < 2; i++) { if (lz->act[i]) cudaFree(lz->act[i]); lz->act[i] = nullptr; }
        size_t cap = (size_t)1 << 20; while (cap < need) cap <<= 1;      // generous from the start: growing means cudaFree (context-wide wait)
        for (int i = 0; i < 2; i++) if (cudaMalloc(&lz->act[i], cap) != cudaSuccess) return cc_fail(dev, CC_ERR_CUDA, "lazy: scratch alloc failed");
        lz->act_cap = cap;
    }
    // the megakernels' attention score rows [heads][max_len + 1] (MegaLaunch::scores), from the QK^T products: the K^T view of the cache
    // has row stride hd and batch stride max_len * hd
    size_t score_need = 0;
    for (auto& op : lz->q)
        if (op.kind == L_BMM && op.b.ndim == 3 && op.b.strides[1] == 1 && op.b.strides[2] > 0 && op.b.strides[0] > 0)
            score_need = std::max(score_need, (size_t)op.a.shape[0] * (size_t)(op.b.strides[0] / op.b.strides[2] + 1) * 4);
    if (score_need > lz->scores_cap) {
        cudaStreamSynchronize(dev->stream);
        graph_cache_clear(lz);                       // cached persistent-kernel graphs hold the old score rows
        cudaFree(lz->scores); lz->scores = nullptr; lz->scores_cap = 0;
        size_t cap = (size_t)1 << 20; while (cap < score_need) cap <<= 1;
        if (cudaMalloc(&lz->scores, cap) != cudaSuccess) return cc_fail(dev, CC_ERR_CUDA, "lazy: score scratch alloc failed");
        lz->scores_cap = cap;
    }
    // eager matvec steps (cc_run_op) use dev->act_scratch; growing it drops the cached graphs (cc_ensure_act_scratch)
    for (auto& op : lz->q) if (op.kind == L_MATVEC) {
        int at = cc_partner_type(op.a.buf->dtype);
        int64_t bb = op.b.ndim == 1 ? 1 : op.b.shape[0];
        if (at != CC_F32 && (rc = cc_ensure_act_scratch(dev, cc_act_bytes(at, bb * op.a.shape[1])))) return rc;
    }
    for (auto& op : lz->q) if (op.kind == L_SAMPLE && (rc = cc_ensure_sample_scratch(dev, view_len(&op.a)))) return rc;
    return CC_OK;
}

// per-token values: pinned slot -> device block, as an ordinary stream copy in front of the launches / the graph
static int upload_dyn(cc_device* dev, LazyState* lz, const Plan& P) {
    if (P.dyn.size() > lz->dyn_cap) return cc_fail(dev, CC_ERR_UNSUPPORTED, "lazy: dynamic argument block too large");
    if (P.dyn.empty()) return CC_OK;
    int rc = CC_OK; const int s = lz->dyn_slot;
    lz->dyn_slot = (s + 1) % LZ_DYN_SLOTS;
    cudaEventSynchronize(lz->dyn_ev[s]);          // the copy that last read this slot (LZ_DYN_SLOTS flushes ago) is long done
    memcpy(lz->dyn_host[s], P.dyn.data(), P.dyn.size());
    if (cudaMemcpyAsync(lz->dyn_dev, lz->dyn_host[s], P.dyn.size(), cudaMemcpyHostToDevice, dev->stream) != cudaSuccess) rc = cc_fail(dev, CC_ERR_CUDA, "lazy: dyn upload failed");
    cudaEventRecord(lz->dyn_ev[s], dev->stream);
    return rc;
}

static int run_steps(cc_device* dev, const Plan& P, const std::vector<LOp>& q, const uint8_t* dyn_dev) {
    for (const Plan::Step& st : P.steps)
        if (int r = st.eager ? cc_run_op(dev, q[st.at]) : launch_phase(dev, P.emitted[st.at], dyn_dev)) return r;
    return CC_OK;
}

// the cached graph of this signature, or end() after making room for a new one
using GraphCache = std::unordered_map<uint64_t, GraphEntry>;
static GraphCache::iterator find_graph(cc_device* dev, LazyState* lz, uint64_t key, const std::vector<uint64_t>& sig) {
    auto it = lz->cache.find(key);
    if (it != lz->cache.end() && it->second.sig != sig) {          // 64-bit key collision: never replay the other plan's graph
        lz->collisions++;
        cudaStreamSynchronize(dev->stream);
        graph_entry_free(it->second);
        lz->cache.erase(it);
        it = lz->cache.end();
    }
    if (it == lz->cache.end() && lz->cache.size() >= LZ_MAX_GRAPHS) {   // LRU bound: evict the entry replayed longest ago
        auto victim = lz->cache.begin();
        for (auto c = lz->cache.begin(); c != lz->cache.end(); ++c) if (c->second.last_use < victim->second.last_use) victim = c;
        cudaStreamSynchronize(dev->stream);          // its last launch may still be running
        graph_entry_free(victim->second);
        lz->cache.erase(victim);
        lz->evictions++;
    }
    return it;
}

// capture the plan -- one persistent kernel, or its steps -- into a new cache entry
static int capture(cc_device* dev, LazyState* lz, Plan& P, uint64_t key, GraphCache::iterator* out) {
    int rc = CC_OK; lz->captures++;
    uint64_t l0 = dev->launches; cudaGraph_t graph = nullptr; GraphEntry ge;
    const MegaLaunch L = choose_mega(dev, P.mega_ok, P.phases);
    if (L.variant != MEGA_NONE) {       // phase table lives in device memory for the lifetime of the graph
        if (cudaMalloc(&ge.phases_dev, P.phases.size() * sizeof(MkPhase)) != cudaSuccess ||
            cudaMemcpy(ge.phases_dev, P.phases.data(), P.phases.size() * sizeof(MkPhase), cudaMemcpyHostToDevice) != cudaSuccess)
            rc = cc_fail(dev, CC_ERR_CUDA, "lazy: phase table upload failed");
    }
    cudaError_t e = rc ? cudaSuccess : cudaStreamBeginCapture(dev->stream, cudaStreamCaptureModeRelaxed);
    if (!rc && e != cudaSuccess) rc = cc_fail(dev, CC_ERR_CUDA, "lazy: begin capture: %s", cudaGetErrorString(e));
    if (!rc) {
        if (L.variant != MEGA_NONE && lz->prof_dev && P.phases.size() < 4000) { lz->prof_types.clear(); for (auto& ph : P.phases) lz->prof_types.push_back(ph.type * 16 + (ph.type == MK_MATVEC ? ph.mv.mats.n + 4 * ph.mv.epilogue + 1024 * (ph.mv.k >> 10) : 0)); }
        unsigned long long* prof = P.phases.size() < 4000 ? lz->prof_dev : nullptr;
        if (L.variant == MEGA_NONE) rc = run_steps(dev, P, lz->q, lz->dyn_dev);
        else if (L.variant == MEGA_RING) rc = cc_launch_mega_ring(dev, ge.phases_dev, (int)P.phases.size(), lz->dyn_dev, lz->bar_dev, L, prof, cc_comm_dev(dev));
        else rc = cc_launch_mega(dev, ge.phases_dev, (int)P.phases.size(), lz->dyn_dev, lz->bar_dev, L, prof);
        e = cudaStreamEndCapture(dev->stream, &graph);
        if (!rc && e != cudaSuccess) rc = cc_fail(dev, CC_ERR_CUDA, "lazy: end capture: %s", cudaGetErrorString(e));
    }
    if (!rc) {
        e = cudaGraphInstantiate(&ge.exec, graph, 0);
        if (e != cudaSuccess) rc = cc_fail(dev, CC_ERR_CUDA, "lazy: graph instantiate: %s", cudaGetErrorString(e));
    }
    if (graph) cudaGraphDestroy(graph);
    if (!rc) {
        ge.mega_variant = L.variant;
        ge.dyn_bytes = P.dyn.size();
        ge.sig = P.sig;
        ge.launches = dev->launches - l0;
        dev->launches = l0;            // counted when the graph is launched
        *out = lz->cache.emplace(key, ge).first;
    }
    return rc;
}

int cc_lazy_flush(cc_device* dev) {
    LazyState* lz = dev->lz;
    if (!lz || lz->q.empty()) return CC_OK;
    lz->flushes++;
    int rc = size_scratch(dev, lz); if (rc) return rc;
    auto t_f0 = std::chrono::steady_clock::now();
    Plan P;
    Fuser F{dev, lz, lz->q, P};
    F.run();
    auto t_f1 = std::chrono::steady_clock::now();
    lz->ns_fuse += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(t_f1 - t_f0).count();
    if (P.dyn.size() > lz->dyn_cap) P.cacheable = false;
    rc = upload_dyn(dev, lz, P);
    if (rc) {
    } else if (!P.cacheable) {
        lz->uncached++;
        rc = run_steps(dev, P, lz->q, lz->dyn_dev);
    } else {
        P.S(P.dyn.size());
        uint64_t key = hash_sig(P.sig);
        auto it = find_graph(dev, lz, key, P.sig);
        if (it != lz->cache.end()) lz->graph_hits++;
        else rc = capture(dev, lz, P, key, &it);
        if (!rc) {
            it->second.last_use = lz->flushes;
            if (it->second.mega_variant != MEGA_NONE) lz->mega_variant = it->second.mega_variant;
            cudaError_t e = cudaGraphLaunch(it->second.exec, dev->stream);
            if (e != cudaSuccess) rc = cc_fail(dev, CC_ERR_CUDA, "lazy: graph launch: %s", cudaGetErrorString(e));
            else dev->launches += it->second.launches;
        }
    }
    lz->ns_submit += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t_f1).count();
    // drop the queue's references, last op first (keeps pool pointer assignment identical from token to token)
    std::vector<LOp> old;
    old.swap(lz->q);
    lz->qrefs.clear();
    for (size_t t = old.size(); t-- > 0;) {
        LOp& op = old[t];
        if (op.out) cc_tensor_release(op.out);
        if (op.b.buf) cc_tensor_release(op.b.buf);
        if (op.a.buf) cc_tensor_release(op.a.buf);
    }
    return rc;
}

// Called after a stream synchronize.  A persistent kernel that gave up on a barrier (MkSpin in mega.cu) has raised the host-mapped
// error word: report it, and reset the barrier words (their monotonic counters are inconsistent after a drained launch).
int cc_check_async_error(cc_device* dev) {
    if (!dev || !dev->err_host) return CC_OK;
    const unsigned code = *(volatile unsigned*)dev->err_host;
    if (!code) return CC_OK;
    *(volatile unsigned*)dev->err_host = 0u;
    if (dev->err_dev) cudaMemset(dev->err_dev, 0, 256);
    if (dev->lz && dev->lz->bar_dev) cudaMemset(dev->lz->bar_dev, 0, 4096);
    return cc_fail(dev, CC_ERR_CUDA, "%s timeout (%s): the grid was not co-resident or a peer GPU stopped responding",
                   code == 3u ? "exchange kernel" : "megakernel barrier", code == 1u ? "grid barrier" : code == 4u ? "weight ring" : "cross-GPU handshake");
}

// developer profiling: per-phase start timestamps (ns) of the last megakernel run + phase type codes
extern "C" CC_API int cc_lazy_mega_profile(cc_device* dev, unsigned long long* ts, int* types, int cap, int* n_out) {
    if (!dev || !dev->lz || !dev->lz->prof_dev || !ts || !types || !n_out) return CC_ERR_ARG;
    cudaStreamSynchronize(dev->stream);
    int n = (int)dev->lz->prof_types.size();
    if ((n + 1) * MK_PROF_SLOTS > cap) return CC_ERR_ARG;
    if (cudaMemcpy(ts, dev->lz->prof_dev, (size_t)(n + 1) * MK_PROF_SLOTS * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return CC_ERR_CUDA;
    for (int i = 0; i < n; i++) types[i] = dev->lz->prof_types[i];
    *n_out = n;
    return CC_OK;
}

extern "C" CC_API int cc_lazy_mega_variant(cc_device* dev) { return dev && dev->lz ? dev->lz->mega_variant : 0; }

extern "C" CC_API int cc_lazy_stats(cc_device* dev, uint64_t* out4) {
    if (!dev || !dev->lz || !out4) return CC_ERR_ARG;
    out4[0] = dev->lz->flushes; out4[1] = dev->lz->graph_hits; out4[2] = dev->lz->captures; out4[3] = dev->lz->uncached;
    out4[4] = dev->lz->ns_record; out4[5] = dev->lz->ns_fuse; out4[6] = dev->lz->ns_submit; out4[7] = dev->lz->n_ops;
    return CC_OK;
}
