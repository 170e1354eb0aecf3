// common.cuh -- internal declarations shared by the CUDA translation units of libcrabml_cuda.
// H100 (sm_90a) only.  No CPU fallback anywhere in this library.
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/crabml_cuda.h"

#define QK_K 256

// ------------------------------------------------------------------------------------------
// Device-side storage layouts (DESIGN.md "Data layout in HBM").  GGUF stores a weight matrix
// as rows of AoS blocks whose size is only 2-byte aligned (34 / 18 / 22 / 210 ... bytes).
// from_cpu repacks each matrix ONCE into planes so that every hot-loop load is a 16-byte,
// fully coalesced LDG.128; total bytes are unchanged (the f16 scales move to their own plane).
//
//   type   plane0                         plane1                 plane2            plane3
//   Q8_0   qs  int8  [rows][k] (*)        d   f16 [rows][S]        (*) inside each group of 32 blocks the 16 B
//                                                                  first halves precede the second halves
//   Q4_0   qs  u8    [rows][k/32][16]     d   f16 [rows][S]        S = CC_D_STRIDE(k/32): rows padded to 16 bytes
//   Q4_1   qs  u8    [rows][k/32][16]     d,m f16x2
//   Q5_0   qs  u8    [rows][k/32][16]     d   f16                qh u32 [rows][k/32]
//   Q5_1   qs  u8    [rows][k/32][16]     d,m f16x2              qh u32
//   Q2_K   qs  u8    [rows][k/256][64]    scales u8 [..][16]     d,dmin f16x2
//   Q3_K   qs  u8    [rows][k/256][64]    hmask u8 [..][32]      scales u8 [..][12]   d f16
//   Q4_K   AoS 144 B blocks (already 16 B aligned: 16 B header + 128 B qs)
//   Q5_K   AoS 176 B blocks (16 B header + 32 B qh + 128 B qs)
//   Q6_K   ql  u8    [rows][k/256][128]   qh u8 [..][64]         scales i8 [..][16]   d f16
//   Q8_K   qs  int8  [rows][k]            d   f32 [rows][k/256]
// ------------------------------------------------------------------------------------------
// Q8_0 / Q4_0: the rows of the f16 scale plane are padded to a multiple of 8 blocks (16 bytes), so that any row segment is a legal bulk
// copy (TMA: 16-byte aligned address, 16-byte multiple size) for every k -- the column-split shards of the sharded path included
// (k = 11008 / N: 172, 86, 43 blocks per row).  The padding is never read by arithmetic.
#define CC_D_STRIDE(nb) ((((nb) + 7) / 8) * 8)
#define CC_HAS_PADDED_D(t) ((t) == CC_Q8_0 || (t) == CC_Q4_0)
#define CC_MAX_PLANES 4
#define CC_N_SLOTS 16
#define CC_HISTORY_CAP 65536

struct cc_device;

struct cc_buf {
    cc_device* dev = nullptr;
    std::atomic<int> refs{1};
    int32_t dtype = CC_F32;
    int64_t nelems = 0;        // capacity in elements
    void* base = nullptr;      // allocation base (plane[0] for quantized types)
    size_t bytes = 0;          // allocation size
    bool pooled = false;       // came from the activation pool (size class = bytes)
    int64_t rows = 0, cols = 0;  // quantized matrices
    uint8_t* plane[CC_MAX_PLANES] = {nullptr, nullptr, nullptr, nullptr};
    uint8_t* raw = nullptr;    // GGUF-layout copy, kept only on exact_order devices (exact.cu)
    void* f16 = nullptr;       // dequantised f16 [rows][cols] tile source of the prefill GEMM, built at first use (prefill_gemm.cu)
};

// On-device activation formats: what buf/api.rs:195-228 `quantize` produces, as SoA.
struct ActQ8_0 {          // partner of Q8_0 / Q4_0 / Q5_0 (buf_q8_0.rs:87-134)
    int8_t* qs;           // [b][k]
    float* d;             // [b][k/32]   = f32(f16(d))
    int32_t* isum;        // [b][k/32]   sum of the block's quants (for the -8 / -16 offsets)
};
struct ActQ8_1 {          // partner of Q4_1 / Q5_1 (buf_q8_1.rs:90-129)
    int8_t* qs;           // [b][k]
    __half2* ds;          // [b][k/32]   (d, s) as stored f16 values
};
struct ActQ8_K {          // partner of all K-quants (buf_q8_k.rs:84-131)
    int8_t* qs;           // [b][k]
    float* d;             // [b][k/256]
    int16_t* bsums;       // [b][k/16]
};

// ---- comm.cu: exchange step of the sharded decode path ---------------------------------------------------
#define CC_COMM_MAX_RANKS 8
#define CC_COMM_MAX_ELEMS 32768          // f32 elements per exchange per rank (a [dim] row, or a vocab/N logit slice)
struct CommDev {                         // by-value kernel argument: where every rank's window lives in THIS rank's address space
    int rank, world;
    float* data[CC_COMM_MAX_RANKS];      // data[p] + ((parity * 8 + src_rank) * CC_COMM_MAX_ELEMS)
    unsigned* flag[CC_COMM_MAX_RANKS];   // flag[p][src_rank * 32]
    unsigned* seq;                       // local: number of finished exchanges
};
struct cc_comm;

struct cc_device {
    int ordinal = 0;
    cc_comm* comm = nullptr;
    cudaStream_t stream = nullptr;
    bool debug_named_tensors = false;
    bool lazy = false;
    bool exact = false;       // cc_device_options.exact_order
    bool pdl = true;          // launch fused-path kernels with programmatic dependent launch
    bool mega = false;        // lazy mode 2: one persistent kernel per token (mega.cu)
    struct LazyState* lz = nullptr;   // non-null in lazy mode (lazy.cu)
    std::string last_error;
    uint64_t launches = 0;
    int sm_count = 132;          // H100 SXM; replaced by the device's count at creation

    // f16 LUTs (cpu_device.rs:108-124), computed on the host with libm and uploaded
    uint16_t* exp_lut = nullptr;
    uint16_t* gelu_lut = nullptr;

    // activation scratch for matmul_vec (grown on demand; stream-ordered reuse)
    void* act_scratch = nullptr;
    size_t act_scratch_bytes = 0;

    // stream-ordered size-class pool for activations
    std::mutex mu;
    std::unordered_map<size_t, std::set<uintptr_t>> free_lists;   // per size class, ordered: allocation takes the LOWEST free address
    size_t pool_live_bytes = 0;

    void* dev_idx = nullptr;      // device copy of row indices
    size_t dev_idx_bytes = 0;

    cudaEvent_t ev_begin = nullptr, ev_end = nullptr;    // cc_bench_timer_*
    // greedy decode without host round trips (capi.cu cc_argmax_to_slot / cc_copy_rows_from_slot): token-id slots and the history
    // of sampled ids, both in device memory
    int64_t* slots = nullptr;         // [CC_N_SLOTS]
    int64_t* history = nullptr;       // [CC_HISTORY_CAP]
    void* sample_scratch = nullptr;   // temperature / top-p sampler (sample_dev.cuh): probabilities and the sort's key arrays
    size_t sample_scratch_bytes = 0;
    unsigned* err_host = nullptr;     // host-mapped word a kernel raises when one of its bounded spins times out (mega.cu, comm.cu)
    unsigned* err_dev = nullptr;      // device copy polled by the other spinners of the same GPU

    // weight upload (Tensor::from_cpu): double-buffered pinned staging so that reading the caller's bytes (page-faulting a GGUF mmap)
    // overlaps the DMA of the previous chunk and the repack kernels of the previous tensor
    void* up_pinned[2] = {nullptr, nullptr};
    cudaEvent_t up_ev[2] = {nullptr, nullptr};

    // debug tap
    std::map<std::string, std::vector<float>> debug_tensors;
};

// Every extern "C" entry point that touches CUDA makes its device current for the duration of the call and restores the caller's
// afterwards: a cc_device may be driven from any host thread, and one process may own several of them (one per GPU).
struct CcDeviceGuard {
    int prev = -1;
    explicit CcDeviceGuard(const cc_device* dev) {
        if (!dev) return;
        int cur = -1;
        if (cudaGetDevice(&cur) == cudaSuccess && cur != dev->ordinal) { prev = cur; cudaSetDevice(dev->ordinal); }
    }
    ~CcDeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
    CcDeviceGuard(const CcDeviceGuard&) = delete;
    CcDeviceGuard& operator=(const CcDeviceGuard&) = delete;
};
#define CC_CAT2(a, b) a##b
#define CC_CAT(a, b) CC_CAT2(a, b)
#define CC_ENTER(dev) CcDeviceGuard CC_CAT(cc_guard_, __LINE__)(dev)

// ---- error plumbing ------------------------------------------------------------------------
int cc_fail(cc_device* dev, int code, const char* fmt, ...);
#define CC_CUDA(dev, call)                                                                  \
    do {                                                                                    \
        cudaError_t _e = (call);                                                            \
        if (_e != cudaSuccess)                                                              \
            return cc_fail((dev), CC_ERR_CUDA, "%s failed: %s (%s:%d)", #call,              \
                           cudaGetErrorString(_e), __FILE__, __LINE__);                     \
    } while (0)
#define CC_REQUIRE(dev, cond, ...)                                                          \
    do {                                                                                    \
        if (!(cond)) return cc_fail((dev), CC_ERR_TENSOR, __VA_ARGS__);                     \
    } while (0)
#define CC_LAUNCH_CHECK(dev)                                                                \
    do {                                                                                    \
        (dev)->launches++;                                                                  \
        cudaError_t _e = cudaPeekAtLastError();                                             \
        if (_e != cudaSuccess)                                                              \
            return cc_fail((dev), CC_ERR_CUDA, "kernel launch failed: %s (%s:%d)",          \
                           cudaGetErrorString(_e), __FILE__, __LINE__);                     \
    } while (0)

// launch with programmatic dependent launch (pdl: cc_device::pdl): the kernel may start while the previous one in the stream drains
template <class... KArgs, class... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// counter-based generator of the synthetic weights (repack.cu) and of the sampler's coin (sample_dev.cuh)
__host__ __device__ inline uint64_t cc_splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// ---- type facts ------------------------------------------------------------------------------
int cc_block_elems(int t);
size_t cc_block_bytes(int t);          // GGUF block size
int cc_partner_type(int t);            // buf/api.rs:142-159
bool cc_is_quant(int t);

// ---- device.cu ---------------------------------------------------------------------------------
int cc_pool_alloc(cc_device* dev, size_t bytes, void** out, size_t* cls);
void cc_pool_free(cc_device* dev, void* p, size_t cls);
int cc_new_activation(cc_device* dev, int64_t nelems, int dtype, bool zero, cc_buf** out);
int cc_ensure_act_scratch(cc_device* dev, size_t bytes);
int cc_ensure_dev_idx(cc_device* dev, size_t bytes);

// ---- repack.cu -----------------------------------------------------------------------------------
size_t cc_device_layout_bytes(int t, int64_t rows, int64_t cols);
void cc_assign_planes(cc_buf* b);
int cc_launch_repack(cc_device* dev, const uint8_t* gguf_dev, cc_buf* dst);           // GGUF AoS -> planes
int cc_launch_unrepack(cc_device* dev, const cc_buf* src, uint8_t* gguf_dev);          // planes -> GGUF AoS
struct DeqPlanes { const uint8_t* p[CC_MAX_PLANES]; int64_t cols; };
// the planes of b as the dequantising kernels read them; cols is the row length of an unquantised (f32 / f16) b
inline DeqPlanes cc_deq_planes(const cc_buf* b, int64_t cols) {
    DeqPlanes P;
    for (int i = 0; i < CC_MAX_PLANES; i++) P.p[i] = b->plane[i];
    P.cols = b->cols > 0 ? b->cols : cols;
    return P;
}
int cc_launch_dequant_rows(cc_device* dev, const DeqPlanes& src, int src_dtype, const int64_t* rows_dev, int n_rows,
                           int64_t cols, void* dst, int dst_dtype);                    // copy_rows_from
int cc_launch_synth(cc_device* dev, uint8_t* gguf_dev, int t, int64_t nblocks, uint64_t seed, uint64_t tid, float scale);

// ---- quantize.cu ---------------------------------------------------------------------------------
size_t cc_act_bytes(int act_type, int64_t n);
ActQ8_0 cc_act_q8_0(void* scratch, int64_t n);
ActQ8_1 cc_act_q8_1(void* scratch, int64_t n);
ActQ8_K cc_act_q8_k(void* scratch, int64_t n);
int cc_launch_quantize(cc_device* dev, const float* x, int64_t n, int act_type, void* scratch);
int cc_launch_act_to_blocks(cc_device* dev, const void* scratch, int64_t n, int act_type, uint8_t* blocks_dev);

// ---- matvec.cu -----------------------------------------------------------------------------------
int cc_launch_matvec(cc_device* dev, const cc_buf* w, const void* act_scratch, const float* x_f32,
                     float* out, int64_t m, int64_t k, int64_t b);

// ---- prefill_gemm.cu: batched matmul_vec on the tensor cores (TMA + wgmma, f16 operand tiles, f32 register accumulator) ----
bool cc_prefill_supported(int wtype, int64_t m, int64_t k, int64_t b);
int cc_launch_prefill_matmul(cc_device* dev, const cc_buf* w, const void* act_q8_k, const float* x_f32, float* out, int64_t m, int64_t k, int64_t b);
void cc_prefill_release(cc_device* dev);

// ---- ops.cu --------------------------------------------------------------------------------------
int cc_launch_rms_norm(cc_device* dev, float* x, int64_t rows, int64_t cols, float eps);
int cc_launch_softmax(cc_device* dev, float* x, int64_t rows, int64_t cols);
int cc_launch_silu(cc_device* dev, float* x, int64_t n);
int cc_launch_gelu(cc_device* dev, float* x, int64_t n);
int cc_launch_binary(cc_device* dev, float* x, int64_t n, const float* y, int64_t ny, int op);   // 0 add, 1 mul
int cc_launch_scale(cc_device* dev, float* x, int64_t n, float s);
int cc_launch_argmax(cc_device* dev, const float* x, int64_t n, int64_t* slot, int64_t* hist, const int64_t* hist_index_dev, int64_t hist_index);
int cc_ensure_slots(cc_device* dev);
// ---- sample.cu: temperature + top-p sampling into a slot (sample_dev.cuh) ----
struct SampleDyn;
int cc_ensure_sample_scratch(cc_device* dev, int64_t n);
int cc_launch_sample(cc_device* dev, const float* x, int64_t n, const SampleDyn* args, const SampleDyn* args_dev, int64_t* slot, int64_t* hist);
int cc_launch_strided_copy(cc_device* dev, const void* src, int src_dtype, const int64_t* sshape,
                           const int64_t* sstrides, void* dst, int dst_dtype, const int64_t* dstrides,
                           int64_t dst_offset, int ndim);
int cc_launch_batch_matmul(cc_device* dev, const float* a, const void* b, int b_dtype, float* c,
                           int64_t a_batch, int64_t b_batch, int64_t m, int64_t k, int64_t n,
                           int64_t sb0, int64_t sb1, int64_t sb2);

// ---- matvec_stream.cu --------------------------------------------------------------------------------
struct StreamMats {           // up to 3 weight matrices sharing one activation (wq,wk,wv / gate,up)
    const uint8_t* qs[3];     // plane 0 (quants)
    const uint16_t* d[3];     // plane 1 (Q8_0 / Q4_0: f16 scales)
    const uint8_t* p2[3];     // planes 2 and 3 of the K-quant layouts (generic MATVEC phase of the megakernel)
    const uint8_t* p3[3];
    float* out[3];
    int m[3];
    int n;
};
struct StreamArgs {
    StreamMats mats;
    const void* act;         // ActQ8_0 scratch (quantize.cu layout) of k elements
    int k;
    int epilogue;            // 0 store, 1 add residual[mat] (llama2.rs residual adds, qwen2 q/k/v biases), 2 silu(mat0 row) * (mat1 row),
                             // 3 store into every rank's exchange slot (megakernel)
    const float* residual[3];   // epilogue 1: out[mat][r] = dot + residual[mat][r], one f32 vector per matrix
};
struct AttnArgs {            // fused decode attention (fused.cu)
    const float *q, *k, *v;  // raw matvec outputs [n_heads*hd], [n_kv*hd], [n_kv*hd]
    void *kcache, *vcache;   // [n_kv, seq_max, hd] F32 or F16
    float* out;              // [n_heads*hd]
    void* act_scratch;       // Q8_0 quantisation of out
    int n_heads, n_kv, hd, rope_dim, max_len, kv_f16;
    int64_t seq_stride;
    float scale;
    int split;               // megakernels: CTAs per head (lazy.cu: the most the score scratch allows, then cc_attn_split); the fused kernel ignores it
    int rope_neox;           // RoPE pairs: 0 llama (2j, 2j+1), 1 neox (j, j + hd/2), j < rope_dim/2 (rope.rs:47-80)
};
// MkPhase is 512 bytes: the persistent kernels keep ten copies of it in shared memory, so its size moves the weight ring's fit
// Attention phase of the megakernels split over `split` CTAs per head: CTA c scores its own range of the head's positions and
// accumulates PV for its hd / split output dimensions; the score rows meet in MegaLaunch::scores ([n_heads][max_len + 1] f32).  Head h's CTAs count their arrivals in
// word AT_ARRIVE_WORD + 8 h of the grid-barrier block (4096 bytes), AT_SPLIT_MAX per phase whatever the split.
#define AT_SPLIT_MAX 4
#define AT_SPLIT_MIN_KV 320       // below this many cached positions the exchange costs more than the split saves: one CTA per head
#define AT_ARRIVE_WORD 128
#define AT_SPLIT_MAX_HEADS ((1024 - AT_ARRIVE_WORD) / 8)
int cc_attn_split(const AttnArgs& a, int grid);
// megakernel phase descriptor (mega.cu); built by lazy.cu
enum { MK_NORMQ = 0, MK_MATVEC = 1, MK_ATTN = 2, MK_ROWS = 3, MK_REDUCE = 4, MK_GATHER = 5, MK_ARGMAX = 6, MK_SAMPLE = 7 };
struct MkPhase {
    int type, wtype, write_back, next_matvec;  // next_matvec: index of the next MATVEC phase (mega.cu stages its norm weights early), -1 if none
    int xgpu, red_n; const float* next_norm_w; float* red_dst; const float* red_res;   // cross-GPU barrier after this phase ; norm weights of the next
                                        // fused-norm MATVEC phase after this one (mega_ring.cu stages them one phase ahead), null if none ; REDUCE/GATHER phase operands
    // NORMQ (and the output quantisation of ATTN)
    float* x; float* orig; const float* norm_w; float eps; int n; ActQ8_0 act;
    int act_type, next_norm_n;          // MATVEC: CC_Q8_0 (streaming phases) or CC_Q8_K (generic phases: K-quant weights) ; length of next_norm_w
    StreamArgs mv;                      // MATVEC
    AttnArgs at;                        // ATTN
    unsigned long long dyn_off, rope_off;   // ATTN {pos, kv_len} / ROWS row list ; RoPE table
    DeqPlanes planes; int src_dtype, dst_dtype, n_rows, pad; long long cols; void* dst;   // ROWS
    const long long* rows_dev;          // ROWS: row indices in device memory (a token slot) instead of the dyn block ; ARGMAX: x = input, n = length,
    long long* slot_dev; long long* hist_dev;   //   slot_dev / hist_dev = where the index goes (hist index at dyn_off, < 0: none)
                                        // SAMPLE: as ARGMAX, with a SampleDyn at dyn_off and the sampler scratch at dst
    int norm_ahead, pad2;               // fused norm: no op of the table writes norm_w (model weights), so it may be staged before earlier phases end
};
#define MK_PROF_SLOTS 10     // developer profiling: u64 stamps per phase (CTA 0 / thread 0): 0 start, 1 activation ready, 2 rows done, 3 arrived, 4 x staged, 5 rms known,
                             // 6-7 ring consumer counters, 8 norm weights available, 9 ring occupancy as the barrier in front of the phase opened
                             // (mega_ring.cu); read by tools/mega_profile*.py
size_t cc_mega_smem_for_phase(const MkPhase& ph);      // working area, without the norm-weight staging area on top of it
const CommDev* cc_comm_dev(cc_device* dev);
bool cc_comm_is_nccl(cc_device* dev);
int cc_comm_world(cc_device* dev);
void cc_comm_destroy(cc_device* dev);
int cc_launch_all_reduce(cc_device* dev, float* x, int64_t n, const float* residual);
int cc_launch_all_gather(cc_device* dev, const float* src, int64_t n, float* dst);
extern "C" CC_API int cc_test_mega_barrier_floor(cc_device* dev, int n, float* us_per_phase);
// the persistent kernel that runs a phase table; the values are those of cc_lazy_mega_variant
enum MegaVariant { MEGA_NONE = 0, MEGA_REGISTER = 1, MEGA_RING = 2 };     // CUDA-graph mode ; mega_kernel (mega.cu) ; mega_ring_kernel (mega_ring.cu)
struct MegaLaunch {                 // launch description of one phase table (lazy.cu choose_mega)
    MegaVariant variant = MEGA_NONE;
    size_t smem = 1024, wstage = 0;  // working area (largest phase) ; norm-weight stage on top of it (largest n * 4 of a fused-norm phase)
    int slot_bytes = 0, nslots = 0, at_ch = 64;  // MEGA_RING: weight-ring slot size and count (cc_mega_ring_slots), attention chunk
    bool generic = false, sample = false;        // the instantiation that carries the generic (K-quant) MATVEC phase / the sampler's call
    bool qwen2 = false;                          // ... Neox attention phases and per-matrix epilogue vectors (MEGA_RING only)
    float* scores = nullptr;                     // the attention phase's score rows (AttnArgs::split > 1)
};
int cc_launch_mega(cc_device* dev, const MkPhase* phases_dev, int n_phases, const uint8_t* dyn_dev, unsigned* bar_dev, const MegaLaunch& L,
                   unsigned long long* prof);
bool cc_mega_test_stall();
// mega_ring.cu: the same phase table run by the kernel whose weights arrive through a TMA-fed shared-memory ring
bool cc_mega_ring_phase_ok(const MkPhase& ph);
int cc_mega_ring_at_ch(const MkPhase& ph);
size_t cc_mega_ring_smem_for_phase(const MkPhase& ph);
int cc_mega_ring_slots(const MegaLaunch& L);
int cc_launch_mega_ring(cc_device* dev, const MkPhase* phases_dev, int n_phases, const uint8_t* dyn_dev, unsigned* bar_dev, const MegaLaunch& L,
                        unsigned long long* prof, const CommDev* comm);
int cc_check_async_error(cc_device* dev);     // after a stream synchronize: did a persistent kernel give up on a barrier?
int cc_launch_normq(cc_device* dev, float* x, float* orig, const float* norm_w, float eps, int64_t n, ActQ8_0 act, bool write_back);
int cc_launch_attn_decode(cc_device* dev, const AttnArgs& a, const int64_t* dyn /* {pos, kv_len} */, const float* rope_tab /* cos[pairs], sin[pairs] */);
bool cc_attn_decode_fits(int64_t hd, int64_t max_len);      // can the single-pass attention kernel hold the score row of this cache?
struct LazyState;
LazyState* cc_lazy_create(cc_device* dev);
void cc_lazy_destroy(cc_device* dev);
int cc_lazy_flush(cc_device* dev);
int cc_lazy_invalidate(cc_device* dev);        // drop the cached graphs, reset the grid barrier (no-op without lazy state); stream idle
bool cc_stream_supported(int type, int64_t k);
bool cc_mega_generic_supported(int type, int64_t k);      // K-quant weights: generic MATVEC phase of the megakernel (mega.cu)
int cc_launch_matvec_stream(cc_device* dev, int type, const StreamArgs& A);
int cc_launch_matvec_stream_plain(cc_device* dev, const cc_buf* w, const void* act, float* out, int64_t m, int64_t k);

// ---- exact.cu (exact_order verification mode) -------------------------------------------------------
int cc_launch_matvec_exact(cc_device* dev, int t, const uint8_t* w_gguf, const uint8_t* act_blocks, float* out,
                           int64_t m, int64_t k, int64_t b);
int cc_launch_rms_norm_exact(cc_device* dev, float* x, int64_t rows, int64_t cols, float eps);
int cc_launch_softmax_exact(cc_device* dev, float* x, int64_t rows, int64_t cols);
int cc_launch_rope_exact(cc_device* dev, float* x, int64_t n_batch, int64_t batch_stride, int64_t head_dim, int mode,
                         int64_t pos, int64_t rope_dim);
// the cos / sin of the `pairs` rotation angles of one position, on the host with the reference's libm calls (rope.rs:47-80); read by the
// eager rope kernel and by the fused attention of both lazy modes
void cc_rope_table(int mode, int64_t pos, int64_t head_dim, int pairs, float* cos_out, float* sin_out);
int cc_launch_bmm_kcontig_exact(cc_device* dev, const float* a, const void* b, int b_dtype, float* c, int64_t ab, int64_t bb,
                                int64_t m, int64_t k, int64_t n, int64_t sb0, int64_t sb2);

// one segment (16 super-blocks) of a K-quant weight row in registers, loaded as one batch by T::seg_load (vecdot.cuh) so that the
// generic MATVEC phase keeps the next segment in flight: 8 x 16-byte loads + 4 f16 scales per lane (Q4_K: a = block headers,
// b = quants; Q6_K: a = ql, b = qh, s = d)
struct KSeg { int4 a[4], b[4]; uint16_t s[4]; };

// ---- small device helpers -------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// ---- canonical reduction orders ---------------------------------------------------------------------------------
// Every execution mode (eager ops.cu, fused kernels of the CUDA-graph mode, phases of the megakernel) reduces a row with
// the SAME grouping, so the three modes are bit-identical to each other (tests/test_gpu_runner.py):
//   a CTA of CC_RED_THREADS = 512 threads; thread t accumulates the items t, t + 512, t + 1024, ... in that order
//   (for sums of squares an item is a float4 chunk: ss += x*x + y*y + z*z + w*w, left to right), then the xor-butterfly
//   warp_sum, then the 16 warp sums are added in warp order 0..15 by every thread.
#define CC_RED_THREADS 512
#define CC_RED_WARPS 16
__device__ __forceinline__ float cc_block_sum_512(float v, float* s_red /* [16] */) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.0f;
#pragma unroll
    for (int w = 0; w < CC_RED_WARPS; w++) t += s_red[w];
    __syncthreads();                       // s_red may be reused by the caller
    return t;
}
__device__ __forceinline__ float cc_block_max_512(float v, float* s_red /* [16] */) {
    v = warp_max(v);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = s_red[0];
#pragma unroll
    for (int w = 1; w < CC_RED_WARPS; w++) t = fmaxf(t, s_red[w]);
    __syncthreads();
    return t;
}
__device__ __forceinline__ float cc_sq4(const float4& v) { return v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w; }

// streaming 128-bit load of weight data: read exactly once per token, keep it out of L1
__device__ __forceinline__ int4 ld_stream_16(const void* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ void cc_st_release_sys(unsigned* p, unsigned v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned cc_ld_acquire_sys(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// ---- bounded spins: no wait in this library can hang the GPU -----------------------------------------------------------------
// After CC_SPIN_TIMEOUT_NS without progress (a CTA that never became resident because another tenant holds an SM, a peer GPU that
// died) the waiter raises the error words -- the device copy for the other spinners, the host-mapped copy for
// cc_check_async_error, which reports CC_ERR_CUDA "... timeout" at the next synchronising call -- and the kernel drains.
#define CC_SPIN_CHECK 0x7FFFu                // iterations between two looks at the clock / the error word
#define CC_SPIN_TIMEOUT_NS 4000000000ull     // a healthy barrier or handshake takes microseconds
__device__ __forceinline__ unsigned long long cc_globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
struct CcSpin {
    unsigned it = 0; unsigned long long t0 = 0;
    __device__ __forceinline__ bool expired(unsigned* err_dev, unsigned* err_host, unsigned code) {
        if ((++it & CC_SPIN_CHECK) != 0) return false;
        if (err_dev && *(volatile unsigned*)err_dev) return true;
        const unsigned long long t = cc_globaltimer_ns();
        if (!t0) { t0 = t; return false; }
        if (t - t0 < CC_SPIN_TIMEOUT_NS) return false;
        if (err_dev) atomicExch(err_dev, code);
        if (err_host) { *(volatile unsigned*)err_host = code; __threadfence_system(); }
        return true;
    }
};
__device__ __forceinline__ float h2f_bits(uint16_t h) { return __half2float(__ushort_as_half(h)); }
__device__ __forceinline__ uint16_t f2h_bits(float f) { return __half_as_ushort(__float2half_rn(f)); }
#endif
