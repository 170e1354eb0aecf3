/*
 * crabml_cuda.h -- C ABI of the H100-native CUDA backend for crabml's quantized tensor-op path.
 *
 * This is the drop-in boundary: one entry point per method of the reference's `Tensor` trait
 * (crabml-core/src/tensor/api.rs:11-79).  A Rust `crabml-cuda` crate binds these with
 * `extern "C"` (see INTEGRATION.md); in this repo they are driven by the C++ host mirror
 * (crabml_b200/csrc/host/) and by Python ctypes in tests/ and bench.py.
 *
 * Conventions
 *  - Plain pointers and sizes only.  No torch types, no C++ types, nothing throws.
 *  - Every function returns a status: 0 = ok, non-zero = error.  CC_ERR_TENSOR maps to the
 *    reference's ErrorKind::TensorError (crabml-core/src/error.rs:24-25); the message is
 *    available from cc_last_error().  Internal invariant violations that are `assert!`s in the
 *    reference (e.g. primitives/matmul_vec.rs:17-19) are reported as CC_ERR_TENSOR too.
 *  - A tensor on the Rust side is {Arc<buffer>, TensorStrider, device, name}
 *    (cf. crabml-wgpu/src/wgpu_tensor.rs:20-28).  The strider stays host-side: metadata-only
 *    trait methods (reshape / transpose / with_strider / resize / shape / strider,
 *    api.rs:28-44) never cross this ABI.  Ops take a `cc_view` = buffer handle + the strider's
 *    shape and strides (in elements).
 *  - All work is enqueued on the device's single stream; only cc_tensor_export_f32,
 *    cc_debug_tensor_tap and cc_device_synchronize block (api.rs:52; llama2.rs:209).
 *  - There is NO CPU fallback: without a CUDA device cc_device_create fails.
 */
#ifndef CRABML_CUDA_H
#define CRABML_CUDA_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define CC_API __attribute__((visibility("default")))
#else
#define CC_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define CC_OK 0
#define CC_ERR_TENSOR 1   /* ErrorKind::TensorError */
#define CC_ERR_CUDA 2     /* a CUDA runtime call failed (text in cc_last_error) */
#define CC_ERR_ARG 3      /* NULL / malformed argument */
#define CC_ERR_UNSUPPORTED 4

/* GGMLType ids, crabml-core/src/gguf.rs:86-108 */
enum cc_ggml_type {
    CC_F32 = 0, CC_F16 = 1, CC_Q4_0 = 2, CC_Q4_1 = 3, CC_Q5_0 = 6, CC_Q5_1 = 7,
    CC_Q8_0 = 8, CC_Q8_1 = 9, CC_Q2_K = 10, CC_Q3_K = 11, CC_Q4_K = 12,
    CC_Q5_K = 13, CC_Q6_K = 14, CC_Q8_K = 15
};

/* RopeMode, api.rs:5-9 */
enum cc_rope_mode { CC_ROPE_LLAMA = 0, CC_ROPE_NEOX = 1 };

#define CC_MAX_DIMS 4

typedef struct cc_device cc_device;   /* T::DeviceRef */
typedef struct cc_buf cc_buf;         /* refcounted device storage (the Arc<Buffer> of a tensor) */

/* TensorStrider (crabml-core/src/tensor/strider.rs:5-9) passed by value with the buffer. */
typedef struct cc_view {
    cc_buf* buf;
    int32_t ndim;
    int64_t shape[CC_MAX_DIMS];
    int64_t strides[CC_MAX_DIMS];   /* in elements */
} cc_view;

/* CpuTensorDeviceOptions / WgpuTensorDeviceOptions analogue (cpu_device.rs:13-48). */
typedef struct cc_device_options {
    int32_t device_ordinal;        /* CUDA device index */
    int32_t debug_named_tensors;   /* with_name() snapshots tensors to host (cpu_tensor.rs:232-241) */
    int32_t lazy;                  /* 0 = eager: one launch per trait call; 1 = record + fuse + CUDA-graph replay;
                                      2 = as 1, and a fused token runs as ONE persistent kernel (mega_ring.cu, mega.cu) */
    int32_t exact_order;           /* 1 = verification mode: every reduction in the reference's scalar order,
                                      bit-identical to the scalar CPU path (slow; see csrc/exact.cu) */
    uint64_t pool_bytes;           /* activation pool size hint, 0 = default */
} cc_device_options;

/* ---- device ---------------------------------------------------------------------------- */
CC_API int cc_device_create(const cc_device_options* opts, cc_device** out);
CC_API void cc_device_destroy(cc_device* dev);
CC_API const char* cc_last_error(cc_device* dev);          /* NULL dev: last creation error */
CC_API int cc_device_synchronize(cc_device* dev);
/* lazy mode: execute everything queued so far (asynchronously); a no-op in eager mode.  The runner calls it at the
 * end of forward() when the logits are not exported. */
CC_API int cc_device_flush(cc_device* dev);
/* lazy mode statistics, 8 values: {flushes, graph replays, graph captures, uncached (eager) flushes,
 * host ns spent recording, fusing, submitting, ops recorded} */
CC_API int cc_lazy_stats(cc_device* dev, uint64_t* out8);
/* developer hook: per-phase floor of the megakernel (descriptor fetch + grid barrier), microseconds */
CC_API int cc_test_mega_barrier_floor(cc_device* dev, int n, float* us_per_phase);
/* developer profiling (CRABML_MEGA_PROF=1): phase start timestamps of the last megakernel run */
CC_API int cc_lazy_mega_profile(cc_device* dev, unsigned long long* ts, int* types, int cap, int* n_out);
/* which persistent kernel ran the last megakernel flush: 0 none yet, 1 mega_kernel (tables without a Q8_0 / Q4_0 matvec, mega.cu),
 * 2 mega_ring_kernel (Q8_0 / Q4_0 weights through the TMA-fed shared-memory ring, mega_ring.cu) */
CC_API int cc_lazy_mega_variant(cc_device* dev);
/* counters: kernels launched by this library since creation (bench.py "gpu_launches") */
CC_API uint64_t cc_device_launch_count(cc_device* dev);
/* persistent kernels of this device use at most n SMs (test / co-tenancy hook: two devices of one process side by side on one GPU).
 * In lazy mode a change waits for the queued work and drops the graphs captured at the old grid. */
CC_API int cc_device_set_sm_limit(cc_device* dev, int32_t n);
/* raw cudaStream_t of the device, for event timing by the caller */
CC_API void* cc_device_stream(cc_device* dev);

/* ---- storage: Tensor::from_cpu / alloc / Clone / Drop (api.rs:14-23) -------------------- */
/* from_cpu: copies `nbytes` host bytes of GGUF-layout data (row-major rows of quant blocks,
 * model.rs:462-477).  `shape` is [rows, cols] (or 1-D).  Quantized types are repacked once
 * into the device layout documented in DESIGN.md (same algorithmic bytes). */
CC_API int cc_tensor_from_cpu(cc_device* dev, const void* bytes, size_t nbytes, const int64_t* shape,
                       int32_t ndim, int32_t ggml_type, cc_buf** out);
/* alloc: F32 zero-filled, or F16 (cpu_tensor.rs:138-165); other dtypes -> CC_ERR_TENSOR */
CC_API int cc_tensor_alloc(cc_device* dev, const int64_t* shape, int32_t ndim, int32_t ggml_type, cc_buf** out);
CC_API void cc_tensor_retain(cc_buf* buf);
CC_API void cc_tensor_release(cc_buf* buf);
CC_API int32_t cc_tensor_dtype(const cc_buf* buf);          /* api.rs:30 */
CC_API int64_t cc_tensor_capacity(const cc_buf* buf);       /* elements of backing storage (resize bound, cpu_tensor.rs:180) */

/* ---- data movement ------------------------------------------------------------------------ */
CC_API int cc_tensor_dup(cc_device* dev, const cc_view* src, cc_buf** out);                 /* api.rs:55 */
CC_API int cc_tensor_export_f32(cc_device* dev, const cc_view* src, float* dst, size_t n);  /* api.rs:52 */
CC_API int cc_copy_rows_from(cc_device* dev, const cc_view* dst, const cc_view* src,
                      const int64_t* rows, int32_t n_rows);                          /* api.rs:50 */
/* concatenate writes rhs at offset shape[axis] along `axis` using self's strides
 * (concatenate.rs:12-77); the caller then bumps its strider's shape[axis]. */
CC_API int cc_concatenate(cc_device* dev, const cc_view* self, const cc_view* rhs, int32_t axis);  /* api.rs:46 */
CC_API int cc_contiguous(cc_device* dev, const cc_view* src, cc_buf** out);                 /* api.rs:40 */

/* ---- in-place elementwise ops (api.rs:57-74) ---------------------------------------------- */
CC_API int cc_rope_inplace(cc_device* dev, const cc_view* x, int32_t mode, int64_t pos, int64_t rope_dims);
CC_API int cc_rms_norm_inplace(cc_device* dev, const cc_view* x, float eps);
CC_API int cc_softmax_inplace(cc_device* dev, const cc_view* x, int32_t axis);
CC_API int cc_silu_inplace(cc_device* dev, const cc_view* x);
CC_API int cc_gelu_inplace(cc_device* dev, const cc_view* x);
CC_API int cc_mul_inplace(cc_device* dev, const cc_view* x, const cc_view* rhs);
CC_API int cc_add_inplace(cc_device* dev, const cc_view* x, const cc_view* rhs);
CC_API int cc_scale_inplace(cc_device* dev, const cc_view* x, float rhs);

/* ---- the hot path (api.rs:76-78) ------------------------------------------------------------ */
/* matmul_vec: W (m,k) any dtype, x F32 (k,) or (b,k) -> new F32 (m,) / (b,m).
 * The activation is quantized on the fly to W's partner type (buf/api.rs:142-159). */
CC_API int cc_matmul_vec(cc_device* dev, const cc_view* w, const cc_view* x, cc_buf** out);
CC_API int cc_batch_matmul(cc_device* dev, const cc_view* a, const cc_view* b, cc_buf** out);

/* ---- debug tap: with_name / dump_debug_tensor (cpu_tensor.rs:232-241, cpu_device.rs:96-98) -- */
CC_API int cc_debug_tensor_tap(cc_device* dev, const char* name, const cc_view* x);
/* returns element count via *n; copies min(*n_in, count) floats when dst != NULL */
CC_API int cc_dump_debug_tensor(cc_device* dev, const char* name, float* dst, size_t* n);

/* ---- greedy decoding without a host round trip per token (extension; not part of the reference's trait) ----------------
 * The sampled token id stays on the device: cc_argmax_to_slot (sampler.rs:109-116, the LAST maximum) writes it to one of 16 slots
 * and, when hist_index >= 0, to a device-side history; cc_copy_rows_from_slot is copy_rows_from with the single row index taken
 * from a slot (the next token's embedding lookup).  The host can therefore submit token t+1 before token t has finished;
 * cc_read_history synchronises and returns the ids.  cc_tensor_export_f32_async enqueues an export without waiting (dst should
 * be pinned: cc_host_alloc) -- it is complete after the next synchronising call. */
CC_API int cc_argmax_to_slot(cc_device* dev, const cc_view* x, int32_t slot, int64_t hist_index);
CC_API int cc_copy_rows_from_slot(cc_device* dev, const cc_view* dst, const cc_view* src, int32_t slot);
/* Llama2Sampler::sample (sampler.rs:27-107) on the device, into a slot like cc_argmax_to_slot: softmax of x / temperature, then the
 * reference's top-p walk over the probabilities sorted ASCENDING (quirk B21: topp < 1 keeps the low-probability tail).  The coin is
 * (splitmix64(seed ^ splitmix64(coin_index)) >> 40) * 2^-24, so one seed reproduces one run.  temperature == 0 is cc_argmax_to_slot.
 * Where the reference panics (no probability reaches the cutoff) the argmax is taken.  x is not modified.  A NaN or negative
 * temperature, a NaN topp, and a non-f32 or non-contiguous x are CC_ERR_TENSOR. */
CC_API int cc_sample_to_slot(cc_device* dev, const cc_view* x, float temperature, float topp, uint64_t seed, int64_t coin_index,
                             int32_t slot, int64_t hist_index);
CC_API int cc_slot_set(cc_device* dev, int32_t slot, int64_t value);
CC_API int cc_read_history(cc_device* dev, int64_t first, int64_t count, int64_t* out);
CC_API int cc_tensor_export_f32_async(cc_device* dev, const cc_view* src, float* dst, size_t n);
CC_API int cc_host_alloc(cc_device* dev, size_t bytes, void** out);
CC_API void cc_host_free(cc_device* dev, void* p);

/* ---- test / bench hooks (not part of the trait) ---------------------------------------------- */
/* quantize an F32 vector exactly as matmul_vec does internally and return the reference-layout
 * activation blocks (Q8_0 / Q8_1 / Q8_K bytes) to the host: parity tests of a3-a5 (SURVEY §8a). */
CC_API int cc_test_quantize_activation(cc_device* dev, const cc_view* x, int32_t act_type, void* dst, size_t nbytes);
/* ---- sharded decode (SURVEY 8e): the exchange step ---------------------------------------------------------
 * The reference is single-device; its unit of parallelism is the output row (matmul_vec.rs:41-76 splits rows over
 * the thread pool).  Across GPUs the same split leaves two exchanges per layer: a sum of [dim] partials after the
 * column-split `wo` and `ffn_down`, and a gather of the row-split classifier's logit slices.
 * One process per GPU.  cc_comm_create allocates this rank's exchange window and returns its 64-byte CUDA IPC handle;
 * the caller distributes the handles (torch.distributed / any side channel) and passes all of them to
 * cc_comm_connect.  cc_comm_init_nccl switches the transport to NCCL (baseline; id from cc_comm_nccl_unique_id on rank 0). */
CC_API int cc_comm_create(cc_device* dev, int32_t rank, int32_t world, uint8_t* handle_out_64);
CC_API int cc_comm_connect(cc_device* dev, const uint8_t* handles_world_x_64);
/* ranks that are devices of ONE process, one per GPU (peers[r] = the cc_device of rank r): windows are wired directly, no IPC handles.
 * NOTE: ranks of one process share a CUDA context per GPU; put them on DIFFERENT GPUs -- on the same GPU a context-wide wait of one rank
 * (first-use allocation, module load, cudaFree) can deadlock against the other rank's spinning exchange. */
CC_API int cc_comm_connect_local(cc_device* dev, cc_device* const* peers);
CC_API int cc_comm_nccl_unique_id(cc_device* dev, uint8_t* id_out_128);
CC_API int cc_comm_init_nccl(cc_device* dev, const uint8_t* id_128);
CC_API int32_t cc_comm_rank(cc_device* dev);
CC_API int32_t cc_comm_world_size(cc_device* dev);
/* x (contiguous f32, <= 32768 elements, multiple of 4) = sum over ranks of x, same bits on every rank */
CC_API int cc_all_reduce_sum_inplace(cc_device* dev, const cc_view* x);
/* dst[r * n + i] = src of rank r [i]; src: n contiguous f32 (same n on every rank), dst: world * n */
CC_API int cc_all_gather(cc_device* dev, const cc_view* dst, const cc_view* src);
/* synthetic shard: rows [row0, row0+nrows) x columns [col0, col0+ncols) of the tensor cc_tensor_synth would make */
CC_API int cc_tensor_synth_slice(cc_device* dev, const int64_t* shape, int32_t ndim, int32_t ggml_type, uint64_t seed,
                                 uint64_t tensor_id, float scale, int64_t row0, int64_t nrows, int64_t col0,
                                 int64_t ncols, cc_buf** out);

/* synthetic weights generated on device in the device layout (SURVEY §8d config 3): counter-based
 * RNG, identical bytes to tests/synth.py's CPU generator for the same (seed, tensor_id). */
CC_API int cc_tensor_synth(cc_device* dev, const int64_t* shape, int32_t ndim, int32_t ggml_type,
                    uint64_t seed, uint64_t tensor_id, float scale, cc_buf** out);
/* CUDA-event timer on the device's stream (bench.py): begin records an event; end records, synchronises
 * and returns the elapsed milliseconds between the two */
CC_API int cc_bench_timer_begin(cc_device* dev);
CC_API int cc_bench_timer_end(cc_device* dev, float* ms);
/* copy a quantized tensor back in GGUF block layout (inverse of the load-time repack) */
CC_API int cc_test_export_blocks(cc_device* dev, const cc_buf* buf, void* dst, size_t nbytes);

#ifdef __cplusplus
}
#endif
#endif /* CRABML_CUDA_H */
