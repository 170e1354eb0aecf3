//! Raw bindings of `include/crabml_cuda.h` -- one `extern "C"` item per declaration of the header, in the header's order.
//! Hand-written (no bindgen in the build) and checked mechanically: `tests/test_capi_exports.py` parses this file and the
//! header and compares every function's name, arity and argument / return C types.
#![allow(non_camel_case_types)]

use std::os::raw::c_char;
use std::os::raw::c_int;
use std::os::raw::c_void;

pub const CC_OK: c_int = 0;
/// `ErrorKind::TensorError` (crabml-core/src/error.rs:24-25)
pub const CC_ERR_TENSOR: c_int = 1;
/// a CUDA runtime call failed, or a persistent kernel gave up on a barrier (text in `cc_last_error`)
pub const CC_ERR_CUDA: c_int = 2;
pub const CC_ERR_ARG: c_int = 3;
pub const CC_ERR_UNSUPPORTED: c_int = 4;

pub const CC_ROPE_LLAMA: i32 = 0;
pub const CC_ROPE_NEOX: i32 = 1;

pub const CC_MAX_DIMS: usize = 4;

/// `T::DeviceRef` on the C side
#[repr(C)]
pub struct cc_device {
    _private: [u8; 0],
}

/// refcounted device storage (the `Arc<Buffer>` of a tensor)
#[repr(C)]
pub struct cc_buf {
    _private: [u8; 0],
}

/// `TensorStrider` (crabml-core/src/tensor/strider.rs:5-9) passed by value with the buffer; strides in elements
#[repr(C)]
#[derive(Clone, Copy)]
pub struct cc_view {
    pub buf: *mut cc_buf,
    pub ndim: i32,
    pub shape: [i64; CC_MAX_DIMS],
    pub strides: [i64; CC_MAX_DIMS],
}

#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct cc_device_options {
    pub device_ordinal: i32,
    pub debug_named_tensors: i32,
    pub lazy: i32,
    pub exact_order: i32,
    pub pool_bytes: u64,
}

extern "C" {
    // ---- device ----
    pub fn cc_device_create(opts: *const cc_device_options, out: *mut *mut cc_device) -> c_int;
    pub fn cc_device_destroy(dev: *mut cc_device);
    pub fn cc_last_error(dev: *mut cc_device) -> *const c_char;
    pub fn cc_device_synchronize(dev: *mut cc_device) -> c_int;
    pub fn cc_device_flush(dev: *mut cc_device) -> c_int;
    pub fn cc_lazy_stats(dev: *mut cc_device, out8: *mut u64) -> c_int;
    pub fn cc_test_mega_barrier_floor(dev: *mut cc_device, n: c_int, us_per_phase: *mut f32) -> c_int;
    pub fn cc_lazy_mega_profile(
        dev: *mut cc_device,
        ts: *mut u64,
        types: *mut c_int,
        cap: c_int,
        n_out: *mut c_int,
    ) -> c_int;
    pub fn cc_lazy_mega_variant(dev: *mut cc_device) -> c_int;
    pub fn cc_device_launch_count(dev: *mut cc_device) -> u64;
    pub fn cc_device_set_sm_limit(dev: *mut cc_device, n: i32) -> c_int;
    pub fn cc_device_stream(dev: *mut cc_device) -> *mut c_void;

    // ---- storage: Tensor::from_cpu / alloc / Clone / Drop (api.rs:14-23) ----
    pub fn cc_tensor_from_cpu(
        dev: *mut cc_device,
        bytes: *const c_void,
        nbytes: usize,
        shape: *const i64,
        ndim: i32,
        ggml_type: i32,
        out: *mut *mut cc_buf,
    ) -> c_int;
    pub fn cc_tensor_alloc(
        dev: *mut cc_device,
        shape: *const i64,
        ndim: i32,
        ggml_type: i32,
        out: *mut *mut cc_buf,
    ) -> c_int;
    pub fn cc_tensor_retain(buf: *mut cc_buf);
    pub fn cc_tensor_release(buf: *mut cc_buf);
    pub fn cc_tensor_dtype(buf: *const cc_buf) -> i32;
    pub fn cc_tensor_capacity(buf: *const cc_buf) -> i64;

    // ---- data movement ----
    pub fn cc_tensor_dup(dev: *mut cc_device, src: *const cc_view, out: *mut *mut cc_buf) -> c_int;
    pub fn cc_tensor_export_f32(dev: *mut cc_device, src: *const cc_view, dst: *mut f32, n: usize) -> c_int;
    pub fn cc_copy_rows_from(
        dev: *mut cc_device,
        dst: *const cc_view,
        src: *const cc_view,
        rows: *const i64,
        n_rows: i32,
    ) -> c_int;
    pub fn cc_concatenate(dev: *mut cc_device, this: *const cc_view, rhs: *const cc_view, axis: i32) -> c_int;
    pub fn cc_contiguous(dev: *mut cc_device, src: *const cc_view, out: *mut *mut cc_buf) -> c_int;

    // ---- in-place elementwise ops (api.rs:57-74) ----
    pub fn cc_rope_inplace(dev: *mut cc_device, x: *const cc_view, mode: i32, pos: i64, rope_dims: i64) -> c_int;
    pub fn cc_rms_norm_inplace(dev: *mut cc_device, x: *const cc_view, eps: f32) -> c_int;
    pub fn cc_softmax_inplace(dev: *mut cc_device, x: *const cc_view, axis: i32) -> c_int;
    pub fn cc_silu_inplace(dev: *mut cc_device, x: *const cc_view) -> c_int;
    pub fn cc_gelu_inplace(dev: *mut cc_device, x: *const cc_view) -> c_int;
    pub fn cc_mul_inplace(dev: *mut cc_device, x: *const cc_view, rhs: *const cc_view) -> c_int;
    pub fn cc_add_inplace(dev: *mut cc_device, x: *const cc_view, rhs: *const cc_view) -> c_int;
    pub fn cc_scale_inplace(dev: *mut cc_device, x: *const cc_view, rhs: f32) -> c_int;

    // ---- the hot path (api.rs:76-78) ----
    pub fn cc_matmul_vec(dev: *mut cc_device, w: *const cc_view, x: *const cc_view, out: *mut *mut cc_buf) -> c_int;
    pub fn cc_batch_matmul(dev: *mut cc_device, a: *const cc_view, b: *const cc_view, out: *mut *mut cc_buf) -> c_int;

    // ---- debug tap: with_name / dump_debug_tensor ----
    pub fn cc_debug_tensor_tap(dev: *mut cc_device, name: *const c_char, x: *const cc_view) -> c_int;
    pub fn cc_dump_debug_tensor(dev: *mut cc_device, name: *const c_char, dst: *mut f32, n: *mut usize) -> c_int;

    // ---- greedy decoding without a host round trip per token (extension) ----
    pub fn cc_argmax_to_slot(dev: *mut cc_device, x: *const cc_view, slot: i32, hist_index: i64) -> c_int;
    pub fn cc_copy_rows_from_slot(dev: *mut cc_device, dst: *const cc_view, src: *const cc_view, slot: i32) -> c_int;
    pub fn cc_sample_to_slot(
        dev: *mut cc_device,
        x: *const cc_view,
        temperature: f32,
        topp: f32,
        seed: u64,
        coin_index: i64,
        slot: i32,
        hist_index: i64,
    ) -> c_int;
    pub fn cc_slot_set(dev: *mut cc_device, slot: i32, value: i64) -> c_int;
    pub fn cc_read_history(dev: *mut cc_device, first: i64, count: i64, out: *mut i64) -> c_int;
    pub fn cc_tensor_export_f32_async(dev: *mut cc_device, src: *const cc_view, dst: *mut f32, n: usize) -> c_int;
    pub fn cc_host_alloc(dev: *mut cc_device, bytes: usize, out: *mut *mut c_void) -> c_int;
    pub fn cc_host_free(dev: *mut cc_device, p: *mut c_void);

    // ---- test / bench hooks ----
    pub fn cc_test_quantize_activation(
        dev: *mut cc_device,
        x: *const cc_view,
        act_type: i32,
        dst: *mut c_void,
        nbytes: usize,
    ) -> c_int;

    // ---- sharded decode: the exchange step ----
    pub fn cc_comm_create(dev: *mut cc_device, rank: i32, world: i32, handle_out_64: *mut u8) -> c_int;
    pub fn cc_comm_connect(dev: *mut cc_device, handles_world_x_64: *const u8) -> c_int;
    pub fn cc_comm_connect_local(dev: *mut cc_device, peers: *const *mut cc_device) -> c_int;
    pub fn cc_comm_nccl_unique_id(dev: *mut cc_device, id_out_128: *mut u8) -> c_int;
    pub fn cc_comm_init_nccl(dev: *mut cc_device, id_128: *const u8) -> c_int;
    pub fn cc_comm_rank(dev: *mut cc_device) -> i32;
    pub fn cc_comm_world_size(dev: *mut cc_device) -> i32;
    pub fn cc_all_reduce_sum_inplace(dev: *mut cc_device, x: *const cc_view) -> c_int;
    pub fn cc_all_gather(dev: *mut cc_device, dst: *const cc_view, src: *const cc_view) -> c_int;
    pub fn cc_tensor_synth_slice(
        dev: *mut cc_device,
        shape: *const i64,
        ndim: i32,
        ggml_type: i32,
        seed: u64,
        tensor_id: u64,
        scale: f32,
        row0: i64,
        nrows: i64,
        col0: i64,
        ncols: i64,
        out: *mut *mut cc_buf,
    ) -> c_int;

    // ---- synthetic weights, timing, block export ----
    pub fn cc_tensor_synth(
        dev: *mut cc_device,
        shape: *const i64,
        ndim: i32,
        ggml_type: i32,
        seed: u64,
        tensor_id: u64,
        scale: f32,
        out: *mut *mut cc_buf,
    ) -> c_int;
    pub fn cc_bench_timer_begin(dev: *mut cc_device) -> c_int;
    pub fn cc_bench_timer_end(dev: *mut cc_device, ms: *mut f32) -> c_int;
    pub fn cc_test_export_blocks(dev: *mut cc_device, buf: *const cc_buf, dst: *mut c_void, nbytes: usize) -> c_int;
}
