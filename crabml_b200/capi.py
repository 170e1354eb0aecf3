"""ctypes binding of include/crabml_cuda.h (the drop-in C ABI)."""
from __future__ import annotations

import ctypes as C
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libcrabml_cuda.so")
HEADER = os.path.join(os.path.dirname(HERE), "include", "crabml_cuda.h")
RUNNER_HEADER = os.path.join(os.path.dirname(HERE), "include", "crabml_runner.h")

CC_OK, CC_ERR_TENSOR, CC_ERR_CUDA, CC_ERR_ARG, CC_ERR_UNSUPPORTED = 0, 1, 2, 3, 4
CC_MAX_DIMS = 4

# GGMLType ids (crabml-core/src/gguf.rs:86-108)
F32, F16, Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, Q8_1 = 0, 1, 2, 3, 6, 7, 8, 9
Q2_K, Q3_K, Q4_K, Q5_K, Q6_K, Q8_K = 10, 11, 12, 13, 14, 15
ROPE_LLAMA, ROPE_NEOX = 0, 1


class TensorError(Exception):
    """ErrorKind::TensorError (crabml-core/src/error.rs:24-25)."""


class CudaError(RuntimeError):
    pass


class cc_view(C.Structure):
    _fields_ = [("buf", C.c_void_p), ("ndim", C.c_int32), ("shape", C.c_int64 * CC_MAX_DIMS), ("strides", C.c_int64 * CC_MAX_DIMS)]


class cc_device_options(C.Structure):
    _fields_ = [("device_ordinal", C.c_int32), ("debug_named_tensors", C.c_int32), ("lazy", C.c_int32),
                ("exact_order", C.c_int32), ("pool_bytes", C.c_uint64)]


def declared_symbols():
    """Every CC_API prototype name in the headers (used by the CPU-side export test)."""
    out = []
    for h in (HEADER, RUNNER_HEADER):
        with open(h) as f:
            out += re.findall(r"^CC_API [\w\s\*]+?\b(ccr?_\w*)\(", f.read(), flags=re.M)
    return out


class ccr_llama_config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_heads", "n_kv_heads", "n_layers", "embedding_dim", "hidden_dim", "seq_len", "vocab_size", "rope_dim")] + \
               [("rms_norm_eps", C.c_float), ("use_f16_kv_cache", C.c_int32), ("shard_rank", C.c_int32), ("shard_world", C.c_int32), ("hidden_local", C.c_int32),
                ("arch", C.c_int32)]


class ccr_llama_weights(C.Structure):
    _pp = C.POINTER(C.c_void_p)
    _fields_ = [("token_embed", C.c_void_p), ("wq", _pp), ("wk", _pp), ("wv", _pp), ("wo", _pp), ("ffn_gate", _pp),
                ("ffn_down", _pp), ("ffn_up", _pp), ("rms_att", _pp), ("rms_ffn", _pp), ("rms_final", C.c_void_p),
                ("output_weight", C.c_void_p), ("bq", _pp), ("bk", _pp), ("bv", _pp)]


_lib = None


def load_library(build_if_missing: bool = True):
    """Loads the in-tree .so; builds it with nvcc first when it is missing or stale."""
    global _lib
    if _lib is not None:
        return _lib
    alt = os.environ.get("CRABML_CUDA_LIB")          # developer A/B: another build of the same library
    if alt:
        build_if_missing = False
    if build_if_missing:
        from . import build as _build
        if _build.needs_build():
            _build.build()
    if not os.path.exists(LIB_PATH):
        raise CudaError(f"{LIB_PATH} is missing: run `python -m crabml_b200.build` (no CPU fallback exists)")
    L = C.CDLL(alt if alt else LIB_PATH)
    vp, i32, i64, u64, sz, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64, C.c_size_t, C.c_float
    pv = C.POINTER(cc_view)
    pp = C.POINTER(C.c_void_p)
    sig = {
        "cc_device_create": (i32, [C.POINTER(cc_device_options), pp]),
        "cc_device_destroy": (None, [vp]),
        "cc_last_error": (C.c_char_p, [vp]),
        "cc_device_synchronize": (i32, [vp]),
        "cc_device_launch_count": (u64, [vp]),
        "cc_device_flush": (i32, [vp]),
        "cc_lazy_stats": (i32, [vp, C.POINTER(u64)]),
        "cc_test_mega_barrier_floor": (i32, [vp, i32, C.POINTER(f32)]),
        "cc_lazy_mega_profile": (i32, [vp, C.POINTER(u64), C.POINTER(i32), i32, C.POINTER(i32)]),
        "cc_lazy_mega_variant": (i32, [vp]),
        "cc_device_stream": (vp, [vp]),
        "cc_tensor_from_cpu": (i32, [vp, vp, sz, C.POINTER(i64), i32, i32, pp]),
        "cc_tensor_alloc": (i32, [vp, C.POINTER(i64), i32, i32, pp]),
        "cc_tensor_retain": (None, [vp]),
        "cc_tensor_release": (None, [vp]),
        "cc_tensor_dtype": (i32, [vp]),
        "cc_tensor_capacity": (i64, [vp]),
        "cc_tensor_dup": (i32, [vp, pv, pp]),
        "cc_tensor_export_f32": (i32, [vp, pv, vp, sz]),
        "cc_copy_rows_from": (i32, [vp, pv, pv, C.POINTER(i64), i32]),
        "cc_concatenate": (i32, [vp, pv, pv, i32]),
        "cc_contiguous": (i32, [vp, pv, pp]),
        "cc_rope_inplace": (i32, [vp, pv, i32, i64, i64]),
        "cc_rms_norm_inplace": (i32, [vp, pv, f32]),
        "cc_softmax_inplace": (i32, [vp, pv, i32]),
        "cc_silu_inplace": (i32, [vp, pv]),
        "cc_gelu_inplace": (i32, [vp, pv]),
        "cc_mul_inplace": (i32, [vp, pv, pv]),
        "cc_add_inplace": (i32, [vp, pv, pv]),
        "cc_scale_inplace": (i32, [vp, pv, f32]),
        "cc_matmul_vec": (i32, [vp, pv, pv, pp]),
        "cc_batch_matmul": (i32, [vp, pv, pv, pp]),
        "cc_debug_tensor_tap": (i32, [vp, C.c_char_p, pv]),
        "cc_dump_debug_tensor": (i32, [vp, C.c_char_p, vp, C.POINTER(sz)]),
        "cc_test_quantize_activation": (i32, [vp, pv, i32, vp, sz]),
        "cc_tensor_synth": (i32, [vp, C.POINTER(i64), i32, i32, u64, u64, f32, pp]),
        "cc_test_export_blocks": (i32, [vp, vp, vp, sz]),
        "cc_tensor_synth_slice": (i32, [vp, C.POINTER(i64), i32, i32, u64, u64, f32, i64, i64, i64, i64, pp]),
        "cc_comm_create": (i32, [vp, i32, i32, vp]),
        "cc_comm_connect": (i32, [vp, vp]),
        "cc_comm_nccl_unique_id": (i32, [vp, vp]),
        "cc_comm_connect_local": (i32, [vp, vp]),
        "cc_device_set_sm_limit": (i32, [vp, i32]),
        "cc_comm_init_nccl": (i32, [vp, vp]),
        "cc_comm_rank": (i32, [vp]),
        "cc_comm_world_size": (i32, [vp]),
        "cc_all_reduce_sum_inplace": (i32, [vp, pv]),
        "cc_all_gather": (i32, [vp, pv, pv]),
        "cc_bench_timer_begin": (i32, [vp]),
        "cc_bench_timer_end": (i32, [vp, C.POINTER(f32)]),
    }
    sig.update({
        "ccr_runner_create": (i32, [vp, C.POINTER(ccr_llama_config), C.POINTER(ccr_llama_weights), i32, pp]),
        "ccr_runner_destroy": (None, [vp]),
        "ccr_runner_last_error": (C.c_char_p, [vp]),
        "ccr_runner_forward": (i32, [vp, C.POINTER(i64), i32, i64, vp]),
        "ccr_runner_kv_cache_len": (i64, [vp]),
        "ccr_runner_generate_greedy": (i32, [vp, C.POINTER(i64), i32, i32, i64, C.POINTER(i64), C.POINTER(i32)]),
        "ccr_runner_generate_greedy_ex": (i32, [vp, C.POINTER(i64), i32, i32, i64, C.POINTER(i64), C.POINTER(i32), vp]),
        "cc_argmax_to_slot": (i32, [vp, pv, i32, i64]),
        "cc_sample_to_slot": (i32, [vp, pv, f32, f32, u64, i64, i32, i64]),
        "ccr_runner_generate_ex": (i32, [vp, C.POINTER(i64), i32, i32, i64, f32, f32, u64, C.POINTER(i64), C.POINTER(i32), vp]),
        "cc_copy_rows_from_slot": (i32, [vp, pv, pv, i32]),
        "cc_slot_set": (i32, [vp, i32, i64]),
        "cc_read_history": (i32, [vp, i64, i64, C.POINTER(i64)]),
        "cc_tensor_export_f32_async": (i32, [vp, pv, vp, C.c_size_t]),
        "cc_host_alloc": (i32, [vp, C.c_size_t, pp]),
        "cc_host_free": (None, [vp, vp]),
    })
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    # optional entry points (later build stages); bound when present
    _lib = L
    return L
