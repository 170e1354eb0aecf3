"""ctypes binding + numpy helpers for the CPU oracle (oracle/crabml_oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs.  Never imported by crabml_b200/.

Parity status: PINNED -- see tests/test_oracle_kats.py (reference KATs) and
tests/test_oracle_golden_text.py (reference golden generations).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "build", "libcrabml_oracle.so")

# GGML type ids (crabml-core/src/gguf.rs:86-108)
F32, F16, Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, Q8_1 = 0, 1, 2, 3, 6, 7, 8, 9
Q2_K, Q3_K, Q4_K, Q5_K, Q6_K, Q8_K = 10, 11, 12, 13, 14, 15
TYPE_NAMES = {F32: "F32", F16: "F16", Q4_0: "Q4_0", Q4_1: "Q4_1", Q5_0: "Q5_0", Q5_1: "Q5_1",
              Q8_0: "Q8_0", Q8_1: "Q8_1", Q2_K: "Q2_K", Q3_K: "Q3_K", Q4_K: "Q4_K", Q5_K: "Q5_K",
              Q6_K: "Q6_K", Q8_K: "Q8_K"}
QUANT_TYPES = [Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, Q2_K, Q3_K, Q4_K, Q5_K, Q6_K, Q8_K]

BUGCOMPAT = 1
ORDER_AVX2 = 2


def build(force: bool = False) -> str:
    """Compile the oracle with the committed Makefile (gcc only)."""
    src = os.path.join(_HERE, "crabml_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, sz, i32, f32 = C.c_void_p, C.c_size_t, C.c_int, C.c_float
        L.oc_block_elems.argtypes = [i32]; L.oc_block_elems.restype = i32
        L.oc_block_bytes.argtypes = [i32]; L.oc_block_bytes.restype = sz
        L.oc_vec_dot_rhs_type.argtypes = [i32]; L.oc_vec_dot_rhs_type.restype = i32
        L.oc_f16_to_f32.argtypes = [vp, vp, sz]
        L.oc_f32_to_f16.argtypes = [vp, vp, sz]
        L.oc_exp_lut.argtypes = [vp]
        L.oc_gelu_lut.argtypes = [vp]
        L.oc_dequantize.argtypes = [i32, vp, sz, vp, i32]; L.oc_dequantize.restype = i32
        L.oc_quantize.argtypes = [i32, vp, sz, vp]; L.oc_quantize.restype = i32
        L.oc_vec_dot.argtypes = [i32, vp, vp, sz, i32]; L.oc_vec_dot.restype = f32
        L.oc_gemv.argtypes = [i32, vp, sz, sz, vp, sz, vp, i32, i32]; L.oc_gemv.restype = i32
        L.oc_gemv_q.argtypes = [i32, vp, sz, sz, vp, sz, vp, i32, i32]; L.oc_gemv_q.restype = i32
        L.oc_rms_norm.argtypes = [vp, sz, sz, f32]
        L.oc_rope.argtypes = [vp, sz, sz, sz, i32, sz, sz]
        L.oc_softmax.argtypes = [vp, sz, sz, vp]
        L.oc_silu.argtypes = [vp, sz, vp]
        L.oc_gelu.argtypes = [vp, sz, vp]
        L.oc_add.argtypes = [vp, sz, vp, sz]
        L.oc_mul.argtypes = [vp, sz, vp, sz]
        L.oc_batch_matmul_f32.argtypes = [vp, vp, vp] + [sz] * 8
        L.oc_batch_matmul_f16.argtypes = [vp, vp, vp] + [sz] * 8
        L.oc_hw_threads.restype = i32
        L.oc_synth_blocks.argtypes = [i32, sz, C.c_uint64, C.c_uint64, f32, vp]; L.oc_synth_blocks.restype = i32
        _lib = L
    return _lib


def big_empty(nbytes: int) -> np.ndarray:
    """uint8 buffer backed by a pre-faulted anonymous mapping (MAP_POPULATE): first-touch page faults are very
    slow in some virtual machines, which would dominate host-side weight generation."""
    import mmap
    if nbytes < (8 << 20):
        return np.empty(nbytes, np.uint8)
    m = mmap.mmap(-1, nbytes, flags=mmap.MAP_PRIVATE | mmap.MAP_ANONYMOUS | getattr(mmap, "MAP_POPULATE", 0x8000))
    return np.frombuffer(m, np.uint8)


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def block_elems(t): return lib().oc_block_elems(t)
def block_bytes(t): return lib().oc_block_bytes(t)
def rhs_type(t): return lib().oc_vec_dot_rhs_type(t)
def hw_threads(): return lib().oc_hw_threads()


def nbytes_for(t: int, n_elems: int) -> int:
    be = block_elems(t)
    assert n_elems % be == 0, (TYPE_NAMES[t], n_elems)
    return n_elems // be * block_bytes(t)


_EXP_LUT = None
_GELU_LUT = None


def exp_lut() -> np.ndarray:
    global _EXP_LUT
    if _EXP_LUT is None:
        _EXP_LUT = np.empty(65536, np.uint16)
        lib().oc_exp_lut(_p(_EXP_LUT))
    return _EXP_LUT


def gelu_lut() -> np.ndarray:
    global _GELU_LUT
    if _GELU_LUT is None:
        _GELU_LUT = np.empty(65536, np.uint16)
        lib().oc_gelu_lut(_p(_GELU_LUT))
    return _GELU_LUT


def dequantize(t: int, blocks: np.ndarray, n: int, flags: int = 0) -> np.ndarray:
    blocks = np.ascontiguousarray(blocks).view(np.uint8).reshape(-1)
    assert blocks.size >= nbytes_for(t, n)
    out = np.empty(n, np.float32)
    rc = lib().oc_dequantize(t, _p(blocks), n, _p(out), flags)
    assert rc == 0
    return out


def quantize(act_type: int, x: np.ndarray) -> np.ndarray:
    x = np.ascontiguousarray(x, np.float32).reshape(-1)
    out = np.empty(nbytes_for(act_type, x.size), np.uint8)
    rc = lib().oc_quantize(act_type, _p(x), x.size, _p(out))
    assert rc == 0
    return out


def vec_dot(w_type: int, w: np.ndarray, act: np.ndarray, n: int, flags: int = 0) -> np.float32:
    w = np.ascontiguousarray(w).view(np.uint8).reshape(-1)
    act = np.ascontiguousarray(act).view(np.uint8).reshape(-1)
    return np.float32(lib().oc_vec_dot(w_type, _p(w), _p(act), n, flags))


def gemv(w_type: int, w: np.ndarray, m: int, k: int, x: np.ndarray, threads: int = 1, flags: int = 0) -> np.ndarray:
    """(m,k) @ (b,k) -> (b,m) ; x of shape (k,) gives (m,)."""
    w = np.ascontiguousarray(w).view(np.uint8).reshape(-1)
    assert w.size >= nbytes_for(w_type, m * k), (w.size, nbytes_for(w_type, m * k))
    x = np.ascontiguousarray(x, np.float32)
    b = x.size // k
    out = np.empty(b * m, np.float32)
    rc = lib().oc_gemv(w_type, _p(w), m, k, _p(x), b, _p(out), threads, flags)
    assert rc == 0
    return out.reshape(x.shape[:-1] + (m,)) if x.ndim > 1 else out


def gemv_q(w_type, w, m, k, act, b=1, threads=1, flags=0):
    w = np.ascontiguousarray(w).view(np.uint8).reshape(-1)
    act = np.ascontiguousarray(act).view(np.uint8).reshape(-1)
    out = np.empty(b * m, np.float32)
    rc = lib().oc_gemv_q(w_type, _p(w), m, k, _p(act), b, _p(out), threads, flags)
    assert rc == 0
    return out


def f16_to_f32(h: np.ndarray) -> np.ndarray:
    h = np.ascontiguousarray(h).view(np.uint16)
    out = np.empty(h.shape, np.float32)
    lib().oc_f16_to_f32(_p(h), _p(out), h.size)
    return out


def f32_to_f16(x: np.ndarray) -> np.ndarray:
    x = np.ascontiguousarray(x, np.float32)
    out = np.empty(x.shape, np.uint16)
    lib().oc_f32_to_f16(_p(x), _p(out), x.size)
    return out


# in-place primitives on contiguous float32 arrays -------------------------------------------
def rms_norm_(x: np.ndarray, eps: float):
    rows, cols = (1, x.shape[0]) if x.ndim == 1 else (x.shape[0], x.shape[1])
    lib().oc_rms_norm(_p(x), rows, cols, eps)


def rope_(x: np.ndarray, mode: int, pos: int, rope_dim: int):
    if x.ndim == 2:
        n_batch, stride, hd = 1, x.size, x.shape[1]
    else:
        n_batch, stride, hd = x.shape[0], x.shape[1] * x.shape[2], x.shape[2]
    lib().oc_rope(_p(x), n_batch, stride, hd, mode, pos, rope_dim)


def softmax_(x: np.ndarray):
    cols = x.shape[-1]
    lib().oc_softmax(_p(x), x.size // cols, cols, _p(exp_lut()))


def silu_(x: np.ndarray):
    lib().oc_silu(_p(x), x.size, _p(exp_lut()))


def gelu_(x: np.ndarray):
    lib().oc_gelu(_p(x), x.size, _p(gelu_lut()))


def add_(x: np.ndarray, y: np.ndarray):
    lib().oc_add(_p(x), x.size, _p(y), y.size)


def mul_(x: np.ndarray, y: np.ndarray):
    lib().oc_mul(_p(x), x.size, _p(y), y.size)


def batch_matmul(a: np.ndarray, b_buf: np.ndarray, b_shape, b_strides, b_is_f16: bool) -> np.ndarray:
    """a: dense (ab,m,k) f32; b: flat buffer with explicit (shape, strides) in elements."""
    ab, m, k = a.shape
    bb, k2, n = b_shape
    assert k == k2 and ab % bb == 0
    c = np.zeros((ab, m, n), np.float32)
    fn = lib().oc_batch_matmul_f16 if b_is_f16 else lib().oc_batch_matmul_f32
    fn(_p(np.ascontiguousarray(a)), _p(b_buf), _p(c), ab, bb, m, k, n, *[int(s) for s in b_strides])
    return c
