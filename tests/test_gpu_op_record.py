"""Every trait op on its own, each on a fresh device, in eager mode and in lazy modes 1 and 2: the outputs are bit-identical.  The inputs
are flushed before the op and the op is flushed alone, so a lazy device runs it as an unmatched step of its plan (through the same eager
launch as eager mode), or as the fused step that takes a lone op of its kind (a row pick, an argmax, a sampler, a K-quant matvec)."""
import ctypes as C

import numpy as np
import pytest

from crabml_b200.capi import ROPE_LLAMA, ROPE_NEOX
from oracle import oracle as oc
from tests.blockgen import random_weight
from tests.gpu_common import assert_same_bits, run_modes

pytestmark = pytest.mark.gpu


def _new(dev, shape, seed, scale=1.0):
    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(seed)
    return CudaTensor.new((rng.standard_normal(int(np.prod(shape))) * scale).astype(np.float32), list(shape), dev)


def _f16(dev, shape, seed):
    """an f16 tensor [rows, cols], filled through the f32 -> f16 row copy"""
    from crabml_b200 import CudaTensor
    t = CudaTensor.alloc(list(shape), oc.F16, dev)
    t.copy_rows_from(_new(dev, shape, seed), list(range(shape[0])))
    return t


def _f16_rows(dev, t):
    """the f32 values of a contiguous 2d f16 tensor, widened through the row copy"""
    from crabml_b200 import CudaTensor
    rows, cols = t.shape()
    out = CudaTensor.alloc([rows, cols], oc.F32, dev)
    dev.flush()
    out.copy_rows_from(t, list(range(rows)))
    return out.export()


# Each case builds its inputs, flushes, runs ONE op, flushes, and returns the outputs.
def case_dup(dev):
    x = _new(dev, [3, 64], 1); dev.flush()
    d = x.dup(); dev.flush()
    return [d.export()]


def case_contiguous_f32(dev):
    x = _new(dev, [4, 6, 8], 2).transpose([1, 0, 2]); dev.flush()
    c = x.contiguous(); dev.flush()
    return [c.export()]


def case_contiguous_f16(dev):
    x = _f16(dev, [6, 40], 3).transpose([1, 0]); dev.flush()
    c = x.contiguous(); dev.flush()
    return [_f16_rows(dev, c)]


def case_concatenate(dev):
    from crabml_b200 import CudaTensor
    full = CudaTensor.alloc([2, 5, 8], oc.F32, dev)
    cache = full.resize(1, 0)
    k = _new(dev, [1, 2, 8], 4); dev.flush()
    cache.concatenate(k.transpose([1, 0, 2]), 1); dev.flush()
    return [full.export()]


def case_copy_rows_f32(dev):
    from crabml_b200 import CudaTensor
    src = _new(dev, [5, 16], 5)
    dst = CudaTensor.alloc([3, 16], oc.F32, dev); dev.flush()
    dst.copy_rows_from(src, [4, 0, 2]); dev.flush()
    return [dst.export()]


def case_copy_rows_quant(dev):
    from crabml_b200 import CudaTensor
    raw = random_weight(oc.Q4_K, 5, 256, np.random.default_rng(6))
    w = CudaTensor.from_cpu(raw, [5, 256], oc.Q4_K, dev)
    dst = CudaTensor.alloc([2, 256], oc.F32, dev); dev.flush()
    dst.copy_rows_from(w, [3, 1]); dev.flush()
    return [dst.export()]


def case_copy_rows_from_slot(dev):
    from crabml_b200 import CudaTensor
    tab = _new(dev, [5, 32], 7)
    row = CudaTensor.alloc([32], oc.F32, dev)
    dev.check(dev.lib.cc_slot_set(dev.handle, 2, 3)); dev.flush()
    dev.check(dev.lib.cc_copy_rows_from_slot(dev.handle, C.byref(row._view()), C.byref(tab._view()), 2)); dev.flush()
    return [row.export()]


def _rope(mode):
    def case(dev):
        x = _new(dev, [2, 4, 32], 8); dev.flush()
        x.rope_inplace(mode, 7, 16); dev.flush()
        return [x.export()]
    return case


def _unary(name, *args):
    def case(dev):
        x = _new(dev, [100], 9, 3.0); dev.flush()
        getattr(x, name)(*args); dev.flush()
        return [x.export()]
    return case


def case_rms_norm(dev):
    x = _new(dev, [2, 64], 10); dev.flush()
    x.rms_norm_inplace(1e-5); dev.flush()
    return [x.export()]


def case_softmax(dev):
    x = _new(dev, [3, 2, 37], 11, 4.0); dev.flush()
    x.softmax_inplace(2); dev.flush()
    return [x.export()]


def _binary(name):
    def case(dev):
        # 30 elements against a row of 10: chunks_exact(4) leaves the last 2 of x and of the row alone
        x, y = _new(dev, [3, 10], 12), _new(dev, [10], 13); dev.flush()
        getattr(x, name)(y); dev.flush()
        return [x.export()]
    return case


def _bmm(kcontig):
    def case(dev):
        cache = _new(dev, [4, 6, 8], 14)
        if kcontig:                                   # q [4, 1, 8] x K^T [4, 8, 6]: rhs contiguous on k
            a, b = _new(dev, [4, 1, 8], 15), cache.transpose([0, 2, 1])
        else:                                         # w [4, 1, 6] x V [4, 6, 8]: rhs contiguous on n
            a, b = _new(dev, [4, 1, 6], 15), cache
        dev.flush()
        c = a.batch_matmul(b); dev.flush()
        return [c.export()]
    return case


def _matvec(wt, rows):
    def case(dev):
        from crabml_b200 import CudaTensor
        m, k = 64, 512
        w = CudaTensor.from_cpu(random_weight(wt, m, k, np.random.default_rng(16)), [m, k], wt, dev)
        x = _new(dev, [rows, k] if rows > 1 else [k], 17); dev.flush()
        out = w.matmul_vec(x); dev.flush()
        return [out.export()]
    return case


def case_argmax_to_slot(dev):
    x = _new(dev, [300], 18); dev.flush()
    dev.check(dev.lib.cc_argmax_to_slot(dev.handle, C.byref(x._view()), 1, 0)); dev.flush()
    return [dev.read_history(0, 1)]


def case_sample_to_slot(dev):
    x = _new(dev, [300], 19, 2.0); dev.flush()
    x.sample_to_slot(0.8, 0.9, 7, 3, 1, 0); dev.flush()
    return [dev.read_history(0, 1)]


CASES = {
    "dup": case_dup, "contiguous_f32": case_contiguous_f32, "contiguous_f16": case_contiguous_f16, "concatenate": case_concatenate,
    "copy_rows_f32": case_copy_rows_f32, "copy_rows_q4_k": case_copy_rows_quant, "copy_rows_from_slot": case_copy_rows_from_slot,
    "rope_llama": _rope(ROPE_LLAMA), "rope_neox": _rope(ROPE_NEOX),
    "rms_norm": case_rms_norm, "softmax": case_softmax, "silu": _unary("silu_inplace"), "gelu": _unary("gelu_inplace"),
    "add_tail": _binary("add_inplace"), "mul_tail": _binary("mul_inplace"), "scale": _unary("scale_inplace", 0.3),
    "bmm_kcontig": _bmm(True), "bmm_ncontig": _bmm(False),
    "matvec_q4_k": _matvec(oc.Q4_K, 1), "matvec_q8_0_batched": _matvec(oc.Q8_0, 3),
    "argmax_to_slot": case_argmax_to_slot, "sample_to_slot": case_sample_to_slot,
}


@pytest.mark.parametrize("name", list(CASES))
def test_op_alone_is_bit_identical_in_every_mode(name):
    res = run_modes(CASES[name])
    for lazy in (1, 2):
        assert_same_bits(res[lazy], res[0], f"{name}: lazy={lazy} vs eager")
