"""Host logic of the sampled generate loop (ccr_runner_generate_ex, crabml_b200/csrc/host/llama2_sampler.cpp) on CPU, built against
the recording mock of the C ABI (tests/host/mock_abi.cpp + mock_sampler.cpp): with temperature > 0 it issues the greedy loop's op
sequence (ccr_runner_generate_greedy_ex) with cc_sample_to_slot where cc_argmax_to_slot was, the coin index being the generated-token
index; with temperature 0 it is the greedy loop call for call; a bad setting is rejected before any op."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from crabml_b200 import capi
from oracle import oracle as oc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "crabml_b200", "csrc", "host")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("mocksampler") / "librunner_sampler_mock.so")
    srcs = [os.path.join(HOST, "llama2_runner.cpp"), os.path.join(HOST, "llama2_sampler.cpp"),
            os.path.join(ROOT, "tests", "host", "mock_abi.cpp"), os.path.join(ROOT, "tests", "host", "mock_sampler.cpp")]
    subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", *srcs, "-o", out], check=True, capture_output=True, timeout=300)
    L = C.CDLL(out)
    L.mock_device.restype = C.c_void_p
    L.mock_new_buf.restype, L.mock_new_buf.argtypes = C.c_void_p, [C.c_int, C.c_int64]
    L.mock_trace_size.restype = C.c_int64
    L.mock_trace_copy.argtypes = [C.c_char_p]
    L.ccr_runner_create.argtypes = [C.c_void_p, C.POINTER(capi.ccr_llama_config), C.POINTER(capi.ccr_llama_weights), C.c_int32, C.POINTER(C.c_void_p)]
    L.ccr_runner_last_error.restype, L.ccr_runner_last_error.argtypes = C.c_char_p, [C.c_void_p]
    L.ccr_runner_destroy.argtypes = [C.c_void_p]
    i64p, i32p = C.POINTER(C.c_int64), C.POINTER(C.c_int32)
    L.ccr_runner_generate_greedy_ex.argtypes = [C.c_void_p, i64p, C.c_int32, C.c_int32, C.c_int64, i64p, i32p, C.c_void_p]
    L.ccr_runner_generate_ex.argtypes = [C.c_void_p, i64p, C.c_int32, C.c_int32, C.c_int64, C.c_float, C.c_float, C.c_uint64, i64p, i32p, C.c_void_p]
    return L


def _trace(L, call):
    """a fresh tinyllamas-shaped runner (2 layers, vocab 32000, context 32); `call(h)` runs one generate; returns (rc, ids, trace)"""
    nl, dim, hid, vocab, wt = 2, 288, 768, 32000, oc.Q8_0
    keep = []

    def arr(dtype, n):
        a = (C.c_void_p * nl)(*[L.mock_new_buf(dtype, n) for _ in range(nl)])
        keep.append(a)
        return C.cast(a, C.POINTER(C.c_void_p))
    w = capi.ccr_llama_weights(L.mock_new_buf(wt, vocab * dim), arr(wt, dim * dim), arr(wt, dim * dim), arr(wt, dim * dim), arr(wt, dim * dim),
                               arr(wt, hid * dim), arr(wt, dim * hid), arr(wt, hid * dim), arr(oc.F32, dim), arr(oc.F32, dim), L.mock_new_buf(oc.F32, dim),
                               L.mock_new_buf(wt, vocab * dim))
    cconf = capi.ccr_llama_config(6, 6, nl, dim, hid, 256, vocab, 48, 1e-5, 0, 0, 1, hid)
    h = C.c_void_p()
    assert L.ccr_runner_create(L.mock_device(), C.byref(cconf), C.byref(w), 32, C.byref(h)) == 0
    L.mock_trace_clear()
    out = (C.c_int64 * 8)()
    n = C.c_int32(0)
    rc = call(h, out, C.byref(n))
    buf = C.create_string_buffer(int(L.mock_trace_size()) + 1)
    L.mock_trace_copy(buf)
    err = L.ccr_runner_last_error(h).decode()
    L.ccr_runner_destroy(h)
    return rc, list(out[:n.value]), buf.value.decode().splitlines(), err


PROMPT = (C.c_int64 * 2)(1, 365)


@pytest.mark.parametrize("eos", [-1, 7])
@pytest.mark.parametrize("temperature,topp,seed", [(0.8, 0.9, 42), (1.0, 1.0, 2**64 - 1), (1.7, 0.0, 0)])
def test_sampled_loop_is_the_greedy_loop_with_the_sampler_in_place_of_the_argmax(lib, eos, temperature, topp, seed):
    L = lib
    rc0, ids0, greedy, _ = _trace(L, lambda h, out, n: L.ccr_runner_generate_greedy_ex(h, PROMPT, 2, 4, eos, out, n, None))
    rc1, ids1, sampled, err = _trace(L, lambda h, out, n: L.ccr_runner_generate_ex(h, PROMPT, 2, 4, eos, temperature, topp, seed, out, n, None))
    assert rc0 == 0 and rc1 == 0, err
    assert ids1 == ids0          # the mock's device always samples token 7
    calls = [ln for ln in sampled if ln.startswith("tap sample_to_slot")]
    assert len(calls) == (4 if eos < 0 else 2)
    for i, ln in enumerate(calls):
        assert ln == "tap sample_to_slot n=32000 slot=0 hist=%d T=%.9g topp=%.9g seed=%d coin=%d" % (i, np.float32(temperature), np.float32(topp), seed, i)
    it = iter(calls)
    assert [next(it) if ln.startswith("argmax_to_slot") else ln for ln in greedy] == sampled
    assert not [ln for ln in sampled if ln.startswith("argmax_to_slot")]


@pytest.mark.parametrize("eos", [-1, 7])
def test_temperature_zero_is_the_greedy_loop_call_for_call(lib, eos):
    L = lib
    _, ids0, greedy, _ = _trace(L, lambda h, out, n: L.ccr_runner_generate_greedy_ex(h, PROMPT, 2, 4, eos, out, n, None))
    rc, ids1, sampled, err = _trace(L, lambda h, out, n: L.ccr_runner_generate_ex(h, PROMPT, 2, 4, eos, 0.0, 0.9, 5, out, n, None))
    assert rc == 0, err
    assert ids1 == ids0 and sampled == greedy


@pytest.mark.parametrize("temperature,topp", [(float("nan"), 0.9), (-0.5, 0.9), (1.0, float("nan"))])
def test_bad_settings_are_rejected_before_any_op(lib, temperature, topp):
    L = lib
    rc, ids, trace, err = _trace(L, lambda h, out, n: L.ccr_runner_generate_ex(h, PROMPT, 2, 4, -1, temperature, topp, 1, out, n, None))
    assert rc == capi.CC_ERR_TENSOR and ids == [] and trace == [] and "temperature" in err
