"""THE hot path: matmul_vec for every GGUF quant type vs the oracle's gemv (SURVEY §8a a1-a11)."""
import numpy as np
import pytest

from oracle import oracle as oc
from tests.blockgen import random_weight
from tests.gpu_common import make_device

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gdev():
    d = make_device()
    yield d
    d.close()


def gemv_budget(t, raw, m, k, x):
    """Error budget of a matvec against oc.gemv: f32 summation-order noise, 1e-6 * sum_i |w_i a_i| per output (the integer block dots
    are exact), with a the quantised activation the kernel multiplies.  x: [k] or [b, k] -> [b * m] (row-major like the output).
    The weights are dequantised a slab of rows at a time, so that large matrices stay cheap in host memory."""
    at = oc.rhs_type(t)
    xb = np.asarray(x, np.float32).reshape(-1, k)
    ad = np.stack([np.abs(oc.dequantize(at, oc.quantize(at, r), k)) for r in xb]).astype(np.float64)
    rows_per = max(1, (1 << 22) // k)
    row_bytes = raw.size // m
    sums = np.empty((xb.shape[0], m), np.float64)
    for r0 in range(0, m, rows_per):
        r1 = min(m, r0 + rows_per)
        wd = np.abs(oc.dequantize(t, raw[r0 * row_bytes:r1 * row_bytes], (r1 - r0) * k).reshape(r1 - r0, k)).astype(np.float64)
        sums[:, r0:r1] = ad @ wd.T
    return sums.reshape(-1) * 1e-6 + 1e-30


def run_case(gdev, t, m, k, b=None, seed=0, scale=0.02):
    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(seed)
    raw = random_weight(t, m, k, rng, scale)
    xs = [k] if b is None else [b, k]
    x = rng.standard_normal(int(np.prod(xs))).astype(np.float32)
    gw = CudaTensor.from_cpu(raw, [m, k], t, gdev)
    got = gw.matmul_vec(CudaTensor.new(x, xs, gdev))
    assert got.shape() == ([m] if b is None else [b, m])
    want = oc.gemv(t, raw, m, k, x.reshape(xs))
    budget = gemv_budget(t, raw, m, k, x)
    if t in (oc.Q4_1, oc.Q5_1):
        budget = budget * 1.0          # same f16-rounded products as the reference; no extra slack
    diff = np.abs(got.export().astype(np.float64) - want.reshape(-1).astype(np.float64))
    assert (diff <= budget).all(), (oc.TYPE_NAMES[t], m, k, float((diff / budget).max()))
    return got.export(), want.reshape(-1)


@pytest.mark.parametrize("t", oc.QUANT_TYPES)
def test_matvec_all_types_small(gdev, t):
    k = 512 if oc.block_elems(t) == 256 else 288          # 288 = tinyllamas dim: 9 blocks/row, odd tail
    run_case(gdev, t, 37, k, seed=t)


@pytest.mark.parametrize("t", oc.QUANT_TYPES)
def test_matvec_all_types_7b_rows(gdev, t):
    # Llama-2-7B row lengths: 4096 and 11008 (=43 super-blocks, 344 blocks: not a multiple of 32 lanes)
    run_case(gdev, t, 64, 4096, seed=100 + t)
    run_case(gdev, t, 40, 11008, seed=200 + t)


@pytest.mark.parametrize("t", [oc.Q8_0, oc.Q4_0, oc.Q4_K, oc.Q6_K])
def test_matvec_batched_rhs(gdev, t):
    # (m,k) @ (b,k) -> (b,m)  (matmul_vec.rs:6-8)
    run_case(gdev, t, 33, 1024, b=3, seed=300 + t)


@pytest.mark.parametrize("t", [oc.Q8_0, oc.Q4_0])
def test_matvec_vocab_rows(gdev, t):
    # classifier shape: many rows (grid-stride path)
    run_case(gdev, t, 32000, 288, seed=400 + t)


def test_matvec_f16_weights(gdev):
    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(1)
    m, k = 50, 64
    w = rng.standard_normal((m, k)).astype(np.float16)
    x = rng.standard_normal(k).astype(np.float32)
    got = CudaTensor.from_cpu(w, [m, k], oc.F16, gdev).matmul_vec(CudaTensor.new(x, [k], gdev)).export()
    want = oc.gemv(oc.F16, w.view(np.uint16), m, k, x)
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5)


def test_matvec_errors(gdev):
    from crabml_b200 import CudaTensor, TensorError
    rng = np.random.default_rng(2)
    w = CudaTensor.from_cpu(random_weight(oc.Q8_0, 4, 64, rng), [4, 64], oc.Q8_0, gdev)
    with pytest.raises(TensorError):
        w.matmul_vec(CudaTensor.new(np.zeros(32), [32], gdev))                     # last dims differ
    with pytest.raises(TensorError):
        w.transpose([1, 0]).matmul_vec(CudaTensor.new(np.zeros(4), [4], gdev))     # not contiguous
    with pytest.raises(TensorError):
        CudaTensor.from_cpu(np.zeros(10, np.uint8), [4, 64], oc.Q8_0, gdev)         # too few bytes


def test_truncation_vs_rounding_is_visible(gdev):
    """Guards quirk B1: with round-to-nearest activation quantisation the result would differ by far
    more than the parity budget -- i.e. this test suite would catch a 'fixed' quantizer."""
    rng = np.random.default_rng(3)
    m, k = 16, 4096
    raw = random_weight(oc.Q8_0, m, k, rng)
    x = rng.standard_normal(k).astype(np.float32)
    got, want = run_case(gdev, oc.Q8_0, m, k, seed=3)
    blk = x.reshape(-1, 32)
    d = np.abs(blk).max(1, keepdims=True) / np.float32(127.0)
    q_round = np.rint(blk / d)
    w = oc.dequantize(oc.Q8_0, raw, m * k).reshape(m, k)
    rounded = w @ (q_round * d.astype(np.float16).astype(np.float32)).reshape(-1)
    assert np.abs(rounded - want).max() > 50 * np.abs(got - want).max()


@pytest.mark.parametrize("t", oc.QUANT_TYPES)
def test_matvec_exact_order_bit_identical(t):
    """exact_order mode: the scalar reference order (buf_q*.rs vec_dot_*_fallback) -> bit-identical rows."""
    from crabml_b200 import CudaTensor
    dev = make_device(exact_order=True)
    try:
        rng = np.random.default_rng(500 + t)
        for (m, k) in ((19, 512), (5, 4096)):
            raw = random_weight(t, m, k, rng)
            x = rng.standard_normal(k).astype(np.float32)
            got = CudaTensor.from_cpu(raw, [m, k], t, dev).matmul_vec(CudaTensor.new(x, [k], dev)).export()
            want = oc.gemv(t, raw, m, k, x)
            np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32), err_msg=oc.TYPE_NAMES[t])
    finally:
        dev.close()
