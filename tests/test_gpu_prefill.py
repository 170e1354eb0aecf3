"""The dense (prefill) path of matmul_vec: (m, k) @ (b, k) for b >= 32 rows runs as TMA + wgmma tiles
(csrc/prefill_gemm.cu).  Reference behaviour: the batched rhs of primitives/matmul_vec.rs:6-8,26-78 (every output element
is vec_dot(W row, Q8_0-quantised activation row)).

The tensor-core path multiplies f16(w) * f16(q * d) with f32 accumulation, where w is the reference's dequantised weight and
q * d the reference's quantised activation: each operand carries one f16 rounding (relative 2^-11), so
    |got - want| <= 2 * 2^-11 * sum_k |w_k a_k|  (+ f32 accumulation noise)
is a rigorous bound; the test asserts 1.2e-3 * sum|terms| elementwise and reports the achieved ratio."""
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


def run_dense(gdev, t, m, k, b, seed=0):
    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(seed)
    raw = random_weight(t, m, k, rng, 0.02)
    x = rng.standard_normal(b * k).astype(np.float32)
    l0 = gdev.launch_count()
    got = CudaTensor.from_cpu(raw, [m, k], t, gdev).matmul_vec(CudaTensor.new(x, [b, k], gdev))
    assert got.shape() == [b, m]
    got = got.export().reshape(b, m).astype(np.float64)
    want = oc.gemv(t, raw, m, k, x.reshape(b, k)).reshape(b, m).astype(np.float64)
    at = oc.rhs_type(t)
    assert at in (oc.Q8_0, oc.Q8_K)
    wd = np.abs(oc.dequantize(t, raw, m * k).reshape(m, k)).astype(np.float64)
    ad = np.stack([np.abs(oc.dequantize(at, oc.quantize(at, r), k)) for r in x.reshape(b, k)]).astype(np.float64)
    budget = (ad @ wd.T) * 1.2e-3 + 1e-30
    diff = np.abs(got - want)
    assert (diff <= budget).all(), (oc.TYPE_NAMES[t], m, k, b, float((diff / budget).max()))
    # and in the usual sense: a fraction of the typical output magnitude
    assert diff.max() <= 2e-3 * np.abs(want).max()
    return float((diff / budget).max())


@pytest.mark.parametrize("t", [oc.Q8_0, oc.Q4_0, oc.Q5_0])
def test_prefill_dense_small_tiles(gdev, t):
    # one 128-row weight tile, N tile of 64 with a ragged batch (40 of 64 rows) and k = 4 stages exactly / more than the ring
    run_dense(gdev, t, 128, 256, 40, seed=10 + t)
    run_dense(gdev, t, 128, 1024, 64, seed=20 + t)


@pytest.mark.parametrize("t", [oc.Q4_K, oc.Q6_K])
def test_prefill_dense_k_quants(gdev, t):
    # K-quant weights: the activation is quantised to Q8_K (buf_q8_k.rs:84-131) and q * d enters the GEMM
    run_dense(gdev, t, 256, 1024, 96, seed=60 + t)
    run_dense(gdev, t, 128, 4096, 64, seed=70 + t)


def test_prefill_dense_ragged_edges(gdev):
    # m not a multiple of 128 (out-of-bounds rows read as zero, stores guarded), b not a multiple of the N tile, all three N tiles
    run_dense(gdev, oc.Q8_0, 200, 512, 100, seed=31)       # N tile 128
    run_dense(gdev, oc.Q8_0, 333, 512, 250, seed=32)       # N tile 256, ragged
    run_dense(gdev, oc.Q8_0, 96, 4096, 33, seed=33)        # fewer rows than one tile


@pytest.mark.parametrize("t", [oc.Q8_0, oc.Q4_0])
def test_prefill_dense_7b_shapes(gdev, t):
    # Llama-2-7B / Mistral-7B row lengths; enough tiles to wrap the 4-stage ring many times (k = 11008 -> 172 k-blocks)
    r1 = run_dense(gdev, t, 512, 4096, 256, seed=40 + t)
    r2 = run_dense(gdev, t, 256, 11008, 192, seed=50 + t)
    print("prefill error / budget:", r1, r2)


def test_prefill_dense_256_row_cta_tiles(gdev):
    # several 128-row CTA tiles (one 64-row half per consumer warpgroup) with a ragged last tile (1000 = 7 x 128 + 104) and all three
    # N tiles (64, 128, 256 batch rows)
    run_dense(gdev, oc.Q8_0, 640, 512, 64, seed=81)
    run_dense(gdev, oc.Q8_0, 1000, 1024, 130, seed=82)
    run_dense(gdev, oc.Q4_0, 1024, 2048, 300, seed=83)


def test_prefill_small_batches_keep_the_exact_block_path(gdev):
    """b below the dense threshold still takes the per-row quantised dot (1e-6 * sum|terms| parity, test_gpu_matvec.py)"""
    from tests.test_gpu_matvec import run_case
    run_case(gdev, oc.Q8_0, 33, 1024, b=3, seed=301)
