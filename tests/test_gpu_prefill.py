"""The dense (prefill) path of matmul_vec: (m, k) @ (b, k) for b >= 32 rows runs as TMA + wgmma tiles
(csrc/prefill_gemm.cu).  Reference behaviour: the batched rhs of primitives/matmul_vec.rs:6-8,26-78 (every output element
is vec_dot(W row, quantised activation row)).

The tensor-core path multiplies f16(w) * f16(q * d) with f32 accumulation, where w is the reference's dequantised weight and
q * d the reference's quantised activation (Q8_0, or Q8_K for K-quant weights).  Two checks, elementwise:

1. Against the exact operands.  Block unpacking and activation quantisation are bit-exact to the oracle and the build uses no
   FMA contraction or flush-to-zero, so the host rebuilds the f16 operands the kernel multiplies,
       W16 = f16(dequantize(w)),   A16 = f16(q * d * 2^-e) * 2^e,
   (e = 0 unless the row's largest |q * d| reaches 2^15, see act_operand), and their f64 product is exact up to f64 rounding.
   The only remaining deviation is the tensor core's f32 accumulation: at most one rounding per 16-wide K step, counted twice
   for truncating adders,
       |got - A16 @ W16^T| <= (k / 16 + 16) * 2^-22 * (|A16| @ |W16|^T).
   An error the size of one dropped K step or of a truncating f16 conversion does not fit this bound.
2. Against the oracle's gemv, which is what the path means: each operand carries one f16 rounding (relative 2^-11), so
       |got - want| <= 1.2e-3 * sum_k |w_k a_k|.

Each check reports its worst error / bound ratio (run with -s to see them)."""
import time

import numpy as np
import pytest

from oracle import oracle as oc
from tests.blockgen import random_weight
from tests.gpu_common import assert_same_bits, fresh_device, run_modes

pytestmark = pytest.mark.gpu

DENSE_TYPES_Q8_0 = [oc.Q8_0, oc.Q4_0, oc.Q5_0]                            # activation partner Q8_0
DENSE_TYPES_Q8_K = [oc.Q2_K, oc.Q3_K, oc.Q4_K, oc.Q5_K, oc.Q6_K, oc.Q8_K]  # activation partner Q8_K
CHUNK = 2048                                                              # weight rows per step of the f64 reference


@pytest.fixture(scope="module")
def gdev():
    with fresh_device() as d:
        yield d


@pytest.fixture(scope="module", autouse=True)
def report_time():
    t0 = time.perf_counter()
    yield
    print(f"\ntest_gpu_prefill: {time.perf_counter() - t0:.1f} s")


def act_operand(at, x):
    """(b, k) f32 rows -> (A16 as f64, q * d as f32): the activation operand the dense path multiplies.  A row whose largest |q * d|
    reaches 2^15 enters at 2^-e (the smallest e that brings it below 2^15) and its outputs are scaled back by 2^e."""
    b, k = x.shape
    a = oc.dequantize(at, oc.quantize(at, x), b * k).reshape(b, k)
    amax = np.abs(a).max(1)
    e = np.zeros(b, np.int64)
    big = np.isfinite(amax) & (amax >= np.float32(2 ** 15))
    e[big] = np.frexp(amax[big])[1] - 15
    scaled = (a * np.ldexp(np.float32(1), -e).astype(np.float32)[:, None]).astype(np.float16)
    return scaled.astype(np.float64) * np.ldexp(1.0, e)[:, None], a


def check_dense(t, raw, m, k, x, got, oracle_rows=None, what=""):
    """got: (rows, m) outputs of the dense path for the (rows, k) activation x.  Asserts both bounds of the module docstring (the oracle
    bound only on oracle_rows, default all) and returns the two worst ratios."""
    at = oc.rhs_type(t)
    assert at in (oc.Q8_0, oc.Q8_K)
    got = got.astype(np.float64)
    assert np.isfinite(got).all(), (what, "non-finite outputs in rows", sorted(set(np.nonzero(~np.isfinite(got))[0].tolist())))
    a16, a = act_operand(at, x)
    ad = np.abs(a).astype(np.float64)
    w = oc.dequantize(t, raw, m * k).reshape(m, k)
    ref = np.empty(got.shape)
    absref = np.empty(got.shape)
    terms = np.empty(got.shape)
    for r0 in range(0, m, CHUNK):
        w16 = w[r0:r0 + CHUNK].astype(np.float16).astype(np.float64)
        ref[:, r0:r0 + CHUNK] = a16 @ w16.T
        absref[:, r0:r0 + CHUNK] = np.abs(a16) @ np.abs(w16).T
        terms[:, r0:r0 + CHUNK] = ad @ np.abs(w[r0:r0 + CHUNK]).astype(np.float64).T
    bound = (k / 16 + 16) * 2.0 ** -22 * absref
    diff = np.abs(got - ref)
    bad = diff > bound
    ratio = diff / np.where(bound > 0, bound, 1.0)
    assert not bad.any(), (what, "vs exact operands", float(ratio.max()), np.argwhere(bad)[:8].tolist())
    rows = np.arange(x.shape[0]) if oracle_rows is None else np.asarray(oracle_rows)
    want = oc.gemv(t, raw, m, k, x[rows], threads=oc.hw_threads()).reshape(len(rows), m).astype(np.float64)
    budget = terms[rows] * 1.2e-3 + 1e-30
    odiff = np.abs(got[rows] - want)
    oratio = float((odiff / budget).max()) if len(rows) else 0.0
    assert (odiff <= budget).all(), (what, "vs oracle", oratio)
    print(f"{what}: error / bound {float(ratio.max()):.3f} (exact operands), {oratio:.2e} (oracle)")
    return float(ratio.max()), oratio


def coherent_row(t, raw, k):
    """weight row 0, scaled to the size of a normal activation: its output sums k positive terms, so a rounding biased toward zero
    adds up there instead of cancelling"""
    w0 = oc.dequantize(t, raw[:oc.nbytes_for(t, k)], k)
    return w0 * np.float32(3 / np.abs(w0).max())


def run_dense(gdev, t, m, k, b, seed=0, x=None, oracle_rows=None):
    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(seed)
    raw = random_weight(t, m, k, rng, 0.02)
    if x is None:
        x = rng.standard_normal((b, k)).astype(np.float32)
        x[0] = coherent_row(t, raw, k)
    got = CudaTensor.from_cpu(raw, [m, k], t, gdev).matmul_vec(CudaTensor.new(x, [b, k], gdev))
    assert got.shape() == [b, m]
    return check_dense(t, raw, m, k, x, got.export().reshape(b, m), oracle_rows, f"{oc.TYPE_NAMES[t]} m={m} k={k} b={b}")


@pytest.mark.parametrize("t", DENSE_TYPES_Q8_0)
def test_prefill_dense_small_tiles(gdev, t):
    # one 128-row weight tile, N tile of 64 with a ragged batch (40 of 64 rows) and k = 4 stages exactly / more than the ring
    run_dense(gdev, t, 128, 256, 40, seed=10 + t)
    run_dense(gdev, t, 128, 1024, 64, seed=20 + t)


@pytest.mark.parametrize("t", DENSE_TYPES_Q8_K)
def test_prefill_dense_k_quants(gdev, t):
    # K-quant weights: the activation is quantised to Q8_K (buf_q8_k.rs:84-131) and q * d enters the GEMM
    run_dense(gdev, t, 256, 1024, 96, seed=60 + t)
    run_dense(gdev, t, 128, 4096, 64, seed=70 + t)


def test_prefill_dense_ragged_edges(gdev):
    # m not a multiple of 128 (out-of-bounds rows read as zero, stores guarded), b not a multiple of the N tile, all three N tiles
    run_dense(gdev, oc.Q8_0, 200, 512, 100, seed=31)       # N tile 128
    run_dense(gdev, oc.Q8_0, 333, 512, 250, seed=32)       # N tile 256, ragged
    run_dense(gdev, oc.Q8_0, 96, 4096, 33, seed=33)        # fewer rows than one tile


@pytest.mark.parametrize("b", [32, 63, 64, 65, 95, 96, 191, 192, 255, 256, 257])
def test_prefill_dense_batch_edges(gdev, b):
    # the dense threshold (32), every N-tile switch (64 below 96, 128 below 192, 256 from there) and ragged last N tiles
    run_dense(gdev, oc.Q8_0, 192, 320, b, seed=1000 + b)


@pytest.mark.parametrize("m", [1, 63, 64, 65, 127, 128, 129])
def test_prefill_dense_row_edges(gdev, m):
    # the 64-row half tile of one consumer warpgroup, and ragged 128-row CTA tiles
    run_dense(gdev, oc.Q8_0, m, 256, 70, seed=2000 + m)


@pytest.mark.parametrize("t,k", [(oc.Q8_0, 64), (oc.Q8_0, 128), (oc.Q8_0, 256), (oc.Q8_0, 320), (oc.Q8_0, 14336),
                                 (oc.Q4_K, 256), (oc.Q6_K, 14336)])
def test_prefill_dense_k_blocks(gdev, t, k):
    # fewer k-blocks than ring stages (1, 2), exactly the 4 stages, one past them, and 224 k-blocks (56 ring wraps)
    run_dense(gdev, t, 130, k, 70, seed=3000 + k + t)


@pytest.mark.parametrize("t", [oc.Q8_0, oc.Q4_0])
def test_prefill_dense_7b_shapes(gdev, t):
    # Llama-2-7B / Mistral-7B row lengths; enough tiles to wrap the 4-stage ring many times (k = 11008 -> 172 k-blocks)
    run_dense(gdev, t, 512, 4096, 256, seed=40 + t)
    run_dense(gdev, t, 256, 11008, 192, seed=50 + t)


def test_prefill_dense_256_row_cta_tiles(gdev):
    # several 128-row CTA tiles (one 64-row half per consumer warpgroup) with a ragged last tile (1000 = 7 x 128 + 104) and all three
    # N tiles (64, 128, 256 batch rows)
    run_dense(gdev, oc.Q8_0, 640, 512, 64, seed=81)
    run_dense(gdev, oc.Q8_0, 1000, 1024, 130, seed=82)
    run_dense(gdev, oc.Q4_0, 1024, 2048, 300, seed=83)


def sample_rows(b, rng, tile=256):
    """the first and last row and two random rows of every 256-row N tile"""
    rows = set()
    for n0 in range(0, b, tile):
        n1 = min(b, n0 + tile)
        rows.update([n0, n1 - 1])
        rows.update(rng.integers(n0, n1, 2).tolist())
    return np.array(sorted(rows))


# the matrices bench.py's prefill workloads time: (model, weight name, tensor id in runner.synthetic_weights order, batch).  Llama-2-7B's
# wq is Mistral-7B's (same shape, seed and tensor id), so it is not repeated.
BENCH_MATRICES = [("MISTRAL_7B", "wq", 1, 4096), ("MISTRAL_7B", "wk", 2, 4096), ("MISTRAL_7B", "wk", 2, 4097),
                  ("MISTRAL_7B", "ffn_up", 6, 4096), ("MISTRAL_7B", "ffn_down", 7, 4096),
                  ("LLAMA2_7B", "wk", 2, 4096),
                  ("LLAMA2_7B", "ffn_up", 6, 4096), ("LLAMA2_7B", "ffn_down", 7, 4096)]


@pytest.mark.parametrize("model,name,tid,b", BENCH_MATRICES)
def test_prefill_benchmark_shapes(gdev, model, name, tid, b):
    """Synthetic Q8_0 weights of the benchmarked models at b = 4096 prompt rows (16 N tiles of 256) and once at 4097 (a 17th tile of one
    row): every output of a sample of batch rows that covers each CTA tile's first and last row"""
    from crabml_b200 import CudaTensor
    from crabml_b200 import runner as R
    from oracle.synth import synth_weight
    conf = getattr(R, model)
    dim, hid, kv = conf.embedding_dim, conf.hidden_dim, conf.head_size() * conf.n_kv_heads
    m, k = {"wq": (dim, dim), "wk": (kv, dim), "ffn_up": (hid, dim), "ffn_down": (dim, hid)}[name]
    t, seed = oc.Q8_0, 0x5EED
    scale = R.synth_scale(t, k)
    rng = np.random.default_rng(b + tid)
    raw = synth_weight(t, m, k, seed, tid, scale)
    x = rng.standard_normal((b, k), dtype=np.float32)
    x[0] = coherent_row(t, raw, k)
    w = CudaTensor.synth([m, k], t, gdev, seed, tid, scale)
    got = w.matmul_vec(CudaTensor.new(x, [b, k], gdev)).export().reshape(b, m)
    del w
    rows = sample_rows(b, rng)
    check_dense(t, raw, m, k, x[rows], got[rows], what=f"{model} {name} m={m} k={k} b={b} ({len(rows)} rows)")


def test_prefill_small_batches_keep_the_exact_block_path(gdev):
    """b below the dense threshold, weight types without a dense path (Q8_1 partners, F16) and k not a multiple of 64 all take the
    per-row quantised dot (1e-6 * sum|terms| parity, test_gpu_matvec.py)"""
    from crabml_b200 import CudaTensor
    from tests.test_gpu_matvec import run_case
    run_case(gdev, oc.Q8_0, 33, 1024, b=3, seed=301)
    run_case(gdev, oc.Q4_1, 33, 1024, b=40, seed=302)
    run_case(gdev, oc.Q5_1, 33, 1024, b=40, seed=303)
    run_case(gdev, oc.Q8_0, 33, 288, b=40, seed=304)           # 9 blocks of 32: not a whole 64-wide k-block
    rng = np.random.default_rng(305)
    m, k, b = 33, 1024, 40
    w = rng.standard_normal((m, k)).astype(np.float16)
    x = rng.standard_normal((b, k)).astype(np.float32)
    got = CudaTensor.from_cpu(w, [m, k], oc.F16, gdev).matmul_vec(CudaTensor.new(x, [b, k], gdev)).export().reshape(b, m)
    want = oc.gemv(oc.F16, w.view(np.uint16), m, k, x).reshape(b, m)
    budget = np.abs(x.astype(np.float16).astype(np.float64)) @ np.abs(w.astype(np.float64)).T * 1e-6
    assert (np.abs(got.astype(np.float64) - want) <= budget).all(), float((np.abs(got - want) / budget).max())


@pytest.mark.parametrize("t", oc.QUANT_TYPES)
def test_prefill_exact_order_bit_identical(t):
    """exact_order mode never takes the tensor cores: a batch of 40 rows is bit-identical to the reference's gemv"""
    from crabml_b200 import CudaTensor
    with fresh_device(exact_order=True) as dev:
        rng = np.random.default_rng(600 + t)
        m, k, b = 19, 512, 40
        raw = random_weight(t, m, k, rng)
        x = rng.standard_normal((b, k)).astype(np.float32)
        got = CudaTensor.from_cpu(raw, [m, k], t, dev).matmul_vec(CudaTensor.new(x, [b, k], dev)).export()
        want = oc.gemv(t, raw, m, k, x).reshape(-1)
        assert_same_bits(got, want, oc.TYPE_NAMES[t])


def dense_once(t, raw, m, k, x, **dev_kw):
    """the (b, m) result of one batched matmul_vec on a fresh device"""
    from crabml_b200 import CudaTensor
    with fresh_device(**dev_kw) as dev:
        return CudaTensor.from_cpu(raw, [m, k], t, dev).matmul_vec(CudaTensor.new(x, list(x.shape), dev)).export()


@pytest.mark.parametrize("t", [oc.Q8_0, oc.Q4_K])
def test_prefill_lazy_modes_match_eager(t):
    """lazy modes 1 and 2 run a batched matmul_vec through their own dense step (lazy.cu L_MATVEC) with the eager bits, in a plan that
    is never captured into a graph"""
    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(700 + t)
    m, k, b = 200, 1024, 96
    raw = random_weight(t, m, k, rng, 0.02)
    x = rng.standard_normal((b, k)).astype(np.float32)
    eager = dense_once(t, raw, m, k, x)

    def body(dev):
        w = CudaTensor.from_cpu(raw, [m, k], t, dev)
        xt = CudaTensor.new(x, [b, k], dev)
        outs, uncached = [], []
        for _ in range(2):
            u0 = dev.lazy_stats()["uncached"]
            outs.append(w.matmul_vec(xt).export())
            uncached.append(dev.lazy_stats()["uncached"] - u0)
        return outs, uncached
    res = run_modes(body, modes=(1, 2))
    for lazy in (1, 2):
        assert res[lazy][1] == [1, 1], (lazy, "uncached flushes", res[lazy][1])
        assert_same_bits(res[lazy][0], [eager, eager], f"lazy={lazy} {oc.TYPE_NAMES[t]} vs eager")


def test_prefill_cached_weights_and_row_views(gdev):
    """The f16 copy of a full weight is made on the first dense call and reused; a prefix-of-rows view (resize(0, m')) never uses it and
    goes through the scratch buffer instead.  Every result is bit-identical to the same call on a fresh device, and a view's outputs
    are bit-identical to the first m' outputs of the full matrix (an output depends only on its own row and column)."""
    from crabml_b200 import CudaTensor
    t, m, k, b = oc.Q8_0, 300, 1024, 80
    rng = np.random.default_rng(800)
    raw = random_weight(t, m, k, rng, 0.02)
    x = rng.standard_normal((b, k)).astype(np.float32)
    full_fresh = dense_once(t, raw, m, k, x).reshape(b, m)
    views = (64, 200)
    view_fresh = {mv: dense_once(t, raw[:oc.nbytes_for(t, mv * k)], mv, k, x).reshape(b, mv) for mv in views}
    for mv in views:
        assert_same_bits(view_fresh[mv], full_fresh[:, :mv], f"rows [0, {mv}) vs the full matrix")
    with fresh_device() as dev:
        w = CudaTensor.from_cpu(raw, [m, k], t, dev)
        xt = CudaTensor.new(x, [b, k], dev)
        before = {mv: w.resize(0, mv).matmul_vec(xt).export().reshape(b, mv) for mv in views}     # scratch grows from 64 to 200 rows
        first = w.matmul_vec(xt).export().reshape(b, m)                                            # makes the cached f16 copy
        second = w.matmul_vec(xt).export().reshape(b, m)                                           # reuses it
        after = {mv: w.resize(0, mv).matmul_vec(xt).export().reshape(b, mv) for mv in views[::-1]}
        assert_same_bits((first, second), (full_fresh, full_fresh), "first and second call vs a fresh device")
        for mv in views:
            assert_same_bits((before[mv], after[mv]), (view_fresh[mv], view_fresh[mv]), f"view of {mv} rows before and after vs a fresh device")
        check_dense(t, raw, m, k, x, second, what="cached weight, second call")


def test_prefill_scratch_regrowth(gdev):
    """The activation scratch grows when a larger batch follows (pg_ensure frees and reallocates it) and is reused when a smaller one
    follows: both orders are bit-identical to fresh devices"""
    from crabml_b200 import CudaTensor
    t, m, k = oc.Q4_K, 130, 2048
    rng = np.random.default_rng(900)
    raw = random_weight(t, m, k, rng, 0.02)
    xs = {b: rng.standard_normal((b, k)).astype(np.float32) for b in (40, 1000)}
    fresh = {b: dense_once(t, raw, m, k, x) for b, x in xs.items()}
    for order in ((40, 1000, 40), (1000, 40, 1000)):
        with fresh_device() as dev:
            w = CudaTensor.from_cpu(raw, [m, k], t, dev)
            for b in order:
                assert_same_bits(w.matmul_vec(CudaTensor.new(xs[b], [b, k], dev)).export(), fresh[b], (order, b))
    check_dense(t, raw, m, k, xs[1000], fresh[1000].reshape(1000, m), what="Q4_K b=1000")


def range_rows(k, rng):
    """(rows, tiny) activation rows across the range: zero rows; 1e4-sized 32-element blocks beside 1e-3-sized ones; tiny rows whose
    f16 operands are subnormal; rows whose largest element, alone or as the scale of the whole row, is 6.55e4, 65504 (the largest f16),
    1e5 and 8e6 -- at and above the f16 range, where the unscaled operand q * d would overflow to inf"""
    rows, tiny = [], []
    rows += [np.zeros(k, np.float32)] * 2
    for _ in range(2):
        r = 1e-3 * rng.standard_normal(k)
        for blk in rng.choice(k // 32, 3, replace=False):
            r[blk * 32:(blk + 1) * 32] = 1e4 * rng.standard_normal(32)
        rows.append(r)
    for s in (1e-5, 2e-6):
        tiny.append(len(rows))
        rows.append(s * rng.standard_normal(k))
    for v in (6.55e4, 65504.0, 1e5, 8e6):
        r = rng.standard_normal(k)
        r[rng.integers(k)] = v * rng.choice([-1.0, 1.0])
        rows.append(r)
        r = rng.standard_normal(k)
        rows.append(r * (v / np.abs(r).max()))
    rows += [rng.standard_normal(k) for _ in range(40 - len(rows))]
    return np.stack(rows).astype(np.float32), tiny


@pytest.mark.parametrize("t", [oc.Q8_0, oc.Q4_0, oc.Q4_K, oc.Q6_K])
def test_prefill_activation_range(gdev, t):
    """Zero, mixed-scale, subnormal and out-of-f16-range activation rows, with Q8_0 and Q8_K partners: every output is finite and within
    both bounds (the oracle bound is not meant for rows whose operands lose bits to f16 subnormals).  Rows whose largest |q * d| reaches
    2^15 enter the GEMM scaled by a power of two (prefill_gemm.cu); without that scale f16(q * d) is inf and the whole output row is
    inf or NaN."""
    k = 1024
    rng = np.random.default_rng(1100 + t)
    x, tiny = range_rows(k, rng)
    b = x.shape[0]
    run_dense(gdev, t, 192, k, b, seed=1200 + t, x=x, oracle_rows=[r for r in range(b) if r not in tiny])
