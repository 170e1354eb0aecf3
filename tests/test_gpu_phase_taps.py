"""Per-phase parity of the megakernel (VERDICT r1, item 1b): one Llama-2-7B-shaped decode layer driven through the trait mirror in
lazy mode 2 with debug taps (`with_name`, cpu_tensor.rs:232-241 -- the reference's own cross-backend check works the same way,
llama2.rs:768-784).  A tap forces a flush, so the token is cut into several megakernel launches whose outputs are visible:

 * FINE taps (after every stage): each stage is checked against the oracle fed THE SAME INPUT (the GPU's own previous tap), so the
   truncating quantiser cannot amplify upstream noise -- matvec stages within 1e-6 * sum|terms|, residual adds exactly, norm /
   attention / silu stages within one LUT bucket.
 * COARSE taps (only where the decode layer's fused phases end: q/k/v, x after wo + residual, h after gate/up + silu*mul, x after
   down + residual): the phases now run with their fused prologues and epilogues, and every tap must equal the fine run BIT FOR BIT."""
import numpy as np
import pytest

from oracle import oracle as oc
from oracle.synth import synth_weight
from oracle.tensor_ref import OracleDevice, OracleTensor
from tests.gpu_common import make_device

pytestmark = pytest.mark.gpu

DIM, HID, HEADS, HD, VOCAB = 4096, 11008, 32, 128, 32000
SEED = 0x7A95


def build(T, dev, wt, synth):
    from crabml_b200 import runner as R
    rng = np.random.default_rng(SEED)
    nw = lambda: T.from_cpu((1.0 + 0.05 * rng.standard_normal(DIM)).astype(np.float32), [DIM], oc.F32, dev)      # noqa: E731
    w = {k: synth(rows, cols, i + 1) for i, (k, rows, cols) in enumerate(
        [("embed", VOCAB, DIM), ("wq", DIM, DIM), ("wk", DIM, DIM), ("wv", DIM, DIM), ("wo", DIM, DIM), ("gate", HID, DIM), ("up", HID, DIM), ("down", DIM, HID)])}
    w["rms_att"], w["rms_ffn"] = nw(), nw()
    return w


def layer(T, dev, w, kc, vc, token, pos, tap):
    """One decode layer in the reference's op order (llama2.rs:213-281, 527-638); tap(name, tensor) returns the tensor."""
    x = T.alloc([1, DIM], oc.F32, dev)
    x.copy_rows_from(w["embed"], [token])
    x = tap("x0", x)
    x_orig = x.dup()
    x = x.rms_norm_inplace(1e-5).mul_inplace(w["rms_att"])
    x = tap("xn", x)
    q, k, v = w["wq"].matmul_vec(x), w["wk"].matmul_vec(x), w["wv"].matmul_vec(x)
    q, k, v = tap("q", q), tap("k", k), tap("v", v)
    q = q.reshape([1, HEADS, HD]).rope_inplace(0, pos, HD)
    k = k.reshape([1, HEADS, HD]).rope_inplace(0, pos, HD)
    kc.concatenate(k.reshape([1, HEADS, HD]).transpose([1, 0, 2]), 1)
    vc.concatenate(v.reshape([1, HEADS, HD]).transpose([1, 0, 2]), 1)
    q = q.reshape([1, HEADS, HD]).transpose([1, 0, 2]).contiguous().scale_inplace(1.0 / np.sqrt(np.float32(HD)))
    att = q.batch_matmul(kc.transpose([0, 2, 1])).softmax_inplace(2)
    a = att.batch_matmul(vc).reshape([1, DIM])
    del q, k, v, att          # like the moves of the Rust / C++ runner: the fuser only folds intermediates nobody else can observe
    a = tap("att", a)
    o = w["wo"].matmul_vec(a)
    o = tap("o", o)
    x = o.add_inplace(x_orig)
    x = tap("x1", x)
    x_orig2 = x.dup()
    x = x.rms_norm_inplace(1e-5).mul_inplace(w["rms_ffn"])
    x = tap("hn", x)
    g, u = w["gate"].matmul_vec(x), w["up"].matmul_vec(x)
    g, u = tap("g", g), tap("u", u)
    h = g.silu_inplace().mul_inplace(u)
    del g, u
    h = tap("h", h)
    y = w["down"].matmul_vec(h)
    y = tap("y", y)
    x = y.add_inplace(x_orig2)
    return tap("x2", x)


def gpu_run(wt, tokens, names):
    """-> {pos: {tap: values}} for the taps in `names` (others are not tapped, i.e. do not cut the plan)"""
    from crabml_b200 import CudaTensor
    from crabml_b200 import runner as R
    dev = make_device(lazy=2, debug_named_tensors=True)
    try:
        w = build(CudaTensor, dev, wt, lambda r, c, tid: CudaTensor.synth([r, c], wt, dev, SEED, tid, R.synth_scale(wt, c)))
        kc = CudaTensor.alloc([HEADS, 8, HD], oc.F32, dev).resize(1, 0)
        vc = CudaTensor.alloc([HEADS, 8, HD], oc.F32, dev).resize(1, 0)
        out = {}
        for pos, t in enumerate(tokens):
            def tap(name, x):
                return x.with_name(f"{name}:{pos}") if name in names else x
            layer(CudaTensor, dev, w, kc, vc, t, pos, tap).export()
            out[pos] = {n: dev.dump_debug_tensor(f"{n}:{pos}").copy() for n in names}
        return out, dev.lazy_stats()
    finally:
        dev.close()


FINE = ["x0", "xn", "q", "k", "v", "att", "o", "x1", "hn", "g", "u", "h", "y", "x2"]
COARSE = ["x0", "q", "k", "v", "x1", "h", "x2"]


@pytest.mark.parametrize("wt", [oc.Q8_0, oc.Q4_0, oc.Q2_K, oc.Q3_K, oc.Q4_K, oc.Q5_K, oc.Q6_K, oc.Q8_K])
def test_megakernel_phase_taps_vs_oracle_on_the_same_inputs(wt):
    from crabml_b200 import runner as R
    tokens = [1, 31999, 777]
    fine, _ = gpu_run(wt, tokens, FINE)
    coarse, st = gpu_run(wt, tokens, COARSE)
    assert st["uncached"] == 0
    # ---- coarse (fused phases) == fine (split phases), bit for bit ----
    for pos in range(len(tokens)):
        for n in COARSE:
            np.testing.assert_array_equal(coarse[pos][n].view(np.uint32), fine[pos][n].view(np.uint32), err_msg=f"{oc.TYPE_NAMES[wt]} pos {pos} tap {n}")
    # ---- fine taps vs the oracle fed the GPU's own inputs ----
    odev = OracleDevice()
    raw = {}

    def osyn(r, c, tid):
        raw[tid] = (synth_weight(wt, r, c, SEED, tid, R.synth_scale(wt, c)), r, c)
        return OracleTensor.from_cpu(raw[tid][0], [r, c], wt, odev)
    ow = build(OracleTensor, odev, wt, osyn)
    ids = {"embed": 1, "wq": 2, "wk": 3, "wv": 4, "wo": 5, "gate": 6, "up": 7, "down": 8}
    at = oc.rhs_type(wt)

    def matvec_check(name_w, x, got, what):
        blocks, m, k = raw[ids[name_w]]
        want = oc.gemv(wt, blocks, m, k, x)
        wd = np.abs(oc.dequantize(wt, blocks, m * k).reshape(m, k)).astype(np.float64)
        ad = np.abs(oc.dequantize(at, oc.quantize(at, x), k)).astype(np.float64)
        budget = (wd @ ad) * 1e-6 + 1e-30
        diff = np.abs(got.astype(np.float64) - want.astype(np.float64))
        assert (diff <= budget).all(), (oc.TYPE_NAMES[wt], what, float((diff / budget).max()))

    okc = OracleTensor.alloc([HEADS, 8, HD], oc.F32, odev).resize(1, 0)
    ovc = OracleTensor.alloc([HEADS, 8, HD], oc.F32, odev).resize(1, 0)
    for pos, t in enumerate(tokens):
        f = fine[pos]
        # embedding row: bit-exact block unpack
        want = OracleTensor.alloc([1, DIM], oc.F32, odev)
        want.copy_rows_from(ow["embed"], [t])
        np.testing.assert_array_equal(f["x0"].view(np.uint32), want.export().view(np.uint32))
        # norm stages: same input, f32 tree vs sequential sum of squares
        for src, dst, wn in (("x0", "xn", "rms_att"), ("x1", "hn", "rms_ffn")):
            want = OracleTensor.new(f[src], [1, DIM], odev).rms_norm_inplace(1e-5).mul_inplace(ow[wn]).export()
            np.testing.assert_allclose(f[dst], want, rtol=2e-6, atol=1e-7, err_msg=f"pos {pos} {dst}")
        for name_w, src, dst in (("wq", "xn", "q"), ("wk", "xn", "k"), ("wv", "xn", "v"), ("wo", "att", "o"), ("gate", "hn", "g"), ("up", "hn", "u"), ("down", "h", "y")):
            matvec_check(name_w, f[src], f[dst], f"pos {pos} {dst}")
        # residual adds: exact
        np.testing.assert_array_equal(f["x1"].view(np.uint32), (f["o"] + f["x0"]).view(np.uint32))
        np.testing.assert_array_equal(f["x2"].view(np.uint32), (f["y"] + f["x1"]).view(np.uint32))
        # attention from the GPU's q, k, v (the oracle's cache holds the GPU's earlier k, v: rope is bit-exact)
        oq = OracleTensor.new(f["q"], [1, HEADS, HD], odev).rope_inplace(0, pos, HD)
        ok = OracleTensor.new(f["k"], [1, HEADS, HD], odev).rope_inplace(0, pos, HD)
        okc.concatenate(ok.reshape([1, HEADS, HD]).transpose([1, 0, 2]), 1)
        ovc.concatenate(OracleTensor.new(f["v"], [1, HEADS, HD], odev).transpose([1, 0, 2]), 1)
        oq = oq.transpose([1, 0, 2]).contiguous().scale_inplace(1.0 / np.sqrt(np.float32(HD)))
        want = oq.batch_matmul(okc.transpose([0, 2, 1])).softmax_inplace(2).batch_matmul(ovc).reshape([1, DIM]).export()
        assert np.abs(f["att"] - want).max() <= 2e-3 * np.abs(want).max() + 1e-7, (pos, float(np.abs(f["att"] - want).max()))
        # silu(gate) * up through the f16 exp LUT: within one LUT bucket of the oracle on the same g, u
        want = OracleTensor.new(f["g"], [1, HID], odev).silu_inplace().mul_inplace(OracleTensor.new(f["u"], [1, HID], odev)).export()
        np.testing.assert_array_equal(f["h"].view(np.uint32), want.view(np.uint32), err_msg=f"pos {pos} silu*mul is elementwise: exact")
