"""Per-phase parity of the megakernel (VERDICT r1, item 1b): one Llama-2-7B-shaped decode layer driven through the trait mirror in
lazy mode 2 with debug taps (`with_name`, cpu_tensor.rs:232-241 -- the reference's own cross-backend check works the same way,
llama2.rs:768-784).  A tap forces a flush, so the token is cut into several megakernel launches whose outputs are visible:

 * FINE taps (after every stage): each stage is checked against the oracle fed THE SAME INPUT (the GPU's own previous tap), so the
   truncating quantiser cannot amplify upstream noise -- matvec stages within 1e-6 * sum|terms|, residual adds exactly, norm /
   attention / silu stages within one LUT bucket.
 * COARSE taps (only where the decode layer's fused phases end: q/k/v, x after wo + residual, h after gate/up + silu*mul, x after
   down + residual): the phases now run with their fused prologues and epilogues, and every tap must equal the fine run BIT FOR BIT."""
from dataclasses import dataclass

import numpy as np
import pytest

from oracle import oracle as oc
from oracle.synth import synth_weight
from oracle.tensor_ref import OracleDevice, OracleTensor
from crabml_b200.tensor import MEGA_RING
from tests.gpu_common import make_device
from tests.test_gpu_qwen2 import SPLIT_FROM

pytestmark = pytest.mark.gpu

SEED = 0x7A95


@dataclass(frozen=True)
class Shape:
    """one decode layer: Llama-2-7B by default; `bias` adds q/k/v biases after the matvecs (Qwen2, llama2.rs:315-317)"""
    heads: int = 32
    n_kv: int = 32
    hd: int = 128
    hid: int = 11008
    vocab: int = 32000
    bias: bool = False
    rope_mode: int = 0                  # 0: llama (adjacent pairs), 1: neox (pairs (j, j + rope_dim / 2))
    rope_dim: int = 128
    eps: float = 1e-5                   # of the attention norm; the ffn norm's is the reference's literal 1e-5

    @property
    def dim(self):
        return self.heads * self.hd


LLAMA = Shape()


def build(T, dev, wt, synth, sh=LLAMA):
    rng = np.random.default_rng(SEED)
    D, KVD = sh.dim, sh.n_kv * sh.hd
    nw = lambda: T.from_cpu((1.0 + 0.05 * rng.standard_normal(D)).astype(np.float32), [D], oc.F32, dev)      # noqa: E731
    w = {k: synth(rows, cols, i + 1) for i, (k, rows, cols) in enumerate(
        [("embed", sh.vocab, D), ("wq", D, D), ("wk", KVD, D), ("wv", KVD, D), ("wo", D, D), ("gate", sh.hid, D), ("up", sh.hid, D), ("down", D, sh.hid)])}
    w["rms_att"], w["rms_ffn"] = nw(), nw()
    if sh.bias:
        for k, n in (("bq", D), ("bk", KVD), ("bv", KVD)):
            w[k] = T.from_cpu((0.5 * rng.standard_normal(n)).astype(np.float32), [n], oc.F32, dev)
    return w


def layer(T, dev, w, kc, vc, token, pos, tap, sh=LLAMA):
    """One decode layer in the reference's op order (llama2.rs:213-281, 283-352, 527-638); tap(name, tensor) returns the tensor."""
    D, H, KV, HD = sh.dim, sh.heads, sh.n_kv, sh.hd
    x = T.alloc([1, D], oc.F32, dev)
    x.copy_rows_from(w["embed"], [token])
    x = tap("x0", x)
    x_orig = x.dup()
    x = x.rms_norm_inplace(sh.eps).mul_inplace(w["rms_att"])
    x = tap("xn", x)
    q, k, v = w["wq"].matmul_vec(x), w["wk"].matmul_vec(x), w["wv"].matmul_vec(x)
    q, k, v = tap("q", q), tap("k", k), tap("v", v)
    if sh.bias:
        q, k, v = q.add_inplace(w["bq"]), k.add_inplace(w["bk"]), v.add_inplace(w["bv"])
        q, k, v = tap("qb", q), tap("kb", k), tap("vb", v)
    q = tap("qr", q.reshape([1, H, HD]).rope_inplace(sh.rope_mode, pos, sh.rope_dim))
    k = tap("kr", k.reshape([1, KV, HD]).rope_inplace(sh.rope_mode, pos, sh.rope_dim))
    kc.concatenate(k.reshape([1, KV, HD]).transpose([1, 0, 2]), 1)
    vc.concatenate(v.reshape([1, KV, HD]).transpose([1, 0, 2]), 1)
    q = q.reshape([1, H, HD]).transpose([1, 0, 2]).contiguous().scale_inplace(1.0 / np.sqrt(np.float32(HD)))
    att = q.batch_matmul(kc.transpose([0, 2, 1])).softmax_inplace(2)
    a = att.batch_matmul(vc).reshape([1, D])
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


def cache_fill(sh, step, n):
    """[2, n_kv, n, hd] rows that fill the K and V caches before step `step`: f16 values, so an f16 cache holds them exactly"""
    rng = np.random.default_rng(SEED + 1 + step)
    return rng.standard_normal((2, sh.n_kv, n, sh.hd)).astype(np.float16).astype(np.float32)


def positions(steps):
    """steps: [(rows filled into the caches first, token)] -> the position each token decodes at"""
    pos, out = 0, []
    for n, _ in steps:
        pos += n
        out.append(pos)
        pos += 1
    return out


def cache_len(steps):
    """rows allocated per KV cache: 8 at least, as for the Llama layer's three positions"""
    return max(8, positions(steps)[-1] + 1)


def gpu_run(wt, steps, names, sh=LLAMA, kv_type=oc.F32):
    """-> ({step: {tap: values}}, lazy stats, persistent kernel variant) for the taps in `names` (others are not tapped, i.e. do
    not cut the plan)"""
    from crabml_b200 import CudaTensor
    from crabml_b200 import runner as R
    dev = make_device(lazy=2, debug_named_tensors=True)
    try:
        w = build(CudaTensor, dev, wt, lambda r, c, tid: CudaTensor.synth([r, c], wt, dev, SEED, tid, R.synth_scale(wt, c)), sh)
        cap = cache_len(steps)
        kc = CudaTensor.alloc([sh.n_kv, cap, sh.hd], kv_type, dev).resize(1, 0)
        vc = CudaTensor.alloc([sh.n_kv, cap, sh.hd], kv_type, dev).resize(1, 0)
        out = {}
        for i, ((n, t), pos) in enumerate(zip(steps, positions(steps))):
            if n:
                f = cache_fill(sh, i, n)
                kc.concatenate(CudaTensor.new(f[0].reshape(-1), [sh.n_kv, n, sh.hd], dev), 1)
                vc.concatenate(CudaTensor.new(f[1].reshape(-1), [sh.n_kv, n, sh.hd], dev), 1)

            def tap(name, x):
                return x.with_name(f"{name}:{pos}") if name in names else x
            layer(CudaTensor, dev, w, kc, vc, t, pos, tap, sh).export()
            out[i] = {n: dev.dump_debug_tensor(f"{n}:{pos}").copy() for n in names}
        return out, dev.lazy_stats(), dev.mega_variant()
    finally:
        dev.close()


FINE = ["x0", "xn", "q", "k", "v", "att", "o", "x1", "hn", "g", "u", "h", "y", "x2"]
COARSE = ["x0", "q", "k", "v", "x1", "h", "x2"]


def assert_coarse_equals_fine(wt, coarse, fine, names):
    for i in fine:
        for n in names:
            np.testing.assert_array_equal(coarse[i][n].view(np.uint32), fine[i][n].view(np.uint32), err_msg=f"{oc.TYPE_NAMES[wt]} step {i} tap {n}")


def check_fine_vs_oracle(wt, fine, steps, sh=LLAMA, kv_type=oc.F32):
    """every fine tap against the oracle fed the GPU's own inputs"""
    from crabml_b200 import runner as R
    D, H, KV, HD = sh.dim, sh.heads, sh.n_kv, sh.hd
    odev = OracleDevice()
    raw = {}

    def osyn(r, c, tid):
        raw[tid] = (synth_weight(wt, r, c, SEED, tid, R.synth_scale(wt, c)), r, c)
        return OracleTensor.from_cpu(raw[tid][0], [r, c], wt, odev)
    ow = build(OracleTensor, odev, wt, osyn, sh)
    ids = {"embed": 1, "wq": 2, "wk": 3, "wv": 4, "wo": 5, "gate": 6, "up": 7, "down": 8}
    at = oc.rhs_type(wt)
    absw = {}                   # |dequantised weight|, once per matrix

    def matvec_check(name_w, x, got, what):
        blocks, m, k = raw[ids[name_w]]
        want = oc.gemv(wt, blocks, m, k, x)
        if name_w not in absw:
            absw[name_w] = np.abs(oc.dequantize(wt, blocks, m * k).reshape(m, k)).astype(np.float64)
        ad = np.abs(oc.dequantize(at, oc.quantize(at, x), k)).astype(np.float64)
        budget = (absw[name_w] @ ad) * 1e-6 + 1e-30
        diff = np.abs(got.astype(np.float64) - want.astype(np.float64))
        assert (diff <= budget).all(), (oc.TYPE_NAMES[wt], what, float((diff / budget).max()))
        return float((diff / budget).max())

    cap = cache_len(steps)
    okc = OracleTensor.alloc([KV, cap, HD], kv_type, odev).resize(1, 0)
    ovc = OracleTensor.alloc([KV, cap, HD], kv_type, odev).resize(1, 0)
    qn, kn, vn = ("qb", "kb", "vb") if sh.bias else ("q", "k", "v")
    for i, ((n, t), pos) in enumerate(zip(steps, positions(steps))):
        f = fine[i]
        if n:
            fill = cache_fill(sh, i, n)
            okc.concatenate(OracleTensor.new(fill[0].reshape(-1), [KV, n, HD], odev), 1)
            ovc.concatenate(OracleTensor.new(fill[1].reshape(-1), [KV, n, HD], odev), 1)
        # embedding row: bit-exact block unpack
        want = OracleTensor.alloc([1, D], oc.F32, odev)
        want.copy_rows_from(ow["embed"], [t])
        np.testing.assert_array_equal(f["x0"].view(np.uint32), want.export().view(np.uint32))
        # norm stages: same input, f32 tree vs sequential sum of squares
        for src, dst, wn, eps in (("x0", "xn", "rms_att", sh.eps), ("x1", "hn", "rms_ffn", 1e-5)):
            want = OracleTensor.new(f[src], [1, D], odev).rms_norm_inplace(eps).mul_inplace(ow[wn]).export()
            np.testing.assert_allclose(f[dst], want, rtol=2e-6, atol=1e-7, err_msg=f"pos {pos} {dst}")
        mv = max(matvec_check(name_w, f[src], f[dst], f"pos {pos} {dst}") for name_w, src, dst in (
            ("wq", "xn", "q"), ("wk", "xn", "k"), ("wv", "xn", "v"), ("wo", "att", "o"), ("gate", "hn", "g"), ("up", "hn", "u"), ("down", "h", "y")))
        # bias and residual adds: exact
        if sh.bias:
            for src, dst, b in (("q", "qb", "bq"), ("k", "kb", "bk"), ("v", "vb", "bv")):
                np.testing.assert_array_equal(f[dst].view(np.uint32), (f[src] + ow[b].export()).view(np.uint32), err_msg=f"pos {pos} {dst}")
        np.testing.assert_array_equal(f["x1"].view(np.uint32), (f["o"] + f["x0"]).view(np.uint32))
        np.testing.assert_array_equal(f["x2"].view(np.uint32), (f["y"] + f["x1"]).view(np.uint32))
        # attention from the GPU's q, k, v (the oracle's cache holds the GPU's earlier k, v: rope is bit-exact)
        oq = OracleTensor.new(f[qn], [1, H, HD], odev).rope_inplace(sh.rope_mode, pos, sh.rope_dim)
        ok = OracleTensor.new(f[kn], [1, KV, HD], odev).rope_inplace(sh.rope_mode, pos, sh.rope_dim)
        for got, want, name in (("qr", oq, "q"), ("kr", ok, "k")):
            if got in f:
                np.testing.assert_array_equal(f[got].view(np.uint32), want.export().view(np.uint32), err_msg=f"pos {pos} rope of {name}")
        okc.concatenate(ok.reshape([1, KV, HD]).transpose([1, 0, 2]), 1)
        ovc.concatenate(OracleTensor.new(f[vn], [1, KV, HD], odev).transpose([1, 0, 2]), 1)
        oq = oq.transpose([1, 0, 2]).contiguous().scale_inplace(1.0 / np.sqrt(np.float32(HD)))
        want = oq.batch_matmul(okc.transpose([0, 2, 1])).softmax_inplace(2).batch_matmul(ovc).reshape([1, D]).export()
        err, bound = float(np.abs(f["att"] - want).max()), 2e-3 * float(np.abs(want).max()) + 1e-7
        assert err <= bound, (pos, err)
        print(f"{oc.TYPE_NAMES[wt]} {sh.heads}/{sh.n_kv} heads rope {sh.rope_mode}:{sh.rope_dim} kv {oc.TYPE_NAMES[kv_type]} pos {pos}: "
              f"matvecs at {mv:.3f} and attention at {err / bound:.3f} of their bounds")
        # silu(gate) * up through the f16 exp LUT: within one LUT bucket of the oracle on the same g, u
        want = OracleTensor.new(f["g"], [1, sh.hid], odev).silu_inplace().mul_inplace(OracleTensor.new(f["u"], [1, sh.hid], odev)).export()
        np.testing.assert_array_equal(f["h"].view(np.uint32), want.view(np.uint32), err_msg=f"pos {pos} silu*mul is elementwise: exact")


@pytest.mark.parametrize("wt", [oc.Q8_0, oc.Q4_0, oc.Q2_K, oc.Q3_K, oc.Q4_K, oc.Q5_K, oc.Q6_K, oc.Q8_K])
def test_megakernel_phase_taps_vs_oracle_on_the_same_inputs(wt):
    steps = [(0, 1), (0, 31999), (0, 777)]
    fine, _, _ = gpu_run(wt, steps, FINE)
    coarse, st, _ = gpu_run(wt, steps, COARSE)
    assert st["uncached"] == 0
    # ---- coarse (fused phases) == fine (split phases), bit for bit ----
    assert_coarse_equals_fine(wt, coarse, fine, COARSE)
    # ---- fine taps vs the oracle fed the GPU's own inputs ----
    check_fine_vs_oracle(wt, fine, steps)


# ---- a Qwen2-7B layer: q/k/v biases, Neox RoPE (full and partial), 28 heads on 4 kv heads, long caches ----------------------------
FINE_QWEN2 = ["x0", "xn", "q", "k", "v", "qb", "kb", "vb", "qr", "kr", "att", "o", "x1", "hn", "g", "u", "h", "y", "x2"]
COARSE_QKV = ["x0", "qb", "kb", "vb", "x1", "h", "x2"]          # q/k/v after the ring kernel's fused bias epilogue; attention + wo fused
COARSE_ATT = ["x0", "att", "x1", "h", "x2"]                    # the ring kernel's Neox attention phase, in one flush with the q/k/v phase


@pytest.mark.parametrize("wt", [oc.Q8_0, oc.Q4_0])
@pytest.mark.parametrize("rope_dim", [128, 64])
@pytest.mark.parametrize("kv_type", [oc.F32, oc.F16])
def test_qwen2_layer_phase_taps_vs_oracle_on_the_same_inputs(wt, rope_dim, kv_type):
    """A Qwen2-7B decode layer (dim 3584, GQA group 7, hidden 18944, biases of sigma 0.5) at two steps: one whose attention covers
    fewer than SPLIT_FROM cached positions, one past it, the caches filled with random rows in between.  The fine run taps every stage
    (its RoPE and attention then run as the per-op kernels): each is checked against the oracle on the same input, the bias adds and the
    Neox RoPE bit for bit.  The coarse runs cut the layer only where the ring kernel's fused phases end, and equal the fine run bit for
    bit."""
    sh = Shape(heads=28, n_kv=4, hid=18944, bias=True, rope_mode=1, rope_dim=rope_dim, eps=1e-6)
    steps = [(SPLIT_FROM - 20, 1), (40, 31999)]
    assert positions(steps)[0] + 1 < SPLIT_FROM < positions(steps)[1]
    fine, _, _ = gpu_run(wt, steps, FINE_QWEN2, sh, kv_type)
    for names in (COARSE_QKV, COARSE_ATT):
        coarse, _, variant = gpu_run(wt, steps, names, sh, kv_type)
        assert variant == MEGA_RING
        assert_coarse_equals_fine(wt, coarse, fine, names)
    check_fine_vs_oracle(wt, fine, steps, sh, kv_type)
