"""Decode attention past the first KV chunk, at long contexts, in every execution mode.

The megakernels do not read the KV cache directly: their attention phase (csrc/mega_phases.cuh phase_attn) streams a head's K rows,
then its V rows, through a ring of AT_NBUF = 3 shared-memory buffers of `at_ch` positions each (32 for f32 and 64 for f16 caches in
the ring kernel, 64 in the register kernel), one bulk copy per chunk, with mbarrier parity carried across heads and layers.  The
tests here put that phase, the fused single-pass kernel of the CUDA-graph mode and the eager per-op kernels at KV lengths on every
side of every chunk and buffer boundary, and at contexts where the fuser switches kernels.

1. Retrieval with an exact answer.  q, K and V are built so that each head's softmax is one-hot: head h has a single non-zero q
   coordinate, in its own column c(h) = h, scaled to a score of about 32; K holds a 1 in that column in exactly one row t per kv
   group and 0 in every other row, so every other score is exactly 0, exp LUT(0) = 1 and LUT(-32) rounds to 0 in f16.  The output
   is then one V row bit for bit.  V rows are small integers (exact in f16) that encode (group, row), so a mismatch reports which
   row of which group was read instead.  Targets sit at rows 0, at_ch - 1, at_ch, 2 at_ch - 1, 3 at_ch (the first reuse of buffer 0)
   for both chunk sizes, at kv_len - 1, and at the current token.  A second step targets row kv_len, which the first step's owner
   CTA wrote into the cache and which must now come back through a bulk copy.
2. Random data at long KV lengths: every mode equals the eager kernels bit for bit, exact_order mode equals the CPU oracle bit for
   bit, and the megakernel is within a derived bound of an f64 softmax attention with the true exp.
3. The context-length switches of lazy mode 2, found by probing: a flush with a Q8_0 matvec goes from the ring kernel to the CUDA
   graph of fused kernels, attention alone from the register kernel to the graph; and contexts past what the single-pass fused
   kernel can hold."""
import numpy as np
import pytest

from oracle import oracle as oc
from oracle.tensor_ref import OracleDevice, OracleTensor
from crabml_b200.tensor import MEGA_NONE, MEGA_REGISTER, MEGA_RING
from tests.gpu_common import MODE_DEVICE, assert_same_bits, fresh_device

CURRENT = -1                                        # target: this token's own k / v row
SCORE = 32.0                                        # the target's scaled score
MV_K, MV_M, MV_SEED = 4096, 256, 0xA77E             # the unrelated Q8_0 matvec that makes a flush take the ring kernel
MAX_LEN = 4100
KV_LENS = [1, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 191, 192, 193, 1000, 4095, MAX_LEN - 1]
HEADS = [(48, 6, 6), (64, 8, 8), (128, 32, 32), (128, 32, 8), (256, 8, 2)]      # (head_dim, n_heads, n_kv)
# rows 0, at_ch - 1, at_ch, 2 at_ch - 1 and 3 at_ch for at_ch = 32 and 64
BOUNDARY_ROWS = sorted({r for ch in (32, 64) for r in (0, ch - 1, ch, 2 * ch - 1, 3 * ch)})
# execution mode (its device: MODE_DEVICE) -> (ring matvec in the flush, expected mega_variant)
MODES = {"eager": (False, MEGA_NONE), "graph": (False, MEGA_NONE), "register": (False, MEGA_REGISTER), "ring": (True, MEGA_RING),
         "exact": (False, MEGA_NONE)}


def group_of(h, n_heads, n_kv, f16):
    """kv head read by query head h: h % n_kv for f32 caches (batch_matmul.rs:63), h / (n_heads / n_kv) for f16 (:89-91)"""
    return h // (n_heads // n_kv) if f16 else h % n_kv


def v_rows(g, rows, hd):
    """V[g][s] for s in rows: integers |v| <= 1023 (exact in f16); columns 0..2 encode (s mod 1024, s / 1024, g)"""
    s = np.asarray(rows, np.int64)[:, None]
    d = np.arange(hd, dtype=np.int64)[None, :]
    v = (s * 7 + g * 131 + d * 29) % 2047 - 1023
    v[:, 0:1] = s % 1024
    v[:, 1:2] = s // 1024
    v[:, 2:3] = g
    return v.astype(np.float32)


def decode_row(vec):
    return int(vec[2]), int(vec[0]) + 1024 * int(vec[1])


class Retrieval:
    """The construction of part 1 for one (head_dim, n_heads, n_kv, kv_len).  Column h carries head h's step-1 score; column
    n_heads + h its step-2 score, for which only the first step's own row (cache row kv_len) holds a 1.  Columns from 2 n_heads on
    hold junk that no query reads."""

    def __init__(self, hd, n_heads, n_kv, kv_len):
        assert 2 * n_heads <= hd and n_heads % n_kv == 0
        self.hd, self.n_heads, self.n_kv, self.kv_len = hd, n_heads, n_kv, kv_len
        cands = sorted({r for r in BOUNDARY_ROWS if r < kv_len} | {kv_len - 1}) + [CURRENT]
        # which rows are targets rotates with kv_len, so that over the sweep every candidate is hit by heads of every group
        self.target = np.array([cands[(h + kv_len) % len(cands)] for h in range(n_heads)])
        u = 2 * n_heads
        s = np.arange(kv_len, dtype=np.int64)[:, None]
        junk = ((s * 3 + np.arange(hd - u)[None, :] * 5) % 15 - 7).astype(np.float32)
        self.K = np.zeros((n_kv, kv_len, hd), np.float32)
        self.K[:, :, u:] = junk[None]
        self.V = np.stack([v_rows(g, range(kv_len), hd) for g in range(n_kv)]) if kv_len else np.zeros((n_kv, 0, hd), np.float32)
        self.k1 = np.zeros((n_kv, hd), np.float32)
        self.k2 = np.zeros((n_kv, hd), np.float32)
        self.k1[:, u:] = self.k2[:, u:] = junk[0] if kv_len else 1.0
        self.k1[:, n_heads:u] = 1.0                    # step 2's target: this step's row
        for h, t in enumerate(self.target):
            if t == CURRENT:
                self.k1[:, h] = 1.0                   # every group: whichever group head h reads
            else:
                self.K[:, t, h] = 1.0
        self.v1 = np.stack([v_rows(g, [kv_len], hd)[0] for g in range(n_kv)])
        self.v2 = np.stack([v_rows(g, [kv_len + 1], hd)[0] for g in range(n_kv)])
        a = np.float32(SCORE) * np.sqrt(np.float32(hd))
        self.q1 = np.zeros((n_heads, hd), np.float32)
        self.q2 = np.zeros((n_heads, hd), np.float32)
        for h in range(n_heads):
            self.q1[h, h] = a
            self.q2[h, n_heads + h] = a

    def expected(self, step, f16):
        out = np.zeros((self.n_heads, self.hd), np.float32)
        rows = []
        for h in range(self.n_heads):
            g = group_of(h, self.n_heads, self.n_kv, f16)
            t = self.kv_len if step == 2 or self.target[h] == CURRENT else int(self.target[h])
            out[h] = v_rows(g, [t], self.hd)[0]
            rows.append((g, t))
        return out, rows

    def check(self, got, step, f16, what):
        want, rows = self.expected(step, f16)
        got = got.reshape(self.n_heads, self.hd)
        bad = [h for h in range(self.n_heads) if not np.array_equal(got[h].view(np.uint32), want[h].view(np.uint32))]
        if bad:
            lines = []
            for h in bad[:6]:
                gw, sw = rows[h]
                if not got[h].any():
                    lines.append(f"head {h}: want group {gw} row {sw}, got zeros")
                elif np.array_equal(got[h], np.round(got[h])) and np.abs(got[h]).max() <= 1023:
                    gg, sg = decode_row(got[h])
                    lines.append(f"head {h}: want group {gw} row {sw}, read group {gg} row {sg}")
                else:
                    lines.append(f"head {h}: want group {gw} row {sw}, got a mixture {got[h][:4]}")
            pytest.fail(f"{what} step {step}, kv_len {self.kv_len}: {len(bad)} of {self.n_heads} heads wrong\n  " + "\n  ".join(lines))


def attention(T, dev, kc, vc, q, k, v, n_heads, n_kv, hd, pos=0):
    """One decode step's attention in the reference's op order (llama2.rs:252-256, 541-590): the pattern the fuser replaces.
    q [n_heads, hd], k / v [n_kv, hd] are host arrays; returns the [n_heads, 1, hd] output tensor (not yet exported)."""
    qt = T.new(q, [1, n_heads, hd], dev)
    kt = T.new(k, [1, n_kv, hd], dev)
    vt = T.new(v, [1, n_kv, hd], dev)
    qt = qt.rope_inplace(0, pos, hd)
    kt = kt.rope_inplace(0, pos, hd)
    kc.concatenate(kt.transpose([1, 0, 2]), 1)
    vc.concatenate(vt.transpose([1, 0, 2]), 1)
    qt = qt.transpose([1, 0, 2]).contiguous().scale_inplace(1.0 / np.sqrt(np.float32(hd)))
    att = qt.batch_matmul(kc.transpose([0, 2, 1])).softmax_inplace(2)
    out = att.batch_matmul(vc)
    del qt, kt, vt, att           # the fuser only folds intermediates nobody else can observe
    return out


def fill(T, dev, kc_full, vc_full, K, V):
    """caches of max_len rows, filled with the kv_len rows of K, V in one concatenate each"""
    n_kv, kv_len, hd = K.shape
    kc, vc = kc_full.resize(1, 0), vc_full.resize(1, 0)
    if kv_len:
        kc.concatenate(T.new(K, [n_kv, kv_len, hd], dev), 1)
        vc.concatenate(T.new(V, [n_kv, kv_len, hd], dev), 1)
    if hasattr(dev, "flush"):
        dev.flush()
    return kc, vc


# ---- CPU: the construction itself, through the oracle ---------------------------------------------------------------------------------
@pytest.mark.parametrize("f16", [False, True])
@pytest.mark.parametrize("hd,n_heads,n_kv", [(48, 6, 6), (128, 32, 8), (256, 8, 2)])
@pytest.mark.parametrize("kv_len", [1, 33, 129, 193, 300])
def test_retrieval_construction_on_the_oracle(hd, n_heads, n_kv, kv_len, f16):
    """The one-hot construction, run through the CPU oracle's trait ops (no GPU): a GPU failure of the same construction is then
    the kernel's, not the test's."""
    odev = OracleDevice()
    R = Retrieval(hd, n_heads, n_kv, kv_len)
    dt = oc.F16 if f16 else oc.F32
    kc_full, vc_full = OracleTensor.alloc([n_kv, kv_len + 2, hd], dt, odev), OracleTensor.alloc([n_kv, kv_len + 2, hd], dt, odev)
    kc, vc = fill(OracleTensor, odev, kc_full, vc_full, R.K, R.V)
    R.check(attention(OracleTensor, odev, kc, vc, R.q1, R.k1, R.v1, n_heads, n_kv, hd).export(), 1, f16, "oracle")
    R.check(attention(OracleTensor, odev, kc, vc, R.q2, R.k2, R.v2, n_heads, n_kv, hd).export(), 2, f16, "oracle")
    # and the construction is sharp: the wrong head-to-group mapping or a target one row off would be reported
    if n_kv < n_heads:
        want, _ = R.expected(1, not f16)
        assert not np.array_equal(want, R.expected(1, f16)[0])


# ---- GPU -------------------------------------------------------------------------------------------------------------------------------
def ring_matvec(dev):
    """the unrelated Q8_0 matvec (k = 4096) whose streaming phase makes lazy mode 2 pick the ring kernel"""
    from crabml_b200 import CudaTensor
    from crabml_b200 import runner as R
    W = CudaTensor.synth([MV_M, MV_K], oc.Q8_0, dev, MV_SEED, 1, R.synth_scale(oc.Q8_0, MV_K))
    x = np.random.default_rng(MV_SEED).standard_normal(MV_K).astype(np.float32)
    return W.matmul_vec(CudaTensor.new(x, [MV_K], dev))


_EAGER_MV = {}


def eager_matvec():
    if "y" not in _EAGER_MV:
        with fresh_device(lazy=0) as dev:
            _EAGER_MV["y"] = ring_matvec(dev).export()
    return _EAGER_MV["y"]


def run_retrieval(dev, mode, f16, hd, n_heads, n_kv, max_len, kv_lens, second_step=True):
    """every kv_len on one device (one max_len, one flush shape: the same kernel variant throughout)"""
    from crabml_b200 import CudaTensor
    with_mv, variant = MODES[mode]
    dt = oc.F16 if f16 else oc.F32
    kc_full = CudaTensor.alloc([n_kv, max_len, hd], dt, dev)
    vc_full = CudaTensor.alloc([n_kv, max_len, hd], dt, dev)
    outs = []
    for kv_len in kv_lens:
        R = Retrieval(hd, n_heads, n_kv, kv_len)
        kc, vc = fill(CudaTensor, dev, kc_full, vc_full, R.K, R.V)
        steps = [(R.q1, R.k1, R.v1)] + ([(R.q2, R.k2, R.v2)] if second_step and kv_len + 2 <= max_len else [])
        for step, (q, k, v) in enumerate(steps, 1):
            y = ring_matvec(dev) if with_mv else None
            out = attention(CudaTensor, dev, kc, vc, q, k, v, n_heads, n_kv, hd).export()
            what = f"{mode} {'f16' if f16 else 'f32'} hd {hd} heads {n_heads}/{n_kv} max_len {max_len}"
            if dev.lazy == 2:
                assert dev.mega_variant() == variant, (what, kv_len, dev.mega_variant())
            R.check(out, step, f16, what)
            if y is not None:
                assert_same_bits(y.export(), eager_matvec(), f"{what}: matvec vs eager")
            outs.append(out)
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("hd,n_heads,n_kv", HEADS)
@pytest.mark.parametrize("f16", [False, True], ids=["f32", "f16"])
@pytest.mark.parametrize("mode", list(MODES))
def test_retrieval_across_chunk_and_buffer_boundaries(mode, f16, hd, n_heads, n_kv):
    """Part 1: every kv_len in KV_LENS (crossing the first, second and third chunk of both chunk sizes, the first reuse of a buffer,
    and up to max_len - 1), two steps each, bit-exact against the analytic answer in every mode."""
    with fresh_device(**MODE_DEVICE[mode]) as dev:
        run_retrieval(dev, mode, f16, hd, n_heads, n_kv, MAX_LEN, KV_LENS)


# ---- part 2: random data -----------------------------------------------------------------------------------------------------------
def rope_f64(x, pos, hd):
    """RoPE with the reference's f32 angle recurrence (rope.rs:47-63: theta *= theta_scale in f32) and f64 cos / sin"""
    import ctypes
    import ctypes.util
    powf = ctypes.CDLL(ctypes.util.find_library("m")).powf          # the host call that builds the kernels' table (lazy.cu)
    powf.restype, powf.argtypes = ctypes.c_float, [ctypes.c_float, ctypes.c_float]
    x = x.astype(np.float64).reshape(-1, hd).copy()
    theta_scale = np.float32(powf(10000.0, float(np.float32(-2.0) / np.float32(hd))))
    theta = np.float32(pos)
    for j in range(hd // 2):
        c, s = np.cos(np.float64(theta)), np.sin(np.float64(theta))
        a, b = x[:, 2 * j].copy(), x[:, 2 * j + 1].copy()
        x[:, 2 * j], x[:, 2 * j + 1] = a * c - b * s, a * s + b * c
        theta = np.float32(theta * theta_scale)
    return x


def f64_attention_with_budget(q, k, v, K, V, pos, n_heads, n_kv, hd):
    """softmax attention in f64 with the true exp, and the bound on |kernel - f64| per output.

    The kernels evaluate exp as LUT[f16(x)] with x = s - m <= 0 (softmax.rs:39-54): the argument is rounded to f16 (relative error
    <= 2^-11, so exp(x) is off by a factor exp(2^-11 |x|)) and the result is rounded to f16 (relative 2^-11 while >= 2^-14,
    absolute <= 2^-25 in the subnormal range and for what flushes to 0).  So each weight e_s carries a relative error
    r_s <= 2^-11 (1 + |x_s|) + eps_s, plus the absolute 2^-25, where eps_s bounds the f32 score noise: hd products and sums, the
    scale and RoPE (angles identical, cosf / sinf within an ulp), <= 2^-24 (hd + 10) sum_i |q_i k_si| / sqrt(hd).
    Normalising by the sum (of L terms in f32: relative L 2^-24) moves every p_s by the weighted mean D = sum_s p_s r_s + L 2^-24,
    and the f32 PV sum of L terms adds L 2^-24 sum_s p_s |v_sd|.  With Sum e >= 1 (the maximum's weight is 1):
        |out_d - ref_d| <= sum_s p_s r_s |v_sd| + (D + L 2^-24) sum_s p_s |v_sd| + 2^-25 sum_s |v_sd|
    The budget is twice that, for the second-order terms."""
    qr = rope_f64(q, pos, hd)                                        # [n_heads, hd]
    kr = rope_f64(k, pos, hd)                                        # [n_kv, hd]
    ref = np.zeros((n_heads, hd))
    budget = np.zeros((n_heads, hd))
    L = K.shape[1] + 1
    u = 2.0 ** -24
    for h in range(n_heads):
        g = h % n_kv
        Kg = np.concatenate([K[g].astype(np.float64), kr[g:g + 1]])
        Vg = np.concatenate([V[g].astype(np.float64), v[g:g + 1].astype(np.float64)])
        s = Kg @ qr[h] / np.sqrt(hd)
        x = s - s.max()
        e = np.exp(x)
        p = e / e.sum()
        ref[h] = p @ Vg
        eps = u * (hd + 10) * (np.abs(Kg) @ np.abs(qr[h])) / np.sqrt(hd)
        r = 2.0 ** -11 * (1.0 + np.abs(x)) + eps
        D = float(p @ r) + L * u
        pv = p @ np.abs(Vg)
        budget[h] = 2.0 * ((p * r) @ np.abs(Vg) + (D + L * u) * pv + 2.0 ** -25 * np.abs(Vg).sum(0) / e.sum())
    return ref.reshape(-1), budget.reshape(-1)


RANDOM_KV = [96, 200, 1000, 4095]


def random_case(hd, n_heads, n_kv, kv_len):
    rng = np.random.default_rng(1000 + kv_len + hd)
    K = rng.standard_normal((n_kv, kv_len, hd)).astype(np.float32)
    V = rng.standard_normal((n_kv, kv_len, hd)).astype(np.float32)
    q = (2.0 * rng.standard_normal((n_heads, hd))).astype(np.float32)
    k = rng.standard_normal((n_kv, hd)).astype(np.float32)
    v = rng.standard_normal((n_kv, hd)).astype(np.float32)
    return K, V, q, k, v


@pytest.mark.gpu
@pytest.mark.parametrize("hd,n_heads,n_kv", [(128, 32, 8), (48, 6, 6)])
@pytest.mark.parametrize("f16", [False, True], ids=["f32", "f16"])
@pytest.mark.parametrize("kv_len", RANDOM_KV)
def test_random_attention_step_modes_oracle_and_f64(kv_len, f16, hd, n_heads, n_kv, capsys):
    """Part 2: random q, K, V with pos = kv_len (RoPE not the identity).  Graph, register and ring kernels equal the eager kernels bit for
    bit; exact_order mode equals the CPU oracle bit for bit; for f32 caches the megakernel is within the f64 budget above (skipped for
    f16 caches, where the reference's own f16 accumulation dominates)."""
    from crabml_b200 import CudaTensor
    K, V, q, k, v = random_case(hd, n_heads, n_kv, kv_len)
    dt = oc.F16 if f16 else oc.F32
    max_len = kv_len + 4
    got = {}
    for mode, (with_mv, variant) in MODES.items():
        with fresh_device(**MODE_DEVICE[mode]) as dev:
            kc, vc = fill(CudaTensor, dev, CudaTensor.alloc([n_kv, max_len, hd], dt, dev), CudaTensor.alloc([n_kv, max_len, hd], dt, dev), K, V)
            y = ring_matvec(dev) if with_mv else None
            got[mode] = attention(CudaTensor, dev, kc, vc, q, k, v, n_heads, n_kv, hd, pos=kv_len).export()
            if dev.lazy == 2:
                assert dev.mega_variant() == variant, (mode, dev.mega_variant())
            del y
    odev = OracleDevice()
    okc, ovc = fill(OracleTensor, odev, OracleTensor.alloc([n_kv, max_len, hd], dt, odev), OracleTensor.alloc([n_kv, max_len, hd], dt, odev), K, V)
    want = attention(OracleTensor, odev, okc, ovc, q, k, v, n_heads, n_kv, hd, pos=kv_len).export()
    assert np.isfinite(got["eager"]).all() and np.abs(got["eager"]).max() > 1e-3
    for mode in ("graph", "register", "ring"):
        assert_same_bits(got[mode], got["eager"], f"{mode} vs eager, kv_len {kv_len}")
    assert_same_bits(got["exact"], want, f"exact_order vs oracle, kv_len {kv_len}")
    if not f16:
        ref, budget = f64_attention_with_budget(q, k, v, K, V, kv_len, n_heads, n_kv, hd)
        ratio = float((np.abs(got["ring"].astype(np.float64) - ref) / budget).max())
        with capsys.disabled():
            print(f"\nf64 attention, hd {hd} heads {n_heads}/{n_kv} kv_len {kv_len}: max |ring - f64| / budget = {ratio:.3f}")
        assert ratio <= 1.0, ratio


# ---- part 4: the context-length switches -------------------------------------------------------------------------------------------
# Three flush shapes, all with head_dim 128: the ring kernel's flush of part 1 with 8 heads; the same attention with 32 query heads
# after the qkv phase of a Llama-2-7B layer (rms_norm * w of a 4096 row, three Q8_0 4096 x 4096 matvecs: its norm weights are staged in
# shared memory beside the working area, as in the real layer); and the 8-head attention alone, which runs the register kernel.  The
# decision depends on head_dim and max_len, not on n_kv.  (head_dim, n_heads, n_kv, other phase: None = the ring matvec, 0 = none,
# else the qkv phase of that dim; the persistent kernel below the switch)
SWITCH_SHAPES = {"small": (128, 8, 2, None, MEGA_RING), "7b": (128, 32, 8, 4096, MEGA_RING), "attn": (128, 8, 2, 0, MEGA_REGISTER)}


def qkv_phase(dev, dim):
    from crabml_b200 import CudaTensor
    from crabml_b200 import runner as R
    rng = np.random.default_rng(dim)
    x = CudaTensor.new(rng.standard_normal(dim).astype(np.float32), [dim], dev)
    w = CudaTensor.new((1.0 + 0.05 * rng.standard_normal(dim)).astype(np.float32), [dim], dev)
    x = x.rms_norm_inplace(1e-5).mul_inplace(w)
    ys = [CudaTensor.synth([dim, dim], oc.Q8_0, dev, 0x7B, i + 1, R.synth_scale(oc.Q8_0, dim)).matmul_vec(x) for i in range(3)]
    del x
    return ys


def switch_step(shape, lazy, f16, max_len, kv_len, R=None):
    """fresh device; one step of the shape's flush at this max_len -> (variant, attention output, outputs of the other phase)"""
    from crabml_b200 import CudaTensor
    hd, n_heads, n_kv, dim, _ = SWITCH_SHAPES[shape]
    dt = oc.F16 if f16 else oc.F32
    R = R or Retrieval(hd, n_heads, n_kv, kv_len)
    with fresh_device(lazy=lazy) as dev:
        kc, vc = fill(CudaTensor, dev, CudaTensor.alloc([n_kv, max_len, hd], dt, dev), CudaTensor.alloc([n_kv, max_len, hd], dt, dev), R.K, R.V)
        ys = qkv_phase(dev, dim) if dim else [] if dim == 0 else [ring_matvec(dev)]
        out = attention(CudaTensor, dev, kc, vc, R.q1, R.k1, R.v1, n_heads, n_kv, hd).export()
        return dev.mega_variant(), out, [y.export() for y in ys]


def first_max_len(shape, pred, lo, hi):
    """smallest max_len in (lo, hi] with pred(variant), given not pred at lo and pred at hi (variant is monotone in max_len)"""
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if pred(switch_step(shape, 2, False, mid, 1)[0]):
            hi = mid
        else:
            lo = mid
    return hi


_SWITCHES = {}


def switches(shape):
    """-> first max_len that leaves the persistent kernel for the CUDA graph"""
    if shape not in _SWITCHES:
        lo, hi = 256, 50808
        assert switch_step(shape, 2, False, lo, 1)[0] == SWITCH_SHAPES[shape][4] and switch_step(shape, 2, False, hi, 1)[0] == MEGA_NONE
        _SWITCHES[shape] = first_max_len(shape, lambda v: v == MEGA_NONE, lo, hi)
    return _SWITCHES[shape]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SWITCH_SHAPES))
def test_each_side_of_the_context_length_switches(shape, capsys):
    """Probe (one step per candidate, a fresh device each) the max_len at which lazy mode 2 leaves its persistent kernel for the CUDA
    graph; then on each side of the switch fill the cache to max_len - 1 and require the analytic answer and the eager bits, for both
    cache types."""
    graph = switches(shape)
    hd, n_heads, n_kv, _, kernel = SWITCH_SHAPES[shape]
    with capsys.disabled():
        print(f"\n{shape}: lazy=2 runs the {'ring' if kernel == MEGA_RING else 'register'} kernel up to max_len {graph - 1}, "
              f"the CUDA graph of fused kernels from {graph}")
    for max_len in (graph - 1, graph):
        for f16 in (False, True):
            R = Retrieval(hd, n_heads, n_kv, max_len - 1)
            variant, out, ys = switch_step(shape, 2, f16, max_len, max_len - 1, R)
            assert variant == (kernel if max_len < graph else MEGA_NONE), (max_len, variant)
            R.check(out, 1, f16, f"{shape} lazy=2 max_len {max_len} variant {variant}")
            _, out0, ys0 = switch_step(shape, 0, f16, max_len, max_len - 1, R)
            assert_same_bits((out, ys), (out0, ys0), f"{shape} lazy=2 vs eager, max_len {max_len} f16={f16}")


@pytest.mark.gpu
@pytest.mark.parametrize("max_len", [50808, 50809, 65536])
@pytest.mark.parametrize("lazy", [1, 2])
def test_context_past_the_single_pass_kernel(lazy, max_len):
    """The fused single-pass kernel holds the whole score row in shared memory: 50 808 positions at head_dim 128.  Past that the fuser
    must leave attention to the per-op kernels, as in eager mode, instead of failing the token; same bits as eager."""
    R = Retrieval(128, 8, 2, max_len - 1)
    variant, out, ys = switch_step("small", lazy, False, max_len, max_len - 1, R)
    assert variant == MEGA_NONE
    R.check(out, 1, False, f"lazy={lazy} max_len {max_len}")
    _, out0, ys0 = switch_step("small", 0, False, max_len, max_len - 1, R)
    assert_same_bits((out, ys[0]), (out0, ys0[0]), f"lazy={lazy} vs eager, max_len {max_len}")
