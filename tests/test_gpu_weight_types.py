"""The persistent kernels' K-quant (generic) MATVEC phase on every weight type, and models whose layers mix weight types.

The suite pins the eager kernels to the oracle for every weight type (test_gpu_matvec.py, test_gpu_ops.py) and the lazy modes to the eager
kernels bit for bit; that covers the benchmarked kernels only for the weight types and phase tables a lazy-mode test actually runs.  Here:

 (a) raw op sequences through the Python mirror, flushed in lazy modes 0, 1 and 2: 1-3 matrices on one row, the gate/up pair epilogue and
     the residual epilogue, with and without a fused [dup] rms_norm * w prologue, at row lengths that hit the phase's edges (one
     super-block; 1-5 segments of 16 super-blocks with a partial last one; the 32768-column limit) and row counts of 1, a few, and more
     than the grid has warps -- for Q2_K, Q3_K, Q4_K, Q5_K, Q6_K and Q8_K.  Each case checks the persistent kernel and its phase table
     (so it cannot pass without reaching the phase under test), bit-identity with the eager kernels, and, where no norm or pair is
     fused, the oracle's gemv within the per-op budget of test_gpu_matvec.py.
 (b) small models laid out like llama.cpp's K-quant files (Q4_K_M, Q5_K_M, Q3_K_M, Q2_K: a few tensors in another type), with the
     Q8_0 / Q5_0 fallback tensors a dimension that is not a multiple of 256 gets, and the 32-block types, decoded through the C++ runner:
     exact_order logits equal the oracle replay, lazy modes 0-2 are bit-identical, and the expected persistent kernel ran."""
import os

import numpy as np
import pytest

from oracle import oracle as oc
from oracle.llama_replay import Llama2Runner, LlamaConfig as OConf, LlamaWeights
from oracle.synth import synth_weight
from oracle.tensor_ref import OracleDevice, OracleTensor
from crabml_b200.runner import synth_scale
from crabml_b200.tensor import MEGA_NONE, MEGA_REGISTER, MEGA_RING
from tests.gpu_common import assert_same_bits, fresh_device, run_modes
from tests.test_gpu_matvec import gemv_budget

pytestmark = pytest.mark.gpu

GENERIC = [oc.Q2_K, oc.Q3_K, oc.Q4_K, oc.Q5_K, oc.Q6_K, oc.Q8_K]
WSEED = 0x6E7
EPS = 1e-5
ORACLE_THREADS = max(1, min(8, len(os.sched_getaffinity(0))))


def _mv_code(n, epilogue, k):
    return 16 + n + 4 * epilogue + 1024 * (k >> 10)


# ---- (a) the generic phase, op by op ------------------------------------------------------------------------------------------------
NMAT = {"one": 1, "two": 2, "three": 3, "pair": 2, "res": 1}
EPILOGUE = {"one": 0, "two": 0, "three": 0, "pair": 2, "res": 1}
# Row lengths: 256 = one super-block; 2816 / 4352 / 11008 / 14336 / 18944 = 1 / 2 / 3 / 4 / 5 segments of 16 super-blocks with a partial
# last one; 4096 = exactly one segment; 32768 = the generic phase's limit (cc_mega_generic_supported), whose working area leaves no room
# for a fused norm's weight stage.  Every type meets every length: its five plain cases and its five fused-norm cases rotate over these.
K_PLAIN = [32768, 256, 2816, 4352, 14336]
K_NORM = [4096, 11008, 18944, 2816, 4352]
# more rows than the grid has warps (132 SMs x 16 warps on an H100 SXM), so warps own several rows and the deferred epilogue store of
# one row is written while the next one is reduced
MANY = 2240


def _rows(sel, k, shape):
    """a few rows: 37 (odd), but 36 for an epilogue -- the reference's add / mul of a row longer than 1 skips the tail past the last
    multiple of 4 (chunks_exact(4)), which a fused epilogue cannot do: TAIL_CASES pin that such a group is not fused"""
    return [1, 36 if EPILOGUE[shape] else 37, 4096 if k <= 4352 else MANY][sel]


def _ms(shape, m):
    """rows of each matrix of the group: q/k/v-shaped (unequal) for three, equal otherwise"""
    if shape == "three":
        return [m, (m + 3) // 4, (m + 3) // 4]
    return [m] * NMAT[shape]


def _cases():
    out = []
    for ti, t in enumerate(GENERIC):
        for norm in (False, True):
            for si, shape in enumerate(NMAT):
                k = (K_NORM if norm else K_PLAIN)[(si + ti) % 5]
                m = _rows((ti + si + 2 * norm) % 3, k, shape)
                dup = norm and (shape == "res" or ti % 2 == 0)      # [dup]: the prologue also copies the raw row out (CTA 0)
                out.append((t, shape, norm, dup, k, _ms(shape, m)))
        out.append((t, "three", True, True, 4096, [4096, 1024, 1024]))       # Llama-2 q/k/v under 4:1 grouped-query attention
    return out


# 37 rows and an add / mul that skips the last one: the epilogue stays an eager op, so the flush runs in the CUDA-graph mode (Q8_0: the
# streaming kernel's epilogue follows the same rule)
TAIL_CASES = [(t, shape, False, False, 4352, [37] * NMAT[shape]) for t in GENERIC + [oc.Q8_0] for shape in ("pair", "res")]
CASES = _cases() + TAIL_CASES


def _tail(n):
    """rows an add / mul of an n-element rhs touches (capi.cu binary(), arithmetic.rs:5-68)"""
    return n if n == 1 else n - n % 4


def _case_id(c):
    t, shape, norm, dup, k, ms = c
    return f"{oc.TYPE_NAMES[t]}-{shape}-{'dupnorm' if dup else 'norm' if norm else 'plain'}-k{k}-m{ms[0]}"


class _Flush:
    """Tensors of the flushes on one device: weights synthesised on the device once (seed WSEED, tensor id `tid`), f32 rows uploaded."""

    def __init__(self, dev):
        self.dev, self.weights = dev, {}

    def W(self, m, k, t, tid):
        from crabml_b200 import CudaTensor
        if (m, k, t, tid) not in self.weights:
            self.weights[m, k, t, tid] = CudaTensor.synth([m, k], t, self.dev, WSEED, tid, synth_scale(t, k))
        return self.weights[m, k, t, tid]

    def T(self, v):
        from crabml_b200 import CudaTensor
        return CudaTensor.new(np.asarray(v, np.float32), [len(v)], self.dev)


ROUNDS = 2


def _host_inputs(k, shape, rnd):
    """x, norm weights, residual row of round `rnd`: new values every round, so that a replayed graph cannot pass on a stale result"""
    rng = np.random.default_rng([k, len(shape), rnd])
    x = rng.standard_normal(k).astype(np.float32)
    nw = (1.0 + 0.05 * rng.standard_normal(k)).astype(np.float32)
    r = rng.standard_normal(max(4096, k)).astype(np.float32)
    return x, nw, r


def _generic_body(case):
    """-> body(flush, round): the ops of one case.  Uploads: x, the norm weights, the residual row (in that order, each if used).  The
    normalised row is dropped before the export, as the runner's moves do: the fuser folds the norm into the phase's prologue only when
    nobody else can read it."""
    t, shape, norm, dup, k, ms = case

    def body(f, rnd):
        x_h, nw_h, r_h = _host_inputs(k, shape, rnd)
        x = f.T(x_h)
        outs = []
        if norm:
            nw = f.T(nw_h)
        if shape == "res":
            res = f.T(r_h[:ms[0]])
        if norm:
            if dup:
                outs.append(x.dup())
            x.rms_norm_inplace(EPS).mul_inplace(nw)
        ys = [f.W(m, k, t, i + 1).matmul_vec(x) for i, m in enumerate(ms)]
        del x
        if shape == "pair":
            g, u = ys
            g.silu_inplace().mul_inplace(u)
            del u
            ys = [g]
        elif shape == "res":
            ys[0].add_inplace(res)
        return np.concatenate([y.export() for y in ys + outs])
    return body


def _uploads(case):
    t, shape, norm, dup, k, ms = case
    return 1 + norm + (shape == "res")


def _expected_plan(case):
    """(mode-2 variant, phase table fingerprint): one generic phase after the uploads, without a NORMQ (0) phase when the norm is
    fused -- or no persistent kernel at all when the epilogue would have to skip a tail"""
    t, shape, norm, dup, k, ms = case
    if EPILOGUE[shape] and _tail(ms[0]) != ms[0]:
        return MEGA_NONE, ()
    return MEGA_REGISTER, (48,) * _uploads(case) + (_mv_code(NMAT[shape], EPILOGUE[shape], k),)


def flushes(body, grid=0, comm=False, rounds=ROUNDS):
    """-> body(dev) for run_modes: the flush `rounds` times (the first captures the graph, the last replays it) at SM limit `grid`, with
    a world of one if `comm` -> (variant, phase types in mode 2, lazy stats, launches of the last round, its output)"""
    def run(dev):
        if grid:
            dev.set_sm_limit(grid)
        if comm:
            dev.init_comm(0, 1)
        f = _Flush(dev)
        for rnd in range(rounds):
            l0 = dev.launch_count()
            out = body(f, rnd)
            n = dev.launch_count() - l0
        return dev.mega_variant(), dev.mega_phase_types() if dev.lazy == 2 else (), dev.lazy_stats(), n, np.asarray(out).copy()
    return run


def _assert_modes(body, variant, fingerprint, what):
    """lazy modes 1 and 2 bit-identical to eager; mode 2 ran `variant` with phase table `fingerprint`.  -> the eager output"""
    res = run_modes(flushes(body))
    ref = res[0][4]
    for mode in (1, 2):
        assert res[mode][2]["uncached"] == 0, (what, mode, res[mode][2])
        assert_same_bits(res[mode][4], ref, f"{what}: lazy={mode} vs eager")
    assert res[2][:2] == (variant, fingerprint), (what, res[2][:2])
    assert np.isfinite(ref).all() and np.abs(ref).max() > 1e-3
    return ref


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_generic_phase_vs_eager_and_oracle(case, monkeypatch):
    monkeypatch.setenv("CRABML_MEGA_PROF", "1")
    t, shape, norm, dup, k, ms = case
    ref = _assert_modes(_generic_body(case), *_expected_plan(case), _case_id(case))
    if norm or shape == "pair":
        return                   # the eager rms_norm, silu and mul kernels are pinned to the oracle elsewhere; bit-identity is the check
    x, _, r = _host_inputs(k, shape, ROUNDS - 1)
    o = 0
    for i, m in enumerate(ms):
        raw = synth_weight(t, m, k, WSEED, i + 1, synth_scale(t, k))
        want = oc.gemv(t, raw, m, k, x, threads=ORACLE_THREADS).astype(np.float64)
        budget = gemv_budget(t, raw, m, k, x)
        got = ref[o:o + m].astype(np.float64)
        if shape == "res":       # + the residual row where the add reaches: one more f32 rounding of the sum
            n = _tail(m)
            want[:n] = want[:n] + r[:n]
            budget = budget + np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
        diff = np.abs(got - want)
        assert (diff <= budget).all(), (_case_id(case), i, float((diff / budget).max()))
        o += m


def test_generic_phases_of_every_type_in_the_ring_kernel(monkeypatch):
    """A Q8_0 matvec in the flush puts the table on the ring kernel (mega_ring_kernel with generic phases): one generic phase of every
    K-quant type between streaming phases, and a fused-norm generic phase whose norm weights the kernel stages early (from the first
    phase on, across the plain generic and streaming phases before it)."""
    monkeypatch.setenv("CRABML_MEGA_PROF", "1")
    k = 4096

    def body(f, rnd):
        x_h, nw_h, r_h = _host_inputs(k, "ring", rnd)
        x, nw, r = f.T(x_h), f.T(nw_h), f.T(r_h[:k])
        ys = [f.W(512, k, oc.Q8_0, 1).matmul_vec(x)]                                       # streaming, plain quantise merged
        ys += [f.W(37 + 64 * i, k, t, 2 + i).matmul_vec(x) for i, t in enumerate(GENERIC)]   # one generic phase per type
        ys.append(x.dup())
        x.rms_norm_inplace(EPS).mul_inplace(nw)
        z = f.W(k, k, oc.Q5_K, 9).matmul_vec(x).add_inplace(r)                             # fused [dup] norm + residual
        del x
        ys += [z, f.W(300, k, oc.Q8_0, 10).matmul_vec(z)]                                  # streaming again, on the generic output
        return np.concatenate([y.export() for y in ys])
    code = _mv_code(1, 0, k)
    _assert_modes(body, MEGA_RING, (48, 48, 48, code) + (code,) * len(GENERIC) + (_mv_code(1, 1, k), code), "ring")


# ---- (b) mixed-type models end to end ----------------------------------------------------------------------------------------------
SMALL = dict(n_heads=16, n_kv=4, n_layers=4, dim=1024, hidden=2816, vocab=4096)


def _qkm(body, high):
    """llama.cpp's *_K_M: wv and ffn_down in a higher type on the first and last layer"""
    return lambda name, l, nl: high if name in ("wv", "ffn_down") and l in (0, nl - 1) else body


def _q3km(name, l, nl):
    if name in ("wv", "ffn_down"):
        return oc.Q5_K if l < 2 else oc.Q4_K
    return oc.Q4_K if name == "wo" else oc.Q3_K


def _q2k(name, l, nl):
    return {"wv": oc.Q4_K, "wo": oc.Q3_K, "ffn_down": oc.Q3_K}.get(name, oc.Q2_K)


def _fallback(t):
    return lambda name, l, nl: t if name == "ffn_down" else oc.Q4_K


def _uniform(t):
    return lambda name, l, nl: t


# id: (type of (tensor, layer, n_layers), classifier type, shape overrides, f16 KV cache, expected mode-2 variant)
LAYOUTS = {
    "q4_k_m": (_qkm(oc.Q4_K, oc.Q6_K), oc.Q6_K, {}, False, MEGA_REGISTER),
    "q5_k_m": (_qkm(oc.Q5_K, oc.Q6_K), oc.Q6_K, {}, True, MEGA_REGISTER),
    "q3_k_m": (_q3km, oc.Q6_K, {}, False, MEGA_REGISTER),
    "q2_k": (_q2k, oc.Q6_K, {}, True, MEGA_REGISTER),
    "q8_k": (_uniform(oc.Q8_K), oc.Q8_K, {}, False, MEGA_REGISTER),
    "q4_k-q8_0-fallback": (_fallback(oc.Q8_0), oc.Q6_K, {"hidden": 2720}, False, MEGA_RING),     # ring kernel with generic phases
    "q4_k-q5_0-fallback": (_fallback(oc.Q5_0), oc.Q6_K, {"hidden": 2720}, True, MEGA_NONE),      # an eager-only matvec: CUDA graph
    "q4_1": (_uniform(oc.Q4_1), oc.Q6_K, {}, False, MEGA_NONE),
    "q5_0": (_uniform(oc.Q5_0), oc.Q6_K, {}, True, MEGA_NONE),
    "q5_1": (_uniform(oc.Q5_1), oc.Q6_K, {}, False, MEGA_NONE),
    "mistral-q4_k_m": (_qkm(oc.Q4_K, oc.Q6_K), oc.Q6_K, dict(n_heads=32, n_kv=8, n_layers=1, dim=4096, hidden=14336, vocab=32000), True,
                       MEGA_REGISTER),
}


def _shape(overrides):
    s = dict(SMALL)
    s.update(overrides)
    return s


def mixed_weights(type_of, ct, s, make, norm_tensor):
    """The weight set of a model whose tensors have the types type_of(name, layer, n_layers) (token embedding: that of wq; classifier:
    ct).  make(rows, cols, type, tensor id) builds one weight and norm_tensor(values) one f32 row, so the same call gives the
    CudaTensor set for LlamaRunner (synthesised on the device) and the bit-identical OracleTensor twin for the oracle's Llama2Runner.
    -> dict in runner.synthetic_weights' layout."""
    dim, hid, nl = s["dim"], s["hidden"], s["n_layers"]
    kv = dim // s["n_heads"] * s["n_kv"]
    rng = np.random.default_rng(WSEED)
    tid = [0]

    def syn(rows, cols, t):
        tid[0] += 1
        return make(rows, cols, t, tid[0])

    # norm weights around 1/4: with weights around 1 the gate/up products of these synthetic blocks reach a few thousand, and the f16
    # block sum of a Q8_1 activation (the partner of Q4_1 / Q5_1 weights) overflows -- in the reference as on the GPU
    def norm():
        return norm_tensor((0.25 + 0.0125 * rng.standard_normal(dim)).astype(np.float32))
    w = {k: [] for k in ("wq", "wk", "wv", "wo", "ffn_gate", "ffn_up", "ffn_down", "rms_att", "rms_ffn")}
    for l in range(nl):
        for name, rows, cols in (("wq", dim, dim), ("wk", kv, dim), ("wv", kv, dim), ("wo", dim, dim), ("ffn_gate", hid, dim),
                                 ("ffn_up", hid, dim), ("ffn_down", dim, hid)):
            w[name].append(syn(rows, cols, type_of(name, l, nl)))
        w["rms_att"].append(norm()); w["rms_ffn"].append(norm())
    w["token_embed"] = syn(s["vocab"], dim, type_of("wq", 0, nl))
    w["output_weight"] = syn(s["vocab"], dim, ct)
    w["rms_final"] = norm()
    return w


def _gpu_logits(layout, tokens):
    """-> body(dev): the logits of every token, lazy stats, variant"""
    from crabml_b200 import CudaTensor
    from crabml_b200 import runner as R
    type_of, ct, over, f16_kv, _ = LAYOUTS[layout]
    s = _shape(over)

    def body(dev):
        w = mixed_weights(type_of, ct, s, lambda r, c, t, i: CudaTensor.synth([r, c], t, dev, WSEED, i, synth_scale(t, c)),
                          lambda v: CudaTensor.from_cpu(v, [v.size], oc.F32, dev))
        conf = R.LlamaConfig(s["n_heads"], s["n_kv"], s["n_layers"], s["dim"], s["hidden"], 64, s["vocab"], EPS, s["dim"] // s["n_heads"])
        r = R.LlamaRunner(dev, conf, w, 16, f16_kv=f16_kv)
        out = np.stack([r.forward([t], p).copy() for p, t in enumerate(tokens)])
        r.close()
        return out, dev.lazy_stats(), dev.mega_variant()
    return body


def _oracle_logits(layout, tokens):
    type_of, ct, over, f16_kv, _ = LAYOUTS[layout]
    s = _shape(over)
    odev = OracleDevice(thread_num=ORACLE_THREADS)
    w = mixed_weights(type_of, ct, s, lambda r, c, t, i: OracleTensor.from_cpu(synth_weight(t, r, c, WSEED, i, synth_scale(t, c)), [r, c], t, odev),
                      lambda v: OracleTensor.from_cpu(v, [v.size], oc.F32, odev))
    lw = LlamaWeights(w["token_embed"], w["wq"], w["wk"], w["wv"], w["wo"], w["ffn_gate"], w["ffn_down"], w["ffn_up"], w["rms_att"], w["rms_ffn"],
                      w["rms_final"], w["output_weight"])
    ro = Llama2Runner(OracleTensor, OConf(s["n_heads"], s["n_kv"], s["n_layers"], s["dim"], s["hidden"], 64, s["vocab"], EPS, s["dim"] // s["n_heads"]),
                      lw, odev, 16, use_f16_kv_cache=f16_kv)
    return np.stack([ro.forward([t], p).copy() for p, t in enumerate(tokens)])


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_mixed_type_model(layout):
    _, _, over, _, variant = LAYOUTS[layout]
    tokens = [1] + [int(t) for t in np.random.default_rng(len(layout)).integers(2, _shape(over)["vocab"], 9)]
    want = _oracle_logits(layout, tokens)
    with fresh_device(exact_order=True) as dev:
        exact, _, _ = _gpu_logits(layout, tokens)(dev)
    assert_same_bits(exact, want, f"{layout}: exact_order vs the oracle")
    fast = run_modes(_gpu_logits(layout, tokens))
    for mode in (1, 2):
        assert fast[mode][1]["uncached"] == 0, (layout, mode, fast[mode][1])
        assert_same_bits(fast[mode][0], fast[0][0], f"{layout}: lazy={mode} vs eager")
    assert fast[2][2] == variant, (layout, fast[2][2])      # each token is one flush: MEGA_NONE means no token ran a persistent kernel
    ref = fast[0][0]
    assert np.isfinite(ref).all() and np.abs(ref).max() > 1e-3
    rel = float(np.abs(ref - want).max() / np.abs(want).max())
    assert rel < 3e-2, (layout, rel)
