"""Which ops the lazy fuser (lazy.cu) fuses, and which persistent kernel runs them.  Bit-identity alone cannot see a fusion that
silently stops happening, since an unfused op gives the same bits through its eager kernel.  So each case pins, besides eager logits:
lazy mode 1's kernel launches per token and its uncached flushes, and lazy mode 2's kernel variant and phase table fingerprint.  A
fingerprint lists the phase type codes of CudaTensorDevice.mega_phase_types(): 16 * type (0 NORMQ, 1 MATVEC, 2 ATTN, 3 ROWS, 4 REDUCE, 5 GATHER,
6 ARGMAX, 7 SAMPLE), plus for a MATVEC phase its matrix count + 4 * epilogue + 1024 * (k >> 10)."""
import numpy as np
import pytest

from oracle import oracle as oc
from crabml_b200.tensor import MEGA_NONE, MEGA_REGISTER, MEGA_RING
from tests.gpu_common import assert_same_bits, run_modes

pytestmark = pytest.mark.gpu

PROMPT = [1, 365, 2354]
L7B = (32, 32, 1, 4096, 11008, 64, 32000, 1e-5, 128)


def _decode(weights, sample=False):
    """Decode from a slot (ROWS phase first, ARGMAX or SAMPLE last): launches of one generated token, and the logits."""
    def case(dev):
        from crabml_b200 import runner as R
        conf, w = weights(dev)
        counts, logits = [], None
        for steps in (3, 4):
            r = R.LlamaRunner(dev, conf, w, 16)
            l0 = dev.launch_count()
            if sample:
                _, logits = r.generate_logits(PROMPT, steps, 1.0, 0.9, 7)
            else:
                _, logits = r.generate_greedy_logits(PROMPT, steps)
            counts.append(dev.launch_count() - l0)
            r.close()
        return counts[1] - counts[0], logits
    return case


def _synth(wt, ct):
    def weights(dev):
        from crabml_b200 import runner as R
        conf = R.LlamaConfig(*L7B)
        return conf, R.synthetic_weights(dev, conf, wt, ct, seed=0xF5)
    return weights


def _synth_q4_k_m(dev):
    """the 7B-shaped Q4_K layer laid out like llama.cpp's Q4_K_M: wv and ffn_down in Q6_K"""
    from crabml_b200 import CudaTensor
    from crabml_b200 import runner as R
    conf, w = _synth(oc.Q4_K, oc.Q6_K)(dev)
    for tid, key in enumerate(("wv", "ffn_down"), 100):
        rows, cols = w[key][0].shape()
        w[key][0] = CudaTensor.synth([rows, cols], oc.Q6_K, dev, 0xF5, tid, R.synth_scale(oc.Q6_K, cols))
    return conf, w


def _fixture(path):
    def weights(dev):
        from crabml_b200 import runner as R
        conf, w, _ = R.load_gguf(path, dev)
        return conf, w
    return weights


def _ops(body, comm=False, rounds=3):
    """Replay an op sequence `rounds` times; each round ends in an export (one flush).  Launches of the last round, and its outputs."""
    def case(dev):
        from crabml_b200 import CudaTensor, capi
        from crabml_b200.runner import synth_scale
        if comm:
            dev.init_comm(0, 1)
        rng, weights = np.random.default_rng(9), {}

        def W(m, k, t, i):                 # made in the first round, which the measured last round does not see
            if (m, k, t, i) not in weights:
                weights[m, k, t, i] = CudaTensor.synth([m, k], t, dev, 3, i, synth_scale(t, k))
            return weights[m, k, t, i]
        T = lambda v: CudaTensor.new(np.asarray(v, np.float32), [len(v)], dev)                           # noqa: E731
        env = dict(dev=dev, rng=rng, T=T, W=W, capi=capi, CudaTensor=CudaTensor)
        for _ in range(rounds):
            l0 = dev.launch_count()
            out = body(env)
            n = dev.launch_count() - l0
        return n, out
    return case


def _gate_up_no_silu(e):            # two matvecs on one row, nothing after them
    x = e["T"](e["rng"].standard_normal(512))
    ys = [e["W"](256, 512, e["capi"].Q8_0, i).matmul_vec(x) for i in (1, 2)]
    return np.concatenate([y.export() for y in ys])


def _three_then_silu(e):            # q, k, v on one row, then silu on the first
    x = e["T"](e["rng"].standard_normal(512))
    ys = [e["W"](256, 512, e["capi"].Q8_0, i).matmul_vec(x) for i in (1, 2, 3)]
    ys[0].silu_inplace()
    return np.concatenate([y.export() for y in ys])


def _kquant_self_residual(e):       # K-quant matvec + its own input row
    x = e["T"](e["rng"].standard_normal(512))
    return e["W"](512, 512, e["capi"].Q4_K, 1).matmul_vec(x).add_inplace(x).export()


def _norm_weight_written(e):        # the fused norm's weight row is the output of an earlier matvec of the same flush
    z, x = e["T"](e["rng"].standard_normal(512)), e["T"](e["rng"].standard_normal(512))
    nw = e["W"](512, 512, e["capi"].Q8_0, 1).matmul_vec(z)
    x.rms_norm_inplace(1e-5)
    x.mul_inplace(nw)
    return e["W"](256, 512, e["capi"].Q8_0, 2).matmul_vec(x).export()


def _exchange(gather):              # world of one: matvec -> all_reduce -> + residual, or matvec -> all_gather
    def body(e):
        x, r = e["T"](e["rng"].standard_normal(4096)), e["T"](e["rng"].standard_normal(1024))
        y = e["W"](1024, 4096, e["capi"].Q8_0, 5).matmul_vec(x)
        if gather:
            return e["CudaTensor"].alloc([1024], e["capi"].F32, e["dev"]).all_gather_from(y).export()
        return y.all_reduce_sum_inplace().add_inplace(r).export()
    return body


def _samplers(n):
    def body(e):
        t = e["T"](2.0 * e["rng"].standard_normal(64))
        for i in range(n):
            t.sample_to_slot(1.0, 0.9, 5, i, i, i)
        return e["dev"].read_history(0, n)
    return body


def _tinyllamas(fixture_path):
    return _decode(_fixture(fixture_path("tinyllamas-stories-15m-q8_0.gguf")))


# id: (case, mode-1 launches per token, mode-1 uncached flushes, mode-2 variant (0: CUDA graph), mode-2 fingerprint).  Codes: 48 ROWS (a
# CudaTensor.new upload, too), 32 ATTN, 0 NORMQ, 96 ARGMAX, 112 SAMPLE, 64 REDUCE, 80 GATHER; 16 + n + 4 * epilogue + 1024 * (k >> 10) MATVEC.
DECODE_7B = (48, 4115, 32, 4117, 4122, 10261, 0, 48, 4113, 96)     # embedding row; qkv + prologue, attn, wo + res, gate/up + prologue,
#                                          down (k 11008) + res; final norm, a row copy, classifier + prologue, argmax
TINY_LAYER = (19, 32, 0, 21, 26, 21)      # head_dim 48: qkv + prologue, attn, plain quantise of its output, wo + res, gate/up, down + res
CASES = {
    "7b-q8_0": (lambda fp: _decode(_synth(oc.Q8_0, oc.Q8_0)), 14, 0, MEGA_RING, DECODE_7B),
    "7b-q4_0-q6k": (lambda fp: _decode(_synth(oc.Q4_0, oc.Q6_K)), 14, 0, MEGA_RING, DECODE_7B),      # Q6_K classifier: a generic phase in the ring table
    "7b-q4_k": (lambda fp: _decode(_synth(oc.Q4_K, oc.Q6_K)), 29, 0, MEGA_REGISTER, DECODE_7B),      # mode 1 runs K-quant ops eagerly
    # mixed q/k/v (wv Q6_K): the norm cannot fold into the wq/wk phase while wv still reads its row, so it is written back by a NORMQ
    # phase, then wq + wk (2 matrices) and wv (1) run as separate generic phases
    "7b-q4_k_m": (lambda fp: _decode(_synth_q4_k_m), 28, 0, MEGA_REGISTER, (48, 0, 4114, 4113) + DECODE_7B[2:]),
    "tinyllamas-q8_0": (_tinyllamas, 60, 0, MEGA_RING, (48,) + TINY_LAYER * 6 + (0, 48, 17, 96)),
    "7b-q8_0-sampled": (lambda fp: _decode(_synth(oc.Q8_0, oc.Q8_0), sample=True), 14, 0, MEGA_RING, DECODE_7B[:-1] + (112,)),
    "two-samplers": (lambda fp: _ops(_samplers(2)), 3, 0, MEGA_NONE, ()),                             # upload + 2 samplers, in the graph
    "allreduce-add": (lambda fp: _ops(_exchange(False), comm=True), 5, 0, MEGA_RING, (48, 48, 4125, 64)),   # x, r; matvec into the exchange, reduce + r
    "allgather": (lambda fp: _ops(_exchange(True), comm=True), 5, 0, MEGA_RING, (48, 48, 4125, 80)),
    "gate-up-no-silu": (lambda fp: _ops(_gate_up_no_silu), 3, 0, MEGA_RING, (48, 18)),               # x; one 2-matrix phase with a plain quantise
    "three-then-silu": (lambda fp: _ops(_three_then_silu), 8, 0, MEGA_NONE, ()),                      # silu is an eager op: no persistent kernel
    "kquant-self-residual": (lambda fp: _ops(_kquant_self_residual), 4, 0, MEGA_NONE, ()),             # the add is an eager op
    "norm-weight-written": (lambda fp: _ops(_norm_weight_written), 6, 0, MEGA_RING, (48, 48, 17, 0, 17)),    # z, x; nw; norm written back (x lives on), matvec
}


@pytest.mark.parametrize("name", list(CASES))
def test_fusion_plan(name, fixture_path, monkeypatch):
    monkeypatch.setenv("CRABML_MEGA_PROF", "1")
    case, launches, uncached, variant, fingerprint = CASES[name]

    def body(dev):
        n, out = case(fixture_path)(dev)
        st = dev.lazy_stats()
        return n, st and st["uncached"], dev.mega_variant(), dev.mega_phase_types() if dev.lazy == 2 else (), np.asarray(out).copy()
    res = run_modes(body)
    assert res[1][:2] == (launches, uncached), (name, "mode 1 (launches per token, uncached)", res[1][:2])
    assert res[2][2:4] == (variant, fingerprint), (name, "mode 2 (variant, fingerprint)", res[2][2:4])
    for mode in (1, 2):
        assert_same_bits(res[mode][4], res[0][4], f"{name}: lazy={mode} vs eager")
