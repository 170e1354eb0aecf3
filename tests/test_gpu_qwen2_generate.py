"""Qwen2 generation end to end: the device-resident loop of the runner (ccr_runner_generate_greedy / _greedy_ex / _ex), where every
step after the first takes its embedding row from the device slot the previous step sampled into, the sampler inside a qwen2 flush
(the ring kernel's sample phase in lazy mode 2), and the tied classifier, which is then both the slot-indexed embedding table and the
logits matvec.

 * exact_order: the ids are those of the oracle replay picked by the reference sampler, and the exported logits are the oracle's,
   bit for bit.
 * fast modes: eager, lazy 1 and lazy 2 give the same ids and logits bit for bit, over enough steps that the persistent attention
   runs on both sides of its split; every id is the fast sampler's pick on the exported logits; the device loop equals a host loop
   (forward -> export -> pick on the host) bit for bit; EOS stops every mode where the reference stops.
 * Qwen2-7B shapes on synthetic weights: the same identities at vocab 152 064, and the fast mode inside the band between the
   reference's own two summation orders (tests/test_gpu_runner.py restates the yardstick for Llama)."""
import dataclasses
import os

import numpy as np
import pytest

from oracle import oracle as oc
from oracle.llama_replay import Llama2Runner, LlamaConfig as OConf, LlamaWeights
from oracle.synth import synth_weight
from oracle.tensor_ref import OracleDevice, OracleTensor
from tests import sampler_ref as S
from crabml_b200.tensor import MEGA_NONE, MEGA_RING
from tests.blockgen import random_weight
from tests.gpu_common import assert_same_bits, fresh_device, run_modes
from tests.test_gpu_qwen2 import DIM, HEADS, HID, KV, NL, SPLIT_FROM, VOCAB, _gpu_from_raw, make_model

pytestmark = pytest.mark.gpu

SEED = 0x5A3D1E
SAMPLERS = [(0.8, 0.9), (1.0, 1.0), (0.0, 0.0)]        # (temperature, topp); temperature 0 is the greedy entry point
ROPE_DIM = 64                                          # head_dim 64, as Qwen2-0.5B

# name -> (layer weight type, classifier type, tied).  A tied model's classifier is its embedding table.
MODELS = {"q8_0": (oc.Q8_0, oc.Q8_0, False), "q8_0-tied": (oc.Q8_0, oc.Q8_0, True), "q4_0": (oc.Q4_0, oc.Q4_0, False),
          "q4_0-tied": (oc.Q4_0, oc.Q4_0, True), "q4_k+q6_k": (oc.Q4_K, oc.Q6_K, False)}
# classifier block scales that put the logits at a few units, so that top-p keeps many candidates and the coin decides
CLS_SCALE = {oc.Q8_0: 0.002, oc.Q4_0: 0.03, oc.Q6_K: 0.0002}

# Kernel launches per generated token with eos < 0 (every step submitted without a host wait), one-token prompt, measured on an H100
# (the same for greedy and sampled steps, f32 and f16 caches, tied and untied classifiers): {streaming weights: {lazy mode: launches}}.
# See test_small_device_loop_fast_modes.
LAUNCHES_PER_TOKEN = {True: {0: 75, 1: 22, 2: 1}, False: {0: 75, 1: 58, 2: 58}}


def small_model(wt, ct, tied, from_raw):
    """make_model's qwen2 (dim 512, 8 heads on 2 kv heads, vocab 1000, 2 layers) with a classifier of type ct at a scale that
    keeps the logits within a few units; tied: that matrix is the embedding table and there is no output weight"""
    w = make_model(wt, from_raw)
    cls = from_raw(random_weight(ct, VOCAB, DIM, np.random.default_rng(77), CLS_SCALE[ct]), [VOCAB, DIM], ct)
    if tied:
        w["token_embed"], w["output_weight"] = cls, None
    else:
        w["output_weight"] = cls
    return w


def small_conf():
    from crabml_b200 import runner as R
    return R.LlamaConfig(HEADS, KV, NL, DIM, HID, 512, VOCAB, 1e-6, ROPE_DIM, "qwen2")


def oracle_small(wt, ct, tied, f16_kv, kv_len):
    odev = OracleDevice()
    w = small_model(wt, ct, tied, lambda raw, shape, t: OracleTensor.from_cpu(raw, shape, t, odev))
    lw = LlamaWeights(w["token_embed"], w["wq"], w["wk"], w["wv"], w["wo"], w["ffn_gate"], w["ffn_down"], w["ffn_up"], w["rms_att"], w["rms_ffn"],
                      w["rms_final"], w["output_weight"], w["bq"], w["bk"], w["bv"])
    return Llama2Runner(OracleTensor, OConf(HEADS, KV, NL, DIM, HID, 512, VOCAB, 1e-6, ROPE_DIM, "qwen2"), lw, odev, kv_len, use_f16_kv_cache=f16_kv)


def device_loop(r, prompt, steps, temperature, topp):
    """(ids, logits[steps, vocab]) of the runner's device-resident loop: generate_greedy_logits for temperature 0, else
    generate_logits"""
    if temperature == 0.0:
        return r.generate_greedy_logits(prompt, steps)
    return r.generate_logits(prompt, steps, temperature, topp, SEED)


def host_loop(r, prompt, steps, temperature, topp, pick):
    """forward -> logits on the host -> pick(logits, temperature, topp, seed, i) -> next forward; r is a runner or the oracle replay"""
    for p, t in enumerate(prompt):
        lg = r.forward([t], p).copy()
    pos, ids, lgs = len(prompt), [], []
    for i in range(steps):
        nxt = pick(lg, temperature, topp, SEED, i)
        ids.append(nxt)
        lgs.append(lg)
        if i + 1 < steps:
            lg = r.forward([nxt], pos).copy()
            pos += 1
    return ids, np.stack(lgs)


def eos_stop(ids, eos):
    """the reference's rule (llama2.rs:141-172): the first id, from the prompt pass, is always yielded; every later step stops before
    yielding EOS"""
    return next((i for i in range(1, len(ids)) if ids[i] == eos), len(ids))


# ---- 1. small qwen2, exact_order: the oracle replay and the reference sampler ---------------------------------------------------------
@pytest.mark.parametrize("model", list(MODELS))
@pytest.mark.parametrize("f16_kv", [False, True])
def test_exact_order_generation_equals_the_oracle_replay(model, f16_kv):
    """generate_logits at (0.8, 0.9) and (1.0, 1.0) and generate_greedy_logits on an exact_order device: the ids of the oracle
    replay picked by sampler_ref.sample (argmax_last for greedy), and the exported logits of every generated position equal to the
    oracle's forward logits at that position, bit for bit"""
    from crabml_b200 import runner as R
    wt, ct, tied = MODELS[model]
    prompt, steps = [1, 600, 42], 24
    kv_len = len(prompt) + steps + 4
    with fresh_device(exact_order=True) as dev:
        w = small_model(wt, ct, tied, _gpu_from_raw(dev))
        for temperature, topp in SAMPLERS:
            r = R.LlamaRunner(dev, small_conf(), w, kv_len, f16_kv=f16_kv)
            ids, logits = device_loop(r, prompt, steps, temperature, topp)
            assert r.kv_cache_len() == len(prompt) + steps - 1
            r.close()
            want_ids, want_logits = host_loop(oracle_small(wt, ct, tied, f16_kv, kv_len), prompt, steps, temperature, topp, S.sample)
            assert np.isfinite(want_logits).all() and np.abs(want_logits).max() > 1e-3
            assert ids == want_ids, (temperature, topp)
            assert_same_bits(logits, want_logits, f"T={temperature} topp={topp}: exported logits vs the oracle replay")
            if temperature == 0.8:
                assert len(set(ids)) > 4, ids                       # the coin decides, the run is not stuck on one id


# ---- 1. small qwen2, fast modes: one another, the fast sampler, the host loop, EOS -----------------------------------------------------
@pytest.mark.parametrize("model", list(MODELS))
@pytest.mark.parametrize("f16_kv", [False, True])
def test_small_device_loop_fast_modes(model, f16_kv):
    """A one-token prompt and SPLIT_FROM + 8 generated tokens, so the persistent attention runs with one CTA per head and then with
    several.  Eager, lazy 1 and lazy 2 give the same ids and logits bit for bit; each id is sample_fast of its exported logits; the
    device loop equals the host loop; EOS (the fifth generated id) stops every mode before yielding it, with the KV cache as long as
    the reference leaves it.  Lazy 2 runs the ring kernel, except for the all-K-quant model, and every flush of both lazy modes is a
    cached graph.

    Launches per token (LAUNCHES_PER_TOKEN): eager runs the replay's per-op kernels, 75 for two layers, the classifier and the
    sampler.  Lazy 1 replays one CUDA graph of 22 fused kernels.  Lazy 2 is one ring-kernel launch per token: the embedding row read
    from the sampled slot, both layers, the classifier and the sample phase.  The Q4_K + Q6_K model launches 58 in both lazy modes:
    its K-quant matvecs and its bias adds stay eager kernels inside the graph, and lazy 2 runs that graph too, because the qwen2
    phases exist only in the ring kernel, which needs a Q8_0 / Q4_0 matvec."""
    from crabml_b200 import runner as R
    wt, ct, tied = MODELS[model]
    streaming = wt in (oc.Q8_0, oc.Q4_0)
    prompt, steps = [7], SPLIT_FROM + 8
    conf = small_conf()
    for temperature, topp in SAMPLERS:
        stop = []                        # (eos, k): the fifth id of eager mode, and where the reference stops on it

        def body(dev):
            w = small_model(wt, ct, tied, _gpu_from_raw(dev))
            r = R.LlamaRunner(dev, conf, w, steps + 4, f16_kv=f16_kv)
            l0 = dev.launch_count()
            ids, logits = device_loop(r, prompt, steps, temperature, topp)
            launches = (dev.launch_count() - l0) / len(ids)
            assert len(ids) == steps and r.kv_cache_len() == len(prompt) + steps - 1
            r.close()
            print(f"{model} f16_kv={f16_kv} T={temperature} topp={topp} lazy={dev.lazy}: {launches:g} launches per token")
            st, variant, host = dev.lazy_stats(), dev.mega_variant(), None
            if dev.lazy == 2:
                r = R.LlamaRunner(dev, conf, w, steps + 4, f16_kv=f16_kv)
                host = host_loop(r, prompt, steps, temperature, topp, S.sample_fast)
                r.close()
            if not stop:
                stop.append((ids[4], eos_stop(ids, ids[4])))
                assert stop[0][1] < steps
            eos, k = stop[0]
            r = R.LlamaRunner(dev, conf, w, steps + 4, f16_kv=f16_kv)
            e_ids = r.generate_greedy(prompt, steps, eos=eos) if temperature == 0.0 else r.generate(prompt, steps, temperature, topp, SEED, eos=eos)
            assert e_ids == ids[:k], (dev.lazy, eos, e_ids, ids[:k + 1])
            assert r.kv_cache_len() == len(prompt) + k        # the step that sampled EOS ran; nothing after it
            r.close()
            return ids, logits, launches, st, variant, host
        runs = run_modes(body)
        ids, logits = runs[0][:2]
        for m in (0, 1, 2):
            assert runs[m][2] == LAUNCHES_PER_TOKEN[streaming][m], (m, runs[m][2])
        for m in (1, 2):
            assert runs[m][0] == ids, f"lazy={m} vs eager ids"
            assert_same_bits(runs[m][1], logits, f"lazy={m} vs eager logits")
            assert runs[m][3]["uncached"] == 0, runs[m][3]
        assert runs[2][4] == (MEGA_RING if streaming else MEGA_NONE), runs[2][4]
        h_ids, h_logits = runs[2][5]
        assert h_ids == runs[2][0], "device loop vs host loop"
        assert_same_bits(runs[2][1], h_logits, "device loop vs host loop")
        assert np.isfinite(logits).all() and np.abs(logits).max() > 1e-3
        assert ids == [S.sample_fast(logits[i], temperature, topp, SEED, i) for i in range(steps)]
        if temperature == 0.8:
            assert len(set(ids)) > 8, ids


# ---- 2. Qwen2-7B shapes on synthetic weights ---------------------------------------------------------------------------------------
def conf_7b(n_layers):
    from crabml_b200 import runner as R
    return R.LlamaConfig(28, 4, n_layers, 3584, 18944, 4096, 152064, 1e-6, 128, "qwen2")


@pytest.mark.parametrize("wt,ct", [(oc.Q8_0, oc.Q8_0), (oc.Q4_0, oc.Q6_K)])
def test_qwen2_7b_device_loop_modes_bit_identical(wt, ct):
    """Greedy and sampled generation, SPLIT_FROM + 8 steps from a one-token prompt, two layers at Qwen2-7B shapes: eager, lazy 1 and
    the ring kernel give the same ids and logits bit for bit, and every id is sample_fast of its logits at vocab 152 064"""
    from crabml_b200 import runner as R
    conf = conf_7b(2)
    steps = SPLIT_FROM + 8
    samplers = [(0.0, 0.0), (0.8, 0.9)]
    def body(dev):
        w = R.synthetic_weights(dev, conf, wt, ct, seed=0x0E2)
        loops = {}
        for temperature, topp in samplers:
            r = R.LlamaRunner(dev, conf, w, steps + 4)
            loops[temperature] = device_loop(r, [1], steps, temperature, topp)
            r.close()
        return loops, dev.lazy_stats(), dev.mega_variant()
    res = run_modes(body)
    for m in (1, 2):
        assert res[m][1]["uncached"] == 0, (m, res[m][1])
    assert res[2][2] == MEGA_RING, res[2][2]
    for temperature, topp in samplers:
        ids, logits = res[0][0][temperature]
        assert len(ids) == steps and np.isfinite(logits).all() and np.abs(logits).max() > 1e-3
        for m in (1, 2):
            assert res[m][0][temperature][0] == ids, f"T={temperature}: lazy={m} vs eager ids"
            assert_same_bits(res[m][0][temperature][1], logits, f"T={temperature}: lazy={m} vs eager logits")
        assert ids == [S.sample_fast(logits[i], temperature, topp, SEED, i) for i in range(steps)], temperature
        if temperature:
            assert len(set(ids)) > 16, ids


def synthetic_twin(conf, wt, ct, seed):
    """runner.synthetic_weights for arch "qwen2" on the host, as LlamaWeights of (raw, shape, type): the same tensor ids in the same
    order (runner.py:234-241), the norms and biases drawn from the same rng in the same order (per-layer norms, rms_final, then every
    bq, every bk, every bv)"""
    from crabml_b200 import runner as R
    dim, hid, kv, L = conf.embedding_dim, conf.hidden_dim, conf.head_size() * conf.n_kv_heads, conf.n_layers
    tid = [0]

    def syn(rows, cols, t):
        tid[0] += 1
        return synth_weight(t, rows, cols, seed, tid[0], R.synth_scale(t, cols)), [rows, cols], t
    rng = np.random.default_rng(seed)

    def vec(v):
        return v.astype(np.float32), [v.size], oc.F32
    lw = LlamaWeights(None, [], [], [], [], [], [], [], [], [], None, None, [], [], [])
    for _ in range(L):
        lw.wq.append(syn(dim, dim, wt)); lw.wk.append(syn(kv, dim, wt)); lw.wv.append(syn(kv, dim, wt)); lw.wo.append(syn(dim, dim, wt))
        lw.ffn_gate_weight.append(syn(hid, dim, wt)); lw.ffn_up_weight.append(syn(hid, dim, wt)); lw.ffn_down_weight.append(syn(dim, hid, wt))
        lw.rms_att_weight.append(vec(1.0 + 0.05 * rng.standard_normal(dim))); lw.rms_ffn_weight.append(vec(1.0 + 0.05 * rng.standard_normal(dim)))
    lw.token_embed = syn(conf.vocab_size, dim, wt)
    lw.output_weight = syn(conf.vocab_size, dim, ct)
    lw.rms_final_weight = vec(1.0 + 0.05 * rng.standard_normal(dim))
    for key, n in (("bq", dim), ("bk", kv), ("bv", kv)):
        getattr(lw, key).extend(vec(0.5 * rng.standard_normal(n)) for _ in range(L))
    return lw


def upload(lw, odev):
    """the (raw, shape, type) LlamaWeights of synthetic_twin as oracle tensors on odev"""
    def up(v):
        return OracleTensor.from_cpu(*v, odev)
    return LlamaWeights(*[[up(v) for v in f] if isinstance(f, list) else up(f) for f in (getattr(lw, d.name) for d in dataclasses.fields(lw))])


def test_qwen2_7b_fast_mode_logits_inside_the_reference_order_band():
    """The ring kernel on Qwen2-7B shapes (GQA group 7, dim 3584, vocab 152 064, q/k/v biases of sigma 0.5), 2 layers, 24 positions,
    f32 and f16 KV cache: per position, the distance of the GPU logits from the reference's AVX2-order logits against the distance
    between the reference's own scalar and AVX2 orders on the same weights, with the assertions of the Llama-2-7B test
    (tests/test_gpu_runner.py).  The synthetic weights are generated once on the host and shared by both orders."""
    from crabml_b200 import runner as R
    nl = 2
    conf = conf_7b(nl)
    seed, wt = 0x0E2, oc.Q8_0
    toks = [int(t) for t in np.random.default_rng(5).integers(1, conf.vocab_size, 24)]
    threads = max(1, min(16, len(os.sched_getaffinity(0))))
    raw = synthetic_twin(conf, wt, wt, seed)
    oconf = OConf(28, 4, nl, 3584, 18944, 4096, 152064, 1e-6, 128, "qwen2")
    for f16_kv in (False, True):
        logits = {}
        for name, flags in (("avx2", oc.ORDER_AVX2), ("scalar", 0)):
            odev = OracleDevice(thread_num=threads, flags=flags)
            lw = upload(raw, odev)
            ro = Llama2Runner(OracleTensor, oconf, lw, odev, 32, use_f16_kv_cache=f16_kv)
            logits[name] = np.stack([ro.forward([t], p).copy() for p, t in enumerate(toks)])
            del ro, lw
        with fresh_device(lazy=2) as dev:
            w = R.synthetic_weights(dev, conf, wt, wt, seed=seed)
            r = R.LlamaRunner(dev, conf, w, 32, f16_kv=f16_kv)
            logits["gpu"] = np.stack([r.forward([t], p).copy() for p, t in enumerate(toks)])
            assert dev.mega_variant() == MEGA_RING and dev.lazy_stats()["uncached"] == 0
            r.close()
        scale = np.abs(logits["avx2"]).max(axis=1)
        ours = np.abs(logits["gpu"] - logits["avx2"]).max(axis=1) / scale
        band = np.abs(logits["scalar"] - logits["avx2"]).max(axis=1) / scale
        q = lambda a: [float(np.percentile(a, p)) for p in (0, 25, 50, 75, 100)]      # noqa: E731
        print(f"qwen2-7B-shaped {nl}-layer model, f16_kv={f16_kv}, {len(toks)} positions:")
        print("  |gpu - ref(avx2 order)| / max|logit|   min/25/50/75/max =", ["%.2e" % v for v in q(ours)])
        print("  |ref(scalar) - ref(avx2)| / max|logit| min/25/50/75/max =", ["%.2e" % v for v in q(band)])
        assert np.isfinite(logits["gpu"]).all()
        assert np.median(ours) <= 1.0 * np.median(band) * 1.5 and ours.max() <= 1.5 * band.max(), (q(ours), q(band))
        same = logits["scalar"].argmax(1) == logits["avx2"].argmax(1)
        assert (logits["gpu"].argmax(1)[same] == logits["avx2"].argmax(1)[same]).mean() >= 0.9
