"""The other architectures' forwards (SURVEY 8f-4; llama2.rs:283-352 qwen2, :455-524 gemma) through the C++ runner on the GPU:
q/k/v bias adds, Neox RoPE, GeLU ffn through the f16 LUT, the sqrt(dim) embedding scale and the tied classifier, with grouped-query
attention.  exact_order mode must reproduce the oracle replay of the same forward bit for bit; the fast modes must agree with each
other bit for bit and stay close to the oracle."""
import numpy as np
import pytest

from oracle import oracle as oc
from oracle.llama_replay import Llama2Runner, LlamaConfig as OConf, LlamaWeights
from oracle.tensor_ref import OracleDevice, OracleTensor
from tests.blockgen import random_weight
from tests.gpu_common import assert_same_bits, fresh_device, run_modes

pytestmark = pytest.mark.gpu

DIM, HID, HEADS, KV, HD, VOCAB, NL = 256, 512, 8, 4, 32, 640, 3


def make_model(arch, T, dev, wt, from_raw):
    rng = np.random.default_rng(77)
    raws = {}

    def qw(name, rows, cols):
        raws[name] = random_weight(wt, rows, cols, rng, 0.05)
        return from_raw(raws[name], [rows, cols], wt)

    def f32(n, mean=0.0, std=0.1):
        return from_raw((mean + std * rng.standard_normal(n)).astype(np.float32), [n], oc.F32)
    w = dict(token_embed=qw("embed", VOCAB, DIM), wq=[], wk=[], wv=[], wo=[], ffn_gate=[], ffn_up=[], ffn_down=[], rms_att=[], rms_ffn=[], bq=[], bk=[], bv=[])
    for l in range(NL):
        w["wq"].append(qw(f"wq{l}", HEADS * HD, DIM)); w["wk"].append(qw(f"wk{l}", KV * HD, DIM)); w["wv"].append(qw(f"wv{l}", KV * HD, DIM))
        w["wo"].append(qw(f"wo{l}", DIM, HEADS * HD)); w["ffn_gate"].append(qw(f"g{l}", HID, DIM)); w["ffn_up"].append(qw(f"u{l}", HID, DIM))
        w["ffn_down"].append(qw(f"d{l}", DIM, HID)); w["rms_att"].append(f32(DIM, 1.0, 0.05)); w["rms_ffn"].append(f32(DIM, 1.0, 0.05))
        w["bq"].append(f32(HEADS * HD)); w["bk"].append(f32(KV * HD)); w["bv"].append(f32(KV * HD))
    w["rms_final"] = f32(DIM, 1.0, 0.05)
    w["output_weight"] = None if arch == "gemma" else qw("out", VOCAB, DIM)
    if arch != "qwen2":
        for k in ("bq", "bk", "bv"):
            del w[k]
    return w


def oracle_logits(arch, wt, tokens, f16_kv):
    odev = OracleDevice()
    w = make_model(arch, OracleTensor, odev, wt, lambda raw, shape, t: OracleTensor.from_cpu(raw, shape, t, odev))
    lw = LlamaWeights(w["token_embed"], w["wq"], w["wk"], w["wv"], w["wo"], w["ffn_gate"], w["ffn_down"], w["ffn_up"], w["rms_att"], w["rms_ffn"],
                      w["rms_final"], w["output_weight"], w.get("bq"), w.get("bk"), w.get("bv"))
    r = Llama2Runner(OracleTensor, OConf(HEADS, KV, NL, DIM, HID, 64, VOCAB, 1e-6, HD, arch), lw, odev, 32, use_f16_kv_cache=f16_kv)
    return np.stack([r.forward([t], p).copy() for p, t in enumerate(tokens)])


def gpu_logits(arch, wt, tokens, f16_kv):
    """-> body(dev): the logits of every token"""
    from crabml_b200 import CudaTensor
    from crabml_b200 import runner as R

    def body(dev):
        w = make_model(arch, CudaTensor, dev, wt, lambda raw, shape, t: CudaTensor.from_cpu(raw, shape, t, dev))
        conf = R.LlamaConfig(HEADS, KV, NL, DIM, HID, 64, VOCAB, 1e-6, HD, arch)
        r = R.LlamaRunner(dev, conf, w, 32, f16_kv=f16_kv)
        out = np.stack([r.forward([t], p).copy() for p, t in enumerate(tokens)])
        r.close()
        return out
    return body


@pytest.mark.parametrize("arch", ["qwen2", "gemma"])
@pytest.mark.parametrize("wt", [oc.Q8_0, oc.Q4_K])
def test_other_architectures_exact_and_fast(arch, wt):
    tokens = [1, 77, 300, 5, 639, 42]
    f16_kv = True                              # grouped-query attention (8 heads on 4 kv heads) with the f16 cache, the CLI default (main.rs:250)
    want = oracle_logits(arch, wt, tokens, f16_kv)
    assert np.isfinite(want).all() and np.abs(want).max() > 1e-3
    with fresh_device(exact_order=True) as dev:
        exact = gpu_logits(arch, wt, tokens, f16_kv)(dev)
    assert_same_bits(exact, want, f"{arch}: exact_order vs the oracle replay")
    fast = run_modes(gpu_logits(arch, wt, tokens, f16_kv))
    for m in (1, 2):
        assert_same_bits(fast[m], fast[0], f"{arch}: lazy={m} vs eager")
    rel = float(np.abs(fast[0] - want).max() / np.abs(want).max())
    assert rel < 3e-2, (arch, rel)
