"""Qwen2 (llama2.rs:283-352) through every execution mode: the q/k/v bias adds fused into the streaming q/k/v matvec as its per-matrix
epilogue, Neox RoPE in the fused and persistent attention, and one persistent kernel per token in lazy mode 2.  Eager, lazy 1 and lazy 2
must agree bit for bit; exact_order must reproduce the oracle replay bit for bit; the fast modes must stay inside the order band of the
Llama tests.  Also: qwen2 GGUF files (tied and untied classifier) load into the same logits as the same weights passed in directly, and a
sharded qwen2 load is refused."""
import numpy as np
import pytest

from oracle import oracle as oc
from oracle.llama_replay import Llama2Runner, LlamaConfig as OConf, LlamaWeights
from oracle.tensor_ref import OracleDevice, OracleTensor
from crabml_b200.tensor import MEGA_RING
from tests.blockgen import random_weight
from tests.gpu_common import assert_same_bits, fresh_device, run_modes

pytestmark = pytest.mark.gpu

SPLIT_FROM = 320                        # AT_SPLIT_MIN_KV: from this many cached positions the persistent attention runs S CTAs per head


def _run_modes(make, conf, tokens, checkpoints, f16_kv, kv_len):
    """logits at `checkpoints` for each lazy mode, bit-identical; in mode 2 every checkpoint is one persistent ring kernel"""
    from crabml_b200 import runner as R

    def body(dev):
        r = R.LlamaRunner(dev, conf, make(dev), kv_len, f16_kv=f16_kv)
        got, kernels = [], []
        for p, t in enumerate(tokens):
            if p not in checkpoints:
                r.forward([t], p, export=False)
                continue
            l0 = dev.launch_count()
            got.append(r.forward([t], p).copy())
            kernels.append((p, dev.launch_count() - l0, dev.mega_variant()))
        st = dev.lazy_stats()
        r.close()
        return np.stack(got), kernels, st
    out = run_modes(body)
    for p, launches, variant in out[2][1]:
        assert (launches, variant) == (1, MEGA_RING), (p, launches, variant)
    for m in (1, 2):
        assert out[m][2]["uncached"] == 0, (m, out[m][2])
    assert np.isfinite(out[0][0]).all() and np.abs(out[0][0]).max() > 1e-3
    for m in (1, 2):
        assert_same_bits(out[m][0], out[0][0], f"lazy={m} vs lazy=0")
    return {m: v[0] for m, v in out.items()}


# ---- Qwen2-7B shapes: dim 3584, 28 heads on 4 kv heads, head_dim 128, hidden 18944, vocab 152064; two layers ------------------------
@pytest.mark.parametrize("wt,ct", [(oc.Q8_0, oc.Q8_0), (oc.Q4_0, oc.Q6_K)])
@pytest.mark.parametrize("f16_kv", [False, True])
def test_qwen2_7b_shapes_modes_bit_identical(wt, ct, f16_kv):
    from crabml_b200 import runner as R
    conf = R.LlamaConfig(28, 4, 2, 3584, 18944, 4096, 152064, 1e-6, 128, "qwen2")
    rng = np.random.default_rng(11)
    n = SPLIT_FROM + 8
    tokens = [int(t) for t in rng.integers(0, conf.vocab_size, n)]
    checkpoints = {0, 1, 2, 63, 200, SPLIT_FROM - 1, SPLIT_FROM, SPLIT_FROM + 1, n - 1}       # both attention instantiations
    _run_modes(lambda dev: R.synthetic_weights(dev, conf, wt, ct, seed=0x0E2), conf, tokens, checkpoints, f16_kv, n + 4)


# ---- small shapes on random blocks, against the oracle replay --------------------------------------------------------------------------
DIM, HID, HEADS, KV, VOCAB, NL = 512, 1024, 8, 2, 1000, 2           # head_dim 64, as Qwen2-0.5B


def make_model(wt, from_raw, seed=5):
    rng = np.random.default_rng(seed)
    hd = DIM // HEADS

    def qw(rows, cols):
        return from_raw(random_weight(wt, rows, cols, rng, 0.05), [rows, cols], wt)

    def f32(n, mean=0.0, std=0.1):
        return from_raw((mean + std * rng.standard_normal(n)).astype(np.float32), [n], oc.F32)
    w = dict(token_embed=qw(VOCAB, DIM), wq=[], wk=[], wv=[], wo=[], ffn_gate=[], ffn_up=[], ffn_down=[], rms_att=[], rms_ffn=[], bq=[], bk=[], bv=[])
    for _ in range(NL):
        w["wq"].append(qw(DIM, DIM)); w["wk"].append(qw(KV * hd, DIM)); w["wv"].append(qw(KV * hd, DIM)); w["wo"].append(qw(DIM, DIM))
        w["ffn_gate"].append(qw(HID, DIM)); w["ffn_up"].append(qw(HID, DIM)); w["ffn_down"].append(qw(DIM, HID))
        w["rms_att"].append(f32(DIM, 1.0, 0.05)); w["rms_ffn"].append(f32(DIM, 1.0, 0.05))
        w["bq"].append(f32(DIM, 0.0, 0.5)); w["bk"].append(f32(KV * hd, 0.0, 0.5)); w["bv"].append(f32(KV * hd, 0.0, 0.5))
    w["rms_final"] = f32(DIM, 1.0, 0.05)
    w["output_weight"] = qw(VOCAB, DIM)
    return w


def _gpu_from_raw(dev):
    from crabml_b200 import CudaTensor
    return lambda raw, shape, t: CudaTensor.from_cpu(raw, shape, t, dev)


def oracle_logits(wt, rope_dim, tokens, f16_kv, flags=0):
    odev = OracleDevice(flags=flags)
    w = make_model(wt, lambda raw, shape, t: OracleTensor.from_cpu(raw, shape, t, odev))
    lw = LlamaWeights(w["token_embed"], w["wq"], w["wk"], w["wv"], w["wo"], w["ffn_gate"], w["ffn_down"], w["ffn_up"], w["rms_att"], w["rms_ffn"],
                      w["rms_final"], w["output_weight"], w["bq"], w["bk"], w["bv"])
    r = Llama2Runner(OracleTensor, OConf(HEADS, KV, NL, DIM, HID, 512, VOCAB, 1e-6, rope_dim, "qwen2"), lw, odev, len(tokens) + 4, use_f16_kv_cache=f16_kv)
    return np.stack([r.forward([t], p).copy() for p, t in enumerate(tokens)])


def _small_fast_modes(wt, rope_dim, f16_kv, tokens, checkpoints):
    from crabml_b200 import runner as R
    conf = R.LlamaConfig(HEADS, KV, NL, DIM, HID, 512, VOCAB, 1e-6, rope_dim, "qwen2")
    return _run_modes(lambda dev: make_model(wt, _gpu_from_raw(dev)), conf, tokens, checkpoints, f16_kv, len(tokens) + 4)


def _tokens(wt, rope_dim):
    return [int(t) for t in np.random.default_rng(rope_dim + wt).integers(0, VOCAB, SPLIT_FROM + 6)]


@pytest.mark.parametrize("wt", [oc.Q8_0, oc.Q4_0])
@pytest.mark.parametrize("rope_dim", [32, 64])            # 32: partial neox, pairs (j, j + head_dim/2) for j < 16
@pytest.mark.parametrize("f16_kv", [False, True])
def test_qwen2_small_exact_and_modes(wt, rope_dim, f16_kv):
    """exact_order is the oracle replay bit for bit; eager, lazy 1 and lazy 2 agree bit for bit on both sides of the split threshold"""
    from crabml_b200 import runner as R
    conf = R.LlamaConfig(HEADS, KV, NL, DIM, HID, 512, VOCAB, 1e-6, rope_dim, "qwen2")
    tokens = _tokens(wt, rope_dim)
    n_oracle = 12
    want = oracle_logits(wt, rope_dim, tokens[:n_oracle], f16_kv)
    with fresh_device(exact_order=True) as dev:
        r = R.LlamaRunner(dev, conf, make_model(wt, _gpu_from_raw(dev)), n_oracle + 4, f16_kv=f16_kv)
        got = np.stack([r.forward([t], p).copy() for p, t in enumerate(tokens[:n_oracle])])
        r.close()
    assert_same_bits(got, want, "exact_order vs the oracle replay")
    _small_fast_modes(wt, rope_dim, f16_kv, tokens, {0, 1, 2, SPLIT_FROM - 1, SPLIT_FROM, len(tokens) - 1})


@pytest.mark.parametrize("rope_dim", [32, 64])
def test_qwen2_fast_modes_inside_the_llama_order_band(fixture_path, rope_dim):
    """the fast modes stay as close to the oracle replay as the Llama tests require of Llama (tests/test_gpu_llama.py)"""
    from tests.test_gpu_llama import _band
    fixture_path("tinyllamas-stories-15m-q8_0.gguf")          # the band is taken on it
    wt, f16_kv, n = oc.Q8_0, True, 12
    tokens = _tokens(wt, rope_dim)[:n]
    want = oracle_logits(wt, rope_dim, tokens, f16_kv)
    fast = _small_fast_modes(wt, rope_dim, f16_kv, tokens, set(range(n)))
    rel = float((np.abs(fast[0] - want).max(1) / np.abs(want).max(1)).max())
    band = _band()
    print(f"qwen2 rope_dim {rope_dim}: fast modes vs the oracle replay {rel:.3e}; llama order band {band:.3e}")
    assert rel <= 1.5 * band, (rel, band)


# ---- GGUF ---------------------------------------------------------------------------------------------------------------------------
def _write_gguf(path, wt, rope_dim, tied):
    import gguf
    rng = np.random.default_rng(9)
    hd = DIM // HEADS
    raw = {}
    wr = gguf.GGUFWriter(path, "qwen2")
    wr.add_block_count(NL); wr.add_context_length(512); wr.add_embedding_length(DIM); wr.add_feed_forward_length(HID)
    wr.add_head_count(HEADS); wr.add_head_count_kv(KV); wr.add_layer_norm_rms_eps(1e-6); wr.add_rope_dimension_count(rope_dim)
    wr.add_rope_freq_base(1000000.0)                     # present in real qwen2 files; the reference (and this project) run at 10000
    wr.add_tokenizer_model("gpt2")
    wr.add_token_list([f"t{i}" for i in range(VOCAB)]); wr.add_token_scores([0.0] * VOCAB)
    wr.add_bos_token_id(1); wr.add_eos_token_id(2)

    def q(name, rows, cols):
        b = random_weight(wt, rows, cols, rng, 0.05)
        raw[name] = (b, [rows, cols], wt)
        wr.add_tensor(name, b.reshape(rows, -1), raw_dtype=gguf.GGMLQuantizationType(wt))

    def f(name, n, mean, std):
        v = (mean + std * rng.standard_normal(n)).astype(np.float32)
        raw[name] = (v, [n], oc.F32)
        wr.add_tensor(name, v)
    q("token_embd.weight", VOCAB, DIM)
    for l in range(NL):
        q(f"blk.{l}.attn_q.weight", DIM, DIM); q(f"blk.{l}.attn_k.weight", KV * hd, DIM); q(f"blk.{l}.attn_v.weight", KV * hd, DIM)
        f(f"blk.{l}.attn_q.bias", DIM, 0.0, 0.5); f(f"blk.{l}.attn_k.bias", KV * hd, 0.0, 0.5); f(f"blk.{l}.attn_v.bias", KV * hd, 0.0, 0.5)
        q(f"blk.{l}.attn_output.weight", DIM, DIM)
        q(f"blk.{l}.ffn_gate.weight", HID, DIM); q(f"blk.{l}.ffn_up.weight", HID, DIM); q(f"blk.{l}.ffn_down.weight", DIM, HID)
        f(f"blk.{l}.attn_norm.weight", DIM, 1.0, 0.05); f(f"blk.{l}.ffn_norm.weight", DIM, 1.0, 0.05)
    f("output_norm.weight", DIM, 1.0, 0.05)
    if not tied:
        q("output.weight", VOCAB, DIM)
    wr.write_header_to_file(); wr.write_kv_data_to_file(); wr.write_tensors_to_file(); wr.close()
    return raw


@pytest.mark.parametrize("tied", [False, True])
@pytest.mark.parametrize("lazy", [0, 1, 2])
def test_qwen2_gguf_loads_into_the_same_logits(tmp_path, tied, lazy):
    from crabml_b200 import runner as R
    path = str(tmp_path / "qwen2.gguf")
    raw = _write_gguf(path, oc.Q8_0, 32, tied)
    tokens = [1, 77, 300, 5, 999, 42, 7]
    with fresh_device(lazy=lazy) as dev:
        conf, w, tok = R.load_gguf(path, dev)
        assert (conf.arch, conf.n_heads, conf.n_kv_heads, conf.n_layers, conf.embedding_dim, conf.hidden_dim, conf.seq_len, conf.vocab_size,
                conf.rope_dim) == ("qwen2", HEADS, KV, NL, DIM, HID, 512, VOCAB, 32)
        assert conf.rms_norm_eps == np.float32(1e-6) and tok["bos"] == 1 and tok["eos"] == 2
        assert (w["output_weight"] is None) == tied and len(w["bq"]) == NL
        r = R.LlamaRunner(dev, conf, w, 16)
        got = np.stack([r.forward([t], p).copy() for p, t in enumerate(tokens)])
        r.close()
        up = _gpu_from_raw(dev)

        def up_raw(name):
            return up(*raw[name])
        names = {"wq": "attn_q.weight", "wk": "attn_k.weight", "wv": "attn_v.weight", "wo": "attn_output.weight", "ffn_gate": "ffn_gate.weight",
                 "ffn_up": "ffn_up.weight", "ffn_down": "ffn_down.weight", "rms_att": "attn_norm.weight", "rms_ffn": "ffn_norm.weight",
                 "bq": "attn_q.bias", "bk": "attn_k.bias", "bv": "attn_v.bias"}
        direct = {k: [up_raw(f"blk.{l}.{v}") for l in range(NL)] for k, v in names.items()}
        direct.update(token_embed=up_raw("token_embd.weight"), rms_final=up_raw("output_norm.weight"),
                      output_weight=None if tied else up_raw("output.weight"))
        r = R.LlamaRunner(dev, conf, direct, 16)
        want = np.stack([r.forward([t], p).copy() for p, t in enumerate(tokens)])
        r.close()
    assert np.isfinite(want).all() and np.abs(want).max() > 1e-3
    assert_same_bits(got, want, "the gguf load vs the same weights passed in")


def test_qwen2_gguf_sharded_load_is_refused(tmp_path):
    from crabml_b200 import runner as R
    from crabml_b200.capi import TensorError
    path = str(tmp_path / "qwen2.gguf")
    _write_gguf(path, oc.Q8_0, 64, True)
    with fresh_device() as dev, pytest.raises(TensorError, match="sharding"):
        R.load_gguf(path, dev, shard=(0, 2))
