"""Python handle on the C++ Llama2Runner replay (crabml_b200/csrc/host/llama2_runner.cpp) plus the two ways
this repo builds a model: from a GGUF file (python `gguf` reader -> Tensor::from_cpu, the quantized relaxation of
crabml-llama2/src/model.rs:817-837) and synthetic weights generated on the device (SURVEY §8d configs 3-5)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import capi, sharding
from .capi import CudaError, TensorError
from .tensor import CudaTensor, CudaTensorDevice


@dataclass
class LlamaConfig:                      # crabml-llama2/src/model.rs:30-53
    n_heads: int
    n_kv_heads: int
    n_layers: int
    embedding_dim: int
    hidden_dim: int
    seq_len: int
    vocab_size: int
    rms_norm_eps: float = 1e-5
    rope_dim: int = 0
    arch: str = "llama"                 # ModelArchitecture (model.rs:21-27): "llama" | "qwen2" | "gemma"

    def head_size(self):
        return self.embedding_dim // self.n_heads


LLAMA2_7B = LlamaConfig(32, 32, 32, 4096, 11008, 4096, 32000, 1e-5, 128)
MISTRAL_7B = LlamaConfig(32, 8, 32, 4096, 14336, 4096, 32000, 1e-5, 128)
TINYLLAMAS_15M = LlamaConfig(6, 6, 6, 288, 768, 256, 32000, 1e-5, 48)

# GGUF block bytes / elements (SURVEY Appendix A) -- for algorithmic byte accounting
BLOCK = {capi.F32: (4, 1), capi.F16: (2, 1), capi.Q4_0: (18, 32), capi.Q4_1: (20, 32), capi.Q5_0: (22, 32), capi.Q5_1: (24, 32),
         capi.Q8_0: (34, 32), capi.Q2_K: (84, 256), capi.Q3_K: (110, 256), capi.Q4_K: (144, 256), capi.Q5_K: (176, 256),
         capi.Q6_K: (210, 256), capi.Q8_K: (292, 256)}


def weight_bytes(dtype, rows, cols):
    bb, be = BLOCK[dtype]
    return rows * (cols // be) * bb


class LlamaRunner:
    def __init__(self, device: CudaTensorDevice, conf: LlamaConfig, weights: dict, kv_seq_len: int, f16_kv: bool = False,
                 plan: "sharding.ShardPlan | None" = None):
        """plan: this rank's ShardPlan when `weights` are shards (device.init_comm must have been called)."""
        self.device, self.conf, self.weights, self.plan = device, conf, weights, plan          # keep the tensors alive
        L = conf.n_layers
        cconf = capi.ccr_llama_config(conf.n_heads, conf.n_kv_heads, L, conf.embedding_dim, conf.hidden_dim, conf.seq_len,
                                      conf.vocab_size, conf.rope_dim or 0, conf.rms_norm_eps, int(f16_kv),
                                      plan.rank if plan else 0, plan.world if plan else 1, plan.hidden_local if plan else conf.hidden_dim,
                                      {"llama": 0, "qwen2": 1, "gemma": 2}[conf.arch])

        def arr(key):
            a = (C.c_void_p * L)(*[t.buf.handle.value for t in weights[key]])
            self._keep.append(a)
            return C.cast(a, C.POINTER(C.c_void_p))
        self._keep = []
        cw = capi.ccr_llama_weights(weights["token_embed"].buf.handle, arr("wq"), arr("wk"), arr("wv"), arr("wo"), arr("ffn_gate"),
                                    arr("ffn_down"), arr("ffn_up"), arr("rms_att"), arr("rms_ffn"), weights["rms_final"].buf.handle,
                                    weights["output_weight"].buf.handle if weights.get("output_weight") is not None else None,
                                    arr("bq") if "bq" in weights else None, arr("bk") if "bk" in weights else None, arr("bv") if "bv" in weights else None)
        h = C.c_void_p()
        rc = device.lib.ccr_runner_create(device.handle, C.byref(cconf), C.byref(cw), kv_seq_len, C.byref(h))
        if rc != capi.CC_OK:
            raise CudaError(f"ccr_runner_create failed [{rc}]: {device.lib.cc_last_error(device.handle).decode()}")
        self.handle = h
        self.logits = np.zeros(conf.vocab_size, np.float32)

    def _check(self, rc):
        if rc == capi.CC_OK:
            return
        msg = self.device.lib.ccr_runner_last_error(self.handle).decode()
        raise (TensorError if rc == capi.CC_ERR_TENSOR else CudaError)(msg)

    def forward(self, tokens, pos, export=True):
        """Llama2Runner::forward (llama2.rs:184-211).  export=False skips the device->host logits copy."""
        arr = (C.c_int64 * len(tokens))(*[int(t) for t in tokens])
        out = self.logits.ctypes.data_as(C.c_void_p) if export else None
        self._check(self.device.lib.ccr_runner_forward(self.handle, arr, len(tokens), pos, out))
        return self.logits

    def kv_cache_len(self):
        return int(self.device.lib.ccr_runner_kv_cache_len(self.handle))

    def generate_greedy(self, prompt, steps, eos=-1):
        p = (C.c_int64 * len(prompt))(*[int(t) for t in prompt])
        out = (C.c_int64 * max(1, steps))()
        n = C.c_int32(0)
        self._check(self.device.lib.ccr_runner_generate_greedy(self.handle, p, len(prompt), steps, eos, out, C.byref(n)))
        return [int(out[i]) for i in range(n.value)]

    def generate_greedy_logits(self, prompt, steps):
        """ccr_runner_generate_greedy_ex with eos < 0: every step is submitted without waiting for the host (sampling on the device, the
        sampled id feeds the next step from a device slot); returns (ids, logits[steps, vocab]) -- the logits of every generated
        position are exported asynchronously through a pinned staging ring."""
        p = (C.c_int64 * len(prompt))(*[int(t) for t in prompt])
        out = (C.c_int64 * max(1, steps))()
        n = C.c_int32(0)
        logits = np.zeros((max(1, steps), self.conf.vocab_size), np.float32)
        self._check(self.device.lib.ccr_runner_generate_greedy_ex(self.handle, p, len(prompt), steps, -1, out, C.byref(n),
                                                                  logits.ctypes.data_as(C.c_void_p)))
        return [int(out[i]) for i in range(n.value)], logits[:n.value]

    def _generate_ex(self, prompt, steps, temperature, topp, seed, eos, logits):
        p = (C.c_int64 * len(prompt))(*[int(t) for t in prompt])
        out = (C.c_int64 * max(1, steps))()
        n = C.c_int32(0)
        self._check(self.device.lib.ccr_runner_generate_ex(self.handle, p, len(prompt), steps, eos, float(temperature), float(topp),
                                                           int(seed) & (2**64 - 1), out, C.byref(n),
                                                           None if logits is None else logits.ctypes.data_as(C.c_void_p)))
        return [int(out[i]) for i in range(n.value)]

    def generate(self, prompt, steps, temperature, topp, seed, eos=-1):
        """ccr_runner_generate_ex: the greedy loop with Llama2Sampler (sampler.rs:27-107) on the device; the coin of generated
        token i is coin index i of `seed`.  temperature 0 is generate_greedy."""
        return self._generate_ex(prompt, steps, temperature, topp, seed, eos, None)

    def generate_logits(self, prompt, steps, temperature, topp, seed, eos=-1):
        """generate, also returning the logits of every generated position (as generate_greedy_logits): (ids, logits[n, vocab])."""
        logits = np.zeros((max(1, steps), self.conf.vocab_size), np.float32)
        ids = self._generate_ex(prompt, steps, temperature, topp, seed, eos, logits)
        return ids, logits[:len(ids)]

    def close(self):
        if self.handle:
            self.device.lib.ccr_runner_destroy(self.handle)
            self.handle = None

    # algorithmic weight bytes streamed per decoded token (SURVEY §8d): every matmul weight once (THIS rank's shards)
    def weight_bytes_per_token(self):
        w = self.weights
        total = 0
        for key in ("wq", "wk", "wv", "wo", "ffn_gate", "ffn_up", "ffn_down"):
            for t in w[key]:
                r, c = t.shape()
                total += weight_bytes(t.dtype(), r, c)
        ow = w.get("output_weight") if w.get("output_weight") is not None else w["token_embed"]
        r, c = ow.shape()
        return total + weight_bytes(ow.dtype(), r, c)


def load_gguf(path: str, device: CudaTensorDevice, shard=None, f16_kv=False):
    """-> (LlamaConfig, weights dict, tokenizer dict).  Dims are reversed into [rows, cols] (model.rs:474).
    shard = (rank, world): upload only this rank's rows / block columns (sharding.py); the plan is returned as w["plan"]."""
    import gguf
    rd = gguf.GGUFReader(path)
    f = rd.fields

    def scalar(k):
        return f[k].parts[f[k].data[0]][0]
    arch = bytes(f["general.architecture"].parts[f["general.architecture"].data[0]]).decode()
    if arch not in ("llama", "qwen2"):                    # model.rs:285-351, 559
        raise TensorError(f"unsupported architecture {arch}")
    if arch == "qwen2" and shard is not None and shard[1] > 1:
        raise TensorError("sharding: only the llama forward is sharded")
    tokens = [bytes(f["tokenizer.ggml.tokens"].parts[i]).decode("utf-8") for i in f["tokenizer.ggml.tokens"].data]
    conf = LlamaConfig(int(scalar(f"{arch}.attention.head_count")), int(scalar(f"{arch}.attention.head_count_kv")),
                       int(scalar(f"{arch}.block_count")), int(scalar(f"{arch}.embedding_length")),
                       int(scalar(f"{arch}.feed_forward_length")), int(scalar(f"{arch}.context_length")), len(tokens),
                       float(np.float32(scalar(f"{arch}.attention.layer_norm_rms_epsilon"))),
                       int(scalar(f"{arch}.rope.dimension_count")) if f"{arch}.rope.dimension_count" in f else 0, arch)
    # RoPE runs at base 10000 for every architecture, as in the reference (rope.rs:48,69 hard-code it): `{arch}.rope.freq_base` is
    # deliberately not read, so a qwen2 file decodes as the reference decodes it (DESIGN.md §7)
    tensors = {t.name: t for t in rd.tensors}

    plan = None
    if shard is not None and shard[1] > 1:
        plan = sharding.make_plan(conf.n_heads, conf.n_kv_heads, conf.embedding_dim, conf.hidden_dim, conf.vocab_size,
                                  int(tensors["blk.0.ffn_down.weight"].tensor_type), shard[0], shard[1], f16_kv)

    def load(name, kind=None):
        t = tensors[name]
        shape = [int(d) for d in reversed(t.shape.tolist())]
        data = np.ascontiguousarray(t.data).view(np.uint8).reshape(-1)
        if plan is not None and kind is not None:
            data, shape = sharding.shard_bytes(kind, data, shape[0], shape[1], int(t.tensor_type), plan)
        return CudaTensor.from_cpu(data, shape, int(t.tensor_type), device)
    L = conf.n_layers
    names = {"wq": "attn_q", "wk": "attn_k", "wv": "attn_v", "wo": "attn_output", "ffn_gate": "ffn_gate", "ffn_down": "ffn_down",
             "ffn_up": "ffn_up", "rms_att": "attn_norm", "rms_ffn": "ffn_norm"}
    w = {k: [load(f"blk.{l}.{v}.weight", k) for l in range(L)] for k, v in names.items()}
    if arch == "qwen2":
        for k, v in (("bq", "attn_q"), ("bk", "attn_k"), ("bv", "attn_v")):
            w[k] = [load(f"blk.{l}.{v}.bias") for l in range(L)]
    w["token_embed"] = load("token_embd.weight")
    w["rms_final"] = load("output_norm.weight")
    if "output.weight" in tensors:
        w["output_weight"] = load("output.weight", "output_weight")
    else:           # tied classifier (llama2.rs:201-206): the sharded path needs its own row shard of token_embd
        w["output_weight"] = load("token_embd.weight", "output_weight") if plan is not None else None
    w["plan"] = plan
    tok = {"tokens": tokens, "scores": [float(f["tokenizer.ggml.scores"].parts[i][0]) for i in f["tokenizer.ggml.scores"].data],
           "bos": int(scalar("tokenizer.ggml.bos_token_id")), "eos": int(scalar("tokenizer.ggml.eos_token_id"))}
    return conf, w, tok


# central f16 scale of synthetic blocks so that a dequantized row has sigma_w ~ 1/sqrt(k) (SURVEY §8d-3)
_Q_SIGMA = {capi.Q8_0: 73.9, capi.Q4_0: 4.61, capi.Q4_1: 4.61, capi.Q5_0: 9.23, capi.Q5_1: 9.23,
            capi.Q2_K: 1.12 * 8.0, capi.Q3_K: 2.29 * 18.5, capi.Q4_K: 4.61 * 31.5, capi.Q5_K: 9.23 * 31.5, capi.Q6_K: 18.5 * 73.9, capi.Q8_K: 73.9}


def synth_scale(dtype, k):
    return float(1.0 / (_Q_SIGMA[dtype] * np.sqrt(k)))


def synthetic_weights(device: CudaTensorDevice, conf: LlamaConfig, wtype: int, classifier_type: int | None = None,
                      seed: int = 0x5EED, plan: "sharding.ShardPlan | None" = None):
    """Valid, non-degenerate random blocks generated ON the device (never shipped from the host).
    plan: generate only this rank's shard of every tensor (same bytes as the corresponding slice of the full model)."""
    ct = wtype if classifier_type is None else classifier_type
    dim, hid, kv = conf.embedding_dim, conf.hidden_dim, conf.head_size() * conf.n_kv_heads
    tid = [0]

    def syn(rows, cols, t, kind=None):
        tid[0] += 1
        if plan is None or plan.world == 1 or kind not in sharding.CUTS:
            return CudaTensor.synth([rows, cols], t, device, seed, tid[0], synth_scale(t, cols))
        how, attr = sharding.CUTS[kind]
        first, count = getattr(plan, attr)
        r0, nr, c0, nc = (first, count, 0, cols) if how == "rows" else (0, rows, first, count)
        return CudaTensor.synth_slice([rows, cols], t, device, seed, tid[0], synth_scale(t, cols), r0, nr, c0, nc)
    rng = np.random.default_rng(seed)

    def norm():
        return CudaTensor.from_cpu((1.0 + 0.05 * rng.standard_normal(dim)).astype(np.float32), [dim], capi.F32, device)
    L = conf.n_layers
    w = {"wq": [], "wk": [], "wv": [], "wo": [], "ffn_gate": [], "ffn_down": [], "ffn_up": [], "rms_att": [], "rms_ffn": []}
    for _ in range(L):
        w["wq"].append(syn(dim, dim, wtype, "wq")); w["wk"].append(syn(kv, dim, wtype, "wk")); w["wv"].append(syn(kv, dim, wtype, "wv"))
        w["wo"].append(syn(dim, dim, wtype, "wo"))
        w["ffn_gate"].append(syn(hid, dim, wtype, "ffn_gate")); w["ffn_up"].append(syn(hid, dim, wtype, "ffn_up"))
        w["ffn_down"].append(syn(dim, hid, wtype, "ffn_down"))
        w["rms_att"].append(norm()); w["rms_ffn"].append(norm())
    w["token_embed"] = syn(conf.vocab_size, dim, wtype)
    w["output_weight"] = syn(conf.vocab_size, dim, ct, "output_weight")
    w["rms_final"] = norm()
    if conf.arch == "qwen2":                # q/k/v biases (llama2.rs:315-317), of the size of a matvec output element
        for k, n in (("bq", dim), ("bk", kv), ("bv", kv)):
            w[k] = [CudaTensor.from_cpu((0.5 * rng.standard_normal(n)).astype(np.float32), [n], capi.F32, device) for _ in range(L)]
    return w
