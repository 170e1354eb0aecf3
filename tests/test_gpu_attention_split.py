"""The persistent kernels' attention phase split over S CTAs per head (mega_phases.cuh phase_attn, split plan cc_attn_split: restated in
tests/test_attn_split_plan.py).  The split keeps every summation order, so the attention output and the Q8_0 quantisation of it that
the wo matvec consumes must equal eager mode and the CUDA-graph mode bit for bit.  Compared here, for f32 and f16 caches (whose query
heads map to kv groups differently, h % n_kv and h / (n_heads / n_kv)):
  * shapes with S = 4 (head_dim 128, 32 / 8 heads), S = 2 (head_dim 64, 8 / 2 heads) and S = 1 (head_dim 48, 6 / 6 heads) on the full
    grid, and the S = 4 shape at SM limits 64 (S = 2) and 20 (S = 1, fewer CTAs than heads);
  * KV lengths on each side of AT_SPLIT_MIN_KV = 320 (below it one CTA does each head), lengths not divisible by S, on each side of the
    K chunk (32 / 64 rows) and V chunk (S x 32 / S x 64 rows) edges, up to several refills of the three chunk buffers, and the short
    lengths 0, 1, 2, 3, 4 of the one-CTA path;
  * the ring kernel (wo is a Q8_0 matvec: its input quants come from the attention phase) and the register kernel (attention alone);
  * 120 consecutive decode steps through one replayed graph, from 310 to 429 cached positions: the switch to the split, then 110 phases
    of the monotonic per-head arrival words."""
import numpy as np
import pytest

from oracle import oracle as oc
from crabml_b200.tensor import MEGA_NONE, MEGA_REGISTER, MEGA_RING
from tests.gpu_common import MODE_DEVICE, assert_same_bits, fresh_device
from tests.test_gpu_attention_long import attention, fill

WO_SEED = 0x5A17
MAX_LEN = 1100
# (head_dim, n_heads, n_kv, SM limit)
SHAPES = {"split4": (128, 32, 8, None), "split2": (64, 8, 2, None), "split1": (48, 6, 6, None),
          "split4-grid64": (128, 32, 8, 64), "split4-grid20": (128, 32, 8, 20)}
KV_LENS = [0, 1, 2, 3, 4, 33, 129, 319, 320, 321, 322, 323, 351, 352, 353, 383, 384, 385, 447, 448, 449, 511, 512, 513, 600, 1000]
# execution mode (its device: MODE_DEVICE) -> (wo matvec in the flush, expected mega_variant)
MODES = {"eager": (True, MEGA_NONE), "graph": (True, MEGA_NONE), "ring": (True, MEGA_RING), "register": (False, MEGA_REGISTER)}


def case(hd, n_heads, n_kv, kv_len, step=0):
    rng = np.random.default_rng(7000 + 31 * kv_len + hd + 1000003 * step)
    K = rng.standard_normal((n_kv, kv_len, hd)).astype(np.float32)
    V = rng.standard_normal((n_kv, kv_len, hd)).astype(np.float32)
    q = (2.0 * rng.standard_normal((n_heads, hd))).astype(np.float32)
    k = rng.standard_normal((n_kv, hd)).astype(np.float32)
    v = rng.standard_normal((n_kv, hd)).astype(np.float32)
    return K, V, q, k, v


def wo_weight(dev, dim):
    from crabml_b200 import CudaTensor
    from crabml_b200 import runner as R
    return CudaTensor.synth([dim, dim], oc.Q8_0, dev, WO_SEED, 1, R.synth_scale(oc.Q8_0, dim))


def step(dev, kc, vc, q, k, v, n_heads, n_kv, hd, pos, W):
    """attention, then (W given) the wo matvec on its output, as the Llama layer does -> host copies (out, y or None)"""
    from crabml_b200 import CudaTensor
    out = attention(CudaTensor, dev, kc, vc, q, k, v, n_heads, n_kv, hd, pos=pos)
    y = W.matmul_vec(out.reshape([1, n_heads * hd])) if W is not None else None
    o = out.export()
    return o, (y.export() if y is not None else None)


def run_mode(mode, f16, shape):
    from crabml_b200 import CudaTensor
    hd, n_heads, n_kv, limit = SHAPES[shape]
    with_wo, variant = MODES[mode]
    dt = oc.F16 if f16 else oc.F32
    with fresh_device(**MODE_DEVICE[mode]) as dev:
        if limit:
            dev.set_sm_limit(limit)
        W = wo_weight(dev, n_heads * hd) if with_wo else None
        kc_full, vc_full = CudaTensor.alloc([n_kv, MAX_LEN, hd], dt, dev), CudaTensor.alloc([n_kv, MAX_LEN, hd], dt, dev)
        res = []
        for kv_len in KV_LENS:
            K, V, q, k, v = case(hd, n_heads, n_kv, kv_len)
            kc, vc = fill(CudaTensor, dev, kc_full, vc_full, K, V)
            res.append(step(dev, kc, vc, q, k, v, n_heads, n_kv, hd, kv_len, W))
            if dev.lazy == 2:
                assert dev.mega_variant() == variant, (mode, shape, kv_len, dev.mega_variant())
        return res


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("f16", [False, True], ids=["f32", "f16"])
def test_split_attention_and_wo_quants_equal_eager(shape, f16):
    got = {mode: run_mode(mode, f16, shape) for mode in MODES}
    assert np.isfinite(got["eager"][-1][0]).all() and np.abs(got["eager"][-1][0]).max() > 1e-3
    for mode in ("graph", "ring", "register"):
        for kv_len, (o, y), (o0, y0) in zip(KV_LENS, got[mode], got["eager"]):
            assert_same_bits(o, o0, f"{mode} {shape} f16={f16} kv_len {kv_len}: attention output vs eager")
            if y is not None:
                assert_same_bits(y, y0, f"{mode} {shape} f16={f16} kv_len {kv_len}: wo output vs eager")


@pytest.mark.gpu
@pytest.mark.parametrize("f16", [False, True], ids=["f32", "f16"])
def test_120_replayed_steps_equal_eager(f16):
    """One growing cache, 120 decode steps: lazy mode 2 replays one graph of the ring kernel (S = 4) every step."""
    from crabml_b200 import CudaTensor
    hd, n_heads, n_kv, _ = SHAPES["split4"]
    dt = oc.F16 if f16 else oc.F32
    with fresh_device(lazy=0) as eager, fresh_device(lazy=2) as ring:
        devs = {"eager": eager, "ring": ring}
        st = {}
        for name, dev in devs.items():
            kc_full, vc_full = CudaTensor.alloc([n_kv, 440, hd], dt, dev), CudaTensor.alloc([n_kv, 440, hd], dt, dev)
            K, V, _, _, _ = case(hd, n_heads, n_kv, 310)
            kc, vc = fill(CudaTensor, dev, kc_full, vc_full, K, V)
            st[name] = (kc, vc, wo_weight(dev, n_heads * hd))
        s0 = devs["ring"].lazy_stats()
        for t in range(120):
            _, _, q, k, v = case(hd, n_heads, n_kv, 0, step=t + 1)
            r = {name: step(dev, st[name][0], st[name][1], q, k, v, n_heads, n_kv, hd, 310 + t, st[name][2]) for name, dev in devs.items()}
            assert devs["ring"].mega_variant() == MEGA_RING
            assert_same_bits(r["ring"], r["eager"], f"step {t}: (attention output, wo output) vs eager")
        s1 = devs["ring"].lazy_stats()
        delta = {k: s1[k] - s0[k] for k in ("flushes", "graph_captures", "graph_replays", "uncached")}
        assert delta["graph_replays"] >= 100 and delta["uncached"] == 0, delta
