"""Temperature + top-p sampling on the device (cc_sample_to_slot, ccr_runner_generate_ex) against the sequential restatement of
Llama2Sampler (tests/sampler_ref.py): exact_order picks bit for bit, the fast modes bit for bit against the emulation of their
summation orders and bit-identical to each other, lazy mode 2 with several samplers per flush, end to end on the tinyllamas fixtures,
the runner's contract, and the coin's distribution."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle.llama_replay import GGUFModel, Llama2Runner, load_weights
from oracle.tensor_ref import OracleDevice, OracleTensor
from tests import sampler_ref as S
from crabml_b200.tensor import MEGA_REGISTER, MEGA_RING
from tests.gpu_common import assert_same_bits, fresh_device, run_modes

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NS = [1, 2, 33, 511, 512, 513, 32000, 152064]
TS = [0.1, 0.8, 1.0, 1.7]
TOPPS = [0.0, 0.01, 0.5, 0.9, 1.0, 1.5]
KINDS = ["peaked", "flat", "tied", "neginf", "uniform"]


def _row(kind, n, rng):
    if kind == "peaked":
        x = rng.standard_normal(n).astype(np.float32)
        x[rng.integers(0, n)] += 12.0
    elif kind == "flat":
        x = (3.0 * rng.standard_normal(n)).astype(np.float32)
    elif kind == "tied":
        x = rng.integers(0, 4, n).astype(np.float32)
    elif kind == "neginf":
        x = (2.0 * rng.standard_normal(n)).astype(np.float32)
        x[rng.random(n) < 0.4] = -np.inf
        x[rng.integers(0, n)] = 1.0
    else:                                   # near-uniform: topp < 1/n leaves nothing above the cutoff (n0 == 0)
        x = (1e-3 * rng.standard_normal(n)).astype(np.float32)
    return x


def _sample_many(dev, t, temperature, topp, seed, count):
    for i in range(count):
        t.sample_to_slot(temperature, topp, seed, i, 0, i)
    return dev.read_history(0, count).tolist()


def test_exact_order_picks_equal_the_reference_bit_for_bit():
    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(5)
    with fresh_device(exact_order=True) as dev:
        for n in NS:
            for kind in KINDS:
                x = _row(kind, n, rng)
                t = CudaTensor.new(x, [n], dev)
                seed = int(rng.integers(0, 2**63))
                for T in TS:
                    p = S.probs(x, T)
                    for topp in TOPPS:
                        walk = S.topp_walk(p, topp)
                        want = [S.argmax_last(x) if walk is None else S.pick(walk, S.coin(seed, i)) for i in range(64)]
                        got = _sample_many(dev, t, T, topp, seed, 64)
                        assert got == want, (n, kind, T, topp)
                assert_same_bits(t.export(), x, "the sampler modified the logits")


def test_fast_order_picks_equal_the_emulation_of_its_sums_bit_for_bit():
    """Fast devices sum in the canonical tree / tiled-scan orders.  Their picks equal the bit-exact emulation of those orders
    (tests/sampler_ref.py probs_fast / topp_walk_fast; tests/test_sampler_ref.py bounds that emulation's distance from the sequential
    reference entry by entry); how many picks differ from the sequential reference is reported."""
    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(6)
    diffs, total = 0, 0
    with fresh_device() as dev:
        for n in NS:
            for kind in KINDS:
                x = _row(kind, n, rng)
                t = CudaTensor.new(x, [n], dev)
                seed = int(rng.integers(0, 2**63))
                for T in TS:
                    pf, pr = S.probs_fast(x, T), S.probs(x, T)
                    for topp in TOPPS:
                        wf, wr = S.topp_walk_fast(pf, topp), S.topp_walk(pr, topp)
                        got = _sample_many(dev, t, T, topp, seed, 64)
                        want = [S.argmax_last(x) if wf is None else S.pick(wf, S.coin(seed, i)) for i in range(64)]
                        assert got == want, (n, kind, T, topp)
                        ref = [S.argmax_last(x) if wr is None else S.pick(wr, S.coin(seed, i)) for i in range(64)]
                        diffs += sum(g != r for g, r in zip(got, ref))
                        total += 64
    print(f"fast order: {diffs} of {total} picks differ from the sequential reference")


def test_lazy_megakernel_runs_one_sample_per_token_and_hands_the_rest_to_the_graph():
    """lazy mode 2 records cc_sample_to_slot without flushing.  A flush holding one sampler as its last op runs in the megakernel; a
    flush holding several samplers, or ops queued behind one (tokens submitted ahead: the next embedding lookup reads the slot), must
    still run every op: each history entry equals the eager device's."""
    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(12)
    n = 64
    x = (2.0 * rng.standard_normal(n)).astype(np.float32)
    table = (2.0 * rng.standard_normal((n, n))).astype(np.float32)

    def run(dev):
        t = CudaTensor.new(x, [n], dev)
        tab = CudaTensor.new(table.reshape(-1), [n, n], dev)
        row = CudaTensor.alloc([n], 0, dev)
        t.sample_to_slot(1.0, 0.9, 5, 0, 0, 0)                # a flush with one sampler, the last op
        dev.read_history(0, 1)
        variant = dev.mega_variant()
        for i in range(1, 7):                                   # six samplers before one flush, into slots 1..6
            t.sample_to_slot(0.8, 0.9, 5, i, i, i)
        for i in range(7, 11):                                  # sample -> embedding row from the slot -> sample that row ...
            dev.check(dev.lib.cc_copy_rows_from_slot(dev.handle, C.byref(row._view()), C.byref(tab._view()), 0))
            row.sample_to_slot(1.0, 0.5, 5, i, 0, i)
        return dev.read_history(0, 11).tolist(), variant
    res = run_modes(run, modes=(0, 2))
    eager, (lazy, variant) = res[0][0], res[2]
    assert variant == MEGA_REGISTER                                 # the single-sampler flush ran in the (register) megakernel
    assert lazy == eager
    want = [S.sample_fast(x, 1.0, 0.9, 5, 0)] + [S.sample_fast(x, 0.8, 0.9, 5, i) for i in range(1, 7)]
    prev = want[0]
    for i in range(7, 11):
        prev = S.sample_fast(table[prev], 1.0, 0.5, 5, i)
        want.append(prev)
    assert eager == want


def test_fast_modes_sample_bit_identical_ids_on_ring_and_k_quant_kernels(tmp_path, fixture_path):
    """eager, CUDA graph and megakernel: same ids and logits over 96 tinyllamas steps and 66 steps of a Llama-2-7B-shaped layer in
    Q8_0 (the ring megakernel) and in Q4_K + Q6_K (the register megakernel, mega.cu), each mode in its own process; lazy mode 2
    stays in its persistent kernel while sampling."""
    gguf = fixture_path("tinyllamas-stories-15m-q8_0.gguf")
    got = {}
    for name, lazy in (("eager", 0), ("graph", 1), ("mega", 2)):
        env = dict(os.environ)
        env.pop("CRABML_MEGA_FLAGS", None)
        out = str(tmp_path / f"{name}.npz")
        subprocess.run([sys.executable, os.path.join(ROOT, "tests", "sampling_mode_worker.py"), str(lazy), gguf, out], check=True, cwd=ROOT,
                       env=env, timeout=900)
        got[name] = np.load(out)
    assert int(got["mega"]["l7b_variant"]) == MEGA_RING and int(got["mega"]["tiny_variant"]) in (MEGA_REGISTER, MEGA_RING)
    assert int(got["mega"]["l7bk_variant"]) == MEGA_REGISTER
    for key in ("tiny", "l7b", "l7bk"):
        ref_ids, ref_lg = got["eager"][f"{key}_ids"], got["eager"][f"{key}_logits"]
        assert ref_ids.size >= 64 and len(set(ref_ids.tolist())) > 8, ref_ids
        for name in ("graph", "mega"):
            np.testing.assert_array_equal(got[name][f"{key}_ids"], ref_ids, err_msg=f"{key}: {name} vs eager")
            assert_same_bits(got[name][f"{key}_logits"], ref_lg, f"{key}: {name} vs eager")


@pytest.mark.parametrize("fname", ["tinyllamas-stories-15m-q8_0.gguf", "tinyllamas-stories-15m-q4_0.gguf"])
@pytest.mark.parametrize("temperature,topp", [(0.8, 0.9), (1.0, 1.0)])
def test_exact_order_generation_equals_the_oracle_replay(fixture_path, fname, temperature, topp):
    """exact_order generate_ex = the oracle's forward + the reference sampler, token for token; the exported logits are the ones the
    greedy path computes for the same ids (sampling leaves them untouched)."""
    from crabml_b200 import runner as R
    path = fixture_path(fname)
    prompt, steps, seed = [1, 365, 1424], 24, 31337
    with fresh_device(exact_order=True) as dev:
        conf, w, _ = R.load_gguf(path, dev)
        r = R.LlamaRunner(dev, conf, w, 64)
        ids, logits = r.generate_logits(prompt, steps, temperature, topp, seed)
        r.close()
        r = R.LlamaRunner(dev, conf, w, 64)
        seq = prompt + ids
        for pos, tok in enumerate(seq[:-1]):
            lg = r.forward([tok], pos).copy()
            if pos >= len(prompt) - 1:
                assert_same_bits(lg, logits[pos - len(prompt) + 1], f"pos {pos}")
        r.close()
    gm = GGUFModel(path)
    odev = OracleDevice()
    ro = Llama2Runner(OracleTensor, gm.conf, load_weights(gm, OracleTensor, odev), odev, 64)
    want, tok, pos = [], None, 0
    for tok in prompt:
        lg = ro.forward([tok], pos)
        pos += 1
    for i in range(steps):
        nxt = S.sample(np.array(lg, np.float32), temperature, topp, seed, i)
        want.append(nxt)
        if i + 1 < steps:
            lg = ro.forward([nxt], pos)
            pos += 1
    assert ids == want


def test_runner_contract(fixture_path):
    from crabml_b200 import runner as R
    from crabml_b200.capi import TensorError
    path = fixture_path("tinyllamas-stories-15m-q8_0.gguf")
    with fresh_device(lazy=2) as dev:
        conf, w, _ = R.load_gguf(path, dev)

        def fresh():
            return R.LlamaRunner(dev, conf, w, 96)
        r = fresh(); g_ids, g_lg = r.generate_greedy_logits([1, 365], 40); r.close()
        r = fresh(); z_ids, z_lg = r.generate_logits([1, 365], 40, 0.0, 0.9, 5); r.close()
        assert z_ids == g_ids
        assert_same_bits(z_lg, g_lg, "temperature 0 vs greedy")
        r = fresh(); a = r.generate([1, 365], 40, 1.0, 0.9, 2024); r.close()
        r = fresh(); b = r.generate([1, 365], 40, 1.0, 0.9, 2024); r.close()
        r = fresh(); c = r.generate([1, 365], 40, 1.0, 0.9, 2025); r.close()
        assert a == b and a != c
        k = next(i for i in range(1, len(a)) if a[i] not in a[1:i])
        r = fresh(); e = r.generate([1, 365], 40, 1.0, 0.9, 2024, eos=a[k]); r.close()
        assert e == a[:k]                  # stops before yielding EOS, like the greedy loop (llama2.rs:160-163)
        r = fresh()
        for T, p in ((float("nan"), 0.9), (-1.0, 0.9), (1.0, float("nan"))):
            with pytest.raises(TensorError):
                r.generate([1], 4, T, p, 1)
        assert r.kv_cache_len() == 0      # rejected before the prompt ran
        r.close()


def test_sample_to_slot_argument_errors():
    from crabml_b200 import CudaTensor
    from crabml_b200.capi import TensorError
    with fresh_device() as dev:
        x = CudaTensor.new(np.arange(64, dtype=np.float32), [8, 8], dev)
        v = CudaTensor.new(np.arange(64, dtype=np.float32), [64], dev)
        v.sample_to_slot(1.0, 0.9, 1, 0)
        for bad in (lambda: v.sample_to_slot(float("nan"), 0.9, 1, 0), lambda: v.sample_to_slot(-0.5, 0.9, 1, 0),
                    lambda: v.sample_to_slot(1.0, float("nan"), 1, 0), lambda: x.transpose([1, 0]).sample_to_slot(1.0, 0.9, 1, 0),
                    lambda: v.sample_to_slot(1.0, 0.9, 1, 0, slot=16), lambda: v.sample_to_slot(1.0, 0.9, 1, 0, slot=-1),
                    lambda: v.sample_to_slot(1.0, 0.9, 1, 0, hist_index=65536)):
            with pytest.raises(TensorError):
                bad()
        h = CudaTensor.alloc([64], 1, dev)          # f16
        with pytest.raises(TensorError):
            h.sample_to_slot(1.0, 0.9, 1, 0)
        # NaN logits are outside the contract: the kernel still ends and writes an index in range
        nanrow = np.full(64, np.nan, np.float32); nanrow[3] = 1.0
        CudaTensor.new(nanrow, [64], dev).sample_to_slot(1.0, 0.9, 1, 0, 0, 0)
        CudaTensor.new(np.full(64, np.nan, np.float32), [64], dev).sample_to_slot(1.0, 0.9, 1, 1, 0, 1)
        assert all(0 <= i < 64 for i in dev.read_history(0, 2))


def test_coin_distribution_fits_the_reference_tail_distribution():
    """20 000 coin indices on one 64-token row (T = 1, p = 0.9): the empirical frequencies fit the reference's (ascending, tail)
    distribution -- q_j = (C_j - C_{j-1}) / C_last over the walked positions -- by chi-square."""
    from scipy.stats import chisquare

    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(9)
    x = (1.5 * rng.standard_normal(64)).astype(np.float32)
    with fresh_device() as dev:
        got = np.array(_sample_many(dev, CudaTensor.new(x, [64], dev), 1.0, 0.9, 424242, 20000))
    order, Cs, last = S.topp_walk(S.probs(x, 1.0), 0.9)
    q = np.diff(np.concatenate([[0.0], Cs[:last + 1].astype(np.float64)])) / float(Cs[last])
    ids = order[:last + 1]
    assert set(got.tolist()) <= set(ids.tolist())
    obs = np.array([(got == i).sum() for i in ids], np.float64)
    exp = q * got.size
    big = exp >= 5                                          # merge the sparse bins
    obs_m, exp_m = np.append(obs[big], obs[~big].sum()), np.append(exp[big], exp[~big].sum())
    if exp_m[-1] == 0:
        obs_m, exp_m = obs_m[:-1], exp_m[:-1]
    stat, pval = chisquare(obs_m, exp_m * obs_m.sum() / exp_m.sum())
    print(f"chi-square over {len(obs_m)} bins: {stat:.1f}, p = {pval:.3f}")
    assert pval > 1e-3
