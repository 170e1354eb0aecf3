"""Lazy modes 1 and 2 replay a cached CUDA graph whenever a flush's plan signature repeats (lazy.cu).  A graph bakes in every pointer,
type and launch dimension it was captured with, so a replay is right only if each of them is in the signature, or the cache is dropped
when it changes.  The other lazy-mode tests repeat one flush on the same buffers and change only the input values; here, between a
capture and a later flush of the same plan, what a graph bakes in changes:

  * the eager activation scratch (dev->act_scratch, read by the matvec steps a graph runs as eager kernels) is regrown by a batched
    matvec -- a prompt after decoding has started;
  * an f16 buffer takes the pooled address an f32 buffer of the same size class had (CONTIGUOUS, row copies);
  * the persistent grid changes (cc_device_set_sm_limit);
  * more plans than the cache holds (LZ_MAX_GRAPHS), so the least recently used graphs are evicted.

Every case runs one call sequence on a fresh device in eager mode and in lazy modes 1 and 2.  Each output is bit-identical to eager, the
inputs change every round, and the lazy_stats() deltas of every flush pin whether it captured, replayed or ran uncached."""
import numpy as np
import pytest

from oracle import oracle as oc
from crabml_b200.runner import synth_scale
from crabml_b200.tensor import MEGA_REGISTER, MEGA_RING
from tests.gpu_common import assert_same_bits, full_grid, run_modes

pytestmark = pytest.mark.gpu

WSEED = 0x9A7
INITIAL_SCRATCH = 4 << 20          # dev->act_scratch as cc_device_create sizes it (device.cu)
LZ_MAX_GRAPHS = 64                 # cached graphs per device (lazy.cu)
CAPTURE, REPLAY, UNCACHED = (1, 0, 0), (0, 1, 0), (0, 0, 1)


class _Run:
    """One call sequence on one device: the outputs of every step and, in the lazy modes, each step's lazy_stats() deltas."""

    def __init__(self, dev):
        self.lazy, self.dev, self.outs, self.delta = dev.lazy, dev, [], None

    def step(self, what, fn, want=None):
        """fn() -> None, an array or a tuple of arrays (host copies, read after the step's flush).  want: (captures, replays, uncached)
        of the step in both lazy modes; the deltas are kept in self.delta either way."""
        s0 = self.dev.lazy_stats() if self.lazy else None
        out = fn()
        for i, o in enumerate(out if isinstance(out, tuple) else () if out is None else (out,)):
            self.outs.append((f"{what}[{i}]", np.array(o, copy=True)))
        if self.lazy:
            s1 = self.dev.lazy_stats()
            self.delta = tuple(s1[k] - s0[k] for k in ("graph_captures", "graph_replays", "uncached"))
            if want is not None:
                assert self.delta == want, (what, f"lazy={self.lazy}", "(captures, replays, uncached)", self.delta, "want", want)
        return out


def _assert_modes(scenario):
    """the scenario on a fresh device in eager mode and lazy modes 1 and 2 (which check their own deltas): every output bit-identical
    to eager -> eager's [(step, output)]"""
    def body(dev):
        run = _Run(dev)
        scenario(run)
        return run.outs
    res = run_modes(body)
    for mode in (1, 2):
        assert [w for w, _ in res[mode]] == [w for w, _ in res[0]], mode
        for (what, g), (_, r) in zip(res[mode], res[0]):
            assert_same_bits(g, r, f"lazy={mode} vs eager: {what}")
    return res[0]


def _weight(dev, m, k, t, tid):
    from crabml_b200 import CudaTensor
    return CudaTensor.synth([m, k], t, dev, WSEED, tid, synth_scale(t, k))


def _table(dev, rows, k, seed, scale=1.0):
    """a non-pooled f32 [rows, k] table of inputs; a row copy out of it takes its row index from the flush's dynamic block, so one graph
    serves every round while the values change"""
    from crabml_b200 import CudaTensor
    v = (scale * np.random.default_rng(seed).standard_normal((rows, k))).astype(np.float32)
    return CudaTensor.from_cpu(v, [rows, k], oc.F32, dev), v


def _row(dev, table, r, k):
    from crabml_b200 import CudaTensor
    x = CudaTensor.alloc([k], oc.F32, dev)
    x.copy_rows_from(table, [r])
    return x


def _act_bytes_lower_bound(wt, n):
    """bytes of n activations quantised to the weight's partner type, in GGUF blocks -- the device layout is at least this large"""
    at = oc.rhs_type(wt)
    return n // oc.block_elems(at) * oc.block_bytes(at)


# ---- 1. the eager activation scratch regrows under cached graphs ------------------------------------------------------------------
DECODE_K4 = (64, 4096, oc.Q4_K)        # a K-quant matvec: an eager step in mode 1 (quantise into dev->act_scratch + warp-per-row kernel)
DECODE_K8 = (64, 32800, oc.Q8_0)       # a Q8_0 row past the streaming limit (32768): an eager step in both lazy modes
# one batched matvec whose quantised activations outgrow the initial scratch: Q4_K (Q8_K activations, the prefill GEMM quantises into
# the scratch) and Q8_0 (the prefill GEMM quantises itself; size_scratch still grows the scratch for it).  32 rows: the [1024, 32]
# output (128 KiB) lands in a pool size class no decode buffer uses, so the decode flushes get their buffers back at the same addresses.
GROWERS = {"q4_k": (32, 4096, 1024, oc.Q4_K), "q8_0": (32, 4096, 1024, oc.Q8_0)}


@pytest.mark.parametrize("grower", list(GROWERS))
def test_scratch_regrowth_between_replays(grower):
    """Decode flushes of a Q4_K and of a past-the-limit Q8_0 matvec are captured and replayed; a batched matvec then regrows the
    activation scratch; the first decode flush of each plan afterwards must re-capture (its cached graph quantised into the freed
    scratch), and every output equals eager."""
    from crabml_b200 import CudaTensor
    gm, gk, gb, gt = GROWERS[grower]
    assert _act_bytes_lower_bound(gt, gb * gk) > INITIAL_SCRATCH
    assert all(_act_bytes_lower_bound(t, k) < INITIAL_SCRATCH for _, k, t in (DECODE_K4, DECODE_K8))

    def scenario(run):
        dev = run.dev
        probes = []
        for i, (m, k, t) in enumerate((DECODE_K4, DECODE_K8)):
            table, _ = _table(dev, 4, k, [k, 1])
            probes.append((_weight(dev, m, k, t, 1 + i), table, k))

        def decode(p, r):
            w, table, k = probes[p]
            return lambda: w.matmul_vec(_row(dev, table, r, k)).export()
        for r, want in ((0, CAPTURE), (1, REPLAY)):
            for p in range(2):
                run.step(f"decode{p}-r{r}", decode(p, r), want)
        xs = np.random.default_rng([gk, 2]).standard_normal((gb, gk)).astype(np.float32)
        x = CudaTensor.from_cpu(xs, [gb, gk], oc.F32, dev)
        run.step("batched", lambda: _weight(dev, gm, gk, gt, 3).matmul_vec(x).export(), UNCACHED)
        del x
        for r, want in ((2, CAPTURE), (3, REPLAY)):
            for p in range(2):
                run.step(f"decode{p}-r{r}", decode(p, r), want)
    ref = dict(_assert_modes(scenario))
    assert all(np.isfinite(v).all() and np.abs(v).max() > 1e-3 for v in ref.values())


L7B_LONG = (32, 32, 1, 4096, 11008, 512, 32000, 1e-5, 128)       # one Llama-2-7B layer, a context long enough for the 400-token prompt
PROMPT_A = [1, 365, 2354, 931]
PROMPT_B = [1] + [int(t) for t in np.random.default_rng(400).integers(2, 32000, 399)]


def test_second_prompt_regrows_scratch_under_decode_graphs():
    """A Q4_K (Q6_K classifier) model decodes prompt A; a new runner on the same device forwards the 400-token prompt B in one batch --
    ffn_down's Q8_K activations (k = 11008) outgrow the scratch the decode graphs were captured with -- and decodes greedily from it.
    Ids and logits equal eager; the batch is one uncached flush; B's decode captures its two plans (prompt-token and slot-token step)
    afresh instead of replaying A's; mode 2 keeps the mega_kernel."""
    from crabml_b200 import runner as R
    conf = R.LlamaConfig(*L7B_LONG)
    assert _act_bytes_lower_bound(oc.Q4_K, len(PROMPT_B) * conf.hidden_dim) > INITIAL_SCRATCH

    def scenario(run):
        dev = run.dev
        w = R.synthetic_weights(dev, conf, oc.Q4_K, oc.Q6_K, seed=0xF5)
        r = R.LlamaRunner(dev, conf, w, conf.seq_len)
        run.step("A", lambda: r.generate_greedy_logits(PROMPT_A, 6))
        if run.lazy:
            assert run.delta[2] == 0 and run.delta[0] >= 2, run.delta
        if run.lazy == 2:
            assert dev.mega_variant() == MEGA_REGISTER
        r.close()
        r = R.LlamaRunner(dev, conf, w, conf.seq_len)
        lg = run.step("B-prompt", lambda: r.forward(PROMPT_B, 0), UNCACHED)
        nxt = len(lg) - 1 - int(np.argmax(lg[::-1]))        # the sampler's argmax: the last maximum
        run.step("B-decode", lambda: r.generate_greedy_logits([nxt], 6), (2, 4, 0))
        if run.lazy == 2:
            assert dev.mega_variant() == MEGA_REGISTER
        r.close()
    ref = dict(_assert_modes(scenario))
    assert np.isfinite(ref["B-decode[1]"]).all() and len(ref["B-decode[0]"]) == 6


# ---- 2. an f16 buffer at the address of an f32 one ---------------------------------------------------------------------------------
def test_type_change_at_one_pooled_address():
    """Each round, on [8, 8] tensors of one type (each op flushed alone): fill t from a row of an f32 table, CONTIGUOUS of t transposed,
    read that back through a row copy into f32, and copy two rows of t into f32.  Every buffer is in the pool's smallest size class, so
    an f16 round gets the f32 rounds' addresses -- and its CONTIGUOUS and row copies the f32 plans' signatures, but for the types.  f32
    rounds 1-3 (the third replays every plan: the pool hands back the same addresses), an f16 round that must capture, an f32 round
    that replays its own graphs again; the values are the table's, through f16 in the f16 round."""
    from crabml_b200 import CudaTensor
    rounds = [(oc.F32, CAPTURE), (oc.F32, None), (oc.F32, REPLAY), (oc.F16, CAPTURE), (oc.F32, REPLAY)]

    def scenario(run):
        dev = run.dev
        table, tv = _table(dev, len(rounds), 64, 8, 3.0)
        for rnd, (dt, want) in enumerate(rounds):
            tag = f"r{rnd}-{oc.TYPE_NAMES[dt]}"
            t = CudaTensor.alloc([8, 8], dt, dev)
            hold = {}

            def fill():
                t.reshape([64]).copy_rows_from(table, [rnd])
                dev.flush()

            def contiguous():
                hold["c"] = t.transpose([1, 0]).contiguous()
                dev.flush()

            def read_back():
                hold["o"] = CudaTensor.alloc([64], oc.F32, dev)
                hold["o"].copy_rows_from(hold["c"].reshape([1, 64]), [0])
                dev.flush()
                return hold["o"].export()

            rows = [rnd % 8, (rnd + 5) % 8]

            def table_rows():
                hold["o2"] = CudaTensor.alloc([2, 8], oc.F32, dev)
                hold["o2"].copy_rows_from(t, rows)
                dev.flush()
                return hold["o2"].export()
            run.step(f"{tag}-fill", fill, want)
            run.step(f"{tag}-contiguous", contiguous, want)
            got_t = run.step(f"{tag}-read-back", read_back, want)
            got_rows = run.step(f"{tag}-table-rows", table_rows, want)
            v = tv[rnd] if dt == oc.F32 else tv[rnd].astype(np.float16).astype(np.float32)
            np.testing.assert_array_equal(got_t, v.reshape(8, 8).T.reshape(-1), err_msg=f"{tag} lazy={run.lazy}: contiguous")
            np.testing.assert_array_equal(got_rows, v.reshape(8, 8)[rows].reshape(-1), err_msg=f"{tag} lazy={run.lazy}: row copy")
            del t, hold                      # every buffer of the round back to the pool before the next one
    _assert_modes(scenario)


# ---- 3. the persistent grid changes after a capture --------------------------------------------------------------------------------
L7B = (32, 32, 1, 4096, 11008, 64, 32000, 1e-5, 128)
SM_CASES = {"q8_0-ring": (oc.Q8_0, oc.Q8_0, MEGA_RING), "q4_k-mega": (oc.Q4_K, oc.Q6_K, MEGA_REGISTER)}


@pytest.mark.parametrize("case", list(SM_CASES))
def test_sm_limit_after_capture(case):
    """One-layer 7B-shaped token flushes (the ring kernel for Q8_0, the mega_kernel for Q4_K) captured at the full grid, then at sm
    limits 5 and 1 and the full grid again: the first flush after each change re-captures, the next replays, and the logits do not
    change bits (the kernels do not depend on the grid).  The grid barrier's arrival counter advances by the grid size per barrier, so
    the change restarts it: a kernel at a smaller grid would otherwise pass barriers it should wait at, one at a larger grid wait for
    ever (until its bounded spin reports a barrier timeout)."""
    from crabml_b200 import runner as R
    wt, ct, variant = SM_CASES[case]
    tokens = [1] + [int(t) for t in np.random.default_rng(5).integers(2, 32000, 8)]

    def scenario(run):
        dev = run.dev
        conf = R.LlamaConfig(*L7B)
        r = R.LlamaRunner(dev, conf, R.synthetic_weights(dev, conf, wt, ct, seed=0xF5), 16)
        pos = [0]

        def token():
            p = pos[0]
            pos[0] += 1
            return r.forward([tokens[p]], p)
        run.step("warm0", token)
        run.step("warm1", token)                  # the pool's first allocations settle into lowest-address order
        run.step("full", token, REPLAY)
        for n in (5, 1, full_grid()):
            dev.set_sm_limit(n)
            run.step(f"sm{n}-first", token, CAPTURE)
            run.step(f"sm{n}-again", token, REPLAY)
            if run.lazy == 2:
                assert dev.mega_variant() == variant, (n, dev.mega_variant())
        r.close()
    ref = _assert_modes(scenario)
    assert all(np.isfinite(v).all() for _, v in ref)


# ---- 4. more plans than the cache holds ------------------------------------------------------------------------------------------
N_PLANS = 70


def _lru_sequence():
    """(plan, expected) flush by flush, with LZ_MAX_GRAPHS = 64: every plan once (the first 6 are evicted), the newest 64 again (all
    replays); then 0 re-captures (evicting 6, the least recently used); 7 is touched just before 1 re-captures, so 8 is evicted and 7
    survives; 8 and 6 re-capture (evicting 9 and 10), 0 and 1 replay, 9 re-captures."""
    assert LZ_MAX_GRAPHS == 64 and N_PLANS == 70
    seq = [(i, CAPTURE) for i in range(N_PLANS)] + [(i, REPLAY) for i in range(N_PLANS - LZ_MAX_GRAPHS, N_PLANS)]
    seq += [(0, CAPTURE), (7, REPLAY), (1, CAPTURE), (7, REPLAY), (8, CAPTURE), (6, CAPTURE), (0, REPLAY), (1, REPLAY), (9, CAPTURE)]
    return seq


def test_lru_bound_of_the_graph_cache():
    """70 single-matvec plans (a row copy + one small Q8_0 matvec each, distinct weights) through the 64-graph cache: exact capture /
    replay of every flush per _lru_sequence, and every output equals eager.  Mode 2 runs each plan in the ring kernel, whose phase
    table an eviction frees."""
    seq = _lru_sequence()
    m, k = 32, 256

    def scenario(run):
        dev = run.dev
        ws = [_weight(dev, m, k, oc.Q8_0, 1 + i) for i in range(N_PLANS)]
        table, _ = _table(dev, len(seq), k, 70)
        for n, (p, want) in enumerate(seq):
            run.step(f"{n}:plan{p}", lambda: ws[p].matmul_vec(_row(dev, table, n, k)).export(), want)
        if run.lazy == 2:
            assert dev.mega_variant() == MEGA_RING
    _assert_modes(scenario)
