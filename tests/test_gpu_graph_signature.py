"""Lazy modes 1 and 2 replay a cached CUDA graph only for a flush with the same plan signature (lazy.cu).  A fused step's signature
words are its whole phase descriptor, so everything the step's graph bakes in is covered.  The other lazy-mode tests keep every
setting of a flush fixed; here one thing a graph bakes in changes while every other pointer stays where it was:

  * a Q8_0 matrix is released and synthesised again with more rows at the same address: a row copy out of it reads the f16 scales,
    whose plane starts after rows x k quant bytes, so the copy's graph is stale;
  * two flushes at identical buffers differ in one recorded setting: llama vs Neox RoPE pairs in the fused attention, and the eps of
    the rms_norm fused into a matvec's prologue.

Every case runs one call sequence on a fresh device in eager mode and in lazy modes 1 and 2.  Each output is bit-identical to eager, and
the lazy_stats() deltas of the flushes pin whether each captured or replayed (None: a round in which the pool's first allocations
settle into lowest-address order)."""
import numpy as np
import pytest

from oracle import oracle as oc
from crabml_b200.capi import ROPE_LLAMA, ROPE_NEOX
from crabml_b200.runner import synth_scale
from tests.test_gpu_graph_replay import CAPTURE, REPLAY, _assert_modes, _row, _table

pytestmark = pytest.mark.gpu

WSEED = 0x51C


# ---- 1. a matrix re-created at its old address with more rows -------------------------------------------------------------------
K = 4096
R, R2 = 256, 384                       # 1.1 and 1.6 MB: both below 2 MB, so the allocator may hand out the old base again
COPIED = [3, R - 1]                    # rows that both matrices have


def test_recreated_matrix_with_more_rows():
    """A flush that only copies two rows out of a [R, K] Q8_0 matrix, captured and replayed; the matrix is released and a [R2, K] one
    synthesised, which the allocator may place at the same base address; the same flush must re-capture, and the rows equal eager.
    The planes start at 256-byte boundaries (cc_assign_planes): the scales of R rows start at R x K bytes, those of R2 rows further
    on, and the whole old scale plane lies inside the new matrix, so a stale graph would read quant bytes as scales without a fault."""
    from crabml_b200 import CudaTensor
    d_row = (K // 32 + 7) // 8 * 8 * 2                       # bytes of one row of f16 scales, padded to 8 blocks (CC_D_STRIDE)
    assert R * K % 256 == 0 and R2 * K != R * K               # the scale plane moves ...
    assert R * K + R * d_row <= R2 * K                        # ... and the old one lies inside the new quant plane

    def scenario(run):
        dev = run.dev
        rounds = [(R, 1, None), (R, 1, REPLAY), (R2, 2, CAPTURE), (R2, 2, REPLAY)]
        w = None
        for n, (rows, tid, want) in enumerate(rounds):
            if w is None or rows != w.shape()[0]:
                w = None                                      # release the old matrix before the new one is allocated
                w = CudaTensor.synth([rows, K], oc.Q8_0, dev, WSEED, tid, synth_scale(oc.Q8_0, K))

            def copy():
                out = CudaTensor.alloc([len(COPIED), K], oc.F32, dev)
                out.copy_rows_from(w, COPIED)
                return out.export()
            run.step(f"{n}:rows{rows}", copy, want)
    ref = dict(_assert_modes(scenario))
    assert not np.array_equal(ref[f"1:rows{R}[0]"], ref[f"2:rows{R2}[0]"])      # the two matrices differ in the copied rows


# ---- 2. one recorded setting changed at identical buffers --------------------------------------------------------------------------
EPS = (1e-5, 1e-6)


def test_norm_eps_at_identical_buffers():
    """rms_norm with eps 1e-5 or 1e-6, the weight mul and a Q8_0 matvec (fused into one normalise-quantise + streaming matvec step),
    on a row copied from a table: every buffer is the same in every round.  The rows are small (mean square 1e-6), so eps changes the
    result; the first flush with the other eps must capture, then each eps replays its own graph."""
    from crabml_b200 import CudaTensor
    rounds = [(0, None), (0, REPLAY), (1, CAPTURE), (1, REPLAY), (0, REPLAY)]

    def scenario(run):
        dev = run.dev
        table, _ = _table(dev, len(rounds), K, 11, 1e-3)
        nw, _ = _table(dev, 1, K, 12)
        w = CudaTensor.synth([64, K], oc.Q8_0, dev, WSEED, 3, synth_scale(oc.Q8_0, K))
        for n, (e, want) in enumerate(rounds):
            def step():
                x = _row(dev, table, n, K)
                x.rms_norm_inplace(EPS[e])
                x.mul_inplace(nw.reshape([K]))
                return w.matmul_vec(x).export()
            run.step(f"{n}:eps{EPS[e]}", step, want)
    ref = _assert_modes(scenario)
    assert all(np.isfinite(v).all() and np.abs(v).max() > 0 for _, v in ref)


NH, HD, KV, MAX_LEN = 4, 64, 9, 16


def _attention(dev, table, n, kc, vc, mode):
    """one decode step's attention in the reference's op order (tests/test_gpu_attention_long.py attention) on q, k, v rows copied
    from a table, at position KV -> the exported [NH, 1, HD] output"""
    qt, kt, vt = (_row(dev, table, 3 * n + j, NH * HD).reshape([1, NH, HD]) for j in range(3))
    qt = qt.rope_inplace(mode, KV, HD)
    kt = kt.rope_inplace(mode, KV, HD)
    kc.concatenate(kt.transpose([1, 0, 2]), 1)
    vc.concatenate(vt.transpose([1, 0, 2]), 1)
    qt = qt.transpose([1, 0, 2]).contiguous().scale_inplace(1.0 / np.sqrt(np.float32(HD)))
    att = qt.batch_matmul(kc.transpose([0, 2, 1])).softmax_inplace(2)
    out = att.batch_matmul(vc)
    del qt, kt, vt, att               # the fuser only folds intermediates nobody else can observe
    return out.export()


def test_rope_mode_at_identical_buffers():
    """The fused attention with llama or Neox RoPE pairs, on q, k, v rows copied from a table into the same buffers and appended at
    the same cache position every round: the first Neox flush must capture, then each mode replays its own graph."""
    from crabml_b200 import CudaTensor
    from tests.test_gpu_attention_long import fill
    rounds = [(ROPE_LLAMA, None), (ROPE_LLAMA, None), (ROPE_LLAMA, REPLAY), (ROPE_NEOX, CAPTURE), (ROPE_NEOX, REPLAY),
              (ROPE_LLAMA, REPLAY)]

    def scenario(run):
        dev = run.dev
        rng = np.random.default_rng(13)
        kc_full, vc_full = CudaTensor.alloc([NH, MAX_LEN, HD], oc.F32, dev), CudaTensor.alloc([NH, MAX_LEN, HD], oc.F32, dev)
        fill(CudaTensor, dev, kc_full, vc_full, *rng.standard_normal((2, NH, KV, HD)).astype(np.float32))
        table, _ = _table(dev, 3 * len(rounds), NH * HD, 14)
        for n, (mode, want) in enumerate(rounds):
            def step():
                return _attention(dev, table, n, kc_full.resize(1, KV), vc_full.resize(1, KV), mode)
            run.step(f"{n}:rope{mode}", step, want)
    ref = _assert_modes(scenario)
    assert all(np.isfinite(v).all() for _, v in ref)
