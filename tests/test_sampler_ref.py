"""Known answers for the sampler reference (tests/sampler_ref.py), worked by hand from crabml-llama2/src/sampler.rs:27-129, its
agreement with a literal transcription of that file, and the distance of the fast devices' summation orders from it.  CPU only."""
import numpy as np
import pytest

from oracle import oracle as oc
from tests import sampler_ref as S

f32 = np.float32


def walk_pick(p, topp, c):
    w = S.topp_walk(np.array(p, np.float32), topp)
    return None if w is None else S.pick(w, c)


def test_topp_keeps_the_low_probability_tail_in_ascending_order():
    # p = [0.5, 0.3, 0.2], topp 0.5: cutoff 0.25 keeps (0.5, 0) and (0.3, 1); ascending: (0.3, 1), (0.5, 0); C = [0.3, 0.8];
    # C > 0.5 first at 1, so cumulative = 0.8 and r = coin * 0.8 (quirk B21: the most likely token is reached only for r >= 0.3)
    order, C, last = S.topp_walk(np.array([0.5, 0.3, 0.2], np.float32), 0.5)
    assert list(order) == [1, 0] and last == 1 and C[1] == f32(0.3) + f32(0.5)
    assert walk_pick([0.5, 0.3, 0.2], 0.5, 0.1) == 1          # r = 0.08 < 0.3
    assert walk_pick([0.5, 0.3, 0.2], 0.5, 0.5) == 0          # r = 0.4
    # CLI default p = 0.9 on a peaked row: the tail (0.0625, 0.0625, 0.125) holds only 0.25, so the walk runs into the peak at last = 3
    order, C, last = S.topp_walk(np.array([0.0625, 0.75, 0.125, 0.0625], np.float32), 0.9)
    assert list(order) == [0, 3, 2, 1] and last == 3


def test_ties_keep_index_order():
    # p = [0.375, 0.125, 0.125, 0.375] exact in f32, topp 0.5: cutoff 0.5 / 3 keeps 0 and 3; the tie (0.375, 0), (0.375, 3) stays in
    # index order; C = [0.375, 0.75], last = 1, r = coin * 0.75
    order, C, last = S.topp_walk(np.array([0.375, 0.125, 0.125, 0.375], np.float32), 0.5)
    assert list(order) == [0, 3] and last == 1
    assert walk_pick([0.375, 0.125, 0.125, 0.375], 0.5, 0.4) == 0     # r = 0.3 < 0.375
    assert walk_pick([0.375, 0.125, 0.125, 0.375], 0.5, 0.6) == 3     # r = 0.45
    # four equal entries, topp 1: all kept in index order, C = [0.25, 0.5, 0.75, 1]
    assert [walk_pick([0.25] * 4, 1.0, c) for c in (0.0, 0.3, 0.6, 0.99)] == [0, 1, 2, 3]


def test_cumulative_break_at_the_first_entry_above_topp():
    # p = [0.125, 0.5, 0.375], topp 0.5: cutoff 0.25 keeps (0.5, 1), (0.375, 2); ascending (0.375, 2), (0.5, 1); C = [0.375, 0.875]
    order, C, last = S.topp_walk(np.array([0.125, 0.5, 0.375], np.float32), 0.5)
    assert list(order) == [2, 1] and last == 1 and C[last] == f32(0.875)
    assert walk_pick([0.125, 0.5, 0.375], 0.5, 0.4) == 2          # r = 0.35
    assert walk_pick([0.125, 0.5, 0.375], 0.5, 0.5) == 1          # r = 0.4375
    # topp 0.3: C[0] = 0.375 > 0.3 already, the walk stops at 0 and only index 2 can be returned
    assert S.topp_walk(np.array([0.125, 0.5, 0.375], np.float32), 0.3)[2] == 0
    assert {walk_pick([0.125, 0.5, 0.375], 0.3, c) for c in (0.0, 0.5, 0.99)} == {2}


def test_rounding_fallbacks():
    # no prefix exceeds topp (topp 1, the sum is exactly 1): last_idx = n0 - 1 and cumulative is the whole sum
    order, C, last = S.topp_walk(np.array([0.125, 0.5, 0.375], np.float32), 1.0)
    assert list(order) == [0, 2, 1] and last == 2 and C[2] == f32(1.0)
    assert [walk_pick([0.125, 0.5, 0.375], 1.0, c) for c in (0.1, 0.3, 0.6)] == [0, 2, 1]
    # no cdf exceeds r: prob_index[last_idx].1 is returned.  r = coin * C[last] < C[last] for every coin < 1 of a normal C, so the
    # walk is driven here with coin 1.0 (the same statement the reference reaches through rounding)
    assert walk_pick([0.125, 0.5, 0.375], 0.5, 1.0) == 1
    assert walk_pick([0.125, 0.5, 0.375], 1.0, 1.0) == 1


def test_topp_at_or_below_zero_and_at_or_above_one():
    p = [0.125, 0.5, 0.375]
    # topp 0: cutoff (1 - 0) / 2 = 0.5 keeps index 1 only, C = [0.5] > 0
    assert {walk_pick(p, 0.0, c) for c in (0.0, 0.7)} == {1}
    # topp -0.5: cutoff 0.75, nothing kept -> n0 == 0 (the reference panics)
    assert S.topp_walk(np.array(p, np.float32), -0.5) is None
    # topp 1.5: cutoff -0.25 keeps everything, nothing exceeds 1.5: the same draw as topp 1 (sample_multi's result is discarded, B19)
    assert [walk_pick(p, 1.5, c) for c in (0.1, 0.3, 0.6)] == [0, 2, 1]


def test_n0_zero_returns_the_argmax_of_the_logits():
    # a uniform row with topp < 1/n: cutoff 0.999 / 99 > 0.01 = every p
    x = np.zeros(100, np.float32)
    assert S.topp_walk(S.probs(x, 1.0), 0.001) is None
    assert S.sample(x, 1.0, 0.001, 1, 0) == 99                 # the LAST maximum
    with pytest.raises(ValueError):
        S.sample_literal(x, 1.0, 0.001, 0.5)
    x[17] = 0.5
    assert S.sample(x, 0.7, -1.0, 3, 4) == 17


@pytest.mark.parametrize("topp", [0.0, 0.5, 0.9, 1.0, 1.5])
def test_n_equals_one(topp):
    # p = [1]; cutoff (1 - topp) / 0 is +inf (topp < 1), NaN (topp 1) or -inf (topp > 1): only topp > 1 keeps the entry
    x = np.array([3.0], np.float32)
    assert (S.topp_walk(S.probs(x, 1.0), topp) is None) == (topp <= 1.0)
    assert S.sample(x, 1.0, topp, 9, 0) == 0


def test_temperature_zero_is_the_last_maximum():
    x = np.array([1.0, 5.0, 2.0, 5.0, -1.0], np.float32)
    assert S.sample(x, 0.0, 0.9, 1, 0) == 3


def test_coin():
    assert S.splitmix64(0) == 0xE220A8397B1DCDAF                     # the generator's first output from state 0
    pinned = {(0, 0): 10946269, (42, 0): 5086015, (42, 1): 8303539, (2**64 - 1, 7): 11118955, (0x5EED, 123456): 2005025}
    for (seed, i), bits in pinned.items():
        assert S.coin(seed, i) == f32(bits * 2.0 ** -24)
    assert f32((2**24 - 1) * 2.0 ** -24) < f32(1.0)
    cs = np.array([S.coin(7, i) for i in range(4096)])
    assert cs.max() < 1.0 and cs.min() >= 0.0 and abs(cs.mean() - 0.5) < 0.02


def test_probabilities_equal_the_oracle_softmax_of_the_scaled_logits():
    rng = np.random.default_rng(1)
    x = (rng.standard_normal(3001) * 4).astype(np.float32)
    for T in (0.1, 0.8, 1.0, 1.7):
        want = (x / f32(T)).astype(np.float32).reshape(1, -1).copy()
        oc.softmax_(want)
        assert np.array_equal(S.probs(x, T).view(np.uint32), want.reshape(-1).view(np.uint32))


def test_sums_are_sequential():
    # np.add.accumulate must be the reference's left-to-right f32 sum, not numpy's pairwise np.sum
    rng = np.random.default_rng(2)
    v = rng.random(20000).astype(np.float32)
    acc = f32(0.0)
    for a in v:
        acc = f32(acc + a)
    assert np.add.accumulate(v, dtype=np.float32)[-1] == acc


@pytest.mark.parametrize("n", [1, 2, 33, 300])
def test_vectorised_restatement_equals_the_literal_transcription(n):
    rng = np.random.default_rng(n)
    rows = [(rng.standard_normal(n) * 3).astype(np.float32), np.round(rng.standard_normal(n)).astype(np.float32),
            np.zeros(n, np.float32)]
    for x in rows:
        for T in (0.1, 0.8, 1.0, 1.7):
            for topp in (0.0, 0.01, 0.5, 0.9, 1.0, 1.5):
                p = S.probs(x, T)
                w = S.topp_walk(p, topp)
                for i in range(4):
                    c = S.coin(11, i)
                    if w is None:
                        with pytest.raises(ValueError):
                            S.sample_literal(x, T, topp, c)
                    else:
                        assert S.pick(w, c) == S.sample_literal(x, T, topp, c), (n, T, topp, i)


U = 2.0 ** -24


@pytest.mark.parametrize("n", [33, 513, 4097, 32000, 152064])
def test_fast_orders_stay_within_the_derived_reordering_bound(n):
    """The fast devices' sums (emulated bit for bit by probs_fast / topp_walk_fast; the GPU test holds the kernel to the emulation)
    against the sequential reference, entry by entry, with first-order bounds derived from the two summation trees:
      p: the sequential softmax sum is within (n - 1) u of the exact one, the tree sum (n / 512 per thread, 5 butterfly levels, 16 warp
         sums) within (n / 512 + 21) u, and each side rounds its division once: |p_fast - p_ref| <= (n + n / 512 + 22) u p_ref;
      C_j: the reference's sequential prefix is within j u, the tile scan within its depth (8 local + 5 scan levels + 16 warp offsets
         + 3 combining adds + 16 + 5 + 8 inside each earlier tile total + one add per earlier tile: 61 + tiles) u, on top of the
         probabilities' own spread: |C_fast - C_ref| <= (n + n / 512 + 22 + j + 61 + tiles) u C_ref.
    Where the kept sets differ, every entry that differs lies within the probabilities' spread of the cutoff."""
    rng = np.random.default_rng(n)
    worst_p = worst_c = 0.0
    for kind in range(4):
        x = [(3.0 * rng.standard_normal(n)), rng.standard_normal(n) + 12.0 * (np.arange(n) == rng.integers(0, n)),
             rng.integers(0, 4, n).astype(np.float64), 1e-3 * rng.standard_normal(n)][kind].astype(np.float32)
        for T in (0.8, 1.0, 1.7):
            pr, pf = S.probs(x, T), S.probs_fast(x, T)
            kp = (n + n / 512 + 22) * U
            nz = pr > 0
            assert np.array_equal(pf == 0, pr == 0)
            ratio = float((np.abs(pf[nz] - pr[nz]) / (kp * pr[nz])).max())
            worst_p = max(worst_p, ratio)
            assert ratio <= 1.0, (kind, T, ratio)
            for topp in (0.01, 0.5, 0.9, 1.0):
                wr, wf = S.topp_walk(pr, topp), S.topp_walk_fast(pf, topp)
                if wr is None or wf is None:
                    assert wr is None and wf is None
                    continue
                cutoff = np.float32(np.float32(1.0) - np.float32(topp)) / np.float32(n - 1)
                if len(wr[0]) != len(wf[0]) or not np.array_equal(np.sort(wr[0]), np.sort(wf[0])):
                    diff = np.setxor1d(wr[0], wf[0])
                    assert (np.abs(pr[diff] - cutoff) <= kp * cutoff).all(), (kind, T, topp)
                    continue
                Cr, Cf = wr[1].astype(np.float64), wf[1].astype(np.float64)
                done = ~np.isnan(Cf) & (Cr > 0)
                j = np.arange(Cr.size)
                bound = (n + n / 512 + 22 + j + 61 + -(-Cr.size // 4096)) * U * Cr
                r = (np.abs(Cf - Cr)[done] / bound[done]).max() if done.any() else 0.0
                worst_c = max(worst_c, float(r))
                assert r <= 1.0, (kind, T, topp, r)
    print(f"n={n}: worst |p_fast - p_ref| / bound = {worst_p:.3g}, worst |C_fast - C_ref| / bound = {worst_c:.3g}")


def test_fast_emulation_equals_the_reference_where_the_orders_coincide():
    # fewer than 512 entries: every thread adds at most one term, so the tree sum of the softmax differs from the sequential one only
    # through the butterfly; a row of powers of two keeps every partial sum exact, so both orders must agree bit for bit
    x = np.log2(np.array([1, 2, 4, 8, 16, 32, 64, 128], np.float32)) * np.float32(np.log(2.0))
    for T in (1.0,):
        assert np.array_equal(S.probs_fast(x, T), S.probs(x, T))
    p = np.array([0.125, 0.5, 0.375, 0.0625, 0.0625, 0.25], np.float32)
    for topp in (0.3, 0.5, 1.0, 1.5):
        wr, wf = S.topp_walk(p, topp), S.topp_walk_fast(p, topp)
        assert np.array_equal(wr[0], wf[0]) and wr[2] == wf[2]
        assert np.array_equal(wr[1][:wr[2] + 1], wf[1][:wf[2] + 1])
