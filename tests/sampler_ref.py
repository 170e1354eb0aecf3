"""Reference for the device sampler (cc_sample_to_slot): Llama2Sampler::sample (crabml-llama2/src/sampler.rs:27-129) restated in f32
numpy, with the project's coin, and an emulation of the fast devices' two summation orders (sample_dev.cuh).  Test infrastructure only.

Every sum is SEQUENTIAL, as in the reference: np.add.accumulate runs left to right in the array's dtype (unlike np.sum, which pairs);
tests/test_sampler_ref.py checks this restatement against a literal loop-by-loop transcription of sampler.rs.  The one deliberate
divergence: where the reference panics (n0 == 0 -- no probability reaches the cutoff), the argmax of the logits is returned."""
from __future__ import annotations

import numpy as np

from oracle import oracle as oc

_M64 = (1 << 64) - 1


def splitmix64(x: int) -> int:
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def coin(seed: int, index: int) -> np.float32:
    """(splitmix64(seed ^ splitmix64(index)) >> 40) * 2^-24: 24 random bits, in [0, 1 - 2^-24]"""
    return np.float32((splitmix64((seed & _M64) ^ splitmix64(index & _M64)) >> 40) * 2.0 ** -24)


def argmax_last(logits: np.ndarray) -> int:
    """sampler.rs:109-116: max_by keeps the LAST maximum"""
    x = np.asarray(logits, np.float32)
    if np.isnan(x).any():
        best = 0
        for i in range(1, x.size):
            if not (x[i] < x[best]):
                best = i
        return best
    return int(x.size - 1 - np.argmax(x[::-1]))


def probs(logits: np.ndarray, temperature: float) -> np.ndarray:
    """sampler.rs:34-38 (logits / T) + softmax (:119-129) with the f16 exp LUT and a sequential sum"""
    with np.errstate(all="ignore"):
        v = np.asarray(logits, np.float32) / np.float32(temperature)
        m = np.fmax.reduce(v)                                   # fold from NaN with f32::max: NaN is ignored
        e = oc.f16_to_f32(oc.exp_lut()[oc.f32_to_f16((v - m).astype(np.float32))])
        s = np.add.accumulate(e, dtype=np.float32)[-1]
        return (e / s).astype(np.float32)


def topp_walk(p: np.ndarray, topp: float):
    """sampler.rs:76-95: the kept (p, index) pairs sorted ascending (stable), their sequential prefix sums C, and last_idx.
    None when n0 == 0."""
    n = p.size
    with np.errstate(all="ignore"):
        cutoff = np.float32(np.float32(1.0) - np.float32(topp)) / np.float32(n - 1)
        keep = np.nonzero(p >= cutoff)[0]
    if keep.size == 0:
        return None
    order = keep[np.argsort(p[keep], kind="stable")]
    C = np.add.accumulate(p[order], dtype=np.float32)
    over = np.nonzero(C > np.float32(topp))[0]
    last = int(over[0]) if over.size else order.size - 1
    return order, C, last


def pick(walk, c) -> int:
    """sampler.rs:97-106: r = coin * cumulative_prob; the first kept entry whose running cdf exceeds r, else prob_index[last_idx]"""
    order, C, last = walk
    r = np.float32(c) * C[last]
    hit = np.nonzero(C[:last + 1] > r)[0]
    return int(order[hit[0]]) if hit.size else int(order[last])


def sample(logits: np.ndarray, temperature: float, topp: float, seed: int, index: int) -> int:
    """what cc_sample_to_slot picks on an exact_order device"""
    if temperature == 0.0:
        return argmax_last(logits)
    walk = topp_walk(probs(logits, temperature), topp)
    return argmax_last(logits) if walk is None else pick(walk, coin(seed, index))


def sample_literal(logits, temperature: float, topp: float, c) -> int:
    """sampler.rs:27-129 transcribed statement by statement on f32 scalars (slow; small rows only).  Raises where the reference panics."""
    f = np.float32
    x = [f(v) for v in np.asarray(logits, np.float32)]
    if temperature == 0.0:
        return argmax_last(np.array(x, np.float32))
    with np.errstate(all="ignore"):
        x = [v / f(temperature) for v in x]
        mx = f("nan")
        for v in x:
            mx = v if np.isnan(mx) else (mx if np.isnan(v) else max(mx, v))
        lut = oc.exp_lut()
        total = f(0.0)
        for i, v in enumerate(x):
            x[i] = f(oc.f16_to_f32(lut[oc.f32_to_f16(np.array([v - mx], np.float32))])[0])
            total = f(total + x[i])
        x = [v / total for v in x]
        cutoff = (f(1.0) - f(topp)) / f(len(x) - 1)
    prob_index = [(v, i) for i, v in enumerate(x) if v >= cutoff]
    if not prob_index:
        raise ValueError("n0 == 0: the reference panics")
    prob_index.sort(key=lambda t: t[0])                         # stable, like slice::sort_by
    cum, last = f(0.0), len(prob_index) - 1
    for i, (pv, _) in enumerate(prob_index):
        cum = f(cum + pv)
        if cum > f(topp):
            last = i
            break
    r = f(c) * cum
    cdf = f(0.0)
    for pv, i in prob_index[:last + 1]:
        cdf = f(cdf + pv)
        if cdf > r:
            return i
    return prob_index[last][1]


# ---- the fast devices' orders (crabml_b200/csrc/sample_dev.cuh), emulated bit for bit -------------------------------------------------
def probs_fast(logits: np.ndarray, temperature: float) -> np.ndarray:
    """softmax with cc_block_sum_512's order: thread t adds t, t + 512, ... from 0; lane 0 of the xor butterfly; the 16 warp sums in order"""
    with np.errstate(all="ignore"):
        v = np.asarray(logits, np.float32) / np.float32(temperature)
        m = np.fmax.reduce(v)
        e = oc.f16_to_f32(oc.exp_lut()[oc.f32_to_f16((v - m).astype(np.float32))])
        pad = np.zeros(-(-e.size // 512) * 512, np.float32)
        pad[:e.size] = e
        per = np.add.accumulate(pad.reshape(-1, 512), axis=0, dtype=np.float32)[-1].reshape(16, 32)
        lanes = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            per = (per + per[:, lanes ^ o]).astype(np.float32)
        s = np.float32(0.0)
        for w in range(16):
            s = np.float32(s + per[w, 0])
        return (e / s).astype(np.float32)


def topp_walk_fast(p: np.ndarray, topp: float):
    """topp_walk with the tiled block scan: tiles of 4096 = 512 threads x 8 consecutive entries; C = carry + ((warp offset + lane
    offset) + local prefix), warp offsets and the tile total summed in warp order, lane offsets by a Hillis-Steele scan; the scan stops
    after the tile where C first exceeds topp (entries beyond it are never read)"""
    n = p.size
    with np.errstate(all="ignore"):
        cutoff = np.float32(np.float32(1.0) - np.float32(topp)) / np.float32(n - 1)
        keep = np.nonzero(p >= cutoff)[0]
    if keep.size == 0:
        return None
    order = keep[np.argsort(p[keep], kind="stable")]
    q = p[order]
    n0 = q.size
    C = np.full(n0, np.nan, np.float32)
    carry = np.float32(0.0)
    lanes = np.arange(32)
    for base in range(0, n0, 4096):
        tile = np.zeros(4096, np.float32)
        tile[:min(4096, n0 - base)] = q[base:base + 4096]
        loc = np.add.accumulate(tile.reshape(512, 8), axis=1, dtype=np.float32)
        inc = loc[:, 7].reshape(16, 32).copy()
        for o in (1, 2, 4, 8, 16):
            y = np.zeros_like(inc)
            y[:, o:] = inc[:, :-o]
            inc = np.where(lanes >= o, (inc + y).astype(np.float32), inc)
        ex = np.zeros_like(inc)
        ex[:, 1:] = inc[:, :-1]
        woff, tot = np.zeros(16, np.float32), np.float32(0.0)
        for w in range(16):
            woff[w] = tot
            tot = np.float32(tot + inc[w, 31])
        off = (woff[:, None] + ex).astype(np.float32).reshape(512, 1)
        c = (carry + (off + loc).astype(np.float32)).astype(np.float32).reshape(-1)[:min(4096, n0 - base)]
        C[base:base + c.size] = c
        carry = np.float32(carry + tot)
        if (c > np.float32(topp)).any():
            break
    done = ~np.isnan(C)
    over = np.nonzero(done & (C > np.float32(topp)))[0]
    last = int(over[0]) if over.size else n0 - 1
    return order, C, last


def sample_fast(logits: np.ndarray, temperature: float, topp: float, seed: int, index: int) -> int:
    """what cc_sample_to_slot picks on a fast device (every mode: eager, CUDA graph, both megakernels)"""
    if temperature == 0.0:
        return argmax_last(logits)
    walk = topp_walk_fast(probs_fast(logits, temperature), topp)
    return argmax_last(logits) if walk is None else pick(walk, coin(seed, index))
