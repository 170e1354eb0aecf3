"""Cost of the device sampler (cc_sample_to_slot).  Needs a GPU; prints the card and its power limit first.
  1. the standalone one-CTA kernel (CUDA events over many launches) at vocab 32 000 and 152 064, fast and exact_order sums;
  2. Llama-2-7B Q8_0 synthetic decode in lazy mode 2 (one megakernel per token), greedy against sampled (T = 1, p = 0.9), alternating
     A B A B: ms per token, and the sampled token's extra time as a share of it.
usage: python tools/sample_bench.py [--tokens 64] [--rounds 3]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from crabml_b200 import CudaTensor, CudaTensorDevice  # noqa: E402
from crabml_b200 import runner as R  # noqa: E402
from oracle import oracle as oc  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi unavailable)"


def kernel_us(n, exact, launches=200):
    dev = CudaTensorDevice(0, exact_order=exact)
    try:
        x = CudaTensor.new((2.0 * np.random.default_rng(n).standard_normal(n)).astype(np.float32), [n], dev)
        for i in range(10):
            x.sample_to_slot(1.0, 0.9, 1, i)
        dev.timer_begin()
        for i in range(launches):
            x.sample_to_slot(1.0, 0.9, 1, i)
        return dev.timer_end() * 1e3 / launches
    finally:
        dev.close()


def decode_ms(r, dev, tokens, temperature):
    r.generate([1], 4, temperature, 0.9, 7)           # warm: captures
    dev.synchronize()
    t0 = time.perf_counter()
    ids = r.generate([1], tokens, temperature, 0.9, 7)
    dev.synchronize()
    return (time.perf_counter() - t0) * 1e3 / len(ids)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    print("card (name, power limit, max SM clock):", card())
    for n in (32000, 152064):
        for exact in (False, True):
            print(f"sampler kernel n={n:6d} {'exact_order' if exact else 'fast       '}: {kernel_us(n, exact):8.1f} us per call")
    dev = CudaTensorDevice(0, lazy=2)
    try:
        conf = R.LlamaConfig(32, 32, 32, 4096, 11008, 4096, 32000, 1e-5, 128)
        w = R.synthetic_weights(dev, conf, oc.Q8_0, oc.Q8_0, seed=7)
        res = {"greedy": [], "sampled": []}
        for _ in range(a.rounds):
            for name, T in (("greedy", 0.0), ("sampled", 1.0)):
                r = R.LlamaRunner(dev, conf, w, a.tokens + 8)
                res[name].append(decode_ms(r, dev, a.tokens, T))
                if name == "sampled":
                    assert dev.mega_variant() in (1, 2)
                r.close()
                print(f"  {name:7s} {res[name][-1]:.3f} ms/token (prompt + {a.tokens} tokens, lazy 2, megakernel variant {dev.mega_variant()})")
        g, s = min(res["greedy"]), min(res["sampled"])
        print(f"Llama-2-7B Q8_0 lazy 2: greedy {g:.3f} ms/token, sampled (T=1, p=0.9) {s:.3f} ms/token; the sampler phase: {s - g:.3f} ms = "
              f"{100 * (s - g) / s:.1f} % of a sampled token (best of {a.rounds} alternating rounds)")
    finally:
        dev.close()


if __name__ == "__main__":
    main()
