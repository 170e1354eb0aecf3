"""Decode speed of a Qwen2-7B-SHAPED model (28 layers, dim 3584, 28 heads on 4 kv heads, head_dim 128, hidden 18944, vocab 152064;
synthetic weights generated on the device) in lazy mode 1 (fused kernels in a CUDA graph) and lazy mode 2 (one persistent kernel per
token), for Q8_0 and for Q4_0 with a Q6_K classifier.

    python tools/qwen2_decode_bench.py [--steps 128] [--warmup 16] [--parent-lib PATH]

--parent-lib: another build of libcrabml_cuda.so (for example one of an earlier commit) timed beside this one in lazy mode 2, each
configuration in a process of its own, the two libraries alternating.  Prints one JSON line per measurement and the card's name and
power limit, which belong beside every number."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WEIGHTS = {"q8_0": ("Q8_0", "Q8_0"), "q4_0": ("Q4_0", "Q6_K")}


def measure(wname, lazy, steps, warmup):
    sys.path.insert(0, ROOT)
    from crabml_b200 import CudaTensorDevice, capi
    from crabml_b200 import runner as R
    wt, ct = (getattr(capi, n) for n in WEIGHTS[wname])
    conf = R.LlamaConfig(28, 4, 28, 3584, 18944, 4096, 152064, 1e-6, 128, "qwen2")
    dev = CudaTensorDevice(0, lazy=lazy)
    try:
        r = R.LlamaRunner(dev, conf, R.synthetic_weights(dev, conf, wt, ct, seed=0x0E2), steps + warmup + 8)
        r.generate_greedy([1], warmup)                       # captures the token graphs
        l0 = dev.launch_count()
        t0 = time.perf_counter()
        ids = r.generate_greedy([1], steps)                  # returns once the last token is on the host
        dt = time.perf_counter() - t0
        launches = (dev.launch_count() - l0) / max(1, len(ids))
        variant = dev.mega_variant()
        r.close()
    finally:
        dev.close()
    return {"weights": wname, "lazy": lazy, "steps": len(ids), "tok_s": len(ids) / dt, "launches_per_token": launches, "mega_variant": variant}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=2, help="alternating rounds of every configuration")
    ap.add_argument("--parent-lib", help="another libcrabml_cuda.so, timed in lazy mode 2 beside this build")
    ap.add_argument("--one", nargs=2, metavar=("WEIGHTS", "LAZY"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.one:
        print(json.dumps(measure(a.one[0], int(a.one[1]), a.steps, a.warmup)))
        return
    print(json.dumps({"card": card()}))
    runs = [(w, lazy, None) for w in WEIGHTS for lazy in (1, 2)]
    if a.parent_lib:
        runs += [(w, 2, os.path.abspath(a.parent_lib)) for w in WEIGHTS]
    for rnd in range(a.rounds):
        for w, lazy, lib in runs:
            env = dict(os.environ)
            env.pop("CRABML_CUDA_LIB", None)
            if lib:
                env["CRABML_CUDA_LIB"] = lib
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", w, str(lazy), "--steps", str(a.steps), "--warmup", str(a.warmup)],
                               env=env, capture_output=True, text=True)
            if p.returncode != 0:
                sys.stderr.write(p.stderr)
                raise SystemExit(f"{w} lazy={lazy} failed")
            res = json.loads(p.stdout.strip().splitlines()[-1])
            res.update(round=rnd, library="parent" if lib else "this")
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
