"""Worker of tests/test_gpu_sampling.py::test_fast_modes_sample_bit_identical_ids_on_ring_and_k_quant_kernels: sampled generation
(temperature / top-p on the device) in one execution mode; saves the ids, the exported logits and the persistent kernel that ran.
The prompt is one token, so every flush of the run contains the sampler."""
import sys

import numpy as np

sys.path.insert(0, ".")
from crabml_b200 import CudaTensorDevice  # noqa: E402
from crabml_b200 import runner as R  # noqa: E402
from oracle import oracle as oc  # noqa: E402


def run(lazy, build, steps, temperature, topp, seed):
    dev = CudaTensorDevice(0, lazy=lazy)
    try:
        conf, w, kv = build(dev)
        r = R.LlamaRunner(dev, conf, w, kv)
        ids, logits = r.generate_logits([1], steps, temperature, topp, seed)
        variant = dev.mega_variant() if lazy else 0
        r.close()
    finally:
        dev.close()
    return np.array(ids, np.int64), logits, np.int64(variant)


def main():
    lazy, gguf, out = int(sys.argv[1]), sys.argv[2], sys.argv[3]
    res = {}

    def tiny(dev):
        conf, w, _ = R.load_gguf(gguf, dev)
        return conf, w, 128

    def l7b(wt, ct):       # one Llama-2-7B-shaped layer on bench.py's synthetic weights
        def build(dev):
            conf = R.LlamaConfig(32, 32, 1, 4096, 11008, 4096, 32000, 1e-5, 128)
            return conf, R.synthetic_weights(dev, conf, wt, ct, seed=7), 80
        return build
    res["tiny_ids"], res["tiny_logits"], res["tiny_variant"] = run(lazy, tiny, 96, 0.8, 0.9, 1234)
    res["l7b_ids"], res["l7b_logits"], res["l7b_variant"] = run(lazy, l7b(oc.Q8_0, oc.Q8_0), 66, 1.0, 0.9, 99)
    res["l7bk_ids"], res["l7bk_logits"], res["l7bk_variant"] = run(lazy, l7b(oc.Q4_K, oc.Q6_K), 66, 1.0, 0.9, 99)
    np.savez(out, **res)


if __name__ == "__main__":
    main()
