"""Profiling driver: the four Llama-2-7B matvec shapes, cycling over enough distinct matrices to defeat L2.
Usage:  ncu --set full -k regex:matvec_kernel -s 8 -c 4 -o mv python tools/prof_matvec.py Q8_0 11008 4096"""
import sys

import numpy as np

sys.path.insert(0, ".")
from crabml_b200 import CudaTensor, CudaTensorDevice, capi  # noqa: E402
from crabml_b200.runner import synth_scale, weight_bytes  # noqa: E402

T = {"Q8_0": capi.Q8_0, "Q4_0": capi.Q4_0, "Q4_K": capi.Q4_K, "Q6_K": capi.Q6_K, "Q4_1": capi.Q4_1, "Q5_0": capi.Q5_0,
     "Q5_1": capi.Q5_1, "Q2_K": capi.Q2_K, "Q3_K": capi.Q3_K, "Q5_K": capi.Q5_K}
tname = sys.argv[1] if len(sys.argv) > 1 else "Q8_0"
shapes = [(int(sys.argv[2]), int(sys.argv[3]))] if len(sys.argv) > 3 else [(4096, 4096), (11008, 4096), (4096, 11008), (32000, 4096)]
reps = int(sys.argv[4]) if len(sys.argv) > 4 else 5
dev = CudaTensorDevice()
t = T[tname]
for (m, k) in shapes:
    nbytes = weight_bytes(t, m, k)
    nmat = max(2, int(400e6 // nbytes))
    mats = [CudaTensor.synth([m, k], t, dev, 1, i + 1, synth_scale(t, k)) for i in range(nmat)]
    x = CudaTensor.new(np.random.default_rng(0).standard_normal(k).astype(np.float32), [k], dev)
    for w in mats[:2]:
        w.matmul_vec(x)
    dev.synchronize()
    l0 = dev.launch_count()
    dev.timer_begin()
    for _ in range(reps):
        for w in mats:
            w.matmul_vec(x)
    ms = dev.timer_end()
    n = reps * nmat
    print(f"{tname} {m}x{k}: {ms / n * 1e3:.2f} us per matmul_vec ({(dev.launch_count() - l0) / n:.0f} launches), "
          f"{nbytes / (ms / n * 1e-3) / 1e9:.0f} GB/s algorithmic")
dev.close()
