"""Profiling driver of the dense (prefill) matmul_vec: one weight matrix against a (b, k) activation, a few repetitions.
Usage:  python tools/prof_prefill.py Q8_0 4096 4096 4096   (the GEMM kernel is wgmma_gemm_kernel)"""
import sys

import numpy as np

sys.path.insert(0, ".")
from crabml_b200 import CudaTensor, CudaTensorDevice, capi  # noqa: E402
from crabml_b200.runner import synth_scale  # noqa: E402

T = {"Q8_0": capi.Q8_0, "Q4_0": capi.Q4_0, "Q4_K": capi.Q4_K, "Q6_K": capi.Q6_K}
tname = sys.argv[1] if len(sys.argv) > 1 else "Q8_0"
m, k, b = (int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])) if len(sys.argv) > 4 else (4096, 4096, 4096)
reps = int(sys.argv[5]) if len(sys.argv) > 5 else 5
dev = CudaTensorDevice()
w = CudaTensor.synth([m, k], T[tname], dev, 1, 1, synth_scale(T[tname], k))
x = CudaTensor.new(np.random.default_rng(0).standard_normal(b * k).astype(np.float32), [b, k], dev)
for _ in range(2):
    w.matmul_vec(x)
dev.synchronize()
l0 = dev.launch_count()
dev.timer_begin()
for _ in range(reps):
    w.matmul_vec(x)
ms = dev.timer_end()
print(f"{tname} ({m},{k}) @ ({b},{k}): {ms / reps * 1e3:.1f} us per matmul_vec ({(dev.launch_count() - l0) / reps:.0f} launches: quantise, dequantise, "
      f"f16 activation, GEMM) = {2.0 * m * k * b / (ms / reps * 1e-3) / 1e12:.0f} TFLOP/s over the whole call")
dev.close()
