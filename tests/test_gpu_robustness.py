"""The persistent megakernel must fail loudly, never hang: every spin in it is bounded (MkSpin, csrc/mega.cu) and a timed-out
barrier surfaces as CudaError at the next synchronising call.  VERDICT r1 #6 / ADVICE r1 (mega.cu:888)."""
import os
import subprocess
import sys
import time

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import sys, time
sys.path.insert(0, %r)
from crabml_b200 import CudaTensorDevice, CudaError, TensorError
from crabml_b200 import capi, runner as R
dev = CudaTensorDevice(0, lazy=2)
conf = R.LlamaConfig(8, 8, 2, 1024, 2048, 64, 512, 1e-5, 128)
wt = getattr(capi, sys.argv[1]) if len(sys.argv) > 1 else capi.Q8_0
w = R.synthetic_weights(dev, conf, wt, wt, seed=3)
r = R.LlamaRunner(dev, conf, w, 16)
t0 = time.time()
try:
    r.forward([1], 0)
    print("NO-ERROR")
except (CudaError, TensorError) as e:      # the C++ runner reports every failed trait call as its TensorError, like the reference
    print("ERROR:", e, "after %%.1f s" %% (time.time() - t0))
r.close(); dev.close()
print("CLEAN-EXIT")
""" % ROOT


# Q4_K weights run mega_kernel (mega.cu), Q8_0 weights the ring kernel (mega_ring.cu)
@pytest.mark.parametrize("wt", ["Q4_K", "Q8_0"], ids=["register-pipe kernel", "ring kernel"])
def test_deserting_cta_is_a_timeout_error_not_a_hang(wt):
    """test hook MK_F_TESTSTALL (0x80): the last CTA leaves before the third grid barrier, i.e. the grid behaves as if one CTA had
    never become resident (another tenant on the GPU).  Every other CTA must give up after the spin bound, the kernel must drain
    (ring kernel: the producer warps stop, bulk copies in flight land before the CTA's shared memory goes away), and the host must
    see CC_ERR_CUDA 'megakernel barrier timeout' -- within seconds."""
    env = dict(os.environ, CRABML_MEGA_FLAGS=str(0x80))          # the only bit of the word that has an effect
    t0 = time.time()
    p = subprocess.run([sys.executable, "-c", CHILD, wt], env=env, capture_output=True, text=True, timeout=120)
    out = p.stdout + p.stderr
    assert "ERROR:" in out and "barrier timeout" in out, out
    assert "CLEAN-EXIT" in out, out
    assert time.time() - t0 < 90


def test_same_child_without_the_hook_runs():
    p = subprocess.run([sys.executable, "-c", CHILD], env=dict(os.environ), capture_output=True, text=True, timeout=120)
    assert "NO-ERROR" in p.stdout and "CLEAN-EXIT" in p.stdout, p.stdout + p.stderr


def test_context_too_long_for_the_persistent_kernels_falls_back_to_the_graph_mode():
    """A 40 K-token KV cache: the attention phase's score row alone (160 KB) leaves no room for its chunk buffers in shared memory, so
    lazy = 2 must run the token as the CUDA graph of fused kernels instead of failing -- same bits as the eager kernels."""
    import numpy as np
    from crabml_b200 import capi
    from crabml_b200 import runner as R
    from crabml_b200.tensor import MEGA_NONE
    from tests.gpu_common import assert_same_bits, run_modes
    conf = R.LlamaConfig(32, 32, 1, 4096, 11008, 40000, 32000, 1e-5, 128)

    def body(dev):
        w = R.synthetic_weights(dev, conf, capi.Q8_0, capi.Q8_0, seed=5)
        r = R.LlamaRunner(dev, conf, w, 40000)
        logits = np.stack([r.forward([t], p).copy() for p, t in enumerate([1, 9, 31999])])
        r.close()
        return logits, dev.mega_variant(), dev.lazy_stats()
    res = run_modes(body, modes=(0, 2))
    assert res[2][1] == MEGA_NONE, "expected the CUDA-graph fallback"
    assert res[2][2]["uncached"] == 0, res[2][2]
    assert_same_bits(res[2][0], res[0][0], "lazy=2 vs eager")
