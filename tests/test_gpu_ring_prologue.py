"""The ring kernel's fused prologues (mega_ring.cu) against the eager kernels: the norm weights of each fused-norm phase are staged
in shared memory one such phase ahead (the first at kernel start), and the input row is requested into shared memory as the grid
barrier opens.  Only where the inputs arrive changes, so lazy mode 2 must reproduce eager logits bit for bit at every token, on
tables where the weight producers run several phases ahead (tiny rows), on 7B rows, with a K-quant classifier that reads the same
stage, and with an ffn_down row wider than 8192 and no norm."""
import numpy as np
import pytest

from oracle import oracle as oc
from crabml_b200.tensor import MEGA_RING
from tests.gpu_common import assert_same_bits, run_modes

pytestmark = pytest.mark.gpu

TOKENS = 24


def _logits(conf, wt, ct):
    """-> body(dev): the logits of TOKENS tokens and the persistent kernel that ran"""
    from crabml_b200 import runner as R

    def body(dev):
        w = R.synthetic_weights(dev, conf, wt, ct, seed=0x5A6E)
        r = R.LlamaRunner(dev, conf, w, 64)
        toks = [int(t) for t in np.random.default_rng(5).integers(1, conf.vocab_size, TOKENS)]
        out = np.stack([r.forward([t], p).copy() for p, t in enumerate(toks)])
        variant = dev.mega_variant()
        r.close()
        return out, variant
    return body


@pytest.mark.parametrize("shape,wt,ct", [
    ((4, 4, 4, 256, 768, 64, 512), oc.Q8_0, oc.Q8_0),            # tiny multi-layer Q8_0: producers many phases ahead
    ((4, 4, 4, 256, 768, 64, 512), oc.Q4_0, oc.Q4_0),            # tiny multi-layer Q4_0
    ((32, 32, 2, 4096, 11008, 64, 2048), oc.Q8_0, oc.Q8_0),      # Llama-2-7B rows, two layers
    ((8, 8, 2, 512, 1536, 64, 1024), oc.Q4_0, oc.Q6_K),          # Q6_K classifier: a generic phase reading the stage
    ((4, 4, 2, 256, 9216, 64, 512), oc.Q8_0, oc.Q8_0),           # ffn_down: k = 9216 > 8192, no norm
], ids=["tiny-q8_0", "tiny-q4_0", "7b-rows-q8_0", "q4_0-q6k", "wide-ffn-down"])
def test_ring_prologue_matches_eager(shape, wt, ct):
    from crabml_b200 import runner as R
    conf = R.LlamaConfig(*shape, 1e-5, shape[3] // shape[0])
    res = run_modes(_logits(conf, wt, ct), modes=(0, 2))
    (ref, _), (got, variant) = res[0], res[2]
    assert variant == MEGA_RING, "expected the ring kernel"
    assert np.isfinite(ref).all() and np.abs(ref).max() > 1e-3
    assert_same_bits(got, ref, "lazy=2 vs eager")
