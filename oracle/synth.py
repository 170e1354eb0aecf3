"""CPU twin of the on-device synthetic weight generator (crabml_b200/csrc/repack.cu: synth_kernel /
synth_scales_kernel), implemented in oracle/crabml_oracle.c (oc_synth_blocks).  TEST INFRASTRUCTURE: lets the
oracle and the CPU baseline run on exactly the weights the GPU synthesised (SURVEY §8d configs 3-5) without
shipping gigabytes of weights.  Bit-equality with the device generator: tests/test_gpu_synth.py."""
from __future__ import annotations

import numpy as np

from . import oracle as oc


def synth_blocks(t: int, nblocks: int, seed: int, tensor_id: int, scale: float) -> np.ndarray:
    """-> uint8 array of nblocks * block_bytes(t) bytes in GGUF layout, identical to cc_tensor_synth."""
    out = oc.big_empty(nblocks * oc.block_bytes(t))
    rc = oc.lib().oc_synth_blocks(t, nblocks, seed, tensor_id, float(np.float32(scale)), out.ctypes.data_as(oc.C.c_void_p))
    assert rc == 0
    return out


def synth_weight(t: int, rows: int, cols: int, seed: int, tensor_id: int, scale: float) -> np.ndarray:
    return synth_blocks(t, rows * (cols // oc.block_elems(t)), seed, tensor_id, scale)
