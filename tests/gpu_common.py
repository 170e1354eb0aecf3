import contextlib

import numpy as np

from oracle.tensor_ref import OracleTensor

# execution modes by name -> device options; "register" and "ring" differ in what the test puts in the flush
MODE_DEVICE = {"eager": dict(lazy=0), "graph": dict(lazy=1), "register": dict(lazy=2), "ring": dict(lazy=2), "exact": dict(exact_order=True)}


def make_device(**kw):
    from crabml_b200 import CudaTensorDevice
    return CudaTensorDevice(**kw)


@contextlib.contextmanager
def fresh_device(**kw):
    dev = make_device(**kw)
    try:
        yield dev
    finally:
        dev.close()


def run_modes(body, modes=(0, 1, 2), **device_kw):
    """body(dev) on a fresh device in each lazy mode -> {mode: what body returned}"""
    out = {}
    for m in modes:
        with fresh_device(lazy=m, **device_kw) as dev:
            out[m] = body(dev)
    return out


def assert_same_bits(got, want, what):
    """got and want (arrays, or tuples / lists of them) have the same dtype, shape and bytes"""
    if isinstance(want, (tuple, list)):
        assert isinstance(got, (tuple, list)) and len(got) == len(want), (what, "lengths", len(got) if isinstance(got, (tuple, list)) else got, len(want))
        for i, (g, w) in enumerate(zip(got, want)):
            assert_same_bits(g, w, f"{what}[{i}]")
        return
    g, w = np.asarray(got), np.asarray(want)
    assert g.dtype == w.dtype and g.shape == w.shape, (what, g.dtype, g.shape, "want", w.dtype, w.shape)
    n = (g.size, g.dtype.itemsize)
    differ = (np.ascontiguousarray(g).view(np.uint8).reshape(n) != np.ascontiguousarray(w).view(np.uint8).reshape(n)).any(1)
    assert not differ.any(), (what, f"{int(differ.sum())} of {g.size} differ, first at flat indices {np.flatnonzero(differ)[:8].tolist()}")


_SMS = []


def full_grid():
    """SMs of the device: the persistent grid when no limit is set"""
    if not _SMS:
        import torch
        _SMS.append(torch.cuda.get_device_properties(0).multi_processor_count)
    return _SMS[0]


def both(values, shape, gdev, odev):
    from crabml_b200 import CudaTensor
    v = np.asarray(values, np.float32)
    return CudaTensor.new(v, shape, gdev), OracleTensor.new(v, shape, odev)
