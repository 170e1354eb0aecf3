"""Sharded decode path on real GPUs (SURVEY §8e).  The one-process tests run the exchange protocol with a world of 1 (the
peer stores, flag handshake and slot reduction all execute, against this GPU's own window), so they also run on a
single-GPU box; the N-process test needs >= 2 GPUs (`python -m pytest tests/test_gpu_sharded.py -m gpu` on a 2-GPU machine)."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from tests.gpu_common import make_device

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("lazy", [0, 1, 2])
def test_exchange_ops_world_of_one(lazy):
    """matvec -> all_reduce -> + residual and matvec -> all_gather through every execution mode: with one rank the
    exchange is the identity, so the result must equal the plain ops bit for bit."""
    from crabml_b200 import CudaTensor, capi
    from crabml_b200.runner import synth_scale
    ref_dev = make_device(lazy=0)
    dev = make_device(lazy=lazy)
    try:
        dev.init_comm(0, 1)
        rng = np.random.default_rng(3)
        k, m = 4096, 1024
        xs = [rng.standard_normal(k).astype(np.float32) for _ in range(4)]
        res = rng.standard_normal(m).astype(np.float32)
        outs = {}
        for name, d in (("ref", ref_dev), ("dut", dev)):
            w = CudaTensor.synth([m, k], capi.Q8_0, d, 5, 1, synth_scale(capi.Q8_0, k))
            got = []
            for x in xs:           # several rounds: sequence numbers / slot parity advance, graphs are replayed
                xt = CudaTensor.new(x, [k], d)
                r = CudaTensor.new(res, [m], d)
                y = w.matmul_vec(xt)
                if name == "dut":
                    y = y.all_reduce_sum_inplace()
                y = y.add_inplace(r)
                z = w.matmul_vec(xt)
                if name == "dut":
                    z = CudaTensor.alloc([m], capi.F32, d).all_gather_from(z)
                got.append(np.concatenate([y.export(), z.export()]))
            outs[name] = np.stack(got)
        ref, dut = outs["ref"], outs["dut"]
        tol = 1e-6 * float(np.abs(ref).max()) * 64      # eager ref uses the warp-per-row kernel, lazy the streaming one
        np.testing.assert_allclose(dut, ref, rtol=0, atol=tol)
        if lazy:
            st = dev.lazy_stats()
            assert st["uncached"] == 0, st
    finally:
        dev.close()
        ref_dev.close()


def test_exchange_requires_a_communicator():
    from crabml_b200 import CudaTensor, TensorError
    dev = make_device()
    try:
        with pytest.raises(TensorError):
            CudaTensor.new(np.zeros(32, np.float32), [32], dev).all_reduce_sum_inplace()
    finally:
        dev.close()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_two_gpus_sharded_llama_matches_single_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    n = min(int(os.environ.get("CRABML_TEST_WORLD", "2")), torch.cuda.device_count())
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n), "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "sharded_worker.py"), "--mode", "gpu"]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]


@pytest.mark.parametrize("n", [2, 8])
def test_processes_on_one_gpu_sharded_llama(n):
    """World of 2 / 8 on ONE GPU, one process per rank (time-sliced contexts, peers' windows mapped through CUDA IPC exactly as across
    GPUs): the exchange ops bit-exact against the rank-ordered numpy sum, and the 2-layer Llama-2-7B-shaped sharded model in the
    eager, CUDA-graph and megakernel modes -- ranks bit-identical, modes bit-identical, close to the unsharded logits.
    This is the multi-GPU path's parity test on a single-GPU lease (tests/sharded_worker.py --one-gpu); world 8 runs the shard shapes
    of the 8-GPU box (k = 512 / 1376: one short, ragged segment per row) through the same kernels."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n), "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "sharded_worker.py"), "--mode", "gpu", "--one-gpu"]
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
    assert "sharded parity vs single GPU" in p.stdout
