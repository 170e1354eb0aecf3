"""Per-phase time inside the megakernel on the SHARDED path: run under torchrun with N ranks (one per GPU); rank 0 prints its profile.
  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/mega_profile_sharded.py"""
import collections
import os
import sys

os.environ["CRABML_MEGA_PROF"] = "1"
sys.path.insert(0, ".")
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
from crabml_b200 import CudaTensorDevice, capi, sharding  # noqa: E402
from crabml_b200 import runner as R  # noqa: E402

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("cpu:gloo,cuda:nccl", device_id=torch.device("cuda", rank))


def exchange(blob):
    out = [None] * world
    dist.all_gather_object(out, blob)
    return out


dev = CudaTensorDevice(rank, lazy=2)
conf = R.LLAMA2_7B
plan = sharding.make_plan(conf.n_heads, conf.n_kv_heads, conf.embedding_dim, conf.hidden_dim, conf.vocab_size, capi.Q8_0, rank, world)
dev.init_comm(rank, world, exchange, "p2p")
w = R.synthetic_weights(dev, conf, capi.Q8_0, capi.Q8_0, plan=plan)
r = R.LlamaRunner(dev, conf, w, 128, plan=plan)
pos = 0
for i in range(40):
    r.forward([1 + i], pos, export=False); pos += 1
dev.synchronize(); dist.barrier()
dev.timer_begin()
for i in range(40):
    r.forward([100 + i], pos, export=False); pos += 1
ms = dev.timer_end()
stamps, ty = dev.mega_profile()
n = len(ty)
if rank == 0:
    raw = stamps.astype(np.float64)
    t = raw[:, 0]
    d = np.diff(t) / 1e3
    base = {0: "normq", 16 + 3: "qkv", 16 + 1 + 4: "mv+res", 16 + 2 + 8: "gate/up", 16 + 1: "mv", 32: "attn", 48: "rows", 16 + 1 + 12: "mv->xchg", 64: "reduce", 80: "gather"}
    agg = collections.defaultdict(list); sub = collections.defaultdict(list)
    for i in range(n):
        k = f"{base.get(ty[i] & 1023, str(ty[i] & 1023))} k={ty[i] >> 10}K"
        agg[k].append(d[i])
        s0, s1, s2, s3 = raw[i, :4]
        sub[k].append(((s1 - s0) / 1e3 if s1 > 0 else 0.0, (s2 - max(s0, s1)) / 1e3, (s3 - s2) / 1e3, (raw[i + 1, 0] - s3) / 1e3))
    print(f"world {world}: {ms / 40 * 1e3:.1f} us per token (events); phases {n}, token total {(t[-1] - t[0]) / 1e3:.1f} us")
    print("  activation ready | rows done | arrive | barrier wait (incl. the cross-GPU handshake on exchange phases)")
    for k, v in sorted(agg.items(), key=lambda kv: -sum(kv[1])):
        m = np.mean(np.array(sub[k]), axis=0)
        print(f"  {k:18s} n={len(v):3d}  sum {sum(v):8.1f} us  avg {np.mean(v):6.2f}   | {m[0]:5.2f} | {m[1]:5.2f} | {m[2]:5.2f} | {m[3]:5.2f}")
dist.barrier()
r.close(); dev.close()
dist.destroy_process_group()
