"""Per-phase time inside the megakernel (CRABML_MEGA_PROF=1): which phases/barriers the token time goes to."""
import collections
import os
import sys

os.environ["CRABML_MEGA_PROF"] = "1"
sys.path.insert(0, ".")
import numpy as np  # noqa: E402
from crabml_b200 import CudaTensorDevice, capi  # noqa: E402
from crabml_b200 import runner as R  # noqa: E402

wl = sys.argv[1] if len(sys.argv) > 1 else "Q8_0"
wt = {"Q8_0": capi.Q8_0, "Q4_0": capi.Q4_0, "Q4_K": capi.Q4_K, "Q6_K": capi.Q6_K, "Q4_0-Q6K": capi.Q4_0}[wl]      # body type
ct = capi.Q6_K if wl in ("Q4_K", "Q4_0-Q6K") else wt                                                                # classifier type
dev = CudaTensorDevice(0, lazy=2)
conf = R.LLAMA2_7B
w = R.synthetic_weights(dev, conf, wt, ct)
WARM = int(os.environ.get("MEGA_PROFILE_WARM", "40"))          # tokens decoded before the timed 40 (sets the KV length the profile sees)
r = R.LlamaRunner(dev, conf, w, WARM + 88)
pos = 0
for i in range(WARM):
    r.forward([1 + i], pos, export=False); pos += 1
dev.synchronize()
dev.timer_begin()
for i in range(40):
    r.forward([100 + i], pos, export=False); pos += 1
ms = dev.timer_end()
print(f"40 tokens back to back: {ms / 40 * 1e3:.1f} us per token by CUDA events (kernel time below + inter-launch gap)")
stamps, ty = dev.mega_profile()
n = len(ty)
raw = stamps.astype(np.float64)
t = raw[:, 0]
d = np.diff(t) / 1e3
base = {0: "normq", 16 + 3: "qkv", 16 + 1 + 4: "mv+res", 16 + 2 + 8: "gate/up", 16 + 1: "mv", 32: "attn", 48: "rows",
        16 + 1 + 12: "mv->xchg", 64: "reduce", 80: "gather"}


def name(code):
    k = code >> 10
    b = base.get(code & 1023, str(code & 1023))
    return f"{b} k={k}K" if k else b


agg = collections.defaultdict(list)
sub = collections.defaultdict(list)
for i in range(n):
    k = name(ty[i])
    agg[k].append(d[i])
    s0, s1, s2, s3, s4, s5 = raw[i, :6]
    s8 = raw[i, 8]
    act = (s1 - s0) / 1e3 if s1 > 0 else 0.0            # activation staging / fused prologue (MATVEC only)
    wa = (s8 - s0) / 1e3 if s8 > 0 else 0.0             # prologue: norm weights available (ring kernel: the stage filled a phase ago)
    xs = (s4 - s0) / 1e3 if s4 > 0 else 0.0             # prologue: x landed in shared memory (mega.cu: x and weights)
    rm = (s5 - s4) / 1e3 if s5 > 0 and s4 > 0 else 0.0  # prologue: rms known
    qz = (s1 - s5) / 1e3 if s5 > 0 and s1 > 0 else 0.0  # prologue: quantised
    cw, pk = int(stamps[i, 6]), int(stamps[i, 7])          # ring kernel: warp 0 wait cycles ; (row-loop cycles << 20) | entries
    sub[k].append((act, (s2 - max(s0, s1)) / 1e3, (s3 - s2) / 1e3, (raw[i + 1, 0] - s3) / 1e3, xs, rm, qz, cw, pk >> 20, pk & 0xFFF, wa))
print(f"phases {n}, token total {(t[-1] - t[0]) / 1e3:.1f} us (phase time includes the barrier that ends it)")
print("  CTA 0 per phase: activation ready | rows of warp 0 done | arrive | barrier wait || prologue, from phase start: weights available | x landed"
      " || then: rms known | quantised")
for k, v in sorted(agg.items(), key=lambda kv: -sum(kv[1])):
    m = np.mean(np.array(sub[k]), axis=0)
    ringinfo = f" || ring w0: {m[9]:4.1f} entries, {m[8] / max(m[9], 1):6.0f} cyc/entry, waiting {100 * m[7] / max(m[8], 1):3.0f} %" if m[9] > 0 else ""
    print(f"  {k:16s} n={len(v):3d}  sum {sum(v):8.1f} us  avg {np.mean(v):6.2f}  min {min(v):6.2f}  max {max(v):6.2f}   | {m[0]:5.2f} | {m[1]:5.2f} | {m[2]:5.2f} | {m[3]:5.2f} || {m[10]:5.2f} | {m[4]:5.2f} || {m[5]:5.2f} | {m[6]:5.2f}{ringinfo}")
tail = [int(stamps[n, i]) for i in range(1, 5)]      # producer trips, cycles, entries; ring slots
if tail[0]:
    print(f"  ring producer (CTA 0, lane 0): {tail[0]} trips, {tail[2]} entries issued, {tail[1] / tail[0]:.0f} cycles per trip, {tail[1] / 1.965e3:.0f} us inside streaming phases")
    # ring occupancy of CTA 0 (slot 9) as the barrier in front of a phase opened: entries beyond the consumers' position that the producers
    # had issued / that had landed.  No slot is handed back before the phase's rows start, so a ring full here stays full, and this SM
    # reads no weights, through the prologue (and, for an attention phase, the whole phase)
    nslots = tail[3]
    print(f"  ring occupancy as the barrier in front of the phase opened (CTA 0, entries landed / issued ahead of the consumers; {nslots} slots):")
    occ = collections.defaultdict(list)
    for i in range(1, n):
        o = int(stamps[i, 9])
        occ[name(ty[i])].append((o >> 8 & 0xFF, o & 0xFF))
    for k, v in occ.items():
        a = np.array(v, dtype=np.float64)
        print(f"    {k:16s} {np.mean(a[:, 0]):5.1f} / {np.mean(a[:, 1]):5.1f}   full in {100 * np.mean(a[:, 0] >= nslots):3.0f} % of {len(a)}")
dev.close()
