"""Regenerates tests/golden/*_logits.npz from the reference's GGUF fixtures with the CPU oracle.

Run after __graft_entry__.build() has copied the fixtures (oracle/fixtures.py):  python tests/golden/make_golden.py
The reference (nightly Rust) is not built here; these vectors are outputs of the
oracle, which is itself pinned by the reference's KATs and golden strings (tests/test_oracle_*).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.conftest import find_fixture  # noqa: E402
from tests.test_oracle_golden_text import CASES, run_oracle  # noqa: E402

STEPS = np.array([0, 1, 5, 10])

for fname, text, ids in CASES:
    path = find_fixture(fname)
    assert path, fname
    gm, tok, prompt_ids, out, logits, dev = run_oracle(path, debug=True)
    assert out == ids
    taps = {k.replace(":", "_"): v for k, v in dev.debug_tensors.items()
            if k in ("attn_rmsnorm:0:0", "x_debug:0:0", "attn_out:0:0", "ffn_out:0:0", "ffn_out:5:9", "final_rmsnorm:9")}
    np.savez_compressed(os.path.join(HERE, fname.replace(".gguf", "_logits.npz")),
                        prompt_ids=np.array(prompt_ids), generated_ids=np.array(out), steps=STEPS,
                        logits=np.stack(logits)[STEPS], **taps)
    print(fname, "ok", {k: v.shape for k, v in taps.items()})
