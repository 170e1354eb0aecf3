"""Copies the upstream crabml test models (GGUF, 14-27 MB each, too large to commit) into oracle/_ref/testdata, which git ignores.

The upstream checkout is found at $CRABML_REFERENCE, next to this repository (../reference), or at /root/reference, its
default location.  Tests look for the models only under oracle/_ref/testdata; the built tree carries them to
wherever the tests run, including machines without the upstream checkout."""
from __future__ import annotations

import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref", "testdata")
FIXTURES = ["tinyllamas-stories-15m-q8_0.gguf", "tinyllamas-stories-15m-q4_0.gguf"]


def reference_testdata():
    for d in (os.environ.get("CRABML_REFERENCE"), os.path.join(os.path.dirname(ROOT), "reference"), "/root/reference"):
        if d and os.access(os.path.join(d, "testdata"), os.R_OK | os.X_OK):
            return os.path.join(d, "testdata")
    return None


def copy_fixtures() -> list[str]:
    """-> the fixtures present under oracle/_ref/testdata afterwards."""
    src = reference_testdata()
    if src:
        os.makedirs(DST, exist_ok=True)
        for f in FIXTURES:
            s, d = os.path.join(src, f), os.path.join(DST, f)
            if os.path.exists(s) and (not os.path.exists(d) or os.path.getsize(d) != os.path.getsize(s)):
                shutil.copyfile(s, d)
    return [f for f in FIXTURES if os.path.exists(os.path.join(DST, f))]
