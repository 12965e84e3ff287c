"""Per-phase device time of the persistent local-BA kernel (OV2_BA_TRACE=1 prints one line per solve on stderr, with the
plan, Schur mode included, that each window's shape selects) at several group sizes."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
os.environ["OV2_BA_TRACE"] = "1"
from ov2slam_b200 import api, synth  # noqa: E402

ctx = api.Context(0)
opt = api.Optimizer(ctx)
clone = lambda d: {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in d.items()}
c3 = synth.make_ba_problem(3, 10, 2000, 8000)
c5 = synth.make_ba_problem(5, 50, 20000, 150000)
for name, pb, gs in (("C3", c3, ("16", "32", "64", "148")), ("C5", c5, ("296",))):
    for g in gs:
        os.environ["OV2_BA_CTAS"] = g
        for _ in range(3):
            print(name, "ctas", g, file=sys.stderr, flush=True)
            opt.local_ba(clone(pb))
