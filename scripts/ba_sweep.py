"""C3 / C5 solve rate of the persistent local-BA kernel vs the number of CTAs per window (OV2_BA_CTAS), single solves and
batches.  Prints one JSON line per configuration."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from ov2slam_b200 import api, synth  # noqa: E402

ctx = api.Context(0)
opt = api.Optimizer(ctx)
clone = lambda d: {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in d.items()}


def rate(pb, reps):
    for _ in range(3):
        opt.local_ba(clone(pb))
    pbs = [clone(pb) for _ in range(reps)]
    ctx.sync()
    t0 = time.perf_counter()
    for p in pbs:
        r, _ = opt.local_ba(p)
    ctx.sync()
    return reps / (time.perf_counter() - t0), r


c3 = synth.make_ba_problem(3, 10, 2000, 8000)
c5 = synth.make_ba_problem(5, 50, 20000, 150000)
for name, pb, reps, ctas_list in (("C3", c3, 40, ["1", "4", "8", "16", "32", "64", "96", "148", None]), ("C5", c5, 5, ["32", "74", "148", None])):
    for ctas in ctas_list:
        if ctas is None:
            os.environ.pop("OV2_BA_CTAS", None)
        else:
            os.environ["OV2_BA_CTAS"] = ctas
        try:
            v, r = rate(pb, reps)
            print(json.dumps({"window": name, "ctas": ctas, "solves_per_s": round(v, 1), "ms": round(1e3 / v, 4),
                              "iters": [r["iters_robust"], r["iters_refine"]], "final_cost": r["final_cost"]}), flush=True)
        except Exception as e:
            print(json.dumps({"window": name, "ctas": ctas, "error": str(e)[:200]}), flush=True)
base = [synth.make_ba_problem(100 + i, 10, 2000, 8000) for i in range(8)]
for K in (16, 64, 128, 256):
    for ctas in ("1", "2", "4", "8", None):
        if ctas is None:
            os.environ.pop("OV2_BA_CTAS", None)
        else:
            os.environ["OV2_BA_CTAS"] = ctas
        try:
            mk = lambda: [clone(base[i % 8]) for i in range(K)]
            api.local_ba_batch(ctx, mk())
            sets = [mk() for _ in range(3)]
            ctx.sync()
            t0 = time.perf_counter()
            for st in sets:
                api.local_ba_batch(ctx, st)
            ctx.sync()
            dt = time.perf_counter() - t0
            print(json.dumps({"batch": K, "ctas": ctas, "solves_per_s": round(3 * K / dt, 1), "ms_per_launch": round(1e3 * dt / 3, 3)}), flush=True)
        except Exception as e:
            print(json.dumps({"batch": K, "ctas": ctas, "error": str(e)[:200]}), flush=True)
