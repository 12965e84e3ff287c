"""Wall time and per-kernel CUDA-event times of one localBA configuration.
    python scripts/ba_profile.py NCAM NPTS NOBS [reps]"""
import json, os, sys, time
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np
from ov2slam_b200 import api, synth
ncam, npts, nobs = (int(a) for a in sys.argv[1:4])
reps = int(sys.argv[4]) if len(sys.argv) > 4 else 5
pb0 = synth.make_ba_problem(5, ncam, npts, nobs)
clone = lambda d: {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in d.items()}
ctx = api.Context(0)
opt = api.Optimizer(ctx)
res, _ = opt.local_ba(clone(pb0))
pbs = [clone(pb0) for _ in range(reps)]
ctx.sync(); t0 = time.perf_counter()
for p in pbs:
    res, _ = opt.local_ba(p)
ctx.sync(); wall = (time.perf_counter() - t0) / reps
ctx.profile(True)
for p in [clone(pb0) for _ in range(reps)]:
    opt.local_ba(p)
rep = ctx.profile_report(); ctx.profile(False)
print(json.dumps({"config": f"{ncam} KF x {npts} pts x {nobs} obs", "wall_ms_per_solve": 1e3 * wall, "lm_iterations": res["iters_robust"] + res["iters_refine"],
                  "final_cost": res["final_cost"],
                  "kernel_ms_per_solve": {k: round(v[0] / reps, 4) for k, v in rep.items()},
                  "launches_per_solve": {k: v[1] / reps for k, v in rep.items()}}))
