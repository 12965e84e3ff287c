import sys, os; sys.path.insert(0, '.')
import numpy as np
from ov2slam_b200 import api, synth
from oracle import ba_ref as B
ctx = api.Context(0)
pb0 = synth.make_ba_problem(41, 8, 400, 1600, stereo=True)
for keep_types in ((0, 1), (0, 2), (0,), (0, 1, 2)):
    sel = np.isin(pb0["obs_type"], keep_types)
    pb = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in pb0.items()}
    for k in ("obs_cam", "obs_lm", "obs_px", "obs_type"):
        pb[k] = np.ascontiguousarray(pb0[k][sel])
    ref = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in pb.items()}
    log = []
    r = B.local_ba(ref, log=log, max_iters_robust=1, apply_l2_after_robust=False)
    gpu = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in pb.items()}
    g, flags = api.Optimizer(ctx).local_ba(gpu, max_iters_robust=1, apply_l2_after_robust=0)
    print(keep_types, 'ref cand %.8f mcc %.8f' % (log[0]['cand_cost'], log[0]['mcc']), 'pose diff', np.abs(gpu['pose'] - ref['pose']).max(), 'invd', np.abs(gpu['lm_invdepth'] - ref['lm_invdepth']).max())
