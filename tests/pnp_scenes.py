"""Pose problems for MultiViewGeometry::ceresPnP (oracle/pnp_ref.py, csrc/pnp_math.cuh, csrc/pnp_solver.cu), and the near-tie guard.

A scene is one seeded draw: a camera pose, points in front of it projected through a shipped calibration (rounded to float, as the
reference passes fx, fy, cx, cy), pixel noise, optional gross outliers, points mirrored behind the camera, per-keypoint pyramid
levels and a start pose.  A point mirrored through the camera centre projects to the same pixel as the original, so its residual
is small and only the depth test rejects it.

The device solve forms the normal equations with FMA contraction and another summation order than the oracle's QR, so a decision
that sits on its edge may go either way.  `margin` measures, from the oracle's decision log, how far every decision of a solve lies
from its threshold; `draw` redraws a scene from the next seed until that margin is at least MIN_MARGIN, and checks that the
redrawn scene still has the property the case is about."""
from __future__ import annotations

import numpy as np

from oracle import ba_ref as B
from oracle import pnp_ref as P

# fx fy cx cy of the shipped configurations (parameters_files/*/euroc/euroc_*.yaml, */kitti/kitti_*.yaml)
CALIBS = {
    "euroc_left": (458.654, 457.296, 367.215, 248.375),
    "euroc_right": (457.587, 456.134, 379.999, 255.238),
    "kitti_00-02": (718.856, 718.856, 607.1928, 185.2157),
    "kitti_03": (721.5377, 721.5377, 609.5593, 172.854),
    "kitti_04-12": (707.0912, 707.0912, 601.8873, 183.1104),
}
CALIB_K = {k: np.array(v, np.float32).astype(np.float64) for k, v in CALIBS.items()}
CHI2TH = (3.2189, 5.9915, 9.2103)           # the 20 %, 5 % and 1 % values of the shipped robust_mono_th comment
MIN_MARGIN = 1e-6


def make(seed, n, calib="euroc_left", noise=0.6, nout=0, behind=0, far=False, scales=False, start="near", quat="unit", spread=1.0):
    """One problem.  far: KITTI-scale geometry (|t| = 500 m, points 500 to 1 000 m away).  start: "near" (a perturbed truth) or
    "optimum" (the truth itself, noise-free pixels).  quat: "unit", "wneg" (the same rotation with w < 0) or "nonunit" (the start's
    quaternion scaled by 1.7).  behind: that many points mirrored behind the camera (n: all of them).  scales: False (none), True
    (pyramid levels 0 to 3 drawn per point, pixel noise scaled by 2^level) or one level for every point.  spread scales the
    start's offset from the truth (5 cm and 0.02 rad; 50 cm at KITTI scale)."""
    rng = np.random.default_rng(seed)
    K = CALIB_K[calib]
    axis = rng.standard_normal(3)
    axis /= np.linalg.norm(axis)
    ang = 0.6 * rng.random()
    q = np.concatenate([axis * np.sin(ang / 2), [np.cos(ang / 2)]])
    t = rng.normal(0, 0.5, 3)
    if far:
        t = 500.0 * t / np.linalg.norm(t)
    z = rng.uniform(500, 1000, n) if far else rng.uniform(2, 10, n)
    pc = np.stack([rng.uniform(-0.7, 0.7, n) * z, rng.uniform(-0.4, 0.4, n) * z, z], 1)
    px = np.stack([K[0] * pc[:, 0] / pc[:, 2] + K[2], K[1] * pc[:, 1] / pc[:, 2] + K[3]], 1)
    sc = None if scales is False else rng.integers(0, 4, n).astype(np.int32) if scales is True else np.full(n, scales, np.int32)
    if start != "optimum":
        px += rng.normal(0, noise, (n, 2)) * (1 if sc is None else np.power(2.0, sc)[:, None])
    out = rng.choice(n, min(nout, n), replace=False)
    px[out] += rng.uniform(15, 60, (len(out), 2)) * rng.choice([-1, 1], (len(out), 2))
    back = rng.choice(n, min(behind, n), replace=False)
    pc[back] *= -1.0
    w = pc @ B.quat_to_rot(q).T + t
    truth = np.concatenate([t, q])
    if start == "optimum":
        T0 = truth.copy()
    else:
        s = 10.0 if far else 1.0
        T0 = B.pose_plus(truth, spread * np.concatenate([rng.normal(0, 0.05 * s, 3), rng.normal(0, 0.02, 3)]))
    if quat == "wneg":
        T0[3:] = -T0[3:]
    elif quat == "nonunit":
        T0[3:] *= 1.7
    return dict(px=np.ascontiguousarray(px), w=np.ascontiguousarray(w), scales=sc, K=K, T0=T0, n=n)


def unit_start(sc):
    """The start as Sophus stores it: SE3d(q, t) keeps a unit quaternion.  The kernel normalises the start it is given; the oracle
    is run on the normalised start (Ceres, given a unit quaternion, never sees another)."""
    T = sc["T0"].copy()
    T[3:] = B.quat_normalize(T[3:])
    return T


def solve(sc, nmaxiter=5, chi2th=5.9915, use_robust=True, apply_l2=True):
    """The oracle on one scene: (success, pose, outlier indices, info) of pnp_ref.ceres_pnp(..., summary=True)."""
    return P.ceres_pnp(sc["px"], sc["w"], unit_start(sc), sc["K"], nmaxiter=nmaxiter, chi2th=chi2th, use_robust=use_robust,
                       apply_l2_after_robust=apply_l2, scales=sc["scales"], summary=True)


def _rel(v, th):
    return abs(v - th) / max(abs(v), abs(th), 1e-300)


def margin(info):
    """The smallest relative distance of any decision the oracle took to its threshold: the outlier scan (chi2 against chi2th),
    and per solve the gradient test (gmax against 1e-10), the step-norm test, the function-tolerance test (|delta cost| against
    1e-3 cost) and the step acceptance (rho against 1e-3)."""
    m = min((_rel(c, info["chi2th"]) for c in info["chi2"]), default=1.0)
    for log in info["log"]:
        for e in log:
            if "gmax" in e:
                m = min(m, _rel(e["gmax"], 1e-10))
            elif e["valid"]:
                m = min(m, _rel(e["step_norm"], 1e-8 * (e["xnorm"] + 1e-8)), _rel(abs(e["x_cost"] - e["cand_cost"]), 1e-3 * e["x_cost"]))
                if e["rho"] is not None:
                    m = min(m, _rel(e["rho"], 1e-3))
    return m


def draw(seed, keep=None, opts=None, **kw):
    """make(seed, **kw), redrawn from seed + 1000, seed + 2000 ... while the oracle's margin is below MIN_MARGIN.  keep(result) must hold
    for the scene that is kept (the property the case is about).  Returns (scene, oracle result, number of redraws)."""
    opts = opts or {}
    for k in range(50):
        sc = make(seed + 1000 * k, **kw)
        res = solve(sc, **opts)
        if margin(res[3]) >= MIN_MARGIN:
            assert keep is None or keep(res), (seed, kw, opts)
            return sc, res, k
    raise AssertionError(f"no scene with a decision margin of {MIN_MARGIN} in 50 draws: {kw} {opts}")
