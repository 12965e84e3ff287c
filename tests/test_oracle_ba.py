"""CPU tests pinning the BA oracle (oracle/ba_ref.py) piecewise: Ceres' own known answers for the
Huber loss / corrector / LM radius rules, numeric differentiation of the analytic Jacobians, a
dense solve of the full normal equations against the Schur path, and ground-truth recovery."""
import numpy as np
import pytest

from oracle import ba_ref as B
from ov2slam_b200 import synth


def test_huber_known_answers():
    """loss_function_test.cc:92-103 (HuberLoss values both sides of the knee), closed form."""
    for a in (0.7, 1.3):
        for s in (0.357, 1.792, 0.3, a * a, 5.0):
            rho = B.huber(s, a)
            if s <= a * a:
                assert rho[0] == s and rho[1] == 1.0 and rho[2] == 0.0
            else:
                r = np.sqrt(s)
                assert np.isclose(rho[0], 2 * a * r - a * a, rtol=0, atol=1e-15)
                assert np.isclose(rho[1], a / r) and np.isclose(rho[2], -a / (2 * r * s))
            # numeric derivative of rho (loss_function_test.cc AssertLossFunctionIsValid)
            h = 1e-6
            fd1 = (B.huber(s + h, a)[0] - B.huber(s - h, a)[0]) / (2 * h)
            if abs(s - a * a) > 1e-3:
                assert abs(fd1 - rho[1]) < 1e-6


def test_corrector_known_answers():
    """corrector_test.cc:57-135 scalar cases."""
    # ScalarCorrection: sq_norm 3+4, rho = {sq_norm/2, 0.5, 0.0} (zero second derivative)
    sq = 3.0 + 4.0
    sr, rs, al = B.corrector(sq, [sq / 2.0, 0.5, 0.0])
    assert np.isclose(rs, np.sqrt(0.5)) and al == 0.0
    # ScalarCorrectionZeroResidual / negative second derivative -> alpha 0, pure sqrt(rho') scaling
    sr, rs, al = B.corrector(0.0, [0.0, 0.5, 0.25])
    assert al == 0.0 and np.isclose(rs, np.sqrt(0.5))
    sr, rs, al = B.corrector(sq, [1.0, 0.5, -0.1])
    assert al == 0.0 and np.isclose(rs, np.sqrt(0.5))
    # ScalarCorrectionAlphaClamped-style positive rho'': general branch formula
    rho = [1.0, 2.0, 0.05]
    D = 1 + 2 * sq * rho[2] / rho[1]
    alpha = 1 - np.sqrt(D)
    sr, rs, al = B.corrector(sq, rho)
    assert np.isclose(rs, np.sqrt(2.0) / (1 - alpha)) and np.isclose(al, alpha / sq)
    # Huber never reaches the general branch
    for s in (0.1, 3.0, 50.0):
        rho = B.huber(s, 1.5)
        assert B.corrector(s, rho)[2] == 0.0


def test_lm_radius_rules():
    """levenberg_marquardt_strategy_test.cc TrustRegionStepBounds: rejected steps halve, quarter,
    ... the radius; an accepted step with quality 0.75 divides by max(1/3, 1-(2q-1)^3) and resets."""
    r, f = 2.0, 2.0
    r, f = B.lm_step_rejected(r, f)
    assert (r, f) == (1.0, 4.0)
    r, f = B.lm_step_rejected(r, f)
    assert (r, f) == (0.25, 8.0)
    r = B.lm_step_accepted(0.25, 0.75)
    assert np.isclose(r, 0.25 / (1 - 0.5 ** 3))
    assert np.isclose(B.lm_step_accepted(1.0, 1.0), 3.0)           # clamp at 1/3
    assert B.lm_step_accepted(1e16, 1.0) == 1e16                   # max_radius
    assert np.isclose(B.lm_step_accepted(1.0, 0.25), 1.0 / (1 - (-0.5) ** 3))


def test_se3_exp_group_identities():
    rng = np.random.default_rng(0)
    d = rng.normal(0, 0.3, (20, 6))
    t, q = B.se3_exp(d)
    assert np.allclose(np.linalg.norm(q, axis=1), 1.0)
    # exp(d) * exp(-d) = identity
    p = np.concatenate([t, q], -1)
    back = B.pose_plus(p, -d)
    assert np.allclose(back[:, :3], 0, atol=1e-12) and np.allclose(np.abs(back[:, 6]), 1, atol=1e-12)
    # small-angle branch is continuous with the closed form
    dsm = np.array([[0.1, -0.2, 0.3, 1e-11, -2e-11, 1e-11]])
    t2, q2 = B.se3_exp(dsm)
    assert np.allclose(t2[0], dsm[0, :3], atol=1e-10)


def test_jacobians_vs_central_differences():
    pb = synth.make_ba_problem(1, 6, 120, 480)
    pose, invd = pb["pose"].copy(), pb["lm_invdepth"].copy()
    idx = np.arange(0, 480, 7)
    ev = B.evaluate(pb, pose, invd, idx, True)
    h = 1e-6
    for which, J in (("a", ev["Ja"]), ("o", ev["Jo"])):
        num = np.zeros_like(J)
        cams = ev["ca"] if which == "a" else ev["co"]
        for k in range(6):
            d = np.zeros(6)
            d[k] = h
            rp = np.zeros((len(idx), 2))
            rm = np.zeros((len(idx), 2))
            for j, (i, c) in enumerate(zip(idx, cams)):
                pp = pose.copy()
                pp[c] = B.pose_plus(pose[c][None], d[None])[0]
                rp[j] = B.evaluate(pb, pp, invd, np.array([i]), False)["r"][0]
                pm = pose.copy()
                pm[c] = B.pose_plus(pose[c][None], -d[None])[0]
                rm[j] = B.evaluate(pb, pm, invd, np.array([i]), False)["r"][0]
            num[:, :, k] = (rp - rm) / (2 * h)
        assert np.abs(num - J).max() <= 1e-5 * max(1.0, np.abs(J).max()), which
    num = np.zeros_like(ev["Jl"])
    for j, i in enumerate(idx):
        l = pb["obs_lm"][i]
        hh = 1e-7
        ip, im = invd.copy(), invd.copy()
        ip[l] += hh
        im[l] -= hh
        num[j] = (B.evaluate(pb, pose, ip, np.array([i]), False)["r"][0] -
                  B.evaluate(pb, pose, im, np.array([i]), False)["r"][0]) / (2 * hh)
    assert np.abs(num - ev["Jl"]).max() <= 1e-5 * max(1.0, np.abs(ev["Jl"]).max())


def test_schur_step_equals_dense_normal_equations():
    pb = synth.make_ba_problem(2, 5, 60, 240)
    log = []
    B.ceres_solve(pb, pb["pose"], pb["lm_invdepth"], np.ones(240, bool), 1, float(np.sqrt(np.float32(5.9915))), log=log)
    step = [e for e in log if not e.get("ctl")][0]["step"]
    # rebuild the same LM system densely
    idx = np.arange(240)
    ev = B.evaluate(pb, pb["pose"], pb["lm_invdepth"], idx, True)
    w = np.sqrt(B.huber(ev["chi2"], float(np.sqrt(np.float32(5.9915))))[1])
    const = pb["pose_const"].astype(bool)
    cams = np.nonzero(~const)[0]
    slot = {c: k for k, c in enumerate(cams)}
    ncv, nl = len(cams), 60
    J = np.zeros((480, ncv * 6 + nl))
    r = (ev["r"] * w[:, None]).reshape(-1)
    for n in range(240):
        for c, Jb in ((ev["ca"][n], ev["Ja"][n]), (ev["co"][n], ev["Jo"][n])):
            if c in slot:
                J[2 * n:2 * n + 2, 6 * slot[c]:6 * slot[c] + 6] += Jb * w[n]
        J[2 * n:2 * n + 2, ncv * 6 + ev["lm"][n]] = ev["Jl"][n] * w[n]
    scale = 1.0 / (1.0 + np.sqrt((J * J).sum(0)))
    Js = J * scale
    diag = np.clip((Js * Js).sum(0), 1e-6, 1e32)
    A = Js.T @ Js + np.diag(diag / 1e4)
    y = np.linalg.solve(A, Js.T @ r)
    dense_step = -y * scale
    assert np.abs(dense_step - step).max() <= 1e-9 * max(1.0, np.abs(step).max())


def test_noise_free_recovery_and_monotone_cost():
    pb = synth.make_ba_problem(3, 8, 300, 1500, outlier_frac=0.0, px_noise=0.0)
    res = B.local_ba(pb, max_iters_robust=30, function_tolerance=1e-12)
    tr = res["summaries"][0]["trace"]
    costs = [t["cost"] for t in tr if t["ok"]]
    assert all(b <= a + 1e-12 for a, b in zip(costs, costs[1:]))
    assert res["final_cost"] < 1e-3 * res["summaries"][0]["initial_cost"]
    # the scale gauge is fixed by the two constant cameras: poses come back to truth
    assert np.abs(pb["pose"][:, :3] - pb["truth_pose"][:, :3]).max() < 2e-3


def test_outlier_flags_and_two_stage():
    pb = synth.make_ba_problem(4, 10, 400, 1600)
    res = B.local_ba(pb)
    assert res["iters_robust"] <= 5 and res["iters_refine"] <= 10
    assert res["n_outliers_first"] > 20            # 5 % gross outliers were injected
    assert (res["flags"] & 1).sum() == res["n_outliers_first"]
    assert res["n_outliers_second"] <= res["n_outliers_first"]


def test_unused_and_constant_blocks_drop_out():
    pb = synth.make_ba_problem(5, 6, 100, 300)
    pb["pose_const"][:] = 1                          # every pose constant: only inverse depths move
    p0 = pb["pose"].copy()
    res = B.local_ba(pb)
    assert np.array_equal(pb["pose"], p0)
    assert res["final_cost"] <= res["summaries"][0]["initial_cost"]


def _c_port_window(name):
    if name in ("unused_keyframes", "keyframe_leaves_refinement", "landmarks_without_residuals"):
        import ba_windows
        return ba_windows.small_shrinking_windows()[name]
    return synth.make_ba_problem(*[int(v) for v in name.split("-")])


@pytest.mark.parametrize("window", ["3-10-2000-8000", "11-6-300-1200", "5-6-100-300",
                                    "unused_keyframes", "keyframe_leaves_refinement", "landmarks_without_residuals"])
def test_c_port_matches_numpy_oracle(window):
    """oracle/ba_ref_c.c (the single-threaded CPU baseline bench.py times) == oracle/ba_ref.py, also on windows whose
    program is smaller than the declared one (tests/ba_windows.py; the C restatement is mono only)."""
    from oracle import ba_ref_c
    pb = _c_port_window(window)
    a = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in pb.items()}
    b = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in pb.items()}
    ra = B.local_ba(a)
    rb = ba_ref_c.local_ba(b)
    for k in ("iters_robust", "iters_refine", "n_outliers_first", "n_outliers_second", "termination"):
        assert ra[k] == rb[k], k
    assert abs(ra["final_cost"] - rb["final_cost"]) <= 1e-9 * max(1.0, ra["final_cost"])
    assert np.abs(a["pose"] - b["pose"]).max() <= 1e-9
    assert np.abs(a["lm_invdepth"] - b["lm_invdepth"]).max() <= 1e-9
    assert np.array_equal(ra["flags"], rb["flags"])


def test_stereo_jacobians_vs_central_differences():
    """The two right-camera residual blocks (ceres_parametrization.cpp:476-577, :579-712)."""
    pb = synth.make_ba_problem(2, 5, 60, 200, stereo=True)
    pose, invd = pb["pose"].copy(), pb["lm_invdepth"].copy()
    idx = np.arange(0, len(pb["obs_cam"]), 3)
    ev = B.evaluate(pb, pose, invd, idx, True)
    assert set(ev["typ"].tolist()) == {0, 1, 2}
    h = 1e-6
    for which, J, cams in (("a", ev["Ja"], ev["ca"]), ("o", ev["Jo"], ev["co"])):
        num = np.zeros_like(J)
        for k in range(6):
            d = np.zeros(6)
            d[k] = h
            for j, (i, c) in enumerate(zip(idx, cams)):
                if ev["typ"][j] == 2:
                    continue       # no pose dependence by construction (the pose is not a parameter block)
                pp, pm = pose.copy(), pose.copy()
                pp[c] = B.pose_plus(pose[c][None], d[None])[0]
                pm[c] = B.pose_plus(pose[c][None], -d[None])[0]
                num[j, :, k] = (B.evaluate(pb, pp, invd, np.array([i]), False)["r"][0] -
                                B.evaluate(pb, pm, invd, np.array([i]), False)["r"][0]) / (2 * h)
        assert np.abs(num - J).max() <= 1e-5 * max(1.0, np.abs(J).max()), which
    num = np.zeros_like(ev["Jl"])
    for j, i in enumerate(idx):
        l = pb["obs_lm"][i]
        ip, im = invd.copy(), invd.copy()
        ip[l] += 1e-7
        im[l] -= 1e-7
        num[j] = (B.evaluate(pb, pose, ip, np.array([i]), False)["r"][0] -
                  B.evaluate(pb, pose, im, np.array([i]), False)["r"][0]) / 2e-7
    assert np.abs(num - ev["Jl"]).max() <= 1e-5 * max(1.0, np.abs(ev["Jl"]).max())


def test_stereo_window_converges_and_refines_with_trivial_loss():
    pb = synth.make_ba_problem(9, 8, 300, 1200, stereo=True)
    res = B.local_ba(pb)
    assert res["final_cost"] > 0 and res["n_outliers_first"] > 20
    pb2 = synth.make_ba_problem(9, 8, 300, 1200, stereo=True, outlier_frac=0.0, px_noise=0.0)
    r2 = B.local_ba(pb2, max_iters_robust=30, function_tolerance=1e-12)
    assert np.abs(pb2["pose"][:, :3] - pb2["truth_pose"][:, :3]).max() < 2e-3
    assert np.abs(pb2["lm_invdepth"] - pb2["truth_invdepth"]).max() < 5e-3


def test_oracles_agree_and_converge_on_the_bal_structure_fixture():
    """The observation graph / geometry of Ceres' own bundle-adjustment test problem (problem-16-22106-pre.txt, converted by
    scripts/make_bal_fixture.py; measurements re-synthesised through OV2SLAM's residual, tests/ba_fixture.py): track lengths
    2 .. 14 and an uneven covisibility pattern that the synthetic generator does not produce.  The numpy restatement and the C
    restatement take the same LM decisions on a 2 000-landmark subset, and the full window (22 106 landmarks, 61 612 residual
    blocks) converges: cost down, keyframe positions 20x closer to the ground truth."""
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).parent))
    import ba_fixture as F
    from oracle import ba_ref_c
    clone = lambda d: {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in d.items()}
    small = F.bal_window(seed=1, max_pts=2000)
    a, b = clone(small), clone(small)
    ra = B.local_ba(a)
    rb = ba_ref_c.local_ba(b)
    assert (ra["iters_robust"], ra["iters_refine"], ra["termination"]) == (rb["iters_robust"], rb["iters_refine"], rb["termination"])
    assert abs(ra["final_cost"] - rb["final_cost"]) <= 1e-9 * ra["final_cost"]
    assert np.abs(a["pose"] - b["pose"]).max() <= 1e-8 and np.abs(a["lm_invdepth"] - b["lm_invdepth"]).max() <= 1e-8
    assert np.array_equal(ra["flags"], rb["flags"])
    full = F.bal_window(seed=0)
    c = clone(full)
    rc = ba_ref_c.local_ba(c)
    assert rc["final_cost"] < rc["initial_cost"] and rc["n_outliers_first"] > 2000
    e0 = np.abs(full["pose"][:, :3] - full["truth_pose"][:, :3]).max()
    e1 = np.abs(c["pose"][:, :3] - full["truth_pose"][:, :3]).max()
    assert e1 < e0 / 20
