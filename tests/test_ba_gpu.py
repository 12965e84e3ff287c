"""GPU parity tests of ov2_localba_solve (through the C ABI) vs the float64 oracle (oracle/ba_ref.py).

Tolerance policy (SURVEY.md 8c): summation order differs (fp64 atomics vs numpy), so compare at
matched LM decisions: iteration counts and termination equal, costs within 1e-9 relative, final
poses / inverse depths within 1e-7 relative, outlier flag sets identical except observations whose
chi2 lies within 1e-6 of the 5.9915 threshold."""
import numpy as np
import pytest

from ov2slam_b200 import api, synth
from oracle import ba_ref as B

pytestmark = pytest.mark.gpu


def _clone(pb):
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in pb.items()}


def _check(ctx, pb, **opts):
    ref = _clone(pb)
    rres = B.local_ba(ref, **{k: v for k, v in opts.items()})
    gpu = _clone(pb)
    gopts = {k: (int(v) if isinstance(v, bool) else v) for k, v in opts.items()}
    if "refine_trivial_loss" in gopts:
        gopts["refine_loss"] = gopts.pop("refine_trivial_loss")
    gres, flags = api.Optimizer(ctx).local_ba(gpu, **gopts)
    assert gres["iters_robust"] == rres["iters_robust"], (gres, {k: v for k, v in rres.items() if k not in ("flags", "summaries")})
    assert gres["iters_refine"] == rres["iters_refine"]
    term = {"CONVERGENCE": 0, "NO_CONVERGENCE": 1, "FAILURE": 2}[rres["termination"]]
    assert gres["termination"] == term
    assert abs(gres["initial_cost"] - rres["initial_cost"]) <= 1e-9 * max(1.0, abs(rres["initial_cost"]))
    assert abs(gres["final_cost"] - rres["final_cost"]) <= 1e-9 * max(1.0, abs(rres["final_cost"]))
    assert np.abs(gpu["pose"] - ref["pose"]).max() <= 1e-7 * max(1.0, np.abs(ref["pose"]).max())
    assert np.abs(gpu["lm_invdepth"] - ref["lm_invdepth"]).max() <= 1e-7 * max(1.0, np.abs(ref["lm_invdepth"]).max())
    diff = np.nonzero(flags != rres["flags"])[0]
    assert len(diff) <= 2, len(diff)      # only threshold-borderline observations may differ
    assert gres["n_outliers_first"] == rres["n_outliers_first"] or len(diff) > 0
    return gres, rres


@pytest.mark.parametrize("seed,ncam,npts,nobs", [(3, 10, 2000, 8000), (11, 6, 300, 1200), (12, 20, 1500, 9000)])
def test_localba_matches_oracle(ctx, seed, ncam, npts, nobs):
    pb = synth.make_ba_problem(seed, ncam, npts, nobs)
    g, r = _check(ctx, pb)
    assert g["final_cost"] < g["initial_cost"] or g["iters_refine"] > 0


def test_localba_no_robust_and_single_stage(ctx):
    pb = synth.make_ba_problem(21, 8, 500, 2500, outlier_frac=0.0)
    _check(ctx, pb, use_robust=False)
    _check(ctx, pb, apply_l2_after_robust=False)


def test_localba_more_iterations_noise_free_recovers_truth(ctx):
    pb = synth.make_ba_problem(3, 8, 300, 1500, outlier_frac=0.0, px_noise=0.0)
    g, r = _check(ctx, pb, max_iters_robust=30, function_tolerance=1e-12)
    gpu = _clone(pb)
    api.Optimizer(ctx).local_ba(gpu, max_iters_robust=30, function_tolerance=1e-12)
    assert np.abs(gpu["pose"][:, :3] - pb["truth_pose"][:, :3]).max() < 2e-3


def test_localba_all_poses_constant(ctx):
    pb = synth.make_ba_problem(5, 6, 100, 300)
    pb["pose_const"][:] = 1
    p0 = pb["pose"].copy()
    gpu = _clone(pb)
    res, _ = api.Optimizer(ctx).local_ba(gpu)
    assert np.array_equal(gpu["pose"], p0)
    _check(ctx, pb)


def test_localba_rejects_unsorted_observations(ctx):
    pb = synth.make_ba_problem(6, 5, 50, 150)
    pb["obs_lm"] = pb["obs_lm"][::-1].copy()
    with pytest.raises(api.Ov2Error):
        api.Optimizer(ctx).local_ba(pb)


@pytest.mark.parametrize("seed,ncam,npts,nobs", [(41, 8, 400, 1600), (42, 10, 1000, 4000)])
def test_localba_stereo_window_matches_oracle(ctx, seed, ncam, npts, nobs):
    """Stereo windows: left + right-camera residual blocks (ceres_parametrization.cpp:361-712), the
    refinement drops to the trivial loss as optimizer.cpp:606-608 decides."""
    pb = synth.make_ba_problem(seed, ncam, npts, nobs, stereo=True)
    assert set(pb["obs_type"].tolist()) == {0, 1, 2}
    g, r = _check(ctx, pb)
    assert g["n_outliers_first"] > 0


def test_localba_stereo_noise_free_recovers_truth(ctx):
    pb = synth.make_ba_problem(43, 8, 300, 1200, stereo=True, outlier_frac=0.0, px_noise=0.0)
    gpu = _clone(pb)
    api.Optimizer(ctx).local_ba(gpu, max_iters_robust=30, function_tolerance=1e-12)
    assert np.abs(gpu["pose"][:, :3] - pb["truth_pose"][:, :3]).max() < 2e-3
    assert np.abs(gpu["lm_invdepth"] - pb["truth_invdepth"]).max() < 5e-3


def test_localba_refine_loss_override(ctx):
    pb = synth.make_ba_problem(44, 8, 400, 1600)
    _check(ctx, pb, refine_trivial_loss=True)


def _check_oracle(ctx, pb, oracle=None):
    """Against the C restatement of the oracle (oracle/ba_ref_c.c, itself pinned to oracle/ba_ref.py; mono windows only) or
    the given oracle module: same LM decisions, cost 1e-8, states 1e-6, flags equal up to threshold-borderline observations."""
    if oracle is None:
        from oracle import ba_ref_c as oracle
    ref = _clone(pb)
    r = oracle.local_ba(ref)
    gpu = _clone(pb)
    g, flags = api.Optimizer(ctx).local_ba(gpu)
    assert (g["iters_robust"], g["iters_refine"]) == (r["iters_robust"], r["iters_refine"])
    assert abs(g["final_cost"] - r["final_cost"]) <= 1e-8 * max(1.0, r["final_cost"])
    assert np.abs(gpu["pose"] - ref["pose"]).max() <= 1e-6
    assert np.abs(gpu["lm_invdepth"] - ref["lm_invdepth"]).max() <= 1e-6
    assert (flags != r["flags"]).sum() <= 2


@pytest.mark.parametrize("ncam,npts,nobs", [(16, 1200, 7000), (22, 1500, 9000), (50, 4000, 30000)])
def test_localba_all_reduced_solver_paths(ctx, ncam, npts, nobs):
    """Reduced camera systems of 84, 120 and 288 unknowns: shared-memory Gauss-Jordan for n <= 96, blocked Cholesky with
    the FP64 tensor-core trailing update beyond."""
    _check_oracle(ctx, synth.make_ba_problem(70 + ncam, ncam, npts, nobs))


def _keyframe_table_in_shared_memory(ncam, ncv):
    """plan_window (csrc/ba_lm.cu) for n > 96: the keyframe table (12 doubles + 1 int per keyframe) stays in shared memory
    when it fits next to the larger of the Schur scratch and the blocked-Cholesky solve area in 200 KB."""
    warps, sch, ch_nb, n = 8, 8, 32, 6 * ncv
    assert n > 96
    tab = (100 * ncam + 15) & ~15
    schur = (warps * 6 * (ncv + 1) * 8 + (((warps * (ncv + 1) + 1) >> 1) << 3) + warps * 28 * sch * 8 + warps * sch * 4 + 16 + 15) & ~15
    solve = ch_nb * (((n + 15) & ~15) + 8) * 8
    return tab + max(schur, solve) + 16 <= 200 * 1024


@pytest.mark.parametrize("seed,ncam,npts,stereo,shared", [(81, 300, 1200, False, True), (84, 2000, 5000, False, False),
                                                          (83, 1200, 3000, True, False)])
def test_localba_windows_beyond_256_keyframes(ctx, seed, ncam, npts, stereo, shared):
    """Windows of more than 256 keyframes, the last 64 optimised (Optimizer::fullBA / looseBA put a whole map or keyframe
    range in one window; the oldest keyframes are held constant): the keyframe table stays in shared memory up to about a
    thousand keyframes and moves to one copy per CTA in global memory beyond.  Stereo is checked against the numpy oracle."""
    assert _keyframe_table_in_shared_memory(ncam, 64) == shared
    pb = synth.make_ba_problem(seed, ncam, npts, 2 * npts, nconst=ncam - 64, stereo=stereo)
    assert len(np.unique(np.concatenate([pb["obs_cam"], pb["lm_anchor_cam"]]))) == ncam   # every keyframe observes something
    _check_oracle(ctx, pb, B if stereo else None)       # the C restatement has no stereo residual blocks


def test_localba_c5_size_150k_observations(ctx):
    """BASELINE.json configs[4] size on one GPU: 50 KF x 20 000 landmarks x 150 000 observations (288 x 288 reduced
    system) against the C restatement of the oracle: same LM decisions, cost 1e-8, states 1e-6, flags equal up to
    threshold-borderline observations."""
    from oracle import ba_ref_c
    pb = synth.make_ba_problem(5, 50, 20000, 150000)
    ref = _clone(pb)
    r = ba_ref_c.local_ba(ref)
    gpu = _clone(pb)
    g, flags = api.Optimizer(ctx).local_ba(gpu)
    assert (g["iters_robust"], g["iters_refine"]) == (r["iters_robust"], r["iters_refine"])
    assert abs(g["final_cost"] - r["final_cost"]) <= 1e-8 * max(1.0, r["final_cost"])
    assert np.abs(gpu["pose"] - ref["pose"]).max() <= 1e-6
    assert np.abs(gpu["lm_invdepth"] - ref["lm_invdepth"]).max() <= 1e-6
    assert (flags != r["flags"]).sum() <= 4
    assert g["n_outliers_first"] > 5000


def test_localba_stereo_150k_blocks_matches_golden(ctx):
    """Stereo window with 150 000 residual blocks (all three residual types) against the committed result of the numpy
    oracle (tests/golden/ba_stereo_150k.npz, scripts/make_golden_ba.py; the oracle needs about a minute for it)."""
    from pathlib import Path
    g = np.load(Path(__file__).parent / "golden" / "ba_stereo_150k.npz")
    pb = synth.make_ba_problem(int(g["seed"]), int(g["ncam"]), int(g["npts"]), int(g["nobs"]), stereo=True)
    assert len(pb["obs_cam"]) == 150000
    res, flags = api.Optimizer(ctx).local_ba(pb)
    assert [res["iters_robust"], res["iters_refine"]] == g["iters"].tolist()
    assert res["termination"] == int(g["termination"][0])
    assert abs(res["final_cost"] - g["costs"][1]) <= 1e-8 * max(1.0, g["costs"][1])
    assert np.abs(pb["pose"] - g["pose"]).max() <= 1e-6
    assert np.abs(pb["lm_invdepth"] - g["lm_invdepth"]).max() <= 1e-6
    f1 = np.unpackbits(g["flags"])[:150000]
    assert ((flags & 1) != f1).sum() <= 4
    assert abs(res["n_outliers_first"] - int(g["n_outliers"][0])) <= 4


@pytest.mark.parametrize("ctas", ["1", "3", "40", None])
def test_localba_persistent_kernel_group_sizes(ctx, monkeypatch, ctas):
    """The persistent solve kernel with 1, 3, 40 CTAs per window and its own choice: the group barrier, the redundant
    controller and the phase split must give the same solve whatever the group size (mono and stereo windows)."""
    if ctas is None:
        monkeypatch.delenv("OV2_BA_CTAS", raising=False)
    else:
        monkeypatch.setenv("OV2_BA_CTAS", ctas)
    _check(ctx, synth.make_ba_problem(3, 10, 2000, 8000))
    _check(ctx, synth.make_ba_problem(41, 8, 400, 1600, stereo=True))


def test_localba_batch_equals_single_solves(ctx):
    """ov2_localba_solve_batch: windows of different sizes (mono, stereo, all poses constant, one tiny window) in one
    launch; every window equals its own single solve."""
    specs = [(3, 10, 2000, 8000, False), (11, 6, 300, 1200, False), (41, 8, 400, 1600, True), (12, 20, 1500, 9000, False),
             (5, 6, 100, 300, False), (44, 8, 400, 1600, False)] * 3
    pbs = [synth.make_ba_problem(s, c, p, o, stereo=st) for s, c, p, o, st in specs]
    pbs[4]["pose_const"][:] = 1
    singles = [_clone(pb) for pb in pbs]
    refs = [api.Optimizer(ctx).local_ba(pb) for pb in singles]
    batch = [_clone(pb) for pb in pbs]
    res, flags = api.local_ba_batch(ctx, batch)
    assert len(res) == len(pbs)
    for k in range(len(pbs)):
        r1, f1 = refs[k]
        assert (res[k]["iters_robust"], res[k]["iters_refine"], res[k]["termination"]) == (r1["iters_robust"], r1["iters_refine"], r1["termination"]), k
        assert abs(res[k]["final_cost"] - r1["final_cost"]) <= 1e-9 * max(1.0, r1["final_cost"])
        assert np.abs(batch[k]["pose"] - singles[k]["pose"]).max() <= 1e-8
        assert np.abs(batch[k]["lm_invdepth"] - singles[k]["lm_invdepth"]).max() <= 1e-8
        assert (flags[k] != f1).sum() <= 2


def test_localba_stop_request_skips_the_refinement(ctx):
    """Optimizer::signalStopLocalBA (optimizer.cpp:2334-2343): the flag is polled before solve #2 (optimizer.cpp:603-604)."""
    pb = synth.make_ba_problem(3, 10, 2000, 8000)
    a = _clone(pb)
    r0, _ = api.Optimizer(ctx).local_ba(a)
    assert r0["iters_refine"] > 0
    api.request_stop_local_ba(ctx, True)
    b = _clone(pb)
    r1, f1 = api.Optimizer(ctx).local_ba(b)
    assert r1["iters_refine"] == 0 and r1["iters_robust"] == r0["iters_robust"] and r1["n_outliers_first"] == r0["n_outliers_first"]
    ref = _clone(pb)
    rr = B.local_ba(ref, apply_l2_after_robust=False)
    assert np.abs(b["pose"] - ref["pose"]).max() <= 1e-7
    api.request_stop_local_ba(ctx, False)
    c = _clone(pb)
    r2, _ = api.Optimizer(ctx).local_ba(c)
    assert r2["iters_refine"] == r0["iters_refine"]


def test_localba_bal_structure_fixture(ctx):
    """GPU vs the C restatement on the window built from Ceres' BAL test problem's observation graph (tests/ba_fixture.py:
    16 keyframes, 22 106 landmarks with 2 .. 14 views, 61 612 residual blocks, 84 x 84 reduced system)."""
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).parent))
    import ba_fixture as F
    from oracle import ba_ref_c
    pb = F.bal_window(seed=0)
    ref = _clone(pb)
    r = ba_ref_c.local_ba(ref)
    gpu = _clone(pb)
    g, flags = api.Optimizer(ctx).local_ba(gpu)
    assert (g["iters_robust"], g["iters_refine"]) == (r["iters_robust"], r["iters_refine"])
    assert abs(g["final_cost"] - r["final_cost"]) <= 1e-8 * max(1.0, r["final_cost"])
    assert np.abs(gpu["pose"] - ref["pose"]).max() <= 1e-6
    assert np.abs(gpu["lm_invdepth"] - ref["lm_invdepth"]).max() <= 1e-6
    assert (flags != r["flags"]).sum() <= 3
