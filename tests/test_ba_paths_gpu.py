"""ov2_localba_solve(_batch) on every branch of the solve kernel's per-window plan (plan_window, csrc/ba_lm.cu), on windows
whose Ceres program differs from the declared one, and on device-resident windows.

Branches of the plan: the Schur phase (mode 2: private per-warp blocks, the single-window default when they fit; mode 3:
owner mode for n <= 96 and <= 256 keyframes, with 3, 6 or 10 tiles per warp for n <= 48, <= 72, <= 96; mode 0: RED), the
reduced solve (Gauss-Jordan for n <= 96, blocked Cholesky over the CTA group beyond), the lanes per landmark (4, 8 or 32
from the mean residual count per landmark), the keyframe table (shared memory or one copy per CTA in global memory) and the
group size.  `plan` restates those formulas; every case asserts the branch it lands on, and single windows also read the
branch the product took from its OV2_BA_TRACE line.

Tolerance policy as tests/test_ba_gpu.py: same LM iteration counts and terminations; against the numpy oracle (stereo
windows) costs within 1e-9 and states within 1e-7, against its C restatement (mono windows) 1e-8 and 1e-6; outlier flags
equal except threshold-borderline observations.  Batch against single solves: 1e-8."""
import ctypes as C
import re

import numpy as np
import pytest

import ba_windows as W
from ov2slam_b200 import api, synth
from oracle import ba_ref as B
from oracle import ba_ref_c as BC

pytestmark = pytest.mark.gpu

TERM = {"CONVERGENCE": 0, "NO_CONVERGENCE": 1, "FAILURE": 2}
WARPS, SCH, CH_NB, PCH, SMEM_BUDGET = 8, 8, 32, 32, 200 * 1024


# ----------------------------------------------------------------------------- plan restatement
def _owner_tile_pitch(n):
    n8 = (n + 7) & ~7
    return n8 + ((4 - n8) % 16 + 16) % 16


def plan(ncam, ncv, nobs, npts, single):
    """plan_window for a window of `ncam` keyframes of which `ncv` are optimised (used, see ba_windows.used_keyframes),
    `nobs` residuals and `npts` landmarks, solved alone (`single`) or in a batch: Schur mode (2, 3 or 0), owner tiles per
    warp (nt, mode 3 only), blocked Cholesky or Gauss-Jordan, lanes per landmark, where the keyframe table lives."""
    n = 6 * ncv
    blk = max(3 * n + n * n, 1)
    blocked = n > 96
    avg = nobs / npts if npts > 0 else 0.0
    sg = 4 if avg <= 5.0 else (8 if avg <= 12.0 else 32)
    tab = (100 * ncam + 15) & ~15                         # 12 doubles + 1 int per keyframe
    schur = (WARPS * 6 * (ncv + 1) * 8 + (((WARPS * (ncv + 1) + 1) >> 1) << 3) + WARPS * 28 * SCH * 8 + WARPS * SCH * 4 + 16 + 15) & ~15
    solve = CH_NB * (((n + 15) & ~15) + 8) * 8 if blocked else n * (n + 2) * 8
    mode = 0
    if n > 0 and tab + schur + WARPS * blk * 8 <= 190 * 1024 and single:
        mode = 2
        schur += WARPS * blk * 8
    if 0 < n <= 96 and ncam <= 256 and not (single and mode == 2):
        R = WARPS * (32 // sg)
        tile = max((R * _owner_tile_pitch(n) + 2 * R) * 8, WARPS * PCH * 26 * 8)
        mode = 3
        schur = (tile + 15) & ~15
    camtab = "global" if tab + max(schur, solve) + 16 > SMEM_BUDGET else "shared"
    nt = (3 if n <= 48 else 6 if n <= 72 else 10) if mode == 3 else None
    return dict(mode=mode, nt=nt, blocked=int(blocked), sg=sg, camtab=camtab)


def plan_of(pb, single=True):
    return plan(len(pb["pose"]), int(W.used_keyframes(pb).sum()), len(pb["obs_cam"]), len(pb["lm_invdepth"]), single)


_TRACE = re.compile(r"\[ba trace\] G=(\d+) grid=(\d+) smem=(\d+) smemS=(\d+) camtab=(\w+) blocked=(\d+) sg=(\d+)")


def _read_trace(capfd):
    m = _TRACE.findall(capfd.readouterr().err)
    assert len(m) == 1, m
    G, grid, smem, mode, camtab, blocked, sg = m[0]
    return dict(G=int(G), grid=int(grid), smem=int(smem), mode=int(mode), camtab=camtab, blocked=int(blocked), sg=int(sg))


def traced_solve(ctx, capfd, monkeypatch, pb, **opts):
    """One solve with OV2_BA_TRACE=1: the plan the product took, as its trace line reports it."""
    monkeypatch.setenv("OV2_BA_TRACE", "1")
    capfd.readouterr()
    try:
        api.Optimizer(ctx).local_ba(W.clone(pb), **opts)
    finally:
        monkeypatch.delenv("OV2_BA_TRACE")
    return _read_trace(capfd)


def assert_plan(ctx, capfd, monkeypatch, pb, **want):
    """The restated plan has the wanted branch, and a traced single solve took the same one."""
    p = plan_of(pb)
    assert {k: p[k] for k in want} == want, p
    tr = traced_solve(ctx, capfd, monkeypatch, pb)
    assert (tr["mode"], tr["blocked"], tr["sg"], tr["camtab"]) == (p["mode"], p["blocked"], p["sg"], p["camtab"]), (tr, p)
    return p


# ----------------------------------------------------------------------------- comparisons
def _check(ctx, pb, **opts):
    """Against the numpy oracle: same LM decisions, costs 1e-9, states 1e-7, flags up to threshold-borderline observations."""
    ref = W.clone(pb)
    rres = B.local_ba(ref, **opts)
    gpu = W.clone(pb)
    gres, flags = api.Optimizer(ctx).local_ba(gpu, **{k: (int(v) if isinstance(v, bool) else v) for k, v in opts.items()})
    assert (gres["iters_robust"], gres["iters_refine"]) == (rres["iters_robust"], rres["iters_refine"]), (gres, rres["termination"])
    assert gres["termination"] == TERM[rres["termination"]]
    assert abs(gres["initial_cost"] - rres["initial_cost"]) <= 1e-9 * max(1.0, abs(rres["initial_cost"]))
    assert abs(gres["final_cost"] - rres["final_cost"]) <= 1e-9 * max(1.0, abs(rres["final_cost"]))
    assert np.abs(gpu["pose"] - ref["pose"]).max() <= 1e-7 * max(1.0, np.abs(ref["pose"]).max())
    assert np.abs(gpu["lm_invdepth"] - ref["lm_invdepth"]).max() <= 1e-7 * max(1.0, np.abs(ref["lm_invdepth"]).max())
    diff = np.nonzero(flags != rres["flags"])[0]
    assert len(diff) <= 2, len(diff)
    assert gres["n_outliers_first"] == rres["n_outliers_first"] or len(diff) > 0
    return gres, rres, gpu, ref


def _check_oracle(ctx, pb, **opts):
    """Against the C restatement of the oracle (mono windows): same LM decisions, cost 1e-8, states 1e-6, flags equal up to
    threshold-borderline observations."""
    ref = W.clone(pb)
    r = BC.local_ba(ref, **opts)
    gpu = W.clone(pb)
    g, flags = api.Optimizer(ctx).local_ba(gpu, **opts)
    assert (g["iters_robust"], g["iters_refine"]) == (r["iters_robust"], r["iters_refine"]), (g, r["termination"])
    assert g["termination"] == TERM[r["termination"]]
    assert abs(g["final_cost"] - r["final_cost"]) <= 1e-8 * max(1.0, r["final_cost"])
    assert np.abs(gpu["pose"] - ref["pose"]).max() <= 1e-6
    assert np.abs(gpu["lm_invdepth"] - ref["lm_invdepth"]).max() <= 1e-6
    assert (flags != r["flags"]).sum() <= 2
    return g, r, gpu, ref


def check(ctx, pb, **opts):
    """The C restatement for mono windows, the numpy oracle for stereo ones."""
    return (_check if pb.get("obs_type") is not None else _check_oracle)(ctx, pb, **opts)


def assert_same_as_single(res, flags, solved, single):
    """Batch window against its single solve: same decisions, costs and states within 1e-8, flags up to two."""
    r1, f1, s1 = single
    assert (res["iters_robust"], res["iters_refine"], res["termination"]) == (r1["iters_robust"], r1["iters_refine"], r1["termination"])
    assert abs(res["final_cost"] - r1["final_cost"]) <= 1e-8 * max(1.0, r1["final_cost"])
    assert np.abs(solved["pose"] - s1["pose"]).max() <= 1e-8
    assert np.abs(solved["lm_invdepth"] - s1["lm_invdepth"]).max() <= 1e-8
    assert (flags != f1).sum() <= 2


def single_solve(ctx, pb, **opts):
    s = W.clone(pb)
    r, f = api.Optimizer(ctx).local_ba(s, **opts)
    return r, f, s


# ----------------------------------------------------------------------------- windows
def boundary_window(ncv, stereo, ncam=None, per=None):
    """`ncv` optimised keyframes (all used), two constant ones unless `ncam` asks for more; `per` non-anchor observations per
    landmark, by default four in a mono window (four residuals) and two in a stereo one (five residuals: each observation
    with its right-camera twin, and the anchor's right one)."""
    ncam = ncv + 2 if ncam is None else ncam
    per = (2 if stereo else 4) if per is None else per
    npts = 60 * ncv
    return synth.make_ba_problem(100 + 7 * ncv + ncam + (1 if stereo else 0), ncam, npts, per * npts, nconst=ncam - ncv,
                                 stereo=stereo)


PUSHED_KF = {17: 6, 13: 5, 9: 5}     # keyframes that anchor landmarks and whose moved residuals the first scan all flags


def pushed_window(ncv):
    """`ncv` optimised keyframes; every residual observed in or anchored in keyframe PUSHED_KF[ncv] is moved by 40 px, so the
    first scan flags them all and the refinement optimises ncv - 1 keyframes."""
    pb = synth.make_ba_problem(200 + ncv, ncv + 2, 60 * ncv, 240 * ncv)
    return W.push_keyframe(pb, PUSHED_KF[ncv]), PUSHED_KF[ncv]


def stage2_used(pb, flags):
    return int(W.used_keyframes(pb, (flags & 1) == 0).sum())


BOUNDARY = [  # ncv, ncam, branch
    (8, 10, dict(mode=2, blocked=0, camtab="shared")),
    (8, 200, dict(mode=3, nt=3, blocked=0)),
    (9, 11, dict(mode=3, nt=6, blocked=0)),
    (12, 14, dict(mode=3, nt=6, blocked=0)),
    (13, 15, dict(mode=3, nt=10, blocked=0)),
    (16, 18, dict(mode=3, nt=10, blocked=0)),
    (17, 19, dict(mode=0, blocked=1)),
    (16, 300, dict(mode=0, blocked=0, camtab="shared")),
    (8, 300, dict(mode=0, blocked=0, camtab="shared")),
]


@pytest.mark.parametrize("stereo", [False, True], ids=["mono", "stereo"])
@pytest.mark.parametrize("ncv,ncam,branch", BOUNDARY, ids=["mode2-n48", "mode3-nt3-200kf", "mode3-nt6-n54", "mode3-nt6-n72", "mode3-nt10-n78",
                                                           "mode3-nt10-n96-gj", "red-blocked-n102", "red-gj-300kf", "red-gj-n48-300kf"])
def test_plan_branch_boundaries(ctx, capfd, monkeypatch, ncv, ncam, branch, stereo):
    """Each side of every single-window branch boundary: mode 2 up to 8 optimised keyframes (and <= 195 in all), owner mode
    with 3, 6 and 10 tiles, the largest Gauss-Jordan (n = 96) and the smallest blocked Cholesky (n = 102), and RED with
    Gauss-Jordan on windows of more than 256 keyframes (owner mode is barred there) at n = 96 and n = 48."""
    pb = boundary_window(ncv, stereo, ncam)
    assert W.used_keyframes(pb).sum() == ncv
    assert_plan(ctx, capfd, monkeypatch, pb, sg=4, **branch)
    check(ctx, pb)


TRACK_WINDOWS = {  # branch: (keyframes, non-anchor observations per landmark) of the mono and of the stereo window
    "mode3-nt3-sg8": (dict(mode=3, nt=3, sg=8), (200, 8), (200, 4)),
    "mode2-sg8": (dict(mode=2, sg=8), (10, 8), (10, 4)),
    "mode2-sg32": (dict(mode=2, sg=32), (20, 14), (10, 9)),
}


@pytest.mark.parametrize("stereo", [False, True], ids=["mono", "stereo"])
@pytest.mark.parametrize("which", list(TRACK_WINDOWS))
def test_lanes_per_landmark_at_n48(ctx, capfd, monkeypatch, which, stereo):
    """8 optimised keyframes (n = 48) with longer tracks than the boundary windows: owner mode with 3 tiles and 8 lanes per
    landmark (the 200-keyframe table bars mode 2), and the private per-warp blocks of mode 2 with 8 and with 32 lanes (every
    landmark of the stereo window is seen by all 10 keyframes, 19 residuals; the mono one by 15 of 20, 14 residuals)."""
    branch, *shapes = TRACK_WINDOWS[which]
    ncam, per = shapes[stereo]
    pb = boundary_window(8, stereo, ncam, per)
    assert W.used_keyframes(pb).sum() == 8
    assert_plan(ctx, capfd, monkeypatch, pb, blocked=0, **branch)
    check(ctx, pb)


@pytest.mark.parametrize("mean,sg", [(5, 4), (6, 8), (12, 8), (13, 32)])
def test_lanes_per_landmark_from_the_data(ctx, capfd, monkeypatch, mean, sg):
    """The plan's lanes per landmark at both sides of its thresholds: mean residual counts per landmark of 5, 6, 12 and 13
    (14 optimised keyframes: owner mode, 10 tiles)."""
    pb = synth.make_ba_problem(310 + mean, 16, 300, 300 * mean)
    assert_plan(ctx, capfd, monkeypatch, pb, sg=sg, mode=3, nt=10)
    check(ctx, pb)


@pytest.mark.parametrize("stereo", [False, True], ids=["mono-20", "stereo-33to35"])
def test_long_tracks_take_32_lanes(ctx, capfd, monkeypatch, stereo):
    """Long tracks as fullBA / looseBA windows have them: 30 keyframes (28 optimised, n = 168: RED + blocked Cholesky), every
    landmark seen by 21 keyframes; in the stereo window every landmark has 33 to 35 residuals, more than a warp has lanes."""
    pb = synth.make_ba_problem(302, 30, 200, 3300, stereo=True) if stereo else synth.make_ba_problem(301, 30, 300, 6000)
    counts = np.bincount(pb["obs_lm"])
    assert counts.min() >= 20 and (counts.min() > 32) == stereo
    assert_plan(ctx, capfd, monkeypatch, pb, sg=32, mode=0, blocked=1)
    check(ctx, pb)


GROUP_WINDOWS = {"nt6-n72": (12, 14, 700), "blocked-n102": (17, 19, 1000), "blocked-n288": (48, 50, 2500)}


@pytest.mark.parametrize("ctas", ["1", "2", "3", "40"])
@pytest.mark.parametrize("which", list(GROUP_WINDOWS))
def test_group_sizes(ctx, capfd, monkeypatch, which, ctas):
    """The blocked Cholesky spread over groups of 1, 2, 3 and 40 CTAs (n = 102 and n = 288), and an owner-mode window with
    6 tiles on the same group sizes: the group barrier and the panel split must give the same solve whatever G is."""
    ncv, ncam, npts = GROUP_WINDOWS[which]
    pb = synth.make_ba_problem(400 + ncv, ncam, npts, 4 * npts)
    monkeypatch.setenv("OV2_BA_CTAS", ctas)
    p = plan_of(pb)
    assert p["blocked"] == (ncv > 16) and (p["nt"] == 6) == (ncv == 12)
    assert traced_solve(ctx, capfd, monkeypatch, pb)["G"] == int(ctas)
    check(ctx, pb)


# ----------------------------------------------------------------------------- programs that shrink
def test_unused_nonconstant_keyframes_drop_out(ctx, capfd, monkeypatch):
    """Non-constant keyframes no residual touches are not in the program (Ceres' RemoveFixedBlocks): 12 used + 3 unused
    plans as 12 (owner mode, 6 tiles, not 10), and the unused poses come back bit-identical."""
    base = boundary_window(12, False)
    pb = W.add_unused_keyframes(base, 3)
    assert (pb["pose_const"] == 0).sum() == 15 and W.used_keyframes(pb).sum() == 12
    assert_plan(ctx, capfd, monkeypatch, pb, mode=3, nt=6)
    g, r, gpu, ref = check(ctx, pb)
    assert np.array_equal(gpu["pose"][-3:], pb["pose"][-3:]) and np.array_equal(ref["pose"][-3:], pb["pose"][-3:])
    assert np.abs(gpu["pose"][:-3] - base["pose"]).max() > 0


@pytest.mark.parametrize("ncv,before,after", [(17, "blocked", "gj-n96"), (13, "nt10", "nt6"), (9, "nt6", "nt3")])
def test_keyframe_leaves_the_refinement(ctx, capfd, monkeypatch, ncv, before, after):
    """Every residual observed in or anchored in one keyframe is 40 px off, so the first scan flags them all and the
    refinement optimises one keyframe fewer: 17 -> 16 (the blocked solver runs n = 96), 13 -> 12 (owner mode, 10 -> 6
    tiles), 9 -> 8 (6 -> 3 tiles).  The landmarks anchored in that keyframe have no residual left either: their inverse
    depths, and the keyframe's pose, must keep the values the first solve left (the same window solved without the
    refinement, on the device and in the oracle)."""
    pb, kf = pushed_window(ncv)
    p = assert_plan(ctx, capfd, monkeypatch, pb)
    assert (p["blocked"], p["nt"]) == ((1, None) if ncv == 17 else (0, 10 if ncv == 13 else 6))
    g, r, gpu, ref = check(ctx, pb)
    assert stage2_used(pb, r["flags"]) == ncv - 1 and g["iters_refine"] > 0
    gone = np.nonzero(pb["lm_anchor_cam"] == kf)[0]
    assert len(gone) > 0 and ((r["flags"][np.isin(pb["obs_lm"], gone)] & 1) == 1).all()
    g1, r1, gpu1, ref1 = check(ctx, pb, apply_l2_after_robust=False)
    assert np.abs(gpu["lm_invdepth"][gone] - gpu1["lm_invdepth"][gone]).max() <= 1e-8
    assert np.abs(gpu["pose"][kf] - gpu1["pose"][kf]).max() <= 1e-8
    assert np.array_equal(ref["lm_invdepth"][gone], ref1["lm_invdepth"][gone]) and np.array_equal(ref["pose"][kf], ref1["pose"][kf])
    assert np.abs(gpu["pose"][kf] - pb["pose"][kf]).max() > 0           # the first solve did move it


def test_stereo_keyframe_touched_only_by_anchor_frame_right_residuals(ctx, capfd, monkeypatch):
    """A stereo keyframe whose only residuals are right-camera residuals in their own anchor frame (they depend on the
    inverse depth alone): the keyframe is not in the program and comes back bit-identical, its landmarks are optimised."""
    base = synth.make_ba_problem(501, 12, 500, 2000, stereo=True)
    kf = 6
    pb = W.type2_only_keyframe(base, kf)
    u = W.used_keyframes(pb)
    assert not u[kf] and u.sum() == 9 and (pb["obs_cam"] == kf).sum() == (pb["lm_anchor_cam"] == kf).sum() > 0
    assert_plan(ctx, capfd, monkeypatch, pb, mode=3, nt=6)
    g, r, gpu, ref = check(ctx, pb)
    assert np.array_equal(gpu["pose"][kf], pb["pose"][kf])
    mine = pb["lm_anchor_cam"] == kf
    assert np.abs(gpu["lm_invdepth"][mine] - pb["lm_invdepth"][mine]).min() > 0


def test_landmarks_without_residuals(ctx, capfd, monkeypatch):
    """Fewer residuals than landmarks: two landmarks in three have no residual block; they come back bit-identical."""
    base = synth.make_ba_problem(502, 10, 900, 1800)
    lone = np.arange(900)[np.arange(900) % 3 != 0]
    pb = W.drop_landmark_residuals(base, lone)
    assert len(pb["obs_cam"]) < len(pb["lm_invdepth"]) and W.used_keyframes(pb).sum() == 8
    assert_plan(ctx, capfd, monkeypatch, pb, mode=2, sg=4)
    g, r, gpu, ref = check(ctx, pb)
    assert np.array_equal(gpu["lm_invdepth"][lone], pb["lm_invdepth"][lone])


# ----------------------------------------------------------------------------- capacity
def test_capacity_counts_used_keyframes(ctx, capfd, monkeypatch):
    """70 declared non-constant keyframes of which 64 are used solve as Ceres would (64 optimised: n = 384); 65 used are
    refused with OV2_ERR_CAPACITY before anything is launched."""
    base = synth.make_ba_problem(305, 66, 2000, 6000)
    pb = W.add_unused_keyframes(base, 6)
    assert (pb["pose_const"] == 0).sum() == 70 and W.used_keyframes(pb).sum() == 64
    assert_plan(ctx, capfd, monkeypatch, pb, mode=0, blocked=1)
    g, r, gpu, ref = check(ctx, pb)
    assert np.array_equal(gpu["pose"][-6:], pb["pose"][-6:])
    over = synth.make_ba_problem(306, 67, 2000, 6000)
    assert W.used_keyframes(over).sum() == 65
    n0 = ctx.launch_count()
    with pytest.raises(api.Ov2Error, match="CAPACITY"):
        api.Optimizer(ctx).local_ba(W.clone(over))
    assert ctx.launch_count() == n0


# ----------------------------------------------------------------------------- device-resident windows
def _device_window(pb, torch, on_device):
    """An ov2_ba_problem over the window's arrays; those named in `on_device` are CUDA tensors.  Returns (struct, keep)."""
    keys = list(api._BA_KEYS) + (["obs_type", "Kr", "Trl"] if pb.get("obs_type") is not None else [])
    keep = {}
    for k in keys:
        a = np.ascontiguousarray(pb[k]).copy()
        keep[k] = torch.from_numpy(a).cuda() if k in on_device else a
    ptr = {k: (v.data_ptr() if hasattr(v, "data_ptr") else v.ctypes.data) for k, v in keep.items()}
    st = api.BaProblem(len(pb["pose"]), len(pb["lm_invdepth"]), len(pb["obs_cam"]), *[ptr[k] for k in api._BA_KEYS],
                       ptr.get("obs_type"), ptr.get("Kr"), ptr.get("Trl"))
    torch.cuda.synchronize()
    return st, keep


def _host(keep, k):
    v = keep[k]
    return v.cpu().numpy() if hasattr(v, "cpu") else v


ALL = ("K", "pose", "pose_const", "lm_anchor_cam", "lm_anchor_px", "lm_invdepth", "obs_cam", "obs_lm", "obs_px", "obs_type", "Kr", "Trl")


@pytest.mark.parametrize("stereo", [False, True], ids=["mono", "stereo"])
@pytest.mark.parametrize("on_device,flags_on", [(ALL, "device"), (ALL, "host"), (ALL, None), (("pose", "lm_invdepth"), "host"),
                                                (("pose",), "device")],
                         ids=["all-device-flags-device", "all-device-flags-host", "all-device-no-flags", "states-device", "pose-device-flags-device"])
def test_device_resident_window(ctx, on_device, flags_on, stereo):
    """Windows whose arrays are CUDA tensors (every array, or the poses and inverse depths with host observations), outlier
    flags written to device memory, host memory or nowhere: the same solve as the host window, and the states land in the
    device tensors."""
    import torch
    pb = synth.make_ba_problem(601, 10, 800, 3200, stereo=stereo)
    r1, f1, s1 = single_solve(ctx, pb)
    st, keep = _device_window(pb, torch, on_device)
    nobs = len(pb["obs_cam"])
    out = {"device": torch.zeros(nobs, dtype=torch.uint8, device="cuda"), "host": np.zeros(nobs, np.uint8), None: None}[flags_on]
    optr = None if out is None else (out.data_ptr() if hasattr(out, "data_ptr") else out.ctypes.data)
    res = api.BaResult()
    ctx.check(ctx.lib.ov2_localba_solve(ctx.h, C.byref(st), C.byref(api.BaOpts(**api.DEFAULT_BA_OPTS)), C.byref(res), optr))
    torch.cuda.synchronize()
    r = {f: getattr(res, f) for f, _ in api.BaResult._fields_}
    flags = f1 if out is None else (out.cpu().numpy() if hasattr(out, "cpu") else out)
    assert_same_as_single(r, flags, dict(pose=_host(keep, "pose"), lm_invdepth=_host(keep, "lm_invdepth")), (r1, f1, s1))
    assert hasattr(keep["pose"], "cpu") and np.abs(_host(keep, "pose") - pb["pose"]).max() > 0
    if out is not None:
        assert flags.sum() > 0


def test_batch_mixing_host_and_device_windows(ctx):
    """One batch launch with host windows and device windows (every array on the device / device states over host
    observations; flags to device memory, host memory or nowhere): every window equals its host single solve."""
    import torch
    pbs = [synth.make_ba_problem(610 + i, 8 + i, 400, 1600, stereo=(i % 2 == 1)) for i in range(6)]
    singles = [single_solve(ctx, pb) for pb in pbs]
    layouts = [(), ALL, ("pose", "lm_invdepth"), ALL, (), ("pose",)]
    flag_to = ["host", "device", None, "host", None, "device"]
    structs, keeps, outs = [], [], []
    for pb, lay, ft in zip(pbs, layouts, flag_to):
        st, keep = _device_window(pb, torch, lay)
        structs.append(st)
        keeps.append(keep)
        n = len(pb["obs_cam"])
        outs.append({"device": torch.zeros(n, dtype=torch.uint8, device="cuda"), "host": np.zeros(n, np.uint8), None: None}[ft])
    arr = (api.BaProblem * len(pbs))(*structs)
    res = (api.BaResult * len(pbs))()
    fl = (C.c_void_p * len(pbs))(*[None if o is None else (o.data_ptr() if hasattr(o, "data_ptr") else o.ctypes.data) for o in outs])
    ctx.check(ctx.lib.ov2_localba_solve_batch(ctx.h, len(pbs), arr, C.byref(api.BaOpts(**api.DEFAULT_BA_OPTS)), res, fl))
    torch.cuda.synchronize()
    for k in range(len(pbs)):
        r = {f: getattr(res[k], f) for f, _ in api.BaResult._fields_}
        o = outs[k]
        flags = singles[k][1] if o is None else (o.cpu().numpy() if hasattr(o, "cpu") else o)
        assert_same_as_single(r, flags, dict(pose=_host(keeps[k], "pose"), lm_invdepth=_host(keeps[k], "lm_invdepth")), singles[k])


# ----------------------------------------------------------------------------- batches
def _mixed_windows():
    """(name, window, batch plan): every batch plan of the windows above in one list."""
    big_table = W.add_constant_keyframes(boundary_window(17, False), 1800)
    all_const = synth.make_ba_problem(5, 6, 100, 300)
    all_const["pose_const"][:] = 1
    out = [
        ("nt3", boundary_window(8, False), dict(mode=3, nt=3)),
        ("nt3-stereo", boundary_window(8, True), dict(mode=3, nt=3)),
        ("nt6", boundary_window(12, False), dict(mode=3, nt=6)),
        ("nt10-n96", boundary_window(16, False), dict(mode=3, nt=10, blocked=0)),
        ("red-blocked", boundary_window(17, False), dict(mode=0, blocked=1, camtab="shared")),
        ("red-gj-300kf", boundary_window(16, False, 300), dict(mode=0, blocked=0)),
        ("table-global", big_table, dict(mode=0, blocked=1, camtab="global")),
        ("all-constant", all_const, dict(mode=0)),
        ("unused-kf", W.add_unused_keyframes(boundary_window(12, False), 3), dict(mode=3, nt=6)),
        ("push-17", pushed_window(17)[0], dict(blocked=1)),
        ("push-13", pushed_window(13)[0], dict(mode=3, nt=10)),
        ("push-9", pushed_window(9)[0], dict(mode=3, nt=6)),
        ("type2-only", W.type2_only_keyframe(synth.make_ba_problem(501, 12, 500, 2000, stereo=True), 6), dict(mode=3, nt=6)),
        ("lone-landmarks", W.drop_landmark_residuals(synth.make_ba_problem(502, 10, 900, 1800), np.arange(900)[np.arange(900) % 3 != 0]),
         dict(mode=3, nt=3)),
    ]
    for name, pb, want in out:
        p = plan_of(pb, single=False)
        assert {k: p[k] for k in want} == want, (name, p)
    return out


def _batch_equals_singles(ctx, pbs):
    singles = [single_solve(ctx, pb) for pb in pbs]
    batch = [W.clone(pb) for pb in pbs]
    res, flags = api.local_ba_batch(ctx, batch)
    for k in range(len(pbs)):
        assert_same_as_single(res[k], flags[k], batch[k], singles[k])
    return batch


def test_batch_mixing_every_plan(ctx):
    """One launch with owner mode (3, 6 and 10 tiles), RED, Gauss-Jordan and blocked Cholesky, the keyframe table in shared
    and in global memory, stereo, all poses constant and the shrinking programs: every window equals its single solve."""
    wins = _mixed_windows()
    batch = _batch_equals_singles(ctx, [pb for _, pb, _ in wins])
    for (name, pb, _), got in zip(wins, batch):
        if name == "table-global":
            assert np.array_equal(got["pose"][-1800:], pb["pose"][-1800:])
        if name == "all-constant":
            assert np.array_equal(got["pose"], pb["pose"])


def test_batch_reuses_groups(ctx, capfd, monkeypatch):
    """600 small windows: more than the co-resident groups (the resident CTA count is what cudaOccupancyMaxActiveBlocks-
    PerMultiprocessor gives the host, read from the trace of a launch with one CTA per group), so groups solve several
    windows each.  Every window equals its single solve; the distinct windows match the C restatement."""
    base = [synth.make_ba_problem(700 + i, 5 + i % 4, 60 + 10 * i, 240 + 40 * i) for i in range(12)]
    for pb in base:
        _check_oracle(ctx, pb)
    pbs = [base[i % len(base)] for i in range(600)]
    singles = [single_solve(ctx, pb) for pb in base]
    monkeypatch.setenv("OV2_BA_CTAS", "1")
    monkeypatch.setenv("OV2_BA_TRACE", "1")
    capfd.readouterr()
    batch = [W.clone(pb) for pb in pbs]
    res, flags = api.local_ba_batch(ctx, batch)
    monkeypatch.delenv("OV2_BA_TRACE")
    tr = _read_trace(capfd)
    # one group per resident CTA: the smallest batch that reuses groups is one window more than that
    assert tr["G"] == 1 and len(pbs) >= tr["grid"] + 1, tr
    for k in range(len(pbs)):
        assert_same_as_single(res[k], flags[k], batch[k], singles[k % len(base)])


# ----------------------------------------------------------------------------- options at their edges
OPTIONS = [dict(max_iters_robust=1), dict(max_iters_refine=1), dict(huber_th=3.84), dict(huber_th=0.5), dict(function_tolerance=0.0)]


@pytest.mark.parametrize("opts", OPTIONS, ids=["robust1", "refine1", "huber3.84", "huber0.5", "ftol0"])
@pytest.mark.parametrize("ncv", [12, 17], ids=["nt6", "blocked"])
def test_options_at_their_edges(ctx, ncv, opts):
    """One iteration per stage, a tighter and a very tight Huber threshold (a third of the residuals become outliers), no
    function tolerance: on an owner-mode window with 6 tiles and on a blocked-Cholesky window."""
    pb = boundary_window(ncv, False)
    g, r, _, _ = check(ctx, pb, **opts)
    if opts.get("huber_th") == 0.5:
        assert r["n_outliers_first"] > len(pb["obs_cam"]) // 4
    assert g["iters_robust"] <= opts.get("max_iters_robust", 5) and g["iters_refine"] <= opts.get("max_iters_refine", 10)
