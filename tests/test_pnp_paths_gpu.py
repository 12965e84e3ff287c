"""ov2_pnp_solve (csrc/pnp_solver.cu, csrc/pnp_math.cuh) against oracle/pnp_ref.py on every path and edge of ceresPnP: problems of
1 to 20 000 points (below a warp, around the 128-thread block, many points per thread), a distinct float-rounded shipped calibration
per problem, pyramid levels 0 to 3 and no levels, every option the two callers vary (robust loss, L2 pass, 0 / 1 / 5 / 10
iterations, the three shipped chi2 thresholds), points behind the camera, a start at the optimum, KITTI-scale geometry, non-unit
and w < 0 quaternions, batches of more than 1 000 problems with empty ones, device-resident buffers, the refusals of bad offsets,
and the drop-in MultiViewGeometry::ceresPnP overloads.

Every problem must give the oracle's success flag, rejected blocks and LM iteration count exactly, and its pose to 1e-9.  The
oracle is pinned to the real Ceres, iteration counts included (tests/test_oracle_vs_reference_ceres.py).  The device sums in
another order and contracts to FMA, so the scenes are drawn through the near-tie guard of tests/pnp_scenes.py: no decision of the
oracle lies within a relative 1e-6 of its threshold."""
import struct
import subprocess

import numpy as np
import pytest

import pnp_scenes as S
from ov2slam_b200 import api, build

pytestmark = pytest.mark.gpu

OV2_ERR_INVALID = 3
POSE_TOL = 1e-9
CALIB_NAMES = sorted(S.CALIBS)
DEFAULT = dict(nmaxiter=5, chi2th=5.9915, use_robust=True, apply_l2=True)
REDRAWS = []


def _has_outliers(r):
    return len(r[2]) > 0


def _batch(cases, opts, scales=True):
    """cases: list of (seed, make() arguments, keep) or None for an empty problem.  Returns the scenes (None for empty ones) and
    the oracle results.  A problem without pyramid levels gets level 0 when the batch passes levels (scales=True)."""
    scenes, refs = [], []
    for i, c in enumerate(cases):
        if c is None:
            scenes.append(None)
            refs.append(None)
            continue
        seed, kw, keep = c
        kw = dict(kw)
        kw.setdefault("calib", CALIB_NAMES[i % len(CALIB_NAMES)])
        if not scales:
            kw["scales"] = False
        sc, res, k = S.draw(seed, keep=keep, opts=opts, **kw)
        REDRAWS.append(k)
        if scales and sc["scales"] is None:
            sc = dict(sc, scales=np.zeros(sc["n"], np.int32))       # level 0 scales a residual by exactly 1
        scenes.append(sc)
        refs.append(res)
    return scenes, refs


def _flatten(scenes, scales=True):
    sizes = [0 if s is None else s["n"] for s in scenes]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    live = [s for s in scenes if s is not None]
    unpx = np.ascontiguousarray(np.concatenate([s["px"] for s in live]))
    wpts = np.ascontiguousarray(np.concatenate([s["w"] for s in live]))
    sc = np.ascontiguousarray(np.concatenate([s["scales"] for s in live]).astype(np.int32)) if scales else None
    start = np.stack([S.make(0, 1)["T0"] if s is None else s["T0"] for s in scenes])
    K = np.stack([S.CALIB_K["euroc_left"] if s is None else s["K"] for s in scenes])
    return off, unpx, wpts, sc, np.ascontiguousarray(K), np.ascontiguousarray(start)


def _run(ctx, scenes, opts, scales=True):
    off, unpx, wpts, sc, K, start = _flatten(scenes, scales)
    poses = start.copy()
    ok, flags, its = api.MultiViewGeometry(ctx).ceres_pnp_batch(off, unpx, wpts, K, poses, opts["nmaxiter"], opts["chi2th"], opts["use_robust"],
                                                                 opts["apply_l2"], sc)
    return dict(off=off, start=start, ok=ok.copy(), flags=flags.copy(), its=its.copy(), pose=poses)


def _check(scenes, refs, got):
    off = got["off"]
    worst = 0.0
    for k, (sc, ref) in enumerate(zip(scenes, refs)):
        if sc is None:
            assert got["ok"][k] == 0 and got["its"][k] == 0 and np.array_equal(got["pose"][k], got["start"][k]), k
            continue
        ok, pose, outliers, info = ref
        assert bool(got["ok"][k]) == ok, k
        assert np.array_equal(np.nonzero(got["flags"][off[k]:off[k + 1]])[0], outliers), (k, sc["n"])
        assert got["its"][k] == info["summary"]["iterations"], (k, sc["n"], got["its"][k], info["summary"]["iterations"])
        if len(outliers) == sc["n"]:          # every block rejected: false, the pose as given, bit for bit
            assert not ok and got["pose"][k].tobytes() == got["start"][k].tobytes(), k
        else:
            d = np.abs(got["pose"][k] - pose).max()
            assert d <= POSE_TOL, (k, sc["n"], d)
            worst = max(worst, d)
    return worst


SIZES = [1, 2, 3, 4, 5, 31, 32, 33, 127, 128, 129, 700, 5000, 20000]


def _ragged_cases():
    cases = [None]                                                                           # an empty problem first
    cases += [(100 + i, dict(n=n, nout=n // 10, scales=bool(i % 2)), None) for i, n in enumerate(SIZES)]
    cases += [
        (200, dict(n=120, behind=15, nout=5), lambda r: len(r[2]) >= 15),                    # depth test rejects points
        (201, dict(n=60, behind=60), lambda r: not r[0] and len(r[2]) == 60),                # every point behind the camera
        None,                                                                                # an empty problem in the middle
        (202, dict(n=8, scales=3, start="optimum"), lambda r: r[3]["summary"]["iterations"] == 0),
        (203, dict(n=300, far=True, calib="kitti_00-02", nout=30), _has_outliers),           # KITTI scale: |t| = 500 m
        (204, dict(n=300, far=True, calib="kitti_04-12", scales=True), None),
        (205, dict(n=150, quat="nonunit", nout=10), None),
        (206, dict(n=150, quat="wneg", nout=10), None),
        (207, dict(n=400, nout=100, scales=True), _has_outliers),
        (208, dict(n=64, noise=0.6, nout=0), None),
        None,                                                                                # and last
    ]
    return cases


@pytest.mark.parametrize("scales", [True, False], ids=["levels", "no_levels"])
def test_ragged_batch_matches_oracle(ctx, scales):
    """One launch over every problem size, calibration, depth, start and geometry edge, with and without pyramid levels."""
    scenes, refs = _batch(_ragged_cases(), DEFAULT, scales)
    worst = _check(scenes, refs, _run(ctx, scenes, DEFAULT, scales))
    print(f"ragged batch: largest pose difference {worst:.2e}, redraws so far {sum(REDRAWS)} of {len(REDRAWS)} scenes")


OPTION_SETS = [dict(nmaxiter=m, chi2th=th, use_robust=r, apply_l2=l2) for r in (True, False) for l2 in (True, False)
               for m in (0, 1, 5, 10) for th in S.CHI2TH]


@pytest.mark.parametrize("opts", OPTION_SETS, ids=lambda o: f"robust{int(o['use_robust'])}_l2{int(o['apply_l2'])}_it{o['nmaxiter']}_th{o['chi2th']}")
def test_options_match_oracle(ctx, opts):
    """Every use_robust x apply_l2 combination with 0, 1, 5 and 10 iterations and the three shipped chi2 thresholds."""
    base = 300 + 17 * OPTION_SETS.index(opts)
    cases = [(base, dict(n=3), None), (base + 1, dict(n=40, nout=4), None), (base + 2, dict(n=150, nout=15, scales=True), None),
             (base + 3, dict(n=600, nout=60, behind=10), None), (base + 4, dict(n=33, far=True, calib="kitti_03"), None),
             (base + 5, dict(n=129, scales=True), None)]
    if opts["nmaxiter"] == 10:
        # a start far enough from the truth that the solve needs more than 5 iterations
        cases.append((3, dict(n=200, nout=20, spread=15.0, calib="euroc_left"), lambda r: max(s["iterations"] for s in r[3]["solves"]) > 5))
    scenes, refs = _batch(cases, opts)
    _check(scenes, refs, _run(ctx, scenes, opts))


def test_chi2_exactly_on_the_threshold_is_kept(ctx):
    """chi2 > chi2th rejects, chi2 == chi2th keeps.  Identity start, points on the optical axis: every projection is exact, so the
    residual (2, 0) of point 1 gives chi2 = 4 = chi2th in any summation order, with or without FMA (no near-tie guard needed)."""
    K = S.CALIB_K["euroc_left"]
    w = np.array([[0.0, 0.0, 4.0], [0.0, 0.0, 6.0], [0.0, 0.0, 9.0]])
    px = np.array([[K[2], K[3]], [K[2] - 2.0, K[3]], [K[2] - 4.0, K[3]]])
    T0 = np.array([0.0, 0, 0, 0, 0, 0, 1])
    sc = dict(px=px, w=w, scales=None, K=K, T0=T0, n=3)
    opts = dict(nmaxiter=0, chi2th=4.0, use_robust=True, apply_l2=False)
    ref = S.solve(sc, **opts)
    assert list(ref[2]) == [2] and ref[3]["chi2"][1] == 4.0
    _check([sc], [ref], _run(ctx, [sc], opts, scales=False))


def _many():
    rng = np.random.default_rng(77)
    cases = []
    for i in range(1100):
        if i in (0, 550, 1099) or rng.random() < 0.02:
            cases.append(None)
        else:
            cases.append((5000 + i, dict(n=int(rng.integers(1, 70)), nout=int(rng.integers(0, 4)), scales=bool(rng.random() < 0.5)), None))
    return cases


def test_more_than_a_thousand_problems_with_empty_ones(ctx):
    scenes, refs = _batch(_many(), DEFAULT)
    assert len(scenes) > 1000 and scenes[0] is None and scenes[550] is None and scenes[-1] is None
    _check(scenes, refs, _run(ctx, scenes, DEFAULT))


def test_batch_is_deterministic_and_equals_problems_solved_alone(ctx):
    scenes, refs = _batch(_ragged_cases(), DEFAULT)
    a, b = _run(ctx, scenes, DEFAULT), _run(ctx, scenes, DEFAULT)
    for key in ("ok", "flags", "its", "pose"):
        assert a[key].tobytes() == b[key].tobytes(), key
    for k, sc in enumerate(scenes):
        if sc is None:
            continue
        one = _run(ctx, [sc], DEFAULT)
        assert one["ok"][0] == a["ok"][k] and one["its"][0] == a["its"][k], k
        assert one["flags"].tobytes() == a["flags"][a["off"][k]:a["off"][k + 1]].tobytes(), k
        assert one["pose"][0].tobytes() == a["pose"][k].tobytes(), k


def _call(ctx, off, unpx, wpts, sc, K, pose, flags, ok, its, opts=DEFAULT):
    return ctx.lib.ov2_pnp_solve(ctx.h, len(off) - 1, api._ptr(off), api._ptr(unpx), api._ptr(wpts), api._ptr(sc), api._ptr(K), api._ptr(pose),
                                 opts["nmaxiter"], opts["chi2th"], int(opts["use_robust"]), int(opts["apply_l2"]), api._ptr(flags), api._ptr(ok),
                                 api._ptr(its))


def test_device_buffers_and_null_iterations_give_the_host_bits(ctx):
    torch = pytest.importorskip("torch")
    scenes, refs = _batch([(900, dict(n=300, nout=30, scales=True), None), None, (901, dict(n=40, behind=4), None),
                           (902, dict(n=2000, nout=100, scales=True), None)], DEFAULT)
    host = _run(ctx, scenes, DEFAULT)
    _check(scenes, refs, host)
    off, unpx, wpts, sc, K, start = _flatten(scenes)
    dev = [torch.from_numpy(a).cuda() for a in (unpx, wpts, sc, K, start.copy())]
    n, nprob = int(off[-1]), len(off) - 1
    dflags = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
    dok = torch.full((nprob,), 7, dtype=torch.uint8, device="cuda")
    dits = torch.full((nprob,), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    assert _call(ctx, off, *dev, dflags, dok, dits) == api.OV2_OK
    ctx.sync()
    assert dev[4].cpu().numpy().tobytes() == host["pose"].tobytes()
    assert dflags.cpu().numpy().tobytes() == host["flags"].tobytes()
    assert dok.cpu().numpy().tobytes() == host["ok"].tobytes() and dits.cpu().numpy().tobytes() == host["its"].tobytes()
    # iterations_out = NULL, host buffers
    pose, flags, ok = start.copy(), np.zeros(n, np.uint8), np.zeros(nprob, np.uint8)
    assert _call(ctx, off, unpx, wpts, sc, K, pose, flags, ok, None) == api.OV2_OK
    assert pose.tobytes() == host["pose"].tobytes() and flags.tobytes() == host["flags"].tobytes() and ok.tobytes() == host["ok"].tobytes()


@pytest.mark.parametrize("offsets", [[1, 10], [0, 50, 10], [0, -5, 10], [0, 5, -1], "device"])
def test_bad_offsets_are_refused_with_outputs_untouched(ctx, offsets):
    """A device offsets array, a first offset other than 0, a descending interior offset and negative offsets return INVALID
    before anything is staged or launched; the outputs keep their bytes and the context stays usable."""
    sc = S.make(950, 10)
    unpx, wpts, K = sc["px"], sc["w"], np.ascontiguousarray(np.stack([sc["K"]] * 2))
    if offsets == "device":
        torch = pytest.importorskip("torch")
        off_arg = torch.tensor([0, 5, 10], dtype=torch.int32, device="cuda")
        nprob = 2
    else:
        off_arg = np.array(offsets, np.int32)
        nprob = len(offsets) - 1
    pose = np.ascontiguousarray(np.stack([sc["T0"]] * 2))
    flags, ok, its = np.full(64, 0xAB, np.uint8), np.full(2, 0xAB, np.uint8), np.full(2, -7, np.int32)
    before = [a.tobytes() for a in (pose, flags, ok, its)]
    st = ctx.lib.ov2_pnp_solve(ctx.h, nprob, api._ptr(off_arg), unpx.ctypes.data, wpts.ctypes.data, None, K.ctypes.data, pose.ctypes.data, 5, 5.9915,
                               1, 1, flags.ctypes.data, ok.ctypes.data, its.ctypes.data)
    assert st == OV2_ERR_INVALID
    assert [a.tobytes() for a in (pose, flags, ok, its)] == before
    scenes, refs = _batch([(951, dict(n=50, nout=5), None)], DEFAULT)
    _check(scenes, refs, _run(ctx, scenes, DEFAULT))


def _dropin(tmp_path, sc, opts, scales):
    exe = build.build_optimizer_shim()
    n = sc["n"]
    with open(tmp_path / "p.bin", "wb") as f:
        f.write(struct.pack("4i", n, opts["nmaxiter"], int(opts["use_robust"]), int(opts["apply_l2"])))
        f.write(struct.pack("5f", opts["chi2th"], *sc["K"]))
        f.write(np.ascontiguousarray(sc["T0"], np.float64).tobytes())
        f.write(np.ascontiguousarray(sc["px"], np.float64).tobytes() + np.ascontiguousarray(sc["w"], np.float64).tobytes())
        f.write(np.ascontiguousarray(scales, np.int32).tobytes())
    out = subprocess.run([str(exe), "pnp", str(tmp_path / "p.bin"), str(tmp_path / "r.bin")], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    raw, pos, res = (tmp_path / "r.bin").read_bytes(), 0, []
    for _ in range(2):
        rc, = struct.unpack_from("i", raw, pos)
        T = np.frombuffer(raw, np.float64, 7, pos + 4).copy()
        nout, = struct.unpack_from("i", raw, pos + 60)
        idx = np.frombuffer(raw, np.int32, nout, pos + 64).copy()
        pos += 64 + 4 * nout
        res.append((bool(rc), T, idx))
    return res


@pytest.mark.parametrize("case", ["l2", "no_l2", "all_rejected", "empty", "levels"])
def test_dropin_ceres_pnp_overloads(tmp_path, case):
    """MultiViewGeometry::ceresPnP (host/multi_view_geometry_pnp_gpu.cpp) called through both overloads, K rounded to float as the
    reference passes it: the return value, Twc and voutliersidx of the oracle; the scale-less overload equals levels of 0; every
    block rejected returns false with Twc untouched and every index listed; an empty input returns false."""
    opts = dict(DEFAULT, apply_l2=case != "no_l2")
    if case == "empty":
        sc = dict(S.make(960, 1), n=0)
        sc.update(px=np.zeros((0, 2)), w=np.zeros((0, 3)))
        for ok, T, idx in _dropin(tmp_path, sc, opts, np.zeros(0, np.int32)):
            assert not ok and np.abs(T - sc["T0"]).max() <= 1e-15 and len(idx) == 0
        return
    kw = dict(l2=dict(n=200, nout=20), no_l2=dict(n=200, nout=20), all_rejected=dict(n=30, behind=30), levels=dict(n=200, nout=20, scales=True))[case]
    keep = (lambda r: not r[0] and len(r[2]) == 30) if case == "all_rejected" else _has_outliers
    sc, (ok_r, pose_r, out_r, _), _ = S.draw(961, keep=keep, opts=opts, **kw)
    levels = sc["scales"] if sc["scales"] is not None else np.zeros(sc["n"], np.int32)
    (ok1, T1, idx1), (ok2, T2, idx2) = _dropin(tmp_path, sc, opts, levels)
    assert ok1 == ok_r and np.array_equal(idx1, out_r)
    if case == "all_rejected":
        assert np.array_equal(idx1, np.arange(sc["n"])) and np.abs(T1 - sc["T0"]).max() <= 1e-15
    else:
        # the drop-in hands Twc back through SE3d(q, t), which normalises the quaternion once more
        assert np.abs(T1 - pose_r).max() <= POSE_TOL
    if case != "levels":                      # the scale-less overload is the scaled one at level 0
        assert ok2 == ok1 and np.array_equal(idx2, idx1) and T2.tobytes() == T1.tobytes()
