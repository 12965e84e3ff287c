"""The drop-in VisualFrontEnd::kltTracking (host/visual_front_end_klt_gpu.cpp) through its self-test driver
(host/klt_tracking_selftest.cpp, stand-in front-end and map classes):

  - on the CPU, with the device calls replaced by a recorder with canned answers (tests/helpers/klt_tracking_mock.c, LD_PRELOAD):
    each image is uploaded once, ONE ov2_klt_tracking call carries the frame's keypoints, map points, pose, calibration and the
    SlamParams / FeatureTracker settings, and the answers become updateKeypoint / removeObsFromCurFrameById / bp3preq_;
  - on the GPU: what the drop-in leaves in the frame equals FeatureTracker.klt_tracking on the same scene;
  - against the reference's own headers (oracle/ref_build/check_shims.py), like the other drop-ins.
"""
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

from ov2slam_b200 import api, build, synth

ROOT = Path(__file__).resolve().parent.parent
W, H = 320, 240


def _scene(seed, n, distorted):
    sc = synth.make_klt_tracking_scene(seed, [n], W, H, distorted=distorted)
    R, t = sc["Tcw"][0, :9].reshape(3, 3), sc["Tcw"][0, 9:]
    Rwc = R.T
    sc["Twc"] = np.concatenate([-Rwc @ t, synth._rot_to_quat_xyzw(Rwc)])
    sc["lmid"] = np.arange(n, dtype=np.int32) * 7 + 3
    return sc


def _write(path, sc, use_prior, win=9, nlvl=3):
    n = len(sc["px"])
    dist = sc["dist"]
    with open(path, "wb") as f:
        f.write(np.array([n, W, H, int(use_prior), win, nlvl, int(dist is not None)], np.int32).tobytes())
        f.write(np.asarray(sc["K"][0], np.float64).tobytes())
        f.write(np.asarray(dist[0, :4] if dist is not None else np.zeros(4), np.float64).tobytes())
        f.write(np.asarray(sc["Twc"], np.float64).tobytes())
        for i in range(n):
            f.write(np.array([sc["lmid"][i], sc["is3d"][i]], np.int32).tobytes())
            f.write(np.asarray(sc["px"][i], np.float32).tobytes())
            f.write(np.asarray(sc["wpt"][i], np.float64).tobytes())
        f.write(np.ascontiguousarray(sc["prevs"][0]).tobytes())
        f.write(np.ascontiguousarray(sc["curs"][0]).tobytes())


def _read(path):
    raw = np.fromfile(path, np.uint8)
    n = int(raw[:4].view(np.int32)[0])
    T = raw[4:100].view(np.float64)
    bp3p = int(raw[100:104].view(np.int32)[0])
    rec = raw[104:104 + 16 * n].reshape(n, 16)
    ids_alive = rec[:, :8].copy().view(np.int32).reshape(n, 2)
    px = rec[:, 8:].copy().view(np.float32).reshape(n, 2)
    return T, bp3p, ids_alive[:, 0], ids_alive[:, 1].astype(bool), px


def _read_log(path):
    raw = open(path, "rb").read()
    calls, o = [], 0
    while o < len(raw):
        tag = raw[o:o + 1].decode()
        o += 1
        if tag == "B":
            calls.append(("build",))
            continue
        hd = np.frombuffer(raw, np.int32, 10, o); o += 40
        pf = np.frombuffer(raw, np.float32, 3, o); o += 12
        T = np.frombuffer(raw, np.float64, 12, o); o += 96
        K = np.frombuffer(raw, np.float64, 4, o); o += 32
        D = np.frombuffer(raw, np.float64, 5, o); o += 40
        n = int(hd[2])
        px, wpt, is3d = np.zeros((n, 2), np.float32), np.zeros((n, 3)), np.zeros(n, np.uint8)
        for i in range(n):
            px[i] = np.frombuffer(raw, np.float32, 2, o); o += 8
            wpt[i] = np.frombuffer(raw, np.float64, 3, o); o += 24
            is3d[i] = raw[o]; o += 1
        calls.append(("klt", hd, pf, T, K, D, px, wpt, is3d))
    return calls


def _run(exe, scene, result, env=None):
    out = subprocess.run([str(exe), str(scene), str(result)], capture_output=True, text=True, timeout=120, env=env)
    assert out.returncode == 0, out.stdout + out.stderr
    return out


@pytest.mark.parametrize("use_prior,distorted", [(1, False), (0, True), (1, True)])
def test_klt_tracking_shim_flow(tmp_path, use_prior, distorted):
    exe = build.build_klt_tracking_shim()
    mock = tmp_path / "libmock.so"
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-O1", "-o", str(mock), str(ROOT / "tests" / "helpers" / "klt_tracking_mock.c")])
    sc = _scene(81 + distorted, 90, distorted)
    _write(tmp_path / "s.bin", sc, use_prior, win=11, nlvl=2)
    env = dict(os.environ, LD_PRELOAD=str(mock), OV2_MOCK_LOG=str(tmp_path / "log.bin"))
    _run(exe, tmp_path / "s.bin", tmp_path / "r.bin", env)
    T, bp3p, ids, alive, px_out = _read(tmp_path / "r.bin")
    calls = _read_log(tmp_path / "log.bin")
    assert [c[0] for c in calls] == ["build", "build", "klt"]          # each image uploaded once, one tracking call
    _, hd, pf, Tl, K, D, px, wpt, is3d = calls[2]
    first, count, n, win, max_iter, nlvl, up, has_dist, iw, ih = (int(v) for v in hd)
    assert (first, count, n, win, max_iter, nlvl, up, has_dist, iw, ih) == (0, 1, 90, 11, 30, 2, use_prior, int(distorted), W, H)
    assert pf[0] == np.float32(0.01) and pf[1] == 30.0 and pf[2] == np.float32(0.5)
    assert np.array_equal(Tl, T) and np.abs(Tl - sc["Tcw"][0]).max() < 1e-12
    assert np.array_equal(K, sc["K"][0])
    assert np.array_equal(D, np.concatenate([sc["dist"][0, :4], [0.0]]) if distorted else np.zeros(5))
    # the flattened keypoints, in the frame's map order: each scene keypoint exactly once with its map point and 3-D flag
    where = {tuple(p): i for i, p in enumerate(sc["px"].tolist())}
    order = np.array([where[tuple(p)] for p in px.tolist()])
    assert sorted(order.tolist()) == list(range(90))
    assert np.array_equal(is3d, sc["is3d"][order])
    assert np.array_equal(wpt[is3d == 1], sc["wpt"][order][is3d == 1]) and not wpt[is3d == 0].any()
    # the mock's answers applied: pass-1 and pass-2 tracks moved, pass-2 failures removed, the P3P request raised
    assert bp3p == use_prior
    pos = {int(s): k for k, s in enumerate(order)}
    for j in range(90):
        k = pos[j]
        p1 = is3d[k] and k % 2 == 0
        want_alive = p1 or k % 3 != 0
        assert alive[j] == want_alive, j
        if want_alive:
            assert np.array_equal(px_out[j], sc["px"][j] + (np.float32([1, 2]) if p1 else np.float32([3, 4])))


def test_klt_tracking_shim_compiles_against_the_reference_own_headers():
    """host/visual_front_end_klt_gpu.cpp against /root/reference/include itself (visual_front_end.hpp, frame.hpp, map_manager.hpp,
    camera_calibration.hpp, slam_params.hpp; the drop-in feature_tracker.hpp in place of the reference's), as
    tests/test_host_shim.py::test_shims_compile_against_the_reference_own_headers checks the other drop-ins.  The reference's
    visual_front_end.hpp defines MotionModel inline and calls Eigen's isZero, which the reduced Eigen of oracle/ref_build/mini lacks:
    the check maps that one call to squaredNorm() (a syntax check, nothing is evaluated)."""
    from oracle.ref_build import check_shims
    if not check_shims.available():
        pytest.skip("/root/reference is not present")
    check_shims.make_overlay()
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-w", "-iquote", str(check_shims.OVERLAY), *check_shims.include_flags(),
                        "-include", "cstdint", "-DisZero(eps)=squaredNorm()", str(check_shims.HOST / "visual_front_end_klt_gpu.cpp")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[:3000]


@pytest.mark.gpu
@pytest.mark.parametrize("use_prior,distorted", [(1, False), (1, True), (0, False)])
def test_klt_tracking_shim_equals_binding(ctx, tmp_path, use_prior, distorted):
    """The drop-in on the device leaves in the frame exactly what FeatureTracker.klt_tracking returns for the same scene: tracked
    keypoints at the tracked position, the others removed, bp3preq_ as p3p_req."""
    exe = build.build_klt_tracking_shim()
    sc = _scene(91 + distorted, 300, distorted)
    _write(tmp_path / "s.bin", sc, use_prior)
    _run(exe, tmp_path / "s.bin", tmp_path / "r.bin")
    T, bp3p, ids, alive, px_out = _read(tmp_path / "r.bin")
    pp, cp = api.Pyramid(ctx, 1, W, H, 3), api.Pyramid(ctx, 1, W, H, 3)
    pp.build(sc["prevs"][:1])
    cp.build(sc["curs"][:1])
    dist = None if sc["dist"] is None else np.concatenate([sc["dist"][:, :4], np.zeros((1, 1))], 1)
    ref = api.FeatureTracker(ctx, 30, 0.01).klt_tracking(pp, cp, 9, 3, 30.0, 0.5, np.array([0, 300], np.int32), T.reshape(1, 12),
                                                         sc["K"], sc["img_wh"], sc["px"], sc["wpt"], sc["is3d"], dist=dist,
                                                         use_prior=use_prior)
    assert np.array_equal(ids, sc["lmid"])
    assert np.array_equal(alive, ref["status"] == 1)
    assert np.array_equal(px_out[alive].view(np.uint32), ref["tracked"][alive].view(np.uint32))
    assert bp3p == int(ref["p3p_req"][0])
    assert 100 < alive.sum() < 300
    if use_prior:
        assert (ref["passes"] == 1).any() and ((ref["passes"] == 2) & (sc["is3d"] == 1)).any()
