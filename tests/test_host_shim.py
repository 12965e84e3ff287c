"""The drop-in C++ classes (ov2slam_b200/host/) behave like the Python binding of the same C ABI:
CPU part = they compile and link; GPU part = same keypoints / descriptors / tracks."""
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

import stereo_scenes as SS
from oracle import image_ref as R_img
from ov2slam_b200 import api, build, synth

ROOT = Path(__file__).resolve().parents[1]


def test_host_shims_compile_and_link():
    exe = build.build_host_shims()
    assert exe.exists()


@pytest.mark.gpu
def test_host_shims_match_python_binding(ctx, tmp_path):
    exe = build.build_host_shims()
    w, h = 640, 480
    prev, cur, _ = synth.make_pair(77, w, h)
    (tmp_path / "p.raw").write_bytes(prev.tobytes())
    (tmp_path / "c.raw").write_bytes(cur.tobytes())
    out = subprocess.run([str(exe), str(tmp_path / "p.raw"), str(tmp_path / "c.raw"), str(w), str(h)],
                         capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    tok = out.stdout.split()
    got = dict(nkps=int(tok[1]), th=int(tok[3]), kx=float(tok[5]), ky=float(tok[6]), ndesc=int(tok[8]), dsum=int(tok[10]),
               ngood=int(tok[12]))
    pp = api.Pyramid(ctx, 1, w, h, 3)
    cp = api.Pyramid(ctx, 1, w, h, 3)
    pp.build(prev[None])
    cp.build(cur[None])
    fe = api.FeatureExtractor(ctx, nfast_th=10)
    pts, _ = fe.detect_grid_fast_frame(pp, 0, 50, np.zeros((0, 2), np.float32))
    d = np.zeros((len(pts), 32), np.uint8)
    v = np.zeros(len(pts), np.uint8)
    fe.describe_brief(pp, pts, d, v)
    pri = pts.copy()
    st = np.zeros(len(pts), np.uint8)
    api.FeatureTracker(ctx, 30, 0.01).fb_klt_tracking(pp, cp, 9, 3, 30.0, 0.5, pts, pri, st)
    assert got["nkps"] == len(pts) and got["th"] == fe.nfast_th_
    assert abs(got["kx"] - float(pts[:, 0].astype(np.float64).sum())) < 1e-2
    assert got["ndesc"] == int(v.sum())
    assert got["dsum"] == int((d[v.astype(bool)].astype(np.int64) * np.arange(1, 33)).sum())
    assert got["ngood"] == int(st.sum())


_rect_subpix_template = R_img.get_rect_subpix_u8_ref
_line_min_sad_ref = R_img.line_min_sad_ref


def test_get_line_min_sad_matches_the_reference_function():
    """The drop-in FeatureTracker::getLineMinSAD (host C++) against a restatement of the reference's function with
    OpenCV's 8-bit getRectSubPix template: identical priors and errors - sub-pixel points, border window shrink, both
    scan directions (round 1 rounded the point, scanned the other way and dropped the shrink rule: ADVICE r1).  With
    cv2's own getRectSubPix (an IPP build: +-1 grey level on ~0.7 % of the pixels) the errors agree to 0.05 and the
    priors almost always."""
    exe = build.build_host_shims()
    w, h = 320, 240
    left = synth.make_frame(5, w, h, nrect=60)
    right = np.ascontiguousarray(np.roll(left, -7, axis=1))
    rng = np.random.default_rng(3)
    pts = [(rng.uniform(0, w - 1), rng.uniform(0, h - 1), 7, int(rng.integers(0, 2))) for _ in range(40)]
    pts += [(2.3, 100.7, 7, 1), (w - 2.2, 50.1, 7, 0), (150.5, 1.4, 7, 1), (150.5, h - 1.6, 7, 0), (60.0, 60.0, 8, 1), (0.4, 0.3, 7, 1)]
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        (open(f"{d}/l.raw", "wb")).write(left.tobytes())
        (open(f"{d}/r.raw", "wb")).write(right.tobytes())
        args = [str(exe), "--sad", f"{d}/l.raw", f"{d}/r.raw", str(w), str(h), str(len(pts))]
        for x, y, ws, gl in pts:
            args += [repr(float(np.float32(x))), repr(float(np.float32(y))), str(ws), str(gl)]
        out = subprocess.run(args, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    got = [tuple(float(v) for v in line.split()) for line in out.stdout.strip().splitlines()]
    assert len(got) == len(pts)
    try:
        import cv2
        cv_sub = lambda im, ws, cx, cy: cv2.getRectSubPix(im, (ws, ws), (float(cx), float(cy)))
    except Exception:
        cv_sub = None
    agree = 0
    for (x, y, ws, gl), (gx, ge) in zip(pts, got):
        rx, re = _line_min_sad_ref(left, right, (x, y), ws, bool(gl), _rect_subpix_template)
        if re is None:
            assert gx == -1.0
            continue
        assert np.float32(gx) == np.float32(rx) and np.float32(ge) == np.float32(re), ((x, y, ws, gl), (gx, ge), (rx, re))
        if cv_sub is not None:
            cx, ce = _line_min_sad_ref(left, right, (x, y), ws, bool(gl), cv_sub)
            assert abs(ge - ce) <= 0.05
            agree += np.float32(gx) == np.float32(cx)
    if cv_sub is not None:
        assert agree >= 0.8 * len(pts)


def _write_window(path, pb):
    import struct
    stereo = pb.get("obs_type") is not None
    ncam, npts, nobs = len(pb["pose"]), len(pb["lm_invdepth"]), len(pb["obs_cam"])
    with open(path, "wb") as f:
        f.write(struct.pack("4i", ncam, npts, nobs, int(stereo)))
        f.write(np.asarray(pb["K"], np.float64).tobytes())
        f.write(np.asarray(pb["Kr"] if stereo else pb["K"], np.float64).tobytes())
        f.write(np.asarray(pb["Trl"] if stereo else [0, 0, 0, 0, 0, 0, 1], np.float64).tobytes())
        for k, dt in (("pose", np.float64), ("pose_const", np.uint8), ("lm_anchor_cam", np.int32), ("lm_anchor_px", np.float64),
                      ("lm_invdepth", np.float64), ("obs_cam", np.int32), ("obs_lm", np.int32), ("obs_px", np.float64)):
            f.write(np.ascontiguousarray(pb[k], dt).tobytes())
        f.write(np.ascontiguousarray(pb["obs_type"] if stereo else np.zeros(nobs), np.uint8).tobytes())


def _drop_landmarks_seen_only_by_constant_keyframes(pb):
    """Optimizer::localBA collects its landmarks from the 3D keypoints of the OPTIMISED keyframes (optimizer.cpp:178-180): a
    landmark whose anchor and observers are all constant keyframes is not part of the reference's window."""
    const = pb["pose_const"].astype(bool)
    npts = len(pb["lm_invdepth"])
    seen = ~const[pb["lm_anchor_cam"]]
    np.logical_or.at(seen, pb["obs_lm"], ~const[pb["obs_cam"]])
    keep_l = np.nonzero(seen)[0]
    remap = -np.ones(npts, np.int64)
    remap[keep_l] = np.arange(len(keep_l))
    keep_o = np.nonzero(seen[pb["obs_lm"]])[0]
    out = dict(pb)
    for k in ("lm_anchor_cam", "lm_anchor_px", "lm_invdepth"):
        out[k] = np.ascontiguousarray(pb[k][keep_l])
    for k in ("obs_cam", "obs_px") + (("obs_type",) if pb.get("obs_type") is not None else ()):
        out[k] = np.ascontiguousarray(pb[k][keep_o])
    out["obs_lm"] = np.ascontiguousarray(remap[pb["obs_lm"][keep_o]].astype(np.int32))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("stereo,stop", [(False, False), (True, False), (False, True)])
def test_optimizer_localba_shim_updates_the_map_like_the_flat_solve(ctx, tmp_path, stereo, stop):
    """The drop-in Optimizer::localBA (host/optimizer_localba_gpu.cpp, compiled against the stand-in map classes) on a
    synthetic map: window selection over the covisibility map, anchored inverse-depth flattening (mono / stereo), GPU solve,
    write-back - the keyframe poses and landmark inverse depths left in the map equal ov2_localba_solve on the flat window;
    a stop request raised before the call skips the refinement and is consumed (ADVICE r1: bstop_localba_ was never cleared)."""
    exe = build.build_optimizer_shim()
    pb = _drop_landmarks_seen_only_by_constant_keyframes(synth.make_ba_problem(61 + stereo, 9, 600, 2400, stereo=stereo))
    _write_window(tmp_path / "w.bin", pb)
    out = subprocess.run([str(exe), str(tmp_path / "w.bin"), str(tmp_path / "r.bin")] + (["stop"] if stop else []),
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    ncam, npts = len(pb["pose"]), len(pb["lm_invdepth"])
    raw = np.fromfile(tmp_path / "r.bin", np.uint8)
    pose = raw[:ncam * 56].view(np.float64).reshape(ncam, 7)
    invd = raw[ncam * 56:ncam * 56 + npts * 8].view(np.float64)
    ref = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in pb.items()}
    if stop:
        api.request_stop_local_ba(ctx, True)
    res, flags = api.Optimizer(ctx).local_ba(ref)
    api.request_stop_local_ba(ctx, False)
    if stop:
        assert res["iters_refine"] == 0
    # the shim stores unit quaternions through Sophus (sign / normalisation): compare rotations up to sign
    for c in range(ncam):
        assert np.abs(pose[c, :3] - ref["pose"][c, :3]).max() <= 1e-7
        q, r = pose[c, 3:], ref["pose"][c, 3:] / np.linalg.norm(ref["pose"][c, 3:])
        assert min(np.abs(q - r).max(), np.abs(q + r).max()) <= 1e-7
    alive = invd >= 0
    assert alive.mean() > 0.9
    assert np.abs(invd[alive] - ref["lm_invdepth"][alive]).max() <= 1e-7


@pytest.mark.gpu
@pytest.mark.parametrize("mode,stereo", [("loose", False), ("loose", True), ("full", False), ("full", True)])
def test_optimizer_loose_and_full_ba_shims(ctx, tmp_path, mode, stereo):
    """8f-4: the drop-in Optimizer::looseBA / fullBA (optimizer.cpp:900-1671 / 1674-2331; same residual blocks as localBA over a
    keyframe RANGE: the first two (mono) / one (stereo) keyframes constant, all others optimised, one 5-iteration solve with
    function_tolerance 1e-4 for looseBA, up to 100 + 100 iterations at Ceres' default 1e-6 for fullBA) on a synthetic map:
    the map they leave behind equals ov2_localba_solve on the flat window with those options; looseBA also moves the current
    frame rigidly with the loop keyframe (checked inside the self-test)."""
    exe = build.build_optimizer_shim()
    pb = synth.make_ba_problem(71 + stereo, 9, 600, 2400, stereo=stereo)
    pb["pose_const"] = np.zeros_like(pb["pose_const"])
    pb["pose_const"][:1 if stereo else 2] = 1
    pb = _drop_landmarks_seen_only_by_constant_keyframes(pb)
    _write_window(tmp_path / "w.bin", pb)
    out = subprocess.run([str(exe), str(tmp_path / "w.bin"), str(tmp_path / "r.bin"), mode], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    ncam, npts = len(pb["pose"]), len(pb["lm_invdepth"])
    raw = np.fromfile(tmp_path / "r.bin", np.uint8)
    pose = raw[:ncam * 56].view(np.float64).reshape(ncam, 7)
    invd = raw[ncam * 56:ncam * 56 + npts * 8].view(np.float64)
    ref = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in pb.items()}
    if mode == "loose":
        res, flags = api.Optimizer(ctx).local_ba(ref, max_iters_robust=5, max_iters_refine=0, function_tolerance=1e-4, apply_l2_after_robust=0)
        assert res["iters_refine"] == 0
    else:
        res, flags = api.Optimizer(ctx).local_ba(ref, max_iters_robust=100, max_iters_refine=100, function_tolerance=1e-6)
    assert res["final_cost"] < res["initial_cost"]
    for c in range(ncam):
        assert np.abs(pose[c, :3] - ref["pose"][c, :3]).max() <= 1e-7
        q, r = pose[c, 3:], ref["pose"][c, 3:] / np.linalg.norm(ref["pose"][c, 3:])
        assert min(np.abs(q - r).max(), np.abs(q + r).max()) <= 1e-7
    alive = invd >= 0
    assert alive.mean() > 0.9
    assert np.abs(invd[alive] - ref["lm_invdepth"][alive]).max() <= 1e-6 * np.abs(ref["lm_invdepth"][alive]).max() + 1e-7


# ---------------------------------------------------------------------------------------------- Mapper::matchToMap drop-in
def _write_match_scene(path, sc):
    hd = np.array([len(sc["kp_px"]), len(sc["mp_xyz"]), len(sc["desc"]), len(sc["obs_kf"]), len(sc["kf_Tcw"]), len(sc["cand_mp"]),
                   len(sc["cell_ptr"]) - 1, sc["nbwcells"], sc["ncellsize"], sc["img_w"], sc["img_h"], sc["dist"] is not None], np.int32)
    dist = np.zeros(5) if sc["dist"] is None else np.asarray(sc["dist"], np.float64)
    with open(path, "wb") as f:
        f.write(hd.tobytes())
        for a, t in ((sc["K"], np.float64), (dist, np.float64), (sc["Tcw"], np.float64), (sc["kf_Tcw"], np.float64), (sc["mp_xyz"], np.float64),
                     (sc["kp_px"], np.float32), (sc["obs_px"], np.float32), (sc["cell_ptr"], np.int32), (sc["cell_kp"], np.int32),
                     (sc["kp_lm"], np.int32), (sc["mp_desc_ptr"], np.int32), (sc["mp_obs_ptr"], np.int32), (sc["obs_kf"], np.int32),
                     (sc["cand_mp"], np.int32), (sc["desc"], np.uint8)):
            f.write(np.ascontiguousarray(a, t).tobytes())


def _read_match_result(path):
    raw = np.fromfile(path, np.int32)
    n = int(raw[0])
    order = raw[1:1 + n]
    m = int(raw[1 + n])
    pairs = raw[2 + n:2 + n + 2 * m].reshape(m, 2)
    return order, {(int(a), int(b)) for a, b in pairs}, int(raw[2 + n + 2 * m])


def _read_match_dump(path):
    raw = np.fromfile(path, np.uint8)
    hd = raw[:48].view(np.int32)
    nkps, nmps, ndesc, nobs, nkfs, ncand, ncells, nbw, cs, w, h, has_dist = (int(v) for v in hd)
    fl = raw[48:60].view(np.float32)
    off = [60]

    def take(n, t):
        b = n * np.dtype(t).itemsize
        a = raw[off[0]:off[0] + b].view(t).copy()
        off[0] += b
        return a
    sc = dict(img_w=w, img_h=h, ncellsize=cs, nbwcells=nbw, dmaxpxdist=fl[0], fdistratio=fl[1], view_th=fl[2])
    sc["K"] = take(4, np.float64)
    d = take(5, np.float64)
    sc["dist"] = d if has_dist else None
    sc["Tcw"] = take(12, np.float64)
    sc["kf_Tcw"] = take(12 * nkfs, np.float64).reshape(nkfs, 12)
    sc["mp_xyz"] = take(3 * nmps, np.float64).reshape(nmps, 3)
    sc["kp_px"] = take(2 * nkps, np.float32).reshape(nkps, 2)
    sc["obs_px"] = take(2 * nobs, np.float32).reshape(nobs, 2)
    sc["cell_ptr"] = take(ncells + 1, np.int32)
    sc["cell_kp"] = take(int(sc["cell_ptr"][-1]), np.int32)
    sc["kp_lm"] = take(nkps, np.int32)
    sc["mp_desc_ptr"] = take(nmps + 1, np.int32)
    sc["mp_obs_ptr"] = take(nmps + 1, np.int32)
    sc["obs_kf"] = take(nobs, np.int32)
    sc["cand_mp"] = take(ncand, np.int32)
    sc["mp_kfmask"] = take(4 * nmps, np.uint64).reshape(nmps, 4)
    sc["desc"] = take(32 * ndesc, np.uint8).reshape(ndesc, 32)
    assert off[0] == len(raw)
    return sc


def _match_pairs_by_identity(sc, kp_match):
    """(keypoint, map point) pairs named by what they ARE (pixel + own map point's position; candidate's position), so that two
    flattenings of the same map with different index orders can be compared."""
    out = set()
    for j, c in enumerate(kp_match):
        if c >= 0:
            out.add((tuple(sc["kp_px"][j]), tuple(sc["mp_xyz"][sc["kp_lm"][j]]), tuple(sc["mp_xyz"][sc["cand_mp"][c]])))
    return out


@pytest.mark.parametrize("distorted", [True, False])
def test_mapper_match_shim_flattens_the_map_like_the_scene(tmp_path, distorted):
    """The drop-in Mapper::matchToMap (host/mapper_match_gpu.cpp, against the stand-in map classes) on a synthetic map, with the
    GPU call replaced by a recorder (tests/helpers/match_dump.c, LD_PRELOAD): the flat problem it builds from the frame grid, the
    keyframes and the map points gives, through the oracle, the matches of the scene the map was built from (candidates in the
    order the shim walked the id set); map points without descriptor are filtered, keypoints whose map point is gone are dropped
    from the map (mapper.cpp:667-672), the search radius doubles for a frame with fewer than 30 3-D keypoints."""
    from oracle import match_ref as M
    exe = build.build_mapper_shim()
    rec = tmp_path / "librec.so"
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-O1", "-o", str(rec), str(ROOT / "tests" / "helpers" / "match_dump.c")])
    sc = synth.make_match_scene(5 + distorted, nkps=500, ncand=260, nkfs=9, distorted=distorted)
    _write_match_scene(tmp_path / "s.bin", sc)
    env = dict(os.environ, LD_PRELOAD=str(rec), OV2_MATCH_DUMP=str(tmp_path / "d.bin"))
    out = subprocess.run([str(exe), str(tmp_path / "s.bin"), str(tmp_path / "r.bin")], capture_output=True, text=True, timeout=120, env=env)
    assert out.returncode == 0, out.stdout + out.stderr
    order, pairs, ndropped = _read_match_result(tmp_path / "r.bin")
    assert not pairs and ndropped == int((sc["kp_lm"] < 0).sum())
    dump = _read_match_dump(tmp_path / "d.bin")
    assert dump["dmaxpxdist"] == sc["dmaxpxdist"] and dump["fdistratio"] == sc["fdistratio"]
    assert abs(float(dump["view_th"]) - float(sc["view_th"])) <= 1e-6
    ndesc_of = np.diff(sc["mp_desc_ptr"])
    assert len(dump["cand_mp"]) == int((ndesc_of[sc["cand_mp"]] > 0).sum())
    ref = dict(sc, cand_mp=np.asarray(order, np.int32))
    want = _match_pairs_by_identity(ref, M.match_to_map(ref)[2])
    got = _match_pairs_by_identity(dump, M.match_to_map(dump)[2])
    assert len(want) > 40
    # poses travel through unit quaternions (as in the reference's map): last-bit differences in the projections
    assert len(want ^ got) <= max(1, len(want) // 100)


def _shim_against_the_oracle(tmp_path, sc):
    """Runs the drop-in twice on the map built from `sc`: once with the recorder to capture the flat problem it hands to
    ov2_match_to_map, once on the GPU.  Returns the (keypoint lmid, map-point lmid) pairs it returned, the pairs the oracle
    gives on the recorded problem (named through the recorded map-point table), and the recorded problem."""
    from oracle import match_ref as M
    exe = build.build_mapper_shim()
    rec = tmp_path / "librec.so"
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-O1", "-o", str(rec), str(ROOT / "tests" / "helpers" / "match_dump.c")])
    _write_match_scene(tmp_path / "s.bin", sc)
    env = dict(os.environ, LD_PRELOAD=str(rec), OV2_MATCH_DUMP=str(tmp_path / "d.bin"))
    out = subprocess.run([str(exe), str(tmp_path / "s.bin"), str(tmp_path / "rd.bin")], capture_output=True, text=True, timeout=120, env=env)
    assert out.returncode == 0, out.stdout + out.stderr
    out = subprocess.run([str(exe), str(tmp_path / "s.bin"), str(tmp_path / "r.bin")], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    _, pairs, _ = _read_match_result(tmp_path / "r.bin")
    dump = _read_match_dump(tmp_path / "d.bin")
    # the self-test gives map point m the id m, and the shim copies each map point's position as it is: name the recorded
    # map-point table by position
    lmid_of_xyz = {row.tobytes(): m for m, row in enumerate(np.asarray(sc["mp_xyz"], np.float64))}
    assert len(lmid_of_xyz) == len(sc["mp_xyz"])
    lmid = [lmid_of_xyz[row.tobytes()] for row in dump["mp_xyz"]]
    _, _, kp_match, _ = M.match_to_map(dump)
    want = {(lmid[dump["kp_lm"][j]], lmid[dump["cand_mp"][c]]) for j, c in enumerate(kp_match) if c >= 0}
    return pairs, want, dump


@pytest.mark.gpu
def test_mapper_match_shim_matches_python_binding(ctx, tmp_path):
    """The same drop-in end to end on the GPU: the (keypoint id -> map-point id) map it returns equals the oracle on the flat
    problem it hands over (recorded in a first run of the same binary, which walks the same id set the same way)."""
    sc = synth.make_match_scene(9, nkps=1200, ncand=700, nkfs=12, distorted=True)
    pairs, want, _ = _shim_against_the_oracle(tmp_path, sc)
    assert len(want) > 100
    assert pairs == want


@pytest.mark.gpu
def test_mapper_match_shim_with_150_keyframes(ctx, tmp_path):
    """A map of 150 keyframes: the shim's own keyframe numbering fills words 0-2 of the observation masks."""
    sc = synth.make_match_scene(10, nkps=1200, ncand=700, nkfs=150, distorted=True)
    pairs, want, dump = _shim_against_the_oracle(tmp_path, sc)
    assert len(dump["kf_Tcw"]) == 150 and np.all(dump["mp_kfmask"][:, :3].any(axis=0)) and not dump["mp_kfmask"][:, 3].any()
    assert len(want) > 100
    assert pairs == want


# ---------------------------------------------------------------------------------------------- MapManager::stereoMatching drop-in
def _read_stereo_log(path):
    """The calls tests/helpers/frontend_mock.c recorded: ("build",) per pyramid upload, ("stereo", {argument: value}) per
    ov2_stereo_matching."""
    raw = np.fromfile(path, np.uint8)
    off, calls = 0, []

    def take(k, t):
        nonlocal off
        a = raw[off:off + k * np.dtype(t).itemsize].view(t).copy()
        off += k * np.dtype(t).itemsize
        return a
    while off < len(raw):
        tag = int(take(1, np.int32)[0])
        if tag == 3:
            calls.append(("build",))
            continue
        assert tag == 5
        first, count, n, win, max_iter, rectified, nlvl, has_dist, has_grid, iw, ih, ncells = (int(v) for v in take(12, np.int32))
        a = dict(first=first, count=count, win=win, max_iter=max_iter, rectified=rectified, nklt_pyr_lvl=nlvl, img_wh=(iw, ih))
        a["eps"], a["ferr"], a["fb_dist"] = take(3, np.float32)
        a["Tcw"], a["K"], dist, a["Trl"], a["Frl"] = take(12, np.float64), take(4, np.float64), take(5, np.float64), take(12, np.float64), take(9, np.float64)
        a["dist"] = dist if has_dist else None
        grid = take(2, np.int32)
        a["grid"] = grid if has_grid else None
        a["cell_ptr"], a["cell_kps"] = (take(ncells + 1, np.int32), take(n, np.int32)) if has_grid else (None, None)
        a["px"], a["unpx"] = take(2 * n, np.float32).reshape(n, 2), take(2 * n, np.float32).reshape(n, 2)
        a["bv"] = take(3 * n, np.float64).reshape(n, 3)
        a["is3d"], a["has_mp"] = take(n, np.uint8), take(n, np.uint8)
        a["wpt"] = take(3 * n, np.float64).reshape(n, 3)
        calls.append(("stereo", a))
    return calls


@pytest.mark.parametrize("distorted", [False, True])
@pytest.mark.parametrize("rect", [1, 0])
def test_stereo_matching_shim_makes_one_call(tmp_path, rect, distorted):
    """The drop-in MapManager::stereoMatching (host/map_manager_stereo_gpu.cpp, against the stand-in map classes) on a synthetic stereo
    keyframe, the right camera undistorted or distorted, with the device calls replaced by a recorder with rule-based answers
    (tests/helpers/frontend_mock.c, LD_PRELOAD): each image is uploaded once and ONE ov2_stereo_matching call carries the keyframe's
    keypoints in Frame::getKeypoints() order with their map points, the pose, the rig, the right calibration, the grid (rigs that
    are not rectified) and the SlamParams / FeatureTracker settings; keypoints whose map point is gone are dropped from the map; exactly
    the recorder's stereo answers become stereo keypoints, at its right pixels."""
    exe = build.build_stereo_shim()
    mock = tmp_path / "libmock.so"
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-O1", "-o", str(mock), str(ROOT / "tests" / "helpers" / "frontend_mock.c")])
    sc = SS.stereo_scene(31 + rect, rect, Dr=[-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05] if distorted else None)
    SS.write_stereo_scene(tmp_path / "s.bin", sc)
    log = tmp_path / "log.bin"
    env = dict(os.environ, LD_PRELOAD=str(mock), OV2_MOCK_LOG=str(log))
    out = subprocess.run([str(exe), str(tmp_path / "s.bin"), str(tmp_path / "r.bin")], capture_output=True, text=True, timeout=120, env=env)
    assert out.returncode == 0, out.stdout + out.stderr
    r = SS.read_stereo_result(tmp_path / "r.bin")
    order, is_stereo, rpx, removed = r["order"], r["is_stereo"], r["rpx"], r["removed"]
    calls = _read_stereo_log(log)
    assert [c[0] for c in calls] == ["build", "build", "stereo"]          # left and right image: one upload each; one call
    a = calls[2][1]
    fl = SS.flat_scene(sc, order)
    n = len(order)
    assert (a["first"], a["count"], a["rectified"], a["nklt_pyr_lvl"], a["img_wh"]) == (0, 1, rect, 3, (sc["w"], sc["h"]))
    assert (a["win"], a["max_iter"], a["eps"], a["ferr"], a["fb_dist"]) == (9, 30, np.float32(0.01), 30.0, np.float32(0.5))
    for k in ("px", "unpx", "bv", "is3d", "has_mp"):
        assert np.array_equal(a[k], fl[k]), k
    mp = fl["has_mp"] == 1
    assert np.array_equal(a["wpt"][mp], fl["wpt"][mp]) and not a["wpt"][~mp].any()
    assert np.array_equal(a["K"], fl["K"][0]) and np.array_equal(a["Frl"], fl["Frl"][0])
    if distorted:
        assert np.array_equal(a["dist"], fl["dist"][0]) and a["dist"][4] == 0.0
    else:
        assert a["dist"] is None
    # the poses travel through unit quaternions (as in the reference's map)
    assert np.array_equal(a["Tcw"], r["Tcw"]) and np.array_equal(a["Trl"], r["Trl"])
    assert np.abs(a["Tcw"] - fl["Tcw"][0]).max() < 1e-12 and np.abs(a["Trl"] - fl["Trl"][0]).max() < 1e-12
    if rect:
        assert a["grid"] is None and a["cell_ptr"] is None
    else:
        assert np.array_equal(a["grid"], fl["grid"][0]) and np.array_equal(a["cell_ptr"], fl["cell_ptr"])
        assert np.array_equal(a["cell_kps"], np.concatenate([fl["cell_kps"], np.zeros(n - len(fl["cell_kps"]), np.int32)]))
    # the recorder's answers applied: keypoint i is a stereo match iff it was tracked and i % 3 != 0
    gone = (fl["is3d"] == 1) & ~mp
    assert removed == int(gone.sum()) and removed > 5
    i = np.arange(n)
    want = ~gone & (i % 3 != 0)
    assert np.array_equal(is_stereo, want) and 60 < want.sum() < n - 40
    want_rpx = fl["px"] + np.stack([np.float32(-10) - (i % 7).astype(np.float32), np.full(n, 0.25, np.float32)], 1)
    assert np.array_equal(rpx[want], want_rpx[want]) and not rpx[~want].any()


@pytest.mark.gpu
def test_stereo_matching_shim_on_the_device(tmp_path):
    """The same drop-in end to end on the GPU, on a synthetic rectified pair (a smooth texture and its copy 16 px to the left = a
    fronto-parallel plane; map points on that plane): keypoints with a map point are tracked from their projected prior on two
    levels, the others from the batched row-search prior on the full pyramid; away from the left border nearly all become stereo
    keypoints 16 px to the left on the same row."""
    exe = build.build_stereo_shim()
    disp = 16.0
    K0, base = 458.654, 0.11
    sc = SS.stereo_scene(77, 1, depth=K0 * base / disp)
    SS.write_stereo_scene(tmp_path / "s.bin", sc)
    out = subprocess.run([str(exe), str(tmp_path / "s.bin"), str(tmp_path / "r.bin"), str(disp)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    r = SS.read_stereo_result(tmp_path / "r.bin")
    order, is_stereo, rpx = r["order"], r["is_stereo"], r["rpx"]
    idx = {int(l): i for i, l in enumerate(sc["lmid"])}
    px = np.stack([sc["px"][idx[int(l)]] for l in order])
    alive = np.array([not (sc["is3d"][idx[int(l)]] and not sc["has_mp"][idx[int(l)]]) for l in order])
    inner = alive & (px[:, 0] > 60) & (px[:, 0] < sc["w"] - 20) & (px[:, 1] > 20) & (px[:, 1] < sc["h"] - 20)
    assert inner.sum() > 150
    assert is_stereo[inner].mean() > 0.9, out.stdout + out.stderr
    err = np.abs(rpx[inner & is_stereo] - (px[inner & is_stereo] - np.array([disp, 0.0], np.float32)))
    assert np.median(err[:, 0]) < 0.05 and (err[:, 0] < 0.5).mean() > 0.97 and err[:, 1].max() == 0.0
    assert not is_stereo[~alive].any()


def test_clahe_adapter_routes_cv_clahe_calls_to_the_device_call(tmp_path):
    """The cv::CLAHE adapter (host/clahe_gpu.cpp; replaces the reference's one cv::createCLAHE call, ov2slam.cpp:87) with the device
    call mocked (dst = 255 - src): a ROI source (row step > width) into a fresh destination and an in-place call both reach
    ov2_clahe with the image size, ONE row stride valid for both buffers, clip limit 3 and the W/50 x H/50 tile grid; an empty
    image gives an empty result."""
    build.build_host_shims()
    exe = build.LIB / "clahe_selftest"
    mock = tmp_path / "libmock.so"
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-O1", "-o", str(mock), str(ROOT / "tests" / "helpers" / "frontend_mock.c"), "-lm"])
    w, h = 173, 121
    env = dict(os.environ, LD_PRELOAD=str(mock), OV2_MOCK_LOG=str(tmp_path / "log.bin"))
    out = subprocess.run([str(exe), str(w), str(h), str(tmp_path / "o.bin")], capture_output=True, text=True, timeout=60, env=env)
    assert out.returncode == 0, out.stdout + out.stderr
    yy, xx = np.mgrid[0:h, 0:w]
    src = ((xx * 7 + yy * 13 + (xx * yy) % 5) & 255).astype(np.uint8)
    got = np.fromfile(tmp_path / "o.bin", np.uint8).reshape(2, h, w)
    assert np.array_equal(got[0], 255 - src) and np.array_equal(got[1], 255 - src)
    log = np.fromfile(tmp_path / "log.bin", np.int32).reshape(-1, 9)
    assert len(log) == 2 and (log[:, 0] == 4).all()
    for rec in log:
        assert tuple(rec[1:3]) == (w, h) and rec[3] == w and rec[4] == 1 and rec[5] == 3000 and tuple(rec[6:8]) == (w // 50, h // 50)
        assert rec[8] == 1          # both calls equalise in place in the destination's layout (the source was copied there first / is it)


@pytest.mark.parametrize("shim", ["feature_extractor.cpp", "feature_tracker.cpp", "clahe_gpu.cpp", "optimizer_localba_gpu.cpp", "multi_view_geometry_pnp_gpu.cpp",
                                  "mapper_match_gpu.cpp", "map_manager_stereo_gpu.cpp"])
def test_shims_compile_against_the_reference_own_headers(shim):
    """Every drop-in translation unit against /root/reference/include itself (optimizer.hpp, map_manager.hpp, mapper.hpp, frame.hpp,
    multi_view_geometry.hpp ...; the two drop-in class headers in place of the reference's feature_extractor.hpp / feature_tracker.hpp),
    with this container's stand-ins only for the third-party headers it lacks (oracle/ref_build/check_shims.py).  The self-tests above
    use reduced stand-ins of the map classes; this check is what says the member and method names the shims rely on exist."""
    from oracle.ref_build import check_shims
    if not check_shims.available():
        pytest.skip("/root/reference is not present")
    err = check_shims.check(shim)
    assert not err, err[:3000]
