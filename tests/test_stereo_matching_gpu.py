"""GPU tests of ov2_stereo_matching (MapManager::stereoMatching for a batch of keyframes): right pixels, stereo flags, passes and
per-keyframe counts bit-equal to oracle/stereo_matching_ref.py::stereo_matching_ref.

Covered: rectified and other rigs, the right camera undistorted and radial-tangential; windows 9 and 15, nklt_pyr_lvl 3 and 2;
ragged batches, empty keyframes, keyframes without 3-D keypoints, empty slots; 3-D keypoints whose map point is gone; priors on
every right-image edge and points behind the camera; neighbour cells on grid row and column 0, duplicate unpx (the NaN depth
prior) and keypoints without a 3-D neighbour; row-search columns equal to px.x and xprior = -1 (a column past px.x cannot
arise: the scan starts at px.x * downpyrcoef and moves left, and both scalings are exact); epipolar errors exactly 2 and one
float step above; failed guided tracks retried at full depth; host and device arrays, run-to-run equality and a first slot
above 0; every refusal.  A second test runs the drop-in MapManager::stereoMatching (host/stereo_selftest.cpp) on the GPU and
checks that the batched call gives the same stereo keypoints and bit-equal right pixels.

Scenes whose oracle decisions (epipolar errors) lie within a relative 1e-6 of the threshold are redrawn.
"""
import os
import subprocess

import numpy as np
import pytest

import stereo_scenes as SS
from ov2slam_b200 import api, build, synth
from oracle import image_ref as R
from oracle import stereo_matching_ref as S

pytestmark = pytest.mark.gpu

W, H = 320, 240
KEYS = ("right", "stereo", "passes", "nstereo")
PER_KF = ("Tcw", "K", "Trl", "Frl", "img_wh", "grid")


def _pyramids(ctx, sc, levels=3):
    nf = len(sc["lefts"])
    lp, rp = api.Pyramid(ctx, nf, W, H, levels), api.Pyramid(ctx, nf, W, H, levels)
    lp.build(np.asarray(sc["lefts"]))
    rp.build(np.asarray(sc["rights"]))
    return lp, rp


def _args(sc):
    return dict(dist=sc["dist"], Frl=sc["Frl"], cell_offsets=sc["cell_offsets"], grid=sc["grid"], cell_ptr=sc["cell_ptr"],
                cell_kps=sc["cell_kps"])


def _gpu(ctx, sc, win=9, nlvl=3, first=0, pyrs=None, out=None, arrays=None):
    lp, rp = pyrs or _pyramids(ctx, sc)
    a = dict(sc, **(arrays or {}))
    return api.FeatureTracker(ctx, 30, 0.01).stereo_matching(
        lp, rp, win, nlvl, 30.0, 0.5, sc["rectified"], sc["offsets"], a["Tcw"], a["K"], a["Trl"], a["img_wh"], a["px"], a["unpx"],
        a["bv"], a["is3d"], a["has_mp"], a["wpt"], dist=a["dist"], Frl=a["Frl"], cell_offsets=sc["cell_offsets"], grid=a["grid"],
        cell_ptr=a["cell_ptr"], cell_kps=a["cell_kps"], first=first, out=out)


def _ref(sc, win=9, nlvl=3, first=0):
    return S.stereo_matching_ref(sc["lefts"], sc["rights"], sc["offsets"], sc["Tcw"], sc["K"], sc["Trl"], sc["img_wh"], sc["px"],
                                 sc["unpx"], sc["bv"], sc["is3d"], sc["has_mp"], sc["wpt"], sc["rectified"], win=win,
                                 nklt_pyr_lvl=nlvl, first=first, **_args(sc))


def _assert_same(got, ref, what=""):
    for k in KEYS:
        g, r = np.asarray(got[k]), np.asarray(ref[k])
        assert g.shape == r.shape, (what, k, g.shape, r.shape)
        if k == "right":
            bad = (g.view(np.uint32) != r.view(np.uint32)).any(axis=1)
            assert not bad.any(), (what, k, np.nonzero(bad)[0][:20], float(np.abs(g - r).max()))
        else:
            assert np.array_equal(g, r), (what, k, np.nonzero(g != r)[0][:20])


def _near_tie(ref):
    e = ref["epi"][np.isfinite(ref["epi"])].astype(np.float64)
    return bool((np.abs(e - 2.0) <= 2e-6).any())


def _camera_point(T, w):
    return np.asarray(T[:9]).reshape(3, 3) @ w + T[9:]


def _scene(seed, counts, rect, distorted=False, no3d=(), empty_slots=3, win=9, nlvl=3):
    """A scene with the special keypoints of the module docstring; redrawn (next seed) while an epipolar error is a near tie."""
    for s in range(seed, seed + 20):
        sc = synth.make_stereo_matching_scene(s, counts, W, H, rectified=rect, distorted=distorted)
        rng = np.random.default_rng(s)
        for f in no3d:
            sc["is3d"][sc["offsets"][f]:sc["offsets"][f + 1]] = 0
            sc["has_mp"][sc["offsets"][f]:sc["offsets"][f + 1]] = 0
        f0, f1 = sc["offsets"][0], sc["offsets"][1]
        for f in range(len(counts)):                        # a 3-D keypoint whose map point is gone in every keyframe
            d3 = np.nonzero(sc["is3d"][sc["offsets"][f]:sc["offsets"][f + 1]])[0]
            if len(d3) > 6:
                sc["has_mp"][sc["offsets"][f] + d3[-1]] = 0
        # behind the camera: the camera point mirrored through the centre keeps its pixel
        for i in range(f0, min(f0 + 6, f1)):
            if sc["is3d"][i] and sc["has_mp"][i]:
                T = sc["Tcw"][0]
                R_ = T[:9].reshape(3, 3)
                sc["wpt"][i] = R_.T @ (-_camera_point(T, sc["wpt"][i]) - T[9:])
        # duplicate unpx: a 2-D keypoint on top of a 3-D neighbour of its own cell (NaN depth prior), and keypoints near row /
        # column 0 of the grid
        d3 = [i for i in range(f0, f1) if sc["is3d"][i] and sc["has_mp"][i]]
        d2 = [i for i in range(f0, f1) if not sc["is3d"][i]]
        if len(d2) >= 4 and len(d3) >= 2:
            for a, b in zip(d2[:2], d3[-2:]):
                sc["px"][a] = sc["px"][b] + np.float32(0.25)
                sc["unpx"][a] = sc["unpx"][b]
            sc["px"][d2[2]] = (5.0, 150.0)                  # xprior = -1: the search window shrinks to nothing
            sc["px"][d2[3]] = (3.0, 2.0)
            sc["unpx"][[d2[2], d2[3]]] = sc["px"][[d2[2], d2[3]]]
        _regrid(sc)
        if empty_slots:
            sc["px"][rng.choice(np.arange(f1, len(sc["px"])), empty_slots, replace=False)] = -1.0
        ref = _ref(sc, win, nlvl)
        if not _near_tie(ref):
            return sc, ref
    raise AssertionError("no scene without a near tie")


def _regrid(sc):
    """The grid CSR rebuilt from px (cells in index order), after keypoints were moved."""
    cs, nbw = int(sc["grid"][0][0]), int(sc["grid"][0][1])
    ncell = int(sc["cell_offsets"][1])
    ptr, kps = [0], []
    for f in range(len(sc["offsets"]) - 1):
        cells = [[] for _ in range(ncell)]
        for i in range(sc["offsets"][f], sc["offsets"][f + 1]):
            if sc["px"][i, 0] >= 0:
                cells[int(np.floor(sc["px"][i, 1] / np.float32(cs))) * nbw + int(np.floor(sc["px"][i, 0] / np.float32(cs)))].append(i)
        for c in cells:
            kps += c
            ptr.append(len(kps))
        kps += [0] * (sc["offsets"][f + 1] - sc["offsets"][f] - (len(kps) - sc["offsets"][f]))
    sc["cell_ptr"], sc["cell_kps"] = np.array(ptr, np.int32), np.array(kps, np.int32)


@pytest.mark.parametrize("nlvl", [3, 2])
@pytest.mark.parametrize("win", [9, 15])
@pytest.mark.parametrize("distorted", [False, True])
@pytest.mark.parametrize("rect", [1, 0])
def test_stereo_matching_equals_oracle(ctx, rect, distorted, win, nlvl):
    sc, ref = _scene(11 + 2 * win + nlvl, [40, 0, 23, 31, 1], rect, distorted, no3d=(3,), win=win, nlvl=nlvl)
    _assert_same(_gpu(ctx, sc, win, nlvl), ref)
    passes, st = ref["passes"], ref["stereo"].astype(bool)
    gone = sc["is3d"].astype(bool) & ~sc["has_mp"].astype(bool)
    assert (passes[gone] == 0).all() and not st[gone].any() and gone.any()
    assert (passes == 1).any() and (passes == 2).any() and st.any() and (~st & (passes > 0)).any()
    assert ref["nstereo"][1] == 0 and ref["nstereo"][3] == st[sc["offsets"][3]:sc["offsets"][4]].sum()
    # failed guided tracks retried at full depth: a 3-D keypoint with an in-image prior in pass 2
    dist = (lambda f: None) if sc["dist"] is None else (lambda f: sc["dist"][f])
    retried = [i for f in range(len(sc["offsets"]) - 1) for i in range(sc["offsets"][f], sc["offsets"][f + 1])
               if passes[i] == 2 and sc["is3d"][i] and sc["has_mp"][i] and
               S.right_prior(sc["Trl"][f], sc["K"][f], dist(f), W, H, _camera_point(sc["Tcw"][f], sc["wpt"][i]))[2]]
    assert retried
    f0 = sc["offsets"][0]
    behind = [i for i in range(f0, f0 + 6) if sc["is3d"][i] and sc["has_mp"][i]]
    assert behind and all(_camera_point(sc["Tcw"][0], sc["wpt"][i])[2] < 0 for i in behind)
    if not rect:
        args = (sc["Tcw"][0], sc["px"], sc["unpx"], sc["is3d"], sc["has_mp"], sc["wpt"], sc["cell_offsets"], sc["grid"],
                sc["cell_ptr"], sc["cell_kps"])
        depths = [S.neighbour_depth(0, i, f0, sc["offsets"][1], *args) for i in range(f0, sc["offsets"][1]) if not sc["is3d"][i]]
        assert any(d is None for d in depths) and any(d is not None and np.isnan(d) for d in depths)


def test_stereo_matching_device_buffers_and_repeat(ctx):
    torch = pytest.importorskip("torch")
    sc, ref = _scene(5, [60, 17, 0, 44], 0, distorted=True)
    pyrs = _pyramids(ctx, sc)
    host = _gpu(ctx, sc, pyrs=pyrs)
    _assert_same(host, ref, "host")
    _assert_same(_gpu(ctx, sc, pyrs=pyrs), host, "repeat")
    names = ("Tcw", "K", "dist", "Trl", "Frl", "img_wh", "grid", "cell_ptr", "cell_kps", "px", "unpx", "bv", "is3d", "has_mp", "wpt")
    dev = {k: torch.from_numpy(np.ascontiguousarray(sc[k])).cuda() for k in names}
    n, nf = len(sc["px"]), len(sc["offsets"]) - 1
    out = dict(right=torch.full((n, 2), 7.0, device="cuda"), stereo=torch.full((n,), 7, dtype=torch.uint8, device="cuda"),
               passes=torch.full((n,), 7, dtype=torch.uint8, device="cuda"), nstereo=torch.full((nf,), 7, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    _gpu(ctx, sc, pyrs=pyrs, out=out, arrays=dev)
    ctx.sync()
    _assert_same({k: v.cpu().numpy() for k, v in out.items()}, ref, "device")
    with pytest.raises(api.Ov2Error, match="must be float64"):
        _gpu(ctx, sc, pyrs=pyrs, arrays=dict(dev, wpt=dev["wpt"].float()))


def test_stereo_matching_first_slot(ctx):
    """Keyframes [2, 4) of a four-slot pyramid pair."""
    sc, _ = _scene(23, [0, 0, 35, 20], 1, empty_slots=0)
    pyrs = _pyramids(ctx, sc)
    sub = dict(sc, offsets=np.array([0, 35, 55], np.int32), **{k: sc[k][2:] for k in PER_KF})
    _assert_same(_gpu(ctx, sub, first=2, pyrs=pyrs), _ref(sub, first=2))


@pytest.mark.parametrize("rect", [1, 0])
def test_stereo_matching_prior_edges_and_behind_camera(ctx, rect):
    """Priors exactly on each right-image edge and points behind the camera.  Keyframe 0 has Tcw = Trl = [I | 0] and K = (1, 1,
    0, 0), so a map point (x, y, 1) projects to exactly (x, y), and (-x, -y, -1) projects there too from behind the camera."""
    base, _ = _scene(51, [0, 24], rect, empty_slots=0)
    cases = [((0.0, 100.0), True), ((100.0, 0.0), True), ((float(W), 100.0), False), ((100.0, float(H)), False),
             ((W - 2 ** -8, 50.0), True), ((-2 ** -20, 60.0), False), ((150.0, H - 2 ** -9), True), ((200.0, -1e-3), False)]
    rng = np.random.default_rng(51)
    px, wpt, expect = [], [], []
    for behind in (False, True):
        for (x, y), inside in cases:
            px.append((min(max(x, 10.0), W - 10.0), min(max(y, 10.0), H - 10.0)))
            wpt.append((-x, -y, -1.0) if behind else (x, y, 1.0))
            expect.append(inside)
    for _ in range(8):
        x, y = rng.uniform(20, W - 20), rng.uniform(20, H - 20)
        px.append((x + rng.normal(0, 1), y + rng.normal(0, 1)))
        wpt.append((-x * 3.0, -y * 3.0, -3.0))
        expect.append(True)
    n0 = len(px)
    sc = dict(base)
    sc["offsets"] = np.array([0, n0, n0 + 24], np.int32)
    for k, v, dt in (("px", px, np.float32), ("wpt", wpt, np.float64)):
        sc[k] = np.concatenate([np.array(v, dt), base[k]])
    sc["unpx"] = sc["px"].copy()
    sc["bv"] = np.concatenate([np.tile([0.0, 0.0, 1.0], (n0, 1)), base["bv"]])
    sc["is3d"] = np.concatenate([np.ones(n0, np.uint8), base["is3d"]])
    sc["has_mp"] = np.concatenate([np.ones(n0, np.uint8), base["has_mp"]])
    for k in ("Tcw", "Trl", "K"):
        sc[k] = base[k].copy()
    sc["Tcw"][0] = sc["Trl"][0] = [1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0]
    sc["K"][0] = [1.0, 1.0, 0.0, 0.0]
    _regrid(sc)
    ref = _ref(sc)
    for i, inside in enumerate(expect):
        assert S.right_prior(sc["Trl"][0], sc["K"][0], None, W, H, sc["wpt"][i])[2] == inside, i
    _assert_same(_gpu(ctx, sc), ref)


def test_stereo_matching_row_search_and_gate_edges(ctx):
    """Rectified rig.  Keyframe 1's right image is its left one (no shift): the row search keeps its first column, so the
    accepted prior equals px.x; keypoints at x < 8 get xprior = -1.  Then the left keypoints' unpx.y is set so that the
    row differences of gated tracks are exactly 2 (kept) and one float step above 2 (rejected); unpx does not move a track."""
    sc, _ = _scene(61, [30, 40], 1, empty_slots=0)
    sc["rights"][1] = sc["lefts"][1]
    sc["is3d"][30:] = 0
    sc["has_mp"][30:] = 0
    sc["px"][31] = sc["unpx"][31] = (5.0, 100.0)
    _regrid(sc)
    lv = R.build_pyramid_ref(sc["lefts"][1], 3)[3]
    cols = np.array([R.line_min_sad_ref(lv, lv, (p[0] * np.float32(0.125), p[1] * np.float32(0.125)), 7, True)[0] for p in sc["px"][30:]],
                    np.float32) * np.float32(8)
    assert (cols == sc["px"][30:, 0]).sum() > 20 and (cols == -8.0).any()
    ref = _ref(sc)
    gated = np.nonzero(np.isfinite(ref["epi"]))[0]
    assert len(gated) > 10
    sc2 = dict(sc, unpx=sc["unpx"].copy())
    edge, above = [], []
    for k, i in enumerate(gated):
        ry = ref["run"][i, 1]
        y2 = np.float32(ry + np.float32(2.0))
        if np.float32(y2 - ry) != np.float32(2.0):
            continue
        if k % 2 == 0:
            sc2["unpx"][i, 1] = y2
            edge.append(i)
        else:
            sc2["unpx"][i, 1] = np.nextafter(y2, np.float32(np.inf))
            above.append(i)
    ref2 = _ref(sc2)
    assert edge and above
    assert (ref2["epi"][edge] == np.float32(2.0)).all() and ref2["stereo"][edge].all()
    assert (ref2["epi"][above] > np.float32(2.0)).all() and not ref2["stereo"][above].any()
    _assert_same(_gpu(ctx, sc), ref)
    _assert_same(_gpu(ctx, sc2), ref2)


def test_stereo_matching_refusals(ctx):
    torch = pytest.importorskip("torch")
    sc, _ = _scene(7, [20, 20], 0, empty_slots=0)
    lp, rp = _pyramids(ctx, sc)
    ft = api.FeatureTracker(ctx, 30, 0.01)
    out = dict(right=np.full((40, 2), 7, np.float32), stereo=np.full(40, 7, np.uint8), passes=np.full(40, 7, np.uint8),
               nstereo=np.full(2, 7, np.int32))

    def call(win=9, nlvl=3, rect=None, pyrs=(lp, rp), **kw):
        a = dict(sc, **kw)
        return ft.stereo_matching(pyrs[0], pyrs[1], win, nlvl, 30.0, 0.5, sc["rectified"] if rect is None else rect, a["offsets"],
                                  a["Tcw"], a["K"], a["Trl"], a["img_wh"], a["px"], a["unpx"], a["bv"], a["is3d"], a["has_mp"],
                                  a["wpt"], dist=a["dist"], Frl=a["Frl"], cell_offsets=a["cell_offsets"], grid=a["grid"],
                                  cell_ptr=a["cell_ptr"], cell_kps=a["cell_kps"], first=kw.get("first", 0), out=out)
    refused = [dict(offsets=np.array([0, 25, 20], np.int32)), dict(offsets=np.array([1, 20, 40], np.int32)),
               dict(cell_offsets=np.array([0, 90, 80], np.int32)), dict(cell_offsets=np.array([3, 90, 180], np.int32)),
               dict(first=1), dict(win=2), dict(win=33)]
    small = api.Pyramid(ctx, 2, W // 2, H // 2, 3)
    small.build(np.ascontiguousarray(sc["lefts"][:, ::2, ::2]))
    shallow = api.Pyramid(ctx, 2, W, H, 2), api.Pyramid(ctx, 2, W, H, 2)
    shallow[0].build(sc["lefts"])
    shallow[1].build(sc["rights"])
    unbuilt = api.Pyramid(ctx, 2, W, H, 3)
    refused += [dict(pyrs=(lp, small)), dict(pyrs=(unbuilt, rp)), dict(pyrs=(lp, unbuilt)), dict(rect=1, nlvl=4),
                dict(rect=1, nlvl=3, pyrs=shallow)]
    for kw in refused:
        with pytest.raises(api.Ov2Error, match="INVALID"):
            call(**kw)
    assert (out["passes"] == 7).all() and (out["nstereo"] == 7).all() and (out["right"] == 7).all()
    call(rect=0, nlvl=3, pyrs=shallow)                  # other rigs need no row search: the tracker clamps the depth
    out["passes"][:] = 7
    prm = api.C.byref(api.KltParams(9, 30, float(np.float32(0.01)), 30.0, 0.5))
    for offs, cells in ((torch.from_numpy(sc["offsets"]).cuda(), sc["cell_offsets"]),
                        (sc["offsets"], torch.from_numpy(sc["cell_offsets"]).cuda())):
        p = api._ptr
        st = ctx.lib.ov2_stereo_matching(ctx.h, lp.h_, rp.h_, prm, 0, 2, p(offs), p(sc["Tcw"]), p(sc["K"]), None, p(sc["Trl"]),
                                         p(sc["Frl"]), p(sc["img_wh"]), p(cells), p(sc["grid"]), p(sc["cell_ptr"]), p(sc["cell_kps"]),
                                         p(sc["px"]), p(sc["unpx"]), p(sc["bv"]), p(sc["is3d"]), p(sc["has_mp"]), p(sc["wpt"]), 0, 3,
                                         p(out["right"]), p(out["stereo"]), p(out["passes"]), p(out["nstereo"]))
        assert st == 3
    assert (out["passes"] == 7).all()


@pytest.mark.parametrize("rect", [1, 0])
def test_batched_call_equals_the_drop_in(ctx, tmp_path, rect):
    """host/stereo_selftest.cpp's synthetic keyframe (a smooth texture and its copy 16 px to the left) through the drop-in
    MapManager::stereoMatching on the GPU, and through one ov2_stereo_matching call on the same keyframe flattened here: the drop-in
    makes that very call (with the pose and the rig as it flattened them), so the stereo keypoints and their right pixels are
    bit-equal, and the observations it removed are those of the 3-D keypoints without a map point."""
    exe = build.build_stereo_shim()
    disp = 16.0
    sc = SS.stereo_scene(77 + rect, rect, depth=458.654 * 0.11 / disp)
    SS.write_stereo_scene(tmp_path / "s.bin", sc)
    res = subprocess.run([str(exe), str(tmp_path / "s.bin"), str(tmp_path / "r.bin"), str(disp)], capture_output=True, text=True,
                         timeout=120, env=dict(os.environ))
    assert res.returncode == 0, res.stdout + res.stderr
    r = SS.read_stereo_result(tmp_path / "r.bin")
    order, is_stereo, rpx = r["order"], r["is_stereo"], r["rpx"]
    n = len(order)
    w, h = sc["w"], sc["h"]
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    tex = lambda u: np.rint(128 + 50 * np.sin(0.11 * u + 0.07 * yy) + 40 * np.sin(0.05 * u - 0.13 * yy + 1) + 30 * np.sin(0.31 * u + 0.23 * yy + 2)).astype(np.uint8)
    lp, rp = api.Pyramid(ctx, 1, w, h, 3), api.Pyramid(ctx, 1, w, h, 3)
    lp.build(tex(xx)[None])
    rp.build(tex(xx + disp)[None])
    fl = SS.flat_scene(sc, order)
    fl["Tcw"], fl["Trl"] = r["Tcw"][None], r["Trl"][None]          # as the drop-in flattens them (through unit quaternions)
    got = api.FeatureTracker(ctx, 30, 0.01).stereo_matching(
        lp, rp, 9, 3, 30.0, 0.5, fl["rectified"], fl["offsets"], fl["Tcw"], fl["K"], fl["Trl"], fl["img_wh"], fl["px"], fl["unpx"],
        fl["bv"], fl["is3d"], fl["has_mp"], fl["wpt"], dist=fl["dist"], Frl=fl["Frl"], cell_offsets=fl["cell_offsets"], grid=fl["grid"],
        cell_ptr=fl["cell_ptr"], cell_kps=fl["cell_kps"])
    st = got["stereo"].astype(bool)
    assert np.array_equal(st, is_stereo) and st.sum() > 0.5 * n, (st.sum(), is_stereo.sum())
    assert np.array_equal(got["right"][st].view(np.uint32), rpx[st].view(np.uint32))
    assert got["nstereo"][0] == is_stereo.sum()
    assert r["removed"] == int(((fl["is3d"] == 1) & (fl["has_mp"] == 0)).sum()) and r["removed"] > 0
