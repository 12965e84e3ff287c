"""GPU tests of ov2_klt_tracking (VisualFrontEnd::kltTracking for a batch of frames): tracked positions, statuses, passes,
P3P requests and pass-1 counts bit-equal to oracle/klt_tracking_ref.py::klt_tracking_ref.

Covered: windows 9 and 15; ragged frames, empty frames and frames without 3-D keypoints; use_prior 0 and 1; bad priors that
send tracks to the full-depth retry; frames below the 33 % rule and exactly on it (100 pass-1 keypoints: 33 good keep the
retries' priors, 32 reset them); priors on every image edge (x == img_w and y == img_h rejected, x == 0 and y == 0 kept);
map points behind the camera; no distortion and radial-tangential; empty slots (px.x < 0); host and device buffers;
run-to-run equality; a first frame slot > 0; the refused offsets.
"""
import numpy as np
import pytest

from ov2slam_b200 import api, synth
from oracle import image_ref as R
from oracle import klt_tracking_ref as KT

pytestmark = pytest.mark.gpu

W, H = 320, 240
KEYS = ("tracked", "status", "passes", "p3p_req", "nbgood", "nbkps")


def _pyramids(ctx, sc):
    prevs, curs = np.asarray(sc["prevs"]), np.asarray(sc["curs"])
    nf = len(prevs)
    pp, cp = api.Pyramid(ctx, nf, W, H, 3), api.Pyramid(ctx, nf, W, H, 3)
    pp.build(prevs)
    cp.build(curs)
    return pp, cp


def _gpu(ctx, sc, win=9, use_prior=True, nlvl=3, first=0, pyrs=None):
    pp, cp = pyrs or _pyramids(ctx, sc)
    return api.FeatureTracker(ctx, 30, 0.01).klt_tracking(pp, cp, win, nlvl, 30.0, 0.5, sc["offsets"], sc["Tcw"], sc["K"],
                                                           sc["img_wh"], sc["px"], sc["wpt"], sc["is3d"], dist=sc["dist"],
                                                           use_prior=use_prior, first=first)


def _ref(sc, win=9, use_prior=True, nlvl=3, first=0):
    return KT.klt_tracking_ref(sc["prevs"], sc["curs"], sc["offsets"], sc["Tcw"], sc["K"], sc["img_wh"], sc["px"], sc["wpt"],
                               sc["is3d"], dist=sc["dist"], win=win, nklt_pyr_lvl=nlvl, use_prior=use_prior, first=first)


def _assert_same(got, ref, what=""):
    for k in KEYS:
        g, r = np.asarray(got[k]), np.asarray(ref[k])
        assert g.shape == r.shape, (what, k, g.shape, r.shape)
        if k == "tracked":
            bad = (g.view(np.uint32) != r.view(np.uint32)).any(axis=1)
            assert not bad.any(), (what, k, np.nonzero(bad)[0][:20], float(np.abs(g - r).max()))
        else:
            assert np.array_equal(g, r), (what, k, np.nonzero(g != r)[0][:20])


def _scene(seed, counts, distorted=False, no3d_frames=(), empty_slots=0):
    sc = synth.make_klt_tracking_scene(seed, counts, W, H, distorted=distorted)
    for f in no3d_frames:
        sc["is3d"][sc["offsets"][f]:sc["offsets"][f + 1]] = 0
    if empty_slots:
        sc["px"][np.random.default_rng(seed).choice(len(sc["px"]), empty_slots, replace=False)] = -1.0
    return sc


@pytest.mark.parametrize("distorted", [False, True])
@pytest.mark.parametrize("use_prior", [1, 0])
@pytest.mark.parametrize("win", [9, 15])
def test_klt_tracking_equals_oracle(ctx, win, use_prior, distorted):
    sc = _scene(11 + win, [40, 0, 23, 31, 1], distorted, no3d_frames=(3,), empty_slots=3)
    ref = _ref(sc, win, use_prior)
    _assert_same(_gpu(ctx, sc, win, use_prior), ref)
    if use_prior:
        assert ref["nbkps"][3] == 0 and ref["p3p_req"][3] == 0            # a frame without 3-D keypoints skips pass 1
        retried = (ref["passes"] == 2) & sc["is3d"].astype(bool)
        assert retried.any() and (ref["passes"] == 1).any()               # the bad priors send tracks to the retry
    else:
        assert not ref["nbkps"].any() and not (ref["passes"] == 1).any()
    assert (ref["passes"] == 0).sum() == 3 and not ref["status"][ref["passes"] == 0].any()


def test_klt_tracking_device_buffers_and_repeat(ctx):
    torch = pytest.importorskip("torch")
    sc = _scene(5, [60, 17, 0, 44], distorted=True)
    ref = _ref(sc)
    pyrs = _pyramids(ctx, sc)
    host = _gpu(ctx, sc, pyrs=pyrs)
    _assert_same(host, ref, "host")
    _assert_same(_gpu(ctx, sc, pyrs=pyrs), host, "repeat")
    dev = {k: torch.from_numpy(np.ascontiguousarray(sc[k])).cuda() for k in ("Tcw", "K", "dist", "img_wh", "px", "wpt", "is3d")}
    n, nf = len(sc["px"]), len(sc["offsets"]) - 1
    out = dict(tracked=torch.full((n, 2), 7.0, device="cuda"), status=torch.full((n,), 7, dtype=torch.uint8, device="cuda"),
               passes=torch.full((n,), 7, dtype=torch.uint8, device="cuda"),
               p3p_req=torch.full((nf,), 7, dtype=torch.uint8, device="cuda"),
               nbgood=torch.full((nf,), 7, dtype=torch.int32, device="cuda"), nbkps=torch.full((nf,), 7, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    pp, cp = pyrs
    api.FeatureTracker(ctx, 30, 0.01).klt_tracking(pp, cp, 9, 3, 30.0, 0.5, sc["offsets"], dev["Tcw"], dev["K"], dev["img_wh"],
                                                   dev["px"], dev["wpt"], dev["is3d"], dist=dev["dist"], out=out)
    ctx.sync()
    _assert_same({k: v.cpu().numpy() for k, v in out.items()}, ref, "device")


def test_klt_tracking_first_slot(ctx):
    """Frames [2, 4) of a four-slot pyramid pair."""
    sc = _scene(23, [0, 0, 35, 20])
    pyrs = _pyramids(ctx, sc)
    sub = dict(sc, offsets=np.array([0, 35, 55], np.int32), Tcw=sc["Tcw"][2:], K=sc["K"][2:], img_wh=sc["img_wh"][2:])
    _assert_same(_gpu(ctx, sub, first=2, pyrs=pyrs), _ref(sub, first=2))


def _pass1_outcomes(sc, f, idx, pri):
    prev, cur = sc["prevs"][f], sc["curs"][f]
    return R.fb_klt_ref(prev, cur, sc["px"][idx], pri, 9, 1)[1]


@pytest.mark.parametrize("ngood", [33, 32, 10])
def test_klt_tracking_p3p_rule_edge(ctx, ngood):
    """100 pass-1 keypoints of which exactly `ngood` track: 33 is not below 0.33 * 100 (priors kept), 32 is (reset)."""
    pool = synth.make_klt_tracking_scene(40, [400], W, H, frac3d=1.0, bad_frac=0.5)
    idx = np.arange(400)
    pri = np.zeros((400, 2), np.float32)
    for i in idx:
        x, y, inside = KT.prior(pool["Tcw"][0], pool["K"][0], None, W, H, pool["wpt"][i])
        pri[i] = (x, y) if inside else (-1, -1)
    ok_prior = pri[:, 0] >= 0
    st = np.zeros(400, np.uint8)
    st[ok_prior] = _pass1_outcomes(pool, 0, idx[ok_prior], pri[ok_prior])
    good, bad = idx[ok_prior & (st == 1)], idx[ok_prior & (st == 0)]
    assert len(good) >= 33 and len(bad) >= 90, (len(good), len(bad))
    pick = np.concatenate([good[:ngood], bad[:100 - ngood]])
    sc = dict(pool, offsets=np.array([0, 100], np.int32), px=pool["px"][pick].copy(), wpt=pool["wpt"][pick].copy(),
              is3d=pool["is3d"][pick].copy())
    ref = _ref(sc)
    assert ref["nbkps"][0] == 100 and ref["nbgood"][0] == ngood
    assert ref["p3p_req"][0] == (ngood < 33)
    _assert_same(_gpu(ctx, sc), ref)


def test_klt_tracking_prior_edges_and_behind_camera(ctx):
    """Priors exactly on each image edge and points behind the camera.  Frame 0 has Tcw = [I | 0] and K = (1, 1, 0, 0), so a
    map point (x, y, 1) projects to exactly (x, y) and (-x, -y, -1) projects there too, from behind the camera."""
    base = synth.make_klt_tracking_scene(51, [0, 24], W, H)
    cases = [((0.0, 100.0), True), ((100.0, 0.0), True), ((float(W), 100.0), False), ((100.0, float(H)), False),
             ((W - 2 ** -8, 50.0), True), ((-2 ** -20, 60.0), False), ((150.0, H - 2 ** -9), True), ((200.0, -1e-3), False)]
    rng = np.random.default_rng(51)
    px, wpt, expect = [], [], []
    for behind in (False, True):
        for (x, y), inside in cases:
            px.append((min(max(x, 10.0), W - 10.0), min(max(y, 10.0), H - 10.0)))
            wpt.append((-x, -y, -1.0) if behind else (x, y, 1.0))
            expect.append(inside)
    for _ in range(8):                                  # 3-D keypoints behind the camera whose prior lies in the image
        x, y = rng.uniform(20, W - 20), rng.uniform(20, H - 20)
        px.append((x + rng.normal(0, 1), y + rng.normal(0, 1)))
        wpt.append((-x * 3.0, -y * 3.0, -3.0))
        expect.append(True)
    n0 = len(px)
    sc = dict(base)
    sc["offsets"] = np.array([0, n0, n0 + 24], np.int32)
    sc["px"] = np.concatenate([np.array(px, np.float32), base["px"]])
    sc["wpt"] = np.concatenate([np.array(wpt), base["wpt"]])
    sc["is3d"] = np.concatenate([np.ones(n0, np.uint8), base["is3d"]])
    sc["Tcw"] = base["Tcw"].copy()
    sc["Tcw"][0] = [1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0]
    sc["K"] = base["K"].copy()
    sc["K"][0] = [1.0, 1.0, 0.0, 0.0]
    ref = _ref(sc)
    for i, inside in enumerate(expect):
        assert KT.prior(sc["Tcw"][0], sc["K"][0], None, W, H, sc["wpt"][i])[2] == inside, i
    assert ref["nbkps"][0] == sum(expect)
    _assert_same(_gpu(ctx, sc), ref)


def test_klt_tracking_refusals(ctx):
    torch = pytest.importorskip("torch")
    sc = _scene(7, [10, 10])
    pp, cp = _pyramids(ctx, sc)
    ft = api.FeatureTracker(ctx, 30, 0.01)
    out = dict(tracked=np.full((20, 2), 7, np.float32), status=np.full(20, 7, np.uint8), passes=np.full(20, 7, np.uint8),
               p3p_req=np.full(2, 7, np.uint8), nbgood=np.full(2, 7, np.int32), nbkps=np.full(2, 7, np.int32))
    for offs in ([0, 15, 10], [1, 10, 20]):
        with pytest.raises(api.Ov2Error, match="INVALID"):
            ft.klt_tracking(pp, cp, 9, 3, 30.0, 0.5, np.array(offs, np.int32), sc["Tcw"], sc["K"], sc["img_wh"], sc["px"],
                            sc["wpt"], sc["is3d"], out=out)
    with pytest.raises(api.Ov2Error, match="INVALID"):      # more frames than pyramid slots
        ft.klt_tracking(pp, cp, 9, 3, 30.0, 0.5, sc["offsets"], sc["Tcw"], sc["K"], sc["img_wh"], sc["px"], sc["wpt"], sc["is3d"],
                        first=1, out=out)
    with pytest.raises(api.Ov2Error, match="INVALID"):
        ft.klt_tracking(pp, cp, 33, 3, 30.0, 0.5, sc["offsets"], sc["Tcw"], sc["K"], sc["img_wh"], sc["px"], sc["wpt"], sc["is3d"],
                        out=out)
    assert (out["status"] == 7).all() and (out["nbkps"] == 7).all()
    d_offs = torch.from_numpy(sc["offsets"]).cuda()
    st = ctx.lib.ov2_klt_tracking(ctx.h, pp.h_, cp.h_, api.C.byref(api.KltParams(9, 30, float(np.float32(0.01)), 30.0, 0.5)), 0, 2,
                                  d_offs.data_ptr(), sc["Tcw"].ctypes.data, sc["K"].ctypes.data, None, sc["img_wh"].ctypes.data,
                                  sc["px"].ctypes.data, sc["wpt"].ctypes.data, sc["is3d"].ctypes.data, 3, 1,
                                  out["tracked"].ctypes.data, out["status"].ctypes.data, out["passes"].ctypes.data,
                                  out["p3p_req"].ctypes.data, out["nbgood"].ctypes.data, out["nbkps"].ctypes.data)
    assert st == 3 and (out["status"] == 7).all()
