"""The stereoMatching oracle (oracle/stereo_matching_ref.py) pinned two ways:
  * undistort_points_ref against cv2.undistortPoints(pt, K, D, P=K), bit for bit, on EuRoC and KITTI coefficients, on strong
    distortion and on points where the iteration leaves through OpenCV's icdist < 0 exit;
  * the whole flow, run around cv2's tracker and cv2.getRectSubPix, against the REFERENCE'S OWN MapManager::stereoMatching
    compiled in place (oracle/_ref/libov2ref_map.so, or its outputs stored in tests/golden/reference_map.npz), on both branches:
    the same stereo keypoints, and right pixels within 1e-4 px."""
import ctypes as C

import numpy as np
import pytest

import stereo_scenes as SS
from oracle import image_ref as R
from oracle import stereo_matching_ref as S
from reference_golden import ReferenceOutputs

cv2 = pytest.importorskip("cv2")

CALIBS = {
    "euroc": ([458.654, 457.296, 367.215, 248.375], [-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 0.0]),
    "kitti": ([718.856, 718.856, 607.1928, 185.2157], [-0.3728755, 0.2037299, 0.002219027, 0.001383707, -0.07233722]),
    "strong": ([400.0, 410.0, 320.0, 240.0], [-0.9, 0.8, 0.01, -0.02, -0.5]),
}


def _first_icdist(u, v, K, D):
    x, y = (u - K[2]) / K[0], (v - K[3]) / K[1]
    r2 = x * x + y * y
    return 1.0 / (1 + ((D[4] * r2 + D[1]) * r2 + D[0]) * r2)


@pytest.mark.parametrize("calib", sorted(CALIBS))
def test_undistort_points_equals_cv2(calib):
    K, D = CALIBS[calib]
    rng = np.random.default_rng(len(calib))
    pts = np.stack([rng.uniform(-300, 1600, 4000), rng.uniform(-300, 900, 4000)], 1).astype(np.float32)
    pts[:4] = [[K[2], K[3]], [0, 0], [1279.5, 719.5], [np.float32(K[2]) + np.float32(1e-3), 0.25]]
    Km = np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1.0]])
    want = cv2.undistortPoints(pts.reshape(-1, 1, 2), Km, np.array(D), P=Km).reshape(-1, 2)
    got = np.array([S.undistort_points_ref(u, v, K, D) for u, v in pts], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    exits = np.array([_first_icdist(float(u), float(v), K, D) < 0 for u, v in pts])
    if calib == "strong":
        assert exits.sum() > 100                       # the icdist < 0 exit is taken, and equal too
    assert np.array_equal(np.array(S.undistort_points_ref(3.5, 7.25, K, None)), np.array([3.5, 7.25], np.float32))


@pytest.fixture(scope="module")
def lib():
    """The reference's outputs: live from the library where it is built, else as stored in tests/golden (read only here)."""
    from oracle.ref_build import build_map_ref, cv_callbacks as CB
    so = build_map_ref.build()
    handle = None
    if so is not None:
        handle = C.CDLL(str(so))
        cb = CB._Callbacks(*[C.cast(f, C.c_void_p) for f in CB._KEEP])
        handle.ov2ref_cv_set_callbacks(C.byref(cb))
    return ReferenceOutputs("map", handle)


@pytest.mark.parametrize("rect", [1, 0])
def test_stereo_matching_flow_equals_the_reference_source(lib, rect):
    """The reference's stereoMatching on a synthetic stereo keyframe (tests/stereo_scenes.py) over a textured pair 16 px apart, 260
    keypoints: the oracle's flow, around the same cv2 functions, makes the same keypoints stereo keypoints, with the same right
    pixels."""
    w, h, disp = 752, 480, 16.0
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    tex = lambda u: np.rint(128 + 50 * np.sin(0.11 * u + 0.07 * yy) + 40 * np.sin(0.05 * u - 0.13 * yy + 1) + 30 * np.sin(0.31 * u + 0.23 * yy + 2)).astype(np.uint8)
    left, right = tex(xx), tex(xx + disp)
    sc = SS.stereo_scene(91 + rect, rect, nkps=260, depth=458.654 * 0.11 / disp)
    lv_l, lv_r = [left], [right]
    for _ in range(3):
        lv_l.append(cv2.pyrDown(lv_l[-1]))
        lv_r.append(cv2.pyrDown(lv_r[-1]))
    n = len(sc["lmid"])
    D, I, U = C.POINTER(C.c_double), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)

    def live(L):
        PP = U * 4
        pl, pr = PP(*[a.ctypes.data_as(U) for a in lv_l]), PP(*[a.ctypes.data_as(U) for a in lv_r])
        rows, cols = np.array([a.shape[0] for a in lv_l], np.int32), np.array([a.shape[1] for a in lv_l], np.int32)
        order, st, rpx = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros((n, 2), np.float32)
        a = dict(K=np.ascontiguousarray(sc["K"], np.float64), rig=np.ascontiguousarray(np.concatenate([sc["trig"], SS.quat_of(sc["Rrig"])]), np.float64),
                 Twc=np.ascontiguousarray(np.concatenate([sc["twc"], SS.quat_of(sc["Rwc"])]), np.float64), lmid=np.ascontiguousarray(sc["lmid"], np.int32),
                 is3d=np.ascontiguousarray(sc["is3d"], np.int32), has=np.ascontiguousarray(sc["has_mp"], np.int32), px=np.ascontiguousarray(sc["px"], np.float32),
                 wpt=np.ascontiguousarray(sc["wpt"], np.float64))
        L.ov2ref_stereo_matching.restype = C.c_int
        m = L.ov2ref_stereo_matching(n, rect, a["K"].ctypes.data_as(D), a["K"].ctypes.data_as(D), a["rig"].ctypes.data_as(D), a["Twc"].ctypes.data_as(D), w, h, 35,
                                     a["lmid"].ctypes.data_as(I), a["is3d"].ctypes.data_as(I), a["has"].ctypes.data_as(I), a["px"].ctypes.data_as(C.POINTER(C.c_float)),
                                     a["wpt"].ctypes.data_as(D), pl, pr, rows.ctypes.data_as(I), cols.ctypes.data_as(I), order.ctypes.data_as(I),
                                     st.ctypes.data_as(I), rpx.ctypes.data_as(C.POINTER(C.c_float)))
        return dict(m=m, order=order, st=st, rpx=rpx)
    r = lib(f"stereo_matching{rect}", live)
    order, st, rpx = r["order"], r["st"], r["rpx"]
    assert int(r["m"]) == n
    fl = SS.flat_scene(sc, order)
    subpix = lambda src, ws, cx, cy: cv2.getRectSubPix(src, (ws, ws), (float(cx), float(cy)))
    out = S.stereo_matching_ref([left], [right], fl.pop("offsets"), fl.pop("Tcw"), fl.pop("K"), fl.pop("Trl"), fl.pop("img_wh"),
                                fl.pop("px"), fl.pop("unpx"), fl.pop("bv"), fl.pop("is3d"), fl.pop("has_mp"), fl.pop("wpt"),
                                fl.pop("rectified"), fb=R.fb_klt_cv2, subpix=subpix, sad_levels=lambda k: (lv_l[3], lv_r[3]), **fl)
    got = out["stereo"].astype(bool)
    want = st.astype(bool)
    assert np.array_equal(got, want) and want.sum() > 0.6 * len(order)
    assert np.abs(out["right"][want] - rpx[want]).max() <= 1e-4
    assert out["nstereo"][0] == want.sum()
    if rect:
        assert ((out["passes"] == 2) & got).any()      # row-search priors made stereo keypoints
    assert ((out["passes"] == 1) & got).any() and (out["passes"] == 0).sum() == int((sc["is3d"] & ~sc["has_mp"]).sum())
