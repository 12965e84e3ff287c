"""CPU ORACLE for the rectification path (CameraCalibration::rectifyImage).  TEST INFRASTRUCTURE ONLY.

Only tests/ and __graft_entry__.smoke() import this module.  The product path (ov2slam_b200/) never does.

The reference rectifies with cv::remap(img, rect, undist_map_x_, undist_map_y_, cv::INTER_LINEAR) and the default
BORDER_CONSTANT 0 (/root/reference/src/camera_calibration.cpp:233-241).  Its maps are CV_16SC2 + CV_16UC1 from
setUndistStereoMap (:141) or two CV_32FC1 from setUndistMap (:92).  As image_ref.py does for the other image operators, parity
is pinned to cv2 4.13.0 in two layers:

  remap_cv2()  - the reference's call, executed by the real library.
  remap_ref()  - a numpy restatement, pinned against remap_cv2() by tests/test_remap_oracle.py:
      float maps:      X32 = rint(x * 32) (half to even, int32; out of range / NaN -> INT_MIN), X = sat16(X32 >> 5), a = X32 & 31
                       (what cv::convertMaps(.., CV_16SC2) computes; cv::remap with float maps equals that path)
      fixed maps:      (X, Y) = map1, a = map2 & 31, b = (map2 >> 5) & 31
      s   = (32-a)(32-b) p(Y,X) + a(32-b) p(Y,X+1) + (32-a)b p(Y+1,X) + ab p(Y+1,X+1)       (p = 0 outside the image)
      out = clamp((32 s + 2^14) >> 15, 0, 255)
"""
from __future__ import annotations

import numpy as np

try:  # the restatement does not need cv2
    import cv2
except Exception:  # pragma: no cover
    cv2 = None


def fixed_from_float(mx: np.ndarray, my: np.ndarray):
    """(map1 int16 [H, W, 2], map2 uint16 [H, W]) as cv::convertMaps(mx, my, CV_16SC2) returns them."""
    def q(v):
        s = np.asarray(v, np.float32) * np.float32(32.0)
        ok = np.isfinite(s) & (s > -2147483648.0) & (s < 2147483648.0)
        r = np.where(ok, np.rint(np.where(ok, s, 0)), 0).astype(np.int64)
        return np.where(ok, r, -(1 << 31))
    qx, qy = q(mx), q(my)
    m1 = np.stack([np.clip(qx >> 5, -32768, 32767), np.clip(qy >> 5, -32768, 32767)], -1).astype(np.int16)
    m2 = ((qx & 31) | ((qy & 31) << 5)).astype(np.uint16)
    return m1, m2


def remap_ref(img: np.ndarray, map1: np.ndarray, map2: np.ndarray) -> np.ndarray:
    """cv::remap(img, out, map1, map2, INTER_LINEAR, BORDER_CONSTANT 0) on an 8-bit one-channel image.
    map1 / map2: int16 [H, W, 2] + uint16 [H, W] (CV_16SC2 + CV_16UC1) or float32 [H, W] x / y (CV_32FC1)."""
    img = np.asarray(img, np.uint8)
    if map1.dtype == np.float32:
        map1, map2 = fixed_from_float(map1, map2)
    X = map1[..., 0].astype(np.int64)
    Y = map1[..., 1].astype(np.int64)
    f = map2.astype(np.int64) & 1023
    a, b = f & 31, f >> 5
    h, w = img.shape

    def p(yy, xx):
        ok = (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
        return np.where(ok, img[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)].astype(np.int64), 0)

    s = (32 - a) * (32 - b) * p(Y, X) + a * (32 - b) * p(Y, X + 1) + (32 - a) * b * p(Y + 1, X) + a * b * p(Y + 1, X + 1)
    return np.clip((32 * s + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def remap_cv2(img: np.ndarray, map1: np.ndarray, map2: np.ndarray) -> np.ndarray:
    """The reference's call: cv::remap(img, rect, map_x, map_y, cv::INTER_LINEAR)."""
    cv2.setNumThreads(1)
    return cv2.remap(img, map1, map2, cv2.INTER_LINEAR)


# ------------------------------------------------------------------ synthetic rigs (numpy; no calibration files)
EUROC_LIKE = dict(K0=(458.654, 457.296, 367.215, 248.375), D0=(-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 0.0),
                  K1=(457.587, 456.134, 379.999, 255.238), D1=(-0.28368365, 0.07451284, -0.00010473, -3.55590700e-05, 0.0),
                  rvec=(0.0020, -0.0060, 0.0030), t=(-0.110074, 0.000399, -0.000853))
"""Intrinsics like EuRoC's cam0 / cam1 (752 x 480) and a slightly rotated right camera 11 cm to the side."""


def stereo_maps_cv2(w: int, h: int, rig: dict = EUROC_LIKE, m1type: int = 11, alpha: float = 0.0):
    """Rectification maps of both cameras as the reference's setupStereoCalibration builds them (cv::stereoRectify +
    cv::initUndistortRectifyMap per camera, src/ov2slam.cpp:342-395, camera_calibration.cpp:141), m1type 11 = CV_16SC2 or
    5 = CV_32FC1.  Returns [(map1, map2) left, (map1, map2) right]."""
    K0 = np.array([[rig["K0"][0], 0, rig["K0"][2]], [0, rig["K0"][1], rig["K0"][3]], [0, 0, 1]], np.float64)
    K1 = np.array([[rig["K1"][0], 0, rig["K1"][2]], [0, rig["K1"][1], rig["K1"][3]], [0, 0, 1]], np.float64)
    D0, D1 = np.array(rig["D0"], np.float64), np.array(rig["D1"], np.float64)
    R, _ = cv2.Rodrigues(np.array(rig["rvec"], np.float64))
    t = np.array(rig["t"], np.float64)
    R0, R1, P0, P1, _, _, _ = cv2.stereoRectify(K0, D0, K1, D1, (w, h), R, t, flags=cv2.CALIB_ZERO_DISPARITY, alpha=alpha)
    return [cv2.initUndistortRectifyMap(K0, D0, R0, P0, (w, h), m1type),
            cv2.initUndistortRectifyMap(K1, D1, R1, P1, (w, h), m1type)]


def radial_map_np(w: int, h: int, k1: float = 0.25, k2: float = 0.05, f: float | None = None, shift=(0.0, 0.0)):
    """A pinhole undistortion map computed in numpy alone (CV_32FC1 x / y): for every output pixel the distorted source
    position under radial coefficients k1, k2 (cv2 not needed).  Its outer pixels map outside the image."""
    f = f if f is not None else 0.6 * max(w, h)
    cx, cy = (w - 1) / 2.0, (h - 1) / 2.0
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    u, v = (xx - cx) / f, (yy - cy) / f
    r2 = u * u + v * v
    g = 1.0 + k1 * r2 + k2 * r2 * r2
    return ((u * g * f + cx + shift[0]).astype(np.float32), (v * g * f + cy + shift[1]).astype(np.float32))


def edge_maps(w, h, seed=0):
    """Float maps whose entries sit exactly on the last row / column, half a pixel beyond them, on -1 / -0.5, on exact halves
    of 1/32 (the rounding ties), far outside and NaN, mixed with ordinary entries."""
    rng = np.random.default_rng(seed)
    mx = rng.uniform(-3, w + 2, (h, w)).astype(np.float32)
    my = rng.uniform(-3, h + 2, (h, w)).astype(np.float32)
    special_x = np.array([w - 1, w - 1.5, w - 0.5, w, -1, -0.5, -1.5, 0, 1e9, -1e9, 40000, -40000, np.nan,
                          3 + 1 / 64, 3 + 3 / 64, 5 - 1 / 64], np.float32)
    special_y = np.array([h - 1, h - 1.5, h - 0.5, h, -1, -0.5, -1.5, 0, 3, 1e9, 2, -40000, 5,
                          7 + 1 / 64, 2 + 5 / 64, h - 1], np.float32)
    k = len(special_x)
    idx = rng.choice(w * h, size=(8, k), replace=False)
    for r in range(8):
        mx.reshape(-1)[idx[r]] = special_x
        my.reshape(-1)[idx[r]] = np.roll(special_y, r)
    mx[0, :k], my[0, :k] = special_x, special_y
    mx[-1, -k:], my[-1, -k:] = special_x, special_y
    return mx, my
