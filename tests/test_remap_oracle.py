"""oracle/remap_ref.py: the numpy restatement of cv::remap (INTER_LINEAR, BORDER_CONSTANT 0) that the rectification kernel is
checked against, pinned bit for bit to cv2.remap on the maps the reference builds (CameraCalibration::rectifyImage)."""
import numpy as np
import pytest

from oracle import remap_ref as RR

cv2 = pytest.importorskip("cv2")


def _img(w, h, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    smooth = 128 + 60 * np.sin(xx / 7.0) * np.cos(yy / 11.0)
    return np.clip(smooth + rng.normal(0, 25, (h, w)), 0, 255).astype(np.uint8)


@pytest.mark.parametrize("size", [(752, 480), (1241, 376), (333, 217)])
@pytest.mark.parametrize("m1type", [11, 5])
@pytest.mark.parametrize("alpha", [0.0, 1.0])
def test_remap_ref_equals_cv2_on_stereo_rectification_maps(size, m1type, alpha):
    """cv2.stereoRectify + initUndistortRectifyMap of a distorted, rotated rig (CV_16SC2 + CV_16UC1 as setUndistStereoMap builds
    them, and CV_32FC1): both cameras, bit-exact; alpha 1 keeps the whole source view, so many outputs read outside the image."""
    w, h = size
    img = _img(w, h, w + h)
    for m1, m2 in RR.stereo_maps_cv2(w, h, m1type=m1type, alpha=alpha):
        assert np.array_equal(RR.remap_ref(img, m1, m2), RR.remap_cv2(img, m1, m2))


@pytest.mark.parametrize("alpha", [0.0, 1.0])
def test_remap_ref_equals_cv2_on_fisheye_and_undistortion_maps(alpha):
    """A cv2.fisheye map (the reference's Fisheye model, camera_calibration.cpp:97,145) and a pinhole setUndistMap-style
    CV_32FC1 map from getOptimalNewCameraMatrix."""
    w, h = 752, 480
    img = _img(w, h, 3)
    K = np.array([[380.0, 0, 376.0], [0, 380.0, 240.0], [0, 0, 1]])
    D = np.array([-0.01, 0.02, -0.005, 0.001])
    newK = cv2.fisheye.estimateNewCameraMatrixForUndistortRectify(K, D, (w, h), np.eye(3), balance=alpha)
    for t in (cv2.CV_16SC2, cv2.CV_32FC1):
        m1, m2 = cv2.fisheye.initUndistortRectifyMap(K, D, np.eye(3), newK, (w, h), t)
        assert np.array_equal(RR.remap_ref(img, m1, m2), RR.remap_cv2(img, m1, m2))
    K0 = np.array([[458.654, 0, 367.215], [0, 457.296, 248.375], [0, 0, 1]])
    D0 = np.array(RR.EUROC_LIKE["D0"])
    nK, _ = cv2.getOptimalNewCameraMatrix(K0, D0, (w, h), alpha, (w, h))
    mx, my = cv2.initUndistortRectifyMap(K0, D0, None, nK, (w, h), cv2.CV_32FC1)
    assert np.array_equal(RR.remap_ref(img, mx, my), RR.remap_cv2(img, mx, my))
    assert np.array_equal(RR.fixed_from_float(mx, my)[0], cv2.convertMaps(mx, my, cv2.CV_16SC2)[0])
    assert np.array_equal(RR.fixed_from_float(mx, my)[1], cv2.convertMaps(mx, my, cv2.CV_16SC2)[1])


@pytest.mark.parametrize("size", [(333, 217), (64, 48)])
def test_remap_ref_equals_cv2_on_edge_entries(size):
    w, h = size
    img = _img(w, h, 7)
    img[-1, :] = 255
    img[:, -1] = 201
    mx, my = RR.edge_maps(w, h)
    assert np.array_equal(RR.remap_ref(img, mx, my), RR.remap_cv2(img, mx, my))
    m1, m2 = cv2.convertMaps(mx, my, cv2.CV_16SC2)
    assert np.array_equal(RR.remap_ref(img, m1, m2), RR.remap_cv2(img, m1, m2))


def test_numpy_radial_map_equals_cv2():
    """The cv2-free map smoke() uses: remap_ref equals cv2.remap on it, and some of its outputs read outside the image."""
    w, h = 320, 240
    img = _img(w, h, 9)
    mx, my = RR.radial_map_np(w, h)
    assert ((mx < -1) | (mx > w)).any()
    assert np.array_equal(RR.remap_ref(img, mx, my), RR.remap_cv2(img, mx, my))
