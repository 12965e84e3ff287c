"""CPU test: oracle/klt_tracking_ref.py::klt_tracking_ref (VisualFrontEnd::kltTracking composed from fb_klt_ref, which
ov2_klt_tracking is checked against bit for bit) against the same flow around cv2.calcOpticalFlowPyrLK (fb_klt_cv2, the
fbKltTracking orchestration pinned to the reference's own feature_tracker.cpp).

Passes, P3P requests, pass-1 counts and statuses must be identical; tracked positions of tracked keypoints may differ by the
fbKltTracking oracle's stated bound against cv2 (5.6e-3 px, DESIGN §5: cv2 adds its float32 window sums in SIMD lane order)."""
import numpy as np
import pytest

from ov2slam_b200 import synth
from oracle import image_ref as R
from oracle import klt_tracking_ref as KT

pytestmark = pytest.mark.skipif(not R.HAVE_CV2, reason="cv2 not importable")

KLT_BOUND_PX = 5.6e-3


def _both(sc, **kw):
    args = (sc["prevs"], sc["curs"], sc["offsets"], sc["Tcw"], sc["K"], sc["img_wh"], sc["px"], sc["wpt"], sc["is3d"])
    return KT.klt_tracking_ref(*args, dist=sc["dist"], **kw), KT.klt_tracking_ref(*args, dist=sc["dist"], fb=R.fb_klt_cv2, **kw)


@pytest.mark.parametrize("use_prior", [True, False])
@pytest.mark.parametrize("distorted", [False, True])
@pytest.mark.parametrize("win", [9, 15])
def test_oracle_equals_cv2_flow(win, distorted, use_prior):
    sc = synth.make_klt_tracking_scene(60 + win, [45, 0, 30, 38], 320, 240, distorted=distorted)
    ref, cv = _both(sc, win=win, use_prior=use_prior)
    for k in ("passes", "status", "p3p_req", "nbgood", "nbkps"):
        assert np.array_equal(ref[k], cv[k]), (k, np.nonzero(ref[k] != cv[k])[0][:20])
    ok = ref["status"] == 1
    assert ok.sum() >= 60, ok.sum()
    assert np.abs(ref["tracked"][ok] - cv["tracked"][ok]).max(initial=0.0) <= KLT_BOUND_PX
    if use_prior:
        assert (ref["passes"] == 1).any() and ((ref["passes"] == 2) & sc["is3d"].astype(bool)).any()


def test_oracle_p3p_request_resets_retry_priors():
    """A frame whose priors are all bad: fewer than a third of pass 1 tracks, so the retries start from their own position."""
    sc = synth.make_klt_tracking_scene(71, [60], 320, 240, frac3d=1.0, bad_frac=1.0)
    ref, cv = _both(sc)
    assert ref["p3p_req"][0] == 1 and cv["p3p_req"][0] == 1
    assert ref["nbgood"][0] < 0.33 * ref["nbkps"][0]
    assert np.array_equal(ref["status"], cv["status"])


def test_prior_projection_and_in_image():
    """The prior is match_ref's projection; isInImage compares the float pixel against the int image size."""
    T = [1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0]
    K = [1.0, 1.0, 0.0, 0.0]
    assert KT.prior(T, K, None, 320, 240, (0.0, 5.0, 1.0))[2]
    assert not KT.prior(T, K, None, 320, 240, (320.0, 5.0, 1.0))[2]
    assert KT.prior(T, K, None, 320, 240, (-319.0, -5.0, -1.0))[:2] == (np.float32(319.0), np.float32(5.0))   # behind the camera
    assert not KT.prior(T, K, None, 320, 240, (1.0, 1.0, 0.0))[2]                                              # z == 0
