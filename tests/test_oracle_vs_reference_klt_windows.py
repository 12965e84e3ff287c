"""FeatureTracker::fbKltTracking as the reference writes it (oracle/_ref/libov2ref_frontend.so: src/feature_tracker.cpp compiled in
place, its calcOpticalFlowPyrLK answered by the real OpenCV through callbacks) at window sizes other than 9: 5, 15, 21 and the even
sizes 4 and 10.  The reference's own orchestration (depth clamp against the pyramid's entries, forward track from the priors, the
minEig / ferr filter whose divisor depends on the window, the border test, the level-0 backward track, the forward-backward distance)
must equal the oracle's composition oracle/image_ref.py::_fb_klt around the same cv2 call bit for bit, and the exact-integer
composition fb_klt_ref, which the GPU tracker equals bit for bit, must give the same statuses and positions within the bound of
DESIGN §5.

Without the reference tree the library's outputs come from tests/golden/reference_klt_windows.npz, written by
scripts/make_golden_klt_windows.py from the cases below."""
import ctypes as C

import numpy as np
import pytest

from oracle import image_ref as R
from ov2slam_b200 import synth
from reference_golden import ReferenceOutputs

cv2 = pytest.importorskip("cv2")

MAX_ABS_DIFF_PX = 2e-3        # exact-integer vs cv2 float window sums, as tests/test_oracle_klt_windows.py bounds it

# (w, h, nwinsize, nbpyrlvl, pyramid entries the caller holds): 96 x 72 at 21 is an image whose levels the window outgrows,
# 4 entries clamp nbpyrlvl 3 to 1 (feature_tracker.cpp:50-52)
CASES = [(640, 480, 5, 3, 8), (640, 480, 4, 1, 8), (752, 480, 10, 3, 8), (640, 480, 15, 3, 4), (640, 480, 21, 3, 8),
         (96, 72, 21, 3, 8)]


def case_inputs(w, h, win):
    prev, cur, flow = synth.make_pair(80 + win, w, h)
    rng = np.random.default_rng(win)
    n = 160
    kps = np.stack([rng.uniform(0, w, n), rng.uniform(0, h, n)], 1).astype(np.float32)
    kps[:6] = [[0.5, 0.5], [w - 1.2, h - 1.2], [3, h / 2], [w / 2, 2], [w - 3, 10], [20, h - 2.5]]      # border points
    pri = (kps + np.asarray(flow, np.float32) + rng.normal(0, 1.5, (n, 2))).astype(np.float32)
    return prev, cur, kps, pri


def case_key(w, h, win, nbpyrlvl, entries):
    return f"fb_klt_{w}x{h}_win{win}_{nbpyrlvl}_{entries}"


def reference_call(rec, w, h, win, nbpyrlvl, entries):
    """The reference's fbKltTracking on one case: live where the library is built, else as stored."""
    prev, cur, kps, pri = case_inputs(w, h, win)
    n = len(kps)

    def live(lib):
        from oracle.ref_build import cv_callbacks as CB
        got_pri, st = pri.copy(), np.zeros(n, np.uint8)
        m = lib.ov2ref_ft_fb_klt(prev.ctypes.data_as(CB.U8P), cur.ctypes.data_as(CB.U8P), h, w, entries, win, nbpyrlvl,
                                 C.c_float(30.0), C.c_float(0.5), 30, C.c_float(0.01), kps.ctypes.data_as(CB.F32P),
                                 got_pri.ctypes.data_as(CB.F32P), n, st.ctypes.data_as(CB.U8P))
        return dict(m=m, pri=got_pri, st=st)
    return rec(case_key(w, h, win, nbpyrlvl, entries), live)


@pytest.fixture(scope="module")
def ref():
    from oracle.ref_build import cv_callbacks as CB
    rec = ReferenceOutputs("klt_windows", CB.load())
    yield rec
    rec.save()


@pytest.mark.parametrize("w,h,win,nbpyrlvl,entries", CASES)
def test_fb_klt_tracking_windows_equal_the_reference_source(ref, w, h, win, nbpyrlvl, entries):
    prev, cur, kps, pri = case_inputs(w, h, win)
    r = reference_call(ref, w, h, win, nbpyrlvl, entries)
    got_pri, st = r["pri"], r["st"]
    assert int(r["m"]) == len(kps)
    eff = min(nbpyrlvl, entries // 2 - 1)                     # the reference's clamp to the pyramid it is given
    want_pri, want_st = R._fb_klt(R._lk_cv2, prev, cur, kps, pri, win, eff, 30.0, 0.5, 30, R.KLT_EPS)
    assert np.array_equal(st, want_st) and 0.3 < st.mean() < 1.0, st.mean()
    assert np.array_equal(got_pri.view(np.uint32), want_pri.view(np.uint32))
    ref_pri, ref_st = R.fb_klt_ref(prev, cur, kps, pri, win, eff)
    assert np.array_equal(ref_st, st), np.nonzero(ref_st != st)[0]
    both = st > 0
    assert np.abs(ref_pri[both] - got_pri[both]).max() <= MAX_ABS_DIFF_PX
