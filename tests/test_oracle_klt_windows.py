"""CPU test: oracle/image_ref.py::fb_klt_ref (the exact-integer restatement of calcOpticalFlowPyrLK the GPU trackers are
checked against bit for bit) against cv2.calcOpticalFlowPyrLK through the reference's fbKltTracking sequence, for every
window size from 3 to 31, at depths 0 - 3, with keypoints near every border.

Statuses must be identical.  Positions differ where cv2 adds its float32 window sums in its SIMD lane order instead of
forming them exactly (DESIGN §5); the difference and the share of bit-equal positions are bounded by what was measured
here (the share falls as the window grows, because a larger window has more terms to round)."""
import numpy as np
import pytest

from ov2slam_b200 import synth
from oracle import image_ref as R

pytestmark = pytest.mark.skipif(not R.HAVE_CV2, reason="cv2 not importable")

MAX_ABS_DIFF_PX = 2e-3        # largest |oracle - cv2| position difference at any window (measured 1.06e-3, DESIGN §5)
MIN_BIT_EQUAL = 0.8           # smallest share of bit-equal tracked positions at any window (measured 0.828, at 24)


@pytest.fixture(scope="module")
def pair():
    w, h = 320, 240
    prev, cur, flow = synth.make_pair(77, w, h)
    rng = np.random.default_rng(77)
    kps = np.stack([rng.uniform(0, w, 40), rng.uniform(0, h, 40)], 1).astype(np.float32)
    kps[:8] = [[0.5, 0.5], [w - 1.0, 3.0], [2.0, h - 1.5], [w - 2.5, h - 2.5], [1.0, 120.0], [w - 1.0, 60.0],
               [160.0, 0.25], [100.0, h - 0.5]]
    pri = (kps + flow + rng.normal(0, 1.0, kps.shape)).astype(np.float32)
    return prev, cur, kps, pri


@pytest.mark.parametrize("win", list(range(3, 32)))
def test_oracle_equals_cv2_statuses_every_window(pair, win):
    prev, cur, kps, pri = pair
    diffs, equal, tracked = [], 0, 0
    for lvl in range(4):
        rp, rs = R.fb_klt_ref(prev, cur, kps, pri, win, lvl)
        cp, cs = R.fb_klt_cv2(prev, cur, kps, pri, win, lvl)
        assert np.array_equal(rs, cs), (win, lvl, np.nonzero(rs != cs)[0])
        ok = rs == 1
        diffs.append(np.abs(rp[ok] - cp[ok]).max(initial=0.0))
        equal += int((rp[ok] == cp[ok]).all(axis=1).sum())
        tracked += int(ok.sum())
    assert tracked >= 40, tracked            # of 160 tracks (40 keypoints x 4 depths); 42 at the 3 x 3 window
    assert max(diffs) <= MAX_ABS_DIFF_PX, max(diffs)
    assert equal / tracked >= MIN_BIT_EQUAL, equal / tracked
