"""CPU ORACLE for VisualFrontEnd::kltTracking (ov2_klt_tracking).  TEST INFRASTRUCTURE ONLY.

/root/reference/src/visual_front_end.cpp:132-275 restated per frame of a ragged batch, composed from the fbKltTracking oracle
(image_ref.fb_klt_ref, or fb_klt_cv2 for the same flow around cv2.calcOpticalFlowPyrLK) and match_ref's projection:

  prior    Frame::projWorldToImageDist (src/frame.cpp:825-828): match_ref.camera_point (Tcw * X, each row summed left to
           right) and match_ref.project_dist (pinhole, or cv::projectPoints on the float-rounded normalised point).  The
           reference does not test z, so a point behind the camera whose projection lands in the image gets a prior.  A point
           with z == 0 projects to inf / nan in IEEE arithmetic, which no image contains.
  in image Frame::isInImage (src/frame.cpp:840-843): float coordinates against the int image size.
  pass 1   3-D keypoints with an in-image prior, tracked from it at depth 1 (:189-199), when use_prior.
  rule     nbgood < 0.33 * nbkps raises the P3P request and resets the retries' priors to their own position (:228-233).
  pass 2   2-D keypoints, 3-D keypoints without an in-image prior and failed pass-1 keypoints at depth nklt_pyr_lvl (:235-252).

fbKltTracking tracks every keypoint independently, so a pass over a frame's members in index order gives the same per-keypoint
results as the reference's order (the failed pass-1 keypoints appended after the others).  A keypoint with x < 0 is an empty
slot of the batch (ov2_fb_klt's rule): never tracked, pass 0, status 0, tracked = px.

PINNING STATUS: the flow against the same flow around cv2.calcOpticalFlowPyrLK (tests/test_oracle_klt_tracking.py).  The
reference's own VisualFrontEnd::kltTracking is not compiled in place (DESIGN.md section 5).
"""
from __future__ import annotations

import numpy as np

from oracle import image_ref as R
from oracle import match_ref as M

f32 = np.float32


def prior(T, K, dist, img_w: int, img_h: int, wpt):
    """(x, y, in_image) of the world point's projection into the frame (float32 pixel)."""
    X, Y, Z = M.camera_point(T, wpt)
    if Z == 0.0:
        return f32(np.nan), f32(np.nan), False
    with np.errstate(over="ignore", invalid="ignore"):
        x, y = M.project_dist((X, Y, Z), K, dist)
    inside = bool(x >= 0 and y >= 0 and x < f32(img_w) and y < f32(img_h))
    return x, y, inside


def klt_tracking_ref(prevs, curs, offsets, Tcw, K, img_wh, px, wpt, is3d, dist=None, win=9, nklt_pyr_lvl=3, use_prior=True,
                     ferr=30.0, fb_dist=0.5, maxit=30, eps=R.KLT_EPS, first=0, fb=R.fb_klt_ref):
    """Frames [first, first + count) of the image lists prevs / curs.  Returns dict(tracked float32[n, 2], status uint8[n],
    passes uint8[n], p3p_req uint8[count], nbgood int32[count], nbkps int32[count])."""
    offsets = np.asarray(offsets, np.int64)
    count = len(offsets) - 1
    px = np.asarray(px, f32).reshape(-1, 2)
    wpt = np.asarray(wpt, np.float64).reshape(-1, 3)
    is3d = np.asarray(is3d).reshape(-1).astype(bool)
    n = len(px)
    tracked = px.copy()
    status = np.zeros(n, np.uint8)
    passes = np.zeros(n, np.uint8)
    p3p = np.zeros(count, np.uint8)
    nbgood = np.zeros(count, np.int32)
    nbkps = np.zeros(count, np.int32)
    Tcw = np.asarray(Tcw, np.float64).reshape(-1, 12)
    K = np.asarray(K, np.float64).reshape(-1, 4)
    img_wh = np.asarray(img_wh).reshape(-1, 2)

    def track(f, idx, pri, lvl):
        return fb(prevs[first + f], curs[first + f], px[idx], pri, win, lvl, ferr, fb_dist, maxit, eps)

    for f in range(count):
        idx = np.arange(offsets[f], offsets[f + 1])
        idx = idx[px[idx, 0] >= 0]
        d = None if dist is None else np.asarray(dist, np.float64).reshape(-1, 5)[f]
        mem1, pri1 = [], []
        if use_prior:
            for i in idx:
                if is3d[i]:
                    x, y, inside = prior(Tcw[f], K[f], d, int(img_wh[f, 0]), int(img_wh[f, 1]), wpt[i])
                    if inside:
                        mem1.append(i)
                        pri1.append((x, y))
        mem1 = np.array(mem1, np.int64)
        retry_prior = {}
        if len(mem1):
            tr1, st1 = track(f, mem1, np.array(pri1, f32), 1)
            nbgood[f], nbkps[f] = int(st1.sum()), len(mem1)
            p3p[f] = nbgood[f] < 0.33 * nbkps[f]
            for j, i in enumerate(mem1):
                if st1[j]:
                    tracked[i], status[i], passes[i] = tr1[j], 1, 1
                else:
                    retry_prior[i] = px[i] if p3p[f] else tr1[j]
        mem2 = np.array([i for i in idx if passes[i] != 1], np.int64)
        if len(mem2):
            pri2 = np.array([retry_prior.get(i, px[i]) for i in mem2], f32).reshape(-1, 2)
            tr2, st2 = track(f, mem2, pri2, nklt_pyr_lvl)
            tracked[mem2], status[mem2], passes[mem2] = tr2, st2, 2
    return dict(tracked=tracked, status=status, passes=passes, p3p_req=p3p, nbgood=nbgood, nbkps=nbkps)
