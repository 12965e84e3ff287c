"""CPU ORACLE for MapManager::stereoMatching (ov2_stereo_matching).  TEST INFRASTRUCTURE ONLY.

/root/reference/src/map_manager.cpp:367-611 restated per keyframe of a ragged batch, composed from the fbKltTracking oracle
(image_ref.fb_klt_ref, or the same flow around cv2.calcOpticalFlowPyrLK), the getLineMinSAD oracle (image_ref.line_min_sad_ref),
klt_tracking_ref's projection and the two restatements below, every double formed in the kernel's order:

  prior    a 3-D keypoint with a map point: Frame::projWorldToRightImageDist (src/frame.cpp:835-838), Tcw then
           right_prior (klt_tracking_ref.prior) through Trl with the right camera and Frame::isInRightImage (:845-848).  A 3-D
           keypoint without a map point is dropped: pass 0, no stereo.
  rect     the remaining keypoints' row search on level nklt_pyr_lvl (window 7, leftwards) at px * downpyrcoef; the column
           times uppyrcoef (float) replaces the prior's x iff 0 <= x <= px.x (:421-436).
  other    the remaining keypoints' neighbour-depth prior (:438-483) over Frame::getSurroundingKeypoints (src/frame.cpp:594-622):
           cells (rk-1..rk) x (ck-1..ck) in loop order, then list order, the keypoint itself skipped; a cell with r < 0, c < 0
           or idx >= the keyframe's cell count is skipped (the reference's .at() throws at idx == size).  Weights
           1 / cv::norm(unpx_j - unpx) (float difference, double squares); IEEE semantics, so equal unpx give a NaN prior.
  pass 1   the keypoints with an in-image prior at depth 1 (fbKltTracking clamps it as :503-505 do).
  pass 2   the other kept keypoints from their prior and the failed pass-1 keypoints from their forward result, at depth
           nklt_pyr_lvl (:531-535, :545-576).
  gate     undistort_points_ref of the right pixel; rectified: |lun.y - run.y| in float, then y := lun.y; other rigs:
           sampson_ref.  A stereo match iff the error is <= 2 (:583-603).

fbKltTracking and getLineMinSAD treat every keypoint independently, so one pass over a keyframe's members in index order
gives the reference's per-keypoint results.

PINNING STATUS: undistort_points_ref equals cv2.undistortPoints bit for bit (tests/test_oracle_stereo_matching.py, EuRoC and
KITTI coefficients, strong distortion, the icdist < 0 exit).  The flow, run around cv2's tracker and cv2.getRectSubPix, gives
the stereo keypoints and the right pixels (within 1e-4 px) of the reference's own stereoMatching compiled in place, on both
branches (golden tests/golden/reference_map.npz, calls stereo_matching0 / stereo_matching1).
"""
from __future__ import annotations

import numpy as np

from oracle import image_ref as R
from oracle import klt_tracking_ref as KT
from oracle import match_ref as M

f32 = np.float32
SAD_WIN = 7

# Frame::projCamToRightImageDist and isInRightImage: the camera point through Trl into the right camera, the projection and
# in-image test of klt_tracking_ref.prior.
right_prior = KT.prior


def undistort_points_ref(u, v, K, dist):
    """CameraCalibration::undistortImagePoint, pinhole: cv::undistortPoints([(u, v)], K, D, K) with the default criteria
    (5 iterations, no tolerance test), D = (k1, k2, p1, p2, k3); the pixel itself when dist is None.  float32 (x, y)."""
    if dist is None:
        return f32(u), f32(v)
    fx, fy, cx, cy = (float(a) for a in K)
    k1, k2, p1, p2, k3 = (float(a) for a in dist)
    ifx, ify = 1.0 / fx, 1.0 / fy
    x0, y0 = (float(f32(u)) - cx) * ifx, (float(f32(v)) - cy) * ify
    x, y = x0, y0
    for _ in range(5):
        r2 = x * x + y * y
        icdist = 1.0 / (1 + ((k3 * r2 + k2) * r2 + k1) * r2)
        if icdist < 0:
            x, y = x0, y0
            break
        dx = 2 * p1 * x * y + p2 * (r2 + 2 * x * x)
        dy = p1 * (r2 + 2 * y * y) + 2 * p2 * x * y
        x = (x0 - dx) * icdist
        y = (y0 - dy) * icdist
    return f32(fx * x + cx), f32(fy * y + cy)


def sampson_ref(F, l, r):
    """MultiViewGeometry::computeSampsonDistance(Frl, lun, run) (src/multi_view_geometry.cpp:798-821): the products in double,
    r^T F before the product with l, each result rounded to float, the rest in float."""
    F = [float(a) for a in np.asarray(F, np.float64).reshape(9)]
    lx, ly, rx, ry = float(l[0]), float(l[1]), float(r[0]), float(r[1])
    t0 = rx * F[0] + ry * F[3] + F[6]
    t1 = rx * F[1] + ry * F[4] + F[7]
    t2 = rx * F[2] + ry * F[5] + F[8]
    num = f32(t0 * lx + t1 * ly + t2)
    num = num * num
    x1, y1 = f32(t0), f32(t1)
    x2, y2 = f32(F[0] * lx + F[1] * ly + F[2]), f32(F[3] * lx + F[4] * ly + F[5])
    den = x1 * x1 + y1 * y1 + x2 * x2 + y2 * y2
    return np.sqrt(num / den)


def neighbour_depth(f, i, o0, o1, Tcw, px, unpx, is3d, has_mp, wpt, cell_offsets, grid, cell_ptr, cell_kps):
    """The weighted mean depth of keypoint i's 3-D neighbours (map_manager.cpp:438-471), or None without one."""
    ncs, nbw = int(grid[f][0]), int(grid[f][1])
    c0, ncells = int(cell_offsets[f]), int(cell_offsets[f + 1] - cell_offsets[f])
    rk, ck = int(np.floor(px[i, 1] / f32(ncs))), int(np.floor(px[i, 0] / f32(ncs)))
    with np.errstate(all="ignore"):
        return _neighbour_sum(f, i, o0, o1, Tcw, rk, ck, nbw, c0, ncells, unpx, is3d, has_mp, wpt, cell_ptr, cell_kps)


def _neighbour_sum(f, i, o0, o1, Tcw, rk, ck, nbw, c0, ncells, unpx, is3d, has_mp, wpt, cell_ptr, cell_kps):
    zsum, wsum, used = np.float64(0), np.float64(0), False
    for r in (rk - 1, rk):
        for c in (ck - 1, ck):
            idx = r * nbw + c
            if r < 0 or c < 0 or idx >= ncells:
                continue
            for q in range(max(int(cell_ptr[c0 + idx]), o0), min(int(cell_ptr[c0 + idx + 1]), o1)):
                j = int(cell_kps[q])
                if j == i or j < o0 or j >= o1 or not is3d[j] or not has_mp[j]:
                    continue
                d = unpx[j] - unpx[i]                                    # float32 difference
                coef = np.float64(1.0) / np.sqrt(np.float64(d[0]) * np.float64(d[0]) + np.float64(d[1]) * np.float64(d[1]))
                wsum = wsum + coef
                zsum = zsum + coef * np.float64(M.camera_point(Tcw, wpt[j])[2])
                used = True
    return float(zsum / wsum) if used else None


def stereo_matching_ref(lefts, rights, offsets, Tcw, K, Trl, img_wh, px, unpx, bv, is3d, has_mp, wpt, rectified, dist=None,
                        Frl=None, cell_offsets=None, grid=None, cell_ptr=None, cell_kps=None, win=9, nklt_pyr_lvl=3, ferr=30.0,
                        fb_dist=0.5, maxit=30, eps=R.KLT_EPS, first=0, fb=R.fb_klt_ref, subpix=R.get_rect_subpix_u8_ref,
                        sad_levels=None):
    """Keyframes [first, first + count) of the image lists lefts / rights.  sad_levels(k) -> (left, right) images of level
    nklt_pyr_lvl of keyframe slot k (default: image_ref.pyr_down_ref).  Returns dict(right float32[n, 2], stereo uint8[n],
    passes uint8[n], nstereo int32[count], epi float32[n] and run float32[n, 2]: the
    epipolar error and the undistorted right pixel of each gated track, NaN elsewhere)."""
    offsets = np.asarray(offsets, np.int64)
    count = len(offsets) - 1
    px = np.asarray(px, f32).reshape(-1, 2)
    unpx = np.asarray(unpx, f32).reshape(-1, 2)
    bv = np.asarray(bv, np.float64).reshape(-1, 3)
    wpt = np.asarray(wpt, np.float64).reshape(-1, 3)
    is3d = np.asarray(is3d).reshape(-1).astype(bool)
    has_mp = np.asarray(has_mp).reshape(-1).astype(bool)
    Tcw = np.asarray(Tcw, np.float64).reshape(-1, 12)
    Trl = np.asarray(Trl, np.float64).reshape(-1, 12)
    K = np.asarray(K, np.float64).reshape(-1, 4)
    img_wh = np.asarray(img_wh).reshape(-1, 2)
    n = len(px)
    right = px.copy()
    stereo = np.zeros(n, np.uint8)
    passes = np.zeros(n, np.uint8)
    nstereo = np.zeros(count, np.int32)
    epi = np.full(n, np.nan, f32)
    runpx = np.full((n, 2), np.nan, f32)
    up = f32(2.0 ** nklt_pyr_lvl)
    down = f32(1.0 / float(up))

    def levels(k):
        if sad_levels is not None:
            return sad_levels(k)
        return tuple(R.build_pyramid_ref(im, nklt_pyr_lvl)[nklt_pyr_lvl] for im in (lefts[k], rights[k]))

    for f in range(count):
        o0, o1 = int(offsets[f]), int(offsets[f + 1])
        d = None if dist is None else np.asarray(dist, np.float64).reshape(-1, 5)[f]
        w, h = int(img_wh[f, 0]), int(img_wh[f, 1])
        mem1, pri1, blind = [], [], []
        for i in range(o0, o1):
            if not (px[i, 0] >= 0) or (is3d[i] and not has_mp[i]):
                continue
            if is3d[i]:
                x, y, inside = right_prior(Trl[f], K[f], d, w, h, M.camera_point(Tcw[f], wpt[i]))
                if inside:
                    mem1.append(i)
                    pri1.append((x, y))
                    continue
            if not rectified:
                depth = neighbour_depth(f, i, o0, o1, Tcw[f], px, unpx, is3d, has_mp, wpt, cell_offsets, grid, cell_ptr, cell_kps)
                if depth is not None:
                    with np.errstate(all="ignore"):
                        b = bv[i]
                        campt = (depth * (b[0] / b[2]), depth * (b[1] / b[2]), depth * (b[2] / b[2]))
                        x, y, inside = right_prior(Trl[f], K[f], d, w, h, campt)
                    if inside:
                        mem1.append(i)
                        pri1.append((x, y))
                        continue
            blind.append(i)
        retry = {i: px[i].copy() for i in blind}
        if rectified and blind:
            iml, imr = levels(first + f)
            for i in blind:
                xp = f32(R.line_min_sad_ref(iml, imr, (px[i, 0] * down, px[i, 1] * down), SAD_WIN, True, subpix=subpix)[0]) * up
                if xp >= 0 and xp <= px[i, 0]:
                    retry[i][0] = xp
        ok = {}
        if mem1:
            tr1, st1 = fb(lefts[first + f], rights[first + f], px[mem1], np.array(pri1, f32), win, 1, ferr, fb_dist, maxit, eps)
            for j, i in enumerate(mem1):
                if st1[j]:
                    right[i], passes[i], ok[i] = tr1[j], 1, True
                else:
                    retry[i] = tr1[j]
        mem2 = sorted(retry)
        if mem2:
            pri2 = np.array([retry[i] for i in mem2], f32).reshape(-1, 2)
            tr2, st2 = fb(lefts[first + f], rights[first + f], px[mem2], pri2, win, nklt_pyr_lvl, ferr, fb_dist, maxit, eps)
            for j, i in enumerate(mem2):
                right[i], passes[i] = tr2[j], 2
                if st2[j]:
                    ok[i] = True
        for i in sorted(ok):
            run = undistort_points_ref(right[i, 0], right[i, 1], K[f], d)
            runpx[i] = run
            with np.errstate(all="ignore"):
                if rectified:
                    err = abs(f32(unpx[i, 1] - run[1]))
                    right[i, 1] = unpx[i, 1]
                else:
                    err = sampson_ref(np.asarray(Frl, np.float64).reshape(-1, 9)[f], unpx[i], run)
            epi[i] = err
            if err <= 2.0:
                stereo[i] = 1
                nstereo[f] += 1
    return dict(right=right, stereo=stereo, passes=passes, nstereo=nstereo, epi=epi, run=runpx)
