"""CPU ORACLE for Mapper::matchToMap (local-map matching).  TEST INFRASTRUCTURE ONLY.

Last "next" row of the scope table (SURVEY.md 8f-4): /root/reference/src/mapper.cpp:576-774 restated on the FLATTENED
arrays ov2_match_to_map takes (the map walking that produces them is the host shim's job):

  projection                 Frame::projWorldToCam + CameraCalibration::projectCamToImageDist
                             (src/frame.cpp:811-828, src/camera_calibration.cpp:254-281): pinhole, or pinhole +
                             cv::projectPoints on the float-rounded normalised point for a radial-tangential model
                             (restated from OpenCV's cvProjectPoints2Internal; pinned against cv2.projectPoints by
                             tests/test_oracle_match.py); fisheye is not restated
  culling                    depth < 0.1, |z / norm| < cos(max half fov), outside the image (:618-637)
  candidate keypoints        Frame::getSurroundingKeypoints(pt) (src/frame.cpp:624-650): the FOUR cells
                             (r-1 .. r) x (c-1 .. c) around the projection, cell lists in insertion order
  per candidate              pixel distance, "never observed together" (keyframe sets disjoint), mean co-projection
                             error of the map point into the keyframes that observe the keypoint's map point,
                             minimal Hamming distance over all descriptor pairs (src/map_point.cpp:236-252) (:654-724)
  best / second, 0.9 ratio   (:726-744)
  per keypoint               the candidate with the smallest distance, later candidates win ties (:758-772)

The reference iterates an unordered_set of map-point ids; the order of `cand_mp` is used here (and by the kernel).
Every double is formed in the kernel's operation order (csrc/match_map.cu, built with -fmad=false): each row of the
camera-frame point is the left-to-right sum T0*w0 + T1*w1 + T2*w2 + T9 of Python doubles (IEEE, no contraction), the
norm is sqrt(X*X + Y*Y + Z*Z) left to right, and float steps round through numpy float32.  Division and sqrt are correctly
rounded on both sides, so the oracle reproduces the kernel bit for bit: every output is compared for equality, and a
test can put a value exactly on a threshold.  The reference goes through Sophus' quaternion product instead: last-bit
differences in the camera-frame point against it.

PINNING STATUS: the distortion model is pinned against cv2; the flow against the reference's own Mapper::matchToMap (src/mapper.cpp
compiled in place with the reference's Frame / MapManager / MapPoint, oracle/ref_build/build_map_ref.py) on maps built from flattened
scenes with an undistorted calibration: the same pairs for the same candidate order (tests/test_oracle_vs_reference_map.py); hand-built
cases in tests/test_oracle_match.py.
"""
from __future__ import annotations

import math

import numpy as np

f32 = np.float32


def project_dist(campt, K, dist):
    """CameraCalibration::projectCamToImageDist for the pinhole model: float32 pixel (x, y)."""
    fx, fy, cx, cy = (float(v) for v in K)
    invz = 1.0 / float(campt[2])
    x, y = float(campt[0]) * invz, float(campt[1]) * invz
    if dist is None:
        return f32(fx * x + cx), f32(fy * y + cy)
    # cv::Point3f(x, y, 1.) -> cv::projectPoints with zero rotation / translation
    x, y = float(f32(x)), float(f32(y))
    k1, k2, p1, p2, k3 = (float(v) for v in dist)
    r2 = x * x + y * y
    r4 = r2 * r2
    r6 = r4 * r2
    a1 = 2 * x * y
    a2 = r2 + 2 * x * x
    a3 = r2 + 2 * y * y
    cdist = 1 + k1 * r2 + k2 * r4 + k3 * r6
    xd = x * cdist + p1 * a1 + p2 * a2
    yd = y * cdist + p1 * a3 + p2 * a1
    return f32(xd * fx + cx), f32(yd * fy + cy)


def _norm2(dx, dy):
    """cv::norm(cv::Point2f): sqrt in double of the float components."""
    return math.sqrt(float(dx) * float(dx) + float(dy) * float(dy))


def camera_point(T, w):
    """transform() of match_map.cu: T = (row-major R, t) as 12 doubles, each row summed left to right."""
    T = [float(v) for v in T]
    w0, w1, w2 = float(w[0]), float(w[1]), float(w[2])
    return (T[0] * w0 + T[1] * w1 + T[2] * w2 + T[9],
            T[3] * w0 + T[4] * w1 + T[5] * w2 + T[10],
            T[6] * w0 + T[7] * w1 + T[8] * w2 + T[11])


def view_angle(X, Y, Z):
    """z / |p| of the camera-frame point, rounded to float (mapper.cpp:634)."""
    return f32(Z / math.sqrt(X * X + Y * Y + Z * Z))


def pixel_distance(px, py, kx, ky):
    """Distance of the projection to a keypoint: float components, norm in double, rounded to float (mapper.cpp:667)."""
    return f32(_norm2(f32(f32(px) - f32(kx)), f32(f32(py) - f32(ky))))


def coprojection(sc, wpt, lm):
    """(mean co-projection error as a float, nb): the map point `wpt` projected into every keyframe observing map point `lm`,
    float accumulation of the double norms (mapper.cpp:698-716).  The mean is None when no keyframe observes `lm`."""
    kf_T = np.asarray(sc["kf_Tcw"], np.float64).reshape(-1, 12)
    coproj, nb = f32(0.0), 0
    for o in range(int(sc["mp_obs_ptr"][lm]), int(sc["mp_obs_ptr"][lm + 1])):
        qx, qy = project_dist(camera_point(kf_T[int(sc["obs_kf"][o])], wpt), sc["K"], sc.get("dist"))
        ox, oy = sc["obs_px"][o]
        coproj = f32(float(coproj) + _norm2(f32(ox - qx), f32(oy - qy)))
        nb += 1
    return (f32(coproj / f32(nb)) if nb else None), nb


def min_dist(fdistratio):
    """The starting best / second distance: desc_.cols * fdistratio * 8. with a 32-byte descriptor (mapper.cpp:650)."""
    return f32(float(f32(32 * f32(fdistratio))) * 8.0)


def _desc_ints(desc):
    return [int.from_bytes(bytes(row), "little") for row in np.asarray(desc, np.uint8).reshape(-1, 32)]


def match_to_map(sc: dict):
    """Returns (best_kp int32[ncand], best_dist float32[ncand], kp_match int32[nkps], kp_dist float32[nkps])."""
    K, dist = sc["K"], sc.get("dist")
    Tcw = np.asarray(sc["Tcw"], np.float64).reshape(-1)
    cs, nbw = int(sc["ncellsize"]), int(sc["nbwcells"])
    ncells = len(sc["cell_ptr"]) - 1
    w, h = int(sc["img_w"]), int(sc["img_h"])
    dmax, view_th = f32(sc["dmaxpxdist"]), f32(sc["view_th"])
    ncand = len(sc["cand_mp"])
    best_kp = -np.ones(ncand, np.int32)
    best_dist = np.zeros(ncand, np.float32)
    mindist = min_dist(sc["fdistratio"])
    desc = _desc_ints(sc["desc"])
    desc_ptr = [int(v) for v in sc["mp_desc_ptr"]]
    kfmask = [tuple(int(v) for v in row) for row in np.asarray(sc["mp_kfmask"], np.uint64).reshape(-1, 4)]
    for ci, mp in enumerate(int(v) for v in sc["cand_mp"]):
        wpt = sc["mp_xyz"][mp]
        X, Y, Z = camera_point(Tcw, wpt)
        if Z < 0.1:
            continue
        if abs(view_angle(X, Y, Z)) < view_th:
            continue
        px, py = project_dist((X, Y, Z), K, dist)
        if not (px >= 0 and py >= 0 and px < w and py < h):
            continue
        rkp, ckp = int(math.floor(float(f32(py / f32(cs))))), int(math.floor(float(f32(px / f32(cs)))))
        bestid = secid = -1
        bestdist = secdist = mindist
        for r in (rkp - 1, rkp):
            for c in (ckp - 1, ckp):
                idx = r * nbw + c
                if r < 0 or c < 0 or idx >= ncells:
                    continue
                for j in sc["cell_kp"][sc["cell_ptr"][idx]:sc["cell_ptr"][idx + 1]]:
                    lm = int(sc["kp_lm"][j])
                    if lm < 0:
                        continue
                    kx, ky = sc["kp_px"][j]
                    if pixel_distance(px, py, kx, ky) > dmax:
                        continue
                    d0, d1 = desc_ptr[lm], desc_ptr[lm + 1]
                    if d1 == d0:
                        continue
                    if any(a & b for a, b in zip(kfmask[mp], kfmask[lm])):
                        continue
                    mean, nb = coprojection(sc, wpt, lm)
                    if nb > 0 and mean > dmax:
                        continue
                    dd = 1000
                    for a in desc[desc_ptr[mp]:desc_ptr[mp + 1]]:
                        for b in desc[d0:d1]:
                            dd = min(dd, (a ^ b).bit_count())
                    dd = f32(dd)
                    if dd <= bestdist:
                        secdist, secid = bestdist, bestid
                        bestdist, bestid = dd, int(j)
                    elif dd <= secdist:
                        secdist, secid = dd, int(j)
        if bestid != -1 and secid != -1 and 0.9 * float(secdist) < float(bestdist):
            bestid = -1
        if bestid >= 0:
            best_kp[ci] = bestid
            best_dist[ci] = bestdist
    nk = len(sc["kp_px"])
    kp_match = -np.ones(nk, np.int32)
    kp_dist = np.full(nk, 1024.0, np.float32)
    for ci in range(ncand):
        j = best_kp[ci]
        if j >= 0 and best_dist[ci] <= kp_dist[j]:
            kp_dist[j] = best_dist[ci]
            kp_match[j] = ci
    return best_kp, best_dist, kp_match, kp_dist
