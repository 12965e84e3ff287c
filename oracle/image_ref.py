"""CPU ORACLE for the front-end image path.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  The product path (ov2slam_b200/) never does.

The reference delegates every image-side computation to OpenCV
(/root/reference/src/feature_extractor.cpp:443-570,224-285; src/feature_tracker.cpp:35-137;
src/visual_front_end.cpp:1143-1177).  OpenCV's source is NOT under /root/reference and its
version is unpinned by the reference (CMakeLists.txt:73-77: find_package(OpenCV REQUIRED), >=3).
Parity is therefore pinned to **cv2 4.13.0** (the OpenCV in this image) run with
cv2.setNumThreads(1), in two layers:

  *_cv2()  - the reference's exact OpenCV call sequence, executed by the real library.
  *_ref()  - a numpy restatement of what that sequence computes (SURVEY.md Appendix A), which
             tests/test_oracle_image.py pins against *_cv2() on seeded inputs.  The restatement
             is what documents the semantics the CUDA kernels implement and is what runs where
             cv2 is unavailable (the committed golden vectors under tests/golden/ come from
             *_cv2()).

The reference has no tests or golden vectors of its own for this path (SURVEY.md section 4), so
"pinned" here means pinned to the third-party library the reference calls, not to a fixture
of the reference.  The ORCHESTRATION around those calls (grid walk, masks, sort order, threshold /
quality adaptation, descriptor re-alignment, the forward-backward tracking flow, the row search) is
in addition checked against the reference's own src/feature_extractor.cpp and src/feature_tracker.cpp,
compiled where they lie on stand-in OpenCV containers whose arithmetic calls are answered by cv2
(oracle/ref_build/mini_cv, cv_callbacks.py; tests/test_oracle_vs_reference_frontend.py).
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from pathlib import Path

import numpy as np

from .orb_pattern import ORB_PATTERN

try:  # cv2 is present in this image; the restatements below do not need it
    import cv2
    cv2.setNumThreads(1)
    HAVE_CV2 = True
except Exception:  # pragma: no cover
    cv2 = None
    HAVE_CV2 = False

_HERE = Path(__file__).resolve().parent
_BUILD = _HERE / "_build"

KLT_EPS = float(np.float32(0.01))  # FeatureTracker stores fmax_px_precision as float (feature_tracker.hpp:37-41)


# ------------------------------------------------------------------ libstdc++ std::sort helper
_sortlib = None


def build_helpers(force: bool = False) -> Path:
    """g++ -shared oracle/stdsort_helper.cpp -> oracle/_build/libov2oracle_sort.so"""
    _BUILD.mkdir(exist_ok=True)
    so = _BUILD / "libov2oracle_sort.so"
    src = _HERE / "stdsort_helper.cpp"
    if force or not so.exists() or so.stat().st_mtime < src.stat().st_mtime:
        # compiled under a private name and renamed: several processes may get here at once on a fresh checkout (the CPU arm's workers)
        tmp = so.with_name(f"{so.name}.{os.getpid()}.tmp")
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", str(tmp), str(src)])
        os.replace(tmp, so)
    return so


def stdsort_desc(resp) -> np.ndarray:
    """Index order libstdc++ std::sort(v.begin(), v.end(), compare_response) produces
    (feature_extractor.cpp:75-77,518)."""
    global _sortlib
    if _sortlib is None:
        _sortlib = ctypes.CDLL(str(build_helpers()))
        _sortlib.ov2_oracle_sort_desc.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    r = np.ascontiguousarray(resp, np.float32)
    out = np.empty(len(r), np.int32)
    _sortlib.ov2_oracle_sort_desc(r.ctypes.data, len(r), out.ctypes.data)
    return out


# ------------------------------------------------------------------ P: pyramid + Scharr
def _reflect101(idx, n):
    """cv::borderInterpolate(idx, n, BORDER_REFLECT_101): reflected until inside [0, n) (an index can overshoot by
    more than n on a level narrower than the window); n == 1 maps everything to 0."""
    idx = np.asarray(idx)
    if n == 1:
        return np.zeros_like(idx)
    while True:
        idx = np.abs(idx)
        over = idx >= n
        if not over.any():
            return idx
        idx = np.where(over, 2 * (n - 1) - idx, idx)


def optflow_levels(w: int, h: int, win: int = 9, maxlevel: int = 3) -> int:
    """The pyramid depth cv::buildOpticalFlowPyramid(img, pyr, Size(win, win), maxlevel) reaches (its return value): it
    stops before a level whose width or height would be <= win.  calcOpticalFlowPyrLK tracks from that depth, and the
    reference clamps nbpyrlvl to it (feature_tracker.cpp:50-52)."""
    for level in range(maxlevel):
        w, h = (w + 1) // 2, (h + 1) // 2
        if w <= win or h <= win:
            return level
    return maxlevel


def pyr_down_ref(img: np.ndarray) -> np.ndarray:
    """cv::pyrDown: separable [1 4 6 4 1], BORDER_REFLECT_101, (sum + 128) >> 8, even samples,
    output ((W+1)/2, (H+1)/2)  (SURVEY.md A.3)."""
    h, w = img.shape
    oh, ow = (h + 1) // 2, (w + 1) // 2
    k = np.array([1, 4, 6, 4, 1], np.int32)
    src = img.astype(np.int32)
    xs = 2 * np.arange(ow)[:, None] + np.arange(-2, 3)[None, :]
    xs = _reflect101(xs, w)
    rows = (src[:, xs] * k[None, None, :]).sum(axis=2)  # (h, ow)
    ys = 2 * np.arange(oh)[:, None] + np.arange(-2, 3)[None, :]
    ys = _reflect101(ys, h)
    out = (rows[ys, :] * k[None, :, None]).sum(axis=1)  # (oh, ow)
    return ((out + 128) >> 8).astype(np.uint8)


def build_pyramid_ref(img: np.ndarray, nlevels_extra: int = 3):
    """Images of cv::buildOpticalFlowPyramid(img, pyr, Size(9,9), 3) (visual_front_end.cpp:1172):
    [L0, L1, L2, L3].  The derivative Mats are recomputed on the fly by the tracker."""
    pyr = [np.ascontiguousarray(img)]
    for _ in range(nlevels_extra):
        pyr.append(pyr_down_ref(pyr[-1]))
    return pyr


def build_pyramid_cv2(img: np.ndarray, nlevels_extra: int = 3):
    pyr = [np.ascontiguousarray(img)]
    for _ in range(nlevels_extra):
        pyr.append(cv2.pyrDown(pyr[-1]))
    return pyr


def scharr_ref(img: np.ndarray):
    """calcScharrDeriv: Ix = [3 10 3]^T (x) [-1 0 1], Iy = [-1 0 1]^T (x) [3 10 3], int16,
    REFLECT_101 at the image edge."""
    h, w = img.shape
    s = img.astype(np.int32)
    ym = _reflect101(np.arange(h) - 1, h)
    yp = _reflect101(np.arange(h) + 1, h)
    xm = _reflect101(np.arange(w) - 1, w)
    xp = _reflect101(np.arange(w) + 1, w)
    t0 = (s[ym] + s[yp]) * 3 + s * 10
    t1 = s[yp] - s[ym]
    ix = t0[:, xp] - t0[:, xm]
    iy = (t1[:, xp] + t1[:, xm]) * 3 + t1 * 10
    return ix.astype(np.int16), iy.astype(np.int16)


# ------------------------------------------------------------------ F: FAST-9/16 + grid logic
_RING = np.array([(0, -3), (1, -3), (2, -2), (3, -1), (3, 0), (3, 1), (2, 2), (1, 3), (0, 3), (-1, 3),
                  (-2, 2), (-3, 1), (-3, 0), (-3, -1), (-2, -2), (-1, -3)], np.int32)


def fast_score_ref(roi: np.ndarray) -> np.ndarray:
    """Corner score s (SURVEY.md A.1) for every pixel of the ROI with a full ring inside it;
    0 elsewhere.  Pixel is a FAST-9/16 corner at threshold t iff s > t; response = s - 1."""
    h, w = roi.shape
    s = np.zeros((h, w), np.int32)
    if h < 7 or w < 7:
        return s
    v = roi.astype(np.int32)
    c = v[3:h - 3, 3:w - 3]
    d = np.stack([c - v[3 + dy:h - 3 + dy, 3 + dx:w - 3 + dx] for dx, dy in _RING], axis=0)  # (16, ..)
    d2 = np.concatenate([d, d[:8]], axis=0)
    best = np.zeros(c.shape, np.int32)
    for k in range(16):
        arc = d2[k:k + 9]
        mn = arc.min(axis=0)
        mx = arc.max(axis=0)
        best = np.maximum(best, np.maximum(mn, -mx))
    s[3:h - 3, 3:w - 3] = np.maximum(best, 0)
    return s


def fast_detect_ref(roi: np.ndarray, th: int):
    """cv::FastFeatureDetector(th, nonmaxSuppression=true, TYPE_9_16).detect(roi): list of
    (x, y, response) in row-major scan order."""
    s = fast_score_ref(roi)
    resp = np.where(s > th, s - 1, 0)
    h, w = roi.shape
    p = np.pad(resp, 1)
    keep = resp > 0 if th >= 0 else np.ones_like(resp, bool)
    keep = (s > th)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dx == 0 and dy == 0:
                continue
            keep &= resp > p[1 + dy:1 + dy + h, 1 + dx:1 + dx + w]
    # interior only (3-px border of the ROI never holds a keypoint)
    inner = np.zeros_like(keep)
    inner[3:h - 3, 3:w - 3] = True
    keep &= inner
    ys, xs = np.nonzero(keep)
    return [(int(x), int(y), float(resp[y, x])) for y, x in zip(ys, xs)]


def fast_detect_cv2(roi: np.ndarray, th: int):
    det = cv2.FastFeatureDetector_create(int(th))
    kps = det.detect(np.ascontiguousarray(roi), None)
    return [(int(k.pt[0]), int(k.pt[1]), float(k.response)) for k in kps]


def circle_halfwidths(radius: int) -> np.ndarray:
    """Filled cv::circle(img, c, radius, color, -1) rasterisation (OpenCV's midpoint circle):
    row c.y + dy is filled over x in [c.x - hw[|dy|], c.x + hw[|dy|]].  Not the Euclidean disc."""
    hw = np.full(radius + 1, -1, np.int32)
    err, dx, dy, plus, minus = 0, radius, 0, 1, (radius << 1) - 1
    while dx >= dy:
        hw[dy] = max(hw[dy], dx)
        hw[dx] = max(hw[dx], dy)
        dy += 1
        err += plus
        plus += 2
        mask = -1 if err > 0 else 0  # (err <= 0) - 1
        err -= minus & mask
        dx += mask
        minus -= mask & 2
    return hw


def paint_disc(mask: np.ndarray, cx: int, cy: int, hw: np.ndarray) -> None:
    h, w = mask.shape
    r = len(hw) - 1
    for dy in range(-r, r + 1):
        y = cy + dy
        if 0 <= y < h:
            x0 = max(cx - int(hw[abs(dy)]), 0)
            x1 = min(cx + int(hw[abs(dy)]), w - 1)
            if x0 <= x1:
                mask[y, x0:x1 + 1] = 0


def _cv_round(v) -> int:
    """cvRound / saturate_cast<int>(float): round-half-to-even."""
    return int(np.rint(np.float32(v)))


def detect_grid_fast_nosubpix(im: np.ndarray, cellsize: int, curkps, fast_th: int, use_cv2: bool, stats=None):
    """FeatureExtractor::detectGridFAST up to (not including) cornerSubPix
    (feature_extractor.cpp:443-552), with the *sequential* ascending cell order as the defined
    semantics (the reference's parallel_for_ body races on `mask`; SURVEY.md section 2.1).

    Returns (pts int32[N, 2] in cell order, new_fast_th, nbempty).  `stats`, if a list, receives
    (cell, survivors, survivors with the maximal response) for every cell that had a survivor.
    """
    rows, cols = im.shape
    r4 = cellsize // 4
    nh, nw = rows // cellsize, cols // cellsize
    occ = np.zeros((nh + 1, nw + 1), bool)
    # CV_32F ones mask; detect() reads it as bytes (SURVEY.md A.2)
    mask = np.ones((rows, cols), np.float32)
    hw = circle_halfwidths(r4)
    for px in np.asarray(curkps, np.float32).reshape(-1, 2):
        # voccupcells[px.y / ncellsize][px.x / ncellsize]: float divide, truncation
        occ[int(np.float32(px[1]) / np.float32(cellsize)), int(np.float32(px[0]) / np.float32(cellsize))] = True
        if use_cv2:
            cv2.circle(mask, (_cv_round(px[0]), _cv_round(px[1])), r4, 0, -1)
        else:
            paint_disc(mask, _cv_round(px[0]), _cv_round(px[1]), hw)
    det = cv2.FastFeatureDetector_create(int(fast_th)) if use_cv2 else None
    out = []
    nbempty = 0
    for i in range(nh * nw):
        r, c = i // nw, i % nw
        if occ[r, c]:
            continue
        nbempty += 1
        x, y = c * cellsize, r * cellsize
        if not (x + cellsize < cols - 1 and y + cellsize < rows - 1):
            continue
        roi = im[y:y + cellsize, x:x + cellsize]
        if use_cv2:
            kps = det.detect(roi, mask[y:y + cellsize, x:x + cellsize])
            cand = [(int(k.pt[0]), int(k.pt[1]), float(k.response)) for k in kps]
        else:
            mbytes = mask[y:y + cellsize, x:x + cellsize]
            # byte kx of the float row = byte kx%4 of float kx//4 of the sub-matrix row
            cand = []
            for (kx, ky, resp) in fast_detect_ref(roi, fast_th):
                b = np.ascontiguousarray(mbytes[ky, kx // 4:kx // 4 + 1]).view(np.uint8)[kx % 4]
                if b != 0:
                    cand.append((kx, ky, resp))
        if not cand:
            continue
        if stats is not None:
            top = max(k[2] for k in cand)
            stats.append((i, len(cand), sum(k[2] == top for k in cand)))
        order = stdsort_desc([k[2] for k in cand])
        best = cand[int(order[0])]
        if best[2] >= 20:
            px, py = best[0] + x, best[1] + y
            if use_cv2:
                cv2.circle(mask, (px, py), r4, 0, -1)
            else:
                paint_disc(mask, px, py, hw)
            out.append((px, py))
    nbkps = len(out)
    th = int(fast_th)
    if nbkps < 0.5 * nbempty and nbempty > 10:
        th = int(th * 0.66)  # int member *= double (feature_extractor.cpp:546-552)
    elif nbkps == nbempty:
        th = int(th * 1.5)
    return np.array(out, np.int32).reshape(-1, 2), th, nbempty


# ------------------------------------------------------------------ S: cornerSubPix
def corner_subpix_cv2(im: np.ndarray, pts: np.ndarray) -> np.ndarray:
    if len(pts) == 0:
        return np.zeros((0, 2), np.float32)
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 1, 2).copy()
    cv2.cornerSubPix(im, p, (3, 3), (-1, -1), (cv2.TERM_CRITERIA_EPS + cv2.TERM_CRITERIA_MAX_ITER, 30, 0.01))
    return p.reshape(-1, 2)


def _fma32(a, b, c):
    """float32 fused multiply-add (exact product in float64, one rounding to float32 apart from
    a vanishingly rare double rounding)."""
    return np.float32(np.float64(a) * np.float64(b) + np.float64(c))


def _get_rect_subpix_9(im: np.ndarray, cx: np.float32, cy: np.float32) -> np.ndarray:
    """cv::getRectSubPix(im, Size(9,9), c, dst, CV_32F) for an 8-bit source, float32 bilinear with
    a replicated border, in the exact float grouping cv2 4.13 uses (found by exhaustive probing,
    100 % bit-equal on 3 000 random windows incl. borders):
      interior pixel          (p00*a11 + p01*a12) + (p10*a21 + p11*a22)       no FMA
      x-clamped column        p0*(1-b) + p1*b  on the clamped column           no FMA
      y-clamped row           fma(p1, a, p0*(1-a)) on the clamped row
      quirk: in rows above the image the right-clamped columns sample column W-2, not W-1.
    """
    h, w = im.shape
    f32 = np.float32
    f1 = f32(1.0)
    x = f32(f32(cx) - f32(4.0))
    y = f32(f32(cy) - f32(4.0))
    ix, iy = int(np.floor(x)), int(np.floor(y))
    a = f32(x - f32(ix))
    b = f32(y - f32(iy))
    out = np.zeros((9, 9), f32)
    a11 = f32(f32(f1 - a) * f32(f1 - b))
    a12 = f32(a * f32(f1 - b))
    a21 = f32(f32(f1 - a) * b)
    a22 = f32(a * b)
    if 0 <= ix and ix + 9 < w and 0 <= iy and iy + 9 < h:
        p = im[iy:iy + 10, ix:ix + 10].astype(f32)
        return ((p[:9, :9] * a11 + p[:9, 1:] * a12).astype(f32)
                + (p[1:, :9] * a21 + p[1:, 1:] * a22).astype(f32)).astype(f32)
    b1 = f32(f1 - b)
    b2 = b
    rx = min(-ix, 9) if ix < 0 else 0
    rw = 9 if ix < w - 9 else max(w - ix - 1, 0)
    ry = -iy if iy < 0 else 0
    rh = 9 if iy < h - 9 else max(h - iy - 1, 0)
    for i in range(9):
        r0 = min(max(iy + i, 0), h - 1)
        r1 = min(max(iy + i + 1, 0), h - 1)
        yclamp = i < ry or i >= rh
        s0 = im[r0].astype(f32)
        s1 = im[r1].astype(f32)
        for j in range(9):
            if j < rx or j >= rw:
                c = 0 if j < rx else (w - 2 if i < ry else w - 1)
                c = min(max(c, 0), w - 1)
                out[i, j] = f32(f32(s0[c] * b1) + f32(s1[c] * b2))
            elif yclamp:
                c = ix + j
                out[i, j] = _fma32(s0[c + 1], a, f32(s0[c] * f32(f1 - a)))
            else:
                c = ix + j
                out[i, j] = f32(f32(f32(s0[c] * a11) + f32(s0[c + 1] * a12))
                                + f32(f32(s1[c] * a21) + f32(s1[c + 1] * a22)))
    return out


def corner_subpix_ref(im: np.ndarray, pts: np.ndarray) -> np.ndarray:
    """cv::cornerSubPix(im, pts, (3,3), (-1,-1), (EPS|MAX_ITER, 30, 0.01)) (SURVEY.md A.4)."""
    h, w = im.shape
    k = np.arange(-3, 4, dtype=np.float32) / np.float32(3)
    m1 = np.exp(-(k * k)).astype(np.float32)
    mask = (m1[:, None] * m1[None, :]).astype(np.float32)
    px = np.arange(-3, 4, dtype=np.float64)[None, :]
    py = np.arange(-3, 4, dtype=np.float64)[:, None]
    out = np.array(pts, np.float32).reshape(-1, 2).copy()
    for n in range(len(out)):
        ct = out[n].copy()
        ci = ct.copy()
        for _ in range(30):
            sub = _get_rect_subpix_9(im, ci[0], ci[1])
            tgx = (sub[1:8, 2:9] - sub[1:8, 0:7]).astype(np.float64)
            tgy = (sub[2:9, 1:8] - sub[0:7, 1:8]).astype(np.float64)
            mm = mask.astype(np.float64)
            gxx = tgx * tgx * mm
            gxy = tgx * tgy * mm
            gyy = tgy * tgy * mm
            a, b, c = gxx.sum(), gxy.sum(), gyy.sum()
            bb1 = (gxx * px + gxy * py).sum()
            bb2 = (gxy * px + gyy * py).sum()
            det = a * c - b * b
            if abs(det) <= np.finfo(np.float64).eps ** 2:
                break
            scale = 1.0 / det
            ci2 = np.array([np.float32(ci[0] + c * scale * bb1 - b * scale * bb2),
                            np.float32(ci[1] - b * scale * bb1 + a * scale * bb2)], np.float32)
            ex = np.float32(ci2[0] - ci[0])
            ey = np.float32(ci2[1] - ci[1])
            err = float(np.float32(np.float32(ex * ex) + np.float32(ey * ey)))
            # cv2 4.13 tests the *new* point and leaves the loop before adopting it
            if ci2[0] < 0 or ci2[0] >= w or ci2[1] < 0 or ci2[1] >= h:
                break
            ci = ci2
            if err <= 0.01 * 0.01:
                break
        if abs(ci[0] - ct[0]) > 3 or abs(ci[1] - ct[1]) > 3:
            ci = ct
        out[n] = ci
    return out


# ------------------------------------------------------------------ B: ORB-fallback descriptor
_GK7 = None


def gauss7_kernel() -> np.ndarray:
    """cv::getGaussianKernel(7, 2, CV_32F)."""
    global _GK7
    if _GK7 is None:
        x = np.arange(7, dtype=np.float64) - 3.0
        kd = np.exp(-0.5 * (x / 2.0) ** 2)
        kd = kd / kd.sum()
        _GK7 = kd.astype(np.float32)
    return _GK7


def describe_cv2(im: np.ndarray, pts: np.ndarray):
    """FeatureExtractor::describeBRIEF, non-contrib branch (feature_extractor.cpp:224-285,245):
    cv::ORB::create(500, 1., 0).compute on KeyPoint::convert'ed points.  Returns
    (desc uint8[N, 32], valid uint8[N]); rows of dropped points are zero."""
    pts = np.asarray(pts, np.float32).reshape(-1, 2)
    n = len(pts)
    desc = np.zeros((n, 32), np.uint8)
    valid = np.zeros(n, np.uint8)
    if n == 0:
        return desc, valid
    orb = cv2.ORB_create(500, 1.0, 0)
    kps = [cv2.KeyPoint(float(x), float(y), 1.0) for x, y in pts]
    kps2, d = orb.compute(im, kps)
    k = 0
    for i in range(n):
        if k < len(kps2) and kps2[k].pt[0] == pts[i, 0] and kps2[k].pt[1] == pts[i, 1]:
            desc[i] = d[k]
            valid[i] = 1
            k += 1
    return desc, valid


def smooth7_ref(im: np.ndarray) -> np.ndarray:
    """ORB's GaussianBlur(7x7, sigma 2, BORDER_REFLECT_101) as cv2 4.13 evaluates it on this
    image's CPU dispatch (== cv2.sepFilter2D with the float32 kernel; found by probing, 0 wrong
    pixels): float32 rows  acc = x[-3]*k0; acc = fma(x[j], k[j], acc) for j = -2..3;
    columns  acc = r[0]*k3; acc = fma(r[-j] + r[j], k[3+j], acc) for j = 1..3;  rint -> u8."""
    kf = gauss7_kernel()
    h, w = im.shape
    src = im.astype(np.float32)
    xs = _reflect101(np.arange(-3, w + 3), w)
    p = src[:, xs]
    row = (p[:, 0:w] * kf[0]).astype(np.float32)
    for j in range(1, 7):
        row = _fma32(p[:, j:j + w], kf[j], row)
    ys = _reflect101(np.arange(-3, h + 3), h)
    q = row[ys, :]
    col = (q[3:3 + h] * kf[3]).astype(np.float32)
    for j in (1, 2, 3):
        col = _fma32((q[3 - j:3 - j + h] + q[3 + j:3 + j + h]).astype(np.float32), kf[3 + j], col)
    return np.clip(np.rint(col), 0, 255).astype(np.uint8)


def describe_ref(im: np.ndarray, pts: np.ndarray):
    """numpy restatement of describe_cv2 (SURVEY.md A.5)."""
    pts = np.asarray(pts, np.float32).reshape(-1, 2)
    h, w = im.shape
    n = len(pts)
    desc = np.zeros((n, 32), np.uint8)
    valid = np.zeros(n, np.uint8)
    if n == 0:
        return desc, valid
    sm = smooth7_ref(im)
    pat = ORB_PATTERN.astype(np.int32)
    for i in range(n):
        x, y = pts[i]
        # KeyPointsFilter::runByImageBorder(.., 31) tests the *rounded* point
        # (Rect::contains(Point2f -> Point)): 31 <= cvRound(x) < W - 31
        cx, cy = _cv_round(x), _cv_round(y)
        if cx < 31 or cy < 31 or cx >= w - 31 or cy >= h - 31:
            continue
        a = sm[cy + pat[:, 1], cx + pat[:, 0]]
        b = sm[cy + pat[:, 3], cx + pat[:, 2]]
        bits = (a < b).astype(np.uint8).reshape(32, 8)
        desc[i] = (bits << np.arange(8, dtype=np.uint8)[None, :]).sum(axis=1).astype(np.uint8)
        valid[i] = 1
    return desc, valid


def brief32_ref(im: np.ndarray, pts: np.ndarray, pairs: np.ndarray):
    """FeatureExtractor::describeBRIEF, DEFAULT (contrib) branch: cv::xfeatures2d::BriefDescriptorExtractor::create()
    (feature_extractor.cpp:242-243; 32 bytes, use_orientation = false) as opencv_contrib's
    modules/xfeatures2d/src/brief.cpp computes it:
      KeyPointsFilter::runByImageBorder(kps, size, PATCH_SIZE/2 + KERNEL_SIZE/2 = 24 + 4)   (rounded point),
      integral(gray, sum, CV_32S),
      smoothedSum(pt, y, x) = box sum of the 9 x 9 pixels centred on ((int)(pt.y + 0.5) + y, (int)(pt.x + 0.5) + x),
      desc[i] = sum_k (SMOOTHED(y0, x0) < SMOOTHED(y1, x1)) << (7 - k) over the 8 tests of byte i (generated_32.i).
    `pairs` int8[256][4] = (y0, x0, y1, x1) in generated_32.i order.  opencv_contrib is not installed in this image:
    this restatement is NOT pinned against cv2.xfeatures2d ("parity unpinned" for the BRIEF-32 mode); the ORB-fallback
    mode above is pinned."""
    pts = np.asarray(pts, np.float32).reshape(-1, 2)
    pairs = np.asarray(pairs, np.int32).reshape(256, 4)
    h, w = im.shape
    n = len(pts)
    desc = np.zeros((n, 32), np.uint8)
    valid = np.zeros(n, np.uint8)
    if n == 0:
        return desc, valid
    # one replicated column / row: at a .5 tie (int)(pt + 0.5) can exceed the rounded centre by one, so a box can reach
    # one pixel past the image when W - 29 (H - 29) is even.  OpenCV reads the integral image out of its row there
    # (meaningless values); the kernel and this restatement replicate the edge pixel instead.
    imp = np.pad(im, ((0, 1), (0, 1)), mode="edge").astype(np.int64)
    integ = np.zeros((h + 2, w + 2), np.int64)
    integ[1:, 1:] = np.cumsum(np.cumsum(imp, axis=0), axis=1)
    weights = (1 << (7 - np.arange(8))).astype(np.int32)
    for i in range(n):
        x, y = pts[i]
        rx, ry = _cv_round(x), _cv_round(y)
        if rx < 28 or ry < 28 or rx >= w - 28 or ry >= h - 28:
            continue
        cx, cy = int(float(x) + 0.5), int(float(y) + 0.5)

        def smoothed(dy, dx):
            yy = cy + dy
            xx = cx + dx
            return (integ[yy + 5, xx + 5] - integ[yy + 5, xx - 4] - integ[yy - 4, xx + 5] + integ[yy - 4, xx - 4])

        a = smoothed(pairs[:, 0], pairs[:, 1])
        b = smoothed(pairs[:, 2], pairs[:, 3])
        bits = (a < b).astype(np.int32).reshape(32, 8)
        desc[i] = (bits * weights[None, :]).sum(axis=1).astype(np.uint8)
        valid[i] = 1
    return desc, valid


# ------------------------------------------------------------------ K: forward/backward LK
def _lk_cv2(prev, cur, pts, init, maxlevel, win, maxit, eps):
    p0 = np.ascontiguousarray(pts, np.float32).reshape(-1, 1, 2)
    p1 = np.ascontiguousarray(init, np.float32).reshape(-1, 1, 2).copy()
    nxt, st, err = cv2.calcOpticalFlowPyrLK(
        prev, cur, p0, p1, winSize=(win, win), maxLevel=int(maxlevel),
        criteria=(cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, int(maxit), float(eps)),
        flags=cv2.OPTFLOW_USE_INITIAL_FLOW + cv2.OPTFLOW_LK_GET_MIN_EIGENVALS)
    return nxt.reshape(-1, 2), st.reshape(-1).astype(np.uint8), err.reshape(-1)


def _in_border(pt, w, h) -> bool:
    return 1.0 <= pt[0] < w - 1.0 and 1.0 <= pt[1] < h - 1.0


def _fb_klt(lk, prev, cur, kps, priors, win, nbpyrlvl, ferr, fb_dist, maxit, eps):
    kps = np.asarray(kps, np.float32).reshape(-1, 2)
    pri = np.asarray(priors, np.float32).reshape(-1, 2).copy()
    n = len(kps)
    status = np.zeros(n, np.uint8)
    if n == 0:
        return pri, status
    h, w = cur.shape
    # pyramid built with at most 3 extra levels, fewer on small images (feature_tracker.cpp:50-52)
    nbpyrlvl = min(int(nbpyrlvl), optflow_levels(w, h, win, 3))
    fwd, st, err = lk(prev, cur, kps, pri, nbpyrlvl, win, maxit, eps)
    pri[:] = fwd  # vpriorkps is in/out
    idx = []
    for i in range(n):
        if not st[i] or err[i] > ferr or not _in_border(fwd[i], w, h):
            continue
        status[i] = 1
        idx.append(i)
    if not idx:
        return pri, status
    idx = np.array(idx)
    back, st2, _ = lk(cur, prev, fwd[idx], kps[idx], 0, win, maxit, eps)
    for j, i in enumerate(idx):
        if not st2[j]:
            status[i] = 0
            continue
        d = kps[i] - back[j]
        # cv::norm(Point2f) evaluates sqrt((double)x*x + (double)y*y)
        if np.sqrt(float(d[0]) * float(d[0]) + float(d[1]) * float(d[1])) > fb_dist:
            status[i] = 0
    return pri, status


def fb_klt_cv2(prev, cur, kps, priors, win=9, nbpyrlvl=3, ferr=30.0, fb_dist=0.5, maxit=30, eps=KLT_EPS):
    """FeatureTracker::fbKltTracking (feature_tracker.cpp:35-137) through cv2.  The Python
    binding of calcOpticalFlowPyrLK takes images, not pyramids; OpenCV then builds the identical
    pyramid internally (SURVEY.md 8c).  Returns (tracked float32[N, 2] = vpriorkps out,
    status uint8[N] = vkpstatus)."""
    return _fb_klt(_lk_cv2, prev, cur, kps, priors, win, nbpyrlvl, ferr, fb_dist, maxit, eps)


def _cvround_arr(x):
    return np.rint(x).astype(np.int64)


def _lk_ref(prev, cur, pts, init, maxlevel, win, maxit, eps):
    """numpy restatement of cv::calcOpticalFlowPyrLK with USE_INITIAL_FLOW | GET_MIN_EIGENVALS
    (SURVEY.md A.3).  Integer window sums are accumulated exactly and converted to float32 once."""
    f32 = np.float32
    pp = build_pyramid_ref(prev, 3)
    cp = build_pyramid_ref(cur, 3)
    pts = np.asarray(pts, f32).reshape(-1, 2)
    nxt = np.asarray(init, f32).reshape(-1, 2).copy()
    n = len(pts)
    status = np.ones(n, np.uint8)
    err = np.zeros(n, f32)
    half = f32((win - 1) * 0.5)
    eps2 = float(eps) * float(eps)
    flt_scale = f32(1.0 / (1 << 20))
    derivs = [scharr_ref(p) for p in pp]
    wy, wx = np.meshgrid(np.arange(win + 1), np.arange(win + 1), indexing="ij")

    def gather_u8(img, ix, iy):
        h, w = img.shape
        xs = _reflect101(ix + np.arange(win + 1), w)
        ys = _reflect101(iy + np.arange(win + 1), h)
        return img[np.ix_(ys, xs)].astype(np.int64)

    def gather_d(d, ix, iy):
        h, w = d.shape
        xs = ix + np.arange(win + 1)
        ys = iy + np.arange(win + 1)
        okx = (xs >= 0) & (xs < w)
        oky = (ys >= 0) & (ys < h)
        g = d[np.ix_(np.clip(ys, 0, h - 1), np.clip(xs, 0, w - 1))].astype(np.int64)
        return g * (oky[:, None] & okx[None, :])

    def weights(a, b):
        one = f32(1.0)
        s = f32(1 << 14)
        iw00 = int(np.rint(f32(f32(f32(one - a) * f32(one - b)) * s)))
        iw01 = int(np.rint(f32(f32(a * f32(one - b)) * s)))
        iw10 = int(np.rint(f32(f32(f32(one - a) * b) * s)))
        iw11 = (1 << 14) - iw00 - iw01 - iw10
        return iw00, iw01, iw10, iw11

    def interp(g, wts, shift):
        iw00, iw01, iw10, iw11 = wts
        v = g[:-1, :-1] * iw00 + g[:-1, 1:] * iw01 + g[1:, :-1] * iw10 + g[1:, 1:] * iw11
        return (v + (1 << (shift - 1))) >> shift

    for i in range(n):
        for level in range(maxlevel, -1, -1):
            I = pp[level]
            J = cp[level]
            dIx, dIy = derivs[level]
            h, w = I.shape
            sc = f32(1.0 / (1 << level))
            prevpt = np.array([f32(pts[i, 0] * sc), f32(pts[i, 1] * sc)], f32)
            if level == maxlevel:
                nextpt = np.array([f32(nxt[i, 0] * sc), f32(nxt[i, 1] * sc)], f32)
            else:
                nextpt = np.array([f32(nxt[i, 0] * f32(2)), f32(nxt[i, 1] * f32(2))], f32)
            nxt[i] = nextpt
            prevpt = prevpt - half
            ix, iy = int(np.floor(prevpt[0])), int(np.floor(prevpt[1]))
            if ix < -win or ix >= w or iy < -win or iy >= h:
                if level == 0:
                    status[i] = 0
                    err[i] = 0
                continue
            a = f32(prevpt[0] - f32(ix))
            b = f32(prevpt[1] - f32(iy))
            wts = weights(a, b)
            Iw = interp(gather_u8(I, ix, iy), wts, 14 - 5)
            Ixw = interp(gather_d(dIx, ix, iy), wts, 14)
            Iyw = interp(gather_d(dIy, ix, iy), wts, 14)
            A11 = f32(f32(int((Ixw * Ixw).sum())) * flt_scale)
            A12 = f32(f32(int((Ixw * Iyw).sum())) * flt_scale)
            A22 = f32(f32(int((Iyw * Iyw).sum())) * flt_scale)
            D = f32(f32(A11 * A22) - f32(A12 * A12))
            t = f32(f32(f32(A11 - A22) * f32(A11 - A22)) + f32(f32(f32(4) * A12) * A12))
            mineig = f32(f32(f32(A22 + A11) - f32(np.sqrt(t))) / f32(2 * win * win))
            err[i] = mineig
            if mineig < f32(1e-4) or D < np.finfo(f32).eps:
                if level == 0:
                    status[i] = 0
                continue
            D = f32(f32(1.0) / D)
            nextpt = nextpt - half
            prevdelta = np.zeros(2, f32)
            for j in range(maxit):
                jx, jy = int(np.floor(nextpt[0])), int(np.floor(nextpt[1]))
                if jx < -win or jx >= w or jy < -win or jy >= h:
                    if level == 0:
                        status[i] = 0
                    break
                a = f32(nextpt[0] - f32(jx))
                b = f32(nextpt[1] - f32(jy))
                wts = weights(a, b)
                Jw = interp(gather_u8(J, jx, jy), wts, 14 - 5)
                diff = Jw - Iw
                b1 = f32(f32(int((diff * Ixw).sum())) * flt_scale)
                b2 = f32(f32(int((diff * Iyw).sum())) * flt_scale)
                dx = f32(f32(f32(A12 * b2) - f32(A22 * b1)) * D)
                dy = f32(f32(f32(A12 * b1) - f32(A11 * b2)) * D)
                nextpt = np.array([f32(nextpt[0] + dx), f32(nextpt[1] + dy)], f32)
                nxt[i] = nextpt + half
                if float(dx) * float(dx) + float(dy) * float(dy) <= eps2:
                    break
                if j > 0 and abs(float(f32(dx + prevdelta[0]))) < 0.01 and abs(float(f32(dy + prevdelta[1]))) < 0.01:
                    nxt[i] = np.array([f32(nxt[i, 0] - f32(dx * f32(0.5))), f32(nxt[i, 1] - f32(dy * f32(0.5)))], f32)
                    break
                prevdelta = np.array([dx, dy], f32)
    return nxt, status, err


def fb_klt_ref(prev, cur, kps, priors, win=9, nbpyrlvl=3, ferr=30.0, fb_dist=0.5, maxit=30, eps=KLT_EPS):
    return _fb_klt(_lk_ref, prev, cur, kps, priors, win, nbpyrlvl, ferr, fb_dist, maxit, eps)


# ------------------------------------------------------------------ C: CLAHE
def clahe_cv2(im: np.ndarray, clip: float = 3.0, tiles=None) -> np.ndarray:
    """pclahe_->apply with cv::createCLAHE(fclahe_val, Size(W/50, H/50)) (ov2slam.cpp:85-89)."""
    h, w = im.shape
    tx, ty = tiles if tiles is not None else (w // 50, h // 50)
    return cv2.createCLAHE(clip, (tx, ty)).apply(im)


def clahe_ref(im: np.ndarray, clip: float = 3.0, tiles=None) -> np.ndarray:
    """numpy restatement of cv::CLAHE (SURVEY.md A.6)."""
    f32 = np.float32
    h, w = im.shape
    tx, ty = tiles if tiles is not None else (w // 50, h // 50)
    ew, eh = w, h
    if w % tx != 0 or h % ty != 0:
        ew, eh = w + (tx - w % tx), h + (ty - h % ty)
    ext = im[np.ix_(_reflect101(np.arange(eh), h), _reflect101(np.arange(ew), w))]
    tw, th = ew // tx, eh // ty
    area = tw * th
    cl = max(int(clip * area / 256), 1) if clip > 0 else 1 << 30
    lut = np.zeros((ty, tx, 256), np.uint8)
    scale = f32(255) / f32(area)
    for j in range(ty):
        for i in range(tx):
            hist = np.bincount(ext[j * th:(j + 1) * th, i * tw:(i + 1) * tw].ravel(), minlength=256).astype(np.int64)
            excess = int(np.maximum(hist - cl, 0).sum())
            hist = np.minimum(hist, cl)
            batch = excess // 256
            resid = excess - batch * 256
            hist += batch
            if resid:
                step = max(256 // resid, 1)
                idx = np.arange(0, 256, step)[:resid]
                hist[idx] += 1
            lut[j, i] = np.clip(np.rint(np.cumsum(hist).astype(f32) * scale), 0, 255).astype(np.uint8)
    inv_tw, inv_th = f32(1.0) / f32(tw), f32(1.0) / f32(th)
    txf = (np.arange(w, dtype=f32) * inv_tw - f32(0.5)).astype(f32)
    tyf = (np.arange(h, dtype=f32) * inv_th - f32(0.5)).astype(f32)
    tx1 = np.floor(txf).astype(np.int64)
    ty1 = np.floor(tyf).astype(np.int64)
    xa = (txf - tx1.astype(f32)).astype(f32)[None, :]
    ya = (tyf - ty1.astype(f32)).astype(f32)[:, None]
    tx2 = np.minimum(tx1 + 1, tx - 1)
    ty2 = np.minimum(ty1 + 1, ty - 1)
    tx1 = np.maximum(tx1, 0)
    ty1 = np.maximum(ty1, 0)
    v = im.astype(np.int64)
    g = lambda a, b: lut[a[:, None], b[None, :], v].astype(f32)
    xa1, ya1 = (f32(1) - xa).astype(f32), (f32(1) - ya).astype(f32)
    top = ((g(ty1, tx1) * xa1).astype(f32) + (g(ty1, tx2) * xa).astype(f32)).astype(f32)
    bot = ((g(ty2, tx1) * xa1).astype(f32) + (g(ty2, tx2) * xa).astype(f32)).astype(f32)
    res = ((top * ya1).astype(f32) + (bot * ya).astype(f32)).astype(f32)
    return np.clip(np.rint(res), 0, 255).astype(np.uint8)


# ------------------------------------------------------------------ whole per-frame sequence
def detect_grid_fast_cv2(im, cellsize, curkps, fast_th):
    """detectGridFAST including cornerSubPix; returns (pts float32[N,2], int pts, new_th)."""
    ipts, th, _ = detect_grid_fast_nosubpix(im, cellsize, curkps, fast_th, use_cv2=True)
    return corner_subpix_cv2(im, ipts.astype(np.float32)), ipts, th


def detect_grid_fast_ref(im, cellsize, curkps, fast_th):
    ipts, th, _ = detect_grid_fast_nosubpix(im, cellsize, curkps, fast_th, use_cv2=False)
    return corner_subpix_ref(im, ipts.astype(np.float32)), ipts, th


# ------------------------------------------------------------------ D: detectSingleScale ("next" row, SURVEY.md 8f-1)
# FeatureExtractor::detectSingleScale (/root/reference/src/feature_extractor.cpp:288-440): per cell
# GaussianBlur(im(hroi), 3x3) -> cornerMinEigenVal(3, 3) -> arg-max of (response * mask) twice with the
# same disc mask as detectGridFAST, adaptive dmaxquality_, then cornerSubPix.
#
# Pinned OpenCV semantics (cv2 4.13, x86 SIMD128 build, found by probing; tests/test_oracle_image.py):
#  * cv::GaussianBlur on a SUB-MATRIX (im(hroi) is one, unless the cell is the whole image) does not take
#    the fixed-point path (smooth.dispatch.cpp: only when !isSubmatrix() or BORDER_ISOLATED); it runs
#    sepFilter2D with [0.25 0.5 0.25] on the 8-bit integer engine, border pixels taken from the PARENT
#    image (REFLECT_101 only at the image edge).  The exact value is S/16, S = [1 2 1]x[1 2 1] window sum;
#    the vectorised column filter rounds it half-to-EVEN for the first 16*floor(cs/16) columns of the
#    cell, the scalar tail rounds half-UP.  (Python cannot hand OpenCV a sub-matrix with a parent, so the
#    parent-border rule is OpenCV's documented FilterEngine behaviour, not probed; the rounding rule is
#    probed on isolated cs-wide arrays.)
#  * cornerMinEigenVal(filtered, 3, 3) on the cell's own Mat (REFLECT_101 at the CELL border), float32:
#    scale s = 1/(4*3*255); k1 = float32(s), k2 = float32(2 s);
#    Dx = fma(r(y-1)+r(y+1), k1, r(y)*k2), r = right - left (exact);
#    Dy = q(y+1) - q(y-1), q = row filter [k1 k2 k1]: fma(k1,C, fma(k2,B, k1*A)) for the first
#    32*floor(cs/32) columns, ((k1*A + k2*B) + k1*C) without contraction for the tail;
#    products Dx*Dx, Dx*Dy, Dy*Dy in float32; 3x3 box sums accumulated in float64 (exact) -> float32;
#    response = (a + c) - sqrt((a - c)^2 + b^2), a = Sxx/2, c = Syy/2, b = Sxy, no contraction.
#  * cv::minMaxLoc returns the FIRST maximum in row-major order.


def blur3_cell_ref(im: np.ndarray, x: int, y: int, cs: int) -> np.ndarray:
    """GaussianBlur(im(Rect(x, y, cs, cs)), 3x3, 0) as the reference's sub-matrix call evaluates it."""
    h, w = im.shape
    ys = _reflect101(np.arange(y - 1, y + cs + 1), h)
    xs = _reflect101(np.arange(x - 1, x + cs + 1), w)
    p = im[np.ix_(ys, xs)].astype(np.int32)
    rows = p[:, :-2] + 2 * p[:, 1:-1] + p[:, 2:]
    S = rows[:-2] + 2 * rows[1:-1] + rows[2:]
    even = np.rint(S / 16.0).astype(np.int32)      # numpy rint = half-to-even
    up = (S + 8) >> 4
    nvec = (cs // 16) * 16
    out = up.copy()
    out[:, :nvec] = even[:, :nvec]
    return out.astype(np.uint8)


def blur3_cell_cv2(im: np.ndarray, x: int, y: int, cs: int) -> np.ndarray:
    """Same, composed from cv2 calls: whole-image sepFilter2D (vector path: half-even everywhere for
    widths that are multiples of 16) and whole-image GaussianBlur (fixed point: half-up)."""
    k = np.array([0.25, 0.5, 0.25], np.float32)
    h, w = im.shape
    pad = (-w) % 16
    src = cv2.copyMakeBorder(im, 0, 0, 0, pad, cv2.BORDER_REFLECT_101) if pad else im
    # (REFLECT_101 padding puts column w-2 at column w: the right neighbour the image edge would use)
    even = cv2.sepFilter2D(src, cv2.CV_8U, k, k)[:, :w]
    up = cv2.GaussianBlur(im, (3, 3), 0)
    nvec = (cs // 16) * 16
    out = up[y:y + cs, x:x + cs].copy()
    out[:, :nvec] = even[y:y + cs, x:x + nvec]
    return out


_SS_K1 = np.float32(1.0 / (4 * 3 * 255.0))
_SS_K2 = np.float32(2.0 / (4 * 3 * 255.0))


def min_eigen_ref(cell: np.ndarray) -> np.ndarray:
    """cv::cornerMinEigenVal(cell, dst, 3, 3) (8-bit cell, BORDER_REFLECT_101), float32, exact op order."""
    hh, ww = cell.shape
    p = np.pad(cell.astype(np.int32), 1, mode="reflect").astype(np.float32)
    k1, k2 = _SS_K1, _SS_K2
    r = p[:, 2:] - p[:, :-2]
    dx = _fma32(r[:-2] + r[2:], k1, (r[1:-1] * k2).astype(np.float32))
    A, B, C = p[:, :-2], p[:, 1:-1], p[:, 2:]
    qf = _fma32(k1, C, _fma32(k2, B, (k1 * A).astype(np.float32)))
    qp = (((k1 * A).astype(np.float32) + (k2 * B).astype(np.float32)).astype(np.float32) + (k1 * C).astype(np.float32)).astype(np.float32)
    nvec = (ww // 32) * 32
    q = qp.copy()
    q[:, :nvec] = qf[:, :nvec]
    dy = (q[2:] - q[:-2]).astype(np.float32)

    def box(v):
        pp = np.pad(v.astype(np.float64), 1, mode="reflect")
        acc = np.zeros((hh, ww), np.float64)
        for i in range(3):
            for j in range(3):
                acc += pp[i:i + hh, j:j + ww]
        return acc.astype(np.float32)

    sxx, sxy, syy = box((dx * dx).astype(np.float32)), box((dx * dy).astype(np.float32)), box((dy * dy).astype(np.float32))
    a = (sxx * np.float32(0.5)).astype(np.float32)
    c = (syy * np.float32(0.5)).astype(np.float32)
    t = (a - c).astype(np.float32)
    qq = ((t * t).astype(np.float32) + (sxy * sxy).astype(np.float32)).astype(np.float32)
    return ((a + c).astype(np.float32) - np.sqrt(qq).astype(np.float32)).astype(np.float32)


def _first_max(hm: np.ndarray):
    """cv::minMaxLoc's maximum: value and (x, y) of the first occurrence in row-major order."""
    i = int(np.argmax(hm))          # numpy returns the first occurrence as well
    return float(hm.flat[i]), i % hm.shape[1], i // hm.shape[1]


def detect_single_scale_nosubpix(im: np.ndarray, cellsize: int, curkps, roi, dmaxquality: float, use_cv2: bool):
    """detectSingleScale up to (not including) cornerSubPix, sequential ascending cell order (the
    reference's parallel_for_ body races on `mask` and `nboccup`).  roi = (x, y, w, h).
    Returns (pts int32[N,2]: first detections in cell order then the admitted second detections,
    new dmaxquality, nboccup)."""
    rows, cols = im.shape
    r4 = cellsize // 4
    nh, nw = rows // cellsize, cols // cellsize
    nbcells = nh * nw
    occ = np.zeros((nh + 1, nw + 1), bool)
    mask = np.ones((rows, cols), np.float32)
    hw = circle_halfwidths(r4)
    for px in np.asarray(curkps, np.float32).reshape(-1, 2):
        occ[int(np.float32(px[1]) / np.float32(cellsize)), int(np.float32(px[0]) / np.float32(cellsize))] = True
        if use_cv2:
            cv2.circle(mask, (_cv_round(px[0]), _cv_round(px[1])), r4, 0, -1)
        else:
            paint_disc(mask, _cv_round(px[0]), _cv_round(px[1]), hw)
    rx, ry, rw, rh = (int(v) for v in roi)
    first = [[] for _ in range(nbcells)]
    second = [[] for _ in range(nbcells)]
    nboccup = 0

    def paint(px, py):
        if use_cv2:
            cv2.circle(mask, (px, py), r4, 0, -1)
        else:
            paint_disc(mask, px, py, hw)

    for i in range(nbcells):
        r, c = i // nw, i % nw
        if occ[r, c]:
            nboccup += 1
            continue
        x, y = c * cellsize, r * cellsize
        if not (x + cellsize < cols - 1 and y + cellsize < rows - 1):
            continue
        if use_cv2:
            hmap = cv2.cornerMinEigenVal(blur3_cell_cv2(im, x, y, cellsize), 3, 3)
        else:
            hmap = min_eigen_ref(blur3_cell_ref(im, x, y, cellsize))
        for store in (first, second):
            prod = (hmap * mask[y:y + cellsize, x:x + cellsize]).astype(np.float32)
            if use_cv2:
                _, mx, _, loc = cv2.minMaxLoc(prod)
                px, py = loc[0] + x, loc[1] + y
            else:
                mx, lx, ly = _first_max(prod)
                px, py = lx + x, ly + y
            if px < rx or py < ry or px >= rx + rw or py >= ry + rh:
                break            # `continue` of the cell loop: no second detection either
            if mx >= dmaxquality:
                store[i].append((px, py))
                paint(px, py)
    out = [p for v in first for p in v]
    nbkps = len(out)
    if nbkps + nboccup < nbcells:
        nbsec = nbcells - (nbkps + nboccup)
        k = 0
        for v in second:
            if v:
                out.append(v[-1])
                k += 1
                if k == nbsec:
                    break
    nbkps = len(out)
    q = float(dmaxquality)
    if nbkps < 0.33 * (nbcells - nboccup):
        q /= 2.0
    elif nbkps > 0.9 * (nbcells - nboccup):
        q *= 1.5
    return np.array(out, np.int32).reshape(-1, 2), q, nboccup


def detect_single_scale_cv2(im, cellsize, curkps, roi, dmaxquality):
    ipts, q, _ = detect_single_scale_nosubpix(im, cellsize, curkps, roi, dmaxquality, use_cv2=True)
    return corner_subpix_cv2(im, ipts.astype(np.float32)) if len(ipts) else np.zeros((0, 2), np.float32), ipts, q


def detect_single_scale_ref(im, cellsize, curkps, roi, dmaxquality):
    ipts, q, _ = detect_single_scale_nosubpix(im, cellsize, curkps, roi, dmaxquality, use_cv2=False)
    return corner_subpix_ref(im, ipts.astype(np.float32)) if len(ipts) else np.zeros((0, 2), np.float32), ipts, q


def frontend_frame_cv2(prev, cur, kps, priors, is3d, cellsize, fast_th):
    """The per-frame reference sequence the benchmark times on the CPU (SURVEY.md 8d):
    pyramids (visual_front_end.cpp:1172), two fbKltTracking calls (:196 nbpyrlvl=1 on the
    3D-prior subset, :242 nbpyrlvl=3 on the rest), then createKeyframe's detect + describe
    (map_manager.cpp:286-341) on the current image with the surviving tracks as vcurkps."""
    cv2.buildOpticalFlowPyramid(prev, (9, 9), 3)
    cv2.buildOpticalFlowPyramid(cur, (9, 9), 3)
    kps = np.asarray(kps, np.float32).reshape(-1, 2)
    n = len(kps)
    tracked = np.asarray(priors, np.float32).reshape(-1, 2).copy()
    status = np.zeros(n, np.uint8)
    i3 = np.nonzero(is3d)[0]
    i2 = np.nonzero(~np.asarray(is3d, bool))[0]
    if len(i3):
        tracked[i3], status[i3] = fb_klt_cv2(prev, cur, kps[i3], tracked[i3], 9, 1)
    if len(i2):
        tracked[i2], status[i2] = fb_klt_cv2(prev, cur, kps[i2], tracked[i2], 9, 3)
    alive = tracked[status.astype(bool)]
    d_old, v_old = describe_cv2(cur, alive)
    newpts, ipts, th = detect_grid_fast_cv2(cur, cellsize, alive, fast_th)
    d_new, v_new = describe_cv2(cur, newpts)
    return dict(tracked=tracked, status=status, newpts=newpts, newpts_int=ipts, fast_th=th,
                desc_old=d_old, valid_old=v_old, desc_new=d_new, valid_new=v_new)


# ------------------------------------------------------------------ 8f-3: getLineMinSAD
def get_rect_subpix_u8_ref(src, ws, cx, cy):
    """cv::getRectSubPix 8u->8u as OpenCV's own template computes it (imgproc/samplers.cpp: 16-bit fixed-point bilinear
    weights, (sum + 2^15) >> 16, replicated border) - float32 arithmetic mirrored step by step.  (IPP builds of OpenCV
    route this call to ippiCopySubpix, which differs by one grey level on ~0.7 % of the pixels.)"""
    f = np.float32
    cx = f(cx) - f((ws - 1) * 0.5)
    cy = f(cy) - f((ws - 1) * 0.5)
    ipx, ipy = int(np.floor(cx)), int(np.floor(cy))
    a, b = f(cx - f(ipx)), f(cy - f(ipy))
    one = f(1.0)
    rnd = lambda v: int(np.rint(f(v)))
    a11, a12 = rnd((one - a) * (one - b) * f(65536)), rnd(a * (one - b) * f(65536))
    a21, a22 = rnd((one - a) * b * f(65536)), rnd(a * b * f(65536))
    h, w = src.shape
    ys = np.clip(np.arange(ipy, ipy + ws + 1), 0, h - 1)
    xs = np.clip(np.arange(ipx, ipx + ws + 1), 0, w - 1)
    p = src[np.ix_(ys, xs)].astype(np.int64)
    v = p[:-1, :-1] * a11 + p[:-1, 1:] * a12 + p[1:, :-1] * a21 + p[1:, 1:] * a22
    return ((v + (1 << 15)) >> 16).astype(np.uint8)


def line_min_sad_ref(iml, imr, pt, nwinsize, goleft, subpix=get_rect_subpix_u8_ref):
    """FeatureTracker::getLineMinSAD (/root/reference/src/feature_tracker.cpp:138-204) restated; `subpix` = the
    getRectSubPix to use (the OpenCV template above, or cv2's).  Returns (xprior, l1err); l1err is None where the
    reference returns before setting it."""
    f = np.float32
    if nwinsize % 2 == 0:
        return -1.0, None
    x, y = f(pt[0]), f(pt[1])
    hw = nwinsize // 2
    rows, cols = imr.shape
    if x - hw < 0:
        hw = int(f(hw) + (x - f(hw)))
    if x + hw >= cols:
        hw = int(f(hw) + (x + f(hw) - f(cols) - f(1)))
    if y - hw < 0:
        hw = int(f(hw) + (y - f(hw)))
    if y + hw >= rows:
        hw = int(f(hw) + (y + f(hw) - f(rows) - f(1)))
    if hw <= 0:
        return -1.0, None
    ws = 2 * hw + 1
    patch = subpix(iml, ws, x, y).astype(np.int64)
    minsad, xprior = f(255.0), f(-1.0)
    c = x
    while (c >= hw) if goleft else (c < cols - hw):
        e = f(f(np.abs(patch - subpix(imr, ws, c, y).astype(np.int64)).sum()) / f(ws * ws))
        if e < minsad:
            minsad, xprior = e, c
        c = f(c - f(1)) if goleft else f(c + f(1))
    return float(xprior), float(minsad)
