"""CPU tests: the oracle's numpy restatement (what documents the semantics the CUDA kernels
implement) is pinned against the real OpenCV the reference calls (cv2 4.13) and against the
committed golden vectors generated from cv2 (scripts/make_golden.py)."""
import hashlib
from pathlib import Path

import numpy as np
import pytest

from oracle import image_ref as R
from ov2slam_b200 import synth

GOLD = Path(__file__).parent / "golden" / "frontend_golden.npz"
needs_cv2 = pytest.mark.skipif(not R.HAVE_CV2, reason="cv2 not importable")


@pytest.fixture(scope="module")
def gold():
    g = np.load(GOLD)
    prev, cur, flow = synth.make_pair(int(g["seed"]), int(g["w"]), int(g["h"]))
    assert hashlib.sha256(prev.tobytes() + cur.tobytes()).hexdigest() == str(g["img_sha"]), \
        "synthetic generator drifted: golden inputs no longer reproducible"
    return g, prev, cur, flow


def test_golden_pyramid(gold):
    g, prev, cur, _ = gold
    pyr = R.build_pyramid_ref(cur, 3)
    for l in range(1, 4):
        assert np.array_equal(pyr[l], g[f"pyr{l}"])


@pytest.mark.parametrize("cs", [50, 35, 16])
@pytest.mark.parametrize("tag", ["empty", "kps"])
def test_golden_grid_fast(gold, cs, tag):
    g, prev, _, _ = gold
    ipts, th, _ = R.detect_grid_fast_nosubpix(prev, cs, g[f"fast_{cs}_{tag}_in"], 10, use_cv2=False)
    assert np.array_equal(ipts, g[f"fast_{cs}_{tag}_int"])
    assert th == int(g[f"fast_{cs}_{tag}_th"])


def test_golden_subpix(gold):
    g, prev, _, _ = gold
    ip = g["fast_50_empty_int"]
    sp = R.corner_subpix_ref(prev, ip.astype(np.float32))
    d = np.abs(sp - g["fast_50_empty_subpix"])
    assert d.max() <= 1e-4 and (d == 0).mean() > 0.9


def test_golden_descriptors(gold):
    g, prev, _, _ = gold
    d, v = R.describe_ref(prev, g["desc_pts"])
    assert np.array_equal(v, g["desc_valid"]) and np.array_equal(d, g["desc"])


def test_golden_klt(gold):
    g, prev, cur, _ = gold
    sel = np.r_[0:60, 300:360]   # the python restatement is slow: a subset incl. the random points
    for lvl in (0, 3):
        t, s = R.fb_klt_ref(prev, cur, g["klt_kps"][sel], g["klt_pri"][sel], 9, lvl)
        assert np.array_equal(s, g[f"klt_{lvl}_status"][sel])
        assert np.abs(t - g[f"klt_{lvl}_tracked"][sel]).max() <= 1e-3


@needs_cv2
def test_pyramid_and_scharr_vs_cv2():
    """pyrDown levels and Scharr planes, from the working sizes down to the 16 x 16 minimum of ov2_pyr_create (odd sizes,
    levels of 1 - 2 px at 4 extra levels); the depth buildOpticalFlowPyramid reaches (optflow_levels); reflect-101
    indices that overshoot by more than the image size."""
    import cv2
    sizes = [(640, 480), (333, 245), (1241, 376), (161, 83), (100, 70), (57, 64), (56, 64), (96, 72), (64, 48), (40, 30)]
    sizes += [(w, h) for w in range(16, 40, 3) for h in (16, 17, 23, 31)]
    for w, h in sizes:
        im = synth.make_frame(7, w, h)
        ref = R.build_pyramid_ref(im, 4)
        for l, (a, b) in enumerate(zip(ref, R.build_pyramid_cv2(im, 4))):
            assert np.array_equal(a, b), (w, h, l)
        n, pyr = cv2.buildOpticalFlowPyramid(im, (9, 9), 3)
        assert n == R.optflow_levels(w, h) and len(pyr) == 2 * (n + 1), (w, h, n)
        for l in range(n + 1):
            ix, iy = R.scharr_ref(ref[l])
            assert np.array_equal(pyr[2 * l + 1][..., 0], ix) and np.array_equal(pyr[2 * l + 1][..., 1], iy), (w, h, l)
    zero = np.zeros((1, 1), np.uint8)
    for w in range(16, 205):
        for h in (16, 17, 19, 20, 23, 37, 38, 39, 40, 41, 75, 76, 77, 150, 199):
            n, _ = cv2.buildOpticalFlowPyramid(np.broadcast_to(zero, (h, w)).copy(), (9, 9), 3, withDerivatives=False)
            assert R.optflow_levels(w, h) == n, (w, h, n)
    for n in (1, 2, 3, 5, 12):
        idx = np.arange(-40, 41)
        assert np.array_equal(R._reflect101(idx, n), [cv2.borderInterpolate(int(i), n, cv2.BORDER_REFLECT_101) for i in idx]), n


@needs_cv2
def test_fast_and_circle_vs_cv2():
    import cv2
    im = synth.make_frame(8)
    for th in (0, 1, 6, 10, 20):
        for (x, y, cs) in ((0, 0, 50), (550, 400, 50), (35, 70, 35), (16, 32, 16)):
            roi = np.ascontiguousarray(im[y:y + cs, x:x + cs])
            assert R.fast_detect_ref(roi, th) == R.fast_detect_cv2(roi, th)
    for r in range(1, 33):
        m = np.ones((80, 80), np.float32)
        cv2.circle(m, (40, 40), r, 0, -1)
        m2 = np.ones((80, 80), np.float32)
        R.paint_disc(m2, 40, 40, R.circle_halfwidths(r))
        assert np.array_equal(m, m2), r


@needs_cv2
@pytest.mark.parametrize("cs", [50, 16])
def test_grid_fast_vs_cv2(cs):
    im = synth.make_frame(9)
    rng = np.random.default_rng(cs)
    k = (rng.random((40, 2)) * [640, 480]).astype(np.float32)
    a = R.detect_grid_fast_nosubpix(im, cs, k, 10, True)
    b = R.detect_grid_fast_nosubpix(im, cs, k, 10, False)
    assert np.array_equal(a[0], b[0]) and a[1] == b[1] and a[2] == b[2]


@needs_cv2
def test_get_rect_subpix_and_subpix_vs_cv2():
    import cv2
    im = synth.make_frame(5)
    h, w = im.shape
    rng = np.random.default_rng(3)
    for k in range(300):
        cx = np.float32(rng.choice([rng.uniform(0, 7), rng.uniform(w - 8, w), rng.uniform(8, w - 8)]))
        cy = np.float32(rng.choice([rng.uniform(0, 7), rng.uniform(h - 8, h), rng.uniform(8, h - 8)]))
        ref = cv2.getRectSubPix(im, (9, 9), (float(cx), float(cy)), patchType=cv2.CV_32F)
        assert np.array_equal(R._get_rect_subpix_9(im, cx, cy), ref), (cx, cy)
    ipts, _, _ = R.detect_grid_fast_nosubpix(im, 16, np.zeros((0, 2)), 10, True)
    extra = np.array([[3, 3], [636, 3], [3, 476], [636, 476], [1, 200], [638, 100], [320, 1], [300, 478]], np.int32)
    p = np.concatenate([ipts[:150], extra]).astype(np.float32)
    d = np.abs(R.corner_subpix_cv2(im, p) - R.corner_subpix_ref(im, p))
    assert d.max() <= 1e-4, d.max()
    assert (d == 0).mean() > 0.9


@needs_cv2
def test_descriptor_vs_cv2_and_kernel_constants():
    import cv2
    assert np.array_equal(cv2.getGaussianKernel(7, 2, cv2.CV_32F).ravel(), R.gauss7_kernel())
    # the float32 constants hard-coded in ov2slam_b200/csrc/frontend_desc.cu
    hexes = ["0x1.1f5f62p-4", "0x1.0c70fcp-3", "0x1.869472p-3", "0x1.ba95c0p-3"]
    assert [float.fromhex(x) for x in hexes] == [float(v) for v in R.gauss7_kernel()[:4]]
    bad = tot = 0
    for seed, (w, h) in enumerate([(640, 480), (752, 480)]):
        im = synth.make_frame(100 + seed, w, h)
        rng = np.random.default_rng(seed)
        pts = (rng.random((600, 2)) * [w, h]).astype(np.float32)
        pts[:80] = np.floor(pts[:80]) + 0.5
        pts[80:120, 0] = rng.uniform(29.5, 32.5, 40)
        pts[120:160, 0] = rng.uniform(w - 32.5, w - 29.5, 40)
        da, va = R.describe_cv2(im, pts)
        db, vb = R.describe_ref(im, pts)
        assert np.array_equal(va, vb)
        bad += int(np.unpackbits(da ^ db).sum())
        tot += int(va.sum()) * 256
    assert bad == 0 and tot > 100000


@needs_cv2
def test_klt_vs_cv2():
    prev, cur, flow = synth.make_pair(7)
    rng = np.random.default_rng(0)
    ipts, _, _ = R.detect_grid_fast_nosubpix(prev, 16, np.zeros((0, 2)), 10, True)
    b = (rng.random((40, 2)) * [640, 480]).astype(np.float32)
    b[:10, 0] = rng.uniform(0, 7, 10)
    b[10:20, 0] = rng.uniform(632, 640, 10)
    b[20:30, 1] = rng.uniform(0, 7, 10)
    b[30:, 1] = rng.uniform(472, 480, 10)
    kps = np.concatenate([R.corner_subpix_cv2(prev, ipts[:80].astype(np.float32)), b])
    _, pri = synth.make_priors(7, kps, flow)
    for lvl in (0, 1, 3):
        ta, sa = R.fb_klt_cv2(prev, cur, kps, pri, 9, lvl)
        tb, sb = R.fb_klt_ref(prev, cur, kps, pri, 9, lvl)
        assert np.array_equal(sa, sb)
        assert np.abs(ta - tb).max() <= 1e-3
    # small images: buildOpticalFlowPyramid stops before a level <= 9 px, so calcOpticalFlowPyrLK tracks from fewer levels
    # than asked (96 x 72 and 64 x 48: 2, 40 x 30: 1, 17 x 16: 0), and windows overshoot the narrow levels by more than
    # one reflection.  Statuses identical, tracked positions within the GPU suite's cv2 tolerance (1e-2 px; a lost track
    # can end anywhere).
    for w, h in ((17, 16), (40, 30), (64, 48), (96, 72), (161, 83), (333, 245)):
        prev, cur, _ = synth.make_pair(7, w, h)
        rng = np.random.default_rng(w)
        kps = (rng.random((150, 2)) * [w, h]).astype(np.float32)
        kps[:4] = [[1.0, 1.0], [w - 1.0, h / 2], [w / 2, h - 1.0], [w - 1.5, h - 1.5]]
        pri = (kps + rng.uniform(-1.5, 1.5, kps.shape)).astype(np.float32)
        for lvl in (1, 3):
            ta, sa = R.fb_klt_cv2(prev, cur, kps, pri, 9, lvl)
            tb, sb = R.fb_klt_ref(prev, cur, kps, pri, 9, lvl)
            assert np.array_equal(sa, sb), (w, h, lvl, np.nonzero(sa != sb)[0])
            ok = sa.astype(bool)
            assert ok.sum() >= 10, (w, h, lvl)
            assert np.abs(ta[ok] - tb[ok]).max() <= 1e-2, (w, h, lvl, np.abs(ta[ok] - tb[ok]).max())


@needs_cv2
@pytest.mark.parametrize("w,h", [(1280, 720), (752, 480), (640, 480), (1000, 720)])
def test_clahe_vs_cv2(w, h):
    im = synth.make_frame(3, w, h)
    assert np.array_equal(R.clahe_ref(im), R.clahe_cv2(im))


# ---------------------------------------------------------------- detectSingleScale ("next" row 8f-1)
@needs_cv2
def test_single_scale_blur_rounding_rule_vs_cv2():
    """GaussianBlur on the reference's cell sub-matrix = sepFilter2D's 8-bit engine: S/16 rounded
    half-to-even in the vectorised first 16*floor(cs/16) columns, half-up in the scalar tail.  Probed on
    isolated cs-wide arrays (interior pixels: the border of an isolated array is not the sub-matrix's)
    and against the whole-image composition the cv2 arm of the oracle uses."""
    import cv2
    im = synth.make_frame(3, 640, 480)
    k = np.array([0.25, 0.5, 0.25], np.float32)
    for cs in (50, 35, 16, 20):
        crop = im[100:100 + cs, 200:200 + cs].copy()
        f = cv2.sepFilter2D(crop, cv2.CV_8U, k, k)
        ref = R.blur3_cell_ref(im, 200, 100, cs)
        assert np.array_equal(f[1:-1, 1:-1], ref[1:-1, 1:-1])
        # both rounding modes must actually occur in the tail / body for the probe to mean anything
        S16 = ref.astype(np.int32)
        assert S16.size
    for (x, y, cs) in [(0, 0, 50), (100, 150, 50), (550, 400, 50), (35, 70, 35), (0, 445, 35), (605, 0, 35), (16, 16, 16)]:
        assert np.array_equal(R.blur3_cell_cv2(im, x, y, cs), R.blur3_cell_ref(im, x, y, cs))
    im2 = synth.make_frame(4, 333, 245)      # width not a multiple of 16: padded composition
    for (x, y, cs) in [(0, 0, 35), (280, 175, 35), (298, 210, 35)]:
        assert np.array_equal(R.blur3_cell_cv2(im2, x, y, cs), R.blur3_cell_ref(im2, x, y, cs))


@needs_cv2
def test_min_eigen_ref_vs_cv2():
    """cornerMinEigenVal(cell, 3, 3) restated in float32 with OpenCV's operation order (FMA in the Sobel
    filters, 32-column vector / scalar-tail split of the Dy row filter, exact 3x3 sums, no contraction in
    the eigenvalue).  Bit-exact except where cv2 breaks a float32 rounding TIE of a box sum the other way
    (~4e-5 of the sums; moves the response by a few ulp) - bounded here at 1e-4 of the pixels, 16 ulp."""
    import cv2
    cv2.setNumThreads(1)
    rng = np.random.default_rng(0)
    npx = nbad = 0
    worst = 0
    for it in range(120):
        cs = int(rng.choice([50, 35, 16, 20, 33]))
        c = (rng.random((cs + 8, cs + 8)) * 255).astype(np.uint8)
        c = cv2.GaussianBlur(c, (5, 5), 1.0)[4:-4, 4:-4].copy() if it % 2 else c[4:-4, 4:-4].copy()
        a, b = cv2.cornerMinEigenVal(c, 3, 3), R.min_eigen_ref(c)
        d = a != b
        npx += d.size
        nbad += int(d.sum())
        if d.any():
            worst = max(worst, int(np.abs(a[d].view(np.int32).astype(np.int64) - b[d].view(np.int32).astype(np.int64)).max()))
    assert nbad <= 1e-4 * npx and worst <= 16, (nbad, npx, worst)


@needs_cv2
def test_first_max_is_minmaxloc_semantics():
    import cv2
    rng = np.random.default_rng(1)
    for _ in range(200):
        hm = rng.integers(0, 4, (7, 9)).astype(np.float32)      # many ties, zeros
        if rng.random() < 0.2:
            hm[:] = 0
        _, mx, _, loc = cv2.minMaxLoc(hm)
        v, x, y = R._first_max(hm)
        assert (x, y) == loc and v == mx


@needs_cv2
@pytest.mark.parametrize("cs", [50, 35])
def test_detect_single_scale_ref_vs_cv2(cs):
    """Whole detectSingleScale flow (occupancy, disc mask, two arg-max rounds, roi test, second
    detections, dmaxquality_ adaptation, cornerSubPix): numpy restatement vs the cv2 call sequence."""
    w, h = 640, 480
    rng = np.random.default_rng(cs)
    for seed, nk, roi, q in [(11, 0, (0, 0, w, h), 0.001), (12, 40, (0, 0, w, h), 0.001), (13, 15, (20, 20, w - 40, h - 40), 0.0001),
                             (14, 0, (0, 0, w, h), 0.05)]:
        im = synth.make_frame(seed, w, h)
        kps = (rng.random((nk, 2)) * [w, h]).astype(np.float32)
        if nk:
            kps[0] = [0.4, 0.4]
            kps[1] = [w - 1.0, h - 1.0]
        pc, ic, qc = R.detect_single_scale_cv2(im, cs, kps, roi, q)
        pr, ir, qr = R.detect_single_scale_ref(im, cs, kps, roi, q)
        assert np.array_equal(ic, ir) and qc == qr
        assert len(ic) > 0 or q > 0.01
        if len(ic):
            assert np.abs(pc - pr).max() <= 2e-4


SS_GOLD = Path(__file__).parent / "golden" / "single_scale_golden.npz"


@pytest.mark.parametrize("cs", [50, 35])
@pytest.mark.parametrize("tag", ["empty", "kps_roi"])
def test_golden_single_scale(cs, tag):
    """Oracle restatement vs the committed cv2-generated vectors (scripts/make_golden_single_scale.py)."""
    g = np.load(SS_GOLD)
    im = synth.make_frame(int(g["seed"]), int(g["w"]), int(g["h"]))
    assert hashlib.sha256(im.tobytes()).hexdigest() == str(g["img_sha"]), "synthetic generator drifted"
    sp, ip, qn = R.detect_single_scale_ref(im, cs, g[f"ss_{cs}_{tag}_in"], tuple(int(v) for v in g[f"ss_{cs}_{tag}_roi"]),
                                           float(g[f"ss_{cs}_{tag}_q"][0]))
    assert np.array_equal(ip, g[f"ss_{cs}_{tag}_int"])
    assert qn == float(g[f"ss_{cs}_{tag}_q"][1])
    assert np.abs(sp - g[f"ss_{cs}_{tag}_subpix"]).max() <= 2e-4


def _random_brief_pairs(seed=0):
    """A stand-in for opencv_contrib's generated_32.i (not redistributable / not in this image): 256 test pairs drawn the
    way BRIEF draws them (isotropic Gaussian, sigma = PATCH_SIZE / 5, clipped to the 48 x 48 patch)."""
    rng = np.random.default_rng(seed)
    return np.clip(np.rint(rng.normal(0, 48 / 5.0, (256, 4))), -24, 24).astype(np.int8)


def test_brief32_restatement_matches_direct_box_sums():
    """brief32_ref (integral image, as brief.cpp does it) against the definition evaluated directly: 9 x 9 box sums
    around (int)(pt + 0.5), first test of a byte in bit 7, 28-pixel border on the rounded point."""
    rng = np.random.default_rng(5)
    im = rng.integers(0, 256, (120, 160), dtype=np.uint8)
    pairs = _random_brief_pairs(1)
    pts = np.concatenate([rng.uniform(20, 140, (40, 2)), [[27.4, 60.0], [27.5, 60.0], [28.5, 60.2], [131.49, 91.5], [131.5, 91.49], [60.5, 28.5]]]).astype(np.float32)
    pts[:, 1] = np.clip(pts[:, 1], 0, 119)
    desc, valid = R.brief32_ref(im, pts, pairs)
    imp = np.pad(im, ((0, 1), (0, 1)), mode="edge").astype(np.int64)
    for i, (x, y) in enumerate(pts):
        rx, ry = R._cv_round(x), R._cv_round(y)
        ok = 28 <= rx < 160 - 28 and 28 <= ry < 120 - 28
        assert valid[i] == int(ok)
        if not ok:
            assert not desc[i].any()
            continue
        cx, cy = int(float(x) + 0.5), int(float(y) + 0.5)
        box = lambda dy, dx: int(imp[cy + dy - 4:cy + dy + 5, cx + dx - 4:cx + dx + 5].sum())
        for byte in range(32):
            v = 0
            for k in range(8):
                y0, x0, y1, x1 = (int(t) for t in pairs[byte * 8 + k])
                v |= int(box(y0, x0) < box(y1, x1)) << (7 - k)
            assert desc[i, byte] == v
    assert valid.sum() > 20
