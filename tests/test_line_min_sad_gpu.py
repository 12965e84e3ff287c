"""GPU tests of ov2_line_min_sad (FeatureTracker::getLineMinSAD for a batch of points): columns and errors equal float for float
to oracle/image_ref.py::line_min_sad_ref.

Covered: every odd window from 3 to 15 on levels 0-3 of the EuRoC, KITTI, 1280 x 720 and TartanAir pyramids, both scan
directions; points within the last float steps below the right and bottom edges, where the reference's border rule grows the
half window (to 4 h0 - 3 under float rounding: 23 on EuRoC's level 3 and 25 on a 64 x 64 level for window 15); points past
the right and bottom edges on both sides of the built bound of 25; ragged frame indices, fixed strides with a partial last
frame, first_frame > 0 and frames that differ; empty slots, NaN coordinates and n = 0; ties on constant and periodic pairs
(the first minimum in scan order wins, across lanes and rounds of the warp scan) and errors saturated at 255; every refusal,
with the outputs left untouched.
"""
import numpy as np
import pytest

from ov2slam_b200 import api, synth
from oracle import image_ref as R

gpu = pytest.mark.gpu

f32 = np.float32
WINDOWS = range(3, 17, 2)
MAX_HW = 25                         # the half window ov2_line_min_sad is built for (include/ov2b200.h)
GEOMETRIES = {"euroc": (752, 480), "kitti": (1241, 376), "c4": (1280, 720), "tartanair": (640, 480)}


def grown_halfwin(x, y, cols, rows, nwinsize):
    """The half window getLineMinSAD tracks after its four border tests, in the reference's float32 arithmetic."""
    x, y = f32(x), f32(y)
    hw = nwinsize // 2
    if x - f32(hw) < 0:
        hw = int(f32(hw) + (x - f32(hw)))
    if x + f32(hw) >= f32(cols):
        hw = int(f32(hw) + (x + f32(hw) - f32(cols) - f32(1)))
    if y - f32(hw) < 0:
        hw = int(f32(hw) + (y - f32(hw)))
    if y + f32(hw) >= f32(rows):
        hw = int(f32(hw) + (y + f32(hw) - f32(rows) - f32(1)))
    return hw


def test_grown_halfwin_reaches_4h0_minus_3():
    """The float rounding the kernel's bound rests on (runs without a GPU)."""
    x, y = np.nextafter(f32(94), f32(0)), np.nextafter(f32(60), f32(0))
    assert (x, y) == (f32(93.99999237), f32(59.99999619)) and grown_halfwin(x, y, 94, 60, 15) == 23
    e = np.nextafter(f32(64), f32(0))
    assert grown_halfwin(e, e, 64, 64, 15) == 25
    for ws in WINDOWS:
        worst = max(grown_halfwin(x, y, c, r, ws) for c, r in ((94, 60), (64, 64), (80, 60), (156, 47), (188, 120))
                    for x, y in _edge_points(c, r, ws // 2))
        assert worst == 4 * (ws // 2) - 3, ws


def _pair(seed, w, h, frames=1, shift=9):
    """Left images and their right copies moved `shift` px to the left (random columns fill the right edge)."""
    lefts = np.stack([synth.make_frame(seed + k, w, h, nrect=80) for k in range(frames)])
    rights = np.ascontiguousarray(np.roll(lefts, -shift, axis=2))
    rights[:, :, -shift:] = np.random.default_rng(seed).integers(0, 256, (frames, h, shift)).astype(np.uint8)
    return lefts, rights


def _pyramids(ctx, lefts, rights, extra=3):
    nf, h, w = lefts.shape
    pl, pr = api.Pyramid(ctx, nf, w, h, extra), api.Pyramid(ctx, nf, w, h, extra)
    pl.build(lefts)
    pr.build(rights)
    return pl, pr


def _run(ctx, pl, pr, level, pts, ws, goleft, **addr):
    n = len(pts)
    xp, er = np.full(n, 7.0, f32), np.full(n, 7.0, f32)
    api.FeatureTracker(ctx).line_min_sad(pl, pr, level, np.ascontiguousarray(pts, f32), ws, goleft, xp, er, **addr)
    return xp, er


def _ref(L, Rr, pt, ws, goleft):
    x, e = R.line_min_sad_ref(L, Rr, pt, ws, goleft)
    return f32(x), f32(255.0 if e is None else e)


def _assert_ref(xp, er, levels, pts, ws, goleft, frames=None, what=""):
    for i, p in enumerate(pts):
        L, Rr = levels[0 if frames is None else frames[i]]
        rx, re = _ref(L, Rr, p, ws, goleft)
        assert xp[i].view(np.uint32) == rx.view(np.uint32) and er[i].view(np.uint32) == re.view(np.uint32), \
            (what, ws, goleft, i, tuple(p), float(xp[i]), float(rx), float(er[i]), float(re))


@pytest.fixture(scope="module")
def geometry_pyramids(ctx):
    out = {}
    for name, (w, h) in GEOMETRIES.items():
        lefts, rights = _pair(91, w, h)
        pl, pr = _pyramids(ctx, lefts, rights)
        out[name] = pl, pr, [(pl.download(0, lv), pr.download(0, lv)) for lv in range(4)]
    yield out
    for pl, pr, _ in out.values():
        pl.close()
        pr.close()


@pytest.mark.parametrize("geometry", list(GEOMETRIES))
@gpu
def test_every_window_and_level(ctx, geometry_pyramids, geometry):
    pl, pr, levels = geometry_pyramids[geometry]
    rng = np.random.default_rng(len(geometry))
    for lv in range(4):
        L, Rr = levels[lv]
        rows, cols = L.shape
        npts = (3, 6, 12, 20)[lv]            # the oracle scans the whole row
        pts = (rng.random((npts, 2)) * [cols - 1, rows - 1]).astype(f32)
        pts[0] = np.rint(pts[0])
        pts[1] = (2.3, rows / 2 + 0.3)         # a window shrunk by the left edge
        for ws in WINDOWS:
            for gl in (True, False):
                xp, er = _run(ctx, pl, pr, lv, pts, ws, gl)
                _assert_ref(xp, er, [levels[lv]], pts, ws, gl, what=(geometry, lv))
                assert (xp >= 0).any()


def _edge_points(cols, rows, h0):
    """In-image points near every edge: the last three floats below cols / rows, edge - 1, edge - h0, 0 and an interior value
    on each axis, all combinations (the corners included)."""
    def axis(e):
        v = [f32(e)]
        for _ in range(3):
            v.append(np.nextafter(v[-1], f32(0)))
        return v[1:] + [f32(e - 1), f32(e - h0), f32(0), f32(e // 2) + f32(0.25)]
    return [(x, y) for x in axis(cols) for y in axis(rows)]


@pytest.fixture(scope="module")
def edge_levels(ctx):
    """Levels of the shipped pyramids whose size the growth reaches furthest, and a 64 x 64 level."""
    out = []
    for (w, h), lv in (((752, 480), 3), ((752, 480), 2), ((640, 480), 3), ((1241, 376), 3), ((256, 256), 2)):
        lefts, rights = _pair(17 + w, w, h, shift=2)
        pl, pr = _pyramids(ctx, lefts, rights)
        out.append((pl, pr, lv, (pl.download(0, lv), pr.download(0, lv))))
    yield out
    for pl, pr, _, _ in out:
        pl.close()
        pr.close()


@gpu
def test_growth_edge(ctx, edge_levels):
    """Within one pixel of the right and bottom edges the half window grows past the exact-arithmetic bound 4 h0 - 6 (22 for
    window 15): every such point must still get the reference's column."""
    seen = set()
    for pl, pr, lv, level in edge_levels:
        rows, cols = level[0].shape
        for ws in WINDOWS:
            pts = _edge_points(cols, rows, ws // 2)
            hws = [grown_halfwin(x, y, cols, rows, ws) for x, y in pts]
            assert max(hws) <= 4 * (ws // 2) - 3
            if ws == 15:
                seen.update((cols, rows, hw) for hw in hws)
            for gl in (True, False):
                xp, er = _run(ctx, pl, pr, lv, pts, ws, gl)
                _assert_ref(xp, er, [level], pts, ws, gl, what=(cols, rows, lv))
                if gl and ws == 15:
                    grown = [i for i, hw in enumerate(hws) if hw > 22]
                    assert (xp[grown] >= 0).all(), (cols, rows, xp[grown])
    assert (94, 60, 23) in seen and (64, 64, 25) in seen and any(hw == 22 for _, _, hw in seen)


@gpu
def test_points_outside_the_right_image(ctx, edge_levels):
    """x >= cols or y >= rows: the reference's result while the grown half window is <= 25, (-1, 255) beyond."""
    pl, pr, lv, level = edge_levels[0]                  # EuRoC level 3, 94 x 60
    rows, cols = level[0].shape
    within, beyond = set(), set()
    for ws in (7, 11, 15):
        pts = [(f32(x), f32(y)) for x in (cols, cols + 0.5, cols + 2, cols + 4.75, cols + 9, 50.5)
               for y in (20.25, rows, rows + 1, rows + 3.5) if x >= cols or y >= rows]
        xp, er = _run(ctx, pl, pr, lv, pts, ws, True)
        for i, p in enumerate(pts):
            hw = grown_halfwin(*p, cols, rows, ws)
            if hw > MAX_HW:
                beyond.add(hw)
                assert (xp[i], er[i]) == (-1.0, 255.0), (ws, p, hw, xp[i], er[i])
            else:
                within.add(hw)
                _assert_ref(xp[i:i + 1], er[i:i + 1], [level], [p], ws, True, what=("outside", hw))
                assert hw <= 0 or xp[i] >= 0, (ws, p, hw)
    assert MAX_HW in within and MAX_HW + 1 in beyond and max(within) == MAX_HW, (within, beyond)


@pytest.fixture(scope="module")
def four_frames(ctx):
    lefts, rights = _pair(301, 320, 240, frames=4)
    pl, pr = _pyramids(ctx, lefts, rights)
    yield pl, pr, [[(pl.download(k, lv), pr.download(k, lv)) for k in range(4)] for lv in range(4)]
    pl.close()
    pr.close()


@gpu
def test_frame_addressing(ctx, four_frames):
    """Ragged frame indices, a fixed stride with a partial last frame and first_frame > 0, on frames that differ."""
    pl, pr, levels = four_frames
    lv = 2
    rows, cols = levels[lv][0][0].shape
    rng = np.random.default_rng(8)
    pts = (rng.random((40, 2)) * [cols - 1, rows - 1]).astype(f32)
    fidx = rng.integers(0, 4, 40).astype(np.int32)
    fidx[:4] = [3, 0, 2, 1]
    xp, er = _run(ctx, pl, pr, lv, pts, 7, True, frame_idx=fidx)
    _assert_ref(xp, er, levels[lv], pts, 7, True, frames=fidx, what="ragged")
    # the same points read from another frame give other results: a wrong frame index cannot pass
    xs, es = _run(ctx, pl, pr, lv, pts, 7, True, frame_idx=(fidx + 1) % 4)
    assert (xs != xp).any() or (es != er).any()
    for first, per, n in ((0, 11, 40), (1, 13, 30), (2, 7, 14), (3, 40, 25)):
        xp, er = _run(ctx, pl, pr, lv, pts[:n], 9, False, first_frame=first, per_frame=per)
        _assert_ref(xp, er, levels[lv], pts[:n], 9, False, frames=[first + i // per for i in range(n)], what=(first, per))


@gpu
def test_empty_slots_nan_and_no_points(ctx, four_frames):
    pl, pr, levels = four_frames
    rows, cols = levels[3][0][0].shape
    pts = np.array([[-1, -1], [-0.5, 10.0], [np.nan, 10.0], [np.nan, np.nan], [30.5, 20.25]], f32)
    xp, er = _run(ctx, pl, pr, 3, pts, 7, True, frame_idx=np.array([0, 1, 2, 3, 1], np.int32))
    assert (xp[:4] == -1).all() and (er[:4] == 255).all()
    _assert_ref(xp[4:], er[4:], levels[3], pts[4:], 7, True, frames=[1])
    assert xp[4] >= 0
    xp, er = np.full(3, 7.0, f32), np.full(3, 7.0, f32)
    api.FeatureTracker(ctx).line_min_sad(pl, pr, 3, pts, 7, True, xp, er, n=0)
    assert (xp == 7).all() and (er == 7).all()


@gpu
def test_constant_pair_keeps_the_first_column(ctx):
    img = np.full((1, 128, 256), 100, np.uint8)
    pl, pr = _pyramids(ctx, img, img)
    pts = np.array([[100.0, 60.0], [100.5, 60.25], [200.75, 33.5], [12.0, 100.0]], f32)
    for ws in (3, 7, 15):
        for gl in (True, False):
            xp, er = _run(ctx, pl, pr, 0, pts, ws, gl)
            assert np.array_equal(xp, pts[:, 0]) and (er == 0).all(), (ws, gl, xp, er)
            _assert_ref(xp, er, [(img[0], img[0])], pts, ws, gl)
    pl.close()
    pr.close()


@pytest.mark.parametrize("period", [16, 20, 32])
@gpu
def test_periodic_ties_keep_the_first_in_scan_order(ctx, period):
    """A texture periodic in x and its copy moved 5 px: exact matches (error 0) at candidates k0, k0 + period, k0 + 2 period,
    ..., in other lanes and rounds of the warp scan; the first wins."""
    h, w = 96, 320
    tile = np.random.default_rng(period).integers(0, 256, (h, period)).astype(np.uint8)
    left = np.ascontiguousarray(np.tile(tile, (1, w // period + 1))[:, :w])
    right = np.ascontiguousarray(np.roll(left, -5, axis=1))
    pl, pr = _pyramids(ctx, left[None], right[None])
    pts = np.array([[160.0, 48.0], [170.0, 20.0], [150.0, 70.0]], f32)
    for ws in (5, 9, 15):
        for gl, k0 in ((True, 5), (False, period - 5)):
            xp, er = _run(ctx, pl, pr, 0, pts, ws, gl)
            step = -1 if gl else 1
            assert np.array_equal(xp, pts[:, 0] + step * k0) and (er == 0).all(), (period, ws, gl, xp, er)
            _assert_ref(xp, er, [(left, right)], pts, ws, gl)
    pl.close()
    pr.close()


@gpu
def test_saturated_errors_give_no_column(ctx):
    """0 against 255: every candidate's error is exactly 255, which is not below the start value."""
    left, right = np.zeros((1, 64, 128), np.uint8), np.full((1, 64, 128), 255, np.uint8)
    pl, pr = _pyramids(ctx, left, right)
    pts = np.array([[60.0, 30.0], [90.5, 10.25]], f32)
    for gl in (True, False):
        xp, er = _run(ctx, pl, pr, 0, pts, 7, gl)
        assert (xp == -1).all() and (er == 255).all()
        _assert_ref(xp, er, [(left[0], right[0])], pts, 7, gl)
    pl.close()
    pr.close()


@gpu
def test_refusals_leave_the_outputs(ctx, four_frames):
    pl, pr, _ = four_frames
    deep = _pyramids(ctx, *_pair(5, 320, 240), extra=4)
    shallow = _pyramids(ctx, *_pair(5, 320, 240), extra=2)
    pts = np.array([[40.5, 30.0]] * 25, f32)
    ft = api.FeatureTracker(ctx)
    xp, er = np.full(25, 7.0, f32), np.full(25, 7.0, f32)
    cases = [("INVALID", (pl, pr, 3), dict(nwinsize=8)), ("CAPACITY", (pl, pr, 3), dict(nwinsize=17)),
             ("INVALID", (*deep, 4), {}), ("INVALID", (*shallow, 3), {}), ("INVALID", (pl, shallow[1], 3), {}),
             ("INVALID", (pl, pr, 3), dict(per_frame=5)), ("INVALID", (pl, pr, 3), dict(first_frame=1, per_frame=7)),
             ("INVALID", (pl, pr, -1), {})]
    for status, (a, b, lv), kw in cases:
        with pytest.raises(api.Ov2Error, match=status):
            ft.line_min_sad(a, b, lv, pts, kw.pop("nwinsize", 7), True, xp, er, **kw)
        assert (xp == 7).all() and (er == 7).all(), (status, lv, kw)
    for p in (*deep, *shallow):
        p.close()
