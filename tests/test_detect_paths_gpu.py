"""Grid FAST, detectSingleScale, cornerSubPix and CLAHE on every run-time path and on the reference's shipped geometries.

The host code picks kernels and load paths from the image size, the cell size and the buffer alignment; each case below
names the branch it reaches and, where the branch follows from a size formula, recomputes that formula from the same inputs
and asserts the case lands on the intended side.  Bars (against oracle/image_ref.py, its cv2 forms where cv2 imports):
integer keypoints, FAST thresholds, single-scale dmaxquality_ and CLAHE bit-exact; refined points within SUBPIX_TOL.
Oracle results are computed once per input (module-scoped cache) and shared between parametrisations.
"""
import numpy as np
import pytest

from ov2slam_b200 import api, synth
from oracle import image_ref as R

pytestmark = pytest.mark.gpu

SUBPIX_TOL = 1e-5 if R.HAVE_CV2 else 2e-4      # as tests/test_frontend_gpu.py


# ---------------------------------------------------------------------------------------------------------- inputs
def _frame(name, w, h):
    """Seeded test images by name."""
    kind, _, seed = name.partition(":")
    seed = int(seed or 0)
    if kind == "tex":
        return synth.make_frame(seed, w, h)
    if kind == "noise":
        return np.random.default_rng(seed).integers(0, 256, (h, w)).astype(np.uint8)
    if kind == "hc":                               # 0 / 255 noise: every cell has strong corners
        return np.where(np.random.default_rng(seed).random((h, w)) > 0.5, 255, 0).astype(np.uint8)
    if kind == "flat":
        return np.full((h, w), 128, np.uint8)
    if kind == "lattice":                          # 200 on 40 at x = 2 (mod 4), even y: every dot a FAST candidate
        im = np.full((h, w), 40, np.uint8)
        im[0::2, 2::4] = 200
        return im
    if kind == "halfflat":                         # texture on the left half, flat on the right
        im = synth.make_frame(seed, w, h)
        im[:, w // 2:] = 90
        return im
    if kind == "periodic":                         # period-8 block pattern: equal responses repeat inside a cell
        yy, xx = np.mgrid[0:h, 0:w]
        return np.where(((xx // 4) + (yy // 4)) % 2 == 0, 60, 180).astype(np.uint8)
    raise ValueError(name)


def _cell_cap(cs):
    """Candidates a cell can hold: one per column group {4k + 2, 4k + 3} meeting [3, cs - 3), every second interior row."""
    groups = len({x // 4 for x in range(3, cs - 3) if x % 4 in (2, 3)})
    return groups * ((cs - 6 + 1) // 2)


def _kps(seed, w, h, n, cs=None):
    """Ragged existing keypoints: random, plus points on cell boundaries, in the partial last row / column and within 0.5 px
    of the image edge."""
    rng = np.random.default_rng(seed)
    k = (rng.random((n, 2)) * [w, h]).astype(np.float32)
    extra = [[0.4, 0.4], [w - 1.0, h - 1.0], [w - 0.6, 3.0], [2.0, h - 0.6], [100.5, 200.5]]
    if cs:
        extra += [[cs * 2.0, cs * 1.0], [cs * 3.0 - 1e-3, 10.0], [(w // cs) * cs + 0.5, 20.0], [30.0, (h // cs) * cs + 0.5]]
    return np.concatenate([k, np.array(extra, np.float32)]).astype(np.float32)


class _Oracle:
    """Memoised oracle calls keyed by the input's name and size (the images are regenerated from them)."""

    def __init__(self):
        self.memo = {}

    def _get(self, key, fn):
        if key not in self.memo:
            self.memo[key] = fn()
        return self.memo[key]

    def image(self, name, w, h):
        return self._get(("img", name, w, h), lambda: _frame(name, w, h))

    def clahe(self, name, w, h, clip=3.0, tiles=None):
        im = self.image(name, w, h)
        f = R.clahe_cv2 if R.HAVE_CV2 else R.clahe_ref
        return self._get(("clahe", name, w, h, clip, tiles), lambda: f(im, clip, tiles))

    def fast(self, im_key, im, cs, kps_key, kps, th):
        return self._get(("fast", im_key, im.shape, cs, kps_key, th),
                         lambda: R.detect_grid_fast_nosubpix(im, cs, kps, th, use_cv2=R.HAVE_CV2)[:2])

    def sscale(self, im_key, im, cs, kps_key, kps, roi, q):
        return self._get(("ss", im_key, im.shape, cs, kps_key, tuple(roi), q),
                         lambda: R.detect_single_scale_nosubpix(im, cs, kps, roi, q, use_cv2=R.HAVE_CV2)[:2])

    def subpix(self, im_key, im, ipts):
        f = R.corner_subpix_cv2 if R.HAVE_CV2 else R.corner_subpix_ref
        return self._get(("sp", im_key, im.shape, ipts.tobytes()), lambda: f(im, ipts.astype(np.float32)))


@pytest.fixture(scope="module")
def oracle():
    return _Oracle()


# ---------------------------------------------------------------------------------------------------------- formulas
def _fast_sweep_smem(w, h, cs, nw):
    """Shared memory of fast_sweep_kernel at nw warps (grid_sweep.cuh SweepSmem, frontend_fast.cu fast_sweep_smem): the
    bitmap, min(cap, 128) sort keys per warp, row progress counters when nw > 1, occupancy.  Vectorised over w and h."""
    nwc, nhc = w // cs, h // cs
    wpr = (w + 31) // 32
    return (h * wpr * 4 + nw * min(_cell_cap(cs), 128) * 4 + np.where(nw > 1, nhc * 4, 0) + (nhc + 1) * (nwc + 1) + 15) & ~15


def _fast_sweep_warps(w, h, cs):
    """Warps ov2_grid_fast gives fast_sweep_kernel: the most, up to one per cell row and 16, whose shared memory fits 227 KB;
    0: refused with OV2_ERR_CAPACITY.  Vectorised over w and h (at least one cell row)."""
    nhc = np.asarray(h) // cs
    nw = np.zeros(np.broadcast(np.asarray(w), nhc).shape, np.int64)
    for k in range(1, 17):          # the layout grows with the warp count
        nw = np.where((k <= nhc) & (_fast_sweep_smem(w, h, cs, k) <= 227 * 1024), k, nw)
    return int(nw) if nw.ndim == 0 else nw


def _sscale_fits(w, h, cs):
    nwc, nhc = w // cs, h // cs
    wpr = (w + 31) // 32
    smem = (((h * wpr + 1) & ~1) * 4 + nwc * nhc * 16 + (nhc * 4 if nhc > 1 else 0) + (nhc + 1) * (nwc + 1) + 15) & ~15
    return smem <= 227 * 1024


def _fast_tma(pitch, fstride, base):
    """launch_fast_cells stages cells with TMA only for 16-byte aligned bases, pitches and frame strides."""
    return base % 16 == 0 and pitch % 16 == 0 and fstride % 16 == 0


def _clahe_word_tiles(w, h, tx, ty, pitch, base):
    """Tiles clahe_lut_kernel counts with 32-bit word loads (the rest take the byte path)."""
    ew, eh = (w, h) if (w % tx == 0 and h % ty == 0) else (w + tx - w % tx, h + ty - h % ty)
    tw, th = ew // tx, eh // ty
    n = 0
    for j in range(ty):
        for i in range(tx):
            x0, y0 = i * tw, j * th
            n += x0 + tw <= w and y0 + th <= h and tw % 4 == 0 and x0 % 4 == 0 and pitch % 4 == 0 and base % 4 == 0
    return n, tx * ty


# ---------------------------------------------------------------------------------------------------------- runners
def _offsets(kps_list):
    off = np.concatenate([[0], np.cumsum([len(k) for k in kps_list])]).astype(np.int32)
    allk = np.concatenate(kps_list).astype(np.float32) if off[-1] else None
    return off, allk


def _grid_fast(ctx, pyr, cs, first, count, ths, kps_list=None, do_subpix=True):
    ncell = (pyr.h // cs) * (pyr.w // cs)
    pts = np.empty((count, ncell, 2), np.float32)
    ipts = np.empty((count, ncell, 2), np.int32)
    cnt = np.zeros(count, np.int32)
    off, allk = _offsets(kps_list) if kps_list is not None else (None, None)
    api.FeatureExtractor(ctx).detect_grid_fast(pyr, cs, first, count, ths, pts, cnt, off, allk, ipts, do_subpix=do_subpix)
    return pts, ipts, cnt


def _check_fast(oracle, names, imgs, cs, kps_list, th_in, out, th_out, tag=""):
    pts, ipts, cnt = out
    for f, im in enumerate(imgs):
        kk = kps_list[f] if kps_list is not None else np.zeros((0, 2), np.float32)
        ref_i, ref_th = oracle.fast(names[f], im, cs, (tag, f, len(kk)), kk, int(th_in[f]))
        assert cnt[f] == len(ref_i), (names[f], cs, f, cnt[f], len(ref_i))
        assert np.array_equal(ipts[f, :cnt[f]], ref_i), (names[f], cs, f)
        assert th_out[f] == ref_th, (names[f], cs, f, th_out[f], ref_th)
        assert (pts[f, cnt[f]:] == -1).all()
        if cnt[f]:
            d = np.abs(pts[f, :cnt[f]] - oracle.subpix(names[f], im, ref_i))
            assert d.max() <= SUBPIX_TOL, (names[f], cs, f, d.max())


def _sscale(ctx, pyr, cs, first, count, q, kps_list=None, roi=None, do_subpix=True):
    ncell = (pyr.h // cs) * (pyr.w // cs)
    pts = np.empty((count, ncell, 2), np.float32)
    ipts = np.empty((count, ncell, 2), np.int32)
    cnt = np.zeros(count, np.int32)
    off, allk = _offsets(kps_list) if kps_list is not None else (None, None)
    api.FeatureExtractor(ctx).detect_single_scale(pyr, cs, first, count, q, pts, cnt, off, allk, roi, ipts, do_subpix=do_subpix)
    return pts, ipts, cnt


def _check_sscale(oracle, names, imgs, cs, kps_list, roi, q_in, out, q_out, tag=""):
    pts, ipts, cnt = out
    h, w = imgs[0].shape
    r = roi if roi is not None else (0, 0, w, h)
    for f, im in enumerate(imgs):
        kk = kps_list[f] if kps_list is not None else np.zeros((0, 2), np.float32)
        ref_i, ref_q = oracle.sscale(names[f], im, cs, (tag, f, len(kk)), kk, r, float(q_in[f]))
        assert cnt[f] == len(ref_i), (names[f], cs, f, cnt[f], len(ref_i))
        assert np.array_equal(ipts[f, :cnt[f]], ref_i), (names[f], cs, f)
        assert q_out[f] == ref_q, (names[f], cs, f, q_out[f], ref_q)
        assert (pts[f, cnt[f]:] == -1).all()
        if cnt[f]:
            d = np.abs(pts[f, :cnt[f]] - oracle.subpix(names[f], im, ref_i))
            assert d.max() <= SUBPIX_TOL, (names[f], cs, f, d.max())


def _pyr(ctx, imgs, device=False, nlev=0):
    n, h, w = imgs.shape
    p = api.Pyramid(ctx, n, w, h, nlev)
    if device:
        torch = pytest.importorskip("torch")
        p.build(torch.from_numpy(imgs).cuda())
        ctx.sync()
    else:
        p.build(imgs)
    return p


# ---------------------------------------------------------------------------------------------------------- shipped geometries
SHIPPED = [(752, 480), (1241, 376), (640, 480)]


@pytest.mark.parametrize("src", ["host", "device"])
@pytest.mark.parametrize("chain", ["accurate", "average", "fast"])
@pytest.mark.parametrize("w,h", SHIPPED)
def test_shipped_configurations(ctx, oracle, w, h, chain, src):
    """The reference's parameter files on EuRoC 752x480, KITTI 1241x376 and TartanAir 640x480 frames:
    accurate/ = CLAHE (tiles W/50 x H/50) then detectSingleScale at cell 35; average/ = detectSingleScale at cell 45 on the raw
    image; fast/ = grid FAST at cell 50.  Three frames per call with per-frame state, with and without existing keypoints,
    from host buffers and from device-aliased frames.  At 1241 wide the aliased frames' pitch is not 16-byte aligned, so
    grid FAST stages its cells with plain loads instead of TMA, and host-buffer CLAHE takes the byte paths."""
    names = [f"tex:{300 + i}" for i in range(3)]
    raw = np.stack([oracle.image(n, w, h) for n in names])
    if chain == "accurate":
        eq = np.empty_like(raw)
        if src == "host":
            api.clahe(ctx, raw, eq, w, h, count=3)
            if w == 1241:
                assert _clahe_word_tiles(w, h, w // 50, h // 50, w, 0)[0] == 0
        else:
            torch = pytest.importorskip("torch")
            d_out = torch.empty((3, h, w), dtype=torch.uint8, device="cuda")
            api.clahe(ctx, torch.from_numpy(raw).cuda(), d_out, w, h, count=3)
            ctx.sync()
            eq = d_out.cpu().numpy()
        for f in range(3):
            assert np.array_equal(eq[f], oracle.clahe(names[f], w, h)), (f, int((eq[f] != oracle.clahe(names[f], w, h)).sum()))
        imgs, inames = eq, [n + "/clahe" for n in names]
    else:
        imgs, inames = raw, names
    if src == "device":
        assert _fast_tma(w, w * h, 0) == (w % 16 == 0)
    pyr = _pyr(ctx, imgs, device=src == "device")
    for with_kps in (False, True):
        cs = {"accurate": 35, "average": 45, "fast": 50}[chain]
        kl = [_kps(7 + f, w, h, [0, 40, 90][f], cs) for f in range(3)] if with_kps else None
        if chain == "fast":
            th = np.array([10, 6, 20], np.int32)
            th_in = th.copy()
            out = _grid_fast(ctx, pyr, cs, 0, 3, th, kl)
            _check_fast(oracle, inames, imgs, cs, kl, th_in, out, th, tag=("ship", with_kps))
        else:
            q = np.array([0.001, 0.0001, 0.05], np.float64)
            q_in = q.copy()
            out = _sscale(ctx, pyr, cs, 0, 3, q, kl)
            _check_sscale(oracle, inames, imgs, cs, kl, None, q_in, out, q, tag=("ship", with_kps))
        assert out[2].sum() > 0
    pyr.close()


# ---------------------------------------------------------------------------------------------------------- grid FAST sweeps
@pytest.mark.parametrize("w,h,cs,nw", [(1280, 720, 8, 16), (1600, 1000, 50, 16), (1600, 1150, 50, 3), (1600, 1153, 50, 1)])
def test_grid_fast_sweep_warps_from_budget(ctx, oracle, w, h, cs, nw):
    """fast_sweep_kernel takes as many warps as its shared memory allows: 16 at 1280x720 cell 8 (14 400 cells) and at
    1600x1000 cell 50; 3 at 1600x1150 cell 50, where the bitmap leaves room for few sort-key areas; 1 at 1600x1153 cell 50,
    which sweeps the rows in order without progress counters."""
    assert _fast_sweep_warps(w, h, cs) == nw
    names = [f"tex:{60 + cs}"]
    imgs = np.stack([oracle.image(n, w, h) for n in names])
    pyr = _pyr(ctx, imgs)
    kl = [_kps(cs, w, h, 50, cs)]
    th = np.array([10], np.int32)
    out = _grid_fast(ctx, pyr, cs, 0, 1, th, kl)
    _check_fast(oracle, names, imgs, cs, kl, [10], out, th, tag="budget")
    assert out[2][0] > 0
    pyr.close()


def test_grid_fast_capacity_refusal_then_recovers(ctx, oracle):
    """1920x1080: the mask bitmap alone is over 227 KB, so ov2_grid_fast refuses with OV2_ERR_CAPACITY (decided on the host,
    before anything is enqueued); the same context then runs a normal call correctly."""
    assert _fast_sweep_warps(1920, 1080, 50) == 0
    big = api.Pyramid(ctx, 1, 1920, 1080, 0)
    big.build(synth.make_frame(3, 1920, 1080)[None])
    th = np.array([10], np.int32)
    with pytest.raises(api.Ov2Error, match="CAPACITY"):
        _grid_fast(ctx, big, 50, 0, 1, th)
    assert th[0] == 10
    big.close()
    names = ["tex:41"]
    imgs = np.stack([oracle.image(n, 640, 480) for n in names])
    pyr = _pyr(ctx, imgs)
    th = np.array([10], np.int32)
    out = _grid_fast(ctx, pyr, 50, 0, 1, th)
    _check_fast(oracle, names, imgs, 50, None, [10], out, th)
    pyr.close()


# ---------------------------------------------------------------------------------------------------------- grid FAST paths
@pytest.mark.parametrize("cs", [8, 16, 45, 64, 65, 96, 128])
def test_grid_fast_cell_sizes(ctx, oracle, cs):
    """Cell sizes end to end: the 32-thread cell CTA (8, 16), both pair-row layouts of fast_cells_kernel (<= 64 and
    65..128), more than 32 cell rows (cell 8: 60 rows, so each wave warp owns 3 or 4 of them) and one to a few cell rows
    (128); host frames with ragged keypoints and device-aliased frames without."""
    w, h = 640, 480
    names = [f"tex:{500 + i}" for i in range(2)]
    imgs = np.stack([oracle.image(n, w, h) for n in names])
    kl = [_kps(cs + 100 + f, w, h, [20, 3][f], cs) for f in range(2)]
    for device in (False, True):
        pyr = _pyr(ctx, imgs, device=device)
        th = np.array([10, 3], np.int32)
        k = None if device else kl
        out = _grid_fast(ctx, pyr, cs, 0, 2, th, k)
        _check_fast(oracle, names, imgs, cs, k, [10, 3], out, th, tag="sizes")
        assert out[2].sum() > 0
        pyr.close()
    if cs == 8:
        assert h // cs > 32


def test_grid_fast_first_frame_offset(ctx, oracle):
    """first > 0 with count < batch: frames 1 and 2 of a 4-frame pyramid; the outputs are the answers for those frames."""
    w, h = 752, 480
    names = [f"tex:{600 + i}" for i in range(4)]
    imgs = np.stack([oracle.image(n, w, h) for n in names])
    pyr = _pyr(ctx, imgs)
    kl = [_kps(61, w, h, 25, 50), _kps(62, w, h, 0, 50)]
    th = np.array([10, 15], np.int32)
    out = _grid_fast(ctx, pyr, 50, 1, 2, th, kl)
    _check_fast(oracle, names[1:3], imgs[1:3], 50, kl, [10, 15], out, th, tag="first")
    pyr.close()


def test_grid_fast_threshold_branches(ctx, oracle):
    """nfast_th_ adaptation (feature_extractor.cpp:546-552): a textureless frame detects nothing (x 0.66: 10 -> 6); a 0/255
    noise frame detects in every empty cell (x 1.5: 10 -> 15); a frame textured on its left half only detects in 62 of
    108 cells and keeps the threshold."""
    w, h = 640, 480
    names = ["flat", "hc:5", "halfflat:9"]
    imgs = np.stack([oracle.image(n, w, h) for n in names])
    pyr = _pyr(ctx, imgs)
    th = np.array([10, 10, 10], np.int32)
    out = _grid_fast(ctx, pyr, 50, 0, 3, th)
    _check_fast(oracle, names, imgs, 50, None, [10, 10, 10], out, th)
    assert list(th) == [6, 15, 10]
    assert out[2][0] == 0 and out[2][1] == (h // 50) * (w // 50)
    pyr.close()


def _tie_cells(im, cs, th):
    st = []
    R.detect_grid_fast_nosubpix(im, cs, np.zeros((0, 2)), th, use_cv2=R.HAVE_CV2, stats=st)
    return sum(1 for _, n, m in st if n > 16 and m > 1)


def test_grid_fast_tie_sort(ctx, oracle):
    """Cells where more than 16 candidates survive the mask and the top response is tied: the winner is the one the
    libstdc++ std::sort emulation (stdsort_emul.h) puts first.  The dot lattice (every candidate has the same response)
    has 54 such cells at cell 50; uniform noise frames (seeds 0 and 1) have 9 between them at threshold 10.  The test
    asserts at least 50 and 8."""
    w, h = 640, 480
    names = ["lattice", "noise:0", "noise:1"]
    imgs = np.stack([oracle.image(n, w, h) for n in names])
    ties = oracle._get(("ties",), lambda: [_tie_cells(im, 50, 10) for im in imgs])
    assert ties[0] >= 50 and ties[1] + ties[2] >= 8, ties
    pyr = _pyr(ctx, imgs)
    th = np.array([10, 10, 10], np.int32)
    out = _grid_fast(ctx, pyr, 50, 0, 3, th)
    _check_fast(oracle, names, imgs, 50, None, [10, 10, 10], out, th)
    pyr.close()


# ---------------------------------------------------------------------------------------------------------- capacity
CAPACITY_CASES = [("lattice", 45, 10), ("lattice", 50, 10), ("noise:0", 50, 0), ("noise:0", 64, 0), ("noise:0", 128, 0)]


def _max_candidates(im, cs, th):
    h, w = im.shape
    return max(len([k for k in R.fast_detect_ref(im[y:y + cs, x:x + cs], th) if k[0] % 4 in (2, 3)])
               for y in range(0, h - cs - 1, cs) for x in range(0, w - cs - 1, cs))


@pytest.mark.parametrize("name,cs,th0", CAPACITY_CASES)
def test_grid_fast_dense_cells(ctx, oracle, name, cs, th0):
    """Cells with up to the full candidate capacity (the lattice reaches the bound exactly at cell 45: 200; noise at
    threshold 0 reaches 128 at cell 50, 213 at 64 and 820 at 128): every candidate is kept (no OV2_ERR_CAPACITY) and the
    result equals the oracle, through ov2_grid_fast and through batch mode.  Above 128 candidates the sweep reads the
    cell's list from global memory and sorts in its global key area."""
    w, h = 640, 480
    im = oracle.image(name, w, h)
    mc = oracle._get(("maxcand", name, cs, th0), lambda: _max_candidates(im, cs, th0))
    assert mc <= _cell_cap(cs) and mc >= {45: 200, 50: 128, 64: 200, 128: 800}[cs], mc
    imgs = im[None]
    pyr = _pyr(ctx, imgs)
    th = np.array([th0], np.int32)
    out = _grid_fast(ctx, pyr, cs, 0, 1, th)
    _check_fast(oracle, [name], imgs, cs, None, [th0], out, th)
    ncell = (h // cs) * (w // cs)
    bth = np.array([th0], np.int32)
    bout = (np.empty((1, ncell, 2), np.float32), np.empty((1, ncell, 2), np.int32), np.zeros(1, np.int32))
    ctx.batch_begin()
    api.FeatureExtractor(ctx).detect_grid_fast(pyr, cs, 0, 1, bth, bout[0], bout[2], out_pts_int=bout[1])
    ctx.batch_end()
    for a, b in zip(out, bout):
        assert np.array_equal(a, b)
    assert bth[0] == th[0]
    assert api.FeatureExtractor(ctx).fast_cell_capacity(cs) == _cell_cap(cs)
    pyr.close()


def test_frontend_step_dense_cells(ctx, oracle):
    """ov2_frontend_step at cell 50 on current frames with dense cells (the lattice, noise at threshold 0 through the
    threshold state) equals the operator entry points called one by one, and its detections equal the oracle."""
    w, h, nfr, nk = 640, 480, 2, 128
    curs = np.stack([oracle.image("lattice", w, h), oracle.image("noise:0", w, h)])
    prevs = np.stack([synth.make_frame(95 + f, w, h) for f in range(nfr)])
    rng = np.random.default_rng(4)
    kps = np.stack([rng.uniform(12, w - 12, nfr * nk), rng.uniform(12, h - 12, nfr * nk)], axis=1).astype(np.float32)
    lv = np.full(nfr * nk, 3, np.uint8)
    ncell = (h // 50) * (w // 50)
    th0 = np.array([10, 0], np.int32)

    def outputs():
        return dict(pri=kps.copy(), st=np.zeros(nfr * nk, np.uint8), th=th0.copy(),
                    new=np.empty((nfr * ncell, 2), np.float32), cnt=np.zeros(nfr, np.int32),
                    dt=np.zeros((nfr * nk, 32), np.uint8), vt=np.zeros(nfr * nk, np.uint8),
                    dn=np.zeros((nfr * ncell, 32), np.uint8), vn=np.zeros(nfr * ncell, np.uint8))

    pp = api.Pyramid(ctx, nfr, w, h, 3)
    cp = api.Pyramid(ctx, nfr, w, h, 3)
    a = outputs()
    pp.build(prevs)
    cp.build(curs)
    ft, fe = api.FeatureTracker(ctx, 30, 0.01), api.FeatureExtractor(ctx)
    ft.fb_klt_tracking(pp, cp, 9, lv, 30.0, 0.5, kps, a["pri"], a["st"], per_frame=nk)
    ipts = np.empty((nfr, ncell, 2), np.int32)
    fe.detect_grid_fast(cp, 50, 0, nfr, a["th"], a["new"], a["cnt"], out_pts_int=ipts, max_per_frame=ncell)
    fe.describe_brief(cp, a["pri"], a["dt"], a["vt"], per_frame=nk)
    fe.describe_brief(cp, a["new"], a["dn"], a["vn"], per_frame=ncell)
    _check_fast(oracle, ["lattice", "noise:0"], curs, 50, None, th0, (a["new"].reshape(nfr, ncell, 2), ipts, a["cnt"]), a["th"])
    b = outputs()
    args = api.FrontendStepArgs(prevs.ctypes.data, curs.ctypes.data, w, w * h, nfr, api.KltParams(9, 30, float(np.float32(0.01)), 30.0, 0.5),
                                nfr * nk, nk, None, 3, kps.ctypes.data, b["pri"].ctypes.data, b["st"].ctypes.data, 50,
                                b["th"].ctypes.data, ncell, b["new"].ctypes.data, b["cnt"].ctypes.data, b["dt"].ctypes.data,
                                b["vt"].ctypes.data, b["dn"].ctypes.data, b["vn"].ctypes.data)
    for rep in range(3):           # eager, graph capture, replay
        b["pri"][...] = kps
        b["th"][...] = th0
        api.frontend_step(ctx, pp, cp, args)
        for k in a:
            assert np.array_equal(a[k], b[k]), (rep, k)
    pp.close()
    cp.close()


# ---------------------------------------------------------------------------------------------------------- single scale
@pytest.mark.parametrize("cs", [8, 16, 32, 33, 35, 36, 45, 50, 64])
def test_single_scale_cell_sizes(ctx, oracle, cs):
    """ss_sweep_kernel's arg-max: held in registers for cs <= 35 (the lane stride over the cell is one row plus 32 - cs
    pixels for cs < 32, exactly a row at 32, under a row above) and cell_argmax_warp for cs >= 36; cell 8 and 16 give more
    than 32 cell rows at 480 px (60 and 30 rows: 8 only), so wave warps own several rows.  Two frames, ragged keypoints."""
    w, h = 640, 480
    names = [f"tex:{700 + i}" for i in range(2)]
    imgs = np.stack([oracle.image(n, w, h) for n in names])
    pyr = _pyr(ctx, imgs)
    kl = [_kps(cs + 200 + f, w, h, [15, 0][f], cs) for f in range(2)]
    q = np.array([0.001, 0.0005], np.float64)
    q_in = q.copy()
    out = _sscale(ctx, pyr, cs, 0, 2, q, kl)
    _check_sscale(oracle, names, imgs, cs, kl, None, q_in, out, q, tag="sizes")
    assert out[2].sum() > 0
    assert (cs * cs <= 40 * 32) == (cs <= 35)
    pyr.close()


def test_single_scale_ties_flat_cells_and_masked_maxima(ctx, oracle):
    """A periodic block texture whose responses tie inside each cell (the first maximum in row-major order wins), a frame
    half flat (cells whose maximum is 0 skip the cell-maximum shortcut and rescan) and keypoints placed so their discs cover
    the maximum of the next cell to the right (the shortcut is refused and the cell is rescanned)."""
    w, h, cs = 640, 480, 35
    names = ["periodic", "halfflat:9", "tex:710"]
    imgs = np.stack([oracle.image(n, w, h) for n in names])
    pyr = _pyr(ctx, imgs)
    free, _ = oracle.sscale(names[2], imgs[2], cs, "none", np.zeros((0, 2), np.float32), (0, 0, w, h), 0.001)
    r = cs // 4
    mk = []
    for px, py in free:
        c = px // cs
        if c >= 1 and px - (c * cs - 1) <= r and len(mk) < 30:
            mk.append([c * cs - 1.0, float(py)])          # in the left neighbour: its disc covers (px, py)
    assert len(mk) >= 5, len(mk)
    kl = [np.zeros((0, 2), np.float32), np.zeros((0, 2), np.float32), np.array(mk, np.float32)]
    q = np.array([0.001, 0.001, 0.001], np.float64)
    q_in = q.copy()
    out = _sscale(ctx, pyr, cs, 0, 3, q, kl)
    _check_sscale(oracle, names, imgs, cs, kl, None, q_in, out, q, tag="ties")
    pyr.close()


def test_single_scale_roi_quality_and_first(ctx, oracle):
    """roi forms (an offset roi; a small roi that rejects the first detection of most cells, which then get no second one
    either; a zero-area roi), the three dmaxquality_ branches (x 1.5 when more than 90 % of the free cells detect, / 2 below
    33 %, unchanged between) and first > 0 with count < batch."""
    w, h, cs = 752, 480, 45
    names = [f"tex:{720 + i}" for i in range(4)]
    imgs = np.stack([oracle.image(n, w, h) for n in names])
    pyr = _pyr(ctx, imgs)
    for roi in ((20, 24, w - 45, h - 50), (100, 90, 300, 200), (0, 0, 0, 0)):
        q = np.array([0.0001, 0.05], np.float64)
        q_in = q.copy()
        out = _sscale(ctx, pyr, cs, 1, 2, q, None, roi)
        _check_sscale(oracle, names[1:3], imgs[1:3], cs, None, roi, q_in, out, q, tag="roi")
        if roi[2] == 0:
            assert out[2].sum() == 0 and list(q) == [q_in[0] / 2, q_in[1] / 2]
    branches = set()
    for q0 in (0.0001, 0.01, 1e9):
        q = np.array([q0], np.float64)
        out = _sscale(ctx, pyr, cs, 3, 1, q)
        _check_sscale(oracle, names[3:], imgs[3:], cs, None, None, [q0], out, q, tag="q")
        branches.add(round(q[0] / q0, 6))
    assert branches == {0.5, 1.0, 1.5}, branches
    pyr.close()


def test_single_scale_capacity_refusal_then_recovers(ctx, oracle):
    """1280x720 at cell 8: two detections per cell for 14 400 cells plus the bitmap are over 227 KB of shared memory, so
    ov2_detect_single_scale refuses with OV2_ERR_CAPACITY; the same context then runs a normal call correctly."""
    assert not _sscale_fits(1280, 720, 8) and _sscale_fits(1280, 720, 16)
    big = api.Pyramid(ctx, 1, 1280, 720, 0)
    big.build(synth.make_frame(4, 1280, 720)[None])
    q = np.array([0.001], np.float64)
    with pytest.raises(api.Ov2Error, match="CAPACITY"):
        _sscale(ctx, big, 8, 0, 1, q)
    big.close()
    names = ["tex:701"]
    imgs = np.stack([oracle.image(n, 640, 480) for n in names])
    pyr = _pyr(ctx, imgs)
    q = np.array([0.001], np.float64)
    out = _sscale(ctx, pyr, 35, 0, 1, q)
    _check_sscale(oracle, names, imgs, 35, None, None, [0.001], out, q)
    pyr.close()


# ---------------------------------------------------------------------------------------------------------- cornerSubPix
def test_subpix_at_every_border(ctx, oracle):
    """Detections within 4 px of each border and in each corner region: getRectSubPix's replicated-border path of
    rect_subpix_px.  642x482 at cell 32 lets detectSingleScale's last cells reach 3 px from the right and bottom edges;
    the frame has bright squares whose corners sit there.  do_subpix = 0 returns the integer points."""
    w, h, cs = 642, 482, 32
    im = synth.make_frame(811, w, h) // 4
    for x, y in ((1, 1), (w - 4, 1), (1, h - 4), (w - 4, h - 4), (1, 200), (w - 4, 300), (300, 1), (400, h - 4), (30, 2), (2, 40)):
        im[y:y + 3, x:x + 3] = 250
    name = "borders"
    oracle.memo[("img", name, w, h)] = im
    pyr = _pyr(ctx, im[None])
    q = np.array([0.0001], np.float64)
    out = _sscale(ctx, pyr, cs, 0, 1, q)
    _check_sscale(oracle, [name], im[None], cs, None, None, [0.0001], out, q)
    ip = out[1][0, :out[2][0]]
    near = dict(left=ip[:, 0] < 4, right=ip[:, 0] >= w - 4, top=ip[:, 1] < 4, bottom=ip[:, 1] >= h - 4)
    assert all(v.any() for v in near.values()), {k: int(v.sum()) for k, v in near.items()}
    corners = ((ip[:, 0] < 8) | (ip[:, 0] >= w - 8)) & ((ip[:, 1] < 8) | (ip[:, 1] >= h - 8))
    assert corners.sum() >= 2
    q = np.array([0.0001], np.float64)
    raw = _sscale(ctx, pyr, cs, 0, 1, q, do_subpix=False)
    assert np.array_equal(raw[1], out[1]) and np.array_equal(raw[0][0, :out[2][0]], ip.astype(np.float32))
    th = np.array([10], np.int32)
    graw = _grid_fast(ctx, pyr, 16, 0, 1, th, do_subpix=False)
    assert np.array_equal(graw[0][0, :graw[2][0]], graw[1][0, :graw[2][0]].astype(np.float32))
    pyr.close()


# ---------------------------------------------------------------------------------------------------------- CLAHE
def _clahe_ref(im, clip, tiles):
    return (R.clahe_cv2 if R.HAVE_CV2 else R.clahe_ref)(im, clip, tiles)


CLAHE_SIZES = [(1241, 376), (800, 600), (1000, 500), (1000, 480), (333, 245), (50, 50)]


@pytest.mark.parametrize("w,h", CLAHE_SIZES)
def test_clahe_sizes_clips_and_content(ctx, oracle, w, h):
    """cv::CLAHE at sizes with and without OpenCV's reflected extension (800x600 and 1000x500 divide by the default grid;
    1000x480 divides in W only, and OpenCV then extends both), odd sizes and a single tile (50x50); clip limits 3, 0 (no
    clipping), 0.01 (clip = 1, a large residual) and 40; constant, two-level, noise and textured images.  Host buffers
    (word LUT path where the tile rows are 4-byte addressable) and the same images as device tensors."""
    tiles = (max(w // 50, 1), max(h // 50, 1))
    yy, xx = np.mgrid[0:h, 0:w]
    imgs = np.stack([np.full((h, w), 77, np.uint8), np.where(xx < w // 3, 30, 220).astype(np.uint8),
                     np.random.default_rng(w).integers(0, 256, (h, w)).astype(np.uint8), synth.make_frame(w + h, w, h)])
    extended = w % tiles[0] != 0 or h % tiles[1] != 0
    assert extended == ((w, h) not in ((800, 600), (1000, 500), (50, 50)))
    if w == 1241:
        assert _clahe_word_tiles(w, h, *tiles, w, 0)[0] == 0          # odd pitch: byte path everywhere
    torch = pytest.importorskip("torch")
    d_in = torch.from_numpy(imgs).cuda()
    for clip in (3.0, 0.0, 0.01, 40.0):
        out = np.empty_like(imgs)
        api.clahe(ctx, imgs, out, w, h, count=len(imgs), clip_limit=clip, tiles=tiles)
        d_out = torch.empty_like(d_in)
        api.clahe(ctx, d_in, d_out, w, h, count=len(imgs), clip_limit=clip, tiles=tiles)
        ctx.sync()
        for f in range(len(imgs)):
            ref = _clahe_ref(imgs[f], clip, tiles)
            assert np.array_equal(out[f], ref), (clip, f, int((out[f] != ref).sum()))
        assert np.array_equal(d_out.cpu().numpy(), out), clip


@pytest.mark.parametrize("tiles", [(8, 8), (1, 1), (64, 2), (10, 8), (65, 2)])
def test_clahe_explicit_grids(ctx, tiles):
    """Explicit tile grids: 1 to 64 tile columns are built (clahe_apply_kernel stages two LUT rows of up to 64 tiles);
    65 columns return OV2_ERR_CAPACITY.  (10, 8) gives 100 x 60 tiles without extension, so every tile histogram takes the
    32-bit word path; (8, 8) (125-pixel tiles) takes the byte path."""
    w, h = 1000, 480
    im = synth.make_frame(17, w, h)
    out = np.empty_like(im)
    if tiles[0] > 64:
        with pytest.raises(api.Ov2Error, match="CAPACITY"):
            api.clahe(ctx, im[None], out[None], w, h, tiles=tiles)
        return
    words, total = _clahe_word_tiles(w, h, *tiles, w, 0)
    if tiles == (10, 8):
        assert words == total
    if tiles == (8, 8):
        assert words == 0
    api.clahe(ctx, im[None], out[None], w, h, tiles=tiles)
    assert np.array_equal(out, _clahe_ref(im, 3.0, tiles))


def test_clahe_strides_alignment_and_in_place(ctx):
    """Odd row strides wider than the image and padded frame strides (byte paths of both kernels), a device view one byte
    past an aligned base, count > 1, and in place (src is dst) for host and device buffers, as the reference calls
    apply(img, img).  The bytes between a strided image's rows and frames (other pixels of a ROI's parent) come back
    unchanged in a host destination."""
    torch = pytest.importorskip("torch")
    w, h, n = 333, 245, 3
    imgs = np.stack([synth.make_frame(900 + i, w, h) for i in range(n)])
    refs = [_clahe_ref(im, 3.0, (w // 50, h // 50)) for im in imgs]
    rs, fs = w + 6, (w + 6) * h + 5                 # odd row stride, padded frame stride
    assert rs % 2 == 1 and _clahe_word_tiles(w, h, w // 50, h // 50, rs, 0)[0] == 0
    buf = np.full(fs * n, 3, np.uint8)
    for f in range(n):
        buf[f * fs:f * fs + rs * h].reshape(h, rs)[:, :w] = imgs[f]
    dst = np.zeros_like(buf)
    api.clahe(ctx, buf, dst, w, h, count=n, row_stride=rs, frame_stride=fs)
    for f in range(n):
        assert np.array_equal(dst[f * fs:f * fs + rs * h].reshape(h, rs)[:, :w], refs[f]), f
        assert (dst[f * fs:f * fs + rs * h].reshape(h, rs)[:, w:] == 0).all(), f     # a ROI's neighbours are not written
    inplace = buf.copy()
    api.clahe(ctx, inplace, inplace, w, h, count=n, row_stride=rs, frame_stride=fs)
    for f in range(n):
        blk = inplace[f * fs:f * fs + rs * h].reshape(h, rs)
        assert np.array_equal(blk[:, :w], refs[f]), f
        assert (blk[:, w:] == 3).all()                   # bytes between rows untouched
    # device: a view one byte past a 256-byte aligned allocation
    d = torch.from_numpy(np.concatenate([np.zeros(1, np.uint8), buf])).cuda()
    view = d[1:]
    assert view.data_ptr() % 4 == 1
    d_out = torch.zeros_like(view)
    api.clahe(ctx, view, d_out, w, h, count=n, row_stride=rs, frame_stride=fs)
    ctx.sync()
    assert np.array_equal(d_out.cpu().numpy(), dst)
    api.clahe(ctx, view, view, w, h, count=n, row_stride=rs, frame_stride=fs)
    ctx.sync()
    got = view.cpu().numpy()
    for f in range(n):
        assert np.array_equal(got[f * fs:f * fs + rs * h].reshape(h, rs)[:, :w], refs[f]), f


def test_preprocess_without_clahe_and_first(ctx):
    """ov2_preprocess with use_clahe = 0 (level 0 of the output is the raw level 0, the levels are exact pyrDown images of
    it) and with CLAHE on frames [1, 3) of a 3-frame batch (frame 0 of the output is left alone).  An output pyramid
    stays in the mode of its first call (aliasing the raw level 0, or owning an equalised one)."""
    w, h = 752, 480
    imgs = np.stack([synth.make_frame(950 + i, w, h) for i in range(3)])
    raw = api.Pyramid(ctx, 3, w, h, 0)
    raw.build(imgs)
    out = api.Pyramid(ctx, 3, w, h, 3)
    api.preprocess(ctx, raw, out, 0, 3, use_clahe=False)
    for f in range(3):
        ref = R.build_pyramid_ref(imgs[f], 3)
        for lvl in range(4):
            assert np.array_equal(out.download(f, lvl), ref[lvl]), (f, lvl)
    out2 = api.Pyramid(ctx, 3, w, h, 3)
    api.preprocess(ctx, raw, out2, 0, 1, use_clahe=True, tiles=(5, 4))
    before = [out2.download(0, lvl) for lvl in range(4)]
    assert np.array_equal(before[0], _clahe_ref(imgs[0], 3.0, (5, 4)))
    api.preprocess(ctx, raw, out2, 1, 2, use_clahe=True)
    for lvl in range(4):
        assert np.array_equal(out2.download(0, lvl), before[lvl]), lvl
    for f in (1, 2):
        eq = _clahe_ref(imgs[f], 3.0, (w // 50, h // 50))
        ref = R.build_pyramid_ref(eq, 3)
        for lvl in range(4):
            assert np.array_equal(out2.download(f, lvl), ref[lvl]), (f, lvl)
    for p in (raw, out, out2):
        p.close()
