"""GPU tests of every run-time dispatch path of the KLT tracker (ov2_fb_klt) and the pyramid build (ov2_pyr_build).

ov2_fb_klt tracks every keypoint with one fb_klt_kernel launch, one warp per keypoint, and picks its code paths from the
input: a global work counter once the grid exceeds the resident CTAs; word-aligned or byte / reflected template and search
reads; 32-bit or split 64-bit mismatch sums.
The pyramid runs a fused TMA kernel only for 3 extra levels, level 3 >= 8 x 8 and a 16-byte-aligned level 0, and
pyr_down_kernel otherwise.  Every case here is compared bit for bit with oracle/image_ref.py (fb_klt_ref,
build_pyramid_ref) and, where cv2 is importable, the KLT statuses with fb_klt_cv2.  Oracle results are computed once per
module and shared between parametrisations (fb_klt_ref costs ~3 ms per keypoint).
"""
from contextlib import contextmanager

import numpy as np
import pytest

from ov2slam_b200 import api, synth
from oracle import image_ref as R
from test_frontend_gpu import _klt_assert, _klt_inputs, unaligned_device_frames

pytestmark = pytest.mark.gpu


@contextmanager
def _launches(ctx):
    """Kernel name -> launch count of the calls inside the block (the context's per-launch profiler)."""
    got = {}
    ctx.profile(True)
    try:
        yield got
        got.update({k: n for k, (_, n) in ctx.profile_report().items()})
    finally:
        ctx.profile(False)


def _oracle(prevs, curs, kps, pri, lv, fidx, idx=None):
    """fb_klt_ref over a ragged batch, one call per (frame, depth) group, for the keypoints `idx` (default: all).  Empty
    slots (x < 0) keep their prior with status 0.  Where cv2 is importable the statuses are checked against fb_klt_cv2."""
    idx = np.arange(len(kps)) if idx is None else np.asarray(idx)
    out, st = pri[idx].copy(), np.zeros(len(idx), np.uint8)
    for f in np.unique(fidx[idx]):
        for lvl in np.unique(lv[idx]):
            m = np.nonzero((fidx[idx] == f) & (lv[idx] == lvl) & (kps[idx, 0] >= 0))[0]
            if not len(m):
                continue
            k = idx[m]
            out[m], st[m] = R.fb_klt_ref(prevs[f], curs[f], kps[k], pri[k], 9, int(lvl))
            if R.HAVE_CV2:
                _, cs = R.fb_klt_cv2(prevs[f], curs[f], kps[k], pri[k], 9, int(lvl))
                assert np.array_equal(st[m], cs), ("oracle vs cv2", int(f), int(lvl), k[st[m] != cs])
    return out, st


def _track(ctx, pp, cp, kps, pri, lv, **kw):
    out = pri.copy()
    st = np.full(len(kps), 7, np.uint8)         # every slot must be written
    api.FeatureTracker(ctx, 30, 0.01).fb_klt_tracking(pp, cp, 9, lv, 30.0, 0.5, kps, out, st, **kw)
    return out, st


def _assert_same(got, ref, what=""):
    (out, st), (rp, rs) = got, ref
    assert np.array_equal(st, rs), (what, np.nonzero(st != rs)[0][:20])
    assert np.array_equal(out, rp), (what, float(np.abs(out - rp).max()), int((out != rp).any(axis=1).sum()))


def _pyramids(ctx, prevs, curs, extra=3):
    nf, h, w = prevs.shape
    pp, cp = api.Pyramid(ctx, nf, w, h, extra), api.Pyramid(ctx, nf, w, h, extra)
    pp.build(prevs)
    cp.build(curs)
    return pp, cp


def _assert_pyr(pyr, imgs, extra):
    for f in range(len(imgs)):
        ref = R.build_pyramid_ref(imgs[f], extra)
        for lvl in range(extra + 1):
            got = pyr.download(f, lvl)
            assert np.array_equal(got, ref[lvl]), (f, lvl, int((got != ref[lvl]).sum()))


# ---------------------------------------------------------------- 1. pyramid geometry and level-0 alignment
@pytest.mark.parametrize("extra", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("w,h", [(16, 16), (17, 31), (56, 64), (57, 64), (100, 70), (1241, 376)])
def test_pyramid_sizes_and_depths(ctx, w, h, extra):
    """Host images from the 16 x 16 minimum up: odd sizes, levels of 1 - 2 px, 0 - 4 extra levels.  56 x 64 (level 3 is
    7 x 8) takes pyr_down_kernel, 57 x 64 (level 3 is 8 x 8) the fused kernel with a TMA box larger than the image."""
    imgs = np.stack([synth.make_frame(200 + i, w, h) for i in range(2)])
    pyr = api.Pyramid(ctx, 2, w, h, extra)
    with _launches(ctx) as k:
        pyr.build(imgs)
    fused = extra == 3 and (w, h) != (16, 16) and (w, h) != (17, 31) and (w, h) != (56, 64)
    assert ("pyr_levels_kernel" in k) == fused and k.get("pyr_down_kernel", 0) == (0 if fused else extra), k
    _assert_pyr(pyr, imgs, extra)
    pyr.close()


@pytest.mark.parametrize("extra", [1, 3, 4])
@pytest.mark.parametrize("src", ["w332", "w333", "w334", "w335", "roi", "base+1"])
def test_pyramid_device_level0_alignment(ctx, src, extra):
    """Level 0 aliasing device images that TMA cannot address: contiguous widths 332 - 335 (pitch % 16 != 0, pitch % 4 =
    0 - 3), a column ROI of a wider tensor (row_stride > w, base 5 bytes into a row) and a base one byte past a 16-byte
    boundary (pitch and frame stride multiples of 16).  All go through pyr_down_kernel and give the oracle's bytes."""
    torch = pytest.importorskip("torch")
    nf, h = 2, 245
    w = int(src[1:]) if src.startswith("w") else (333 if src == "roi" else 352)
    imgs = np.stack([synth.make_frame(300 + i, w, h) for i in range(nf)])
    pyr = api.Pyramid(ctx, nf, w, h, extra)
    if src.startswith("w"):
        d = torch.from_numpy(imgs).cuda()
        args = dict(images=d)
    elif src == "roi":
        W, x0 = 352, 5
        wide = np.random.default_rng(1).integers(0, 256, (nf, h, W), dtype=np.uint8)
        wide[:, :, x0:x0 + w] = imgs
        d = torch.from_numpy(wide).cuda()
        args = dict(images=d.data_ptr() + x0, count=nf, row_stride=W, frame_stride=W * h)
    else:
        d, args = unaligned_device_frames(imgs)
    torch.cuda.synchronize()
    with _launches(ctx) as k:
        pyr.build(**args)
    assert "pyr_levels_kernel" not in k and k.get("pyr_down_kernel", 0) == extra, k
    _assert_pyr(pyr, imgs, extra)
    pyr.close()
    del d


@pytest.mark.parametrize("extra", [2, 3])
def test_pyramid_build_one_slot_leaves_the_others(ctx, extra):
    """build(first=1, count=1) into a 3-frame pyramid rewrites slot 1 only (pyr_down_kernel and the fused kernel)."""
    w, h = 640, 480
    a = np.stack([synth.make_frame(400 + i, w, h) for i in range(3)])
    b = synth.make_frame(410, w, h)
    pyr = api.Pyramid(ctx, 3, w, h, extra)
    pyr.build(a)
    pyr.build(b[None], first=1, count=1)
    _assert_pyr(pyr, np.stack([a[0], b, a[2]]), extra)
    pyr.close()


@pytest.mark.parametrize("w,h", [(640, 480), (752, 480)])
def test_pyramid_unaligned_level0_equals_fused(ctx, w, h):
    """The same images built from an aligned level 0 (the fused kernel) and from a device view one byte past a 16-byte
    boundary (one pyr_down_kernel launch per level) give the same bytes."""
    imgs = np.stack([synth.make_frame(420 + i, w, h) for i in range(3)])
    got = {}
    for unfused in (False, True):
        pyr = api.Pyramid(ctx, 3, w, h, 3)
        d, args = unaligned_device_frames(imgs) if unfused else (None, dict(images=imgs))
        with _launches(ctx) as k:
            pyr.build(**args)
        assert ("pyr_levels_kernel" in k) != unfused and k.get("pyr_down_kernel", 0) == (3 if unfused else 0), k
        got[unfused] = [[pyr.download(f, lvl) for lvl in range(4)] for f in range(3)]
        pyr.close()
        del d
    for f in range(3):
        ref = R.build_pyramid_ref(imgs[f], 3)
        for lvl in range(4):
            assert np.array_equal(got[False][f][lvl], got[True][f][lvl]), (f, lvl)
            assert np.array_equal(got[True][f][lvl], ref[lvl]), (f, lvl)


# ---------------------------------------------------------------- 2. KLT: the default launch on one input set
@pytest.fixture(scope="module")
def klt_set():
    """640 x 480, 3 frames, ~1 100 keypoints (FAST corners + border bands), per-keypoint depths 0 - 3, a few empty slots,
    ragged frame_idx; oracle results of every keypoint."""
    w, h = 640, 480
    data = [_klt_inputs(60 + f, w, h, 40) for f in range(3)]
    prevs = np.stack([d[0] for d in data])
    curs = np.stack([d[1] for d in data])
    kps = np.concatenate([d[3] for d in data])
    pri = np.concatenate([d[5] for d in data])
    fidx = np.concatenate([np.full(len(d[3]), f, np.int32) for f, d in enumerate(data)])
    rng = np.random.default_rng(11)
    lv = rng.integers(0, 4, len(kps)).astype(np.uint8)
    kps[rng.choice(len(kps), 9, replace=False)] = -1.0
    ref = _oracle(prevs, curs, kps, pri, lv, fidx)
    assert ref[1].mean() > 0.5
    return dict(prevs=prevs, curs=curs, kps=kps, pri=pri, lv=lv, fidx=fidx, ref=ref)


@pytest.fixture(scope="module")
def klt_pyr(ctx, klt_set):
    pp, cp = _pyramids(ctx, klt_set["prevs"], klt_set["curs"])
    yield pp, cp
    pp.close()
    cp.close()


def test_klt_default_launch(ctx, klt_set, klt_pyr):
    """The whole set in one fb_klt_kernel launch: the same bits as the oracle for every keypoint."""
    s = klt_set
    with _launches(ctx) as k:
        got = _track(ctx, *klt_pyr, s["kps"], s["pri"], s["lv"], frame_idx=s["fidx"])
    _assert_same(got, s["ref"])
    assert k == {"fb_klt_kernel": 1}, k


# ---------------------------------------------------------------- 3. unaligned (device-aliased) level 0
@pytest.fixture(scope="module")
def unaligned_set():
    """Two 333 x 245 and two 334 x 245 frame pairs, 150 keypoints per frame, all inside the image; oracle results."""
    out = {}
    for w in (333, 334):
        h = 245
        pairs = [synth.make_pair(80 + f + w, w, h) for f in range(2)]
        prevs = np.stack([p[0] for p in pairs])
        curs = np.stack([p[1] for p in pairs])
        rng = np.random.default_rng(w)
        kps = np.stack([rng.uniform(0, w, 300), rng.uniform(0, h, 300)], 1).astype(np.float32)
        flows = np.repeat(np.stack([p[2] for p in pairs]), 150, axis=0)
        pri = (kps + flows + rng.normal(0, 1, kps.shape)).astype(np.float32)
        lv = rng.choice(np.array([1, 3], np.uint8), 300)
        fidx = np.repeat(np.arange(2, dtype=np.int32), 150)
        ref = _oracle(prevs, curs, kps, pri, lv, fidx)
        assert ref[1].mean() > 0.5
        out[w] = dict(prevs=prevs, curs=curs, kps=kps, pri=pri, lv=lv, fidx=fidx, ref=ref)
    return out


@pytest.mark.parametrize("src", ["w333", "w334", "roi"])
def test_klt_unaligned_level0(ctx, unaligned_set, src):
    """Pyramids aliasing device images whose level 0 is not word aligned (odd or 2-mod-4 pitch, a column ROI 3 bytes into
    a 352-byte row): the byte / reflected template staging and the plain search gather.  Equal to the oracle and to the
    same frames tracked from host-built pyramids."""
    torch = pytest.importorskip("torch")
    w = 333 if src == "roi" else int(src[1:])
    s = unaligned_set[w]
    nf, h = 2, 245
    hp, hc = _pyramids(ctx, s["prevs"], s["curs"])
    host = _track(ctx, hp, hc, s["kps"], s["pri"], s["lv"], frame_idx=s["fidx"])
    _assert_same(host, s["ref"], "host-built")
    dp, dc = api.Pyramid(ctx, nf, w, h, 3), api.Pyramid(ctx, nf, w, h, 3)
    keep = []
    for pyr, imgs in ((dp, s["prevs"]), (dc, s["curs"])):
        if src == "roi":
            W, x0 = 352, 3
            wide = np.random.default_rng(2).integers(0, 256, (nf, h, W), dtype=np.uint8)
            wide[:, :, x0:x0 + w] = imgs
            d = torch.from_numpy(wide).cuda()
            torch.cuda.synchronize()
            pyr.build(d.data_ptr() + x0, count=nf, row_stride=W, frame_stride=W * h)
        else:
            d = torch.from_numpy(imgs).cuda()
            torch.cuda.synchronize()
            pyr.build(d)
        keep.append(d)
    got = _track(ctx, dp, dc, s["kps"], s["pri"], s["lv"], frame_idx=s["fidx"])
    _assert_same(got, host, "device-aliased vs host-built")
    for p in (hp, hc, dp, dc):
        p.close()
    del keep


# ---------------------------------------------------------------- 4. high-gradient windows (split 64-bit sums)
KLT_B32_BOUND = 262000      # frontend_klt.cu: below it the mismatch sums fit one 32-bit reduction


def _block_texture(seed, w, h, shift):
    """Random 0 / 255 blocks of 2 x 2 px, and the same texture moved by `shift` (bilinear), each with +-1 grey of noise."""
    rng = np.random.default_rng(seed)
    base = np.kron(rng.integers(0, 2, ((h + 1) // 2, (w + 1) // 2)) * 255.0, np.ones((2, 2)))[:h, :w]
    prev = base + rng.integers(-1, 2, base.shape)
    cur = synth.shift_image(base, *shift) + rng.integers(-1, 2, base.shape)
    return (np.ascontiguousarray(np.clip(prev, 0, 255), np.uint8),
            np.ascontiguousarray(np.clip(np.rint(cur), 0, 255), np.uint8))


def _window_gradient_sums(img):
    """sum(|Ix| + |Iy|) (Scharr, the tracker's derivative units) of every 9 x 9 window, indexed by its top-left pixel."""
    ix, iy = R.scharr_ref(img)
    g = np.pad((np.abs(ix.astype(np.int64)) + np.abs(iy.astype(np.int64))).cumsum(0).cumsum(1), ((1, 0), (1, 0)))
    return g[9:, 9:] - g[:-9, 9:] - g[9:, :-9] + g[:-9, :-9]


@pytest.fixture(scope="module")
def high_gradient_set():
    """Two 320 x 240 block-texture pairs, 120 keypoints each on integer positions (so the level-0 template window is the
    integer window the Scharr box sums describe, with no bilinear averaging of the alternating derivatives)."""
    w, h, shift = 320, 240, (0.37, -0.61)
    pairs = [_block_texture(5 + f, w, h, shift) for f in range(2)]
    prevs = np.stack([p[0] for p in pairs])
    curs = np.stack([p[1] for p in pairs])
    boxes = [_window_gradient_sums(p) for p in prevs]
    share = np.mean([(b >= KLT_B32_BOUND).mean() for b in boxes])
    assert share > 0.8, share
    rng = np.random.default_rng(3)
    n = 240
    kps = np.stack([rng.integers(12, w - 12, n), rng.integers(12, h - 12, n)], 1).astype(np.float32)
    pri = (kps + np.float32(shift) + rng.uniform(-0.3, 0.3, kps.shape)).astype(np.float32)
    # depths 0 and 1: at coarser levels the blocks average out, and cv2's float window sums round away from the exact ones
    lv = rng.integers(0, 2, n).astype(np.uint8)
    fidx = np.repeat(np.arange(2, dtype=np.int32), n // 2)
    # keypoints whose forward level-0 template window needs the 64-bit sums (window top-left = keypoint - 4)
    xy = kps.astype(np.int64) - 4
    high = np.array([boxes[f][y, x] >= KLT_B32_BOUND for f, (x, y) in zip(fidx, xy)])
    assert high.mean() > 0.75, high.mean()
    ref = _oracle(prevs, curs, kps, pri, lv, fidx)
    assert ref[1].mean() > 0.8
    return dict(prevs=prevs, curs=curs, kps=kps, pri=pri, lv=lv, fidx=fidx, ref=ref)


def test_klt_high_gradient_windows(ctx, high_gradient_set):
    """Windows with sum(|Ix| + |Iy|) >= 262 000, where the mismatch sums need the split 64-bit reduction: bit-exact."""
    s = high_gradient_set
    pp, cp = _pyramids(ctx, s["prevs"], s["curs"])
    got = _track(ctx, pp, cp, s["kps"], s["pri"], s["lv"], frame_idx=s["fidx"])
    _assert_same(got, s["ref"])
    pp.close()
    cp.close()


# ---------------------------------------------------------------- 5. a batch larger than any resident grid
@pytest.fixture(scope="module")
def large_batch():
    """16 frames x 800 keypoints (fixed stride): 720 interior, 40 in the 8-px border bands, 40 empty slots interleaved;
    depths 0 - 3.  Oracle: a seeded sample of 1 500 interior keypoints plus every border one."""
    nfr, per, w, h = 16, 800, 640, 480
    prevs, curs, flows = synth.make_batch(700, nfr, w, h)
    rng = np.random.default_rng(5)
    kps = np.stack([rng.uniform(8, w - 8, (nfr, per)), rng.uniform(8, h - 8, (nfr, per))], -1).astype(np.float32)
    border = np.zeros((nfr, per), bool)
    border[:, 1::20] = True
    b = kps[border]
    side = rng.integers(0, 4, len(b))
    lo, hi = rng.uniform(0, 8, len(b)), rng.uniform(-8, 0, len(b))
    b[:, 0] = np.where(side == 0, lo, np.where(side == 1, w + hi, b[:, 0]))
    b[:, 1] = np.where(side == 2, lo, np.where(side == 3, h + hi, b[:, 1]))
    kps[border] = b
    empty = np.zeros((nfr, per), bool)
    empty[:, 10::20] = True
    kps[empty] = -1.0
    pri = (kps + flows[:, None, :] + rng.normal(0, 1, kps.shape)).astype(np.float32)
    kps, pri = kps.reshape(-1, 2), pri.reshape(-1, 2)
    border, empty = border.reshape(-1), empty.reshape(-1)
    lv = rng.integers(0, 4, nfr * per).astype(np.uint8)
    fidx = np.repeat(np.arange(nfr, dtype=np.int32), per)
    inner = np.nonzero(~border & ~empty)[0]
    idx = np.sort(np.concatenate([np.random.default_rng(6).choice(inner, 1500, replace=False), np.nonzero(border)[0]]))
    ref = _oracle(prevs, curs, kps, pri, lv, fidx, idx)
    return dict(prevs=prevs, curs=curs, kps=kps, pri=pri, lv=lv, per=per, idx=idx, empty=np.nonzero(empty)[0], ref=ref)


def test_klt_large_batch_work_counter(ctx, large_batch):
    """12 800 keypoints: 1 600 CTAs of 8 warps, more than an H100 holds resident (at most 2 048 threads per SM), so the
    launch takes the global work-counter path.  Equal to the oracle on its sample; empty slots get status 0 and keep
    their prior."""
    torch = pytest.importorskip("torch")
    s = large_batch
    n = len(s["kps"])
    assert (n + 7) // 8 > 8 * torch.cuda.get_device_properties(0).multi_processor_count
    pp, cp = _pyramids(ctx, s["prevs"], s["curs"])
    out, st = _track(ctx, pp, cp, s["kps"], s["pri"], s["lv"], per_frame=s["per"])
    _assert_same((out[s["idx"]], st[s["idx"]]), s["ref"], "oracle sample")
    assert not st[s["empty"]].any() and np.array_equal(out[s["empty"]], s["pri"][s["empty"]])
    assert st.mean() > 0.5
    pp.close()
    cp.close()


# ---------------------------------------------------------------- 6. small images at OpenCV's pyramid depth
SMALL = [(16, 16), (17, 16), (40, 30), (64, 48), (96, 72), (161, 83)]


@pytest.fixture(scope="module")
def small_sets():
    """Per size: one frame pair, 120 keypoints (random, plus the corners of the in-border test), priors within 1.5 px;
    oracle results for nbpyrlvl 1, 3 and the per-keypoint depths {0, 2, 4, 9, 255}."""
    out = {}
    for w, h in SMALL:
        prev, cur, _ = synth.make_pair(7, w, h)
        rng = np.random.default_rng(w * h)
        kps = (rng.random((120, 2)) * [w, h]).astype(np.float32)
        kps[:4] = [[1.0, 1.0], [w - 1.0, h / 2], [w / 2, h - 1.0], [w - 1.5, h - 1.5]]
        pri = (kps + rng.uniform(-1.5, 1.5, kps.shape)).astype(np.float32)
        fidx = np.zeros(120, np.int32)
        lvs = {1: np.full(120, 1, np.uint8), 3: np.full(120, 3, np.uint8),
               "mixed": rng.choice(np.array([0, 2, 4, 9, 255], np.uint8), 120)}
        refs = {k: _oracle(prev[None], cur[None], kps, pri, lv, fidx) for k, lv in lvs.items()}
        out[(w, h)] = dict(prev=prev, cur=cur, kps=kps, pri=pri, lvs=lvs, refs=refs)
    return out


@pytest.mark.parametrize("w,h", SMALL)
def test_klt_small_images_opencv_depth(ctx, small_sets, w, h):
    """cv::buildOpticalFlowPyramid stops before a level <= 9 px, and calcOpticalFlowPyrLK / the reference track from the
    depth it reached (17 x 16: 0, 40 x 30: 1, 64 x 48 and 96 x 72: 2, 161 x 83: 3), whatever nbpyrlvl says and however many
    levels the pyramid holds: equal to the oracle (whose statuses equal cv2's)."""
    s = small_sets[(w, h)]
    pp, cp = _pyramids(ctx, s["prev"][None], s["cur"][None])
    for key, lv in s["lvs"].items():
        got = _track(ctx, pp, cp, s["kps"], s["pri"], key if isinstance(key, int) else lv)
        _assert_same(got, s["refs"][key], key)
    pp.close()
    cp.close()


# ---------------------------------------------------------------- 7. inputs at the edges
@pytest.fixture(scope="module")
def edge_inputs(klt_set):
    """Keypoints on the klt_set frames: priors far outside the image (out of range at the coarsest level too), keypoints
    and priors exactly on the in-border bounds (1.0 and w - 1), empty-slot markers interleaved."""
    w, h = 640, 480
    rng = np.random.default_rng(21)
    kps = np.stack([rng.uniform(20, w - 20, 120), rng.uniform(20, h - 20, 120)], 1).astype(np.float32)
    pri = kps.copy()
    pri[0:12] = [[-1000, -1000], [5000, 3000], [w + 100, h / 2], [-100, h / 2], [w / 2, h + 120], [w / 2, -90],
                 [w + 9 * 8, 20], [-9 * 8 - 1, 20], [1e6, 1e6], [-1e6, 5], [w + 30, h + 30], [-30, -30]]
    kps[12:24] = [[1.0, 240], [w - 1.0, 240], [320, 1.0], [320, h - 1.0], [1.0, 1.0], [w - 1.0, h - 1.0],
                  [0.999, 100], [w - 1.001, 100], [300, 0.999], [300, h - 1.001], [0.0, 0.0], [w - 0.5, h - 0.5]]
    pri[12:24] = kps[12:24]
    pri[24:120] = kps[24:120] + rng.normal(0, 1.5, (96, 2)).astype(np.float32)
    empty = np.arange(30, 120, 9)
    kps[empty] = -1.0
    lv = rng.choice(np.array([1, 3], np.uint8), 120)          # the reference's two depths (visual_front_end.cpp:196,242)
    return dict(kps=kps, pri=pri, lv=lv, empty=empty)


def _edge_check(s, got, kps, pri, lv, frames):
    out, st = got
    full = np.ones(len(kps), bool)
    full[s["empty"]] = False
    assert not st[~full].any() and np.array_equal(out[~full], pri[~full])
    for f in np.unique(frames):
        for lvl in np.unique(lv):
            m = np.nonzero(full & (frames == f) & (lv == lvl))[0]
            if len(m):
                _klt_assert(out[m], st[m], s["prevs"][f], s["curs"][f], kps[m], pri[m], 9, int(lvl), min_frac=0.9)


def test_klt_edge_inputs_first_frame(ctx, klt_set, klt_pyr, edge_inputs):
    """Fixed-stride addressing from first_frame = 1 with per_frame = 120 (frames 1 and 2 of a 3-frame pyramid)."""
    e = edge_inputs
    kps, pri, lv = np.concatenate([e["kps"]] * 2), np.concatenate([e["pri"]] * 2), np.concatenate([e["lv"]] * 2)
    got = _track(ctx, *klt_pyr, kps, pri, lv, first_frame=1, per_frame=120)
    s = dict(klt_set, empty=np.concatenate([e["empty"], e["empty"] + 120]))
    _edge_check(s, got, kps, pri, lv, np.repeat(np.array([1, 2]), 120))


def test_klt_edge_inputs_ragged_frames(ctx, klt_set, klt_pyr, edge_inputs):
    """A ragged, non-monotonic frame_idx (2, 0, 1, 0, 2, ...)."""
    e = edge_inputs
    fidx = np.random.default_rng(4).integers(0, 3, 120).astype(np.int32)
    fidx[:5] = [2, 0, 1, 0, 2]
    got = _track(ctx, *klt_pyr, e["kps"], e["pri"], e["lv"], frame_idx=fidx)
    _edge_check(dict(klt_set, empty=e["empty"]), got, e["kps"], e["pri"], e["lv"], fidx)
