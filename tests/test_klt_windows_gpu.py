"""GPU tests of fbKltTracking with every window size from 3 to 31 other than 9 (fb_klt_win_kernel): statuses and
tracked positions bit-equal to oracle/image_ref.py::fb_klt_ref, which restates calcOpticalFlowPyrLK for any window.

Covered: 640 x 480 and 752 x 480 pairs with known flow, mixed per-keypoint depths, keypoints within `win` of every edge
and corner, priors whose search window starts past -win, empty slots, a ragged frame_idx, small images where the window
clamps the pyramid depth, host and device buffers, a device level 0 at an odd address and pitch, the one-shot and the
persistent (work-counter) launch, ov2_frontend_step with klt.win = 15, the counting hook, and the refusals of sizes
outside 3 .. 31.  Oracle results are computed once per module, with each image's pyramid and derivative planes cached.
"""
import numpy as np
import pytest

from ov2slam_b200 import api, synth
from oracle import image_ref as R
from test_frontend_gpu import _klt_inputs, unaligned_device_frames
from test_klt_counts_gpu import _CountingNumpy
from test_klt_pyr_paths_gpu import _launches

pytestmark = pytest.mark.gpu

WINDOWS = [w for w in range(3, 32) if w != 9]


@pytest.fixture(scope="module")
def cached_oracle():
    """fb_klt_ref with each image's pyramid and Scharr planes built once (the tracking loop is unchanged)."""
    pyr_cache, d_cache = {}, {}
    build, scharr = R.build_pyramid_ref, R.scharr_ref

    def build_cached(img, nlev=3):
        key = (id(img), nlev)
        if key not in pyr_cache:
            pyr_cache[key] = (img, build(img, nlev))
        return pyr_cache[key][1]

    def scharr_cached(img):
        if id(img) not in d_cache:
            d_cache[id(img)] = (img, scharr(img))
        return d_cache[id(img)][1]

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(R, "build_pyramid_ref", build_cached)
        mp.setattr(R, "scharr_ref", scharr_cached)
        yield R.fb_klt_ref


def _oracle(fb, prevs, curs, kps, pri, lv, fidx, win):
    """fb_klt_ref over a ragged batch, one call per (frame, depth) group; empty slots keep their prior with status 0."""
    out, st = pri.copy(), np.zeros(len(kps), np.uint8)
    for f in np.unique(fidx):
        for lvl in np.unique(lv):
            m = np.nonzero((fidx == f) & (lv == lvl) & (kps[:, 0] >= 0))[0]
            if len(m):
                out[m], st[m] = fb(prevs[f], curs[f], kps[m], pri[m], win, int(lvl))
    return out, st


def _track(ctx, pp, cp, win, kps, pri, lv, **kw):
    out = pri.copy()
    st = np.full(len(kps), 7, np.uint8)          # every slot must be written
    api.FeatureTracker(ctx, 30, 0.01).fb_klt_tracking(pp, cp, win, lv, 30.0, 0.5, kps, out, st, **kw)
    return out, st


def _assert_same(got, ref, what=""):
    (out, st), (rp, rs) = got, ref
    assert np.array_equal(st, rs), (what, np.nonzero(st != rs)[0][:20])
    assert np.array_equal(out.view(np.uint32), rp.view(np.uint32)), (what, float(np.abs(out - rp).max()),
                                                                       int((out != rp).any(axis=1).sum()))


def _pyramids(ctx, prevs, curs):
    nf, h, w = prevs.shape
    pp, cp = api.Pyramid(ctx, nf, w, h, 3), api.Pyramid(ctx, nf, w, h, 3)
    pp.build(prevs)
    cp.build(curs)
    return pp, cp


def _edge_keypoints(rng, w, h, win, n):
    """n keypoints within `win` of the edges and corners (inside the image), and the four corners themselves."""
    e = rng.uniform(0, win, (n, 2))
    side = rng.integers(0, 4, n)
    x = np.where(side == 0, e[:, 0], np.where(side == 1, w - 1e-3 - e[:, 0], rng.uniform(0, w, n)))
    y = np.where(side == 2, e[:, 1], np.where(side == 3, h - 1e-3 - e[:, 1], rng.uniform(0, h, n)))
    k = np.stack([x, y], 1)
    k[:4] = [[0.0, 0.0], [w - 0.5, 0.25], [0.5, h - 0.75], [w - 1.0, h - 1.0]]
    return k.astype(np.float32)


@pytest.fixture(scope="module")
def window_sets(cached_oracle):
    """Per window: two 640 x 480 frames and one 752 x 480 frame, each with 14 FAST keypoints (known flow, noisy priors),
    8 edge / corner keypoints, 2 priors far past -win (their search window leaves the image at every level) and 2 empty
    slots; per-keypoint depths 0 - 3; a shuffled (ragged) frame_idx.  Oracle results for each."""
    inputs = {}
    for w, h, seeds in ((640, 480, (31, 32)), (752, 480, (33,))):
        data = [_klt_inputs(s, w, h, 24) for s in seeds]
        inputs[(w, h)] = dict(prevs=np.stack([d[0] for d in data]), curs=np.stack([d[1] for d in data]),
                              kps=[d[3] for d in data], pri=[d[5] for d in data])
    sets = {}
    for win in WINDOWS:
        rng = np.random.default_rng(win)
        per_size = {}
        for (w, h), d in inputs.items():
            ks, ps, fs = [], [], []
            for f in range(len(d["kps"])):
                idx = rng.choice(len(d["kps"][f]) - 24, 14, replace=False)
                k = np.concatenate([d["kps"][f][idx], _edge_keypoints(rng, w, h, win, 8),
                                    rng.uniform(40, 200, (2, 2)).astype(np.float32), np.full((2, 2), -1, np.float32)])
                p = np.concatenate([d["pri"][f][idx], np.zeros((12, 2))])
                p[14:22] = k[14:22] + rng.normal(0, 1.0, (8, 2))
                p[22:24] = [[-3.0 * win - 200, 50.0], [60.0, -5.0 * win - 300]]
                p[24:26] = 5.0
                ks.append(k)
                ps.append(p.astype(np.float32))
                fs.append(np.full(len(k), f, np.int32))
            k, p, fi = np.concatenate(ks), np.concatenate(ps), np.concatenate(fs)
            order = rng.permutation(len(k))                      # ragged, non-monotonic frame_idx
            k, p, fi = np.ascontiguousarray(k[order]), np.ascontiguousarray(p[order]), np.ascontiguousarray(fi[order])
            lv = rng.integers(0, 4, len(k)).astype(np.uint8)
            ref = _oracle(cached_oracle, d["prevs"], d["curs"], k, p, lv, fi, win)
            per_size[(w, h)] = dict(kps=k, pri=p, lv=lv, fidx=fi, ref=ref)
        sets[win] = per_size
    tracked = np.mean([s[sz]["ref"][1].mean() for s in sets.values() for sz in s])
    assert tracked > 0.4, tracked
    return inputs, sets


@pytest.fixture(scope="module")
def window_pyrs(ctx, window_sets):
    inputs, _ = window_sets
    pyrs = {sz: _pyramids(ctx, d["prevs"], d["curs"]) for sz, d in inputs.items()}
    yield pyrs
    for pp, cp in pyrs.values():
        pp.close()
        cp.close()


@pytest.mark.parametrize("win", WINDOWS)
def test_klt_window_bit_exact(ctx, window_sets, window_pyrs, win):
    """640 x 480 and 752 x 480, one launch each of fb_klt_win_kernel: every keypoint's status and position equal the
    oracle's bits, empty slots keep their prior with status 0."""
    _, sets = window_sets
    for sz, s in sets[win].items():
        pp, cp = window_pyrs[sz]
        with _launches(ctx) as k:
            got = _track(ctx, pp, cp, win, s["kps"], s["pri"], s["lv"], frame_idx=s["fidx"])
        assert k == {"fb_klt_win_kernel": 1}, k
        _assert_same(got, s["ref"], (win, sz))
        empty = s["kps"][:, 0] < 0
        assert not got[1][empty].any() and np.array_equal(got[0][empty], s["pri"][empty])


@pytest.mark.parametrize("win", [4, 15, 31])
def test_klt_window_device_buffers(ctx, window_sets, window_pyrs, win):
    """The same keypoints, priors, depths, frame indices and statuses in device memory give the host-buffer bits."""
    torch = pytest.importorskip("torch")
    _, sets = window_sets
    s = sets[win][(640, 480)]
    pp, cp = window_pyrs[(640, 480)]
    dk, dp = torch.from_numpy(s["kps"]).cuda(), torch.from_numpy(s["pri"].copy()).cuda()
    dl, df = torch.from_numpy(s["lv"]).cuda(), torch.from_numpy(s["fidx"]).cuda()
    dst = torch.full((len(s["kps"]),), 7, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    api.FeatureTracker(ctx, 30, 0.01).fb_klt_tracking(pp, cp, win, dl, 30.0, 0.5, dk, dp, dst, frame_idx=df)
    ctx.sync()
    _assert_same((dp.cpu().numpy(), dst.cpu().numpy()), s["ref"], win)


SMALL = [(40, 30, 15), (96, 72, 21), (64, 48, 31), (17, 16, 4), (161, 83, 11)]


@pytest.mark.parametrize("w,h,win", SMALL)
def test_klt_window_small_images(ctx, cached_oracle, w, h, win):
    """Images whose levels the window outgrows: cv::buildOpticalFlowPyramid stops before a level <= win px and the track
    starts at that depth (40 x 30 at 15 and 96 x 72 at 21: level 1; 64 x 48 at 31: level 0), whatever nbpyrlvl says."""
    assert R.optflow_levels(w, h, win, 3) < 3
    prev, cur, _ = synth.make_pair(w + h + win, w, h)
    rng = np.random.default_rng(win)
    kps = (rng.random((60, 2)) * [w, h]).astype(np.float32)
    kps[:4] = [[1.0, 1.0], [w - 1.0, h / 2], [w / 2, h - 1.0], [w - 1.5, h - 1.5]]
    pri = (kps + rng.uniform(-1.5, 1.5, kps.shape)).astype(np.float32)
    lv = rng.choice(np.array([0, 1, 3, 9], np.uint8), 60)
    fidx = np.zeros(60, np.int32)
    ref = _oracle(cached_oracle, prev[None], cur[None], kps, pri, lv, fidx, win)
    pp, cp = _pyramids(ctx, prev[None], cur[None])
    _assert_same(_track(ctx, pp, cp, win, kps, pri, lv), ref, (w, h, win))
    pp.close()
    cp.close()


@pytest.mark.parametrize("win", [5, 21])
def test_klt_window_unaligned_level0(ctx, cached_oracle, win):
    """Pyramids aliasing device frames of width 333 (odd pitch) one byte past a 16-byte boundary: equal to the oracle."""
    pytest.importorskip("torch")
    w, h = 333, 245
    pairs = [synth.make_pair(500 + f, w, h) for f in range(2)]
    prevs, curs = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    rng = np.random.default_rng(win)
    kps = np.stack([rng.uniform(0, w, 80), rng.uniform(0, h, 80)], 1).astype(np.float32)
    pri = (kps + np.repeat(np.stack([p[2] for p in pairs]), 40, axis=0) + rng.normal(0, 1, kps.shape)).astype(np.float32)
    lv = rng.choice(np.array([1, 3], np.uint8), 80)
    fidx = np.repeat(np.arange(2, dtype=np.int32), 40)
    ref = _oracle(cached_oracle, prevs, curs, kps, pri, lv, fidx, win)
    dp, dc = api.Pyramid(ctx, 2, w, h, 3), api.Pyramid(ctx, 2, w, h, 3)
    bp, ap = unaligned_device_frames(prevs)
    bc, ac = unaligned_device_frames(curs)
    dp.build(**ap)
    dc.build(**ac)
    _assert_same(_track(ctx, dp, dc, win, kps, pri, lv, frame_idx=fidx), ref, win)
    dp.close()
    dc.close()
    del bp, bc


@pytest.mark.parametrize("win", [15, 21])
def test_klt_window_persistent_launch(ctx, cached_oracle, win):
    """16 frames x 256 keypoints (fixed stride, every 16th slot empty): more warps than the GPU holds resident, so the
    launch pulls keypoints from the work counter.  Equal to the oracle on a 160-keypoint sample, and each sampled
    keypoint tracked alone (one-shot launch) gives the same bits."""
    torch = pytest.importorskip("torch")
    nfr, per, w, h = 16, 256, 640, 480
    prevs, curs, flows = synth.make_batch(900 + win, nfr, w, h)
    rng = np.random.default_rng(win)
    kps = np.stack([rng.uniform(0, w, (nfr, per)), rng.uniform(0, h, (nfr, per))], -1).astype(np.float32)
    kps[:, ::16] = -1.0
    pri = (kps + flows[:, None, :] + rng.normal(0, 1, kps.shape)).astype(np.float32)
    kps, pri = kps.reshape(-1, 2), pri.reshape(-1, 2)
    lv = rng.integers(0, 4, nfr * per).astype(np.uint8)
    n = len(kps)
    # 4-warp CTAs of 45 088 B shared memory: at most 5 resident per SM (228 KB)
    assert (n + 3) // 4 > 5 * torch.cuda.get_device_properties(0).multi_processor_count
    pp, cp = _pyramids(ctx, prevs, curs)
    got = _track(ctx, pp, cp, win, kps, pri, lv, per_frame=per)
    idx = np.sort(np.random.default_rng(1).choice(n, 160, replace=False))
    fidx = (np.arange(n) // per).astype(np.int32)
    ref = _oracle(cached_oracle, prevs, curs, kps[idx], pri[idx], lv[idx], fidx[idx], win)
    _assert_same((got[0][idx], got[1][idx]), ref, "persistent vs oracle")
    one = _track(ctx, pp, cp, win, np.ascontiguousarray(kps[idx]), np.ascontiguousarray(pri[idx]),
                 np.ascontiguousarray(lv[idx]), frame_idx=fidx[idx])
    _assert_same(one, ref, "one-shot vs oracle")
    assert not got[1][kps[:, 0] < 0].any() and got[1].mean() > 0.4
    pp.close()
    cp.close()


def test_frontend_step_window_15(ctx):
    """ov2_frontend_step with klt.win = 15 equals the operator entry points called one by one."""
    w, h, nfr, nk = 640, 480, 2, 256
    data = [synth.make_pair(190 + f, w, h) for f in range(nfr)]
    prevs = np.stack([d[0] for d in data])
    curs = np.stack([d[1] for d in data])
    rng = np.random.default_rng(15)
    kps = np.stack([rng.uniform(0, w, nfr * nk), rng.uniform(0, h, nfr * nk)], axis=1).astype(np.float32)
    pri0 = (kps + np.repeat(np.stack([d[2] for d in data]), nk, axis=0)).astype(np.float32)
    lv = rng.integers(0, 4, nfr * nk).astype(np.uint8)
    ncell = (h // 50) * (w // 50)

    def outputs():
        return dict(pri=pri0.copy(), st=np.zeros(nfr * nk, np.uint8), th=np.full(nfr, 10, np.int32),
                    new=np.empty((nfr * ncell, 2), np.float32), cnt=np.zeros(nfr, np.int32),
                    dt=np.zeros((nfr * nk, 32), np.uint8), vt=np.zeros(nfr * nk, np.uint8),
                    dn=np.zeros((nfr * ncell, 32), np.uint8), vn=np.zeros(nfr * ncell, np.uint8))

    pp, cp = api.Pyramid(ctx, nfr, w, h, 3), api.Pyramid(ctx, nfr, w, h, 3)
    a = outputs()
    pp.build(prevs)
    cp.build(curs)
    ft, fe = api.FeatureTracker(ctx, 30, 0.01), api.FeatureExtractor(ctx)
    ft.fb_klt_tracking(pp, cp, 15, lv, 30.0, 0.5, kps, a["pri"], a["st"], per_frame=nk)
    fe.detect_grid_fast(cp, 50, 0, nfr, a["th"], a["new"], a["cnt"], max_per_frame=ncell)
    fe.describe_brief(cp, a["pri"], a["dt"], a["vt"], per_frame=nk)
    fe.describe_brief(cp, a["new"], a["dn"], a["vn"], per_frame=ncell)
    assert a["st"].mean() > 0.5
    b = outputs()
    args = api.FrontendStepArgs(prevs.ctypes.data, curs.ctypes.data, w, w * h, nfr,
                                api.KltParams(15, 30, float(np.float32(0.01)), 30.0, 0.5),
                                nfr * nk, nk, lv.ctypes.data, 0, kps.ctypes.data, b["pri"].ctypes.data, b["st"].ctypes.data, 50,
                                b["th"].ctypes.data, ncell, b["new"].ctypes.data, b["cnt"].ctypes.data, b["dt"].ctypes.data,
                                b["vt"].ctypes.data, b["dn"].ctypes.data, b["vn"].ctypes.data)
    for rep in range(2):
        b["pri"][...] = pri0
        b["th"][...] = 10
        with _launches(ctx) as k:
            api.frontend_step(ctx, pp, cp, args)
        assert rep > 0 or k.get("fb_klt_win_kernel") == 1, k
        for key in a:
            assert np.array_equal(a[key], b[key]), (rep, key)
    pp.close()
    cp.close()


def _oracle_counts(monkeypatch, prev, cur, kps, pri, nbpyrlvl, win):
    """Per keypoint: fb_klt_ref's result and its level set-ups / iterations, counted as tests/test_klt_counts_gpu.py
    counts them (clip calls / 4 and reflect calls / 2 - set-ups), for a win x win window."""
    reflect = R._reflect101
    counts = {"clip": 0, "reflect": 0}

    def reflect_counted(idx, n):
        counts["reflect"] += 1
        return reflect(idx, n)

    for im in (prev, cur):                        # fill the module's pyramid / derivative caches before counting
        for lvl in R.build_pyramid_ref(im, 3):
            R.scharr_ref(lvl)
    monkeypatch.setattr(R, "_reflect101", reflect_counted)
    monkeypatch.setattr(R, "np", _CountingNumpy(counts))
    n = len(kps)
    out, st, work = pri.copy(), np.zeros(n, np.uint8), np.zeros((n, 2), np.int32)
    for i in range(n):
        counts["clip"] = counts["reflect"] = 0
        o, s = R.fb_klt_ref(prev, cur, kps[i:i + 1], pri[i:i + 1], win, nbpyrlvl)
        out[i], st[i] = o[0], s[0]
        assert counts["clip"] % 4 == 0 and counts["reflect"] % 2 == 0, counts
        setups = counts["clip"] // 4
        work[i] = setups, counts["reflect"] // 2 - setups
    monkeypatch.undo()
    return out, st, work


@pytest.mark.parametrize("win", [3, 7, 21, 31])
def test_klt_window_counts(ctx, cached_oracle, monkeypatch, win):
    """The counting instantiation of fb_klt_win_kernel tracks as the product launch does, and reports the oracle's
    level set-ups and iterations for every keypoint (interior, border, one empty slot)."""
    w, h = 640, 480
    prev, cur, flow, kps, is3d, pri = _klt_inputs(11, w, h, 24)
    kps, pri = np.ascontiguousarray(kps[-48:]), np.ascontiguousarray(pri[-48:])
    kps[5] = (-1.0, -1.0)
    pp, cp = _pyramids(ctx, prev[None], cur[None])
    ft = api.FeatureTracker(ctx, 30, 0.01)
    n = len(kps)
    out, st = pri.copy(), np.zeros(n, np.uint8)
    ft.fb_klt_tracking(pp, cp, win, 3, 30.0, 0.5, kps, out, st)
    cout, cst, cnt = pri.copy(), np.zeros(n, np.uint8), np.full((n, 2), -1, np.int32)
    ft.fb_klt_tracking(pp, cp, win, 3, 30.0, 0.5, kps, cout, cst, counts_out=cnt)
    pp.close()
    cp.close()
    assert np.array_equal(cout.view(np.uint32), out.view(np.uint32)) and np.array_equal(cst, st)
    valid = kps[:, 0] >= 0
    rout, rst, rcnt = _oracle_counts(monkeypatch, prev, cur, kps[valid], pri[valid], 3, win)
    assert np.array_equal(out[valid].view(np.uint32), rout.view(np.uint32)) and np.array_equal(st[valid], rst)
    assert np.array_equal(cnt[~valid], np.zeros((1, 2), np.int32))
    bad = np.nonzero((cnt[valid] != rcnt).any(axis=1))[0]
    assert bad.size == 0, (bad, cnt[valid][bad], rcnt[bad])
    assert rcnt[:, 0].max() >= 2 and rcnt[:, 1].sum() > 3 * len(rcnt)


def test_klt_window_refusals(ctx, window_sets, window_pyrs):
    """Sizes 0, 2, 32 and -1 are refused with a message naming the range, outputs untouched; the same context then
    tracks at 15 and 9 as before."""
    _, sets = window_sets
    s = sets[15][(640, 480)]
    pp, cp = window_pyrs[(640, 480)]
    ft = api.FeatureTracker(ctx, 30, 0.01)
    for bad in (0, 2, 32, -1):
        out, st = s["pri"].copy(), np.full(len(s["kps"]), 7, np.uint8)
        with pytest.raises(api.Ov2Error, match=r"3 \.\. 31"):
            ft.fb_klt_tracking(pp, cp, bad, s["lv"], 30.0, 0.5, s["kps"], out, st, frame_idx=s["fidx"])
        assert np.array_equal(out, s["pri"]) and (st == 7).all()
    _assert_same(_track(ctx, pp, cp, 15, s["kps"], s["pri"], s["lv"], frame_idx=s["fidx"]), s["ref"], "after refusals")
    with _launches(ctx) as k:
        _track(ctx, pp, cp, 9, s["kps"], s["pri"], s["lv"], frame_idx=s["fidx"])
    assert k == {"fb_klt_kernel": 1}, k
