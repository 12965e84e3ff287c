"""GPU tests of the fb-KLT counting hook (ov2_debug_klt_counts): the counting instantiation of fb_klt_kernel tracks exactly
as the product launch does, and the level set-ups and iterations it reports for each keypoint are those of the oracle
(oracle/image_ref.py::_lk_ref) on the same points.

The oracle's work is counted from the outside, without changing it: each level set-up gathers the template patch once
(_reflect101 twice) and both derivative patches (np.clip twice each), and each iteration gathers one search patch
(_reflect101 twice).  So set-ups = clip calls / 4 and iterations = reflect calls / 2 - set-ups, per fb_klt_ref call on one
keypoint, with the pyramids and derivative planes computed beforehand so that only the tracking loop is counted.
"""
import numpy as np
import pytest

from ov2slam_b200 import api
from oracle import image_ref as R
from test_frontend_gpu import _klt_inputs

pytestmark = pytest.mark.gpu


class _CountingNumpy:
    """numpy for image_ref's module globals, counting np.clip calls."""

    def __init__(self, counts):
        self._counts = counts

    def clip(self, *a, **k):
        self._counts["clip"] += 1
        return np.clip(*a, **k)

    def __getattr__(self, name):
        return getattr(np, name)


def _oracle_counts(monkeypatch, prev, cur, kps, pri, nbpyrlvl):
    """(tracked, status, counts (n, 2) int32) of fb_klt_ref, one keypoint at a time, counted as the module docstring says."""
    pyr_cache, d_cache = {}, {}
    build, scharr, reflect = R.build_pyramid_ref, R.scharr_ref, R._reflect101

    def build_cached(img, nlev=3):
        key = (id(img), nlev)
        if key not in pyr_cache:
            pyr_cache[key] = (img, build(img, nlev))
        return pyr_cache[key][1]

    def scharr_cached(img):
        if id(img) not in d_cache:
            d_cache[id(img)] = (img, scharr(img))
        return d_cache[id(img)][1]

    for im in (prev, cur):          # warm both caches before counting starts
        for lvl in build_cached(im, 3):
            scharr_cached(lvl)
    counts = {"clip": 0, "reflect": 0}

    def reflect_counted(idx, n):
        counts["reflect"] += 1
        return reflect(idx, n)

    monkeypatch.setattr(R, "build_pyramid_ref", build_cached)
    monkeypatch.setattr(R, "scharr_ref", scharr_cached)
    monkeypatch.setattr(R, "_reflect101", reflect_counted)
    monkeypatch.setattr(R, "np", _CountingNumpy(counts))
    n = len(kps)
    out, st, work = pri.copy(), np.zeros(n, np.uint8), np.zeros((n, 2), np.int32)
    for i in range(n):
        counts["clip"] = counts["reflect"] = 0
        o, s = R.fb_klt_ref(prev, cur, kps[i:i + 1], pri[i:i + 1], 9, nbpyrlvl)
        out[i], st[i] = o[0], s[0]
        assert counts["clip"] % 4 == 0 and counts["reflect"] % 2 == 0, counts
        setups = counts["clip"] // 4
        work[i] = setups, counts["reflect"] // 2 - setups
    monkeypatch.undo()
    return out, st, work


@pytest.mark.parametrize("nbpyrlvl", [0, 3])
def test_klt_counts_match_oracle(ctx, monkeypatch, nbpyrlvl):
    """Per keypoint, interior and border windows: the counting kernel's tracks equal the product launch's and the oracle's
    bit for bit, and its set-up and iteration counts equal the oracle's."""
    w, h = 640, 480
    prev, cur, flow, kps, is3d, pri = _klt_inputs(11, w, h, 24)
    kps, pri = np.ascontiguousarray(kps[-64:]), np.ascontiguousarray(pri[-64:])     # 40 interior + 24 border keypoints
    kps[5] = (-1.0, -1.0)                                                             # an empty slot: no work
    pp = api.Pyramid(ctx, 1, w, h, 3)
    cp = api.Pyramid(ctx, 1, w, h, 3)
    pp.build(prev[None])
    cp.build(cur[None])
    ft = api.FeatureTracker(ctx, 30, 0.01)
    n = len(kps)
    out, st = pri.copy(), np.zeros(n, np.uint8)
    ft.fb_klt_tracking(pp, cp, 9, nbpyrlvl, 30.0, 0.5, kps, out, st)
    cout, cst, cnt = pri.copy(), np.zeros(n, np.uint8), np.full((n, 2), -1, np.int32)
    ft.fb_klt_tracking(pp, cp, 9, nbpyrlvl, 30.0, 0.5, kps, cout, cst, counts_out=cnt)
    pp.close()
    cp.close()
    assert np.array_equal(cout.view(np.uint32), out.view(np.uint32)) and np.array_equal(cst, st)

    valid = kps[:, 0] >= 0
    rout, rst, rcnt = _oracle_counts(monkeypatch, prev, cur, kps[valid], pri[valid], nbpyrlvl)
    assert np.array_equal(out[valid].view(np.uint32), rout.view(np.uint32)) and np.array_equal(st[valid], rst)
    assert np.array_equal(cnt[~valid], np.zeros((1, 2), np.int32))
    bad = np.nonzero((cnt[valid] != rcnt).any(axis=1))[0]
    assert bad.size == 0, (bad, cnt[valid][bad], rcnt[bad])
    # the set exercises more than one level and many iterations
    assert rcnt[:, 0].max() >= 2 and rcnt[:, 1].sum() > 3 * len(rcnt)


def test_klt_counts_batched_persistent(ctx):
    """A batch larger than the resident warps (the work-counter launch): the counting kernel returns the product launch's
    tracks, and every keypoint's counts are plausible (a tracked keypoint set up at least its forward level 0 and the
    backward level, and iterated at least once on each)."""
    w, h, nfr, per = 320, 240, 24, 256
    data = [_klt_inputs(300 + f, w, h, 40) for f in range(nfr)]
    kps = np.zeros((nfr * per, 2), np.float32) - 1
    pri = kps.copy()
    for f, d in enumerate(data):
        m = min(per, len(d[3]))
        kps[f * per:f * per + m], pri[f * per:f * per + m] = d[3][:m], d[5][:m]
    pp = api.Pyramid(ctx, nfr, w, h, 3)
    cp = api.Pyramid(ctx, nfr, w, h, 3)
    pp.build(np.stack([d[0] for d in data]))
    cp.build(np.stack([d[1] for d in data]))
    ft = api.FeatureTracker(ctx, 30, 0.01)
    n = len(kps)
    out, st = pri.copy(), np.zeros(n, np.uint8)
    ft.fb_klt_tracking(pp, cp, 9, 3, 30.0, 0.5, kps, out, st, per_frame=per)
    cout, cst, cnt = pri.copy(), np.zeros(n, np.uint8), np.full((n, 2), -1, np.int32)
    ft.fb_klt_tracking(pp, cp, 9, 3, 30.0, 0.5, kps, cout, cst, per_frame=per, counts_out=cnt)
    pp.close()
    cp.close()
    assert np.array_equal(cout.view(np.uint32), out.view(np.uint32)) and np.array_equal(cst, st)
    assert (cnt >= 0).all()
    assert (cnt[kps[:, 0] < 0] == 0).all()
    ok = st == 1
    assert ok.sum() > n // 4
    assert (cnt[ok, 0] >= 2).all() and (cnt[ok, 1] >= 2).all()
    assert (cnt[:, 0] <= 5).all() and (cnt[:, 1] <= 5 * 30).all()
