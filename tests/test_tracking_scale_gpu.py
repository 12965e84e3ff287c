"""ov2_klt_tracking and ov2_stereo_matching at the frame sizes and keypoint counts of the shipped configurations, bit-equal to
oracle/klt_tracking_ref.py and oracle/stereo_matching_ref.py on every output.

Each call runs one CTA of 256 threads per frame, and each thread strides over the frame's keypoints, so these tests use frames
of 0, 1, 255, 256, 257, 512, 513 keypoints and one keypoint per grid cell of the configuration (EuRoC 752 x 480, KITTI
1241 x 376 and TartanAir 640 x 480 with cell size 35: 308, 396 and 266), the P3P rule on counts gathered over every warp and
stride (300 and 1 100 pass-1 keypoints, 99 / 98 and 363 / 362 good), and a 132-keyframe batch of about 1 120 keypoints per
frame at 1280 x 720 on a fresh context (its scratch arena grows during the call), then again on the same context.  That batch
is checked against the oracle on sampled frames (first, middle, last, largest, the 257-keypoint frame), each through a call
of its own: a frame's results depend on its own inputs only.  Both calls are also run inside a batch the caller opened, with
host outputs read after ov2_batch_end, and with CUDA tensors.
"""
import functools

import numpy as np
import pytest

from ov2slam_b200 import api, synth
from oracle import image_ref as R
from oracle import klt_tracking_ref as KT
from oracle import stereo_matching_ref as S
from test_klt_tracking_gpu import KEYS as KT_KEYS, _assert_same as _assert_klt
from test_stereo_matching_gpu import KEYS as SM_KEYS, _assert_same as _assert_stereo, _near_tie, _regrid

pytestmark = pytest.mark.gpu

STRIDE_COUNTS = [0, 1, 255, 256, 257, 512, 513]
KLT_SIZES = {"euroc": (752, 480), "kitti": (1241, 376), "tartanair": (640, 480)}
# (size, rectified, distorted, cell size): EuRoC's rig is not rectified; KITTI's accurate / average configurations rectify
# (cell size 35) and its fast one does not (50); C4 is the shape scripts/bench_stereo_matching.py times.
STEREO_GEOMETRIES = {"euroc-35": ((752, 480), 0, 1, 35), "euroc-45": ((752, 480), 0, 1, 45), "euroc-50": ((752, 480), 0, 1, 50),
                     "kitti-rect-35": ((1241, 376), 1, 0, 35), "kitti-50": ((1241, 376), 0, 0, 50),
                     "c4-rect-35": ((1280, 720), 1, 0, 35)}
BW, BH, BNF = 1280, 720, 132
PER_KF = ("Tcw", "K", "dist", "Trl", "Frl", "img_wh", "grid")


def _cells(w, h, cs):
    return -(-w // cs) * -(-h // cs)


def _pyramids(ctx, a, b):
    nf, h, w = np.asarray(a).shape
    pa, pb = api.Pyramid(ctx, nf, w, h, 3), api.Pyramid(ctx, nf, w, h, 3)
    pa.build(np.asarray(a))
    pb.build(np.asarray(b))
    return pa, pb


def _klt(ctx, pyrs, sc, use_prior=True, first=0, out=None, arrays=None):
    a = dict(sc, **(arrays or {}))
    return api.FeatureTracker(ctx, 30, 0.01).klt_tracking(pyrs[0], pyrs[1], 9, 3, 30.0, 0.5, sc["offsets"], a["Tcw"], a["K"],
                                                           a["img_wh"], a["px"], a["wpt"], a["is3d"], dist=a["dist"],
                                                           use_prior=use_prior, first=first, out=out)


def _klt_ref(sc, use_prior=True, first=0):
    return KT.klt_tracking_ref(sc["prevs"], sc["curs"], sc["offsets"], sc["Tcw"], sc["K"], sc["img_wh"], sc["px"], sc["wpt"],
                               sc["is3d"], dist=sc["dist"], win=9, nklt_pyr_lvl=3, use_prior=use_prior, first=first)


def _stereo(ctx, pyrs, sc, first=0, out=None, arrays=None):
    a = dict(sc, **(arrays or {}))
    return api.FeatureTracker(ctx, 30, 0.01).stereo_matching(
        pyrs[0], pyrs[1], 9, 3, 30.0, 0.5, sc["rectified"], sc["offsets"], a["Tcw"], a["K"], a["Trl"], a["img_wh"], a["px"],
        a["unpx"], a["bv"], a["is3d"], a["has_mp"], a["wpt"], dist=a["dist"], Frl=a["Frl"], cell_offsets=sc["cell_offsets"],
        grid=a["grid"], cell_ptr=a["cell_ptr"], cell_kps=a["cell_kps"], first=first, out=out)


def _stereo_ref(sc, first=0):
    return S.stereo_matching_ref(sc["lefts"], sc["rights"], sc["offsets"], sc["Tcw"], sc["K"], sc["Trl"], sc["img_wh"], sc["px"],
                                 sc["unpx"], sc["bv"], sc["is3d"], sc["has_mp"], sc["wpt"], sc["rectified"], dist=sc["dist"],
                                 Frl=sc["Frl"], cell_offsets=sc["cell_offsets"], grid=sc["grid"], cell_ptr=sc["cell_ptr"],
                                 cell_kps=sc["cell_kps"], win=9, nklt_pyr_lvl=3, first=first)


def _frame(sc, f, per_frame):
    """Frame f alone: one-frame offsets and per-frame arrays, the keypoint arrays and the images of the whole batch (the
    oracle and the call index them by first + 0)."""
    o0, o1 = int(sc["offsets"][f]), int(sc["offsets"][f + 1])
    sub = dict(sc, offsets=np.array([0, o1 - o0], np.int32), **{k: None if sc[k] is None else sc[k][f:f + 1] for k in per_frame})
    for k in ("px", "unpx", "bv", "wpt", "is3d", "has_mp"):
        if k in sc:
            sub[k] = sc[k][o0:o1]
    if "cell_offsets" in sc:
        c0, c1 = int(sc["cell_offsets"][f]), int(sc["cell_offsets"][f + 1])
        sub["cell_offsets"] = np.array([0, c1 - c0], np.int32)
        sub["cell_ptr"] = sc["cell_ptr"][c0:c1 + 1] - sc["cell_ptr"][c0]
        sub["cell_kps"] = sc["cell_kps"][o0:o1] - o0
    return sub, slice(o0, o1)


# ----------------------------------------------------------------------------------------------------------- kltTracking
@functools.lru_cache(maxsize=None)
def _klt_scene(size, distorted):
    w, h = KLT_SIZES[size]
    return synth.make_klt_tracking_scene(300 + w, STRIDE_COUNTS + [_cells(w, h, 35)], w, h, distorted=distorted)


@pytest.mark.parametrize("use_prior", [1, 0])
@pytest.mark.parametrize("distorted", [False, True])
@pytest.mark.parametrize("size", list(KLT_SIZES))
def test_klt_tracking_stride_boundaries(ctx, size, distorted, use_prior):
    sc = _klt_scene(size, distorted)
    ref = _klt_ref(sc, use_prior)
    pyrs = _pyramids(ctx, sc["prevs"], sc["curs"])
    _assert_klt(_klt(ctx, pyrs, sc, use_prior), ref, (size, distorted, use_prior))
    offs = sc["offsets"]
    for f in range(2, len(offs) - 1):                   # every frame of more than one stride tracks in both passes
        sl = slice(offs[f], offs[f + 1])
        assert (ref["passes"][sl] == 2).any() and ref["status"][sl].any() and not ref["status"][sl].all(), f
        assert (ref["passes"][sl] == 1).any() == bool(use_prior) and (ref["nbkps"][f] > 0) == bool(use_prior), f
    for p in pyrs:
        p.close()


def _pass1_pool(seed, n, w, h):
    """A frame of n 3-D keypoints with in-image priors, and each one's pass-1 outcome by the oracle."""
    pool = synth.make_klt_tracking_scene(seed, [n], w, h, frac3d=1.0, bad_frac=0.6)
    pri = np.zeros((n, 2), np.float32)
    inside = np.zeros(n, bool)
    for i in range(n):
        x, y, inside[i] = KT.prior(pool["Tcw"][0], pool["K"][0], None, w, h, pool["wpt"][i])
        pri[i] = (x, y)
    idx = np.nonzero(inside)[0]
    st = np.zeros(n, np.uint8)
    st[idx] = R.fb_klt_ref(pool["prevs"][0], pool["curs"][0], pool["px"][idx], pri[idx], 9, 1)[1]
    return pool, idx[st[idx] == 1], idx[st[idx] == 0]


@functools.lru_cache(maxsize=None)
def _p3p_pool():
    return _pass1_pool(77, 2000, 640, 480)


@pytest.mark.parametrize("side", ["kept", "reset"])
def test_klt_tracking_p3p_rule_across_strides(ctx, side):
    """Frames of 300 and 1 100 pass-1 keypoints whose good tracks are spread over every warp and stride: 99 and 363 good are
    not below 0.33 * nbkps (the retries keep their priors), 98 and 362 are (reset)."""
    pool, good, bad = _p3p_pool()
    assert len(good) >= 363 and len(bad) >= 738, (len(good), len(bad))
    rng = np.random.default_rng(5)
    picks, at = [], []
    for nbkps, ngood in ((300, 99), (1100, 363)):
        ngood -= side == "reset"
        slots = np.round(np.linspace(0, nbkps - 1, ngood)).astype(int)
        pick = np.empty(nbkps, np.int64)
        mask = np.zeros(nbkps, bool)
        mask[slots] = True
        pick[mask] = rng.permutation(good)[:ngood]
        pick[~mask] = rng.permutation(bad)[:nbkps - ngood]
        assert len(set((slots % 256) // 32)) == 8 and (slots >= 256).any()
        picks.append(pick)
        at.append(ngood)
    pick = np.concatenate(picks)
    two = lambda a: np.concatenate([a, a])
    sc = dict(pool, prevs=two(pool["prevs"]), curs=two(pool["curs"]), offsets=np.array([0, 300, 1400], np.int32),
              Tcw=two(pool["Tcw"]), K=two(pool["K"]), img_wh=two(pool["img_wh"]), px=pool["px"][pick].copy(),
              wpt=pool["wpt"][pick].copy(), is3d=pool["is3d"][pick].copy())
    ref = _klt_ref(sc)
    assert list(ref["nbkps"]) == [300, 1100] and list(ref["nbgood"]) == at
    assert list(ref["p3p_req"]) == [side == "reset"] * 2
    pyrs = _pyramids(ctx, sc["prevs"], sc["curs"])
    _assert_klt(_klt(ctx, pyrs, sc), ref, side)
    for p in pyrs:
        p.close()


# -------------------------------------------------------------------------------------------------------- stereoMatching
def _stereo_scene(seed, counts, w, h, rect, distorted, cs, ref_frames=None):
    """A stereo scene whose right images sit about 2 px below the left ones, so that the row gate both keeps and rejects, with a
    2-D keypoint at x = 5 in every keyframe (its row search window shrinks to nothing: xprior = -1).  Redrawn while the
    oracle's epipolar errors on ref_frames (all frames by default) hold a near tie; returns the scene and those frames'
    oracle results."""
    for s in range(seed, seed + 20):
        rng = np.random.default_rng(s)
        shifts = [(rng.uniform(-8, -1), rng.choice([-1, 1]) * rng.uniform(1.6, 2.4)) for _ in counts]
        sc = synth.make_stereo_matching_scene(s, counts, w, h, rectified=rect, distorted=distorted, cs=cs, shifts=shifts)
        for f in range(len(counts)):
            o0, o1 = sc["offsets"][f], sc["offsets"][f + 1]
            two_d = np.nonzero(sc["is3d"][o0:o1] == 0)[0]
            if len(two_d):
                i = o0 + two_d[0]
                sc["px"][i] = sc["unpx"][i] = (5.0, sc["px"][i, 1])
        _regrid(sc)
        if ref_frames is None:
            refs = {None: _stereo_ref(sc)}
        else:
            refs = {f: _stereo_ref(_frame(sc, f, PER_KF)[0], first=f) for f in ref_frames}
        if not any(_near_tie(r) for r in refs.values()):
            return sc, refs
    raise AssertionError("no scene without a near tie")



def _assert_both_ways(sc, f, passes, stereo):
    """Keyframe f's outcomes (its slices of the passes and stereo outputs) go both ways: passes 1 and 2, stereo and rejected
    tracks, and on rectified rigs accepted row searches and xprior = -1."""
    st = stereo.astype(bool)
    assert (passes == 1).any() and (passes == 2).any(), f
    assert st.any() and (~st & (passes > 0)).any(), (f, st.sum(), (passes > 0).sum())
    if not sc["rectified"]:
        return
    lv = [R.build_pyramid_ref(im[f], 3)[3] for im in (sc["lefts"], sc["rights"])]
    down, up = np.float32(0.125), np.float32(8)
    seen = set()
    for i in range(sc["offsets"][f], sc["offsets"][f + 1]):
        if sc["is3d"][i]:
            continue
        p = sc["px"][i]
        xp = np.float32(R.line_min_sad_ref(lv[0], lv[1], (p[0] * down, p[1] * down), S.SAD_WIN, True)[0]) * up
        seen.add(bool(0 <= xp <= p[0]))
        if len(seen) == 2:
            return
    raise AssertionError((f, seen))


@pytest.mark.parametrize("geometry", list(STEREO_GEOMETRIES))
def test_stereo_matching_stride_boundaries(ctx, geometry):
    (w, h), rect, distorted, cs = STEREO_GEOMETRIES[geometry]
    sc, refs = _stereo_scene(400 + cs, STRIDE_COUNTS + [_cells(w, h, cs)], w, h, rect, distorted, cs)
    ref = refs[None]
    pyrs = _pyramids(ctx, sc["lefts"], sc["rights"])
    _assert_stereo(_stereo(ctx, pyrs, sc), ref, geometry)
    for f in range(2, len(sc["offsets"]) - 1):
        sl = slice(sc["offsets"][f], sc["offsets"][f + 1])
        _assert_both_ways(sc, f, ref["passes"][sl], ref["stereo"][sl])
    for p in pyrs:
        p.close()


# ----------------------------------------------------------------------------------------------------- bench-shaped batch
def _bench_counts():
    counts = np.random.default_rng(132).integers(1000, 1201, BNF)
    counts[40], counts[41] = 0, 257
    return [int(c) for c in counts]


def _sampled(counts):
    return sorted({0, BNF // 2, BNF - 1, 41, int(np.argmax(counts))})


@pytest.fixture(scope="module")
def fresh_ctx():
    """A context of this module's own, so that its scratch arena first grows inside the calls below."""
    c = api.Context(0)
    yield c
    c.close()


def test_klt_tracking_bench_batch(fresh_ctx):
    counts = _bench_counts()
    sc = synth.make_klt_tracking_scene(132, counts, BW, BH)
    pyrs = _pyramids(fresh_ctx, sc["prevs"], sc["curs"])
    first = _klt(fresh_ctx, pyrs, sc)
    _assert_klt(_klt(fresh_ctx, pyrs, sc), first, "consolidated arena")
    for f in _sampled(counts):
        sub, sl = _frame(sc, f, ("Tcw", "K", "dist", "img_wh"))
        ref = _klt_ref(sub, first=f)
        got = {k: first[k][sl] if k in ("tracked", "status", "passes") else first[k][f:f + 1] for k in KT_KEYS}
        _assert_klt(got, ref, f)
        assert counts[f] == 0 or ((ref["passes"] == 1).any() and (ref["passes"] == 2).any()), f
    for p in pyrs:
        p.close()


@pytest.mark.parametrize("rect", [1, 0])
def test_stereo_matching_bench_batch(fresh_ctx, rect):
    counts = _bench_counts()
    sampled = _sampled(counts)
    sc, refs = _stereo_scene(500 + rect, counts, BW, BH, rect, 0, 35, ref_frames=sampled)
    pyrs = _pyramids(fresh_ctx, sc["lefts"], sc["rights"])
    first = _stereo(fresh_ctx, pyrs, sc)
    _assert_stereo(_stereo(fresh_ctx, pyrs, sc), first, "consolidated arena")
    for f in sampled:
        sl = slice(sc["offsets"][f], sc["offsets"][f + 1])
        got = {k: first[k][sl] if k != "nstereo" else first[k][f:f + 1] for k in SM_KEYS}
        _assert_stereo(got, refs[f], f)
        if counts[f] > 256:
            _assert_both_ways(sc, f, refs[f]["passes"], refs[f]["stereo"])
    for p in pyrs:
        p.close()


# ------------------------------------------------------------------------------------- caller's batch and device arrays
@functools.lru_cache(maxsize=None)
def _device_scenes():
    counts = [1120, 0, 1119]
    kl = synth.make_klt_tracking_scene(9, counts, BW, BH, distorted=True)
    st = synth.make_stereo_matching_scene(9, counts, BW, BH, rectified=True, shifts=[(-4.0, 2.0)] * 3)
    return kl, st


def test_callers_batch_and_device_arrays(ctx):
    torch = pytest.importorskip("torch")
    kl, st = _device_scenes()
    kp, sp = _pyramids(ctx, kl["prevs"], kl["curs"]), _pyramids(ctx, st["lefts"], st["rights"])
    k_host, s_host = _klt(ctx, kp, kl), _stereo(ctx, sp, st)
    assert k_host["status"].any() and s_host["stereo"].any()
    n, nf = len(kl["px"]), 3
    k_out = dict(tracked=np.full((n, 2), 7, np.float32), status=np.full(n, 7, np.uint8), passes=np.full(n, 7, np.uint8),
                 p3p_req=np.full(nf, 7, np.uint8), nbgood=np.full(nf, 7, np.int32), nbkps=np.full(nf, 7, np.int32))
    s_out = dict(right=np.full((n, 2), 7, np.float32), stereo=np.full(n, 7, np.uint8), passes=np.full(n, 7, np.uint8),
                 nstereo=np.full(nf, 7, np.int32))
    ctx.batch_begin()
    try:
        _klt(ctx, kp, kl, out=k_out)
        _stereo(ctx, sp, st, out=s_out)
    finally:
        ctx.batch_end()
    _assert_klt(k_out, k_host, "caller's batch")
    _assert_stereo(s_out, s_host, "caller's batch")
    cuda = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
    k_dev = {k: cuda(kl[k]) for k in ("Tcw", "K", "dist", "img_wh", "px", "wpt", "is3d")}
    s_dev = {k: cuda(st[k]) for k in ("Tcw", "K", "dist", "Trl", "Frl", "img_wh", "grid", "cell_ptr", "cell_kps", "px", "unpx", "bv",
                                      "is3d", "has_mp", "wpt")}
    k_out = {k: torch.full(v.shape, 7, dtype=getattr(torch, v.dtype.name), device="cuda") for k, v in k_host.items()}
    s_out = {k: torch.full(v.shape, 7, dtype=getattr(torch, v.dtype.name), device="cuda") for k, v in s_host.items()}
    torch.cuda.synchronize()
    _klt(ctx, kp, kl, out=k_out, arrays=k_dev)
    _stereo(ctx, sp, st, out=s_out, arrays=s_dev)
    ctx.sync()
    _assert_klt({k: v.cpu().numpy() for k, v in k_out.items()}, k_host, "device")
    _assert_stereo({k: v.cpu().numpy() for k, v in s_out.items()}, s_host, "device")
    for p in (*kp, *sp):
        p.close()
