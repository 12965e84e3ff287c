"""ORB-fallback descriptors on both of ov2_describe's paths: the per-window kernel (each keypoint smooths its own
26 x 26 window) and the dense one (each frame smoothed once, then gathered).  OV2_DESC_DENSE forces a path; unset,
the density rule picks one.  Every path must give the oracle's bytes, and so the same bytes as each other."""
import numpy as np
import pytest

from ov2slam_b200 import api, synth
from oracle import image_ref as R

pytestmark = pytest.mark.gpu

MODES = {"per-window": "0", "dense": "1", "rule": None}
KERNELS = {"0": {"describe_kernel"}, "1": {"desc_smooth_kernel", "describe_dense_kernel"}}


def _limit_points(w, h):
    """Rounded centres exactly at the 31 px limits on all four sides and one pixel outside them, and half-pixel
    positions next to the limits that round both ways (cvRound is round-half-even)."""
    mx, my = w // 2, h // 2
    xs = [31, 30, w - 32, w - 31, 30.5, 31.5, 32.5, w - 32.5, w - 31.5, w - 30.5, 31.49, 30.51]
    ys = [31, 30, h - 32, h - 31, 30.5, 31.5, 32.5, h - 32.5, h - 31.5, h - 30.5, 31.49, 30.51]
    pts = [(x, my) for x in xs] + [(mx, y) for y in ys]
    pts += [(31, 31), (w - 32, h - 32), (31, h - 32), (w - 32, 31), (30, 31), (w - 31, h - 32)]
    return np.array(pts, np.float32)


def _points(rng, w, h, n):
    lim = _limit_points(w, h)
    pts = np.empty((n, 2), np.float32)
    pts[:] = (rng.random((n, 2)) * [w, h]).astype(np.float32)
    k = min(len(lim), n)
    pts[:k] = lim[:k]
    half = slice(k, k + n // 8)
    pts[half] = np.floor(pts[half]) + 0.5
    pts[rng.random(n) < 0.1] = [-1.0, -1.0]          # empty slots
    return pts


def _reference(im, pts):
    if R.HAVE_CV2:
        q = pts.copy()
        q[q[:, 0] < 0] = 0.0                          # cv2 drops (0, 0) by the border rule as the kernel drops x < 0
        return R.describe_cv2(im, q)
    return R.describe_ref(im, pts)


def _describe_all_modes(ctx, monkeypatch, pyr, pts, per_frame, first_frame=0):
    fe = api.FeatureExtractor(ctx)
    out = {}
    for name, env in MODES.items():
        if env is None:
            monkeypatch.delenv("OV2_DESC_DENSE", raising=False)
        else:
            monkeypatch.setenv("OV2_DESC_DENSE", env)
        desc = np.full((len(pts), 32), 0xA5, np.uint8)
        valid = np.full(len(pts), 7, np.uint8)
        ctx.profile(True)
        fe.describe_brief(pyr, pts, desc, valid, first_frame=first_frame, per_frame=per_frame)
        ran = {k for k in ctx.profile_report()}
        ctx.profile(False)
        if env is not None:
            assert ran == KERNELS[env], (name, ran)
        out[name] = (desc, valid, ran)
    monkeypatch.delenv("OV2_DESC_DENSE", raising=False)
    return out


def _check(out, imgs, pts, per_frame, first_frame=0):
    for f in range(len(pts) // per_frame):
        sl = slice(f * per_frame, (f + 1) * per_frame)
        rd, rv = _reference(imgs[first_frame + f], pts[sl])
        for name, (desc, valid, _) in out.items():
            assert np.array_equal(valid[sl], rv), (name, f)
            assert np.array_equal(desc[sl], rd), (name, f, int(np.unpackbits(desc[sl] ^ rd).sum()))
    base = out["per-window"]
    for name, (desc, valid, _) in out.items():
        assert np.array_equal(desc, base[0]) and np.array_equal(valid, base[1]), name


@pytest.mark.parametrize("w,h", [(640, 480), (752, 480), (1241, 376), (1280, 720), (63, 63)])
@pytest.mark.parametrize("per_frame", [40, 1300])
def test_describe_paths_bit_exact(ctx, monkeypatch, w, h, per_frame):
    nfr = 2
    imgs = np.stack([synth.make_frame(70 + i, w, h) for i in range(nfr)])
    imgs[1] = np.random.default_rng(w + h).integers(0, 256, (h, w)).astype(np.uint8)   # raw noise
    pyr = api.Pyramid(ctx, nfr, w, h, 0)
    pyr.build(imgs)
    rng = np.random.default_rng(per_frame * 7 + w)
    pts = np.concatenate([_points(rng, w, h, per_frame) for _ in range(nfr)])
    out = _describe_all_modes(ctx, monkeypatch, pyr, pts, per_frame)
    _check(out, imgs, pts, per_frame)
    pyr.close()


def test_describe_rule_sides_of_crossover(ctx, monkeypatch):
    """At C2's geometry the rule takes the dense path for a dense set (1024 per frame) and the per-window path for
    a sparse one (108 per frame, the new keypoints of 40 px cells)."""
    w, h = 640, 480
    imgs = synth.make_frame(90, w, h)[None]
    pyr = api.Pyramid(ctx, 1, w, h, 0)
    pyr.build(imgs)
    rng = np.random.default_rng(3)
    for per_frame, want in ((1024, "1"), (108, "0")):
        pts = _points(rng, w, h, per_frame)
        out = _describe_all_modes(ctx, monkeypatch, pyr, pts, per_frame)
        assert out["rule"][2] == KERNELS[want], (per_frame, out["rule"][2])
        _check(out, imgs, pts, per_frame)
    pyr.close()


def test_describe_paths_first_frame(ctx, monkeypatch):
    """A multi-frame batch that starts at pyramid slot 2 of 5: the dense path smooths only frames 2..4 and reads
    frame f's plane for keypoint f * per_frame + k."""
    w, h = 640, 480
    nfr, first, per_frame = 5, 2, 600
    imgs = np.stack([synth.make_frame(100 + i, w, h) for i in range(nfr)])
    pyr = api.Pyramid(ctx, nfr, w, h, 0)
    pyr.build(imgs)
    rng = np.random.default_rng(11)
    pts = np.concatenate([_points(rng, w, h, per_frame) for _ in range(nfr - first)])
    out = _describe_all_modes(ctx, monkeypatch, pyr, pts, per_frame, first_frame=first)
    _check(out, imgs, pts, per_frame, first_frame=first)
    pyr.close()


@pytest.mark.parametrize("kind", ["constant", "binary"])
def test_describe_paths_ties_and_clamp(ctx, monkeypatch, kind):
    """A constant frame makes every comparison a tie (all bits 0); a 0/255 frame drives the smoothed values to both
    ends of the u8 range."""
    w, h = 320, 240
    rng = np.random.default_rng(17)
    if kind == "constant":
        im = np.full((h, w), 200, np.uint8)
    else:
        im = (rng.integers(0, 2, (h, w)) * 255).astype(np.uint8)
        im[:, : w // 3] = 255
        im[h // 2:, w // 2:] = 0
    pyr = api.Pyramid(ctx, 1, w, h, 0)
    pyr.build(im[None])
    per_frame = 500
    pts = _points(rng, w, h, per_frame)
    out = _describe_all_modes(ctx, monkeypatch, pyr, pts, per_frame)
    _check(out, im[None], pts, per_frame)
    if kind == "constant":
        assert not out["dense"][0].any()
    pyr.close()
