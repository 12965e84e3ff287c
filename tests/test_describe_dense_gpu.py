"""ORB-fallback descriptors on both of ov2_describe's paths: the per-window kernel (each keypoint smooths its own
26 x 26 window) and the dense one (each frame smoothed once, then gathered).  A ragged frame_idx call always takes the
per-window path; a fixed-stride call on the same points takes the path the density rule picks.  Every path must give
the oracle's bytes, and so the same bytes as each other."""
import numpy as np
import pytest

from ov2slam_b200 import api, synth
from oracle import image_ref as R

pytestmark = pytest.mark.gpu

KERNELS = {"per-window": {"describe_kernel"}, "dense": {"desc_smooth_kernel", "describe_dense_kernel"}}


def _rule(per_frame, w, h):
    """The density rule of frontend_desc.cu (use_dense) for a fixed-stride call."""
    dense = w >= 63 and h >= 63 and per_frame * 26.0 * 26.0 >= float(np.float32(1.4)) * (w - 36) * (h - 36)
    return "dense" if dense else "per-window"


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


def _describe_both_calls(ctx, pyr, pts, per_frame, first_frame=0):
    """{"per-window": the ragged call, "rule": the fixed-stride call}, each (desc, valid, kernels that ran)."""
    fe = api.FeatureExtractor(ctx)
    fidx = np.repeat(np.arange(first_frame, first_frame + len(pts) // per_frame, dtype=np.int32), per_frame)
    out = {}
    for name, kw in (("per-window", dict(frame_idx=fidx)), ("rule", dict(first_frame=first_frame, per_frame=per_frame))):
        desc = np.full((len(pts), 32), 0xA5, np.uint8)
        valid = np.full(len(pts), 7, np.uint8)
        ctx.profile(True)
        fe.describe_brief(pyr, pts, desc, valid, **kw)
        ran = {k for k in ctx.profile_report()}
        ctx.profile(False)
        out[name] = (desc, valid, ran)
    assert out["per-window"][2] == KERNELS["per-window"], out["per-window"][2]
    w, h = pyr.w, pyr.h
    assert out["rule"][2] == KERNELS[_rule(per_frame, w, h)], (per_frame, w, h, out["rule"][2])
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
def test_describe_calls_bit_exact(ctx, w, h, per_frame):
    """The rule sends 1300 per frame to the dense path at every size but 1280 x 720, and 40 per frame to the per-window
    path at every size but 63 x 63."""
    nfr = 2
    imgs = np.stack([synth.make_frame(70 + i, w, h) for i in range(nfr)])
    imgs[1] = np.random.default_rng(w + h).integers(0, 256, (h, w)).astype(np.uint8)   # raw noise
    pyr = api.Pyramid(ctx, nfr, w, h, 0)
    pyr.build(imgs)
    rng = np.random.default_rng(per_frame * 7 + w)
    pts = np.concatenate([_points(rng, w, h, per_frame) for _ in range(nfr)])
    out = _describe_both_calls(ctx, pyr, pts, per_frame)
    _check(out, imgs, pts, per_frame)
    pyr.close()


def test_describe_rule_takes_each_side_of_crossover(ctx):
    """At C2's geometry the rule takes the dense path for a dense set (1024 per frame) and the per-window path for
    a sparse one (108 per frame, the new keypoints of 40 px cells)."""
    w, h = 640, 480
    imgs = synth.make_frame(90, w, h)[None]
    pyr = api.Pyramid(ctx, 1, w, h, 0)
    pyr.build(imgs)
    rng = np.random.default_rng(3)
    for per_frame, want in ((1024, "dense"), (108, "per-window")):
        pts = _points(rng, w, h, per_frame)
        out = _describe_both_calls(ctx, pyr, pts, per_frame)
        assert out["rule"][2] == KERNELS[want], (per_frame, out["rule"][2])
        _check(out, imgs, pts, per_frame)
    pyr.close()


def test_describe_calls_first_frame(ctx):
    """A multi-frame batch that starts at pyramid slot 2 of 5: the dense path smooths only frames 2..4 and reads
    frame f's plane for keypoint f * per_frame + k."""
    w, h = 640, 480
    nfr, first, per_frame = 5, 2, 600
    assert _rule(per_frame, w, h) == "dense"
    imgs = np.stack([synth.make_frame(100 + i, w, h) for i in range(nfr)])
    pyr = api.Pyramid(ctx, nfr, w, h, 0)
    pyr.build(imgs)
    rng = np.random.default_rng(11)
    pts = np.concatenate([_points(rng, w, h, per_frame) for _ in range(nfr - first)])
    out = _describe_both_calls(ctx, pyr, pts, per_frame, first_frame=first)
    _check(out, imgs, pts, per_frame, first_frame=first)
    pyr.close()


@pytest.mark.parametrize("kind", ["constant", "binary"])
def test_describe_calls_ties_and_clamp(ctx, kind):
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
    assert _rule(per_frame, w, h) == "dense"
    pts = _points(rng, w, h, per_frame)
    out = _describe_both_calls(ctx, pyr, pts, per_frame)
    _check(out, im[None], pts, per_frame)
    if kind == "constant":
        assert not out["rule"][0].any()
    pyr.close()
