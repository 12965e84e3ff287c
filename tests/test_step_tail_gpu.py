"""cornerSubPix (subpix_kernel) on the cases its staged patch branches on.

subpix_kernel stages the 10 x 10 pixels under the patch once per integer origin and re-interpolates from shared memory
while the origin stays; it goes pixel by pixel through getRectSubPix's border rules within 4 px of a border.  The cases:
points whose centre crosses an integer boundary between iterations (the block is staged again), points in every border
band and corner, points that walk more than 3 px (returned unrefined), empty slots, do_subpix = 0, and level 0 as an
odd-pitch, odd-address view of a device buffer.  Bars: bit-equal to tests/golden/step_tail_golden.npz, which holds what
the kernel returned before it staged anything (every iteration read its 81 x 4 pixels from global memory), and within
SUBPIX_TOL of the oracle.

`python tests/test_step_tail_gpu.py --write-golden [PATH]` writes the golden from the library as built.
"""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from ov2slam_b200 import api, synth  # noqa: E402
from oracle import image_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = ROOT / "tests" / "golden" / "step_tail_golden.npz"
SUBPIX_TOL = 1e-5 if R.HAVE_CV2 else 2e-4      # as tests/test_frontend_gpu.py
SP_W, SP_H = 323, 243                           # odd width: rows of a packed frame start at every byte alignment


# ---------------------------------------------------------------------------------------------------------- cornerSubPix
def _subpix_images():
    w, h = SP_W, SP_H
    tex = synth.make_frame(21, w, h)
    soft = (synth.make_frame(22, w, h, nrect=20) // 6 + 100).astype(np.uint8)     # weak gradients: long walks
    noise = np.random.default_rng(23).integers(0, 256, (h, w)).astype(np.uint8)
    return np.stack([tex, soft, noise])


def _subpix_points():
    """Integer points per frame (same slots for every frame): every border band and corner, a random interior set, and
    empty slots in between."""
    w, h = SP_W, SP_H
    pts = []
    for b in range(4):
        pts += [(b, y) for y in range(0, h, 7)] + [(w - 1 - b, y) for y in range(3, h, 7)]
        pts += [(x, b) for x in range(0, w, 7)] + [(x, h - 1 - b) for x in range(3, w, 7)]
    pts += [(x, y) for x in (0, 1, 2, 3, w - 4, w - 3, w - 2, w - 1) for y in (0, 1, 2, 3, h - 4, h - 3, h - 2, h - 1)]
    rng = np.random.default_rng(24)
    pts += [(int(x), int(y)) for x, y in zip(rng.integers(4, w - 4, 900), rng.integers(4, h - 4, 900))]
    p = np.array(pts, np.int32)
    p[rng.random(len(p)) < 0.05] = -1
    return p


def _run_subpix(ctx, imgs, ipts, view=False):
    """cornerSubPix alone on `ipts` in every frame: (refined (F, P, 2), iterations (F, P)).  view: level 0 aliases a device
    buffer at an odd address with a pitch of w + 5 bytes."""
    n, h, w = imgs.shape
    pyr = api.Pyramid(ctx, n, w, h, 0)
    if view:
        torch = pytest.importorskip("torch")
        pitch, fs = w + 5, (w + 5) * h + 3
        buf = torch.zeros(1 + n * fs, dtype=torch.uint8, device="cuda")
        for f in range(n):
            buf[1 + f * fs:1 + f * fs + pitch * h].view(h, pitch)[:, :w] = torch.from_numpy(imgs[f]).cuda()
        d0 = buf[1:]
        assert d0.data_ptr() % 2 == 1
        pyr.build(d0, count=n, row_stride=pitch, frame_stride=fs)
    else:
        pyr.build(imgs)
    allp = np.ascontiguousarray(np.broadcast_to(ipts, (n,) + ipts.shape)).reshape(-1, 2)
    out = np.empty(allp.shape, np.float32)
    its = np.empty(len(allp), np.int32)
    api.FeatureExtractor(ctx).debug_subpix_iters(pyr, 0, n, len(ipts), allp, out, its)
    pyr.close()
    return out.reshape(n, -1, 2), its.reshape(n, -1)


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("view", [False, True], ids=["owned", "unaligned-view"])
def test_subpix_bit_equal_to_unstaged_kernel(ctx, golden, view):
    imgs, ipts = _subpix_images(), _subpix_points()
    out, its = _run_subpix(ctx, imgs, ipts, view)
    assert np.array_equal(out.view(np.uint32), golden["subpix_out"].view(np.uint32)), int((out != golden["subpix_out"]).sum())
    assert np.array_equal(its, golden["subpix_iters"])
    live = ipts[:, 0] >= 0
    assert (out[:, ~live] == -1).all() and (its[:, ~live] == -1).all()
    assert its[:, live].min() >= 1 and its.max() == 30
    fp = ipts.astype(np.float32)[None]
    # the cases: the final centre's patch origin differs from the first one after at least three iterations (the block was
    # staged again and then reused), border bands, and walks of more than 3 px (returned unrefined)
    moved = (np.floor(out - 4) != fp - 4).any(axis=2) & live[None]
    assert (moved & (its >= 3)).sum() >= 50
    band = ((ipts[:, 0] < 4) | (ipts[:, 0] >= SP_W - 4) | (ipts[:, 1] < 4) | (ipts[:, 1] >= SP_H - 4)) & live
    assert band.sum() >= 400 and (its[:, band] >= 2).any()
    reverted = (out == fp).all(axis=2) & (its >= 2) & live[None]
    assert reverted.sum() >= 10


def test_subpix_against_oracle(ctx):
    imgs, ipts = _subpix_images(), _subpix_points()
    ipts = ipts[ipts[:, 0] >= 0]
    out, _ = _run_subpix(ctx, imgs, ipts)
    f = R.corner_subpix_cv2 if R.HAVE_CV2 else R.corner_subpix_ref
    for k in range(len(imgs)):
        p = ipts if R.HAVE_CV2 else ipts[::8]
        got = out[k] if R.HAVE_CV2 else out[k][::8]
        d = np.abs(got - f(imgs[k], p.astype(np.float32)))
        assert d.max() <= SUBPIX_TOL, (k, d.max(), p[d.max(axis=1).argmax()])


def test_no_subpix_returns_integer_points(ctx):
    imgs = _subpix_images()[:1]
    pyr = api.Pyramid(ctx, 1, SP_W, SP_H, 0)
    pyr.build(imgs)
    ncell = (SP_H // 20) * (SP_W // 20)
    res = {}
    for sub in (True, False):
        pts, ip, cnt = np.empty((ncell, 2), np.float32), np.empty((ncell, 2), np.int32), np.zeros(1, np.int32)
        api.FeatureExtractor(ctx).detect_grid_fast(pyr, 20, 0, 1, np.array([10], np.int32), pts, cnt, out_pts_int=ip, do_subpix=sub)
        res[sub] = (pts, ip, int(cnt[0]))
    pyr.close()
    pts, ip, n = res[False]
    assert n > 20 and np.array_equal(pts[:n], ip[:n].astype(np.float32)) and (pts[n:] == -1).all()
    assert np.array_equal(ip, res[True][1]) and not np.array_equal(pts, res[True][0])


def _write_golden(path):
    ctx = api.Context(0)
    out, its = _run_subpix(ctx, _subpix_images(), _subpix_points())
    ctx.close()
    np.savez_compressed(path, subpix_out=out, subpix_iters=its)
    print("wrote", path, out.shape, "mean iterations", its[its > 0].mean(), "max", its.max())


if __name__ == "__main__":
    if "--write-golden" in sys.argv:
        _write_golden(sys.argv[sys.argv.index("--write-golden") + 1] if len(sys.argv) > 2 else GOLDEN)
