"""ov2_remap / ov2_pyr_build_remap (csrc/frontend_remap.cu) on the GPU against oracle/remap_ref.py: bit-exact, both map types,
host and device buffers, batched frames with strides, in place; the pyramid built through a map and CLAHE on it."""
import numpy as np
import pytest

from oracle import image_ref as R
from oracle import remap_ref as RR
from ov2slam_b200 import api

pytestmark = pytest.mark.gpu


def _imgs(n, w, h, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    out = []
    for k in range(n):
        smooth = 128 + 70 * np.sin(xx / (5.0 + k) + k) * np.cos(yy / 9.0)
        out.append(np.clip(smooth + rng.normal(0, 20, (h, w)), 0, 255).astype(np.uint8))
    return np.stack(out)


def _maps(w, h):
    """(fixed CV_16SC2 + CV_16UC1, float CV_32FC1) of a numpy radial map plus the edge entries of the oracle test."""
    mx, my = RR.radial_map_np(w, h, shift=(3.25, -2.5))
    ex, ey = RR.edge_maps(w, h, seed=w)
    sel = np.random.default_rng(1).random((h, w)) < 0.05
    mx, my = np.where(sel, ex, mx).astype(np.float32), np.where(sel, ey, my).astype(np.float32)
    return RR.fixed_from_float(mx, my), (mx, my)


@pytest.mark.parametrize("size", [(752, 480), (333, 217)])
@pytest.mark.parametrize("kind", ["fixed", "float"])
def test_remap_host_buffers_equal_the_oracle(ctx, size, kind):
    w, h = size
    m16, f32 = _maps(w, h)
    m = m16 if kind == "fixed" else f32
    rm = api.RemapMap(ctx, *m)
    imgs = _imgs(3, w, h, 5)
    want = np.stack([RR.remap_ref(im, *m) for im in imgs])
    out = np.zeros_like(imgs)
    api.remap(ctx, rm, imgs, out)
    assert np.array_equal(out, want)
    one = np.zeros((h, w), np.uint8)
    api.remap(ctx, rm, imgs[1], one)
    assert np.array_equal(one, want[1])
    inplace = imgs.copy()
    api.remap(ctx, rm, inplace, inplace)                       # rectifyImage(im0, im0)
    assert np.array_equal(inplace, want)
    # strided frames: rows of pitch w + 9 inside frames of h + 3 rows, destination with its own pitch; the gaps stay untouched
    sp, dp = w + 9, w + 20
    src = np.full((3, h + 3, sp), 77, np.uint8)
    src[:, :h, :w] = imgs
    dst = np.full((3, h + 1, dp), 5, np.uint8)
    api.remap(ctx, rm, src, dst, count=3, src_row_stride=sp, src_frame_stride=sp * (h + 3), dst_row_stride=dp,
              dst_frame_stride=dp * (h + 1))
    assert np.array_equal(dst[:, :h, :w], want)
    assert (dst[:, :h, w:] == 5).all() and (dst[:, h:, :] == 5).all()
    rm.close()


@pytest.mark.parametrize("kind", ["fixed", "float"])
def test_remap_device_buffers_and_device_maps(ctx, kind):
    torch = pytest.importorskip("torch")
    w, h = 752, 480
    m16, f32 = _maps(w, h)
    m = m16 if kind == "fixed" else f32
    d1, d2 = torch.from_numpy(m[0]).cuda(), torch.from_numpy(m[1]).cuda()
    torch.cuda.synchronize()
    rm = api.RemapMap(ctx, d1, d2)                                                            # maps on the device
    imgs = _imgs(5, w, h, 8)
    want = np.stack([RR.remap_ref(im, *m) for im in imgs])
    src = torch.from_numpy(imgs).cuda()
    dst = torch.zeros_like(src)
    torch.cuda.synchronize()                                   # torch's copies run on its own stream
    api.remap(ctx, rm, src, dst)
    ctx.sync()
    assert np.array_equal(dst.cpu().numpy(), want)
    # device source, host destination and the reverse
    out = np.zeros_like(imgs)
    api.remap(ctx, rm, src, out)
    assert np.array_equal(out, want)
    dst.zero_()
    torch.cuda.synchronize()
    api.remap(ctx, rm, imgs, dst)
    ctx.sync()
    assert np.array_equal(dst.cpu().numpy(), want)
    rm.close()


def test_remap_rejects_images_above_2046_px(ctx):
    w, h = 2047, 16
    mx, my = np.zeros((h, w), np.float32), np.zeros((h, w), np.float32)
    with pytest.raises(api.Ov2Error, match="CAPACITY"):
        api.RemapMap(ctx, mx, my)


@pytest.mark.parametrize("device_images", [False, True])
def test_pyramid_built_through_a_map_equals_the_oracle(ctx, device_images):
    """Every level of ov2_pyr_build_remap equals build_pyramid_ref(remap_ref(img)); CLAHE through ov2_preprocess on that pyramid
    equals clahe_ref of the rectified image (and the pyramid over it build_pyramid_ref of that)."""
    w, h = 752, 480
    m16, _ = _maps(w, h)
    rm = api.RemapMap(ctx, *m16)
    imgs = _imgs(3, w, h, 21)
    rect = [RR.remap_ref(im, *m16) for im in imgs]
    pyr = api.Pyramid(ctx, 4, w, h, 3)
    if device_images:
        torch = pytest.importorskip("torch")
        dimgs = torch.from_numpy(imgs).cuda()
        torch.cuda.synchronize()
        pyr.build_remap(rm, dimgs, first=1)
        ctx.sync()
    else:
        pyr.build_remap(rm, imgs, first=1)
    for k in range(3):
        for lvl, ref in enumerate(R.build_pyramid_ref(rect[k], 3)):
            assert np.array_equal(pyr.download(1 + k, lvl), ref), (k, lvl)
    eq = api.Pyramid(ctx, 4, w, h, 3)
    api.preprocess(ctx, pyr, eq, first=1, count=3)
    for k in range(3):
        cl = R.clahe_ref(rect[k])
        for lvl, ref in enumerate(R.build_pyramid_ref(cl, 3)):
            assert np.array_equal(eq.download(1 + k, lvl), ref), (k, lvl)
    eq.close()
    pyr.close()
    rm.close()
