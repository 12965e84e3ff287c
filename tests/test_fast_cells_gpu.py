"""The per-cell FAST candidate lists of stage F1 (ov2_debug_fast_cells) against oracle/image_ref.py::fast_detect_ref.

The grid tests only see one winner per cell; this pins every candidate: position, response and scan order, after the
CV_32F-mask byte filter (cell-local x % 4 in {2, 3}).  Cell sizes cover the default 50, odd interior widths (35, 65), the
32-thread CTA (8, 16) and both pair-row layouts of the kernel (<= 64 and above, up to 128); thresholds go down to 0, and a
high-contrast frame with 0 / 255 pixels drives scores to 255.  A dot lattice fills cells up to the capacity the hook
reports (ov2_fast_cell_capacity, checked against the bound derived here), and every list is compared whole.
"""
import numpy as np
import pytest

from ov2slam_b200 import api, synth
from oracle import image_ref as R
from test_frontend_gpu import unaligned_device_frames

pytestmark = pytest.mark.gpu

W, H = 640, 480
THRESHOLDS = (10, 6, 3, 1, 0)


def _frames():
    tex = synth.make_frame(30, W, H)
    hc = np.where(synth.make_frame(31, W, H) > 127, 255, 0).astype(np.uint8)
    rng = np.random.default_rng(31)
    salt = rng.random((H, W))
    hc[salt < 0.01] = 0
    hc[salt > 0.99] = 255
    lattice = np.full((H, W), 40, np.uint8)          # a candidate at every x = 2 (mod 4), even y: up to the full capacity
    lattice[0::2, 2::4] = 200
    return {"textured": tex, "high_contrast": hc, "lattice": lattice}


def _cap(cs):
    """One candidate per column group {4k + 2, 4k + 3} meeting the interior [3, cs - 3), every second interior row."""
    groups = len({x // 4 for x in range(3, cs - 3) if x % 4 in (2, 3)})
    return groups * ((cs - 6 + 1) // 2)


@pytest.mark.parametrize("staging", ["tma", "plain"])
@pytest.mark.parametrize("cs", [50, 35, 16, 8, 64, 65, 128])
def test_fast_cell_full_candidate_lists_match_oracle(ctx, cs, staging):
    """`plain`: the same frames through a device-aliased level 0 whose base the TMA rules reject (plain-load staging)."""
    nw, cap = W // cs, _cap(cs)
    top = 0
    for name, im in _frames().items():
        pyr = api.Pyramid(ctx, 1, W, H, 0)
        if staging == "plain":
            d, args = unaligned_device_frames(im[None])
            pyr.build(**args)
        else:
            pyr.build(im[None])
        fe = api.FeatureExtractor(ctx)
        for th in THRESHOLDS:
            cells = fe.debug_fast_cells(pyr, 0, cs, th)
            assert fe.last_fast_cell_cap == cap == fe.fast_cell_capacity(cs)
            assert len(cells) == (H // cs) * nw
            for ci, got in enumerate(cells):
                x, y = (ci % nw) * cs, (ci // nw) * cs
                if not (x + cs < W - 1 and y + cs < H - 1):
                    assert got == [], (name, th, ci)
                    continue
                ref = [k for k in R.fast_detect_ref(im[y:y + cs, x:x + cs], th) if k[0] % 4 in (2, 3)]
                assert len(ref) <= cap and got == ref, (name, th, ci, got[:6], ref[:6], len(got), len(ref))
                if got:
                    top = max(top, max(k[2] for k in got))
        pyr.close()
    assert top == 254.0            # response = score - 1: the 0 / 255 frame reaches the largest score
