"""The hand-placed matchToMap scenes of tests/match_scenes.py sit where they claim to: the oracle (oracle/match_ref.py)
sees each threshold exactly on its edge, each projection on its pixel, each case decided the way it was built.  The GPU
tests (tests/test_match_paths_gpu.py) compare the kernel with the oracle on the same scenes."""
import numpy as np
import pytest

import match_scenes as S
from oracle import match_ref as M

f32 = np.float32


@pytest.mark.parametrize("kind", S.THRESHOLDS)
@pytest.mark.parametrize("on_edge", [True, False])
def test_threshold_scenes_sit_on_the_edge(kind, on_edge):
    sc, at_edge, kept = S.threshold_scene(kind, on_edge)
    assert at_edge
    bk, bd, km, kd = M.match_to_map(sc)
    assert (bk[0] == 0) == kept and (bk[0] == -1) == (not kept)
    if kind == "no_descriptor" and kept:
        assert bd[0] == 1000.0 and km[0] == 0 and kd[0] == 1000.0


@pytest.mark.parametrize("case", sorted(S.LANE_CASES))
def test_lane_scenes(case):
    counts, dists, best = S.LANE_CASES[case]
    sc, ids = S.lane_scene(counts, dists)
    bk, _, _, _ = M.match_to_map(sc)
    assert bk[0] == (ids[best] if best is not None else -1)
    # the four cells hold the keypoints in the order they were added
    r0, c0, nbw = 3, 4, sc["nbwcells"]
    for i, (dr, dc) in enumerate(S.CORNER):
        cell = (r0 + dr) * nbw + c0 + dc
        assert list(sc["cell_kp"][sc["cell_ptr"][cell]:sc["cell_ptr"][cell + 1]]) == [ids[(i, q)] for q in range(counts[i])]


@pytest.mark.parametrize("nkfs", [64, 65, 128, 256])
def test_mask_scenes(nkfs):
    sc, disjoint = S.mask_scene(nkfs)
    bk, _, _, _ = M.match_to_map(sc)
    assert list(bk >= 0) == disjoint and not all(disjoint) and any(disjoint)
    words = (nkfs + 63) // 64
    assert np.all(sc["mp_kfmask"][:, words:] == 0) and np.all(sc["mp_kfmask"][:, :words].any(axis=0))


@pytest.mark.parametrize("distorted", [False, True])
@pytest.mark.parametrize("cs", [35, 45, 50])
@pytest.mark.parametrize("geom", sorted(S.GEOMETRIES))
def test_grid_edge_scenes(geom, cs, distorted):
    sc, placed = S.grid_edge_scene(geom, cs, distorted)
    bk, _, _, _ = M.match_to_map(sc)
    first_kp = [int(np.nonzero(sc["kp_lm"] == sc["cand_mp"][c] + 1)[0][0]) for c in range(len(placed))]
    for c, ((u, v), p, inside) in enumerate(placed):
        for t, q in ((u, p[0]), (v, p[1])):
            if not distorted and t != 0:
                assert q == t, (c, (u, v), p)               # a pinhole projection lands on the pixel itself
            else:
                assert abs(float(q) - float(t)) <= 2e-4, (c, (u, v), p)
        assert bk[c] == (first_kp[c] if inside else -1), (c, (u, v), p)
    w, h = sc["img_w"], sc["img_h"]
    assert sum(inside for _, _, inside in placed) >= 11
    if not distorted:
        assert sum(p[0] == 0 or p[1] == 0 for _, p, _ in placed) >= 2
        assert any(p[0] == np.nextafter(f32(w), f32(0)) for _, p, inside in placed if inside)
        assert any(p[0] == w for _, p, inside in placed if not inside)


def test_descriptor_set_scene():
    sc, want = S.descriptor_set_scene()
    bk, bd, _, _ = M.match_to_map(sc)
    assert np.all(bk == np.arange(len(want))) and list(bd) == want
    assert set(np.diff(sc["mp_desc_ptr"])) == {1, 7, 16}


def test_keypoint_pass_scene():
    sc, kp_of = S.keypoint_pass_scene()
    bk, bd, km, kd = M.match_to_map(sc)
    assert list(bk) == kp_of
    last = lambda k: max(c for c, j in enumerate(kp_of) if j == k)
    assert km[0] == last(0) and kd[0] == 9.0
    assert kd[1] == 4.0 and bd[km[1]] == 4.0 and km[1] != last(1)
    assert km[2] == last(2) and kd[2] == 1000.0
