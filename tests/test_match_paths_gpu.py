"""ov2_match_to_map (csrc/match_map.cu) against oracle/match_ref.py on hand-placed scenes (tests/match_scenes.py): cells that
take several rounds of 32 lanes, keyframe sets in every word of the 256-bit mask, every threshold on and one step past its
edge, the grid and image edges of the shipped geometries, descriptor sets up to 16 x 16 pairs, the per-keypoint pass under
many candidates, a grid-stride-sized scene and empty sides.  Every comparison is exact on all four outputs."""
import numpy as np
import pytest

import match_scenes as S
from oracle import match_ref as M
from ov2slam_b200 import api, synth

pytestmark = pytest.mark.gpu


def _same(ctx, sc):
    want = M.match_to_map(sc)
    got = api.match_to_map(ctx, sc)
    for name, g, w in zip(("best_kp", "best_dist", "kp_match", "kp_dist"), got, want):
        assert g.dtype == w.dtype and np.array_equal(g, w), (name, np.nonzero(g != w)[0][:10], g[g != w][:10], w[g != w][:10])
    return want


@pytest.mark.parametrize("case", sorted(S.LANE_CASES))
def test_lane_rounds(ctx, case):
    counts, dists, best = S.LANE_CASES[case]
    sc, ids = S.lane_scene(counts, dists)
    bk, _, _, _ = _same(ctx, sc)
    assert bk[0] == (ids[best] if best is not None else -1)


@pytest.mark.parametrize("nkfs", [64, 65, 128, 256])
def test_keyframe_masks(ctx, nkfs):
    sc, disjoint = S.mask_scene(nkfs)
    bk, _, _, _ = _same(ctx, sc)
    assert list(bk >= 0) == disjoint


def test_more_than_256_keyframes_is_refused_and_the_context_stays_usable(ctx):
    sc, _ = S.mask_scene(256)
    big = dict(sc, kf_Tcw=np.tile(S.IDENTITY, (257, 1)))
    with pytest.raises(api.Ov2Error, match="INVALID"):
        api.match_to_map(ctx, big)
    _same(ctx, sc)


@pytest.mark.parametrize("on_edge", [True, False])
@pytest.mark.parametrize("kind", S.THRESHOLDS)
def test_thresholds(ctx, kind, on_edge):
    sc, at_edge, kept = S.threshold_scene(kind, on_edge)
    assert at_edge
    bk, _, _, _ = _same(ctx, sc)
    assert (bk[0] >= 0) == kept


@pytest.mark.parametrize("distorted", [False, True])
@pytest.mark.parametrize("cs", [35, 45, 50])
@pytest.mark.parametrize("geom", sorted(S.GEOMETRIES))
def test_grid_and_image_edges(ctx, geom, cs, distorted):
    sc, placed = S.grid_edge_scene(geom, cs, distorted)
    bk, _, _, _ = _same(ctx, sc)
    assert list(bk >= 0) == [inside for _, _, inside in placed]


def test_descriptor_sets(ctx):
    sc, want = S.descriptor_set_scene()
    _, bd, _, _ = _same(ctx, sc)
    assert list(bd) == want


def test_keypoint_pass_under_many_candidates(ctx):
    sc, kp_of = S.keypoint_pass_scene()
    bk, _, km, kd = _same(ctx, sc)
    assert list(bk) == kp_of and list(kd) == [9.0, 4.0, 1000.0]


def test_grid_stride_sized_scene(ctx):
    sc = synth.make_match_scene(21, nkps=5000, ncand=20000, distorted=True)
    bk, _, km, _ = _same(ctx, sc)
    assert (bk >= 0).sum() > 2000 and (km >= 0).sum() > 1000


def test_empty_sides_and_depth_culls(ctx):
    sc = synth.make_match_scene(22, nkps=300, ncand=120)
    no_cand = dict(sc, cand_mp=sc["cand_mp"][:0])
    bk, bd, km, kd = _same(ctx, no_cand)
    assert len(bk) == 0 and np.all(km == -1) and np.all(kd == 1024.0)
    nbc = len(sc["cell_ptr"]) - 1
    no_kps = dict(sc, kp_px=np.zeros((0, 2), np.float32), kp_lm=np.zeros(0, np.int32), cell_kp=np.zeros(0, np.int32),
                  cell_ptr=np.zeros(nbc + 1, np.int32))
    bk, _, km, _ = _same(ctx, no_kps)
    assert np.all(bk == -1) and len(km) == 0
    both = dict(no_kps, cand_mp=sc["cand_mp"][:0])
    bk, _, km, _ = _same(ctx, both)
    assert len(bk) == 0 and len(km) == 0
    # candidates behind the camera and at depth exactly 0, next to ones that match
    s = S.Scene()
    for i, z in enumerate((2.0, 0.0, -2.0, 2.0, -0.0)):
        D = s.random_desc()
        xyz = s.point_at(100.5 + 80 * i, 200.5, z=2.0)
        s.keypoint(s.project(xyz), s.map_point(xyz, [S.flip(D, 3)]))
        xyz[2] = z
        s.candidate(s.map_point(xyz, [D]))
    bk, _, _, _ = _same(ctx, s.scene())
    assert list(bk) == [0, -1, -1, 3, -1]
