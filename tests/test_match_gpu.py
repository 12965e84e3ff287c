"""8f-4: ov2_match_to_map (the data-parallel core of Mapper::matchToMap, mapper.cpp:576-774) against oracle/match_ref.py
through the C ABI."""
import numpy as np
import pytest

from ov2slam_b200 import api, synth
from oracle import match_ref as M

pytestmark = pytest.mark.gpu


def _compare(ctx, sc):
    """All four outputs identical: the oracle forms every double in the kernel's operation order."""
    rbk, rbd, rkm, rkd = M.match_to_map(sc)
    bk, bd, km, kd = api.match_to_map(ctx, sc)
    bad = np.nonzero(bk != rbk)[0]
    assert len(bad) == 0, (len(bad), bad[:10], bk[bad[:10]], rbk[bad[:10]])
    assert np.array_equal(bd, rbd)
    assert np.array_equal(km, rkm) and np.array_equal(kd, rkd)
    return (bk >= 0).sum(), (km >= 0).sum()


def test_hand_built_scene(ctx):
    from test_oracle_match import _tiny_scene
    sc = _tiny_scene()
    bk, bd, km, kd = api.match_to_map(ctx, sc)
    assert list(bk) == [0, 0] and list(bd) == [1.0, 2.0] and list(km) == [0, -1, -1] and kd[0] == 1.0 and kd[1] == 1024.0
    _compare(ctx, sc)


@pytest.mark.parametrize("seed,nkps,ncand,distorted", [(1, 800, 400, True), (2, 800, 400, False), (3, 300, 160, True), (4, 2000, 1600, True)])
def test_match_to_map_matches_oracle(ctx, seed, nkps, ncand, distorted):
    sc = synth.make_match_scene(seed, nkps, ncand, distorted=distorted)
    nmatch, nkp = _compare(ctx, sc)
    assert nmatch > 0.1 * ncand and nkp > 0


def test_empty_and_degenerate_inputs(ctx):
    sc = synth.make_match_scene(5, 200, 50)
    e = dict(sc)
    e["cand_mp"] = sc["cand_mp"][:0]
    bk, bd, km, kd = api.match_to_map(ctx, e)
    assert len(bk) == 0 and np.all(km == -1) and np.all(kd == 1024.0)
    far = dict(sc)
    far["dmaxpxdist"] = np.float32(0.0)        # nothing within zero pixels
    _compare(ctx, far)
