"""Multi-GPU localBA (SURVEY.md 8e): landmark partitioning + an in-kernel sum of the reduced camera
system over peer memory every LM iteration.

CPU: the partition is a partition.
GPU (one device): the ranks' shards run concurrently on contexts of one process and must reproduce
the unsharded solve; windows the exchange buffer cannot hold are refused before any launch."""
import threading

import numpy as np
import pytest

from ov2slam_b200 import api, synth


def test_partition_is_a_balanced_partition():
    pb = synth.make_ba_problem(7, 8, 500, 3000)
    for world in (2, 3, 8):
        shards = api.partition_ba_problem(pb, world)
        all_l = np.concatenate([s[1] for s in shards])
        all_o = np.concatenate([s[2] for s in shards])
        assert sorted(all_l.tolist()) == list(range(500)) and sorted(all_o.tolist()) == list(range(3000))
        loads = [len(s[2]) for s in shards]
        assert max(loads) - min(loads) <= 0.05 * 3000 / world + 8
        for sh, lms, obs in shards:
            assert (np.diff(sh["obs_lm"]) >= 0).all()                      # still CSR by landmark
            assert np.array_equal(lms[sh["obs_lm"]], pb["obs_lm"][obs])     # remap is consistent
            assert np.array_equal(sh["obs_px"], pb["obs_px"][obs])
            assert np.array_equal(sh["pose"], pb["pose"])


@pytest.mark.gpu
@pytest.mark.parametrize("world,empty", [(2, False), (3, False), (3, True)])
def test_p2p_sharded_solve_matches_unsharded(ctx, monkeypatch, world, empty):
    """(All ranks share ONE GPU here, so their persistent kernels must be co-resident: 24 CTAs each.)
    ov2_localba_solve_p2p: `world` ranks as contexts of ONE process on one GPU (communicators connected with direct
    pointers); every rank's persistent kernel sums the partial reduced systems out of the other ranks' exchange buffers.
    Must reproduce the unsharded solve; with `empty` the last rank owns no landmark at all (ADVICE r1: an empty shard
    used to fail with a zero-block launch and hang the others)."""
    monkeypatch.setenv("OV2_BA_CTAS", "24")
    pb = synth.make_ba_problem(31, 12, 1500, 9000)
    ref = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in pb.items()}
    rres, rflags = api.Optimizer(ctx).local_ba(ref)
    shards = api.partition_ba_problem(pb, world - 1 if empty else world)
    if empty:
        e = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in shards[0][0].items()}
        for k in ("lm_anchor_cam", "lm_anchor_px", "lm_invdepth", "obs_cam", "obs_lm", "obs_px"):
            e[k] = e[k][:0].copy()
        shards.append((e, np.zeros(0, np.int64), np.zeros(0, np.int64)))
    ctxs = [api.Context(0) for _ in range(world)]
    for c in ctxs:
        # every context allocates its arenas / pinned staging on its first solve; do that BEFORE the concurrent solves: a
        # cudaMalloc / cudaHostAlloc issued while another rank's kernel spins in a rank barrier on the SAME device can block
        # behind that kernel (ranks on different devices, the real configuration, do not share this hazard)
        api.Optimizer(c).local_ba({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in pb.items()})
    comms = [api.BaComm(ctxs[r], r, world) for r in range(world)]
    api.BaComm.connect_local(comms)
    for rep in range(2):                       # twice: epochs of consecutive launches must not collide
        work = [{k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in sh[0].items()} for sh in shards]
        results = [None] * world
        errs = []

        def run(rank):
            try:
                results[rank] = comms[rank].local_ba(work[rank])
            except Exception as ex:  # pragma: no cover
                errs.append((rank, ex))

        ths = [threading.Thread(target=run, args=(r,)) for r in range(world)]
        for t in ths:
            t.start()
        for t in ths:
            t.join(timeout=180)
        assert not errs, errs
        invd = np.zeros(len(pb["lm_invdepth"]))
        flags = np.zeros(len(pb["obs_cam"]), np.uint8)
        for r, (sh, lms, obs) in enumerate(shards):
            res, fl = results[r]
            assert (res["iters_robust"], res["iters_refine"]) == (rres["iters_robust"], rres["iters_refine"]), (r, res)
            assert abs(res["final_cost"] - rres["final_cost"]) <= 1e-9 * max(1.0, rres["final_cost"])
            assert np.abs(work[r]["pose"] - ref["pose"]).max() <= 1e-7
            assert np.array_equal(work[r]["pose"], work[0]["pose"])          # bit-identical decisions on every rank
            invd[lms] = work[r]["lm_invdepth"]
            flags[obs] = fl
        assert np.abs(invd - ref["lm_invdepth"]).max() <= 1e-7
        assert (flags != rflags).sum() <= 2
    for c in comms:
        c.close()
    for c in ctxs:
        c.close()


@pytest.mark.gpu
def test_p2p_refuses_windows_beyond_256_keyframes_before_launch(ctx):
    """The exchange buffer holds 256 keyframes: with world > 1 every rank must refuse a larger window on the host, so no rank
    launches a kernel that would wait in a rank barrier for a peer that never started."""
    pb = synth.make_ba_problem(84, 300, 1200, 2400, nconst=236)
    shards = api.partition_ba_problem(pb, 2)
    ctxs = [api.Context(0) for _ in range(2)]
    comms = [api.BaComm(ctxs[r], r, 2) for r in range(2)]
    api.BaComm.connect_local(comms)
    launches = [c.launch_count() for c in ctxs]
    errs = [None, None]

    def run(rank):
        try:
            comms[rank].local_ba(shards[rank][0])
        except api.Ov2Error as ex:
            errs[rank] = ex

    ths = [threading.Thread(target=run, args=(r,)) for r in range(2)]
    for t in ths:
        t.start()
    for t in ths:
        t.join(timeout=120)
    assert all(isinstance(e, api.Ov2Error) for e in errs), errs
    assert [c.launch_count() for c in ctxs] == launches
    for c in comms:
        c.close()
    for c in ctxs:
        c.close()
