"""MapManager::stereoMatching on a C4-shaped stereo stage, on one GPU: ov2_stereo_matching against the flow keyframe by keyframe.

    python scripts/bench_stereo_matching.py [--keyframes 132] [--steps 10] [--warmup 2] [--cv2-keyframes 8]

132 stereo keyframes of 1280 x 720 (the C4 leg of bench_legs.py: 400 tracked keypoints, 60 % of them 3-D, and up to 720
new ones per keyframe, so 1 120 keypoints), accurate/ parameters (window 9, nklt_pyr_lvl 3), built by
synth.make_stereo_matching_scene (8 distinct keyframes tiled over the batch), for a rectified rig and for another rig.
Three paths, each reported as ms per keyframe:

  device_ms   one ov2_stereo_matching call over all keyframes, every array on the device: the median of `steps` calls,
              each timed by the host clock from its start to the end of a stream synchronisation
  binding_ms  the flow through the Python binding, keyframe by keyframe: the projected priors on the host (numpy), the
              row search (rectified rig) and the two tracker calls on host arrays, each waiting for its result, the retry
              lists and the epipolar gate on the host.  The neighbour-depth prior of the other rig is not computed here
              (those keypoints start blind), so that path does less host work than the reference
  cv2_ms      the two tracker passes of the same lists with cv2.calcOpticalFlowPyrLK on the host cores (no row search,
              no gate), over the first `cv2-keyframes` keyframes

and the card name, power limit and SM clock read in the same run, then one JSON line.  Writes nothing."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

W, H, NKPS, FRAC3D, WIN, LVL = 1280, 720, 1120, 0.6 * 400 / 1120, 9, 3


def tiled_scene(nkf, rect, distinct=8):
    from ov2slam_b200 import synth
    src = synth.make_stereo_matching_scene(2026 + rect, [NKPS] * distinct, W, H, rectified=bool(rect), frac3d=FRAC3D)
    pick = np.arange(nkf) % distinct
    sc = dict(src, lefts=src["lefts"][pick], rights=src["rights"][pick], offsets=(np.arange(nkf + 1) * NKPS).astype(np.int32),
              cell_offsets=(np.arange(nkf + 1) * src["cell_offsets"][1]).astype(np.int32))
    for k in ("Tcw", "K", "Trl", "Frl", "img_wh", "grid"):
        sc[k] = np.ascontiguousarray(src[k][pick])
    for k in ("px", "unpx", "bv", "is3d", "has_mp", "wpt"):
        sc[k] = np.ascontiguousarray(np.concatenate([src[k][p * NKPS:(p + 1) * NKPS] for p in pick]))
    ncell = int(src["cell_offsets"][1])
    ptr = [src["cell_ptr"][p * ncell:(p + 1) * ncell] - p * NKPS + f * NKPS for f, p in enumerate(pick)]
    sc["cell_ptr"] = np.concatenate(ptr + [[nkf * NKPS]]).astype(np.int32)
    sc["cell_kps"] = np.concatenate([src["cell_kps"][p * NKPS:(p + 1) * NKPS] - p * NKPS + f * NKPS
                                     for f, p in enumerate(pick)]).astype(np.int32)
    return sc


def host_priors(sc, f):
    """The projected 3-D priors of keyframe f (vectorised numpy): members of pass 1 and their priors."""
    sl = slice(sc["offsets"][f], sc["offsets"][f + 1])
    T, Tr, K = sc["Tcw"][f], sc["Trl"][f], sc["K"][f]
    c = sc["wpt"][sl] @ T[:9].reshape(3, 3).T + T[9:]
    c = c @ Tr[:9].reshape(3, 3).T + Tr[9:]
    with np.errstate(all="ignore"):
        x = (K[0] * c[:, 0] / c[:, 2] + K[2]).astype(np.float32)
        y = (K[1] * c[:, 1] / c[:, 2] + K[3]).astype(np.float32)
    ok = sc["is3d"][sl].astype(bool) & sc["has_mp"][sl].astype(bool) & (x >= 0) & (y >= 0) & (x < W) & (y < H)
    return ok, np.stack([x, y], 1)


def binding_flow(ctx, ft, lp, rp, sc, f, rect):
    sl = slice(sc["offsets"][f], sc["offsets"][f + 1])
    px, unpx = sc["px"][sl], sc["unpx"][sl]
    guided, pri = host_priors(sc, f)
    keep = ~(sc["is3d"][sl].astype(bool) & ~sc["has_mp"][sl].astype(bool))
    blind = keep & ~guided
    bpri = px[blind].copy()
    if rect and blind.any():
        sp = np.ascontiguousarray(bpri * np.float32(0.125))
        col, err = np.zeros(len(sp), np.float32), np.zeros(len(sp), np.float32)
        ft.line_min_sad(lp, rp, LVL, sp, 7, True, col, err, per_frame=len(sp), first_frame=f)
        x = col * np.float32(8)
        ok = (x >= 0) & (x <= bpri[:, 0])
        bpri[ok, 0] = x[ok]
    g_px, g_pri = np.ascontiguousarray(px[guided]), np.ascontiguousarray(pri[guided])
    st1 = np.zeros(len(g_px), np.uint8)
    if len(g_px):
        ft.fb_klt_tracking(lp, rp, WIN, 1, 30.0, 0.5, g_px, g_pri, st1, per_frame=len(g_px), first_frame=f)
    failed = st1 == 0
    p2 = np.ascontiguousarray(np.concatenate([px[blind], g_px[failed]]))
    r2 = np.ascontiguousarray(np.concatenate([bpri, g_pri[failed]]))
    st2 = np.zeros(len(p2), np.uint8)
    if len(p2):
        ft.fb_klt_tracking(lp, rp, WIN, LVL, 30.0, 0.5, p2, r2, st2, per_frame=len(p2), first_frame=f)
    lun = np.concatenate([unpx[guided][~failed], unpx[blind], unpx[guided][failed]])[np.concatenate([st1[~failed], st2]) > 0]
    run = np.concatenate([g_pri[~failed], r2])[np.concatenate([st1[~failed], st2]) > 0]
    if rect:
        return int((np.abs(lun[:, 1] - run[:, 1]) <= 2).sum())
    F = sc["Frl"][f].reshape(3, 3)
    lh, rh = np.c_[lun, np.ones(len(lun))], np.c_[run, np.ones(len(run))]
    Fl, Ftr = lh @ F.T, rh @ F
    e = np.sqrt(np.einsum("ij,ij->i", rh, Fl) ** 2 / (Ftr[:, 0] ** 2 + Ftr[:, 1] ** 2 + Fl[:, 0] ** 2 + Fl[:, 1] ** 2))
    return int((e <= 2).sum())


def cv2_flow(sc, f):
    from oracle import image_ref as R
    sl = slice(sc["offsets"][f], sc["offsets"][f + 1])
    px = sc["px"][sl]
    guided, pri = host_priors(sc, f)
    keep = ~(sc["is3d"][sl].astype(bool) & ~sc["has_mp"][sl].astype(bool))
    tr1, st1 = R.fb_klt_cv2(sc["lefts"][f], sc["rights"][f], px[guided], pri[guided], WIN, 1)
    p2 = np.concatenate([px[keep & ~guided], px[guided][st1 == 0]])
    r2 = np.concatenate([px[keep & ~guided], tr1[st1 == 0]])
    R.fb_klt_cv2(sc["lefts"][f], sc["rights"][f], p2, r2, WIN, LVL)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, default=132)
    ap.add_argument("--steps", type=int, default=10, help="timed calls of the device path")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cv2-keyframes", type=int, default=8)
    args = ap.parse_args()
    import torch
    from ov2slam_b200 import api
    if not torch.cuda.is_available():
        raise SystemExit("bench_stereo_matching.py: no CUDA device; there is no CPU fallback")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    ctx = api.Context(0)
    ft = api.FeatureTracker(ctx, 30, 0.01)
    nkf = args.keyframes
    res = dict(metric="stereo_matching_ms_per_keyframe", keyframes=nkf, keypoints_per_keyframe=NKPS, size=[W, H],
               gpu=smi[0] if smi else "unknown")
    for rect in (1, 0):
        sc = tiled_scene(nkf, rect)
        lp, rp = api.Pyramid(ctx, nkf, W, H, 3), api.Pyramid(ctx, nkf, W, H, 3)
        lp.build(sc["lefts"])
        rp.build(sc["rights"])
        names = ("Tcw", "K", "Trl", "Frl", "img_wh", "grid", "cell_ptr", "cell_kps", "px", "unpx", "bv", "is3d", "has_mp", "wpt")
        d = {k: torch.from_numpy(np.ascontiguousarray(sc[k])).cuda() for k in names}
        n = len(sc["px"])
        out = dict(right=torch.empty((n, 2), device="cuda"), stereo=torch.empty(n, dtype=torch.uint8, device="cuda"),
                   passes=torch.empty(n, dtype=torch.uint8, device="cuda"), nstereo=torch.empty(nkf, dtype=torch.int32, device="cuda"))

        def device():
            ft.stereo_matching(lp, rp, WIN, LVL, 30.0, 0.5, rect, sc["offsets"], d["Tcw"], d["K"], d["Trl"], d["img_wh"], d["px"],
                               d["unpx"], d["bv"], d["is3d"], d["has_mp"], d["wpt"], Frl=d["Frl"], cell_offsets=sc["cell_offsets"],
                               grid=d["grid"], cell_ptr=d["cell_ptr"], cell_kps=d["cell_kps"], out=out)
            ctx.sync()
        times = []
        for s in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            device()
            if s >= args.warmup:
                times.append(time.perf_counter() - t0)
        tag = "rect" if rect else "other"
        res[f"{tag}_device_ms"] = 1e3 * float(np.median(times)) / nkf
        res[f"{tag}_device_stereo"] = int(out["nstereo"].sum().item())
        for f in range(min(nkf, 2)):
            binding_flow(ctx, ft, lp, rp, sc, f, rect)                    # warm-up of the per-keyframe shapes
        t0 = time.perf_counter()
        nst = sum(binding_flow(ctx, ft, lp, rp, sc, f, rect) for f in range(nkf))
        res[f"{tag}_binding_ms"] = 1e3 * (time.perf_counter() - t0) / nkf
        res[f"{tag}_binding_stereo"] = nst
        ncv = min(nkf, args.cv2_keyframes)
        t0 = time.perf_counter()
        for f in range(ncv):
            cv2_flow(sc, f)
        res[f"{tag}_cv2_ms"] = 1e3 * (time.perf_counter() - t0) / max(ncv, 1)
    for line in smi:
        print("#", line)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
