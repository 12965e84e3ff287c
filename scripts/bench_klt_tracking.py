"""VisualFrontEnd::kltTracking on the C2 tracking shapes, on one GPU: ov2_klt_tracking against today's batched path.

    python scripts/bench_klt_tracking.py [--batch 256] [--steps 20] [--warmup 3]

256 pairs of 640 x 480 frames, 1 024 keypoints per frame, 60 % of them 3-D with map points that project near the true
flow, a fifth of those 12 - 30 px off, so that pass 1 fails on some and pass 2 retries them (synth.make_klt_tracking_scene;
16 distinct image pairs, tiled over the batch).  Every array lives on the device.  Reports:

  klt_tracking_ms   ms per ov2_klt_tracking call over the whole batch: the median of `steps` calls, each timed by the host clock
                    from its start to the end of a stream synchronisation (both paths are timed the same way)
  fb_klt_ms         the same keypoints through one ov2_fb_klt with per-keypoint depth (1 for a 3-D keypoint with an
                    in-image prior, starting from it; nklt_pyr_lvl for the rest), the path without the retry
  tracked / tracked_fb_klt   keypoints with status 1 on each path
  retry_gained      failed pass-1 tracks that pass 2 recovers
  p3p_frames        share of frames with p3p_req

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256, help="frame pairs per call")
    ap.add_argument("--kps", type=int, default=1024, help="keypoints per frame")
    ap.add_argument("--steps", type=int, default=20, help="timed calls per path")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    from ov2slam_b200 import api, synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_klt_tracking.py: no CUDA device; there is no CPU fallback")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    w, h, nf = 640, 480, args.batch
    pairs = synth.make_batch(2024, 16, w, h)
    tile = lambda a: np.ascontiguousarray(np.resize(a, (nf,) + a.shape[1:]))
    sc = synth.make_klt_tracking_scene(2024, [args.kps] * nf, w, h, images=tuple(tile(a) for a in pairs))
    n = len(sc["px"])

    ctx = api.Context(0)
    pp, cp = api.Pyramid(ctx, nf, w, h, 3), api.Pyramid(ctx, nf, w, h, 3)
    pp.build(sc["prevs"])
    cp.build(sc["curs"])
    dev = {k: torch.from_numpy(np.ascontiguousarray(sc[k])).cuda() for k in ("Tcw", "K", "img_wh", "px", "wpt", "is3d")}
    out = dict(tracked=torch.zeros((n, 2), device="cuda"), status=torch.zeros(n, dtype=torch.uint8, device="cuda"),
               passes=torch.zeros(n, dtype=torch.uint8, device="cuda"), p3p_req=torch.zeros(nf, dtype=torch.uint8, device="cuda"),
               nbgood=torch.zeros(nf, dtype=torch.int32, device="cuda"), nbkps=torch.zeros(nf, dtype=torch.int32, device="cuda"))
    ft = api.FeatureTracker(ctx, 30, 0.01)
    torch.cuda.synchronize()

    def tracking():
        ft.klt_tracking(pp, cp, 9, 3, 30.0, 0.5, sc["offsets"], dev["Tcw"], dev["K"], dev["img_wh"], dev["px"], dev["wpt"],
                        dev["is3d"], out=out)

    # today's batched path: pass-1 members (read from one ov2_klt_tracking run) at depth 1 from their prior, the rest at 3
    tracking()
    ctx.sync()
    passes = out["passes"].cpu().numpy()
    status = out["status"].cpu().numpy()
    member1 = np.zeros(n, bool)
    from oracle import klt_tracking_ref as KT   # noqa: E402  (the projection only; numpy)
    pri0 = sc["px"].copy()
    for f in range(nf):
        for i in range(sc["offsets"][f], sc["offsets"][f + 1]):
            if sc["is3d"][i]:
                x, y, inside = KT.prior(sc["Tcw"][f], sc["K"][f], None, w, h, sc["wpt"][i])
                if inside:
                    member1[i] = True
                    pri0[i] = (x, y)
    lv = torch.from_numpy(np.where(member1, 1, 3).astype(np.uint8)).cuda()
    d_pri0 = torch.from_numpy(pri0).cuda()
    d_pri = d_pri0.clone()
    d_st = torch.zeros(n, dtype=torch.uint8, device="cuda")
    fidx = torch.from_numpy(np.repeat(np.arange(nf, dtype=np.int32), args.kps)).cuda()
    torch.cuda.synchronize()

    def fb_klt():
        ft.fb_klt_tracking(pp, cp, 9, lv, 30.0, 0.5, dev["px"], d_pri, d_st, n=n, frame_idx=fidx)

    def reset_priors():
        d_pri.copy_(d_pri0)     # the tracker writes its priors in place: every timed call starts from the same ones

    def timed(fn, reset=lambda: None):
        for _ in range(args.warmup):
            reset()
            fn()
        ctx.sync()
        ts = []
        for _ in range(args.steps):
            reset()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            ctx.sync()
            ts.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(ts)), float(min(ts)), float(max(ts))

    kt = timed(tracking)
    fb = timed(fb_klt, reset_priors)
    st_fb = d_st.cpu().numpy()
    res = dict(gpu=smi[0] if smi else "unknown", batch=nf, kps_per_frame=args.kps, keypoints=n,
               klt_tracking_ms=round(kt[0], 3), klt_tracking_ms_range=[round(kt[1], 3), round(kt[2], 3)],
               fb_klt_ms=round(fb[0], 3), fb_klt_ms_range=[round(fb[1], 3), round(fb[2], 3)],
               tracked=int(status.sum()), tracked_fb_klt=int(st_fb.sum()),
               pass1_members=int(member1.sum()), pass1_members_kernel=int(out["nbkps"].sum().item()),
               retry_gained=int((member1 & (passes == 2) & (status == 1)).sum()),
               p3p_frames=round(float(out["p3p_req"].float().mean().item()), 4))
    print("gpu (name, power limit, SM clock, max SM clock):", res["gpu"], flush=True)
    print(json.dumps(res), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
