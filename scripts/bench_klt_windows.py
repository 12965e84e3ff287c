"""fbKltTracking at window sizes 5 to 31 on the C2 tracking shapes, on one GPU, against the cv2 call sequence on the host.

    python scripts/bench_klt_windows.py [--batch 256] [--steps 20] [--warmup 3] [--cpu-frames 2]

Builds bench.py's own Workload (imported, so shapes, priors and depths cannot drift apart: 640 x 480 pairs, 1 024
keypoints per frame, 60 % at nbpyrlvl 1 with a motion prior, the rest at 3) and, for each window, tracks every keypoint
of the batch `steps` times with the context's per-kernel CUDA events on.  Per window it reports:

  kernel            fb_klt_kernel (9) or fb_klt_win_kernel (every other size)
  kernel_ms         ms per call (one call tracks the whole batch)
  keypoints_per_s   batch * 1 024 / kernel time
  setups / iters    level set-ups and Lucas-Kanade iterations per keypoint, forward and backward tracks together
                    (counting instantiation, run once on the same keypoints)
  tracked           share of keypoints with status 1
  cpu_ms_per_frame  FeatureTracker::fbKltTracking's two cv2.calcOpticalFlowPyrLK call pairs on one host core, per frame:
                    the median over `cpu_rounds` timed rounds of `cpu_frames` frames of the same batch, with the rounds'
                    min and max (cpu_ms_range) as the spread; cpu_keypoints_per_s_per_core from the median

and prints the card name, power limit and SM clock read in the same run, then one JSON line.  Writes nothing."""
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

WINDOWS = [5, 7, 9, 11, 15, 21, 31]


def cpu_klt(R, prevs, curs, kps, pri, lv, win):
    """The reference's forward / backward calls for one frame (two depth groups, as bench.py's CPU arm issues them)."""
    for lvl in (1, 3):
        m = lv == lvl
        if m.any():
            R.fb_klt_cv2(prevs, curs, kps[m], pri[m], win, lvl)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256, help="frame pairs per call")
    ap.add_argument("--steps", type=int, default=20, help="timed calls per window")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-frames", type=int, default=8, help="frames per round for the cv2 sequence (0: skip)")
    ap.add_argument("--cpu-rounds", type=int, default=3, help="timed rounds of the cv2 sequence per window")
    args = ap.parse_args()
    import torch
    import bench
    from ov2slam_b200 import api
    if not torch.cuda.is_available():
        raise SystemExit("bench_klt_windows.py: no CUDA device; there is no CPU fallback")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print("gpu:", smi[0] if smi else "unknown", flush=True)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx = api.Context(0, stream=stream.cuda_stream)
    wl = bench.Workload(torch, api, ctx, 0, args.batch)
    wl.step_resident()                                   # builds the batch's pyramids
    B, n = args.batch, args.batch * bench.NKP
    ft = api.FeatureTracker(ctx, 30, 0.01)
    d_pri = wl.d_pri0.clone()
    d_st = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_cnt = torch.empty((n, 2), dtype=torch.int32, device="cuda")

    def track(counts=None):
        d_pri.copy_(wl.d_pri0)
        ft.fb_klt_tracking(wl.pyr_prev_d, wl.pyr_cur_d, win, wl.d_lv, 30.0, 0.5, wl.d_kps, d_pri, d_st, n=n,
                           per_frame=bench.NKP, counts_out=counts)

    cpu = None
    if args.cpu_frames:
        import cv2
        from oracle import image_ref as R
        cv2.setNumThreads(1)
        frames = []
        for i in range(args.cpu_frames):
            f = slice(i * bench.NKP, (i + 1) * bench.NKP)
            frames.append((wl.pyr_prev_d.download(i, 0), wl.pyr_cur_d.download(i, 0), wl.h_kps[f].numpy(),
                           wl.h_pri0[f].numpy(), wl.h_lv[f].numpy()))
        cpu = (R, frames)

    rows = []
    for win in WINDOWS:
        for _ in range(args.warmup):
            track()
        torch.cuda.synchronize()
        ctx.profile(True)
        for _ in range(args.steps):
            track()
        rep = ctx.profile_report()
        ctx.profile(False)
        name = "fb_klt_kernel" if win == 9 else "fb_klt_win_kernel"
        ms = rep[name][0] / rep[name][1]
        track(d_cnt)
        torch.cuda.synchronize()
        cnt = d_cnt.cpu().numpy()
        full = wl.h_kps.numpy()[:, 0] >= 0
        row = {"win": win, "kernel": name, "kernel_ms": ms, "keypoints_per_s": n / (ms * 1e-3),
               "setups_per_kp": float(cnt[full, 0].mean()), "iters_per_kp": float(cnt[full, 1].mean()),
               "tracked": float(d_st.float().mean().item())}
        if cpu:
            R, frames = cpu
            for fr in frames:                                # untimed round: cv2 paging, allocations
                cpu_klt(R, *fr, win)
            rounds = []
            for _ in range(args.cpu_rounds):
                t0 = time.perf_counter()
                for fr in frames:
                    cpu_klt(R, *fr, win)
                rounds.append((time.perf_counter() - t0) * 1e3 / len(frames))
            cms = float(np.median(rounds))
            row.update(cpu_ms_per_frame=cms, cpu_ms_range=[min(rounds), max(rounds)],
                       cpu_keypoints_per_s_per_core=bench.NKP / (cms * 1e-3))
        else:
            row.update(cpu_ms_per_frame="not measured")
        rows.append(row)
        print(f"win {win:2d} {name:18s} {ms:8.3f} ms  {row['keypoints_per_s'] / 1e6:7.1f} M kp/s  set-ups "
              f"{row['setups_per_kp']:.2f}  iters {row['iters_per_kp']:.2f}  tracked {row['tracked']:.3f}  cpu "
              f"{row.get('cpu_ms_per_frame')} {row.get('cpu_ms_range', '')}", flush=True)
    ctx.close()
    print(json.dumps({"gpu": smi, "batch": B, "keypoints_per_frame": bench.NKP, "steps": args.steps, "windows": rows}))


if __name__ == "__main__":
    main()
