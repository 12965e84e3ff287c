"""Per-kernel times of the resident C2 step that bench.py measures, on one GPU.

    python scripts/bench_step_kernels.py [--batch 256] [--steps 20] [--warmup 5]

Builds bench.py's own Workload (imported, so the shapes cannot drift apart), runs `steps` resident steps with the
context's per-kernel CUDA events on (they serialise the launches: this is a breakdown, not the step time; bench.py gives
that) and prints one JSON line:

  kernels_ms_per_step   every kernel name -> ms per step (sum over its launches in a step), and launches per step
  step_ms               the same steps timed with the events off, for the share each kernel has of it
  pyramid               achieved GB/s of pyr_levels_kernel against the bytes the algorithm needs: level 0 read once,
                        levels 1-3 written once, for both images of every pair
  subpix                mean and histogram of cornerSubPix iterations per detected point (counting instantiation of the
                        kernel, run once on the step's integer detections; the product launch carries no counter)
  klt                   level set-ups and Lucas-Kanade iterations per keypoint, forward and backward tracks together: means
                        and histograms (counting instantiation of fb_klt_kernel, run once on the step's own keypoints,
                        priors and depths; the product launch carries no counter)
  gpu                   card name, power limit and maximum SM clock, read in the same run

Writes nothing."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)


def pyramid_bytes(frames: int, w: int, h: int) -> int:
    """Level 0 read once and the three pyrDown levels written once, per frame."""
    n, lw, lh = w * h, w, h
    for _ in range(3):
        lw, lh = (lw + 1) // 2, (lh + 1) // 2
        n += lw * lh
    return frames * n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256, help="frame pairs per step")
    ap.add_argument("--steps", type=int, default=20, help="profiled steps (at least 20 for a stable mean)")
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    import bench
    from ov2slam_b200 import api
    if not torch.cuda.is_available():
        raise SystemExit("bench_step_kernels.py: no CUDA device; there is no CPU fallback")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx = api.Context(0, stream=stream.cuda_stream)
    wl = bench.Workload(torch, api, ctx, 0, args.batch)
    B, W, H = args.batch, bench.W_IMG, bench.H_IMG

    for _ in range(args.warmup):
        wl.step_resident()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(args.steps):
        wl.step_resident()
    e1.record(stream)
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / args.steps

    ctx.profile(True)
    for _ in range(args.steps):
        wl.step_resident()
    rep = ctx.profile_report()
    ctx.profile(False)
    kernels = {k: {"ms_per_step": v[0] / args.steps, "launches_per_step": v[1] / args.steps,
                   "share_of_step": v[0] / args.steps / step_ms} for k, v in sorted(rep.items(), key=lambda kv: -kv[1][0])}
    ksum = sum(v["ms_per_step"] for v in kernels.values())

    pyr = None
    if "pyr_levels_kernel" in kernels:
        nbytes = pyramid_bytes(2 * B, W, H)
        ms = kernels["pyr_levels_kernel"]["ms_per_step"]
        pyr = {"algorithmic_bytes_per_step": nbytes, "ms_per_step": ms, "achieved_gbs": nbytes / (ms * 1e-3) / 1e9,
               "datasheet_hbm_gbs": 3350.0}

    # cornerSubPix iterations on the step's own detections (same frames, same threshold, same integer points)
    ncell = wl.ncell
    d_int = torch.empty((B * ncell, 2), dtype=torch.int32, device="cuda")
    d_pts = torch.empty((B * ncell, 2), dtype=torch.float32, device="cuda")
    d_it = torch.empty(B * ncell, dtype=torch.int32, device="cuda")
    wl.d_th.fill_(bench.FAST_TH)
    wl.fe.detect_grid_fast(wl.pyr_cur_d, bench.CELL, 0, B, wl.d_th, wl.d_new, wl.d_cnt, out_pts_int=d_int, max_per_frame=ncell)
    wl.fe.debug_subpix_iters(wl.pyr_cur_d, 0, B, ncell, d_int, d_pts, d_it)
    torch.cuda.synchronize()
    same = bool(torch.equal(d_pts, wl.d_new))
    it = d_it.cpu().numpy()
    it = it[it >= 0]
    subpix = {"slots": int(B * ncell), "points": int(it.size), "mean_iterations": float(it.mean()) if it.size else None,
              "histogram": {str(k): int(v) for k, v in enumerate(np.bincount(it, minlength=31)) if v},
              "counting_kernel_matches_product": same}

    # fb-KLT work on the step's own keypoints, priors and pyramid depths
    n = B * bench.NKP
    d_pri = wl.d_pri0.clone()
    d_st = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_cnt = torch.empty((n, 2), dtype=torch.int32, device="cuda")
    wl.ft.fb_klt_tracking(wl.pyr_prev_d, wl.pyr_cur_d, 9, wl.d_lv, 30.0, 0.5, wl.d_kps, d_pri, d_st, n=n, per_frame=bench.NKP,
                          counts_out=d_cnt)
    wl.d_pri.copy_(wl.d_pri0)
    wl.ft.fb_klt_tracking(wl.pyr_prev_d, wl.pyr_cur_d, 9, wl.d_lv, 30.0, 0.5, wl.d_kps, wl.d_pri, wl.d_status, n=n,
                          per_frame=bench.NKP)
    torch.cuda.synchronize()
    cnt = d_cnt.cpu().numpy()
    klt = {"keypoints": int(n), "mean_setups": float(cnt[:, 0].mean()), "mean_iterations": float(cnt[:, 1].mean()),
           "setups_histogram": {str(k): int(v) for k, v in enumerate(np.bincount(cnt[:, 0])) if v},
           "iterations_histogram": {str(k): int(v) for k, v in enumerate(np.bincount(cnt[:, 1])) if v},
           "counting_kernel_matches_product": bool(torch.equal(d_pri, wl.d_pri) and torch.equal(d_st, wl.d_status))}

    wl.close()
    ctx.close()
    print(json.dumps({"gpu": gpu[0] if gpu else None, "batch": B, "image": [W, H], "steps": args.steps, "step_ms": step_ms,
                      "kernels_ms_sum": ksum, "kernels_ms_per_step": kernels, "pyramid": pyr, "subpix": subpix, "klt": klt,
                      "command": "python scripts/bench_step_kernels.py " + " ".join(sys.argv[1:])}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
