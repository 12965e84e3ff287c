"""Rectification benchmark: CameraCalibration::rectifyImage (bit-exact cv::remap) fused into the pyramid build, on one GPU.

    python scripts/bench_rect.py [--pairs 132] [--steps 10] [--warmup 3]

One step = `pairs` unrectified 752 x 480 stereo pairs from a synthetic distorted rig (intrinsics like EuRoC's, written below; no
calibration files are read), resident on the device: ov2_pyr_build_remap of the left and of the right batch (rectification into
level 0 + levels 1-3), next to ov2_pyr_build of the same images without rectification.  The CV_16SC2 maps are built by cv2 at
set-up, outside the timed region.  Also reported: the same call from pageable host images (upload every step), remap_kernel's
time and achieved GB/s against its algorithmic bytes, cv2.remap on the host cores, and the card's name and power limit read in
the same run.  Prints one JSON line; writes nothing."""
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

RECT_W, RECT_H = 752, 480
# a distorted, unrectified stereo rig with intrinsics like EuRoC's cam0 / cam1 (fx, fy, cx, cy; k1, k2, p1, p2, k3) and a right
# camera 11 cm to the side, rotated by a few milliradians: what the reference rectifies with bdo_stereo_rect = 1
RECT_RIG = dict(K0=(458.654, 457.296, 367.215, 248.375), D0=(-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 0.0),
                K1=(457.587, 456.134, 379.999, 255.238), D1=(-0.28368365, 0.07451284, -0.00010473, -3.55590700e-05, 0.0),
                rvec=(0.0020, -0.0060, 0.0030), t=(-0.110074, 0.000399, -0.000853))


def remap_algorithmic_bytes(count: int, w: int, h: int) -> float:
    """remap_kernel, per launch of `count` frames sharing one map: each source pixel read once, each output pixel written once,
    the map's packed 4-byte entry per pixel once."""
    return count * w * h * 2.0 + w * h * 4.0


def rect_maps(cv2, w: int = RECT_W, h: int = RECT_H, rig: dict = RECT_RIG):
    """CV_16SC2 + CV_16UC1 maps of both cameras as SlamManager::setupStereoCalibration builds them (cv::stereoRectify with
    CALIB_ZERO_DISPARITY, alpha 0, then CameraCalibration::setUndistStereoMap's initUndistortRectifyMap, m1type 11)."""
    K = [np.array([[k[0], 0, k[2]], [0, k[1], k[3]], [0, 0, 1]], np.float64) for k in (rig["K0"], rig["K1"])]
    D = [np.array(rig["D0"], np.float64), np.array(rig["D1"], np.float64)]
    R, _ = cv2.Rodrigues(np.array(rig["rvec"], np.float64))
    R0, R1, P0, P1, _, _, _ = cv2.stereoRectify(K[0], D[0], K[1], D[1], (w, h), R, np.array(rig["t"], np.float64),
                                                flags=cv2.CALIB_ZERO_DISPARITY, alpha=0.0)
    return [cv2.initUndistortRectifyMap(K[0], D[0], R0, P0, (w, h), cv2.CV_16SC2),
            cv2.initUndistortRectifyMap(K[1], D[1], R1, P1, (w, h), cv2.CV_16SC2)]


def run(torch, api, ctx, stream, args, peaks, usable_cores):
    """`rect_pairs` unrectified 752 x 480 stereo pairs per step, resident on the device: ov2_pyr_build_remap of the left and the
    right batch (rectification into level 0 + levels 1-3) next to ov2_pyr_build of the same images (no rectification), the
    remap kernel's time and bandwidth, and cv2.remap on the host cores.  The maps are built by cv2 at set-up, untimed."""
    import cv2
    from ov2slam_b200 import synth
    w, h, n = RECT_W, RECT_H, args.pairs
    maps = rect_maps(cv2)
    uniq = [synth.make_frame(3100 + k, w, h) for k in range(8)]
    left = np.stack([uniq[k % 8] for k in range(n)])
    right = np.stack([uniq[(k + 3) % 8] for k in range(n)])
    dl, dr = torch.from_numpy(left).cuda(), torch.from_numpy(right).cuda()
    torch.cuda.synchronize()
    rm = [api.RemapMap(ctx, *m) for m in maps]
    pyr_rect = [api.Pyramid(ctx, n, w, h, 3) for _ in range(2)]
    pyr_plain = [api.Pyramid(ctx, n, w, h, 3) for _ in range(2)]

    def step_rect():
        pyr_rect[0].build_remap(rm[0], dl)
        pyr_rect[1].build_remap(rm[1], dr)

    def step_plain():
        pyr_plain[0].build(dl)
        pyr_plain[1].build(dr)

    def timed(fn, steps, warmup):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    steps, warmup = max(args.steps, 10), max(args.warmup, 2)
    ms = {"rect": [], "plain": []}
    for _ in range(3):                                       # alternated, median of three
        ms["rect"].append(timed(step_rect, steps, warmup))
        ms["plain"].append(timed(step_plain, steps, warmup))
    ms_rect, ms_plain = sorted(ms["rect"])[1], sorted(ms["plain"])[1]
    checked = all(np.array_equal(pyr_rect[s].download(k, 0), cv2.remap(imgs[k], *maps[s], cv2.INTER_LINEAR))
                  for s, imgs in enumerate((left, right)) for k in (0, n - 1))
    # host images: each step uploads the unrectified pairs (pageable numpy arrays) once
    ms_host = timed(lambda: (pyr_rect[0].build_remap(rm[0], left), pyr_rect[1].build_remap(rm[1], right)), 3, 1)
    ctx.profile(True)
    for _ in range(5):
        step_rect()
    rep = ctx.profile_report()
    ctx.profile(False)
    k_ms, k_n = rep.get("remap_kernel", (0.0, 0))
    kernel_ms = k_ms / max(k_n, 1)
    alg = remap_algorithmic_bytes(n, w, h)
    peak, peak_src = peaks
    achieved = alg / (kernel_ms * 1e-3) / 1e9 if kernel_ms > 0 else None
    # cv2.remap on the host: the reference's per-frame call, both images of a pair
    cores = usable_cores()
    sample = 32

    def cpu_rate(threads):
        cv2.setNumThreads(threads)
        for k in range(2):
            cv2.remap(left[k], *maps[0], cv2.INTER_LINEAR)
        t0 = time.perf_counter()
        for k in range(sample):
            cv2.remap(left[k], *maps[0], cv2.INTER_LINEAR)
            cv2.remap(right[k], *maps[1], cv2.INTER_LINEAR)
        return sample / (time.perf_counter() - t0)

    cpu_all, cpu_one = cpu_rate(cores), cpu_rate(1)
    cv2.setNumThreads(1)
    for p in pyr_rect + pyr_plain + rm:
        p.close()
    return {"metric": "rectified stereo pairs/sec (resident)", "value": n / (ms_rect * 1e-3), "unit": "pairs/s",
            "ms_per_step": ms_rect, "pairs_per_step": n, "image": [w, h],
            "pyr_build_value": n / (ms_plain * 1e-3), "pyr_build_ms_per_step": ms_plain,
            "host_images_value": n / (ms_host * 1e-3),
            "repeats_ms": ms, "bit_exact_vs_cv2_remap": bool(checked),
            "what": "ov2_pyr_build_remap of the left and the right batch (remap into level 0 + levels 1-3) vs ov2_pyr_build of the "
                    "same unrectified images; host_images_value: the same with pageable host images uploaded every step",
            "kernel": {"name": "remap_kernel", "ms_per_launch": kernel_ms, "launches_per_step": 2,
                       "algorithmic_bytes_per_launch": alg, "achieved": achieved, "peak": peak, "unit": "GB/s",
                       "frac": achieved / peak if achieved else None, "peak_source": peak_src, "bound": "hbm",
                       "byte_model": "count*W*H*2 + W*H*4 per launch"},
            "cpu_baseline": {"value": cpu_all, "unit": "pairs/s", "cores": cores, "single_core_value": cpu_one, "kind": "library",
                             "sample": f"cv2.remap INTER_LINEAR (OpenCV {cv2.__version__}) of {sample} pairs, CV_16SC2 maps, "
                                       f"cv2.setNumThreads({cores}) / (1)"}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=132, help="unrectified stereo pairs per step")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    from ov2slam_b200 import api
    from bench import _peaks, usable_cores
    if not torch.cuda.is_available():
        raise SystemExit("bench_rect.py: no CUDA device; there is no CPU fallback")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx = api.Context(0, stream=stream.cuda_stream)
    out = run(torch, api, ctx, stream, args, _peaks(), usable_cores)
    out["gpu"] = gpu[0] if gpu else None
    out["command"] = "python scripts/bench_rect.py " + " ".join(sys.argv[1:])
    ctx.close()
    print(json.dumps(out), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
