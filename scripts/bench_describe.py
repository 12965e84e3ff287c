"""Descriptor benchmark: ov2_describe (ORB fallback) on its per-window and its dense path, on one GPU.

    python scripts/bench_describe.py [--batch 256] [--launches 50] [--warmup 5]

Workload: C2's geometry (640 x 480 frames, 40 px cells), resident on the device: the tracked set (1024 keypoints per
frame) and the new set (one slot per cell, 12 x 16 = 192 per frame, about 108 valid).  Each set is described by a ragged
frame_idx call, which always takes the per-window path (describe_kernel), and by a fixed-stride call on the same points,
which takes the path the density rule in frontend_desc.cu picks, alternated in one process and timed with CUDA events
over `launches` calls after warm-up (median of three windows).  dense_ms is the fixed-stride time where the rule picks
the dense path, and null where it does not.  Then, in a separate pass with per-kernel events, the dense path's smoothing
and gather kernel times.  Then a sweep of per_frame at the same batch over the rule's crossover: cover =
per_frame * 26^2 / ((w - 36)(h - 36)).  Checks that both calls return the same bytes on every set.  Prints the card's
name, power limit and SM clock read in the same run, and one JSON line; writes nothing."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

W_IMG, H_IMG, CELL, NKP = 640, 480, 40, 1024
SWEEP = (32, 64, 108, 160, 192, 256, 320, 384, 448, 512, 768, 1024)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256, help="frames per call")
    ap.add_argument("--launches", type=int, default=50, help="timed calls per window")
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    from ov2slam_b200 import api, synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_describe.py: no CUDA device; there is no CPU fallback")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx = api.Context(0, stream=stream.cuda_stream)
    fe = api.FeatureExtractor(ctx)
    B, w, h = args.batch, W_IMG, H_IMG
    uniq = [synth.make_frame(4200 + k, w, h) for k in range(16)]
    pyr = api.Pyramid(ctx, B, w, h, 0)
    pyr.build(np.stack([uniq[k % 16] for k in range(B)]))
    rng = np.random.default_rng(0)
    ncell = (h // CELL) * (w // CELL)

    def point_set(per_frame, frac_valid=1.0):
        p = np.stack([rng.uniform(12, w - 12, B * per_frame), rng.uniform(12, h - 12, B * per_frame)], axis=1).astype(np.float32)
        p[rng.random(len(p)) >= frac_valid] = -1.0           # empty slots (x < 0)
        return torch.from_numpy(p).cuda()

    def call(pts, per_frame, out, fidx):
        """The ragged call when `fidx` is given (always the per-window path), else the fixed-stride call."""
        if fidx is not None:
            fe.describe_brief(pyr, pts, out[0], out[1], n=pts.shape[0], frame_idx=fidx)
        else:
            fe.describe_brief(pyr, pts, out[0], out[1], n=pts.shape[0], per_frame=per_frame)

    def outputs(n):
        return (torch.empty((n, 32), dtype=torch.uint8, device="cuda"), torch.empty(n, dtype=torch.uint8, device="cuda"))

    def timed(fn, launches, warmup):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(launches):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / launches

    def kernels(pts, per_frame, fidx, reps=1):
        """{kernel: (total ms, launches)} of `reps` calls (per-kernel events serialise the launches)."""
        out = outputs(pts.shape[0])
        call(pts, per_frame, out, fidx)
        ctx.profile(True)
        for _ in range(reps):
            call(pts, per_frame, out, fidx)
        rep = ctx.profile_report()
        ctx.profile(False)
        return rep

    def compare(pts, per_frame, launches, warmup, windows=3):
        """ms per call of the ragged (per-window) and the fixed-stride call (median of `windows` alternated windows), the
        latter null unless the rule picks the dense path, and whether the bytes agree."""
        # frame_idx[i] = i // per_frame: the frames of the fixed-stride call
        fidx = torch.arange(pts.shape[0] // per_frame, dtype=torch.int32, device="cuda").repeat_interleave(per_frame)
        assert set(kernels(pts, per_frame, fidx)) == {"describe_kernel"}
        dense = "describe_dense_kernel" in kernels(pts, per_frame, None)
        res, ms = {}, {True: [], False: []}
        for _ in range(windows):
            for ragged in (True, False):
                out = outputs(pts.shape[0])
                f = fidx if ragged else None
                ms[ragged].append(timed(lambda: call(pts, per_frame, out, f), launches, warmup))
                res[ragged] = out
        same = bool(torch.equal(res[True][0], res[False][0]) and torch.equal(res[True][1], res[False][1]))
        return sorted(ms[True])[windows // 2], sorted(ms[False])[windows // 2] if dense else None, same

    sets = {"tracked": (point_set(NKP), NKP), "new": (point_set(ncell, 108 / ncell), ncell)}
    report = {}
    for name, (pts, per_frame) in sets.items():
        pw, dn, same = compare(pts, per_frame, args.launches, args.warmup)
        # kernel times of the dense path, per call
        rep = kernels(pts, per_frame, None, 10) if dn is not None else None
        report[name] = {"per_frame": per_frame, "n": int(pts.shape[0]), "per_window_ms": pw, "dense_ms": dn,
                        "speedup_dense": pw / dn if dn is not None else None, "bit_equal": same,
                        "dense_kernels_ms": {k: v[0] / v[1] for k, v in rep.items()} if rep is not None else None}
    band = (w - 36) * (h - 36)
    sweep = []
    for per_frame in SWEEP:
        pts = point_set(per_frame)
        pw, dn, same = compare(pts, per_frame, max(args.launches // 2, 10), 2, windows=1)
        sweep.append({"per_frame": per_frame, "cover": round(per_frame * 26 * 26 / band, 3), "per_window_ms": pw, "dense_ms": dn,
                      "bit_equal": same})
    pyr.close()
    ctx.close()
    print(json.dumps({"gpu": gpu[0] if gpu else None, "batch": B, "image": [w, h], "sets": report, "sweep": sweep,
                      "command": "python scripts/bench_describe.py " + " ".join(sys.argv[1:])}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
