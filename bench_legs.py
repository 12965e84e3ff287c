"""bench_legs.py - the C4 (stereo 1280x720, accurate parameters) and C5 (localBA 50 KF x 20k pts x 150k obs,
landmarks split over the ranks) legs of bench.py (BASELINE.json configs[3] and configs[4]).

C4, one step = one batch of stereo units (prev-left, cur-left, cur-right), per unit what the reference does for
a stereo keyframe with parameters_files/accurate (use_clahe 1, use_singlescale_detector 1, nmaxdist 35):

    C+P  preprocessImage of the three images: CLAHE(clip 3, tiles W/50 x H/50) + buildOpticalFlowPyramid
         (visual_front_end.cpp:1143-1177; right image: mapper.cpp:75-81)
    K    temporal fb-KLT prev-left -> cur-left, NTRK keypoints (60 % with a motion prior at nbpyrlvl 1, the rest
         at nbpyrlvl 3; visual_front_end.cpp:196,242)
    D    detectSingleScale + cornerSubPix on the equalised cur-left, tracked keypoints as vcurkps
         (feature_extractor.cpp:288-440; map_manager.cpp:316)
    B    describeBRIEF on the RAW cur-left of the tracked and of the new keypoints (map_manager.cpp:301-303,326-329)
    K'   stereo fb-KLT cur-left -> cur-right of every keypoint (tracked: 60 % with a disparity prior at nbpyrlvl 1,
         the rest and all new keypoints at nbpyrlvl 3; map_manager.cpp:510,550)

Nothing here touches oracle/ except the cpu_baseline functions (run_c4_cpu, the C5 C restatement).
"""
from __future__ import annotations

import json
import os
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent

C4_W, C4_H, C4_CELL, C4_NTRK, C4_Q = 1280, 720, 35, 400, 0.001
C4_NCELL = (C4_H // C4_CELL) * (C4_W // C4_CELL)     # 36 x 20 = 720
C4_FRAC3D = 0.6
C4_TILES = (C4_W // 50, C4_H // 50)


# ----------------------------------------------------------------------------- C4 inputs
def make_stereo_unit(seed: int):
    """(prev_left, cur_left, cur_right, kps, temporal priors, temporal levels, stereo prior offsets, stereo levels).
    cur_right(x, y) = cur_left(x + d, y) + noise with a seeded disparity d in [5, 30] px."""
    from ov2slam_b200 import synth
    prev, cur, flow = synth.make_pair(seed, C4_W, C4_H)
    rng = np.random.default_rng(seed + 31)
    disp = float(rng.uniform(5.0, 30.0))
    right = synth.shift_image(cur, -disp, 0.0) + rng.normal(0.0, 1.5, size=cur.shape)
    right = np.ascontiguousarray(np.clip(np.rint(right), 0, 255).astype(np.uint8))
    kps = np.stack([rng.uniform(40, C4_W - 40, C4_NTRK), rng.uniform(40, C4_H - 40, C4_NTRK)], axis=1).astype(np.float32)
    is3d, pri = synth.make_priors(seed, kps, flow, C4_FRAC3D)
    lv = np.where(is3d, 1, 3).astype(np.uint8)
    soff = np.zeros((C4_NTRK, 2), np.float32)
    soff[is3d, 0] = (-disp + rng.normal(0.0, 1.0, size=int(is3d.sum()))).astype(np.float32)
    return prev, cur, right, kps, pri, lv, soff, lv.copy()


def _unit_job(seed):
    return make_stereo_unit(seed)


def make_stereo_batch(first_seed: int, batch: int, unique: int, nproc: int = 1):
    """`batch` units from `unique` generated ones (the rest are vertical flips / repeats of them at distinct
    addresses: generation costs ~0.7 s per unit and the batch only has to exceed L2 in footprint)."""
    unique = max(1, min(unique, batch))
    seeds = [first_seed + i for i in range(unique)]
    if nproc > 1:
        import multiprocessing as mp
        with mp.get_context("fork").Pool(min(nproc, unique)) as pool:
            base = pool.map(_unit_job, seeds)
    else:
        base = [make_stereo_unit(s) for s in seeds]
    out = dict(prev=np.empty((batch, C4_H, C4_W), np.uint8), cur=np.empty((batch, C4_H, C4_W), np.uint8),
               right=np.empty((batch, C4_H, C4_W), np.uint8), kps=np.empty((batch, C4_NTRK, 2), np.float32),
               pri=np.empty((batch, C4_NTRK, 2), np.float32), lv=np.empty((batch, C4_NTRK), np.uint8),
               soff=np.empty((batch, C4_NTRK, 2), np.float32), slv=np.empty((batch, C4_NTRK), np.uint8))
    for i in range(batch):
        p, c, r, k, pr, lv, so, slv = base[i % unique]
        if (i // unique) % 2 == 1:      # vertical flip: a different image with the same statistics
            p, c, r = p[::-1], c[::-1], r[::-1]
            k = k.copy(); pr = pr.copy()
            k[:, 1] = (C4_H - 1) - k[:, 1]
            pr[:, 1] = (C4_H - 1) - pr[:, 1]
        out["prev"][i], out["cur"][i], out["right"][i] = p, c, r
        out["kps"][i], out["pri"][i], out["lv"][i], out["soff"][i], out["slv"][i] = k, pr, lv, so, slv
    return out


# ----------------------------------------------------------------------------- C4 CPU reference sequence
def _detect_single_scale_timing(cv2, im, cellsize, curkps, dmaxquality):
    """detectSingleScale's per-cell OpenCV call sequence (feature_extractor.cpp:288-440) for TIMING: the same calls
    with the same sizes as the reference (GaussianBlur 3x3 on the cell, cornerMinEigenVal(3, 3), multiply by the mask
    cell, minMaxLoc, circle - twice per cell), then cornerSubPix.  Python hands OpenCV the cell without its parent,
    so the blur border is reflected inside the cell (the parity oracle, oracle/image_ref.py, models the parent-aware
    border; the cost is identical)."""
    rows, cols = im.shape
    r4 = cellsize // 4
    nh, nw = rows // cellsize, cols // cellsize
    occ = np.zeros((nh + 1, nw + 1), bool)
    mask = np.ones((rows, cols), np.float32)
    for px in curkps:
        occ[int(px[1] / cellsize), int(px[0] / cellsize)] = True
        cv2.circle(mask, (int(round(float(px[0]))), int(round(float(px[1])))), r4, 0, -1)
    pts, second, nboccup = [], [], 0
    for i in range(nh * nw):
        r, c = divmod(i, nw)
        if occ[r, c]:
            nboccup += 1
            continue
        x, y = c * cellsize, r * cellsize
        if not (x + cellsize < cols - 1 and y + cellsize < rows - 1):
            continue
        cell = cv2.GaussianBlur(im[y:y + cellsize, x:x + cellsize], (3, 3), 0)
        hmap = cv2.cornerMinEigenVal(cell, 3, 3)
        for rnd in range(2):
            prod = cv2.multiply(hmap, mask[y:y + cellsize, x:x + cellsize])
            _, mx, _, loc = cv2.minMaxLoc(prod)
            if mx >= dmaxquality:
                (pts if rnd == 0 else second).append((loc[0] + x, loc[1] + y))
                cv2.circle(mask, (loc[0] + x, loc[1] + y), r4, 0, -1)
    nbsec = nh * nw - (len(pts) + nboccup)          # second detections fill the cells that stayed empty (:400-412)
    pts += second[:max(nbsec, 0)]
    p = np.array(pts, np.float32).reshape(-1, 1, 2)
    if len(p):
        cv2.cornerSubPix(im, p, (3, 3), (-1, -1), (cv2.TERM_CRITERIA_EPS + cv2.TERM_CRITERIA_MAX_ITER, 30, 0.01))
    return p.reshape(-1, 2)


def _c4_cpu_unit(R, cv2, clahe, u):
    prev, cur, right, kps, pri, lv, soff, slv = u
    eP, eC, eR = clahe.apply(prev), clahe.apply(cur), clahe.apply(right)
    tracked = pri.copy()
    status = np.zeros(len(kps), np.uint8)
    for lvl in (1, 3):
        idx = np.nonzero(lv == lvl)[0]
        if len(idx):
            tracked[idx], status[idx] = R.fb_klt_cv2(eP, eC, kps[idx], tracked[idx], 9, lvl)
    alive = tracked[status.astype(bool)]              # the reference hands only the surviving tracks on (the GPU arm: all slots)
    R.describe_cv2(cur, alive)
    newpts = _detect_single_scale_timing(cv2, eC, C4_CELL, alive, C4_Q)
    R.describe_cv2(cur, newpts)
    spri = tracked + soff
    for lvl in (1, 3):
        idx = np.nonzero(slv == lvl)[0]
        if len(idx):
            R.fb_klt_cv2(eC, eR, tracked[idx], spri[idx], 9, lvl)
    if len(newpts):
        R.fb_klt_cv2(eC, eR, newpts, newpts.copy(), 9, 3)
    return int(status.sum()), len(newpts)


def _c4_cpu_worker(seeds):
    import cv2
    cv2.setNumThreads(1)
    from oracle import image_ref as R
    clahe = cv2.createCLAHE(3.0, C4_TILES)
    units = [make_stereo_unit(s) for s in seeds]
    if units:
        _c4_cpu_unit(R, cv2, clahe, units[0])   # untimed warm-up of this process
    t0 = time.perf_counter()
    n = 0
    for u in units:
        _c4_cpu_unit(R, cv2, clahe, u)
        n += 1
    return time.perf_counter() - t0, n


def run_c4_cpu(nunits: int, nproc: int, first_seed: int = 7000):
    """stereo units/s of the OpenCV reference sequence with `nproc` single-threaded processes."""
    import multiprocessing as mp
    nproc = max(1, min(nproc, nunits))
    seeds = [first_seed + i for i in range(nunits)]
    shares = [seeds[i::nproc] for i in range(nproc)]
    if nproc == 1:
        res = [_c4_cpu_worker(shares[0])]
    else:
        with mp.get_context("fork").Pool(nproc) as pool:
            res = pool.map(_c4_cpu_worker, shares)
    tmax = max(r[0] for r in res)
    n = sum(r[1] for r in res)
    return n / tmax, tmax, n


# ----------------------------------------------------------------------------- C4 GPU workload
class C4Workload:
    def __init__(self, torch, api, ctx, rank: int, batch: int, unique: int, nproc: int):
        self.torch, self.api, self.ctx, self.B = torch, api, ctx, batch
        dev = torch.device("cuda", torch.cuda.current_device())
        d = make_stereo_batch(4000 + rank * 100003, batch, unique, nproc)
        n, nn = batch * C4_NTRK, batch * C4_NCELL
        pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
        self.h = dict(prev=pin(d["prev"]), cur=pin(d["cur"]), right=pin(d["right"]), kps=pin(d["kps"].reshape(-1, 2)),
                      pri0=pin(d["pri"].reshape(-1, 2)), lv=pin(d["lv"].reshape(-1)), soff=pin(d["soff"].reshape(-1, 2)),
                      slv=pin(d["slv"].reshape(-1)))
        e = lambda *s, dt=torch.float32: torch.empty(s, dtype=dt).pin_memory()
        self.h.update(pri=e(n, 2), st=e(n, dt=torch.uint8), q=e(batch, dt=torch.float64), new=e(nn, 2), cnt=e(batch, dt=torch.int32),
                      desc_t=e(n, 32, dt=torch.uint8), val_t=e(n, dt=torch.uint8), desc_n=e(nn, 32, dt=torch.uint8),
                      val_n=e(nn, dt=torch.uint8), spri=e(n, 2), sst=e(n, dt=torch.uint8), npri=e(nn, 2), nst=e(nn, dt=torch.uint8),
                      off=pin(np.arange(0, (batch + 1) * C4_NTRK, C4_NTRK, dtype=np.int32)))
        self.d = {k: v.to(dev) for k, v in self.h.items()}
        mk = lambda lv: api.Pyramid(ctx, batch, C4_W, C4_H, lv)
        self.raw = dict(prev=mk(0), cur=mk(0), right=mk(0))
        self.pyr = dict(prev=mk(3), cur=mk(3), right=mk(3))
        self.ft = api.FeatureTracker(ctx, 30, 0.01)
        self.fe = api.FeatureExtractor(ctx, nmaxdist=C4_CELL, dmaxquality=C4_Q)
        img = 3 * batch * C4_W * C4_H
        self.h2d = img + n * (8 + 8 + 1 + 8 + 1) + batch * 8 + (batch + 1) * 4 + n * 8 + nn * 8
        self.d2h = n * (8 + 1) + batch * (8 + 4) + nn * 8 + (n + nn) * 33 + n * (8 + 1) + nn * (8 + 1)

    # one step on one context; `t` = dict of tensors (device-resident or pinned host), `sl` = (frame0, frames)
    def _run(self, ctx, ft, fe, raw, pyr, t, f0, cnt, host: bool):
        api = self.api
        k0, k1 = f0 * C4_NTRK, (f0 + cnt) * C4_NTRK
        c0, c1 = f0 * C4_NCELL, (f0 + cnt) * C4_NCELL
        n, nn = k1 - k0, c1 - c0
        t["pri"][k0:k1].copy_(t["pri0"][k0:k1])          # vpriorkps is in/out: fresh guess every step
        t["q"][f0:f0 + cnt].fill_(C4_Q)                   # constant work per step
        if host:
            ctx.batch_begin()
        for name in ("prev", "cur", "right"):
            raw[name].build(t[name][f0:f0 + cnt], first=0, count=cnt)
            api.preprocess(ctx, raw[name], pyr[name], 0, cnt, True, 3.0, C4_TILES)
        ft.fb_klt_tracking(pyr["prev"], pyr["cur"], 9, t["lv"][k0:k1], 30.0, 0.5, t["kps"][k0:k1], t["pri"][k0:k1],
                           t["st"][k0:k1], n=n, per_frame=C4_NTRK)
        fe.detect_single_scale(pyr["cur"], C4_CELL, 0, cnt, t["q"][f0:f0 + cnt], t["new"][c0:c1], t["cnt"][f0:f0 + cnt],
                               t["off_local"][:cnt + 1], t["pri"][k0:k1], None, None, max_per_frame=C4_NCELL)
        fe.describe_brief(raw["cur"], t["pri"][k0:k1], t["desc_t"][k0:k1], t["val_t"][k0:k1], n=n, per_frame=C4_NTRK)
        fe.describe_brief(raw["cur"], t["new"][c0:c1], t["desc_n"][c0:c1], t["val_n"][c0:c1], n=nn, per_frame=C4_NCELL)
        if host:
            ctx.batch_end()       # the tracked / new keypoints are on the host now: the mapper computes its priors there
            np.add(t["pri_np"][k0:k1], t["soff_np"][k0:k1], out=t["spri_np"][k0:k1])
            t["npri_np"][c0:c1] = t["new_np"][c0:c1]
            ctx.batch_begin()
        else:
            self.torch.add(t["pri"][k0:k1], t["soff"][k0:k1], out=t["spri"][k0:k1])
            t["npri"][c0:c1].copy_(t["new"][c0:c1])
        ft.fb_klt_tracking(pyr["cur"], pyr["right"], 9, t["slv"][k0:k1], 30.0, 0.5, t["pri"][k0:k1], t["spri"][k0:k1],
                           t["sst"][k0:k1], n=n, per_frame=C4_NTRK)
        ft.fb_klt_tracking(pyr["cur"], pyr["right"], 9, 3, 30.0, 0.5, t["new"][c0:c1], t["npri"][c0:c1], t["nst"][c0:c1],
                           n=nn, per_frame=C4_NCELL)
        if host:
            ctx.batch_end()

    def step_resident(self):
        self.d["off_local"] = self.d["off"]
        self._run(self.ctx, self.ft, self.fe, self.raw, self.pyr, self.d, 0, self.B, host=False)

    # ---- end-to-end arm: chunks of the batch on their own contexts / host threads (copies overlap kernels)
    def init_e2e(self, nchunks: int):
        import concurrent.futures as cf
        api, torch = self.api, self.torch
        while self.B % nchunks:
            nchunks -= 1
        self.nchunks, self.cs = nchunks, self.B // nchunks
        self.chunks = []
        for _ in range(nchunks):
            c = api.Context(torch.cuda.current_device())
            mk = lambda lv: api.Pyramid(c, self.cs, C4_W, C4_H, lv)
            self.chunks.append(dict(ctx=c, raw=dict(prev=mk(0), cur=mk(0), right=mk(0)), pyr=dict(prev=mk(3), cur=mk(3), right=mk(3)),
                                    ft=api.FeatureTracker(c, 30, 0.01), fe=api.FeatureExtractor(c, nmaxdist=C4_CELL, dmaxquality=C4_Q)))
        self.h["off_local"] = self.h["off"]
        for k in ("pri", "soff", "spri", "new", "npri"):
            self.h[k + "_np"] = self.h[k].numpy()
        self.pool = cf.ThreadPoolExecutor(max_workers=nchunks)

    def _e2e_chunk(self, k: int):
        ch = self.chunks[k]
        self._run(ch["ctx"], ch["ft"], ch["fe"], ch["raw"], ch["pyr"], self.h, k * self.cs, self.cs, host=True)
        return int(self.h["cnt"][k * self.cs:(k + 1) * self.cs].sum())   # the step's result is read on the host

    def step_e2e(self):
        return sum(self.pool.map(self._e2e_chunk, range(self.nchunks)))

    def stream_e2e(self, steps: int):
        def run(k):
            return sum(self._e2e_chunk(k) for _ in range(steps))
        return sum(self.pool.map(run, range(self.nchunks)))

    def e2e_launches(self):
        return sum(ch["ctx"].launch_count() for ch in self.chunks)

    def close(self):
        if hasattr(self, "pool"):
            self.pool.shutdown(wait=True)
        for ch in getattr(self, "chunks", []):
            for p in list(ch["raw"].values()) + list(ch["pyr"].values()):
                p.close()
            ch["ctx"].close()
        for p in list(self.raw.values()) + list(self.pyr.values()):
            p.close()


def c4_algorithmic_bytes(kernel: str, batch: int, nnew: float) -> float:
    """SURVEY.md 8(d) algorithmic bytes per STEP (all launches of that kernel in one step), C4 sizes."""
    wh = C4_W * C4_H
    if kernel == "clahe_lut_kernel":
        return 3.0 * batch * wh                                   # histogram pass reads every image once
    if kernel == "clahe_apply_kernel":
        return 3.0 * batch * 2.0 * wh                             # read + write
    if kernel in ("pyr_down_kernel", "pyr_levels_kernel"):
        return 3.0 * batch * wh * (1 + 0.25 + 0.0625 + 0.015625) + 3.0 * batch * wh * (0.25 + 0.0625)   # read l, write l+1 (re-read l1, l2 unless fused)
    if kernel == "fb_klt_kernel":
        return batch * ((C4_NTRK * 2 + nnew) * 1120.0)            # temporal + stereo(tracked) + stereo(new)
    if kernel == "ss_response_kernel":
        return batch * (wh + 4.0 * wh)                            # read the image, write the float32 response map
    if kernel == "ss_sweep_kernel":
        return batch * 4.0 * wh                                   # reads the response map once
    if kernel == "subpix_kernel":
        return batch * nnew * (81.0 * 4 + 16)
    if kernel == "describe_kernel":
        return batch * (C4_NTRK + nnew) * 1064.0
    return 0.0


def c4_leg(torch, api, dist, ctx, stream, rank, world, args, peaks, usable_cores, ncu_traffic):
    """The C4 leg: value (resident), e2e (host buffers), roofline of the dominant kernel, cv2 cpu_baseline."""
    t_gen = time.perf_counter()
    wl = C4Workload(torch, api, ctx, rank, args.c4_batch, args.c4_unique, min(usable_cores(), 16))
    gen_s = time.perf_counter() - t_gen

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def allmax(v):
        t = torch.tensor([v], dtype=torch.float64, device="cuda")
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t[0])

    steps, warm = args.c4_steps, max(3, args.warmup)
    for _ in range(warm):
        wl.step_resident()
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    l0 = ctx.launch_count()
    e0.record(stream)
    for _ in range(steps):
        wl.step_resident()
    e1.record(stream)
    torch.cuda.synchronize()
    ms_res = allmax(e0.elapsed_time(e1))
    launches = ctx.launch_count() - l0
    nnew = float(wl.d["cnt"].float().mean().item())
    ntracked = float(wl.d["st"].float().mean().item())
    nstereo = float(wl.d["sst"].float().mean().item())
    # e2e: stepped once for warm-up, then the pipelined stream timed three times (median)
    nch = args.e2e_chunks if args.e2e_chunks > 0 else (8 if world == 1 else max(4, min(8, usable_cores())))
    wl.init_e2e(nch)
    for _ in range(2):
        wl.step_e2e()
    wl.stream_e2e(1)
    reps = []
    for _ in range(3):
        barrier()
        t0 = time.perf_counter()
        wl.stream_e2e(steps)
        torch.cuda.synchronize()
        reps.append(allmax((time.perf_counter() - t0) * 1000.0))
    ms_e2e = sorted(reps)[1]
    units = world * args.c4_batch * steps
    out = None
    if rank == 0:
        ctx.profile(True)
        for _ in range(2):
            wl.step_resident()
        rep = ctx.profile_report()
        ctx.profile(False)
        peak, peak_src = peaks
        tot = sum(v[0] for v in rep.values()) or 1.0
        shares = {k: round(v[0] / tot, 4) for k, v in rep.items()}
        dname, (dms, dn) = max(rep.items(), key=lambda kv: kv[1][0])
        per_step_ms = dms / 2.0
        alg = c4_algorithmic_bytes(dname, args.c4_batch, nnew)
        achieved = alg / (per_step_ms * 1e-3) / 1e9
        per_kernel = {}
        for k, (ms, nl) in rep.items():
            a = c4_algorithmic_bytes(k, args.c4_batch, nnew)
            if a > 0:
                per_kernel[k] = {"ms_per_step": round(ms / 2.0, 4), "launches_per_step": nl // 2,
                                 "achieved_gbs": round(a / (ms / 2.0 * 1e-3) / 1e9, 1), "frac": round(a / (ms / 2.0 * 1e-3) / 1e9 / peak, 4)}
        roof = {"bound": "hbm", "kernel": dname, "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                "traffic": ncu_traffic("c4:" + dname), "peak_source": peak_src, "ms_per_step_all_launches": per_step_ms,
                "launches_per_step": dn // 2, "algorithmic_bytes_per_step": alg, "kernel_time_shares": shares,
                "per_kernel": per_kernel}
        cpu = None
        if world == 1 and not args.no_cpu:
            cores = usable_cores()
            nun = int(min(max(8 * cores, 16), 768))
            ups, t, n = run_c4_cpu(nun, cores)
            ups1, t1, n1 = run_c4_cpu(4, 1)
            cpu = {"value": ups, "unit": "stereo frames/s", "cores": cores, "kind": "port",
                   "sample": f"{n} stereo units, OpenCV call sequence (CLAHE x3, fb-KLT temporal + stereo, per-cell single-scale "
                             f"detector, cornerSubPix, ORB-fallback descriptors) in {cores} processes x 1 cv2 thread; calcOpticalFlowPyrLK "
                             f"rebuilds its pyramids per call (the reference builds each once): single core {ups1:.2f} units/s on {n1}"}
        out = {"metric": "stereo front-end frames/sec", "value": units / (ms_res / 1e3), "unit": "stereo frames/s", "n_gpus": world,
               "steps": steps, "warmup": warm, "ms_per_step": ms_res / steps, "higher_is_better": True, "scaling": "weak",
               "dtype": "u8/i32/f32",
               "config": {"workload": "C4: stereo 1280x720, parameters_files/accurate (CLAHE, single-scale detector cell 35), "
                                      "batch of %d stereo units (prev-left, cur-left, cur-right) per GPU" % args.c4_batch,
                          "tracked_keypoints_per_frame": C4_NTRK, "new_keypoints_per_frame": round(nnew, 1),
                          "temporal_tracks_ok": round(ntracked, 3), "stereo_tracks_ok": round(nstereo, 3),
                          "unique_units": args.c4_unique, "l2": "inputs 3 x %d x 0.92 MB = %.0f MB per step exceed the 50 MB L2"
                                                                % (args.c4_batch, 3 * args.c4_batch * C4_W * C4_H / 1e6),
                          "input_generation_s": round(gen_s, 1)},
               "e2e": {"value": units / (ms_e2e / 1e3), "unit": "stereo frames/s", "h2d_bytes_per_step": int(wl.h2d),
                       "d2h_bytes_per_step": int(wl.d2h), "ms_per_step": ms_e2e / steps, "chunks": wl.nchunks,
                       "mode": "pipelined chunk threads, two syncs per chunk-step (front-end results, then the mapper's stereo pass)",
                       "repeats": [units / (m / 1e3) for m in reps]},
               "gpu_launches": int(launches), "roofline": roof, "cpu_baseline": cpu}
    wl.close()
    return out


# ----------------------------------------------------------------------------- C5: localBA 50 x 20k x 150k
C5 = (50, 20000, 150000)


def ba_bytes_per_iteration(nobs: int, npts: int) -> float:
    """SURVEY.md 8(d): one Jacobian pass + one cost pass + Schur + back-substitution, J never counted."""
    return 67.0 * nobs + 64.0 * npts


def c5_leg(torch, api, dist, ctx, rank, world, args, peaks, ncu_traffic=None):
    """1 GPU: ov2_localba_solve on the C5 window (host buffers in/out).  N GPUs: landmarks (with their observations)
    split N ways, reduced camera system summed over NVLink peer memory inside the solve kernel every LM iteration
    (ov2_localba_solve_p2p)."""
    from ov2slam_b200 import synth
    ncam, npts, nobs = C5 if not args.c5_small else (20, 3000, 18000)
    pb = synth.make_ba_problem(5, ncam, npts, nobs)
    clone = lambda d: {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in d.items()}
    reps = args.c5_reps
    out = {"metric": "local-BA solves/sec", "unit": "solves/s", "n_gpus": world, "dtype": "f64", "higher_is_better": True,
           "scaling": "strong", "config": {"workload": f"C5: localBA {ncam} KF x {npts} pts x {nobs} obs, 5 % gross outliers, two-stage solve"
                                                         + ("" if world == 1 else f", landmarks split {world}-way")}}
    if world == 1:
        opt = api.Optimizer(ctx)
        for _ in range(2):
            res, _ = opt.local_ba(clone(pb))
        pbs = [clone(pb) for _ in range(reps)]
        torch.cuda.synchronize()
        l0 = ctx.launch_count()
        t0 = time.perf_counter()
        for p in pbs:
            res, _ = opt.local_ba(p)
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / reps
        launches = (ctx.launch_count() - l0) / reps
        ref_pose = pbs[-1]["pose"]
    else:
        shards = api.partition_ba_problem(pb, world)
        solver = api.ShardedOptimizer(ctx, dist, torch, rank, world)
        mine = clone(shards[rank][0])
        for _ in range(2):
            solver.local_ba(clone(shards[rank][0]))
        torch.cuda.synchronize()
        dist.barrier()
        l0 = ctx.launch_count()
        t0 = time.perf_counter()
        for _ in range(reps):
            mine = clone(shards[rank][0])
            res, flags = solver.local_ba(mine)
        torch.cuda.synchronize()
        tt = torch.tensor([time.perf_counter() - t0], dtype=torch.float64, device="cuda")
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        dt = float(tt[0]) / reps
        launches = (ctx.launch_count() - l0) / reps
        ref_pose = mine["pose"]
        out["collective"] = solver.describe()
    its = res["iters_robust"] + res["iters_refine"]
    out.update(value=1.0 / dt, ms_per_solve=1e3 * dt, lm_iterations=its, iters=[res["iters_robust"], res["iters_refine"]],
               final_cost=res["final_cost"], gpu_launches_per_solve=launches)
    peak, peak_src = peaks
    bytes_per_solve = its * ba_bytes_per_iteration(nobs, npts)
    out["roofline"] = {"bound": "hbm", "kernel": "localBA solve (all kernels of one two-stage solve)", "achieved": bytes_per_solve / dt / 1e9,
                       "peak": peak * world, "unit": "GB/s", "frac": bytes_per_solve / dt / 1e9 / (peak * world),
                       "traffic": ncu_traffic("c5:ba_lm_kernel") if (ncu_traffic and world == 1 and not args.c5_small) else None,
                       "peak_source": peak_src, "algorithmic_bytes_per_solve": bytes_per_solve,
                       "note": "67 N_obs + 64 N_pts bytes per LM iteration (SURVEY 8d) x iterations run; includes the H2D of the window "
                               "and the D2H of the states (host buffers in/out)"}
    if rank == 0:
        # same decisions as the unsharded / oracle solve
        try:
            from oracle import ba_ref_c
            ts = []
            for _ in range(3):
                ref = clone(pb)
                t = time.perf_counter()
                r = ba_ref_c.local_ba(ref)
                ts.append(time.perf_counter() - t)
            out["cpu_baseline"] = {"value": 1.0 / float(np.median(ts)), "unit": "solves/s", "cores": 1, "kind": "port",
                                   "sample": "3 solves of the same window, oracle/ba_ref_c.c single thread (restatement, not Ceres; the "
                                             "reference sets num_threads = 1, optimizer.cpp:460)",
                                   "lm_iterations": r["iters_robust"] + r["iters_refine"]}
            out["same_iterations_as_cpu"] = [r["iters_robust"], r["iters_refine"]] == out["iters"]
            out["max_pose_diff_vs_cpu"] = float(np.abs(ref_pose - ref["pose"]).max())
        except Exception as e:  # pragma: no cover
            out["cpu_baseline"] = {"error": str(e)[:160]}
    return out
