"""CPU tests of host-side logic: the libstdc++ std::sort restatement used by the grid-FAST sweep,
and that the C-ABI library loads and exports every symbol include/ov2b200.h declares."""
import ctypes
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


def test_stdsort_emulation_matches_libstdcxx_16bit_index(tmp_path):
    """ov2slam_b200/csrc/stdsort_emul.h compiled for the host vs the real std::sort (and
    std::partial_sort for the heapsort fallback) on tie-heavy inputs.  Keys are (response << 16) | index; every fourth
    input is up to 2 100 long, past the 1 891 candidates a 128-pixel FAST cell can hold, so indices above 255 and the
    deep introsort / heapsort paths are pinned too."""
    src = tmp_path / "t.cpp"
    src.write_text(r'''
#include "%s/ov2slam_b200/csrc/stdsort_emul.h"
#include <algorithm>
#include <vector>
#include <random>
#include <cstdio>
struct Kp { float r; int idx; };
static bool cmp(Kp a, Kp b) { return a.r > b.r; }
int main() {
  std::mt19937 rng(7); long bad = 0, badh = 0, nlong = 0;
  for (int it = 0; it < 60000; ++it) {
    int n = 1 + rng() %% (it %% 4 ? 200 : 2100), nv = 1 + rng() %% (it %% 3 ? 6 : 40), pat = rng() %% 3;
    nlong += n > 1891;
    std::vector<Kp> v(n); std::vector<int> k(n);
    for (int i = 0; i < n; ++i) { int r = pat == 1 ? i %% nv : pat == 2 ? (n - i) / (1 + (int)(rng() %% 3)) : (int)(rng() %% nv);
      r = 20 + r %% 235;                                   // responses 20 .. 254, as FAST gives
      v[i] = {(float)r, i}; k[i] = (r << 16) | i; }
    std::vector<Kp> w = v; std::vector<int> k2 = k;
    std::sort(v.begin(), v.end(), cmp); ov2sort::sort_desc(k.data(), n);
    for (int i = 0; i < n; ++i) if ((k[i] & 0xFFFF) != v[i].idx) { bad++; break; }
    std::partial_sort(w.begin(), w.end(), w.end(), cmp); ov2sort::heap_sort(k2.data(), 0, n);
    for (int i = 0; i < n; ++i) if ((k2[i] & 0xFFFF) != w[i].idx) { badh++; break; }
  }
  printf("%%ld %%ld %%ld\n", bad, badh, nlong); return (bad || badh || nlong < 1000) ? 1 : 0;
}''' % ROOT)
    exe = tmp_path / "t"
    subprocess.check_call(["g++", "-O2", "-o", str(exe), str(src)])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout


def test_oracle_sort_helper_is_real_std_sort():
    from oracle import image_ref as R
    r = np.array([30, 20, 30, 25, 30], np.float32)
    o = R.stdsort_desc(r)
    assert list(o) == [0, 2, 4, 3, 1]          # <= 16 elements: stable insertion sort
    rng = np.random.default_rng(0)
    r = rng.integers(20, 24, 100).astype(np.float32)
    o = R.stdsort_desc(r)
    assert sorted(o.tolist()) == list(range(100)) and (np.diff(r[o]) <= 0).all()


def test_abi_library_exports_every_declared_symbol():
    from ov2slam_b200 import api, build
    so = build.build()
    lib = ctypes.CDLL(str(so))
    hdr = (ROOT / "include" / "ov2b200.h").read_text()
    declared = set(re.findall(r"OV2_API\s+[\w\s\*]+?\b(ov2_\w+)\s*\(", hdr))
    assert len(declared) >= 18, declared
    for sym in declared:
        assert hasattr(lib, sym), f"{sym} declared in include/ov2b200.h but not exported"
    assert set(api.ABI_SYMBOLS) <= declared
    assert lib.ov2_version is not None


def test_no_cpu_fallback_without_device():
    """Product path fails loudly without a CUDA device (no CPU fallback, nothing routed via oracle/)."""
    import torch
    from ov2slam_b200 import api
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(api.Ov2Error):
        api.Context(0)


def test_product_never_imports_oracle():
    for p in (ROOT / "ov2slam_b200").rglob("*"):
        if p.suffix in (".py", ".cu", ".cuh", ".h", ".cpp", ".hpp") and "lib" not in p.parts:
            txt = p.read_text()
            assert not re.search(r"^\s*(from|import)\s+oracle", txt, re.M), p
            assert not re.search(r'#include\s+"[^"]*oracle/', txt), p


def test_product_reads_only_non_selecting_environment_variables():
    """Every kernel path is chosen from the input.  The library and the host shims read three variables, none of which
    picks a path: OV2_BA_TRACE (per-phase times and the plan on stderr), OV2_BA_CTAS (the local-BA group size, which ranks
    sharing one GPU need so that their kernels are co-resident) and OV2_DEVICE (the GPU of the drop-in classes, whose
    reference signatures take none).  The mocks under tests/helpers read their log paths and are not product code."""
    names = set()
    for d in ("csrc", "host"):
        for p in (ROOT / "ov2slam_b200" / d).rglob("*"):
            if p.suffix in (".cu", ".cuh", ".h", ".cpp", ".hpp"):
                txt = p.read_text()
                calls = re.findall(r"\bgetenv\s*\(([^)]*)\)", txt)
                assert all(re.fullmatch(r'\s*"\w+"\s*', c) for c in calls), (p, calls)
                names |= {c.strip().strip('"') for c in calls}
    assert names == {"OV2_BA_TRACE", "OV2_BA_CTAS", "OV2_DEVICE"}, names


def test_klt_level_setup_lane_code_matches_definition(tmp_path):
    """ov2slam_b200/csrc/klt_setup.cuh (the per-lane staging / Scharr / template code the KLT kernel
    runs) compiled for the host and checked against the definition (reflect-101 neighbourhood, Scharr
    with zero planes outside the image, OpenCV's fixed-point bilinear template) on random images and
    window positions: interior, every border, word-aligned and unaligned rows."""
    src = tmp_path / "k.cpp"
    src.write_text(r'''
#include "%s/ov2slam_b200/csrc/klt_setup.cuh"
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>
using namespace kltsetup;
static int refl(int i, int n) { return reflect101_any(i, n); }
int main() {
  std::mt19937 rng(11); long bad = 0, n_int = 0, n_brd = 0;
  for (int it = 0; it < 20000; ++it) {
    int lw = 14 + rng() %% 50, lh = 14 + rng() %% 40;
    bool al = rng() %% 4 != 0;
    int pitch = al ? ((lw + 3) & ~3) + 4 * (rng() %% 3) : lw + (rng() %% 3);
    std::vector<uint32_t> store((size_t)(pitch * lh + 64) / 4 + 4);
    uint8_t* img = reinterpret_cast<uint8_t*>(store.data()) + (al ? 0 : 1 + rng() %% 3);
    for (int i = 0; i < pitch * lh; ++i) img[i] = (uint8_t)(rng() >> 7);
    bool aligned = ((reinterpret_cast<uintptr_t>(img) | (uintptr_t)pitch) & 3) == 0;
    int ix = (int)(rng() %% (lw + WIN)) - WIN, iy = (int)(rng() %% (lh + WIN)) - WIN;   // the kernel's admissible range
    if (it %% 3 == 0) { ix = 1 + rng() %% (lw - 11); iy = 1 + rng() %% (lh - 11); }
    (patch_interior(ix, iy, lw, lh) ? n_int : n_brd)++;
    float a = (rng() %% 1000) / 1000.f, b = (rng() %% 1000) / 1000.f;
    int iw00 = (int)((1.f - a) * (1.f - b) * 16384.f + .5f), iw01 = (int)(a * (1.f - b) * 16384.f + .5f),
        iw10 = (int)((1.f - a) * b * 16384.f + .5f), iw11 = 16384 - iw00 - iw01 - iw10;
    if (it %% 50 == 0) { iw11 = -1; iw00 += 1; }
    alignas(16) uint8_t sP[SP_BYTES]; int sD[SD_INTS];
    memset(sP, 0xCD, sizeof sP); memset(sD, 0x5A, sizeof sD);
    int off = 0;
    for (int l = 0; l < 32; ++l) off = stage_patch(l, img, pitch, lw, lh, ix, iy, aligned, sP);
    for (int l = 0; l < 32; ++l) scharr_rows(l, sP, off, ix, iy, lw, lh, sD);
    // definition
    auto P = [&](int r, int c) { return (int)img[(size_t)refl(iy - 1 + r, lh) * pitch + refl(ix - 1 + c, lw)]; };
    for (int r = 0; r < PW; ++r) for (int c = 0; c < PW; ++c) if (sP[r * SP_PITCH + off + c] != P(r, c)) bad++;
    int dxr[DW][DW], dyr[DW][DW];
    for (int r = 0; r < DW; ++r) for (int c = 0; c < DW; ++c) {
      int y = iy + r, x = ix + c, dx = 0, dy = 0;
      if (x >= 0 && x < lw && y >= 0 && y < lh) {
        dx = (P(r, c + 2) + P(r + 2, c + 2)) * 3 + P(r + 1, c + 2) * 10 - ((P(r, c) + P(r + 2, c)) * 3 + P(r + 1, c) * 10);
        dy = ((P(r + 2, c) - P(r, c)) + (P(r + 2, c + 2) - P(r, c + 2))) * 3 + (P(r + 2, c + 1) - P(r, c + 1)) * 10;
      }
      dxr[r][c] = dx; dyr[r][c] = dy;
      int v = sD[r * SD_PITCH + c];
      if ((int)(short)(v & 0xFFFF) != dx || (v >> 16) != dy) bad++;
    }
    long A11 = 0, A12 = 0, A22 = 0, g11 = 0, g12 = 0, g22 = 0;
    for (int l = 0; l < 32; ++l) {
      short Iv[3], Ix[3], Iy[3]; int s11, s12, s22;
      template_rows(l, sP, off, sD, iw00, iw01, iw10, iw11, Iv, Ix, Iy, s11, s12, s22);
      g11 += s11; g12 += s12; g22 += s22;
      for (int k = 0; k < 3; ++k) {
        int p = 3 * l + k;
        if (p >= WIN * WIN) { if (Iv[k] || Ix[k] || Iy[k]) bad++; continue; }
        int y = p / WIN, x = p %% WIN;
        int iv = (P(y + 1, x + 1) * iw00 + P(y + 1, x + 2) * iw01 + P(y + 2, x + 1) * iw10 + P(y + 2, x + 2) * iw11 + 256) >> 9;
        int ixv = (dxr[y][x] * iw00 + dxr[y][x + 1] * iw01 + dxr[y + 1][x] * iw10 + dxr[y + 1][x + 1] * iw11 + 8192) >> 14;
        int iyv = (dyr[y][x] * iw00 + dyr[y][x + 1] * iw01 + dyr[y + 1][x] * iw10 + dyr[y + 1][x + 1] * iw11 + 8192) >> 14;
        if (Iv[k] != (short)iv || Ix[k] != (short)ixv || Iy[k] != (short)iyv) bad++;
        A11 += (long)ixv * ixv; A12 += (long)ixv * iyv; A22 += (long)iyv * iyv;
      }
    }
    if (A11 != g11 || A12 != g12 || A22 != g22) bad++;
    // interior fast path: template_direct (interpolate first, differentiate after) must give the same integers
    if (aligned && patch_interior(ix, iy, lw, lh)) {
      long d11 = 0, d12 = 0, d22 = 0;
      for (int l = 0; l < 32; ++l) {
        short Iv[3], Ix[3], Iy[3], Jv[3], Jx[3], Jy[3]; int s11, s12, s22, t11, t12, t22;
        template_rows(l, sP, off, sD, iw00, iw01, iw10, iw11, Iv, Ix, Iy, s11, s12, s22);
        template_direct(l, sP, off, iw00, iw01, iw10, iw11, Jv, Jx, Jy, t11, t12, t22);
        for (int k = 0; k < 3; ++k) if (Iv[k] != Jv[k] || Ix[k] != Jx[k] || Iy[k] != Jy[k]) bad++;
        if (s11 != t11 || s12 != t12 || s22 != t22) bad++;
        d11 += t11; d12 += t12; d22 += t22;
      }
      if (A11 != d11 || A12 != d12 || A22 != d22) bad++;
    }
  }
  printf("%%ld bad, %%ld interior, %%ld border\n", bad, n_int, n_brd);
  return (bad || n_int < 1000 || n_brd < 1000) ? 1 : 0;
}''' % ROOT)
    exe = tmp_path / "k"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", str(exe), str(src)])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr


def test_single_scale_cell_math_matches_oracle(tmp_path):
    """ov2slam_b200/csrc/sscale_math.cuh (the per-cell blur / Sobel / minimal-eigenvalue phases the
    ss_response_kernel runs) compiled for the host with contraction off and run thread by thread, vs
    oracle min_eigen_ref(blur3_cell_ref(.)): bit-exact float32 responses for every reference cell size."""
    import numpy as np
    from oracle import image_ref as R
    src = tmp_path / "s.cpp"
    src.write_text(r'''
#include "%s/ov2slam_b200/csrc/sscale_math.cuh"
#include <vector>
extern "C" void cell_response(const unsigned char* raw, int cs, float* out, int* best) {
    std::vector<unsigned char> bl(cs * cs);
    std::vector<double> cov(3 * cs * cs);
    const int nt = 256;
    for (int t = 0; t < nt; ++t) sscale::phase_blur(t, nt, raw, bl.data(), cs);
    for (int t = 0; t < nt; ++t) sscale::phase_cov(t, nt, bl.data(), cov.data(), cs);
    float bv = -INFINITY; int bi = 0x7fffffff;
    for (int t = 0; t < nt; ++t) sscale::phase_response(t, nt, cov.data(), out, cs, bv, bi);
    *best = bi;
}''' % ROOT)
    so = tmp_path / "libs.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", str(so), str(src)])
    lib = ctypes.CDLL(str(so))
    lib.cell_response.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    rng = np.random.default_rng(21)
    for it in range(60):
        cs = int(rng.choice([50, 35, 16, 20, 33, 64, 8]))
        raw = (rng.random((cs + 2, cs + 2)) * 255).astype(np.uint8)
        if it % 2:
            raw = np.clip(raw.astype(np.int32) // 8 + 100, 0, 255).astype(np.uint8)    # low contrast: many exact ties / zeros
        out = np.empty((cs, cs), np.float32)
        best = np.zeros(1, np.int32)
        lib.cell_response(raw.ctypes.data, cs, out.ctypes.data, best.ctypes.data)
        ref = R.min_eigen_ref(R.blur3_cell_ref(raw, 1, 1, cs))
        assert np.array_equal(out.view(np.int32), ref.view(np.int32)), (it, cs, int((out != ref).sum()))
        assert int(best[0]) == int(np.argmax(ref))          # first maximum in row-major order (np.argmax returns the first)


def test_pnp_solver_code_matches_oracle(tmp_path):
    """ov2slam_b200/csrc/pnp_math.cuh (the ceresPnP solve the GPU kernel instantiates with a thread-block
    context) compiled for the host with the single-lane context, vs oracle/pnp_ref.py: same success flag,
    same rejected blocks, same LM iteration count, pose to 1e-9 (normal equations vs the oracle's QR)."""
    import numpy as np
    from oracle import ba_ref, pnp_ref
    src = tmp_path / "p.cpp"
    src.write_text(r'''
#include "%s/ov2slam_b200/csrc/pnp_math.cuh"
#include <vector>
extern "C" int pnp_host(int n, const double* unpx, const double* wpts, const double* K, double* pose, int nmaxiter,
                        float chi2th, int use_robust, int apply_l2, unsigned char* flags, int* iterations) {
    pnp::Problem P; P.n = n; P.unpx = unpx; P.wpts = wpts; P.scales = nullptr;
    for (int i = 0; i < 4; ++i) P.K[i] = K[i];
    std::vector<double> chi2(n); std::vector<unsigned char> dep(n), work(n);
    pnp::SerialPar par; pnp::Summary S;
    bool ok = pnp::ceres_pnp(par, P, pose, nmaxiter, chi2th, use_robust != 0, apply_l2 != 0, chi2.data(), dep.data(), flags, work.data(), S);
    *iterations = S.iterations;
    return ok ? 1 : 0;
}''' % ROOT)
    so = tmp_path / "libp.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", str(so), str(src)])
    lib = ctypes.CDLL(str(so))
    vp = ctypes.c_void_p
    lib.pnp_host.argtypes = [ctypes.c_int, vp, vp, vp, vp, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int, vp, vp]
    K = np.array([458.0, 457.0, 367.0, 248.0])
    rng = np.random.default_rng(3)
    for case in range(12):
        n = int(rng.integers(30, 400))
        axis = rng.standard_normal(3); axis /= np.linalg.norm(axis)
        ang = 0.3 * rng.random()
        pose = np.concatenate([rng.standard_normal(3) * 0.5, axis * np.sin(ang / 2), [np.cos(ang / 2)]])
        R = ba_ref.quat_to_rot(pose[3:])
        pc = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(2, 10, n)], 1)
        wpts = np.ascontiguousarray(pc @ R.T + pose[:3])
        px = np.stack([K[0] * pc[:, 0] / pc[:, 2] + K[2], K[1] * pc[:, 1] / pc[:, 2] + K[3]], 1)
        px += rng.standard_normal(px.shape) * (0.0 if case % 3 == 0 else 0.6)
        nbad = 0 if case % 2 == 0 else n // 8
        bad = rng.choice(n, nbad, replace=False)
        px[bad] += rng.uniform(15, 60, (nbad, 2))
        if case == 11:
            px += 500.0                                            # everything is an outlier
        px = np.ascontiguousarray(px)
        start = ba_ref.pose_plus(pose, np.concatenate([rng.standard_normal(3) * 0.05, rng.standard_normal(3) * 0.02]))
        for apply_l2 in (1, 0):
            ok_r, est_r, out_r, info = pnp_ref.ceres_pnp(px, wpts, start, K, 5, 5.9915, True, bool(apply_l2), summary=True)
            est = start.copy()
            flags = np.zeros(n, np.uint8)
            its = ctypes.c_int()
            ok = lib.pnp_host(n, px.ctypes.data, wpts.ctypes.data, K.ctypes.data, est.ctypes.data, 5, 5.9915, 1, apply_l2,
                              flags.ctypes.data, ctypes.byref(its))
            assert bool(ok) == ok_r, case
            assert np.array_equal(np.nonzero(flags)[0], out_r), case
            assert np.abs(est - est_r).max() <= 1e-9, (case, np.abs(est - est_r).max())
            assert its.value == info["summary"]["iterations"], (case, its.value, info["summary"]["iterations"])


def test_device_lm_controller_replays_the_oracle_decisions(tmp_path):
    """csrc/ba_lm_ctl.cuh (the trust-region controller every CTA of the persistent solve kernel replays on the device)
    compiled for the host and driven with the per-iteration scalars of the oracle (oracle/ba_ref.py): same iteration
    counts, termination types, final costs and radius sequence for both solves of several windows - including windows
    that end on the function tolerance, on the iteration cap, and with rejected steps."""
    src = tmp_path / "ctl.cpp"
    src.write_text(r'''
#include "%s/ov2slam_b200/csrc/ba_lm_ctl.cuh"
extern "C" int replay(int n, const double* rec, int max_iters, double ftol, double* out) {
  // rec: n x 7 = x_cost, cand_cost, mcc, step2, candx2, gmax, invalid
  lmctl::State s; lmctl::init(s);
  int k = 0;
  for (;;) {
    if (!lmctl::begin_iteration(s, max_iters)) break;
    if (k >= n) return -1;
    const double* r = rec + 7 * k++;
    out[8 + s.iteration] = s.radius;
    lmctl::Action a = lmctl::end_iteration(s, r[0], r[1], r[2], r[3], r[4], r[5], r[6] != 0.0, ftol);
    if (a == lmctl::ACT_STOP) break;
  }
  out[0] = s.iteration; out[1] = s.termination; out[2] = lmctl::final_cost(s); out[3] = s.initial_cost; out[4] = k;
  return 0;
}''' % ROOT)
    so = tmp_path / "libctl.so"
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", str(so), str(src)])
    lib = ctypes.CDLL(str(so))
    lib.replay.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_void_p]
    from ov2slam_b200 import synth
    from oracle import ba_ref as B
    seen_term = set()
    rejected = 0
    cases = [(3, 6, 300, 1200, {}), (11, 6, 300, 1200, dict(max_iters_robust=2)), (21, 8, 500, 2500, dict(use_robust=False)),
             (5, 8, 300, 1500, dict(max_iters_robust=30, function_tolerance=1e-12)), (41, 8, 400, 1600, dict(stereo=True))]
    for seed, ncam, npts, nobs, kw in cases:
        stereo = kw.pop("stereo", False)
        pb = synth.make_ba_problem(seed, ncam, npts, nobs, stereo=stereo)
        log = []
        res = B.local_ba(pb, log=log, **kw)
        ctl = [e for e in log if e.get("ctl")]
        # split the records of solve #1 and #2: the iteration counter restarts at 1
        cuts = [i for i, e in enumerate(ctl) if e["it"] == 1]
        parts = [ctl[a:b] for a, b in zip(cuts, cuts[1:] + [len(ctl)])]
        assert len(parts) == len(res["summaries"])
        for part, summ, max_it in zip(parts, res["summaries"], (kw.get("max_iters_robust", 5), kw.get("max_iters_refine", 10))):
            rec = np.array([[e["x_cost"], e["cand_cost"], e["mcc"], e["step2"], e["candx2"], e["gmax"], float(e["invalid"])] for e in part])
            out = np.zeros(64)
            rc = lib.replay(len(rec), np.ascontiguousarray(rec).ctypes.data, max_it, kw.get("function_tolerance", 1e-3), out.ctypes.data)
            assert rc == 0
            term = {"CONVERGENCE": 0, "NO_CONVERGENCE": 1, "FAILURE": 2}[summ["termination"]]
            assert int(out[0]) == summ["iterations"] and int(out[1]) == term, (seed, out[:5], summ["iterations"], summ["termination"])
            assert out[2] == summ["final_cost"] and out[3] == summ["initial_cost"]
            assert int(out[4]) == len(rec)                      # every oracle iteration was consumed, none missing
            radii = [t["radius"] for t in summ["trace"]]        # radius at the start of iteration k+1 = trace[k]
            for it in range(1, summ["iterations"] + 1):
                assert abs(out[8 + it] - radii[it - 1]) <= 1e-12 * radii[it - 1], (seed, it)
            seen_term.add(summ["termination"])
            rejected += sum(1 for t in summ["trace"][1:] if not t["ok"])
    assert {"CONVERGENCE", "NO_CONVERGENCE"} <= seen_term


def test_device_lm_controller_solves_ceres_powell_known_answer(tmp_path):
    """Ceres' own known-answer test of the trust-region loop (internal/ceres/trust_region_minimizer_test.cc:223-291,
    PowellsSingularFunctionUsingLevenbergMarquardt): Powell's singular function from (3, -1, 0, 1) with each of the 14
    column-activation patterns the Ceres test runs must reach the minimum at 0 within 1e-3.  Here the iteration is driven
    by the DEVICE controller (csrc/ba_lm_ctl.cuh: step acceptance, radius update, invalid-step handling, tolerances) around
    a dense LM step with Ceres' Jacobi scaling and LM-diagonal clamp (levenberg_marquardt_strategy.cc:66-160) - the same
    decision code the persistent solve kernel replays."""
    src = tmp_path / "powell.cpp"
    src.write_text(r'''
#include "%s/ov2slam_b200/csrc/ba_lm_ctl.cuh"
#include <cmath>
#include <cstdio>
static void eval(const double* x, double* r, double J[4][4]) {
  r[0] = x[0] + 10 * x[1]; r[1] = sqrt(5.0) * (x[2] - x[3]); r[2] = (x[1] - 2 * x[2]) * (x[1] - 2 * x[2]); r[3] = sqrt(10.0) * (x[0] - x[3]) * (x[0] - x[3]);
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) J[i][j] = 0;
  J[0][0] = 1; J[0][1] = 10; J[1][2] = sqrt(5.0); J[1][3] = -sqrt(5.0);
  J[2][1] = 2 * (x[1] - 2 * x[2]); J[2][2] = -4 * (x[1] - 2 * x[2]);
  J[3][0] = 2 * sqrt(10.0) * (x[0] - x[3]); J[3][3] = -2 * sqrt(10.0) * (x[0] - x[3]);
}
static bool solve4(double A[4][4], double* b, int n) {   // Cholesky-free Gauss elimination with the LLT failure rule
  for (int j = 0; j < n; ++j) {
    if (!(A[j][j] > 0)) return false;
    for (int r = j + 1; r < n; ++r) { double f = A[r][j] / A[j][j]; for (int c = j; c < n; ++c) A[r][c] -= f * A[j][c]; b[r] -= f * b[j]; }
  }
  for (int j = n - 1; j >= 0; --j) { for (int c = j + 1; c < n; ++c) b[j] -= A[j][c] * b[c]; b[j] /= A[j][j]; }
  return true;
}
int main(int argc, char** argv) {
  int worst_iters = 0; double worst = 0;
  for (int mask = 1; mask < 16; ++mask) {
    if (mask == 0xB) continue;                       // <true, true, false, true>: excluded by the Ceres test (local minimum)
    int act[4], na = 0; for (int k = 0; k < 4; ++k) if (mask & (1 << k)) act[na++] = k;
    double x[4] = {3, -1, 0, 1.0};
    for (int k = 0; k < 4; ++k) if (!(mask & (1 << k))) x[k] = 0.0;
    lmctl::State s; lmctl::init(s);
    double scale[4] = {1, 1, 1, 1}, diag[4] = {0, 0, 0, 0};
    for (;;) {
      if (!lmctl::begin_iteration(s, 50)) break;
      double r[4], J[4][4]; eval(x, r, J);
      double cost = 0; for (int i = 0; i < 4; ++i) cost += 0.5 * r[i] * r[i];
      double gmax = 0; for (int a = 0; a < na; ++a) { double g = 0; for (int i = 0; i < 4; ++i) g += J[i][act[a]] * r[i]; gmax = fmax(gmax, fabs(g)); }
      if (s.first_iter) for (int a = 0; a < na; ++a) { double cn = 0; for (int i = 0; i < 4; ++i) cn += J[i][act[a]] * J[i][act[a]]; scale[a] = 1.0 / (1.0 + sqrt(cn)); }
      if (s.x_is_new) for (int a = 0; a < na; ++a) { double cn = 0; for (int i = 0; i < 4; ++i) cn += J[i][act[a]] * J[i][act[a]] * scale[a] * scale[a]; diag[a] = fmin(fmax(cn, 1e-6), 1e32); }
      double A[4][4], b[4];
      for (int a = 0; a < na; ++a) { b[a] = 0; for (int i = 0; i < 4; ++i) b[a] += J[i][act[a]] * scale[a] * r[i];
        for (int c = 0; c < na; ++c) { A[a][c] = 0; for (int i = 0; i < 4; ++i) A[a][c] += J[i][act[a]] * scale[a] * J[i][act[c]] * scale[c]; }
        A[a][a] += diag[a] / s.radius; }
      bool ok = solve4(A, b, na);
      double xc[4] = {x[0], x[1], x[2], x[3]}, mcc = 0, st2 = 0, cx2 = 0, cc = 0;
      if (ok) {
        double Js[4] = {0, 0, 0, 0};
        for (int a = 0; a < na; ++a) { double d = -b[a] * scale[a]; xc[act[a]] = x[act[a]] + d; st2 += d * d; for (int i = 0; i < 4; ++i) Js[i] += J[i][act[a]] * d; }
        for (int i = 0; i < 4; ++i) mcc -= Js[i] * (r[i] + 0.5 * Js[i]);
        for (int a = 0; a < na; ++a) cx2 += xc[act[a]] * xc[act[a]];
        double rc[4], Jc[4][4]; eval(xc, rc, Jc); for (int i = 0; i < 4; ++i) cc += 0.5 * rc[i] * rc[i];
      }
      lmctl::Action act_ = lmctl::end_iteration(s, cost, cc, mcc, st2, cx2, gmax, !ok, 1e-26);
      if (act_ == lmctl::ACT_CONTINUE_ACCEPTED) for (int k = 0; k < 4; ++k) x[k] = xc[k];
      if (act_ == lmctl::ACT_STOP) break;
    }
    for (int k = 0; k < 4; ++k) worst = fmax(worst, fabs(x[k]));
    if (s.iteration > worst_iters) worst_iters = s.iteration;
  }
  printf("%%.6g %%d\n", worst, worst_iters);
  return worst < 1e-3 ? 0 : 1;
}''' % ROOT)
    exe = tmp_path / "powell"
    subprocess.check_call(["g++", "-O2", "-o", str(exe), str(src)])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout
    worst, iters = out.stdout.split()
    assert float(worst) < 1e-3 and int(iters) <= 50


def test_brief_table_extractor_parses_generated_32_format():
    """scripts/brief_table_from_contrib.py (the one step a contrib build needs for BRIEF-32): a file in generated_32.i's format
    comes back as the int8[256][4] table in test order, and a file whose shifts break the bit-order assumption is refused."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("brief_tab", str(ROOT / "scripts" / "brief_table_from_contrib.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    rng = np.random.default_rng(0)
    t = rng.integers(-24, 25, (256, 4))
    lines = []
    for i in range(32):
        terms = " + ".join("((SMOOTHED(%d, %d) < SMOOTHED(%d, %d)) << %d)" % (*t[i * 8 + k], 7 - k) for k in range(8))
        lines.append("    desc[%d] = (uchar)(%s);" % (i, terms))
    txt = "\n".join(lines)
    assert np.array_equal(mod.parse(txt), t.astype(np.int8))
    with pytest.raises(SystemExit):
        mod.parse(txt.replace("<< 7)", "<< 6)", 1))


def test_fast_sweep_refuses_no_geometry_the_two_kernel_sweep_ran():
    """Grid FAST's sweep used to pick between a wavefront kernel (when its shared memory was at most 200 KB) and a one-warp
    kernel (at most 227 KB); both formulas are kept here as they were.  Every geometry either of them ran, the one
    wavefront kernel runs, and every geometry the old wavefront kernel ran keeps its warp count (cells 8 to 128, images up
    to 4096 x 4096)."""
    from test_detect_paths_gpu import _cell_cap, _fast_sweep_warps
    ws = np.arange(8, 4097, 5)[:, None]
    for cs in range(8, 129):
        w = ws[ws >= cs][:, None]
        h = w.T
        nwc, nhc = w // cs, h // cs
        wpr = (w + 31) // 32
        cap = _cell_cap(cs)
        old_nw = np.minimum(nhc, 16)
        wave = ((((h * wpr + 1) & ~1) * 4 + nwc * nhc * 8 + old_nw * min(cap, 128) * 4 + nhc * 4 + (nhc + 1) * (nwc + 1) + 15)
                & ~15) <= 200 * 1024
        seq = ((h * wpr * 4 + cap * 4 + (nhc + 1) * (nwc + 1) + 15) & ~15) <= 227 * 1024
        nw = _fast_sweep_warps(w, h, cs)
        assert (nw > 0)[wave | seq].all(), cs
        assert (nw == old_nw)[wave].all(), cs
