"""CPU test of the any-window KLT lane code (ov2slam_b200/csrc/klt_setup.cuh, win_*), which fb_klt_win_kernel runs for
every window size from 3 to 31 but 9: compiled for the host, run lane by lane, and checked against the definition
(reflect-101 neighbourhood, Scharr with zero planes outside the image, OpenCV's fixed-point bilinear template, the
iterations' mismatch sums) for every window size, on random images and window origins inside, across and past every
border."""
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]


def test_klt_any_window_lane_code_matches_definition(tmp_path):
    src = tmp_path / "w.cpp"
    src.write_text(r'''
#include "%s/ov2slam_b200/csrc/klt_setup.cuh"
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>
using namespace kltsetup;
int main() {
  std::mt19937 rng(5); long bad = 0, n_int = 0, n_brd = 0;
  for (int it = 0; it < 6000; ++it) {
    const int win = 3 + it %% 29;
    int lw = 4 + rng() %% 70, lh = 4 + rng() %% 60;
    int pitch = lw + rng() %% 5;
    std::vector<uint8_t> img((size_t)pitch * lh);
    for (auto& v : img) v = (uint8_t)(rng() >> 7);
    if (it %% 7 == 0) for (auto& v : img) v = (rng() & 1) ? 255 : 0;        // extreme gradients
    int ix = (int)(rng() %% (lw + 2 * win)) - win - win / 2, iy = (int)(rng() %% (lh + 2 * win)) - win - win / 2;
    if (it %% 3 == 0 && lw > win + 3 && lh > win + 3) { ix = 1 + rng() %% (lw - win - 2); iy = 1 + rng() %% (lh - win - 2); }
    (ix >= 1 && iy >= 1 && ix + win + 2 <= lw && iy + win + 2 <= lh ? n_int : n_brd)++;
    float a = (rng() %% 1000) / 1000.f, b = (rng() %% 1000) / 1000.f;
    int iw00 = (int)((1.f - a) * (1.f - b) * 16384.f + .5f), iw01 = (int)(a * (1.f - b) * 16384.f + .5f),
        iw10 = (int)((1.f - a) * b * 16384.f + .5f), iw11 = 16384 - iw00 - iw01 - iw10;
    if (it %% 50 == 0) { iw11 = -1; iw00 += 1; }
    auto P = [&](int y, int x) { return (int)img[(size_t)reflect101_any(y, lh) * pitch + reflect101_any(x, lw)]; };
    uint8_t sN[WN_BYTES]; int sD[WD_INTS], sG[WT_ELEMS]; short sI[WT_ELEMS];
    memset(sN, 0xCD, sizeof sN); memset(sD, 0x5A, sizeof sD);
    for (int l = 0; l < 32; ++l) win_stage(l, img.data(), pitch, lw, lh, ix - 1, iy - 1, win + 3, sN);
    for (int r = 0; r < win + 3; ++r) for (int c = 0; c < win + 3; ++c) if (sN[r * WN_PITCH + c] != P(iy - 1 + r, ix - 1 + c)) bad++;
    for (int l = 0; l < 32; ++l) win_scharr(l, sN, ix, iy, lw, lh, win, sD);
    std::vector<int> dxr((win + 1) * (win + 1)), dyr((win + 1) * (win + 1));
    for (int r = 0; r <= win; ++r) for (int c = 0; c <= win; ++c) {
      int y = iy + r, x = ix + c, dx = 0, dy = 0;
      if (x >= 0 && x < lw && y >= 0 && y < lh) {
        dx = (P(y - 1, x + 1) + P(y + 1, x + 1)) * 3 + P(y, x + 1) * 10 - ((P(y - 1, x - 1) + P(y + 1, x - 1)) * 3 + P(y, x - 1) * 10);
        dy = ((P(y + 1, x - 1) - P(y - 1, x - 1)) + (P(y + 1, x + 1) - P(y - 1, x + 1))) * 3 + (P(y + 1, x) - P(y - 1, x)) * 10;
      }
      dxr[r * (win + 1) + c] = dx; dyr[r * (win + 1) + c] = dy;
      int v = sD[r * WG_PITCH + c];
      if ((int)(short)(v & 0xFFFF) != dx || (v >> 16) != dy) bad++;
    }
    long A11 = 0, A12 = 0, A22 = 0, g11 = 0, g12 = 0, g22 = 0;
    std::vector<int> Ir(win * win), Xr(win * win), Yr(win * win);
    for (int l = 0; l < 32; ++l) {
      int s11, s12, s22;
      win_template(l, sN, sD, win, iw00, iw01, iw10, iw11, sI, sG, s11, s12, s22);
      g11 += s11; g12 += s12; g22 += s22;
    }
    auto D = [&](const std::vector<int>& d, int r, int c) { return d[r * (win + 1) + c]; };
    for (int r = 0; r < win; ++r) for (int c = 0; c < win; ++c) {
      int iv = (P(iy + r, ix + c) * iw00 + P(iy + r, ix + c + 1) * iw01 + P(iy + r + 1, ix + c) * iw10 + P(iy + r + 1, ix + c + 1) * iw11 + 256) >> 9;
      int ixv = (D(dxr, r, c) * iw00 + D(dxr, r, c + 1) * iw01 + D(dxr, r + 1, c) * iw10 + D(dxr, r + 1, c + 1) * iw11 + 8192) >> 14;
      int iyv = (D(dyr, r, c) * iw00 + D(dyr, r, c + 1) * iw01 + D(dyr, r + 1, c) * iw10 + D(dyr, r + 1, c + 1) * iw11 + 8192) >> 14;
      Ir[r * win + c] = iv; Xr[r * win + c] = ixv; Yr[r * win + c] = iyv;
      int g = sG[r * WG_PITCH + c];
      if (sI[r * WG_PITCH + c] != (short)iv || (int)(short)(g & 0xFFFF) != ixv || (g >> 16) != iyv) bad++;
      A11 += (long)ixv * ixv; A12 += (long)ixv * iyv; A22 += (long)iyv * iyv;
    }
    if (A11 != g11 || A12 != g12 || A22 != g22) bad++;
    // one iteration: search origin anywhere the kernel admits it, new sub-pixel weights
    int jx = (int)(rng() %% (lw + win)) - win, jy = (int)(rng() %% (lh + win)) - win;
    float a2 = (rng() %% 1000) / 1000.f, b2 = (rng() %% 1000) / 1000.f;
    int jw00 = (int)((1.f - a2) * (1.f - b2) * 16384.f + .5f), jw01 = (int)(a2 * (1.f - b2) * 16384.f + .5f),
        jw10 = (int)((1.f - a2) * b2 * 16384.f + .5f), jw11 = 16384 - jw00 - jw01 - jw10;
    for (int l = 0; l < 32; ++l) win_stage(l, img.data(), pitch, lw, lh, jx, jy, win + 1, sN);
    long B1 = 0, B2 = 0, h1 = 0, h2 = 0;
    for (int r = 0; r < win; ++r) for (int c = 0; c < win; ++c) {
      int jv = (P(jy + r, jx + c) * jw00 + P(jy + r, jx + c + 1) * jw01 + P(jy + r + 1, jx + c) * jw10 + P(jy + r + 1, jx + c + 1) * jw11 + 256) >> 9;
      long d = jv - Ir[r * win + c];
      B1 += d * Xr[r * win + c]; B2 += d * Yr[r * win + c];
    }
    for (int l = 0; l < 32; ++l) {
      int s1, s2;
      win_mismatch(l, sN, sI, sG, win, jw00, jw01, jw10, jw11, s1, s2);
      if (l >= win && (s1 || s2)) bad++;
      h1 += s1; h2 += s2;
    }
    if (B1 != h1 || B2 != h2) bad++;
  }
  printf("%%ld bad, %%ld interior, %%ld border\n", bad, n_int, n_brd);
  return (bad || n_int < 1000 || n_brd < 1000) ? 1 : 0;
}''' % ROOT)
    exe = tmp_path / "w"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", str(exe), str(src)])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
