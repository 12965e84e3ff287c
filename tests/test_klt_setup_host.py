"""CPU tests of the KLT level set-up code in ov2slam_b200/csrc/klt_setup.cuh compiled for the host: the int-output template
functions and the split staging that fb_klt_kernel calls, lane by lane against the definition, and the host thresholds that
replace the trackers' minEig division and forward-backward square root, decision by decision against the expressions they
replace."""
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]


def _run(tmp_path, name, code):
    src = tmp_path / (name + ".cpp")
    src.write_text(code.replace("@ROOT@", str(ROOT)))
    exe = tmp_path / name
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", str(exe), str(src)])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    return out.stdout


def test_klt_thresholds_decide_as_the_division_and_sqrt(tmp_path):
    """q < klt_eig_q(win, T) <=> q / (2 win^2) < T, q > klt_ferr_q(win, ferr) <=> q / (2 win^2) > ferr and
    s > klt_fb_s(fb) <=> sqrt(s) > fb, for every win from 3 to 31, ferr / fb_dist of 30, 0.5, 0, -0, negative, +-inf, NaN and
    random ones, on every float / double within 3000 ULPs of each threshold and random values over the whole range."""
    out = _run(tmp_path, "thr", r'''
#include "@ROOT@/ov2slam_b200/csrc/klt_setup.cuh"
#include <cmath>
#include <cstdio>
#include <limits>
#include <random>
#include <vector>
using namespace kltsetup;
static float fbits(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static double dbits(uint64_t u) { double f; memcpy(&f, &u, 8); return f; }
static uint32_t bitsf(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static uint64_t bitsd(double f) { uint64_t u; memcpy(&u, &f, 8); return u; }
// the floats k ULPs around x in increasing order (crossing zero and the infinities' neighbours)
static float fstep(float x, long k) {
  long long key = (long long)(bitsf(x) & 0x7fffffffu) * ((bitsf(x) >> 31) ? -1 : 1) + k;
  if (key > 0x7f800000LL) key = 0x7f800000LL;
  if (key < -0x7f800000LL) key = -0x7f800000LL;
  return key >= 0 ? fbits((uint32_t)key) : fbits(0x80000000u | (uint32_t)(-key));
}
int main() {
  const float inf = std::numeric_limits<float>::infinity(), nan = std::numeric_limits<float>::quiet_NaN();
  std::mt19937_64 rng(5);
  std::vector<float> vals = {30.f, 0.5f, 0.f, -0.f, -1.f, -30.f, inf, -inf, nan, 0x1.a36e3p-14f, 1e-30f, 3e38f,
                             std::numeric_limits<float>::denorm_min(), std::numeric_limits<float>::max()};
  for (int i = 0; i < 20; ++i) vals.push_back(std::ldexp((float)(rng() % 100000) / 1000.f, (int)(rng() % 40) - 20));
  for (int i = 0; i < 4; ++i) vals.push_back(fbits((uint32_t)rng()));
  long bad = 0, checks = 0;
  auto probe_f = [&](float q, float d, float Q, float G, float ferr) {
    if ((q / d < 0x1.a36e3p-14f) != (q < Q)) bad++;
    if ((q / d > ferr) != (q > G)) bad++;
    checks++;
  };
  for (int win = 3; win <= 31; ++win) {
    const float d = (float)(2 * win * win);
    const float Q = klt_eig_q(win, 0x1.a36e3p-14f);
    for (float ferr : vals) {
      const float G = klt_ferr_q(win, ferr);
      std::vector<float> qs = {0.f, -0.f, inf, -inf, nan, 1.f, -1.f};
      for (long k = -3000; k <= 3000; ++k) { qs.push_back(fstep(Q, k)); qs.push_back(fstep(G, k)); qs.push_back(fstep(0.f, k)); }
      for (int i = 0; i < 20000; ++i) qs.push_back(fbits((uint32_t)rng()));
      for (int i = 0; i < 20000; ++i) qs.push_back(std::ldexp((float)(rng() % 1000000) / 1000.f, (int)(rng() % 30) - 20));
      for (float q : qs) probe_f(q, d, Q, G, ferr);
    }
  }
  for (float fb : vals) {
    const double S = klt_fb_s(fb);
    std::vector<double> ss = {0.0, std::numeric_limits<double>::infinity(), std::numeric_limits<double>::quiet_NaN()};
    const double bases[] = {S, 0.0, (double)fb * (double)fb};
    for (double b : bases) {
      if (!(b >= 0.0) || std::isinf(b)) continue;
      const uint64_t u = bitsd(b);
      for (long k = -3000; k <= 3000; ++k) if ((long long)u + k >= 0) ss.push_back(dbits(u + k));
    }
    for (int i = 0; i < 50000; ++i) ss.push_back(dbits(rng() & 0x7fffffffffffffffULL));
    for (int i = 0; i < 50000; ++i) {
      const float dx = (float)((long)(rng() % 2000001) - 1000000) / 1000.f, dy = (float)((long)(rng() % 2001) - 1000) / 1000.f;
      ss.push_back((double)dx * (double)dx + (double)dy * (double)dy);
    }
    for (double s : ss) {
      if ((std::sqrt(s) > (double)fb) != (s > S)) bad++;
      checks++;
    }
  }
  printf("%ld bad of %ld\n", bad, checks);
  return bad ? 1 : 0;
}''')
    assert out.startswith("0 bad")


def test_klt_setup_int_lane_code_matches_definition(tmp_path):
    """stage_interior / stage_border and the int-output template_direct / template_rows (the functions fb_klt_kernel calls),
    lane by lane, against the definition (reflect-101 neighbourhood, Scharr with zero planes outside the image, OpenCV's
    fixed-point bilinear template as sign-extended int16) on random images and window positions: interior, every border,
    word-aligned and unaligned rows."""
    _run(tmp_path, "lane", r'''
#include "@ROOT@/ov2slam_b200/csrc/klt_setup.cuh"
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>
using namespace kltsetup;
int main() {
  std::mt19937 rng(23); long bad = 0, n_int = 0, n_brd = 0;
  for (int it = 0; it < 20000; ++it) {
    int lw = 14 + rng() % 50, lh = 14 + rng() % 40;
    bool al = rng() % 4 != 0;
    int pitch = al ? ((lw + 3) & ~3) + 4 * (rng() % 3) : lw + (rng() % 3);
    // the image ends exactly at its last row's pitch: a staged word past the buffer would be read outside it
    std::vector<uint32_t> store((size_t)(pitch * lh + 8) / 4 + 2);
    uint8_t* img = reinterpret_cast<uint8_t*>(store.data()) + (al ? 0 : 1 + rng() % 3);
    for (int i = 0; i < pitch * lh; ++i) img[i] = (uint8_t)(rng() >> 7);
    bool aligned = ((reinterpret_cast<uintptr_t>(img) | (uintptr_t)pitch) & 3) == 0;
    int ix = (int)(rng() % (lw + WIN)) - WIN, iy = (int)(rng() % (lh + WIN)) - WIN;
    if (it % 3 == 0) { ix = 1 + rng() % (lw - 11); iy = 1 + rng() % (lh - 11); }
    if (it % 7 == 0) { ix = lw - 11; iy = lh - 11; }                 // the last interior origin
    const bool interior = aligned && patch_interior(ix, iy, lw, lh);
    (interior ? n_int : n_brd)++;
    float a = (rng() % 1000) / 1000.f, b = (rng() % 1000) / 1000.f;
    int iw00 = (int)((1.f - a) * (1.f - b) * 16384.f + .5f), iw01 = (int)(a * (1.f - b) * 16384.f + .5f),
        iw10 = (int)((1.f - a) * b * 16384.f + .5f), iw11 = 16384 - iw00 - iw01 - iw10;
    if (it % 50 == 0) { iw11 = -1; iw00 += 1; }
    alignas(16) uint8_t sP[SP_BYTES]; int sD[SD_INTS];
    memset(sP, 0xCD, sizeof sP); memset(sD, 0x5A, sizeof sD);
    const int off = interior ? (ix - 1) & 3 : 0;
    for (int l = 0; l < 32; ++l) {
      if (interior) stage_interior(l, img, pitch, lw, ix, iy, sP);
      else stage_border(l, img, pitch, lw, lh, ix, iy, sP);
    }
    auto P = [&](int r, int c) {
      return (int)img[(size_t)reflect101_any(iy - 1 + r, lh) * pitch + reflect101_any(ix - 1 + c, lw)];
    };
    for (int r = 0; r < PW; ++r) for (int c = 0; c < PW; ++c) if (sP[r * SP_PITCH + off + c] != P(r, c)) bad++;
    int dxr[DW][DW], dyr[DW][DW];
    for (int r = 0; r < DW; ++r) for (int c = 0; c < DW; ++c) {
      int y = iy + r, x = ix + c, dx = 0, dy = 0;
      if (x >= 0 && x < lw && y >= 0 && y < lh) {
        dx = (P(r, c + 2) + P(r + 2, c + 2)) * 3 + P(r + 1, c + 2) * 10 - ((P(r, c) + P(r + 2, c)) * 3 + P(r + 1, c) * 10);
        dy = ((P(r + 2, c) - P(r, c)) + (P(r + 2, c + 2) - P(r, c + 2))) * 3 + (P(r + 2, c + 1) - P(r, c + 1)) * 10;
      }
      dxr[r][c] = dx; dyr[r][c] = dy;
    }
    if (!interior) for (int l = 0; l < 32; ++l) scharr_rows(l, sP, off, ix, iy, lw, lh, sD);
    long g11 = 0, g12 = 0, g22 = 0, A11 = 0, A12 = 0, A22 = 0;
    for (int l = 0; l < 32; ++l) {
      int Iv[3], Ix[3], Iy[3], s11, s12, s22;
      if (interior) template_direct(l, sP, off, iw00, iw01, iw10, iw11, Iv, Ix, Iy, s11, s12, s22);
      else template_rows(l, sP, off, sD, iw00, iw01, iw10, iw11, Iv, Ix, Iy, s11, s12, s22);
      g11 += s11; g12 += s12; g22 += s22;
      for (int k = 0; k < 3; ++k) {
        int p = 3 * l + k;
        if (p >= WIN * WIN) { if (Iv[k] || Ix[k] || Iy[k]) bad++; continue; }
        int y = p / WIN, x = p % WIN;
        int iv = (P(y + 1, x + 1) * iw00 + P(y + 1, x + 2) * iw01 + P(y + 2, x + 1) * iw10 + P(y + 2, x + 2) * iw11 + 256) >> 9;
        int ixv = (dxr[y][x] * iw00 + dxr[y][x + 1] * iw01 + dxr[y + 1][x] * iw10 + dxr[y + 1][x + 1] * iw11 + 8192) >> 14;
        int iyv = (dyr[y][x] * iw00 + dyr[y][x + 1] * iw01 + dyr[y + 1][x] * iw10 + dyr[y + 1][x + 1] * iw11 + 8192) >> 14;
        // OpenCV keeps int16: the int outputs are those values sign-extended
        if (Iv[k] != (int)(short)iv || Ix[k] != (int)(short)ixv || Iy[k] != (int)(short)iyv) bad++;
        if (iv != (short)iv || ixv != (short)ixv || iyv != (short)iyv) bad++;
        A11 += (long)ixv * ixv; A12 += (long)ixv * iyv; A22 += (long)iyv * iyv;
      }
    }
    if (A11 != g11 || A12 != g12 || A22 != g22) bad++;
  }
  printf("%ld bad, %ld interior, %ld border\n", bad, n_int, n_brd);
  return (bad || n_int < 1000 || n_brd < 1000) ? 1 : 0;
}''')
