"""ov2sort::sort_desc_front (ov2slam_b200/csrc/stdsort_emul.h): the element std::sort leaves first, found by following
only the leftmost chain of introsort partitions.  Compiled for the host and compared with the real std::sort on the
inputs tests/test_host_logic.py uses for sort_desc: tie-heavy responses, ramps and saw-tooth orders, lengths up to 2 100
(deep partition chains), plus organ-pipe orders that drive introsort to its depth limit and the heapsort fallback."""
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def test_sort_desc_front_matches_std_sort(tmp_path):
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
  std::mt19937 rng(11); long bad = 0, nlong = 0;
  for (int it = 0; it < 60000; ++it) {
    int n = 1 + rng() %% (it %% 4 ? 200 : 2100), nv = 1 + rng() %% (it %% 3 ? 6 : 40), pat = rng() %% 4;
    nlong += n > 1891;
    std::vector<Kp> v(n); std::vector<int> k(n);
    for (int i = 0; i < n; ++i) {
      int r = pat == 1 ? i %% nv : pat == 2 ? (n - i) / (1 + (int)(rng() %% 3)) : pat == 3 ? (i < n / 2 ? i : n - i) : (int)(rng() %% nv);
      r = 20 + r %% 235;
      v[i] = {(float)r, i}; k[i] = (r << 16) | i; }
    std::sort(v.begin(), v.end(), cmp);
    if ((ov2sort::sort_desc_front(k.data(), n) & 0xFFFF) != v[0].idx) bad++;
  }
  printf("%%ld %%ld\n", bad, nlong); return (bad || nlong < 1000) ? 1 : 0;
}''' % ROOT)
    exe = tmp_path / "t"
    subprocess.check_call(["g++", "-O2", "-o", str(exe), str(src)])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout
