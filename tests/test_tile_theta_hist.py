"""The bucket and edge mapping of k_tile's running threshold (th_hist_bucket / th_hist_edge in tq_layout.h), compiled on the host
from the header the kernel uses: for every base that matters (none yet, small, the benchmark's, near the top of the key space) and
keys of every key >> 16 value with low halves 0, 1 and 0xFFFF, edge(bucket(key)) <= key, bucket and edge never decrease, buckets
stay in [0, 2048), keys at or below the base land in bucket 0 (edge 0) and keys above the window in the top bucket."""
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tantivy_b200", "csrc")

_SRC = r"""
#include "tq_layout.h"
#include <cstdio>
using namespace tq;
int main() {
  const uint32_t bases[] = {0u, 1u, 0x8000u, 0xBD80u, 0xC0A3u, 0xFFF0u, 0xFFFFu};
  unsigned long long bad_edge = 0, bad_mono = 0, bad_range = 0, bad_low = 0, bad_top = 0, n = 0;
  for (uint32_t bw : bases) {
    const uint32_t base = th_hist_base(bw);
    uint32_t prev_b = 0, prev_e = 0;
    for (uint32_t hi = 0; hi <= 0xFFFFu; ++hi)
      for (uint32_t lo : {0u, 1u, 0xFFFFu}) {
        const uint32_t key = hi << 16 | lo, b = th_hist_bucket(key, base), e = th_hist_edge(b, base);
        ++n;
        bad_edge += e > key;
        bad_mono += b < prev_b || e < prev_e;
        bad_range += b >= kThHistFine;
        bad_low += hi <= base && (b != 0u || e != 0u);
        bad_top += hi >= base + kThHistFine - 1u && b != kThHistFine - 1u;
        prev_b = b; prev_e = e;
      }
    for (uint32_t b = 1; b < kThHistFine; ++b) bad_mono += th_hist_edge(b, base) < th_hist_edge(b - 1u, base);
  }
  printf("%llu %llu %llu %llu %llu %llu %u %u %u\n", n, bad_edge, bad_mono, bad_range, bad_low, bad_top, th_hist_base(0u),
         th_hist_bucket(0xBF800000u, 0xBF00u), th_hist_edge(3u, 0xBF00u));
}
"""


def _cuda_include():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), "include")


def test_bucket_and_edge_mapping(tmp_path):
    src = tmp_path / "th_hist.cpp"
    src.write_text(_SRC)
    exe = tmp_path / "th_hist"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", CSRC, "-I", _cuda_include(), "-o", str(exe), str(src)])
    n, bad_edge, bad_mono, bad_range, bad_low, bad_top, fallback, b_one, e_three = (int(x) for x in subprocess.check_output([str(exe)]).split())
    assert n == 7 * 65536 * 3
    assert (bad_edge, bad_mono, bad_range, bad_low, bad_top) == (0, 0, 0, 0, 0)
    assert fallback == 0xBD80  # no threshold yet: the window starts at 2^-4 (score key 0xBD800000)
    assert b_one == 0x80 and e_three == 0xBF03 << 16  # 1.0f is 128 buckets (one binade) above the key of 0.5f
