"""Host-side check of the balanced bulk launch: `bulk_build_jobs` (starway_b200/csrc/bulk_jobs.h) and the
per-CTA byte-range iterator `SwJobRangeIter` (sw_device.h) that the sm_90a kernel
`sw_bulk_tma_jobs_kernel` runs unchanged.  A C++ harness (compiled here with g++) replays every CTA of
randomized launches on the CPU and checks: every byte copied exactly once, pieces 16-byte aligned,
within one job, at most stage_bytes long, grid <= max CTAs, shares equal within 1 KiB."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HARNESS = r"""
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <random>
#include <vector>
#include "starway_b200/csrc/bulk_jobs.h"
using namespace swgpu;
int main() {
  std::mt19937_64 rng(0xB200);
  int launches = 0, fallbacks = 0;
  for (int iter = 0; iter < 1500; iter++) {
    // a launch: some messages, each cut into segments the way the engine does
    const int nmsg = 1 + (int)(rng() % (iter % 7 == 0 ? 400 : 70));
    const uint64_t seg = 1024ull * (4 + rng() % 128);
    std::vector<uint8_t> src_mem, dst_mem;
    std::vector<SwSeg> segs;
    std::vector<std::pair<uint64_t, uint64_t>> msgs;   // (offset, len) in the arenas
    uint64_t arena = 0;
    for (int m = 0; m < nmsg; m++) {
      uint64_t len = 16 * (1 + rng() % (iter % 25 == 0 ? 60000 : 1500));
      if (rng() % 9 == 0) len = 16 * (1 + rng() % 4);
      const uint64_t gap = (rng() % 3 == 0) ? 0 : 16 * (rng() % 64);   // gap 0: adjacent messages merge into one job
      arena += gap;
      msgs.push_back({arena, len});
      arena += len;
    }
    src_mem.resize(arena + 64);
    dst_mem.assign(arena + 64, 0);
    { uint64_t x = rng(); for (auto& b : src_mem) { x = x * 6364136223846793005ull + 1442695040888963407ull; b = (uint8_t)(x >> 56); } }
    std::vector<uint32_t> hits(arena + 64, 0);
    const uint64_t sbase = (uint64_t)(uintptr_t)src_mem.data(), dbase = (uint64_t)(uintptr_t)dst_mem.data();
    const uint64_t sal = (16 - (sbase & 15)) & 15, dal = (16 - (dbase & 15)) & 15;
    uint64_t total = 0;
    for (auto& m : msgs) {
      for (uint64_t off = 0; off < m.second; off += seg)
        segs.push_back(SwSeg{sbase + sal + m.first + off, dbase + dal + m.first + off, std::min(seg, m.second - off), 0});
      total += m.second;
    }
    if (iter % 11 == 0 && !segs.empty()) segs.insert(segs.begin() + rng() % segs.size(), SwSeg{0, 0, 0, 0});  // empty segment
    const uint32_t stage = 16 * (64 + rng() % 1536), max_ctas = 1 + rng() % 296;
    SwBulkJobArgs a;
    uint32_t grid = 0;
    if (!bulk_build_jobs(segs.data(), (uint32_t)segs.size(), max_ctas, stage, 8, &a, &grid)) {
      fallbacks++;
      continue;
    }
    launches++;
    if (grid == 0 || grid > max_ctas || a.njobs == 0 || a.njobs > SW_BULK_INLINE_JOBS || (a.share & 1023) ||
        a.end[a.njobs - 1] != total || (uint64_t)grid * a.share < total || (uint64_t)(grid - 1) * a.share >= total) {
      printf("FAIL header iter %d grid %u max %u njobs %u share %llu total %llu\n", iter, grid, max_ctas, a.njobs,
             (unsigned long long)a.share, (unsigned long long)total);
      return 1;
    }
    for (uint32_t cta = 0; cta < grid; cta++) {
      SwJobRangeIter it;
      it.init(a, cta);
      uint64_t s, d, mine = 0;
      uint32_t n;
      while (it.next(a, s, d, n)) {
        if (((s | d | n) & 15) || n == 0 || n > stage) { printf("FAIL piece iter %d\n", iter); return 1; }
        if (s - (sbase + sal) != d - (dbase + dal)) { printf("FAIL src/dst skew iter %d\n", iter); return 1; }
        const uint64_t off = d - (dbase + dal);
        if (off + n > arena) { printf("FAIL range iter %d\n", iter); return 1; }
        memcpy((void*)(uintptr_t)d, (const void*)(uintptr_t)s, n);
        for (uint32_t k = 0; k < n; k += 16) hits[off + k]++;
        mine += n;
      }
      if (mine > a.share) { printf("FAIL share iter %d\n", iter); return 1; }
    }
    for (auto& m : msgs) {
      if (memcmp(src_mem.data() + sal + m.first, dst_mem.data() + dal + m.first, m.second)) { printf("FAIL bytes iter %d\n", iter); return 1; }
      for (uint64_t k = 0; k < m.second; k += 16)
        if (hits[m.first + k] != 1) { printf("FAIL coverage iter %d\n", iter); return 1; }
    }
  }
  printf("OK launches=%d fallbacks=%d\n", launches, fallbacks);
  return launches > 800 && fallbacks > 10 ? 0 : 2;
}
"""


def test_job_range_iterator_covers_every_launch_exactly_once(tmp_path):
    src = tmp_path / "harness.cpp"
    src.write_text(HARNESS)
    exe = tmp_path / "harness"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", ROOT, "-o", str(exe), str(src)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.startswith("OK"), out.stdout
