// tests/gpu_probe/probe.cu — GPU-side unit tests and micro-benchmarks for the starway_b200
// kernels (TEST INFRASTRUCTURE).  Needs a GPU (built for sm_90a by `make probe`):
//   sw_probe correctness           bulk-copy parity (TMA and SIMT kernels, aligned and unaligned segments)
//   sw_probe bench                 single-GPU bulk copy bandwidth sweep (TMA vs SIMT tunings)
//   sw_probe peer                  2-GPU in-process peer pull/push bandwidth, cudaMemcpyPeer ceiling
//   sw_probe ipc                   2-process CUDA-IPC mapping check + pull bandwidth
//   sw_probe latency               launch + completion-poll latency of the put kernels
//   sw_probe balance               bulk copy of n x 1 MiB messages: segment-list kernel vs balanced job-range kernel
//   sw_probe floor                 launch -> completion-seen floor: event vs flag in pinned memory
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/wait.h>
#include <unistd.h>
#include <algorithm>
#include <chrono>
#include <random>
#include <string>
#include <vector>

#include "../../starway_b200/csrc/gpu.h"

using namespace swgpu;

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e__ = (call);                                                                      \
    if (e__ != cudaSuccess) {                                                                      \
      fprintf(stderr, "CUDA error %s at %s:%d: %s\n", #call, __FILE__, __LINE__, cudaGetErrorString(e__)); \
      exit(2);                                                                                     \
    }                                                                                              \
  } while (0)
#define REQ(cond)                                                          \
  do {                                                                     \
    if (!(cond)) {                                                         \
      fprintf(stderr, "FAILED: %s at %s:%d (%s)\n", #cond, __FILE__, __LINE__, last_error()); \
      exit(3);                                                             \
    }                                                                      \
  } while (0)

static double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// ------------------------------------------------------------------ bulk helpers
static std::vector<SwSeg> make_segs(uint64_t src, uint64_t dst, uint64_t len, uint64_t seg_bytes) {
  std::vector<SwSeg> v;
  for (uint64_t off = 0; off < len; off += seg_bytes) {
    SwSeg s;
    s.src = src + off;
    s.dst = dst + off;
    s.len = std::min(seg_bytes, len - off);
    s.pad = 0;
    v.push_back(s);
  }
  return v;
}

static float time_bulk(stream_t st, const SwSeg* segs_pinned, uint32_t nseg, const BulkTuning& t, int iters,
                       void* flush, size_t flush_bytes) {
  event_t a = event_create(1), b = event_create(1);
  float best = 1e30f;
  for (int i = 0; i < iters + 2; i++) {
    if (flush) CK(cudaMemsetAsync(flush, i, flush_bytes, (cudaStream_t)st));
    event_record(a, st);
    REQ(launch_bulk(st, segs_pinned, nseg, &t) == 0);
    event_record(b, st);
    REQ(event_sync(b) == 0);
    float ms = event_elapsed_ms(a, b);
    if (i >= 2 && ms < best) best = ms;
  }
  event_destroy(a);
  event_destroy(b);
  return best;
}

static void fill_pattern(std::vector<uint8_t>& v, uint32_t seed) {
  uint32_t x = seed * 2654435761u + 12345u;
  for (size_t i = 0; i < v.size(); i++) {
    x = x * 1664525u + 1013904223u;
    v[i] = (uint8_t)(x >> 24);
  }
}

static void test_bulk_correctness() {
  printf("[bulk] correctness\n");
  stream_t st = stream_create();
  const size_t POOL = 96u << 20;
  uint8_t *src = (uint8_t*)dev_alloc(POOL), *dst = (uint8_t*)dev_alloc(POOL);
  REQ(src && dst);
  std::vector<uint8_t> hsrc(POOL), hdst(POOL), ref(POOL);
  fill_pattern(hsrc, 7);
  CK(cudaMemcpy(src, hsrc.data(), POOL, cudaMemcpyHostToDevice));
  SwSeg* segs = (SwSeg*)host_alloc(sizeof(SwSeg) * 65536);
  std::mt19937_64 rng(42);
  for (int mode = 0; mode < 2; mode++) {
    for (int trial = 0; trial < 12; trial++) {
      CK(cudaMemset(dst, 0xEE, POOL));
      std::fill(ref.begin(), ref.end(), 0xEE);
      // carve random non-overlapping jobs
      std::vector<SwSeg> all;
      size_t soff = 0, doff = 0;
      int njobs = 1 + (int)(rng() % 40);
      for (int j = 0; j < njobs; j++) {
        uint64_t len;
        switch (rng() % 6) {
          case 0: len = 16 * (1 + rng() % 8); break;
          case 1: len = 16 * (1 + rng() % 4096); break;
          case 2: len = (1 + rng() % 64) << 16; break;
          case 3: len = 1 + rng() % 5000; break;
          case 4: len = (1u << 20) + 16 * (rng() % 1000); break;
          default: len = 16 * (1 + rng() % 200000); break;
        }
        uint64_t sa = 0, da = 0;
        if (mode == 0) {
          len &= ~15ull;
          if (!len) len = 16;
        } else {
          int k = rng() % 4;  // alignment class
          sa = rng() % 16;
          da = (k == 0) ? sa : (k == 1 ? (sa + 4 * (rng() % 4)) % 16 : rng() % 16);
        }
        soff = (soff + 255) & ~255ull;
        doff = (doff + 255) & ~255ull;
        if (soff + sa + len + 256 > POOL || doff + da + len + 256 > POOL) break;
        uint64_t segb = (mode == 0) ? (uint64_t)(16 * (64 + rng() % 8192)) : (uint64_t)(1 + rng() % (1 << 20));
        if (mode == 0) segb &= ~15ull;
        auto v = make_segs((uint64_t)(src + soff + sa), (uint64_t)(dst + doff + da), len, segb);
        all.insert(all.end(), v.begin(), v.end());
        memcpy(ref.data() + doff + da, hsrc.data() + soff + sa, len);
        soff += sa + len;
        doff += da + len;
      }
      REQ(all.size() < 65536);
      memcpy(segs, all.data(), sizeof(SwSeg) * all.size());
      BulkTuning t;
      t.mode = mode;
      t.stages = 2 + (int)(rng() % 7);
      t.stage_bytes = 16 * (int)(64 + rng() % 1500);
      t.ctas_per_sm = 1 + (int)(rng() % 3);
      t.balance = trial & 1;   // odd trials: jobs as kernel parameters, equal byte range per CTA
      REQ(launch_bulk(st, segs, (uint32_t)all.size(), &t) == 0);
      REQ(stream_sync(st) == 0);
      CK(cudaMemcpy(hdst.data(), dst, POOL, cudaMemcpyDeviceToHost));
      if (memcmp(hdst.data(), ref.data(), POOL) != 0) {
        size_t i = 0;
        while (hdst[i] == ref[i]) i++;
        fprintf(stderr, "bulk mismatch mode=%d trial=%d at byte %zu (stages=%d stage_bytes=%d)\n", mode, trial, i,
                t.stages, t.stage_bytes);
        exit(4);
      }
    }
    printf("[bulk] mode %d (%s) ok\n", mode, mode == 0 ? "tma" : "simt");
  }
  host_free(segs);
  dev_free(src);
  dev_free(dst);
  stream_destroy(st);
}

// ------------------------------------------------------------------ benchmarks
static void bench_bulk_table(const char* label, uint8_t* src, uint8_t* dst, size_t maxbytes, bool peer,
                             FILE* json) {
  stream_t st = stream_create();
  SwSeg* segs = (SwSeg*)host_alloc(sizeof(SwSeg) * (1u << 16));
  const size_t FLUSH = 256u << 20;
  void* flush = dev_alloc(FLUSH);
  struct Cfg {
    int mode, stages, stage_bytes, ctas;
    uint64_t seg;
  };
  std::vector<Cfg> cfgs = {
      {0, 4, 16384, 2, 1 << 18}, {0, 4, 32768, 1, 1 << 18}, {0, 6, 32768, 1, 1 << 18}, {0, 4, 8192, 4, 1 << 17},
      {0, 3, 16384, 4, 1 << 17}, {0, 8, 24576, 1, 1 << 19}, {0, 4, 49152, 1, 1 << 19}, {1, 0, 0, 4, 1 << 16},
      {1, 0, 0, 8, 1 << 16},     {1, 0, 0, 8, 1 << 18},
  };
  std::vector<size_t> sizes = {1u << 20, 4u << 20, 16u << 20, 64u << 20, 256u << 20, 1024u << 20};
  for (size_t bytes : sizes) {
    if (bytes > maxbytes) break;
    for (auto& c : cfgs) {
      uint64_t seg = c.seg;
      while (bytes / seg > 60000) seg <<= 1;
      auto v = make_segs((uint64_t)src, (uint64_t)dst, bytes, seg);
      memcpy(segs, v.data(), v.size() * sizeof(SwSeg));
      BulkTuning t{c.mode, c.stages, c.stage_bytes, c.ctas};
      bool need_flush = !peer && bytes <= (128u << 20);
      float ms = time_bulk(st, segs, (uint32_t)v.size(), t, 5, need_flush ? flush : nullptr, FLUSH);
      double gbs = bytes / (ms * 1e-3) / 1e9;
      printf("[%s] %8.1f MiB mode=%s stages=%d stage=%6d ctas/sm=%d seg=%7llu nseg=%5zu : %8.3f ms  %8.1f GB/s payload\n",
             label, bytes / 1048576.0, c.mode ? "simt" : "tma ", c.stages, c.stage_bytes, c.ctas,
             (unsigned long long)seg, v.size(), ms, gbs);
      if (json)
        fprintf(json,
                "{\"bench\":\"%s\",\"bytes\":%zu,\"mode\":\"%s\",\"stages\":%d,\"stage_bytes\":%d,\"ctas_per_sm\":%d,"
                "\"seg\":%llu,\"ms\":%.4f,\"gbs\":%.1f}\n",
                label, bytes, c.mode ? "simt" : "tma", c.stages, c.stage_bytes, c.ctas, (unsigned long long)seg, ms,
                gbs);
    }
    // cudaMemcpyAsync reference
    {
      event_t a = event_create(1), b = event_create(1);
      float best = 1e30f;
      for (int i = 0; i < 6; i++) {
        if (!peer && bytes <= (128u << 20)) CK(cudaMemsetAsync(flush, i, FLUSH, (cudaStream_t)st));
        event_record(a, st);
        CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)st));
        event_record(b, st);
        event_sync(b);
        float ms = event_elapsed_ms(a, b);
        if (i >= 1 && ms < best) best = ms;
      }
      printf("[%s] %8.1f MiB cudaMemcpyAsync: %8.3f ms %8.1f GB/s payload\n", label, bytes / 1048576.0, best,
             bytes / (best * 1e-3) / 1e9);
      if (json)
        fprintf(json, "{\"bench\":\"%s\",\"bytes\":%zu,\"mode\":\"cudaMemcpyAsync\",\"ms\":%.4f,\"gbs\":%.1f}\n", label,
                bytes, best, bytes / (best * 1e-3) / 1e9);
      event_destroy(a);
      event_destroy(b);
    }
  }
  dev_free(flush);
  host_free(segs);
  stream_destroy(st);
}

static void bench_single(FILE* json) {
  const size_t N = 1024u << 20;
  uint8_t *a = (uint8_t*)dev_alloc(N), *b = (uint8_t*)dev_alloc(N);
  REQ(a && b);
  bench_bulk_table("loopback", a, b, N, false, json);
  dev_free(a);
  dev_free(b);
}

static void bench_peer(FILE* json) {
  int n = device_count();
  if (n < 2) {
    printf("[peer] skipped: %d device(s)\n", n);
    return;
  }
  const size_t N = 1024u << 20;
  CK(cudaSetDevice(1));
  uint8_t* remote = nullptr;
  CK(cudaMalloc(&remote, N));
  CK(cudaMemset(remote, 0x5A, N));
  CK(cudaDeviceEnablePeerAccess(0, 0));
  CK(cudaSetDevice(0));
  CK(cudaDeviceEnablePeerAccess(1, 0));
  uint8_t* local = (uint8_t*)dev_alloc(N);
  CK(cudaMemset(local, 0x11, N));
  CK(cudaDeviceSynchronize());
  bench_bulk_table("pull(remote->local)", remote, local, N, true, json);
  bench_bulk_table("push(local->remote)", local, remote, N, true, json);
  // correctness of a pull
  std::vector<uint8_t> h(1 << 20);
  CK(cudaMemcpy(h.data(), local, h.size(), cudaMemcpyDeviceToHost));
  for (auto x : h) REQ(x == 0x11 || x == 0x5A);
  dev_free(local);
  CK(cudaSetDevice(1));
  CK(cudaFree(remote));
  CK(cudaSetDevice(0));
}

static void bench_latency(FILE* json) {
  stream_t st = stream_create();
  SwPutDesc* descs = (SwPutDesc*)host_alloc(sizeof(SwPutDesc) * 1024);
  uint8_t* ring = (uint8_t*)dev_alloc(1024 * SW_SLOT_BYTES);
  uint8_t* src = (uint8_t*)dev_alloc(1 << 20);
  for (int n : {1, 64, 1024}) {
    for (int len : {64, 1024, 8128}) {
      for (int i = 0; i < n; i++) {
        descs[i].src = (uint64_t)src;
        descs[i].dst = (uint64_t)(ring + (size_t)i * SW_SLOT_BYTES);
        descs[i].tag = 1;
        descs[i].seq = i + 1;
        descs[i].len = len;
        descs[i].kind = SW_KIND_EAGER;
        descs[i].msg_len = len;
      }
      event_t ev = event_create(0);
      double best = 1e9;
      for (int it = 0; it < 50; it++) {
        double t0 = now_s();
        launch_put(st, descs, n);
        event_record(ev, st);
        while (event_query(ev) == 1) {
        }
        double t1 = now_s();
        if (it > 5) best = std::min(best, t1 - t0);
      }
      printf("[latency] put n=%4d len=%5d: launch+poll %.2f us (%.2f Mmsg/s)\n", n, len, best * 1e6, n / best / 1e6);
      if (json)
        fprintf(json, "{\"bench\":\"put_latency\",\"n\":%d,\"len\":%d,\"us\":%.2f}\n", n, len, best * 1e6);
      event_destroy(ev);
      if (n <= 32) {   // the single-CTA variant announces completion through a flag in pinned memory
        static uint64_t* flag = (uint64_t*)host_alloc(64);
        static uint64_t seq = 0;
        double bestf = 1e9;
        for (int it = 0; it < 50; it++) {
          DoneFlag df{flag, ++seq};
          double t0 = now_s();
          REQ(launch_put(st, descs, n, &df) == 1);
          while (*(volatile uint64_t*)flag != seq) {
          }
          double t1 = now_s();
          if (it > 5) bestf = std::min(bestf, t1 - t0);
        }
        printf("[latency] put n=%4d len=%5d: launch+flag %.2f us\n", n, len, bestf * 1e6);
        if (json)
          fprintf(json, "{\"bench\":\"put_latency_flag\",\"n\":%d,\"len\":%d,\"us\":%.2f}\n", n, len, bestf * 1e6);
      }
    }
  }
}

// ------------------------------------------------------------------ tuning sweep of the TMA bulk kernel
static void bench_tune(FILE* json) {
  const size_t N = 64u << 20;
  uint8_t* a = (uint8_t*)dev_alloc(N);
  uint8_t* b = (uint8_t*)dev_alloc(N);
  uint8_t* remote = nullptr;
  if (device_count() > 1) {
    CK(cudaSetDevice(1));
    CK(cudaMalloc(&remote, N));
    CK(cudaMemset(remote, 1, N));
    CK(cudaDeviceEnablePeerAccess(0, 0));
    CK(cudaSetDevice(0));
    CK(cudaDeviceEnablePeerAccess(1, 0));
  }
  stream_t st = stream_create();
  SwSeg* segs = (SwSeg*)host_alloc(sizeof(SwSeg) * 65536);
  const size_t FLUSH = 256u << 20;
  void* flush = dev_alloc(FLUSH);
  for (int where = 0; where < (remote ? 2 : 1); where++) {
    for (size_t bytes : {size_t(16) << 20, size_t(32) << 20, size_t(64) << 20}) {
      struct R { float ms; int st, sb, ct; uint64_t seg; };
      std::vector<R> res;
      for (int stages : {3, 4, 6, 8})
        for (int sb : {8192, 16384, 24576, 32768, 49152})
          for (int ctas : {1, 2, 3, 4})
            for (uint64_t seg : {uint64_t(32) << 10, uint64_t(64) << 10, uint64_t(128) << 10, uint64_t(256) << 10}) {
              if ((size_t)stages * sb * ctas > 220 * 1024) continue;
              if (seg % sb != 0 && seg > (uint64_t)sb) continue;
              auto v = make_segs((uint64_t)(where ? remote : a), (uint64_t)b, bytes, seg);
              memcpy(segs, v.data(), v.size() * sizeof(SwSeg));
              BulkTuning t{0, stages, sb, ctas};
              float ms = time_bulk(st, segs, (uint32_t)v.size(), t, 4, where ? nullptr : flush, FLUSH);
              res.push_back(R{ms, stages, sb, ctas, seg});
            }
      std::sort(res.begin(), res.end(), [](const R& x, const R& y) { return x.ms < y.ms; });
      for (size_t i = 0; i < res.size() && i < 6; i++) {
        printf("[tune %s %3zu MiB] #%zu stages=%d stage=%5d ctas=%d seg=%6llu: %.3f ms %.1f GB/s\n", where ? "pull" : "loop",
               bytes >> 20, i, res[i].st, res[i].sb, res[i].ct, (unsigned long long)res[i].seg, res[i].ms,
               bytes / (res[i].ms * 1e-3) / 1e9);
        if (json)
          fprintf(json, "{\"bench\":\"tune\",\"where\":\"%s\",\"bytes\":%zu,\"rank\":%zu,\"stages\":%d,\"stage_bytes\":%d,\"ctas\":%d,\"seg\":%llu,\"ms\":%.4f}\n",
                  where ? "pull" : "loop", bytes, i, res[i].st, res[i].sb, res[i].ct, (unsigned long long)res[i].seg, res[i].ms);
      }
      // the engine's default
      for (auto& r : res)
        if (r.st == 8 && r.sb == 24576 && r.ct == 1 && r.seg == (128u << 10))
          printf("[tune %s %3zu MiB] default(8x24K,1cta,seg128K): %.3f ms %.1f GB/s\n", where ? "pull" : "loop", bytes >> 20,
                 r.ms, bytes / (r.ms * 1e-3) / 1e9);
    }
  }
}

// ------------------------------------------------------------------ pinned host memory paths
static void bench_hostmem(FILE* json) {
  stream_t st = stream_create();
  const size_t N = 64u << 20;
  uint8_t *hs = (uint8_t*)host_alloc(N), *hd = (uint8_t*)host_alloc(N);
  uint8_t *ds = (uint8_t*)dev_alloc(N), *dd = (uint8_t*)dev_alloc(N);
  REQ(hs && hd && ds && dd);
  for (size_t i = 0; i < N; i++) hs[i] = (uint8_t)(i * 7 + (i >> 11));
  CK(cudaMemcpy(ds, hs, N, cudaMemcpyHostToDevice));
  SwSeg* segs = (SwSeg*)host_alloc(sizeof(SwSeg) * 65536);
  struct Case {
    const char* name;
    uint8_t *src, *dst;
  } cases[] = {{"host->host", hs, hd}, {"host->dev", hs, dd}, {"dev->host", ds, hd}};
  for (auto& c : cases) {
    for (int mode = 0; mode < 3; mode++) {
      float best = 1e30f;
      const char* mname = mode == 0 ? "tma" : (mode == 1 ? "simt" : "cudaMemcpyAsync");
      for (uint64_t seg : {uint64_t(1) << 16, uint64_t(1) << 18, uint64_t(1) << 20}) {
        if (mode == 2 && seg != (1u << 16)) continue;
        memset(hd, 0, N);
        CK(cudaMemset(dd, 0, N));
        auto v = make_segs((uint64_t)c.src, (uint64_t)c.dst, N, seg);
        memcpy(segs, v.data(), v.size() * sizeof(SwSeg));
        event_t a = event_create(1), b = event_create(1);
        float bb = 1e30f;
        for (int it = 0; it < 5; it++) {
          event_record(a, st);
          if (mode == 2) {
            CK(cudaMemcpyAsync(c.dst, c.src, N, cudaMemcpyDefault, (cudaStream_t)st));
          } else {
            BulkTuning t{mode, 8, 24576, mode ? 8 : 1};
            REQ(launch_bulk(st, segs, (uint32_t)v.size(), &t) == 0);
          }
          event_record(b, st);
          REQ(event_sync(b) == 0);
          float ms = event_elapsed_ms(a, b);
          if (it > 0 && ms < bb) bb = ms;
        }
        // verify
        std::vector<uint8_t> chk(N);
        if (c.dst == hd) memcpy(chk.data(), hd, N); else CK(cudaMemcpy(chk.data(), dd, N, cudaMemcpyDeviceToHost));
        REQ(memcmp(chk.data(), hs, N) == 0);
        printf("[hostmem] %-10s %-16s seg=%7llu: %8.3f ms %7.1f GB/s\n", c.name, mname, (unsigned long long)seg, bb, N / (bb * 1e-3) / 1e9);
        if (json)
          fprintf(json, "{\"bench\":\"hostmem\",\"path\":\"%s\",\"mode\":\"%s\",\"seg\":%llu,\"ms\":%.4f,\"gbs\":%.1f}\n", c.name, mname,
                  (unsigned long long)seg, bb, N / (bb * 1e-3) / 1e9);
        if (bb < best) best = bb;
        event_destroy(a);
        event_destroy(b);
      }
    }
  }
}


// ------------------------------------------------------------------ PCIe duplex: host->device and device->host at once
// What the e2e path (host buffers) can hope for: both directions of the link busy at the same time, by the copy
// engines, by the bulk kernels (few CTAs each, so that both kernels are resident together), or one of each.
static void bench_duplex(FILE* json) {
  const size_t N = 256u << 20;
  uint8_t *hs = (uint8_t*)host_alloc(N), *hd = (uint8_t*)host_alloc(N);
  uint8_t *ds = (uint8_t*)dev_alloc(N), *dd = (uint8_t*)dev_alloc(N);
  REQ(hs && hd && ds && dd);
  memset(hs, 0x3C, N);
  CK(cudaMemset(ds, 0x5A, N));
  stream_t s1 = stream_create(), s2 = stream_create();
  const uint64_t seg = 1u << 20;
  auto up = make_segs((uint64_t)hs, (uint64_t)dd, N, seg), down = make_segs((uint64_t)ds, (uint64_t)hd, N, seg);
  SwSeg* sup = (SwSeg*)host_alloc(sizeof(SwSeg) * up.size());
  SwSeg* sdown = (SwSeg*)host_alloc(sizeof(SwSeg) * down.size());
  memcpy(sup, up.data(), sizeof(SwSeg) * up.size());
  memcpy(sdown, down.data(), sizeof(SwSeg) * down.size());
  stream_t xs[4] = {stream_create(), stream_create(), stream_create(), stream_create()};
  auto down64 = make_segs((uint64_t)ds, (uint64_t)hd, N, 65536);
  SwSeg* small = (SwSeg*)host_alloc(sizeof(SwSeg) * down64.size());
  memcpy(small, down64.data(), sizeof(SwSeg) * down64.size());
  const size_t small_n = down64.size();
  struct Mode {
    const char* name;
    int up, down;   // 0: none, 1: copy engine, 2: bulk TMA kernel, 3: SIMT kernel, 4: 1 MiB copies, 5/6: 4 MiB TMA/SIMT kernels
  } modes[] = {{"H2D copy engine alone", 1, 0},   {"D2H copy engine alone", 0, 1},    {"H2D + D2H copy engines", 1, 1},
               {"H2D kernel alone", 2, 0},        {"D2H kernel alone", 0, 2},         {"H2D + D2H kernels (TMA)", 2, 2},
               {"H2D copy engine + D2H kernel", 1, 2}, {"H2D kernel + D2H copy engine", 2, 1}, {"H2D + D2H kernels (SIMT)", 3, 3},
               // the engine's pattern for host buffers: 1 MiB copies on four streams; 4 MiB kernels of 64 KiB pieces
               {"H2D 1 MiB copies alone", 4, 0}, {"D2H 4 MiB TMA kernels alone", 0, 5}, {"H2D 1 MiB copies + D2H 4 MiB TMA kernels", 4, 5},
               {"H2D 1 MiB copies + D2H 4 MiB SIMT kernels", 4, 6}, {"H2D 1 MiB copies + D2H copy engine", 4, 1},
               {"H2D 1 MiB copies, one stream + D2H 4 MiB TMA kernels", 7, 5},
               {"H2D 4 MiB copies, one stream + D2H 4 MiB TMA kernels", 9, 5}, {"H2D 16 MiB copies, one stream + D2H 4 MiB TMA kernels", 10, 5},
               {"H2D kernel 8 CTAs + D2H 4 MiB TMA kernels", 11, 5}, {"H2D kernel 8 CTAs + D2H kernel 8 CTAs", 11, 11},
               {"H2D 1 MiB copies, batch API alone", 8, 0}, {"H2D 1 MiB copies, batch API + D2H 4 MiB TMA kernels", 8, 5}};
  for (const Mode& m : modes) {
    float best = 1e30f, best_up = 0, best_down = 0;
    for (int it = 0; it < 4; it++) {
      event_t a = event_create(1), b1 = event_create(1), b2 = event_create(1);
      CK(cudaDeviceSynchronize());
      event_record(a, s1);
      CK(cudaStreamWaitEvent((cudaStream_t)s2, (cudaEvent_t)a, 0));
      auto go = [&](int how, stream_t st, SwSeg* segs, size_t nseg, void* dst, const void* src) {
        if (how == 1) CK(cudaMemcpyAsync(dst, src, N, cudaMemcpyDefault, (cudaStream_t)st));
        if (how == 2) {
          BulkTuning t{0, 8, 24576, 1, 0};
          REQ(launch_bulk(st, segs, 32, &t) == 0);   // 32 CTAs ...
          for (size_t o = 32; o < nseg; o += 32) REQ(launch_bulk(st, segs + o, (uint32_t)std::min<size_t>(32, nseg - o), &t) == 0);
        }
        if (how == 3) {
          BulkTuning t{1, 8, 24576, 1, 0};
          for (size_t o = 0; o < nseg; o += 64) REQ(launch_bulk(st, segs + o, (uint32_t)std::min<size_t>(64, nseg - o), &t) == 0);
        }
        if (how == 4) {   // 1 MiB copies, groups of four per stream, four streams
          for (size_t o = 0; o < N; o += 1u << 20)
            CK(cudaMemcpyAsync((uint8_t*)dst + o, (const uint8_t*)src + o, 1u << 20, cudaMemcpyDefault, (cudaStream_t)xs[(o >> 22) & 3]));
        }
        if (how == 7 || how == 9 || how == 10) {   // copies of 1 / 4 / 16 MiB on one stream
          const size_t piece = how == 7 ? (1u << 20) : (how == 9 ? (4u << 20) : (16u << 20));
          for (size_t o = 0; o < N; o += piece)
            CK(cudaMemcpyAsync((uint8_t*)dst + o, (const uint8_t*)src + o, piece, cudaMemcpyDefault, (cudaStream_t)st));
        }
        if (how == 8) {   // the same 1 MiB copies through cudaMemcpyBatchAsync, 64 per call
          static std::vector<void*> bd, bs;
          static std::vector<size_t> bz;
          bd.clear(); bs.clear(); bz.clear();
          for (size_t o = 0; o < N; o += 1u << 20) {
            bd.push_back((uint8_t*)dst + o);
            bs.push_back((uint8_t*)const_cast<void*>(src) + o);
            bz.push_back(1u << 20);
          }
          cudaMemcpyAttributes at;
          memset(&at, 0, sizeof at);
          at.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
          size_t ai = 0, fail = 0;
          for (size_t o = 0; o < bd.size(); o += 64)
            CK(cudaMemcpyBatchAsync(bd.data() + o, bs.data() + o, bz.data() + o, std::min<size_t>(64, bd.size() - o), &at, &ai, 1, &fail, (cudaStream_t)st));
        }
        if (how == 11) {   // bulk TMA kernel on 8 CTAs, 8 MiB per launch
          BulkTuning t{0, 8, 24576, 1, 0};
          for (size_t o = 0; o < nseg; o += 8) REQ(launch_bulk(st, segs + o, (uint32_t)std::min<size_t>(8, nseg - o), &t) == 0);
        }
        if (how == 5 || how == 6) {   // 4 MiB per launch, 64 KiB pieces
          BulkTuning t{how == 5 ? 0 : 1, 8, 24576, how == 5 ? 1 : 8, 0};
          for (size_t o = 0; o < small_n; o += 64) REQ(launch_bulk(st, small + o, (uint32_t)std::min<size_t>(64, small_n - o), &t) == 0);
        }
      };
      if (m.up == 4 || m.down == 4)
        for (int k = 0; k < 4; k++) CK(cudaStreamWaitEvent((cudaStream_t)xs[k], (cudaEvent_t)a, 0));
      go(m.up, s1, sup, up.size(), dd, hs);
      if (m.up == 4)
        for (int k = 0; k < 4; k++) {
          event_t j = event_create(0);
          event_record(j, xs[k]);
          CK(cudaStreamWaitEvent((cudaStream_t)s1, (cudaEvent_t)j, 0));
          event_destroy(j);
        }
      go(m.down, s2, sdown, down.size(), hd, ds);
      if (m.down == 4)
        for (int k = 0; k < 4; k++) {
          event_t j = event_create(0);
          event_record(j, xs[k]);
          CK(cudaStreamWaitEvent((cudaStream_t)s2, (cudaEvent_t)j, 0));
          event_destroy(j);
        }
      event_record(b1, s1);
      event_record(b2, s2);
      REQ(event_sync(b1) == 0 && event_sync(b2) == 0);
      const float ms = std::max(event_elapsed_ms(a, b1), event_elapsed_ms(a, b2));
      if (it > 0 && ms < best) {
        best = ms;
        best_up = event_elapsed_ms(a, b1);
        best_down = event_elapsed_ms(a, b2);
      }
      event_destroy(a);
      event_destroy(b1);
      event_destroy(b2);
    }
    const double dirs = (m.up ? 1 : 0) + (m.down ? 1 : 0);
    printf("[duplex] %-44s %8.3f ms  %6.1f GB/s per direction, %6.1f GB/s total  (up %.3f ms, down %.3f ms)\n", m.name, best, N / (best * 1e-3) / 1e9,
           dirs * N / (best * 1e-3) / 1e9, best_up, best_down);
    if (json) fprintf(json, "{\"bench\":\"duplex\",\"mode\":\"%s\",\"ms\":%.4f,\"gbs_per_direction\":%.1f}\n", m.name, best, N / (best * 1e-3) / 1e9);
  }
}

// ------------------------------------------------------------------ 2-process CUDA IPC
static int ipc_child(const char* path) {
  int n = device_count();
  int dev = n > 1 ? 1 : 0;
  REQ(init(dev) == 0);
  FILE* f = fopen(path, "rb");
  REQ(f);
  uint8_t handle[64];
  uint64_t off = 0, len = 0;
  REQ(fread(handle, 1, 64, f) == 64 && fread(&off, 8, 1, f) == 1 && fread(&len, 8, 1, f) == 1);
  fclose(f);
  void* base = nullptr;
  REQ(ipc_open(handle, &base) == 0);
  uint8_t* remote = (uint8_t*)base + off;
  uint8_t* local = (uint8_t*)dev_alloc(len);
  stream_t st = stream_create();
  SwSeg* segs = (SwSeg*)host_alloc(sizeof(SwSeg) * 65536);
  auto v = make_segs((uint64_t)remote, (uint64_t)local, len, 1 << 18);
  memcpy(segs, v.data(), v.size() * sizeof(SwSeg));
  for (int mode = 0; mode < 2; mode++) {
    BulkTuning t{mode, 4, 32768, mode ? 8 : 1};
    CK(cudaMemset(local, 0, len));
    float ms = time_bulk(st, segs, (uint32_t)v.size(), t, 5, nullptr, 0);
    std::vector<uint8_t> h(len);
    CK(cudaMemcpy(h.data(), local, len, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < len; i += 4097) REQ(h[i] == (uint8_t)((i + off) * 131u >> 3));
    printf("[ipc] child dev%d pulled %.0f MiB over IPC mapping, mode=%s: %.3f ms %.1f GB/s, pattern ok\n", dev,
           len / 1048576.0, mode ? "simt" : "tma", ms, len / (ms * 1e-3) / 1e9);
  }
  // write into the parent's buffer (push) so the parent can check visibility
  CK(cudaMemset(remote, 0xC3, 4096));
  CK(cudaDeviceSynchronize());
  REQ(ipc_close(base) == 0);
  return 0;
}

static void test_ipc(const char* self) {
  const size_t ALLOC = 600u << 20;
  const uint64_t off = 4096 + 512, len = 512u << 20;
  uint8_t* buf = (uint8_t*)dev_alloc(ALLOC);
  std::vector<uint8_t> h(ALLOC);
  for (size_t i = 0; i < ALLOC; i++) h[i] = (uint8_t)(i * 131u >> 3);
  CK(cudaMemcpy(buf, h.data(), ALLOC, cudaMemcpyHostToDevice));
  PtrInfo pi;
  REQ(ptr_info(buf + off, &pi) == 0);
  printf("[ipc] ptr_info: is_device=%d dev=%d base=%llx size=%llu (alloc %p)\n", pi.is_device, pi.device,
         (unsigned long long)pi.base, (unsigned long long)pi.size, buf);
  REQ(pi.is_device && pi.base == (uint64_t)buf && pi.size >= ALLOC);
  uint8_t handle[64];
  REQ(ipc_get(buf, handle) == 0);
  // same-process open is expected to fail (documented CUDA behaviour) -> engine uses direct pointers
  void* self_open = nullptr;
  int r = ipc_open(handle, &self_open);
  printf("[ipc] same-process cudaIpcOpenMemHandle -> %s\n", r == 0 ? "ok (unexpected)" : last_error());
  if (r == 0) ipc_close(self_open);
  char path[64];
  snprintf(path, sizeof(path), "/tmp/sw_ipc_%d.bin", (int)getpid());
  FILE* f = fopen(path, "wb");
  fwrite(handle, 1, 64, f);
  fwrite(&off, 8, 1, f);
  fwrite(&len, 8, 1, f);
  fclose(f);
  pid_t pid = fork();  // fork before... no: CUDA is already initialised here, so exec a fresh process
  if (pid == 0) {
    execl(self, self, "ipc-child", path, (char*)nullptr);
    _exit(127);
  }
  int status = 0;
  waitpid(pid, &status, 0);
  REQ(WIFEXITED(status) && WEXITSTATUS(status) == 0);
  std::vector<uint8_t> chk(4096);
  CK(cudaMemcpy(chk.data(), buf + off, 4096, cudaMemcpyDeviceToHost));
  for (auto x : chk) REQ(x == 0xC3);
  printf("[ipc] parent sees the child's peer stores: ok\n");
  unlink(path);
  dev_free(buf);
}



// ------------------------------------------------------------------ segment-list vs balanced job-range launch
// Launch shapes as the engine produces them for windows of 1 MiB messages: n messages, each cut into
// segments of ceil(total / (4 * SMs)) rounded to the stage size (pump_bulk), separate allocations.
static void bench_balance(FILE* json) {
  stream_t st = stream_create();
  const size_t MSG = 1u << 20, GAP = 256, MAXN = 96;
  uint8_t* src = (uint8_t*)dev_alloc(MAXN * (MSG + GAP));
  uint8_t* dst = (uint8_t*)dev_alloc(MAXN * (MSG + GAP));
  const size_t FLUSH = 256u << 20;
  void* flush = dev_alloc(FLUSH);
  REQ(src && dst && flush);
  std::vector<uint8_t> h(MAXN * (MSG + GAP));
  fill_pattern(h, 3);
  CK(cudaMemcpy(src, h.data(), h.size(), cudaMemcpyHostToDevice));
  SwSeg* segs = (SwSeg*)host_alloc(sizeof(SwSeg) * 65536);
  for (int n : {1, 2, 4, 8, 16, 32, 43, 64, 96}) {
    const uint64_t total = (uint64_t)n * MSG;
    const uint64_t unit = 24576, target = (uint64_t)sm_count() * 4;
    uint64_t seg = (total + target - 1) / target;
    seg = ((seg + unit - 1) / unit) * unit;
    seg = std::max<uint64_t>(seg, 49152);
    std::vector<SwSeg> v;
    for (int m = 0; m < n; m++) {
      auto p = make_segs((uint64_t)(src + (size_t)m * (MSG + GAP)), (uint64_t)(dst + (size_t)m * (MSG + GAP)), MSG, seg);
      v.insert(v.end(), p.begin(), p.end());
    }
    memcpy(segs, v.data(), v.size() * sizeof(SwSeg));
    float ms[2];
    for (int bal = 0; bal < 2; bal++) {
      CK(cudaMemset(dst, 0, MAXN * (MSG + GAP)));
      BulkTuning t{0, 8, 24576, 1, bal};
      ms[bal] = time_bulk(st, segs, (uint32_t)v.size(), t, 7, flush, FLUSH);
      std::vector<uint8_t> chk((size_t)n * (MSG + GAP));
      CK(cudaMemcpy(chk.data(), dst, chk.size(), cudaMemcpyDeviceToHost));
      for (int m = 0; m < n; m++) REQ(memcmp(chk.data() + (size_t)m * (MSG + GAP), h.data() + (size_t)m * (MSG + GAP), MSG) == 0);
    }
    printf("[balance] %3d x 1 MiB (%5zu segments of %7llu B): segment list %7.2f us %7.1f GB/s | job ranges %7.2f us %7.1f GB/s\n", n,
           v.size(), (unsigned long long)seg, ms[0] * 1e3, total / (ms[0] * 1e-3) / 1e9, ms[1] * 1e3, total / (ms[1] * 1e-3) / 1e9);
    if (json)
      fprintf(json, "{\"bench\":\"balance\",\"msgs\":%d,\"nseg\":%zu,\"seglist_us\":%.2f,\"jobs_us\":%.2f}\n", n, v.size(), ms[0] * 1e3,
              ms[1] * 1e3);
  }
  host_free(segs);
  dev_free(src);
  dev_free(dst);
  dev_free(flush);
  stream_destroy(st);
}

// ------------------------------------------------------------------ launch/completion floor
// What one launch -> "host knows it finished" costs on this box, by completion mechanism.
__global__ void floor_empty_kernel() {}
__global__ void floor_flag_kernel(volatile uint64_t* flag, uint64_t value) {
  __threadfence_system();
  *flag = value;
}

static double median(std::vector<double>& v) {
  std::sort(v.begin(), v.end());
  return v[v.size() / 2];
}

static void bench_floor(FILE* json) {
  cudaStream_t st;
  CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  uint64_t* flag;
  CK(cudaHostAlloc((void**)&flag, 64, cudaHostAllocPortable | cudaHostAllocMapped));
  *flag = 0;
  const int iters = 400;
  auto report = [&](const char* name, std::vector<double>& total, std::vector<double>* api = nullptr) {
    const double m = median(total) * 1e6;
    std::vector<double> s = total;
    const double p10 = s[s.size() / 10] * 1e6;
    if (api) {
      printf("[floor] %-58s median %6.2f us  p10 %6.2f us  (API calls %5.2f us)\n", name, m, p10, median(*api) * 1e6);
    } else {
      printf("[floor] %-58s median %6.2f us  p10 %6.2f us\n", name, m, p10);
    }
    if (json) fprintf(json, "{\"bench\":\"floor\",\"case\":\"%s\",\"us\":%.2f,\"p10_us\":%.2f}\n", name, m, p10);
  };
  for (int timing = 0; timing < 2; timing++) {
    cudaEvent_t ev;
    CK(cudaEventCreateWithFlags(&ev, timing ? cudaEventDefault : cudaEventDisableTiming));
    std::vector<double> tot, api;
    for (int i = 0; i < iters; i++) {
      const double t0 = now_s();
      floor_empty_kernel<<<1, 32, 0, st>>>();
      CK(cudaEventRecord(ev, st));
      const double t1 = now_s();
      while (cudaEventQuery(ev) == cudaErrorNotReady) {
      }
      const double t2 = now_s();
      if (i >= 20) {
        tot.push_back(t2 - t0);
        api.push_back(t1 - t0);
      }
    }
    report(timing ? "empty kernel + event (timing enabled), cudaEventQuery spin" : "empty kernel + event (timing disabled), cudaEventQuery spin",
           tot, &api);
    CK(cudaEventDestroy(ev));
  }
  uint64_t seq = 0;
  {
    std::vector<double> tot, api;
    for (int i = 0; i < iters; i++) {
      const double t0 = now_s();
      floor_flag_kernel<<<1, 32, 0, st>>>(flag, ++seq);
      const double t1 = now_s();
      while (*(volatile uint64_t*)flag != seq) {
      }
      const double t2 = now_s();
      if (i >= 20) {
        tot.push_back(t2 - t0);
        api.push_back(t1 - t0);
      }
    }
    report("flag kernel (fence.sys + store to pinned host), host spins on the flag", tot, &api);
  }
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(st));
  CK(cudaFreeHost(flag));
  CK(cudaStreamDestroy(st));
}

// ------------------------------------------------------------------ hostlat: what device <-> host-memory hops cost
// One CTA, two warps.  Warp 1 (optional) keeps PCIe reads of pinned host memory in flight, like the link warp of
// sw_progress_kernel.  Warp 0 lane 0 measures with clock64:
//   mode 0: latency of one ld.relaxed.sys from pinned host memory
//   mode 1: store to pinned host memory + fence.sys (the completion-record pattern)
//   mode 2: store to device memory + fence.sys
//   mode 3: store to device memory + fence.gpu
//   mode 4: host -> device signalling through pinned memory: the host bumps a word, the kernel echoes it (RTT seen by the host)
__global__ void hostlat_kernel(volatile uint64_t* host_words, uint64_t* dev_words, int mode, int iters, int bg, uint64_t* out,
                               volatile uint64_t* stop) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 1) {
    if (!bg || lane) return;
    uint64_t acc = 0;
    while (*reinterpret_cast<volatile uint64_t*>(dev_words + 64) == 0) {
      uint64_t v;
      asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(host_words + 32) : "memory");
      acc += v;
    }
    out[63] = acc;
    return;
  }
  if (lane) return;
  long long total = 0, worst = 0;
  if (mode == 4) {
    uint64_t seen = 0;
    while (!*stop) {
      uint64_t v;
      asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(host_words) : "memory");
      if (v != seen) {
        seen = v;
        asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(host_words + 8), "l"(v) : "memory");
      }
    }
  } else {
    for (int i = 0; i < iters; i++) {
      const long long t0 = clock64();
      if (mode == 0) {
        uint64_t v;
        asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(host_words + (i & 7)) : "memory");
        total += (v & 1);
      } else if (mode == 1) {
        asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(host_words + 16 + (i & 7)), "l"((uint64_t)i) : "memory");
        __threadfence_system();
      } else if (mode == 2) {
        dev_words[i & 7] = i;
        __threadfence_system();
      } else {
        dev_words[i & 7] = i;
        __threadfence();
      }
      const long long dt = clock64() - t0;
      total += dt;
      worst = dt > worst ? dt : worst;
    }
  }
  out[0] = (uint64_t)total;
  out[1] = (uint64_t)worst;
  __threadfence();
  *reinterpret_cast<volatile uint64_t*>(dev_words + 64) = 1;
}

static void bench_hostlat(FILE* json) {
  uint64_t* host = (uint64_t*)host_alloc(4096);
  uint64_t* dev = (uint64_t*)dev_alloc(4096);
  uint64_t* out = (uint64_t*)host_alloc(4096);
  int khz = 0;
  CK(cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0));
  const double mhz = khz / 1000.0;
  const char* names[] = {"ld.sys of pinned host memory", "st pinned host + fence.sys", "st device + fence.sys", "st device + fence.gpu"};
  for (int bg = 0; bg < 2; bg++)
    for (int mode = 0; mode < 4; mode++) {
      CK(cudaMemset(dev, 0, 4096));
      const int iters = 2000;
      hostlat_kernel<<<1, 64>>>(host, dev, mode, iters, bg, out, host + 40);
      CK(cudaDeviceSynchronize());
      printf("hostlat %-32s background PCIe reads %d: mean %.2f us  worst %.2f us\n", names[mode], bg, out[0] / mhz / iters, out[1] / mhz);
      if (json) fprintf(json, "{\"probe\":\"hostlat\",\"what\":\"%s\",\"bg_reads\":%d,\"mean_us\":%.3f,\"worst_us\":%.3f}\n", names[mode], bg, out[0] / mhz / iters, out[1] / mhz);
    }
  // host -> device -> host echo through pinned memory (the post-ring / completion-ring hop pair)
  CK(cudaMemset(dev, 0, 4096));
  host[0] = host[8] = host[40] = 0;
  hostlat_kernel<<<1, 64>>>(host, dev, 4, 0, 0, out, host + 40);
  std::vector<double> rtt;
  for (int i = 1; i <= 2000; i++) {
    const double t0 = now_s();
    __atomic_store_n(&host[0], (uint64_t)i, __ATOMIC_RELEASE);
    while (__atomic_load_n(&host[8], __ATOMIC_ACQUIRE) != (uint64_t)i) {
    }
    rtt.push_back((now_s() - t0) * 1e6);
  }
  __atomic_store_n(&host[40], 1, __ATOMIC_RELEASE);
  CK(cudaDeviceSynchronize());
  std::sort(rtt.begin(), rtt.end());
  printf("hostlat host word -> kernel poll -> echo word -> host: median %.2f us  p10 %.2f  p90 %.2f\n", rtt[rtt.size() / 2], rtt[rtt.size() / 10], rtt[rtt.size() * 9 / 10]);
  if (json) fprintf(json, "{\"probe\":\"hostlat\",\"what\":\"host->kernel->host echo\",\"median_us\":%.3f}\n", rtt[rtt.size() / 2]);
  host_free(host);
  host_free(out);
  dev_free(dev);
}

// ------------------------------------------------------------------ pull: the resident pull kernel on its own
// Publishes batches of whole messages from the device (the way a matcher does) and lets sw_pull_kernel serve them:
// payload GB/s while a batch is active (first chunk claimed -> records written), per batch shape.  `ncu --set full`
// of this command profiles the kernel itself (launch = a resident period that serves the published batches).
static void bench_pull(FILE* json, int nbatches_fixed) {
  const size_t POOL = 2ull << 30;
  uint8_t* src = (uint8_t*)dev_alloc_raw(POOL);
  uint8_t* dst = (uint8_t*)dev_alloc_raw(POOL);
  uint8_t* scratch = (uint8_t*)dev_alloc(4096 + sizeof(SwCqEnt) * SW_CQ_RING);
  REQ(src && dst && scratch);
  CK(cudaMemset(src, 0x5A, POOL));
  SwPullQueue* q = pull_queue_create();
  SwPullCtl* ctl = (SwPullCtl*)host_alloc(sizeof(SwPullCtl));
  SwSeg* msgs = (SwSeg*)host_alloc(sizeof(SwSeg) * SW_PULL_JOBS * 64);
  stream_t sp = stream_create(), sq = stream_create();
  BulkTuning tune{0, 8, 24576, 1, 1};
  const uint32_t ctas = (uint32_t)pull_default_ctas();
  // SW_PROBE_PULL_LINGER_US=1: the kernel leaves as soon as the batch is done (ncu captures: duration = start-up + batch)
  const uint32_t linger_us = getenv("SW_PROBE_PULL_LINGER_US") ? (uint32_t)atoi(getenv("SW_PROBE_PULL_LINGER_US")) : 40;
  struct Shape {
    uint32_t nmsg;
    uint64_t len;
    uint32_t nbatch;
  };
  const Shape shapes[] = {{1, 1u << 20, 8}, {8, 1u << 20, 8}, {16, 1u << 20, 8}, {64, 1u << 20, 8}, {64, 4u << 20, 6}, {16, 64u << 20, 2}, {1, 1u << 30, 2}, {52, 16384, 8}, {52, 65536, 8}};
  uint64_t seq = 0;
  for (const Shape& sh : shapes) {
    const uint32_t nb = nbatches_fixed ? (uint32_t)nbatches_fixed : sh.nbatch;
    uint64_t s0[8], s1[8];
    pull_queue_read_stats(q, s0);
    // (larger than the 50 MB L2 of an H100: batches of a shape use disjoint parts of the 2 GiB pools, wrapping)
    uint64_t off = 0;
    for (uint32_t b = 0; b < nb; b++) {
      SwSeg* m = msgs + (size_t)b * SW_PULL_JOBS;
      for (uint32_t j = 0; j < sh.nmsg; j++) {
        if (off + sh.len > POOL) off = 0;
        m[j] = SwSeg{(uint64_t)(uintptr_t)(src + off), (uint64_t)(uintptr_t)(dst + off), sh.len, 0};
        off += sh.len;
      }
    }
    // one batch per resident period: publish it, start the pull kernel, which serves it and leaves after 40 us of
    // silence (its statistics count the active interval of the batch only)
    for (uint32_t b = 0; b < nb; b++) {
      REQ(probe_publish_batch(sq, q, msgs + (size_t)b * SW_PULL_JOBS, sh.nmsg, ctas, scratch) == 0);
      REQ(stream_sync(sq) == 0);
      ctl->stop = 0;
      REQ(launch_pull(sp, q, ctl, ++seq, ctas, linger_us, 100000, &tune) == 0);
      REQ(stream_sync(sp) == 0);
      uint64_t st[8];
      REQ(pull_queue_read_stats(q, st) == 0);
      if (st[2] - s0[2] != b + 1) {
        fprintf(stderr, "pull probe: batch %u of shape %u x %llu not completed (batches %llu, alloc %llu, exited %llu)\n", b, sh.nmsg,
                (unsigned long long)sh.len, (unsigned long long)(st[2] - s0[2]), (unsigned long long)st[7], (unsigned long long)ctl->exited);
        exit(4);
      }
    }
    pull_queue_read_stats(q, s1);
    const double nbat = (double)(s1[2] - s0[2]), bytes = (double)(s1[0] - s0[0]), busy = (double)(s1[1] - s0[1]);
    printf("pull %2u x %9llu B per batch: %6.1f us per batch, %7.1f GB/s payload while active (x2 = HBM traffic); phases %.1f / %.1f / %.1f us\n",
           sh.nmsg, (unsigned long long)sh.len, busy / nbat * 1e-3, bytes / busy, (s1[4] - s0[4]) / nbat * 1e-3, (s1[5] - s0[5]) / nbat * 1e-3,
           (s1[6] - s0[6]) / nbat * 1e-3);
    if (json)
      fprintf(json, "{\"probe\":\"pull\",\"msgs\":%u,\"msg_bytes\":%llu,\"us_per_batch\":%.2f,\"payload_gbs\":%.1f,\"pickup_us\":%.2f,\"copy_us\":%.2f,\"records_us\":%.2f}\n",
              sh.nmsg, (unsigned long long)sh.len, busy / nbat * 1e-3, bytes / busy, (s1[4] - s0[4]) / nbat * 1e-3, (s1[5] - s0[5]) / nbat * 1e-3,
              (s1[6] - s0[6]) / nbat * 1e-3);
  }
  // spot check
  std::vector<uint8_t> h(4096);
  CK(cudaMemcpy(h.data(), dst, 4096, cudaMemcpyDeviceToHost));
  for (auto x : h) REQ(x == 0x5A);
}

int main(int argc, char** argv) {
  std::string cmd = argc > 1 ? argv[1] : "correctness";
  if (cmd == "ipc-child") return ipc_child(argv[2]);
  REQ(init(0) == 0);
  printf("backend %s, %d device(s), %d SMs\n", backend_name(), device_count(), sm_count());
  FILE* json = nullptr;
  if (argc > 2 && strcmp(argv[2], "-") != 0) json = fopen(argv[2], "a");
  if (cmd == "correctness" || cmd == "all") test_bulk_correctness();
  if (cmd == "latency" || cmd == "all") bench_latency(json);
  if (cmd == "bench" || cmd == "all") bench_single(json);
  if (cmd == "floor") bench_floor(json);
  if (cmd == "balance") bench_balance(json);
  if (cmd == "hostmem") bench_hostmem(json);
  if (cmd == "duplex") bench_duplex(json);
  if (cmd == "hostlat") bench_hostlat(json);
  if (cmd == "pull") bench_pull(json, argc > 3 ? atoi(argv[3]) : 0);
  if (cmd == "tune") bench_tune(json);
  if (cmd == "ipc" || cmd == "all") test_ipc(argv[0]);
  if (cmd == "peer" || cmd == "all") bench_peer(json);
  if (json) fclose(json);
  printf("PROBE %s DONE\n", cmd.c_str());
  return 0;
}
