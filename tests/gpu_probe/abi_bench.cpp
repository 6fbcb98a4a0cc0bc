// tests/gpu_probe/abi_bench.cpp — drives libstarway_b200.so through its C ABI from C++ (no Python,
// no asyncio) to show what the engine + kernels sustain on their own: the same window workload as
// bench.py (receiver posts W receives, sender issues W sends + flush, wait for every completion),
// Server and Client on one GPU, device buffers, sizes 64 B .. 256 MiB.
//   abi_bench [out.jsonl]
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <chrono>
#include <unordered_map>
#include <vector>

#include "../../include/starway_b200.h"

static double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
#define REQ(c)                                                                        \
  do {                                                                                \
    if (!(c)) {                                                                       \
      fprintf(stderr, "FAILED %s at line %d: %s\n", #c, __LINE__, sw_last_error()); \
      exit(2);                                                                        \
    }                                                                                 \
  } while (0)

static std::unordered_map<uint64_t, sw_completion> done;
static void wait_for(sw_ctx* ctx, const std::vector<uint64_t>& ops) {
  sw_completion buf[256];
  for (uint64_t op : ops) {
    while (!done.count(op)) {
      int n = sw_wait(ctx, buf, 256, 100);
      for (int i = 0; i < n; i++) done[buf[i].op_id] = buf[i];
    }
    REQ(done[op].status == 0);
    done.erase(op);
  }
}

int main(int argc, char** argv) {
  FILE* out = argc > 1 ? fopen(argv[1], "a") : nullptr;
  sw_ctx* ctx = sw_ctx_create(0);
  REQ(ctx);
  sw_set_option(ctx, "profile", 1);
  sw_worker_t srv = sw_worker_create(ctx, SW_WORKER_SERVER), cli = sw_worker_create(ctx, SW_WORKER_CLIENT);
  REQ(sw_listen_address(ctx, srv) == 0);
  char blob[512];
  int64_t blen = sw_get_address(ctx, srv, blob, sizeof(blob));
  REQ(blen > 0);
  uint64_t cop = sw_connect_address(ctx, cli, blob, (size_t)blen);
  REQ(cop);
  wait_for(ctx, {cop});
  done.clear();

  const size_t POOL = 1ull << 30;
  uint8_t *src, *dst;
  REQ(cudaMalloc(&src, POOL) == cudaSuccess && cudaMalloc(&dst, POOL) == cudaSuccess);
  cudaMemset(src, 0x5A, POOL);
  cudaMemset(dst, 0, POOL);
  cudaDeviceSynchronize();

  const size_t n_min = getenv("ABI_MIN") ? (size_t)atoll(getenv("ABI_MIN")) : 64, n_max = getenv("ABI_MAX") ? (size_t)atoll(getenv("ABI_MAX")) : (256u << 20);
  for (size_t n = 64; n <= (256u << 20); n *= 4) {
    if (n < n_min || n > n_max) continue;
    size_t window = std::min<size_t>(256, std::max<size_t>(1, (512u << 20) / n));
    if (n <= 8192) window = 1024;
    int steps = n >= (16u << 20) ? 8 : 20;
    double best = 1e9;
    sw_stats s0, s1;
    for (int rep = 0; rep < 3; rep++) {
      sw_stats_get(ctx, &s0);
      double t0 = now_s();
      for (int st = 0; st < steps; st++) {
        std::vector<uint64_t> ops;
        ops.reserve(2 * window + 1);
        for (size_t j = 0; j < window; j++) {
          size_t off = (j * n) % (POOL - n + 1);
          ops.push_back(sw_post_recv(ctx, srv, dst + off, n, 1, 0xFFFF, SW_MEM_DEVICE));
        }
        for (size_t j = 0; j < window; j++) {
          size_t off = (j * n) % (POOL - n + 1);
          ops.push_back(sw_post_send(ctx, cli, 0, src + off, n, 1, SW_MEM_DEVICE));
        }
        ops.push_back(sw_post_flush(ctx, cli));
        wait_for(ctx, ops);
      }
      cudaDeviceSynchronize();
      double el = now_s() - t0;
      sw_stats_get(ctx, &s1);
      if (rep > 0 && el < best) best = el;
    }
    double msgs = (double)window * steps;
    double gbs = msgs * n / best / 1e9;
    uint64_t launches = s1.put_launches - s0.put_launches + s1.bulk_tma_launches - s0.bulk_tma_launches +
                        s1.bulk_simt_launches - s0.bulk_simt_launches;
    launches += s1.prog_launches - s0.prog_launches + s1.pull_launches - s0.pull_launches;
    const double pb = (double)(s1.pull_batches - s0.pull_batches), pbusy = s1.pull_busy_ms - s0.pull_busy_ms;
    printf("[c-abi loopback] %10zu B window=%4zu: %9.3f GB/s  %8.4f Mmsg/s  %8.2f us/msg  (%llu launches/step)", n, window,
           gbs, msgs / best / 1e6, best / msgs * 1e6, (unsigned long long)(launches / steps));
    if (pb > 0)
      printf("  pull: %.0f batches of %.2f MB, %.1f us each, %.0f GB/s while active; phases %.1f / %.1f / %.1f us", pb,
             (double)(s1.pull_bytes - s0.pull_bytes) / pb / 1e6, pbusy * 1e3 / pb, (double)(s1.pull_bytes - s0.pull_bytes) / (pbusy * 1e-3) / 1e9,
             (s1.pull_pickup_ms - s0.pull_pickup_ms) * 1e3 / pb, (s1.pull_copy_ms - s0.pull_copy_ms) * 1e3 / pb, (s1.pull_fin_ms - s0.pull_fin_ms) * 1e3 / pb);
    printf("\n");
    if (out)
      fprintf(out, "{\"bench\":\"c_abi_loopback\",\"msg_bytes\":%zu,\"window\":%zu,\"gbs\":%.3f,\"mmsg_s\":%.4f,\"us_per_msg\":%.3f}\n",
              n, window, gbs, msgs / best / 1e6, best / msgs * 1e6);
  }
  // spot check of the last transfer
  std::vector<uint8_t> h(4096);
  cudaMemcpy(h.data(), dst, 4096, cudaMemcpyDeviceToHost);
  for (auto x : h) REQ(x == 0x5A);
  uint64_t c1 = sw_close(ctx, cli);
  wait_for(ctx, {c1});
  uint64_t c2 = sw_close(ctx, srv);
  wait_for(ctx, {c2});
  sw_ctx_destroy(ctx);
  if (out) fclose(out);
  printf("ABI_BENCH DONE\n");
  return 0;
}
