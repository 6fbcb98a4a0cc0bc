// tests/gpu_kernels/kernels_test.cu — TEST INFRASTRUCTURE: flat extern "C" entry points over the CUDA backend
// (gpu_cuda.cu) so that tests/test_gpu_kernels.py can launch the data-movement kernels one at a time, at launch
// shapes of its own choosing, and compare them with a host reference.  Linked with build/gpu_cuda.o into
// libsw_kernels_test.so (`make probe`); never part of libstarway_b200.so.
//
// Callers pass arrays of plain integers; the wrappers build SwSeg / SwPutDesc themselves and write them into pinned
// host memory the caller owns (`pinned`, `pinned_bytes`), which must stay allocated until the launch has completed.
// Every wait is bounded: swk_wait returns -2 when its deadline passes, it never blocks for ever.
#include <cuda_runtime.h>
#include <stdint.h>
#include <time.h>

#include "../../starway_b200/csrc/gpu.h"

using namespace swgpu;

namespace {

thread_local const char* g_shim_err = nullptr;   // set by the wrappers themselves (argument checks)

int shim_fail(const char* what) {
  g_shim_err = what;
  return -1;
}

double now_s() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

// Segment list in the caller's pinned memory; nullptr when it does not fit.
SwSeg* build_segs(const uint64_t* src, const uint64_t* dst, const uint64_t* len, uint32_t n, void* pinned,
                  size_t pinned_bytes) {
  if (!pinned || (size_t)n * sizeof(SwSeg) > pinned_bytes) return nullptr;
  SwSeg* s = static_cast<SwSeg*>(pinned);
  for (uint32_t i = 0; i < n; i++) {
    s[i].src = src[i];
    s[i].dst = dst[i];
    s[i].len = len[i];
    s[i].pad = 0;
  }
  return s;
}

// One resident pull kernel and what it needs: the queue (device), its control words (pinned), a scratch completion
// ring that nobody reads, and pinned message lists, one per published batch.
struct PullSession {
  SwPullQueue* q;
  SwPullCtl* ctl;
  void* scratch;
  SwSeg* msgs;
  uint32_t max_batches, published;
};

}  // namespace

extern "C" {

// Also launches the batch publisher once, on a queue of its own: with lazy module loading (the CUDA 12 default) the
// first launch of a kernel loads it, and that load waits for kernels already running -- a resident pull kernel that
// is waiting for the very batch being published.
int swk_init(int device) {
  g_shim_err = nullptr;
  if (init(device) != 0) return -1;
  SwPullQueue* q = pull_queue_create();
  void* scratch = dev_alloc(4096 + sizeof(SwCqEnt) * SW_CQ_RING);
  SwSeg* msgs = static_cast<SwSeg*>(host_alloc(sizeof(SwSeg)));
  stream_t s = stream_create();
  int r = q && scratch && msgs && s ? 0 : -1;
  if (r == 0) r = probe_publish_batch(s, q, msgs, 0, 2, scratch);
  if (r == 0) r = stream_sync(s);
  if (s) stream_destroy(s);
  host_free(msgs);
  dev_free(scratch);
  pull_queue_destroy(q);
  return r;
}
const char* swk_last_error() { return g_shim_err ? g_shim_err : last_error(); }
int swk_bulk_smem_limit() { return bulk_smem_limit(); }
int swk_pull_default_ctas() { return pull_default_ctas(); }
int swk_pull_jobs() { return (int)SW_PULL_JOBS; }
int swk_pull_slots() { return (int)SW_PULL_SLOTS; }

void* swk_host_alloc(size_t bytes) { return host_alloc(bytes); }
int swk_host_free(void* p) { return host_free(p); }
void* swk_stream_create() { return stream_create(); }
int swk_stream_destroy(void* s) { return stream_destroy(s); }

// 0: everything queued on `s` has completed; -1: a launch on it failed; -2: still running at the deadline.
int swk_wait(void* s, double timeout_s) {
  const double deadline = now_s() + timeout_s;
  for (;;) {
    const int r = stream_query(s);
    if (r <= 0) return r;
    if (now_s() > deadline) {
      g_shim_err = "swk_wait: deadline passed with work still pending";
      return -2;
    }
    struct timespec ts = {0, 200000};
    nanosleep(&ts, nullptr);
  }
}

int swk_launch_bulk(void* s, const uint64_t* src, const uint64_t* dst, const uint64_t* len, uint32_t n, void* pinned,
                    size_t pinned_bytes, int mode, int stages, int stage_bytes, int ctas_per_sm, int balance) {
  g_shim_err = nullptr;
  const SwSeg* segs = build_segs(src, dst, len, n, pinned, pinned_bytes);
  if (!segs) return shim_fail("swk_launch_bulk: segment list does not fit the pinned buffer");
  BulkTuning t{mode, stages, stage_bytes, ctas_per_sm, balance};
  return launch_bulk(s, segs, n, &t);
}

int swk_launch_reduce(void* s, const uint64_t* src, const uint64_t* dst, const uint64_t* len, uint32_t n, void* pinned,
                      size_t pinned_bytes, int dtype, int mode, int stages, int stage_bytes, int ctas_per_sm) {
  g_shim_err = nullptr;
  const SwSeg* segs = build_segs(src, dst, len, n, pinned, pinned_bytes);
  if (!segs) return shim_fail("swk_launch_reduce: segment list does not fit the pinned buffer");
  BulkTuning t{mode, stages, stage_bytes, ctas_per_sm, 0};
  return launch_reduce(s, segs, n, dtype, &t);
}

// rts[i] != 0: message i is a rendezvous request whose 128-byte body is at src[i] (pinned host memory).
// Returns launch_put's result: 1 when the launch writes `done_value` to `*done_flag`, 0 when it does not, < 0 on error.
int swk_launch_put(void* s, const uint64_t* src, const uint64_t* dst, const uint64_t* tag, const uint64_t* seq,
                   const uint32_t* len, const uint8_t* rts, const uint64_t* msg_len, uint32_t n, void* pinned,
                   size_t pinned_bytes, uint64_t* done_flag, uint64_t done_value) {
  g_shim_err = nullptr;
  if (!pinned || (size_t)n * sizeof(SwPutDesc) > pinned_bytes)
    return shim_fail("swk_launch_put: descriptors do not fit the pinned buffer");
  SwPutDesc* d = static_cast<SwPutDesc*>(pinned);
  for (uint32_t i = 0; i < n; i++) {
    if (rts[i] && len[i] != sizeof(SwRts)) return shim_fail("swk_launch_put: an RTS body is 128 bytes");
    if (len[i] > SW_EAGER_MAX) return shim_fail("swk_launch_put: payload larger than a slot");
    d[i].src = src[i];
    d[i].dst = dst[i];
    d[i].tag = tag[i];
    d[i].seq = seq[i];
    d[i].len = len[i];
    d[i].kind = rts[i] ? SW_KIND_RTS : SW_KIND_EAGER;
    d[i].msg_len = msg_len[i];
  }
  DoneFlag df{done_flag, done_value};
  return launch_put(s, d, n, done_flag ? &df : nullptr);
}

// ---- pull session
void* swk_pull_create(uint32_t max_batches) {
  g_shim_err = nullptr;
  PullSession* p = new PullSession();
  p->q = pull_queue_create();
  p->ctl = static_cast<SwPullCtl*>(host_alloc(sizeof(SwPullCtl)));
  p->scratch = dev_alloc(4096 + sizeof(SwCqEnt) * SW_CQ_RING);
  p->msgs = static_cast<SwSeg*>(host_alloc(sizeof(SwSeg) * SW_PULL_JOBS * (size_t)max_batches));
  p->max_batches = max_batches;
  p->published = 0;
  if (!p->q || !p->ctl || !p->scratch || !p->msgs) {
    pull_queue_destroy(p->q);
    host_free(p->ctl);
    dev_free(p->scratch);
    host_free(p->msgs);
    delete p;
    return nullptr;
  }
  return p;
}

// Starts the resident pull kernel.  It serves published batches until swk_pull_stop; linger_us and max_life_us only
// bound its life should the caller never get there.
int swk_pull_launch(void* h, void* s, uint32_t ctas, int stages, int stage_bytes, uint32_t linger_us,
                    uint32_t max_life_us) {
  g_shim_err = nullptr;
  PullSession* p = static_cast<PullSession*>(h);
  if (ctas < 2) return shim_fail("swk_pull_launch: the pull grid needs CTA 0 and at least one copy CTA");
  BulkTuning t{0, stages, stage_bytes, 1, 1};
  p->ctl->stop = 0;
  return launch_pull(s, p->q, p->ctl, 1, ctas, linger_us, max_life_us, &t);
}

// Publishes one batch of whole messages (src and dst 16-byte aligned, any length) from the device.
int swk_pull_publish(void* h, void* s, const uint64_t* src, const uint64_t* dst, const uint64_t* len, uint32_t n,
                     uint32_t pull_ctas) {
  g_shim_err = nullptr;
  PullSession* p = static_cast<PullSession*>(h);
  if (p->published >= p->max_batches) return shim_fail("swk_pull_publish: session has no message list left");
  if (n > SW_PULL_JOBS) return shim_fail("swk_pull_publish: more messages than a batch holds");
  for (uint32_t j = 0; j < n; j++)
    if ((src[j] | dst[j]) & 15) return shim_fail("swk_pull_publish: src and dst must be 16-byte aligned");
  SwSeg* m = build_segs(src, dst, len, n, p->msgs + (size_t)p->published * SW_PULL_JOBS, sizeof(SwSeg) * SW_PULL_JOBS);
  const int r = probe_publish_batch(s, p->q, m, n, pull_ctas, p->scratch);
  if (r == 0) p->published++;
  return r;
}

void swk_pull_stop(void* h) { __atomic_store_n(&static_cast<PullSession*>(h)->ctl->stop, 1, __ATOMIC_RELEASE); }

// out: bytes, busy_ns, batches, jobs, pickup_ns, copy_ns, fin_ns, alloc (tickets taken, EXIT markers included)
int swk_pull_stats(void* h, uint64_t* out) { return pull_queue_read_stats(static_cast<PullSession*>(h)->q, out); }

// Only once every launch on the session has completed.
int swk_pull_destroy(void* h) {
  PullSession* p = static_cast<PullSession*>(h);
  int r = 0;
  r |= pull_queue_destroy(p->q);
  r |= host_free(p->ctl);
  r |= dev_free(p->scratch);
  r |= host_free(p->msgs);
  delete p;
  return r;
}

}  // extern "C"
