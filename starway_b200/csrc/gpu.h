// starway_b200 — the narrow interface between the host progress engine
// (engine.cpp) and the device backend.  The product backend is gpu_cuda.cu
// (hand-written sm_90a kernels).  tests/hostsim/gpu_sim.cpp is a test-only
// stand-in that lets the CPU test-suite exercise the host protocol logic
// without a GPU; it is never linked into the product library.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "sw_device.h"

namespace swgpu {

typedef void* stream_t;
typedef void* event_t;

struct PtrInfo {
  int is_device;      // 1: device memory, 0: host (pageable or pinned)
  int is_pinned;      // host memory registered/pinned with CUDA (device accessible)
  int device;         // ordinal for device memory
  uint64_t base;      // allocation base (device memory)
  uint64_t size;      // allocation size (device memory)
  uint64_t buffer_id; // unique id of the allocation (changes when the address is re-allocated); 0: unknown
};

struct BulkTuning {
  int mode;           // 0: TMA-staged (cp.async.bulk), 1: SIMT vectorised
  int stages;         // TMA smem stages per CTA (2..8)
  int stage_bytes;    // bytes per stage (multiple of 16)
  int ctas_per_sm;    // resident CTAs per SM targeted
  int balance;        // TMA mode: 1 = equal byte range per CTA when the launch has <= 96 jobs (see bulk_jobs.h)
};

const char* backend_name();
const char* last_error();

int device_count();
int init(int device);                 // binds the calling thread to `device`
int bind_thread(int device);          // cudaSetDevice for helper threads
int sm_count();
int clock_mhz();                       // SM clock that converts device cycle counts to time
int device_pci_bus_id(int device, char* out, int cap);   // "0000:1b:00.0"; < 0 when unknown

void* dev_alloc(size_t bytes);        // IPC-shareable device allocation, zeroed
void* dev_alloc_raw(size_t bytes);    // same, contents undefined (large staging buffers)
int dev_free(void* p);
void* host_alloc(size_t bytes);       // pinned, device-mapped host memory, zeroed
int host_free(void* p);

int ipc_get(const void* alloc_base, uint8_t handle[64]);
int ipc_open(const uint8_t handle[64], void** out);
int ipc_close(void* p);
int ptr_info(const void* p, PtrInfo* out);

stream_t stream_create();
int stream_destroy(stream_t s);
int stream_sync(stream_t s);
int stream_query(stream_t s);   // 0: idle, 1: work pending, < 0: a launch on the stream failed
event_t event_create(int timing);
int event_destroy(event_t e);
int event_record(event_t e, stream_t s);
int event_query(event_t e);           // 0: complete, 1: not ready, <0: error
int event_sync(event_t e);
float event_elapsed_ms(event_t a, event_t b);

int memcpy_h2d(void* dst, const void* src, size_t n, stream_t s);
// n host -> device copies as ONE copy-engine submission (cudaMemcpyBatchAsync): separate 1 MiB copies each pay a start-up
// cost that grows while the other direction of the link is busy, the batch pays it once (`sw_probe duplex` compares them)
int memcpy_h2d_batch(void* const* dsts, const void* const* srcs, const size_t* sizes, size_t n, stream_t s);
int memcpy_batch(void* const* dsts, const void* const* srcs, const size_t* sizes, size_t n, stream_t s);   // any direction
int memcpy_d2h(void* dst, const void* src, size_t n, stream_t s);
int memcpy_d2d(void* dst, const void* src, size_t n, stream_t s);
int memset_dev(void* dst, int v, size_t n, stream_t s);
int upload(void* dst_dev, const void* src_host, size_t n);   // synchronous small upload

// Build/destroy the device-resident queues of one worker.
SwMatchState* match_state_create(uint32_t heap_small_blocks, uint32_t heap_big_blocks);
int match_state_destroy(SwMatchState* st);
int match_state_set_ring(SwMatchState* st, uint32_t ep, void* ring_base, uint32_t slots, uint32_t gen = 0);

// Kernel launches (asynchronous on `s`).
// Completion flag: a word in pinned host memory that a single-CTA launch stores `value` to (system
// scope, after all its other stores) so that the host can spin on memory instead of on a CUDA event.
// launch_put returns 1 when the launch will write the flag, 0 when the batch is too large for the
// flag-writing variant (the caller records an event instead), < 0 on error.
struct DoneFlag {
  volatile uint64_t* flag;
  uint64_t value;            // non-zero
};
int launch_put(stream_t s, const SwPutDesc* descs, uint32_t n, const DoneFlag* done = nullptr);
int launch_bulk(stream_t s, const SwSeg* segs, uint32_t nseg, const BulkTuning* tune);

// ---------------------------------------------------------------- resident progress path
// 1: launch_progress / launch_pull start kernels that stay resident and watch device / host memory on their
// own (the CUDA backend); 0: each launch performs one pass over what is there and returns (the CPU stand-in).
int resident_lingers();
// Page-locks an existing host mapping (the POSIX-shm control block of a connection) and returns the address
// device code uses for it; nullptr on failure.
void* host_register(void* p, size_t bytes);
int host_unregister(void* p);
// per-endpoint words of a worker's match state the control kernel publishes to (device-visible addresses)
int match_state_set_ep_words(SwMatchState* st, uint32_t ep, void* credit_word, void* fin_words);
SwPullQueue* pull_queue_create();
int pull_queue_destroy(SwPullQueue* q);
SwMapEnt* map_table_create();
int map_table_destroy(SwMapEnt* t);
// insert (exporting context, buffer id) -> (remote base, local mapped base); < 0 when the probe window is full
int map_table_insert(SwMapEnt* t, stream_t s, uint64_t uuid, uint64_t buf_id, uint64_t remote_base, uint64_t local_base);
int map_table_clear(SwMapEnt* t);

struct ProgressLaunch {
  SwMatchState* st;
  SwProgCtl* ctl;
  SwPostEnt* posts;
  SwCqEnt* cq;
  SwCqEnt* cqr;
  SwHrEnt* hr;
  SwSendLL* sends;
  SwPullQueue* pq;
  SwMapEnt* map;
  uint64_t ctx_uuid, launch_seq;
  uint32_t pid, n_eps, linger_us, max_life_us, pull_ctas;
};
int launch_progress(stream_t s, const ProgressLaunch* a);
int launch_pull(stream_t s, SwPullQueue* q, SwPullCtl* ctl, uint64_t launch_seq, uint32_t ctas, uint32_t linger_us,
                uint32_t max_life_us, const BulkTuning* tune);
int pull_default_ctas();
// measurement hook (tests/gpu_probe): publishes ONE batch of whole messages (src, dst, len; 16-byte aligned) to the
// pull queue from the device, the way a matcher does; completion records of the batch are dropped
int probe_publish_batch(stream_t s, SwPullQueue* q, const SwSeg* msgs_pinned, uint32_t n, uint32_t pull_ctas, void* scratch_dev);
int pull_queue_read_stats(SwPullQueue* q, uint64_t out[8]);   // bytes, busy_ns, batches, jobs, pickup_ns, copy_ns, fin_ns, alloc

}  // namespace swgpu
