// tests/hostsim/gpu_sim.cpp — TEST INFRASTRUCTURE, never part of the product library.
//
// A CPU stand-in for the swgpu device backend (starway_b200/csrc/gpu.h) so that the
// `pytest -m "not gpu"` suite can drive the REAL host progress engine (engine.cpp:
// connection handshake, credits, rendezvous protocol, flush, close, cancellation,
// 2-process operation) on a machine without a GPU.  "Device memory" is POSIX shared
// memory (so the CUDA-IPC exchange has something real to exercise), "kernels" run
// synchronously on the calling thread (or, with SWSIM_LINGER=1, the control kernel as a
// thread that stays for a while: see resident_lingers()), and the match step is a plain sequential
// restatement of the semantics in oracle/tagmatch.c over the same queue layout the
// CUDA kernels use.  libstarway_hostsim.so is only ever loaded by tests/.
#include <fcntl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <chrono>
#include <map>
#include <mutex>
#include <thread>
#include <string>
#include <vector>

#include "../../starway_b200/csrc/bulk_jobs.h"
#include "../../starway_b200/csrc/gpu.h"

namespace swgpu {

static thread_local std::string g_err;
// shared words of the 'device': relaxed atomic accesses where the host and a lingering 'kernel' thread may meet (on the
// GPU these are plain loads / cudaMemcpy stores; the protocol does not depend on their order, see Pass::snapshot)
template <class T>
static inline void st_rlx(T* p, T v) { __atomic_store_n(p, v, __ATOMIC_RELAXED); }
template <class T>
static inline T ld_rlx(const T* p) { return __atomic_load_n(p, __ATOMIC_RELAXED); }
static std::mutex g_mu;
struct DevAlloc {
  size_t size;
  std::string name;
  uint64_t id;
  bool noexport = false;   // stands for memory of the CUDA virtual-memory-management API: ipc_get refuses it
};
static std::map<uintptr_t, DevAlloc> g_allocs;       // our "device" allocations (shm backed)
static std::map<uintptr_t, size_t> g_opened;         // mappings opened through ipc_open
static int g_counter = 0;
static int g_device = 0;
static const bool g_linger = getenv("SWSIM_LINGER") && atoi(getenv("SWSIM_LINGER")) != 0;   // see resident_lingers()
static std::atomic<int> g_residents{0};   // 'kernels' that are still running (threads)

const char* backend_name() { return "hostsim (test only)"; }
const char* last_error() { return g_err.c_str(); }
int device_count() {
  const char* e = getenv("SW_SIM_DEVICES");
  return e ? atoi(e) : 2;
}
int init(int device) {
  if (device < 0 || device >= device_count()) {
    g_err = "CUDA device ordinal out of range";
    return -1;
  }
  g_device = device;
  return 0;
}
int bind_thread(int) { return 0; }
int sm_count() { return 8; }
int clock_mhz() { return 1000; }
int device_pci_bus_id(int, char*, int) { return -1; }

static void cleanup_all() {
  for (int i = 0; i < 2000 && g_residents.load() > 0; i++) usleep(100);   // let lingering 'kernels' leave first
  std::lock_guard<std::mutex> lk(g_mu);
  for (auto& kv : g_allocs) shm_unlink(kv.second.name.c_str());
}

void* dev_alloc_raw(size_t bytes) {
  static bool registered = false;
  std::lock_guard<std::mutex> lk(g_mu);
  if (!registered) {
    atexit(cleanup_all);
    registered = true;
  }
  char name[64];
  snprintf(name, sizeof(name), "/swsim-%d-%d", (int)getpid(), g_counter++);
  int fd = shm_open(name, O_CREAT | O_EXCL | O_RDWR, 0600);
  if (fd < 0) {
    g_err = "shm_open failed";
    return nullptr;
  }
  size_t sz = ((bytes ? bytes : 16) + 4095) & ~(size_t)4095;
  if (ftruncate(fd, (off_t)sz) != 0) {
    close(fd);
    shm_unlink(name);
    g_err = "ftruncate failed";
    return nullptr;
  }
  void* p = mmap(nullptr, sz, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (p == MAP_FAILED) {
    shm_unlink(name);
    g_err = "mmap failed";
    return nullptr;
  }
  g_allocs[(uintptr_t)p] = DevAlloc{sz, name, ((uint64_t)getpid() << 32) | (uint64_t)g_counter};
  return p;
}
void* dev_alloc(size_t bytes) { return dev_alloc_raw(bytes); }  // fresh shm is zero-filled
int dev_free(void* p) {
  if (!p) return 0;
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_allocs.find((uintptr_t)p);
  if (it == g_allocs.end()) {
    g_err = "dev_free: unknown pointer";
    return -1;
  }
  shm_unlink(it->second.name.c_str());
  munmap(p, it->second.size);
  g_allocs.erase(it);
  return 0;
}
void* host_alloc(size_t bytes) {
  void* p = nullptr;
  if (posix_memalign(&p, 4096, bytes ? bytes : 16) != 0) return nullptr;
  memset(p, 0, bytes);
  return p;
}
int host_free(void* p) {
  free(p);
  return 0;
}

int ipc_get(const void* alloc_base, uint8_t handle[64]) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_allocs.find((uintptr_t)alloc_base);
  if (it == g_allocs.end()) {
    g_err = "ipc_get: not the base of a device allocation";
    return -1;
  }
  if (it->second.noexport) {
    g_err = "ipc_get: invalid argument (allocation cannot be exported)";
    return -1;
  }
  memset(handle, 0, 64);
  snprintf((char*)handle, 48, "%s", it->second.name.c_str());
  uint64_t sz = it->second.size;
  memcpy(handle + 48, &sz, 8);
  uint32_t pid = (uint32_t)getpid();
  memcpy(handle + 56, &pid, 4);
  return 0;
}
int ipc_open(const uint8_t handle[64], void** out) {
  uint32_t pid;
  memcpy(&pid, handle + 56, 4);
  if (pid == (uint32_t)getpid()) {
    // CUDA refuses to open a handle in the process that exported it
    g_err = "ipc_open: invalid device context (same process)";
    return -1;
  }
  char name[49];
  memcpy(name, handle, 48);
  name[48] = 0;
  uint64_t sz;
  memcpy(&sz, handle + 48, 8);
  int fd = shm_open(name, O_RDWR, 0600);
  if (fd < 0) {
    g_err = "ipc_open: shm_open failed";
    return -1;
  }
  void* p = mmap(nullptr, sz, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (p == MAP_FAILED) {
    g_err = "ipc_open: mmap failed";
    return -1;
  }
  std::lock_guard<std::mutex> lk(g_mu);
  g_opened[(uintptr_t)p] = sz;
  *out = p;
  return 0;
}
int ipc_close(void* p) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_opened.find((uintptr_t)p);
  if (it == g_opened.end()) return -1;
  munmap(p, it->second);
  g_opened.erase(it);
  return 0;
}
int ptr_info(const void* p, PtrInfo* out) {
  memset(out, 0, sizeof(*out));
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_allocs.upper_bound((uintptr_t)p);
  if (it != g_allocs.begin()) {
    --it;
    if ((uintptr_t)p < it->first + it->second.size) {
      out->is_device = 1;
      out->device = g_device;
      out->base = it->first;
      out->size = it->second.size;
      out->buffer_id = it->second.id;
    }
  }
  return 0;
}

stream_t stream_create() { return (stream_t)(uintptr_t)1; }
int stream_destroy(stream_t) { return 0; }
int stream_sync(stream_t) { return 0; }
int stream_query(stream_t) { return 0; }
event_t event_create(int) { return (event_t)(uintptr_t)1; }
int event_destroy(event_t) { return 0; }
int event_record(event_t, stream_t) { return 0; }
int event_query(event_t) { return 0; }
int event_sync(event_t) { return 0; }
float event_elapsed_ms(event_t, event_t) { return 0.001f; }
int memcpy_h2d(void* d, const void* s, size_t n, stream_t) { memcpy(d, s, n); return 0; }
int memcpy_batch(void* const* d, const void* const* s, const size_t* z, size_t n, stream_t) {
  for (size_t i = 0; i < n; i++) memcpy(d[i], s[i], z[i]);
  return 0;
}
int memcpy_h2d_batch(void* const* d, const void* const* s, const size_t* z, size_t n, stream_t) {
  for (size_t i = 0; i < n; i++) memcpy(d[i], s[i], z[i]);
  return 0;
}
int memcpy_d2h(void* d, const void* s, size_t n, stream_t) { memcpy(d, s, n); return 0; }
int memcpy_d2d(void* d, const void* s, size_t n, stream_t) { memmove(d, s, n); return 0; }
int memset_dev(void* d, int v, size_t n, stream_t) { memset(d, v, n); return 0; }
int upload(void* d, const void* s, size_t n) { memcpy(d, s, n); return 0; }

// ---------------------------------------------------------------- match state (host memory)
SwMatchState* match_state_create(uint32_t hs, uint32_t hb) {
  SwMatchState* st = (SwMatchState*)calloc(1, sizeof(SwMatchState));
  st->p_tag = (uint64_t*)calloc(SW_PQ_CAP, 8);
  st->p_mask = (uint64_t*)calloc(SW_PQ_CAP, 8);
  st->p_buf = (uint64_t*)calloc(SW_PQ_CAP, 8);
  st->p_cap = (uint64_t*)calloc(SW_PQ_CAP, 8);
  st->p_op = (uint64_t*)calloc(SW_PQ_CAP, 8);
  st->p_valid = (uint32_t*)calloc(SW_PQ_CAP, 4);
  st->u_tag = (uint64_t*)calloc(SW_UQ_CAP, 8);
  st->u_len = (uint64_t*)calloc(SW_UQ_CAP, 8);
  st->u_data = (uint64_t*)calloc(SW_UQ_CAP, 8);
  st->u_meta = (uint32_t*)calloc(SW_UQ_CAP, 4);
  st->u_blk = (uint32_t*)calloc(SW_UQ_CAP, 4);
  st->cap_small = hs;
  st->cap_big = hb;
  st->heap_small = (uint8_t*)calloc((size_t)hs, SW_HEAP_SMALL_BYTES);
  st->heap_big = (uint8_t*)calloc((size_t)hb, SW_HEAP_BIG_BYTES);
  st->free_small = (uint32_t*)calloc(hs, 4);
  st->free_big = (uint32_t*)calloc(hb, 4);
  for (uint32_t i = 0; i < hs; i++) st->free_small[i] = i;
  for (uint32_t i = 0; i < hb; i++) st->free_big[i] = i;
  st->n_free_small = hs;
  st->n_free_big = hb;
  return st;
}
int match_state_destroy(SwMatchState* st) {
  if (!st) return -1;
  void* ptrs[] = {st->p_tag, st->p_mask, st->p_buf, st->p_cap, st->p_op, st->p_valid, st->u_tag, st->u_len, st->u_data,
                  st->u_meta, st->u_blk, st->heap_small, st->heap_big, st->free_small, st->free_big};
  for (void* p : ptrs) free(p);
  free(st);
  return 0;
}
int match_state_set_ring(SwMatchState* st, uint32_t ep, void* ring_base, uint32_t slots, uint32_t gen) {
  if (ep >= SW_MAX_EPS) return -1;
  st_rlx(&st->ring_gen[ep], gen);
  st_rlx(&st->ring_base[ep], (uint64_t)(uintptr_t)ring_base);
  st_rlx(&st->ring_slots[ep], slots);
  st_rlx(&st->ring_cons[ep], (uint64_t)0);
  return 0;
}

// ---------------------------------------------------------------- "kernels"
int launch_put(stream_t, const SwPutDesc* descs, uint32_t n, const DoneFlag* done) {
  for (uint32_t i = 0; i < n; i++) {
    const SwPutDesc& d = descs[i];
    uint8_t* slot = (uint8_t*)(uintptr_t)d.dst;
    if (d.len) memcpy(slot + SW_SLOT_HDR, (const void*)(uintptr_t)d.src, d.len);
    SwSlotHdr h;
    memset(&h, 0, sizeof(h));
    h.tag = d.tag;
    h.len = d.msg_len;
    h.seq = d.seq;
    h.kind = d.kind;
    h.magic = SW_SLOT_MAGIC;
    // same order as sw_put_header: tag / length / kind / magic, then the sequence word (the arrival flag) with
    // release semantics
    memcpy(slot, &h, 16);
    memcpy(slot + 24, &h.kind, 8);
    __atomic_store_n(reinterpret_cast<uint64_t*>(slot + 16), h.seq, __ATOMIC_RELEASE);
  }
  // same split as the CUDA backend: only the small (single-CTA) variant announces itself by flag
  uint32_t n_rts = 0;
  for (uint32_t i = 0; i < n; i++) n_rts += descs[i].kind == SW_KIND_RTS;
  if (done && n <= 32 && n_rts <= 16) {
    __atomic_store_n((uint64_t*)done->flag, done->value, __ATOMIC_RELEASE);
    return 1;
  }
  return 0;
}

int launch_bulk(stream_t, const SwSeg* segs, uint32_t nseg, const BulkTuning* t) {
  // Balanced launches run the SAME job builder and per-CTA range iterator as the CUDA kernel
  // (bulk_jobs.h, SwJobRangeIter): one loop iteration per CTA, memcpy in place of the TMA pipeline.
  SwBulkJobArgs ja;
  uint32_t grid = 0;
  if (t && t->mode == 0 && t->balance &&
      bulk_build_jobs(segs, nseg, 132, (uint32_t)(t->stage_bytes & ~15), (uint32_t)t->stages, &ja, &grid)) {
    if (getenv("SW_SIM_TRACE_BULK")) fprintf(stderr, "simjobs njobs=%u grid=%u share=%llu total=%llu\n", ja.njobs, grid, (unsigned long long)ja.share, (unsigned long long)ja.end[ja.njobs - 1]);
    uint64_t copied = 0, want = ja.end[ja.njobs - 1];
    for (uint32_t cta = 0; cta < grid; cta++) {
      SwJobRangeIter it;
      it.init(ja, cta);
      uint64_t src, dst;
      uint32_t bytes;
      while (it.next(ja, src, dst, bytes)) {
        if (((src | dst | bytes) & 15) || bytes > ja.stage_bytes) {
          g_err = "bulk job iterator produced a misaligned / oversized piece";
          return -1;
        }
        memcpy((void*)(uintptr_t)dst, (const void*)(uintptr_t)src, bytes);
        copied += bytes;
      }
    }
    if (copied != want) {
      g_err = "bulk job iterator did not cover the launch";
      return -1;
    }
    return 0;
  }
  for (uint32_t i = 0; i < nseg; i++)
    memcpy((void*)(uintptr_t)segs[i].dst, (const void*)(uintptr_t)segs[i].src, segs[i].len);
  return 0;
}

// ---------------------------------------------------------------- resident progress path (one pass per launch)
// The CUDA backend keeps sw_progress_kernel / sw_pull_kernel resident; this stand-in performs ONE pass of the
// same protocol per launch, synchronously: post ring -> matching -> eager delivery / rendezvous copy through the
// mapping table -> completion rings, credit words and FIN words -> exit word.  The host engine cannot tell the
// difference except that nothing happens between launches (resident_lingers() == 0).
// SWSIM_LINGER=1: a launch becomes a THREAD that repeats the pass until the host asks it to stop, linger_us of silence or
// max_life_us have passed -- the resident behaviour of the CUDA kernels (engine.cpp then uses everything that depends on a
// kernel being there: puts handed over through the stamped send ring, the armed relaunch policy, stop / epoch hand-shakes
// with a kernel that runs concurrently).  Default: one synchronous pass per launch.
int resident_lingers() { return g_linger ? 1 : 0; }
void* host_register(void* p, size_t) { return p; }
int host_unregister(void*) { return 0; }
int match_state_set_ep_words(SwMatchState* st, uint32_t ep, void* credit_word, void* fin_words) {
  if (ep >= SW_MAX_EPS) return -1;
  st_rlx(&st->credit_ptr[ep], (uint64_t)(uintptr_t)credit_word);
  st_rlx(&st->fin_ptr[ep], (uint64_t)(uintptr_t)fin_words);
  return 0;
}
SwPullQueue* pull_queue_create() { return (SwPullQueue*)calloc(1, sizeof(SwPullQueue)); }
int pull_queue_destroy(SwPullQueue* q) {
  free(q);
  return 0;
}
SwMapEnt* map_table_create() { return (SwMapEnt*)calloc(SW_MAP_SLOTS, sizeof(SwMapEnt)); }
int map_table_destroy(SwMapEnt* t) {
  free(t);
  return 0;
}
int map_table_clear(SwMapEnt* t) {
  memset(t, 0, sizeof(SwMapEnt) * SW_MAP_SLOTS);
  return 0;
}
int map_table_insert(SwMapEnt* t, stream_t, uint64_t uuid, uint64_t buf_id, uint64_t remote_base, uint64_t local_base) {
  const uint32_t home = sw_map_home(uuid, buf_id);
  for (uint32_t k = 0; k < SW_MAP_PROBE; k++) {
    SwMapEnt& e = t[(home + k) & (SW_MAP_SLOTS - 1)];
    if (e.buf_id) continue;
    e.remote_base = remote_base;
    e.local_base = local_base;
    e.uuid = uuid;
    __atomic_store_n(&e.buf_id, buf_id, __ATOMIC_RELEASE);
    return 0;
  }
  g_err = "mapping table: probe window full";
  return -1;
}
int pull_default_ctas() { return 8; }
int probe_publish_batch(stream_t, SwPullQueue*, const SwSeg*, uint32_t, uint32_t, void*) { return -1; }
int pull_queue_read_stats(SwPullQueue*, uint64_t*) { return -1; }

namespace {
template <class T>
static inline T ld(const volatile T* p) { return __atomic_load_n(const_cast<const T*>(p), __ATOMIC_ACQUIRE); }

struct Pass {
  const ProgressLaunch* a;
  SwMatchState* st;
  SwProgCtl* ctl;
  // ring geometry and cursors as of the launch (the CUDA kernel keeps them in shared memory): a ring attached while
  // this launch runs is not seen, and only the cursors of the rings it knew go back to the match state
  uint64_t ring_base[SW_MAX_EPS], cons[SW_MAX_EPS], credit_ptr[SW_MAX_EPS], fin_ptr[SW_MAX_EPS];
  uint32_t ring_slots[SW_MAX_EPS], ring_gen[SW_MAX_EPS];
  void snapshot() {
    for (uint32_t e = 0; e < SW_MAX_EPS; e++) {
      ring_base[e] = ld_rlx(&st->ring_base[e]);
      ring_slots[e] = ld_rlx(&st->ring_slots[e]);
      ring_gen[e] = ld_rlx(&st->ring_gen[e]);
      cons[e] = ld_rlx(&st->ring_cons[e]);
      credit_ptr[e] = ld_rlx(&st->credit_ptr[e]);
      fin_ptr[e] = ld_rlx(&st->fin_ptr[e]);
    }
  }
  void write_back() {
    for (uint32_t e = 0; e < SW_MAX_EPS; e++)
      if (ring_base[e]) st_rlx(&st->ring_cons[e], cons[e]);
  }
  bool rings_full() const {
    return st->cq_alloc - ld(&ctl->cq_head) + 8 > SW_CQ_RING || st->cqr_alloc - ld(&ctl->cqr_head) + 8 > SW_CQ_RING ||
           st->hr_alloc - ld(&ctl->hr_head) + 8 > SW_HR_RING;
  }
  static void cqe(SwCqEnt* ring, uint64_t idx, uint64_t op, uint64_t tag, uint64_t len, int32_t status) {
    SwCqEnt* e = &ring[idx % SW_CQ_RING];
    e->op_id = op;
    e->tag = tag;
    e->len = len;
    const uint64_t w = ((uint64_t)sw_ring_pass(idx, SW_CQ_RING) << 32) | (uint32_t)status;
    __atomic_store_n(reinterpret_cast<uint64_t*>(&e->status), w, __ATOMIC_RELEASE);
  }
  void deliver(uint64_t src, uint64_t dst, uint64_t msg_len, uint64_t cap, uint64_t op, uint64_t tag) {
    const bool trunc = msg_len > cap;
    if (!trunc && msg_len) memcpy((void*)(uintptr_t)dst, (const void*)(uintptr_t)src, msg_len);
    cqe(a->cq, st->cq_alloc++, op, tag, msg_len, trunc ? SW_ERR_MESSAGE_TRUNCATED : SW_OK);
  }
  uint64_t map_lookup(uint64_t uuid, uint64_t buf_id, uint64_t remote_base) const {
    if (!a->map || !buf_id) return 0;
    const uint32_t home = sw_map_home(uuid, buf_id);
    for (uint32_t k = 0; k < SW_MAP_PROBE; k++) {
      const SwMapEnt& e = a->map[(home + k) & (SW_MAP_SLOTS - 1)];
      if (__atomic_load_n(&e.buf_id, __ATOMIC_ACQUIRE) == buf_id && e.uuid == uuid) return e.remote_base == remote_base ? e.local_base : 0;
    }
    return 0;
  }
  // same decision as sw_res_rts
  void rts(uint64_t payload, uint64_t stag, uint64_t msg_len, uint32_t epf, uint64_t buf, uint64_t cap, uint64_t op, uint32_t pflags) {
    SwRts r;
    memcpy(&r, (const void*)(uintptr_t)payload, sizeof(r));
    const uint32_t ep = epf & ((1u << SW_EP_IDX_BITS) - 1);
    const bool trunc = msg_len > cap;
    bool device_path = a->pq && a->pull_ctas && !trunc && !(pflags & SW_POST_HOSTPATH) && !(r.pad[0] & SW_RTS_PINNED_SRC) &&
                       !((ld(&ctl->dead_mask) >> ep) & 1) && fin_ptr[ep] && (epf >> SW_EP_IDX_BITS) == (ring_gen[ep] & SW_EP_GEN_MASK);
    uint64_t src = 0;
    if (device_path) {
      if (r.ctx_uuid == a->ctx_uuid && r.src_pid == a->pid) {
        src = r.src_ptr;
      } else {
        const uint64_t local = map_lookup(r.ctx_uuid, r.pad[1], r.alloc_base);
        if (local && r.src_ptr >= r.alloc_base && r.src_ptr - r.alloc_base + msg_len <= r.alloc_size) src = local + (r.src_ptr - r.alloc_base);
      }
      if (!src || ((src | buf) & 15)) device_path = false;
    }
    if (device_path) {
      // what the pull CTAs do: copy, completion record, FIN word of the sender, statistics
      if (msg_len) memcpy((void*)(uintptr_t)buf, (const void*)(uintptr_t)src, msg_len);
      cqe(a->cqr, st->cqr_alloc++, op, stag, msg_len, SW_OK);
      __atomic_store_n(reinterpret_cast<uint64_t*>(fin_ptr[ep] + 8ull * (r.send_seq % SW_FIN_SLOTS)), (r.send_seq << 2) | 1, __ATOMIC_RELEASE);
      st->pull_jobs++;
      __atomic_fetch_add(&a->pq->bytes, msg_len & ~15ull, __ATOMIC_RELAXED);   // one queue per context: several workers
      __atomic_fetch_add(&a->pq->busy_ns, (uint64_t)1000, __ATOMIC_RELAXED);
      __atomic_fetch_add(&a->pq->batches, (uint64_t)1, __ATOMIC_RELAXED);
      __atomic_fetch_add(&a->pq->jobs, (uint64_t)1, __ATOMIC_RELAXED);
      return;
    }
    SwHrEnt* h = &a->hr[st->hr_alloc % SW_HR_RING];
    h->rec.rts = r;
    h->rec.op_id = op;
    h->rec.dst = buf;
    h->rec.cap = cap;
    h->rec.tag = stag;
    h->rec.len = msg_len;
    h->rec.ep = epf;
    h->rec.status = trunc ? SW_ERR_MESSAGE_TRUNCATED : SW_OK;
    h->pad = 0;
    __atomic_store_n(&h->seq, sw_ring_pass(st->hr_alloc, SW_HR_RING), __ATOMIC_RELEASE);
    st->hr_alloc++;
  }
};
}  // namespace

namespace {
// One pass of the control kernel.  Returns whether anything was consumed (receives, arrivals, puts).
bool run_pass(Pass& p) {
  const ProgressLaunch* a = p.a;
  const uint64_t PQM = SW_PQ_CAP - 1, UQM = SW_UQ_CAP - 1;
  SwMatchState* st = p.st;
  SwProgCtl* ctl = p.ctl;
  const uint64_t epoch = __atomic_load_n(&ctl->host_epoch, __ATOMIC_ACQUIRE);
  bool stalled = false, did = false;
  // ---- puts handed over by the host (only a kernel that stays gets any): stamped units -> entry -> slot
  if (g_linger && a->sends) {
    const uint64_t tail = __atomic_load_n(&ctl->send_tail, __ATOMIC_ACQUIRE);
    while (st->send_consumed < tail) {
      const SwSendLL* le = &a->sends[st->send_consumed % SW_SEND_RING];
      uint32_t w[SW_SEND_UNITS * 3];
      for (uint32_t k = 0; k < SW_SEND_UNITS; k++) {
        memcpy(&w[3 * k], le->u[k], 12);
        if (le->u[k][3] != sw_send_stamp(st->send_consumed)) ctl->err = ctl->err | 2;   // the host's encoding is wrong
      }
      SwSendEnt e;
      memcpy(&e, w, sizeof e);
      SwPutDesc d = e.d;
      d.kind &= ~SW_KIND_SAME_GPU;
      if (d.src == 0) d.src = (uint64_t)(uintptr_t)e.inl;
      launch_put(nullptr, &d, 1, nullptr);
      st->send_consumed++;
      did = true;
    }
    ctl->send_head = st->send_consumed;
    __atomic_store_n(&ctl->send_done, st->send_consumed, __ATOMIC_RELEASE);
  }
  // ---- new receives, in post order, against the unexpected queue (earliest arrival first)
  while (st->post_consumed < __atomic_load_n(&ctl->post_tail, __ATOMIC_ACQUIRE) && !p.rings_full()) {
    const SwPostEnt e = a->posts[st->post_consumed % SW_POST_RING];
    st->post_consumed++;
    did = true;
    bool found = false;
    for (uint64_t idx = st->u_head; idx < st->u_tail; idx++) {
      const uint64_t s = idx & UQM;
      const uint32_t meta = st->u_meta[s];
      if (!(meta & SW_UMETA_VALID) || !sw_tag_match(st->u_tag[s], e.tag, e.mask)) continue;
      st->u_meta[s] = 0;
      st->u_count--;
      if (meta & SW_UMETA_RTS)
        p.rts(st->u_data[s], st->u_tag[s], st->u_len[s], meta & SW_UMETA_EPMASK, e.buf, e.cap, e.op_id, e.flags);
      else
        p.deliver(st->u_data[s], e.buf, st->u_len[s], e.cap, e.op_id, st->u_tag[s]);
      if (meta & SW_UMETA_BIG)
        st->free_big[st->n_free_big++] = st->u_blk[s];
      else
        st->free_small[st->n_free_small++] = st->u_blk[s];
      found = true;
      break;
    }
    while (st->u_head < st->u_tail && !(st->u_meta[st->u_head & UQM] & SW_UMETA_VALID)) st->u_head++;
    if (found) continue;
    if (st->p_tail - st->p_head >= SW_PQ_CAP) {
      Pass::cqe(a->cq, st->cq_alloc++, e.op_id, 0, 0, SW_ERR_NO_MEMORY);
      continue;
    }
    const uint64_t s = st->p_tail & PQM;
    st->p_tag[s] = e.tag;
    st->p_mask[s] = e.mask;
    st->p_buf[s] = e.buf;
    st->p_cap[s] = e.cap;
    st->p_op[s] = e.op_id;
    st->p_valid[s] = 1u | (e.flags << 8);
    st->p_tail++;
    st->p_count++;
  }
  __atomic_store_n(&ctl->post_head, st->post_consumed, __ATOMIC_RELEASE);
  // ---- arrivals: a slot has arrived when its header carries the expected sequence number
  for (uint32_t k = 0; k < a->n_eps; k++) {
    const uint32_t ep = (st->rr_ep + k) % a->n_eps;
    if (!p.ring_base[ep]) continue;
    const uint32_t epf = ep | ((p.ring_gen[ep] & SW_EP_GEN_MASK) << SW_EP_IDX_BITS);
    uint64_t cons = p.cons[ep];
    for (;;) {
      if (p.rings_full()) break;
      const uint8_t* slot = (const uint8_t*)(uintptr_t)(p.ring_base[ep] + (cons & (p.ring_slots[ep] - 1)) * SW_SLOT_BYTES);
      if (__atomic_load_n(reinterpret_cast<const uint64_t*>(slot + 16), __ATOMIC_ACQUIRE) != cons + 1) break;
      SwSlotHdr h;
      memcpy(&h, slot, 32);
      if (h.magic != SW_SLOT_MAGIC) ctl->err |= 1;
      const bool is_rts = h.kind == SW_KIND_RTS;
      const uint64_t payload = (uint64_t)(uintptr_t)(slot + SW_SLOT_HDR);
      bool found = false;
      for (uint64_t idx = st->p_head; idx < st->p_tail; idx++) {
        const uint64_t s = idx & PQM;
        if (!st->p_valid[s] || !sw_tag_match(h.tag, st->p_tag[s], st->p_mask[s])) continue;
        const uint32_t pflags = st->p_valid[s] >> 8;
        st->p_valid[s] = 0;
        st->p_count--;
        if (is_rts)
          p.rts(payload, h.tag, h.len, epf, st->p_buf[s], st->p_cap[s], st->p_op[s], pflags);
        else
          p.deliver(payload, st->p_buf[s], h.len, st->p_cap[s], st->p_op[s], h.tag);
        found = true;
        break;
      }
      while (st->p_head < st->p_tail && !st->p_valid[st->p_head & PQM]) st->p_head++;
      if (!found) {
        const uint64_t need = is_rts ? sizeof(SwRts) : h.len;
        const bool big = need > SW_HEAP_SMALL_BYTES;
        if ((big ? st->n_free_big : st->n_free_small) == 0 || st->u_tail - st->u_head >= SW_UQ_CAP) {
          stalled = true;   // back-pressure: the message stays in its ring slot
          break;
        }
        const uint32_t blk = big ? st->free_big[--st->n_free_big] : st->free_small[--st->n_free_small];
        const uint64_t haddr = big ? (uint64_t)(uintptr_t)st->heap_big + (uint64_t)blk * SW_HEAP_BIG_BYTES
                                   : (uint64_t)(uintptr_t)st->heap_small + (uint64_t)blk * SW_HEAP_SMALL_BYTES;
        if (need) memcpy((void*)(uintptr_t)haddr, (const void*)(uintptr_t)payload, need);
        const uint64_t s = st->u_tail & UQM;
        st->u_tag[s] = h.tag;
        st->u_len[s] = h.len;
        st->u_data[s] = haddr;
        st->u_blk[s] = blk;
        st->u_meta[s] = SW_UMETA_VALID | (big ? SW_UMETA_BIG : 0) | (is_rts ? SW_UMETA_RTS : 0) | (epf & SW_UMETA_EPMASK);
        st->u_tail++;
        st->u_count++;
      }
      cons++;
      st->arrivals++;
    }
    if (cons != p.cons[ep]) {
      p.cons[ep] = cons;
      did = true;
      if (p.credit_ptr[ep]) __atomic_store_n(reinterpret_cast<uint64_t*>(p.credit_ptr[ep]), cons, __ATOMIC_RELEASE);
    }
  }
  st->rr_ep++;
  __atomic_store_n(&ctl->pull_jobs, st->pull_jobs, __ATOMIC_RELEASE);
  __atomic_store_n(&ctl->arrivals, st->arrivals, __ATOMIC_RELAXED);
  __atomic_store_n(&ctl->n_posted, st->p_count, __ATOMIC_RELAXED);
  __atomic_store_n(&ctl->n_unexp, st->u_count, __ATOMIC_RELAXED);
  __atomic_store_n(&ctl->stalled, (uint64_t)(stalled ? 1 : 0), __ATOMIC_RELAXED);
  __atomic_store_n(&ctl->iterations, ctl->iterations + 1, __ATOMIC_RELAXED);
  __atomic_store_n(&ctl->dev_epoch, epoch, __ATOMIC_RELEASE);
  return did;
}

void finish_launch(Pass& p, uint64_t reason, uint64_t life_us) {
  p.write_back();
  p.ctl->exit_reason = reason;
  p.ctl->life_us = life_us;
  __atomic_store_n(&p.ctl->exit_seq, p.a->launch_seq, __ATOMIC_RELEASE);   // last: the host may free everything now
}
}  // namespace

int launch_progress(stream_t, const ProgressLaunch* a) {
  if (!g_linger) {
    Pass p;
    p.a = a;
    p.st = a->st;
    p.ctl = a->ctl;
    p.snapshot();
    run_pass(p);
    finish_launch(p, 2, 1);
    return 0;
  }
  g_residents.fetch_add(1);
  const ProgressLaunch args = *a;
  std::thread([args]() {
    using clock = std::chrono::steady_clock;
    auto us_since = [](clock::time_point t) { return std::chrono::duration_cast<std::chrono::microseconds>(clock::now() - t).count(); };
    Pass* p = new Pass;   // (two 512-entry tables: not on a small thread stack)
    p->a = &args;
    p->st = args.st;
    p->ctl = args.ctl;
    p->snapshot();
    const auto t0 = clock::now();
    auto last = t0;
    uint64_t reason = 0;
    while (!reason) {
      const bool did = run_pass(*p);
      if (did) last = clock::now();
      if (__atomic_load_n(&args.ctl->stop, __ATOMIC_ACQUIRE)) reason = 1;
      else if (us_since(last) > (long long)args.linger_us) reason = 2;
      else if (us_since(t0) > (long long)args.max_life_us) reason = 3;
      else if (!did) std::this_thread::sleep_for(std::chrono::microseconds(3));
    }
    const uint64_t life = (uint64_t)us_since(t0);
    finish_launch(*p, reason, life ? life : 1);
    delete p;
    g_residents.fetch_sub(1);
  }).detach();
  return 0;
}

// the copies were made by the pass that matched them: the "pull kernel" only reports and leaves
int launch_pull(stream_t, SwPullQueue* q, SwPullCtl* ctl, uint64_t launch_seq, uint32_t, uint32_t, uint32_t, const BulkTuning*) {
  ctl->bytes = __atomic_load_n(&q->bytes, __ATOMIC_RELAXED);
  ctl->busy_ns = __atomic_load_n(&q->busy_ns, __ATOMIC_RELAXED);
  ctl->batches = __atomic_load_n(&q->batches, __ATOMIC_RELAXED);
  ctl->jobs = __atomic_load_n(&q->jobs, __ATOMIC_RELAXED);
  __atomic_store_n(&ctl->exited, launch_seq, __ATOMIC_RELEASE);
  return 0;
}

}  // namespace swgpu

// Test-only exports (tests/hostsim/exports_sim.map): "device" buffers for the Python tests, so that the
// engine's device-buffer paths (zero-copy rendezvous between user buffers, IPC export of user
// allocations, handle / mapping caches) run on the CPU as well.
extern "C" void* swsim_dev_alloc(size_t bytes) { return swgpu::dev_alloc(bytes); }
// a 'device' buffer the IPC export refuses (what cudaIpcGetMemHandle does for cuMemCreate / expandable-segment memory)
extern "C" void* swsim_dev_alloc_noexport(size_t bytes) {
  void* p = swgpu::dev_alloc(bytes);
  if (p) {
    std::lock_guard<std::mutex> lk(swgpu::g_mu);
    swgpu::g_allocs[(uintptr_t)p].noexport = true;
  }
  return p;
}
extern "C" int swsim_dev_free(void* p) { return swgpu::dev_free(p); }

