// starway_b200 — host progress engine behind the C ABI in include/starway_b200.h.
//
// Replaces the reference's per-object UCX worker thread
// (Client::start_working / Server::start_working, reference src/bindings/main.cpp:234-550,
// 1063-1373) with ONE progress thread per context that
//   * drains a submission queue filled by sw_post_* (reference Channel<T> mailboxes, chan.hpp:84-120),
//   * batches sends into sw_put_kernel launches (eager payloads / RTS descriptors stored straight
//     into the peer's device-resident inbound ring through a CUDA-IPC mapping),
//   * feeds new receives to the resident control kernel of each worker (sw_progress_kernel), which
//     matches them against ring arrivals in device-resident posted/unexpected queues,
//   * keeps the resident pull CTAs (sw_pull_kernel) alive while rendezvous payloads are to be PULLED from
//     the sender's buffer (IPC mapping) into the caller's receive buffer, and turns the rendezvous matches
//     the device leaves to the host into sw_bulk_*_kernel launches,
//   * resolves operations by polling CUDA events (replaces ucp_worker_progress + UCX callbacks).
// Host<->host signalling (doorbells, credits, FIN/CLOSE) uses a small POSIX shared-memory
// control block per connection; the worker-address handshake (main.cpp:292-317, 912-985)
// becomes an exchange of CUDA IPC handles over a TCP / abstract-unix bootstrap socket.
//
// This file contains no CUDA: the device is reached through gpu.h only.
#include <pthread.h>
#include <sched.h>
#include "starway_b200.h"

#include <arpa/inet.h>
#include <errno.h>
#include <fcntl.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <poll.h>
#include <signal.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <linux/futex.h>
#include <sys/eventfd.h>
#include <sys/ioctl.h>
#include <sys/mman.h>
#include <sys/prctl.h>
#include <sys/socket.h>
#include <sys/stat.h>
#include <sys/syscall.h>
#include <sys/un.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <random>
#include <set>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "gpu.h"
#include "sw_device.h"
#if defined(__SSE2__)
#include <emmintrin.h>
#endif

namespace {

// ============================================================================ utilities
thread_local std::string g_last_error;
void set_error(const std::string& s) { g_last_error = s; }

// A pull grid of one CTA is CTA 0 alone, which completes batches but copies nothing: the control kernel would still
// hand rendezvous matches to it (pull_ctas != 0) and those receives would never complete.
const char* const kPullCtasOne = "1 is not a valid value: the pull kernel needs CTA 0 plus at least one copy CTA";

double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
uint64_t rand64() {
  static std::mutex mu;
  static std::mt19937_64 rng(std::random_device{}() ^ ((uint64_t)getpid() << 32) ^
                             (uint64_t)std::chrono::steady_clock::now().time_since_epoch().count());
  std::lock_guard<std::mutex> lk(mu);
  return rng();
}
bool pid_alive(uint32_t pid) { return pid == 0 || kill((pid_t)pid, 0) == 0 || errno == EPERM; }

// ============================================================================ shared control block
constexpr uint32_t SHM_MAGIC = 0x53574333u;  // "SWC3"
constexpr uint32_t CTL_RING = 256;
enum : uint32_t { CTL_FIN = 1, CTL_CLOSE = 2, CTL_CLOSE_ACK = 3, CTL_CANCEL_RTS = 4, CTL_CANCEL_ACK = 5 };

struct CtlMsg {
  uint32_t type;
  int32_t status;
  uint64_t a;
  uint64_t b;
  uint64_t pad;
};

struct alignas(64) ShmDir {  // one direction: sender side X -> receiver side Y
  alignas(64) std::atomic<uint64_t> produced;  // ring slots completely written by X (after put kernels finished)
  alignas(64) std::atomic<uint64_t> consumed;  // ring slots released by Y (credits)
  alignas(64) std::atomic<uint64_t> ctl_head;  // control messages written by X
  alignas(64) std::atomic<uint64_t> ctl_tail;  // control messages consumed by Y
  alignas(64) CtlMsg ctl[CTL_RING];
  // Rendezvous FIN words, written by Y's pull CTAs (device stores into this page-locked block), read by X:
  // word [seq % SW_FIN_SLOTS] == (seq << 2) | 1 once rendezvous `seq` of this direction has been pulled.
  alignas(64) std::atomic<uint64_t> gfin[SW_FIN_SLOTS];
};

struct ShmCtl {
  uint32_t magic;
  uint32_t version;
  uint32_t pid[2];  // [0] client, [1] server
  ShmDir dir[2];    // [0] client -> server, [1] server -> client
};

// ============================================================================ wire format (bootstrap socket)
constexpr uint32_t WIRE_MAGIC = 0x53574231u;  // "SWB1"
constexpr uint32_t ADDR_MAGIC = 0x53574144u;  // "SWAD"

struct WireHello {
  uint32_t magic, version;
  uint32_t pid;
  int32_t device;
  uint64_t ctx_uuid;
  uint64_t worker_id;
  uint8_t ring_handle[64];
  uint64_t ring_ptr;
  uint32_t ring_slots;
  uint32_t pad;
  char shm_name[64];
};
struct WireWelcome {
  uint32_t magic;
  int32_t status;
  uint32_t pid;
  int32_t device;
  uint64_t ctx_uuid;
  uint64_t worker_id;
  uint8_t ring_handle[64];
  uint64_t ring_ptr;
  uint32_t ring_slots;
  uint32_t ep_index;
};
struct AddrBlob {  // what listen_address()/get_worker_address() return (reference: UCX worker address bytes)
  uint32_t magic, version;
  uint32_t pid;
  int32_t device;
  uint64_t ctx_uuid;
  uint64_t worker_id;
  char unix_name[64];  // abstract-namespace bootstrap socket ("" for clients)
  char host[32];
};

bool write_all(int fd, const void* p, size_t n) {
  const char* c = (const char*)p;
  while (n) {
    ssize_t r = ::send(fd, c, n, MSG_NOSIGNAL);
    if (r < 0) {
      if (errno == EINTR) continue;
      return false;
    }
    c += r;
    n -= (size_t)r;
  }
  return true;
}
bool read_all(int fd, void* p, size_t n) {
  char* c = (char*)p;
  while (n) {
    ssize_t r = ::recv(fd, c, n, 0);
    if (r == 0) return false;
    if (r < 0) {
      if (errno == EINTR) continue;
      return false;
    }
    c += r;
    n -= (size_t)r;
  }
  return true;
}
void set_sock_timeout(int fd, double sec) {
  struct timeval tv;
  tv.tv_sec = (long)sec;
  tv.tv_usec = (long)((sec - (long)sec) * 1e6);
  setsockopt(fd, SOL_SOCKET, SO_RCVTIMEO, &tv, sizeof(tv));
  setsockopt(fd, SOL_SOCKET, SO_SNDTIMEO, &tv, sizeof(tv));
}

// ============================================================================ pinned bounce pool (host receive buffers)
struct HostPool {
  static constexpr int NCLS = 3;
  const size_t cls_bytes[NCLS] = {256, 4096, 65536};
  const size_t chunk_blocks[NCLS] = {4096, 512, 64};
  std::vector<void*> free_list[NCLS];
  std::vector<void*> chunks;
  int cls_of(size_t n) const {
    for (int i = 0; i < NCLS; i++)
      if (n <= cls_bytes[i]) return i;
    return -1;
  }
  void* get(size_t n) {
    int c = cls_of(n ? n : 1);
    if (c < 0) return nullptr;
    if (free_list[c].empty()) {
      uint8_t* chunk = (uint8_t*)swgpu::host_alloc(cls_bytes[c] * chunk_blocks[c]);
      if (!chunk) return nullptr;
      chunks.push_back(chunk);
      for (size_t i = 0; i < chunk_blocks[c]; i++) free_list[c].push_back(chunk + i * cls_bytes[c]);
    }
    void* p = free_list[c].back();
    free_list[c].pop_back();
    return p;
  }
  void put(void* p, size_t n) {
    int c = cls_of(n ? n : 1);
    if (c >= 0 && p) free_list[c].push_back(p);
  }
  void destroy() {
    for (void* c : chunks) swgpu::host_free(c);
    chunks.clear();
  }
};

// ============================================================================ device staging pool
// Large host-memory sends/receives are staged through device buffers.  cudaMalloc/cudaFree
// per message would serialise the device (cudaFree synchronises), so freed blocks are kept.
struct StagingPool {
  std::multimap<size_t, void*> free_blocks;
  size_t cached = 0;
  static constexpr size_t MAX_CACHED = 6ull << 30;
  void* get(size_t n, size_t* got) {
    const size_t need = (n + 0xFFFFF) & ~(size_t)0xFFFFF;  // blocks come in 1 MiB granules
    auto it = free_blocks.lower_bound(need);
    if (it != free_blocks.end() && it->first <= 2 * need) {
      void* p = it->second;
      *got = it->first;
      cached -= it->first;
      free_blocks.erase(it);
      return p;
    }
    size_t sz = need;
    void* p = swgpu::dev_alloc_raw(sz);
    if (!p && !free_blocks.empty()) {
      destroy();
      p = swgpu::dev_alloc_raw(sz);
    }
    *got = sz;
    return p;
  }
  void put(void* p, size_t sz) {
    if (!p) return;
    if (cached + sz > MAX_CACHED) {
      swgpu::dev_free(p);
      return;
    }
    free_blocks.emplace(sz, p);
    cached += sz;
  }
  void destroy() {
    for (auto& kv : free_blocks) swgpu::dev_free(kv.second);
    free_blocks.clear();
    cached = 0;
  }
};

// Device landing blocks of reducing receives: the matcher copies an eager payload (at most SW_EAGER_MAX bytes) into
// the receive's block, a reduce launch then adds it into the caller's buffer.  Fixed blocks carved from larger
// allocations, so that thousands of receives in flight cost one slot each rather than a staging granule.
struct LandingPool {
  static constexpr size_t BLOCK = SW_SLOT_BYTES, PER_CHUNK = 256;
  std::vector<void*> free_list, chunks;
  void* get() {
    if (free_list.empty()) {
      uint8_t* chunk = (uint8_t*)swgpu::dev_alloc_raw(BLOCK * PER_CHUNK);
      if (!chunk) return nullptr;
      chunks.push_back(chunk);
      for (size_t i = 0; i < PER_CHUNK; i++) free_list.push_back(chunk + i * BLOCK);
    }
    void* p = free_list.back();
    free_list.pop_back();
    return p;
  }
  void put(void* p) {
    if (p) free_list.push_back(p);
  }
  void destroy() {
    for (void* c : chunks) swgpu::dev_free(c);
    chunks.clear();
    free_list.clear();
  }
};

// ============================================================================ pageable host buffers
// cudaMemcpyAsync from / to pageable memory is a synchronous, single-threaded staging loop inside the driver
// (slow, and it blocks the progress thread).  Large pageable buffers are moved by a few
// helper threads between the caller's memory and page-locked staging instead (chunked memcpy), and the copy
// engine only ever sees page-locked memory.  The payload still travels host -> GPU -> (NVLink) -> GPU -> host.
struct CopyPool {
  struct Task {
    uint8_t* dst;
    const uint8_t* src;
    size_t n;
    std::atomic<int>* pending;
  };
  static constexpr size_t CHUNK = 256 << 10;
  std::mutex mu;
  std::condition_variable cv;
  std::deque<Task> q;
  std::vector<std::thread> threads;
  bool stop = false;
  void start(int n, int device) {
    for (int i = 0; i < n; i++)
      threads.emplace_back([this, device] {
        (void)device;
        for (;;) {
          Task t;
          {
            std::unique_lock<std::mutex> lk(mu);
            cv.wait(lk, [&] { return stop || !q.empty(); });
            if (q.empty()) return;
            t = q.front();
            q.pop_front();
          }
          memcpy(t.dst, t.src, t.n);
          t.pending->fetch_sub(1, std::memory_order_acq_rel);
        }
      });
  }
  // copies n bytes in CHUNK pieces; *pending reaches 0 when every piece is done
  void submit(void* dst, const void* src, size_t n, std::atomic<int>* pending) {
    const int pieces = (int)((n + CHUNK - 1) / CHUNK);
    pending->store(pieces, std::memory_order_release);
    {
      std::lock_guard<std::mutex> lk(mu);
      for (size_t off = 0; off < n; off += CHUNK) q.push_back(Task{(uint8_t*)dst + off, (const uint8_t*)src + off, std::min(CHUNK, n - off), pending});
    }
    cv.notify_all();
  }
  void shutdown() {
    {
      std::lock_guard<std::mutex> lk(mu);
      stop = true;
    }
    cv.notify_all();
    for (auto& t : threads) t.join();
    threads.clear();
  }
};

struct PinnedPool {   // page-locked staging for pageable buffers (cudaHostAlloc costs milliseconds: blocks are kept)
  std::multimap<size_t, void*> free_blocks;
  size_t cached = 0;
  static constexpr size_t MAX_CACHED = 1ull << 30;
  void* get(size_t n, size_t* got) {
    const size_t need = (n + 0xFFFFF) & ~(size_t)0xFFFFF;
    auto it = free_blocks.lower_bound(need);
    if (it != free_blocks.end() && it->first <= 2 * need) {
      void* p = it->second;
      *got = it->first;
      cached -= it->first;
      free_blocks.erase(it);
      return p;
    }
    *got = need;
    return swgpu::host_alloc(need);
  }
  void put(void* p, size_t sz) {
    if (!p) return;
    if (cached + sz > MAX_CACHED) {
      swgpu::host_free(p);
      return;
    }
    free_blocks.emplace(sz, p);
    cached += sz;
  }
  void destroy() {
    for (auto& kv : free_blocks) swgpu::host_free(kv.second);
    free_blocks.clear();
    cached = 0;
  }
};

// ============================================================================ engine objects
struct Worker;
struct Ctx;

// Intrusive node of the lock-free multi-producer submission queue (replaces the reference's
// 1-slot Channel<T> mailboxes, chan.hpp:84-120: any number of ops can be in flight).
struct SqNode {
  SqNode* next = nullptr;
  int kind = 0;
  Worker* w = nullptr;
  void* p = nullptr;
  bool heap = false;
};

// Operation records are allocated on the posting thread and freed on the progress thread; going
// through malloc that is a cross-thread free per operation.  Freed blocks go onto a lock-free
// return stack instead (push only: no ABA), and an allocating thread takes the WHOLE stack into a
// thread-local cache when its cache runs dry.
template <class T>
struct OpPool {
  struct Node {
    Node* next;
  };
  static inline std::atomic<Node*> returned{nullptr};
  static inline thread_local Node* cache = nullptr;
  static void* get() {
    Node* n = cache;
    if (!n) n = returned.exchange(nullptr, std::memory_order_acquire);
    if (n) {
      cache = n->next;
      return n;
    }
    return ::operator new(sizeof(T) < sizeof(Node) ? sizeof(Node) : sizeof(T));
  }
  static void put(void* p) {
    Node* n = static_cast<Node*>(p);
    Node* h = returned.load(std::memory_order_relaxed);
    do {
      n->next = h;
    } while (!returned.compare_exchange_weak(h, n, std::memory_order_release, std::memory_order_relaxed));
  }
};

struct SendOp {
  static void* operator new(size_t) { return OpPool<SendOp>::get(); }
  static void operator delete(void* p) { OpPool<SendOp>::put(p); }
  SqNode sqn;
  uint64_t op_id = 0;
  Worker* w = nullptr;
  struct Ep* ep = nullptr;
  const uint8_t* ptr = nullptr;
  size_t len = 0;
  uint64_t tag = 0;
  int mem = SW_MEM_AUTO;
  uint64_t sseq = 0;        // per-endpoint send sequence, for flush
  bool user_done = false;   // user-visible completion already delivered
  void* dev_staging = nullptr;
  size_t staging_size = 0;
  uint64_t rndv_seq = 0;
  // The put block that carries this send's slot still refers to the record until poll_puts retires it: a
  // FIN / close that ends the send earlier only notes the outcome here and poll_puts finishes the record.
  void* pin_stage = nullptr;           // pageable host source: page-locked copy made by the helper threads
  size_t pin_stage_size = 0;
  std::atomic<int> pin_pending{0};     // chunks of that copy still running
  bool stage_d2d = false;   // device source that CUDA IPC cannot export (cuMemCreate / expandable segments):
                            // copied into an exportable staging buffer first
  bool in_put = false;
  bool ended_early = false;
  int32_t early_status = 0;
};

constexpr int MEM_PINNED = 3;  // internal: host memory the device can address directly (cudaHostAlloc)

struct RecvOp {
  static void* operator new(size_t) { return OpPool<RecvOp>::get(); }
  static void operator delete(void* p) { OpPool<RecvOp>::put(p); }
  SqNode sqn;
  uint64_t op_id = 0;
  Worker* w = nullptr;
  uint8_t* ptr = nullptr;
  size_t cap = 0;
  uint64_t tag = 0, mask = 0;
  int mem = SW_MEM_AUTO;
  void* pinned_bounce = nullptr;  // small host receives land here (device-mapped pinned memory)
  void* dev_staging = nullptr;    // large host receives land here, then D2H
  size_t staging_size = 0;
  bool rndv_capable = false;      // resident path: counted in Worker::rndv_recvs while posted
  void* pin_stage = nullptr;      // pageable host destination: page-locked landing zone of the device -> host copy
  size_t pin_stage_size = 0;
  std::atomic<int> pin_pending{0};
  int dtype = 0;                  // reducing receive (sw_post_recv_reduce): SW_DT_* of the caller's buffer; 0: plain receive
  void* landing = nullptr;        // reducing receive: device block the matcher copies an eager payload into
};

struct FlushOp {
  SqNode sqn;
  uint64_t op_id = 0;
  struct Ep* ep = nullptr;               // nullptr: every endpoint of the worker
  std::map<struct Ep*, uint64_t> marks;  // per-endpoint: sends with sseq < mark must be complete
};

struct Mapping;

struct BulkJob {
  double t_enq = 0;
  bool host_side = false;  // source or destination is pinned host memory
  bool src_host = false;   // the source is pinned host memory (read over PCIe by the copying kernel)
  Worker* w = nullptr;
  struct Ep* ep = nullptr;
  uint64_t recv_op = 0;
  uint64_t dst = 0, cap = 0, tag = 0, len = 0;
  SwRts rts;
  uint64_t src = 0;
  Mapping* mapping = nullptr;
  bool failed = false;
  int32_t fail_status = 0;
  int dtype = 0;            // reducing receive: dst += src with elements of this SW_DT_* type (0: copy)
  bool src_ready = false;   // `src` is a local device address already (an eager payload in a landing block)
};

constexpr uint32_t EP_MAGIC = 0x53574550u, WORKER_MAGIC = 0x5357574Bu, DEAD_MAGIC = 0x44454144u;

// Worker / endpoint handles are pointers into TYPE-STABLE storage tagged with a 16-bit generation
// (bits 48-63): the storage of a destroyed object is never returned to malloc, it goes onto a free
// list and is reused for the next object of the same type with the generation bumped.  A stale
// handle therefore always dereferences valid memory and fails the magic / generation check,
// while a process that keeps creating and closing Clients / Servers does not grow (each record is
// 2-3 KB: two std::deque members alone are 1.2 KB).  Both types start with {magic, gen}.
constexpr uint64_t HANDLE_PTR_MASK = 0x0000FFFFFFFFFFFFull;
template <class T>
struct Slab {
  static inline std::mutex mu;
  static inline std::vector<void*> free_list;
  static T* make() {
    void* mem = nullptr;
    uint32_t gen = 1;
    {
      std::lock_guard<std::mutex> lk(mu);
      if (!free_list.empty()) {
        mem = free_list.back();
        free_list.pop_back();
        gen = (static_cast<uint32_t*>(mem)[1] + 1) & 0xFFFFu;
        if (!gen) gen = 1;
      }
    }
    if (!mem) mem = ::operator new(sizeof(T));
    T* t = new (mem) T();
    t->gen = gen;
    t->id = (uint64_t)(uintptr_t)t | ((uint64_t)gen << 48);
    return t;
  }
  static void recycle(T* t) {
    const uint32_t gen = t->gen;
    t->~T();
    static_cast<uint32_t*>(static_cast<void*>(t))[0] = DEAD_MAGIC;
    static_cast<uint32_t*>(static_cast<void*>(t))[1] = gen;
    std::lock_guard<std::mutex> lk(mu);
    free_list.push_back(t);
  }
};

struct Ep {
  uint32_t magic = EP_MAGIC;
  uint32_t gen = 0;
  uint64_t id = 0;
  Worker* owner = nullptr;
  uint32_t index = 0;  // index of the inbound ring in the owner's match state
  bool is_client_side = false;
  // peer identity
  uint32_t peer_pid = 0;
  int32_t peer_device = -1;
  uint64_t peer_ctx_uuid = 0;
  uint64_t peer_worker_id = 0;
  bool in_process = false;
  // our inbound ring (owned) and the peer's inbound ring (mapped)
  uint8_t* ring = nullptr;
  uint32_t ring_slots = 0;
  uint8_t* peer_ring = nullptr;
  bool ring_same_gpu = false;         // the peer's ring is in the memory of this context's GPU (pointer attributes of the mapping)
  void* peer_ring_mapping = nullptr;  // base returned by ipc_open (nullptr when in-process)
  uint32_t peer_ring_slots = 0;
  // control block
  ShmCtl* shm = nullptr;
  uint8_t* shm_dev = nullptr;   // device-visible alias of the control block (nullptr: not page-locked)
  size_t shm_size = 0;
  ShmDir* out = nullptr;  // we are the sender side of this direction
  ShmDir* in = nullptr;   // we are the receiver side of this direction
  std::deque<CtlMsg> ctl_backlog;
  // send side
  std::deque<SendOp*> sendq;
  uint64_t out_sent = 0;       // slots handed to put kernels
  uint64_t out_published = 0;  // slots published in out->produced
  uint64_t next_sseq = 1;
  std::set<uint64_t> out_seqs;  // outstanding sends (sseq)
  uint64_t rndv_next = 1;
  std::map<uint64_t, SendOp*> rndv_wait;  // rendezvous sends waiting for FIN
  std::set<uint64_t> cancel_wait;          // CANCEL_RTS sent, waiting for ack / FIN
  uint32_t puts_inflight = 0;
  // receive side
  std::set<uint64_t> canceled_rts;  // sender cancelled these rendezvous ids
  // resident path: withdrawals (CANCEL_RTS) wait here until the control kernel has seen the endpoint's dead bit
  // and every device-side pull issued before that is complete; then they move to canceled_rts and are acked
  std::vector<uint64_t> cancel_quiesce;
  uint64_t cancel_epoch = 0;        // host_epoch value the control kernel has to echo
  uint64_t cancel_pull_mark = 0;    // device pull jobs that must have completed
  bool retired = false;             // resources released, ring index reusable (the record stays listed)
  uint32_t ring_gen = 0;            // generation of `index` (device side: SwMatchState::ring_gen)
  // lifecycle
  bool peer_closed = false;
  bool close_ack_owed = false;
  bool close_sent = false;
  bool close_acked = false;
  // metadata (reference ServerEndpoint, main.hpp:292-304)
  sw_ep_info info;
};

struct Worker {
  uint32_t magic = WORKER_MAGIC;
  uint32_t gen = 0;
  uint64_t id = 0;
  int kind = 0;
  Ctx* ctx = nullptr;
  std::atomic<int> status{SW_ST_VOID};
  // device-resident queues
  SwMatchState* mstate = nullptr;
  std::vector<Ep*> eps;  // index == Ep::index
  // receives
  std::deque<RecvOp*> new_posts;
  std::unordered_map<uint64_t, RecvOp*> recvs;  // handed to the device, not completed
  // flush
  std::vector<FlushOp*> flushes;
  // listeners
  int tcp_fd = -1, unix_fd = -1;
  struct PendingHello {   // accepted bootstrap connection whose hello has not arrived yet
    int fd;
    bool tcp;
    double deadline;
  };
  std::vector<PendingHello> pending_hello;
  std::string unix_name;
  AddrBlob blob;
  std::atomic<bool> blob_ready{false};
  // close
  uint64_t close_op = 0;
  int close_phase = 0;
  double close_deadline = 0;
  bool registered = false;
  std::atomic<bool> register_queued{false};  // an SQ_REGISTER for this worker was pushed
  std::atomic<bool> retired{false};          // the progress thread has dropped its last reference
  std::thread connector;
  uint32_t bulk_inflight = 0;
  // ---- resident path (sw_progress_kernel): host-visible rings and control words of this worker
  SwProgCtl* pctl = nullptr;
  SwPostEnt* post_ring = nullptr;
  SwCqEnt* cq_ring = nullptr;
  SwCqEnt* cqr_ring = nullptr;
  SwHrEnt* hr_ring = nullptr;
  SwSendLL* send_ring = nullptr;    // puts executed by the resident kernel (small batches, no launch), stamped units
  uint64_t sends_written = 0;
  swgpu::stream_t s_ctl = nullptr;
  uint64_t prog_seq = 0;          // launches so far
  bool prog_running = false;
  bool cfg_dirty = false;         // ring set changed: the running kernel must leave and be relaunched
  uint64_t posts_written = 0, cq_head = 0, cqr_head = 0, hr_head = 0;
  uint64_t host_epoch = 0;
  double last_activity = 0, prog_launched_at = 0, last_send = -1;
  uint32_t prog_spins = 0;
  // a launch that ended with a ring blocked on the unexpected heap is repeated only when something changed
  bool prog_stalled = false;
  uint64_t stall_posts = 0, stall_seen = 0;
  uint32_t rndv_recvs = 0;        // posted receives that a rendezvous message could land in
  uint64_t arrivals_seen = 0;
  std::vector<uint32_t> free_ring_idx;   // ring indices of retired endpoints
  uint32_t ring_gen_ctr[SW_MAX_EPS] = {};
  std::vector<Ep*> tombs;                // retired endpoint records whose ring index has been taken over
};

enum : int { SQ_SEND = 1, SQ_RECV = 2, SQ_FLUSH = 3, SQ_CLOSE = 4, SQ_NEW_EP = 5, SQ_REGISTER = 6 };

struct PutItem {
  Ep* ep;
  SendOp* op;
  bool rndv;
};
constexpr uint32_t STAGE_SEGS = 1024;
struct PutBlock {
  SwSeg* segs = nullptr;   // pinned-host -> device staging uploads of this batch (TMA kernel)
  uint32_t nsegs = 0;
  SwPutDesc* descs = nullptr;
  SwRts* rts = nullptr;
  uint8_t* stage = nullptr;
  swgpu::event_t ev = nullptr, ev_start = nullptr;   // timing pair (option profile >= 2)
  swgpu::event_t ev_fast = nullptr;                  // completion only (timing disabled)
  uint64_t* done = nullptr;                          // pinned host: completion flag of small launches
  uint64_t done_seq = 0;
  uint32_t spins = 0;
  bool flag_mode = false, timed = false;
  bool busy = false;
  // executed by the sending worker's resident control kernel instead of a launch: done when the kernel's
  // send_done counter has passed res_end
  Worker* res_worker = nullptr;
  uint64_t res_end = 0;
  // every block launches on a stream of its own: put kernels are latency-bound (a handful of stores behind a
  // launch), so consecutive batches overlap instead of queueing behind each other; blocks still retire in order
  swgpu::stream_t s = nullptr;
  std::vector<PutItem> items;
  // host -> staging uploads of this batch, submitted as one copy-engine batch in front of the put
  std::vector<void*> up_dst;
  std::vector<const void*> up_src;
  std::vector<size_t> up_len;
};
struct BulkBlock {
  SwSeg* segs = nullptr;
  swgpu::event_t ev = nullptr, ev_start = nullptr;   // timing pair (option profile >= 1)
  swgpu::event_t ev_fast = nullptr;                  // completion only (timing disabled)
  bool timed = false;
  bool busy = false;
  std::vector<BulkJob> jobs;
  std::vector<SwSeg> tma, simt;  // scratch, capacity retained across launches
  std::vector<SwSeg> rtma[7], rsimt[7];   // the same for reducing receives, indexed by SW_DT_*
  std::vector<void*> ce_dst;     // copies of this block made by the copy engine (device -> pinned host)
  std::vector<const void*> ce_src;
  std::vector<size_t> ce_len;
  uint64_t bytes = 0;
};
struct PostCopy {  // device staging -> host user buffer after delivery
  swgpu::event_t ev;
  RecvOp* op;
  uint64_t tag, len;
  int32_t status;
  int phase = 0;   // 0: device -> page-locked copy in flight; 1: helper threads copy page-locked -> caller's memory
};
struct Mapping {
  void* base;
  uint32_t refs;
  double last_use;
  uint64_t uuid, buf_id, remote_base;   // key / value of the device-resident table entry (buf_id 0: none)
};
struct MapKey {   // (exporting pid, cudaIpcMemHandle_t bytes)
  uint32_t pid;
  uint8_t handle[64];
  bool operator==(const MapKey& o) const { return pid == o.pid && memcmp(handle, o.handle, 64) == 0; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    uint64_t h = 0xcbf29ce484222325ull ^ k.pid;
    const uint64_t* w = reinterpret_cast<const uint64_t*>(k.handle);
    for (int i = 0; i < 8; i++) h = (h ^ w[i]) * 0x100000001b3ull;
    return (size_t)h;
  }
};

constexpr uint32_t PUT_BATCH = 512;
constexpr int N_PUT_BLOCKS = 4;
constexpr int N_BULK_BLOCKS = 3;
constexpr uint32_t MAX_SEGS = 8192;
constexpr size_t HOST_BOUNCE_MAX = 65536;
constexpr size_t MAX_MAPPINGS = 4096;
constexpr uint64_t STAGE_BATCH_BYTES = 4ull << 20;
constexpr uint64_t STAGE_SEG_BYTES = 32768;

struct Ctx {
  int device = 0;
  uint64_t uuid = 0;
  // handle tables
  std::mutex mu;
  std::unordered_map<uint64_t, Worker*> workers;
  std::unordered_map<uint64_t, Ep*> eps;
  // The words that posting threads, the progress thread and a polling consumer hammer on live on
  // cache lines of their own (no false sharing between the submission and the completion side).
  alignas(64) std::atomic<uint64_t> next_id{1};  // posting threads
  // submission queue: written by posting threads, polled by the progress thread
  alignas(64) std::atomic<SqNode*> sq_head{nullptr};
  std::atomic<int> sleeping{0};  // the progress thread naps on this word (futex); a submission wakes it
  // completion queue: written by the progress thread, polled by the consumer
  alignas(64) std::atomic<uint32_t> cq_count{0};  // == cq.size(), readable without the lock
  std::atomic<int> efd_signaled{0};               // the eventfd counter is non-zero
  alignas(64) std::atomic<int> consumer_polling{0};  // option "consumer_polling": skip the eventfd wake-up
  std::atomic<int> cq_waiters{0};                    // threads blocked in sw_wait
  alignas(64) std::mutex cq_mu;
  std::condition_variable cq_cv;
  std::deque<sw_completion> cq;
  std::vector<sw_completion> cq_local;  // progress-thread staging
  int efd = -1;
  // progress thread
  std::thread thr;
  std::atomic<bool> stop{false};
  std::vector<Worker*> active;  // progress-thread private
  bool need_prune = false;      // progress-thread private: a worker reached close phase 4
  // device resources
  swgpu::stream_t s_put = nullptr, s_bulk = nullptr;
  PutBlock put_blocks[N_PUT_BLOCKS];
  uint32_t put_head = 0, put_tail = 0;  // ring of in-flight put blocks
  BulkBlock bulk_blocks[N_BULK_BLOCKS];
  uint32_t bulk_head = 0, bulk_tail = 0;
  std::deque<BulkJob> pending_bulk;
  std::deque<PostCopy> post_copies;
  HostPool host_pool;
  StagingPool staging;
  LandingPool landing;
  PinnedPool pinned_pool;
  CopyPool copy_pool;
  std::atomic<int64_t> opt_copy_threads{4};   // helper threads for pageable host buffers (0: cudaMemcpyAsync on pageable memory)
  size_t pin_inflight = 0;                    // bytes of page-locked staging in use by sends
  std::unordered_map<MapKey, Mapping, MapKeyHash> mappings;  // node addresses are stable
  struct HandleEnt {
    uint64_t base;
    uint8_t handle[64];
    bool exportable = true;   // false: cudaIpcGetMemHandle refuses this allocation (virtual-memory-management API)
  };
  std::unordered_map<uint64_t, HandleEnt> handle_cache;  // CUDA buffer id -> exported IPC handle
  // options
  std::atomic<int64_t> opt_eager_max{SW_EAGER_MAX};
  std::atomic<int64_t> opt_ring_slots{SW_RING_SLOTS_DEFAULT};
  std::atomic<int64_t> opt_bulk_mode{0}, opt_bulk_stages{8}, opt_bulk_stage_bytes{24576}, opt_bulk_ctas{1};
  std::atomic<int64_t> opt_coalesce_us{40}, opt_coalesce_bytes{32 << 20};
  // 1: launches of <= 96 messages carry the messages as kernel parameters and every CTA copies an equal
  // byte range (sw_bulk_tma_jobs_kernel); 0: segment list in pinned host memory (sw_bulk_tma_kernel)
  std::atomic<int64_t> opt_bulk_balance{1};
  // small put launches announce completion through a flag in pinned host memory
  // (seen sooner than through a timing event; `sw_probe floor` measures both)
  std::atomic<int64_t> opt_done_flags{1};
  uint64_t flag_seq = 0;
  std::atomic<int64_t> opt_heap_small{4096}, opt_heap_big{512};
  std::atomic<int64_t> opt_profile{0};
  // 1: same-process pinned host sources are read in place by the receiver's kernel (one host->host
  // kernel, ~37 GB/s); 0: stage them through device memory so upload and download overlap (PCIe duplex)
  std::atomic<int64_t> opt_pinned_send_direct{1};
  std::atomic<int64_t> opt_pull_keep_us{60};   // the pull kernel stays through gaps between needs up to this long (0: asked to leave at once)
  // 1: upload pinned host sources with the TMA bulk kernel; 0 (default): copy engine (cudaMemcpyAsync).
  // The copy engine leaves the SMs and more of the PCIe duplex budget to the concurrent download kernel.
  std::atomic<int64_t> opt_stage_upload_kernel{0};
  std::atomic<int64_t> opt_stage_batch_bytes{(int64_t)STAGE_BATCH_BYTES};   // staged sends are announced in batches of this size
  std::atomic<int64_t> opt_max_mappings{(int64_t)MAX_MAPPINGS};   // peer allocations kept mapped (LRU quarter dropped when full)
  std::atomic<int64_t> opt_hostdst_ce{0};    // device -> pinned-host copies by the copy engine (batched) instead of a kernel
  std::atomic<int64_t> opt_hostdst_tma{0};   // device -> pinned-host copies by the TMA kernel instead of the SIMT kernel
  // ---- resident path: receives are driven by resident control kernels (sw_progress_kernel) and rendezvous
  // copies by the resident pull CTAs (sw_pull_kernel)
  std::atomic<int64_t> opt_linger_us{150}, opt_max_life_us{2000}, opt_armed_ms{30}, opt_pull_ctas{0};
  // batches of at most this many sends of ONE worker whose control kernel is resident are executed by that
  // kernel (descriptor ring in pinned memory) instead of a put launch; 0: always launch
  std::atomic<int64_t> opt_resident_puts{24};
  std::atomic<int64_t> opt_yield_us{30};   // progress thread yields between looks after this much silence with only resident kernels out (0: never)
  SwPullQueue* pq = nullptr;
  SwMapEnt* map_tbl = nullptr;
  SwPullCtl* pull_ctl = nullptr;
  swgpu::stream_t s_pull = nullptr, s_map = nullptr;
  swgpu::event_t pull_ev = nullptr;
  uint64_t pull_seq = 0;
  bool pull_running = false, pull_stop_sent = false;
  double pull_launched_at = 0, pull_last_need = 0;
  uint64_t pull_bytes_seen = 0, pull_busy_seen = 0, pull_batches_seen = 0, pull_jobs_seen = 0;
  std::atomic<int> stats_flush{0};
  bool evict_pending = false;   // the mapping cache is waiting for the device-side users to drain
  // stats
  std::mutex st_mu;
  sw_stats stats;
  // optional event trace of the progress thread (STARWAY_TRACE=<file>): time-stamped pipeline events
  struct TraceRec {
    double t;
    const char* what;
    uint64_t a, b;
  };
  std::vector<TraceRec> trace;
  std::string trace_path;
  bool tracing = false;
};

inline void trace(Ctx* c, const char* what, uint64_t a = 0, uint64_t b = 0) {
  if (c->tracing && c->trace.size() < (1u << 22)) c->trace.push_back(Ctx::TraceRec{now_s(), what, a, b});
}

std::mutex g_ctx_mu;
std::vector<Ctx*> g_ctxs;

// ============================================================================ completions
// Completions produced by the progress thread are staged locally and published once per loop
// iteration: one lock, one condvar signal, one eventfd write per batch.
thread_local bool tls_is_progress = false;

void publish_completions(Ctx* c, const sw_completion* comps, size_t n) {
  if (!n) return;
  {
    std::lock_guard<std::mutex> lk(c->cq_mu);
    const bool was_empty = c->cq.empty();
    for (size_t i = 0; i < n; i++) c->cq.push_back(comps[i]);
    c->cq_count.store((uint32_t)c->cq.size(), std::memory_order_seq_cst);
    // A consumer that announced it is busy-polling (option "consumer_polling") needs no wake-up: it
    // clears the flag and polls once more before it goes back to sleeping on the eventfd.  The
    // eventfd is written and cleared (sw_poll) under cq_mu only: "counter non-zero" <=> efd_signaled.
    if (was_empty && c->efd >= 0 && !c->consumer_polling.load(std::memory_order_seq_cst)) {
      c->efd_signaled.store(1, std::memory_order_release);
      uint64_t one = 1;
      ssize_t r = write(c->efd, &one, sizeof(one));
      (void)r;
    }
  }
  if (c->cq_waiters.load(std::memory_order_seq_cst)) c->cq_cv.notify_one();
  std::lock_guard<std::mutex> lk(c->st_mu);
  c->stats.completions += n;
}

void push_completion(Ctx* c, const sw_completion& comp) {
  if (tls_is_progress) {
    c->cq_local.push_back(comp);
    return;
  }
  publish_completions(c, &comp, 1);
}

void flush_completions(Ctx* c) {
  if (c->cq_local.empty()) return;
  trace(c, "publish", c->cq_local.size());
  publish_completions(c, c->cq_local.data(), c->cq_local.size());
  c->cq_local.clear();
}
void complete(Ctx* c, Worker* w, uint64_t op_id, uint32_t kind, int32_t status, uint64_t tag = 0, uint64_t len = 0,
              uint64_t ep = 0) {
  sw_completion comp;
  memset(&comp, 0, sizeof(comp));
  comp.op_id = op_id;
  comp.status = status;
  comp.kind = kind;
  comp.sender_tag = tag;
  comp.length = len;
  comp.worker = w ? w->id : 0;
  comp.ep = ep;
  push_completion(c, comp);
}

// ============================================================================ control messages
bool ctl_try_send(Ep* ep, const CtlMsg& m) {
  ShmDir* d = ep->out;
  uint64_t head = d->ctl_head.load(std::memory_order_relaxed);
  uint64_t tail = d->ctl_tail.load(std::memory_order_acquire);
  if (head - tail >= CTL_RING) return false;
  d->ctl[head % CTL_RING] = m;
  d->ctl_head.store(head + 1, std::memory_order_release);
  return true;
}
void ctl_send(Ep* ep, uint32_t type, int32_t status, uint64_t a, uint64_t b = 0) {
  if (!ep->shm) return;
  CtlMsg m;
  m.type = type;
  m.status = status;
  m.a = a;
  m.b = b;
  m.pad = 0;
  if (!ep->ctl_backlog.empty() || !ctl_try_send(ep, m)) ep->ctl_backlog.push_back(m);
}
void ctl_flush_backlog(Ep* ep) {
  while (!ep->ctl_backlog.empty() && ctl_try_send(ep, ep->ctl_backlog.front())) ep->ctl_backlog.pop_front();
}

// ============================================================================ send-op bookkeeping
void send_finished(Ctx* c, SendOp* op, int32_t status) {
  if (!op->user_done) {
    complete(c, op->w, op->op_id, SW_OP_SEND, status);
    op->user_done = true;
  }
  if (op->dev_staging) c->staging.put(op->dev_staging, op->staging_size);
  if (op->pin_stage) {
    while (op->pin_pending.load(std::memory_order_acquire) > 0) sched_yield();   // (cancelled while the helpers still copy)
    c->pinned_pool.put(op->pin_stage, op->pin_stage_size);
    c->pin_inflight -= std::min(c->pin_inflight, op->pin_stage_size);
  }
  op->ep->out_seqs.erase(op->sseq);
  delete op;
}

void recv_release(Ctx* c, RecvOp* r) {
  if (r->rndv_capable && r->w && r->w->rndv_recvs) r->w->rndv_recvs--;
  if (r->pin_stage) c->pinned_pool.put(r->pin_stage, r->pin_stage_size);
  if (r->pinned_bounce) c->host_pool.put(r->pinned_bounce, r->cap);
  if (r->dev_staging) c->staging.put(r->dev_staging, r->staging_size);
  c->landing.put(r->landing);
  delete r;
}

// finish a receive whose payload (if any) already sits in its landing buffer
void recv_finish(Ctx* c, Worker* w, uint64_t op_id, int32_t status, uint64_t tag, uint64_t len) {
  auto it = w->recvs.find(op_id);
  if (it == w->recvs.end()) return;
  RecvOp* r = it->second;
  if (status == SW_OK && len && r->pinned_bounce) {
    memcpy(r->ptr, r->pinned_bounce, (size_t)std::min<uint64_t>(len, r->cap));
    std::lock_guard<std::mutex> lk(c->st_mu);
    c->stats.d2h_bytes += len;
  }
  if (status == SW_OK && len && r->dev_staging) {
    // large host receive: bring the bytes down, complete when the copy has finished
    w->recvs.erase(it);
    swgpu::event_t ev = swgpu::event_create(0);
    if (!c->copy_pool.threads.empty() && len >= (256u << 10)) {
      // pageable destination: DMA into page-locked staging, the helper threads finish the job (poll_bulk)
      r->pin_stage = c->pinned_pool.get((size_t)len, &r->pin_stage_size);
    }
    swgpu::memcpy_d2h(r->pin_stage ? r->pin_stage : (void*)r->ptr, r->dev_staging, (size_t)len, c->s_bulk);
    swgpu::event_record(ev, c->s_bulk);
    c->post_copies.push_back(PostCopy{ev, r, tag, len, status});
    std::lock_guard<std::mutex> lk(c->st_mu);
    c->stats.d2h_bytes += len;
    return;
  }
  w->recvs.erase(it);
  complete(c, w, op_id, SW_OP_RECV, status, tag, len);
  recv_release(c, r);
}

// ============================================================================ worker resources
bool worker_alloc_device(Ctx* c, Worker* w) {
  w->mstate = swgpu::match_state_create((uint32_t)c->opt_heap_small.load(), (uint32_t)c->opt_heap_big.load());
  if (!w->mstate) {
    set_error(std::string("match_state_create: ") + swgpu::last_error());
    return false;
  }
  w->pctl = (SwProgCtl*)swgpu::host_alloc(sizeof(SwProgCtl));
  w->post_ring = (SwPostEnt*)swgpu::host_alloc(sizeof(SwPostEnt) * SW_POST_RING);
  w->cq_ring = (SwCqEnt*)swgpu::host_alloc(sizeof(SwCqEnt) * SW_CQ_RING);
  w->cqr_ring = (SwCqEnt*)swgpu::host_alloc(sizeof(SwCqEnt) * SW_CQ_RING);
  w->hr_ring = (SwHrEnt*)swgpu::host_alloc(sizeof(SwHrEnt) * SW_HR_RING);
  w->send_ring = (SwSendLL*)swgpu::host_alloc(sizeof(SwSendLL) * SW_SEND_RING);
  if (w->send_ring) memset(w->send_ring, 0, sizeof(SwSendLL) * SW_SEND_RING);   // stamp 0: never an entry
  w->s_ctl = swgpu::stream_create();
  if (!w->pctl || !w->post_ring || !w->cq_ring || !w->cqr_ring || !w->hr_ring || !w->send_ring || !w->s_ctl) {
    set_error(std::string("worker resident-path alloc: ") + swgpu::last_error());
    return false;
  }
  w->last_activity = now_s();
  return true;
}

// per-endpoint words the control kernel publishes to: the sender-visible credit word and the FIN words of the
// inbound direction, through the page-locked alias of the control block
bool ep_publish_words(Worker* w, Ep* ep) {
  if (!ep->shm_dev) return false;   // sw_ctx_create probed page-locking: this is an error
  const size_t off = (uint8_t*)ep->in - (uint8_t*)ep->shm;
  return swgpu::match_state_set_ep_words(w->mstate, ep->index, ep->shm_dev + off + offsetof(ShmDir, consumed),
                                         ep->shm_dev + off + offsetof(ShmDir, gfin)) == 0;
}

void fill_blob(Ctx* c, Worker* w) {
  memset(&w->blob, 0, sizeof(w->blob));
  w->blob.magic = ADDR_MAGIC;
  w->blob.version = SW_ABI_VERSION;
  w->blob.pid = (uint32_t)getpid();
  w->blob.device = c->device;
  w->blob.ctx_uuid = c->uuid;
  w->blob.worker_id = w->id;
  snprintf(w->blob.unix_name, sizeof(w->blob.unix_name), "%s", w->unix_name.c_str());
  gethostname(w->blob.host, sizeof(w->blob.host) - 1);
  w->blob_ready.store(true, std::memory_order_release);
}

Ep* ep_new(Ctx* c, Worker* w) {
  Ep* ep = Slab<Ep>::make();
  ep->owner = w;
  memset(&ep->info, 0, sizeof(ep->info));
  return ep;
}

bool ep_alloc_ring(Ctx* c, Ep* ep) {
  uint32_t slots = (uint32_t)c->opt_ring_slots.load();
  uint32_t p2 = 1;
  while (p2 < slots) p2 <<= 1;
  ep->ring_slots = p2;
  ep->ring = (uint8_t*)swgpu::dev_alloc((size_t)p2 * SW_SLOT_BYTES);
  if (!ep->ring) {
    set_error(std::string("ring alloc: ") + swgpu::last_error());
    return false;
  }
  return true;
}

// Control blocks are mapped ONCE per process and name (both ends of an in-process connection share the
// mapping) and page-locked with the CUDA driver, so that kernels can store credits and FIN words into them.
struct ShmMapping {
  ShmCtl* host = nullptr;
  uint8_t* dev = nullptr;   // device-visible alias (nullptr: registration failed, the host forwards instead)
  size_t size = 0;
  int refs = 0;
};
std::mutex g_shm_mu;
std::map<std::string, ShmMapping> g_shm;

constexpr size_t shm_bytes() { return (sizeof(ShmCtl) + 4095) & ~(size_t)4095; }

ShmCtl* shm_adopt(const std::string& name, void* p, size_t sz, uint8_t** dev_out) {
  ShmMapping m;
  m.host = (ShmCtl*)p;
  m.size = sz;
  m.refs = 1;
  m.dev = (uint8_t*)swgpu::host_register(p, sz);
  if (!m.dev) fprintf(stderr, "starway_b200: control block not page-locked (%s)\n", swgpu::last_error());
  g_shm[name] = m;
  *dev_out = m.dev;
  return m.host;
}

ShmCtl* shm_create(std::string& name_out, size_t& size_out, uint8_t** dev_out) {
  char name[64];
  snprintf(name, sizeof(name), "/swb200-%d-%llx", (int)getpid(), (unsigned long long)rand64());
  int fd = shm_open(name, O_CREAT | O_EXCL | O_RDWR, 0600);
  if (fd < 0) return nullptr;
  size_t sz = shm_bytes();
  if (ftruncate(fd, (off_t)sz) != 0) {
    close(fd);
    shm_unlink(name);
    return nullptr;
  }
  void* p = mmap(nullptr, sz, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (p == MAP_FAILED) {
    shm_unlink(name);
    return nullptr;
  }
  memset(p, 0, sz);
  ShmCtl* s = (ShmCtl*)p;
  s->magic = SHM_MAGIC;
  s->version = SW_ABI_VERSION;
  name_out = name;
  size_out = sz;
  std::lock_guard<std::mutex> lk(g_shm_mu);
  return shm_adopt(name, p, sz, dev_out);
}
ShmCtl* shm_attach(const char* name, size_t& size_out, uint8_t** dev_out) {
  std::lock_guard<std::mutex> lk(g_shm_mu);
  auto it = g_shm.find(name);
  if (it != g_shm.end()) {   // the creator lives in this process
    it->second.refs++;
    size_out = it->second.size;
    *dev_out = it->second.dev;
    return it->second.host;
  }
  int fd = shm_open(name, O_RDWR, 0600);
  if (fd < 0) return nullptr;
  size_t sz = shm_bytes();
  void* p = mmap(nullptr, sz, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (p == MAP_FAILED) return nullptr;
  ShmCtl* s = (ShmCtl*)p;
  if (s->magic != SHM_MAGIC) {
    munmap(p, sz);
    return nullptr;
  }
  size_out = sz;
  return shm_adopt(name, p, sz, dev_out);
}
void shm_release(ShmCtl* s) {
  if (!s) return;
  std::lock_guard<std::mutex> lk(g_shm_mu);
  for (auto it = g_shm.begin(); it != g_shm.end(); ++it) {
    if (it->second.host != s) continue;
    if (--it->second.refs == 0) {
      if (it->second.dev) swgpu::host_unregister(it->second.host);
      munmap(it->second.host, it->second.size);
      g_shm.erase(it);
    }
    return;
  }
}

void sq_push(Ctx* c, int kind, Worker* w, void* p, SqNode* n = nullptr) {
  if (!n) {
    n = new SqNode();
    n->heap = true;
  }
  n->kind = kind;
  n->w = w;
  n->p = p;
  SqNode* head = c->sq_head.load(std::memory_order_relaxed);
  do {
    n->next = head;
  } while (!c->sq_head.compare_exchange_weak(head, n, std::memory_order_release, std::memory_order_relaxed));
  // an idle progress thread naps between polls of the peers' doorbells: cut the nap short
  if (c->sleeping.load(std::memory_order_seq_cst) && c->sleeping.exchange(0, std::memory_order_seq_cst))
    syscall(SYS_futex, reinterpret_cast<int*>(&c->sleeping), FUTEX_WAKE_PRIVATE, 1, nullptr, nullptr, 0);
}

// ============================================================================ connection: server side
int make_unix_listener(std::string& name_out) {
  int fd = socket(AF_UNIX, SOCK_STREAM | SOCK_CLOEXEC, 0);
  if (fd < 0) return -1;
  char name[64];
  snprintf(name, sizeof(name), "starway-b200-%d-%llx", (int)getpid(), (unsigned long long)rand64());
  struct sockaddr_un sa;
  memset(&sa, 0, sizeof(sa));
  sa.sun_family = AF_UNIX;
  size_t n = strlen(name);
  memcpy(sa.sun_path + 1, name, n);  // abstract namespace
  if (bind(fd, (struct sockaddr*)&sa, (socklen_t)(offsetof(struct sockaddr_un, sun_path) + 1 + n)) != 0 ||
      listen(fd, 128) != 0) {
    close(fd);
    return -1;
  }
  fcntl(fd, F_SETFL, fcntl(fd, F_GETFL) | O_NONBLOCK);
  name_out = name;
  return fd;
}
int make_tcp_listener(const char* addr, uint16_t port) {
  int fd = socket(AF_INET, SOCK_STREAM | SOCK_CLOEXEC, 0);
  if (fd < 0) return -1;
  int one = 1;
  setsockopt(fd, SOL_SOCKET, SO_REUSEADDR, &one, sizeof(one));
  struct sockaddr_in sa;
  memset(&sa, 0, sizeof(sa));
  sa.sin_family = AF_INET;
  sa.sin_port = htons(port);
  if (inet_pton(AF_INET, addr, &sa.sin_addr) != 1) {
    close(fd);
    errno = EINVAL;
    return -1;
  }
  if (bind(fd, (struct sockaddr*)&sa, sizeof(sa)) != 0 || listen(fd, 128) != 0) {
    int e = errno;
    close(fd);
    errno = e;
    return -1;
  }
  fcntl(fd, F_SETFL, fcntl(fd, F_GETFL) | O_NONBLOCK);
  return fd;
}

void describe_transport(Ctx* c, Ep* ep) {
  ep->info.num_transports = 1;
  snprintf(ep->info.transport_device[0], 32, "cuda:%d", c->device);
  if (ep->in_process)
    snprintf(ep->info.transport_name[0], 32, "cuda_loopback");
  else if (ep->peer_device == c->device)
    snprintf(ep->info.transport_name[0], 32, "cuda_ipc");
  else
    snprintf(ep->info.transport_name[0], 32, "nvlink_ipc");
}

// Runs on the progress thread: accept one bootstrap connection and perform the handshake.
void server_handshake(Ctx* c, Worker* w, int fd, bool tcp) {
  set_sock_timeout(fd, 2.0);
  if (!tcp) {
    // abstract unix sockets carry no file permissions: accept peers of the same user only
    struct ucred cred;
    socklen_t cl = sizeof(cred);
    if (getsockopt(fd, SOL_SOCKET, SO_PEERCRED, &cred, &cl) != 0 || cred.uid != geteuid()) {
      close(fd);
      return;
    }
  }
  WireHello h;
  WireWelcome wl;
  memset(&wl, 0, sizeof(wl));
  wl.magic = WIRE_MAGIC;
  wl.status = SW_ERR_INVALID_PARAM;
  Ep* ep = nullptr;
  do {
    if (!read_all(fd, &h, sizeof(h)) || h.magic != WIRE_MAGIC) break;
    h.shm_name[sizeof(h.shm_name) - 1] = 0;
    if (w->eps.size() >= SW_MAX_EPS && w->free_ring_idx.empty()) {
      wl.status = SW_ERR_NO_MEMORY;   // SW_MAX_EPS connections OPEN at the same time
      break;
    }
    ep = ep_new(c, w);
    // ring index: a fresh one, or the index of an endpoint whose connection has ended and drained
    ep->index = w->free_ring_idx.empty() ? (uint32_t)w->eps.size() : w->free_ring_idx.back();
    ep->ring_gen = ++w->ring_gen_ctr[ep->index] & SW_EP_GEN_MASK;
    ep->peer_pid = h.pid;
    ep->peer_device = h.device;
    ep->peer_ctx_uuid = h.ctx_uuid;
    ep->peer_worker_id = h.worker_id;
    ep->in_process = (h.pid == (uint32_t)getpid() && h.ctx_uuid == c->uuid);
    ep->shm = shm_attach(h.shm_name, ep->shm_size, &ep->shm_dev);
    if (!ep->shm) {
      wl.status = SW_ERR_IO_ERROR;
      break;
    }
    ep->shm->pid[1] = (uint32_t)getpid();
    ep->out = &ep->shm->dir[1];
    ep->in = &ep->shm->dir[0];
    if (!ep_alloc_ring(c, ep)) {
      wl.status = SW_ERR_NO_MEMORY;
      break;
    }
    if (ep->in_process) {
      ep->peer_ring = (uint8_t*)(uintptr_t)h.ring_ptr;
      ep->ring_same_gpu = true;   // same context, same GPU
    } else {
      void* base = nullptr;
      if (swgpu::ipc_open(h.ring_handle, &base) != 0) {
        fprintf(stderr, "starway_b200: cannot map the client's inbound ring: %s\n", swgpu::last_error());
        wl.status = SW_ERR_UNREACHABLE;
        break;
      }
      ep->peer_ring_mapping = base;
      ep->peer_ring = (uint8_t*)base;
      {
        // CUDA ordinals of two processes need not agree (CUDA_VISIBLE_DEVICES): ask where the mapping lives
        swgpu::PtrInfo rpi;
        swgpu::ptr_info(ep->peer_ring, &rpi);
        ep->ring_same_gpu = rpi.is_device && rpi.device == c->device;
      }
      if (swgpu::ipc_get(ep->ring, wl.ring_handle) != 0) {
        wl.status = SW_ERR_IO_ERROR;
        break;
      }
    }
    ep->peer_ring_slots = h.ring_slots;
    if (swgpu::match_state_set_ring(w->mstate, ep->index, ep->ring, ep->ring_slots, ep->ring_gen) != 0) {
      wl.status = SW_ERR_IO_ERROR;
      break;
    }
    if (!ep_publish_words(w, ep)) {
      wl.status = SW_ERR_IO_ERROR;
      break;
    }
    w->cfg_dirty = true;   // a running control kernel does not know this ring yet
    // endpoint metadata (reference handle_new_endpoint, main.cpp:867-910)
    snprintf(ep->info.name, sizeof(ep->info.name), "starway-ep-%u[pid %u gpu %d]", ep->index, h.pid, h.device);
    if (tcp) {
      struct sockaddr_in la, ra;
      socklen_t ll = sizeof(la), rl = sizeof(ra);
      if (getsockname(fd, (struct sockaddr*)&la, &ll) == 0) {
        inet_ntop(AF_INET, &la.sin_addr, ep->info.local_addr, sizeof(ep->info.local_addr));
        ep->info.local_port = ntohs(la.sin_port);
      }
      if (getpeername(fd, (struct sockaddr*)&ra, &rl) == 0) {
        inet_ntop(AF_INET, &ra.sin_addr, ep->info.remote_addr, sizeof(ep->info.remote_addr));
        ep->info.remote_port = ntohs(ra.sin_port);
      }
    }
    describe_transport(c, ep);
    wl.status = SW_OK;
    wl.pid = (uint32_t)getpid();
    wl.device = c->device;
    wl.ctx_uuid = c->uuid;
    wl.worker_id = w->id;
    wl.ring_ptr = (uint64_t)(uintptr_t)ep->ring;
    wl.ring_slots = ep->ring_slots;
    wl.ep_index = ep->index;
  } while (0);

  if (wl.status == SW_OK) {
    // the endpoint is visible (list_clients) before the client learns the connect succeeded
    if (ep->index < w->eps.size()) {
      w->free_ring_idx.pop_back();
      w->tombs.push_back(w->eps[ep->index]);   // the retired record stays listed (list_clients never shrinks)
      w->eps[ep->index] = ep;
      if (w->pctl)   // the index starts a new life: its requests may go down the device path again
        __atomic_store_n(&w->pctl->dead_mask, w->pctl->dead_mask & ~(1ull << ep->index), __ATOMIC_RELEASE);
    } else {
      w->eps.push_back(ep);
    }
    {
      std::lock_guard<std::mutex> lk(c->mu);
      c->eps[ep->id] = ep;
    }
    if (!write_all(fd, &wl, sizeof(wl))) ep->peer_closed = true;
    complete(c, w, 0, SW_OP_ACCEPT, SW_OK, 0, 0, ep->id);
  } else {
    write_all(fd, &wl, sizeof(wl));
    if (ep) {
      if (ep->peer_ring_mapping) swgpu::ipc_close(ep->peer_ring_mapping);
      if (ep->ring) swgpu::dev_free(ep->ring);
      if (ep->shm) shm_release(ep->shm);
      Slab<Ep>::recycle(ep);
    }
  }
  close(fd);
}

void poll_listeners(Ctx* c, Worker* w) {
  if (w->status.load(std::memory_order_acquire) != SW_ST_RUNNING) return;
  for (int k = 0; k < 2; k++) {
    int lfd = k == 0 ? w->unix_fd : w->tcp_fd;
    if (lfd < 0) continue;
    for (int n = 0; n < 8 && w->pending_hello.size() < 64; n++) {
      int fd = accept4(lfd, nullptr, nullptr, SOCK_CLOEXEC);
      if (fd < 0) break;
      if (k == 1) {
        // The bootstrap exchanges CUDA IPC handles and the name of a shared-memory block: it only makes sense within
        // one host.  A connection made on this host has the same address at both ends.
        struct sockaddr_in la, ra;
        socklen_t ll = sizeof(la), rl = sizeof(ra);
        if (getsockname(fd, (struct sockaddr*)&la, &ll) != 0 || getpeername(fd, (struct sockaddr*)&ra, &rl) != 0 ||
            la.sin_addr.s_addr != ra.sin_addr.s_addr) {
          close(fd);
          continue;
        }
      }
      w->pending_hello.push_back(Worker::PendingHello{fd, k == 1, now_s() + 2.0});
    }
  }
  // The handshake runs on this thread (it touches the worker's endpoint tables): start it only once the client's
  // hello is in the socket buffer, so that a peer that connects and says nothing holds up nobody.
  for (size_t i = 0; i < w->pending_hello.size();) {
    Worker::PendingHello ph = w->pending_hello[i];
    int avail = 0;
    char probe;
    bool ready = ioctl(ph.fd, FIONREAD, &avail) == 0 && avail >= (int)sizeof(WireHello);
    bool dead = !ready && (now_s() > ph.deadline || recv(ph.fd, &probe, 1, MSG_PEEK | MSG_DONTWAIT) == 0);
    if (!ready && !dead) {
      i++;
      continue;
    }
    w->pending_hello.erase(w->pending_hello.begin() + (long)i);
    if (ready) server_handshake(c, w, ph.fd, ph.tcp);
    else close(ph.fd);
  }
}

// ============================================================================ connection: client side
struct ConnectReq {
  int mode;  // 0 tcp, 1 address blob
  std::string addr;
  uint16_t port;
  AddrBlob blob;
  uint64_t op_id;
};

void client_connect_thread(Ctx* c, Worker* w, ConnectReq req) {
  swgpu::bind_thread(c->device);
  int32_t status = SW_ERR_NOT_CONNECTED;
  int fd = -1;
  Ep* ep = nullptr;
  std::string shm_name;
  do {
    // ---- bootstrap socket
    if (req.mode == 0) {
      fd = socket(AF_INET, SOCK_STREAM | SOCK_CLOEXEC, 0);
      if (fd < 0) break;
      struct sockaddr_in sa;
      memset(&sa, 0, sizeof(sa));
      sa.sin_family = AF_INET;
      sa.sin_port = htons(req.port);
      if (inet_pton(AF_INET, req.addr.c_str(), &sa.sin_addr) != 1) {
        status = SW_ERR_INVALID_PARAM;
        break;
      }
      set_sock_timeout(fd, 5.0);
      if (connect(fd, (struct sockaddr*)&sa, sizeof(sa)) != 0) {
        status = (errno == ETIMEDOUT || errno == EINPROGRESS) ? SW_ERR_TIMED_OUT : SW_ERR_NOT_CONNECTED;
        break;
      }
      int one = 1;
      setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof(one));
    } else {
      if (req.blob.magic != ADDR_MAGIC || req.blob.unix_name[0] == 0) {
        status = SW_ERR_INVALID_PARAM;
        break;
      }
      fd = socket(AF_UNIX, SOCK_STREAM | SOCK_CLOEXEC, 0);
      if (fd < 0) break;
      struct sockaddr_un sa;
      memset(&sa, 0, sizeof(sa));
      sa.sun_family = AF_UNIX;
      req.blob.unix_name[sizeof(req.blob.unix_name) - 1] = 0;
      size_t n = strlen(req.blob.unix_name);
      memcpy(sa.sun_path + 1, req.blob.unix_name, n);
      set_sock_timeout(fd, 5.0);
      if (connect(fd, (struct sockaddr*)&sa, (socklen_t)(offsetof(struct sockaddr_un, sun_path) + 1 + n)) != 0) {
        status = SW_ERR_NOT_CONNECTED;
        break;
      }
    }
    // ---- local resources: device queues, inbound ring, control block
    status = SW_ERR_NO_MEMORY;
    if (!worker_alloc_device(c, w)) break;
    ep = ep_new(c, w);
    ep->index = 0;
    ep->is_client_side = true;
    if (!ep_alloc_ring(c, ep)) break;
    if (swgpu::match_state_set_ring(w->mstate, 0, ep->ring, ep->ring_slots) != 0) break;
    ep->shm = shm_create(shm_name, ep->shm_size, &ep->shm_dev);
    if (!ep->shm) {
      status = SW_ERR_IO_ERROR;
      break;
    }
    ep->shm->pid[0] = (uint32_t)getpid();
    ep->out = &ep->shm->dir[0];
    ep->in = &ep->shm->dir[1];
    if (!ep_publish_words(w, ep)) {
      status = SW_ERR_IO_ERROR;
      break;
    }
    // ---- handshake
    WireHello h;
    memset(&h, 0, sizeof(h));
    h.magic = WIRE_MAGIC;
    h.version = SW_ABI_VERSION;
    h.pid = (uint32_t)getpid();
    h.device = c->device;
    h.ctx_uuid = c->uuid;
    h.worker_id = w->id;
    h.ring_ptr = (uint64_t)(uintptr_t)ep->ring;
    h.ring_slots = ep->ring_slots;
    snprintf(h.shm_name, sizeof(h.shm_name), "%s", shm_name.c_str());
    if (swgpu::ipc_get(ep->ring, h.ring_handle) != 0) {
      // not fatal for an in-process peer; a remote peer will fail to map and refuse
      memset(h.ring_handle, 0, sizeof(h.ring_handle));
    }
    status = SW_ERR_NOT_CONNECTED;
    if (!write_all(fd, &h, sizeof(h))) break;
    WireWelcome wl;
    if (!read_all(fd, &wl, sizeof(wl)) || wl.magic != WIRE_MAGIC) break;
    if (wl.status != SW_OK) {
      status = wl.status;
      break;
    }
    ep->peer_pid = wl.pid;
    ep->peer_device = wl.device;
    ep->peer_ctx_uuid = wl.ctx_uuid;
    ep->peer_worker_id = wl.worker_id;
    ep->in_process = (wl.pid == (uint32_t)getpid() && wl.ctx_uuid == c->uuid);
    ep->peer_ring_slots = wl.ring_slots;
    if (ep->in_process) {
      ep->peer_ring = (uint8_t*)(uintptr_t)wl.ring_ptr;
      ep->ring_same_gpu = true;   // same context, same GPU
    } else {
      void* base = nullptr;
      if (swgpu::ipc_open(wl.ring_handle, &base) != 0) {
        fprintf(stderr, "starway_b200: cannot map the server's inbound ring: %s\n", swgpu::last_error());
        status = SW_ERR_UNREACHABLE;
        break;
      }
      ep->peer_ring_mapping = base;
      ep->peer_ring = (uint8_t*)base;
      {
        // CUDA ordinals of two processes need not agree (CUDA_VISIBLE_DEVICES): ask where the mapping lives
        swgpu::PtrInfo rpi;
        swgpu::ptr_info(ep->peer_ring, &rpi);
        ep->ring_same_gpu = rpi.is_device && rpi.device == c->device;
      }
    }
    snprintf(ep->info.name, sizeof(ep->info.name), "starway-server[pid %u gpu %d]", wl.pid, wl.device);
    describe_transport(c, ep);
    status = SW_OK;
  } while (0);
  if (fd >= 0) close(fd);
  if (!shm_name.empty()) shm_unlink(shm_name.c_str());  // both sides have it mapped (or the attempt failed)

  if (status == SW_OK) {
    w->eps.push_back(ep);
    {
      std::lock_guard<std::mutex> lk(c->mu);
      c->eps[ep->id] = ep;
    }
    w->status.store(SW_ST_INIT, std::memory_order_release);
    w->register_queued.store(true, std::memory_order_release);
    sq_push(c, SQ_REGISTER, w, (void*)(uintptr_t)req.op_id);
  } else {
    if (ep) {
      if (ep->peer_ring_mapping) swgpu::ipc_close(ep->peer_ring_mapping);
      if (ep->ring) swgpu::dev_free(ep->ring);
      if (ep->shm) shm_release(ep->shm);
      Slab<Ep>::recycle(ep);
    }
    if (w->mstate) {
      swgpu::match_state_destroy(w->mstate);
      w->mstate = nullptr;
    }
    w->status.store(SW_ST_CLOSED, std::memory_order_release);
    complete(c, w, req.op_id, SW_OP_CONNECT, status);
  }
}

// ============================================================================ progress: sends
// One put entry into the stamped ring (SwSendLL, sw_device.h): every 16-byte unit goes out in one store, so the
// control kernel -- which may read the entry before the cursor announces it -- only ever sees whole units.
static inline void send_ring_write(SwSendLL* dst, const SwSendEnt& e, uint64_t index) {
  const uint32_t stamp = sw_send_stamp(index);
  uint32_t w[SW_SEND_UNITS * 3] = {0};
  memcpy(w, &e, sizeof e);
  for (uint32_t k = 0; k < SW_SEND_UNITS; k++) {
#if defined(__SSE2__)
    _mm_store_si128(reinterpret_cast<__m128i*>(dst->u[k]),
                    _mm_set_epi32((int)stamp, (int)w[3 * k + 2], (int)w[3 * k + 1], (int)w[3 * k]));
#else
    dst->u[k][0] = w[3 * k];
    dst->u[k][1] = w[3 * k + 1];
    dst->u[k][2] = w[3 * k + 2];
    __atomic_store_n(&dst->u[k][3], stamp, __ATOMIC_RELEASE);
#endif
  }
}

bool pump_sends(Ctx* c) {
  if ((c->put_tail - c->put_head) >= (uint32_t)N_PUT_BLOCKS) return false;
  PutBlock& b = c->put_blocks[c->put_tail % N_PUT_BLOCKS];
  uint32_t n = 0;
  uint64_t bytes = 0, h2d = 0, staged_bytes = 0;
  bool batch_full = false, stream_ordered = false;
  const uint64_t eager_max = (uint64_t)std::min<int64_t>(c->opt_eager_max.load(), SW_EAGER_MAX);
  b.items.clear();
  b.nsegs = 0;
  b.res_worker = nullptr;
  b.up_dst.clear();
  b.up_src.clear();
  b.up_len.clear();
  for (Worker* w : c->active) {
    for (Ep* ep : w->eps) {
      while (!ep->sendq.empty() && n < PUT_BATCH) {
        SendOp* op = ep->sendq.front();
        if (ep->peer_closed) {
          ep->sendq.pop_front();
          send_finished(c, op, SW_ERR_CONNECTION_RESET);
          continue;
        }
        uint64_t consumed = ep->out->consumed.load(std::memory_order_acquire);
        if (ep->out_sent - consumed >= ep->peer_ring_slots) break;  // no credit
        // the FIN words of a connection are indexed by the rendezvous sequence number modulo SW_FIN_SLOTS
        if (op->len > eager_max && ep->rndv_wait.size() >= SW_FIN_SLOTS - 1) break;
        SwPutDesc& d = b.descs[n];
        d.tag = op->tag;
        d.msg_len = op->len;
        bool rndv = false;
        if (op->len <= eager_max) {
          if (op->mem == SW_MEM_HOST) {
            memcpy(b.stage + (size_t)n * SW_SLOT_BYTES, op->ptr, op->len);
            d.src = (uint64_t)(uintptr_t)(b.stage + (size_t)n * SW_SLOT_BYTES);
            h2d += op->len;
          } else {
            d.src = (uint64_t)(uintptr_t)op->ptr;
          }
          d.len = (uint32_t)op->len;
          d.kind = SW_KIND_EAGER;
        } else {
          // ---- rendezvous: publish a descriptor of the source, the receiver pulls
          rndv = true;
          SwRts& r = b.rts[n];
          memset(&r, 0, sizeof(r));
          uint64_t base = 0, size = 0, buffer_id = 0;
          int srcdev = c->device;
          if (op->mem == SW_MEM_HOST && ep->in_process && c->opt_pinned_send_direct.load()) {
            swgpu::PtrInfo pi;
            swgpu::ptr_info(op->ptr, &pi);
            if (pi.is_pinned) op->mem = MEM_PINNED;  // same process: the receiver's kernel reads it in place
          }
          if (op->mem == MEM_PINNED) {
            base = (uint64_t)(uintptr_t)op->ptr;
            size = op->len;
            r.src_ptr = base;
            r.pad[0] = SW_RTS_PINNED_SRC;
          } else if (op->mem != SW_MEM_HOST && !ep->in_process && !op->stage_d2d && !op->dev_staging) {
            // device source, peer in another process: can the allocation be exported?  (answer cached per allocation)
            swgpu::PtrInfo pi;
            swgpu::ptr_info(op->ptr, &pi);
            if (!pi.is_device || pi.base == 0) {
              ep->sendq.pop_front();
              set_error("rendezvous source is not a CUDA device allocation");
              send_finished(c, op, SW_ERR_INVALID_PARAM);
              continue;
            }
            auto hit = pi.buffer_id ? c->handle_cache.find(pi.buffer_id) : c->handle_cache.end();
            if (hit != c->handle_cache.end() && hit->second.base == pi.base) {
              op->stage_d2d = !hit->second.exportable;
            } else {
              Ctx::HandleEnt he;
              he.base = pi.base;
              he.exportable = swgpu::ipc_get((void*)(uintptr_t)pi.base, he.handle) == 0;
              if (pi.buffer_id) {
                if (c->handle_cache.size() > 8192) c->handle_cache.clear();
                c->handle_cache[pi.buffer_id] = he;
              }
              op->stage_d2d = !he.exportable;
            }
          }
          if (op->mem == MEM_PINNED) {
            // (handled above)
          } else if (op->mem == SW_MEM_HOST || op->stage_d2d) {
            // Staged sends are published batch by batch: keep batches small so that the receiver can
            // start pulling the first payloads while later ones are still being uploaded.
            // (Host memory; or device memory from the CUDA virtual-memory-management API -- PyTorch's expandable
            // segments -- which cudaIpcGetMemHandle cannot export: one device-to-device copy into an exportable
            // staging buffer, at HBM speed, keeps such tensors usable as rendezvous sources.)
            if (!op->dev_staging && n > 0 && staged_bytes + op->len > (uint64_t)c->opt_stage_batch_bytes.load()) {
              batch_full = true;
              break;
            }
            if (op->mem == SW_MEM_HOST && !op->stage_d2d && !op->dev_staging && !c->copy_pool.threads.empty()) {
              // pageable source: helper threads copy it into page-locked staging first (started here, for this
              // operation and the next few of the queue), the upload then is a plain DMA
              if (!op->pin_stage) {
                swgpu::PtrInfo hpi;
                swgpu::ptr_info(op->ptr, &hpi);
                if (!hpi.is_pinned) {
                  size_t ahead = 0;
                  for (SendOp* o2 : ep->sendq) {
                    if (ahead++ >= 8 || c->pin_inflight > (512u << 20)) break;
                    if (o2->pin_stage || o2->mem != SW_MEM_HOST || o2->len <= eager_max || o2->dev_staging) continue;
                    o2->pin_stage = c->pinned_pool.get(o2->len, &o2->pin_stage_size);
                    if (!o2->pin_stage) break;
                    c->pin_inflight += o2->pin_stage_size;
                    c->copy_pool.submit(o2->pin_stage, o2->ptr, o2->len, &o2->pin_pending);
                  }
                }
              }
              if (op->pin_stage && op->pin_pending.load(std::memory_order_acquire) > 0) break;   // not copied yet
            }
            if (!op->dev_staging) staged_bytes += op->len;
            if (!op->dev_staging) {
              op->dev_staging = c->staging.get(op->len, &op->staging_size);
              if (!op->dev_staging) {
                ep->sendq.pop_front();
                send_finished(c, op, SW_ERR_NO_MEMORY);
                continue;
              }
              if (op->stage_d2d) {
                trace(c, "d2d_stage", op->len);
                swgpu::memcpy_d2d(op->dev_staging, op->ptr, op->len, b.s);
                stream_ordered = true;
              } else {
              swgpu::PtrInfo hpi;
              swgpu::ptr_info(op->ptr, &hpi);
              const uint64_t pieces = (op->len + STAGE_SEG_BYTES - 1) / STAGE_SEG_BYTES;
              if (c->opt_stage_upload_kernel.load() && hpi.is_pinned && ((uintptr_t)op->ptr & 15) == 0 &&
                  b.nsegs + pieces + 1 <= STAGE_SEGS) {
                // pinned source: the upload is part of this batch's device work (TMA bulk kernel
                // reading host memory), no per-message copy-engine operation
                const uint64_t body = op->len & ~15ull;
                for (uint64_t off = 0; off < body; off += STAGE_SEG_BYTES)
                  b.segs[b.nsegs++] = SwSeg{(uint64_t)(uintptr_t)op->ptr + off, (uint64_t)(uintptr_t)op->dev_staging + off,
                                            std::min<uint64_t>(STAGE_SEG_BYTES, body - off), 0};
                stream_ordered = true;
                if (op->len > body)
                  swgpu::memcpy_h2d((uint8_t*)op->dev_staging + body, op->ptr + body, op->len - body, b.s);
              } else {
                b.up_dst.push_back(op->dev_staging);
                b.up_src.push_back(op->pin_stage ? (const void*)op->pin_stage : (const void*)op->ptr);
                b.up_len.push_back((size_t)op->len);
                stream_ordered = true;   // the RTS may only become visible after this copy: needs the put launch behind it
              }
              h2d += op->len;
              }
            }
            base = (uint64_t)(uintptr_t)op->dev_staging;
            size = op->staging_size;
            r.src_ptr = base;
            if (!ep->in_process) {
              swgpu::PtrInfo spi;
              swgpu::ptr_info(op->dev_staging, &spi);
              buffer_id = spi.buffer_id;
            }
          } else {
            r.src_ptr = (uint64_t)(uintptr_t)op->ptr;
            if (!ep->in_process) {
              // a peer in another process maps the allocation: it needs base, size and an IPC handle
              swgpu::PtrInfo pi;
              swgpu::ptr_info(op->ptr, &pi);
              base = pi.base;
              size = pi.size;
              srcdev = pi.device;
              buffer_id = pi.buffer_id;
            }
          }
          if (!ep->in_process) {
            // IPC handles are cached per allocation (CUDA buffer id: changes if the address is re-allocated)
            auto hit = buffer_id ? c->handle_cache.find(buffer_id) : c->handle_cache.end();
            if (hit != c->handle_cache.end() && hit->second.base == base) {
              memcpy(r.ipc_handle, hit->second.handle, 64);
            } else if (swgpu::ipc_get((void*)(uintptr_t)base, r.ipc_handle) != 0) {
              fprintf(stderr, "starway_b200: cudaIpcGetMemHandle failed: %s\n", swgpu::last_error());
              ep->sendq.pop_front();
              send_finished(c, op, SW_ERR_INVALID_PARAM);
              continue;
            } else if (buffer_id) {
              if (c->handle_cache.size() > 8192) c->handle_cache.clear();
              Ctx::HandleEnt he;
              he.base = base;
              memcpy(he.handle, r.ipc_handle, 64);
              c->handle_cache[buffer_id] = he;
            }
          }
          r.alloc_base = base;
          r.alloc_size = size;
          r.pad[1] = buffer_id;   // key of the receiver's device-resident mapping table
          r.ctx_uuid = c->uuid;
          r.src_pid = (uint32_t)getpid();
          r.src_dev = srcdev;
          op->rndv_seq = ep->rndv_next++;
          r.send_seq = op->rndv_seq;
          d.src = (uint64_t)(uintptr_t)&r;
          d.len = (uint32_t)sizeof(SwRts);
          d.kind = SW_KIND_RTS;
        }
        d.dst = (uint64_t)(uintptr_t)(ep->peer_ring + (size_t)(ep->out_sent % ep->peer_ring_slots) * SW_SLOT_BYTES);
        d.seq = ep->out_sent + 1;
        ep->out_sent++;
        ep->puts_inflight++;
        ep->sendq.pop_front();
        if (rndv) ep->rndv_wait[op->rndv_seq] = op;
        op->in_put = true;
        b.items.push_back(PutItem{ep, op, rndv});
        bytes += d.len;
        n++;
      }
      if (n >= PUT_BATCH || batch_full) break;
    }
    if (n >= PUT_BATCH || batch_full) break;
  }
  if (!n) return false;
  if (!b.up_dst.empty()) {
    // the uploads of this batch in one copy-engine submission, in front of the put that announces them
    trace(c, "h2d_batch", b.up_dst.size(), staged_bytes);
    if (swgpu::memcpy_h2d_batch(b.up_dst.data(), b.up_src.data(), b.up_len.data(), b.up_dst.size(), b.s) != 0)
      fprintf(stderr, "starway_b200: staging upload failed: %s\n", swgpu::last_error());
  }
  // ---- small batch of one worker whose control kernel is resident: hand the descriptors to that kernel
  if (n <= (uint32_t)c->opt_resident_puts.load() && !stream_ordered && b.nsegs == 0 && swgpu::resident_lingers()) {
    Worker* w0 = b.items[0].op->w;
    bool one = w0->prog_running && c->opt_profile.load() < 2 &&
               w0->sends_written + n - __atomic_load_n(&w0->pctl->send_done, __ATOMIC_ACQUIRE) <= SW_SEND_RING;
    for (uint32_t i = 1; one && i < n; i++) one = b.items[i].op->w == w0;
    // the put warp takes a lane per put for RTS descriptors and payloads up to 256 B; larger eager payloads are
    // copied by the whole warp one after the other -- a launch (a warp per message) is faster for more than two
    uint32_t large = 0;
    for (uint32_t i = 0; i < n; i++) large += b.descs[i].kind == SW_KIND_EAGER && b.descs[i].len > 256;
    one = one && large <= 2;
    if (one) {
      for (uint32_t i = 0; i < n; i++) {
        SwSendEnt e;
        memset(&e, 0, sizeof e);
        e.d = b.descs[i];
        // RTS descriptors and small host payloads travel inside the entry: the kernel fetches descriptor and
        // payload in one PCIe round trip
        const bool staged_payload = e.d.src >= (uint64_t)(uintptr_t)b.stage && e.d.src < (uint64_t)(uintptr_t)b.stage + (uint64_t)PUT_BATCH * SW_SLOT_BYTES;
        if (e.d.kind == SW_KIND_RTS || (staged_payload && e.d.len <= sizeof(e.inl))) {
          memcpy(e.inl, (const void*)(uintptr_t)e.d.src, e.d.len);
          e.d.src = 0;
        }
        if (b.items[i].op->ep && b.items[i].op->ep->ring_same_gpu) e.d.kind |= SW_KIND_SAME_GPU;
        send_ring_write(&w0->send_ring[(w0->sends_written + i) % SW_SEND_RING], e, w0->sends_written + i);
      }
      w0->sends_written += n;
      __atomic_store_n(&w0->pctl->send_tail, w0->sends_written, __ATOMIC_RELEASE);
      trace(c, "put_resident", n, bytes + h2d);
      b.res_worker = w0;
      b.res_end = w0->sends_written;
      b.flag_mode = false;
      b.timed = false;
      b.busy = true;
      c->put_tail++;
      w0->last_activity = now_s();
      std::lock_guard<std::mutex> lk(c->st_mu);
      c->stats.put_resident++;
      c->stats.put_msgs += n;
      c->stats.put_bytes += bytes;
      c->stats.h2d_bytes += h2d;
      return true;
    }
  }
  b.timed = c->opt_profile.load() >= 2;
  if (b.timed) swgpu::event_record(b.ev_start, b.s);
  if (b.nsegs) {
    swgpu::BulkTuning up{0, 8, 24576, 1, 0};
    trace(c, "stage_upload_launch", b.nsegs, staged_bytes);
    if (swgpu::launch_bulk(b.s, b.segs, b.nsegs, &up) != 0)
      fprintf(stderr, "starway_b200: staging upload launch failed: %s\n", swgpu::last_error());
  }
  trace(c, "put_launch", n, bytes + h2d);
  swgpu::DoneFlag df{b.done, ++c->flag_seq};
  const int lr = swgpu::launch_put(b.s, b.descs, n, (b.timed || !c->opt_done_flags.load()) ? nullptr : &df);
  if (lr < 0) fprintf(stderr, "starway_b200: put launch failed: %s\n", swgpu::last_error());
  b.flag_mode = lr == 1;
  b.done_seq = df.value;
  b.spins = 0;
  if (!b.flag_mode) swgpu::event_record(b.timed ? b.ev : b.ev_fast, b.s);
  b.busy = true;
  c->put_tail++;
  std::lock_guard<std::mutex> lk(c->st_mu);
  c->stats.put_launches++;
  c->stats.put_msgs += n;
  c->stats.put_bytes += bytes;
  c->stats.h2d_bytes += h2d;
  return true;
}

bool poll_puts(Ctx* c) {
  bool any = false;
  while (c->put_head != c->put_tail) {
    PutBlock& b = c->put_blocks[c->put_head % N_PUT_BLOCKS];
    int q;
    if (b.res_worker) {
      // the resident kernel of the sending worker executes these puts (if it left first, the relaunch does)
      q = __atomic_load_n(&b.res_worker->pctl->send_done, __ATOMIC_ACQUIRE) >= b.res_end ? 0 : 1;
    } else if (b.flag_mode) {
      q = __atomic_load_n(b.done, __ATOMIC_ACQUIRE) == b.done_seq ? 0 : 1;
      // a faulted launch never writes its flag: look at the stream now and then
      if (q == 1 && (++b.spins & 0x3FF) == 0 && swgpu::stream_query(b.s) < 0) q = -1;
    } else {
      q = swgpu::event_query(b.timed ? b.ev : b.ev_fast);
    }
    if (q == 1) break;
    if (q < 0) fprintf(stderr, "starway_b200: put kernel failed: %s\n", swgpu::last_error());
    if (b.timed) {
      float ms = swgpu::event_elapsed_ms(b.ev_start, b.ev);
      if (ms >= 0) {
        std::lock_guard<std::mutex> lk(c->st_mu);
        c->stats.put_event_ms += ms;
        c->stats.put_event_launches++;
      }
    }
    trace(c, "put_done", b.items.size());
    // publish the slots (doorbell), then complete the eager sends
    for (PutItem& it : b.items) {
      it.ep->out_published++;
      it.ep->puts_inflight--;
    }
    for (PutItem& it : b.items) {
      Ep* ep = it.ep;
      if (ep->out->produced.load(std::memory_order_relaxed) != ep->out_published)
        ep->out->produced.store(ep->out_published, std::memory_order_release);
    }
    for (PutItem& it : b.items) {
      SendOp* op = it.op;
      op->in_put = false;
      if (op->ended_early) {
        send_finished(c, op, op->early_status);
      } else if (!it.rndv) {
        send_finished(c, op, q < 0 ? SW_ERR_IO_ERROR : SW_OK);
      } else if (op->dev_staging && !op->user_done) {
        // host buffer has been staged on the device: the caller may reuse it (UCX eager-bcopy semantics)
        complete(c, op->w, op->op_id, SW_OP_SEND, SW_OK);
        op->user_done = true;
      }
    }
    b.items.clear();
    b.busy = false;
    c->put_head++;
    any = true;
  }
  return any;
}

// ============================================================================ progress: rendezvous pulls
uint64_t pull_outstanding(Ctx* c);
// device-side users of the mapping table / of mapped addresses: running control kernels, unfinished pulls
bool mappings_in_use_on_device(Ctx* c) {
  for (Worker* w : c->active)
    if (w->prog_running) return true;
  return pull_outstanding(c) != 0;
}

// Maps the sender's allocation (cached).  New mappings are also entered into the device-resident table, so
// that the next rendezvous from that allocation is resolved by the control kernel without the host.
// *retry: the cache is full and entries can only be dropped while no resident kernel runs -- try again later.
void* resolve_mapping(Ctx* c, BulkJob& j, bool* retry) {
  *retry = false;
  MapKey key;
  key.pid = j.rts.src_pid;
  memcpy(key.handle, j.rts.ipc_handle, 64);
  auto it = c->mappings.find(key);
  if (it == c->mappings.end()) {
    // Bound the cache (PyTorch's caching allocator hands out many small segments: a few hundred
    // distinct IPC handles are normal).  Opening/closing a mapping costs ~100s of us, so only
    // the least recently used idle quarter is dropped when the bound is hit.
    if (c->mappings.size() >= (size_t)std::max<int64_t>(1, c->opt_max_mappings.load())) {
      if (mappings_in_use_on_device(c)) {
        // A control kernel may be resolving through the table, a pull may be reading through a mapping:
        // have the control kernels leave (no relaunch while evict_pending), let the pulls drain, come back.
        c->evict_pending = true;
        for (Worker* w : c->active)
          if (w->prog_running) __atomic_store_n(&w->pctl->stop, 1, __ATOMIC_RELEASE);
        *retry = true;
        return nullptr;
      }
      c->evict_pending = false;
      std::vector<std::pair<double, MapKey>> idle;
      for (auto& kv : c->mappings)
        if (kv.second.refs == 0) idle.emplace_back(kv.second.last_use, kv.first);
      std::sort(idle.begin(), idle.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
      size_t drop = std::max<size_t>(1, idle.size() / 4);
      trace(c, "map_evict", std::min(drop, idle.size()), c->mappings.size());
      for (size_t i = 0; i < drop && i < idle.size(); i++) {
        auto m = c->mappings.find(idle[i].second);
        swgpu::ipc_close(m->second.base);
        c->mappings.erase(m);
      }
      // rebuild the device table from what is left
      swgpu::map_table_clear(c->map_tbl);
      for (auto& kv : c->mappings)
        if (kv.second.buf_id)
          swgpu::map_table_insert(c->map_tbl, c->s_map, kv.second.uuid, kv.second.buf_id, kv.second.remote_base,
                                  (uint64_t)(uintptr_t)kv.second.base);
    }
    void* base = nullptr;
    if (swgpu::ipc_open(j.rts.ipc_handle, &base) != 0) {
      fprintf(stderr, "starway_b200: cannot map the sender's buffer: %s\n", swgpu::last_error());
      return nullptr;
    }
    Mapping m{base, 0, now_s(), j.rts.ctx_uuid, j.rts.pad[1], j.rts.alloc_base};
    if (m.buf_id &&
        swgpu::map_table_insert(c->map_tbl, c->s_map, m.uuid, m.buf_id, m.remote_base, (uint64_t)(uintptr_t)base) != 0)
      m.buf_id = 0;   // probe window full: this allocation keeps going through the host
    it = c->mappings.emplace(key, m).first;
  }
  it->second.refs++;
  it->second.last_use = now_s();
  j.mapping = &it->second;
  return it->second.base;
}
void release_mapping(Ctx* c, BulkJob& j) {
  (void)c;
  if (j.mapping && j.mapping->refs) j.mapping->refs--;
  j.mapping = nullptr;
}

void bulk_job_done(Ctx* c, BulkJob& j, int32_t status) {
  recv_finish(c, j.w, j.recv_op, status, j.tag, j.len);
  if (j.ep) {
    bool was_cancelled = j.ep->canceled_rts.erase(j.rts.send_seq) > 0;
    (void)was_cancelled;
    // FIN: the sender's buffer is no longer needed (UCX: rendezvous ATS).  A message the receive refused (too long,
    // or not a whole number of elements for a reducing receive) was still consumed: the send succeeded.
    const bool refused = status == SW_ERR_MESSAGE_TRUNCATED || (j.dtype && status == SW_ERR_INVALID_PARAM);
    ctl_send(j.ep, CTL_FIN, refused ? SW_OK : status, j.rts.send_seq);
  }
  release_mapping(c, j);
  if (j.w->bulk_inflight) j.w->bulk_inflight--;
}

bool pump_bulk(Ctx* c) {
  if (c->pending_bulk.empty()) {
    c->evict_pending = false;
    return false;
  }
  if ((c->bulk_tail - c->bulk_head) >= (uint32_t)N_BULK_BLOCKS) return false;
  {
    // Coalesce: while more matches are on their way (ops queued, puts in flight, receives not yet handed to
    // the device), hold the launch until enough bytes are pending or the oldest job has waited opt_coalesce_us.
    bool upstream = c->sq_head.load(std::memory_order_acquire) != nullptr || c->put_head != c->put_tail;
    for (Worker* w : c->active) upstream |= !w->new_posts.empty();
    if (upstream) {
      uint64_t bytes = 0;
      for (auto& j : c->pending_bulk) bytes += j.len;
      double age_us = (now_s() - c->pending_bulk.front().t_enq) * 1e6;
      if (bytes < (uint64_t)c->opt_coalesce_bytes.load() && age_us < (double)c->opt_coalesce_us.load()) return false;
    }
  }
  BulkBlock& b = c->bulk_blocks[c->bulk_tail % N_BULK_BLOCKS];
  b.jobs.clear();
  b.bytes = 0;
  const uint64_t MAX_BYTES = 8ull << 30;
  // ---- choose the jobs of this launch
  while (!c->pending_bulk.empty() && b.jobs.size() < 2048 && b.bytes < MAX_BYTES) {
    BulkJob j = c->pending_bulk.front();
    c->pending_bulk.pop_front();
    j.w->bulk_inflight++;
    if (!j.failed && j.ep && j.ep->canceled_rts.count(j.rts.send_seq)) {
      j.failed = true;
      j.fail_status = SW_ERR_CONNECTION_RESET;
    }
    if (!j.failed && !j.src_ready) {
      if (j.rts.ctx_uuid == c->uuid && j.rts.src_pid == (uint32_t)getpid()) {
        j.src = j.rts.src_ptr;
      } else {
        bool retry = false;
        void* base = resolve_mapping(c, j, &retry);
        if (retry) {   // the mapping cache has to wait for the resident kernels to leave
          j.w->bulk_inflight--;
          c->pending_bulk.push_front(j);
          break;
        }
        if (!base) {
          j.failed = true;
          j.fail_status = SW_ERR_UNREACHABLE;
        } else {
          j.src = (uint64_t)(uintptr_t)base + (j.rts.src_ptr - j.rts.alloc_base);
        }
      }
    }
    if (j.failed) {
      if (j.fail_status == SW_ERR_CONNECTION_RESET) {
        // cancelled by the sender: no FIN, the CANCEL_ACK was already sent
        recv_finish(c, j.w, j.recv_op, j.fail_status, j.tag, j.len);
        if (j.ep) j.ep->canceled_rts.erase(j.rts.send_seq);
        j.w->bulk_inflight--;
      } else {
        bulk_job_done(c, j, j.fail_status);
      }
      continue;
    }
    b.bytes += j.len;
    b.jobs.push_back(j);
  }
  if (b.jobs.empty()) return true;
  // ---- segment list: [0, ntma) TMA-eligible pieces, [ntma, nseg) generic pieces
  swgpu::BulkTuning tune;
  tune.mode = (int)c->opt_bulk_mode.load();
  tune.stages = (int)c->opt_bulk_stages.load();
  tune.stage_bytes = (int)c->opt_bulk_stage_bytes.load();
  tune.ctas_per_sm = (int)c->opt_bulk_ctas.load();
  tune.balance = (int)c->opt_bulk_balance.load();
  const uint64_t sms = (uint64_t)swgpu::sm_count();
  uint64_t target = sms * (uint64_t)std::max(1, tune.ctas_per_sm) * 4;
  uint64_t seg = (b.bytes + target - 1) / target;
  const uint64_t unit = tune.mode == 0 ? (uint64_t)std::max(1024, tune.stage_bytes & ~15) : 65536;
  seg = ((seg + unit - 1) / unit) * unit;
  seg = std::max<uint64_t>(seg, std::max<uint64_t>(unit, 65536 / unit * unit));
  seg = std::min<uint64_t>(seg, 4u << 20);
  while ((b.bytes / seg) + 2 * b.jobs.size() + 2 > MAX_SEGS) seg *= 2;
  std::vector<SwSeg>& tma = b.tma;
  std::vector<SwSeg>& simt = b.simt;
  tma.clear();
  simt.clear();
  b.ce_dst.clear();
  b.ce_src.clear();
  b.ce_len.clear();
  for (int dt = 0; dt < 7; dt++) {
    b.rtma[dt].clear();
    b.rsimt[dt].clear();
  }
  for (BulkJob& j : b.jobs) {
    uint64_t src = j.src, dst = j.dst, len = j.len;
    if (j.host_side && !j.src_host && c->opt_hostdst_ce.load()) {
      // device (local or peer staging) -> pinned host: the copy engine, one batched submission per launch block --
      // with the other direction of the PCIe link busy it keeps ~50 GB/s where a copying kernel drops to ~35
      b.ce_dst.push_back((void*)(uintptr_t)dst);
      b.ce_src.push_back((const void*)(uintptr_t)src);
      b.ce_len.push_back((size_t)len);
      continue;
    }
    // receives into host memory were redirected to device staging at post time (a reducing receive's destination
    // is always device memory: host_side means a pinned-host source there)
    const bool tma_ok = !j.host_side || (!j.src_host && c->opt_hostdst_tma.load());   // device -> pinned host: bulk stores over PCIe
    std::vector<SwSeg>& to_tma = j.dtype ? b.rtma[j.dtype] : tma;
    std::vector<SwSeg>& to_simt = j.dtype ? b.rsimt[j.dtype] : simt;
    if (tune.mode == 0 && tma_ok && ((src | dst) & 15) == 0 && len >= 16) {
      uint64_t body = len & ~15ull;
      for (uint64_t off = 0; off < body; off += seg) to_tma.push_back(SwSeg{src + off, dst + off, std::min(seg, body - off), 0});
      if (len > body) to_simt.push_back(SwSeg{src + body, dst + body, len - body, 0});
    } else {
      for (uint64_t off = 0; off < len; off += seg) to_simt.push_back(SwSeg{src + off, dst + off, std::min(seg, len - off), 0});
    }
  }
  uint32_t ntma = (uint32_t)tma.size(), nsimt = (uint32_t)simt.size();
  if (ntma) memcpy(b.segs, tma.data(), sizeof(SwSeg) * ntma);
  if (nsimt) memcpy(b.segs + ntma, simt.data(), sizeof(SwSeg) * nsimt);
  b.timed = c->opt_profile.load() != 0;
  if (b.timed) swgpu::event_record(b.ev_start, c->s_bulk);
  trace(c, "bulk_launch", b.jobs.size(), b.bytes);
  int rc = 0;
  if (ntma) rc |= swgpu::launch_bulk(c->s_bulk, b.segs, ntma, &tune);
  if (nsimt) {
    swgpu::BulkTuning t2 = tune;
    t2.mode = 1;
    t2.ctas_per_sm = 8;
    rc |= swgpu::launch_bulk(c->s_bulk, b.segs + ntma, nsimt, &t2);
  }
  if (!b.ce_dst.empty()) rc |= swgpu::memcpy_batch(b.ce_dst.data(), b.ce_src.data(), b.ce_len.data(), b.ce_dst.size(), c->s_bulk);
  // reducing receives: one launch per element type and kernel, their segments after the copies' in b.segs
  uint32_t nseg = ntma + nsimt, nred_tma = 0, nred_simt = 0;
  for (int dt = 1; dt < 7; dt++) {
    for (int simt_k = 0; simt_k < 2; simt_k++) {
      const std::vector<SwSeg>& v = simt_k ? b.rsimt[dt] : b.rtma[dt];
      if (v.empty()) continue;
      memcpy(b.segs + nseg, v.data(), sizeof(SwSeg) * v.size());
      swgpu::BulkTuning t2 = tune;
      if (simt_k) {
        t2.mode = 1;
        t2.ctas_per_sm = 8;
      }
      rc |= swgpu::launch_reduce(c->s_bulk, b.segs + nseg, (uint32_t)v.size(), dt, &t2);
      nseg += (uint32_t)v.size();
      (simt_k ? nred_simt : nred_tma)++;
    }
  }
  if (rc) fprintf(stderr, "starway_b200: bulk launch failed: %s\n", swgpu::last_error());
  swgpu::event_record(b.timed ? b.ev : b.ev_fast, c->s_bulk);
  b.busy = true;
  c->bulk_tail++;
  std::lock_guard<std::mutex> lk(c->st_mu);
  if (ntma) c->stats.bulk_tma_launches++;
  if (nsimt) c->stats.bulk_simt_launches++;
  c->stats.bulk_tma_launches += nred_tma;
  c->stats.bulk_simt_launches += nred_simt;
  c->stats.bulk_jobs += b.jobs.size();
  c->stats.bulk_bytes += b.bytes;
  return true;
}

bool poll_bulk(Ctx* c) {
  bool any = false;
  while (c->bulk_head != c->bulk_tail) {
    BulkBlock& b = c->bulk_blocks[c->bulk_head % N_BULK_BLOCKS];
    int q = swgpu::event_query(b.timed ? b.ev : b.ev_fast);
    if (q == 1) break;
    if (q < 0) fprintf(stderr, "starway_b200: bulk kernel failed: %s\n", swgpu::last_error());
    if (b.timed) {
      float ms = swgpu::event_elapsed_ms(b.ev_start, b.ev);
      if (ms >= 0) {
        std::lock_guard<std::mutex> lk(c->st_mu);
        c->stats.bulk_event_ms += ms;
        c->stats.bulk_event_launches++;
        c->stats.bulk_event_bytes += b.bytes;
      }
    }
    trace(c, "bulk_done", b.jobs.size(), b.bytes);
    for (BulkJob& j : b.jobs) bulk_job_done(c, j, q < 0 ? SW_ERR_IO_ERROR : SW_OK);
    b.jobs.clear();
    b.busy = false;
    c->bulk_head++;
    any = true;
  }
  // host receives: device -> page-locked copies finish in order; the helper threads' second hop may not, so the
  // queue is scanned (it is short: one entry per large host receive in flight)
  for (size_t i = 0; i < c->post_copies.size();) {
    PostCopy& pc = c->post_copies[i];
    if (pc.phase == 0) {
      int q = swgpu::event_query(pc.ev);
      if (q == 1) break;   // later entries' copies are behind this one on the stream
      swgpu::event_destroy(pc.ev);
      pc.ev = nullptr;
      if (q < 0) pc.status = SW_ERR_IO_ERROR;
      if (pc.op->pin_stage && q == 0) {
        c->copy_pool.submit(pc.op->ptr, pc.op->pin_stage, (size_t)pc.len, &pc.op->pin_pending);
        pc.phase = 1;
        any = true;
        i++;
        continue;
      }
      pc.phase = 2;
    }
    if (pc.phase == 1) {
      if (pc.op->pin_pending.load(std::memory_order_acquire) > 0) {
        i++;
        continue;
      }
      pc.phase = 2;
    }
    complete(c, pc.op->w, pc.op->op_id, SW_OP_RECV, pc.status, pc.tag, pc.len);
    recv_release(c, pc.op);
    c->post_copies.erase(c->post_copies.begin() + (long)i);
    any = true;
  }
  return any;
}

// ============================================================================ progress: resident control kernel
// The host only feeds the post ring, drains the completion rings and keeps the kernels alive while work is
// expected.
uint64_t unseen_arrivals(Worker* w) {
  uint64_t unseen = 0;
  for (Ep* ep : w->eps) {
    if (!ep->in) continue;
    const uint64_t p = ep->in->produced.load(std::memory_order_acquire);
    const uint64_t cns = ep->in->consumed.load(std::memory_order_acquire);
    if (p > cns) unseen += p - cns;
  }
  return unseen;
}

inline bool cq_ready(const SwCqEnt* e, uint64_t idx, int32_t* status) {
  // status and pass number share one 8-byte word, stored last by the device
  const uint64_t w = __atomic_load_n(reinterpret_cast<const uint64_t*>(&e->status), __ATOMIC_ACQUIRE);
  if (static_cast<uint32_t>(w >> 32) != sw_ring_pass(idx, SW_CQ_RING)) return false;
  *status = static_cast<int32_t>(static_cast<uint32_t>(w));
  return true;
}

// An eager message matched by a reducing receive sits in the receive's landing block: it becomes a bulk job from there
// into the caller's buffer, launched with whatever else is pending (bulk_job_done then completes the receive).
// Returns false when the receive completes as it is: not a reducing receive, an error, or length 0.
bool reduce_landed(Ctx* c, Worker* w, uint64_t op_id, int32_t status, uint64_t tag, uint64_t len) {
  auto it = w->recvs.find(op_id);
  if (it == w->recvs.end() || !it->second->dtype || status != SW_OK || !len) return false;
  RecvOp* r = it->second;
  if (len % sw_dtype_size(r->dtype)) {
    recv_finish(c, w, op_id, SW_ERR_INVALID_PARAM, tag, len);
    return true;
  }
  BulkJob j;
  j.w = w;
  j.recv_op = op_id;
  j.dst = (uint64_t)(uintptr_t)r->ptr;
  j.cap = r->cap;
  j.tag = tag;
  j.len = len;
  j.src = (uint64_t)(uintptr_t)r->landing;
  j.src_ready = true;
  j.dtype = r->dtype;
  j.t_enq = now_s();
  c->pending_bulk.push_back(j);
  return true;
}

bool poll_progress_rings(Ctx* c, Worker* w) {
  bool any = false;
  // ---- eager completions
  uint64_t h = w->cq_head;
  for (;;) {
    const SwCqEnt* e = &w->cq_ring[h % SW_CQ_RING];
    int32_t status;
    if (!cq_ready(e, h, &status)) break;
    trace(c, "cqe_eager", e->op_id, e->len);
    if (!reduce_landed(c, w, e->op_id, status, e->tag, e->len)) recv_finish(c, w, e->op_id, status, e->tag, e->len);
    h++;
  }
  if (h != w->cq_head) {
    w->cq_head = h;
    __atomic_store_n(&w->pctl->cq_head, h, __ATOMIC_RELEASE);
    any = true;
  }
  // ---- rendezvous completions of the pull CTAs (the sender's FIN word has been written by the same CTA)
  h = w->cqr_head;
  for (;;) {
    const SwCqEnt* e = &w->cqr_ring[h % SW_CQ_RING];
    int32_t status;
    if (!cq_ready(e, h, &status)) break;
    trace(c, "pull_done", e->op_id, e->len);
    recv_finish(c, w, e->op_id, status, e->tag, e->len);
    h++;
  }
  if (h != w->cqr_head) {
    w->cqr_head = h;
    __atomic_store_n(&w->pctl->cqr_head, h, __ATOMIC_RELEASE);
    any = true;
  }
  // ---- rendezvous matches the device left to the host (source not mapped yet, host-side or unaligned
  //      buffers, truncation, withdrawn senders)
  h = w->hr_head;
  for (;;) {
    const SwHrEnt* e = &w->hr_ring[h % SW_HR_RING];
    if (__atomic_load_n(&e->seq, __ATOMIC_ACQUIRE) != sw_ring_pass(h, SW_HR_RING)) break;
    const SwRndvRec& r = e->rec;
    BulkJob j;
    j.w = w;
    const uint32_t idx = r.ep & ((1u << SW_EP_IDX_BITS) - 1), gen = r.ep >> SW_EP_IDX_BITS;
    j.ep = idx < w->eps.size() ? w->eps[idx] : nullptr;
    j.recv_op = r.op_id;
    j.dst = r.dst;
    j.cap = r.cap;
    j.tag = r.tag;
    j.len = r.len;
    j.rts = r.rts;
    j.t_enq = now_s();
    {
      auto rit = w->recvs.find(r.op_id);
      j.src_host = (r.rts.pad[0] & SW_RTS_PINNED_SRC) != 0;
      j.host_side = j.src_host || (rit != w->recvs.end() && rit->second->mem == MEM_PINNED);
      if (rit != w->recvs.end() && rit->second->dtype) {
        j.dtype = rit->second->dtype;
        j.dst = (uint64_t)(uintptr_t)rit->second->ptr;   // reduced straight into the caller's buffer
      }
    }
    if (r.status != SW_OK) {
      j.failed = true;
      j.fail_status = r.status;
    } else if (j.dtype && r.len % sw_dtype_size(j.dtype)) {
      j.failed = true;
      j.fail_status = SW_ERR_INVALID_PARAM;
    }
    if (!j.ep || j.ep->retired || j.ep->ring_gen != gen) {
      // a request parked in the unexpected queue by a connection that has ended since: its source is gone
      j.ep = nullptr;
      j.failed = true;
      j.fail_status = SW_ERR_CONNECTION_RESET;
    }
    c->pending_bulk.push_back(j);
    h++;
  }
  if (h != w->hr_head) {
    w->hr_head = h;
    __atomic_store_n(&w->pctl->hr_head, h, __ATOMIC_RELEASE);
    any = true;
  }
  if (any) w->last_activity = now_s();
  return any;
}

bool pump_progress(Ctx* c, Worker* w) {
  if (!w->mstate || !w->pctl) return false;
  const int st = w->status.load(std::memory_order_acquire);
  if (st != SW_ST_RUNNING && st != SW_ST_CLOSING) return false;
  bool any = false;
  // ---- has the last launch ended?
  if (w->prog_running) {
    if (__atomic_load_n(&w->pctl->exit_seq, __ATOMIC_ACQUIRE) == w->prog_seq) {
      w->prog_running = false;
      trace(c, "prog_exit", w->prog_seq, w->pctl->arrivals);
      if (w->pctl->err) fprintf(stderr, "starway_b200: device matcher reported inconsistency 0x%llx\n", (unsigned long long)w->pctl->err);
      w->prog_stalled = w->pctl->stalled != 0;
      w->stall_posts = w->posts_written;
      w->stall_seen = unseen_arrivals(w);
      {
        const uint64_t arr = w->pctl->arrivals, why = w->pctl->exit_reason, life = w->pctl->life_us;
        std::lock_guard<std::mutex> lk(c->st_mu);
        c->stats.match_arrivals += arr - w->arrivals_seen;
        w->arrivals_seen = arr;
        (why == 1 ? c->stats.prog_exit_stop : why == 2 ? c->stats.prog_exit_idle : c->stats.prog_exit_life)++;
        c->stats.prog_life_ms += (double)life * 1e-3;
      }
      any = true;
    } else if ((++w->prog_spins & 0xFFF) == 0 && swgpu::stream_query(w->s_ctl) < 0) {
      fprintf(stderr, "starway_b200: control kernel failed: %s\n", swgpu::last_error());
      w->prog_running = false;
    }
  }
  any |= poll_progress_rings(c, w);
  // ---- new receives -> post ring
  uint32_t np = 0;
  if (w->close_phase == 0) {
    while (!w->new_posts.empty() && w->posts_written - __atomic_load_n(&w->pctl->post_head, __ATOMIC_ACQUIRE) < SW_POST_RING &&
           w->recvs.size() < SW_PQ_CAP / 2) {
      RecvOp* r = w->new_posts.front();
      uint64_t buf = (uint64_t)(uintptr_t)r->ptr;
      if (r->dtype && r->cap) {
        // reducing receive: an eager payload lands in a block of its own (reduce_landed), a rendezvous match takes the
        // host path (pump_bulk reduces the sender's buffer straight into the caller's)
        r->landing = c->landing.get();
        buf = (uint64_t)(uintptr_t)r->landing;
        if (!buf) {
          w->new_posts.pop_front();
          complete(c, w, r->op_id, SW_OP_RECV, SW_ERR_NO_MEMORY);
          delete r;
          continue;
        }
      }
      if (r->mem == SW_MEM_HOST && r->cap > HOST_BOUNCE_MAX) {
        swgpu::PtrInfo pi;
        swgpu::ptr_info(r->ptr, &pi);
        if (pi.is_pinned) r->mem = MEM_PINNED;  // a host-launched copy writes the caller's pinned buffer directly
      }
      if (r->mem == SW_MEM_HOST) {
        if (r->cap <= HOST_BOUNCE_MAX) {
          r->pinned_bounce = c->host_pool.get(r->cap);
          buf = (uint64_t)(uintptr_t)r->pinned_bounce;
        } else {
          r->dev_staging = c->staging.get(r->cap, &r->staging_size);
          buf = (uint64_t)(uintptr_t)r->dev_staging;
        }
        if (!buf) {
          w->new_posts.pop_front();
          complete(c, w, r->op_id, SW_OP_RECV, SW_ERR_NO_MEMORY);
          delete r;
          continue;
        }
      }
      SwPostEnt& p = w->post_ring[w->posts_written % SW_POST_RING];
      p.tag = r->tag;
      p.mask = r->mask;
      p.buf = buf;
      p.cap = r->cap;
      p.op_id = r->op_id;
      p.flags = r->mem == MEM_PINNED || r->dtype ? (uint32_t)SW_POST_HOSTPATH : 0u;
      if (r->pinned_bounce) p.flags |= SW_POST_HOSTBUF;
      p.pad = 0;
      if (!p.flags && r->cap > (uint64_t)c->opt_eager_max.load()) {
        r->rndv_capable = true;   // a rendezvous may land here: keep the pull CTAs of the context resident
        w->rndv_recvs++;
      }
      w->recvs[r->op_id] = r;
      w->new_posts.pop_front();
      w->posts_written++;
      np++;
    }
    if (np) {
      __atomic_store_n(&w->pctl->post_tail, w->posts_written, __ATOMIC_RELEASE);
      w->last_activity = now_s();
      std::lock_guard<std::mutex> lk(c->st_mu);
      c->stats.match_posts += np;
      any = true;
    }
  }
  if (w->prog_running) {
    if (w->cfg_dirty || w->close_phase >= 2) __atomic_store_n(&w->pctl->stop, 1, __ATOMIC_RELEASE);
    return any;
  }
  // ---- (re)launch?  Work: receives the kernel has not taken yet, or ring slots it has not consumed (host
  // doorbell of the peers).  Armed: receives are outstanding and the connection was active recently -- the
  // kernel then watches the rings itself and a message needs no doorbell, no launch.
  if (w->close_phase >= 3 || c->evict_pending) return any;
  const uint64_t unseen = unseen_arrivals(w);
  const bool posts_pending = w->posts_written != __atomic_load_n(&w->pctl->post_head, __ATOMIC_ACQUIRE);
  const bool sends_pending = w->sends_written != __atomic_load_n(&w->pctl->send_done, __ATOMIC_ACQUIRE);
  bool work = posts_pending || unseen != 0;
  if (w->prog_stalled && w->stall_posts == w->posts_written && w->stall_seen == unseen) work = false;
  work |= sends_pending;   // puts handed to a kernel that left before it took them
  const double now = now_s();
  if (w->last_send == 0) w->last_send = now;   // a send was queued since the last look
  // armed: receives are outstanding and the connection was active recently, or the worker has been sending within
  // the last millisecond (its next small batch of puts then needs no launch)
  const bool armed = swgpu::resident_lingers() && w->close_phase == 0 &&
                     ((!w->recvs.empty() && now - w->last_activity < (double)c->opt_armed_ms.load() * 1e-3) ||
                      (c->opt_resident_puts.load() > 0 && now - w->last_send < 1e-3));
  if (!work && !armed) return any;
  swgpu::ProgressLaunch a;
  a.st = w->mstate;
  a.ctl = w->pctl;
  a.posts = w->post_ring;
  a.cq = w->cq_ring;
  a.cqr = w->cqr_ring;
  a.hr = w->hr_ring;
  a.sends = w->send_ring;
  a.pq = c->pq;
  a.map = c->map_tbl;
  a.ctx_uuid = c->uuid;
  a.launch_seq = ++w->prog_seq;
  a.pid = (uint32_t)getpid();
  a.n_eps = (uint32_t)w->eps.size();
  a.linger_us = (uint32_t)c->opt_linger_us.load();
  a.max_life_us = (uint32_t)c->opt_max_life_us.load();
  a.pull_ctas = (uint32_t)c->opt_pull_ctas.load();
  __atomic_store_n(&w->pctl->stop, 0, __ATOMIC_RELEASE);
  w->cfg_dirty = false;
  trace(c, "prog_launch", w->prog_seq, unseen);
  if (swgpu::launch_progress(w->s_ctl, &a) != 0) {
    fprintf(stderr, "starway_b200: control kernel launch failed: %s\n", swgpu::last_error());
    w->prog_seq--;
    return any;
  }
  w->prog_running = true;
  w->prog_spins = 0;
  w->prog_launched_at = now;
  if (work) w->last_activity = now;
  std::lock_guard<std::mutex> lk(c->st_mu);
  c->stats.prog_launches++;
  return true;
}

// ---- the pull CTAs of the context: alive while device-side rendezvous copies are outstanding or expected
uint64_t pull_outstanding(Ctx* c) {
  uint64_t n = 0;
  for (Worker* w : c->active) {
    if (!w->pctl) continue;
    const uint64_t pub = __atomic_load_n(&w->pctl->pull_jobs, __ATOMIC_ACQUIRE);
    if (pub > w->cqr_head) n += pub - w->cqr_head;
  }
  return n;
}

void pull_collect_stats(Ctx* c) {
  if (!c->pull_ctl) return;
  const uint64_t bytes = c->pull_ctl->bytes, busy = c->pull_ctl->busy_ns, batches = c->pull_ctl->batches, jobs = c->pull_ctl->jobs;
  std::lock_guard<std::mutex> lk(c->st_mu);
  c->stats.pull_pickup_ms = (double)c->pull_ctl->pickup_ns * 1e-6;   // totals since the context was created
  c->stats.pull_copy_ms = (double)c->pull_ctl->copy_ns * 1e-6;
  c->stats.pull_fin_ms = (double)c->pull_ctl->fin_ns * 1e-6;
  c->stats.pull_bytes += bytes - c->pull_bytes_seen;
  c->stats.pull_busy_ms += (double)(busy - c->pull_busy_seen) * 1e-6;
  c->stats.pull_batches += batches - c->pull_batches_seen;
  c->stats.pull_jobs += jobs - c->pull_jobs_seen;
  c->pull_bytes_seen = bytes;
  c->pull_busy_seen = busy;
  c->pull_batches_seen = batches;
  c->pull_jobs_seen = jobs;
}

bool pump_pull(Ctx* c) {
  bool any = false;
  if (c->pull_running) {
    if (__atomic_load_n(&c->pull_ctl->exited, __ATOMIC_ACQUIRE) == c->pull_seq && swgpu::event_query(c->pull_ev) != 1) {
      c->pull_running = false;
      c->pull_stop_sent = false;
      pull_collect_stats(c);
      trace(c, "pull_exit", c->pull_seq);
      any = true;
    }
  }
  const uint64_t outstanding = pull_outstanding(c);
  bool expected = false;   // a running control kernel may hand over a rendezvous match at any moment
  for (Worker* w : c->active) expected |= w->prog_running && w->rndv_recvs > 0;
  const double now = now_s();
  if (outstanding || expected) c->pull_last_need = now;
  if (c->pull_running) {
    const bool flush = c->stats_flush.load(std::memory_order_acquire) != 0;
    // No need right now is not a reason to leave: the next receive of a ping-pong or of the next window is
    // posted a few microseconds later, and a relaunch (old kernel out, new one in: ~15 us) would be paid by
    // every such message.  The host asks the kernel to leave when nothing has needed it for pull_keep_us
    // (shorter than the control kernels' linger: a device-wide synchronisation after the last message waits
    // for those anyway), or when statistics are wanted now; the kernel's own linger is the backstop.
    const bool unneeded = !outstanding && !expected && now - c->pull_last_need > (double)c->opt_pull_keep_us.load() * 1e-6;
    if (!c->pull_stop_sent && (unneeded || flush)) {
      __atomic_store_n(&c->pull_ctl->stop, 1, __ATOMIC_RELEASE);
      c->pull_stop_sent = true;
    }
    return any;
  }
  if (c->stats_flush.load(std::memory_order_acquire)) c->stats_flush.store(0, std::memory_order_release);
  if (!outstanding && !(expected && swgpu::resident_lingers())) return any;
  swgpu::BulkTuning tune;
  tune.mode = 0;
  tune.stages = (int)c->opt_bulk_stages.load();
  tune.stage_bytes = (int)c->opt_bulk_stage_bytes.load();
  tune.ctas_per_sm = 1;
  tune.balance = 1;
  __atomic_store_n(&c->pull_ctl->stop, 0, __ATOMIC_RELEASE);
  c->pull_seq++;
  trace(c, "pull_launch", c->pull_seq, outstanding);
  if (swgpu::launch_pull(c->s_pull, c->pq, c->pull_ctl, c->pull_seq, (uint32_t)c->opt_pull_ctas.load(),
                         (uint32_t)c->opt_linger_us.load() * 2, (uint32_t)c->opt_max_life_us.load(), &tune) != 0) {
    fprintf(stderr, "starway_b200: pull kernel launch failed: %s\n", swgpu::last_error());
    c->pull_seq--;
    return any;
  }
  swgpu::event_record(c->pull_ev, c->s_pull);
  c->pull_running = true;
  c->pull_stop_sent = false;
  c->pull_launched_at = now;
  std::lock_guard<std::mutex> lk(c->st_mu);
  c->stats.pull_launches++;
  return true;
}

// ============================================================================ progress: control ring, flush, close
// End a rendezvous send that has left the queue.  While the put block that carried its RTS is still in flight
// the block refers to the record (poll_puts reads it): only note the outcome, poll_puts finishes it.
void rndv_end(Ctx* c, SendOp* op, int32_t status) {
  if (op->in_put) {
    op->ended_early = true;
    op->early_status = status;
    return;
  }
  send_finished(c, op, status);
}

void fail_ep_sends(Ctx* c, Ep* ep, int32_t status) {
  while (!ep->sendq.empty()) {
    SendOp* op = ep->sendq.front();
    ep->sendq.pop_front();
    send_finished(c, op, status);
  }
  for (auto& kv : ep->rndv_wait) rndv_end(c, kv.second, status);
  ep->rndv_wait.clear();
  ep->cancel_wait.clear();
}

// FIN words written by the receiver's pull CTAs (device stores into the page-locked control block)
bool poll_fin_words(Ctx* c, Ep* ep) {
  if (!ep->out || ep->rndv_wait.empty()) return false;
  bool any = false;
  int looked = 0;
  for (auto it = ep->rndv_wait.begin(); it != ep->rndv_wait.end() && looked < 64; looked++) {
    const uint64_t seq = it->first;
    const uint64_t v = ep->out->gfin[seq % SW_FIN_SLOTS].load(std::memory_order_acquire);
    if ((v >> 2) != seq) {
      ++it;
      continue;
    }
    trace(c, "fin_word", seq);
    SendOp* op = it->second;
    it = ep->rndv_wait.erase(it);
    ep->cancel_wait.erase(seq);
    rndv_end(c, op, (v & 3) == 1 ? SW_OK : SW_ERR_IO_ERROR);
    any = true;
  }
  return any;
}

bool poll_ctl(Ctx* c, Ep* ep) {
  if (!ep->shm) return false;
  ctl_flush_backlog(ep);
  ShmDir* d = ep->in;
  bool any = false;
  for (;;) {
    uint64_t tail = d->ctl_tail.load(std::memory_order_relaxed);
    uint64_t head = d->ctl_head.load(std::memory_order_acquire);
    if (tail == head) break;
    CtlMsg m = d->ctl[tail % CTL_RING];
    d->ctl_tail.store(tail + 1, std::memory_order_release);
    any = true;
    switch (m.type) {
      case CTL_FIN: {
        trace(c, "fin_recv", m.a);
        ep->cancel_wait.erase(m.a);
        auto it = ep->rndv_wait.find(m.a);
        if (it != ep->rndv_wait.end()) {
          SendOp* op = it->second;
          ep->rndv_wait.erase(it);
          rndv_end(c, op, m.status);
        }
        break;
      }
      case CTL_CANCEL_ACK:
        ep->cancel_wait.erase(m.a);
        break;
      case CTL_CANCEL_RTS: {
        // the sender is closing and withdraws rendezvous m.a
        // The control kernel may match (and the pull CTAs may copy) this request at any moment: raise the
        // endpoint's dead bit -- matches of its requests then come to the host -- and acknowledge once
        // the kernel has seen the bit and every pull it issued before that has completed
        // (progress_cancels).
        Worker* w = ep->owner;
        ep->cancel_quiesce.push_back(m.a);
        __atomic_store_n(&w->pctl->dead_mask, w->pctl->dead_mask | (1ull << (ep->index & 63)), __ATOMIC_RELEASE);
        __atomic_store_n(&w->pctl->host_epoch, ++w->host_epoch, __ATOMIC_RELEASE);
        ep->cancel_epoch = w->host_epoch;
        ep->cancel_pull_mark = ~0ull;
        break;
      }
      case CTL_CLOSE:
        ep->peer_closed = true;
        ep->close_ack_owed = true;
        fail_ep_sends(c, ep, SW_ERR_CONNECTION_RESET);
        break;
      case CTL_CLOSE_ACK:
        ep->close_acked = true;
        break;
      default:
        break;
    }
  }
  if (ep->close_ack_owed && ep->puts_inflight == 0) {
    // nothing of ours targets the peer's ring any more: it may free it
    ctl_send(ep, CTL_CLOSE_ACK, SW_OK, 0);
    ep->close_ack_owed = false;
  }
  return any;
}

// A connection whose peer has closed and whose traffic has drained gives its ring, control block and peer
// mapping back; the ring index is reused by a later connection (with a new generation).  The record itself
// stays listed (reference: list_clients never shrinks, tests/test_basic.py:53-56).
bool retire_eps(Ctx* c, Worker* w) {
  if (w->kind != SW_WORKER_SERVER || w->close_phase != 0) return false;
  bool any = false;
  for (Ep* ep : w->eps) {
    if (ep->retired || !ep->peer_closed || ep->close_ack_owed || !ep->shm) continue;
    if (!ep->ctl_backlog.empty() || !ep->sendq.empty() || !ep->rndv_wait.empty() || ep->puts_inflight) continue;
    if (!ep->cancel_quiesce.empty() || !ep->out_seqs.empty()) continue;
    if (ep->in->produced.load(std::memory_order_acquire) != ep->in->consumed.load(std::memory_order_acquire)) continue;
    bool busy = false;
    for (auto& j : c->pending_bulk) busy |= j.ep == ep;
    for (uint32_t k = c->bulk_head; k != c->bulk_tail; k++)
      for (BulkJob& j : c->bulk_blocks[k % N_BULK_BLOCKS].jobs) busy |= j.ep == ep;
    for (FlushOp* f : w->flushes) busy |= f->marks.count(ep) != 0;
    if (busy || pull_outstanding(c)) continue;
    if (w->prog_running) {   // the control kernel polls this ring: have it leave first
      w->cfg_dirty = true;
      continue;
    }
    swgpu::match_state_set_ring(w->mstate, ep->index, nullptr, 0, 0);
    swgpu::match_state_set_ep_words(w->mstate, ep->index, nullptr, nullptr);
    if (ep->peer_ring_mapping) swgpu::ipc_close(ep->peer_ring_mapping);
    ep->peer_ring_mapping = nullptr;
    ep->peer_ring = nullptr;
    if (ep->ring) swgpu::dev_free(ep->ring);   // the peer's CLOSE came after its last put had completed
    ep->ring = nullptr;
    shm_release(ep->shm);
    ep->shm = nullptr;
    ep->shm_dev = nullptr;
    ep->in = ep->out = nullptr;
    ep->retired = true;
    w->free_ring_idx.push_back(ep->index);
    trace(c, "ep_retired", ep->index);
    any = true;
  }
  return any;
}

// withdrawals wait until the device cannot touch the withdrawn sources any more
bool progress_cancels(Ctx* c, Worker* w) {
  bool any = false;
  for (Ep* ep : w->eps) {
    if (ep->cancel_quiesce.empty()) continue;
    const bool seen = !w->prog_running || __atomic_load_n(&w->pctl->dev_epoch, __ATOMIC_ACQUIRE) >= ep->cancel_epoch;
    if (!seen) continue;
    if (ep->cancel_pull_mark == ~0ull) ep->cancel_pull_mark = __atomic_load_n(&w->pctl->pull_jobs, __ATOMIC_ACQUIRE);
    if (w->cqr_head < ep->cancel_pull_mark) continue;   // pulls issued before the dead bit was seen: still copying
    for (uint64_t seq : ep->cancel_quiesce) {
      bool in_flight = false;
      for (uint32_t k = c->bulk_head; k != c->bulk_tail; k++)
        for (BulkJob& j : c->bulk_blocks[k % N_BULK_BLOCKS].jobs)
          if (j.ep == ep && j.rts.send_seq == seq) in_flight = true;
      if (in_flight) continue;   // the FIN of the running host-launched pull acknowledges it
      ep->canceled_rts.insert(seq);
      ctl_send(ep, CTL_CANCEL_ACK, SW_OK, seq);
    }
    ep->cancel_quiesce.clear();
    any = true;
  }
  return any;
}

void check_flushes(Ctx* c, Worker* w) {
  for (size_t i = 0; i < w->flushes.size();) {
    FlushOp* f = w->flushes[i];
    bool done = true;
    for (auto& kv : f->marks) {
      Ep* ep = kv.first;
      if (!ep->out_seqs.empty() && *ep->out_seqs.begin() < kv.second) {
        done = false;
        break;
      }
    }
    if (done) {
      complete(c, w, f->op_id, f->ep ? SW_OP_FLUSH_EP : SW_OP_FLUSH, SW_OK);
      delete f;
      w->flushes.erase(w->flushes.begin() + (long)i);
    } else {
      i++;
    }
  }
}

void worker_release(Ctx* c, Worker* w, bool leak_rings) {
  if (c->tracing && w->pctl && w->pctl->dbg[0]) {
    const double mhz = (double)swgpu::clock_mhz(), n = (double)w->pctl->dbg[0];
    fprintf(stderr, "starway_b200 resident puts (worker %llx): %llu; seen->staged %.2f us, staged->released %.2f us, released->published %.2f us; link round %.2f us\n",
            (unsigned long long)w->id, (unsigned long long)w->pctl->dbg[0], w->pctl->dbg[1] / n / mhz, w->pctl->dbg[2] / n / mhz,
            w->pctl->dbg[3] / n / mhz, w->pctl->dbg[4] ? w->pctl->dbg[5] / (double)w->pctl->dbg[4] / mhz : 0.0);
  }
  for (Ep* ep : w->eps) {
    if (ep->retired) continue;
    if (ep->peer_ring_mapping) {
      swgpu::ipc_close(ep->peer_ring_mapping);
      ep->peer_ring_mapping = nullptr;
    }
    ep->peer_ring = nullptr;
    bool safe = ep->close_acked || ep->in_process || !pid_alive(ep->peer_pid) || !leak_rings;
    if (ep->ring && safe) swgpu::dev_free(ep->ring);
    ep->ring = nullptr;
    if (ep->shm) {
      shm_release(ep->shm);
      ep->shm = nullptr;
      ep->shm_dev = nullptr;
      ep->in = ep->out = nullptr;
    }
  }
  if (w->mstate) {
    swgpu::match_state_destroy(w->mstate);
    w->mstate = nullptr;
  }
  if (w->s_ctl) {
    swgpu::stream_sync(w->s_ctl);
    swgpu::stream_destroy(w->s_ctl);
  }
  swgpu::host_free(w->pctl);
  swgpu::host_free(w->post_ring);
  swgpu::host_free(w->cq_ring);
  swgpu::host_free(w->cqr_ring);
  swgpu::host_free(w->hr_ring);
  swgpu::host_free(w->send_ring);
  w->send_ring = nullptr;
  w->s_ctl = nullptr;
  w->pctl = nullptr;
  w->post_ring = nullptr;
  w->cq_ring = w->cqr_ring = nullptr;
  w->hr_ring = nullptr;
  if (w->tcp_fd >= 0) close(w->tcp_fd);
  if (w->unix_fd >= 0) close(w->unix_fd);
  w->tcp_fd = w->unix_fd = -1;
  for (auto& ph : w->pending_hello) close(ph.fd);
  w->pending_hello.clear();
}

// reference shutdown sequence: main.cpp:469-550 (client), 1269-1373 (server)
bool progress_close(Ctx* c, Worker* w) {
  if (w->close_phase == 0) return false;
  if (w->close_phase == 1) {
    // ---- cancel everything that has not reached the device / the wire
    while (!w->new_posts.empty()) {
      RecvOp* r = w->new_posts.front();
      w->new_posts.pop_front();
      complete(c, w, r->op_id, SW_OP_RECV, SW_ERR_CANCELED);
      delete r;
    }
    for (FlushOp* f : w->flushes) {
      complete(c, w, f->op_id, f->ep ? SW_OP_FLUSH_EP : SW_OP_FLUSH, SW_ERR_CANCELED);
      delete f;
    }
    w->flushes.clear();
    for (Ep* ep : w->eps) {
      while (!ep->sendq.empty()) {
        SendOp* op = ep->sendq.front();
        ep->sendq.pop_front();
        send_finished(c, op, SW_ERR_CANCELED);
      }
      // withdraw unmatched rendezvous sends; their buffers stay valid until the peer acknowledges
      for (auto& kv : ep->rndv_wait) {
        if (!ep->peer_closed) {
          ctl_send(ep, CTL_CANCEL_RTS, SW_OK, kv.first);
          ep->cancel_wait.insert(kv.first);
        }
      }
    }
    w->close_phase = 2;
    w->close_deadline = now_s() + 3.0;
    return true;
  }
  if (w->close_phase == 2) {
    // ---- wait for in-flight device work and for the cancel acknowledgements
    bool busy = w->bulk_inflight > 0;
    if (w->pctl) {
      // the control kernel is asked to leave (pump_progress raises `stop` from phase 2 on); rendezvous copies
      // it handed to the pull CTAs run to completion -- they write into receive buffers of this worker
      busy |= w->prog_running;
      busy |= __atomic_load_n(&w->pctl->pull_jobs, __ATOMIC_ACQUIRE) > w->cqr_head;
    }
    for (Ep* ep : w->eps) {
      if (ep->puts_inflight) busy = true;
      if (!ep->cancel_quiesce.empty()) busy = true;   // withdrawals of our peers that we still have to acknowledge
      if (!ep->cancel_wait.empty() && !ep->peer_closed && pid_alive(ep->peer_pid) && now_s() < w->close_deadline)
        busy = true;
    }
    for (auto& j : c->pending_bulk)
      if (j.w == w) busy = true;
    for (auto& pc : c->post_copies)
      if (pc.op->w == w) busy = true;
    if (busy) return false;
    for (Ep* ep : w->eps) {
      for (auto& kv : ep->rndv_wait) rndv_end(c, kv.second, SW_ERR_CANCELED);
      ep->rndv_wait.clear();
      ep->cancel_wait.clear();
    }
    // pending receives fail with "Request canceled" (reference main.cpp:498-502)
    std::vector<uint64_t> ids;
    for (auto& kv : w->recvs) ids.push_back(kv.first);
    for (uint64_t id : ids) recv_finish(c, w, id, SW_ERR_CANCELED, 0, 0);
    for (Ep* ep : w->eps) {
      if (!ep->peer_closed && ep->shm) {
        ctl_send(ep, CTL_CLOSE, SW_OK, 0);
        ep->close_sent = true;
      }
    }
    w->close_phase = 3;
    w->close_deadline = now_s() + 2.0;
    return true;
  }
  if (w->close_phase == 3) {
    // ---- wait until no peer can still be writing into our rings
    bool waiting = false;
    for (Ep* ep : w->eps) {
      ctl_flush_backlog(ep);
      if (ep->close_sent && !ep->close_acked && pid_alive(ep->peer_pid) && now_s() < w->close_deadline) waiting = true;
      if (ep->close_ack_owed || !ep->ctl_backlog.empty()) {
        if (now_s() < w->close_deadline) waiting = true;
      }
    }
    if (waiting) return false;
    worker_release(c, w, true);
    w->close_phase = 4;
    c->need_prune = true;
    w->status.store(SW_ST_CLOSED, std::memory_order_release);
    if (w->close_op) complete(c, w, w->close_op, SW_OP_CLOSE, SW_OK);
    return true;
  }
  return false;
}

// ============================================================================ progress thread
void drain_sq(Ctx* c) {
  if (c->sq_head.load(std::memory_order_acquire) == nullptr) return;
  SqNode* list = c->sq_head.exchange(nullptr, std::memory_order_acquire);
  trace(c, "sq_drain");
  // the stack is LIFO: reverse it to recover submission order
  SqNode* rev = nullptr;
  while (list) {
    SqNode* nx = list->next;
    list->next = rev;
    rev = list;
    list = nx;
  }
  struct Item {
    int kind;
    Worker* w;
    void* p;
  };
  while (rev) {
    SqNode* node = rev;
    rev = rev->next;
    Item it{node->kind, node->w, node->p};  // the op that embeds `node` may be freed below
    if (node->heap) delete node;
    Worker* w = it.w;
    switch (it.kind) {
      case SQ_REGISTER: {
        if (!w->registered) {
          c->active.push_back(w);
          w->registered = true;
        }
        if (w->kind == SW_WORKER_CLIENT) {
          w->status.store(SW_ST_RUNNING, std::memory_order_release);
          complete(c, w, (uint64_t)(uintptr_t)it.p, SW_OP_CONNECT, SW_OK);
        }
        break;
      }
      case SQ_SEND: {
        SendOp* op = (SendOp*)it.p;
        int st = w->status.load(std::memory_order_acquire);
        if (st != SW_ST_RUNNING || w->close_phase != 0) {
          // The op was accepted while the worker was running and close overtook it in the queue:
          // like a mailbox-resident op in the reference it is cancelled (main.cpp:680-701).  Ops
          // posted after close began are refused synchronously by sw_post_* (reference: RuntimeError).
          complete(c, w, op->op_id, SW_OP_SEND, SW_ERR_CANCELED);
          delete op;
          break;
        }
        op->sseq = op->ep->next_sseq++;
        op->ep->out_seqs.insert(op->sseq);
        op->ep->sendq.push_back(op);
        w->last_send = 0;   // stamped by pump_progress (one clock read per loop, not per op)
        break;
      }
      case SQ_RECV: {
        RecvOp* r = (RecvOp*)it.p;
        int st = w->status.load(std::memory_order_acquire);
        if (st != SW_ST_RUNNING || w->close_phase != 0) {
          complete(c, w, r->op_id, SW_OP_RECV, SW_ERR_CANCELED);
          delete r;
          break;
        }
        w->new_posts.push_back(r);
        break;
      }
      case SQ_FLUSH: {
        FlushOp* f = (FlushOp*)it.p;
        int st = w->status.load(std::memory_order_acquire);
        if (st != SW_ST_RUNNING || w->close_phase != 0) {
          complete(c, w, f->op_id, f->ep ? SW_OP_FLUSH_EP : SW_OP_FLUSH, SW_ERR_CANCELED);
          delete f;
          break;
        }
        if (f->ep)
          f->marks[f->ep] = f->ep->next_sseq;
        else
          for (Ep* ep : w->eps) f->marks[ep] = ep->next_sseq;
        w->flushes.push_back(f);
        break;
      }
      case SQ_CLOSE: {
        w->close_op = (uint64_t)(uintptr_t)it.p;
        if (w->close_phase == 0) w->close_phase = 1;
        if (!w->registered) {
          c->active.push_back(w);
          w->registered = true;
        }
        break;
      }
      default:
        break;
    }
  }
}

// ============================================================================ NUMA placement
// GPU-local CPUs from sysfs (what `nvidia-smi topo -m` prints as CPU affinity).  Pinned control
// blocks and staging buffers are allocated, and the progress thread runs, next to the GPU's PCIe
// root: on a 2-socket host a rank whose host memory sits on the other socket moves its
// host<->device traffic over the inter-socket link.
std::string device_cpulist(int device) {
  char bus[64];
  if (swgpu::device_pci_bus_id(device, bus, sizeof bus) != 0) return "";
  std::string path = std::string("/sys/bus/pci/devices/") + bus + "/local_cpulist";
  FILE* f = fopen(path.c_str(), "r");
  if (!f) return "";
  char line[1024];
  std::string out;
  if (fgets(line, sizeof line, f)) out = line;
  fclose(f);
  while (!out.empty() && (out.back() == '\n' || out.back() == ' ')) out.pop_back();
  return out;
}

bool parse_cpulist(const std::string& s, cpu_set_t* set) {
  CPU_ZERO(set);
  int n = 0;
  size_t i = 0;
  while (i < s.size()) {
    char* end = nullptr;
    long a = strtol(s.c_str() + i, &end, 10);
    if (end == s.c_str() + i) return false;
    long b = a;
    i = (size_t)(end - s.c_str());
    if (i < s.size() && s[i] == '-') {
      b = strtol(s.c_str() + i + 1, &end, 10);
      i = (size_t)(end - s.c_str());
    }
    for (long k = a; k <= b && k < CPU_SETSIZE; k++) {
      CPU_SET((int)k, set);
      n++;
    }
    if (i < s.size() && s[i] == ',') i++;
  }
  return n > 0;
}

// GPU-local CPUs that this process is allowed to run on; false when there is nothing to do
bool device_cpuset(int device, cpu_set_t* out) {
  if (const char* e = getenv("STARWAY_AFFINITY"))
    if (atoi(e) == 0) return false;
  cpu_set_t local, allowed;
  if (!parse_cpulist(device_cpulist(device), &local)) return false;
  if (sched_getaffinity(0, sizeof allowed, &allowed) != 0) return false;
  CPU_AND(out, &local, &allowed);
  return CPU_COUNT(out) > 0 && !CPU_EQUAL(out, &allowed);
}

// binds the calling thread to the GPU-local CPUs for the lifetime of the object (allocations made
// meanwhile are first-touched on that node)
struct ScopedAffinity {
  cpu_set_t saved;
  bool active = false;
  explicit ScopedAffinity(int device) {
    cpu_set_t want;
    if (!device_cpuset(device, &want)) return;
    if (pthread_getaffinity_np(pthread_self(), sizeof saved, &saved) != 0) return;
    active = pthread_setaffinity_np(pthread_self(), sizeof want, &want) == 0;
  }
  ~ScopedAffinity() {
    if (active) pthread_setaffinity_np(pthread_self(), sizeof saved, &saved);
  }
};

void progress_main(Ctx* c) {
  swgpu::bind_thread(c->device);
  {
    cpu_set_t want;
    if (device_cpuset(c->device, &want)) pthread_setaffinity_np(pthread_self(), sizeof want, &want);
  }
  prctl(PR_SET_TIMERSLACK, 1000UL, 0, 0, 0);  // 1 us timer slack: short sleeps stay short
  tls_is_progress = true;
  uint64_t iter = 0;
  double last_active = now_s(), last_event = last_active;
  while (!c->stop.load(std::memory_order_acquire)) {
    bool active = false;
    drain_sq(c);
    active |= poll_puts(c);
    active |= pump_sends(c);
    for (Worker* w : c->active) {
      if (w->close_phase >= 4) continue;
      for (Ep* ep : w->eps) {
        active |= poll_ctl(c, ep);
        active |= poll_fin_words(c, ep);
      }
      active |= pump_progress(c, w);
      active |= progress_cancels(c, w);
      if ((iter & 255) == 0) active |= retire_eps(c, w);
      check_flushes(c, w);
      active |= progress_close(c, w);
      if ((iter & 31) == 0 && w->kind == SW_WORKER_SERVER) poll_listeners(c, w);
    }
    active |= poll_bulk(c);
    active |= pump_bulk(c);
    active |= pump_pull(c);
    flush_completions(c);
    // forget fully closed workers; `retired` tells sw_worker_destroy that this thread holds no
    // reference any more and the record may be recycled
    if (c->need_prune) {
      c->need_prune = false;
      auto dead = std::stable_partition(c->active.begin(), c->active.end(), [](Worker* w) { return w->close_phase < 4; });
      for (auto it = dead; it != c->active.end(); ++it) (*it)->retired.store(true, std::memory_order_release);
      c->active.erase(dead, c->active.end());
    }
    iter++;
    bool inflight = (c->put_head != c->put_tail) || (c->bulk_head != c->bulk_tail) || !c->post_copies.empty();
    bool resident_only = !inflight;   // nothing but resident kernels on the device
    inflight |= c->pull_running;
    bool expecting = false;  // operations whose completion depends on a peer's doorbell / FIN
    for (Worker* w : c->active) {
      inflight |= w->prog_running;
      if (w->close_phase >= 4) continue;
      expecting |= !w->recvs.empty() || !w->flushes.empty() || w->close_phase != 0;
      for (Ep* ep : w->eps) expecting |= !ep->rndv_wait.empty() || !ep->sendq.empty();
    }
    if (active) last_event = now_s();
    if (active || inflight) {
      last_active = now_s();
      if (!active) {
        for (int k = 0; k < 8; k++) __builtin_ia32_pause();  // polling device events: yield the core's pipeline
        // Only resident kernels are out and nothing has happened for a while: they may stay for milliseconds
        // waiting for a peer.  Keep polling their rings, but let other runnable threads (the Python thread of
        // this rank, other ranks of a crowded host) have the CPU between looks.
        if (resident_only && c->opt_yield_us.load(std::memory_order_relaxed) > 0 &&
            last_active - last_event > (double)c->opt_yield_us.load(std::memory_order_relaxed) * 1e-6)
          sched_yield();
      }
    } else {
      // The reference's worker threads spin at 100 % (main.cpp:361, 1126).  Here: spin while work is
      // outstanding or was seen recently, then back off progressively.
      double idle = now_s() - last_active;
      // be a polite hyper-thread sibling: the Python thread of this rank may share the core
      for (int k = 0; k < 32; k++) __builtin_ia32_pause();
      if (expecting && idle < 0.25) {
        if (idle > 0.002) sched_yield();
      } else if (idle > 0.02) {
        // nap: 30 us, 300 us after a second of silence.  Remote doorbells are only seen when the nap
        // ends; a local submission ends it at once (sq_push -> futex wake).
        struct timespec ts = {0, idle > 1.0 ? 300000 : 30000};
        c->sleeping.store(1, std::memory_order_seq_cst);
        if (c->sq_head.load(std::memory_order_seq_cst) == nullptr)
          syscall(SYS_futex, reinterpret_cast<int*>(&c->sleeping), FUTEX_WAIT_PRIVATE, 1, &ts, nullptr, 0);
        c->sleeping.store(0, std::memory_order_seq_cst);
      } else if (idle > 0.002) {
        sched_yield();
      }
    }
  }
  flush_completions(c);
}

Worker* find_worker(Ctx* c, sw_worker_t id) {
  Worker* w = (Worker*)(uintptr_t)(id & HANDLE_PTR_MASK);
  return (w && w->magic == WORKER_MAGIC && w->gen == (uint32_t)(id >> 48) && w->ctx == c) ? w : nullptr;
}
Ep* find_ep(Ctx* c, sw_ep_t id) {
  Ep* ep = (Ep*)(uintptr_t)(id & HANDLE_PTR_MASK);
  return (ep && ep->magic == EP_MAGIC && ep->gen == (uint32_t)(id >> 48) && ep->owner && ep->owner->ctx == c) ? ep
                                                                                                              : nullptr;
}

// returns the records of a closed worker and of its endpoints to their slabs (caller: no other
// thread references them any more)
void recycle_worker(Ctx* c, Worker* w) {
  if (w->connector.joinable()) w->connector.join();
  {
    std::lock_guard<std::mutex> lk(c->mu);
    c->workers.erase(w->id);
    for (Ep* ep : w->eps) c->eps.erase(ep->id);
    for (Ep* ep : w->tombs) c->eps.erase(ep->id);
  }
  for (Ep* ep : w->eps) Slab<Ep>::recycle(ep);
  for (Ep* ep : w->tombs) Slab<Ep>::recycle(ep);
  w->eps.clear();
  w->tombs.clear();
  Slab<Worker>::recycle(w);
}

int classify_mem(const void* ptr, int mem_kind) {
  if (mem_kind == SW_MEM_HOST || mem_kind == SW_MEM_DEVICE) return mem_kind;
  swgpu::PtrInfo pi;
  swgpu::ptr_info(ptr, &pi);
  return pi.is_device ? SW_MEM_DEVICE : SW_MEM_HOST;
}

}  // namespace

// ================================================================================== C ABI
extern "C" {

int sw_abi_version(void) { return SW_ABI_VERSION; }
const char* sw_backend_name(void) { return swgpu::backend_name(); }
const char* sw_last_error(void) { return g_last_error.c_str(); }
int sw_device_count(void) { return swgpu::device_count(); }

const char* sw_status_string(int32_t status) {
  switch (status) {
    case SW_STATUS_OK: return "Success";
    case SW_STATUS_IO_ERROR: return "Input/output error";
    case SW_STATUS_NO_MEMORY: return "Out of memory";
    case SW_STATUS_INVALID_PARAM: return "Invalid parameter";
    case SW_STATUS_UNREACHABLE: return "Destination is unreachable";
    case SW_STATUS_MESSAGE_TRUNCATED: return "Message truncated";
    case SW_STATUS_BUSY: return "Device is busy";
    case SW_STATUS_CANCELED: return "Request canceled";
    case SW_STATUS_TIMED_OUT: return "Operation timed out";
    case SW_STATUS_NOT_CONNECTED: return "Endpoint is not connected";
    case SW_STATUS_CONNECTION_RESET: return "Connection reset by remote peer";
    default: return "Unknown error";
  }
}

sw_ctx* sw_ctx_create(int device) {
  if (swgpu::init(device) != 0) {
    set_error(std::string("sw_ctx_create: ") + swgpu::last_error());
    return nullptr;
  }
  ScopedAffinity numa(device);
  Ctx* c = new Ctx();
  c->device = device;
  c->uuid = rand64() | 1;
  memset(&c->stats, 0, sizeof(c->stats));
  c->efd = eventfd(0, EFD_NONBLOCK | EFD_CLOEXEC);
  c->s_put = swgpu::stream_create();
  c->s_bulk = swgpu::stream_create();
  bool ok = c->s_put && c->s_bulk;
  for (int i = 0; ok && i < N_PUT_BLOCKS; i++) {
    PutBlock& b = c->put_blocks[i];
    b.descs = (SwPutDesc*)swgpu::host_alloc(sizeof(SwPutDesc) * PUT_BATCH);
    b.rts = (SwRts*)swgpu::host_alloc(sizeof(SwRts) * PUT_BATCH);
    b.stage = (uint8_t*)swgpu::host_alloc((size_t)PUT_BATCH * SW_SLOT_BYTES);
    b.segs = (SwSeg*)swgpu::host_alloc(sizeof(SwSeg) * STAGE_SEGS);
    b.ev = swgpu::event_create(1);
    b.ev_start = swgpu::event_create(1);
    b.ev_fast = swgpu::event_create(0);
    b.done = (uint64_t*)swgpu::host_alloc(64);
    if (b.done) *b.done = 0;
    b.s = i == 0 ? c->s_put : swgpu::stream_create();
    ok = b.descs && b.rts && b.stage && b.segs && b.ev && b.ev_start && b.ev_fast && b.done && b.s;
  }
  for (int i = 0; ok && i < N_BULK_BLOCKS; i++) {
    BulkBlock& b = c->bulk_blocks[i];
    b.segs = (SwSeg*)swgpu::host_alloc(sizeof(SwSeg) * MAX_SEGS);
    b.ev = swgpu::event_create(1);
    b.ev_start = swgpu::event_create(1);
    b.ev_fast = swgpu::event_create(0);
    ok = b.segs && b.ev && b.ev_start && b.ev_fast;
  }
  if (!ok) {
    set_error(std::string("sw_ctx_create: ") + swgpu::last_error());
    delete c;
    return nullptr;
  }
  // ---- resident path: pull queue, mapping table.  The control kernels publish credits and FIN words through
  // page-locked aliases of the connections' shared control blocks: check once that such mappings can be locked.
  {
    void* probe = mmap(nullptr, 4096, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
    bool can_lock = false;
    if (probe != MAP_FAILED) {
      can_lock = swgpu::host_register(probe, 4096) != nullptr;
      if (can_lock) swgpu::host_unregister(probe);
      munmap(probe, 4096);
    }
    if (!can_lock) {
      set_error(std::string("sw_ctx_create: cannot page-lock shared host mappings: ") + swgpu::last_error());
      delete c;
      return nullptr;
    }
  }
  c->pq = swgpu::pull_queue_create();
  c->map_tbl = swgpu::map_table_create();
  c->pull_ctl = (SwPullCtl*)swgpu::host_alloc(sizeof(SwPullCtl));
  c->s_pull = swgpu::stream_create();
  c->s_map = swgpu::stream_create();
  c->pull_ev = swgpu::event_create(0);
  c->opt_pull_ctas = swgpu::pull_default_ctas();
  if (!c->pq || !c->map_tbl || !c->pull_ctl || !c->s_pull || !c->s_map || !c->pull_ev) {
    set_error(std::string("sw_ctx_create (resident path): ") + swgpu::last_error());
    delete c;
    return nullptr;
  }
  if (const char* e = getenv("STARWAY_COPY_THREADS")) c->opt_copy_threads = std::max<int64_t>(0, atoll(e));
  {
    // helper threads for pageable buffers sit next to the GPU like the progress thread (ScopedAffinity above)
    int n = (int)c->opt_copy_threads.load();
    const int hw = (int)std::thread::hardware_concurrency();
    if (hw > 0 && n > hw / 4) n = std::max(hw >= 4 ? 1 : 0, hw / 4);
    if (n > 0) c->copy_pool.start(n, device);
  }
  if (const char* e = getenv("STARWAY_LINGER_US")) c->opt_linger_us = std::max<int64_t>(1, atoll(e));
  if (const char* e = getenv("STARWAY_MAX_LIFE_US")) c->opt_max_life_us = std::max<int64_t>(10, atoll(e));
  if (const char* e = getenv("STARWAY_ARMED_MS")) c->opt_armed_ms = std::max<int64_t>(0, atoll(e));
  if (const char* e = getenv("STARWAY_PULL_CTAS")) {
    if (atoll(e) == 1)
      fprintf(stderr, "starway_b200: STARWAY_PULL_CTAS=1 ignored: %s\n", kPullCtasOne);
    else
      c->opt_pull_ctas = std::max<int64_t>(0, atoll(e));
  }
  // environment knobs
  if (const char* e = getenv("STARWAY_EAGER_MAX")) c->opt_eager_max = std::min<int64_t>(atoll(e), SW_EAGER_MAX);
  if (const char* e = getenv("STARWAY_RING_SLOTS")) c->opt_ring_slots = std::max<int64_t>(atoll(e), 4);
  if (const char* e = getenv("STARWAY_BULK_MODE")) c->opt_bulk_mode = atoll(e);
  if (const char* e = getenv("STARWAY_BULK_STAGES")) c->opt_bulk_stages = atoll(e);
  if (const char* e = getenv("STARWAY_BULK_STAGE_BYTES")) c->opt_bulk_stage_bytes = atoll(e);
  if (const char* e = getenv("STARWAY_BULK_CTAS")) c->opt_bulk_ctas = atoll(e);
  if (const char* e = getenv("STARWAY_BULK_BALANCE")) c->opt_bulk_balance = atoll(e);
  if (const char* e = getenv("STARWAY_PINNED_SEND_DIRECT")) c->opt_pinned_send_direct = atoll(e);
  if (const char* e = getenv("STARWAY_HOSTDST_TMA")) c->opt_hostdst_tma = atoll(e);
  if (const char* e = getenv("STARWAY_PULL_KEEP_US")) c->opt_pull_keep_us = std::max<int64_t>(0, atoll(e));
  if (const char* e = getenv("STARWAY_OPTS")) {   // "key=value,key=value": any sw_set_option key
    std::string all(e);
    size_t pos = 0;
    while (pos < all.size()) {
      size_t end = all.find(',', pos);
      if (end == std::string::npos) end = all.size();
      const std::string kv = all.substr(pos, end - pos);
      const size_t eq = kv.find('=');
      if (eq != std::string::npos && sw_set_option((sw_ctx*)c, kv.substr(0, eq).c_str(), atoll(kv.c_str() + eq + 1)) != 0)
        fprintf(stderr, "starway_b200: STARWAY_OPTS: '%s' ignored: unknown option or invalid value\n", kv.c_str());
      pos = end + 1;
    }
  }
  if (const char* e = getenv("STARWAY_TRACE")) {
    c->trace_path = std::string(e) + "." + std::to_string((int)getpid());
    c->tracing = true;
    c->trace.reserve(1u << 20);
  }
  c->thr = std::thread(progress_main, c);
  std::lock_guard<std::mutex> lk(g_ctx_mu);
  g_ctxs.push_back(c);
  return (sw_ctx*)c;
}

int sw_ctx_device(sw_ctx* ctx) { return ((Ctx*)ctx)->device; }

int sw_device_local_cpus(int device, char* out, size_t cap) {
  if (swgpu::init(device) != 0) {
    set_error(std::string("sw_device_local_cpus: ") + swgpu::last_error());
    return -1;
  }
  std::string s = device_cpulist(device);
  if (s.empty() || s.size() + 1 > cap) return -1;
  memcpy(out, s.c_str(), s.size() + 1);
  return (int)s.size();
}

void sw_ctx_destroy(sw_ctx* ctx) {
  Ctx* c = (Ctx*)ctx;
  if (!c) return;
  // close every running worker first (reference ~Client/~Server force status 3 and join)
  std::vector<Worker*> ws;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    for (auto& kv : c->workers) ws.push_back(kv.second);
  }
  for (Worker* w : ws) sw_worker_destroy(ctx, w->id);
  c->stop.store(true, std::memory_order_release);
  if (c->thr.joinable()) c->thr.join();
  // whatever sw_worker_destroy could not recycle (still closing when it gave up) goes now
  ws.clear();
  {
    std::lock_guard<std::mutex> lk(c->mu);
    for (auto& kv : c->workers) ws.push_back(kv.second);
    c->workers.clear();
    c->eps.clear();
  }
  if (c->tracing) {
    if (FILE* f = fopen(c->trace_path.c_str(), "w")) {
      for (auto& r : c->trace) fprintf(f, "%.7f %s %llu %llu\n", r.t, r.what, (unsigned long long)r.a, (unsigned long long)r.b);
      fclose(f);
    }
  }
  swgpu::bind_thread(c->device);
  for (int i = 0; i < N_PUT_BLOCKS; i++) {
    PutBlock& b = c->put_blocks[i];
    swgpu::host_free(b.descs);
    swgpu::host_free(b.rts);
    swgpu::host_free(b.stage);
    swgpu::host_free(b.segs);
    swgpu::host_free(b.done);
    if (i > 0 && b.s) swgpu::stream_destroy(b.s);
    if (b.ev) swgpu::event_destroy(b.ev);
    if (b.ev_start) swgpu::event_destroy(b.ev_start);
    if (b.ev_fast) swgpu::event_destroy(b.ev_fast);
  }
  for (int i = 0; i < N_BULK_BLOCKS; i++) {
    BulkBlock& b = c->bulk_blocks[i];
    swgpu::host_free(b.segs);
    if (b.ev_fast) swgpu::event_destroy(b.ev_fast);
    if (b.ev) swgpu::event_destroy(b.ev);
    if (b.ev_start) swgpu::event_destroy(b.ev_start);
  }
  for (auto& kv : c->mappings) swgpu::ipc_close(kv.second.base);
  if (c->s_pull) {
    // the pull CTAs leave on their own (silence / lifetime); a stop request makes it quick
    if (c->pull_ctl) __atomic_store_n(&c->pull_ctl->stop, 1, __ATOMIC_RELEASE);
    swgpu::stream_sync(c->s_pull);
    swgpu::stream_destroy(c->s_pull);
  }
  if (c->s_map) {
    swgpu::stream_sync(c->s_map);
    swgpu::stream_destroy(c->s_map);
  }
  if (c->pull_ev) swgpu::event_destroy(c->pull_ev);
  if (c->pq) swgpu::pull_queue_destroy(c->pq);
  if (c->map_tbl) swgpu::map_table_destroy(c->map_tbl);
  swgpu::host_free(c->pull_ctl);
  c->copy_pool.shutdown();
  c->pinned_pool.destroy();
  c->host_pool.destroy();
  c->staging.destroy();
  c->landing.destroy();
  swgpu::stream_destroy(c->s_put);
  swgpu::stream_destroy(c->s_bulk);
  if (c->efd >= 0) close(c->efd);
  {
    std::lock_guard<std::mutex> lk(g_ctx_mu);
    g_ctxs.erase(std::remove(g_ctxs.begin(), g_ctxs.end(), c), g_ctxs.end());
  }
  for (Worker* w : ws) {
    if (w->connector.joinable()) w->connector.join();
    for (Ep* ep : w->eps) Slab<Ep>::recycle(ep);
    for (Ep* ep : w->tombs) Slab<Ep>::recycle(ep);
    w->eps.clear();
    w->tombs.clear();
    Slab<Worker>::recycle(w);
  }
  delete c;
}

int sw_set_option(sw_ctx* ctx, const char* key, int64_t value) {
  Ctx* c = (Ctx*)ctx;
  std::string k(key);
  if (k == "eager_max") c->opt_eager_max = std::max<int64_t>(0, std::min<int64_t>(value, SW_EAGER_MAX));
  else if (k == "ring_slots") c->opt_ring_slots = std::max<int64_t>(4, value);
  else if (k == "bulk_mode") c->opt_bulk_mode = value;
  else if (k == "bulk_stages") c->opt_bulk_stages = value;
  else if (k == "bulk_stage_bytes") c->opt_bulk_stage_bytes = value;
  else if (k == "bulk_ctas_per_sm") c->opt_bulk_ctas = value;
  else if (k == "heap_small_blocks") c->opt_heap_small = std::max<int64_t>(1, value);
  else if (k == "heap_big_blocks") c->opt_heap_big = std::max<int64_t>(1, value);
  else if (k == "profile") c->opt_profile = value;
  else if (k == "pinned_send_direct") c->opt_pinned_send_direct = value;
  else if (k == "pull_keep_us") c->opt_pull_keep_us = std::max<int64_t>(0, value);
  else if (k == "stage_upload_kernel") c->opt_stage_upload_kernel = value;
  else if (k == "hostdst_tma") c->opt_hostdst_tma = value;
  else if (k == "hostdst_ce") c->opt_hostdst_ce = value;
  else if (k == "max_mappings") c->opt_max_mappings = std::max<int64_t>(1, value);
  else if (k == "stage_batch_bytes") c->opt_stage_batch_bytes = std::max<int64_t>(65536, value);
  else if (k == "coalesce_us") c->opt_coalesce_us = value;
  else if (k == "coalesce_bytes") c->opt_coalesce_bytes = value;
  else if (k == "done_flags") c->opt_done_flags = value;
  else if (k == "bulk_balance") c->opt_bulk_balance = value;
  else if (k == "consumer_polling") c->consumer_polling.store(value != 0, std::memory_order_seq_cst);
  else if (k == "linger_us") c->opt_linger_us = std::max<int64_t>(1, value);
  else if (k == "max_life_us") c->opt_max_life_us = std::max<int64_t>(10, value);
  else if (k == "armed_ms") c->opt_armed_ms = std::max<int64_t>(0, value);
  else if (k == "pull_ctas" && value != 1) c->opt_pull_ctas = std::max<int64_t>(0, value);
  else if (k == "resident_puts") c->opt_resident_puts = std::max<int64_t>(0, value);
  else if (k == "yield_us") c->opt_yield_us = std::max<int64_t>(0, value);
  else {
    set_error(k == "pull_ctas" ? "pull_ctas: " + std::string(kPullCtasOne) : "unknown option " + k);
    return -1;
  }
  return 0;
}
int64_t sw_get_option(sw_ctx* ctx, const char* key) {
  Ctx* c = (Ctx*)ctx;
  std::string k(key);
  if (k == "ring_slots") return c->opt_ring_slots;
  if (k == "bulk_mode") return c->opt_bulk_mode;
  if (k == "bulk_stages") return c->opt_bulk_stages;
  if (k == "bulk_stage_bytes") return c->opt_bulk_stage_bytes;
  if (k == "bulk_ctas_per_sm") return c->opt_bulk_ctas;
  if (k == "heap_small_blocks") return c->opt_heap_small;
  if (k == "heap_big_blocks") return c->opt_heap_big;
  if (k == "profile") return c->opt_profile;
  if (k == "sm_count") return swgpu::sm_count();
  if (k == "resident") return 1;   // receives always run on the resident control kernels (read-only)
  if (k == "linger_us") return c->opt_linger_us;
  if (k == "max_life_us") return c->opt_max_life_us;
  if (k == "armed_ms") return c->opt_armed_ms;
  if (k == "pull_ctas") return c->opt_pull_ctas;
  if (k == "pull_keep_us") return c->opt_pull_keep_us;
  if (k == "max_mappings") return c->opt_max_mappings;
  if (k == "eager_max") return c->opt_eager_max;
  return -1;
}

sw_worker_t sw_worker_create(sw_ctx* ctx, int kind) {
  Ctx* c = (Ctx*)ctx;
  if (kind != SW_WORKER_SERVER && kind != SW_WORKER_CLIENT) {
    set_error("bad worker kind");
    return 0;
  }
  ScopedAffinity numa(c->device);
  Worker* w = Slab<Worker>::make();
  w->kind = kind;
  w->ctx = c;
  std::lock_guard<std::mutex> lk(c->mu);
  c->workers[w->id] = w;
  return w->id;
}

int sw_worker_status(sw_ctx* ctx, sw_worker_t wid) {
  Worker* w = find_worker((Ctx*)ctx, wid);
  return w ? w->status.load(std::memory_order_acquire) : -1;
}

static int server_start(Ctx* c, Worker* w, const char* addr, uint16_t port, bool tcp) {
  int expected = SW_ST_VOID;
  if (w->kind != SW_WORKER_SERVER || !w->status.compare_exchange_strong(expected, SW_ST_INIT)) {
    // reference main.cpp:818-820
    set_error("Server: already listening. You can only listen once, and cannot listen again after close.");
    return -1;
  }
  swgpu::bind_thread(c->device);
  if (!worker_alloc_device(c, w)) {
    w->status.store(SW_ST_VOID);
    return -1;
  }
  w->unix_fd = make_unix_listener(w->unix_name);
  if (w->unix_fd < 0) {
    set_error("Server: failed to create the bootstrap socket");
    worker_release(c, w, false);
    w->status.store(SW_ST_VOID);
    return -1;
  }
  if (tcp) {
    w->tcp_fd = make_tcp_listener(addr, port);
    if (w->tcp_fd < 0) {
      set_error(std::string("UCP error: failed to create listener - ") + strerror(errno));
      worker_release(c, w, false);
      w->status.store(SW_ST_VOID);
      return -1;
    }
  }
  fill_blob(c, w);
  w->status.store(SW_ST_RUNNING, std::memory_order_release);
  w->register_queued.store(true, std::memory_order_release);
  sq_push(c, SQ_REGISTER, w, nullptr);
  return 0;
}

int sw_listen(sw_ctx* ctx, sw_worker_t wid, const char* addr, uint16_t port) {
  Ctx* c = (Ctx*)ctx;
  Worker* w = find_worker(c, wid);
  if (!w) {
    set_error("bad worker handle");
    return -1;
  }
  return server_start(c, w, addr, port, true);
}
int sw_listen_address(sw_ctx* ctx, sw_worker_t wid) {
  Ctx* c = (Ctx*)ctx;
  Worker* w = find_worker(c, wid);
  if (!w) {
    set_error("bad worker handle");
    return -1;
  }
  return server_start(c, w, nullptr, 0, false);
}

int64_t sw_get_address(sw_ctx* ctx, sw_worker_t wid, void* out, size_t cap) {
  Worker* w = find_worker((Ctx*)ctx, wid);
  if (!w || !w->blob_ready.load(std::memory_order_acquire) || w->status.load() == SW_ST_CLOSED) {
    // reference main.cpp:587-590, 854-857
    set_error(w && w->kind == SW_WORKER_CLIENT ? "Client: worker address not ready. Connect first before querying."
                                               : "Server: worker address not ready. Start listening first.");
    return -1;
  }
  if (cap < sizeof(AddrBlob)) return (int64_t)sizeof(AddrBlob);
  memcpy(out, &w->blob, sizeof(AddrBlob));
  return (int64_t)sizeof(AddrBlob);
}

static uint64_t client_start(Ctx* c, Worker* w, ConnectReq req) {
  int expected = SW_ST_VOID;
  if (w->kind != SW_WORKER_CLIENT || !w->status.compare_exchange_strong(expected, SW_ST_INIT)) {
    // reference main.cpp:554-555
    set_error("Client: already connected. You can only connect once, and cannot reconnect after close.");
    return 0;
  }
  req.op_id = c->next_id.fetch_add(1);
  fill_blob(c, w);
  w->connector = std::thread(client_connect_thread, c, w, req);
  return req.op_id;
}

uint64_t sw_connect(sw_ctx* ctx, sw_worker_t wid, const char* addr, uint16_t port) {
  Ctx* c = (Ctx*)ctx;
  Worker* w = find_worker(c, wid);
  if (!w) {
    set_error("bad worker handle");
    return 0;
  }
  ConnectReq req;
  req.mode = 0;
  req.addr = addr ? addr : "";
  req.port = port;
  memset(&req.blob, 0, sizeof(req.blob));
  return client_start(c, w, req);
}
uint64_t sw_connect_address(sw_ctx* ctx, sw_worker_t wid, const void* blob, size_t len) {
  Ctx* c = (Ctx*)ctx;
  Worker* w = find_worker(c, wid);
  if (!w) {
    set_error("bad worker handle");
    return 0;
  }
  ConnectReq req;
  req.mode = 1;
  req.port = 0;
  memset(&req.blob, 0, sizeof(req.blob));
  if (blob && len >= sizeof(AddrBlob)) memcpy(&req.blob, blob, sizeof(AddrBlob));
  return client_start(c, w, req);
}

uint64_t sw_close(sw_ctx* ctx, sw_worker_t wid) {
  Ctx* c = (Ctx*)ctx;
  Worker* w = find_worker(c, wid);
  int expected = SW_ST_RUNNING;
  if (!w || !w->status.compare_exchange_strong(expected, SW_ST_CLOSING)) {
    // reference main.cpp:596-597, 1377-1378
    set_error(w && w->kind == SW_WORKER_SERVER ? "Server: not running. You can only close once, after listen."
                                               : "Client: not running. You can only close once, after connect done.");
    return 0;
  }
  uint64_t op = c->next_id.fetch_add(1);
  sq_push(c, SQ_CLOSE, w, (void*)(uintptr_t)op);
  return op;
}

int sw_worker_destroy(sw_ctx* ctx, sw_worker_t wid) {
  Ctx* c = (Ctx*)ctx;
  Worker* w = find_worker(c, wid);
  if (!w) return -1;
  // a connect may still be running
  if (w->connector.joinable()) w->connector.join();
  double deadline = now_s() + 2.0;
  while (w->status.load() == SW_ST_INIT && now_s() < deadline) sched_yield();
  int expected = SW_ST_RUNNING;
  if (w->status.compare_exchange_strong(expected, SW_ST_CLOSING)) sq_push(c, SQ_CLOSE, w, nullptr);
  deadline = now_s() + 10.0;
  while (w->status.load() == SW_ST_CLOSING && now_s() < deadline) {
    struct timespec ts = {0, 100000};
    nanosleep(&ts, nullptr);
  }
  // Recycle the record once nothing references it: never handed to the progress thread, or handed
  // over and already dropped by it.  (A worker stuck in CLOSING keeps its tombstone.)
  const int st = w->status.load(std::memory_order_acquire);
  if (st == SW_ST_VOID || st == SW_ST_CLOSED) {
    bool free_now = !w->register_queued.load(std::memory_order_acquire);
    if (!free_now) {
      deadline = now_s() + 0.5;
      while (!w->retired.load(std::memory_order_acquire) && now_s() < deadline) {
        struct timespec ts = {0, 50000};
        nanosleep(&ts, nullptr);
      }
      free_now = w->retired.load(std::memory_order_acquire);
    }
    if (free_now) recycle_worker(c, w);
  }
  return 0;
}

static uint64_t not_running(Worker* w, const char* verb) {
  // reference main.cpp:607-608, 629-630, 651-652, 1389-1390, 1413-1414, 1435-1436, 1455-1456
  bool server = w && w->kind == SW_WORKER_SERVER;
  set_error(std::string(server ? "Server" : "Client") + ": not running. You can only " + verb + ", after " +
            (server ? "listen." : "connect."));
  return 0;
}

uint64_t sw_post_send(sw_ctx* ctx, sw_worker_t wid, sw_ep_t epid, const void* ptr, size_t len, uint64_t tag,
                      int mem_kind) {
  Ctx* c = (Ctx*)ctx;
  Worker* w = find_worker(c, wid);
  if (!w || w->status.load(std::memory_order_acquire) != SW_ST_RUNNING) return not_running(w, "send");
  Ep* ep = nullptr;
  if (w->kind == SW_WORKER_CLIENT) {
    ep = w->eps.empty() ? nullptr : w->eps[0];
  } else {
    ep = find_ep(c, epid);
    if (ep && ep->owner != w) ep = nullptr;
  }
  if (!ep) {
    set_error("send: unknown endpoint");
    return 0;
  }
  SendOp* op = new SendOp();
  op->op_id = c->next_id.fetch_add(1);
  op->w = w;
  op->ep = ep;
  op->ptr = (const uint8_t*)ptr;
  op->len = len;
  op->tag = tag;
  op->mem = len ? classify_mem(ptr, mem_kind) : SW_MEM_DEVICE;
  uint64_t id = op->op_id;
  sq_push(c, SQ_SEND, w, op, &op->sqn);
  return id;
}

uint64_t sw_post_recv(sw_ctx* ctx, sw_worker_t wid, void* ptr, size_t cap, uint64_t tag, uint64_t tag_mask,
                      int mem_kind) {
  Ctx* c = (Ctx*)ctx;
  Worker* w = find_worker(c, wid);
  if (!w || w->status.load(std::memory_order_acquire) != SW_ST_RUNNING) return not_running(w, "recv");
  RecvOp* r = new RecvOp();
  r->op_id = c->next_id.fetch_add(1);
  r->w = w;
  r->ptr = (uint8_t*)ptr;
  r->cap = cap;
  r->tag = tag;
  r->mask = tag_mask;
  r->mem = cap ? classify_mem(ptr, mem_kind) : SW_MEM_DEVICE;
  uint64_t id = r->op_id;
  sq_push(c, SQ_RECV, w, r, &r->sqn);
  return id;
}

static_assert((int)SW_DTYPE_F32 == (int)SW_DT_F32 && (int)SW_DTYPE_F16 == (int)SW_DT_F16 &&
                  (int)SW_DTYPE_BF16 == (int)SW_DT_BF16 && (int)SW_DTYPE_F64 == (int)SW_DT_F64 &&
                  (int)SW_DTYPE_I32 == (int)SW_DT_I32 && (int)SW_DTYPE_I64 == (int)SW_DT_I64,
              "element type numbering of the C ABI and the kernels");

uint64_t sw_post_recv_reduce(sw_ctx* ctx, sw_worker_t wid, void* ptr, size_t cap, uint64_t tag, uint64_t tag_mask,
                             int dtype) {
  Ctx* c = (Ctx*)ctx;
  Worker* w = find_worker(c, wid);
  if (!w || w->status.load(std::memory_order_acquire) != SW_ST_RUNNING) return not_running(w, "recv");
  const uint32_t isz = sw_dtype_size(dtype);
  if (!isz) {
    set_error("recv_reduce: unknown element type");
    return 0;
  }
  if (cap % isz || (uintptr_t)ptr % isz) {
    set_error("recv_reduce: buffer address and size must be multiples of the element size");
    return 0;
  }
  if (cap) {
    swgpu::PtrInfo pi;
    swgpu::ptr_info(ptr, &pi);
    if (!pi.is_device || pi.device != c->device) {
      set_error("recv_reduce: the buffer is not device memory of the context's device");
      return 0;
    }
  }
  RecvOp* r = new RecvOp();
  r->op_id = c->next_id.fetch_add(1);
  r->w = w;
  r->ptr = (uint8_t*)ptr;
  r->cap = cap;
  r->tag = tag;
  r->mask = tag_mask;
  r->mem = SW_MEM_DEVICE;
  r->dtype = dtype;
  uint64_t id = r->op_id;
  sq_push(c, SQ_RECV, w, r, &r->sqn);
  return id;
}

uint64_t sw_post_flush(sw_ctx* ctx, sw_worker_t wid) {
  Ctx* c = (Ctx*)ctx;
  Worker* w = find_worker(c, wid);
  if (!w || w->status.load(std::memory_order_acquire) != SW_ST_RUNNING) return not_running(w, "flush");
  FlushOp* f = new FlushOp();
  f->op_id = c->next_id.fetch_add(1);
  uint64_t id = f->op_id;
  sq_push(c, SQ_FLUSH, w, f, &f->sqn);
  return id;
}
uint64_t sw_post_flush_ep(sw_ctx* ctx, sw_worker_t wid, sw_ep_t epid) {
  Ctx* c = (Ctx*)ctx;
  Worker* w = find_worker(c, wid);
  if (!w || w->status.load(std::memory_order_acquire) != SW_ST_RUNNING) return not_running(w, "flush");
  Ep* ep = find_ep(c, epid);
  if (!ep || ep->owner != w) {
    set_error("flush_ep: unknown endpoint");
    return 0;
  }
  FlushOp* f = new FlushOp();
  f->op_id = c->next_id.fetch_add(1);
  f->ep = ep;
  uint64_t id = f->op_id;
  sq_push(c, SQ_FLUSH, w, f, &f->sqn);
  return id;
}

static void clear_efd_if_empty(Ctx* c) {  // cq_mu held
  if (c->cq.empty() && c->efd >= 0 && c->efd_signaled.exchange(0, std::memory_order_acq_rel)) {
    uint64_t v;
    ssize_t r = read(c->efd, &v, sizeof(v));
    (void)r;
  }
}

int sw_poll(sw_ctx* ctx, sw_completion* out, int max) {
  Ctx* c = (Ctx*)ctx;
  // nothing queued and no stale eventfd signal: no lock, no system call (busy-polling consumers)
  if (c->cq_count.load(std::memory_order_seq_cst) == 0 && !c->efd_signaled.load(std::memory_order_acquire)) return 0;
  std::lock_guard<std::mutex> lk(c->cq_mu);
  int n = 0;
  while (n < max && !c->cq.empty()) {
    out[n++] = c->cq.front();
    c->cq.pop_front();
  }
  c->cq_count.store((uint32_t)c->cq.size(), std::memory_order_seq_cst);
  clear_efd_if_empty(c);
  return n;
}

int sw_wait(sw_ctx* ctx, sw_completion* out, int max, int timeout_ms) {
  Ctx* c = (Ctx*)ctx;
  std::unique_lock<std::mutex> lk(c->cq_mu);
  if (c->cq.empty()) {
    c->cq_waiters.fetch_add(1, std::memory_order_seq_cst);
    c->cq_cv.wait_for(lk, std::chrono::milliseconds(timeout_ms), [&] { return !c->cq.empty(); });
    c->cq_waiters.fetch_sub(1, std::memory_order_seq_cst);
  }
  int n = 0;
  while (n < max && !c->cq.empty()) {
    out[n++] = c->cq.front();
    c->cq.pop_front();
  }
  c->cq_count.store((uint32_t)c->cq.size(), std::memory_order_seq_cst);
  clear_efd_if_empty(c);
  return n;
}

int sw_event_fd(sw_ctx* ctx) { return ((Ctx*)ctx)->efd; }

int sw_list_eps(sw_ctx* ctx, sw_worker_t wid, sw_ep_t* out, int max) {
  Ctx* c = (Ctx*)ctx;
  std::lock_guard<std::mutex> lk(c->mu);
  auto it = c->workers.find(wid);
  if (it == c->workers.end()) return -1;
  int n = 0;
  // endpoints are never removed (reference: tests/test_basic.py:53-56)
  std::vector<uint64_t> ids;
  for (auto& kv : c->eps)
    if (kv.second->owner == it->second) ids.push_back(kv.first);
  std::sort(ids.begin(), ids.end());
  for (uint64_t id : ids) {
    if (n < max) out[n] = id;
    n++;
  }
  return n;
}

int sw_ep_info_get(sw_ctx* ctx, sw_worker_t wid, sw_ep_t epid, sw_ep_info* out) {
  Ep* ep = find_ep((Ctx*)ctx, epid);
  if (!ep || ep->owner->id != wid) return -1;
  *out = ep->info;
  return 0;
}

// reference evaluate_perf (main.cpp:452-467, 666-678) returns UCX's analytic time estimate for a
// message size.  Here: latency + size / bandwidth, with the latencies of `bench_scenarios.py pingpong` and the
// 1 GiB loopback rate of the bench sweep, measured on one H100 SXM (80 GB, 400 W power limit), seconds.
double sw_evaluate_perf(sw_ctx* ctx, sw_worker_t wid, sw_ep_t epid, size_t msg_size) {
  Ctx* c = (Ctx*)ctx;
  Worker* w = find_worker(c, wid);
  if (!w || w->status.load() != SW_ST_RUNNING) {
    set_error("Server: not running. You can only evaluate perf, after listen.");
    return -1.0;
  }
  Ep* ep = epid ? find_ep(c, epid) : (w->eps.empty() ? nullptr : w->eps[0]);
  const bool same_gpu = !ep || ep->in_process || ep->peer_device == c->device;
  const bool eager = msg_size <= (size_t)c->opt_eager_max.load();
  // One-way latency through the asyncio API on one GPU: 64 B 29.9 us, 1 MiB 52.3 us.
  // A peer over NVLink has not been measured on H100; its estimate takes the same latency.
  const double lat = eager ? 29.9e-6 : 52.3e-6;
  // copy rate of one large message: HBM copy on one GPU (1.16 TB/s payload at 1 GiB, measured), NVLink 4 pull
  // between GPUs (450 GB/s per direction, nominal: not measured)
  const double bw = same_gpu ? 1.16e12 : 4.5e11;
  return lat + (double)msg_size / bw;
}

int sw_stats_get(sw_ctx* ctx, sw_stats* out) {
  Ctx* c = (Ctx*)ctx;
  if (!tls_is_progress) {
    // the pull CTAs publish their byte / busy-time counters when they leave: ask them to (they are relaunched
    // at once if copies are outstanding), bounded wait
    c->stats_flush.store(1, std::memory_order_release);
    sq_push(c, 0, nullptr, nullptr);   // wake a napping progress thread
    const double deadline = now_s() + 0.25;
    while (c->stats_flush.load(std::memory_order_acquire) && now_s() < deadline) {
      struct timespec ts = {0, 20000};
      nanosleep(&ts, nullptr);
    }
  }
  std::lock_guard<std::mutex> lk(c->st_mu);
  *out = c->stats;
  return 0;
}
int sw_stats_reset(sw_ctx* ctx) {
  Ctx* c = (Ctx*)ctx;
  std::lock_guard<std::mutex> lk(c->st_mu);
  memset(&c->stats, 0, sizeof(c->stats));
  return 0;
}

}  // extern "C"
