// starway_b200 — resident progress kernels (sm_90a): the receive side without the host on the data path.
//
//   sw_progress_kernel  ONE CTA per worker (Client / Server object), resident for a bounded time:
//                         warp 0   matcher: polls the slot headers of the inbound rings (ld.acquire.sys on the
//                                  sequence word the peer's put kernel releases last), takes new receives staged
//                                  by warp 1, runs the tag matching over the device-resident posted / unexpected
//                                  queues, copies small payloads itself, writes completion records and credits
//                                  straight to host-visible memory, hands rendezvous matches to the pull queue
//                         warp 1   host link: polls the worker's control words and the post ring in pinned host
//                                  memory (PCIe reads off the matcher's critical path), decides when to leave
//                         warp 2   puts: small batches of sends the host hands over while the kernel is resident
//                                  (payload + released header into the peer's ring, no launch on the sender side)
//                         warp 3+  helpers: eager payloads above SW_INLINE_DELIVER bytes
//                       (replaces ucp_worker_progress + the matching inside ucp_tag_recv_nbx,
//                        reference src/bindings/main.cpp:362,1127 and :404,1172)
//   sw_pull_kernel      resident pull CTAs of the context (one elected thread each drives the cp.async.bulk
//                       pipeline): claim chunks of published batches, copy sender buffer -> receive buffer through
//                       the CUDA-IPC peer mapping, the CTA that completes a batch writes the completion records
//                       and the FIN words of the senders (replaces the rendezvous leg of ucp_tag_send_nbx,
//                       reference main.cpp:370,1136)
//
// Both kernels leave on their own (linger / maximum lifetime / host request), always with consistent state in
// device memory; the host relaunches them while work is expected.  Pure data movement and uint64
// xor/and/compare: no tensor cores, no floating point.
#pragma once
#include "kernels.cuh"

// ------------------------------------------------------------------ memory-model helpers
__device__ __forceinline__ uint64_t sw_ld_acquire_sys(const void* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t sw_ld_relaxed_sys(const void* p) {
  uint64_t v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void sw_st_release_sys(void* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void sw_st_relaxed_sys(void* p, uint64_t v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t sw_ld_acquire_gpu(const void* p) {
  uint64_t v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void sw_st_release_gpu(void* p, uint64_t v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t sw_globaltimer() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ int4 sw_ld16_sys(const void* p) {   // host-visible memory: never served from L1
  int4 r;
  asm volatile("ld.relaxed.sys.global.v4.s32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}

// one completion record: body first, system-scope fence (payload copies of this warp included), then the word
// that carries status + pass number -- the host reads that word first
// `host_dst`: the payload went to host memory: payload and record travel the same way and get a system-scope
// fence between them (~1.5 us, `sw_probe hostlat`).  A payload in device memory only has to be performed at gpu
// scope before the record leaves (L2 is where every later reader of that buffer looks; 0.3 us); the fence also
// keeps the record's body ahead of its pass word on the way out (posted writes of one requester stay in order).
__device__ __forceinline__ void sw_write_cqe(SwCqEnt* ring, uint64_t idx, uint64_t op, uint64_t tag, uint64_t len,
                                             int32_t status, bool host_dst = true) {
  SwCqEnt* e = &ring[idx % SW_CQ_RING];
  e->op_id = op;
  e->tag = tag;
  e->len = len;
  if (host_dst)
    __threadfence_system();
  else
    __threadfence();
  const uint64_t w = (static_cast<uint64_t>(sw_ring_pass(idx, SW_CQ_RING)) << 32) | static_cast<uint32_t>(status);
  sw_st_relaxed_sys(&e->status, w);
}

// single-thread copy of a small payload (the lane-per-message path of the matcher)
__device__ __forceinline__ void sw_copy_lane(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint32_t len) {
  const uint64_t a = reinterpret_cast<uint64_t>(src) | reinterpret_cast<uint64_t>(dst);
  uint32_t i = 0;
  if ((a & 15) == 0) {
    for (; i + 16 <= len; i += 16) sw_st16(dst + i, sw_ld16(src + i));
  } else if ((a & 3) == 0) {
    for (; i + 4 <= len; i += 4) *reinterpret_cast<uint32_t*>(dst + i) = *reinterpret_cast<const uint32_t*>(src + i);
  }
  for (; i < len; i++) dst[i] = src[i];
}

// ------------------------------------------------------------------ launch parameters
struct SwProgArgs {
  SwMatchState* st;
  SwProgCtl* ctl;            // pinned host
  const SwPostEnt* posts;    // pinned host, SW_POST_RING entries
  SwCqEnt* cq;               // pinned host, SW_CQ_RING entries: eager completions (index allocated by the matcher)
  SwCqEnt* cqr;              // pinned host, SW_CQ_RING entries: rendezvous completions (allocated by pull CTAs)
  SwHrEnt* hr;               // pinned host, SW_HR_RING entries
  const SwSendLL* sends;     // pinned host, SW_SEND_RING stamped entries
  SwPullQueue* pq;           // device memory (nullptr: every rendezvous goes to the host)
  const SwMapEnt* map;       // device memory
  uint64_t ctx_uuid;
  uint64_t launch_seq;
  uint32_t pid, n_eps;
  uint32_t linger_us, max_life_us;
  uint32_t pull_ctas, clk_mhz;
};

constexpr uint32_t SW_PROG_THREADS = 256;
constexpr uint32_t SW_PROG_PUTTERS = 1;
constexpr uint32_t SW_PROG_HELPERS = SW_PROG_THREADS / 32 - 2 - SW_PROG_PUTTERS;
constexpr uint32_t SW_SSEND_RING = 32;
constexpr uint32_t SW_DJOB_RING = 64;
constexpr uint32_t SW_SPOST_RING = 64;
constexpr uint32_t SW_PEND_RING = 128;

struct SwDJob {      // matcher -> helper warp
  uint64_t src, dst, len, op_id, tag, msg_len, cq_idx;
  int32_t status;
  uint32_t pad;
};
struct SwPend {      // something that may only be released once helper job `job` has finished
  uint64_t job;
  uint64_t cons_after;   // kind 0: ring cursor to publish
  uint32_t kind;         // 0: ring credit (arg = endpoint), 1: small heap block, 2: big heap block (arg = block)
  uint32_t arg;
};

struct SwProgShared {
  SwPostEnt posts[SW_SPOST_RING];
  SwSendEnt sends[SW_SSEND_RING];
  uint64_t fin_ptr[SW_MAX_EPS];
  SwDJob jobs[SW_DJOB_RING];
  SwPend pend[SW_PEND_RING];
  uint64_t ring_base[SW_MAX_EPS];
  uint64_t cons[SW_MAX_EPS];
  uint64_t credit[SW_MAX_EPS];       // cursor published to the sender so far
  uint64_t releasable[SW_MAX_EPS];   // cursor that may be published (no helper still reads a slot below it)
  uint32_t ring_mask[SW_MAX_EPS];
  uint32_t ring_gen[SW_MAX_EPS];
  uint32_t pend_cnt[SW_MAX_EPS];
  // rendezvous batch under construction
  uint64_t pb_end[SW_PULL_JOBS], pb_src[SW_PULL_JOBS], pb_dst[SW_PULL_JOBS];
  SwPullMeta pb_meta[SW_PULL_JOBS];
  // cross-warp words
  volatile uint64_t post_tail;    // staged by the link warp
  volatile uint64_t post_head;    // consumed by the matcher
  volatile uint64_t job_tail;     // jobs emitted by the matcher
  volatile uint64_t send_tail;    // put descriptors staged by the link warp
  volatile uint64_t send_done;    // every put below this index has been executed (and published to the host)
  volatile uint64_t send_base;    // index of the first put of this launch
  volatile long long t_staged, t_released;   // latency budget of resident puts (last put)
  volatile uint64_t cq_head, cqr_head, hr_head, dead_mask, host_epoch;   // copies of the host's words
  volatile long long active_clk;  // last time the matcher did something
  volatile uint32_t helper_done[SW_PROG_HELPERS];
  volatile uint32_t exit_req;     // link warp -> matcher
  volatile uint32_t helpers_exit; // matcher -> helpers
};

struct SwResCtx {   // warp-uniform state of the matcher, in registers for the life of the kernel
  uint64_t p_head, p_tail, u_head, u_tail;
  uint32_t p_count, u_count, n_free_small, n_free_big;
  uint64_t cq_alloc, hr_alloc, jobs_emitted, pull_jobs, arrivals, post_head;
  uint32_t pend_head, pend_tail, pb_n, err;
  bool stalled;
  SwPullSlot* last_slot;   // where sw_res_flush_pull published last
  uint64_t last_ticket;
};

// ------------------------------------------------------------------ matcher building blocks
__device__ __forceinline__ uint64_t sw_warp_min64(uint64_t v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const uint64_t x = sw_shfl64(v, (threadIdx.x & 31) ^ o);
    v = x < v ? x : v;
  }
  return v;
}

// smallest helper-job index that has not finished
__device__ __forceinline__ uint64_t sw_done_prefix(const SwProgShared& sh, uint32_t lane) {
  uint64_t v = ~0ull;
  if (lane < SW_PROG_HELPERS) v = lane + static_cast<uint64_t>(sh.helper_done[lane]) * SW_PROG_HELPERS;
  return sw_warp_min64(v);
}

__device__ __forceinline__ void sw_publish_credit(SwMatchState* st, SwProgShared& sh, uint32_t ep, uint64_t cons, uint32_t lane) {
  if (lane == 0 && cons > sh.credit[ep]) {
    sh.credit[ep] = cons;
    if (st->credit_ptr[ep]) sw_st_release_sys(reinterpret_cast<void*>(st->credit_ptr[ep]), cons);
  }
}

// releases whose helper job has finished: ring credits, heap blocks
__device__ __forceinline__ void sw_retire(SwMatchState* st, SwProgShared& sh, SwResCtx& c, uint32_t lane, bool wait_all) {
  while (c.pend_head != c.pend_tail) {
    const uint64_t prefix = sw_done_prefix(sh, lane);
    bool any = false;
    while (c.pend_head != c.pend_tail) {
      const SwPend p = sh.pend[c.pend_head % SW_PEND_RING];
      if (p.job >= prefix) break;
      if (p.kind == 0) {
        // the slots up to this job's are free again (published lazily: a release costs a system-scope fence)
        if (lane == 0) {
          sh.pend_cnt[p.arg]--;
          const uint64_t r = sh.pend_cnt[p.arg] == 0 ? sh.cons[p.arg] : p.cons_after;
          if (r > sh.releasable[p.arg]) sh.releasable[p.arg] = r;
        }
        __syncwarp();
      } else if (p.kind == 1) {
        if (lane == 0) st->free_small[c.n_free_small] = p.arg;
        c.n_free_small++;
      } else {
        if (lane == 0) st->free_big[c.n_free_big] = p.arg;
        c.n_free_big++;
      }
      c.pend_head++;
      any = true;
    }
    __syncwarp();
    if (!wait_all) break;
    if (!any) __nanosleep(50);
  }
}

__device__ __forceinline__ void sw_cq_room(const SwProgShared& sh, const SwResCtx& c, uint32_t n) {
  while (c.cq_alloc + n - sh.cq_head > SW_CQ_RING) __nanosleep(100);   // the link warp refreshes cq_head
}

// Complete a receive whose payload (copy_len bytes, already clipped / 0 on error) is at `src`.
// src_kind 0: ring slot of endpoint `arg` (its cursor after this slot is cons_after), 1 / 2: heap block `arg`.
// Returns true when the source was released at once (copied by the matcher), false when a helper owns it.
__device__ __forceinline__ bool sw_res_deliver(SwMatchState* st, SwProgShared& sh, const SwProgArgs& a, SwResCtx& c,
                                               uint32_t lane, uint64_t src, uint64_t dst, uint64_t copy_len, uint64_t op,
                                               uint64_t tag, uint64_t msg_len, int32_t status, uint32_t src_kind,
                                               uint32_t arg, uint64_t cons_after, uint32_t pflags) {
  sw_cq_room(sh, c, 1);
  const uint64_t cq_idx = c.cq_alloc++;
  if (copy_len <= SW_INLINE_DELIVER) {
    sw_copy(reinterpret_cast<uint8_t*>(dst), reinterpret_cast<const uint8_t*>(src), copy_len, lane, 32);
    __syncwarp();
    if (lane == 0) sw_write_cqe(a.cq, cq_idx, op, tag, msg_len, status, (pflags & SW_POST_HOSTBUF) != 0);
    if (src_kind == 1) {
      if (lane == 0) st->free_small[c.n_free_small] = arg;
      c.n_free_small++;
    } else if (src_kind == 2) {
      if (lane == 0) st->free_big[c.n_free_big] = arg;
      c.n_free_big++;
    }
    return true;
  }
  // helper job: wait for room in the job ring and in the pending-release ring
  while (c.jobs_emitted - sw_done_prefix(sh, lane) >= SW_DJOB_RING || c.pend_tail - c.pend_head >= SW_PEND_RING) {
    sw_retire(st, sh, c, lane, false);
    __nanosleep(50);
  }
  if (lane == 0) {
    SwDJob* j = &sh.jobs[c.jobs_emitted % SW_DJOB_RING];
    j->src = src;
    j->dst = dst;
    j->len = copy_len;
    j->op_id = op;
    j->tag = tag;
    j->msg_len = msg_len;
    j->cq_idx = cq_idx;
    j->status = status;
    j->pad = pflags;
    SwPend* p = &sh.pend[c.pend_tail % SW_PEND_RING];
    p->job = c.jobs_emitted;
    p->cons_after = cons_after;
    p->kind = src_kind;
    p->arg = arg;
    if (src_kind == 0) sh.pend_cnt[arg]++;
    __threadfence_block();
    sh.job_tail = c.jobs_emitted + 1;
  }
  c.jobs_emitted++;
  c.pend_tail++;
  __syncwarp();
  return false;
}

// publish the rendezvous batch under construction to the pull CTAs of the context
__device__ __forceinline__ void sw_res_flush_pull(SwMatchState* st, SwProgShared& sh, const SwProgArgs& a, SwResCtx& c,
                                                  uint32_t lane) {
  if (c.pb_n == 0) return;
  SwPullQueue* q = a.pq;
  uint64_t ticket = 0;
  if (lane == 0) ticket = atomicAdd(reinterpret_cast<unsigned long long*>(&q->alloc), 1ull);
  ticket = sw_shfl64(ticket, 0);
  SwPullSlot* s = &q->slot[ticket % SW_PULL_SLOTS];
  const uint64_t want = ticket >= SW_PULL_SLOTS ? ticket - SW_PULL_SLOTS + 1 : 0;
  while (sw_ld_acquire_gpu(&s->free_seq) != want) __nanosleep(100);   // the previous occupant has been retired
  const uint32_t n = c.pb_n;
  for (uint32_t j = lane; j < n; j += 32) {
    s->end[j] = sh.pb_end[j];
    s->src[j] = sh.pb_src[j];
    s->dst[j] = sh.pb_dst[j];
    s->meta[j] = sh.pb_meta[j];
  }
  if (lane == 0) {
    const uint64_t total = sh.pb_end[n - 1];
    // chunk: about one per copy CTA (claims are dynamic: a CTA that is still busy with an earlier batch simply
    // takes none), 8 KiB .. 256 KiB, a multiple of 1 KiB
    uint64_t chunk = total / (a.pull_ctas > 1 ? a.pull_ctas - 1 : 1) + 1023;
    chunk &= ~1023ull;
    if (chunk < 8192) chunk = 8192;
    if (chunk > 262144) chunk = 262144;
    uint64_t nch = (total + chunk - 1) / chunk;
    if (nch == 0) nch = 1;
    s->njobs = n;
    s->nchunks = static_cast<uint32_t>(nch);
    s->exit = 0;
    s->chunk_bytes = chunk;
    s->total = total;
    s->next_chunk = 0;
    s->done_chunks = 0;
    s->retire = 0;
    s->t_first = 0;
    s->t_pub = sw_globaltimer();
    s->cqr_ring = reinterpret_cast<uint64_t>(a.cqr);
    s->cqr_alloc = reinterpret_cast<uint64_t>(&st->cqr_alloc);
    s->cqr_head_dev = reinterpret_cast<uint64_t>(&st->cqr_head);
    s->cqr_head_host = reinterpret_cast<uint64_t>(&a.ctl->cqr_head);
  }
  __syncwarp();
  if (lane == 0) {
    __threadfence();
    sw_st_release_gpu(&s->seq, ticket + 1);
    a.ctl->pull_jobs = c.pull_jobs;   // the host keeps the pull kernel alive while jobs are outstanding
  }
  c.last_slot = s;
  c.last_ticket = ticket;
  c.pb_n = 0;
  __syncwarp();
}

// warp-wide probe of the (exporter, allocation) -> mapped base table; 0: not mapped here (yet)
__device__ __forceinline__ uint64_t sw_map_lookup(const SwMapEnt* map, uint64_t uuid, uint64_t buf_id, uint64_t remote_base,
                                                  uint32_t lane) {
  if (!map || !buf_id) return 0;
  const SwMapEnt* e = &map[(sw_map_home(uuid, buf_id) + lane) & (SW_MAP_SLOTS - 1)];
  const int4 k = sw_ld16(e);
  const uint64_t e_uuid = (static_cast<uint64_t>(static_cast<uint32_t>(k.y)) << 32) | static_cast<uint32_t>(k.x);
  const uint64_t e_buf = (static_cast<uint64_t>(static_cast<uint32_t>(k.w)) << 32) | static_cast<uint32_t>(k.z);
  const uint32_t hit = __ballot_sync(0xffffffffu, e_uuid == uuid && e_buf == buf_id);
  if (!hit) return 0;
  const int L = __ffs(hit) - 1;
  uint64_t rb = 0, lb = 0;
  if (static_cast<int>(lane) == L) {
    rb = e->remote_base;
    lb = e->local_base;
  }
  rb = sw_shfl64(rb, L);
  lb = sw_shfl64(lb, L);
  return rb == remote_base ? lb : 0;
}

// A rendezvous request (the 128 B SwRts at `payload`: ring slot or heap copy) met the receive (buf, cap, op).
__device__ __forceinline__ void sw_res_rts(SwMatchState* st, SwProgShared& sh, const SwProgArgs& a, SwResCtx& c,
                                           uint32_t lane, uint64_t payload, uint64_t stag, uint64_t msg_len, uint32_t epf,
                                           uint64_t buf, uint64_t cap, uint64_t op, uint32_t pflags) {
  const uint32_t w = reinterpret_cast<const volatile uint32_t*>(payload)[lane];   // 128 B descriptor, 4 B per lane, not from L1
  auto f64 = [&](int word) {
    const uint32_t lo = __shfl_sync(0xffffffffu, w, word), hi = __shfl_sync(0xffffffffu, w, word + 1);
    return (static_cast<uint64_t>(hi) << 32) | lo;
  };
  const uint64_t alloc_base = f64(16), alloc_size = f64(18), src_ptr = f64(20), send_seq = f64(22);
  const uint64_t uuid = f64(24), rflags = f64(28), buf_id = f64(30);
  const uint32_t src_pid = __shfl_sync(0xffffffffu, w, 26);
  const bool trunc = msg_len > cap;
  uint64_t src = 0;
  const uint32_t ep = epf & ((1u << SW_EP_IDX_BITS) - 1);   // ring index; the rest of the field is its generation
  bool device_path = a.pq != nullptr && a.pull_ctas != 0 && !trunc && !(pflags & SW_POST_HOSTPATH) &&
                     !(rflags & SW_RTS_PINNED_SRC) && !((sh.dead_mask >> ep) & 1) && sh.fin_ptr[ep] != 0 &&
                     (epf >> SW_EP_IDX_BITS) == sh.ring_gen[ep];
  if (device_path) {
    if (uuid == a.ctx_uuid && src_pid == a.pid) {
      src = src_ptr;   // same process, same context: the sender's pointer is ours
    } else {
      const uint64_t local = sw_map_lookup(a.map, uuid, buf_id, alloc_base, lane);
      if (local && src_ptr >= alloc_base && src_ptr - alloc_base + msg_len <= alloc_size) src = local + (src_ptr - alloc_base);
    }
    if (!src || ((src | buf) & 15)) device_path = false;   // not mapped yet / generic alignment: the host copies
  }
  if (device_path) {
    if (lane == 0) {
      const uint32_t j = c.pb_n;
      const uint64_t body = msg_len & ~15ull;
      sh.pb_end[j] = (j ? sh.pb_end[j - 1] : 0) + body;
      sh.pb_src[j] = src;
      sh.pb_dst[j] = buf;
      SwPullMeta m;
      m.op_id = op;
      m.tag = stag;
      m.len = msg_len;
      m.fin_addr = sh.fin_ptr[ep] + 8ull * (send_seq % SW_FIN_SLOTS);
      m.fin_val = (send_seq << 2) | 1;
      sh.pb_meta[j] = m;
    }
    c.pb_n++;
    c.pull_jobs++;
    __syncwarp();
    if (c.pb_n == SW_PULL_JOBS) sw_res_flush_pull(st, sh, a, c, lane);
    return;
  }
  // host path: the record travels to the host, which maps the source / launches the generic copy
  while (c.hr_alloc + 1 - sh.hr_head > SW_HR_RING) __nanosleep(100);
  SwHrEnt* h = &a.hr[c.hr_alloc % SW_HR_RING];
  reinterpret_cast<uint32_t*>(&h->rec.rts)[lane] = w;
  if (lane == 0) {
    h->rec.op_id = op;
    h->rec.dst = buf;
    h->rec.cap = cap;
    h->rec.tag = stag;
    h->rec.len = msg_len;
    h->rec.ep = epf;
    h->rec.status = trunc ? SW_ERR_MESSAGE_TRUNCATED : SW_OK;
  }
  __syncwarp();
  if (lane == 0) {
    __threadfence_system();
    sw_st_relaxed_sys(&h->pad, static_cast<uint64_t>(sw_ring_pass(c.hr_alloc, SW_HR_RING)) << 32);
  }
  c.hr_alloc++;
  __syncwarp();
}

// ------------------------------------------------------------------ phase 1: new receives (n <= 32, staged in shared memory)
__device__ __forceinline__ void sw_res_posts(SwMatchState* __restrict__ st, SwProgShared& sh, const SwProgArgs& a,
                                             SwResCtx& c, const uint32_t lane, const uint32_t n) {
  const uint64_t PQM = SW_PQ_CAP - 1, UQM = SW_UQ_CAP - 1;
  SwPostEnt mine;
  mine.tag = mine.mask = mine.buf = mine.cap = mine.op_id = 0;
  mine.flags = 0;
  if (lane < n) mine = sh.posts[(c.post_head + lane) % SW_SPOST_RING];
  if (c.u_count == 0 && SW_PQ_CAP - (c.p_tail - c.p_head) >= n) {
    // nothing is waiting in the unexpected queue: every receive is simply appended, one lane each
    if (lane < n) {
      const uint64_t s = (c.p_tail + lane) & PQM;
      st->p_tag[s] = mine.tag;
      st->p_mask[s] = mine.mask;
      st->p_buf[s] = mine.buf;
      st->p_cap[s] = mine.cap;
      st->p_op[s] = mine.op_id;
      st->p_valid[s] = 1u | (mine.flags << 8);
    }
    c.p_tail += n;
    c.p_count += n;
    __syncwarp();
    return;
  }
  // register window over the unexpected queue: lane L caches entry (wb + L)
  uint64_t wb = c.u_head;
  uint64_t w_tag = 0, w_len = 0, w_data = 0;
  uint32_t w_meta = 0, w_blk = 0;
  auto load_uwin = [&]() {
    const uint64_t idx = wb + lane;
    w_meta = 0;
    if (idx < c.u_tail) {
      const uint64_t s = idx & UQM;
      w_meta = st->u_meta[s];
      w_tag = st->u_tag[s];
      w_len = st->u_len[s];
      w_data = st->u_data[s];
      w_blk = st->u_blk[s];
    }
  };
  load_uwin();
  for (uint32_t j = 0; j < n; j++) {
    const uint64_t tag = sw_shfl64(mine.tag, j), mask = sw_shfl64(mine.mask, j);
    const uint64_t buf = sw_shfl64(mine.buf, j), cap = sw_shfl64(mine.cap, j);
    const uint64_t op = sw_shfl64(mine.op_id, j);
    const uint32_t pflags = __shfl_sync(0xffffffffu, mine.flags, j);
    bool found = false;
    uint64_t f_tag = 0, f_len = 0, f_data = 0;
    uint32_t f_meta = 0, f_blk = 0;
    if (c.u_count) {
      while (__ballot_sync(0xffffffffu, (w_meta & SW_UMETA_VALID) != 0) == 0 && wb + 32 <= c.u_tail) {
        wb += 32;
        load_uwin();
      }
      const bool hit = (w_meta & SW_UMETA_VALID) && sw_tag_match(w_tag, tag, mask);
      uint32_t bal = __ballot_sync(0xffffffffu, hit);
      if (bal) {
        const int L = __ffs(bal) - 1;
        f_tag = sw_shfl64(w_tag, L);
        f_len = sw_shfl64(w_len, L);
        f_data = sw_shfl64(w_data, L);
        f_meta = __shfl_sync(0xffffffffu, w_meta, L);
        f_blk = __shfl_sync(0xffffffffu, w_blk, L);
        if (static_cast<int>(lane) == L) {
          w_meta = 0;
          st->u_meta[(wb + L) & UQM] = 0;
        }
        found = true;
      } else {
        for (uint64_t b = wb + 32; b < c.u_tail && !found; b += 32) {
          const uint64_t idx = b + lane;
          uint32_t meta = 0;
          uint64_t t = 0;
          if (idx < c.u_tail) {
            meta = st->u_meta[idx & UQM];
            t = st->u_tag[idx & UQM];
          }
          const bool h2 = (meta & SW_UMETA_VALID) && sw_tag_match(t, tag, mask);
          bal = __ballot_sync(0xffffffffu, h2);
          if (bal) {
            const int L = __ffs(bal) - 1;
            uint64_t l = 0, dta = 0;
            uint32_t blk = 0;
            if (static_cast<int>(lane) == L) {
              l = st->u_len[idx & UQM];
              dta = st->u_data[idx & UQM];
              blk = st->u_blk[idx & UQM];
              st->u_meta[idx & UQM] = 0;
            }
            f_tag = sw_shfl64(t, L);
            f_len = sw_shfl64(l, L);
            f_data = sw_shfl64(dta, L);
            f_meta = __shfl_sync(0xffffffffu, meta, L);
            f_blk = __shfl_sync(0xffffffffu, blk, L);
            found = true;
          }
        }
      }
    }
    if (found) {
      c.u_count--;
      const bool big = (f_meta & SW_UMETA_BIG) != 0;
      if (f_meta & SW_UMETA_RTS) {
        sw_res_rts(st, sh, a, c, lane, f_data, f_tag, f_len, f_meta & SW_UMETA_EPMASK, buf, cap, op, pflags);
        // the descriptor has been read: its heap block is free again
        if (lane == 0) (big ? st->free_big[c.n_free_big] : st->free_small[c.n_free_small]) = f_blk;
        if (big)
          c.n_free_big++;
        else
          c.n_free_small++;
      } else {
        const bool trunc = f_len > cap;
        sw_res_deliver(st, sh, a, c, lane, f_data, buf, trunc ? 0 : f_len, op, f_tag, f_len,
                       trunc ? SW_ERR_MESSAGE_TRUNCATED : SW_OK, big ? 2u : 1u, f_blk, 0, pflags);
      }
    } else if (c.p_tail - c.p_head >= SW_PQ_CAP) {
      c.err |= 2;   // posted queue overflow (the host throttles before this can happen)
      sw_cq_room(sh, c, 1);
      if (lane == 0) sw_write_cqe(a.cq, c.cq_alloc, op, 0, 0, SW_ERR_NO_MEMORY);
      c.cq_alloc++;
    } else {
      if (lane == 0) {
        const uint64_t s = c.p_tail & PQM;
        st->p_tag[s] = tag;
        st->p_mask[s] = mask;
        st->p_buf[s] = buf;
        st->p_cap[s] = cap;
        st->p_op[s] = op;
        st->p_valid[s] = 1u | (pflags << 8);
      }
      c.p_tail++;
      c.p_count++;
    }
  }
  while (__ballot_sync(0xffffffffu, (w_meta & SW_UMETA_VALID) != 0) == 0 && wb + 32 <= c.u_tail) {
    wb += 32;
    load_uwin();
  }
  c.u_head = wb;
  __syncwarp();
}

// ------------------------------------------------------------------ phase 2: arrivals on one ring
// Looks at up to 32 slots from the ring cursor; a slot has arrived when its header carries the expected
// sequence number (written last, with release semantics, by the peer's put kernel).  Returns the number of
// slots consumed.
__device__ __forceinline__ uint32_t sw_res_arrivals(SwMatchState* __restrict__ st, SwProgShared& sh, const SwProgArgs& a,
                                                    SwResCtx& c, const uint32_t lane, const uint32_t ep) {
  const uint64_t PQM = SW_PQ_CAP - 1, UQM = SW_UQ_CAP - 1;
  uint64_t cons = sh.cons[ep];
  const uint32_t epf = ep | (sh.ring_gen[ep] << SW_EP_IDX_BITS);
  const uint64_t ring = sh.ring_base[ep];
  const uint64_t smask = sh.ring_mask[ep];
  const uint64_t my_slot = ring + ((cons + lane) & smask) * SW_SLOT_BYTES;
  const uint64_t seqw = sw_ld_acquire_sys(reinterpret_cast<const void*>(my_slot + 16));
  const uint32_t okb = __ballot_sync(0xffffffffu, seqw == cons + lane + 1);
  const uint32_t chunk = okb == 0xffffffffu ? 32u : static_cast<uint32_t>(__ffs(~okb) - 1);
  if (!chunk) return 0;
  uint64_t h_tag = 0, h_len = 0;
  uint32_t h_kind = 0, h_magic = 0;
  if (lane < chunk) {
    const int4 h0 = sw_ld16(reinterpret_cast<const void*>(my_slot));
    const uint64_t km = *reinterpret_cast<const volatile uint64_t*>(my_slot + 24);
    h_tag = (static_cast<uint64_t>(static_cast<uint32_t>(h0.y)) << 32) | static_cast<uint32_t>(h0.x);
    h_len = (static_cast<uint64_t>(static_cast<uint32_t>(h0.w)) << 32) | static_cast<uint32_t>(h0.z);
    h_kind = static_cast<uint32_t>(km);
    h_magic = static_cast<uint32_t>(km >> 32);
  }
  if (__ballot_sync(0xffffffffu, lane < chunk && h_magic != SW_SLOT_MAGIC)) c.err |= 1;

  // register window over the posted queue
  uint64_t wb = c.p_head;
  uint64_t w_tag = 0, w_mask = 0, w_buf = 0, w_cap = 0, w_op = 0;
  uint32_t w_valid = 0;
  auto load_pwin = [&]() {
    const uint64_t idx = wb + lane;
    w_valid = 0;
    if (idx < c.p_tail) {
      const uint64_t s = idx & PQM;
      w_valid = st->p_valid[s];
      w_tag = st->p_tag[s];
      w_mask = st->p_mask[s];
      w_buf = st->p_buf[s];
      w_cap = st->p_cap[s];
      w_op = st->p_op[s];
    }
  };
  if (c.p_count) load_pwin();
  const uint64_t cons0 = cons;
  bool blocked = false;
  uint32_t j0 = 0;
  // ---- pairing step: when the first k valid receives of the window accept every one of the next k arrivals
  // (all wildcard masks, or one common tag they all accept) arrival j goes to the j-th of them -- exactly what
  // the sequential rule (earliest-posted matching receive) yields.
  while (j0 < chunk && c.p_count) {
    while (__ballot_sync(0xffffffffu, w_valid != 0) == 0 && wb + 32 <= c.p_tail) {
      wb += 32;
      load_pwin();
    }
    const uint32_t V = __ballot_sync(0xffffffffu, w_valid != 0);
    if (!V) break;
    const uint32_t lt = (1u << lane) - 1;
    const uint32_t k = min(chunk - j0, static_cast<uint32_t>(__popc(V)));
    const uint32_t rnk = __popc(V & lt);
    const bool in_k = w_valid && rnk < k;
    bool compat = __ballot_sync(0xffffffffu, in_k && w_mask != 0) == 0;
    if (!compat) {
      const uint64_t T = sw_shfl64(h_tag, j0);
      const bool same = __ballot_sync(0xffffffffu, lane >= j0 && lane < j0 + k && h_tag != T) == 0;
      if (same) compat = __ballot_sync(0xffffffffu, in_k && !sw_tag_match(T, w_tag, w_mask)) == 0;
    }
    if (!compat) break;
    const int srcl = static_cast<int>(min(j0 + rnk, 31u));
    const uint64_t a_tag = sw_shfl64(h_tag, srcl), a_len = sw_shfl64(h_len, srcl);
    const uint64_t a_slot = sw_shfl64(my_slot, srcl);
    const uint32_t a_kind = __shfl_sync(0xffffffffu, h_kind, srcl);
    const bool a_rts = a_kind == SW_KIND_RTS;
    const bool trunc = a_len > w_cap;
    const uint64_t copy_len = trunc ? 0 : a_len;
    const bool small = in_k && !a_rts && copy_len <= SW_INLINE_DELIVER;
    const uint32_t small_m = __ballot_sync(0xffffffffu, small);
    // rendezvous requests the pull CTAs can serve (source in this process or already in the mapping table, 16 B
    // alignment): one lane per request builds its entry of the pull batch
    bool rfast = false;
    uint64_t r_src = 0, r_seq = 0;
    if (in_k && a_rts && !trunc && a.pq != nullptr && a.pull_ctas != 0 && !((w_valid >> 8) & SW_POST_HOSTPATH) &&
        !((sh.dead_mask >> ep) & 1) && sh.fin_ptr[ep] != 0) {
      const uint64_t rp = a_slot + SW_SLOT_HDR;   // the SwRts in the slot
      const int4 q0 = sw_ld16(reinterpret_cast<const void*>(rp + 64));    // alloc_base, alloc_size
      const int4 q1 = sw_ld16(reinterpret_cast<const void*>(rp + 80));    // src_ptr, send_seq
      const int4 q2 = sw_ld16(reinterpret_cast<const void*>(rp + 96));    // ctx_uuid, src_pid | src_dev
      const int4 q3 = sw_ld16(reinterpret_cast<const void*>(rp + 112));   // flags, buffer id
      auto u64of = [](int lo, int hi) { return (static_cast<uint64_t>(static_cast<uint32_t>(hi)) << 32) | static_cast<uint32_t>(lo); };
      const uint64_t alloc_base = u64of(q0.x, q0.y), alloc_size = u64of(q0.z, q0.w), src_ptr = u64of(q1.x, q1.y);
      const uint64_t uuid = u64of(q2.x, q2.y), rflags = u64of(q3.x, q3.y), buf_id = u64of(q3.z, q3.w);
      r_seq = u64of(q1.z, q1.w);
      if (!(rflags & SW_RTS_PINNED_SRC)) {
        if (uuid == a.ctx_uuid && static_cast<uint32_t>(q2.z) == a.pid) {
          r_src = src_ptr;
        } else if (a.map && buf_id && src_ptr >= alloc_base && src_ptr - alloc_base + a_len <= alloc_size) {
          const uint32_t home = sw_map_home(uuid, buf_id);
          for (uint32_t k = 0; k < SW_MAP_PROBE; k++) {
            const SwMapEnt* me = &a.map[(home + k) & (SW_MAP_SLOTS - 1)];
            const int4 key = sw_ld16(me);
            const uint64_t e_buf = u64of(key.z, key.w);
            if (!e_buf) break;   // entries are only ever added: an empty slot ends the probe
            if (e_buf == buf_id && u64of(key.x, key.y) == uuid) {
              const int4 val = sw_ld16(reinterpret_cast<const int4*>(me) + 1);
              if (u64of(val.x, val.y) == alloc_base) r_src = u64of(val.z, val.w) + (src_ptr - alloc_base);
              break;
            }
          }
        }
      }
      rfast = r_src != 0 && ((r_src | w_buf) & 15) == 0;
    }
    const uint32_t rfast_m = __ballot_sync(0xffffffffu, rfast);
    if (rfast_m) {
      const uint32_t cnt = __popc(rfast_m);
      if (c.pb_n + cnt > SW_PULL_JOBS) sw_res_flush_pull(st, sh, a, c, lane);
      // cumulative body bytes: inclusive scan over the participating lanes
      const uint64_t body = rfast ? (a_len & ~15ull) : 0;
      uint64_t scan = body;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint64_t up = sw_shfl64(scan, static_cast<int>(lane) - o < 0 ? static_cast<int>(lane) : static_cast<int>(lane) - o);
        if (static_cast<int>(lane) >= o) scan += up;
      }
      const uint64_t base_end = c.pb_n ? sh.pb_end[c.pb_n - 1] : 0;
      __syncwarp();
      if (rfast) {
        const uint32_t j = c.pb_n + __popc(rfast_m & lt);
        sh.pb_end[j] = base_end + scan;
        sh.pb_src[j] = r_src;
        sh.pb_dst[j] = w_buf;
        SwPullMeta m;
        m.op_id = w_op;
        m.tag = a_tag;
        m.len = a_len;
        m.fin_addr = sh.fin_ptr[ep] + 8ull * (r_seq % SW_FIN_SLOTS);
        m.fin_val = (r_seq << 2) | 1;
        sh.pb_meta[j] = m;
      }
      c.pb_n += cnt;
      c.pull_jobs += cnt;
      __syncwarp();
    }
    const uint32_t other_m = __ballot_sync(0xffffffffu, in_k && !small && !rfast);
    // small eager payloads: one lane per message, completion records in pairing order
    const uint32_t n_small = __popc(small_m);
    if (n_small) {
      sw_cq_room(sh, c, n_small);
      if (small) {
        sw_copy_lane(reinterpret_cast<uint8_t*>(w_buf), reinterpret_cast<const uint8_t*>(a_slot + SW_SLOT_HDR),
                     static_cast<uint32_t>(copy_len));
        sw_write_cqe(a.cq, c.cq_alloc + __popc(small_m & lt), w_op, a_tag, a_len, trunc ? SW_ERR_MESSAGE_TRUNCATED : SW_OK,
                     ((w_valid >> 8) & SW_POST_HOSTBUF) != 0);
      }
      c.cq_alloc += n_small;
    }
    if (in_k) {
      st->p_valid[(wb + lane) & PQM] = 0;
    }
    // everything else (larger eager payloads, rendezvous requests) one after the other, in pairing order
    uint32_t rest = other_m;
    while (rest) {
      const int L = __ffs(rest) - 1;
      rest &= rest - 1;
      const uint64_t o_tag = sw_shfl64(a_tag, L), o_len = sw_shfl64(a_len, L), o_slot = sw_shfl64(a_slot, L);
      const uint64_t o_buf = sw_shfl64(w_buf, L), o_cap = sw_shfl64(w_cap, L), o_op = sw_shfl64(w_op, L);
      const uint32_t o_valid = __shfl_sync(0xffffffffu, w_valid, L);
      const bool o_rts = __shfl_sync(0xffffffffu, static_cast<uint32_t>(a_rts), L) != 0;
      const uint32_t o_rank = __shfl_sync(0xffffffffu, rnk, L);
      if (o_rts) {
        sw_res_rts(st, sh, a, c, lane, o_slot + SW_SLOT_HDR, o_tag, o_len, epf, o_buf, o_cap, o_op, o_valid >> 8);
      } else {
        const bool t2 = o_len > o_cap;
        sw_res_deliver(st, sh, a, c, lane, o_slot + SW_SLOT_HDR, o_buf, t2 ? 0 : o_len, o_op, o_tag, o_len,
                       t2 ? SW_ERR_MESSAGE_TRUNCATED : SW_OK, 0, ep, cons + o_rank + 1, o_valid >> 8);
      }
    }
    if (in_k) w_valid = 0;
    c.p_count -= k;
    j0 += k;
    cons += k;
  }
  // ---- one arrival at a time
  for (uint32_t j = j0; j < chunk && !blocked; j++) {
    const uint64_t stag = sw_shfl64(h_tag, j), mlen = sw_shfl64(h_len, j);
    const uint32_t kind = __shfl_sync(0xffffffffu, h_kind, j);
    const uint64_t slot = sw_shfl64(my_slot, j);
    const uint64_t payload = slot + SW_SLOT_HDR;
    const bool is_rts = kind == SW_KIND_RTS;
    bool found = false;
    uint64_t f_buf = 0, f_cap = 0, f_op = 0;
    uint32_t f_valid = 0;
    if (c.p_count) {
      while (__ballot_sync(0xffffffffu, w_valid != 0) == 0 && wb + 32 <= c.p_tail) {
        wb += 32;
        load_pwin();
      }
      const bool hit = w_valid && sw_tag_match(stag, w_tag, w_mask);
      uint32_t bal = __ballot_sync(0xffffffffu, hit);
      if (bal) {
        const int L = __ffs(bal) - 1;
        f_buf = sw_shfl64(w_buf, L);
        f_cap = sw_shfl64(w_cap, L);
        f_op = sw_shfl64(w_op, L);
        f_valid = __shfl_sync(0xffffffffu, w_valid, L);
        if (static_cast<int>(lane) == L) {
          w_valid = 0;
          st->p_valid[(wb + L) & PQM] = 0;
        }
        found = true;
      } else {
        for (uint64_t b = wb + 32; b < c.p_tail && !found; b += 32) {
          const uint64_t idx = b + lane;
          uint32_t v = 0;
          uint64_t t = 0, m = 0;
          if (idx < c.p_tail) {
            v = st->p_valid[idx & PQM];
            t = st->p_tag[idx & PQM];
            m = st->p_mask[idx & PQM];
          }
          const bool h2 = v && sw_tag_match(stag, t, m);
          bal = __ballot_sync(0xffffffffu, h2);
          if (bal) {
            const int L = __ffs(bal) - 1;
            uint64_t bf = 0, cp = 0, op = 0;
            if (static_cast<int>(lane) == L) {
              bf = st->p_buf[idx & PQM];
              cp = st->p_cap[idx & PQM];
              op = st->p_op[idx & PQM];
              st->p_valid[idx & PQM] = 0;
            }
            f_buf = sw_shfl64(bf, L);
            f_cap = sw_shfl64(cp, L);
            f_op = sw_shfl64(op, L);
            f_valid = __shfl_sync(0xffffffffu, v, L);
            found = true;
          }
        }
      }
    }
    if (found) {
      c.p_count--;
      if (is_rts) {
        sw_res_rts(st, sh, a, c, lane, payload, stag, mlen, epf, f_buf, f_cap, f_op, f_valid >> 8);
      } else {
        const bool trunc = mlen > f_cap;
        sw_res_deliver(st, sh, a, c, lane, payload, f_buf, trunc ? 0 : mlen, f_op, stag, mlen,
                       trunc ? SW_ERR_MESSAGE_TRUNCATED : SW_OK, 0, ep, cons + 1, f_valid >> 8);
      }
    } else {
      // unexpected: park the payload (or the RTS descriptor) on the heap -- copied by this warp at once, so the
      // slot is free again and a later receive finds the bytes in place
      const uint64_t need = is_rts ? sizeof(SwRts) : mlen;
      const bool big = need > SW_HEAP_SMALL_BYTES;
      const bool have = big ? (c.n_free_big > 0) : (c.n_free_small > 0);
      if (!have || c.u_tail - c.u_head >= SW_UQ_CAP) {
        blocked = true;   // back-pressure: the message stays in its ring slot until receives free the heap
        c.stalled = true;
        break;
      }
      uint32_t blk = 0;
      if (lane == 0) blk = big ? st->free_big[c.n_free_big - 1] : st->free_small[c.n_free_small - 1];
      blk = __shfl_sync(0xffffffffu, blk, 0);
      if (big)
        c.n_free_big--;
      else
        c.n_free_small--;
      const uint64_t haddr = big ? reinterpret_cast<uint64_t>(st->heap_big) + uint64_t(blk) * SW_HEAP_BIG_BYTES
                                 : reinterpret_cast<uint64_t>(st->heap_small) + uint64_t(blk) * SW_HEAP_SMALL_BYTES;
      sw_copy(reinterpret_cast<uint8_t*>(haddr), reinterpret_cast<const uint8_t*>(payload), need, lane, 32);
      if (lane == 0) {
        const uint64_t s = c.u_tail & UQM;
        st->u_tag[s] = stag;
        st->u_len[s] = mlen;
        st->u_data[s] = haddr;
        st->u_blk[s] = blk;
        st->u_meta[s] = SW_UMETA_VALID | (big ? SW_UMETA_BIG : 0) | (is_rts ? SW_UMETA_RTS : 0) | (epf & SW_UMETA_EPMASK);
      }
      c.u_tail++;
      c.u_count++;
      __syncwarp();
    }
    cons++;
  }
  if (c.p_count) {
    while (__ballot_sync(0xffffffffu, w_valid != 0) == 0 && wb + 32 <= c.p_tail) {
      wb += 32;
      load_pwin();
    }
    c.p_head = wb;
  } else {
    c.p_head = c.p_tail;
  }
  const uint32_t used = static_cast<uint32_t>(cons - cons0);
  if (used) {
    if (lane == 0) sh.cons[ep] = cons;
    __syncwarp();
    c.arrivals += used;
    // Credits cost a system-scope release (~1.5 us): while messages keep coming they are returned a quarter of
    // the ring at a time; the matcher's main loop returns the rest as soon as an iteration finds nothing new.
    // Slots whose payload a helper still reads stay owned until that job retires.
    if (sh.pend_cnt[ep] == 0 && lane == 0) sh.releasable[ep] = cons;
    __syncwarp();
    if (sh.releasable[ep] - sh.credit[ep] >= (smask + 1) / 4) sw_publish_credit(st, sh, ep, sh.releasable[ep], lane);
  }
  return used;
}

// compaction of a queue when tombstones dominate (more than half its capacity between head and tail): the valid
// entries move down to the head in their order, the tail follows them and the vacated entries are cleared
__device__ __forceinline__ void sw_res_compact(SwMatchState* __restrict__ st, SwResCtx& c, const uint32_t lane) {
  const uint64_t PQM = SW_PQ_CAP - 1, UQM = SW_UQ_CAP - 1;
  if (c.p_tail - c.p_head > SW_PQ_CAP / 2) {
    uint64_t j = c.p_head;
    for (uint64_t b = c.p_head; b < c.p_tail; b += 32) {
      const uint64_t idx = b + lane;
      uint32_t v = 0;
      uint64_t t = 0, m = 0, bf = 0, cp = 0, op = 0;
      if (idx < c.p_tail) {
        const uint64_t s = idx & PQM;
        v = st->p_valid[s];
        if (v) {
          t = st->p_tag[s];
          m = st->p_mask[s];
          bf = st->p_buf[s];
          cp = st->p_cap[s];
          op = st->p_op[s];
        }
      }
      const uint32_t bal = __ballot_sync(0xffffffffu, v != 0);
      const uint64_t pos = j + __popc(bal & ((1u << lane) - 1));
      __syncwarp();
      if (v) {
        const uint64_t s = pos & PQM;
        st->p_tag[s] = t;
        st->p_mask[s] = m;
        st->p_buf[s] = bf;
        st->p_cap[s] = cp;
        st->p_op[s] = op;
        st->p_valid[s] = v;
      }
      j += __popc(bal);
      __syncwarp();
    }
    for (uint64_t idx = j + lane; idx < c.p_tail; idx += 32) st->p_valid[idx & PQM] = 0;
    c.p_tail = j;
    __syncwarp();
  }
  if (c.u_tail - c.u_head > SW_UQ_CAP / 2) {
    uint64_t j = c.u_head;
    for (uint64_t b = c.u_head; b < c.u_tail; b += 32) {
      const uint64_t idx = b + lane;
      uint32_t meta = 0, blk = 0;
      uint64_t t = 0, l = 0, dta = 0;
      if (idx < c.u_tail) {
        const uint64_t s = idx & UQM;
        meta = st->u_meta[s];
        if (meta & SW_UMETA_VALID) {
          t = st->u_tag[s];
          l = st->u_len[s];
          dta = st->u_data[s];
          blk = st->u_blk[s];
        }
      }
      const bool v = (meta & SW_UMETA_VALID) != 0;
      const uint32_t bal = __ballot_sync(0xffffffffu, v);
      const uint64_t pos = j + __popc(bal & ((1u << lane) - 1));
      __syncwarp();
      if (v) {
        const uint64_t s = pos & UQM;
        st->u_tag[s] = t;
        st->u_len[s] = l;
        st->u_data[s] = dta;
        st->u_blk[s] = blk;
        st->u_meta[s] = meta;
      }
      j += __popc(bal);
      __syncwarp();
    }
    for (uint64_t idx = j + lane; idx < c.u_tail; idx += 32) st->u_meta[idx & UQM] = 0;
    c.u_tail = j;
    __syncwarp();
  }
}

// ------------------------------------------------------------------ the control kernel
__global__ void __launch_bounds__(SW_PROG_THREADS, 1) sw_progress_kernel(const __grid_constant__ SwProgArgs a) {
  __shared__ SwProgShared sh;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  SwMatchState* st = a.st;
  const long long clk0 = clock64();
  // ---- set-up: ring geometry and cursors from the match state
  for (uint32_t e = threadIdx.x; e < SW_MAX_EPS; e += blockDim.x) {
    sh.ring_base[e] = st->ring_base[e];
    sh.ring_mask[e] = st->ring_slots[e] ? st->ring_slots[e] - 1 : 0;
    sh.ring_gen[e] = st->ring_gen[e] & SW_EP_GEN_MASK;
    sh.fin_ptr[e] = st->fin_ptr[e];
    sh.cons[e] = st->ring_cons[e];
    sh.credit[e] = st->ring_cons[e];
    sh.releasable[e] = st->ring_cons[e];
    sh.pend_cnt[e] = 0;
  }
  if (threadIdx.x == 0) {
    sh.post_tail = sh.post_head = st->post_consumed;
    sh.send_tail = sh.send_done = sh.send_base = st->send_consumed;
    sh.job_tail = 0;
    sh.cq_head = a.ctl->cq_head;
    sh.cqr_head = a.ctl->cqr_head;
    sh.hr_head = a.ctl->hr_head;
    sh.dead_mask = a.ctl->dead_mask;
    sh.host_epoch = a.ctl->host_epoch;
    sh.active_clk = clk0;
    sh.exit_req = 0;
    sh.helpers_exit = 0;
    for (uint32_t h = 0; h < SW_PROG_HELPERS; h++) sh.helper_done[h] = 0;
  }
  __syncthreads();

  if (warp == 0) {
    // ================================================================ matcher
    SwResCtx c;
    c.p_head = st->p_head;
    c.p_tail = st->p_tail;
    c.u_head = st->u_head;
    c.u_tail = st->u_tail;
    c.p_count = st->p_count;
    c.u_count = st->u_count;
    c.n_free_small = st->n_free_small;
    c.n_free_big = st->n_free_big;
    c.cq_alloc = st->cq_alloc;
    c.hr_alloc = st->hr_alloc;
    c.pull_jobs = st->pull_jobs;
    c.arrivals = st->arrivals;
    c.post_head = st->post_consumed;
    c.jobs_emitted = 0;
    c.pend_head = c.pend_tail = 0;
    c.pb_n = 0;
    c.err = 0;
    c.last_slot = nullptr;
    c.last_ticket = 0;
    uint64_t echoed = ~0ull, iters = 0;
    SwPullSlot* pb_prev = nullptr;   // the batch this matcher published last
    uint64_t pb_prev_ticket = 0;
    uint32_t pb_wait = 0;
    uint32_t rr = st->rr_ep;
    const uint32_t n_eps = a.n_eps;
    for (;;) {
      bool did = false;
      c.stalled = false;
      // The host bumps host_epoch AFTER changing dead_mask and waits for the echo: read the epoch before anything
      // of this iteration looks at dead_mask, echo it once the iteration (and what it handed on) is done.
      const uint64_t he = sh.host_epoch;
      __threadfence_block();
      sw_res_compact(st, c, lane);
      // ---- new receives staged by the link warp
      for (;;) {
        const uint64_t pt = sh.post_tail;
        if (c.post_head >= pt) break;
        __threadfence_block();
        const uint32_t n = static_cast<uint32_t>(min(static_cast<uint64_t>(32), pt - c.post_head));
        sw_res_posts(st, sh, a, c, lane, n);
        c.post_head += n;
        if (lane == 0) sh.post_head = c.post_head;
        did = true;
      }
      const bool leaving = sh.exit_req != 0;
      // ---- arrivals: every ring, round robin; a busy ring is drained in a few steps before the next one
      if (!leaving) {
        for (uint32_t e = 0; e < n_eps; e++) {
          const uint32_t ep = (rr + e) % n_eps;
          if (!sh.ring_base[ep]) continue;
          for (int rep = 0; rep < 4; rep++) {
            const uint32_t used = sw_res_arrivals(st, sh, a, c, lane, ep);
            did |= used != 0;
            if (used < 32) break;
          }
        }
        rr++;
      }
      if (c.pb_n) {
        // Publish the batch at once when the pull CTAs have nothing of ours to do; while the previous batch is still
        // being copied, let this one grow (bounded: 32 messages or a few iterations) -- batches then size
        // themselves to the load, and a lone message never waits.
        bool go = c.pb_n >= 32 || !pb_prev || ++pb_wait > 6;
        if (!go) {
          uint64_t fin = 0, seq = 0;
          if (lane == 0) {
            seq = sw_ld_acquire_gpu(&pb_prev->seq);
            fin = *reinterpret_cast<volatile uint64_t*>(&pb_prev->fin_seq);
          }
          seq = sw_shfl64(seq, 0);
          fin = sw_shfl64(fin, 0);
          go = seq != pb_prev_ticket + 1 || fin == seq;   // slot reused, or completed
        }
        if (go) {
          sw_res_flush_pull(st, sh, a, c, lane);
          pb_prev = c.last_slot;
          pb_prev_ticket = c.last_ticket;
          pb_wait = 0;
        }
      }
      if (c.pend_head != c.pend_tail) sw_retire(st, sh, c, lane, false);
      if (he != echoed) {   // nothing matched under an older dead_mask is left in this warp
        echoed = he;
        if (lane == 0) {
          __threadfence_system();
          a.ctl->dev_epoch = he;
        }
      }
      iters++;
      if (leaving) {
        // the link warp stops staging before it raises exit_req: once nothing staged is left, leave
        if (c.post_head >= sh.post_tail) break;
        continue;
      }
      if (did) {
        if (lane == 0) sh.active_clk = clock64();
      } else {
        // quiet: return the credits that were held back
        for (uint32_t e = 0; e < n_eps; e++)
          if (sh.ring_base[e] && sh.releasable[e] != sh.credit[e]) sw_publish_credit(st, sh, e, sh.releasable[e], lane);
        __nanosleep(40);
      }
    }
    // ---- wind down: helpers finish, every deferred release happens, state goes back to device memory
    sw_res_flush_pull(st, sh, a, c, lane);
    sw_retire(st, sh, c, lane, true);
    for (uint32_t e = 0; e < n_eps; e++)
      if (sh.ring_base[e]) sw_publish_credit(st, sh, e, sh.cons[e], lane);   // every helper has finished
    __syncwarp();
    for (uint32_t e = lane; e < SW_MAX_EPS; e += 32)
      if (sh.ring_base[e]) st->ring_cons[e] = sh.cons[e];   // (a ring attached while this launch ran is not ours to touch)
    if (lane == 0) {
      st->p_head = c.p_head;
      st->p_tail = c.p_tail;
      st->u_head = c.u_head;
      st->u_tail = c.u_tail;
      st->p_count = c.p_count;
      st->u_count = c.u_count;
      st->n_free_small = c.n_free_small;
      st->n_free_big = c.n_free_big;
      st->cq_alloc = c.cq_alloc;
      st->hr_alloc = c.hr_alloc;
      st->pull_jobs = c.pull_jobs;
      st->arrivals = c.arrivals;
      st->post_consumed = c.post_head;
      st->rr_ep = rr;
      a.ctl->pull_jobs = c.pull_jobs;
      a.ctl->arrivals = c.arrivals;
      a.ctl->n_posted = c.p_count;
      a.ctl->n_unexp = c.u_count;
      a.ctl->err = a.ctl->err | c.err;
      a.ctl->stalled = c.stalled ? 1 : 0;
      a.ctl->iterations = a.ctl->iterations + iters;
      __threadfence_block();
      sh.helpers_exit = 1;
    }
  } else if (warp == 1) {
    // ================================================================ host link
    // Every look at host memory costs a PCIe round trip (~1 us) and a thread's system-scope loads do not overlap:
    // each round is ONE warp-wide load instruction (a lane per 16-byte unit), then one more for the entries.
    const long long linger_clk = static_cast<long long>(a.linger_us) * a.clk_mhz;
    const long long life_clk = static_cast<long long>(a.max_life_us) * a.clk_mhz;
    uint64_t staged = sh.post_tail, sstaged = sh.send_tail;
    uint64_t he_prev = sh.host_epoch;
    uint64_t dbg_n = 0, dbg_stage = 0, dbg_rounds = 0;
    bool leaving = false;
    const uint8_t* ctl_bytes = reinterpret_cast<const uint8_t*>(const_cast<const SwProgCtl*>(a.ctl));
    auto u64of = [](int lo, int hi) { return (static_cast<uint64_t>(static_cast<uint32_t>(hi)) << 32) | static_cast<uint32_t>(lo); };
    for (;;) {
      // units of the two host->kernel lines: 0 {post_tail, cq_head} 1 {cqr_head, hr_head} 2 {send_tail, -}
      //                                      4 {stop, dead_mask} 5 {host_epoch, -}
      // lanes 6 .. 20: the units of the next put entry the host will write (or has written), speculatively
      int4 v = make_int4(0, 0, 0, 0);
      if (lane < 6) v = sw_ld16_sys(ctl_bytes + 16 * lane);
      else if (lane < 6 + SW_SEND_UNITS) v = sw_ld16_sys(&a.sends[sstaged % SW_SEND_RING].u[lane - 6][0]);
      auto unit_lo = [&](int u) { return u64of(__shfl_sync(0xffffffffu, v.x, u), __shfl_sync(0xffffffffu, v.y, u)); };
      auto unit_hi = [&](int u) { return u64of(__shfl_sync(0xffffffffu, v.z, u), __shfl_sync(0xffffffffu, v.w, u)); };
      const uint64_t host_tail = unit_lo(0), cq_head = unit_hi(0), cqr_head = unit_lo(1), hr_head = unit_hi(1);
      const uint64_t host_stail = unit_lo(2), stop = unit_lo(4), dead_mask = unit_hi(4), he = unit_lo(5);
      if (lane == 0) {
        sh.cq_head = cq_head;
        if (cqr_head != sh.cqr_head) {
          sh.cqr_head = cqr_head;
          st->cqr_head = cqr_head;   // the pull CTAs read the device copy
        }
        sh.hr_head = hr_head;
        sh.dead_mask = dead_mask;
        // The epoch handed to the matcher is the one read in the PREVIOUS round: this round's dead_mask was
        // requested after that read had returned, so it is at least as new as the epoch that vouches for it.
        __threadfence_block();
        sh.host_epoch = he_prev;
      }
      he_prev = he;
      dbg_rounds++;
      if (leaving) {
        // the matcher winds down (it may still need room in the completion rings): keep the host's cursors fresh;
        // the put warp finishes what is staged
        if (sh.helpers_exit && sh.send_done == sstaged) {
          if (lane == 0) {
            a.ctl->dbg[0] = a.ctl->dbg[0] + dbg_n;
            a.ctl->dbg[1] = a.ctl->dbg[1] + dbg_stage;
            a.ctl->dbg[4] = a.ctl->dbg[4] + dbg_rounds;
            a.ctl->dbg[5] = a.ctl->dbg[5] + static_cast<uint64_t>(clock64() - clk0);
          }
          break;
        }
        continue;
      }
      // ---- stage new receives: up to 32 per round, 16-byte units spread over the lanes (3 units per entry)
      const uint64_t consumed = sh.post_head;
      const uint64_t room = SW_SPOST_RING - (staged - consumed);
      uint64_t n = host_tail - staged;
      if (n > room) n = room;
      if (n > 32) n = 32;
      for (uint32_t x = lane; x < 3 * n; x += 32) {
        const uint32_t e = x / 3, u = x % 3;
        const int4* src = reinterpret_cast<const int4*>(&a.posts[(staged + e) % SW_POST_RING]);
        reinterpret_cast<int4*>(&sh.posts[(staged + e) % SW_SPOST_RING])[u] = sw_ld16_sys(src + u);
      }
      __syncwarp();
      if (n) {
        staged += n;
        if (lane == 0) {
          __threadfence_block();
          sh.post_tail = staged;
          a.ctl->post_head = staged;   // the host may reuse these ring entries
        }
      }
      // ---- stage puts for the put warp.  The entry read with the control words is taken when all its units carry
      //      its stamp (the host's cursor may not have been seen to cover it yet: the entry is complete all the same);
      //      what the cursor announces beyond it costs one more round trip, two entries per load instruction.
      const uint64_t sdone = sh.send_done;
      uint64_t sroom = SW_SSEND_RING - (sstaged - sdone);
      const long long t_seen = clock64();
      auto stage_unit = [&](uint64_t idx, uint32_t unit, const int4& d) {
        uint32_t* dst = reinterpret_cast<uint32_t*>(&sh.sends[idx % SW_SSEND_RING]) + 3 * unit;
        dst[0] = static_cast<uint32_t>(d.x);
        dst[1] = static_cast<uint32_t>(d.y);
        if (3 * unit + 2 < SW_SEND_WORDS) dst[2] = static_cast<uint32_t>(d.z);
      };
      const bool is_unit = lane >= 6 && lane < 6 + SW_SEND_UNITS;
      const bool stamped = !is_unit || static_cast<uint32_t>(v.w) == sw_send_stamp(sstaged);
      uint64_t ns = 0;
      if (__all_sync(0xffffffffu, stamped) && sroom) {
        if (is_unit) stage_unit(sstaged, lane - 6, v);
        ns = 1;
      }
      if (host_stail > sstaged + ns) {
        uint64_t more = host_stail - (sstaged + ns);
        if (more > sroom - ns) more = sroom - ns;
        for (uint64_t base = 0; base < more; base += 2) {
          const uint32_t e = lane / SW_SEND_UNITS, u = lane % SW_SEND_UNITS;
          if (e < 2 && base + e < more) {
            const uint64_t idx = sstaged + ns + base + e;
            stage_unit(idx, u, sw_ld16_sys(&a.sends[idx % SW_SEND_RING].u[u][0]));
          }
        }
        ns += more;
      }
      __syncwarp();
      if (ns) {
        sstaged += ns;
        if (lane == 0) {
          __threadfence_block();
          sh.send_tail = sstaged;
          a.ctl->send_head = sstaged;
          const long long ts = clock64();
          sh.active_clk = ts;
          sh.t_staged = ts;
          dbg_stage += ts - t_seen;
          dbg_n += ns;
        }
      }
      const long long now = clock64();
      const bool idle = n == 0 && ns == 0 && host_tail == staged && staged == sh.post_head && host_stail <= sstaged &&
                        sstaged == sh.send_done && now - sh.active_clk > linger_clk;
      if (stop || idle || now - clk0 > life_clk) {
        if (lane == 0) {
          a.ctl->exit_reason = stop ? 1 : (idle ? 2 : 3);
          a.ctl->life_us = static_cast<uint64_t>(now - clk0) / (a.clk_mhz ? a.clk_mhz : 1);
          __threadfence_block();
          sh.exit_req = 1;   // after the last staging store: the matcher drains what is staged and leaves
        }
        leaving = true;
      }
    }
  } else if (warp == 2) {
    // ================================================================ puts handed over by the host
    // (the sender side of ucp_tag_send_nbx for small batches while this kernel is resident: no launch)
    uint64_t i = sh.send_base;
    uint64_t dbg_put = 0, dbg_pub = 0;
    for (;;) {
      uint64_t tail;
      while ((tail = sh.send_tail) <= i) {
        if (sh.helpers_exit) {   // raised after the link warp has stopped staging: nothing is left behind
          if (lane == 0) {
            a.ctl->dbg[2] = a.ctl->dbg[2] + dbg_put;
            a.ctl->dbg[3] = a.ctl->dbg[3] + dbg_pub;
          }
          goto out;
        }
        __nanosleep(20);
      }
      __threadfence_block();
      const uint32_t n = static_cast<uint32_t>(tail - i < 32 ? tail - i : 32);
      // a lane per put when the payload is small (inline in the entry, or <= 256 B): payload, then the header
      // with release semantics; larger payloads by the whole warp, one after the other
      const SwSendEnt* e = &sh.sends[(i + lane) % SW_SSEND_RING];
      SwPutDesc d;
      d.src = d.dst = d.tag = d.seq = d.msg_len = 0;
      d.len = d.kind = 0;
      if (lane < n) d = e->d;
      const bool same_gpu = (d.kind & SW_KIND_SAME_GPU) != 0;
      d.kind &= ~SW_KIND_SAME_GPU;
      auto put_header = [&]() {
        uint8_t* hdr = reinterpret_cast<uint8_t*>(d.dst);
        if (same_gpu) sw_put_header_same_gpu(hdr, d.tag, d.msg_len, d.seq, d.kind);
        else sw_put_header(hdr, d.tag, d.msg_len, d.seq, d.kind);
      };
      const bool mine = lane < n && (d.src == 0 || d.len <= 256);
      if (mine) {
        uint8_t* slot = reinterpret_cast<uint8_t*>(d.dst);
        if (d.src) {
          sw_copy_lane(slot + SW_SLOT_HDR, reinterpret_cast<const uint8_t*>(d.src), d.len);
        } else {
          for (uint32_t k = 0; k * 16 < d.len; k++) sw_st16(slot + SW_SLOT_HDR + 16 * k, reinterpret_cast<const int4*>(e->inl)[k]);
        }
        put_header();
      }
      const uint32_t big = __ballot_sync(0xffffffffu, lane < n && !mine);
      uint32_t rest = big;
      while (rest) {
        const int L = __ffs(rest) - 1;
        rest &= rest - 1;
        const uint64_t src = sw_shfl64(d.src, L), dst = sw_shfl64(d.dst, L);
        const uint32_t len = __shfl_sync(0xffffffffu, d.len, L);
        sw_copy(reinterpret_cast<uint8_t*>(dst) + SW_SLOT_HDR, reinterpret_cast<const uint8_t*>(src), len, lane, 32);
        __syncwarp();
        if (static_cast<int>(lane) == L) put_header();
      }
      __syncwarp();
      i += n;
      if (lane == 0) {
        const long long t1 = clock64();
        sw_st_release_sys(const_cast<uint64_t*>(&a.ctl->send_done), i);   // every header before it: the host rings the doorbell on it
        __threadfence_block();
        sh.send_done = i;
        const long long t2 = clock64();
        sh.active_clk = t2;
        dbg_put += t1 - sh.t_staged;
        dbg_pub += t2 - t1;
      }
      __syncwarp();
    }
  } else {
    // ================================================================ helpers: larger eager payloads
    const uint32_t h = warp - 2 - SW_PROG_PUTTERS;
    uint64_t i = h;
    uint32_t done = 0;
    for (;;) {
      while (sh.job_tail <= i) {
        if (sh.helpers_exit) goto out;
        __nanosleep(30);
      }
      __threadfence_block();
      {
        const SwDJob j = sh.jobs[i % SW_DJOB_RING];
        sw_copy(reinterpret_cast<uint8_t*>(j.dst), reinterpret_cast<const uint8_t*>(j.src), j.len, lane, 32);
        __syncwarp();
        if (lane == 0) {
          sw_write_cqe(a.cq, j.cq_idx, j.op_id, j.tag, j.msg_len, j.status, (j.pad & SW_POST_HOSTBUF) != 0);
          sh.helper_done[h] = ++done;
        }
        __syncwarp();
      }
      i += SW_PROG_HELPERS;
    }
  }
out:
  __syncthreads();
  if (threadIdx.x == 0) {
    st->send_consumed = sh.send_done;
    __threadfence_system();
    a.ctl->exit_seq = a.launch_seq;
  }
}

// ------------------------------------------------------------------ the pull kernel
struct SwPullArgs {
  SwPullQueue* q;
  SwPullCtl* ctl;          // pinned host
  uint64_t launch_seq;
  uint32_t stage_bytes, nstages;
  uint32_t linger_us, max_life_us, clk_mhz, pad;
};

// ---- completion of a batch (CTA 0 of the pull kernel, a full warp, no copy traffic of its own): tails, completion
// records into the receiving worker's rendezvous CQ, FIN words into the senders' control blocks, statistics.
// The copy CTAs signal with plain atomics (their bulk stores have completed when they do); the fences are here.
__device__ __forceinline__ void sw_pull_finalize(SwPullQueue* q, SwPullSlot* sp, uint32_t lane) {
  volatile SwPullSlot* s = sp;   // written by a matcher on another SM: never from this SM's L1
  const uint32_t n = s->njobs;
  const uint64_t t_copied = sw_globaltimer();
  for (uint32_t j = lane; j < n; j += 32) {
    const uint64_t len = s->meta[j].len, body = len & ~15ull;
    for (uint64_t k = body; k < len; k++)
      reinterpret_cast<uint8_t*>(s->dst[j])[k] = reinterpret_cast<const volatile uint8_t*>(s->src[j])[k];
  }
  __syncwarp();
  if (n) {
    SwCqEnt* ring = reinterpret_cast<SwCqEnt*>(s->cqr_ring);
    uint64_t base = 0;
    if (lane == 0) {
      base = atomicAdd(reinterpret_cast<unsigned long long*>(s->cqr_alloc), static_cast<unsigned long long>(n));
      // room: the device copy of the host's cursor is refreshed by the worker's control kernel; when that one is
      // not running, read the host's word itself
      while (base + n - sw_ld_relaxed_sys(reinterpret_cast<const void*>(s->cqr_head_dev)) > SW_CQ_RING) {
        const uint64_t hh = sw_ld_relaxed_sys(reinterpret_cast<const void*>(s->cqr_head_host));
        if (base + n - hh <= SW_CQ_RING) break;
        __nanosleep(500);
      }
    }
    base = sw_shfl64(base, 0);
    for (uint32_t j = lane; j < n; j += 32) {
      SwCqEnt* e = &ring[(base + j) % SW_CQ_RING];
      e->op_id = s->meta[j].op_id;
      e->tag = s->meta[j].tag;
      e->len = s->meta[j].len;
    }
    // ONE system-scope fence per batch: the chunks (complete before their CTAs counted them), the tails and the
    // bodies of the records, before the pass words and the FIN words
    __threadfence_system();
    for (uint32_t j = lane; j < n; j += 32) {
      const uint64_t idx = base + j;
      sw_st_relaxed_sys(&ring[idx % SW_CQ_RING].status, static_cast<uint64_t>(sw_ring_pass(idx, SW_CQ_RING)) << 32);
      if (s->meta[j].fin_addr) sw_st_relaxed_sys(reinterpret_cast<void*>(s->meta[j].fin_addr), s->meta[j].fin_val);
    }
  }
  __syncwarp();
  if (lane == 0) {
    // statistics: bytes and the union of the batches' active intervals
    const uint64_t t1 = sw_globaltimer(), t0 = s->t_first ? s->t_first : t_copied;
    if (t1 > q->last_end) {   // (only this warp writes the statistics)
      q->busy_ns += t1 - (t0 > q->last_end ? t0 : q->last_end);
      q->last_end = t1;
    }
    q->bytes += s->total;
    q->batches += 1;
    q->jobs += n;
    if (s->t_pub && t0 >= s->t_pub) q->pickup_ns += t0 - s->t_pub;
    if (t_copied >= t0) q->copy_ns += t_copied - t0;
    q->fin_ns += t1 - t_copied;
  }
}

// A slot is free again when every copy CTA has left the batch (no more chunks for it) and CTA 0 has completed it.
__device__ __forceinline__ void sw_pull_retire(SwPullSlot* s, uint64_t ticket) {
  const uint32_t r = atomicAdd(&s->retire, 1u) + 1;
  if (r == gridDim.x) sw_st_release_gpu(&s->free_seq, ticket + 1);
}

__global__ void __launch_bounds__(64) sw_pull_kernel(const __grid_constant__ SwPullArgs a) {
  extern __shared__ __align__(128) uint8_t sw_smem[];
  __shared__ __align__(8) uint64_t full[SW_BULK_MAX_STAGES];
  // batch descriptors, double-buffered: warp 1 of a copy CTA fetches batch b + 1 (a lane per message) while
  // thread 0 streams batch b
  __shared__ uint64_t s_endb[2][SW_PULL_JOBS], s_srcb[2][SW_PULL_JOBS], s_dstb[2][SW_PULL_JOBS];
  __shared__ uint64_t s_chunk[2], s_total[2];
  __shared__ uint32_t s_nchunks[2], s_exitb[2];
  __shared__ volatile uint64_t s_ready;      // descriptors of every ticket below this one are in shared memory
  __shared__ volatile uint64_t s_released;   // thread 0 has finished with every ticket below this one
  SwPullQueue* q = a.q;
  const uint64_t first = sw_ld_acquire_gpu(&q->start);   // first ticket of this launch
  const long long clk0 = clock64();
  const long long linger_clk = static_cast<long long>(a.linger_us) * a.clk_mhz;
  const long long life_clk = static_cast<long long>(a.max_life_us) * a.clk_mhz;

  if (blockIdx.x == 0) {
    // ================================================================ CTA 0: completions, and when the grid leaves
    if (threadIdx.x >= 32) return;   // one warp
    const uint32_t lane = threadIdx.x;
    uint64_t finalized = 0;        // batches of this launch completed so far
    uint64_t exit_ticket = 0;
    bool exit_taken = false, exit_published = false;
    long long last_work = clk0;
    uint32_t polls = 0;
    for (;;) {
      // ---- a batch is complete when every chunk has been counted
      bool did = false;
      for (uint32_t k = 0; k < SW_PULL_SLOTS; k++) {
        SwPullSlot* s = &q->slot[k];
        uint32_t ready = 0;
        if (lane == 0) {
          const uint64_t seq = sw_ld_acquire_gpu(&s->seq);
          // published, of this launch, not an EXIT marker, not completed yet, all chunks counted
          if (seq > first && !s->exit && s->fin_seq != seq && (!exit_taken || seq - 1 < exit_ticket) &&
              *reinterpret_cast<volatile uint32_t*>(&s->done_chunks) == *reinterpret_cast<volatile uint32_t*>(&s->nchunks))
            ready = 1;
        }
        ready = __shfl_sync(0xffffffffu, ready, 0);
        if (!ready) continue;
        sw_pull_finalize(q, s, lane);
        if (lane == 0) {
          s->fin_seq = s->seq;
          sw_pull_retire(s, s->seq - 1);
        }
        __syncwarp();
        finalized++;
        did = true;
      }
      const long long now = clock64();
      if (did) last_work = now;
      // ---- leaving: take a ticket from the counter the matchers use -- every batch before it is served by this
      // grid, every batch after it by the next launch -- and publish the EXIT batch as soon as that ticket's
      // slot is free; the copy CTAs leave when they reach it, this CTA when everything before it is completed
      if (!exit_published && (++polls & 3) == 0) {
        uint32_t go = 0;
        if (lane == 0) {
          if (!exit_taken) {
            const bool stop = sw_ld_relaxed_sys(const_cast<const uint64_t*>(&a.ctl->stop)) != 0;
            const uint64_t alloc = *reinterpret_cast<volatile uint64_t*>(&q->alloc);
            const bool quiet = alloc == first + finalized;   // nothing allocated that is not completed
            if (stop || (quiet && now - last_work > linger_clk) || now - clk0 > life_clk) {
              exit_ticket = atomicAdd(reinterpret_cast<unsigned long long*>(&q->alloc), 1ull);
              exit_taken = true;
            }
          }
          if (exit_taken) {
            SwPullSlot* xs = &q->slot[exit_ticket % SW_PULL_SLOTS];
            const uint64_t want = exit_ticket >= SW_PULL_SLOTS ? exit_ticket - SW_PULL_SLOTS + 1 : 0;
            if (sw_ld_acquire_gpu(&xs->free_seq) == want) {
              xs->njobs = 0;
              xs->nchunks = 0;
              xs->exit = 1;
              xs->total = 0;
              xs->next_chunk = xs->done_chunks = xs->retire = 0;
              __threadfence();
              sw_st_release_gpu(&xs->seq, exit_ticket + 1);
              go = 2;
            } else {
              go = 1;
            }
          }
        }
        go = __shfl_sync(0xffffffffu, go, 0);
        exit_taken = go != 0;
        exit_published = go == 2;
        exit_ticket = sw_shfl64(exit_ticket, 0);
      }
      if (exit_published && first + finalized == exit_ticket) break;
      if (!did) __nanosleep(100);
    }
    // the EXIT batch: every CTA passes it once; the last one hands the next launch its first ticket
    if (lane == 0) {
      SwPullSlot* s = &q->slot[exit_ticket % SW_PULL_SLOTS];
      a.ctl->bytes = q->bytes;
      a.ctl->busy_ns = q->busy_ns;
      a.ctl->batches = q->batches;
      a.ctl->jobs = q->jobs;
      a.ctl->pickup_ns = q->pickup_ns;
      a.ctl->copy_ns = q->copy_ns;
      a.ctl->fin_ns = q->fin_ns;
      __threadfence_system();
      const uint32_t r = atomicAdd(&s->retire, 1u) + 1;
      if (r == gridDim.x) {
        s->exit = 0;
        q->start = exit_ticket + 1;
        __threadfence();
        sw_st_release_gpu(&s->free_seq, exit_ticket + 1);
      }
      a.ctl->exited = a.launch_seq;   // (the host also waits for the stream: the other CTAs may still be leaving)
    }
    return;
  }

  // ================================================================ copy CTAs
  // warp 0, thread 0: drives the TMA pipeline.  warp 1: watches the queue and brings the descriptors of the next
  // batch into shared memory ahead of time (a lane per message: one round trip to L2 instead of 3 x messages).
  if (threadIdx.x == 0) {
    s_ready = first;
    s_released = first;
  }
  __syncthreads();
  if (threadIdx.x >= 32) {
    const uint32_t lane = threadIdx.x & 31;
    for (uint64_t t = first;; t++) {
      SwPullSlot* s = &q->slot[t % SW_PULL_SLOTS];
      while (t >= s_released + 2) __nanosleep(50);                       // the buffer (t & 1) is still in use
      while (sw_ld_acquire_gpu(&s->seq) != t + 1) __nanosleep(100);    // not published yet
      const uint32_t k = t & 1, nj = s->njobs, ex = s->exit;
      for (uint32_t j = lane; j < nj; j += 32) {
        s_endb[k][j] = s->end[j];
        s_srcb[k][j] = s->src[j];
        s_dstb[k][j] = s->dst[j];
      }
      if (lane == 0) {
        s_chunk[k] = s->chunk_bytes;
        s_total[k] = s->total;
        s_nchunks[k] = s->nchunks;
        s_exitb[k] = ex;
      }
      __syncwarp();
      if (lane == 0) {
        __threadfence_block();
        s_ready = t + 1;
      }
      if (ex) return;
    }
  }
  if (threadIdx.x != 0) return;
  const uint32_t nstages = a.nstages, stage_bytes = a.stage_bytes;
  for (uint32_t i = 0; i < nstages; i++) sw_mbar_init(&full[i], 1);
  sw_fence_mbar_init();
  sw_fence_proxy_async();

  constexpr uint32_t TRK = 16;   // pieces tracked between load issue and accounted completion (> look-ahead + lag)
  constexpr uint32_t LAG = 6;    // store groups that may be outstanding when completions are accounted: waiting for
                                 // fewer would make every iteration wait for a store issued two pieces ago
  uint64_t st_dst[SW_BULK_MAX_STAGES];
  uint32_t st_bytes[SW_BULK_MAX_STAGES];
  SwPullSlot* tr_slot[TRK];      // != nullptr: this piece is the last of a chunk of that slot
  for (uint32_t i = 0; i < TRK; i++) tr_slot[i] = nullptr;
  const uint32_t lookahead = nstages - 2;
  uint64_t issued = 0, stored = 0, retired = 0;

  // generator state
  uint64_t b = first;                          // ticket looked at next
  SwPullSlot* cur = nullptr;                   // batch being worked on
  uint32_t nchunks = 0, j = 0, kb = 0;
  uint64_t chunk_bytes = 0, total = 0, pos = 0, cend = 0;
  bool have_chunk = false, leave = false;
  const uint64_t *s_end = s_endb[0], *s_src = s_srcb[0], *s_dst = s_dstb[0];

  // a chunk is counted once its bulk stores have completed (cp.async.bulk.wait_group): plain atomic, no fence --
  // CTA 0 fences once per batch before it publishes the completion records
  auto chunk_done = [&](SwPullSlot* s) { atomicAdd(&s->done_chunks, 1u); };
  // next piece of work, without blocking: 1 = piece, 0 = nothing right now
  auto try_next = [&](uint64_t& src, uint64_t& dst, uint32_t& bytes, bool& last) -> int {
    for (;;) {
      if (have_chunk) {
        if (pos < cend) {
          while (s_end[j] <= pos) j++;
          const uint64_t begin = j ? s_end[j - 1] : 0;
          const uint64_t stop = s_end[j] < cend ? s_end[j] : cend;
          const uint64_t left = stop - pos;
          bytes = left < stage_bytes ? static_cast<uint32_t>(left) : stage_bytes;
          src = s_src[j] + (pos - begin);
          dst = s_dst[j] + (pos - begin);
          pos += bytes;
          last = pos >= cend;
          if (last) have_chunk = false;
          return 1;
        }
        have_chunk = false;
        chunk_done(cur);   // an empty chunk (a batch of tails only)
      }
      if (!cur) {
        if (s_ready <= b) return 0;   // warp 1 has not seen batch b yet
        __threadfence_block();
        kb = b & 1;
        if (s_exitb[kb]) {
          leave = true;
          return 0;
        }
        cur = &q->slot[b % SW_PULL_SLOTS];
        nchunks = s_nchunks[kb];
        chunk_bytes = s_chunk[kb];
        total = s_total[kb];
        s_end = s_endb[kb];
        s_src = s_srcb[kb];
        s_dst = s_dstb[kb];
      }
      const uint32_t cidx = atomicAdd(&cur->next_chunk, 1u);
      if (cidx >= nchunks) {
        sw_pull_retire(cur, b);   // nothing left for this CTA in batch b
        cur = nullptr;
        b++;
        // pieces of batch b - 1 may still be in flight, but their addresses are in st_dst / the TMA unit: the
        // descriptor buffer can be refilled
        s_released = b;
        continue;
      }
      if (cidx == 0) cur->t_first = sw_globaltimer();
      pos = static_cast<uint64_t>(cidx) * chunk_bytes;
      cend = pos + chunk_bytes < total ? pos + chunk_bytes : total;
      j = 0;
      have_chunk = true;
    }
  };
  auto account = [&](uint64_t piece) {
    SwPullSlot* s = tr_slot[piece % TRK];
    if (s) chunk_done(s);
  };

  for (;;) {
    // ---- issue loads up to the look-ahead
    bool idle = false;
    while (issued - stored < lookahead && issued - retired < TRK - 1) {
      uint64_t src, dst;
      uint32_t bytes;
      bool last;
      if (!try_next(src, dst, bytes, last)) {
        idle = true;
        break;
      }
      if (issued >= nstages) sw_bulk_wait_read<1>();   // the store that last used this stage has read it
      const uint32_t stg = issued % nstages;
      sw_mbar_expect_tx(&full[stg], bytes);
      sw_bulk_g2s(sw_smem + size_t(stg) * stage_bytes, reinterpret_cast<const void*>(src), bytes, &full[stg]);
      st_dst[stg] = dst;
      st_bytes[stg] = bytes;
      tr_slot[issued % TRK] = last ? cur : nullptr;   // (`cur` is the batch the piece belongs to)
      issued++;
    }
    // ---- store the oldest loaded piece
    if (stored < issued) {
      const uint32_t stg = stored % nstages;
      sw_mbar_wait(&full[stg], (stored / nstages) & 1);
      sw_bulk_s2g(reinterpret_cast<void*>(st_dst[stg]), sw_smem + size_t(stg) * stage_bytes, st_bytes[stg]);
      sw_bulk_commit();
      stored++;
    }
    // ---- account completions: all but the LAG most recent store groups have been written
    if (stored - retired > LAG) {
      asm volatile("cp.async.bulk.wait_group %0;" ::"n"(LAG) : "memory");
      while (retired + LAG < stored) account(retired++);
    }
    if (idle && stored == issued) {
      if (retired < stored) {
        sw_bulk_wait_all();
        while (retired < stored) account(retired++);
      }
      if (leave) break;
      __nanosleep(100);
    }
  }
  // the EXIT batch: every CTA passes it once; the last one hands the next launch its first ticket
  {
    SwPullSlot* s = &q->slot[b % SW_PULL_SLOTS];
    const uint32_t r = atomicAdd(&s->retire, 1u) + 1;
    if (r == gridDim.x) {
      s->exit = 0;
      q->start = b + 1;
      __threadfence();
      sw_st_release_gpu(&s->free_seq, b + 1);
    }
  }
}
