// starway_b200 — hand-written sm_90a kernels for the tagged-messaging hot path.
//
//   sw_put_kernel       eager / RTS put: vectorised stores into the peer's inbound ring
//   sw_put_inline_kernel  same, descriptors + RTS payloads as kernel parameters (batches <= 32)
//                       (replaces the eager leg of ucp_tag_send_nbx, reference main.cpp:370,1136)
//   sw_match_kernel     device-resident posted / unexpected queues + tag matching
//                       (replaces ucp_tag_recv_nbx + the matching inside ucp_worker_progress,
//                        reference main.cpp:404,1172,362,1127)
//   sw_deliver_kernel   slot/heap -> user buffer copies + completion records
//   sw_match_deliver_kernel  both in one launch for small batches (job list in shared memory)
//   sw_bulk_tma_kernel  rendezvous / loopback bulk copy, cp.async.bulk global->smem->global
//                       with an mbarrier pipeline (replaces the rendezvous leg of ucp_tag_send_nbx)
//   sw_bulk_simt_kernel generic-alignment bulk copy (fallback + comparison)
//
// Pure data movement and uint64 xor/and/compare: no tensor cores, no floating point.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "sw_device.h"

// ------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t sw_smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void sw_mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sw_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void sw_fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void sw_fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void sw_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sw_smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void sw_mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "SW_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra SW_DONE;\n\t"
      "bra SW_WAIT;\n\t"
      "SW_DONE:\n\t"
      "}" ::"r"(sw_smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// TMA bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void sw_bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          sw_smem_u32(smem_dst)),
      "l"(__cvta_generic_to_global(gsrc)), "r"(bytes), "r"(sw_smem_u32(bar))
      : "memory");
}
// TMA bulk copy shared -> global, tracked by bulk async-groups
__device__ __forceinline__ void sw_bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(__cvta_generic_to_global(gdst)),
               "r"(sw_smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void sw_bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void sw_bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void sw_bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ int4 sw_ld16(const void* p) {
  int4 r;
  asm volatile("ld.global.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void sw_st16(void* p, const int4& v) {
  asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}

// ------------------------------------------------------------------ cooperative byte copy
// Copies len bytes with `nthr` cooperating threads (a warp or a CTA).  Loads never allocate in L1 (a resident
// kernel reads ring slots that peers rewrite while it runs).  Uses 16 B
// vectors when src and dst are mutually 16 B aligned, 4 B words when mutually
// 4 B aligned, bytes otherwise.  Heads/tails are peeled with byte copies.
__device__ __forceinline__ void sw_copy(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint64_t len,
                                        uint32_t tid, uint32_t nthr) {
  if (len == 0) return;
  const uint64_t s = reinterpret_cast<uint64_t>(src), d = reinterpret_cast<uint64_t>(dst);
  if (((s ^ d) & 15) == 0) {
    uint64_t head = (16 - (s & 15)) & 15;
    if (head > len) head = len;
    if (tid < head) dst[tid] = __ldcg(src + tid);
    const uint64_t body = (len - head) >> 4;
    const int4* s4 = reinterpret_cast<const int4*>(src + head);
    int4* d4 = reinterpret_cast<int4*>(dst + head);
    uint64_t i = tid;
    for (; i + 3ull * nthr < body; i += 4ull * nthr) {
      int4 a = sw_ld16(s4 + i), b = sw_ld16(s4 + i + nthr), c = sw_ld16(s4 + i + 2ull * nthr),
           e = sw_ld16(s4 + i + 3ull * nthr);
      sw_st16(d4 + i, a);
      sw_st16(d4 + i + nthr, b);
      sw_st16(d4 + i + 2ull * nthr, c);
      sw_st16(d4 + i + 3ull * nthr, e);
    }
    for (; i < body; i += nthr) sw_st16(d4 + i, sw_ld16(s4 + i));
    const uint64_t done = head + (body << 4);
    const uint64_t tail = len - done;
    if (tid < tail) dst[done + tid] = __ldcg(src + done + tid);
  } else if (((s ^ d) & 3) == 0) {
    uint64_t head = (4 - (s & 3)) & 3;
    if (head > len) head = len;
    if (tid < head) dst[tid] = __ldcg(src + tid);
    const uint64_t body = (len - head) >> 2;
    const uint32_t* s1 = reinterpret_cast<const uint32_t*>(src + head);
    uint32_t* d1 = reinterpret_cast<uint32_t*>(dst + head);
    for (uint64_t i = tid; i < body; i += nthr) d1[i] = __ldcg(s1 + i);
    const uint64_t done = head + (body << 2);
    const uint64_t tail = len - done;
    if (tid < tail) dst[done + tid] = __ldcg(src + done + tid);
  } else {
    for (uint64_t i = tid; i < len; i += nthr) dst[i] = __ldcg(src + i);
  }
}

// Slot header: tag / length / kind / magic first, then the sequence word -- the arrival flag -- with release
// semantics at system scope.  The payload stores of the other lanes are ordered before it by the __syncwarp the
// callers execute first (release is cumulative), so a receiver that observes the flag with an acquire load
// (sw_progress_kernel) sees header and payload; a receiver launched after the host doorbell sees them anyway.
__device__ __forceinline__ void sw_put_header(uint8_t* slot, uint64_t tag, uint64_t msg_len, uint64_t seq, uint32_t kind) {
  int4 h0;
  h0.x = static_cast<int>(tag & 0xffffffffu);
  h0.y = static_cast<int>(tag >> 32);
  h0.z = static_cast<int>(msg_len & 0xffffffffu);
  h0.w = static_cast<int>(msg_len >> 32);
  sw_st16(slot, h0);
  const uint64_t km = (static_cast<uint64_t>(SW_SLOT_MAGIC) << 32) | kind;
  asm volatile("st.global.u64 [%0], %1;" ::"l"(slot + 24), "l"(km) : "memory");
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(slot + 16), "l"(seq) : "memory");
}

// The same header for a ring in this GPU's own memory: the receiver's acquire load (any scope) runs on this GPU,
// a device-scope release is enough.
__device__ __forceinline__ void sw_put_header_same_gpu(uint8_t* slot, uint64_t tag, uint64_t msg_len, uint64_t seq, uint32_t kind) {
  int4 h0;
  h0.x = static_cast<int>(tag & 0xffffffffu);
  h0.y = static_cast<int>(tag >> 32);
  h0.z = static_cast<int>(msg_len & 0xffffffffu);
  h0.w = static_cast<int>(msg_len >> 32);
  sw_st16(slot, h0);
  const uint64_t km = (static_cast<uint64_t>(SW_SLOT_MAGIC) << 32) | kind;
  asm volatile("st.global.u64 [%0], %1;" ::"l"(slot + 24), "l"(km) : "memory");
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(slot + 16), "l"(seq) : "memory");
}

// ------------------------------------------------------------------ K1: eager / RTS put
// One warp per message.  Payload first (16 B vector stores into the peer ring slot),
// then a system-scope fence, then the 64 B header whose last word carries the
// sequence number / magic (flag).  Grid-stride over the descriptor batch.
__global__ void __launch_bounds__(256) sw_put_kernel(const SwPutDesc* __restrict__ descs, uint32_t n) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t i = warp; i < n; i += nwarps) {
    const SwPutDesc d = descs[i];
    uint8_t* slot = reinterpret_cast<uint8_t*>(d.dst);
    sw_copy(slot + SW_SLOT_HDR, reinterpret_cast<const uint8_t*>(d.src), d.len, lane, 32);
    __syncwarp();
    if (lane == 0) sw_put_header(slot, d.tag, d.msg_len, d.seq, d.kind);
  }
}

// Small batches: descriptors and RTS payloads travel as kernel parameters (no PCIe read on the
// latency-critical path).
constexpr uint32_t SW_PUT_INLINE = 32;
constexpr uint32_t SW_PUT_INLINE_RTS = 16;   // keeps the parameter block under the classic 4 KiB
struct SwPutArgs {
  uint32_t n, pad;
  uint64_t done_flag;           // pinned-host word (0: none) that receives done_value when every slot is written
  uint64_t done_value;
  SwPutDesc d[SW_PUT_INLINE];   // for kind == SW_KIND_RTS, d[i].src is an index into r[]
  SwRts r[SW_PUT_INLINE_RTS];
};
static_assert(sizeof(SwPutArgs) <= 4096, "inline put parameters");
// ONE CTA, one warp per message.  Completion is announced by a flag in pinned host memory: the
// barrier collects every warp's stores, thread 0's system-scope fence orders them (cumulatively)
// before the flag, which the host sees sooner than a timing event (`sw_probe floor` measures both).
__global__ void __launch_bounds__(SW_PUT_INLINE * 32) sw_put_inline_kernel(const __grid_constant__ SwPutArgs a) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t nwarps = blockDim.x >> 5;
  for (uint32_t i = warp; i < a.n; i += nwarps) {
    const SwPutDesc d = a.d[i];
    uint8_t* slot = reinterpret_cast<uint8_t*>(d.dst);
    if (d.kind == SW_KIND_RTS) {
      if (lane < 8) {
        const int4 v = reinterpret_cast<const int4*>(&a.r[d.src & (SW_PUT_INLINE_RTS - 1)])[lane];
        sw_st16(slot + SW_SLOT_HDR + 16 * lane, v);
      }
    } else {
      sw_copy(slot + SW_SLOT_HDR, reinterpret_cast<const uint8_t*>(d.src), d.len, lane, 32);
    }
    __syncwarp();
    if (lane == 0) sw_put_header(slot, d.tag, d.msg_len, d.seq, d.kind);
  }
  if (a.done_flag) {
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence_system();
      *reinterpret_cast<volatile uint64_t*>(a.done_flag) = a.done_value;
    }
  }
}

// ------------------------------------------------------------------ K2: tag match
// One warp per worker.  The queues live in device memory; the warp keeps a 32-entry
// register window over the head of the queue it is searching so that FIFO traffic
// costs one global-memory round trip per 32 events instead of one per event.
//
// Order of events inside one launch (any serialisation of concurrent posts and
// arrivals is legal; this one removes intra-launch copy dependencies):
//   phase 1: every new receive, in post order, takes the EARLIEST-ARRIVED matching
//            unexpected message, else is appended to the posted queue;
//   phase 2: every new arrival, per ring in ring order (rings round-robin), is given
//            to the EARLIEST-POSTED matching receive, else is stashed on the heap and
//            appended to the unexpected queue.
struct SwMatchRegs {   // warp-uniform scalars kept in registers for the whole launch
  uint64_t p_head, p_tail, u_head, u_tail;
  uint32_t p_count, u_count;
  uint32_t n_jobs, n_rndv, err;
  uint32_t n_free_small, n_free_big, n_pend_small, n_pend_big;
};

__device__ __forceinline__ uint64_t sw_shfl64(uint64_t v, int src) {
  uint32_t lo = __shfl_sync(0xffffffffu, static_cast<uint32_t>(v), src);
  uint32_t hi = __shfl_sync(0xffffffffu, static_cast<uint32_t>(v >> 32), src);
  return (static_cast<uint64_t>(hi) << 32) | lo;
}

__device__ __forceinline__ void sw_emit_job(SwJob* jobs, SwMatchRegs& r, uint32_t lane, uint64_t src,
                                            uint64_t dst, uint64_t len, uint64_t op, uint64_t tag, uint64_t msg_len,
                                            int32_t status, uint32_t kind) {
  if (lane == 0) {
    SwJob* j = &jobs[r.n_jobs];
    j->src = src;
    j->dst = dst;
    j->len = len;
    j->op_id = op;
    j->tag = tag;
    j->msg_len = msg_len;
    j->status = status;
    j->kind = kind;
  }
  r.n_jobs++;
}

// Hand a matched message to the receive (buf, cap, op).  `payload` points at the eager
// bytes or at the SwRts (slot payload or heap block).
__device__ __forceinline__ void sw_emit_match(SwJob* jobs, SwMatchOut* out, SwMatchRegs& r, uint32_t lane,
                                              bool is_rts, uint64_t payload, uint64_t stag, uint64_t msg_len,
                                              uint32_t ep, uint64_t buf, uint64_t cap, uint64_t op) {
  const bool trunc = msg_len > cap;
  if (!is_rts) {
    sw_emit_job(jobs, r, lane, payload, buf, trunc ? 0 : msg_len, op, stag, msg_len,
                trunc ? SW_ERR_MESSAGE_TRUNCATED : SW_OK, SW_JOB_DELIVER);
  } else {
    SwRndvRec* rec = &out->rndv[r.n_rndv];
    // 128 B descriptor: 32 lanes x 4 B
    reinterpret_cast<uint32_t*>(&rec->rts)[lane] = reinterpret_cast<const uint32_t*>(payload)[lane];
    if (lane == 0) {
      rec->op_id = op;
      rec->dst = buf;
      rec->cap = cap;
      rec->tag = stag;
      rec->len = msg_len;
      rec->ep = ep;
      rec->status = trunc ? SW_ERR_MESSAGE_TRUNCATED : SW_OK;
    }
    r.n_rndv++;
  }
}

// Launch scalars travel as kernel parameters (constant bank) instead of being read from pinned host
// memory over PCIe: with <= SW_INLINE_EPS rings and <= SW_INLINE_POSTS new receives a match launch
// performs no host-memory read at all.
constexpr uint32_t SW_INLINE_EPS = 8;
constexpr uint32_t SW_INLINE_POSTS = 32;
struct SwMatchArgs {
  uint32_t n_posts, n_eps, max_arrivals, pad;
  uint64_t done_value;   // fused launch: value stored to SwMatchOut::done_seq at the very end (0: none)
  uint64_t produced[SW_INLINE_EPS];
  SwMatchScalars sc;   // sc.valid: queue cursors + ring cursors by value (host mirror of the last launch)
  SwPost posts[SW_INLINE_POSTS];
};
static_assert(SW_SC_EPS == SW_INLINE_EPS, "cursor mirror covers the inline endpoints");

// returns the number of jobs emitted into `jobs`
__device__ __forceinline__ uint32_t sw_match_body(SwMatchState* __restrict__ st, const SwMatchIn* __restrict__ in,
                                              SwMatchOut* __restrict__ out, const SwMatchArgs& a,
                                              SwJob* __restrict__ jobs, const uint32_t lane) {
  SwMatchRegs r;
  const bool by_value = a.sc.valid != 0 && a.n_eps <= SW_SC_EPS;
  if (by_value) {
    r.p_head = a.sc.p_head;
    r.p_tail = a.sc.p_tail;
    r.u_head = a.sc.u_head;
    r.u_tail = a.sc.u_tail;
    r.p_count = a.sc.p_count;
    r.u_count = a.sc.u_count;
    r.n_free_small = a.sc.n_free_small;
    r.n_free_big = a.sc.n_free_big;
    r.n_pend_small = a.sc.n_pend_small;
    r.n_pend_big = a.sc.n_pend_big;
  } else {
    r.p_head = st->p_head;
    r.p_tail = st->p_tail;
    r.u_head = st->u_head;
    r.u_tail = st->u_tail;
    r.p_count = st->p_count;
    r.u_count = st->u_count;
    r.n_free_small = st->n_free_small;
    r.n_free_big = st->n_free_big;
    r.n_pend_small = st->n_pend_small;
    r.n_pend_big = st->n_pend_big;
  }
  r.n_jobs = 0;
  r.n_rndv = 0;
  r.err = 0;

  // deferred heap frees of the previous launch become allocatable now (its deliver
  // kernel has finished: same stream)
  for (uint32_t i = lane; i < r.n_pend_small; i += 32) st->free_small[r.n_free_small + i] = st->pend_small[i];
  for (uint32_t i = lane; i < r.n_pend_big; i += 32) st->free_big[r.n_free_big + i] = st->pend_big[i];
  r.n_free_small += r.n_pend_small;
  r.n_free_big += r.n_pend_big;
  r.n_pend_small = 0;
  r.n_pend_big = 0;
  __syncwarp();

  const uint64_t PQM = SW_PQ_CAP - 1, UQM = SW_UQ_CAP - 1;

  // ---------------- compaction of the posted queue when tombstones dominate
  if (r.p_tail - r.p_head > SW_PQ_CAP / 2) {
    uint64_t j = r.p_head;
    for (uint64_t b = r.p_head; b < r.p_tail; b += 32) {
      const uint64_t idx = b + lane;
      uint32_t v = 0;
      uint64_t t = 0, m = 0, bf = 0, cp = 0, op = 0;
      if (idx < r.p_tail) {
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
        st->p_valid[s] = 1;
      }
      j += __popc(bal);
      __syncwarp();
    }
    for (uint64_t idx = j + lane; idx < r.p_tail; idx += 32) st->p_valid[idx & PQM] = 0;
    r.p_tail = j;
    __syncwarp();
  }
  // ---------------- same for the unexpected queue
  if (r.u_tail - r.u_head > SW_UQ_CAP / 2) {
    uint64_t j = r.u_head;
    for (uint64_t b = r.u_head; b < r.u_tail; b += 32) {
      const uint64_t idx = b + lane;
      uint32_t meta = 0, blk = 0;
      uint64_t t = 0, l = 0, dta = 0;
      if (idx < r.u_tail) {
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
    for (uint64_t idx = j + lane; idx < r.u_tail; idx += 32) st->u_meta[idx & UQM] = 0;
    r.u_tail = j;
    __syncwarp();
  }

  // ================================================================ phase 1: new receives
  const uint32_t n_posts = a.n_posts;
  if (n_posts) {
    // register window over the unexpected queue: lane L caches entry (wb + L)
    uint64_t wb = r.u_head;
    uint64_t w_tag = 0, w_len = 0, w_data = 0;
    uint32_t w_meta = 0, w_blk = 0;
    auto load_uwin = [&]() {
      const uint64_t idx = wb + lane;
      w_meta = 0;
      if (idx < r.u_tail) {
        const uint64_t s = idx & UQM;
        w_meta = st->u_meta[s];
        w_tag = st->u_tag[s];
        w_len = st->u_len[s];
        w_data = st->u_data[s];
        w_blk = st->u_blk[s];
      }
    };
    load_uwin();
    for (uint32_t base = 0; base < n_posts; base += 32) {
      SwPost mine;
      mine.tag = mine.mask = mine.buf = mine.cap = mine.op_id = 0;
      if (base + lane < n_posts) mine = (n_posts <= SW_INLINE_POSTS) ? a.posts[base + lane] : in->posts[base + lane];
      const uint32_t cnt = min(32u, n_posts - base);
      if (r.u_count == 0 && SW_PQ_CAP - (r.p_tail - r.p_head) >= cnt) {
        // fast path: nothing is waiting in the unexpected queue, so every receive of this chunk
        // is simply appended -- 32 receives per step, one lane each
        if (lane < cnt) {
          const uint64_t s = (r.p_tail + lane) & PQM;
          st->p_tag[s] = mine.tag;
          st->p_mask[s] = mine.mask;
          st->p_buf[s] = mine.buf;
          st->p_cap[s] = mine.cap;
          st->p_op[s] = mine.op_id;
          st->p_valid[s] = 1;
        }
        r.p_tail += cnt;
        r.p_count += cnt;
        continue;
      }
      for (uint32_t j = 0; j < cnt; j++) {
        const uint64_t tag = sw_shfl64(mine.tag, j), mask = sw_shfl64(mine.mask, j);
        const uint64_t buf = sw_shfl64(mine.buf, j), cap = sw_shfl64(mine.cap, j);
        const uint64_t op = sw_shfl64(mine.op_id, j);
        bool found = false;
        uint64_t f_tag = 0, f_len = 0, f_data = 0;
        uint32_t f_meta = 0, f_blk = 0;
        if (r.u_count) {
          // drop fully consumed windows
          while (__ballot_sync(0xffffffffu, (w_meta & SW_UMETA_VALID) != 0) == 0 && wb + 32 <= r.u_tail) {
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
            if (lane == L) {
              w_meta = 0;
              st->u_meta[(wb + L) & UQM] = 0;
            }
            found = true;
          } else {
            for (uint64_t b = wb + 32; b < r.u_tail && !found; b += 32) {
              const uint64_t idx = b + lane;
              uint32_t meta = 0;
              uint64_t t = 0;
              if (idx < r.u_tail) {
                meta = st->u_meta[idx & UQM];
                t = st->u_tag[idx & UQM];
              }
              const bool h2 = (meta & SW_UMETA_VALID) && sw_tag_match(t, tag, mask);
              bal = __ballot_sync(0xffffffffu, h2);
              if (bal) {
                const int L = __ffs(bal) - 1;
                uint64_t l = 0, dta = 0;
                uint32_t blk = 0;
                if (lane == L) {
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
          r.u_count--;
          sw_emit_match(jobs, out, r, lane, (f_meta & SW_UMETA_RTS) != 0, f_data, f_tag, f_len,
                        f_meta & SW_UMETA_EPMASK, buf, cap, op);
          // the heap block is released one launch later (after this launch's deliver kernel)
          if (lane == 0) {
            if (f_meta & SW_UMETA_BIG)
              st->pend_big[r.n_pend_big] = f_blk;
            else
              st->pend_small[r.n_pend_small] = f_blk;
          }
          if (f_meta & SW_UMETA_BIG)
            r.n_pend_big++;
          else
            r.n_pend_small++;
        } else {
          if (r.p_tail - r.p_head >= SW_PQ_CAP) {
            r.err |= 2;   // posted queue overflow (the host throttles before this can happen)
            sw_emit_job(jobs, r, lane, 0, 0, 0, op, 0, 0, SW_ERR_NO_MEMORY, SW_JOB_DELIVER);
          } else {
            if (lane == 0) {
              const uint64_t s = r.p_tail & PQM;
              st->p_tag[s] = tag;
              st->p_mask[s] = mask;
              st->p_buf[s] = buf;
              st->p_cap[s] = cap;
              st->p_op[s] = op;
              st->p_valid[s] = 1;
            }
            r.p_tail++;
            r.p_count++;
          }
        }
      }
    }
    // every entry before the window base is a tombstone
    while (__ballot_sync(0xffffffffu, (w_meta & SW_UMETA_VALID) != 0) == 0 && wb + 32 <= r.u_tail) {
      wb += 32;
      load_uwin();
    }
    r.u_head = wb;
    __syncwarp();
  }

  // ================================================================ phase 2: new arrivals
  {
    uint64_t wb = r.p_head;
    uint64_t w_tag = 0, w_mask = 0, w_buf = 0, w_cap = 0, w_op = 0;
    uint32_t w_valid = 0;
    auto load_pwin = [&]() {
      const uint64_t idx = wb + lane;
      w_valid = 0;
      if (idx < r.p_tail) {
        const uint64_t s = idx & PQM;
        w_valid = st->p_valid[s];
        w_tag = st->p_tag[s];
        w_mask = st->p_mask[s];
        w_buf = st->p_buf[s];
        w_cap = st->p_cap[s];
        w_op = st->p_op[s];
      }
    };
    load_pwin();
    const uint32_t n_eps = a.n_eps;
    uint32_t budget = min(a.max_arrivals, SW_MAX_ARRIVALS);
    uint32_t consumed_total = 0;
    const uint32_t rr = n_eps ? ((by_value ? a.sc.rr_ep : st->rr_ep) % n_eps) : 0;
    for (uint32_t e = 0; e < n_eps; e++) {
      const uint32_t ep = (rr + e) % n_eps;
      uint64_t cons = by_value ? a.sc.ring_cons[ep] : st->ring_cons[ep];
      const uint64_t prod = (n_eps <= SW_INLINE_EPS) ? a.produced[ep] : in->produced[ep];
      const uint64_t ring = by_value ? a.sc.ring_base[ep] : st->ring_base[ep];
      const uint64_t smask = (by_value ? a.sc.ring_slots[ep] : st->ring_slots[ep]) - 1;
      bool blocked = false;
      while (cons < prod && budget > 0 && !blocked) {
        const uint32_t chunk = static_cast<uint32_t>(min(static_cast<uint64_t>(min(32u, budget)), prod - cons));
        // lanes prefetch 32 slot headers at once
        uint64_t h_tag = 0, h_len = 0, h_seq = 0;
        uint32_t h_kind = 0, h_magic = 0;
        const uint64_t my_slot = ring + ((cons + lane) & smask) * SW_SLOT_BYTES;
        if (lane < chunk) {
          const int4 a = sw_ld16(reinterpret_cast<const void*>(my_slot));
          const int4 b = sw_ld16(reinterpret_cast<const void*>(my_slot + 16));
          h_tag = (static_cast<uint64_t>(static_cast<uint32_t>(a.y)) << 32) | static_cast<uint32_t>(a.x);
          h_len = (static_cast<uint64_t>(static_cast<uint32_t>(a.w)) << 32) | static_cast<uint32_t>(a.z);
          h_seq = (static_cast<uint64_t>(static_cast<uint32_t>(b.y)) << 32) | static_cast<uint32_t>(b.x);
          h_kind = static_cast<uint32_t>(b.z);
          h_magic = static_cast<uint32_t>(b.w);
        }
        // ---- fast path: pair up to 32 arrivals with the first posted receives in ONE step when every
        // one of those receives accepts every one of those arrivals (all wildcard masks, or all
        // arrivals carry the same tag): arrival j then goes to the j-th valid posted entry, exactly
        // what the sequential rule (earliest-posted matching receive) produces.
        uint32_t j0 = 0;
        while (j0 < chunk && r.p_count) {
          while (__ballot_sync(0xffffffffu, w_valid != 0) == 0 && wb + 32 <= r.p_tail) {
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
          if (__ballot_sync(0xffffffffu, lane >= j0 && lane < j0 + k &&
                                             (h_magic != SW_SLOT_MAGIC || h_seq != cons + (lane - j0) + 1)))
            r.err |= 1;
          const int srcl = static_cast<int>(min(j0 + rnk, 31u));
          const uint64_t a_tag = sw_shfl64(h_tag, srcl), a_len = sw_shfl64(h_len, srcl);
          const uint64_t a_slot = sw_shfl64(my_slot, srcl);
          const uint32_t a_kind = __shfl_sync(0xffffffffu, h_kind, srcl);
          const bool a_rts = a_kind == SW_KIND_RTS;
          const uint32_t eager_m = __ballot_sync(0xffffffffu, in_k && !a_rts);
          const uint32_t rts_m = __ballot_sync(0xffffffffu, in_k && a_rts);
          if (in_k) {
            const bool trunc = a_len > w_cap;
            if (!a_rts) {
              SwJob* jb = &jobs[r.n_jobs + __popc(eager_m & lt)];
              jb->src = a_slot + SW_SLOT_HDR;
              jb->dst = w_buf;
              jb->len = trunc ? 0 : a_len;
              jb->op_id = w_op;
              jb->tag = a_tag;
              jb->msg_len = a_len;
              jb->status = trunc ? SW_ERR_MESSAGE_TRUNCATED : SW_OK;
              jb->kind = SW_JOB_DELIVER;
            } else {
              SwRndvRec* rec = &out->rndv[r.n_rndv + __popc(rts_m & lt)];
              const int4* sp = reinterpret_cast<const int4*>(a_slot + SW_SLOT_HDR);
              int4* dp = reinterpret_cast<int4*>(&rec->rts);
#pragma unroll
              for (int q = 0; q < 8; q++) dp[q] = sw_ld16(sp + q);
              rec->op_id = w_op;
              rec->dst = w_buf;
              rec->cap = w_cap;
              rec->tag = a_tag;
              rec->len = a_len;
              rec->ep = ep;
              rec->status = trunc ? SW_ERR_MESSAGE_TRUNCATED : SW_OK;
            }
            w_valid = 0;
            st->p_valid[(wb + lane) & PQM] = 0;
          }
          r.n_jobs += __popc(eager_m);
          r.n_rndv += __popc(rts_m);
          r.p_count -= k;
          j0 += k;
          cons += k;
          budget -= k;
          consumed_total += k;
        }
        for (uint32_t j = j0; j < chunk && !blocked; j++) {
          const uint64_t stag = sw_shfl64(h_tag, j), mlen = sw_shfl64(h_len, j), seq = sw_shfl64(h_seq, j);
          const uint32_t kind = __shfl_sync(0xffffffffu, h_kind, j);
          const uint32_t magic = __shfl_sync(0xffffffffu, h_magic, j);
          const uint64_t slot = sw_shfl64(my_slot, j);
          const uint64_t payload = slot + SW_SLOT_HDR;
          if (magic != SW_SLOT_MAGIC || seq != cons + 1) r.err |= 1;
          const bool is_rts = kind == SW_KIND_RTS;
          bool found = false;
          uint64_t f_buf = 0, f_cap = 0, f_op = 0;
          if (r.p_count) {
            while (__ballot_sync(0xffffffffu, w_valid != 0) == 0 && wb + 32 <= r.p_tail) {
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
              if (lane == L) {
                w_valid = 0;
                st->p_valid[(wb + L) & PQM] = 0;
              }
              found = true;
            } else {
              for (uint64_t b = wb + 32; b < r.p_tail && !found; b += 32) {
                const uint64_t idx = b + lane;
                uint32_t v = 0;
                uint64_t t = 0, m = 0;
                if (idx < r.p_tail) {
                  v = st->p_valid[idx & PQM];
                  t = st->p_tag[idx & PQM];
                  m = st->p_mask[idx & PQM];
                }
                const bool h2 = v && sw_tag_match(stag, t, m);
                bal = __ballot_sync(0xffffffffu, h2);
                if (bal) {
                  const int L = __ffs(bal) - 1;
                  uint64_t bf = 0, cp = 0, op = 0;
                  if (lane == L) {
                    bf = st->p_buf[idx & PQM];
                    cp = st->p_cap[idx & PQM];
                    op = st->p_op[idx & PQM];
                    st->p_valid[idx & PQM] = 0;
                  }
                  f_buf = sw_shfl64(bf, L);
                  f_cap = sw_shfl64(cp, L);
                  f_op = sw_shfl64(op, L);
                  found = true;
                }
              }
            }
          }
          if (found) {
            r.p_count--;
            sw_emit_match(jobs, out, r, lane, is_rts, payload, stag, mlen, ep, f_buf, f_cap, f_op);
          } else {
            // unexpected: park the payload (or the RTS descriptor) on the heap, free the slot
            const uint64_t need = is_rts ? sizeof(SwRts) : mlen;
            const bool big = need > SW_HEAP_SMALL_BYTES;
            const bool have = big ? (r.n_free_big > 0) : (r.n_free_small > 0);
            if (!have || r.u_tail - r.u_head >= SW_UQ_CAP) {
              blocked = true;   // back-pressure: leave the message in its ring slot
              break;
            }
            uint32_t blk = 0;
            if (lane == 0) blk = big ? st->free_big[r.n_free_big - 1] : st->free_small[r.n_free_small - 1];
            blk = __shfl_sync(0xffffffffu, blk, 0);
            if (big)
              r.n_free_big--;
            else
              r.n_free_small--;
            const uint64_t haddr = big ? reinterpret_cast<uint64_t>(st->heap_big) + uint64_t(blk) * SW_HEAP_BIG_BYTES
                                       : reinterpret_cast<uint64_t>(st->heap_small) + uint64_t(blk) * SW_HEAP_SMALL_BYTES;
            sw_emit_job(jobs, r, lane, payload, haddr, need, 0, stag, mlen, SW_OK, SW_JOB_STASH);
            if (lane == 0) {
              const uint64_t s = r.u_tail & UQM;
              st->u_tag[s] = stag;
              st->u_len[s] = mlen;
              st->u_data[s] = haddr;
              st->u_blk[s] = blk;
              st->u_meta[s] = SW_UMETA_VALID | (big ? SW_UMETA_BIG : 0) | (is_rts ? SW_UMETA_RTS : 0) |
                              (ep & SW_UMETA_EPMASK);
            }
            r.u_tail++;
            r.u_count++;
          }
          cons++;
          budget--;
          consumed_total++;
        }
      }
      if (lane == 0) {
        st->ring_cons[ep] = cons;
        out->consumed[ep] = cons;
      }
    }
    while (__ballot_sync(0xffffffffu, w_valid != 0) == 0 && wb + 32 <= r.p_tail) {
      wb += 32;
      load_pwin();
    }
    r.p_head = wb;
    if (lane == 0) {
      st->rr_ep = rr + 1;
      out->sc.rr_ep = rr + 1;
      out->n_arrivals = consumed_total;
    }
  }

  if (lane == 0) {
    st->p_head = r.p_head;
    st->p_tail = r.p_tail;
    st->u_head = r.u_head;
    st->u_tail = r.u_tail;
    st->p_count = r.p_count;
    st->u_count = r.u_count;
    st->n_jobs = r.n_jobs;
    st->n_free_small = r.n_free_small;
    st->n_free_big = r.n_free_big;
    st->n_pend_small = r.n_pend_small;
    st->n_pend_big = r.n_pend_big;
    out->n_jobs = r.n_jobs;
    out->n_rndv = r.n_rndv;
    out->n_posted = r.p_count;
    out->n_unexp = r.u_count;
    out->err = r.err;
    out->heap_small_free = r.n_free_small;
    out->heap_big_free = r.n_free_big;
    out->sc.p_head = r.p_head;
    out->sc.p_tail = r.p_tail;
    out->sc.u_head = r.u_head;
    out->sc.u_tail = r.u_tail;
    out->sc.p_count = r.p_count;
    out->sc.u_count = r.u_count;
    out->sc.n_free_small = r.n_free_small;
    out->sc.n_free_big = r.n_free_big;
    out->sc.n_pend_small = r.n_pend_small;
    out->sc.n_pend_big = r.n_pend_big;
    out->sc.valid = 1;
  }
  return r.n_jobs;
}

__global__ void __launch_bounds__(32) sw_match_kernel(SwMatchState* __restrict__ st, const SwMatchIn* __restrict__ in,
                                                      SwMatchOut* __restrict__ out,
                                                      const __grid_constant__ SwMatchArgs a) {
  (void)sw_match_body(st, in, out, a, st->jobs, threadIdx.x);
}

__device__ __forceinline__ void sw_deliver_one(const SwJob& j, SwMatchOut* __restrict__ out, uint32_t i,
                                               uint32_t lane) {
  sw_copy(reinterpret_cast<uint8_t*>(j.dst), reinterpret_cast<const uint8_t*>(j.src), j.len, lane, 32);
  if (lane == 0) {
    // the host reads the record only after the launch has completed (CUDA event, or the done flag)
    SwCqe c;
    c.op_id = j.op_id;
    c.tag = j.tag;
    c.len = j.msg_len;
    c.status = j.status;
    c.kind = j.kind;
    out->cq[i] = c;
  }
}

// Fused variant for small batches: warp 0 matches, then the whole CTA delivers -- one launch
// instead of two on the latency-critical path.
constexpr uint32_t SW_FUSED_THREADS = 512;
constexpr uint32_t SW_FUSED_MAX_JOBS = 192;   // the host uses the fused launch only for batches this small
__global__ void __launch_bounds__(SW_FUSED_THREADS) sw_match_deliver_kernel(SwMatchState* __restrict__ st,
                                                                            const SwMatchIn* __restrict__ in,
                                                                            SwMatchOut* __restrict__ out,
                                                                            const __grid_constant__ SwMatchArgs a) {
  // the job list of a fused launch lives in shared memory: no global round trip between the phases
  __shared__ SwJob s_jobs[SW_FUSED_MAX_JOBS];
  __shared__ uint32_t s_njobs;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 0) {
    const uint32_t nj = sw_match_body(st, in, out, a, s_jobs, lane);
    if (lane == 0) s_njobs = nj;
  }
  __syncthreads();
  const uint32_t n = s_njobs;
  for (uint32_t i = warp; i < n; i += SW_FUSED_THREADS / 32) sw_deliver_one(s_jobs[i], out, i, lane);
  if (a.done_value) {
    // completion flag in pinned host memory (see sw_put_inline_kernel): queue state, delivered
    // payloads and completion records of every warp are ordered before it
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence_system();
      *reinterpret_cast<volatile uint64_t*>(&out->done_seq) = a.done_value;
    }
  }
}

// ------------------------------------------------------------------ deliver
// One warp per job: copy the eager payload (ring slot or heap block) into the posted
// receive buffer, then publish the completion record into pinned host memory.
__global__ void __launch_bounds__(256) sw_deliver_kernel(SwMatchState* __restrict__ st, SwMatchOut* __restrict__ out) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t n = st->n_jobs;
  for (uint32_t i = warp; i < n; i += nwarps) sw_deliver_one(st->jobs[i], out, i, lane);
}

// ------------------------------------------------------------------ K3/K5: bulk copy, TMA staged
// Each CTA walks the segments s = blockIdx.x, blockIdx.x + gridDim.x, ... and streams
// them through an smem ring: cp.async.bulk global->shared (mbarrier complete_tx) then
// cp.async.bulk shared->global (bulk async-group).  One elected thread issues
// everything; the TMA engine moves the bytes.  src/dst/len of every segment must be
// multiples of 16 B (the host routes anything else to sw_bulk_simt_kernel).
constexpr int SW_BULK_MAX_STAGES = 8;

// The copy pipeline, shared by the entry points below.  `next(src, dst, bytes)` yields this CTA's
// pieces (each at most stage_bytes, 16-byte aligned) until it returns false.
template <class Next>
__device__ __forceinline__ void sw_bulk_tma_pipeline(Next next, uint32_t stage_bytes, uint32_t nstages) {
  extern __shared__ __align__(128) uint8_t sw_smem[];
  __shared__ __align__(8) uint64_t full[SW_BULK_MAX_STAGES];
  if (threadIdx.x != 0) return;
  for (uint32_t i = 0; i < nstages; i++) sw_mbar_init(&full[i], 1);
  sw_fence_mbar_init();
  sw_fence_proxy_async();

  uint64_t st_dst[SW_BULK_MAX_STAGES];
  uint32_t st_bytes[SW_BULK_MAX_STAGES];

  const uint32_t lookahead = nstages - 2;   // loads in flight ahead of the store front
  uint32_t issued = 0, done = 0;
  bool more = true;

  auto issue_load = [&]() -> bool {
    uint64_t src, dst;
    uint32_t bytes;
    if (!next(src, dst, bytes)) return false;
    const uint32_t stg = issued % nstages;
    sw_mbar_expect_tx(&full[stg], bytes);
    sw_bulk_g2s(sw_smem + size_t(stg) * stage_bytes, reinterpret_cast<const void*>(src), bytes, &full[stg]);
    st_dst[stg] = dst;
    st_bytes[stg] = bytes;
    issued++;
    return true;
  };

  while (more && issued < lookahead) more = issue_load();
  for (;;) {
    if (more && issued - done <= lookahead) {
      // the stage about to be refilled was stored >= 2 pieces ago: all but the most
      // recent store group must have finished reading shared memory
      sw_bulk_wait_read<1>();
      more = issue_load();
    }
    if (done == issued) break;
    const uint32_t stg = done % nstages;
    sw_mbar_wait(&full[stg], (done / nstages) & 1);
    sw_bulk_s2g(reinterpret_cast<void*>(st_dst[stg]), sw_smem + size_t(stg) * stage_bytes, st_bytes[stg]);
    sw_bulk_commit();
    done++;
  }
  sw_bulk_wait_all();
}

// Segment-list source: CTA b walks segments b, b + gridDim.x, ...
template <class SegAt>
__device__ __forceinline__ void sw_bulk_tma_body(SegAt seg_at, uint32_t nseg, uint32_t stage_bytes, uint32_t nstages) {
  uint32_t s = blockIdx.x;
  uint64_t off = 0;
  SwSeg cur;
  cur.src = cur.dst = cur.len = 0;
  if (threadIdx.x == 0 && s < nseg) cur = seg_at(s);
  sw_bulk_tma_pipeline(
      [&](uint64_t& src, uint64_t& dst, uint32_t& bytes) -> bool {
        while (s < nseg && off >= cur.len) {
          s += gridDim.x;
          off = 0;
          if (s < nseg) cur = seg_at(s);
        }
        if (s >= nseg) return false;
        const uint64_t left = cur.len - off;
        bytes = left < stage_bytes ? static_cast<uint32_t>(left) : stage_bytes;
        src = cur.src + off;
        dst = cur.dst + off;
        off += bytes;
        return true;
      },
      stage_bytes, nstages);
}

__global__ void __launch_bounds__(32) sw_bulk_tma_kernel(const SwSeg* __restrict__ segs, uint32_t nseg,
                                                         uint32_t stage_bytes, uint32_t nstages) {
  sw_bulk_tma_body([segs](uint32_t i) { return segs[i]; }, nseg, stage_bytes, nstages);
}

// Launches with few segments carry the list in the kernel parameter bank: the first bulk load of
// every CTA is not preceded by a read of pinned host memory over PCIe.
// Only the latency-critical small launches take this route: the parameter block stays under the
// classic 4 KiB limit: a much larger parameter block costs more host time per launch than the
// first-segment PCIe read it saves.
constexpr uint32_t SW_BULK_INLINE_SEGS_SMALL = 96;   // 3 KiB
template <uint32_t N>
struct SwSegArgs {
  uint32_t nseg, stage_bytes, nstages, pad;
  SwSeg seg[N];
};
template <uint32_t N>
__global__ void __launch_bounds__(32) sw_bulk_tma_inline_kernel(const __grid_constant__ SwSegArgs<N> a) {
  sw_bulk_tma_body([&a](uint32_t i) { return a.seg[i]; }, a.nseg, a.stage_bytes, a.nstages);
}

// Balanced variant: the jobs (whole messages) travel as kernel parameters and CTA b copies the byte
// range [b * share, (b + 1) * share) of their concatenation (SwJobRangeIter, sw_device.h).  Every SM
// gets the same amount of work whatever the number and size of the messages, and a single 1 MiB
// message is spread over 32 CTAs instead of 2.
__global__ void __launch_bounds__(32) sw_bulk_tma_jobs_kernel(const __grid_constant__ SwBulkJobArgs a) {
  SwJobRangeIter it;
  it.pos = it.range_end = 0;
  it.j = 0;
  if (threadIdx.x == 0) it.init(a, blockIdx.x);
  sw_bulk_tma_pipeline([&](uint64_t& src, uint64_t& dst, uint32_t& bytes) -> bool { return it.next(a, src, dst, bytes); },
                       a.stage_bytes, a.nstages);
}

// ------------------------------------------------------------------ bulk copy, SIMT vectorised
// Generic alignment; one CTA per segment (grid-stride).
__global__ void __launch_bounds__(256) sw_bulk_simt_kernel(const SwSeg* __restrict__ segs, uint32_t nseg) {
  for (uint32_t s = blockIdx.x; s < nseg; s += gridDim.x) {
    const SwSeg g = segs[s];
    sw_copy(reinterpret_cast<uint8_t*>(g.dst), reinterpret_cast<const uint8_t*>(g.src), g.len, threadIdx.x,
            blockDim.x);
  }
}
