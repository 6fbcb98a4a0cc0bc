// starway_b200 — hand-written sm_90a kernels for the tagged-messaging hot path.
//
//   sw_put_kernel       eager / RTS put: vectorised stores into the peer's inbound ring
//   sw_put_inline_kernel  same, descriptors + RTS payloads as kernel parameters (batches <= 32)
//                       (replaces the eager leg of ucp_tag_send_nbx, reference main.cpp:370,1136)
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

__device__ __forceinline__ uint64_t sw_shfl64(uint64_t v, int src) {
  uint32_t lo = __shfl_sync(0xffffffffu, static_cast<uint32_t>(v), src);
  uint32_t hi = __shfl_sync(0xffffffffu, static_cast<uint32_t>(v >> 32), src);
  return (static_cast<uint64_t>(hi) << 32) | lo;
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
