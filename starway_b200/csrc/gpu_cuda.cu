// starway_b200 — CUDA (sm_90a) implementation of the swgpu backend interface.
// Compiled with: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

#include "bulk_jobs.h"
#include "gpu.h"
#include "kernels.cuh"
#include "progress.cuh"

namespace swgpu {

static thread_local std::string g_err;
static int g_sms = 132;
static int g_max_smem_optin = 0;
static int g_smem_per_sm = 228 * 1024;
static int g_clk_mhz = 1980;

static int fail(cudaError_t e, const char* what) {
  char buf[256];
  snprintf(buf, sizeof(buf), "%s: %s (%d)", what, cudaGetErrorString(e), (int)e);
  g_err = buf;
  cudaGetLastError();  // clear sticky-less errors
  return -1;
}
#define SW_CUDA(call)                            \
  do {                                           \
    cudaError_t e__ = (call);                    \
    if (e__ != cudaSuccess) return fail(e__, #call); \
  } while (0)

const char* backend_name() { return "cuda-sm_90a"; }
const char* last_error() { return g_err.c_str(); }

int device_count() {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

int init(int device) {
  int n = device_count();
  if (n <= 0) {
    g_err = "no CUDA device visible: starway_b200 has no CPU fallback";
    return -1;
  }
  if (device < 0 || device >= n) {
    g_err = "CUDA device ordinal out of range";
    return -1;
  }
  SW_CUDA(cudaSetDevice(device));
  SW_CUDA(cudaFree(0));
  cudaDeviceProp prop;
  SW_CUDA(cudaGetDeviceProperties(&prop, device));
  g_sms = prop.multiProcessorCount;
  g_max_smem_optin = (int)prop.sharedMemPerBlockOptin;
  g_smem_per_sm = (int)prop.sharedMemPerMultiprocessor;
  {
    int khz = 0;
    if (cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, device) == cudaSuccess && khz > 0) g_clk_mhz = khz / 1000;
    cudaFuncAttributes pa;
    SW_CUDA(cudaFuncGetAttributes(&pa, sw_pull_kernel));
    SW_CUDA(cudaFuncSetAttribute(sw_pull_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)prop.sharedMemPerBlockOptin - (int)pa.sharedSizeBytes));
  }
  cudaFuncAttributes fa;
  SW_CUDA(cudaFuncGetAttributes(&fa, sw_bulk_tma_kernel));
  g_max_smem_optin -= (int)fa.sharedSizeBytes;   // static mbarrier storage counts against the opt-in limit
  SW_CUDA(cudaFuncSetAttribute(sw_bulk_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, g_max_smem_optin));
  SW_CUDA(cudaFuncSetAttribute(sw_bulk_tma_jobs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, g_max_smem_optin));
  SW_CUDA(cudaFuncSetAttribute(sw_bulk_tma_inline_kernel<SW_BULK_INLINE_SEGS_SMALL>,
                               cudaFuncAttributeMaxDynamicSharedMemorySize, g_max_smem_optin));
  SW_CUDA(cudaFuncSetAttribute(sw_reduce_tma_kernel<SW_DT_F32>, cudaFuncAttributeMaxDynamicSharedMemorySize, g_max_smem_optin));
  SW_CUDA(cudaFuncSetAttribute(sw_reduce_tma_kernel<SW_DT_F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, g_max_smem_optin));
  SW_CUDA(cudaFuncSetAttribute(sw_reduce_tma_kernel<SW_DT_BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, g_max_smem_optin));
  SW_CUDA(cudaFuncSetAttribute(sw_reduce_tma_kernel<SW_DT_F64>, cudaFuncAttributeMaxDynamicSharedMemorySize, g_max_smem_optin));
  SW_CUDA(cudaFuncSetAttribute(sw_reduce_tma_kernel<SW_DT_I32>, cudaFuncAttributeMaxDynamicSharedMemorySize, g_max_smem_optin));
  SW_CUDA(cudaFuncSetAttribute(sw_reduce_tma_kernel<SW_DT_I64>, cudaFuncAttributeMaxDynamicSharedMemorySize, g_max_smem_optin));
  return 0;
}
int bind_thread(int device) {
  SW_CUDA(cudaSetDevice(device));
  return 0;
}
int sm_count() { return g_sms; }
int clock_mhz() { return g_clk_mhz; }
int bulk_smem_limit() { return g_max_smem_optin; }
int device_pci_bus_id(int device, char* out, int cap) {
  if (cap < 16) return -1;
  cudaError_t r = cudaDeviceGetPCIBusId(out, cap, device);
  if (r != cudaSuccess) return fail(r, "cudaDeviceGetPCIBusId");
  for (char* p = out; *p; p++)
    if (*p >= 'A' && *p <= 'Z') *p = (char)(*p - 'A' + 'a');   // sysfs spells it in lower case
  return 0;
}

void* dev_alloc(size_t bytes) {
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes ? bytes : 16);
  if (e != cudaSuccess) {
    fail(e, "cudaMalloc");
    return nullptr;
  }
  e = cudaMemset(p, 0, bytes);
  if (e != cudaSuccess) {
    fail(e, "cudaMemset");
    cudaFree(p);
    return nullptr;
  }
  return p;
}
void* dev_alloc_raw(size_t bytes) {
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes ? bytes : 16);
  if (e != cudaSuccess) {
    fail(e, "cudaMalloc");
    return nullptr;
  }
  return p;
}
int dev_free(void* p) {
  if (p) SW_CUDA(cudaFree(p));
  return 0;
}
void* host_alloc(size_t bytes) {
  void* p = nullptr;
  cudaError_t e = cudaHostAlloc(&p, bytes ? bytes : 16, cudaHostAllocPortable | cudaHostAllocMapped);
  if (e != cudaSuccess) {
    fail(e, "cudaHostAlloc");
    return nullptr;
  }
  memset(p, 0, bytes);
  return p;
}
int host_free(void* p) {
  if (p) SW_CUDA(cudaFreeHost(p));
  return 0;
}

int ipc_get(const void* alloc_base, uint8_t handle[64]) {
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ipc handle size");
  cudaIpcMemHandle_t h;
  SW_CUDA(cudaIpcGetMemHandle(&h, const_cast<void*>(alloc_base)));
  memcpy(handle, &h, 64);
  return 0;
}
int ipc_open(const uint8_t handle[64], void** out) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, 64);
  SW_CUDA(cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}
int ipc_close(void* p) {
  SW_CUDA(cudaIpcCloseMemHandle(p));
  return 0;
}

// One driver call (cuPointerGetAttributes, resolved through cudaGetDriverEntryPoint so that the
// library has no link-time libcuda dependency) answers everything the engine needs about a pointer.
int ptr_info(const void* p, PtrInfo* out) {
  memset(out, 0, sizeof(*out));
  typedef int (*attrs_fn)(unsigned int, int*, void**, unsigned long long);
  static attrs_fn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuPointerGetAttributes", &f, cudaEnableDefault, &qr) == cudaSuccess &&
        qr == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<attrs_fn>(f);
    else
      cudaGetLastError();
  });
  if (fn) {
    // CU_POINTER_ATTRIBUTE_MEMORY_TYPE=2, DEVICE_ORDINAL=9, RANGE_START_ADDR=11, RANGE_SIZE=12, BUFFER_ID=7
    int attrs[5] = {2, 9, 11, 12, 7};
    unsigned int mem_type = 0;
    int ordinal = -1;
    unsigned long long start = 0, buffer_id = 0;
    size_t range = 0;
    void* data[5] = {&mem_type, &ordinal, &start, &range, &buffer_id};
    if (fn(5, attrs, data, (unsigned long long)(uintptr_t)p) == 0) {
      if (mem_type == 2 /* CU_MEMORYTYPE_DEVICE */) {
        out->is_device = 1;
        out->device = ordinal;
        out->base = start;
        out->size = range;
        out->buffer_id = buffer_id;
      } else if (mem_type == 1 /* CU_MEMORYTYPE_HOST: pinned / registered */) {
        out->is_pinned = 1;
      } else if (mem_type == 4 /* CU_MEMORYTYPE_UNIFIED */) {
        out->is_device = 1;
        out->device = ordinal;
      }
      return 0;
    }
  }
  cudaPointerAttributes a;
  cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return 0;  // plain host memory unknown to CUDA
  }
  if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) {
    out->is_device = 1;
    out->device = a.device;
  } else if (a.type == cudaMemoryTypeHost) {
    out->is_pinned = 1;
  }
  return 0;
}

stream_t stream_create() {
  cudaStream_t s;
  cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    fail(e, "cudaStreamCreate");
    return nullptr;
  }
  return (stream_t)s;
}
int stream_destroy(stream_t s) {
  SW_CUDA(cudaStreamDestroy((cudaStream_t)s));
  return 0;
}
int stream_query(stream_t s) {
  cudaError_t r = cudaStreamQuery((cudaStream_t)s);
  if (r == cudaSuccess) return 0;
  if (r == cudaErrorNotReady) return 1;
  return fail(r, "cudaStreamQuery");
}
int stream_sync(stream_t s) {
  SW_CUDA(cudaStreamSynchronize((cudaStream_t)s));
  return 0;
}
event_t event_create(int timing) {
  cudaEvent_t e;
  cudaError_t r = cudaEventCreateWithFlags(&e, timing ? cudaEventDefault : cudaEventDisableTiming);
  if (r != cudaSuccess) {
    fail(r, "cudaEventCreate");
    return nullptr;
  }
  return (event_t)e;
}
int event_destroy(event_t e) {
  SW_CUDA(cudaEventDestroy((cudaEvent_t)e));
  return 0;
}
int event_record(event_t e, stream_t s) {
  SW_CUDA(cudaEventRecord((cudaEvent_t)e, (cudaStream_t)s));
  return 0;
}
int event_query(event_t e) {
  cudaError_t r = cudaEventQuery((cudaEvent_t)e);
  if (r == cudaSuccess) return 0;
  if (r == cudaErrorNotReady) return 1;
  return fail(r, "cudaEventQuery");
}
int event_sync(event_t e) {
  SW_CUDA(cudaEventSynchronize((cudaEvent_t)e));
  return 0;
}
float event_elapsed_ms(event_t a, event_t b) {
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, (cudaEvent_t)a, (cudaEvent_t)b) != cudaSuccess) {
    cudaGetLastError();
    return -1.f;
  }
  return ms;
}

int memcpy_h2d(void* dst, const void* src, size_t n, stream_t s) {
  SW_CUDA(cudaMemcpyAsync(dst, src, n, cudaMemcpyHostToDevice, (cudaStream_t)s));
  return 0;
}
int memcpy_batch(void* const* dsts, const void* const* srcs, const size_t* sizes, size_t n, stream_t s) {
  if (n == 0) return 0;
#if CUDART_VERSION >= 12080
  if (n > 1) {
    cudaMemcpyAttributes at;
    memset(&at, 0, sizeof at);
    at.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
    size_t attr_idx = 0, fail = 0;
    cudaError_t e = cudaMemcpyBatchAsync(const_cast<void**>(dsts), (void**)srcs,
                                         const_cast<size_t*>(sizes), n, &at, &attr_idx, 1, &fail, (cudaStream_t)s);
    if (e == cudaSuccess) return 0;
    (void)cudaGetLastError();   // not supported by this driver / for these operands: one copy at a time
  }
#endif
  for (size_t i = 0; i < n; i++) SW_CUDA(cudaMemcpyAsync(dsts[i], srcs[i], sizes[i], cudaMemcpyDefault, (cudaStream_t)s));
  return 0;
}
int memcpy_h2d_batch(void* const* dsts, const void* const* srcs, const size_t* sizes, size_t n, stream_t s) {
  return memcpy_batch(dsts, srcs, sizes, n, s);
}
int memcpy_d2h(void* dst, const void* src, size_t n, stream_t s) {
  SW_CUDA(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, (cudaStream_t)s));
  return 0;
}
int memcpy_d2d(void* dst, const void* src, size_t n, stream_t s) {
  SW_CUDA(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToDevice, (cudaStream_t)s));
  return 0;
}
int memset_dev(void* dst, int v, size_t n, stream_t s) {
  SW_CUDA(cudaMemsetAsync(dst, v, n, (cudaStream_t)s));
  return 0;
}
int upload(void* dst_dev, const void* src_host, size_t n) {
  SW_CUDA(cudaMemcpy(dst_dev, src_host, n, cudaMemcpyHostToDevice));
  return 0;
}

// ---------------------------------------------------------------- match state
struct StateOwner {   // host-side bookkeeping so destroy can free every array
  SwMatchState host;
  SwMatchState* dev;
};
static std::mutex g_states_mu;
static std::vector<StateOwner*> g_states;

SwMatchState* match_state_create(uint32_t heap_small_blocks, uint32_t heap_big_blocks) {
  StateOwner* o = new StateOwner();
  SwMatchState& h = o->host;
  memset(&h, 0, sizeof(h));
#define SW_ALLOC(field, type, count)                       \
  h.field = (type*)dev_alloc(sizeof(type) * (size_t)(count)); \
  if (!h.field) return nullptr;
  SW_ALLOC(p_tag, uint64_t, SW_PQ_CAP);
  SW_ALLOC(p_mask, uint64_t, SW_PQ_CAP);
  SW_ALLOC(p_buf, uint64_t, SW_PQ_CAP);
  SW_ALLOC(p_cap, uint64_t, SW_PQ_CAP);
  SW_ALLOC(p_op, uint64_t, SW_PQ_CAP);
  SW_ALLOC(p_valid, uint32_t, SW_PQ_CAP);
  SW_ALLOC(u_tag, uint64_t, SW_UQ_CAP);
  SW_ALLOC(u_len, uint64_t, SW_UQ_CAP);
  SW_ALLOC(u_data, uint64_t, SW_UQ_CAP);
  SW_ALLOC(u_meta, uint32_t, SW_UQ_CAP);
  SW_ALLOC(u_blk, uint32_t, SW_UQ_CAP);
  h.cap_small = heap_small_blocks;
  h.cap_big = heap_big_blocks;
  SW_ALLOC(heap_small, uint8_t, (size_t)heap_small_blocks * SW_HEAP_SMALL_BYTES);
  SW_ALLOC(heap_big, uint8_t, (size_t)heap_big_blocks * SW_HEAP_BIG_BYTES);
  SW_ALLOC(free_small, uint32_t, heap_small_blocks);
  SW_ALLOC(free_big, uint32_t, heap_big_blocks);
#undef SW_ALLOC
  {
    std::vector<uint32_t> idx(heap_small_blocks > heap_big_blocks ? heap_small_blocks : heap_big_blocks);
    for (size_t i = 0; i < idx.size(); i++) idx[i] = (uint32_t)i;
    if (heap_small_blocks && upload(h.free_small, idx.data(), sizeof(uint32_t) * heap_small_blocks)) return nullptr;
    if (heap_big_blocks && upload(h.free_big, idx.data(), sizeof(uint32_t) * heap_big_blocks)) return nullptr;
  }
  h.n_free_small = heap_small_blocks;
  h.n_free_big = heap_big_blocks;
  o->dev = (SwMatchState*)dev_alloc(sizeof(SwMatchState));
  if (!o->dev) return nullptr;
  if (upload(o->dev, &h, sizeof(h))) return nullptr;
  std::lock_guard<std::mutex> lk(g_states_mu);
  g_states.push_back(o);
  return o->dev;
}

int match_state_destroy(SwMatchState* st) {
  StateOwner* o = nullptr;
  {
    std::lock_guard<std::mutex> lk(g_states_mu);
    for (size_t i = 0; i < g_states.size(); i++)
      if (g_states[i]->dev == st) {
        o = g_states[i];
        g_states.erase(g_states.begin() + i);
        break;
      }
  }
  if (!o) return -1;
  SwMatchState& h = o->host;
  void* ptrs[] = {h.p_tag,  h.p_mask, h.p_buf,      h.p_cap,    h.p_op,       h.p_valid, h.u_tag, h.u_len, h.u_data,
                  h.u_meta, h.u_blk,  h.heap_small, h.heap_big, h.free_small, h.free_big, o->dev};
  for (void* p : ptrs) dev_free(p);
  delete o;
  return 0;
}

int match_state_set_ring(SwMatchState* st, uint32_t ep, void* ring_base, uint32_t slots, uint32_t gen) {
  if (ep >= SW_MAX_EPS) return -1;
  uint64_t base = (uint64_t)(uintptr_t)ring_base;
  uint64_t zero = 0;
  SW_CUDA(cudaMemcpy(&st->ring_gen[ep], &gen, sizeof(gen), cudaMemcpyHostToDevice));
  SW_CUDA(cudaMemcpy(&st->ring_base[ep], &base, sizeof(base), cudaMemcpyHostToDevice));
  SW_CUDA(cudaMemcpy(&st->ring_slots[ep], &slots, sizeof(slots), cudaMemcpyHostToDevice));
  SW_CUDA(cudaMemcpy(&st->ring_cons[ep], &zero, sizeof(zero), cudaMemcpyHostToDevice));
  return 0;
}

// ---------------------------------------------------------------- launches
int launch_put(stream_t s, const SwPutDesc* descs, uint32_t n, const DoneFlag* done) {
  if (!n) return 0;
  const uint32_t warps_per_cta = 8;
  uint32_t n_rts = 0;
  if (n <= SW_PUT_INLINE)
    for (uint32_t i = 0; i < n; i++) n_rts += descs[i].kind == SW_KIND_RTS;
  if (n <= SW_PUT_INLINE && n_rts <= SW_PUT_INLINE_RTS) {
    // descriptors (and RTS payloads, which live in host memory next to them) by value
    SwPutArgs a;
    a.n = n;
    a.pad = 0;
    a.done_flag = done ? (uint64_t)(uintptr_t)done->flag : 0;
    a.done_value = done ? done->value : 0;
    uint32_t r = 0;
    for (uint32_t i = 0; i < n; i++) {
      a.d[i] = descs[i];
      if (descs[i].kind == SW_KIND_RTS) {
        memcpy(&a.r[r], (const void*)(uintptr_t)descs[i].src, sizeof(SwRts));
        a.d[i].src = r++;
      }
    }
    sw_put_inline_kernel<<<1, n * 32, 0, (cudaStream_t)s>>>(a);   // one CTA, one warp per message
    SW_CUDA(cudaGetLastError());
    return done ? 1 : 0;
  }
  uint32_t grid = (n + warps_per_cta - 1) / warps_per_cta;
  const uint32_t cap = (uint32_t)g_sms * 8;
  if (grid > cap) grid = cap;
  sw_put_kernel<<<grid, warps_per_cta * 32, 0, (cudaStream_t)s>>>(descs, n);
  SW_CUDA(cudaGetLastError());
  return 0;
}

int launch_bulk(stream_t s, const SwSeg* segs, uint32_t nseg, const BulkTuning* t) {
  if (!nseg) return 0;
  if (t->mode == 0) {
    int stages = t->stages < 2 ? 2 : (t->stages > SW_BULK_MAX_STAGES ? SW_BULK_MAX_STAGES : t->stages);
    int sb = t->stage_bytes & ~15;
    if (sb < 1024) sb = 1024;
    size_t smem = (size_t)stages * sb;
    if ((int)smem > g_max_smem_optin) {
      g_err = "bulk tuning exceeds shared memory";
      return -1;
    }
    int ctas = t->ctas_per_sm > 0 ? t->ctas_per_sm : 1;
    const int fit = (int)((size_t)g_smem_per_sm / (smem + 1024 + 128));   // CTAs of this size resident per SM
    if (ctas > fit) ctas = fit < 1 ? 1 : fit;
    uint32_t grid = (uint32_t)(g_sms * ctas);
    SwBulkJobArgs ja;
    uint32_t jgrid = 0;
    if (t->balance && bulk_build_jobs(segs, nseg, grid, (uint32_t)sb, (uint32_t)stages, &ja, &jgrid)) {
      sw_bulk_tma_jobs_kernel<<<jgrid, 32, smem, (cudaStream_t)s>>>(ja);
      SW_CUDA(cudaGetLastError());
      return 0;
    }
    if (grid > nseg) grid = nseg;
    if (nseg <= SW_BULK_INLINE_SEGS_SMALL) {
      SwSegArgs<SW_BULK_INLINE_SEGS_SMALL> a;
      a.nseg = nseg;
      a.stage_bytes = (uint32_t)sb;
      a.nstages = (uint32_t)stages;
      a.pad = 0;
      memcpy(a.seg, segs, sizeof(SwSeg) * nseg);
      sw_bulk_tma_inline_kernel<SW_BULK_INLINE_SEGS_SMALL><<<grid, 32, smem, (cudaStream_t)s>>>(a);
    } else {
      sw_bulk_tma_kernel<<<grid, 32, smem, (cudaStream_t)s>>>(segs, nseg, (uint32_t)sb, (uint32_t)stages);
    }
  } else {
    uint32_t grid = (uint32_t)(g_sms * (t->ctas_per_sm > 0 ? t->ctas_per_sm : 4));
    if (grid > nseg) grid = nseg;
    sw_bulk_simt_kernel<<<grid, 256, 0, (cudaStream_t)s>>>(segs, nseg);
  }
  SW_CUDA(cudaGetLastError());
  return 0;
}

template <int DT>
static void launch_reduce_as(cudaStream_t s, const SwSeg* segs, uint32_t nseg, int tma, uint32_t grid, size_t smem,
                             uint32_t sb, uint32_t stages) {
  if (tma)
    sw_reduce_tma_kernel<DT><<<grid, 32, smem, s>>>(segs, nseg, sb, stages);
  else
    sw_reduce_simt_kernel<DT><<<grid, 256, 0, s>>>(segs, nseg);
}

int launch_reduce(stream_t s, const SwSeg* segs, uint32_t nseg, int dtype, const BulkTuning* t) {
  if (!nseg) return 0;
  const int tma = t->mode == 0;
  int stages = t->stages < 2 ? 2 : (t->stages > SW_BULK_MAX_STAGES ? SW_BULK_MAX_STAGES : t->stages);
  int sb = t->stage_bytes & ~15;
  if (sb < 1024) sb = 1024;
  const size_t smem = (size_t)stages * sb;
  int ctas = t->ctas_per_sm > 0 ? t->ctas_per_sm : 1;
  if (tma) {
    if ((int)smem > g_max_smem_optin) {
      g_err = "bulk tuning exceeds shared memory";
      return -1;
    }
    const int fit = (int)((size_t)g_smem_per_sm / (smem + 1024 + 128));   // CTAs of this size resident per SM
    if (ctas > fit) ctas = fit < 1 ? 1 : fit;
  }
  uint32_t grid = (uint32_t)(g_sms * ctas);
  if (grid > nseg) grid = nseg;
  cudaStream_t cs = (cudaStream_t)s;
  switch (dtype) {
    case SW_DT_F32: launch_reduce_as<SW_DT_F32>(cs, segs, nseg, tma, grid, smem, (uint32_t)sb, (uint32_t)stages); break;
    case SW_DT_F16: launch_reduce_as<SW_DT_F16>(cs, segs, nseg, tma, grid, smem, (uint32_t)sb, (uint32_t)stages); break;
    case SW_DT_BF16: launch_reduce_as<SW_DT_BF16>(cs, segs, nseg, tma, grid, smem, (uint32_t)sb, (uint32_t)stages); break;
    case SW_DT_F64: launch_reduce_as<SW_DT_F64>(cs, segs, nseg, tma, grid, smem, (uint32_t)sb, (uint32_t)stages); break;
    case SW_DT_I32: launch_reduce_as<SW_DT_I32>(cs, segs, nseg, tma, grid, smem, (uint32_t)sb, (uint32_t)stages); break;
    case SW_DT_I64: launch_reduce_as<SW_DT_I64>(cs, segs, nseg, tma, grid, smem, (uint32_t)sb, (uint32_t)stages); break;
    default:
      g_err = "launch_reduce: unknown element type";
      return -1;
  }
  SW_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------- resident progress path
int resident_lingers() { return 1; }

void* host_register(void* p, size_t bytes) {
  cudaError_t e = cudaHostRegister(p, bytes, cudaHostRegisterPortable | cudaHostRegisterMapped);
  if (e != cudaSuccess) {
    fail(e, "cudaHostRegister");
    return nullptr;
  }
  void* d = nullptr;
  e = cudaHostGetDevicePointer(&d, p, 0);
  if (e != cudaSuccess) {
    fail(e, "cudaHostGetDevicePointer");
    cudaHostUnregister(p);
    return nullptr;
  }
  return d;
}
int host_unregister(void* p) {
  if (p) SW_CUDA(cudaHostUnregister(p));
  return 0;
}

int match_state_set_ep_words(SwMatchState* st, uint32_t ep, void* credit_word, void* fin_words) {
  if (ep >= SW_MAX_EPS) return -1;
  uint64_t c = (uint64_t)(uintptr_t)credit_word, f = (uint64_t)(uintptr_t)fin_words;
  SW_CUDA(cudaMemcpy(&st->credit_ptr[ep], &c, sizeof(c), cudaMemcpyHostToDevice));
  SW_CUDA(cudaMemcpy(&st->fin_ptr[ep], &f, sizeof(f), cudaMemcpyHostToDevice));
  return 0;
}

SwPullQueue* pull_queue_create() { return (SwPullQueue*)dev_alloc(sizeof(SwPullQueue)); }
int pull_queue_destroy(SwPullQueue* q) { return dev_free(q); }
SwMapEnt* map_table_create() { return (SwMapEnt*)dev_alloc(sizeof(SwMapEnt) * SW_MAP_SLOTS); }
int map_table_destroy(SwMapEnt* t) { return dev_free(t); }
static void map_shadow_reset(SwMapEnt* t);
int map_table_clear(SwMapEnt* t) {
  SW_CUDA(cudaMemset(t, 0, sizeof(SwMapEnt) * SW_MAP_SLOTS));
  map_shadow_reset(t);
  return 0;
}
// The host keeps a shadow of the occupied slots; entries are only ever added (or the table is cleared while no
// control kernel runs).  Body first, then the key the device compares: two stream-ordered copies.
static std::mutex g_map_mu;
static std::vector<std::pair<SwMapEnt*, std::vector<uint8_t>>> g_map_shadow;
int map_table_insert(SwMapEnt* t, stream_t s, uint64_t uuid, uint64_t buf_id, uint64_t remote_base, uint64_t local_base) {
  std::lock_guard<std::mutex> lk(g_map_mu);
  std::vector<uint8_t>* used = nullptr;
  for (auto& kv : g_map_shadow)
    if (kv.first == t) used = &kv.second;
  if (!used) {
    g_map_shadow.emplace_back(t, std::vector<uint8_t>(SW_MAP_SLOTS, 0));
    used = &g_map_shadow.back().second;
  }
  const uint32_t home = sw_map_home(uuid, buf_id);
  for (uint32_t k = 0; k < SW_MAP_PROBE; k++) {
    const uint32_t i = (home + k) & (SW_MAP_SLOTS - 1);
    if ((*used)[i]) continue;
    (*used)[i] = 1;
    uint64_t body[2] = {remote_base, local_base}, key[2] = {uuid, buf_id};
    SW_CUDA(cudaMemcpyAsync(&t[i].remote_base, body, sizeof(body), cudaMemcpyHostToDevice, (cudaStream_t)s));
    SW_CUDA(cudaMemcpyAsync(&t[i].uuid, key, sizeof(key), cudaMemcpyHostToDevice, (cudaStream_t)s));
    return 0;
  }
  g_err = "mapping table: probe window full";
  return -1;
}

static void map_shadow_reset(SwMapEnt* t) {
  std::lock_guard<std::mutex> lk(g_map_mu);
  for (auto& kv : g_map_shadow)
    if (kv.first == t) std::fill(kv.second.begin(), kv.second.end(), 0);
}

// ---- measurement hook: one batch published from the device, like sw_res_flush_pull does
__global__ void sw_probe_publish_kernel(SwPullQueue* q, const SwSeg* msgs, uint32_t n, uint32_t pull_ctas, uint8_t* scratch) {
  if (threadIdx.x) return;
  const uint64_t ticket = atomicAdd(reinterpret_cast<unsigned long long*>(&q->alloc), 1ull);
  SwPullSlot* s = &q->slot[ticket % SW_PULL_SLOTS];
  const uint64_t want = ticket >= SW_PULL_SLOTS ? ticket - SW_PULL_SLOTS + 1 : 0;
  while (sw_ld_acquire_gpu(&s->free_seq) != want) __nanosleep(100);
  uint64_t total = 0;
  for (uint32_t j = 0; j < n; j++) {
    total += msgs[j].len & ~15ull;
    s->end[j] = total;
    s->src[j] = msgs[j].src;
    s->dst[j] = msgs[j].dst;
    s->meta[j].op_id = j;
    s->meta[j].tag = 0;
    s->meta[j].len = msgs[j].len;
    s->meta[j].fin_addr = 0;
    s->meta[j].fin_val = 0;
  }
  uint64_t chunk = total / (pull_ctas > 1 ? pull_ctas - 1 : 1) + 1023;
  chunk &= ~1023ull;
  if (chunk < 8192) chunk = 8192;
  if (chunk > 262144) chunk = 262144;
  uint64_t nch = (total + chunk - 1) / chunk;
  if (!nch) nch = 1;
  s->njobs = n;
  s->nchunks = (uint32_t)nch;
  s->exit = 0;
  s->chunk_bytes = chunk;
  s->total = total;
  s->next_chunk = s->done_chunks = s->retire = 0;
  s->t_first = 0;
  s->t_pub = sw_globaltimer();
  // completion records of the probe go to a scratch ring nobody reads; its "host cursor" follows the allocation
  // cursor, so the ring never looks full
  s->cqr_ring = reinterpret_cast<uint64_t>(scratch + 4096);
  s->cqr_alloc = reinterpret_cast<uint64_t>(scratch);
  s->cqr_head_dev = reinterpret_cast<uint64_t>(scratch + 8);
  s->cqr_head_host = reinterpret_cast<uint64_t>(scratch + 8);
  *reinterpret_cast<volatile uint64_t*>(scratch + 8) = *reinterpret_cast<volatile uint64_t*>(scratch);
  __threadfence();
  sw_st_release_gpu(&s->seq, ticket + 1);
}
int probe_publish_batch(stream_t s, SwPullQueue* q, const SwSeg* msgs_pinned, uint32_t n, uint32_t pull_ctas, void* scratch_dev) {
  if (n > SW_PULL_JOBS) return -1;
  sw_probe_publish_kernel<<<1, 32, 0, (cudaStream_t)s>>>(q, msgs_pinned, n, pull_ctas, (uint8_t*)scratch_dev);
  SW_CUDA(cudaGetLastError());
  return 0;
}
int pull_queue_read_stats(SwPullQueue* q, uint64_t out[8]) {
  SwPullQueue h;
  SW_CUDA(cudaMemcpy(&h, q, offsetof(SwPullQueue, slot), cudaMemcpyDeviceToHost));
  out[0] = h.bytes;
  out[1] = h.busy_ns;
  out[2] = h.batches;
  out[3] = h.jobs;
  out[4] = h.pickup_ns;
  out[5] = h.copy_ns;
  out[6] = h.fin_ns;
  out[7] = h.alloc;
  return 0;
}

int pull_default_ctas() { return g_sms > 4 ? g_sms - 2 : g_sms; }

int launch_progress(stream_t s, const ProgressLaunch* p) {
  SwProgArgs a;
  a.st = p->st;
  a.ctl = p->ctl;
  a.posts = p->posts;
  a.cq = p->cq;
  a.cqr = p->cqr;
  a.hr = p->hr;
  a.sends = p->sends;
  a.pq = p->pq;
  a.map = p->map;
  a.ctx_uuid = p->ctx_uuid;
  a.launch_seq = p->launch_seq;
  a.pid = p->pid;
  a.n_eps = p->n_eps;
  a.linger_us = p->linger_us;
  a.max_life_us = p->max_life_us;
  a.pull_ctas = p->pull_ctas;
  a.clk_mhz = (uint32_t)g_clk_mhz;
  sw_progress_kernel<<<1, SW_PROG_THREADS, 0, (cudaStream_t)s>>>(a);
  SW_CUDA(cudaGetLastError());
  return 0;
}

int launch_pull(stream_t s, SwPullQueue* q, SwPullCtl* ctl, uint64_t launch_seq, uint32_t ctas, uint32_t linger_us,
                uint32_t max_life_us, const BulkTuning* t) {
  int stages = t->stages < 3 ? 3 : (t->stages > SW_BULK_MAX_STAGES ? SW_BULK_MAX_STAGES : t->stages);
  int sb = t->stage_bytes & ~15;
  if (sb < 1024) sb = 1024;
  SwPullArgs a;
  a.q = q;
  a.ctl = ctl;
  a.launch_seq = launch_seq;
  a.stage_bytes = (uint32_t)sb;
  a.nstages = (uint32_t)stages;
  a.linger_us = linger_us;
  a.max_life_us = max_life_us;
  a.clk_mhz = (uint32_t)g_clk_mhz;
  a.pad = 0;
  sw_pull_kernel<<<ctas, 64, (size_t)stages * sb, (cudaStream_t)s>>>(a);
  SW_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace swgpu
