// starway_b200 — layouts shared by the host progress engine and the sm_90a kernels.
//
// Everything in this file is plain-old-data that lives either in device memory
// (rings, queues, job lists), in pinned host memory (per-launch input/output
// blocks) or in POSIX shared memory (control block between two workers).
//
// Reference being replaced: the wire/queue state that libucp keeps behind
// ucp_tag_send_nbx / ucp_tag_recv_nbx / ucp_worker_progress
// (reference src/bindings/main.cpp:370,404,362 and :1136,1172,1127).
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define SW_HD __host__ __device__
#else
#define SW_HD
#endif

// ---------------------------------------------------------------- inbound ring
// One ring per inbound endpoint, owned by the receiving worker, written by the
// sending worker's put kernel through a peer mapping (NVLink stores) or a plain
// pointer (same process).  A slot is a fixed 8 KiB landing zone.
constexpr uint32_t SW_SLOT_BYTES = 8192;
constexpr uint32_t SW_SLOT_HDR = 64;
constexpr uint32_t SW_EAGER_MAX = SW_SLOT_BYTES - SW_SLOT_HDR;  // 8128 B payload
constexpr uint32_t SW_RING_SLOTS_DEFAULT = 1024;                // 8 MiB per endpoint

enum : uint32_t { SW_KIND_EAGER = 1, SW_KIND_RTS = 2 };
// SwSendEnt only (puts executed by the resident control kernel): the destination ring is in the memory of the GPU the
// kernel runs on, so the arrival flag is released at device scope (~0.3 us) instead of system scope (~1.5 us)
constexpr uint32_t SW_KIND_SAME_GPU = 0x80000000u;

struct SwSlotHdr {     // 64 B, 16 B aligned, written after the payload by the put kernel
  uint64_t tag;        // sender tag (full uint64)
  uint64_t len;        // message length in bytes (for RTS: length of the remote payload)
  uint64_t seq;        // 1-based slot sequence number on this ring: the ARRIVAL FLAG, stored last with release
                       // semantics at system scope; the receiver's control kernel polls it with ld.acquire.sys
  uint32_t kind;       // SW_KIND_*
  uint32_t magic;      // SW_SLOT_MAGIC
  uint64_t pad[4];
};
constexpr uint32_t SW_SLOT_MAGIC = 0x53574d47u;  // "SWMG"

// Rendezvous request-to-send descriptor; travels as the payload of an RTS slot so
// that it stays ordered with the eager messages of the same sender (non-overtaking).
struct SwRts {            // 128 B
  uint8_t ipc_handle[64];  // cudaIpcMemHandle_t of the allocation holding the source
  uint64_t alloc_base;     // sender-side virtual address of the allocation base
  uint64_t alloc_size;     // size of that allocation
  uint64_t src_ptr;        // sender-side virtual address of the payload
  uint64_t send_seq;       // sender's rendezvous sequence number (echoed in FIN)
  uint64_t ctx_uuid;       // sender context id (same value => same process => direct ptr)
  uint32_t src_pid;
  int32_t src_dev;         // CUDA ordinal of the source memory (-1: unknown)
  uint64_t pad[2];         // [0]: SW_RTS_* flags; [1]: CUDA buffer id of the source allocation (key of the receiver's
                           //      device-resident mapping table; 0: unknown)
};
static_assert(sizeof(SwRts) == 128, "SwRts layout");
static_assert(sizeof(SwSlotHdr) == 64, "SwSlotHdr layout");

// ---------------------------------------------------------------- put kernel input
struct SwPutDesc {   // pinned host, read by the put kernel
  uint64_t src;      // payload source (device ptr, or pinned-host staging ptr)
  uint64_t dst;      // destination slot base (peer-mapped or local device ptr)
  uint64_t tag;
  uint64_t seq;      // ring sequence number for the slot header
  uint32_t len;      // payload bytes to copy into the slot (<= SW_EAGER_MAX)
  uint32_t kind;     // SW_KIND_*
  uint64_t msg_len;  // value for SwSlotHdr.len (== len for eager; remote length for RTS)
};
static_assert(sizeof(SwPutDesc) == 48, "SwPutDesc layout");

// ---------------------------------------------------------------- matching
constexpr uint32_t SW_MAX_EPS = 64;          // inbound endpoints per worker

// Completion status codes (values mirror the UCX codes the reference forwards
// through ucs_status_string; see sw_status_string in the C-ABI).
enum : int32_t {
  SW_OK = 0,
  SW_ERR_MESSAGE_TRUNCATED = -9,
  SW_ERR_CANCELED = -16,
  SW_ERR_NOT_CONNECTED = -24,
  SW_ERR_CONNECTION_RESET = -25,
  SW_ERR_INVALID_PARAM = -5,
  SW_ERR_NO_MEMORY = -4,
  SW_ERR_IO_ERROR = -3,
  SW_ERR_UNREACHABLE = -6,
  SW_ERR_TIMED_OUT = -20,
  SW_ERR_BUSY = -15,
};

struct SwRndvRec {  // a rendezvous match handed to the host (inside SwHrEnt): the receiver pulls the payload
  uint64_t op_id;
  uint64_t dst;
  uint64_t cap;
  uint64_t tag;
  uint64_t len;
  uint32_t ep;
  int32_t status;   // SW_OK or SW_ERR_MESSAGE_TRUNCATED
  SwRts rts;
};

// ---------------------------------------------------------------- device-resident queues
// Posted-receive queue and unexpected-message queue of one worker.  Both are
// power-of-two rings addressed by monotonically increasing logical indices;
// removal from the middle leaves a tombstone (valid = 0).
constexpr uint32_t SW_PQ_CAP = 1u << 16;
constexpr uint32_t SW_UQ_CAP = 1u << 16;
constexpr uint32_t SW_HEAP_SMALL_BYTES = 256;
constexpr uint32_t SW_HEAP_BIG_BYTES = SW_EAGER_MAX;

struct SwMatchState {   // device memory, one per worker
  // posted queue (SoA)
  uint64_t p_head, p_tail;
  uint64_t* p_tag;
  uint64_t* p_mask;
  uint64_t* p_buf;
  uint64_t* p_cap;
  uint64_t* p_op;
  uint32_t* p_valid;
  uint32_t p_count;      // valid entries
  // unexpected queue (SoA)
  uint32_t u_count;
  uint64_t u_head, u_tail;
  uint64_t* u_tag;
  uint64_t* u_len;       // full message length
  uint64_t* u_data;      // heap block holding the eager payload / the SwRts
  uint32_t* u_meta;      // bit31 valid | bit30 big-block | bit29 RTS | low bits: ep
  uint32_t* u_blk;       // heap block index
  // inbound rings
  uint64_t ring_base[SW_MAX_EPS];
  uint32_t ring_slots[SW_MAX_EPS];   // power of two
  uint64_t ring_cons[SW_MAX_EPS];    // slots consumed so far
  uint64_t credit_ptr[SW_MAX_EPS];   // resident path: device-visible address of the sender-visible `consumed` word
  uint64_t fin_ptr[SW_MAX_EPS];      // resident path: device-visible address of the FIN words of that connection
  uint32_t ring_gen[SW_MAX_EPS];     // generation of the ring index (a retired endpoint's index is reused): travels
                                     // with unexpected rendezvous requests so that a stale one is never pulled
  // unexpected heap: two size classes, stacks of free block indices.  The control kernel pushes a block back once
  // nothing reads it any more: at once when the matcher warp has copied the payload or read the rendezvous
  // descriptor, else when the helper warp that copies the payload has finished.
  uint8_t* heap_small;  uint32_t* free_small;  uint32_t n_free_small;  uint32_t cap_small;
  uint8_t* heap_big;    uint32_t* free_big;    uint32_t n_free_big;    uint32_t cap_big;
  uint32_t rr_ep;        // round-robin start endpoint
  // resident path: cursors that survive from one launch of the control kernel to the next
  uint64_t cq_alloc;       // eager completion records written so far
  uint64_t hr_alloc;       // host-path rendezvous records written so far
  uint64_t pull_jobs;      // rendezvous jobs handed to the pull queue so far
  uint64_t arrivals;       // ring slots consumed so far
  uint64_t post_consumed;  // receives taken from the post ring so far
  uint64_t cqr_alloc;      // rendezvous completion records allocated by pull CTAs (atomic)
  uint64_t cqr_head;       // device copy of the host's cursor into the rendezvous completion ring
  uint64_t send_consumed;  // put descriptors taken from the send ring so far
};

constexpr uint32_t SW_UMETA_VALID = 1u << 31;
constexpr uint32_t SW_UMETA_BIG = 1u << 30;
constexpr uint32_t SW_UMETA_RTS = 1u << 29;
constexpr uint32_t SW_UMETA_EPMASK = 0xFFFFu;   // bits 0-5: ring index, bits 6-15: generation of that index
constexpr uint32_t SW_EP_IDX_BITS = 6, SW_EP_GEN_MASK = 0x3FFu;
static_assert(SW_MAX_EPS <= (1u << SW_EP_IDX_BITS), "ring index field");

// ---------------------------------------------------------------- resident progress path
// The receive side of a worker is driven by a RESIDENT (bounded-lifetime) control kernel: it polls the slot headers of the inbound rings in device memory
// (release/acquire on the header's sequence word -- no host doorbell on the data path), takes new
// receives from a ring in pinned host memory, matches, delivers eager payloads, publishes credits and
// completion records straight to host-visible memory, and hands rendezvous matches to a pool of
// resident pull CTAs (sw_pull_kernel) through a queue in device memory.  The kernels exit on their own
// after `linger` of silence or `max_life`, so device-wide synchronisations of the application
// (cudaFree, cudaDeviceSynchronize) never wait long; the host relaunches them while work is expected.
constexpr uint32_t SW_POST_RING = 4096;     // host -> device: new receives (pinned host memory)
constexpr uint32_t SW_CQ_RING = 16384;      // device -> host: completion records (pinned host memory)
constexpr uint32_t SW_HR_RING = 2048;       // device -> host: rendezvous matches the host must copy
constexpr uint32_t SW_FIN_SLOTS = 1024;     // rendezvous FIN words per direction (control block)
constexpr uint32_t SW_PULL_SLOTS = 8;       // pull batches in flight per context
constexpr uint32_t SW_PULL_JOBS = 64;       // messages per pull batch
constexpr uint32_t SW_MAP_SLOTS = 8192;     // device-resident (exporter, allocation) -> mapped base table
constexpr uint32_t SW_MAP_PROBE = 32;       // one warp-wide probe
constexpr uint32_t SW_INLINE_DELIVER = 256; // eager payloads up to this size are copied by the matcher warp itself
constexpr uint32_t SW_SEND_RING = 64;       // host -> device: put descriptors executed by the resident control kernel

enum : uint32_t {
  SW_POST_HOSTPATH = 1,   // a rendezvous into this receive is copied by a host-launched kernel
  SW_POST_HOSTBUF = 2,    // the landing buffer is host memory (pinned bounce): payload and record need a system-scope fence
};
enum : uint64_t { SW_RTS_PINNED_SRC = 1 };  // SwRts::pad[0]: the source is pinned host memory

struct SwSendEnt {   // pinned host: one put for the resident control kernel of the sending worker
  SwPutDesc d;       // d.src == 0: the payload (<= 128 B: an RTS descriptor, a small host payload) is in `inl`
  uint8_t inl[128];
};
static_assert(sizeof(SwSendEnt) == 176, "SwSendEnt layout");

// The ring itself holds the entry in 16-byte units of 12 data bytes + a 4-byte stamp (the entry's index): the link
// warp reads the next expected entry in the SAME load instruction as the control words, without waiting for the
// host's cursor to cover it, and takes it when every unit carries the stamp.  A unit is written with one 16-byte
// store and read in one piece, so a stamped unit is a whole unit; units of an older entry carry an older stamp.
constexpr uint32_t SW_SEND_WORDS = sizeof(SwSendEnt) / 4;            // 44
constexpr uint32_t SW_SEND_UNITS = (SW_SEND_WORDS + 2) / 3;         // 15
struct alignas(16) SwSendLL {
  uint32_t u[16][4];   // unit k: words 3k .. 3k+2 of the SwSendEnt, then the stamp; unit 15 is unused
};
static_assert(sizeof(SwSendLL) == 256, "SwSendLL layout");
SW_HD inline uint32_t sw_send_stamp(uint64_t index) { return (static_cast<uint32_t>(index + 1) & 0x7fffffffu) | 0x80000000u; }

struct SwPostEnt {   // pinned host: one posted receive on its way to the control kernel
  uint64_t tag, mask, buf, cap, op_id;
  uint32_t flags, pad;
};
static_assert(sizeof(SwPostEnt) == 48, "SwPostEnt layout");

struct SwCqEnt {     // pinned host: `seq` (pass number of the ring, never 0) is written last
  uint64_t op_id, tag, len;
  int32_t status;
  uint32_t seq;
};
static_assert(sizeof(SwCqEnt) == 32, "SwCqEnt layout");
SW_HD static inline uint32_t sw_ring_pass(uint64_t idx, uint32_t cap) { return static_cast<uint32_t>(idx / cap) + 1; }

struct SwHrEnt {     // pinned host: a rendezvous match handed to the host (`seq` written last)
  SwRndvRec rec;
  uint32_t pad;
  uint32_t seq;
};

struct SwMapEnt {    // device memory: key = (exporting context, CUDA buffer id of the allocation)
  uint64_t uuid, buf_id;   // buf_id == 0: empty
  uint64_t remote_base, local_base;
};
SW_HD static inline uint32_t sw_map_home(uint64_t uuid, uint64_t buf_id) {
  uint64_t h = (uuid ^ (buf_id * 0x9E3779B97F4A7C15ull)) * 0xD6E8FEB86659FD93ull;
  return static_cast<uint32_t>(h >> 40) & (SW_MAP_SLOTS - 1);
}

// Words shared between the host engine and the control kernel of one worker (pinned host memory).
struct SwProgCtl {
  // host -> kernel
  alignas(64) volatile uint64_t post_tail;   // receives written into the post ring so far
  volatile uint64_t cq_head;                 // eager completion records consumed by the host
  volatile uint64_t cqr_head;                // rendezvous completion records consumed by the host
  volatile uint64_t hr_head;                 // host-path rendezvous records consumed by the host
  volatile uint64_t send_tail;               // put descriptors written into the send ring so far
  volatile uint64_t pad_s;
  alignas(64) volatile uint64_t stop;        // != 0: leave as soon as the state is consistent
  volatile uint64_t dead_mask;               // endpoints (bit = ring index) whose rendezvous go to the host
  volatile uint64_t host_epoch;              // bumped by the host; echoed in dev_epoch by a later iteration
  volatile uint64_t pad0;
  // kernel -> host
  alignas(64) volatile uint64_t post_head;   // receives taken from the post ring
  volatile uint64_t dev_epoch;
  volatile uint64_t exit_seq;                // launch number of the last launch that has ended
  volatile uint64_t pull_jobs;               // rendezvous jobs handed to the pull queue so far
  volatile uint64_t arrivals;                // ring slots consumed so far
  volatile uint64_t n_posted, n_unexp;       // queue depths at exit
  volatile uint64_t err;                     // consistency errors seen by the matcher
  volatile uint64_t stalled;                 // a ring is blocked on the unexpected heap (needs new receives)
  volatile uint64_t iterations;
  volatile uint64_t send_head;               // put descriptors taken from the send ring
  volatile uint64_t send_done;               // put descriptors executed (slot written, header released)
  volatile uint64_t exit_reason;             // why the last launch left: 1 host request, 2 silence (linger), 3 lifetime
  volatile uint64_t life_us;                 // how long it ran
  // clock sums for the latency budget of resident puts (SM clocks; [0] count, [1] first sight of a new descriptor
  // -> staged in shared memory, [2] staged -> slot written and header released, [3] released -> send_done
  // published, [4] link-warp rounds, [5] link-warp clocks)
  volatile uint64_t dbg[8];
};

// ---- pull queue: rendezvous copies executed by the resident pull CTAs of the context
struct SwPullMeta {       // completion of one pulled message
  uint64_t op_id, tag, len;
  uint64_t fin_addr;      // word in the sender-visible control block (0: none)
  uint64_t fin_val;
};
struct SwPullSlot {
  uint64_t seq;           // ticket + 1 once published (release); compared by the workers
  uint64_t free_seq;      // ticket + 1 of the last batch retired from this slot
  uint64_t fin_seq;       // == seq once CTA 0 of the pull kernel has completed the batch
  uint32_t njobs, nchunks, exit, pad;
  uint64_t chunk_bytes, total;
  uint32_t next_chunk, done_chunks, retire, pad2;
  uint64_t t_first;       // globaltimer of the first claim
  uint64_t t_pub;         // globaltimer when the matcher published the batch
  // where the completion records of this batch go (the receiving worker's rendezvous CQ)
  uint64_t cqr_ring, cqr_alloc, cqr_head_dev, cqr_head_host;
  uint64_t end[SW_PULL_JOBS], src[SW_PULL_JOBS], dst[SW_PULL_JOBS];
  SwPullMeta meta[SW_PULL_JOBS];
};
struct SwPullQueue {      // device memory, one per context
  uint64_t alloc;         // next ticket (atomic)
  uint64_t start;         // first ticket the next pull launch looks at
  uint64_t bytes, busy_ns, last_end, batches, jobs;   // statistics (roofline: bytes / busy_ns)
  uint64_t pickup_ns, copy_ns, fin_ns;                // per-batch phases: published -> first claim -> last chunk -> records out
  SwPullSlot slot[SW_PULL_SLOTS];
};
struct SwPullCtl {        // pinned host, one per context
  alignas(64) volatile uint64_t stop;     // host -> kernel: publish an EXIT batch
  alignas(64) volatile uint64_t exited;   // kernel -> host: launch number of the last launch whose CTA 0 left
  volatile uint64_t bytes, busy_ns, batches, jobs;   // copies of the queue statistics at exit
  volatile uint64_t pickup_ns, copy_ns, fin_ns;
};

// ---------------------------------------------------------------- bulk copy input
struct SwSeg {        // one contiguous piece of a rendezvous/loopback copy
  uint64_t src;
  uint64_t dst;
  uint64_t len;
  uint64_t pad;
};

// Balanced bulk copy: the launch carries its jobs (whole messages, at most SW_BULK_INLINE_JOBS of them)
// in the kernel parameter bank and every CTA takes an equal, contiguous byte range of their
// concatenation -- no segment list in host memory, no idle SMs when the launch has fewer segments
// than the GPU has SMs.  The iterator below is the ONLY place that maps (CTA, progress) to addresses;
// the CPU stand-in backend runs the same code, so every host-logic test exercises it.
constexpr uint32_t SW_BULK_INLINE_JOBS = 96;
struct SwBulkJobArgs {
  uint32_t njobs, stage_bytes, nstages, pad;
  uint64_t share;                        // bytes per CTA (multiple of 1024)
  uint64_t end[SW_BULK_INLINE_JOBS];     // end[j] = total bytes of jobs 0..j
  uint64_t src[SW_BULK_INLINE_JOBS];
  uint64_t dst[SW_BULK_INLINE_JOBS];
};
static_assert(sizeof(SwBulkJobArgs) <= 4096 - 512, "bulk job parameters stay under the classic 4 KiB parameter limit");

struct SwJobRangeIter {
  uint64_t pos, range_end;
  uint32_t j;
  SW_HD void init(const SwBulkJobArgs& a, uint32_t cta) {
    const uint64_t total = a.njobs ? a.end[a.njobs - 1] : 0;
    pos = static_cast<uint64_t>(cta) * a.share;
    if (pos > total) pos = total;
    range_end = pos + a.share;
    if (range_end > total) range_end = total;
    j = 0;
    while (j < a.njobs && a.end[j] <= pos) j++;
  }
  // next piece of at most stage_bytes that stays inside one job and inside this CTA's range
  SW_HD bool next(const SwBulkJobArgs& a, uint64_t& src, uint64_t& dst, uint32_t& bytes) {
    if (pos >= range_end) return false;
    while (a.end[j] <= pos) j++;   // pos < range_end <= end[njobs-1]: terminates inside the array
    const uint64_t begin = j ? a.end[j - 1] : 0;
    const uint64_t stop = a.end[j] < range_end ? a.end[j] : range_end;
    const uint64_t left = stop - pos;
    bytes = left < a.stage_bytes ? static_cast<uint32_t>(left) : a.stage_bytes;
    src = a.src[j] + (pos - begin);
    dst = a.dst[j] + (pos - begin);
    pos += bytes;
    return true;
  }
};

// Match rule of the UCP tag API as used at reference main.cpp:404,1172:
// a receive (tag, mask) accepts a message with sender tag `stag` iff
// ((stag ^ tag) & mask) == 0.
SW_HD static inline bool sw_tag_match(uint64_t stag, uint64_t tag, uint64_t mask) {
  return ((stag ^ tag) & mask) == 0;
}
