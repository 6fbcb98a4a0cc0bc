/* starway_b200.h — C ABI of the GPU-native (sm_90a) tagged-messaging engine.
 *
 * This is the drop-in boundary for the reference's `_bindings` extension module
 * (reference src/starway/_bindings.pyi:7-88, bound at src/bindings/main.cpp:1538-1581).
 * The reference exposes nanobind classes whose methods take Python callbacks; here
 * every call is plain C (handles, pointers, sizes), every asynchronous operation
 * returns an op id, and completions are drained with sw_poll()/sw_wait() — the
 * replacement for the UCX completion callbacks (main.cpp:172-232, 990-1061) that the
 * reference fires from its per-object progress thread.
 *
 * No torch / Python / CUDA types appear in any signature.  The library has no CPU
 * fallback: sw_ctx_create() fails when no CUDA device is visible.
 */
#ifndef STARWAY_B200_H
#define STARWAY_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SW_ABI_VERSION 1

typedef struct sw_ctx sw_ctx;
typedef uint64_t sw_worker_t; /* 0 is never a valid handle */
typedef uint64_t sw_ep_t;

/* worker kinds: reference classes Server (main.hpp:306) and Client (main.hpp:131) */
enum { SW_WORKER_SERVER = 1, SW_WORKER_CLIENT = 2 };

/* worker status, same numbering as the reference's status_ (main.hpp:173-174, 356-357):
 * 0 void, 1 initialized, 2 running, 3 closing, 4 closed */
enum { SW_ST_VOID = 0, SW_ST_INIT = 1, SW_ST_RUNNING = 2, SW_ST_CLOSING = 3, SW_ST_CLOSED = 4 };

/* where a buffer lives; AUTO asks the CUDA runtime (cudaPointerGetAttributes) */
enum { SW_MEM_AUTO = 0, SW_MEM_HOST = 1, SW_MEM_DEVICE = 2 };

/* completion kinds */
enum {
  SW_OP_SEND = 1,     /* reference ClientSendFuture / ServerSendFuture */
  SW_OP_RECV = 2,     /* reference ClientRecvFuture / ServerRecvFuture: (sender_tag, length) */
  SW_OP_FLUSH = 3,    /* reference ClientFlushFuture / ServerFlushFuture */
  SW_OP_FLUSH_EP = 4, /* reference ServerFlushEpFuture */
  SW_OP_CONNECT = 5,  /* reference Client connect_callback_(status string) */
  SW_OP_CLOSE = 6,    /* reference close_callback_() */
  SW_OP_ACCEPT = 7    /* reference Server accept_callback_(ServerEndpoint); op_id == 0 */
};

/* status codes: the UCX codes whose ucs_status_string() the reference forwards to
 * fail callbacks (main.cpp:94-98 etc.) */
enum {
  SW_STATUS_OK = 0,
  SW_STATUS_IO_ERROR = -3,
  SW_STATUS_NO_MEMORY = -4,
  SW_STATUS_INVALID_PARAM = -5,
  SW_STATUS_UNREACHABLE = -6,
  SW_STATUS_MESSAGE_TRUNCATED = -9,
  SW_STATUS_BUSY = -15,
  SW_STATUS_CANCELED = -16,
  SW_STATUS_TIMED_OUT = -20,
  SW_STATUS_NOT_CONNECTED = -24,
  SW_STATUS_CONNECTION_RESET = -25
};

typedef struct sw_completion {
  uint64_t op_id;      /* id returned by the posting call (0 for SW_OP_ACCEPT) */
  int32_t status;      /* SW_STATUS_* */
  uint32_t kind;       /* SW_OP_* */
  uint64_t sender_tag; /* SW_OP_RECV */
  uint64_t length;     /* SW_OP_RECV */
  uint64_t worker;     /* worker the completion belongs to */
  uint64_t ep;         /* SW_OP_ACCEPT: the new endpoint */
} sw_completion;

/* reference ServerEndpoint (main.hpp:292-304): name, local/remote sockaddr, transports */
typedef struct sw_ep_info {
  char name[64];
  char local_addr[48];
  char remote_addr[48];
  uint16_t local_port;
  uint16_t remote_port;
  uint32_t num_transports;
  char transport_device[4][32];
  char transport_name[4][32];
} sw_ep_info;

typedef struct sw_stats {
  uint64_t put_launches, put_msgs, put_bytes;
  uint64_t match_launches, deliver_launches;   /* always 0: receives are matched by the resident control kernels */
  uint64_t match_posts, match_arrivals;       /* receives handed to the device, ring slots consumed */
  uint64_t bulk_tma_launches, bulk_simt_launches, bulk_jobs, bulk_bytes;
  uint64_t h2d_bytes, d2h_bytes;
  uint64_t completions;
  double bulk_event_ms;       /* CUDA-event time of bulk launches (profiling on) */
  uint64_t bulk_event_launches;
  uint64_t bulk_event_bytes;
  double put_event_ms;
  uint64_t put_event_launches;
  double match_event_ms;      /* always 0, like match_launches */
  uint64_t match_event_launches;
  /* resident path: control-kernel / pull-kernel launches, and what the pull CTAs copied (bytes) in how much
   * time (union of the batches' active intervals, device timer) -- the roofline numerator / denominator */
  uint64_t prog_launches, pull_launches, pull_batches, pull_jobs, pull_bytes;
  double pull_busy_ms;
  uint64_t prog_exit_stop, prog_exit_idle, prog_exit_life; /* why control-kernel launches ended */
  double prog_life_ms;                                     /* total time control kernels were resident */
  uint64_t put_resident;                                   /* put batches executed by a resident control kernel (no launch) */
  double pull_pickup_ms, pull_copy_ms, pull_fin_ms;        /* pull batches, summed since context creation: published -> first
                                                              chunk claimed -> last chunk written -> records and FIN words out */
} sw_stats;

/* ---- library / context (reference Context, main.cpp:71-79) */
int sw_abi_version(void);
const char* sw_backend_name(void);
const char* sw_last_error(void);              /* thread-local message of the last failed call */
const char* sw_status_string(int32_t status); /* ucs_status_string() equivalents */
int sw_device_count(void);
/* CPUs on the NUMA node the GPU hangs off, as a Linux cpulist ("0-31,64-95"); returns its length, or
 * -1 when unknown.  The progress thread of a context binds itself to these CPUs (as UCX/NCCL helper
 * threads do); a launcher that wants host buffers NUMA-local binds the rank's process the same way. */
int sw_device_local_cpus(int device, char* out, size_t cap);
sw_ctx* sw_ctx_create(int device);            /* NULL on failure (no GPU => failure, no fallback) */
void sw_ctx_destroy(sw_ctx* ctx);
int sw_ctx_device(sw_ctx* ctx);
int sw_set_option(sw_ctx* ctx, const char* key, int64_t value);
int64_t sw_get_option(sw_ctx* ctx, const char* key);

/* ---- workers (reference Server::Server / Client::Client, main.cpp:811, 139) */
sw_worker_t sw_worker_create(sw_ctx* ctx, int kind);
int sw_worker_destroy(sw_ctx* ctx, sw_worker_t w); /* reference ~Client/~Server: implicit close + join */
int sw_worker_status(sw_ctx* ctx, sw_worker_t w);

/* reference Server::listen (main.cpp:815-832): blocks until running */
int sw_listen(sw_ctx* ctx, sw_worker_t w, const char* addr, uint16_t port);
/* reference Server::listen_address (main.cpp:834-851) */
int sw_listen_address(sw_ctx* ctx, sw_worker_t w);
/* reference get_worker_address (main.cpp:586-593, 853-860): returns length, <0 when not ready */
int64_t sw_get_address(sw_ctx* ctx, sw_worker_t w, void* out, size_t cap);
/* reference Client::connect / connect_address (main.cpp:552-585): completion kind SW_OP_CONNECT */
uint64_t sw_connect(sw_ctx* ctx, sw_worker_t w, const char* addr, uint16_t port);
uint64_t sw_connect_address(sw_ctx* ctx, sw_worker_t w, const void* blob, size_t len);
/* reference close (main.cpp:594-601, 1375-1382): completion kind SW_OP_CLOSE; 0 when not running */
uint64_t sw_close(sw_ctx* ctx, sw_worker_t w);

/* ---- the hot path.  All return an op id, or 0 with sw_last_error() set when the
 *      worker is not running (the reference throws std::runtime_error there). */
/* reference Client::send / Server::send (main.cpp:603-624, 1384-1407); ep ignored for clients */
uint64_t sw_post_send(sw_ctx* ctx, sw_worker_t w, sw_ep_t ep, const void* ptr, size_t len, uint64_t tag,
                      int mem_kind);
/* reference Client::recv / Server::recv (main.cpp:625-647, 1409-1431) */
uint64_t sw_post_recv(sw_ctx* ctx, sw_worker_t w, void* ptr, size_t cap, uint64_t tag, uint64_t tag_mask,
                      int mem_kind);
/* reference flush / flush_ep (main.cpp:649-665, 1433-1471) */
uint64_t sw_post_flush(sw_ctx* ctx, sw_worker_t w);
uint64_t sw_post_flush_ep(sw_ctx* ctx, sw_worker_t w, sw_ep_t ep);

/* ---- completions (replaces the UCX callbacks + GIL hand-off) */
int sw_poll(sw_ctx* ctx, sw_completion* out, int max);
int sw_wait(sw_ctx* ctx, sw_completion* out, int max, int timeout_ms);
int sw_event_fd(sw_ctx* ctx); /* readable while completions are pending */

/* ---- endpoints (reference list_clients / ServerEndpoint / evaluate_perf) */
int sw_list_eps(sw_ctx* ctx, sw_worker_t w, sw_ep_t* out, int max);
int sw_ep_info_get(sw_ctx* ctx, sw_worker_t w, sw_ep_t ep, sw_ep_info* out);
double sw_evaluate_perf(sw_ctx* ctx, sw_worker_t w, sw_ep_t ep, size_t msg_size);

/* ---- measurement hooks used by bench.py */
int sw_stats_get(sw_ctx* ctx, sw_stats* out);
int sw_stats_reset(sw_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* STARWAY_B200_H */
