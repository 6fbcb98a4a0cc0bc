"""ctypes shim + asyncio API over the starway_b200 C ABI (include/starway_b200.h).

Mirrors the reference's public surface — ``Server`` / ``Client`` /
``ServerEndpoint`` with ``asend / arecv / aflush / aflush_ep / aconnect /
aconnect_address / aclose / listen / listen_address`` (reference
``src/starway/__init__.py:71-345``) — over the drop-in replacement for its
``_bindings`` extension (reference ``src/starway/_bindings.pyi:7-88``).

Differences that are deliberate:
  * buffers may live on the GPU (torch CUDA tensors, ``__cuda_array_interface__``)
    as well as on the host (NumPy); the reference accepts CPU arrays only;
  * futures are resolved from ONE completion-poller thread per context, one
    ``call_soon_threadsafe`` per batch, instead of one UCX callback + GIL
    acquisition + ``call_soon_threadsafe`` per operation
    (reference ``src/bindings/main.cpp:172-232`` and ``__init__.py:124-128``);
  * the buffer object is kept alive until the operation completes (the
    reference keeps only the raw pointer, ``main.cpp:610-611``).

``bind(lib)`` builds the API classes on top of an already loaded ctypes
library.  The package binds it to ``libstarway_b200.so`` (CUDA, no fallback);
the CPU test-suite binds it to the host-logic simulator under ``tests/hostsim``.
"""
from __future__ import annotations

import asyncio
import atexit
import ctypes
import os
import threading
import time
import weakref
from collections.abc import Callable
from types import SimpleNamespace
from typing import Any

import numpy as np

try:  # C fast path of the binding layer (starway_b200/csrc/fastpath.c); the ctypes code below is the fallback
    from . import _fastpath
except ImportError:  # pragma: no cover
    _fastpath = None

# ----------------------------------------------------------------------------- C structs
SW_WORKER_SERVER = 1
SW_WORKER_CLIENT = 2
SW_MEM_HOST = 1
SW_MEM_DEVICE = 2
SW_OP_SEND, SW_OP_RECV, SW_OP_FLUSH, SW_OP_FLUSH_EP, SW_OP_CONNECT, SW_OP_CLOSE, SW_OP_ACCEPT = 1, 2, 3, 4, 5, 6, 7


class SwCompletion(ctypes.Structure):
    _fields_ = [
        ("op_id", ctypes.c_uint64),
        ("status", ctypes.c_int32),
        ("kind", ctypes.c_uint32),
        ("sender_tag", ctypes.c_uint64),
        ("length", ctypes.c_uint64),
        ("worker", ctypes.c_uint64),
        ("ep", ctypes.c_uint64),
    ]


class SwEpInfo(ctypes.Structure):
    _fields_ = [
        ("name", ctypes.c_char * 64),
        ("local_addr", ctypes.c_char * 48),
        ("remote_addr", ctypes.c_char * 48),
        ("local_port", ctypes.c_uint16),
        ("remote_port", ctypes.c_uint16),
        ("num_transports", ctypes.c_uint32),
        ("transport_device", (ctypes.c_char * 32) * 4),
        ("transport_name", (ctypes.c_char * 32) * 4),
    ]


class SwStats(ctypes.Structure):
    _fields_ = [
        ("put_launches", ctypes.c_uint64),
        ("put_msgs", ctypes.c_uint64),
        ("put_bytes", ctypes.c_uint64),
        ("match_launches", ctypes.c_uint64),
        ("deliver_launches", ctypes.c_uint64),
        ("match_posts", ctypes.c_uint64),
        ("match_arrivals", ctypes.c_uint64),
        ("bulk_tma_launches", ctypes.c_uint64),
        ("bulk_simt_launches", ctypes.c_uint64),
        ("bulk_jobs", ctypes.c_uint64),
        ("bulk_bytes", ctypes.c_uint64),
        ("h2d_bytes", ctypes.c_uint64),
        ("d2h_bytes", ctypes.c_uint64),
        ("completions", ctypes.c_uint64),
        ("bulk_event_ms", ctypes.c_double),
        ("bulk_event_launches", ctypes.c_uint64),
        ("bulk_event_bytes", ctypes.c_uint64),
        ("put_event_ms", ctypes.c_double),
        ("put_event_launches", ctypes.c_uint64),
        ("match_event_ms", ctypes.c_double),
        ("match_event_launches", ctypes.c_uint64),
        ("prog_launches", ctypes.c_uint64),
        ("pull_launches", ctypes.c_uint64),
        ("pull_batches", ctypes.c_uint64),
        ("pull_jobs", ctypes.c_uint64),
        ("pull_bytes", ctypes.c_uint64),
        ("pull_busy_ms", ctypes.c_double),
        ("prog_exit_stop", ctypes.c_uint64),
        ("prog_exit_idle", ctypes.c_uint64),
        ("prog_exit_life", ctypes.c_uint64),
        ("prog_life_ms", ctypes.c_double),
        ("put_resident", ctypes.c_uint64),
        ("pull_pickup_ms", ctypes.c_double),
        ("pull_copy_ms", ctypes.c_double),
        ("pull_fin_ms", ctypes.c_double),
    ]


# every symbol include/starway_b200.h declares: name -> (restype, argtypes)
_u64, _i64, _i32, _int, _vp, _cp, _sz = (
    ctypes.c_uint64,
    ctypes.c_int64,
    ctypes.c_int32,
    ctypes.c_int,
    ctypes.c_void_p,
    ctypes.c_char_p,
    ctypes.c_size_t,
)
C_ABI = {
    "sw_abi_version": (_int, []),
    "sw_backend_name": (_cp, []),
    "sw_last_error": (_cp, []),
    "sw_status_string": (_cp, [_i32]),
    "sw_device_count": (_int, []),
    "sw_ctx_create": (_vp, [_int]),
    "sw_ctx_destroy": (None, [_vp]),
    "sw_ctx_device": (_int, [_vp]),
    "sw_device_local_cpus": (_int, [_int, ctypes.c_char_p, _sz]),
    "sw_set_option": (_int, [_vp, _cp, _i64]),
    "sw_get_option": (_i64, [_vp, _cp]),
    "sw_worker_create": (_u64, [_vp, _int]),
    "sw_worker_destroy": (_int, [_vp, _u64]),
    "sw_worker_status": (_int, [_vp, _u64]),
    "sw_listen": (_int, [_vp, _u64, _cp, ctypes.c_uint16]),
    "sw_listen_address": (_int, [_vp, _u64]),
    "sw_get_address": (_i64, [_vp, _u64, _vp, _sz]),
    "sw_connect": (_u64, [_vp, _u64, _cp, ctypes.c_uint16]),
    "sw_connect_address": (_u64, [_vp, _u64, _vp, _sz]),
    "sw_close": (_u64, [_vp, _u64]),
    "sw_post_send": (_u64, [_vp, _u64, _u64, _vp, _sz, _u64, _int]),
    "sw_post_recv": (_u64, [_vp, _u64, _vp, _sz, _u64, _u64, _int]),
    "sw_post_recv_reduce": (_u64, [_vp, _u64, _vp, _sz, _u64, _u64, _int]),
    "sw_post_flush": (_u64, [_vp, _u64]),
    "sw_post_flush_ep": (_u64, [_vp, _u64, _u64]),
    "sw_poll": (_int, [_vp, ctypes.POINTER(SwCompletion), _int]),
    "sw_wait": (_int, [_vp, ctypes.POINTER(SwCompletion), _int, _int]),
    "sw_event_fd": (_int, [_vp]),
    "sw_list_eps": (_int, [_vp, _u64, ctypes.POINTER(_u64), _int]),
    "sw_ep_info_get": (_int, [_vp, _u64, _u64, ctypes.POINTER(SwEpInfo)]),
    "sw_evaluate_perf": (ctypes.c_double, [_vp, _u64, _u64, _sz]),
    "sw_stats_get": (_int, [_vp, ctypes.POINTER(SwStats)]),
    "sw_stats_reset": (_int, [_vp]),
}


def declare(lib: ctypes.CDLL) -> ctypes.CDLL:
    """Attach restype/argtypes for every C-ABI entry point; raises if one is missing."""
    for name, (res, args) in C_ABI.items():
        fn = getattr(lib, name)  # AttributeError => the library does not export the ABI
        fn.restype = res
        fn.argtypes = args
    return lib


# ----------------------------------------------------------------------------- buffers
def _is_torch_tensor(obj: Any) -> bool:
    mod = type(obj).__module__
    return mod == "torch" or mod.startswith("torch.")


_U8 = np.dtype(np.uint8)
_np_cache: dict[int, tuple] = {}  # id(array) -> (weakref, ptr, nbytes, writeable): preallocated buffers are reused


def _np_fast(arr: np.ndarray):
    import weakref

    key = id(arr)
    hit = _np_cache.get(key)
    if hit is not None and hit[0]() is arr:
        return hit
    if len(_np_cache) > 8192:
        _np_cache.clear()
    hit = (weakref.ref(arr), arr.__array_interface__["data"][0], arr.nbytes, arr.flags.writeable)
    _np_cache[key] = hit
    return hit


def as_buffer(obj: Any, writable: bool):
    """-> (ptr, nbytes, mem_kind, keepalive).  1-D contiguous uint8, host or device."""
    tp = type(obj)
    if tp is np.ndarray:
        arr = obj
        if arr.dtype is _U8 and arr.strides == (1,):
            _, ptr, nbytes, wr = _np_fast(arr)
            if writable and not wr:
                raise TypeError("recv buffer must be a writable, contiguous 1-D uint8 array")
            return ptr, nbytes, SW_MEM_HOST, arr
        if arr.dtype != np.uint8 or arr.ndim != 1 or not arr.flags.c_contiguous:
            if writable:
                raise TypeError("recv buffer must be a writable, contiguous 1-D uint8 array")
            if arr.ndim != 1:
                raise TypeError("send buffer must be 1-D")
            if arr.dtype != np.uint8:
                # nanobind's ndarray caster converts implicitly (reference tests pass int64 arrays,
                # tests/test_basic.py:562); the temporary is kept alive until completion
                arr = arr.astype(np.uint8)
            arr = np.ascontiguousarray(arr)
        elif writable and not arr.flags.writeable:
            raise TypeError("recv buffer must be a writable, contiguous 1-D uint8 array")
        return arr.__array_interface__["data"][0], arr.nbytes, SW_MEM_HOST, arr
    if _is_torch_tensor(obj):
        t = obj
        if t.dim() != 1 or not t.is_contiguous():
            raise TypeError("tensor buffers must be 1-D and contiguous")
        if t.element_size() != 1:
            if writable:
                raise TypeError("recv buffer must be a uint8 tensor")
            t = t.view(-1).contiguous().view(dtype=__import__("torch").uint8)
        return t.data_ptr(), t.numel(), (SW_MEM_DEVICE if t.is_cuda else SW_MEM_HOST), t
    if isinstance(obj, np.ndarray):
        return as_buffer(np.asarray(obj), writable)
    cai = getattr(obj, "__cuda_array_interface__", None)
    if cai is not None:
        shape = cai["shape"]
        if len(shape) != 1 or cai.get("strides") not in (None, (np.dtype(cai["typestr"]).itemsize,)):
            raise TypeError("device buffers must be 1-D and contiguous")
        ptr, readonly = cai["data"]
        if writable and readonly:
            raise TypeError("recv buffer is read-only")
        return int(ptr), int(shape[0]) * np.dtype(cai["typestr"]).itemsize, SW_MEM_DEVICE, obj
    raise TypeError(f"unsupported buffer type {type(obj)!r}: expected numpy.ndarray, torch.Tensor or a CUDA array")


# element types of arecv_reduce (SW_DTYPE_* in include/starway_b200.h)
SW_DTYPE_F32, SW_DTYPE_F16, SW_DTYPE_BF16, SW_DTYPE_F64, SW_DTYPE_I32, SW_DTYPE_I64 = 1, 2, 3, 4, 5, 6
_REDUCE_TORCH = {"torch.float32": 1, "torch.float16": 2, "torch.bfloat16": 3, "torch.float64": 4, "torch.int32": 5,
                 "torch.int64": 6}
_REDUCE_TYPESTR = {"<f4": 1, "<f2": 2, "<f8": 4, "<i4": 5, "<i8": 6}  # bfloat16 has no typestr: torch only


def as_reduce_buffer(obj: Any, device: int):
    """-> (ptr, nbytes, dtype, keepalive) for arecv_reduce: a contiguous CUDA tensor on `device` (any shape) or a
    contiguous ``__cuda_array_interface__`` object of a supported element type.  Anything else: TypeError."""
    if _is_torch_tensor(obj):
        dt = _REDUCE_TORCH.get(str(obj.dtype))
        if dt is None:
            raise TypeError(f"arecv_reduce: unsupported dtype {obj.dtype}")
        if not obj.is_cuda or obj.device.index != device:
            raise TypeError(f"arecv_reduce: the buffer must be a CUDA tensor on cuda:{device}")
        if not obj.is_contiguous():
            raise TypeError("arecv_reduce: the buffer must be contiguous")
        return obj.data_ptr(), obj.numel() * obj.element_size(), dt, obj
    cai = None if isinstance(obj, np.ndarray) else getattr(obj, "__cuda_array_interface__", None)
    if cai is None:
        raise TypeError(f"arecv_reduce: expected a CUDA tensor or a CUDA array, got {type(obj)!r}")
    dt = _REDUCE_TYPESTR.get(cai["typestr"])
    if dt is None:
        raise TypeError(f"arecv_reduce: unsupported typestr {cai['typestr']!r}")
    shape = tuple(int(x) for x in cai["shape"])
    itemsize = np.dtype(cai["typestr"]).itemsize
    strides = cai.get("strides")
    if strides is not None:
        want, acc = [], itemsize
        for dim in reversed(shape):
            want.append(acc)
            acc *= dim
        if tuple(strides) != tuple(reversed(want)) and int(np.prod(shape)) > 1:
            raise TypeError("arecv_reduce: the buffer must be contiguous")
    ptr, readonly = cai["data"]
    if readonly:
        raise TypeError("arecv_reduce: the buffer is read-only")
    return int(ptr), int(np.prod(shape)) * itemsize, dt, obj


# ----------------------------------------------------------------------------- API factory
def _banner(msg: str) -> None:
    """The reference prints "Connected!" / "Client closed!" / "Server closed!" (__init__.py:91,224,256).
    Kept for drop-in behaviour; STARWAY_QUIET=1 silences them (benchmarks print one JSON line)."""
    import os

    if os.environ.get("STARWAY_QUIET") != "1":
        print(msg)


def _weak_method(obj, func):
    """`func` bound to `obj` through a weak reference (the C callable stored on the object must not keep it alive)."""
    ref = weakref.ref(obj)

    def call(*args, **kwargs):
        o = ref()
        if o is None:
            raise ReferenceError("starway_b200 object is gone")
        return func(o, *args, **kwargs)

    return call


def bind(lib: ctypes.CDLL, default_device: Callable[[], int] | None = None, use_fastpath: bool = True) -> SimpleNamespace:
    """Build Context/Server/Client/ServerEndpoint classes on top of a loaded C-ABI library."""
    declare(lib)
    _post_send, _post_recv = lib.sw_post_send, lib.sw_post_recv
    _get_running_loop = asyncio.get_running_loop
    _monotonic_ns = time.monotonic_ns
    _U64MASK = 0xFFFFFFFFFFFFFFFF

    def _err() -> str:
        s = lib.sw_last_error()
        return s.decode() if s else "unknown error"

    def status_string(code: int) -> str:
        return lib.sw_status_string(code).decode()

    class Context:
        """One per (process, device): owns the native context and completion delivery.

        Replaces the reference's global ``Context()`` (``__init__.py:68``) plus the per-object UCX
        progress threads.  Completions are drained by the asyncio loop itself: the native
        completion queue signals an eventfd that is registered with ``loop.add_reader``, so futures
        are resolved on the loop thread in batches with no thread hand-off ("asyncio futures resolve
        from CUDA-event polling").  A fallback poller thread serves raw-callback users and loops the
        context was not registered with."""

        def __init__(self, device: int | None = None):
            if device is None:
                device = default_device() if default_device else 0
            self.device = device
            self._h = lib.sw_ctx_create(device)
            if not self._h:
                raise RuntimeError(_err())
            self._lock = threading.Lock()
            self._ops: dict[int, tuple] = {}
            # weak: a Server the caller dropped must be collectable (its __del__ closes the native worker)
            self._servers: weakref.WeakValueDictionary = weakref.WeakValueDictionary()
            self._efd = lib.sw_event_fd(self._h)
            self._readers: dict[Any, bool] = {}
            self._bufs: dict[Any, Any] = {}  # loop -> completion batch buffer (ctypes drain path)
            self._stop = False
            self._wake = threading.Event()
            self._fp = None
            self._spin_ns = int(float(os.environ.get("STARWAY_SPIN_US", "200")) * 1000)
            self._spin_loop = None
            self._spin_seen = -1
            self._spin_deadline = 0
            if _fastpath is not None and use_fastpath:
                addr = lambda f: ctypes.cast(f, ctypes.c_void_p).value  # noqa: E731
                self._fp = _fastpath.Binding(addr(lib.sw_post_send), addr(lib.sw_post_recv), addr(lib.sw_poll), self._h,
                                             self._ops, as_buffer, self.ensure_reader, self._slow, _err, status_string)
                self._fp.kick = self._kick
            self._thread = threading.Thread(target=self._poll_loop, name="starway-b200-poller", daemon=True)
            self._thread.start()

        # -- submission helpers ------------------------------------------------
        def submit(self, post: Callable[[], int], entry: tuple) -> int:
            if not self._h:
                raise RuntimeError("starway_b200 context is closed")
            with self._lock:
                op = post()
                if not op:
                    raise RuntimeError(_err())
                self._ops[op] = entry
            if self._spin_loop is None:
                self._kick()
            return op

        def ensure_reader(self, loop) -> None:
            """Register the completion eventfd with `loop` (must be called on the loop's thread)."""
            if loop in self._readers or self._efd < 0:
                return
            try:
                if asyncio.get_running_loop() is not loop:
                    return
                loop.add_reader(self._efd, self._drain, loop)
                self._readers[loop] = True
                sl = self._spin_loop
                if sl is not None and sl is not loop and not sl.is_running():
                    self._stop_spin(None)
                loop.call_soon(self._drain, loop)  # anything published before the reader existed
            except (RuntimeError, NotImplementedError, OSError):
                pass

        # -- completion side ---------------------------------------------------
        def _dispatch(self, n: int, buf, here) -> None:
            """Deliver n polled completions.  `here` is the loop whose thread we are on (or None)."""
            with self._lock:
                pop = self._ops.pop
                entries = [pop(buf[i].op_id, None) for i in range(n)]
            fp = self._fp
            if fp is not None and None in entries:
                # operations posted through the C fast path live in its own table
                entries = [e if e is not None else fp.take(buf[i].op_id) for i, e in enumerate(entries)]
            batches: dict[Any, list] | None = None
            for i in range(n):
                entry = entries[i]
                c = buf[i]
                kind = c.kind
                if entry is None:
                    if kind == SW_OP_ACCEPT:
                        srv = self._servers.get(c.worker)
                        if srv is not None:
                            srv._on_accept(c.ep)
                    continue
                status = c.status
                if entry[0] == "fut":
                    _, loop, fut, _keep, post_ok = entry
                    if status == 0:
                        if post_ok is not None:
                            post_ok()
                        val = (c.sender_tag, c.length) if kind == SW_OP_RECV else None
                        if loop is here:
                            if not fut.done():
                                fut.set_result(val)
                            continue
                        item = (fut, True, val)
                    else:
                        if loop is here:
                            if not fut.done():
                                fut.set_exception(Exception(status_string(status)))
                            continue
                        item = (fut, False, status_string(status))
                    if batches is None:
                        batches = {}
                    batches.setdefault(loop, []).append(item)
                else:  # raw callbacks (reference: invoked on the native worker thread)
                    _, done, fail, _keep = entry
                    try:
                        if status == 0:
                            if kind == SW_OP_RECV:
                                done(c.sender_tag, c.length)
                            elif kind == SW_OP_CONNECT:
                                done("")
                            else:
                                done()
                        else:
                            if kind == SW_OP_CONNECT:
                                done(status_string(status))
                            elif fail is not None:
                                fail(status_string(status))
                    except Exception as exc:  # never kill the dispatcher
                        print(f"starway_b200: exception in user callback: {exc!r}")
            if batches:
                for loop, lst in batches.items():
                    try:
                        loop.call_soon_threadsafe(_resolve_batch, lst)
                    except RuntimeError:
                        pass  # loop already closed

        def _slow(self, entry, kind, status, sender_tag, length, worker, ep, here, op_id=0) -> None:
            """One completion the C fast path does not handle itself (accept, raw callbacks, other loops)."""
            if entry is None and op_id:
                # An operation posted through submit() from another thread: sw_post_* runs with the GIL
                # released and the entry is registered right after it, both under self._lock.  Taking
                # the lock here therefore waits for the registration (completions must never be dropped).
                with self._lock:
                    entry = self._ops.pop(op_id, None)
            if entry is None:
                if kind == SW_OP_ACCEPT:
                    srv = self._servers.get(worker)
                    if srv is not None:
                        srv._on_accept(ep)
                return
            c = SwCompletion(0, status, kind, sender_tag, length, worker, ep)
            buf = (SwCompletion * 1)(c)
            op = -1 - id(entry)  # re-insert under a private key so that _dispatch finds it
            with self._lock:
                self._ops[op & 0xFFFFFFFFFFFFFFFF] = entry
            buf[0].op_id = op & 0xFFFFFFFFFFFFFFFF
            self._dispatch(1, buf, here)

        def _drain(self, loop) -> int:
            """eventfd reader callback: runs on `loop`'s thread.  Returns the number of completions."""
            h = self._h
            if not h:
                return 0
            if self._fp is not None:
                return self._fp.drain(loop)
            buf = self._bufs.get(loop)  # one batch buffer per loop (= per draining thread)
            if buf is None:
                buf = self._bufs[loop] = (SwCompletion * 512)()
            total = 0
            while True:
                n = lib.sw_poll(h, buf, 512)
                if n <= 0:
                    return total
                total += n
                self._dispatch(n, buf, loop)
                if n < 512:
                    return total

        # -- adaptive busy-polling of the completion queue ---------------------------------------
        # Waking a thread that sleeps in epoll on the eventfd costs 10-40 us, several times the device
        # pipeline of a small message.  After a submission the loop therefore polls the completion
        # queue from a self-re-arming call_soon callback (other callbacks and I/O keep running between
        # polls) until nothing has happened for `spin_us`; then it returns to the eventfd.  While it
        # polls, the engine skips the eventfd write (option "consumer_polling").
        def _kick(self) -> None:
            if self._spin_loop is not None or self._spin_ns <= 0:
                return
            try:
                loop = _get_running_loop()
            except RuntimeError:
                return
            if loop not in self._readers or not self._h:
                return
            self._spin_loop = loop
            if self._fp is not None:
                self._fp.spinning = 1
            self._spin_seen = -1
            self._spin_deadline = _monotonic_ns() + self._spin_ns
            lib.sw_set_option(self._h, b"consumer_polling", 1)
            try:
                loop.call_soon(self._spin, loop)
            except RuntimeError:
                self._stop_spin(None)

        def _spin(self, loop) -> None:
            if self._spin_loop is not loop:
                return
            again = False
            try:
                n = self._drain(loop)
                pending = len(self._ops) + (self._fp.pending() if self._fp is not None else 0)
                if pending and self._h:
                    now = _monotonic_ns()
                    if n or pending != self._spin_seen:
                        self._spin_seen = pending
                        self._spin_deadline = now + self._spin_ns
                    if now < self._spin_deadline:
                        loop.call_soon(self._spin, loop)
                        again = True
            finally:
                if not again:
                    self._stop_spin(loop)

        def _stop_spin(self, loop) -> None:
            self._spin_loop = None
            if self._fp is not None:
                self._fp.spinning = 0
            if self._h:
                lib.sw_set_option(self._h, b"consumer_polling", 0)
                if loop is not None:
                    self._drain(loop)  # completions published while the wake-up was suppressed

        def _poll_loop(self):
            buf = (SwCompletion * 512)()
            while not self._stop:
                sl = self._spin_loop
                if sl is not None and not sl.is_running():
                    # the polling loop stopped with its callback still queued: hand delivery back
                    self._stop_spin(None)
                    for lp in list(self._readers):
                        if not lp.is_closed():
                            try:
                                lp.call_soon_threadsafe(self._drain, lp)
                            except RuntimeError:
                                pass
                if self._readers:
                    # an asyncio loop drains the queue itself; only watch for loops that went away
                    for lp in list(self._readers):
                        if lp.is_closed():
                            self._readers.pop(lp, None)
                            self._bufs.pop(lp, None)
                    if self._readers:
                        self._wake.wait(0.05)
                        continue
                n = lib.sw_wait(self._h, buf, 512, 50)
                if n > 0:
                    self._dispatch(n, buf, None)

        def stats(self) -> dict:
            s = SwStats()
            lib.sw_stats_get(self._h, ctypes.byref(s))
            return {name: getattr(s, name) for name, _ in SwStats._fields_}

        def reset_stats(self) -> None:
            lib.sw_stats_reset(self._h)

        def set_option(self, key: str, value: int) -> None:
            if lib.sw_set_option(self._h, key.encode(), int(value)) != 0:
                raise ValueError(_err())

        def get_option(self, key: str) -> int:
            return int(lib.sw_get_option(self._h, key.encode()))

        def close(self):
            if self._h:
                if self._fp is not None:
                    self._fp.closed = 1  # objects bound to the fast path (Client.asend ...) fall back to the Python methods
                self._fp = None  # the C fast path holds the raw context pointer
                self._stop = True
                self._wake.set()
                self._thread.join(timeout=2.0)
                for lp in list(self._readers):
                    try:
                        if not lp.is_closed():
                            lp.remove_reader(self._efd)
                    except Exception:
                        pass
                self._readers.clear()
                h, self._h = self._h, None
                lib.sw_ctx_destroy(h)

    def _resolve_batch(lst):
        for fut, ok, val in lst:
            if fut.done():
                continue
            if ok:
                fut.set_result(val)
            else:
                fut.set_exception(Exception(val))

    def local_cpus(device: int | None = None) -> set[int]:
        """CPUs on the NUMA node of `device` (empty when unknown)."""
        if device is None:
            device = default_device() if default_device else 0
        buf = ctypes.create_string_buffer(1024)
        if lib.sw_device_local_cpus(int(device), buf, 1024) <= 0:
            return set()
        cpus: set[int] = set()
        for part in buf.value.decode().split(","):
            lo, _, hi = part.partition("-")
            cpus.update(range(int(lo), int(hi or lo) + 1))
        return cpus

    def bind_to_device_numa(device: int | None = None) -> bool:
        """Restrict the calling thread (and the threads it starts later) to the CPUs next to `device`,
        so that host buffers it allocates are NUMA-local to the GPU's PCIe root — what a launcher
        does with `numactl --cpunodebind`.  Returns False when nothing was changed."""
        try:
            want = local_cpus(device) & os.sched_getaffinity(0)
            if not want or want == os.sched_getaffinity(0):
                return False
            os.sched_setaffinity(0, want)
            return True
        except (OSError, AttributeError, ValueError):
            return False

    _state = SimpleNamespace(ctx=None)
    _state_lock = threading.Lock()

    def get_context() -> Context:
        with _state_lock:
            if _state.ctx is None:
                _state.ctx = Context()
                atexit.register(shutdown)
            return _state.ctx

    def shutdown():
        with _state_lock:
            ctx, _state.ctx = _state.ctx, None
        if ctx is not None:
            ctx.close()

    class ServerEndpoint:
        """Reference ``ServerEndpoint`` (``main.hpp:292-304``, ``_bindings.pyi:10-21``)."""

        __slots__ = ("_ctx", "_worker", "_id", "_info")

        def __init__(self, ctx: Context, worker: int, ep_id: int):
            self._ctx = ctx
            self._worker = worker
            self._id = ep_id
            info = SwEpInfo()
            lib.sw_ep_info_get(ctx._h, worker, ep_id, ctypes.byref(info))
            self._info = info

        name = property(lambda self: self._info.name.decode())
        local_addr = property(lambda self: self._info.local_addr.decode())
        local_port = property(lambda self: int(self._info.local_port))
        remote_addr = property(lambda self: self._info.remote_addr.decode())
        remote_port = property(lambda self: int(self._info.remote_port))

        def view_transports(self) -> list[tuple[str, str]]:
            n = self._info.num_transports
            return [
                (self._info.transport_device[i].value.decode(), self._info.transport_name[i].value.decode())
                for i in range(n)
            ]

        def __hash__(self):
            return hash(self._id)

        def __eq__(self, other):
            return isinstance(other, ServerEndpoint) and other._id == self._id

        def __repr__(self):
            return f"<ServerEndpoint {self.name!r}>"

    class _Base:
        _kind = 0

        def __init__(self, ctx: Context | None = None):
            self._ctx = ctx if ctx is not None else get_context()
            self._w = lib.sw_worker_create(self._ctx._h, self._kind)
            if not self._w:
                raise RuntimeError(_err())
            fp = self._ctx._fp
            if fp is not None:
                # the hot calls as C callables bound to this worker (no Python frame per message); anything but the
                # plain call shape goes to the Python method of the same name
                cls = type(self)
                self.arecv = fp.bound(self._w, 0, True, _weak_method(self, cls.arecv))
                if self._kind == SW_WORKER_CLIENT:
                    self.asend = fp.bound(self._w, 0, False, _weak_method(self, cls.asend))

        def __del__(self):
            # reference ~Client/~Server: implicit close + join (main.cpp:703-719, 1519-1536)
            try:
                ctx = self._ctx
                if ctx._h:
                    lib.sw_worker_destroy(ctx._h, self._w)
                    ctx._servers.pop(self._w, None)
            except Exception:
                pass

        # -- helpers -------------------------------------------------------------
        def _future(self, loop):
            if loop is None:
                loop = asyncio.get_running_loop()
            ctx = self._ctx
            if loop not in ctx._readers:
                ctx.ensure_reader(loop)
            return loop, loop.create_future()

        def _post_recv(self, buffer, tag, tag_mask, entry_of):
            ptr, n, mem, keep = as_buffer(buffer, writable=True)
            h, w = self._ctx._h, self._w
            return self._ctx.submit(
                lambda: lib.sw_post_recv(h, w, ptr, n, tag & 0xFFFFFFFFFFFFFFFF, tag_mask & 0xFFFFFFFFFFFFFFFF, mem),
                entry_of(keep),
            )

        def recv(self, buffer, tag: int, tag_mask: int, done_callback, fail_callback):
            self._post_recv(buffer, tag, tag_mask, lambda keep: ("cb", done_callback, fail_callback, keep))

        def arecv(self, buffer, tag: int, tag_mask: int, loop: asyncio.AbstractEventLoop | None = None):
            # hot path: no helper calls / closures
            ctx = self._ctx
            if loop is None and ctx._fp is not None:
                fut = ctx._fp.arecv(self._w, buffer, tag, tag_mask)
                if ctx._spin_loop is None:
                    ctx._kick()
                return fut
            if loop is None:
                loop = _get_running_loop()
            if loop not in ctx._readers:
                ctx.ensure_reader(loop)
            fut = loop.create_future()
            ptr, n, mem, keep = as_buffer(buffer, True)
            if not ctx._h:
                raise RuntimeError("starway_b200 context is closed")
            with ctx._lock:
                op = _post_recv(ctx._h, self._w, ptr, n, tag & _U64MASK, tag_mask & _U64MASK, mem)
                if not op:
                    raise RuntimeError(_err())
                ctx._ops[op] = ("fut", loop, fut, keep, None)
            if ctx._spin_loop is None:
                ctx._kick()
            return fut

        def arecv_reduce(self, buffer, tag: int, tag_mask: int, loop: asyncio.AbstractEventLoop | None = None):
            """Receive a message and ADD it into `buffer` instead of overwriting it (an extension beyond the
            reference's API).  Matches exactly like `arecv`.  The message's bytes, read as elements of the buffer's
            dtype, are added into the first ``length // itemsize`` elements; the future resolves to
            ``(sender_tag, length)`` once the sum is visible on every stream.  `buffer`: a contiguous CUDA tensor on
            the context's device (float32, float16, bfloat16, float64, int32, int64) or a contiguous
            ``__cuda_array_interface__`` object; anything else raises TypeError.  Work queued on `buffer` must be
            finished before the call."""
            ctx = self._ctx
            ptr, n, dtype, keep = as_reduce_buffer(buffer, ctx.device)
            loop, fut = self._future(loop)
            if not ctx._h:
                raise RuntimeError("starway_b200 context is closed")
            with ctx._lock:
                op = lib.sw_post_recv_reduce(ctx._h, self._w, ptr, n, tag & _U64MASK, tag_mask & _U64MASK, dtype)
                if not op:
                    msg = _err()
                    raise (TypeError if msg.startswith("recv_reduce:") else RuntimeError)(msg)
                ctx._ops[op] = ("fut", loop, fut, keep, None)
            if ctx._spin_loop is None:
                ctx._kick()
            return fut

        def flush(self, done_callback, fail_callback):
            h, w = self._ctx._h, self._w
            self._ctx.submit(lambda: lib.sw_post_flush(h, w), ("cb", done_callback, fail_callback, None))

        def aflush(self, loop: asyncio.AbstractEventLoop | None = None):
            loop, fut = self._future(loop)
            h, w = self._ctx._h, self._w
            self._ctx.submit(lambda: lib.sw_post_flush(h, w), ("fut", loop, fut, None, None))
            return fut

        def get_worker_address(self) -> bytes:
            buf = ctypes.create_string_buffer(512)
            n = lib.sw_get_address(self._ctx._h, self._w, buf, 512)
            if n < 0:
                raise RuntimeError(_err())
            return buf.raw[:n]

        def close(self, callback: Callable[[], None]):
            """Binding-level close (reference ``_bindings.pyi:31,69``, bound at ``main.cpp:1538-1581``): returns at
            once, ``callback()`` fires when the worker has shut down.  Raises RuntimeError when not running."""
            h, w = self._ctx._h, self._w
            self._ctx.submit(lambda: lib.sw_close(h, w), ("cb", callback, None, None))

        def _aclose(self, loop, banner):
            loop, fut = self._future(loop)
            h, w = self._ctx._h, self._w
            self._ctx.submit(lambda: lib.sw_close(h, w), ("fut", loop, fut, None, lambda: _banner(banner)))
            return fut

    class Server(_Base):
        """Reference ``Server`` (``src/starway/__init__.py:71-209``)."""

        _kind = SW_WORKER_SERVER

        def __init__(self, ctx: Context | None = None):
            super().__init__(ctx)
            self._accept_cb = None
            self._eps: dict[int, ServerEndpoint] = {}
            self._ctx._servers[self._w] = self

        def _ep(self, ep_id: int) -> ServerEndpoint:
            ep = self._eps.get(ep_id)
            if ep is None:
                ep = self._eps[ep_id] = ServerEndpoint(self._ctx, self._w, ep_id)
            return ep

        def _on_accept(self, ep_id: int):
            ep = self._ep(ep_id)
            cb = self._accept_cb
            if cb is not None:
                try:
                    cb(ep)
                except Exception as exc:
                    print(f"starway_b200: exception in accept callback: {exc!r}")

        def listen(self, addr: str, port: int):
            if lib.sw_listen(self._ctx._h, self._w, addr.encode(), port) != 0:
                raise RuntimeError(_err())

        def listen_address(self) -> bytes:
            if lib.sw_listen_address(self._ctx._h, self._w) != 0:
                raise RuntimeError(_err())
            return self.get_worker_address()

        def set_accept_cb(self, on_accept: Callable[[ServerEndpoint], None]):
            self._accept_cb = on_accept

        set_accept_callback = set_accept_cb

        def aclose(self, loop: asyncio.AbstractEventLoop | None = None):
            return self._aclose(loop, "Server closed!")

        def list_clients(self) -> set[ServerEndpoint]:
            arr = (ctypes.c_uint64 * 256)()
            n = lib.sw_list_eps(self._ctx._h, self._w, arr, 256)
            return {self._ep(arr[i]) for i in range(max(0, min(n, 256)))}

        def _post_send(self, client_ep, buffer, tag, entry_of):
            if not isinstance(client_ep, ServerEndpoint):
                raise TypeError("client_ep must be a ServerEndpoint")
            ptr, n, mem, keep = as_buffer(buffer, writable=False)
            h, w, e = self._ctx._h, self._w, client_ep._id
            return self._ctx.submit(
                lambda: lib.sw_post_send(h, w, e, ptr, n, tag & 0xFFFFFFFFFFFFFFFF, mem), entry_of(keep)
            )

        def send(self, client_ep, buffer, tag: int, done_callback, fail_callback):
            self._post_send(client_ep, buffer, tag, lambda keep: ("cb", done_callback, fail_callback, keep))

        def asend(self, client_ep, buffer, tag: int, loop: asyncio.AbstractEventLoop | None = None):
            ctx = self._ctx
            if loop is None and ctx._fp is not None:
                fut = ctx._fp.asend(self._w, client_ep._id, buffer, tag)
                if ctx._spin_loop is None:
                    ctx._kick()
                return fut
            if loop is None:
                loop = _get_running_loop()
            if loop not in ctx._readers:
                ctx.ensure_reader(loop)
            fut = loop.create_future()
            ptr, n, mem, keep = as_buffer(buffer, False)
            if not ctx._h:
                raise RuntimeError("starway_b200 context is closed")
            with ctx._lock:
                op = _post_send(ctx._h, self._w, client_ep._id, ptr, n, tag & _U64MASK, mem)
                if not op:
                    raise RuntimeError(_err())
                ctx._ops[op] = ("fut", loop, fut, keep, None)
            if ctx._spin_loop is None:
                ctx._kick()
            return fut

        def flush_ep(self, client_ep, done_callback, fail_callback):
            h, w, e = self._ctx._h, self._w, client_ep._id
            self._ctx.submit(lambda: lib.sw_post_flush_ep(h, w, e), ("cb", done_callback, fail_callback, None))

        def aflush_ep(self, client_ep, loop: asyncio.AbstractEventLoop | None = None):
            loop, fut = self._future(loop)
            h, w, e = self._ctx._h, self._w, client_ep._id
            self._ctx.submit(lambda: lib.sw_post_flush_ep(h, w, e), ("fut", loop, fut, None, None))
            return fut

        def evaluate_perf(self, client_ep, msg_size: int) -> float:
            t = lib.sw_evaluate_perf(self._ctx._h, self._w, client_ep._id, msg_size)
            if t < 0:
                raise RuntimeError(_err())
            return t

    class Client(_Base):
        """Reference ``Client`` (``src/starway/__init__.py:212-345``)."""

        _kind = SW_WORKER_CLIENT

        def connect(self, addr: str, port: int, callback: Callable[[str], None]):
            h, w = self._ctx._h, self._w
            self._ctx.submit(lambda: lib.sw_connect(h, w, addr.encode(), port), ("cb", callback, None, None))

        def connect_address(self, remote_address: bytes, callback: Callable[[str], None]):
            h, w = self._ctx._h, self._w
            blob = bytes(remote_address)
            self._ctx.submit(lambda: lib.sw_connect_address(h, w, blob, len(blob)), ("cb", callback, None, blob))

        def aconnect(self, addr: str, port: int, loop: asyncio.AbstractEventLoop | None = None):
            loop, fut = self._future(loop)
            h, w = self._ctx._h, self._w
            self._ctx.submit(
                lambda: lib.sw_connect(h, w, addr.encode(), port), ("fut", loop, fut, None, lambda: _banner("Connected!"))
            )
            return fut

        def aconnect_address(self, remote_address: bytes, loop: asyncio.AbstractEventLoop | None = None):
            loop, fut = self._future(loop)
            h, w = self._ctx._h, self._w
            blob = bytes(remote_address)
            self._ctx.submit(
                lambda: lib.sw_connect_address(h, w, blob, len(blob)),
                ("fut", loop, fut, blob, lambda: _banner("Connected!")),
            )
            return fut

        def aclose(self, loop: asyncio.AbstractEventLoop | None = None):
            return self._aclose(loop, "Client closed!")

        def _post_send(self, buffer, tag, entry_of):
            ptr, n, mem, keep = as_buffer(buffer, writable=False)
            h, w = self._ctx._h, self._w
            return self._ctx.submit(
                lambda: lib.sw_post_send(h, w, 0, ptr, n, tag & 0xFFFFFFFFFFFFFFFF, mem), entry_of(keep)
            )

        def send(self, buffer, tag: int, done_callback, fail_callback):
            self._post_send(buffer, tag, lambda keep: ("cb", done_callback, fail_callback, keep))

        def asend(self, buffer, tag: int, loop: asyncio.AbstractEventLoop | None = None):
            ctx = self._ctx
            if loop is None and ctx._fp is not None:
                fut = ctx._fp.asend(self._w, 0, buffer, tag)
                if ctx._spin_loop is None:
                    ctx._kick()
                return fut
            if loop is None:
                loop = _get_running_loop()
            if loop not in ctx._readers:
                ctx.ensure_reader(loop)
            fut = loop.create_future()
            ptr, n, mem, keep = as_buffer(buffer, False)
            if not ctx._h:
                raise RuntimeError("starway_b200 context is closed")
            with ctx._lock:
                op = _post_send(ctx._h, self._w, 0, ptr, n, tag & _U64MASK, mem)
                if not op:
                    raise RuntimeError(_err())
                ctx._ops[op] = ("fut", loop, fut, keep, None)
            if ctx._spin_loop is None:
                ctx._kick()
            return fut

        def evaluate_perf(self, msg_size: int) -> float:
            t = lib.sw_evaluate_perf(self._ctx._h, self._w, 0, msg_size)
            if t < 0:
                raise RuntimeError(_err())
            return t

    return SimpleNamespace(
        lib=lib,
        Context=Context,
        Server=Server,
        Client=Client,
        ServerEndpoint=ServerEndpoint,
        get_context=get_context,
        shutdown=shutdown,
        status_string=status_string,
        backend_name=lambda: lib.sw_backend_name().decode(),
        device_count=lambda: lib.sw_device_count(),
        local_cpus=local_cpus,
        bind_to_device_numa=bind_to_device_numa,
    )
