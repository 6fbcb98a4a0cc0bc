"""CPU suite: the reference's integration tests (tests/cases_basic.py) driven through the
REAL host progress engine linked against the test-only device simulator (tests/hostsim).
Covers connection, eager / rendezvous protocol, credits, flush, close, cancellation and
world_size-2 (two processes) operation without a GPU."""
import asyncio

import numpy as np
import pytest

from tests import cases_basic as cb


def run(coro):
    return asyncio.run(asyncio.wait_for(coro, timeout=120))


@pytest.mark.parametrize("case", cb.SINGLE_PROCESS_CASES, ids=lambda c: c.__name__)
def test_reference_case(sim_api, port, case):
    run(case(sim_api, port))


@pytest.mark.parametrize("size", [1, 1024, 4096, 8128, 8129, 65536, 1 << 20, (1 << 22) + 13])
def test_message_integrity(sim_api, port, size):
    run(cb.case_message_integrity(sim_api, port, size))


@pytest.mark.parametrize("mode", ["flush", "flush_ep"])
def test_two_process_server_send_with_flush_good(sim_api, port, mode):
    run(cb.case_server_send_with_flush_good(sim_api, port, "sim", mode))


def test_two_process_client_send_with_flush_good(sim_api, port):
    run(cb.case_client_send_with_flush_good(sim_api, port, "sim"))


@pytest.mark.parametrize("seed", range(12))
def test_random_schedule_vs_oracle(sim_api, port, seed):
    run(cb.case_random_schedule_vs_oracle(sim_api, port, seed, quiesce=0.002))


def _proc_connect_and_die(port, q):
    import os
    import signal

    api = cb.load_api("sim")

    async def inner():
        client = api.Client()
        await client.aconnect(cb.SERVER_ADDR, port)
        await client.asend(__import__("numpy").arange(100, dtype="uint8"), 5)  # eager: delivered
        big = __import__("numpy").ones(1 << 20, dtype="uint8")
        client.asend(big, 6)  # rendezvous: never matched before we die
        await asyncio.sleep(0.2)
        q.put("ready")
        await asyncio.sleep(30)

    try:
        asyncio.run(inner())
    finally:
        os.kill(os.getpid(), signal.SIGKILL)


def test_peer_killed_does_not_hang_close(sim_api, port):
    """Failure handling the reference leaves to UCX (SURVEY 5): a peer that dies without closing must
    not wedge the survivor — delivered eager data stays readable and aclose() returns."""
    import multiprocessing as mp

    import numpy as np

    async def go():
        server = sim_api.Server()
        server.listen(cb.SERVER_ADDR, port)
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        p = ctx.Process(target=_proc_connect_and_die, args=(port, q))
        p.start()
        loop = asyncio.get_running_loop()
        assert await loop.run_in_executor(None, q.get, True, 60) == "ready"
        p.kill()
        p.join()
        buf = np.zeros(100, dtype=np.uint8)
        assert await asyncio.wait_for(server.arecv(buf, 5, (1 << 64) - 1), 10) == (5, 100)
        np.testing.assert_array_equal(buf, np.arange(100, dtype=np.uint8))
        pending = server.arecv(np.zeros(8, dtype=np.uint8), 77, (1 << 64) - 1)
        await asyncio.wait_for(server.aclose(), 15)
        with pytest.raises(Exception, match="cancel"):
            await pending

    run(go())


@pytest.mark.parametrize("seed", range(4))
def test_multi_sender_invariants(sim_api, port, seed):
    run(cb.case_multi_sender_invariants(sim_api, port, seed))


def test_stalled_ring_does_not_block_other_senders(sim_api, port):
    """Unexpected-heap exhaustion back-pressures ONE ring; traffic of other endpoints that matches
    posted receives must still flow (no head-of-line blocking across senders)."""
    import numpy as np

    async def go():
        ctx = sim_api.get_context()
        old = ctx.get_option("heap_big_blocks")
        ctx.set_option("heap_big_blocks", 2)
        try:
            server = sim_api.Server()
            server.listen(cb.SERVER_ADDR, port)
        finally:
            ctx.set_option("heap_big_blocks", old)
        a, b = sim_api.Client(), sim_api.Client()
        await a.aconnect(cb.SERVER_ADDR, port)
        await b.aconnect(cb.SERVER_ADDR, port)
        want = np.zeros(4096, dtype=np.uint8)
        fut = server.arecv(want, 0x77, (1 << 64) - 1)
        floods = [asyncio.ensure_future(a.asend(np.full(4096, i, dtype=np.uint8), 0x10 + i)) for i in range(10)]
        await asyncio.sleep(0.2)  # ring A is now stalled behind a full heap
        await b.asend(np.full(4096, 0xAB, dtype=np.uint8), 0x77)
        assert await asyncio.wait_for(fut, 10) == (0x77, 4096)
        assert (want == 0xAB).all()
        # draining the flood releases the stall, in order
        for i in range(10):
            buf = np.zeros(4096, dtype=np.uint8)
            assert await asyncio.wait_for(server.arecv(buf, 0, 0), 10) == (0x10 + i, 4096)
            assert (buf == i).all()
        await asyncio.gather(*floods)
        await a.aclose()
        await b.aclose()
        await server.aclose()

    run(go())


@pytest.mark.parametrize("opts", [{"done_flags": 0}, {"profile": 2}, {"profile": 1}],
                         ids=["events_only", "timed_events", "bulk_timing"])
def test_completion_detection_modes(sim_api, port, opts):
    """Engine side of the completion-flag / event split (the GPU suite runs the same on hardware)."""
    from tests.conftest import free_port

    ctx = sim_api.get_context()
    try:
        for k, v in opts.items():
            ctx.set_option(k, v)
        run(cb.case_random_schedule_vs_oracle(sim_api, port, 11))
        run(cb.case_chaos(sim_api, free_port(), 21))
    finally:
        ctx.set_option("done_flags", 1)
        ctx.set_option("profile", 0)


def test_connection_churn_recycles_native_records(sim_api, port):
    """Creating and dropping Servers / Clients must not grow the process: the native worker and
    endpoint records are type-stable slabs (handle = pointer | generation << 48) that are reused once
    the owner is gone, and the context keeps only weak references to Server objects."""
    import gc

    import numpy as np

    ptr_mask = (1 << 48) - 1
    seen_server, seen_ep, handles = set(), set(), []

    async def cycle(i):
        server = sim_api.Server()
        addr = server.listen_address()
        clients = [sim_api.Client() for _ in range(2)]
        for c in clients:
            await c.aconnect_address(addr)
        buf = np.zeros(64, dtype=np.uint8)
        fut = server.arecv(buf, 5, 0xFF)
        await clients[0].asend(np.full(64, i & 0xFF, dtype=np.uint8), 5)
        assert await fut == (5, 64) and (buf == (i & 0xFF)).all()
        for _ in range(200):
            if len(server.list_clients()) == 2:
                break
            await asyncio.sleep(0.005)
        eps = list(server.list_clients())
        assert len(eps) == 2
        seen_server.add(server._w & ptr_mask)
        handles.append(server._w)
        for ep in eps:
            seen_ep.add(ep._id & ptr_mask)
        for c in clients:
            await c.aclose()
        await server.aclose()
        return eps[0]  # an endpoint object that outlives its server

    stale = None
    for i in range(40):
        stale = run(cycle(i))
        gc.collect()
    assert len(set(handles)) == len(handles)           # every handle value is unique (generation tag) ...
    assert len(seen_server) <= 6 and len(seen_ep) <= 12  # ... while the storage behind them is reused
    # a handle of a recycled record fails the generation check instead of aliasing the new owner
    lib = sim_api.lib
    import ctypes

    buf = (ctypes.c_uint64 * 8)()
    assert lib.sw_list_eps(sim_api.get_context()._h, handles[0], buf, 8) == -1
    assert stale.name  # metadata was copied at creation; the object stays usable


# ---------------------------------------------------------------- 'device' buffers on the CPU stand-in
# The stand-in's device allocator hands out memory its pointer query reports as device memory
# (tests/hostsim SimDev): the engine's device-buffer paths run on the CPU as well — eager payloads read
# straight from the user buffer, zero-copy rendezvous between user buffers, IPC export of user
# allocations with its handle cache, truncation into device buffers.
@pytest.mark.parametrize("seed", [21, 22, 23])
def test_simdev_random_schedules_vs_oracle(sim_api, port, seed):
    from tests.hostsim import SimDev

    run(cb.case_random_schedule_vs_oracle(sim_api, port, seed, SimDev))


@pytest.mark.parametrize("seed", [0, 1])
def test_simdev_multi_sender_invariants(sim_api, port, seed):
    from tests.hostsim import SimDev

    run(cb.case_multi_sender_invariants(sim_api, port, seed, SimDev))


@pytest.mark.parametrize("seed", [31, 32, 33])
def test_simdev_chaos(sim_api, port, seed):
    from tests.hostsim import SimDev

    run(cb.case_chaos(sim_api, port, seed, bufs=SimDev))


@pytest.mark.parametrize("size", [1, 8128, 8129, 65536 + 3, (4 << 20) + 16])
def test_simdev_mixed_host_and_device_buffers(sim_api, port, size):
    """device -> host, host -> device and device -> device, same bytes every way."""
    import numpy as np

    from tests.hostsim import SimDev

    async def go():
        async with cb.gen_server_client(sim_api, port) as (server, client):
            ep = next(iter(server.list_clients()))
            src = np.random.default_rng(size).integers(0, 256, size, dtype=np.uint8)
            dsrc = SimDev.from_np(src)
            # device -> host
            hdst = np.zeros(size + 5, dtype=np.uint8)
            f = server.arecv(hdst, 1, 0xFF)
            await client.asend(dsrc, 1)
            assert await f == (1, size)
            np.testing.assert_array_equal(hdst[:size], src)
            assert (hdst[size:] == 0).all()
            # host -> device
            ddst = SimDev.alloc(size + 5)
            f = client.arecv(ddst, 2, 0xFF)
            await server.asend(ep, src, 2)
            assert await f == (2, size)
            np.testing.assert_array_equal(SimDev.to_np(ddst)[:size], src)
            assert (SimDev.to_np(ddst)[size:] == 0xEE).all()
            # device -> device
            ddst2 = SimDev.alloc(size)
            f = server.arecv(ddst2, 3, 0xFF)
            await client.asend(dsrc, 3)
            assert await f == (3, size)
            np.testing.assert_array_equal(SimDev.to_np(ddst2), src)
            await asyncio.gather(client.aflush(), server.aflush())

    run(go())


@pytest.mark.parametrize("exportable", [True, False], ids=["ipc-exportable", "not-exportable"])
def test_simdev_two_process_device_buffers(sim_api, port, exportable):
    """Rendezvous pulls straight out of another process's user 'device' allocation (IPC export by
    the sender, mapping cache on the receiver), three rounds over the same allocations."""
    run(cb.case_simdev_two_process_device_buffers(sim_api, port, exportable))


def test_round_trip_after_a_long_idle_period(sim_api, port):
    """After more than a second of silence the progress thread naps (futex, 300 us at a time) and the
    asyncio loop sleeps in epoll; a submission wakes the former at once.  Functional check: the first
    round trip after the pause completes promptly (thread wake-ups cost ~0.1-0.3 ms on a busy CI host,
    so the bound is loose) and carries the right bytes."""
    import time

    import numpy as np

    async def go():
        async with cb.gen_server_client(sim_api, port) as (server, client):
            buf, src = np.zeros(8, dtype=np.uint8), np.arange(8, dtype=np.uint8)

            async def rtt(tag):
                src[0] = tag
                t0 = time.perf_counter()
                f = server.arecv(buf, tag, 0xFF)
                await client.asend(src, tag)
                assert await f == (tag, 8)
                assert (buf == src).all()
                return time.perf_counter() - t0

            for i in range(20):
                await rtt(i)
            for i in range(3):
                await asyncio.sleep(1.2)
                assert await rtt(100 + i) < 0.05

    run(go())


@pytest.mark.parametrize("opts", [{"hostdst_ce": 1, "pinned_send_direct": 0}, {"stage_batch_bytes": 65536}, {"pull_keep_us": 0},
                                  {"hostdst_tma": 1, "stage_upload_kernel": 1}],
                         ids=["ce_download", "small_stage_batches", "pull_leaves_at_once", "tma_host_legs"])
def test_host_buffer_and_pull_options(sim_api, port, opts):
    """The tunables of the host-buffer legs and of the pull kernel's stay (INTEGRATION.md) keep every message intact:
    mixed host / device buffers, eager and rendezvous sizes, and a random schedule against the oracle."""
    from tests.conftest import free_port

    ctx = sim_api.get_context()
    defaults = {k: ctx.get_option(k) for k in ("pull_keep_us",)}
    try:
        for k, v in opts.items():
            ctx.set_option(k, v)
        for size in (100, 70000, 3 << 20):
            run(cb.case_message_integrity(sim_api, free_port(), size))
        run(cb.case_random_schedule_vs_oracle(sim_api, port, 5))
    finally:
        for k, v in {"hostdst_ce": 0, "hostdst_tma": 0, "stage_upload_kernel": 0, "pinned_send_direct": 1,
                     "stage_batch_bytes": 4 << 20, **defaults}.items():
            ctx.set_option(k, v)


def test_options_from_the_environment(port):
    """STARWAY_OPTS="key=value,..." is applied when a context is created; unknown keys are reported, not fatal."""
    import os
    import subprocess
    import sys

    code = ("from tests import hostsim; sw = hostsim.load(); c = sw.get_context(); "
            "print(c.get_option('pull_keep_us'), c.get_option('linger_us')); sw.shutdown()")
    env = dict(os.environ, STARWAY_OPTS="pull_keep_us=7,linger_us=33,no_such_option=1", STARWAY_QUIET="1")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", code], env=env, cwd=root, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    assert out.stdout.split()[-2:] == ["7", "33"], out.stdout
    assert "no_such_option" in out.stderr


def test_pull_ctas_of_one_is_refused(sim_api):
    """A pull grid of one CTA is CTA 0 alone, which copies nothing: rendezvous receives handed to it would never
    complete.  `sw_set_option("pull_ctas", 1)` fails and leaves the value as it was; 0 and 2 are accepted.
    STARWAY_PULL_CTAS=1 is ignored with a warning."""
    import os
    import subprocess
    import sys

    ctx = sim_api.get_context()
    old = ctx.get_option("pull_ctas")
    try:
        ctx.set_option("pull_ctas", 2)
        with pytest.raises(ValueError, match="pull_ctas"):
            ctx.set_option("pull_ctas", 1)
        assert ctx.get_option("pull_ctas") == 2
        ctx.set_option("pull_ctas", 0)
        assert ctx.get_option("pull_ctas") == 0
    finally:
        ctx.set_option("pull_ctas", old)

    code = ("from tests import hostsim; sw = hostsim.load(); c = sw.get_context(); "
            "print(c.get_option('pull_ctas')); sw.shutdown()")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    outs = {}
    for name, value in (("STARWAY_PULL_CTAS", "1"), ("STARWAY_OPTS", "pull_ctas=1"), ("STARWAY_PULL_CTAS", "3")):
        env = dict(os.environ, STARWAY_QUIET="1")
        env.pop("STARWAY_PULL_CTAS", None)
        env.pop("STARWAY_OPTS", None)
        env[name] = value
        out = subprocess.run([sys.executable, "-c", code], env=env, cwd=root, capture_output=True, text=True, timeout=120)
        assert out.returncode == 0, out.stderr
        outs[(name, value)] = (int(out.stdout.split()[-1]), out.stderr)
    default = outs[("STARWAY_PULL_CTAS", "1")][0]
    assert default not in (0, 1), outs
    assert outs[("STARWAY_OPTS", "pull_ctas=1")][0] == default, outs
    assert outs[("STARWAY_PULL_CTAS", "3")][0] == 3 and "ignored" not in outs[("STARWAY_PULL_CTAS", "3")][1], outs
    for key in (("STARWAY_PULL_CTAS", "1"), ("STARWAY_OPTS", "pull_ctas=1")):
        assert "pull_ctas" in outs[key][1].lower() and "ignored" in outs[key][1], outs


@pytest.mark.parametrize("bound", [1, 2])
def test_mapping_cache_eviction(sim_api, port, bound):
    """More peer allocations than the receiver keeps mapped (`max_mappings`): the least recently used idle mappings are
    dropped — after the resident control kernels have left and outstanding pulls have drained — the device table is
    rebuilt, and an allocation whose mapping was dropped is simply mapped again.  Three rendezvous-size sources, three
    rounds over them, every payload checked."""
    ctx = sim_api.get_context()
    old = ctx.get_option("max_mappings")
    try:
        ctx.set_option("max_mappings", bound)
        run(cb.case_simdev_two_process_device_buffers(sim_api, port, True))
    finally:
        ctx.set_option("max_mappings", old)


class _DevSlice:
    """A window of a 'device' allocation of the stand-in (one allocation, many messages)."""

    def __init__(self, pool, off, n):
        self.ptr, self.n, self._pool = pool.ptr + off, n, pool
        self.np = pool.np[off:off + n]

    @property
    def __cuda_array_interface__(self):
        return {"shape": (self.n,), "typestr": "|u1", "data": (self.ptr, False), "version": 2}


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("first", ["sends_first", "receives_first"])
def test_more_rendezvous_in_flight_than_ring_slots_and_fin_words(sim_api, port, first, mem):
    """2500 rendezvous-size messages on one connection, posted faster than they can complete: more than the 1024 ring
    slots, the 1023 FIN words per direction and the 64-entry pull batches hold at once.  Credits, the FIN-word window and
    the unexpected queue's heap (RTS descriptors) have to back-pressure without losing or reordering anything."""
    n, size = 2500, 9000

    async def go():
        async with cb.gen_server_client(sim_api, port) as (server, client):
            if mem == "host":
                src = [np.full(size, i & 0xFF, dtype=np.uint8) for i in range(n)]
                dst = [np.zeros(size, dtype=np.uint8) for _ in range(n)]
            else:   # device buffers: matched, copied and completed (FIN words) by the 'kernels'
                from tests.hostsim import SimDev

                stride = (size + 255) & ~255
                spool, dpool = SimDev.alloc(n * stride), SimDev.alloc(n * stride)
                src = [_DevSlice(spool, i * stride, size) for i in range(n)]
                dst = [_DevSlice(dpool, i * stride, size) for i in range(n)]
                for i, s_ in enumerate(src):
                    s_.np[:] = i & 0xFF
                dpool.np[:] = 0
            if first == "sends_first":
                sends = [client.asend(s, 5) for s in src]
                await asyncio.sleep(0.05)
                recvs = [server.arecv(d, 5, 0xFFFF) for d in dst]
            else:
                recvs = [server.arecv(d, 5, 0xFFFF) for d in dst]
                sends = [client.asend(s, 5) for s in src]
            for f in recvs:
                assert await asyncio.wait_for(f, 120) == (5, size)
            await asyncio.wait_for(asyncio.gather(*sends), 120)
            await client.aflush()
            for i, d in enumerate(dst):      # per-sender FIFO: message i lands in receive i
                a = d if mem == "host" else d.np
                assert a[0] == (i & 0xFF) and a[-1] == (i & 0xFF), i

    run(go())
