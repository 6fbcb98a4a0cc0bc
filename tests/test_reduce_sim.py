"""CPU suite for arecv_reduce: the real host engine against the test-only device stand-in (tests/hostsim), with
'device' buffers from its allocator.  Covers the landing blocks of eager messages, the host-path routing of
rendezvous messages, FIN / sender completion on refused messages, close, mixed schedules against the tag-matching
oracle and a two-process sender."""
import asyncio

import numpy as np
import pytest

from tests import cases_basic as cb
from tests.hostsim import SimDev

U64 = (1 << 64) - 1
# name -> (numpy storage type, typestr, SW_DTYPE_*); bfloat16 is stored as uint16 and has no typestr
DTYPES = {
    "float32": (np.float32, "<f4", 1),
    "float16": (np.float16, "<f2", 2),
    "bfloat16": (np.uint16, None, 3),
    "float64": (np.float64, "<f8", 4),
    "int32": (np.int32, "<i4", 5),
    "int64": (np.int64, "<i8", 6),
}


def run(coro):
    return asyncio.run(asyncio.wait_for(coro, timeout=120))


class Typed:
    """A typed 1-D 'device' array of the stand-in backend, exposed through __cuda_array_interface__."""

    def __init__(self, name, n, offset=0, typestr=None):
        self.name = name
        st, ts, _ = DTYPES[name]
        self.st = np.dtype(st)
        self.typestr = typestr or ts
        self.raw = SimDev.Buf(SimDev.lib(), n * self.st.itemsize + offset)
        self.offset = offset
        self.n = n
        self.np = self.raw.np[offset:offset + n * self.st.itemsize].view(self.st)

    @property
    def ptr(self):
        return self.raw.ptr + self.offset

    @property
    def __cuda_array_interface__(self):
        return {"shape": (self.n,), "typestr": self.typestr, "data": (self.ptr, False), "version": 2}


def values(name, n, rng):
    st = DTYPES[name][0]
    if name == "bfloat16":
        return f32_to_bf16(rng.standard_normal(n).astype(np.float32))
    if name.startswith("int"):
        return rng.integers(-1000, 1000, n).astype(st)
    return rng.standard_normal(n).astype(st)


def bf16_to_f32(u):
    return (u.astype(np.uint32) << 16).view(np.float32)


def f32_to_bf16(f):
    u = f.view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def add(name, a, b):
    """a + b as one rounded add of the type (integers wrap)."""
    if name == "bfloat16":
        return f32_to_bf16(bf16_to_f32(a) + bf16_to_f32(b))
    with np.errstate(over="ignore"):
        return (a + b).astype(a.dtype)


def arecv_reduce(api, worker, buf, tag, mask):
    """bfloat16 has no typestr: post it through the C ABI and register the future the way the binding does."""
    if buf.typestr is not None:
        return worker.arecv_reduce(buf, tag, mask)
    ctx = worker._ctx
    loop = asyncio.get_running_loop()
    ctx.ensure_reader(loop)
    fut = loop.create_future()
    with ctx._lock:
        op = api.lib.sw_post_recv_reduce(ctx._h, worker._w, buf.ptr, buf.n * 2, tag, mask, DTYPES[buf.name][2])
        assert op, api.lib.sw_last_error()
        ctx._ops[op] = ("fut", loop, fut, buf, None)
    ctx._kick()
    return fut


async def pair(api, port):
    server, client = api.Server(), api.Client()
    server.listen(cb.SERVER_ADDR, port)
    await client.aconnect(cb.SERVER_ADDR, port)
    return server, client


def sizes(name):
    isz = np.dtype(DTYPES[name][0]).itemsize
    return [1, 8128 // isz, 8128 // isz + 1, (1 << 20) // isz + 7]


@pytest.mark.parametrize("arrival", ["expected", "unexpected"])
@pytest.mark.parametrize("name", list(DTYPES))
def test_reduce_values(sim_api, port, name, arrival):
    async def go():
        server, client = await pair(sim_api, port)
        rng = np.random.default_rng(7)
        for n in sizes(name):
            for src_kind in ("device", "host"):
                extra = 5   # the message fills part of the buffer: the rest stays as it was
                dst = Typed(name, n + extra)
                dst.np[:] = values(name, n + extra, rng)
                dst0 = dst.np.copy()
                data = values(name, n, rng)
                src = SimDev.from_np(data.view(np.uint8)) if src_kind == "device" else data.view(np.uint8)
                if arrival == "expected":
                    fut = arecv_reduce(sim_api, server, dst, 3, U64)
                    send = client.asend(src, 3)
                else:
                    send = asyncio.ensure_future(client.asend(src, 3))
                    await asyncio.sleep(0.01)
                    fut = arecv_reduce(sim_api, server, dst, 3, U64)
                assert await asyncio.wait_for(fut, 20) == (3, data.nbytes), (n, src_kind)
                await asyncio.wait_for(send, 20)
                want = dst0.copy()
                want[:n] = add(name, dst0[:n], data)
                np.testing.assert_array_equal(dst.np.view(np.uint8), want.view(np.uint8), err_msg=f"{n} {src_kind}")
        await client.aclose()
        await server.aclose()

    run(go())


@pytest.mark.parametrize("n_bytes", [40, 8124, 30000])
def test_reduce_refused_messages_leave_the_buffer_alone(sim_api, port, n_bytes):
    """Too long -> "Message truncated", not whole elements -> "Invalid parameter", length 0 -> (tag, 0); the
    buffer keeps its bytes and the sender's send succeeds in all three cases."""

    async def go():
        server, client = await pair(sim_api, port)
        dst = Typed("float32", n_bytes // 4)
        dst.np[:] = np.arange(dst.n, dtype=np.float32)
        before = dst.np.copy()
        cases = [(n_bytes + 4, "truncated"), (n_bytes - 2, "Invalid parameter"), (0, None)]
        for length, err in cases:
            fut = server.arecv_reduce(dst, 9, U64)
            send = client.asend(SimDev.from_np(np.full(length, 0x3F, dtype=np.uint8)), 9)
            if err is None:
                assert await asyncio.wait_for(fut, 20) == (9, 0)
            else:
                with pytest.raises(Exception, match=err):
                    await asyncio.wait_for(fut, 20)
            assert await asyncio.wait_for(send, 20) is None
            np.testing.assert_array_equal(dst.np, before)
        await client.aclose()
        await server.aclose()

    run(go())


def test_reduce_pending_at_close_is_canceled(sim_api, port):
    async def go():
        server, client = await pair(sim_api, port)
        dst = Typed("int32", 64)
        fut = client.arecv_reduce(dst, 1, U64)
        await client.aclose()
        with pytest.raises(Exception, match="Request canceled"):
            await asyncio.wait_for(fut, 20)
        await server.aclose()

    run(go())


def test_reduce_buffer_checks(sim_api, port):
    """Buffers the reduce cannot take raise TypeError at the call and post nothing."""

    async def go():
        server, client = await pair(sim_api, port)
        host = np.zeros(16, dtype=np.float32)

        class HostCAI:   # host memory dressed up as a CUDA array: the engine's pointer query tells
            __cuda_array_interface__ = {"shape": (16,), "typestr": "<f4", "data": (host.ctypes.data, False), "version": 2}

        bad = [
            host,                                   # NumPy array
            HostCAI(),                              # not device memory
            Typed("float32", 8, typestr="|u1"),     # unsupported element type
            Typed("float32", 8, offset=2),          # not aligned to the element size
        ]
        for b in bad:
            with pytest.raises(TypeError):
                server.arecv_reduce(b, 0, 0)
        lib, ctx = sim_api.lib, server._ctx
        d = Typed("float32", 8)
        assert lib.sw_post_recv_reduce(ctx._h, server._w, d.ptr, 32, 0, 0, 99) == 0
        assert b"element type" in lib.sw_last_error()
        assert lib.sw_post_recv_reduce(ctx._h, server._w, d.ptr, 30, 0, 0, 1) == 0
        assert b"multiples" in lib.sw_last_error()
        # nothing was posted: a message finds no receive
        buf = SimDev.alloc(4)
        f = server.arecv(buf, 0, 0)
        await client.asend(SimDev.from_np(np.arange(4, dtype=np.uint8)), 5)
        assert await asyncio.wait_for(f, 20) == (5, 4)
        await client.aclose()
        await server.aclose()

    run(go())


@pytest.mark.parametrize("seed", range(8))
def test_reduce_random_schedule_vs_oracle(sim_api, port, seed):
    """arecv / arecv_reduce (int32) / asend issued one at a time; every receive pairs with the oracle's message.
    A reducing receive's oracle mirror is a scratch buffer that is added into the expected tensor."""
    from oracle.tagmatch import ORC_OK, COracle

    async def go():
        rng = np.random.default_rng(seed)
        masks = [0, U64, 0xFF, 0xF0, 0xFFFF]
        lens = [0, 1, 8, 16, 100, 256, 4096, 8128, 8132, 20000, 70000]
        server, client = await pair(sim_api, port)
        orc = COracle()
        futs, bufs, mirror, expect, kind, sends, keep, want = {}, {}, {}, {}, {}, [], [], {}
        op = 1
        for _ in range(48):
            if rng.random() < 0.5:
                tag, mask = int(rng.integers(0, 5)), masks[int(rng.integers(0, 5))]
                cap = int(rng.choice([0, 8, 300, 8128, 100000]))
                mirror[op] = np.full(cap, 0xEE, dtype=np.uint8)
                if rng.random() < 0.5:
                    kind[op] = "reduce"
                    bufs[op] = Typed("int32", cap // 4)
                    bufs[op].np[:] = rng.integers(-(1 << 31), 1 << 31, cap // 4, dtype=np.int64).astype(np.int32)
                    expect[op] = bufs[op].np.copy()
                    futs[op] = server.arecv_reduce(bufs[op], tag, mask)
                else:
                    kind[op] = "copy"
                    bufs[op] = SimDev.alloc(cap)
                    futs[op] = server.arecv(bufs[op], tag, mask)
                m = orc.post_recv(op, tag, mask, mirror[op])
                op += 1
            else:
                stag = int(rng.integers(0, 5)) | (int(rng.integers(0, 2)) << 8)
                data = rng.integers(0, 256, int(rng.choice(lens)), dtype=np.uint8)
                t = SimDev.from_np(data)
                keep.append(t)
                sends.append(asyncio.ensure_future(client.asend(t, stag)))
                m = orc.arrive(0, stag, data)
            if m is not None:
                want[m.op_id] = m
            await asyncio.sleep(0.002)
        for o, m in want.items():
            if m.status == ORC_OK and (kind[o] == "copy" or m.length % 4 == 0):
                assert await asyncio.wait_for(futs[o], 20) == (m.sender_tag, m.length), (seed, o)
                if kind[o] == "reduce":
                    k = m.length // 4
                    expect[o][:k] = add("int32", expect[o][:k], mirror[o][: m.length].view(np.int32))
            else:
                err = "truncated" if m.status != ORC_OK else "Invalid parameter"
                with pytest.raises(Exception, match=err):
                    await asyncio.wait_for(futs[o], 20)
        await asyncio.sleep(0.05)
        for o in futs:
            if o not in want:
                assert not futs[o].done(), (seed, o)
            if kind[o] == "reduce":
                np.testing.assert_array_equal(bufs[o].np, expect[o])
            else:
                np.testing.assert_array_equal(SimDev.to_np(bufs[o]), mirror[o])
        await client.aclose()
        await server.aclose()
        res = await asyncio.gather(*sends, *[f for o, f in futs.items() if o not in want], return_exceptions=True)
        for r in res:
            assert r is None or "cancel" in str(r) or "reset" in str(r), r

    run(go())


def _proc_reduce_sender(port, n_eager, n_rndv):
    api = cb.load_api("sim")

    async def inner():
        client = api.Client()
        await client.aconnect(cb.SERVER_ADDR, port)
        for n, tag in ((n_eager, 1), (n_rndv, 2)):
            data = np.arange(n, dtype=np.float32)
            await client.asend(SimDev.from_np(data.view(np.uint8)), tag)   # device source: mapped by the receiver
            await client.asend(data.view(np.uint8), tag)                    # host source: staged by the sender
        await client.aflush()
        await client.aclose()

    asyncio.run(inner())


def test_reduce_two_processes(sim_api, port):
    import multiprocessing as mp

    async def go():
        server = sim_api.Server()
        server.listen(cb.SERVER_ADDR, port)
        n_eager, n_rndv = 1000, 100003
        dst_e, dst_r = Typed("float32", n_eager), Typed("float32", n_rndv)
        dst_e.np[:] = 1.0
        dst_r.np[:] = 1.0
        futs = [server.arecv_reduce(d, t, U64) for d, t in ((dst_e, 1), (dst_e, 1), (dst_r, 2), (dst_r, 2))]
        p = mp.get_context("spawn").Process(target=_proc_reduce_sender, args=(port, n_eager, n_rndv))
        p.start()
        res = await asyncio.wait_for(asyncio.gather(*futs), 60)
        assert res == [(1, 4 * n_eager)] * 2 + [(2, 4 * n_rndv)] * 2
        for d, n in ((dst_e, n_eager), (dst_r, n_rndv)):
            np.testing.assert_array_equal(d.np, 1.0 + 2.0 * np.arange(n, dtype=np.float32))
        loop = asyncio.get_running_loop()
        await loop.run_in_executor(None, p.join, 60)
        assert p.exitcode == 0
        await server.aclose()

    run(go())

