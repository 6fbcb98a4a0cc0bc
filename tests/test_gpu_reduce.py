"""arecv_reduce on the GPU: sums computed by the sm_90a reduce kernels (bulk reductions for the 16-byte-aligned
body, element-wise atomics for the rest) compared bit-exactly with torch's own add in the same dtype."""
import asyncio
import multiprocessing as mp

import numpy as np
import pytest

from tests import cases_basic as cb

pytestmark = pytest.mark.gpu

U64 = (1 << 64) - 1
NAMES = ["float32", "float16", "bfloat16", "float64", "int32", "int64"]


def run(coro, timeout=300):
    return asyncio.run(asyncio.wait_for(coro, timeout=timeout))


def torch_cuda():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch


def dt(name):
    return getattr(torch_cuda(), name)


def bits(t):
    """Integer view of a tensor for bit-exact comparison."""
    torch = torch_cuda()
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def values(name, n, gen, scale=1.0):
    torch = torch_cuda()
    if name.startswith("int"):
        return torch.randint(-1000, 1000, (n,), generator=gen, device="cuda", dtype=dt(name))
    return (torch.randn(n, generator=gen, device="cuda") * scale).to(dt(name))


def sizes(name):
    isz = torch_cuda().empty(0, dtype=dt(name)).element_size()
    return [1, 8128 // isz, 8128 // isz + 1, (1 << 20) // isz + 7, (64 << 20) // isz + 7]


async def pair(api, port):
    server, client = api.Server(), api.Client()
    server.listen(cb.SERVER_ADDR, port)
    await client.aconnect(cb.SERVER_ADDR, port)
    return server, client


async def reduce_one(server, client, dst, src, tag=3, unexpected=False):
    torch = torch_cuda()
    torch.cuda.synchronize()
    if unexpected:
        send = asyncio.ensure_future(client.asend(src, tag))
        await asyncio.sleep(0.005)
        fut = server.arecv_reduce(dst, tag, U64)
    else:
        fut = server.arecv_reduce(dst, tag, U64)
        send = client.asend(src, tag)
    got = await asyncio.wait_for(fut, 60)
    await asyncio.wait_for(send, 60)
    return got


@pytest.mark.parametrize("name", NAMES)
def test_reduce_values(cuda_api, port, name):
    torch = torch_cuda()

    async def go():
        server, client = await pair(cuda_api, port)
        gen = torch.Generator(device="cuda").manual_seed(11)
        for n in sizes(name):
            for unexpected in (False, True):
                dst = values(name, n + 3, gen)
                dst0 = dst.clone()
                src = values(name, n, gen)
                got = await reduce_one(server, client, dst, src, unexpected=unexpected)
                assert got == (3, src.numel() * src.element_size()), (n, unexpected)
                want = dst0.clone()
                want[:n] = dst0[:n] + src
                torch.cuda.synchronize()
                assert torch.equal(bits(dst), bits(want)), (name, n, unexpected)
        await client.aclose()
        await server.aclose()

    run(go())


@pytest.mark.parametrize("name", ["float32", "bfloat16", "int64"])
def test_reduce_alignment(cuda_api, port, name):
    """Destinations at element offsets 1 and 3, senders at an odd byte offset: the bulk path cannot take these, or
    only part of them; body and tail both carry data."""
    torch = torch_cuda()

    async def go():
        server, client = await pair(cuda_api, port)
        gen = torch.Generator(device="cuda").manual_seed(5)
        isz = torch.empty(0, dtype=dt(name)).element_size()
        for n in (8128 // isz - 1, (1 << 20) // isz + 3, (4 << 20) // isz + 5):
            for dst_off in (0, 1, 3):
                for src_off in (0, 1):
                    base = values(name, n + 8, gen)
                    base0 = base.clone()
                    dst = base[dst_off:dst_off + n]
                    data = values(name, n, gen)
                    raw = torch.zeros(n * isz + 16, dtype=torch.uint8, device="cuda")
                    src = raw[src_off:src_off + n * isz]
                    src.copy_(data.view(torch.uint8))
                    assert await reduce_one(server, client, dst, src) == (3, n * isz)
                    want = base0.clone()
                    want[dst_off:dst_off + n] += data
                    torch.cuda.synchronize()
                    assert torch.equal(bits(base), bits(want)), (n, dst_off, src_off)
        await client.aclose()
        await server.aclose()

    run(go())


@pytest.mark.parametrize("name", ["float32", "float16"])
def test_reduce_subnormals(cuda_api, port, name):
    """Subnormal operands and sums are kept, not flushed to zero, on the bulk path and the element-wise path."""
    torch = torch_cuda()
    tiny = torch.finfo(dt(name)).tiny

    async def go():
        server, client = await pair(cuda_api, port)
        gen = torch.Generator(device="cuda").manual_seed(3)
        for n in (8128 // 4 + 1, (1 << 20) + 5):
            # about half the elements subnormal in each operand, signs mixed; the rest normal-range
            a = values(name, n, gen).float() * tiny * 0.5
            b = values(name, n, gen).float() * tiny * 0.5
            keep = torch.rand(n, generator=gen, device="cuda") < 0.5
            a = torch.where(keep, a, a * 1e3).to(dt(name))
            b = torch.where(keep, b, b * 1e3).to(dt(name))
            assert (a != 0).logical_and(a.abs() < tiny).sum() > n // 8
            want = a + b
            assert (want != 0).logical_and(want.abs() < tiny).sum() > n // 8
            assert await reduce_one(server, client, a, b) == (3, b.numel() * b.element_size())
            torch.cuda.synchronize()
            assert torch.equal(bits(a), bits(want)), n
        await client.aclose()
        await server.aclose()

    run(go())


@pytest.mark.parametrize("name", ["float32", "int32", "bfloat16"])
def test_reduce_many_into_one(cuda_api, port, name):
    """Three clients sending four messages each and one client sending 32, every message matched by an
    arecv_reduce with a wildcard mask on ONE tensor, eager and rendezvous sizes.  Integer-valued data: the sum is
    the same in any order."""
    torch = torch_cuda()

    async def go():
        server = cuda_api.Server()
        server.listen(cb.SERVER_ADDR, port)
        clients = [cuda_api.Client() for _ in range(4)]
        for c in clients:
            await c.aconnect(cb.SERVER_ADDR, port)
        gen = torch.Generator(device="cuda").manual_seed(9)
        counts = [4, 4, 4, 32]
        for n in (1000, (2 << 20) + 3):
            # |any partial sum| <= 2 + 44 * 2: exact in every type, bfloat16 included
            acc = torch.randint(-2, 3, (n,), generator=gen, device="cuda").to(dt(name))
            srcs = [[torch.randint(-2, 3, (n,), generator=gen, device="cuda").to(dt(name)) for _ in range(k)]
                    for k in counts]
            want = acc.clone()
            for lst in srcs:
                for s in lst:
                    want += s
            torch.cuda.synchronize()
            futs = [server.arecv_reduce(acc, 0, 0) for _ in range(sum(counts))]
            sends = [c.asend(s, 100 + i) for i, (c, lst) in enumerate(zip(clients, srcs)) for s in lst]
            res = await asyncio.wait_for(asyncio.gather(*futs), 120)
            await asyncio.wait_for(asyncio.gather(*sends), 120)
            assert sorted(t for t, _ in res) == sorted(100 + i for i, k in enumerate(counts) for _ in range(k))
            assert all(ln == n * acc.element_size() for _, ln in res)
            torch.cuda.synchronize()
            assert torch.equal(bits(acc), bits(want)), n
        for c in clients:
            await c.aclose()
        await server.aclose()

    run(go())


@pytest.mark.parametrize("seed", range(4))
def test_reduce_random_schedule_vs_oracle(cuda_api, port, seed):
    """arecv (uint8) / arecv_reduce (int32) / asend issued one at a time against the tag-matching oracle; a reducing
    receive's oracle mirror is a scratch buffer added into the expected tensor."""
    torch = torch_cuda()
    from oracle.tagmatch import ORC_OK, COracle

    async def go():
        rng = np.random.default_rng(seed)
        masks = [0, U64, 0xFF, 0xF0, 0xFFFF]
        lens = [0, 1, 8, 16, 100, 256, 4096, 8128, 8132, 20000, 70000, 1 << 20]
        server, client = await pair(cuda_api, port)
        orc = COracle()
        futs, bufs, mirror, expect, kind, sends, keep, want = {}, {}, {}, {}, {}, [], [], {}
        op = 1
        for _ in range(48):
            if rng.random() < 0.5:
                tag, mask = int(rng.integers(0, 5)), masks[int(rng.integers(0, 5))]
                cap = int(rng.choice([0, 8, 300, 8128, 100000, 2 << 20]))
                mirror[op] = np.full(cap, 0xEE, dtype=np.uint8)
                if rng.random() < 0.5:
                    kind[op] = "reduce"
                    init = rng.integers(-(1 << 31), 1 << 31, cap // 4, dtype=np.int64).astype(np.int32)
                    expect[op] = init.copy()
                    bufs[op] = torch.from_numpy(init).cuda()
                    torch.cuda.synchronize()
                    futs[op] = server.arecv_reduce(bufs[op], tag, mask)
                else:
                    kind[op] = "copy"
                    bufs[op] = torch.full((cap,), 0xEE, dtype=torch.uint8, device="cuda")
                    torch.cuda.synchronize()
                    futs[op] = server.arecv(bufs[op], tag, mask)
                m = orc.post_recv(op, tag, mask, mirror[op])
                op += 1
            else:
                stag = int(rng.integers(0, 5)) | (int(rng.integers(0, 2)) << 8)
                data = rng.integers(0, 256, int(rng.choice(lens)), dtype=np.uint8)
                t = torch.from_numpy(data).cuda()
                keep.append(t)
                torch.cuda.synchronize()
                sends.append(asyncio.ensure_future(client.asend(t, stag)))
                m = orc.arrive(0, stag, data)
            if m is not None:
                want[m.op_id] = m
            await asyncio.sleep(0.004)
        for o, m in want.items():
            if m.status == ORC_OK and (kind[o] == "copy" or m.length % 4 == 0):
                assert await asyncio.wait_for(futs[o], 30) == (m.sender_tag, m.length), (seed, o)
                if kind[o] == "reduce":
                    k = m.length // 4
                    expect[o][:k] = (expect[o][:k].astype(np.int64) + mirror[o][: m.length].view(np.int32)).astype(np.int32)
            else:
                err = "truncated" if m.status != ORC_OK else "Invalid parameter"
                with pytest.raises(Exception, match=err):
                    await asyncio.wait_for(futs[o], 30)
        await asyncio.sleep(0.05)
        torch.cuda.synchronize()
        for o in futs:
            if o not in want:
                assert not futs[o].done(), (seed, o)
            if kind[o] == "reduce":
                np.testing.assert_array_equal(bufs[o].cpu().numpy(), expect[o])
            else:
                np.testing.assert_array_equal(bufs[o].cpu().numpy(), mirror[o])
        await client.aclose()
        await server.aclose()
        res = await asyncio.gather(*sends, *[f for o, f in futs.items() if o not in want], return_exceptions=True)
        for r in res:
            assert r is None or "cancel" in str(r) or "reset" in str(r), r

    run(go())


def test_reduce_host_sources(cuda_api, port):
    """NumPy (pageable, staged by the sender) and pinned-host senders into a device arecv_reduce."""
    torch = torch_cuda()

    async def go():
        server, client = await pair(cuda_api, port)
        for n in (1000, (1 << 20) + 7, (16 << 20) + 1):
            data = torch.arange(n, dtype=torch.float32) % 1000
            for src in (data.numpy().view(np.uint8), data.view(torch.uint8).pin_memory()):
                acc = torch.ones(n, dtype=torch.float32, device="cuda")
                assert await reduce_one(server, client, acc, src) == (3, 4 * n)
                torch.cuda.synchronize()
                assert torch.equal(acc.cpu(), data + 1), (n, type(src))
        await client.aclose()
        await server.aclose()

    run(go())


def _proc_sender(port, ns):
    import torch

    api = cb.load_api("cuda")

    async def inner():
        client = api.Client()
        await client.aconnect(cb.SERVER_ADDR, port)
        for i, n in enumerate(ns):
            src = (torch.arange(n, dtype=torch.float32, device="cuda") % 1000)
            torch.cuda.synchronize()
            await client.asend(src, i)
        await client.aflush()
        await client.aclose()

    asyncio.run(inner())


def test_reduce_two_processes(cuda_api, port):
    """The sender's buffer lives in another process: the receiver maps it (CUDA IPC) and reduces from the mapping."""
    torch = torch_cuda()

    async def go():
        server = cuda_api.Server()
        server.listen(cb.SERVER_ADDR, port)
        ns = [1000, (1 << 20) + 7, (16 << 20) + 1]
        accs = [torch.full((n,), 2.0, device="cuda") for n in ns]
        torch.cuda.synchronize()
        futs = [server.arecv_reduce(a, i, U64) for i, a in enumerate(accs)]
        p = mp.get_context("spawn").Process(target=_proc_sender, args=(port, ns))
        p.start()
        res = await asyncio.wait_for(asyncio.gather(*futs), 240)
        assert res == [(i, 4 * n) for i, n in enumerate(ns)]
        torch.cuda.synchronize()
        for a, n in zip(accs, ns):
            assert torch.equal(a, torch.arange(n, dtype=torch.float32, device="cuda") % 1000 + 2.0), n
        await asyncio.get_running_loop().run_in_executor(None, p.join, 120)
        assert p.exitcode == 0
        await server.aclose()

    run(go())


@pytest.mark.parametrize("n_bytes", [40, 8124, 1 << 20])
def test_reduce_refused_messages(cuda_api, port, n_bytes):
    """Truncated, not whole elements, zero length: the tensor keeps its bytes and the sender's send succeeds."""
    torch = torch_cuda()

    async def go():
        server, client = await pair(cuda_api, port)
        dst = torch.arange(n_bytes // 4, dtype=torch.float32, device="cuda")
        before = dst.clone()
        for length, err in ((n_bytes + 4, "truncated"), (n_bytes - 2, "Invalid parameter"), (0, None)):
            torch.cuda.synchronize()
            fut = server.arecv_reduce(dst, 9, U64)
            send = client.asend(torch.full((length,), 0x3F, dtype=torch.uint8, device="cuda"), 9)
            if err is None:
                assert await asyncio.wait_for(fut, 30) == (9, 0)
            else:
                with pytest.raises(Exception, match=err):
                    await asyncio.wait_for(fut, 30)
            assert await asyncio.wait_for(send, 30) is None
            torch.cuda.synchronize()
            assert torch.equal(dst, before), (length, err)
        fut = server.arecv_reduce(dst, 1, U64)
        await client.aclose()
        await server.aclose()
        with pytest.raises(Exception, match="Request canceled"):
            await asyncio.wait_for(fut, 30)

    run(go())


def test_reduce_rejects_unsupported_buffers(cuda_api, port):
    torch = torch_cuda()

    async def go():
        server, client = await pair(cuda_api, port)
        bad = [
            np.zeros(16, dtype=np.float32),
            torch.zeros(16),                                              # host tensor
            torch.zeros(16, dtype=torch.uint8, device="cuda"),            # unsupported dtype
            torch.zeros(16, 4, device="cuda").t(),                        # not contiguous
        ]
        if torch.cuda.device_count() > 1:
            bad.append(torch.zeros(16, device="cuda:1"))
        for b in bad:
            with pytest.raises(TypeError):
                server.arecv_reduce(b, 0, 0)
        two_d = torch.zeros(4, 8, device="cuda")   # any shape is fine when contiguous
        f = server.arecv_reduce(two_d, 0, 0)
        await client.asend(torch.ones(32, device="cuda"), 1)
        assert await asyncio.wait_for(f, 30) == (1, 128)
        torch.cuda.synchronize()
        assert torch.equal(two_d, torch.ones(4, 8, device="cuda"))
        await client.aclose()
        await server.aclose()

    run(go())
