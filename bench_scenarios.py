#!/usr/bin/env python
"""bench_scenarios.py — the BASELINE.json configurations beyond the headline bench line.

  python bench_scenarios.py sweep                       config 3, 1 GPU loopback (uni + bidirectional)
  torchrun --nproc-per-node 2 bench_scenarios.py sweep  config 3, 2 GPUs over NVLink (rank0 <-> rank1)
  torchrun --nproc-per-node 8 bench_scenarios.py allpairs   config 4: each rank asends 4 MiB to 7 peers, wildcard recv
  torchrun --nproc-per-node 8 bench_scenarios.py storm      config 5: 1 M x 64 B, server.asend + aflush_ep per peer

Every mode prints one JSON line per data point on rank 0 (and appends it to --out).  Device
buffers, public asyncio API; GB/s is payload bytes delivered / wall time; `nvlink_frac` is per-GPU
egress / 450 GB/s (H100 SXM, NVLink 4: the nominal per-direction figure of the data sheet).
"""
from __future__ import annotations

import argparse
import asyncio
import json
import os
import statistics
import sys
import time

NVLINK_NOMINAL_GBS = 450.0  # H100 SXM, NVLink 4, per direction (data sheet)
HBM_DATASHEET_GBS = 3350.0  # H100 SXM HBM3 (data sheet); a loopback copy moves 2 bytes of HBM per payload byte

ROOT = os.path.dirname(os.path.abspath(__file__))
os.environ.setdefault("STARWAY_QUIET", "1")  # no "Connected!" banners: stdout carries JSON lines only
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

U64 = (1 << 64) - 1
DATA_TAG, ACK_TAG, GO_TAG = 0x2B00, 0x1AA2, 0x1AA1


def env():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))


def emit(args, rec):
    line = json.dumps(rec)
    print(line, flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")


def runner():
    try:
        import uvloop

        return uvloop.run
    except Exception:
        return asyncio.run


def setup():
    import torch

    rank, world, local = env()
    torch.cuda.set_device(local)
    os.environ["STARWAY_DEVICE"] = str(local)
    import starway_b200 as sw

    dist = None
    if world > 1:
        import torch.distributed as dist

        dist.init_process_group("gloo", rank=rank, world_size=world)
    return torch, sw, dist, rank, world, local


# ----------------------------------------------------------------------------------------- config 3
def mode_sweep(args):
    torch, sw, dist, rank, world, local = setup()
    assert world in (1, 2)
    dev = torch.device("cuda", local)
    sizes = [1 << k for k in range(6, 31)]
    if args.max_bytes:
        sizes = [s for s in sizes if s <= args.max_bytes]

    async def main():
        server = sw.Server()
        addr = server.listen_address()
        addrs = [addr]
        if dist:
            addrs = [None] * world
            dist.all_gather_object(addrs, addr)
        peer = (rank + 1) % world
        client = sw.Client()
        await client.aconnect_address(addrs[peer])
        for _ in range(2000):
            if server.list_clients():
                break
            await asyncio.sleep(0.005)
        ep = next(iter(server.list_clients()))
        ack = torch.zeros(8, dtype=torch.uint8, device=dev)
        pool_bytes = 1 << 30
        src_pool = torch.empty(pool_bytes, dtype=torch.uint8, device=dev)
        src_pool.view(torch.int64).copy_((torch.arange(pool_bytes // 8, device=dev, dtype=torch.int64) * 2654435761 + rank))
        dst_pool = torch.full((pool_bytes,), 0xEE, dtype=torch.uint8, device=dev)
        torch.cuda.synchronize()

        async def sender(n, window, iters):
            """client -> peer server: `iters` windows of `window` messages, aflush per window, then wait for the ack."""
            bufs = [src_pool[(j * n) % (pool_bytes - n + 1):][:n] for j in range(window)] if n * window <= pool_bytes else [src_pool[:n]] * window
            a = client.arecv(ack, ACK_TAG, U64)
            t0 = time.perf_counter()
            for _ in range(iters):
                sends = [client.asend(b, DATA_TAG) for b in bufs]
                for f in sends:
                    await f
                await client.aflush()
            await a
            return time.perf_counter() - t0

        async def receiver(n, window, iters):
            """server side: pre-post every receive, ack when the last one completed."""
            bufs = [dst_pool[(j * n) % (pool_bytes - n + 1):][:n] for j in range(window)] if n * window <= pool_bytes else [dst_pool[:n]] * window
            recvs = [server.arecv(bufs[j % window], DATA_TAG, U64) for j in range(window * iters)]
            for f in recvs:
                assert await f == (DATA_TAG, n)
            await server.asend(ep, ack, ACK_TAG)

        async def sync():
            if dist:
                await asyncio.get_running_loop().run_in_executor(None, dist.barrier)

        for n in sizes:
            window = min(64, max(1, (1 << 28) // n))
            iters = max(5, min(400, (1 << 31) // (n * window)))
            if n <= 4096:
                iters = max(iters, 100)
                iters = min(iters, 300)
            for direction in ("uni", "bi"):
                times = []
                for rep in range(args.reps + 1):
                    await sync()
                    if world == 1:
                        if direction == "bi":
                            continue
                        r = asyncio.ensure_future(receiver(n, window, iters))
                        t = await sender(n, window, iters)
                        await r
                    else:
                        if direction == "uni":
                            if rank == 0:
                                t = await sender(n, window, iters)
                            else:
                                await receiver(n, window, iters)
                                t = None
                        else:
                            r = asyncio.ensure_future(receiver(n, window, iters))
                            t = await sender(n, window, iters)
                            await r
                    if rep > 0 and t is not None:
                        times.append(t)
                if world == 1 and direction == "bi":
                    continue
                if direction == "bi" and dist:
                    tt = torch.tensor([max(times)], dtype=torch.float64)
                    dist.all_reduce(tt, op=dist.ReduceOp.MAX)
                    worst = float(tt[0])
                if rank == 0:
                    best, med = min(times), statistics.median(times)
                    nbytes = n * window * iters
                    rec = {
                        "scenario": "sweep", "direction": direction, "n_gpus": world, "msg_bytes": n, "window": window,
                        "iters": iters, "gbs_best": round(nbytes / best / 1e9, 3), "gbs_median": round(nbytes / med / 1e9, 3),
                        "mmsg_s_best": round(window * iters / best / 1e6, 4), "us_per_msg": round(best / (window * iters) * 1e6, 3),
                        "per_direction": True,
                    }
                    if world > 1:
                        rec["nvlink_frac"] = round(rec["gbs_best"] / NVLINK_NOMINAL_GBS, 4)
                    else:
                        rec["hbm_frac"] = round(2 * rec["gbs_best"] / HBM_DATASHEET_GBS, 4)
                    if direction == "bi":
                        rec["aggregate_gbs_best"] = round(2 * nbytes / worst / 1e9, 3)
                    emit(args, rec)
        # bit-exactness of the last transfer (size-independent check at the largest size)
        await sync()
        await client.aclose()
        await sync()
        await server.aclose()

    runner()(main())
    sw.shutdown()


# ----------------------------------------------------------------------------------------- config 4
def mode_allpairs(args):
    torch, sw, dist, rank, world, local = setup()
    dev = torch.device("cuda", local)
    n = args.msg_bytes or (4 << 20)
    rounds, warm = args.rounds, 10

    async def main():
        server = sw.Server()
        addr = server.listen_address()
        addrs = [None] * world
        dist.all_gather_object(addrs, addr)
        peers = [p for p in range(world) if p != rank]
        clients = {}
        for p in peers:
            c = sw.Client()
            await c.aconnect_address(addrs[p])
            clients[p] = c
        for _ in range(4000):
            if len(server.list_clients()) >= len(peers):
                break
            await asyncio.sleep(0.005)
        assert len(server.list_clients()) == len(peers)
        src = {p: torch.full((n,), (rank * 16 + p) & 0xFF, dtype=torch.uint8, device=dev) for p in peers}
        dst = [torch.zeros(n, dtype=torch.uint8, device=dev) for _ in peers]
        torch.cuda.synchronize()
        loop = asyncio.get_running_loop()

        async def one_round():
            recvs = [server.arecv(d, 0, 0) for d in dst]          # wildcard: source identified by sender_tag
            sends = [clients[p].asend(src[p], rank) for p in peers]
            res = [await f for f in recvs]
            for f in sends:
                await f
            return res

        counts = {}
        for i in range(warm + rounds):
            if i == warm:
                await loop.run_in_executor(None, dist.barrier)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
            res = await one_round()
            for tag, length in res:
                assert length == n and 0 <= tag < world and tag != rank
                counts[tag] = counts.get(tag, 0) + 1
        torch.cuda.synchronize()
        el = time.perf_counter() - t0
        assert sorted(counts) == peers and all(v == warm + rounds for v in counts.values()), counts
        # the last round's payloads: every destination holds the fill pattern of the peer its sender_tag names
        # (ranks drift apart without a barrier per round: a round's seven wildcard receives may well hold two
        # messages of a fast peer -- the tag says which; tests/test_gpu_multi.py compares full payloads)
        for d, (tag, _) in zip(dst, res):
            assert int(d[0]) == ((tag * 16 + rank) & 0xFF) and int(d[-1]) == int(d[0]), (tag, int(d[0]))
        t = torch.tensor([el], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        el = float(t[0])
        if rank == 0:
            per_gpu = len(peers) * n * rounds / el / 1e9
            emit(args, {"scenario": "allpairs", "n_gpus": world, "msg_bytes": n, "rounds": rounds,
                        "per_gpu_egress_gbs": round(per_gpu, 2), "aggregate_gbs": round(per_gpu * world, 2),
                        "nvlink_frac": round(per_gpu / NVLINK_NOMINAL_GBS, 4), "ms_per_round": round(el / rounds * 1e3, 4)})
        await loop.run_in_executor(None, dist.barrier)
        for c in clients.values():
            await c.aclose()
        await loop.run_in_executor(None, dist.barrier)
        await server.aclose()

    runner()(main())
    sw.shutdown()


# ----------------------------------------------------------------------------------------- config 5
def mode_storm(args):
    torch, sw, dist, rank, world, local = setup()
    dev = torch.device("cuda", local)
    total = args.total_msgs
    per_pair = total // (world * (world - 1))
    n = 64

    async def main():
        server = sw.Server()
        addr = server.listen_address()
        addrs = [None] * world
        dist.all_gather_object(addrs, addr)
        peers = [p for p in range(world) if p != rank]
        clients = {}
        for p in peers:
            c = sw.Client()
            await c.aconnect_address(addrs[p])
            clients[p] = c
        for _ in range(4000):
            if len(server.list_clients()) >= len(peers):
                break
            await asyncio.sleep(0.005)
        eps = list(server.list_clients())
        assert len(eps) == len(peers)
        src = torch.arange(n, dtype=torch.uint8, device=dev)
        dst = {p: torch.zeros(n, dtype=torch.uint8, device=dev) for p in peers}
        torch.cuda.synchronize()
        ctx = sw.get_context()
        ctx.set_option("profile", 1)
        loop = asyncio.get_running_loop()
        await loop.run_in_executor(None, dist.barrier)
        ctx.reset_stats()
        t0 = time.perf_counter()
        # receivers: every client pre-posts its receives (full mask on the per-peer tag prefix is not
        # needed: one sender per client worker) -- wildcard receives
        recvs = [clients[p].arecv(dst[p], 0, 0) for p in peers for _ in range(per_pair)]
        # senders: the Server sends to each of its 7 endpoints, then aflush_ep per peer
        sends = [server.asend(ep, src, (rank << 32) | i) for i in range(per_pair) for ep in eps]
        for f in sends:  # awaiting in order is cheaper than gather over 10^5 futures
            await f
        for f in [server.aflush_ep(ep) for ep in eps]:
            await f
        res = [await f for f in recvs]
        torch.cuda.synchronize()
        el = time.perf_counter() - t0
        assert all(length == n for _, length in res)
        assert len({t for t, _ in res}) == len(res)
        st = ctx.stats()
        t = torch.tensor([el], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        el = float(t[0])
        if rank == 0:
            msgs = per_pair * world * (world - 1)
            emit(args, {"scenario": "storm", "n_gpus": world, "msg_bytes": n, "total_msgs": msgs,
                        "api_mmsg_s": round(msgs / el / 1e6, 4), "seconds": round(el, 3),
                        "kernel_level": {
                            "put_msgs": st["put_msgs"], "put_launches": st["put_launches"],
                            "put_mmsg_s": round(st["put_msgs"] / max(st["put_event_ms"], 1e-9) / 1e3, 2),
                            "match_arrivals": st["match_arrivals"],
                            "note": "rank 0 counters; device time of the launches from CUDA events"}})
        await loop.run_in_executor(None, dist.barrier)
        for c in clients.values():
            await c.aclose()
        await loop.run_in_executor(None, dist.barrier)
        await server.aclose()

    runner()(main())
    sw.shutdown()


# ----------------------------------------------------------------------------------------- configs 1 + 2 (latency)
def mode_pingpong(args):
    """Round-trip latency: config 1 (4 B host NumPy buffers, tag=1 tag_mask=0xFFFF) and config 2
    (one 1 MiB device buffer), reference scenario shape `pingpong-flag` (scenarios.py:238-266).
    world 1: Server+Client in one process on one GPU; world 2: rank 0 client <-> rank 1 server."""
    import numpy as np

    torch, sw, dist, rank, world, local = setup()
    assert world in (1, 2)
    dev = torch.device("cuda", local)

    async def main():
        server = sw.Server()
        addr = server.listen_address()
        addrs = [addr]
        if dist:
            addrs = [None] * world
            dist.all_gather_object(addrs, addr)
        client = sw.Client()
        await client.aconnect_address(addrs[(rank + 1) % world])
        for _ in range(2000):
            if server.list_clients():
                break
            await asyncio.sleep(0.005)
        ep = next(iter(server.list_clients()))
        cases = [("config1: 4 B host NumPy", 4, "host", 100, 1000), ("64 B device", 64, "dev", 100, 1000),
                 ("8 KiB device (eager max)", 8128, "dev", 50, 500), ("config2: 1 MiB device", 1 << 20, "dev", 20, 200),
                 ("64 MiB device", 64 << 20, "dev", 5, 30)]
        for name, n, where, warm, iters in cases:
            if where == "host":
                mk = lambda: np.arange(n, dtype=np.uint8)  # noqa: E731
            else:
                mk = lambda: torch.arange(n, dtype=torch.uint8, device=dev) if n <= 256 else torch.ones(n, dtype=torch.uint8, device=dev)  # noqa: E731
            ping, pong, rping, rpong = mk(), mk(), mk(), mk()
            if where == "dev":
                torch.cuda.synchronize()
            if dist:
                await asyncio.get_running_loop().run_in_executor(None, dist.barrier)
            samples = []
            for i in range(warm + iters):
                t0 = time.perf_counter()
                if world == 1:
                    f = server.arecv(rping, 1, 0xFFFF)
                    await client.asend(ping, 1)
                    await f
                    f = client.arecv(rpong, 2, 0xFFFF)
                    await server.asend(ep, pong, 2)
                    await f
                elif rank == 0:
                    f = client.arecv(rpong, 2, 0xFFFF)
                    await client.asend(ping, 1)
                    await f
                else:
                    await server.arecv(rping, 1, 0xFFFF)
                    await server.asend(ep, pong, 2)
                if i >= warm:
                    samples.append(time.perf_counter() - t0)
            if rank == 0:
                samples.sort()
                med = samples[len(samples) // 2]
                emit(args, {"scenario": "pingpong", "case": name, "n_gpus": world, "msg_bytes": n, "buffers": where,
                            "rtt_us_median": round(med * 1e6, 2), "rtt_us_p10": round(samples[len(samples) // 10] * 1e6, 2),
                            "one_way_us": round(med * 5e5, 2), "iters": iters,
                            "gbs_one_way": round(n / (med / 2) / 1e9, 3)})
        if dist:
            await asyncio.get_running_loop().run_in_executor(None, dist.barrier)
        await client.aclose()
        if dist:
            await asyncio.get_running_loop().run_in_executor(None, dist.barrier)
        await server.aclose()

    runner()(main())
    sw.shutdown()
    if rank == 0:
        # the restated reference on host cores, same shape (config 1 is the reference's own CPU-runnable case)
        from oracle import starway_cpu as cpu

        async def cpu_main():
            port = 45000 + os.getpid() % 10000
            s, c = cpu.make_pair(port)
            await c.aconnect("127.0.0.1", port)
            for n, warm, iters in ((4, 100, 1000), (1 << 20, 20, 200)):
                a, b, ra, rb = (np.arange(n, dtype=np.uint8) for _ in range(4))
                samples = []
                for i in range(warm + iters):
                    t0 = time.perf_counter()
                    f = s.arecv(ra, 1, 0xFFFF)
                    await c.asend(a, 1)
                    await f
                    f = c.arecv(rb, 2, 0xFFFF)
                    await s.asend(0, b, 2)
                    await f
                    if i >= warm:
                        samples.append(time.perf_counter() - t0)
                samples.sort()
                med = samples[len(samples) // 2]
                emit(args, {"scenario": "pingpong", "impl": "cpu_baseline (restated reference, oracle/cpu_engine.cpp)",
                            "msg_bytes": n, "buffers": "host", "rtt_us_median": round(med * 1e6, 2),
                            "one_way_us": round(med * 5e5, 2), "cores": 3, "host_cpus": len(os.sched_getaffinity(0))})
            await c.aclose()
            await s.aclose()

        runner()(cpu_main())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=["sweep", "allpairs", "storm", "pingpong"])
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-bytes", type=int, default=0)
    ap.add_argument("--msg-bytes", type=int, default=0)
    ap.add_argument("--rounds", type=int, default=50)
    ap.add_argument("--total-msgs", type=int, default=1_000_000)
    args = ap.parse_args()
    {"sweep": mode_sweep, "allpairs": mode_allpairs, "storm": mode_storm, "pingpong": mode_pingpong}[args.mode](args)


if __name__ == "__main__":
    main()
