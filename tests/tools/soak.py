"""Leak / stability soak: repeated listen / connect / mixed traffic / close cycles.
  python tests/tools/soak.py sim 200      CPU host-logic simulator
  python tests/tools/soak.py cuda 200     CUDA device (prints device memory in use)
Reports file descriptors, POSIX-shm segments, resident set and (cuda) device memory per 50 cycles;
all of them must stay flat."""
import asyncio
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from tests.cases_basic import load_api  # noqa: E402

backend = sys.argv[1] if len(sys.argv) > 1 else "sim"
cycles = int(sys.argv[2]) if len(sys.argv) > 2 else 200
api = load_api(backend)


def snapshot():
    fds = len(os.listdir("/proc/self/fd"))
    shm = len([f for f in os.listdir("/dev/shm") if f.startswith(("swsim", "swb200"))])
    rss = int(open("/proc/self/statm").read().split()[1]) * 4096 >> 20
    dev = None
    if backend == "cuda":
        import torch

        free, total = torch.cuda.mem_get_info()
        dev = (total - free) >> 20
    return fds, shm, rss, dev


async def main():
    hist = []
    dev_bufs = None
    if backend == "cuda":
        import torch

        dev_bufs = (torch.ones(300000, dtype=torch.uint8, device="cuda"), torch.zeros(300000, dtype=torch.uint8, device="cuda"))
        torch.cuda.synchronize()
    sim_dev = None
    if backend == "sim":
        from tests.hostsim import SimDev as sim_dev
    for cyc in range(cycles):
        server = api.Server()
        addr = server.listen_address()
        clients = [api.Client() for _ in range(3)]
        for c in clients:
            await c.aconnect_address(addr)
        buf = np.zeros(100000, dtype=np.uint8)
        futs = [server.arecv(buf, 0, 0) for _ in clients]
        for i, c in enumerate(clients):
            await c.asend(np.ones(50000 if i else 10, dtype=np.uint8), i)
        for f in futs:
            await f
        if dev_bufs is not None:
            f = server.arecv(dev_bufs[1], 7, 0xFFFF)
            await clients[0].asend(dev_bufs[0], 7)
            await f
        if sim_dev is not None:  # fresh 'device' allocations every cycle: handle / mapping caches must not grow
            a, b = sim_dev.from_np(np.ones(300000, dtype=np.uint8)), sim_dev.alloc(300000)
            f = server.arecv(b, 7, 0xFFFF)
            await clients[0].asend(a, 7)
            await f
            assert (sim_dev.to_np(b) == 1).all()
            del a, b
        for c in clients:
            await c.aclose()
        await server.aclose()
        del server, clients
        if cyc % 50 == 49:
            s = snapshot()
            hist.append(s)
            print(f"cycle {cyc + 1}: fds={s[0]} shm={s[1]} rss={s[2]} MiB dev={s[3]} MiB", flush=True)
    if len(hist) >= 3:
        assert hist[-1][0] <= hist[1][0] + 2, "file descriptors leak"
        assert hist[-1][1] <= hist[1][1] + 2, "shm segments leak"
        if hist[-1][3] is not None:
            assert hist[-1][3] <= hist[1][3] + 64, "device memory leak"
        if len(hist) >= 6:  # pools, caches and malloc arenas fill up during the first 150-200 cycles
            assert hist[-1][2] <= hist[3][2] + 16, "resident set grows (records of closed workers / endpoints must be recycled)"
    print("SOAK OK")


asyncio.run(main())
api.shutdown()
