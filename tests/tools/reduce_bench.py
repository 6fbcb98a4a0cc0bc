"""Loopback measurement of arecv_reduce on one GPU, through the asyncio API.

Three arms run in the same process, alternating step by step, on the same seeded messages:
  (a) reduce:   arecv_reduce into the accumulators;
  (b) two_step: arecv into scratch tensors, synchronise, dst.add_(scratch), synchronise (what a caller writes today);
  (c) copy:     plain arecv into scratch tensors (the transfer alone).
One step = a window of --window messages posted, sent, received and synchronised.  Prints one JSON line per
(dtype, size) with message GB/s and microseconds per step (median over --steps), plus ping-pong round trips of
64 B and 8128 B for arecv_reduce next to arecv, and the card's name and power limit.

--profile: a separate run of arm (a) under torch.profiler; reports the time of the reduce kernels and, from it, the
achieved HBM rate as 3 N bytes per message (read src, read dst, write dst) over kernel time, against the H100 SXM
data-sheet 3.35 TB/s.  Keep it apart from the timed run: tracing slows the host.

  python tests/tools/reduce_bench.py [--sizes 65536,1048576,16777216,268435456] [--dtypes float32,bfloat16]
                                     [--steps 20] [--warmup 3] [--window 16] [--profile] [--out DIR]
"""
import argparse
import asyncio
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
os.environ.setdefault("STARWAY_QUIET", "1")

HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                      text=True, timeout=30)
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


async def setup(sw):
    server, client = sw.Server(), sw.Client()
    await client.aconnect_address(server.listen_address())
    for _ in range(400):
        if server.list_clients():
            break
        await asyncio.sleep(0.005)
    return server, client, next(iter(server.list_clients()))


async def step(torch, server, client, arm, srcs, dsts, scratch):
    if arm == "reduce":
        futs = [server.arecv_reduce(d, i, (1 << 64) - 1) for i, d in enumerate(dsts)]
    else:
        futs = [server.arecv(s, i, (1 << 64) - 1) for i, s in enumerate(scratch)]
    sends = [client.asend(s, i) for i, s in enumerate(srcs)]
    await asyncio.gather(*futs, *sends)
    torch.cuda.synchronize()
    if arm == "two_step":
        for d, s in zip(dsts, scratch):
            d.add_(s.view(d.dtype))
        torch.cuda.synchronize()


async def pingpong(torch, server, client, ep, n, reduce, iters):
    a = torch.zeros(n // 4, dtype=torch.float32, device="cuda")
    b = torch.zeros(n // 4, dtype=torch.float32, device="cuda")
    ab, bb = a.view(torch.uint8), b.view(torch.uint8)
    torch.cuda.synchronize()
    ts = []
    for k in range(iters):
        t0 = time.perf_counter()
        f1 = server.arecv_reduce(a, 1, (1 << 64) - 1) if reduce else server.arecv(ab, 1, (1 << 64) - 1)
        await client.asend(bb, 1)
        await f1
        f2 = client.arecv_reduce(b, 2, (1 << 64) - 1) if reduce else client.arecv(bb, 2, (1 << 64) - 1)
        await server.asend(ep, ab, 2)
        await f2
        ts.append(time.perf_counter() - t0)
    ts = ts[iters // 10:]
    return statistics.median(ts) * 1e6


async def main(args):
    import torch

    import starway_b200 as sw

    assert torch.cuda.is_available(), "reduce_bench measures on a GPU"
    server, client, ep = await setup(sw)
    results = []
    gen = torch.Generator(device="cuda").manual_seed(1)
    for name in args.dtypes.split(","):
        dt = getattr(torch, name)
        isz = torch.empty(0, dtype=dt).element_size()
        for size in (int(s) for s in args.sizes.split(",")):
            n = size // isz
            srcs = [torch.randn(n, generator=gen, device="cuda").to(dt) for _ in range(args.window)]
            dsts = [torch.zeros(n, device="cuda", dtype=dt) for _ in range(args.window)]
            scratch = [torch.empty(size, dtype=torch.uint8, device="cuda") for _ in range(args.window)]
            arms = ["reduce"] if args.profile else ["reduce", "two_step", "copy"]
            for _ in range(args.warmup):
                for arm in arms:
                    await step(torch, server, client, arm, srcs, dsts, scratch)
            rec = {"dtype": name, "size": size, "window": args.window, "steps": args.steps}
            if args.profile:
                from torch.profiler import ProfilerActivity, profile

                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.steps):
                        await step(torch, server, client, "reduce", srcs, dsts, scratch)
                    torch.cuda.synchronize()
                us = {"sw_reduce_tma_kernel": 0.0, "sw_reduce_simt_kernel": 0.0}
                launches = {k: 0 for k in us}
                for ev in prof.key_averages():
                    for k in us:
                        if k in ev.key:
                            us[k] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
                            launches[k] += ev.count
                kernel_s = sum(us.values()) * 1e-6
                hbm = 3.0 * size * args.window * args.steps
                rec.update({"kernel_us": {k: round(v, 1) for k, v in us.items()}, "launches": launches,
                            "kernel_us_per_step": round(sum(us.values()) / args.steps, 1),
                            "hbm_GBps": round(hbm / kernel_s / 1e9, 1) if kernel_s else None,
                            "hbm_share_of_3.35TBps": round(hbm / kernel_s / HBM_PEAK, 3) if kernel_s else None})
                if args.out:
                    prof.export_chrome_trace(os.path.join(args.out, f"reduce_{name}_{size}.pt.trace.json"))
            else:
                times = {arm: [] for arm in arms}
                for _ in range(args.steps):
                    for arm in arms:   # alternating: the arms see the same host noise
                        t0 = time.perf_counter()
                        await step(torch, server, client, arm, srcs, dsts, scratch)
                        times[arm].append(time.perf_counter() - t0)
                for arm in arms:
                    med = statistics.median(times[arm])
                    rec[arm] = {"us_per_step": round(med * 1e6, 1), "msg_GBps": round(size * args.window / med / 1e9, 1)}
            results.append(rec)
            print(json.dumps(rec), flush=True)
            del srcs, dsts, scratch
            torch.cuda.empty_cache()
    if not args.profile:
        rtt = {}
        for n in (64, 8128):
            for reduce in (False, True):
                await pingpong(torch, server, client, ep, n, reduce, 200)   # warm-up
                rtt[f"{'arecv_reduce' if reduce else 'arecv'}_{n}B_us"] = round(
                    await pingpong(torch, server, client, ep, n, reduce, args.rtt_iters), 1)
        print(json.dumps({"pingpong_rtt_median": rtt}), flush=True)
        results.append({"pingpong_rtt_median": rtt})
    await client.aclose()
    await server.aclose()
    info = {"card": card(), "profile": args.profile}
    print(json.dumps(info), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "reduce_bench_profile.json" if args.profile else "reduce_bench.json"), "w") as f:
            json.dump({"info": info, "results": results}, f, indent=1)
    sw.shutdown()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="65536,1048576,16777216,268435456")
    ap.add_argument("--dtypes", default="float32,bfloat16")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--window", type=int, default=16)
    ap.add_argument("--rtt-iters", type=int, default=2000)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    asyncio.run(main(a))
