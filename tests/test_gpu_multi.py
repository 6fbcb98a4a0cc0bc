"""Multi-GPU parity (one process per GPU, NVLink peer path): BASELINE configs 2-5 at test size, every
received byte and every (sender_tag, length) checked against the CPU oracle (tests/multi_gpu_worker.py).

Skipped when the machine has fewer GPUs than the test's world size: a 2-GPU machine runs the world-2 case,
an 8-GPU machine worlds 2, 4 and 8."""
import multiprocessing as mp
import queue as queue_mod

import pytest

from tests.conftest import free_port
from tests.multi_gpu_worker import rank_main

pytestmark = pytest.mark.gpu

ALL = ("s2", "s3", "s4", "s5")


def run_world(world, scenarios, backend="cuda", scale=1.0, timeout=1700):
    ctx = mp.get_context("spawn")
    barrier, q = ctx.Barrier(world), ctx.Queue()
    base_port = free_port()
    procs = [ctx.Process(target=rank_main, args=(r, world, base_port, barrier, q, scenarios, backend, scale)) for r in range(world)]
    for p in procs:
        p.start()
    results = {}
    try:
        for _ in range(world):
            try:
                rank, status, detail = q.get(timeout=timeout)
            except queue_mod.Empty:
                break
            results[rank] = (status, detail)
    finally:
        for p in procs:
            p.join(20)
            if p.is_alive():
                p.kill()
                p.join()
    errors = {r: d for r, (s, d) in results.items() if s != "ok"}
    missing = [r for r in range(world) if r not in results]
    assert not errors and not missing, "\n".join([f"--- rank {r} ---\n{d}" for r, d in sorted(errors.items())] +
                                                 [f"no result from ranks {missing}"] * bool(missing))
    return {r: d for r, (s, d) in results.items()}


@pytest.mark.parametrize("world", [2, 4, 8])
def test_configs_2_to_5_vs_oracle(world):
    import torch

    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    stats = run_world(world, ALL)
    for r, st in stats.items():
        # the product kernels moved the data: eager puts, device matching and rendezvous pulls on every rank
        assert st["put_msgs"] > 0 and st["match_arrivals"] > 0 and st["bulk_bytes"] > 0, (r, st)
