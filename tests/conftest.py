import os
import random
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with `-m gpu`)")
    # the native pieces are built in-tree by `make` (== __graft_entry__.build()); build them on demand
    needed = ["starway_b200/libstarway_b200.so", "starway_b200/_fastpath.so", "oracle/liboracle_tagmatch.so",
              "oracle/libstarway_cpu.so", "tests/hostsim/libstarway_hostsim.so"]
    if any(not os.path.exists(os.path.join(ROOT, p)) for p in needed):
        import subprocess

        subprocess.check_call(["make", "-C", ROOT, "-j", "8", "lib", "oracle", "hostsim"])


def free_port():
    # reference tests/test_basic.py:18-20 draws random.randint(10000, 50000); that collides now and then
    # with a live socket ("Address already in use"), so ask the kernel for a port that is free right now
    import socket

    for _ in range(20):
        cand = random.randint(10000, 30000)  # below the ephemeral range (32768+): no outgoing socket lands here
        with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
            try:
                s.bind(("127.0.0.1", cand))
                return cand
            except OSError:
                continue
    return random.randint(10000, 30000)


@pytest.fixture
def port():
    return free_port()


@pytest.fixture(scope="session")
def sim_api():
    """API classes bound to the host-logic simulator (CPU, test-only)."""
    from tests.hostsim import load

    api = load()
    yield api
    api.shutdown()


@pytest.fixture(scope="session")
def cuda_api():
    """API classes bound to the product library (CUDA, sm_90a)."""
    import types

    import starway_b200 as sw

    api = types.SimpleNamespace(
        Server=sw.Server,
        Client=sw.Client,
        ServerEndpoint=sw.ServerEndpoint,
        get_context=sw.get_context,
        shutdown=sw.shutdown,
        backend_name=sw.backend_name,
        local_cpus=sw.local_cpus,
        bind_to_device_numa=sw.bind_to_device_numa,
    )
    yield api
    sw.shutdown()


def _sweep_stale_shm():
    """Tests kill peer processes on purpose (dead-peer paths); a killed process cannot unlink the POSIX
    shared-memory segments it created (hostsim 'device memory', control blocks).  Remove the ones whose
    creating pid no longer exists, so that repeated runs do not fill /dev/shm."""
    try:
        names = os.listdir("/dev/shm")
    except OSError:
        return
    for name in names:
        if not name.startswith(("swsim-", "swb200-")):
            continue
        try:
            pid = int(name.split("-")[1])
        except (IndexError, ValueError):
            continue
        if pid == os.getpid() or os.path.exists(f"/proc/{pid}"):
            continue
        try:
            os.unlink(os.path.join("/dev/shm", name))
        except OSError:
            pass


def pytest_sessionstart(session):
    _sweep_stale_shm()


def pytest_sessionfinish(session, exitstatus):
    _sweep_stale_shm()
