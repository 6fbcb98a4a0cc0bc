"""starway_b200 — Hopper-native (H100, sm_90a) tagged point-to-point messaging.

Drop-in for the reference package's public surface (reference
``src/starway/__init__.py:351-358``): ``Server``, ``Client``, ``ServerEndpoint``.
The hot path under it is hand-written sm_90a CUDA reached through the C ABI in
``include/starway_b200.h``; there is NO CPU fallback: if ``libstarway_b200.so``
is missing this import fails, and if no CUDA device is visible the first
``Server()`` / ``Client()`` raises.
"""
from __future__ import annotations

import ctypes
import os
import sys

from . import _core

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libstarway_b200.so")


def _load() -> ctypes.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `make lib` (or `python -c 'import __graft_entry__ as g; g.build()'`). "
            "starway_b200 has no CPU fallback."
        )
    return ctypes.CDLL(LIB_PATH)


def _default_device() -> int:
    for key in ("STARWAY_DEVICE", "LOCAL_RANK"):
        v = os.environ.get(key)
        if v is not None and v.strip().lstrip("-").isdigit():
            n = _api.device_count()
            return int(v) % n if n > 0 else int(v)
    torch = sys.modules.get("torch")
    if torch is not None:
        try:
            if torch.cuda.is_available():
                return int(torch.cuda.current_device())
        except Exception:
            pass
    return 0


_api = _core.bind(_load(), _default_device)

Context = _api.Context
Server = _api.Server
Client = _api.Client
ServerEndpoint = _api.ServerEndpoint
get_context = _api.get_context
shutdown = _api.shutdown
status_string = _api.status_string
backend_name = _api.backend_name
device_count = _api.device_count
local_cpus = _api.local_cpus
bind_to_device_numa = _api.bind_to_device_numa


def check_sys_libs() -> str:
    """Reference ``check_sys_libs`` reports which libucx was loaded; here: the CUDA backend."""
    return backend_name()


__all__ = [
    "Server",
    "Client",
    "ServerEndpoint",
    "Context",
    "check_sys_libs",
    "get_context",
    "shutdown",
    "local_cpus",
    "bind_to_device_numa",
    "status_string",
    "backend_name",
    "device_count",
]
