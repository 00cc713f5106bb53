"""ctypes front-end of the control plane's oracle (oracle/control_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  control_oracle.c is compiled together with raft_oracle.c into its own
library, libcontrol_oracle.so: next to the sources when that directory is writable, else in a per-user temporary
directory.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SOURCES = ("control_oracle.c", "raft_oracle.c")
_HEADERS = ("control_oracle.h", "raft_oracle.h")
CFLAGS = ["-O3", "-march=x86-64-v3", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-pthread"]

CTL_CMD_DTYPE = np.dtype([("group", "<u4"), ("op", "u1"), ("peer_slot", "u1"), ("arg", "<u2"), ("a", "<u8", (4,))])
CTL_RESULT_DTYPE = np.dtype([("status", "<i4"), ("value", "<i4")])


def build(force: bool = False) -> str:
    """Compile libcontrol_oracle.so when it is missing or older than its sources; returns its path."""
    out_dir = _HERE if os.access(_HERE, os.W_OK) else os.path.join(tempfile.gettempdir(), f"control_oracle_{os.getuid()}")
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "libcontrol_oracle.so")
    newest = max(os.path.getmtime(os.path.join(_HERE, f)) for f in _SOURCES + _HEADERS)
    if force or not os.path.exists(path) or os.path.getmtime(path) < newest:
        tmp = f"{path}.{os.getpid()}"
        subprocess.run([os.environ.get("CC", "gcc"), *CFLAGS, "-shared", "-o", tmp,
                        *[os.path.join(_HERE, f) for f in _SOURCES]], check=True)
        os.replace(tmp, path)
    return path


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.ro_arena_control.argtypes = [C.POINTER(O.ArenaView), C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        L.ro_arena_control.restype = None
        _lib = L
    return _lib


def arena_control(c, votes: np.ndarray, cmds: np.ndarray) -> np.ndarray:
    """Every control command in list order (ro_arena_control); groups [0, c.n_groups) are the allocated ones.
    `votes` ([SLOTS][cap] u8) is updated in place.  Returns the {status, value} results."""
    assert votes.dtype == np.uint8 and votes.shape == (O.SLOTS, c.cap) and votes.flags.c_contiguous
    assert cmds.dtype.itemsize == CTL_CMD_DTYPE.itemsize and cmds.flags.c_contiguous
    res = np.zeros(len(cmds), dtype=CTL_RESULT_DTYPE)
    v = O.view(c)
    lib().ro_arena_control(C.byref(v), votes.ctypes.data, cmds.ctypes.data, len(cmds), res.ctypes.data)
    return res
