"""ctypes front-end of the control plane's oracle (oracle/control_oracle.c).

TEST INFRASTRUCTURE ONLY, like oracle.py.  control_oracle.c is part of libraft_oracle.so; lib() declares its functions
on oracle.lib().
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import oracle as O

CTL_CMD_DTYPE = np.dtype([("group", "<u4"), ("op", "u1"), ("peer_slot", "u1"), ("arg", "<u2"), ("a", "<u8", (4,))])
CTL_RESULT_DTYPE = np.dtype([("status", "<i4"), ("value", "<i4")])


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = O.lib()
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
