"""raft-rs_b200: H100-native batched commit-index engine for multi-raft.

The product is ``libraftgpu.so`` (hand-written sm_90a CUDA behind the C-ABI in
``include/raftgpu.h``) plus the C++ mirror of the raft-rs tracker surface in
``host/``.  This Python package is only the ctypes plumbing the tests and
``bench.py`` use; import it with ``importlib.import_module("raft-rs_b200")``.
"""
from .binding import *  # noqa: F401,F403
from . import binding  # noqa: F401
from . import wire  # noqa: F401
