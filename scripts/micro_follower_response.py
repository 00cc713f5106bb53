#!/usr/bin/env python
"""The responses that reach followers and candidates (raftgpu_follower_response_wire[_device]): a deposition burst of
about 1M frames over `groups` groups x 5 voters at term 7 (half Followers, a quarter each PreCandidates and Candidates),
`per` frames per group, shuffled:
  - the late MsgAppendResponse / MsgHeartbeatResponse frames of leaderships the groups lost, at term 7 (dropped);
  - late vote responses at term 6 (stale) and 7 (a candidate's own are left for raftgpu_vote_wire);
  - for a third of the groups one rejection at term 8 (become_follower: the claimant resets its group).

Each pass runs on reloaded state (a SET_TERM + RESET control list, outside the timed region), `runs` passes after two
warm-up passes, between CUDA events; then the host form end to end (its 64 B x groups voter table crosses PCIe on every
call) and the batch oracle (oracle/follow_resp_oracle.c) on one host core.  The device result is checked against the
batch oracle at full size.  Prints the GPU's name and power limit read in the same run.

    python scripts/micro_follower_response.py [--groups N] [--per K] [--runs R]
"""
import argparse
import importlib
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
B = importlib.import_module("raft-rs_b200").binding
from oracle import oracle as O  # noqa: E402
from oracle import control_oracle as CO  # noqa: E402
from oracle import follow_resp_oracle as FR  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--groups", type=int, default=250_000)
p.add_argument("--per", type=int, default=4)
p.add_argument("--runs", type=int, default=20)
args = p.parse_args()
n, per, runs = args.groups, args.per, args.runs
rng = np.random.default_rng(0x7750)

ar = B.Arena(n)   # RaftGpuError(ERR_NO_DEVICE) without a GPU: no fallback
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(ar.info.device)],
                     capture_output=True, text=True).stdout.strip()
ar.group_alloc_range(n)
g = np.arange(n, dtype=np.uint32)
last = rng.integers(10, 1 << 30, n).astype(np.uint64)
com = last - rng.integers(0, 10, n).astype(np.uint64)
setup = np.zeros(3 * n, B.CTL_CMD_DTYPE)
setup["group"] = np.tile(g, 3)
setup["op"][:n], setup["a"][:n, 0], setup["a"][:n, 3] = B.CTL_SET_CONF, 0x1F, last + 1
setup["op"][n:2 * n], setup["a"][n:2 * n, 0] = B.CTL_SET_TERM, 7
setup["op"][2 * n:] = B.CTL_RESET
setup["a"][2 * n:] = np.stack([np.full(n, B.NO_TERM_START, np.uint64), last, com, last], 1)
restore = np.ascontiguousarray(setup[n:])
assert np.all(ar.control(setup)["status"] == 0)
c0 = O.new_columns(n, n)
c0.term_start[:] = B.NO_TERM_START
v0 = np.zeros((O.SLOTS, n), np.uint8)
CO.arena_control(c0, v0, setup)

role = rng.choice(3, n, p=(0.5, 0.25, 0.25))   # Follower, PreCandidate, Candidate
table = np.zeros(n, B.VOTER_DTYPE)
table["id"], table["last_term"], table["persisted"] = 1, 7, last
table["flags"] = B.VOTER_SELECT | np.where(role == 1, B.VOTER_CANDIDATE | B.VOTER_PRE_CANDIDATE,
                                           np.where(role == 2, B.VOTER_CANDIDATE, 0))

# 12-byte frames: the u32 header, then {msg_type, to 1, from, term}; a rejection adds reject = true (2 bytes)
hdr = (np.repeat(g, per) << 4 | np.tile(np.arange(1, per + 1, dtype=np.uint32) % 5, n)).astype(np.uint32)
typ = rng.choice(np.array([4, 9, 6, 18], np.uint8), n * per)
term = rng.choice(np.array([6, 7, 7], np.uint8), n * per)
up = np.repeat(rng.random(n) < 1 / 3, per) & (np.tile(np.arange(per), n) == 0)
typ[up], term[up] = np.where(role[np.repeat(g, per)[up]] == 1, 18, 6), 8
k = n * per
rows = np.zeros((k, 14), np.uint8)
rows[:, :4] = hdr.astype("<u4").view(np.uint8).reshape(k, 4)
rows[:, 4:] = [0x08, 0, 0x10, 1, 0x18, 0, 0x20, 0, 0x50, 1]
rows[:, 5], rows[:, 9], rows[:, 11] = typ, (hdr & 15) + 1, term
size = np.where(up, 14, 12)
order = rng.permutation(k)
blob = np.concatenate([rows[order][np.arange(14)[None, :] < size[order][:, None]], np.zeros(16, np.uint8)])
off = np.concatenate([[0], np.cumsum(size[order])]).astype(np.uint32)
nb = int(off[-1])

L, h = ar._L, ar._h
stream = torch.cuda.Stream()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
bufs = [ar.device_alloc(x) for x in (len(blob), off.nbytes, table.nbytes, k, 8 * k)]
d_b, d_o, d_v, d_st, d_out = bufs
ar.h2d(d_b, blob)
ar.h2d(d_o, off)
ar.h2d(d_v, table)

t_dev = []
for r in range(runs + 2):   # the first two runs warm up
    ar.control(restore)
    ar.synchronize()
    ev0.record(stream)
    rc = L.raftgpu_follower_response_wire_device(h, stream.cuda_stream, d_b, nb, d_o, k, d_v, d_st, d_out)
    assert rc == B.OK, rc
    ev1.record(stream)
    stream.synchronize()
    if r >= 2:
        t_dev.append(ev0.elapsed_time(ev1) * 1e-3)
st, out = np.zeros(k, np.uint8), np.zeros(k, np.uint64)
ar.d2h(st, d_st)
ar.d2h(out, d_out)
c, v = O.copy_columns(c0), v0.copy()
want = FR.batch(c, None, v, blob[:nb], off, table, bench=True)
assert np.array_equal(want[0], st) and np.array_equal(want[1], out), "the device differs from the oracle"
assert np.array_equal(ar.column_read(B.COL_TERM, 0, 0, n, np.uint64), c.term[:n])
cols = ar.read_columns(n)
for col in ("term_start", "committed", "last_index", "matched", "next_idx", "peer_committed", "pflags"):
    assert np.array_equal(getattr(cols, col), getattr(c, col)[..., :n]), col


def us(t):
    a = np.array(t) * 1e6
    return f"{np.median(a):.1f} us (range {a.min():.1f}-{a.max():.1f})"


fr = type("Frames", (), {"bytes": blob, "n_bytes": nb, "offsets": off, "n": k})
t_host = []
for r in range(min(runs, 5) + 1):
    ar.control(restore)
    t0 = time.perf_counter()
    hres = ar.follower_response_wire(fr, table)
    t1 = time.perf_counter()
    if r >= 1:
        t_host.append(t1 - t0)
assert np.array_equal(hres[0], st) and np.array_equal(hres[1], out), "the host form differs from the oracle"
kinds = np.bincount(st >> 4, minlength=16)
print(f"GPU: {gpu}")
print(f"{n} groups x 5 voters at term 7 ({per} frames each), {k} frames of 12-14 bytes; {runs} runs")
print(f"  {int(kinds[B.WIRE_OK])} OK ({np.count_nonzero(st & B.FTERM_BUMPED)} bumped), {int(kinds[B.WIRE_IGNORED])} "
      f"IGNORED, {int(kinds[B.WIRE_STALE])} STALE")
print(f"  raftgpu_follower_response_wire_device: {us(t_dev)}")
print(f"  raftgpu_follower_response_wire (host form, end to end, {min(runs, 5)} runs): {us(t_host)}")
print(f"  batch oracle, one host core: {want[-1] * 1e6:.1f} us")
print("the pass matches the batch oracle at full size: status, out and the reset columns")
for ptr in bufs:
    ar.device_free(ptr)
ar.close()
