#!/usr/bin/env python
"""Vote requests at a leader (raftgpu_leader_vote_request_wire[_device]): 1M leader groups x 5 voters at term 7, three
bursts of shuffled frames:
  - late: the losing candidates' MsgRequestVote at the winner's own term, one per leader plus a second for half of
    them, all rejected with the leader's commit info;
  - pre-vote: a healed partition's MsgRequestPreVote at term 8 to every leader, half of them in lease (IGNORED), the
    others granted or rejected at an unchanged term;
  - vote: MsgRequestVote at term 8 to a third of the leaders, out of lease: each deposes its leader (become_follower's
    arena reset) and is granted or rejected at term 8.

Each pass runs on reloaded state (a SET_TERM + RESET + BECOME_LEADER control list, outside the timed region), `runs`
passes after two warm-up passes, between CUDA events; then the host form end to end (its 64 B x groups voter table
crosses PCIe on every call) and the batch oracle (oracle/leader_vote_request_oracle.c) on one host core.  The device
result is checked against the batch oracle at full size.  Prints the GPU's name and power limit read in the same run.

    python scripts/micro_leader_vote_request.py [--groups N] [--runs K]
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
from oracle import leader_vote_request_oracle as LV  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--groups", type=int, default=1_000_000)
p.add_argument("--runs", type=int, default=20)
args = p.parse_args()
n, runs = args.groups, args.runs
rng = np.random.default_rng(0x7604)

ar = B.Arena(n)   # RaftGpuError(ERR_NO_DEVICE) without a GPU: no fallback
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(ar.info.device)],
                     capture_output=True, text=True).stdout.strip()
ar.group_alloc_range(n)
g = np.arange(n, dtype=np.uint32)
last = rng.integers(10, 1 << 30, n).astype(np.uint64)
com = last - rng.integers(0, 10, n).astype(np.uint64)
setup = np.zeros(4 * n, B.CTL_CMD_DTYPE)
setup["group"] = np.tile(g, 4)
setup["op"][:n], setup["a"][:n, 0], setup["a"][:n, 3] = B.CTL_SET_CONF, 0x1F, last + 1
setup["op"][n:2 * n], setup["a"][n:2 * n, 0] = B.CTL_SET_TERM, 7
setup["op"][2 * n:3 * n] = B.CTL_RESET
setup["a"][2 * n:3 * n] = np.stack([last + 1, last, com, last], 1)
setup["op"][3 * n:] = B.CTL_BECOME_LEADER
restore = np.ascontiguousarray(setup[n:])
assert np.all(ar.control(setup)["status"] == 0)
c0 = O.new_columns(n, n)
c0.term_start[:] = B.NO_TERM_START
v0 = np.zeros((O.SLOTS, n), np.uint8)
CO.arena_control(c0, v0, setup)
li = c0.last_index[:n].copy()   # the leader's empty entry at term_start

table = np.zeros(n, B.VOTER_DTYPE)
table["id"], table["vote"], table["last_term"], table["persisted"], table["commit_term"] = 1, 1, 7, last, 7
table["flags"] = B.VOTER_LEADER
lease = table.copy()
lease["flags"][rng.random(n) < 0.5] |= B.VOTER_LEASE


def requests(gs, typ, term):
    """Shuffled requests to groups gs from candidates 2-5 whose log is the leader's or one entry short."""
    e = np.zeros(len(gs), B.SYNTH_VOTE_REQUEST_DTYPE)
    e["hdr"], e["msg_type"], e["to"], e["from"] = gs << 4 | 1, typ, 1, rng.integers(2, 6, len(gs))
    e["term"], e["log_term"], e["index"] = term, 7, li[gs] - rng.integers(0, 2, len(gs)).astype(np.uint64)
    return B.synth_encode_vote_requests(e[rng.permutation(len(e))])


bursts = (("late", requests(np.concatenate([g, np.flatnonzero(rng.random(n) < 0.5).astype(np.uint32)]), 5, 7), table),
          ("pre-vote", requests(g, 17, 8), lease),
          ("vote", requests(np.flatnonzero(rng.random(n) < 1 / 3).astype(np.uint32), 5, 8), table))

L, h = ar._L, ar._h
stream = torch.cuda.Stream()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
nmax = max(len(off) for _, (_, off), _ in bursts) - 1
bmax = max(len(blob) for _, (blob, _), _ in bursts)
bound = B.vote_request_wire_bound(nmax)
sizes = (bmax + 16, 4 * (nmax + 1), table.nbytes, nmax, 16 * nmax, bound, 4 * (nmax + 1), 16)
bufs = [ar.device_alloc(x) for x in sizes]
d_b, d_o, d_v, d_st, d_out, d_rb, d_ro, d_t = bufs


def timed(nb, nf):
    t = []
    for k in range(runs + 2):   # the first two runs warm up
        ar.control(restore)
        ar.synchronize()
        ev0.record(stream)
        rc = L.raftgpu_leader_vote_request_wire_device(h, stream.cuda_stream, d_b, nb, d_o, nf, d_v, d_st, d_out, d_rb,
                                                       bound, d_ro, d_t)
        ev1.record(stream)
        assert rc == B.OK, rc
        stream.synchronize()
        if k >= 2:
            t.append(ev0.elapsed_time(ev1) * 1e-3)
    return t


def us(t):
    a = np.array(t) * 1e6
    return f"{np.median(a):.1f} us (range {a.min():.1f}-{a.max():.1f})"


print(f"GPU: {gpu}")
print(f"{n} leader groups x 5 voters at term 7; {runs} runs")
for name, (blob, off), tab in bursts:
    nf, nb = len(off) - 1, int(off[-1])
    ar.h2d(d_b, blob)
    ar.h2d(d_o, off)
    ar.h2d(d_v, tab)
    t_dev = timed(nb, nf)
    tot = np.zeros(2, np.uint64)
    ar.d2h(tot, d_t)
    st, out = np.zeros(nf, np.uint8), np.zeros((nf, 2), np.uint64)
    rb, ro = np.zeros(int(tot[1]), np.uint8), np.zeros(int(tot[0]) + 1, np.uint32)
    for arr, ptr in ((st, d_st), (out, d_out), (rb, d_rb), (ro, d_ro)):
        if arr.size:
            ar.d2h(arr, ptr)
    c, v = O.copy_columns(c0), v0.copy()
    want = LV.batch(c, None, v, blob, off, tab, bench=True, n_bytes=nb)
    for w, x, what in zip(want, (st, out, rb, ro, tot), ("status", "out", "bytes", "offsets", "totals")):
        assert np.array_equal(w, x), (name, what)
    assert np.array_equal(ar.column_read(B.COL_TERM, 0, 0, n, np.uint64), c.term[:n])
    cols = ar.read_columns(n)
    for col in ("term_start", "committed", "last_index", "matched", "next_idx", "peer_committed", "pflags"):
        assert np.array_equal(getattr(cols, col), getattr(c, col)[..., :n]), (name, col)
    kinds = np.bincount(st >> 4, minlength=16)
    print(f"{name}: {nf} frames, {nb} bytes; {int(kinds[B.WIRE_OK])} OK ({np.count_nonzero(st & B.VREQ_GRANTED)} granted, "
          f"{np.count_nonzero(st & B.VREQ_BUMPED)} bumped), {int(kinds[B.WIRE_IGNORED])} IGNORED, "
          f"{int(kinds[B.WIRE_DUP])} DUP; {int(tot[0])} responses, {int(tot[1])} bytes")
    print(f"  raftgpu_leader_vote_request_wire_device: {us(t_dev)}")
    fr = type("Frames", (), {"bytes": blob, "n_bytes": nb, "offsets": off, "n": nf})
    t_host = []
    for k in range(min(runs, 5) + 1):
        ar.control(restore)
        t0 = time.perf_counter()
        hres = ar.leader_vote_request_wire(fr, tab)
        t1 = time.perf_counter()
        if k >= 1:
            t_host.append(t1 - t0)
    assert all(np.array_equal(x, y) for x, y in zip(hres, want[:5])), "the host form differs from the oracle"
    print(f"  raftgpu_leader_vote_request_wire (host form, end to end, {min(runs, 5)} runs): {us(t_host)}")
    print(f"  batch oracle, one host core: {want[-1] * 1e6:.1f} us")
print("the pass matches the batch oracle at full size in every burst: status, out, responses, offsets and the columns")
for ptr in bufs:
    ar.device_free(ptr)
ar.close()
