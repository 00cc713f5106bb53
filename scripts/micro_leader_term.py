#!/usr/bin/env python
"""The term prefix at a leader (raftgpu_leader_term_wire[_device]): 1M leader groups x 5 voters at term 7, two batches:
  - steady: one MsgAppendResponse per peer cell at the term (4M frames), what running the pass every tick costs: every
    frame is left to the wire step;
  - partition heal: one MsgAppendResponse at term 8 for a third of the leaders (a follower that campaigned while cut
    off), a late MsgRequestVoteResponse at term 7 for every leader, and a stale MsgHeartbeat at term 6 for 5% of them
    from deposed leaders, shuffled.  Every group checks the quorum, so each stale heartbeat is answered.

Each pass runs on reloaded state (a SET_TERM + RESET + BECOME_LEADER control list, outside the timed region), `runs`
passes after two warm-up passes, between CUDA events; then the host form end to end (its 64 B x groups voter table
crosses PCIe on every call) and the batch oracle (oracle/leader_term_oracle.c) on one host core.  The device result is
checked against the batch oracle at full size.  Prints the GPU's name and power limit read in the same run.

    python scripts/micro_leader_term.py [--groups N] [--runs K]
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
from oracle import leader_term_oracle as LT  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--groups", type=int, default=1_000_000)
p.add_argument("--runs", type=int, default=20)
args = p.parse_args()
n, runs = args.groups, args.runs
rng = np.random.default_rng(0x7504)

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

table = np.zeros(n, B.VOTER_DTYPE)
table["id"], table["last_term"], table["persisted"] = 1, 7, last
table["flags"] = B.VOTER_STALE_REPLY


def batch(hdr, typ, frm, term):
    """12-byte frames: the u32 header, then {msg_type, to 1, from, term}."""
    k = len(hdr)
    rows = np.zeros((k, 12), np.uint8)
    rows[:, :4] = hdr.astype("<u4").view(np.uint8).reshape(k, 4)
    rows[:, 4:] = [0x08, 0, 0x10, 1, 0x18, 0, 0x20, 0]
    rows[:, 5], rows[:, 9], rows[:, 11] = typ, frm, term
    return np.concatenate([rows.reshape(-1), np.zeros(16, np.uint8)]), (12 * np.arange(k + 1)).astype(np.uint32)


cells = np.repeat(g, 4), np.tile(np.arange(1, 5, dtype=np.uint32), n)
steady = batch(cells[0] << 4 | cells[1], 4, cells[1] + 1, 7)
up = np.flatnonzero(rng.random(n) < 1 / 3).astype(np.uint32)
stale = np.flatnonzero(rng.random(n) < 0.05).astype(np.uint32)
hdr = np.concatenate([up << 4 | 2, g << 4 | 3, stale << 4 | 1])
typ = np.concatenate([np.full(len(up), 4), np.full(n, 6), np.full(len(stale), 8)]).astype(np.uint8)
frm = np.concatenate([np.full(len(up), 3), np.full(n, 4), np.full(len(stale), 9)]).astype(np.uint8)
term = np.concatenate([np.full(len(up), 8), np.full(n, 7), np.full(len(stale), 6)]).astype(np.uint8)
order = rng.permutation(len(hdr))
heal = batch(hdr[order], typ[order], frm[order], term[order])

L, h = ar._L, ar._h
stream = torch.cuda.Stream()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
nmax = max(len(steady[1]), len(heal[1])) - 1
bound = B.follower_term_wire_bound(nmax)
sizes = (12 * nmax + 16, 4 * (nmax + 1), table.nbytes, nmax, 16 * nmax, bound, 4 * (nmax + 1), 16)
bufs = [ar.device_alloc(x) for x in sizes]
d_b, d_o, d_v, d_st, d_out, d_rb, d_ro, d_t = bufs
ar.h2d(d_v, table)


def timed(nf):
    def run():
        rc = L.raftgpu_leader_term_wire_device(h, stream.cuda_stream, d_b, 12 * nf, d_o, nf, d_v, d_st, d_out, d_rb,
                                               bound, d_ro, d_t)
        assert rc == B.OK, rc
    t = []
    for k in range(runs + 2):   # the first two runs warm up
        ar.control(restore)
        ar.synchronize()
        ev0.record(stream)
        run()
        ev1.record(stream)
        stream.synchronize()
        if k >= 2:
            t.append(ev0.elapsed_time(ev1) * 1e-3)
    return t


def us(t):
    a = np.array(t) * 1e6
    return f"{np.median(a):.1f} us (range {a.min():.1f}-{a.max():.1f})"


print(f"GPU: {gpu}")
print(f"{n} leader groups x 5 voters at term 7, 12-byte frames; {runs} runs")
for name, (blob, off) in (("steady", steady), ("partition heal", heal)):
    nf = len(off) - 1
    ar.h2d(d_b, blob)
    ar.h2d(d_o, off)
    t_dev = timed(nf)
    tot = np.zeros(2, np.uint64)
    ar.d2h(tot, d_t)
    st, out = np.zeros(nf, np.uint8), np.zeros((nf, 2), np.uint64)
    rb, ro = np.zeros(int(tot[1]), np.uint8), np.zeros(int(tot[0]) + 1, np.uint32)
    for arr, ptr in ((st, d_st), (out, d_out), (rb, d_rb), (ro, d_ro)):
        if arr.size:
            ar.d2h(arr, ptr)
    c, v = O.copy_columns(c0), v0.copy()
    want = LT.batch(c, None, v, blob[:12 * nf], off, table, bench=True)
    for w, x, what in zip(want, (st, out, rb, ro, tot), ("status", "out", "bytes", "offsets", "totals")):
        assert np.array_equal(w, x), (name, what)
    assert np.array_equal(ar.column_read(B.COL_TERM, 0, 0, n, np.uint64), c.term[:n])
    cols = ar.read_columns(n)
    for col in ("term_start", "committed", "last_index", "matched", "next_idx", "peer_committed", "pflags"):
        assert np.array_equal(getattr(cols, col), getattr(c, col)[..., :n]), (name, col)
    kinds = np.bincount(st >> 4, minlength=16)
    print(f"{name}: {nf} frames; {int(kinds[B.WIRE_OK])} OK ({np.count_nonzero(st & B.FTERM_BUMPED)} bumped), "
          f"{int(kinds[B.WIRE_IGNORED])} IGNORED, {int(kinds[B.WIRE_STALE])} STALE ({int(tot[0])} replies)")
    print(f"  raftgpu_leader_term_wire_device: {us(t_dev)}")
    fr = type("Frames", (), {"bytes": blob, "n_bytes": 12 * nf, "offsets": off, "n": nf})
    t_host = []
    for k in range(min(runs, 5) + 1):
        ar.control(restore)
        t0 = time.perf_counter()
        hres = ar.leader_term_wire(fr, table)
        t1 = time.perf_counter()
        if k >= 1:
            t_host.append(t1 - t0)
    assert all(np.array_equal(x, y) for x, y in zip(hres, want[:5])), "the host form differs from the oracle"
    print(f"  raftgpu_leader_term_wire (host form, end to end, {min(runs, 5)} runs): {us(t_host)}")
    print(f"  batch oracle, one host core: {want[-1] * 1e6:.1f} us")
print("the pass matches the batch oracle at full size in both cases: status, out, replies, offsets and the reset columns")
for ptr in bufs:
    ar.device_free(ptr)
ar.close()
