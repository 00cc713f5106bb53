#!/usr/bin/env python
"""The term prefix at a follower (raftgpu_follower_term_wire[_device]) after a store restarts: 1M follower groups x 5
voters at term 7; one MsgHeartbeat per group, at term 8 for one group in three (its leader was elected while the store
was down) and at term 7 for the rest, plus 5% stale heartbeats at term 6 from deposed leaders, shuffled.  Every group
checks the quorum, so each stale frame is answered.

Each pass runs on reloaded state (a SET_TERM + RESET control list, outside the timed region), 20 passes after two
warm-up passes, between CUDA events:
  - this pass alone;
  - this pass followed by raftgpu_follower_heartbeat_device, against raftgpu_follower_heartbeat_device alone on the same
    batch (which hands every frame at term 8 and 6 back as TERM);
  - the host form end to end (its 64 B x groups voter table crosses PCIe on every call);
  - the batch oracle (oracle/follow_term_oracle.c) on one host core.
The device result is checked against the batch oracle at full size.  Prints the GPU's name and power limit read in
the same run.

    python scripts/micro_follower_term.py [--groups N] [--runs K]
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
from oracle import follow_term_oracle as FT  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--groups", type=int, default=1_000_000)
p.add_argument("--runs", type=int, default=20)
args = p.parse_args()
n, runs = args.groups, args.runs
rng = np.random.default_rng(0x7404)

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
setup["op"][n:2 * n] = B.CTL_RESET
setup["a"][n:2 * n] = np.stack([np.full(n, B.NO_TERM_START, np.uint64), last, com, last], 1)
setup["op"][2 * n:], setup["a"][2 * n:, 0] = B.CTL_SET_TERM, 7
restore = np.ascontiguousarray(np.concatenate([setup[2 * n:], setup[n:2 * n]]))
assert np.all(ar.control(setup)["status"] == 0)
c0 = O.new_columns(n, n)
c0.term_start[:] = B.NO_TERM_START
v0 = np.zeros((O.SLOTS, n), np.uint8)
CO.arena_control(c0, v0, setup)

table = np.zeros(n, B.VOTER_DTYPE)
table["id"], table["last_term"], table["persisted"] = 1, 7, last
table["flags"] = B.VOTER_SELECT | B.VOTER_STALE_REPLY
ids = np.ones(n, np.uint64)
select = np.full((n + 31) // 32, 0xFFFFFFFF, np.uint32)

# the batch: MsgHeartbeat {to 1, from, term} at 12 bytes a frame
stale = np.flatnonzero(rng.random(n) < 0.05).astype(np.uint32)
gs = np.concatenate([g, stale])
nf = len(gs)
term = np.where(rng.random(n) < 1 / 3, 8, 7).astype(np.uint8)
terms = np.concatenate([term, np.full(len(stale), 6, np.uint8)])
order = rng.permutation(nf)
gs, terms = gs[order], terms[order]
rows = np.zeros((nf, 12), np.uint8)
rows[:, :4] = (gs << 4 | 1).astype("<u4").view(np.uint8).reshape(nf, 4)
rows[:, 4:] = [0x08, 8, 0x10, 1, 0x18, 0, 0x20, 0]
rows[:, 9] = np.where(terms == 6, 9, 2 + terms % 3)   # one `from` per term
rows[:, 11] = terms
blob = np.concatenate([rows.reshape(-1), np.zeros(16, np.uint8)])
off = (12 * np.arange(nf + 1)).astype(np.uint32)
n_bytes = 12 * nf

L, h = ar._L, ar._h
stream = torch.cuda.Stream()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
bound, hb_bound = B.follower_term_wire_bound(nf), B.follower_heartbeat_bound(nf)
sizes = (len(blob), 4 * (nf + 1), table.nbytes, nf, 16 * nf, bound, 4 * (nf + 1), 16, select.nbytes, 8 * n, nf, 8 * nf,
         hb_bound, 4 * (nf + 1), 16)
bufs = [ar.device_alloc(x) for x in sizes]
d_b, d_o, d_v, d_st, d_out, d_rb, d_ro, d_t, d_sel, d_ids, d_hst, d_from, d_hrb, d_hro, d_ht = bufs
for ptr, x in ((d_b, blob), (d_o, off), (d_v, table), (d_sel, select), (d_ids, ids)):
    ar.h2d(ptr, x)


def term_pass():
    rc = L.raftgpu_follower_term_wire_device(h, stream.cuda_stream, d_b, n_bytes, d_o, nf, d_v, d_st, d_out, d_rb, bound,
                                             d_ro, d_t)
    assert rc == B.OK, rc


def heartbeat_pass():
    rc = L.raftgpu_follower_heartbeat_device(h, stream.cuda_stream, d_b, n_bytes, d_o, nf, d_sel, d_ids, d_hst, d_from,
                                             d_hrb, hb_bound, d_hro, d_ht)
    assert rc == B.OK, rc


def timed(*passes):
    t = []
    for k in range(runs + 2):   # the first two runs warm up
        ar.control(restore)
        ar.synchronize()
        ev0.record(stream)
        for f in passes:
            f()
        ev1.record(stream)
        stream.synchronize()
        if k >= 2:
            t.append(ev0.elapsed_time(ev1) * 1e-3)
    return t


def us(t):
    a = np.array(t) * 1e6
    return f"{np.median(a):.1f} us (range {a.min():.1f}-{a.max():.1f})"


print(f"GPU: {gpu}")
t_term = timed(term_pass)
tot = np.zeros(2, np.uint64)
ar.d2h(tot, d_t)
st, out = np.zeros(nf, np.uint8), np.zeros((nf, 2), np.uint64)
rb, ro = np.zeros(int(tot[1]), np.uint8), np.zeros(int(tot[0]) + 1, np.uint32)
for arr, ptr in ((st, d_st), (out, d_out), (rb, d_rb), (ro, d_ro)):
    ar.d2h(arr, ptr)
c, v = O.copy_columns(c0), v0.copy()
want = FT.batch(c, None, v, blob[:n_bytes], off, table, bench=True)
for w, x, name in zip(want, (st, out, rb, ro, tot), ("status", "out", "bytes", "offsets", "totals")):
    assert np.array_equal(w, x), name
assert np.array_equal(ar.column_read(B.COL_TERM, 0, 0, n, np.uint64), c.term[:n])
cols = ar.read_columns(n)
for name in ("term_start", "committed", "last_index", "matched", "next_idx", "peer_committed", "pflags"):
    assert np.array_equal(getattr(cols, name), getattr(c, name)[..., :n]), name
kinds = np.bincount(st >> 4, minlength=16)
print(f"{n} follower groups x 5 voters at term 7, {nf} heartbeats ({np.count_nonzero(terms == 8)} at term 8, "
      f"{len(stale)} stale at term 6), 12 bytes a frame; {runs} runs")
print(f"verdicts: {int(kinds[B.WIRE_OK])} OK ({np.count_nonzero(st & B.FTERM_BUMPED)} bumped), "
      f"{int(kinds[B.WIRE_STALE])} STALE ({int(tot[0])} replies, {int(tot[1])} bytes)")
print(f"  raftgpu_follower_term_wire_device alone: {us(t_term)}")
t_both = timed(term_pass, heartbeat_pass)
hst = np.zeros(nf, np.uint8)
ar.d2h(hst, d_hst)
print(f"  then raftgpu_follower_heartbeat_device: {us(t_both)}; heartbeats answered on the device: "
      f"{np.count_nonzero(hst & B.RES_OK)}")
t_hb = timed(heartbeat_pass)
ar.d2h(hst, d_hst)
print(f"  raftgpu_follower_heartbeat_device alone on the same batch: {us(t_hb)}; answered: "
      f"{np.count_nonzero(hst & B.RES_OK)}, TERM: {np.count_nonzero(hst >> 4 == B.WIRE_TERM)}")
fr = type("Frames", (), {"bytes": blob, "n_bytes": n_bytes, "offsets": off, "n": nf})
t_host = []
for k in range(min(runs, 5) + 1):
    ar.control(restore)
    t0 = time.perf_counter()
    hres = ar.follower_term_wire(fr, table)
    t1 = time.perf_counter()
    if k >= 1:
        t_host.append(t1 - t0)
assert all(np.array_equal(x, y) for x, y in zip(hres, want[:5])), "the host form differs from the oracle"
print(f"  raftgpu_follower_term_wire (host form, end to end, {min(runs, 5)} runs): {us(t_host)}")
print(f"  batch oracle, one host core: {want[-1] * 1e6:.1f} us")
print("the pass matches the batch oracle at full size: status, out, replies, offsets and the reset columns")
for ptr in bufs:
    ar.device_free(ptr)
ar.close()
