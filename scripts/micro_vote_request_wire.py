#!/usr/bin/env python
"""Vote requests at a voter (raftgpu_vote_request_wire[_device]) in an election storm: 1M follower groups x 5 voters at
term 7, one candidate's request per group plus a second candidate's for one group in eight (the DUP path), shuffled.

  - The pre-vote round (MsgRequestPreVote at term 8) changes nothing the pass writes, so it is timed over 20 passes after
    two warm-up passes: the device form between CUDA events and from the call to the end of a synchronise, and the host
    form end to end (its 64 B x groups voter table crosses PCIe on every call).
  - The vote round (MsgRequestVote at term 8) bumps every term, so each pass runs on restored state: the restore (a
    SET_TERM + RESET control list) is outside the timed region.
  - The batch oracle (oracle/vote_request_oracle.c) on one host core is the CPU reference.

Both rounds are checked against the batch oracle at full size (status, out, response bytes and offsets, the arena
columns a reset touches).  Prints the GPU's name and power limit read in the same run.

    python scripts/micro_vote_request_wire.py [--groups N] [--runs K]
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
from oracle import vote_request_oracle as VR  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--groups", type=int, default=1_000_000)
p.add_argument("--runs", type=int, default=20)
args = p.parse_args()
n, runs = args.groups, args.runs
rng = np.random.default_rng(0x7202)

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
restore = np.ascontiguousarray(np.concatenate([setup[2 * n:], setup[n:2 * n]]))  # what every vote-round pass starts from
assert np.all(ar.control(setup)["status"] == 0)
c0 = O.new_columns(n, n)
c0.term_start[:] = B.NO_TERM_START
v0 = np.zeros((O.SLOTS, n), np.uint8)
CO.arena_control(c0, v0, setup)

table = np.zeros(n, B.VOTER_DTYPE)
table["id"], table["last_term"], table["commit_term"], table["persisted"] = 1, 7, 7, last
table["flags"] = B.VOTER_SELECT
second = np.flatnonzero(rng.random(n) < 0.125).astype(np.uint32)
gs = np.concatenate([g, second])
nf = len(gs)


def frames(typ):
    e = np.zeros(nf, B.SYNTH_VOTE_REQUEST_DTYPE)
    e["hdr"], e["msg_type"], e["to"], e["from"] = gs << 4 | 1, typ, 1, rng.integers(2, 6, nf)
    e["term"], e["log_term"], e["index"] = 8, 7, last[gs] + rng.integers(0, 2, nf).astype(np.uint64) - 1
    e["commit"], e["commit_term"] = com[gs], 7
    return B.synth_encode_vote_requests(e[rng.permutation(nf)])


bound = B.vote_request_wire_bound(nf)
L, h = ar._L, ar._h
stream = torch.cuda.Stream()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
COLS = ("term_start", "committed", "last_index", "matched", "next_idx", "peer_committed", "pflags")


def device_round(blob, off, restore_first):
    bufs = [ar.device_alloc(x) for x in (len(blob), 4 * (nf + 1), table.nbytes, nf, 16 * nf, bound, 4 * (nf + 1), 16)]
    d_b, d_o, d_v, d_st, d_out, d_rb, d_ro, d_t = bufs
    for ptr, x in ((d_b, blob), (d_o, off), (d_v, table)):
        ar.h2d(ptr, x)
    t_dev, t_call = [], []
    for k in range(runs + 2):   # the first two runs warm up
        if restore_first:
            ar.control(restore)
        ar.synchronize()
        t0 = time.perf_counter()
        ev0.record(stream)
        rc = L.raftgpu_vote_request_wire_device(h, stream.cuda_stream, d_b, int(off[-1]), d_o, nf, d_v, d_st, d_out, d_rb,
                                                bound, d_ro, d_t)
        ev1.record(stream)
        assert rc == B.OK, rc
        stream.synchronize()
        t1 = time.perf_counter()
        if k >= 2:
            t_dev.append(ev0.elapsed_time(ev1) * 1e-3)
            t_call.append(t1 - t0)
    tot = np.zeros(2, np.uint64)
    ar.d2h(tot, d_t)
    st, out = np.zeros(nf, np.uint8), np.zeros((nf, 2), np.uint64)
    rb, ro = np.zeros(int(tot[1]), np.uint8), np.zeros(int(tot[0]) + 1, np.uint32)
    for arr, ptr in ((st, d_st), (out, d_out), (rb, d_rb), (ro, d_ro)):
        ar.d2h(arr, ptr)
    for ptr in bufs:
        ar.device_free(ptr)
    return (st, out, rb, ro, tot), t_dev, t_call


def check(got, blob, off, what):
    c, v = O.copy_columns(c0), v0.copy()
    want = VR.batch(c, None, v, blob[: off[-1]], off, table, bench=True)
    for w, x, name in zip(want, got, ("status", "out", "bytes", "offsets", "totals")):
        assert np.array_equal(w, x), (what, name)
    cols = ar.read_columns(n)
    for name in COLS:
        assert np.array_equal(getattr(cols, name), getattr(c, name)[..., :n]), (what, name)
    assert np.array_equal(ar.column_read(B.COL_TERM, 0, 0, n, np.uint64), c.term[:n]), what
    return want[-1]


def us(t):
    a = np.array(t) * 1e6
    return f"{np.median(a):.1f} us (range {a.min():.1f}-{a.max():.1f})"


print(f"GPU: {gpu}")
pre_blob, pre_off = frames(17)
got, t_dev, t_call = device_round(pre_blob, pre_off, False)
secs = check(got, pre_blob, pre_off, "pre-vote round")
kinds = np.bincount(got[0] >> 4, minlength=16)
print(f"{n} follower groups x 5 voters, {nf} frames ({len(second)} second candidates: DUP), "
      f"{pre_off[-1] / nf:.1f} bytes per request, {got[4][1] / max(1, got[4][0]):.1f} per response; {runs} runs")
print(f"pre-vote round: {int(kinds[B.WIRE_OK])} OK ({int((got[0] & B.VREQ_GRANTED).astype(bool).sum())} granted), "
      f"{int(kinds[B.WIRE_DUP])} DUP")
print(f"  raftgpu_vote_request_wire_device: {us(t_dev)} between CUDA events; {us(t_call)} to the end of a synchronise")
fr = type("Frames", (), {"bytes": pre_blob, "n_bytes": int(pre_off[-1]), "offsets": pre_off, "n": nf})
t_host = []
for k in range(min(runs, 5) + 1):
    t0 = time.perf_counter()
    hst = ar.vote_request_wire(fr, table)
    t1 = time.perf_counter()
    if k >= 1:
        t_host.append(t1 - t0)
assert all(np.array_equal(x, y) for x, y in zip(hst, got)), "the host form differs from the device form"
print(f"  raftgpu_vote_request_wire (host form, end to end, {min(runs, 5)} runs): {us(t_host)}")
print(f"  batch oracle, one host core: {secs * 1e6:.1f} us")
vote_blob, vote_off = frames(5)
got, t_dev, t_call = device_round(vote_blob, vote_off, True)
secs = check(got, vote_blob, vote_off, "vote round")
kinds = np.bincount(got[0] >> 4, minlength=16)
print(f"vote round: {int(kinds[B.WIRE_OK])} OK ({int((got[0] & B.VREQ_BUMPED).astype(bool).sum())} bumped, "
      f"{int((got[0] & B.VREQ_VOTED).astype(bool).sum())} voted), {int(kinds[B.WIRE_DUP])} DUP")
print(f"  raftgpu_vote_request_wire_device: {us(t_dev)} between CUDA events; {us(t_call)} to the end of a synchronise "
      f"(restore outside)")
print(f"  batch oracle, one host core: {secs * 1e6:.1f} us")
print("both rounds match the batch oracle at full size: status, out, responses, offsets and the reset columns")
ar.close()
