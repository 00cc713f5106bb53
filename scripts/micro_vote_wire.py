#!/usr/bin/env python
"""Vote responses at a candidate (raftgpu_vote_wire_device) in scripts/micro_control.py's election storm: 1M groups x 5
voters, every group a Candidate whose self vote is in, and 4M shuffled MsgRequestVoteResponse frames (each peer answers
once).  Before every pass an untimed control list resets the votes and records the self votes.  Timed over 20 passes,
median and range: the pass between CUDA events, the pass from the call to the end of a synchronise, and the same votes
as INTEGRATION.md section 6 step 2's control list (RECORD_VOTE + VOTE_RESULT per response, raftgpu_control: copy, run,
copy back).  Checks that the two forms leave the same votes and decide the same groups, and prints the GPU's name and
power limit read in the same run.

    python scripts/micro_vote_wire.py [--groups N] [--runs K]
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

p = argparse.ArgumentParser()
p.add_argument("--groups", type=int, default=1_000_000)
p.add_argument("--runs", type=int, default=20)
args = p.parse_args()
n, runs = args.groups, args.runs
rng = np.random.default_rng(0x707A)

ar = B.Arena(n)   # RaftGpuError(ERR_NO_DEVICE) without a GPU: no fallback
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(ar.info.device)],
                     capture_output=True, text=True).stdout.strip()
ar.group_alloc_range(n)
g = np.arange(n, dtype=np.uint32)
term = rng.integers(1, 1 << 30, n).astype(np.uint64)
setup = np.zeros(3 * n, B.CTL_CMD_DTYPE)
setup["group"] = np.tile(g, 3)
setup["op"][:n], setup["a"][:n, 0], setup["a"][:n, 3] = B.CTL_SET_CONF, 0x1F, 11
setup["op"][n:2 * n], setup["a"][n:2 * n] = B.CTL_RESET, (B.NO_TERM_START, 10, 5, 10)
setup["op"][2 * n:], setup["a"][2 * n:, 0] = B.CTL_SET_TERM, term
assert np.all(ar.control(setup)["status"] == 0)
fresh = np.zeros(2 * n, B.CTL_CMD_DTYPE)          # reset_votes + the self vote: what every pass starts from
fresh["group"] = np.repeat(g, 2)
fresh["op"][0::2], fresh["op"][1::2], fresh["arg"][1::2] = B.CTL_RESET_VOTES, B.CTL_RECORD_VOTE, 1

gs = np.repeat(g, 4)
slots = np.tile(np.arange(1, 5, dtype=np.uint32), n)
granted = (rng.random(4 * n) < 0.55).astype(np.uint32)
perm = rng.permutation(4 * n)
gs, slots, granted = gs[perm], slots[perm], granted[perm]
e = np.zeros(4 * n, B.SYNTH_VOTE_DTYPE)
e["hdr"], e["msg_type"], e["to"], e["from"] = gs << 4 | slots, 6, 1, slots + 1
e["term"], e["reject"] = term[gs], 1 - granted
blob, off = B.synth_encode_votes(e)
nf = 4 * n
step2 = np.zeros(2 * nf, B.CTL_CMD_DTYPE)
step2["group"] = np.repeat(gs, 2)
step2["op"][0::2], step2["op"][1::2] = B.CTL_RECORD_VOTE, B.CTL_VOTE_RESULT
step2["peer_slot"][0::2], step2["arg"][0::2] = slots, granted

sel = np.packbits(np.ones(n + (-n) % 32, bool), bitorder="little").view(np.uint32).copy()
bufs = [ar.device_alloc(x) for x in (len(blob), 4 * (nf + 1), sel.nbytes, nf, 8 * n, 8)]
d_b, d_o, d_s, d_st, d_out, d_c = bufs
for ptr, x in ((d_b, blob), (d_o, off), (d_s, sel)):
    ar.h2d(ptr, x)
L, h = ar._L, ar._h
stream = torch.cuda.Stream()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
t_dev, t_call, t_list = [], [], []
for k in range(runs + 2):   # the first two runs warm up
    ar.control(fresh)
    ar.synchronize()
    t0 = time.perf_counter()
    ev0.record(stream)
    rc = L.raftgpu_vote_wire_device(h, stream.cuda_stream, d_b, len(blob), d_o, nf, d_s, None, d_st, d_out, n, d_c)
    ev1.record(stream)
    assert rc == B.OK, rc
    stream.synchronize()
    t1 = time.perf_counter()
    if k >= 2:
        t_dev.append(ev0.elapsed_time(ev1) * 1e-3)
        t_call.append(t1 - t0)
cnt, st = np.zeros(1, np.uint64), np.zeros(nf, np.uint8)
ar.d2h(cnt, d_c), ar.d2h(st, d_st)
out = np.zeros(int(cnt[0]), B.VOTE_OUTCOME_DTYPE)
ar.d2h(out, d_out)
votes_pass = np.stack([ar.column_read(B.COL_VOTES, s, 0, n, np.uint8) for s in range(5)])
assert np.all(st == (B.WIRE_OK << 4 | B.RES_OK))
for k in range(runs + 2):
    ar.control(fresh)
    ar.synchronize()
    t0 = time.perf_counter()
    res = ar.control(step2)
    t1 = time.perf_counter()
    if k >= 2:
        t_list.append(t1 - t0)
votes_list = np.stack([ar.column_read(B.COL_VOTES, s, 0, n, np.uint8) for s in range(5)])
last = np.zeros(n, np.uint32)
last[gs] = res["value"][1::2].astype(np.uint32)
decided = np.flatnonzero(last & 0xFF != B.VOTE_PENDING)
assert np.array_equal(votes_pass, votes_list), "the pass and the control list disagree on the votes"
assert np.array_equal(out["group"], decided) and np.array_equal(out["result"], last[decided]), "outcomes differ"


def us(t):
    a = np.array(t) * 1e6
    return f"{np.median(a):.1f} us (range {a.min():.1f}-{a.max():.1f})"


won = int(((out["result"] & 0xFF) == B.VOTE_WON).sum())
print(f"GPU: {gpu}")
print(f"{n} candidate groups x 5 voters, {nf} MsgRequestVoteResponse frames (shuffled), {len(blob) / nf:.1f} bytes per "
      f"frame; {len(out)} decided ({won} won); {runs} runs")
print(f"raftgpu_vote_wire_device: {us(t_dev)} between CUDA events; {us(t_call)} from the call to the end of a synchronise")
print(f"section 6 step 2 control list ({2 * nf} commands, raftgpu_control): {us(t_list)}")
print("the pass and the list agree: same votes, same decided groups and words")
for ptr in bufs:
    ar.device_free(ptr)
ar.close()
