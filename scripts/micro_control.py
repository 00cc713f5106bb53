"""Micro-benchmark: the control plane's list form against its single-group calls, on a cfg3-shaped arena (1M groups x
5 peers).  (a) the store-wide election of INTEGRATION 6 as raftgpu_control lists -- every group campaigns (RESET +
SET_TERM + RESET_VOTES + RECORD_VOTE(self) + VOTE_RESULT), the vote responses (4 x RECORD_VOTE + VOTE_RESULT), the
winners' RESET + BECOME_LEADER -- wall clock to each call's final synchronise; (b) the same commands of a 10 000-group
sample as single calls (one launch + synchronise each, called through ctypes).  Prints commands/s and us per command,
with the GPU name and power limit read in the same run.  Without a GPU it fails with RAFTGPU_ERR_NO_DEVICE."""
import ctypes as C
import importlib
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

B = importlib.import_module("raft-rs_b200").binding

n = int(os.environ.get("N", 1_000_000))
sample = min(n, int(os.environ.get("SAMPLE", 10_000)))
ar = B.Arena(n)   # RaftGpuError(ERR_NO_DEVICE) without a GPU: no fallback
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(ar.info.device)],
                     capture_output=True, text=True).stdout.strip()
s = B.Synth(n, 0x5EED0003)
ar.group_alloc_range(n)
ar.load_columns(s.initial)
rng = np.random.default_rng(0x57041)
init = s.initial
g = np.arange(n, dtype=np.uint32)
li = init.last_index[:n]

campaign = np.zeros((n, 5), dtype=B.CTL_CMD_DTYPE)
campaign["group"] = g[:, None]
campaign["op"] = [B.CTL_RESET, B.CTL_SET_TERM, B.CTL_RESET_VOTES, B.CTL_RECORD_VOTE, B.CTL_VOTE_RESULT]
campaign["a"][:, 0, 0], campaign["a"][:, 0, 1], campaign["a"][:, 0, 2], campaign["a"][:, 0, 3] = \
    B.NO_TERM_START, li, init.committed[:n], li
campaign["a"][:, 1, 0] = 2
campaign["arg"][:, 3] = 1
responses = np.zeros((n, 5), dtype=B.CTL_CMD_DTYPE)
responses["group"] = g[:, None]
responses["op"][:, :4], responses["op"][:, 4] = B.CTL_RECORD_VOTE, B.CTL_VOTE_RESULT
responses["peer_slot"][:, :4] = np.arange(1, 5)
responses["arg"][:, :4] = rng.random((n, 4)) < 0.6


def leaders(res_responses, groups):
    won = groups[(res_responses.reshape(len(groups), 5)[:, 4]["value"] & 0xFF) == B.VOTE_WON]
    out = np.zeros((len(won), 2), dtype=B.CTL_CMD_DTYPE)
    out["group"] = won[:, None]
    out["op"] = [B.CTL_RESET, B.CTL_BECOME_LEADER]
    out["a"][:, 0, 0], out["a"][:, 0, 1], out["a"][:, 0, 2], out["a"][:, 0, 3] = \
        li[won] + 1, li[won], init.committed[won], li[won]
    return out.reshape(-1)


# warm-up: every op of the storm once through the list form and once through the single calls
warm = np.concatenate([campaign[:64].reshape(-1), responses[:64].reshape(-1)])
ar.control(warm)

# (a) the storm as three lists
t_lists, n_cmds = [], 0
for lst in (campaign.reshape(-1), responses.reshape(-1)):
    t0 = time.perf_counter()
    res = ar.control(lst)
    t_lists.append(time.perf_counter() - t0)
    n_cmds += len(lst)
    assert (res["status"] == B.OK).all()
lead = leaders(res, g)
t0 = time.perf_counter()
assert (ar.control(lead)["status"] == B.OK).all()
t_lists.append(time.perf_counter() - t0)
n_cmds += len(lead)
t_a = sum(t_lists)

# (b) the same commands of the first `sample` groups as single calls, on a fresh copy of their state
ar.load_columns(s.initial)
L, h = ar._L, ar._h
out, gr, rj = C.c_int32(), C.c_uint32(), C.c_uint32()


def single(m):
    op, gg, sl, arg, a = int(m["op"]), int(m["group"]), int(m["peer_slot"]), int(m["arg"]), [int(x) for x in m["a"]]
    if op == B.CTL_RESET:
        return L.raftgpu_group_reset(h, gg, *a)
    if op == B.CTL_SET_TERM:
        return L.raftgpu_group_set_term(h, gg, a[0])
    if op == B.CTL_RESET_VOTES:
        return L.raftgpu_reset_votes(h, gg)
    if op == B.CTL_RECORD_VOTE:
        return L.raftgpu_record_vote(h, gg, sl, arg)
    if op == B.CTL_VOTE_RESULT:
        return L.raftgpu_vote_result(h, gg, C.byref(out), C.byref(gr), C.byref(rj))
    return L.raftgpu_group_become_leader(h, gg)


for m in warm[:10]:
    single(m)
sample_lists = [campaign[:sample].reshape(-1), responses[:sample].reshape(-1)]
n_single, t0 = 0, time.perf_counter()
for lst in sample_lists:
    for m in lst:
        assert single(m) == B.OK
    n_single += len(lst)
lead_s = lead[np.isin(lead["group"], g[:sample])]
for m in lead_s:
    assert single(m) == B.OK
n_single += len(lead_s)
t_b = time.perf_counter() - t0

print(f"GPU: {gpu}")
print(f"(a) raftgpu_control, election storm over {n} groups: {n_cmds} commands in {t_a * 1e3:.1f} ms "
      f"(campaign {t_lists[0] * 1e3:.1f}, responses {t_lists[1] * 1e3:.1f}, leaders {t_lists[2] * 1e3:.1f}): "
      f"{n_cmds / t_a / 1e6:.2f} M commands/s, {t_a / n_cmds * 1e6:.3f} us per command")
print(f"(b) single calls, {sample}-group sample: {n_single} commands in {t_b * 1e3:.1f} ms: "
      f"{n_single / t_b / 1e3:.1f} k commands/s, {t_b / n_single * 1e6:.2f} us per command")
print(f"ratio (b)/(a) per command: {(t_b / n_single) / (t_a / n_cmds):.0f}x")
