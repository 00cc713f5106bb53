"""Micro-benchmark: ReadIndex (ReadOnlyOption::Safe) on a cfg3-shaped arena (1M groups x 5 peers) with read queues
(max_pending = 8).  Every tick, one MsgReadIndex per group (raftgpu_read_index_request_device), then the 4M heartbeat
responses of the four followers carrying that tick's context, in shuffled order (raftgpu_read_index_ack_device);
beside them, raftgpu_heartbeat_resp_device's tracker pass over the same device records.  Each pass is timed on the
host clock from its call to the end of a device synchronise, so a figure includes one launch and one synchronise.
Prints us per pass (median and range over the ticks), requests/s and reads released/s, with the GPU name and power
limit read in the same run.  Without a GPU it fails with RAFTGPU_ERR_NO_DEVICE."""
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
ticks = int(os.environ.get("TICKS", 20))
P = 8
ar = B.Arena(n)   # RaftGpuError(ERR_NO_DEVICE) without a GPU: no fallback
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(ar.info.device)],
                     capture_output=True, text=True).stdout.strip()
ar.enable_read_index(P)
s = B.Synth(n, 0x5EED0003)
ar.group_alloc_range(n)
ar.load_columns(s.initial)
L, h = ar._L, ar._h
rng = np.random.default_rng(0x4EAD)

g = np.arange(n, dtype=np.uint32)
reqs = np.zeros(n, dtype=B.READ_REQ_DTYPE)
reqs["group"] = g
recs = np.zeros(4 * n, dtype=B.APPEND_RESP_DTYPE)
recs["group"] = np.repeat(g, 4)
recs["peer_slot"] = np.tile(np.arange(1, 5, dtype=np.uint8), n)
recs["flags"] = B.REC_HEARTBEAT | B.REC_READ_CTX
recs["commit"] = np.repeat(s.initial.committed[:n], 4)
perm = rng.permutation(4 * n)
cap_ack = n * P

d_req, d_res = ar.device_alloc(reqs.nbytes), ar.device_alloc(n)
d_rec, d_hres = ar.device_alloc(recs.nbytes), ar.device_alloc(4 * n)
d_out, d_cnt, d_bad = ar.device_alloc(24 * cap_ack), ar.device_alloc(8), ar.device_alloc(4)
cnt = np.zeros(1, np.uint64)


def timed(fn):
    t0 = time.perf_counter()
    rc = fn()
    assert rc == B.OK, rc
    ar.synchronize()
    return time.perf_counter() - t0


t_req, t_ack, t_hb, n_queued, n_released = [], [], [], 0, 0
for tick in range(ticks + 2):   # the first two ticks warm up
    reqs["ctx"] = np.uint64(tick) * np.uint64(n) + g + 1
    recs["index"] = np.repeat(reqs["ctx"], 4)
    ar.h2d(d_req, reqs)
    ar.h2d(d_rec, recs[perm])
    tr = timed(lambda: L.raftgpu_read_index_request_device(h, None, d_req, n, d_res, d_out, n, d_cnt, d_bad))
    res = np.zeros(n, np.uint8)
    ar.d2h(res, d_res)
    ta = timed(lambda: L.raftgpu_read_index_ack_device(h, None, d_rec, 4 * n, d_out, cap_ack, d_cnt))
    ar.d2h(cnt, d_cnt)
    th = timed(lambda: L.raftgpu_heartbeat_resp_device(h, None, d_rec, 4 * n, d_hres, None))
    if tick >= 2:
        t_req.append(tr), t_ack.append(ta), t_hb.append(th)
        n_queued += int((res == B.READ_QUEUED).sum())
        n_released += int(cnt[0])
pend = ar.read_index_read(0, n)[0]


def us(t):
    a = np.array(t) * 1e6
    return f"{np.median(a):.1f} us (range {a.min():.1f}-{a.max():.1f})"


print(f"GPU: {gpu}")
print(f"{n} groups x 5 peers, max_pending {P}, {ticks} ticks: {n_queued / ticks:.0f} reads queued per tick, "
      f"{n_released / ticks:.0f} released per tick, {int(pend.sum())} pending at the end")
print(f"request pass ({n} requests): {us(t_req)}; {n / np.median(t_req) / 1e6:.1f} M requests/s")
print(f"ack pass ({4 * n} heartbeat responses, shuffled): {us(t_ack)}; "
      f"{n_released / ticks / np.median(t_ack) / 1e6:.1f} M reads released/s")
print(f"raftgpu_heartbeat_resp pass over the same records: {us(t_hb)}")
