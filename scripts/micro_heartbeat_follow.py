"""Micro-benchmark: MsgHeartbeat frames at the follower (raftgpu_follower_heartbeat) on a cfg3-sized follower arena (1M
groups), one heartbeat per group in a shuffled order, three quarters of them with an 8-byte context; every group
selected, at the heartbeat's term, with its log past m.commit.  Times the device pass (raftgpu_follower_heartbeat_device,
CUDA events around the call, and from the call to the end of a synchronise) over the same frames each run -- after
the first run commit_to moves nothing, which costs the pass the same bytes -- median and range.  Prints the
algorithmic bytes per frame, the fraction of the data sheet's 3.35 TB/s, the GPU's name and power limit read in the
same run, and the C oracle's single-thread time over the same batch.  Without a GPU it fails with RAFTGPU_ERR_NO_DEVICE."""
import importlib
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np
import torch

from oracle import oracle as O
from oracle import read_oracle as RO
from oracle import hb_frames_oracle as HF
from oracle import hb_follow_oracle as HL
import hb_follow as FL

pkg = importlib.import_module("raft-rs_b200")
B = pkg.binding

n = int(os.environ.get("N", 1_000_000))
runs = int(os.environ.get("RUNS", 20))
rng = np.random.default_rng(0x4EF6)

# the frames: one heartbeat from each of n leaders (one peer each), 3/4 with a pending read id as the context
lc = O.new_columns(n, n)
lc.meta[:] = B.make_meta(0b11, 0, 0, 0)
lc.term_start[:] = 1
lc.term[:] = rng.integers(1, 1 << 33, n)
lc.committed[:] = rng.integers(1 << 20, 1 << 40, n)
lc.matched[1] = lc.committed
q = RO.ReadQueues(n, 1)
q.allocated[:] = 1
q.count[:] = rng.random(n) < 0.75
q.ctx[:, 0] = rng.integers(1, 1 << 63, n, dtype=np.uint64)
hb, hoff, htot = HF.bcast_heartbeats(lc, q, 0, n, rng.integers(1, 1 << 63, (9, n), dtype=np.uint64))
order = rng.permutation(n)                                    # shuffled: frame k comes from leader order[k]
lens = np.diff(hoff.astype(np.int64))
starts = hoff[:-1].astype(np.int64)[order]
idx = np.repeat(starts - np.concatenate([[0], np.cumsum(lens[order])[:-1]]), lens[order]) + np.arange(int(lens.sum()))
blob = hb[idx]
off = np.concatenate([[0], np.cumsum(lens[order])]).astype(np.uint32)
perm = rng.permutation(n).astype(np.uint32)                   # leader g's follower: group perm[g]
blob = FL.with_headers(blob, off, perm[order] << 4 | 1)
commit = lc.committed

ar = B.Arena(n)   # RaftGpuError(ERR_NO_DEVICE) without a GPU: no fallback
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(ar.info.device)],
                     capture_output=True, text=True).stdout.strip()
ar.group_alloc_range(n)
terms, last = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
terms[perm] = lc.term
last[perm] = commit + np.uint64(100)
committed = last - np.uint64(200)
for col, arr in ((B.COL_TERM, terms), (B.COL_LAST_INDEX, last), (B.COL_COMMITTED, committed),
                 (B.COL_TERM_START, np.full(n, B.NO_TERM_START, np.uint64))):
    ar.column_write(col, 0, 0, arr)
sel = FL.bitmap(np.ones(n, bool))
ids = rng.integers(1, 1 << 20, n, dtype=np.uint64)

# the C oracle, single thread, over the same batch and the same starting state
c = O.new_columns(n, n)
c.meta[:], c.term_start[:], c.term[:], c.last_index[:], c.committed[:] = 0, B.NO_TERM_START, terms, last, committed
st_o, _, _, _, tot_o, t_oracle = HL.follower_heartbeats(c, None, blob, off, sel, ids, bench=True)

bound = B.follower_heartbeat_bound(n)
bufs = [ar.device_alloc(x) for x in (len(blob) + 16, 4 * (n + 1), sel.nbytes, ids.nbytes, n, 8 * n, bound, 4 * (n + 1), 16)]
d_b, d_o, d_s, d_i, d_st, d_f, d_rb, d_ro, d_t = bufs
for p, x in ((d_b, blob), (d_o, off), (d_s, sel), (d_i, ids)):
    ar.h2d(p, x)
L, h = ar._L, ar._h
stream = torch.cuda.Stream()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
t_dev, t_call = [], []
for k in range(runs + 2):   # the first two runs warm up (the first one also moves committed)
    t0 = time.perf_counter()
    ev0.record(stream)
    rc = L.raftgpu_follower_heartbeat_device(h, stream.cuda_stream, d_b, len(blob), d_o, n, d_s, d_i, d_st, d_f, d_rb, bound,
                                             d_ro, d_t)
    ev1.record(stream)
    assert rc == B.OK, rc
    stream.synchronize()
    t1 = time.perf_counter()
    if k >= 2:
        t_dev.append(ev0.elapsed_time(ev1) * 1e-3)
        t_call.append(t1 - t0)
tot, st = np.zeros(2, np.uint64), np.zeros(n, np.uint8)
ar.d2h(tot, d_t), ar.d2h(st, d_st)
assert np.array_equal(st, st_o) and int(tot[0]) == n and tot.tolist() == tot_o.tolist(), (tot, tot_o)


def us(t):
    a = np.array(t) * 1e6
    return f"{np.median(a):.1f} us (range {a.min():.1f}-{a.max():.1f})"


nbytes = int(tot[1])
frame_bytes = len(blob) / n
# per frame: the frame and its 4-byte offset (+ the next block's first offset), the status byte (written by the scan,
# read and rewritten by the apply pass, read by the write pass), meta 4 + term_start 8 + term 8 + committed 8 +
# last_index 8 + the select word 4 + the self id 8 (scan), the 48-byte record (written by the scan, read by the apply
# and write passes, commit rewritten: 8), first_frame 4 (atomic in the scan, read in the apply pass), committed +
# last_index 16 read and committed 8 written (apply), from 8 written, the response and its 4-byte offset written;
# plus the 4 bytes per group slot of the first_frame reset.
read_pf = frame_bytes + 4 + 1 + 1 + 48 + 8 + 8 + 8 + 8 + 4 + 8 + 48 + 48 + 4 + 16 + 4
write_pf = 1 + 1 + 48 + 8 + 4 + 8 + 8 + nbytes / n + 4 + 4
med = np.median(t_dev)
print(f"GPU: {gpu}")
print(f"{n} follower groups, {n} MsgHeartbeat frames (shuffled, {int(q.count.sum())} with an 8-byte context), "
      f"{frame_bytes:.1f} bytes per frame in, {nbytes / n:.1f} per response out; {runs} runs")
print(f"algorithmic bytes per frame: {read_pf:.0f} read, {write_pf:.0f} written")
print(f"raftgpu_follower_heartbeat_device: {us(t_dev)} between CUDA events "
      f"({(read_pf + write_pf) * n / med / 1e9:.0f} GB/s algorithmic, {(read_pf + write_pf) * n / med / 3.35e12 * 100:.1f}% "
      f"of 3.35 TB/s); {us(t_call)} from the call to the end of a synchronise")
print(f"C oracle (hfl_follower_heartbeats, one thread): {t_oracle * 1e3:.1f} ms over the same batch")
