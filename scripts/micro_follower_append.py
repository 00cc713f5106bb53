"""Micro-benchmark: entry-less MsgAppend frames at the follower (raftgpu_follower_append) on a cfg3-sized follower arena
(1M groups), one caught-up frame per group from raftgpu_append_frames, in a shuffled order; every group selected, at the
frame's term, its log ending at m.index in a run of m.log_term.  Times the device pass (raftgpu_follower_append_device,
CUDA events around the call) over the same frames each run -- after the first run commit_to moves nothing, which costs
the pass the same bytes -- median and range, then the host form end to end (copies in, the pass, copies back) and the C
batch oracle on one core over the same batch.  Prints the GPU's name and power limit read in the same run.  Without a
GPU it fails with RAFTGPU_ERR_NO_DEVICE.

--entries K [--payload B]: raftgpu_follower_append_entries instead, one MsgAppend per group with K entries of B data
bytes each at the log's tail (index = last_index, log_term = run_term = the term), so every frame appends.  The table
and last_index are restored before every pass (outside the CUDA events), so every timed pass appends.

    python scripts/micro_follower_append.py                                  # 1M groups, entry-less
    python scripts/micro_follower_append.py --entries 1 --payload 128        # 1M groups
    N=100000 python scripts/micro_follower_append.py --entries 8 --payload 1024"""
import argparse
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
from oracle import app_follow_oracle as AL
import hb_follow as FL
import hb_frames as F

pkg = importlib.import_module("raft-rs_b200")
B = pkg.binding

n = int(os.environ.get("N", 1_000_000))
runs = int(os.environ.get("RUNS", 20))
rng = np.random.default_rng(0xAF60)
ap = argparse.ArgumentParser()
ap.add_argument("--entries", type=int, default=0)
ap.add_argument("--payload", type=int, default=0)
args = ap.parse_args()
if args.entries:
    import micro_follower_append_entries as ME
    ME.main(B, n, runs, args.entries, args.payload, rng)
    sys.exit(0)

# the frames: raftgpu_append_frames of n leaders with one caught-up peer each (slot 1)
lc = O.new_columns(n, n)
lc.meta[:] = B.make_meta(0b11, 0, 0, 0)
lc.term[:] = rng.integers(1, 1 << 33, n)
lc.last_index[:] = rng.integers(1 << 20, 1 << 40, n)
lc.term_start[:] = lc.last_index - rng.integers(0, 1000, n).astype(np.uint64)
lc.committed[:] = lc.last_index - rng.integers(0, 50, n).astype(np.uint64)
lc.matched[1] = lc.last_index
lc.next_idx[1] = lc.last_index + 1
lc.pflags[1] = B.STATE_REPLICATE
la = B.Arena(n)   # RaftGpuError(ERR_NO_DEVICE) without a GPU: no fallback
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(la.info.device)],
                     capture_output=True, text=True).stdout.strip()
la.group_alloc_range(n)
la.load_columns(lc)
la.column_write(B.COL_TERM, 0, 0, lc.term.copy())
rc, fb, foff, _, ftot = la.append_frames(0, n, rng.integers(1, 1 << 63, (9, n), dtype=np.uint64))
assert rc == B.OK and int(ftot[0]) == n, ftot
la.close()
order = rng.permutation(n)                                    # shuffled: frame k comes from leader order[k]
lens = np.diff(foff.astype(np.int64))
starts = foff[:-1].astype(np.int64)[order]
idx = np.repeat(starts - np.concatenate([[0], np.cumsum(lens[order])[:-1]]), lens[order]) + np.arange(int(lens.sum()))
blob = np.asarray(fb)[idx]
off = np.concatenate([[0], np.cumsum(lens[order])]).astype(np.uint32)
perm = rng.permutation(n).astype(np.uint32)                   # leader g's follower: group perm[g]
blob = FL.with_headers(blob, off, perm[order] << 4 | 1)

ar = B.Arena(n)
ar.group_alloc_range(n)
terms, last, committed = np.zeros(n, np.uint64), np.zeros(n, np.uint64), np.zeros(n, np.uint64)
terms[perm], last[perm] = lc.term, lc.last_index
committed[perm] = lc.committed - rng.integers(0, 100, n).astype(np.uint64)
for col, arr in ((B.COL_TERM, terms), (B.COL_LAST_INDEX, last), (B.COL_COMMITTED, committed),
                 (B.COL_TERM_START, np.full(n, B.NO_TERM_START, np.uint64))):
    ar.column_write(col, 0, 0, arr)
table = np.zeros(n, AL.LOG_DTYPE)
table["id"], table["flags"] = rng.integers(1, 1 << 20, n, dtype=np.uint64), AL.SELECT
table["run_start"], table["run_term"] = last - np.minimum(last, np.uint64(10)), terms

# the C oracle, single thread, over the same batch and the same starting state
c = O.new_columns(n, n)
c.term_start[:], c.term[:], c.last_index[:], c.committed[:] = B.NO_TERM_START, terms, last, committed
st_o, _, _, _, tot_o, t_oracle = AL.batch(c, None, table, blob, off, bench=True)
assert np.all(st_o == (B.WIRE_OK << 4 | B.RES_OK))

bound = B.follower_append_bound(n)
bufs = [ar.device_alloc(x) for x in (len(blob) + 16, 4 * (n + 1), table.nbytes, n, 8 * n, bound, 4 * (n + 1), 16)]
d_b, d_o, d_t, d_st, d_f, d_rb, d_ro, d_tot = bufs
for p, x in ((d_b, blob), (d_o, off), (d_t, table)):
    ar.h2d(p, x)
L, h = ar._L, ar._h
stream = torch.cuda.Stream()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
t_dev = []
for k in range(runs + 2):   # the first two runs warm up (the first one also moves committed)
    ev0.record(stream)
    rc = L.raftgpu_follower_append_device(h, stream.cuda_stream, d_b, len(blob), d_o, n, d_t, d_st, d_f, d_rb, bound, d_ro,
                                          d_tot)
    ev1.record(stream)
    assert rc == B.OK, rc
    stream.synchronize()
    if k >= 2:
        t_dev.append(ev0.elapsed_time(ev1) * 1e-3)
tot, st = np.zeros(2, np.uint64), np.zeros(n, np.uint8)
ar.d2h(tot, d_tot), ar.d2h(st, d_st)
assert np.array_equal(st, st_o) and tot.tolist() == tot_o.tolist(), (tot, tot_o)
for p in bufs:
    ar.device_free(p)

# the host form end to end: pageable input, the copies in, the pass, the copies back
hb = F.Frames([])
hb.bytes, hb.offsets, hb.n, hb.n_bytes = np.concatenate([blob, np.zeros(16, np.uint8)]), off, n, len(blob)
t_host = []
for k in range(5):
    t0 = time.perf_counter()
    got = ar.follower_append(hb, table)
    t_host.append(time.perf_counter() - t0)
assert np.array_equal(got[0], st_o)


def us(t):
    a = np.array(t) * 1e6
    return f"{np.median(a):.1f} us (range {a.min():.1f}-{a.max():.1f})"


print(f"GPU: {gpu}")
print(f"{n} follower groups, {n} MsgAppend frames from raftgpu_append_frames (shuffled), {len(blob) / n:.1f} bytes per "
      f"frame in, {int(tot[1]) / n:.1f} per response out")
print(f"raftgpu_follower_append_device: {us(t_dev)} over {runs} passes between CUDA events")
print(f"raftgpu_follower_append (host form, end to end): {us(t_host)} over 5 calls")
print(f"C batch oracle (afl_batch, one thread): {t_oracle * 1e3:.1f} ms over the same batch")
