"""Micro-benchmark: the commit broadcast's MsgAppend frames (raftgpu_append_frames_device) on a cfg3-shaped arena (1M
groups x 5 peers, every group a leader with a term), next to raftgpu_send_list_device on the same selection.  Two
states: after three bench.py-style steps of synthetic traffic, selected by the last step's advanced bitmap (most sends
need entries: mostly rest entries), and the same arena with every follower caught up (next_idx = last_index + 1,
Replicate) and every group selected (all frames).  CUDA events around each call, median and range over the runs.
Prints the frame / rest split and the GPU name and power limit read in the same run.  Without a GPU it fails with
RAFTGPU_ERR_NO_DEVICE."""
import importlib
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

pkg = importlib.import_module("raft-rs_b200")
B = pkg.binding

n = int(os.environ.get("N", 1_000_000))
runs = int(os.environ.get("RUNS", 20))
ar = B.Arena(n)   # RaftGpuError(ERR_NO_DEVICE) without a GPU: no fallback
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(ar.info.device)],
                     capture_output=True, text=True).stdout.strip()
s = B.Synth(n, 0x5EED0003)
ar.group_alloc_range(n)
ar.load_columns(s.initial)
ar.column_write(B.COL_TERM, 0, 0, np.full(n, 7, np.uint64))
for _ in range(3):
    ar.step_begin_records(s.next_round().copy(), B.STEP_READ_COMMITTED)
    ar.step_wait()
adv = ar.step_results(n)[0].copy()
ids = np.random.default_rng(0xA99).integers(1, 1 << 20, (9, n), dtype=np.uint64)

bound = B.append_frames_bound(n)
d_ids, d_bytes, d_off = ar.device_alloc(ids.nbytes), ar.device_alloc(bound), ar.device_alloc(4 * (8 * n + 1))
d_rest, d_tot, d_sel = ar.device_alloc(16 * 8 * n), ar.device_alloc(32), ar.device_alloc(adv.nbytes)
d_list, d_cnt = ar.device_alloc(16 * 8 * n), ar.device_alloc(8)
ar.h2d(d_ids, ids)
L, h = ar._L, ar._h
stream = torch.cuda.Stream()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def timed(call):
    t = []
    for k in range(runs + 2):   # the first two runs warm up
        ev0.record(stream)
        assert call() == B.OK
        ev1.record(stream)
        stream.synchronize()
        if k >= 2:
            t.append(ev0.elapsed_time(ev1) * 1e3)
    return np.array(t)


def us(t):
    return f"{np.median(t):.1f} us (range {t.min():.1f}-{t.max():.1f})"


def measure(label, sel):
    if sel is not None:
        ar.h2d(d_sel, sel)
    ps = d_sel if sel is not None else None
    t_app = timed(lambda: L.raftgpu_append_frames_device(h, stream.cuda_stream, 0, n, ps, d_ids, d_bytes, bound, d_off, 8 * n,
                                                         d_rest, 8 * n, d_tot))
    t_list = timed(lambda: L.raftgpu_send_list_device(h, stream.cuda_stream, 0, n, ps, d_list, 8 * n, d_cnt))
    tot, cnt = np.zeros(4, np.uint64), np.zeros(1, np.uint64)
    ar.d2h(tot, d_tot)
    ar.d2h(cnt, d_cnt)
    frames, nbytes, rest = int(tot[0]), int(tot[1]), int(tot[2])
    print(f"{label}: {frames} frames ({nbytes} bytes, {nbytes / max(frames, 1):.1f} per frame) + {rest} rest entries "
          f"= {frames + rest} sends; the send list has {int(cnt[0])}")
    print(f"  raftgpu_append_frames_device: {us(t_app)}")
    print(f"  raftgpu_send_list_device:     {us(t_list)}")


print(f"GPU: {gpu}")
print(f"{n} groups x 5 peers, {runs} runs each, {int(np.unpackbits(adv.view(np.uint8)).sum())} groups advanced in the last step")
measure("after 3 steps, the advanced bitmap", adv)
c = ar.read_columns(n)
for k in range(B.SLOTS):
    ar.column_write(B.COL_NEXT_IDX, k, 0, (c.last_index + 1).astype(np.uint64))
    ar.column_write(B.COL_PFLAGS, k, 0, np.where((c.pflags[k] & 3) == B.STATE_SNAPSHOT, c.pflags[k],
                                                 B.STATE_REPLICATE).astype(np.uint8))
measure("every follower caught up, every group", None)
