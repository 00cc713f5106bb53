"""Micro-benchmark: MsgHeartbeat frames (raftgpu_heartbeat_frames) on a cfg3-shaped arena (1M groups x 5 peers, every
group a leader with a term) with read queues (max_pending = 8) and one pending read per group, so every frame carries
an 8-byte context.  Times the device pass (raftgpu_heartbeat_frames_device, CUDA events around the call) and the host
form (raftgpu_heartbeat_frames: the H2D of the id table, the pass, the D2H of offsets and bytes, on the host clock),
median and range over the runs.  Prints the output per group and the algorithmic bytes the pass reads and writes per
group, with the GPU name and power limit read in the same run.  Without a GPU it fails with RAFTGPU_ERR_NO_DEVICE."""
import importlib
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

pkg = importlib.import_module("raft-rs_b200")
B = pkg.binding

n = int(os.environ.get("N", 1_000_000))
runs = int(os.environ.get("RUNS", 20))
P = 8
ar = B.Arena(n)   # RaftGpuError(ERR_NO_DEVICE) without a GPU: no fallback
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(ar.info.device)],
                     capture_output=True, text=True).stdout.strip()
ar.enable_read_index(P)
s = B.Synth(n, 0x5EED0003)
ar.group_alloc_range(n)
ar.load_columns(s.initial)
ar.column_write(B.COL_TERM, 0, 0, np.full(n, 7, np.uint64))
reqs = np.zeros(n, dtype=B.READ_REQ_DTYPE)
reqs["group"], reqs["ctx"] = np.arange(n), np.arange(1, n + 1)
res, _ = ar.read_index_request(reqs)
rng = np.random.default_rng(0x4EB)
ids = rng.integers(1, 1 << 20, (9, n), dtype=np.uint64)

bound = B.heartbeat_frames_bound(n)
d_ids, d_bytes = ar.device_alloc(ids.nbytes), ar.device_alloc(bound)
d_off, d_tot = ar.device_alloc(4 * (8 * n + 1)), ar.device_alloc(24)
ar.h2d(d_ids, ids)
L, h = ar._L, ar._h
stream = torch.cuda.Stream()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
tot = np.zeros(3, np.uint64)

t_dev, t_call = [], []
for k in range(runs + 2):   # the first two runs warm up
    t0 = time.perf_counter()
    ev0.record(stream)
    rc = L.raftgpu_heartbeat_frames_device(h, stream.cuda_stream, 0, n, None, d_ids, d_bytes, bound, d_off, 8 * n, d_tot)
    ev1.record(stream)
    assert rc == B.OK, rc
    stream.synchronize()
    t1 = time.perf_counter()
    if k >= 2:
        t_dev.append(ev0.elapsed_time(ev1) * 1e-3)
        t_call.append(t1 - t0)
ar.d2h(tot, d_tot)
frames, nbytes = int(tot[0]), int(tot[1])

bytes_out = np.zeros(nbytes, np.uint8)
offsets_out = np.zeros(frames + 1, np.uint32)
t_host = []
for k in range(runs + 2):
    t0 = time.perf_counter()
    rc, blob, off, t = ar.heartbeat_frames(0, n, ids, bytes_out=bytes_out, offsets_out=offsets_out)
    t1 = time.perf_counter()
    assert rc == B.OK and int(t[0]) == frames
    if k >= 2:
        t_host.append(t1 - t0)


def us(t):
    a = np.array(t) * 1e6
    return f"{np.median(a):.1f} us (range {a.min():.1f}-{a.max():.1f})"


pending = int((res == B.READ_QUEUED).sum())
peers = frames / n
# per group, each of the two passes that read the arena: meta 4 + term_start 8 + term 8 + committed 8 + from 8 + the
# queue word 4 (+ its last ctx 8 when a read is pending) + per peer matched 8 + id 8; the write pass also reads the
# size pass's 8-byte count.  Written: the 8-byte count, the frames and their 4-byte offsets.
read_pg = 2 * (40 + 8 * pending / n + 16 * peers) + 8
write_pg = 8 + nbytes / n + 4 * frames / n
print(f"GPU: {gpu}")
print(f"{n} groups x 5 peers, max_pending {P}, {pending} groups with a pending read; {runs} runs")
print(f"output: {frames} frames, {nbytes} bytes ({nbytes / frames:.1f} per frame, {nbytes / n:.1f} + {4 * frames / n:.1f} "
      f"offset bytes per group)")
print(f"algorithmic bytes per group: {read_pg:.0f} read, {write_pg:.0f} written")
print(f"raftgpu_heartbeat_frames_device: {us(t_dev)} between CUDA events; {(read_pg + write_pg) * n / np.median(t_dev) / 1e9:.0f} "
      f"GB/s algorithmic; {us(t_call)} from the call to the end of a synchronise")
print(f"raftgpu_heartbeat_frames (H2D of {ids.nbytes >> 20} MiB ids + pass + D2H of {(nbytes + 4 * frames) >> 20} MiB): "
      f"{us(t_host)}")
