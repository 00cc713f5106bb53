"""Micro-benchmark: MsgHeartbeatResponse frames on a cfg3-shaped arena (1M groups x 5 peers) with read queues
(max_pending = 8).  Every tick runs two halves, each after one MsgReadIndex per group
(raftgpu_read_index_request_device): the 4M heartbeat responses of the four followers, carrying that request's
context, in shuffled order, once as 24-byte records through raftgpu_heartbeat_resp_device +
raftgpu_read_index_ack_device, once as serialized frames (8-byte contexts) through raftgpu_heartbeat_wire_device.
Each pass is timed on the host clock from its call to the end of a device synchronise, so a figure includes its
launches and one synchronise.  Prints the bytes per frame against the 24-byte record, us per pass (median and range
over the ticks) and reads released per tick, with the GPU name and power limit read in the same run.  Without a GPU it
fails with RAFTGPU_ERR_NO_DEVICE."""
import importlib
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

pkg = importlib.import_module("raft-rs_b200")
B, W = pkg.binding, pkg.wire

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
cap = n * P
wb = W.WireBuffers(ar, 4 * n, bytes_per_record=32)

d_req, d_res = ar.device_alloc(reqs.nbytes), ar.device_alloc(n)
d_rec, d_hres = ar.device_alloc(recs.nbytes), ar.device_alloc(4 * n)
d_bytes, d_off, d_st = ar.device_alloc(len(wb.bytes)), ar.device_alloc(4 * (4 * n + 1)), ar.device_alloc(4 * n)
d_out, d_cnt, d_bad = ar.device_alloc(24 * cap), ar.device_alloc(8), ar.device_alloc(4)
cnt = np.zeros(1, np.uint64)


def timed(fn):
    t0 = time.perf_counter()
    rc = fn()
    assert rc == B.OK, rc
    ar.synchronize()
    return time.perf_counter() - t0


def request(tick, half):
    reqs["ctx"] = np.uint64(2 * tick + half) * np.uint64(n) + g + 1
    ar.h2d(d_req, reqs)
    assert timed(lambda: L.raftgpu_read_index_request_device(h, None, d_req, n, d_res, d_out, n, d_cnt, d_bad)) > 0
    recs["index"] = np.repeat(reqs["ctx"], 4)
    return recs[perm]


t_hb, t_ack, t_wire, rel_rec, rel_wire, frame_bytes = [], [], [], 0, 0, 0
for tick in range(ticks + 2):   # the first two ticks warm up
    ar.h2d(d_rec, request(tick, 0))
    th = timed(lambda: L.raftgpu_heartbeat_resp_device(h, None, d_rec, 4 * n, d_hres, None))
    ta = timed(lambda: L.raftgpu_read_index_ack_device(h, None, d_rec, 4 * n, d_out, cap, d_cnt))
    ar.d2h(cnt, d_cnt)
    r_rec = int(cnt[0])
    wb.encode_heartbeats(request(tick, 1))
    ar.h2d(d_bytes, wb.bytes[: wb.n_bytes])
    ar.h2d(d_off, wb.offsets[: wb.n + 1])
    tw = timed(lambda: L.raftgpu_heartbeat_wire_device(h, None, d_bytes, wb.n_bytes, d_off, wb.n, d_st, d_out, cap, d_cnt))
    ar.d2h(cnt, d_cnt)
    st = np.zeros(wb.n, np.uint8)
    ar.d2h(st, d_st)
    assert np.all((st >> 4) == B.WIRE_OK)
    if tick >= 2:
        t_hb.append(th), t_ack.append(ta), t_wire.append(tw)
        rel_rec += r_rec
        rel_wire += int(cnt[0])
        frame_bytes = wb.n_bytes


def us(t):
    a = np.array(t) * 1e6
    return f"{np.median(a):.1f} us (range {a.min():.1f}-{a.max():.1f})"


print(f"GPU: {gpu}")
print(f"{n} groups x 5 peers, max_pending {P}, {ticks} ticks of {4 * n} shuffled heartbeat responses")
print(f"bytes per response: {frame_bytes / (4 * n):.1f} frame + 4 offset = {frame_bytes / (4 * n) + 4:.1f}, "
      f"against the 24-byte record")
print(f"raftgpu_heartbeat_wire_device (decode + tracker + read): {us(t_wire)}; {rel_wire / ticks:.0f} reads released per tick")
print(f"records: raftgpu_heartbeat_resp_device {us(t_hb)} + raftgpu_read_index_ack_device {us(t_ack)} = "
      f"{np.median(np.array(t_hb) + np.array(t_ack)) * 1e6:.1f} us (median of sums); {rel_rec / ticks:.0f} released per tick")
wb.free()
