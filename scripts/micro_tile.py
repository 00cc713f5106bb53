"""Micro-benchmark of a fused tile kernel alone: 1M groups x 5 peers, 4 arenas rotated (inputs larger than L2), R rounds
each, one CUDA graph of all launches, CUDA events.  KERNEL=packed (default) times step_tile_kernel
(raftgpu_step_sorted_device on packed records); KERNEL=compact times step_tile_compact_kernel
(raftgpu_step_compact_device on the same rounds packed with raftgpu_pack_compact, tile index built beforehand), which
the end-to-end legs of bench.py hide behind PCIe.  With RAFTGPU_TILE_DEBUG=1 in the environment the kernel's phase
cycle counters are printed too."""
import importlib, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np, torch
B = importlib.import_module("raft-rs_b200").binding
n = int(os.environ.get("N", 1_000_000))
R = int(os.environ.get("R", 6))
joint = os.environ.get("JOINT", "0") == "1"
kernel = os.environ.get("KERNEL", "packed")
assert kernel in ("packed", "compact"), kernel
NA = 4
arenas, rounds, outs = [], [], []
pack_buf = np.empty((7 * n + 64, 2), dtype=np.uint64)
for a in range(NA):
    s = B.Synth(n, 0x5EED0003 + 0x100 * a, k_peers=5, joint=joint)
    ar = B.Arena(n, n_rings=1, ring_records=4096)
    ar.group_alloc_range(n); ar.load_columns(s.initial)
    # the step's outputs (advanced bitmap, commit index of every group), written as bench.py's fused leg writes them
    outs.append({"d_adv": ar.device_alloc(4 * ((n + 31) // 32 + 1)), "d_commit": ar.device_alloc(8 * n)})
    rr = []
    for _ in range(R):
        recs = s.next_round()
        if kernel == "packed":
            k = ar.pack_records(recs, pack_buf)
            p = ar.device_alloc(16 * k); ar.h2d(p, pack_buf[:k])
            off = B.tile_index(pack_buf, k, n)
            po = ar.device_alloc(off.nbytes); ar.h2d(po, off)
            rr.append(((p, k, po), {}))
        else:
            blob = np.zeros(B.compact_bound(len(recs)), dtype=np.uint8)
            nb, _ = B.pack_compact(np.ascontiguousarray(recs), blob)
            d_blob = ar.device_alloc(nb); ar.h2d(d_blob, blob[:nb])
            d_off = ar.device_alloc(4 * (3 * (ar.cap // B.tile_groups() + 2) + 2))
            d_dup = ar.device_alloc(4); ar.h2d(d_dup, np.zeros(1, dtype=np.uint32))
            ar.compact_tile_index_device(d_blob, blob, d_off, d_dup)
            ordered = not (blob[:64].view(B.COMPACT_HDR_DTYPE)[0]["flags"] & B.COMPACT_ONE_WAVE)
            rr.append(((d_blob, blob, d_off), {"d_dup": d_dup, "ordered": bool(ordered)}))
    arenas.append(ar); rounds.append(rr)
st = torch.cuda.Stream(); sh = st.cuda_stream
sched = [(i % NA, i // NA) for i in range(NA * R)]
warm = NA          # the first round of every arena, untimed
k = len(sched) - warm
snapshots = [ar.read_columns(n) for ar in arenas]


def launch(a, r):
    args, kw = rounds[a][r]
    if kernel == "packed":
        arenas[a].step_sorted_device(*args, stream=sh, **outs[a])
    else:
        arenas[a].step_compact_device(*args, stream=sh, **outs[a], **kw)


with torch.cuda.stream(st):
    for a, r in sched[:warm]:
        launch(a, r)
    torch.cuda.synchronize()
    d0 = sum(ar.debug_read().astype(np.float64) for ar in arenas)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        for a, r in sched[warm:]:
            launch(a, r)
    best = 1e9
    for rep in range(3):
        if rep:
            for ar, snap in zip(arenas, snapshots):
                ar.load_columns(snap)
            for a, r in sched[:warm]:
                launch(a, r)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(st); g.replay(); e1.record(st)
        torch.cuda.synchronize()
        best = min(best, 1e3 * e0.elapsed_time(e1) / k)
msg = f"{kernel}: {best:.2f} us per launch (best of 3 x {k} launches)"
if os.environ.get("RAFTGPU_TILE_DEBUG"):
    d = sum(ar.debug_read().astype(np.float64) for ar in arenas) - d0
    tiles = max(d[4], 1)
    msg += "; cycles per tile (tid 0 of the consumer group): wait %.0f, records %.0f, recompute %.0f, hand-off %.0f; tiles %d" % (
        d[0] / tiles, d[1] / tiles, d[2] / tiles, d[3] / tiles, tiles)
print(msg, flush=True)
