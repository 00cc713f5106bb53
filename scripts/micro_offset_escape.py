"""What escaped offsets cost the fused step: step_tile_kernel on cfg3 (1M groups x 5 peers, 4 arenas rotated, R rounds
each, one CUDA graph, CUDA events, as micro_tile.py) where a fraction p of the follower cells start with
next_idx - matched in (2^15, 2^31).  Such a next_idx fits a 32-bit offset but not a 16-bit one (k_common.cuh): at 16
bits the cell's records take the general path, whose exact values are dependent HBM loads.  P="0,0.01,0.1" by default;
prints the GPU name and power limit."""
import importlib, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np, torch
B = importlib.import_module("raft-rs_b200").binding
from oracle import oracle as O

n = int(os.environ.get("N", 1_000_000))
R = int(os.environ.get("R", 6))
P = [float(x) for x in os.environ.get("P", "0,0.01,0.1").split(",")]
NA = 4
try:
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
except FileNotFoundError:
    print("nvidia-smi not found", flush=True)
pack_buf = np.empty((7 * n + 64, 2), dtype=np.uint64)


def far_next(c, rng, p):
    """next_idx of a fraction p of the present follower cells moved 2^15 + 1 .. 2^31 - 1 past matched."""
    meta = c.meta[:n].astype(np.int64)
    slot = np.arange(O.SLOTS)[:, None]
    present = (((meta | meta >> 8 | meta >> 16) & 0xff) >> slot) & 1 == 1
    own = ((meta & O.META_HAS_SELF) != 0) & (((meta >> 24) & 7) == slot)
    pick = present & ~own & (rng.random((O.SLOTS, n)) < p)
    far = c.matched[:, :n] + rng.integers((1 << 15) + 1, 1 << 31, (O.SLOTS, n)).astype(np.uint64)
    c.next_idx[:, :n] = np.where(pick, far, c.next_idx[:, :n])
    return np.count_nonzero(pick) / max(np.count_nonzero(present & ~own), 1)


for p in P:
    arenas, rounds, outs, snapshots, frac = [], [], [], [], []
    for a in range(NA):
        s = B.Synth(n, 0x5EED0003 + 0x100 * a, k_peers=5)
        init = O.copy_columns(s.initial)
        frac.append(far_next(init, np.random.default_rng(a), p))
        ar = B.Arena(n, n_rings=1, ring_records=4096)
        ar.group_alloc_range(n)
        ar.load_columns(init)
        outs.append({"d_adv": ar.device_alloc(4 * ((n + 31) // 32 + 1)), "d_commit": ar.device_alloc(8 * n)})
        rr = []
        for _ in range(R):
            k = ar.pack_records(s.next_round(), pack_buf)
            d = ar.device_alloc(16 * k); ar.h2d(d, pack_buf[:k])
            off = B.tile_index(pack_buf, k, n)
            do = ar.device_alloc(off.nbytes); ar.h2d(do, off)
            rr.append((d, k, do))
        arenas.append(ar); rounds.append(rr); snapshots.append(init)
    st = torch.cuda.Stream(); sh = st.cuda_stream
    sched = [(i % NA, i // NA) for i in range(NA * R)]
    warm = NA
    k = len(sched) - warm
    with torch.cuda.stream(st):
        for a, r in sched[:warm]:
            arenas[a].step_sorted_device(*rounds[a][r], stream=sh, **outs[a])
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for a, r in sched[warm:]:
                arenas[a].step_sorted_device(*rounds[a][r], stream=sh, **outs[a])
        best = 1e9
        for rep in range(3):
            if rep:
                for ar, snap in zip(arenas, snapshots):
                    ar.load_columns(snap)
                for a, r in sched[:warm]:
                    arenas[a].step_sorted_device(*rounds[a][r], stream=sh, **outs[a])
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(st); g.replay(); e1.record(st)
            torch.cuda.synchronize()
            best = min(best, 1e3 * e0.elapsed_time(e1) / k)
    print(f"p = {p:g} ({100 * np.mean(frac):.2f} % of follower cells far ahead): {best:.2f} us per launch "
          f"(best of 3 x {k} launches)", flush=True)
    del g
    for ar in arenas:
        ar.close()
