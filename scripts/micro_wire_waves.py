"""Micro-benchmark: the wire step and the follower's append pass at raftgpu_arena_set_wire_waves (DESIGN 3.19),
device-resident batches, CUDA events, median (range) of 20 passes:
  1. the wire step, 1M leaders x 4 followers, k in {1, 2, 4} accept frames per cell: k calls at waves = 1 (one frame per
     cell each) against one call at waves = k (all of them, in arrival order);
  2. raftgpu_follower_append_entries_device, 1M follower groups, k in {1, 2, 4} pipelined frames of 1 entry x 128 B each,
     compared the same way;
  3. the cost of waves that find nothing: a batch with one frame per cell at waves in {1, 4, 16, 64}.
Also the wave oracle (oracle/wire_waves_oracle.c) on one core for item 1.  Every frame of a batch has the same layout
(indexes with 3-byte varints), so the batches are built with numpy.  Prints the card and its power limit."""
import importlib, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
pkg = importlib.import_module("raft-rs_b200")
B = pkg.binding
from oracle import oracle as O
from oracle import app_follow_oracle as AL
from oracle import wire_waves_oracle as WW

n = int(os.environ.get("N", 1_000_000))
P, TERM, L0 = 5, 5, 1 << 15                                       # L0 + small: 3-byte varints
PASSES = 20


def v3(x):
    """x (array, 2^14 <= x < 2^21) as 3-byte varints -> (len, 3) u8."""
    x = np.asarray(x, np.uint64)
    return np.stack([(x & 0x7F) | 0x80, ((x >> 7) & 0x7F) | 0x80, x >> 14], axis=1).astype(np.uint8)


def frames_to_batch(rows):
    """(N, w) u8 frames of one width -> (blob, offsets)."""
    N, w = rows.shape
    return rows.reshape(-1).copy(), (np.arange(N + 1, dtype=np.uint64) * w).astype(np.uint32)


def accepts(k):
    """k accept frames per (group, slot 1..4) cell, round-major (arrival order): round j at index L0 + j."""
    g = np.tile(np.repeat(np.arange(n, dtype=np.uint32), P - 1), k)
    s = np.tile(np.tile(np.arange(1, P, dtype=np.uint32), n), k)
    j = np.repeat(np.arange(k), n * (P - 1))
    hdr = (g << 4 | s).astype("<u4").view(np.uint8).reshape(-1, 4)
    fixed = np.array([0x08, 4, 0x10, 1, 0x18, 0, 0x20, TERM, 0x30], np.uint8)
    rows = np.concatenate([hdr, np.tile(fixed, (len(g), 1)), v3(L0 + j)], axis=1)
    rows[:, 9] = s + 1                                           # from
    return frames_to_batch(rows)


def appends(k, data=128):
    """k pipelined MsgAppend frames per follower group, round-major: round j at index L0 + j with one entry L0 + j + 1 of
    `data` bytes, commit L0 + j."""
    g = np.tile(np.arange(n, dtype=np.uint32), k)
    j = np.repeat(np.arange(k), n)
    idx = L0 + j
    hdr = (g << 4).astype("<u4").view(np.uint8).reshape(-1, 4)
    ent = 2 + 4 + 3 + data                                       # term, index, data (2-byte length) = 137
    head = np.array([0x08, 3, 0x10, 2, 0x18, 1, 0x20, TERM, 0x28, TERM, 0x30], np.uint8)
    N = len(g)
    parts = [hdr, np.tile(head, (N, 1)), v3(idx),
             np.tile(np.array([0x3A, (ent & 0x7F) | 0x80, ent >> 7, 0x10, TERM, 0x18], np.uint8), (N, 1)), v3(idx + 1),
             np.tile(np.array([0x22, (data & 0x7F) | 0x80, data >> 7], np.uint8), (N, 1)), np.full((N, data), 0xAB, np.uint8),
             np.tile(np.array([0x40], np.uint8), (N, 1)), v3(idx)]
    return frames_to_batch(np.concatenate(parts, axis=1))


def fmt(us):
    return f"{np.median(us):.1f} us ({min(us):.1f}-{max(us):.1f})"


class Dev:
    """A batch in device memory for one arena."""

    def __init__(self, a, blob, off):
        self.a, self.n = a, len(off) - 1
        nb = (len(blob) + 15) & ~15
        self.d_b, self.d_o = a.device_alloc(nb + 16), a.device_alloc(4 * len(off))
        buf = np.zeros(nb, np.uint8)
        buf[: len(blob)] = blob
        a.h2d(self.d_b, buf), a.h2d(self.d_o, off)
        self.n_bytes = len(blob)

    def free(self):
        self.a.device_free(self.d_b), self.a.device_free(self.d_o)


def timed(st, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(st):
        e0.record(st); fn(); e1.record(st)
    st.synchronize()
    return 1e3 * e0.elapsed_time(e1)


try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
except OSError:
    q = "nvidia-smi unavailable"
print(f"card: {torch.cuda.get_device_name(0)}; nvidia-smi: {q}")
st = torch.cuda.Stream()
sp = st.cuda_stream

# ---- 1 + 3: the wire step
c = O.new_columns(n, n)
c.term[:n], c.term_start[:n], c.last_index[:n] = TERM, L0 - 100, L0 + 64
c.meta[:n] = O.make_meta((1 << P) - 1, self_slot=0)
for s in range(1, P):
    c.matched[s, :n], c.next_idx[s, :n] = L0 - 1, L0
    c.pflags[s, :n] = B.STATE_REPLICATE
la = B.Arena(n)
la.group_alloc_range(n)
la.column_write(B.COL_TERM, 0, 0, c.term[:n].copy())
d_st = la.device_alloc(4 * n * (P - 1) + 16)
for k in (1, 2, 4):
    blob, off = accepts(k)
    m = n * (P - 1)                                              # frames per round, 16 bytes each
    rounds = [Dev(la, blob[j * m * 16:(j + 1) * m * 16].copy(), off[: m + 1].copy()) for j in range(k)]
    full = Dev(la, blob, off)
    us1, usk = [], []
    for p in range(2 * PASSES + 2):
        la.load_columns(c)
        if p % 2 == 0:
            la.set_wire_waves(1)
            us1.append(timed(st, lambda: [la.wire_apply_device(r.d_b, r.n_bytes, r.d_o, r.n, d_st, stream=sp) for r in rounds]))
        else:
            la.set_wire_waves(k)
            usk.append(timed(st, lambda: la.wire_apply_device(full.d_b, full.n_bytes, full.d_o, full.n, d_st, stream=sp)))
    stt = np.zeros(full.n, np.uint8)
    la.d2h(stt, d_st)
    assert (stt >> 4 == B.WIRE_OK).all()
    print(f"wire step, {n} x {P - 1} cells, k = {k}: {k} calls at waves 1 {fmt(us1[1:])}; one call at waves {k} "
          f"{fmt(usk[1:])}")
    ref = O.copy_columns(c)
    _, secs = WW.leader(ref, None, *accepts(k), k, bench=True)
    print(f"  wave oracle, one core, waves {k}: {1e6 * secs:.0f} us")
    for r in rounds + [full]:
        r.free()
one = Dev(la, *accepts(1))
line = []
for waves in (1, 4, 16, 64):
    la.set_wire_waves(waves)
    us = [timed(st, lambda: la.wire_apply_device(one.d_b, one.n_bytes, one.d_o, one.n, d_st, stream=sp))
          for _ in range(PASSES + 1)]
    line.append(f"waves {waves} {fmt(us[1:])}")
print(f"wire step, one frame per cell ({one.n} frames): " + "; ".join(line))
one.free()
la.close()

# ---- 2: the follower's pass with entries
fa = B.Arena(n)
fa.group_alloc_range(n)
fc_last = np.full(n, L0, np.uint64)
table = np.zeros(n, AL.LOG_DTYPE)
table["id"], table["flags"], table["run_start"], table["run_term"] = 2, AL.SELECT, 1, TERM


def follower_state():
    fa.column_write(B.COL_TERM, 0, 0, np.full(n, TERM, np.uint64))
    fa.column_write(B.COL_LAST_INDEX, 0, 0, fc_last)
    fa.column_write(B.COL_COMMITTED, 0, 0, fc_last - 1)
    fa.column_write(B.COL_TERM_START, 0, 0, np.full(n, (1 << 64) - 1, np.uint64))
    fa.h2d(d_t, table)


kmax = 4
d_t = fa.device_alloc(table.nbytes)
d_fst, d_f, d_ap = fa.device_alloc(kmax * n + 16), fa.device_alloc(8 * kmax * n), fa.device_alloc(40 * kmax * n)
bound = B.follower_append_bound(kmax * n)
d_rb, d_ro, d_tot = fa.device_alloc(bound), fa.device_alloc(4 * (kmax * n + 1)), fa.device_alloc(16)


def follow(d):
    fa.follower_append_entries_device(d.d_b, d.n_bytes, d.d_o, d.n, d_t, d_fst, d_f, d_ap, d_rb,
                                      B.follower_append_bound(d.n), d_ro, d_tot, stream=sp)


for k in (1, 2, 4):
    blob, off = appends(k)
    w = len(blob) // (k * n)
    rounds = []
    for j in range(k):
        rounds.append(Dev(fa, blob[j * n * w:(j + 1) * n * w].copy(), off[: n + 1].copy()))
    full = Dev(fa, blob, off)
    us1, usk = [], []
    for p in range(2 * PASSES + 2):
        follower_state()
        fa.synchronize()
        if p % 2 == 0:
            fa.set_wire_waves(1)
            us1.append(timed(st, lambda: [follow(r) for r in rounds]))
        else:
            fa.set_wire_waves(k)
            usk.append(timed(st, lambda: follow(full)))
    tot = np.zeros(2, np.uint64)
    fa.d2h(tot, d_tot)
    assert int(tot[0]) == k * n, tot
    print(f"follower append with entries, {n} groups, k = {k} frames of 1 x 128 B ({w} B each): {k} calls at waves 1 "
          f"{fmt(us1[1:])}; one call at waves {k} {fmt(usk[1:])}")
    for r in rounds + [full]:
        r.free()
fa.close()
