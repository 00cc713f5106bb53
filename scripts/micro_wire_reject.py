"""Micro-benchmark: the wire step on arenas with leader runs (DESIGN 3.18), 1M leaders x 5 peers (4 followers each),
device-resident batches through raftgpu_wire_apply_device, CUDA events, median (range) of 20 passes:
  - an all-accept batch on an arena with runs and on one without, alternated in one run (the accept path of the <true>
    kernels against the <false> ones);
  - a batch where every follower rejects with log_term > 0 after an election, decided on the device from 2 stated runs;
  - the oracle's batch form (oracle/leader_runs_oracle.c) on one core for the same rejection batch.
Also the share of the rejections decided at 0, 1 and 2 stated runs.  Prints the card and its power limit."""
import importlib, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
pkg = importlib.import_module("raft-rs_b200")
B = pkg.binding
from oracle import oracle as O
from oracle import leader_runs_oracle as LR

n = int(os.environ.get("N", 1_000_000))
P = 5
rng = np.random.default_rng(1)
# leaders after an election: terms t0 < t1 < t2 < term; runs of 1-8 entries; every follower lags or diverges
runs_len = rng.integers(1, 9, size=(n, 4)).astype(np.uint64)
t = np.cumsum(rng.integers(1, 4, size=(n, 4)), axis=1).astype(np.uint64)
last = runs_len.sum(axis=1)
ts = last - runs_len[:, 3] + 1
rs0 = ts - runs_len[:, 2]
rs1 = rs0 - runs_len[:, 1]
c = O.new_columns(n, n)
c.term[:n], c.term_start[:n], c.last_index[:n] = t[:, 3], ts, last
c.meta[:n] = O.make_meta((1 << P) - 1, self_slot=0)
for s in range(P):
    c.next_idx[s, :n] = last + 1
rows = np.zeros(n, LR.ROW_DTYPE)
rows["group"] = np.arange(n)
rows["term"], rows["term_start"] = t[:, 3], ts
rows["run_start"][:, 0], rows["run_start"][:, 1] = rs0, rs1
rows["run_term"][:, 0], rows["run_term"][:, 1] = t[:, 2], t[:, 1]


def varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80); v >>= 7
    out.append(v)
    return bytes(out)


def resp(g, s, term, index, reject=False, hint=0, lt=0):
    body = b"".join(varint(no << 3) + varint(v) for no, v in ((1, 4), (2, 1), (3, s + 1), (4, term), (5, lt), (6, index),
                                                              (10, int(reject)), (11, hint)) if v)
    return np.array([g << 4 | s], "<u4").tobytes() + body


def batch(kind):
    frames = []
    for g in range(n):
        for s in range(1, P):
            if kind == "accept":
                frames.append(resp(g, s, int(t[g, 3]), int(last[g])))
            else:  # the follower's last term is one of the leader's earlier terms, or a term between them
                lt = int(t[g, rng.integers(0, 3)]) - int(rng.integers(0, 2))
                frames.append(resp(g, s, int(t[g, 3]), int(last[g]), True, int(last[g]) - int(rng.integers(0, 4)), max(lt, 1)))
    blob = np.frombuffer(b"".join(frames), np.uint8).copy()
    off = np.concatenate([[0], np.cumsum([len(f) for f in frames])]).astype(np.uint32)
    return blob, off


def arena(runs):
    a = B.Arena(n)
    if runs:
        a.enable_leader_runs()
    a.group_alloc_range(n); a.load_columns(c); a.column_write(B.COL_TERM, 0, 0, c.term[:n].copy())
    if runs:
        assert (a.leader_runs_set(rows) == 0).all()
    return a


def upload(a, blob, off):
    nb = (len(blob) + 15) & ~15
    d_b, d_o, d_s = a.device_alloc(nb + 16), a.device_alloc(4 * len(off)), a.device_alloc(len(off))
    buf = np.zeros(nb, np.uint8); buf[: len(blob)] = blob
    a.h2d(d_b, buf); a.h2d(d_o, off)
    return d_b, len(blob), d_o, len(off) - 1, d_s


def time_pass(a, args, st):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(st):
        e0.record(st); a.wire_apply_device(*args, stream=st.cuda_stream); e1.record(st)
    st.synchronize()
    return 1e3 * e0.elapsed_time(e1)


def fmt(us):
    return f"{np.median(us):.1f} us ({min(us):.1f}-{max(us):.1f})"


try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
except OSError:
    q = "nvidia-smi unavailable"
print(f"card: {torch.cuda.get_device_name(0)}; nvidia-smi: {q}")
st = torch.cuda.Stream()
acc = batch("accept")
ar, a0 = arena(True), arena(False)
xr, x0 = upload(ar, *acc), upload(a0, *acc)
us_r, us_0 = [], []
for k in range(22):  # the accepts change nothing after the first pass; alternated, the first two dropped
    (us_r if k % 2 == 0 else us_0).append(time_pass(ar if k % 2 == 0 else a0, xr if k % 2 == 0 else x0, st))
print(f"all-accept, {len(acc[1]) - 1} frames ({len(acc[0])} bytes): with runs {fmt(us_r[1:])}, without {fmt(us_0[1:])}")
rej = batch("reject")
shares = []
for k in range(3):
    rk = rows.copy()
    if k < 2:
        rk["run_start"][:, k:] = 0
        rk["run_term"][:, k:] = 0
    s, _, _, _ = LR.decode_batch(c, rk, *rej)
    shares.append(float((s == O.WIRE_OK).mean()))
print("rejections decided at 0, 1, 2 stated runs: " + ", ".join(f"{100 * x:.1f}%" for x in shares))
us = []
for k in range(20):  # a fresh arena state each pass: the next_idx the batch probes at
    ar.load_columns(c)
    xr2 = upload(ar, *rej)
    us.append(time_pass(ar, xr2, st))
    stt = np.zeros(len(rej[1]) - 1, np.uint8); ar.d2h(stt, xr2[4])
    for p in (xr2[0], xr2[2], xr2[4]):
        ar.device_free(p)
want, _, _, _ = LR.decode_batch(c, rows, *rej)
assert np.array_equal(stt >> 4, want), "device statuses differ from the oracle's"
print(f"all-reject after an election, {len(rej[1]) - 1} frames, {100 * (want == 0).mean():.1f}% decided: "
      f"device {fmt(us)}")
secs = LR.bench(c, rows, *rej, iters=3)
print(f"oracle batch form, one core, same batch: {1e6 * secs:.0f} us")
