"""Follower runs (DESIGN 3.22) on the device: raftgpu_follower_append[_entries]_device on arenas with and without
follower runs.  Device time from CUDA events, median and range over `runs` passes after two warm-up passes, the arena
state reloaded before each pass; the card's name and power limit read in the same run.

  steady  n followers, one MsgAppend each with one 128-byte entry at the log's tail (the accept path never reads a
          row), on an arena without follower runs and one with them, alternated pass by pass;
  reject  n diverged followers (log runs at terms 2, 4, 6; the table states the last) answer the new leader's first
          probe (log_term 7, 5 or 3, a third each): the share decided with 0, 1 and 2 stated runs, and the time;
  probe   the leader's next probe inside run 1 (term 4) or inside run 2 (term 2), half each, with three entries at
          term 5 and the leader's own at term 8: the log is truncated inside run 1 or run 2; the share decided and the
          time.
The C batch oracle (fro_batch, one thread) runs over the same batches.

    python scripts/micro_follower_runs.py [--n 1000000] [--runs 20]
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from helpers import B  # noqa: E402
from oracle import app_follow_oracle as AL  # noqa: E402
from oracle import follower_runs_oracle as FR  # noqa: E402
from oracle import oracle as O  # noqa: E402
import app_entries as E  # noqa: E402
import app_follow as A  # noqa: E402


def arena(n, runs, cols):
    ar = B.Arena(n)  # RaftGpuError(ERR_NO_DEVICE) without a GPU: no fallback
    if runs:
        ar.enable_follower_runs()
    ar.group_alloc_range(n)
    for col, arr in cols.items():
        ar.column_write(col, 0, 0, arr)
    return ar


class Pass:
    """One device form over one batch on one arena, with its buffers; time() = seconds of one pass between events."""

    def __init__(self, ar, entries, blob, off, table, cols):
        self.ar, self.entries, self.table, self.cols, self.n = ar, entries, table, cols, len(off) - 1
        self.n_bytes = len(blob)
        n = self.n
        self.bound = B.follower_append_bound(n)
        self.bufs = [ar.device_alloc(x) for x in (len(blob) + 16, 4 * (n + 1), table.nbytes, n, 8 * n, 40 * n,
                                                  self.bound, 4 * (n + 1), 16)]
        ar.h2d(self.bufs[0], blob), ar.h2d(self.bufs[1], off)
        self.stream = torch.cuda.Stream()
        self.ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def time(self, rows=None):
        ar, (d_b, d_o, d_t, d_st, d_f, d_ap, d_rb, d_ro, d_tot) = self.ar, self.bufs
        ar.h2d(d_t, self.table)
        for col, arr in self.cols.items():
            ar.column_write(col, 0, 0, arr)
        if rows is not None:
            ar.follower_runs_set(rows)
        ar.synchronize()
        self.ev[0].record(self.stream)
        if self.entries:
            rc = ar._L.raftgpu_follower_append_entries_device(ar._h, self.stream.cuda_stream, d_b, self.n_bytes, d_o,
                                                              self.n, d_t, d_st, d_f, d_ap, d_rb, self.bound, d_ro, d_tot)
        else:
            rc = ar._L.raftgpu_follower_append_device(ar._h, self.stream.cuda_stream, d_b, self.n_bytes, d_o, self.n,
                                                      d_t, d_st, d_f, d_rb, self.bound, d_ro, d_tot)
        self.ev[1].record(self.stream)
        assert rc == B.OK, rc
        self.stream.synchronize()
        return self.ev[0].elapsed_time(self.ev[1]) * 1e-3

    def status(self):
        st = np.zeros(self.n, np.uint8)
        self.ar.d2h(st, self.bufs[3])
        return st


def us(t):
    a = np.array(t) * 1e6
    return f"{np.median(a):.1f} us (range {a.min():.1f}-{a.max():.1f})"


def steady(n, runs, rng):
    terms = rng.integers(1, 1 << 33, n).astype(np.uint64)
    last = rng.integers(1 << 20, 1 << 40, n).astype(np.uint64)
    committed = last - rng.integers(0, 100, n).astype(np.uint64)
    cols = {B.COL_TERM: terms, B.COL_LAST_INDEX: last, B.COL_COMMITTED: committed,
            B.COL_TERM_START: np.full(n, B.NO_TERM_START, np.uint64)}
    table = np.zeros(n, AL.LOG_DTYPE)
    table["id"], table["flags"] = rng.integers(1, 1 << 20, n, dtype=np.uint64), AL.SELECT
    table["run_start"], table["run_term"] = last - np.uint64(10), terms
    data = bytes(128 * [0x5A])
    frames = [A.frame(g, 1, E.message(int(terms[g]), int(terms[g]), int(last[g]), int(last[g]) + 1, 7,
                                      [E.record(E.entry(int(terms[g]), int(last[g]) + 1, data=data))]))
              for g in rng.permutation(n).tolist()]
    blob, off = A.batch(frames)
    del frames
    rows = FR.rows_for(n)
    rows["anchor_start"], rows["anchor_term"] = table["run_start"], terms
    rows["run_start"][:, 0], rows["run_term"][:, 0] = 1, 1
    passes = [Pass(arena(n, r, cols), True, blob, off, table, cols) for r in (False, True)]
    passes[1].ar.follower_runs_set(rows)
    t = [[], []]
    for r in range(runs + 2):
        for k, p in enumerate(passes):
            x = p.time()
            if r >= 2:
                t[k].append(x)
    for p in passes:
        assert np.all(p.status() == (B.WIRE_OK << 4 | B.RES_OK | B.FAPP_APPENDED))
    secs = []
    for r in (None, rows):
        cc = O.new_columns(n, n)
        cc.term_start[:], cc.term[:], cc.last_index[:], cc.committed[:] = B.NO_TERM_START, terms, last, committed
        secs.append(FR.batch(cc, None, table.copy(), None if r is None else r.copy(), blob, off, True, bench=True)[-1])
    print(f"steady accepts, {n} followers, one 128-byte entry each: without follower runs {us(t[0])}, "
          f"with {us(t[1])}; C batch oracle (one thread) {secs[0] * 1e3:.1f} ms without rows, {secs[1] * 1e3:.1f} ms with")
    for p in passes:
        for b in p.bufs:
            p.ar.device_free(b)
        del p.ar


def burst(n, runs, rng):
    a = rng.integers(10, 1000, n).astype(np.uint64)
    b = a + rng.integers(2, 100, n).astype(np.uint64)
    c = b + rng.integers(1, 100, n).astype(np.uint64)
    L = b + np.uint64(1) + (rng.random(n) * (c - b).astype(np.float64)).astype(np.uint64)
    lt = rng.choice(np.array([7, 5, 3], np.uint64), n)
    term = np.uint64(8)
    cols = {B.COL_TERM: np.full(n, term, np.uint64), B.COL_LAST_INDEX: c, B.COL_COMMITTED: a // np.uint64(2),
            B.COL_TERM_START: np.full(n, B.NO_TERM_START, np.uint64)}
    table = np.zeros(n, AL.LOG_DTYPE)
    table["id"], table["flags"] = np.arange(1, n + 1, dtype=np.uint64), AL.SELECT
    table["run_start"], table["run_term"] = b + np.uint64(1), 6
    rows = []
    for k in range(3):
        r = FR.rows_for(n)
        r["anchor_start"], r["anchor_term"] = b + np.uint64(1), 6
        if k >= 1:
            r["run_start"][:, 0], r["run_term"][:, 0] = a + np.uint64(1), 4
        if k >= 2:
            r["run_start"][:, 1], r["run_term"][:, 1] = 1, 2
        rows.append(r)
    order = rng.permutation(n).tolist()
    rej = [A.frame(g, 1, A.message(3, term=8, log_term=int(lt[g]), index=int(L[g]), commit=int(a[g]) // 2, frm=1))
           for g in order]
    # a cut strictly inside run 1 ([a + 1, b]) or run 2 ([1, a]): m.index below the run's end, the entries' terms new
    in1 = rng.random(n) < 0.5
    at = np.where(in1, a + np.uint64(1) + (rng.random(n) * (b - a - np.uint64(1)).astype(np.float64)).astype(np.uint64),
                 a // np.uint64(2) + (rng.random(n) * (a - a // np.uint64(2)).astype(np.float64)).astype(np.uint64))
    probe = [A.frame(g, 1, E.message(8, 4 if in1[g] else 2, int(at[g]), int(a[g]) // 2, 1,
                                     [E.record(E.entry(5, int(at[g]) + 1 + j, data=bytes(16))) for j in range(3)] +
                                     [E.record(E.entry(8, int(at[g]) + 4, data=bytes(16)))]))
             for g in order]
    ar = arena(n, True, cols)
    for name, frames, entries in (("rejection", rej, False), ("next probe (cut inside run 1 or run 2)", probe, True)):
        blob, off = A.batch(frames)
        p = Pass(ar, entries, blob, off, table, cols)
        for k in range(3):
            t = []
            for r in range(runs + 2):
                x = p.time(rows[k])
                if r >= 2:
                    t.append(x)
            st = p.status()
            cc = O.new_columns(n, n)
            cc.term_start[:] = B.NO_TERM_START
            cc.term[:], cc.last_index[:], cc.committed[:] = term, c, a // np.uint64(2)
            res = FR.batch(cc, None, table.copy(), rows[k].copy(), blob, off, entries, bench=True)
            assert np.array_equal(res[0], st)
            share = float(np.mean(st >> 4 == B.WIRE_OK))
            print(f"{name} batch, {n} diverged followers, {k} stated runs: {share:.3f} decided on the device; "
                  f"device {us(t)}; C batch oracle (one thread) {res[-1] * 1e3:.1f} ms")
        for x in p.bufs:
            ar.device_free(x)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--runs", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device: there is no CPU measurement")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    print(f"GPU: {gpu}")
    rng = np.random.default_rng(1)
    steady(args.n, args.runs, rng)
    burst(args.n, args.runs, rng)


if __name__ == "__main__":
    main()
