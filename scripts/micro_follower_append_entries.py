"""The --entries mode of micro_follower_append.py: raftgpu_follower_append_entries on n follower groups, one MsgAppend
each with k entries of `payload` data bytes at the log's tail, so every frame appends (see that script)."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from oracle import oracle as O  # noqa: E402
from oracle import app_entries_oracle as AE  # noqa: E402
from oracle import app_follow_oracle as AL  # noqa: E402
import app_entries as E  # noqa: E402
import app_follow as A  # noqa: E402
import hb_frames as F  # noqa: E402


def main(B, n, runs, k, payload, rng):
    ar = B.Arena(n)   # RaftGpuError(ERR_NO_DEVICE) without a GPU: no fallback
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                          str(ar.info.device)], capture_output=True, text=True).stdout.strip()
    ar.group_alloc_range(n)
    terms = rng.integers(1, 1 << 33, n).astype(np.uint64)
    last = rng.integers(1 << 20, 1 << 40, n).astype(np.uint64)
    committed = last - rng.integers(0, 100, n).astype(np.uint64)
    for col, arr in ((B.COL_TERM, terms), (B.COL_LAST_INDEX, last), (B.COL_COMMITTED, committed),
                     (B.COL_TERM_START, np.full(n, B.NO_TERM_START, np.uint64))):
        ar.column_write(col, 0, 0, arr)
    table = np.zeros(n, AL.LOG_DTYPE)
    table["id"], table["flags"] = rng.integers(1, 1 << 20, n, dtype=np.uint64), AL.SELECT
    table["run_start"], table["run_term"] = last - np.minimum(last, np.uint64(10)), terms
    data = bytes(payload * [0x5A])
    order = rng.permutation(n)
    frames = []
    for g in order.tolist():
        t, i = int(terms[g]), int(last[g])
        recs = [E.record(E.entry(t, i + 1 + j, data=data)) for j in range(k)]
        frames.append(A.frame(g, 1, E.message(t, t, i, i + k, int(rng.integers(1, 1 << 40)), recs)))
    blob, off = A.batch(frames)
    del frames

    c = O.new_columns(n, n)
    c.term_start[:], c.term[:], c.last_index[:], c.committed[:] = B.NO_TERM_START, terms, last, committed
    st_o, _, _, _, _, tot_o, t_oracle = AE.batch(c, None, table.copy(), blob, off, bench=True)
    assert np.all(st_o == (B.WIRE_OK << 4 | B.RES_OK | B.FAPP_APPENDED))

    bound = B.follower_append_bound(n)
    bufs = [ar.device_alloc(x) for x in (len(blob) + 16, 4 * (n + 1), table.nbytes, n, 8 * n, 40 * n, bound,
                                         4 * (n + 1), 16)]
    d_b, d_o, d_t, d_st, d_f, d_ap, d_rb, d_ro, d_tot = bufs
    ar.h2d(d_b, blob), ar.h2d(d_o, off)
    L, h = ar._L, ar._h
    stream = torch.cuda.Stream()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t_dev = []
    for r in range(runs + 2):   # the first two runs warm up; every pass starts from the same state
        ar.h2d(d_t, table)
        ar.column_write(B.COL_LAST_INDEX, 0, 0, last)
        ar.column_write(B.COL_COMMITTED, 0, 0, committed)
        ar.synchronize()
        ev0.record(stream)
        rc = L.raftgpu_follower_append_entries_device(h, stream.cuda_stream, d_b, len(blob), d_o, n, d_t, d_st, d_f, d_ap,
                                                      d_rb, bound, d_ro, d_tot)
        ev1.record(stream)
        assert rc == B.OK, rc
        stream.synchronize()
        if r >= 2:
            t_dev.append(ev0.elapsed_time(ev1) * 1e-3)
    tot, st = np.zeros(2, np.uint64), np.zeros(n, np.uint8)
    ar.d2h(tot, d_tot), ar.d2h(st, d_st)
    assert np.array_equal(st, st_o) and tot.tolist() == tot_o.tolist(), (tot, tot_o)
    for p in bufs:
        ar.device_free(p)

    hb = F.Frames([])
    hb.bytes, hb.offsets, hb.n, hb.n_bytes = np.concatenate([blob, np.zeros(16, np.uint8)]), off, n, len(blob)
    t_host = []
    for r in range(5):
        ar.column_write(B.COL_LAST_INDEX, 0, 0, last)
        ar.column_write(B.COL_COMMITTED, 0, 0, committed)
        tb = table.copy()
        t0 = time.perf_counter()
        got = ar.follower_append_entries(hb, tb)
        t_host.append(time.perf_counter() - t0)
        assert np.array_equal(got[0], st_o)

    def us(t):
        a = np.array(t) * 1e6
        return f"{np.median(a):.1f} us (range {a.min():.1f}-{a.max():.1f})"

    print(f"GPU: {gpu}")
    print(f"{n} follower groups, one MsgAppend each with {k} entries of {payload} data bytes (shuffled), "
          f"{len(blob) / n:.1f} bytes per frame in, {int(tot[1]) / n:.1f} per response out")
    print(f"raftgpu_follower_append_entries_device: {us(t_dev)} over {runs} passes between CUDA events")
    print(f"raftgpu_follower_append_entries (host form, end to end): {us(t_host)} over 5 calls")
    print(f"C batch oracle (aeo_batch, one thread): {t_oracle * 1e3:.1f} ms over the same batch")
