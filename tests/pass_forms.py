"""Both forms of every wire pass from one table: device(a, name, ...) runs raftgpu_<name>_device over buffers from
raftgpu_device_alloc, host(a, name, ...) the host form over the same batch, and refusals(a, name, ...) holds the
buffers of a test that checks what the device form refuses before it launches anything."""
import contextlib
import types

import numpy as np

from helpers import B
import hb_frames as F

ST = (("st", np.uint8, ()),)
OUT = (("out", np.uint64, (2,)),)
FROM = (("f", np.uint64, ()),)
REPLY = ("rb", "cap", "ro", "t")       # response bytes, their capacity, response offsets, totals u64[2]
LISTED = ("out", "cap", "c")           # a list, its capacity, its length u64[1]
STATUS_SENTINEL, COUNT_SENTINEL = 0xEE, 77


def _frame_pass(tables, outs, tail=(), bound=None, listed=None, updates_table=False):
    """tables: (argument name, dtype) of the inputs after n; outs: (argument name, dtype, shape per frame) of the outputs
    with one row per frame; tail: REPLY (capacity bound(n)) or LISTED (listed = (dtype, capacity(a, n)))."""
    args = ("b", "nb", "o", "n") + tuple(t for t, _ in tables) + tuple(o for o, _, _ in outs) + tail
    return types.SimpleNamespace(args=args, tables=tables, outs=outs, tail=tail, bound=bound, listed=listed,
                                 updates_table=updates_table)


VOTERS, LOG = (("v", B.VOTER_DTYPE),), (("l", B.FOLLOWER_LOG_DTYPE),)
PASSES = {
    "wire_apply": _frame_pass((), ST),
    "heartbeat_wire": _frame_pass((), ST, LISTED,
                                  listed=(B.READ_STATE_DTYPE, lambda a, n: n * getattr(a, "read_max_pending", 0))),
    "vote_wire": _frame_pass((("s", np.uint32), ("p", np.uint32)), ST, LISTED,
                             listed=(B.VOTE_OUTCOME_DTYPE, lambda a, n: min(n, a.get_info().n_alloc))),
    "vote_request_wire": _frame_pass(VOTERS, ST + OUT, REPLY, B.vote_request_wire_bound),
    "follower_heartbeat": _frame_pass((("s", np.uint32), ("i", np.uint64)), ST + FROM, REPLY, B.follower_heartbeat_bound),
    "follower_term_wire": _frame_pass(VOTERS, ST + OUT, REPLY, B.follower_term_wire_bound),
    "leader_term_wire": _frame_pass(VOTERS, ST + OUT, REPLY, B.follower_term_wire_bound),
    "follower_append": _frame_pass(LOG, ST + FROM, REPLY, B.follower_append_bound),
    "follower_append_entries": _frame_pass(LOG, ST + FROM + (("ap", B.FOLLOWER_APPENDED_DTYPE, ()),), REPLY,
                                           B.follower_append_bound, updates_table=True),
}
# The broadcast passes build frames for groups [first, first + n) from ids u64[9][n] and a select bitmap: the bound of
# their bytes, the words of their totals, and whether they list the sends that need the log (append_frames' rest).
BROADCASTS = {"heartbeat_frames": (B.heartbeat_frames_bound, 3, False),
              "append_frames": (B.append_frames_bound, 4, True)}


@contextlib.contextmanager
def device_buffers(a):
    """Yields put(nbytes, data=None, fill=None): a device buffer of at least nbytes (and 16) bytes holding data, or
    filled with the array fill; every buffer is freed on the way out."""
    ptrs = []

    def put(nbytes, data=None, fill=None):
        ptrs.append(a.device_alloc(max(16, int(nbytes))))
        for x in (data, fill):
            if x is not None and x.nbytes:
                a.h2d(ptrs[-1], x)
        return ptrs[-1]

    try:
        yield put
    finally:
        for p in ptrs:
            a.device_free(p)


def _args(a, put, p, blob, off, tables, n_bytes, capacity, sentinel):
    """The device form's arguments by name, over buffers from put; the status and the count / totals hold the refusal
    sentinels when sentinel is set."""
    n, off = len(off) - 1, np.ascontiguousarray(off, np.uint32)
    blob = np.concatenate([np.asarray(blob, np.uint8), np.zeros(16, np.uint8)])
    d = {"b": put(len(blob), blob), "nb": len(blob) - 16 if n_bytes is None else n_bytes, "o": put(off.nbytes, off), "n": n}
    for (name, dt), x in zip(p.tables, tables):
        d[name] = None if x is None else put(max(64, np.asarray(x).nbytes), np.ascontiguousarray(x, dt))
    for name, dt, shape in p.outs:
        fill = np.full(n, STATUS_SENTINEL, np.uint8) if sentinel and name == "st" else None
        d[name] = put(np.dtype(dt).itemsize * int(np.prod(shape)) * max(1, n), fill=fill)
    words = {REPLY: 2, LISTED: 1}.get(p.tail, 0)
    count = np.full(words, COUNT_SENTINEL, np.uint64) if sentinel else None
    if p.tail == REPLY:
        cap = p.bound(n) if capacity is None else capacity
        d.update(rb=put(cap + 64), cap=cap, ro=put(4 * (n + 1)), t=put(8 * words, fill=count))
    elif p.tail == LISTED:
        cap = p.listed[1](a, n) if capacity is None else capacity
        d.update(out=put(p.listed[0].itemsize * max(1, cap)), cap=cap, c=put(8 * words, fill=count))
    return d


def _read(a, d2h_arr, ptr):
    if d2h_arr.size:
        a.d2h(d2h_arr, ptr)
    return d2h_arr


def device(a, name, blob, off, *tables, n_bytes=None, capacity=None):
    """raftgpu_<name>_device over the batch (blob followed by 16 zero bytes on the device; n_bytes: all of blob by
    default) and the tables in the C function's order -> the per-frame outputs, then (response blob, response offsets,
    totals) for a reply pass or the listed outputs for vote_wire / heartbeat_wire.  follower_append_entries updates its
    table in place from the device's copy."""
    p = PASSES[name]
    with device_buffers(a) as put:
        d = _args(a, put, p, blob, off, tables, n_bytes, capacity, False)
        getattr(a, name + "_device")(*[d[k] for k in p.args])
        a.synchronize()
        n = d["n"]
        got = [_read(a, np.zeros((n,) + shape, dt), d[k]) for k, dt, shape in p.outs]
        if p.updates_table and tables[0].nbytes:
            a.d2h(tables[0], d["l"])
        if p.tail == REPLY:
            tot = _read(a, np.zeros(2, np.uint64), d["t"])
            got += [_read(a, np.zeros(int(tot[1]), np.uint8), d["rb"]),
                    _read(a, np.zeros(int(tot[0]) + 1, np.uint32), d["ro"]), tot]
        elif p.tail == LISTED:
            cnt = _read(a, np.zeros(1, np.uint64), d["c"])
            got.append(_read(a, np.zeros(int(cnt[0]), p.listed[0]), d["out"]))
    return tuple(got)


def host_batch(blob, off, n_bytes=None):
    """What the host forms read: .bytes (the batch and 16 spare bytes), .n_bytes, .offsets, .n, no records."""
    n_bytes = len(blob) if n_bytes is None else n_bytes
    fb = F.Frames([])
    fb.bytes = np.concatenate([np.asarray(blob[:n_bytes], np.uint8), np.zeros(16, np.uint8)])
    fb.offsets, fb.n, fb.n_bytes = np.ascontiguousarray(off, np.uint32), len(off) - 1, int(n_bytes)
    return fb


def host(a, name, blob, off, *tables, n_bytes=None):
    """The host form (Arena.<name>) over host_batch(blob, off, n_bytes)."""
    return getattr(a, name)(host_batch(blob, off, n_bytes), *tables)


def run(a, name, blob, off, *tables, device, n_bytes=None):
    """The device form when device is set, else the host form."""
    return _FORMS[device](a, name, blob, off, *tables, n_bytes=n_bytes)


_FORMS = {True: device, False: host}


def split(blob, off):
    return [blob[a:b].tobytes() for a, b in zip(off[:-1].tolist(), off[1:].tolist())]


def equal(want, got, names, what):
    for w, g, name in zip(want, got, names):
        assert w.shape == g.shape and np.array_equal(w, g), (what, name, np.flatnonzero(w != g)[:5] if w.shape == g.shape
                                                              else (w.shape, g.shape))


def broadcast(a, name, first, n, ids, select, bytes_capacity=None, frames_capacity=None, rest_capacity=None):
    """raftgpu_<name>_device for heartbeat_frames / append_frames with the outputs sized at the bound -> (blob, offsets,
    [rest,] totals)."""
    bound, words, rest = BROADCASTS[name]
    with device_buffers(a) as put:
        d_ids, d_bytes, d_off = put(max(8, ids.nbytes), ids), put(bound(n)), put(4 * (8 * n + 1))
        d_rest, d_tot = put(16 * 8 * n) if rest else None, put(8 * words)
        d_sel = put(select.nbytes, select) if select is not None else None
        caps = [bound(n) if bytes_capacity is None else bytes_capacity, 8 * n if frames_capacity is None else frames_capacity]
        args = [first, n, d_sel, d_ids, d_bytes, caps[0], d_off, caps[1]]
        if rest:
            args += [d_rest, 8 * n if rest_capacity is None else rest_capacity]
        getattr(a, name + "_device")(*args, d_tot)
        a.synchronize()
        tot = _read(a, np.zeros(words, np.uint64), d_tot)
        got = [_read(a, np.zeros(int(tot[1]), np.uint8), d_bytes), _read(a, np.zeros(int(tot[0]) + 1, np.uint32), d_off)]
        if rest:
            got.append(_read(a, np.zeros(int(tot[2]), B.SEND_ENTRY_DTYPE), d_rest))
    return (*got, tot)


@contextlib.contextmanager
def refusals(a, name, blob, off, *tables, n_bytes=None, capacity=None):
    """Buffers for the device form over the batch, its status filled with STATUS_SENTINEL and its count / totals with
    COUNT_SENTINEL -> r: r.args, the arguments by name; r.call(**overrides), the raw C function's return code with the
    named arguments replaced; r.read(name, arr), an output read back; r.untouched(), whether the sentinels are still
    there (nothing was launched).  The buffers are freed on the way out."""
    p = PASSES[name]
    fn = getattr(a._L, "raftgpu_" + name + "_device")
    words = {REPLY: 2, LISTED: 1}[p.tail]
    count = {REPLY: "t", LISTED: "c"}[p.tail]
    with device_buffers(a) as put:
        d = _args(a, put, p, blob, off, tables, n_bytes, capacity, True)

        def read(k, arr):
            a.synchronize()
            a.d2h(arr, d[k])
            return arr

        def untouched():
            st, cnt = read("st", np.zeros(d["n"], np.uint8)), read(count, np.zeros(words, np.uint64))
            return bool(np.all(st == STATUS_SENTINEL)) and cnt.tolist() == [COUNT_SENTINEL] * words

        yield types.SimpleNamespace(args=d, read=read, untouched=untouched,
                                    call=lambda **k: fn(a._h, None, *[k.get(x, d[x]) for x in p.args]))
