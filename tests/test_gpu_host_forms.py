"""The host forms of the batch passes on the GPU: each one is admitted only while no records are enqueued for a step.
With one record enqueued, every form is refused with ERR_BUSY and changes nothing -- the columns, the votes and the
read queues stay as they were, and the caller's outputs hold only what the call writes before admission.  After the
step the same call succeeds.  Run with -m gpu."""
import ctypes as C

import numpy as np
import pytest

from helpers import B, COMPARE_COLUMNS
import hb_frames as F
import read_cases as R
import vote_frames as V

pytestmark = pytest.mark.gpu

N, P = 16, 8
JUNK = 0xAB  # every byte of an output before the call


def _out(n, dtype):
    return np.full(max(1, n) * np.dtype(dtype).itemsize, JUNK, np.uint8).view(dtype)


def _junk(x):
    return bool(np.all(x.view(np.uint8) == JUNK))


def _arena():
    """N groups with read queues, each a leader over voters {0, 1, 2} with one pending read."""
    d = R.ArenaDriver(N, P)
    for g in range(N):
        R.leader(d, g, 0b111, committed=1, last_index=3)
    d.a.read_index_request(R.reqs(*[(g, 100 + g) for g in range(N)]))
    return d.a


def _state(a):
    cols = a.read_columns(N)
    votes = [a.column_read(B.COL_VOTES, s, 0, N, np.uint8) for s in range(B.SLOTS)]
    return cols, votes, a.column_read(B.COL_TERM, 0, 0, N, np.uint64), a.read_index_read(0, N)


def _same_state(x, y):
    for name in COMPARE_COLUMNS:
        assert np.array_equal(getattr(x[0], name), getattr(y[0], name)), name
    for s in range(B.SLOTS):
        assert np.array_equal(x[1][s], y[1][s]), f"votes of slot {s}"
    assert np.array_equal(x[2], y[2]), "term"
    for name, u, v in zip(("count", "ctx", "index", "acks"), x[3], y[3]):
        assert np.array_equal(u, v), f"read queue {name}"


def _heartbeat_resp(a):
    recs = np.zeros(1, B.APPEND_RESP_DTYPE)
    recs[0] = (1, 1, B.REC_HEARTBEAT, 0, 0, 0)
    res = _out(1, np.uint8)

    def call():
        return a._L.raftgpu_heartbeat_resp(a._h, recs.ctypes.data, 1, res.ctypes.data)

    return call, lambda: _junk(res)


def _update_state(a):
    ent = np.zeros(1, B.SEND_ENTRY_DTYPE)
    ent[0] = (1, 2, 0, 0, 4)
    res = _out(1, np.uint8)

    def call():
        return a._L.raftgpu_update_state(a._h, ent.ctypes.data, 1, res.ctypes.data)

    return call, lambda: _junk(res)


def _read_index_request(a):
    reqs = R.reqs((2, 200))
    res, rel, n = _out(1, np.uint8), _out(1, B.READ_STATE_DTYPE), C.c_uint64(2**64 - 1)

    def call():
        return a._L.raftgpu_read_index_request(a._h, reqs.ctypes.data, 1, res.ctypes.data, rel.ctypes.data, 1, C.byref(n))

    return call, lambda: _junk(res) and _junk(rel) and n.value == 0


def _read_index_ack(a):
    recs = R.acks((2, 1, 102))
    rel, n = _out(P, B.READ_STATE_DTYPE), C.c_uint64(2**64 - 1)

    def call():
        return a._L.raftgpu_read_index_ack(a._h, recs.ctypes.data, 1, rel.ctypes.data, P, C.byref(n))

    return call, lambda: _junk(rel) and n.value == 0


def _read_index_recheck(a):
    groups = np.array([3], np.uint32)
    rel, n = _out(P, B.READ_STATE_DTYPE), C.c_uint64(2**64 - 1)

    def call():
        return a._L.raftgpu_read_index_recheck(a._h, groups.ctypes.data, 1, rel.ctypes.data, P, C.byref(n))

    return call, lambda: _junk(rel) and n.value == 0


def _heartbeat_wire(a):
    fb = F.Frames([F.frame(4, 1, F.message(F.HEARTBEAT_RESPONSE, term=1, context=F.ctx_bytes(104)))])
    status, rel, n = _out(1, np.uint8), _out(P, B.READ_STATE_DTYPE), C.c_uint64(2**64 - 1)

    def call():
        return a._L.raftgpu_heartbeat_wire(a._h, fb.bytes.ctypes.data, fb.n_bytes, fb.offsets.ctypes.data, 1,
                                           status.ctypes.data, rel.ctypes.data, P, C.byref(n))

    return call, lambda: _junk(status) and _junk(rel) and n.value == 0


def _heartbeat_frames(a):
    k = 4
    ids = np.arange(1, (B.SLOTS + 1) * k + 1, dtype=np.uint64).reshape(B.SLOTS + 1, k)
    blob, offs = _out(B.heartbeat_frames_bound(k), np.uint8), _out(B.SLOTS * k + 1, np.uint32)
    totals = _out(3, np.uint64)

    def call():
        return a._L.raftgpu_heartbeat_frames(a._h, 0, k, None, ids.ctypes.data, blob.ctypes.data, len(blob),
                                             offs.ctypes.data, len(offs) - 1, totals.ctypes.data)

    return call, lambda: _junk(blob) and _junk(offs) and not totals.any()


def _follower_heartbeat(a):
    fb = F.Frames([F.frame(5, 1, F.message(8, term=1, commit=1, frm=2))])  # MsgHeartbeat
    sel, ids = V.bitmap(np.ones(a.cap, bool)), np.arange(1, a.cap + 1, dtype=np.uint64)
    status, frm = _out(1, np.uint8), _out(1, np.uint64)
    resp, roff, totals = _out(B.follower_heartbeat_bound(1), np.uint8), _out(2, np.uint32), _out(2, np.uint64)

    def call():
        return a._L.raftgpu_follower_heartbeat(a._h, fb.bytes.ctypes.data, fb.n_bytes, fb.offsets.ctypes.data, 1,
                                               sel.ctypes.data, ids.ctypes.data, status.ctypes.data, frm.ctypes.data,
                                               resp.ctypes.data, len(resp), roff.ctypes.data, totals.ctypes.data)

    return call, lambda: (_junk(status) and _junk(frm) and _junk(resp) and roff[0] == 0 and _junk(roff[1:])
                          and not totals.any())


def _vote_wire(a):
    fb = F.Frames([F.frame(6, 1, V.message(V.VOTE_RESPONSE, term=1))])
    sel = V.bitmap(np.ones(N, bool))
    status, out, n = _out(1, np.uint8), _out(1, B.VOTE_OUTCOME_DTYPE), C.c_uint64(2**64 - 1)

    def call():
        return a._L.raftgpu_vote_wire(a._h, fb.bytes.ctypes.data, fb.n_bytes, fb.offsets.ctypes.data, 1, sel.ctypes.data,
                                      None, status.ctypes.data, out.ctypes.data, 1, C.byref(n))

    return call, lambda: _junk(status) and _junk(out) and n.value == 0


FORMS = [_heartbeat_resp, _update_state, _read_index_request, _read_index_ack, _read_index_recheck, _heartbeat_wire,
         _heartbeat_frames, _follower_heartbeat, _vote_wire]


@pytest.mark.parametrize("form", FORMS, ids=[f.__name__[1:] for f in FORMS])
def test_refused_while_records_are_enqueued(form):
    a = _arena()
    call, untouched = form(a)
    before = _state(a)
    recs = np.zeros(1, B.APPEND_RESP_DTYPE)
    recs[0] = (0, 1, 0, 0, 2, 0)
    a.enqueue(recs)
    assert call() == B.ERR_BUSY
    _same_state(_state(a), before)
    assert untouched(), "the refused call wrote the caller's outputs"
    a.step()
    assert call() == B.OK
    a.close()
