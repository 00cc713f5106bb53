"""Wire batches at the edges of the prologue every wire-frame pass shares (k_wire.cuh: wire_stage_block, wire_open,
wire_decode): the stage rule restated, ballast frames that place a batch's blocks on both sides of the 16 KiB stage,
hostile offset layouts, and the golden decoder vectors retargeted to another message type.  Pure numpy: the CPU tests
check what these batches reach, the GPU tests (test_gpu_wire_batches.py) run them."""
import json
import os

import numpy as np

import hb_frames as F

THREADS, STAGE = 256, 16 * 1024            # kWireThreads, kWireStage
STAGED, SPAN, ORDER, PAST = "staged", "span", "order", "past"
MSG_APPEND, MSG_SNAPSHOT = 3, 7            # the ballast types: SKIP_TYPE in every pass
HERE = os.path.dirname(os.path.abspath(__file__))


def stage_blocks(offsets, n_bytes):
    """wire_stage_block for every block of 256 frames: STAGED when offsets[first] <= offsets[last] <= n_bytes and
    offsets[last] - (offsets[first] & ~15) <= 16384, else why not -- ORDER, PAST or SPAN, checked in that order."""
    off = np.asarray(offsets, np.int64)
    n = len(off) - 1
    out = []
    for first in range(0, n, THREADS):
        lo, hi = int(off[first]), int(off[min(first + THREADS, n)])
        out.append(ORDER if lo > hi else PAST if hi > n_bytes else SPAN if hi - (lo & ~15) > STAGE else STAGED)
    return out


def geometry(offsets, n_bytes):
    """The stage geometries a batch reaches: the set of stage_blocks' verdicts, plus ("span", span, lo % 16, staged) for
    blocks that span exactly 16384 or 16385 bytes, "partial" for a last block of fewer than 256 frames, and "frame>16K" /
    "frame>64K" for frames (inside the batch) that long."""
    off = np.asarray(offsets, np.int64)
    n = len(off) - 1
    got = set(stage_blocks(off, n_bytes))
    for first in range(0, n, THREADS):
        lo, hi = int(off[first]), int(off[min(first + THREADS, n)])
        if hi - (lo & ~15) in (STAGE, STAGE + 1):
            got.add(("span", hi - (lo & ~15), lo % 16, hi - (lo & ~15) <= STAGE))
    if n % THREADS:
        got.add("partial")
    sizes = np.diff(off)[(np.diff(off) > 0) & (off[1:] <= n_bytes)]
    if (sizes > STAGE).any():
        got.add("frame>16K")
    if (sizes > 64 * 1024).any():
        got.add("frame>64K")
    return got


# every geometry the GPU tests must reach (the stage rule's four verdicts, both sides of its span limit at both ends of
# a 16-byte line, a partial last block and frames past 16 KiB and 64 KiB)
WANT_GEOMETRY = {STAGED, SPAN, ORDER, PAST, "partial", "frame>16K", "frame>64K"} | \
    {("span", s, r, s == STAGE) for s in (STAGE, STAGE + 1) for r in (0, 15)}


def _payload(k):
    return (np.arange(k, dtype=np.int64) * 37 % 251).astype(np.uint8).tobytes()


def ballast(size, kind=MSG_APPEND, group=0):
    """A frame of exactly `size` (>= 8) bytes, header included, naming `group` slot 0: a MsgAppend whose entries field
    (7) holds the bytes, or a MsgSnapshot whose snapshot field (9) does.  Every pass skips it (SKIP_TYPE)."""
    field = 7 if kind == MSG_APPEND else 9
    for pad in (b"", F.varint(6 << 3) + b"\x01"):      # index = 1 bridges the sizes a longer length varint skips
        head = bytes([0x08, kind]) + pad + F.varint(field << 3 | 2)
        for vl in (1, 2, 3, 4):
            p = size - 4 - len(head) - vl
            if p >= 0 and len(F.varint(p)) == vl:
                return F.frame(group, 0, head + F.varint(p) + _payload(p))
    raise ValueError(size)


def across_the_stage(frames, rng, group=0):
    """The frames in order with ballast frames interleaved so that the batch reaches WANT_GEOMETRY's valid geometries:
    blocks spanning exactly 16384 and 16385 bytes from offsets[first] % 16 = 0 and 15 (each after a staged block whose
    last frame is the ballast that sets that residue), a block holding a frame past 16 KiB, one holding a frame past
    64 KiB, small ballast frames everywhere else, and a partial last block -> (frames, ballast mask)."""
    out, mask, it = [], [], iter(frames)
    pos = 0

    def put(f, is_ballast):
        nonlocal pos
        out.append(f)
        mask.append(is_ballast)
        pos += len(f)

    def take(k):
        got = [next(it) for _ in range(k)]
        return got, sum(len(f) for f in got)

    def block(kind, size_of):
        """255 scenario frames and one ballast frame at a random place in the block, sized by size_of(bytes of the 255)"""
        got, nb = take(THREADS - 1)
        at = int(rng.integers(0, THREADS))
        for f in got[:at] + [None] + got[at:]:
            put(ballast(size_of(nb), kind, group) if f is None else f, f is None)

    for k, (span, r) in enumerate([(STAGE, 0), (STAGE, 15), (STAGE + 1, 0), (STAGE + 1, 15), (None, 0), (None, 1)]):
        got, nb = take(THREADS - 1)                    # a staged block that ends on the residue r
        for f in got:
            put(f, False)
        put(ballast(24 + (r - pos - 24) % 16, MSG_SNAPSHOT, group), True)
        assert pos % 16 == r
        kind = MSG_APPEND if k % 2 else MSG_SNAPSHOT
        if span is not None:
            block(kind, lambda nb: span - r - nb)
        else:                                          # one frame past 16 KiB, or past 64 KiB
            big = STAGE + 1 if r == 0 else 64 * 1024 + 1
            block(kind, lambda nb: big + int(rng.integers(0, 4096)))
    for f in it:
        put(f, False)
        if rng.random() < 0.02:
            put(ballast(int(rng.integers(8, 400)), int(rng.choice([MSG_APPEND, MSG_SNAPSHOT])), group), True)
    if len(out) % THREADS == 0:
        put(ballast(40, MSG_APPEND, group), True)
    return out, np.array(mask, bool)


def slack(frames, at_least=4096):
    """Valid frames of at least `at_least` bytes, for the bytes a device buffer holds past n_bytes -> (bytes, the frame
    boundaries relative to n_bytes)."""
    got, nb = [], 0
    for f in frames:
        if nb >= at_least:
            break
        got.append(f)
        nb += len(f)
    assert nb >= at_least
    return b"".join(got), np.concatenate([[0], np.cumsum([len(f) for f in got])]).astype(np.int64)


def hostile(frames, rng, n, residue, past):
    """n frames over a batch of n_bytes = residue (mod 16) bytes, with a valid frame and some bytes before offsets[0],
    descending offset pairs, frames of 0 to 3 bytes and frames that end past n_bytes.  past: the offsets past n_bytes a
    frame may use, relative to n_bytes and > 0 (the boundaries of the valid frames of `slack`, or the bytes the host
    form copies in after the batch).  The last offset is past n_bytes when residue // 4 is 0, below offsets[0] when it
    is 1 -> (blob of n_bytes bytes, offsets u32[n + 1])."""
    frames = [frames[k % len(frames)] for k in range(n + 1)]
    body = frames[1:]
    nb = len(frames[0]) + sum(len(f) for f in body)
    prefix = frames[0] + bytes(int(rng.integers(0, 16)) * 16 + (residue - nb) % 16)
    blob = np.frombuffer(prefix + b"".join(body), np.uint8).copy()
    n_bytes = len(blob)
    assert n_bytes % 16 == residue
    off = np.concatenate([[len(prefix)], len(prefix) + np.cumsum([len(f) for f in body])]).astype(np.int64)
    past = np.asarray([p for p in past if p > 0], np.int64)
    edits = rng.choice(n, max(1, n // 12), replace=False) if n > 1 else [0]
    for i in edits:
        kind = int(rng.integers(3)) if n > 1 else residue % 3
        if kind == 0:          # a frame of 0 to 3 bytes (the next one starts inside this one's bytes)
            off[i + 1] = min(off[i] + int(rng.integers(0, 4)), n_bytes)
        elif kind == 1:        # a descending pair
            off[i + 1] = max(0, off[i] - int(rng.integers(1, 64)))
        elif i + 1 < n:        # a frame from a slack boundary to the next one, past n_bytes
            k = int(rng.integers(0, len(past) - 1))
            off[i], off[i + 1] = n_bytes + past[k] if k else off[i], n_bytes + past[k + 1]
    if residue // 4 == 0:
        off[n] = n_bytes + int(past[-1])
    elif residue // 4 == 1:
        off[n] = off[0] - 1
    assert off.min() >= 0 and off.max() <= n_bytes + past.max()
    return blob, off.astype(np.uint32)


def hostile_cases():
    """(n, residue) of the hostile batches: every residue of n_bytes mod 16, n cycling through 1, 255, 256 and 257."""
    return [((1, 255, 256, 257)[r % 4], r) for r in range(16)]


# --------------------------------------------------------------------------- the golden decoder vectors


def golden():
    with open(os.path.join(HERE, "golden", "wire", "messages.json")) as f:
        return json.load(f)["vectors"]


def retarget(vector, msg_type):
    """A messages.json vector as a message of type msg_type: an accepted one gets 0x08 <type> appended (field 1 is a
    scalar, so the last value wins and every other field keeps python-protobuf's verdict), a rejected one stays as it
    is -> (Message bytes, its fields with msg_type replaced, or None for a rejected vector)."""
    raw = bytes.fromhex(vector["hex"])
    if not vector["ok"]:
        return raw, None
    return raw + bytes([0x08, msg_type]), dict(vector["fields"], msg_type=msg_type)
