#!/usr/bin/env python
"""Golden vectors for the MsgHeartbeatResponse wire decode (raftgpu_heartbeat_wire): the scalar fields and the context.

Like scripts/gen_wire_golden.py, the verdicts come from an independent implementation of the published format,
python-protobuf, over the same descriptor restating eraftpb.proto:23-92.  A heartbeat that carries read id x has the
8 bytes of x, little-endian, as its context, and the follower echoes it (raft.rs:2461).

    python scripts/gen_wire_hb_golden.py          # rewrites tests/golden/wire/heartbeat_responses.json

Every vector: {"kind", "hex": serialized bytes, "ok": python-protobuf parsed it, "fields": the scalar fields,
"context": the context's hex (None when not ok)}.  Covered: canonical responses with contexts of length 0, 8 and
others and ids 0, 1, 2^64 - 1; a repeated context field (the last wins); field 12 sent as a varint (an unknown field:
the context stays empty); unknown fields; other message types that carry a context; truncated lengths."""
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_wire_golden import build_classes, fields_of, varint  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "wire", "heartbeat_responses.json")


def ctx_field(data: bytes) -> bytes:
    return varint(12 << 3 | 2) + varint(len(data)) + data


def main():
    Message = build_classes()
    rng = random.Random(0x4EA27)
    vectors = []

    def add(kind, raw):
        m = Message()
        try:
            m.ParseFromString(raw)
            ok = True
        except Exception:
            ok = False
        f = fields_of(m) if ok else None
        if f:
            f["msg_type"] &= 0xFFFFFFFF
        vectors.append({"kind": kind, "hex": raw.hex(), "ok": ok, "fields": f, "context": m.context.hex() if ok else None})

    ids = [0, 1, 2, 255, 256, 1 << 32, (1 << 63), (1 << 64) - 1]
    # 1. canonical responses (what handle_heartbeat sends: to, term, commit, the echoed context)
    for k in range(96):
        m = Message()
        m.msg_type = 9
        m.to = rng.randint(1, 9)
        setattr(m, "from", rng.randint(1, 9))
        m.term = rng.choice([1, 7, rng.randint(1, 1 << 20)])
        m.commit = rng.choice([0, 1, rng.getrandbits(20), rng.getrandbits(64)])
        r = k % 4
        if r == 1:
            m.context = (ids[(k // 4) % len(ids)] if k < 40 else rng.getrandbits(64)).to_bytes(8, "little")
        elif r == 2:
            m.context = rng.randbytes(rng.choice([1, 7, 9, 16, 33]))
        elif r == 3:
            m.context = rng.getrandbits(64).to_bytes(8, "little")
        add("canonical", m.SerializeToString())
    # 2. a repeated context field: the last occurrence wins, whatever the lengths
    base = varint(1 << 3) + varint(9) + varint(4 << 3) + varint(7) + varint(8 << 3) + varint(99)
    for a, b in [(8, 8), (8, 0), (0, 8), (3, 8), (8, 12), (8, 8)]:
        add("repeated_context", base + ctx_field(rng.randbytes(a)) + varint(8 << 3) + varint(5) + ctx_field(rng.randbytes(b)))
    # 3. field 12 as a varint: an unknown field for a parser, the context stays as it was
    add("context_varint", base + varint(12 << 3 | 0) + varint(8))
    add("context_varint", base + ctx_field((5).to_bytes(8, "little")) + varint(12 << 3 | 0) + varint(1 << 40))
    add("context_varint", base + varint(12 << 3 | 0) + varint(3) + ctx_field((6).to_bytes(8, "little")))
    # 4. unknown fields of every wire type around a context
    for k in range(12):
        parts = [varint(1 << 3) + varint(9), varint(4 << 3) + varint(rng.randint(1, 9)), varint(8 << 3) + varint(rng.getrandbits(30)),
                 ctx_field(rng.getrandbits(64).to_bytes(8, "little") if k % 3 else rng.randbytes(rng.randint(0, 12)))]
        for _ in range(rng.randint(1, 3)):
            no, wt = rng.choice([16, 17, 100, 1000, 536870911]), rng.choice([0, 1, 2, 5])
            body = {0: varint(rng.getrandbits(40)), 1: rng.randbytes(8), 5: rng.randbytes(4)}.get(wt)
            if wt == 2:
                blob = rng.randbytes(rng.randint(0, 20))
                body = varint(len(blob)) + blob
            parts.insert(rng.randint(0, len(parts)), varint(no << 3 | wt) + body)
        add("unknown_fields", b"".join(parts))
    # 5. other message types carrying a context (MsgHeartbeat, MsgReadIndex, MsgReadIndexResp, MsgAppendResponse, ...)
    for t in [8, 15, 16, 4, 0, 3, 18]:
        m = Message()
        m.msg_type = t
        m.term, m.commit, m.index = 7, rng.getrandbits(20), rng.getrandbits(20)
        m.context = rng.getrandbits(64).to_bytes(8, "little")
        add("other_type", m.SerializeToString())
    # 6. truncated and overlong lengths, python-protobuf's verdict as is
    ctx8 = (1234).to_bytes(8, "little")
    for raw in [base + varint(12 << 3 | 2) + varint(8) + ctx8[:5],          # length runs past the end
                base + varint(12 << 3 | 2) + varint(9) + ctx8,              # one byte short
                base + varint(12 << 3 | 2),                                  # tag without length
                base + varint(12 << 3 | 2) + b"\x88",                        # truncated length varint
                base + varint(12 << 3 | 2) + b"\x88\x80\x80\x80\x80\x80\x80\x80\x80\x80\x00" + ctx8,   # 11-byte length
                base + varint(12 << 3 | 2) + b"\x88\x00" + ctx8,             # over-long but legal length (2 bytes)
                (base + ctx_field(ctx8))[:-1],                               # the frame cut one byte early
                varint(1 << 3) + varint(9) + varint(12 << 3 | 2) + b"\xff\xff\xff\xff\x0f"]:   # huge length
        add("truncated", raw)
    with open(OUT, "w") as f:
        json.dump({"source": "python-protobuf %s from a descriptor restating eraftpb.proto:23-92" %
                             __import__("google.protobuf").protobuf.__version__, "vectors": vectors}, f, indent=0)
    print(f"wrote {len(vectors)} vectors to {OUT}")


if __name__ == "__main__":
    main()
