#!/usr/bin/env python
"""Golden vectors for the MsgHeartbeat encoder (raftgpu_heartbeat_frames): the bytes an independent protobuf encoder,
python-protobuf, writes for eraftpb.Message with msg_type = MsgHeartbeat (8) and the fields send_heartbeat and send set
(raft.rs:602-661, 822-844): to, from, term, commit and the context.  The descriptor is gen_wire_golden.py's, restating
eraftpb.proto:23-92.  A heartbeat that carries read id x has the 8 bytes of x, little-endian, as its context; id 0 is
no context.

    python scripts/gen_wire_heartbeat_golden.py   # rewrites tests/golden/wire/heartbeats.json

Every vector: {"to", "from", "term", "commit", "ctx": the read id or None (no context field at all), "hex": the
serialized Message}.  Covered: each field zero and non-zero; ids and terms at 1, 127, 128, 2^32, 2^63 and 2^64 - 1;
commit 0 and 2^64 - 1; no context, and read ids 0, 1 and 2^64 - 1."""
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_wire_golden import build_classes  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "wire", "heartbeats.json")
EDGES = [1, 127, 128, 1 << 32, 1 << 63, (1 << 64) - 1]
CTXS = [None, 0, 1, (1 << 64) - 1]


def main():
    Message = build_classes()
    rng = random.Random(0x4EA28)
    vectors = []

    def add(to, frm, term, commit, ctx):
        m = Message()
        m.msg_type = 8
        m.to = to
        setattr(m, "from", frm)
        m.term = term
        m.commit = commit
        if ctx:  # id 0 is no context
            m.context = ctx.to_bytes(8, "little")
        vectors.append({"to": to, "from": frm, "term": term, "commit": commit, "ctx": ctx, "hex": m.SerializeToString().hex()})

    # 1. every field zero and non-zero, with every context form
    for mask in range(16):
        for ctx in CTXS:
            v = [rng.choice(EDGES) if (mask >> k) & 1 else 0 for k in range(4)]
            add(*v, ctx)
    # 2. each of to, from, term at every edge value; commit 0 and 2^64 - 1
    for field in range(3):
        for e in EDGES:
            for commit in (0, (1 << 64) - 1):
                v = [rng.randint(1, 9), rng.randint(1, 9), rng.randint(1, 1 << 20)]
                v[field] = e
                add(*v, commit, CTXS[(e + commit) % len(CTXS)])
    # 3. random heartbeats as a leader sends them
    for _ in range(64):
        add(rng.choice([rng.randint(1, 9), rng.getrandbits(64)]), rng.choice([rng.randint(1, 9), rng.getrandbits(64)]),
            rng.choice([1, 7, rng.getrandbits(20), rng.getrandbits(64)]), rng.choice([0, 1, rng.getrandbits(20), rng.getrandbits(64)]),
            rng.choice([None, 0, rng.getrandbits(64)]))
    with open(OUT, "w") as f:
        json.dump({"source": "python-protobuf %s from a descriptor restating eraftpb.proto:23-92" %
                             __import__("google.protobuf").protobuf.__version__, "vectors": vectors}, f, indent=0)
    print(f"wrote {len(vectors)} vectors to {OUT}")


if __name__ == "__main__":
    main()
