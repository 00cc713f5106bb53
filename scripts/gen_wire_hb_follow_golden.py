#!/usr/bin/env python
"""Golden vectors for the MsgHeartbeatResponse encoder of the follower's heartbeat pass (raftgpu_follower_heartbeat):
the bytes an independent protobuf encoder, python-protobuf, writes for eraftpb.Message with msg_type =
MsgHeartbeatResponse (9) and the fields handle_heartbeat and send set (raft.rs:602-661, 2452-2464): to, from, term,
commit and the context echoed from the heartbeat.  The descriptor is gen_wire_golden.py's, restating eraftpb.proto:23-92.

    python scripts/gen_wire_hb_follow_golden.py   # rewrites tests/golden/wire/heartbeat_follow.json

Every vector: {"to", "from", "term", "commit", "ctx": None (no context field at all) or the 8 context bytes as hex,
"hex": the serialized Message}.  Covered: each field zero and non-zero; to, from, term and commit at 0, 1, 127, 128,
2^32, 2^63 and 2^64 - 1; no context, and the contexts of read ids 0, 1 and 2^64 - 1 (8 bytes each, so id 0 is a
present context of 8 zero bytes)."""
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_wire_golden import build_classes  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "wire", "heartbeat_follow.json")
EDGES = [0, 1, 127, 128, 1 << 32, 1 << 63, (1 << 64) - 1]
CTXS = [None] + [x.to_bytes(8, "little") for x in (0, 1, (1 << 64) - 1)]


def main():
    Message = build_classes()
    rng = random.Random(0x4EF0)
    vectors = []

    def add(to, frm, term, commit, ctx):
        m = Message()
        m.msg_type = 9
        m.to = to
        setattr(m, "from", frm)
        m.term = term
        m.commit = commit
        if ctx is not None:
            m.context = ctx
        vectors.append({"to": to, "from": frm, "term": term, "commit": commit, "ctx": None if ctx is None else ctx.hex(),
                        "hex": m.SerializeToString().hex()})

    # 1. every field zero and non-zero, with every context form
    for mask in range(16):
        for ctx in CTXS:
            add(*[rng.choice(EDGES[1:]) if (mask >> k) & 1 else 0 for k in range(4)], ctx)
    # 2. each field at every edge value, the others small, with each context form in turn
    for field in range(4):
        for k, e in enumerate(EDGES):
            v = [rng.randint(1, 9), rng.randint(1, 9), rng.randint(1, 1 << 20), rng.randint(0, 1 << 20)]
            v[field] = e
            add(*v, CTXS[(field + k) % len(CTXS)])
    # 3. random responses as a follower sends them
    for _ in range(64):
        add(rng.choice([rng.randint(1, 9), rng.getrandbits(64)]), rng.choice([rng.randint(1, 9), rng.getrandbits(64)]),
            rng.choice([1, 7, rng.getrandbits(20), rng.getrandbits(64)]), rng.choice([0, 1, rng.getrandbits(20), rng.getrandbits(64)]),
            rng.choice([None, rng.getrandbits(64).to_bytes(8, "little")]))
    with open(OUT, "w") as f:
        json.dump({"source": "python-protobuf %s from a descriptor restating eraftpb.proto:23-92" %
                             __import__("google.protobuf").protobuf.__version__, "vectors": vectors}, f, indent=0)
    print(f"wrote {len(vectors)} vectors to {OUT}")


if __name__ == "__main__":
    main()
