#!/usr/bin/env python
"""Golden vectors for the follower's MsgAppendResponse encoder (raftgpu_follower_append) and for its entries flag: the
bytes an independent protobuf encoder, python-protobuf, writes for eraftpb.Message.  The descriptor is
gen_wire_golden.py's, restating eraftpb.proto:23-92.

    python scripts/gen_wire_append_resp_golden.py   # rewrites tests/golden/wire/append_responses.json

"responses": {"to", "from", "term", "log_term", "index", "commit", "reject", "reject_hint", "hex"} with msg_type 4 and
the fields handle_append_entries sets (raft.rs:2389-2448).  Covered: each field zero and non-zero; every field at 0, 1,
127, 128, 2^32, 2^63 and 2^64 - 1; reject with reject_hint 0 and log_term 0.
"appends": {"term", "log_term", "index", "commit", "entries": [[term, index], ..], "hex"}: MsgAppend (3) with 0, 1 and 3
entries, an empty Entry included, for the decoder's field-7 flag."""
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_wire_golden import build_classes  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "wire", "append_responses.json")
EDGES = [0, 1, 127, 128, 1 << 32, 1 << 63, (1 << 64) - 1]
FIELDS = ("to", "from", "term", "log_term", "index", "commit", "reject", "reject_hint")


def main():
    Message = build_classes()
    rng = random.Random(0xA99F)
    responses, appends = [], []

    def add(*vals):
        m = Message()
        m.msg_type = 4
        for name, v in zip(FIELDS, vals):
            setattr(m, name, bool(v) if name == "reject" else v)
        responses.append(dict(zip(FIELDS, [int(v) for v in vals]), hex=m.SerializeToString().hex()))

    big = lambda: rng.choice([rng.randint(1, 9), rng.getrandbits(64) or 1])
    # 1. every field zero and non-zero
    for mask in range(256):
        add(*[(1 if k == 6 else rng.choice(EDGES[1:])) if (mask >> k) & 1 else 0 for k in range(8)])
    # 2. each field at every edge value, the others small or large
    for field in range(8):
        for e in (EDGES if field != 6 else [0, 1]):
            v = [big() for _ in range(8)]
            v[6] = rng.randint(0, 1)
            v[field] = e
            add(*v)
    # 3. rejections with reject_hint 0 and log_term 0
    for _ in range(16):
        add(big(), big(), big(), 0, big(), big(), 1, 0)
    add(big(), big(), big(), 0, 0, 0, 1, 0)
    # MsgAppend with 0, 1 and 3 entries (an empty Entry among them)
    for k in (0, 1, 1, 3, 3):
        for empty in (False, True):
            m = Message()
            m.msg_type = 3
            m.term, m.log_term, m.index, m.commit = big(), big(), big(), big()
            ents = []
            for j in range(k):
                e = m.entries.add()
                if not (empty and j == k // 2):
                    e.term, e.index = big(), m.index + j + 1
                ents.append([e.term, e.index])
            appends.append({"term": m.term, "log_term": m.log_term, "index": m.index, "commit": m.commit, "entries": ents,
                            "hex": m.SerializeToString().hex()})
    with open(OUT, "w") as f:
        json.dump({"source": "python-protobuf %s from a descriptor restating eraftpb.proto:23-92" %
                             __import__("google.protobuf").protobuf.__version__,
                   "responses": responses, "appends": appends}, f, indent=0)
    print(f"wrote {len(responses)} responses and {len(appends)} appends to {OUT}")


if __name__ == "__main__":
    main()
