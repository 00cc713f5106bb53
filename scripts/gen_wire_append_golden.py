#!/usr/bin/env python
"""Golden vectors for the entry-less MsgAppend encoder (raftgpu_append_frames): the bytes an independent protobuf
encoder, python-protobuf, writes for eraftpb.Message with msg_type = MsgAppend (3) and the fields prepare_send_entries
and send set when there are no entries (raft.rs:602-661, 714-730): to, from, term, log_term, index and commit.  The
descriptor is gen_wire_golden.py's, restating eraftpb.proto:23-92 (Message: eraftpb.proto:71-92).

    python scripts/gen_wire_append_golden.py   # rewrites tests/golden/wire/appends.json

Every vector: {"to", "from", "term", "log_term", "index", "commit", "hex": the serialized Message}.  Covered: each field
zero and non-zero; every field at 0, 1, 127, 128, 2^32, 2^63 and 2^64 - 1; log_term 0 and index 0 with the others set."""
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_wire_golden import build_classes  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "wire", "appends.json")
EDGES = [0, 1, 127, 128, 1 << 32, 1 << 63, (1 << 64) - 1]
FIELDS = ("to", "from", "term", "log_term", "index", "commit")


def main():
    Message = build_classes()
    rng = random.Random(0xA99E)
    vectors = []

    def add(*vals):
        m = Message()
        m.msg_type = 3
        for name, v in zip(FIELDS, vals):
            setattr(m, name, v)
        vectors.append(dict(zip(FIELDS, vals), hex=m.SerializeToString().hex()))

    # 1. every field zero and non-zero
    for mask in range(64):
        add(*[rng.choice(EDGES[1:]) if (mask >> k) & 1 else 0 for k in range(6)])
    # 2. each field at every edge value, the others small or large
    for field in range(6):
        for e in EDGES:
            v = [rng.choice([rng.randint(1, 9), rng.getrandbits(64) or 1]) for _ in range(6)]
            v[field] = e
            add(*v)
    # 3. as the commit broadcast sends them: index = next_idx - 1, log_term = term at last_index, 0 above it
    for _ in range(64):
        term, last = rng.choice([1, 7, rng.getrandbits(20), rng.getrandbits(64)]), rng.choice([0, 5, rng.getrandbits(40)])
        index = last + rng.choice([0, 0, 1, rng.getrandbits(16)])
        add(rng.randint(1, 9), rng.randint(1, 9), term, term if index <= last else 0, index, rng.randint(0, index))
    with open(OUT, "w") as f:
        json.dump({"source": "python-protobuf %s from a descriptor restating eraftpb.proto:23-92" %
                             __import__("google.protobuf").protobuf.__version__, "vectors": vectors}, f, indent=0)
    print(f"wrote {len(vectors)} vectors to {OUT}")


if __name__ == "__main__":
    main()
