#!/usr/bin/env python
"""Golden vectors for the stale replies of raftgpu_follower_term_wire and for the frames it reads: the bytes an
independent protobuf encoder, python-protobuf, writes for eraftpb.Message.  The descriptor is gen_wire_golden.py's,
restating eraftpb.proto:23-92.

    python scripts/gen_wire_follower_term_golden.py   # rewrites tests/golden/wire/follower_terms.json

"replies": {"to", "from", "term", "hex"}: the empty MsgAppendResponse (4) of raft.rs:1375-1376, every field at 0, 1,
127, 128, 2^32, 2^63 and 2^64 - 1 in every combination.
"frames": {"msg_type", "from", "term", "commit", "hex"}: MsgAppend (3) and MsgHeartbeat (8) with from and term at those
values, for the decoder's msg_type, from and term."""
import itertools
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_wire_golden import build_classes  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "wire", "follower_terms.json")
EDGES = [0, 1, 127, 128, 1 << 32, 1 << 63, (1 << 64) - 1]


def main():
    Message = build_classes()
    rng = random.Random(0xF7E8)
    replies, frames = [], []
    for to, frm, term in itertools.product(EDGES, EDGES, EDGES):
        m = Message()
        m.msg_type, m.to, m.term = 4, to, term
        setattr(m, "from", frm)
        replies.append({"to": to, "from": frm, "term": term, "hex": m.SerializeToString().hex()})
    for msg_type in (3, 8):
        for frm, term in itertools.product(EDGES, EDGES):
            m = Message()
            m.msg_type, m.to, m.term = msg_type, rng.choice(EDGES[1:]), term
            setattr(m, "from", frm)
            m.commit = rng.choice(EDGES)
            if msg_type == 3:
                m.log_term, m.index = rng.choice(EDGES), rng.choice(EDGES)
            frames.append({"msg_type": msg_type, "from": frm, "term": term, "commit": m.commit,
                           "hex": m.SerializeToString().hex()})
    with open(OUT, "w") as f:
        json.dump({"source": "python-protobuf %s from a descriptor restating eraftpb.proto:23-92" %
                             __import__("google.protobuf").protobuf.__version__,
                   "replies": replies, "frames": frames}, f, indent=0)
    print(f"wrote {len(replies)} replies and {len(frames)} frames to {OUT}")


if __name__ == "__main__":
    main()
