#!/usr/bin/env python
"""Golden vectors for the vote-response encoders of the vote pass's tests and bench input (tests/vote_frames.py and
raftgpu_synth_wire_encode_votes): the bytes an independent protobuf encoder, python-protobuf, writes for eraftpb.Message
with msg_type = MsgRequestVoteResponse (6) or MsgRequestPreVoteResponse (18) and the fields a voter sets
(raft.rs:1413-1470, 602-661): to, from, term, reject, commit and commit_term.  The descriptor is gen_wire_golden.py's,
restating eraftpb.proto:23-92.

    python scripts/gen_wire_vote_golden.py   # rewrites tests/golden/wire/vote_responses.json

Every vector: {"msg_type", "to", "from", "term", "reject", "commit", "commit_term", "hex": the serialized Message}.
Covered: both types, reject on and off, and term, commit and commit_term each at 0, 1, 127, 128, 2^32 and 2^64 - 1."""
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_wire_golden import build_classes  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "wire", "vote_responses.json")
EDGES = [0, 1, 127, 128, 1 << 32, (1 << 64) - 1]


def main():
    Message = build_classes()
    rng = random.Random(0x5E7E)
    vectors = []

    def add(msg_type, to, frm, term, reject, commit, commit_term):
        m = Message()
        m.msg_type = msg_type
        m.to = to
        setattr(m, "from", frm)
        m.term = term
        m.reject = reject
        m.commit = commit
        m.commit_term = commit_term
        vectors.append({"msg_type": msg_type, "to": to, "from": frm, "term": term, "reject": reject, "commit": commit,
                        "commit_term": commit_term, "hex": m.SerializeToString().hex()})

    # 1. both types, reject on and off, term / commit / commit_term over every edge combination
    for msg_type in (6, 18):
        for reject in (False, True):
            for term in EDGES:
                for commit in EDGES:
                    for commit_term in EDGES:
                        add(msg_type, rng.choice([0, 1, rng.getrandbits(64)]), rng.choice([0, 2, rng.getrandbits(64)]),
                            term, reject, commit, commit_term)
    # 2. random responses as voters send them
    for _ in range(64):
        add(rng.choice([6, 18]), rng.randint(1, 9), rng.randint(1, 9), rng.getrandbits(rng.choice([8, 20, 64])),
            rng.random() < 0.3, rng.choice([0, rng.getrandbits(20)]), rng.choice([0, rng.getrandbits(16)]))
    with open(OUT, "w") as f:
        json.dump({"source": "python-protobuf %s from a descriptor restating eraftpb.proto:23-92" %
                             __import__("google.protobuf").protobuf.__version__, "vectors": vectors}, f, indent=0)
    print(f"wrote {len(vectors)} vectors to {OUT}")


if __name__ == "__main__":
    main()
