#!/usr/bin/env python
"""Golden vectors for the vote-request encoders of the voter pass's tests and bench input (tests/vote_request_frames.py
and raftgpu_synth_wire_encode_vote_requests): the bytes an independent protobuf encoder, python-protobuf, writes for
eraftpb.Message with msg_type = MsgRequestVote (5) or MsgRequestPreVote (17) and the fields a candidate sets
(campaign, raft.rs:1217-1263, and send, :602-661): to, from, term, log_term, index, commit, commit_term, priority and
context.  The descriptor is gen_wire_golden.py's, restating eraftpb.proto:23-92.

    python scripts/gen_wire_vote_request_golden.py   # rewrites tests/golden/wire/vote_requests.json

Every vector: {"msg_type", "to", "from", "term", "log_term", "index", "commit", "commit_term", "priority", "context" (hex),
"hex": the serialized Message}.  Covered: both types; term, log_term, index, commit, commit_term and priority each at
0, 1, 127, 128, 2^32 and 2^64 - 1; the contexts empty, CampaignTransfer, CampaignElection, CampaignPreElection and
arbitrary bytes; random requests shaped as campaign builds them."""
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_wire_golden import build_classes  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "wire", "vote_requests.json")
EDGES = [0, 1, 127, 128, 1 << 32, (1 << 64) - 1]
CONTEXTS = [b"", b"CampaignTransfer", b"CampaignElection", b"CampaignPreElection", bytes([0, 0xFF, 0x80, 7]), b"\0" * 24]
FIELDS = ("to", "from", "term", "log_term", "index", "commit", "commit_term", "priority")


def main():
    Message = build_classes()
    rng = random.Random(0x5E7F)
    vectors = []

    def add(msg_type, context, **v):
        m = Message()
        m.msg_type = msg_type
        for k in FIELDS:
            setattr(m, k, v[k])
        m.context = context
        vectors.append({"msg_type": msg_type, **{k: v[k] for k in FIELDS}, "context": context.hex(),
                        "hex": m.SerializeToString().hex()})

    def rnd():
        return rng.choice([0, 1, rng.getrandbits(rng.choice([7, 20, 40, 64]))])

    # 1. both types; every field at every edge, the others random, each context
    for msg_type in (5, 17):
        for k in ("term", "log_term", "index", "commit", "commit_term", "priority"):
            for e in EDGES:
                for ctx in CONTEXTS:
                    v = {f: rnd() for f in FIELDS}
                    v[k] = e
                    add(msg_type, ctx, **v)
        for e in EDGES:   # all six at once
            add(msg_type, rng.choice(CONTEXTS), to=rnd(), **{"from": rnd()},
                **{k: e for k in ("term", "log_term", "index", "commit", "commit_term", "priority")})
    # 2. random requests as campaign builds them: to a peer, from self, term (+1 for a pre-vote), the last log
    # position, the commit info (raft.rs:1246-1251), the priority (send, :656-660), the campaign type as context
    # only for a transfer (:1255-1258)
    for _ in range(128):
        pre = rng.random() < 0.5
        term = rng.getrandbits(rng.choice([8, 20, 64 - 1]))
        index = rng.getrandbits(rng.choice([8, 20, 40]))
        commit = rng.randint(0, index)
        add(17 if pre else 5, b"CampaignTransfer" if rng.random() < 0.2 else b"", to=rng.randint(1, 9),
            **{"from": rng.randint(1, 9)}, term=term + 1, log_term=rng.randint(0, term), index=index, commit=commit,
            commit_term=rng.randint(0, term) if commit else 0, priority=rng.choice([0, 0, rng.getrandbits(8)]))
    with open(OUT, "w") as f:
        json.dump({"source": "python-protobuf %s from a descriptor restating eraftpb.proto:23-92" %
                             __import__("google.protobuf").protobuf.__version__, "vectors": vectors}, f, indent=0)
    print(f"wrote {len(vectors)} vectors to {OUT}")


if __name__ == "__main__":
    main()
