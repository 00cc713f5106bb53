#!/usr/bin/env python
"""Golden vectors for the eraftpb.Message wire decoder (SURVEY 8(f4)).

The reference serializes messages with rust-protobuf 2 / prost 0.7 (proto/Cargo.toml:21-27), neither
vendored nor buildable here, and holds no wire-format goldens for this path.  The vectors are therefore
produced by an INDEPENDENT implementation of the same published format: Google's python-protobuf,
from a descriptor that restates `message Message` / `Entry` / `Snapshot` of
the reference's proto/proto/eraftpb.proto:23-92 field for field (numbers and types).  "Parity unpinned by
the reference" (DESIGN.md 6): what is pinned is proto3 wire compatibility.

    python scripts/gen_wire_golden.py            # rewrites tests/golden/wire/messages.json

Every vector: {"hex": serialized bytes, "fields": the scalar fields a decoder must recover}.  Besides
python-protobuf's canonical encodings the file holds hand-built non-canonical but legal encodings
(fields out of order, repeated scalar fields -- last one wins --, unknown fields of every wire type,
over-long varints) and malformed inputs (truncated varint / length, wire types 3/4/6/7, field 0)."""
import json
import os
import random

from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "wire", "messages.json")

T = descriptor_pb2.FieldDescriptorProto


def build_classes():
    fd = descriptor_pb2.FileDescriptorProto(name="eraftpb_golden.proto", package="eraftpb", syntax="proto3")
    et = fd.enum_type.add(name="EntryType")                    # eraftpb.proto:7-11
    for i, n in enumerate(["EntryNormal", "EntryConfChange", "EntryConfChangeV2"]):
        et.value.add(name=n, number=i)
    mt = fd.enum_type.add(name="MessageType")                  # eraftpb.proto:49-69
    for i, n in enumerate(["MsgHup", "MsgBeat", "MsgPropose", "MsgAppend", "MsgAppendResponse", "MsgRequestVote",
                           "MsgRequestVoteResponse", "MsgSnapshot", "MsgHeartbeat", "MsgHeartbeatResponse",
                           "MsgUnreachable", "MsgSnapStatus", "MsgCheckQuorum", "MsgTransferLeader", "MsgTimeoutNow",
                           "MsgReadIndex", "MsgReadIndexResp", "MsgRequestPreVote", "MsgRequestPreVoteResponse"]):
        mt.value.add(name=n, number=i)

    def msg(name, fields):
        m = fd.message_type.add(name=name)
        for fname, num, typ, tname, rep in fields:
            f = m.field.add(name=fname, number=num, type=typ,
                            label=T.LABEL_REPEATED if rep else T.LABEL_OPTIONAL)
            if tname:
                f.type_name = tname
    msg("Entry", [("entry_type", 1, T.TYPE_ENUM, ".eraftpb.EntryType", False), ("term", 2, T.TYPE_UINT64, None, False),
                  ("index", 3, T.TYPE_UINT64, None, False), ("data", 4, T.TYPE_BYTES, None, False),
                  ("context", 6, T.TYPE_BYTES, None, False), ("sync_log", 5, T.TYPE_BOOL, None, False)])   # :23-34
    msg("ConfState", [("voters", 1, T.TYPE_UINT64, None, True), ("learners", 2, T.TYPE_UINT64, None, True)])
    msg("SnapshotMetadata", [("conf_state", 1, T.TYPE_MESSAGE, ".eraftpb.ConfState", False),
                             ("index", 2, T.TYPE_UINT64, None, False), ("term", 3, T.TYPE_UINT64, None, False)])  # :36-42
    msg("Snapshot", [("data", 1, T.TYPE_BYTES, None, False),
                     ("metadata", 2, T.TYPE_MESSAGE, ".eraftpb.SnapshotMetadata", False)])               # :44-47
    msg("Message", [("msg_type", 1, T.TYPE_ENUM, ".eraftpb.MessageType", False), ("to", 2, T.TYPE_UINT64, None, False),
                    ("from", 3, T.TYPE_UINT64, None, False), ("term", 4, T.TYPE_UINT64, None, False),
                    ("log_term", 5, T.TYPE_UINT64, None, False), ("index", 6, T.TYPE_UINT64, None, False),
                    ("entries", 7, T.TYPE_MESSAGE, ".eraftpb.Entry", True), ("commit", 8, T.TYPE_UINT64, None, False),
                    ("commit_term", 15, T.TYPE_UINT64, None, False), ("snapshot", 9, T.TYPE_MESSAGE, ".eraftpb.Snapshot", False),
                    ("request_snapshot", 13, T.TYPE_UINT64, None, False), ("reject", 10, T.TYPE_BOOL, None, False),
                    ("reject_hint", 11, T.TYPE_UINT64, None, False), ("context", 12, T.TYPE_BYTES, None, False),
                    ("priority", 14, T.TYPE_UINT64, None, False)])                                       # :71-92
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName("eraftpb.Message"))


SCALARS = ["msg_type", "to", "from", "term", "log_term", "index", "commit", "commit_term", "request_snapshot",
           "reject", "reject_hint", "priority"]
FIELD_NO = {"msg_type": 1, "to": 2, "from": 3, "term": 4, "log_term": 5, "index": 6, "commit": 8, "commit_term": 15,
            "request_snapshot": 13, "reject": 10, "reject_hint": 11, "priority": 14}


def fields_of(m):
    return {k: int(getattr(m, k)) for k in SCALARS}


def varint(v, pad=0, limit=10):
    """LEB128; pad > 0 appends that many redundant continuation bytes (a legal over-long encoding)
    as long as the whole varint stays within `limit` bytes."""
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            break
    if pad and len(out) + pad <= limit:
        out[-1] |= 0x80
        out += b"\x80" * (pad - 1) + b"\x00"
    return bytes(out)


def main():
    Message = build_classes()
    rng = random.Random(0xE4AF7)
    edge = [0, 1, 127, 128, 255, 256, 16383, 16384, (1 << 21) - 1, 1 << 21, (1 << 28) - 1, 1 << 28, (1 << 32) - 1, 1 << 32,
            (1 << 35) - 1, 1 << 35, (1 << 42), (1 << 49) - 1, (1 << 56), (1 << 63) - 1, 1 << 63, (1 << 64) - 1]

    def u64():
        r = rng.random()
        if r < 0.3:
            return rng.choice(edge)
        if r < 0.6:
            return rng.getrandbits(rng.choice([7, 14, 21, 28, 35, 42, 49, 56, 63, 64]))
        return rng.getrandbits(40)

    vectors = []
    # 1. canonical AppendResponses, the shape of the synthetic stream: accepts and rejects
    for k in range(160):
        m = Message()
        m.msg_type = 4
        m.to, setattr_from, m.term = u64() if k % 5 == 0 else rng.randint(1, 9), None, rng.randint(1, 1 << 20)
        setattr(m, "from", u64() if k % 7 == 0 else rng.randint(1, 9))
        m.index = u64()
        m.commit = u64() if k % 3 == 0 else max(0, m.index - rng.randint(0, 300))
        if k % 4 == 0:
            m.reject = True
            m.reject_hint = u64() if k % 8 == 0 else max(0, m.index - rng.randint(0, 9))
            if k % 12 == 0:
                m.log_term = rng.randint(1, 1 << 20)
            if k % 16 == 0:
                m.request_snapshot = u64()
        vectors.append({"kind": "append_response", "hex": m.SerializeToString().hex(), "fields": fields_of(m), "ok": True})
    # 2. every message type, every field at random (entries / snapshot / context present: skipped by the decoder)
    for k in range(120):
        m = Message()
        m.msg_type = rng.randint(0, 18)
        for f in SCALARS[1:]:
            if rng.random() < 0.6:
                setattr(m, f, (rng.random() < 0.5) if f == "reject" else u64())
        if rng.random() < 0.5:
            for _ in range(rng.randint(1, 3)):
                e = m.entries.add()
                e.term, e.index, e.data = u64(), u64(), rng.randbytes(rng.randint(0, 200))
        if rng.random() < 0.3:
            m.snapshot.data = rng.randbytes(rng.randint(0, 300))
            m.snapshot.metadata.index = u64()
        if rng.random() < 0.3:
            m.context = rng.randbytes(rng.randint(0, 40))
        vectors.append({"kind": "any", "hex": m.SerializeToString().hex(), "fields": fields_of(m), "ok": True})
    # 3. legal but non-canonical encodings, checked by python-protobuf's own parser
    for k in range(80):
        vals = {f: ((1 if rng.random() < 0.5 else 0) if f == "reject" else (rng.randint(0, 18) if f == "msg_type" else u64()))
                for f in SCALARS if rng.random() < 0.7}
        parts = []
        for f, v in vals.items():
            if rng.random() < 0.3:      # an earlier value of the same field: the last one wins
                parts.append(varint(FIELD_NO[f] << 3) + varint(rng.getrandbits(20)))
            parts.append(varint(FIELD_NO[f] << 3, pad=rng.choice([0, 0, 1, 2]), limit=5) + varint(v, pad=rng.choice([0, 0, 0, 1, 3])))
        rng.shuffle(parts)
        for _ in range(rng.randint(0, 3)):  # unknown fields of the four legal wire types
            no = rng.choice([16, 17, 100, 1000, 536870911])
            wt = rng.choice([0, 1, 2, 5])
            body = {0: varint(u64()), 1: rng.randbytes(8), 5: rng.randbytes(4)}.get(wt)
            if wt == 2:
                blob = rng.randbytes(rng.randint(0, 30))
                body = varint(len(blob)) + blob
            parts.insert(rng.randint(0, len(parts)), varint(no << 3 | wt) + body)
        raw = b"".join(parts)
        m = Message()
        m.ParseFromString(raw)          # python-protobuf decides what the bytes mean
        vectors.append({"kind": "non_canonical", "hex": raw.hex(), "fields": fields_of(m), "ok": True})
    # 4. malformed: python-protobuf must refuse them too
    bad = [
        b"\x08",                                   # tag without value
        b"\x08\x80",                               # truncated varint
        b"\x30" + b"\xff" * 10 + b"\x01",          # 11-byte varint
        b"\x3a\x05abc",                            # length runs past the end
        b"\x3a\xff\xff\xff\xff\x0f",               # huge length
        b"\x0b",                                   # wire type 3 (start group) on field 1
        b"\x0c",                                   # wire type 4
        b"\x0e\x00",                               # wire type 6
        b"\x0f\x00",                               # wire type 7
        b"\x00\x00",                               # field number 0
        b"\x09\x01\x02\x03",                       # fixed64 truncated
        b"\x0d\x01",                               # fixed32 truncated
        b"\x08\x04\x30",                           # valid prefix, then a tag without value
    ]
    for raw in bad:
        m = Message()
        try:
            m.ParseFromString(raw)
            ok = True
        except Exception:
            ok = False
        vectors.append({"kind": "malformed", "hex": raw.hex(), "fields": fields_of(m) if ok else None, "ok": ok})
    # 5. edge semantics, python-protobuf's verdict recorded as is: the 10th varint byte counts with its lowest bit
    # only, bool = any non-zero varint, enum = the varint truncated to 32 bits, a known field number with another
    # wire type is an unknown field, tags are at most 5 bytes / field numbers below 2^29, the empty message is legal
    edge_raw = [
        b"\x30" + b"\xff" * 9 + b"\x7f", b"\x30" + b"\xff" * 9 + b"\x01", b"\x30" + b"\xff" * 9 + b"\x02",
        b"\x50\x02", b"\x50" + varint(1 << 32), b"\x50" + varint(1 << 63), b"\x08" + varint((1 << 32) + 4),
        b"\x08" + varint(1 << 31), b"\x08" + varint((1 << 64) - 1), varint((0x1fffffff << 3) | 0) + b"\x01",
        b"\x88\x80\x80\x80\x80\x00\x01", varint((0x20000000 << 3) | 0) + b"\x01", b"", b"\x0a\x01\x04", b"\x38\x05",
        b"\x31" + b"\x01" * 8, b"\x35\x01\x02\x03\x04\x08\x04", b"\x08\x04\x08\x09", b"\x08\x09\x08\x04",
        b"\x08\x04\x20\x07\x30\x64\x40\x63",   # the plain accept: type 4, term 7, index 100, commit 99
    ]
    for raw in edge_raw:
        m = Message()
        try:
            m.ParseFromString(raw)
            ok = True
        except Exception:
            ok = False
        f_ = fields_of(m) if ok else None
        if f_:
            f_["msg_type"] &= 0xFFFFFFFF   # enums are int32 in python: compare as the 32-bit pattern
        vectors.append({"kind": "edge", "hex": raw.hex(), "fields": f_, "ok": ok})
    with open(OUT, "w") as f:
        json.dump({"source": "python-protobuf %s from a descriptor restating eraftpb.proto:23-92" %
                             __import__("google.protobuf").protobuf.__version__, "vectors": vectors}, f, indent=0)
    print(f"wrote {len(vectors)} vectors to {OUT}; malformed accepted by python-protobuf:",
          [v["hex"] for v in vectors if v["kind"] == "malformed" and v["ok"]])


if __name__ == "__main__":
    main()
