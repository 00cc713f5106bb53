#!/usr/bin/env python
"""Golden vectors for the follower's entry walk (raftgpu_follower_append_entries): MsgAppend Messages with entries as an
independent protobuf implementation, python-protobuf, writes and parses them.  The descriptor is gen_wire_golden.py's,
restating eraftpb.proto:23-92.

    python scripts/gen_wire_append_entries_golden.py   # rewrites tests/golden/wire/append_entries.json

"vectors": {"name", "hex", "parses", "entries": [[term, index, off, end], ..]}: `parses` is python-protobuf's verdict
on the bytes; where they parse, every Entry's term and index as it reads them and the byte span [off, end) of its
field-7 record (tag, length, Entry) in the Message.  Covered: 0, 1, 3 and 64 entries; each Entry field zero and
non-zero; term and index at 0, 1, 127, 128, 2^32, 2^63 and 2^64 - 1; data of 0, 1, 127, 128 and 20 000 bytes and a
context; and hand-built hostile bytes: a truncated inner Entry, a bad inner wire type, field 7 as a varint and an
Entry split from the next by another field."""
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_wire_golden import build_classes  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "wire", "append_entries.json")
EDGES = [0, 1, 127, 128, 1 << 32, 1 << 63, (1 << 64) - 1]


def varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def main():
    Message = build_classes()
    Entry = type(Message().entries.add())
    rng = random.Random(0xAE77)
    vectors = []

    def verdict(raw):
        m = Message()
        try:
            m.ParseFromString(raw)
        except Exception:
            return None
        return m

    def add(name, head: bytes, records, tail: bytes = b""):
        """head + the field-7 records (each bytes, or (bytes between, record)) + tail, as built; parsed back."""
        raw, spans = bytearray(head), []
        for r in records:
            between, rec = r if isinstance(r, tuple) else (b"", r)
            raw += between
            spans.append((len(raw), len(raw) + len(rec)))
            raw += rec
        raw += tail
        m = verdict(bytes(raw))
        ents = []
        if m is not None:
            assert len(m.entries) <= len(spans)
            ents = [[e.term, e.index, a, b] for e, (a, b) in zip(m.entries, spans)]
        vectors.append({"name": name, "hex": bytes(raw).hex(), "parses": m is not None, "entries": ents})

    def head(term, log_term, index, frm=2):
        m = Message()
        m.msg_type, m.to, m.term, m.log_term, m.index = 3, 1, term, log_term, index
        setattr(m, "from", frm)
        return m.SerializeToString()

    def tail(commit):
        m = Message()
        m.commit = commit
        return m.SerializeToString()

    def rec(**kw):
        e = Entry()
        for k, v in kw.items():
            setattr(e, k, v)
        b = e.SerializeToString()
        return varint(7 << 3 | 2) + varint(len(b)) + b

    big = lambda: rng.choice([rng.randint(1, 9), rng.getrandbits(64) or 1])
    # 0, 1, 3 and 64 entries at consecutive indexes
    for k in (0, 1, 3, 64):
        t, i = big(), rng.randint(0, 1 << 40)
        add(f"{k} entries", head(t, t, i), [rec(term=t, index=i + 1 + j) for j in range(k)], tail(big()))
    # each Entry field zero and non-zero
    for mask in range(64):
        kw = {}
        for bit, (f, v) in enumerate((("entry_type", 1), ("term", big()), ("index", big()), ("data", b"xyz"),
                                      ("context", b"c"), ("sync_log", True))):
            if (mask >> bit) & 1:
                kw[f] = v
        add(f"fields {mask:06b}", head(5, 5, 9), [rec(**kw)], tail(3))
    # term and index at the varint edges
    for e in EDGES:
        add(f"term {e}", head(1, 1, 1), [rec(term=e, index=2)])
        add(f"index {e}", head(1, 1, 1), [rec(term=1, index=e)])
    # data sizes and a context
    for n in (0, 1, 127, 128, 20_000):
        add(f"data {n}", head(3, 3, 10), [rec(term=3, index=11, data=bytes([0xA5]) * n), rec(term=4, index=12)], tail(11))
    add("context", head(3, 3, 10), [rec(term=3, index=11, context=b"ctx" * 50)])
    # hostile bytes
    ok = rec(term=2, index=2)
    add("truncated entry", head(2, 2, 1), [ok[:-1]])
    add("entry length past the end", head(2, 2, 1), [varint(7 << 3 | 2) + varint(9) + b"\x10\x02"])
    add("entry truncated varint", head(2, 2, 1), [varint(7 << 3 | 2) + b"\x02\x10\x82"])
    add("entry bad wire type 3", head(2, 2, 1), [varint(7 << 3 | 2) + b"\x02\x13\x00"])
    add("entry bad wire type 7", head(2, 2, 1), [varint(7 << 3 | 2) + b"\x02\x17\x00"])
    add("entry field 0", head(2, 2, 1), [varint(7 << 3 | 2) + b"\x02\x00\x01"])
    add("entry term as bytes", head(2, 2, 1), [varint(7 << 3 | 2) + b"\x05\x12\x01\x05\x18\x02"])
    add("entry repeated term", head(2, 2, 1), [varint(7 << 3 | 2) + b"\x06\x10\x01\x10\x02\x18\x02"])
    add("field 7 as a varint", head(2, 2, 1), [ok, varint(7 << 3) + varint(5)])
    add("field 7 as fixed64", head(2, 2, 1), [varint(7 << 3 | 1) + bytes(8)])
    add("entries split by another field", head(2, 2, 1), [ok, (varint(11 << 3) + varint(4), rec(term=2, index=3))],
        tail(1))
    add("entries after commit", head(2, 2, 1), [(tail(1), ok)])
    with open(OUT, "w") as f:
        json.dump({"source": "python-protobuf %s from a descriptor restating eraftpb.proto:23-92" %
                             __import__("google.protobuf").protobuf.__version__, "vectors": vectors}, f, indent=0)
    print(f"wrote {len(vectors)} vectors to {OUT}")


if __name__ == "__main__":
    main()
