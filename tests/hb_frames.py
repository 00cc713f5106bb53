"""Wire frames for the heartbeat-response tests: u32 LE (group << 4 | peer_slot) + a serialized eraftpb.Message, built
field by field (proto3: zero scalars are not written), and batches of them as (blob, offsets)."""
import numpy as np

HEARTBEAT_RESPONSE, APPEND_RESPONSE = 9, 4


def varint(v: int) -> bytes:
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def message(msg_type, term=0, commit=0, index=0, reject=False, reject_hint=0, context=None, frm=0) -> bytes:
    out = b""
    for no, v in ((1, msg_type), (2, 1), (3, frm), (4, term), (6, index), (8, commit), (10, int(reject)), (11, reject_hint)):
        if v:
            out += varint(no << 3) + varint(v)
    if context:
        out += varint(12 << 3 | 2) + varint(len(context)) + context
    return out


def frame(group, slot, body: bytes) -> bytes:
    return np.array([group << 4 | slot], dtype="<u4").tobytes() + body


def ctx_bytes(x: int) -> bytes:
    """The context of a heartbeat that carries read id x."""
    return int(x).to_bytes(8, "little")


def batch(frames):
    blob = np.frombuffer(b"".join(frames), dtype=np.uint8).copy()
    offsets = np.concatenate([[0], np.cumsum([len(f) for f in frames])]).astype(np.uint32)
    return blob, offsets


class Frames:
    """A batch with the attributes Arena.heartbeat_wire / step_begin_wire read."""

    def __init__(self, frames):
        self.bytes, self.offsets = batch(frames)
        self.n, self.n_bytes, self.n_records = len(frames), len(self.bytes), 0
        if self.n_bytes == 0:
            self.bytes = np.zeros(16, np.uint8)
