// k_wire.cuh -- the step from serialized eraftpb.Message frames (SURVEY 8(f) rank 4): proto3 varint decode on
// the device + the per-message prefix of handle_append_response, one thread per frame.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).
//
// A wire batch is what a transport holds: frames back to back,
//      frame i = bytes[offsets[i], offsets[i+1]) = u32 LE (group << 4 | peer_slot) + serialized Message
// (proto/proto/eraftpb.proto:71-92: fields 1-6, 8, 10, 11, 13-15 are varints; entries (7), snapshot (9) and
// context (12) are length-delimited and skipped).  The host does NOT parse anything: it appends frames and
// their end offsets, the blob crosses PCIe as it is (an AppendResponse is ~20-26 bytes on the wire, the same
// as the 24-byte record the host would otherwise have to build), and the GPU decodes.
//
// Two passes, because a batch may hold several messages of one (group, peer) cell and they must be applied
// in arrival order (the reject path does not commute with the accept path): the scan pass decodes every
// frame, classifies it and records -- atomicMin -- the FIRST frame of every cell; the apply pass decodes
// again (cheaper than carrying 40 bytes per frame through HBM), applies the frame that is first on its cell
// (apply_one, raft.rs:1663-1743) and reports every later one as RAFTGPU_WIRE_DUP for the next batch.
// What cannot be decided here goes back to the host as a status: other message types, a term that is not
// the group's (Raft::step's term rules), a rejection with log_term > 0 (its next_probe_index needs the
// leader's log, raft.rs:1562-1661), malformed bytes.
//
// HBM-bound byte work: every block stages the contiguous byte range of its 256 frames into shared memory
// with 16-byte loads (frames are ~26 bytes, unaligned) and the threads parse from there.

struct WireSrc {
    const uint8_t *bytes;     // 16-byte aligned
    const uint32_t *offsets;  // [n + 1]
    uint64_t n_bytes;
    uint32_t n;
    uint32_t n_groups;        // frames naming a group >= n_groups are malformed
};

struct WireMsg {  // the scalar fields this path looks at
    uint32_t msg_type;
    bool reject;
    uint64_t term, log_term, index, commit, reject_hint, request_snapshot;
    uint32_t ctx_off, ctx_len;  // wire_decode<true> only: bytes [ctx_off, ctx_off + ctx_len) are the last context (12)
    uint64_t from;              // wire_decode<true, true> only: field 3
};

constexpr uint32_t kWireThreads = 256;
constexpr uint32_t kWireStage = 16u * 1024u;  // staged bytes per block (256 frames of <= 64 bytes)

// Base-128 varint: at most `max_bytes` (10; 5 for tags), the tenth byte counts with its lowest bit.
__device__ __forceinline__ bool wire_varint(const uint8_t *p, uint32_t &pos, uint32_t end, uint32_t max_bytes, uint64_t &out) {
    uint64_t v = 0;
    for (uint32_t k = 0; k < max_bytes && pos < end; k++) {
        const uint32_t b = p[pos++];
        v |= (k < 9) ? (static_cast<uint64_t>(b & 0x7fu) << (7 * k)) : (static_cast<uint64_t>(b & 1u) << 63);
        if (!(b & 0x80u)) {
            out = v;
            return true;
        }
    }
    return false;
}

// One serialized Message -> WireMsg.  false = not a well-formed protobuf message.  kContext: also the context's
// position (the heartbeat-response path, k_hb_wire.cuh); the AppendResponse kernels instantiate it without.  kFrom:
// also `from` (the follower's heartbeat path, k_hb_follow.cuh).
template <bool kContext = false, bool kFrom = false>
__device__ __forceinline__ bool wire_decode(const uint8_t *p, uint32_t len, WireMsg &m) {
    m.msg_type = 0;
    m.reject = false;
    m.term = m.log_term = m.index = m.commit = m.reject_hint = m.request_snapshot = 0;
    if constexpr (kContext) m.ctx_off = m.ctx_len = 0;
    if constexpr (kFrom) m.from = 0;
    uint32_t pos = 0;
    while (pos < len) {
        uint64_t tag;
        if (!wire_varint(p, pos, len, 5, tag) || tag > 0xffffffffull) return false;
        const uint32_t field = static_cast<uint32_t>(tag >> 3), wt = static_cast<uint32_t>(tag & 7u);
        if (field == 0) return false;
        if (wt == 0) {
            uint64_t v;
            if (!wire_varint(p, pos, len, 10, v)) return false;
            // eraftpb.proto:71-92; a repeated scalar keeps its last value
            if (field == 1) m.msg_type = static_cast<uint32_t>(v);
            else if (field == 4) m.term = v;
            else if (field == 5) m.log_term = v;
            else if (field == 6) m.index = v;
            else if (field == 8) m.commit = v;
            else if (field == 10) m.reject = v != 0;
            else if (field == 11) m.reject_hint = v;
            else if (field == 13) m.request_snapshot = v;
            if constexpr (kFrom) {
                if (field == 3) m.from = v;
            }
        } else if (wt == 1) {
            if (len - pos < 8) return false;
            pos += 8;
        } else if (wt == 5) {
            if (len - pos < 4) return false;
            pos += 4;
        } else if (wt == 2) {
            uint64_t l;
            if (!wire_varint(p, pos, len, 10, l) || l > len - pos) return false;
            if constexpr (kContext) {
                if (field == 12) {  // bytes context = 12; a repeated one keeps its last value, as a parser does
                    m.ctx_off = pos;
                    m.ctx_len = static_cast<uint32_t>(l);
                }
            }
            pos += static_cast<uint32_t>(l);
        } else {
            return false;  // groups (3, 4) are not proto3; 6, 7 do not exist
        }
    }
    return true;
}

// The block's frames -> shared memory (when their byte range is sane and fits); returns through smem.
struct WireStage {
    uint32_t base, lo, hi;
    bool staged;
};

__device__ __forceinline__ WireStage wire_stage_block(const WireSrc &w, uint32_t first, uint32_t last, uint8_t *stage) {
    WireStage s;
    s.lo = w.offsets[first];
    s.hi = w.offsets[last];
    s.base = s.lo & ~15u;
    s.staged = s.lo <= s.hi && s.hi <= w.n_bytes && s.hi - s.base <= kWireStage;
    if (s.staged) {
        const uint32_t nb = s.hi - s.base;
        for (uint32_t o = threadIdx.x * 16u; o < nb; o += kWireThreads * 16u) {
            if (static_cast<uint64_t>(s.base) + o + 16u <= w.n_bytes) {
                *reinterpret_cast<uint4 *>(stage + o) = *reinterpret_cast<const uint4 *>(w.bytes + s.base + o);
            } else {
                for (uint32_t k = 0; k < 16u && static_cast<uint64_t>(s.base) + o + k < w.n_bytes; k++)
                    stage[o + k] = w.bytes[s.base + o + k];
            }
        }
    }
    __syncthreads();
    return s;
}

// Frame i's bytes (from the stage when they are there), its length and its u32 LE header; nullptr = not a frame
// (offsets out of order or past the batch, shorter than the header).
__device__ __forceinline__ const uint8_t *wire_frame_at(const WireSrc &w, const WireStage &s, const uint8_t *stage, uint32_t i,
                                                        uint32_t &hdr, uint32_t &len) {
    const uint32_t a = w.offsets[i], b = w.offsets[i + 1];
    if (b < a || b > w.n_bytes || b - a < 4u) return nullptr;
    const uint8_t *p = (s.staged && a >= s.lo && b <= s.hi) ? stage + (a - s.base) : w.bytes + a;
    hdr = p[0] | (static_cast<uint32_t>(p[1]) << 8) | (static_cast<uint32_t>(p[2]) << 16) | (static_cast<uint32_t>(p[3]) << 24);
    len = b - a;
    return p;
}

// Frame i: its status before the duplicate rule, the record, the REJECT's hint / request_snapshot.
__device__ __forceinline__ uint32_t wire_frame(const Columns &c, const WireSrc &w, const WireStage &s, const uint8_t *stage,
                                               uint32_t i, RecRegs &rec, uint64_t &hint, uint64_t &request_snapshot) {
    uint32_t hdr, len;
    const uint8_t *p = wire_frame_at(w, s, stage, i, hdr, len);
    if (!p) return RAFTGPU_WIRE_MALFORMED;
    const uint32_t group = hdr >> 4, slot = hdr & 15u;
    WireMsg m;
    if (group >= w.n_groups || !wire_decode(p + 4, len - 4u, m)) return RAFTGPU_WIRE_MALFORMED;
    if (m.msg_type != 4u) return RAFTGPU_WIRE_SKIP_TYPE;  // MsgAppendResponse, eraftpb.proto:54
    const uint64_t gterm = c.term[group];
    if (gterm != 0 && m.term != gterm) return RAFTGPU_WIRE_TERM;
    if (m.reject && m.log_term > 0) return RAFTGPU_WIRE_NEEDS_LOG;  // raft.rs:1562
    rec.w0 = static_cast<uint64_t>(group) | (static_cast<uint64_t>(slot) << 32) |
             (static_cast<uint64_t>(m.reject ? RAFTGPU_REC_REJECT : 0u) << 40);
    rec.index = m.index;
    rec.commit = m.commit;
    hint = m.reject_hint;                  // raft.rs:1560
    request_snapshot = m.request_snapshot;  // raft.rs:1709
    return RAFTGPU_WIRE_OK;
}

// Pass 1: classify every frame; first_frame[cell] = the lowest frame index that wants the cell.
__global__ void __launch_bounds__(kWireThreads) wire_scan_kernel(Columns c, WireSrc w, uint8_t *__restrict__ status,
                                                                 uint32_t *__restrict__ first_frame) {
    __shared__ __align__(16) uint8_t stage[kWireStage + 16];
    const uint32_t first = blockIdx.x * kWireThreads;
    if (first >= w.n) return;
    const uint32_t last = min(first + kWireThreads, w.n);
    const WireStage s = wire_stage_block(w, first, last, stage);
    const uint32_t i = first + threadIdx.x;
    if (i >= last) return;
    RecRegs rec;
    uint64_t hint, snap;
    const uint32_t st = wire_frame(c, w, s, stage, i, rec, hint, snap);
    status[i] = static_cast<uint8_t>(st << 4);
    if (st == RAFTGPU_WIRE_OK) {
        const uint32_t g = static_cast<uint32_t>(rec.w0), slot = static_cast<uint32_t>(rec.w0 >> 32) & 0xffu;
        if (slot < kSlots) atomicMin(&first_frame[static_cast<size_t>(slot) * c.cap + g], i);
    }
}

// Pass 2: the first frame of every cell is applied (raft.rs:1663-1743), later ones are RAFTGPU_WIRE_DUP.
// status[i] = wire status << 4 | RAFTGPU_RES_* of the applied message.
__global__ void __launch_bounds__(kWireThreads) wire_apply_kernel(Columns c, WireSrc w, uint8_t *__restrict__ status,
                                                                  const uint32_t *__restrict__ first_frame,
                                                                  unsigned long long *__restrict__ counters,
                                                                  uint32_t *__restrict__ dup_count) {
    __shared__ __align__(16) uint8_t stage[kWireStage + 16];
    uint32_t local[5] = {0, 0, 0, 0, 0};  // records, updates, rejects, decrements, no_progress
    const uint32_t first = blockIdx.x * kWireThreads;
    if (first < w.n) {
        const uint32_t last = min(first + kWireThreads, w.n);
        const WireStage s = wire_stage_block(w, first, last, stage);
        const uint32_t i = first + threadIdx.x;
        if (i < last && status[i] == (RAFTGPU_WIRE_OK << 4)) {
            RecRegs rec;
            uint64_t hint, snap;
            wire_frame(c, w, s, stage, i, rec, hint, snap);  // same verdict as in the scan pass
            const uint32_t g = static_cast<uint32_t>(rec.w0), slot = static_cast<uint32_t>(rec.w0 >> 32) & 0xffu;
            if (slot < kSlots && first_frame[static_cast<size_t>(slot) * c.cap + g] != i) {
                status[i] = static_cast<uint8_t>(RAFTGPU_WIRE_DUP << 4);
                if (dup_count) atomicAdd(dup_count, 1u);
            } else {
                const CellRegs cell = load_cell(c, rec);
                const CellPtrs gp = global_cell_ptrs(c, rec);
                const uint32_t res = apply_one<2>(c, nullptr, hint, snap, rec, cell, gp, local);
                status[i] = static_cast<uint8_t>((RAFTGPU_WIRE_OK << 4) | (res & 0xfu));
            }
        }
    }
    const int which[5] = {kCntRecords, kCntUpdates, kCntRejects, kCntDecrements, kCntNoProgress};
    block_flush_counts<5>(local, which, counters, nullptr);
}
