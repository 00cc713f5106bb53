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
// leader's log, raft.rs:1562-1661) unless the leader's term runs decide it (the <true> kernels, DESIGN 3.18),
// malformed bytes.
//
// HBM-bound byte work: every block stages the contiguous byte range of its 256 frames into shared memory
// with 16-byte loads (frames are ~26 bytes, unaligned) and the threads parse from there.
//
// The file holds the frame format in both directions: the decoder and the block staging every wire pass uses
// (wire_open, wire_block_frame), and the heartbeat-kind encoder with the block-output code that the leader's
// MsgHeartbeat frames (k_hb_frames.cuh) and the follower's MsgHeartbeatResponse frames (k_hb_follow.cuh) share; the
// voter's vote responses (k_vote_request.cuh) use that block-output code with their own encoder.

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
    uint64_t commit_term;       // wire_decode<.., .., true> only: field 15
    uint64_t priority;          // wire_decode<.., .., .., true> only: field 14
    bool entries;               // wire_decode<.., .., .., .., true> only: a field 7 (entries) is present
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
// also `from` (the follower's heartbeat path, k_hb_follow.cuh).  kCommitTerm: also commit_term (the vote responses,
// k_vote_wire.cuh).  kPriority: also priority (the vote requests, k_vote_request.cuh).  kEntries: also whether any
// field 7 occurs, in any wire type (the follower's MsgAppend path, k_app_follow.cuh).
template <bool kContext = false, bool kFrom = false, bool kCommitTerm = false, bool kPriority = false, bool kEntries = false>
__device__ __forceinline__ bool wire_decode(const uint8_t *p, uint32_t len, WireMsg &m) {
    m.msg_type = 0;
    m.reject = false;
    m.term = m.log_term = m.index = m.commit = m.reject_hint = m.request_snapshot = 0;
    if constexpr (kContext) m.ctx_off = m.ctx_len = 0;
    if constexpr (kFrom) m.from = 0;
    if constexpr (kCommitTerm) m.commit_term = 0;
    if constexpr (kPriority) m.priority = 0;
    if constexpr (kEntries) m.entries = false;
    uint32_t pos = 0;
    while (pos < len) {
        uint64_t tag;
        if (!wire_varint(p, pos, len, 5, tag) || tag > 0xffffffffull) return false;
        const uint32_t field = static_cast<uint32_t>(tag >> 3), wt = static_cast<uint32_t>(tag & 7u);
        if (field == 0) return false;
        if constexpr (kEntries) {
            if (field == 7) m.entries = true;  // repeated Entry entries = 7, an empty Entry included
        }
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
            if constexpr (kCommitTerm) {
                if (field == 15) m.commit_term = v;
            }
            if constexpr (kPriority) {
                if (field == 14) m.priority = v;
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

// The entries of a MsgAppend whose log matches at idx (k_app_follow.cuh, raftgpu_follower_append_entries): every field 7
// of the Message p[0, len) (already well formed: wire_decode) walked once, each length-delimited one decoded as an
// eraftpb.Entry (term = 2, index = 3, eraftpb.proto:16-21; other fields skipped by their length, a repeated scalar
// keeps its last value).  term(j) for j > idx is the follower's: run_term up to last, 0 above (raft_log.rs:125).
struct WireEntries {
    uint32_t count;               // field-7 records
    uint32_t conflict;            // find_conflict (raft_log.rs:182-198): 1 + the position of the first entry whose term
                                  // is not term(index) (index idx + conflict), 0 when every entry matches
    uint32_t tail;                // 1 + the position of the trailing block of appended entries with the last one's term
    uint32_t span_off, span_end;  // from p: the first appended entry's tag, the end of the last appended one
    uint64_t tail_term;           // the last appended entry's term
    bool uniform;                 // every appended entry has term tail_term
};
constexpr uint32_t kEntsOk = 0, kEntsMalformed = 1, kEntsNeedsLog = 2;

// The walk of raftgpu_follower_append_entries on an arena with follower runs (k_app_follow.cuh, DESIGN 3.22): term(j)
// for idx < j <= last is run_term on the table's run [run_start, last], t1 on the row's run 1 (down to s1) and t2 below
// it (term(idx) is known, so every such j lies in one of them); pre / pre_term = the block of appended entries before
// the trailing one (as tail / tail_term; 0 when the appended entries hold one term).
struct WireEntriesRuns : WireEntries {
    uint32_t pre;
    uint64_t pre_term;
};

template <bool kRuns, class E>
__device__ __forceinline__ uint32_t wire_entries_walk(const uint8_t *p, uint32_t len, uint64_t idx, uint64_t last,
                                                      uint64_t run_start, uint64_t run_term, uint64_t s1, uint64_t t1,
                                                      uint64_t t2, E &e) {
    e.count = e.conflict = e.tail = e.span_off = e.span_end = 0;
    e.tail_term = 0;
    e.uniform = true;
    if constexpr (kRuns) {
        e.pre = 0;
        e.pre_term = 0;
    }
    bool needs_log = false;
    uint32_t pos = 0;
    while (pos < len) {
        const uint32_t at = pos;
        uint64_t tag, l;
        if (!wire_varint(p, pos, len, 5, tag)) return kEntsMalformed;
        const uint32_t field = static_cast<uint32_t>(tag >> 3), wt = static_cast<uint32_t>(tag & 7u);
        if (wt != 2) {  // a scalar: skipped (the Message is well formed)
            if (field == 7) needs_log = true;
            if (wt == 0) wire_varint(p, pos, len, 10, l);
            else pos += wt == 1 ? 8u : 4u;
            continue;
        }
        if (!wire_varint(p, pos, len, 10, l)) return kEntsMalformed;
        const uint32_t end = pos + static_cast<uint32_t>(l);
        if (field != 7) {
            pos = end;
            continue;
        }
        uint64_t term = 0, index = 0;
        while (pos < end) {  // the Entry
            uint64_t t, v;
            if (!wire_varint(p, pos, end, 5, t) || t > 0xffffffffull || (t >> 3) == 0) return kEntsMalformed;
            const uint32_t f = static_cast<uint32_t>(t >> 3), w = static_cast<uint32_t>(t & 7u);
            if (w == 0) {
                if (!wire_varint(p, pos, end, 10, v)) return kEntsMalformed;
                if (f == 2) term = v;
                else if (f == 3) index = v;
            } else if (w == 1 || w == 5) {
                const uint32_t k = w == 1 ? 8u : 4u;
                if (end - pos < k) return kEntsMalformed;
                pos += k;
            } else if (w == 2) {
                if (!wire_varint(p, pos, end, 10, v) || v > end - pos) return kEntsMalformed;
                pos += static_cast<uint32_t>(v);
            } else {
                return kEntsMalformed;
            }
        }
        const uint32_t k = ++e.count;  // this entry is index idx + k
        if (index != idx + k || term == 0) {
            needs_log = true;
        } else if (!e.conflict) {
            uint64_t have = run_term;  // term(idx + k), for idx + k <= last
            if constexpr (kRuns) have = idx + k >= run_start ? run_term : idx + k >= s1 ? t1 : t2;
            if (idx + k > last || term != have) {  // the first entry the log takes
                e.conflict = e.tail = k;
                e.tail_term = term;
                e.span_off = at;
                e.span_end = end;
            }
        } else {
            if (at != e.span_end) needs_log = true;
            e.span_end = end;
            if (term != e.tail_term) {
                if constexpr (kRuns) {
                    e.pre = e.tail;
                    e.pre_term = e.tail_term;
                }
                e.tail = k;
                e.tail_term = term;
                e.uniform = false;
            }
        }
    }
    return needs_log ? kEntsNeedsLog : kEntsOk;
}

// kEntsMalformed: an Entry is not a well-formed protobuf message.  kEntsNeedsLog: a field 7 that is not length-
// delimited, an index other than idx + 1, idx + 2, ..., a term 0, or appended entries with another field between them.
__device__ __noinline__ uint32_t wire_entries(const uint8_t *p, uint32_t len, uint64_t idx, uint64_t last,
                                                 uint64_t run_term, WireEntries &e) {
    return wire_entries_walk<false>(p, len, idx, last, 0, run_term, 0, 0, 0, e);
}

// The same walk with the follower's runs (WireEntriesRuns).
__device__ __noinline__ uint32_t wire_entries_runs(const uint8_t *p, uint32_t len, uint64_t idx, uint64_t last,
                                                      uint64_t run_start, uint64_t run_term, uint64_t s1, uint64_t t1,
                                                      uint64_t t2, WireEntriesRuns &e) {
    return wire_entries_walk<true>(p, len, idx, last, run_start, run_term, s1, t1, t2, e);
}

// The context convention of the heartbeat paths (DESIGN 3.10): a read id travels as the 8 bytes of the context,
// little-endian.  q = the context's first byte (WireMsg::ctx_off from the Message's start).
__device__ __forceinline__ uint64_t wire_ctx_u64(const uint8_t *q) {
    uint64_t x = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) x |= static_cast<uint64_t>(q[k]) << (8 * k);
    return x;
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

// The prologue of every staging kernel (kWireThreads frames per block): stages the block's frames and returns the
// thread's frame index, or kNoFrame past the batch.  A block past the batch returns at once, without staging.
constexpr uint32_t kNoFrame = 0xffffffffu;  // (a frame index is below w.n <= 0xfffffff0)

__device__ __forceinline__ uint32_t wire_block_frame(const WireSrc &w, uint8_t *stage, WireStage &s) {
    const uint32_t first = blockIdx.x * kWireThreads;
    if (first >= w.n) return kNoFrame;
    const uint32_t last = min(first + kWireThreads, w.n);
    s = wire_stage_block(w, first, last, stage);
    const uint32_t i = first + threadIdx.x;
    return i < last ? i : kNoFrame;
}

// Frame i opened: its u32 LE header, its Message (msg, from the stage when the bytes are there) decoded into m.
// RAFTGPU_WIRE_MALFORMED when it is not a frame (offsets out of order or past the batch, shorter than the header),
// names a group >= n_groups or is not a well-formed protobuf message; RAFTGPU_WIRE_OK otherwise.  The flags are
// wire_decode's.
template <bool kContext = false, bool kFrom = false, bool kCommitTerm = false, bool kPriority = false, bool kEntries = false>
__device__ __forceinline__ uint32_t wire_open(const WireSrc &w, const WireStage &s, const uint8_t *stage, uint32_t i,
                                              uint32_t &hdr, const uint8_t *&msg, WireMsg &m) {
    const uint32_t a = w.offsets[i], b = w.offsets[i + 1];
    if (b < a || b > w.n_bytes || b - a < 4u) return RAFTGPU_WIRE_MALFORMED;
    const uint8_t *p = (s.staged && a >= s.lo && b <= s.hi) ? stage + (a - s.base) : w.bytes + a;
    hdr = p[0] | (static_cast<uint32_t>(p[1]) << 8) | (static_cast<uint32_t>(p[2]) << 16) | (static_cast<uint32_t>(p[3]) << 24);
    msg = p + 4;
    if ((hdr >> 4) >= w.n_groups || !wire_decode<kContext, kFrom, kCommitTerm, kPriority, kEntries>(msg, b - a - 4u, m))
        return RAFTGPU_WIRE_MALFORMED;
    return RAFTGPU_WIRE_OK;
}

// The leader's term runs (raftgpu_arena_enable_leader_runs, DESIGN 3.18): one row per group slot, 48 bytes, read as three
// 16-byte loads -- {term, term_start} (the anchor), {run_start[0], run_start[1]}, {run_term[0], run_term[1]}.  Run 1
// is [run_start[0], term_start - 1] at run_term[0], run 2 [run_start[1], run_start[0] - 1] at run_term[1]; a start of 0
// is not stated.  raftgpu_leader_runs_set stores only rows with 0 < run_start[1] < run_start[0] < term_start and
// 0 < run_term[1] < run_term[0] < term where stated.  A pair's row lives on its low half.
struct LeaderRuns {
    ulonglong2 anchor, start, term;
};

// next_probe_index = find_conflict_by_term(h, lt) (raft.rs:1562, raft_log.rs:209-235) of group g's leader, from the
// arena and its row: term(i) = term on [term_start, last_index] (DESIGN 1), run_term[k] on run k, 0 at 0.  A pair reads
// its low half's term, term_start and row, and the larger last_index (as DESIGN 3.15).  false = undecided: the row is
// not anchored to the group's leadership (a leader, a term, the row's (term, term_start)), or the walk leaves the stated
// runs at an index whose bound -- the lowest stated run's term, terms being monotone -- is above lt.
__device__ __forceinline__ bool wire_probe_by_runs(const Columns &c, const LeaderRuns *__restrict__ runs, uint32_t g,
                                                   uint64_t h, uint64_t lt, uint64_t &out) {
    const uint32_t meta = c.meta[g];
    const uint32_t lo = (meta & RAFTGPU_META_WIDE_HI) ? g - 1 : g;
    const uint64_t ts = c.term_start[lo], term = c.term[lo];
    if (ts == RAFTGPU_NO_TERM_START || term == 0) return false;
    const ulonglong2 anchor = runs[lo].anchor;
    if (anchor.x != term || anchor.y != ts) return false;
    uint64_t last = c.last_index[lo];
    if (meta & (RAFTGPU_META_WIDE_LO | RAFTGPU_META_WIDE_HI)) last = umax64(last, c.last_index[lo + 1]);
    out = h;
    if (h > last) return true;  // raft_log.rs:213-221
    // the segments from the top: [ts, last] at term, run 1, run 2; i walks down to the first one whose term is <= lt
    uint64_t i = h;
    if (term <= lt) return true;  // (i >= ts, or i below ts whose term is <= term)
    i = umin64(i, ts - 1);
    uint64_t bound = term;  // every index at or below i has a term <= bound
    const ulonglong2 rs = runs[lo].start, rt = runs[lo].term;
    if (rs.x) {
        if (i >= rs.x && rt.x <= lt) {
            out = i;
            return true;
        }
        bound = rt.x;
        if (rs.x <= i) i = rs.x - 1;
        if (rs.y) {
            if (i >= rs.y && rt.y <= lt) {
                out = i;
                return true;
            }
            bound = rt.y;
            if (rs.y <= i) i = rs.y - 1;
        }
    }
    out = i;
    return i == 0 || bound <= lt;  // term(0) = 0 < lt
}

// Frame i: its status before the duplicate rule, the record, the REJECT's hint / request_snapshot.  kRuns: a rejection
// with log_term > 0 is decided from the leader's runs (wire_probe_by_runs) where they say enough.
template <bool kRuns>
__device__ __forceinline__ uint32_t wire_frame(const Columns &c, const LeaderRuns *runs, const WireSrc &w, const WireStage &s,
                                               const uint8_t *stage, uint32_t i, RecRegs &rec, uint64_t &hint,
                                               uint64_t &request_snapshot) {
    uint32_t hdr;
    const uint8_t *msg;
    WireMsg m;
    if (wire_open(w, s, stage, i, hdr, msg, m) != RAFTGPU_WIRE_OK) return RAFTGPU_WIRE_MALFORMED;
    const uint32_t group = hdr >> 4, slot = hdr & 15u;
    if (m.msg_type != 4u) return RAFTGPU_WIRE_SKIP_TYPE;  // MsgAppendResponse, eraftpb.proto:54
    const uint64_t gterm = c.term[group];
    if (gterm != 0 && m.term != gterm) return RAFTGPU_WIRE_TERM;
    uint64_t h = m.reject_hint;  // raft.rs:1560
    if (m.reject && m.log_term > 0) {  // raft.rs:1562
        if constexpr (!kRuns) return RAFTGPU_WIRE_NEEDS_LOG;
        else if (!wire_probe_by_runs(c, runs, group, m.reject_hint, m.log_term, h)) return RAFTGPU_WIRE_NEEDS_LOG;
    }
    rec.w0 = static_cast<uint64_t>(group) | (static_cast<uint64_t>(slot) << 32) |
             (static_cast<uint64_t>(m.reject ? RAFTGPU_REC_REJECT : 0u) << 40);
    rec.index = m.index;
    rec.commit = m.commit;
    hint = h;
    request_snapshot = m.request_snapshot;  // raft.rs:1709
    return RAFTGPU_WIRE_OK;
}

// Pass 1: classify every frame; first_frame[cell] = the lowest frame index that wants the cell.  runs: the arena's rows
// (kRuns only; the last parameter, so that the others keep their offsets).
template <bool kRuns>
__device__ __forceinline__ void wire_scan(const Columns &c, const WireSrc &w, uint8_t *__restrict__ status,
                                          uint32_t *__restrict__ first_frame, const LeaderRuns *__restrict__ runs) {
    __shared__ __align__(16) uint8_t stage[kWireStage + 16];
    WireStage s;
    const uint32_t i = wire_block_frame(w, stage, s);
    if (i == kNoFrame) return;
    RecRegs rec;
    uint64_t hint, snap;
    const uint32_t st = wire_frame<kRuns>(c, runs, w, s, stage, i, rec, hint, snap);
    status[i] = static_cast<uint8_t>(st << 4);
    if (st == RAFTGPU_WIRE_OK) {
        const uint32_t g = static_cast<uint32_t>(rec.w0), slot = static_cast<uint32_t>(rec.w0 >> 32) & 0xffu;
        if (slot < kSlots) atomicMin(&first_frame[static_cast<size_t>(slot) * c.cap + g], i);
    }
}
// With the runs, at least 6 blocks per SM, so ptxas works to a cap of 40 registers (it takes 35, allocated as 40: 6 blocks
// of 256 threads per SM, where the 32-register <false> kernel fits 8).  At __launch_bounds__(kWireThreads) alone ptxas
// settles on 32 registers and spills 24 bytes, as it does in hb_wire_scan_kernel.
template <bool kRuns>
__global__ void __launch_bounds__(kWireThreads, kRuns ? 6 : 0) wire_scan_kernel(Columns c, WireSrc w, uint8_t *__restrict__ status,
                                                                 uint32_t *__restrict__ first_frame,
                                                                 const LeaderRuns *__restrict__ runs) {
    wire_scan<kRuns>(c, w, status, first_frame, runs);
}

// Pass 2: the first frame of every cell is applied (raft.rs:1663-1743), later ones are RAFTGPU_WIRE_DUP.
// status[i] = wire status << 4 | RAFTGPU_RES_* of the applied message.
template <bool kRuns>
__global__ void __launch_bounds__(kWireThreads) wire_apply_kernel(Columns c, WireSrc w, uint8_t *__restrict__ status,
                                                                  const uint32_t *__restrict__ first_frame,
                                                                  unsigned long long *__restrict__ counters,
                                                                  uint32_t *__restrict__ dup_count,
                                                                  const LeaderRuns *__restrict__ runs) {
    __shared__ __align__(16) uint8_t stage[kWireStage + 16];
    uint32_t local[5] = {0, 0, 0, 0, 0};  // records, updates, rejects, decrements, no_progress
    // the prologue of wire_block_frame written out: through the helper, ptxas spills in this kernel
    const uint32_t first = blockIdx.x * kWireThreads;
    if (first < w.n) {  // (every thread goes on to block_flush_counts)
        const uint32_t last = min(first + kWireThreads, w.n);
        const WireStage s = wire_stage_block(w, first, last, stage);
        const uint32_t i = first + threadIdx.x;
        if (i < last && status[i] == (RAFTGPU_WIRE_OK << 4)) {
            RecRegs rec;
            uint64_t hint, snap;
            wire_frame<kRuns>(c, runs, w, s, stage, i, rec, hint, snap);  // same verdict as in the scan pass
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

// ---------------------------------------------------------------------------
// Waves (raftgpu_arena_set_wire_waves, DESIGN 3.19): the pass above repeated over the frames it left DUP, in their batch
// order, until `waves` runs are done or no frame is left.  Wave 1 is the scan kernel above and wire_wave_apply_kernel
// over the whole batch; every later wave is wire_wave_claim_kernel<false> and wire_wave_apply_kernel over the list the wave
// before it wrote, so its cost follows its frames, not the batch or the arena.  The first-frame table is filled with
// 0xff once per call: the frame that takes a cell clears the cell's entry again, so the next wave finds it free.
// kNoFrame = free; kWaveStop (k_app_follow.cuh's waves only) = the group's claimant was not applied.
constexpr uint32_t kWaveStop = 0xfffffffeu;

// A wave's frames: its list (nullptr = the whole batch, wave 1) and count, and the list and count of the frames it
// leaves DUP for the next wave.
struct WaveIo {
    const uint32_t *in, *in_n;
    uint32_t *out, *out_n;
};

// Every lane of a full warp: frame i goes on the next wave's list when dup.
__device__ __forceinline__ void wave_enlist(const WaveIo &io, bool dup, uint32_t i) {
    const uint32_t at = warp_reserve(io.out_n, dup ? 1u : 0u);
    if (dup) io.out[at] = i;
}

// The u32 LE header of frame i, read from the batch (a frame on a wave list was opened by wave 1).
__device__ __forceinline__ uint32_t wire_header(const WireSrc &w, uint32_t i) {
    const uint8_t *p = w.bytes + w.offsets[i];
    return p[0] | (static_cast<uint32_t>(p[1]) << 8) | (static_cast<uint32_t>(p[2]) << 16) | (static_cast<uint32_t>(p[3]) << 24);
}

// Wave j >= 2, pass 1: every frame on the list claims its cell (kGroup: its group, k_app_follow.cuh's waves, unless the
// group is stopped).  A listed frame reached the decision in every wave before -- what it is decided on beyond that
// (committed, last_index, the run, matched) does not move it out -- so the lowest listed frame of a cell is the one that
// takes it, and the header alone names the cell.
template <bool kGroup>
__global__ void __launch_bounds__(kWireThreads) wire_wave_claim_kernel(WireSrc w, uint32_t cap, uint32_t *__restrict__ first_frame,
                                                                       const uint32_t *__restrict__ list,
                                                                       const uint32_t *__restrict__ list_n) {
    const uint32_t n = *list_n;
    for (uint32_t k = blockIdx.x * kWireThreads + threadIdx.x; k < n; k += gridDim.x * kWireThreads) {
        const uint32_t i = list[k], hdr = wire_header(w, i);
        if constexpr (kGroup) {
            if (first_frame[hdr >> 4] != kWaveStop) atomicMin(&first_frame[hdr >> 4], i);  // (a stopped entry never moves)
        } else {
            atomicMin(&first_frame[static_cast<size_t>(hdr & 15u) * cap + (hdr >> 4)], i);  // (slot < kSlots: it was DUP)
        }
    }
}

// The apply pass of a wave: wire_apply_kernel's rule, the cell's entry cleared by the frame that takes it, and every DUP
// frame put on io.out.  io.in == nullptr (wave 1): every frame of the batch the scan left OK, staged as there; else the
// frames of io.in, read from global memory, over a grid-stride loop (a wave that finds no frame returns at once), where
// a frame that does not take its cell stays DUP untouched.
template <bool kRuns>
__global__ void __launch_bounds__(kWireThreads) wire_wave_apply_kernel(Columns c, WireSrc w, uint8_t *__restrict__ status,
                                                                       uint32_t *__restrict__ first_frame,
                                                                       unsigned long long *__restrict__ counters,
                                                                       const LeaderRuns *__restrict__ runs, WaveIo io) {
    __shared__ __align__(16) uint8_t stage[kWireStage + 16];
    uint32_t local[5] = {0, 0, 0, 0, 0};  // records, updates, rejects, decrements, no_progress
    const uint32_t n = io.in ? *io.in_n : w.n;
    if (n == 0) return;
    const uint32_t stride = io.in ? gridDim.x * kWireThreads : w.n;  // (wave 1: one tile per block, the stage used once)
    for (uint32_t k0 = blockIdx.x * kWireThreads; k0 < n; k0 += stride) {  // (uniform per block)
        const uint32_t last = min(k0 + kWireThreads, n), k = k0 + threadIdx.x;
        WireStage s{0, 0, 0, false};
        if (!io.in) s = wire_stage_block(w, k0, last, stage);
        const uint32_t i = k < last ? (io.in ? io.in[k] : k) : kNoFrame;
        bool dup = false;
        uint32_t *cell = nullptr;
        if (i != kNoFrame && io.in) {  // a listed frame is DUP already: only the one that takes its cell is decoded
            const uint32_t hdr = wire_header(w, i);
            cell = &first_frame[static_cast<size_t>(hdr & 15u) * c.cap + (hdr >> 4)];
            dup = *cell != i;
        }
        if (i != kNoFrame && !dup && (io.in || status[i] == (RAFTGPU_WIRE_OK << 4))) {
            RecRegs rec;
            uint64_t hint, snap;
            wire_frame<kRuns>(c, runs, w, s, stage, i, rec, hint, snap);  // same verdict as in wave 1's scan
            const uint32_t g = static_cast<uint32_t>(rec.w0), slot = static_cast<uint32_t>(rec.w0 >> 32) & 0xffu;
            if (!io.in) cell = slot < kSlots ? &first_frame[static_cast<size_t>(slot) * c.cap + g] : nullptr;
            if (cell && *cell != i) {
                status[i] = static_cast<uint8_t>(RAFTGPU_WIRE_DUP << 4);
                dup = true;
            } else {
                if (cell) *cell = kNoFrame;  // (the cell's other frames read i or kNoFrame: DUP either way)
                const CellRegs cr = load_cell(c, rec);
                const CellPtrs gp = global_cell_ptrs(c, rec);
                const uint32_t res = apply_one<2>(c, nullptr, hint, snap, rec, cr, gp, local);
                status[i] = static_cast<uint8_t>((RAFTGPU_WIRE_OK << 4) | (res & 0xfu));
            }
        }
        wave_enlist(io, dup, i);
    }
    const int which[5] = {kCntRecords, kCntUpdates, kCntRejects, kCntDecrements, kCntNoProgress};
    block_flush_counts<5>(local, which, counters, nullptr);
}

// Clears or states leader-run rows: rows[i] of the list go to row group[i] (raftgpu_leader_runs_set, after its checks).
__global__ void leader_runs_set_kernel(LeaderRuns *__restrict__ dst, const raftgpu_leader_runs *__restrict__ rows, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const raftgpu_leader_runs r = rows[i];
    dst[r.group] = LeaderRuns{make_ulonglong2(r.term, r.term_start), make_ulonglong2(r.run_start[0], r.run_start[1]),
                              make_ulonglong2(r.run_term[0], r.run_term[1])};
}

// ---------------------------------------------------------------------------
// The encoder: heartbeat-kind frames (MsgHeartbeat at the leader, MsgHeartbeatResponse at the follower), and the
// block-output code of the passes that write them -- a block scan of {frames, bytes}, the one-block scan of the block
// sums (block_starts_kernel) and the 16-byte store of a block's contiguous output.

constexpr uint32_t kWireHbFrameMax = 60;  // 4-byte header + at most 56 bytes of Message
constexpr uint32_t kScanThreads = 1024;  // block_starts_kernel

// bytes of v as a base-128 varint
__device__ __forceinline__ uint32_t wire_varint_len(uint64_t v) {
    return v ? (70u - static_cast<uint32_t>(__clzll(static_cast<long long>(v)))) / 7u : 1u;
}

// Bytes of a heartbeat-kind frame (MsgHeartbeat, k_hb_frames.cuh; MsgHeartbeatResponse, k_hb_follow.cuh) before its
// `to` and `commit`: header, msg_type, from, term (never 0 on these paths) and the 8-byte context when there is one.
__device__ __forceinline__ uint32_t wire_hb_fixed_len(uint64_t from, uint64_t term, bool has_ctx) {
    return 4u + 2u + (from ? 1u + wire_varint_len(from) : 0u) + 1u + wire_varint_len(term) + (has_ctx ? 10u : 0u);
}

// Bytes of the frame to a peer with id `to` and commit `commit`, after the fields its group's frames share (`fixed`,
// wire_hb_fixed_len).
__device__ __forceinline__ uint32_t wire_hb_len(uint32_t fixed, uint64_t to, uint64_t commit) {
    return fixed + (to ? 1u + wire_varint_len(to) : 0u) + (commit ? 1u + wire_varint_len(commit) : 0u);
}

__device__ __forceinline__ uint8_t *wire_put_varint(uint8_t *p, uint64_t v) {
    while (v >= 0x80u) {
        *p++ = static_cast<uint8_t>(v | 0x80u);
        v >>= 7;
    }
    *p++ = static_cast<uint8_t>(v);
    return p;
}

// What every frame starts with: the u32 LE header, then the Message's field 1, msg_type (never 0 on these paths).
__device__ __forceinline__ uint8_t *wire_put_head(uint8_t *p, uint32_t hdr, uint8_t type) {
    p[0] = static_cast<uint8_t>(hdr);
    p[1] = static_cast<uint8_t>(hdr >> 8);
    p[2] = static_cast<uint8_t>(hdr >> 16);
    p[3] = static_cast<uint8_t>(hdr >> 24);
    p[4] = 0x08;  // field 1, varint
    p[5] = type;
    return p + 6;
}

// One heartbeat-kind frame: u32 LE header, then eraftpb.Message (eraftpb.proto:71-92) in field-number order with zero
// scalars omitted: 1 msg_type = kType (MsgHeartbeat 8, MsgHeartbeatResponse 9, eraftpb.proto:58-59), 2 to, 3 from,
// 4 term (never 0 on these paths), 8 commit, 12 context (the 8 little-endian bytes of ctx when has_ctx).
template <uint8_t kType>
__device__ __forceinline__ uint8_t *wire_put_hb_frame(uint8_t *p, uint32_t hdr, uint64_t to, uint64_t from, uint64_t term,
                                                 uint64_t commit, bool has_ctx, uint64_t ctx) {
    p = wire_put_head(p, hdr, kType);
    if (to) {
        *p++ = 0x10;
        p = wire_put_varint(p, to);
    }
    if (from) {
        *p++ = 0x18;
        p = wire_put_varint(p, from);
    }
    *p++ = 0x20;
    p = wire_put_varint(p, term);
    if (commit) {
        *p++ = 0x40;
        p = wire_put_varint(p, commit);
    }
    if (has_ctx) {
        p[0] = 0x62;
        p[1] = 8;
#pragma unroll
        for (int k = 0; k < 8; k++) p[2 + k] = static_cast<uint8_t>(ctx >> (8 * k));
        p += 10;
    }
    return p;
}

// A vote response (MsgRequestVoteResponse 6, MsgRequestPreVoteResponse 18; k_vote_request.cuh): u32 LE header, then
// eraftpb.Message in field-number order with zero scalars omitted, as raftgpu_synth_wire_encode_votes writes it:
// 1 msg_type, 2 to, 3 from, 4 term, 8 commit, 10 reject, 15 commit_term.  At most 4 + 2 + 5 * 11 + 2 = 63 bytes.
constexpr uint32_t kWireVoteFrameMax = 64;

// bytes of the frame, header included
__device__ __forceinline__ uint32_t wire_vote_len(uint64_t to, uint64_t from, uint64_t term, uint64_t commit, bool reject,
                                                  uint64_t commit_term) {
    return 6u + (to ? 1u + wire_varint_len(to) : 0u) + (from ? 1u + wire_varint_len(from) : 0u) +
           (term ? 1u + wire_varint_len(term) : 0u) + (commit ? 1u + wire_varint_len(commit) : 0u) + (reject ? 2u : 0u) +
           (commit_term ? 1u + wire_varint_len(commit_term) : 0u);
}

__device__ __forceinline__ uint8_t *wire_put_vote_frame(uint8_t *p, uint32_t hdr, uint8_t type, uint64_t to, uint64_t from,
                                                        uint64_t term, uint64_t commit, bool reject, uint64_t commit_term) {
    p = wire_put_head(p, hdr, type);
    const uint8_t tags[4] = {0x10, 0x18, 0x20, 0x40};  // fields 2, 3, 4, 8
    const uint64_t vals[4] = {to, from, term, commit};
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (vals[k]) {
            *p++ = tags[k];
            p = wire_put_varint(p, vals[k]);
        }
    }
    if (reject) {
        p[0] = 0x50;  // field 10
        p[1] = 1;
        p += 2;
    }
    if (commit_term) {
        *p++ = 0x78;  // field 15
        p = wire_put_varint(p, commit_term);
    }
    return p;
}

// An entry-less MsgAppend (msg_type 3; k_app_frames.cuh): u32 LE header, then eraftpb.Message in field-number order
// with zero scalars omitted: 1 msg_type, 2 to, 3 from, 4 term, 5 log_term, 6 index, 8 commit.  At most 4 + 2 + 6 * 11 =
// 72 bytes.
constexpr uint32_t kWireAppFrameMax = 72;

// bytes of the frame, header included
__device__ __forceinline__ uint32_t wire_app_len(uint64_t to, uint64_t from, uint64_t term, uint64_t log_term, uint64_t index,
                                                 uint64_t commit) {
    const uint64_t vals[6] = {to, from, term, log_term, index, commit};
    uint32_t len = 6u;
#pragma unroll
    for (int k = 0; k < 6; k++) len += vals[k] ? 1u + wire_varint_len(vals[k]) : 0u;
    return len;
}

// kType: MsgAppend 3 here; MsgAppendResponse 4 (eraftpb.proto:53-54) writes these fields before its own.
template <uint8_t kType>
__device__ __forceinline__ uint8_t *wire_put_append_frame(uint8_t *p, uint32_t hdr, uint64_t to, uint64_t from, uint64_t term,
                                                          uint64_t log_term, uint64_t index, uint64_t commit) {
    p = wire_put_head(p, hdr, kType);
    const uint8_t tags[6] = {0x10, 0x18, 0x20, 0x28, 0x30, 0x40};  // fields 2, 3, 4, 5, 6, 8
    const uint64_t vals[6] = {to, from, term, log_term, index, commit};
#pragma unroll
    for (int k = 0; k < 6; k++) {
        if (vals[k]) {
            *p++ = tags[k];
            p = wire_put_varint(p, vals[k]);
        }
    }
    return p;
}

// A MsgAppendResponse (msg_type 4; k_app_follow.cuh): u32 LE header, then eraftpb.Message in field-number order with
// zero scalars omitted, as raftgpu_synth_wire_encode writes it: 1 msg_type, 2 to, 3 from, 4 term, 5 log_term, 6 index,
// 8 commit, 10 reject, 11 reject_hint.  At most 4 + 2 + 6 * 11 + 2 + 11 = 85 bytes.
constexpr uint32_t kWireAppRespFrameMax = 85;

// bytes of the frame, header included
__device__ __forceinline__ uint32_t wire_app_resp_len(uint64_t to, uint64_t from, uint64_t term, uint64_t log_term,
                                                      uint64_t index, uint64_t commit, bool reject, uint64_t reject_hint) {
    return wire_app_len(to, from, term, log_term, index, commit) + (reject ? 2u : 0u) +
           (reject_hint ? 1u + wire_varint_len(reject_hint) : 0u);
}

__device__ __forceinline__ uint8_t *wire_put_app_resp_frame(uint8_t *p, uint32_t hdr, uint64_t to, uint64_t from,
                                                            uint64_t term, uint64_t log_term, uint64_t index,
                                                            uint64_t commit, bool reject, uint64_t reject_hint) {
    p = wire_put_append_frame<4>(p, hdr, to, from, term, log_term, index, commit);
    if (reject) {
        p[0] = 0x50;  // field 10
        p[1] = 1;
        p += 2;
    }
    if (reject_hint) {
        *p++ = 0x58;  // field 11
        p = wire_put_varint(p, reject_hint);
    }
    return p;
}

// Exclusive scan of two u32 counts over a block of W warps; *tot_a / *tot_b = the block's sums (every thread).
template <uint32_t W>
__device__ __forceinline__ void wire_block_scan(uint32_t &a, uint32_t &b, uint32_t &tot_a, uint32_t &tot_b) {
    __shared__ uint32_t wa[W], wb[W];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    uint32_t ia = a, ib = b;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t va = __shfl_up_sync(0xffffffffu, ia, d), vb = __shfl_up_sync(0xffffffffu, ib, d);
        if (lane >= static_cast<uint32_t>(d)) {
            ia += va;
            ib += vb;
        }
    }
    if (lane == 31) {
        wa[warp] = ia;
        wb[warp] = ib;
    }
    __syncthreads();
    if (warp == 0) {
        uint32_t xa = lane < W ? wa[lane] : 0u, xb = lane < W ? wb[lane] : 0u;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t va = __shfl_up_sync(0xffffffffu, xa, d), vb = __shfl_up_sync(0xffffffffu, xb, d);
            if (lane >= static_cast<uint32_t>(d)) {
                xa += va;
                xb += vb;
            }
        }
        if (lane < W) {  // inclusive -> the warps' exclusive starts, the sums behind them
            wa[lane] = xa;
            wb[lane] = xb;
        }
    }
    __syncthreads();
    tot_a = wa[W - 1];
    tot_b = wb[W - 1];
    const uint32_t sa = warp ? wa[warp - 1] : 0u, sb = warp ? wb[warp - 1] : 0u;
    a = sa + ia - a;
    b = sb + ib - b;
    __syncthreads();  // wa / wb may be reused by the caller's next scan
}

// One block: blk's counts become each block's exclusive starts.  K = u32 per block in blk: {count} (K = 1), {frames,
// bytes} (K = 2) or {frames, bytes, leaders without a term} (K = 3); totals = the K sums.  offsets (K >= 2, nullable):
// offsets[frames] = bytes, the end of the last frame, for a caller whose outputs always fit; a pass that may not fit
// writes it where it decides the fit.
template <uint32_t K>
__global__ void __launch_bounds__(kScanThreads) block_starts_kernel(uint32_t *__restrict__ blk, uint32_t nb,
                                                                    uint64_t *__restrict__ totals,
                                                                    uint32_t *__restrict__ offsets) {
    static_assert(K >= 1 && K <= 3, "blk holds {count} or {frames, bytes[, leaders without a term]} per block");
    uint32_t carry_f = 0, carry_b = 0, no_term = 0;
    for (uint32_t j0 = 0; j0 < nb; j0 += kScanThreads) {  // (uniform trip count: every thread reaches the scan)
        const uint32_t j = j0 + threadIdx.x;
        uint32_t f = 0, b = 0;
        if (j < nb) {
            f = blk[K * j];
            if constexpr (K >= 2) b = blk[K * j + 1];
            if constexpr (K == 3) no_term += blk[K * j + 2];
        }
        uint32_t tf, tb;
        wire_block_scan<kScanThreads / 32>(f, b, tf, tb);
        if (j < nb) {
            blk[K * j] = carry_f + f;
            if constexpr (K >= 2) blk[K * j + 1] = carry_b + b;
        }
        carry_f += tf;
        carry_b += tb;
    }
    if constexpr (K == 1) {
        if (threadIdx.x == 0) totals[0] = carry_f;
        return;
    }
    uint64_t t = 0;
    if constexpr (K == 3) {
        no_term = __reduce_add_sync(0xffffffffu, no_term);
        __shared__ uint32_t nt[kScanThreads / 32];
        if ((threadIdx.x & 31u) == 0) nt[threadIdx.x >> 5] = no_term;
        __syncthreads();
        if (threadIdx.x == 0)
            for (uint32_t w = 0; w < kScanThreads / 32; w++) t += nt[w];
    }
    if (threadIdx.x == 0) {
        totals[0] = carry_f;
        totals[1] = carry_b;
        if constexpr (K == 3) totals[2] = t;
        if (offsets) offsets[carry_f] = carry_b;
    }
}

// A block's contiguous output [b0, b0 + nbytes) from shared memory, where it was assembled at buf + (b0 & 15): whole
// 16-byte chunks go out as uint4 stores, only the two chunks shared with the neighbouring blocks byte by byte.
template <uint32_t kThreads>
__device__ __forceinline__ void wire_store_block(uint8_t *__restrict__ out, const uint8_t *buf, uint32_t b0, uint32_t nbytes) {
    const uint32_t a0 = b0 & ~15u, end = b0 + nbytes;
    for (uint32_t q = a0 + 16u * threadIdx.x; q < end; q += 16u * kThreads) {
        const uint8_t *src = buf + (q - a0);
        if (q >= b0 && q + 16u <= end) {
            *reinterpret_cast<uint4 *>(out + q) = *reinterpret_cast<const uint4 *>(src);
        } else {
            for (uint32_t k = 0; k < 16u; k++)
                if (q + k >= b0 && q + k < end) out[q + k] = src[k];
        }
    }
}

// The last pass of a pass that answers frames with frames (k_hb_follow.cuh, k_vote_request.cuh), after block_starts_kernel<2>
// turned blk into block starts: every block encodes its responses, in frame order, into shared memory at their offset
// from the 16-byte boundary below the block's start and stores them with wire_store_block; offsets [blk start, + its
// responses).  P holds what the pass knows at compile time: Rec (its record per frame), kFrameMax (bytes of its
// largest response), answers(status) (the frame has a response), len(rec) and put(p, rec) (the response's bytes and its
// encoder).  Launched with kWireThreads threads per block, as the pass's scan and apply kernels.  Reads 1 per frame +
// sizeof(Rec) per response; writes the responses and 4 per response.
template <class P>
__global__ void __launch_bounds__(kWireThreads) reply_write_kernel(uint32_t n, const uint8_t *__restrict__ status,
                                                                   const typename P::Rec *__restrict__ recs,
                                                                   const uint32_t *__restrict__ blk, uint8_t *__restrict__ out,
                                                                   uint32_t *__restrict__ offsets) {
    __shared__ __align__(16) uint8_t buf[kWireThreads * P::kFrameMax + 16];
    __shared__ uint32_t offs[kWireThreads];
    const uint32_t i = blockIdx.x * kWireThreads + threadIdx.x;
    const bool has = i < n && P::answers(status[i]);
    typename P::Rec r{};
    if (has) r = recs[i];
    uint32_t lf = has, lb = has ? P::len(r) : 0u, nf, nbytes;
    wire_block_scan<kWireThreads / 32>(lf, lb, nf, nbytes);
    const uint32_t f0 = blk[2 * blockIdx.x], b0 = blk[2 * blockIdx.x + 1], pad = b0 & 15u;
    if (has) {
        offs[lf] = b0 + lb;
        P::put(buf + pad + lb, r);
    }
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < nf; j += kWireThreads) offsets[f0 + j] = offs[j];
    wire_store_block<kWireThreads>(out, buf, b0, nbytes);
}
