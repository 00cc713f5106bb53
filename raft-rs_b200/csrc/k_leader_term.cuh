// k_leader_term.cuh -- the term prefix of Raft::step (raft.rs:1280-1411) and the drop arms of step_leader (:2111-2119)
// and step_follower for the frames that reach a leader (DESIGN 3.21): MsgAppend (3), MsgAppendResponse (4),
// MsgHeartbeat (8), MsgHeartbeatResponse (9), MsgRequestVoteResponse (6) and MsgRequestPreVoteResponse (18).  A higher
// term is become_follower(T, ..)'s arena part, a lower-term MsgAppend / MsgHeartbeat gets the empty MsgAppendResponse
// check_quorum or pre_vote asks for, and every frame step_leader or (after the bump) step_follower drops is settled here.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).
//
// Leadership is the arena's own: term_start != RAFTGPU_NO_TERM_START.  The caller's raftgpu_voter table gives id,
// persisted and RAFTGPU_VOTER_STALE_REPLY.  Types 4, 6, 9 and 18 carry the leader's cell (a wide pair's high half stands
// for the pair's low half); types 3 and 8 the group's own slot (group << 4 | x), with x copied into the reply.  Every
// frame gets its verdict in one call, from T = max(the group's term, every passing m.term that can raise it).
//
// Five kernels and no waiting between blocks: ltm_scan_kernel stages and decodes every frame once, classifies it,
// settles the pre-vote grants (which never raise the term, raft.rs:1319-1320), writes a FtmRec per other passing frame
// and atomicMax-es T into a per-group u64 table; ftm_claim_kernel (k_follow_term.cuh) lets the lowest frame at T > term
// claim its group; ltm_apply_kernel bumps the claimed groups and settles every frame from T, its own m.term and the
// bits its record carries, and sums the stale replies per block; block_starts_kernel<2> and reply_write_kernel<FtmReply>
// (k_wire.cuh) write the replies.  Every kernel takes kWireThreads frames per block.

// Bits of a record's w0 beyond k_follow_term.cuh's: the header (low 32 bits) is (pair's low half << 4 | x) and
// kFtmReply is set for a MsgAppend / MsgHeartbeat of a group with RAFTGPU_VOTER_STALE_REPLY.  kLtmAtTerm: m.term was
// the group's term when the pass began (the apply kernel must not read the term, which a claimant writes there);
// kLtmFollow: a MsgAppend or MsgHeartbeat (step_follower takes it after a bump); kLtmOwn: a MsgAppendResponse or
// MsgHeartbeatResponse (its own leader pass decides it at the term).  `to` = m.from for types 3 and 8, 0 otherwise:
// become_follower's leader_id (raft.rs:1340-1347) and the stale reply's to.
constexpr uint64_t kLtmAtTerm = 1ull << 33, kLtmFollow = 1ull << 34, kLtmOwn = 1ull << 35;

// Frame i: its status (checks in the order of raftgpu.h) and, for a frame left RAFTGPU_WIRE_OK, its record and T's
// candidate: the larger of m.term and the group's term.  A MsgRequestPreVoteResponse that grants is settled here:
// RAFTGPU_WIRE_STALE below the group's term, RAFTGPU_WIRE_IGNORED at or above it.
__device__ __forceinline__ uint32_t ltm_frame(const Columns &c, const WireSrc &w, const raftgpu_voter *__restrict__ voters,
                                              const WireStage &s, const uint8_t *stage, uint32_t i, FtmRec &r, uint64_t &top) {
    uint32_t hdr;
    const uint8_t *msg;
    WireMsg m;
    if (wire_open<false, true>(w, s, stage, i, hdr, msg, m) != RAFTGPU_WIRE_OK) return RAFTGPU_WIRE_MALFORMED;
    const uint32_t g = hdr >> 4, t = m.msg_type;
    const bool high = (c.meta[g] & RAFTGPU_META_WIDE_HI) != 0, follow = t == 3u || t == 8u;
    if (follow && high) return RAFTGPU_WIRE_MALFORMED;  // the follower's own slot: a pair is addressed by its low half
    if (!follow && t != 4u && t != 6u && t != 9u && t != 18u) return RAFTGPU_WIRE_SKIP_TYPE;  // eraftpb.proto:53-68
    const uint32_t lo = high ? g - 1 : g;
    if (c.term_start[lo] == RAFTGPU_NO_TERM_START) return RAFTGPU_WIRE_ROLE;
    const uint64_t term = c.term[lo];
    if (term == 0 || m.term == 0) return RAFTGPU_WIRE_TERM;  // m.term 0 is a local message
    if (t == 18u && !m.reject) return m.term < term ? RAFTGPU_WIRE_STALE : RAFTGPU_WIRE_IGNORED;
    r.w0 = (lo << 4 | (hdr & 15u)) | (m.term == term ? kLtmAtTerm : 0ull) |
           (follow ? kLtmFollow | ((voters[lo].flags & RAFTGPU_VOTER_STALE_REPLY) ? kFtmReply : 0ull) : 0ull) |
           ((t == 4u || t == 9u) ? kLtmOwn : 0ull);
    r.to = follow ? m.from : 0ull;
    r.term = m.term;
    top = umax64(m.term, term);
    return RAFTGPU_WIRE_OK;
}

// Pass 1: classify every frame; status[i] = wire status << 4; a passing frame's record (w0, to, term) and
// top[group] = max(top, m.term, term).  top covers [0, hi) and is zero before the pass.  Launched with kWireThreads
// threads per block.
__global__ void __launch_bounds__(kWireThreads) ltm_scan_kernel(Columns c, WireSrc w, const raftgpu_voter *__restrict__ voters,
                                                                uint8_t *__restrict__ status, FtmRec *__restrict__ recs,
                                                                unsigned long long *__restrict__ top) {
    __shared__ __align__(16) uint8_t stage[kWireStage + 16];
    WireStage s;
    const uint32_t i = wire_block_frame(w, stage, s);
    if (i == kNoFrame) return;
    FtmRec r;
    uint64_t t;
    const uint32_t st = ltm_frame(c, w, voters, s, stage, i, r, t);
    status[i] = static_cast<uint8_t>(st << 4);
    if (st != RAFTGPU_WIRE_OK) return;
    recs[i].w0 = r.w0;
    recs[i].to = r.to;
    recs[i].term = r.term;
    const uint32_t g = static_cast<uint32_t>(r.w0) >> 4;
    if (top[g] < t) atomicMax(&top[g], static_cast<unsigned long long>(t));
}

// Pass 2 is ftm_claim_kernel (k_follow_term.cuh): the lowest passing frame with m.term == T > term claims its group.

// Pass 3: the verdict of every passing frame, from T = top[group], its m.term and its record's bits -- never from the
// group's term, which the claimant writes in this kernel.  The claimant runs become_follower(T, ..)'s arena part
// (become_follower_arena) and keeps RAFTGPU_WIRE_OK | RAFTGPU_FTERM_BUMPED with out = {leader_id, T}.  A frame at the
// leader's term: RAFTGPU_WIRE_OK for types 4 and 9 (their own pass decided them), RAFTGPU_WIRE_IGNORED for the others
// (step_leader drops them).  Another frame at T > term: RAFTGPU_WIRE_OK for types 3 and 8 (the follower passes take
// them), RAFTGPU_WIRE_IGNORED for the others (step_follower drops them).  Any other frame is below T:
// RAFTGPU_WIRE_STALE, | RAFTGPU_RES_OK with its reply's record completed (from = the table's id, term = T) when
// kFtmReply is set.  out[2 i..] (nullable) = 0 for every frame but a claimant.  blk[2 * block + {0, 1}] = the block's
// replies and their bytes.  Algorithmic bytes per frame: 1 read + 1 written (+ 16 out); per passing frame 24 (record)
// + 8 (T) + 4 (first_frame) read; per stale reply 8 (id) read and 16 (record) written; per bump the reset of its group.
__global__ void __launch_bounds__(kWireThreads) ltm_apply_kernel(Columns c, uint32_t n, const raftgpu_voter *__restrict__ voters,
                                                                 uint8_t *__restrict__ status, FtmRec *__restrict__ recs,
                                                                 const unsigned long long *__restrict__ top,
                                                                 const uint32_t *__restrict__ first_frame,
                                                                 uint64_t *__restrict__ out, uint32_t *__restrict__ blk) {
    const uint32_t i = blockIdx.x * kWireThreads + threadIdx.x;
    uint32_t resp = 0, bytes = 0;
    if (i < n) {
        uint64_t from = 0, term = 0;
        if (status[i] == (RAFTGPU_WIRE_OK << 4)) {
            FtmRec r = recs[i];
            const uint32_t g = static_cast<uint32_t>(r.w0) >> 4;
            const uint64_t t = top[g];
            uint32_t st = RAFTGPU_WIRE_OK << 4;
            if (first_frame[g] == i) {
                become_follower_arena(c, g, t, voters);
                st |= RAFTGPU_FTERM_BUMPED;
                from = r.to;
                term = t;
            } else if (r.w0 & kLtmAtTerm) {
                if (!(r.w0 & kLtmOwn)) st = RAFTGPU_WIRE_IGNORED << 4;
            } else if (r.term == t) {
                if (!(r.w0 & kLtmFollow)) st = RAFTGPU_WIRE_IGNORED << 4;
            } else if (r.w0 & kFtmReply) {
                r.from = voters[g].id;  // send: from = self.id, term = self.term (raft.rs:610-650)
                recs[i].from = r.from;
                recs[i].term = r.term = t;
                st = (RAFTGPU_WIRE_STALE << 4) | RAFTGPU_RES_OK;
                resp = 1;
                bytes = ftm_len(r);
            } else {
                st = RAFTGPU_WIRE_STALE << 4;
            }
            status[i] = static_cast<uint8_t>(st);
        }
        if (out) {
            out[2ull * i] = from;
            out[2ull * i + 1] = term;
        }
    }
    block_sums<2, kWireThreads>({resp, bytes}, blk);
}

// Pass 5 is reply_write_kernel<FtmReply> (k_wire.cuh, k_follow_term.cuh): the stale MsgAppend / MsgHeartbeat frames the
// apply pass marked RAFTGPU_RES_OK answer.
