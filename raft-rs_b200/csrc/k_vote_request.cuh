// k_vote_request.cuh -- MsgRequestVote / MsgRequestPreVote frames at a voter (DESIGN 3.14): Raft::step's term rules
// (raft.rs:1280-1411), then the MsgRequestVote | MsgRequestPreVote arm (raft.rs:1418-1462) and one response through
// send (raft.rs:602-661) for the first frame of every group that reaches the term rules.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).
//
// Role, vote, leader and lease stay with the caller: its table (raftgpu_voter, one row per group slot) is read only.
// The frame's header is the voter's own (group << 4 | x); x is not read and goes back unchanged in the response's header.
// A group's frames are decided one per batch, in frame order: each decision reads what an earlier one may change.
//
// Four kernels and no waiting between blocks: vrq_scan_kernel stages and decodes every frame once, classifies and
// decides it and writes a 48-byte record per frame that reached the term rules; vrq_apply_kernel marks the later frames
// of a group DUP, raises the term and resets the group where the first one bumps it, and sums the responses per block;
// block_starts_kernel<2> (k_wire.cuh) turns the sums into block starts; reply_write_kernel<VrqReply> (k_wire.cuh) encodes
// the responses (wire_put_vote_frame) and stores them through shared memory.  Every kernel takes kWireThreads frames per
// block: one block sum per scan block.
//
// kLeader (DESIGN 3.24): the same frames at a leader (term_start != RAFTGPU_NO_TERM_START; SELECT is not read).  Only
// a group's claimant b(g) changes state -- its first MsgRequestVote above the term that the lease does not drop, or a
// granted MsgRequestVote at the term -- so the frames before it are decided against the unchanged leader, b(g) is
// applied, and only the frames after it are DUP.  COMMIT_VOTE is tested on the bumped path alone: maybe_commit_by_vote
// returns at once for a Leader (raft.rs:2131).

// A decided frame's record: w0 = its header | the kVrq* bits; the response's to (= m.from), from (the table's id),
// term, commit and commit_term.  A bumped frame's new term is its response's term (m.term: a bump is only decided at
// m.term, and its grant and its rejection both answer at it).
constexpr uint64_t kVrqPre = 1ull << 32, kVrqReject = 1ull << 33, kVrqBumped = 1ull << 34, kVrqVoted = 1ull << 35;
struct __align__(16) VrqRec {
    uint64_t w0, to, from, term, commit, commit_term;
};

__device__ __forceinline__ uint32_t vrq_len(const VrqRec &r) {
    return wire_vote_len(r.to, r.from, r.term, r.commit, (r.w0 & kVrqReject) != 0, r.commit_term);
}

// m.context == CAMPAIGN_TRANSFER (raft.rs:57, 1288): the 16 bytes "CampaignTransfer" as two little-endian words
__device__ __forceinline__ bool vrq_transfer(const WireMsg &m, const uint8_t *msg) {
    return m.ctx_len == 16u && wire_ctx_u64(msg + m.ctx_off) == 0x6e676961706d6143ull &&
           wire_ctx_u64(msg + m.ctx_off + 8) == 0x726566736e617254ull;
}

// Frame i: its status before the duplicate rule (checks in the order of raftgpu.h) and, for the frames that reach the
// term rules (OK, IGNORED, COMMIT_VOTE), its record (w0 alone for the last two).  kLeader: a claimant's w0 has
// kVrqBumped or kVrqVoted.
template <bool kLeader>
__device__ __forceinline__ uint32_t vrq_frame(const Columns &c, const WireSrc &w, const raftgpu_voter *__restrict__ voters,
                                              const WireStage &s, const uint8_t *stage, uint32_t i, VrqRec &r) {
    uint32_t hdr;
    const uint8_t *msg;
    WireMsg m;
    if (wire_open<true, true, true, true>(w, s, stage, i, hdr, msg, m) != RAFTGPU_WIRE_OK) return RAFTGPU_WIRE_MALFORMED;
    const uint32_t g = hdr >> 4, meta = c.meta[g];
    if (meta & RAFTGPU_META_WIDE_HI) return RAFTGPU_WIRE_MALFORMED;
    if (m.msg_type != 5u && m.msg_type != 17u) return RAFTGPU_WIRE_SKIP_TYPE;  // eraftpb.proto:55, 67
    const raftgpu_voter &v = voters[g];
    const uint32_t flags = v.flags;
    if constexpr (kLeader) {
        if (c.term_start[g] == RAFTGPU_NO_TERM_START) return RAFTGPU_WIRE_ROLE;
    } else {
        if (!(flags & RAFTGPU_VOTER_SELECT) || c.term_start[g] != RAFTGPU_NO_TERM_START) return RAFTGPU_WIRE_ROLE;
    }
    const uint64_t term = c.term[g];
    if (term == 0 || m.term == 0) return RAFTGPU_WIRE_TERM;
    const bool pre = m.msg_type == 17u;
    r.w0 = hdr | (pre ? kVrqPre : 0ull);
    r.to = m.from;  // new_message(m.from, ..) (raft.rs:1395, 1441, 1453)
    r.from = v.id;  // send: from = self.id (raft.rs:610-612)
    r.commit = r.commit_term = 0;
    uint64_t vote = v.vote;
    bool leader = flags & RAFTGPU_VOTER_LEADER;
    if (m.term > term) {
        // raft.rs:1288-1316: in lease and not forced, the request is dropped
        if ((flags & RAFTGPU_VOTER_LEASE) && !vrq_transfer(m, msg))
            return RAFTGPU_WIRE_IGNORED;
        if (!pre) {  // become_follower(m.term, INVALID_ID) (raft.rs:1346): vote and leader_id are reset
            r.w0 |= kVrqBumped;
            vote = 0;
            leader = false;
        }
    } else if (m.term < term) {
        if (!pre) return RAFTGPU_WIRE_IGNORED;  // raft.rs:1399-1409
        r.w0 |= kVrqReject;                     // raft.rs:1395-1398: rejected at our term, no commit fields
        r.term = term;
        return RAFTGPU_WIRE_OK;
    }
    uint64_t last = c.last_index[g], committed = c.committed[g];
    if (meta & RAFTGPU_META_WIDE_LO) {
        last = umax64(last, c.last_index[g + 1]);
        committed = umax64(committed, c.committed[g + 1]);
    }
    const uint64_t last_term = v.last_term;
    // raft.rs:1420-1428: can_vote, is_up_to_date (raft_log.rs:412-414), the priority rule
    const bool can_vote = vote == m.from || (vote == 0 && !leader) || (pre && m.term > term);
    if (can_vote && (m.log_term > last_term || (m.log_term == last_term && m.index >= last)) &&
        (m.index > last || v.priority <= m.priority)) {
        r.term = m.term;
        if (!pre) r.w0 |= kVrqVoted;
        return RAFTGPU_WIRE_OK;
    }
    // maybe_commit_by_vote (raft.rs:2126-2164) would read the caller's log; a leader's returns at once (:2131)
    if ((!kLeader || (r.w0 & kVrqBumped)) && m.commit != 0 && m.commit_term != 0 && m.commit > committed)
        return RAFTGPU_WIRE_COMMIT_VOTE;
    r.w0 |= kVrqReject;
    r.term = (r.w0 & kVrqBumped) ? m.term : term;
    r.commit = committed;  // raft_log.commit_info() (raft.rs:1456-1458)
    r.commit_term = v.commit_term;
    return RAFTGPU_WIRE_OK;
}

// Pass 1: classify every frame; status[i] = wire status << 4; the record of a frame that reached the term rules,
// first_frame[group] = the lowest such frame of the group.  Launched with kWireThreads threads per block.
// kLeader: first_frame[group] = the group's claimant b(g), and out[2 i..] (nullable) = {m.from, the group's term} of
// every OK frame, 0 otherwise -- the term before b(g)'s bump, which the apply pass of the frames before b(g) could not
// read while b(g) writes it.
template <bool kLeader>
__global__ void __launch_bounds__(kWireThreads) vrq_scan_kernel(Columns c, WireSrc w, const raftgpu_voter *__restrict__ voters,
                                                                uint8_t *__restrict__ status, VrqRec *__restrict__ recs,
                                                                uint32_t *__restrict__ first_frame, uint64_t *__restrict__ out) {
    __shared__ __align__(16) uint8_t stage[kWireStage + 16];
    WireStage s;
    const uint32_t i = wire_block_frame(w, stage, s);
    if (i == kNoFrame) return;
    VrqRec r;
    const uint32_t st = vrq_frame<kLeader>(c, w, voters, s, stage, i, r);
    status[i] = static_cast<uint8_t>(st << 4);
    if constexpr (kLeader) {
        if (out) {
            const bool ok = st == RAFTGPU_WIRE_OK;
            out[2ull * i] = ok ? r.to : 0;
            out[2ull * i + 1] = ok ? c.term[static_cast<uint32_t>(r.w0) >> 4] : 0;
        }
    }
    if (st == RAFTGPU_WIRE_OK) recs[i] = r;
    else if (st == RAFTGPU_WIRE_IGNORED || st == RAFTGPU_WIRE_COMMIT_VOTE) recs[i].w0 = r.w0;
    else return;
    if (!kLeader || (r.w0 & (kVrqBumped | kVrqVoted))) atomicMin(&first_frame[static_cast<uint32_t>(r.w0) >> 4], i);
}

// become_follower(term, ..)'s arena part (raft.rs:1087-1096) for group g, a wide pair by its low half: the term, then
// reset_group on both halves with RAFTGPU_CTL_RESET's arguments -- no term_start, last_index and committed (the larger
// of the halves'), the table's persisted -- exactly as RAFTGPU_CTL_SET_TERM + RAFTGPU_CTL_RESET.  Shared by the two
// passes that raise a follower's term: vrq_apply_kernel here and ftm_apply_kernel (k_follow_term.cuh).
__device__ __forceinline__ void become_follower_arena(const Columns &c, uint32_t g, uint64_t term,
                                                      const raftgpu_voter *__restrict__ voters) {
    const bool wide = c.meta[g] & RAFTGPU_META_WIDE_LO;
    uint64_t last = c.last_index[g], committed = c.committed[g];
    if (wide) {
        last = umax64(last, c.last_index[g + 1]);
        committed = umax64(committed, c.committed[g + 1]);
    }
    const uint64_t persisted = voters[g].persisted;
    c.term[g] = term;
    reset_group(c, g, RAFTGPU_NO_TERM_START, last, committed, persisted);
    if (wide) {
        c.term[g + 1] = term;
        reset_group(c, g + 1, RAFTGPU_NO_TERM_START, last, committed, persisted);
    }
}

// Pass 2: a later frame of a group is RAFTGPU_WIRE_DUP.  The first one, when OK, is applied: a bump sets the term and
// resets both halves of a pair (reset_group with RAFTGPU_CTL_RESET's arguments: no term_start, last_index, committed,
// the table's persisted), exactly as RAFTGPU_CTL_SET_TERM + RAFTGPU_CTL_RESET.  out[2 i..] (nullable) = {m.from, the
// term after} of an applied frame, 0 otherwise.  blk[2 * block + {0, 1}] = the block's responses and their bytes.
// kLeader: the frames after b(g) are DUP, b(g) is applied as the first frame is, and the OK frames before it answer
// with nothing applied (their out is the scan's).
// Algorithmic bytes per frame: 1 read + 1 written (+ 16 out); per frame that reached the term rules 8 (w0) + 4
// (first_frame) read; per applied one 40 (record) + 8 (term) read, and a bump's reset of its group.  kLeader: per
// frame 16 out written by the scan, here only for DUP frames and b(g); per OK frame before b(g) 40 (record) read.
template <bool kLeader>
__global__ void __launch_bounds__(kWireThreads) vrq_apply_kernel(Columns c, uint32_t n, const raftgpu_voter *__restrict__ voters,
                                                                 uint8_t *__restrict__ status, const VrqRec *__restrict__ recs,
                                                                 const uint32_t *__restrict__ first_frame,
                                                                 uint64_t *__restrict__ out, uint32_t *__restrict__ blk) {
    const uint32_t i = blockIdx.x * kWireThreads + threadIdx.x;
    uint32_t resp = 0, bytes = 0;
    if (i < n) {
        uint64_t from = 0, term = 0;
        bool put = !kLeader;  // kLeader: out is written for DUP frames and b(g) only
        const uint32_t st = status[i] >> 4;
        if (st == RAFTGPU_WIRE_OK || st == RAFTGPU_WIRE_IGNORED || st == RAFTGPU_WIRE_COMMIT_VOTE) {
            const uint64_t w0 = recs[i].w0;
            const uint32_t g = static_cast<uint32_t>(w0) >> 4, first = first_frame[g];
            if (kLeader ? i > first : first != i) {
                status[i] = static_cast<uint8_t>(RAFTGPU_WIRE_DUP << 4);
                put = true;
            } else if (st == RAFTGPU_WIRE_OK) {
                const VrqRec r = recs[i];
                if (!kLeader || i == first) {
                    term = c.term[g];
                    put = true;
                }
                if (w0 & kVrqBumped) {
                    term = r.term;
                    become_follower_arena(c, g, term, voters);
                }
                const uint32_t f = ((w0 & kVrqReject) ? 0u : RAFTGPU_VREQ_GRANTED) | ((w0 & kVrqVoted) ? RAFTGPU_VREQ_VOTED : 0u) |
                                   ((w0 & kVrqBumped) ? RAFTGPU_VREQ_BUMPED : 0u);
                status[i] = static_cast<uint8_t>((RAFTGPU_WIRE_OK << 4) | f);
                from = r.to;
                resp = 1;
                bytes = vrq_len(r);
            }
        }
        if (out && put) {
            out[2ull * i] = from;
            out[2ull * i + 1] = term;
        }
    }
    block_sums<2, kWireThreads>({resp, bytes}, blk);
}

// Pass 4 is reply_write_kernel<VrqReply> (k_wire.cuh): the frames that are still RAFTGPU_WIRE_OK after the apply pass
// answer.
struct VrqReply {
    using Rec = VrqRec;
    static constexpr uint32_t kFrameMax = kWireVoteFrameMax;
    __device__ __forceinline__ static bool answers(uint8_t status) { return (status >> 4) == RAFTGPU_WIRE_OK; }
    __device__ __forceinline__ static uint32_t len(const VrqRec &r) { return vrq_len(r); }
    __device__ __forceinline__ static uint8_t *put(uint8_t *p, const VrqRec &r) {  // vote_resp_msg_type, raft.rs:307-313
        return wire_put_vote_frame(p, static_cast<uint32_t>(r.w0), (r.w0 & kVrqPre) ? 18u : 6u, r.to, r.from, r.term, r.commit,
                                   (r.w0 & kVrqReject) != 0, r.commit_term);
    }
};
