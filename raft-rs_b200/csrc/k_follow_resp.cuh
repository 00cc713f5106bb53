// k_follow_resp.cuh -- the term prefix of Raft::step (raft.rs:1280-1348) and the drop arms of step_follower and
// step_candidate (:2205-2255) for the responses that reach a Follower, PreCandidate or Candidate (DESIGN 3.23):
// MsgAppendResponse (4), MsgRequestVoteResponse (6), MsgHeartbeatResponse (9) and MsgRequestPreVoteResponse (18).  A
// higher term is become_follower(T, INVALID_ID)'s arena part, the frames of the group's own candidacy at its term are
// left for raftgpu_vote_wire, and every other frame is dropped.  None of them is answered.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).
//
// Role comes from the caller's raftgpu_voter table (RAFTGPU_VOTER_SELECT, _CANDIDATE, _PRE_CANDIDATE), leadership from
// the arena (term_start != RAFTGPU_NO_TERM_START).  Frames carry the receiver's cell: a wide pair's high half stands for
// the pair's low half.  Every frame gets its verdict in one call, from T = max(the group's term, every passing m.term
// that can raise it).
//
// Three kernels and no waiting between blocks: frp_scan_kernel stages and decodes every frame once, classifies it,
// writes a FtmRec per passing frame and atomicMax-es T into a per-group u64 table; ftm_claim_kernel (k_follow_term.cuh)
// lets the lowest frame at T > term claim its group; frp_apply_kernel bumps the claimed groups and settles every frame
// from T, its own m.term and its record's bits.  Every kernel takes kWireThreads frames per block.

// A passing frame's record: w0 = its header (the pair's low half << 4 | slot) | kFrpOwn when the frame belongs to the
// group's own candidacy (a MsgRequestVoteResponse at a Candidate, a MsgRequestPreVoteResponse at a PreCandidate);
// to = m.term; term = m.term, but 0 for a MsgRequestPreVoteResponse with reject = false, which never raises the term
// (raft.rs:1319-1320) and so must never claim.  `from` is not used.
constexpr uint64_t kFrpOwn = 1ull << 33;

// Frame i: its status (checks in the order of raftgpu.h) and, for a passing frame (RAFTGPU_WIRE_OK here), its record
// and T's candidate: the larger of m.term and the group's term, the group's term alone for a granting pre-vote.
__device__ __forceinline__ uint32_t frp_frame(const Columns &c, const WireSrc &w, const raftgpu_voter *__restrict__ voters,
                                              const WireStage &s, const uint8_t *stage, uint32_t i, FtmRec &r, uint64_t &top) {
    uint32_t hdr;
    const uint8_t *msg;
    WireMsg m;
    if (wire_open<false, true>(w, s, stage, i, hdr, msg, m) != RAFTGPU_WIRE_OK) return RAFTGPU_WIRE_MALFORMED;
    const uint32_t g = hdr >> 4, t = m.msg_type;
    if (t != 4u && t != 6u && t != 9u && t != 18u) return RAFTGPU_WIRE_SKIP_TYPE;  // eraftpb.proto:54-68
    const uint32_t lo = (c.meta[g] & RAFTGPU_META_WIDE_HI) ? g - 1 : g;
    const uint32_t flags = voters[lo].flags;
    if (!(flags & RAFTGPU_VOTER_SELECT) || c.term_start[lo] != RAFTGPU_NO_TERM_START) return RAFTGPU_WIRE_ROLE;
    const uint64_t term = c.term[lo];
    if (term == 0 || m.term == 0) return RAFTGPU_WIRE_TERM;  // m.term 0 is a local message
    const bool grant = t == 18u && !m.reject, pre = (flags & RAFTGPU_VOTER_PRE_CANDIDATE) != 0;
    const bool own = (flags & RAFTGPU_VOTER_CANDIDATE) && (t == 18u ? pre : t == 6u && !pre);  // step_candidate, :2230-2240
    r.w0 = (lo << 4 | (hdr & 15u)) | (own ? kFrpOwn : 0ull);
    r.to = m.term;
    r.term = grant ? 0ull : m.term;
    top = grant ? term : umax64(m.term, term);
    return RAFTGPU_WIRE_OK;
}

// Pass 1: classify every frame; status[i] = wire status << 4; a passing frame's record (w0, to, term) and
// top[group] = max(top, T's candidate).  top covers [0, hi) and is zero before the pass.  Launched with kWireThreads
// threads per block.
__global__ void __launch_bounds__(kWireThreads) frp_scan_kernel(Columns c, WireSrc w, const raftgpu_voter *__restrict__ voters,
                                                                uint8_t *__restrict__ status, FtmRec *__restrict__ recs,
                                                                unsigned long long *__restrict__ top) {
    __shared__ __align__(16) uint8_t stage[kWireStage + 16];
    WireStage s;
    const uint32_t i = wire_block_frame(w, stage, s);
    if (i == kNoFrame) return;
    FtmRec r;
    uint64_t t;
    const uint32_t st = frp_frame(c, w, voters, s, stage, i, r, t);
    status[i] = static_cast<uint8_t>(st << 4);
    if (st != RAFTGPU_WIRE_OK) return;
    recs[i].w0 = r.w0;
    recs[i].to = r.to;
    recs[i].term = r.term;
    const uint32_t g = static_cast<uint32_t>(r.w0) >> 4;
    if (top[g] < t) atomicMax(&top[g], static_cast<unsigned long long>(t));
}

// Pass 2 is ftm_claim_kernel (k_follow_term.cuh): the lowest passing frame with m.term == T > term claims its group.

// Pass 3: the verdict of every passing frame, from T = top[group], whether its group has a claimant, its m.term and
// its record's bits -- never from the group's term, which the claimant writes in this kernel.  The claimant runs
// become_follower(T, INVALID_ID)'s arena part (become_follower_arena) and keeps RAFTGPU_WIRE_OK | RAFTGPU_FTERM_BUMPED
// with out = T.  A frame below T is RAFTGPU_WIRE_STALE.  A frame of the group's own candidacy at T, in a group without
// a claimant (T is the term), stays RAFTGPU_WIRE_OK for raftgpu_vote_wire -- a granting pre-vote above T too; every other
// frame is RAFTGPU_WIRE_IGNORED.  out[i] (nullable) = 0 for every frame but a claimant.  Algorithmic bytes per frame:
// 1 read (+ 8 out); per passing frame 24 (record) + 8 (T) + 4 (first_frame) read and 1 written; per bump the reset of
// its group.
__global__ void __launch_bounds__(kWireThreads) frp_apply_kernel(Columns c, uint32_t n, const raftgpu_voter *__restrict__ voters,
                                                                 uint8_t *__restrict__ status, const FtmRec *__restrict__ recs,
                                                                 const unsigned long long *__restrict__ top,
                                                                 const uint32_t *__restrict__ first_frame,
                                                                 uint64_t *__restrict__ out) {
    const uint32_t i = blockIdx.x * kWireThreads + threadIdx.x;
    if (i >= n) return;
    uint64_t term = 0;
    if (status[i] == (RAFTGPU_WIRE_OK << 4)) {
        const FtmRec r = recs[i];
        const uint32_t g = static_cast<uint32_t>(r.w0) >> 4, first = first_frame[g];
        const uint64_t t = top[g];
        uint32_t st = RAFTGPU_WIRE_OK << 4;
        if (first == i) {
            become_follower_arena(c, g, t, voters);
            st |= RAFTGPU_FTERM_BUMPED;
            term = t;
        } else if (r.to < t) {
            st = RAFTGPU_WIRE_STALE << 4;
        } else if (first != kNoFrame || !(r.w0 & kFrpOwn)) {
            st = RAFTGPU_WIRE_IGNORED << 4;
        }
        status[i] = static_cast<uint8_t>(st);
    }
    if (out) out[i] = term;
}
