// k_follow_term.cuh -- the term prefix of Raft::step (raft.rs:1280-1376) for MsgAppend and MsgHeartbeat frames at a
// Follower, PreCandidate or Candidate (DESIGN 3.20): become_follower(T, m.from)'s arena part for a group whose frames
// name a higher term, and the empty MsgAppendResponse a lower-term frame gets when check_quorum or pre_vote is on
// (raft.rs:1349-1376).  The frames at the group's (new) term are left for raftgpu_follower_heartbeat and
// raftgpu_follower_append[_entries].
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).
//
// Role, vote and leader stay with the caller: its raftgpu_voter table (one row per group slot) is read only.  The
// frame's header is the follower's own (group << 4 | x); x is not read and goes back unchanged in the response's header.
// Every frame gets its verdict in one call: T = max(the group's term, the largest m.term among its passing frames) does
// not depend on the order in which they are applied, and the first one applied at T does the bump.  A row with
// RAFTGPU_VOTER_CANDIDATE opts in to step_candidate's step-down (raft.rs:2215-2224): when T is the group's term, the
// first frame at T makes the (Pre)Candidate a Follower, become_follower(term, m.from), whose arena part is the reset.
//
// Five kernels and no waiting between blocks: ftm_scan_kernel stages and decodes every frame once, classifies it,
// writes a 24-byte record per passing frame and atomicMax-es T into a per-group u64 table; ftm_claim_kernel lets the
// lowest passing frame at T > term claim its group; ftm_apply_kernel bumps the claimed groups, settles every frame
// from T and its own m.term, and sums the stale replies per block; block_starts_kernel<2> (k_wire.cuh) turns the sums
// into block starts; reply_write_kernel<FtmReply> (k_wire.cuh) encodes the replies (wire_put_app_resp_frame) and
// stores them through shared memory.  Every kernel takes kWireThreads frames per block: one block sum per scan block.

// A passing frame's record: w0 = its header | kFtmReply when the table's RAFTGPU_VOTER_STALE_REPLY is set | kFtmCand
// when its RAFTGPU_VOTER_CANDIDATE is; to = m.from; term = m.term (the apply pass overwrites it with T for a stale
// reply); from = the table's id (written by the apply pass for a stale reply only).  No other pass sets kFtmCand, so
// ftm_claim_kernel claims their groups at a raised term only.
constexpr uint64_t kFtmReply = 1ull << 32, kFtmCand = 1ull << 36;
struct __align__(16) FtmRec {
    uint64_t w0, to, term, from;
};

// bytes of a stale reply, header included: an empty MsgAppendResponse {to, from, term} (raft.rs:1375-1376)
__device__ __forceinline__ uint32_t ftm_len(const FtmRec &r) { return wire_app_resp_len(r.to, r.from, r.term, 0, 0, 0, false, 0); }
constexpr uint32_t kWireStaleFrameMax = 39;  // 4-byte header + msg_type (2) + to, from, term at 11 bytes each

// Frame i: its status before the per-group verdict (checks in the order of raftgpu.h) and, for a passing frame
// (RAFTGPU_WIRE_OK here), its record and T's candidate: the larger of m.term and the group's term.
__device__ __forceinline__ uint32_t ftm_frame(const Columns &c, const WireSrc &w, const raftgpu_voter *__restrict__ voters,
                                              const WireStage &s, const uint8_t *stage, uint32_t i, FtmRec &r, uint64_t &top) {
    uint32_t hdr;
    const uint8_t *msg;
    WireMsg m;
    if (wire_open<false, true>(w, s, stage, i, hdr, msg, m) != RAFTGPU_WIRE_OK) return RAFTGPU_WIRE_MALFORMED;
    const uint32_t g = hdr >> 4;
    if (c.meta[g] & RAFTGPU_META_WIDE_HI) return RAFTGPU_WIRE_MALFORMED;
    if (m.msg_type != 3u && m.msg_type != 8u) return RAFTGPU_WIRE_SKIP_TYPE;  // MsgAppend, MsgHeartbeat: eraftpb.proto:53, 58
    const uint32_t flags = voters[g].flags;
    // a leader's step-down has host-side consequences; the three other roles share step's term rules
    if (!(flags & RAFTGPU_VOTER_SELECT) || c.term_start[g] != RAFTGPU_NO_TERM_START) return RAFTGPU_WIRE_ROLE;
    const uint64_t term = c.term[g];
    if (term == 0 || m.term == 0) return RAFTGPU_WIRE_TERM;  // m.term 0 is a local message
    r.w0 = hdr | ((flags & RAFTGPU_VOTER_STALE_REPLY) ? kFtmReply : 0ull) | ((flags & RAFTGPU_VOTER_CANDIDATE) ? kFtmCand : 0ull);
    r.to = m.from;  // become_follower's leader_id, the stale reply's to (raft.rs:1347, 1375)
    r.term = m.term;
    top = umax64(m.term, term);
    return RAFTGPU_WIRE_OK;
}

// Pass 1: classify every frame; status[i] = wire status << 4; a passing frame's record (w0, to, term) and
// top[group] = max(top, m.term, term).  top covers [0, hi) and is zero before the pass.  Launched with kWireThreads
// threads per block.
__global__ void __launch_bounds__(kWireThreads) ftm_scan_kernel(Columns c, WireSrc w, const raftgpu_voter *__restrict__ voters,
                                                                uint8_t *__restrict__ status, FtmRec *__restrict__ recs,
                                                                unsigned long long *__restrict__ top) {
    __shared__ __align__(16) uint8_t stage[kWireStage + 16];
    WireStage s;
    const uint32_t i = wire_block_frame(w, stage, s);
    if (i == kNoFrame) return;
    FtmRec r;
    uint64_t t;
    const uint32_t st = ftm_frame(c, w, voters, s, stage, i, r, t);
    status[i] = static_cast<uint8_t>(st << 4);
    if (st != RAFTGPU_WIRE_OK) return;
    recs[i].w0 = r.w0;
    recs[i].to = r.to;
    recs[i].term = r.term;
    const uint32_t g = static_cast<uint32_t>(r.w0) >> 4;
    if (top[g] < t) atomicMax(&top[g], static_cast<unsigned long long>(t));
}

// Pass 2: a passing frame with m.term == T > term, or with m.term == T and kFtmCand, claims its group: first_frame[group]
// = the lowest such frame.  Algorithmic bytes per frame: 1 read; per passing frame 16 (w0, term) + 8 (T) read; per
// frame at T 8 (term) read and 4 (first_frame) written.
__global__ void __launch_bounds__(kWireThreads) ftm_claim_kernel(Columns c, uint32_t n, const uint8_t *__restrict__ status,
                                                                 const FtmRec *__restrict__ recs,
                                                                 const unsigned long long *__restrict__ top,
                                                                 uint32_t *__restrict__ first_frame) {
    const uint32_t i = blockIdx.x * kWireThreads + threadIdx.x;
    if (i >= n || status[i] != (RAFTGPU_WIRE_OK << 4)) return;
    const uint32_t g = static_cast<uint32_t>(recs[i].w0) >> 4;
    const uint64_t t = recs[i].term;
    if (t == top[g] && (t > c.term[g] || (recs[i].w0 & kFtmCand))) atomicMin(&first_frame[g], i);
}

// Pass 3: the verdict of every passing frame, from T = top[group] and its own m.term -- never from the group's term,
// which the claimant writes in this kernel (only the claimant reads it, before).  The claimant runs
// become_follower(T, m.from)'s arena part (become_follower_arena) and keeps RAFTGPU_WIRE_OK | RAFTGPU_FTERM_BUMPED, or
// RAFTGPU_FTERM_STEPPED when T is the term (the reset alone); any other frame at T stays RAFTGPU_WIRE_OK
// with nothing written; a frame below T is RAFTGPU_WIRE_STALE, | RAFTGPU_RES_OK with its reply's record completed
// (from = the table's id, term = T) when kFtmReply is set.  out[2 i..] (nullable) = {m.from, T} of the claimant, 0
// otherwise.  blk[2 * block + {0, 1}] = the block's replies and their bytes.  Algorithmic bytes per frame: 1 read + 1
// written (+ 16 out); per passing frame 24 (record) + 8 (T) + 4 (first_frame) read; per stale reply 8 (id) read and 16
// (record) written; per bump the reset of its group (become_follower_arena).
__global__ void __launch_bounds__(kWireThreads) ftm_apply_kernel(Columns c, uint32_t n, const raftgpu_voter *__restrict__ voters,
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
            if (first_frame[g] == i) {
                const uint32_t how = t > c.term[g] ? RAFTGPU_FTERM_BUMPED : RAFTGPU_FTERM_STEPPED;
                become_follower_arena(c, g, t, voters);
                status[i] = static_cast<uint8_t>((RAFTGPU_WIRE_OK << 4) | how);
                from = r.to;
                term = t;
            } else if (r.term < t) {
                if (r.w0 & kFtmReply) {
                    r.from = voters[g].id;  // send: from = self.id, term = self.term (raft.rs:610-650)
                    r.term = t;
                    recs[i].from = r.from;
                    recs[i].term = t;
                    status[i] = static_cast<uint8_t>((RAFTGPU_WIRE_STALE << 4) | RAFTGPU_RES_OK);
                    resp = 1;
                    bytes = ftm_len(r);
                } else {
                    status[i] = static_cast<uint8_t>(RAFTGPU_WIRE_STALE << 4);
                }
            }
        }
        if (out) {
            out[2ull * i] = from;
            out[2ull * i + 1] = term;
        }
    }
    block_sums<2, kWireThreads>({resp, bytes}, blk);
}

// Pass 5 is reply_write_kernel<FtmReply> (k_wire.cuh): the stale frames the apply pass marked RAFTGPU_RES_OK answer.
struct FtmReply {
    using Rec = FtmRec;
    static constexpr uint32_t kFrameMax = kWireStaleFrameMax;
    __device__ __forceinline__ static bool answers(uint8_t status) { return status == ((RAFTGPU_WIRE_STALE << 4) | RAFTGPU_RES_OK); }
    __device__ __forceinline__ static uint32_t len(const FtmRec &r) { return ftm_len(r); }
    __device__ __forceinline__ static uint8_t *put(uint8_t *p, const FtmRec &r) {  // MsgAppendResponse, raft.rs:1375-1376
        return wire_put_app_resp_frame(p, static_cast<uint32_t>(r.w0), r.to, r.from, r.term, 0, 0, 0, false, 0);
    }
};
