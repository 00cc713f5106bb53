// k_vote_wire.cuh -- MsgRequestVoteResponse / MsgRequestPreVoteResponse frames at a candidate (DESIGN 3.13): Raft::step's
// term rules and step_candidate's type check as statuses, then poll's record_vote (tracker.rs:308-310) for the first
// passing frame of every (group, peer) cell, and one tally_votes (tracker.rs:313-340) per group the batch touched.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).
//
// Role stays with the caller: one bitmap selects the groups whose Raft is a PreCandidate or a Candidate, a second one
// marks the PreCandidates among them.  The transitions poll would make (become_leader, become_follower, campaign) are
// the caller's too: the pass lists each touched group whose tally is decided, and the caller runs its control list.
// One tally per batch is exact because votes only accumulate (DESIGN 3.13).
//
// Five kernels and no waiting between blocks: vw_scan_kernel stages and decodes every frame once, classifies it and
// writes an 8-byte record per passing frame; vw_apply_kernel marks the later frames of a cell DUP, writes the first
// one's vote and marks its group (pair) touched; vw_count_kernel tallies every touched group and sums the decided ones
// per block; block_starts_kernel<1> (k_wire.cuh) turns the sums into block starts; vw_write_kernel lists the decided groups
// in ascending order.

constexpr uint32_t kVwThreads = 256;  // frames (scan, apply) or group slots (count, write) per block

// The caller's bitmaps, in the layout of d_adv_bitmap: select (required) and pre (nullable: no PreCandidates).
struct VwSrc {
    const uint32_t *select;
    const uint32_t *pre;
};

// A passing frame's record: its header, bit 32 = granted (!m.reject), bit 33 = the header names a wide pair's high half.
constexpr uint64_t kVwGranted = 1ull << 32, kVwHigh = 1ull << 33;

__device__ __forceinline__ bool vw_bit(const uint32_t *bm, uint32_t g) { return (bm[g >> 5] >> (g & 31u)) & 1u; }

// Frame i: its status before the duplicate rule (checks in the order of raftgpu.h) and, for RAFTGPU_WIRE_OK, its record.
__device__ __forceinline__ uint32_t vw_frame(const Columns &c, const WireSrc &w, const VwSrc &v, const WireStage &s,
                                             const uint8_t *stage, uint32_t i, uint64_t &rec) {
    uint32_t hdr;
    const uint8_t *msg;
    WireMsg m;
    if (wire_open<false, false, true>(w, s, stage, i, hdr, msg, m) != RAFTGPU_WIRE_OK) return RAFTGPU_WIRE_MALFORMED;
    if (m.msg_type != 6u && m.msg_type != 18u) return RAFTGPU_WIRE_SKIP_TYPE;  // eraftpb.proto:56, 68
    const uint32_t g = hdr >> 4, meta = c.meta[g];
    const bool high = (meta & RAFTGPU_META_WIDE_HI) != 0;
    const uint32_t lo = high ? g - 1 : g;  // a pair's role, term and committed are its low half's
    if (!vw_bit(v.select, lo) || c.term_start[lo] != RAFTGPU_NO_TERM_START) return RAFTGPU_WIRE_ROLE;
    // a pair without voters -- a freed slot (raftgpu_group_free leaves meta 0), or one not configured yet -- is the
    // host's: its tally would be Won (majority.rs:131-136), and only allocated groups may reach the outcome list
    const uint32_t meta_lo = high ? c.meta[lo] : meta;
    uint32_t voters = RAFTGPU_META_IN(meta_lo) | RAFTGPU_META_OUT(meta_lo);
    if (high || (meta_lo & RAFTGPU_META_WIDE_LO)) voters |= RAFTGPU_META_IN(c.meta[lo + 1]) | RAFTGPU_META_OUT(c.meta[lo + 1]);
    if (voters == 0) return RAFTGPU_WIRE_ROLE;
    const bool pre = v.pre && vw_bit(v.pre, lo);
    if (pre != (m.msg_type == 18u)) return RAFTGPU_WIRE_ROLE;  // step_candidate ignores the other type, raft.rs:2230-2240
    const uint64_t term = c.term[lo];
    if (term == 0 || m.term == 0) return RAFTGPU_WIRE_TERM;
    // raft.rs:1280-1349: a Candidate polls at its own term; a PreCandidate also takes a granted pre-vote from its future
    // term (:1319-1330) -- a higher-term rejection is become_follower, a lower term is ignored
    if (pre ? (m.term < term || (m.reject && m.term > term)) : m.term != term) return RAFTGPU_WIRE_TERM;
    uint64_t committed = c.committed[lo];
    if (c.meta[lo] & RAFTGPU_META_WIDE_LO) committed = umax64(committed, c.committed[lo + 1]);
    // maybe_commit_by_vote (raft.rs:2126-2164) would read raft_log.term(m.commit): the caller's log
    if (m.commit != 0 && m.commit_term != 0 && m.commit > committed) return RAFTGPU_WIRE_COMMIT_VOTE;
    rec = hdr | (m.reject ? 0ull : kVwGranted) | (high ? kVwHigh : 0ull);
    return RAFTGPU_WIRE_OK;
}

// Pass 1: classify every frame; status[i] = wire status << 4; a passing frame's record, first_frame[cell] = the lowest
// passing frame of the cell.  Launched with kVwThreads threads per block; __maxnreg__ as hb_wire_scan_kernel, because
// ptxas, left alone, settles on 32 registers and spills.
__global__ void __maxnreg__(40) vw_scan_kernel(Columns c, WireSrc w, VwSrc v, uint8_t *__restrict__ status,
                                               uint64_t *__restrict__ recs, uint32_t *__restrict__ first_frame) {
    static_assert(kVwThreads == kWireThreads, "wire_block_frame stages kWireThreads frames per block");
    __shared__ __align__(16) uint8_t stage[kWireStage + 16];
    WireStage s;
    const uint32_t i = wire_block_frame(w, stage, s);
    if (i == kNoFrame) return;
    uint64_t r = 0;
    const uint32_t st = vw_frame(c, w, v, s, stage, i, r);
    status[i] = static_cast<uint8_t>(st << 4);
    if (st == RAFTGPU_WIRE_OK) {
        recs[i] = r;
        const uint32_t g = static_cast<uint32_t>(r) >> 4, slot = static_cast<uint32_t>(r) & 15u;
        if (slot < kSlots) atomicMin(&first_frame[static_cast<size_t>(slot) * c.cap + g], i);
    }
}

// Pass 2: the first passing frame of every cell records its vote -- entry(id).or_insert(vote), tracker.rs:308-310, as
// RAFTGPU_CTL_RECORD_VOTE -- and a later one is RAFTGPU_WIRE_DUP.  A slot past the group's 8 (no such peer) records
// nothing: RAFTGPU_RES_NO_PROGRESS.  Every applied frame sets its group's (its pair's low half's) touched bit.
// Algorithmic bytes per frame: 1 read + 1 written; per passing frame 8 (record) + 4 (first_frame) read; per applied
// one 1 (votes) read, at most 1 written, and a touched word.
__global__ void __launch_bounds__(kVwThreads) vw_apply_kernel(Columns c, uint32_t n, uint8_t *__restrict__ status,
                                                              const uint64_t *__restrict__ recs,
                                                              const uint32_t *__restrict__ first_frame,
                                                              uint32_t *__restrict__ touched) {
    const uint32_t i = blockIdx.x * kVwThreads + threadIdx.x;
    if (i >= n || status[i] != (RAFTGPU_WIRE_OK << 4)) return;
    const uint64_t r = recs[i];
    const uint32_t g = static_cast<uint32_t>(r) >> 4, slot = static_cast<uint32_t>(r) & 15u;
    uint32_t res = RAFTGPU_RES_NO_PROGRESS;
    if (slot < kSlots) {
        const size_t cell = static_cast<size_t>(slot) * c.cap + g;
        if (first_frame[cell] != i) {
            status[i] = static_cast<uint8_t>(RAFTGPU_WIRE_DUP << 4);
            return;
        }
        res = 0;
        if (c.votes[cell] == 0) {  // (the only frame of this batch that touches the cell)
            c.votes[cell] = (r & kVwGranted) ? 2 : 1;
            res = RAFTGPU_RES_OK;
        }
    }
    status[i] = static_cast<uint8_t>((RAFTGPU_WIRE_OK << 4) | res);
    const uint32_t lo = (r & kVwHigh) ? g - 1 : g;
    atomicOr(&touched[lo >> 5], 1u << (lo & 31u));
}

// Pass 3, one thread per group slot of [0, n): a touched group's tally (tally_group, both halves of a pair) goes to
// words[g]; blk[block] = the block's touched groups whose tally is WON or LOST.  Each tally adds one to votes_tallied.
__global__ void __launch_bounds__(kVwThreads) vw_count_kernel(Columns c, uint32_t n, const uint32_t *__restrict__ touched,
                                                              uint32_t *__restrict__ words, uint32_t *__restrict__ blk,
                                                              unsigned long long *__restrict__ counters) {
    const uint32_t g = blockIdx.x * kVwThreads + threadIdx.x;
    uint32_t decided = 0, tallied = 0;
    if (g < n && vw_bit(touched, g)) {
        const uint32_t r = tally_group(c, g);
        words[g] = r;
        decided = (r & 0xffu) != RAFTGPU_VOTE_PENDING;
        tallied = 1;
    }
    block_sums<1, kVwThreads>({decided}, blk);
    const uint32_t local[1] = {tallied};
    const int which[1] = {kCntVotes};
    block_flush_counts<1>(local, which, counters, nullptr);
}

// Pass 5 (after block_starts_kernel<1> turned blk into block starts): every decided group's outcome, in ascending group order;
// an outcome at or past `capacity` is not written (the count, *d_count, stays the true one).
__global__ void __launch_bounds__(kVwThreads) vw_write_kernel(uint32_t n, const uint32_t *__restrict__ touched,
                                                              const uint32_t *__restrict__ words,
                                                              const uint32_t *__restrict__ blk,
                                                              raftgpu_vote_outcome *__restrict__ out, uint64_t capacity) {
    const uint32_t g = blockIdx.x * kVwThreads + threadIdx.x;
    uint32_t r = 0, pos = 0, zero = 0, tot, tot0;
    if (g < n && vw_bit(touched, g)) {
        r = words[g];
        pos = (r & 0xffu) != RAFTGPU_VOTE_PENDING;
    }
    const bool decided = pos;
    wire_block_scan<kVwThreads / 32>(pos, zero, tot, tot0);
    if (decided) {
        const uint32_t at = blk[blockIdx.x] + pos;
        if (at < capacity) out[at] = raftgpu_vote_outcome{g, r};
    }
}
