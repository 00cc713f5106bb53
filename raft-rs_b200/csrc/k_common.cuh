// k_common.cuh -- the arena columns, counters, the quorum selection (MajorityConfig / JointConfig::committed_index), block-level
// counter flush and sums, the warp-level reservation of output slots.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).

constexpr int kSlots = RAFTGPU_SLOTS;

// Device view of the arena: per-peer columns are [kSlots][cap], per-group [cap].
struct Columns {
    uint32_t cap;
    uint64_t *matched;
    // next_idx and peer_committed of a cell are stored as offsets from its matched (next_d, pc_d; off_* below); the
    // u64 columns hold the exact value of the cells whose offset is kOffEscape and are not read for any other cell
    int16_t *next_d;
    int16_t *pc_d;
    uint64_t *next_idx;
    uint64_t *peer_committed;
    uint64_t *pending_snapshot;
    uint64_t *pending_req_snapshot;
    uint64_t *commit_group_id;
    uint8_t *pflags;
    uint8_t *votes;
    uint32_t *meta;
    uint64_t *committed;
    uint64_t *term_start;
    uint64_t *last_index;
    uint64_t *term;  // Raft::term, 0 = unknown (wire path only)
    // Inflights on the device (raftgpu_arena_enable_inflights; SURVEY 8(f) rank 2): ins_cap = window size
    // (Config::max_inflight_msgs), 0 = off (INS_FULL is then the host's to report); ins_meta [kSlots][cap] =
    // start | count << 16 (inflights.rs:21-23); ins_buf [kSlots][cap][ins_cap] the rings
    uint32_t ins_cap;
    uint32_t *ins_meta;
    uint64_t *ins_buf;
    // ReadIndex queues (raftgpu_arena_enable_read_index, k_read.cuh): rq_cap = max_pending, 0 = off; rq_hc [cap] =
    // head | count << 8 | kRqAlloc; rq_ctx / rq_index / rq_acks [rq_cap][cap] the ring entries (read_only.rs:58-63)
    uint32_t rq_cap;
    uint32_t *rq_hc;
    uint64_t *rq_ctx;
    uint64_t *rq_index;
    uint16_t *rq_acks;
};

enum Counter : int {
    kCntRecomputes = 0,
    kCntAdvanced,
    kCntRecords,
    kCntUpdates,
    kCntRejects,
    kCntDecrements,
    kCntNoProgress,
    kCntVotes,
    kCntCount
};

// Fire-and-forget L2 prefetch: costs no destination register, so it deepens the memory pipeline
// beyond what registers x occupancy allow (the kernels here are long-scoreboard bound).
__device__ __forceinline__ void prefetch_l2(const void *p) {
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

__device__ __forceinline__ uint64_t umin64(uint64_t a, uint64_t b) { return a < b ? a : b; }
__device__ __forceinline__ uint64_t umax64(uint64_t a, uint64_t b) { return a > b ? a : b; }

// ---------------------------------------------------------------------------
// The offset codec of next_idx and peer_committed.  In a live group both sit within the inflight window of the same
// cell's matched, so each is stored as a signed 16-bit offset from it (next_d, pc_d): a fused step then moves 4 bytes
// per cell for the two instead of 16.  A value the offset cannot express -- more than 32 767 entries ahead of matched
// or behind it, or a peer right after Raft::reset, whose matched is 0 -- is stored as kOffEscape, with the
// exact value in the u64 column; such a cell takes the general path, correct but slower.  The format is lossless for
// every u64 value.  Offsets are relative to matched, so every write of matched re-encodes both offsets of its cell
// (hot_write); nothing outside this section does the arithmetic.
constexpr int16_t kOffEscape = INT16_MIN;

__device__ __forceinline__ bool off_escaped(int16_t d) { return d == kOffEscape; }
// the value of an offset that is not kOffEscape
__device__ __forceinline__ uint64_t off_value(int16_t d, uint64_t matched) {
    return matched + static_cast<uint64_t>(static_cast<int64_t>(d));
}
__device__ __forceinline__ uint64_t off_decode(int16_t d, uint64_t matched, const uint64_t *esc) {
    return off_escaped(d) ? *esc : off_value(d, matched);
}
// the offset to store for value v; a value that does not fit goes to *esc (a plain store, no read)
__device__ __forceinline__ int16_t off_encode(uint64_t v, uint64_t matched, uint64_t *esc) {
    const uint64_t d = v - matched;  // in the window (kOffEscape, INT16_MAX] iff d + INT16_MAX <= 2 * INT16_MAX, mod 2^64
    if (d + static_cast<uint64_t>(INT16_MAX) <= 2u * static_cast<uint64_t>(INT16_MAX)) return static_cast<int16_t>(d);
    *esc = v;
    return kOffEscape;
}

// Where one cell's matched and offsets live -- HBM, or a fused kernel's shared-memory rows -- and its index in the
// arena, which addresses its escape slots (always in HBM).
struct HotPtrs {
    uint64_t *matched;
    int16_t *next_d, *pc_d;
    size_t cell;
};
struct HotVals {
    uint64_t matched, next_idx, peer_committed;
};
__device__ __forceinline__ HotPtrs hot_ptrs(const Columns &c, size_t cell) {
    return HotPtrs{c.matched + cell, c.next_d + cell, c.pc_d + cell, cell};
}
__device__ __forceinline__ HotVals hot_load(const Columns &c, const HotPtrs &p) {
    HotVals h;
    h.matched = *p.matched;
    h.next_idx = off_decode(*p.next_d, h.matched, c.next_idx + p.cell);
    h.peer_committed = off_decode(*p.pc_d, h.matched, c.peer_committed + p.cell);
    return h;
}
// The cell's new values over its old ones: writes what changed, and both offsets when matched changed.
__device__ __forceinline__ void hot_write(const Columns &c, const HotPtrs &p, const HotVals &old, const HotVals &v) {
    const bool m_new = v.matched != old.matched;
    if (m_new) *p.matched = v.matched;
    if (m_new || v.next_idx != old.next_idx) *p.next_d = off_encode(v.next_idx, v.matched, c.next_idx + p.cell);
    if (m_new || v.peer_committed != old.peer_committed)
        *p.pc_d = off_encode(v.peer_committed, v.matched, c.peer_committed + p.cell);
}
// The same from the cell's stored form (matched and the two offsets as loaded): writes what differs.
__device__ __forceinline__ void hot_write_over(const Columns &c, const HotPtrs &p, uint64_t old_matched, int16_t old_next_d,
                                               int16_t old_pc_d, const HotVals &v) {
    if (v.matched != old_matched) *p.matched = v.matched;
    const int16_t nd = off_encode(v.next_idx, v.matched, c.next_idx + p.cell);
    if (nd != old_next_d) *p.next_d = nd;
    const int16_t pd = off_encode(v.peer_committed, v.matched, c.peer_committed + p.cell);
    if (pd != old_pc_d) *p.pc_d = pd;
}
__device__ __forceinline__ void hot_store(const Columns &c, const HotPtrs &p, const HotVals &v) {
    *p.matched = v.matched;
    *p.next_d = off_encode(v.next_idx, v.matched, c.next_idx + p.cell);
    *p.pc_d = off_encode(v.peer_committed, v.matched, c.peer_committed + p.cell);
}
__device__ __forceinline__ void hot_set_next(const Columns &c, const HotPtrs &p, uint64_t next_idx) {
    *p.next_d = off_encode(next_idx, *p.matched, c.next_idx + p.cell);
}
// Progress::update_committed (progress.rs:153-157)
__device__ __forceinline__ void hot_update_committed(const Columns &c, const HotPtrs &p, uint64_t committed) {
    const uint64_t m = *p.matched;
    if (committed > off_decode(*p.pc_d, m, c.peer_committed + p.cell))
        *p.pc_d = off_encode(committed, m, c.peer_committed + p.cell);
}
// Column IO of an offset column (raftgpu_column_read / _write): materialize the decoded values of cells [first,
// first + n) in their u64 column, or encode the values the host has put there.
__global__ void offset_column_kernel(const uint64_t *__restrict__ matched, int16_t *__restrict__ d,
                                     uint64_t *__restrict__ esc, size_t first, uint32_t n, bool encode) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        const size_t cell = first + i;
        if (encode)
            d[cell] = off_encode(esc[cell], matched[cell], &esc[cell]);
        else
            esc[cell] = off_decode(d[cell], matched[cell], &esc[cell]);
    }
}

// ---------------------------------------------------------------------------
// Inflights (src/tracker/inflights.rs) of one cell, when the arena keeps the windows on the device.  The flag bit
// RAFTGPU_PF_INS_FULL mirrors ins.full() (what Progress::is_paused reads, progress.rs:213): every function
// takes the caller's copy of the flag byte and keeps the bit right.
__device__ __forceinline__ void ins_reset(const Columns &c, size_t cell) {  // :119-123
    if (c.ins_cap) c.ins_meta[cell] = 0;
}
// :85-110 free_to
__device__ __noinline__ void ins_free_to(const Columns &c, size_t cell, uint64_t to, uint32_t &flags) {
    const uint32_t m = c.ins_meta[cell];
    uint32_t start = m & 0xffffu, count = m >> 16;
    const uint64_t *ring = c.ins_buf + cell * c.ins_cap;
    if (count == 0 || to < ring[start]) return;  // out of the left side of the window
    uint32_t i = 0, idx = start;
    while (i < count) {
        if (to < ring[idx]) break;  // found the first large inflight
        idx += 1;
        if (idx >= c.ins_cap) idx -= c.ins_cap;
        i += 1;
    }
    c.ins_meta[cell] = idx | ((count - i) << 16);
    if (i) flags &= ~RAFTGPU_PF_INS_FULL;
}
// :113-116 free_first_one
__device__ __forceinline__ void ins_free_first_one(const Columns &c, size_t cell, uint32_t &flags) {
    const uint32_t m = c.ins_meta[cell];
    if ((m >> 16) == 0) return;
    ins_free_to(c, cell, c.ins_buf[cell * c.ins_cap + (m & 0xffffu)], flags);
}
// :65-82 add; false where the reference panics (the window is full)
__device__ __forceinline__ bool ins_add(const Columns &c, size_t cell, uint64_t inflight, uint32_t &flags) {
    const uint32_t m = c.ins_meta[cell];
    const uint32_t start = m & 0xffffu, count = m >> 16;
    if (count == c.ins_cap) return false;
    uint32_t next = start + count;
    if (next >= c.ins_cap) next -= c.ins_cap;
    c.ins_buf[cell * c.ins_cap + next] = inflight;
    c.ins_meta[cell] = start | ((count + 1) << 16);
    if (count + 1 == c.ins_cap) flags |= RAFTGPU_PF_INS_FULL;
    return true;
}

// ---------------------------------------------------------------------------
// ReadIndex queues (src/read_only.rs), when the arena keeps them (Columns::rq_cap != 0).  A group's queue is a ring
// of rq_cap entries; its word rq_hc holds the front's position, the entry count and kRqAlloc (the group slot is
// allocated: group alloc / free set and clear it).  The kernels are in k_read.cuh; the control-plane hooks below.
constexpr uint32_t kRqAlloc = 0x80000000u;
__device__ __forceinline__ uint32_t rq_count(uint32_t hc) { return (hc >> 8) & 0xffu; }
// the cell of queue entry k (0 = the front) of group g
__device__ __forceinline__ size_t rq_at(const Columns &c, uint32_t g, uint32_t hc, uint32_t k) {
    uint32_t p = (hc & 0xffu) + k;
    if (p >= c.rq_cap) p -= c.rq_cap;
    return static_cast<size_t>(p) * c.cap + g;
}
// Raft::reset replaces the ReadOnly (raft.rs:957): the queue is emptied
__device__ __forceinline__ void rq_reset(const Columns &c, uint32_t g) {
    if (c.rq_cap) c.rq_hc[g] &= kRqAlloc;
}
// apply_conf removed the peers `removed` of half g (new meta `meta`): their bits leave every pending read's acks, so
// that a slot reused for a new peer does not inherit an old ack (DESIGN 3.9)
__device__ __forceinline__ void rq_conf_removed(const Columns &c, uint32_t g, uint32_t meta, uint32_t removed) {
    if (!c.rq_cap || !removed) return;
    const bool hi = (meta & RAFTGPU_META_WIDE_HI) != 0;
    const uint32_t qg = hi ? g - 1 : g, keep = ~(removed << (hi ? 8 : 0));
    const uint32_t hc = c.rq_hc[qg];
    for (uint32_t k = 0; k < rq_count(hc); k++) {
        uint16_t *p = &c.rq_acks[rq_at(c, qg, hc, k)];
        *p = static_cast<uint16_t>(*p & keep);
    }
}

// ---------------------------------------------------------------------------
// MajorityConfig::committed_index without group commit (majority.rs:70-101):
// the q-th largest acked index of the voters in `mask`, q = n/2 + 1
// (util.rs:118-120); the empty config yields u64::MAX (majority.rs:71-75).

// General form (any masks, joint configurations): quorum_index_joint in quorum_select.h -- the 8 slots are ordered
// once as predecessor bit masks (28 compares) and the q-th largest member of each half is the member with q - 1
// predecessors inside its mask.  (Until round 2 each half sorted the zero-padded slots with a 19-comparator network.)

// The common 5-voter case (q = 3): the median, by the classic 10 min/max form
// med5(a..e) = med3(e, max(min(a,b),min(c,d)), min(max(a,b),max(c,d))).
__device__ __forceinline__ uint64_t median5(uint64_t a, uint64_t b, uint64_t c, uint64_t d,
                                            uint64_t e) {
    const uint64_t lo = umax64(umin64(a, b), umin64(c, d));
    const uint64_t hi = umin64(umax64(a, b), umax64(c, d));
    return umax64(umin64(lo, hi), umin64(umax64(lo, hi), e));
}

// MajorityConfig::committed_index WITH group commit (majority.rs:70-124), the
// literal algorithm: gather, stable descending sort, then the scan of :102-123.
// Rare path (ProgressTracker::group_commit is off by default), kept out of line
// so its local arrays do not cost the common path registers.
__device__ __noinline__ void majority_group_commit(const uint64_t *v, const uint64_t *gid,
                                                   uint32_t mask, uint64_t *out_index,
                                                   bool *out_use_gc) {
    if (mask == 0) {  // :71-75
        *out_index = UINT64_MAX;
        *out_use_gc = true;
        return;
    }
    uint64_t idx[kSlots], grp[kSlots];
    int n = 0;
    for (int s = 0; s < kSlots; s++) {
        if ((mask >> s) & 1u) {  // :77-85 (voters without progress do not occur in a tracker)
            idx[n] = v[s];
            grp[n] = gid[s];
            n++;
        }
    }
    for (int i = 1; i < n; i++) {  // :95 stable sort, descending by index
        uint64_t xi = idx[i], xg = grp[i];
        int j = i;
        while (j > 0 && idx[j - 1] < xi) {
            idx[j] = idx[j - 1];
            grp[j] = grp[j - 1];
            j--;
        }
        idx[j] = xi;
        grp[j] = xg;
    }
    const int quorum = n / 2 + 1;  // :97
    const uint64_t quorum_commit_index = idx[quorum - 1];
    uint64_t checked_group_id = grp[quorum - 1];
    bool single_group = true;
    for (int i = 0; i < n; i++) {  // :105-118
        if (grp[i] == 0) {
            single_group = false;
            continue;
        }
        if (checked_group_id == 0) {
            checked_group_id = grp[i];
            continue;
        }
        if (checked_group_id == grp[i]) continue;
        *out_index = umin64(idx[i], quorum_commit_index);
        *out_use_gc = true;
        return;
    }
    *out_index = single_group ? quorum_commit_index : idx[n - 1];  // :119-123
    *out_use_gc = false;
}

// ProgressTracker::maximal_committed_index (tracker.rs:294-298) of group g:
// JointConfig::committed_index (joint.rs:47-51) over both majority halves, reading
// matched / commit_group_id through the ProgressMap AckedIndexer (tracker.rs:183-190).
__device__ __forceinline__ void group_mci(const Columns &c, uint32_t g, uint32_t meta, uint64_t &mci,
                                          bool &use_gc) {
    const uint32_t in = RAFTGPU_META_IN(meta), out = RAFTGPU_META_OUT(meta);
    const uint32_t voters = in | out;
    uint64_t v[kSlots];
#pragma unroll
    for (int s = 0; s < kSlots; s++)
        v[s] = ((voters >> s) & 1u) ? c.matched[static_cast<size_t>(s) * c.cap + g] : 0ull;
    if (!(meta & RAFTGPU_META_GROUP_COMMIT)) {
        uint64_t i_idx, o_idx;
        quorum_index_joint(v, in, out, i_idx, o_idx);  // quorum_select.h; empty outgoing => u64::MAX
        mci = umin64(i_idx, o_idx);                    // joint.rs:50
        // a non-empty half reports false (majority.rs:99-101), an empty one true (:71-75)
        use_gc = (in == 0) && (out == 0);
    } else {
        uint64_t gid[kSlots];
        for (int s = 0; s < kSlots; s++)
            gid[s] = ((voters >> s) & 1u) ? c.commit_group_id[static_cast<size_t>(s) * c.cap + g] : 0ull;
        uint64_t i_idx, o_idx;
        bool i_gc, o_gc;
        majority_group_commit(v, gid, in, &i_idx, &i_gc);
        majority_group_commit(v, gid, out, &o_idx, &o_gc);
        mci = umin64(i_idx, o_idx);
        use_gc = i_gc && o_gc;  // joint.rs:50
    }
}

// ---------------------------------------------------------------------------
// WIDE groups (RAFTGPU_META_WIDE_LO / _HI): up to 16 peers over two consecutive group slots.  Rare (a joint change of
// a large configuration with learners), so the code is the literal algorithm on 16 values, out of line.

// MajorityConfig::committed_index over up to 16 voters: gather, stable descending insertion sort (majority.rs:95), the
// quorum element, then -- with group commit -- the scan of majority.rs:102-123.
__device__ __noinline__ void majority_committed_index16(const uint64_t *v, const uint64_t *gid, uint32_t mask, bool group_commit,
                                                        uint64_t *out_index, bool *out_use_gc) {
    if (mask == 0) {  // majority.rs:71-75
        *out_index = UINT64_MAX;
        *out_use_gc = true;
        return;
    }
    uint64_t idx[16], grp[16];
    int n = 0;
    for (int s = 0; s < 16; s++)
        if ((mask >> s) & 1u) {
            idx[n] = v[s];
            grp[n] = gid ? gid[s] : 0;
            n++;
        }
    for (int i = 1; i < n; i++) {
        const uint64_t xi = idx[i], xg = grp[i];
        int j = i;
        while (j > 0 && idx[j - 1] < xi) {
            idx[j] = idx[j - 1];
            grp[j] = grp[j - 1];
            j--;
        }
        idx[j] = xi;
        grp[j] = xg;
    }
    const int quorum = n / 2 + 1;  // util.rs:118-120
    const uint64_t quorum_commit_index = idx[quorum - 1];
    if (!group_commit) {  // majority.rs:99-101
        *out_index = quorum_commit_index;
        *out_use_gc = false;
        return;
    }
    uint64_t checked_group_id = grp[quorum - 1];
    bool single_group = true;
    for (int i = 0; i < n; i++) {  // :105-118
        if (grp[i] == 0) {
            single_group = false;
            continue;
        }
        if (checked_group_id == 0) {
            checked_group_id = grp[i];
            continue;
        }
        if (checked_group_id == grp[i]) continue;
        *out_index = umin64(idx[i], quorum_commit_index);
        *out_use_gc = true;
        return;
    }
    *out_index = single_group ? quorum_commit_index : idx[n - 1];  // :119-123
    *out_use_gc = false;
}

// maximal_committed_index of the wide group whose low half is g (tracker.rs:294-298, joint.rs:47-51)
__device__ __noinline__ void wide_mci(const Columns &c, uint32_t g, uint32_t meta_lo, uint64_t &mci, bool &use_gc) {
    const uint32_t meta_hi = c.meta[g + 1];
    const uint32_t in = RAFTGPU_META_IN(meta_lo) | (RAFTGPU_META_IN(meta_hi) << 8);
    const uint32_t out = RAFTGPU_META_OUT(meta_lo) | (RAFTGPU_META_OUT(meta_hi) << 8);
    const uint32_t voters = in | out;
    const bool gc = (meta_lo & RAFTGPU_META_GROUP_COMMIT) != 0;
    uint64_t v[16], gid[16];
    for (int s = 0; s < 16; s++) {
        const size_t cell = static_cast<size_t>(s & 7) * c.cap + g + (s >> 3);
        const bool member = (voters >> s) & 1u;
        v[s] = member ? c.matched[cell] : 0ull;
        gid[s] = (member && gc) ? c.commit_group_id[cell] : 0ull;
    }
    uint64_t i_idx, o_idx;
    bool i_gc, o_gc;
    majority_committed_index16(v, gid, in, gc, &i_idx, &i_gc);
    majority_committed_index16(v, gid, out, gc, &o_idx, &o_gc);
    mci = umin64(i_idx, o_idx);  // joint.rs:50
    use_gc = i_gc && o_gc;
}

// Side-effect-free single-group query (thread 0 of one warp).
__global__ void mci_kernel(Columns c, uint32_t g, uint64_t *out_mci, uint8_t *out_gc) {
    if (threadIdx.x != 0) return;
    uint64_t mci;
    bool use_gc;
    const uint32_t meta = c.meta[g];
    if (meta & RAFTGPU_META_WIDE_LO)
        wide_mci(c, g, meta, mci, use_gc);
    else
        group_mci(c, g, meta, mci, use_gc);
    *out_mci = mci;
    *out_gc = use_gc ? 1 : 0;
}

// Block-level counter flush: per-thread tallies -> warp shuffle reduce -> shared
// -> ONE global atomic per counter per block.  (v1 issued one atomic per warp per
// counter; ~10^5 same-address atomics serialise in L2 and dominated both kernels.)
template <int kN>
__device__ __forceinline__ void block_flush_counts(const uint32_t (&local)[kN], const int (&which)[kN],
                                                   unsigned long long *counters,
                                                   uint32_t *extra_u32 /* nullable, gets local[1] */) {
    __shared__ uint32_t s_cnt[kN];
    if (threadIdx.x < kN) s_cnt[threadIdx.x] = 0;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kN; k++) {
        const uint32_t w = __reduce_add_sync(0xffffffffu, local[k]);
        if ((threadIdx.x & 31) == 0 && w) atomicAdd(&s_cnt[k], w);
    }
    __syncthreads();
    if (threadIdx.x < kN && s_cnt[threadIdx.x]) {
        atomicAdd(&counters[which[threadIdx.x]], static_cast<unsigned long long>(s_cnt[threadIdx.x]));
        if (extra_u32 && threadIdx.x == 1) atomicAdd(extra_u32, s_cnt[1]);
    }
}

// Per-thread u32 values -> the block's K sums at out[K * blockIdx.x + k]: a warp reduce, one shared word per warp and
// value, then thread k adds the warps' words of value k.  Every thread of the block (kThreads of them) calls it.
template <uint32_t K, uint32_t kThreads>
__device__ __forceinline__ void block_sums(const uint32_t (&v)[K], uint32_t *__restrict__ out) {
    __shared__ uint32_t sum[K][kThreads / 32];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    uint32_t r[K];
#pragma unroll
    for (uint32_t k = 0; k < K; k++) r[k] = __reduce_add_sync(0xffffffffu, v[k]);
    if (lane == 0) {
#pragma unroll
        for (uint32_t k = 0; k < K; k++) sum[k][warp] = r[k];
    }
    __syncthreads();
    if (threadIdx.x < K) {
        uint32_t t = 0;
#pragma unroll
        for (uint32_t w = 0; w < kThreads / 32; w++) t += sum[threadIdx.x][w];
        out[K * blockIdx.x + threadIdx.x] = t;
    }
}

// Every lane of a full warp asks for `want` consecutive slots of *count: a warp scan, ONE atomic per warp (a million
// same-address atomics, one per group, would serialise in L2), and each lane gets the first of its slots.
template <typename T>
__device__ __forceinline__ T warp_reserve(T *count, uint32_t want) {
    const uint32_t lane = threadIdx.x & 31;
    uint32_t incl = want;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= static_cast<uint32_t>(d)) incl += v;
    }
    const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
    T base = 0;
    if (lane == 31 && total) base = atomicAdd(count, static_cast<T>(total));
    return __shfl_sync(0xffffffffu, base, 31) + static_cast<T>(incl - want);
}
