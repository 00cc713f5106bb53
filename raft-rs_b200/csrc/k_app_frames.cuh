// k_app_frames.cuh -- bcast_append to the wire (DESIGN 3.15): for a range of group slots, the commit broadcast's
// entry-less MsgAppend frames, in ascending (group, slot) order in the frame format of k_wire.cuh, and the sends that
// need the leader's log as a rest list of raftgpu_send_entry, in the same order.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).
//
// The structure of k_hb_frames.cuh, with a second output: apf_size_kernel counts every group's frames, bytes and rest
// entries and sums them per block, hbf_scan_kernel<3> (frames, bytes, leaders without a term) and hbf_scan_kernel<1>
// (rest entries) turn the block sums into block starts and totals, apf_write_kernel decides whether all three outputs
// fit, re-derives each group's sends, stores its rest entries in place and lays its frames out in shared memory for
// wire_store_block.  Nothing in the arena is written.

constexpr uint32_t kApfThreads = 128;                                           // group slots per block of the size and write kernels
constexpr uint32_t kApfBufBytes = kApfThreads * kSlots * kWireAppFrameMax + 16;  // + the block's misalignment
constexpr uint32_t kApfSmem = kApfBufBytes + kApfThreads * kSlots * 4;          // + the block's frame offsets

// What group slot first + i sends: `peers` = the slots bcast_append visits, and the fields its decisions read.
struct ApfGroup {
    uint32_t peers;
    bool no_term;  // a selected leader whose term is 0 (set on the low half only: counted once per group)
    uint64_t from, term, term_start, committed, last_index;
};

// bcast_append's choices for one slot (raft.rs:857-865): a leader (term_start set) that is allocated, selected and has
// a term visits every present peer but itself -- the selection of hbf_group.  A wide group's high half takes the low
// half's selection bit, term, term_start and `from`; committed and last_index are the pair's (max of both halves).
__device__ __forceinline__ ApfGroup apf_group(const Columns &c, const HbfSrc &s, uint32_t i) {
    ApfGroup r{};
    const uint32_t g = s.first + i;
    const uint32_t meta = c.meta[g];
    const bool hi_half = (meta & RAFTGPU_META_WIDE_HI) != 0;
    const uint32_t lo = hi_half ? g - 1 : g;  // (the host refuses a range that splits a pair: lo >= first)
    if (lo >= s.hi) return r;
    if (s.select && !((s.select[lo >> 5] >> (lo & 31u)) & 1u)) return r;
    if (c.rq_cap && !(c.rq_hc[lo] & kRqAlloc)) return r;
    r.term_start = c.term_start[lo];
    if (r.term_start == RAFTGPU_NO_TERM_START) return r;  // not a leader
    r.term = c.term[lo];
    if (r.term == 0) {
        r.no_term = !hi_half;
        return r;
    }
    uint32_t peers = RAFTGPU_META_IN(meta) | RAFTGPU_META_OUT(meta) | RAFTGPU_META_LEARN(meta);
    if (meta & RAFTGPU_META_HAS_SELF) peers &= ~(1u << RAFTGPU_META_SELF(meta));  // raft.rs:863 id != self_id
    r.peers = peers;
    if (!peers) return r;
    const bool wide = hi_half || (meta & RAFTGPU_META_WIDE_LO);
    r.committed = wide ? umax64(c.committed[lo], c.committed[lo + 1]) : c.committed[g];
    r.last_index = wide ? umax64(c.last_index[lo], c.last_index[lo + 1]) : c.last_index[g];
    r.from = s.ids[static_cast<size_t>(kSlots) * s.n + (lo - s.first)];
    return r;
}

// Progress::is_paused (progress.rs:210-216) of a flag byte: Probe -> paused, Replicate -> ins.full(), Snapshot ->
// always.  send_list_kernel states the same test inline: written through this helper it compiles to different SASS
// (56 fewer instructions, other registers), so the step path's kernel is left as it is.
__device__ __forceinline__ bool pf_paused(uint32_t f) {
    const uint32_t state = f & RAFTGPU_PF_STATE_MASK;
    return state == RAFTGPU_STATE_PROBE ? (f & RAFTGPU_PF_PAUSED) != 0
                                        : (state == RAFTGPU_STATE_REPLICATE ? (f & RAFTGPU_PF_INS_FULL) != 0 : true);
}

// maybe_send_append(to, allow_empty = true) for a present peer (raft.rs:764-819): nothing for a paused peer; the rest
// list when a snapshot is requested, when entries follow next_idx (raft_log.rs:382-387), or when the term of
// next_idx - 1 lies before the leader's term and so needs the log; a frame otherwise.  `next` = next_idx.
enum : uint32_t { kApfNone, kApfRest, kApfFrame };
__device__ __forceinline__ uint32_t apf_peer(const Columns &c, const ApfGroup &h, size_t cell, uint64_t &next, uint32_t &flags) {
    const uint32_t f = c.pflags[cell];
    const uint64_t matched = c.matched[cell], prs = c.pending_req_snapshot[cell];
    const int16_t nd = c.next_d[cell];
    if (pf_paused(f)) return kApfNone;
    next = off_decode(nd, matched, c.next_idx + cell);
    flags = prs != RAFTGPU_INVALID_INDEX ? RAFTGPU_SEND_SNAPSHOT : 0u;  // raft.rs:792-797, as send_list_kernel reports it
    return (flags || next <= h.last_index || next - 1 < h.term_start) ? kApfRest : kApfFrame;
}

// The frame of a peer that gets one (prepare_send_entries without entries, raft.rs:714-730, then send): index =
// next_idx - 1, log_term = the term when index <= last_index (DESIGN 1's range form of raft_log.term), 0 above it.
__device__ __forceinline__ uint64_t apf_log_term(const ApfGroup &h, uint64_t next) { return next - 1 <= h.last_index ? h.term : 0; }

// Pass 1: cnt[i] = {frames | rest entries << 16, bytes} of group slot first + i; blk[3 * block + {0, 1, 2}] = the
// block's frames, bytes and leaders without a term, blk_rest[block] = its rest entries.  Algorithmic bytes per slot:
// 4 (meta) + 8 (term_start) + 8 (term) read; per leader 16-32 (committed, last_index) + 8 (from) + per peer 1 (pflags)
// + 8 (matched) + 2 (the next_idx offset) + 8 (pending_request_snapshot) (+ 8 (its id) per frame); 8 written.
__global__ void __launch_bounds__(kApfThreads) apf_size_kernel(Columns c, HbfSrc s, uint2 *__restrict__ cnt,
                                                               uint32_t *__restrict__ blk, uint32_t *__restrict__ blk_rest) {
    const uint32_t i = blockIdx.x * kApfThreads + threadIdx.x;
    uint32_t frames = 0, bytes = 0, rest = 0, no_term = 0;
    if (i < s.n) {
        const ApfGroup h = apf_group(c, s, i);
        no_term = h.no_term;
        const uint32_t g = s.first + i;
#pragma unroll
        for (int k = 0; k < kSlots; k++) {
            if (!((h.peers >> k) & 1u)) continue;
            uint64_t next;
            uint32_t flags;
            const uint32_t d = apf_peer(c, h, static_cast<size_t>(k) * c.cap + g, next, flags);
            if (d == kApfRest) rest++;
            if (d != kApfFrame) continue;
            const uint64_t to = s.ids[static_cast<size_t>(k) * s.n + i];
            frames++;
            bytes += wire_app_len(to, h.from, h.term, apf_log_term(h, next), next - 1, h.committed);
        }
        cnt[i] = make_uint2(frames | (rest << 16), bytes);
    }
    block_sums<3, kApfThreads>({frames, bytes, no_term}, blk);
    block_sums<1, kApfThreads>({rest}, blk_rest);
}

// Where apf_write_kernel puts its three outputs, and their capacities.
struct ApfOut {
    uint8_t *bytes;
    uint32_t *offsets;
    raftgpu_send_entry *rest;
    uint64_t bytes_cap, frames_cap, rest_cap;
    uint64_t *totals;  // u64[4]: frames, bytes, rest entries, leaders without a term
};

// (Pass 2 is hbf_scan_kernel<3> on blk and hbf_scan_kernel<1> on blk_rest, k_wire.cuh: tot = {frames, bytes, leaders
// without a term, rest entries}.)
// Pass 3: block 0 writes the totals; when all three outputs fit (offsets given, each total within its capacity), it
// also writes offsets[frames] = bytes and every block writes its groups' rest entries -- [blk_rest start, + its
// entries) -- straight to `rest`, and its frames -- bytes [blk start, + its bytes), offsets [blk start, + its frames)
// -- through shared memory as hbf_write_kernel does.  Reads as pass 1 (+ 8 per slot of cnt); writes the frames and 16
// per rest entry.
__global__ void __launch_bounds__(kApfThreads) apf_write_kernel(Columns c, HbfSrc s, const uint2 *__restrict__ cnt,
                                                                const uint32_t *__restrict__ blk,
                                                                const uint32_t *__restrict__ blk_rest,
                                                                const uint64_t *__restrict__ tot, ApfOut o) {
    extern __shared__ __align__(16) uint8_t apf_smem[];
    const uint64_t frames = tot[0], bytes = tot[1], rest = tot[3];
    const bool fits = o.offsets && frames <= o.frames_cap && bytes <= o.bytes_cap && rest <= o.rest_cap;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        o.totals[0] = frames;
        o.totals[1] = bytes;
        o.totals[2] = rest;
        o.totals[3] = tot[2];
        if (fits) o.offsets[frames] = static_cast<uint32_t>(bytes);
    }
    if (!fits) return;
    uint8_t *buf = apf_smem;
    uint32_t *offs = reinterpret_cast<uint32_t *>(apf_smem + kApfBufBytes);
    const uint32_t i = blockIdx.x * kApfThreads + threadIdx.x;
    const uint2 fb = i < s.n ? cnt[i] : make_uint2(0u, 0u);
    // frames and rest entries scan as one u32: a block's sums of either stay below 2^16 (kApfThreads * kSlots)
    uint32_t lfr = fb.x, lb = fb.y, nfr, nbytes;
    wire_block_scan<kApfThreads / 32>(lfr, lb, nfr, nbytes);
    uint32_t lf = lfr & 0xffffu, lr = lfr >> 16;
    const uint32_t nf = nfr & 0xffffu;
    const uint32_t f0 = blk[3 * blockIdx.x], b0 = blk[3 * blockIdx.x + 1], r0 = blk_rest[blockIdx.x], pad = b0 & 15u;
    if (fb.x) {
        const ApfGroup h = apf_group(c, s, i);
        const uint32_t g = s.first + i;
        uint8_t *p = buf + pad + lb;
#pragma unroll 1
        for (uint32_t k = 0; k < kSlots; k++) {
            if (!((h.peers >> k) & 1u)) continue;
            uint64_t next;
            uint32_t flags;
            const uint32_t d = apf_peer(c, h, static_cast<size_t>(k) * c.cap + g, next, flags);
            if (d == kApfRest) {  // the send list's entry (send_list_kernel)
                uint64_t *e = reinterpret_cast<uint64_t *>(o.rest + r0 + lr++);
                e[0] = static_cast<uint64_t>(g) | (static_cast<uint64_t>(k) << 32) | (static_cast<uint64_t>(flags) << 40);
                e[1] = next;
            } else if (d == kApfFrame) {
                const uint64_t to = s.ids[static_cast<size_t>(k) * s.n + i];
                offs[lf++] = b0 + static_cast<uint32_t>(p - buf - pad);
                p = wire_put_append_frame(p, (g << 4) | k, to, h.from, h.term, apf_log_term(h, next), next - 1, h.committed);
            }
        }
    }
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < nf; j += kApfThreads) o.offsets[f0 + j] = offs[j];
    wire_store_block<kApfThreads>(o.bytes, buf, b0, nbytes);
}
