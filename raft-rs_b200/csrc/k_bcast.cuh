// k_bcast.cuh -- the leader's broadcast pipeline (DESIGN 3.11): for a range of group slots, the frames a broadcast
// sends, in ascending (group, slot) order in the frame format of k_wire.cuh, and for a pass that has one, the sends that
// need the host as a rest list of raftgpu_send_entry in the same order.  Nothing in the arena is written.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).
//
// Three kernels and no waiting between blocks (a decoupled look-back would spin across blocks): bcast_size_kernel<P>
// counts every group's frames, bytes and rest entries and sums them per block, block_starts_kernel (k_wire.cuh, one
// block) turns the block sums into block starts and totals, bcast_write_kernel<P> decides whether every output fits,
// re-derives each group's sends, stores its rest entries in place and lays its frames out in shared memory for
// wire_store_block.  P is the pass's broadcast policy, a struct of compile-time facts:
//   kFrameMax  bytes of its largest frame
//   kRest      whether it has a rest list
//   Group      what a group sends: BcastLeader and the pass's own fields, read by group(c, s, i) with bcast_leader
//   Send       what one peer's decision found, filled by peer(c, h, cell, d): kBcastNone, kBcastRest or kBcastFrame
//   len(h, d, to) / put(p, hdr, h, d, to)   the peer's frame: its bytes and its encoder
// The kernels branch on P::kRest at compile time only, where the rest list is: its block sums, its entry store and the
// totals; HbBcast (k_hb_frames.cuh) has none, AppBcast (k_app_frames.cuh) has one.

constexpr uint32_t kBcastThreads = 128;  // group slots per block of the size and write kernels
// dynamic shared memory of bcast_write_kernel<P>: the block's frames (+ its misalignment), then its frame offsets
template <class P>
constexpr uint32_t kBcastBufBytes = kBcastThreads * kSlots * P::kFrameMax + 16;
template <class P>
constexpr uint32_t kBcastSmem = kBcastBufBytes<P> + kBcastThreads * kSlots * 4;

// The range and the caller's tables: select = bitmap from group 0 (nullptr = all), ids = u64 [kSlots + 1][n].
struct BcastSrc {
    uint32_t first, n, hi;
    const uint32_t *select;
    const uint64_t *ids;
};

// Who sends for group slot first + i: `peers` = the slots the broadcast visits, and the fields every pass reads.
struct BcastLeader {
    uint32_t lo, peers;
    bool wide;     // a pair: committed (and a pass's own pair fields) are the max of both halves
    bool no_term;  // a selected leader whose term is 0 (set on the low half only: counted once per group)
    uint64_t from, term, term_start, committed;
};

// bcast_heartbeat's and bcast_append's choice of senders (raft.rs:857-889): a leader (term_start set) that is allocated,
// selected and has a term visits every present peer but itself.  A wide group's high half takes the low half (`lo`):
// its selection bit, term, term_start and `from`; committed is the pair's (max of both halves).  r starts zeroed.
// Returns whether the group sends, for the pass's group() to read its own fields in the same branch: behind a second
// test of r.peers, those loads wait one more round trip to memory in every block of the write kernel.
__device__ __forceinline__ bool bcast_leader(const Columns &c, const BcastSrc &s, uint32_t i, BcastLeader &r) {
    const uint32_t g = s.first + i;
    const uint32_t meta = c.meta[g];
    const bool hi_half = (meta & RAFTGPU_META_WIDE_HI) != 0;
    r.lo = hi_half ? g - 1 : g;  // (the host refuses a range that splits a pair: lo >= first)
    if (r.lo >= s.hi) return false;
    if (s.select && !((s.select[r.lo >> 5] >> (r.lo & 31u)) & 1u)) return false;
    if (c.rq_cap && !(c.rq_hc[r.lo] & kRqAlloc)) return false;
    r.term_start = c.term_start[r.lo];
    if (r.term_start == RAFTGPU_NO_TERM_START) return false;  // not a leader: ping and bcast_append do nothing
    r.term = c.term[r.lo];
    if (r.term == 0) {
        r.no_term = !hi_half;
        return false;
    }
    uint32_t peers = RAFTGPU_META_IN(meta) | RAFTGPU_META_OUT(meta) | RAFTGPU_META_LEARN(meta);
    if (meta & RAFTGPU_META_HAS_SELF) peers &= ~(1u << RAFTGPU_META_SELF(meta));  // raft.rs:863, 887 id != self_id
    r.peers = peers;
    if (!peers) return false;
    r.wide = hi_half || (meta & RAFTGPU_META_WIDE_LO);
    r.committed = r.wide ? umax64(c.committed[r.lo], c.committed[r.lo + 1]) : c.committed[g];
    r.from = s.ids[static_cast<size_t>(kSlots) * s.n + (r.lo - s.first)];
    return true;
}

enum : uint32_t { kBcastNone, kBcastRest, kBcastFrame };  // what P::peer decides for one peer

// Pass 1: cnt[i] = {frames | rest entries << 16, bytes} of group slot first + i; blk[3 * block + {0, 1, 2}] = the
// block's frames, bytes and leaders without a term, blk_rest[block] = its rest entries (P::kRest).  Algorithmic bytes
// per slot: 4 (meta) + 8 (term_start) + 8 (term) read; per leader 8-16 (committed) + 8 (from) + the pass's; 8 written.
template <class P>
__global__ void __launch_bounds__(kBcastThreads) bcast_size_kernel(Columns c, BcastSrc s, uint2 *__restrict__ cnt,
                                                                   uint32_t *__restrict__ blk, uint32_t *__restrict__ blk_rest) {
    const uint32_t i = blockIdx.x * kBcastThreads + threadIdx.x;
    uint32_t frames = 0, bytes = 0, rest = 0, no_term = 0;
    if (i < s.n) {
        const typename P::Group h = P::group(c, s, i);
        no_term = h.no_term;
        const uint32_t g = s.first + i;
#pragma unroll
        for (int k = 0; k < kSlots; k++) {
            if (!((h.peers >> k) & 1u)) continue;
            typename P::Send d;
            const uint32_t kind = P::peer(c, h, static_cast<size_t>(k) * c.cap + g, d);
            if (kind == kBcastRest) rest++;
            if (kind != kBcastFrame) continue;
            const uint64_t to = s.ids[static_cast<size_t>(k) * s.n + i];
            frames++;
            bytes += P::len(h, d, to);
        }
        cnt[i] = make_uint2(frames | (rest << 16), bytes);
    }
    block_sums<3, kBcastThreads>({frames, bytes, no_term}, blk);
    if constexpr (P::kRest) block_sums<1, kBcastThreads>({rest}, blk_rest);
}

// Where bcast_write_kernel puts its outputs, and their capacities (rest: P::kRest only).
struct BcastOut {
    uint8_t *bytes;
    uint32_t *offsets;
    raftgpu_send_entry *rest;
    uint64_t bytes_cap, frames_cap, rest_cap;
    uint64_t *totals;  // kBcastTotals<P>
};
// totals: {frames, bytes, leaders without a term}; with a rest list {frames, bytes, rest entries, leaders without a term}
template <class P>
constexpr uint32_t kBcastTotals = P::kRest ? 4 : 3;

// (Pass 2 is block_starts_kernel<3> on blk and, with a rest list, block_starts_kernel<1> on blk_rest, k_wire.cuh: tot =
// {frames, bytes, leaders without a term[, rest entries]}.)
// Pass 3: block 0 writes the totals; when every output fits (offsets given, each total within its capacity), it also
// writes offsets[frames] = bytes and every block writes its groups' rest entries -- [blk_rest start, + its entries) --
// straight to `rest`, and its frames -- bytes [blk start, + its bytes), offsets [blk start, + its frames) -- through
// shared memory: the frames are assembled there at their offset from the 16-byte boundary below the block's start, so
// whole 16-byte chunks go out as uint4 stores and only the two chunks shared with the neighbouring blocks byte by
// byte.  Reads as pass 1 (+ 8 per slot of cnt); writes the frames, 4 per frame and 16 per rest entry.
template <class P>
__global__ void __launch_bounds__(kBcastThreads) bcast_write_kernel(Columns c, BcastSrc s, const uint2 *__restrict__ cnt,
                                                                    const uint32_t *__restrict__ blk,
                                                                    const uint32_t *__restrict__ blk_rest,
                                                                    const uint64_t *__restrict__ tot, BcastOut o) {
    extern __shared__ __align__(16) uint8_t bcast_smem[];
    const uint64_t frames = tot[0], bytes = tot[1];
    bool fits = o.offsets && frames <= o.frames_cap && bytes <= o.bytes_cap;
    if constexpr (P::kRest) {
        const uint64_t rest = tot[3];  // (loaded before the test: behind it, every block would wait one more round trip)
        fits = fits && rest <= o.rest_cap;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        o.totals[0] = frames;
        o.totals[1] = bytes;
        if constexpr (P::kRest) {
            o.totals[2] = tot[3];
            o.totals[3] = tot[2];
        } else {
            o.totals[2] = tot[2];
        }
        if (fits) o.offsets[frames] = static_cast<uint32_t>(bytes);
    }
    if (!fits) return;
    uint8_t *buf = bcast_smem;
    uint32_t *offs = reinterpret_cast<uint32_t *>(bcast_smem + kBcastBufBytes<P>);
    const uint32_t i = blockIdx.x * kBcastThreads + threadIdx.x;
    const uint2 fb = i < s.n ? cnt[i] : make_uint2(0u, 0u);
    // frames and rest entries scan as one u32: a block's sums of either stay below 2^16 (kBcastThreads * kSlots)
    uint32_t lfr = fb.x, lb = fb.y, nfr, nbytes;
    wire_block_scan<kBcastThreads / 32>(lfr, lb, nfr, nbytes);
    uint32_t lf = lfr & 0xffffu, lr = lfr >> 16;
    const uint32_t nf = nfr & 0xffffu;
    const uint32_t f0 = blk[3 * blockIdx.x], b0 = blk[3 * blockIdx.x + 1], r0 = P::kRest ? blk_rest[blockIdx.x] : 0u;
    const uint32_t pad = b0 & 15u;
    if (fb.x) {
        const typename P::Group h = P::group(c, s, i);
        const uint32_t g = s.first + i;
        uint8_t *p = buf + pad + lb;
#pragma unroll 1
        for (uint32_t k = 0; k < kSlots; k++) {
            if (!((h.peers >> k) & 1u)) continue;
            typename P::Send d;
            const uint32_t kind = P::peer(c, h, static_cast<size_t>(k) * c.cap + g, d);
            if constexpr (P::kRest) {
                if (kind == kBcastRest) {  // the send list's entry (send_list_kernel)
                    uint64_t *e = reinterpret_cast<uint64_t *>(o.rest + r0 + lr++);
                    e[0] = static_cast<uint64_t>(g) | (static_cast<uint64_t>(k) << 32) | (static_cast<uint64_t>(d.flags) << 40);
                    e[1] = d.next;
                    continue;  // (as an else of the frame's test: reconverging before it costs every peer)
                }
            }
            if (kind != kBcastFrame) continue;
            const uint64_t to = s.ids[static_cast<size_t>(k) * s.n + i];
            offs[lf++] = b0 + static_cast<uint32_t>(p - buf - pad);
            p = P::put(p, (g << 4) | k, h, d, to);
        }
    }
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < nf; j += kBcastThreads) o.offsets[f0 + j] = offs[j];
    wire_store_block<kBcastThreads>(o.bytes, buf, b0, nbytes);
}
