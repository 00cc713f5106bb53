// k_hb_frames.cuh -- bcast_heartbeat to the wire (DESIGN 3.11): serialized MsgHeartbeat frames for a range of group
// slots, in ascending (group, slot) order, in the frame format of k_wire.cuh.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).
//
// Three kernels and no waiting between blocks (a decoupled look-back would spin across blocks): hbf_size_kernel
// counts every group's frames and bytes and sums them per block, hbf_scan_kernel (one block) turns the block sums
// into block starts and the totals, hbf_write_kernel re-derives each group's frames, lays out the block's contiguous
// output in shared memory and stores it with 16-byte stores.  Nothing in the arena is written.  The encoder, the scan
// kernel and the block store are k_wire.cuh's, shared with the follower's responses (k_hb_follow.cuh).

constexpr uint32_t kHbfThreads = 128;                                           // group slots per block of the size and write kernels
constexpr uint32_t kHbfBufBytes = kHbfThreads * kSlots * kWireHbFrameMax + 16;  // + the block's misalignment
constexpr uint32_t kHbfSmem = kHbfBufBytes + kHbfThreads * kSlots * 4;          // + the block's frame offsets

// The range and the caller's tables: select = bitmap from group 0 (nullptr = all), ids = u64 [kSlots + 1][n].
struct HbfSrc {
    uint32_t first, n, hi;
    const uint32_t *select;
    const uint64_t *ids;
};

// What group slot first + i sends: `peers` = the slots that get a frame, and the fields every frame shares.
struct HbfGroup {
    uint32_t peers;
    bool no_term;  // a selected leader whose term is 0 (set on the low half only: counted once per group)
    uint64_t from, term, committed, ctx;
};

// bcast_heartbeat's choices for one slot (raft.rs:868-889): a leader (term_start set) that is allocated, selected and
// has a term sends to every present peer but itself.  A wide group's high half takes the low half's selection bit,
// term, term_start, `from` and read queue; committed is the pair's (max of both halves).
__device__ __forceinline__ HbfGroup hbf_group(const Columns &c, const HbfSrc &s, uint32_t i) {
    HbfGroup r{};
    const uint32_t g = s.first + i;
    const uint32_t meta = c.meta[g];
    const bool hi_half = (meta & RAFTGPU_META_WIDE_HI) != 0;
    const uint32_t lo = hi_half ? g - 1 : g;  // (the host refuses a range that splits a pair: lo >= first)
    if (lo >= s.hi) return r;
    if (s.select && !((s.select[lo >> 5] >> (lo & 31u)) & 1u)) return r;
    if (c.rq_cap && !(c.rq_hc[lo] & kRqAlloc)) return r;
    if (c.term_start[lo] == RAFTGPU_NO_TERM_START) return r;  // not a leader: ping does nothing
    r.term = c.term[lo];
    if (r.term == 0) {
        r.no_term = !hi_half;
        return r;
    }
    uint32_t peers = RAFTGPU_META_IN(meta) | RAFTGPU_META_OUT(meta) | RAFTGPU_META_LEARN(meta);
    if (meta & RAFTGPU_META_HAS_SELF) peers &= ~(1u << RAFTGPU_META_SELF(meta));  // raft.rs:887 id != self_id
    r.peers = peers;
    if (!peers) return r;
    const bool wide = hi_half || (meta & RAFTGPU_META_WIDE_LO);
    r.committed = wide ? umax64(c.committed[lo], c.committed[lo + 1]) : c.committed[g];
    r.from = s.ids[static_cast<size_t>(kSlots) * s.n + (lo - s.first)];
    if (c.rq_cap) {  // read_only.rs:132-135 last_pending_request_ctx
        const uint32_t hc = c.rq_hc[lo], cnt = rq_count(hc);
        if (cnt) r.ctx = c.rq_ctx[rq_at(c, lo, hc, cnt - 1)];
    }
    return r;
}

// The bytes every frame of the group shares (header, msg_type, from, term, context); wire_hb_len adds `to` and `commit`.
__device__ __forceinline__ uint32_t hbf_fixed(const HbfGroup &h) { return wire_hb_fixed_len(h.from, h.term, h.ctx != 0); }
// One MsgHeartbeat frame with header (group << 4 | slot); the read id travels as the context (DESIGN 3.10), id 0 as none.
__device__ __forceinline__ uint8_t *hbf_frame(uint8_t *p, uint32_t g, uint32_t slot, const HbfGroup &h, uint64_t to,
                                              uint64_t commit) {
    return wire_put_hb_frame<8>(p, (g << 4) | slot, to, h.from, h.term, commit, h.ctx != 0, h.ctx);
}

// Pass 1: cnt[i] = {frames, bytes} of group slot first + i; blk[3 * block + {0, 1, 2}] = the block's frames, bytes and
// leaders without a term.  Algorithmic bytes per slot: 4 (meta) + 8 (term_start) + 8 (term) read; per leader 8-16
// (committed) + 8 (from) + 4 (+ 8) (the read queue) + per peer 8 (matched) + 8 (its id); 8 written.
__global__ void __launch_bounds__(kHbfThreads) hbf_size_kernel(Columns c, HbfSrc s, uint2 *__restrict__ cnt,
                                                               uint32_t *__restrict__ blk) {
    const uint32_t i = blockIdx.x * kHbfThreads + threadIdx.x;
    uint32_t frames = 0, bytes = 0, no_term = 0;
    if (i < s.n) {
        const HbfGroup h = hbf_group(c, s, i);
        no_term = h.no_term;
        const uint32_t fixed = hbf_fixed(h), g = s.first + i;
#pragma unroll
        for (int k = 0; k < kSlots; k++) {
            if (!((h.peers >> k) & 1u)) continue;
            const uint64_t to = s.ids[static_cast<size_t>(k) * s.n + i];
            const uint64_t commit = umin64(c.matched[static_cast<size_t>(k) * c.cap + g], h.committed);  // raft.rs:838-840
            frames++;
            bytes += wire_hb_len(fixed, to, commit);
        }
        cnt[i] = make_uint2(frames, bytes);
    }
    block_sums<3, kHbfThreads>({frames, bytes, no_term}, blk);
}

// (Pass 2 is hbf_scan_kernel<3>, k_wire.cuh.)
// Pass 3: when the output fits, every block writes its groups' frames -- bytes [blk start, + its bytes) of `out` and
// offsets [blk start, + its frames) -- through shared memory: the frames are assembled there at their offset from the
// 16-byte boundary below the block's start, so whole 16-byte chunks go out as uint4 stores and only the two chunks
// shared with the neighbouring blocks byte by byte.  Reads as pass 1 (+ 8 per slot of cnt); writes the frames.
__global__ void __launch_bounds__(kHbfThreads) hbf_write_kernel(Columns c, HbfSrc s, const uint2 *__restrict__ cnt,
                                                                const uint32_t *__restrict__ blk,
                                                                const uint32_t *__restrict__ flag, uint8_t *__restrict__ out,
                                                                uint32_t *__restrict__ offsets) {
    extern __shared__ __align__(16) uint8_t hbf_smem[];
    if (!flag[0]) return;
    uint8_t *buf = hbf_smem;
    uint32_t *offs = reinterpret_cast<uint32_t *>(hbf_smem + kHbfBufBytes);
    const uint32_t i = blockIdx.x * kHbfThreads + threadIdx.x;
    const uint2 fb = i < s.n ? cnt[i] : make_uint2(0u, 0u);
    uint32_t lf = fb.x, lb = fb.y, nf, nbytes;
    wire_block_scan<kHbfThreads / 32>(lf, lb, nf, nbytes);
    const uint32_t f0 = blk[3 * blockIdx.x], b0 = blk[3 * blockIdx.x + 1], pad = b0 & 15u;
    if (fb.x) {
        const HbfGroup h = hbf_group(c, s, i);
        const uint32_t g = s.first + i;
        uint8_t *p = buf + pad + lb;
#pragma unroll 1
        for (uint32_t k = 0; k < kSlots; k++) {
            if (!((h.peers >> k) & 1u)) continue;
            const uint64_t to = s.ids[static_cast<size_t>(k) * s.n + i];
            const uint64_t commit = umin64(c.matched[static_cast<size_t>(k) * c.cap + g], h.committed);
            offs[lf++] = b0 + static_cast<uint32_t>(p - buf - pad);
            p = hbf_frame(p, g, k, h, to, commit);
        }
    }
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < nf; j += kHbfThreads) offsets[f0 + j] = offs[j];
    wire_store_block<kHbfThreads>(out, buf, b0, nbytes);
}
