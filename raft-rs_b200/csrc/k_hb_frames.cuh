// k_hb_frames.cuh -- bcast_heartbeat to the wire (DESIGN 3.11): serialized MsgHeartbeat frames for a range of group
// slots, in ascending (group, slot) order, in the frame format of k_wire.cuh.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).
//
// Three kernels and no waiting between blocks (a decoupled look-back would spin across blocks): hbf_size_kernel
// counts every group's frames and bytes and sums them per block, hbf_scan_kernel (one block) turns the block sums
// into block starts and the totals, hbf_write_kernel re-derives each group's frames, lays out the block's contiguous
// output in shared memory and stores it with 16-byte stores.  Nothing in the arena is written.

constexpr uint32_t kHbfThreads = 128;                           // group slots per block of the size and write kernels
constexpr uint32_t kHbfFrameMax = 60;                           // 4-byte header + at most 56 bytes of Message
constexpr uint32_t kHbfBufBytes = kHbfThreads * kSlots * kHbfFrameMax + 16;  // + the block's misalignment
constexpr uint32_t kHbfSmem = kHbfBufBytes + kHbfThreads * kSlots * 4;      // + the block's frame offsets
constexpr uint32_t kHbfScanThreads = 1024;

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

// bytes of v as a base-128 varint
__device__ __forceinline__ uint32_t hbf_vlen(uint64_t v) {
    return v ? (70u - static_cast<uint32_t>(__clzll(static_cast<long long>(v)))) / 7u : 1u;
}

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

// Bytes of a heartbeat-kind frame (MsgHeartbeat here, MsgHeartbeatResponse in k_hb_follow.cuh) before its `to` and
// `commit`: header, msg_type, from, term (never 0 on this path) and the 8-byte context when there is one.
__device__ __forceinline__ uint32_t hb_msg_fixed(uint64_t from, uint64_t term, bool has_ctx) {
    return 4u + 2u + (from ? 1u + hbf_vlen(from) : 0u) + 1u + hbf_vlen(term) + (has_ctx ? 10u : 0u);
}

// Bytes of the frame to a peer with id `to` and commit `commit`, after the fields its group's frames share (`fixed`:
// header, msg_type, from, term, context).
__device__ __forceinline__ uint32_t hbf_fixed(const HbfGroup &h) { return hb_msg_fixed(h.from, h.term, h.ctx != 0); }
__device__ __forceinline__ uint32_t hbf_len(uint32_t fixed, uint64_t to, uint64_t commit) {
    return fixed + (to ? 1u + hbf_vlen(to) : 0u) + (commit ? 1u + hbf_vlen(commit) : 0u);
}

__device__ __forceinline__ uint8_t *hbf_varint(uint8_t *p, uint64_t v) {
    while (v >= 0x80u) {
        *p++ = static_cast<uint8_t>(v | 0x80u);
        v >>= 7;
    }
    *p++ = static_cast<uint8_t>(v);
    return p;
}

// One heartbeat-kind frame: u32 LE header, then eraftpb.Message (eraftpb.proto:71-92) in field-number order with zero
// scalars omitted: 1 msg_type = kType (MsgHeartbeat 8, MsgHeartbeatResponse 9, eraftpb.proto:58-59), 2 to, 3 from,
// 4 term (never 0 on this path), 8 commit, 12 context (the 8 little-endian bytes of ctx when has_ctx).
template <uint8_t kType>
__device__ __forceinline__ uint8_t *hb_msg_frame(uint8_t *p, uint32_t hdr, uint64_t to, uint64_t from, uint64_t term,
                                                 uint64_t commit, bool has_ctx, uint64_t ctx) {
    p[0] = static_cast<uint8_t>(hdr);
    p[1] = static_cast<uint8_t>(hdr >> 8);
    p[2] = static_cast<uint8_t>(hdr >> 16);
    p[3] = static_cast<uint8_t>(hdr >> 24);
    p[4] = 0x08;  // field 1, varint
    p[5] = kType;
    p += 6;
    if (to) {
        *p++ = 0x10;
        p = hbf_varint(p, to);
    }
    if (from) {
        *p++ = 0x18;
        p = hbf_varint(p, from);
    }
    *p++ = 0x20;
    p = hbf_varint(p, term);
    if (commit) {
        *p++ = 0x40;
        p = hbf_varint(p, commit);
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

// One MsgHeartbeat frame with header (group << 4 | slot); the read id travels as the context (DESIGN 3.10), id 0 as none.
__device__ __forceinline__ uint8_t *hbf_frame(uint8_t *p, uint32_t g, uint32_t slot, const HbfGroup &h, uint64_t to,
                                              uint64_t commit) {
    return hb_msg_frame<8>(p, (g << 4) | slot, to, h.from, h.term, commit, h.ctx != 0, h.ctx);
}

// Exclusive scan of two u32 counts over a block of W warps; *tot_a / *tot_b = the block's sums (every thread).
template <uint32_t W>
__device__ __forceinline__ void hbf_block_scan(uint32_t &a, uint32_t &b, uint32_t &tot_a, uint32_t &tot_b) {
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
            bytes += hbf_len(fixed, to, commit);
        }
        cnt[i] = make_uint2(frames, bytes);
    }
    __shared__ uint32_t sum[3][kHbfThreads / 32];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    frames = __reduce_add_sync(0xffffffffu, frames);
    bytes = __reduce_add_sync(0xffffffffu, bytes);
    no_term = __reduce_add_sync(0xffffffffu, no_term);
    if (lane == 0) {
        sum[0][warp] = frames;
        sum[1][warp] = bytes;
        sum[2][warp] = no_term;
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        uint32_t t = 0;
#pragma unroll
        for (uint32_t w = 0; w < kHbfThreads / 32; w++) t += sum[threadIdx.x][w];
        blk[3 * blockIdx.x + threadIdx.x] = t;
    }
}

// Pass 2, one block: blk's frames and bytes become each block's exclusive starts.  K = u32 per block in blk: {frames,
// bytes} (K = 2, k_hb_follow.cuh) or {frames, bytes, leaders without a term} (K = 3); totals = the K sums.  flag[0] =
// the output fits (d_offsets given, frames <= frames_cap, bytes <= bytes_cap); then offsets[frames] = bytes, the end of
// the last frame.
template <uint32_t K>
__global__ void __launch_bounds__(kHbfScanThreads) hbf_scan_kernel(uint32_t *__restrict__ blk, uint32_t nb, uint64_t bytes_cap,
                                                                   uint64_t frames_cap, uint64_t *__restrict__ totals,
                                                                   uint32_t *__restrict__ offsets, uint32_t *__restrict__ flag) {
    static_assert(K == 2 || K == 3, "blk holds {frames, bytes[, leaders without a term]} per block");
    uint32_t carry_f = 0, carry_b = 0, no_term = 0;
    for (uint32_t j0 = 0; j0 < nb; j0 += kHbfScanThreads) {  // (uniform trip count: every thread reaches the scan)
        const uint32_t j = j0 + threadIdx.x;
        uint32_t f = 0, b = 0;
        if (j < nb) {
            f = blk[K * j];
            b = blk[K * j + 1];
            if constexpr (K == 3) no_term += blk[K * j + 2];
        }
        uint32_t tf, tb;
        hbf_block_scan<kHbfScanThreads / 32>(f, b, tf, tb);
        if (j < nb) {
            blk[K * j] = carry_f + f;
            blk[K * j + 1] = carry_b + b;
        }
        carry_f += tf;
        carry_b += tb;
    }
    uint64_t t = 0;
    if constexpr (K == 3) {
        no_term = __reduce_add_sync(0xffffffffu, no_term);
        __shared__ uint32_t nt[kHbfScanThreads / 32];
        if ((threadIdx.x & 31u) == 0) nt[threadIdx.x >> 5] = no_term;
        __syncthreads();
        if (threadIdx.x == 0)
            for (uint32_t w = 0; w < kHbfScanThreads / 32; w++) t += nt[w];
    }
    if (threadIdx.x == 0) {
        totals[0] = carry_f;
        totals[1] = carry_b;
        if constexpr (K == 3) totals[2] = t;
        const bool fits = offsets && carry_f <= frames_cap && carry_b <= bytes_cap;
        flag[0] = fits;
        if (fits) offsets[carry_f] = carry_b;
    }
}

// A block's contiguous output [b0, b0 + nbytes) from shared memory, where it was assembled at buf + (b0 & 15): whole
// 16-byte chunks go out as uint4 stores, only the two chunks shared with the neighbouring blocks byte by byte.
template <uint32_t kThreads>
__device__ __forceinline__ void hbf_store_block(uint8_t *__restrict__ out, const uint8_t *buf, uint32_t b0, uint32_t nbytes) {
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
    hbf_block_scan<kHbfThreads / 32>(lf, lb, nf, nbytes);
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
    hbf_store_block<kHbfThreads>(out, buf, b0, nbytes);
}
