// k_read.cuh -- ReadIndex with ReadOnlyOption::Safe (DESIGN 3.9): the request, ack, advance, recheck and last-ctx
// kernels over the arena's read queues (Columns::rq_*, helpers in k_common.cuh).  Every quorum test is
// quorum_group's has_quorum (k_control.cuh).
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).

// The configuration a read needs of group g (the low half of a wide group): its voter halves over 16 peer slots, the
// self bit (read_only.rs:97 acks = {self_id}; 0 when the leader holds no slot), and the log bounds of the range-form
// commit_to_current_term (raft.rs:581-585: term(committed) == term <=> term_start <= committed <= last_index).  The
// halves of a wide group agree on their log columns up to what one half alone has seen (wide_sync).
struct RqGroup {
    uint32_t in, out, self_bit;
    uint64_t committed;
    bool in_term;
};
__device__ __forceinline__ RqGroup rq_group(const Columns &c, uint32_t g, uint32_t meta) {
    const bool wide = (meta & RAFTGPU_META_WIDE_LO) != 0;
    const uint32_t meta_hi = wide ? c.meta[g + 1] : 0u;
    RqGroup r;
    r.in = RAFTGPU_META_IN(meta) | (RAFTGPU_META_IN(meta_hi) << 8);
    r.out = RAFTGPU_META_OUT(meta) | (RAFTGPU_META_OUT(meta_hi) << 8);
    r.self_bit = (meta & RAFTGPU_META_HAS_SELF) ? 1u << RAFTGPU_META_SELF(meta)
                 : (meta_hi & RAFTGPU_META_HAS_SELF) ? 1u << (8 + RAFTGPU_META_SELF(meta_hi)) : 0u;
    r.committed = wide ? umax64(c.committed[g], c.committed[g + 1]) : c.committed[g];
    const uint64_t last = wide ? umax64(c.last_index[g], c.last_index[g + 1]) : c.last_index[g];
    const uint64_t ts = c.term_start[g];
    r.in_term = ts <= r.committed && r.committed <= last;
    return r;
}

__device__ __forceinline__ void rq_emit(raftgpu_read_state *out, unsigned long long pos, unsigned long long capacity,
                                        uint32_t g, uint64_t ctx, uint64_t index) {
    if (pos >= capacity) return;  // (the host entry points size `out` so that this never happens)
    uint64_t *p = reinterpret_cast<uint64_t *>(out + pos);
    p[0] = g;
    p[1] = ctx;
    p[2] = index;
}

// Pop the first m entries of group g's queue (ReadOnly::advance, read_only.rs:115-129) into out[pos, pos + m), in
// queue order.
__device__ __forceinline__ void rq_release(const Columns &c, uint32_t g, uint32_t hc, uint32_t m, raftgpu_read_state *out,
                                           unsigned long long capacity, unsigned long long pos) {
    for (uint32_t k = 0; k < m; k++) {
        const size_t cell = rq_at(c, g, hc, k);
        rq_emit(out, pos + k, capacity, g, c.rq_ctx[cell], c.rq_index[cell]);
    }
    uint32_t head = (hc & 0xffu) + m;
    if (head >= c.rq_cap) head -= c.rq_cap;
    c.rq_hc[g] = (hc & kRqAlloc) | ((rq_count(hc) - m) << 8) | head;
}

// ---------------------------------------------------------------------------
// read_order_kernel: the requests must be in non-decreasing group order (queue order is arrival order).  A violation
// sets *flag (which read_request_kernel reads before it applies anything) and bumps *bad once.
__global__ void __launch_bounds__(256)
read_order_kernel(const raftgpu_read_req *__restrict__ reqs, uint64_t n, uint32_t *__restrict__ flag, uint32_t *__restrict__ bad) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x + 1; i < n; i += stride)
        if (reqs[i].group < reqs[i - 1].group && atomicExch(flag, 1u) == 0u && bad) atomicAdd(bad, 1u);
}

// read_request_kernel: MsgReadIndex at the leader (raft.rs:2056-2091) for a batch in group order.  The thread of the
// first request of each group's run walks the run in order: commit_to_current_term (:2057-2062), is_singleton
// (:2064-2070, joint.rs:77-79: outgoing empty, one incoming voter), else ReadOnly::add_request (read_only.rs:86-99:
// a pending ctx changes nothing; a new one goes to the back with index = committed, acks = {self}).  Reads a
// singleton releases are reserved with one atomic per run and written in request order.  Algorithmic bytes per
// request: 16 read, 1 written; per queued read 18 written; per group 4 + 8 (hc, meta) + 24 (log bounds) read, and
// the ctx of every pending entry for the duplicate test.
__global__ void __launch_bounds__(256)
read_request_kernel(Columns c, const raftgpu_read_req *__restrict__ reqs, uint64_t n, uint8_t *__restrict__ results,
                    raftgpu_read_state *__restrict__ out, unsigned long long capacity, unsigned long long *__restrict__ count,
                    const uint32_t *__restrict__ flag) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    const bool refused = *flag != 0;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        if (refused) {  // out of group order: nothing is applied
            if (results) results[i] = 0;
            continue;
        }
        const uint32_t g = reqs[i].group;
        if (i > 0 && reqs[i - 1].group == g) continue;  // not the first request of its group's run
        uint64_t end = i + 1;
        while (end < n && reqs[end].group == g) end++;
        const uint32_t hc0 = g < c.cap ? c.rq_hc[g] : 0u;
        const uint32_t meta = (hc0 & kRqAlloc) ? c.meta[g] : 0u;
        if (!(hc0 & kRqAlloc) || (meta & RAFTGPU_META_WIDE_HI)) {
            for (uint64_t j = i; j < end; j++)
                if (results) results[j] = RAFTGPU_READ_NO_GROUP;
            continue;
        }
        const RqGroup q = rq_group(c, g, meta);
        const bool singleton = q.out == 0 && __popc(q.in) == 1;
        if (q.in_term && singleton) {  // every request with a ctx is ready at once, index = committed
            uint32_t m = 0;
            for (uint64_t j = i; j < end; j++) m += reqs[j].ctx != 0;
            unsigned long long pos = m ? atomicAdd(count, static_cast<unsigned long long>(m)) : 0ull;
            for (uint64_t j = i; j < end; j++) {
                const uint64_t ctx = reqs[j].ctx;
                if (ctx) rq_emit(out, pos++, capacity, g, ctx, q.committed);
                if (results) results[j] = ctx ? RAFTGPU_READ_READY : RAFTGPU_READ_NO_CTX;
            }
            continue;
        }
        uint32_t hc = hc0;
        for (uint64_t j = i; j < end; j++) {
            const uint64_t ctx = reqs[j].ctx;
            uint32_t r;
            if (!ctx) {
                r = RAFTGPU_READ_NO_CTX;
            } else if (!q.in_term) {
                r = RAFTGPU_READ_DROPPED;
            } else {
                const uint32_t cnt = rq_count(hc);
                r = RAFTGPU_READ_QUEUED;
                for (uint32_t k = 0; k < cnt; k++)
                    if (c.rq_ctx[rq_at(c, g, hc, k)] == ctx) {
                        r = RAFTGPU_READ_DUP;
                        break;
                    }
                if (r == RAFTGPU_READ_QUEUED && cnt == c.rq_cap) r = RAFTGPU_READ_FULL;
                if (r == RAFTGPU_READ_QUEUED) {
                    const size_t cell = rq_at(c, g, hc, cnt);
                    c.rq_ctx[cell] = ctx;
                    c.rq_index[cell] = q.committed;
                    c.rq_acks[cell] = static_cast<uint16_t>(q.self_bit);
                    hc += 1u << 8;
                }
            }
            if (results) results[j] = static_cast<uint8_t>(r);
        }
        if (hc != hc0) c.rq_hc[g] = hc;
    }
}

// ---------------------------------------------------------------------------
// read_ack_kernel: recv_ack (read_only.rs:104-110) for every RAFTGPU_REC_HEARTBEAT | RAFTGPU_REC_READ_CTX record, one
// thread each (raft.rs:1805-1812: a responder without Progress, :1779-1789, and an empty context are ignored).  The
// responder's bit is ORed into its ctx's pending entry -- peer s of a wide group's high half is bit 8 + s of the
// low half's queue -- the entry's ring position is marked in hit[group], and the group goes, once, onto the touched
// list for read_advance_kernel.  Acks commute, so the records need no order and no waves (DESIGN 3.9).  Algorithmic
// bytes per record: 24 read, + 4 (meta) + 4 (hc) + 8 per pending entry scanned, and two atomics (the entry's acks,
// the group's hit mask) when its ctx is pending.
__global__ void __launch_bounds__(256)
read_ack_kernel(Columns c, const raftgpu_append_resp *__restrict__ recs, uint64_t n, unsigned long long *__restrict__ hit,
                uint32_t *__restrict__ list, uint32_t *__restrict__ list_n) {
    constexpr uint32_t kWant = RAFTGPU_REC_HEARTBEAT | RAFTGPU_REC_READ_CTX;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    // warp-uniform trip count: the whole warp reaches warp_reserve together
    for (uint64_t i0 = static_cast<uint64_t>(blockIdx.x) * blockDim.x + (threadIdx.x & ~31u); i0 < n; i0 += stride) {
        const uint64_t i = i0 + (threadIdx.x & 31);
        uint32_t qg = 0, first = 0;  // first: this record put its group on the touched list
        if (i < n) {
            const uint64_t *p = reinterpret_cast<const uint64_t *>(recs + i);
            const uint64_t w0 = p[0], ctx = p[1];
            const uint32_t g = static_cast<uint32_t>(w0), slot = static_cast<uint32_t>(w0 >> 32) & 0xffu;
            const bool want = ((static_cast<uint32_t>(w0 >> 40) & kWant) == kWant) && ctx != 0 && g < c.cap && slot < kSlots;
            const uint32_t meta = want ? c.meta[g] : 0u;
            const uint32_t present = RAFTGPU_META_IN(meta) | RAFTGPU_META_OUT(meta) | RAFTGPU_META_LEARN(meta);
            if ((present >> slot) & 1u) {
                const bool hi = (meta & RAFTGPU_META_WIDE_HI) != 0;
                qg = hi ? g - 1 : g;
                const uint32_t bit = hi ? 8 + slot : slot;
                const uint32_t hc = c.rq_hc[qg];
                for (uint32_t k = 0; k < rq_count(hc); k++) {
                    const size_t cell = rq_at(c, qg, hc, k);
                    if (c.rq_ctx[cell] != ctx) continue;
                    // u16 acks: the OR goes to the aligned 32-bit word that holds them
                    atomicOr(reinterpret_cast<uint32_t *>(c.rq_acks) + (cell >> 1), (1u << bit) << (16 * (cell & 1)));
                    first = atomicOr(&hit[qg], 1ull << (cell / c.cap)) == 0ull;
                    break;
                }
            }
        }
        const uint32_t pos = warp_reserve(list_n, first);
        if (first) list[pos] = qg;
    }
}

// read_advance_kernel: per touched group, the last queue entry that an ack of the batch named and whose acks have a
// quorum (has_quorum, tracker.rs:367-372, tested from the back), and ReadOnly::advance to it (read_only.rs:115-129):
// it and every entry in front of it are released, contiguously and in queue order.  An entry no ack named is not
// tested: in the reference only the entry a response names is (raft.rs:1812-1815), and one that already has a
// quorum (a configuration change can give it one) waits for that.  hit[g] is cleared for the next batch.
// Algorithmic bytes per touched group: 4 (hc) + 8 (hit) + 4-8 (meta) + 2 per entry tested read, 8 written; 24
// written and 16 read per released read.
__global__ void __launch_bounds__(256)
read_advance_kernel(Columns c, unsigned long long *__restrict__ hit, const uint32_t *__restrict__ list,
                    const uint32_t *__restrict__ list_n, raftgpu_read_state *__restrict__ out, unsigned long long capacity,
                    unsigned long long *__restrict__ count) {
    const uint32_t stride = gridDim.x * blockDim.x, m = *list_n;
    for (uint32_t t0 = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); t0 < m; t0 += stride) {  // warp-uniform
        const uint32_t t = t0 + (threadIdx.x & 31);
        uint32_t g = 0, hc = 0, upto = 0;
        if (t < m) {
            g = list[t];
            hc = c.rq_hc[g];
            const unsigned long long named = hit[g];
            hit[g] = 0ull;
            for (uint32_t k = rq_count(hc); k > 0; k--) {
                const size_t cell = rq_at(c, g, hc, k - 1);
                if (((named >> (cell / c.cap)) & 1ull) && quorum_group(c, g, 0, c.rq_acks[cell])) {
                    upto = k;
                    break;
                }
            }
        }
        const unsigned long long pos = warp_reserve(count, upto);
        if (upto) rq_release(c, g, hc, upto, out, capacity, pos);
    }
}

// read_recheck_kernel: the tail of post_conf_change (raft.rs:2648-2664) for the listed (distinct) groups: recv_ack(self,
// last_pending_request_ctx) and, when the new configuration gives that entry a quorum, advance(last ctx) releases
// the whole queue.
__global__ void __launch_bounds__(256)
read_recheck_kernel(Columns c, const uint32_t *__restrict__ groups, uint64_t n, raftgpu_read_state *__restrict__ out,
                    unsigned long long capacity, unsigned long long *__restrict__ count) {
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t i0 = static_cast<uint64_t>(blockIdx.x) * blockDim.x + (threadIdx.x & ~31u); i0 < n; i0 += stride) {
        const uint64_t i = i0 + (threadIdx.x & 31);
        uint32_t g = 0, hc = 0, cnt = 0;
        bool release = false;
        if (i < n) {
            g = groups[i];
            hc = c.rq_hc[g];
            cnt = rq_count(hc);
            if (cnt) {
                const size_t last = rq_at(c, g, hc, cnt - 1);
                const uint32_t acks = c.rq_acks[last] | rq_group(c, g, c.meta[g]).self_bit;
                c.rq_acks[last] = static_cast<uint16_t>(acks);
                release = quorum_group(c, g, 0, acks) != 0;
            }
        }
        const unsigned long long pos = warp_reserve(count, release ? cnt : 0u);
        if (release) rq_release(c, g, hc, cnt, out, capacity, pos);
    }
}

// read_last_ctx_kernel: ReadOnly::last_pending_request_ctx (read_only.rs:132-135) per group, the ctx bcast_heartbeat
// attaches (raft.rs:876); 0 for none.  Algorithmic bytes per group: 4 read (+ 8 when a read is pending), 8 written.
__global__ void __launch_bounds__(256)
read_last_ctx_kernel(Columns c, uint32_t first, uint32_t n, uint64_t *__restrict__ out) {
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint32_t g = first + i, hc = c.rq_hc[g], cnt = rq_count(hc);
        out[i] = cnt ? c.rq_ctx[rq_at(c, g, hc, cnt - 1)] : 0ull;
    }
}

// Group alloc / free: the allocated bit of groups [first, first + n), with an empty queue.
__global__ void read_mark_kernel(uint32_t *__restrict__ hc, uint32_t first, uint32_t n, uint32_t value) {
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) hc[first + i] = value;
}
