// k_app_frames.cuh -- bcast_append to the wire (DESIGN 3.15): for a range of group slots, the commit broadcast's
// entry-less MsgAppend frames through the broadcast pipeline (k_bcast.cuh), and the sends that need the leader's log as
// its rest list.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).

// Progress::is_paused (progress.rs:210-216) of a flag byte: Probe -> paused, Replicate -> ins.full(), Snapshot ->
// always.  send_list_kernel states the same test inline: written through this helper it compiles to different SASS
// (56 fewer instructions, other registers), so the step path's kernel is left as it is.
__device__ __forceinline__ bool pf_paused(uint32_t f) {
    const uint32_t state = f & RAFTGPU_PF_STATE_MASK;
    return state == RAFTGPU_STATE_PROBE ? (f & RAFTGPU_PF_PAUSED) != 0
                                        : (state == RAFTGPU_STATE_REPLICATE ? (f & RAFTGPU_PF_INS_FULL) != 0 : true);
}

struct AppBcast {
    static constexpr uint32_t kFrameMax = kWireAppFrameMax;
    static constexpr bool kRest = true;

    struct Group : BcastLeader {
        uint64_t last_index;
    };
    struct Send {
        uint64_t next;   // next_idx
        uint32_t flags;  // the rest entry's RAFTGPU_SEND_* flags
    };

    // last_index is the pair's (max of both halves), as committed.
    static __device__ __forceinline__ Group group(const Columns &c, const BcastSrc &s, uint32_t i) {
        Group r{};
        if (bcast_leader(c, s, i, r))
            r.last_index = r.wide ? umax64(c.last_index[r.lo], c.last_index[r.lo + 1]) : c.last_index[r.lo];
        return r;
    }
    // maybe_send_append(to, allow_empty = true) for a present peer (raft.rs:764-819): nothing for a paused peer; the rest
    // list when a snapshot is requested, when entries follow next_idx (raft_log.rs:382-387), or when the term of
    // next_idx - 1 lies before the leader's term and so needs the log; a frame otherwise.  Algorithmic bytes per peer:
    // 1 (pflags) + 8 (matched) + 2 (the next_idx offset) + 8 (pending_request_snapshot); per leader 8-16 (last_index).
    static __device__ __forceinline__ uint32_t peer(const Columns &c, const Group &h, size_t cell, Send &d) {
        const uint32_t f = c.pflags[cell];
        const uint64_t matched = c.matched[cell], prs = c.pending_req_snapshot[cell];
        const int16_t nd = c.next_d[cell];
        if (pf_paused(f)) return kBcastNone;
        d.next = off_decode(nd, matched, c.next_idx + cell);
        d.flags = prs != RAFTGPU_INVALID_INDEX ? RAFTGPU_SEND_SNAPSHOT : 0u;  // raft.rs:792-797, as send_list_kernel reports it
        return (d.flags || d.next <= h.last_index || d.next - 1 < h.term_start) ? kBcastRest : kBcastFrame;
    }
    // The frame of a peer that gets one (prepare_send_entries without entries, raft.rs:714-730, then send): index =
    // next_idx - 1, log_term = the term when index <= last_index (DESIGN 1's range form of raft_log.term), 0 above it.
    static __device__ __forceinline__ uint64_t log_term(const Group &h, uint64_t next) {
        return next - 1 <= h.last_index ? h.term : 0;
    }
    static __device__ __forceinline__ uint32_t len(const Group &h, const Send &d, uint64_t to) {
        return wire_app_len(to, h.from, h.term, log_term(h, d.next), d.next - 1, h.committed);
    }
    static __device__ __forceinline__ uint8_t *put(uint8_t *p, uint32_t hdr, const Group &h, const Send &d, uint64_t to) {
        return wire_put_append_frame<3>(p, hdr, to, h.from, h.term, log_term(h, d.next), d.next - 1, h.committed);
    }
};
