// k_hb_frames.cuh -- bcast_heartbeat to the wire (DESIGN 3.11): serialized MsgHeartbeat frames for a range of group
// slots through the broadcast pipeline (k_bcast.cuh).  The encoder is k_wire.cuh's, shared with the follower's
// responses (k_hb_follow.cuh).
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).

struct HbBcast {
    static constexpr uint32_t kFrameMax = kWireHbFrameMax;
    static constexpr bool kRest = false;

    struct Group : BcastLeader {
        uint64_t ctx;    // the read id the frames carry as their context, 0 for none
        uint32_t fixed;  // the bytes every frame of the group shares (wire_hb_fixed_len)
    };
    struct Send {
        uint64_t commit;
    };

    // A leader's frames also carry its last pending read id (read_only.rs:132-135 last_pending_request_ctx); a wide
    // group's high half takes the low half's read queue.
    static __device__ __forceinline__ Group group(const Columns &c, const BcastSrc &s, uint32_t i) {
        Group r{};
        if (bcast_leader(c, s, i, r) && c.rq_cap) {
            const uint32_t hc = c.rq_hc[r.lo], cnt = rq_count(hc);
            if (cnt) r.ctx = c.rq_ctx[rq_at(c, r.lo, hc, cnt - 1)];
        }
        r.fixed = wire_hb_fixed_len(r.from, r.term, r.ctx != 0);
        return r;
    }
    // send_heartbeat (raft.rs:822-844): every peer gets a frame, commit = min(matched, committed) (raft.rs:838-840).
    static __device__ __forceinline__ uint32_t peer(const Columns &c, const Group &h, size_t cell, Send &d) {
        d.commit = umin64(c.matched[cell], h.committed);
        return kBcastFrame;
    }
    static __device__ __forceinline__ uint32_t len(const Group &h, const Send &d, uint64_t to) {
        return wire_hb_len(h.fixed, to, d.commit);
    }
    // The read id travels as the context (DESIGN 3.10), id 0 as none.
    static __device__ __forceinline__ uint8_t *put(uint8_t *p, uint32_t hdr, const Group &h, const Send &d, uint64_t to) {
        return wire_put_hb_frame<8>(p, hdr, to, h.from, h.term, d.commit, h.ctx != 0, h.ctx);
    }
};
