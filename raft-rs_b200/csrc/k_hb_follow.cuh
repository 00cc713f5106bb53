// k_hb_follow.cuh -- MsgHeartbeat frames at the follower (DESIGN 3.12): Raft::step's term rules as statuses, then
// handle_heartbeat (raft.rs:2452-2464) -- commit_to(m.commit) and one MsgHeartbeatResponse back through send
// (raft.rs:602-661) -- for the first passing frame of every group.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).
//
// Role stays with the caller: a bitmap selects the groups whose Raft is a Follower without a pending
// request_snapshot, and the ids (`from` of the responses) come from the caller's table.  The frame's header is the
// follower's own (group << 4 | x); x is not read and goes back unchanged in the response's header.
//
// Four kernels and no waiting between blocks: hfw_scan_kernel stages and decodes every frame once, classifies it and
// writes a 48-byte record per passing frame; hfw_apply_kernel marks the later frames of a group DUP, runs commit_to
// on the first one and sums the responses per block; block_starts_kernel<2> (k_wire.cuh) turns the sums into block
// starts; reply_write_kernel<HfwReply> (k_wire.cuh) encodes the responses (wire_put_hb_frame<9>) and stores them
// through shared memory.  Every kernel takes kWireThreads frames per block: one block sum per scan block.

// The caller's tables: select = bitmap from group 0 (required), self_ids = u64 [group slots].
struct HfwSrc {
    const uint32_t *select;
    const uint64_t *self_ids;
};

// A passing frame: w0 = its header | has_ctx << 32; to = m.from; from = the group's id; term; commit = m.commit (the
// new committed after the apply pass); ctx = the context's 8 bytes, little-endian.
struct __align__(16) HfwRec {
    uint64_t w0, to, from, term, commit, ctx;
};

__device__ __forceinline__ uint32_t hfw_len(const HfwRec &r) {
    return wire_hb_len(wire_hb_fixed_len(r.from, r.term, (r.w0 >> 32) & 1u), r.to, r.commit);
}

// Frame i: its status before the duplicate rule (checks in the order of raftgpu.h) and, for RAFTGPU_WIRE_OK, its
// record.
__device__ __forceinline__ uint32_t hfw_frame(const Columns &c, const WireSrc &w, const HfwSrc &f, const WireStage &s,
                                              const uint8_t *stage, uint32_t i, HfwRec &r) {
    uint32_t hdr;
    const uint8_t *msg;
    WireMsg m;
    if (wire_open<true, true>(w, s, stage, i, hdr, msg, m) != RAFTGPU_WIRE_OK) return RAFTGPU_WIRE_MALFORMED;
    const uint32_t g = hdr >> 4;
    const uint32_t meta = c.meta[g];
    if ((meta & RAFTGPU_META_WIDE_HI) || (c.rq_cap && !(c.rq_hc[g] & kRqAlloc))) return RAFTGPU_WIRE_MALFORMED;
    if (m.msg_type != 8u) return RAFTGPU_WIRE_SKIP_TYPE;  // MsgHeartbeat, eraftpb.proto:58
    // a Follower (the caller's bit) and not a leader here: step_follower (raft.rs:2276-2280) is the only path taken
    if (!((f.select[g >> 5] >> (g & 31u)) & 1u) || c.term_start[g] != RAFTGPU_NO_TERM_START) return RAFTGPU_WIRE_ROLE;
    const uint64_t term = c.term[g];
    if (term == 0 || m.term != term) return RAFTGPU_WIRE_TERM;  // raft.rs:1280-1411 decide those on the host
    if (m.ctx_len && m.ctx_len != 8u) return RAFTGPU_WIRE_CONTEXT;
    uint64_t top = umax64(c.committed[g], c.last_index[g]);
    if (meta & RAFTGPU_META_WIDE_LO) top = umax64(top, umax64(c.committed[g + 1], c.last_index[g + 1]));  // (wide_sync)
    if (m.commit > top) return RAFTGPU_WIRE_COMMIT_RANGE;  // commit_to would be fatal!, raft_log.rs:291-298
    r.w0 = hdr | (static_cast<uint64_t>(m.ctx_len != 0) << 32);
    r.to = m.from;                             // raft.rs:2462 to = m.from
    r.from = f.self_ids[g];                    // send: from = self.id (raft.rs:612)
    r.term = term;                             // send: term = self.term (raft.rs:650)
    r.commit = m.commit;
    r.ctx = m.ctx_len ? wire_ctx_u64(msg + m.ctx_off) : 0;
    return RAFTGPU_WIRE_OK;
}

// Pass 1: classify every frame; status[i] = wire status << 4; a passing frame's record, first_frame[group] = the
// lowest passing frame of the group.  Launched with kWireThreads threads per block; __maxnreg__ as hb_wire_scan_kernel,
// because ptxas, left alone, settles on 32 registers and spills.
__global__ void __maxnreg__(40) hfw_scan_kernel(Columns c, WireSrc w, HfwSrc f, uint8_t *__restrict__ status,
                                                               HfwRec *__restrict__ recs, uint32_t *__restrict__ first_frame) {
    __shared__ __align__(16) uint8_t stage[kWireStage + 16];
    WireStage s;
    const uint32_t i = wire_block_frame(w, stage, s);
    if (i == kNoFrame) return;
    HfwRec r;
    const uint32_t st = hfw_frame(c, w, f, s, stage, i, r);
    status[i] = static_cast<uint8_t>(st << 4);
    if (st == RAFTGPU_WIRE_OK) {
        recs[i] = r;
        atomicMin(&first_frame[static_cast<uint32_t>(r.w0) >> 4], i);
    }
}

// Pass 2: the first passing frame of every group runs commit_to (raft.rs:2453) -- on both halves of a wide pair, after
// wide_sync, as RAFTGPU_CTL_COMMIT_TO does -- and keeps the new committed in its record; a later one is
// RAFTGPU_WIRE_DUP.  from_out[i] (nullable) = m.from of an applied frame, 0 otherwise.  blk[2 * block + {0, 1}] = the
// block's responses and their bytes.  Algorithmic bytes per frame: 1 read + 1 written (+ 8 from_out); per passing
// frame 48 (record) + 4 (first_frame) read; per applied one 16-32 (committed, last_index) read, 8-16 (committed) + 8
// (record) written.
__global__ void __launch_bounds__(kWireThreads) hfw_apply_kernel(Columns c, uint32_t n, uint8_t *__restrict__ status,
                                                                 HfwRec *__restrict__ recs, const uint32_t *__restrict__ first_frame,
                                                                 uint64_t *__restrict__ from_out, uint32_t *__restrict__ blk) {
    const uint32_t i = blockIdx.x * kWireThreads + threadIdx.x;
    uint32_t resp = 0, bytes = 0;
    if (i < n) {
        uint64_t from = 0;
        if (status[i] == (RAFTGPU_WIRE_OK << 4)) {
            HfwRec r = recs[i];
            const uint32_t g = static_cast<uint32_t>(r.w0) >> 4;
            if (first_frame[g] != i) {
                status[i] = static_cast<uint8_t>(RAFTGPU_WIRE_DUP << 4);
            } else {
                if (c.meta[g] & RAFTGPU_META_WIDE_LO) {
                    wide_sync(c, g);
                    commit_to_group(c, g + 1, r.commit);
                }
                commit_to_group(c, g, r.commit);  // (in range: the scan checked it)
                r.commit = c.committed[g];        // raft.rs:2462 commit = raft_log.committed
                recs[i].commit = r.commit;
                status[i] = static_cast<uint8_t>((RAFTGPU_WIRE_OK << 4) | RAFTGPU_RES_OK);
                from = r.to;
                resp = 1;
                bytes = hfw_len(r);
            }
        }
        if (from_out) from_out[i] = from;
    }
    block_sums<2, kWireThreads>({resp, bytes}, blk);
}

// Pass 4 is reply_write_kernel<HfwReply> (k_wire.cuh): the frames the apply pass marked RAFTGPU_RES_OK answer.
struct HfwReply {
    using Rec = HfwRec;
    static constexpr uint32_t kFrameMax = kWireHbFrameMax;
    __device__ __forceinline__ static bool answers(uint8_t status) { return status & RAFTGPU_RES_OK; }
    __device__ __forceinline__ static uint32_t len(const HfwRec &r) { return hfw_len(r); }
    __device__ __forceinline__ static uint8_t *put(uint8_t *p, const HfwRec &r) {  // MsgHeartbeatResponse, raft.rs:2458-2463
        return wire_put_hb_frame<9>(p, static_cast<uint32_t>(r.w0), r.to, r.from, r.term, r.commit, (r.w0 >> 32) & 1u, r.ctx);
    }
};
