// k_hb_wire.cuh -- MsgHeartbeatResponse frames (DESIGN 3.10): the wire batch of k_wire.cuh, decoded with the context
// field, then the tracker part of handle_heartbeat_response (heartbeat_resp_one, k_control.cuh) on the first frame
// of every cell, and the read part as read_ack_kernel + read_advance_kernel (k_read.cuh) over the records the decode
// wrote.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).
//
// The context of a heartbeat that carries read id x is the 8 bytes of x, little-endian (the caller builds the
// heartbeat and the follower echoes its context, raft.rs:2461).  A frame whose context is anything else, or that has
// a context on an arena without read queues, is RAFTGPU_WIRE_CONTEXT: the host's own ReadOnly gets it whole.
//
// Two kernels, like the AppendResponse path, but the bytes are decoded once: the scan writes one 24-byte record per
// frame into the pass's scratch (flags 0 for a frame that is not applied), the apply pass reads the record back.

// Frame i as a heartbeat response: its status before the duplicate rule and, for RAFTGPU_WIRE_OK, its record
// (w0 = group | slot << 32 | flags << 40, ctx, commit = m.commit).
__device__ __forceinline__ uint32_t hb_wire_frame(const Columns &c, const WireSrc &w, const WireStage &s, const uint8_t *stage,
                                                  uint32_t i, uint64_t &w0, uint64_t &ctx, uint64_t &commit) {
    uint32_t hdr;
    const uint8_t *msg;
    WireMsg m;
    if (wire_open<true>(w, s, stage, i, hdr, msg, m) != RAFTGPU_WIRE_OK) return RAFTGPU_WIRE_MALFORMED;
    const uint32_t group = hdr >> 4, slot = hdr & 15u;
    if (m.msg_type != 9u) return RAFTGPU_WIRE_SKIP_TYPE;  // MsgHeartbeatResponse, eraftpb.proto:59
    const uint64_t gterm = c.term[group];
    if (gterm != 0 && m.term != gterm) return RAFTGPU_WIRE_TERM;
    uint32_t flags = RAFTGPU_REC_HEARTBEAT;
    if (m.ctx_len) {
        if (m.ctx_len != 8u || !c.rq_cap) return RAFTGPU_WIRE_CONTEXT;
        ctx = wire_ctx_u64(msg + m.ctx_off);
        flags |= RAFTGPU_REC_READ_CTX;  // raft.rs:1805-1818 runs for this response
    }
    w0 = static_cast<uint64_t>(group) | (static_cast<uint64_t>(slot) << 32) | (static_cast<uint64_t>(flags) << 40);
    commit = m.commit;
    return RAFTGPU_WIRE_OK;
}

// Pass 1: classify every frame, write its record (zero unless RAFTGPU_WIRE_OK), first_frame[cell] = the lowest
// frame index that wants the cell.  status[i] = wire status << 4.  Launched with kWireThreads threads per block;
// __maxnreg__ instead of __launch_bounds__ because ptxas, left alone, settles on 32 registers and spills.
__global__ void __maxnreg__(40) hb_wire_scan_kernel(Columns c, WireSrc w, uint8_t *__restrict__ status,
                                                                    raftgpu_append_resp *__restrict__ recs,
                                                                    uint32_t *__restrict__ first_frame) {
    __shared__ __align__(16) uint8_t stage[kWireStage + 16];
    WireStage s;
    const uint32_t i = wire_block_frame(w, stage, s);
    if (i == kNoFrame) return;
    uint64_t w0 = 0, ctx = 0, commit = 0;
    const uint32_t st = hb_wire_frame(c, w, s, stage, i, w0, ctx, commit);
    status[i] = static_cast<uint8_t>(st << 4);
    uint64_t *r = reinterpret_cast<uint64_t *>(recs + i);
    if (st != RAFTGPU_WIRE_OK) w0 = ctx = commit = 0;
    r[0] = w0;
    r[1] = ctx;
    r[2] = commit;
    if (st == RAFTGPU_WIRE_OK) {
        const uint32_t g = static_cast<uint32_t>(w0), slot = static_cast<uint32_t>(w0 >> 32) & 0xffu;
        if (slot < kSlots) atomicMin(&first_frame[static_cast<size_t>(slot) * c.cap + g], i);
    }
}

// Pass 2: the first frame of every cell runs the tracker part (raft.rs:1777-1804); a later one is RAFTGPU_WIRE_DUP and
// its record loses its flags, so the read part skips it too.  status[i] = wire status << 4 | RAFTGPU_RES_*.
// Algorithmic bytes per frame: 1 + 24 + 4 read; per applied frame what heartbeat_resp_kernel moves for a record.
__global__ void __launch_bounds__(256) hb_wire_apply_kernel(Columns c, uint32_t n, uint8_t *__restrict__ status,
                                                            raftgpu_append_resp *__restrict__ recs,
                                                            const uint32_t *__restrict__ first_frame) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || status[i] != (RAFTGPU_WIRE_OK << 4)) return;
    uint64_t *r = reinterpret_cast<uint64_t *>(recs + i);
    const uint64_t w0 = r[0], commit = r[2];
    const uint32_t g = static_cast<uint32_t>(w0), slot = static_cast<uint32_t>(w0 >> 32) & 0xffu;
    if (slot < kSlots && first_frame[static_cast<size_t>(slot) * c.cap + g] != i) {
        r[0] = w0 & 0xffffffffffull;
        status[i] = static_cast<uint8_t>(RAFTGPU_WIRE_DUP << 4);
        return;
    }
    const uint32_t res = heartbeat_resp_one(c, g, slot, commit, []() { return true; });
    status[i] = static_cast<uint8_t>((RAFTGPU_WIRE_OK << 4) | (res & 0xfu));
}
