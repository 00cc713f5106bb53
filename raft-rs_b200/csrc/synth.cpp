// synth.cpp -- deterministic synthetic AppendResponse workload (SURVEY 8(d)).
//
// A follower SIMULATION, not a tracker: it remembers what every follower has
// acknowledged and what the leader has appended, and emits the messages such
// followers would send.  It never evaluates a quorum or a Progress transition,
// so the engine and the oracle both consume it as opaque input.
#include <cstdint>
#include <cstring>

#include "raftgpu_synth.h"

namespace {

inline uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// stateless stream: draw k of (seed, a, b)
struct Rng {
    uint64_t s;
    Rng(uint64_t seed, uint64_t a, uint64_t b) : s(splitmix64(splitmix64(seed ^ a) + b)) {}
    uint64_t next() { return s = splitmix64(s); }
    uint64_t below(uint64_t n) { return next() % n; }
};

inline uint64_t sub_sat(uint64_t a, uint64_t b) { return a > b ? a - b : 0; }

}  // namespace

extern "C" {

int32_t raftgpu_synth_init(const raftgpu_synth_columns *c, uint64_t seed, uint32_t k_peers,
                           int32_t joint) {
    if (!c || c->n_groups > c->cap) return RAFTGPU_ERR_INVALID;
    const uint32_t n_slots = joint ? 7u : k_peers;
    if (n_slots < 1 || n_slots > RAFTGPU_SLOTS) return RAFTGPU_ERR_INVALID;
    const uint32_t in_mask = joint ? 0x1fu : ((1u << k_peers) - 1u);
    const uint32_t out_mask = joint ? 0x67u : 0u;  // slots {0,1,2,5,6}
    const size_t cap = c->cap;
    for (uint32_t g = 0; g < c->n_groups; g++) {
        Rng r(seed, g, 0);
        const uint64_t base = 1 + (r.next() & ((1ull << 40) - 1));
        for (uint32_t s = 0; s < RAFTGPU_SLOTS; s++) {
            const size_t cell = s * cap + g;
            uint64_t m = 0, nx = 0;
            uint8_t f = 0;
            if (s < n_slots) {
                if (s == 0) {
                    m = base;
                    nx = base + 1;
                    f = RAFTGPU_STATE_REPLICATE;
                } else {
                    m = sub_sat(base, r.below(1024));
                    nx = m + 1 + r.below(8);
                    if (r.below(100) < 95) {
                        f = RAFTGPU_STATE_REPLICATE;
                    } else {
                        f = RAFTGPU_STATE_PROBE | (r.below(2) ? RAFTGPU_PF_PAUSED : 0);
                    }
                }
            }
            c->matched[cell] = m;
            c->next_idx[cell] = nx;
            c->pflags[cell] = f;
            c->sim_acked[cell] = m;
            c->sim_flags[cell] = 0;
        }
        c->meta[g] = in_mask | (out_mask << 8) | RAFTGPU_META_HAS_SELF;  // self slot 0
        c->term[g] = 1 + (r.next() & ((1ull << 20) - 1));
        uint64_t ts = sub_sat(base, r.below(2048));
        c->term_start[g] = ts < 1 ? 1 : ts;
        c->last_index[g] = base;
        c->sim_last[g] = base;
        // some follower's acked index, minus a little: above the quorum index for
        // some groups (exercises the `>` guard), below it for others
        const uint32_t pick = n_slots > 1 ? 1 + static_cast<uint32_t>(r.below(n_slots - 1)) : 0;
        const uint64_t committed = sub_sat(c->matched[pick * cap + g], r.below(4));
        c->committed[g] = committed;
        for (uint32_t s = 0; s < RAFTGPU_SLOTS; s++) {
            const size_t cell = s * cap + g;
            uint64_t pc = 0;
            if (s == 0)
                pc = committed;
            else if (s < n_slots) {
                pc = sub_sat(committed, r.below(4));
                if (pc > c->matched[cell]) pc = c->matched[cell];
            }
            c->peer_committed[cell] = pc;
        }
    }
    return RAFTGPU_OK;
}

int32_t raftgpu_synth_round(const raftgpu_synth_columns *c, uint64_t seed, uint32_t round,
                            uint32_t k_peers, raftgpu_append_resp *out, uint64_t max_records,
                            uint64_t *out_n) {
    if (!c || !out || !out_n || k_peers < 1 || k_peers > RAFTGPU_SLOTS) return RAFTGPU_ERR_INVALID;
    const size_t cap = c->cap;
    const uint32_t followers = k_peers - 1;
    uint64_t n = 0;
    auto emit = [&](uint32_t g, uint32_t slot, uint8_t flags, uint64_t index, uint64_t commit) {
        raftgpu_append_resp &r = out[n++];
        r.group = g;
        r.peer_slot = static_cast<uint8_t>(slot);
        r.flags = flags;
        r.reserved = 0;
        r.index = index;
        r.commit = commit;
    };
    for (uint32_t g = 0; g < c->n_groups; g++) {
        if (n + 2ull * followers + 1 > max_records) {
            *out_n = n;
            return RAFTGPU_ERR_FULL;
        }
        Rng r(seed, g, 1 + round);
        const uint64_t last = c->sim_last[g];
        if (followers) {
            const uint32_t nresp = 1 + static_cast<uint32_t>(r.below(followers));
            const uint32_t start = static_cast<uint32_t>(r.below(followers));
            for (uint32_t j = 0; j < nresp; j++) {
                const uint32_t slot = 1 + (start + j) % followers;
                const size_t cell = slot * cap + g;
                const uint64_t acked = c->sim_acked[cell];
                const uint64_t p = r.below(100);
                if (p < 88) {  // accept: the follower appended up to `index` (<= leader's last)
                    uint64_t index = acked + 1 + r.below(63);
                    if (index > last) index = last;
                    if (index < acked) index = acked;
                    emit(g, slot, 0, index, sub_sat(index, r.below(4)));
                    c->sim_acked[cell] = index;
                    c->sim_flags[cell] = 0;
                } else if (p < 98) {  // stale accept (duplicate / reordered response)
                    const uint64_t index = sub_sat(acked, r.below(8));
                    emit(g, slot, 0, index, sub_sat(index, r.below(4)));
                } else {  // reject + hint
                    const bool again = c->sim_flags[cell] & 1u;
                    const uint64_t index = again ? acked : acked + 1 + r.below(4);
                    const uint64_t hint = again ? sub_sat(acked, r.below(4)) : acked + r.below(4);
                    const uint64_t request_snapshot = r.below(8) == 0 ? acked + 1 : 0;
                    emit(g, slot, RAFTGPU_REC_REJECT, index, sub_sat(acked, r.below(4)));
                    emit(g, slot, RAFTGPU_REC_EXT, hint, request_snapshot);
                    c->sim_flags[cell] = 1;
                }
            }
        }
        // the leader appends U[0,64) entries and persists (almost) all of them
        const uint64_t new_last = last + r.below(64);
        uint64_t persisted = sub_sat(new_last, r.below(4));
        if (persisted < c->sim_acked[g]) persisted = c->sim_acked[g];
        emit(g, 0, RAFTGPU_REC_LOCAL, persisted, new_last);
        c->sim_last[g] = new_last;
        c->sim_acked[g] = persisted;
    }
    *out_n = n;
    return RAFTGPU_OK;
}


// One synthetic round as a TRANSPORT would hold it (SURVEY 8(f4)): every follower record becomes a
// serialized eraftpb.Message (proto/proto/eraftpb.proto:71-92; proto3: zero fields are not written) behind
// a 4-byte frame header (group << 4 | peer_slot); a REJECT's EXT record folds into reject_hint /
// request_snapshot.  Leader-local records are not messages and are returned as they are.
static inline uint8_t *put_varint(uint8_t *p, uint64_t v) {
    while (v >= 0x80) {
        *p++ = static_cast<uint8_t>(v) | 0x80;
        v >>= 7;
    }
    *p++ = static_cast<uint8_t>(v);
    return p;
}
static inline uint8_t *put_field(uint8_t *p, uint32_t field, uint64_t v) {
    if (v == 0) return p;
    p = put_varint(p, static_cast<uint64_t>(field) << 3);
    return put_varint(p, v);
}

int32_t raftgpu_synth_wire_encode(const raftgpu_append_resp *recs, uint64_t n, const uint64_t *term, uint8_t *out_bytes,
                                  uint64_t bytes_cap, uint32_t *out_offsets, uint64_t *out_n_frames, uint64_t *out_n_bytes,
                                  raftgpu_append_resp *out_local, uint64_t *out_n_local) {
    if ((!recs && n) || !out_bytes || !out_offsets || !out_n_frames || !out_n_bytes || !out_local || !out_n_local)
        return RAFTGPU_ERR_INVALID;
    uint64_t nf = 0, nl = 0;
    uint8_t *p = out_bytes;
    out_offsets[0] = 0;
    for (uint64_t i = 0; i < n; i++) {
        const raftgpu_append_resp &r = recs[i];
        if (r.flags & RAFTGPU_REC_EXT) continue;
        if (r.flags & RAFTGPU_REC_LOCAL) {
            out_local[nl++] = r;
            continue;
        }
        if (static_cast<uint64_t>(p - out_bytes) + 80 > bytes_cap) return RAFTGPU_ERR_FULL;
        const bool has_ext = (r.flags & RAFTGPU_REC_REJECT) && i + 1 < n && (recs[i + 1].flags & RAFTGPU_REC_EXT);
        const uint32_t hdr = (r.group << 4) | (r.peer_slot & 15u);
        memcpy(p, &hdr, 4);
        p += 4;
        p = put_field(p, 1, 4);                                     // msg_type = MsgAppendResponse
        p = put_field(p, 2, 1);                                     // to: the leader
        p = put_field(p, 3, static_cast<uint64_t>(r.peer_slot) + 1); // from
        p = put_field(p, 4, term ? term[r.group] : 1);              // term
        p = put_field(p, 6, r.index);
        p = put_field(p, 8, r.commit);
        if (r.flags & RAFTGPU_REC_REJECT) {
            p = put_field(p, 10, 1);
            if (has_ext) {
                p = put_field(p, 11, recs[i + 1].index);   // reject_hint
                p = put_field(p, 13, recs[i + 1].commit);  // request_snapshot
            }
        }
        out_offsets[++nf] = static_cast<uint32_t>(p - out_bytes);
    }
    *out_n_frames = nf;
    *out_n_bytes = static_cast<uint64_t>(p - out_bytes);
    *out_n_local = nl;
    return RAFTGPU_OK;
}

// Heartbeat responses as a transport holds them: every RAFTGPU_REC_HEARTBEAT record becomes a MsgHeartbeatResponse
// (handle_heartbeat, raft.rs:2452-2464: term, commit, the heartbeat's context echoed); the ctx id of a
// RAFTGPU_REC_READ_CTX record is the context, 8 bytes little-endian, when it is non-zero.
int32_t raftgpu_synth_wire_encode_heartbeats(const raftgpu_append_resp *recs, uint64_t n, const uint64_t *term,
                                             uint8_t *out_bytes, uint64_t bytes_cap, uint32_t *out_offsets,
                                             uint64_t *out_n_frames, uint64_t *out_n_bytes) {
    if ((!recs && n) || !out_bytes || !out_offsets || !out_n_frames || !out_n_bytes) return RAFTGPU_ERR_INVALID;
    uint64_t nf = 0;
    uint8_t *p = out_bytes;
    out_offsets[0] = 0;
    for (uint64_t i = 0; i < n; i++) {
        const raftgpu_append_resp &r = recs[i];
        if (!(r.flags & RAFTGPU_REC_HEARTBEAT)) continue;
        if (static_cast<uint64_t>(p - out_bytes) + 64 > bytes_cap) return RAFTGPU_ERR_FULL;
        const uint32_t hdr = (r.group << 4) | (r.peer_slot & 15u);
        memcpy(p, &hdr, 4);
        p += 4;
        p = put_field(p, 1, 9);                                     // msg_type = MsgHeartbeatResponse
        p = put_field(p, 2, 1);                                     // to: the leader
        p = put_field(p, 3, static_cast<uint64_t>(r.peer_slot) + 1); // from
        p = put_field(p, 4, term ? term[r.group] : 1);              // term
        p = put_field(p, 8, r.commit);                              // commit
        if ((r.flags & RAFTGPU_REC_READ_CTX) && r.index) {
            *p++ = (12u << 3) | 2u;                                 // context, length-delimited
            *p++ = 8;
            for (int k = 0; k < 8; k++) *p++ = static_cast<uint8_t>(r.index >> (8 * k));
        }
        out_offsets[++nf] = static_cast<uint32_t>(p - out_bytes);
    }
    *out_n_frames = nf;
    *out_n_bytes = static_cast<uint64_t>(p - out_bytes);
    return RAFTGPU_OK;
}

int32_t raftgpu_synth_wire_encode_votes(const raftgpu_synth_vote *votes, uint64_t n, uint8_t *out_bytes, uint64_t bytes_cap,
                                        uint32_t *out_offsets, uint64_t *out_n_bytes) {
    if ((!votes && n) || !out_bytes || !out_offsets || !out_n_bytes) return RAFTGPU_ERR_INVALID;
    uint8_t *p = out_bytes;
    out_offsets[0] = 0;
    for (uint64_t i = 0; i < n; i++) {
        const raftgpu_synth_vote &v = votes[i];
        if (static_cast<uint64_t>(p - out_bytes) + 64 > bytes_cap) return RAFTGPU_ERR_FULL;
        memcpy(p, &v.hdr, 4);
        p += 4;
        p = put_field(p, 1, v.msg_type);
        p = put_field(p, 2, v.to);
        p = put_field(p, 3, v.from);
        p = put_field(p, 4, v.term);
        p = put_field(p, 8, v.commit);
        p = put_field(p, 10, v.reject != 0);
        p = put_field(p, 15, v.commit_term);
        out_offsets[i + 1] = static_cast<uint32_t>(p - out_bytes);
    }
    *out_n_bytes = static_cast<uint64_t>(p - out_bytes);
    return RAFTGPU_OK;
}

int32_t raftgpu_synth_wire_encode_vote_requests(const raftgpu_synth_vote_request *reqs, uint64_t n, uint8_t *out_bytes,
                                                uint64_t bytes_cap, uint32_t *out_offsets, uint64_t *out_n_bytes) {
    if ((!reqs && n) || !out_bytes || !out_offsets || !out_n_bytes) return RAFTGPU_ERR_INVALID;
    uint8_t *p = out_bytes;
    out_offsets[0] = 0;
    for (uint64_t i = 0; i < n; i++) {
        const raftgpu_synth_vote_request &r = reqs[i];
        if (r.context_len > sizeof(r.context)) return RAFTGPU_ERR_INVALID;
        if (static_cast<uint64_t>(p - out_bytes) + 120 > bytes_cap) return RAFTGPU_ERR_FULL;
        memcpy(p, &r.hdr, 4);
        p += 4;
        p = put_field(p, 1, r.msg_type);
        p = put_field(p, 2, r.to);
        p = put_field(p, 3, r.from);
        p = put_field(p, 4, r.term);
        p = put_field(p, 5, r.log_term);
        p = put_field(p, 6, r.index);
        p = put_field(p, 8, r.commit);
        if (r.context_len) {
            *p++ = (12u << 3) | 2u;  // context, length-delimited
            *p++ = static_cast<uint8_t>(r.context_len);
            memcpy(p, r.context, r.context_len);
            p += r.context_len;
        }
        p = put_field(p, 14, r.priority);
        p = put_field(p, 15, r.commit_term);
        out_offsets[i + 1] = static_cast<uint32_t>(p - out_bytes);
    }
    *out_n_bytes = static_cast<uint64_t>(p - out_bytes);
    return RAFTGPU_OK;
}

}  // extern "C"
