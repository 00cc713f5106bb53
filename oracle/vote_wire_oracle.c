/* vote_wire_oracle.c -- see vote_wire_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#include "vote_wire_oracle.h"

#include <stdlib.h>
#include <string.h>

#define NO_TERM_START UINT64_MAX

static inline size_t cell(const ro_arena_view *a, uint32_t slot, uint32_t g) { return (size_t)slot * a->cap + g; }
static inline int bit(const uint32_t *bm, uint32_t g) { return (int)((bm[g / 32] >> (g % 32)) & 1u); }
static uint64_t max64(uint64_t x, uint64_t y) { return x > y ? x : y; }

/* Frame i: its header and Message; 0 when it is not a frame, names a group >= n_groups or is not a protobuf message. */
static int open_frame(const ro_arena_view *a, const uint8_t *bytes, const uint32_t *offsets, uint64_t n_bytes, size_t i, uint32_t *hdr,
                      wo_message *m) {
    const uint32_t lo = offsets[i], hi = offsets[i + 1];
    if (hi < lo || hi > n_bytes || hi - lo < 4) return 0;
    memcpy(hdr, bytes + lo, 4); /* little-endian host */
    return (*hdr >> 4) < a->n_groups && wo_decode_message(bytes + lo + 4, hi - lo - 4, m);
}

/* the low half of the pair g belongs to (g itself for a narrow group) */
static uint32_t low_half(const ro_arena_view *a, uint32_t g) { return (a->meta[g] & RO_META_WIDE_HI) ? g - 1 : g; }

/* committed as raftgpu_group_get reports it: the larger of a pair's halves */
static uint64_t pair_committed(const ro_arena_view *a, uint32_t lo) {
    return (a->meta[lo] & RO_META_WIDE_LO) ? max64(a->committed[lo], a->committed[lo + 1]) : a->committed[lo];
}

static uint32_t tally(const ro_arena_view *a, const uint8_t *votes, uint32_t lo) {
    uint32_t gr, rj;
    const int v = ro_arena_vote_result(a, votes, lo, &gr, &rj);
    return (uint32_t)v | gr << 8 | rj << 16;
}

void vwo_batch(ro_arena_view *a, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes,
               const uint32_t *select, const uint32_t *pre, uint8_t *status, vwo_outcome *out, uint64_t *n_out,
               uint64_t *tallied) {
    uint8_t *applied = (uint8_t *)calloc((size_t)RO_SLOTS * a->cap + 1, 1), *touched = (uint8_t *)calloc(a->cap + 1, 1);
    for (size_t i = 0; i < n; i++) {
        uint32_t hdr;
        wo_message m;
        status[i] = WO_WIRE_MALFORMED << 4;
        if (!open_frame(a, bytes, offsets, n_bytes, i, &hdr, &m)) continue;
        if (m.msg_type != 6 && m.msg_type != 18) { /* MsgRequestVoteResponse, MsgRequestPreVoteResponse */
            status[i] = WO_WIRE_SKIP_TYPE << 4;
            continue;
        }
        const uint32_t g = hdr >> 4, slot = hdr & 15u, lo = low_half(a, g);
        const int is_pre = pre && bit(pre, lo);
        uint32_t voters = RO_META_IN(a->meta[lo]) | RO_META_OUT(a->meta[lo]);
        if (a->meta[lo] & RO_META_WIDE_LO) voters |= RO_META_IN(a->meta[lo + 1]) | RO_META_OUT(a->meta[lo + 1]);
        /* a pair without voters (a freed slot, or not configured yet) is the host's */
        if (!bit(select, lo) || a->term_start[lo] != NO_TERM_START || !voters || is_pre != (m.msg_type == 18)) {
            status[i] = VWO_WIRE_ROLE << 4;
            continue;
        }
        const uint64_t term = a->term[lo];
        if (term == 0 || m.term == 0 || (is_pre ? (m.term < term || (m.reject && m.term > term)) : m.term != term)) {
            status[i] = WO_WIRE_TERM << 4;
            continue;
        }
        if (m.commit != 0 && m.commit_term != 0 && m.commit > pair_committed(a, lo)) {
            status[i] = VWO_WIRE_COMMIT_VOTE << 4;
            continue;
        }
        uint8_t res = 4; /* RAFTGPU_RES_NO_PROGRESS: no peer in that slot */
        if (slot < RO_SLOTS) {
            const size_t c = cell(a, slot, g);
            if (applied[c]) {
                status[i] = WO_WIRE_DUP << 4;
                continue;
            }
            applied[c] = 1;
            res = 0;
            if (!votes[c]) { /* tracker.rs:308-310 entry(id).or_insert(vote) */
                votes[c] = m.reject ? 1 : 2;
                res = 1;
            }
        }
        status[i] = (uint8_t)(WO_WIRE_OK << 4 | res);
        touched[lo] = 1;
    }
    uint64_t k = 0, t = 0;
    for (uint32_t g = 0; g < a->n_groups; g++) {
        if (!touched[g]) continue;
        t++;
        const uint32_t w = tally(a, votes, g);
        if ((w & 0xff) != RO_VOTE_PENDING) out[k++] = (vwo_outcome){g, w};
    }
    *n_out = k;
    *tallied = t;
    free(applied);
    free(touched);
}

/* ---- the literal form -------------------------------------------------------------------------------------------- */

static int32_t ctl(ro_arena_view *a, uint8_t *votes, uint32_t g, uint8_t op, uint8_t slot, uint16_t arg, uint64_t a0,
                   uint64_t a1, uint64_t a2, uint64_t a3) {
    const ro_ctl_cmd c = {g, op, slot, arg, {a0, a1, a2, a3}};
    ro_ctl_result r;
    ro_arena_control(a, votes, &c, 1, &r);
    return r.value;
}

/* Raft::reset's arena part with INTEGRATION.md section 6's arguments (raft.rs:942-971) */
static void reset(ro_arena_view *a, uint8_t *votes, uint32_t lo, uint64_t term_start) {
    const uint64_t last = a->last_index[lo];
    ctl(a, votes, lo, RO_CTL_RESET, 0, 0, term_start, last, pair_committed(a, lo), last);
}

/* become_follower(term, INVALID_ID) (raft.rs:1087-1096) */
static void become_follower(ro_arena_view *a, uint8_t *votes, uint8_t *role, uint32_t lo, uint64_t term) {
    reset(a, votes, lo, NO_TERM_START);
    if (a->term[lo] != term) ctl(a, votes, lo, RO_CTL_SET_TERM, 0, 0, term, 0, 0, 0);
    role[lo] = VWO_FOLLOWER;
}

/* become_leader (raft.rs:1162-1203): reset with term_start = the index of the empty entry it appends */
static void become_leader(ro_arena_view *a, uint8_t *votes, uint8_t *role, uint32_t lo) {
    reset(a, votes, lo, a->last_index[lo] + 1);
    ctl(a, votes, lo, RO_CTL_BECOME_LEADER, 0, 0, 0, 0, 0, 0);
    role[lo] = VWO_LEADER;
}

/* poll's transitions (raft.rs:2182-2199) for the tally word w */
static void transition(ro_arena_view *a, uint8_t *votes, uint8_t *role, uint32_t lo, uint32_t w);

/* campaign(CAMPAIGN_ELECTION) (raft.rs:1233-1278): become_candidate (term + 1, reset), then poll(self.id, true) */
static void campaign(ro_arena_view *a, uint8_t *votes, uint8_t *role, uint32_t lo) {
    const uint64_t term = a->term[lo] + 1;
    reset(a, votes, lo, NO_TERM_START);
    ctl(a, votes, lo, RO_CTL_SET_TERM, 0, 0, term, 0, 0, 0);
    role[lo] = VWO_CANDIDATE;
    uint32_t self = 0xff;
    if (a->meta[lo] & RO_META_HAS_SELF) self = RO_META_SELF(a->meta[lo]);
    else if ((a->meta[lo] & RO_META_WIDE_LO) && (a->meta[lo + 1] & RO_META_HAS_SELF)) self = 8 + RO_META_SELF(a->meta[lo + 1]);
    if (self != 0xff) ctl(a, votes, lo, RO_CTL_RECORD_VOTE, (uint8_t)self, 1, 0, 0, 0, 0);
    transition(a, votes, role, lo, tally(a, votes, lo));
}

static void transition(ro_arena_view *a, uint8_t *votes, uint8_t *role, uint32_t lo, uint32_t w) {
    if ((w & 0xff) == RO_VOTE_WON) {
        if (role[lo] == VWO_PRE_CANDIDATE) campaign(a, votes, role, lo);
        else become_leader(a, votes, role, lo);
    } else if ((w & 0xff) == RO_VOTE_LOST) {
        become_follower(a, votes, role, lo, a->term[lo]);
    }
}

void vwo_literal(ro_arena_view *a, uint8_t *votes, uint8_t *role, const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes,
                 uint32_t *first) {
    for (size_t i = 0; i < n; i++) {
        uint32_t hdr;
        wo_message m;
        if (!open_frame(a, bytes, offsets, n_bytes, i, &hdr, &m) || (m.msg_type != 6 && m.msg_type != 18)) continue;
        const uint32_t g = hdr >> 4, slot = hdr & 15u, lo = low_half(a, g);
        const uint64_t term = a->term[lo];
        /* Raft::step's term rules (raft.rs:1280-1349); m.term == 0 is a local message and goes on */
        if (m.term > term) {
            /* a granted pre-vote response keeps the term (:1319-1330); anything else steps down */
            if (!(m.msg_type == 18 && !m.reject)) {
                become_follower(a, votes, role, lo, m.term);
                continue; /* step_follower ignores vote responses */
            }
        } else if (m.term != 0 && m.term < term) {
            continue; /* a lower term: ignored (:1349-1411) */
        }
        /* step_candidate (raft.rs:2230-2243); the other roles ignore vote responses */
        if (role[lo] == VWO_PRE_CANDIDATE ? m.msg_type != 18 : (role[lo] != VWO_CANDIDATE || m.msg_type != 6)) continue;
        /* poll (raft.rs:2166-2201): record_vote, tally_votes, the transition */
        if (slot < RO_SLOTS && !votes[cell(a, slot, g)]) votes[cell(a, slot, g)] = m.reject ? 1 : 2;
        const uint32_t w = tally(a, votes, lo);
        if ((w & 0xff) != RO_VOTE_PENDING && first[lo] == 0xffffffffu) first[lo] = w;
        transition(a, votes, role, lo, w);
    }
}
