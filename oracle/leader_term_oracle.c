/* leader_term_oracle.c -- see leader_term_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#define _POSIX_C_SOURCE 199309L
#include "leader_term_oracle.h"

#include <stdlib.h>
#include <string.h>
#include <time.h>

#define NO_TERM_START UINT64_MAX

static uint64_t max64(uint64_t x, uint64_t y) { return x > y ? x : y; }

static int follow_type(uint32_t t) { return t == 3 || t == 8; } /* MsgAppend, MsgHeartbeat */
static int leader_type(uint32_t t) { return follow_type(t) || t == 4 || t == 6 || t == 9 || t == 18; }

/* Frame i opened: its header and Message; 0 when it is not a frame, names a group >= n_groups or is not a protobuf
 * message. */
static int open_frame(const ro_arena_view *a, const uint8_t *bytes, const uint32_t *offsets, uint64_t n_bytes, size_t i,
                      uint32_t *hdr, wo_message *m) {
    const uint32_t lo = offsets[i], hi = offsets[i + 1];
    if (hi < lo || hi > n_bytes || hi - lo < 4) return 0;
    memcpy(hdr, bytes + lo, 4); /* little-endian host */
    return (*hdr >> 4) < a->n_groups && wo_decode_message(bytes + lo + 4, hi - lo - 4, m);
}

static void ctl(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, uint32_t g, uint8_t op, uint64_t a0, uint64_t a1,
                uint64_t a2, uint64_t a3) {
    const ro_ctl_cmd c = {g, op, 0, 0, {a0, a1, a2, a3}};
    ro_ctl_result r;
    if (q) ro_read_control(a, q, votes, &c, 1, &r);
    else ro_arena_control(a, votes, &c, 1, &r);
}

static uint64_t pair_max(const ro_arena_view *a, const uint64_t *col, uint32_t g) {
    return (a->meta[g] & RO_META_WIDE_LO) ? max64(col[g], col[g + 1]) : col[g];
}

/* become_follower(term, ..)'s arena part (raft.rs:1087-1096): the term, then Raft::reset (raft.rs:942-971) */
static void bump(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, uint32_t g, uint64_t term, uint64_t persisted) {
    const uint64_t last = pair_max(a, a->last_index, g), committed = pair_max(a, a->committed, g);
    ctl(a, q, votes, g, RO_CTL_SET_TERM, term, 0, 0, 0);
    ctl(a, q, votes, g, RO_CTL_RESET, NO_TERM_START, last, committed, persisted);
}

/* the empty MsgAppendResponse of raft.rs:1375-1376 */
static void respond(uint8_t *resp, uint32_t *resp_offsets, uint64_t *totals, uint32_t hdr, uint64_t to, uint64_t from,
                    uint64_t term) {
    uint8_t *p = resp + totals[1];
    memcpy(p, &hdr, 4);
    const size_t k = 4 + afl_encode_response(to, from, term, 0, 0, 0, 0, 0, p + 4);
    resp_offsets[totals[0]++] = (uint32_t)totals[1];
    totals[1] += k;
    resp_offsets[totals[0]] = (uint32_t)totals[1];
}

void lto_batch(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
               size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp,
               uint32_t *resp_offsets, uint64_t *totals) {
    uint64_t *top = (uint64_t *)calloc(a->n_groups ? a->n_groups : 1, sizeof(uint64_t));
    uint64_t *mterm = (uint64_t *)calloc(n ? n : 1, sizeof(uint64_t)), *mfrom = (uint64_t *)calloc(n ? n : 1, sizeof(uint64_t));
    uint32_t *hdrs = (uint32_t *)calloc(n ? n : 1, sizeof(uint32_t)), *lows = (uint32_t *)calloc(n ? n : 1, sizeof(uint32_t));
    uint32_t *types = (uint32_t *)calloc(n ? n : 1, sizeof(uint32_t));
    uint8_t *at_term = (uint8_t *)calloc(n ? n : 1, 1), *claimed = (uint8_t *)calloc(a->n_groups ? a->n_groups : 1, 1);
    totals[0] = totals[1] = 0;
    resp_offsets[0] = 0;
    /* the checks in the order of raftgpu.h; T per group over the passing frames that can raise the term */
    for (size_t i = 0; i < n; i++) {
        uint32_t hdr;
        wo_message m;
        status[i] = WO_WIRE_MALFORMED << 4;
        out[2 * i] = out[2 * i + 1] = 0;
        if (!open_frame(a, bytes, offsets, n_bytes, i, &hdr, &m)) continue;
        const uint32_t g = hdr >> 4, high = (a->meta[g] & RO_META_WIDE_HI) != 0;
        if (follow_type(m.msg_type) && high) continue;
        if (!leader_type(m.msg_type)) {
            status[i] = WO_WIRE_SKIP_TYPE << 4;
            continue;
        }
        const uint32_t lo = high ? g - 1 : g;
        if (a->term_start[lo] == NO_TERM_START) {
            status[i] = VRO_WIRE_ROLE << 4;
            continue;
        }
        const uint64_t term = a->term[lo];
        if (term == 0 || m.term == 0) {
            status[i] = WO_WIRE_TERM << 4;
            continue;
        }
        if (m.msg_type == 18 && !m.reject) { /* raft.rs:1319-1320: never raises the term */
            status[i] = (m.term < term ? FTO_WIRE_STALE : LTO_WIRE_IGNORED) << 4;
            continue;
        }
        status[i] = WO_WIRE_OK << 4;
        hdrs[i] = hdr;
        lows[i] = lo;
        types[i] = m.msg_type;
        mterm[i] = m.term;
        mfrom[i] = follow_type(m.msg_type) ? m.from : 0;
        at_term[i] = m.term == term;
        top[lo] = max64(top[lo], max64(m.term, term));
    }
    /* the verdicts in frame order: the first frame at T > term bumps */
    for (size_t i = 0; i < n; i++) {
        if (status[i] != WO_WIRE_OK << 4) continue;
        const uint32_t g = lows[i];
        const uint64_t t = top[g];
        const int follow = follow_type(types[i]), own = types[i] == 4 || types[i] == 9;
        if (at_term[i]) {
            if (!own) status[i] = LTO_WIRE_IGNORED << 4;
        } else if (mterm[i] == t) {
            if (!claimed[g]) {
                claimed[g] = 1;
                bump(a, q, votes, g, t, voters[g].persisted);
                status[i] |= FTO_BUMPED;
                out[2 * i] = mfrom[i];
                out[2 * i + 1] = t;
            } else if (!follow) {
                status[i] = LTO_WIRE_IGNORED << 4;
            }
        } else if (follow && (voters[g].flags & FTO_STALE_REPLY)) {
            respond(resp, resp_offsets, totals, hdrs[i], mfrom[i], voters[g].id, t);
            status[i] = FTO_WIRE_STALE << 4 | AFL_RES_OK;
        } else {
            status[i] = FTO_WIRE_STALE << 4;
        }
    }
    free(top);
    free(mterm);
    free(mfrom);
    free(hdrs);
    free(lows);
    free(types);
    free(at_term);
    free(claimed);
}

void lto_literal(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, uint8_t *role, uint64_t *leader, vro_voter *voters,
                 const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes, uint8_t *outcome, uint8_t *resp,
                 uint32_t *resp_offsets, uint64_t *totals) {
    totals[0] = totals[1] = 0;
    resp_offsets[0] = 0;
    for (size_t i = 0; i < n; i++) {
        uint32_t hdr;
        wo_message m;
        outcome[i] = FTO_NONE;
        if (!open_frame(a, bytes, offsets, n_bytes, i, &hdr, &m) || !leader_type(m.msg_type)) continue;
        const uint32_t g = hdr >> 4, high = (a->meta[g] & RO_META_WIDE_HI) != 0;
        if (follow_type(m.msg_type)) {
            if (high) continue; /* the follower's own slot: a pair is addressed by its low half */
            if (role[g] == 3 && m.term != 0 && m.term == a->term[g]) {
                outcome[i] = LTO_IGNORED; /* step_leader's `_` arm */
                continue;
            }
            /* every other case is Raft::step's term prefix, then step_follower: fto_literal's */
            uint32_t ro[2];
            uint64_t tot[2];
            fto_literal(a, q, votes, role, leader, voters, bytes, offsets + i, 1, n_bytes, outcome + i, resp + totals[1], ro,
                        tot);
            if (tot[0]) {
                resp_offsets[totals[0]++] = (uint32_t)totals[1];
                totals[1] += tot[1];
                resp_offsets[totals[0]] = (uint32_t)totals[1];
            }
            continue;
        }
        const uint32_t lo = high ? g - 1 : g;
        vro_voter *v = &voters[lo];
        const uint64_t term = a->term[lo];
        if (m.term != 0 && m.term < term) { /* raft.rs:1399-1409: ignored */
            outcome[i] = FTO_DROPPED;
            continue;
        }
        if (m.term > term && !(m.msg_type == 18 && !m.reject)) { /* raft.rs:1319-1347: become_follower(m.term, INVALID_ID) */
            bump(a, q, votes, lo, m.term, v->persisted);
            role[lo] = 0;
            leader[lo] = 0;
            v->vote = 0;
            v->flags &= ~(uint32_t)(VRO_LEADER | VRO_LEASE);
        }
        /* step_leader handles the responses of its own passes and drops the vote responses; step_follower drops all */
        outcome[i] = (role[lo] == 3 && (m.msg_type == 4 || m.msg_type == 9)) ? FTO_PASS : LTO_IGNORED;
    }
}

double lto_bench(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
                 size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp,
                 uint32_t *resp_offsets, uint64_t *totals) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    lto_batch(a, q, votes, bytes, offsets, n, n_bytes, voters, status, out, resp, resp_offsets, totals);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}
