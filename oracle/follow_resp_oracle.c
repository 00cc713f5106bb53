/* follow_resp_oracle.c -- see follow_resp_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#define _POSIX_C_SOURCE 199309L
#include "follow_resp_oracle.h"

#include <stdlib.h>
#include <string.h>
#include <time.h>

#define NO_TERM_START UINT64_MAX

static uint64_t max64(uint64_t x, uint64_t y) { return x > y ? x : y; }

static int resp_type(uint32_t t) { return t == 4 || t == 6 || t == 9 || t == 18; }

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

/* become_follower(term, ..)'s arena part (raft.rs:1087-1096): the term (a no-op at the group's own), then Raft::reset
 * (raft.rs:942-971) */
static void bump(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, uint32_t g, uint64_t term, uint64_t persisted) {
    const uint64_t last = pair_max(a, a->last_index, g), committed = pair_max(a, a->committed, g);
    ctl(a, q, votes, g, RO_CTL_SET_TERM, term, 0, 0, 0);
    ctl(a, q, votes, g, RO_CTL_RESET, NO_TERM_START, last, committed, persisted);
}

/* does the frame belong to the candidacy of a group with these flags (step_candidate, raft.rs:2230-2240)? */
static int own(uint32_t flags, uint32_t t) {
    const int pre = (flags & FRP_PRE_CANDIDATE) != 0;
    return (flags & FRP_CANDIDATE) && (t == 18 ? pre : (t == 6 && !pre));
}

void frp_batch(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
               size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out) {
    uint64_t *top = (uint64_t *)calloc(a->n_groups ? a->n_groups : 1, sizeof(uint64_t));
    uint64_t *mterm = (uint64_t *)calloc(n ? n : 1, sizeof(uint64_t)), *gterm = (uint64_t *)calloc(n ? n : 1, sizeof(uint64_t));
    uint32_t *lows = (uint32_t *)calloc(n ? n : 1, sizeof(uint32_t));
    uint8_t *mine = (uint8_t *)calloc(n ? n : 1, 1), *grant = (uint8_t *)calloc(n ? n : 1, 1);
    uint8_t *claimed = (uint8_t *)calloc(a->n_groups ? a->n_groups : 1, 1);
    /* the checks in the order of raftgpu.h; T per group over the passing frames that can raise the term */
    for (size_t i = 0; i < n; i++) {
        uint32_t hdr;
        wo_message m;
        status[i] = WO_WIRE_MALFORMED << 4;
        out[i] = 0;
        if (!open_frame(a, bytes, offsets, n_bytes, i, &hdr, &m)) continue;
        if (!resp_type(m.msg_type)) {
            status[i] = WO_WIRE_SKIP_TYPE << 4;
            continue;
        }
        const uint32_t g = hdr >> 4, lo = (a->meta[g] & RO_META_WIDE_HI) ? g - 1 : g;
        if (!(voters[lo].flags & VRO_SELECT) || a->term_start[lo] != NO_TERM_START) {
            status[i] = VRO_WIRE_ROLE << 4;
            continue;
        }
        const uint64_t term = a->term[lo];
        if (term == 0 || m.term == 0) {
            status[i] = WO_WIRE_TERM << 4;
            continue;
        }
        status[i] = WO_WIRE_OK << 4;
        lows[i] = lo;
        mterm[i] = m.term;
        gterm[i] = term;
        grant[i] = m.msg_type == 18 && !m.reject; /* raft.rs:1319-1320: never raises the term */
        mine[i] = (uint8_t)own(voters[lo].flags, m.msg_type);
        top[lo] = max64(top[lo], grant[i] ? term : max64(m.term, term));
    }
    /* the verdicts in frame order: the first frame at T > term bumps */
    for (size_t i = 0; i < n; i++) {
        if (status[i] != WO_WIRE_OK << 4) continue;
        const uint32_t g = lows[i];
        const uint64_t t = top[g];
        if (!grant[i] && mterm[i] == t && t > gterm[i] && !claimed[g]) {
            claimed[g] = 1;
            bump(a, q, votes, g, t, voters[g].persisted);
            status[i] |= FTO_BUMPED;
            out[i] = t;
        } else if (mterm[i] < t) {
            status[i] = FTO_WIRE_STALE << 4;
        } else if (t > gterm[i] || !mine[i]) {
            status[i] = LTO_WIRE_IGNORED << 4;
        }
    }
    free(top);
    free(mterm);
    free(gterm);
    free(lows);
    free(mine);
    free(grant);
    free(claimed);
}

/* become_follower's host side as the caller keeps it in the table: no candidacy, leader_id = leader */
static void follower_row(vro_voter *v, uint64_t leader) {
    v->flags &= ~(uint32_t)(VRO_LEADER | VRO_LEASE | FRP_CANDIDATE | FRP_PRE_CANDIDATE);
    if (leader) v->flags |= VRO_LEADER;
}

void frp_literal(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, uint8_t *role, uint64_t *leader, vro_voter *voters,
                 const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes, uint8_t *outcome, uint8_t *resp,
                 uint32_t *resp_offsets, uint64_t *totals) {
    totals[0] = totals[1] = 0;
    resp_offsets[0] = 0;
    for (size_t i = 0; i < n; i++) {
        uint32_t hdr;
        wo_message m;
        outcome[i] = FTO_NONE;
        if (!open_frame(a, bytes, offsets, n_bytes, i, &hdr, &m)) continue;
        const uint32_t g = hdr >> 4, t = m.msg_type, high = (a->meta[g] & RO_META_WIDE_HI) != 0;
        if (t == 3 || t == 8) {
            if (high || role[g] == 3) continue; /* a pair is addressed by its low half; a Leader's is lto_literal's */
            if ((role[g] == 1 || role[g] == 2) && m.term != 0 && m.term == a->term[g]) {
                /* step_candidate (raft.rs:2215-2224): become_follower(term, m.from) -- the vote stays, the term is
                 * the same -- then the follower's handler */
                bump(a, q, votes, g, m.term, voters[g].persisted);
                role[g] = 0;
                leader[g] = m.from;
                follower_row(&voters[g], m.from);
                outcome[i] = FTO_PASS;
                continue;
            }
            uint32_t ro[2];
            uint64_t tot[2];
            fto_literal(a, q, votes, role, leader, voters, bytes, offsets + i, 1, n_bytes, outcome + i, resp + totals[1], ro,
                        tot);
            if (tot[0]) {
                resp_offsets[totals[0]++] = (uint32_t)totals[1];
                totals[1] += tot[1];
                resp_offsets[totals[0]] = (uint32_t)totals[1];
            }
            if (role[g] == 0) voters[g].flags &= ~(uint32_t)(FRP_CANDIDATE | FRP_PRE_CANDIDATE);
            continue;
        }
        if (!resp_type(t)) continue;
        const uint32_t lo = high ? g - 1 : g;
        if (role[lo] == 3) continue;
        vro_voter *v = &voters[lo];
        const uint64_t term = a->term[lo];
        if (m.term != 0 && m.term < term) { /* raft.rs:1399-1409: ignored */
            outcome[i] = FTO_DROPPED;
            continue;
        }
        if (m.term > term && !(t == 18 && !m.reject)) { /* raft.rs:1319-1347: become_follower(m.term, INVALID_ID) */
            bump(a, q, votes, lo, m.term, v->persisted);
            role[lo] = 0;
            leader[lo] = 0;
            v->vote = 0;
            follower_row(v, 0);
        }
        /* step_candidate polls its own candidacy's responses; it and step_follower drop everything else */
        outcome[i] = ((role[lo] == 1 && t == 18) || (role[lo] == 2 && t == 6)) ? FTO_PASS : LTO_IGNORED;
    }
}

void frp_term_batch(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
                    size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp,
                    uint32_t *resp_offsets, uint64_t *totals) {
    uint64_t *term0 = (uint64_t *)malloc((a->n_groups ? a->n_groups : 1) * sizeof(uint64_t));
    uint8_t *claimed = (uint8_t *)calloc(a->n_groups ? a->n_groups : 1, 1);
    memcpy(term0, a->term, a->n_groups * sizeof(uint64_t));
    fto_batch(a, q, votes, bytes, offsets, n, n_bytes, voters, status, out, resp, resp_offsets, totals);
    /* a frame left OK with no low nibble is at T; T is the term where fto_batch raised nothing */
    for (size_t i = 0; i < n; i++) {
        uint32_t hdr;
        wo_message m;
        if (status[i] != WO_WIRE_OK << 4 || !open_frame(a, bytes, offsets, n_bytes, i, &hdr, &m)) continue;
        const uint32_t g = hdr >> 4;
        if (!(voters[g].flags & FRP_CANDIDATE) || a->term[g] != term0[g] || claimed[g]) continue;
        claimed[g] = 1;
        bump(a, q, votes, g, m.term, voters[g].persisted); /* m.term == term: the reset alone */
        status[i] |= FRP_STEPPED;
        out[2 * i] = m.from;
        out[2 * i + 1] = m.term;
    }
    free(term0);
    free(claimed);
}

double frp_bench(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
                 size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    frp_batch(a, q, votes, bytes, offsets, n, n_bytes, voters, status, out);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}
