/* vote_request_oracle.c -- see vote_request_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#define _POSIX_C_SOURCE 199309L
#include "vote_request_oracle.h"

#include <stdlib.h>
#include <string.h>
#include <time.h>

#define NO_TERM_START UINT64_MAX

static uint64_t max64(uint64_t x, uint64_t y) { return x > y ? x : y; }

static uint8_t *put_varint(uint8_t *p, uint64_t v) {
    while (v >= 0x80) {
        *p++ = (uint8_t)(v | 0x80);
        v >>= 7;
    }
    *p++ = (uint8_t)v;
    return p;
}

size_t vro_encode_response(uint32_t msg_type, uint64_t to, uint64_t from, uint64_t term, uint64_t commit, int reject,
                           uint64_t commit_term, uint8_t *out) {
    const uint32_t field[7] = {1, 2, 3, 4, 8, 10, 15};
    const uint64_t val[7] = {msg_type, to, from, term, commit, reject ? 1u : 0u, commit_term};
    uint8_t *p = out;
    for (int k = 0; k < 7; k++) {
        if (!val[k]) continue; /* proto3: a zero scalar is not written */
        p = put_varint(p, (uint64_t)field[k] << 3);
        p = put_varint(p, val[k]);
    }
    return (size_t)(p - out);
}

/* m.context == CAMPAIGN_TRANSFER (raft.rs:57, 1288) */
static int transfer(const uint8_t *msg, uint32_t off, uint32_t len) {
    return len == 16 && memcmp(msg + off, "CampaignTransfer", 16) == 0;
}

/* Frame i opened: its header, Message and context; 0 when it is not a frame, names a group >= n_groups or is not a
 * protobuf message. */
static int open_frame(const ro_arena_view *a, const uint8_t *bytes, const uint32_t *offsets, uint64_t n_bytes, size_t i, uint32_t *hdr,
                      wo_message *m, int *force) {
    const uint32_t lo = offsets[i], hi = offsets[i + 1];
    if (hi < lo || hi > n_bytes || hi - lo < 4) return 0;
    memcpy(hdr, bytes + lo, 4); /* little-endian host */
    hwo_message h;
    if ((*hdr >> 4) >= a->n_groups || !hwo_decode_message(bytes + lo + 4, hi - lo - 4, &h)) return 0;
    *m = h.m;
    *force = transfer(bytes + lo + 4, h.ctx_off, h.ctx_len);
    return 1;
}

static void ctl(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, uint32_t g, uint8_t op, uint64_t a0, uint64_t a1,
                uint64_t a2, uint64_t a3) {
    const ro_ctl_cmd c = {g, op, 0, 0, {a0, a1, a2, a3}};
    ro_ctl_result r;
    if (q) ro_read_control(a, q, votes, &c, 1, &r);
    else ro_arena_control(a, votes, &c, 1, &r);
}

/* last_index and committed as raftgpu_group_get reports them: the larger of a pair's halves */
static uint64_t pair_max(const ro_arena_view *a, const uint64_t *col, uint32_t g) {
    return (a->meta[g] & RO_META_WIDE_LO) ? max64(col[g], col[g + 1]) : col[g];
}

/* become_follower(term, INVALID_ID)'s arena part (raft.rs:1087-1096): the term, then Raft::reset (raft.rs:942-971) */
static void bump(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, uint32_t g, uint64_t term, uint64_t persisted) {
    const uint64_t last = pair_max(a, a->last_index, g), committed = pair_max(a, a->committed, g);
    ctl(a, q, votes, g, RO_CTL_SET_TERM, term, 0, 0, 0);
    ctl(a, q, votes, g, RO_CTL_RESET, NO_TERM_START, last, committed, persisted);
}

/* The decision both forms share once the term rules have run (raft.rs:1420-1428): 1 grant, 0 reject. */
static int decide(const ro_arena_view *a, const vro_voter *v, uint32_t g, const wo_message *m, uint64_t term_before,
                  uint64_t vote, int leader) {
    const int pre = m->msg_type == 17;
    const uint64_t last = pair_max(a, a->last_index, g);
    const int can_vote = vote == m->from || (vote == 0 && !leader) || (pre && m->term > term_before);
    const int up_to_date = m->log_term > v->last_term || (m->log_term == v->last_term && m->index >= last);
    return can_vote && up_to_date && (m->index > last || v->priority <= m->priority);
}

static void respond(uint8_t *resp, uint32_t *resp_offsets, uint64_t *totals, uint32_t hdr, uint32_t type, uint64_t to,
                    uint64_t from, uint64_t term, uint64_t commit, int reject, uint64_t commit_term) {
    uint8_t *p = resp + totals[1];
    memcpy(p, &hdr, 4);
    const size_t k = 4 + vro_encode_response(type, to, from, term, commit, reject, commit_term, p + 4);
    resp_offsets[totals[0]++] = (uint32_t)totals[1];
    totals[1] += k;
    resp_offsets[totals[0]] = (uint32_t)totals[1];
}

void vro_batch(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
               size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp, uint32_t *resp_offsets,
               uint64_t *totals) {
    uint8_t *claimed = (uint8_t *)calloc(a->n_groups ? a->n_groups : 1, 1);
    totals[0] = totals[1] = 0;
    resp_offsets[0] = 0;
    for (size_t i = 0; i < n; i++) {
        uint32_t hdr;
        wo_message m;
        int force;
        status[i] = WO_WIRE_MALFORMED << 4;
        out[2 * i] = out[2 * i + 1] = 0;
        if (!open_frame(a, bytes, offsets, n_bytes, i, &hdr, &m, &force)) continue;
        const uint32_t g = hdr >> 4;
        if (a->meta[g] & RO_META_WIDE_HI) continue;
        if (m.msg_type != 5 && m.msg_type != 17) { /* MsgRequestVote, MsgRequestPreVote */
            status[i] = WO_WIRE_SKIP_TYPE << 4;
            continue;
        }
        const vro_voter *v = &voters[g];
        if (!(v->flags & VRO_SELECT) || a->term_start[g] != NO_TERM_START) {
            status[i] = VRO_WIRE_ROLE << 4;
            continue;
        }
        const uint64_t term = a->term[g];
        if (term == 0 || m.term == 0) {
            status[i] = WO_WIRE_TERM << 4;
            continue;
        }
        if (claimed[g]) { /* the group's decision waits for the next batch */
            status[i] = WO_WIRE_DUP << 4;
            continue;
        }
        claimed[g] = 1;
        const int pre = m.msg_type == 17;
        const uint32_t type = pre ? 18 : 6;
        if (m.term < term) {
            if (pre) { /* raft.rs:1395-1398 */
                respond(resp, resp_offsets, totals, hdr, type, m.from, v->id, term, 0, 1, 0);
                status[i] = WO_WIRE_OK << 4;
                out[2 * i] = m.from;
                out[2 * i + 1] = term;
            } else {
                status[i] = VRO_WIRE_IGNORED << 4;
            }
            continue;
        }
        if (m.term > term && (v->flags & VRO_LEASE) && !force) {
            status[i] = VRO_WIRE_IGNORED << 4;
            continue;
        }
        const int bumped = m.term > term && !pre;
        const int grant = decide(a, v, g, &m, term, bumped ? 0 : v->vote, bumped ? 0 : (v->flags & VRO_LEADER) != 0);
        if (!grant && m.commit != 0 && m.commit_term != 0 && m.commit > pair_max(a, a->committed, g)) {
            status[i] = VRO_WIRE_COMMIT_VOTE << 4;
            continue;
        }
        if (bumped) bump(a, q, votes, g, m.term, v->persisted);
        if (grant) respond(resp, resp_offsets, totals, hdr, type, m.from, v->id, m.term, 0, 0, 0);
        else respond(resp, resp_offsets, totals, hdr, type, m.from, v->id, a->term[g], pair_max(a, a->committed, g), 1,
                     v->commit_term);
        status[i] = (uint8_t)(WO_WIRE_OK << 4 | (grant ? VRO_GRANTED : 0) | (grant && !pre ? VRO_VOTED : 0) |
                              (bumped ? VRO_BUMPED : 0));
        out[2 * i] = m.from;
        out[2 * i + 1] = a->term[g];
    }
    free(claimed);
}

void vro_literal(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, uint8_t *role, vro_voter *voters,
                 const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes, uint8_t *resp, uint32_t *resp_offsets,
                 uint64_t *totals) {
    totals[0] = totals[1] = 0;
    resp_offsets[0] = 0;
    for (size_t i = 0; i < n; i++) {
        uint32_t hdr;
        wo_message m;
        int force;
        if (!open_frame(a, bytes, offsets, n_bytes, i, &hdr, &m, &force) || (m.msg_type != 5 && m.msg_type != 17)) continue;
        const uint32_t g = hdr >> 4;
        if (a->meta[g] & RO_META_WIDE_HI) continue; /* a pair is addressed by its low half */
        vro_voter *v = &voters[g];
        const int pre = m.msg_type == 17;
        const uint32_t type = pre ? 18 : 6;
        const uint64_t term = a->term[g];
        /* Raft::step's term rules (raft.rs:1280-1411); m.term == 0 is a local message and goes on */
        if (m.term > term) {
            if (!force && (v->flags & VRO_LEASE)) continue; /* :1288-1316 */
            if (!pre) {                                     /* :1346 become_follower(m.term, INVALID_ID) */
                bump(a, q, votes, g, m.term, v->persisted);
                v->vote = 0;
                v->flags &= ~(uint32_t)(VRO_LEADER | VRO_LEASE);
                role[g] = 0;
            }
        } else if (m.term != 0 && m.term < term) {
            if (pre) respond(resp, resp_offsets, totals, hdr, type, m.from, v->id, term, 0, 1, 0); /* :1377-1398 */
            continue;
        }
        /* the vote arm (raft.rs:1418-1462); maybe_commit_by_vote is the host's */
        if (decide(a, v, g, &m, term, v->vote, (v->flags & VRO_LEADER) != 0)) {
            respond(resp, resp_offsets, totals, hdr, type, m.from, v->id, m.term, 0, 0, 0);
            if (!pre) { /* :1445-1449 election_elapsed = 0, vote = m.from */
                v->vote = m.from;
                if ((v->flags & VRO_LEADER) && (v->flags & VRO_CHECK_QUORUM)) v->flags |= VRO_LEASE;
            }
        } else {
            respond(resp, resp_offsets, totals, hdr, type, m.from, v->id, a->term[g], pair_max(a, a->committed, g), 1,
                    v->commit_term);
        }
    }
}

double vro_bench(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
                 size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp, uint32_t *resp_offsets,
                 uint64_t *totals) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    vro_batch(a, q, votes, bytes, offsets, n, n_bytes, voters, status, out, resp, resp_offsets, totals);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}
