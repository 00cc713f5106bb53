/* leader_vote_request_oracle.c -- see leader_vote_request_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#define _POSIX_C_SOURCE 199309L
#include "leader_vote_request_oracle.h"

#include <stdlib.h>
#include <string.h>
#include <time.h>

#define NO_TERM_START UINT64_MAX

static uint64_t max64(uint64_t x, uint64_t y) { return x > y ? x : y; }

/* last_index and committed as raftgpu_group_get reports them: the larger of a pair's halves */
static uint64_t pair_max(const ro_arena_view *a, const uint64_t *col, uint32_t g) {
    return (a->meta[g] & RO_META_WIDE_LO) ? max64(col[g], col[g + 1]) : col[g];
}

/* Frame i opened: its header, Message and whether the context is CAMPAIGN_TRANSFER (raft.rs:57, 1288); 0 when it is
 * not a frame, names a group >= n_groups or is not a protobuf message. */
static int open_frame(const ro_arena_view *a, const uint8_t *bytes, const uint32_t *offsets, uint64_t n_bytes, size_t i,
                      uint32_t *hdr, wo_message *m, int *force) {
    const uint32_t lo = offsets[i], hi = offsets[i + 1];
    if (hi < lo || hi > n_bytes || hi - lo < 4) return 0;
    memcpy(hdr, bytes + lo, 4); /* little-endian host */
    hwo_message h;
    if ((*hdr >> 4) >= a->n_groups || !hwo_decode_message(bytes + lo + 4, hi - lo - 4, &h)) return 0;
    *m = h.m;
    *force = h.ctx_len == 16 && memcmp(bytes + lo + 4 + h.ctx_off, "CampaignTransfer", 16) == 0;
    return 1;
}

static void ctl(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, uint32_t g, uint8_t op, uint64_t a0, uint64_t a1,
                uint64_t a2, uint64_t a3) {
    const ro_ctl_cmd c = {g, op, 0, 0, {a0, a1, a2, a3}};
    ro_ctl_result r;
    if (q) ro_read_control(a, q, votes, &c, 1, &r);
    else ro_arena_control(a, votes, &c, 1, &r);
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

void lvro_batch(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
                size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp,
                uint32_t *resp_offsets, uint64_t *totals) {
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
        if (!claimed[g] && a->term_start[g] == NO_TERM_START) { /* not a leader (a claimant's bump is not seen here) */
            status[i] = VRO_WIRE_ROLE << 4;
            continue;
        }
        const vro_voter *v = &voters[g];
        const uint64_t term = a->term[g];
        if (term == 0 || m.term == 0) {
            status[i] = WO_WIRE_TERM << 4;
            continue;
        }
        if (claimed[g]) { /* after the group's claimant: decided once its host side is done */
            status[i] = WO_WIRE_DUP << 4;
            continue;
        }
        const int pre = m.msg_type == 17;
        const uint32_t type = pre ? 18 : 6;
        if (m.term < term) {
            if (pre) { /* raft.rs:1395-1398 */
                respond(resp, resp_offsets, totals, hdr, type, m.from, v->id, term, 0, 1, 0);
                status[i] = WO_WIRE_OK << 4;
                out[2 * i] = m.from;
                out[2 * i + 1] = term;
            } else {
                status[i] = VRO_WIRE_IGNORED << 4; /* :1399-1409 */
            }
            continue;
        }
        if (m.term > term && (v->flags & VRO_LEASE) && !force) { /* :1288-1316 */
            status[i] = VRO_WIRE_IGNORED << 4;
            continue;
        }
        /* a MsgRequestVote above the term runs become_follower(m.term, INVALID_ID) first (:1346) */
        const int bumped = m.term > term && !pre;
        const uint64_t vote = bumped ? 0 : v->vote;
        const int leader = bumped ? 0 : (v->flags & VRO_LEADER) != 0;
        const uint64_t last = pair_max(a, a->last_index, g), committed = pair_max(a, a->committed, g);
        /* the vote arm (:1418-1462): can_vote, is_up_to_date, the priority rule */
        const int can_vote = vote == m.from || (vote == 0 && !leader) || (pre && m.term > term);
        const int grant = can_vote && (m.log_term > v->last_term || (m.log_term == v->last_term && m.index >= last)) &&
                          (m.index > last || v->priority <= m.priority);
        if (bumped || (grant && !pre)) claimed[g] = 1; /* the claimant: the only frame that changes state */
        /* maybe_commit_by_vote returns at once for a Leader (:2131), not for the Follower a bump makes */
        if (bumped && !grant && m.commit != 0 && m.commit_term != 0 && m.commit > committed) {
            status[i] = VRO_WIRE_COMMIT_VOTE << 4;
            continue;
        }
        if (bumped) {
            ctl(a, q, votes, g, RO_CTL_SET_TERM, m.term, 0, 0, 0);
            ctl(a, q, votes, g, RO_CTL_RESET, NO_TERM_START, last, committed, v->persisted);
        }
        if (grant) respond(resp, resp_offsets, totals, hdr, type, m.from, v->id, m.term, 0, 0, 0);
        else respond(resp, resp_offsets, totals, hdr, type, m.from, v->id, a->term[g], committed, 1, v->commit_term);
        status[i] = (uint8_t)(WO_WIRE_OK << 4 | (grant ? VRO_GRANTED : 0) | (grant && !pre ? VRO_VOTED : 0) |
                              (bumped ? VRO_BUMPED : 0));
        out[2 * i] = m.from;
        out[2 * i + 1] = a->term[g];
    }
    free(claimed);
}

double lvro_bench(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
                  size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp,
                  uint32_t *resp_offsets, uint64_t *totals) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    lvro_batch(a, q, votes, bytes, offsets, n, n_bytes, voters, status, out, resp, resp_offsets, totals);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}
