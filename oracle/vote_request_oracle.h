/*
 * vote_request_oracle.h -- CPU ORACLE of vote requests at a voter. TEST INFRASTRUCTURE ONLY (see raft_oracle.h).
 *
 * Two forms over the arena view, its votes column and (nullable) its read queues, both decoding with hb_wire_oracle.c
 * (wire_oracle.c's fields -- 5, 6, 14 and 15 pinned by tests/golden/wire/vote_requests.json -- and the context, 12):
 *
 *  - the batch form restates what raftgpu_vote_request_wire does: the statuses in the order of include/raftgpu.h, one
 *    decided frame per group in frame order (IGNORED and COMMIT_VOTE claim the group too, later frames are DUP), the
 *    bump's SET_TERM + RESET through the control oracle, and the responses;
 *  - the literal form restates the reference one frame at a time, for every role: RawNode::step -> Raft::step's term
 *    rules (raft.rs:1280-1411: the lease, become_follower(m.term, INVALID_ID) through SET_TERM + RESET, the lower-term
 *    pre-vote rejection), then the vote arm (raft.rs:1418-1462: can_vote, is_up_to_date, the priority rule, the vote
 *    write, the response through send).  maybe_commit_by_vote is left out: it needs the log, and both forms leave it to
 *    the host.
 *
 * The caller's per-group table is vro_voter (== raftgpu_voter).  The literal form changes its vote and flags as the
 * reference changes vote, leader_id and the lease; it reads VRO_CHECK_QUORUM, an oracle-only flag bit, to recompute the
 * lease after a granted vote resets election_elapsed.
 *
 * Built together with the other oracle sources into libraft_oracle.so (oracle/vote_request_oracle.py).
 */
#ifndef VOTE_REQUEST_ORACLE_H
#define VOTE_REQUEST_ORACLE_H

#include "hb_wire_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* statuses beyond wire_oracle.h's (== RAFTGPU_WIRE_ROLE / _COMMIT_VOTE / _IGNORED) */
enum { VRO_WIRE_ROLE = 7, VRO_WIRE_COMMIT_VOTE = 9, VRO_WIRE_IGNORED = 10 };
/* the table's flags (== RAFTGPU_VOTER_*), the oracle's check_quorum bit, the applied frame's flags (== RAFTGPU_VREQ_*) */
enum { VRO_SELECT = 1, VRO_LEADER = 2, VRO_LEASE = 4, VRO_CHECK_QUORUM = 0x100 };
enum { VRO_GRANTED = 1, VRO_VOTED = 2, VRO_BUMPED = 4 };

typedef struct {
    uint64_t id, vote, last_term, commit_term, persisted, priority;
    uint32_t flags, reserved;
    uint64_t reserved2;
} vro_voter;

/* A vote response's Message bytes (no header): fields 1, 2, 3, 4, 8, 10, 15 in number order, zeros omitted. */
size_t vro_encode_response(uint32_t msg_type, uint64_t to, uint64_t from, uint64_t term, uint64_t commit, int reject,
                           uint64_t commit_term, uint8_t *out);

/* The batch form.  q (nullable): the arena's read queues, which a bump's reset clears.  status[i] = WO_WIRE_* /
 * VRO_WIRE_* << 4 | VRO_GRANTED.. of an applied frame; out[2 i..] = {m.from, the term after} of an applied frame, 0
 * otherwise; the responses (header + Message) back to back in resp (64 n bytes), resp_offsets [responses + 1],
 * totals = {responses, bytes}. */
void vro_batch(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
               size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp, uint32_t *resp_offsets,
               uint64_t *totals);

/* The literal form: every frame in order, as the reference steps it.  role[g] (0 Follower, 1 PreCandidate, 2 Candidate,
 * 3 Leader; the low half's for a pair), voters (vote, flags) and the arena change as the reference would change them;
 * the responses go to resp / resp_offsets / totals as in the batch form (resp: 64 n bytes). */
void vro_literal(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, uint8_t *role, vro_voter *voters,
                 const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes, uint8_t *resp, uint32_t *resp_offsets,
                 uint64_t *totals);

/* vro_batch's seconds on one core (the micro-benchmark's CPU reference). */
double vro_bench(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
                 size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp, uint32_t *resp_offsets,
                 uint64_t *totals);

#ifdef __cplusplus
}
#endif
#endif /* VOTE_REQUEST_ORACLE_H */
