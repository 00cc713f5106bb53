/*
 * follow_resp_oracle.h -- CPU ORACLE of the term prefix of the responses that reach a Follower, PreCandidate or
 * Candidate -- MsgAppendResponse (4), MsgRequestVoteResponse (6), MsgHeartbeatResponse (9) and
 * MsgRequestPreVoteResponse (18) -- and of step_candidate's step-down at the candidate's own term.  TEST
 * INFRASTRUCTURE ONLY (see raft_oracle.h).
 *
 * Two forms over the arena view, its votes column, (nullable) its read queues and the caller's voter table (vro_voter
 * == raftgpu_voter), decoding with wire_oracle.c:
 *
 *  - the literal form steps one frame at a time through Raft::step at a non-leader: for types 4, 6, 9 and 18 the
 *    term rules (raft.rs:1280-1411: a lower term is dropped, a higher one is become_follower(m.term, INVALID_ID) but
 *    for a granted pre-vote), then step_candidate's vote arm (:2230-2243: a Candidate's MsgRequestVoteResponse and a
 *    PreCandidate's MsgRequestPreVoteResponse reach poll, FTO_PASS) or the drop arms of step_follower and
 *    step_candidate (LTO_IGNORED).  For types 3 and 8 step_candidate's MsgAppend / MsgHeartbeat arms at the term
 *    (:2215-2224: become_follower(term, m.from), then the follower's handler, FTO_PASS), and fto_literal otherwise;
 *  - the batch form restates what raftgpu_follower_response_wire does: the statuses in the order of
 *    include/raftgpu.h, T per group over its passing frames (a granted pre-vote left out), the lowest frame at
 *    T > term as the claimant, and the verdict of every other frame from T, its m.term and the group's candidacy;
 *  - the step-down's batch form restates raftgpu_follower_term_wire for rows with FRP_CANDIDATE: fto_batch, then the
 *    lowest frame at a flagged group's unchanged term as the step-down's claimant.
 *
 * Built together with the other oracle sources into libraft_oracle.so (oracle/follow_resp_oracle.py).
 */
#ifndef FOLLOW_RESP_ORACLE_H
#define FOLLOW_RESP_ORACLE_H

#include "leader_term_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the table's candidate flags (== RAFTGPU_VOTER_CANDIDATE, RAFTGPU_VOTER_PRE_CANDIDATE) and the step-down's low nibble
 * (== RAFTGPU_FTERM_STEPPED) */
enum { FRP_CANDIDATE = 0x10, FRP_PRE_CANDIDATE = 0x20 };
enum { FRP_STEPPED = 0x8 };

/* The batch form.  q (nullable): the arena's read queues, which a bump's reset clears.  status[i] = WO_WIRE_* /
 * VRO_WIRE_ROLE / LTO_WIRE_IGNORED / FTO_WIRE_STALE << 4 | FTO_BUMPED; out[i] = T of a claimant, 0 otherwise. */
void frp_batch(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
               size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out);

/* The literal form: every frame in order, as the reference steps it at a Follower (role 0), PreCandidate (1) or
 * Candidate (2).  role[g], leader[g] (leader_id), voters (vote, flags: a group that becomes a Follower loses
 * FRP_CANDIDATE and FRP_PRE_CANDIDATE) and the arena change as the reference would change them (a pair's on its low
 * half); outcome[i] = FTO_* or LTO_IGNORED (FTO_NONE for a frame that is not one of the six types, not a frame, a type
 * 3 or 8 to a pair's high half, or a frame to a Leader); the replies of fto_literal's stale frames go to resp /
 * resp_offsets / totals as in fto_batch. */
void frp_literal(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, uint8_t *role, uint64_t *leader, vro_voter *voters,
                 const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes, uint8_t *outcome, uint8_t *resp,
                 uint32_t *resp_offsets, uint64_t *totals);

/* The batch form of raftgpu_follower_term_wire with the step-down: fto_batch, then, for every group whose row has
 * FRP_CANDIDATE and whose term fto_batch did not raise, the lowest frame left OK (m.term == T == term) claims it:
 * become_follower(term, m.from)'s arena part (the reset alone), status | FRP_STEPPED, out[2 i..] = {m.from, term}.
 * Arguments and outputs as fto_batch's. */
void frp_term_batch(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
                    size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp,
                    uint32_t *resp_offsets, uint64_t *totals);

/* frp_batch's seconds on one core (the micro-benchmark's CPU reference). */
double frp_bench(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
                 size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out);

#ifdef __cplusplus
}
#endif
#endif /* FOLLOW_RESP_ORACLE_H */
