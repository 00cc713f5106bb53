/*
 * leader_term_oracle.h -- CPU ORACLE of the term prefix of the frames that reach a leader: MsgAppend (3),
 * MsgAppendResponse (4), MsgRequestVoteResponse (6), MsgHeartbeat (8), MsgHeartbeatResponse (9) and
 * MsgRequestPreVoteResponse (18).  TEST INFRASTRUCTURE ONLY (see raft_oracle.h).
 *
 * Two forms over the arena view, its votes column, (nullable) its read queues and the caller's voter table (vro_voter
 * == raftgpu_voter), decoding with wire_oracle.c and encoding replies as follow_term_oracle.c does:
 *
 *  - the literal form steps one frame at a time through Raft::step's term rules (raft.rs:1280-1411) and the drop arms
 *    of step_leader (:2111-2119) and step_follower, at a Leader or at the Follower a higher term made of it.  Types 3
 *    and 8 go through fto_literal, which handles them for every role, except at a leader at its own term, where
 *    step_leader drops them.  Types 4, 6, 9 and 18: a lower term is dropped; a higher one is become_follower(m.term,
 *    INVALID_ID) but for a granted pre-vote; then a Leader hands types 4 and 9 to their own passes (LTO_PASS) and drops
 *    the others, a Follower drops all four;
 *  - the batch form restates what raftgpu_leader_term_wire does: the statuses in the order of include/raftgpu.h, T
 *    per group over its passing frames, the lowest frame at T > term as the claimant, the verdict of every other frame
 *    from T and its own m.term, and the replies in frame order.
 *
 * Built together with the other oracle sources into libraft_oracle.so (oracle/leader_term_oracle.py).
 */
#ifndef LEADER_TERM_ORACLE_H
#define LEADER_TERM_ORACLE_H

#include "follow_term_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the status beyond the others (== RAFTGPU_WIRE_IGNORED) */
enum { LTO_WIRE_IGNORED = 10 };
/* the literal form's outcome per frame: FTO_NONE, FTO_PASS, FTO_ANSWERED, FTO_DROPPED (a lower term) and: */
enum { LTO_IGNORED = 4 }; /* the role's handler drops it */

/* The batch form.  q (nullable): the arena's read queues, which a bump's reset clears.  status[i] = WO_WIRE_* /
 * VRO_WIRE_ROLE / LTO_WIRE_IGNORED / FTO_WIRE_STALE << 4 | FTO_BUMPED or AFL_RES_OK; out[2 i..] = {leader_id, T} of a
 * claimant, 0 otherwise; the replies (header + Message) back to back in resp (39 n bytes), resp_offsets [replies + 1],
 * totals = {replies, bytes}. */
void lto_batch(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
               size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp,
               uint32_t *resp_offsets, uint64_t *totals);

/* The literal form: every frame in order, as the reference steps it at a Leader (role 3) or a Follower (role 0).
 * role[g], leader[g] (leader_id), voters (vote, flags) and the arena change as the reference would change them (a
 * pair's on its low half); outcome[i] = FTO_* or LTO_IGNORED (FTO_NONE for a frame that is not one of the six types,
 * not a frame, or a type 3 or 8 to a pair's high half); the replies go to resp / resp_offsets / totals as in the batch
 * form. */
void lto_literal(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, uint8_t *role, uint64_t *leader, vro_voter *voters,
                 const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes, uint8_t *outcome, uint8_t *resp,
                 uint32_t *resp_offsets, uint64_t *totals);

/* lto_batch's seconds on one core (the micro-benchmark's CPU reference). */
double lto_bench(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
                 size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp,
                 uint32_t *resp_offsets, uint64_t *totals);

#ifdef __cplusplus
}
#endif
#endif /* LEADER_TERM_ORACLE_H */
