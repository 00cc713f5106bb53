/*
 * follow_term_oracle.h -- CPU ORACLE of the term prefix of MsgAppend / MsgHeartbeat frames at a follower. TEST
 * INFRASTRUCTURE ONLY (see raft_oracle.h).
 *
 * Two forms over the arena view, its votes column, (nullable) its read queues and the caller's voter table (vro_voter
 * == raftgpu_voter), both decoding with wire_oracle.c and encoding replies with app_follow_oracle.c's
 * afl_encode_response:
 *
 *  - the literal form restates Raft::step's term rules (raft.rs:1280-1376) one frame at a time, for every role:
 *    m.term 0 is a local message and goes on; a higher term is become_follower(m.term, m.from) -- the arena part through
 *    the control oracle's SET_TERM + RESET, the role, vote and leader in the caller's arrays; a lower one is answered
 *    with an empty MsgAppendResponse at the group's term when check_quorum || pre_vote (FTO_STALE_REPLY), dropped
 *    otherwise; the rest reaches the role's handler (FTO_PASS), which is not restated here;
 *  - the batch form restates what raftgpu_follower_term_wire does: the statuses in the order of include/raftgpu.h, T
 *    per group over its passing frames, the lowest frame at T > term as the claimant, the verdict of every other frame
 *    from T, and the replies in frame order.
 *
 * Built together with the other oracle sources into libraft_oracle.so (oracle/follow_term_oracle.py).
 */
#ifndef FOLLOW_TERM_ORACLE_H
#define FOLLOW_TERM_ORACLE_H

#include "app_follow_oracle.h"
#include "vote_request_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the status beyond the others (== RAFTGPU_WIRE_STALE), the table's flag (== RAFTGPU_VOTER_STALE_REPLY), the
 * claimant's low nibble (== RAFTGPU_FTERM_BUMPED) */
enum { FTO_WIRE_STALE = 11 };
enum { FTO_STALE_REPLY = 0x8 };
enum { FTO_BUMPED = 0x4 };
/* the literal form's outcome per frame */
enum { FTO_NONE = 0, FTO_PASS = 1, FTO_ANSWERED = 2, FTO_DROPPED = 3 };

/* The batch form.  q (nullable): the arena's read queues, which a bump's reset clears.  status[i] = WO_WIRE_* /
 * VRO_WIRE_ROLE / FTO_WIRE_STALE << 4 | FTO_BUMPED or AFL_RES_OK; out[2 i..] = {m.from, T} of a claimant, 0 otherwise;
 * the replies (header + Message) back to back in resp (39 n bytes), resp_offsets [replies + 1], totals = {replies,
 * bytes}. */
void fto_batch(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
               size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp,
               uint32_t *resp_offsets, uint64_t *totals);

/* The literal form: every frame in order, as the reference's term rules step it.  role[g] (0 Follower, 1 PreCandidate,
 * 2 Candidate, 3 Leader; the low half's for a pair), leader[g] (leader_id), voters (vote, flags) and the arena change
 * as the reference would change them; outcome[i] = FTO_*; the replies go to resp / resp_offsets / totals as in the
 * batch form. */
void fto_literal(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, uint8_t *role, uint64_t *leader, vro_voter *voters,
                 const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes, uint8_t *outcome, uint8_t *resp,
                 uint32_t *resp_offsets, uint64_t *totals);

/* fto_batch's seconds on one core (the micro-benchmark's CPU reference). */
double fto_bench(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
                 size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp,
                 uint32_t *resp_offsets, uint64_t *totals);

#ifdef __cplusplus
}
#endif
#endif /* FOLLOW_TERM_ORACLE_H */
