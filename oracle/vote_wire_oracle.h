/*
 * vote_wire_oracle.h -- CPU ORACLE of vote responses at a candidate. TEST INFRASTRUCTURE ONLY (see raft_oracle.h).
 *
 * Two forms over the arena view and its votes column ([RO_SLOTS][cap], 0 missing / 1 no / 2 yes), both decoding with
 * wire_oracle.c (whose decoder messages.json pins on types 6 and 18 and on commit_term):
 *
 *  - the batch form restates what raftgpu_vote_wire does: the statuses in the order of include/raftgpu.h, the or_insert
 *    vote of the first passing frame of every (group, peer) cell (a pair without voters is ROLE), and one tally per
 *    touched group (pair) after the batch, listed when it is Won or Lost;
 *  - the literal form restates the reference one frame at a time, transitions included: RawNode::step -> Raft::step's
 *    term rules for types 6 and 18 (raft.rs:1280-1349) -> step_candidate (raft.rs:2230-2243) -> poll (raft.rs:2166-2201)
 *    with become_leader, become_follower and, for a PreCandidate that won, campaign(CAMPAIGN_ELECTION) (term + 1,
 *    reset, the self vote and its poll).  The arena part of each transition runs through the control oracle with
 *    INTEGRATION.md section 6's RESET arguments: persisted = last_index, term_start = last_index + 1 for a leader and
 *    UINT64_MAX otherwise.  maybe_commit_by_vote is not restated: it needs the log, and a frame that would reach it
 *    (m.commit > committed with commit_term != 0) is the host's in both forms.
 *
 * Built together with the other oracle sources into libraft_oracle.so (oracle/vote_wire_oracle.py).
 */
#ifndef VOTE_WIRE_ORACLE_H
#define VOTE_WIRE_ORACLE_H

#include "control_oracle.h"
#include "wire_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* statuses beyond wire_oracle.h's (== RAFTGPU_WIRE_ROLE / RAFTGPU_WIRE_COMMIT_VOTE) */
enum { VWO_WIRE_ROLE = 7, VWO_WIRE_COMMIT_VOTE = 9 };
/* the literal form's roles (raft.rs StateRole) */
enum { VWO_FOLLOWER = 0, VWO_PRE_CANDIDATE = 1, VWO_CANDIDATE = 2, VWO_LEADER = 3 };

/* raftgpu_vote_outcome: the group (a pair's low half) and VoteResult | granted << 8 | rejected << 16 */
typedef struct {
    uint32_t group;
    uint32_t result;
} vwo_outcome;

/* The batch form.  select / pre: bitmaps from group 0 (pre nullable); status[i] = WO_WIRE_* / VWO_WIRE_* << 4 | the
 * applied frame's result (1 recorded, 0 the cell had a vote, 4 a slot >= 8); out (room for min(n, n_groups)) gets the
 * decided groups in ascending order, *n_out how many, *tallied the touched groups. */
void vwo_batch(ro_arena_view *a, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes,
               const uint32_t *select, const uint32_t *pre, uint8_t *status, vwo_outcome *out, uint64_t *n_out,
               uint64_t *tallied);

/* The literal form.  role[g] (VWO_*, the low half's for a pair) and the arena (a->term included) change as the reference
 * would change them.  first[g] = the first Won or Lost word poll returned for group g in this batch, left alone where
 * none did (the caller fills it with 0xffffffff). */
void vwo_literal(ro_arena_view *a, uint8_t *votes, uint8_t *role, const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes,
                 uint32_t *first);

#ifdef __cplusplus
}
#endif
#endif /* VOTE_WIRE_ORACLE_H */
