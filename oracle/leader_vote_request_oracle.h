/*
 * leader_vote_request_oracle.h -- CPU ORACLE of vote requests at a leader.  TEST INFRASTRUCTURE ONLY (see
 * raft_oracle.h).
 *
 * The batch form restates what raftgpu_leader_vote_request_wire does, over the arena view, its votes column, (nullable)
 * its read queues and the caller's voter table (vro_voter == raftgpu_voter), decoding with hb_wire_oracle.c: the
 * statuses in the order of include/raftgpu.h, each leader's frames in frame order against its unchanged state up to
 * its claimant (the first MsgRequestVote above the term that the lease does not drop, or a granted MsgRequestVote at
 * the term), the claimant's bump through the control oracle (SET_TERM + RESET), later frames DUP, and the responses.
 * The reference is vro_literal (vote_request_oracle.h), which steps leaders too.
 *
 * Built together with the other oracle sources into libraft_oracle.so (oracle/leader_vote_request_oracle.py).
 */
#ifndef LEADER_VOTE_REQUEST_ORACLE_H
#define LEADER_VOTE_REQUEST_ORACLE_H

#include "vote_request_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The batch form.  status[i] = WO_WIRE_* / VRO_WIRE_* << 4 | VRO_GRANTED.. of an OK frame; out[2 i..] = {m.from, the
 * term after} of an OK frame, 0 otherwise; the responses as vro_batch writes them (resp: 64 n bytes). */
void lvro_batch(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
                size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp,
                uint32_t *resp_offsets, uint64_t *totals);

/* lvro_batch's seconds on one core (the micro-benchmark's CPU reference). */
double lvro_bench(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const uint8_t *bytes, const uint32_t *offsets,
                  size_t n, uint64_t n_bytes, const vro_voter *voters, uint8_t *status, uint64_t *out, uint8_t *resp,
                  uint32_t *resp_offsets, uint64_t *totals);

#ifdef __cplusplus
}
#endif
#endif /* LEADER_VOTE_REQUEST_ORACLE_H */
