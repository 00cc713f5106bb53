/*
 * hb_follow_oracle.h -- CPU ORACLE of MsgHeartbeat frames at the follower. TEST INFRASTRUCTURE ONLY (see raft_oracle.h).
 *
 * What it restates, one frame at a time in frame order, over the arena view: RawNode::step -> Raft::step's term rules
 * (raft.rs:1280-1411: a frame whose term is not the group's goes back to the host) -> step_follower (raft.rs:2276-2280)
 * -> handle_heartbeat (raft.rs:2452-2464): RaftLog::commit_to(m.commit) (raft_log.rs:286-300, through the control
 * oracle's COMMIT_TO, which also keeps a wide pair's halves equal), then one MsgHeartbeatResponse through send
 * (raft.rs:602-661: to = m.from, from = self.id, term = self.term, commit = raft_log.committed, context = m.context),
 * in the canonical proto3 encoding of hb_frames_oracle.c.  Role is the caller's: `select` marks the groups whose Raft
 * is a Follower without a pending request_snapshot.
 *
 * Built together with hb_frames_oracle.c, hb_wire_oracle.c, wire_oracle.c, read_oracle.c, control_oracle.c and
 * raft_oracle.c into its own library (oracle/hb_follow_oracle.py).
 */
#ifndef HB_FOLLOW_ORACLE_H
#define HB_FOLLOW_ORACLE_H

#include "hb_frames_oracle.h"
#include "hb_wire_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* statuses beyond hb_wire_oracle.h's (== RAFTGPU_WIRE_ROLE / RAFTGPU_WIRE_COMMIT_RANGE) */
enum { HFL_WIRE_ROLE = 7, HFL_WIRE_COMMIT_RANGE = 8 };

/* The serialized MsgHeartbeatResponse (eraftpb.Message, msg_type 9) with these fields and, when ctx != NULL, the
 * 8-byte context ctx[0..8).  Returns its length (at most 56 bytes). */
size_t hfl_encode_response(uint64_t to, uint64_t from, uint64_t term, uint64_t commit, const uint8_t *ctx, uint8_t *out);

/* The follower's side of every frame of a wire batch (u32 LE group << 4 | x, then the Message; `group` is the
 * follower's slot, x is copied into the response's header).  select: bitmap from group 0 (bit g = the caller's Raft
 * of group g is a Follower without a pending request_snapshot); self_ids[g] = group g's Raft::id; q (nullable): read
 * queues, whose `allocated` then decides which groups exist.  status[i] = WO_WIRE_* / HFL_WIRE_* << 4, | 1
 * (RAFTGPU_RES_OK) when a response was written; checks in this order: MALFORMED (frame, group >= n_groups or not
 * allocated, a wide pair's high half, protobuf), SKIP_TYPE (not 8), ROLE (select bit clear, or term_start !=
 * UINT64_MAX), TERM (a->term 0 or m.term != a->term), CONTEXT (present and not 8 bytes), COMMIT_RANGE (m.commit >
 * max(committed, last_index) over both halves of a wide pair), DUP (a group that already had a frame applied).
 * from[i] = m.from of an applied frame, 0 otherwise.  resp [60 n] / resp_offsets [n + 1]: the responses, in frame
 * order, framed with the input header; totals = {responses, bytes}. */
void hfl_follower_heartbeats(ro_arena_view *a, const ro_read_queues *q, const uint8_t *bytes, const uint32_t *offsets,
                             size_t n, uint64_t n_bytes, const uint32_t *select, const uint64_t *self_ids, uint8_t *status, uint64_t *from,
                             uint8_t *resp, uint32_t *resp_offsets, uint64_t *totals);

/* CPU baseline: the same pass over the same inputs, timed with CLOCK_MONOTONIC; returns seconds.  The arena view is
 * changed as hfl_follower_heartbeats changes it. */
double hfl_bench(ro_arena_view *a, const ro_read_queues *q, const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes,
                 const uint32_t *select, const uint64_t *self_ids, uint8_t *status, uint64_t *from, uint8_t *resp,
                 uint32_t *resp_offsets, uint64_t *totals);

#ifdef __cplusplus
}
#endif
#endif /* HB_FOLLOW_ORACLE_H */
