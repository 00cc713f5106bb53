/*
 * hb_frames_oracle.h -- CPU ORACLE of MsgHeartbeat frames to the wire. TEST INFRASTRUCTURE ONLY (see raft_oracle.h).
 *
 * What it restates, one group at a time in group order: Raft::ping / MsgBeat -> bcast_heartbeat (raft.rs:868-878;
 * leaders only, the context = ReadOnly::last_pending_request_ctx, read_only.rs:132-135) -> bcast_heartbeat_with_ctx
 * (raft.rs:881-889: every Progress but self) -> send_heartbeat (raft.rs:822-844: msg_type MsgHeartbeat, to, commit =
 * min(pr.matched, raft_log.committed), the context when there is one) -> send (raft.rs:602-661: from = self.id,
 * term = self.term), and the canonical proto3 encoding of eraftpb.Message (eraftpb.proto:71-92).  Each message goes
 * out as a frame of the wire batch format: u32 LE (group << 4 | peer_slot), then the Message.  A read id x travels as
 * the 8 little-endian bytes of x (DESIGN.md 3.10); id 0 is no context.
 *
 * Built together with read_oracle.c, control_oracle.c and raft_oracle.c into its own library
 * (oracle/hb_frames_oracle.py).
 */
#ifndef HB_FRAMES_ORACLE_H
#define HB_FRAMES_ORACLE_H

#include "read_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The serialized MsgHeartbeat (eraftpb.Message, msg_type 8) with these fields; ctx 0 = no context.  Returns its
 * length (at most 56 bytes). */
size_t hfo_encode_heartbeat(uint64_t to, uint64_t from, uint64_t term, uint64_t commit, uint64_t ctx, uint8_t *out);

/* bcast_heartbeat for every group of [first, first + n) whose bit is set in `select` (bit g = group g, words from group
 * 0; NULL = all) and that is allocated (g < a->n_groups, and q->allocated when q != NULL), a leader (term_start !=
 * UINT64_MAX) and has a term (a->term != 0; a leader without one sends nothing and is counted in totals[2]).
 * ids = u64 [RO_SLOTS + 1][n]: row s < 8 the id of the peer in slot s of group first + i, row 8 the group's own id.
 * A wide pair (RO_META_WIDE_LO / _HI) is one group: peer 8 + s is cell (g + 1, s); its selection bit, term,
 * term_start, id and read queue are the low half's, committed is the larger of both halves'.  q == NULL: no read
 * queues, no context.  bytes [n * 8 * 60], offsets [n * 8 + 1]; totals = {frames, bytes, leaders without a term}. */
void hfo_bcast_heartbeats(const ro_arena_view *a, const ro_read_queues *q, uint32_t first, uint32_t n, const uint32_t *select,
                          const uint64_t *ids, uint8_t *bytes, uint32_t *offsets, uint64_t *totals);

#ifdef __cplusplus
}
#endif
#endif /* HB_FRAMES_ORACLE_H */
