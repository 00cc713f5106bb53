/*
 * app_frames_oracle.h -- CPU ORACLE of the commit broadcast's entry-less MsgAppend frames. TEST INFRASTRUCTURE ONLY
 * (see raft_oracle.h).
 *
 * What it restates, one group at a time in group order: Raft::maybe_commit -> bcast_append (raft.rs:1745-1748,
 * 857-865: every Progress but self) -> send_append -> maybe_send_append(to, allow_empty = true) (raft.rs:764-819:
 * is_paused, progress.rs:210-216; pending_request_snapshot; raft_log.entries(next_idx), raft_log.rs:382-387;
 * raft_log.term(next_idx - 1), raft_log.rs:122-127) -> prepare_send_entries (raft.rs:714-730: msg_type MsgAppend,
 * index, log_term, commit; no update_state without entries) -> send (raft.rs:602-661: from = self.id, term =
 * self.term), and the canonical proto3 encoding of eraftpb.Message (eraftpb.proto:71-92).  The log is the arena's
 * range form (DESIGN.md 1): the term of an index in [term_start, last_index] is the group's term, above last_index
 * 0, and below term_start only the log knows it.  A send the log has to add to -- entries, a snapshot, or a term below
 * term_start -- goes to the rest list as the send list's entry; every other one is a frame of the wire batch format:
 * u32 LE (group << 4 | peer_slot), then the Message.
 *
 * Part of libraft_oracle.so (oracle/Makefile); oracle/app_frames_oracle.py declares its functions.
 */
#ifndef APP_FRAMES_ORACLE_H
#define APP_FRAMES_ORACLE_H

#include "read_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The serialized entry-less MsgAppend (eraftpb.Message, msg_type 3) with these fields.  Returns its length (at most
 * 68 bytes). */
size_t afo_encode_append(uint64_t to, uint64_t from, uint64_t term, uint64_t log_term, uint64_t index, uint64_t commit,
                         uint8_t *out);

/* bcast_append for every group of [first, first + n) whose bit is set in `select` (bit g = group g, words from group 0;
 * NULL = all) and that is allocated (g < a->n_groups, and q->allocated when q != NULL), a leader (term_start !=
 * UINT64_MAX) and has a term (a->term != 0; a leader without one sends nothing and is counted in totals[3]).
 * ids = u64 [RO_SLOTS + 1][n]: row s < 8 the id of the peer in slot s of group first + i, row 8 the group's own id.
 * A wide pair (RO_META_WIDE_LO / _HI) is one group: peer 8 + s is cell (g + 1, s); its selection bit, term, term_start
 * and id are the low half's, committed and last_index the larger of both halves'.  bytes [n * 8 * 72], offsets
 * [n * 8 + 1], rest [n * 8]; totals = {frames, bytes, rest entries, leaders without a term}. */
void afo_bcast_append(const ro_arena_view *a, const ro_read_queues *q, uint32_t first, uint32_t n, const uint32_t *select,
                      const uint64_t *ids, uint8_t *bytes, uint32_t *offsets, ro_send_entry *rest, uint64_t *totals);

#ifdef __cplusplus
}
#endif
#endif /* APP_FRAMES_ORACLE_H */
