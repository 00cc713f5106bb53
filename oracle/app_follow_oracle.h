/*
 * app_follow_oracle.h -- CPU ORACLE of MsgAppend frames at the follower. TEST INFRASTRUCTURE ONLY (see raft_oracle.h).
 *
 * Two forms, both decoding with wire_oracle.c (fields 3, 5 and 6 included) plus a walk of the entries (field 7, each
 * an eraftpb.Entry whose term is field 2 and index field 3, eraftpb.proto:16-21):
 *
 *  - the literal form restates the reference one frame at a time over each group's literal term array: RawNode::step ->
 *    Raft::step's term rules (raft.rs:1280-1411: m.term 0 is local, a higher term is become_follower, a lower one is
 *    answered at :1349-1376 when check_quorum or pre_vote is on) -> step_follower (raft.rs:2271-2275) ->
 *    handle_append_entries (raft.rs:2389-2448) with RaftLog::term (raft_log.rs:122-140, no compaction: the dummy entry
 *    is index 0), maybe_append (:241-279, entries appended literally), find_conflict_by_term (:209-239) and commit_to
 *    (:286-300).  No arena: it keeps its own term, committed and log per group;
 *  - the batch form restates what raftgpu_follower_append does over the arena view and the caller's run table: the
 *    statuses in the order of include/raftgpu.h, one decided frame per group in frame order (NEEDS_LOG and
 *    COMMIT_RANGE claim the group too, later frames are DUP), commit_to through the control oracle's COMMIT_TO (which
 *    also keeps a wide pair's halves equal), and the responses.
 *
 * Built together with the other oracle sources into libraft_oracle.so (oracle/app_follow_oracle.py).
 */
#ifndef APP_FOLLOW_ORACLE_H
#define APP_FOLLOW_ORACLE_H

#include "hb_wire_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* statuses beyond wire_oracle.h's (== RAFTGPU_WIRE_ROLE / RAFTGPU_WIRE_COMMIT_RANGE) */
enum { AFL_WIRE_ROLE = 7, AFL_WIRE_COMMIT_RANGE = 8 };
/* the run table's flag (== RAFTGPU_FOLLOWER_SELECT) and an applied frame's low nibble (== RAFTGPU_RES_OK,
 * RAFTGPU_FAPP_REJECT, RAFTGPU_FAPP_STALE) */
enum { AFL_SELECT = 1 };
enum { AFL_RES_OK = 1, AFL_REJECT = 2, AFL_STALE = 4 };

/* == raftgpu_follower_log */
typedef struct {
    uint64_t id, run_start, run_term;
    uint32_t flags, reserved;
} afl_log;

/* The literal form's group: its Raft's id, term and committed, and its log terms[0 .. last_index] (terms[0] is the
 * dummy entry's).  flags: AFL_G_FOLLOWER (a Follower without pending_request_snapshot: other roles are not stepped
 * here), AFL_G_LOWER_REPLY (check_quorum || pre_vote). */
enum { AFL_G_FOLLOWER = 1, AFL_G_LOWER_REPLY = 2 };
typedef struct {
    uint64_t id, term, committed, last_index;
    uint32_t flags, reserved;
} afl_group;
/* the literal form's outcome per frame */
enum { AFL_NONE = 0, AFL_ANSWERED = 1, AFL_DROPPED = 2, AFL_FATAL = 3 };

/* A MsgAppendResponse's Message bytes (no header): fields 1 (4), 2, 3, 4, 5, 6, 8, 10, 11 in number order, zeros
 * omitted.  At most 81 bytes. */
size_t afl_encode_response(uint64_t to, uint64_t from, uint64_t term, uint64_t log_term, uint64_t index, uint64_t commit,
                           int reject, uint64_t reject_hint, uint8_t *out);

/* 1 when the bytes are a well-formed protobuf message (wo_decode_message's verdict); *n_fields7 = the field-7 occurrences
 * in any wire type; the first max_ents length-delimited ones' Entry term / index go to ent_term / ent_index. */
int afl_decode(const uint8_t *buf, size_t len, wo_message *m, size_t *n_fields7, uint64_t *ent_term, uint64_t *ent_index,
               size_t max_ents);

/* The batch form.  q (nullable): the arena's read queues, whose `allocated` then decides which groups exist.
 * status[i] = WO_WIRE_* / AFL_WIRE_* << 4 | AFL_RES_OK.. of an applied frame; from[i] = m.from of an applied frame, 0
 * otherwise; the responses (header + Message) back to back in resp (85 n bytes), resp_offsets [responses + 1],
 * totals = {responses, bytes}. */
void afl_batch(ro_arena_view *a, const ro_read_queues *q, const afl_log *logs, const uint8_t *bytes, const uint32_t *offsets,
               size_t n, uint64_t n_bytes, uint8_t *status, uint64_t *from, uint8_t *resp, uint32_t *resp_offsets,
               uint64_t *totals);

/* The literal form: every frame in order, as the reference steps it, over groups[0 .. n_groups) and their logs
 * (terms + g * log_cap).  A frame with entries past log_cap is AFL_FATAL.  outcome[i] = AFL_*; the responses go to resp /
 * resp_offsets / totals as in the batch form (resp: 85 n bytes); a fatal frame changes nothing. */
void afl_literal(afl_group *groups, uint64_t *terms, uint64_t log_cap, size_t n_groups, const uint8_t *bytes,
                 const uint32_t *offsets, size_t n, uint64_t n_bytes, uint8_t *outcome, uint8_t *resp, uint32_t *resp_offsets,
                 uint64_t *totals);

/* afl_batch's seconds on one core (the micro-benchmark's CPU reference). */
double afl_bench(ro_arena_view *a, const ro_read_queues *q, const afl_log *logs, const uint8_t *bytes, const uint32_t *offsets,
                 size_t n, uint64_t n_bytes, uint8_t *status, uint64_t *from, uint8_t *resp, uint32_t *resp_offsets,
                 uint64_t *totals);

#ifdef __cplusplus
}
#endif
#endif /* APP_FOLLOW_ORACLE_H */
