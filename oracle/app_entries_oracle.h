/*
 * app_entries_oracle.h -- CPU ORACLE of MsgAppend frames with entries at the follower. TEST INFRASTRUCTURE ONLY (see
 * raft_oracle.h).
 *
 * The batch form of raftgpu_follower_append_entries, restated over the arena view and the caller's run table: the
 * statuses of afl_batch (app_follow_oracle.h) in the order of include/raftgpu.h, plus the entries: every field 7 of a
 * frame past TERM decoded as an eraftpb.Entry (an Entry that is not a well-formed message: MALFORMED, no claim), and
 * for the claiming frame whose log matches at m.index maybe_append (raft_log.rs:249-279) with find_conflict
 * (:182-198) read from the run -- NEEDS_LOG for what the pass hands back, COMMIT_RANGE for the fatal! ones, else the
 * new last_index through the control oracle's SET_LOG_BOUNDS, commit_to through its COMMIT_TO, the new run written
 * into the table, the appended record and the response.
 *
 * Built together with the other oracle sources into libraft_oracle.so (oracle/app_entries_oracle.py).
 */
#ifndef APP_ENTRIES_ORACLE_H
#define APP_ENTRIES_ORACLE_H

#include "app_follow_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* an applied frame's low-nibble bit (== RAFTGPU_FAPP_APPENDED) */
enum { AEO_APPENDED = 8 };

/* == raftgpu_follower_appended */
typedef struct {
    uint64_t first_index, last_index, run_start, run_term;
    uint32_t span_off, span_len;
} aeo_appended;

/* One field 7 of a Message, in frame order: its Entry's term (2) and index (3) when it is length-delimited (ld), and
 * its record [off, end) from the Message's start (tag included). */
typedef struct {
    uint64_t term, index;
    uint32_t off, end;
    uint32_t ld, reserved;
} aeo_entry;

/* The Message buf[0, len): 0 when it, or one of its length-delimited field 7s as an Entry, is not a well-formed
 * protobuf message; else 1, *m decoded and the first max_ents field 7s in ents (*n = how many there are). */
int aeo_decode(const uint8_t *buf, size_t len, wo_message *m, aeo_entry *ents, size_t max_ents, size_t *n);

/* The batch form: afl_batch's arguments, the table read-write, and appended[n] (all zero but for the appended
 * frames). */
void aeo_batch(ro_arena_view *a, const ro_read_queues *q, afl_log *logs, const uint8_t *bytes, const uint32_t *offsets,
               size_t n, uint64_t n_bytes, uint8_t *status, uint64_t *from, aeo_appended *appended, uint8_t *resp,
               uint32_t *resp_offsets, uint64_t *totals);

/* aeo_batch's seconds on one core (the micro-benchmark's CPU reference). */
double aeo_bench(ro_arena_view *a, const ro_read_queues *q, afl_log *logs, const uint8_t *bytes, const uint32_t *offsets,
                 size_t n, uint64_t n_bytes, uint8_t *status, uint64_t *from, aeo_appended *appended, uint8_t *resp,
                 uint32_t *resp_offsets, uint64_t *totals);

#ifdef __cplusplus
}
#endif
#endif /* APP_ENTRIES_ORACLE_H */
