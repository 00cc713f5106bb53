/*
 * leader_runs_oracle.h -- CPU ORACLE for the leader-runs decision of the wire step (DESIGN 3.18).  TEST INFRASTRUCTURE
 * ONLY (same rules as raft_oracle.h: only tests/, smoke() and bench.py's checker legs may use it).
 *
 * What it restates: the leader's side of a rejected MsgAppendResponse, raft.rs:1559-1562 and
 * RaftLog::find_conflict_by_term (raft_log.rs:209-235) with RaftLog::term (raft_log.rs:122-140), in two forms:
 *   - the literal form walks a leader's whole term array one index at a time, as the reference does;
 *   - the batch form restates the device rule: the arena's (term, term_start, last_index) and a row of at most two
 *     earlier term runs, the anchor test, and the undecided case that leaves a frame RAFTGPU_WIRE_NEEDS_LOG.
 * Both decode each Message with wire_oracle.c's wo_decode_message and restate wo_decode_batch's loop around it: the
 * frame checks, the statuses, the term rule and the duplicate rule (the first passing frame of a (group, peer) cell
 * wins).  With no rows the batch form equals wo_decode_batch (tests/test_oracle_append_reject.py).  Parity: the decode is pinned by python-protobuf vectors (wire_oracle.h); the
 * walk by the reference's test_fast_log_rejection, restated in tests/test_oracle_append_reject.py.
 */
#ifndef LEADER_RUNS_ORACLE_H
#define LEADER_RUNS_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#include "raft_oracle.h"
#include "wire_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One group's row (include/raftgpu.h raftgpu_leader_runs, restated): the anchor (term, term_start), run 1 =
 * [run_start[0], term_start - 1] at run_term[0], run 2 = [run_start[1], run_start[0] - 1] at run_term[1]; a start of
 * 0 states no run. */
typedef struct {
    uint32_t group, reserved;
    uint64_t term, term_start;
    uint64_t run_start[2];
    uint64_t run_term[2];
} lro_row;

/* The setter's check of one row: 0 (stored), -5 (RAFTGPU_ERR_RANGE: not allocated, or a wide pair's high half) or -1
 * (RAFTGPU_ERR_INVALID: term 0, term_start 0 or u64::MAX, run 2 without run 1, starts not strictly descending below
 * term_start, run terms 0 or not strictly descending below term). */
int32_t lro_row_status(const lro_row *r, int allocated, int wide_hi);

/* find_conflict_by_term(h, lt) on a log whose terms[i] is the term of entry i for first_index - 1 <= i <= last_index
 * (RaftLog::term is 0 outside that range).  Returns the conflict index (.0 of the reference's result). */
uint64_t lro_find_conflict_by_term(const uint64_t *terms, uint64_t first_index, uint64_t last_index, uint64_t h, uint64_t lt);

/* The device rule for one group: 1 and *out = the conflict index when the leader's (term, term_start, last_index) and
 * its row decide it, 0 when not (no row, a row anchored to another leadership, or a walk that leaves the stated runs
 * above lt).  row NULL = an arena without runs. */
int lro_probe_by_runs(uint64_t term, uint64_t term_start, uint64_t last_index, const lro_row *row, uint64_t h, uint64_t lt,
                      uint64_t *out);

/* The batch form over the arena view c: wo_decode_batch's statuses, records, hints and request_snapshots, with the term
 * test on c->term, and every rejection with log_term > 0 decided by lro_probe_by_runs (a wide pair: the low half's term,
 * term_start and row, the larger last_index) or left WO_WIRE_NEEDS_LOG.  rows [c->n_groups] or NULL. */
void lro_decode_batch(const ro_arena_view *c, const lro_row *rows, const uint8_t *bytes, const uint32_t *offsets, size_t n,
                      uint64_t n_bytes, uint8_t *status, wo_record *recs, uint64_t *hint, uint64_t *request_snapshot);

/* The literal form: as lro_decode_batch, but every rejection with log_term > 0 passes, with its hint from
 * lro_find_conflict_by_term on group g's log: terms log_terms[log_off[g] .. log_off[g + 1]) for entries 0 .., last
 * index log_off[g + 1] - log_off[g] - 1, first index first_index[g].  group_term: as wo_decode_batch's. */
void lro_literal_batch(const uint64_t *log_off, const uint64_t *log_terms, const uint64_t *first_index,
                       const uint64_t *group_term, uint32_t n_groups, const uint8_t *bytes, const uint32_t *offsets,
                       size_t n, uint64_t n_bytes, uint8_t *status, wo_record *recs, uint64_t *hint,
                       uint64_t *request_snapshot);

/* lro_decode_batch `iters` times on one thread; seconds per batch. */
double lro_bench(const ro_arena_view *c, const lro_row *rows, const uint8_t *bytes, const uint32_t *offsets, size_t n,
                 uint64_t n_bytes, uint8_t *status, wo_record *recs, uint64_t *hint, uint64_t *request_snapshot, int iters);

#ifdef __cplusplus
}
#endif
#endif
