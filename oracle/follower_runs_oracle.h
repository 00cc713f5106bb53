/* follower_runs_oracle.h -- the follower's earlier term runs (DESIGN 3.22, include/raftgpu.h
 * raftgpu_arena_enable_follower_runs) on the CPU: raftgpu_follower_append and raftgpu_follower_append_entries as they
 * decide on an arena with follower runs, one batch (one wave) at a time.  TEST INFRASTRUCTURE ONLY.
 *
 * The rule restated over the arena view, the table and the rows: term(i) is 0 above last_index, run_term on the table's
 * run [run_start, last_index], and -- when the group's row is anchored there (the table's run non-empty and equal to
 * the row's anchor, with a non-zero term) -- the row's run 1 and run 2 below it.  Every read of a term goes through
 * that lookup: the match at m.index, the rejection's find_conflict_by_term walk (a walk that leaves the lowest stated
 * run is NEEDS_LOG) and find_conflict over the entries.  An append that does not keep the table's run rewrites the
 * table and the row from the top of the new log: the appended blocks (at most the last two), then -- when they are all
 * the appended entries -- the segment that held conflict - 1, cut there, and the runs below it; equal neighbours
 * merge; the row takes the two segments below the top while their terms strictly decrease. */
#ifndef FOLLOWER_RUNS_ORACLE_H
#define FOLLOWER_RUNS_ORACLE_H

#include "app_entries_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* == raftgpu_follower_runs */
typedef struct {
    uint32_t group, reserved;
    uint64_t anchor_start, anchor_term;
    uint64_t run_start[2], run_term[2];
} fro_row;

/* One batch: afl_batch (entries == 0) or aeo_batch (entries != 0) with rows[g] per group slot (NULL: an arena without
 * follower runs, where it is exactly those).  The table (logs), the rows and the arena view change in place as the
 * device's do; appended (n records) is written for entries != 0 only. */
void fro_batch(ro_arena_view *a, const ro_read_queues *q, afl_log *logs, fro_row *rows, int entries, const uint8_t *bytes,
               const uint32_t *offsets, size_t n, uint64_t n_bytes, uint8_t *status, uint64_t *from, aeo_appended *appended,
               uint8_t *resp, uint32_t *resp_offsets, uint64_t *totals);

/* fro_batch's seconds on one core (the micro-benchmark's CPU reference). */
double fro_bench(ro_arena_view *a, const ro_read_queues *q, afl_log *logs, fro_row *rows, int entries, const uint8_t *bytes,
                 const uint32_t *offsets, size_t n, uint64_t n_bytes, uint8_t *status, uint64_t *from, aeo_appended *appended,
                 uint8_t *resp, uint32_t *resp_offsets, uint64_t *totals);

#ifdef __cplusplus
}
#endif
#endif /* FOLLOWER_RUNS_ORACLE_H */
