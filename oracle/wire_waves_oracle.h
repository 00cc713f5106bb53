/*
 * wire_waves_oracle.h -- CPU ORACLE of the passes at raftgpu_arena_set_wire_waves > 1 (DESIGN 3.19).  TEST INFRASTRUCTURE
 * ONLY (see raft_oracle.h).
 *
 * It restates only the wave loop and the follower's stop rule of include/raftgpu.h: F1 = every frame of the batch; run j
 * is the existing batch form over the frames Fj, re-packed as a batch of their own in their batch order, whose statuses,
 * records and responses are mapped back to the frames' positions; Fj+1 = the frames run j returned DUP (the follower's
 * passes: but for those of groups whose claimant in run j was NEEDS_LOG or COMMIT_RANGE).  The batch forms it calls:
 *   - the wire step: lro_decode_batch (leader_runs_oracle.h; no rows = wo_decode_batch), then every OK frame's record,
 *     and a REJECT's EXT with its hint, through ro_arena_apply in frame order;
 *   - the follower's entry-less pass: afl_batch (app_follow_oracle.h);
 *   - the follower's pass with entries: aeo_batch (app_entries_oracle.h).
 *
 * Built together with the other oracle sources into libraft_oracle.so (oracle/wire_waves_oracle.py).
 */
#ifndef WIRE_WAVES_ORACLE_H
#define WIRE_WAVES_ORACLE_H

#include "app_entries_oracle.h"
#include "leader_runs_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The wire step at `waves` over the arena view c (changed in place; no maybe_commit: the caller runs it once after, as
 * the device does).  rows [c->n_groups] or NULL.  status[i] = WO_WIRE_* << 4 | the result's low nibble of an applied
 * frame. */
void wwo_leader(ro_arena_view *c, const lro_row *rows, const uint8_t *bytes, const uint32_t *offsets, size_t n,
                uint64_t n_bytes, uint32_t waves, uint8_t *status);

/* wwo_leader's seconds on one core (the micro-benchmark's CPU reference). */
double wwo_leader_bench(ro_arena_view *c, const lro_row *rows, const uint8_t *bytes, const uint32_t *offsets, size_t n,
                        uint64_t n_bytes, uint32_t waves, uint8_t *status);

/* The follower's append pass at `waves`: afl_batch (entries 0; appended may be NULL) or aeo_batch (entries 1), their
 * arguments and outputs for the whole batch.  The responses of every run go to resp in frame order (85 n bytes),
 * resp_offsets [responses + 1], totals = {responses, bytes}. */
void wwo_follower(ro_arena_view *c, const ro_read_queues *q, afl_log *logs, int entries, const uint8_t *bytes,
                  const uint32_t *offsets, size_t n, uint64_t n_bytes, uint32_t waves, uint8_t *status, uint64_t *from,
                  aeo_appended *appended, uint8_t *resp, uint32_t *resp_offsets, uint64_t *totals);

#ifdef __cplusplus
}
#endif
#endif /* WIRE_WAVES_ORACLE_H */
