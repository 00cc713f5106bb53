/*
 * raft_oracle.h -- CPU ORACLE. TEST INFRASTRUCTURE ONLY.
 *
 * A plain-C restatement of the commit-index hot path of pingcap/raft-rs
 * (crate `raft` 0.6.0 @ 7c21f8d).  Nothing in the product path (libraftgpu.so,
 * the host mirror, bench.py's GPU arm) may include, link or call this file;
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * `--impl reference` legs do, and there only as the checker / the CPU
 * baseline.
 *
 * Parity status: PINNED.  The functions below are replayed against the
 * reference's own golden vectors (tests/golden/quorum/ .txt files, copied from
 * src/quorum/testdata/) and against the table tests listed next to each
 * function (tests/test_oracle_*.py).  The reference itself is Rust and cannot
 * be built without a Rust toolchain, which the project does not assume, so there is no oracle/_ref.
 *
 * Every function cites the reference file:line it restates (paths relative to
 * the reference checkout).
 */
#ifndef RAFT_ORACLE_H
#define RAFT_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- src/quorum.rs ------------------------------------------------------ */

/* quorum.rs:12-20 -- enum order is Pending, Lost, Won. */
enum { RO_VOTE_PENDING = 0, RO_VOTE_LOST = 1, RO_VOTE_WON = 2 };

/* quorum.rs:35-38 */
typedef struct {
    uint64_t index;
    uint64_t group_id;
} ro_index;

/* quorum.rs:67-74 `AckIndexer = HashMap<u64, Index>`: parallel arrays. */
typedef struct {
    const uint64_t *ids;
    const ro_index *idx;
    size_t n;
} ro_ack_indexer;

/* votes: HashMap<u64,bool>; vote[i] in {0 = no, 1 = yes}. */
typedef struct {
    const uint64_t *ids;
    const uint8_t *vote;
    size_t n;
} ro_vote_map;

/* util.rs:118-120 */
size_t ro_majority(size_t total);

/* quorum.rs:69-74: returns 1 and fills *out when `voter` has an entry. */
int ro_acked_index(const ro_ack_indexer *l, uint64_t voter, ro_index *out);

/* majority.rs:70-124.  `voters` is the set in iteration order. */
void ro_majority_committed_index(const uint64_t *voters, size_t n_voters,
                                 int use_group_commit, const ro_ack_indexer *l,
                                 uint64_t *out_index, int *out_use_gc);

/* joint.rs:47-51 */
void ro_joint_committed_index(const uint64_t *incoming, size_t n_in,
                              const uint64_t *outgoing, size_t n_out,
                              int use_group_commit, const ro_ack_indexer *l,
                              uint64_t *out_index, int *out_use_gc);

/* majority.rs:130-154 */
int ro_majority_vote_result(const uint64_t *voters, size_t n_voters,
                            const ro_vote_map *votes);
/* joint.rs:56-67 */
int ro_joint_vote_result(const uint64_t *incoming, size_t n_in,
                         const uint64_t *outgoing, size_t n_out,
                         const ro_vote_map *votes);

/* ---- src/tracker/progress.rs, src/tracker/state.rs ---------------------- */

/* state.rs:22-29 */
enum { RO_STATE_PROBE = 0, RO_STATE_REPLICATE = 1, RO_STATE_SNAPSHOT = 2 };

/* raft.rs:81 */
#define RO_INVALID_INDEX 0ull

/* src/tracker/inflights.rs:19-110: the sliding window of in-flight MsgAppends of one peer (the last index of each),
 * a ring of `cap` entries (Config::max_inflight_msgs, config.rs:112).  Pinned by the reference's own table tests
 * (inflights.rs:131-256) in tests/test_oracle_tables.py. */
typedef struct {
    uint32_t start; /* inflights.rs:21 */
    uint32_t count; /* :23 */
    uint32_t cap;   /* buffer.capacity() */
    uint64_t *buffer;
} ro_inflights;
int ro_inflights_full(const ro_inflights *in);            /* :54-56 */
int ro_inflights_add(ro_inflights *in, uint64_t v);       /* :65-82; -1 where the reference panics (full) */
void ro_inflights_free_to(ro_inflights *in, uint64_t to); /* :85-110 */
void ro_inflights_free_first_one(ro_inflights *in);       /* :113-116 */
void ro_inflights_reset(ro_inflights *in);                /* :119-123 */

/* progress.rs:8-56.  `ins`: when the caller models the Inflights ring (`ins` != NULL) every place the
 * reference touches it does; otherwise the single bit the path reads from it, `ins.full()`
 * (progress.rs:213), is carried as `ins_full`, cleared wherever the reference calls ins.reset(). */
typedef struct {
    uint64_t matched;
    uint64_t next_idx;
    uint64_t pending_snapshot;
    uint64_t pending_request_snapshot;
    uint64_t commit_group_id;
    uint64_t committed_index;
    uint8_t state;
    uint8_t paused;
    uint8_t recent_active;
    uint8_t ins_full;
    ro_inflights *ins; /* optional */
} ro_progress;

void ro_progress_new(ro_progress *p, uint64_t next_idx);       /* progress.rs:60-73 */
void ro_progress_reset(ro_progress *p, uint64_t next_idx);     /* progress.rs:82-92 */
void ro_progress_become_probe(ro_progress *p);                 /* progress.rs:95-107 */
void ro_progress_become_replicate(ro_progress *p);             /* progress.rs:110-114 */
void ro_progress_become_snapshot(ro_progress *p, uint64_t i);  /* progress.rs:117-121 */
void ro_progress_snapshot_failure(ro_progress *p);             /* progress.rs:124-127 */
int ro_progress_maybe_snapshot_abort(const ro_progress *p);    /* progress.rs:131-134 */
int ro_progress_maybe_update(ro_progress *p, uint64_t n);      /* progress.rs:138-150 */
void ro_progress_update_committed(ro_progress *p, uint64_t c); /* progress.rs:153-157 */
void ro_progress_optimistic_update(ro_progress *p, uint64_t n);/* progress.rs:160-163 */
int ro_progress_maybe_decr_to(ro_progress *p, uint64_t rejected, uint64_t match_hint,
                              uint64_t request_snapshot);      /* progress.rs:168-206 */
int ro_progress_is_paused(const ro_progress *p);               /* progress.rs:210-216 */
void ro_progress_resume(ro_progress *p);                       /* progress.rs:219-222 */
void ro_progress_pause(ro_progress *p);                        /* progress.rs:225-228 */
/* progress.rs:231-243; returns -1 where the reference panics (Snapshot). */
int ro_progress_update_state(ro_progress *p, uint64_t last);

/* ---- src/raft_log.rs (commit bookkeeping only) -------------------------- */

/* A literal log model: entries first_index..first_index+n-1 with terms[],
 * plus the dummy entry (first_index-1, dummy_term) the storage keeps
 * (storage.rs MemStorage; raft_log.rs:124 `dummy_idx = first_index - 1`). */
typedef struct {
    uint64_t first_index;
    uint64_t dummy_term;
    const uint64_t *terms;
    size_t n;
    uint64_t committed;
} ro_raft_log;

uint64_t ro_log_last_index(const ro_raft_log *l);
uint64_t ro_log_term(const ro_raft_log *l, uint64_t idx);            /* raft_log.rs:122-140 */
/* raft_log.rs:286-300; returns -1 where the reference `fatal!`s. */
int ro_log_commit_to(ro_raft_log *l, uint64_t to_commit);
int ro_log_maybe_commit(ro_raft_log *l, uint64_t max_index, uint64_t term); /* raft_log.rs:487-499 */

/* ---- the batched arena view (same SoA layout as the GPU arena) ---------- */

/* per-peer flag byte */
#define RO_PF_STATE_MASK 0x03u
#define RO_PF_PAUSED 0x04u
#define RO_PF_RECENT_ACTIVE 0x08u
#define RO_PF_INS_FULL 0x10u

/* per-group meta word: [0,8) incoming voters, [8,16) outgoing voters,
 * [16,24) learners (learners + learners_next), [24,27) self slot,
 * bit 27 = has self slot, bit 28 = group_commit enabled. */
#define RO_META_IN(m) ((m) & 0xffu)
#define RO_META_OUT(m) (((m) >> 8) & 0xffu)
#define RO_META_LEARN(m) (((m) >> 16) & 0xffu)
#define RO_META_SELF(m) (((m) >> 24) & 0x7u)
#define RO_META_HAS_SELF 0x08000000u
#define RO_META_GROUP_COMMIT 0x10000000u
/* A wide group (up to 16 peers) = two consecutive group slots: g (even, WIDE_LO, peers 0..7) and g + 1 (WIDE_HI,
 * peers 8..15).  Cells are addressed per half; quorum, votes and maybe_commit are evaluated on the low half over
 * both halves' peers (ids 1..16), and the group's log / commit columns are kept equal on both. */
#define RO_META_WIDE_LO 0x20000000u
#define RO_META_WIDE_HI 0x40000000u

#define RO_SLOTS 8

/* Columns are [RO_SLOTS][cap] (peer columns) or [cap] (group columns). */
typedef struct {
    uint32_t cap;      /* column stride in groups */
    uint32_t n_groups; /* groups in use: 0..n_groups-1 */
    uint64_t *matched;
    uint64_t *next_idx;
    uint64_t *peer_committed;
    uint64_t *pending_snapshot;
    uint64_t *pending_request_snapshot;
    uint64_t *commit_group_id;
    uint8_t *pflags;
    uint32_t *meta;
    uint64_t *committed;
    uint64_t *term_start; /* first index of the leader's own term; UINT64_MAX = not leader */
    uint64_t *last_index;
    uint64_t *term;       /* only used by the literal synthetic-log check */
    /* optional device-side Inflights (SURVEY 8(f2)): ins_cap = window size (0 = not modelled, the ins_full bit is
     * then host-reported); ins_meta [RO_SLOTS][cap] = start | count << 16; ins_buf [RO_SLOTS][cap][ins_cap] */
    uint32_t ins_cap;
    uint32_t *ins_meta;
    uint64_t *ins_buf;
} ro_arena_view;

/* AppendResponse record, 24 bytes (SURVEY 8(d)); a REJECT record is followed
 * by one EXT record whose `index` = next_probe_index (raft.rs:1560-1661) and
 * whose `commit` = request_snapshot. */
typedef struct {
    uint32_t group;
    uint8_t peer_slot;
    uint8_t flags;
    uint16_t reserved;
    uint64_t index;
    uint64_t commit;
} ro_append_resp;
#define RO_REC_REJECT 0x01u
/* leader-local record: `commit` (when non-zero) is the new last_index after
 * Raft::append_entry (raft.rs:974-991), `index` the newly persisted index fed to
 * on_persist_entries (raft.rs:994-1016: prs[self].maybe_update(index) &&
 * maybe_commit()); peer_slot is the leader's own slot. */
#define RO_REC_LOCAL 0x02u
#define RO_REC_EXT 0x80u

/* per-record result byte */
#define RO_RES_OK 0x01u          /* maybe_update / maybe_decr_to returned true */
#define RO_RES_OLD_PAUSED 0x02u  /* is_paused() before maybe_update (raft.rs:1724) */
#define RO_RES_NO_PROGRESS 0x04u /* raft.rs:1663-1673: unknown responder */
#define RO_RES_SEND 0x08u        /* reject path reached send_append (raft.rs:1719) */

/* maximal_committed_index for one group of the arena (tracker.rs:294-298 via
 * tracker.rs:183-190, joint.rs:47-51, majority.rs:70-124): literal version,
 * builds the voter id lists and an AckIndexer and calls the functions above. */
void ro_arena_mci(const ro_arena_view *a, uint32_t g, uint64_t *out_index, int *out_use_gc);

/* Raft::maybe_commit for one group (raft.rs:893-904), range formulation of
 * RaftLog::maybe_commit: term(mci)==term  <=>  term_start <= mci <= last_index. */
int ro_arena_maybe_commit(ro_arena_view *a, uint32_t g);
/* Same, through the literal synthetic log model: term_of(idx) = 0 if
 * idx > last_index; term[g] if idx >= term_start; else term[g]-1 (SURVEY 8(d)). */
int ro_arena_maybe_commit_literal(ro_arena_view *a, uint32_t g);

/* handle_append_response sequencing for ONE record (raft.rs:1663-1751), with
 * (per_message_commit != 0) or without the trailing self.maybe_commit().
 * `ext` is the following EXT record for rejects (may be NULL otherwise).
 * Returns the result byte; *advanced is set when maybe_commit returned true. */
uint8_t ro_arena_handle_append_response(ro_arena_view *a, const ro_append_resp *rec,
                                        const ro_append_resp *ext, int per_message_commit,
                                        int *advanced);

/* Apply n records in arrival order.  mode 0 = batched (no per-message
 * commit), mode 1 = literal per-message maybe_commit.  results may be NULL. */
void ro_arena_apply(ro_arena_view *a, const ro_append_resp *recs, size_t n, int mode,
                    uint8_t *results);

/* Recompute pass over groups [first, first+n): maybe_commit each group, set
 * bit g of adv_bitmap (u32 words) when it advanced, store mci/use_gc when the
 * out arrays are non-NULL.  Returns the number of advanced groups. */
uint64_t ro_arena_recompute(ro_arena_view *a, uint32_t first, uint32_t n, uint32_t *adv_bitmap,
                            uint64_t *mci_out, uint8_t *gc_out);

/* Vote tally for the arena (tracker.rs:313-340 / majority.rs:130-154 /
 * joint.rs:56-67): votes[slot*cap+g] in {0 missing, 1 no, 2 yes}. */
int ro_arena_vote_result(const ro_arena_view *a, const uint8_t *votes, uint32_t g,
                         uint32_t *granted, uint32_t *rejected);

/* Post-commit send decisions: bcast_append (raft.rs:857-865) for the groups of [first, first+n)
 * whose bit is set in adv_bitmap (NULL = all), each send_append gated by Progress::is_paused
 * (raft.rs:780-788, progress.rs:210-216).  One entry per (group, peer != self, not paused), in
 * (group, slot) order; returns the number of entries (only the first `cap` are stored). */
typedef struct {
    uint32_t group;
    uint8_t peer_slot;
    uint8_t flags; /* 1 = pending_request_snapshot != INVALID_INDEX (raft.rs:792-797) */
    uint16_t reserved;
    uint64_t next_idx;
} ro_send_entry;
uint64_t ro_arena_send_list(const ro_arena_view *a, uint32_t first, uint32_t n, const uint32_t *adv_bitmap,
                            ro_send_entry *out, uint64_t cap);

/* bcast_heartbeat (raft.rs:875-889) -> send_heartbeat commit = min(pr.matched, committed)
 * (raft.rs:838-840) for every present peer but the group's own slot; UINT64_MAX elsewhere.
 * out[slot * n + (g - first)]. */
void ro_arena_heartbeat_commits(const ro_arena_view *a, uint32_t first, uint32_t n, uint64_t *out);

/* handle_heartbeat_response for ONE record (raft.rs:1777-1819, the tracker part: the read-index tail
 * :1806-1818 is outside the path): rec->commit = m.commit.  update_committed, recent_active = true,
 * resume(); a Replicate peer whose inflights window is full frees its first entry (:1797-1799 -- a full
 * window that loses an entry is no longer full, so the carried ins_full bit clears); RO_RES_SEND when the
 * reference calls send_append: pr.matched < last_index || pending_request_snapshot != INVALID_INDEX
 * (:1801-1804).  RO_RES_OK marks a record that found its Progress. */
#define RO_REC_HEARTBEAT 0x04u
uint8_t ro_arena_handle_heartbeat_response(ro_arena_view *a, const ro_append_resp *rec);
void ro_arena_apply_heartbeat(ro_arena_view *a, const ro_append_resp *recs, size_t n, uint8_t *results);

/* Progress::update_state(last) (progress.rs:231-243) for every entry {group, peer_slot, next_idx = last}:
 * what send_append does after it built a MsgAppend (raft.rs:753-760): Replicate -> optimistic_update(last)
 * (+ ins.add(last), host side), Probe -> pause().  results[i]: 1 done, 0xff where the reference panics
 * (Snapshot state), RO_RES_NO_PROGRESS for an unknown peer. */
void ro_arena_update_state(ro_arena_view *a, const ro_send_entry *entries, size_t n, uint8_t *results);

/* ---- CPU baseline timing (bench.py cpu_baseline / --impl reference) ----- */

/* Runs `iters` recompute passes over the whole arena with n_threads pthreads
 * (static range partition) and returns wall seconds (CLOCK_MONOTONIC). */
double ro_bench_recompute(ro_arena_view *a, int n_threads, int iters, uint64_t *advanced_total);
/* One full step: apply recs (batched mode, range-partitioned by group: recs
 * must be sorted by group) then recompute, n_threads pthreads. */
double ro_bench_step(ro_arena_view *a, const ro_append_resp *recs, size_t n_recs, int n_threads,
                     uint64_t *advanced_total);
/* Same step through the tuned CPU path (in-place column updates, direct selection):
 * identical results, what the CPU baseline arm times. */
double ro_bench_step_fast(ro_arena_view *a, const ro_append_resp *recs, size_t n_recs, int n_threads,
                          uint64_t *advanced_total);

#ifdef __cplusplus
}
#endif
#endif /* RAFT_ORACLE_H */
