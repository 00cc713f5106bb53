/*
 * raftgpu.h -- C-ABI boundary of the H100 batched multi-raft commit-index engine.
 *
 * raft-rs (pingcap/raft-rs, crate `raft` 0.6.0 @ 7c21f8d) has no FFI/plugin
 * interface for this path: the boundary is the Rust method surface of
 * ProgressTracker / Progress / quorum::{MajorityConfig,JointConfig} /
 * RaftLog::maybe_commit / Raft::maybe_commit.  Each entry point below names the
 * reference interface (file:line, relative to the reference checkout) it
 * replaces; the Rust-side binding a maintainer would add is in INTEGRATION.md.
 *
 * Conventions
 *  - plain C: pointers and sizes only, no C++/torch types;
 *  - every function returns an int32_t status (RAFTGPU_OK or a negative
 *    RAFTGPU_ERR_*); nothing throws or aborts across the boundary.  The hot-path
 *    functions of the reference are infallible (they return bool / tuples);
 *    the codes here cover misuse and CUDA failures, plus the two places the
 *    reference itself errors: StepPeerNotFound (raw_node.rs:402-411) and the
 *    `fatal!` in RaftLog::commit_to (raft_log.rs:291-298);
 *  - there is NO CPU fallback: without a CUDA device every compute entry point
 *    returns RAFTGPU_ERR_NO_DEVICE;
 *  - `stream` parameters are a cudaStream_t passed as void* (NULL = the arena's
 *    own compute stream);
 *  - threading follows the reference (raw_node.rs:284 "RawNode is a
 *    thread-unsafe Node", raft.rs:292-294 `Raft: Send`): calls that touch ONE
 *    group may run concurrently for DIFFERENT groups; raftgpu_step*,
 *    raftgpu_control (it may change many groups' configurations, and with them
 *    the launch plan of the next step) and the arena lifecycle calls need
 *    exclusive access.
 *
 * Data layout in HBM (struct-of-arrays, see DESIGN.md): per-peer columns are
 * [RAFTGPU_SLOTS][cap] u64 / u8, per-group columns are [cap]; a "group" is one
 * raft group (one ProgressTracker), a "peer slot" one Progress of that group.
 * next_idx and peer_committed are held on the device as signed 16-bit offsets
 * from the same cell's matched, with the exact u64 kept aside for a value the
 * offset cannot express; raftgpu_column_read / _write convert, so every column
 * call still sees u64 values (and a write of matched keeps the cells' next_idx
 * and peer_committed values).
 */
#ifndef RAFTGPU_H
#define RAFTGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RAFTGPU_ABI_VERSION 1
#define RAFTGPU_SLOTS 8 /* peer slots per group (voters + learners, both halves of a joint config) */

/* ---- status codes ------------------------------------------------------- */
#define RAFTGPU_OK 0
#define RAFTGPU_ERR_INVALID (-1)        /* bad argument */
#define RAFTGPU_ERR_CUDA (-2)           /* CUDA runtime error; see raftgpu_last_error */
#define RAFTGPU_ERR_NOMEM (-3)          /* host / device allocation failed, or arena full */
#define RAFTGPU_ERR_NO_DEVICE (-4)      /* no CUDA device: there is no CPU fallback */
#define RAFTGPU_ERR_RANGE (-5)          /* group / peer slot out of range or not allocated */
#define RAFTGPU_ERR_FULL (-6)           /* staging ring full: call raftgpu_step first */
#define RAFTGPU_ERR_PEER_NOT_FOUND (-7) /* Error::StepPeerNotFound, raw_node.rs:402-411 */
#define RAFTGPU_ERR_COMMIT_RANGE (-8)   /* RaftLog::commit_to fatal!, raft_log.rs:291-298 */
#define RAFTGPU_ERR_BUSY (-9)           /* a step is still in flight on this buffer */
/* A group would need more peer slots than it has: 8 (RAFTGPU_SLOTS) for an ordinary group, 16 for a wide one
 * (raftgpu_group_alloc_wide).  Peers = voters of both halves of a joint configuration + learners + learners_next
 * (tracker.rs:37-92).  The reference has no limit (majority.rs:86-93 sorts any number of voters on the heap); 16
 * covers two disjoint 7-voter sets in a joint change plus learners.  Beyond that the caller keeps the group on the
 * stock ProgressTracker (arena groups are independent). */
#define RAFTGPU_ERR_TOO_MANY_PEERS (-10)

const char *raftgpu_strerror(int32_t status);
uint32_t raftgpu_abi_version(void);

/* ---- constants shared with the reference -------------------------------- */
/* ProgressState, src/tracker/state.rs:22-29 */
#define RAFTGPU_STATE_PROBE 0
#define RAFTGPU_STATE_REPLICATE 1
#define RAFTGPU_STATE_SNAPSHOT 2
/* INVALID_INDEX, src/raft.rs:81 */
#define RAFTGPU_INVALID_INDEX 0ull
/* VoteResult, src/quorum.rs:12-20 (declaration order) */
#define RAFTGPU_VOTE_PENDING 0
#define RAFTGPU_VOTE_LOST 1
#define RAFTGPU_VOTE_WON 2
/* "not a leader": no index is of the current term */
#define RAFTGPU_NO_TERM_START UINT64_MAX

/* per-peer flag byte (column RAFTGPU_COL_PFLAGS) */
#define RAFTGPU_PF_STATE_MASK 0x03u
#define RAFTGPU_PF_PAUSED 0x04u        /* Progress::paused, progress.rs:24 */
#define RAFTGPU_PF_RECENT_ACTIVE 0x08u /* Progress::recent_active, progress.rs:41 */
#define RAFTGPU_PF_INS_FULL 0x10u      /* Inflights::full(), inflights.rs:54-56: reported by the host, or (with
                                          raftgpu_arena_enable_inflights) kept by the device */

/* per-group meta word (column RAFTGPU_COL_META): the tracker::Configuration
 * (tracker.rs:37-92) as bit masks over peer slots. */
#define RAFTGPU_META_IN(m) ((m) & 0xffu)            /* voters.incoming, joint.rs:13 */
#define RAFTGPU_META_OUT(m) (((m) >> 8) & 0xffu)    /* voters.outgoing, joint.rs:14 */
#define RAFTGPU_META_LEARN(m) (((m) >> 16) & 0xffu) /* learners | learners_next */
#define RAFTGPU_META_SELF(m) (((m) >> 24) & 0x7u)   /* slot of Raft::id */
#define RAFTGPU_META_HAS_SELF 0x08000000u
#define RAFTGPU_META_GROUP_COMMIT 0x10000000u       /* ProgressTracker::group_commit, tracker.rs:207 */
/* A WIDE group (raftgpu_group_alloc_wide: up to 16 peers) occupies two consecutive group slots: `g` (even) holds
 * peers 0..7 and carries WIDE_LO, `g + 1` holds peers 8..15 and carries WIDE_HI.  Each half's masks describe its own
 * eight peers; quorum / votes / commit are evaluated once, on the low half, over both. */
#define RAFTGPU_META_WIDE_LO 0x20000000u
#define RAFTGPU_META_WIDE_HI 0x40000000u

/* ---- plain data types --------------------------------------------------- */
typedef struct raftgpu_arena raftgpu_arena; /* opaque; owns all device + pinned memory */

/* One Progress (src/tracker/progress.rs:8-56) minus `ins` (Inflights stays host-side). */
typedef struct {
    uint64_t matched;                  /* progress.rs:10 */
    uint64_t next_idx;                 /* progress.rs:12 */
    uint64_t pending_snapshot;         /* progress.rs:31 */
    uint64_t pending_request_snapshot; /* progress.rs:35 */
    uint64_t commit_group_id;          /* progress.rs:52 */
    uint64_t committed_index;          /* progress.rs:55 */
    uint8_t state;                     /* progress.rs:22 */
    uint8_t paused;                    /* progress.rs:25 */
    uint8_t recent_active;             /* progress.rs:41 */
    uint8_t ins_full;                  /* Inflights::full() as last reported by the host */
    uint8_t present;                   /* 1 when the slot holds a Progress */
    uint8_t reserved[3];
} raftgpu_progress;

/* Per-group log / commit bookkeeping: the part of RaftLog (raft_log.rs:33-59)
 * RaftLog::maybe_commit needs, in range form (DESIGN.md "term test"). */
typedef struct {
    uint32_t meta;
    uint32_t reserved;
    uint64_t committed;  /* RaftLog::committed, raft_log.rs:45 */
    uint64_t term_start; /* first index whose entry carries the leader's current term */
    uint64_t last_index; /* RaftLog::last_index() */
} raftgpu_group_state;

/* One MsgAppendResponse as handle_append_response consumes it (raft.rs:1559-1775,
 * eraftpb.proto:71-92): 24 bytes.  A REJECT record is followed by ONE EXT record
 * with the same group/peer_slot whose `index` is next_probe_index (m.reject_hint,
 * or find_conflict_by_term(..).0 when m.log_term > 0 -- that lookup needs the
 * leader's log and is done by the caller, raft.rs:1560-1661) and whose `commit`
 * is m.request_snapshot. */
typedef struct {
    uint32_t group;     /* group slot */
    uint8_t peer_slot;  /* slot of m.from */
    uint8_t flags;      /* RAFTGPU_REC_* */
    uint16_t reserved;
    uint64_t index;     /* m.index */
    uint64_t commit;    /* m.commit */
} raftgpu_append_resp;
#define RAFTGPU_REC_REJECT 0x01u /* m.reject */
/* Leader-local record (not a message): `commit`, when non-zero, is the new
 * last_index after Raft::append_entry (raft.rs:974-991); `index` is the newly
 * persisted index of Raft::on_persist_entries (raft.rs:994-1016), which runs
 * prs[self].maybe_update(index); peer_slot is the leader's own slot. */
#define RAFTGPU_REC_LOCAL 0x02u
#define RAFTGPU_REC_EXT 0x80u    /* extension record of the preceding REJECT */
/* A MsgHeartbeatResponse (raft.rs:1777-1819): `commit` = m.commit, `index` unused.  Only
 * raftgpu_heartbeat_resp[_device] takes such records; the append-response paths ignore them. */
#define RAFTGPU_REC_HEARTBEAT 0x04u

/* The packed 16-byte wire form of a record (raftgpu_pack_records); layout in DESIGN.md 2. */
typedef struct {
    uint64_t w0, w1;
} raftgpu_packed_rec;

/* per-record result byte */
#define RAFTGPU_RES_OK 0x01u          /* maybe_update / maybe_decr_to returned true */
#define RAFTGPU_RES_OLD_PAUSED 0x02u  /* pr.is_paused() before maybe_update, raft.rs:1724 */
#define RAFTGPU_RES_NO_PROGRESS 0x04u /* prs.get_mut(m.from) == None, raft.rs:1663-1673 */
#define RAFTGPU_RES_SEND 0x08u        /* reject path reached self.send_append(m.from), raft.rs:1719 */

/* column ids for bulk IO */
enum {
    RAFTGPU_COL_MATCHED = 0,              /* u64 [SLOTS][cap] */
    RAFTGPU_COL_NEXT_IDX = 1,             /* u64 [SLOTS][cap] */
    RAFTGPU_COL_PEER_COMMITTED = 2,       /* u64 [SLOTS][cap]  Progress::committed_index */
    RAFTGPU_COL_PENDING_SNAPSHOT = 3,     /* u64 [SLOTS][cap] */
    RAFTGPU_COL_PENDING_REQ_SNAPSHOT = 4, /* u64 [SLOTS][cap] */
    RAFTGPU_COL_COMMIT_GROUP_ID = 5,      /* u64 [SLOTS][cap] */
    RAFTGPU_COL_PFLAGS = 6,               /* u8  [SLOTS][cap] */
    RAFTGPU_COL_VOTES = 7,                /* u8  [SLOTS][cap]  0 missing, 1 no, 2 yes */
    RAFTGPU_COL_META = 8,                 /* u32 [cap] */
    RAFTGPU_COL_COMMITTED = 9,            /* u64 [cap] */
    RAFTGPU_COL_TERM_START = 10,          /* u64 [cap] */
    RAFTGPU_COL_LAST_INDEX = 11,          /* u64 [cap] */
    RAFTGPU_COL_TERM = 12,                /* u64 [cap]  Raft::term (raft.rs:227), 0 = unknown; only the wire path reads it */
    RAFTGPU_COL_INS_META = 13,            /* u32 [SLOTS][cap]  Inflights start | count << 16 (raftgpu_arena_enable_inflights) */
    RAFTGPU_COL__COUNT = 14
};

typedef struct {
    uint32_t abi_version;
    int32_t device;
    uint32_t cap;          /* max groups */
    uint32_t slots;        /* RAFTGPU_SLOTS */
    uint32_t n_alloc;      /* groups currently allocated */
    uint32_t hi;           /* allocated groups live in [0, hi) */
    uint32_t sm_count;
    uint32_t reserved;
    uint64_t l2_bytes;
    uint64_t device_bytes; /* HBM held by this arena */
    uint64_t pinned_bytes;
} raftgpu_info;

/* monotonically increasing device-side counters (what the multi-GPU run gathers) */
typedef struct {
    uint64_t recomputes;      /* per-group Raft::maybe_commit evaluations */
    uint64_t advanced;        /* of which advanced `committed` */
    uint64_t records;         /* AppendResponse records applied */
    uint64_t updates;         /* maybe_update returned true */
    uint64_t rejects;         /* reject records seen */
    uint64_t decrements;      /* maybe_decr_to returned true */
    uint64_t no_progress;     /* records for an unknown responder */
    uint64_t votes_tallied;   /* per-group vote_result evaluations */
} raftgpu_counters;

typedef struct {
    uint64_t n_records;  /* records submitted in this step (EXT records included) */
    uint32_t n_waves;    /* kernel waves the records were split into (see raftgpu_enqueue_append_resp) */
    uint32_t n_groups;   /* groups recomputed */
    uint64_t n_advanced; /* groups whose committed index advanced */
    uint64_t h2d_bytes;  /* bytes DMAed host -> device for this step (packed staging records) */
    uint64_t d2h_bytes;  /* bytes DMAed device -> host (advanced bitmap, commit indexes, results) */
    uint64_t n_duplicates; /* zero-copy steps: records dropped because their cell already had one */
} raftgpu_step_result;

/* ---- arena lifecycle ---------------------------------------------------- */

/* ProgressTracker::with_capacity (tracker.rs:217-236) for `max_groups` trackers
 * at once: allocates every column in HBM plus the pinned staging buffers.
 * slots_per_group must be RAFTGPU_SLOTS (8): the unit of the arena is the 8-slot group, and a group that needs up
 * to 16 peers takes two of them (raftgpu_group_alloc_wide); any other value is RAFTGPU_ERR_TOO_MANY_PEERS.  ring_records = capacity of each of
 * the `n_rings` host staging rings (0 = default). */
int32_t raftgpu_arena_create(int32_t device, uint32_t max_groups, uint32_t slots_per_group,
                             uint32_t n_rings, uint32_t ring_records, raftgpu_arena **out);
int32_t raftgpu_arena_destroy(raftgpu_arena *arena);
int32_t raftgpu_arena_info(const raftgpu_arena *arena, raftgpu_info *out);
/* Last CUDA / argument error text for this arena (never NULL). */
const char *raftgpu_last_error(const raftgpu_arena *arena);

/* ---- group lifecycle (control plane; synchronous, small copies) --------- */

/* Raft::new (raft.rs:318-400) / drop: one slot per ProgressTracker. */
int32_t raftgpu_group_alloc(raftgpu_arena *arena, uint32_t *out_group);
int32_t raftgpu_group_alloc_range(raftgpu_arena *arena, uint32_t n, uint32_t *out_first);
/* A WIDE group: up to 16 peer slots (a joint configuration of large voter sets with learners; the reference has no
 * limit, majority.rs:86-93).  It occupies two consecutive group slots: *out_group (even) and *out_group + 1.  Every
 * single-group call takes the group id with peer slots 0..15 and 16-bit masks; in RECORDS (and send-list entries,
 * wire frames, column IO) peer 8 + s of wide group g is addressed as (group g + 1, slot s) -- the per-cell paths do
 * not know about wide groups at all.  Quorum, votes and Raft::maybe_commit are evaluated once, on the low half, over
 * both halves' peers; the advanced bit and the commit index are the low half's.  While an arena holds wide groups its
 * steps run through the scatter + recompute kernels (the fused tile kernel evaluates 8-slot groups); a 17th peer is
 * RAFTGPU_ERR_TOO_MANY_PEERS. */
int32_t raftgpu_group_alloc_wide(raftgpu_arena *arena, uint32_t *out_group);
int32_t raftgpu_group_free(raftgpu_arena *arena, uint32_t group);

/* ProgressTracker::apply_conf (tracker.rs:380-397) / confchange::restore
 * (confchange/restore.rs:91-107): replace the Configuration.  Slots that become
 * present get Progress::new(next_idx, ..) with recent_active = true
 * (tracker.rs:385-390); slots that disappear are removed (tracker.rs:392-394). */
int32_t raftgpu_group_set_conf(raftgpu_arena *arena, uint32_t group, uint32_t incoming_mask,
                               uint32_t outgoing_mask, uint32_t learner_mask, int32_t self_slot,
                               uint64_t next_idx);

/* Raft::reset (raft.rs:942-971) followed by become_leader's bookkeeping
 * (raft.rs:1162-1203): every Progress is reset(last_index + 1); the self slot
 * gets matched = persisted, committed_index = committed (raft.rs:964-970).
 * term_start = RAFTGPU_NO_TERM_START for a non-leader. */
int32_t raftgpu_group_reset(raftgpu_arena *arena, uint32_t group, uint64_t term_start,
                            uint64_t last_index, uint64_t committed, uint64_t persisted);

/* The tracker side of Raft::become_leader (raft.rs:1162-1203), after
 * raftgpu_group_reset: prs[self].become_replicate() (raft.rs:1180), then the
 * empty entry of the new term is appended (raft.rs:1192), so last_index += 1 and
 * term_start = that index. */
int32_t raftgpu_group_become_leader(raftgpu_arena *arena, uint32_t group);

/* Raft::append_entry (raft.rs:974-991): the log grew; entries of the current
 * term are [term_start, last_index]. */
int32_t raftgpu_group_set_log_bounds(raftgpu_arena *arena, uint32_t group, uint64_t term_start,
                                     uint64_t last_index);
/* RaftLog::commit_to (raft_log.rs:286-300): never decreases; RAFTGPU_ERR_COMMIT_RANGE
 * where the reference `fatal!`s (to_commit > last_index). */
int32_t raftgpu_group_commit_to(raftgpu_arena *arena, uint32_t group, uint64_t to_commit);
int32_t raftgpu_group_get(raftgpu_arena *arena, uint32_t group, raftgpu_group_state *out);

/* ProgressTracker::get / get_mut (tracker.rs:267-275): Progress has pub fields,
 * so the Rust shim reads a copy and writes it back. */
int32_t raftgpu_progress_get(raftgpu_arena *arena, uint32_t group, uint32_t peer_slot,
                             raftgpu_progress *out);
int32_t raftgpu_progress_set(raftgpu_arena *arena, uint32_t group, uint32_t peer_slot,
                             const raftgpu_progress *in);

/* Any single method of Progress (src/tracker/progress.rs:75-243) on one peer, executed on the
 * device columns; a0..a2 are the method's arguments, *out_result its bool (or -1 where the
 * reference panics: update_state in Snapshot).  This is what the host mirror's ProgressRef
 * calls; batches of maybe_update / maybe_decr_to go through raftgpu_enqueue_* instead. */
enum {
    RAFTGPU_POP_MAYBE_UPDATE = 0,         /* (n)                                  progress.rs:138-150 */
    RAFTGPU_POP_MAYBE_DECR_TO = 1,        /* (rejected, match_hint, request_snapshot)     :168-206 */
    RAFTGPU_POP_UPDATE_COMMITTED = 2,     /* (committed_index)                            :153-157 */
    RAFTGPU_POP_OPTIMISTIC_UPDATE = 3,    /* (n)                                          :160-163 */
    RAFTGPU_POP_BECOME_PROBE = 4,         /*                                              :95-107  */
    RAFTGPU_POP_BECOME_REPLICATE = 5,     /*                                              :110-114 */
    RAFTGPU_POP_BECOME_SNAPSHOT = 6,      /* (snapshot_idx)                               :117-121 */
    RAFTGPU_POP_SNAPSHOT_FAILURE = 7,     /*                                              :124-127 */
    RAFTGPU_POP_MAYBE_SNAPSHOT_ABORT = 8, /*                                              :131-134 */
    RAFTGPU_POP_IS_PAUSED = 9,            /*                                              :210-216 */
    RAFTGPU_POP_RESUME = 10,              /*                                              :219-222 */
    RAFTGPU_POP_PAUSE = 11,               /*                                              :225-228 */
    RAFTGPU_POP_UPDATE_STATE = 12,        /* (last)                                       :231-243 */
    RAFTGPU_POP_RESET = 13,               /* (next_idx)                                   :82-92   */
    /* Inflights (src/tracker/inflights.rs) of the peer's window, arenas with raftgpu_arena_enable_inflights only
     * (*out_result = -3 otherwise) */
    RAFTGPU_POP_INS_ADD = 14,             /* (inflight); -1 where the reference panics    inflights.rs:65-82 */
    RAFTGPU_POP_INS_FREE_TO = 15,         /* (to)                                         :85-110  */
    RAFTGPU_POP_INS_FREE_FIRST_ONE = 16,  /*                                              :113-116 */
    RAFTGPU_POP_INS_RESET = 17,           /*                                              :119-123 */
    RAFTGPU_POP_INS_FULL = 18             /*                                              :54-56   */
};
int32_t raftgpu_progress_op(raftgpu_arena *arena, uint32_t group, uint32_t peer_slot, int32_t op,
                            uint64_t a0, uint64_t a1, uint64_t a2, int32_t *out_result);

/* ProgressTracker::has_quorum (tracker.rs:367-372) for a set of peer slots, and
 * quorum_recently_active (tracker.rs:346-361; clears recent_active like the reference). */
int32_t raftgpu_has_quorum(raftgpu_arena *arena, uint32_t group, uint32_t slot_mask, int32_t *out);
int32_t raftgpu_quorum_recently_active(raftgpu_arena *arena, uint32_t group, uint32_t perspective_of_slot,
                                       int32_t *out);

/* RaftLog::maybe_commit(max_index, term) (raft_log.rs:487-499) for term == the leader's
 * current term, i.e. the range test on [term_start, last_index]. */
int32_t raftgpu_group_maybe_commit_to(raftgpu_arena *arena, uint32_t group, uint64_t max_index,
                                      int32_t *out_advanced);

/* ProgressTracker::enable_group_commit (tracker.rs:238-241) and
 * Raft::assign_commit_groups / clear_commit_group (raft.rs:531-552). */
int32_t raftgpu_set_group_commit(raftgpu_arena *arena, uint32_t group, int32_t enable);
int32_t raftgpu_assign_commit_group(raftgpu_arena *arena, uint32_t group, uint32_t peer_slot,
                                    uint64_t commit_group_id);

/* Bulk column IO for [first_group, first_group + n) of one column (peer_slot is
 * ignored for per-group columns): restoring / inspecting many groups at once. */
int32_t raftgpu_column_write(raftgpu_arena *arena, int32_t column, uint32_t peer_slot,
                             uint32_t first_group, uint32_t n, const void *host_src);
int32_t raftgpu_column_read(raftgpu_arena *arena, int32_t column, uint32_t peer_slot,
                            uint32_t first_group, uint32_t n, void *host_dst);

/* ---- the hot path ------------------------------------------------------- */

/* ProgressTracker::maximal_committed_index (tracker.rs:294-298) for one group:
 * JointConfig::committed_index (joint.rs:47-51) over MajorityConfig::committed_index
 * (majority.rs:70-124).  Runs the batched kernel on a 1-group range. */
int32_t raftgpu_maximal_committed_index(raftgpu_arena *arena, uint32_t group, uint64_t *out_index,
                                        int32_t *out_use_group_commit);

/* Raft::maybe_commit (raft.rs:893-904) for one group: maximal_committed_index ->
 * RaftLog::maybe_commit (raft_log.rs:487-499) -> prs[self].update_committed. */
int32_t raftgpu_maybe_commit(raftgpu_arena *arena, uint32_t group, int32_t *out_advanced,
                             uint64_t *out_committed);

/* Batched Raft::maybe_commit over groups [first, first + n): ONE kernel pass.
 * Asynchronous on `stream`.  d_adv_bitmap (device, u32 words indexed by
 * group >> 5 from group 0; may be NULL) gets bit g set iff group g advanced;
 * d_commit_out (device u64 [cap], may be NULL) gets the new committed index of
 * advanced groups (entries of other groups are unspecified: the fused step kernels
 * copy every group's commit index there, this pass only the advanced ones); d_mci_out / d_gc_out (may be NULL) get maximal_committed_index
 * for every group. */
int32_t raftgpu_recompute(raftgpu_arena *arena, void *stream, uint32_t first, uint32_t n,
                          uint32_t *d_adv_bitmap, uint64_t *d_commit_out, uint64_t *d_mci_out,
                          uint8_t *d_gc_out);

/* Batched handle_append_response prefix (raft.rs:1663-1743: recent_active,
 * update_committed, maybe_decr_to | maybe_update + state transition) over `n`
 * records ALREADY IN HBM.  Precondition: at most one non-EXT record per
 * (group, peer_slot) in the range -- one "wave"; raftgpu_enqueue_append_resp
 * builds waves for arbitrary streams.  d_results (device, n bytes) may be NULL.
 * Asynchronous on `stream`. */
int32_t raftgpu_apply_device(raftgpu_arena *arena, void *stream,
                             const raftgpu_append_resp *d_records, uint64_t n, uint8_t *d_results);

/* Same, for records that are already in the packed 16-byte wire form (raftgpu_pack_records,
 * the format the staging path ships over PCIe) in HBM: a third less record traffic. */
int32_t raftgpu_apply_device_packed(raftgpu_arena *arena, void *stream, const void *d_packed_records,
                                    uint64_t n_packed, uint8_t *d_results);

/* The FUSED step for batches in group order: apply + recompute in one kernel whose HBM traffic is
 * all dense bulk transfers (DESIGN.md 3.4).  d_packed_records are packed records in
 * non-decreasing group order (EXT payloads directly behind their record); d_tile_off[t] is the
 * index of the first record whose group is >= t * RAFTGPU_TILE_GROUPS, for t = 0..n_tiles
 * (raftgpu_tile_index builds and validates it on the host).  One wave per call, like
 * raftgpu_apply_device; processes all allocated groups [0, hi).  A record found outside its tile
 * is not applied and reported as RAFTGPU_RES_NO_PROGRESS.  Asynchronous on `stream`. */
#ifndef RAFTGPU_TILE_GROUPS
#define RAFTGPU_TILE_GROUPS 256
#endif
uint32_t raftgpu_tile_groups(void); /* the value the library was built with */
int32_t raftgpu_step_sorted_device(raftgpu_arena *arena, void *stream, const void *d_packed_records,
                                   uint64_t n_packed, const uint32_t *d_tile_off, uint8_t *d_results,
                                   uint32_t *d_adv_bitmap, uint64_t *d_commit_out);
/* Host helper: out[t] for t = 0..n_tiles where n_tiles = ceil(n_groups / RAFTGPU_TILE_GROUPS)
 * (out has n_tiles + 1 entries).  RAFTGPU_ERR_INVALID if the records are not in group order,
 * RAFTGPU_ERR_RANGE if one names a group >= n_groups (no tile would visit it). */
int32_t raftgpu_tile_index(const raftgpu_packed_rec *packed, uint64_t n_packed, uint32_t n_groups,
                           uint32_t *out, uint64_t out_capacity);

/* Stage host records for the next step (RawNode::step -> Raft::step ->
 * handle_append_response, raw_node.rs:402-411 / raft.rs:1559).  Records for one
 * (group, peer) keep their arrival order: a second record for a cell that
 * already has one in the pending step is placed in a later wave.  `ring`
 * selects one of the arena's staging rings; different threads use different
 * rings (and, as in the reference, different groups). */
int32_t raftgpu_enqueue_append_resp(raftgpu_arena *arena, uint32_t ring,
                                    const raftgpu_append_resp *records, uint64_t n);

/* Bulk form of the above for a caller that already holds a whole batch in host memory:
 * the library splits it over its own staging threads (pinned to the GPU-local CPUs; count
 * from RAFTGPU_HOST_THREADS, default 16, at most the arena's ring count), one ring each.
 * The records of one (group, peer) cell keep their arrival order when the group's records are contiguous in
 * the batch (what a ready loop produces); a cell whose records are scattered through an unordered batch
 * belongs on one ring through raftgpu_enqueue_append_resp.
 * RAFTGPU_BULK_SORTED: the caller promises records are in non-decreasing group order, which
 * lets the threads skip atomics on the per-cell bookkeeping; the order is verified and
 * RAFTGPU_ERR_INVALID returned (nothing is applied; call raftgpu_step to discard) if not. */
#define RAFTGPU_BULK_SORTED 0x1u
int32_t raftgpu_enqueue_bulk(raftgpu_arena *arena, const raftgpu_append_resp *records, uint64_t n,
                             uint32_t flags);

/* ---- zero-copy submission ---------------------------------------------------
 * For callers that build their batch directly in DMA-able memory: raftgpu_host_alloc returns
 * pinned memory on the GPU-local NUMA node, raftgpu_pack_records converts public records to
 * the 16-byte packed wire form (a REJECT and its EXT become 2-3 packed records; returns the
 * packed count), and raftgpu_step_begin_packed ships such a buffer with no staging copy:
 * H2D straight from the caller's buffer, ONE apply wave, the recompute pass, D2H of the
 * results.  The one-record-per-(group, peer) precondition cannot be checked on the host
 * without reading the batch, so the GPU checks it: a duplicate is not applied, counted in
 * raftgpu_step_result.n_duplicates, and raftgpu_step_wait returns RAFTGPU_ERR_INVALID.
 * The buffer must stay untouched until that step's raftgpu_step_wait returns. */
int32_t raftgpu_host_alloc(raftgpu_arena *arena, uint64_t bytes, void **out_pinned);
int32_t raftgpu_host_free(raftgpu_arena *arena, void *pinned);
int32_t raftgpu_pack_records(const raftgpu_append_resp *records, uint64_t n, raftgpu_packed_rec *out,
                             uint64_t out_capacity, uint64_t *out_n);
int32_t raftgpu_step_begin_packed(raftgpu_arena *arena, const raftgpu_packed_rec *pinned_records,
                                  uint64_t n_packed, uint32_t flags);

/* ---- compact stream (the narrow wire form) -------------------------------------
 * PCIe is the end-to-end bottleneck of a step (DESIGN.md 5), so the bytes per record are the
 * end-to-end cost.  The compact stream carries a batch as 4-byte units instead of 16-byte
 * packed records: the records of one group (consecutive in the input, as a multi-raft ready
 * loop produces them) form a RUN
 *      [HDR_A][HDR_B] rec rec rec ...          (at most 8 units after the header)
 * whose header names the group and a 48-bit base index, and each record is a slot, a 14-bit
 * index delta above the base and an 8-bit commit delta:
 *      unit & 3 == 0  REC    [2] LOCAL  [3,6) back  [6,9) peer slot  [9] REJECT  [10,24) index - base
 *                            [24,32) message: index - commit; LOCAL: commit - index (255 = none)
 *                            (the run's header sits at unit positions i-back-2 and i-back-1; a
 *                            REJECT is followed by a payload unit with its next_probe_index hint)
 *      unit & 3 == 1  HDR_A  [2,32) base bits [0,30)
 *      unit & 3 == 2  HDR_B  [2,14) group - g_base[block of HDR_A]   [14,32) base bits [30,48)
 *      unit & 3 == 3  ESC    [2,32) < 0x1fffffff: index into the side table; == 0x1fffffff: padding;
 *                            bit 31 set: the payload of the REJECT in front, [2,31) = hint - index (signed)
 * g_base[] holds one group id per block of RAFTGPU_COMPACT_BLOCK units.  Whatever does not fit
 * (a REJECT that asks for a snapshot, an index more than 8192 away from the run's first, a commit
 * delta above 254, a base above 2^48, a group more than 4095 above its block's g_base, flag bits
 * the format does not know) is an ESC unit pointing at the full 24-byte public record (and its
 * EXT) in the side table -- the format is lossless for ANY input, only less compact for hostile
 * ones.  A 5-peer round is ~22 bytes per group instead of ~57.  The blob is position
 * independent: header, g_base[], units[] (padded to 16 bytes), side[].
 * Same contract as raftgpu_step_begin_packed: pinned buffer (raftgpu_host_alloc), ONE wave
 * checked on the GPU, buffer untouched until the step's raftgpu_step_wait returns.  Result
 * bytes (RAFTGPU_STEP_READ_RESULTS) are per UNIT; raftgpu_pack_compact can report the unit
 * of every public record. */
#define RAFTGPU_COMPACT_MAGIC 0x31434752u /* "RGC1" */
#define RAFTGPU_COMPACT_BLOCK 2048u
typedef struct raftgpu_compact_hdr {
    uint32_t magic;
    uint32_t n_units;   /* 4-byte units */
    uint32_t n_blocks;  /* ceil(n_units / RAFTGPU_COMPACT_BLOCK) */
    uint32_t n_side;    /* 24-byte records in the side table */
    uint64_t n_records; /* public records represented (EXT continuations not counted) */
    uint64_t off_blocks, off_units, off_side; /* byte offsets from the start of the blob, 16-byte aligned */
    uint64_t total_bytes;
    uint32_t flags;     /* RAFTGPU_COMPACT_TILEABLE */
    uint32_t reserved;
} raftgpu_compact_hdr;
/* Set by raftgpu_pack_compact when the groups of the runs ascend and every run has a header
 * (records of one group contiguous, groups in increasing order, no group too far from its
 * block's g_base): the fused tile kernel can then take the stream -- and, because one thread
 * walks a group's records in order, such a stream may hold SEVERAL records per (group, peer). */
#define RAFTGPU_COMPACT_TILEABLE 0x1u
/* ... and no (group, peer) cell occurs twice: the fused kernel may then use one thread per unit
 * (faster than the ordered per-group walk); the kernel still verifies it. */
#define RAFTGPU_COMPACT_ONE_WAVE 0x2u
/* Upper bound of the blob size for n public records (EXT records included in n). */
uint64_t raftgpu_compact_bound(uint64_t n);
/* records[0..n) -> blob at out (out_capacity bytes; any host memory, pinned for the zero-copy
 * step).  unit_of_record: optional [n], the unit index holding record i's result byte
 * (UINT32_MAX for EXT records). */
int32_t raftgpu_pack_compact(const raftgpu_append_resp *records, uint64_t n, void *out, uint64_t out_capacity,
                             uint64_t *out_bytes, uint32_t *unit_of_record);
int32_t raftgpu_step_begin_compact(raftgpu_arena *arena, const void *pinned_blob, uint64_t blob_bytes,
                                   uint32_t flags);
/* Records in ordinary (pageable) host memory -> one step: the library's staging threads pack
 * slices of the batch into the compact stream in pinned memory (cut at group boundaries, so the
 * records of a group must be contiguous for the result to be tileable; any other order still
 * works through the scatter kernel, one record per cell), then the step is submitted like
 * raftgpu_step_begin_compact.  Nothing may have been enqueued for this step.  `records` can be
 * reused as soon as the call returns.  A batch too hostile for the compact form (every record
 * escaping to the side table) goes through raftgpu_enqueue_bulk + raftgpu_step_begin instead, and
 * so does a batch with several records per cell that the fused kernel cannot take: one that is
 * not group-ordered or too sparse to tile (a unit block of the stream spanning more than 4095
 * groups), or any such batch on an arena that cannot run the fused kernel (device-side Inflights,
 * wide groups; RAFTGPU_STEP_ASYNC is ignored on such arenas).  With RAFTGPU_STEP_ASYNC the batch
 * is packed after the call has returned, too late to change paths: a batch that needs the general
 * path is refused instead, its raftgpu_step_wait returns RAFTGPU_ERR_FULL and nothing of it is
 * applied; submit it again without RAFTGPU_STEP_ASYNC.
 * raft.rs:1663-1743 + 893-904 for a whole tick, as one call. */
int32_t raftgpu_step_begin_records(raftgpu_arena *arena, const raftgpu_append_resp *records, uint64_t n,
                                   uint32_t flags);
/* The same step for a blob that already sits in device memory (hdr = a host copy of its
 * header): raftgpu_compact_tile_index_device builds the tile table in d_tile_off -- room for
 * 3 * (ceil(n_groups / RAFTGPU_TILE_GROUPS) + 2) + 2 u32: the first unit of every tile, then each
 * tile's group-id bases -- and bumps *d_bad if the stream is not tileable after all, then
 * raftgpu_step_compact_device runs ONE fused kernel: the records of every tile applied to
 * its rows in shared memory, Raft::maybe_commit for its groups, rows stored back. */
int32_t raftgpu_compact_tile_index_device(raftgpu_arena *arena, void *stream, const void *d_blob,
                                          const raftgpu_compact_hdr *hdr, uint32_t *d_tile_off, uint32_t *d_bad);
/* flags: RAFTGPU_COMPACT_STEP_ORDERED forces the per-group walk (records of a cell applied in stream
 * order); otherwise a ONE_WAVE stream gets one thread per unit, and d_dup_count (nullable) is bumped
 * for every record that turns out to be the second one on its cell (such a record is not applied). */
#define RAFTGPU_COMPACT_STEP_ORDERED 0x1u
int32_t raftgpu_step_compact_device(raftgpu_arena *arena, void *stream, const void *d_blob,
                                    const raftgpu_compact_hdr *hdr, const uint32_t *d_tile_off, uint8_t *d_results,
                                    uint32_t *d_adv_bitmap, uint64_t *d_commit_out, uint32_t *d_dup_count,
                                    uint32_t flags);
/* Result bytes of the last completed ZERO-COPY step (packed: one per packed record, compact:
 * one per unit; 0 for EXT payloads / headers), valid until the next raftgpu_step_wait
 * (RAFTGPU_ERR_INVALID while two steps are in flight, as raftgpu_step_results).  Needs
 * RAFTGPU_STEP_READ_RESULTS.  raft.rs:1663-1743: what handle_append_response decided per message. */
int32_t raftgpu_step_slot_results(raftgpu_arena *arena, const uint8_t **results, uint64_t *n_slots);

/* One batched step over everything enqueued: H2D of the staged records, the
 * apply kernel per wave, ONE recompute pass over all allocated groups, D2H of
 * the results.  raftgpu_step = raftgpu_step_begin + raftgpu_step_wait.  Between
 * begin and wait the caller may already enqueue the NEXT step's records, and may even
 * begin it: up to TWO steps can be in flight (three staging sets), so the H2D of step
 * j+1 overlaps the kernels and D2H of step j.  raftgpu_step_wait completes the oldest. */
#define RAFTGPU_STEP_READ_COMMITTED 0x1u /* also copy back the new committed index of advanced groups */
#define RAFTGPU_STEP_READ_RESULTS 0x2u   /* also copy back the per-record result bytes */
/* raftgpu_step_begin_records only: return as soon as the staging threads have the batch; packing, the H2D copies
 * and the kernel launches are queued by the arena's submitter thread.  `records` must then stay untouched until
 * this step's raftgpu_step_wait returns, a submission error is reported by that raftgpu_step_wait, and until
 * then the only arena calls allowed are raftgpu_step_wait and the next raftgpu_step_begin_* (which first waits
 * for the pending submission).  This overlaps ALL host work of tick j+1 with the GPU work of tick j. */
#define RAFTGPU_STEP_ASYNC 0x4u
/* raftgpu_step_begin_records only: ship the 24-byte records AS THEY ARE (one H2D straight from the caller's buffer,
 * which should be pinned: raftgpu_host_alloc) and apply them with the scatter kernel -- no host packing at all.
 * 3.7x the PCIe bytes of the compact stream, zero CPU: the better choice when the caller's CPU share is small
 * (several GPUs per socket: packing is CPU-bound, DESIGN.md 4/7).  Contract of
 * the zero-copy paths: at most ONE record per (group, peer) cell, verified on the GPU (a duplicate is not applied,
 * counted in n_duplicates, raftgpu_step_wait returns RAFTGPU_ERR_INVALID); `records` stays untouched until the
 * step's raftgpu_step_wait returns. */
#define RAFTGPU_STEP_RAW 0x8u
/* raftgpu_step_begin_records only, `records` in PINNED host memory (ignored otherwise, and with RAFTGPU_STEP_RAW or
 * RAFTGPU_STEP_READ_RESULTS): HYBRID staging.  Packing costs host CPU time, the raw form costs PCIe time; with few
 * staging threads per GPU (eight GPUs share the host's cores) neither alone keeps up.  The library packs the first
 * part of the batch (cut at a group boundary) into the compact stream while the DMA engine ships the rest as 24-byte
 * records straight from the caller's buffer, sized so that both finish together (model: RAFTGPU_HYBRID_PACK_NS per
 * record and thread, and RAFTGPU_HYBRID_PCIE_GBS: both measured on every step unless set; or RAFTGPU_HYBRID_PACK_PCT to fix the
 * split).  The batch must be in group order with at most ONE record per (group, peer) cell in its tail (a tick with
 * several acknowledgements per peer belongs to the plain form, whose fused kernel walks them in order); both are
 * verified on the device and a violation fails the step's raftgpu_step_wait.  The raw part goes through the scatter kernel, then the
 * fused kernel applies the packed part and recomputes every group.  `records` must stay untouched until
 * raftgpu_step_wait returns. */
#define RAFTGPU_STEP_HYBRID 0x10u
int32_t raftgpu_step_begin(raftgpu_arena *arena, uint32_t flags);
int32_t raftgpu_step_wait(raftgpu_arena *arena, raftgpu_step_result *out);
int32_t raftgpu_step(raftgpu_arena *arena, uint32_t flags, raftgpu_step_result *out);

/* Results of the last completed step, in arena-owned pinned memory, valid until
 * the next raftgpu_step_wait.  While two steps are in flight the third staging set,
 * which held them, stages the next batch: from the begin that leaves two in flight
 * until the next wait this call returns RAFTGPU_ERR_INVALID, as do
 * raftgpu_step_slot_results, raftgpu_step_record_results and raftgpu_step_send_list.
 * adv_bitmap has bit g set iff group g advanced
 * (LightReady.commit_index, raw_node.rs:643-650); committed[g] is meaningful
 * for advanced groups when RAFTGPU_STEP_READ_COMMITTED was set. */
int32_t raftgpu_step_results(raftgpu_arena *arena, const uint32_t **adv_bitmap,
                             const uint64_t **committed);
/* Per-record result bytes (RAFTGPU_RES_*) of the last completed step for the
 * records enqueued on `ring`, in that ring's enqueue order (EXT records get 0);
 * needs RAFTGPU_STEP_READ_RESULTS.  *out_n = records enqueued on the ring; with
 * out == NULL only the count is returned. */
int32_t raftgpu_step_record_results(raftgpu_arena *arena, uint32_t ring, uint8_t *out,
                                    uint64_t out_capacity, uint64_t *out_n);

/* ---- post-commit send decisions (SURVEY 8(f) rank 2) --------------------- */

/* The step right after the path: when a group's commit index advanced the leader calls
 * bcast_append (raft.rs:1745-1748, 1012-1013 -> raft.rs:857-865), i.e. send_append for every
 * peer but itself, and maybe_send_append drops the paused ones first (raft.rs:780-788;
 * Progress::is_paused, progress.rs:210-216: Probe -> paused, Replicate -> ins.full(),
 * Snapshot -> always).  raftgpu_send_list_device turns the advanced bitmap of a step into that
 * work list -- one entry per (group, peer) the host has to build a MsgAppend for -- with a
 * stream-compaction kernel: groups [first, first+n) whose bit is set in d_adv_bitmap (NULL = every
 * group: a plain bcast_append), peers = voters and learners of the group except its own slot.
 * Entries come out in no particular order (neither does HashMap iteration in the reference).
 * *d_count = number of entries the pass produced (u64, zeroed here first); entries beyond
 * `capacity` are dropped, so count > capacity means "call again with a larger buffer". */
typedef struct raftgpu_send_entry {
    uint32_t group;
    uint8_t peer_slot;
    uint8_t flags;     /* RAFTGPU_SEND_SNAPSHOT */
    uint16_t reserved;
    uint64_t next_idx; /* Progress::next_idx: entries from here (raft.rs:799) */
} raftgpu_send_entry;
/* pending_request_snapshot != INVALID_INDEX: prepare_send_snapshot comes first (raft.rs:792-797) */
#define RAFTGPU_SEND_SNAPSHOT 0x1u
int32_t raftgpu_send_list_device(raftgpu_arena *arena, void *stream, uint32_t first, uint32_t n,
                                 const uint32_t *d_adv_bitmap, raftgpu_send_entry *d_out, uint64_t capacity,
                                 uint64_t *d_count);
/* The same for the last completed step (its advanced bitmap, all allocated groups), entries
 * copied to host memory; synchronous.  The pause flags and next_idx are read when the kernel runs:
 * call it before the NEXT step is submitted if the list has to reflect exactly this step.  RAFTGPU_ERR_FULL (with *out_n = the number needed) when
 * `capacity` is too small. */
int32_t raftgpu_step_send_list(raftgpu_arena *arena, raftgpu_send_entry *out, uint64_t capacity, uint64_t *out_n);

/* ---- heartbeat commits (SURVEY 8(f) rank 3, leader side) ------------------- */

/* bcast_heartbeat (raft.rs:875-889) calls send_heartbeat for every peer but the leader itself, and
 * send_heartbeat attaches commit = min(pr.matched, raft_log.committed) (raft.rs:826-848: the
 * leader must not forward a follower's commit past what that follower has).  One dense pass
 * over groups [first, first+n): d_out[slot * n + (g - first)] = that commit for every present
 * peer (voter or learner) other than the group's own slot, RAFTGPU_NO_HEARTBEAT elsewhere. */
#define RAFTGPU_NO_HEARTBEAT UINT64_MAX
int32_t raftgpu_heartbeat_commits_device(raftgpu_arena *arena, void *stream, uint32_t first, uint32_t n,
                                         uint64_t *d_out);

/* ---- wire decode (SURVEY 8(f) rank 4) ------------------------------------- */

/* The step from what a transport holds: serialized eraftpb.Message frames (proto/proto/eraftpb.proto:71-92;
 * the reference decodes them with rust-protobuf / prost before RawNode::step, raw_node.rs:402-411).  The host
 * appends frames and their end offsets and parses NOTHING; the GPU decodes the varints and runs the same
 * per-message prefix of handle_append_response (raft.rs:1663-1743) + Raft::maybe_commit.
 *      frame i = bytes[offsets[i], offsets[i+1]) = u32 little-endian (group << 4 | peer_slot), then the Message
 * offsets[0..n] ascend.  Per frame one status byte comes back: RAFTGPU_WIRE_* << 4 | RAFTGPU_RES_* (the latter
 * for applied frames).  Frames the device cannot decide are NOT applied and are the host's to handle: */
#define RAFTGPU_WIRE_OK 0u         /* a MsgAppendResponse, applied (low nibble: RAFTGPU_RES_*) */
#define RAFTGPU_WIRE_SKIP_TYPE 1u  /* any other MessageType: Raft::step on the host */
#define RAFTGPU_WIRE_TERM 2u       /* m.term != the group's term (raftgpu_group_set_term; 0 = not checked): Raft::step's term rules */
#define RAFTGPU_WIRE_NEEDS_LOG 3u  /* reject with log_term > 0: next_probe_index = find_conflict_by_term(..) needs the leader's
                                      log (raft.rs:1562-1661); the host computes it and submits the 24-byte REJECT + EXT records.
                                      On an arena with leader runs (raftgpu_arena_enable_leader_runs) only the rejections
                                      the stated runs cannot decide come back so.
                                      At raftgpu_follower_append: a MsgAppend with entries, or whose answer needs a term of
                                      the follower's log outside the caller's run (and, on an arena with follower runs,
                                      outside the row's two runs below it): RawNode::step on the host */
#define RAFTGPU_WIRE_MALFORMED 4u  /* not a protobuf message, a bad frame, or a group that is not allocated */
#define RAFTGPU_WIRE_DUP 5u        /* a later frame of a (group, peer) cell that already has one in this batch: cells are
                                      applied in arrival order, one message per step -- resubmit it with the next batch */
#define RAFTGPU_WIRE_CONTEXT 6u    /* (raftgpu_heartbeat_wire only) a context that is not an 8-byte read id, or any context
                                      on an arena without read queues: the host's own ReadOnly handles the frame */
#define RAFTGPU_WIRE_ROLE 7u       /* (raftgpu_follower_heartbeat, raftgpu_follower_append, raftgpu_vote_wire,
                                      raftgpu_vote_request_wire, raftgpu_follower_term_wire) the group is not selected for the role the pass serves,
                                      or is a leader; at raftgpu_vote_wire also a response type that is not the
                                      candidate's own (step_candidate ignores it); at raftgpu_leader_term_wire the group
                                      is not a leader; at raftgpu_follower_response_wire it is unselected or a leader;
                                      at raftgpu_leader_vote_request_wire the group is not a leader: Raft::step on the
                                      host */
#define RAFTGPU_WIRE_COMMIT_RANGE 8u /* (raftgpu_follower_heartbeat, raftgpu_follower_append) the commit_to the frame asks
                                        for -- m.commit, or min(m.commit, m.index) of a matching MsgAppend -- beyond
                                        max(committed, last_index): commit_to would be fatal! (raft_log.rs:291-298) */
#define RAFTGPU_WIRE_COMMIT_VOTE 9u  /* (raftgpu_vote_wire, raftgpu_vote_request_wire, raftgpu_leader_vote_request_wire)
                                        m.commit != 0, m.commit_term != 0 and m.commit beyond committed -- at the vote
                                        request passes for a rejected request (at a leader: one that deposes it):
                                        maybe_commit_by_vote (raft.rs:2126-2164) needs the caller's log */
#define RAFTGPU_WIRE_IGNORED 10u     /* (raftgpu_vote_request_wire, raftgpu_leader_vote_request_wire,
                                        raftgpu_leader_term_wire, raftgpu_follower_response_wire)
                                        the reference drops the frame: a vote request in lease (raft.rs:1288-1316) or a
                                        MsgRequestVote at a lower term (:1399-1409); a frame step_leader, step_candidate
                                        or step_follower has no arm for */
#define RAFTGPU_WIRE_STALE 11u       /* (raftgpu_follower_term_wire, raftgpu_leader_term_wire,
                                        raftgpu_follower_response_wire) m.term below the group's (new)
                                        term: settled by the pass, which answered it when the low nibble is
                                        RAFTGPU_RES_OK; drop the frame */
typedef struct raftgpu_wire_batch {
    const uint8_t *bytes;    /* the frames, back to back */
    uint64_t n_bytes;
    const uint32_t *offsets; /* [n + 1] */
    uint64_t n;              /* frames */
    /* 24-byte records that travel with the batch and are applied BEFORE the frames: the leader's own
     * RAFTGPU_REC_LOCAL events (append_entry / on_persist_entries are calls, not messages) and REJECTs whose
     * next_probe_index the host has resolved (RAFTGPU_WIRE_NEEDS_LOG of an earlier step).  At most one
     * record per (group, peer) cell, verified on the GPU like raftgpu_step_begin_packed.  May be NULL / 0.
     * On an arena with leader runs, a rejection the runs decide is applied from its frame and needs no record. */
    const raftgpu_append_resp *records;
    uint64_t n_records;
} raftgpu_wire_batch;
/* Raft::term (raft.rs:227) of a group, for the wire path's term test; 0 (the initial value) = the caller filters. */
int32_t raftgpu_group_set_term(raftgpu_arena *arena, uint32_t group, uint64_t term);
/* Decode + apply for a batch that already sits in device memory (d_bytes 16-byte aligned, d_offsets [n + 1]);
 * d_status [n] is required.  Two kernels (scan: classify + first frame of every cell; apply), asynchronous on
 * `stream`; run raftgpu_recompute afterwards for Raft::maybe_commit. */
int32_t raftgpu_wire_apply_device(raftgpu_arena *arena, void *stream, const void *d_bytes, uint64_t n_bytes,
                                  const uint32_t *d_offsets, uint64_t n, uint8_t *d_status);
/* One step from a wire batch in host memory (pinned -- raftgpu_host_alloc -- for an asynchronous copy): H2D of
 * bytes + offsets, decode + apply, the recompute pass, D2H of the results and the status bytes.  Same
 * begin / wait protocol and result accessors as raftgpu_step_begin; the buffers must stay untouched until
 * raftgpu_step_wait returns.  raftgpu_step_wire_status: the status bytes of the last completed wire step. */
int32_t raftgpu_step_begin_wire(raftgpu_arena *arena, const raftgpu_wire_batch *batch, uint32_t flags);
int32_t raftgpu_step_wire_status(raftgpu_arena *arena, const uint8_t **status, uint64_t *n);

/* ---- waves: pipelined frames of one cell or group in one call -------------- */

/* A leader sends as many MsgAppend to a peer as its inflight window allows (raft.rs:1755-1761), so one received batch
 * may hold several MsgAppend for one follower group, and several MsgAppendResponse for one leader cell.  At `waves` = k
 * the passes below decide up to k of them per cell (the wire step: raftgpu_wire_apply_device, raftgpu_step_begin_wire)
 * or per group (raftgpu_follower_append[_device], raftgpu_follower_append_entries[_device]) in one call, in arrival
 * order.  Let F1 be every frame of the batch; run j is the pass as it is at one wave, over the frames Fj in their batch
 * order; a call at k waves returns what up to k runs return:
 *   - the wire step: Fj+1 = the frames run j returned RAFTGPU_WIRE_DUP (a frame that is not OK claims no cell: the
 *     host's resubmission with no host work between);
 *   - the follower's append passes: Fj+1 = the frames run j returned DUP, but for those of groups whose claiming frame in
 *     run j was RAFTGPU_WIRE_NEEDS_LOG or RAFTGPU_WIRE_COMMIT_RANGE: they stay DUP, as the host handles the claimant
 *     first.  A frame of a later run is decided against the group's state after the earlier runs: committed,
 *     last_index and (the _device form with entries) the table's run.
 * A frame's status byte is that of the last run that saw it (a frame still DUP after run k stays DUP); its `from` and
 * appended record come from the run that decided it, zero for a frame left DUP.  The responses of every run go to one
 * output in frame order, the totals summed: a frame is answered at most once, so raftgpu_follower_append_bound(n)
 * still bounds them.  The wire step runs one Raft::maybe_commit pass after the last run; its counters count every run.
 *
 * 1 (the default) is the passes as they are.  Each wave costs two kernel launches whether or not it finds frames, so
 * k bounds the cost of a call; a cell or group with more frames than k gets DUP for the rest.  The heartbeat and vote
 * passes keep one frame per cell or group: they bring at most one message per peer per tick or election.
 * raftgpu_arena_set_wire_waves takes effect for the calls queued after it (a step already begun keeps its value);
 * RAFTGPU_ERR_INVALID for a NULL arena, 0 or more than RAFTGPU_WIRE_WAVES_MAX. */
#define RAFTGPU_WIRE_WAVES_MAX 64u
int32_t raftgpu_arena_set_wire_waves(raftgpu_arena *arena, uint32_t waves);

/* ---- the leader's term runs: rejections decided in the wire step ---------- */

/* A rejected MsgAppendResponse with log_term > 0 needs find_conflict_by_term(m.reject_hint, m.log_term) on the leader's
 * log (raft.rs:1562, raft_log.rs:209-235).  The arena already knows the leader's own term: term(i) = term on
 * [term_start, last_index] and 0 above last_index.  A row per group states up to two earlier term runs below
 * term_start; with it raftgpu_wire_apply_device and raftgpu_step_begin_wire decide such a frame on the device whenever
 * the walk ends inside what is known, and apply it as RAFTGPU_WIRE_OK with the result as next_probe_index.  The others
 * stay RAFTGPU_WIRE_NEEDS_LOG, handled by the host as before.  Accepts never read the rows.
 *
 * A row is used only while its group is a leader (term_start != RAFTGPU_NO_TERM_START) with a non-zero term and
 * (term, term_start) equal the row's anchor; any call that changes either (reset, become_leader, set_log_bounds,
 * set_term, a vote-request pass's become_follower, ...) leaves the row inert until it is stated again.  Group alloc and
 * free clear the row.  A wide pair's row is stated on its low half and read with the pair's term_start and the larger
 * last_index.
 *
 * Opt-in: call before groups are allocated.  Memory: 48 bytes per group slot (48 MB per million).  An arena that does
 * not call it behaves exactly as without the feature. */
int32_t raftgpu_arena_enable_leader_runs(raftgpu_arena *arena);

/* One group's row: 56 bytes.  Run 1 is [run_start[0], term_start - 1] at run_term[0], run 2 is [run_start[1],
 * run_start[0] - 1] at run_term[1]; a run_start of 0 states no run.  Every stated run must still be readable by the
 * leader's RaftLog::term (at or above first_index - 1): on compaction, restate the row or drop runs.  Fewer runs are
 * never wrong; they leave more frames to the host. */
typedef struct raftgpu_leader_runs {
    uint32_t group;        /* the group (the low half of a wide pair) */
    uint32_t reserved;     /* ignored */
    uint64_t term;         /* the anchor: Raft::term and term_start of the leadership the runs belong to */
    uint64_t term_start;
    uint64_t run_start[2];
    uint64_t run_term[2];
} raftgpu_leader_runs;

/* State rows for many groups (a store-wide election: right after the raftgpu_control list that makes them leaders, in
 * either order).  status[i] per row, and a refused row is not stored:
 *   RAFTGPU_ERR_RANGE    the group is not allocated, or is the high half of a wide pair;
 *   RAFTGPU_ERR_INVALID  term is 0, term_start is 0 or RAFTGPU_NO_TERM_START, run 2 without run 1, starts that do not
 *                        satisfy 0 < run_start[1] < run_start[0] < term_start where stated, or run terms that do not
 *                        satisfy 0 < run_term[1] < run_term[0] < term where stated.
 * Returns RAFTGPU_OK when the list ran (n == 0 included), RAFTGPU_ERR_INVALID for an arena without leader runs or a
 * NULL rows / status with n > 0.  The rows take effect at the call, in submission order with steps in flight (like
 * the control calls); synchronous.  A later row of the same group wins. */
int32_t raftgpu_leader_runs_set(raftgpu_arena *arena, const raftgpu_leader_runs *rows, uint64_t n, int32_t *status);

/* ---- heartbeat responses (SURVEY 8(f) rank 3, response side) ---------------- */

/* The tracker part of Raft::handle_heartbeat_response (raft.rs:1777-1804) for a batch of RAFTGPU_REC_HEARTBEAT
 * records: pr.update_committed(m.commit), recent_active = true, resume(), a full inflights window of a
 * Replicate peer frees its first entry (INS_FULL clears), and the result byte says whether the reference would
 * call send_append: RAFTGPU_RES_OK | RAFTGPU_RES_SEND when pr.matched < last_index or a snapshot was requested
 * (raft.rs:1800-1803); RAFTGPU_RES_NO_PROGRESS for an unknown peer.  The read-index tail (:1806-1818) is
 * raftgpu_read_index_ack over the same records (RAFTGPU_REC_READ_CTX, ignored here).  A heartbeat batch is its own pass, ordered by the caller between steps (it reads last_index,
 * which a step's LOCAL records write): "all heartbeat responses of the tick after its append responses" is
 * one of the delivery orders raft allows.  One record per (group, peer) cell; a second one is not applied,
 * gets result 0 and -- in the host form -- makes the call return RAFTGPU_ERR_INVALID.
 * _device: records and results in device memory, asynchronous on `stream` (d_dup_count nullable, u32, zeroed by
 * the caller); the host form copies, runs and waits. */
int32_t raftgpu_heartbeat_resp_device(raftgpu_arena *arena, void *stream, const raftgpu_append_resp *d_records,
                                      uint64_t n, uint8_t *d_results, uint32_t *d_dup_count);
int32_t raftgpu_heartbeat_resp(raftgpu_arena *arena, const raftgpu_append_resp *records, uint64_t n, uint8_t *results);

/* Progress::update_state(last) (progress.rs:231-243) for a list of MsgAppends the host has just built -- the
 * follow-up of every send-list entry (raft.rs:753-760): a Replicate peer's next_idx jumps to last + 1
 * (optimistic_update; the matching ins.add(last) is the host's Inflights), a Probe peer is paused until its
 * next response.  entries[i].next_idx carries `last`, the index of the last entry sent to that peer.
 * results[i] (nullable): 1 done, 0xff where the reference panics (a Snapshot-state peer), RAFTGPU_RES_NO_PROGRESS. */
int32_t raftgpu_update_state_device(raftgpu_arena *arena, void *stream, const raftgpu_send_entry *d_entries, uint64_t n,
                                    uint8_t *d_results);
int32_t raftgpu_update_state(raftgpu_arena *arena, const raftgpu_send_entry *entries, uint64_t n, uint8_t *results);

/* ---- Inflights on the device (SURVEY 8(f) rank 2) --------------------------- */

/* Keep every peer's Inflights window (src/tracker/inflights.rs:19-110: the last index of each in-flight MsgAppend, a
 * ring of Config::max_inflight_msgs entries, config.rs:112) in HBM, so that nothing about flow control is left to
 * per-message host work: raftgpu_update_state adds (progress.rs:231-236), an accepted append response frees up to
 * its index (raft.rs:1742), a heartbeat response frees the first entry of a full window (raft.rs:1796-1798), every
 * state change resets (progress.rs:75-80), and RAFTGPU_PF_INS_FULL -- what Progress::is_paused reads in Replicate
 * state -- mirrors ins.full() (raftgpu_progress.ins_full is then an output only).  Call before groups are
 * allocated.  Memory: 8 slots x max_groups x max_inflight x 8 bytes (256 entries: 16 KB per group), which is why
 * it is opt-in.  With windows on, steps run through the scatter kernels (the fused tile kernels keep their rows in
 * shared memory and do not carry the rings): raftgpu_step_sorted_device / raftgpu_step_compact_device return
 * RAFTGPU_ERR_INVALID, every raftgpu_step_begin_* form works. */
int32_t raftgpu_arena_enable_inflights(raftgpu_arena *arena, uint32_t max_inflight);
/* One peer's window: *start, *count (inflights.rs:21-23) and, when buffer != NULL, its `capacity` ring entries. */
int32_t raftgpu_inflights_get(raftgpu_arena *arena, uint32_t group, uint32_t peer_slot, uint32_t *start, uint32_t *count,
                              uint64_t *buffer, uint32_t capacity);

/* ---- ReadIndex, ReadOnlyOption::Safe (SURVEY 8(f) rank 3, read side) -------- */

/* The leader side of MsgReadIndex (raft.rs:2056-2091) and the read-index tail of Raft::handle_heartbeat_response
 * (raft.rs:1805-1818) as batched device passes: each group's ReadOnly (read_only.rs:86-139) is a queue in HBM.
 * Contexts are opaque bytes in the reference; here they are u64 context ids the caller assigns (equal bytes, equal
 * id; 0 = no context, m.context.is_empty()), and the caller keeps id -> (bytes, original Message) for
 * handle_ready_read_index (raft.rs:2790-2805).  A pending read's acks are a 16-bit peer-slot mask (a wide group's
 * peer 8 + s is bit 8 + s); the self bit is set when it is queued.  Deviations from the reference, both documented
 * in DESIGN.md 3.9: the queue holds at most max_pending reads (RAFTGPU_READ_FULL; the reference's is unbounded),
 * and a peer removed by a configuration change loses its acks (a peer removed and re-added while a read is
 * pending must ack again; this can delay a read, never release one early).  The queue of a wide group lives on
 * its low half.
 *
 * Opt-in, like device-side Inflights: call before groups are allocated.  Memory: max_pending x 18 bytes + 16 per
 * group slot (8 pending reads: about 160 bytes).  Arenas that do not call it behave exactly as without the feature;
 * the step kernels never read the queues, so every step form (the fused tile kernels included) stays available. */
#define RAFTGPU_READ_MAX_PENDING 64u
int32_t raftgpu_arena_enable_read_index(raftgpu_arena *arena, uint32_t max_pending);

/* RAFTGPU_REC_HEARTBEAT records with this flag carry the response's context id in `index` (0 = none).
 * raftgpu_heartbeat_resp[_device] ignores the bit, so the tracker pass and the read pass can run over the same
 * device buffer. */
#define RAFTGPU_REC_READ_CTX 0x08u

/* One MsgReadIndex at the leader: 16 bytes. */
typedef struct {
    uint32_t group;     /* the group id (the low half of a wide group) */
    uint32_t reserved;
    uint64_t ctx;       /* context id, non-zero */
} raftgpu_read_req;
/* One released read (ReadIndexStatus minus the message, read_only.rs:58-63): 24 bytes. */
typedef struct {
    uint32_t group;
    uint32_t reserved;
    uint64_t ctx;
    uint64_t index;     /* the commit index the read was queued with */
} raftgpu_read_state;

/* per-request result byte */
#define RAFTGPU_READ_QUEUED 1u   /* add_request: a new entry at the back of the queue, acks = {self} */
#define RAFTGPU_READ_READY 2u    /* is_singleton(): released at once with index = committed (raft.rs:2064-2070) */
#define RAFTGPU_READ_DUP 3u      /* the ctx is already pending: nothing changes (read_only.rs:89-91); the reference
                                    still broadcasts the heartbeat */
#define RAFTGPU_READ_DROPPED 4u  /* !commit_to_current_term() (raft.rs:2057-2062): term_start <= committed <=
                                    last_index does not hold (a non-leader's requests are always dropped) */
#define RAFTGPU_READ_FULL 5u     /* the queue already holds max_pending reads: resubmit after a release */
#define RAFTGPU_READ_NO_GROUP 6u /* an unallocated group, or the high half of a wide group */
#define RAFTGPU_READ_NO_CTX 7u   /* ctx == 0: 0 is "no context" and cannot be acked */

/* Requests (raft.rs:2056-2091) for many groups: d_reqs in non-decreasing group order (queue order is arrival
 * order), verified on the device before anything is applied -- on a violation nothing is applied, every result
 * is 0 and *d_bad (u32, nullable) is bumped once.  d_results (n bytes, nullable) gets RAFTGPU_READ_*; READY reads
 * go to d_released, *d_count (u64) = how many (zeroed here first).  capacity must be at least n
 * (RAFTGPU_ERR_INVALID before any launch otherwise): a release cannot be regenerated.  Asynchronous on `stream`. */
int32_t raftgpu_read_index_request_device(raftgpu_arena *arena, void *stream, const raftgpu_read_req *d_reqs, uint64_t n,
                                          uint8_t *d_results, raftgpu_read_state *d_released, uint64_t capacity,
                                          uint64_t *d_count, uint32_t *d_bad);
/* Host form: copies, runs and waits; RAFTGPU_ERR_INVALID (nothing applied) when the requests are out of group
 * order; *out_n = released reads copied to `released`. */
int32_t raftgpu_read_index_request(raftgpu_arena *arena, const raftgpu_read_req *reqs, uint64_t n, uint8_t *results,
                                   raftgpu_read_state *released, uint64_t capacity, uint64_t *out_n);

/* The read-index tail of handle_heartbeat_response (raft.rs:1805-1818) for a batch of RAFTGPU_REC_HEARTBEAT |
 * RAFTGPU_REC_READ_CTX records (every other record is ignored, and so is a responder without Progress or ctx 0):
 * recv_ack (read_only.rs:104-110) ORs the responder's bit into its ctx's pending entry, then per group the last
 * entry that a record named and whose acks have a quorum (ProgressTracker::has_quorum, tracker.rs:367-372) is
 * advanced to (read_only.rs:115-129): it and every entry in front of it are released, contiguously and in queue
 * order.
 * Any number of records per cell, in any order: the result is what applying them one at a time in any order
 * gives (DESIGN.md 3.9).  *d_count (u64) = released reads, zeroed here first.  capacity must be at least
 * min(n, allocated groups) x max_pending (RAFTGPU_ERR_INVALID before any launch otherwise), so a release is never
 * lost.  Asynchronous on `stream`. */
int32_t raftgpu_read_index_ack_device(raftgpu_arena *arena, void *stream, const raftgpu_append_resp *d_records, uint64_t n,
                                      raftgpu_read_state *d_released, uint64_t capacity, uint64_t *d_count);
int32_t raftgpu_read_index_ack(raftgpu_arena *arena, const raftgpu_append_resp *records, uint64_t n,
                               raftgpu_read_state *released, uint64_t capacity, uint64_t *out_n);

/* The tail of post_conf_change (raft.rs:2648-2664) for the listed groups (a group listed twice counts once):
 * recv_ack(self, last pending ctx) and, when the new configuration gives that entry a quorum, every pending read
 * is released.  List only groups whose configuration just changed: on any other group it could release a read
 * the reference would not.  capacity must be at least n x max_pending.  Synchronous. */
int32_t raftgpu_read_index_recheck(raftgpu_arena *arena, const uint32_t *groups, uint64_t n, raftgpu_read_state *out,
                                   uint64_t capacity, uint64_t *out_n);

/* ReadOnly::last_pending_request_ctx (read_only.rs:132-135) for groups [first, first + n): the ctx bcast_heartbeat
 * attaches (raft.rs:876), d_out[g - first] = 0 for none.  Asynchronous on `stream`. */
int32_t raftgpu_read_index_last_ctx_device(raftgpu_arena *arena, void *stream, uint32_t first, uint32_t n, uint64_t *d_out);

/* Inspection: one group's pending reads in queue order (*count = pending_read_count, raft.rs:437; up to
 * `capacity` entries of ctx / index / acks, each nullable), and the same for groups [first, first + n) at once:
 * counts[n], and ctx / index / acks as [n][max_pending] (group i's entry k at i * max_pending + k). */
int32_t raftgpu_read_index_get(raftgpu_arena *arena, uint32_t group, uint32_t *count, uint64_t *ctx, uint64_t *index,
                               uint16_t *acks, uint32_t capacity);
int32_t raftgpu_read_index_read(raftgpu_arena *arena, uint32_t first, uint32_t n, uint32_t *counts, uint64_t *ctx,
                                uint64_t *index, uint16_t *acks);

/* ---- heartbeat responses from the wire ---------------------------------------- */

/* Raft::handle_heartbeat_response (raft.rs:1777-1819) for the MsgHeartbeatResponse frames (msg_type 9) of a wire
 * batch, in the format of raftgpu_wire_batch (u32 LE group << 4 | peer_slot, then the serialized Message; peer
 * 8 + s of a wide group is cell (g + 1, s)).  The context of a heartbeat that carries read id x is the 8 bytes of x,
 * little-endian (the caller builds the heartbeat; the follower echoes its context, raft.rs:2461).  Field 12 decodes
 * as a parser does: the last length-delimited occurrence wins, a varint field 12 is skipped.  Per frame:
 *   - no context: the tracker part, exactly raftgpu_heartbeat_resp for a RAFTGPU_REC_HEARTBEAT record with
 *     commit = m.commit;
 *   - an 8-byte context on an arena with read queues: the tracker part, and the read part, exactly
 *     raftgpu_read_index_ack for the same record with RAFTGPU_REC_READ_CTX and the id in `index` (id 0 acks nothing);
 *   - any other context, or any context on an arena without read queues: RAFTGPU_WIRE_CONTEXT, nothing applied.
 * status[i] = RAFTGPU_WIRE_* << 4 | RAFTGPU_RES_* (RAFTGPU_RES_OK [| RAFTGPU_RES_SEND] or RAFTGPU_RES_NO_PROGRESS for
 * an applied frame).  RAFTGPU_WIRE_SKIP_TYPE for every other message type (MsgAppendResponse included: the same
 * bytes can go through raftgpu_wire_apply_device as well, and each frame is applied by exactly one of the two),
 * RAFTGPU_WIRE_TERM, RAFTGPU_WIRE_MALFORMED and RAFTGPU_WIRE_DUP (a later frame of a cell that already has one in the
 * batch) as for the AppendResponse path.  A frame is applied whole or not at all: a DUP, TERM, CONTEXT or MALFORMED
 * frame touches neither the tracker nor the read queue; the host may deliver it later.  Like raftgpu_heartbeat_resp,
 * the pass runs between steps (it reads last_index).
 * Released reads go to d_released, *d_count (u64) = how many, zeroed here first; capacity must be at least
 * min(n, allocated groups) x max_pending (RAFTGPU_ERR_INVALID before any launch otherwise).  On an arena without read
 * queues d_released / capacity / d_count may be NULL / 0.  d_bytes 16-byte aligned, n and n_bytes below 4 GiB.
 * Asynchronous on `stream`.  The pass keeps its own decode scratch (not a staging set's) and shares the read
 * passes' per-group scratch: run it on one stream with the other read-index passes. */
int32_t raftgpu_heartbeat_wire_device(raftgpu_arena *arena, void *stream, const void *d_bytes, uint64_t n_bytes,
                                      const uint32_t *d_offsets, uint64_t n, uint8_t *d_status,
                                      raftgpu_read_state *d_released, uint64_t capacity, uint64_t *d_count);
/* Host form: copies, runs and waits; status (n bytes) nullable; *out_n = released reads copied to `released`
 * (released / capacity / out_n may be NULL / 0 on an arena without read queues). */
int32_t raftgpu_heartbeat_wire(raftgpu_arena *arena, const void *bytes, uint64_t n_bytes, const uint32_t *offsets, uint64_t n,
                               uint8_t *status, raftgpu_read_state *released, uint64_t capacity, uint64_t *out_n);

/* ---- heartbeats to the wire ---------------------------------------------------- */

/* Raft::ping / MsgBeat -> bcast_heartbeat (raft.rs:868-889) -> send_heartbeat (raft.rs:822-844) -> send (raft.rs:602-661)
 * for groups [first, first + n), as serialized MsgHeartbeat frames ready for the transport.  A read-only pass: the
 * tracker and the read queues are not changed.
 *
 * Selection.  d_select is a bitmap in the layout of d_adv_bitmap (bit g = group g, words counted from group 0); NULL =
 * every group of the range.  A selected group sends only when it is allocated, a leader (term_start !=
 * RAFTGPU_NO_TERM_START) and its term (raftgpu_group_set_term) is non-zero.  A leader whose term is 0 sends nothing --
 * a term-less heartbeat would be read as a local message -- and is counted in totals[2], so a missing
 * raftgpu_group_set_term shows; a non-leader is skipped silently, as `ping` skips it.
 * Peers.  One MsgHeartbeat per present peer (voter of either half of a joint configuration, or learner) other than
 * the group's own slot.  The ids are the caller's (the arena keeps slots): d_ids is u64 [RAFTGPU_SLOTS + 1][n], row
 * s < 8 = the id of the peer in slot s of group first + i, row 8 = that group's Raft::id, the `from` (a leader that
 * has removed itself has no self slot and still sends).
 * Wide groups.  Peer 8 + s is cell (g + 1, s), as in the wire batches.  Selection bit, term, term_start, the `from`
 * (row 8) and the context are the low half's; commit uses committed = max of both halves (what raftgpu_group_get
 * reports).  A range that splits a wide group is RAFTGPU_ERR_INVALID before any launch.
 * The message: msg_type = MsgHeartbeat (8), to, from, term = Raft::term, commit = min(pr.matched, committed) and, on
 * an arena with read queues whose queue is not empty, context = the 8 little-endian bytes of the last pending ctx id
 * (read_only.rs:132-135: what raftgpu_heartbeat_wire decodes); no context otherwise.  Canonical proto3 encoding of
 * eraftpb.Message, fields in number order, zero scalars omitted: at most 56 bytes.
 * Output.  The frames of raftgpu_wire_batch: u32 LE (group << 4 | peer_slot), then the Message; in ascending
 * (group, slot) order, so the output is deterministic.  d_bytes (16-byte aligned, so the blob can go to the wire
 * entry points as is) holds the frames back to back; d_offsets [frames + 1] their starts and the end, d_offsets[0] =
 * 0.  d_totals (u64[3]) = {frames, bytes, leaders without a term}, always the full need.  When frames >
 * frames_capacity (d_offsets has room for frames_capacity + 1 values) or bytes > bytes_capacity, NOTHING is written to
 * d_bytes or d_offsets; the pass only reads state, so calling again with larger buffers is always safe.
 * raftgpu_heartbeat_frames_bound(n) is enough for any n groups; a range whose bound exceeds what u32 offsets address
 * is RAFTGPU_ERR_INVALID.
 * Ordering.  The pass reads matched and committed, which steps write: order it against steps on the stream, as for
 * raftgpu_heartbeat_commits_device.  _device: asynchronous on `stream`, with its own scratch in the arena (run it on
 * one stream at a time).  The host form copies select / ids, runs and waits: RAFTGPU_ERR_FULL with *out_totals filled
 * in when a capacity is short. */
/* Worst-case bytes of raftgpu_heartbeat_frames* output for n group slots (8 frames x 60 bytes per slot). */
uint64_t raftgpu_heartbeat_frames_bound(uint32_t n);
int32_t raftgpu_heartbeat_frames_device(raftgpu_arena *arena, void *stream, uint32_t first, uint32_t n,
                                        const uint32_t *d_select, const uint64_t *d_ids,
                                        uint8_t *d_bytes, uint64_t bytes_capacity,
                                        uint32_t *d_offsets, uint64_t frames_capacity, uint64_t *d_totals);
int32_t raftgpu_heartbeat_frames(raftgpu_arena *arena, uint32_t first, uint32_t n, const uint32_t *select,
                                 const uint64_t *ids, uint8_t *bytes, uint64_t bytes_capacity, uint32_t *offsets,
                                 uint64_t frames_capacity, uint64_t *out_totals);

/* ---- the commit broadcast to the wire -------------------------------------------- */

/* Raft::maybe_commit -> bcast_append (raft.rs:1745-1748, 857-865) -> send_append -> maybe_send_append(to, allow_empty =
 * true) (raft.rs:764-819) -> prepare_send_entries (raft.rs:714-730) -> send (raft.rs:602-661) for groups [first,
 * first + n), split by what the leader's log has to add: the entry-less MsgAppend frames, ready for the transport, and
 * a rest list of the sends that need the log.  A read-only pass: no update_state (the reference calls it only when
 * entries were sent), nothing in the arena is written.
 *
 * Selection.  As raftgpu_heartbeat_frames: d_select in the layout of d_adv_bitmap (normally the step's advanced
 * bitmap, raftgpu_step_results), NULL = every group of the range; a selected group takes part only when it is
 * allocated and a leader (term_start != RAFTGPU_NO_TERM_START); a non-leader is skipped silently, a leader whose term
 * (raftgpu_group_set_term) is 0 sends nothing and is counted in totals[3].
 * Peers.  Every present peer (voter of either half, or learner) other than the group's own slot -- the peers
 * raftgpu_send_list_device visits -- in this order:
 *   Progress::is_paused (progress.rs:210-216; with device Inflights RAFTGPU_PF_INS_FULL is the derived bit): nothing;
 *   pending_request_snapshot != RAFTGPU_INVALID_INDEX: a rest entry with RAFTGPU_SEND_SNAPSHOT;
 *   next_idx <= last_index (entries to send) or next_idx - 1 < term_start (its term needs the log): a rest entry;
 *   otherwise one MsgAppend frame: msg_type 3, to, from, term = Raft::term, log_term = the term when next_idx - 1 <=
 *   last_index and 0 above it (raft_log.rs:122-127), index = next_idx - 1, commit = committed, no entries.  Canonical
 *   proto3 encoding of eraftpb.Message, fields in number order, zero scalars omitted: at most 68 bytes.
 * The ids are the caller's: d_ids u64 [RAFTGPU_SLOTS + 1][n] as in raftgpu_heartbeat_frames (row 8 = the `from`).
 * Wide groups.  Peer 8 + s is cell (g + 1, s), its frame header (g + 1) << 4 | s.  Selection bit, term, term_start and
 * the `from` are the low half's; committed and last_index the larger of both halves' values.  A range that splits a
 * wide group is RAFTGPU_ERR_INVALID before any launch.
 * Output.  In ascending (group, slot) order each, so the output is deterministic: the frames in the format of
 * raftgpu_wire_batch (d_bytes 16-byte aligned, d_offsets [frames + 1], d_offsets[0] = 0), and d_rest, the rest list
 * as raftgpu_send_entry {group, peer_slot, RAFTGPU_SEND_SNAPSHOT or 0, next_idx}: the send list of the same selection
 * minus the peers that got a frame.  The host builds the rest list's messages from its log and then calls
 * raftgpu_update_state for those that carried entries, as it does with the send list.  d_totals (u64[4]) = {frames,
 * bytes, rest entries, leaders without a term}, always the full need.  When frames > frames_capacity, bytes >
 * bytes_capacity or rest entries > rest_capacity, NOTHING is written to d_bytes, d_offsets or d_rest; the pass only
 * reads state, so calling again with larger buffers is always safe.  raftgpu_append_frames_bound(n) bytes are enough
 * for any n groups and 8 n is enough frames or rest entries; a range whose bound exceeds what u32 offsets address is
 * RAFTGPU_ERR_INVALID.
 * Ordering.  The pass reads what steps write: order it against steps on the stream.  _device: asynchronous on
 * `stream`, with its own scratch in the arena (run it on one stream at a time).  The host form copies select / ids,
 * runs and waits, and sees the arena as if every submitted step had completed: RAFTGPU_ERR_FULL with *out_totals
 * filled in when a capacity is short. */
/* Worst-case bytes of raftgpu_append_frames* output for n group slots (8 frames x 72 bytes per slot). */
uint64_t raftgpu_append_frames_bound(uint32_t n);
int32_t raftgpu_append_frames_device(raftgpu_arena *arena, void *stream, uint32_t first, uint32_t n,
                                     const uint32_t *d_select, const uint64_t *d_ids,
                                     uint8_t *d_bytes, uint64_t bytes_capacity,
                                     uint32_t *d_offsets, uint64_t frames_capacity,
                                     raftgpu_send_entry *d_rest, uint64_t rest_capacity, uint64_t *d_totals);
int32_t raftgpu_append_frames(raftgpu_arena *arena, uint32_t first, uint32_t n, const uint32_t *select,
                              const uint64_t *ids, uint8_t *bytes, uint64_t bytes_capacity, uint32_t *offsets,
                              uint64_t frames_capacity, raftgpu_send_entry *rest, uint64_t rest_capacity,
                              uint64_t *out_totals);

/* ---- heartbeats at the follower ------------------------------------------------ */

/* RawNode::step -> Raft::step (raft.rs:1280-1411) -> step_follower (raft.rs:2276-2280) -> handle_heartbeat
 * (raft.rs:2452-2464) for the MsgHeartbeat frames (msg_type 8) of a wire batch that reach this arena's followers:
 * commit_to(m.commit) (raft_log.rs:286-300: never decreases) and one MsgHeartbeatResponse through send (raft.rs:602-661).
 * Input.  The frames of raftgpu_wire_batch, but the header is u32 LE (group << 4 | x) with `group` the follower's own
 * group slot in this arena (the transport rewrites the leader's header on the way in); x is not read and is copied
 * into the response's header.  d_bytes 16-byte aligned, n and n_bytes below 4 GiB.
 * Role.  d_select (required) is a bitmap in the layout of d_adv_bitmap: bit g set when the caller's Raft of group g is
 * a Follower (not a Candidate or PreCandidate) without a pending_request_snapshot -- host state the arena does not
 * keep.  d_self_ids (u64, indexed by group slot) holds each group's Raft::id, the `from` of its response (send takes
 * it from self.id, not from m.to).
 * Status.  status[i] = RAFTGPU_WIRE_* << 4, | RAFTGPU_RES_OK when a response was written; the first failing check decides:
 *   MALFORMED    a bad frame or protobuf, a group at or past the highest allocated slot (on an arena with read queues:
 *                any unallocated group), or the high half of a wide pair (a pair is addressed by its low half);
 *   SKIP_TYPE    any type but MsgHeartbeat;
 *   ROLE         the select bit is clear, or the group is a leader (term_start != RAFTGPU_NO_TERM_START);
 *   TERM         the group's term (raftgpu_group_set_term) is 0 or m.term differs: a higher term is become_follower, a
 *                lower one may need a MsgAppendResponse (raft.rs:1349-1376), m.term 0 is a local message;
 *   CONTEXT      a context that is present and not 8 bytes;
 *   COMMIT_RANGE m.commit > max(committed, last_index) (both halves of a wide pair);
 *   DUP          a later frame of a group whose first passing frame is applied here.
 * A frame that does not pass changes nothing: run RawNode::step on it.  d_from (u64[n], nullable) = m.from of every
 * applied frame (0 for the others), for step_follower's leader_id = m.from and election_elapsed = 0.
 * Apply.  committed = max(committed, m.commit), on both halves of a wide pair (as raftgpu_group_commit_to).
 * Output.  One MsgHeartbeatResponse per applied frame, in frame order: the input frame's header, then msg_type 9, to =
 * m.from, from = the group's id, term, commit = the new committed and, when the heartbeat had one, its 8 context bytes;
 * canonical proto3 as raftgpu_heartbeat_frames writes (at most 56 bytes + the header).  d_resp_bytes (16-byte aligned)
 * holds them back to back, d_resp_offsets (n + 1 values) their starts and the end; d_totals (u64[2]) = {responses,
 * bytes}.  A response cannot be regenerated once committed has moved, so resp_bytes_capacity must be at least
 * raftgpu_follower_heartbeat_bound(n) and that bound must be addressable by u32 offsets: RAFTGPU_ERR_INVALID before
 * any launch otherwise.
 * Ordering.  Runs between steps on `stream`, with its own scratch in the arena (run it on one stream at a time).  The
 * host form copies (select and self_ids cover the arena's max_groups; only the groups below the highest allocated one
 * are read), runs and waits; status, from, resp_bytes / resp_offsets as above, totals u64[2]. */
/* 60 bytes per frame: enough for the responses to any n frames. */
uint64_t raftgpu_follower_heartbeat_bound(uint64_t n);
int32_t raftgpu_follower_heartbeat_device(raftgpu_arena *arena, void *stream, const void *d_bytes, uint64_t n_bytes,
                                          const uint32_t *d_offsets, uint64_t n, const uint32_t *d_select,
                                          const uint64_t *d_self_ids, uint8_t *d_status, uint64_t *d_from,
                                          uint8_t *d_resp_bytes, uint64_t resp_bytes_capacity, uint32_t *d_resp_offsets,
                                          uint64_t *d_totals);
int32_t raftgpu_follower_heartbeat(raftgpu_arena *arena, const void *bytes, uint64_t n_bytes, const uint32_t *offsets,
                                   uint64_t n, const uint32_t *select, const uint64_t *self_ids, uint8_t *status,
                                   uint64_t *from, uint8_t *resp_bytes, uint64_t resp_bytes_capacity,
                                   uint32_t *resp_offsets, uint64_t *totals);

/* ---- vote responses at a candidate ---------------------------------------------- */

/* RawNode::step -> Raft::step (raft.rs:1280-1349) -> step_candidate (raft.rs:2230-2243) -> poll's record_vote and
 * tally_votes (raft.rs:2166-2168, tracker.rs:308-340) for the MsgRequestVoteResponse (6) and MsgRequestPreVoteResponse
 * (18) frames of a wire batch.  The transitions poll makes on a decided tally are NOT applied: become_leader appends to
 * the caller's log, and role, leader_id and vote are the caller's.  The pass lists the decided groups instead, and the
 * caller runs its control lists for them (INTEGRATION.md section 6).
 * Input.  The frames of raftgpu_wire_batch (u32 LE group << 4 | peer_slot, then the Message; peer 8 + s of a wide pair
 * is cell (g + 1, s)).  d_bytes 16-byte aligned, n and n_bytes below 4 GiB.
 * Role.  d_select (required) and d_pre (nullable: no PreCandidates) are bitmaps in the layout of d_adv_bitmap: d_select
 * marks the groups whose Raft is a PreCandidate or a Candidate, d_pre the PreCandidates among them.  A frame addressed
 * to the high half of a wide pair is checked against the low half's bits, term, term_start and committed (the larger
 * of both halves', as raftgpu_group_get reports).
 * Status.  status[i] = RAFTGPU_WIRE_* << 4 | RAFTGPU_RES_*; the first failing check decides:
 *   MALFORMED    a bad frame or protobuf, or a group at or past the highest allocated slot;
 *   SKIP_TYPE    any type but 6 and 18 (append and heartbeat responses are left to their own passes);
 *   ROLE         the select bit is clear, the group is a leader (term_start != RAFTGPU_NO_TERM_START), the pair has no
 *                voter (a freed slot, or a group not configured yet), or type 6 at a PreCandidate / 18 at a Candidate;
 *   TERM         the group's term (raftgpu_group_set_term) or m.term is 0; at a Candidate m.term != term; at a
 *                PreCandidate m.term < term, or a rejection with m.term > term (become_follower).  A granted pre-vote
 *                with m.term > term passes and leaves the term alone (raft.rs:1319-1330);
 *   COMMIT_VOTE  m.commit != 0, m.commit_term != 0 and m.commit > committed;
 *   DUP          a later frame of a (group, peer) cell whose first passing frame is applied here.
 * A frame that does not pass changes nothing: run RawNode::step on it.  An applied frame's low nibble: RAFTGPU_RES_OK
 * when its vote was recorded, 0 when the cell already held a vote (record_vote is or_insert, as RAFTGPU_CTL_RECORD_VOTE),
 * RAFTGPU_RES_NO_PROGRESS for a header slot of 8 or more (nothing recorded).  A vote of a non-voter slot is recorded
 * and the tally ignores it, as in the reference.
 * Output.  One raftgpu_vote_outcome per group (pair: the low half) that an applied frame names and whose tally after the
 * pass is RAFTGPU_VOTE_WON or RAFTGPU_VOTE_LOST, in ascending group order; *d_count (u64) = how many.  Every touched
 * group adds one to votes_tallied.  Votes only accumulate, so one tally after the batch is the first decided result
 * that applying the frames one at a time would reach, in any order (DESIGN.md 3.13).  capacity must be at least
 * min(n, allocated groups), which bounds the outcomes: RAFTGPU_ERR_INVALID before any launch otherwise, as are a missing
 * d_count, d_select, d_status, d_bytes or d_offsets.  No outcome is written at or past capacity.
 * Ordering.  Runs between steps on `stream`, with its own scratch in the arena (run it on one stream at a time).  The
 * host form copies (select and pre cover the groups below the highest allocated one), runs and waits; status (n bytes)
 * nullable, *out_n = the outcomes copied to `out`. */
typedef struct raftgpu_vote_outcome {
    uint32_t group;  /* low half for a wide pair */
    uint32_t result; /* VoteResult | granted << 8 | rejected << 16, raftgpu_tally_votes' word */
} raftgpu_vote_outcome;
int32_t raftgpu_vote_wire_device(raftgpu_arena *arena, void *stream, const void *d_bytes, uint64_t n_bytes,
                                 const uint32_t *d_offsets, uint64_t n, const uint32_t *d_select, const uint32_t *d_pre,
                                 uint8_t *d_status, raftgpu_vote_outcome *d_out, uint64_t capacity, uint64_t *d_count);
int32_t raftgpu_vote_wire(raftgpu_arena *arena, const void *bytes, uint64_t n_bytes, const uint32_t *offsets, uint64_t n,
                          const uint32_t *select, const uint32_t *pre, uint8_t *status, raftgpu_vote_outcome *out,
                          uint64_t capacity, uint64_t *out_n);

/* ---- vote requests at a voter -------------------------------------------------- */

/* RawNode::step -> Raft::step (raft.rs:1280-1411, then the MsgRequestVote | MsgRequestPreVote arm at :1418-1462, with
 * send at :602-661) for the MsgRequestVote (5) and MsgRequestPreVote (17) frames of a wire batch: the term rules, the
 * grant decision and one response per decided frame.
 * Input.  The frames of raftgpu_wire_batch, but the header is u32 LE (group << 4 | x) with `group` the voter's own group
 * slot in this arena (the transport rewrites the header on the way in); x is not read and is copied into the response's
 * header.  d_bytes 16-byte aligned, n and n_bytes below 4 GiB.  d_voters (16-byte aligned, read only) has one
 * raftgpu_voter per group slot below the highest allocated one: the per-group facts the arena does not keep.  term,
 * term_start, committed and last_index come from the arena; for a wide pair (addressed by its low half) committed and
 * last_index are the larger of both halves', as raftgpu_group_get reports.
 * Status.  status[i] = RAFTGPU_WIRE_* << 4 | RAFTGPU_VREQ_* for an applied frame; the first failing check decides:
 *   MALFORMED    a bad frame or protobuf, a group at or past the highest allocated slot, or a wide pair's high half;
 *   SKIP_TYPE    any type but 5 and 17;
 *   ROLE         RAFTGPU_VOTER_SELECT is clear, or the group is a leader (term_start != RAFTGPU_NO_TERM_START): a leader
 *                that steps down has host-side consequences (raftgpu_leader_vote_request_wire decides its frames);
 *   TERM         the group's term (raftgpu_group_set_term) is 0, or m.term is 0 (a local message);
 * then the first frame of each group in frame order that got this far is decided by the term rules:
 *   IGNORED      m.term > term in lease (RAFTGPU_VOTER_LEASE, and the context is not "CampaignTransfer"), or a
 *                MsgRequestVote with m.term < term: the reference drops it;
 *   COMMIT_VOTE  a rejection with m.commit != 0, m.commit_term != 0 and m.commit > committed (maybe_commit_by_vote
 *                needs the log);
 *   OK           decided and applied: a MsgRequestVote with m.term > term first runs become_follower(m.term,
 *                INVALID_ID)'s arena part (term = m.term, and RAFTGPU_CTL_RESET's reset on both halves with term_start
 *                RAFTGPU_NO_TERM_START, last_index, committed and the table's persisted) and is decided with vote 0 and no
 *                leader; a MsgRequestPreVote at a lower term is rejected at the group's term (raft.rs:1395-1398); else
 *                can_vote, is_up_to_date(m.index, m.log_term) and the priority rule (:1420-1428) grant or reject;
 *   DUP          every later frame of a group whose first frame reached the term rules in this batch: its decision
 *                depends on what the first one changes; resubmit DUP frames, in order, with the next batch.
 * A frame that is not OK changes nothing: run RawNode::step on it (IGNORED ones may be dropped).  d_out (nullable,
 * u64[2 n]) = {m.from, the group's term after the frame} per applied frame, zero for the others.
 * Output.  One response per applied frame, in frame order: the input header, then eraftpb.Message with msg_type 6 or 18,
 * to = m.from, from = the table's id, term (m.term on a grant, the group's term otherwise), reject, and on a rejection
 * of the vote arm commit and commit_term; canonical proto3 as raftgpu_synth_wire_encode_votes writes (at most 63 bytes
 * with the header).  d_resp_bytes (16-byte aligned) holds them back to back, d_resp_offsets (n + 1 values) their starts
 * and the end, d_totals (u64[2]) = {responses, bytes}.  The pass writes terms and resets groups, so a response cannot be
 * produced again: resp_bytes_capacity must be at least raftgpu_vote_request_wire_bound(n), and that bound addressable
 * by u32 offsets: RAFTGPU_ERR_INVALID before any launch otherwise, as are a missing d_voters, d_status, d_bytes or
 * d_offsets with n > 0 and misaligned buffers.  The caller sends the responses only after it has made the changed
 * HardState (term, vote) durable.
 * Ordering.  Runs between steps on `stream`, with its own scratch in the arena (run it on one stream at a time).  The
 * host form copies (voters covers the groups below the highest allocated one), runs and waits; status, out,
 * resp_bytes / resp_offsets as above, totals u64[2]. */
#define RAFTGPU_VOTER_SELECT 0x1u /* the pass decides this group: a Follower, PreCandidate or Candidate */
#define RAFTGPU_VOTER_LEADER 0x2u /* leader_id != INVALID_ID */
#define RAFTGPU_VOTER_LEASE 0x4u  /* check_quorum && leader_id != INVALID_ID && election_elapsed < election_timeout */
#define RAFTGPU_VOTER_STALE_REPLY 0x8u /* check_quorum || pre_vote (raft.rs:1350): raftgpu_follower_term_wire answers a
                                          lower-term frame; raftgpu_vote_request_wire does not read it */
#define RAFTGPU_VOTER_CANDIDATE 0x10u  /* a PreCandidate or a Candidate: raftgpu_follower_response_wire's role, and
                                          raftgpu_follower_term_wire's step-down at the group's own term; the other
                                          passes do not read it */
#define RAFTGPU_VOTER_PRE_CANDIDATE 0x20u /* a PreCandidate (with RAFTGPU_VOTER_CANDIDATE): raftgpu_follower_response_wire */
#define RAFTGPU_VREQ_GRANTED 0x1u /* the response has reject = false */
#define RAFTGPU_VREQ_VOTED 0x2u   /* a granted MsgRequestVote: the caller sets vote = m.from, election_elapsed = 0 */
#define RAFTGPU_VREQ_BUMPED 0x4u  /* the term was raised: the caller runs become_follower(m.term, INVALID_ID)'s host side */
typedef struct raftgpu_voter {
    uint64_t id;          /* Raft::id: the response's from */
    uint64_t vote;        /* Raft::vote, 0 = INVALID_ID */
    uint64_t last_term;   /* raft_log.last_term() */
    uint64_t commit_term; /* raft_log.commit_info().1, the term of `committed` */
    uint64_t persisted;   /* raft_log.persisted: the self cell's matched after a term bump's reset (raft.rs:967) */
    uint64_t priority;    /* Raft::priority */
    uint32_t flags;       /* RAFTGPU_VOTER_* */
    uint32_t reserved;    /* 0 */
    uint64_t reserved2;   /* 0 */
} raftgpu_voter;
/* 64 bytes per frame: enough for the responses to any n frames. */
uint64_t raftgpu_vote_request_wire_bound(uint64_t n);
int32_t raftgpu_vote_request_wire_device(raftgpu_arena *arena, void *stream, const void *d_bytes, uint64_t n_bytes,
                                         const uint32_t *d_offsets, uint64_t n, const raftgpu_voter *d_voters,
                                         uint8_t *d_status, uint64_t *d_out, uint8_t *d_resp_bytes,
                                         uint64_t resp_bytes_capacity, uint32_t *d_resp_offsets, uint64_t *d_totals);
int32_t raftgpu_vote_request_wire(raftgpu_arena *arena, const void *bytes, uint64_t n_bytes, const uint32_t *offsets,
                                  uint64_t n, const raftgpu_voter *voters, uint8_t *status, uint64_t *out,
                                  uint8_t *resp_bytes, uint64_t resp_bytes_capacity, uint32_t *resp_offsets,
                                  uint64_t *totals);

/* ---- the term prefix of MsgAppend and MsgHeartbeat at a follower --------------- */

/* RawNode::step -> Raft::step's term rules (raft.rs:1280-1376) for the MsgAppend (3) and MsgHeartbeat (8) frames of a
 * wire batch at a Follower, PreCandidate or Candidate: become_follower(m.term, m.from)'s arena part for a higher term,
 * the empty MsgAppendResponse check_quorum or pre_vote asks for at a lower one.  Nothing past the term prefix: the
 * frames this pass lets through meet raftgpu_follower_heartbeat and raftgpu_follower_append[_entries] at the group's
 * (new) term.
 * Input.  The frames of those passes: u32 LE header (group << 4 | x) with `group` the follower's own group slot; x is
 * not read and is copied into the response's header.  d_bytes 16-byte aligned, n and n_bytes below 4 GiB.  d_voters
 * (16-byte aligned, read only) is raftgpu_vote_request_wire's table: the pass reads id, persisted and the flags
 * (RAFTGPU_VOTER_SELECT: a Follower, PreCandidate or Candidate, the roles whose term rule is the same;
 * RAFTGPU_VOTER_STALE_REPLY: check_quorum || pre_vote; RAFTGPU_VOTER_CANDIDATE: a PreCandidate or Candidate, which a
 * frame at its own term steps down -- opt-in: a row without it is decided as if the group were a Follower).
 * Status.  status[i] = RAFTGPU_WIRE_* << 4 | a low nibble; the first failing check decides:
 *   MALFORMED    a bad frame or protobuf, a group at or past the highest allocated slot, or a wide pair's high half;
 *   SKIP_TYPE    any type but 3 and 8 (MsgSnapshot and MsgTimeoutNow stay with the host);
 *   ROLE         RAFTGPU_VOTER_SELECT is clear, or the group is a leader (term_start != RAFTGPU_NO_TERM_START): a leader
 *                that steps down has host-side consequences;
 *   TERM         the group's term (raftgpu_group_set_term) is 0, or m.term is 0 (a local message);
 * then every passing frame is decided per group.  Let T be the larger of the group's term and the largest m.term
 * among its passing frames:
 *   OK           m.term == T: the frame is left for the follower passes, nothing is written for it.  When T is above
 *                the group's term the lowest such frame is the group's claimant, with the low nibble
 *                RAFTGPU_FTERM_BUMPED: it runs become_follower(T, m.from)'s arena part (term = T, and RAFTGPU_CTL_RESET's
 *                reset on both halves of a pair with term_start RAFTGPU_NO_TERM_START, last_index, committed -- the
 *                larger of the halves' -- and the table's persisted), exactly RAFTGPU_CTL_SET_TERM + RAFTGPU_CTL_RESET.
 *                When T equals the term of a group whose row has RAFTGPU_VOTER_CANDIDATE, the lowest frame at T is the
 *                claimant too, with the low nibble RAFTGPU_FTERM_STEPPED: step_candidate's become_follower(term, m.from)
 *                (raft.rs:2215-2224), whose arena part is RAFTGPU_CTL_RESET's reset alone (term unchanged, votes
 *                cleared);
 *   STALE        m.term < T: settled here; drop the frame.  With RAFTGPU_VOTER_STALE_REPLY the pass answers it with one
 *                MsgAppendResponse {to = m.from, from = the table's id, term = T}, every other field zero
 *                (raft.rs:1375-1376), and the low nibble is RAFTGPU_RES_OK; without it the reference ignores the frame.
 * There is no DUP: every frame gets its verdict in one call.  d_out (nullable, u64[2 n]) = {m.from, T} for each
 * claimant, zero for every other frame.
 * What the result equals.  For a group whose frames at T carry one `from`, as a real leader's do, the reference reaches
 * the same state when its frames are delivered in this order: the heartbeats at T in batch order, the appends at T in
 * batch order, then the stale frames -- the order in which this pass, raftgpu_follower_heartbeat and
 * raftgpu_follower_append[_entries] apply them.  The first frame delivered at T does the bump, and the bump does not
 * depend on which frame it is.  When the frames at T carry different `from`s, leader_id is the claimant's m.from.
 * Output.  The replies in frame order: the input header, then eraftpb.Message with msg_type 4, to, from and term;
 * canonical proto3 as raftgpu_synth_wire_encode writes (zero fields omitted, at most 39 bytes with the header).
 * d_resp_bytes (16-byte aligned) holds them back to back, d_resp_offsets (n + 1 values) their starts and the end,
 * d_totals (u64[2]) = {responses, bytes}.  The pass writes terms and resets groups, so its responses cannot be
 * produced again: resp_bytes_capacity must be at least raftgpu_follower_term_wire_bound(n), and that bound addressable
 * by u32 offsets: RAFTGPU_ERR_INVALID before any launch otherwise, as are a missing d_voters, d_status, d_bytes or
 * d_offsets with n > 0 and misaligned buffers.  The caller sends the replies only after it has made the changed
 * HardState (term) durable.
 * Host side.  For every RAFTGPU_FTERM_BUMPED frame the caller runs become_follower's host side -- role Follower,
 * leader_id = m.from, vote = 0, election_elapsed = 0 -- and updates its select bitmap, log table and voter row before
 * the next call that reads them: a voter row left stale could grant a vote the reference, now following m.from,
 * refuses.  For every RAFTGPU_FTERM_STEPPED frame: role Follower, leader_id = m.from, election_elapsed = 0, the vote
 * kept (the term is the same); clear RAFTGPU_VOTER_CANDIDATE and RAFTGPU_VOTER_PRE_CANDIDATE and set the group's
 * follower select bits, so that the follower passes on the same buffer decide the frame.
 * Ordering.  Runs between steps on `stream`, with its own scratch in the arena (run it on one stream at a time).  When
 * one received buffer goes through several passes: raftgpu_vote_request_wire first, then raftgpu_follower_response_wire
 * and its host side, then this pass, then the follower passes (their types are disjoint).  A candidate this pass bumps
 * or steps down is a Follower only once the caller says so: the follower passes of the same sequence return ROLE for it
 * until then, and the host steps those frames.  The host form copies (voters covers the groups below the highest
 * allocated one), runs and waits; status, out, resp_bytes / resp_offsets as above, totals u64[2]. */
#define RAFTGPU_FTERM_BUMPED 0x4u /* the claimant: the term was raised, the caller runs become_follower(T, m.from)'s
                                     host side */
#define RAFTGPU_FTERM_STEPPED 0x8u /* (raftgpu_follower_term_wire) the claimant at a (Pre)Candidate's own term: the
                                      caller runs become_follower(term, m.from)'s host side */
/* 39 bytes per frame: enough for the responses to any n frames. */
uint64_t raftgpu_follower_term_wire_bound(uint64_t n);
int32_t raftgpu_follower_term_wire_device(raftgpu_arena *arena, void *stream, const void *d_bytes, uint64_t n_bytes,
                                          const uint32_t *d_offsets, uint64_t n, const raftgpu_voter *d_voters,
                                          uint8_t *d_status, uint64_t *d_out, uint8_t *d_resp_bytes,
                                          uint64_t resp_bytes_capacity, uint32_t *d_resp_offsets, uint64_t *d_totals);
int32_t raftgpu_follower_term_wire(raftgpu_arena *arena, const void *bytes, uint64_t n_bytes, const uint32_t *offsets,
                                   uint64_t n, const raftgpu_voter *voters, uint8_t *status, uint64_t *out,
                                   uint8_t *resp_bytes, uint64_t resp_bytes_capacity, uint32_t *resp_offsets,
                                   uint64_t *totals);

/* ---- the term prefix of the frames that reach a leader -------------------------- */

/* RawNode::step -> Raft::step's term rules (raft.rs:1280-1411), step_leader's drop arm (:2111-2119) and, after a
 * step-down, step_follower's, for the MsgAppend (3), MsgAppendResponse (4), MsgRequestVoteResponse (6), MsgHeartbeat
 * (8), MsgHeartbeatResponse (9) and MsgRequestPreVoteResponse (18) frames of a wire batch at a leader:
 * become_follower(T, ..)'s arena part for a higher term, the empty MsgAppendResponse check_quorum or pre_vote asks for
 * at a lower-term MsgAppend / MsgHeartbeat, and a verdict for every frame the reference drops.  The frames at the
 * leader's term of types 4 and 9 are their own passes' (the wire step, raftgpu_heartbeat_wire).
 * Input.  Types 4, 6, 9 and 18 carry the leader's cell (group << 4 | slot), as the wire step and raftgpu_vote_wire take
 * them: a wide pair's high half stands for its pair's low half.  Types 3 and 8 carry the group's own slot (group << 4 |
 * x), as the follower passes take them; x is copied into the reply's header.  d_bytes 16-byte aligned, n and n_bytes
 * below 4 GiB.  d_voters (16-byte aligned, read only) is raftgpu_vote_request_wire's table, one row per group slot below
 * the highest allocated one (a pair's row is its low half's): the pass reads id, persisted and
 * RAFTGPU_VOTER_STALE_REPLY.  Leadership is the arena's own: term_start != RAFTGPU_NO_TERM_START.
 * Status.  status[i] = RAFTGPU_WIRE_* << 4 | a low nibble; the first failing check decides:
 *   MALFORMED    a bad frame or protobuf, a group at or past the highest allocated slot, or a wide pair's high half in
 *                the header of type 3 or 8;
 *   SKIP_TYPE    any type but 3, 4, 6, 8, 9 and 18;
 *   ROLE         the group (a pair: its low half) is not a leader;
 *   TERM         the group's term (raftgpu_group_set_term) is 0, or m.term is 0 (a local message);
 * then every passing frame is decided per group.  A MsgRequestPreVoteResponse with reject = false never raises the term
 * (raft.rs:1319-1320): it is STALE below the group's term and IGNORED at or above it.  Let T be the larger of the
 * group's term and the largest m.term among its other passing frames:
 *   OK | RAFTGPU_FTERM_BUMPED  T is above the term and this is the lowest frame at T: it runs become_follower(T, ..)'s
 *                arena part, exactly RAFTGPU_CTL_SET_TERM + RAFTGPU_CTL_RESET (as raftgpu_follower_term_wire's claimant).
 *                A claimant of type 3 or 8 is left for the follower passes;
 *   OK           a frame of type 4 or 9 at the leader's term (its own pass decided it), or another frame of type 3 or 8
 *                at T above the term (left for the follower passes);
 *   IGNORED      a frame of type 3, 6, 8 or 18 at the leader's term (step_leader drops it), or another frame of type 4,
 *                6, 9 or 18 at T above the term (step_follower drops it);
 *   STALE        any other frame, below T: settled here; drop it.  A MsgAppend or MsgHeartbeat of a group with
 *                RAFTGPU_VOTER_STALE_REPLY is answered with one MsgAppendResponse {to = m.from, from = the table's id,
 *                term = T}, every other field zero (raft.rs:1375-1376), and the low nibble is RAFTGPU_RES_OK.
 * There is no DUP: every frame gets its verdict in one call.  d_out (nullable, u64[2 n]) = {leader_id, T} for each
 * claimant -- leader_id = m.from for types 3 and 8, 0 for the others (raft.rs:1340-1347) -- zero for every other frame.
 * What the result equals.  The reference reaches the same state when a group's frames are delivered in this order: the
 * frames at the leader's term, the claimant, the other frames at T in batch order (types 3 and 8 through the follower
 * passes), then the stale frames; the granting pre-vote responses anywhere.
 * Output.  The replies in frame order, as raftgpu_follower_term_wire writes them (at most 39 bytes with the header):
 * d_resp_bytes (16-byte aligned) holds them back to back, d_resp_offsets (n + 1 values) their starts and the end,
 * d_totals (u64[2]) = {responses, bytes}.  resp_bytes_capacity must be at least raftgpu_follower_term_wire_bound(n), and
 * that bound addressable by u32 offsets: RAFTGPU_ERR_INVALID before any launch otherwise, as are a missing d_voters,
 * d_status, d_bytes or d_offsets with n > 0 and misaligned buffers.  The caller sends the replies only after it has
 * made the changed HardState (term) durable.
 * Host side.  For every RAFTGPU_FTERM_BUMPED frame the caller runs become_follower (raft.rs:1082-1093) and the host part
 * of reset (:942-971) for the group: role Follower, leader_id as out gives it, vote = 0, election_elapsed = 0, no
 * leadership transferee, no pending conf index, the read-index map emptied; and updates its voter row and select
 * bitmaps before the next call that reads them.
 * Ordering.  Runs between steps on `stream`, with its own scratch in the arena (run it on one stream at a time).  When
 * one received buffer goes through several passes: raftgpu_vote_request_wire, raftgpu_follower_response_wire,
 * raftgpu_follower_term_wire, raftgpu_vote_wire, the leader passes (the wire step and raftgpu_heartbeat_wire), then
 * this pass, then the host side
 * of every BUMPED of raftgpu_follower_term_wire and of this pass, then the follower passes.  This pass must come after
 * the leader passes, which would apply the frames at T after a bump; after a step's begin is enough.  The follower
 * term pass must come before it, or a group bumped here could be answered twice.  Merging statuses: this pass's
 * STALE, IGNORED and the BUMPED of types 4, 6, 9 and 18 are settled; its OK leaves the frame to its own pass's status;
 * a frame of a bumped group that a leader pass left DUP, NEEDS_LOG or CONTEXT is stale: drop it.  The host form copies
 * (voters covers the groups below the highest allocated one), runs and waits; status, out, resp_bytes / resp_offsets
 * as above, totals u64[2]. */
int32_t raftgpu_leader_term_wire_device(raftgpu_arena *arena, void *stream, const void *d_bytes, uint64_t n_bytes,
                                        const uint32_t *d_offsets, uint64_t n, const raftgpu_voter *d_voters,
                                        uint8_t *d_status, uint64_t *d_out, uint8_t *d_resp_bytes,
                                        uint64_t resp_bytes_capacity, uint32_t *d_resp_offsets, uint64_t *d_totals);
int32_t raftgpu_leader_term_wire(raftgpu_arena *arena, const void *bytes, uint64_t n_bytes, const uint32_t *offsets,
                                 uint64_t n, const raftgpu_voter *voters, uint8_t *status, uint64_t *out,
                                 uint8_t *resp_bytes, uint64_t resp_bytes_capacity, uint32_t *resp_offsets,
                                 uint64_t *totals);

/* ---- vote requests at a leader ------------------------------------------------- */

/* RawNode::step -> Raft::step's term rules (raft.rs:1280-1411), then the MsgRequestVote | MsgRequestPreVote arm
 * (:1418-1462) and one response through send, for the MsgRequestVote (5) and MsgRequestPreVote (17) frames of a wire
 * batch at a leader: a winner's answer to the losing candidates, the lease against a healed partition, and the
 * step-down at a higher-term vote.  raftgpu_vote_request_wire returns ROLE for these frames; this pass takes them.
 * Input.  raftgpu_vote_request_wire's frames (the header names the group's own slot, x is copied back), its table and
 * its buffers.  The pass reads id, vote, last_term, commit_term, persisted, priority and the flags RAFTGPU_VOTER_LEADER
 * (the leader's own leader_id: set) and RAFTGPU_VOTER_LEASE; RAFTGPU_VOTER_SELECT is not read.  Leadership is the
 * arena's own: term_start != RAFTGPU_NO_TERM_START, a pair's by its low half.
 * Status.  status[i] = RAFTGPU_WIRE_* << 4 | RAFTGPU_VREQ_* for an answered frame; the first failing check decides:
 *   MALFORMED    a bad frame or protobuf, a group at or past the highest allocated slot, or a wide pair's high half;
 *   SKIP_TYPE    any type but 5 and 17;
 *   ROLE         the group is not a leader;
 *   TERM         the group's term (raftgpu_group_set_term) is 0, or m.term is 0 (a local message);
 * then each group's frames in frame order.  The group's claimant b(g) is its first frame that changes state: a
 * MsgRequestVote with m.term > term that the lease does not drop, or a granted MsgRequestVote at the term (only a frame
 * whose m.from is the leader's own vote gets one).  The frames before b(g) are decided against the unchanged leader:
 *   IGNORED      m.term > term in lease (RAFTGPU_VOTER_LEASE, and the context is not "CampaignTransfer"), or a
 *                MsgRequestVote with m.term < term: the reference drops it;
 *   OK           a MsgRequestPreVote at a lower term is rejected at the group's term (raft.rs:1395-1398); a
 *                MsgRequestPreVote above the term (the term stays) and any frame at the term meet can_vote,
 *                is_up_to_date and the priority rule: a grant answers at m.term, a rejection at the term with
 *                commit_info() (maybe_commit_by_vote returns at once for a Leader, :2131);
 * b(g) is decided as raftgpu_vote_request_wire decides a bumped frame:
 *   COMMIT_VOTE  a MsgRequestVote above the term that is rejected with m.commit != 0, m.commit_term != 0 and m.commit
 *                beyond committed (maybe_commit_by_vote at the Follower it becomes needs the log): nothing is applied;
 *   OK           applied: above the term, become_follower(m.term, INVALID_ID)'s arena part (term = m.term, and
 *                RAFTGPU_CTL_RESET's reset on both halves with term_start RAFTGPU_NO_TERM_START, last_index, committed and
 *                the table's persisted), then the grant with vote 0 and no leader (RAFTGPU_VREQ_BUMPED, and
 *                RAFTGPU_VREQ_VOTED on a grant) or the rejection at m.term; at the term, the grant (RAFTGPU_VREQ_VOTED);
 *   DUP          every frame after b(g): its decision depends on b(g)'s host side.  Resubmit DUP frames, in order,
 *                after it: through raftgpu_vote_request_wire once the group is a Follower, through this pass otherwise.
 * A frame that is not OK changes nothing: run RawNode::step on it (IGNORED ones may be dropped).  d_out (nullable,
 * u64[2 n]) = {m.from, the group's term after the frame} per OK frame, zero for the others.
 * Output, bound and refusals.  raftgpu_vote_request_wire's: one response per OK frame in frame order, resp_bytes_capacity
 * at least raftgpu_vote_request_wire_bound(n), RAFTGPU_ERR_INVALID before any launch otherwise, as for a missing
 * d_voters, d_status, d_bytes or d_offsets with n > 0, misaligned buffers and a batch past 4 GiB.  The caller sends the
 * responses only after it has made the changed HardState (term, vote) durable.
 * Host side.  For a RAFTGPU_VREQ_BUMPED frame the caller runs become_follower (raft.rs:1082-1093) and the host part of
 * reset (:942-971): role Follower, no leader, vote = 0 -- then m.from for RAFTGPU_VREQ_VOTED --, election_elapsed = 0,
 * no leadership transferee, no pending conf index, the read-index map emptied; it clears RAFTGPU_VOTER_LEADER and
 * RAFTGPU_VOTER_LEASE, sets the group's follower select bits and updates its voter row before the next call that reads
 * them.  For RAFTGPU_VREQ_VOTED at the term: vote = m.from, election_elapsed = 0.
 * Ordering.  Runs between steps on `stream`, with its own scratch in the arena (run it on one stream at a time).  When
 * one received buffer goes through several passes, this pass is the last of the leader side: after
 * raftgpu_leader_term_wire and its host side.  A group raftgpu_leader_term_wire deposed is ROLE here: once the caller
 * has made it a Follower, it resubmits those frames through raftgpu_vote_request_wire, after the follower passes.  The
 * reference reaches the same state when a leader's frames are delivered in that order: its other frames, then its vote
 * requests in frame order.  The host form copies (voters covers the groups below the highest allocated one), runs and
 * waits; status, out, resp_bytes / resp_offsets as above, totals u64[2]. */
int32_t raftgpu_leader_vote_request_wire_device(raftgpu_arena *arena, void *stream, const void *d_bytes,
                                                uint64_t n_bytes, const uint32_t *d_offsets, uint64_t n,
                                                const raftgpu_voter *d_voters, uint8_t *d_status, uint64_t *d_out,
                                                uint8_t *d_resp_bytes, uint64_t resp_bytes_capacity,
                                                uint32_t *d_resp_offsets, uint64_t *d_totals);
int32_t raftgpu_leader_vote_request_wire(raftgpu_arena *arena, const void *bytes, uint64_t n_bytes,
                                         const uint32_t *offsets, uint64_t n, const raftgpu_voter *voters,
                                         uint8_t *status, uint64_t *out, uint8_t *resp_bytes,
                                         uint64_t resp_bytes_capacity, uint32_t *resp_offsets, uint64_t *totals);

/* ---- the responses that reach a follower or a candidate ------------------------ */

/* RawNode::step -> Raft::step's term rules (raft.rs:1280-1348) and the drop arms of step_follower and step_candidate
 * (:2205-2255) for the MsgAppendResponse (4), MsgRequestVoteResponse (6), MsgHeartbeatResponse (9) and
 * MsgRequestPreVoteResponse (18) frames of a wire batch at a Follower, PreCandidate or Candidate: the late responses
 * of a deposed leader, the late votes of a lost or abandoned election, and a higher-term rejection at a candidate.
 * become_follower(T, INVALID_ID)'s arena part for a higher term, and a verdict for every frame the reference drops.
 * None of these frames is ever answered.
 * Input.  The frames carry the receiver's cell (group << 4 | slot), as the wire step, raftgpu_vote_wire and
 * raftgpu_leader_term_wire take them: a wide pair's high half stands for its pair's low half.  d_bytes 16-byte aligned,
 * n and n_bytes below 4 GiB.  d_voters (16-byte aligned, read only) is raftgpu_vote_request_wire's table, one row per
 * group slot below the highest allocated one (a pair's row is its low half's): the pass reads persisted and the flags
 * (RAFTGPU_VOTER_SELECT; RAFTGPU_VOTER_CANDIDATE: a PreCandidate or Candidate; RAFTGPU_VOTER_PRE_CANDIDATE: a
 * PreCandidate).  Leadership is the arena's own: term_start != RAFTGPU_NO_TERM_START.
 * Status.  status[i] = RAFTGPU_WIRE_* << 4 | a low nibble; the first failing check decides:
 *   MALFORMED    a bad frame or protobuf, or a group at or past the highest allocated slot;
 *   SKIP_TYPE    any type but 4, 6, 9 and 18;
 *   ROLE         RAFTGPU_VOTER_SELECT is clear, or the group (a pair: its low half) is a leader;
 *   TERM         the group's term (raftgpu_group_set_term) is 0, or m.term is 0 (a local message);
 * then every passing frame is decided per group.  A MsgRequestPreVoteResponse with reject = false never raises the term
 * (raft.rs:1319-1320).  Let T be the larger of the group's term and the largest m.term among its other passing frames:
 *   OK | RAFTGPU_FTERM_BUMPED  T is above the term and this is the lowest frame at T: it runs
 *                become_follower(T, INVALID_ID)'s arena part, exactly RAFTGPU_CTL_SET_TERM + RAFTGPU_CTL_RESET (as
 *                raftgpu_follower_term_wire's claimant);
 *   OK           T is the group's term and the frame belongs to the group's own candidacy: a MsgRequestVoteResponse
 *                at a Candidate at the term, or a MsgRequestPreVoteResponse at a PreCandidate at the term -- or, when
 *                it grants, above it (raft.rs:1319-1330).  Nothing is written: raftgpu_vote_wire takes the frame;
 *   IGNORED      any other frame at T, a granting pre-vote response at or above T included: step_follower and
 *                step_candidate drop it;
 *   STALE        m.term below T: settled here; drop the frame (no reply: raft.rs:1349-1411).
 * There is no DUP: every frame gets its verdict in one call.  d_out (nullable, u64[n]) = T for each claimant, zero for
 * every other frame.
 * What the result equals.  The reference reaches the same state when a group's frames are delivered in this order: the
 * claimant, the other frames at T, then the stale frames.  When there is no claimant, the frames left OK go through
 * raftgpu_vote_wire.
 * Refusals.  RAFTGPU_ERR_INVALID before any launch for a missing d_voters, d_status, d_bytes or d_offsets with n > 0,
 * misaligned buffers, and the batch limits of the other wire passes.
 * Host side.  For every RAFTGPU_FTERM_BUMPED frame the caller runs become_follower(T, INVALID_ID) (raft.rs:1082-1093)
 * and the host part of reset (:942-971): role Follower, no leader, vote = 0, election_elapsed = 0; it clears
 * RAFTGPU_VOTER_CANDIDATE and RAFTGPU_VOTER_PRE_CANDIDATE, sets the group's follower select bits and updates its
 * voter row before the next call that reads them.
 * Ordering.  Runs between steps on `stream`, with its own scratch in the arena (run it on one stream at a time).  When
 * one received buffer goes through several passes: raftgpu_vote_request_wire, this pass and its host side,
 * raftgpu_follower_term_wire and its host side, raftgpu_vote_wire, the leader passes, raftgpu_leader_term_wire and its
 * host side, then the follower passes.  Merging statuses: this pass's STALE, IGNORED and BUMPED are settled; its OK
 * defers to raftgpu_vote_wire's status, but for a group raftgpu_follower_term_wire then bumps or steps down: its
 * step-down comes first, and step_follower drops the frame (settled as IGNORED; do not hand it to raftgpu_vote_wire).  The host form copies (voters covers the groups below the highest allocated
 * one), runs and waits; status and out as above. */
int32_t raftgpu_follower_response_wire_device(raftgpu_arena *arena, void *stream, const void *d_bytes, uint64_t n_bytes,
                                              const uint32_t *d_offsets, uint64_t n, const raftgpu_voter *d_voters,
                                              uint8_t *d_status, uint64_t *d_out);
int32_t raftgpu_follower_response_wire(raftgpu_arena *arena, const void *bytes, uint64_t n_bytes, const uint32_t *offsets,
                                       uint64_t n, const raftgpu_voter *voters, uint8_t *status, uint64_t *out);

/* ---- MsgAppend at the follower ------------------------------------------------ */

/* RawNode::step -> Raft::step (raft.rs:1280-1411) -> step_follower (raft.rs:2271-2275) -> handle_append_entries
 * (raft.rs:2389-2448, with maybe_append and find_conflict_by_term, raft_log.rs:209-279) for the entry-less MsgAppend
 * frames (msg_type 3) of a wire batch -- the commit broadcast raftgpu_append_frames writes: commit_to and one
 * MsgAppendResponse per decided frame.  No entry is ever written and last_index is never changed: a frame that carries
 * entries, or whose answer needs a term of the log the pass does not know, goes back to the host whole.
 * Input.  The frames of raftgpu_wire_batch, but the header is u32 LE (group << 4 | x) with `group` the follower's own
 * group slot in this arena (the transport rewrites the header on the way in); x is not read and is copied into the
 * response's header.  d_bytes 16-byte aligned, n and n_bytes below 4 GiB.  d_log (16-byte aligned, read only) has one
 * raftgpu_follower_log per group slot below the highest allocated one.  term, term_start, committed and last_index come
 * from the arena (the caller keeps last_index current with RAFTGPU_CTL_SET_LOG_BOUNDS, term start
 * RAFTGPU_NO_TERM_START); for a wide pair (addressed by its low half) committed and last_index are the larger of both
 * halves'.
 * The run.  run_start / run_term state the last term run of the caller's log: raft_log.term(i) == run_term for every i
 * in [run_start, last_index] (run_start > last_index: no run).  term(i) is known to the pass there and above last_index
 * (0, raft_log.rs:125), nowhere else; a shorter run is always correct and only hands back more frames.
 * Status.  status[i] = RAFTGPU_WIRE_* << 4 | RAFTGPU_RES_OK [| RAFTGPU_FAPP_*] for an applied frame; the first failing
 * check decides:
 *   MALFORMED    a bad frame or protobuf, a group at or past the highest allocated slot (on an arena with read queues:
 *                any unallocated group), or the high half of a wide pair;
 *   SKIP_TYPE    any type but 3;
 *   ROLE         RAFTGPU_FOLLOWER_SELECT is clear, or the group is a leader (term_start != RAFTGPU_NO_TERM_START);
 *   TERM         the group's term (raftgpu_group_set_term) is 0 or m.term differs: a higher term is
 *                become_follower(m.term, m.from), a lower one may need a MsgAppendResponse (raft.rs:1349-1376);
 * then the first frame of each group in frame order that got this far is decided:
 *   NEEDS_LOG    the frame carries entries (any field 7, an empty Entry included), or the decision reads a term
 *                outside the run: run RawNode::step on it;
 *   COMMIT_RANGE the log matches and min(m.commit, m.index) > max(committed, last_index): commit_to would be fatal!
 *                (raft_log.rs:291-298);
 *   OK           decided and applied:
 *                - m.index < committed: the response is {index = committed, commit = committed} (RAFTGPU_FAPP_STALE);
 *                - term(m.index) == m.log_term: commit_to(min(m.commit, m.index)) on both halves of a pair, as
 *                  RAFTGPU_CTL_COMMIT_TO; the response is {index = m.index, commit = committed after};
 *                - otherwise, with h = min(m.index, last_index) in the run and run_term <= m.log_term: the response is
 *                  {reject, index = m.index, reject_hint = h, log_term = run_term, commit = committed}
 *                  (RAFTGPU_FAPP_REJECT); every other rejection walks below the run and is NEEDS_LOG -- on an arena
 *                  with follower runs the match and the walk also read the row's runs below the table's run
 *                  (raftgpu_arena_enable_follower_runs; this pass never writes the rows);
 *   DUP          every later frame of a group whose first frame reached the decision in this batch: resubmit DUP
 *                frames, in order, with the next batch.
 * A frame that is not OK changes nothing.  d_from (nullable, u64[n]) = m.from of every applied frame (0 for the
 * others), for step_follower's leader_id = m.from and election_elapsed = 0.  This pass and
 * raftgpu_follower_heartbeat take disjoint types, so one received buffer can go through both; a group's heartbeats
 * and appends are then not answered in the batch's own order (Raft allows it; split the buffer to keep that order).
 * Output.  One MsgAppendResponse per applied frame, in frame order: the input header, then eraftpb.Message with
 * msg_type 4, to = m.from, from = the table's id, term, log_term, index, commit, reject and reject_hint; canonical
 * proto3 as raftgpu_synth_wire_encode writes (at most 85 bytes with the header).  d_resp_bytes (16-byte aligned) holds
 * them back to back, d_resp_offsets (n + 1 values) their starts and the end, d_totals (u64[2]) = {responses, bytes}.  A
 * response cannot be produced again once committed has moved: resp_bytes_capacity must be at least
 * raftgpu_follower_append_bound(n), and that bound addressable by u32 offsets: RAFTGPU_ERR_INVALID before any launch
 * otherwise, as are a missing d_log, d_status, d_bytes or d_offsets with n > 0 and misaligned buffers.
 * Ordering.  Runs between steps on `stream`, with its own scratch in the arena (run it on one stream at a time).  The
 * host form copies (log covers the groups below the highest allocated one), runs and waits; status, from,
 * resp_bytes / resp_offsets as above, totals u64[2]. */
#define RAFTGPU_FOLLOWER_SELECT 0x1u /* a Follower without pending_request_snapshot: the pass decides this group */
#define RAFTGPU_FAPP_REJECT 0x2u     /* the response rejects (reject_hint, log_term = run_term) */
#define RAFTGPU_FAPP_STALE 0x4u      /* m.index < committed: the response names committed, nothing changed */
typedef struct raftgpu_follower_log {
    uint64_t id;        /* Raft::id: the response's from */
    uint64_t run_start; /* every index i in [run_start, last_index] has raft_log.term(i) == run_term */
    uint64_t run_term;  /* (run_start > last_index: no run; only indexes above last_index are known, term 0) */
    uint32_t flags;     /* RAFTGPU_FOLLOWER_* */
    uint32_t reserved;  /* 0 */
} raftgpu_follower_log;
/* 85 bytes per frame: enough for the responses to any n frames. */
uint64_t raftgpu_follower_append_bound(uint64_t n);
int32_t raftgpu_follower_append_device(raftgpu_arena *arena, void *stream, const void *d_bytes, uint64_t n_bytes,
                                       const uint32_t *d_offsets, uint64_t n, const raftgpu_follower_log *d_log,
                                       uint8_t *d_status, uint64_t *d_from, uint8_t *d_resp_bytes,
                                       uint64_t resp_bytes_capacity, uint32_t *d_resp_offsets, uint64_t *d_totals);
int32_t raftgpu_follower_append(raftgpu_arena *arena, const void *bytes, uint64_t n_bytes, const uint32_t *offsets,
                                uint64_t n, const raftgpu_follower_log *log, uint8_t *status, uint64_t *from,
                                uint8_t *resp_bytes, uint64_t resp_bytes_capacity, uint32_t *resp_offsets,
                                uint64_t *totals);

/* ---- MsgAppend with entries at the follower ------------------------------------ */

/* raftgpu_follower_append, and for a frame that carries entries maybe_append (raft_log.rs:249-279) at the log's tail:
 * find_conflict (raft_log.rs:182-198) from the run, the new last_index, commit_to and the MsgAppendResponse.  The log
 * stays with the caller: the pass says which bytes of the frame the log takes (the appended records' span) and keeps
 * the table's run current.
 * The input, the header, MALFORMED, SKIP_TYPE, ROLE, TERM, the claim and DUP rule, the stale rule (m.index < committed
 * is answered whatever entries the frame carries), the rejections (the entries are ignored), the responses, the bound
 * (raftgpu_follower_append_bound), the refusals and the ordering are raftgpu_follower_append's.  What differs:
 * Entries.  Each field 7 of a frame past TERM is decoded as an eraftpb.Entry (term = 2, index = 3; other fields
 * skipped, a repeated scalar keeps its last value): an Entry whose bytes are not a well-formed protobuf message makes
 * the frame MALFORMED (it does not claim its group).  A claiming frame whose log matches at m.index then runs
 * maybe_append, in this order:
 *   NEEDS_LOG    a field 7 that is not length-delimited; indexes that are not m.index + 1, m.index + 2, ...; an entry
 *                of term 0; m.index > last_index (a gap: truncate_and_append panics); appended entries that are not
 *                back to back in the frame (another field between them);
 *   COMMIT_RANGE find_conflict's index is at or below committed (raft_log.rs:259-265 fatal!), or commit_to would be;
 *   OK           find_conflict's index is the first entry whose index is <= last_index and whose term is not run_term,
 *                or the first above last_index.  When there is one (`conflict`), last_index = m.index + entries (both
 *                halves of a pair, as RAFTGPU_CTL_SET_LOG_BOUNDS) and the low nibble is RAFTGPU_RES_OK |
 *                RAFTGPU_FAPP_APPENDED; when every entry matched nothing is appended and it is RAFTGPU_RES_OK.  Then
 *                commit_to(min(m.commit, m.index + entries)); the response is {index = m.index + entries, commit =
 *                committed after}.
 * The run.  For an appended frame, let t be the last entry's term and k the first index of the trailing block of
 * appended entries with term t.  When every appended entry has term t, t == run_term and conflict - 1 >= run_start,
 * the run stays; otherwise it becomes [k, last_index] with term t.  The device form writes d_log's row (the table is
 * read-write); the host form writes the caller's `log` rows of the appended frames from their records.  On an arena
 * with follower runs (raftgpu_arena_enable_follower_runs) find_conflict also reads the row's runs, the log may be
 * truncated into them, and an append that does not keep the run rewrites the run (which may then merge with the
 * segment below, starting before k) and the row.
 * Appended.  d_appended (u64-aligned, n records) = raftgpu_follower_appended of every RAFTGPU_FAPP_APPENDED frame, all
 * zero for every other frame.  The span points into the caller's batch: the host hands those bytes to its log engine
 * (or decodes only them for RaftLog::unstable), lowers persisted to first_index - 1 (raft_log.rs:269-272) and sends the
 * response once the entries are durable.  The host form's `appended` has n records. */
#define RAFTGPU_FAPP_APPENDED 0x8u /* the log took entries from this frame: see raftgpu_follower_appended */
typedef struct raftgpu_follower_appended {
    uint64_t first_index; /* find_conflict's index: the first entry the log took from this frame */
    uint64_t last_index;  /* the log's last index after the append (m.index + number of entries) */
    uint64_t run_start;   /* the log's last term run after the append (also written into the table) */
    uint64_t run_term;
    uint32_t span_off;    /* byte offset in the batch of that entry's field-7 tag */
    uint32_t span_len;    /* the appended Entry records (tag, length, Entry), back to back */
} raftgpu_follower_appended; /* all zero for every frame without RAFTGPU_FAPP_APPENDED */
int32_t raftgpu_follower_append_entries_device(raftgpu_arena *arena, void *stream, const void *d_bytes, uint64_t n_bytes,
                                               const uint32_t *d_offsets, uint64_t n, raftgpu_follower_log *d_log,
                                               uint8_t *d_status, uint64_t *d_from, raftgpu_follower_appended *d_appended,
                                               uint8_t *d_resp_bytes, uint64_t resp_bytes_capacity,
                                               uint32_t *d_resp_offsets, uint64_t *d_totals);
int32_t raftgpu_follower_append_entries(raftgpu_arena *arena, const void *bytes, uint64_t n_bytes, const uint32_t *offsets,
                                        uint64_t n, raftgpu_follower_log *log, uint8_t *status, uint64_t *from,
                                        raftgpu_follower_appended *appended, uint8_t *resp_bytes,
                                        uint64_t resp_bytes_capacity, uint32_t *resp_offsets, uint64_t *totals);

/* ---- the follower's earlier term runs: MsgAppend decided below the table's run ---- */

/* The two passes above know term(i) on the table's run and above last_index.  After an election or a healed partition
 * a follower's answer usually reads an older term: a rejection whose find_conflict_by_term walk (raft.rs:2429-2444,
 * raft_log.rs:209-235) leaves the run, and the leader's next probe, whose m.index lies below it.  A row per group
 * states up to two earlier term runs of the follower's log below the table's run; with it raftgpu_follower_append[_device]
 * and raftgpu_follower_append_entries[_device] read term(i) there too:
 *   - a match at m.index in run 1 or run 2: commit_to(min(m.commit, m.index)), or maybe_append with find_conflict
 *     through every stated run (the log may be truncated into run 1 or run 2);
 *   - a rejection: the walk goes down the table's run, run 1 and run 2 from h = min(m.index, last_index); the first
 *     whose term is <= m.log_term answers {reject_hint = min(h, its end), log_term = its term}.  A walk that leaves the
 *     lowest stated run stays RAFTGPU_WIRE_NEEDS_LOG (index 0 included: the pass cannot tell a compacted log).
 * Everything else -- the statuses, the gap and entry-shape rules, the responses -- is as above.
 *
 * A row is used only while the arena has follower runs, the table's run is non-empty (run_start <= last_index, the
 * pair's larger) and (run_start, run_term) equal the row's anchor with a non-zero term.  By the Log Matching Property
 * the log below that entry is then the one the row was stated for, so a row survives term changes and
 * become_follower.  A host-side change that moves the table's run off the anchor (a truncation or append that rewrites
 * it, a snapshot) leaves the row inert until it is stated again.  Group alloc and free clear the row; a wide pair's row
 * is on its low half.
 *
 * raftgpu_follower_append reads rows and never writes them.  raftgpu_follower_append_entries rewrites the row of every
 * group it appends to so that, with the table's run, it describes the new log from the top: the appended blocks, the
 * segment that held conflict - 1 cut there and the runs below it, equal neighbours merged, terms strictly decreasing
 * downward.  Appended entries with more than two terms leave run 2, or both runs, unstated.  The table's new run (also
 * raftgpu_follower_appended.run_start / run_term) may then start lower than the trailing block: it is still the log's
 * last term run.  An append without an anchored row writes an anchored one from what the pass knows.
 *
 * Opt-in: call before groups are allocated.  Memory: 48 bytes per group slot.  An arena that does not call it behaves
 * exactly as without the feature. */
int32_t raftgpu_arena_enable_follower_runs(raftgpu_arena *arena);

/* One group's row: 56 bytes.  Run 1 is [run_start[0], anchor_start - 1] at run_term[0], run 2 is [run_start[1],
 * run_start[0] - 1] at run_term[1]; a run_start of 0 states no run.  Every stated run must still be readable by the
 * follower's RaftLog::term (at or above first_index - 1): on compaction, restate the row or drop runs.  Fewer runs are
 * never wrong; they leave more frames to the host. */
typedef struct raftgpu_follower_runs {
    uint32_t group;        /* the group (the low half of a wide pair) */
    uint32_t reserved;     /* ignored; 0 from raftgpu_follower_runs_get */
    uint64_t anchor_start; /* the table's run this row belongs to: raftgpu_follower_log.run_start ... */
    uint64_t anchor_term;  /* ... and run_term */
    uint64_t run_start[2];
    uint64_t run_term[2];
} raftgpu_follower_runs;

/* State rows for many groups.  status[i] per row, and a refused row is not stored:
 *   RAFTGPU_ERR_RANGE    the group is not allocated, or is the high half of a wide pair;
 *   RAFTGPU_ERR_INVALID  anchor_term is 0, anchor_start is 0 or RAFTGPU_NO_TERM_START, run 2 without run 1, starts that
 *                        do not satisfy 0 < run_start[1] < run_start[0] < anchor_start where stated, or run terms that
 *                        do not satisfy 0 < run_term[1] < run_term[0] < anchor_term where stated.
 * Returns RAFTGPU_OK when the list ran (n == 0 included), RAFTGPU_ERR_INVALID for an arena without follower runs or a
 * NULL rows / status with n > 0.  The rows take effect at the call, in submission order on the compute stream;
 * synchronous.  A later row of the same group wins. */
int32_t raftgpu_follower_runs_set(raftgpu_arena *arena, const raftgpu_follower_runs *rows, uint64_t n, int32_t *status);

/* The device's rows of groups [first, first + n) (group filled in), after the work already submitted on the compute
 * stream: the entries pass rewrites rows on its own, and this is how a caller sees them.  The copy is not ordered after
 * work on other streams: after raftgpu_follower_append_entries_device on a stream of the caller's, synchronise that
 * stream first.  RAFTGPU_ERR_INVALID for an arena without follower runs or NULL rows with n > 0, RAFTGPU_ERR_RANGE past
 * the arena's capacity. */
int32_t raftgpu_follower_runs_get(raftgpu_arena *arena, uint32_t first, uint32_t n, raftgpu_follower_runs *rows);

/* ---- votes (SURVEY 8(f) rank 1) ----------------------------------------- */

/* ProgressTracker::reset_votes / record_vote (tracker.rs:301-310). */
int32_t raftgpu_reset_votes(raftgpu_arena *arena, uint32_t group);
int32_t raftgpu_record_vote(raftgpu_arena *arena, uint32_t group, uint32_t peer_slot, int32_t vote);
/* Batched ProgressTracker::tally_votes (tracker.rs:313-340) over [first, first+n):
 * d_out[g] = VoteResult | granted << 8 | rejected << 16.  Asynchronous. */
int32_t raftgpu_tally_votes(raftgpu_arena *arena, void *stream, uint32_t first, uint32_t n,
                            uint32_t *d_out);
/* Single-group form (synchronous). */
int32_t raftgpu_vote_result(raftgpu_arena *arena, uint32_t group, int32_t *out_result,
                            uint32_t *out_granted, uint32_t *out_rejected);

/* ---- batched control plane ------------------------------------------------ */

/* One command of a raftgpu_control list: one single-group control call and its arguments.  40 bytes. */
typedef struct {
    uint32_t group;     /* group id as the single-group calls take it (the low half of a wide group) */
    uint8_t op;         /* RAFTGPU_CTL_* */
    uint8_t peer_slot;  /* 0..15 where the op names a peer; SET_CONF: the self slot, 0xff = none */
    uint16_t arg;       /* PROGRESS_OP: RAFTGPU_POP_*; RECORD_VOTE: 0 no / 1 yes; SET_GROUP_COMMIT: enable */
    uint64_t a[4];      /* the single call's u64 arguments, in its order */
} raftgpu_ctl_cmd;

/* What the command's single call would have returned. */
typedef struct {
    int32_t status;     /* exactly the single call's status */
    int32_t value;      /* its out value: has_quorum / quorum_recently_active / maybe_commit_to 0|1, progress_op's
                           result, vote_result as VoteResult | granted << 8 | rejected << 16; else 0 */
} raftgpu_ctl_result;

/* op                                    single call                      arguments */
#define RAFTGPU_CTL_SET_CONF 0              /* raftgpu_group_set_conf        a = {incoming, outgoing, learners, next_idx}, peer_slot = self */
#define RAFTGPU_CTL_RESET 1                 /* raftgpu_group_reset           a = {term_start, last_index, committed, persisted} */
#define RAFTGPU_CTL_BECOME_LEADER 2         /* raftgpu_group_become_leader   - */
#define RAFTGPU_CTL_SET_LOG_BOUNDS 3        /* raftgpu_group_set_log_bounds  a = {term_start, last_index} */
#define RAFTGPU_CTL_SET_TERM 4              /* raftgpu_group_set_term        a[0] */
#define RAFTGPU_CTL_COMMIT_TO 5             /* raftgpu_group_commit_to       a[0] */
#define RAFTGPU_CTL_MAYBE_COMMIT_TO 6       /* raftgpu_group_maybe_commit_to a[0] */
#define RAFTGPU_CTL_SET_GROUP_COMMIT 7      /* raftgpu_set_group_commit      arg */
#define RAFTGPU_CTL_ASSIGN_COMMIT_GROUP 8   /* raftgpu_assign_commit_group   peer_slot, a[0] */
#define RAFTGPU_CTL_RESET_VOTES 9           /* raftgpu_reset_votes           - */
#define RAFTGPU_CTL_RECORD_VOTE 10          /* raftgpu_record_vote           peer_slot, arg */
#define RAFTGPU_CTL_VOTE_RESULT 11          /* raftgpu_vote_result           - */
#define RAFTGPU_CTL_HAS_QUORUM 12           /* raftgpu_has_quorum            a[0] = slot mask */
#define RAFTGPU_CTL_QUORUM_RECENTLY_ACTIVE 13 /* raftgpu_quorum_recently_active peer_slot = perspective_of */
#define RAFTGPU_CTL_PROGRESS_OP 14          /* raftgpu_progress_op           peer_slot, arg = RAFTGPU_POP_*, a[0..2] */

/* Run a list of control commands for many groups in a few launches (the store-wide election after a restart, the
 * check_quorum sweep, region splits).  The contract: the arena, every results[i], the device counters and the
 * arena's meta mirror end exactly as calling the single-group entry points one at a time, in list order, would
 * leave them.  A command its single call would refuse (an unallocated group, the high half of a wide group, an
 * absent peer, a mask too wide, an unknown RAFTGPU_POP_* code) does nothing and carries that status, and an unknown
 * op carries RAFTGPU_ERR_INVALID whatever its group; the other commands still run.  Returns RAFTGPU_OK when the list ran (n == 0 included), RAFTGPU_ERR_INVALID for a NULL
 * cmds / results with n > 0, RAFTGPU_ERR_BUSY while records are enqueued for a step, RAFTGPU_ERR_CUDA on a CUDA
 * failure.  A list longer than the arena's staging buffer runs in list-order chunks.  Synchronous; needs exclusive
 * access (see the threading note at the top). */
int32_t raftgpu_control(raftgpu_arena *arena, const raftgpu_ctl_cmd *cmds, uint64_t n, raftgpu_ctl_result *results);

/* ---- plumbing ------------------------------------------------------------ */
int32_t raftgpu_counters_read(raftgpu_arena *arena, raftgpu_counters *out);
int32_t raftgpu_synchronize(raftgpu_arena *arena);
/* Diagnostics: 8 u64 slots the fused kernel fills when RAFTGPU_TILE_DEBUG is set (cycle totals
 * of its phases: wait for loads, records, recompute, stores; [4] = tiles). */
int32_t raftgpu_debug_read(raftgpu_arena *arena, uint64_t *out8);
/* Device scratch owned by the arena (for callers that keep record batches in
 * HBM, e.g. the bench's device-resident leg). */
int32_t raftgpu_device_alloc(raftgpu_arena *arena, uint64_t bytes, void **out_device_ptr);
int32_t raftgpu_device_free(raftgpu_arena *arena, void *device_ptr);
int32_t raftgpu_memcpy_h2d(raftgpu_arena *arena, void *device_dst, const void *host_src,
                           uint64_t bytes);
int32_t raftgpu_memcpy_d2h(raftgpu_arena *arena, void *host_dst, const void *device_src,
                           uint64_t bytes);

#ifdef __cplusplus
}
#endif
#endif /* RAFTGPU_H */
