/*
 * control_oracle.h -- CPU ORACLE of the control plane's list form. TEST INFRASTRUCTURE ONLY (see raft_oracle.h).
 *
 * ro_arena_control restates, for a list of control commands laid out as raftgpu_ctl_cmd, each reference method its
 * op names, on the arena view of raft_oracle.h.  It is built together with raft_oracle.c into its own library
 * (oracle/control_oracle.py) and uses that file's Progress, Inflights, quorum and log functions.
 */
#ifndef CONTROL_ORACLE_H
#define CONTROL_ORACLE_H

#include "raft_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One control command, laid out as raftgpu_ctl_cmd (40 bytes); op codes as RAFTGPU_CTL_*. */
typedef struct {
    uint32_t group;
    uint8_t op;
    uint8_t peer_slot; /* 0..15; SET_CONF: the self slot, 0xff = none */
    uint16_t arg;      /* PROGRESS_OP: the Progress method (RAFTGPU_POP_* order); RECORD_VOTE: 0 no / 1 yes; SET_GROUP_COMMIT */
    uint64_t a[4];
} ro_ctl_cmd;
typedef struct {
    int32_t status; /* 0, or the status the engine's single-group call returns (RAFTGPU_ERR_* values) */
    int32_t value;
} ro_ctl_result;
enum {
    RO_CTL_SET_CONF, RO_CTL_RESET, RO_CTL_BECOME_LEADER, RO_CTL_SET_LOG_BOUNDS, RO_CTL_SET_TERM, RO_CTL_COMMIT_TO,
    RO_CTL_MAYBE_COMMIT_TO, RO_CTL_SET_GROUP_COMMIT, RO_CTL_ASSIGN_COMMIT_GROUP, RO_CTL_RESET_VOTES, RO_CTL_RECORD_VOTE,
    RO_CTL_VOTE_RESULT, RO_CTL_HAS_QUORUM, RO_CTL_QUORUM_RECENTLY_ACTIVE, RO_CTL_PROGRESS_OP
};
#define RO_ERR_INVALID (-1)
#define RO_ERR_RANGE (-5)
#define RO_ERR_PEER_NOT_FOUND (-7)
#define RO_ERR_COMMIT_RANGE (-8)
#define RO_ERR_TOO_MANY_PEERS (-10)

/* Every command in list order, each the reference method its op names, on the arena's columns and `votes`
 * ([RO_SLOTS][cap], 0 missing / 1 no / 2 yes): apply_conf (tracker.rs:380-397), Raft::reset (raft.rs:942-971),
 * become_leader (raft.rs:1162-1203), record_vote / tally_votes (tracker.rs:301-340), has_quorum /
 * quorum_recently_active (tracker.rs:346-372), commit_to / maybe_commit (raft_log.rs:286-300, 487-499) and the
 * Progress methods (progress.rs:75-243, inflights.rs:54-123).  Groups [0, n_groups) are the allocated ones; a command
 * the engine's single-group call refuses does nothing and carries that call's status, and an unknown op carries
 * RO_ERR_INVALID whatever its group. */
void ro_arena_control(ro_arena_view *a, uint8_t *votes, const ro_ctl_cmd *cmds, size_t n, ro_ctl_result *results);

#ifdef __cplusplus
}
#endif
#endif /* CONTROL_ORACLE_H */
