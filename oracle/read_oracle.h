/*
 * read_oracle.h -- CPU ORACLE of ReadIndex with ReadOnlyOption::Safe. TEST INFRASTRUCTURE ONLY (see raft_oracle.h).
 *
 * A literal restatement of ReadOnly (src/read_only.rs:86-139) per group -- a FIFO queue, each entry a context, the
 * index it was queued with and its acks -- and of the pieces of src/raft.rs that drive it: the MsgReadIndex arm of
 * step_leader (raft.rs:2056-2091), the tail of handle_heartbeat_response (raft.rs:1805-1818), Raft::reset
 * (raft.rs:957) and the tail of post_conf_change (raft.rs:2648-2664).  Messages are processed one at a time, in the
 * order given.  Contexts are u64 ids (0 = none), acks are peer-slot masks (peer 8 + s of a wide group is bit 8 + s),
 * and a peer removed by a configuration change loses its bits, as on the device (DESIGN.md 3.9 states that
 * deviation); the queue holds at most max_pending entries (RO_READ_FULL).
 *
 * Built together with control_oracle.c and raft_oracle.c into its own library (oracle/read_oracle.py).
 */
#ifndef READ_ORACLE_H
#define READ_ORACLE_H

#include "control_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
    uint32_t group;
    uint32_t reserved;
    uint64_t ctx;
} ro_read_req; /* raftgpu_read_req */
typedef struct {
    uint32_t group;
    uint32_t reserved;
    uint64_t ctx;
    uint64_t index;
} ro_read_state; /* raftgpu_read_state: ReadIndexStatus minus the message, read_only.rs:58-63 */

/* The ReadOnly of every group slot (the low half of a wide group holds the wide group's): entries [0, count[g]) of
 * row g, front first (pending_read_index + read_index_queue, read_only.rs:69-70: a ctx's map entry and its queue
 * position are kept together), and whether the slot is allocated. */
typedef struct {
    uint32_t cap, max_pending;
    uint32_t *count;   /* [cap] */
    uint64_t *ctx;     /* [cap][max_pending] */
    uint64_t *index;   /* [cap][max_pending] */
    uint16_t *acks;    /* [cap][max_pending] */
    uint8_t *allocated; /* [cap] */
} ro_read_queues;

/* per-request result, as RAFTGPU_READ_* */
enum { RO_READ_QUEUED = 1, RO_READ_READY, RO_READ_DUP, RO_READ_DROPPED, RO_READ_FULL, RO_READ_NO_GROUP, RO_READ_NO_CTX };
#define RO_REC_READ_CTX 0x08u

/* MsgReadIndex at the leader for each request in order (raft.rs:2056-2091); ready reads are appended to out. */
void ro_read_request(const ro_arena_view *a, ro_read_queues *q, const ro_read_req *reqs, size_t n, uint8_t *results,
                     ro_read_state *out, uint64_t *n_out);
/* The read tail of handle_heartbeat_response (raft.rs:1805-1818) for each record in order: recv_ack, has_quorum,
 * advance.  Records that are not RO_REC_HEARTBEAT | RO_REC_READ_CTX are skipped. */
void ro_read_ack_seq(const ro_arena_view *a, ro_read_queues *q, const ro_append_resp *recs, size_t n, ro_read_state *out,
                     uint64_t *n_out);
/* The same batch in the device's formulation (DESIGN.md 3.9): every recv_ack first, then per group (in the order
 * groups first appear in the batch) advance to the last entry that an ack of the batch named and whose acks have a
 * quorum. */
void ro_read_ack_batch(const ro_arena_view *a, ro_read_queues *q, const ro_append_resp *recs, size_t n, ro_read_state *out,
                       uint64_t *n_out);
/* post_conf_change's read tail (raft.rs:2648-2664) for each listed group, in order. */
void ro_read_recheck(const ro_arena_view *a, ro_read_queues *q, const uint32_t *groups, size_t n, ro_read_state *out,
                     uint64_t *n_out);
/* ReadOnly::last_pending_request_ctx (read_only.rs:132-135); 0 for none. */
uint64_t ro_read_last_ctx(const ro_read_queues *q, uint32_t g);
/* Every control command in list order (ro_arena_control), with the read state's hooks: RESET replaces the ReadOnly
 * (raft.rs:957), SET_CONF clears the bits of removed peers. */
void ro_read_control(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const ro_ctl_cmd *cmds, size_t n,
                     ro_ctl_result *results);

#ifdef __cplusplus
}
#endif
#endif /* READ_ORACLE_H */
