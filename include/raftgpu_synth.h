/*
 * raftgpu_synth.h -- the synthetic AppendResponse workload of SURVEY.md 8(d) (bench.py, the tests,
 * scripts/).  NOT part of the product boundary: it lives in its own library, libraftgpu_synth.so
 * (csrc/synth.cpp, plain C++, no CUDA), so neither the engine nor a process that only generates
 * input (the CPU baseline arm) maps the other.  Deterministic: splitmix64(seed ^ counter).
 */
#ifndef RAFTGPU_SYNTH_H
#define RAFTGPU_SYNTH_H

#include "raftgpu.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Fills host columns for groups [0, n) of a K-peer configuration (`joint` != 0:
 * 7 slots, incoming = {0..4}, outgoing = {0,1,2,5,6}).  Arrays are [SLOTS][cap]
 * / [cap] like the arena's columns. */
typedef struct {
    uint32_t cap;
    uint32_t n_groups;
    /* initial arena columns: written by raftgpu_synth_init only */
    uint64_t *matched, *next_idx, *peer_committed;
    uint8_t *pflags;
    uint32_t *meta;
    uint64_t *committed, *term_start, *last_index, *term;
    /* follower simulation, advanced by raftgpu_synth_round */
    uint64_t *sim_acked; /* [SLOTS][cap] last index each peer acknowledged */
    uint64_t *sim_last;  /* [cap] the leader's last_index */
    uint8_t *sim_flags;  /* [SLOTS][cap] bit 0: the peer's previous response was a reject */
} raftgpu_synth_columns;
int32_t raftgpu_synth_init(const raftgpu_synth_columns *cols, uint64_t seed, uint32_t k_peers,
                           int32_t joint);
/* Generates ONE round for all groups from the follower simulation: 1 + r mod (K-1)
 * distinct followers answer (88 % accept, 10 % stale accept, 2 % reject = REJECT +
 * EXT), then one RAFTGPU_REC_LOCAL record advances the leader's log / persisted
 * index.  At most one record per (group, peer): a round is one wave.  Records are
 * in group order.  Returns the count in *out_n, or RAFTGPU_ERR_FULL. */
int32_t raftgpu_synth_round(const raftgpu_synth_columns *cols, uint64_t seed, uint32_t round,
                            uint32_t k_peers, raftgpu_append_resp *out, uint64_t max_records,
                            uint64_t *out_n);

/* The records of one round as a transport holds them (SURVEY 8(f4)): follower records -> frames of
 * serialized eraftpb.Message (u32 header group << 4 | peer_slot, then the protobuf bytes; a REJECT's EXT
 * becomes reject_hint / request_snapshot), leader-local records -> out_local as they are.  term: [cap] the
 * groups' terms (NULL = 1).  out_offsets has room for n + 1 entries, out_local for n records. */
int32_t raftgpu_synth_wire_encode(const raftgpu_append_resp *recs, uint64_t n, const uint64_t *term, uint8_t *out_bytes,
                                  uint64_t bytes_cap, uint32_t *out_offsets, uint64_t *out_n_frames, uint64_t *out_n_bytes,
                                  raftgpu_append_resp *out_local, uint64_t *out_n_local);

/* RAFTGPU_REC_HEARTBEAT records -> MsgHeartbeatResponse frames, one per such record in record order (others are
 * skipped): msg_type 9, term (term[group], NULL = 1), commit, and for a RAFTGPU_REC_READ_CTX record with a non-zero
 * ctx id (`index`) the context = the id's 8 bytes, little-endian.  out_offsets has room for n + 1 entries. */
int32_t raftgpu_synth_wire_encode_heartbeats(const raftgpu_append_resp *recs, uint64_t n, const uint64_t *term,
                                             uint8_t *out_bytes, uint64_t bytes_cap, uint32_t *out_offsets,
                                             uint64_t *out_n_frames, uint64_t *out_n_bytes);

/* One vote response as raftgpu_synth_wire_encode_votes writes it (56 bytes). */
typedef struct raftgpu_synth_vote {
    uint32_t hdr;      /* the frame's u32 header: group << 4 | peer_slot */
    uint32_t msg_type; /* MsgRequestVoteResponse (6) or MsgRequestPreVoteResponse (18) */
    uint64_t to, from, term, commit, commit_term;
    uint32_t reject;   /* 0 or 1 */
    uint32_t reserved;
} raftgpu_synth_vote;

/* Vote responses -> frames, one per entry in order: the header, then eraftpb.Message with msg_type, to, from, term,
 * commit, reject and commit_term, fields in number order and zero scalars omitted (the canonical proto3 encoding:
 * at most 63 bytes a frame, header included).  out_offsets has room for n + 1 entries.  RAFTGPU_ERR_FULL when bytes_cap is short. */
int32_t raftgpu_synth_wire_encode_votes(const raftgpu_synth_vote *votes, uint64_t n, uint8_t *out_bytes, uint64_t bytes_cap,
                                        uint32_t *out_offsets, uint64_t *out_n_bytes);

/* One vote request as raftgpu_synth_wire_encode_vote_requests writes it (104 bytes). */
typedef struct raftgpu_synth_vote_request {
    uint32_t hdr;      /* the frame's u32 header: group << 4 | x */
    uint32_t msg_type; /* MsgRequestVote (5) or MsgRequestPreVote (17) */
    uint64_t to, from, term, log_term, index, commit, commit_term, priority;
    uint8_t context[24];  /* the first context_len bytes are the context */
    uint32_t context_len; /* 0 (none) .. 24 */
    uint32_t reserved;
} raftgpu_synth_vote_request;

/* Vote requests -> frames, one per entry in order: the header, then eraftpb.Message with msg_type, to, from, term,
 * log_term, index, commit, context, priority and commit_term, fields in number order and zero scalars and an empty
 * context omitted (the canonical proto3 encoding: at most 120 bytes a frame, header included).  out_offsets has room for
 * n + 1 entries.  RAFTGPU_ERR_FULL when bytes_cap is short, RAFTGPU_ERR_INVALID for a context_len past 24. */
int32_t raftgpu_synth_wire_encode_vote_requests(const raftgpu_synth_vote_request *reqs, uint64_t n, uint8_t *out_bytes,
                                                uint64_t bytes_cap, uint32_t *out_offsets, uint64_t *out_n_bytes);

#ifdef __cplusplus
}
#endif
#endif /* RAFTGPU_SYNTH_H */
