/*
 * hb_wire_oracle.h -- CPU ORACLE of MsgHeartbeatResponse frames on the wire. TEST INFRASTRUCTURE ONLY (see
 * raft_oracle.h).
 *
 * What it restates: the decode of wire_oracle.h with the context field (bytes context = 12, eraftpb.proto:90; the
 * last length-delimited occurrence wins, as a protobuf parser keeps the last value of a singular field), the statuses
 * a heartbeat-response frame can get, and Raft::handle_heartbeat_response (raft.rs:1777-1819) for the frames that
 * are applied, one at a time in frame order: ro_arena_handle_heartbeat_response (the tracker part, raft_oracle.h)
 * and ro_read_ack_seq (the read part, read_oracle.h).  The context of a heartbeat that carries read id x is the 8
 * bytes of x, little-endian.
 *
 * Built together with wire_oracle.c, read_oracle.c, control_oracle.c and raft_oracle.c into its own library
 * (oracle/hb_wire_oracle.py).
 */
#ifndef HB_WIRE_ORACLE_H
#define HB_WIRE_ORACLE_H

#include "read_oracle.h"
#include "wire_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the scalar fields (wo_message) and where the context lies: bytes [ctx_off, ctx_off + ctx_len) of the message */
typedef struct {
    wo_message m;
    uint32_t ctx_off, ctx_len;
} hwo_message;

/* 1 when the bytes are a well-formed protobuf message (wo_decode_message's verdict), 0 otherwise. */
int hwo_decode_message(const uint8_t *buf, size_t len, hwo_message *out);

/* status of a heartbeat-response frame (== RAFTGPU_WIRE_*): WO_WIRE_OK, SKIP_TYPE, TERM, MALFORMED, DUP and */
enum { HWO_WIRE_CONTEXT = 6 }; /* a context that is not 8 bytes, or any context without read queues */

/* Every frame's status and, for WO_WIRE_OK frames, the record the reference's handle_heartbeat_response consumes:
 * RO_REC_HEARTBEAT (| RO_REC_READ_CTX with the id in `index` when the context is 8 bytes), commit = m.commit; zero
 * records for the others.  read_queues: whether the arena keeps read queues.  Checks in order: frame / group /
 * protobuf (MALFORMED), msg_type 9 (SKIP_TYPE), group_term (TERM; NULL or 0 = not checked), the context (CONTEXT),
 * then the first frame of a (group, slot < 8) cell wins and later ones are DUP. */
void hwo_decode_batch(const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes, const uint64_t *group_term, uint32_t n_groups,
                      int read_queues, uint8_t *status, ro_append_resp *recs);

/* Decode, then handle_heartbeat_response for the applied frames in frame order: status[i] = WO_WIRE_* << 4 |
 * RO_RES_* of the tracker part; the read part (q != NULL) appends released reads to out. */
void hwo_apply(ro_arena_view *a, ro_read_queues *q, const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes,
               const uint64_t *group_term, uint8_t *status, ro_read_state *out, uint64_t *n_out);

#ifdef __cplusplus
}
#endif
#endif /* HB_WIRE_ORACLE_H */
