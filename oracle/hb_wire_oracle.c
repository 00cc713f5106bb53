/* hb_wire_oracle.c -- see hb_wire_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#include "hb_wire_oracle.h"

#include <stdlib.h>
#include <string.h>

/* Base-128 varint as in wire_oracle.c; returns the bytes used, 0 = malformed. */
static size_t varint(const uint8_t *p, size_t len, uint64_t *out) {
    uint64_t v = 0;
    for (size_t i = 0; i < len && i < 10; i++) {
        v |= i < 9 ? (uint64_t)(p[i] & 0x7f) << (7 * i) : (uint64_t)(p[i] & 0x01) << 63;
        if (!(p[i] & 0x80)) {
            *out = v;
            return i + 1;
        }
    }
    return 0;
}

int hwo_decode_message(const uint8_t *buf, size_t len, hwo_message *out) {
    out->ctx_off = out->ctx_len = 0;
    if (!wo_decode_message(buf, len, &out->m)) return 0;
    /* a second walk over bytes known to be well-formed: where the last length-delimited field 12 lies */
    size_t pos = 0;
    while (pos < len) {
        uint64_t tag = 0, v = 0;
        pos += varint(buf + pos, len - pos, &tag);
        const uint32_t field = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
        if (wt == 0) {
            pos += varint(buf + pos, len - pos, &v);
        } else if (wt == 1) {
            pos += 8;
        } else if (wt == 5) {
            pos += 4;
        } else { /* wt == 2 */
            pos += varint(buf + pos, len - pos, &v);
            if (field == 12) { /* bytes context = 12 (eraftpb.proto:90); a varint field 12 is an unknown field */
                out->ctx_off = (uint32_t)pos;
                out->ctx_len = (uint32_t)v;
            }
            pos += (size_t)v;
        }
    }
    return 1;
}

void hwo_decode_batch(const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes, const uint64_t *group_term, uint32_t n_groups,
                      int read_queues, uint8_t *status, ro_append_resp *recs) {
    uint8_t *touched = (uint8_t *)calloc(n_groups ? n_groups : 1, 1); /* 8 slot bits per group */
    for (size_t i = 0; i < n; i++) {
        memset(&recs[i], 0, sizeof(recs[i]));
        const uint32_t lo = offsets[i], hi = offsets[i + 1];
        status[i] = WO_WIRE_MALFORMED;
        if (hi < lo || hi > n_bytes || hi - lo < 4) continue;
        uint32_t hdr;
        memcpy(&hdr, bytes + lo, 4);
        const uint32_t group = hdr >> 4, slot = hdr & 15u;
        hwo_message h;
        if (group >= n_groups || !hwo_decode_message(bytes + lo + 4, hi - lo - 4, &h)) continue;
        if (h.m.msg_type != 9) { /* MsgHeartbeatResponse, eraftpb.proto:59 */
            status[i] = WO_WIRE_SKIP_TYPE;
            continue;
        }
        if (group_term && group_term[group] != 0 && h.m.term != group_term[group]) {
            status[i] = WO_WIRE_TERM;
            continue;
        }
        uint64_t ctx = 0;
        if (h.ctx_len) {
            if (h.ctx_len != 8 || !read_queues) {
                status[i] = HWO_WIRE_CONTEXT;
                continue;
            }
            for (int k = 0; k < 8; k++) ctx |= (uint64_t)bytes[lo + 4 + h.ctx_off + k] << (8 * k);
        }
        if (slot < 8) {
            if (touched[group] & (1u << slot)) {
                status[i] = WO_WIRE_DUP;
                continue;
            }
            touched[group] |= (uint8_t)(1u << slot);
        }
        status[i] = WO_WIRE_OK;
        recs[i].group = group;
        recs[i].peer_slot = (uint8_t)slot;
        recs[i].flags = (uint8_t)(RO_REC_HEARTBEAT | (h.ctx_len ? RO_REC_READ_CTX : 0));
        recs[i].index = ctx;
        recs[i].commit = h.m.commit;
    }
    free(touched);
}

void hwo_apply(ro_arena_view *a, ro_read_queues *q, const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes,
               const uint64_t *group_term, uint8_t *status, ro_read_state *out, uint64_t *n_out) {
    ro_append_resp *recs = (ro_append_resp *)malloc((n ? n : 1) * sizeof(ro_append_resp));
    hwo_decode_batch(bytes, offsets, n, n_bytes, group_term, a->n_groups, q != NULL, status, recs);
    size_t m = 0;
    for (size_t i = 0; i < n; i++) {
        if (status[i] == WO_WIRE_OK) {
            recs[m++] = recs[i]; /* (m <= i: a record is moved down before it is overwritten) */
            status[i] = (uint8_t)(ro_arena_handle_heartbeat_response(a, &recs[m - 1]) & 0xf); /* raft.rs:1777-1804 */
        } else {
            status[i] = (uint8_t)(status[i] << 4);
        }
    }
    /* the read part (raft.rs:1805-1818) reads only the configuration, which the tracker part leaves alone: the same
     * records after every tracker update give what interleaving them would */
    *n_out = 0;
    if (q) ro_read_ack_seq(a, q, recs, m, out, n_out);
    free(recs);
}
