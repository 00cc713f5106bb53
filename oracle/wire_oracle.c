/* wire_oracle.c -- see wire_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#include "wire_oracle.h"

#include <stdlib.h>
#include <string.h>

/* Base-128 varint (protobuf encoding guide): 7 bits per byte, least significant group first, the
 * high bit says "more".  At most 10 bytes; the tenth contributes its lowest bit only (what protobuf
 * parsers do with the bits that do not fit 64).  Returns the number of bytes used, 0 = malformed. */
static size_t wo_varint(const uint8_t *p, size_t len, uint64_t *out) {
    uint64_t v = 0;
    for (size_t i = 0; i < len && i < 10; i++) {
        const uint8_t b = p[i];
        if (i < 9)
            v |= (uint64_t)(b & 0x7f) << (7 * i);
        else
            v |= (uint64_t)(b & 0x01) << 63;
        if (!(b & 0x80)) {
            *out = v;
            return i + 1;
        }
    }
    return 0; /* ran out of bytes, or an 11th byte would be needed */
}

int wo_decode_message(const uint8_t *buf, size_t len, wo_message *out) {
    memset(out, 0, sizeof(*out));
    size_t pos = 0;
    while (pos < len) {
        /* tag: a varint of at most 5 bytes whose value fits 32 bits; field number 1 .. 2^29 - 1 */
        uint64_t tag;
        const size_t tl = wo_varint(buf + pos, len - pos < 5 ? len - pos : 5, &tag);
        if (tl == 0 || tag > 0xffffffffull) return 0;
        pos += tl;
        const uint32_t field = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
        if (field == 0) return 0;
        if (wt == 0) {
            uint64_t v;
            const size_t vl = wo_varint(buf + pos, len - pos, &v);
            if (vl == 0) return 0;
            pos += vl;
            switch (field) { /* eraftpb.proto:71-92 */
            case 1: out->msg_type = (uint32_t)v; break;
            case 2: out->to = v; break;
            case 3: out->from = v; break;
            case 4: out->term = v; break;
            case 5: out->log_term = v; break;
            case 6: out->index = v; break;
            case 8: out->commit = v; break;
            case 10: out->reject = v != 0; break;
            case 11: out->reject_hint = v; break;
            case 13: out->request_snapshot = v; break;
            case 14: out->priority = v; break;
            case 15: out->commit_term = v; break;
            default: break; /* unknown field, or a varint where the schema has bytes / a message */
            }
        } else if (wt == 1) {
            if (len - pos < 8) return 0;
            pos += 8;
        } else if (wt == 5) {
            if (len - pos < 4) return 0;
            pos += 4;
        } else if (wt == 2) {
            uint64_t l;
            const size_t ll = wo_varint(buf + pos, len - pos, &l);
            if (ll == 0) return 0;
            pos += ll;
            if (l > len - pos) return 0;
            pos += (size_t)l; /* entries / snapshot / context / unknown bytes: not on this path */
        } else {
            return 0; /* groups (3, 4) are not part of proto3 messages; 6, 7 do not exist */
        }
    }
    return 1;
}

void wo_decode_batch(const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes, const uint64_t *group_term,
                     uint32_t n_groups, uint8_t *status, wo_record *recs, uint64_t *hint, uint64_t *request_snapshot) {
    uint8_t *touched = (uint8_t *)calloc(n_groups ? n_groups : 1, 2); /* 16 slot bits per group */
    for (size_t i = 0; i < n; i++) {
        memset(&recs[i], 0, sizeof(recs[i]));
        hint[i] = 0;
        request_snapshot[i] = 0;
        const uint32_t lo = offsets[i], hi = offsets[i + 1];
        if (hi < lo || hi > n_bytes || hi - lo < 4) {
            status[i] = WO_WIRE_MALFORMED;
            continue;
        }
        uint32_t hdr;
        memcpy(&hdr, bytes + lo, 4);
        const uint32_t group = hdr >> 4, slot = hdr & 15u;
        wo_message m;
        if (group >= n_groups || !wo_decode_message(bytes + lo + 4, hi - lo - 4, &m)) {
            status[i] = WO_WIRE_MALFORMED;
            continue;
        }
        if (m.msg_type != 4) { /* MsgAppendResponse, eraftpb.proto:54 */
            status[i] = WO_WIRE_SKIP_TYPE;
            continue;
        }
        if (group_term && group_term[group] != 0 && m.term != group_term[group]) {
            status[i] = WO_WIRE_TERM;
            continue;
        }
        if (m.reject && m.log_term > 0) { /* raft.rs:1562: next_probe_index comes from the leader's log */
            status[i] = WO_WIRE_NEEDS_LOG;
            continue;
        }
        if (slot < 8) { /* the arena's peer slots; a frame naming another slot finds no Progress (raft.rs:1663-1673) */
            uint16_t t;
            memcpy(&t, touched + 2 * (size_t)group, 2);
            if (t & (1u << slot)) {
                status[i] = WO_WIRE_DUP;
                continue;
            }
            t |= (uint16_t)(1u << slot);
            memcpy(touched + 2 * (size_t)group, &t, 2);
        }
        status[i] = WO_WIRE_OK;
        recs[i].group = group;
        recs[i].peer_slot = (uint8_t)slot;
        recs[i].flags = m.reject ? 0x01 : 0x00;
        recs[i].index = m.index;
        recs[i].commit = m.commit;
        hint[i] = m.reject_hint;               /* raft.rs:1560 */
        request_snapshot[i] = m.request_snapshot; /* raft.rs:1709 */
    }
    free(touched);
}
