/* hb_frames_oracle.c -- see hb_frames_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#include "hb_frames_oracle.h"

#include <string.h>

#define NO_TERM_START UINT64_MAX

static uint8_t *put_varint(uint8_t *p, uint64_t v) {
    do {
        uint8_t b = (uint8_t)(v & 0x7f);
        v >>= 7;
        if (v) b |= 0x80;
        *p++ = b;
    } while (v);
    return p;
}

/* proto3: a scalar field that holds 0 is not written (tag = field number << 3 | wire type) */
static uint8_t *put_u64_field(uint8_t *p, uint32_t field, uint64_t v) {
    if (v == 0) return p;
    p = put_varint(p, (uint64_t)field << 3);
    return put_varint(p, v);
}

size_t hfo_encode_heartbeat(uint64_t to, uint64_t from, uint64_t term, uint64_t commit, uint64_t ctx, uint8_t *out) {
    uint8_t *p = out;
    p = put_u64_field(p, 1, 8); /* msg_type = MsgHeartbeat, eraftpb.proto:58 */
    p = put_u64_field(p, 2, to);
    p = put_u64_field(p, 3, from);
    p = put_u64_field(p, 4, term);
    p = put_u64_field(p, 8, commit);
    if (ctx) { /* bytes context = 12: length-delimited */
        p = put_varint(p, 12u << 3 | 2u);
        p = put_varint(p, 8);
        for (int k = 0; k < 8; k++) *p++ = (uint8_t)(ctx >> (8 * k));
    }
    return (size_t)(p - out);
}

/* One message of send_heartbeat + send, as a frame at bytes + *len. */
typedef struct {
    uint8_t *bytes;
    uint32_t *offsets;
    uint64_t frames, len;
} out_t;

static void emit(out_t *o, uint32_t cell_group, uint32_t slot, uint64_t to, uint64_t from, uint64_t term, uint64_t commit,
                 uint64_t ctx) {
    uint8_t *p = o->bytes + o->len;
    const uint32_t hdr = cell_group << 4 | slot;
    memcpy(p, &hdr, 4); /* little-endian host */
    const size_t m = hfo_encode_heartbeat(to, from, term, commit, ctx, p + 4);
    o->offsets[o->frames++] = (uint32_t)o->len;
    o->len += 4 + m;
}

void hfo_bcast_heartbeats(const ro_arena_view *a, const ro_read_queues *q, uint32_t first, uint32_t n, const uint32_t *select,
                          const uint64_t *ids, uint8_t *bytes, uint32_t *offsets, uint64_t *totals) {
    out_t o = {bytes, offsets, 0, 0};
    uint64_t no_term = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t g = first + i;
        if (a->meta[g] & RO_META_WIDE_HI) continue; /* sent with its low half */
        const int wide = (a->meta[g] & RO_META_WIDE_LO) != 0;
        if (g >= a->n_groups || (q && !q->allocated[g])) continue;
        if (select && !((select[g / 32] >> (g % 32)) & 1u)) continue;
        /* Raft::ping: MsgBeat reaches step_leader only (raft.rs:868-878) */
        if (a->term_start[g] == NO_TERM_START) continue;
        const uint64_t term = a->term[g];
        if (term == 0) { /* a term-less message would be a local one: not sent, reported */
            no_term++;
            continue;
        }
        const uint64_t ctx = q ? ro_read_last_ctx(q, g) : 0;  /* read_only.rs:132-135 */
        uint64_t committed = a->committed[g];
        if (wide && a->committed[g + 1] > committed) committed = a->committed[g + 1];
        const uint64_t self_id = ids[(size_t)RO_SLOTS * n + i];
        /* bcast_heartbeat_with_ctx: every Progress of the tracker (both halves of a wide group) but self */
        for (uint32_t half = 0; half < (wide ? 2u : 1u); half++) {
            const uint32_t h = g + half;
            const uint32_t meta = a->meta[h];
            const uint32_t present = (meta & 0xffu) | ((meta >> 8) & 0xffu) | ((meta >> 16) & 0xffu);
            for (uint32_t s = 0; s < RO_SLOTS; s++) {
                if (!((present >> s) & 1u)) continue;
                if ((meta & 0x08000000u) && ((meta >> 24) & 7u) == s) continue; /* id == self_id */
                const uint64_t matched = a->matched[(size_t)s * a->cap + h];
                const uint64_t commit = matched < committed ? matched : committed; /* raft.rs:838-840 */
                emit(&o, h, s, ids[(size_t)s * n + (h - first)], self_id, term, commit, ctx);
            }
        }
    }
    o.offsets[o.frames] = (uint32_t)o.len;
    totals[0] = o.frames;
    totals[1] = o.len;
    totals[2] = no_term;
}
