/* app_frames_oracle.c -- see app_frames_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#include "app_frames_oracle.h"

#include <string.h>

#define NO_TERM_START UINT64_MAX
#define INVALID_INDEX 0u

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

size_t afo_encode_append(uint64_t to, uint64_t from, uint64_t term, uint64_t log_term, uint64_t index, uint64_t commit,
                         uint8_t *out) {
    uint8_t *p = out;
    p = put_u64_field(p, 1, 3); /* msg_type = MsgAppend, eraftpb.proto:53 */
    p = put_u64_field(p, 2, to);
    p = put_u64_field(p, 3, from);
    p = put_u64_field(p, 4, term);
    p = put_u64_field(p, 5, log_term);
    p = put_u64_field(p, 6, index);
    p = put_u64_field(p, 8, commit); /* no entries (7) */
    return (size_t)(p - out);
}

/* Progress::is_paused, progress.rs:210-216 */
static int is_paused(uint8_t f) {
    switch (f & RO_PF_STATE_MASK) {
    case RO_STATE_PROBE: return (f & RO_PF_PAUSED) != 0;
    case RO_STATE_REPLICATE: return (f & RO_PF_INS_FULL) != 0;
    default: return 1;
    }
}

typedef struct {
    uint8_t *bytes;
    uint32_t *offsets;
    ro_send_entry *rest;
    uint64_t frames, len, n_rest;
} out_t;

void afo_bcast_append(const ro_arena_view *a, const ro_read_queues *q, uint32_t first, uint32_t n, const uint32_t *select,
                      const uint64_t *ids, uint8_t *bytes, uint32_t *offsets, ro_send_entry *rest, uint64_t *totals) {
    out_t o = {bytes, offsets, rest, 0, 0, 0};
    uint64_t no_term = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t g = first + i;
        if (a->meta[g] & RO_META_WIDE_HI) continue; /* sent with its low half */
        const int wide = (a->meta[g] & RO_META_WIDE_LO) != 0;
        if (g >= a->n_groups || (q && !q->allocated[g])) continue;
        if (select && !((select[g / 32] >> (g % 32)) & 1u)) continue;
        /* only a leader's maybe_commit broadcasts (raft.rs:1745-1748) */
        const uint64_t term_start = a->term_start[g];
        if (term_start == NO_TERM_START) continue;
        const uint64_t term = a->term[g];
        if (term == 0) { /* a term-less message would be a local one: not sent, reported */
            no_term++;
            continue;
        }
        uint64_t committed = a->committed[g], last_index = a->last_index[g];
        if (wide && a->committed[g + 1] > committed) committed = a->committed[g + 1];
        if (wide && a->last_index[g + 1] > last_index) last_index = a->last_index[g + 1];
        const uint64_t self_id = ids[(size_t)RO_SLOTS * n + i];
        for (uint32_t half = 0; half < (wide ? 2u : 1u); half++) {
            const uint32_t h = g + half;
            const uint32_t meta = a->meta[h];
            const uint32_t present = RO_META_IN(meta) | RO_META_OUT(meta) | RO_META_LEARN(meta);
            for (uint32_t s = 0; s < RO_SLOTS; s++) {
                if (!((present >> s) & 1u)) continue;
                if ((meta & RO_META_HAS_SELF) && RO_META_SELF(meta) == s) continue; /* :863 id != self_id */
                const size_t c = (size_t)s * a->cap + h;
                if (is_paused(a->pflags[c])) continue; /* :780-788 */
                const uint64_t next_idx = a->next_idx[c];
                const int snapshot = a->pending_request_snapshot[c] != INVALID_INDEX; /* :792-797 */
                /* entries(next_idx) is empty iff next_idx > last_index; term(next_idx - 1) is known without the log iff
                 * next_idx - 1 >= term_start (the group's term up to last_index, 0 above it) */
                if (snapshot || next_idx <= last_index || next_idx - 1 < term_start) {
                    ro_send_entry *e = &o.rest[o.n_rest++];
                    e->group = h;
                    e->peer_slot = (uint8_t)s;
                    e->flags = snapshot ? 1 : 0;
                    e->reserved = 0;
                    e->next_idx = next_idx;
                    continue;
                }
                const uint64_t index = next_idx - 1;
                const uint64_t log_term = index <= last_index ? term : 0;
                uint8_t *p = o.bytes + o.len;
                const uint32_t hdr = h << 4 | s;
                memcpy(p, &hdr, 4); /* little-endian host */
                const size_t m = afo_encode_append(ids[(size_t)s * n + (h - first)], self_id, term, log_term, index,
                                                   committed, p + 4);
                o.offsets[o.frames++] = (uint32_t)o.len;
                o.len += 4 + m;
            }
        }
    }
    o.offsets[o.frames] = (uint32_t)o.len;
    totals[0] = o.frames;
    totals[1] = o.len;
    totals[2] = o.n_rest;
    totals[3] = no_term;
}
