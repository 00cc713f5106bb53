/* app_entries_oracle.c -- see app_entries_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#define _POSIX_C_SOURCE 199309L
#include "app_entries_oracle.h"

#include <stdlib.h>
#include <string.h>
#include <time.h>

#define NO_TERM_START UINT64_MAX

static uint64_t max64(uint64_t x, uint64_t y) { return x > y ? x : y; }
static uint64_t min64(uint64_t x, uint64_t y) { return x < y ? x : y; }

/* a varint of at most max bytes inside [p, p + len): bytes used, 0 = none */
static size_t varint(const uint8_t *p, size_t len, size_t max, uint64_t *out) {
    uint64_t v = 0;
    for (size_t i = 0; i < len && i < max; i++) {
        v |= i < 9 ? (uint64_t)(p[i] & 0x7f) << (7 * i) : (uint64_t)(p[i] & 1) << 63;
        if (!(p[i] & 0x80)) {
            *out = v;
            return i + 1;
        }
    }
    return 0;
}

/* One protobuf message's fields: 0 when it is not well formed.  Entry: term (2) and index (3), the last value of each
 * varint occurrence; other fields and other wire types are skipped. */
static int entry(const uint8_t *p, size_t len, uint64_t *term, uint64_t *index) {
    *term = *index = 0;
    size_t pos = 0;
    while (pos < len) {
        uint64_t tag, v;
        size_t k = varint(p + pos, len - pos, 5, &tag);
        if (!k || tag > 0xffffffffu || (tag >> 3) == 0) return 0;
        pos += k;
        switch (tag & 7) {
        case 0:
            if (!(k = varint(p + pos, len - pos, 10, &v))) return 0;
            pos += k;
            if ((tag >> 3) == 2) *term = v;
            if ((tag >> 3) == 3) *index = v;
            break;
        case 1:
        case 5:
            if (len - pos < ((tag & 7) == 1 ? 8u : 4u)) return 0;
            pos += (tag & 7) == 1 ? 8 : 4;
            break;
        case 2:
            if (!(k = varint(p + pos, len - pos, 10, &v)) || v > len - pos - k) return 0;
            pos += k + (size_t)v;
            break;
        default:
            return 0;
        }
    }
    return 1;
}

int aeo_decode(const uint8_t *buf, size_t len, wo_message *m, aeo_entry *ents, size_t max_ents, size_t *n) {
    *n = 0;
    if (!wo_decode_message(buf, len, m)) return 0;
    size_t pos = 0; /* well formed: every tag, varint and length below is in range */
    while (pos < len) {
        const size_t at = pos;
        uint64_t tag = 0, v = 0;
        pos += varint(buf + pos, len - pos, 5, &tag);
        const uint32_t wt = (uint32_t)(tag & 7);
        aeo_entry e = {0, 0, (uint32_t)at, 0, wt == 2, 0};
        if (wt == 0) {
            pos += varint(buf + pos, len - pos, 10, &v);
        } else if (wt == 2) {
            pos += varint(buf + pos, len - pos, 10, &v);
            if ((tag >> 3) == 7 && !entry(buf + pos, (size_t)v, &e.term, &e.index)) return 0;
            pos += (size_t)v;
        } else {
            pos += wt == 1 ? 8 : 4;
        }
        e.end = (uint32_t)pos;
        if ((tag >> 3) == 7) {
            if (*n < max_ents) ents[*n] = e;
            ++*n;
        }
    }
    return 1;
}

static void respond(uint8_t *resp, uint32_t *resp_offsets, uint64_t *totals, uint32_t hdr, uint64_t to, uint64_t from,
                    uint64_t term, uint64_t log_term, uint64_t index, uint64_t commit, int reject, uint64_t reject_hint) {
    uint8_t *p = resp + totals[1];
    memcpy(p, &hdr, 4); /* little-endian host */
    const size_t k = 4 + afl_encode_response(to, from, term, log_term, index, commit, reject, reject_hint, p + 4);
    resp_offsets[totals[0]++] = (uint32_t)totals[1];
    totals[1] += k;
    resp_offsets[totals[0]] = (uint32_t)totals[1];
}

static uint64_t pair_max(const ro_arena_view *a, const uint64_t *col, uint32_t g) {
    return (a->meta[g] & RO_META_WIDE_LO) ? max64(col[g], col[g + 1]) : col[g];
}

void aeo_batch(ro_arena_view *a, const ro_read_queues *q, afl_log *logs, const uint8_t *bytes, const uint32_t *offsets,
               size_t n, uint64_t n_bytes, uint8_t *status, uint64_t *from, aeo_appended *appended, uint8_t *resp,
               uint32_t *resp_offsets, uint64_t *totals) {
    uint8_t *claimed = (uint8_t *)calloc(a->n_groups ? a->n_groups : 1, 1);
    size_t cap = 64;
    aeo_entry *ents = (aeo_entry *)malloc(cap * sizeof(aeo_entry));
    totals[0] = totals[1] = 0;
    resp_offsets[0] = 0;
    for (size_t i = 0; i < n; i++) {
        status[i] = WO_WIRE_MALFORMED << 4;
        from[i] = 0;
        memset(&appended[i], 0, sizeof appended[i]);
        const uint32_t lo = offsets[i], hi = offsets[i + 1];
        if (hi < lo || hi > n_bytes || hi - lo < 4) continue;
        uint32_t hdr;
        memcpy(&hdr, bytes + lo, 4);
        const uint32_t g = hdr >> 4;
        wo_message m;
        size_t n7 = 0;
        /* the Message alone first: an Entry that does not parse is MALFORMED only past TERM */
        if (g >= a->n_groups || !afl_decode(bytes + lo + 4, hi - lo - 4, &m, &n7, NULL, NULL, 0)) continue;
        if ((q && !q->allocated[g]) || (a->meta[g] & RO_META_WIDE_HI)) continue;
        if (m.msg_type != 3) {
            status[i] = WO_WIRE_SKIP_TYPE << 4;
            continue;
        }
        afl_log *l = &logs[g];
        if (!(l->flags & AFL_SELECT) || a->term_start[g] != NO_TERM_START) {
            status[i] = AFL_WIRE_ROLE << 4;
            continue;
        }
        const uint64_t term = a->term[g];
        if (term == 0 || m.term != term) {
            status[i] = WO_WIRE_TERM << 4;
            continue;
        }
        if (n7 > cap) {
            cap = n7;
            ents = (aeo_entry *)realloc(ents, cap * sizeof(aeo_entry));
        }
        if (!aeo_decode(bytes + lo + 4, hi - lo - 4, &m, ents, cap, &n7)) continue; /* an Entry: MALFORMED, no claim */
        if (claimed[g]) {
            status[i] = WO_WIRE_DUP << 4;
            continue;
        }
        claimed[g] = 1;
        const uint64_t last = pair_max(a, a->last_index, g), committed = pair_max(a, a->committed, g);
        const int known = m.index > last || (m.index >= l->run_start && m.index <= last);
        uint8_t flags = AFL_RES_OK;
        if (m.index < committed) { /* raft.rs:2394-2404, whatever the entries */
            respond(resp, resp_offsets, totals, hdr, m.from, l->id, term, 0, committed, committed, 0, 0);
            flags |= AFL_STALE;
        } else if (!known) {
            status[i] = WO_WIRE_NEEDS_LOG << 4;
            continue;
        } else if ((m.index > last ? 0 : l->run_term) == m.log_term) { /* maybe_append */
            /* what the pass hands back: a scalar field 7, a gap, indexes not m.index + 1.., a term 0 */
            int needs_log = n7 && m.index > last;
            for (size_t k = 0; k < n7; k++)
                if (!ents[k].ld || ents[k].index != m.index + 1 + k || ents[k].term == 0) needs_log = 1;
            /* find_conflict: term(j) = run_term up to last_index, 0 above */
            size_t first = n7;
            for (size_t k = 0; k < n7 && first == n7 && !needs_log; k++)
                if (ents[k].index > last || ents[k].term != l->run_term) first = k;
            for (size_t k = first + 1; k < n7 && !needs_log; k++) /* the appended records form one span */
                if (ents[k].off != ents[k - 1].end) needs_log = 1;
            if (needs_log) {
                status[i] = WO_WIRE_NEEDS_LOG << 4;
                continue;
            }
            const uint64_t conflict = first < n7 ? ents[first].index : 0;
            const uint64_t last_new = m.index + n7, new_last = conflict ? last_new : last;
            const uint64_t to_commit = min64(m.commit, last_new);
            /* the reference's fatal!s (:259-265, :291-298); unreachable past the stale rule (conflict > m.index >=
             * committed, to_commit <= last_new <= new_last), kept as the pass keeps them */
            if ((conflict && conflict <= committed) || to_commit > max64(committed, new_last)) {
                status[i] = AFL_WIRE_COMMIT_RANGE << 4;
                continue;
            }
            if (conflict) {
                const ro_ctl_cmd b = {g, RO_CTL_SET_LOG_BOUNDS, 0, 0, {NO_TERM_START, new_last, 0, 0}};
                ro_ctl_result r;
                ro_arena_control(a, NULL, &b, 1, &r);
                /* the run: the trailing block of appended entries with the last one's term */
                const uint64_t t = ents[n7 - 1].term;
                size_t k = n7 - 1;
                while (k > first && ents[k - 1].term == t) k--;
                if (!(k == first && t == l->run_term && conflict - 1 >= l->run_start)) {
                    l->run_start = ents[k].index;
                    l->run_term = t;
                }
                appended[i] = (aeo_appended){conflict, last_new, l->run_start, l->run_term, lo + 4 + ents[first].off,
                                             ents[n7 - 1].end - ents[first].off};
                flags |= AEO_APPENDED;
            }
            const ro_ctl_cmd c = {g, RO_CTL_COMMIT_TO, 0, 0, {to_commit, 0, 0, 0}};
            ro_ctl_result r;
            ro_arena_control(a, NULL, &c, 1, &r);
            respond(resp, resp_offsets, totals, hdr, m.from, l->id, term, 0, last_new, a->committed[g], 0, 0);
        } else { /* the rejection ignores the entries */
            const uint64_t h = min64(m.index, last);
            if (!(h >= l->run_start && h <= last) || l->run_term > m.log_term) {
                status[i] = WO_WIRE_NEEDS_LOG << 4;
                continue;
            }
            respond(resp, resp_offsets, totals, hdr, m.from, l->id, term, l->run_term, m.index, committed, 1, h);
            flags |= AFL_REJECT;
        }
        status[i] = (uint8_t)(WO_WIRE_OK << 4 | flags);
        from[i] = m.from;
    }
    free(ents);
    free(claimed);
}

double aeo_bench(ro_arena_view *a, const ro_read_queues *q, afl_log *logs, const uint8_t *bytes, const uint32_t *offsets,
                 size_t n, uint64_t n_bytes, uint8_t *status, uint64_t *from, aeo_appended *appended, uint8_t *resp,
                 uint32_t *resp_offsets, uint64_t *totals) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    aeo_batch(a, q, logs, bytes, offsets, n, n_bytes, status, from, appended, resp, resp_offsets, totals);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}
