/* app_follow_oracle.c -- see app_follow_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#define _POSIX_C_SOURCE 199309L
#include "app_follow_oracle.h"

#include <stdlib.h>
#include <string.h>
#include <time.h>

#define NO_TERM_START UINT64_MAX

static uint64_t max64(uint64_t x, uint64_t y) { return x > y ? x : y; }
static uint64_t min64(uint64_t x, uint64_t y) { return x < y ? x : y; }

static uint8_t *put_varint(uint8_t *p, uint64_t v) {
    while (v >= 0x80) {
        *p++ = (uint8_t)(v | 0x80);
        v >>= 7;
    }
    *p++ = (uint8_t)v;
    return p;
}

/* a varint of at most 10 bytes inside [p, p + len): bytes used, 0 = none */
static size_t get_varint(const uint8_t *p, size_t len, uint64_t *out) {
    uint64_t v = 0;
    for (size_t i = 0; i < len && i < 10; i++) {
        v |= i < 9 ? (uint64_t)(p[i] & 0x7f) << (7 * i) : (uint64_t)(p[i] & 1) << 63;
        if (!(p[i] & 0x80)) {
            *out = v;
            return i + 1;
        }
    }
    return 0;
}

size_t afl_encode_response(uint64_t to, uint64_t from, uint64_t term, uint64_t log_term, uint64_t index, uint64_t commit,
                           int reject, uint64_t reject_hint, uint8_t *out) {
    const uint32_t field[9] = {1, 2, 3, 4, 5, 6, 8, 10, 11};
    const uint64_t val[9] = {4, to, from, term, log_term, index, commit, reject ? 1u : 0u, reject_hint};
    uint8_t *p = out;
    for (int k = 0; k < 9; k++) {
        if (!val[k]) continue; /* proto3: a zero scalar is not written */
        p = put_varint(p, (uint64_t)field[k] << 3);
        p = put_varint(p, val[k]);
    }
    return (size_t)(p - out);
}

/* An Entry's term (2) and index (3); a sub-message that does not parse keeps what was read before the fault. */
static void entry_fields(const uint8_t *p, size_t len, uint64_t *term, uint64_t *index) {
    *term = *index = 0;
    size_t pos = 0;
    while (pos < len) {
        uint64_t tag, v;
        size_t k = get_varint(p + pos, len - pos, &tag);
        if (!k) return;
        pos += k;
        const uint32_t wt = (uint32_t)(tag & 7);
        if (wt == 0) {
            if (!(k = get_varint(p + pos, len - pos, &v))) return;
            pos += k;
            if ((tag >> 3) == 2) *term = v;
            if ((tag >> 3) == 3) *index = v;
        } else if (wt == 2) {
            if (!(k = get_varint(p + pos, len - pos, &v)) || v > len - pos - k) return;
            pos += k + (size_t)v;
        } else if (wt == 1 || wt == 5) {
            pos += wt == 1 ? 8 : 4;
        } else {
            return;
        }
    }
}

int afl_decode(const uint8_t *buf, size_t len, wo_message *m, size_t *n_fields7, uint64_t *ent_term, uint64_t *ent_index,
               size_t max_ents) {
    *n_fields7 = 0;
    if (!wo_decode_message(buf, len, m)) return 0;
    /* well formed: every tag, varint and length below is in range */
    size_t pos = 0;
    while (pos < len) {
        uint64_t tag = 0, v = 0;
        pos += get_varint(buf + pos, len - pos, &tag);
        const uint32_t field = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
        const size_t at = *n_fields7;
        if (field == 7) ++*n_fields7;
        if (wt == 0) {
            pos += get_varint(buf + pos, len - pos, &v);
        } else if (wt == 2) {
            pos += get_varint(buf + pos, len - pos, &v);
            if (field == 7 && at < max_ents) entry_fields(buf + pos, (size_t)v, &ent_term[at], &ent_index[at]);
            pos += (size_t)v;
        } else {
            pos += wt == 1 ? 8 : 4;
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

/* last_index and committed as raftgpu_group_get reports them: the larger of a pair's halves */
static uint64_t pair_max(const ro_arena_view *a, const uint64_t *col, uint32_t g) {
    return (a->meta[g] & RO_META_WIDE_LO) ? max64(col[g], col[g + 1]) : col[g];
}

void afl_batch(ro_arena_view *a, const ro_read_queues *q, const afl_log *logs, const uint8_t *bytes, const uint32_t *offsets,
               size_t n, uint64_t n_bytes, uint8_t *status, uint64_t *from, uint8_t *resp, uint32_t *resp_offsets,
               uint64_t *totals) {
    uint8_t *claimed = (uint8_t *)calloc(a->n_groups ? a->n_groups : 1, 1);
    totals[0] = totals[1] = 0;
    resp_offsets[0] = 0;
    for (size_t i = 0; i < n; i++) {
        status[i] = WO_WIRE_MALFORMED << 4;
        from[i] = 0;
        const uint32_t lo = offsets[i], hi = offsets[i + 1];
        if (hi < lo || hi > n_bytes || hi - lo < 4) continue;
        uint32_t hdr;
        memcpy(&hdr, bytes + lo, 4);
        const uint32_t g = hdr >> 4;
        wo_message m;
        size_t n7;
        if (g >= a->n_groups || !afl_decode(bytes + lo + 4, hi - lo - 4, &m, &n7, NULL, NULL, 0)) continue;
        if ((q && !q->allocated[g]) || (a->meta[g] & RO_META_WIDE_HI)) continue;
        if (m.msg_type != 3) { /* MsgAppend, eraftpb.proto:53 */
            status[i] = WO_WIRE_SKIP_TYPE << 4;
            continue;
        }
        const afl_log *l = &logs[g];
        if (!(l->flags & AFL_SELECT) || a->term_start[g] != NO_TERM_START) {
            status[i] = AFL_WIRE_ROLE << 4;
            continue;
        }
        const uint64_t term = a->term[g];
        if (term == 0 || m.term != term) {
            status[i] = WO_WIRE_TERM << 4;
            continue;
        }
        if (claimed[g]) { /* the group's decision waits for the next batch */
            status[i] = WO_WIRE_DUP << 4;
            continue;
        }
        claimed[g] = 1;
        if (n7) {
            status[i] = WO_WIRE_NEEDS_LOG << 4;
            continue;
        }
        const uint64_t last = pair_max(a, a->last_index, g), committed = pair_max(a, a->committed, g);
        /* term(i) where the pass knows it: above last_index 0, in the run run_term */
        const int known = m.index > last || (m.index >= l->run_start && m.index <= last);
        uint8_t flags = AFL_RES_OK;
        if (m.index < committed) { /* raft.rs:2394-2404 */
            respond(resp, resp_offsets, totals, hdr, m.from, l->id, term, 0, committed, committed, 0, 0);
            flags |= AFL_STALE;
        } else if (!known) {
            status[i] = WO_WIRE_NEEDS_LOG << 4;
            continue;
        } else if ((m.index > last ? 0 : l->run_term) == m.log_term) {
            const uint64_t to_commit = min64(m.commit, m.index);
            if (to_commit > max64(committed, last)) { /* raft_log.rs:291-298 fatal! */
                status[i] = AFL_WIRE_COMMIT_RANGE << 4;
                continue;
            }
            const ro_ctl_cmd c = {g, RO_CTL_COMMIT_TO, 0, 0, {to_commit, 0, 0, 0}};
            ro_ctl_result r;
            ro_arena_control(a, NULL, &c, 1, &r);
            respond(resp, resp_offsets, totals, hdr, m.from, l->id, term, 0, m.index, a->committed[g], 0, 0);
        } else {
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
    free(claimed);
}

#define MAX_ENTS 64

void afl_literal(afl_group *groups, uint64_t *terms, uint64_t log_cap, size_t n_groups, const uint8_t *bytes,
                 const uint32_t *offsets, size_t n, uint64_t n_bytes, uint8_t *outcome, uint8_t *resp, uint32_t *resp_offsets,
                 uint64_t *totals) {
    totals[0] = totals[1] = 0;
    resp_offsets[0] = 0;
    uint64_t et[MAX_ENTS], ei[MAX_ENTS];
    for (size_t i = 0; i < n; i++) {
        outcome[i] = AFL_NONE;
        const uint32_t lo = offsets[i], hi = offsets[i + 1];
        if (hi < lo || hi > n_bytes || hi - lo < 4) continue;
        uint32_t hdr;
        memcpy(&hdr, bytes + lo, 4);
        const uint32_t g = hdr >> 4;
        wo_message m;
        size_t ne;
        if (g >= n_groups || !afl_decode(bytes + lo + 4, hi - lo - 4, &m, &ne, et, ei, MAX_ENTS) || m.msg_type != 3) continue;
        afl_group *s = &groups[g];
        if (!(s->flags & AFL_G_FOLLOWER)) continue;
        uint64_t *t = terms + (size_t)g * log_cap;
        /* Raft::step's term rules; m.term 0 is a local message and goes on */
        if (m.term > s->term) {
            s->term = m.term; /* become_follower(m.term, m.from): vote and the rest are the host's */
        } else if (m.term != 0 && m.term < s->term) {
            if (s->flags & AFL_G_LOWER_REPLY) { /* raft.rs:1349-1376: new_message(m.from, MsgAppendResponse) */
                respond(resp, resp_offsets, totals, hdr, m.from, s->id, s->term, 0, 0, 0, 0, 0);
                outcome[i] = AFL_ANSWERED;
            } else {
                outcome[i] = AFL_DROPPED;
            }
            continue;
        }
        /* handle_append_entries (raft.rs:2389-2448) */
        if (m.index < s->committed) {
            respond(resp, resp_offsets, totals, hdr, m.from, s->id, s->term, 0, s->committed, s->committed, 0, 0);
            outcome[i] = AFL_ANSWERED;
            continue;
        }
        const uint64_t last = s->last_index;
#define TERM(x) ((x) > last ? 0 : t[x]) /* RaftLog::term: 0 above last_index; the dummy entry is index 0 */
        if (TERM(m.index) == m.log_term) { /* maybe_append */
            if (ne > MAX_ENTS) {
                outcome[i] = AFL_FATAL;
                continue;
            }
            uint64_t conflict = 0;
            size_t first = 0;
            for (size_t k = 0; k < ne; k++) { /* find_conflict (raft_log.rs:181-203) */
                if (TERM(ei[k]) != et[k]) {
                    conflict = ei[k];
                    first = k;
                    break;
                }
            }
            const uint64_t last_new = m.index + ne;
            const uint64_t to_commit = min64(m.commit, last_new);
            uint64_t new_last = last;
            if (conflict) {
                if (conflict <= s->committed || conflict - 1 + (ne - first) >= log_cap) { /* :251-256 fatal! */
                    outcome[i] = AFL_FATAL;
                    continue;
                }
                new_last = conflict - 1 + (ne - first); /* truncate_and_append(ents[first..]) */
            }
            if (to_commit > s->committed && to_commit > new_last) { /* commit_to, raft_log.rs:291-298 fatal! */
                outcome[i] = AFL_FATAL;
                continue;
            }
            if (conflict) {
                for (size_t k = first; k < ne; k++) t[conflict + (k - first)] = et[k];
                s->last_index = new_last;
            }
            if (to_commit > s->committed) s->committed = to_commit;
            respond(resp, resp_offsets, totals, hdr, m.from, s->id, s->term, 0, last_new, s->committed, 0, 0);
        } else { /* find_conflict_by_term(min(m.index, last_index), m.log_term) */
            uint64_t h = min64(m.index, last);
            while (h > 0 && TERM(h) > m.log_term) h--; /* (term(0) is the dummy's, 0 in every log here) */
            respond(resp, resp_offsets, totals, hdr, m.from, s->id, s->term, TERM(h), m.index, s->committed, 1, h);
        }
#undef TERM
        outcome[i] = AFL_ANSWERED;
    }
}

double afl_bench(ro_arena_view *a, const ro_read_queues *q, const afl_log *logs, const uint8_t *bytes, const uint32_t *offsets,
                 size_t n, uint64_t n_bytes, uint8_t *status, uint64_t *from, uint8_t *resp, uint32_t *resp_offsets,
                 uint64_t *totals) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    afl_batch(a, q, logs, bytes, offsets, n, n_bytes, status, from, resp, resp_offsets, totals);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}
