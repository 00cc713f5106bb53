/* follower_runs_oracle.c -- see follower_runs_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#define _POSIX_C_SOURCE 199309L
#include "follower_runs_oracle.h"

#include <stdlib.h>
#include <string.h>
#include <time.h>

#define NO_TERM_START UINT64_MAX

static uint64_t max64(uint64_t x, uint64_t y) { return x > y ? x : y; }
static uint64_t min64(uint64_t x, uint64_t y) { return x < y ? x : y; }

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

/* The stated segments of a log from the top: [start[k], (k ? start[k - 1] - 1 : last)] at term[k]. */
typedef struct {
    uint64_t start[3], term[3];
    int n;
} segs;

static segs stated(const afl_log *l, const fro_row *row, uint64_t last) {
    segs s = {{0}, {0}, 0};
    if (l->run_start > last) return s; /* no run: only the indexes above last_index are known */
    s.start[0] = l->run_start;
    s.term[0] = l->run_term;
    s.n = 1;
    if (!row || row->anchor_term == 0 || row->anchor_term != l->run_term || row->anchor_start != l->run_start) return s;
    for (int k = 0; k < 2 && row->run_start[k]; k++) {
        s.start[s.n] = row->run_start[k];
        s.term[s.n++] = row->run_term[k];
    }
    return s;
}

/* term(x) for x <= last: 1 when a segment states it */
static int term_of(const segs *s, uint64_t x, uint64_t *t) {
    for (int k = 0; k < s->n; k++)
        if (x >= s->start[k]) {
            *t = s->term[k];
            return 1;
        }
    return 0;
}

/* A top-down list of segments that merges equal neighbours. */
typedef struct {
    uint64_t start[8], term[8];
    int n;
} seglist;

static void push(seglist *v, uint64_t start, uint64_t term) {
    if (v->n && v->term[v->n - 1] == term) {
        v->start[v->n - 1] = start;
    } else {
        v->start[v->n] = start;
        v->term[v->n++] = term;
    }
}

void fro_batch(ro_arena_view *a, const ro_read_queues *q, afl_log *logs, fro_row *rows, int entries, const uint8_t *bytes,
               const uint32_t *offsets, size_t n, uint64_t n_bytes, uint8_t *status, uint64_t *from, aeo_appended *appended,
               uint8_t *resp, uint32_t *resp_offsets, uint64_t *totals) {
    uint8_t *claimed = (uint8_t *)calloc(a->n_groups ? a->n_groups : 1, 1);
    size_t cap = 64;
    aeo_entry *ents = (aeo_entry *)malloc(cap * sizeof(aeo_entry));
    totals[0] = totals[1] = 0;
    resp_offsets[0] = 0;
    for (size_t i = 0; i < n; i++) {
        status[i] = WO_WIRE_MALFORMED << 4;
        from[i] = 0;
        if (entries) memset(&appended[i], 0, sizeof appended[i]);
        const uint32_t lo = offsets[i], hi = offsets[i + 1];
        if (hi < lo || hi > n_bytes || hi - lo < 4) continue;
        uint32_t hdr;
        memcpy(&hdr, bytes + lo, 4);
        const uint32_t g = hdr >> 4;
        wo_message m;
        size_t n7 = 0;
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
        if (entries) {
            if (n7 > cap) {
                cap = n7;
                ents = (aeo_entry *)realloc(ents, cap * sizeof(aeo_entry));
            }
            if (!aeo_decode(bytes + lo + 4, hi - lo - 4, &m, ents, cap, &n7)) continue; /* MALFORMED, no claim */
        }
        if (claimed[g]) {
            status[i] = WO_WIRE_DUP << 4;
            continue;
        }
        claimed[g] = 1;
        if (!entries && n7) {
            status[i] = WO_WIRE_NEEDS_LOG << 4;
            continue;
        }
        const uint64_t last = pair_max(a, a->last_index, g), committed = pair_max(a, a->committed, g);
        fro_row *row = rows ? &rows[g] : NULL;
        const segs s = stated(l, row, last);
        uint64_t tm = 0;
        uint8_t flags = AFL_RES_OK;
        if (m.index < committed) { /* raft.rs:2394-2404, whatever the entries */
            respond(resp, resp_offsets, totals, hdr, m.from, l->id, term, 0, committed, committed, 0, 0);
            flags |= AFL_STALE;
        } else if (m.index <= last && !term_of(&s, m.index, &tm)) {
            status[i] = WO_WIRE_NEEDS_LOG << 4;
            continue;
        } else if (tm == m.log_term) { /* maybe_append */
            int needs_log = n7 && m.index > last;
            for (size_t k = 0; k < n7; k++)
                if (!ents[k].ld || ents[k].index != m.index + 1 + k || ents[k].term == 0) needs_log = 1;
            size_t first = n7; /* find_conflict through the lookup */
            for (size_t k = 0; k < n7 && first == n7 && !needs_log; k++) {
                uint64_t t = 0;
                if (ents[k].index > last || (term_of(&s, ents[k].index, &t), t != ents[k].term)) first = k;
            }
            for (size_t k = first + 1; k < n7 && !needs_log; k++)
                if (ents[k].off != ents[k - 1].end) needs_log = 1;
            if (needs_log) {
                status[i] = WO_WIRE_NEEDS_LOG << 4;
                continue;
            }
            const uint64_t conflict = first < n7 ? ents[first].index : 0;
            const uint64_t last_new = m.index + n7, new_last = conflict ? last_new : last;
            const uint64_t to_commit = min64(m.commit, last_new);
            if ((conflict && conflict <= committed) || to_commit > max64(committed, new_last)) {
                status[i] = AFL_WIRE_COMMIT_RANGE << 4;
                continue;
            }
            if (conflict) {
                const ro_ctl_cmd b = {g, RO_CTL_SET_LOG_BOUNDS, 0, 0, {NO_TERM_START, new_last, 0, 0}};
                ro_ctl_result r;
                ro_arena_control(a, NULL, &b, 1, &r);
                /* the appended blocks from the top: the trailing one [k, ..] and the one before it */
                const uint64_t t = ents[n7 - 1].term;
                size_t k = n7 - 1;
                while (k > first && ents[k - 1].term == t) k--;
                if (!(k == first && t == l->run_term && conflict - 1 >= l->run_start)) { /* the run is not kept */
                    seglist v = {{0}, {0}, 0};
                    push(&v, ents[k].index, t);
                    size_t kp = k;
                    if (k > first) {
                        const uint64_t tp = ents[k - 1].term;
                        kp = k - 1;
                        while (kp > first && ents[kp - 1].term == tp) kp--;
                        push(&v, ents[kp].index, tp);
                    }
                    if (kp == first) /* the blocks are all the appended entries: the old log up to conflict - 1 */
                        for (int j = 0; j < s.n; j++)
                            if (conflict - 1 >= s.start[j]) push(&v, s.start[j], s.term[j]);
                    l->run_start = v.start[0];
                    l->run_term = v.term[0];
                    if (row) {
                        fro_row nr = {g, 0, v.start[0], v.term[0], {0, 0}, {0, 0}};
                        for (int j = 1; j < v.n && j < 3; j++) {
                            if (!v.start[j] || !v.term[j] || v.term[j] >= v.term[j - 1]) break;
                            nr.run_start[j - 1] = v.start[j];
                            nr.run_term[j - 1] = v.term[j];
                        }
                        *row = nr;
                    }
                }
                appended[i] = (aeo_appended){conflict, last_new, l->run_start, l->run_term, lo + 4 + ents[first].off,
                                             ents[n7 - 1].end - ents[first].off};
                flags |= AEO_APPENDED;
            }
            const ro_ctl_cmd c = {g, RO_CTL_COMMIT_TO, 0, 0, {to_commit, 0, 0, 0}};
            ro_ctl_result r;
            ro_arena_control(a, NULL, &c, 1, &r);
            respond(resp, resp_offsets, totals, hdr, m.from, l->id, term, 0, last_new, a->committed[g], 0, 0);
        } else { /* find_conflict_by_term(min(m.index, last_index), m.log_term) down the stated segments */
            uint64_t h = min64(m.index, last), lt = 0;
            int found = 0;
            for (int j = 0; j < s.n && !found; j++) {
                if (h < s.start[j]) continue;
                if (s.term[j] <= m.log_term) {
                    found = 1;
                    lt = s.term[j];
                } else if (s.start[j] == 0) {
                    break;
                } else {
                    h = s.start[j] - 1;
                }
            }
            if (!found) {
                status[i] = WO_WIRE_NEEDS_LOG << 4;
                continue;
            }
            respond(resp, resp_offsets, totals, hdr, m.from, l->id, term, lt, m.index, committed, 1, h);
            flags |= AFL_REJECT;
        }
        status[i] = (uint8_t)(WO_WIRE_OK << 4 | flags);
        from[i] = m.from;
    }
    free(ents);
    free(claimed);
}

double fro_bench(ro_arena_view *a, const ro_read_queues *q, afl_log *logs, fro_row *rows, int entries, const uint8_t *bytes,
                 const uint32_t *offsets, size_t n, uint64_t n_bytes, uint8_t *status, uint64_t *from, aeo_appended *appended,
                 uint8_t *resp, uint32_t *resp_offsets, uint64_t *totals) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    fro_batch(a, q, logs, rows, entries, bytes, offsets, n, n_bytes, status, from, appended, resp, resp_offsets, totals);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}
