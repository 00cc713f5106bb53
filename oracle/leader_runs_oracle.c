/* leader_runs_oracle.c -- see leader_runs_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#define _POSIX_C_SOURCE 199309L
#include "leader_runs_oracle.h"

#include <stdlib.h>
#include <string.h>
#include <time.h>

#define LRO_NO_TERM_START UINT64_MAX
#define LRO_META_WIDE_LO 0x20000000u /* RAFTGPU_META_WIDE_LO / _HI */
#define LRO_META_WIDE_HI 0x40000000u

int32_t lro_row_status(const lro_row *r, int allocated, int wide_hi) {
    if (!allocated || wide_hi) return -5;
    if (r->term == 0 || r->term_start == 0 || r->term_start == LRO_NO_TERM_START) return -1;
    /* the stated runs, top down: each start below the one above it, each term non-zero and below the one above it */
    uint64_t above_start = r->term_start, above_term = r->term;
    int ended = 0;
    for (int k = 0; k < 2; k++) {
        if (r->run_start[k] == 0) {
            ended = 1;
            continue;
        }
        if (ended) return -1; /* run 2 without run 1 */
        if (r->run_start[k] >= above_start || r->run_term[k] == 0 || r->run_term[k] >= above_term) return -1;
        above_start = r->run_start[k];
        above_term = r->run_term[k];
    }
    return 0;
}

/* RaftLog::term (raft_log.rs:122-140) on the literal log */
static uint64_t lit_term(const uint64_t *terms, uint64_t first_index, uint64_t last_index, uint64_t i) {
    if (i + 1 < first_index || i > last_index) return 0;
    return terms[i];
}

uint64_t lro_find_conflict_by_term(const uint64_t *terms, uint64_t first_index, uint64_t last_index, uint64_t h, uint64_t lt) {
    uint64_t conflict_index = h;
    if (h > last_index) return h; /* raft_log.rs:213-221 */
    for (;;) {                     /* :223-234 */
        const uint64_t t = lit_term(terms, first_index, last_index, conflict_index);
        if (t > lt)
            conflict_index -= 1;
        else
            return conflict_index;
    }
}

/* term(i) as the arena and the row state it: 1 with *t and *seg_start (the first index of i's segment of equal
 * terms) when stated, 0 when not. */
static int row_term(uint64_t term, uint64_t ts, uint64_t last, const lro_row *row, uint64_t i, uint64_t *t, uint64_t *seg_start) {
    if (i >= ts) {
        *t = term;
        *seg_start = ts;
        return 1;
    }
    for (int k = 0; k < 2; k++) {
        if (row->run_start[k] != 0 && i >= row->run_start[k]) {
            *t = row->run_term[k];
            *seg_start = row->run_start[k];
            return 1;
        }
        if (row->run_start[k] == 0) break;
    }
    (void)last;
    return 0;
}

int lro_probe_by_runs(uint64_t term, uint64_t term_start, uint64_t last_index, const lro_row *row, uint64_t h, uint64_t lt,
                      uint64_t *out) {
    if (!row || term_start == LRO_NO_TERM_START || term == 0) return 0;
    if (row->term != term || row->term_start != term_start) return 0; /* the anchor */
    if (h > last_index) {
        *out = h;
        return 1;
    }
    /* lowest: the term of the lowest stated segment (the stated runs are contiguous below term_start) */
    uint64_t lowest = term;
    for (int k = 0; k < 2 && row->run_start[k] != 0; k++) lowest = row->run_term[k];
    uint64_t i = h;
    for (;;) {
        if (i == 0) { /* term(0) = 0 <= lt */
            *out = 0;
            return 1;
        }
        uint64_t t, start;
        if (!row_term(term, term_start, last_index, row, i, &t, &start)) break;
        if (t <= lt) {
            *out = i;
            return 1;
        }
        i = start - 1; /* every index of the segment has term t > lt */
    }
    /* i is below every stated run: term(i) <= lowest (terms are monotone, a compacted index reads 0) */
    if (lowest <= lt) {
        *out = i;
        return 1;
    }
    return 0;
}

/* Both forms: frames decoded and classified as wo_decode_batch does; a rejection with log_term > 0 goes to decide(),
 * which returns 1 with the hint, or 0 (WO_WIRE_NEEDS_LOG). */
typedef int (*lro_decide_fn)(const void *ctx, uint32_t group, uint64_t h, uint64_t lt, uint64_t *out);

static void lro_batch(const void *ctx, lro_decide_fn decide, const uint64_t *group_term, uint32_t n_groups,
                      const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes, uint8_t *status,
                      wo_record *recs, uint64_t *hint, uint64_t *request_snapshot) {
    uint16_t *touched = (uint16_t *)calloc(n_groups ? n_groups : 1, sizeof(uint16_t)); /* a bit per peer slot */
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
        if (m.msg_type != 4) {
            status[i] = WO_WIRE_SKIP_TYPE;
            continue;
        }
        if (group_term && group_term[group] != 0 && m.term != group_term[group]) {
            status[i] = WO_WIRE_TERM;
            continue;
        }
        uint64_t h = m.reject_hint; /* raft.rs:1560 */
        if (m.reject && m.log_term > 0 && !decide(ctx, group, m.reject_hint, m.log_term, &h)) {
            status[i] = WO_WIRE_NEEDS_LOG;
            continue;
        }
        if (slot < 8) { /* a frame naming another slot finds no Progress (raft.rs:1663-1673) and claims nothing */
            if (touched[group] & (1u << slot)) {
                status[i] = WO_WIRE_DUP;
                continue;
            }
            touched[group] |= (uint16_t)(1u << slot);
        }
        status[i] = WO_WIRE_OK;
        recs[i].group = group;
        recs[i].peer_slot = (uint8_t)slot;
        recs[i].flags = m.reject ? 0x01 : 0x00;
        recs[i].index = m.index;
        recs[i].commit = m.commit;
        hint[i] = h;
        request_snapshot[i] = m.request_snapshot; /* raft.rs:1709 */
    }
    free(touched);
}

typedef struct {
    const ro_arena_view *c;
    const lro_row *rows;
} runs_ctx;

static int decide_runs(const void *p, uint32_t group, uint64_t h, uint64_t lt, uint64_t *out) {
    const runs_ctx *x = (const runs_ctx *)p;
    const ro_arena_view *c = x->c;
    if (!x->rows) return 0;
    const uint32_t meta = c->meta[group];
    const uint32_t lo = (meta & LRO_META_WIDE_HI) ? group - 1 : group; /* a pair: the low half's row and fields */
    uint64_t last = c->last_index[lo];
    if ((meta & (LRO_META_WIDE_LO | LRO_META_WIDE_HI)) && c->last_index[lo + 1] > last) last = c->last_index[lo + 1];
    return lro_probe_by_runs(c->term[lo], c->term_start[lo], last, &x->rows[lo], h, lt, out);
}

void lro_decode_batch(const ro_arena_view *c, const lro_row *rows, const uint8_t *bytes, const uint32_t *offsets, size_t n,
                      uint64_t n_bytes, uint8_t *status, wo_record *recs, uint64_t *hint, uint64_t *request_snapshot) {
    const runs_ctx x = {c, rows};
    lro_batch(&x, decide_runs, c->term, c->n_groups, bytes, offsets, n, n_bytes, status, recs, hint, request_snapshot);
}

typedef struct {
    const uint64_t *log_off, *log_terms, *first_index;
} literal_ctx;

static int decide_literal(const void *p, uint32_t group, uint64_t h, uint64_t lt, uint64_t *out) {
    const literal_ctx *x = (const literal_ctx *)p;
    const uint64_t *terms = x->log_terms + x->log_off[group];
    const uint64_t last = x->log_off[group + 1] - x->log_off[group] - 1;
    *out = lro_find_conflict_by_term(terms, x->first_index[group], last, h, lt);
    return 1;
}

void lro_literal_batch(const uint64_t *log_off, const uint64_t *log_terms, const uint64_t *first_index,
                       const uint64_t *group_term, uint32_t n_groups, const uint8_t *bytes, const uint32_t *offsets,
                       size_t n, uint64_t n_bytes, uint8_t *status, wo_record *recs, uint64_t *hint,
                       uint64_t *request_snapshot) {
    const literal_ctx x = {log_off, log_terms, first_index};
    lro_batch(&x, decide_literal, group_term, n_groups, bytes, offsets, n, n_bytes, status, recs, hint, request_snapshot);
}

double lro_bench(const ro_arena_view *c, const lro_row *rows, const uint8_t *bytes, const uint32_t *offsets, size_t n,
                 uint64_t n_bytes, uint8_t *status, wo_record *recs, uint64_t *hint, uint64_t *request_snapshot, int iters) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    for (int k = 0; k < iters; k++) lro_decode_batch(c, rows, bytes, offsets, n, n_bytes, status, recs, hint, request_snapshot);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return ((double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec)) / (iters > 0 ? iters : 1);
}
