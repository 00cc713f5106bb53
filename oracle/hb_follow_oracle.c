/* hb_follow_oracle.c -- see hb_follow_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#define _POSIX_C_SOURCE 199309L
#include "hb_follow_oracle.h"

#include <stdlib.h>
#include <string.h>
#include <time.h>

#define NO_TERM_START UINT64_MAX

size_t hfl_encode_response(uint64_t to, uint64_t from, uint64_t term, uint64_t commit, const uint8_t *ctx, uint8_t *out) {
    /* hfo_encode_heartbeat's fields without the context: msg_type is field 1, written first as the two bytes 0x08, 8;
     * a response differs only in that value, and both are one-byte varints */
    size_t k = hfo_encode_heartbeat(to, from, term, commit, 0, out);
    out[1] = 9; /* MsgHeartbeatResponse, eraftpb.proto:59 */
    if (ctx) {  /* bytes context = 12, the last field: length-delimited, echoed byte for byte */
        out[k++] = 12u << 3 | 2u;
        out[k++] = 8;
        memcpy(out + k, ctx, 8);
        k += 8;
    }
    return k;
}

static uint64_t max64(uint64_t x, uint64_t y) { return x > y ? x : y; }

void hfl_follower_heartbeats(ro_arena_view *a, const ro_read_queues *q, const uint8_t *bytes, const uint32_t *offsets,
                             size_t n, uint64_t n_bytes, const uint32_t *select, const uint64_t *self_ids, uint8_t *status, uint64_t *from,
                             uint8_t *resp, uint32_t *resp_offsets, uint64_t *totals) {
    uint8_t *applied = (uint8_t *)calloc(a->n_groups ? a->n_groups : 1, 1);
    uint64_t frames = 0, len = 0;
    for (size_t i = 0; i < n; i++) {
        status[i] = WO_WIRE_MALFORMED << 4;
        from[i] = 0;
        const uint32_t lo = offsets[i], hi = offsets[i + 1];
        if (hi < lo || hi > n_bytes || hi - lo < 4) continue;
        uint32_t hdr;
        memcpy(&hdr, bytes + lo, 4);
        const uint32_t g = hdr >> 4;
        hwo_message h;
        if (g >= a->n_groups || (q && !q->allocated[g]) || (a->meta[g] & RO_META_WIDE_HI)) continue;
        if (!hwo_decode_message(bytes + lo + 4, hi - lo - 4, &h)) continue;
        const wo_message *m = &h.m;
        if (m->msg_type != 8) { /* MsgHeartbeat, eraftpb.proto:58 */
            status[i] = WO_WIRE_SKIP_TYPE << 4;
            continue;
        }
        /* Raft::step reaches step_follower only for a Follower at m.term == term (raft.rs:1280-1411, 2276) */
        if (!((select[g / 32] >> (g % 32)) & 1u) || a->term_start[g] != NO_TERM_START) {
            status[i] = HFL_WIRE_ROLE << 4;
            continue;
        }
        if (a->term[g] == 0 || m->term != a->term[g]) {
            status[i] = WO_WIRE_TERM << 4;
            continue;
        }
        if (h.ctx_len && h.ctx_len != 8) {
            status[i] = HWO_WIRE_CONTEXT << 4;
            continue;
        }
        const int wide = (a->meta[g] & RO_META_WIDE_LO) != 0;
        uint64_t top = max64(a->committed[g], a->last_index[g]);
        if (wide) top = max64(top, max64(a->committed[g + 1], a->last_index[g + 1]));
        if (m->commit > top) { /* raft_log.rs:291-298 fatal! */
            status[i] = HFL_WIRE_COMMIT_RANGE << 4;
            continue;
        }
        if (applied[g]) {
            status[i] = WO_WIRE_DUP << 4;
            continue;
        }
        applied[g] = 1;
        /* handle_heartbeat (raft.rs:2452-2464): commit_to, then send the response */
        const ro_ctl_cmd c = {g, RO_CTL_COMMIT_TO, 0, 0, {m->commit, 0, 0, 0}};
        ro_ctl_result r;
        ro_arena_control(a, NULL, &c, 1, &r);
        uint8_t *p = resp + len;
        memcpy(p, &hdr, 4); /* little-endian host */
        const size_t k = hfl_encode_response(m->from, self_ids[g], a->term[g], a->committed[g],
                                             h.ctx_len ? bytes + lo + 4 + h.ctx_off : NULL, p + 4);
        resp_offsets[frames++] = (uint32_t)len;
        len += 4 + k;
        status[i] = (uint8_t)(WO_WIRE_OK << 4 | 1u);
        from[i] = m->from;
    }
    resp_offsets[frames] = (uint32_t)len;
    totals[0] = frames;
    totals[1] = len;
    free(applied);
}

double hfl_bench(ro_arena_view *a, const ro_read_queues *q, const uint8_t *bytes, const uint32_t *offsets, size_t n, uint64_t n_bytes,
                 const uint32_t *select, const uint64_t *self_ids, uint8_t *status, uint64_t *from, uint8_t *resp,
                 uint32_t *resp_offsets, uint64_t *totals) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    hfl_follower_heartbeats(a, q, bytes, offsets, n, n_bytes, select, self_ids, status, from, resp, resp_offsets, totals);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}
