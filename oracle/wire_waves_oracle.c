/* wire_waves_oracle.c -- see wire_waves_oracle.h.  TEST INFRASTRUCTURE ONLY. */
#define _POSIX_C_SOURCE 199309L
#include "wire_waves_oracle.h"

#include <stdlib.h>
#include <string.h>
#include <time.h>

#define RESP_MAX 85 /* == RAFTGPU_FOLLOWER_APPEND_BOUND per frame */

/* The frames pick[0 .. m) of the batch as a batch of their own: *sub_bytes / *sub_off (m + 1), malloc'd; returns its
 * length.  Every picked frame is a well-formed one (it was DUP), so its bytes lie inside the batch. */
static uint64_t repack(const uint8_t *bytes, const uint32_t *offsets, const uint32_t *pick, size_t m, uint8_t **sub_bytes,
                       uint32_t **sub_off) {
    uint64_t len = 0;
    for (size_t k = 0; k < m; k++) len += offsets[pick[k] + 1] - offsets[pick[k]];
    *sub_bytes = malloc(len ? len : 1);
    *sub_off = malloc(sizeof(uint32_t) * (m + 1));
    uint32_t at = 0;
    for (size_t k = 0; k < m; k++) {
        const uint32_t a = offsets[pick[k]], b = offsets[pick[k] + 1];
        (*sub_off)[k] = at;
        memcpy(*sub_bytes + at, bytes + a, b - a);
        at += b - a;
    }
    (*sub_off)[m] = at;
    return len;
}

static uint32_t *all_frames(size_t n) {
    uint32_t *f = malloc(sizeof(uint32_t) * (n ? n : 1));
    for (size_t i = 0; i < n; i++) f[i] = (uint32_t)i;
    return f;
}

void wwo_leader(ro_arena_view *c, const lro_row *rows, const uint8_t *bytes, const uint32_t *offsets, size_t n,
                uint64_t n_bytes, uint32_t waves, uint8_t *status) {
    uint32_t *frames = all_frames(n);
    size_t m = n;
    uint8_t *st = malloc(n ? n : 1);
    wo_record *recs = malloc(sizeof(wo_record) * (n ? n : 1));
    uint64_t *hint = malloc(sizeof(uint64_t) * (n ? n : 1)), *snap = malloc(sizeof(uint64_t) * (n ? n : 1));
    for (uint32_t j = 0; j < waves && m; j++) {
        uint8_t *sb = NULL;
        uint32_t *so = NULL;
        const uint64_t len = j ? repack(bytes, offsets, frames, m, &sb, &so) : n_bytes;
        lro_decode_batch(c, rows, j ? sb : bytes, j ? so : offsets, m, len, st, recs, hint, snap);
        size_t next = 0;
        for (size_t k = 0; k < m; k++) {
            const uint32_t i = frames[k];
            status[i] = (uint8_t)(st[k] << 4);
            if (st[k] == WO_WIRE_DUP) frames[next++] = i;  /* (k >= next: in place) */
            if (st[k] != WO_WIRE_OK) continue;
            ro_append_resp r[2];
            memcpy(&r[0], &recs[k], sizeof(r[0]));
            r[1] = (ro_append_resp){recs[k].group, recs[k].peer_slot, RO_REC_EXT, 0, hint[k], snap[k]};
            uint8_t res[2];
            ro_arena_apply(c, r, (recs[k].flags & RO_REC_REJECT) ? 2 : 1, 0, res);
            status[i] |= res[0] & 0xf;
        }
        m = next;
        free(sb);
        free(so);
    }
    free(frames);
    free(st);
    free(recs);
    free(hint);
    free(snap);
}

double wwo_leader_bench(ro_arena_view *c, const lro_row *rows, const uint8_t *bytes, const uint32_t *offsets, size_t n,
                        uint64_t n_bytes, uint32_t waves, uint8_t *status) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    wwo_leader(c, rows, bytes, offsets, n, n_bytes, waves, status);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}

void wwo_follower(ro_arena_view *c, const ro_read_queues *q, afl_log *logs, int entries, const uint8_t *bytes,
                  const uint32_t *offsets, size_t n, uint64_t n_bytes, uint32_t waves, uint8_t *status, uint64_t *from,
                  aeo_appended *appended, uint8_t *resp, uint32_t *resp_offsets, uint64_t *totals) {
    const size_t nn = n ? n : 1;
    uint32_t *frames = all_frames(n);
    size_t m = n;
    uint8_t *st = malloc(nn), *sresp = malloc(RESP_MAX * nn), *stopped = calloc(c->cap ? c->cap : 1, 1);
    uint64_t *sfrom = malloc(sizeof(uint64_t) * nn), stot[2];
    uint32_t *soff = malloc(sizeof(uint32_t) * (nn + 1));
    aeo_appended *sapp = calloc(nn, sizeof(aeo_appended));
    /* every frame's response, kept at its position until all runs are done */
    uint8_t *own = malloc(RESP_MAX * nn);
    uint32_t *own_len = calloc(nn, sizeof(uint32_t));
    memset(status, 0, n);
    memset(from, 0, sizeof(uint64_t) * n);
    if (appended) memset(appended, 0, sizeof(aeo_appended) * n);
    for (uint32_t j = 0; j < waves && m; j++) {
        uint8_t *sb = NULL;
        uint32_t *so = NULL;
        const uint64_t len = j ? repack(bytes, offsets, frames, m, &sb, &so) : n_bytes;
        const uint8_t *b = j ? sb : bytes;
        const uint32_t *o = j ? so : offsets;
        if (entries)
            aeo_batch(c, q, logs, b, o, m, len, st, sfrom, sapp, sresp, soff, stot);
        else
            afl_batch(c, q, logs, b, o, m, len, st, sfrom, sresp, soff, stot);
        size_t answered = 0;
        for (size_t k = 0; k < m; k++) {
            const uint32_t i = frames[k], s = st[k] >> 4;
            status[i] = st[k];
            from[i] = sfrom[k];
            if (appended) appended[i] = entries ? sapp[k] : (aeo_appended){0};
            if (appended && appended[i].span_len)  /* the span's offset in the batch, not in the re-packed one */
                appended[i].span_off += offsets[i] - o[k];
            if (s == WO_WIRE_OK && (st[k] & AFL_RES_OK)) {
                own_len[i] = soff[answered + 1] - soff[answered];
                memcpy(own + (size_t)RESP_MAX * i, sresp + soff[answered], own_len[i]);
                answered++;
            }
            if (s == WO_WIRE_NEEDS_LOG || s == AFL_WIRE_COMMIT_RANGE) {  /* a claimant the host handles first */
                uint32_t hdr;
                memcpy(&hdr, b + o[k], 4);
                stopped[hdr >> 4] = 1;
            }
        }
        size_t next = 0;
        for (size_t k = 0; k < m; k++) {
            uint32_t hdr;
            memcpy(&hdr, b + o[k], 4);
            if ((st[k] >> 4) == WO_WIRE_DUP && !stopped[hdr >> 4]) frames[next++] = frames[k];
        }
        m = next;
        free(sb);
        free(so);
    }
    uint64_t nr = 0, at = 0;
    resp_offsets[0] = 0;
    for (size_t i = 0; i < n; i++) {
        if (!own_len[i]) continue;
        memcpy(resp + at, own + (size_t)RESP_MAX * i, own_len[i]);
        at += own_len[i];
        resp_offsets[++nr] = (uint32_t)at;
    }
    totals[0] = nr;
    totals[1] = at;
    free(frames);
    free(st);
    free(sresp);
    free(stopped);
    free(sfrom);
    free(soff);
    free(sapp);
    free(own);
    free(own_len);
}
