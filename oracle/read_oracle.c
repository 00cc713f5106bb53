/*
 * read_oracle.c -- CPU ORACLE of ReadIndex with ReadOnlyOption::Safe. TEST INFRASTRUCTURE ONLY (see read_oracle.h).
 */
#include "read_oracle.h"

#include <stdlib.h>
#include <string.h>

/* ---- the group's configuration, through the arena view --------------------- */

static uint32_t present_of(uint32_t m) { return RO_META_IN(m) | RO_META_OUT(m) | RO_META_LEARN(m); }
static uint32_t hi_meta(const ro_arena_view *a, uint32_t g) { return (a->meta[g] & RO_META_WIDE_LO) ? a->meta[g + 1] : 0; }

/* JointConfig voters over 16 peer slots (peer p has id p + 1) */
static void voter_masks(const ro_arena_view *a, uint32_t g, uint32_t *in, uint32_t *out) {
    uint32_t lo = a->meta[g], hi = hi_meta(a, g);
    *in = RO_META_IN(lo) | (RO_META_IN(hi) << 8);
    *out = RO_META_OUT(lo) | (RO_META_OUT(hi) << 8);
}

/* ProgressTracker::has_quorum (tracker.rs:367-372): conf.voters.vote_result(|id| set.get(id).map(|_| true)) == Won */
static int has_quorum(const ro_arena_view *a, uint32_t g, uint32_t acks) {
    uint32_t in, out;
    voter_masks(a, g, &in, &out);
    uint64_t in_ids[16], out_ids[16], v_ids[16];
    uint8_t v_yes[16];
    size_t n_in = 0, n_out = 0, n_v = 0;
    for (uint32_t p = 0; p < 16; p++) {
        if (in & (1u << p)) in_ids[n_in++] = p + 1;
        if (out & (1u << p)) out_ids[n_out++] = p + 1;
        if (acks & (1u << p)) v_ids[n_v] = p + 1, v_yes[n_v++] = 1;
    }
    ro_vote_map vm = {v_ids, v_yes, n_v};
    return ro_joint_vote_result(in_ids, n_in, out_ids, n_out, &vm) == RO_VOTE_WON;
}

/* JointConfig::is_singleton (joint.rs:77-79): outgoing empty, exactly one incoming voter */
static int is_singleton(const ro_arena_view *a, uint32_t g) {
    uint32_t in, out;
    voter_masks(a, g, &in, &out);
    return out == 0 && __builtin_popcount(in) == 1;
}

/* the slot bit of Raft::id (read_only.rs:97 acks.insert(self_id)); 0 when the leader holds no slot */
static uint32_t self_bit(const ro_arena_view *a, uint32_t g) {
    uint32_t lo = a->meta[g], hi = hi_meta(a, g);
    if (lo & RO_META_HAS_SELF) return 1u << RO_META_SELF(lo);
    if (hi & RO_META_HAS_SELF) return 1u << (8 + RO_META_SELF(hi));
    return 0;
}

/* Raft::commit_to_current_term (raft.rs:581-585) in range form: term(committed) == term <=> term_start <= committed <=
 * last_index.  A wide group's halves carry the same log columns (what one half alone has seen counts). */
static int commit_to_current_term(const ro_arena_view *a, uint32_t g, uint64_t *committed) {
    uint64_t c = a->committed[g], li = a->last_index[g];
    if (a->meta[g] & RO_META_WIDE_LO) {
        if (a->committed[g + 1] > c) c = a->committed[g + 1];
        if (a->last_index[g + 1] > li) li = a->last_index[g + 1];
    }
    *committed = c;
    return a->term_start[g] <= c && c <= li;
}

/* ---- ReadOnly (read_only.rs:86-139) ---------------------------------------- */

static size_t at(const ro_read_queues *q, uint32_t g, uint32_t k) { return (size_t)g * q->max_pending + k; }

/* pending_read_index.get(ctx): the queue position of ctx, -1 when it is not pending */
static int find(const ro_read_queues *q, uint32_t g, uint64_t ctx) {
    for (uint32_t k = 0; k < q->count[g]; k++)
        if (q->ctx[at(q, g, k)] == ctx) return (int)k;
    return -1;
}

/* read_only.rs:86-99 add_request(index, ctx, self): a pending ctx changes nothing; else a new entry at the back with
 * acks = {self}.  Returns the result byte. */
static uint8_t add_request(ro_read_queues *q, uint32_t g, uint64_t ctx, uint64_t index, uint32_t self) {
    if (find(q, g, ctx) >= 0) return RO_READ_DUP; /* :89-91 */
    if (q->count[g] == q->max_pending) return RO_READ_FULL; /* the bounded queue (the reference's is unbounded) */
    size_t c = at(q, g, q->count[g]++);
    q->ctx[c] = ctx, q->index[c] = index, q->acks[c] = (uint16_t)self; /* :93-98 */
    return RO_READ_QUEUED;
}

/* read_only.rs:115-129 advance(ctx): pop the queue up to and including the entry at position `pos` */
static void advance(ro_read_queues *q, uint32_t g, uint32_t pos, ro_read_state *out, uint64_t *n_out) {
    for (uint32_t k = 0; k <= pos; k++) {
        size_t c = at(q, g, k);
        ro_read_state s = {g, 0, q->ctx[c], q->index[c]};
        out[(*n_out)++] = s;
    }
    uint32_t left = q->count[g] - (pos + 1);
    memmove(&q->ctx[at(q, g, 0)], &q->ctx[at(q, g, pos + 1)], left * sizeof(uint64_t));
    memmove(&q->index[at(q, g, 0)], &q->index[at(q, g, pos + 1)], left * sizeof(uint64_t));
    memmove(&q->acks[at(q, g, 0)], &q->acks[at(q, g, pos + 1)], left * sizeof(uint16_t));
    q->count[g] = left;
}

static int is_group(const ro_arena_view *a, const ro_read_queues *q, uint32_t g) {
    return g < q->cap && q->allocated[g] && !(a->meta[g] & RO_META_WIDE_HI);
}

void ro_read_request(const ro_arena_view *a, ro_read_queues *q, const ro_read_req *reqs, size_t n, uint8_t *results,
                     ro_read_state *out, uint64_t *n_out) {
    *n_out = 0;
    for (size_t i = 0; i < n; i++) {
        uint32_t g = reqs[i].group;
        uint64_t ctx = reqs[i].ctx, committed;
        uint8_t r;
        if (!is_group(a, q, g)) {
            r = RO_READ_NO_GROUP;
        } else if (ctx == 0) {
            r = RO_READ_NO_CTX;
        } else if (!commit_to_current_term(a, g, &committed)) { /* raft.rs:2057-2062 */
            r = RO_READ_DROPPED;
        } else if (is_singleton(a, g)) { /* raft.rs:2064-2070: ready with read_index = committed */
            ro_read_state s = {g, 0, ctx, committed};
            out[(*n_out)++] = s;
            r = RO_READ_READY;
        } else { /* raft.rs:2076-2082 */
            r = add_request(q, g, ctx, committed, self_bit(a, g));
        }
        if (results) results[i] = r;
    }
}

/* raft.rs:1777-1789 + 1805-1812: the group slot holding the queue and the responder's bit; 0 = the record is
 * ignored (not a READ_CTX heartbeat, an empty context, a responder without Progress) */
static int ack_target(const ro_arena_view *a, const ro_read_queues *q, const ro_append_resp *r, uint32_t *qg, uint32_t *bit) {
    if ((r->flags & (RO_REC_HEARTBEAT | RO_REC_READ_CTX)) != (RO_REC_HEARTBEAT | RO_REC_READ_CTX)) return 0;
    if (r->index == 0 || r->group >= q->cap || r->peer_slot >= RO_SLOTS) return 0;
    uint32_t m = a->meta[r->group];
    if (!(present_of(m) & (1u << r->peer_slot))) return 0;
    int hi = (m & RO_META_WIDE_HI) != 0;
    *qg = hi ? r->group - 1 : r->group;
    *bit = 1u << (hi ? 8 + r->peer_slot : r->peer_slot);
    return 1;
}

void ro_read_ack_seq(const ro_arena_view *a, ro_read_queues *q, const ro_append_resp *recs, size_t n, ro_read_state *out,
                     uint64_t *n_out) {
    *n_out = 0;
    for (size_t i = 0; i < n; i++) {
        uint32_t g, bit;
        if (!ack_target(a, q, &recs[i], &g, &bit)) continue;
        int k = find(q, g, recs[i].index); /* read_only.rs:104-110 recv_ack */
        if (k < 0) continue;
        q->acks[at(q, g, (uint32_t)k)] |= (uint16_t)bit;
        if (!has_quorum(a, g, q->acks[at(q, g, (uint32_t)k)])) continue; /* raft.rs:1812-1815 */
        advance(q, g, (uint32_t)k, out, n_out);                           /* raft.rs:1817 */
    }
}

void ro_read_ack_batch(const ro_arena_view *a, ro_read_queues *q, const ro_append_resp *recs, size_t n, ro_read_state *out,
                       uint64_t *n_out) {
    *n_out = 0;
    uint32_t *touched = malloc((n ? n : 1) * sizeof(uint32_t));
    uint64_t *hit = calloc(q->cap, sizeof(uint64_t)); /* per group: the queue positions an ack of the batch named */
    size_t n_t = 0;
    for (size_t i = 0; i < n; i++) { /* every recv_ack first */
        uint32_t g, bit;
        if (!ack_target(a, q, &recs[i], &g, &bit)) continue;
        int k = find(q, g, recs[i].index);
        if (k < 0) continue;
        q->acks[at(q, g, (uint32_t)k)] |= (uint16_t)bit;
        if (!hit[g]) touched[n_t++] = g;
        hit[g] |= 1ull << k;
    }
    for (size_t t = 0; t < n_t; t++) { /* then advance to the last named entry whose acks have a quorum */
        uint32_t g = touched[t];
        for (uint32_t k = q->count[g]; k > 0; k--)
            if (((hit[g] >> (k - 1)) & 1u) && has_quorum(a, g, q->acks[at(q, g, k - 1)])) {
                advance(q, g, k - 1, out, n_out);
                break;
            }
    }
    free(touched);
    free(hit);
}

void ro_read_recheck(const ro_arena_view *a, ro_read_queues *q, const uint32_t *groups, size_t n, ro_read_state *out,
                     uint64_t *n_out) {
    *n_out = 0;
    for (size_t i = 0; i < n; i++) {
        uint32_t g = groups[i];
        if (!q->count[g]) continue; /* raft.rs:2650 last_pending_request_ctx() == None */
        size_t c = at(q, g, q->count[g] - 1);
        q->acks[c] |= (uint16_t)self_bit(a, g); /* :2652-2655 recv_ack(self.id, &ctx) */
        if (has_quorum(a, g, q->acks[c])) advance(q, g, q->count[g] - 1, out, n_out); /* :2656-2662 */
    }
}

uint64_t ro_read_last_ctx(const ro_read_queues *q, uint32_t g) {
    return q->count[g] ? q->ctx[at(q, g, q->count[g] - 1)] : 0;
}

void ro_read_control(ro_arena_view *a, ro_read_queues *q, uint8_t *votes, const ro_ctl_cmd *cmds, size_t n,
                     ro_ctl_result *results) {
    for (size_t i = 0; i < n; i++) {
        uint32_t g = cmds[i].group;
        int ok_g = g < a->n_groups;
        uint32_t before_lo = ok_g ? a->meta[g] : 0, before_hi = ok_g ? hi_meta(a, g) : 0;
        ro_arena_control(a, votes, &cmds[i], 1, &results[i]);
        if (results[i].status != 0 || !ok_g || (a->meta[g] & RO_META_WIDE_HI)) continue;
        if (cmds[i].op == RO_CTL_RESET) {
            q->count[g] = 0; /* raft.rs:957 self.read_only = ReadOnly::new(..) */
        } else if (cmds[i].op == RO_CTL_SET_CONF) {
            uint32_t removed = (present_of(before_lo) & ~present_of(a->meta[g])) |
                               ((present_of(before_hi) & ~present_of(hi_meta(a, g))) << 8);
            for (uint32_t k = 0; k < q->count[g]; k++) q->acks[at(q, g, k)] &= (uint16_t)~removed;
        }
    }
}
