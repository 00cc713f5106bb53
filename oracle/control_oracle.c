/*
 * control_oracle.c -- CPU ORACLE of the control plane's list form. TEST INFRASTRUCTURE ONLY (see control_oracle.h).
 */
#include "control_oracle.h"

/* ---- cells of the arena view (the layout of raft_oracle.h) ---------------- */

static inline size_t cell(const ro_arena_view *a, uint32_t slot, uint32_t g) { return (size_t)slot * a->cap + g; }

/* The Progress of one cell.  `ring` backs p->ins when the arena models the Inflights window. */
static void load_progress_ins(const ro_arena_view *a, uint32_t slot, uint32_t g, ro_progress *p, ro_inflights *ring) {
    size_t c = cell(a, slot, g);
    p->ins = NULL;
    if (a->ins_cap && ring) {
        ring->start = a->ins_meta[c] & 0xffffu;
        ring->count = a->ins_meta[c] >> 16;
        ring->cap = a->ins_cap;
        ring->buffer = a->ins_buf + c * (size_t)a->ins_cap;
        p->ins = ring;
    }
    uint8_t f = a->pflags[c];
    p->matched = a->matched[c];
    p->next_idx = a->next_idx[c];
    p->pending_snapshot = a->pending_snapshot[c];
    p->pending_request_snapshot = a->pending_request_snapshot[c];
    p->commit_group_id = a->commit_group_id[c];
    p->committed_index = a->peer_committed[c];
    p->state = f & RO_PF_STATE_MASK;
    p->paused = (f & RO_PF_PAUSED) != 0;
    p->recent_active = (f & RO_PF_RECENT_ACTIVE) != 0;
    p->ins_full = (f & RO_PF_INS_FULL) != 0;
}

static void store_progress(ro_arena_view *a, uint32_t slot, uint32_t g, ro_progress *p) {
    size_t c = cell(a, slot, g);
    if (p->ins) { /* the flag column mirrors ins.full() */
        a->ins_meta[c] = p->ins->start | (p->ins->count << 16);
        p->ins_full = (uint8_t)ro_inflights_full(p->ins);
    }
    a->matched[c] = p->matched;
    a->next_idx[c] = p->next_idx;
    a->pending_snapshot[c] = p->pending_snapshot;
    a->pending_request_snapshot[c] = p->pending_request_snapshot;
    a->commit_group_id[c] = p->commit_group_id;
    a->peer_committed[c] = p->committed_index;
    a->pflags[c] = (uint8_t)((p->state & RO_PF_STATE_MASK) | (p->paused ? RO_PF_PAUSED : 0) |
                             (p->recent_active ? RO_PF_RECENT_ACTIVE : 0) | (p->ins_full ? RO_PF_INS_FULL : 0));
}

/* ---- the control plane --------------------------------------------------- */

static uint32_t present_of(uint32_t m) { return RO_META_IN(m) | RO_META_OUT(m) | RO_META_LEARN(m); }
static uint32_t halves_of(const ro_arena_view *a, uint32_t g) { return (a->meta[g] & RO_META_WIDE_LO) ? 2 : 1; }

/* peer 0..15 of group g -> (half, slot in the half); 0 = the group has no such slot */
static int ctl_resolve(const ro_arena_view *a, uint32_t g, uint32_t peer, uint32_t *g2, uint32_t *s2) {
    if (peer < RO_SLOTS) {
        *g2 = g, *s2 = peer;
        return 1;
    }
    if (peer < 2 * RO_SLOTS && (a->meta[g] & RO_META_WIDE_LO)) {
        *g2 = g + 1, *s2 = peer - RO_SLOTS;
        return 1;
    }
    return 0;
}

/* both halves of a wide group carry the group's log bounds, commit index and term */
static void ctl_wide_sync(ro_arena_view *a, uint32_t g) {
    uint64_t li = a->last_index[g] > a->last_index[g + 1] ? a->last_index[g] : a->last_index[g + 1];
    a->last_index[g] = a->last_index[g + 1] = li;
    uint64_t cm = a->committed[g] > a->committed[g + 1] ? a->committed[g] : a->committed[g + 1];
    a->committed[g] = a->committed[g + 1] = cm;
    a->term_start[g + 1] = a->term_start[g];
    a->term[g + 1] = a->term[g];
}

/* tracker.rs:380-397 on one half: a slot that appears gets Progress::new(next_idx, ..) with recent_active
 * (tracker.rs:385-390), one that disappears is removed (tracker.rs:392-394; an absent cell is all zeros) */
static void ctl_apply_conf(ro_arena_view *a, uint8_t *votes, uint32_t g, uint32_t meta, uint64_t next_idx) {
    uint32_t was = present_of(a->meta[g]), now = present_of(meta);
    for (uint32_t s = 0; s < RO_SLOTS; s++) {
        if (!((was ^ now) & (1u << s))) continue;
        int add = (now >> s) & 1u;
        ro_progress p;
        ro_inflights ring;
        load_progress_ins(a, s, g, &p, &ring);
        ro_inflights *ins = p.ins;
        ro_progress_new(&p, add ? next_idx : 0);
        p.recent_active = (uint8_t)add;
        p.ins = ins;
        if (ins) ro_inflights_reset(ins); /* Inflights::new(max_inflight), progress.rs:70 */
        store_progress(a, s, g, &p);
        votes[cell(a, s, g)] = 0;
    }
    a->meta[g] = meta;
}

/* raft.rs:942-971 on one half: every Progress reset(last_index + 1) (progress.rs:82-92), its vote cleared
 * (prs.reset_votes, :953); the self Progress gets matched = persisted, committed_index = committed (:964-970) */
static void ctl_reset(ro_arena_view *a, uint8_t *votes, uint32_t g, const uint64_t *arg) {
    uint32_t meta = a->meta[g];
    for (uint32_t s = 0; s < RO_SLOTS; s++) {
        if (!(present_of(meta) & (1u << s))) continue;
        ro_progress p;
        ro_inflights ring;
        load_progress_ins(a, s, g, &p, &ring);
        ro_progress_reset(&p, arg[1] + 1);
        if ((meta & RO_META_HAS_SELF) && RO_META_SELF(meta) == s) {
            p.matched = arg[3];
            p.committed_index = arg[2];
        }
        store_progress(a, s, g, &p);
        votes[cell(a, s, g)] = 0;
    }
    a->term_start[g] = arg[0];
    a->last_index[g] = arg[1];
    a->committed[g] = arg[2];
}

/* raft.rs:1176-1192 on one half: prs[self].become_replicate() (progress.rs:110-114), then the empty entry of the
 * new term is appended (append_entry, :1192): last_index + 1, which is the first index of the term */
static void ctl_become_leader(ro_arena_view *a, uint32_t g) {
    uint32_t meta = a->meta[g];
    if (meta & RO_META_HAS_SELF) {
        ro_progress p;
        ro_inflights ring;
        load_progress_ins(a, RO_META_SELF(meta), g, &p, &ring);
        ro_progress_become_replicate(&p);
        store_progress(a, RO_META_SELF(meta), g, &p);
    }
    a->last_index[g] += 1;
    a->term_start[g] = a->last_index[g];
}

/* voter ids (8 * half + slot + 1) of a group over both halves */
static void ctl_voters(const ro_arena_view *a, uint32_t g, uint64_t *in_ids, size_t *n_in, uint64_t *out_ids, size_t *n_out) {
    *n_in = *n_out = 0;
    for (uint32_t h = 0; h < halves_of(a, g); h++) {
        uint32_t m = a->meta[g + h];
        for (uint32_t s = 0; s < RO_SLOTS; s++) {
            if (RO_META_IN(m) & (1u << s)) in_ids[(*n_in)++] = 8 * h + s + 1;
            if (RO_META_OUT(m) & (1u << s)) out_ids[(*n_out)++] = 8 * h + s + 1;
        }
    }
}

/* tracker.rs:367-372 vote_result(|id| set.get(id).map(|_| true)) == Won, the set = peers of `mask` */
static int ctl_quorum(const ro_arena_view *a, uint32_t g, uint32_t mask) {
    uint64_t in_ids[2 * RO_SLOTS], out_ids[2 * RO_SLOTS], v_ids[2 * RO_SLOTS];
    uint8_t v_yes[2 * RO_SLOTS];
    size_t n_in, n_out, n_v = 0;
    ctl_voters(a, g, in_ids, &n_in, out_ids, &n_out);
    for (uint32_t p = 0; p < 2 * RO_SLOTS; p++)
        if (mask & (1u << p)) v_ids[n_v] = p + 1, v_yes[n_v++] = 1;
    ro_vote_map vm = {v_ids, v_yes, n_v};
    return ro_joint_vote_result(in_ids, n_in, out_ids, n_out, &vm) == RO_VOTE_WON;
}

/* tracker.rs:346-361: the perspective's own Progress turns recently active; every other Progress counts when it was
 * and is then cleared */
static int ctl_quorum_recently_active(ro_arena_view *a, uint32_t g, uint32_t perspective) {
    uint32_t active = 0;
    for (uint32_t p = 0; p < halves_of(a, g) * RO_SLOTS; p++) {
        uint32_t h = p / RO_SLOTS, s = p % RO_SLOTS;
        if (!(present_of(a->meta[g + h]) & (1u << s))) continue;
        uint8_t *f = &a->pflags[cell(a, s, g + h)];
        if (p == perspective) {
            *f |= RO_PF_RECENT_ACTIVE;
            active |= 1u << p;
        } else {
            if (*f & RO_PF_RECENT_ACTIVE) active |= 1u << p;
            *f &= (uint8_t)~RO_PF_RECENT_ACTIVE;
        }
    }
    return ctl_quorum(a, g, active);
}

/* one Progress method on cell (s, g): progress.rs:75-243 and, on arenas that keep the windows, inflights.rs:54-123
 * (-3 without them); -1 where the reference panics, -2 for an unknown method */
static int32_t ctl_progress_op(ro_arena_view *a, uint32_t g, uint32_t s, uint32_t op, const uint64_t *x) {
    ro_progress p;
    ro_inflights ring;
    load_progress_ins(a, s, g, &p, &ring);
    int32_t ret = 0;
    switch (op) {
    case 0: ret = ro_progress_maybe_update(&p, x[0]); break;
    case 1: ret = ro_progress_maybe_decr_to(&p, x[0], x[1], x[2]); break;
    case 2: ro_progress_update_committed(&p, x[0]); break;
    case 3: ro_progress_optimistic_update(&p, x[0]); break;
    case 4: ro_progress_become_probe(&p); break;
    case 5: ro_progress_become_replicate(&p); break;
    case 6: ro_progress_become_snapshot(&p, x[0]); break;
    case 7: ro_progress_snapshot_failure(&p); break;
    case 8: ret = ro_progress_maybe_snapshot_abort(&p); break;
    case 9: ret = ro_progress_is_paused(&p); break;
    case 10: ro_progress_resume(&p); break;
    case 11: ro_progress_pause(&p); break;
    case 12: ret = ro_progress_update_state(&p, x[0]); break;
    case 13: ro_progress_reset(&p, x[0]); break;
    case 14: ret = p.ins ? ro_inflights_add(p.ins, x[0]) : -3; break;
    case 15: if (p.ins) ro_inflights_free_to(p.ins, x[0]); else ret = -3; break;
    case 16: if (p.ins) ro_inflights_free_first_one(p.ins); else ret = -3; break;
    case 17: if (p.ins) ro_inflights_reset(p.ins); else ret = -3; break;
    case 18: ret = p.ins ? ro_inflights_full(p.ins) : -3; break;
    default: ret = -2;
    }
    store_progress(a, s, g, &p);
    return ret;
}

static ro_ctl_result ctl_one(ro_arena_view *a, uint8_t *votes, const ro_ctl_cmd *m) {
    ro_ctl_result r = {0, 0};
    uint32_t g = m->group, g2, s2;
    if (m->op > RO_CTL_PROGRESS_OP) return (r.status = RO_ERR_INVALID, r); /* no such call */
    if (g >= a->n_groups) return (r.status = RO_ERR_RANGE, r);
    uint32_t meta = a->meta[g], halves = halves_of(a, g);
    int hi = (meta & RO_META_WIDE_HI) != 0;
    switch (m->op) {
    case RO_CTL_SET_CONF: {
        uint64_t lim = halves == 2 ? 0xffffu : 0xffu;
        int has_self = m->peer_slot != 0xff;
        if (hi) return (r.status = RO_ERR_RANGE, r);
        if ((m->a[0] | m->a[1] | m->a[2]) > lim || (has_self && m->peer_slot >= halves * RO_SLOTS))
            return (r.status = RO_ERR_TOO_MANY_PEERS, r);
        for (uint32_t h = 0; h < halves; h++) {
            uint32_t sh = 8 * h;
            uint32_t nm = (uint32_t)(((m->a[0] >> sh) & 0xffu) | (((m->a[1] >> sh) & 0xffu) << 8) | (((m->a[2] >> sh) & 0xffu) << 16)) |
                          (a->meta[g + h] & (RO_META_GROUP_COMMIT | RO_META_WIDE_LO | RO_META_WIDE_HI));
            if (has_self && m->peer_slot >= sh && m->peer_slot < sh + 8) nm |= ((uint32_t)(m->peer_slot - sh) << 24) | RO_META_HAS_SELF;
            ctl_apply_conf(a, votes, g + h, nm, m->a[3]);
        }
        return r;
    }
    case RO_CTL_SET_TERM: /* either half; a wide group's low half names both */
        a->term[g] = m->a[0];
        if (halves == 2) a->term[g + 1] = m->a[0];
        return r;
    case RO_CTL_VOTE_RESULT: { /* either half */
        uint32_t gr, rj;
        int v = ro_arena_vote_result(a, votes, g, &gr, &rj);
        r.value = (int32_t)((uint32_t)v | gr << 8 | rj << 16);
        return r;
    }
    case RO_CTL_RECORD_VOTE: /* tracker.rs:308-310 votes.entry(id).or_insert(vote) */
        if (!ctl_resolve(a, g, m->peer_slot, &g2, &s2)) return (r.status = RO_ERR_RANGE, r);
        if (!votes[cell(a, s2, g2)]) votes[cell(a, s2, g2)] = m->arg ? 2 : 1;
        return r;
    case RO_CTL_ASSIGN_COMMIT_GROUP: /* raft.rs:531-540: an unknown peer is skipped */
        if (!ctl_resolve(a, g, m->peer_slot, &g2, &s2)) return (r.status = RO_ERR_RANGE, r);
        if (present_of(a->meta[g2]) & (1u << s2)) a->commit_group_id[cell(a, s2, g2)] = m->a[0];
        return r;
    case RO_CTL_PROGRESS_OP:
        if (!ctl_resolve(a, g, m->peer_slot, &g2, &s2)) return (r.status = RO_ERR_RANGE, r);
        if (!(present_of(a->meta[g2]) & (1u << s2))) return (r.status = RO_ERR_PEER_NOT_FOUND, r);
        if (m->arg > 18) return (r.status = RO_ERR_INVALID, r);
        r.value = ctl_progress_op(a, g2, s2, m->arg, m->a);
        return r;
    default:
        break;
    }
    if (hi) return (r.status = RO_ERR_RANGE, r); /* the rest name a wide group by its low half */
    switch (m->op) {
    case RO_CTL_RESET:
        for (uint32_t h = 0; h < halves; h++) ctl_reset(a, votes, g + h, m->a);
        break;
    case RO_CTL_BECOME_LEADER:
        for (uint32_t h = 0; h < halves; h++) ctl_become_leader(a, g + h);
        break;
    case RO_CTL_SET_LOG_BOUNDS: /* raft.rs:974-991 append_entry: the log grew */
        for (uint32_t h = 0; h < halves; h++) a->term_start[g + h] = m->a[0], a->last_index[g + h] = m->a[1];
        break;
    case RO_CTL_COMMIT_TO: /* raft_log.rs:286-300 on the log [1, last_index] */
        if (halves == 2) ctl_wide_sync(a, g);
        for (uint32_t h = 0; h < halves; h++) {
            ro_raft_log l = {1, 0, NULL, (size_t)a->last_index[g + h], a->committed[g + h]};
            if (ro_log_commit_to(&l, m->a[0]) != 0 && h == 0) r.status = RO_ERR_COMMIT_RANGE;
            a->committed[g + h] = l.committed;
        }
        break;
    case RO_CTL_MAYBE_COMMIT_TO: /* raft_log.rs:487-499 at the leader's term: term(i) == term <=> term_start <= i <= last_index */
        if (halves == 2) ctl_wide_sync(a, g);
        for (uint32_t h = 0; h < halves; h++) {
            int adv = m->a[0] > a->committed[g + h] && m->a[0] >= a->term_start[g + h] && m->a[0] <= a->last_index[g + h];
            if (adv) a->committed[g + h] = m->a[0];
            if (h == 0) r.value = adv;
        }
        break;
    case RO_CTL_SET_GROUP_COMMIT: /* tracker.rs:238-241 enable_group_commit */
        for (uint32_t h = 0; h < halves; h++)
            a->meta[g + h] = m->arg ? (a->meta[g + h] | RO_META_GROUP_COMMIT) : (a->meta[g + h] & ~RO_META_GROUP_COMMIT);
        break;
    case RO_CTL_RESET_VOTES: /* tracker.rs:301-304 */
        for (uint32_t h = 0; h < halves; h++)
            for (uint32_t s = 0; s < RO_SLOTS; s++) votes[cell(a, s, g + h)] = 0;
        break;
    case RO_CTL_HAS_QUORUM:
        r.value = ctl_quorum(a, g, (uint32_t)m->a[0] & (halves == 2 ? 0xffffu : 0xffu));
        break;
    case RO_CTL_QUORUM_RECENTLY_ACTIVE:
        if (m->peer_slot >= halves * RO_SLOTS) return (r.status = RO_ERR_RANGE, r);
        r.value = ctl_quorum_recently_active(a, g, m->peer_slot);
        break;
    }
    return r;
}

void ro_arena_control(ro_arena_view *a, uint8_t *votes, const ro_ctl_cmd *cmds, size_t n, ro_ctl_result *results) {
    for (size_t i = 0; i < n; i++) results[i] = ctl_one(a, votes, &cmds[i]);
}
