// k_app_follow.cuh -- entry-less MsgAppend frames at the follower (DESIGN 3.16): Raft::step's term rules as statuses,
// then handle_append_entries (raft.rs:2389-2448) with maybe_append / find_conflict_by_term (raft_log.rs:209-279) and no
// entries -- commit_to(min(m.commit, m.index)) or a rejection with its hint -- and one MsgAppendResponse back through
// send (raft.rs:602-661) for the first frame of every group that reaches the decision.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).
//
// The log stays with the caller: its table (raftgpu_follower_log, one row per group slot) states the log's last term
// run [run_start, last_index] with its term, and the pass reads term(i) only for i in that run (run_term) and above
// last_index (0, raft_log.rs:125).  A frame whose decision needs any other term, or that carries entries, goes back to
// the host whole.  Nothing but committed is ever written.  The frame's header is the follower's own (group << 4 | x);
// x is not read and goes back unchanged in the response's header.
//
// kAppend = true is raftgpu_follower_append_entries (DESIGN 3.17): a matching frame's entries are walked once
// (wire_entries, k_wire.cuh), find_conflict is decided from the run, and the apply pass moves last_index, keeps the
// table's run current and reports the appended span; the log's bytes stay with the caller.
//
// Four kernels and no waiting between blocks: afw_scan_kernel stages and decodes every frame once, classifies and
// decides it and writes a 64-byte record per frame that reached the decision; afw_apply_kernel marks the later frames
// of a group DUP, runs commit_to on the first one where it matched and sums the responses per block;
// block_starts_kernel<2> (k_wire.cuh) turns the sums into block starts; reply_write_kernel<AfwReply> (k_wire.cuh) encodes
// the responses (wire_put_app_resp_frame) and stores them through shared memory.  Every kernel takes kWireThreads
// frames per block: one block sum per scan block.
//
// kRuns = true is an arena with follower runs (DESIGN 3.22): a row per group states up to two term runs below the
// table's run, and the decision reads term(i) there too (afw_runs_*); the entries pass keeps the row current.  The
// <false> kernels are the passes as they were.

// A decided frame's record: w0 = its header | the kAfw* bits; the response's fields.  A matching frame's commit is
// min(m.commit, m.index) until the apply pass replaces it with the committed after commit_to.
constexpr uint64_t kAfwReject = 1ull << 32, kAfwStale = 1ull << 33, kAfwCommit = 1ull << 34, kAfwAppend = 1ull << 35;
constexpr uint64_t kAfwRuns = 1ull << 36;  // (kRuns, appended) the group's row becomes {the new run, AfwRunsIo::next[i]}
struct __align__(16) AfwRec {
    uint64_t w0, to, from, term, log_term, index, commit, reject_hint;
};

__device__ __forceinline__ uint32_t afw_len(const AfwRec &r) {
    return wire_app_resp_len(r.to, r.from, r.term, r.log_term, r.index, r.commit, (r.w0 & kAfwReject) != 0, r.reject_hint);
}

// A matching frame with entries (afw_frame<true>), its walk (ents, e) done: maybe_append from the run.  m.index is at or
// above run_start here (the match is known and m.index <= last_index, or the frame is a gap and goes back to the host),
// or in a stated run of the row (kRuns, which then replaces the run this leaves: afw_runs_after).
__device__ __forceinline__ uint32_t afw_append(const WireSrc &w, AfwRec &r, raftgpu_follower_appended &ap, uint32_t i,
                                               const WireMsg &m, uint32_t ents, const WireEntries &e, uint64_t last,
                                               uint64_t committed, uint64_t run_start, uint64_t run_term) {
    if (ents == kEntsNeedsLog || m.index > last) return RAFTGPU_WIRE_NEEDS_LOG;  // (m.index > last_index: a gap)
    // Both COMMIT_RANGE checks below restate the reference's fatal!s and cannot fire here: past the stale rule
    // m.index >= committed, so conflict >= m.index + 1 > committed; and to_commit <= last_new <= new_last.
    const uint64_t conflict = e.conflict ? m.index + e.conflict : 0;
    if (conflict && conflict <= committed) return RAFTGPU_WIRE_COMMIT_RANGE;  // raft_log.rs:259-265 fatal!
    const uint64_t last_new = m.index + e.count, new_last = conflict ? last_new : last;
    const uint64_t to_commit = umin64(m.commit, last_new);
    if (to_commit > umax64(committed, new_last)) return RAFTGPU_WIRE_COMMIT_RANGE;  // raft_log.rs:291-298 fatal!
    r.w0 |= kAfwCommit;
    r.index = last_new;  // raft.rs:2441 to_send.index = last_idx
    r.commit = to_commit;
    if (conflict) {
        r.w0 |= kAfwAppend;
        const bool keep = e.uniform && e.tail_term == run_term && conflict - 1 >= run_start;
        r.reject_hint = keep ? run_start : m.index + e.tail;
        r.log_term = keep ? run_term : e.tail_term;
        ap.first_index = conflict;
        ap.last_index = last_new;
        ap.run_start = r.reject_hint;
        ap.run_term = r.log_term;
        ap.span_off = w.offsets[i] + 4u + e.span_off;
        ap.span_len = e.span_end - e.span_off;
    }
    return RAFTGPU_WIRE_OK;
}

// Follower runs (raftgpu_arena_enable_follower_runs, DESIGN 3.22): one row per group slot in LeaderRuns' layout, anchor =
// {anchor_term, anchor_start}: run 1 is [s1, anchor_start - 1] at t1, run 2 [s2, s1 - 1] at t2, a start of 0 states no
// run, and stated terms strictly decrease downward.  A row is read only while the table's run is non-empty and equals
// its anchor: by Log Matching the log below (anchor_start, anchor_term) is then the one the row was stated for.  A pair's
// row is on its low half.  next (the entries pass; nullptr in the entry-less one): per frame, the row an appended frame
// with kAfwRuns leaves, for the apply pass to store when the frame claims its group.
struct AfwRuns {
    uint64_t s1, s2, t1, t2;
};
struct AfwRunsIo {
    LeaderRuns *rows;
    AfwRuns *next;
};

// Group g's row below its table run, all zero when it is not anchored there.
__device__ __forceinline__ AfwRuns afw_runs_row(const LeaderRuns *__restrict__ rows, uint32_t g, uint64_t run_start,
                                                uint64_t run_term, uint64_t last) {
    if (run_start > last) return AfwRuns{0, 0, 0, 0};
    const ulonglong2 a = rows[g].anchor;
    if (a.x == 0 || a.x != run_term || a.y != run_start) return AfwRuns{0, 0, 0, 0};
    const ulonglong2 s = rows[g].start, t = rows[g].term;
    return AfwRuns{s.x, s.y, t.x, t.y};
}

// term(x) for x below the table's run from the row; false = not stated.
__device__ __forceinline__ bool afw_runs_term(const AfwRuns &R, uint64_t x, uint64_t &t) {
    if (R.s1 && x >= R.s1) {
        t = R.t1;
        return true;
    }
    if (R.s2 && x >= R.s2) {
        t = R.t2;
        return true;
    }
    return false;
}

// find_conflict_by_term(i, lt) (raft_log.rs:209-235) for i below the table's run: the first of run 1, run 2 at or below i
// whose term is <= lt gives {hint, its term}; false = the walk leaves the lowest stated run.
__device__ __forceinline__ bool afw_runs_walk(const AfwRuns &R, uint64_t i, uint64_t lt, uint64_t &hint, uint64_t &term) {
    if (R.s1 && i >= R.s1) {
        if (R.t1 <= lt) {
            hint = i;
            term = R.t1;
            return true;
        }
        i = R.s1 - 1;
    }
    if (R.s2 && i >= R.s2 && R.t2 <= lt) {
        hint = i;
        term = R.t2;
        return true;
    }
    return false;
}

// The top of the log after an append at conflict c that does not keep the table's run: from the top, the trailing block
// of appended entries [k, ..] at t, the block before it [kp, k - 1] at tp (two: the entries hold two terms or more), and
// -- when those blocks are all the appended entries (whole) -- the segment that held c - 1, cut there, and the stated
// ones below it; equal neighbours merge.  The table's run becomes the top segment (*ts, *tt) and the row the next two
// while their terms strictly decrease (fewer runs are never wrong).
__device__ __forceinline__ void afw_runs_after(uint64_t c, uint64_t k, uint64_t t, uint64_t kp, uint64_t tp, bool two,
                                               bool whole, uint64_t run_start, uint64_t run_term, const AfwRuns &R,
                                               uint64_t &ts, uint64_t &tt, AfwRuns &nr) {
    uint64_t s0 = k, t0 = t, s1 = kp, t1 = tp, s2 = 0, t2 = 0;
    uint32_t n = two ? 2u : 1u;  // segments so far; 4 = full
    const auto push = [&](uint64_t s, uint64_t u) {
        if (n == 1) {
            if (u == t0) s0 = s;
            else s1 = s, t1 = u, n = 2;
        } else if (n == 2) {
            if (u == t1) s1 = s;
            else s2 = s, t2 = u, n = 3;
        } else if (n == 3) {
            if (u == t2) s2 = s;
            else n = 4;
        }
    };
    if (whole) {
        const uint64_t x = c - 1;
        if (x >= run_start) push(run_start, run_term);
        if (x >= run_start || x >= R.s1) {
            if (R.s1) push(R.s1, R.t1);
        }
        if (R.s1 && R.s2) push(R.s2, R.t2);
    }
    ts = s0;
    tt = t0;
    nr = AfwRuns{0, 0, 0, 0};
    if (n >= 2 && s1 && t1 && t1 < t0) {
        nr.s1 = s1;
        nr.t1 = t1;
        if (n >= 3 && s2 && t2 && t2 < t1) {
            nr.s2 = s2;
            nr.t2 = t2;
        }
    }
}

// Frame i: its status before the duplicate rule (checks in the order of raftgpu.h) and, for the frames that reach the
// decision (OK, NEEDS_LOG, COMMIT_RANGE), its record (w0 alone for the last two).  kAppend (raftgpu_follower_append_entries):
// a matching frame's entries are appended (maybe_append, raft_log.rs:249-279); an appended frame's record carries the
// new run in log_term (its term) and reject_hint (its start) to the apply pass, and ap = its raftgpu_follower_appended
// (untouched for every other frame).  kRuns: term(i) is read from group g's row too (io.rows, never inside the table's
// run), and an appended frame whose new log top moves off the table's run or the row gets kAfwRuns, the table's new run
// in its record and ap, and the row's runs in nr.
template <bool kAppend, bool kRuns = false>
__device__ __forceinline__ uint32_t afw_frame(const Columns &c, const WireSrc &w, const raftgpu_follower_log *__restrict__ logs,
                                              const WireStage &s, const uint8_t *stage, uint32_t i, AfwRec &r,
                                              raftgpu_follower_appended &ap, const AfwRunsIo &io = {}, AfwRuns *nr = nullptr) {
    uint32_t hdr;
    const uint8_t *msg;
    WireMsg m;
    if (wire_open<false, true, false, false, true>(w, s, stage, i, hdr, msg, m) != RAFTGPU_WIRE_OK) return RAFTGPU_WIRE_MALFORMED;
    const uint32_t g = hdr >> 4, meta = c.meta[g];
    if ((meta & RAFTGPU_META_WIDE_HI) || (c.rq_cap && !(c.rq_hc[g] & kRqAlloc))) return RAFTGPU_WIRE_MALFORMED;
    if (m.msg_type != 3u) return RAFTGPU_WIRE_SKIP_TYPE;  // MsgAppend, eraftpb.proto:53
    const raftgpu_follower_log &l = logs[g];
    // a Follower (the caller's bit) and not a leader here: step_follower (raft.rs:2271-2275) is the only path taken
    if (!(l.flags & RAFTGPU_FOLLOWER_SELECT) || c.term_start[g] != RAFTGPU_NO_TERM_START) return RAFTGPU_WIRE_ROLE;
    const uint64_t term = c.term[g];
    if (term == 0 || m.term != term) return RAFTGPU_WIRE_TERM;  // raft.rs:1280-1411 decide those on the host
    r.w0 = hdr;
    if constexpr (!kAppend) {
        if (m.entries) return RAFTGPU_WIRE_NEEDS_LOG;
    }
    uint64_t last = c.last_index[g], committed = c.committed[g];
    if (meta & RAFTGPU_META_WIDE_LO) {
        last = umax64(last, c.last_index[g + 1]);
        committed = umax64(committed, c.committed[g + 1]);
    }
    uint32_t ents = kEntsOk;
    std::conditional_t<kRuns, WireEntriesRuns, WireEntries> e;
    AfwRuns R{0, 0, 0, 0};  // (kRuns) the row, read here when m.index is below the table's run, later where needed
    if constexpr (kRuns) {
        if (m.index <= last && m.index < l.run_start) R = afw_runs_row(io.rows, g, l.run_start, l.run_term, last);
    }
    if constexpr (kAppend) {  // every entry of every frame that got this far: an Entry that is not well formed is MALFORMED
        if (m.entries) {
            if constexpr (kRuns)
                ents = wire_entries_runs(msg, w.offsets[i + 1] - w.offsets[i] - 4u, m.index, last, l.run_start, l.run_term,
                                         R.s1, R.t1, R.t2, e);
            else
                ents = wire_entries(msg, w.offsets[i + 1] - w.offsets[i] - 4u, m.index, last, l.run_term, e);
            if (ents == kEntsMalformed) return RAFTGPU_WIRE_MALFORMED;
        }
    }
    r.to = m.from;    // to_send.to = m.from (raft.rs:2400, 2407)
    r.from = l.id;    // send: from = self.id (raft.rs:610-612)
    r.term = term;    // send: term = self.term (raft.rs:650)
    r.log_term = r.reject_hint = 0;
    if (m.index < committed) {  // raft.rs:2394-2404
        r.w0 |= kAfwStale;
        r.index = r.commit = committed;
        return RAFTGPU_WIRE_OK;
    }
    const uint64_t run_start = l.run_start, run_term = l.run_term;
    if constexpr (kRuns) {  // the rule below with term(i) from the row under the table's run
        const bool below = m.index <= last && m.index < run_start;  // (R was read)
        uint64_t tm = m.index > last ? 0ull : run_term;
        if (below && !afw_runs_term(R, m.index, tm)) return RAFTGPU_WIRE_NEEDS_LOG;
        if (tm == m.log_term) {
            if constexpr (kAppend) {
                if (m.entries) {
                    const uint32_t st = afw_append(w, r, ap, i, m, ents, e, last, committed, run_start, run_term);
                    const uint64_t conflict = m.index + e.conflict;
                    if (st != RAFTGPU_WIRE_OK || !(r.w0 & kAfwAppend) ||
                        (e.uniform && e.tail_term == run_term && conflict - 1 >= run_start))
                        return st;  // (the table's run kept: so is the row)
                    if (!below) R = afw_runs_row(io.rows, g, run_start, run_term, last);
                    afw_runs_after(conflict, m.index + e.tail, e.tail_term, m.index + e.pre, e.pre_term, !e.uniform,
                                   e.uniform || e.pre == e.conflict, run_start, run_term, R, r.reject_hint, r.log_term, *nr);
                    r.w0 |= kAfwRuns;
                    ap.run_start = r.reject_hint;
                    ap.run_term = r.log_term;
                    return st;
                }
            }
            const uint64_t to_commit = umin64(m.commit, m.index);
            if (to_commit > umax64(committed, last)) return RAFTGPU_WIRE_COMMIT_RANGE;  // raft_log.rs:291-298 fatal!
            r.w0 |= kAfwCommit;
            r.index = m.index;
            r.commit = to_commit;
            return RAFTGPU_WIRE_OK;
        }
        const uint64_t h = umin64(m.index, last);
        if (h >= run_start && run_term <= m.log_term) {  // the walk stops at once inside the table's run
            r.reject_hint = h;
            r.log_term = run_term;
        } else {
            if (!below) R = afw_runs_row(io.rows, g, run_start, run_term, last);
            if (!afw_runs_walk(R, h >= run_start ? run_start - 1 : h, m.log_term, r.reject_hint, r.log_term))
                return RAFTGPU_WIRE_NEEDS_LOG;  // (run_start 0: no row is anchored there)
        }
        r.w0 |= kAfwReject;
        r.index = m.index;
        r.commit = committed;
        return RAFTGPU_WIRE_OK;
    }
    if (m.index > last || m.index >= run_start) {  // term(m.index) is known: 0 above last_index, run_term in the run
        if ((m.index > last ? 0ull : run_term) == m.log_term) {  // maybe_append matches (raft_log.rs:243)
            if constexpr (kAppend) {
                if (m.entries) return afw_append(w, r, ap, i, m, ents, e, last, committed, run_start, run_term);
            }
            const uint64_t to_commit = umin64(m.commit, m.index);
            if (to_commit > umax64(committed, last)) return RAFTGPU_WIRE_COMMIT_RANGE;  // raft_log.rs:291-298 fatal!
            r.w0 |= kAfwCommit;
            r.index = m.index;  // last_new_index = idx + 0
            r.commit = to_commit;
            return RAFTGPU_WIRE_OK;
        }
    } else {
        return RAFTGPU_WIRE_NEEDS_LOG;
    }
    // the rejection: find_conflict_by_term(min(m.index, last_index), m.log_term) stops at once inside the run
    const uint64_t h = umin64(m.index, last);
    if (h < run_start || run_term > m.log_term) return RAFTGPU_WIRE_NEEDS_LOG;
    r.w0 |= kAfwReject;
    r.index = m.index;
    r.reject_hint = h;
    r.log_term = run_term;
    r.commit = committed;
    return RAFTGPU_WIRE_OK;
}

// The apply side of kAfwRuns: the claimant of group g stores the row its scan left in io.next[i], anchored at the
// table's new run (the record's reject_hint and log_term, before they are cleared).
__device__ __forceinline__ void afw_runs_store(const AfwRunsIo &io, uint32_t g, uint32_t i, uint64_t w0, const AfwRec &r) {
    if (!(w0 & kAfwRuns)) return;
    const AfwRuns nr = io.next[i];
    io.rows[g] = LeaderRuns{make_ulonglong2(r.log_term, r.reject_hint), make_ulonglong2(nr.s1, nr.s2),
                            make_ulonglong2(nr.t1, nr.t2)};
}

// Pass 1: classify and decide every frame; status[i] = wire status << 4; the record of a frame that reached the
// decision, first_frame[group] = the lowest such frame of the group.  kAppend: appended[i] = the frame's
// raftgpu_follower_appended (zero unless it appends; the apply pass zeroes a DUP one).  Launched with kWireThreads
// threads per block.  kRuns: the rows in io (the last parameter, so that the others keep their offsets); kAppend also
// writes io.next[i] of a frame with kAfwRuns.
template <bool kAppend, bool kRuns>
__global__ void __launch_bounds__(kWireThreads) afw_scan_kernel(Columns c, WireSrc w, const raftgpu_follower_log *__restrict__ logs,
                                                                uint8_t *__restrict__ status, AfwRec *__restrict__ recs,
                                                                uint32_t *__restrict__ first_frame,
                                                                raftgpu_follower_appended *__restrict__ appended,
                                                                AfwRunsIo io) {
    __shared__ __align__(16) uint8_t stage[kWireStage + 16];
    WireStage s;
    const uint32_t i = wire_block_frame(w, stage, s);
    if (i == kNoFrame) return;
    AfwRec r;
    raftgpu_follower_appended ap{};
    AfwRuns nr;
    const uint32_t st = afw_frame<kAppend, kRuns>(c, w, logs, s, stage, i, r, ap, io, &nr);
    status[i] = static_cast<uint8_t>(st << 4);
    if constexpr (kAppend) appended[i] = ap;
    if constexpr (kAppend && kRuns) {
        if (st == RAFTGPU_WIRE_OK && (r.w0 & kAfwRuns)) io.next[i] = nr;
    }
    if (st == RAFTGPU_WIRE_OK) recs[i] = r;
    else if (st == RAFTGPU_WIRE_NEEDS_LOG || st == RAFTGPU_WIRE_COMMIT_RANGE) recs[i].w0 = r.w0;
    else return;
    atomicMin(&first_frame[static_cast<uint32_t>(r.w0) >> 4], i);
}

// Pass 2: a later frame of a group is RAFTGPU_WIRE_DUP.  The first one, when OK and matching, runs commit_to -- on both
// halves of a wide pair, after wide_sync, as RAFTGPU_CTL_COMMIT_TO does -- and keeps the new committed in its record.
// kAppend: an appended frame first sets last_index (both halves of a pair, as RAFTGPU_CTL_SET_LOG_BOUNDS) and the
// table's run, and clears the run from its record; a DUP frame's appended record is zeroed.
// from_out[i] (nullable) = m.from of an applied frame, 0 otherwise.  blk[2 * block + {0, 1}] = the block's responses
// and their bytes.  Algorithmic bytes per frame: 1 read + 1 written (+ 8 from_out); per frame that reached the decision
// 8 (w0) + 4 (first_frame) read; per applied one 56 (record) read, and for a match 16-32 (committed, last_index) read,
// 8-16 (committed) + 8 (record) written; per appended one 8-16 (last_index) + 16 (run) + 16 (record) written, and with
// kAfwRuns (kRuns) 32 (io.next) read and 48 (the row) written.
template <bool kAppend, bool kRuns>
__global__ void __launch_bounds__(kWireThreads) afw_apply_kernel(Columns c, uint32_t n, uint8_t *__restrict__ status,
                                                                 AfwRec *__restrict__ recs, const uint32_t *__restrict__ first_frame,
                                                                 uint64_t *__restrict__ from_out, uint32_t *__restrict__ blk,
                                                                 raftgpu_follower_log *__restrict__ logs,
                                                                 raftgpu_follower_appended *__restrict__ appended,
                                                                 AfwRunsIo io) {
    const uint32_t i = blockIdx.x * kWireThreads + threadIdx.x;
    uint32_t resp = 0, bytes = 0;
    if (i < n) {
        uint64_t from = 0;
        const uint32_t st = status[i] >> 4;
        if (st == RAFTGPU_WIRE_OK || st == RAFTGPU_WIRE_NEEDS_LOG || st == RAFTGPU_WIRE_COMMIT_RANGE) {
            const uint64_t w0 = recs[i].w0;
            const uint32_t g = static_cast<uint32_t>(w0) >> 4;
            if (first_frame[g] != i) {
                status[i] = static_cast<uint8_t>(RAFTGPU_WIRE_DUP << 4);
                if constexpr (kAppend) {
                    if (st == RAFTGPU_WIRE_OK && (w0 & kAfwAppend)) appended[i] = raftgpu_follower_appended{};
                }
            } else if (st == RAFTGPU_WIRE_OK) {
                AfwRec r = recs[i];
                if constexpr (kAppend) {
                    if (w0 & kAfwAppend) {  // truncate_and_append: last_index = m.index + entries
                        if (c.meta[g] & RAFTGPU_META_WIDE_LO) {
                            wide_sync(c, g);
                            c.last_index[g + 1] = r.index;
                        }
                        c.last_index[g] = r.index;
                        logs[g].run_start = r.reject_hint;
                        logs[g].run_term = r.log_term;
                        if constexpr (kRuns) afw_runs_store(io, g, i, w0, r);
                        r.log_term = r.reject_hint = 0;  // the response carries neither
                        recs[i].log_term = 0;
                        recs[i].reject_hint = 0;
                    }
                }
                if (w0 & kAfwCommit) {
                    if (c.meta[g] & RAFTGPU_META_WIDE_LO) {
                        wide_sync(c, g);
                        commit_to_group(c, g + 1, r.commit);
                    }
                    commit_to_group(c, g, r.commit);  // (in range: the scan checked it)
                    r.commit = c.committed[g];        // raft.rs:2446 to_send.commit = raft_log.committed
                    recs[i].commit = r.commit;
                }
                uint32_t low = RAFTGPU_RES_OK | ((w0 & kAfwReject) ? RAFTGPU_FAPP_REJECT : 0u) |
                               ((w0 & kAfwStale) ? RAFTGPU_FAPP_STALE : 0u);
                if constexpr (kAppend) low |= (w0 & kAfwAppend) ? RAFTGPU_FAPP_APPENDED : 0u;
                status[i] = static_cast<uint8_t>((RAFTGPU_WIRE_OK << 4) | low);
                from = r.to;
                resp = 1;
                bytes = afw_len(r);
            }
        }
        if (from_out) from_out[i] = from;
    }
    block_sums<2, kWireThreads>({resp, bytes}, blk);
}

// Waves (raftgpu_arena_set_wire_waves, DESIGN 3.19): the decision repeated over the frames it left DUP, each wave against
// the state the waves before it left (committed, last_index, the table's run).  Wave 1 is afw_scan_kernel and
// afw_wave_apply_kernel over the batch; a later wave is wire_wave_claim_kernel<true> (k_wire.cuh) and
// afw_wave_apply_kernel over the list (WaveIo) the wave before it wrote, which decides the claimant only.  A group's claimant leaves the group's first_frame entry kNoFrame
// when it was applied, kWaveStop when it was not (NEEDS_LOG, COMMIT_RANGE): the group's later frames then stay DUP, as
// the host resubmits them only after it has handled the claimant.  block_starts_kernel<2> and reply_write_kernel run
// once after the last wave.

// Frame i after its wave's scan, as afw_apply_kernel decides it, with the claimant's mark on the group's entry.  true =
// DUP and on the next wave's list; *resp_bytes = the bytes of its response (0: none), *from = m.from when applied.
template <bool kAppend, bool kRuns>
__device__ __forceinline__ bool afw_wave_frame(const Columns &c, uint32_t i, uint8_t *__restrict__ status, AfwRec *__restrict__ recs,
                                               uint32_t *__restrict__ first_frame, raftgpu_follower_log *__restrict__ logs,
                                               raftgpu_follower_appended *__restrict__ appended, uint64_t &from,
                                               uint32_t &resp_bytes, const AfwRunsIo &rio) {
    const uint32_t st = status[i] >> 4;
    if (st != RAFTGPU_WIRE_OK && st != RAFTGPU_WIRE_NEEDS_LOG && st != RAFTGPU_WIRE_COMMIT_RANGE) return false;
    const uint64_t w0 = recs[i].w0;
    const uint32_t g = static_cast<uint32_t>(w0) >> 4;
    if (first_frame[g] != i) {  // (reads i, kNoFrame or kWaveStop: the claimant writes its mark during this pass)
        status[i] = static_cast<uint8_t>(RAFTGPU_WIRE_DUP << 4);
        if constexpr (kAppend) {
            if (st == RAFTGPU_WIRE_OK && (w0 & kAfwAppend)) appended[i] = raftgpu_follower_appended{};
        }
        return true;
    }
    first_frame[g] = st == RAFTGPU_WIRE_OK ? kNoFrame : kWaveStop;
    if (st != RAFTGPU_WIRE_OK) return false;
    AfwRec r = recs[i];
    if constexpr (kAppend) {
        if (w0 & kAfwAppend) {  // truncate_and_append: last_index = m.index + entries
            if (c.meta[g] & RAFTGPU_META_WIDE_LO) {
                wide_sync(c, g);
                c.last_index[g + 1] = r.index;
            }
            c.last_index[g] = r.index;
            logs[g].run_start = r.reject_hint;
            logs[g].run_term = r.log_term;
            if constexpr (kRuns) afw_runs_store(rio, g, i, w0, r);
            r.log_term = r.reject_hint = 0;  // the response carries neither
            recs[i].log_term = 0;
            recs[i].reject_hint = 0;
        }
    }
    if (w0 & kAfwCommit) {
        if (c.meta[g] & RAFTGPU_META_WIDE_LO) {
            wide_sync(c, g);
            commit_to_group(c, g + 1, r.commit);
        }
        commit_to_group(c, g, r.commit);
        r.commit = c.committed[g];  // raft.rs:2446 to_send.commit = raft_log.committed
        recs[i].commit = r.commit;
    }
    uint32_t low = RAFTGPU_RES_OK | ((w0 & kAfwReject) ? RAFTGPU_FAPP_REJECT : 0u) | ((w0 & kAfwStale) ? RAFTGPU_FAPP_STALE : 0u);
    if constexpr (kAppend) low |= (w0 & kAfwAppend) ? RAFTGPU_FAPP_APPENDED : 0u;
    status[i] = static_cast<uint8_t>((RAFTGPU_WIRE_OK << 4) | low);
    from = r.to;
    resp_bytes = afw_len(r);
    return false;
}

// The apply pass of a wave.  io.in == nullptr (wave 1): every frame of the batch after afw_scan_kernel, one per thread,
// and blk written as afw_apply_kernel writes it; else the frames of io.in over a grid-stride loop, the claimant of each
// group decided and applied, each response added to its frame's block in blk (a wave that finds no frame returns at
// once).  Every DUP frame goes on io.out.  logs: the table, written by the kAppend kernels only; rio: kRuns' rows.
template <bool kAppend, bool kRuns>
__global__ void __launch_bounds__(kWireThreads) afw_wave_apply_kernel(Columns c, WireSrc w, uint8_t *__restrict__ status,
                                                                      AfwRec *__restrict__ recs, uint32_t *__restrict__ first_frame,
                                                                      uint64_t *__restrict__ from_out, uint32_t *__restrict__ blk,
                                                                      raftgpu_follower_log *__restrict__ logs,
                                                                      raftgpu_follower_appended *__restrict__ appended,
                                                                      WaveIo io, AfwRunsIo rio) {
    if (!io.in) {
        const uint32_t i = blockIdx.x * kWireThreads + threadIdx.x;
        uint32_t bytes = 0;
        bool dup = false;
        if (i < w.n) {
            uint64_t from = 0;
            dup = afw_wave_frame<kAppend, kRuns>(c, i, status, recs, first_frame, logs, appended, from, bytes, rio);
            if (from_out) from_out[i] = from;
        }
        wave_enlist(io, dup, i);
        block_sums<2, kWireThreads>({bytes ? 1u : 0u, bytes}, blk);
        return;
    }
    const uint32_t m = *io.in_n;
    const WireStage s{0, 0, 0, false};
    for (uint32_t k0 = blockIdx.x * kWireThreads; k0 < m; k0 += gridDim.x * kWireThreads) {  // (uniform per warp)
        const uint32_t k = k0 + threadIdx.x, i = k < m ? io.in[k] : kNoFrame;
        uint32_t bytes = 0;
        bool dup = false;
        bool claim = false;
        if (i != kNoFrame) {
            // A listed frame is DUP with a zero appended record and from.  One that does not claim stays so, and leaves
            // the lists once its group is stopped (kWaveStop, written before or during this pass).
            const uint32_t f = first_frame[wire_header(w, i) >> 4];
            claim = f == i;
            dup = !claim && f != kWaveStop;
        }
        if (claim) {  // afw_scan_kernel's decision, then afw_apply_kernel's
            AfwRec r;
            raftgpu_follower_appended ap{};
            AfwRuns nr;
            const uint32_t st = afw_frame<kAppend, kRuns>(c, w, logs, s, nullptr, i, r, ap, rio, &nr);
            status[i] = static_cast<uint8_t>(st << 4);
            if constexpr (kAppend) appended[i] = ap;
            if constexpr (kAppend && kRuns) {
                if (st == RAFTGPU_WIRE_OK && (r.w0 & kAfwRuns)) rio.next[i] = nr;
            }
            if (st == RAFTGPU_WIRE_OK) recs[i] = r;
            else recs[i].w0 = r.w0;  // (NEEDS_LOG, COMMIT_RANGE: a listed frame reaches the decision)
            uint64_t from = 0;
            afw_wave_frame<kAppend, kRuns>(c, i, status, recs, first_frame, logs, appended, from, bytes, rio);
            if (from_out) from_out[i] = from;
            if (bytes) {
                atomicAdd(&blk[2 * (i / kWireThreads)], 1u);
                atomicAdd(&blk[2 * (i / kWireThreads) + 1], bytes);
            }
        }
        wave_enlist(io, dup, i);
    }
}

// Pass 4 is reply_write_kernel<AfwReply> (k_wire.cuh): the frames the apply pass marked RAFTGPU_RES_OK answer.
struct AfwReply {
    using Rec = AfwRec;
    static constexpr uint32_t kFrameMax = kWireAppRespFrameMax;
    __device__ __forceinline__ static bool answers(uint8_t status) { return status & RAFTGPU_RES_OK; }
    __device__ __forceinline__ static uint32_t len(const AfwRec &r) { return afw_len(r); }
    __device__ __forceinline__ static uint8_t *put(uint8_t *p, const AfwRec &r) {  // MsgAppendResponse, raft.rs:2406-2447
        return wire_put_app_resp_frame(p, static_cast<uint32_t>(r.w0), r.to, r.from, r.term, r.log_term, r.index, r.commit,
                                       (r.w0 & kAfwReject) != 0, r.reject_hint);
    }
};
