// raftgpu.hpp -- C++17 mirror of the raft-rs tracker / quorum surface over the C-ABI.
//
// The reference is a Rust crate and the project builds without a Rust toolchain, so the host side above
// include/raftgpu.h is written in C++: same type and method names, argument meaning and error
// behaviour as the crate (file:line of each counterpart is given), every piece of arithmetic
// forwarded to libraftgpu.so -- there is no CPU implementation of the path in here.  The Rust
// shim a raft-rs maintainer would write has this exact shape (INTEGRATION.md).
//
// Single-group calls go through small synchronous kernels and are meant for the control plane
// and for the drop-in tests (host/test_mirror.cpp); the data plane is the batched
// enqueue / step interface (MultiRaftDriver below).
#pragma once

#include <algorithm>
#include <cstdint>
#include <functional>
#include <map>
#include <memory>
#include <optional>
#include <set>
#include <stdexcept>
#include <string>
#include <tuple>
#include <unordered_map>
#include <utility>
#include <vector>

#include "raftgpu.h"

namespace raft {

constexpr uint64_t INVALID_INDEX = RAFTGPU_INVALID_INDEX;  // raft.rs:81
constexpr uint64_t INVALID_ID = 0;                         // raft.rs:79

// util.rs:118-120
constexpr size_t majority(size_t total) { return total / 2 + 1; }

// state.rs:22-29
enum class ProgressState : uint8_t { Probe = 0, Replicate = 1, Snapshot = 2 };
// quorum.rs:12-20
enum class VoteResult : int { Pending = 0, Lost = 1, Won = 2 };

// errors.rs:17-50: recoverable errors are exceptions derived from Error; what the reference
// `fatal!`s (lib.rs:490-503) is Fatal.
struct Error : std::runtime_error {
    int32_t status;
    Error(int32_t st, const std::string &what) : std::runtime_error(what), status(st) {}
};
struct StepPeerNotFound : Error {  // errors.rs, raised by RawNode::step (raw_node.rs:402-411)
    StepPeerNotFound() : Error(RAFTGPU_ERR_PEER_NOT_FOUND, "raft: cannot step as peer not found") {}
};
struct Fatal : Error {
    using Error::Error;
};

// The HBM arena shared by every tracker of a store.
class Arena {
  public:
    static std::shared_ptr<Arena> create(int device, uint32_t max_groups, uint32_t n_rings = 0) {
        raftgpu_arena *a = nullptr;
        const int32_t rc = raftgpu_arena_create(device, max_groups, RAFTGPU_SLOTS, n_rings, 0, &a);
        if (rc != RAFTGPU_OK) throw Error(rc, std::string("raftgpu_arena_create: ") + raftgpu_strerror(rc));
        return std::shared_ptr<Arena>(new Arena(a));
    }
    ~Arena() {
        if (scratch_ != UINT32_MAX) raftgpu_group_free(a_, scratch_);
        raftgpu_arena_destroy(a_);
    }
    raftgpu_arena *raw() const { return a_; }
    void check(int32_t rc, const char *what) const {
        if (rc == RAFTGPU_OK) return;
        if (rc == RAFTGPU_ERR_PEER_NOT_FOUND) throw StepPeerNotFound();
        const std::string msg = std::string(what) + ": " + raftgpu_strerror(rc) + " (" + raftgpu_last_error(a_) + ")";
        if (rc == RAFTGPU_ERR_COMMIT_RANGE) throw Fatal(rc, msg);
        throw Error(rc, msg);
    }
    // a spare group used to evaluate free-standing quorum functions on the device; more than 8 distinct ids take a
    // wide one (allocated only then: while an arena holds a wide group its steps skip the fused tile kernel)
    uint32_t scratch_group(size_t n_ids = 0) {
        if (n_ids > RAFTGPU_SLOTS) {
            if (scratch_wide_ == UINT32_MAX) check(raftgpu_group_alloc_wide(a_, &scratch_wide_), "group_alloc_wide");
            return scratch_wide_;
        }
        if (scratch_ == UINT32_MAX) check(raftgpu_group_alloc(a_, &scratch_), "group_alloc");
        return scratch_;
    }

  private:
    explicit Arena(raftgpu_arena *a) : a_(a) {}
    raftgpu_arena *a_;
    uint32_t scratch_ = UINT32_MAX, scratch_wide_ = UINT32_MAX;
};

// quorum.rs:35-38
struct Index {
    uint64_t index = 0;
    uint64_t group_id = 0;
};
// quorum.rs:67 `AckIndexer = HashMap<u64, Index>`; quorum.rs:63-65 trait AckedIndexer
using AckIndexer = std::unordered_map<uint64_t, Index>;

namespace detail {
// ids -> peer slots of the scratch group (the reference's voter sets hold at most 7 ids on the
// stack path, majority.rs:79; a joint config unions two of them; more than 8 distinct ids use a wide scratch group: 16 slots)
inline std::map<uint64_t, uint32_t> slot_map(const std::set<uint64_t> &a, const std::set<uint64_t> &b) {
    std::map<uint64_t, uint32_t> m;
    for (const auto *s : {&a, &b})
        for (uint64_t id : *s)
            if (!m.count(id)) {
                if (m.size() >= 2 * RAFTGPU_SLOTS) throw Error(RAFTGPU_ERR_TOO_MANY_PEERS, "more than 16 distinct voters");
                const uint32_t slot = static_cast<uint32_t>(m.size());
                m[id] = slot;
            }
    return m;
}
inline uint32_t mask_of(const std::set<uint64_t> &ids, const std::map<uint64_t, uint32_t> &slots) {
    uint32_t m = 0;
    for (uint64_t id : ids) m |= 1u << slots.at(id);
    return m;
}
}  // namespace detail

// majority.rs:14-16: a set of ids that uses majority quorums to make decisions.
class MajorityConfig {
  public:
    MajorityConfig() = default;
    explicit MajorityConfig(std::set<uint64_t> voters) : voters_(std::move(voters)) {}
    const std::set<uint64_t> &ids() const { return voters_; }                  // majority.rs:46-48
    std::vector<uint64_t> slice() const { return {voters_.begin(), voters_.end()}; }  // :51-55 (sorted)
    bool empty() const { return voters_.empty(); }
    size_t len() const { return voters_.size(); }
    bool contains(uint64_t id) const { return voters_.count(id) != 0; }
    void insert(uint64_t id) { voters_.insert(id); }
    void remove(uint64_t id) { voters_.erase(id); }
    void clear() { voters_.clear(); }
    bool operator==(const MajorityConfig &o) const { return voters_ == o.voters_; }

    // majority.rs:70-124, evaluated by the batched kernel on a scratch group
    std::pair<uint64_t, bool> committed_index(Arena &arena, bool use_group_commit, const AckIndexer &l) const;
    // majority.rs:130-154
    VoteResult vote_result(Arena &arena, const std::function<std::optional<bool>(uint64_t)> &check) const;

  private:
    std::set<uint64_t> voters_;
};

// joint.rs:12-15
class JointConfig {
  public:
    MajorityConfig incoming, outgoing;
    JointConfig() = default;
    explicit JointConfig(std::set<uint64_t> voters) : incoming(std::move(voters)) {}            // joint.rs:19-24
    JointConfig(MajorityConfig in, MajorityConfig out) : incoming(std::move(in)), outgoing(std::move(out)) {}

    // joint.rs:47-51
    std::pair<uint64_t, bool> committed_index(Arena &arena, bool use_group_commit, const AckIndexer &l) const {
        const auto slots = detail::slot_map(incoming.ids(), outgoing.ids());
        const uint32_t g = arena.scratch_group(slots.size());
        raftgpu_arena *a = arena.raw();
        arena.check(raftgpu_group_set_conf(a, g, 0, 0, 0, -1, 1), "group_set_conf");
        arena.check(raftgpu_group_set_conf(a, g, detail::mask_of(incoming.ids(), slots),
                                           detail::mask_of(outgoing.ids(), slots), 0, -1, 1), "group_set_conf");
        arena.check(raftgpu_set_group_commit(a, g, use_group_commit), "set_group_commit");
        for (const auto &[id, slot] : slots) {
            raftgpu_progress p{};
            arena.check(raftgpu_progress_get(a, g, slot, &p), "progress_get");
            const auto it = l.find(id);  // a voter without an entry counts as Index::default(), majority.rs:81
            p.matched = it == l.end() ? 0 : it->second.index;
            p.commit_group_id = it == l.end() ? 0 : it->second.group_id;
            arena.check(raftgpu_progress_set(a, g, slot, &p), "progress_set");
        }
        uint64_t idx = 0;
        int32_t gc = 0;
        arena.check(raftgpu_maximal_committed_index(a, g, &idx, &gc), "maximal_committed_index");
        return {idx, gc != 0};
    }
    // joint.rs:56-67
    VoteResult vote_result(Arena &arena, const std::function<std::optional<bool>(uint64_t)> &check) const {
        const auto slots = detail::slot_map(incoming.ids(), outgoing.ids());
        const uint32_t g = arena.scratch_group(slots.size());
        raftgpu_arena *a = arena.raw();
        arena.check(raftgpu_group_set_conf(a, g, 0, 0, 0, -1, 1), "group_set_conf");
        arena.check(raftgpu_group_set_conf(a, g, detail::mask_of(incoming.ids(), slots),
                                           detail::mask_of(outgoing.ids(), slots), 0, -1, 1), "group_set_conf");
        arena.check(raftgpu_reset_votes(a, g), "reset_votes");
        for (const auto &[id, slot] : slots)
            if (const auto v = check(id)) arena.check(raftgpu_record_vote(a, g, slot, *v ? 1 : 0), "record_vote");
        int32_t r = 0;
        arena.check(raftgpu_vote_result(a, g, &r, nullptr, nullptr), "vote_result");
        return static_cast<VoteResult>(r);
    }
    void clear() {  // joint.rs:70-73
        incoming.clear();
        outgoing.clear();
    }
    bool is_singleton() const { return outgoing.empty() && incoming.len() == 1; }  // joint.rs:77-79
    std::set<uint64_t> ids() const {                                               // joint.rs:82-84 (Union)
        std::set<uint64_t> u = incoming.ids();
        u.insert(outgoing.ids().begin(), outgoing.ids().end());
        return u;
    }
    bool contains(uint64_t id) const { return incoming.contains(id) || outgoing.contains(id); }  // :88-90
};

inline std::pair<uint64_t, bool> MajorityConfig::committed_index(Arena &arena, bool use_group_commit,
                                                                 const AckIndexer &l) const {
    // "joining a majority with the empty majority gives the same result" (datadriven_test.rs:187-192)
    return JointConfig(*this, MajorityConfig()).committed_index(arena, use_group_commit, l);
}
inline VoteResult MajorityConfig::vote_result(Arena &arena,
                                              const std::function<std::optional<bool>(uint64_t)> &check) const {
    return JointConfig(*this, MajorityConfig()).vote_result(arena, check);
}

// progress.rs:8-56 -- a value copy of one peer's Progress (pub fields); `ins` (Inflights) stays
// with the caller, its full() bit travels as ins_full.
struct Progress {
    uint64_t matched = 0;
    uint64_t next_idx = 0;
    ProgressState state = ProgressState::Probe;
    bool paused = false;
    uint64_t pending_snapshot = 0;
    uint64_t pending_request_snapshot = 0;
    bool recent_active = false;
    bool ins_full = false;
    uint64_t commit_group_id = 0;
    uint64_t committed_index = 0;
};

// tracker.rs:37-92
struct Configuration {
    JointConfig voters;
    std::set<uint64_t> learners;
    std::set<uint64_t> learners_next;
    bool auto_leave = false;
};
enum class MapChangeType { Add, Remove };                              // confchange.rs
using MapChange = std::vector<std::pair<uint64_t, MapChangeType>>;

class ProgressTracker;

// `&mut Progress` as handed out by ProgressTracker::get_mut (tracker.rs:273-275): methods run on
// the device cell; direct field pokes go through load() / store().
class ProgressRef {
  public:
    Progress load() const;
    void store(const Progress &p) const;
    bool maybe_update(uint64_t n) const { return op(RAFTGPU_POP_MAYBE_UPDATE, n) != 0; }             // progress.rs:138-150
    bool maybe_decr_to(uint64_t rejected, uint64_t match_hint, uint64_t request_snapshot) const {    // :168-206
        return op(RAFTGPU_POP_MAYBE_DECR_TO, rejected, match_hint, request_snapshot) != 0;
    }
    void update_committed(uint64_t ci) const { op(RAFTGPU_POP_UPDATE_COMMITTED, ci); }               // :153-157
    void optimistic_update(uint64_t n) const { op(RAFTGPU_POP_OPTIMISTIC_UPDATE, n); }               // :160-163
    void become_probe() const { op(RAFTGPU_POP_BECOME_PROBE); }                                      // :95-107
    void become_replicate() const { op(RAFTGPU_POP_BECOME_REPLICATE); }                              // :110-114
    void become_snapshot(uint64_t snapshot_idx) const { op(RAFTGPU_POP_BECOME_SNAPSHOT, snapshot_idx); }  // :117-121
    void snapshot_failure() const { op(RAFTGPU_POP_SNAPSHOT_FAILURE); }                              // :124-127
    bool maybe_snapshot_abort() const { return op(RAFTGPU_POP_MAYBE_SNAPSHOT_ABORT) != 0; }          // :131-134
    bool is_paused() const { return op(RAFTGPU_POP_IS_PAUSED) != 0; }                                // :210-216
    void resume() const { op(RAFTGPU_POP_RESUME); }                                                  // :219-222
    void pause() const { op(RAFTGPU_POP_PAUSE); }                                                    // :225-228
    void update_state(uint64_t last) const {                                                         // :231-243
        if (op(RAFTGPU_POP_UPDATE_STATE, last) < 0) throw Fatal(RAFTGPU_ERR_INVALID, "updating progress state in unhandled state Snapshot");
    }
    void reset(uint64_t next_idx) const { op(RAFTGPU_POP_RESET, next_idx); }                         // :82-92

  private:
    friend class ProgressTracker;
    ProgressRef(Arena *arena, uint32_t group, uint32_t slot) : arena_(arena), group_(group), slot_(slot) {}
    int32_t op(int32_t code, uint64_t a0 = 0, uint64_t a1 = 0, uint64_t a2 = 0) const {
        int32_t r = 0;
        arena_->check(raftgpu_progress_op(arena_->raw(), group_, slot_, code, a0, a1, a2, &r), "progress_op");
        return r;
    }
    Arena *arena_;
    uint32_t group_, slot_;
};

// tracker.rs:195-398
class ProgressTracker {
  public:
    // tracker.rs:211-236 new / with_capacity
    // wide = a group of up to 16 peers (raftgpu_group_alloc_wide: two consecutive group slots); the default holds 8
    ProgressTracker(std::shared_ptr<Arena> arena, size_t max_inflight, bool wide = false)
        : arena_(std::move(arena)), max_inflight_(max_inflight), n_slots_(wide ? 2 * RAFTGPU_SLOTS : RAFTGPU_SLOTS) {
        if (wide)
            arena_->check(raftgpu_group_alloc_wide(arena_->raw(), &group_), "group_alloc_wide");
        else
            arena_->check(raftgpu_group_alloc(arena_->raw(), &group_), "group_alloc");
    }
    ~ProgressTracker() { raftgpu_group_free(arena_->raw(), group_); }
    ProgressTracker(const ProgressTracker &) = delete;
    ProgressTracker &operator=(const ProgressTracker &) = delete;

    void enable_group_commit(bool enable) {  // tracker.rs:238-241
        arena_->check(raftgpu_set_group_commit(arena_->raw(), group_, enable), "set_group_commit");
        group_commit_ = enable;
    }
    bool group_commit() const { return group_commit_; }                  // tracker.rs:243-246
    bool is_singleton() const { return conf_.voters.is_singleton(); }    // tracker.rs:256-258
    const Configuration &conf() const { return conf_; }
    size_t max_inflight() const { return max_inflight_; }
    uint32_t group() const { return group_; }
    // how a RECORD names peer slot `slot` of this group: peers 8..15 of a wide group are the cells of group + 1
    uint32_t record_group(uint32_t slot) const { return group_ + (slot >> 3); }
    static uint8_t record_slot(uint32_t slot) { return static_cast<uint8_t>(slot & 7u); }
    std::optional<uint32_t> slot_of(uint64_t id) const {
        const auto it = slots_.find(id);
        return it == slots_.end() ? std::nullopt : std::optional<uint32_t>(it->second);
    }
    // the peer id that lives in `slot` (0 when the slot is free): for results that name slots
    uint64_t id_of(uint32_t slot) const {
        for (const auto &kv : slots_)
            if (kv.second == slot) return kv.first;
        return 0;
    }
    void set_self(uint64_t id) { self_id_ = id; }

    // tracker.rs:261-275 get / get_mut
    std::optional<Progress> get(uint64_t id) const {
        const auto s = slot_of(id);
        if (!s) return std::nullopt;
        return ProgressRef(arena_.get(), group_, *s).load();
    }
    std::optional<ProgressRef> get_mut(uint64_t id) {
        const auto s = slot_of(id);
        if (!s) return std::nullopt;
        return ProgressRef(arena_.get(), group_, *s);
    }
    // tracker.rs:281-293 iter
    std::vector<std::pair<uint64_t, Progress>> iter() const {
        std::vector<std::pair<uint64_t, Progress>> out;
        for (const auto &[id, slot] : slots_) out.emplace_back(id, ProgressRef(arena_.get(), group_, slot).load());
        return out;
    }

    // tracker.rs:294-298
    std::pair<uint64_t, bool> maximal_committed_index() {
        uint64_t idx = 0;
        int32_t gc = 0;
        arena_->check(raftgpu_maximal_committed_index(arena_->raw(), group_, &idx, &gc), "maximal_committed_index");
        return {idx, gc != 0};
    }

    void reset_votes() {  // tracker.rs:301-303
        arena_->check(raftgpu_reset_votes(arena_->raw(), group_), "reset_votes");
        votes_.clear();
    }
    void record_vote(uint64_t id, bool vote) {  // tracker.rs:307-310: first vote wins
        votes_.emplace(id, vote);
        if (const auto s = slot_of(id)) arena_->check(raftgpu_record_vote(arena_->raw(), group_, *s, vote), "record_vote");
    }
    const std::map<uint64_t, bool> &votes() const { return votes_; }
    // tracker.rs:313-332
    std::tuple<size_t, size_t, VoteResult> tally_votes() {
        int32_t r = 0;
        uint32_t granted = 0, rejected = 0;
        arena_->check(raftgpu_vote_result(arena_->raw(), group_, &r, &granted, &rejected), "vote_result");
        return {granted, rejected, static_cast<VoteResult>(r)};
    }
    // tracker.rs:338-340
    VoteResult vote_result(const std::map<uint64_t, bool> &votes) {
        return conf_.voters.vote_result(*arena_, [&](uint64_t id) -> std::optional<bool> {
            const auto it = votes.find(id);
            return it == votes.end() ? std::nullopt : std::optional<bool>(it->second);
        });
    }
    // tracker.rs:346-361
    bool quorum_recently_active(uint64_t perspective_of) {
        const auto s = slot_of(perspective_of);
        if (!s) throw StepPeerNotFound();
        int32_t r = 0;
        arena_->check(raftgpu_quorum_recently_active(arena_->raw(), group_, *s, &r), "quorum_recently_active");
        return r != 0;
    }
    // tracker.rs:367-372
    bool has_quorum(const std::set<uint64_t> &potential_quorum) {
        uint32_t mask = 0;
        for (uint64_t id : potential_quorum)
            if (const auto s = slot_of(id)) mask |= 1u << *s;
        int32_t r = 0;
        arena_->check(raftgpu_has_quorum(arena_->raw(), group_, mask, &r), "has_quorum");
        return r != 0;
    }

    // tracker.rs:380-397
    void apply_conf(Configuration conf, const MapChange &changes, uint64_t next_idx) {
        for (const auto &[id, ty] : changes) {
            if (ty == MapChangeType::Add) {
                if (slots_.count(id)) continue;
                uint32_t slot = 0;
                while (slot < n_slots_ && used_slots_ & (1u << slot)) slot++;
                if (slot == n_slots_) throw Error(RAFTGPU_ERR_TOO_MANY_PEERS, "more peers than the group has slots (8, or 16 for a wide group)");
                used_slots_ |= 1u << slot;
                slots_[id] = slot;
            } else if (const auto it = slots_.find(id); it != slots_.end()) {
                used_slots_ &= ~(1u << it->second);
                slots_.erase(it);
            }
        }
        auto mask = [&](const std::set<uint64_t> &ids) {
            uint32_t m = 0;
            for (uint64_t id : ids)
                if (const auto s = slot_of(id)) m |= 1u << *s;
            return m;
        };
        const auto self = slot_of(self_id_);
        arena_->check(raftgpu_group_set_conf(arena_->raw(), group_, mask(conf.voters.incoming.ids()),
                                             mask(conf.voters.outgoing.ids()),
                                             mask(conf.learners) | mask(conf.learners_next),
                                             self ? static_cast<int32_t>(*self) : -1, next_idx), "group_set_conf");
        conf_ = std::move(conf);
    }

  private:
    std::shared_ptr<Arena> arena_;
    uint32_t group_ = 0;
    size_t max_inflight_;
    uint32_t n_slots_ = RAFTGPU_SLOTS;
    bool group_commit_ = false;
    uint64_t self_id_ = INVALID_ID;
    Configuration conf_;
    std::map<uint64_t, uint32_t> slots_;  // peer id -> slot
    uint32_t used_slots_ = 0;
    std::map<uint64_t, bool> votes_;
};

inline Progress ProgressRef::load() const {
    raftgpu_progress p{};
    arena_->check(raftgpu_progress_get(arena_->raw(), group_, slot_, &p), "progress_get");
    Progress o;
    o.matched = p.matched;
    o.next_idx = p.next_idx;
    o.state = static_cast<ProgressState>(p.state);
    o.paused = p.paused;
    o.pending_snapshot = p.pending_snapshot;
    o.pending_request_snapshot = p.pending_request_snapshot;
    o.recent_active = p.recent_active;
    o.ins_full = p.ins_full;
    o.commit_group_id = p.commit_group_id;
    o.committed_index = p.committed_index;
    return o;
}
inline void ProgressRef::store(const Progress &o) const {
    raftgpu_progress p{};
    p.matched = o.matched;
    p.next_idx = o.next_idx;
    p.state = static_cast<uint8_t>(o.state);
    p.paused = o.paused;
    p.pending_snapshot = o.pending_snapshot;
    p.pending_request_snapshot = o.pending_request_snapshot;
    p.recent_active = o.recent_active;
    p.ins_full = o.ins_full;
    p.commit_group_id = o.commit_group_id;
    p.committed_index = o.committed_index;
    arena_->check(raftgpu_progress_set(arena_->raw(), group_, slot_, &p), "progress_set");
}

// The slice of RaftLog (raft_log.rs:33-59) and Raft (raft.rs:163-274) on the path, for a leader.
class LeaderLog {
  public:
    LeaderLog(std::shared_ptr<Arena> arena, ProgressTracker &prs) : arena_(std::move(arena)), prs_(prs) {}
    // Raft::reset (raft.rs:942-971) then become_leader (raft.rs:1162-1203)
    void reset(uint64_t last_index, uint64_t committed, uint64_t persisted) {
        arena_->check(raftgpu_group_reset(arena_->raw(), prs_.group(), RAFTGPU_NO_TERM_START, last_index, committed, persisted), "group_reset");
    }
    void become_leader() { arena_->check(raftgpu_group_become_leader(arena_->raw(), prs_.group()), "group_become_leader"); }
    // the log as far as the commit rule needs it: entries of the leader's term are [term_start, last_index]
    void set_log_bounds(uint64_t term_start, uint64_t last_index) {
        arena_->check(raftgpu_group_set_log_bounds(arena_->raw(), prs_.group(), term_start, last_index), "group_set_log_bounds");
    }
    raftgpu_group_state state() const {
        raftgpu_group_state s{};
        arena_->check(raftgpu_group_get(arena_->raw(), prs_.group(), &s), "group_get");
        return s;
    }
    uint64_t committed() const { return state().committed; }  // RaftLog::committed, raft_log.rs:45
    // RaftLog::commit_to, raft_log.rs:286-300 (throws Fatal where the reference fatal!s)
    void commit_to(uint64_t to_commit) { arena_->check(raftgpu_group_commit_to(arena_->raw(), prs_.group(), to_commit), "commit_to"); }
    // RaftLog::maybe_commit(max_index, term == the leader's term), raft_log.rs:487-499
    bool maybe_commit_index(uint64_t max_index) {
        int32_t adv = 0;
        arena_->check(raftgpu_group_maybe_commit_to(arena_->raw(), prs_.group(), max_index, &adv), "maybe_commit_to");
        return adv != 0;
    }
    // Raft::maybe_commit, raft.rs:893-904
    bool maybe_commit() {
        int32_t adv = 0;
        uint64_t committed = 0;
        arena_->check(raftgpu_maybe_commit(arena_->raw(), prs_.group(), &adv, &committed), "maybe_commit");
        return adv != 0;
    }

  private:
    std::shared_ptr<Arena> arena_;
    ProgressTracker &prs_;
};

// The batched data plane: what replaces N x handle_append_response + N x maybe_commit per tick.
class MultiRaftDriver {
  public:
    explicit MultiRaftDriver(std::shared_ptr<Arena> arena) : arena_(std::move(arena)) {}
    // Raft::step(MsgAppendResponse) -> staged (raft.rs:1559-1775); next_probe_index as raft.rs:1560-1661
    void step_append_response(const ProgressTracker &prs, uint64_t from, uint64_t index, uint64_t commit,
                              bool reject = false, uint64_t next_probe_index = 0, uint64_t request_snapshot = INVALID_INDEX,
                              uint32_t ring = 0) {
        const auto slot = prs.slot_of(from);
        if (!slot) throw StepPeerNotFound();  // raw_node.rs:402-411
        raftgpu_append_resp r[2] = {};
        r[0] = {prs.record_group(*slot), prs.record_slot(*slot), static_cast<uint8_t>(reject ? RAFTGPU_REC_REJECT : 0), 0, index, commit};
        r[1] = {prs.record_group(*slot), prs.record_slot(*slot), RAFTGPU_REC_EXT, 0, next_probe_index, request_snapshot};
        arena_->check(raftgpu_enqueue_append_resp(arena_->raw(), ring, r, reject ? 2 : 1), "enqueue_append_resp");
    }
    // append_entry + on_persist_entries of the leader (raft.rs:974-1016)
    void local_progress(const ProgressTracker &prs, uint64_t self_id, uint64_t persisted, uint64_t last_index, uint32_t ring = 0) {
        const auto slot = prs.slot_of(self_id);
        if (!slot) throw StepPeerNotFound();
        const raftgpu_append_resp r{prs.record_group(*slot), prs.record_slot(*slot), RAFTGPU_REC_LOCAL, 0, persisted, last_index};
        arena_->check(raftgpu_enqueue_append_resp(arena_->raw(), ring, &r, 1), "enqueue_append_resp");
    }
    // one batched pass; returns how many groups advanced their commit index
    raftgpu_step_result step(uint32_t flags = RAFTGPU_STEP_READ_COMMITTED) {
        raftgpu_step_result res{};
        arena_->check(raftgpu_step(arena_->raw(), flags, &res), "step");
        return res;
    }
    bool advanced(uint32_t group) const {
        const uint32_t *bm = nullptr;
        const uint64_t *com = nullptr;
        arena_->check(raftgpu_step_results(arena_->raw(), &bm, &com), "step_results");
        return (bm[group >> 5] >> (group & 31)) & 1u;
    }

    // ---- one tick as one call: collect the tick's messages, hand them over together -------------
    // (raftgpu_step_begin_records: the library packs them into the compact stream; the records of
    // one group must be pushed back to back for the fused kernel, which then applies several
    // responses of one peer in arrival order)
    void push_append_response(const ProgressTracker &prs, uint64_t from, uint64_t index, uint64_t commit, bool reject = false,
                              uint64_t next_probe_index = 0, uint64_t request_snapshot = INVALID_INDEX) {
        const auto slot = prs.slot_of(from);
        if (!slot) throw StepPeerNotFound();  // raw_node.rs:402-411
        tick_.push_back({prs.record_group(*slot), prs.record_slot(*slot), static_cast<uint8_t>(reject ? RAFTGPU_REC_REJECT : 0), 0, index, commit});
        if (reject) tick_.push_back({prs.record_group(*slot), prs.record_slot(*slot), RAFTGPU_REC_EXT, 0, next_probe_index, request_snapshot});
    }
    void push_local_progress(const ProgressTracker &prs, uint64_t self_id, uint64_t persisted, uint64_t last_index) {
        const auto slot = prs.slot_of(self_id);
        if (!slot) throw StepPeerNotFound();
        tick_.push_back({prs.record_group(*slot), prs.record_slot(*slot), RAFTGPU_REC_LOCAL, 0, persisted, last_index});
    }
    raftgpu_step_result step_tick(uint32_t flags = RAFTGPU_STEP_READ_COMMITTED) {
        raftgpu_step_result res{};
        arena_->check(raftgpu_step_begin_records(arena_->raw(), tick_.data(), tick_.size(), flags), "step_begin_records");
        tick_.clear();
        arena_->check(raftgpu_step_wait(arena_->raw(), &res), "step_wait");
        return res;
    }
    // bcast_append for the groups whose commit index advanced in the last step (raft.rs:1745-1748,
    // 857-865), minus the paused peers (raft.rs:780-788): the MsgAppends the caller has to build
    std::vector<raftgpu_send_entry> send_list() const {
        std::vector<raftgpu_send_entry> out(64);
        uint64_t n = 0;
        int32_t rc = raftgpu_step_send_list(arena_->raw(), out.data(), out.size(), &n);
        if (rc == RAFTGPU_ERR_FULL) {
            out.resize(n);
            rc = raftgpu_step_send_list(arena_->raw(), out.data(), out.size(), &n);
        }
        arena_->check(rc, "step_send_list");
        out.resize(n);
        return out;
    }

  private:
    std::shared_ptr<Arena> arena_;
    std::vector<raftgpu_append_resp> tick_;
};

}  // namespace raft
