// arena.cu -- host side of the engine: the HBM arena, staging rings, streams and
// the extern "C" surface declared in include/raftgpu.h.
//
// The arena owns every byte of device and pinned memory.  There is no CPU
// compute path: without a CUDA device arena creation fails with
// RAFTGPU_ERR_NO_DEVICE and nothing else can be called.
#include <algorithm>
#include <atomic>
#include <cassert>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <thread>
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include <sched.h>
#if defined(__x86_64__)
#include <immintrin.h>
#endif

#include "kernels.cuh"
#include "pack_compact.h"

using namespace raftgpu;

namespace {

constexpr int kNumSets = 3;        // staging sets: one filling, up to two steps in flight
constexpr uint32_t kChunk = 2048;  // records per staging chunk (48 KiB)
constexpr size_t kScratchBytes = 256;  // d_scratch / h_scratch

// A record moved to a later wave: its packed form (1..4 PackedRec) plus where its result goes.
struct OverflowRec {
    PackedRec pk[4];
    int n_pk;
    uint32_t ring;
    uint64_t seq;  // position of the (main) record in the ring's enqueue order
};

// One caller thread's staging ring: a list of chunks of the set's shared pinned
// buffer.  Only its owner thread touches it between steps.
struct Ring {
    std::vector<uint32_t> chunks;        // chunk indices, in fill order
    uint32_t fill = kChunk;              // records used in the last chunk (kChunk = need a new one)
    uint64_t seq = 0;                    // records enqueued on this ring (wave 0 + overflow)
    std::vector<uint64_t> overflow_seq;  // seq numbers that went to a later wave (ascending)
};

struct StagingSet {
    // host (pinned)
    PackedRec *h_recs = nullptr;      // [n_chunks][kChunk] packed wave-0 records, shared by all rings
    PackedRec *h_overflow = nullptr;  // later waves, laid out at submit time
    uint32_t *h_adv_bitmap = nullptr;
    uint64_t *h_committed = nullptr;
    uint8_t *h_results = nullptr;
    uint32_t *h_step_adv = nullptr;
    // host (pageable)
    std::vector<Ring> rings;
    std::atomic<uint32_t> next_chunk{0};
    uint8_t *touched = nullptr;  // [cap] one bit per peer slot: cell has a record in wave 0
    std::mutex overflow_mu;
    std::unordered_map<uint64_t, uint32_t> overflow_depth;      // cell -> waves used beyond 0
    std::vector<std::vector<OverflowRec>> overflow_waves;       // wave w+1 records
    std::vector<std::pair<uint32_t, uint64_t>> overflow_order;  // (ring, seq | UINT64_MAX for EXT) per packed rec
    // device
    PackedRec *d_recs = nullptr;
    uint32_t *d_adv_bitmap = nullptr;
    uint64_t *d_commit_out = nullptr;
    uint8_t *d_results = nullptr;
    uint32_t *d_tile_off = nullptr;  // [cap / kFTile + 2]: tile index of a tileable compact stream
    uint32_t *d_step_adv = nullptr;  // [0] advanced groups of the step, [1] duplicate records (zero-copy)
    uint32_t *d_touched = nullptr;   // [cap/4] zero-copy steps: one bit per (group, slot)
    // wire steps (grown on demand): the frames and their offsets on the device
    uint8_t *d_wire = nullptr;   // also the device copy of a RAFTGPU_STEP_RAW batch
    uint64_t d_wire_cap = 0;
    uint64_t wire_n = 0;             // frames of the wire step this set carried (0 = not a wire step)
    // sync
    cudaEvent_t ev_h2d = nullptr, ev_compute = nullptr, ev_done = nullptr;
    cudaEvent_t ev_raw0 = nullptr, ev_raw1 = nullptr;  // around the hybrid step's raw H2D copy (timing: the effective PCIe rate)
    uint64_t raw_timed_bytes = 0;                      // bytes of that copy, 0 = nothing to read back
    bool in_flight = false;
    std::atomic<bool> dirty{false};  // touched[] has bits set (set by any enqueueing thread)
    uint32_t flags = 0;
    uint64_t wave0_slots = 0;  // staged wave-0 slots (chunks used * kChunk)
    raftgpu_step_result result{};
    // asynchronous steps (RAFTGPU_STEP_ASYNC): 1 = booked, the submitter thread has not queued it yet;
    // 0 = queued (or not an asynchronous step); < 0 = the submission failed with this status
    std::atomic<int32_t> submit_rc{0};
};

// One raftgpu_step_begin_records in progress (shared by the caller, the staging threads and the submitter).
struct RecJob {
    const raftgpu_append_resp *recs = nullptr;
    uint64_t n = 0;
    uint32_t flags = 0;
    bool async = false, trace = false;
    int T = 1, S = 1;
    StagingSet *set = nullptr;
    uint8_t *buf = nullptr;
    uint64_t cap_bytes = 0, meta_bytes = 0, side_bytes = 0, scratch_units = 0, gb_per_slice = 0;
    uint32_t *stream_units = nullptr;  // the unit stream in the set's pinned buffer
    uint64_t stream_cap_units = 0;
    std::chrono::steady_clock::time_point t_begin;
    std::vector<double> tr_a, tr_b;
    std::atomic<uint64_t> busy_ns{0};  // time the staging threads spent packing this job's slices (for the hybrid split)
    uint64_t raw_n = 0;                // RAFTGPU_STEP_HYBRID: records of the batch that sit in the set's d_wire as they are
    uint32_t raw_min_group = 0;        // ... all of groups >= this one (the packed part ends below it)
    double us_since() const { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t_begin).count(); }
};

// The library's own staging workers (raftgpu_enqueue_bulk, raftgpu_step_begin_records): persistent
// threads, pinned to the GPU-local CPUs.  A step arrives every few hundred microseconds, so a worker
// that has just finished a job SPINS on the generation counter for a while (RAFTGPU_SPIN_US, default
// 2000) before it goes to sleep on the condition variable: waking 32 sleepers through a futex costs
// more than the job itself.  The submitter spins on `pending` likewise.
struct HostPool {
    // One sleeper slot per worker: a worker that has spun long enough sleeps on ITS OWN condition variable.
    // (One shared condition variable makes the wake-up a convoy: the woken threads queue on the one mutex and
    // come back one after the other, each paying its core's idle-state exit.)
    struct alignas(128) Sleeper {
        std::mutex mu;
        std::condition_variable cv;
        bool sleeping = false;
    };
    std::vector<std::thread> threads;
    std::unique_ptr<Sleeper[]> sleepers;
    std::atomic<uint64_t> generation{0};
    std::atomic<int> pending{0};
    std::atomic<bool> stop{false};
    std::function<void(int)> job;
    int spin_us = 2000;

    static inline void cpu_relax() {
#if defined(__x86_64__)
        _mm_pause();
#endif
    }
    void wake_all() {
        for (size_t t = 0; t < threads.size(); t++) {
            Sleeper &sl = sleepers[t];
            std::lock_guard<std::mutex> lk(sl.mu);
            if (sl.sleeping) sl.cv.notify_one();
        }
    }
    // start `fn` on every worker and return at once; wait() blocks until all are done
    void start(const std::function<void(int)> &fn) {
        job = fn;
        pending.store(static_cast<int>(threads.size()));
        generation.fetch_add(1);
        wake_all();
    }
    void wait() {
        uint32_t spins = 0;
        while (pending.load(std::memory_order_acquire) != 0) {
            cpu_relax();
            if ((++spins & 63u) == 0) std::this_thread::yield();  // this thread may sit on a worker's CPU
        }
    }
    void run(const std::function<void(int)> &fn) {
        start(fn);
        wait();
    }
    cpu_set_t pool_cpus;      // RAFTGPU_PIN=set: every worker may run on any CPU of the pool's share
    bool pin_set = false;
    void worker(int idx, int cpu) {
        if (pin_set) {
            sched_setaffinity(0, sizeof(pool_cpus), &pool_cpus);
        } else if (cpu >= 0) {  // one CPU per worker (ensure_pool picks them: GPU-local physical cores first)
            cpu_set_t one;
            CPU_ZERO(&one);
            CPU_SET(cpu, &one);
            sched_setaffinity(0, sizeof(one), &one);
        }
        uint64_t seen = 0;
        for (;;) {
            const auto t_idle = std::chrono::steady_clock::now();
            uint32_t spins = 0;
            while (generation.load(std::memory_order_acquire) == seen && !stop.load(std::memory_order_relaxed)) {
                cpu_relax();
                // a spinning worker owns its CPU as far as the scheduler can tell: give way to whatever else is
                // runnable there (the caller's thread, time-sliced against a spinning worker, loses time on
                // every call)
                if ((++spins & 127u) == 0) sched_yield();
                if ((spins & 255u) == 0 &&
                    std::chrono::steady_clock::now() - t_idle > std::chrono::microseconds(spin_us)) {
                    Sleeper &sl = sleepers[idx];
                    std::unique_lock<std::mutex> lk(sl.mu);
                    sl.sleeping = true;  // start() changes `generation` BEFORE it looks at this flag under the lock
                    sl.cv.wait(lk, [&] { return stop.load() || generation.load() != seen; });
                    sl.sleeping = false;
                    break;
                }
            }
            if (stop.load()) return;
            seen = generation.load(std::memory_order_acquire);
            job(idx);
            pending.fetch_sub(1, std::memory_order_release);
        }
    }
    ~HostPool() {
        stop.store(true);
        wake_all();
        for (auto &t : threads) t.join();
    }
};

// The device scratch of one wire pass: `first`, its first-frame table (allocated on first use and refilled with 0xff by
// every run: no frame yet), and `buf`, a buffer grown on demand (`cap` u64 words) that the pass carves where it runs
// (its abi_*.inc); pass_scratch prepares both.  Never shared between passes (DESIGN 3.10): a wire step may be in flight
// on s_compute while another pass runs on the caller's stream.
struct PassScratch {
    uint32_t *first = nullptr;
    uint64_t *buf = nullptr;
    uint64_t cap = 0;
};
enum Pass {
    kPassWireStep,
    kPassHbWire,
    kPassHbFrames,
    kPassHbFollow,
    kPassVoteWire,
    kPassVoteRequest,
    kPassAppFrames,
    kPassAppFollow,
    kPassFollowTerm,
    kPassLeaderTerm,
    kPassFollowResp,
    kPassLeaderVoteRequest,
    kPassCount
};

}  // namespace

struct raftgpu_arena {
    int device = 0;
    uint32_t cap = 0;
    uint32_t n_rings = 0;
    uint32_t n_chunks = 0;  // chunks in each set's shared staging buffer
    uint64_t overflow_records = 0;
    uint32_t voter_hint = 0;                 // superset of every group's voter slots (recompute_kernel)
    int grid_recompute = 0, grid_recompute5 = 0, grid_apply = 0;  // persistent grid sizes (blocks)
    uint32_t hyb_samples = 0;
    double hyb_pcie_gbs = 0.0;               // RAFTGPU_STEP_HYBRID: measured rate of the raw H2D copies (GB/s), 0 = not measured yet
    double hyb_pack_ns = 0.0;                // RAFTGPU_STEP_HYBRID: measured packing cost (ns per record and staging thread), 0 = not measured yet
    uint32_t n_wide = 0;                     // wide groups (two slots each): the fused tile kernels are not used while any exist
    uint32_t n_simple5 = 0;                  // groups whose meta is the plain 5-voter configuration
    bool force_general = false;              // RAFTGPU_FORCE_GENERAL=1: never take the simple5 kernels
    Columns cols{};
    unsigned long long *d_counters = nullptr;
    void *d_scratch = nullptr;  // kScratchBytes for the small results of single calls (scratch<T>)
    void *h_scratch = nullptr;  // pinned mirror
    cudaStream_t s_compute = nullptr, s_h2d = nullptr, s_d2h = nullptr;
    StagingSet sets[kNumSets];
    int fill = 0;        // set currently being filled by enqueue
    int last_done = -1;  // set whose results raftgpu_step_results exposes
    int inflight[2] = {-1, -1};  // sets submitted by step_begin and not yet waited for, oldest first
    int n_inflight = 0;
    // control plane: single-group calls share the scratch buffers and the meta mirror
    std::mutex ctl_mu;
    // raftgpu_control scratch, kept between calls: per group (pair), the commands staged in the current chunk and
    // its running meta; per command of the chunk, its wave (kCtlSkip = not staged) and, in wave order, its index
    std::vector<uint32_t> ctl_count, ctl_meta, ctl_wave, ctl_order;
    // ReadIndex (raftgpu_arena_enable_read_index): the ack pass's per-group mask of the ring positions its acks named
    // [cap] (zero between passes) and touched-group list [cap]; rq_flag[0] = the request pass's order violation,
    // rq_flag[1] = the touched list's length
    unsigned long long *rq_hit = nullptr;
    uint32_t *rq_list = nullptr, *rq_flag = nullptr;
    // leader runs (raftgpu_arena_enable_leader_runs): the rows [cap], nullptr = off; raftgpu_leader_runs_set's device copy
    // of a list (lr_stage_n rows) and, per group, its position in the list being built (UINT32_MAX = none)
    LeaderRuns *lr_rows = nullptr;
    raftgpu_leader_runs *lr_stage = nullptr;
    uint64_t lr_stage_n = 0;
    std::vector<uint32_t> lr_pos;
    // follower runs (raftgpu_arena_enable_follower_runs): the rows [cap], nullptr = off; their setter shares lr_stage and
    // lr_pos
    LeaderRuns *fr_rows = nullptr;
    // raftgpu_arena_set_wire_waves: frames of a cell (the wire step) or group (the follower's append passes) decided per
    // call, read by each call as it is queued
    uint32_t wire_waves = 1;
    PassScratch pass[kPassCount];  // the wire passes' scratch, one each
    // group allocation
    std::mutex alloc_mu;
    std::vector<uint32_t> free_list;
    std::vector<uint8_t> allocated;
    std::vector<uint32_t> h_meta;  // host mirror of the meta column
    uint32_t hi = 0, n_alloc = 0;
    // info
    int sm_count = 0;
    uint64_t l2_bytes = 0, device_bytes = 0, pinned_bytes = 0;
    std::string last_error;
    std::vector<void *> user_allocs;
    std::vector<void *> host_allocs;  // raftgpu_host_alloc
    HostPool *pool = nullptr;  // created on first raftgpu_enqueue_bulk / raftgpu_step_begin_records
    // raftgpu_step_begin_records scratch, kept between steps (no allocation on the step path)
    std::vector<uint64_t> rec_cut;
    std::vector<PackState> rec_pack;
    std::vector<uint32_t> rec_gbase;
    std::vector<std::atomic<int32_t>> rec_done;
    std::vector<std::atomic<uint64_t>> rec_end;  // where every slice ends in the stream (UINT64_MAX = not packed yet)
    std::vector<uint32_t> rec_scratch;           // one private packing buffer per staging thread
    RecJob rec_job;
    std::atomic<int> rec_next{0};  // next slice to pack
    std::chrono::steady_clock::time_point t_created = std::chrono::steady_clock::now();  // RAFTGPU_TRACE timelines
    // the submitter thread of RAFTGPU_STEP_ASYNC steps
    std::thread sub_thread;
    std::mutex sub_mu;
    std::condition_variable sub_cv;
    bool sub_has_job = false, sub_stop = false;
    std::atomic<int> sub_busy{0};
    cpu_set_t local_cpus;      // GPU-local CPUs (empty when unknown)
    bool have_local_cpus = false;
};

namespace {

thread_local std::string g_create_error;

// Pinned staging must live on the NUMA node the GPU's PCIe root hangs off: DMA reads of
// remote-socket memory cross the inter-socket link and lose H2D bandwidth.  cudaHostAlloc
// places pages by first touch, so the allocating thread is moved onto the GPU-local CPUs
// (sysfs local_cpulist of the device) for the duration of the allocations.
struct LocalCpuGuard {
    cpu_set_t saved;
    cpu_set_t local;  // the GPU-local CPUs we are allowed to run on
    bool active = false;
    explicit LocalCpuGuard(int device) {
        char bus[32] = {0};
        if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) return;
        for (char *p = bus; *p; p++) *p = static_cast<char>(tolower(*p));
        std::string path = std::string("/sys/bus/pci/devices/") + bus + "/local_cpulist";
        FILE *f = fopen(path.c_str(), "r");
        if (!f) return;
        char line[512] = {0};
        const bool ok = fgets(line, sizeof(line), f) != nullptr;
        fclose(f);
        if (!ok) return;
        cpu_set_t want;
        CPU_ZERO(&want);
        int n_set = 0;
        for (char *tok = strtok(line, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
            int lo = 0, hi = 0;
            const int k = sscanf(tok, "%d-%d", &lo, &hi);
            if (k == 1) hi = lo;
            if (k < 1) continue;
            for (int c = lo; c <= hi && c < CPU_SETSIZE; c++) {
                CPU_SET(c, &want);
                n_set++;
            }
        }
        if (!n_set) return;
        if (sched_getaffinity(0, sizeof(saved), &saved) != 0) return;
        cpu_set_t both;
        CPU_AND(&both, &want, &saved);  // stay inside the cpuset we are allowed to use
        if (CPU_COUNT(&both) == 0) return;
        local = both;
        if (sched_setaffinity(0, sizeof(both), &both) == 0) active = true;
    }
    ~LocalCpuGuard() {
        if (active) sched_setaffinity(0, sizeof(saved), &saved);
    }
};

int32_t fail(raftgpu_arena *a, int32_t code, const std::string &msg) {
    if (a) a->last_error = msg;
    return code;
}

#define CK(a, call)                                                                          \
    do {                                                                                     \
        cudaError_t e_ = (call);                                                             \
        if (e_ != cudaSuccess) {                                                             \
            return fail((a), RAFTGPU_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
        }                                                                                    \
    } while (0)

#define CKL(a)                                                                                    \
    do {                                                                                          \
        cudaError_t e_ = cudaGetLastError();                                                      \
        if (e_ != cudaSuccess)                                                                    \
            return fail((a), RAFTGPU_ERR_CUDA, std::string("launch: ") + cudaGetErrorString(e_)); \
    } while (0)

template <typename T>
int32_t dev_alloc(raftgpu_arena *a, T **p, size_t count, bool zero = true) {
    const size_t bytes = count * sizeof(T);
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(p), bytes ? bytes : 1);
    if (e != cudaSuccess)
        return fail(a, e == cudaErrorMemoryAllocation ? RAFTGPU_ERR_NOMEM : RAFTGPU_ERR_CUDA,
                    std::string("cudaMalloc: ") + cudaGetErrorString(e));
    a->device_bytes += bytes;
    if (zero) CK(a, cudaMemset(*p, 0, bytes ? bytes : 1));
    return RAFTGPU_OK;
}

template <typename T>
int32_t pin_alloc(raftgpu_arena *a, T **p, size_t count) {
    const size_t bytes = count * sizeof(T);
    cudaError_t e = cudaHostAlloc(reinterpret_cast<void **>(p), bytes ? bytes : 1, cudaHostAllocDefault);
    if (e != cudaSuccess)
        return fail(a, RAFTGPU_ERR_NOMEM, std::string("cudaHostAlloc: ") + cudaGetErrorString(e));
    a->pinned_bytes += bytes;
    memset(*p, 0, bytes);  // first touch decides the NUMA node
    return RAFTGPU_OK;
}

inline double trace_us(const raftgpu_arena *a) {
    return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - a->t_created).count();
}

inline bool group_ok(const raftgpu_arena *a, uint32_t g) { return g < a->cap && a->allocated[g]; }

// PackedRec slots of a staging set's device record buffer (d_recs): wave 0 + the later waves.  Between steps the
// buffer also stages the other forms' batches and the host calls' (HostFrame, raftgpu_step_send_list).
inline uint64_t rec_slots(const raftgpu_arena *a) { return static_cast<uint64_t>(a->n_chunks) * kChunk + a->overflow_records; }

inline uint32_t present_mask(uint32_t meta) {
    return RAFTGPU_META_IN(meta) | RAFTGPU_META_OUT(meta) | RAFTGPU_META_LEARN(meta);
}
inline uint32_t voter_mask(uint32_t meta) { return RAFTGPU_META_IN(meta) | RAFTGPU_META_OUT(meta); }

inline cudaStream_t pick_stream(raftgpu_arena *a, void *stream) {
    return stream ? static_cast<cudaStream_t>(stream) : a->s_compute;
}

inline uint32_t div_up(uint64_t a, uint32_t b) { return static_cast<uint32_t>((a + b - 1) / b); }

// d_scratch or h_scratch as N values of T, from offset 0 (the rule is at their allocation in raftgpu_arena_create)
template <typename T, size_t N = 1>
T *scratch(void *p) {
    static_assert(sizeof(T) * N <= kScratchBytes, "d_scratch / h_scratch hold kScratchBytes");
    return static_cast<T *>(p);
}

// True when every group of [first, first+n) is the plain 5-voter configuration in slots 0..4
// (no joint half, no group commit): the host's meta mirror is authoritative, so the kernels
// specialised for that case need no per-group check.
inline bool is_simple5(uint32_t meta) {
    return (meta & (0xffffu | RAFTGPU_META_GROUP_COMMIT | RAFTGPU_META_WIDE_LO | RAFTGPU_META_WIDE_HI)) == 0x1fu;
}
inline bool wide_lo(const raftgpu_arena *a, uint32_t g) { return (a->h_meta[g] & RAFTGPU_META_WIDE_LO) != 0; }
inline bool wide_hi(const raftgpu_arena *a, uint32_t g) { return (a->h_meta[g] & RAFTGPU_META_WIDE_HI) != 0; }
// peer slot 0..15 of a wide group -> (half, slot in the half); false = no such slot in this group
inline bool resolve_slot(const raftgpu_arena *a, uint32_t g, uint32_t slot, uint32_t *g2, uint32_t *s2) {
    if (slot < RAFTGPU_SLOTS) {
        *g2 = g;
        *s2 = slot;
        return true;
    }
    if (slot < 2 * RAFTGPU_SLOTS && wide_lo(a, g)) {
        *g2 = g + 1;
        *s2 = slot - RAFTGPU_SLOTS;
        return true;
    }
    return false;
}
inline bool range_simple5(const raftgpu_arena *a, uint32_t first, uint32_t n) {
    return a->n_simple5 == a->hi && static_cast<uint64_t>(first) + n <= a->hi;
}
// RAFTGPU_TILE_DEBUG (read once per process): the fused tile kernels add up the cycles of their phases in the 8
// diagnostic slots behind the counters (raftgpu_debug_read)
inline unsigned long long *tile_dbg(raftgpu_arena *a) {
    static const bool on = getenv("RAFTGPU_TILE_DEBUG") != nullptr;
    return on ? a->d_counters + kCntCount : nullptr;
}

// A fused tile kernel's launch over [0, hi): the simple5 specialisation or the general one, the voter slots its
// stages hold (a superset of every group's), its stage count (tile_stages) for a payload of payload_bytes per stage
// and extra_bytes of other dynamic shared memory, and that dynamic shared memory.  stages == 0 when no slot is
// hinted: the kernels would have nothing to stage.
struct TilePlan {
    bool simple5;
    uint32_t hint;
    int stages;
    size_t smem;
};
TilePlan tile_plan(const raftgpu_arena *a, uint32_t payload_bytes, uint32_t extra_bytes) {
    TilePlan p{};
    p.simple5 = range_simple5(a, 0, a->hi) && !a->force_general;
    p.hint = p.simple5 ? 0x1fu : (a->voter_hint & 0xffu);
    const uint32_t H = static_cast<uint32_t>(__builtin_popcount(p.hint));
    if (H == 0) return p;
    p.stages = tile_stages(H, payload_bytes, extra_bytes);
    p.smem = static_cast<size_t>(p.stages) * tile_stage_bytes(H, payload_bytes) + extra_bytes;
    return p;
}

inline void set_meta(raftgpu_arena *a, uint32_t g, uint32_t meta) {
    a->n_simple5 += static_cast<uint32_t>(is_simple5(meta)) - static_cast<uint32_t>(is_simple5(a->h_meta[g]));
    a->n_wide += ((meta & RAFTGPU_META_WIDE_LO) ? 1u : 0u) - ((a->h_meta[g] & RAFTGPU_META_WIDE_LO) ? 1u : 0u);
    a->h_meta[g] = meta;
    a->voter_hint |= voter_mask(meta);
}

int32_t launch_recompute(raftgpu_arena *a, cudaStream_t st, uint32_t first, uint32_t n, uint32_t hint,
                         uint32_t *d_adv, uint64_t *d_commit, uint64_t *d_mci, uint8_t *d_gc,
                         uint32_t *d_step_adv) {
    if (n == 0) return RAFTGPU_OK;
    const bool simple5 = range_simple5(a, first, n) && !a->force_general;
    if (simple5) hint = 0x1fu;
    const uint32_t base = first & ~31u;
    const uint64_t threads = static_cast<uint64_t>(first - base) + n;
    if (simple5) {
        const uint32_t blocks = std::min<uint32_t>(div_up(threads, 256), static_cast<uint32_t>(a->grid_recompute5));
        recompute_kernel<true><<<blocks, 256, 0, st>>>(a->cols, first, n, hint, d_adv, d_commit, d_mci, d_gc,
                                                      d_step_adv, a->d_counters);
    } else {
        const uint32_t blocks = std::min<uint32_t>(div_up(threads, 256), static_cast<uint32_t>(a->grid_recompute));
        recompute_kernel<false><<<blocks, 256, 0, st>>>(a->cols, first, n, hint, d_adv, d_commit, d_mci, d_gc,
                                                       d_step_adv, a->d_counters);
    }
    CKL(a);
    return RAFTGPU_OK;
}

int32_t launch_apply(raftgpu_arena *a, cudaStream_t st, const void *d_recs, uint64_t n, uint8_t *d_results,
                     bool packed) {
    if (n == 0) return RAFTGPU_OK;
    const uint32_t blocks = std::min<uint32_t>(div_up(n, 256), static_cast<uint32_t>(a->grid_apply));
    if (packed)
        apply_kernel<true><<<blocks, 256, 0, st>>>(a->cols, d_recs, n, d_results, a->d_counters);
    else
        apply_kernel<false><<<blocks, 256, 0, st>>>(a->cols, d_recs, n, d_results, a->d_counters);
    CKL(a);
    return RAFTGPU_OK;
}

// The verified one-wave scatter apply of a batch no host code has looked at: a second record of a cell, or a record of
// a group below min_group, is refused and counted in d_step_adv[1].  Src: const raftgpu_append_resp *, const PackedRec *
// or CompactSrc (n = its units).  clear = false: the second part of a wave whose first part has marked d_touched.
template <typename Src>
int32_t launch_verified_apply(raftgpu_arena *a, StagingSet &s, Src src, uint64_t n, uint8_t *d_results,
                              uint32_t min_group = 0, bool clear = true) {
    using Rec = std::remove_cv_t<std::remove_pointer_t<Src>>;
    if (n == 0) return RAFTGPU_OK;
    if (clear) CK(a, cudaMemsetAsync(s.d_touched, 0, a->cap, a->s_compute));
    const uint32_t blocks = std::min<uint32_t>(div_up(n, 256), static_cast<uint32_t>(a->grid_apply));
    if constexpr (std::is_same_v<Src, CompactSrc>)
        apply_compact_kernel<true><<<blocks, 256, 0, a->s_compute>>>(a->cols, src, d_results, a->d_counters, s.d_touched,
                                                                    s.d_step_adv + 1);
    else
        apply_kernel<std::is_same_v<Rec, PackedRec>, true><<<blocks, 256, 0, a->s_compute>>>(
            a->cols, src, n, d_results, a->d_counters, s.d_touched, s.d_step_adv + 1, min_group);
    CKL(a);
    return RAFTGPU_OK;
}

// A device buffer grown on demand (*ptr, *cap elements of T) holds at least `need`: when it does not, st is synchronised
// (nothing may still read the old buffer), the buffer freed and need + a quarter allocated (a batch that grows slowly
// is not reallocated on every call).
template <typename T>
int32_t grow_scratch(raftgpu_arena *a, cudaStream_t st, T **ptr, uint64_t *cap, uint64_t need) {
    if (*cap >= need) return RAFTGPU_OK;
    CK(a, cudaStreamSynchronize(st));
    CK(a, cudaFree(*ptr));
    *ptr = nullptr;
    *cap = 0;
    const uint64_t want = need + need / 4;
    const int32_t rc = dev_alloc(a, ptr, want, false);
    if (rc != RAFTGPU_OK) return rc;
    *cap = want;
    return RAFTGPU_OK;
}

// d_wire holds at least `need` bytes
int32_t grow_wire(raftgpu_arena *a, StagingSet &s, uint64_t need) {
    return grow_scratch(a, a->s_compute, &s.d_wire, &s.d_wire_cap, need);
}

// A wire pass's first-frame table (`n` u32, allocated on first use) filled with 0xff on st: no frame yet.
int32_t reset_first_frames(raftgpu_arena *a, cudaStream_t st, uint32_t **table, size_t n) {
    if (!*table) {
        const int32_t rc = dev_alloc(a, table, n, false);
        if (rc != RAFTGPU_OK) return rc;
    }
    CK(a, cudaMemsetAsync(*table, 0xff, n * sizeof(uint32_t), st));
    return RAFTGPU_OK;
}

// What a wire pass does before its first launch on st: its first-frame table of first_n u32 reset (0: the pass keeps
// none), its buffer holding at least `words` u64.
int32_t pass_scratch(raftgpu_arena *a, cudaStream_t st, PassScratch &p, size_t first_n, uint64_t words) {
    if (first_n) {
        const int32_t rc = reset_first_frames(a, st, &p.first, first_n);
        if (rc != RAFTGPU_OK) return rc;
    }
    return grow_scratch(a, st, &p.buf, &p.cap, words);
}

// The limits of every wire batch: frame offsets and counts are u32 on the device, and the staging kernels read the
// bytes with 16-byte loads (d_bytes = nullptr: not checked here, for a form that copies the bytes to d_wire itself).
int32_t wire_batch_check(raftgpu_arena *a, uint64_t n_bytes, uint64_t n, const void *d_bytes) {
    if (n > 0xfffffff0ull || n_bytes > 0xfffffff0ull) return fail(a, RAFTGPU_ERR_INVALID, "wire batch larger than 4 GiB");
    if (reinterpret_cast<uintptr_t>(d_bytes) & 15u) return fail(a, RAFTGPU_ERR_INVALID, "wire bytes must be 16-byte aligned");
    return RAFTGPU_OK;
}

void free_set(StagingSet &s) {
    cudaFreeHost(s.h_recs);
    cudaFreeHost(s.h_overflow);
    cudaFreeHost(s.h_adv_bitmap);
    cudaFreeHost(s.h_committed);
    cudaFreeHost(s.h_results);
    cudaFreeHost(s.h_step_adv);
    free(s.touched);
    cudaFree(s.d_recs);
    cudaFree(s.d_adv_bitmap);
    cudaFree(s.d_commit_out);
    cudaFree(s.d_results);
    cudaFree(s.d_tile_off);
    cudaFree(s.d_step_adv);
    cudaFree(s.d_touched);
    cudaFree(s.d_wire);
    if (s.ev_h2d) cudaEventDestroy(s.ev_h2d);
    if (s.ev_raw0) cudaEventDestroy(s.ev_raw0);
    if (s.ev_raw1) cudaEventDestroy(s.ev_raw1);
    if (s.ev_compute) cudaEventDestroy(s.ev_compute);
    if (s.ev_done) cudaEventDestroy(s.ev_done);
}

void destroy(raftgpu_arena *a) {
    if (!a) return;
    if (a->sub_thread.joinable()) {
        {
            std::lock_guard<std::mutex> lk(a->sub_mu);
            a->sub_stop = true;
        }
        a->sub_cv.notify_one();
        a->sub_thread.join();
    }
    cudaSetDevice(a->device);
    cudaDeviceSynchronize();
    Columns &c = a->cols;
    cudaFree(c.matched);
    cudaFree(c.next_d);
    cudaFree(c.pc_d);
    cudaFree(c.next_idx);
    cudaFree(c.peer_committed);
    cudaFree(c.pending_snapshot);
    cudaFree(c.pending_req_snapshot);
    cudaFree(c.commit_group_id);
    cudaFree(c.pflags);
    cudaFree(c.votes);
    cudaFree(c.meta);
    cudaFree(c.committed);
    cudaFree(c.term_start);
    cudaFree(c.last_index);
    cudaFree(c.term);
    cudaFree(c.ins_meta);
    cudaFree(c.ins_buf);
    cudaFree(c.rq_hc);
    cudaFree(c.rq_ctx);
    cudaFree(c.rq_index);
    cudaFree(c.rq_acks);
    cudaFree(a->rq_hit);
    cudaFree(a->rq_list);
    cudaFree(a->rq_flag);
    cudaFree(a->lr_rows);
    cudaFree(a->lr_stage);
    cudaFree(a->fr_rows);
    for (PassScratch &p : a->pass) {
        cudaFree(p.first);
        cudaFree(p.buf);
    }
    cudaFree(a->d_counters);
    cudaFree(a->d_scratch);
    cudaFreeHost(a->h_scratch);
    for (void *p : a->user_allocs) cudaFree(p);
    for (void *p : a->host_allocs) cudaFreeHost(p);
    delete a->pool;
    for (auto &s : a->sets) free_set(s);
    if (a->s_compute) cudaStreamDestroy(a->s_compute);
    if (a->s_h2d) cudaStreamDestroy(a->s_h2d);
    if (a->s_d2h) cudaStreamDestroy(a->s_d2h);
    delete a;
}

int32_t create(int32_t device, uint32_t max_groups, uint32_t slots, uint32_t n_rings,
               uint32_t ring_records, raftgpu_arena **out) {
    if (!out || max_groups == 0) return RAFTGPU_ERR_INVALID;
    if (slots != RAFTGPU_SLOTS) return RAFTGPU_ERR_TOO_MANY_PEERS;  // the documented hard limit (raftgpu.h)
    *out = nullptr;
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
        cudaGetLastError();
        return RAFTGPU_ERR_NO_DEVICE;
    }
    if (device < 0 || device >= n_dev) return RAFTGPU_ERR_INVALID;
    raftgpu_arena *a = new (std::nothrow) raftgpu_arena();
    if (!a) return RAFTGPU_ERR_NOMEM;
    a->device = device;
    // pad the column stride so every column (and every slot row of it) is 128-byte aligned
    a->cap = (max_groups + 127u) & ~127u;
    a->n_rings = n_rings ? n_rings : 16;
    // staging capacity per step, shared by all rings: ring_records * n_rings when given, else
    // ~5 records per group (a full round of a 5-peer deployment is ~3.5); plus one partially
    // filled chunk per ring
    const uint64_t want = ring_records ? static_cast<uint64_t>(ring_records) * a->n_rings
                                       : std::max<uint64_t>(4096, 5ull * a->cap);
    a->n_chunks = div_up(want, kChunk) + a->n_rings;
    a->overflow_records = std::max<uint64_t>(4096, a->cap / 4);
    int32_t rc = RAFTGPU_OK;
    auto bail = [&](int32_t code) {
        g_create_error = a->last_error;
        destroy(a);
        return code;
    };
#define TRY(x)                                 \
    do {                                       \
        rc = (x);                              \
        if (rc != RAFTGPU_OK) return bail(rc); \
    } while (0)
#define TRYC(call)                                                              \
    do {                                                                        \
        cudaError_t e_ = (call);                                                \
        if (e_ != cudaSuccess) {                                                \
            a->last_error = std::string(#call) + ": " + cudaGetErrorString(e_); \
            return bail(RAFTGPU_ERR_CUDA);                                      \
        }                                                                       \
    } while (0)
    TRYC(cudaSetDevice(device));
    cudaDeviceProp prop{};
    TRYC(cudaGetDeviceProperties(&prop, device));
    a->sm_count = prop.multiProcessorCount;
    a->l2_bytes = static_cast<uint64_t>(prop.l2CacheSize);
    int occ = 0;
    TRYC(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, recompute_kernel<false>, 256, 0));
    a->grid_recompute = std::max(1, occ) * a->sm_count;
    TRYC(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, recompute_kernel<true>, 256, 0));
    a->grid_recompute5 = std::max(1, occ) * a->sm_count;
    TRYC(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, apply_kernel<true>, 256, 0));
    a->grid_apply = std::max(1, occ) * a->sm_count;
    const int tile_smem = static_cast<int>(kFSmem);
    TRYC(cudaFuncSetAttribute(step_tile_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, tile_smem));
    TRYC(cudaFuncSetAttribute(step_tile_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tile_smem));
    TRYC(cudaFuncSetAttribute(step_tile_compact_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, tile_smem));
    TRYC(cudaFuncSetAttribute(step_tile_compact_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, tile_smem));
    TRYC(cudaFuncSetAttribute(step_tile_compact_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tile_smem));
    TRYC(cudaFuncSetAttribute(step_tile_compact_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tile_smem));
    TRYC(cudaFuncSetAttribute(bcast_write_kernel<HbBcast>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              static_cast<int>(kBcastSmem<HbBcast>)));
    TRYC(cudaFuncSetAttribute(bcast_write_kernel<AppBcast>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              static_cast<int>(kBcastSmem<AppBcast>)));
    {
        const char *f = getenv("RAFTGPU_FORCE_GENERAL");
        a->force_general = f && f[0] == '1';
    }
    TRYC(cudaStreamCreateWithFlags(&a->s_compute, cudaStreamNonBlocking));
    TRYC(cudaStreamCreateWithFlags(&a->s_h2d, cudaStreamNonBlocking));
    TRYC(cudaStreamCreateWithFlags(&a->s_d2h, cudaStreamNonBlocking));

    const size_t cells = static_cast<size_t>(kSlots) * a->cap;
    Columns &c = a->cols;
    c.cap = a->cap;
    TRY(dev_alloc(a, &c.matched, cells));
    TRY(dev_alloc(a, &c.next_d, cells));  // zero offsets: next_idx = peer_committed = matched = 0
    TRY(dev_alloc(a, &c.pc_d, cells));
    TRY(dev_alloc(a, &c.next_idx, cells));
    TRY(dev_alloc(a, &c.peer_committed, cells));
    TRY(dev_alloc(a, &c.pending_snapshot, cells));
    TRY(dev_alloc(a, &c.pending_req_snapshot, cells));
    TRY(dev_alloc(a, &c.commit_group_id, cells));
    TRY(dev_alloc(a, &c.pflags, cells));
    TRY(dev_alloc(a, &c.votes, cells));
    TRY(dev_alloc(a, &c.meta, a->cap));
    TRY(dev_alloc(a, &c.committed, a->cap));
    TRY(dev_alloc(a, &c.term_start, a->cap));
    TRY(dev_alloc(a, &c.last_index, a->cap));
    TRY(dev_alloc(a, &c.term, a->cap));
    TRYC(cudaMemset(c.term_start, 0xff, sizeof(uint64_t) * a->cap));  // RAFTGPU_NO_TERM_START
    TRY(dev_alloc(a, &a->d_counters, kCntCount + 8));  // + 8 diagnostic slots (fused kernel phase cycles)
    // d_scratch / h_scratch: every user sees them as its own type at offset 0 (scratch<T>), because no two users are
    // ever live at once: each holds ctl_mu and synchronises s_compute before it returns, and no step kernel touches
    // d_scratch.
    TRY(dev_alloc(a, reinterpret_cast<uint8_t **>(&a->d_scratch), kScratchBytes));
    TRY(pin_alloc(a, reinterpret_cast<uint8_t **>(&a->h_scratch), kScratchBytes));

    const uint64_t wave0_total = static_cast<uint64_t>(a->n_chunks) * kChunk;
    const uint64_t rec_total = rec_slots(a);
    LocalCpuGuard numa_guard(device);  // pinned pages on the GPU-local NUMA node
    CPU_ZERO(&a->local_cpus);
    if (numa_guard.active) {
        a->local_cpus = numa_guard.local;
        a->have_local_cpus = true;
    }
    for (auto &s : a->sets) {
        TRY(pin_alloc(a, &s.h_recs, wave0_total));
        TRY(pin_alloc(a, &s.h_overflow, a->overflow_records));
        TRY(pin_alloc(a, &s.h_adv_bitmap, a->cap / 32));
        TRY(pin_alloc(a, &s.h_committed, a->cap));
        TRY(pin_alloc(a, &s.h_results, 4 * rec_total));  // one byte per slot; a compact stream has 4-byte units
        TRY(pin_alloc(a, &s.h_step_adv, 4));
        s.rings.assign(a->n_rings, Ring());
        s.touched = static_cast<uint8_t *>(calloc(a->cap, 1));
        if (!s.touched) return bail(RAFTGPU_ERR_NOMEM);
        TRY(dev_alloc(a, &s.d_recs, rec_total, false));
        TRY(dev_alloc(a, &s.d_adv_bitmap, a->cap / 32));
        TRY(dev_alloc(a, &s.d_commit_out, a->cap));
        TRY(dev_alloc(a, &s.d_results, 4 * rec_total));
        TRY(dev_alloc(a, &s.d_tile_off, 3 * (a->cap / kFTile + 2) + 2));
        TRY(dev_alloc(a, &s.d_step_adv, 4));
        TRY(dev_alloc(a, &s.d_touched, a->cap / 4));
        TRYC(cudaEventCreateWithFlags(&s.ev_h2d, cudaEventDisableTiming));
        TRYC(cudaEventCreate(&s.ev_raw0));
        TRYC(cudaEventCreate(&s.ev_raw1));
        TRYC(cudaEventCreateWithFlags(&s.ev_compute, cudaEventDisableTiming));
        TRYC(cudaEventCreateWithFlags(&s.ev_done, cudaEventDisableTiming));
    }
    a->allocated.assign(a->cap, 0);
    a->h_meta.assign(a->cap, 0);
    TRYC(cudaDeviceSynchronize());
#undef TRY
#undef TRYC
    *out = a;
    return RAFTGPU_OK;
}

// Control-plane kernel(s) + sync on the compute stream.
template <typename F>
int32_t sync_op(raftgpu_arena *a, F &&launch) {
    CK(a, cudaSetDevice(a->device));
    launch(a->s_compute);
    CKL(a);
    CK(a, cudaStreamSynchronize(a->s_compute));
    return RAFTGPU_OK;
}

// ReadIndex queues (arenas with raftgpu_arena_enable_read_index only): groups [first, first + n) become allocated with
// an empty queue (value = kRqAlloc) or free (0).
int32_t read_mark(raftgpu_arena *a, uint32_t first, uint32_t n, uint32_t value) {
    if (!a->cols.rq_cap || n == 0) return RAFTGPU_OK;
    const uint32_t blocks = std::min<uint32_t>(div_up(n, 256), 8u * static_cast<uint32_t>(a->sm_count));
    return sync_op(a, [&](cudaStream_t st) { read_mark_kernel<<<blocks, 256, 0, st>>>(a->cols.rq_hc, first, n, value); });
}

// Leader and follower runs (arenas with raftgpu_arena_enable_leader_runs / _follower_runs only): the rows of groups
// [first, first + n) are cleared, so that a slot that is allocated or freed matches no anchor.
int32_t runs_clear(raftgpu_arena *a, uint32_t first, uint32_t n) {
    if ((!a->lr_rows && !a->fr_rows) || n == 0) return RAFTGPU_OK;
    CK(a, cudaSetDevice(a->device));
    if (a->lr_rows) CK(a, cudaMemsetAsync(a->lr_rows + first, 0, sizeof(LeaderRuns) * n, a->s_compute));
    if (a->fr_rows) CK(a, cudaMemsetAsync(a->fr_rows + first, 0, sizeof(LeaderRuns) * n, a->s_compute));
    CK(a, cudaStreamSynchronize(a->s_compute));
    return RAFTGPU_OK;
}

struct ColumnDesc {
    void *base;
    size_t elem;
    bool per_peer;
};

bool column_desc(raftgpu_arena *a, int32_t col, ColumnDesc *d) {
    Columns &c = a->cols;
    switch (col) {
    case RAFTGPU_COL_MATCHED: *d = {c.matched, 8, true}; return true;
    case RAFTGPU_COL_NEXT_IDX: *d = {c.next_idx, 8, true}; return true;
    case RAFTGPU_COL_PEER_COMMITTED: *d = {c.peer_committed, 8, true}; return true;
    case RAFTGPU_COL_PENDING_SNAPSHOT: *d = {c.pending_snapshot, 8, true}; return true;
    case RAFTGPU_COL_PENDING_REQ_SNAPSHOT: *d = {c.pending_req_snapshot, 8, true}; return true;
    case RAFTGPU_COL_COMMIT_GROUP_ID: *d = {c.commit_group_id, 8, true}; return true;
    case RAFTGPU_COL_PFLAGS: *d = {c.pflags, 1, true}; return true;
    case RAFTGPU_COL_VOTES: *d = {c.votes, 1, true}; return true;
    case RAFTGPU_COL_META: *d = {c.meta, 4, false}; return true;
    case RAFTGPU_COL_COMMITTED: *d = {c.committed, 8, false}; return true;
    case RAFTGPU_COL_TERM_START: *d = {c.term_start, 8, false}; return true;
    case RAFTGPU_COL_LAST_INDEX: *d = {c.last_index, 8, false}; return true;
    case RAFTGPU_COL_TERM: *d = {c.term, 8, false}; return true;
    case RAFTGPU_COL_INS_META:
        if (!c.ins_cap) return false;
        *d = {c.ins_meta, 4, true};
        return true;
    default: return false;
    }
}

// next_idx and peer_committed are offsets from matched on the device (k_common.cuh), so their column IO goes through
// the u64 escape columns: decode = materialize the values of cells [slot * cap + first, + n) there, encode = turn the
// values there into offsets.  `column` is RAFTGPU_COL_NEXT_IDX, _PEER_COMMITTED, or _MATCHED for both.
int32_t offset_column_io(raftgpu_arena *a, int32_t column, uint32_t slot, uint32_t first, uint32_t n, bool encode) {
    Columns &c = a->cols;
    const size_t cell0 = static_cast<size_t>(slot) * a->cap + first;
    const int grid = static_cast<int>(std::max<uint64_t>(1, std::min<uint64_t>(8ull * a->sm_count, (n + 255u) / 256u)));
    if (column != RAFTGPU_COL_PEER_COMMITTED)
        offset_column_kernel<<<grid, 256, 0, a->s_compute>>>(c.matched, c.next_d, c.next_idx, cell0, n, encode);
    if (column != RAFTGPU_COL_NEXT_IDX)
        offset_column_kernel<<<grid, 256, 0, a->s_compute>>>(c.matched, c.pc_d, c.peer_committed, cell0, n, encode);
    CKL(a);
    return RAFTGPU_OK;
}

// Move a duplicate-cell record (already packed) to a later wave.
void push_overflow(StagingSet &s, uint64_t cell, const PackedRec *pk, int n_pk, uint32_t ring, uint64_t seq) {
    std::lock_guard<std::mutex> lk(s.overflow_mu);
    const uint32_t depth = s.overflow_depth[cell]++;  // 0 -> wave 1
    if (s.overflow_waves.size() <= depth) s.overflow_waves.resize(depth + 1);
    OverflowRec o{};
    for (int k = 0; k < n_pk; k++) o.pk[k] = pk[k];
    o.n_pk = n_pk;
    o.ring = ring;
    o.seq = seq;
    s.overflow_waves[depth].push_back(o);
}

// make a finished set reusable for filling
int32_t reclaim_set(raftgpu_arena *a, StagingSet &s) {
    if (s.in_flight) return RAFTGPU_ERR_BUSY;
    if (s.dirty.load(std::memory_order_relaxed)) {
        memset(s.touched, 0, a->cap);
        s.dirty.store(false, std::memory_order_relaxed);
    }
    for (auto &r : s.rings) {
        r.chunks.clear();
        r.fill = kChunk;
        r.seq = 0;
        r.overflow_seq.clear();
    }
    s.next_chunk.store(0);
    s.wire_n = 0;
    s.overflow_depth.clear();
    s.overflow_waves.clear();
    s.overflow_order.clear();  // (raftgpu_step_record_results: only a step with later waves has any)
    return RAFTGPU_OK;
}

// host batch -> device scratch (the fill set's record staging, idle between steps) -> kernel -> results
// every entry point that queues work or touches the staging sets first lets a pending asynchronous submission finish
void wait_submitter(raftgpu_arena *a) {
    uint32_t spins = 0;
    while (a->sub_busy.load(std::memory_order_acquire) != 0) {
        HostPool::cpu_relax();
        if ((++spins & 63u) == 0) std::this_thread::yield();
    }
}

// The admission rule of every host batch call: the fill set's staging is idle (no records enqueued for a step).
int32_t host_batch_admit(raftgpu_arena *a, StagingSet **out) {
    wait_submitter(a);
    StagingSet &s = a->sets[a->fill];
    if (s.in_flight || s.next_chunk.load() != 0) return fail(a, RAFTGPU_ERR_BUSY, "records are staged for a step: step first");
    *out = &s;
    return RAFTGPU_OK;
}

// ---- the host frame: every host form of a batch pass (raftgpu_heartbeat_resp, raftgpu_update_state, the three
// raftgpu_read_index_* passes, raftgpu_heartbeat_wire, raftgpu_heartbeat_frames, raftgpu_follower_heartbeat,
// raftgpu_vote_wire, raftgpu_vote_request_wire, raftgpu_append_frames) stages its host buffers in the fill set, idle between steps, runs its `_device` form on s_compute
// and copies the outputs back through one HostFrame:
//   open   admission (host_batch_admit), and the record batch if the form has one: the batch goes to d_recs and one
//          result byte per item to d_results, so it is refused with ERR_FULL past their room;
//   in     a region of d_wire copied from a host buffer; out: a region only reserved; rest: the last region, which
//          takes what d_wire has room for (at least `min` bytes) until enlarge gives it an exact size;
//   run    d_wire grown to hold the regions, the H2D copies (the batch, then the inputs in order), then the pass;
//   back   a D2H copy from d_results, d_wire or the arena's scratch (where the counts go, scratch<T>);
//   wait   the synchronise of s_compute that ends a phase, when the frame queued anything since the last one.
// A null host pointer or a zero length copies nothing.  Regions are offsets: only the pass sees device pointers into
// d_wire, made after the growth that may move it.  The regions start on 16-byte boundaries.
struct WireRegion {
    uint64_t at;
};

// What a frame's pass sees: the batch, the result bytes, d_wire as it is after the growth and the rest region's bytes.
struct Staged {
    const void *recs;
    uint8_t *results;
    uint8_t *wire;
    uint64_t rest;
    template <typename T>
    T *at(WireRegion r) const {
        return reinterpret_cast<T *>(wire + r.at);
    }
};

class HostFrame {
  public:
    explicit HostFrame(raftgpu_arena *a) : a_(a) {}

    int32_t open(const void *recs = nullptr, uint64_t n = 0, size_t elem = 0) {
        const int32_t rc = host_batch_admit(a_, &s_);
        if (rc != RAFTGPU_OK) return rc;
        if (n * elem > rec_slots(a_) * sizeof(PackedRec) || n > 4 * rec_slots(a_))
            return fail(a_, RAFTGPU_ERR_FULL, "batch larger than the staging buffer");
        recs_ = recs;
        rec_bytes_ = n * elem;
        CK(a_, cudaSetDevice(a_->device));
        return RAFTGPU_OK;
    }

    WireRegion in(const void *src, uint64_t bytes) {
        const WireRegion r = take(bytes);
        assert(n_in_ < kInputs);
        in_[n_in_++] = {r.at, src, bytes};
        return r;
    }
    WireRegion out(uint64_t bytes) { return take(bytes); }
    WireRegion rest(uint64_t min) {
        rest_ = take(min);
        return rest_;
    }
    void enlarge(uint64_t bytes) {
        end_ = rest_.at + bytes;
        rest_bytes_ = bytes;
    }

    template <typename Pass>
    int32_t run(Pass &&pass) {
        StagingSet &s = *s_;
        int32_t rc = grow_wire(a_, s, end_);
        if (rc != RAFTGPU_OK) return rc;
        if (recs_ && rec_bytes_) CK(a_, cudaMemcpyAsync(s.d_recs, recs_, rec_bytes_, cudaMemcpyHostToDevice, a_->s_compute));
        for (uint32_t i = 0; i < n_in_; i++)
            if (in_[i].src && in_[i].bytes)
                CK(a_, cudaMemcpyAsync(s.d_wire + in_[i].at, in_[i].src, in_[i].bytes, cudaMemcpyHostToDevice, a_->s_compute));
        queued_ = true;
        const Staged d{s.d_recs, s.d_results, s.d_wire, std::min(rest_bytes_, s.d_wire_cap - rest_.at)};
        return pass(d);
    }

    const uint8_t *results() const { return s_->d_results; }
    int32_t back(void *dst, const void *d_src, uint64_t bytes) {
        if (!dst || !bytes) return RAFTGPU_OK;
        CK(a_, cudaMemcpyAsync(dst, d_src, bytes, cudaMemcpyDeviceToHost, a_->s_compute));
        queued_ = true;
        return RAFTGPU_OK;
    }
    int32_t back(void *dst, WireRegion src, uint64_t bytes) { return back(dst, s_->d_wire + src.at, bytes); }

    int32_t wait() {
        if (!queued_) return RAFTGPU_OK;
        queued_ = false;
        CK(a_, cudaStreamSynchronize(a_->s_compute));
        return RAFTGPU_OK;
    }

  private:
    static constexpr uint32_t kInputs = 4;
    struct Input {
        uint64_t at;
        const void *src;
        uint64_t bytes;
    };
    WireRegion take(uint64_t bytes) {
        const uint64_t at = (end_ + 15u) & ~15ull;
        end_ = at + bytes;
        return {at};
    }

    raftgpu_arena *a_;
    StagingSet *s_ = nullptr;
    const void *recs_ = nullptr;
    uint64_t rec_bytes_ = 0;
    Input in_[kInputs] = {};
    uint32_t n_in_ = 0;
    uint64_t end_ = 0;               // where the last region ends: what d_wire must hold
    WireRegion rest_ = {0};
    uint64_t rest_bytes_ = UINT64_MAX;  // the rest region's size once enlarged (until then: to the end of d_wire)
    bool queued_ = false;               // copies or a pass queued since the last wait
};

// ---- the reply pipeline (DESIGN 3.12): a pass that answers every frame it applies with a frame of its own
// (raftgpu_follower_heartbeat, raftgpu_vote_request_wire, raftgpu_follower_term_wire's and raftgpu_leader_term_wire's stale replies) keeps its decision -- a scan and an apply kernel -- and
// shares the rest: reply_check, reply_run<P> for the `_device` form, reply_host for the host form.  P is the pass's
// reply policy (reply_write_kernel, k_wire.cuh).

// The refusals both forms make before any copy or launch; bound_name: the pass's public bound function, n * frame_max.
int32_t reply_check(raftgpu_arena *a, uint64_t n_bytes, uint64_t n, uint64_t frame_max, uint64_t resp_bytes_capacity,
                    const char *bound_name) {
    const int32_t rc = wire_batch_check(a, n_bytes, n, nullptr);  // (the device form checks the alignment after)
    if (rc != RAFTGPU_OK) return rc;
    if (n * frame_max > 0xffffffffull)
        return fail(a, RAFTGPU_ERR_INVALID, "the responses of this batch may not be addressable by u32 offsets");
    // the pass changes the groups it answers for: a response that did not fit could not be produced again
    if (resp_bytes_capacity < n * frame_max)
        return fail(a, RAFTGPU_ERR_INVALID, std::string("response capacity below ") + bound_name + "(n)");
    return RAFTGPU_OK;
}

// The `_device` form after its checks, on st: no frame gives zero totals and resp_offsets[0] = 0.  Otherwise the
// pass's scratch (u64 words) is carved into one record per frame and the {responses, bytes} of every block, its
// first-frame table (first_n u32) reset, and four passes run with kWireThreads frames per block: passes(blocks, recs,
// first, blk) launches the pass's scan and apply kernels, block_starts_kernel<2> turns the block sums into block starts,
// the totals and the last offset, reply_write_kernel<P> writes the responses.  extra_words: u64 words behind blk that
// the pass uses as it likes (the follower's wave lists); the passes' launch errors, and those of anything else they
// queue, are reported after the last launch.
template <class P, typename Passes>
int32_t reply_run(raftgpu_arena *a, cudaStream_t st, PassScratch &scratch, uint64_t n, const uint8_t *d_status,
                  uint8_t *d_resp_bytes, uint32_t *d_resp_offsets, uint64_t *d_totals, size_t first_n, Passes &&passes,
                  uint64_t extra_words = 0) {
    using Rec = typename P::Rec;
    if (n == 0) {
        CK(a, cudaMemsetAsync(d_totals, 0, 16, st));
        CK(a, cudaMemsetAsync(d_resp_offsets, 0, 4, st));
        return RAFTGPU_OK;
    }
    const uint32_t nb = div_up(n, kWireThreads);
    const int32_t rc = pass_scratch(a, st, scratch, first_n, (sizeof(Rec) / 8) * n + nb + extra_words);
    if (rc != RAFTGPU_OK) return rc;
    Rec *recs = reinterpret_cast<Rec *>(scratch.buf);
    uint32_t *blk = reinterpret_cast<uint32_t *>(scratch.buf + (sizeof(Rec) / 8) * n);
    passes(nb, recs, scratch.first, blk);
    // (the capacities always hold: resp_bytes_capacity >= P::kFrameMax * n was checked, d_resp_offsets has n + 1 values)
    block_starts_kernel<2><<<1, kScanThreads, 0, st>>>(blk, nb, d_totals, d_resp_offsets);
    reply_write_kernel<P><<<nb, kWireThreads, 0, st>>>(static_cast<uint32_t>(n), d_status, recs, blk, d_resp_bytes, d_resp_offsets);
    CKL(a);
    return RAFTGPU_OK;
}

// What reply_host hands the `_device` form: the staged batch and tables, the outputs' places in d_wire, the totals' in
// the arena's scratch.
struct ReplyStaged {
    const uint8_t *bytes;
    const uint32_t *offsets;
    const void *table[2];
    uint8_t *status;
    uint64_t *out;  // nullptr when the caller passed none
    uint8_t *resp_bytes;
    uint32_t *resp_offsets;
    uint64_t *totals;
};
struct ReplyTable {
    const void *src;
    uint64_t bytes;
};

// The host form after its checks (HostFrame): d_wire holds [bytes | offsets | the pass's tables | status | out, out_width
// bytes per frame | response offsets | response bytes, `bound`], the totals go to the arena's scratch.  The totals,
// status and out come back, then the responses the totals give.
template <typename Device>
int32_t reply_host(raftgpu_arena *a, const void *bytes, uint64_t n_bytes, const uint32_t *offsets, uint64_t n,
                   const ReplyTable (&tables)[2], uint8_t *status, uint64_t *out, uint64_t out_width, uint64_t bound,
                   uint8_t *resp_bytes, uint32_t *resp_offsets, uint64_t *totals, Device &&device) {
    totals[0] = totals[1] = 0;
    resp_offsets[0] = 0;
    if (n == 0) return RAFTGPU_OK;
    HostFrame f(a);
    int32_t rc = f.open();
    if (rc != RAFTGPU_OK) return rc;
    const WireRegion bytes_at = f.in(bytes, n_bytes), off_at = f.in(offsets, 4 * (n + 1));
    const WireRegion table_at[2] = {f.in(tables[0].src, tables[0].bytes), f.in(tables[1].src, tables[1].bytes)};
    const WireRegion status_at = f.out(n), out_at = f.out(out_width * n), roff_at = f.out(4 * (n + 1)), rbytes_at = f.out(bound);
    uint64_t *d_totals = scratch<uint64_t, 2>(a->d_scratch), *h_totals = scratch<uint64_t, 2>(a->h_scratch);
    rc = f.run([&](const Staged &d) {
        return device(ReplyStaged{d.at<const uint8_t>(bytes_at), d.at<const uint32_t>(off_at),
                                  {d.at<const void>(table_at[0]), d.at<const void>(table_at[1])}, d.at<uint8_t>(status_at),
                                  out ? d.at<uint64_t>(out_at) : nullptr, d.at<uint8_t>(rbytes_at), d.at<uint32_t>(roff_at),
                                  d_totals});
    });
    if (rc == RAFTGPU_OK) rc = f.back(h_totals, d_totals, 16);
    if (rc == RAFTGPU_OK) rc = f.back(status, status_at, n);
    if (rc == RAFTGPU_OK) rc = f.back(out, out_at, out_width * n);
    if (rc == RAFTGPU_OK) rc = f.wait();
    if (rc != RAFTGPU_OK) return rc;
    totals[0] = h_totals[0];
    totals[1] = h_totals[1];
    rc = f.back(resp_offsets, roff_at, 4 * (totals[0] + 1));
    if (rc == RAFTGPU_OK) rc = f.back(resp_bytes, rbytes_at, totals[1]);
    return rc == RAFTGPU_OK ? f.wait() : rc;
}

// ---- waves (DESIGN 3.19): a pass at raftgpu_arena_set_wire_waves > 1 repeats its decision over the frames it left DUP.
// Its scratch holds two lists of n frames, used in turn, and one count per wave, zeroed on st before wave 1; a pass at
// one wave keeps none.  Wave j >= 2 reads the list wave j - 1 wrote, on a grid of grid_apply blocks at most: its
// kernels loop over whatever the list holds, and return at once when it is empty.
uint64_t wave_list_words(uint64_t n, uint32_t waves) { return waves > 1 ? (2 * n + waves + 1) / 2 : 0; }

// Wave j's lists (0-based; wave 0 reads the whole batch).
WaveIo wave_io(uint32_t *lists, uint64_t n, uint32_t j) {
    uint32_t *cnt = lists + 2 * n;
    return WaveIo{j ? lists + ((j - 1) & 1u) * n : nullptr, j ? cnt + j - 1 : nullptr, lists + (j & 1u) * n, cnt + j};
}

// The wire step (abi_wire.inc): wave 1 is wire_scan_kernel and wire_wave_apply_kernel over the batch, each later wave
// wire_wave_claim_kernel<false> and wire_wave_apply_kernel over its list.
template <bool kRuns>
int32_t launch_wire_waves(raftgpu_arena *a, cudaStream_t st, const WireSrc &w, uint8_t *d_status, uint32_t *first,
                          uint32_t *lists, uint32_t waves) {
    const LeaderRuns *runs = kRuns ? a->lr_rows : nullptr;
    const uint32_t blocks = div_up(w.n, kWireThreads), grid = std::min<uint32_t>(blocks, a->grid_apply);
    CK(a, cudaMemsetAsync(lists + 2ull * w.n, 0, 4ull * waves, st));
    wire_scan_kernel<kRuns><<<blocks, kWireThreads, 0, st>>>(a->cols, w, d_status, first, runs);
    for (uint32_t j = 0; j < waves; j++) {
        const WaveIo io = wave_io(lists, w.n, j);
        if (j) wire_wave_claim_kernel<false><<<grid, kWireThreads, 0, st>>>(w, a->cap, first, io.in, io.in_n);
        wire_wave_apply_kernel<kRuns><<<j ? grid : blocks, kWireThreads, 0, st>>>(a->cols, w, d_status, first, a->d_counters,
                                                                                 runs, io);
    }
    CKL(a);
    return RAFTGPU_OK;
}

// The follower's append passes' decision (abi_app_follow.inc): afw_scan_kernel, then afw_apply_kernel at one wave; at
// more, afw_wave_apply_kernel over the batch, then wire_wave_claim_kernel<true> and afw_wave_apply_kernel over each later
// wave's list.  blk: reply_run's block sums, followed by the pass's extra words: the wave lists, then (kRuns and kAppend)
// the new row of every frame (AfwRuns, 4 words each).  kRuns: an arena with follower runs (DESIGN 3.22).  Called from
// reply_run's passes, which reports the launch errors.
template <bool kAppend, bool kRuns>
void launch_afw(raftgpu_arena *a, cudaStream_t st, const WireSrc &w, const raftgpu_follower_log *d_log, uint8_t *d_status,
                AfwRec *recs, uint32_t *first, uint64_t *d_from, uint32_t nb, uint32_t *blk,
                raftgpu_follower_appended *d_appended, uint32_t waves) {
    // (a later wave's claimant reads the table; only the kAppend kernels write it: raftgpu_follower_append_entries_device's,
    // which is not const)
    raftgpu_follower_log *logs = const_cast<raftgpu_follower_log *>(d_log);
    uint32_t *lists = blk + 2 * nb;
    AfwRunsIo rio{kRuns ? a->fr_rows : nullptr, nullptr};
    if (kRuns && kAppend) rio.next = reinterpret_cast<AfwRuns *>(reinterpret_cast<uint64_t *>(lists) + wave_list_words(w.n, waves));
    afw_scan_kernel<kAppend, kRuns><<<nb, kWireThreads, 0, st>>>(a->cols, w, d_log, d_status, recs, first, d_appended, rio);
    if (waves == 1) {
        afw_apply_kernel<kAppend, kRuns && kAppend><<<nb, kWireThreads, 0, st>>>(a->cols, w.n, d_status, recs, first, d_from,
                                                                               blk, logs, d_appended, rio);
        return;
    }
    const uint32_t grid = std::min<uint32_t>(nb, a->grid_apply);
    cudaMemsetAsync(lists + 2ull * w.n, 0, 4ull * waves, st);
    for (uint32_t j = 0; j < waves; j++) {
        const WaveIo io = wave_io(lists, w.n, j);
        if (j) wire_wave_claim_kernel<true><<<grid, kWireThreads, 0, st>>>(w, a->cap, first, io.in, io.in_n);
        afw_wave_apply_kernel<kAppend, kRuns><<<j ? grid : nb, kWireThreads, 0, st>>>(a->cols, w, d_status, recs, first, d_from,
                                                                                     blk, logs, d_appended, io, rio);
    }
}

// ---- the broadcast pipeline (DESIGN 3.11): a pass that writes a leader's frames from the arena
// (raftgpu_heartbeat_frames, raftgpu_append_frames) is a broadcast policy P (k_bcast.cuh) and shares the rest:
// bcast_check, bcast_device<P> for the `_device` form, bcast_host<P> for the host form.  `pass` is its PassScratch slot,
// `name` the word its messages start with.

// The refusals both forms make before any copy or launch.
int32_t bcast_check(raftgpu_arena *a, uint32_t first, uint32_t n, uint32_t frame_max, const char *name) {
    if (static_cast<uint64_t>(first) + n > a->cap) return RAFTGPU_ERR_RANGE;
    if (static_cast<uint64_t>(n) * kSlots * frame_max > 0xffffffffull)  // the pass's public bound
        return fail(a, RAFTGPU_ERR_INVALID, std::string(name) + " frames of this range may not be addressable by u32 offsets");
    if (n && ((a->h_meta[first] & RAFTGPU_META_WIDE_HI) || (a->h_meta[first + n - 1] & RAFTGPU_META_WIDE_LO)))
        return fail(a, RAFTGPU_ERR_INVALID, "the range splits a wide group");
    return RAFTGPU_OK;
}

// The `_device` form after its null checks, o on the device.  No group gives zero totals and offsets[0] = 0.
template <class P>
int32_t bcast_device(raftgpu_arena *a, void *stream, int pass, const char *name, uint32_t first, uint32_t n,
                     const uint32_t *d_select, const uint64_t *d_ids, const BcastOut &o) {
    int32_t rc = bcast_check(a, first, n, P::kFrameMax, name);
    if (rc != RAFTGPU_OK) return rc;
    if (reinterpret_cast<uintptr_t>(o.bytes) & 15u) return fail(a, RAFTGPU_ERR_INVALID, "frame bytes must be 16-byte aligned");
    CK(a, cudaSetDevice(a->device));
    cudaStream_t st = pick_stream(a, stream);
    constexpr uint32_t kTotals = kBcastTotals<P>;
    if (n == 0) {
        CK(a, cudaMemsetAsync(o.totals, 0, 8 * kTotals, st));
        if (o.offsets) CK(a, cudaMemsetAsync(o.offsets, 0, 4, st));
        return RAFTGPU_OK;
    }
    // scratch in u64 words: {frames | rest << 16, bytes} per slot, the totals of the block starts, then u32: 3 per block
    // (frames, bytes, leaders without a term) and, with a rest list, 1 per block (rest entries)
    const uint32_t nb = div_up(n, kBcastThreads);
    PassScratch &ps = a->pass[pass];
    rc = pass_scratch(a, st, ps, 0, n + kTotals + div_up((P::kRest ? 4ull : 3ull) * nb, 2));
    if (rc != RAFTGPU_OK) return rc;
    uint2 *cnt = reinterpret_cast<uint2 *>(ps.buf);
    uint64_t *tot = ps.buf + n;
    uint32_t *blk = reinterpret_cast<uint32_t *>(tot + kTotals), *blk_rest = blk + 3ull * nb;
    const BcastSrc s{first, n, a->hi, d_select, d_ids};
    bcast_size_kernel<P><<<nb, kBcastThreads, 0, st>>>(a->cols, s, cnt, blk, blk_rest);
    block_starts_kernel<3><<<1, kScanThreads, 0, st>>>(blk, nb, tot, nullptr);
    if constexpr (P::kRest) block_starts_kernel<1><<<1, kScanThreads, 0, st>>>(blk_rest, nb, tot + 3, nullptr);
    bcast_write_kernel<P><<<nb, kBcastThreads, kBcastSmem<P>, st>>>(a->cols, s, cnt, blk, blk_rest, tot, o);
    CKL(a);
    return RAFTGPU_OK;
}

// The host form after its null checks, o on the host (HostFrame): d_wire holds [ids | select | offsets | rest entries,
// none without a rest list | bytes], the totals go to the arena's scratch.  The bytes are the rest region, what d_wire
// already has room for; when the frames need more (and fit the caller's buffer) the region is enlarged to exactly that
// and the pass runs again, so a caller with a steady load runs it once per call.
template <class P>
int32_t bcast_host(raftgpu_arena *a, int pass, const char *name, uint32_t first, uint32_t n, const uint32_t *select,
                   const uint64_t *ids, const BcastOut &o) {
    std::lock_guard<std::mutex> ctl_lock(a->ctl_mu);
    int32_t rc = bcast_check(a, first, n, P::kFrameMax, name);
    if (rc != RAFTGPU_OK) return rc;
    constexpr uint32_t kTotals = kBcastTotals<P>;
    for (uint32_t k = 0; k < kTotals; k++) o.totals[k] = 0;
    if (n == 0) {
        if (!o.offsets) return fail(a, RAFTGPU_ERR_FULL, "no offsets buffer");
        o.offsets[0] = 0;
        return RAFTGPU_OK;
    }
    HostFrame f(a);
    rc = f.open();
    if (rc != RAFTGPU_OK) return rc;
    const uint64_t words = select ? (static_cast<uint64_t>(first) + n + 31) / 32 : 0;
    const uint64_t frames_room = std::min<uint64_t>(o.frames_cap, static_cast<uint64_t>(kSlots) * n);
    const uint64_t rest_room = std::min<uint64_t>(o.rest_cap, static_cast<uint64_t>(kSlots) * n);
    const WireRegion ids_at = f.in(ids, 8ull * (kSlots + 1) * n), sel_at = f.in(select, 4 * words);
    const WireRegion off_at = f.out(4 * (frames_room + 1)), rest_at = f.out(sizeof(raftgpu_send_entry) * rest_room);
    const WireRegion bytes_at = f.rest(16);
    uint64_t *d_totals = scratch<uint64_t, kTotals>(a->d_scratch), *h_totals = scratch<uint64_t, kTotals>(a->h_scratch);
    uint64_t room = 0;
    auto run = [&]() {
        int32_t r = f.run([&](const Staged &d) {
            room = std::min(o.bytes_cap, d.rest);
            return bcast_device<P>(a, a->s_compute, pass, name, first, n, words ? d.at<const uint32_t>(sel_at) : nullptr,
                                   d.at<const uint64_t>(ids_at),
                                   {d.at<uint8_t>(bytes_at), d.at<uint32_t>(off_at), d.at<raftgpu_send_entry>(rest_at),
                                    room, frames_room, rest_room, d_totals});
        });
        if (r == RAFTGPU_OK) r = f.back(h_totals, d_totals, 8 * kTotals);
        return r == RAFTGPU_OK ? f.wait() : r;
    };
    rc = run();
    if (rc != RAFTGPU_OK) return rc;
    const uint64_t rest = P::kRest ? h_totals[2] : 0;
    const bool fits = o.offsets && h_totals[0] <= o.frames_cap && h_totals[1] <= o.bytes_cap && (!P::kRest || rest <= o.rest_cap);
    if (fits && h_totals[1] > room) {  // the caller's buffer is large enough, d_wire was not
        f.enlarge(h_totals[1]);
        rc = run();
        if (rc != RAFTGPU_OK) return rc;
    }
    for (uint32_t k = 0; k < kTotals; k++) o.totals[k] = h_totals[k];
    if (!fits) return fail(a, RAFTGPU_ERR_FULL, std::string(name) + " frames exceed the output buffers");
    rc = f.back(o.offsets, off_at, 4 * (h_totals[0] + 1));
    if (rc == RAFTGPU_OK) rc = f.back(o.rest, rest_at, sizeof(raftgpu_send_entry) * rest);
    if (rc == RAFTGPU_OK) rc = f.back(o.bytes, bytes_at, h_totals[1]);
    return rc == RAFTGPU_OK ? f.wait() : rc;
}

// ---- the step frame: every raftgpu_step_begin* form is step_admit -> the form's own function, which queues its H2D
// copies on s_h2d and its apply kernels on s_compute and says what it queued (StepWork) -> step_finish -> step_book.

// What a form queued, for the rest of the step and its raftgpu_step_result.
struct StepWork {
    uint64_t res_bytes = 0;    // result / status bytes to copy back from d_results
    uint64_t wave0_slots = 0;  // result slots of wave 0 (raftgpu_step_slot_results)
    uint64_t n_records = 0;
    uint64_t h2d_bytes = 0;
    uint32_t later_waves = 0;  // waves after wave 0 (a later wave needs a record of its cell in wave 0)
    bool fused = false;        // the fused tile kernel has applied AND recomputed
};

// RAFTGPU_SYNC_DEBUG (diagnostics, read once per process): wait for every stage of a step and name it
bool sync_debug() {
    static const bool on = getenv("RAFTGPU_SYNC_DEBUG") != nullptr;
    return on;
}
void stage_done(raftgpu_arena *a, const char *what) {
    if (!sync_debug()) return;
    const cudaError_t e = cudaStreamSynchronize(a->s_compute);
    fprintf(stderr, "[raftgpu] @%.0f   stage done: %s (%s)\n", trace_us(a), what, cudaGetErrorString(e));
}

// What every form checks before it touches the fill set (*out).  `form` names a form that brings its own batch, which
// cannot go with records enqueued for the step; nullptr: raftgpu_step_begin, which submits them.
int32_t step_admit(raftgpu_arena *a, const char *form, StagingSet **out) {
    wait_submitter(a);
    if (a->n_inflight >= 2) return fail(a, RAFTGPU_ERR_BUSY, "two steps already in flight: call raftgpu_step_wait");
    StagingSet &s = a->sets[a->fill];
    if (s.in_flight) return RAFTGPU_ERR_BUSY;
    if (form && (s.next_chunk.load() != 0 || !s.overflow_waves.empty()))
        return fail(a, RAFTGPU_ERR_INVALID, std::string("records were enqueued for this step: cannot mix with ") + form);
    CK(a, cudaSetDevice(a->device));
    *out = &s;
    return RAFTGPU_OK;
}

// The step's H2D copies are queued: its kernels start behind them, with d_step_adv cleared.
int32_t compute_after_h2d(raftgpu_arena *a, StagingSet &s) {
    CK(a, cudaEventRecord(s.ev_h2d, a->s_h2d));
    CK(a, cudaStreamWaitEvent(a->s_compute, s.ev_h2d, 0));
    CK(a, cudaMemsetAsync(s.d_step_adv, 0, 8, a->s_compute));
    stage_done(a, "h2d");
    return RAFTGPU_OK;
}

// The end of every step: recompute [0, hi) unless the fused kernel has, the D2H, the events, the set's result.  No
// booking: the caller thread books a step (step_book), an asynchronous one before the submitter thread queues it.
int32_t step_finish(raftgpu_arena *a, StagingSet &s, uint32_t flags, const StepWork &w) {
    const uint32_t hi = a->hi;
    uint64_t *d_commit = (flags & RAFTGPU_STEP_READ_COMMITTED) ? s.d_commit_out : nullptr;
    if (!w.fused) {
        const int32_t rc = launch_recompute(a, a->s_compute, 0, hi, a->voter_hint, s.d_adv_bitmap, d_commit, nullptr, nullptr,
                                            s.d_step_adv);
        if (rc != RAFTGPU_OK) return rc;
    }
    CK(a, cudaEventRecord(s.ev_compute, a->s_compute));
    CK(a, cudaStreamWaitEvent(a->s_d2h, s.ev_compute, 0));
    CK(a, cudaMemcpyAsync(s.h_step_adv, s.d_step_adv, 8, cudaMemcpyDeviceToHost, a->s_d2h));
    if (hi)
        CK(a, cudaMemcpyAsync(s.h_adv_bitmap, s.d_adv_bitmap, 4ull * ((hi + 31) / 32),
                              cudaMemcpyDeviceToHost, a->s_d2h));
    if (d_commit && hi)
        CK(a, cudaMemcpyAsync(s.h_committed, s.d_commit_out, 8ull * hi, cudaMemcpyDeviceToHost, a->s_d2h));
    if (w.res_bytes)
        CK(a, cudaMemcpyAsync(s.h_results, s.d_results, w.res_bytes, cudaMemcpyDeviceToHost, a->s_d2h));
    CK(a, cudaEventRecord(s.ev_done, a->s_d2h));
    s.flags = flags;
    s.wave0_slots = w.wave0_slots;
    s.result.n_records = w.n_records;
    s.result.h2d_bytes = w.h2d_bytes;
    s.result.d2h_bytes = 8 + (hi ? 4ull * ((hi + 31) / 32) : 0) + ((d_commit && hi) ? 8ull * hi : 0) + w.res_bytes;
    s.result.n_waves = (w.n_records ? 1 : 0) + w.later_waves;
    s.result.n_groups = hi;
    return RAFTGPU_OK;
}

// The fill set is now in flight (caller thread only): pick the next one to fill.
int32_t step_book(raftgpu_arena *a) {
    StagingSet &s = a->sets[a->fill];
    s.in_flight = true;
    a->inflight[a->n_inflight++] = a->fill;
    // flip: a set that is neither in flight nor holding the results of the last completed step
    // becomes the fill target (with 3 sets and <= 2 in flight there is always one)
    int other = -1;
    for (int k = 0; k < kNumSets; k++) {
        if (a->sets[k].in_flight) continue;
        if (k == a->last_done && other >= 0) continue;  // prefer keeping the last results alive
        if (other < 0 || k != a->last_done) other = k;
    }
    if (other < 0) return fail(a, RAFTGPU_ERR_BUSY, "no free staging set");
    const int32_t rc = reclaim_set(a, a->sets[other]);
    if (rc != RAFTGPU_OK) return rc;
    if (a->last_done == other) a->last_done = -1;  // its results are gone
    a->fill = other;
    return RAFTGPU_OK;
}

// One synchronous step: admission, the form's queue(StagingSet &, StepWork &), the finish, the booking.
template <typename Queue>
int32_t run_step(raftgpu_arena *a, const char *form, uint32_t flags, Queue &&queue) {
    StagingSet *s = nullptr;
    StepWork w;
    int32_t rc = step_admit(a, form, &s);
    if (rc == RAFTGPU_OK) rc = queue(*s, w);
    if (rc == RAFTGPU_OK) rc = step_finish(a, *s, flags, w);
    return rc == RAFTGPU_OK ? step_book(a) : rc;
}

}  // namespace

// ===========================================================================
extern "C" {

#include "abi_control_batch.inc"
#include "abi_control.inc"
#include "abi_device.inc"
#include "abi_staging.inc"
#include "abi_compact.inc"
#include "abi_wire.inc"
#include "abi_results.inc"
#include "abi_read.inc"
#include "abi_hb_wire.inc"
#include "abi_hb_frames.inc"
#include "abi_app_frames.inc"
#include "abi_hb_follow.inc"
#include "abi_vote_wire.inc"
#include "abi_vote_request.inc"
#include "abi_app_follow.inc"
#include "abi_leader_runs.inc"
#include "abi_follow_term.inc"
#include "abi_leader_term.inc"
#include "abi_follow_resp.inc"

}  // extern "C"
