// k_tile.cuh -- step_tile_kernel: the fused apply + recompute tile kernel on packed records (the headline kernel).
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).

// ---------------------------------------------------------------------------
// step_tile_kernel: apply + recompute FUSED, for batches whose records are in group order.
//
// The scatter apply kernel above keeps many loads in flight but stays far below the HBM peak: its cell
// accesses are sector-granular (8 useful bytes per 32-byte sector request, several rows per
// record), which HBM serves at roughly half the efficiency of dense bursts.  When the batch is
// ordered by group, a tile of kFTile consecutive groups owns a CONTIGUOUS record range, so the
// whole step becomes dense traffic: per tile the producer warp bulk-loads (TMA, cp.async.bulk)
// the tile's rows of matched / next_idx / committed_index / pflags / meta / committed /
// term_start / last_index and its record range into one shared-memory stage; the consumers
//   A. apply every record of the tile to the shared-memory rows (one thread per record;
//      distinct cells per wave, so no conflicts),
//   B. recompute the commit index of the tile's groups from the same shared-memory rows
//      (matched is read from HBM once per step instead of twice),
//   C. bulk-store the rows back (cp.async.bulk.global.shared::cta).
// Peer slots outside `hint` (learners) and the cold columns are handled through HBM directly.
// tile_off[t] = index of the first packed record of tile t (raftgpu_tile_index builds it).
constexpr int kFTile = RAFTGPU_TILE_GROUPS;  // groups per tile
// consumer groups: tile i of a CTA is handled by group i % kNG, so the phases of kNG tiles overlap
// inside one CTA; each group has kCT threads (kCT >= kFTile).  Template parameters of the kernel.
constexpr int kFMaxStages = 8;
// Row strides inside a stage.  Records arrive in group order, so the ~3.5 records of one group sit
// in neighbouring lanes and touch the SAME column index of DIFFERENT rows: with a 256-element row
// stride they would all fall on the same shared-memory banks (4-way conflicts on every access).
// 258 u64 (= 2064 B, still 16-byte aligned for TMA) shifts consecutive rows by 4 banks.
constexpr uint32_t kFRow64 = (kFTile + 2) * 8;   // bytes per u64 row
constexpr uint32_t kFRow8 = kFTile + 16;         // bytes per u8 (pflags) row
constexpr uint32_t kFDefer = 32;                 // deferred (rare-path) records per warp per tile; more are handled inline

__device__ __forceinline__ void named_bar_sync(int id, int n_threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n_threads) : "memory");
}
// A consumer's wait for "the loads of MY tile have landed in this stage".  A consumer group sees only every kNG-th
// tile, so on one stage's `full` barrier it skips phases -- and a parity wait is only exact while the waiter is at
// most ONE phase ahead.  With uniform tiles that always holds; with a batch that covers only part of the groups it
// does not (record-less tiles are done in a microsecond, loads of light and heavy tiles land out of order): a group
// could pass the barrier of a stage still armed for the PREVIOUS tile and work on half-landed rows.  So it first
// waits for the previous use of the stage to be DONE (`done` barrier, previous phase).  That wait is exact: the
// group's own previous tile was loaded, hence the tile n_stages before IT was stored, stores happen in tile order,
// and with n_stages >= kNG that covers the previous user of this stage; and once the previous user is done, the
// `full` barrier is in this tile's phase, so the second wait is exact too.
__device__ __forceinline__ void wait_stage(uint64_t *full_bar, uint64_t *done_bar, uint32_t parity) {
    mbar_wait(done_bar, parity ^ 1u);  // (first use of a stage: the parity-1 wait on a fresh barrier passes at once)
    mbar_wait(full_bar, parity);
}
// 1-D TMA store: shared -> global, tracked by the per-thread bulk async-group
__device__ __forceinline__ void tma_store_1d(void *dst, const void *src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src)),
                 "r"(bytes)
                 : "memory");
}

struct TileArgs {
    const PackedRec *recs;     // packed records in group order
    const uint32_t *tile_off;  // [n_tiles + 1]
    uint32_t n_groups;         // groups [0, n_groups)
    uint32_t hint;
    int n_stages;
    uint32_t rec_cap;          // packed records staged per tile (multiple of 4); the rest is read from HBM
    uint8_t *results;          // nullable, one byte per packed record
    uint32_t *adv_bitmap;      // nullable
    uint64_t *commit_out;      // nullable
    uint32_t *step_advanced;   // nullable
    unsigned long long *counters;
    unsigned long long *dbg;   // nullable: [8] cycle totals per phase (diagnostics, RAFTGPU_TILE_DEBUG=1)
    uint32_t skip;             // diagnostics only (RAFTGPU_TILE_SKIP, results are WRONG): 1 no records, 2 no recompute, 4 no stores
};

// bytes of one stage for H hinted slots (shared by host and device)
__host__ __device__ constexpr uint32_t tile_stage_bytes(uint32_t H, uint32_t rec_cap) {
    return 3u * H * kFRow64 + 3u * kFRow64 + kFTile * 4u + H * kFRow8 + rec_cap * 16u;
}

template <bool kSimple5, int kCT, int kNG>
__global__ void __launch_bounds__(kCT *kNG + 64, 1) step_tile_kernel(Columns c, TileArgs a) {
    static_assert(kCT >= kFTile && kCT % 32 == 0, "a consumer group covers a tile");
    const uint32_t kFRecCap = a.rec_cap;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t full_bar[kFMaxStages];   // loads landed            (load warp -> consumers)
    __shared__ __align__(8) uint64_t done_bar[kFMaxStages];   // rows final in smem      (consumers -> store warp)
    __shared__ __align__(8) uint64_t empty_bar[kFMaxStages];  // rows read by the stores (store warp -> load warp)
    __shared__ uint32_t s_defer[32][kFDefer];                 // per warp: tile-relative indexes of its rare-path records
    __shared__ uint32_t s_ndefer[32];

    const uint32_t hint = kSimple5 ? 0x1fu : (a.hint & 0xffu);
    const uint32_t H = kSimple5 ? 5u : static_cast<uint32_t>(__popc(hint));
    // stage layout (bytes)
    const uint32_t o_matched = 0, o_next = H * kFRow64, o_pc = 2u * H * kFRow64, o_committed = 3u * H * kFRow64,
                   o_ts = o_committed + kFRow64, o_li = o_ts + kFRow64, o_meta = o_li + kFRow64,
                   o_flags = o_meta + kFTile * 4u, o_recs = o_flags + H * kFRow8, stage_bytes = tile_stage_bytes(H, a.rec_cap);
    const uint32_t n_tiles = (a.n_groups + kFTile - 1) / kFTile;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int s = 0; s < a.n_stages; s++) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&done_bar[s], 1);
            mbar_init(&empty_bar[s], 1);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    uint32_t local[7] = {0, 0, 0, 0, 0, 0, 0};  // records, updates, rejects, decrements, no_progress | recomputes, advanced
    if (warp == kNG * kCT / 32 + 1) {
        // ===================== store warp: rows back to HBM, then the stage is free =====================
        const uint32_t n_out = 4u * H + 2u + (a.commit_out ? 1u : 0u);
        uint32_t it = 0;
        for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, it++) {
            const int st = it % a.n_stages;
            const uint32_t ph = (it / a.n_stages) & 1u;
            const uint32_t g0 = tile * kFTile;
            const uint32_t ng = a.n_groups - g0 < kFTile ? a.n_groups - g0 : kFTile;
            const uint32_t ng16 = (ng + 15u) & ~15u;
            uint8_t *sb = smem + static_cast<size_t>(st) * stage_bytes;
            mbar_wait(&done_bar[st], ph);  // every lane waits: the barrier's completion orders the consumers' writes
            for (uint32_t j = lane; j < ((a.skip & 4u) ? 0u : n_out); j += 32) {
                if (j < 4u * H) {
                    const uint32_t col = j / H, r = j % H;
                    uint32_t slot = 0, seen = 0;
                    for (uint32_t s2 = 0; s2 < kSlots; s2++)
                        if ((hint >> s2) & 1u) {
                            if (seen == r) slot = s2;
                            seen++;
                        }
                    const size_t cell = static_cast<size_t>(slot) * c.cap + g0;
                    if (col == 0) tma_store_1d(c.matched + cell, sb + o_matched + r * kFRow64, ng16 * 8u);
                    if (col == 1) tma_store_1d(c.next_idx + cell, sb + o_next + r * kFRow64, ng16 * 8u);
                    if (col == 2) tma_store_1d(c.peer_committed + cell, sb + o_pc + r * kFRow64, ng16 * 8u);
                    if (col == 3) tma_store_1d(c.pflags + cell, sb + o_flags + r * kFRow8, ng16);
                } else if (j == 4u * H) {
                    tma_store_1d(c.committed + g0, sb + o_committed, ng16 * 8u);
                } else if (j == 4u * H + 1u) {
                    tma_store_1d(c.last_index + g0, sb + o_li, ng16 * 8u);
                } else {  // the step's commit-index output: the tile's `committed` row, one dense copy (not 8-byte scatters)
                    tma_store_1d(a.commit_out + g0, sb + o_committed, ng16 * 8u);
                }
            }
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // shared memory has been read
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[st]);
        }
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // all stores have landed
    } else if (warp == kNG * kCT / 32) {
        // ===================== load warp =====================
        const uint32_t n_copies = 4u * H + 5u;
        uint32_t it = 0;
        // the tile index of the NEXT tile is fetched while this one is being issued: a dependent global
        // load at the top of every iteration would sit on the critical path of the ring
        uint32_t nx_beg = blockIdx.x < n_tiles ? a.tile_off[blockIdx.x] : 0u, nx_end = blockIdx.x < n_tiles ? a.tile_off[blockIdx.x + 1] : 0u;
        for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, it++) {
            const int st = it % a.n_stages;
            const uint32_t ph = (it / a.n_stages) & 1u;
            const uint32_t g0 = tile * kFTile;
            const uint32_t ng = a.n_groups - g0 < kFTile ? a.n_groups - g0 : kFTile;
            const uint32_t ng16 = (ng + 15u) & ~15u;  // 16-byte multiples for every row; inside the padded stride
            const uint32_t rbeg = nx_beg, rend = nx_end;
            if (tile + gridDim.x < n_tiles) {
                nx_beg = a.tile_off[tile + gridDim.x];
                nx_end = a.tile_off[tile + gridDim.x + 1];
            }
            const uint32_t staged = rend - rbeg < kFRecCap ? rend - rbeg : kFRecCap;
            if (lane == 0) {
                mbar_wait(&empty_bar[st], ph ^ 1u);
                mbar_expect_tx(&full_bar[st], 3u * H * ng16 * 8u + H * ng16 + 3u * ng16 * 8u + ng16 * 4u + staged * 16u);
            }
            __syncwarp();
            uint8_t *sb = smem + static_cast<size_t>(st) * stage_bytes;
            for (uint32_t j = lane; j < n_copies; j += 32) {
                if (j < 4u * H) {
                    const uint32_t col = j / H, r = j % H;  // col: 0 matched, 1 next_idx, 2 committed_index, 3 pflags
                    uint32_t slot = 0, seen = 0;
                    for (uint32_t s2 = 0; s2 < kSlots; s2++)
                        if ((hint >> s2) & 1u) {
                            if (seen == r) slot = s2;
                            seen++;
                        }
                    const size_t cell = static_cast<size_t>(slot) * c.cap + g0;
                    if (col == 0) tma_load_1d(sb + o_matched + r * kFRow64, c.matched + cell, ng16 * 8u, &full_bar[st]);
                    if (col == 1) tma_load_1d(sb + o_next + r * kFRow64, c.next_idx + cell, ng16 * 8u, &full_bar[st]);
                    if (col == 2) tma_load_1d(sb + o_pc + r * kFRow64, c.peer_committed + cell, ng16 * 8u, &full_bar[st]);
                    if (col == 3) tma_load_1d(sb + o_flags + r * kFRow8, c.pflags + cell, ng16, &full_bar[st]);
                } else if (j == 4u * H) {
                    tma_load_1d(sb + o_committed, c.committed + g0, ng16 * 8u, &full_bar[st]);
                } else if (j == 4u * H + 1) {
                    tma_load_1d(sb + o_ts, c.term_start + g0, ng16 * 8u, &full_bar[st]);
                } else if (j == 4u * H + 2) {
                    tma_load_1d(sb + o_li, c.last_index + g0, ng16 * 8u, &full_bar[st]);
                } else if (j == 4u * H + 3) {
                    tma_load_1d(sb + o_meta, c.meta + g0, ng16 * 4u, &full_bar[st]);
                } else if (staged) {
                    tma_load_1d(sb + o_recs, a.recs + rbeg, staged * 16u, &full_bar[st]);
                }
            }
        }
    } else {
        // ===================== consumers: group cg takes every kFGroups-th tile of this CTA =====================
        const uint32_t cg = warp / (kCT / 32);
        const uint32_t tid = threadIdx.x - cg * kCT;
        const int bar_id = 1 + static_cast<int>(cg);
        constexpr uint32_t R64 = kFRow64 / 8;  // row stride in u64 elements
        uint32_t it = 0;
        const uint32_t first_tile = blockIdx.x + cg * gridDim.x, tile_step = kNG * gridDim.x;
        uint32_t nx_beg = first_tile < n_tiles ? a.tile_off[first_tile] : 0u, nx_end = first_tile < n_tiles ? a.tile_off[first_tile + 1] : 0u;
        it = cg;
        for (uint32_t tile = first_tile; tile < n_tiles; tile += tile_step, it += kNG) {

            const int st = it % a.n_stages;
            const uint32_t ph = (it / a.n_stages) & 1u;
            const uint32_t g0 = tile * kFTile;
            const uint32_t ng = a.n_groups - g0 < kFTile ? a.n_groups - g0 : kFTile;
            const uint32_t rbeg = nx_beg, rend = nx_end;
            if (tile + tile_step < n_tiles) {  // next tile of this consumer group: fetched during this one
                nx_beg = a.tile_off[tile + tile_step];
                nx_end = a.tile_off[tile + tile_step + 1];
            }
            const uint32_t cnt = rend - rbeg, staged = cnt < kFRecCap ? cnt : kFRecCap;
            uint8_t *sb = smem + static_cast<size_t>(st) * stage_bytes;
            uint64_t *s_matched = reinterpret_cast<uint64_t *>(sb + o_matched);
            uint64_t *s_next = reinterpret_cast<uint64_t *>(sb + o_next);
            uint64_t *s_pc = reinterpret_cast<uint64_t *>(sb + o_pc);
            uint64_t *s_committed = reinterpret_cast<uint64_t *>(sb + o_committed);
            uint64_t *s_ts = reinterpret_cast<uint64_t *>(sb + o_ts);
            uint64_t *s_li = reinterpret_cast<uint64_t *>(sb + o_li);
            uint32_t *s_meta = reinterpret_cast<uint32_t *>(sb + o_meta);
            uint8_t *s_flags = sb + o_flags;
            const PackedRec *s_recs = reinterpret_cast<const PackedRec *>(sb + o_recs);
            const ulonglong2 *g_recs = reinterpret_cast<const ulonglong2 *>(a.recs + rbeg);
            // direct records: this thread's first record is requested BEFORE the wait for the stage (its address does
            // not depend on it); the loop then fetches one record ahead.  (Two ahead was slower
            // with scripts/micro_tile.py: the kernel sits near its register ceiling and the consumers are bound by
            // issue latency, not by the record reads.)
            ulonglong2 q_next = make_ulonglong2(kPkExt, 0ull);
            if (staged == 0 && tid < cnt) q_next = g_recs[tid];
            long long t0 = 0, t1 = 0, t2 = 0, t3 = 0, t4 = 0;
            if (a.dbg && tid == 0) t0 = clock64();
            wait_stage(&full_bar[st], &done_bar[st], ph);
            if (a.dbg && tid == 0) t1 = clock64();

            // ---- A: the tile's records against the shared-memory rows (raft.rs:1663-1743)
            // Records come from the stage when they were staged (rec_cap > 0), else straight from HBM /
            // L2 (rec_cap == 0: the stage holds rows only, which buys a fifth stage; the records of a
            // tile were prefetched into L2 while the previous tile was processed, and the loop fetches
            // the records two iterations ahead).
            auto rec_at = [&](uint32_t j) -> ulonglong2 {
                if (j < staged) return reinterpret_cast<const ulonglong2 *>(s_recs)[j];
                if (j < cnt) return g_recs[j];
                return make_ulonglong2(kPkExt, 0ull);
            };
            // The main loop handles the records that make up ~98 % of the traffic -- an accept or a leader-local
            // record for a staged cell of a peer in Replicate or Probe state -- straight on the packed words and the
            // shared-memory cell.  Whatever else turns up (a rejection, a WIDE commit, a Snapshot-state peer, a learner
            // outside the hint, a record that is not this tile's) is put on the WARP's deferred list and handled after
            // the loop with all the warp's lanes working on such records at once, instead of one lane at a time
            // inside the loop (half of all warp-iterations contain a rejection): a wave has at most one record per
            // cell, so the order between the two passes does not matter.
            uint32_t *my_defer = s_defer[warp];
            if (lane == 0) s_ndefer[warp] = 0;
            __syncwarp();
            // A record the straight-line form does not take: a rejection without a snapshot request on a staged
            // Replicate / Probe cell directly (maybe_decr_to, progress.rs:168-206), the rest through apply_one.
            auto slow_record = [&](const uint32_t k) {
                const ulonglong2 q = rec_at(k);
                const uint64_t w0 = q.x;
                const uint32_t slot = static_cast<uint32_t>(w0 >> 32) & 7u;
                const uint32_t g = static_cast<uint32_t>(w0);
                const uint32_t gl = g - g0;
                if (!(w0 & kPkWide) && (w0 & kPkReject) && gl < ng && ((hint >> slot) & 1u)) {
                    const uint32_t r = kSimple5 ? slot : static_cast<uint32_t>(__popc(hint & ((1u << slot) - 1u)));
                    const uint32_t ci = r * R64 + gl;
                    const uint32_t f0 = s_flags[r * kFRow8 + gl];
                    const uint32_t state = f0 & RAFTGPU_PF_STATE_MASK;
                    const bool present = kSimple5 || (((RAFTGPU_META_IN(s_meta[gl]) | RAFTGPU_META_OUT(s_meta[gl]) |
                                                        RAFTGPU_META_LEARN(s_meta[gl])) >> slot) & 1u);
                    if (present && state != RAFTGPU_STATE_SNAPSHOT) {
                        // its EXT payloads: [kind 1 hint] [kind 2 snapshot request]
                        uint64_t hint_idx = 0;
                        bool snapshot_req = false;
                        const ulonglong2 e1 = rec_at(k + 1);   // (past the end: a padding EXT of kind 0)
                        const ulonglong2 e2 = rec_at(k + 2);
                        const bool x1 = (e1.x & kPkExt) != 0, x2 = x1 && (e2.x & kPkExt) != 0;
                        if (x1 && (e1.x >> 40) == 1) hint_idx = e1.y;
                        if ((x1 && (e1.x >> 40) == 2) || (x2 && (e2.x >> 40) == 2)) snapshot_req = true;
                        if (!snapshot_req) {
                            const uint64_t index = q.y;
                            const uint32_t delta = static_cast<uint32_t>(w0 >> 40);
                            uint64_t m = s_matched[ci], nx = s_next[ci];
                            const uint64_t nx0 = nx;
                            uint32_t f = f0 | RAFTGPU_PF_RECENT_ACTIVE, res = 0;         // raft.rs:1674
                            local[0]++;
                            local[2]++;
                            const uint64_t commit = index - delta;
                            if (commit > s_pc[ci]) s_pc[ci] = commit;                   // raft.rs:1677
                            bool ok;
                            if (state == RAFTGPU_STATE_REPLICATE) {
                                ok = index > m;                                          // :173-177 stale otherwise
                                if (ok) nx = m + 1;                                      // :178-179
                            } else if (nx == 0 || nx - 1 != index) {
                                ok = false;                                              // :188-192 stale
                            } else {
                                nx = umin64(index, hint_idx + 1);                        // :195-199
                                if (nx < 1) nx = 1;
                                f &= ~RAFTGPU_PF_PAUSED;                                 // :204
                                ok = true;
                            }
                            if (ok) {
                                local[3]++;
                                res = RAFTGPU_RES_OK | RAFTGPU_RES_SEND;
                                if (state == RAFTGPU_STATE_REPLICATE) {                  // raft.rs:1716-1718 become_probe
                                    f = (f & ~(RAFTGPU_PF_PAUSED | RAFTGPU_PF_INS_FULL | RAFTGPU_PF_STATE_MASK)) | RAFTGPU_STATE_PROBE;
                                    c.pending_snapshot[static_cast<size_t>(slot) * c.cap + g] = 0;
                                    nx = m + 1;
                                }
                            }
                            if (nx != nx0) s_next[ci] = nx;
                            if (f != f0) s_flags[r * kFRow8 + gl] = static_cast<uint8_t>(f);
                            if (a.results) a.results[rbeg + k] = static_cast<uint8_t>(res);
                            return;
                        }
                    }
                }
                // General path: from the stage when the whole tile is staged, else from HBM.
                const bool from_smem = staged == cnt;
                const void *base = from_smem ? static_cast<const void *>(s_recs) : static_cast<const void *>(a.recs + rbeg);
                const uint64_t nn = from_smem ? staged : cnt;
                const RecRegs rec = load_rec<true>(base, k, nn);
                uint32_t res = 0;
                if (!((rec.w0 >> 40) & RAFTGPU_REC_EXT)) {
                    const uint32_t g2 = static_cast<uint32_t>(rec.w0), slot2 = static_cast<uint32_t>(rec.w0 >> 32) & 0xffu;
                    const uint32_t gl2 = g2 - g0;
                    if (gl2 >= ng) {  // not this tile's group: the batch is not in group order / bad index
                        local[0]++;
                        local[4]++;
                        res = RAFTGPU_RES_NO_PROGRESS;
                    } else if (slot2 < kSlots && ((hint >> slot2) & 1u)) {
                        const uint32_t r = __popc(hint & ((1u << slot2) - 1u));
                        CellRegs cd;
                        cd.meta = s_meta[gl2];
                        cd.matched = s_matched[r * R64 + gl2];
                        cd.next_idx = s_next[r * R64 + gl2];
                        cd.flags = s_flags[r * kFRow8 + gl2];
                        cd.peer_committed = s_pc[r * R64 + gl2];
                        const CellPtrs sp{&s_matched[r * R64 + gl2], &s_next[r * R64 + gl2], &s_pc[r * R64 + gl2], &s_li[gl2],
                                          &s_flags[r * kFRow8 + gl2]};
                        res = apply_one<1>(c, base, nn, k, rec, cd, sp, local);
                    } else {  // a peer slot outside the hint (a learner): its cell lives in HBM
                        CellRegs cd = load_cell(c, rec);
                        cd.meta = s_meta[gl2];
                        CellPtrs gp = global_cell_ptrs(c, rec);
                        gp.last_index = &s_li[gl2];
                        res = apply_one<1>(c, base, nn, k, rec, cd, gp, local);
                    }
                }
                if (a.results) a.results[rbeg + k] = static_cast<uint8_t>(res);
            };
            if (staged != 0) q_next = rec_at(tid);
            for (uint32_t k = tid; k < ((a.skip & 1u) ? 0u : cnt); k += kCT) {
                const ulonglong2 q = q_next;
                q_next = rec_at(k + kCT);
                const uint64_t w0 = q.x;
                if (w0 & kPkExt) {
                    if (a.results) a.results[rbeg + k] = 0;
                    continue;
                }
                const uint32_t slot = static_cast<uint32_t>(w0 >> 32) & 7u;
                const uint32_t g = static_cast<uint32_t>(w0);
                const uint32_t gl = g - g0;
                bool done = false;
                if (!(w0 & (kPkWide | kPkReject)) && gl < ng && ((hint >> slot) & 1u)) {
                    const uint32_t r = kSimple5 ? slot : static_cast<uint32_t>(__popc(hint & ((1u << slot) - 1u)));
                    const uint32_t ci = r * R64 + gl;
                    const uint32_t f0 = s_flags[r * kFRow8 + gl];
                    const uint32_t state = f0 & RAFTGPU_PF_STATE_MASK;
                    const bool present = kSimple5 || (((RAFTGPU_META_IN(s_meta[gl]) | RAFTGPU_META_OUT(s_meta[gl]) |
                                                        RAFTGPU_META_LEARN(s_meta[gl])) >> slot) & 1u);
                    if (present && state != RAFTGPU_STATE_SNAPSHOT) {
                        // accept / leader-local: maybe_update (progress.rs:138-150), shared by the accept path
                        // (raft.rs:1674-1677, 1724-1730) and the leader-local path (raft.rs:974-991, 1010-1014);
                        // only an accept looks at is_paused() and may move a probing peer to Replicate.
                        const uint64_t index = q.y;
                        const uint32_t delta = static_cast<uint32_t>(w0 >> 40);
                        const bool is_local = (w0 & kPkLocal) != 0;
                        const uint64_t m = s_matched[ci], nx = s_next[ci], pcv = s_pc[ci];
                        local[0]++;
                        if (is_local && delta != kPkNoCommit) s_li[gl] = index + delta;   // raft.rs:974-991
                        const uint64_t commit = index - delta;
                        if (!is_local && commit > pcv) s_pc[ci] = commit;                 // raft.rs:1677
                        const bool probe = state == RAFTGPU_STATE_PROBE;
                        const bool need = m < index;
                        const bool old_paused = !is_local && (f0 & (probe ? RAFTGPU_PF_PAUSED : RAFTGPU_PF_INS_FULL)) != 0;
                        const bool trans = need && !is_local && probe;                    // raft.rs:1730 become_replicate
                        uint32_t f = is_local ? f0 : (f0 | RAFTGPU_PF_RECENT_ACTIVE);     // raft.rs:1674
                        if (need) f &= ~RAFTGPU_PF_PAUSED;
                        if (trans)
                            f = (f & ~(RAFTGPU_PF_PAUSED | RAFTGPU_PF_INS_FULL | RAFTGPU_PF_STATE_MASK)) | RAFTGPU_STATE_REPLICATE;
                        uint64_t nnx = nx < index + 1 ? index + 1 : nx;
                        if (trans) {
                            nnx = index + 1;                                              // next_idx = matched + 1
                            c.pending_snapshot[static_cast<size_t>(slot) * c.cap + g] = 0;
                        }
                        local[1] += need ? 1u : 0u;
                        if (need) s_matched[ci] = index;
                        if (nnx != nx) s_next[ci] = nnx;
                        if (f != f0) s_flags[r * kFRow8 + gl] = static_cast<uint8_t>(f);
                        if (a.results)
                            a.results[rbeg + k] = static_cast<uint8_t>(need ? (RAFTGPU_RES_OK | (old_paused ? RAFTGPU_RES_OLD_PAUSED : 0u)) : 0u);
                        done = true;
                    }
                }
                if (!done) {   // the rare kinds: onto the warp's list, handled after the loop by all its lanes together
                    const uint32_t at = atomicAdd(&s_ndefer[warp], 1u);
                    if (at < kFDefer)
                        my_defer[at] = k;
                    else
                        slow_record(k);  // the list is full: here and now (correct, only slower)
                }
            }
            __syncwarp();
            {
                const uint32_t nd = s_ndefer[warp] < kFDefer ? s_ndefer[warp] : kFDefer;
                for (uint32_t j = lane; j < nd; j += 32) slow_record(my_defer[j]);
            }
            named_bar_sync(bar_id, kCT);
            if (a.dbg && tid == 0) t2 = clock64();

            // ---- B: Raft::maybe_commit for the tile's groups (raft.rs:893-904)
            if (tid < kFTile && !(a.skip & 2u)) {  // warp-uniform: kFTile is a multiple of 32
                const uint32_t gl = tid;
                const bool active = gl < ng;
                const uint32_t g = g0 + gl;
                bool advanced = false;
                if (active) {
                    const uint32_t meta = s_meta[gl];
                    uint64_t v[kSlots];
                    uint32_t r = 0;
#pragma unroll
                    for (int s2 = 0; s2 < kSlots; s2++) {
                        v[s2] = 0;
                        if ((hint >> s2) & 1u) {
                            v[s2] = s_matched[r * R64 + gl];
                            r++;
                        }
                    }
                    uint64_t mci;
                    bool use_gc;
                    eval_mci<kSimple5>(c, g, meta, v, hint, mci, use_gc);
                    advanced = mci > s_committed[gl] && mci >= s_ts[gl] && mci <= s_li[gl];  // raft_log.rs:488
                    if (advanced) {
                        s_committed[gl] = mci;  // (the store warp copies the row to commit_out too)
                        if (meta & RAFTGPU_META_HAS_SELF) {  // raft.rs:896-900
                            const uint32_t self = RAFTGPU_META_SELF(meta);
                            uint64_t *pc = ((hint >> self) & 1u)
                                               ? &s_pc[__popc(hint & ((1u << self) - 1u)) * R64 + gl]
                                               : &c.peer_committed[static_cast<size_t>(self) * c.cap + g];
                            if (mci > *pc) *pc = mci;
                        }
                    }
                }
                uint32_t lc[2] = {0, 0};
                publish_tile(a.adv_bitmap, static_cast<uint64_t>(g0) + gl, lane, active, advanced, lc);
                local[5] += lc[0];
                local[6] += lc[1];
            }

            // ---- C: hand the stage to the store warp (generic writes -> async proxy: fence, then signal)
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            named_bar_sync(bar_id, kCT);
            if (a.dbg && tid == 0) t3 = clock64();
            if (tid == 0) mbar_arrive(&done_bar[st]);
            if (kFRecCap == 0 && tile + tile_step < n_tiles) {  // direct records: next tile's range -> L2 (one line = 8 records)
                const uint32_t nn = nx_end - nx_beg;
                for (uint32_t k = tid * 8u; k < nn; k += kCT * 8u) prefetch_l2(a.recs + nx_beg + k);
            }
            if (a.dbg && tid == 0) {
                t4 = clock64();
                atomicAdd(&a.dbg[0], static_cast<unsigned long long>(t1 - t0));  // waiting for the TMA loads
                atomicAdd(&a.dbg[1], static_cast<unsigned long long>(t2 - t1));  // A: records
                atomicAdd(&a.dbg[2], static_cast<unsigned long long>(t3 - t2));  // B: recompute (+ fence, barrier)
                atomicAdd(&a.dbg[3], static_cast<unsigned long long>(t4 - t3));  // C: stores + drain
                atomicAdd(&a.dbg[4], 1ull);                                       // tiles
            }
        }
    }
    const int which[7] = {kCntRecords, kCntUpdates, kCntRejects, kCntDecrements, kCntNoProgress, kCntRecomputes, kCntAdvanced};
    block_flush_counts<7>(local, which, a.counters, nullptr);
    if (a.step_advanced) {
        const uint32_t w = __reduce_add_sync(0xffffffffu, local[6]);
        if (lane == 0 && w) atomicAdd(a.step_advanced, w);
    }
}
