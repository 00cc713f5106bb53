// k_tile.cuh -- the stage ring of the fused tile kernels, and step_tile_kernel: the fused apply + recompute tile
// kernel on packed records (the headline kernel).
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).

// ---------------------------------------------------------------------------
// The fused tile kernels: apply + recompute FUSED, for batches whose records are in group order.
//
// The scatter apply kernel above keeps many loads in flight but stays far below the HBM peak: its cell
// accesses are sector-granular (8 useful bytes per 32-byte sector request, several rows per
// record), which HBM serves at roughly half the efficiency of dense bursts.  When the batch is
// ordered by group, a tile of kFTile consecutive groups owns a CONTIGUOUS record range, so the
// whole step becomes dense traffic.  One CTA per SM runs a ring of shared-memory stages:
//   - the load warp bulk-loads (TMA, cp.async.bulk) the tile's rows of matched / the next_idx and
//     committed_index offsets / pflags / meta / committed / term_start / last_index, plus an optional
//     payload (the compact kernel's units), into one stage;
//   - consumer group i % kFGroups takes the CTA's tile i, so the phases of kFGroups tiles overlap:
//     it applies the tile's records to the shared-memory rows (the kernel's own body; the packed kernel's
//     records arrive in a double buffer of the consumer group's own, outside the ring), then
//     recomputes the commit index of the tile's groups from the same rows (matched is read from
//     HBM once per step instead of twice);
//   - the store warp bulk-stores the rows back (cp.async.bulk.global.shared::cta).
// Peer slots outside `hint` (learners), the cold columns and the offset escapes are handled through HBM directly.
// tile_off[t] = index of the first record (packed kernel) or unit (compact kernel) of tile t.
constexpr int kFTile = RAFTGPU_TILE_GROUPS;  // groups per tile = threads per consumer group
constexpr int kFGroups = 3;                  // consumer groups per CTA
constexpr int kFThreads = kFTile * kFGroups + 64;  // + the load warp and the store warp
static_assert(kFTile % 32 == 0 && kFThreads <= 1024, "a consumer group is whole warps, one thread per group of its tile");
constexpr int kFMaxStages = 8;
// Row strides inside a stage.  Records arrive in group order, so the ~3.5 records of one group sit
// in neighbouring lanes and touch the SAME column index of DIFFERENT rows: with a 256-element row
// stride they would all fall on the same shared-memory banks (4-way conflicts on every access).
// 258 u64 (= 2064 B, still 16-byte aligned for TMA) shifts consecutive rows by 4 banks.
constexpr uint32_t kFRow64 = (kFTile + 2) * 8;   // bytes per u64 row
// bytes per 16-bit offset row (next_d, pc_d): 264 elements, 16-byte aligned too, consecutive rows 4 banks apart
constexpr uint32_t kFRow16 = (kFTile + 8) * 2;
constexpr uint32_t kFRow8 = kFTile + 16;         // bytes per u8 (pflags) row
constexpr uint32_t kFDefer = 32;                 // deferred (rare-path) records per warp per tile; more are handled inline
// dynamic shared memory of the fused kernels: 227 KB per CTA minus their static shared memory (barriers, deferred lists)
constexpr uint32_t kFSmem = 227u * 1024u - 5u * 1024u;

// bytes of one stage for H hinted slots and a payload of payload_bytes (shared by host and device)
__host__ __device__ constexpr uint32_t tile_stage_bytes(uint32_t H, uint32_t payload_bytes) {
    return H * kFRow64 + 2u * H * kFRow16 + 3u * kFRow64 + kFTile * 4u + H * kFRow8 + payload_bytes;
}
// The stage count of both fused kernels: the most stages, at most kFMaxStages, that fit in kFSmem
// beside extra_bytes of other dynamic shared memory.
__host__ __device__ constexpr int tile_stages(uint32_t H, uint32_t payload_bytes, uint32_t extra_bytes) {
    const uint32_t fit = (kFSmem - extra_bytes) / tile_stage_bytes(H, payload_bytes);
    return fit < static_cast<uint32_t>(kFMaxStages) ? static_cast<int>(fit) : kFMaxStages;
}
// The compact kernel stages up to kCUnitCap 4-byte units per tile (the rest of a crowded tile is read from HBM) and
// keeps one u32 run index per group of each consumer group behind the stages.
constexpr uint32_t kCUnitCap = 1536;
constexpr uint32_t kCRunBytes = kFGroups * kFTile * 4u;
// The packed kernel copies up to kRecCap packed records of a tile into shared memory (the rest of a crowded tile is
// read from HBM): two buffers per consumer group behind the stages, one for its current tile and one that its next
// tile's records land in meanwhile.  (bench.py's cfg3 stream, 1M groups × 5 peers, has 910 ± 22 records per tile, at
// most 991; cfg4's, 7 slots under joint consensus, 1 172 ± 32, at most 1 287: a larger cap would cost it a stage.)
constexpr uint32_t kRecCap = 4u * kFTile;
constexpr uint32_t kRecBytes = kFGroups * 2u * kRecCap * 16u;
// Every hint width leaves a stage per consumer group (wait_stage relies on it) ...
static_assert(tile_stages(kSlots, 0, kRecBytes) >= kFGroups && tile_stages(kSlots, kCUnitCap * 4u, kCRunBytes) >= kFGroups,
              "a stage per consumer group");
// ... and with 256-group tiles the plans for H = 1..8 hinted slots are
static_assert(kFTile != 256 || (tile_stages(1, 0, kRecBytes) == 8 && tile_stages(2, 0, kRecBytes) == 8 &&
                                tile_stages(3, 0, kRecBytes) == 7 && tile_stages(4, 0, kRecBytes) == 6 &&
                                tile_stages(5, 0, kRecBytes) == 5 && tile_stages(6, 0, kRecBytes) == 4 &&
                                tile_stages(7, 0, kRecBytes) == 4 && tile_stages(8, 0, kRecBytes) == 3),
              "packed kernel: 24 176 B per stage at H = 5, beside 96 KB of record buffers");
static_assert(kFTile != 256 || (tile_stages(1, kCUnitCap * 4u, kCRunBytes) == 8 && tile_stages(2, kCUnitCap * 4u, kCRunBytes) == 8 &&
                                tile_stages(3, kCUnitCap * 4u, kCRunBytes) == 8 && tile_stages(4, kCUnitCap * 4u, kCRunBytes) == 8 &&
                                tile_stages(5, kCUnitCap * 4u, kCRunBytes) == 7 && tile_stages(6, kCUnitCap * 4u, kCRunBytes) == 6 &&
                                tile_stages(7, kCUnitCap * 4u, kCRunBytes) == 6 && tile_stages(8, kCUnitCap * 4u, kCRunBytes) == 5),
              "compact kernel: 30 320 B per stage at H = 5");
static_assert(kFTile != 256 || (tile_stage_bytes(5, 0) == 24176 && tile_stage_bytes(5, kCUnitCap * 4u) == 30320), "stage sizes");

// ---- 1-D TMA and mbarrier primitives
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// 1-D TMA: global -> shared, completion counted in bytes on `bar`
__device__ __forceinline__ void tma_load_1d(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// 1-D TMA store: shared -> global, tracked by the per-thread bulk async-group
__device__ __forceinline__ void tma_store_1d(void *dst, const void *src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int n_threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n_threads) : "memory");
}
// A consumer's wait for "the loads of MY tile have landed in this stage".  A consumer group sees only every kFGroups-th
// tile, so on one stage's `full` barrier it skips phases -- and a parity wait is only exact while the waiter is at
// most ONE phase ahead.  With uniform tiles that always holds; with a batch that covers only part of the groups it
// does not (record-less tiles are done in a microsecond, loads of light and heavy tiles land out of order): a group
// could pass the barrier of a stage still armed for the PREVIOUS tile and work on half-landed rows.  So it first
// waits for the previous use of the stage to be DONE (`done` barrier, previous phase).  That wait is exact: the
// group's own previous tile was loaded, hence the tile n_stages before IT was stored, stores happen in tile order,
// and with n_stages >= kFGroups that covers the previous user of this stage; and once the previous user is done, the
// `full` barrier is in this tile's phase, so the second wait is exact too.
__device__ __forceinline__ void wait_stage(uint64_t *full_bar, uint64_t *done_bar, uint32_t parity) {
    mbar_wait(done_bar, parity ^ 1u);  // (first use of a stage: the parity-1 wait on a fresh barrier passes at once)
    mbar_wait(full_bar, parity);
}

// ---- the ring
// Kernel arguments both fused kernels share.
struct TileRingArgs {
    const uint32_t *tile_off;  // [n_tiles + 1]
    uint32_t n_groups;         // groups [0, n_groups)
    uint32_t hint;
    int n_stages;              // tile_stages(), >= kFGroups
    uint8_t *results;          // nullable, one byte per record / unit
    uint32_t *adv_bitmap;      // nullable
    uint64_t *commit_out;      // nullable
    uint32_t *step_advanced;   // nullable
    unsigned long long *counters;
    unsigned long long *dbg;   // nullable: [8] cycle totals per phase (diagnostics, RAFTGPU_TILE_DEBUG=1)
};

struct TileBarriers {
    uint64_t full[kFMaxStages];   // loads landed            (load warp -> consumers)
    uint64_t done[kFMaxStages];   // rows final in smem      (consumers -> store warp)
    uint64_t empty[kFMaxStages];  // rows read by the stores (store warp -> load warp)
    uint64_t recs[kFGroups][2];   // packed kernel: a consumer group's record buffer filled (its thread 0 -> the group)
    uint32_t clk[kFGroups];       // RAFTGPU_TILE_DEBUG: per consumer group, the end of its wait for the stage
};

// One stage's rows in shared memory.  Row r of a per-peer column is the r-th hinted slot.
struct TileRows {
    uint64_t *matched;
    int16_t *next, *pc;  // the offsets next_d / pc_d, rows kFRow16 bytes apart
    uint64_t *committed, *ts, *li;
    uint32_t *meta;
    uint8_t *flags;
    uint32_t *units;  // the payload
};
// matched and the offsets of the cell staged in row r for group gl (arena cell `cell`)
__device__ __forceinline__ HotPtrs staged_hot(const TileRows &t, uint32_t r, uint32_t gl, size_t cell) {
    return HotPtrs{&t.matched[r * (kFRow64 / 8) + gl], &t.next[r * (kFRow16 / 2) + gl], &t.pc[r * (kFRow16 / 2) + gl], cell};
}

// Where a consumer group is in its walk over the CTA's tiles.
struct TileCursor {
    uint32_t tile, it;  // the tile, and its place in the CTA's sequence of tiles (stage it % n_stages)
    uint32_t u0, u1;    // tile_off[tile], tile_off[tile + 1]
    uint32_t nx0, nx1;  // the same for this group's next tile, fetched during this one
};

// kUnitCap: 4-byte payload units staged per tile (a multiple of 4); the rest of a tile's units is read from HBM.
template <bool kSimple5, uint32_t kUnitCap>
struct TileRing {
    TileRingArgs a;
    TileBarriers *bar;
    uint8_t *smem;
    uint32_t hint, H, stage_bytes, n_tiles;

    __device__ __forceinline__ TileRing(const TileRingArgs &args, TileBarriers *b, uint8_t *dyn_smem)
        : a(args), bar(b), smem(dyn_smem) {
        hint = kSimple5 ? 0x1fu : (a.hint & 0xffu);
        H = kSimple5 ? 5u : static_cast<uint32_t>(__popc(hint));
        stage_bytes = tile_stage_bytes(H, kUnitCap * 4u);
        n_tiles = (a.n_groups + kFTile - 1) / kFTile;
    }
    __device__ __forceinline__ void init_barriers() const {
        if (threadIdx.x == 0) {
            for (int s = 0; s < a.n_stages; s++) {
                mbar_init(&bar->full[s], 1);
                mbar_init(&bar->done[s], 1);
                mbar_init(&bar->empty[s], 1);
            }
            for (int g = 0; g < kFGroups; g++) {
                mbar_init(&bar->recs[g][0], 1);
                mbar_init(&bar->recs[g][1], 1);
            }
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
    }
    // the extra dynamic shared memory behind the stages
    __device__ __forceinline__ uint8_t *extra() const { return smem + static_cast<size_t>(a.n_stages) * stage_bytes; }
    __device__ __forceinline__ uint32_t groups_of(uint32_t g0) const {
        return a.n_groups - g0 < kFTile ? a.n_groups - g0 : kFTile;
    }
    // units of [u0, u1) staged, counted from the 16-byte boundary at or below u0
    __device__ __forceinline__ static uint32_t staged_units(uint32_t u0, uint32_t u1) {
        if constexpr (kUnitCap == 0) {
            return 0u;
        } else {
            const uint32_t cnt4 = (u1 - (u0 & ~3u) + 3u) & ~3u;
            return u1 <= u0 ? 0u : (cnt4 < kUnitCap ? cnt4 : kUnitCap);
        }
    }
    __device__ __forceinline__ TileRows rows(uint32_t it) const {
        uint8_t *sb = smem + static_cast<size_t>(it % a.n_stages) * stage_bytes;
        TileRows t;
        t.matched = reinterpret_cast<uint64_t *>(sb);
        t.next = reinterpret_cast<int16_t *>(sb + H * kFRow64);
        t.pc = reinterpret_cast<int16_t *>(sb + H * (kFRow64 + kFRow16));
        t.committed = reinterpret_cast<uint64_t *>(sb + H * (kFRow64 + 2u * kFRow16));
        t.ts = t.committed + kFRow64 / 8;
        t.li = t.ts + kFRow64 / 8;
        t.meta = reinterpret_cast<uint32_t *>(t.li + kFRow64 / 8);
        t.flags = reinterpret_cast<uint8_t *>(t.meta + kFTile);
        t.units = reinterpret_cast<uint32_t *>(t.flags + H * kFRow8);
        return t;
    }
    // peer slot of the r-th hinted slot
    __device__ __forceinline__ uint32_t hinted_slot(uint32_t r) const {
        uint32_t slot = 0, seen = 0;
        for (uint32_t s2 = 0; s2 < kSlots; s2++)
            if ((hint >> s2) & 1u) {
                if (seen == r) slot = s2;
                seen++;
            }
        return slot;
    }

    // ===================== load warp: rows (and units) of the CTA's tiles into the stages =====================
    __device__ __forceinline__ void load_warp(const Columns &c, const uint32_t *units) const {
        const uint32_t lane = threadIdx.x & 31;
        const uint32_t n_copies = 4u * H + 5u;
        uint32_t it = 0;
        // the tile index of the NEXT tile is fetched while this one is being issued: a dependent global
        // load at the top of every iteration would sit on the critical path of the ring
        uint32_t nx0 = 0, nx1 = 0;
        if (kUnitCap && blockIdx.x < n_tiles) {
            nx0 = a.tile_off[blockIdx.x];
            nx1 = a.tile_off[blockIdx.x + 1];
        }
        for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, it++) {
            const int st = it % a.n_stages;
            const uint32_t ph = (it / a.n_stages) & 1u;
            const uint32_t g0 = tile * kFTile;
            const uint32_t ng16 = (groups_of(g0) + 15u) & ~15u;  // 16-byte multiples for every row; inside the padded stride
            const uint32_t u0 = nx0, u1 = nx1;
            if (kUnitCap && tile + gridDim.x < n_tiles) {
                nx0 = a.tile_off[tile + gridDim.x];
                nx1 = a.tile_off[tile + gridDim.x + 1];
            }
            const uint32_t staged = staged_units(u0, u1);
            if (lane == 0) {
                mbar_wait(&bar->empty[st], ph ^ 1u);
                mbar_expect_tx(&bar->full[st], H * ng16 * (8u + 2u + 2u + 1u) + 3u * ng16 * 8u + ng16 * 4u + staged * 4u);
            }
            __syncwarp();
            const TileRows t = rows(it);
            for (uint32_t j = lane; j < n_copies; j += 32) {
                if (j < 4u * H) {
                    const uint32_t col = j / H, r = j % H;  // col: 0 matched, 1 next_d, 2 pc_d, 3 pflags
                    const size_t cell = static_cast<size_t>(hinted_slot(r)) * c.cap + g0;
                    if (col == 0) tma_load_1d(t.matched + r * (kFRow64 / 8), c.matched + cell, ng16 * 8u, &bar->full[st]);
                    if (col == 1) tma_load_1d(t.next + r * (kFRow16 / 2), c.next_d + cell, ng16 * 2u, &bar->full[st]);
                    if (col == 2) tma_load_1d(t.pc + r * (kFRow16 / 2), c.pc_d + cell, ng16 * 2u, &bar->full[st]);
                    if (col == 3) tma_load_1d(t.flags + r * kFRow8, c.pflags + cell, ng16, &bar->full[st]);
                } else if (j == 4u * H) {
                    tma_load_1d(t.committed, c.committed + g0, ng16 * 8u, &bar->full[st]);
                } else if (j == 4u * H + 1) {
                    tma_load_1d(t.ts, c.term_start + g0, ng16 * 8u, &bar->full[st]);
                } else if (j == 4u * H + 2) {
                    tma_load_1d(t.li, c.last_index + g0, ng16 * 8u, &bar->full[st]);
                } else if (j == 4u * H + 3) {
                    tma_load_1d(t.meta, c.meta + g0, ng16 * 4u, &bar->full[st]);
                } else if (staged) {
                    tma_load_1d(t.units, units + (u0 & ~3u), staged * 4u, &bar->full[st]);
                }
            }
        }
    }

    // ===================== store warp: rows back to HBM, then the stage is free =====================
    __device__ __forceinline__ void store_warp(const Columns &c) const {
        const uint32_t lane = threadIdx.x & 31;
        const uint32_t n_out = 4u * H + 2u + (a.commit_out ? 1u : 0u);
        uint32_t it = 0;
        for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, it++) {
            const int st = it % a.n_stages;
            const uint32_t ph = (it / a.n_stages) & 1u;
            const uint32_t g0 = tile * kFTile;
            const uint32_t ng16 = (groups_of(g0) + 15u) & ~15u;
            const TileRows t = rows(it);
            mbar_wait(&bar->done[st], ph);  // every lane waits: the barrier's completion orders the consumers' writes
            for (uint32_t j = lane; j < n_out; j += 32) {
                if (j < 4u * H) {
                    const uint32_t col = j / H, r = j % H;
                    const size_t cell = static_cast<size_t>(hinted_slot(r)) * c.cap + g0;
                    if (col == 0) tma_store_1d(c.matched + cell, t.matched + r * (kFRow64 / 8), ng16 * 8u);
                    if (col == 1) tma_store_1d(c.next_d + cell, t.next + r * (kFRow16 / 2), ng16 * 2u);
                    if (col == 2) tma_store_1d(c.pc_d + cell, t.pc + r * (kFRow16 / 2), ng16 * 2u);
                    if (col == 3) tma_store_1d(c.pflags + cell, t.flags + r * kFRow8, ng16);
                } else if (j == 4u * H) {
                    tma_store_1d(c.committed + g0, t.committed, ng16 * 8u);
                } else if (j == 4u * H + 1u) {
                    tma_store_1d(c.last_index + g0, t.li, ng16 * 8u);
                } else {  // the step's commit-index output: the tile's `committed` row, one dense copy (not 8-byte scatters)
                    tma_store_1d(a.commit_out + g0, t.committed, ng16 * 8u);
                }
            }
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // shared memory has been read
            __syncwarp();
            if (lane == 0) mbar_arrive(&bar->empty[st]);
        }
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // all stores have landed
    }

    // ===================== consumers: group cg takes every kFGroups-th tile of this CTA =====================
    //   for (TileCursor t = ring.first(cg); t.tile < ring.n_tiles; ring.next(t)) {
    //       const TileRows s = ring.wait(t);  ...apply the tile's records...  ring.finish(c, t, s, local);
    //   }
    __device__ __forceinline__ uint32_t tile_step() const { return kFGroups * gridDim.x; }
    __device__ __forceinline__ TileCursor first(uint32_t cg) const {
        TileCursor t;
        t.tile = blockIdx.x + cg * gridDim.x;
        t.it = cg;
        t.u0 = t.u1 = t.nx0 = t.nx1 = 0;
        if (t.tile < n_tiles) {
            t.u0 = a.tile_off[t.tile];
            t.u1 = a.tile_off[t.tile + 1];
        }
        if (t.tile + tile_step() < n_tiles) {
            t.nx0 = a.tile_off[t.tile + tile_step()];
            t.nx1 = a.tile_off[t.tile + tile_step() + 1];
        }
        return t;
    }
    __device__ __forceinline__ void next(TileCursor &t) const {
        t.tile += tile_step();
        t.it += kFGroups;
        t.u0 = t.nx0;
        t.u1 = t.nx1;
        if (t.tile + tile_step() < n_tiles) {  // next tile of this consumer group: fetched during this one
            t.nx0 = a.tile_off[t.tile + tile_step()];
            t.nx1 = a.tile_off[t.tile + tile_step() + 1];
        }
    }
    __device__ __forceinline__ TileRows wait(TileCursor &t) const {
        const uint32_t tid = threadIdx.x % kFTile;
        const int st = t.it % a.n_stages;
        // (the phase clocks are kept in shared memory: a register live across the consumer body costs spills)
        const long long t0 = a.dbg && tid == 0 ? clock64() : 0;
        wait_stage(&bar->full[st], &bar->done[st], (t.it / a.n_stages) & 1u);
        if (a.dbg && tid == 0) {
            const long long t1 = clock64();
            bar->clk[threadIdx.x / kFTile] = static_cast<uint32_t>(t1);
            atomicAdd(&a.dbg[0], static_cast<unsigned long long>(t1 - t0));  // waiting for the TMA loads
        }
        return rows(t.it);
    }
    // Raft::maybe_commit (raft.rs:893-904) of the tile's group g0 + tid, then the stage goes to the store warp.
    __device__ __forceinline__ void finish(const Columns &c, const TileCursor &t, const TileRows &s, uint32_t (&local)[7]) const {
        constexpr uint32_t R64 = kFRow64 / 8;  // row stride in u64 elements
        const uint32_t tid = threadIdx.x % kFTile, lane = threadIdx.x & 31;
        uint32_t clk = 0;
        if (a.dbg && tid == 0) {
            clk = static_cast<uint32_t>(clock64());
            atomicAdd(&a.dbg[1], static_cast<unsigned long long>(clk - bar->clk[threadIdx.x / kFTile]));  // the records
        }
        const uint32_t g0 = t.tile * kFTile, gl = tid;
        const bool active = gl < groups_of(g0);
        const uint32_t g = g0 + gl;
        bool advanced = false;
        if (active) {
            const uint32_t meta = s.meta[gl];
            uint64_t v[kSlots];
            uint32_t r = 0;
#pragma unroll
            for (int s2 = 0; s2 < kSlots; s2++) {
                v[s2] = 0;
                if ((hint >> s2) & 1u) {
                    v[s2] = s.matched[r * R64 + gl];
                    r++;
                }
            }
            uint64_t mci;
            bool use_gc;
            eval_mci<kSimple5>(c, g, meta, v, hint, mci, use_gc);
            advanced = mci > s.committed[gl] && mci >= s.ts[gl] && mci <= s.li[gl];  // raft_log.rs:488
            if (advanced) {
                s.committed[gl] = mci;  // (the store warp copies the row to commit_out too)
                if (meta & RAFTGPU_META_HAS_SELF) {  // raft.rs:896-900
                    const uint32_t self = RAFTGPU_META_SELF(meta);
                    const size_t cell = static_cast<size_t>(self) * c.cap + g;
                    if ((hint >> self) & 1u)
                        hot_update_committed(c, staged_hot(s, __popc(hint & ((1u << self) - 1u)), gl, cell), mci);
                    else
                        hot_update_committed(c, hot_ptrs(c, cell), mci);
                }
            }
        }
        uint32_t lc[2] = {0, 0};
        publish_tile(a.adv_bitmap, static_cast<uint64_t>(g0) + gl, lane, active, advanced, lc);
        local[5] += lc[0];
        local[6] += lc[1];
        if (a.dbg && tid == 0) {
            const uint32_t now = static_cast<uint32_t>(clock64());
            atomicAdd(&a.dbg[2], static_cast<unsigned long long>(now - clk));  // recompute
            clk = now;
        }

        // hand the stage to the store warp (generic writes -> async proxy: fence, then signal)
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        named_bar_sync(1 + static_cast<int>(threadIdx.x / kFTile), kFTile);
        if (tid == 0) mbar_arrive(&bar->done[t.it % a.n_stages]);
        if (a.dbg && tid == 0) {
            atomicAdd(&a.dbg[3], static_cast<uint32_t>(clock64()) - clk);  // hand-off to the stores
            atomicAdd(&a.dbg[4], 1ull);                                               // tiles
        }
    }

    // records, updates, rejects, decrements, no_progress | recomputes, advanced
    __device__ __forceinline__ void flush(const uint32_t (&local)[7]) const {
        const int which[7] = {kCntRecords, kCntUpdates, kCntRejects, kCntDecrements, kCntNoProgress, kCntRecomputes, kCntAdvanced};
        block_flush_counts<7>(local, which, a.counters, nullptr);
        if (a.step_advanced) {
            const uint32_t w = __reduce_add_sync(0xffffffffu, local[6]);
            if ((threadIdx.x & 31) == 0 && w) atomicAdd(a.step_advanced, w);
        }
    }
};

// ---- the apply paths shared by both kernels
// A record that is not on the fast path (Snapshot state, a REJECT with a snapshot request or a hostile value, a WIDE
// commit, a peer slot outside the hint): the literal apply_one against the shared-memory cell, or against HBM for a
// slot the tile does not stage.
__device__ __forceinline__ uint32_t tile_general_apply(const Columns &c, const RecRegs &rec, uint64_t ext_hint,
                                                    uint64_t ext_snapshot, uint32_t gl, uint32_t hint,
                                                    const TileRows &t, uint32_t *local) {
    const uint32_t slot = static_cast<uint32_t>(rec.w0 >> 32) & 0xffu;
    if (slot < kSlots && ((hint >> slot) & 1u)) {
        const uint32_t r = __popc(hint & ((1u << slot) - 1u));
        const CellPtrs sp{staged_hot(t, r, gl, static_cast<size_t>(slot) * c.cap + static_cast<uint32_t>(rec.w0)), &t.li[gl],
                          &t.flags[r * kFRow8 + gl]};
        const HotVals h = hot_load(c, sp.hot);
        CellRegs cd;
        cd.meta = t.meta[gl];
        cd.matched = h.matched;
        cd.next_idx = h.next_idx;
        cd.flags = t.flags[r * kFRow8 + gl];
        cd.peer_committed = h.peer_committed;
        return apply_one<2>(c, nullptr, ext_hint, ext_snapshot, rec, cd, sp, local);
    }
    CellRegs cd = load_cell(c, rec);
    cd.meta = t.meta[gl];
    CellPtrs gp = global_cell_ptrs(c, rec);
    gp.last_index = &t.li[gl];
    return apply_one<2>(c, nullptr, ext_hint, ext_snapshot, rec, cd, gp, local);
}

// The common records -- accept, leader-local, rejection without a snapshot request -- for a peer
// in Replicate or Probe state whose cell is staged in shared memory: statement for statement the
// branches of apply_one (raft.rs:1674-1677, 1709-1730, 974-991, 1010-1014; progress.rs:95-114,
// 138-157, 168-206).  Returns false (nothing touched) when the record needs the general path, which
// includes a cell whose offsets are escaped: the exact values would be a dependent HBM load.
// `res` is left alone unless the record makes progress.
template <bool kSimple5>
__device__ __forceinline__ bool tile_fast_apply(const Columns &c, const TileRows &t, uint32_t gl, uint32_t g, uint32_t slot,
                                                uint64_t index, uint64_t commit, bool is_local, bool is_reject,
                                                uint64_t ext_hint, uint32_t hint, uint32_t present_mask, uint32_t *local,
                                                uint32_t &res) {
    constexpr uint32_t R64 = kFRow64 / 8, R16 = kFRow16 / 2;
    if (!((hint >> slot) & 1u)) return false;
    const uint32_t r = kSimple5 ? slot : static_cast<uint32_t>(__popc(hint & ((1u << slot) - 1u)));
    const uint32_t ci = r * R64 + gl, di = r * R16 + gl;
    const uint32_t f0 = t.flags[r * kFRow8 + gl];
    const uint32_t state = f0 & RAFTGPU_PF_STATE_MASK;
    const int16_t nd = t.next[di], pd = t.pc[di];
    if (!((present_mask >> slot) & 1u) || state == RAFTGPU_STATE_SNAPSHOT || off_escaped(nd) || off_escaped(pd))
        return false;
    uint64_t m = t.matched[ci];
    const uint64_t m0 = m;
    uint64_t nx = off_value(nd, m0), pc = off_value(pd, m0);
    uint32_t f = f0;
    local[0]++;
    if (is_local) {
        if (commit != 0) t.li[gl] = commit;
    } else {
        f |= RAFTGPU_PF_RECENT_ACTIVE;
        if (commit > pc) pc = commit;
    }
    if (is_reject) {  // maybe_decr_to without a snapshot request
        local[2]++;
        bool ok;
        if (state == RAFTGPU_STATE_REPLICATE) {
            ok = index > m;                              // progress.rs:173-177 stale otherwise
            if (ok) nx = m + 1;                          // :178-179
        } else if (nx == 0 || nx - 1 != index) {
            ok = false;                                  // :188-192 stale
        } else {
            nx = umin64(index, ext_hint + 1);            // :195-199
            if (nx < 1) nx = 1;
            f &= ~RAFTGPU_PF_PAUSED;                     // :204
            ok = true;
        }
        if (ok) {
            local[3]++;
            res = RAFTGPU_RES_OK | RAFTGPU_RES_SEND;
            if (state == RAFTGPU_STATE_REPLICATE) {      // raft.rs:1716-1718 become_probe
                f = (f & ~(RAFTGPU_PF_PAUSED | RAFTGPU_PF_INS_FULL | RAFTGPU_PF_STATE_MASK)) | RAFTGPU_STATE_PROBE;
                c.pending_snapshot[static_cast<size_t>(slot) * c.cap + g] = 0;
                nx = m + 1;
            }
        }
    } else {
        const bool old_paused = !is_local && (state == RAFTGPU_STATE_PROBE ? (f & RAFTGPU_PF_PAUSED) != 0
                                                                           : (f & RAFTGPU_PF_INS_FULL) != 0);
        const bool need = m < index;
        if (need) {
            m = index;
            f &= ~RAFTGPU_PF_PAUSED;
            local[1]++;
            res = RAFTGPU_RES_OK | (old_paused ? RAFTGPU_RES_OLD_PAUSED : 0u);
        }
        if (nx < index + 1) nx = index + 1;
        if (need && !is_local && state == RAFTGPU_STATE_PROBE) {
            f = (f & ~(RAFTGPU_PF_PAUSED | RAFTGPU_PF_INS_FULL | RAFTGPU_PF_STATE_MASK)) | RAFTGPU_STATE_REPLICATE;
            c.pending_snapshot[static_cast<size_t>(slot) * c.cap + g] = 0;
            nx = m + 1;
        }
    }
    hot_write_over(c, staged_hot(t, r, gl, static_cast<size_t>(slot) * c.cap + g), m0, nd, pd, HotVals{m, nx, pc});
    if (f != f0) t.flags[r * kFRow8 + gl] = static_cast<uint8_t>(f);
    return true;
}

__device__ __forceinline__ uint32_t present_of(uint32_t meta) {
    return RAFTGPU_META_IN(meta) | RAFTGPU_META_OUT(meta) | RAFTGPU_META_LEARN(meta);
}

// ---------------------------------------------------------------------------
// step_tile_kernel: the fused step on packed records in group order (tile_off from raftgpu_tile_index).
// The records do not travel through the ring.  Each consumer group owns two record buffers behind the stages: while it
// works on one tile, its thread 0 bulk-copies (cp.async.bulk) the first kRecCap records of the group's next tile into
// the other buffer, on that buffer's own mbarrier.  The apply loop then reads its records from shared memory instead
// of waiting on L2 behind the ring's traffic; the records of a crowded tile past the cap are read from HBM (and
// prefetched into L2 during the previous tile).
struct TileArgs {
    TileRingArgs r;
    const PackedRec *recs;  // packed records in group order
};

template <bool kSimple5>
__global__ void __launch_bounds__(kFThreads, 1) step_tile_kernel(Columns c, TileArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) TileBarriers bars;
    __shared__ uint32_t s_defer[32][kFDefer];  // per warp: tile-relative indexes of its rare-path records
    __shared__ uint32_t s_ndefer[32];

    const TileRing<kSimple5, 0> ring(a.r, &bars, smem);
    ring.init_barriers();
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t hint = ring.hint;

    uint32_t local[7] = {0, 0, 0, 0, 0, 0, 0};
    if (warp == kFGroups * kFTile / 32 + 1) {
        ring.store_warp(c);
    } else if (warp == kFGroups * kFTile / 32) {
        ring.load_warp(c, nullptr);
    } else {
        const uint32_t cg = warp / (kFTile / 32);
        const uint32_t tid = threadIdx.x % kFTile;
        // buffer b of this consumer group (its address is recomputed where used: a register live across the loop spills)
        auto rbuf = [&](uint32_t b) { return reinterpret_cast<ulonglong2 *>(ring.extra()) + (cg * 2u + b) * kRecCap; };
        // (thread 0 of the group) the first kRecCap records of [r0, r1) into buffer b.  Its previous contents were read
        // in the records phase of the group's tile before last, which ended in the group's barrier, and generic reads
        // are followed by an async-proxy write: fence.  A record-less tile arrives with 0 bytes, so the wait passes.
        auto fill = [&](uint32_t b, uint32_t r0, uint32_t r1) {
            const uint32_t n = r1 > r0 ? min(r1 - r0, kRecCap) : 0u;
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            mbar_expect_tx(&bars.recs[cg][b], n * 16u);
            if (n) tma_load_1d(rbuf(b), a.recs + r0, n * 16u, &bars.recs[cg][b]);
        };
        TileCursor t = ring.first(cg);
        if (tid == 0 && t.tile < ring.n_tiles) fill(0, t.u0, t.u1);
        for (; t.tile < ring.n_tiles; ring.next(t)) {
            const uint32_t g0 = t.tile * kFTile;
            const uint32_t ng = ring.groups_of(g0);
            const uint32_t rbeg = t.u0, cnt = t.u1 - t.u0;
            // the group's i-th tile reads buffer i & 1, whose barrier completes one phase per use
            const uint32_t i = t.it / kFGroups;
            if (tid == 0 && t.tile + ring.tile_step() < ring.n_tiles) fill((i + 1u) & 1u, t.nx0, t.nx1);
            const TileRows s = ring.wait(t);
            mbar_wait(&bars.recs[cg][i & 1u], (i >> 1) & 1u);
            const ulonglong2 *s_recs = rbuf(i & 1u);
            const ulonglong2 *g_recs = reinterpret_cast<const ulonglong2 *>(a.recs + rbeg);
            // every read of the tile's record j < cnt: the shared-memory copy, or HBM past the cap
            auto rec_at = [&](uint32_t j) -> ulonglong2 { return j < kRecCap ? s_recs[j] : g_recs[j]; };

            // ---- the tile's records against the shared-memory rows (raft.rs:1663-1743)
            // The main loop handles the records that make up ~98 % of the traffic -- an accept or a leader-local
            // record for a staged cell of a peer in Replicate or Probe state.  Whatever else turns up (a rejection, a
            // WIDE commit, a Snapshot-state peer, a learner outside the hint, a record that is not this tile's) is put
            // on the WARP's deferred list and handled after the loop with all the warp's lanes working on such records
            // at once, instead of one lane at a time inside the loop (half of all warp-iterations contain a
            // rejection): a wave has at most one record per cell, so the order between the two passes does not matter.
            uint32_t *my_defer = s_defer[warp];
            if (lane == 0) s_ndefer[warp] = 0;
            __syncwarp();
            auto slow_record = [&](const uint32_t k) {
                const RecRegs rec = load_packed_rec(rec_at, k, cnt);
                const uint64_t w0 = rec_at(k).x;
                const uint32_t gl = static_cast<uint32_t>(rec.w0) - g0;
                uint32_t res = 0;
                if (gl >= ng) {  // not this tile's group: the batch is not in group order / bad index
                    local[0]++;
                    local[4]++;
                    res = RAFTGPU_RES_NO_PROGRESS;
                } else {
                    // (the loop above has taken every accept and leader-local record the fast path can take)
                    uint64_t ext_hint = 0, ext_snapshot = RAFTGPU_INVALID_INDEX;
                    const bool is_reject = (w0 & kPkReject) != 0;
                    if (is_reject) load_packed_reject_ext(rec_at, k, cnt, ext_hint, ext_snapshot);
                    const bool fast = is_reject && !(w0 & kPkWide) && ext_snapshot == RAFTGPU_INVALID_INDEX &&
                                      tile_fast_apply<kSimple5>(c, s, gl, g0 + gl, static_cast<uint32_t>(rec.w0 >> 32) & 7u,
                                                                rec.index, rec.index - (w0 >> 40), false, true, ext_hint, hint,
                                                                kSimple5 ? 0x1fu : present_of(s.meta[gl]), local, res);
                    if (!fast) res = tile_general_apply(c, rec, ext_hint, ext_snapshot, gl, hint, s, local);
                }
                if (a.r.results) a.r.results[rbeg + k] = static_cast<uint8_t>(res);
            };
            for (uint32_t k = tid; k < cnt; k += kFTile) {
                const ulonglong2 q = rec_at(k);
                const uint64_t w0 = q.x;
                if (w0 & kPkExt) {
                    if (a.r.results) a.r.results[rbeg + k] = 0;
                    continue;
                }
                const uint32_t slot = static_cast<uint32_t>(w0 >> 32) & 7u;
                const uint32_t gl = static_cast<uint32_t>(w0) - g0;
                const uint32_t delta = static_cast<uint32_t>(w0 >> 40);
                const bool is_local = (w0 & kPkLocal) != 0;
                const uint64_t commit = is_local ? (delta == kPkNoCommit ? 0 : q.y + delta) : q.y - delta;
                uint32_t res = 0;
                if (!(w0 & (kPkWide | kPkReject)) && gl < ng &&
                    tile_fast_apply<kSimple5>(c, s, gl, g0 + gl, slot, q.y, commit, is_local, false, 0, hint,
                                              kSimple5 ? 0x1fu : present_of(s.meta[gl]), local, res)) {
                    if (a.r.results) a.r.results[rbeg + k] = static_cast<uint8_t>(res);
                } else {  // the rare kinds: onto the warp's list, handled after the loop by all its lanes together
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
            // the group's cells are final, and its record buffer is read: thread 0 may fill it again
            named_bar_sync(1 + static_cast<int>(cg), kFTile);

            ring.finish(c, t, s, local);
            if (t.tile + ring.tile_step() < ring.n_tiles) {  // next tile's records past the cap -> L2 (one line = 8 records)
                const uint32_t nn = t.nx1 - t.nx0;
                for (uint32_t k = kRecCap + tid * 8u; k < nn; k += kFTile * 8u) prefetch_l2(a.recs + t.nx0 + k);
            }
        }
    }
    ring.flush(local);
}
