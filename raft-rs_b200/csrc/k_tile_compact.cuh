// k_tile_compact.cuh -- step_tile_compact_kernel (+ its tile index kernels): the fused step on the compact stream.
// Part of kernels.cuh (included there, inside namespace raftgpu; not a standalone header).

// step_tile_compact_kernel: the fused step for a TILEABLE compact stream (groups ascending, every
// run headed -- raftgpu_compact_hdr.flags & RAFTGPU_COMPACT_TILEABLE).  Same producer / store
// warps and stage ring (TileRing, k_tile.cuh) as step_tile_kernel; the consumers work per GROUP instead of per record:
//   0. a unit-parallel pre-pass finds, for every group of the tile, the first unit of its first
//      run (shared-memory atomicMin on the run headers),
//   1. thread gl then walks the runs of group g0+gl SEQUENTIALLY -- header decoded once, each
//      record a handful of instructions against the shared-memory cells -- so the records of one
//      cell apply in stream order (no one-wave restriction) and
//   2. goes straight on to the group's Raft::maybe_commit: its cells were written by this very
//      thread, so no barrier separates apply and recompute.
// Against the per-record form this is ~2.5x fewer warp instructions per tile (no per-record
// header/cell address arithmetic, no three-way divergence on the record kind) and a third of the
// record bytes.  tile_off[t] = unit position of the first run header of tile t.
struct CTileArgs {
    TileRingArgs r;
    CompactSrc src;
    const uint2 *tile_gb;      // [n_tiles]: g_base of the unit block tile t starts in, and of the next block
    uint32_t *dup_count;       // nullable (!kOrdered): bumped for a second record on one cell, which is not applied
};

// kOrdered: per-group walk (records of a cell apply in stream order; any number per cell).
// !kOrdered: one thread per unit (faster; at most one record per (group, peer) cell per batch --
// checked on the fly in a shared-memory bitmap when a.dup_count is given).
template <bool kSimple5, bool kOrdered>
__global__ void __launch_bounds__(kFThreads, 1) step_tile_compact_kernel(Columns c, CTileArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) TileBarriers bars;

    const TileRing<kSimple5, kCUnitCap> ring(a.r, &bars, smem);
    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t hint = ring.hint;
    uint32_t *s_run_all = reinterpret_cast<uint32_t *>(ring.extra());
    if (threadIdx.x < kFGroups * kFTile) s_run_all[threadIdx.x] = kOrdered ? 0xffffffffu : 0u;
    ring.init_barriers();

    uint32_t local[7] = {0, 0, 0, 0, 0, 0, 0};
    if (warp == kFGroups * kFTile / 32 + 1) {
        ring.store_warp(c);
    } else if (warp == kFGroups * kFTile / 32) {
        ring.load_warp(c, a.src.units);
    } else {
        // ===================== consumers: thread gl of group cg owns group g0 + gl of its tiles =====================
        const uint32_t cg = warp / (kFTile / 32);
        const uint32_t tid = threadIdx.x % kFTile;
        const int bar_id = 1 + static_cast<int>(cg);
        uint32_t *s_run = s_run_all + cg * kFTile;
        TileCursor t = ring.first(cg);
        // the g_base words of this consumer group's NEXT tile are fetched during the current one
        // (tile_gb[t] = the g_base words of the two unit blocks tile t starts in)
        uint2 nx_gb = t.tile < ring.n_tiles ? a.tile_gb[t.tile] : make_uint2(0u, 0u);
        for (; t.tile < ring.n_tiles; ring.next(t)) {
            const uint32_t g0 = t.tile * kFTile;
            const uint32_t ng = ring.groups_of(g0);
            const uint32_t gb0 = nx_gb.x, gb1 = nx_gb.y;
            if (t.tile + ring.tile_step() < ring.n_tiles) nx_gb = a.tile_gb[t.tile + ring.tile_step()];
            const uint32_t ua = t.u0 & ~3u;
            const uint32_t lead = t.u0 - ua, cnt = t.u1 - ua;  // local unit positions [lead, cnt)
            const uint32_t staged = ring.staged_units(t.u0, t.u1);
            const uint32_t *g_units = a.src.units + ua;
            const uint32_t blk0 = ua / RAFTGPU_COMPACT_BLOCK;
            const TileRows s = ring.wait(t);
            const uint32_t *s_units = s.units;

            // ---- 0: first run header of every group of the tile.  The g_base words of the (at most
            // two, unless the tile is crowded) unit blocks the tile spans were fetched before the wait.
            auto group_of = [&](uint32_t p, uint32_t hb) -> uint32_t {
                const uint32_t blk = (ua + p) / RAFTGPU_COMPACT_BLOCK;
                const uint32_t gb = blk == blk0 ? gb0 : (blk == blk0 + 1u ? gb1 : a.src.g_base[blk]);
                return gb + ((hb >> 2) & 0xfffu);
            };
            const uint32_t gl = tid;
            const bool active = gl < ng;
            const uint32_t g = g0 + gl;
            if constexpr (kOrdered) {
                for (uint32_t p = lead + tid; p < cnt; p += kFTile) {
                    const uint32_t u = p < staged ? s_units[p] : g_units[p];
                    const uint32_t kind = u & 3u;
                    if (kind == kCuEsc) {  // a side-table record: start pulling it towards L1 for the walk below
                        const uint32_t k = u >> 2;
                        if (k < kCuPad && k < a.src.n_side) {
                            asm volatile("prefetch.global.L1 [%0];" ::"l"(a.src.side + k));
                            asm volatile("prefetch.global.L1 [%0];" ::"l"(reinterpret_cast<const uint8_t *>(a.src.side + k) + 40));
                        }
                        continue;
                    }
                    if (kind != kCuHdrA || p + 1u >= cnt) continue;
                    const uint32_t hb = p + 1u < staged ? s_units[p + 1u] : g_units[p + 1u];
                    if ((hb & 3u) != kCuHdrB) continue;
                    const uint32_t gt = group_of(p, hb) - g0;
                    if (gt < ng) atomicMin(&s_run[gt], p);
                }
                named_bar_sync(bar_id, kFTile);

                // ---- 1: the runs of group g, record by record (raft.rs:1663-1743)
                uint32_t p = s_run[gl];
                s_run[gl] = 0xffffffffu;  // ready for this consumer group's next tile
                if (active && p != 0xffffffffu) {
                    const uint32_t present_mask = kSimple5 ? 0x1fu : present_of(s.meta[gl]);
                    uint64_t base = 0;
                    while (p < cnt) {
                        const uint32_t u = p < staged ? s_units[p] : g_units[p];
                        const uint32_t kind = u & 3u;
                        if (kind == kCuHdrA) {  // a run header: ours (the first, or a continuation) or the next group's
                            if (p + 1u >= cnt) break;
                            const uint32_t hb = p + 1u < staged ? s_units[p + 1u] : g_units[p + 1u];
                            if ((hb & 3u) != kCuHdrB) break;
                            if (group_of(p, hb) != g) break;
                            base = static_cast<uint64_t>(u >> 2) | (static_cast<uint64_t>(hb >> 14) << 30);
                            p += 2u;
                            continue;
                        }
                        if (kind == kCuHdrB) break;  // malformed
                        uint32_t res = 0;
                        RecRegs rec;
                        uint64_t ext_hint = 0, ext_snapshot = RAFTGPU_INVALID_INDEX;
                        bool general = false;
                        uint32_t step = 1;
                        if (kind == kCuRec) {
                            const uint32_t slot = (u >> 6) & 7u;
                            const uint64_t index = base + ((u >> 10) & 0x3fffu);
                            const uint32_t cd = u >> 24;
                            const bool is_local = (u & kCuLocal) != 0;
                            const bool is_reject = (u & kCuReject) != 0;
                            const uint64_t commit = is_local ? (cd == kCuNoCommit ? 0 : index + cd) : (index >= cd ? index - cd : 0);
                            if (is_reject && p + 1u < cnt) {  // its hint rides in the next unit
                                const uint32_t pl = p + 1u < staged ? s_units[p + 1u] : g_units[p + 1u];
                                if ((pl & 3u) == kCuEsc && ((pl >> 2) & kCuPayload)) {
                                    ext_hint = compact_hint(index, pl);
                                    step = 2;
                                }
                            }
                            const bool fast = tile_fast_apply<kSimple5>(c, s, gl, g, slot, index, commit, is_local, is_reject, ext_hint,
                                                                        hint, present_mask, local, res);
                            if (!fast) {
                                general = true;
                                rec.w0 = static_cast<uint64_t>(g) | (static_cast<uint64_t>(slot) << 32) |
                                         (static_cast<uint64_t>(is_reject ? RAFTGPU_REC_REJECT : (is_local ? RAFTGPU_REC_LOCAL : 0u)) << 40);
                                rec.index = index;
                                rec.commit = commit;
                            }
                        } else {  // ESC: the full record sits in the side table (a stray payload unit: nothing)
                            const uint32_t k = u >> 2;
                            if (k == kCuPad) break;  // padding only ever follows the last run of a slice
                            if (k < kCuPad && k < a.src.n_side) {
                                const uint64_t *sp = reinterpret_cast<const uint64_t *>(a.src.side + k);
                                rec.w0 = sp[0];
                                rec.index = sp[1];
                                rec.commit = sp[2];
                                if ((rec.w0 >> 40) & RAFTGPU_REC_EXT) {
                                    // a continuation by itself carries nothing
                                } else if (static_cast<uint32_t>(rec.w0) != g) {  // not this run's group: the stream lied
                                    local[0]++;
                                    local[4]++;
                                    res = RAFTGPU_RES_NO_PROGRESS;
                                } else {
                                    general = true;
                                    if ((rec.w0 >> 40) & RAFTGPU_REC_REJECT)
                                        load_reject_ext<false>(a.src.side, k, a.src.n_side, ext_hint, ext_snapshot);
                                }
                            }
                        }
                        if (general) res = tile_general_apply(c, rec, ext_hint, ext_snapshot, gl, hint, s, local);
                        if (a.r.results) a.r.results[ua + p] = static_cast<uint8_t>(res);
                        p += step;
                    }
                }
            } else {
                // ---- 1': one thread per unit; a record finds its run header `back` units behind it
                uint32_t *s_touch = s_run;  // 2048 bits: (group, peer slot) cells seen in this tile
                for (uint32_t k = lead + tid; k < cnt; k += kFTile) {
                    const uint32_t u = k < staged ? s_units[k] : g_units[k];
                    const uint32_t kind = u & 3u;
                    if (kind == kCuHdrA || kind == kCuHdrB) continue;
                    uint32_t res = 0, gt = 0, slot = 0;
                    RecRegs rec;
                    uint64_t ext_hint = 0, ext_snapshot = RAFTGPU_INVALID_INDEX;
                    bool general = false, fast_ok = false, is_local = false, is_reject = false;
                    if (kind == kCuRec) {
                        const uint32_t back = (u >> 3) & 7u;
                        if (k < lead + back + 2u) continue;  // malformed
                        const uint32_t hp = k - back - 2u;
                        const uint32_t ha = hp < staged ? s_units[hp] : g_units[hp];
                        const uint32_t hb = hp + 1u < staged ? s_units[hp + 1u] : g_units[hp + 1u];
                        if ((ha & 3u) != kCuHdrA || (hb & 3u) != kCuHdrB) continue;
                        gt = group_of(hp, hb) - g0;
                        slot = (u >> 6) & 7u;
                        rec.index = (static_cast<uint64_t>(ha >> 2) | (static_cast<uint64_t>(hb >> 14) << 30)) + ((u >> 10) & 0x3fffu);
                        const uint32_t cd = u >> 24;
                        is_local = (u & kCuLocal) != 0;
                        is_reject = (u & kCuReject) != 0;
                        rec.commit = is_local ? (cd == kCuNoCommit ? 0 : rec.index + cd) : (rec.index >= cd ? rec.index - cd : 0);
                        if (is_reject && k + 1u < cnt) {  // its hint rides in the next unit
                            const uint32_t pl = k + 1u < staged ? s_units[k + 1u] : g_units[k + 1u];
                            if ((pl & 3u) == kCuEsc && ((pl >> 2) & kCuPayload)) ext_hint = compact_hint(rec.index, pl);
                        }
                        rec.w0 = static_cast<uint64_t>(g0 + gt) | (static_cast<uint64_t>(slot) << 32) |
                                 (static_cast<uint64_t>(is_reject ? RAFTGPU_REC_REJECT : (is_local ? RAFTGPU_REC_LOCAL : 0u)) << 40);
                        fast_ok = true;
                    } else {  // ESC: the full record sits in the side table (payload units / padding: nothing)
                        const uint32_t k2 = u >> 2;
                        if (k2 >= kCuPad || k2 >= a.src.n_side) continue;
                        const uint64_t *sp = reinterpret_cast<const uint64_t *>(a.src.side + k2);
                        rec.w0 = sp[0];
                        rec.index = sp[1];
                        rec.commit = sp[2];
                        if ((rec.w0 >> 40) & RAFTGPU_REC_EXT) continue;  // a continuation by itself carries nothing
                        gt = static_cast<uint32_t>(rec.w0) - g0;
                        slot = static_cast<uint32_t>(rec.w0 >> 32) & 0xffu;
                        if ((rec.w0 >> 40) & RAFTGPU_REC_REJECT)
                            load_reject_ext<false>(a.src.side, k2, a.src.n_side, ext_hint, ext_snapshot);
                    }
                    if (gt >= ng) {  // not this tile's group: the stream lied
                        local[0]++;
                        local[4]++;
                        res = RAFTGPU_RES_NO_PROGRESS;
                    } else {
                        bool dup = false;
                        if (a.dup_count && slot < kSlots) {
                            const uint32_t bit = 1u << (8u * (gt & 3u) + slot);
                            dup = (atomicOr(&s_touch[gt >> 2], bit) & bit) != 0;
                            if (dup) atomicAdd(a.dup_count, 1u);
                        }
                        if (!dup) {
                            const uint32_t present_mask = kSimple5 ? 0x1fu : present_of(s.meta[gt]);
                            general = !(fast_ok && tile_fast_apply<kSimple5>(c, s, gt, g0 + gt, slot, rec.index, rec.commit, is_local,
                                                                             is_reject, ext_hint, hint, present_mask, local, res));
                            if (general) res = tile_general_apply(c, rec, ext_hint, ext_snapshot, gt, hint, s, local);
                        }
                    }
                    if (a.r.results) a.r.results[ua + k] = static_cast<uint8_t>(res);
                }
                named_bar_sync(bar_id, kFTile);
                if (a.dup_count && tid < kFTile / 4) s_touch[tid] = 0;  // clean for this consumer group's next tile
            }
            __syncwarp();

            // ---- 2: Raft::maybe_commit for this thread's group: its cells were written by this very thread (ordered)
            // or are final after the barrier above; then the stage goes to the store warp
            ring.finish(c, t, s, local);
        }
    }
    ring.flush(local);
}

// Tile index of a tileable compact stream, on the device (the zero-copy step has no host pass
// over the units): tile_off[t] = position of the first run header whose group is >= t * kFTile.
// One thread per unit; a header finds the previous run's group by looking back over at most one
// run (2 + 8 units).  *bad is bumped when groups do not ascend or an ESC unit has no run.
__global__ void __launch_bounds__(256)
compact_tile_index_kernel(CompactSrc src, uint32_t n_groups, uint32_t *__restrict__ tile_off, uint32_t *__restrict__ bad) {
    const uint32_t n_tiles = (n_groups + kFTile - 1) / kFTile;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < src.n_units; i += stride) {
        const uint32_t u = src.units[i];
        if ((u & 3u) == kCuEsc && (u >> 2) < kCuPad) {  // a side-table record must sit inside a run
            bool headed = false;
            for (uint32_t b = 1; b <= 8u && b <= i; b++) {
                const uint32_t k = src.units[i - b] & 3u;
                if (k == kCuHdrB) {
                    headed = true;
                    break;
                }
            }
            if (!headed) atomicAdd(bad, 1u);
            continue;
        }
        if ((u & 3u) != kCuHdrA || i + 1 >= src.n_units) continue;
        const uint32_t hb = src.units[i + 1];
        if ((hb & 3u) != kCuHdrB) continue;
        const uint32_t g = src.g_base[i / RAFTGPU_COMPACT_BLOCK] + ((hb >> 2) & 0xfffu);
        // previous run header, if any: at most one run (2 + 8 units) back, not counting the padding
        // that fills a staging slice up to its block boundary (raftgpu_step_begin_records)
        bool have_prev = false;
        uint32_t gp = 0;
        for (uint32_t b = 2, real = 0; b <= i && real <= 10u; b++) {
            const uint32_t ua = src.units[i - b];
            if (ua == (kCuEsc | (kCuPad << 2))) continue;
            real++;
            if ((ua & 3u) == kCuHdrA && (src.units[i - b + 1] & 3u) == kCuHdrB) {
                gp = src.g_base[(i - b) / RAFTGPU_COMPACT_BLOCK] + ((src.units[i - b + 1] >> 2) & 0xfffu);
                have_prev = true;
                break;
            }
        }
        if (!have_prev) {  // the first run of the stream: everything before it must be padding
            for (uint32_t b = 1; b <= i && b <= 12u; b++)
                if (src.units[i - b] != (kCuEsc | (kCuPad << 2))) {
                    atomicAdd(bad, 1u);
                    break;
                }
        }
        if (have_prev && gp > g) atomicAdd(bad, 1u);       // groups must ascend
        if (g >= n_groups) {
            atomicAdd(bad, 1u);
            continue;
        }
        const uint32_t t_hi = g / kFTile;
        const uint32_t t_lo = have_prev ? (gp / kFTile) + 1u : 0u;  // tiles (prev tile, this tile] start here
        if (!have_prev || gp / kFTile != t_hi)
            for (uint32_t t2 = t_lo; t2 <= t_hi; t2++) tile_off[t2] = i;
    }
    // tiles behind the last run are filled by the host-side launch (tile_off pre-set to n_units)
    (void)n_tiles;
}

// tile_gb[t] = the g_base words of the unit block tile t's (16-byte aligned) first unit lies in and of
// the block after it, so that the fused kernel decodes group ids without dependent global loads.
__global__ void __launch_bounds__(256)
compact_tile_gb_kernel(CompactSrc src, uint32_t n_tiles, const uint32_t *__restrict__ tile_off, uint2 *__restrict__ tile_gb) {
    const uint32_t n_blk = (src.n_units + RAFTGPU_COMPACT_BLOCK - 1) / RAFTGPU_COMPACT_BLOCK;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n_tiles; t += gridDim.x * blockDim.x) {
        const uint32_t blk0 = (tile_off[t] & ~3u) / RAFTGPU_COMPACT_BLOCK;
        tile_gb[t] = make_uint2(blk0 < n_blk ? src.g_base[blk0] : 0u, blk0 + 1u < n_blk ? src.g_base[blk0 + 1u] : 0u);
    }
}
