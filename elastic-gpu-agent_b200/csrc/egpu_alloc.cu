// egpu_alloc.cu — best-fit fractional-GPU allocation on H100 (sm_90a) + its C ABI.
//
// Product path.  There is no CPU fallback in this file and nothing here
// includes or links oracle/: when no CUDA device is usable every entry point
// returns EGPU_ERR_NO_DEVICE.
//
// Reference slot this fills: baseDevicePlugin.GetPreferredAllocation, an empty
// stub in elastic-ai/elastic-gpu-agent (pkg/plugins/base.go:94-96); units from
// pkg/common/const.go:4 and pkg/plugins/gpushare.go:24-33,159-168.  The decision
// rule is the builder-defined spec of DESIGN.md §2 (the reference has none).
#include "egpu_kernels.cuh"

#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <mutex>
#include <new>
#include <vector>

#include "../../include/egpu_alloc.h"

#include "egpu_scan.cuh"
#include "egpu_replay.cuh"

// =============================================================================
// Host side: context + C ABI
// =============================================================================
using namespace egpu;

#include "egpu_ctx.h"

namespace {

constexpr int64_t kMaxRows = (1ll << 31) - 1;  // EGPU_MAX_ROWS

int d_bucket(int D) { return D <= 8 ? 0 : D <= 16 ? 1 : D <= 32 ? 2 : 3; }

RowFormat row_format(int flags) { return (flags & EGPU_F_PACKED) ? kRowsPacked : kRowsInt32; }

// ---- kernel tables: one kernel per family, row format and D bucket ----
template <class Fn>
struct Kernel {
    Fn fn;
    int threads;
    size_t smem;  // dynamic shared memory
    int slot;     // its entry in egpu_ctx::ctas_per_sm
};
template <class Fn>
constexpr Kernel<Fn> kernel(Fn fn, int threads, size_t smem) { return {fn, threads, smem, 0}; }

// Kernel of family F for rows in format FMT in bucket B.  The register scans run 256 threads up to D = 32 and 128 at
// D = 64; the lookup scan is one kernel for every D.  Packed rows run in the packed twin of a scan (P ? twin : int32
// kernel): same CTA size, shared memory and kernel type.  The grid scan reads int32 rows only, the warp-chunk scan
// (kScanPacked) packed words only.  The one-launch kernels run kRoundsThreads per CTA in every bucket, with the register
// scan's SnapSmem or the lookup scan's LutSmem of that CTA size.  The release kernels reuse the register scans' CTA sizes
// and lane-private accumulators at every D (DESIGN.md 4.1h); the sharded one's last CTA exchanges the sums with the
// peers before it decides.
template <int F, RowFormat FMT, int B>
constexpr auto family_kernel() {
    constexpr int DT = 8 << B, T = B == 3 ? 128 : 256, RT = kRoundsThreads;
    constexpr size_t snap = sizeof(SnapSmem<DT, T>), lut = sizeof(LutSmem<256>);
    constexpr size_t rsnap = sizeof(SnapSmem<DT, RT>), rlut = sizeof(LutSmem<RT>);
    constexpr bool P = FMT == kRowsPacked;
    static_assert(F != kScanGrid || !P, "the grid scan has no packed form");
    static_assert(F != kScanPacked || P, "the warp-chunk scan reads packed words");
    if constexpr (F == kScanSorted) return kernel(P ? bestfit_sorted_packed_snap_kernel<DT, T> : bestfit_sorted_kernel<DT, T, false>, T, snap);
    else if constexpr (F == kScanSortedContig) return kernel(P ? bestfit_sorted_packed_contig_kernel<DT, T> : bestfit_sorted_kernel<DT, T, true>, T, snap);
    else if constexpr (F == kScanGrid) return kernel(bestfit_grid_kernel<DT, T>, T, snap);
    else if constexpr (F == kScanLut) return kernel(P ? bestfit_lut_packed_snap_kernel<256> : bestfit_lut_kernel<256, false>, 256, lut);
    else if constexpr (F == kScanLutContig) return kernel(P ? bestfit_lut_packed_contig_kernel<256> : bestfit_lut_kernel<256, true>, 256, lut);
    else if constexpr (F == kScanSortedMulti) return kernel(P ? bestfit_sorted_packed_multi_kernel<DT, T> : bestfit_sorted_multi_kernel<DT, T>, T, snap);
    else if constexpr (F == kScanLutMulti) return kernel(P ? bestfit_lut_packed_multi_kernel<256> : bestfit_lut_multi_kernel<256>, 256, lut);
    else if constexpr (F == kScanPacked) return kernel(bestfit_sorted_packed_kernel<DT, T>, T, snap);
    else if constexpr (F == kRoundsSorted) return kernel(rounds_sorted_kernel<DT, FMT>, RT, rsnap);
    else if constexpr (F == kRoundsLut) return kernel(rounds_lut_kernel<FMT>, RT, rlut);
    else if constexpr (F == kRoundsMultiSorted) return kernel(rounds_sorted_multi_kernel<DT, FMT>, RT, rsnap);
    else if constexpr (F == kRoundsMultiLut) return kernel(rounds_lut_multi_kernel<FMT>, RT, rlut);
    else if constexpr (F == kShardPrefixSorted) return kernel(shard_prefix_multi_sorted_kernel<DT, FMT>, RT, rsnap);
    else if constexpr (F == kShardPrefixLut) return kernel(shard_prefix_multi_lut_kernel<FMT>, RT, rlut);
    else if constexpr (F == kShardRoundsSorted) return kernel(shard_rounds_sorted_kernel<DT, FMT>, RT, rsnap);
    else if constexpr (F == kShardRoundsLut) return kernel(shard_rounds_lut_kernel<FMT>, RT, rlut);
    else if constexpr (F == kRelease) return kernel(release_rows_kernel<DT, T, FMT, false>, T, snap);
    else {
        static_assert(F == kReleaseShard, "a family without kernels");
        return kernel(release_rows_kernel<DT, T, FMT, true>, T, snap);
    }
}
template <int F, RowFormat FMT, int B>
constexpr auto table_entry() {
    auto k = family_kernel<F, FMT, B>();
    k.slot = (F * 2 + FMT) * 4 + B;
    return k;
}
// The table of family F in format FMT, one kernel per D bucket
template <int F, RowFormat FMT>
constexpr decltype(family_kernel<F, FMT, 0>()) kKernels[4] = {table_entry<F, FMT, 0>(), table_entry<F, FMT, 1>(),
                                                              table_entry<F, FMT, 2>(), table_entry<F, FMT, 3>()};

// The kernel a launcher runs for the context's D: family F, or G when `alt` (the lookup scan, the sharded release), in
// row format fmt.  The one place a launcher's run-time choice of table is made.
template <int F, int G = F>
const auto& select_kernel(const egpu_ctx* ctx, bool alt, RowFormat fmt) {
    const int b = d_bucket(ctx->D);
    if constexpr (F == kScanGrid) return kKernels<F, kRowsInt32>[b];  // no packed form: launch_snapshot refuses packed rows
    else if (fmt == kRowsPacked) return alt ? kKernels<G, kRowsPacked>[b] : kKernels<F, kRowsPacked>[b];
    else return alt ? kKernels<G, kRowsInt32>[b] : kKernels<F, kRowsInt32>[b];
}

// Resident CTAs per SM of kernel k.  The first use on a context opts in to the kernel's dynamic shared memory and
// asks the occupancy; the answer stays in the context's occupancy cache.
template <class Fn>
int resident_ctas(egpu_ctx* ctx, const Kernel<Fn>& k, int* per_sm) {
    int& cached = ctx->ctas_per_sm[k.slot];
    if (cached == 0) {
        EGPU_CUDA(ctx, cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(k.smem)));
        int m = 0;
        EGPU_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&m, k.fn, k.threads, k.smem));
        cached = m < 1 ? 1 : m;
    }
    *per_sm = cached;
    return EGPU_OK;
}

// Programmatic dependent launch: the kernel may be scheduled while its predecessor on the stream
// still runs; each scan orders itself with griddepcontrol.wait (see order_scan).
template <class Fn, class... A>
int launch_pdl(egpu_ctx* ctx, const Kernel<Fn>& k, int64_t grid, cudaStream_t s, const A&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(static_cast<unsigned>(grid));
    cfg.blockDim = dim3(static_cast<unsigned>(k.threads));
    cfg.dynamicSmemBytes = k.smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    EGPU_CUDA(ctx, cudaLaunchKernelEx(&cfg, k.fn, args...));
    return EGPU_OK;
}

// blocks of a grid-stride kernel over n items, per_block items a block: at most 8 per SM
unsigned capped_blocks(const egpu_ctx* ctx, int64_t n, int64_t per_block) {
    int64_t blocks = (n + per_block - 1) / per_block;
    const int64_t cap = static_cast<int64_t>(ctx->sm_count) * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return static_cast<unsigned>(blocks);
}

bool lut_variant(const egpu_ctx* ctx) {
    return ctx->variant == EGPU_VARIANT_LUT || (ctx->variant == EGPU_VARIANT_AUTO && ctx->D > 16);
}

// Stream capture (CUDA graphs).  A launch captured into a graph runs at every replay, not now, against whatever
// table the context holds then; so the host bookkeeping of a captured launch must not change as if it had run
// (DESIGN.md 2.9):
//  - a captured lookup scan rebuilds d_lut inside the graph when it is stale (once per capture), and lut_dirty is
//    left as it was: the next eager lookup scan still rebuilds it;
//  - a captured launch that may rewrite the table and leaves d_lut alone is followed, inside the graph, by a
//    rebuild of d_lut, so that a replay leaves d_lut built from the table it installed; lut_dirty is left as it was;
//  - scans pipeline only behind scans of the same capture, or eagerly behind eager ones: a captured scan is never
//    the eager predecessor of the next launch; the epilogue rings still advance, so that slots stay distinct.
// capture_id: the capture sequence `s` belongs to (bit 63 set), 0 when it is not capturing.
unsigned long long capture_id(cudaStream_t s) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    unsigned long long id = 0;
    if (cudaStreamGetCaptureInfo(s, &st, &id) != cudaSuccess) {
        (void)cudaGetLastError();
        return 0;
    }
    return st == cudaStreamCaptureStatusActive ? (id | (1ull << 63)) : 0;
}

int launch_lut_build(egpu_ctx* ctx, cudaStream_t s) {
    lut_build_kernel<<<1, 256, 0, s>>>(ctx->d_state, ctx->d_lut);
    EGPU_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    ctx->prev_is_scan = false;
    return EGPU_OK;
}

// the lookup scans read ctx->d_lut: rebuild it on the launching stream after the table changed
int refresh_lut(egpu_ctx* ctx, cudaStream_t s) {
    const unsigned long long cap = capture_id(s);
    if (!ctx->lut_dirty || (cap && ctx->lut_capture == cap)) return EGPU_OK;
    const int rc = launch_lut_build(ctx, s);
    if (rc != EGPU_OK) return rc;
    if (cap) ctx->lut_capture = cap;
    else ctx->lut_dirty = false;
    return EGPU_OK;
}

// After a launch on `s` that may rewrite the table.  lut_built: the launch itself leaves d_lut built from the
// table it leaves (the persistent lookup kernels).  Eagerly: mark d_lut stale (or, lut_built, current).  Captured:
// rebuild it inside the graph (see capture_id).
int table_changed(egpu_ctx* ctx, cudaStream_t s, bool lut_built = false) {
    const unsigned long long cap = capture_id(s);
    if (!cap) {
        ctx->lut_dirty = !lut_built;
        return EGPU_OK;
    }
    if (!lut_built) {
        const int rc = launch_lut_build(ctx, s);
        if (rc != EGPU_OK) return rc;
    }
    ctx->lut_capture = cap;  // the graph's later lookup scans read the tables it rebuilt
    return EGPU_OK;
}

// Host image of a table: the part of DevState before `peer` (free capacity, D, candidate masks and
// the sorted view that resort_table_cta keeps on the device); oversub may be nullptr (no flags)
void table_image(DevState& h, const int32_t* free_core, const int32_t* free_mem, const int32_t* oversub, int D) {
    std::memset(&h, 0, offsetof(DevState, peer));
    std::memcpy(h.free_core, free_core, sizeof(int32_t) * D);
    std::memcpy(h.free_mem, free_mem, sizeof(int32_t) * D);
    if (oversub)
        for (int d = 0; d < D; ++d) h.oversub[d] = oversub[d] ? 1 : 0;
    h.D = D;
    h.cand_xor = kGuards;
    h.cand_mask = kCandMask;
    for (int j = 0; j < kMaxD; ++j) {
        h.sorted_k[j] = kPadWord;
        h.sorted_dev[j] = -1;
    }
    unsigned long long packed = ~0ull;
    for (int d = 0; d < D; ++d) {
        const uint32_t mine = (static_cast<uint32_t>(h.free_core[d]) << 24) | (static_cast<uint32_t>(h.free_mem[d]) << 6) | d;
        int pos = 0;
        for (int k = 0; k < D; ++k) {
            const uint32_t other = (static_cast<uint32_t>(h.free_core[k]) << 24) | (static_cast<uint32_t>(h.free_mem[k]) << 6) | k;
            pos += other < mine;
        }
        h.sorted_k[pos] = pack_table_word(h.free_core[d], h.free_mem[d]) | (static_cast<uint32_t>(pos) & 31u);
        h.sorted_dev[pos] = d;
        if (pos < 8) packed = (packed & ~(0xffull << (8 * pos))) | (static_cast<unsigned long long>(d) << (8 * pos));
    }
    h.dev_packed = packed;
}

// ---- output ranges of the launches in flight (pipelined launches must not share outputs) ----
using Range = egpu_ctx::Range;
// the outputs of one batch: indices (idx_bytes each: int32, or int8 in the packed format), demand sums, table'
void batch_ranges(Range* r, const void* idx, int64_t R, size_t idx_bytes, const void* delta, const int32_t* table_out, int D) {
    const uintptr_t pi = reinterpret_cast<uintptr_t>(idx), pd = reinterpret_cast<uintptr_t>(delta),
                    pt = reinterpret_cast<uintptr_t>(table_out);
    r[0] = {pi, pi + static_cast<uintptr_t>(R) * idx_bytes};
    r[1] = {pd, pd + (pd ? sizeof(long long) * 2 * D : 0)};
    r[2] = {pt, pt + (pt ? sizeof(int32_t) * 3 * D : 0)};
}
// `r[0..n)`: drops empty ranges, sorts by address; returns the new count, or -1 when two of
// them overlap each other.
int prepare_ranges(Range* r, int n) {
    int m = 0;
    for (int i = 0; i < n; ++i)
        if (r[i].hi > r[i].lo) r[m++] = r[i];
    std::sort(r, r + m, [](const Range& a, const Range& b) { return a.lo < b.lo; });
    for (int i = 1; i < m; ++i)
        if (r[i].lo < r[i - 1].hi) return -1;
    return m;
}
// both sorted and internally disjoint: one sweep
bool overlaps_inflight(const std::vector<Range>& f, const Range* r, int n) {
    size_t i = 0;
    int k = 0;
    while (i < f.size() && k < n) {
        if (f[i].hi <= r[k].lo) ++i;
        else if (r[k].hi <= f[i].lo) ++k;
        else return true;
    }
    return false;
}
// the device descriptor of one batch: of the multi-batch scans, and of the persistent kernels
void set_desc(BatchDesc& d, const int32_t* rc, const int32_t* rm, long long R, int32_t* idx, long long* delta, int32_t* table_out) {
    d = {rc, rm, idx, delta, table_out, R};
}
void set_desc(RoundsBatch& d, const int32_t* rc, const int32_t* rm, long long R, int32_t* idx, long long* delta, int32_t* table_out) {
    d = {rc, rm, R, idx, delta, table_out};
}
// K batches of `bs` in format fmt as device descriptors `out` (packed: no mem array; table_out false: no table'), and
// their outputs in ctx->multi_ranges, prepared.  Returns the number of ranges, or -1 when two batches share an output
// (their order would be undefined); *max_r = the largest R.
template <class Desc>
int batch_descs(egpu_ctx* ctx, const egpu_batch* bs, int K, RowFormat fmt, bool table_out, Desc* out, int64_t* max_r) {
    const bool packed = fmt == kRowsPacked;
    Range* mine = ctx->multi_ranges;
    *max_r = 0;
    for (int b = 0; b < K; ++b) {
        const egpu_batch& in = bs[b];
        long long* delta = reinterpret_cast<long long*>(in.d_delta);
        int32_t* tab = table_out ? in.d_table_out : nullptr;
        set_desc(out[b], in.d_req_core, packed ? nullptr : in.d_req_mem, in.R, in.d_out_idx, delta, tab);
        batch_ranges(mine + 3 * b, in.d_out_idx, in.R, packed ? sizeof(int8_t) : sizeof(int32_t), delta, tab, ctx->D);
        *max_r = std::max<int64_t>(*max_r, in.R);
    }
    return prepare_ranges(mine, 3 * K);
}

void new_group(egpu_ctx* ctx) {
    ctx->group_len = 0;
    ctx->group_mbatches = 0;
    ctx->inflight.clear();
}

// Ordering of a scan behind the launches before it (programmatic dependent launch); returns its
// kFlagLateWait | kFlagBoundary | kFlagEarlyTrigger bits.  Every scan carries the PDL attribute,
// so the hardware may schedule it while its predecessor is still running.  A fully ordered launch
// waits (griddepcontrol.wait) before it touches anything.  A pipelined launch (kFlagLateWait) runs
// scan and epilogue at once - its epilogue state is its own slot - and waits only before exiting.
// That is allowed when
//  - the caller vouches its inputs were complete before the previous launch on this stream
//    (EGPU_F_INPUTS_READY), and `eligible` holds: the launch's own conditions (a single-batch
//    launch must not commit - a committing launch rewrites the table the launches still in flight
//    read and compute their table' from - and must be a plain scan, neither CONTIG nor the grid
//    variant),
//  - the previous launch was a scan of this context on the same stream that does not rewrite
//    the table,
//  - its outputs (indices, demand sums, table') are disjoint from the outputs of every launch
//    since the last fully ordered one, and
//  - fewer than pipe_group launches have been issued since then, which bounds the launches in
//    flight to pipe_group + 1 < kEpiSlots, and the epi_multi slots of those launches and this
//    one's `batches` (0 for a single-batch launch) stay within half of that ring.
// Otherwise the launch is fully ordered and opens a new group.
// `cap`: the launch's capture_id; the previous launch must belong to the same capture, or both be eager.
int order_scan(egpu_ctx* ctx, int user_flags, bool eligible, int batches, cudaStream_t s, const Range* mine, int n_mine,
               unsigned long long cap) {
    int flags = 0;
    const bool pipelined = (user_flags & EGPU_F_INPUTS_READY) && eligible && ctx->prev_capture == cap && ctx->prev_is_scan && !ctx->prev_changes_table &&
                           ctx->prev_stream == s && ctx->group_len > 0 && !overlaps_inflight(ctx->inflight, mine, n_mine);
    if (pipelined) {
        flags |= kFlagLateWait;
        if (ctx->group_len >= ctx->pipe_group || ctx->group_mbatches + batches > kMultiSlots - kMultiMax) {
            // group boundary: this launch still scans alongside its predecessors, but it waits
            // for them before its epilogue and only then lets its successors start; it becomes
            // the first member of the next group
            flags |= kFlagBoundary;
            new_group(ctx);
        }
    } else {
        new_group(ctx);
    }
    // Early trigger (griddepcontrol.launch_dependents before the work is done) only helps when
    // the next launch is another scan of a pipelined stream, so only those launches do it.
    // (What scripts/probes/pdl_event_probe.cu and scripts/eager_probe.py check: events
    // and ordinary kernels enqueued after a PDL launch still wait for its completion.)
    if (user_flags & EGPU_F_INPUTS_READY) flags |= kFlagEarlyTrigger;
    return flags;
}

// Bookkeeping of a scan launched under order_scan: `batches` = 0 for a single-batch launch (one
// epilogue slot of the seq ring), K for a multi-batch one (K slots of the mseq ring); `cap` its capture_id.
void record_scan(egpu_ctx* ctx, cudaStream_t s, const Range* mine, int n_mine, int batches, bool changes_table,
                 unsigned long long cap) {
    ctx->launches += 1;
    if (batches) ctx->mseq += static_cast<uint64_t>(batches);
    else ctx->seq += 1;
    ctx->prev_capture = cap;
    ctx->range_tmp.resize(ctx->inflight.size() + static_cast<size_t>(n_mine));
    std::merge(ctx->inflight.begin(), ctx->inflight.end(), mine, mine + n_mine, ctx->range_tmp.begin(),
               [](const Range& a, const Range& b) { return a.lo < b.lo; });
    ctx->inflight.swap(ctx->range_tmp);
    ctx->group_len += 1;
    ctx->group_mbatches += batches;
    ctx->prev_is_scan = true;
    ctx->prev_changes_table = changes_table;
    ctx->prev_stream = s;
}

// ---- single-batch scans ----
struct Snapshot {
    const int32_t* rc;
    const int32_t* rm;
    int64_t R;
    int32_t* idx;
    long long* delta = nullptr;
    int32_t* table_out = nullptr;
    int user_flags = 0;                          // EGPU_F_COMMIT | EGPU_F_INPUTS_READY
    int rpt_hint = 0;                            // rows per thread, 0 = the default rule below
    unsigned long long push_step_plus1 = 0;      // exchange step + 1 the epilogue pushes the demand to, 0 = none
    int lag = 0;                                 // lagged apply (egpu_bestfit_batch_shard_lag_dev)
    bool contig = false;                         // prefix-commit: contiguous tiles, per-tile sums in ctx->d_tile_sums
    bool packed = false;                         // rc = packed words, rm unused, idx = int8 indices (CONTIG: prefix-commit,
                                                 // otherwise a sharded scan); not in the grid variant
};

template <int F>
int launch_snapshot_as(egpu_ctx* ctx, const Snapshot& a, cudaStream_t s, int* n_tiles_out) {
    constexpr bool lut = F == kScanLut || F == kScanLutContig, grid_variant = F == kScanGrid;
    const auto& k = select_kernel<F>(ctx, false, a.packed ? kRowsPacked : kRowsInt32);
    int per_sm = 0;
    int rc = resident_ctas(ctx, k, &per_sm);
    if (rc != EGPU_OK) return rc;
    if (lut) {
        rc = refresh_lut(ctx, s);
        if (rc != EGPU_OK) return rc;
    }
    Range mine[3];
    batch_ranges(mine, a.idx, a.R, a.packed ? sizeof(int8_t) : sizeof(int32_t), a.delta, a.table_out, ctx->D);
    const int n_mine = prepare_ranges(mine, 3);
    if (n_mine < 0) return EGPU_ERR_INVALID;  // two of this launch's own outputs overlap
    const bool commit = (a.user_flags & EGPU_F_COMMIT) != 0;
    const unsigned long long captured = capture_id(s);
    const int flags = kFlagFinalize | (commit ? kFlagCommit : 0) |
                      order_scan(ctx, a.user_flags, !grid_variant && !a.contig && !commit, 0, s, mine, n_mine, captured);
    const unsigned long long slot = (ctx->seq % kEpiSlots) | (a.push_step_plus1 << 8) | (static_cast<unsigned long long>(a.lag) << 56);

    // Grid: one resident wave at most.  A lone launch wants every SM pulling at once
    // (8 rows per thread, one trip); launches of a pipelined stream overlap each
    // other, so a smaller grid with more rows per thread (48) costs fewer CTA
    // launches, fewer atomics and leaves room for the neighbours (scripts/tune_sweep.sh
    // re-measures the choice at R = 1M).  The zero-copy path passes its own hint (see egpu_bestfit_batch).
    const int64_t nvec = a.R >> 2;
    int rpt = 8;
    // (measured and dropped: giving the launches of a pipelined stream that could not themselves be
    // pipelined - the first of a graph - the lone-launch grid: slower per step)
    if (a.user_flags & EGPU_F_INPUTS_READY) rpt = (lut || ctx->D <= 16) ? 48 : 8;  // measured, scripts/tune_*.sh
    else if (lut) rpt = 32;  // the lookup scan has a 13 KB per-CTA table tile to amortise
    // a lone packed sharded register scan: 5-byte rows want longer CTAs (16 measured faster than 8 at D = 8; twice
    // the other rules measured slower or level, DESIGN.md 4.1c)
    else if (a.packed && !a.contig) rpt = 16;
    if (a.rpt_hint > 0) rpt = a.rpt_hint;
    if (ctx->rows_per_thread > 0) rpt = ctx->rows_per_thread;
    if (grid_variant) rpt = 4;
    const int64_t per_cta = static_cast<int64_t>(k.threads) * ((rpt + 3) / 4);
    int64_t want = (nvec + per_cta - 1) / per_cta;
    if (ctx->ctas_per_sm_cap > 0 && ctx->ctas_per_sm_cap < per_sm) per_sm = ctx->ctas_per_sm_cap;
    // one resident wave; two for a huge batch (the CTA scheduler then evens out the SMs, see launch_multi)
    const int64_t cap = static_cast<int64_t>(ctx->sm_count) * per_sm * ((a.R >= (16ll << 20) && !a.contig) ? 2 : 1);
    if (want > cap) want = cap;
    if (want < 1) want = 1;
    // lane-private sums hold 2^19 rows per lane (kAccShift): keep rows/thread below that
    const int64_t rows_per_thread = a.R / (want * k.threads) + 8;
    if (rows_per_thread >= (1ll << 19)) return EGPU_ERR_INVALID;

    unsigned long long* tile_sums = nullptr;
    if (a.contig) {  // one tile per CTA: make room for their sums
        const size_t bytes = sizeof(unsigned long long) * 2 * kMaxD * static_cast<size_t>(want);
        EGPU_CUDA(ctx, grow(ctx->tile_bytes, bytes, bytes, &ctx->d_tile_sums));
        tile_sums = ctx->d_tile_sums;
        *n_tiles_out = static_cast<int>(want);
    }
    if constexpr (lut)
        rc = launch_pdl(ctx, k, want, s, ctx->d_state, a.rc, a.rm, static_cast<long long>(a.R), a.idx, a.delta, a.table_out, flags,
                        slot, static_cast<const DevLut*>(ctx->d_lut), tile_sums);
    else
        rc = launch_pdl(ctx, k, want, s, ctx->d_state, a.rc, a.rm, static_cast<long long>(a.R), a.idx, a.delta, a.table_out, flags,
                        slot, tile_sums);
    if (rc != EGPU_OK) return rc;
    record_scan(ctx, s, mine, n_mine, 0, commit, captured);
    return commit ? table_changed(ctx, s) : EGPU_OK;
}

// One scan of one batch against the context's table, in the kernel the context's variant picks.
// A CONTIG scan reports its tile count in *n_tiles_out.
int launch_snapshot(egpu_ctx* ctx, const Snapshot& a, cudaStream_t s, int* n_tiles_out = nullptr) {
    if (a.R > kMaxRows) return EGPU_ERR_INVALID;  // the scans index 128-bit vectors with 32 bits
    const bool grid_variant = ctx->variant == EGPU_VARIANT_GRID;
    if ((a.contig || a.packed) && grid_variant) return EGPU_ERR_STATE;  // the literal variant has no prefix-commit mode, no packed form
    if (lut_variant(ctx))
        return a.contig ? launch_snapshot_as<kScanLutContig>(ctx, a, s, n_tiles_out) : launch_snapshot_as<kScanLut>(ctx, a, s, n_tiles_out);
    if (grid_variant) return launch_snapshot_as<kScanGrid>(ctx, a, s, n_tiles_out);
    return a.contig ? launch_snapshot_as<kScanSortedContig>(ctx, a, s, n_tiles_out) : launch_snapshot_as<kScanSorted>(ctx, a, s, n_tiles_out);
}

// Multi-batch launch: K batches, all scored against the current table, one grid (CTA (b, t) =
// tile t of batch b), one epilogue slot per batch.  Pipelines behind its predecessor under the
// conditions of order_scan; a launch group never holds more than half of the epi_multi ring,
// so the slots of everything that can be in flight are distinct.
// push_base = first exchange step + 1 when every batch also pushes its demand vector to the peers.
// EGPU_F_PACKED: the batches are in the packed format (d_req_core = words, d_out_idx = int8 indices)
// and run in the packed twin of family F's kernel; everything else is the same launch.
template <int F>
int launch_multi_as(egpu_ctx* ctx, const egpu_batch* bs, int K, int user_flags, cudaStream_t s, unsigned long long push_base) {
    constexpr bool lut = F == kScanLutMulti;
    const RowFormat fmt = row_format(user_flags);
    const auto& k = select_kernel<F>(ctx, false, fmt);
    int per_sm = 0;
    int rc = resident_ctas(ctx, k, &per_sm);
    if (rc != EGPU_OK) return rc;
    if (lut) {
        rc = refresh_lut(ctx, s);
        if (rc != EGPU_OK) return rc;
    }
    MultiArgs args;
    std::memset(&args, 0, sizeof args);
    Range* mine = ctx->multi_ranges;
    int64_t max_r = 0;
    // sharded: table' comes from an apply call, or (EGPU_F_APPLY) from the batch's own last CTA
    const bool table_out = !push_base || (user_flags & EGPU_F_APPLY);
    const int n_mine = batch_descs(ctx, bs, K, fmt, table_out, args.b, &max_r);
    if (n_mine < 0) return EGPU_ERR_INVALID;
    const unsigned long long captured = capture_id(s);
    const int flags = kFlagFinalize | ((push_base && (user_flags & EGPU_F_APPLY)) ? kFlagApplyNow : 0) |
                      order_scan(ctx, user_flags, true, K, s, mine, n_mine, captured);

    // Tiles per batch.  Batches below 512 Ki rows: enough CTAs that a thread has >= multi_rpt rows,
    // at most the resident capacity of the GPU (one wave: there, every extra CTA costs an epilogue
    // and 100 k-row batches measured slower with more).  Larger batches: about 20 rows per thread
    // (28 in the lookup scan, whose CTAs first copy a 15 KB table), rounded up to whole waves, however
    // many that takes.  The SMs do not stream at the same rate (in one wave the CTAs' exit times
    // spread over a third of the launch); with several waves of small CTAs the hardware scheduler
    // hands the next CTA to whichever SM frees a slot first.  Either way the CTAs are shared out
    // evenly, the first `extra` batches get one more.  Packed rows are 5 bytes instead of 12, and
    // their large batches want longer CTAs: 48 rows per thread (56 in the lookup scan) measured
    // fastest of 20 / 28, 32 / 40 and 48 / 56.  Measured on an H100: DESIGN.md 4.1e.
    const int64_t nvec = max_r >> 2;
    const bool small = max_r < (512ll << 10);
    const int64_t rpt = small ? ctx->multi_rpt : fmt == kRowsPacked ? (lut ? 56 : 48) : (lut ? 28 : 20);
    const int64_t per_cta = static_cast<int64_t>(k.threads) * ((rpt + 3) / 4);
    int64_t tiles = (nvec + per_cta - 1) / per_cta;
    if (tiles < 1) tiles = 1;
    if (ctx->ctas_per_sm_cap > 0 && ctx->ctas_per_sm_cap < per_sm) per_sm = ctx->ctas_per_sm_cap;
    const int64_t wave = static_cast<int64_t>(ctx->sm_count) * per_sm;
    int64_t extra = 0;
    if (!small || tiles * K > wave) {
        const int64_t total = small ? wave : (tiles * K + wave - 1) / wave * wave;
        tiles = total / K;
        extra = total % K;
        if (tiles < 1) {
            tiles = 1;
            extra = 0;
        }
    }
    if (tiles > 0xffff) tiles = 0xffff;
    if (max_r / (tiles * k.threads) + 8 >= (1ll << 19)) return EGPU_ERR_INVALID;  // lane-private sums hold 2^19 rows per lane
    const int tiles_extra = static_cast<int>(tiles | (extra << 16));
    const int64_t n_ctas = tiles * K + extra;

    const unsigned int slot_base = static_cast<unsigned int>(ctx->mseq % kMultiSlots);
    if constexpr (lut)
        rc = launch_pdl(ctx, k, n_ctas, s, ctx->d_state, args, tiles_extra, flags, slot_base, push_base,
                        static_cast<const DevLut*>(ctx->d_lut));
    else
        rc = launch_pdl(ctx, k, n_ctas, s, ctx->d_state, args, tiles_extra, flags, slot_base, push_base);
    if (rc != EGPU_OK) return rc;
    record_scan(ctx, s, mine, n_mine, K, false, captured);
    return EGPU_OK;
}

int launch_multi(egpu_ctx* ctx, const egpu_batch* bs, int K, int user_flags, cudaStream_t s, unsigned long long push_base) {
    if (ctx->variant == EGPU_VARIANT_GRID) return EGPU_ERR_STATE;  // the literal variant has no multi-batch form
    return lut_variant(ctx) ? launch_multi_as<kScanLutMulti>(ctx, bs, K, user_flags, s, push_base)
                            : launch_multi_as<kScanSortedMulti>(ctx, bs, K, user_flags, s, push_base);
}

// First half of a prefix-commit (spec 2.5): the CONTIG scan, which neither commits nor returns
// delta / table' (its sums are the uncapped ones); push_step_plus1 as in Snapshot.  Returns the
// PrefixOut the next kernels fill and the tile count of the scan.  kRowsPacked: d_rc holds the
// packed words (d_rm unused) and d_idx receives int8 indices.
int prefix_scan(egpu_ctx* ctx, const int32_t* d_rc, const int32_t* d_rm, int64_t R, int32_t* d_idx, RowFormat fmt,
                unsigned long long push_step_plus1, cudaStream_t s, PrefixOut** pf, int* n_tiles) {
    if (!ctx->d_prefix_out) EGPU_CUDA(ctx, cudaMalloc(&ctx->d_prefix_out, sizeof(PrefixOut) + sizeof(long long) * 2 * kMaxD));
    *pf = static_cast<PrefixOut*>(ctx->d_prefix_out);
    Snapshot a{d_rc, d_rm, R, d_idx};
    a.push_step_plus1 = push_step_plus1;
    a.contig = true;
    a.packed = fmt == kRowsPacked;
    return launch_snapshot(ctx, a, s, n_tiles);
}

// Prefix-commit pipeline on device buffers (spec 2.5): CONTIG scan -> per-device cut ->
// rewrite of the deferred indices -> delta / table' of the committed rows only.  Rows in
// either format (see prefix_scan); the cut and the rewrite read the scan's format.
int launch_prefix_commit(egpu_ctx* ctx, const int32_t* d_rc, const int32_t* d_rm, int64_t R, int32_t* d_idx,
                         long long* d_delta, int32_t* d_table_out, int user_flags, cudaStream_t s, RowFormat fmt = kRowsInt32) {
    PrefixOut* pf = nullptr;
    int n_tiles = 0;
    const int rc = prefix_scan(ctx, d_rc, d_rm, R, d_idx, fmt, 0, s, &pf, &n_tiles);
    if (rc != EGPU_OK) return rc;
    if (fmt == kRowsPacked) {
        signed char* idx8 = reinterpret_cast<signed char*>(d_idx);
        prefix_cut_packed_kernel<<<ctx->D, 256, 0, s>>>(ctx->d_state, idx8, reinterpret_cast<const uint32_t*>(d_rc), R, n_tiles,
                                                        ctx->d_tile_sums, pf);
        prefix_apply_packed_kernel<<<capped_blocks(ctx, R, 1024), 256, 0, s>>>(pf, ctx->D, R, idx8);
    } else {
        prefix_cut_kernel<<<ctx->D, 256, 0, s>>>(ctx->d_state, d_idx, d_rc, d_rm, R, n_tiles, ctx->d_tile_sums, pf);
        prefix_apply_kernel<<<capped_blocks(ctx, R, 1024), 256, 0, s>>>(pf, ctx->D, R, d_idx);
    }
    prefix_finalize_kernel<<<1, kMaxD, 0, s>>>(ctx->d_state, pf, d_delta, d_table_out, (user_flags & EGPU_F_COMMIT) ? 1 : 0);
    EGPU_CUDA(ctx, cudaGetLastError());
    ctx->launches += 3;
    ctx->prev_is_scan = false;
    return (user_flags & EGPU_F_COMMIT) ? table_changed(ctx, s) : EGPU_OK;
}

// Rounds of committing prefix-commit until nothing is deferred (spec 2.5, "rounds").  Round 1
// runs on the caller's device arrays; the rows it defers are gathered, in order, into dense
// scratch arrays and re-submitted against the table round 1 committed, and so on.  Every round
// needs two numbers on the host (rows still deferred, the round's committed demand), so this
// is a synchronous host loop around asynchronous launches.  Rows in either format (see
// prefix_scan); d_table_out (may be NULL) receives every round's table', so the last one stays.
struct RoundInfo {
    unsigned long long deferred;
    long long delta[2 * kMaxD];
};

// Scratch of the rounds (run_rounds and the one-launch rounds), owned by the context, grow-only,
// sized by R BEFORE anything is committed (a failed allocation must not leave a half-committed
// batch): a head (round info; the one-launch rounds keep their grid-barrier words at kRoundsCtlOff),
// tile counts, and two sets of (core, mem, caller's row, index) arrays - the deferred rows of any
// round are at most R.  Packed: two sets of (words, caller's row, int8 index), 9 bytes per row each.
constexpr size_t kRoundsHead = 2048;
constexpr size_t kRoundsCtlOff = 1536;
constexpr size_t kShardStopOff = 1792;  // the stop word of the multi-batch sharded prefix-commit (ShardPrefixArgs::stop)
constexpr size_t kShardAgainOff = 1800;  // the again word of the sharded rounds (ShardRoundsArgs::again)
static_assert(sizeof(RoundInfo) <= kRoundsCtlOff && kRoundsCtlOff + sizeof(RoundsCtl) <= kShardStopOff &&
                  kShardStopOff + sizeof(unsigned int) <= kShardAgainOff && kShardAgainOff + sizeof(unsigned int) <= kRoundsHead,
              "rounds scratch head");
struct RoundsScratch {
    RoundInfo* info;
    unsigned int* tiles;
    int32_t* set[2][4];  // rc, rm (packed: none), map, idx
};
int rounds_scratch(egpu_ctx* ctx, int64_t R, bool packed, RoundsScratch* out) {
    auto align = [](size_t b) { return (b + 255) & ~static_cast<size_t>(255); };
    const int64_t tiles_cap = (R + kCompactTile - 1) / kCompactTile;
    const size_t tiles_bytes = align(sizeof(unsigned int) * static_cast<size_t>(tiles_cap));
    const size_t per = align(sizeof(int32_t) * static_cast<size_t>(R));
    const size_t sub[4] = {per, packed ? 0 : per, per, packed ? align(static_cast<size_t>(R)) : per};  // rc, rm, map, idx
    const size_t need = kRoundsHead + tiles_bytes + 2 * (sub[0] + sub[1] + sub[2] + sub[3]);
    EGPU_CUDA(ctx, grow(ctx->rounds_bytes, need, need, &ctx->d_rounds));
    char* base = static_cast<char*>(ctx->d_rounds);
    out->info = reinterpret_cast<RoundInfo*>(base);
    out->tiles = reinterpret_cast<unsigned int*>(base + kRoundsHead);
    size_t off = kRoundsHead + tiles_bytes;
    for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 4; ++b) {
            out->set[a][b] = sub[b] ? reinterpret_cast<int32_t*>(base + off) : nullptr;
            off += sub[b];
        }
    return EGPU_OK;
}

// The grid-barrier words of the persistent launches, in the head of the rounds scratch (rounds_scratch first)
int rounds_ctl(egpu_ctx* ctx, cudaStream_t s, RoundsCtl** out) {
    RoundsCtl* ctl = reinterpret_cast<RoundsCtl*>(reinterpret_cast<char*>(ctx->d_rounds) + kRoundsCtlOff);
    if (ctx->rounds_ctl_bytes != ctx->rounds_bytes) {  // fresh scratch: the barrier words start at zero
        EGPU_CUDA(ctx, cudaMemsetAsync(ctl, 0, sizeof(RoundsCtl), s));
        ctx->rounds_ctl_bytes = ctx->rounds_bytes;
    }
    *out = ctl;
    return EGPU_OK;
}

// The RoundsArgs of a one-launch rounds kernel whose (first) batch is b, in format fmt: allocates the rounds scratch
// for R rows and zeroes fresh barrier words on s (rounds_scratch, rounds_ctl); the context's tile sums, PrefixOut and
// lookup tables.
int rounds_args(egpu_ctx* ctx, const egpu_batch& b, int64_t R, RowFormat fmt, cudaStream_t s, RoundsArgs* a) {
    const bool packed = fmt == kRowsPacked;
    RoundsScratch sc;
    int rc = rounds_scratch(ctx, R, packed, &sc);
    if (rc != EGPU_OK) return rc;
    std::memset(a, 0, sizeof *a);
    rc = rounds_ctl(ctx, s, &a->ctl);
    if (rc != EGPU_OK) return rc;
    a->rc = b.d_req_core;
    a->rm = packed ? nullptr : b.d_req_mem;
    a->R = static_cast<long long>(b.R);
    a->idx = b.d_out_idx;
    a->delta_out = reinterpret_cast<long long*>(b.d_delta);
    a->table_out = b.d_table_out;
    a->tile_sums = ctx->d_tile_sums;
    a->pf = static_cast<PrefixOut*>(ctx->d_prefix_out);
    a->total = sc.info->delta;
    a->deferred = &sc.info->deferred;
    a->tile_count = sc.tiles;
    std::memcpy(a->set, sc.set, sizeof a->set);
    a->lut = ctx->d_lut;
    return EGPU_OK;
}

int run_rounds(egpu_ctx* ctx, const int32_t* d_rc, const int32_t* d_rm, int64_t R, int32_t* d_idx, int max_rounds,
               long long* total_delta /* host [2*D] */, int32_t* rounds_out, int64_t* left_out, cudaStream_t s,
               RowFormat fmt = kRowsInt32, int32_t* d_table_out = nullptr) {
    const int D = ctx->D;
    const bool packed = fmt == kRowsPacked;
    for (int j = 0; j < 2 * D; ++j) total_delta[j] = 0;
    *rounds_out = 0;
    *left_out = 0;
    if (R == 0 || max_rounds < 1) return EGPU_OK;
    RoundsScratch sc;
    const int rcs = rounds_scratch(ctx, R, packed, &sc);
    if (rcs != EGPU_OK) return rcs;
    RoundInfo* d_info = sc.info;
    unsigned int* d_tiles = sc.tiles;
    // current round's arrays (round 1: the caller's) and the next round's
    const int32_t* cur_rc = d_rc;
    const int32_t* cur_rm = d_rm;
    const int32_t* cur_map = nullptr;
    int32_t* cur_idx = d_idx;
    int64_t n = R;
    int32_t* (&set)[2][4] = sc.set;
    int which = 0;
    RoundInfo h{};
    auto idx8 = [](const int32_t* p) { return reinterpret_cast<signed char*>(const_cast<int32_t*>(p)); };
    for (int round = 1;; ++round) {
        int rc = launch_prefix_commit(ctx, cur_rc, cur_rm, n, cur_idx, d_info->delta, d_table_out, EGPU_F_COMMIT, s, fmt);
        if (rc != EGPU_OK) return rc;
        if (cur_map) {
            if (packed)
                round_writeback_packed_kernel<<<capped_blocks(ctx, n, 256), 256, 0, s>>>(idx8(cur_idx), cur_map, n, idx8(d_idx));
            else
                round_writeback_kernel<<<capped_blocks(ctx, n, 256), 256, 0, s>>>(cur_idx, cur_map, n, d_idx);
            ctx->launches += 1;
        }
        const int64_t tiles = (n + kCompactTile - 1) / kCompactTile;
        if (packed)
            deferred_count_packed_kernel<<<static_cast<unsigned>(tiles), 256, 0, s>>>(idx8(cur_idx), n, d_tiles);
        else
            deferred_count_kernel<<<static_cast<unsigned>(tiles), 256, 0, s>>>(cur_idx, n, d_tiles);
        deferred_scan_kernel<<<1, 1024, 0, s>>>(d_tiles, tiles, &d_info->deferred);
        ctx->launches += 2;
        EGPU_CUDA(ctx, cudaGetLastError());
        EGPU_CUDA(ctx, cudaMemcpyAsync(&h, d_info, sizeof h, cudaMemcpyDeviceToHost, s));
        EGPU_CUDA(ctx, cudaStreamSynchronize(s));
        for (int j = 0; j < 2 * D; ++j) total_delta[j] += h.delta[j];
        *rounds_out = round;
        *left_out = static_cast<int64_t>(h.deferred);
        if (h.deferred == 0 || round >= max_rounds) return EGPU_OK;
        int32_t** nxt = set[which];
        if (packed)
            deferred_scatter_packed_kernel<<<static_cast<unsigned>(tiles), 256, 0, s>>>(
                idx8(cur_idx), reinterpret_cast<const uint32_t*>(cur_rc), cur_map, n, d_tiles, reinterpret_cast<uint32_t*>(nxt[0]), nxt[2]);
        else
            deferred_scatter_kernel<<<static_cast<unsigned>(tiles), 256, 0, s>>>(cur_idx, cur_rc, cur_rm, cur_map, n, d_tiles, nxt[0],
                                                                                   nxt[1], nxt[2]);
        ctx->launches += 1;
        EGPU_CUDA(ctx, cudaGetLastError());
        cur_rc = nxt[0];
        cur_rm = nxt[1];
        cur_map = nxt[2];
        cur_idx = nxt[3];
        n = static_cast<int64_t>(h.deferred);
        which ^= 1;
    }
}

// EGPU_F_ROUNDS: packed prefix-commit rounds until nothing is deferred, on device words and int8
// indices.  Leaves the demand committed over all rounds in host total[2*D] and, when d_delta is
// given, in d_delta; d_table_out receives the last round's table'.  R = 0 is the packed
// prefix-commit with R = 0.  The caller synchronises `s`.
int launch_packed_rounds(egpu_ctx* ctx, const int32_t* d_words, int64_t R, int32_t* d_idx8, long long* d_delta,
                         int32_t* d_table_out, long long* total /* host [2*D] */, cudaStream_t s) {
    if (ctx->variant == EGPU_VARIANT_GRID) return EGPU_ERR_STATE;  // no prefix-commit mode
    if (R == 0) {
        for (int j = 0; j < 2 * ctx->D; ++j) total[j] = 0;
        return launch_prefix_commit(ctx, d_words, nullptr, 0, d_idx8, d_delta, d_table_out, EGPU_F_COMMIT, s, kRowsPacked);
    }
    int32_t rounds = 0;
    int64_t left = 0;
    const int rc = run_rounds(ctx, d_words, nullptr, R, d_idx8, INT32_MAX, total, &rounds, &left, s, kRowsPacked, d_table_out);
    if (rc != EGPU_OK) return rc;
    if (d_delta) EGPU_CUDA(ctx, cudaMemcpyAsync(d_delta, total, sizeof(long long) * 2 * ctx->D, cudaMemcpyHostToDevice, s));
    return EGPU_OK;
}

// The flags EGPU_F_ROUNDS is valid with: all of kRoundsNeeds, optionally EGPU_F_INPUTS_READY
constexpr int kRoundsNeeds = EGPU_F_PACKED | EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT | EGPU_F_ROUNDS;
bool rounds_flags_ok(int flags, int64_t R) {
    return (flags & ~(kRoundsNeeds | EGPU_F_INPUTS_READY)) == 0 && (flags & kRoundsNeeds) == kRoundsNeeds && R < (1ll << 31);
}

// The flags EGPU_F_DEVICE_ROUNDS is valid with: all of kDeviceRoundsNeeds, optionally EGPU_F_PACKED and
// EGPU_F_INPUTS_READY
constexpr int kDeviceRoundsNeeds = EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT | EGPU_F_ROUNDS | EGPU_F_DEVICE_ROUNDS;
bool device_rounds_flags_ok(int flags, int64_t R) {
    return (flags & ~(kDeviceRoundsNeeds | EGPU_F_PACKED | EGPU_F_INPUTS_READY)) == 0 &&
           (flags & kDeviceRoundsNeeds) == kDeviceRoundsNeeds && R < (1ll << 31);
}

// The flags EGPU_F_RELEASE is valid with: itself, optionally EGPU_F_COMMIT and EGPU_F_PACKED
bool release_flags_ok(int flags, int64_t R) {
    return (flags & ~(EGPU_F_RELEASE | EGPU_F_COMMIT | EGPU_F_PACKED)) == 0 && R < (1ll << 31);
}

// What egpu_bestfit_batch[_dev] does
enum BatchOp { kOpSnapshot, kOpPrefix, kOpRounds, kOpDeviceRounds, kOpRelease };

// The operation of egpu_bestfit_batch[_dev]'s flags for R rows; false when the flags are refused.  Without
// EGPU_F_RELEASE, EGPU_F_DEVICE_ROUNDS or EGPU_F_ROUNDS other bits are ignored, except that EGPU_F_PACKED needs
// EGPU_F_PREFIX_COMMIT.
bool batch_op(int flags, int64_t R, BatchOp* op) {
    *op = (flags & EGPU_F_RELEASE)         ? kOpRelease
          : (flags & EGPU_F_DEVICE_ROUNDS) ? kOpDeviceRounds
          : (flags & EGPU_F_ROUNDS)        ? kOpRounds
          : (flags & EGPU_F_PREFIX_COMMIT) ? kOpPrefix
                                           : kOpSnapshot;
    switch (*op) {
        case kOpRelease: return release_flags_ok(flags, R);
        case kOpDeviceRounds: return device_rounds_flags_ok(flags, R);
        case kOpRounds: return rounds_flags_ok(flags, R);
        case kOpPrefix: return true;
        default: return !(flags & EGPU_F_PACKED);
    }
}

// Grid of a persistent launch (the one-launch rounds, the multi-batch sharded prefix-commit) of kernel k over
// batches of at most R rows: as many CTAs as round 1's CONTIG scan wants at 8 rows per thread (the lone-launch
// rule of launch_snapshot_as), at most one resident wave (the grid barriers need every CTA resident) and at
// least one CTA per device (CTA d cuts device d).  Also sizes the tile sums and PrefixOut for that grid, so
// that, with the caller's own scratch, everything is allocated before the launch and a failure commits nothing.
template <class Fn>
int persistent_grid(egpu_ctx* ctx, const Kernel<Fn>& k, int64_t R, int64_t* grid_out) {
    int per_sm = 0;
    const int rc = resident_ctas(ctx, k, &per_sm);
    if (rc != EGPU_OK) return rc;
    if (ctx->ctas_per_sm_cap > 0 && ctx->ctas_per_sm_cap < per_sm) per_sm = ctx->ctas_per_sm_cap;
    const int64_t wave = static_cast<int64_t>(ctx->sm_count) * per_sm;
    const int64_t per_cta = static_cast<int64_t>(kRoundsThreads) * 2;  // 128-bit vectors of 4 rows
    int64_t grid = ((R >> 2) + per_cta - 1) / per_cta;
    if (grid > wave) grid = wave;
    if (grid < ctx->D) grid = ctx->D;
    if (grid > wave) return EGPU_ERR_STATE;  // fewer resident CTAs than devices: not on an H100
    const size_t sums_bytes = sizeof(unsigned long long) * 2 * kMaxD * static_cast<size_t>(grid);
    EGPU_CUDA(ctx, grow(ctx->tile_bytes, sums_bytes, sums_bytes, &ctx->d_tile_sums));
    if (!ctx->d_prefix_out) EGPU_CUDA(ctx, cudaMalloc(&ctx->d_prefix_out, sizeof(PrefixOut) + sizeof(long long) * 2 * kMaxD));
    *grid_out = grid;
    return EGPU_OK;
}

// The cooperative launch of a persistent kernel on `grid` CTAs (persistent_grid): the runtime refuses a grid it
// cannot co-schedule rather than letting its barriers wait.
template <class Fn, class A>
int launch_persistent(egpu_ctx* ctx, const Kernel<Fn>& k, int64_t grid, cudaStream_t s, const A& args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(static_cast<unsigned>(grid));
    cfg.blockDim = dim3(static_cast<unsigned>(k.threads));
    cfg.dynamicSmemBytes = k.smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    EGPU_CUDA(ctx, cudaLaunchKernelEx(&cfg, k.fn, ctx->d_state, args));
    ctx->launches += 1;
    ctx->prev_is_scan = false;
    return EGPU_OK;
}

// EGPU_F_DEVICE_ROUNDS: the rounds of run_rounds with no round limit, in ONE cooperative launch of
// rounds_sorted_kernel / rounds_lut_kernel (egpu_scan.cuh) and without a host round trip: nothing
// here waits for the device.  Rows in either format (see prefix_scan).  Per batch, d_delta (may be NULL)
// receives the demand committed over all rounds, d_table_out (may be NULL) the last round's table'.
// Scratch is the rounds scratch of run_rounds, sized before the launch.
// multi (egpu_bestfit_batches_dev): the K batches of `bs`, each to its fixed point against the table the
// batches before it committed, in one launch of the multi-batch twins; grid and scratch are those of the
// largest batch.  Otherwise bs[0] alone (K = 1) in the single-batch kernels.
int launch_device_rounds(egpu_ctx* ctx, const egpu_batch* bs, int K, bool multi, cudaStream_t s, RowFormat fmt) {
    if (ctx->variant == EGPU_VARIANT_GRID) return EGPU_ERR_STATE;  // no prefix-commit mode
    const bool lut = lut_variant(ctx);
    RoundsMultiArgs m;
    int64_t R = bs[0].R;
    if (multi) {  // two batches sharing an output: the later one would overwrite the earlier one's
        std::memset(&m, 0, sizeof m);
        if (batch_descs(ctx, bs, K, fmt, true, m.b, &R) < 0) return EGPU_ERR_INVALID;
    }
    const auto& k = select_kernel<kRoundsSorted, kRoundsLut>(ctx, lut, fmt);
    const auto& km = select_kernel<kRoundsMultiSorted, kRoundsMultiLut>(ctx, lut, fmt);
    int64_t grid = 0;
    int rc = multi ? persistent_grid(ctx, km, R, &grid) : persistent_grid(ctx, k, R, &grid);
    if (rc != EGPU_OK) return rc;
    RoundsArgs a;
    rc = rounds_args(ctx, bs[0], R, fmt, s, &a);
    if (rc != EGPU_OK) return rc;
    if (multi) {
        m.a = a;
        m.K = K;
        rc = launch_persistent(ctx, km, grid, s, m);
    } else {
        rc = launch_persistent(ctx, k, grid, s, a);
    }
    if (rc != EGPU_OK) return rc;
    return table_changed(ctx, s, lut);  // the lookup kernels leave d_lut built from the table they committed
}

// Prefix-commit over row shards (one rank per GPU, rank-major row order).  Two exchange
// steps: `step` carries the uncapped demand of every shard (pushed by the scan itself),
// `step + 1` the committed demand after the cut (pushed by prefix_push_kernel).  Rows in either
// format (see prefix_scan); base, push and apply do not see them.
int launch_prefix_commit_shard(egpu_ctx* ctx, const int32_t* d_rc, const int32_t* d_rm, int64_t R, int32_t* d_idx,
                               long long* d_delta, int32_t* d_table_out, int user_flags, uint64_t step, cudaStream_t s,
                               RowFormat fmt) {
    PrefixOut* pf = nullptr;
    int n_tiles = 0;
    const int rc = prefix_scan(ctx, d_rc, d_rm, R, d_idx, fmt, step + 1, s, &pf, &n_tiles);
    if (rc != EGPU_OK) return rc;
    long long* base = reinterpret_cast<long long*>(pf + 1);
    prefix_base_kernel<<<1, kMaxD, 0, s>>>(ctx->d_state, step + 1, base);
    if (fmt == kRowsPacked) {
        signed char* idx8 = reinterpret_cast<signed char*>(d_idx);
        prefix_cut_packed_shard_kernel<<<ctx->D, 256, 0, s>>>(ctx->d_state, idx8, reinterpret_cast<const uint32_t*>(d_rc), R, n_tiles,
                                                              ctx->d_tile_sums, pf, base);
        prefix_apply_packed_kernel<<<capped_blocks(ctx, R, 1024), 256, 0, s>>>(pf, ctx->D, R, idx8);
    } else {
        prefix_cut_kernel<<<ctx->D, 256, 0, s>>>(ctx->d_state, d_idx, d_rc, d_rm, R, n_tiles, ctx->d_tile_sums, pf, base);
        prefix_apply_kernel<<<capped_blocks(ctx, R, 1024), 256, 0, s>>>(pf, ctx->D, R, d_idx);
    }
    prefix_push_kernel<<<1, kMaxD, 0, s>>>(ctx->d_state, pf, step + 2, d_delta);
    ApplyOuts outs{};
    outs.table_out[0] = d_table_out;
    apply_peers_kernel<<<1, kMaxD, 0, s>>>(ctx->d_state, step + 2, 1, outs, (user_flags & EGPU_F_COMMIT) ? 1 : 0);
    EGPU_CUDA(ctx, cudaGetLastError());
    ctx->launches += 5;
    ctx->prev_is_scan = false;
    return (user_flags & EGPU_F_COMMIT) ? table_changed(ctx, s) : EGPU_OK;
}

// K sharded prefix-commits in ONE cooperative launch of shard_prefix_multi_sorted_kernel /
// shard_prefix_multi_lut_kernel (egpu_scan.cuh): batch k is launch_prefix_commit_shard with
// step = first_step + 2k, scored against the table batch k - 1 left (with commit, the one it installed).
// Grid: persistent_grid of the largest batch; scratch: the tile sums, PrefixOut and the head of the rounds
// scratch (barrier words, stop word), all allocated before the launch.
int launch_shard_prefix_multi(egpu_ctx* ctx, const egpu_batch* bs, int K, bool commit, uint64_t first_step, cudaStream_t s,
                              RowFormat fmt) {
    if (ctx->variant == EGPU_VARIANT_GRID) return EGPU_ERR_STATE;  // no prefix-commit mode
    const bool lut = lut_variant(ctx);
    ShardPrefixArgs a;
    std::memset(&a, 0, sizeof a);
    int64_t R = 0;
    // the later batch would overwrite the earlier one's outputs
    if (batch_descs(ctx, bs, K, fmt, true, a.b, &R) < 0) return EGPU_ERR_INVALID;
    const auto& k = select_kernel<kShardPrefixSorted, kShardPrefixLut>(ctx, lut, fmt);
    int64_t grid = 0;
    int rc = persistent_grid(ctx, k, R, &grid);
    if (rc != EGPU_OK) return rc;
    RoundsScratch sc;
    rc = rounds_scratch(ctx, 0, fmt == kRowsPacked, &sc);  // the head only
    if (rc != EGPU_OK) return rc;
    rc = rounds_ctl(ctx, s, &a.ctl);
    if (rc != EGPU_OK) return rc;
    a.tile_sums = ctx->d_tile_sums;
    a.pf = static_cast<PrefixOut*>(ctx->d_prefix_out);
    a.stop = reinterpret_cast<unsigned int*>(static_cast<char*>(ctx->d_rounds) + kShardStopOff);
    a.lut = ctx->d_lut;
    a.first_step_plus1 = first_step + 1;
    a.K = K;
    a.commit = commit ? 1 : 0;
    rc = launch_persistent(ctx, k, grid, s, a);
    if (rc != EGPU_OK) return rc;
    // the lookup kernel leaves d_lut built from the table it last scored against or installed
    return (lut || commit) ? table_changed(ctx, s, lut) : EGPU_OK;
}

// Sharded rounds to the fixed point in ONE cooperative launch of shard_rounds_sorted_kernel / shard_rounds_lut_kernel
// (egpu_scan.cuh): launch_prefix_commit_shard on exchange steps `step` and `step + 1`, committing, then every later
// round on the same two steps, until no rank has a deferred row.  Grid: persistent_grid of this rank's R; scratch:
// the rounds scratch of launch_device_rounds, sized by R, and the barrier, stop and again words in its head, all
// allocated before the launch.  Nothing here waits for the device.
int launch_shard_rounds(egpu_ctx* ctx, const egpu_batch& b, uint64_t step, cudaStream_t s, RowFormat fmt) {
    if (ctx->variant == EGPU_VARIANT_GRID) return EGPU_ERR_STATE;  // no prefix-commit mode
    const bool lut = lut_variant(ctx);
    const auto& k = select_kernel<kShardRoundsSorted, kShardRoundsLut>(ctx, lut, fmt);
    int64_t grid = 0;
    int rc = persistent_grid(ctx, k, b.R, &grid);
    if (rc != EGPU_OK) return rc;
    ShardRoundsArgs a;
    std::memset(&a, 0, sizeof a);
    rc = rounds_args(ctx, b, b.R, fmt, s, &a.a);
    if (rc != EGPU_OK) return rc;
    a.stop = reinterpret_cast<unsigned int*>(static_cast<char*>(ctx->d_rounds) + kShardStopOff);
    a.again = reinterpret_cast<unsigned int*>(static_cast<char*>(ctx->d_rounds) + kShardAgainOff);
    a.step_plus1 = step + 1;
    rc = launch_persistent(ctx, k, grid, s, a);
    if (rc != EGPU_OK) return rc;
    return table_changed(ctx, s, lut);  // the lookup kernel leaves d_lut built from the table it committed
}

// Packed-format scan: always a fully ordered launch (it serves the synchronous host path).
int launch_packed(egpu_ctx* ctx, const uint32_t* d_req, int64_t R, signed char* d_idx8, long long* d_delta,
                  int32_t* d_table_out, int user_flags, cudaStream_t s, int rows_per_thread) {
    const auto& k = kKernels<kScanPacked, kRowsPacked>[d_bucket(ctx->D)];
    int per_sm = 0;
    int rc = resident_ctas(ctx, k, &per_sm);
    if (rc != EGPU_OK) return rc;
    const int64_t nchunk = R >> 9;  // 512 requests per warp trip
    const int64_t per_cta = static_cast<int64_t>(k.threads / 32) * ((rows_per_thread + 15) / 16);
    int64_t want = (nchunk + per_cta - 1) / per_cta;
    const int64_t cap = static_cast<int64_t>(ctx->sm_count) * per_sm;
    if (want > cap) want = cap;
    if (want < 1) want = 1;
    if (R / (want * k.threads) + 16 >= (1ll << 19)) return EGPU_ERR_INVALID;
    const int flags = kFlagFinalize | ((user_flags & EGPU_F_COMMIT) ? kFlagCommit : 0);
    const unsigned long long slot = ctx->seq % kEpiSlots;
    rc = launch_pdl(ctx, k, want, s, ctx->d_state, d_req, static_cast<long long>(R), d_idx8, d_delta, d_table_out, flags, slot);
    if (rc != EGPU_OK) return rc;
    ctx->launches += 1;
    ctx->seq += 1;
    new_group(ctx);
    ctx->prev_is_scan = false;  // the int32 scans do not pipeline behind this one
    return (flags & kFlagCommit) ? table_changed(ctx, s) : EGPU_OK;
}

// EGPU_F_RELEASE (spec 2.8): the R rows (d_rc, d_rm) give back what they hold on device d_idx[r], all or
// nothing, in one launch of release_rows_kernel.  Rows in either format (see prefix_scan); the indices are
// read, never written.  d_delta (may be NULL) receives the sums, d_table_out (may be NULL) table + sums or,
// refused, the table, and the per-device reason words; EGPU_F_COMMIT installs an accepted result.  An ordinary
// launch, fully ordered behind everything on the stream, whatever the context's scan variant.  Grid: the
// lone-launch rule of launch_snapshot_as (8 rows per thread, one resident wave, two from 16 Mi rows).
// step_plus1 (egpu_bestfit_batch_shard_prefix_dev): the rows are this rank's shard, and the decision is taken on
// every rank's sums, exchanged under step step_plus1 - 1 in the last CTA; 0 for one GPU.
int launch_release(egpu_ctx* ctx, const int32_t* d_rc, const int32_t* d_rm, int64_t R, const int32_t* d_idx, long long* d_delta,
                   int32_t* d_table_out, int user_flags, cudaStream_t s, RowFormat fmt, uint64_t step_plus1) {
    const bool commit = (user_flags & EGPU_F_COMMIT) != 0;
    const auto& k = select_kernel<kRelease, kReleaseShard>(ctx, step_plus1 != 0, fmt);
    int per_sm = 0;
    const int rc = resident_ctas(ctx, k, &per_sm);
    if (rc != EGPU_OK) return rc;
    Range mine[3];
    batch_ranges(mine, nullptr, 0, 0, d_delta, d_table_out, ctx->D);
    if (prepare_ranges(mine, 3) < 0) return EGPU_ERR_INVALID;  // the sums and table' overlap
    const int rpt = ctx->rows_per_thread > 0 ? ctx->rows_per_thread : 8;
    const int64_t per_cta = static_cast<int64_t>(k.threads) * ((rpt + 3) / 4);
    int64_t want = ((R >> 2) + per_cta - 1) / per_cta;
    if (ctx->ctas_per_sm_cap > 0 && ctx->ctas_per_sm_cap < per_sm) per_sm = ctx->ctas_per_sm_cap;
    const int64_t cap = static_cast<int64_t>(ctx->sm_count) * per_sm * (R >= (16ll << 20) ? 2 : 1);
    if (want > cap) want = cap;
    if (want < 1) want = 1;
    // lane-private sums hold 2^19 rows per lane (kAccShift)
    if (R / (want * k.threads) + 8 >= (1ll << 19)) return EGPU_ERR_INVALID;
    k.fn<<<static_cast<unsigned>(want), k.threads, k.smem, s>>>(ctx->d_state, d_rc, d_rm, static_cast<long long>(R), d_idx, d_delta,
                                                                d_table_out, commit ? kFlagCommit : 0,
                                                                static_cast<int>(ctx->seq % kEpiSlots), step_plus1);
    EGPU_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    ctx->seq += 1;
    new_group(ctx);
    ctx->prev_is_scan = false;
    return commit ? table_changed(ctx, s) : EGPU_OK;  // a refused launch leaves the table as it was: a rebuild is harmless
}

// staging of the host-buffer entry points: three arrays of at least `rows` int32, doubling
int ensure_staging(egpu_ctx* ctx, int64_t rows) {
    const size_t need = sizeof(int32_t) * static_cast<size_t>(rows);
    size_t bytes = ctx->staging_bytes ? ctx->staging_bytes : sizeof(int32_t) * 1024;
    while (bytes < need) bytes *= 2;
    EGPU_CUDA(ctx, grow(ctx->staging_bytes, need, bytes, &ctx->d_req_core, &ctx->d_req_mem, &ctx->d_idx));
    return EGPU_OK;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// The row arrays of an entry point in format fmt: present when there are rows and, device arrays, 16-byte aligned
// (the scans move 128-bit vectors).  Packed rows are words in rc with rm NULL, so that packed rows handed over
// without EGPU_F_PACKED (rm NULL, R > 0) are refused rather than read as int32 arrays.
bool arrays_ok(RowFormat fmt, int64_t R, const void* rc, const void* rm, const void* idx, bool device = true) {
    auto ok = [&](const void* p) { return (R <= 0 || p) && (!device || aligned16(p)); };
    return ok(rc) && ok(idx) && (fmt == kRowsPacked ? !rm : ok(rm));
}

// Host forms: the caller's rows into the staging arrays (rm: NULL for packed rows; idx: only when the indices are
// an input, idx_bytes each) ...
int stage_in(egpu_ctx* ctx, cudaStream_t s, int64_t R, const void* rc, const void* rm, const void* idx, size_t idx_bytes) {
    const int e = ensure_staging(ctx, R > 0 ? R : 1);
    if (e != EGPU_OK) return e;
    if (R > 0) {
        EGPU_CUDA(ctx, cudaMemcpyAsync(ctx->d_req_core, rc, sizeof(int32_t) * R, cudaMemcpyHostToDevice, s));
        if (rm) EGPU_CUDA(ctx, cudaMemcpyAsync(ctx->d_req_mem, rm, sizeof(int32_t) * R, cudaMemcpyHostToDevice, s));
        if (idx) EGPU_CUDA(ctx, cudaMemcpyAsync(ctx->d_idx, idx, idx_bytes * R, cudaMemcpyHostToDevice, s));
    }
    return EGPU_OK;
}
// ... and back, before the synchronisation: the indices (idx: NULL when they were an input) and, `sums`, the demand
// sums into ctx->h_delta
int stage_out(egpu_ctx* ctx, cudaStream_t s, int64_t R, void* idx, size_t idx_bytes, bool sums) {
    if (idx && R > 0) EGPU_CUDA(ctx, cudaMemcpyAsync(idx, ctx->d_idx, idx_bytes * R, cudaMemcpyDeviceToHost, s));
    if (sums) EGPU_CUDA(ctx, cudaMemcpyAsync(ctx->h_delta, ctx->d_delta, sizeof(long long) * 2 * ctx->D, cudaMemcpyDeviceToHost, s));
    return EGPU_OK;
}
// a call's demand sums (host, core then mem) into the caller's arrays, each of which may be NULL
void sums_out(const egpu_ctx* ctx, const long long* sums, int64_t* core, int64_t* mem) {
    if (core) std::memcpy(core, sums, sizeof(int64_t) * ctx->D);
    if (mem) std::memcpy(mem, sums + ctx->D, sizeof(int64_t) * ctx->D);
}

// egpu_bestfit_batch[_dev] after their checks, on device arrays: the caller's, or the host form's staging.  total:
// host int64[2*D], where the packed rounds leave the demand they committed over all rounds.
int run_batch(egpu_ctx* ctx, BatchOp op, RowFormat fmt, const int32_t* rc, const int32_t* rm, int64_t R, int32_t* idx,
              long long* delta, int32_t* table_out, int flags, cudaStream_t s, long long* total) {
    switch (op) {
        case kOpRelease: return launch_release(ctx, rc, rm, R, idx, delta, table_out, flags, s, fmt, 0);
        case kOpDeviceRounds: {
            const egpu_batch one{rc, rm, R, idx, reinterpret_cast<int64_t*>(delta), table_out};
            return launch_device_rounds(ctx, &one, 1, false, s, fmt);
        }
        case kOpRounds: return launch_packed_rounds(ctx, rc, R, idx, delta, table_out, total, s);
        case kOpPrefix: return launch_prefix_commit(ctx, rc, rm, R, idx, delta, table_out, flags, s, fmt);
        default: return launch_snapshot(ctx, Snapshot{rc, rm, R, idx, delta, table_out, flags}, s);
    }
}

// What an entry point needs of the context, each level including the ones before it.
enum Needs { kNeedsDevice, kNeedsTable, kNeedsPeers };

// The part of an entry point after it took ctx->mu: checks the state it needs, selects the
// context's device and the stream to launch on (the caller's, or the context's for nullptr).
int enter(egpu_ctx* ctx, Needs needs, void* stream, cudaStream_t* s) {
    if (needs >= kNeedsTable && !ctx->has_table) return EGPU_ERR_NO_TABLE;
    if (needs >= kNeedsPeers && !ctx->attached) return EGPU_ERR_STATE;
    EGPU_CUDA(ctx, cudaSetDevice(ctx->dev));
    *s = stream ? static_cast<cudaStream_t>(stream) : ctx->stream;
    return EGPU_OK;
}

// device-visible alias of a pinned (mapped) host allocation, nullptr for anything else
void* mapped_alias(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        (void)cudaGetLastError();
        return nullptr;
    }
    return (a.type == cudaMemoryTypeHost) ? a.devicePointer : nullptr;
}

}  // namespace

extern "C" {

// 1.4: + multi-batch launches, stateless query, start gate (additive)
// 1.5: + egpu_preferred_allocation_batch (additive)
// 1.6: + EGPU_F_PACKED multi-batch launches (additive)
// 1.7: + EGPU_F_PACKED prefix-commit on egpu_bestfit_batch / egpu_bestfit_batch_dev (additive)
// 1.8: + EGPU_F_ROUNDS, packed prefix-commit rounds on the same two entry points (additive)
// 1.9: + EGPU_F_PACKED on egpu_bestfit_batch_shard_dev, _shard_lag_dev and _shard_prefix_dev (additive)
// 1.10: + EGPU_F_DEVICE_ROUNDS, rounds in one launch on egpu_bestfit_batch / egpu_bestfit_batch_dev (additive)
// 1.11: + EGPU_F_DEVICE_ROUNDS on egpu_bestfit_batches_dev, K batches placed in order in one launch (additive)
//       + EGPU_F_PREFIX_COMMIT on egpu_bestfit_batches_shard_dev, K sharded prefix-commits in one launch (a newly
//         accepted flag set on an existing entry point; the version stays 1011, which callers and tests pin)
int egpu_abi_version(void) { return 1011; }

const char* egpu_strerror(int code) {
    switch (code) {
        case EGPU_OK: return "ok";
        case EGPU_ERR_INVALID: return "invalid argument";
        case EGPU_ERR_NO_DEVICE: return "no usable CUDA device (this library has no CPU fallback)";
        case EGPU_ERR_CUDA: return "CUDA runtime error";
        case EGPU_ERR_NOMEM: return "out of memory";
        case EGPU_ERR_NO_TABLE: return "capacity table not set";
        case EGPU_ERR_STATE: return "call not valid in the current state";
        case EGPU_ERR_PARSE: return "malformed device id";
        case EGPU_ERR_UNSAT: return "preferred allocation cannot be satisfied";
        default: return "unknown error";
    }
}

int egpu_ctx_create(int cuda_device, egpu_ctx** out) {
    if (!out) return EGPU_ERR_INVALID;
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        (void)cudaGetLastError();
        return EGPU_ERR_NO_DEVICE;
    }
    if (cuda_device < 0 || cuda_device >= n) return EGPU_ERR_INVALID;
    egpu_ctx* ctx = new (std::nothrow) egpu_ctx();
    if (!ctx) return EGPU_ERR_NOMEM;
    ctx->dev = cuda_device;
    int rc = [&]() -> int {
        EGPU_CUDA(ctx, cudaSetDevice(cuda_device));
        cudaDeviceProp prop;
        EGPU_CUDA(ctx, cudaGetDeviceProperties(&prop, cuda_device));
        ctx->sm_count = prop.multiProcessorCount;
        if (const char* e = std::getenv("EGPU_CTAS_PER_SM")) ctx->ctas_per_sm_cap = std::atoi(e);
        if (const char* e = std::getenv("EGPU_ROWS_PER_THREAD")) ctx->rows_per_thread = std::atoi(e);
        if (const char* e = std::getenv("EGPU_REPLAY_GENERAL")) ctx->replay_general = std::atoi(e) != 0;
        if (const char* e = std::getenv("EGPU_REPLAY_VARIANT")) ctx->replay_variant = std::atoi(e);
        if (const char* e = std::getenv("EGPU_MULTI_RPT")) ctx->multi_rpt = std::max(4, std::min(4096, std::atoi(e)));
        if (const char* e = std::getenv("EGPU_PIPE_GROUP")) {
            const int g = std::atoi(e);
            ctx->pipe_group = g < 1 ? 1 : (g > kPipeGroupMax ? kPipeGroupMax : g);
        }
        EGPU_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
        EGPU_CUDA(ctx, cudaMalloc(&ctx->d_state, sizeof(DevState)));
        EGPU_CUDA(ctx, cudaMemsetAsync(ctx->d_state, 0, sizeof(DevState), ctx->stream));
        EGPU_CUDA(ctx, cudaMalloc(&ctx->d_lut, sizeof(DevLut)));
        EGPU_CUDA(ctx, cudaMalloc(&ctx->d_xchg, sizeof(XchgBuf)));
        EGPU_CUDA(ctx, cudaMemsetAsync(ctx->d_xchg, 0, sizeof(XchgBuf), ctx->stream));
        EGPU_CUDA(ctx, cudaMalloc(&ctx->d_delta, sizeof(long long) * 2 * kMaxD));
        EGPU_CUDA(ctx, cudaMalloc(&ctx->d_table_out, sizeof(int32_t) * 3 * kMaxD));
        EGPU_CUDA(ctx, cudaMallocHost(&ctx->h_delta, sizeof(long long) * 2 * kMaxD));
        EGPU_CUDA(ctx, cudaHostGetDevicePointer(reinterpret_cast<void**>(&ctx->h_delta_dev), ctx->h_delta, 0));
        if (const char* e = std::getenv("EGPU_NO_ZERO_COPY")) ctx->no_zero_copy = std::atoi(e) != 0;
        EGPU_CUDA(ctx, cudaMallocHost(&ctx->h_table, sizeof(int32_t) * 3 * kMaxD));
        EGPU_CUDA(ctx, cudaMallocHost(&ctx->h_qtable, offsetof(DevState, peer)));
        EGPU_CUDA(ctx, cudaMallocHost(&ctx->h_gate, sizeof(unsigned long long)));
        *ctx->h_gate = 0ull;
        EGPU_CUDA(ctx, cudaHostGetDevicePointer(reinterpret_cast<void**>(&ctx->h_gate_dev), ctx->h_gate, 0));
        EGPU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        return EGPU_OK;
    }();
    if (rc != EGPU_OK) {
        egpu_ctx_destroy(ctx);
        return rc;
    }
    *out = ctx;
    return EGPU_OK;
}

void egpu_ctx_destroy(egpu_ctx* ctx) {
    if (!ctx) return;
    if (ctx->dev >= 0) cudaSetDevice(ctx->dev);
    if (ctx->stream) {
        cudaStreamSynchronize(ctx->stream);
        cudaStreamDestroy(ctx->stream);
    }
    for (int r = 0; r < kMaxRanks; ++r)
        if (ctx->peer_open[r]) cudaIpcCloseMemHandle(ctx->peer_open[r]);
    cudaFree(ctx->d_xchg);
    cudaFree(ctx->d_tile_sums);
    cudaFree(ctx->d_rounds);
    cudaFree(ctx->d_prefix_out);
    cudaFree(ctx->arena);
    cudaFree(ctx->d_state);
    cudaFree(ctx->d_lut);
    cudaFree(ctx->d_req_core);
    cudaFree(ctx->d_req_mem);
    cudaFree(ctx->d_idx);
    cudaFree(ctx->d_delta);
    cudaFree(ctx->d_table_out);
    if (ctx->h_delta) cudaFreeHost(ctx->h_delta);
    if (ctx->h_table) cudaFreeHost(ctx->h_table);
    if (ctx->h_gate) cudaFreeHost(ctx->h_gate);
    if (ctx->h_qtable) cudaFreeHost(ctx->h_qtable);
    cudaFree(ctx->d_qstate);
    (void)cudaGetLastError();
    delete ctx;
}

const char* egpu_last_error(egpu_ctx* ctx) { return ctx ? ctx->last_err : ""; }
int egpu_backend(egpu_ctx* ctx) { return ctx ? 1 : EGPU_ERR_INVALID; }
int64_t egpu_launch_count(egpu_ctx* ctx) {
    if (!ctx) return 0;
    std::lock_guard<std::mutex> g(ctx->mu);
    return ctx->launches;
}

int egpu_set_variant(egpu_ctx* ctx, int variant) {
    if (!ctx || variant < EGPU_VARIANT_AUTO || variant > EGPU_VARIANT_LUT) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    ctx->variant = variant;
    return EGPU_OK;
}

int egpu_table_set(egpu_ctx* ctx, const int32_t* free_core, const int32_t* free_mem, int32_t D) {
    if (!ctx || !free_core || !free_mem || D < 1 || D > EGPU_MAX_DEVICES) return EGPU_ERR_INVALID;
    for (int d = 0; d < D; ++d) {
        if (free_core[d] < 0 || free_core[d] > EGPU_CORE_MAX) return EGPU_ERR_INVALID;
        if (free_mem[d] < 0 || free_mem[d] > EGPU_MEM_MAX) return EGPU_ERR_INVALID;
    }
    std::lock_guard<std::mutex> g(ctx->mu);
    return egpu_table_set_locked(ctx, free_core, free_mem, nullptr, D);
}

}  // extern "C"

// for the host-only translation units (egpu_restore.cc), which cannot see egpu_ctx
void egpu_note_error(egpu_ctx* ctx, const char* msg) {
    if (!ctx || !msg) return;
    std::lock_guard<std::mutex> g(ctx->mu);
    std::snprintf(ctx->last_err, sizeof ctx->last_err, "%s", msg);
}

// body of egpu_table_set; the caller holds ctx->mu and has validated the arguments
// (also used by egpu_table_restore_flat, egpu_devhash.cu, which installs its flags too)
int egpu_table_set_locked(egpu_ctx* ctx, const int32_t* free_core, const int32_t* free_mem, const int32_t* oversub, int32_t D) {
    EGPU_CUDA(ctx, cudaSetDevice(ctx->dev));
    DevState h;
    table_image(h, free_core, free_mem, oversub, D);
    // pageable source: the copy is staged before the call returns
    // only the table part: the peer configuration (egpu_peer_attach) and the epilogue slots
    // that follow stay as they are
    EGPU_CUDA(ctx, cudaMemcpyAsync(ctx->d_state, &h, offsetof(DevState, peer), cudaMemcpyHostToDevice, ctx->stream));
    EGPU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->D = D;
    ctx->has_table = true;
    ctx->prev_is_scan = false;
    ctx->lut_dirty = true;
    return EGPU_OK;
}

extern "C" {

int egpu_table_size(egpu_ctx* ctx) {
    if (!ctx) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    return ctx->has_table ? ctx->D : EGPU_ERR_NO_TABLE;
}

int egpu_table_get(egpu_ctx* ctx, int32_t* free_core, int32_t* free_mem, int32_t* oversub) {
    if (!ctx || !free_core || !free_mem) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->has_table) return EGPU_ERR_NO_TABLE;
    EGPU_CUDA(ctx, cudaSetDevice(ctx->dev));
    EGPU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    EGPU_CUDA(ctx, cudaMemcpy(ctx->h_table, ctx->d_state, sizeof(int32_t) * 3 * kMaxD, cudaMemcpyDeviceToHost));
    std::memcpy(free_core, ctx->h_table, sizeof(int32_t) * ctx->D);
    std::memcpy(free_mem, ctx->h_table + kMaxD, sizeof(int32_t) * ctx->D);
    if (oversub) std::memcpy(oversub, ctx->h_table + 2 * kMaxD, sizeof(int32_t) * ctx->D);
    return EGPU_OK;
}

int egpu_host_alloc(egpu_ctx* ctx, void** out, int64_t bytes) {
    if (!ctx || !out || bytes <= 0) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    EGPU_CUDA(ctx, cudaSetDevice(ctx->dev));
    EGPU_CUDA(ctx, cudaMallocHost(out, static_cast<size_t>(bytes)));
    return EGPU_OK;
}

void egpu_host_free(egpu_ctx* ctx, void* p) {
    if (!ctx || !p) return;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaSetDevice(ctx->dev);
    cudaFreeHost(p);
    (void)cudaGetLastError();
}

int egpu_host_register(egpu_ctx* ctx, void* p, int64_t bytes) {
    if (!ctx || !p || bytes <= 0) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    EGPU_CUDA(ctx, cudaSetDevice(ctx->dev));
    EGPU_CUDA(ctx, cudaHostRegister(p, static_cast<size_t>(bytes), cudaHostRegisterMapped | cudaHostRegisterPortable));
    return EGPU_OK;
}

int egpu_host_unregister(egpu_ctx* ctx, void* p) {
    if (!ctx || !p) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    EGPU_CUDA(ctx, cudaSetDevice(ctx->dev));
    EGPU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // nothing of ours may still be reading it
    EGPU_CUDA(ctx, cudaHostUnregister(p));
    return EGPU_OK;
}

int egpu_bestfit_batch_dev(egpu_ctx* ctx, const int32_t* d_req_core, const int32_t* d_req_mem, int64_t R,
                           int32_t* d_out_idx, int64_t* d_delta, int32_t* d_table_out, int flags,
                           void* stream) {
    // EGPU_F_PACKED: prefix-commit only, d_req_core = words, d_req_mem NULL, d_out_idx = int8 indices.
    // EGPU_F_ROUNDS: that, committing, to the fixed point; synchronises the stream.
    // EGPU_F_DEVICE_ROUNDS: rounds to the fixed point in either format, in one launch, asynchronous.
    // EGPU_F_RELEASE [| EGPU_F_COMMIT] [| EGPU_F_PACKED]: the rows give back what they hold on d_out_idx, which is read.
    BatchOp op;
    if (!ctx || R < 0 || !batch_op(flags, R, &op)) return EGPU_ERR_INVALID;
    const RowFormat fmt = row_format(flags);
    if (!arrays_ok(fmt, R, d_req_core, d_req_mem, d_out_idx)) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    int rc = enter(ctx, kNeedsTable, stream, &s);
    if (rc != EGPU_OK) return rc;
    long long total[2 * kMaxD];
    rc = run_batch(ctx, op, fmt, d_req_core, d_req_mem, R, d_out_idx, reinterpret_cast<long long*>(d_delta), d_table_out, flags, s,
                   total);
    if (rc != EGPU_OK || op != kOpRounds) return rc;
    EGPU_CUDA(ctx, cudaStreamSynchronize(s));
    return EGPU_OK;
}

// one check of every batch of a multi-batch call (see arrays_ok)
static int check_batches(const egpu_batch* batches, int32_t K, RowFormat fmt) {
    if (!batches || K < 1 || K > EGPU_MAX_BATCHES) return EGPU_ERR_INVALID;
    for (int k = 0; k < K; ++k) {
        const egpu_batch& b = batches[k];
        if (b.R < 0 || b.R > kMaxRows || !arrays_ok(fmt, b.R, b.d_req_core, b.d_req_mem, b.d_out_idx)) return EGPU_ERR_INVALID;
    }
    return EGPU_OK;
}
int egpu_bestfit_batches_dev(egpu_ctx* ctx, const egpu_batch* batches, int32_t K, int flags, void* stream) {
    // EGPU_F_DEVICE_ROUNDS (with exactly the flags of the single-batch call): the batches placed in order,
    // each committed to its fixed point, in one launch.  Otherwise a snapshot of every batch.
    const bool device_rounds = (flags & EGPU_F_DEVICE_ROUNDS) != 0;
    if (!ctx || (device_rounds ? !device_rounds_flags_ok(flags, 0) : (flags & ~(EGPU_F_INPUTS_READY | EGPU_F_PACKED)) != 0))
        return EGPU_ERR_INVALID;
    int rc = check_batches(batches, K, row_format(flags));
    if (rc != EGPU_OK) return rc;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    rc = enter(ctx, kNeedsTable, stream, &s);
    if (rc != EGPU_OK) return rc;
    if (device_rounds) return launch_device_rounds(ctx, batches, K, true, s, row_format(flags));
    return launch_multi(ctx, batches, K, flags, s, 0);
}

int egpu_bestfit_batches_shard_dev(egpu_ctx* ctx, const egpu_batch* batches, int32_t K, int flags, uint64_t first_step,
                                   void* stream) {
    // EGPU_F_PREFIX_COMMIT [| EGPU_F_COMMIT] [| EGPU_F_PACKED]: K sharded prefix-commits in order, in one launch, on
    // exchange steps first_step .. first_step + 2K - 1.  Otherwise K sharded snapshot steps.
    const bool prefix = (flags & EGPU_F_PREFIX_COMMIT) != 0;
    if (!ctx || first_step >= (1ull << 47) ||
        (flags & ~(prefix ? EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT | EGPU_F_PACKED : EGPU_F_INPUTS_READY | EGPU_F_APPLY)))
        return EGPU_ERR_INVALID;
    int rc = check_batches(batches, K, row_format(flags));
    if (rc != EGPU_OK) return rc;
    if (prefix && first_step + 2ull * static_cast<uint64_t>(K) > (1ull << 47)) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    rc = enter(ctx, kNeedsPeers, stream, &s);
    if (rc != EGPU_OK) return rc;
    if (prefix)
        return launch_shard_prefix_multi(ctx, batches, K, (flags & EGPU_F_COMMIT) != 0, first_step, s, row_format(flags));
    return launch_multi(ctx, batches, K, flags, s, first_step + 1);
}

int egpu_peer_gate_dev(egpu_ctx* ctx, void* stream) {
    if (!ctx) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    const int rc = enter(ctx, kNeedsDevice, stream, &s);
    if (rc != EGPU_OK) return rc;
    gate_kernel<<<1, 32, 0, s>>>(ctx->d_state, ctx->h_gate_dev);
    EGPU_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    ctx->prev_is_scan = false;
    return EGPU_OK;
}

int64_t egpu_peer_gate_timeouts(egpu_ctx* ctx) {
    if (!ctx) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (cudaSetDevice(ctx->dev) != cudaSuccess) return EGPU_ERR_CUDA;
    unsigned long long v = 0;
    if (cudaMemcpy(&v, reinterpret_cast<char*>(ctx->d_state) + offsetof(DevState, gate_timeouts), sizeof v,
                   cudaMemcpyDeviceToHost) != cudaSuccess) {
        (void)cudaGetLastError();
        return EGPU_ERR_CUDA;
    }
    return static_cast<int64_t>(v);
}

int64_t egpu_release_refusals(egpu_ctx* ctx) {
    if (!ctx) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (cudaSetDevice(ctx->dev) != cudaSuccess) return EGPU_ERR_CUDA;
    unsigned long long v = 0;
    // every stream, the non-blocking ones too: the launches counted may sit on any of them
    if (cudaDeviceSynchronize() != cudaSuccess ||
        cudaMemcpy(&v, reinterpret_cast<char*>(ctx->d_state) + offsetof(DevState, release_refusals), sizeof v,
                   cudaMemcpyDeviceToHost) != cudaSuccess) {
        (void)cudaGetLastError();
        return EGPU_ERR_CUDA;
    }
    return static_cast<int64_t>(v);
}

int egpu_peer_gate_open(egpu_ctx* ctx) {
    if (!ctx) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    __atomic_fetch_add(ctx->h_gate, 1ull, __ATOMIC_RELEASE);
    return EGPU_OK;
}

int egpu_bestfit_query(egpu_ctx* ctx, const int32_t* free_core, const int32_t* free_mem, int32_t D, const int32_t* req_core,
                       const int32_t* req_mem, int64_t R, int32_t* out_idx) {
    if (!ctx || !free_core || !free_mem || D < 1 || D > EGPU_MAX_DEVICES || R < 0 || R > kMaxRows) return EGPU_ERR_INVALID;
    if (R > 0 && (!req_core || !req_mem || !out_idx)) return EGPU_ERR_INVALID;
    for (int d = 0; d < D; ++d) {
        if (free_core[d] < 0 || free_core[d] > EGPU_CORE_MAX) return EGPU_ERR_INVALID;
        if (free_mem[d] < 0 || free_mem[d] > EGPU_MEM_MAX) return EGPU_ERR_INVALID;
    }
    if (R == 0) return EGPU_OK;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    int rc = enter(ctx, kNeedsDevice, nullptr, &s);
    if (rc != EGPU_OK) return rc;
    if (!ctx->d_qstate) {
        EGPU_CUDA(ctx, cudaMalloc(&ctx->d_qstate, sizeof(DevState)));
        EGPU_CUDA(ctx, cudaMemsetAsync(ctx->d_qstate, 0, sizeof(DevState), s));
    }
    // the scratch table: same layout and sorted view as the context's own, in its own DevState
    DevState* h = reinterpret_cast<DevState*>(ctx->h_qtable);
    table_image(*h, free_core, free_mem, nullptr, D);
    EGPU_CUDA(ctx, cudaMemcpyAsync(ctx->d_qstate, h, offsetof(DevState, peer), cudaMemcpyHostToDevice, s));
    rc = ensure_staging(ctx, R);
    if (rc != EGPU_OK) return rc;
    EGPU_CUDA(ctx, cudaMemcpyAsync(ctx->d_req_core, req_core, sizeof(int32_t) * R, cudaMemcpyHostToDevice, s));
    EGPU_CUDA(ctx, cudaMemcpyAsync(ctx->d_req_mem, req_mem, sizeof(int32_t) * R, cudaMemcpyHostToDevice, s));
    // the register scan whatever the context's variant: one table, used once - lookup tables would not pay
    const auto& k = kKernels<kScanSorted, kRowsInt32>[d_bucket(D)];
    int per_sm = 0;
    rc = resident_ctas(ctx, k, &per_sm);
    if (rc != EGPU_OK) return rc;
    const int64_t nvec = R >> 2;
    const int64_t per_cta = static_cast<int64_t>(k.threads) * 2;
    int64_t want = (nvec + per_cta - 1) / per_cta;
    const int64_t cap = static_cast<int64_t>(ctx->sm_count) * per_sm;
    if (want > cap) want = cap;
    if (want < 1) want = 1;
    if (R / (want * k.threads) + 8 >= (1ll << 19)) return EGPU_ERR_INVALID;
    // fully ordered launch (no PDL flags), epilogue slot 0 of the scratch state, nothing published
    k.fn<<<static_cast<unsigned>(want), k.threads, k.smem, s>>>(ctx->d_qstate, ctx->d_req_core, ctx->d_req_mem,
                                                                static_cast<long long>(R), ctx->d_idx, nullptr, nullptr,
                                                                kFlagFinalize, 0ull, nullptr);
    EGPU_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    ctx->prev_is_scan = false;
    EGPU_CUDA(ctx, cudaMemcpyAsync(out_idx, ctx->d_idx, sizeof(int32_t) * R, cudaMemcpyDeviceToHost, s));
    EGPU_CUDA(ctx, cudaStreamSynchronize(s));
    return EGPU_OK;
}

int egpu_bestfit_batch(egpu_ctx* ctx, const int32_t* req_core, const int32_t* req_mem, int64_t R,
                       int32_t* out_idx, int64_t* out_delta_core, int64_t* out_delta_mem, int commit) {
    // `commit` carries the flags of egpu_bestfit_batch_dev: EGPU_F_PACKED rows are req_core = words, req_mem NULL,
    // out_idx = int8 indices; with EGPU_F_RELEASE out_idx is an input, the devices the rows were placed on
    BatchOp op;
    if (!ctx || R < 0 || !batch_op(commit, R, &op)) return EGPU_ERR_INVALID;
    const RowFormat fmt = row_format(commit);
    if (!arrays_ok(fmt, R, req_core, req_mem, out_idx, false)) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    int rc = enter(ctx, kNeedsTable, nullptr, &s);
    if (rc != EGPU_OK) return rc;
    const int D = ctx->D;
    const int user_flags = commit & EGPU_F_COMMIT;
    // Zero-copy: when all three caller arrays of a snapshot are pinned (egpu_host_alloc or
    // cudaHostRegister) and 16-byte aligned, the scan reads the requests and writes
    // the indices straight across PCIe — one launch, no staging in HBM, reads and
    // writes overlap on the full-duplex link.  Demand sums land in pinned memory too.
    const bool mapped = R > 0 && op == kOpSnapshot;
    const int32_t* zc = mapped ? static_cast<const int32_t*>(mapped_alias(req_core)) : nullptr;
    const int32_t* zm = mapped ? static_cast<const int32_t*>(mapped_alias(req_mem)) : nullptr;
    int32_t* zi = mapped ? static_cast<int32_t*>(mapped_alias(out_idx)) : nullptr;
    if (zc && zm && zi && aligned16(zc) && aligned16(zm) && aligned16(zi) && !ctx->no_zero_copy) {
        // 64 rows per thread: few CTAs, many trips, so reads of later rows and writes of
        // earlier ones are on the link at the same time (PCIe is full duplex)
        Snapshot a{zc, zm, R, zi, ctx->h_delta_dev, nullptr, user_flags};
        a.rpt_hint = 64;
        rc = launch_snapshot(ctx, a, s);
        if (rc != EGPU_OK) return rc;
        EGPU_CUDA(ctx, cudaStreamSynchronize(s));
        sums_out(ctx, ctx->h_delta, out_delta_core, out_delta_mem);
        return EGPU_OK;
    }
    // Otherwise staged through HBM, per row int32 12 bytes in and 4 out (release: 12 in, nothing out), packed 4 in
    // and 1 out (release: 5 in).  The packed rounds keep their sums on the host (d_delta NULL: no copy to the
    // device); a release's table' carries the reason words of a refusal.
    const bool release = op == kOpRelease;
    const size_t idx_bytes = fmt == kRowsPacked ? sizeof(int8_t) : sizeof(int32_t);
    rc = stage_in(ctx, s, R, req_core, req_mem, release ? out_idx : nullptr, idx_bytes);
    if (rc != EGPU_OK) return rc;
    long long total[2 * kMaxD];
    rc = run_batch(ctx, op, fmt, ctx->d_req_core, ctx->d_req_mem, R, ctx->d_idx, op == kOpRounds ? nullptr : ctx->d_delta,
                   release ? ctx->d_table_out : nullptr, user_flags, s, total);
    if (rc != EGPU_OK) return rc;
    rc = stage_out(ctx, s, R, release ? nullptr : out_idx, idx_bytes, op != kOpRounds);
    if (rc != EGPU_OK) return rc;
    if (release) EGPU_CUDA(ctx, cudaMemcpyAsync(ctx->h_table, ctx->d_table_out, sizeof(int32_t) * 3 * D, cudaMemcpyDeviceToHost, s));
    unsigned long long timeouts = 0;
    if (op == kOpDeviceRounds)
        EGPU_CUDA(ctx, cudaMemcpyAsync(&timeouts, reinterpret_cast<char*>(ctx->d_state) + offsetof(DevState, rounds_timeouts),
                                       sizeof timeouts, cudaMemcpyDeviceToHost, s));
    EGPU_CUDA(ctx, cudaStreamSynchronize(s));
    if (op == kOpDeviceRounds && timeouts != ctx->rounds_timeouts_seen) {  // this launch, or a _dev launch since the last check, gave up
        ctx->rounds_timeouts_seen = timeouts;
        std::snprintf(ctx->last_err, sizeof ctx->last_err,
                      "EGPU_F_DEVICE_ROUNDS: a grid barrier waited more than 2 s and the launch gave up (%llu so far)", timeouts);
        return EGPU_ERR_CUDA;
    }
    sums_out(ctx, op == kOpRounds ? total : ctx->h_delta, out_delta_core, out_delta_mem);
    for (int d = 0; release && d < D; ++d) {
        const int32_t reason = ctx->h_table[2 * D + d];
        if (!reason) continue;
        std::snprintf(ctx->last_err, sizeof ctx->last_err, "EGPU_F_RELEASE refused, nothing released: device %d %s", d,
                      reason == EGPU_REL_FLAGGED ? "is oversubscribed (EGPU_REL_FLAGGED)"
                                                 : "would hold more than the domain allows (EGPU_REL_EXCEEDS)");
        return EGPU_ERR_STATE;
    }
    return EGPU_OK;
}

int egpu_bestfit_batch_rounds(egpu_ctx* ctx, const int32_t* req_core, const int32_t* req_mem, int64_t R, int32_t* out_idx,
                              int64_t* out_delta_core, int64_t* out_delta_mem, int32_t max_rounds, int32_t* out_rounds,
                              int64_t* out_deferred) {
    if (!ctx || R < 0 || R >= (1ll << 31) || max_rounds < 1) return EGPU_ERR_INVALID;
    if (!arrays_ok(kRowsInt32, R, req_core, req_mem, out_idx, false)) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    int rc = enter(ctx, kNeedsTable, nullptr, &s);
    if (rc != EGPU_OK) return rc;
    rc = stage_in(ctx, s, R, req_core, req_mem, nullptr, 0);
    if (rc != EGPU_OK) return rc;
    long long total[2 * kMaxD];
    int32_t rounds = 0;
    int64_t left = 0;
    rc = run_rounds(ctx, ctx->d_req_core, ctx->d_req_mem, R, ctx->d_idx, max_rounds, total, &rounds, &left, s);
    if (rc != EGPU_OK) return rc;
    rc = stage_out(ctx, s, R, out_idx, sizeof(int32_t), false);
    if (rc != EGPU_OK) return rc;
    EGPU_CUDA(ctx, cudaStreamSynchronize(s));
    sums_out(ctx, total, out_delta_core, out_delta_mem);
    if (out_rounds) *out_rounds = rounds;
    if (out_deferred) *out_deferred = left;
    return EGPU_OK;
}

int egpu_bestfit_batch_rounds_dev(egpu_ctx* ctx, const int32_t* d_req_core, const int32_t* d_req_mem, int64_t R,
                                  int32_t* d_out_idx, int64_t* out_delta /* host [2*D] */, int32_t max_rounds,
                                  int32_t* out_rounds, int64_t* out_deferred, void* stream) {
    if (!ctx || R < 0 || R >= (1ll << 31) || max_rounds < 1 || !arrays_ok(kRowsInt32, R, d_req_core, d_req_mem, d_out_idx))
        return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    int rc = enter(ctx, kNeedsTable, stream, &s);
    if (rc != EGPU_OK) return rc;
    long long total[2 * kMaxD];
    int32_t rounds = 0;
    int64_t left = 0;
    rc = run_rounds(ctx, d_req_core, d_req_mem, R, d_out_idx, max_rounds, total, &rounds, &left, s);
    if (rc != EGPU_OK) return rc;
    EGPU_CUDA(ctx, cudaStreamSynchronize(s));
    if (out_delta) std::memcpy(out_delta, total, sizeof(int64_t) * 2 * ctx->D);
    if (out_rounds) *out_rounds = rounds;
    if (out_deferred) *out_deferred = left;
    return EGPU_OK;
}

int egpu_peer_export(egpu_ctx* ctx, void* handle_out) {
    if (!ctx || !handle_out) return EGPU_ERR_INVALID;
    static_assert(sizeof(cudaIpcMemHandle_t) == EGPU_IPC_HANDLE_BYTES, "IPC handle size");
    std::lock_guard<std::mutex> g(ctx->mu);
    EGPU_CUDA(ctx, cudaSetDevice(ctx->dev));
    cudaIpcMemHandle_t h;
    EGPU_CUDA(ctx, cudaIpcGetMemHandle(&h, ctx->d_xchg));
    std::memcpy(handle_out, &h, sizeof h);
    return EGPU_OK;
}

int egpu_peer_attach(egpu_ctx* ctx, int rank, int world, const void* handles) {
    if (!ctx || !handles || world < 1 || world > kMaxRanks || rank < 0 || rank >= world) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (ctx->attached) return EGPU_ERR_STATE;
    EGPU_CUDA(ctx, cudaSetDevice(ctx->dev));
    PeerCfg cfg;
    std::memset(&cfg, 0, sizeof cfg);
    cfg.world = world;
    cfg.rank = rank;
    for (int r = 0; r < world; ++r) {
        if (r == rank) {
            cfg.buf[r] = ctx->d_xchg;
            continue;
        }
        cudaIpcMemHandle_t h;
        std::memcpy(&h, static_cast<const char*>(handles) + static_cast<size_t>(r) * sizeof h, sizeof h);
        void* p = nullptr;
        EGPU_CUDA(ctx, cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        ctx->peer_open[r] = p;
        cfg.buf[r] = static_cast<XchgBuf*>(p);
    }
    EGPU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    EGPU_CUDA(ctx, cudaMemcpy(reinterpret_cast<char*>(ctx->d_state) + offsetof(DevState, peer), &cfg, sizeof cfg,
                              cudaMemcpyHostToDevice));
    ctx->world = world;
    ctx->rank = rank;
    ctx->attached = true;
    return EGPU_OK;
}

int egpu_peer_detach(egpu_ctx* ctx) {
    if (!ctx) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->attached) return EGPU_OK;
    EGPU_CUDA(ctx, cudaSetDevice(ctx->dev));
    EGPU_CUDA(ctx, cudaDeviceSynchronize());
    for (int r = 0; r < kMaxRanks; ++r) {
        if (ctx->peer_open[r]) cudaIpcCloseMemHandle(ctx->peer_open[r]);
        ctx->peer_open[r] = nullptr;
    }
    ctx->attached = false;
    ctx->world = 1;
    ctx->rank = 0;
    return EGPU_OK;
}

int egpu_bestfit_batch_shard_dev(egpu_ctx* ctx, const int32_t* d_req_core, const int32_t* d_req_mem, int64_t R,
                                 int32_t* d_out_idx, int64_t* d_delta, int flags, uint64_t step, void* stream) {
    // the commit happens in apply_peers; prefix-commit over shards has its own entry point;
    // step + 1 travels in 48 bits of the launch word.  EGPU_F_PACKED: words in d_req_core, d_req_mem
    // NULL, int8 indices (as in egpu_bestfit_batch_dev)
    const RowFormat fmt = row_format(flags);
    if (!ctx || R < 0 || (flags & ~(EGPU_F_INPUTS_READY | EGPU_F_PACKED)) || step >= (1ull << 47)) return EGPU_ERR_INVALID;
    if (!arrays_ok(fmt, R, d_req_core, d_req_mem, d_out_idx)) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    const int rc = enter(ctx, kNeedsPeers, stream, &s);
    if (rc != EGPU_OK) return rc;
    Snapshot a{d_req_core, d_req_mem, R, d_out_idx, reinterpret_cast<long long*>(d_delta), nullptr, flags};
    a.push_step_plus1 = step + 1;
    a.packed = fmt == kRowsPacked;
    return launch_snapshot(ctx, a, s);
}

int egpu_bestfit_batch_shard_prefix_dev(egpu_ctx* ctx, const int32_t* d_req_core, const int32_t* d_req_mem, int64_t R,
                                        int32_t* d_out_idx, int64_t* d_delta, int32_t* d_table_out, int flags,
                                        uint64_t step, void* stream) {
    // EGPU_F_ROUNDS / EGPU_F_DEVICE_ROUNDS only as the flag set of the one-launch rounds, without
    // EGPU_F_INPUTS_READY: rounds to the fixed point over the shards, in one launch, on steps step and step + 1.
    // EGPU_F_RELEASE [| EGPU_F_COMMIT] [| EGPU_F_PACKED]: this rank's rows give back what they hold on d_out_idx
    // (read, never written), decided on every rank's sums, in one launch, on step `step`
    const RowFormat fmt = row_format(flags);
    const bool rounds = (flags & (EGPU_F_ROUNDS | EGPU_F_DEVICE_ROUNDS)) != 0;
    const bool release = (flags & EGPU_F_RELEASE) != 0;
    if (!ctx || R < 0 || step >= (1ull << 47)) return EGPU_ERR_INVALID;
    if (release ? !release_flags_ok(flags, R)
        : rounds ? (flags & ~EGPU_F_PACKED) != kDeviceRoundsNeeds || R >= (1ll << 31) || step + 2 > (1ull << 47)
                 : (flags & ~(EGPU_F_COMMIT | EGPU_F_PREFIX_COMMIT | EGPU_F_PACKED)) != 0)
        return EGPU_ERR_INVALID;
    if (!arrays_ok(fmt, R, d_req_core, d_req_mem, d_out_idx)) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    const int rc = enter(ctx, kNeedsPeers, stream, &s);
    if (rc != EGPU_OK) return rc;
    long long* delta = reinterpret_cast<long long*>(d_delta);
    if (release) return launch_release(ctx, d_req_core, d_req_mem, R, d_out_idx, delta, d_table_out, flags, s, fmt, step + 1);
    if (rounds) return launch_shard_rounds(ctx, egpu_batch{d_req_core, d_req_mem, R, d_out_idx, d_delta, d_table_out}, step, s, fmt);
    return launch_prefix_commit_shard(ctx, d_req_core, d_req_mem, R, d_out_idx, delta, d_table_out, flags, step, s, fmt);
}

int egpu_bestfit_batch_shard_lag_dev(egpu_ctx* ctx, const int32_t* d_req_core, const int32_t* d_req_mem, int64_t R,
                                     int32_t* d_out_idx, int64_t* d_delta, int flags, uint64_t step, int lag,
                                     int32_t* d_table_out_lagged, void* stream) {
    // This entry point never checked flags other than EGPU_F_COMMIT, so a call with EGPU_F_PACKED and
    // two int32 arrays has always run as int32 and still does: packed needs the flag AND a NULL d_req_mem.
    const RowFormat fmt = (flags & EGPU_F_PACKED) && !d_req_mem ? kRowsPacked : kRowsInt32;
    if (!ctx || R < 0 || (flags & EGPU_F_COMMIT) || lag < 1 || lag > 16 || step >= (1ull << 47)) return EGPU_ERR_INVALID;
    if (!arrays_ok(fmt, R, d_req_core, d_req_mem, d_out_idx)) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    const int rc = enter(ctx, kNeedsPeers, stream, &s);
    if (rc != EGPU_OK) return rc;
    Snapshot a{d_req_core, d_req_mem, R, d_out_idx, reinterpret_cast<long long*>(d_delta), d_table_out_lagged, flags};
    a.push_step_plus1 = step + 1;
    a.lag = lag;
    a.packed = fmt == kRowsPacked;
    return launch_snapshot(ctx, a, s);
}

int egpu_table_apply_peers_multi_dev(egpu_ctx* ctx, uint64_t first_step, int nsteps, int32_t* const* d_table_outs,
                                     int commit, void* stream) {
    if (!ctx || nsteps < 1 || nsteps > kApplyMax) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    const int rc = enter(ctx, kNeedsPeers, stream, &s);
    if (rc != EGPU_OK) return rc;
    if (commit) ctx->prev_is_scan = false;  // the next scan must see the new table
    ApplyOuts outs;
    for (int k = 0; k < kApplyMax; ++k) outs.table_out[k] = (d_table_outs && k < nsteps) ? d_table_outs[k] : nullptr;
    apply_peers_kernel<<<commit ? 1 : nsteps, kMaxD, 0, s>>>(ctx->d_state, first_step + 1, nsteps, outs, commit);
    EGPU_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    return commit ? table_changed(ctx, s) : EGPU_OK;
}

int egpu_table_apply_peers_dev(egpu_ctx* ctx, uint64_t step, int32_t* d_table_out, int commit, void* stream) {
    int32_t* outs[1] = {d_table_out};
    return egpu_table_apply_peers_multi_dev(ctx, step, 1, outs, commit, stream);
}

int64_t egpu_peer_last_timeout(egpu_ctx* ctx) {
    if (!ctx) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (cudaSetDevice(ctx->dev) != cudaSuccess) return EGPU_ERR_CUDA;
    unsigned long long v = 0;
    if (cudaMemcpy(&v, reinterpret_cast<char*>(ctx->d_state) + offsetof(DevState, peer_timeout), sizeof v,
                   cudaMemcpyDeviceToHost) != cudaSuccess) {
        (void)cudaGetLastError();
        return EGPU_ERR_CUDA;
    }
    return static_cast<int64_t>(v);
}

int egpu_bestfit_batch_packed_dev(egpu_ctx* ctx, const uint32_t* d_req_packed, int64_t R, int8_t* d_out_idx8,
                                  int64_t* d_delta, int32_t* d_table_out, int flags, void* stream) {
    if (!ctx || R < 0 || !arrays_ok(kRowsPacked, R, d_req_packed, nullptr, d_out_idx8)) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    const int rc = enter(ctx, kNeedsTable, stream, &s);
    if (rc != EGPU_OK) return rc;
    // The grid variant has no packed snapshot scan, and the snapshot scans index at most EGPU_MAX_ROWS rows:
    // those calls keep the warp-chunk scan of the host call, fully ordered.
    if (ctx->variant == EGPU_VARIANT_GRID || R > kMaxRows)
        return launch_packed(ctx, d_req_packed, R, reinterpret_cast<signed char*>(d_out_idx8), reinterpret_cast<long long*>(d_delta),
                             d_table_out, flags, s, 16);
    // Otherwise the round-robin packed scan of the sharded calls, in the variant's scan (register scan up to
    // D = 16 under AUTO, lookup scan above), pipelined under EGPU_F_INPUTS_READY as the int32 call is.  Other
    // flag bits are ignored: callers may pass them, and EGPU_F_PREFIX_COMMIT must not turn this into prefix-commit.
    Snapshot a{reinterpret_cast<const int32_t*>(d_req_packed), nullptr, R, reinterpret_cast<int32_t*>(d_out_idx8),
               reinterpret_cast<long long*>(d_delta), d_table_out, flags & (EGPU_F_COMMIT | EGPU_F_INPUTS_READY)};
    a.packed = true;
    return launch_snapshot(ctx, a, s);
}

int egpu_bestfit_batch_packed(egpu_ctx* ctx, const uint32_t* req_packed, int64_t R, int8_t* out_idx8,
                              int64_t* out_delta_core, int64_t* out_delta_mem, int commit) {
    if (!ctx || R < 0 || !arrays_ok(kRowsPacked, R, req_packed, nullptr, out_idx8, false)) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    int rc = enter(ctx, kNeedsTable, nullptr, &s);
    if (rc != EGPU_OK) return rc;
    const uint32_t* zr = R > 0 ? static_cast<const uint32_t*>(mapped_alias(req_packed)) : nullptr;
    signed char* zi = R > 0 ? static_cast<signed char*>(mapped_alias(out_idx8)) : nullptr;
    if (zr && zi && aligned16(zr) && aligned16(zi) && !ctx->no_zero_copy) {  // zero-copy across PCIe, see egpu_bestfit_batch
        rc = launch_packed(ctx, zr, R, zi, ctx->h_delta_dev, nullptr, commit ? EGPU_F_COMMIT : 0, s, 128);
        if (rc != EGPU_OK) return rc;
        EGPU_CUDA(ctx, cudaStreamSynchronize(s));
    } else {
        rc = stage_in(ctx, s, R, req_packed, nullptr, nullptr, 0);  // d_req_core holds the packed words, d_idx the bytes
        if (rc != EGPU_OK) return rc;
        rc = launch_packed(ctx, reinterpret_cast<const uint32_t*>(ctx->d_req_core), R, reinterpret_cast<signed char*>(ctx->d_idx),
                           ctx->d_delta, nullptr, commit ? EGPU_F_COMMIT : 0, s, 16);
        if (rc != EGPU_OK) return rc;
        rc = stage_out(ctx, s, R, out_idx8, sizeof(int8_t), true);
        if (rc != EGPU_OK) return rc;
        EGPU_CUDA(ctx, cudaStreamSynchronize(s));
    }
    sums_out(ctx, ctx->h_delta, out_delta_core, out_delta_mem);
    return EGPU_OK;
}

int egpu_table_apply_deltas_dev(egpu_ctx* ctx, const int64_t* d_deltas, int G, int32_t* d_table_out,
                                int commit, void* stream) {
    if (!ctx || !d_deltas || G < 1) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    const int rc = enter(ctx, kNeedsTable, stream, &s);
    if (rc != EGPU_OK) return rc;
    ctx->prev_is_scan = false;
    apply_deltas_kernel<<<1, kMaxD, 0, s>>>(ctx->d_state, reinterpret_cast<const long long*>(d_deltas), G,
                                            d_table_out, commit);
    EGPU_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    return commit ? table_changed(ctx, s) : EGPU_OK;
}

int egpu_synth_requests_dev(egpu_ctx* ctx, int dist, uint64_t seed, int64_t first_row, int64_t R,
                            int32_t* d_req_core, int32_t* d_req_mem, void* stream) {
    if (!ctx || R < 0 || first_row < 0 || (dist != 2 && dist != 3 && dist != 4)) return EGPU_ERR_INVALID;
    if (R == 0) return EGPU_OK;
    if (!d_req_core || !d_req_mem) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaStream_t s;
    const int rc = enter(ctx, kNeedsDevice, stream, &s);
    if (rc != EGPU_OK) return rc;
    ctx->prev_is_scan = false;
    synth_requests_kernel<<<capped_blocks(ctx, R, 256), 256, 0, s>>>(dist, seed, first_row, R, d_req_core, d_req_mem);
    EGPU_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    return EGPU_OK;
}

int egpu_replay(egpu_ctx* ctx, const int32_t* kind, const int32_t* a, const int32_t* b, int64_t E,
                int32_t* out_idx) {
    if (!ctx || E < 0 || E > 0x7fffffffll) return EGPU_ERR_INVALID;
    if (E > 0 && (!kind || !a || !b || !out_idx)) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->has_table) return EGPU_ERR_NO_TABLE;
    if (E == 0) return EGPU_OK;
    EGPU_CUDA(ctx, cudaSetDevice(ctx->dev));
    // staging comes from the context's grow-only arena (three inputs, one output, the `live`
    // map when it does not fit in shared memory): no cudaMalloc/cudaFree on the call path
    cudaStream_t s = ctx->stream;
    const size_t ebytes = sizeof(int32_t) * static_cast<size_t>(E);
    void *kind_p, *a_p, *b_p, *out_p, *live_p = nullptr;
    const ArenaWant wants[] = {{&kind_p, ebytes}, {&a_p, ebytes}, {&b_p, ebytes}, {&out_p, ebytes}, {&live_p, static_cast<size_t>(E)}};
    EGPU_CUDA(ctx, arena_carve(ctx, wants, E > kReplaySmemEvents ? 5 : 4));
    int32_t* d_kind = static_cast<int32_t*>(kind_p);
    int32_t* d_a = static_cast<int32_t*>(a_p);
    int32_t* d_b = static_cast<int32_t*>(b_p);
    int32_t* d_out = static_cast<int32_t*>(out_p);
    signed char* d_live = static_cast<signed char*>(live_p);
    size_t smem = 0;
    if (E <= kReplaySmemEvents) {
        smem = static_cast<size_t>((E + 15) & ~15ll);
        if (!ctx->replay_configured) {
            EGPU_CUDA(ctx, cudaFuncSetAttribute(replay_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kReplaySmemEvents));
            EGPU_CUDA(ctx, cudaFuncSetAttribute(replay8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kReplaySmemEvents));
            ctx->replay_configured = true;
        }
    }
    EGPU_CUDA(ctx, cudaMemcpyAsync(d_kind, kind, sizeof(int32_t) * E, cudaMemcpyHostToDevice, s));
    EGPU_CUDA(ctx, cudaMemcpyAsync(d_a, a, sizeof(int32_t) * E, cudaMemcpyHostToDevice, s));
    EGPU_CUDA(ctx, cudaMemcpyAsync(d_b, b, sizeof(int32_t) * E, cudaMemcpyHostToDevice, s));
    ctx->prev_is_scan = false;
    ctx->lut_dirty = true;
    if (ctx->D <= 32 && E <= kReplaySmemEvents && ctx->replay_variant == 2) {
        // two warps: decode off the chain, lane = device on it (default wherever it applies); the release path
        // only for streams that hold a release event
        const size_t smem2 = static_cast<size_t>((E + 15) & ~15ll);
        if (!ctx->replay2_configured) {
            EGPU_CUDA(ctx, cudaFuncSetAttribute(replay2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kReplaySmemEvents));
            EGPU_CUDA(ctx, cudaFuncSetAttribute(replay2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kReplaySmemEvents));
            ctx->replay2_configured = true;
        }
        if (std::find(kind, kind + E, EGPU_EV_RELEASE) != kind + E)
            replay2_kernel<true><<<1, 64, smem2, s>>>(ctx->d_state, d_kind, d_a, d_b, E, d_out);
        else
            replay2_kernel<false><<<1, 64, smem2, s>>>(ctx->d_state, d_kind, d_a, d_b, E, d_out);
    } else if (ctx->D <= 8 && !ctx->replay_general)
        replay8_kernel<<<1, 32, smem, s>>>(ctx->d_state, d_kind, d_a, d_b, E, d_out, d_live);
    else
        replay_kernel<<<1, 32, smem, s>>>(ctx->d_state, d_kind, d_a, d_b, E, d_out, d_live);
    EGPU_CUDA(ctx, cudaGetLastError());
    ctx->launches += 1;
    EGPU_CUDA(ctx, cudaMemcpyAsync(out_idx, d_out, sizeof(int32_t) * E, cudaMemcpyDeviceToHost, s));
    EGPU_CUDA(ctx, cudaStreamSynchronize(s));
    return EGPU_OK;
}

}  // extern "C"
