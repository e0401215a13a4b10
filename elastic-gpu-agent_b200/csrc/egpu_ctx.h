// egpu_ctx.h — the context behind the opaque egpu_ctx* of include/egpu_alloc.h, shared by
// the translation units of the library (egpu_alloc.cu, egpu_devhash.cu).  Internal.
#pragma once
#include <cstdint>
#include <cstdio>
#include <mutex>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/egpu_alloc.h"
#include "egpu_kernels.cuh"

using namespace egpu;  // internal header: the context is made of the kernels' types

// The scan kernels the launchers of egpu_alloc.cu choose from, one per D bucket (D <= 8, 16, 32, 64) ...
enum ScanFamily {
    kScanSorted, kScanSortedContig, kScanGrid, kScanLut, kScanLutContig, kScanSortedMulti, kScanLutMulti, kScanPacked,
    kScanFamilies
};
// ... and the kernels of the other launches, numbered on from them.  A family has a table per row format
// (RowFormat), one kernel per D bucket, and every such kernel its own entry in egpu_ctx::ctas_per_sm.
enum LaunchFamily {
    kRoundsSorted = kScanFamilies, kRoundsLut,  // EGPU_F_DEVICE_ROUNDS, one batch
    kRoundsMultiSorted, kRoundsMultiLut,         // ... K batches (egpu_bestfit_batches_dev)
    kShardPrefixSorted, kShardPrefixLut,         // EGPU_F_PREFIX_COMMIT on egpu_bestfit_batches_shard_dev
    kShardRoundsSorted, kShardRoundsLut,         // EGPU_F_DEVICE_ROUNDS on egpu_bestfit_batch_shard_prefix_dev
    kRelease, kReleaseShard,                     // EGPU_F_RELEASE, one GPU and over row shards
    kKernelFamilies
};

struct egpu_ctx {
    std::mutex mu;
    int ctas_per_sm[kKernelFamilies * 2 * 4] = {};  // resident CTAs per SM of each kernel (Kernel::slot), 0 = not asked yet
    void* h_qtable = nullptr;        // pinned host image of that table (the part of DevState before `peer`)
    DevState* d_qstate = nullptr;     // scratch table of egpu_bestfit_query (the context's own table is not touched)
    unsigned long long* h_gate = nullptr;      // pinned: start gates the host has opened (egpu_peer_gate_open)
    unsigned long long* h_gate_dev = nullptr;  // its device-visible alias
    unsigned long long* d_tile_sums = nullptr;  // prefix-commit: per-tile per-device sums [tiles][2*64]
    size_t tile_bytes = 0;
    void* d_prefix_out = nullptr;     // PrefixOut
    void* d_rounds = nullptr;         // scratch of egpu_bestfit_batch_rounds (grow-only)
    size_t rounds_bytes = 0;
    size_t rounds_ctl_bytes = 0;      // rounds_bytes when the grid-barrier words in d_rounds were last zeroed
    unsigned long long rounds_timeouts_seen = 0;  // DevState::rounds_timeouts as the host form last read it
    DevLut* d_lut = nullptr;
    XchgBuf* d_xchg = nullptr;        // this rank's exchange buffer (exported to the peers over CUDA IPC)
    void* peer_open[kMaxRanks] = {};  // peers' buffers as opened here (nullptr for own rank)
    int world = 1, rank = 0;
    bool attached = false;
    bool lut_dirty = true;            // table changed since the lookup tables were built
    unsigned long long lut_capture = 0;  // the capture (capture_id) whose graph rebuilds them after its last table change
    int dev = -1;
    int sm_count = 132;  // H100 SXM; egpu_ctx_create reads the device's own count
    cudaStream_t stream = nullptr;
    DevState* d_state = nullptr;
    bool has_table = false;
    int D = 0;
    int variant = EGPU_VARIANT_AUTO;
    int64_t launches = 0;
    // staging for the host-buffer entry points
    int32_t* d_req_core = nullptr;
    int32_t* d_req_mem = nullptr;
    int32_t* d_idx = nullptr;
    size_t staging_bytes = 0;         // bytes of each of the three
    long long* d_delta = nullptr;     // int64[2*64]
    int32_t* d_table_out = nullptr;   // int32[3*64]
    long long* h_delta = nullptr;     // pinned
    long long* h_delta_dev = nullptr; // its device-visible alias
    bool no_zero_copy = false;        // EGPU_NO_ZERO_COPY=1: always stage through HBM
    int32_t* h_table = nullptr;       // pinned int32[3*64]
    bool replay_configured = false;   // shared-memory opt-in of the replay kernels done
    // bookkeeping for programmatic dependent launch (see order_scan in egpu_alloc.cu)
    bool prev_is_scan = false;        // the last kernel this context launched was a snapshot scan ...
    bool prev_changes_table = false;  // ... and it may rewrite the table (commit)
    cudaStream_t prev_stream = nullptr;
    unsigned long long prev_capture = 0;  // ... and the capture it was recorded in (capture_id), 0 = eager
    uint64_t seq = 0;                 // scans launched (epilogue slot = seq mod kEpiSlots)
    int group_len = 0;                // launches since (and including) the last fully ordered one
    int group_mbatches = 0;           // ... and the epi_multi slots (batches of multi-batch launches) they hold
    uint64_t mseq = 0;                // batches launched through multi-batch launches (slot = mseq mod kMultiSlots)
    struct Range { uintptr_t lo, hi; };
    std::vector<Range> inflight;      // output ranges of those launches, sorted by address, pairwise disjoint
    std::vector<Range> range_tmp;
    Range multi_ranges[3 * kMultiMax];  // scratch of launch_multi
    int multi_rpt = 8;                // multi-batch launches of batches < 512 Ki rows: the fewest rows per thread worth a CTA (EGPU_MULTI_RPT)
    int pipe_group = 24;              // launches per group (EGPU_PIPE_GROUP, <= kPipeGroupMax)
    int ctas_per_sm_cap = 0;          // 0 = occupancy limit (EGPU_CTAS_PER_SM overrides)
    int rows_per_thread = 0;          // grid sizing target (EGPU_ROWS_PER_THREAD), 0 = default
    int replay_variant = 2;           // 2 = two-warp kernel where it applies (EGPU_REPLAY_VARIANT=1: round 1's one-warp kernels)
    bool replay2_configured = false;
    bool sort_sets_configured = false;  // sort_sets_smem_kernel may use 128 KB of dynamic shared memory
    bool replay_general = false;      // EGPU_REPLAY_GENERAL=1: lane = device kernel even for D <= 8 (tests)
    // grow-only device arena for multi-kernel host-buffer pipelines (arena_carve)
    void* arena = nullptr;
    size_t arena_cap = 0;
    char last_err[256] = {0};
};

inline int cuda_fail(egpu_ctx* ctx, cudaError_t e, const char* what) {
    if (ctx) std::snprintf(ctx->last_err, sizeof ctx->last_err, "%s: %s", what, cudaGetErrorString(e));
    (void)cudaGetLastError();
    return e == cudaErrorMemoryAllocation ? EGPU_ERR_NOMEM : EGPU_ERR_CUDA;
}

// Grow-only device scratch: when `need` bytes do not fit in `cap`, frees every buffer in `bufs` and
// gives each `alloc` (>= need) fresh bytes; contents are not kept.  `cap` is 0 until all are allocated.
template <class... T>
cudaError_t grow(size_t& cap, size_t need, size_t alloc, T**... bufs) {
    if (need <= cap) return cudaSuccess;
    cap = 0;
    ((cudaFree(*bufs), *bufs = nullptr), ...);
    cudaError_t e = cudaSuccess;
    ((e = e == cudaSuccess ? cudaMalloc(bufs, alloc) : e), ...);
    if (e == cudaSuccess) cap = alloc;
    return e;
}

// Scratch of one call, carved from the context's arena in 256-byte aligned pieces (an empty want
// still gets one).  Every piece is sized before anything is enqueued, so a failed allocation leaves
// no work half done; the arena grows with 25 % slack and is only touched under ctx->mu.
struct ArenaWant {
    void** p;
    size_t bytes;
};
inline cudaError_t arena_carve(egpu_ctx* ctx, const ArenaWant* wants, int n) {
    auto piece = [](size_t bytes) { return ((bytes ? bytes : 16) + 255) & ~static_cast<size_t>(255); };
    size_t total = 0;
    for (int i = 0; i < n; ++i) total += piece(wants[i].bytes);
    const cudaError_t e = grow(ctx->arena_cap, total, total + total / 4, &ctx->arena);
    if (e != cudaSuccess) return e;
    size_t used = 0;
    for (int i = 0; i < n; ++i) {
        *wants[i].p = static_cast<char*>(ctx->arena) + used;
        used += piece(wants[i].bytes);
    }
    return cudaSuccess;
}

// egpu_alloc.cu: body of egpu_table_set for callers that already hold ctx->mu.  oversub[D] are the
// table's oversubscription flags (nullptr: none, as egpu_table_set installs it).
int egpu_table_set_locked(egpu_ctx* ctx, const int32_t* free_core, const int32_t* free_mem, const int32_t* oversub, int32_t D);

namespace egpu {
// egpu_devhash.cu: the identity pipeline's stable LSD radix sort and exclusive scan, for the other
// pipelines.  Both return the number of kernels they launched on s.
// words of the sort's histogram for n keys
size_t radix_hist_words(long long n);
// sorts (key, val) pairs of n < 2^31 elements by the low n_digits 4-bit digits of key, stably; the
// sorted pairs end in key / val (the pointers are swapped with the scratch pair after every pass)
int radix_sort_pairs(cudaStream_t s, unsigned long long*& key, uint32_t*& val, unsigned long long*& key_tmp,
                     uint32_t*& val_tmp, long long n, int n_digits, uint32_t* hist);
// out[0..n] = exclusive prefix sums of v[0..n); blk holds (n + 1023) / 1024 + 1 words
int exclusive_scan_u32(cudaStream_t s, const uint32_t* v, long long n, unsigned long long* blk, unsigned long long* out);
}  // namespace egpu

#define EGPU_CUDA(ctx, call)                                   \
    do {                                                       \
        cudaError_t e__ = (call);                              \
        if (e__ != cudaSuccess) return cuda_fail(ctx, e__, #call); \
    } while (0)
