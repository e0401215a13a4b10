/*
 * egpu_alloc.h — C ABI of the H100-native best-fit allocation path.
 *
 * This is the drop-in boundary: a Go DaemonSet (elastic-gpu-agent) binds these
 * symbols through cgo; nothing in the signatures is a CUDA, torch or C++ type.
 * All pointers are caller-owned and only read/written for the duration of the
 * call (cgo pointer rule) unless the name ends in `_dev`, in which case they are
 * CUDA device pointers and the call is asynchronous on the given stream.
 *
 * Reference interfaces each entry point stands behind (paths relative to the
 * reference repo elastic-ai/elastic-gpu-agent @ 2609107):
 *
 *   egpu_ctx_create / egpu_ctx_destroy
 *       constructed where the plugin is built, pkg/manager/manager.go:138
 *       (plugins.PluginFactory) and pkg/plugins/base.go:208-233.
 *   egpu_table_set
 *       the capacity table the reference derives at start-up from NVML:
 *       pkg/operator/base.go:19-75 (device count, memory bytes),
 *       pkg/plugins/gpushare.go:24-33 (100 core units per GPU),
 *       pkg/plugins/gpushare.go:159-168 (one memory unit per MiB).
 *   egpu_bestfit_batch / egpu_bestfit_batch_dev
 *       the slot of baseDevicePlugin.GetPreferredAllocation, a stub in the
 *       reference (pkg/plugins/base.go:94-96); request units follow
 *       pkg/common/const.go:4 (GPUPercentEachCard = 100) and the vendored
 *       resource names elasticgpu.io/gpu-core, elasticgpu.io/gpu-memory
 *       (vendor/elasticgpu.io/elastic-gpu/api/v1alpha1/types.go:105-112).
 *   egpu_bestfit_batches_dev / egpu_bestfit_query
 *       the same slot, for a caller with several requests' worth of batches in
 *       hand (one launch for up to 64 of them), and for the stateless what-if
 *       form GetPreferredAllocation needs (pkg/plugins/base.go:94-96: kubelet
 *       passes the available IDs of ONE admission; the node's committed table
 *       must not be touched by it).
 *   egpu_replay
 *       commits serialised under baseDevicePlugin.lock in PreStartContainer
 *       (pkg/plugins/gpushare.go:114,239) and frees issued by
 *       GPUSharePlugin.GC (pkg/plugins/base.go:241-306).
 *   egpu_preferred_allocation
 *       pluginapi.PreferredAllocationRequest/Response
 *       (vendor/k8s.io/kubelet/pkg/apis/deviceplugin/v1beta1/api.pb.go:564-571,
 *       675-677) with the device-ID format "%d-%02d" of
 *       pkg/plugins/gpushare.go:28,163.
 *   egpu_device_hash / egpu_device_hash_batch
 *       types.NewDevice + hash, pkg/types/device.go:17-25,49-54
 *       (sort.Strings, join ":", SHA-256, first 8 hex digits), used by
 *       Allocate (pkg/plugins/gpushare.go:44,179) and by
 *       KubeletDeviceLocator.Locate (pkg/kube/locator.go:62-90).
 *
 * IMPORTANT: the reference contains NO best-fit scoring loop (SURVEY.md §0);
 * the decision rule implemented here is the builder-defined specification in
 * DESIGN.md §2 ("the spec"), restated on the CPU in oracle/.
 *
 * The spec in one paragraph. D devices (1..64), free_core[d] in [0,100]
 * (percent), free_mem[d] in [0, 2^18-1] (MiB).  Request (core, mem) is feasible
 * on d iff 0 <= core <= free_core[d] and 0 <= mem <= free_mem[d].  Best fit =
 * the feasible device with the lexicographically smallest
 * (free_core[d]-core, free_mem[d]-mem, d); idx = -1 when no device is feasible.
 * Snapshot mode scores every request of a batch against the same table and
 * reports per-device demand sums (int64) and table' = table - demand
 * (saturated to int32, oversub flag when negative).  Sequential mode applies
 * each event to the table before the next one is scored.
 */
#ifndef EGPU_ALLOC_H
#define EGPU_ALLOC_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EGPU_MAX_DEVICES   64
#define EGPU_CORE_MAX      100              /* pkg/common/const.go:4 */
#define EGPU_MEM_MAX       ((1 << 18) - 1)  /* MiB; an H100 80GB reports 81559 */
#define EGPU_MAX_ROWS      2147483647       /* requests per batch (R): the scans index with 32 bits */
#define EGPU_IDX_INFEASIBLE (-1)
#define EGPU_IDX_DEFERRED   (-2)            /* prefix-commit mode only */

/* return codes: 0 = OK, negative = error, never aborts the process */
#define EGPU_OK               0
#define EGPU_ERR_INVALID     (-1)   /* bad argument (NULL, range, D, sizes) */
#define EGPU_ERR_NO_DEVICE   (-2)   /* no usable CUDA device / driver */
#define EGPU_ERR_CUDA        (-3)   /* CUDA runtime error (see egpu_last_error) */
#define EGPU_ERR_NOMEM       (-4)   /* host or device allocation failed */
#define EGPU_ERR_NO_TABLE    (-5)   /* egpu_table_set has not been called */
#define EGPU_ERR_STATE       (-6)   /* call not valid in the current state */
#define EGPU_ERR_PARSE       (-7)   /* malformed device-ID string or stored record */
#define EGPU_ERR_UNSAT       (-8)   /* preferred allocation cannot be satisfied */

/* event kinds for egpu_replay */
#define EGPU_EV_ALLOC   0
#define EGPU_EV_FREE    1
#define EGPU_EV_RELEASE 3   /* gives back a placement made before the call; 2 stays a no-op */

/* flags of egpu_bestfit_batch_dev */
#define EGPU_F_COMMIT        1   /* table' replaces the current table */
#define EGPU_F_INPUTS_READY  2   /* the request arrays were complete before the previous
                                    launch on this stream: consecutive scans may overlap
                                    (programmatic dependent launch); anything else
                                    enqueued later on the stream still sees them
                                    complete. */

#define EGPU_F_PREFIX_COMMIT 4   /* spec 2.5: a request commits only while the running demand of
                                    its device (all earlier requests that chose it) still fits;
                                    the others get EGPU_IDX_DEFERRED, the demand sums and table'
                                    count committed requests only, so table' never goes negative.
                                    Single GPU; not with EGPU_VARIANT_GRID.  In egpu_bestfit_batch
                                    pass it in `commit` (EGPU_F_COMMIT | EGPU_F_PREFIX_COMMIT). */

#define EGPU_F_APPLY         8   /* egpu_bestfit_batches_shard_dev only: the CTAs that complete a batch's sums, having pushed the
                                    batch's demand vector, also wait for the peers' vectors of that exchange step and
                                    write table' (= table - sum over ranks) to the batch's d_table_out: no apply call,
                                    no second stream.  Never commits.  Every rank must issue the same launch; start the
                                    ranks together (egpu_peer_gate_dev) or the wait is as long as their skew. */

#define EGPU_F_PACKED       16   /* the packed format of egpu_bestfit_batch_packed (5 bytes per decision
                                    instead of 12) on egpu_bestfit_batches_dev (see there) and, together with
                                    EGPU_F_PREFIX_COMMIT only, on egpu_bestfit_batch / egpu_bestfit_batch_dev:
                                    see egpu_bestfit_batch_dev; and on the sharded single-batch calls
                                    egpu_bestfit_batch_shard_dev, egpu_bestfit_batch_shard_lag_dev and
                                    egpu_bestfit_batch_shard_prefix_dev (see there).
                                    egpu_bestfit_batches_shard_dev refuses it. */

#define EGPU_F_ROUNDS       32   /* egpu_bestfit_batch / egpu_bestfit_batch_dev only, and only as
                                    EGPU_F_PACKED | EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT | EGPU_F_ROUNDS
                                    [| EGPU_F_INPUTS_READY]: packed prefix-commit rounds to the fixed point
                                    (egpu_bestfit_batch_rounds on packed words, no round limit); see
                                    egpu_bestfit_batch_dev.  egpu_bestfit_batches_dev and
                                    egpu_bestfit_batch_shard_prefix_dev refuse it except in the flag set of
                                    EGPU_F_DEVICE_ROUNDS. */

#define EGPU_F_DEVICE_ROUNDS 128 /* egpu_bestfit_batch / egpu_bestfit_batch_dev / egpu_bestfit_batches_dev and
                                    egpu_bestfit_batch_shard_prefix_dev only, and only as
                                    EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT | EGPU_F_ROUNDS | EGPU_F_DEVICE_ROUNDS
                                    [| EGPU_F_PACKED] [| EGPU_F_INPUTS_READY]: rounds to the fixed point, int32 or
                                    packed, in ONE launch with no host round trip per round; the _dev forms do
                                    not synchronise their stream.  See egpu_bestfit_batch_dev (one batch) and
                                    egpu_bestfit_batches_dev (batches placed in order).  Also accepted by
                                    egpu_bestfit_batch_shard_prefix_dev, as that flag set without
                                    EGPU_F_INPUTS_READY: rounds over row shards (see there).  The value is 128,
                                    not 64: callers were told that EGPU_F_ROUNDS with bit 64 is refused, and it
                                    still is.  Bit 64 is unassigned. */

#define EGPU_F_RELEASE      256  /* egpu_bestfit_batch / egpu_bestfit_batch_dev and
                                    egpu_bestfit_batch_shard_prefix_dev only, and only as
                                    EGPU_F_RELEASE [| EGPU_F_COMMIT] [| EGPU_F_PACKED]: the rows give back the
                                    capacity they hold on the devices in the index array, which is an INPUT, all
                                    or nothing, in one launch; see egpu_bestfit_batch_dev, and
                                    egpu_bestfit_batch_shard_prefix_dev for the release over row shards.  Any other
                                    bit with it is EGPU_ERR_INVALID.  egpu_bestfit_batches_dev,
                                    egpu_bestfit_batches_shard_dev and egpu_bestfit_batch_shard_dev refuse it;
                                    egpu_bestfit_batch_packed_dev and egpu_bestfit_batch_shard_lag_dev ignore it, as
                                    they ignore every bit they never checked.  Until this flag was defined the two
                                    calls that take it ignored bit 256 when no rounds bit came with it; it is now
                                    defined, and with it set only EGPU_F_COMMIT commits.  Bit 64 stays unassigned. */

/* per-device reason words of a refused release: the third block of d_table_out */
#define EGPU_REL_FLAGGED     1   /* rows are held on a device whose oversubscription flag is set */
#define EGPU_REL_EXCEEDS     2   /* free + released would exceed EGPU_CORE_MAX or EGPU_MEM_MAX on the device */

/* kernel variants for the snapshot scan (egpu_set_variant) */
#define EGPU_VARIANT_AUTO    0   /* SORTED for D <= 16, LUT above */
#define EGPU_VARIANT_GRID    1   /* direct (device x request) score grid, min over packed keys */
#define EGPU_VARIANT_SORTED  2   /* first feasible device in (core, mem, d)-sorted order, table in registers */
#define EGPU_VARIANT_LUT     3   /* same order, answered by shared-memory lookup tables (large D) */

typedef struct egpu_ctx egpu_ctx;

/* ---- lifetime --------------------------------------------------------- */

/* One context per CUDA device (one process per GPU).  Thread-safe: every entry
 * point takes the context mutex (mirrors baseDevicePlugin.lock) and binds the
 * CUDA device explicitly, so it may be called from any OS thread (goroutines
 * migrate).  Fails with EGPU_ERR_NO_DEVICE when there is no GPU: there is NO
 * CPU fallback in this library. */
int  egpu_ctx_create(int cuda_device, egpu_ctx** out);
void egpu_ctx_destroy(egpu_ctx* ctx);
const char* egpu_strerror(int code);
/* last error detail recorded by this context ("" if none): the failing CUDA call, or the
 * record a parse error was found in.  The pointer stays valid for the life of the context;
 * the text is overwritten by the next failing call. */
const char* egpu_last_error(egpu_ctx* ctx);
/* 1 = CUDA sm_90a path.  (0 is reserved; this library never returns it.) */
int  egpu_backend(egpu_ctx* ctx);
/* number of kernels this context has launched since creation */
int64_t egpu_launch_count(egpu_ctx* ctx);
int  egpu_set_variant(egpu_ctx* ctx, int variant);
/* ABI version: major*1000 + minor.  Minor revisions only add entry points (1.1 placement
 * restore, 1.2 prefix-commit over row shards, 1.3 rounds, 1.4 multi-batch launches, stateless query,
 * start gate, host registration, 1.5 preferred allocation for many container requests from flat ID
 * buffers, 1.6 EGPU_F_PACKED multi-batch launches, 1.7 EGPU_F_PACKED prefix-commit on egpu_bestfit_batch and
 * egpu_bestfit_batch_dev, 1.8 EGPU_F_ROUNDS packed rounds on the same two, 1.9 EGPU_F_PACKED on
 * egpu_bestfit_batch_shard_dev, egpu_bestfit_batch_shard_lag_dev and egpu_bestfit_batch_shard_prefix_dev,
 * 1.10 EGPU_F_DEVICE_ROUNDS rounds in one launch on egpu_bestfit_batch and egpu_bestfit_batch_dev,
 * 1.11 EGPU_F_DEVICE_ROUNDS on egpu_bestfit_batches_dev: K batches placed in order in one launch); a
 * caller built against 1.0 keeps working. */
int  egpu_abi_version(void);

/* ---- capacity table --------------------------------------------------- */

int egpu_table_set(egpu_ctx* ctx, const int32_t* free_core,
                   const int32_t* free_mem, int32_t D);
/* oversub may be NULL.  Synchronises the context's stream. */
int egpu_table_get(egpu_ctx* ctx, int32_t* free_core, int32_t* free_mem,
                   int32_t* oversub);
int egpu_table_size(egpu_ctx* ctx);

/* ---- snapshot mode, host buffers (what a cgo caller uses) -------------- */

/* Scores R requests against the current table.  Copies inputs H2D from the
 * caller's arrays (pinned or pageable), runs the scan, copies idx and deltas
 * back; returns when the outputs are valid.  out_delta_* have D entries and
 * may be NULL.  commit != 0 installs table' as the current table.  `commit` also takes
 * EGPU_F_PREFIX_COMMIT, and with it EGPU_F_PACKED (packed prefix-commit: see egpu_bestfit_batch_dev;
 * the words are staged through HBM, 4 bytes per row in and 1 out), and with those and EGPU_F_COMMIT,
 * EGPU_F_ROUNDS (packed rounds to the fixed point, staged the same way; out_delta_* receive the demand
 * committed over all rounds), and with EGPU_F_ROUNDS, EGPU_F_DEVICE_ROUNDS (rounds in one launch, int32
 * or packed: staged through HBM, int32 8 bytes per row in and 4 out, packed 4 in and 1 out; one launch
 * and one synchronisation; returns EGPU_ERR_CUDA, with egpu_last_error saying so, when a device-rounds
 * launch on this context gave up at a grid barrier since the previous host-form call).  `commit` also takes
 * EGPU_F_RELEASE [| EGPU_F_COMMIT] [| EGPU_F_PACKED] (release: see egpu_bestfit_batch_dev): out_idx is then an
 * input, and the call returns EGPU_ERR_STATE when the release was refused. */
int egpu_bestfit_batch(egpu_ctx* ctx, const int32_t* req_core,
                       const int32_t* req_mem, int64_t R, int32_t* out_idx,
                       int64_t* out_delta_core, int64_t* out_delta_mem,
                       int commit);

/* Batch allocation to a fixed point (SURVEY.md §8(f) n4: "multi-round deferred retry").
 * Round 1 is egpu_bestfit_batch(..., EGPU_F_COMMIT | EGPU_F_PREFIX_COMMIT); every later round
 * re-submits the rows the previous one deferred, in their original order, against the table
 * that round committed.  It stops when a round defers nothing or after max_rounds (>= 1).
 * Every round places at least one row per device that still has takers, so it terminates; the
 * table is always committed and never oversubscribed.
 *   out_idx[r]      device index, EGPU_IDX_INFEASIBLE (in the round the row was last scored),
 *                   or EGPU_IDX_DEFERRED when max_rounds ran out first
 *   out_delta_*[D]  demand committed over all rounds (may be NULL)
 *   *out_rounds     rounds run; *out_deferred = rows still deferred (both may be NULL)
 * Scratch (32 bytes per request, kept by the context) is allocated before round 1: an
 * allocation failure returns EGPU_ERR_NOMEM with nothing committed.
 * R < 2^31.  The _dev form takes device request/index arrays (16-byte aligned) and host
 * out_delta[2*D]; it synchronises `stream` (each round needs its deferred count on the host). */
int egpu_bestfit_batch_rounds(egpu_ctx* ctx, const int32_t* req_core, const int32_t* req_mem,
                              int64_t R, int32_t* out_idx, int64_t* out_delta_core,
                              int64_t* out_delta_mem, int32_t max_rounds, int32_t* out_rounds,
                              int64_t* out_deferred);
int egpu_bestfit_batch_rounds_dev(egpu_ctx* ctx, const int32_t* d_req_core,
                                  const int32_t* d_req_mem, int64_t R, int32_t* d_out_idx,
                                  int64_t* out_delta, int32_t max_rounds, int32_t* out_rounds,
                                  int64_t* out_deferred, void* stream);

/* Packed wire format, for callers bound by PCIe rather than by the scan: 5 bytes per decision
 * instead of 12.  req_packed[r] = EGPU_PACK_REQUEST(core, mem) (core in 0..127, mem in
 * 0..2^18-1; any word >= 2^25, e.g. EGPU_PACKED_INVALID, is an infeasible request);
 * out_idx8[r] = device index 0..63 or -1.  Everything else as egpu_bestfit_batch.  Snapshot mode only:
 * EGPU_F_PREFIX_COMMIT is not implemented here (packed prefix-commit is egpu_bestfit_batch[_dev] with
 * EGPU_F_PACKED | EGPU_F_PREFIX_COMMIT). */
#define EGPU_PACK_REQUEST(core, mem) (((uint32_t)(core) << 18) | (uint32_t)(mem))
#define EGPU_PACKED_INVALID 0xFFFFFFFFu
int egpu_bestfit_batch_packed(egpu_ctx* ctx, const uint32_t* req_packed, int64_t R, int8_t* out_idx8,
                              int64_t* out_delta_core, int64_t* out_delta_mem, int commit);
/* The same snapshot on device buffers, asynchronous on `stream` as egpu_bestfit_batch_dev: d_req_packed R
 * words, d_out_idx8 R int8 indices (both 16-byte aligned when R > 0), d_delta int64[2*D] and d_table_out
 * int32[3*D] (either may be NULL).  flags: EGPU_F_COMMIT (table' replaces the current table) and
 * EGPU_F_INPUTS_READY (as in egpu_bestfit_batch_dev: consecutive non-committing scans of this context on one
 * stream - packed, int32, multi-batch or sharded - may overlap); every other bit is ignored, so
 * EGPU_F_PREFIX_COMMIT does not select prefix-commit here.  The scan follows egpu_set_variant as the int32
 * scan does: the register scan for D <= 16 and the lookup scan above under EGPU_VARIANT_AUTO.  Under
 * EGPU_VARIANT_GRID, and for R > EGPU_MAX_ROWS, the call runs the fully ordered scan of
 * egpu_bestfit_batch_packed instead; the outputs are the same either way.  EGPU_ERR_INVALID: NULL or
 * misaligned words or indices with R > 0, R < 0, and (as in egpu_bestfit_batch_dev) indices, sums and
 * table' that overlap each other. */
int egpu_bestfit_batch_packed_dev(egpu_ctx* ctx, const uint32_t* d_req_packed, int64_t R,
                                  int8_t* d_out_idx8, int64_t* d_delta, int32_t* d_table_out,
                                  int flags, void* stream);

/* Pinned host memory for callers that want zero staging copies. */
int  egpu_host_alloc(egpu_ctx* ctx, void** out, int64_t bytes);
void egpu_host_free(egpu_ctx* ctx, void* p);

/* Pins caller-owned memory in place (cudaHostRegister, mapped) so that buffers the caller already
 * has - a Go slice it keeps for the life of the plugin, say - take the zero-staging path of
 * egpu_bestfit_batch / _packed instead of being copied through HBM.  Registration is slow next to
 * one call, so it pays only for buffers that are reused.  The range must stay allocated until
 * egpu_host_unregister (a cgo caller must not hand over memory the Go runtime may release:
 * allocate it with C.malloc or keep it pinned with runtime.Pinner).  The context does not track
 * registrations. */
int  egpu_host_register(egpu_ctx* ctx, void* p, int64_t bytes);
int  egpu_host_unregister(egpu_ctx* ctx, void* p);

/* ---- snapshot mode, device buffers (bench / multi-GPU plumbing) -------- */

/* CUDA graphs (DESIGN.md 2.9): a _dev call captured into a graph changes nothing at capture time; it runs at
 * every replay against the table the context holds then.  A captured call that may rewrite the table is followed
 * inside the graph by a rebuild of the lookup tables (one more node than the eager call's launches), so eager calls
 * after a replay read the table it left.  A captured lookup scan rebuilds them inside the graph only when they were
 * stale at capture: after changing the table outside the graph (egpu_table_set, an eager commit), run one eager
 * lookup scan before the next replay of such a graph.  EGPU_F_INPUTS_READY pipelines captured scans behind scans of
 * the same capture only: never behind an eager launch, nor an eager one behind them.
 * Calls that synchronise a stream (the host forms, the rounds with EGPU_F_ROUNDS alone) cannot be captured.
 *
 * Asynchronous on `stream` (a cudaStream_t passed as void*; NULL = the
 * context's own non-blocking stream — to name the legacy default stream pass
 * cudaStreamLegacy, not 0).  d_delta is int64[2*D]: core sums then mem sums; it
 * is overwritten, not accumulated.  d_table_out (may be NULL) receives
 * int32[3*D]: free_core', free_mem', oversub.  flags: EGPU_F_*.  The three
 * request/index arrays must be 16-byte aligned (128-bit accesses).
 *
 * Packed prefix-commit (flags EGPU_F_PACKED | EGPU_F_PREFIX_COMMIT [| EGPU_F_COMMIT]
 * [| EGPU_F_INPUTS_READY]):
 *   d_req_core   R packed words (EGPU_PACK_REQUEST; const uint32_t* cast to the argument's type);
 *   d_req_mem    must be NULL;
 *   d_out_idx    R int8 indices (int8_t* cast to the argument's type): device, -1 or EGPU_IDX_DEFERRED.
 * Semantics are the int32 prefix-commit's on the requests the words stand for; words >= 2^25 and
 * core 101..127 are infeasible.  EGPU_ERR_STATE under EGPU_VARIANT_GRID.  EGPU_ERR_INVALID, before
 * anything is launched or written: EGPU_F_PACKED without EGPU_F_PREFIX_COMMIT (packed snapshots are
 * egpu_bestfit_batch_packed[_dev]), a non-NULL d_req_mem, NULL or (_dev) misaligned words or indices
 * with R > 0.  Without EGPU_F_PACKED a NULL d_req_mem with R > 0 is refused, so packed words are never
 * read as int32 arrays.
 *
 * Packed rounds (flags EGPU_F_PACKED | EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT | EGPU_F_ROUNDS
 * [| EGPU_F_INPUTS_READY]): the arguments of packed prefix-commit, and the semantics of
 * egpu_bestfit_batch_rounds with no round limit: committing rounds run until one defers nothing, so
 * every index ends as a device or -1, never EGPU_IDX_DEFERRED, and the table is never oversubscribed
 * (sticky oversubscription flags are kept, as there).  d_delta (may be NULL) receives the demand
 * committed over all rounds, int64[2*D]; d_table_out (may be NULL) the last round's table', oversub
 * words 0.  THIS CALL SYNCHRONISES `stream` before it returns: every round needs its deferred count on
 * the host.  Scratch (18 bytes per request, kept by the context) is allocated before round 1: an
 * allocation failure returns EGPU_ERR_NOMEM with nothing committed.  R = 0 is the packed prefix-commit
 * with R = 0.  EGPU_ERR_STATE under EGPU_VARIANT_GRID.  EGPU_ERR_INVALID, before anything is launched
 * or written: EGPU_F_ROUNDS with any other combination of flags, R >= 2^31, and everything packed
 * prefix-commit refuses.
 *
 * Rounds in one launch (flags EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT | EGPU_F_ROUNDS | EGPU_F_DEVICE_ROUNDS
 * [| EGPU_F_PACKED] [| EGPU_F_INPUTS_READY], the last accepted and without effect): the semantics of
 * egpu_bestfit_batch_rounds_dev with no round limit - every index ends as a device or -1, never
 * EGPU_IDX_DEFERRED, sticky oversubscription flags are kept - on int32 arrays (d_req_core, d_req_mem,
 * int32 d_out_idx) or, with EGPU_F_PACKED, on the arguments of packed prefix-commit (words, NULL
 * d_req_mem, int8 indices).  ASYNCHRONOUS on `stream`, with no synchronisation: every round runs in one
 * persistent launch, so the call can sit in a pipelined stream.  d_delta (may be NULL) receives the
 * demand committed over all rounds, int64[2*D]; d_table_out (may be NULL) the last round's table',
 * oversub words 0; the committed table is installed in stream order.  R = 0 writes zero sums and
 * table' = the current table.  Scratch is that of the rounds (32 bytes per request int32, 18 packed),
 * kept by the context and allocated before the launch: an allocation failure returns EGPU_ERR_NOMEM
 * with nothing committed.  Calls that share a context's scratch (all prefix-commit and rounds calls)
 * must be ordered on one stream, or by the caller.  The launch is cooperative: the runtime refuses a
 * grid it cannot keep resident rather than letting it wait.  Every wait inside the launch gives up
 * after about 2 s; a launch that gave up leaves the rows it did not finish at EGPU_IDX_DEFERRED and is
 * reported by the next host-form call with EGPU_F_DEVICE_ROUNDS (EGPU_ERR_CUDA).  EGPU_ERR_STATE under
 * EGPU_VARIANT_GRID.  EGPU_ERR_INVALID, before anything is launched or written: EGPU_F_DEVICE_ROUNDS
 * with any other combination of flags, R >= 2^31, NULL or misaligned arrays with R > 0, a non-NULL
 * d_req_mem with EGPU_F_PACKED and a NULL one without it.
 *
 * Release (flags EGPU_F_RELEASE [| EGPU_F_COMMIT] [| EGPU_F_PACKED]; DESIGN.md 2.8): the R rows give back what
 * they hold, by index, in ONE launch (egpu_launch_count + 1).  d_out_idx is READ, never written: it is the index
 * array a committing call produced for these rows, or any subset or concatenation of such rows.  Row r holds
 * (core, mem) on device d_out_idx[r] iff 0 <= d_out_idx[r] < D, 0 <= core <= EGPU_CORE_MAX and 0 <= mem <=
 * EGPU_MEM_MAX; every other row (-1, EGPU_IDX_DEFERRED, any other index, an out-of-domain request) holds nothing
 * and is skipped, so the output of a rounds or prefix-commit call can be handed back unfiltered.  U[d] = the int64
 * sums over the rows held on d; a device is touched iff U_core[d] > 0 or U_mem[d] > 0.  The call is REFUSED, as a
 * whole, iff some touched device has its oversubscription flag set (EGPU_REL_FLAGGED: saturation at 0 lost its
 * true deficit) or free + U would exceed EGPU_CORE_MAX or EGPU_MEM_MAX there (EGPU_REL_EXCEEDS).  The context does
 * not know a device's memory capacity: the memory bound is the domain bound only, and a caller who wants a
 * capacity check runs the call without EGPU_F_COMMIT and compares d_table_out with its capacities.  Rows that are
 * truly held on unflagged devices are never refused; a refusal means a double release, foreign rows or an
 * oversubscribed device.  Written whether accepted or refused: d_delta (may be NULL) = U, int64[2*D]; d_table_out
 * (may be NULL) = free + U when accepted and the current table when refused, int32[2*D], followed by D reason
 * words: 0, EGPU_REL_FLAGGED or EGPU_REL_EXCEEDS (any non-zero word: refused).  With EGPU_F_COMMIT an accepted
 * free + U becomes the table, in stream order; the sticky oversubscription flags stay as they are.  Without it
 * nothing is installed (dry run).  A refused launch changes nothing but d_delta, d_table_out and
 * egpu_release_refusals.  With EGPU_F_PACKED the rows are the arguments of packed prefix-commit (words, NULL
 * d_req_mem, int8 indices); a word >= 2^25 or with core 101..127 holds nothing.  R = 0 is accepted: zero sums and
 * d_table_out = the current table.  ASYNCHRONOUS on `stream`, fully ordered behind what the stream holds, and it
 * replays from a CUDA graph.  It does not depend on the scan variant: it works under EGPU_VARIANT_GRID too.
 * EGPU_ERR_NO_TABLE without a table.  EGPU_ERR_INVALID, before anything is launched or written: any other bit
 * with EGPU_F_RELEASE (EGPU_F_INPUTS_READY, EGPU_F_PREFIX_COMMIT, EGPU_F_ROUNDS, EGPU_F_DEVICE_ROUNDS and
 * EGPU_F_APPLY among them), R >= 2^31, NULL or misaligned arrays with R > 0, a non-NULL d_req_mem with
 * EGPU_F_PACKED and a NULL one without it, d_delta and d_table_out that overlap.  The host form
 * egpu_bestfit_batch takes the same flags in `commit`, reads out_idx, stages rows and indices through HBM (12
 * bytes per row in, packed 5, none out), and returns EGPU_ERR_STATE when the release was refused, with
 * egpu_last_error naming the first offending device and the reason; out_delta_* are written either way.  This is
 * a newly accepted flag set on existing entry points: egpu_abi_version() stays 1011. */
int egpu_bestfit_batch_dev(egpu_ctx* ctx, const int32_t* d_req_core,
                           const int32_t* d_req_mem, int64_t R,
                           int32_t* d_out_idx, int64_t* d_delta,
                           int32_t* d_table_out, int flags, void* stream);

/* Several batches in ONE launch.  Every batch is what egpu_bestfit_batch_dev takes - its own
 * request arrays, index array, d_delta (may be NULL) and d_table_out (may be NULL) - and all K
 * (1..EGPU_MAX_BATCHES) are scored against the current table, so the result of each batch is
 * exactly what K separate non-committing calls would produce; only the launch latency, ramp and
 * tail are paid once instead of K times (at R = 1 M that fixed cost is about a third of a lone
 * launch; at R <= 100 k it is nearly all of it).  Asynchronous on `stream`.  flags:
 * EGPU_F_INPUTS_READY only for a snapshot launch, which never commits; the one committing form is
 * the flag set of the rounds in one launch (below).  Outputs of different batches must not
 * overlap (EGPU_ERR_INVALID).  Batches may have different R (R = 0 allowed).
 *
 * Packed batches (flags EGPU_F_PACKED, alone or with EGPU_F_INPUTS_READY): every batch of the call
 * is in the wire format of egpu_bestfit_batch_packed, and the fields are read as
 *   d_req_core   R packed words (const uint32_t* cast to the field's type), 16-byte aligned;
 *   d_req_mem    must be NULL (EGPU_ERR_INVALID otherwise);
 *   d_out_idx    R int8 indices (int8_t* cast to the field's type), 16-byte aligned;
 *   d_delta, d_table_out  as above.
 * Words >= 2^25 and core 101..127 are infeasible requests (-1).  Everything else is as for int32
 * batches - K <= 64, ragged and empty batches, never commits, EGPU_F_INPUTS_READY pipelining (packed
 * and int32 launches may follow each other in one pipelined stream), EGPU_ERR_STATE under
 * EGPU_VARIANT_GRID - and outputs of different batches must not overlap: an index array covers R
 * bytes.  Without the flag a batch with R > 0 and a NULL d_req_mem is refused, so packed batches
 * handed over without it are never read as int32 arrays.  egpu_bestfit_batches_shard_dev refuses
 * the flag on its snapshot steps; it takes it only with EGPU_F_PREFIX_COMMIT (below).
 *
 * Batches placed in order, each to the fixed point, in one launch (flags EGPU_F_PREFIX_COMMIT |
 * EGPU_F_COMMIT | EGPU_F_ROUNDS | EGPU_F_DEVICE_ROUNDS [| EGPU_F_PACKED] [| EGPU_F_INPUTS_READY], the
 * last accepted and without effect): batch k runs the rounds in one launch of egpu_bestfit_batch_dev
 * against the table batches 0..k-1 committed, so the result is, bit for bit, what K consecutive
 * egpu_bestfit_batch_dev calls with the same flags give when issued on one stream in batch order (an
 * ordered admission queue: FIFO, or priority tiers placed one after the other).  This is not one rounds
 * call on the concatenated batches, whose round 1 would let a later batch take the device an earlier
 * batch's deferred row gets in its round 2.  Every index ends as a device or -1; sticky
 * oversubscription flags are kept.  Per batch, d_delta (may be NULL) receives the demand that batch
 * committed over its rounds, int64[2*D], and d_table_out (may be NULL) the table' of its last round,
 * oversub words 0; an empty batch (R = 0) writes zero sums and table' = the table its predecessors left.
 * The rows are int32 arrays, or with EGPU_F_PACKED the packed batch layout above (words, NULL
 * d_req_mem, int8 indices).  ONE launch (egpu_launch_count + 1), ASYNCHRONOUS on `stream` with no
 * synchronisation; the committed table is installed in stream order, and the call replays from a
 * CUDA graph (a replay after egpu_table_set starts from the new table).  Scratch is the rounds scratch
 * of egpu_bestfit_batch_dev, sized by the largest batch before the launch: an allocation failure
 * returns EGPU_ERR_NOMEM with nothing committed.  Every wait inside the launch gives up after about
 * 2 s, counted as for egpu_bestfit_batch_dev and reported by the next host-form call with
 * EGPU_F_DEVICE_ROUNDS (EGPU_ERR_CUDA); then the batch in progress keeps its unfinished rows at
 * EGPU_IDX_DEFERRED, and the batches after it are not reached: their indices, d_delta and d_table_out
 * are left unwritten.  EGPU_ERR_STATE under EGPU_VARIANT_GRID, EGPU_ERR_NO_TABLE without a table.
 * EGPU_ERR_INVALID, before anything is launched or written: EGPU_F_DEVICE_ROUNDS with any other
 * combination of flags, K outside 1..64, a batch with R >= 2^31, NULL or misaligned arrays with R > 0,
 * a non-NULL d_req_mem with EGPU_F_PACKED and a NULL one without it, outputs of two batches that
 * overlap.  egpu_bestfit_batches_shard_dev refuses these flags. */
#define EGPU_MAX_BATCHES 64
typedef struct egpu_batch {
    const int32_t* d_req_core;   /* EGPU_F_PACKED: the packed words */
    const int32_t* d_req_mem;    /* EGPU_F_PACKED: NULL */
    int64_t        R;
    int32_t*       d_out_idx;    /* EGPU_F_PACKED: int8 indices */
    int64_t*       d_delta;      /* int64[2*D] or NULL */
    int32_t*       d_table_out;  /* int32[3*D] or NULL */
} egpu_batch;
int egpu_bestfit_batches_dev(egpu_ctx* ctx, const egpu_batch* batches, int32_t K, int flags,
                             void* stream);

/* Stateless query: scores R requests against the table GIVEN HERE (free_core/free_mem[D], host
 * arrays, same domain as egpu_table_set) and returns the indices.  The context's own table,
 * its oversubscription flags and lookup tables are not read or written, so a context that
 * tracks the node's committed placement can also answer GetPreferredAllocation-style
 * what-if questions (egpu_preferred_allocation uses this).  Host buffers; returns when out_idx
 * is valid. */
int egpu_bestfit_query(egpu_ctx* ctx, const int32_t* free_core, const int32_t* free_mem, int32_t D,
                       const int32_t* req_core, const int32_t* req_mem, int64_t R,
                       int32_t* out_idx);

/* Multi-GPU step 2: after the G per-rank delta vectors (int64[G][2*D], rank
 * major) have been all-gathered, subtract their sum from the current table on
 * this rank: d_table_out (may be NULL) receives int32[3*D] as above, and with
 * commit != 0 the result becomes the current table.  Every rank ends with an
 * identical table'. */
int egpu_table_apply_deltas_dev(egpu_ctx* ctx, const int64_t* d_deltas, int G,
                                int32_t* d_table_out, int commit, void* stream);

/* ---- multi-GPU without a collective library on the data path --------------- */

/* One process per GPU.  Each rank exports a CUDA-IPC handle of its exchange buffer
 * (EGPU_IPC_HANDLE_BYTES bytes), the ranks swap handles by any means (the bench uses
 * torch.distributed.all_gather_object) and attach: handles = world * 64 bytes, rank
 * major.  After that a sharded step is two asynchronous calls:
 *   egpu_bestfit_batch_shard_dev  scans this rank's rows; its last CTA stores the
 *       rank's demand vector into EVERY rank's exchange buffer over NVLink and raises
 *       a release flag - the exchange is fused into the scan kernel;
 *   egpu_table_apply_peers_dev    waits (acquire) until all `world` vectors of `step`
 *       have landed locally, applies their sum: table' (and commit) as in snapshot mode.
 * `step` must increase by one per sharded step on every rank; a rank's scans may run at
 * most 128 steps ahead of its own applies (256 exchange slots: then no peer can be more than
 * 255 steps ahead of what this rank has consumed).  The scan itself never commits.
 *
 * Packed sharded scans (egpu_bestfit_batch_shard_dev flags EGPU_F_PACKED [| EGPU_F_INPUTS_READY]):
 * the arguments of the packed prefix-commit of egpu_bestfit_batch_dev -
 *   d_req_core   R packed words (EGPU_PACK_REQUEST; const uint32_t* cast to the argument's type), 16-byte aligned;
 *   d_req_mem    must be NULL;
 *   d_out_idx    R int8 indices (int8_t* cast to the argument's type), 16-byte aligned: device or -1.
 * Words >= 2^25 and core 101..127 are infeasible.  The demand vector pushed for `step` is the one the
 * int32 call pushes for the requests the words stand for, so the apply calls are the same and ranks
 * may mix formats.  Packed and int32 sharded scans may follow each other in one EGPU_F_INPUTS_READY
 * pipelined stream.  EGPU_ERR_STATE under EGPU_VARIANT_GRID.  EGPU_ERR_INVALID, before anything is
 * launched or written: a non-NULL d_req_mem, NULL words or indices with R > 0, misaligned words or
 * indices. */
#define EGPU_IPC_HANDLE_BYTES 64
#define EGPU_MAX_RANKS 8
int egpu_peer_export(egpu_ctx* ctx, void* handle_out);
int egpu_peer_attach(egpu_ctx* ctx, int rank, int world, const void* handles);
int egpu_peer_detach(egpu_ctx* ctx);
int egpu_bestfit_batch_shard_dev(egpu_ctx* ctx, const int32_t* d_req_core,
                                 const int32_t* d_req_mem, int64_t R,
                                 int32_t* d_out_idx, int64_t* d_delta, int flags,
                                 uint64_t step, void* stream);
int egpu_table_apply_peers_dev(egpu_ctx* ctx, uint64_t step, int32_t* d_table_out,
                               int commit, void* stream);
/* K sharded steps in one launch: batch k is exchange step first_step + k (egpu_bestfit_batches_dev
 * + the fused push of egpu_bestfit_batch_shard_dev).  Without EGPU_F_APPLY d_table_out of the
 * batches is ignored (table' comes from the apply calls); with it the exchange steps are consumed
 * by the launch itself and no apply call must follow.
 *
 * K sharded prefix-commits in one launch (flags EGPU_F_PREFIX_COMMIT [| EGPU_F_COMMIT] [| EGPU_F_PACKED]):
 * batch k, in order for k = 0..K-1, is exactly one egpu_bestfit_batch_shard_prefix_dev call with
 * step = first_step + 2k and the same flags; the result is, bit for bit, what K such calls issued on one
 * stream give, and the call uses exchange steps first_step .. first_step + 2K - 1 (the caller advances
 * by 2K).  Per batch: rows commit while the running demand of their device fits, counted over the whole
 * shards of the lower ranks and this rank's earlier rows of that batch; the others get
 * EGPU_IDX_DEFERRED.  d_delta (may be NULL) receives THIS rank's committed demand, int64[2*D];
 * d_table_out (may be NULL) receives table - committed demand of all ranks, int32[3*D], identical on
 * every rank (unlike the snapshot steps, it is written).  With EGPU_F_COMMIT that table is installed
 * before batch k + 1 is scored; without it every batch is scored against the current table.  Never
 * oversubscribes.  With EGPU_F_PACKED every batch is in the packed batch layout of
 * egpu_bestfit_batches_dev (words, NULL d_req_mem, int8 indices).  The exchange vectors are those of
 * the single call, so ranks may mix formats and may mix this launch with single calls.  ONE launch
 * (egpu_launch_count + 1), ASYNCHRONOUS on `stream` with no synchronisation; it replays from a CUDA
 * graph, and a replay after egpu_table_set starts from the new table.  It shares the prefix-commit and
 * rounds scratch of the context: calls that use it must be ordered on one stream, or by the caller.
 * Every wait inside the launch gives up after about 2 s: a peer vector that does not arrive is recorded
 * as egpu_peer_last_timeout records it, a grid barrier is counted as for EGPU_F_DEVICE_ROUNDS.  The
 * batches after the one in progress are then left unwritten.  If the wait was for the other ranks'
 * uncapped demand (the base), or a grid barrier before the cut, the batch in progress commits nothing:
 * every row of it that is not -1 is EGPU_IDX_DEFERRED, and its d_delta, d_table_out and the table are left
 * as they were.  If it was for the committed demand (the apply), the batch's indices and d_delta are
 * final and, as in the single call, its d_table_out and the table are left alone.  EGPU_ERR_STATE when the context is not attached to peers or under EGPU_VARIANT_GRID,
 * EGPU_ERR_NO_TABLE without a table, EGPU_ERR_NOMEM (nothing committed) when scratch cannot be
 * allocated.  EGPU_ERR_INVALID, before anything is launched or written: EGPU_F_APPLY or
 * EGPU_F_INPUTS_READY with EGPU_F_PREFIX_COMMIT (this form always applies, and the single call refuses
 * EGPU_F_INPUTS_READY too), EGPU_F_PACKED without EGPU_F_PREFIX_COMMIT, any EGPU_F_ROUNDS or
 * EGPU_F_DEVICE_ROUNDS bit, first_step + 2K > 2^47, K outside 1..64, a batch with R >= 2^31, NULL or
 * misaligned arrays with R > 0, a non-NULL d_req_mem with EGPU_F_PACKED and a NULL one without it,
 * outputs of two batches that overlap.  This is a newly accepted flag set on an existing entry point:
 * egpu_abi_version() stays 1011. */
int egpu_bestfit_batches_shard_dev(egpu_ctx* ctx, const egpu_batch* batches, int32_t K, int flags,
                                   uint64_t first_step, void* stream);
/* Start gate for a sharded sequence.  egpu_peer_gate_dev enqueues a one-warp kernel that
 * waits (i) for this rank's host to call egpu_peer_gate_open - which the caller does after it
 * has enqueued everything that follows the gate - and (ii) for every peer's gate to have
 * reached the same point, through flags in peer memory.  The work behind the gate then starts
 * at the same time on every rank without any host in the way: launch skew between the ranks'
 * host threads no longer lands inside the sequence.  Every gate_dev needs exactly one
 * gate_open, on every rank, in the same order.  Works unattached too (host part only).
 * A gate that has waited ~2 s gives up and lets the stream proceed (this happens when kernel
 * launches are blocking - CUDA_LAUNCH_BLOCKING, a profiler - because the host then never gets
 * to open it); egpu_peer_gate_timeouts counts those (synchronises the device). */
int egpu_peer_gate_dev(egpu_ctx* ctx, void* stream);
int egpu_peer_gate_open(egpu_ctx* ctx);
int64_t egpu_peer_gate_timeouts(egpu_ctx* ctx);
/* Release launches (EGPU_F_RELEASE) of this context that were refused on the device, since creation.  An
 * asynchronous caller that passes a NULL d_table_out reads its refusals here.  Synchronises the device. */
int64_t egpu_release_refusals(egpu_ctx* ctx);
/* Prefix-commit (EGPU_F_PREFIX_COMMIT semantics, see egpu_bestfit_batch) over row shards.
 * The batch is the concatenation of the ranks' shards in rank order; request r of rank g
 * commits iff the running demand of its device over ALL earlier rows - the whole shards of
 * ranks < g and the rows before r here - still fits (SURVEY.md Appendix A.5: "rank-major
 * across shards").  One asynchronous call per rank; it uses TWO exchange steps, `step` (the
 * uncapped demand of every shard, pushed by the scan itself; every rank then knows the base
 * offset of its shard) and `step + 1` (the committed demand after the cut), so the caller
 * advances `step` by 2.  Outputs: d_out_idx with EGPU_IDX_DEFERRED for the rows beyond the
 * cut; d_delta[2*D] = THIS rank's committed demand (may be NULL); d_table_out[3*D] =
 * table - committed demand of all ranks, identical on every rank (may be NULL);
 * EGPU_F_COMMIT installs it.  Never oversubscribes.
 * flags EGPU_F_PACKED [| EGPU_F_PREFIX_COMMIT] [| EGPU_F_COMMIT]: the same on packed words, with the
 * arguments and refusals of the packed sharded scan (egpu_bestfit_batch_shard_dev above); d_out_idx
 * receives int8 indices: device, -1 or EGPU_IDX_DEFERRED.  The exchange steps carry the same vectors
 * as in the int32 call.  EGPU_ERR_STATE under EGPU_VARIANT_GRID (in either format).
 *
 * Rounds to the fixed point over row shards in one launch (flags EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT |
 * EGPU_F_ROUNDS | EGPU_F_DEVICE_ROUNDS [| EGPU_F_PACKED]): the result is, bit for bit, egpu_bestfit_batch_rounds
 * with no round limit on the concatenation of the ranks' shards in rank order - every rank's slice of the indices
 * and the table every rank ends with.  Round 1 is the prefix-commit above, committing; round j + 1 re-submits,
 * rank-major, the rows round j deferred against the table round j committed.  Every index ends as a device or -1,
 * never EGPU_IDX_DEFERRED; sticky oversubscription flags are kept.  d_delta (may be NULL) receives THIS rank's
 * demand committed over all rounds, int64[2*D]; d_table_out (may be NULL) the last round's table', int32[3*D] with
 * the oversub words 0, identical on every rank; the committed table is installed in stream order.  If every rank
 * passes R = 0 the call writes zero sums and table' = the current table.  The rows are int32 arrays or, with
 * EGPU_F_PACKED, the packed arguments above (words, NULL d_req_mem, int8 indices).
 * Exchange steps: the call uses `step` and `step + 1`, as the prefix call does, whatever the number of rounds
 * (every round reuses the two), so the caller advances by 2.  Every rank must issue this call with the same
 * `step`; R may differ between ranks, and a rank with no deferred rows left still takes part in every round.  A
 * rank that issues the plain prefix call on that step instead is a usage error: its peers give up after about 2 s.
 * ONE launch (egpu_launch_count + 1), ASYNCHRONOUS on `stream` with no synchronisation; it replays from a CUDA
 * graph, and a replay after egpu_table_set starts from the new table.  The launch is cooperative: the runtime
 * refuses a grid it cannot keep resident rather than letting it wait.  Scratch is the rounds scratch of
 * egpu_bestfit_batch_dev with EGPU_F_DEVICE_ROUNDS, sized by this rank's R and allocated before the launch: an
 * allocation failure returns EGPU_ERR_NOMEM with nothing committed.  The call shares that scratch with every
 * prefix-commit and rounds call of the context, so they must be ordered on one stream, or by the caller.
 * Timeouts: every wait inside the launch gives up after about 2 s and ends the launch.  A pull that gives up is
 * recorded as egpu_peer_last_timeout reports it; a grid barrier that gives up is counted and reported by the next
 * host-form call with EGPU_F_DEVICE_ROUNDS (EGPU_ERR_CUDA).  If the wait is in round 1 before the cut (the other
 * ranks' uncapped demand, or a grid barrier), nothing commits: every row that chose a device is
 * EGPU_IDX_DEFERRED, and the table, d_delta and d_table_out are left as they were, as in the multi-batch form of
 * egpu_bestfit_batches_shard_dev.  If it is round 1's apply, the rows stay as its cut left them and the table is
 * left alone, as in the prefix call.  In a later round the rounds already applied stay installed and the rows not
 * finished stay EGPU_IDX_DEFERRED.  d_delta and d_table_out are written at the fixed point only.
 * EGPU_ERR_STATE when the context is not attached to peers or under EGPU_VARIANT_GRID, EGPU_ERR_NO_TABLE without a
 * table.  EGPU_ERR_INVALID, before anything is launched or written: EGPU_F_ROUNDS or EGPU_F_DEVICE_ROUNDS in any
 * other combination (EGPU_F_INPUTS_READY or EGPU_F_APPLY with them among it), step + 2 > 2^47, R >= 2^31, NULL or
 * misaligned arrays with R > 0, a non-NULL d_req_mem with EGPU_F_PACKED and a NULL one without it.  This is a
 * newly accepted flag set on an existing entry point: egpu_abi_version() stays 1011.  The K-batch form
 * (egpu_bestfit_batches_shard_dev) does not take these flags; K calls on one stream give K batches, one launch
 * each.
 *
 * Release over row shards (flags EGPU_F_RELEASE [| EGPU_F_COMMIT] [| EGPU_F_PACKED]; DESIGN.md 2.8): each rank
 * passes its own rows and index array - typically the slice of the indices this rank's sharded placement call
 * produced - with the row rule and the packed arguments of the single-GPU release (egpu_bestfit_batch_dev): the
 * index array is READ, never written, and rows that hold nothing are skipped.  The result is, bit for bit, the
 * single-GPU release of the concatenation of every rank's rows against the table the ranks share: U = the int64 sum
 * over the ranks of each rank's U_g, the same all-or-nothing test on every touched device (EGPU_REL_FLAGGED,
 * EGPU_REL_EXCEEDS), and the same install of free + U, re-sorted, with the sticky flags kept.  The decision is taken
 * from each rank's own table: ranks whose tables are equal, as every sharded call keeps them, decide the same way
 * and install the same table; a caller who installed different tables on different ranks gets no guarantee.
 * Written whether accepted or refused: d_delta (may be NULL) = THIS rank's U_g, int64[2*D]; d_table_out (may be
 * NULL) = free + U when accepted and the current table when refused, int32[2*D], followed by the D reason words,
 * identical on every rank.  With EGPU_F_COMMIT an accepted result is installed on every rank in stream order.  A
 * refused launch changes nothing but d_delta, d_table_out and egpu_release_refusals, which each rank counts for
 * itself.  Exchange steps: the call uses ONE step, `step`, so the caller advances by 1.  Every rank must issue the
 * call with the same `step`, and every rank launches, with R = 0 too (it contributes zero sums).  A rank that
 * issues a different call on that step (a prefix call, say) is a usage error: its peers give up after about 2 s.
 * ONE launch (egpu_launch_count + 1), ASYNCHRONOUS on `stream`, fully ordered behind what the stream holds; it
 * replays from a CUDA graph and does not depend on the scan variant (it works under EGPU_VARIANT_GRID too).
 * Timeout: a peer whose sums do not arrive makes the launch give up after about 2 s; d_delta is written, d_table_out
 * and the table are left as they were, no refusal is counted, and egpu_peer_last_timeout reports step + 1.  The
 * ranks' tables may then differ (a peer may have installed the release): the caller re-installs a table on every
 * rank (egpu_table_set).  EGPU_ERR_STATE when the context is not attached to peers, EGPU_ERR_NO_TABLE without a
 * table.  EGPU_ERR_INVALID, before anything is launched or written: any other bit with EGPU_F_RELEASE
 * (EGPU_F_PREFIX_COMMIT, EGPU_F_ROUNDS, EGPU_F_DEVICE_ROUNDS, EGPU_F_INPUTS_READY and EGPU_F_APPLY among them),
 * R >= 2^31, step >= 2^47, NULL or misaligned arrays with R > 0, a non-NULL d_req_mem with EGPU_F_PACKED and a
 * NULL one without it, d_delta and d_table_out that overlap.  This is a newly accepted flag set on an existing entry
 * point: egpu_abi_version() stays 1011.  egpu_bestfit_batches_shard_dev, egpu_bestfit_batch_shard_dev,
 * egpu_bestfit_batches_dev and egpu_bestfit_batch_shard_lag_dev keep their handling of EGPU_F_RELEASE. */
int egpu_bestfit_batch_shard_prefix_dev(egpu_ctx* ctx, const int32_t* d_req_core,
                                        const int32_t* d_req_mem, int64_t R,
                                        int32_t* d_out_idx, int64_t* d_delta,
                                        int32_t* d_table_out, int flags, uint64_t step,
                                        void* stream);
/* Scan + lagged apply in ONE launch: as egpu_bestfit_batch_shard_dev, and the same last CTA
 * also applies the exchanged vectors of step (step - lag) (1 <= lag <= 16) and writes that
 * step's table' to d_table_out_lagged (skipped while step < lag).  A whole sharded sequence
 * is then a single stream of scan launches, finished by one
 * egpu_table_apply_peers_multi_dev(first_step = last - lag + 1, lag steps) for the tail.
 * The wait for step - lag is the back-pressure: no rank gets more than `lag` steps ahead
 * of the slowest.  A sequence restarted from step 0 (a replayed CUDA graph) must be
 * separated from the previous one by a barrier across the ranks.  Never commits.
 * Packed: EGPU_F_PACKED AND a NULL d_req_mem run the packed sharded scan (arguments as for
 * egpu_bestfit_batch_shard_dev with EGPU_F_PACKED; the lagged table' is the same in both formats).
 * COMPATIBILITY: this call has never checked flags other than EGPU_F_COMMIT, so EGPU_F_PACKED with a
 * non-NULL d_req_mem still runs the int32 scan on two int32 arrays, as it did before 1.9. */
int egpu_bestfit_batch_shard_lag_dev(egpu_ctx* ctx, const int32_t* d_req_core,
                                     const int32_t* d_req_mem, int64_t R,
                                     int32_t* d_out_idx, int64_t* d_delta, int flags,
                                     uint64_t step, int lag, int32_t* d_table_out_lagged,
                                     void* stream);
/* Same for nsteps (1..64) consecutive steps in one launch; d_table_outs is a HOST array of
 * nsteps device pointers (entries may be NULL).  With commit the steps are applied on top
 * of each other and the last table' is installed. */
int egpu_table_apply_peers_multi_dev(egpu_ctx* ctx, uint64_t first_step, int nsteps,
                                     int32_t* const* d_table_outs, int commit,
                                     void* stream);
/* step + 1 of the last apply that gave up waiting for a peer (~2 s), 0 if none */
int64_t egpu_peer_last_timeout(egpu_ctx* ctx);

/* Deterministic synthetic request generator on the device (same counter-based
 * RNG as the CPU generators; DESIGN.md §6).  dist: 2 = cfg2, 3 = cfg3. */
int egpu_synth_requests_dev(egpu_ctx* ctx, int dist, uint64_t seed,
                            int64_t first_row, int64_t R, int32_t* d_req_core,
                            int32_t* d_req_mem, void* stream);

/* ---- sequential mode --------------------------------------------------- */

/* Applies E events in order to the current table (which is updated).
 * kind[i] = EGPU_EV_ALLOC: a[i] = core, b[i] = mem  -> out_idx[i] = device or -1
 * kind[i] = EGPU_EV_FREE : a[i] = index of the ALLOC event to release
 *                          -> out_idx[i] = device released, or -1 when that
 *                          event is not a live allocation (not an ALLOC, not
 *                          earlier than i, infeasible, or already freed).
 * kind[i] = EGPU_EV_RELEASE: a[i] = device, b[i] = EGPU_PACK_REQUEST(core, mem) read as int32: gives back a
 *                          placement made before this call (an earlier call's ALLOC, a batch row, a restored
 *                          record), with no ledger in the library: the caller keeps (device, request).
 *                          -> out_idx[i] = a[i] when accepted, else -1 and nothing changes.  Accepted iff,
 *                          on the table as events 0..i-1 left it: 0 <= a[i] < D; 0 <= b[i] < 2^25 with
 *                          core <= EGPU_CORE_MAX; the device's oversubscription flag is clear unless the
 *                          request is (0, 0) (EGPU_REL_FLAGGED); and free + live + request stays within
 *                          EGPU_CORE_MAX and EGPU_MEM_MAX on the device (EGPU_REL_EXCEEDS), where live is
 *                          what this call's ALLOC events still hold there: its FREE events may give that
 *                          back later.  The decision is per event: a release that EGPU_F_RELEASE refuses as
 *                          a batch can be a stream whose first events are accepted.  The flags never change.
 * Every other kind is a no-op with out_idx[i] = -1, and so is an EGPU_EV_FREE whose target is not an
 * EGPU_EV_ALLOC.  EGPU_EV_RELEASE is a newly accepted input: egpu_abi_version() stays 1011. */
int egpu_replay(egpu_ctx* ctx, const int32_t* kind, const int32_t* a,
                const int32_t* b, int64_t E, int32_t* out_idx);

#ifdef __cplusplus
}
#endif
#endif /* EGPU_ALLOC_H */
