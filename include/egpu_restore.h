/*
 * egpu_restore.h — C ABI of placement-state restore (SURVEY.md §8 row n3): rebuild the
 * free-capacity table of the best-fit path from what the agent persisted.
 *
 * What the reference persists (elastic-ai/elastic-gpu-agent @ 2609107):
 *   - one Bolt record per pod in bucket "root" (pkg/storage/storage.go:13,53-57):
 *       key  "namespace/name"                          (pkg/types/pod.go:51-53)
 *       val  json.Marshal(map[container]*types.Device)  (pkg/types/pod.go:55-58), i.e.
 *            {"<container>":{"Hash":"1a2b3c4d","List":["0-00","3-07"],"ResourceName":"elasticgpu.io/gpu-core"}}
 *     read back with NewPIFromRaw (pkg/types/pod.go:39-49) inside Storage.ForEach
 *     (pkg/storage/storage.go:79-89);
 *   - one symlink per placed (container, GPU):  /host/dev/elastic-gpu-<Hash>-<i> -> /dev/nvidia<N>
 *     (pkg/operator/gpushare.go:10-14,31-55), created by PreStartContainer with N taken from
 *     the pod annotation (pkg/plugins/gpushare.go:114-128, :239-247).
 * The record says HOW MUCH a container holds (len(List) units of ResourceName: percent of a
 * card for gpu-core, MiB for gpu-memory, pkg/plugins/gpushare.go:24-33,159-168) but its IDs are
 * the kubelet's arbitrary pick from the advertised pool, not the physical GPU; WHERE it sits is
 * only in the symlink.  GPUManager.Restore() is declared and never implemented
 * (pkg/manager/manager.go:20); this is that function for the allocation table.
 *
 * Rule (builder-defined on top of the stored formats; DESIGN.md §2.7):
 *   for every container entry with n = len(List):
 *     gpu-core,   n <= 100: core[gpu(link 0)] += n
 *     gpu-core,   n  > 100: core[gpu(link i)] += 100 for i < n/100   (whole cards; the same
 *                           n/100 the reference uses, pkg/plugins/gpushare.go:62-69, base.go:282-292)
 *     gpu-memory:           mem[gpu(link 0)]  += n
 *   free = capacity - usage, saturated at 0 with an oversubscription flag (as table' in
 *   egpu_bestfit_batch).  An entry whose stored Hash is not the identity of its List
 *   (types.NewDevice, pkg/types/device.go:17-25,49-54; recomputed for all entries at once by
 *   the device-set identity batch of egpu_devhash.h) is stale or corrupt: reported, not
 *   counted.  So is an entry without its symlink (the container never started, or GC removed
 *   the link: pkg/plugins/base.go:281-300).
 *
 * No CPU fallback: the identity batch and the usage sums run on the GPU of the context.
 */
#ifndef EGPU_RESTORE_H
#define EGPU_RESTORE_H

#include <stdint.h>

#include "egpu_alloc.h"
#include "egpu_plugin.h" /* EGPU_RESOURCE_CORE / EGPU_RESOURCE_MEM */

#ifdef __cplusplus
extern "C" {
#endif

/* per-entry status */
#define EGPU_REC_OK            0
#define EGPU_REC_EMPTY         1 /* null entry or empty list: holds nothing */
#define EGPU_REC_FOREIGN       2 /* ResourceName of another plugin: ignored */
#define EGPU_REC_NO_LINK       3 /* a needed symlink is missing or points outside the table */
#define EGPU_REC_HASH_MISMATCH 4 /* stored Hash != identity of the stored List */
#define EGPU_REC_STATUS_COUNT  5

#define EGPU_RESOURCE_FOREIGN (-1)

/* flags */
#define EGPU_RESTORE_VERIFY  1 /* recompute every entry's identity and drop mismatches */
#define EGPU_RESTORE_INSTALL 2 /* make the restored table the context's table, as egpu_table_set does, but
                                  with out_table's oversubscription flags: they stay set until the next
                                  egpu_table_set, as after a committing batch */

/* Charge and release (DESIGN.md §2.7).  The caller's own stored records are the ledger: these flags
 * apply a few of them to the context's CURRENT table instead of rebuilding it from all of them.
 * U = the usage of the given entries, by the rule above and with the same per-entry statuses (only
 * EGPU_REC_OK entries count, in either direction; EGPU_RESTORE_VERIFY is optional, as for a restore).
 *   EGPU_RESTORE_CHARGE   free' = max(free - U, 0), oversub' = oversub | (free - U < 0), per device
 *                         and dimension: charging B on the table a restore of A installed gives exactly
 *                         the table a restore of A and B installs, flags included.  For placements this
 *                         context did not commit itself (the scheduler's pick, stored by PreStartContainer).
 *   EGPU_RESTORE_RELEASE  free' = free + U, flags unchanged: releasing B, a part of A, gives exactly the
 *                         table a restore of A without B installs.  For the records GC is about to delete.
 *                         All or nothing: refused with EGPU_ERR_STATE, installing and writing nothing, when
 *                         on some device d with U[d] > 0 the sticky oversubscription flag is set (the stored
 *                         table saturated at 0 and the deficit is lost: restore the node instead) or
 *                         free + U > cap_core / cap_mem (more is released than is in use).
 * Either one installs its result as EGPU_RESTORE_INSTALL does (sorted view, lookup tables rebuilt
 * before the next lookup scan) and writes it to out_table.  Refused with EGPU_ERR_INVALID before
 * anything is launched: both together, either with EGPU_RESTORE_INSTALL, D other than the context's
 * table size; EGPU_ERR_NO_TABLE without a table.  n_sets = 0 leaves the table as it is and writes it
 * to out_table.
 * Ordering: the current table is read as egpu_table_get reads it, after the context's stream is
 * synchronised and under the context's lock, and the result is installed before the lock is released,
 * as EGPU_RESTORE_INSTALL and egpu_table_set install theirs.  So every host-buffer call and every _dev
 * call on the context's own stream is counted; a committing _dev call on another stream must have
 * completed (synchronise that stream first), or one of the two changes is lost.
 * egpu_abi_version() stays 1011: these are newly accepted flags on existing entry points, as in
 * ABI 1.9-1.11; a library that predates them refuses them with EGPU_ERR_INVALID. */
#define EGPU_RESTORE_CHARGE  4
#define EGPU_RESTORE_RELEASE 8

/* Already-parsed form.  Entries = device-ID sets in the layout of egpu_device_hash_batch:
 *   ids_flat / id_offsets[n_ids + 1] / set_offsets[n_sets + 1]
 *   set_hash8     [n_sets * 8]   the stored Hash, 8 lowercase hex characters, no NUL
 *   set_resource  [n_sets]       EGPU_RESOURCE_CORE / _MEM / _FOREIGN
 *   link_offsets  [n_sets + 1], link_gpu[link_offsets[n_sets]]: link_gpu[link_offsets[s] + i]
 *                 is the N of the target /dev/nvidiaN of symlink "<Hash>-<i>", or -1 if absent
 *   cap_core / cap_mem [D]       capacity per GPU (100 and MiB: egpu_table_set's domain)
 * Outputs: out_table[3 * D] = free_core', free_mem', oversub (any may not be NULL);
 *          out_status[n_sets] (may be NULL). */
int egpu_table_restore_flat(egpu_ctx* ctx, const char* ids_flat, const int64_t* id_offsets, int64_t n_ids,
                            const int64_t* set_offsets, int64_t n_sets, const char* set_hash8,
                            const int32_t* set_resource, const int64_t* link_offsets, const int32_t* link_gpu,
                            const int32_t* cap_core, const int32_t* cap_mem, int32_t D, int flags,
                            int32_t* out_table, int32_t* out_status);

/* Raw form: the (key, value) pairs exactly as bucket.ForEach yields them, and the directory
 * listing of /host/dev as (file name, readlink target) pairs.
 *   link_names[i]   "elastic-gpu-<Hash>-<i>" (a bare "<Hash>-<i>" is accepted too); names of
 *                   other files, including "elastic-gpuctl-*", are skipped
 *   link_targets[i] "/dev/nvidia<N>"; other targets are skipped
 * A key that is not "namespace/name" or a value that is not the JSON above fails the whole
 * call with EGPU_ERR_PARSE, as NewPIFromRaw's error aborts ForEach; egpu_last_error names
 * the record.  Outputs: out_table[3 * D]; out_counts[EGPU_REC_STATUS_COUNT] = entries per
 * status (may be NULL); out_record_status[n_records] = the worst status among the record's
 * entries (may be NULL). */
int egpu_table_restore(egpu_ctx* ctx, const char* const* keys, const int64_t* key_lens, const char* const* vals,
                       const int64_t* val_lens, int64_t n_records, const char* const* link_names,
                       const char* const* link_targets, int64_t n_links, const int32_t* cap_core,
                       const int32_t* cap_mem, int32_t D, int flags, int32_t* out_table, int64_t* out_counts,
                       int32_t* out_record_status);

#ifdef __cplusplus
}
#endif
#endif /* EGPU_RESTORE_H */
