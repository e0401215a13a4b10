/*
 * egpu_plugin.h — C ABI of the plugin-side host logic around the best-fit path:
 * the device-ID codec and GetPreferredAllocation for one container request.
 *
 * Reference interfaces (elastic-ai/elastic-gpu-agent @ 2609107):
 *   egpu_device_id_format / egpu_device_id_parse
 *       the fake device IDs the plugins advertise, fmt.Sprintf("%d-%02d", gpu, j)
 *       (pkg/plugins/gpushare.go:28 for gpu-core, :163 for gpu-memory);
 *   egpu_preferred_allocation
 *       pluginapi.ContainerPreferredAllocationRequest -> ...Response
 *       (vendor/k8s.io/kubelet/pkg/apis/deviceplugin/v1beta1/api.pb.go:564-571, 675-677;
 *       api.proto:133-150), the body baseDevicePlugin.GetPreferredAllocation leaves empty
 *       (pkg/plugins/base.go:94-96).
 *
 * The choice itself is made by the CUDA best-fit scan (egpu_bestfit_query); this file
 * only turns ID strings into the capacity table and the answer back into IDs.  No CPU
 * fallback: without a context (no GPU) the call fails.
 *
 * egpu_preferred_allocation_batch answers every container request of a PreferredAllocationRequest
 * in one call from flat ID buffers; parsing, counting, must-include matching, the best-fit choice
 * and the ID selection all run on the GPU, with the answers of egpu_preferred_allocation.
 */
#ifndef EGPU_PLUGIN_H
#define EGPU_PLUGIN_H

#include <stdint.h>

#include "egpu_alloc.h"

#ifdef __cplusplus
extern "C" {
#endif

#define EGPU_RESOURCE_CORE 0  /* elasticgpu.io/gpu-core:   one ID per percent, 100 per GPU */
#define EGPU_RESOURCE_MEM  1  /* elasticgpu.io/gpu-memory: one ID per MiB */

/* "%d-%02d".  Returns the length written (excluding NUL) or EGPU_ERR_INVALID if it
 * does not fit in cap bytes or an argument is negative. */
int egpu_device_id_format(int32_t gpu, int64_t unit, char* out, int64_t cap);

/* Strict inverse: decimal gpu, '-', decimal unit of at least two digits; nothing else.
 * EGPU_ERR_PARSE otherwise. */
int egpu_device_id_parse(const char* id, int32_t* gpu, int64_t* unit);

/* One ContainerPreferredAllocationRequest.
 *   available_ids[n_available], must_include_ids[n_must]: NUL-terminated ID strings
 *   allocation_size: number of IDs (= units of `resource`) the container asks for
 * The free table is what the available IDs say: per GPU, the number of available units
 * of this resource (the other resource is unconstrained).  The request is
 * allocation_size units; the GPU is the best fit (tightest leftover, lowest index).
 * must_include IDs pin the GPU: they must all sit on one GPU that can hold the request.
 * Output: out_positions[allocation_size] = indices into available_ids of the chosen IDs,
 * must-include IDs first, then the lowest unit numbers of the chosen GPU; *out_gpu = the
 * GPU index.  EGPU_ERR_UNSAT when no single GPU can satisfy the request (kubelet then
 * falls back to its own choice), EGPU_ERR_PARSE on a malformed ID.
 * Whole-card requests (gpu-core, allocation_size > 100): the reference hands such a container
 * allocation_size / 100 whole GPUs (pkg/plugins/gpushare.go:62-69).  The size must be a multiple of
 * 100; the GPUs are chosen one after the other, each the best fit among the cards that are still
 * completely available (must-include GPUs first); the answer lists all 100 IDs of every chosen card,
 * *out_gpu is the first one.
 * The context's own capacity table is not touched (the availability table of the request is
 * scored through egpu_bestfit_query), so the context that tracks the node's committed
 * placement can serve these calls too, concurrently with commits and replays. */
int egpu_preferred_allocation(egpu_ctx* ctx, const char* const* available_ids, int64_t n_available,
                              const char* const* must_include_ids, int64_t n_must,
                              int32_t allocation_size, int resource, int32_t* out_positions,
                              int32_t* out_gpu);

#define EGPU_PREFALLOC_MAX_REQUESTS 65536  /* container requests per egpu_preferred_allocation_batch call */

/* Every ContainerPreferredAllocationRequest of one PreferredAllocationRequest (or of several) in one
 * call, with all ID work on the GPU.
 * IDs: the layout of egpu_device_hash_batch - ids_flat, id_offsets[n_ids + 1] (int64 byte offsets,
 * id_offsets[0] == 0, no separators, no NULs; the buffer is id_offsets[n_ids] bytes long) and
 * set_offsets[2 * n_req + 1] (id indices).  Set 2q holds request q's available IDs, in the message's
 * order; set 2q + 1 holds its must-include IDs.  allocation_size[n_req].
 * Outputs:
 *   out_positions  request q's answer starts at sum_{q' < q} max(allocation_size[q'], 0); entries are
 *                  indices into request q's own available list (0-based), as egpu_preferred_allocation
 *                  returns them; -1 in every slot of a request whose code is not EGPU_OK
 *   out_gpu[n_req] first chosen GPU, -1 when the code is not EGPU_OK (may be NULL)
 *   out_rc[n_req]  exactly what egpu_preferred_allocation returns for that request alone:
 *                  EGPU_OK, EGPU_ERR_UNSAT, EGPU_ERR_PARSE or EGPU_ERR_INVALID
 * Per request, the first rule that applies decides the code (the order egpu_preferred_allocation
 * checks them in):
 *   1. allocation_size < 0: INVALID
 *   2. more must-include IDs than allocation_size: UNSAT, before any ID is parsed
 *   3. the first bad available ID in list order: malformed (including offsets that decrease or leave
 *      the buffer) PARSE, GPU index >= EGPU_MAX_DEVICES INVALID
 *   4. no available IDs: OK when allocation_size is 0, else UNSAT
 *   5. a whole-card size (gpu-core, > 100) that is not a multiple of 100: UNSAT
 *   6. must-include IDs in order, the first failure: malformed PARSE; not among the available IDs
 *      UNSAT; more pinned GPUs than the request takes UNSAT
 *   7. no feasible GPU at some pick: UNSAT
 *   8. fewer IDs to give than asked for: UNSAT
 * Duplicate IDs count as often as they are listed (capped at a card's units); a must-include ID is
 * the first position of its string and is given once however often it is listed.
 * Return: EGPU_OK when out_rc is valid; EGPU_ERR_INVALID for call-level argument errors (NULL ctx, NULL
 * pointers with non-zero counts, bad resource, n_ids >= 2^31, n_req > EGPU_PREFALLOC_MAX_REQUESTS,
 * a negative buffer length, set offsets that do not start at 0, are not monotone or do not end at
 * n_ids); EGPU_ERR_NOMEM / EGPU_ERR_CUDA as elsewhere.  The context's own table is neither read nor
 * written.  The number of kernel launches does not depend on n_req. */
int egpu_preferred_allocation_batch(egpu_ctx* ctx, int resource,
                                    const char* ids_flat, const int64_t* id_offsets, int64_t n_ids,
                                    const int64_t* set_offsets, int64_t n_req,
                                    const int32_t* allocation_size,
                                    int32_t* out_positions, int32_t* out_gpu, int32_t* out_rc);

#ifdef __cplusplus
}
#endif
#endif /* EGPU_PLUGIN_H */
