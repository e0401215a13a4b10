/*
 * egpu_devhash.h — C ABI of the device-set identity batch (SURVEY.md §8 row n2).
 *
 * Reference semantics, exactly (elastic-ai/elastic-gpu-agent @ 2609107):
 *   types.NewDevice  pkg/types/device.go:17-25   curr := clone(list); sort.Strings(curr)
 *   types.hash       pkg/types/device.go:49-54   hex(sha256(strings.Join(curr, ":")))[0:8]
 *   Device.Equals    pkg/types/device.go:27-29   Hash == && List == (&& ResourceName ==)
 * used by Allocate (pkg/plugins/gpushare.go:44,179), PreStartContainer (:92,217) and — once
 * per candidate container on the node — by KubeletDeviceLocator.Locate
 * (pkg/kube/locator.go:62-90), the reference's real CPU hot loop: at node scale the
 * gpu-memory plugin hands out one ID per MiB, so a 16 GiB container is 16384 strings to
 * sort and hash, for every candidate, on every container start.
 *
 * Unlike the best-fit rule this computation IS defined by the reference, so parity is
 * PINNED: byte-exact against oracle/devicehash_oracle.c, Python hashlib and the FIPS 180-4
 * vectors (tests/golden/device_hash.json).
 *
 * GPU formulation: device IDs only contain '-' and digits ("%d-%02d",
 * pkg/plugins/gpushare.go:28,163), so an ID of up to 16 characters packs into 64 bits at
 * 4 bits per character with the byte order preserved (pad 0 < '-' 1 < '0'..'9' 2..11).
 * All sets are sorted at once by an LSD radix sort on (set, packed id), the canonical
 * "a:b:c" strings are rendered from the sorted keys, and SHA-256 runs one message per
 * thread.  IDs with other characters or longer than 16 bytes are rejected
 * (EGPU_ERR_PARSE): they cannot come from this plugin.
 */
#ifndef EGPU_DEVHASH_H
#define EGPU_DEVHASH_H

#include <stdint.h>

#include "egpu_alloc.h"

#ifdef __cplusplus
extern "C" {
#endif

/* n_sets device-ID lists in one call.
 *   ids_flat    all ID strings concatenated, no separators, no NULs
 *   id_offsets  [n_ids + 1] byte offsets into ids_flat (id i = [id_offsets[i], id_offsets[i+1]))
 *   set_offsets [n_sets + 1] id indices (set s = ids [set_offsets[s], set_offsets[s+1]))
 * Outputs (either may be NULL):
 *   out_hash8   [n_sets * 9]  the reference's Device.Hash: 8 lowercase hex digits + NUL
 *   out_digest  [n_sets * 32] the full SHA-256 digest of the joined sorted list
 * An empty set hashes the empty string, as the reference would. */
int egpu_device_hash_batch(egpu_ctx* ctx, const char* ids_flat, const int64_t* id_offsets, int64_t n_ids,
                           const int64_t* set_offsets, int64_t n_sets, char* out_hash8, uint8_t* out_digest);

/* One list of NUL-terminated strings (what NewDevice takes). out_hash8: 9 bytes. */
int egpu_device_hash(egpu_ctx* ctx, const char* const* ids, int64_t n, char* out_hash8);

/* KubeletDeviceLocator.Locate's search (pkg/kube/locator.go:62-90): set 0 is the request,
 * sets 1..n_sets-1 are the candidate containers in the reference's iteration order.
 * *out_match = index (>= 1) of the first candidate whose sorted list equals the request's
 * (Device.Equals: same hash and same list), or -1. */
int egpu_device_locate(egpu_ctx* ctx, const char* ids_flat, const int64_t* id_offsets, int64_t n_ids,
                       const int64_t* set_offsets, int64_t n_sets, int64_t* out_match);

#ifdef __cplusplus
}
#endif
#endif /* EGPU_DEVHASH_H */
