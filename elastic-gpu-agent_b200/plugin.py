"""Python mirror of the plugin-side host logic (include/egpu_plugin.h), used by the tests
the way a Go handler would use the cgo binding: device-ID codec and
GetPreferredAllocation for one container request (pkg/plugins/base.go:94-96).
All work happens in the C/CUDA library."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L

RESOURCE_CORE = 0  # elasticgpu.io/gpu-core
RESOURCE_MEM = 1   # elasticgpu.io/gpu-memory


def format_device_id(gpu: int, unit: int) -> str:
    buf = C.create_string_buffer(40)
    n = L.load().egpu_device_id_format(int(gpu), int(unit), buf, 40)
    if n < 0:
        raise L.EgpuError(n, "egpu_device_id_format")
    return buf.value.decode()


def parse_device_id(s: str) -> tuple[int, int]:
    g, u = C.c_int32(), C.c_int64()
    rc = L.load().egpu_device_id_parse(s.encode(), C.byref(g), C.byref(u))
    if rc != L.OK:
        raise L.EgpuError(rc, f"egpu_device_id_parse({s!r})")
    return g.value, u.value


def _strs(ids):
    arr = (C.c_char_p * max(1, len(ids)))()
    keep = [s.encode() for s in ids]
    for i, b in enumerate(keep):
        arr[i] = b
    return arr, keep


def preferred_allocation(alloc, available: list[str], must_include: list[str], allocation_size: int,
                         resource: int = RESOURCE_CORE) -> tuple[list[str], int]:
    """ContainerPreferredAllocationRequest -> (deviceIDs, gpu index)."""
    av, _k1 = _strs(available)
    mu, _k2 = _strs(must_include)
    out = np.full(max(1, allocation_size), -1, dtype=np.int32)
    gpu = C.c_int32(-1)
    rc = L.load().egpu_preferred_allocation(alloc.handle, av, len(available), mu, len(must_include), int(allocation_size),
                                            int(resource), C.c_void_p(out.ctypes.data), C.byref(gpu))
    if rc != L.OK:
        raise L.EgpuError(rc, "egpu_preferred_allocation")
    return [available[p] for p in out[:allocation_size]], gpu.value


def flatten_requests(requests) -> tuple[bytes, np.ndarray, np.ndarray, np.ndarray]:
    """[(available, must_include, allocation_size)] -> (ids_flat, id_offsets, set_offsets, allocation_size), the
    layout of egpu_preferred_allocation_batch: UTF-8 bytes of every ID without separators, int64 byte offsets
    (n_ids + 1), int64 set offsets (2 * n_req + 1; set 2q = request q's available IDs, 2q + 1 its must-include
    IDs) and int32 sizes.  One join and cumulative lengths: no per-string ctypes objects."""
    ids: list[str] = []
    set_len = np.zeros(2 * len(requests), dtype=np.int64)
    sizes = np.zeros(len(requests), dtype=np.int32)
    for q, (available, must_include, allocation_size) in enumerate(requests):
        ids.extend(available)
        ids.extend(must_include)
        set_len[2 * q] = len(available)
        set_len[2 * q + 1] = len(must_include)
        sizes[q] = allocation_size
    joined = "".join(ids)
    flat = joined.encode()
    if len(flat) == len(joined):  # ASCII (every real ID): characters are bytes
        lens = np.fromiter(map(len, ids), dtype=np.int64, count=len(ids))
    else:
        lens = np.fromiter((len(s.encode()) for s in ids), dtype=np.int64, count=len(ids))
    id_offsets = np.zeros(len(ids) + 1, dtype=np.int64)
    np.cumsum(lens, out=id_offsets[1:])
    set_offsets = np.zeros(2 * len(requests) + 1, dtype=np.int64)
    np.cumsum(set_len, out=set_offsets[1:])
    return flat, id_offsets, set_offsets, sizes


def preferred_allocation_batch_flat(alloc, resource: int, flat, id_offsets: np.ndarray, set_offsets: np.ndarray,
                                    sizes: np.ndarray) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """egpu_preferred_allocation_batch on flat buffers (bytes or any buffer: numpy, pinned memory).  Returns
    (positions, gpu, rc): request q's answer is positions[sum(max(sizes[:q], 0)):][:max(sizes[q], 0)]."""
    id_offsets = np.ascontiguousarray(id_offsets, dtype=np.int64)
    set_offsets = np.ascontiguousarray(set_offsets, dtype=np.int64)
    sizes = np.ascontiguousarray(sizes, dtype=np.int32)
    n_req = sizes.size
    pos = np.empty(max(1, int(np.maximum(sizes, 0).sum())), dtype=np.int32)
    gpu = np.empty(max(1, n_req), dtype=np.int32)
    rc = np.empty(max(1, n_req), dtype=np.int32)
    flat = np.frombuffer(flat, dtype=np.uint8) if not isinstance(flat, np.ndarray) else flat  # no copy
    r = L.load().egpu_preferred_allocation_batch(alloc.handle, int(resource), C.c_void_p(flat.ctypes.data),
                                                 C.c_void_p(id_offsets.ctypes.data), id_offsets.size - 1,
                                                 C.c_void_p(set_offsets.ctypes.data), n_req, C.c_void_p(sizes.ctypes.data),
                                                 C.c_void_p(pos.ctypes.data), C.c_void_p(gpu.ctypes.data),
                                                 C.c_void_p(rc.ctypes.data))
    if r != L.OK:
        raise L.EgpuError(r, "egpu_preferred_allocation_batch")
    return pos, gpu[:n_req], rc[:n_req]


def preferred_allocation_batch(alloc, requests, resource: int = RESOURCE_CORE) -> list[tuple[list[str] | None, int, int]]:
    """Every ContainerPreferredAllocationRequest of a PreferredAllocationRequest in one call:
    requests = [(available, must_include, allocation_size)] -> [(deviceIDs or None, gpu index, return code)],
    each entry what preferred_allocation answers for that request alone (None and -1 where it raises)."""
    flat, id_offsets, set_offsets, sizes = flatten_requests(requests)
    pos, gpu, rc = preferred_allocation_batch_flat(alloc, resource, flat, id_offsets, set_offsets, sizes)
    out, off = [], 0
    for q, (available, _, size) in enumerate(requests):
        n = max(int(size), 0)
        if rc[q] == L.OK:
            out.append(([available[p] for p in pos[off:off + n]], int(gpu[q]), L.OK))
        else:
            out.append((None, -1, int(rc[q])))
        off += n
    return out
