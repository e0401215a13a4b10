"""Python mirror of include/egpu_restore.h: rebuild the free-capacity table from the agent's
stored placement records (Bolt key/value pairs, pkg/types/pod.go:39-58) and the
/host/dev/elastic-gpu-<Hash>-<i> symlinks (pkg/operator/gpushare.go:31-55) — the
GPUManager.Restore() the reference declares and never implements (pkg/manager/manager.go:20)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L

REC_OK, REC_EMPTY, REC_FOREIGN, REC_NO_LINK, REC_HASH_MISMATCH = range(5)
REC_STATUS_COUNT = 5
RESTORE_VERIFY = 1
RESTORE_INSTALL = 2
RESTORE_CHARGE = 4
RESTORE_RELEASE = 8
RESOURCE_CORE, RESOURCE_MEM, RESOURCE_FOREIGN = 0, 1, -1


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _flags(verify, install, charge, release):
    return ((RESTORE_VERIFY if verify else 0) | (RESTORE_INSTALL if install else 0) | (RESTORE_CHARGE if charge else 0)
            | (RESTORE_RELEASE if release else 0))


def restore_table(alloc, records, links, cap_core, cap_mem, verify: bool = True, install: bool = False,
                  charge: bool = False, release: bool = False):
    """egpu_table_restore.  records: iterable of (key bytes, value bytes) as bucket.ForEach yields
    them; links: iterable of (file name, readlink target).  charge / release apply the records'
    usage to the context's current table instead (EGPU_RESTORE_CHARGE / EGPU_RESTORE_RELEASE).
    Returns (free_core, free_mem, oversub, counts[5], record_status[n_records])."""
    records = [(bytes(k), bytes(v)) for k, v in records]
    links = [(n.encode() if isinstance(n, str) else bytes(n), t.encode() if isinstance(t, str) else bytes(t))
             for n, t in links]
    n, nl = len(records), len(links)
    keys = (C.c_char_p * max(1, n))(*[k for k, _ in records])
    vals = (C.c_char_p * max(1, n))(*[v for _, v in records])
    klen = np.asarray([len(k) for k, _ in records] or [0], dtype=np.int64)
    vlen = np.asarray([len(v) for _, v in records] or [0], dtype=np.int64)
    names = (C.c_char_p * max(1, nl))(*[a for a, _ in links])
    targets = (C.c_char_p * max(1, nl))(*[b for _, b in links])
    cc, cm = _i32(cap_core), _i32(cap_mem)
    D = cc.size
    table = np.zeros(3 * D, dtype=np.int32)
    counts = np.zeros(REC_STATUS_COUNT, dtype=np.int64)
    rstat = np.zeros(max(1, n), dtype=np.int32)
    flags = _flags(verify, install, charge, release)
    rc = L.load().egpu_table_restore(alloc.handle, keys, C.c_void_p(klen.ctypes.data), vals, C.c_void_p(vlen.ctypes.data), n,
                                     names, targets, nl, C.c_void_p(cc.ctypes.data), C.c_void_p(cm.ctypes.data), D, flags,
                                     C.c_void_p(table.ctypes.data), C.c_void_p(counts.ctypes.data),
                                     C.c_void_p(rstat.ctypes.data))
    if rc != L.OK:
        raise L.EgpuError(rc, "egpu_table_restore", L.load().egpu_last_error(alloc.handle).decode())
    return table[:D].copy(), table[D:2 * D].copy(), table[2 * D:].copy(), counts, rstat[:n].copy()


def restore_table_flat(alloc, sets, hashes, resources, links, cap_core, cap_mem, verify: bool = True,
                       install: bool = False, charge: bool = False, release: bool = False):
    """egpu_table_restore_flat.  sets: list of ID lists; hashes: stored 8-hex strings; resources:
    RESOURCE_* per set; links: per set, the list of GPU indices of its symlinks (-1 = absent);
    charge / release as in restore_table.  Returns (free_core, free_mem, oversub, status[n_sets])."""
    from .devhash import flatten
    flat, id_off, set_off = flatten(sets)
    n_sets = len(sets)
    h8 = b"".join((h.encode() + b"????????")[:8] for h in hashes)
    res = _i32(resources if n_sets else [0])
    loff = np.zeros(n_sets + 1, dtype=np.int64)
    lg = []
    for i, l in enumerate(links):
        lg.extend(l)
        loff[i + 1] = len(lg)
    lgpu = _i32(lg or [0])
    cc, cm = _i32(cap_core), _i32(cap_mem)
    D = cc.size
    table = np.zeros(3 * D, dtype=np.int32)
    status = np.zeros(max(1, n_sets), dtype=np.int32)
    flags = _flags(verify, install, charge, release)
    rc = L.load().egpu_table_restore_flat(alloc.handle, C.c_char_p(flat), C.c_void_p(id_off.ctypes.data), len(id_off) - 1,
                                          C.c_void_p(set_off.ctypes.data), n_sets, C.c_char_p(h8),
                                          C.c_void_p(res.ctypes.data), C.c_void_p(loff.ctypes.data),
                                          C.c_void_p(lgpu.ctypes.data), C.c_void_p(cc.ctypes.data),
                                          C.c_void_p(cm.ctypes.data), D, flags, C.c_void_p(table.ctypes.data),
                                          C.c_void_p(status.ctypes.data))
    if rc != L.OK:
        raise L.EgpuError(rc, "egpu_table_restore_flat", L.load().egpu_last_error(alloc.handle).decode())
    return table[:D].copy(), table[D:2 * D].copy(), table[2 * D:].copy(), status[:n_sets].copy()
