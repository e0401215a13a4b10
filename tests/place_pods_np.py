"""Restatement of egpu::place_pods (DESIGN.md §2.12), test infrastructure only.

`place` is a plain numpy round loop written from the spec.  Per round, each pending pod is replayed on every table
at once (its containers one after another, each by best fit against what the pod's earlier containers left),
the pod takes the node with the smallest (sum of core leftovers, sum of memory leftovers, n), and per node, in pod
order, a pod commits when none of its devices is closed and its demand on every device it uses fits on top of what
the pods before it committed; a pod that does not commit closes every device it chose.  It shares nothing with the
kernel's word packing, its staging or its barriers.
"""
from __future__ import annotations

import numpy as np

CORE_MAX = 100
MEM_MAX = (1 << 18) - 1
MAX_POD = 8


def offsets_ok(pod_offsets, P: int) -> bool:
    o = np.asarray(pod_offsets, dtype=np.int64)
    if o.size < 1 or o[0] != 0 or o[-1] != P:
        return False
    step = np.diff(o)
    return bool(((step >= 1) & (step <= MAX_POD)).all())


def valid_devices(free_core, free_mem, d_valid):
    """[N, D] bool: the devices of §2.1's domain (d < d_valid[n] of a table whose valid devices are all in range)."""
    fc, fm = np.asarray(free_core), np.asarray(free_mem)
    N, D = fc.shape
    dv = np.asarray(d_valid, dtype=np.int64)
    cols = np.arange(D)[None, :] < dv[:, None]
    in_range = (fc >= 0) & (fc <= CORE_MAX) & (fm >= 0) & (fm <= MEM_MAX)
    table_ok = (dv >= 1) & (dv <= D) & (in_range | ~cols).all(axis=1)
    return cols & table_ok[:, None]


def replay_all(fc, fm, valid, cores, mems):
    """One pod's in-node replay on every table at once.  Returns (fits bool[N], devs int64[N, k], slc, slm int64[N]):
    devs[n, j] is container j's device on table n (meaningful where fits[n])."""
    N = fc.shape[0]
    left_c, left_m = fc.copy(), fm.copy()
    fits = valid.any(axis=1)
    devs = np.zeros((N, len(cores)), np.int64)
    slc = np.zeros(N, np.int64)
    slm = np.zeros(N, np.int64)
    rows = np.arange(N)
    for j, (c, m) in enumerate(zip(cores, mems)):
        lc, lm = left_c - c, left_m - m
        feas = valid & (lc >= 0) & (lm >= 0)
        rank = np.where(feas, lc * (MEM_MAX + 1) + lm, np.iinfo(np.int64).max)
        d = rank.argmin(axis=1)  # the first device of a tie: the lowest d
        fits &= feas.any(axis=1)
        devs[:, j] = d
        slc += lc[rows, d]
        slm += lm[rows, d]
        left_c[rows, d] -= c
        left_m[rows, d] -= m
    return fits, devs, slc, slm


def place(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets, trace=None):
    """Returns (node int32[G], dev int8[P], free_core_out int32[N, D], free_mem_out int32[N, D], info [3]).

    trace: a list, or None.  Each round appends (0, positions, deferred) to it: the pods of the round's pending set
    in the order the kernel lays it out (round 1: every pod, those outside the domain included; later rounds: the
    pods the round before deferred), and the indices into `positions` of the pods this round defers."""
    fc = np.array(free_core, dtype=np.int64, copy=True)
    fm = np.array(free_mem, dtype=np.int64, copy=True)
    rc = np.asarray(req_core, dtype=np.int64)
    rm = np.asarray(req_mem, dtype=np.int64)
    off = np.asarray(pod_offsets, dtype=np.int64)
    N, D = fc.shape
    P, G = rc.size, off.size - 1
    node = np.full(G, -1, np.int32)
    dev = np.full(P, -1, np.int8)
    if N == 0 or P == 0:
        return node, dev, fc.astype(np.int32), fm.astype(np.int32), [0, 0, 0]
    if not offsets_ok(off, P):
        return node, dev, fc.astype(np.int32), fm.astype(np.int32), [0, 0, 1]
    valid = valid_devices(fc, fm, d_valid)
    c_ok = (rc >= 0) & (rc <= CORE_MAX) & (rm >= 0) & (rm <= MEM_MAX)
    pod_ok = np.array([c_ok[off[g]:off[g + 1]].all() for g in range(G)], bool)
    pending = np.flatnonzero(pod_ok)
    rounds = 0
    while pending.size:
        rounds += 1
        chosen = {}  # node -> [(pod, devs)] in pod order
        for g in pending:
            cs = slice(off[g], off[g + 1])
            fits, devs, slc, slm = replay_all(fc, fm, valid, rc[cs], rm[cs])
            if not fits.any():
                continue  # fits no node when scored: -1 for good
            score = np.where(fits, slc * (1 << 21) + slm, np.iinfo(np.int64).max)
            n = int(score.argmin())  # the first node of a tie: the lowest n
            chosen.setdefault(n, []).append((g, devs[n]))
        deferred = []
        for n, pods in chosen.items():
            acc_c = np.zeros(D, np.int64)
            acc_m = np.zeros(D, np.int64)
            closed = np.zeros(D, bool)
            for g, devs in pods:
                cs = slice(off[g], off[g + 1])
                need_c = np.zeros(D, np.int64)
                need_m = np.zeros(D, np.int64)
                np.add.at(need_c, devs, rc[cs])
                np.add.at(need_m, devs, rm[cs])
                used = np.unique(devs)
                ok = not closed[used].any() and (acc_c[used] + need_c[used] <= fc[n, used]).all() and \
                    (acc_m[used] + need_m[used] <= fm[n, used]).all()
                if ok:
                    acc_c += need_c
                    acc_m += need_m
                    node[g] = n
                    dev[cs] = devs
                else:
                    closed[used] = True
                    deferred.append(g)
            fc[n] -= acc_c
            fm[n] -= acc_m
        positions = np.arange(G) if rounds == 1 else pending
        pending = np.array(sorted(deferred), np.int64)
        if trace is not None:
            trace.append((0, positions, np.searchsorted(positions, pending)))
    return node, dev, fc.astype(np.int32), fm.astype(np.int32), [rounds, 0, 0]
