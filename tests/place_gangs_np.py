"""Restatement of egpu::place_gangs (DESIGN.md §2.13), test infrastructure only.

`place` is §2.13's loop over gangs written over its own round loop: per gang, in gang order, rounds of §2.12 (each
pending pod replayed on every table with place_pods_np.replay_all, the node with the smallest (sum of core
leftovers, sum of memory leftovers, n), per node in pod order a pod commits when none of its devices is closed and its
demand fits on top of what the pods before it committed) run against the tables the kept gangs left, while the gang
has pending pods and placed + pending >= gang_min.  A gang with at least gang_min pods placed keeps its placement and
tables; any other gang is -1 throughout and leaves the tables as they were.  The round count is §2.13's: rounds run,
summed over gangs, with the early stop.  It shares nothing with the kernel's word packing, its staging or its
barriers.

`loop` is the literal rule: one place_pods_np.place per gang, kept or thrown away.
"""
from __future__ import annotations

import numpy as np

import place_pods_np
from place_pods_np import CORE_MAX, MEM_MAX, replay_all, valid_devices


def gangs_ok(gang_offsets, gang_min, G: int) -> bool:
    o = np.asarray(gang_offsets, dtype=np.int64)
    m = np.asarray(gang_min, dtype=np.int64)
    if o.size < 1 or o[0] != 0 or o[-1] != G or m.size != o.size - 1:
        return False
    size = np.diff(o)
    return bool(((size >= 1) & (m >= 1) & (m <= size)).all())


def _round(fc, fm, valid, rc, rm, off, pending, node, dev):
    """One §2.12 round over `pending` (pod indices, in pod order) on the tables fc / fm, updated in place.
    Returns (committed pods, deferred pods)."""
    D = fc.shape[1]
    chosen = {}  # node -> [(pod, devs)] in pod order
    for g in pending:
        cs = slice(off[g], off[g + 1])
        fits, devs, slc, slm = replay_all(fc, fm, valid, rc[cs], rm[cs])
        if not fits.any():
            continue  # fits no node when scored: -1 for good
        score = np.where(fits, slc * (1 << 21) + slm, np.iinfo(np.int64).max)
        n = int(score.argmin())  # the first node of a tie: the lowest n
        chosen.setdefault(n, []).append((g, devs[n]))
    committed, deferred = 0, []
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
                committed += 1
            else:
                closed[used] = True
                deferred.append(g)
        fc[n] -= acc_c
        fm[n] -= acc_m
    return committed, sorted(deferred)


def place(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets, gang_offsets, gang_min, trace=None):
    """Returns (node int32[G], dev int8[P], placed int32[J], free_core_out int32[N, D], free_mem_out int32[N, D],
    info [3]).

    trace: a list, or None.  Each round appends (j, positions, deferred) to it: gang j, the pods of the round's
    pending set in the order the kernel lays it out (a gang's round 1: the gang's whole range, pods outside the
    domain included; later rounds: the pods the round before deferred), and the indices into `positions` of the pods
    this round defers."""
    fc = np.array(free_core, dtype=np.int64, copy=True)
    fm = np.array(free_mem, dtype=np.int64, copy=True)
    rc = np.asarray(req_core, dtype=np.int64)
    rm = np.asarray(req_mem, dtype=np.int64)
    off = np.asarray(pod_offsets, dtype=np.int64)
    goff = np.asarray(gang_offsets, dtype=np.int64)
    gmin = np.asarray(gang_min, dtype=np.int64)
    N, D = fc.shape
    P, G, J = rc.size, off.size - 1, goff.size - 1
    node = np.full(G, -1, np.int32)
    dev = np.full(P, -1, np.int8)
    placed = np.zeros(J, np.int32)
    if N == 0 or P == 0:
        return node, dev, placed, fc.astype(np.int32), fm.astype(np.int32), [0, 0, 0]
    if not place_pods_np.offsets_ok(off, P) or not gangs_ok(goff, gmin, G):
        return node, dev, placed, fc.astype(np.int32), fm.astype(np.int32), [0, 0, 1]
    valid = valid_devices(fc, fm, d_valid)
    c_ok = (rc >= 0) & (rc <= CORE_MAX) & (rm >= 0) & (rm <= MEM_MAX)
    rounds = 0
    for j in range(J):
        pods = np.arange(goff[j], goff[j + 1])
        pending = [g for g in pods if c_ok[off[g]:off[g + 1]].all()]
        t_fc, t_fm = fc.copy(), fm.copy()
        t_node = np.full(G, -1, np.int32)
        t_dev = np.full(P, -1, np.int8)
        k = 0
        positions = pods
        while pending and k + len(pending) >= gmin[j]:
            rounds += 1
            committed, pending = _round(t_fc, t_fm, valid, rc, rm, off, pending, t_node, t_dev)
            k += committed
            if trace is not None:
                trace.append((j, positions, np.searchsorted(positions, pending)))
            positions = np.array(pending, np.int64)
        if k >= gmin[j]:  # then nothing is pending: the rounds ran to the fixed point
            fc, fm = t_fc, t_fm
            node[pods] = t_node[pods]
            cs = slice(off[goff[j]], off[goff[j + 1]])
            dev[cs] = t_dev[cs]
            placed[j] = k
    return node, dev, placed, fc.astype(np.int32), fm.astype(np.int32), [rounds, 0, 0]


def loop(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets, gang_offsets, gang_min):
    """The rule as written: place_pods_np.place once per gang, on the gang's containers and its pod offsets rebased
    to 0, kept when at least gang_min pods are placed.  Same outputs as `place`; info[0] sums place_pods' rounds."""
    fc = np.array(free_core, dtype=np.int32, copy=True)
    fm = np.array(free_mem, dtype=np.int32, copy=True)
    rc = np.asarray(req_core)
    rm = np.asarray(req_mem)
    off = np.asarray(pod_offsets, dtype=np.int64)
    goff = np.asarray(gang_offsets, dtype=np.int64)
    gmin = np.asarray(gang_min, dtype=np.int64)
    G, J = off.size - 1, goff.size - 1
    node = np.full(G, -1, np.int32)
    dev = np.full(rc.size, -1, np.int8)
    placed = np.zeros(J, np.int32)
    rounds = 0
    for j in range(J):
        g0, g1 = goff[j], goff[j + 1]
        c0, c1 = off[g0], off[g1]
        r_node, r_dev, r_fc, r_fm, r_info = place_pods_np.place(fc, fm, d_valid, rc[c0:c1], rm[c0:c1],
                                                                off[g0:g1 + 1] - c0)
        rounds += r_info[0]
        k = int((r_node >= 0).sum())
        if k >= gmin[j]:
            node[g0:g1] = r_node
            dev[c0:c1] = r_dev
            fc, fm = r_fc, r_fm
            placed[j] = k
    return node, dev, placed, fc, fm, [rounds, 0, 0]
