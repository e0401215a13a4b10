"""Restatement of egpu::preempt_pods (DESIGN.md §2.14), test infrastructure only.

`place` is a numpy round loop written from the spec.  Per round, each pending pod is replayed on every table at once
(place_pods_np.replay_all).  If some node takes it as it is, it chooses among those nodes by (sum lc, sum lm, n), with
no victim.  Otherwise, on every node at once, C (the alive running pods below the pod's priority) is walked by
(priority descending, h ascending), one replay_all per step, dropping each h without which the pod still fits; the
pod takes the candidate with the smallest (highest victim priority, sum of (priority + 2^31), victims, sum lc, sum lm,
n).  Per node, in pod order: a pod without victims commits as in §2.12; a pod with victims commits only when it is the
first of the round on the node, evicts them and takes its demand, and closes the node.  It shares nothing with the
kernel's warp replay, its records or its barriers.

`single` is the rule for one pod (G = 1) written as plain Python loops per node and device, separately from `place`.
"""
from __future__ import annotations

import numpy as np

import place_pods_np
from place_pods_np import CORE_MAX, MAX_POD, MEM_MAX, replay_all, valid_devices

MAX_RUN = 128
BIAS = 1 << 31


def index_ok(pod_offsets, P, run_offsets, Q, node_offsets, H, N) -> bool:
    ro = np.asarray(run_offsets, dtype=np.int64)
    no = np.asarray(node_offsets, dtype=np.int64)
    if not place_pods_np.offsets_ok(pod_offsets, P):
        return False
    if ro.size != H + 1 or ro[0] != 0 or ro[-1] != Q or no.size != N + 1 or no[0] != 0 or no[-1] != H:
        return False
    rs, ns = np.diff(ro), np.diff(no)
    return bool(((rs >= 1) & (rs <= MAX_POD)).all() and ((ns >= 0) & (ns <= MAX_RUN)).all())


def usable_nodes(fc, fm, dv, qc, qm, qd, roff, noff):
    """bool[N]: the table is in §2.1's domain and the node's running data is consistent."""
    N, D = fc.shape
    valid = valid_devices(fc, fm, dv)
    ok = valid.any(axis=1)
    tot_c, tot_m = fc.astype(np.int64).copy(), fm.astype(np.int64).copy()
    for n in range(N):
        for h in range(noff[n], noff[n + 1]):
            for c in range(roff[h], roff[h + 1]):
                d = int(qd[c])
                if not (0 <= d < min(dv[n], D) and 0 <= qc[c] <= CORE_MAX and 0 <= qm[c] <= MEM_MAX):
                    ok[n] = False
                    continue
                tot_c[n, d] += qc[c]
                tot_m[n, d] += qm[c]
    over = ((tot_c > CORE_MAX) | (tot_m > MEM_MAX)) & valid
    return ok & ~over.any(axis=1)


def _demand(H, D, qc, qm, qd, roff):
    """[H, D] core and memory demand of each running pod per device of its node."""
    dc = np.zeros((H + 1, D), np.int64)  # row H: no pod
    dm = np.zeros((H + 1, D), np.int64)
    pod_of = np.repeat(np.arange(H), np.diff(roff))
    ok = (qd >= 0) & (qd < D)
    np.add.at(dc, (pod_of[ok], qd[ok]), qc[ok])
    np.add.at(dm, (pod_of[ok], qd[ok]), qm[ok])
    return dc, dm


def _victims(fc, fm, valid, cores, mems, p, rprio, alive, noff, dc, dm):
    """§2.14 steps 2 and 3 on every node at once, for a pod that fits no node as it is.  Returns (cand bool[N],
    V list of running pods per node, devs [N, k], slc, slm)."""
    N = fc.shape[0]
    H = rprio.size
    order = []
    for n in range(N):
        hs = [h for h in range(noff[n], noff[n + 1]) if alive[h] and rprio[h] < p]
        order.append(sorted(hs, key=lambda h: (-int(rprio[h]), h)))
    L = max((len(o) for o in order), default=0)
    idx = np.full((N, max(L, 1)), H, np.int64)  # H: no pod
    for n, o in enumerate(order):
        idx[n, :len(o)] = o
    base_c = fc + dc[idx].sum(axis=1)
    base_m = fm + dm[idx].sum(axis=1)
    has_c = np.array([len(o) > 0 for o in order])
    cand, devs, slc, slm = replay_all(base_c, base_m, valid, cores, mems)
    cand &= has_c
    inV = idx < H
    for t in range(L):
        h = idx[:, t]
        tc, tm = base_c - dc[h], base_m - dm[h]
        fits, tdevs, tslc, tslm = replay_all(tc, tm, valid, cores, mems)
        drop = cand & (h < H) & fits
        base_c[drop], base_m[drop] = tc[drop], tm[drop]
        devs[drop], slc[drop], slm[drop] = tdevs[drop], tslc[drop], tslm[drop]
        inV[drop, t] = False
    V = [[int(h) for h in idx[n][inV[n]]] for n in range(N)]
    return cand, V, devs, slc, slm


def place(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets, pod_prio, run_core, run_mem, run_dev,
          run_offsets, run_prio, node_offsets):
    """Returns (node int32[G], dev int8[P], evicted int32[H], free_core_out int32[N, D], free_mem_out int32[N, D],
    info [3])."""
    fc = np.array(free_core, dtype=np.int64, copy=True)
    fm = np.array(free_mem, dtype=np.int64, copy=True)
    dv = np.asarray(d_valid, dtype=np.int64)
    rc, rm = np.asarray(req_core, dtype=np.int64), np.asarray(req_mem, dtype=np.int64)
    off, prio = np.asarray(pod_offsets, dtype=np.int64), np.asarray(pod_prio, dtype=np.int64)
    qc, qm = np.asarray(run_core, dtype=np.int64), np.asarray(run_mem, dtype=np.int64)
    qd = np.asarray(run_dev, dtype=np.int64)
    roff, rprio = np.asarray(run_offsets, dtype=np.int64), np.asarray(run_prio, dtype=np.int64)
    noff = np.asarray(node_offsets, dtype=np.int64)
    N, D = fc.shape
    P, G, H = rc.size, off.size - 1, roff.size - 1
    node = np.full(G, -1, np.int32)
    dev = np.full(P, -1, np.int8)
    evicted = np.full(max(H, 0), -1, np.int32)
    if N == 0 or P == 0:
        return node, dev, evicted, fc.astype(np.int32), fm.astype(np.int32), [0, 0, 0]
    if not index_ok(off, P, roff, qc.size, noff, H, N):
        return node, dev, evicted, fc.astype(np.int32), fm.astype(np.int32), [0, 0, 1]
    valid = valid_devices(fc, fm, dv) & usable_nodes(fc, fm, dv, qc, qm, qd, roff, noff)[:, None]
    dc, dm = _demand(H, D, qc, qm, qd, roff)
    alive = np.ones(H, bool)
    c_ok = (rc >= 0) & (rc <= CORE_MAX) & (rm >= 0) & (rm <= MEM_MAX)
    pending = [g for g in range(G) if c_ok[off[g]:off[g + 1]].all()]
    rounds = 0
    while pending:
        rounds += 1
        chosen = {}  # node -> [(pod, devs, V)] in pod order
        for g in pending:
            cs = slice(off[g], off[g + 1])
            fits, devs, slc, slm = replay_all(fc, fm, valid, rc[cs], rm[cs])
            if fits.any():
                score = np.where(fits, slc * (1 << 21) + slm, np.iinfo(np.int64).max)
                n = int(score.argmin())
                chosen.setdefault(n, []).append((g, devs[n], []))
                continue
            cand, V, devs, slc, slm = _victims(fc, fm, valid, rc[cs], rm[cs], prio[g], rprio, alive, noff, dc, dm)
            if not cand.any():
                continue  # no candidate when scored: -1 for good
            keys = [(max(int(rprio[h]) for h in V[n]), sum(int(rprio[h]) + BIAS for h in V[n]), len(V[n]),
                     int(slc[n]), int(slm[n]), n) for n in np.flatnonzero(cand)]
            n = min(keys)[-1]
            chosen.setdefault(n, []).append((g, devs[n], V[n]))
        deferred = []
        for n, pods in chosen.items():
            acc_c = np.zeros(D, np.int64)
            acc_m = np.zeros(D, np.int64)
            closed = np.zeros(D, bool)
            node_closed = False
            for i, (g, devs, V) in enumerate(pods):
                cs = slice(off[g], off[g + 1])
                need_c = np.zeros(D, np.int64)
                need_m = np.zeros(D, np.int64)
                np.add.at(need_c, devs, rc[cs])
                np.add.at(need_m, devs, rm[cs])
                if node_closed or (V and i > 0):
                    node_closed |= bool(V)
                    deferred.append(g)
                    continue
                if V:  # the first pod of the round on n: evict, then take the demand
                    node_closed = True
                    evicted[V] = g
                    alive[V] = False
                    fc[n] += dc[V].sum(axis=0) - need_c
                    fm[n] += dm[V].sum(axis=0) - need_m
                    node[g] = n
                    dev[cs] = devs
                    continue
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
        pending = sorted(deferred)
    return node, dev, evicted, fc.astype(np.int32), fm.astype(np.int32), [rounds, 0, 0]


def _replay(tc, tm, rows, cores, mems):
    """One pod's in-node replay on one table as plain loops: (devices, sum lc, sum lm), or None."""
    tc, tm = list(tc), list(tm)
    devs, slc, slm = [], 0, 0
    for c, m in zip(cores, mems):
        if not (0 <= c <= CORE_MAX and 0 <= m <= MEM_MAX):
            return None
        best = None
        for d in range(rows):
            lc, lm = tc[d] - c, tm[d] - m
            if lc >= 0 and lm >= 0 and (best is None or (lc, lm, d) < best):
                best = (lc, lm, d)
        if best is None:
            return None
        lc, lm, d = best
        tc[d] -= c
        tm[d] -= m
        devs.append(d)
        slc += lc
        slm += lm
    return devs, slc, slm


def single(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets, pod_prio, run_core, run_mem, run_dev,
           run_offsets, run_prio, node_offsets):
    """The rule for one pending pod (G = 1), node by node: steps 1 to 3, the key, the smallest key commits.  Inputs
    must pass the eager checks except that nodes may be inconsistent (they offer nothing).  Same outputs as `place`."""
    fc = [[int(x) for x in row] for row in np.asarray(free_core)]
    fm = [[int(x) for x in row] for row in np.asarray(free_mem)]
    dv = [int(x) for x in d_valid]
    cores, mems = [int(x) for x in req_core], [int(x) for x in req_mem]
    p = int(pod_prio[0])
    qc, qm, qd = [int(x) for x in run_core], [int(x) for x in run_mem], [int(x) for x in run_dev]
    roff, rprio, noff = [int(x) for x in run_offsets], [int(x) for x in run_prio], [int(x) for x in node_offsets]
    N, D, H = len(fc), np.asarray(free_core).shape[1], len(rprio)
    assert len(pod_offsets) == 2

    def with_demand(n, pods):
        tc, tm = list(fc[n]), list(fm[n])
        for h in pods:
            for c in range(roff[h], roff[h + 1]):
                tc[qd[c]] += qc[c]
                tm[qd[c]] += qm[c]
        return tc, tm

    def consistent(n):
        if not 1 <= dv[n] <= D or any(not (0 <= fc[n][d] <= CORE_MAX and 0 <= fm[n][d] <= MEM_MAX) for d in range(dv[n])):
            return False
        for h in range(noff[n], noff[n + 1]):
            for c in range(roff[h], roff[h + 1]):
                if not (0 <= qd[c] < dv[n] and 0 <= qc[c] <= CORE_MAX and 0 <= qm[c] <= MEM_MAX):
                    return False
        tc, tm = with_demand(n, range(noff[n], noff[n + 1]))
        return all(tc[d] <= CORE_MAX and tm[d] <= MEM_MAX for d in range(dv[n]))

    best = None
    for n in range(N):
        if not consistent(n):
            continue
        r = _replay(fc[n], fm[n], dv[n], cores, mems)
        if r is not None:  # step 1
            key, V = (float("-inf"), 0, 0, r[1], r[2], n), []
        else:
            C = [h for h in range(noff[n], noff[n + 1]) if rprio[h] < p]  # step 2
            if not C or _replay(*with_demand(n, C), dv[n], cores, mems) is None:
                continue
            V = list(C)
            for h in sorted(C, key=lambda h: (-rprio[h], h)):  # step 3
                rest = [x for x in V if x != h]
                if _replay(*with_demand(n, rest), dv[n], cores, mems) is not None:
                    V = rest
            r = _replay(*with_demand(n, V), dv[n], cores, mems)
            key = (max(rprio[h] for h in V), sum(rprio[h] + BIAS for h in V), len(V), r[1], r[2], n)
        if best is None or key < best[0]:
            best = (key, V, r[0])
    node = np.full(1, -1, np.int32)
    dev = np.full(len(cores), -1, np.int8)
    evicted = np.full(H, -1, np.int32)
    out_c, out_m = np.array(fc, np.int32).reshape(N, D), np.array(fm, np.int32).reshape(N, D)
    in_domain = all(0 <= c <= CORE_MAX for c in cores) and all(0 <= m <= MEM_MAX for m in mems)
    if best is not None:
        key, V, devs = best
        n = key[-1]
        tc, tm = with_demand(n, V)
        for d, c, m in zip(devs, cores, mems):
            tc[d] -= c
            tm[d] -= m
        out_c[n], out_m[n] = tc, tm
        node[0] = n
        dev[:] = devs
        evicted[V] = 0
    return node, dev, evicted, out_c, out_m, [1 if in_domain else 0, 0, 0]
