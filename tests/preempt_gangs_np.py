"""Restatement of egpu::preempt_gangs (DESIGN.md §2.15), test infrastructure only.

`place` is §2.13's loop over gangs written over its own round loop, each round §2.14's at the gang's priority:
per pending pod, the nodes that take it as it is (place_pods_np.replay_all) are chosen by (sum lc, sum lm, n);
otherwise preempt_pods_np._victims walks, on every node at once, C capped per running job: of each job's pods in C on
the node only the slack_r that come last in the walk order (priority descending, h ascending) stay, slack_r being
the job's alive pods less its minimum at the start of the round.  Per node, in pod order, §2.14's commit; the
round's first-on-node preemptors then commit in pod order only while, for each job among their victims, their
victims of the job and those of every earlier such preemptor stay within slack_r.  A gang with fewer than gang_min
pods placed is thrown away with every eviction it made: the tables, the alive set and the counts are the copies
taken before it.  It shares nothing with the kernel's slot masks, its budget pass or its atomic rollback.

`loop` is the literal rule for uncapped inputs: one preempt_pods_np.place per gang at the gang's priority, the pods
a kept gang evicted marked gone for later gangs by zero demand and priority INT32_MAX, kept or thrown away.
"""
from __future__ import annotations

import numpy as np

import place_gangs_np
import preempt_pods_np
from place_pods_np import CORE_MAX, MEM_MAX, replay_all, valid_devices
from preempt_pods_np import BIAS, _demand, _victims, usable_nodes

INT32_MAX = 2**31 - 1


def index_ok(pod_offsets, P, gang_offsets, gang_min, run_offsets, Q, node_offsets, H, N, run_gang, run_gang_min):
    rg = np.asarray(run_gang, dtype=np.int64)
    rmin = np.asarray(run_gang_min, dtype=np.int64)
    G = np.asarray(pod_offsets).size - 1
    return (preempt_pods_np.index_ok(pod_offsets, P, run_offsets, Q, node_offsets, H, N)
            and place_gangs_np.gangs_ok(gang_offsets, gang_min, G) and rg.size == H
            and bool(((rg >= -1) & (rg < rmin.size)).all()) and bool((rmin >= 0).all()))


def capped(alive, rprio, rgang, noff, p, slack):
    """bool[H]: the running pods that may be in C this round (§2.15 rule 1).  Of each node's alive pods below p, a
    running job keeps only its slack[r] pods that come last in the walk order."""
    out = alive.copy()
    for n in range(noff.size - 1):
        hs = [h for h in range(noff[n], noff[n + 1]) if alive[h] and rprio[h] < p]
        seen = {}
        for h in sorted(hs, key=lambda h: (-int(rprio[h]), h), reverse=True):  # last in the walk first
            r = int(rgang[h])
            if r < 0:
                continue
            seen[r] = seen.get(r, 0) + 1
            if seen[r] > slack[r]:
                out[h] = False
    return out


def place(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets, gang_offsets, gang_min, gang_prio, run_core,
          run_mem, run_dev, run_offsets, run_prio, node_offsets, run_gang, run_gang_min):
    """Returns (node int32[G], dev int8[P], placed int32[J], evicted int32[H], free_core_out int32[N, D],
    free_mem_out int32[N, D], info [3])."""
    fc = np.array(free_core, dtype=np.int64, copy=True)
    fm = np.array(free_mem, dtype=np.int64, copy=True)
    dv = np.asarray(d_valid, dtype=np.int64)
    rc, rm = np.asarray(req_core, dtype=np.int64), np.asarray(req_mem, dtype=np.int64)
    off = np.asarray(pod_offsets, dtype=np.int64)
    goff, gmin = np.asarray(gang_offsets, dtype=np.int64), np.asarray(gang_min, dtype=np.int64)
    gprio = np.asarray(gang_prio, dtype=np.int64)
    qc, qm = np.asarray(run_core, dtype=np.int64), np.asarray(run_mem, dtype=np.int64)
    qd = np.asarray(run_dev, dtype=np.int64)
    roff, rprio = np.asarray(run_offsets, dtype=np.int64), np.asarray(run_prio, dtype=np.int64)
    noff = np.asarray(node_offsets, dtype=np.int64)
    rgang, rmin = np.asarray(run_gang, dtype=np.int64), np.asarray(run_gang_min, dtype=np.int64)
    N, D = fc.shape
    P, G, J, H, R = rc.size, off.size - 1, goff.size - 1, roff.size - 1, rmin.size
    node = np.full(G, -1, np.int32)
    dev = np.full(P, -1, np.int8)
    placed = np.zeros(J, np.int32)
    evicted = np.full(max(H, 0), -1, np.int32)
    if N == 0 or P == 0:
        return node, dev, placed, evicted, fc.astype(np.int32), fm.astype(np.int32), [0, 0, 0]
    if not index_ok(off, P, goff, gmin, roff, qc.size, noff, H, N, rgang, rmin):
        return node, dev, placed, evicted, fc.astype(np.int32), fm.astype(np.int32), [0, 0, 1]
    valid = valid_devices(fc, fm, dv) & usable_nodes(fc, fm, dv, qc, qm, qd, roff, noff)[:, None]
    dc, dm = _demand(H, D, qc, qm, qd, roff)
    alive = np.ones(H, bool)
    count = np.bincount(rgang[rgang >= 0], minlength=R).astype(np.int64)  # each job's alive pods
    c_ok = (rc >= 0) & (rc <= CORE_MAX) & (rm >= 0) & (rm <= MEM_MAX)
    rounds = 0
    for j in range(J):
        p = gprio[j]
        pending = [g for g in range(goff[j], goff[j + 1]) if c_ok[off[g]:off[g + 1]].all()]
        t_fc, t_fm, t_alive, t_count = fc.copy(), fm.copy(), alive.copy(), count.copy()
        t_node, t_dev, t_ev = node.copy(), dev.copy(), evicted.copy()
        k = 0
        while pending and k + len(pending) >= gmin[j]:
            rounds += 1
            slack = np.maximum(t_count - rmin, 0)
            c_alive = capped(t_alive, rprio, rgang, noff, p, slack)
            chosen = {}  # node -> [(pod, devs, V)] in pod order
            for g in pending:
                cs = slice(off[g], off[g + 1])
                fits, devs, slc, slm = replay_all(t_fc, t_fm, valid, rc[cs], rm[cs])
                if fits.any():
                    score = np.where(fits, slc * (1 << 21) + slm, np.iinfo(np.int64).max)
                    n = int(score.argmin())
                    chosen.setdefault(n, []).append((g, devs[n], []))
                    continue
                cand, V, devs, slc, slm = _victims(t_fc, t_fm, valid, rc[cs], rm[cs], p, rprio, c_alive, noff, dc, dm)
                if not cand.any():
                    continue  # no candidate when scored: -1 for good
                keys = [(max(int(rprio[h]) for h in V[n]), sum(int(rprio[h]) + BIAS for h in V[n]), len(V[n]),
                         int(slc[n]), int(slm[n]), n) for n in np.flatnonzero(cand)]
                n = min(keys)[-1]
                chosen.setdefault(n, []).append((g, devs[n], V[n]))
            deferred, preemptors = [], []
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
                    if V:  # the first pod of the round on n: the round budget decides
                        node_closed = True
                        preemptors.append((g, n, devs, V, need_c, need_m))
                        continue
                    used = np.unique(devs)
                    ok = not closed[used].any() and (acc_c[used] + need_c[used] <= t_fc[n, used]).all() and \
                        (acc_m[used] + need_m[used] <= t_fm[n, used]).all()
                    if ok:
                        acc_c += need_c
                        acc_m += need_m
                        t_node[g] = n
                        t_dev[cs] = devs
                        k += 1
                    else:
                        closed[used] = True
                        deferred.append(g)
                t_fc[n] -= acc_c
                t_fm[n] -= acc_m
            spent = np.zeros(R, np.int64)  # victims per job of this round's preemptors so far, committed or not
            for g, n, devs, V, need_c, need_m in sorted(preemptors, key=lambda x: x[0]):
                jobs = [int(rgang[h]) for h in V if rgang[h] >= 0]
                np.add.at(spent, jobs, 1)
                if any(spent[r] > slack[r] for r in jobs):
                    deferred.append(g)
                    continue
                t_ev[V] = g
                t_alive[V] = False
                np.subtract.at(t_count, jobs, 1)
                t_fc[n] += dc[V].sum(axis=0) - need_c
                t_fm[n] += dm[V].sum(axis=0) - need_m
                t_node[g] = n
                t_dev[off[g]:off[g + 1]] = devs
                k += 1
            pending = sorted(deferred)
        if k >= gmin[j]:  # then nothing is pending
            fc, fm, alive, count = t_fc, t_fm, t_alive, t_count
            node, dev, evicted = t_node, t_dev, t_ev
            placed[j] = k
    return node, dev, placed, evicted, fc.astype(np.int32), fm.astype(np.int32), [rounds, 0, 0]


def loop(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets, gang_offsets, gang_min, gang_prio, run_core,
         run_mem, run_dev, run_offsets, run_prio, node_offsets, run_gang=None, run_gang_min=None):
    """The rule as written when no running job is capped (R = 0): preempt_pods_np.place once per gang at its
    priority, on the gang's containers and its pod offsets rebased to 0, kept when at least gang_min pods are placed.
    A kept gang's victims stay listed for later gangs with zero demand and priority INT32_MAX, so no later pod can
    choose them and their capacity is in the tables.  Same outputs as `place`; info[0] sums preempt_pods' rounds."""
    fc = np.array(free_core, dtype=np.int32, copy=True)
    fm = np.array(free_mem, dtype=np.int32, copy=True)
    rc, rm = np.asarray(req_core), np.asarray(req_mem)
    off = np.asarray(pod_offsets, dtype=np.int64)
    goff, gmin = np.asarray(gang_offsets, dtype=np.int64), np.asarray(gang_min, dtype=np.int64)
    qc = np.array(run_core, dtype=np.int32, copy=True)
    qm = np.array(run_mem, dtype=np.int32, copy=True)
    roff = np.asarray(run_offsets, dtype=np.int64)
    rprio = np.array(run_prio, dtype=np.int32, copy=True)
    G, J, H = off.size - 1, goff.size - 1, roff.size - 1
    node = np.full(G, -1, np.int32)
    dev = np.full(rc.size, -1, np.int8)
    placed = np.zeros(J, np.int32)
    evicted = np.full(H, -1, np.int32)
    rounds = 0
    for j in range(J):
        g0, g1 = goff[j], goff[j + 1]
        c0, c1 = off[g0], off[g1]
        r = preempt_pods_np.place(fc, fm, d_valid, rc[c0:c1], rm[c0:c1], off[g0:g1 + 1] - c0,
                                  np.full(g1 - g0, gang_prio[j], np.int32), qc, qm, run_dev, run_offsets, rprio,
                                  node_offsets)
        r_node, r_dev, r_ev, r_fc, r_fm, r_info = r
        rounds += r_info[0]
        k = int((r_node >= 0).sum())
        if k >= gmin[j]:
            node[g0:g1] = r_node
            dev[c0:c1] = r_dev
            fc, fm = r_fc, r_fm
            placed[j] = k
            for h in np.flatnonzero(r_ev >= 0):
                evicted[h] = g0 + r_ev[h]
                qc[roff[h]:roff[h + 1]] = 0
                qm[roff[h]:roff[h + 1]] = 0
                rprio[h] = INT32_MAX
    return node, dev, placed, evicted, fc, fm, [rounds, 0, 0]
