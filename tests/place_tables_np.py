"""Restatements of egpu::place_tables (DESIGN.md §2.11), test infrastructure only.

`place` is a plain numpy round loop written from the spec: every table's valid devices concatenated node-major,
best fit over that concatenation by (free_core - core, free_mem - mem, position), prefix-commit per device in
request order, the deferred requests scored again against the tables the round left.  It shares nothing with the
kernel's word packing, its scan or its barriers.

`place_torch` is what a caller does without the operator: a torch loop of egpu::bestfit_tables, a min over the
nodes, a stable sort by device, a segmented cumsum and a scatter-subtract, with a host sync per round.  The GPU
tests compare with it at shapes too large for `place`; scripts/place_tables_probe.py times it.
"""
from __future__ import annotations

import numpy as np

CORE_MAX = 100
MEM_MAX = (1 << 18) - 1
NO_KEY = 0x7FFFFFFF


def table_in_domain(fc_row, fm_row, dv: int, D: int) -> bool:
    """§2.1's domain for one table: 1 <= d_valid <= D, and its first d_valid devices in range."""
    if not 1 <= dv <= D:
        return False
    c, m = np.asarray(fc_row[:dv]), np.asarray(fm_row[:dv])
    return bool(((c >= 0) & (c <= CORE_MAX) & (m >= 0) & (m <= MEM_MAX)).all())


def place(free_core, free_mem, d_valid, req_core, req_mem):
    """Returns (node int32[P], dev int8[P], free_core_out int32[N, D], free_mem_out int32[N, D], rounds)."""
    fc = np.array(free_core, dtype=np.int64, copy=True)
    fm = np.array(free_mem, dtype=np.int64, copy=True)
    dv = np.asarray(d_valid, dtype=np.int64)
    rc = np.asarray(req_core, dtype=np.int64)
    rm = np.asarray(req_mem, dtype=np.int64)
    N, D = fc.shape
    P = rc.size
    node = np.full(P, -1, np.int32)
    dev = np.full(P, -1, np.int8)
    # the concatenated table: every valid device of every table in the domain, node-major
    cols = [(n, d) for n in range(N) if table_in_domain(fc[n], fm[n], int(dv[n]), D) for d in range(int(dv[n]))]
    cn = np.array([c[0] for c in cols], np.int64)
    cd = np.array([c[1] for c in cols], np.int64)
    in_domain = (rc >= 0) & (rc <= CORE_MAX) & (rm >= 0) & (rm <= MEM_MAX)
    pending = np.arange(P) if N else np.arange(0)
    rounds = 0
    while pending.size:
        rounds += 1
        c, m = rc[pending][:, None], rm[pending][:, None]
        lc = fc[cn, cd][None, :] - c
        lm = fm[cn, cd][None, :] - m
        feasible = (c >= 0) & (m >= 0) & (lc >= 0) & (lm >= 0)
        # (lc, lm) as one ordered number; argmin takes the first column of a tie, i.e. the lowest (n, d)
        rank = np.where(feasible, lc * (MEM_MAX + 1) + lm, np.iinfo(np.int64).max)
        col = rank.argmin(axis=1) if cols else np.zeros(pending.size, np.int64)
        chose = feasible.any(axis=1) if cols else np.zeros(pending.size, bool)
        deferred = []
        for j in np.unique(col[chose]):
            rows = pending[chose & (col == j)]  # in request order
            n, d = cn[j], cd[j]
            ok = (np.cumsum(rc[rows]) <= fc[n, d]) & (np.cumsum(rm[rows]) <= fm[n, d])
            node[rows[ok]] = n
            dev[rows[ok]] = d
            fc[n, d] -= rc[rows[ok]].sum()
            fm[n, d] -= rm[rows[ok]].sum()
            deferred.extend(rows[~ok].tolist())
        pending = np.array(sorted(deferred), np.int64)
    if not in_domain.any():
        rounds = 0
    return node, dev, fc.astype(np.int32), fm.astype(np.int32), rounds


def place_torch(free_core, free_mem, d_valid, req_core, req_mem):
    """The same placement by a torch loop around egpu::bestfit_tables (the raw operator: no data checks), one
    host sync per round.  CUDA tensors in, (node, dev, free_core_out, free_mem_out, rounds) out, on the device."""
    import torch
    op = torch.ops.egpu.bestfit_tables
    N, D = free_core.shape
    P = req_core.shape[0]
    dv = d_valid
    fc, fm = free_core.clone(), free_mem.clone()
    node = torch.full((P,), -1, dtype=torch.int32, device=fc.device)
    dev = torch.full((P,), -1, dtype=torch.int8, device=fc.device)
    nodes = torch.arange(N, device=fc.device, dtype=torch.int64)[:, None]
    in_domain = bool(((req_core >= 0) & (req_core <= CORE_MAX) & (req_mem >= 0) & (req_mem <= MEM_MAX)).any()) if P else False
    pending = torch.arange(P, device=fc.device) if N else torch.arange(0, device=fc.device)
    rounds = 0
    while pending.numel():
        rounds += 1
        c, m = req_core[pending], req_mem[pending]
        idx, key = op(fc, fm, dv, c, m)  # [N, Pr]
        k = key.to(torch.int64)
        word = ((k >> 6) << 37) | (nodes << 6) | (k & 63)  # (lc, lm, n, d)
        word = torch.where(key == NO_KEY, torch.iinfo(torch.int64).max, word)
        best = word.min(dim=0).values
        chose = best != torch.iinfo(torch.int64).max
        rows, best = pending[chose], best[chose]
        flat = ((best >> 6) & 0x7FFFFFFF) * D + (best & 63)
        order = torch.sort(flat, stable=True).indices  # by device, request order kept within a device
        rows, flat = rows[order], flat[order]
        cc, cm = req_core[rows].to(torch.int64), req_mem[rows].to(torch.int64)
        start = torch.ones_like(flat, dtype=torch.bool)
        start[1:] = flat[1:] != flat[:-1]
        seg = torch.cumsum(start.to(torch.int64), 0) - 1
        csc, csm = torch.cumsum(cc, 0), torch.cumsum(cm, 0)
        first = torch.nonzero(start).flatten()
        pc = csc - (csc[first] - cc[first])[seg]  # segmented inclusive cumsum
        pm = csm - (csm[first] - cm[first])[seg]
        fits = (pc <= fc.view(-1)[flat].to(torch.int64)) & (pm <= fm.view(-1)[flat].to(torch.int64))
        node[rows[fits]] = (flat[fits] // D).to(torch.int32)
        dev[rows[fits]] = (flat[fits] % D).to(torch.int8)
        fc.view(-1).index_add_(0, flat[fits], -cc[fits].to(torch.int32))
        fm.view(-1).index_add_(0, flat[fits], -cm[fits].to(torch.int32))
        pending = torch.sort(rows[~fits]).values  # host sync: the next round's size
    return node, dev, fc, fm, rounds if in_domain else 0
