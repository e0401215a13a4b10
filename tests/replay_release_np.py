"""Plain-Python restatement of sequential mode with release events (DESIGN.md 2.6), independent of the kernels
and of oracle/.  Kinds 0 and 1 follow oracle/bestfit_np.replay; kind 3 gives back a placement made before the call.

TEST INFRASTRUCTURE ONLY: the product never imports this module."""
from __future__ import annotations

import numpy as np

CORE_MAX = 100
MEM_MAX = (1 << 18) - 1
EV_ALLOC, EV_FREE, EV_RELEASE = 0, 1, 3


def pack(core, mem):
    """EGPU_PACK_REQUEST as the int32 that a release event carries in b"""
    return np.int32((int(core) << 18) | int(mem))


def replay(free_core, free_mem, oversub, kind, a, b):
    """(idx int32[E], free_core', free_mem').  oversub (the sticky flags) is read, never changed.

    RELEASE(a = device, b = packed word) is accepted iff 0 <= a < D, 0 <= b < 2^25 with core <= 100, the device is
    unflagged unless the request is (0, 0), and the request fits the device's room: the domain bound minus the table
    minus what this call's live ALLOCs hold on it."""
    fc = [int(x) for x in free_core]
    fm = [int(x) for x in free_mem]
    ov = [int(x) != 0 for x in oversub]
    D = len(fc)
    assert all(0 <= c <= CORE_MAX for c in fc) and all(0 <= m <= MEM_MAX for m in fm) and len(ov) == D
    held_c, held_m = [0] * D, [0] * D  # what live ALLOCs of this call hold per device
    E = len(kind)
    out = np.full(E, -1, dtype=np.int32)
    live = {}
    for i in range(E):
        k, x, y = int(kind[i]), int(a[i]), int(b[i])
        if k == EV_ALLOC:
            if x < 0 or y < 0:
                continue
            fits = [(fc[d] - x, fm[d] - y, d) for d in range(D) if fc[d] >= x and fm[d] >= y]
            if fits:
                d = min(fits)[2]
                fc[d] -= x
                fm[d] -= y
                held_c[d] += x
                held_m[d] += y
                live[i] = d
                out[i] = d
        elif k == EV_FREE:
            if 0 <= x < i and x in live:
                d = live.pop(x)
                c, m = int(a[x]), int(b[x])
                fc[d] += c
                fm[d] += m
                held_c[d] -= c
                held_m[d] -= m
                out[i] = d
        elif k == EV_RELEASE:
            if not (0 <= x < D and 0 <= y < (1 << 25)):
                continue
            c, m = y >> 18, y & MEM_MAX
            if c > CORE_MAX or ((c > 0 or m > 0) and ov[x]):
                continue
            if fc[x] + held_c[x] + c > CORE_MAX or fm[x] + held_m[x] + m > MEM_MAX:
                continue
            fc[x] += c
            fm[x] += m
            out[i] = x
    return out, np.array(fc, dtype=np.int32), np.array(fm, dtype=np.int32)


def releases_of(kind, a, b, out_idx):
    """Release events (kind, a, b) that give back every placement a replay's result still holds, in event order:
    what a caller who keeps (device, request) of each placement hands back later."""
    live = {}
    for i in range(len(kind)):
        if kind[i] == EV_ALLOC and out_idx[i] >= 0:
            live[i] = (int(out_idx[i]), int(a[i]), int(b[i]))
        elif kind[i] == EV_FREE and out_idx[i] >= 0:
            live.pop(int(a[i]))
    rows = [live[t] for t in sorted(live)]
    return (np.full(len(rows), EV_RELEASE, np.int32), np.array([d for d, _, _ in rows], np.int32),
            np.array([pack(c, m) for _, c, m in rows], np.int32))
