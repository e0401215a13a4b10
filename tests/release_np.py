"""numpy restatement of the release rule (DESIGN.md 2.8), independent of tests/release_oracle.c.

TEST INFRASTRUCTURE ONLY: the product never imports this module."""
from __future__ import annotations

import numpy as np

CORE_MAX = 100
MEM_MAX = (1 << 18) - 1
REL_FLAGGED = 1
REL_EXCEEDS = 2


def release(free_core, free_mem, oversub, core, mem, idx):
    """(u int64[2D], table_out int32[3D], accepted).  table_out = free + u when accepted, free when refused,
    then the per-device reason words."""
    fc = np.asarray(free_core, dtype=np.int64)
    fm = np.asarray(free_mem, dtype=np.int64)
    ov = np.asarray(oversub, dtype=np.int64)
    c = np.asarray(core, dtype=np.int64)
    m = np.asarray(mem, dtype=np.int64)
    i = np.asarray(idx, dtype=np.int64)
    D = fc.size
    holds = (i >= 0) & (i < D) & (c >= 0) & (c <= CORE_MAX) & (m >= 0) & (m <= MEM_MAX)
    uc = np.zeros(D, dtype=np.int64)
    um = np.zeros(D, dtype=np.int64)
    np.add.at(uc, i[holds], c[holds])
    np.add.at(um, i[holds], m[holds])
    touched = (uc > 0) | (um > 0)
    reason = np.where(touched & (ov != 0), REL_FLAGGED,
                      np.where(touched & ((fc + uc > CORE_MAX) | (fm + um > MEM_MAX)), REL_EXCEEDS, 0))
    accepted = not reason.any()
    nc, nm = (fc + uc, fm + um) if accepted else (fc, fm)
    return np.concatenate([uc, um]).astype(np.int64), np.concatenate([nc, nm, reason]).astype(np.int32), accepted


def unpack(words):
    """Packed words -> the (core, mem) they stand for; a word >= 2^25 becomes core 127 (holds nothing)."""
    w = np.asarray(words, dtype=np.uint32).astype(np.int64)
    bad = w >= (1 << 25)
    return np.where(bad, 127, (w >> 18) & 127).astype(np.int32), np.where(bad, 0, w & MEM_MAX).astype(np.int32)
