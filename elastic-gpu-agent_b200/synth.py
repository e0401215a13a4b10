"""Deterministic synthetic workloads for the best-fit path (DESIGN.md §6).

A counter-based generator so that numpy (here), C and the on-device CUDA
generator (csrc/egpu_alloc.cu: synth_requests_kernel) produce identical data
without files:

    z  = seed*0x9E3779B97F4A7C15 + stream*0xD1B54A32D192ED03 + i      (mod 2^64)
    z  = splitmix64_finalise(z)
    v  = lo + (((z >> 32) * (hi - lo + 1)) >> 32)

Units follow the reference: core in percent of one card, 100 per card
(pkg/common/const.go:4); memory in MiB (pkg/plugins/gpushare.go:161).  The synthetic
node's cards hold 183359 MiB each, more than an H100 80GB's 81559: the workloads, the
golden vectors and bench results stay the same from build to build, and the ID formats
are exercised past the size of the card that runs them.
"""
from __future__ import annotations

import numpy as np

CAP_CORE = 100
CAP_MEM = 183359  # MiB per card of the synthetic node

_G1 = np.uint64(0x9E3779B97F4A7C15)
_G2 = np.uint64(0xD1B54A32D192ED03)
_M1 = np.uint64(0xBF58476D1CE4E5B9)
_M2 = np.uint64(0x94D049BB133111EB)

STREAM_TABLE_CORE = 0
STREAM_TABLE_MEM = 1
STREAM_REQ_CORE = 2
STREAM_REQ_MEM = 3
STREAM_EV_KIND = 4
STREAM_EV_VICTIM = 5

CFG2_CORES = np.array([5, 10, 20, 25, 50, 100], dtype=np.int32)
CFG2_MEMS = np.array([256, 512, 1024, 2048, 4096, 8192, 16384], dtype=np.int32)


def mix64(seed: int, stream: int, i) -> np.ndarray:
    """splitmix64 finaliser of the (seed, stream, counter) triple; uint64."""
    with np.errstate(over="ignore"):
        i = np.asarray(i, dtype=np.uint64)
        z = np.uint64(seed) * _G1 + np.uint64(stream) * _G2 + i
        z = (z ^ (z >> np.uint64(30))) * _M1
        z = (z ^ (z >> np.uint64(27))) * _M2
        z = z ^ (z >> np.uint64(31))
    return z


def uniform(seed: int, stream: int, i, lo: int, hi: int) -> np.ndarray:
    """Integers in [lo, hi] (inclusive), int32."""
    z = mix64(seed, stream, i)
    n = np.uint64(hi - lo + 1)
    v = ((z >> np.uint64(32)) * n) >> np.uint64(32)
    return (v.astype(np.int64) + lo).astype(np.int32)


def table_full(D: int = 8):
    return (np.full(D, CAP_CORE, dtype=np.int32), np.full(D, CAP_MEM, dtype=np.int32))


def table_fragmented(seed: int, D: int = 8, mem_cap: int = CAP_MEM):
    d = np.arange(D, dtype=np.uint64)
    return (uniform(seed, STREAM_TABLE_CORE, d, 0, CAP_CORE),
            uniform(seed, STREAM_TABLE_MEM, d, 0, mem_cap))


def requests(dist: int, seed: int, R: int, first_row: int = 0):
    """Request rows [first_row, first_row+R) of distribution `dist`.

    dist 2 (cfg2): core from {5,10,20,25,50,100}, mem from {256..16384} powers of 2.
    dist 3 (cfg3): core in [1,100], mem in [1,65536]; rows with r%16==15 are
                   forced infeasible, alternating core=101 / mem=CAP_MEM+1.
    dist 4 (cfg4): as dist 3 with mem in [1,24576] (64 slice rows of <= CAP_MEM/8).
    """
    r = np.arange(first_row, first_row + R, dtype=np.uint64)
    if dist == 2:
        core = CFG2_CORES[uniform(seed, STREAM_REQ_CORE, r, 0, 5)]
        mem = CFG2_MEMS[uniform(seed, STREAM_REQ_MEM, r, 0, 6)]
        return core.astype(np.int32), mem.astype(np.int32)
    if dist in (3, 4):
        mem_hi = 65536 if dist == 3 else 24576
        core = uniform(seed, STREAM_REQ_CORE, r, 1, 100)
        mem = uniform(seed, STREAM_REQ_MEM, r, 1, mem_hi)
        forced = (r % np.uint64(16)) == np.uint64(15)
        alt = ((r // np.uint64(16)) % np.uint64(2)) == np.uint64(0)
        core = np.where(forced & alt, CAP_CORE + 1, core).astype(np.int32)
        mem = np.where(forced & ~alt, CAP_MEM + 1, mem).astype(np.int32)
        return core, mem
    raise ValueError(f"unknown request distribution {dist}")


def churn_events(seed: int, E: int):
    """cfg5: E interleaved Allocate/Free events.

    Event i is FREE with probability 0.5 when any ALLOC event is still
    un-freed, and always when 40 are (victim = position `x % live` of the list
    of un-freed ALLOC events, swap-removed), else ALLOC(core in [1,50], mem in
    [1,32768]).  The un-freed count random-walks over 0..40, so the node swings
    between empty and oversubscribed and both outcomes are exercised.
    The list tracks issued events, not outcomes, so the stream does not depend
    on the algorithm under test.  Returns (kind, a, b) int32 arrays.
    """
    i = np.arange(E, dtype=np.uint64)
    coin = uniform(seed, STREAM_EV_KIND, i, 0, 9999)
    victim = mix64(seed, STREAM_EV_VICTIM, i)
    core = uniform(seed, STREAM_REQ_CORE, i, 1, 50)
    mem = uniform(seed, STREAM_REQ_MEM, i, 1, 32768)
    kind = np.zeros(E, dtype=np.int32)
    a = np.zeros(E, dtype=np.int32)
    b = np.zeros(E, dtype=np.int32)
    live: list[int] = []
    for k in range(E):
        if live and (coin[k] < 5000 or len(live) >= 40):
            p = int(victim[k] % np.uint64(len(live)))
            kind[k] = 1
            a[k] = live[p]
            live[p] = live[-1]
            live.pop()
        else:
            a[k] = core[k]
            b[k] = mem[k]
            live.append(k)
    return kind, a, b


# Named workloads (BASELINE.json configs -> concrete inputs)
def workload(name: str):
    """Returns dict(D, free_core, free_mem, dist, seed, R, mode)."""
    if name == "cfg1":
        fc, fm = table_full(8)
        return dict(D=8, free_core=fc, free_mem=fm, dist=None, seed=1, R=4, mode="sequential")
    if name == "cfg2":
        fc, fm = table_full(8)
        return dict(D=8, free_core=fc, free_mem=fm, dist=2, seed=2, R=1000, mode="snapshot")
    if name == "cfg3":
        fc, fm = table_fragmented(3, 8)
        return dict(D=8, free_core=fc, free_mem=fm, dist=3, seed=3, R=100_000, mode="snapshot")
    if name == "cfg3_1m":
        fc, fm = table_fragmented(3, 8)
        return dict(D=8, free_core=fc, free_mem=fm, dist=3, seed=6, R=1_000_000, mode="snapshot")
    if name == "cfg3_64mi":
        fc, fm = table_fragmented(3, 8)
        return dict(D=8, free_core=fc, free_mem=fm, dist=3, seed=7, R=64 << 20, mode="snapshot")
    if name == "cfg4":
        fc, fm = table_fragmented(4, 64, CAP_MEM // 8)
        return dict(D=64, free_core=fc, free_mem=fm, dist=4, seed=4, R=1_000_000, mode="snapshot")
    if name == "cfg5":
        fc, fm = table_full(8)
        return dict(D=8, free_core=fc, free_mem=fm, dist=None, seed=5, R=100_000, mode="sequential")
    raise ValueError(f"unknown workload {name}")
