"""Release events in sequential replay (EGPU_EV_RELEASE, DESIGN.md 2.6), without a GPU: the restatement of
tests/replay_release_np.py against hand-derived answers, against oracle/bestfit_np on streams without release
events, and the header and binding text."""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import release_np  # noqa: E402
import replay_release_np as rr  # noqa: E402
from replay_release_np import pack  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEM_MAX = rr.MEM_MAX
A, F, REL = 0, 1, 3

FC, FM = [50, 100], [1000, MEM_MAX]

# (name, table (fc, fm, oversub), events [(kind, a, b)], out_idx, (fc', fm'))
CASES = [
    ("accepted", (FC, FM, [0, 0]), [(REL, 0, pack(30, 500))], [0], ([80, 100], [1500, MEM_MAX])),
    ("accepted up to the domain", (FC, FM, [0, 0]), [(REL, 0, pack(50, MEM_MAX - 1000))], [0], ([100, 100], [MEM_MAX, MEM_MAX])),
    ("flagged device", (FC, FM, [1, 0]), [(REL, 0, pack(10, 10)), (REL, 0, pack(0, 1)), (REL, 1, pack(0, 0))], [-1, -1, 1],
     (FC, FM)),
    ("(0, 0) on a flagged device", (FC, FM, [1, 1]), [(REL, 0, pack(0, 0)), (REL, 1, 0)], [0, 1], (FC, FM)),
    ("core past the domain", (FC, FM, [0, 0]), [(REL, 0, pack(51, 0)), (REL, 1, pack(1, 0))], [-1, -1], (FC, FM)),
    ("memory past the domain", (FC, FM, [0, 0]), [(REL, 0, pack(0, MEM_MAX - 999)), (REL, 1, pack(0, 1))], [-1, -1], (FC, FM)),
    ("bad device", (FC, FM, [0, 0]), [(REL, -1, pack(1, 1)), (REL, 2, pack(1, 1)), (REL, 64, pack(1, 1)),
                                      (REL, -(2**31), pack(1, 1))], [-1] * 4, (FC, FM)),
    ("word >= 2^25 or negative", (FC, FM, [0, 0]), [(REL, 0, 1 << 25), (REL, 0, (1 << 25) + 7), (REL, 0, -1),
                                                    (REL, 0, -(2**31)), (REL, 0, 2**31 - 1)], [-1] * 5, (FC, FM)),
    ("core 101..127", ([0, 0], [0, 0], [0, 0]), [(REL, 0, 101 << 18), (REL, 0, (127 << 18) | 5), (REL, 1, (110 << 18) | MEM_MAX),
                                                 (REL, 1, pack(100, 0))], [-1, -1, -1, 1], ([0, 100], [0, 0])),
    ("FREE of a release event", (FC, FM, [0, 0]), [(REL, 0, pack(10, 0)), (F, 0, 0)], [0, -1], ([60, 100], FM)),
    ("kinds 2 and 7 stay no-ops", (FC, FM, [0, 0]), [(2, 0, pack(10, 0)), (7, 0, pack(10, 0)), (F, 1, 0)], [-1] * 3, (FC, FM)),
    # the room counts this call's live ALLOCs: 20 free + 30 live + 60 > 100, then 20 + 30 + 50 = 100 fits
    ("live allocations count against the room", ([50], [1000], [0]),
     [(A, 30, 0), (REL, 0, pack(60, 0)), (REL, 0, pack(50, 0)), (F, 0, 0)], [0, -1, 0, 0], ([100], [1000])),
    ("a freed allocation no longer counts", ([50], [1000], [0]),
     [(A, 30, 0), (F, 0, 0), (REL, 0, pack(50, 0))], [0, 0, 0], ([100], [1000])),
    # per event: the first two fit, the third would pass 100; the same rows as one batch release are refused
    ("a prefix is accepted", ([90], [0], [0]), [(REL, 0, pack(5, 0))] * 3, [0, 0, -1], ([100], [0])),
    ("released capacity is allocatable", ([0, 40], [0, 10], [0, 0]), [(A, 10, 10), (REL, 0, pack(60, 100)), (A, 10, 10)],
     [1, 0, 0], ([50, 30], [90, 0])),
]


def run(table, events):
    fc, fm, ov = table
    kind, a, b = (np.array([e[i] for e in events], np.int64).astype(np.int32) for i in range(3))
    return rr.replay(fc, fm, ov, kind, a, b)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_restatement_hand_derived(case):
    _, table, events, want_idx, (want_fc, want_fm) = case
    idx, fc, fm = run(table, events)
    assert idx.tolist() == want_idx
    assert fc.tolist() == list(want_fc) and fm.tolist() == list(want_fm)


def test_a_prefix_where_the_batch_is_refused():
    """the rows of "a prefix is accepted" as one EGPU_F_RELEASE batch: refused as a whole"""
    _, _, ok = release_np.release([90], [0], [0], [5, 5, 5], [0, 0, 0], [0, 0, 0])
    assert not ok
    _, tab, ok = release_np.release([90], [0], [0], [5, 5], [0, 0], [0, 0])
    assert ok and tab[0] == 100


@pytest.mark.parametrize("seed", range(6))
def test_restatement_is_the_oracle_without_release_events(seed):
    """kinds 0, 1, 2 and 7 only: the restatement is oracle/bestfit_np.replay"""
    from oracle import bestfit_np
    rng = np.random.default_rng(seed)
    D, E = int(rng.integers(1, 12)), 400
    fc = rng.integers(0, 101, D).astype(np.int32)
    fm = rng.integers(0, MEM_MAX + 1, D).astype(np.int32)
    kind = rng.choice([0, 0, 1, 1, 2, 7], E).astype(np.int32)
    a = np.where(kind == 0, rng.integers(-2, 60, E), rng.integers(-3, E + 3, E)).astype(np.int32)
    b = rng.integers(-2, 40_000, E).astype(np.int32)
    got = rr.replay(fc, fm, np.zeros(D), kind, a, b)
    want = bestfit_np.replay(fc, fm, kind, a, b)
    assert all(np.array_equal(x, y) for x, y in zip(got, want))


@pytest.mark.parametrize("seed", range(4))
def test_restatement_round_trip(seed):
    """every placement a call still holds, handed back as release events in a second call in any order, restores
    the table"""
    rng = np.random.default_rng(50 + seed)
    D, E = 9, 300
    fc = rng.integers(0, 101, D).astype(np.int32)
    fm = rng.integers(0, 50_000, D).astype(np.int32)
    kind = rng.choice([0, 0, 0, 1], E).astype(np.int32)
    a = np.where(kind == 0, rng.integers(0, 30, E), rng.integers(0, E, E)).astype(np.int32)
    b = rng.integers(0, 5000, E).astype(np.int32)
    out, fc1, fm1 = rr.replay(fc, fm, np.zeros(D), kind, a, b)
    rk, ra, rb = rr.releases_of(kind, a, b, out)
    assert rk.size > 0
    perm = rng.permutation(rk.size)
    back, fc2, fm2 = rr.replay(fc1, fm1, np.zeros(D), rk[perm], ra[perm], rb[perm])
    assert np.array_equal(back, ra[perm])
    assert np.array_equal(fc2, fc) and np.array_equal(fm2, fm)


def test_header_documents_the_release_kind():
    text = open(os.path.join(ROOT, "include", "egpu_alloc.h")).read()
    kinds = dict(re.findall(r"#define (EGPU_EV_\w+)\s+(\d+)", text))
    assert kinds == {"EGPU_EV_ALLOC": "0", "EGPU_EV_FREE": "1", "EGPU_EV_RELEASE": "3"}  # 2 and 7 stay unassigned
    block = text[text.index("/* Applies E events in order"):text.index("int egpu_replay(")]
    for phrase in ("EGPU_EV_RELEASE", "EGPU_PACK_REQUEST(core, mem) read as int32", "0 <= a[i] < D",
                   "0 <= b[i] < 2^25", "core <= EGPU_CORE_MAX", "EGPU_REL_FLAGGED", "EGPU_REL_EXCEEDS", "(0, 0)",
                   "Every other kind is a no-op", "stays 1011"):
        assert phrase in block, phrase
    from elastic_gpu_agent_b200 import _lib
    assert (_lib.EV_ALLOC, _lib.EV_FREE, _lib.EV_RELEASE) == (0, 1, 3)
