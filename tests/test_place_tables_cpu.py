"""egpu::place_tables without a GPU (DESIGN.md §2.11).

  1. the numpy restatement (tests/place_tables_np.py) against the hand-derived answers of
     tests/golden/place_tables_kat.json;
  2. the restatement against oracle/bestfit_np.rounds run on the concatenated table (every valid device of every
     table in the domain, node-major), for hundreds of seeded cases with at most 64 devices in all: the same
     placements under the map (n, d) -> offset[n] + d, the same tables and the same number of rounds;
  3. the fake implementation's shapes and dtypes, which torch.compile and CUDA-graph tracing see;
  4. the refusals of bestfit_tables, with "place_tables" in the messages, alike through the fake, the compiled
     operator (its CPU registration) and the Python checks.
"""
import json
import os
import sys

import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import place_tables_np as ref  # noqa: E402
import test_tables_cpu as tc  # noqa: E402  (argument builder and the refusal cases of bestfit_tables)

from oracle import bestfit_np  # noqa: E402

MEM_MAX = (1 << 18) - 1
KAT = json.load(open(os.path.join(HERE, "golden", "place_tables_kat.json")))["cases"]


@pytest.fixture(scope="module")
def tables():
    from elastic_gpu_agent_b200 import tables as t
    t.load()
    return t


# ---- 1. known answers ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", range(len(KAT)))
def test_restatement_matches_the_known_answers(case):
    c = KAT[case]
    node, dev, fco, fmo, rounds = ref.place(np.array(c["free_core"]), np.array(c["free_mem"]), c["d_valid"],
                                            c["req_core"], c["req_mem"])
    assert node.tolist() == c["node"] and dev.tolist() == c["dev"], c["name"]
    assert fco.tolist() == c["free_core_out"] and fmo.tolist() == c["free_mem_out"], c["name"]
    assert rounds == c["rounds"], c["name"]


def test_known_answers_cover_the_issue_cases():
    assert len(KAT) == 5 and {c["rounds"] for c in KAT} == {1, 2, 3}


# ---- 2. against the single-table rounds oracle on the concatenation --------------------------------------------
def random_case(g, contended):
    """A few tables with mixed d_valid, at most 64 valid devices in all, out-of-domain padding past d_valid and now
    and then a table outside the domain; requests drawn to collide (contended) or spread."""
    N = int(g.integers(1, 9))
    D = int(g.integers(1, 65 // N + 1))
    dv = g.integers(1, D + 1, N).astype(np.int32)
    fc = g.choice([0, 10, 25, 50, 75, 100], (N, D)).astype(np.int32) if contended else g.integers(0, 101, (N, D)).astype(np.int32)
    fm = g.choice([0, 1024, 4096, 40_000, 81_559], (N, D)).astype(np.int32) if contended else \
        g.integers(0, MEM_MAX + 1, (N, D)).astype(np.int32)
    past = np.arange(D)[None, :] >= dv[:, None]
    fc[past] = g.choice([-3, 101, 500], int(past.sum()))
    fm[past] = g.choice([-1, MEM_MAX + 1], int(past.sum()))
    if g.random() < 0.2:
        bad = int(g.integers(0, N))
        if g.random() < 0.5:
            dv[bad] = g.choice([0, D + 1, -2])
        else:
            fc[bad, 0] = 101
            dv[bad] = max(int(dv[bad]), 1)
    P = int(g.integers(0, 120))
    if contended:
        rc = g.choice([5, 10, 25, 50], P).astype(np.int32)
        rm = g.choice([0, 512, 1024, 4096], P).astype(np.int32)
    else:
        rc = g.integers(0, 101, P).astype(np.int32)
        rm = g.integers(0, 90_000, P).astype(np.int32)
    odd = g.random(P) < 0.05
    rc[odd] = g.choice([-1, 101, 1 << 20], int(odd.sum()))
    return fc, fm, dv, rc, rm


@pytest.mark.parametrize("seed", range(300))
def test_restatement_equals_rounds_on_the_concatenated_table(seed):
    g = np.random.default_rng(9000 + seed)
    fc, fm, dv, rc, rm = random_case(g, contended=seed % 3 != 0)
    N, D = fc.shape
    node, dev, fco, fmo, rounds = ref.place(fc, fm, dv, rc, rm)
    live = [n for n in range(N) if ref.table_in_domain(fc[n], fm[n], int(dv[n]), D)]
    offset = {}
    cat_c, cat_m = [], []
    for n in live:
        offset[n] = len(cat_c)
        cat_c += fc[n, :dv[n]].tolist()
        cat_m += fm[n, :dv[n]].tolist()
    assert len(cat_c) <= 64
    # tables outside the domain, and every column past d_valid, come back unchanged
    for n in range(N):
        keep = slice(None) if n not in offset else slice(int(dv[n]), None)
        np.testing.assert_array_equal(fco[n, keep], fc[n, keep])
        np.testing.assert_array_equal(fmo[n, keep], fm[n, keep])
    placed = node >= 0
    if not cat_c:
        assert not placed.any()
        return
    o_idx, _, _, o_fc, o_fm, o_rounds, o_left = bestfit_np.rounds(np.array(cat_c, np.int32), np.array(cat_m, np.int32), rc, rm)
    assert o_left == 0
    flat = np.array([offset[int(n)] + int(d) if n >= 0 else -1 for n, d in zip(node, dev)], np.int64)
    np.testing.assert_array_equal(flat, o_idx)
    for n in live:
        o = offset[n]
        np.testing.assert_array_equal(fco[n, :dv[n]], o_fc[o:o + dv[n]])
        np.testing.assert_array_equal(fmo[n, :dv[n]], o_fm[o:o + dv[n]])
    in_domain = ((rc >= 0) & (rc <= 100) & (rm >= 0) & (rm <= MEM_MAX)).any()
    assert rounds == (o_rounds if in_domain else 0)


def test_seeds_reach_several_rounds():
    most = 0
    for seed in range(300):
        g = np.random.default_rng(9000 + seed)
        most = max(most, ref.place(*random_case(g, contended=seed % 3 != 0))[4])
    assert most >= 5


# ---- 3. the fake ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,D,P", [(6, 8, 12), (5000, 8, 1024), (512, 64, 8192), (0, 3, 7), (4, 1, 0)])
def test_fake_gives_shapes_and_dtypes(N, D, P, tables):
    with FakeTensorMode():
        node, dev, fco, fmo, info = torch.ops.egpu.place_tables(*tc.args(N, D, P, device="cuda"))
    assert node.shape == dev.shape == (P,) and fco.shape == fmo.shape == (N, D) and info.shape == (2,)
    assert node.dtype == fco.dtype == fmo.dtype == info.dtype == torch.int32 and dev.dtype == torch.int8
    assert all(t.device.type == "cuda" for t in (node, dev, fco, fmo, info))


# ---- 4. refusals ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", range(13))
def test_fake_operator_and_python_checks_refuse_alike(case, tables):
    exc, msg, kw = tc.refusals("cpu")[case]
    msg = "place_tables: .*" + msg
    with pytest.raises(exc, match=msg):
        torch.ops.egpu.place_tables(*tc.args(**kw))  # the compiled operator, CPU tensors: refused before the device check
    with pytest.raises(exc, match=msg):
        tables.check_args(*tc.args(**kw), op="place_tables")
    with pytest.raises(exc, match=msg):
        tables.place_tables(*tc.args(**kw))
    with FakeTensorMode():
        exc_f, msg_f, kw_f = tc.refusals("cuda")[case]
        with pytest.raises(exc_f, match="place_tables: .*" + msg_f):
            torch.ops.egpu.place_tables(*tc.args(device="cuda", **kw_f))


def test_tensors_off_the_gpu_are_refused(tables):
    for call in (torch.ops.egpu.place_tables, tables.place_tables):
        with pytest.raises(RuntimeError, match="place_tables: every tensor must be on one CUDA device"):
            call(*tc.args())
    with FakeTensorMode():
        fc, fm, dv, rc, rm = tc.args(device="cuda")
        with pytest.raises(RuntimeError, match="place_tables: every tensor must be on one CUDA device"):
            torch.ops.egpu.place_tables(fc, fm, dv, torch.zeros(12, dtype=torch.int32), rm)


def test_table_checks_name_the_operator(tables):
    fc, fm, dv, _, _ = tc.args(N=4, D=8)
    f2 = fc.clone()
    f2[3, 0] = 101
    with pytest.raises(ValueError, match="place_tables: 1 table\\(s\\) outside the domain"):
        tables.check_tables(f2, fm, dv, op="place_tables")
    d2 = dv.clone()
    d2[2] = 0
    with pytest.raises(ValueError, match="place_tables: 1 table\\(s\\) with d_valid outside \\[1, 8\\]"):
        tables.check_tables(fc, fm, d2, op="place_tables")
