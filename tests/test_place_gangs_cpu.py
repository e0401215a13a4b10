"""egpu::place_gangs without a GPU (DESIGN.md §2.13).

  1. the numpy restatement (tests/place_gangs_np.py) against the hand-derived answers of
     tests/golden/place_gangs_kat.json;
  2. on 300 seeded cases, the restatement's placement, placed counts and tables equal the literal loop of §2.13 (one
     place_pods_np.place per gang, kept or thrown away), and its round count is at most the loop's;
  3. one gang whose pods are all placed: exactly place_pods_np.place, rounds included;
  4. the fake implementation's shapes and dtypes;
  5. the refusals: place_pods' with "place_gangs" in the messages, then gang_offsets' and gang_min's, alike through
     the fake, the compiled operator (its CPU registration) and the Python checks; bad index values refused eagerly
     and by the restatement.
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
import place_gangs_np as ref  # noqa: E402
import place_pods_np  # noqa: E402
import test_place_pods_cpu as ppc  # noqa: E402  (argument builder and the offsets refusals of place_pods)
import test_tables_cpu as tc  # noqa: E402  (the refusal cases of bestfit_tables)

KAT = json.load(open(os.path.join(HERE, "golden", "place_gangs_kat.json")))["cases"]
KEYS = ("free_core", "free_mem", "d_valid", "req_core", "req_mem", "pod_offsets", "gang_offsets", "gang_min")


@pytest.fixture(scope="module")
def tables():
    from elastic_gpu_agent_b200 import tables as t
    t.load()
    return t


# ---- 1. known answers ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", range(len(KAT)))
def test_restatement_matches_the_known_answers(case):
    c = KAT[case]
    node, dev, placed, fco, fmo, info = ref.place(*[np.array(c[k]) for k in KEYS])
    assert node.tolist() == c["node"] and dev.tolist() == c["dev"] and placed.tolist() == c["placed"], c["name"]
    assert fco.tolist() == c["free_core_out"] and fmo.tolist() == c["free_mem_out"], c["name"]
    assert info == [c["rounds"], 0, 0], c["name"]


def test_known_answers_cover_the_listed_cases():
    assert len(KAT) >= 9 and all(c["why"] for c in KAT)
    assert any(len(c["gang_min"]) == 1 for c in KAT)  # J = 1
    assert any(0 in c["placed"] and c["placed"][-1] > 0 for c in KAT)  # given back, then a later gang placed
    assert any(min(c["gang_min"]) < max(np.diff(c["gang_offsets"])) for c in KAT)  # min < size
    # a gang that stops early: fewer rounds than the literal loop
    assert any(ref.loop(*[np.array(c[k]) for k in KEYS])[5][0] > c["rounds"] for c in KAT)


# ---- 2. the literal loop over place_pods -------------------------------------------------------------------------
def random_gangs(g, G, hi=6):
    """gang_offsets and gang_min for G pods in gangs of 1 to `hi` pods: a third all or nothing, the rest any min."""
    sizes, total = [], 0
    while total < G:
        s = min(int(g.integers(1, hi + 1)), G - total)
        sizes.append(s)
        total += s
    sizes = np.array(sizes, np.int64)
    gmin = np.where(g.random(sizes.size) < 0.33, sizes, g.integers(1, sizes + 1))
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32), gmin.astype(np.int32)


def random_case(g):
    N, D = int(g.integers(1, 7)), int(g.integers(1, 9))
    contended = g.random() < 0.7
    fc = g.choice([0, 10, 25, 50, 75, 100], (N, D)) if contended else g.integers(0, 101, (N, D))
    fm = g.choice([0, 1024, 4096, 40_000], (N, D)) if contended else g.integers(0, 81_560, (N, D))
    dv = g.integers(1, D + 1, N)
    past = np.arange(D)[None, :] >= dv[:, None]
    fc[past] = g.choice([-3, 101], int(past.sum()))
    if g.random() < 0.15:
        fc[int(g.integers(N)), 0] = 120  # a table outside the domain
    off = ppc.random_pods(g, int(g.integers(1, 25)), hi=4)
    P = int(off[-1])
    rc = g.choice([0, 5, 10, 25, 50, 100], P)
    rm = g.choice([0, 512, 1024, 4096], P)
    bad = g.random(P) < 0.04
    rc[bad] = g.choice([-1, 101], int(bad.sum()))
    goff, gmin = random_gangs(g, off.size - 1)
    return [x.astype(np.int32) for x in (fc, fm, dv, rc, rm)] + [off, goff, gmin]


@pytest.mark.parametrize("seed", range(300))
def test_restatement_equals_the_loop_over_place_pods(seed):
    a = random_case(np.random.default_rng(7100 + seed))
    got = ref.place(*a)
    exp = ref.loop(*a)
    for x, y in zip(got[:5], exp[:5]):
        np.testing.assert_array_equal(x, y)
    assert got[5][1:] == [0, 0] and got[5][0] <= exp[5][0]
    placed, gmin, size = got[2], a[7], np.diff(a[6])
    assert ((placed == 0) | ((placed >= gmin) & (placed <= size))).all()


def test_seeded_cases_roll_back_and_stop_early():
    """The seeded cases above exercise what they are there for: gangs given back, and rounds saved by the early stop."""
    rolled = early = 0
    for seed in range(300):
        a = random_case(np.random.default_rng(7100 + seed))
        got, exp = ref.place(*a), ref.loop(*a)
        rolled += int(((got[2] == 0) & (np.diff(a[6]) > 0)).sum())
        early += got[5][0] < exp[5][0]
    assert rolled >= 100 and early >= 30, (rolled, early)


@pytest.mark.parametrize("seed", range(60))
def test_one_gang_with_every_pod_placed_is_place_pods(seed):
    g = np.random.default_rng(8300 + seed)
    N, D = int(g.integers(1, 8)), int(g.integers(1, 17))
    fc = g.integers(50, 101, (N, D)).astype(np.int32)
    fm = g.integers(40_000, 81_560, (N, D)).astype(np.int32)
    dv = g.integers(1, D + 1, N).astype(np.int32)
    off = ppc.random_pods(g, int(g.integers(1, 10)), hi=3)
    P, G = int(off[-1]), off.size - 1
    rc = g.choice([0, 5, 10, 25, 50], P).astype(np.int32)
    rm = g.choice([0, 512, 1024], P).astype(np.int32)
    exp = place_pods_np.place(fc, fm, dv, rc, rm, off)
    got = ref.place(fc, fm, dv, rc, rm, off, [0, G], [int(g.integers(1, G + 1))])
    if (exp[0] < 0).any():
        return  # not every pod placed: the gang may be given back
    for x, y in zip(got[:2] + got[3:5], exp[:4]):
        np.testing.assert_array_equal(x, y)
    assert got[2].tolist() == [G] and got[5] == exp[4]


# ---- 4. the fake ----------------------------------------------------------------------------------------------
def gang_args(N=6, D=8, P=12, G=4, J=2, device="cpu", **kw):
    fc, fm, dv, rc, rm, off = ppc.pod_args(N, D, P, G, device=device)
    z = dict(dtype=torch.int32, device=device)
    a = dict(fc=fc, fm=fm, dv=dv, rc=rc, rm=rm, off=off,
             goff=torch.arange(J + 1, **z) * (G // max(J, 1)), gmin=torch.ones(J, **z))
    a.update(kw)
    return a["fc"], a["fm"], a["dv"], a["rc"], a["rm"], a["off"], a["goff"], a["gmin"]


@pytest.mark.parametrize("N,D,P,G,J", [(6, 8, 12, 4, 2), (5000, 8, 2560, 1024, 128), (512, 64, 8192, 4096, 256),
                                       (0, 3, 7, 7, 7), (4, 1, 0, 0, 0)])
def test_fake_gives_shapes_and_dtypes(N, D, P, G, J, tables):
    with FakeTensorMode():
        node, dev, placed, fco, fmo, info = torch.ops.egpu.place_gangs(*gang_args(N, D, P, G, J, device="cuda"))
    assert node.shape == (G,) and dev.shape == (P,) and placed.shape == (J,) and fco.shape == fmo.shape == (N, D)
    assert info.shape == (3,) and dev.dtype == torch.int8
    assert node.dtype == placed.dtype == fco.dtype == fmo.dtype == info.dtype == torch.int32
    assert all(t.device.type == "cuda" for t in (node, dev, placed, fco, fmo, info))


# ---- 5. refusals ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", range(13))
def test_table_refusals_alike(case, tables):
    exc, msg, kw = tc.refusals("cpu")[case]
    msg = "place_gangs: .*" + msg
    rest = gang_args()[5:]
    with pytest.raises(exc, match=msg):
        torch.ops.egpu.place_gangs(*tc.args(**kw), *rest)  # the compiled operator, CPU tensors
    with pytest.raises(exc, match=msg):
        tables.check_args(*tc.args(**kw), op="place_gangs")
    with pytest.raises(exc, match=msg):
        tables.place_gangs(*tc.args(**kw), *rest)
    with FakeTensorMode():
        exc_f, msg_f, kw_f = tc.refusals("cuda")[case]
        with pytest.raises(exc_f, match="place_gangs: .*" + msg_f):
            torch.ops.egpu.place_gangs(*tc.args(device="cuda", **kw_f), *gang_args(device="cuda")[5:])


def gang_refusals(device):
    z = dict(dtype=torch.int32, device=device)
    return [(exc, msg, {"off": kw["off"]}) for exc, msg, kw in ppc.offsets_refusals(device)] + [
        (RuntimeError, "gang_offsets must be int32", dict(goff=torch.tensor([0, 2, 4], dtype=torch.int64, device=device))),
        (RuntimeError, "gang_min must be int32", dict(gmin=torch.ones(2, dtype=torch.float32, device=device))),
        (RuntimeError, "gang_offsets must be contiguous", dict(goff=torch.arange(6, **z)[::2])),
        (RuntimeError, "gang_min must be contiguous", dict(gmin=torch.ones(4, **z)[::2])),
        (ValueError, "gang_offsets must be \\[J \\+ 1\\]", dict(goff=torch.zeros(0, **z))),
        (ValueError, "gang_offsets must be \\[J \\+ 1\\]", dict(goff=torch.zeros((3, 1), **z))),
        (ValueError, "gang_min must be \\[J\\] = \\[2\\], got \\(3,\\)", dict(gmin=torch.ones(3, **z))),
        (ValueError, "gang_min must be \\[J\\] = \\[2\\], got \\(2, 1\\)", dict(gmin=torch.ones((2, 1), **z))),
    ]


@pytest.mark.parametrize("case", range(12))
def test_index_refusals_alike(case, tables):
    """The index tensors are checked after the other five tensors' device, so with CPU tensors the compiled operator
    and the Python interface both refuse on the device; with CUDA tensors (fake here, real in the GPU tests) the
    fake and the Python checks refuse on the index tensor alike."""
    a = gang_args(**gang_refusals("cpu")[case][2])
    for call in (torch.ops.egpu.place_gangs, tables.place_gangs):
        with pytest.raises(RuntimeError, match="place_gangs: every tensor must be on one CUDA device"):
            call(*a)
    with FakeTensorMode():
        exc, msg, kw = gang_refusals("cuda")[case]
        a = gang_args(device="cuda", **kw)
        with pytest.raises(exc, match="place_gangs: " + msg):
            torch.ops.egpu.place_gangs(*a)
        with pytest.raises(exc, match="place_gangs: " + msg):
            tables.check_pod_args(a[0], a[5], op="place_gangs")
            tables.check_gang_args(a[0], a[6], a[7])


def test_tensors_off_the_gpu_are_refused(tables):
    for call in (torch.ops.egpu.place_gangs, tables.place_gangs):
        with pytest.raises(RuntimeError, match="place_gangs: every tensor must be on one CUDA device"):
            call(*gang_args())
    with FakeTensorMode():
        for k in (6, 7):  # only gang_offsets, or only gang_min, off the GPU
            a = list(gang_args(device="cuda"))
            a[k] = torch.zeros(a[k].shape, dtype=torch.int32)
            for call in (torch.ops.egpu.place_gangs, lambda *x: tables.check_gang_args(x[0], x[6], x[7])):
                with pytest.raises(RuntimeError, match="place_gangs: every tensor must be on one CUDA device"):
                    call(*a)


def bad_gangs(G=4):
    """Every way gang_offsets' and gang_min's values can be wrong, each with the eager check's message."""
    return [
        ([1, 2, 4], [1, 1], "gang_offsets must start at 0, got 1"),
        ([-1, 2, 4], [1, 1], "gang_offsets must start at 0, got -1"),
        ([0, 2, 3], [1, 1], "gang_offsets must end at G = 4, got 3"),
        ([0, 2, 5], [1, 1], "gang_offsets must end at G = 4, got 5"),
        ([0], [], "gang_offsets must end at G = 4, got 0"),
        ([0, 0, 4], [1, 1], "1 gang\\(s\\) with no pod"),
        ([0, 3, 1, 4], [1, 1, 1], "1 gang\\(s\\) with no pod"),
        ([0, -2147483648, 4], [1, 1], "1 gang\\(s\\) with no pod"),
        ([0, 2, 4], [0, 1], "1 gang\\(s\\) with gang_min outside \\[1, gang size\\]"),
        ([0, 2, 4], [3, 1], "1 gang\\(s\\) with gang_min outside \\[1, gang size\\]"),
        ([0, 2, 4], [-1, 2147483647], "2 gang\\(s\\) with gang_min outside \\[1, gang size\\]"),
        ([0, 1, 4], [1, 4], "1 gang\\(s\\) with gang_min outside \\[1, gang size\\]"),
    ]


@pytest.mark.parametrize("case", range(12))
def test_bad_gangs_refused_eagerly_and_by_the_restatement(case, tables):
    goff, gmin, msg = bad_gangs()[case]
    with pytest.raises(ValueError, match="place_gangs: " + msg):
        tables.check_gangs(torch.tensor(goff, dtype=torch.int32), torch.tensor(gmin, dtype=torch.int32), 4)
    assert not ref.gangs_ok(goff, gmin, 4)
    out = ref.place(np.full((2, 2), 50), np.full((2, 2), 100), [2, 2], [10] * 8, [0] * 8, [0, 2, 4, 6, 8], goff, gmin)
    node, dev, placed, fco, fmo, info = out
    assert (node == -1).all() and (dev == -1).all() and (placed == 0).all() and info == [0, 0, 1] and (fco == 50).all()


@pytest.mark.parametrize("case", range(10))
def test_bad_pod_offsets_refused_eagerly_and_by_the_restatement(case, tables):
    off, msg = ppc.bad_offsets()[case]
    t = torch.tensor(off, dtype=torch.int32)
    with pytest.raises(ValueError, match="place_gangs: pod_offsets " + msg if "must" in msg else "place_gangs: " + msg):
        tables.check_pods(t, 12, op="place_gangs")
    G = len(off) - 1
    out = ref.place(np.full((2, 2), 50), np.full((2, 2), 100), [2, 2], [10] * 12, [0] * 12, off, [0, G], [1])
    assert (out[0] == -1).all() and (out[1] == -1).all() and out[2].tolist() == [0] and out[5] == [0, 0, 1]


def test_good_gangs_pass_the_eager_check(tables):
    for goff, gmin, G in (([0, 4], [4], 4), ([0, 1, 2, 3, 4], [1, 1, 1, 1], 4), ([0, 3, 4], [2, 1], 4), ([0], [], 0)):
        tables.check_gangs(torch.tensor(goff, dtype=torch.int32), torch.tensor(gmin, dtype=torch.int32), G)
        assert ref.gangs_ok(goff, gmin, G)


def test_empty_calls_in_the_restatement():
    for N, P in ((0, 4), (3, 0)):
        G = P
        out = ref.place(np.full((N, 2), 50), np.full((N, 2), 9), [2] * N, [10] * P, [0] * P, list(range(P + 1)),
                        [0, G] if G else [0], [1] if G else [])
        assert (out[0] == -1).all() and (out[2] == 0).all() and out[5] == [0, 0, 0]
