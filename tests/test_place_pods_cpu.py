"""egpu::place_pods without a GPU (DESIGN.md §2.12).

  1. the numpy restatement (tests/place_pods_np.py) against the hand-derived answers of
     tests/golden/place_pods_kat.json;
  2. pods of one container: the restatement equals place_tables' restatement (node, device, tables, rounds) on 300
     seeded cases;
  3. one pod: oracle/bestfit_np.replay of the pod's ALLOC events on each table gives the devices and leftovers, and
     the pod goes to the node with the smallest (sum of core leftovers, sum of memory leftovers, n);
  4. the fake implementation's shapes and dtypes;
  5. the refusals: bestfit_tables' with "place_pods" in the messages, then pod_offsets', alike through the fake, the
     compiled operator (its CPU registration) and the Python checks; the eager check of the offsets' values.
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
import place_pods_np as ref  # noqa: E402
import place_tables_np  # noqa: E402
import test_place_tables_cpu as ptc  # noqa: E402  (seeded cases of place_tables)
import test_tables_cpu as tc  # noqa: E402  (argument builder and the refusal cases of bestfit_tables)

from oracle import bestfit_np  # noqa: E402

MEM_MAX = (1 << 18) - 1
KAT = json.load(open(os.path.join(HERE, "golden", "place_pods_kat.json")))["cases"]


@pytest.fixture(scope="module")
def tables():
    from elastic_gpu_agent_b200 import tables as t
    t.load()
    return t


# ---- 1. known answers ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", range(len(KAT)))
def test_restatement_matches_the_known_answers(case):
    c = KAT[case]
    node, dev, fco, fmo, info = ref.place(np.array(c["free_core"]), np.array(c["free_mem"]), c["d_valid"],
                                          c["req_core"], c["req_mem"], c["pod_offsets"])
    assert node.tolist() == c["node"] and dev.tolist() == c["dev"], c["name"]
    assert fco.tolist() == c["free_core_out"] and fmo.tolist() == c["free_mem_out"], c["name"]
    assert info == [c["rounds"], 0, 0], c["name"]


def test_known_answers_cover_the_listed_cases():
    assert len(KAT) == 9 and {c["rounds"] for c in KAT} == {1, 2, 3}
    assert max(len(c["pod_offsets"]) for c in KAT) >= 3 and max(np.diff(c["pod_offsets"]).max() for c in KAT) == 8


# ---- 2. one container per pod: place_tables ---------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(300))
def test_single_container_pods_equal_place_tables(seed):
    g = np.random.default_rng(9000 + seed)
    fc, fm, dv, rc, rm = ptc.random_case(g, contended=seed % 3 != 0)
    P = rc.size
    node, dev, fco, fmo, info = ref.place(fc, fm, dv, rc, rm, np.arange(P + 1))
    e_node, e_dev, e_fc, e_fm, e_rounds = place_tables_np.place(fc, fm, dv, rc, rm)
    if P == 0:  # place_pods gives no launch for P = 0; place_tables' restatement agrees on everything but shapes
        assert info == [0, 0, 0] and node.size == dev.size == 0
        return
    np.testing.assert_array_equal(node, e_node)
    np.testing.assert_array_equal(dev, e_dev)
    np.testing.assert_array_equal(fco, e_fc)
    np.testing.assert_array_equal(fmo, e_fm)
    assert info == [e_rounds, 0, 0]


# ---- 3. one pod: the single-table replay oracle ------------------------------------------------------------------
def random_pods(g, G, lo=1, hi=8):
    sizes = g.integers(lo, hi + 1, G)
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)


@pytest.mark.parametrize("seed", range(100))
def test_one_pod_is_the_replay_on_its_best_node(seed):
    g = np.random.default_rng(4400 + seed)
    N, D = int(g.integers(1, 12)), int(g.integers(1, 17))
    fc = g.choice([0, 10, 25, 50, 75, 100], (N, D)).astype(np.int32)
    fm = g.choice([0, 1024, 4096, 40_000], (N, D)).astype(np.int32)
    dv = g.integers(1, D + 1, N).astype(np.int32)
    off = random_pods(g, 1)
    P = int(off[-1])
    rc = g.choice([0, 5, 10, 25, 50], P).astype(np.int32)
    rm = g.choice([0, 512, 1024, 4096], P).astype(np.int32)
    node, dev, fco, fmo, info = ref.place(fc, fm, dv, rc, rm, off)
    best = None
    for n in range(N):
        idx, o_fc, o_fm = bestfit_np.replay(fc[n, :dv[n]], fm[n, :dv[n]], np.zeros(P, np.int32), rc, rm)
        if (idx < 0).any():
            continue
        # the leftovers at the moment each container is placed: replay the prefixes
        slc = slm = 0
        left_c, left_m = fc[n, :dv[n]].astype(np.int64), fm[n, :dv[n]].astype(np.int64)
        for k, d in enumerate(idx):
            left_c[d] -= rc[k]
            left_m[d] -= rm[k]
            slc += int(left_c[d])
            slm += int(left_m[d])
        np.testing.assert_array_equal(left_c, o_fc)
        np.testing.assert_array_equal(left_m, o_fm)
        if best is None or (slc, slm, n) < best[0]:
            best = ((slc, slm, n), idx, o_fc, o_fm)
    if best is None:
        assert node.tolist() == [-1] and (dev == -1).all() and info[0] == 1
        return
    n = best[0][2]
    assert node.tolist() == [n] and info[0] == 1
    np.testing.assert_array_equal(dev, best[1])
    np.testing.assert_array_equal(fco[n, :dv[n]], best[2])
    np.testing.assert_array_equal(fmo[n, :dv[n]], best[3])
    others = np.arange(N) != n
    np.testing.assert_array_equal(fco[others], fc[others])


def test_a_pod_that_failed_can_fit_a_smaller_table():
    """§2.12: fit is not monotone.  d0 = (50, 100), d1 = (60, 10): the pod (10, 5), (50, 100) fails, because its
    first container takes d0; with d1 shrunk to (15, 10) the same pod fits."""
    off = [0, 2]
    rc, rm = [10, 50], [5, 100]
    assert ref.place(np.array([[50, 60]]), np.array([[100, 10]]), [2], rc, rm, off)[0].tolist() == [-1]
    node, dev, *_ = ref.place(np.array([[50, 15]]), np.array([[100, 10]]), [2], rc, rm, off)
    assert node.tolist() == [0] and dev.tolist() == [1, 0]


# ---- 4. the fake ----------------------------------------------------------------------------------------------
def pod_args(N=6, D=8, P=12, G=None, device="cpu", **kw):
    fc, fm, dv, rc, rm = tc.args(N, D, P, device=device)
    G = P if G is None else G
    a = dict(fc=fc, fm=fm, dv=dv, rc=rc, rm=rm,
             off=torch.arange(G + 1, dtype=torch.int32, device=device) * (P // max(G, 1)))
    a.update(kw)
    return a["fc"], a["fm"], a["dv"], a["rc"], a["rm"], a["off"]


@pytest.mark.parametrize("N,D,P,G", [(6, 8, 12, 4), (5000, 8, 2560, 1024), (512, 64, 8192, 4096), (0, 3, 7, 7),
                                     (4, 1, 0, 0)])
def test_fake_gives_shapes_and_dtypes(N, D, P, G, tables):
    with FakeTensorMode():
        node, dev, fco, fmo, info = torch.ops.egpu.place_pods(*pod_args(N, D, P, G, device="cuda"))
    assert node.shape == (G,) and dev.shape == (P,) and fco.shape == fmo.shape == (N, D) and info.shape == (3,)
    assert node.dtype == fco.dtype == fmo.dtype == info.dtype == torch.int32 and dev.dtype == torch.int8
    assert all(t.device.type == "cuda" for t in (node, dev, fco, fmo, info))


# ---- 5. refusals ------------------------------------------------------------------------------------------------
def offsets_refusals(device):
    z = dict(dtype=torch.int32, device=device)
    return [
        (RuntimeError, "pod_offsets must be int32", dict(off=torch.arange(13, dtype=torch.int64, device=device))),
        (RuntimeError, "pod_offsets must be contiguous", dict(off=torch.arange(26, **z)[::2])),
        (ValueError, "pod_offsets must be \\[G \\+ 1\\]", dict(off=torch.zeros(0, **z))),
        (ValueError, "pod_offsets must be \\[G \\+ 1\\]", dict(off=torch.zeros((13, 1), **z))),
    ]


@pytest.mark.parametrize("case", range(13))
def test_table_refusals_alike(case, tables):
    exc, msg, kw = tc.refusals("cpu")[case]
    msg = "place_pods: .*" + msg
    off = torch.arange(13, dtype=torch.int32)
    with pytest.raises(exc, match=msg):
        torch.ops.egpu.place_pods(*tc.args(**kw), off)  # the compiled operator, CPU tensors: refused before the device check
    with pytest.raises(exc, match=msg):
        tables.check_args(*tc.args(**kw), op="place_pods")
    with pytest.raises(exc, match=msg):
        tables.place_pods(*tc.args(**kw), off)
    with FakeTensorMode():
        exc_f, msg_f, kw_f = tc.refusals("cuda")[case]
        with pytest.raises(exc_f, match="place_pods: .*" + msg_f):
            torch.ops.egpu.place_pods(*tc.args(device="cuda", **kw_f), torch.arange(13, dtype=torch.int32, device="cuda"))


@pytest.mark.parametrize("case", range(4))
def test_offsets_refusals_alike(case, tables):
    """pod_offsets is checked after the other five tensors' device, so with CPU tensors the compiled operator and the
    Python interface both refuse on the device; with CUDA tensors (fake here, real in the GPU tests) the fake and
    the Python checks refuse on the offsets alike."""
    a = pod_args(**offsets_refusals("cpu")[case][2])
    for call in (torch.ops.egpu.place_pods, tables.place_pods):
        with pytest.raises(RuntimeError, match="place_pods: every tensor must be on one CUDA device"):
            call(*a)
    with FakeTensorMode():
        exc, msg, kw = offsets_refusals("cuda")[case]
        a = pod_args(device="cuda", **kw)
        with pytest.raises(exc, match="place_pods: " + msg):
            torch.ops.egpu.place_pods(*a)
        with pytest.raises(exc, match="place_pods: " + msg):
            tables.check_pod_args(a[0], a[5])


def test_tensors_off_the_gpu_are_refused(tables):
    for call in (torch.ops.egpu.place_pods, tables.place_pods):
        with pytest.raises(RuntimeError, match="place_pods: every tensor must be on one CUDA device"):
            call(*pod_args())
    with FakeTensorMode():
        a = list(pod_args(device="cuda"))
        a[5] = torch.arange(13, dtype=torch.int32)  # only the offsets off the GPU
        for call in (torch.ops.egpu.place_pods, lambda *x: tables.check_pod_args(x[0], x[5])):
            with pytest.raises(RuntimeError, match="place_pods: every tensor must be on one CUDA device"):
                call(*a)


def bad_offsets(P=12):
    """Every way pod_offsets' values can be wrong, each with the eager check's message: (offsets, message)."""
    return [
        ([1, 4, 8, 12], "must start at 0, got 1"),
        ([-1, 4, 8, 12], "must start at 0, got -1"),
        ([0, 4, 8, 11], "must end at P = 12, got 11"),
        ([0, 4, 8, 13], "must end at P = 12, got 13"),
        ([0], "must end at P = 12, got 0"),
        ([0, 4, 4, 12], "1 pod\\(s\\) with a container count outside \\[1, 8\\]"),
        ([0, 6, 3, 12], "2 pod\\(s\\) with a container count outside \\[1, 8\\]"),
        ([0, 2, 11, 12], "1 pod\\(s\\) with a container count outside \\[1, 8\\]"),
        ([0, -2147483648, 12], "2 pod\\(s\\) with a container count outside \\[1, 8\\]"),
        ([0, 2147483647, 12], "2 pod\\(s\\) with a container count outside \\[1, 8\\]"),
    ]


@pytest.mark.parametrize("case", range(10))
def test_bad_offsets_refused_eagerly_and_by_the_restatement(case, tables):
    off, msg = bad_offsets()[case]
    t = torch.tensor(off, dtype=torch.int32)
    with pytest.raises(ValueError, match="place_pods: pod_offsets " + msg if "must" in msg else "place_pods: " + msg):
        tables.check_pods(t, 12)
    assert not ref.offsets_ok(off, 12)
    node, dev, fco, fmo, info = ref.place(np.full((2, 2), 50), np.full((2, 2), 100), [2, 2], [10] * 12, [0] * 12, off)
    assert (node == -1).all() and (dev == -1).all() and info == [0, 0, 1] and (fco == 50).all()


def test_good_offsets_pass_the_eager_check(tables):
    for off, P in (([0, 8], 8), ([0, 1, 2, 3], 3), ([0, 3, 11, 12], 12), ([0], 0)):
        tables.check_pods(torch.tensor(off, dtype=torch.int32), P)
        assert ref.offsets_ok(off, P)
