"""egpu::preempt_gangs without a GPU (DESIGN.md §2.15): the numpy restatement against the hand-derived known answers,
against the literal loop of preempt_pods calls when no running job is capped, against place_gangs' restatement when
nothing is evictable and against preempt_pods' restatement for one gang of minimum 1; the fake's shapes; the fake,
the CPU registration and the Python checks refusing alike."""
import json
import os
import sys

import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import place_gangs_np  # noqa: E402
import preempt_gangs_np as ref  # noqa: E402
import preempt_pods_np  # noqa: E402
import test_preempt_pods_cpu as pods  # noqa: E402  (random running pods, refusal cases of preempt_pods)

KAT = json.load(open(os.path.join(HERE, "golden", "preempt_gangs_kat.json")))["cases"]
KEYS = ("free_core", "free_mem", "d_valid", "req_core", "req_mem", "pod_offsets", "gang_offsets", "gang_min",
        "gang_prio", "run_core", "run_mem", "run_dev", "run_offsets", "run_prio", "node_offsets", "run_gang",
        "run_gang_min")
OUTS = ("node", "dev", "placed", "evicted", "free_core_out", "free_mem_out")


def kat_args(c):
    a = [np.array(c[k], np.int8 if k == "run_dev" else np.int32) for k in KEYS]
    a[0] = a[0].reshape(len(c["d_valid"]), -1)
    a[1] = a[1].reshape(a[0].shape)
    return a


def random_case(g, N, D, J, run_hi=6, hi_pod=4, hi_gang=4, evictable=True, full=0.7, bad_nodes=0.0, R=None,
                run_lo=0):
    """preempt_pods' random tables and running pods, its pending pods grouped into J gangs of 1 to hi_gang pods
    with mixed minimums and priorities, and the running pods grouped into R running jobs (about a third of them in
    no job) with minimums from 0 to beyond their size.  R = 0: no running job."""
    sizes = g.integers(1, hi_gang + 1, J)
    goff = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    G = int(goff[-1])
    a = pods.random_case(g, N, D, G, run_hi=run_hi, hi_pod=hi_pod, evictable=evictable, full=full,
                         bad_nodes=bad_nodes, run_lo=run_lo)
    fc, fm, dv, rc, rm, off, prio, qc, qm, qd, roff, rprio, noff = a
    gmin = g.integers(1, sizes + 1).astype(np.int32)
    if evictable:
        gprio = g.choice(pods.PRIOS[2:], J).astype(np.int32)
    else:
        gprio = g.choice([-2**31, -7], J).astype(np.int32)
    H = rprio.size
    if R is None:
        R = int(g.integers(1, max(2, H // 2) + 1))
    rgang = np.where(g.random(H) < 0.35, -1, g.integers(0, max(R, 1), H)).astype(np.int32) if R else \
        np.full(H, -1, np.int32)
    size = np.bincount(rgang[rgang >= 0], minlength=R)
    rgmin = (g.integers(0, size + 2) if R else np.zeros(0, np.int64)).astype(np.int32)
    return [fc, fm, dv, rc, rm, off, goff, gmin, gprio, qc, qm, qd, roff, rprio, noff, rgang, rgmin]


@pytest.mark.parametrize("case", range(len(KAT)))
def test_restatement_known_answers(case):
    c = KAT[case]
    out = ref.place(*kat_args(c))
    for k, x in zip(OUTS, out[:6]):
        assert x.tolist() == c[k], (c["name"], k)
    assert list(out[6]) == c["info"], c["name"]


def test_known_answers_cover_the_rule():
    assert len(KAT) >= 11 and all(c["reason"] for c in KAT)
    assert any(c["raw"] for c in KAT) and any(c["info"][0] >= 3 for c in KAT)
    assert any(0 in c["placed"] and max(c["evicted"]) == -1 and c["info"][0] >= 1 for c in KAT)  # a gang given back


def test_no_running_job_is_the_literal_loop():
    """R = 0: one preempt_pods call per gang, the kept gangs' victims marked gone by zero demand and priority
    INT32_MAX; the restatement removes them from its alive set instead.  Equal outputs, rounds at most the loop's."""
    evicted = given_back = stopped = 0
    for seed in range(300):
        g = np.random.default_rng(seed)
        a = random_case(g, int(g.integers(1, 7)), int(g.integers(1, 6)), int(g.integers(1, 9)), R=0, full=0.9,
                        run_hi=5, bad_nodes=0.2 if seed % 5 == 0 else 0.0)
        got, exp = ref.place(*a), ref.loop(*a)
        for x, y in zip(got[:6], exp[:6]):
            np.testing.assert_array_equal(x, y)
        assert got[6][0] <= exp[6][0]
        evicted += int((got[3] >= 0).any())
        given_back += int((got[2] == 0).any())
        stopped += int(got[6][0] < exp[6][0])
    assert evicted >= 100 and given_back >= 50 and stopped >= 10, (evicted, given_back, stopped)


def test_every_min_zero_is_the_literal_loop():
    """A running job of minimum 0 has all its alive pods as slack, so neither rule ever binds."""
    for seed in range(100):
        g = np.random.default_rng(5000 + seed)
        a = random_case(g, int(g.integers(1, 7)), int(g.integers(1, 6)), int(g.integers(1, 7)), full=0.9)
        a[16][:] = 0
        got, exp = ref.place(*a), ref.loop(*a)
        for x, y in zip(got[:6], exp[:6]):
            np.testing.assert_array_equal(x, y)


def test_nothing_evictable_is_place_gangs():
    rounds = []
    for seed in range(300):
        g = np.random.default_rng(1000 + seed)
        a = random_case(g, int(g.integers(1, 9)), int(g.integers(1, 9)), int(g.integers(1, 10)), evictable=False)
        got = ref.place(*a)
        exp = place_gangs_np.place(*a[:8])
        for x, y in zip(got[:3] + got[4:6], exp[:5]):
            np.testing.assert_array_equal(x, y)
        assert (got[3] == -1).all() and got[6] == exp[5]
        rounds.append(got[6][0])
    assert max(rounds) >= 4


def test_one_gang_of_minimum_1_is_preempt_pods():
    evictions = 0
    for seed in range(300):
        g = np.random.default_rng(2000 + seed)
        a = random_case(g, int(g.integers(1, 8)), int(g.integers(1, 7)), 1, hi_gang=12, full=0.9, R=0)
        a[7][:] = 1
        got = ref.place(*a)
        G = int(a[6][-1])
        exp = preempt_pods_np.place(*a[:6], np.full(G, a[8][0], np.int32), *a[9:15])
        for x, y in zip(got[:2] + got[3:6], exp[:5]):
            np.testing.assert_array_equal(x, y)
        assert got[2].tolist() == [int((exp[0] >= 0).sum())] and got[6] == exp[5]
        evictions += int((got[3] >= 0).any())
    assert evictions >= 100, evictions


def test_running_jobs_never_cut_below_their_minimum():
    capped = 0
    for seed in range(200):
        g = np.random.default_rng(3000 + seed)
        a = random_case(g, int(g.integers(2, 9)), int(g.integers(1, 6)), int(g.integers(1, 9)), full=0.95,
                        run_hi=8)
        node, dev, placed, evicted, *_ = ref.place(*a)
        rgang, rgmin, gmin = a[15], a[16], a[7]
        alive0 = np.bincount(rgang[rgang >= 0], minlength=rgmin.size)
        gone = np.bincount(rgang[(rgang >= 0) & (evicted >= 0)], minlength=rgmin.size)
        assert (gone <= np.maximum(alive0 - rgmin, 0)).all()
        goff = a[6]
        gang_of = np.repeat(np.arange(gmin.size), np.diff(goff))
        kept = placed > 0
        assert (placed[kept] >= gmin[kept]).all()
        assert (~kept[gang_of[evicted[evicted >= 0]]]).sum() == 0  # gangs given back evict nothing
        capped += int((ref.loop(*a)[3] != evicted).any())
    assert capped >= 20, capped


# ---- the fake and the refusals ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tables():
    from elastic_gpu_agent_b200 import tables as t
    t.load()
    return t


def cpu_args(N=5, D=4, P=6, G=3, J=2, Q=4, H=2, R=1, device="cpu"):
    z = dict(dtype=torch.int32, device=device)
    a = pods.cpu_args(N, D, P, G, Q, H, device=device)
    del a["prio"]
    a.update(goff=torch.tensor([0] + [G] * J, **z) if J else torch.zeros(1, **z), gmin=torch.ones(J, **z),
             gprio=torch.ones(J, **z), rgang=torch.zeros(H, **z) if R else torch.full((H,), -1, **z),
             rgmin=torch.ones(R, **z))
    if J:
        a["goff"][1:] = torch.arange(1, J + 1, **z) * (G // J)
        a["goff"][-1] = G
    return a


ORDER = ("fc", "fm", "dv", "rc", "rm", "off", "goff", "gmin", "gprio", "qc", "qm", "qd", "roff", "rprio", "noff",
         "rgang", "rgmin")


def call(fn, a):
    return fn(*[a[k] for k in ORDER])


@pytest.mark.parametrize("N,D,P,G,J,Q,H,R", [(5, 4, 6, 3, 2, 4, 2, 1), (7, 64, 8, 8, 8, 0, 0, 0),
                                             (1, 1, 40, 5, 1, 12, 3, 3)])
def test_fake_gives_shapes_and_dtypes(N, D, P, G, J, Q, H, R, tables):
    with FakeTensorMode():
        a = cpu_args(N, D, P, G, J, Q, H, R, device="cuda")
        node, dev, placed, evicted, fco, fmo, info = call(torch.ops.egpu.preempt_gangs, a)
    assert node.shape == (G,) and dev.shape == (P,) and placed.shape == (J,) and evicted.shape == (H,)
    assert fco.shape == fmo.shape == (N, D) and info.shape == (3,) and dev.dtype == torch.int8
    assert node.dtype == placed.dtype == evicted.dtype == fco.dtype == fmo.dtype == info.dtype == torch.int32
    assert all(t.device.type == "cuda" for t in (node, dev, placed, evicted, fco, fmo, info))


def refusal_cases(device="cpu"):
    """(exception, arguments, message): the checks in the operator's order, device last."""
    def with_(**kw):
        a = cpu_args(device=device)
        a.update(kw)
        return a

    z = dict(dtype=torch.int32, device=device)
    base = cpu_args(device=device)
    out = []
    for exc, pa, msg in pods.refusal_cases(device)[:-1]:  # preempt_pods' own, but for pod_prio
        if "pod_prio" in msg:
            continue
        a = dict(base)
        a.update({k: v for k, v in pa.items() if k != "prio"})
        out.append((exc, a, msg))
    return out[:4] + [
        (RuntimeError, with_(goff=base["goff"].to(torch.int64)), "gang_offsets must be int32"),
        (RuntimeError, with_(gmin=torch.arange(4, **z)[::2]), "gang_min must be contiguous"),
        (ValueError, with_(goff=torch.zeros(0, **z)), "gang_offsets must be \\[J \\+ 1\\]"),
        (ValueError, with_(gmin=torch.ones(3, **z)), "gang_min must be \\[J\\]"),
    ] + out[4:] + [
        (RuntimeError, with_(gprio=base["gprio"].to(torch.int64)), "gang_prio must be int32"),
        (RuntimeError, with_(rgang=base["rgang"].to(torch.int16)), "run_gang must be int32"),
        (RuntimeError, with_(rgmin=torch.arange(4, **z)[::2]), "run_gang_min must be contiguous"),
        (ValueError, with_(gprio=torch.ones(3, **z)), "gang_prio must be \\[J\\] = \\[2\\]"),
        (ValueError, with_(rgang=torch.zeros(3, **z)), "run_gang must be \\[H\\] = \\[2\\]"),
        (ValueError, with_(rgmin=torch.zeros((1, 1), **z)), "run_gang_min must be \\[R\\]"),
        (RuntimeError, with_(rgmin=torch.zeros(1, dtype=torch.int32)), "every tensor must be on one CUDA device"),
    ]


@pytest.mark.parametrize("i", range(len(refusal_cases())))
def test_fake_cpu_registration_and_checks_refuse_alike(i, tables):
    # CPU tensors reach the CPU registration, which refuses them on the device check after the table checks
    exc, a, msg = refusal_cases()[i]
    if i >= 2:
        exc, msg = RuntimeError, "every tensor must be on one CUDA device"
    for fn in (tables.preempt_gangs, torch.ops.egpu.preempt_gangs):
        with pytest.raises(exc, match="preempt_gangs: " + msg):
            call(fn, a)
    with FakeTensorMode():  # CUDA-looking tensors reach every check: the fake and the Python checks
        exc, a, msg = refusal_cases("cuda")[i]
        with pytest.raises(exc, match="preempt_gangs: " + msg):
            call(torch.ops.egpu.preempt_gangs, a)
        with pytest.raises(exc, match="preempt_gangs: " + msg):
            op = "preempt_gangs"
            tables.check_args(a["fc"], a["fm"], a["dv"], a["rc"], a["rm"], op=op)
            tables.check_pod_args(a["fc"], a["off"], op=op)
            tables.check_gang_args(a["fc"], a["goff"], a["gmin"], op=op)
            tables.check_preempt_args(a["fc"], a["off"], None, *[a[k] for k in ("qc", "qm", "qd", "roff", "rprio",
                                                                                 "noff")], op=op)
            tables.check_preempt_gang_args(a["fc"], a["goff"], a["roff"], a["gprio"], a["rgang"], a["rgmin"])


BAD_VALUES = [  # (key, value, message of the eager check)
    ("rgang", [0, 1], "1 running pod\\(s\\) with run_gang outside \\[-1, 1\\)"),
    ("rgang", [-2, 0], "running pod\\(s\\) with run_gang outside"),
    ("rgmin", [-1], "running job\\(s\\) with run_gang_min below 0"),
]


@pytest.mark.parametrize("i", range(len(BAD_VALUES)))
def test_eager_checks_of_the_running_jobs(i, tables):
    a = cpu_args()
    key, value, msg = BAD_VALUES[i]
    a[key] = torch.tensor(value, dtype=torch.int32)
    with pytest.raises(ValueError, match="preempt_gangs: .*" + msg):
        tables.check_running_gangs(a["rgang"], a["rgmin"])
    x = {k: v.numpy() for k, v in a.items()}
    assert not ref.index_ok(x["off"], 6, x["goff"], x["gmin"], x["roff"], 4, x["noff"], 2, 5, x["rgang"], x["rgmin"])


def test_eager_checks_accept_consistent_running_jobs(tables):
    a = cpu_args()
    tables.check_running_gangs(a["rgang"], a["rgmin"])
    tables.check_running_gangs(torch.full((2,), -1, dtype=torch.int32), torch.zeros(0, dtype=torch.int32))
    x = {k: v.numpy() for k, v in a.items()}
    assert ref.index_ok(x["off"], 6, x["goff"], x["gmin"], x["roff"], 4, x["noff"], 2, 5, x["rgang"], x["rgmin"])
