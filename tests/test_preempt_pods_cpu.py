"""egpu::preempt_pods without a GPU (DESIGN.md §2.14): the numpy restatement against the hand-derived known answers,
against place_pods' restatement when no pending pod outranks a running pod, and against the literal single-pod rule;
the fake's shapes; the fake, the CPU registration and the Python checks refusing alike."""
import json
import os
import sys

import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import place_pods_np  # noqa: E402
import preempt_pods_np as ref  # noqa: E402

KAT = json.load(open(os.path.join(HERE, "golden", "preempt_pods_kat.json")))["cases"]
KEYS = ("free_core", "free_mem", "d_valid", "req_core", "req_mem", "pod_offsets", "pod_prio", "run_core", "run_mem",
        "run_dev", "run_offsets", "run_prio", "node_offsets")
PRIOS = np.array([-2**31, -7, 0, 1, 5, 10, 2**31 - 1])


def kat_args(c):
    return [np.array(c[k], np.int8 if k == "run_dev" else np.int32) for k in KEYS]


def random_case(g, N, D, G, run_hi=6, hi_pod=4, evictable=True, full=0.7, bad_nodes=0.0, run_lo=0):
    """Tables of N nodes whose devices hold running pods (consistent by construction), and G pending pods.  With
    evictable=False no pending pod outranks any running pod.  bad_nodes: share of nodes made inconsistent."""
    dv = g.integers(1, D + 1, N).astype(np.int32)
    cap_c = np.full((N, D), 100, np.int64)
    cap_m = np.full((N, D), 80_000, np.int64)
    qc, qm, qd, roff, rprio, noff = [], [], [], [0], [], [0]
    for n in range(N):
        for _ in range(int(g.integers(run_lo, run_hi + 1))):
            k = int(g.integers(1, hi_pod + 1))
            for _ in range(k):
                d = int(g.integers(0, dv[n]))
                c = int(min(cap_c[n, d], g.choice([5, 10, 25, 50, 100])))
                m = int(min(cap_m[n, d], g.choice([0, 1000, 4000, 40_000])))
                cap_c[n, d] -= c
                cap_m[n, d] -= m
                qc.append(c)
                qm.append(m)
                qd.append(d)
            roff.append(roff[-1] + k)
            rprio.append(int(g.choice(PRIOS[1:5])))
        noff.append(len(rprio))
    # part of what the running pods leave is held by pods the caller does not list (not evictable)
    fc = (cap_c - (g.random((N, D)) < full) * g.integers(0, cap_c + 1)).astype(np.int32)
    fm = (cap_m - (g.random((N, D)) < full) * g.integers(0, cap_m + 1)).astype(np.int32)
    bad = np.flatnonzero(g.random(N) < bad_nodes)
    for n in bad:
        if noff[n + 1] > noff[n]:
            c = roff[noff[n]]
            fc[n, qd[c]] = 100  # free + its demand > 100 when the container holds core
            qc[c] = max(qc[c], 1)
    sizes = g.integers(1, hi_pod + 1, G)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    P = int(off[-1])
    rc = g.choice([5, 10, 25, 50, 100], P).astype(np.int32)
    rm = g.choice([0, 1000, 4000, 40_000], P).astype(np.int32)
    rprio = np.array(rprio, np.int32)
    if evictable:
        prio = g.choice(PRIOS[2:], G).astype(np.int32)
    else:
        prio = g.choice([-2**31, -7], G).astype(np.int32)
        rprio = np.maximum(rprio, prio.max(initial=-2**31)).astype(np.int32)
    return [fc, fm, dv, rc, rm, off, prio, np.array(qc, np.int32), np.array(qm, np.int32), np.array(qd, np.int8),
            np.array(roff, np.int32), rprio, np.array(noff, np.int32)]


def equal(x, y):
    for a, b in zip(x[:5], y[:5]):
        np.testing.assert_array_equal(a, b)
    assert list(x[5]) == list(y[5])


@pytest.mark.parametrize("case", range(len(KAT)))
def test_restatement_known_answers(case):
    c = KAT[case]
    node, dev, evicted, fco, fmo, info = ref.place(*kat_args(c))
    assert node.tolist() == c["node"] and dev.tolist() == c["dev"] and evicted.tolist() == c["evicted"], c["name"]
    assert fco.tolist() == c["free_core_out"] and fmo.tolist() == c["free_mem_out"], c["name"]
    assert info == [c["rounds"], 0, 0], c["name"]


def test_known_answers_cover_the_rule():
    assert len(KAT) >= 11 and all(c["reason"] for c in KAT)
    assert any(c["raw"] for c in KAT) and any(c["rounds"] >= 2 for c in KAT)


def test_nothing_evictable_is_place_pods():
    rounds = []
    for seed in range(300):
        g = np.random.default_rng(seed)
        a = random_case(g, int(g.integers(1, 9)), int(g.integers(1, 9)), int(g.integers(1, 25)), evictable=False)
        got = ref.place(*a)
        exp = place_pods_np.place(*a[:6])
        for x, y in zip(got[:2] + got[3:5], exp[:4]):
            np.testing.assert_array_equal(x, y)
        assert (got[2] == -1).all() and got[5] == exp[4]
        rounds.append(got[5][0])
    assert max(rounds) >= 3


def test_single_pod_equals_the_literal_rule():
    evictions = 0
    for seed in range(300):
        g = np.random.default_rng(1000 + seed)
        a = random_case(g, int(g.integers(1, 7)), int(g.integers(1, 6)), 1, run_hi=5, full=0.9,
                        bad_nodes=0.2 if seed % 3 == 0 else 0.0)
        equal(ref.place(*a), ref.single(*a))
        evictions += int((ref.place(*a)[2] >= 0).any())
    assert evictions >= 50, evictions


# ---- the fake and the refusals ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tables():
    from elastic_gpu_agent_b200 import tables as t
    t.load()
    return t


def cpu_args(N=5, D=4, P=6, G=3, Q=4, H=2, device="cpu"):
    z = dict(dtype=torch.int32, device=device)
    return dict(fc=torch.full((N, D), 50, **z), fm=torch.full((N, D), 1000, **z), dv=torch.full((N,), D, **z),
                rc=torch.full((P,), 10, **z), rm=torch.zeros(P, **z), off=torch.arange(G + 1, **z) * (P // G),
                prio=torch.ones(G, **z), qc=torch.full((Q,), 10, **z), qm=torch.zeros(Q, **z),
                qd=torch.zeros(Q, dtype=torch.int8, device=device), roff=torch.arange(H + 1, **z) * (Q // max(H, 1)),
                rprio=torch.zeros(H, **z), noff=torch.tensor([0, H] + [H] * (N - 1), **z))


ORDER = ("fc", "fm", "dv", "rc", "rm", "off", "prio", "qc", "qm", "qd", "roff", "rprio", "noff")


def call(fn, a):
    return fn(*[a[k] for k in ORDER])


@pytest.mark.parametrize("N,D,P,G,Q,H", [(5, 4, 6, 3, 4, 2), (7, 64, 8, 8, 0, 0), (1, 1, 40, 5, 12, 3)])
def test_fake_gives_shapes_and_dtypes(N, D, P, G, Q, H, tables):
    with FakeTensorMode():
        a = cpu_args(N, D, P, G, Q, H, device="cuda")
        node, dev, evicted, fco, fmo, info = call(torch.ops.egpu.preempt_pods, a)
    assert node.shape == (G,) and dev.shape == (P,) and evicted.shape == (H,) and fco.shape == fmo.shape == (N, D)
    assert info.shape == (3,) and dev.dtype == torch.int8
    assert node.dtype == evicted.dtype == fco.dtype == fmo.dtype == info.dtype == torch.int32
    assert all(t.device.type == "cuda" for t in (node, dev, evicted, fco, fmo, info))


def refusal_cases(device="cpu"):
    """(exception, arguments, message): the checks in the operator's order, device last."""
    def with_(**kw):
        a = cpu_args(device=device)
        a.update(kw)
        return a

    def cpu_args_(**kw):
        return cpu_args(device=device, **kw)

    z = dict(dtype=torch.int32, device=device)
    return [
        (RuntimeError, with_(fc=cpu_args_()["fc"].to(torch.int64)), "free_core must be int32"),
        (ValueError, with_(fm=torch.full((5, 3), 1, **z)), "free_core and free_mem"),
        (RuntimeError, with_(off=cpu_args_()["off"].to(torch.int64)), "pod_offsets must be int32"),
        (ValueError, with_(off=torch.zeros(0, **z)), "pod_offsets must be"),
        (RuntimeError, with_(prio=cpu_args_()["prio"].to(torch.int64)), "pod_prio must be int32"),
        (RuntimeError, with_(qc=cpu_args_()["qc"].to(torch.int16)), "run_core must be int32"),
        (RuntimeError, with_(qm=torch.arange(8, **z)[::2]), "run_mem must be contiguous"),
        (RuntimeError, with_(qd=cpu_args_()["qd"].to(torch.int32)), "run_dev must be int8"),
        (RuntimeError, with_(roff=cpu_args_()["roff"].to(torch.int64)), "run_offsets must be int32"),
        (RuntimeError, with_(rprio=cpu_args_()["rprio"].to(torch.float32)), "run_prio must be int32"),
        (RuntimeError, with_(noff=cpu_args_()["noff"].to(torch.int64)), "node_offsets must be int32"),
        (ValueError, with_(prio=torch.ones(2, **z)), "pod_prio must be"),
        (ValueError, with_(qm=torch.zeros(3, **z)), "run_core, run_mem and run_dev"),
        (ValueError, with_(qd=torch.zeros(5, dtype=torch.int8, device=device)), "run_core, run_mem and run_dev"),
        (ValueError, with_(roff=torch.zeros(0, **z)), "run_offsets must be"),
        (ValueError, with_(rprio=torch.zeros(3, **z)), "run_prio must be"),
        (ValueError, with_(noff=torch.zeros(5, **z)), "node_offsets must be"),
        (RuntimeError, with_(noff=torch.zeros(6, dtype=torch.int32)), "every tensor must be on one CUDA device"),
    ]


@pytest.mark.parametrize("i", range(len(refusal_cases())))
def test_fake_cpu_registration_and_checks_refuse_alike(i, tables):
    # CPU tensors reach the CPU registration, which refuses them on the device check after the table checks
    exc, a, msg = refusal_cases()[i]
    if i >= 2:
        exc, msg = RuntimeError, "every tensor must be on one CUDA device"
    for fn in (tables.preempt_pods, torch.ops.egpu.preempt_pods):
        with pytest.raises(exc, match="preempt_pods: " + msg):
            call(fn, a)
    with FakeTensorMode():  # CUDA-looking tensors reach every check: the fake and the Python checks
        exc, a, msg = refusal_cases("cuda")[i]
        with pytest.raises(exc, match="preempt_pods: " + msg):
            call(torch.ops.egpu.preempt_pods, a)
        with pytest.raises(exc, match="preempt_pods: " + msg):
            tables.check_args(a["fc"], a["fm"], a["dv"], a["rc"], a["rm"], op="preempt_pods")
            tables.check_pod_args(a["fc"], a["off"], op="preempt_pods")
            tables.check_preempt_args(*[a[k] for k in ("fc", "off", "prio", "qc", "qm", "qd", "roff", "rprio", "noff")])


BAD_VALUES = [  # (key, value, message of the eager check)
    ("roff", [1, 2, 4], "run_offsets must start at 0"), ("roff", [0, 2, 3], "run_offsets must end at Q = 4"),
    ("roff", [0, 0, 4], "running pod\\(s\\) with a container count"), ("roff", [0, 9, 4], "running pod"),
    ("noff", [1, 2, 2, 2, 2, 2], "node_offsets must start at 0"), ("noff", [0, 1, 1, 1, 1, 1], "must end at H = 2"),
    ("noff", [0, 2, 1, 2, 2, 2], "node\\(s\\) with a running pod count"),
    ("qd", [0, 0, 4, 0], "inconsistent running data"), ("qd", [0, -1, 0, 0], "inconsistent running data"),
    ("qc", [10, 10, 101, 10], "inconsistent running data"), ("qm", [0, -1, 0, 0], "inconsistent running data"),
    ("qc", [10, 41, 10, 10], "inconsistent running data"),  # 50 free + 10 + 41 on device 0 of node 0
]


@pytest.mark.parametrize("i", range(len(BAD_VALUES)))
def test_eager_checks_of_the_running_pods(i, tables):
    a = cpu_args()
    key, value, msg = BAD_VALUES[i]
    a[key] = torch.tensor(value, dtype=a[key].dtype)
    with pytest.raises(ValueError, match="preempt_pods: .*" + msg):
        tables.check_running(a["fc"], a["fm"], a["dv"], a["qc"], a["qm"], a["qd"], a["roff"], a["noff"])
    if key in ("roff", "noff"):
        assert not ref.index_ok(a["off"].numpy(), 6, a["roff"].numpy(), 4, a["noff"].numpy(), 2, 5)
    else:
        x = {k: v.numpy() for k, v in a.items()}
        assert not ref.usable_nodes(x["fc"], x["fm"], x["dv"], x["qc"], x["qm"], x["qd"], x["roff"], x["noff"])[0]


def test_eager_checks_accept_consistent_running_pods(tables):
    a = cpu_args()
    tables.check_running(a["fc"], a["fm"], a["dv"], a["qc"], a["qm"], a["qd"], a["roff"], a["noff"])
    a["qc"][:] = 25  # 50 free + 4 x 25 = 150 > 100 on device 0 of node 0
    with pytest.raises(ValueError, match="preempt_pods: 1 node"):
        tables.check_running(a["fc"], a["fm"], a["dv"], a["qc"], a["qm"], a["qd"], a["roff"], a["noff"])
