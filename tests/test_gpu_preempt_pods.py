"""egpu::preempt_pods on the GPU (DESIGN.md §2.14): pods placed on N capacity tables, evicting the fewest,
lowest-priority running pods of one node where a pod fits no node as it is, in one cooperative launch.

  1. the known answers of tests/golden/preempt_pods_kat.json, exactly;
  2. the numpy restatement at the D buckets and their edges, with padding, inconsistent nodes and contended seeds;
  3. bit-identical to place_pods when no pending pod outranks a running pod, at 5 000 x 8 and 512 x 64;
  4. contended calls of many rounds, ragged tiles, nodes at 0 and 128 running pods;
  5. the invariants (per device: input + evicted demand - placed demand = output; nothing oversubscribed; every
     victim below its evictor and on its node);
  6. empty calls, inputs unchanged, two calls bit-identical;
  7. CUDA-graph capture and replay on new inputs, torch.compile(fullgraph=True);
  8. refusals before any launch, and bad offset tensors given to the raw operator during capture.
"""
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import preempt_pods_np as ref  # noqa: E402
import test_preempt_pods_cpu as cpu  # noqa: E402  (random cases, argument builders, refusal cases)

KAT = cpu.KAT


@pytest.fixture(scope="module")
def tables():
    from elastic_gpu_agent_b200 import tables as t
    t.load()
    return t


def cuda(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def run(tables, a, raw=False):
    fn = torch.ops.egpu.preempt_pods if raw else tables.preempt_pods
    out = fn(*cuda(*a))
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


def check(a, out, exp=None):
    """out equals the restatement's outputs exp (computed here when not given), info included."""
    exp = ref.place(*a) if exp is None else exp
    assert out[0].dtype == np.int32 and out[1].dtype == np.int8 and out[2].dtype == np.int32
    for x, y in zip(out[:5], exp[:5]):
        np.testing.assert_array_equal(x, y)
    assert out[5].tolist() == exp[5]
    return exp


def invariants(a, out):
    fc, fm, dv, rc, rm, off, prio, qc, qm, qd, roff, rprio, noff = a
    node, dev, evicted, fco, fmo, info = [np.asarray(x) for x in out]
    N, D = fc.shape
    assert info[1] == 0 and info[2] == 0 and not (node == -2).any() and not (dev == -2).any()
    pod_of = np.repeat(np.arange(node.size), np.diff(off))
    cnode = node[pod_of]
    assert ((cnode == -1) == (dev == -1)).all()
    run_node = np.repeat(np.arange(N), np.diff(noff))
    gone = evicted >= 0
    assert (node[evicted[gone]] == run_node[gone]).all()  # a victim is on its evictor's node ...
    assert (rprio[gone] < prio[evicted[gone]]).all()  # ... and below its priority
    delta_c = np.zeros((N, D), np.int64)
    delta_m = np.zeros((N, D), np.int64)
    rpod = np.repeat(np.arange(rprio.size), np.diff(roff))
    ev = gone[rpod] if rpod.size else np.zeros(0, bool)
    np.add.at(delta_c, (run_node[rpod[ev]], qd[ev].astype(np.int64)), qc[ev])
    np.add.at(delta_m, (run_node[rpod[ev]], qd[ev].astype(np.int64)), qm[ev])
    kept = cnode >= 0
    np.subtract.at(delta_c, (cnode[kept], dev[kept].astype(np.int64)), rc[kept])
    np.subtract.at(delta_m, (cnode[kept], dev[kept].astype(np.int64)), rm[kept])
    np.testing.assert_array_equal(fc.astype(np.int64) + delta_c, fco)
    np.testing.assert_array_equal(fm.astype(np.int64) + delta_m, fmo)
    valid = np.arange(D)[None, :] < dv[:, None]
    assert (fco[valid] >= 0).all() and (fmo[valid] >= 0).all()
    assert (dev[kept] < dv[cnode[kept]]).all()


# ---- 1. known answers ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(KAT)))
def test_known_answers(case, tables):
    c = KAT[case]
    node, dev, evicted, fco, fmo, info = run(tables, cpu.kat_args(c), raw=c["raw"])
    assert node.tolist() == c["node"] and dev.tolist() == c["dev"] and evicted.tolist() == c["evicted"], c["name"]
    assert fco.tolist() == c["free_core_out"] and fmo.tolist() == c["free_mem_out"], c["name"]
    assert info.tolist() == [c["rounds"], 0, 0], c["name"]


# ---- 2. the D buckets ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 5, 8, 9, 16, 17, 32, 33, 64])
def test_restatement_at_the_d_buckets(D, tables):
    evicted, rounds = 0, []
    for k in range(3):
        g = np.random.default_rng(500 + 10 * D + k)
        a = cpu.random_case(g, 23 + k, D, 60, run_hi=8, full=0.8)
        a[0][g.random(a[0].shape) < 0.05] = 101  # padding past d_valid may be anything; some tables out of domain
        out = run(tables, a, raw=True)
        check(a, out)
        evicted += int((out[2] >= 0).sum())
        rounds.append(int(out[5][0]))
        a = cpu.random_case(g, 17, D, 80, run_hi=6, full=0.9, bad_nodes=0.2)
        out = run(tables, a, raw=True)
        check(a, out)
    assert evicted >= 5 and max(rounds) >= 2, (evicted, rounds)


# ---- 3. nothing evictable: place_pods bit for bit --------------------------------------------------------------
def large(N, D, G, run_lo, run_hi, hi_pod, seed, evictable):
    g = np.random.default_rng(seed)
    a = cpu.random_case(g, N, D, G, run_hi=run_hi, hi_pod=hi_pod, evictable=evictable, full=0.5)
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("N,D,G,run_hi,hi_pod", [(5000, 8, 4096, 8, 4), (512, 64, 8192, 24, 8)])
def test_nothing_evictable_is_place_pods(N, D, G, run_hi, hi_pod, tables):
    a = large(N, D, G, 0, run_hi, hi_pod, N + G, evictable=False)
    args = cuda(*a)
    got = tables.preempt_pods(*args)
    exp = tables.place_pods(*args[:6])
    torch.cuda.synchronize()
    for x, y in zip(got[:2] + got[3:5], exp[:4]):
        assert torch.equal(x, y)
    assert (got[2] == -1).all() and torch.equal(got[5], exp[4])
    assert (got[0] >= 0).any() and got[5][0] >= 1


# ---- 4. contended calls, ragged tiles, 0 and 128 running pods --------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,D,G", [(9, 8, 300), (31, 4, 500), (61, 64, 200), (67, 33, 260), (3, 16, 150)])
def test_contended_and_ragged(N, D, G, tables):
    g = np.random.default_rng(N * 7 + G)
    a = cpu.random_case(g, N, D, G, run_hi=10, full=0.95)
    out = run(tables, a)
    check(a, out)
    invariants(a, out)
    assert out[5][0] >= 3 and (out[2] >= 0).any()


# running pods per node at every slot edge (a node's running pod h0 + lane + 32 i is slot i of the lane)
SLOT_EDGES = [1, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128]


@pytest.mark.gpu
@pytest.mark.parametrize("counts", [[0, 128, 128, 0, 5, 128], SLOT_EDGES], ids=["0_5_128", "slot_edges"])
@pytest.mark.parametrize("D", [8, 64])
def test_nodes_at_0_and_128_running_pods(D, counts, tables):
    """With SLOT_EDGES node n's running priorities are constant over h0 + [0, 16), [16, 48), [48, 80), [80, 112) and
    [112, 128), at (-2, 1, -1, 2, 0) rotated by n: the walk (priority descending, h ascending) jumps between slots,
    and each run of equal priorities but the first and last spans two slots."""
    g = np.random.default_rng(77 + D + (0 if counts[0] == 0 else 1000))
    N, G = len(counts), 120
    fc = np.zeros((N, D), np.int32)
    fm = np.zeros((N, D), np.int32)
    qc, qm, qd, roff, rprio = [], [], [], [0], []
    for n, k in enumerate(counts):
        left = np.full(D, 100)
        for h in range(k):
            d = h % D
            c = int(min(left[d], g.choice([1, 2, 5] if D == 8 else [20, 40])))  # 16 or 2 pods per device
            left[d] -= c
            qc.append(c)
            qm.append(0)
            qd.append(d)
            roff.append(roff[-1] + 1)
            rprio.append(int(g.integers(-3, 4)) if counts[0] == 0 else ((h + 16) // 32 * 3 + n) % 5 - 2)
        fc[n] = left // 4  # most of what the running pods leave is held by pods the caller does not list
        fm[n] = 1000
    noff = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    sizes = g.integers(1, 4, G)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    P = int(off[-1])
    a = [fc, fm, np.full(N, D, np.int32), g.choice([10, 40, 100], P).astype(np.int32), np.zeros(P, np.int32), off,
         g.integers(-2, 6, G).astype(np.int32), np.array(qc, np.int32), np.array(qm, np.int32), np.array(qd, np.int8),
         np.array(roff, np.int32), np.array(rprio, np.int32), noff]
    out = run(tables, a)
    check(a, out)
    invariants(a, out)
    run_node = np.repeat(np.arange(N), counts)
    if counts[0] == 0:
        assert (out[2][np.isin(run_node, [1, 2, 5])] >= 0).any() and (out[2] >= 0).sum() >= 5
    else:  # victims in every slot
        slot = (np.arange(run_node.size) - noff[run_node]) >> 5
        assert set(slot[out[2] >= 0].tolist()) == {0, 1, 2, 3}


# ---- 6. empty calls, inputs unchanged, repeat calls ------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,P,G,H", [(0, 16, 4, 0), (5, 0, 0, 2), (0, 0, 0, 0)])
def test_empty_calls(N, P, G, H, tables):
    z = dict(dtype=torch.int32, device="cuda")
    fc = torch.full((N, 4), 50, **z)
    fm = torch.full((N, 4), 700, **z)
    off = torch.arange(G + 1, **z) * (P // max(G, 1))
    noff = torch.full((N + 1,), H, **z)
    noff[0] = 0
    out = tables.preempt_pods(fc, fm, torch.full((N,), 4, **z), torch.zeros(P, **z), torch.zeros(P, **z), off,
                              torch.zeros(G, **z), torch.ones(H, **z), torch.zeros(H, **z),
                              torch.zeros(H, dtype=torch.int8, device="cuda"), torch.arange(H + 1, **z),
                              torch.zeros(H, **z), noff if N else torch.zeros(1, **z))
    node, dev, evicted, fco, fmo, info = out
    assert node.shape == (G,) and dev.shape == (P,) and evicted.shape == (H,) and fco.shape == (N, 4)
    assert (node == -1).all() and (dev == -1).all() and (evicted == -1).all()
    assert torch.equal(fco, fc) and torch.equal(fmo, fm) and info.tolist() == [0, 0, 0]


@pytest.mark.gpu
def test_inputs_unchanged_and_two_calls_bit_identical(tables):
    a = cpu.random_case(np.random.default_rng(17), 300, 16, 1500, run_hi=12, full=0.9)
    args = cuda(*a)
    first = tables.preempt_pods(*args)
    second = tables.preempt_pods(*args)
    torch.cuda.synchronize()
    for t, x in zip(args, a):
        np.testing.assert_array_equal(t.cpu().numpy(), x)
    for x, y in zip(first, second):
        assert torch.equal(x, y)
    assert first[5][0] >= 2 and (first[2] >= 0).any()


# ---- 7. CUDA graphs and torch.compile --------------------------------------------------------------------------
@pytest.mark.gpu
def test_cuda_graph_capture_and_replay(tables):
    N, D, G = 40, 16, 200
    a0 = cpu.random_case(np.random.default_rng(11), N, D, G, run_hi=6, full=0.9)
    st = cuda(*a0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        tables.preempt_pods(*st)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = tables.preempt_pods(*st)
    for seed in (12, 13):  # new values in place (same shapes), then replay
        ng = np.random.default_rng(seed)
        new = [x.copy() for x in a0]
        new[0] = np.minimum(a0[0], ng.integers(0, 101, a0[0].shape)).astype(np.int32)
        new[3] = ng.choice([5, 10, 25, 50, 100], a0[3].size).astype(np.int32)
        new[6] = ng.choice(cpu.PRIOS, G).astype(np.int32)
        new[11] = ng.choice(cpu.PRIOS[1:5], a0[11].size).astype(np.int32)
        for t, x in zip(st, new):
            t.copy_(torch.from_numpy(x))
        graph.replay()
        torch.cuda.synchronize()
        check(new, [t.cpu().numpy() for t in out])


@pytest.mark.gpu
def test_torch_compile_fullgraph(tables):
    a = cpu.random_case(np.random.default_rng(21), 19, 9, 90, full=0.9)
    out = torch.compile(tables.preempt_pods, fullgraph=True)(*cuda(*a))
    torch.cuda.synchronize()
    check(a, [t.cpu().numpy() for t in out])


# ---- 8. refusals, and bad offsets during capture ---------------------------------------------------------------
@pytest.mark.gpu
def test_refusals(tables):
    for exc, a, msg in cpu.refusal_cases("cuda")[:-1]:
        for fn in (tables.preempt_pods, torch.ops.egpu.preempt_pods):
            with pytest.raises(exc, match="preempt_pods: " + msg):
                cpu.call(fn, a)
    for key, value, msg in cpu.BAD_VALUES:  # the eager value checks
        a = cpu.cpu_args(device="cuda")
        a[key] = torch.tensor(value, dtype=a[key].dtype, device="cuda")
        with pytest.raises(ValueError, match="preempt_pods: .*" + msg):
            cpu.call(tables.preempt_pods, a)


LAUNCH_COUNT = r"""
import sys
sys.path[:0] = [{tests!r}, {root!r}]
import torch
from torch.profiler import ProfilerActivity, profile
import test_preempt_pods_cpu as c
from elastic_gpu_agent_b200 import tables
tables.load()

def launches(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "preempt_pods_kernel" in e.name)

def refuse_all():
    cases = [(exc, a) for exc, a, _ in c.refusal_cases("cuda")[:-1]]
    for key, value, _ in c.BAD_VALUES:
        a = c.cpu_args(device="cuda")
        a[key] = torch.tensor(value, dtype=a[key].dtype, device="cuda")
        cases.append((ValueError, a))
    for exc, a in cases:
        try:
            c.call(tables.preempt_pods, a)
        except exc:
            continue
        raise SystemExit("not refused")

print(launches(refuse_all), launches(lambda: c.call(tables.preempt_pods, c.cpu_args(device="cuda"))))
"""


@pytest.mark.gpu
def test_refusals_launch_nothing():
    import subprocess
    root = os.path.dirname(HERE)
    r = subprocess.run([sys.executable, "-c", LAUNCH_COUNT.format(tests=HERE, root=root)], capture_output=True,
                       text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.split() == ["0", "1"], r.stdout


BAD_OFFSETS = [  # (pod_offsets, run_offsets, node_offsets) with one of them bad; G = 4, H = 3, N = 3
    ([1, 3, 6, 9, 12], [0, 2, 3, 4], [0, 1, 3, 3]), ([0, 3, 6, 9, 13], [0, 2, 3, 4], [0, 1, 3, 3]),
    ([0, 3, 3, 9, 12], [0, 2, 3, 4], [0, 1, 3, 3]), ([0, 3, 6, 9, 12], [1, 2, 3, 4], [0, 1, 3, 3]),
    ([0, 3, 6, 9, 12], [0, 2, 3, 5], [0, 1, 3, 3]), ([0, 3, 6, 9, 12], [0, 2, 2, 4], [0, 1, 3, 3]),
    ([0, 3, 6, 9, 12], [0, 2, 3, 4], [1, 1, 3, 3]), ([0, 3, 6, 9, 12], [0, 2, 3, 4], [0, 1, 3, 2]),
    ([0, 3, 6, 9, 12], [0, 2, 3, 4], [0, 2, 1, 3]), ([0, 3, 6, 9, 12], [0, -2147483648, 3, 4], [0, 1, 3, 3]),
]


@pytest.mark.gpu
def test_bad_offsets_during_capture(tables):
    """The raw operator cannot read the offsets on the host; the kernel refuses them itself: nothing placed or evicted,
    the tables copied, info = [0, 0, 1].  Good offsets in the same graph place as eagerly."""
    fc = np.array([[0, 20], [10, 0], [100, 100]], np.int32)
    fm = np.full((3, 2), 1000, np.int32)
    good = [np.array(x, np.int32) for x in ([0, 3, 6, 9, 12], [0, 2, 3, 4], [0, 1, 3, 3])]
    a = [fc, fm, np.full(3, 2, np.int32), np.full(12, 10, np.int32), np.zeros(12, np.int32), good[0],
         np.array([5, 1, 9, 0], np.int32), np.array([40, 40, 90, 50], np.int32), np.zeros(4, np.int32),
         np.array([0, 1, 0, 1], np.int8), good[1], np.array([0, 2, 1], np.int32), good[2]]
    st = cuda(*a)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.ops.egpu.preempt_pods(*st)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = torch.ops.egpu.preempt_pods(*st)
    for bad in BAD_OFFSETS:
        for i, x in zip((5, 10, 12), bad):
            st[i].copy_(torch.tensor(x, dtype=torch.int32))
        graph.replay()
        torch.cuda.synchronize()
        node, dev, evicted, fco, fmo, info = [t.cpu().numpy() for t in out]
        assert (node == -1).all() and (dev == -1).all() and (evicted == -1).all(), bad
        np.testing.assert_array_equal(fco, fc)
        np.testing.assert_array_equal(fmo, fm)
        assert info.tolist() == [0, 0, 1], bad
    for i, x in zip((5, 10, 12), good):
        st[i].copy_(torch.from_numpy(x))
    graph.replay()
    torch.cuda.synchronize()
    check(a, [t.cpu().numpy() for t in out])
