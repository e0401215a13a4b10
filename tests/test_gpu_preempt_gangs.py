"""egpu::preempt_gangs on the GPU (DESIGN.md §2.15): gangs placed in order on N capacity tables, each at its
priority with preempt_pods' evictions, kept or given back with its evictions, never cutting a running job below its
minimum, in one cooperative launch.

  1. the known answers of tests/golden/preempt_gangs_kat.json, exactly;
  2. the numpy restatement at the D buckets and their edges, with padding, inconsistent nodes and running jobs;
  3. bit-identical to place_gangs when no gang outranks a running pod, and to a torch loop of raw preempt_pods calls
     when there is no running job, at 5 000 x 8 and 512 x 64; one gang of minimum 1 against preempt_pods;
  4. contended and ragged calls with running jobs, nodes at 0 and 128 running pods;
  5. the invariants (jobs kept at their minimum, victims below their evictor's gang, kept gangs at their minimum and
     gangs given back evicting nothing, per device: input + evicted demand - placed demand = output);
  6. empty calls, inputs unchanged, two calls bit-identical;
  7. CUDA-graph capture and replay on new inputs, torch.compile(fullgraph=True);
  8. refusals before any launch, and each bad index tensor given to the raw operator during capture.
"""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import preempt_gangs_np as ref  # noqa: E402
import test_preempt_gangs_cpu as cpu  # noqa: E402  (random cases, argument builders, refusal cases)

KAT = cpu.KAT
INT32_MAX = 2**31 - 1


@pytest.fixture(scope="module")
def tables():
    from elastic_gpu_agent_b200 import tables as t
    t.load()
    return t


def cuda(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def run(tables, a, raw=False):
    fn = torch.ops.egpu.preempt_gangs if raw else tables.preempt_gangs
    out = fn(*cuda(*a))
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


def check(a, out, exp=None):
    """out equals the restatement's outputs exp (computed here when not given), info included."""
    exp = ref.place(*a) if exp is None else exp
    assert out[0].dtype == np.int32 and out[1].dtype == np.int8 and out[3].dtype == np.int32
    for x, y in zip(out[:6], exp[:6]):
        np.testing.assert_array_equal(x, y)
    assert out[6].tolist() == exp[6]
    return exp


def invariants(a, out):
    fc, fm, dv, rc, rm, off, goff, gmin, gprio, qc, qm, qd, roff, rprio, noff, rgang, rgmin = a
    node, dev, placed, evicted, fco, fmo, info = [np.asarray(x) for x in out]
    N, D = fc.shape
    assert info[1] == 0 and info[2] == 0 and not (node == -2).any() and not (dev == -2).any()
    pod_of = np.repeat(np.arange(node.size), np.diff(off))
    gang_of = np.repeat(np.arange(gmin.size), np.diff(goff))
    cnode = node[pod_of]
    assert ((cnode == -1) == (dev == -1)).all()
    kept = placed > 0
    assert (placed[kept] >= gmin[kept]).all() and (node[kept[gang_of] == False] == -1).all()  # noqa: E712
    assert np.array_equal(np.bincount(gang_of[node >= 0], minlength=gmin.size), placed)
    run_node = np.repeat(np.arange(N), np.diff(noff))
    gone = evicted >= 0
    assert kept[gang_of[evicted[gone]]].all()  # only kept gangs evict ...
    assert (node[evicted[gone]] == run_node[gone]).all()  # ... on their pods' nodes ...
    assert (rprio[gone] < gprio[gang_of[evicted[gone]]]).all()  # ... pods below their gang's priority
    alive0 = np.bincount(rgang[rgang >= 0], minlength=rgmin.size)
    lost = np.bincount(rgang[gone & (rgang >= 0)], minlength=rgmin.size)
    assert (lost <= np.maximum(alive0 - rgmin, 0)).all()  # a job at or above its minimum stays there
    delta_c = np.zeros((N, D), np.int64)
    delta_m = np.zeros((N, D), np.int64)
    rpod = np.repeat(np.arange(rprio.size), np.diff(roff))
    ev = gone[rpod] if rpod.size else np.zeros(0, bool)
    np.add.at(delta_c, (run_node[rpod[ev]], qd[ev].astype(np.int64)), qc[ev])
    np.add.at(delta_m, (run_node[rpod[ev]], qd[ev].astype(np.int64)), qm[ev])
    on = cnode >= 0
    np.subtract.at(delta_c, (cnode[on], dev[on].astype(np.int64)), rc[on])
    np.subtract.at(delta_m, (cnode[on], dev[on].astype(np.int64)), rm[on])
    np.testing.assert_array_equal(fc.astype(np.int64) + delta_c, fco)
    np.testing.assert_array_equal(fm.astype(np.int64) + delta_m, fmo)
    valid = np.arange(D)[None, :] < dv[:, None]
    assert (fco[valid] >= 0).all() and (fmo[valid] >= 0).all()


def torch_loop(args, off_h, goff, gmin, gprio):
    """§2.13's loop written with raw preempt_pods calls, one per gang, without a host round trip: each gang's result is
    kept with torch.where when at least gang_min pods are placed; a kept gang's victims stay listed with zero demand
    and priority INT32_MAX.  off_h (pod_offsets), goff, gmin, gprio are host arrays (the slices are shapes).
    Capturable.  Returns preempt_gangs' outputs, info[0] summing the calls' rounds."""
    fc, fm, dv, rc, rm, off, qc, qm, qd, roff, rprio, noff = args
    G, P, H, J = off.numel() - 1, rc.numel(), roff.numel() - 1, len(gmin)
    dev_ = fc.device
    node = torch.full((G,), -1, dtype=torch.int32, device=dev_)
    dv_out = torch.full((P,), -1, dtype=torch.int8, device=dev_)
    placed = torch.zeros(J, dtype=torch.int32, device=dev_)
    evicted = torch.full((H,), -1, dtype=torch.int32, device=dev_)
    rounds = torch.zeros((), dtype=torch.int32, device=dev_)
    run_pod = torch.repeat_interleave(torch.arange(H, device=dev_), roff[1:] - roff[:-1], output_size=qc.numel())
    qc, qm, rprio = qc.clone(), qm.clone(), rprio.clone()
    for j in range(J):
        g0, g1 = int(goff[j]), int(goff[j + 1])
        c0, c1 = int(off_h[g0]), int(off_h[g1])
        prio = torch.full((g1 - g0,), int(gprio[j]), dtype=torch.int32, device=dev_)
        n_, d_, e_, fc_, fm_, info = torch.ops.egpu.preempt_pods(fc, fm, dv, rc[c0:c1], rm[c0:c1], off[g0:g1 + 1] - c0,
                                                                 prio, qc, qm, qd, roff, rprio, noff)
        k = (n_ >= 0).sum().to(torch.int32)
        keep = k >= int(gmin[j])
        node[g0:g1] = torch.where(keep, n_, node[g0:g1])
        dv_out[c0:c1] = torch.where(keep, d_, dv_out[c0:c1])
        fc, fm = torch.where(keep, fc_, fc), torch.where(keep, fm_, fm)
        placed[j] = torch.where(keep, k, 0)
        ev = keep & (e_ >= 0)
        evicted = torch.where(ev, e_ + g0, evicted)
        gone = ev[run_pod]
        qc, qm = torch.where(gone, 0, qc), torch.where(gone, 0, qm)
        rprio = torch.where(ev, INT32_MAX, rprio)
        rounds = rounds + info[0]
    return node, dv_out, placed, evicted, fc, fm, rounds


# ---- 1. known answers ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(KAT)))
def test_known_answers(case, tables):
    c = KAT[case]
    out = run(tables, cpu.kat_args(c), raw=c["raw"])
    for k, x in zip(cpu.OUTS, out[:6]):
        assert x.tolist() == c[k], (c["name"], k)
    assert out[6].tolist() == c["info"], c["name"]


# ---- 2. the D buckets ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 5, 8, 9, 16, 17, 32, 33, 64])
def test_restatement_at_the_d_buckets(D, tables):
    evicted, given_back, rounds = 0, 0, []
    for k in range(3):
        g = np.random.default_rng(700 + 10 * D + k)
        a = cpu.random_case(g, 23 + k, D, 24, run_hi=8, full=0.8)
        a[0][g.random(a[0].shape) < 0.05] = 101  # padding past d_valid may be anything; some tables out of domain
        out = run(tables, a, raw=True)
        check(a, out)
        evicted += int((out[3] >= 0).sum())
        given_back += int((out[2] == 0).sum())
        rounds.append(int(out[6][0]))
        a = cpu.random_case(g, 17, D, 30, run_hi=6, full=0.9, bad_nodes=0.2)
        out = run(tables, a, raw=True)
        check(a, out)
    assert evicted >= 5 and given_back >= 1 and max(rounds) >= 20, (evicted, given_back, rounds)


# ---- 3. place_gangs, the torch loop of preempt_pods, and preempt_pods bit for bit ---------------------------------
def large(N, D, J, hi_gang, run_hi, hi_pod, seed, evictable, R=None):
    g = np.random.default_rng(seed)
    return cpu.random_case(g, N, D, J, run_hi=run_hi, hi_pod=hi_pod, hi_gang=hi_gang, evictable=evictable,
                           full=0.9, R=R)


SHAPES = [(5000, 8, 128, 16, 8, 4), (512, 64, 256, 8, 24, 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,D,J,hi_gang,run_hi,hi_pod", SHAPES)
def test_nothing_evictable_is_place_gangs(N, D, J, hi_gang, run_hi, hi_pod, tables):
    a = large(N, D, J, hi_gang, run_hi, hi_pod, N + J, evictable=False)
    args = cuda(*a)
    got = tables.preempt_gangs(*args)
    exp = tables.place_gangs(*args[:8])
    torch.cuda.synchronize()
    for x, y in zip(got[:3] + got[4:6], exp[:5]):
        assert torch.equal(x, y)
    assert (got[3] == -1).all() and torch.equal(got[6], exp[5])
    assert (got[2] > 0).any() and got[6][0] >= J


@pytest.mark.gpu
@pytest.mark.parametrize("N,D,J,hi_gang,run_hi,hi_pod", SHAPES)
def test_no_running_job_is_the_torch_loop(N, D, J, hi_gang, run_hi, hi_pod, tables):
    a = large(N, D, J, hi_gang, run_hi, hi_pod, 3 * N + J, evictable=True, R=0)
    args = cuda(*a)
    got = tables.preempt_gangs(*args)
    exp = torch_loop(args[:6] + args[9:15], a[5], a[6], a[7], a[8])
    torch.cuda.synchronize()
    for x, y in zip(got[:6], exp[:6]):
        assert torch.equal(x, y)
    assert int(got[6][0]) <= int(exp[6]) and got[6][1:].tolist() == [0, 0]
    assert (got[3] >= 0).sum() >= 10


@pytest.mark.gpu
@pytest.mark.parametrize("D", [8, 64])
def test_one_gang_of_minimum_1_is_preempt_pods(D, tables):
    g = np.random.default_rng(90 + D)
    a = cpu.random_case(g, 300 if D == 8 else 20, D, 1, hi_gang=400, run_hi=10, full=0.97, R=0)
    a[7][:] = 1
    args = cuda(*a)
    got = tables.preempt_gangs(*args)
    G = int(a[6][-1])
    prio = torch.full((G,), int(a[8][0]), dtype=torch.int32, device="cuda")
    exp = tables.preempt_pods(*args[:6], prio, *args[9:15])
    torch.cuda.synchronize()
    for x, y in zip(got[:2] + got[3:7], exp):
        assert torch.equal(x, y)
    assert int(got[2][0]) == int((exp[0] >= 0).sum()) and (got[3] >= 0).any()


# ---- 4. contended calls with running jobs, ragged tiles, 0 and 128 running pods ---------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,D,J", [(9, 8, 60), (31, 4, 90), (11, 64, 80), (67, 33, 50), (3, 16, 40)])
def test_contended_and_ragged(N, D, J, tables):
    g = np.random.default_rng(N * 7 + J)
    a = cpu.random_case(g, N, D, J, run_hi=10, full=0.95)
    out = run(tables, a)
    check(a, out)
    invariants(a, out)
    assert out[6][0] >= J and (out[3] >= 0).any()


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
    N, J = len(counts), 40
    fc = np.zeros((N, D), np.int32)
    fm = np.zeros((N, D), np.int32)
    qc, qm, qd, roff, rprio = [], [], [], [0], []
    for n, k in enumerate(counts):
        left = np.full(D, 100)
        for h in range(k):
            d = h % D
            c = int(min(left[d], g.choice([1, 2, 5] if D == 8 else [20, 40])))
            left[d] -= c
            qc.append(c)
            qm.append(0)
            qd.append(d)
            roff.append(roff[-1] + 1)
            rprio.append(int(g.integers(-3, 4)) if counts[0] == 0 else ((h + 16) // 32 * 3 + n) % 5 - 2)
        fc[n] = left // 4
        fm[n] = 1000
    noff = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    H = len(rprio)
    R = 12
    rgang = np.where(g.random(H) < 0.3, -1, g.integers(0, R, H)).astype(np.int32)
    rgmin = g.integers(0, np.bincount(rgang[rgang >= 0], minlength=R) + 1).astype(np.int32)
    gsz = g.integers(1, 5, J)
    goff = np.concatenate([[0], np.cumsum(gsz)]).astype(np.int32)
    G = int(goff[-1])
    sizes = g.integers(1, 4, G)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    P = int(off[-1])
    a = [fc, fm, np.full(N, D, np.int32), g.choice([10, 40, 100], P).astype(np.int32), np.zeros(P, np.int32), off,
         goff, g.integers(1, gsz + 1).astype(np.int32), g.integers(-2, 6, J).astype(np.int32), np.array(qc, np.int32),
         np.array(qm, np.int32), np.array(qd, np.int8), np.array(roff, np.int32), np.array(rprio, np.int32), noff,
         rgang, rgmin]
    out = run(tables, a)
    check(a, out)
    invariants(a, out)
    run_node = np.repeat(np.arange(N), counts)
    if counts[0] == 0:
        assert (out[3][np.isin(run_node, [1, 2, 5])] >= 0).any() and (out[3] >= 0).sum() >= 5
    else:  # victims in every slot
        slot = (np.arange(run_node.size) - noff[run_node]) >> 5
        assert set(slot[out[3] >= 0].tolist()) == {0, 1, 2, 3}


# ---- 6. empty calls, inputs unchanged, repeat calls ------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,P,G,H", [(0, 16, 4, 0), (5, 0, 0, 2), (0, 0, 0, 0)])
def test_empty_calls(N, P, G, H, tables):
    z = dict(dtype=torch.int32, device="cuda")
    fc = torch.full((N, 4), 50, **z)
    fm = torch.full((N, 4), 700, **z)
    off = torch.arange(G + 1, **z) * (P // max(G, 1))
    J = 1 if G else 0
    goff = torch.tensor([0, G] if G else [0], **z)
    noff = torch.full((N + 1,), H, **z)
    noff[0] = 0
    out = tables.preempt_gangs(fc, fm, torch.full((N,), 4, **z), torch.zeros(P, **z), torch.zeros(P, **z), off, goff,
                               torch.ones(J, **z), torch.zeros(J, **z), torch.ones(H, **z), torch.zeros(H, **z),
                               torch.zeros(H, dtype=torch.int8, device="cuda"), torch.arange(H + 1, **z),
                               torch.zeros(H, **z), noff if N else torch.zeros(1, **z), torch.zeros(H, **z),
                               torch.zeros(1, **z))
    node, dev, placed, evicted, fco, fmo, info = out
    assert node.shape == (G,) and dev.shape == (P,) and placed.shape == (J,) and evicted.shape == (H,)
    assert (node == -1).all() and (dev == -1).all() and (placed == 0).all() and (evicted == -1).all()
    assert torch.equal(fco, fc) and torch.equal(fmo, fm) and info.tolist() == [0, 0, 0]


@pytest.mark.gpu
def test_inputs_unchanged_and_two_calls_bit_identical(tables):
    a = cpu.random_case(np.random.default_rng(17), 300, 16, 400, run_hi=12, full=0.9)
    args = cuda(*a)
    first = tables.preempt_gangs(*args)
    second = tables.preempt_gangs(*args)
    torch.cuda.synchronize()
    for t, x in zip(args, a):
        np.testing.assert_array_equal(t.cpu().numpy(), x)
    for x, y in zip(first, second):
        assert torch.equal(x, y)
    assert first[6][0] >= 2 and (first[3] >= 0).any()


# ---- 7. CUDA graphs and torch.compile --------------------------------------------------------------------------
@pytest.mark.gpu
def test_cuda_graph_capture_and_replay(tables):
    N, D, J = 40, 16, 60
    a0 = cpu.random_case(np.random.default_rng(11), N, D, J, run_hi=6, full=0.9)
    st = cuda(*a0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        tables.preempt_gangs(*st)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = tables.preempt_gangs(*st)
    for seed in (12, 13):  # new values in place (same shapes), then replay
        ng = np.random.default_rng(seed)
        new = [x.copy() for x in a0]
        new[0] = np.minimum(a0[0], ng.integers(0, 101, a0[0].shape)).astype(np.int32)
        new[3] = ng.choice([5, 10, 25, 50, 100], a0[3].size).astype(np.int32)
        new[8] = ng.choice(cpu.pods.PRIOS, J).astype(np.int32)
        new[13] = ng.choice(cpu.pods.PRIOS[1:5], a0[13].size).astype(np.int32)
        new[16] = ng.integers(0, 3, a0[16].size).astype(np.int32)
        for t, x in zip(st, new):
            t.copy_(torch.from_numpy(x))
        graph.replay()
        torch.cuda.synchronize()
        check(new, [t.cpu().numpy() for t in out])


@pytest.mark.gpu
def test_torch_compile_fullgraph(tables):
    a = cpu.random_case(np.random.default_rng(21), 19, 9, 30, full=0.9)
    out = torch.compile(tables.preempt_gangs, fullgraph=True)(*cuda(*a))
    torch.cuda.synchronize()
    check(a, [t.cpu().numpy() for t in out])


# ---- 8. refusals, and bad index tensors during capture ---------------------------------------------------------
@pytest.mark.gpu
def test_refusals(tables):
    for exc, a, msg in cpu.refusal_cases("cuda")[:-1]:
        for fn in (tables.preempt_gangs, torch.ops.egpu.preempt_gangs):
            with pytest.raises(exc, match="preempt_gangs: " + msg):
                cpu.call(fn, a)
    for key, value, msg in cpu.BAD_VALUES:  # the eager value checks
        a = cpu.cpu_args(device="cuda")
        a[key] = torch.tensor(value, dtype=torch.int32, device="cuda")
        with pytest.raises(ValueError, match="preempt_gangs: .*" + msg):
            cpu.call(tables.preempt_gangs, a)


LAUNCH_COUNT = r"""
import sys
sys.path[:0] = [{tests!r}, {root!r}]
import torch
from torch.profiler import ProfilerActivity, profile
import test_preempt_gangs_cpu as c
from elastic_gpu_agent_b200 import tables
tables.load()

def launches(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "preempt_gangs_kernel" in e.name)

def refuse_all():
    cases = [(exc, a) for exc, a, _ in c.refusal_cases("cuda")[:-1]]
    for key, value, _ in c.BAD_VALUES:
        a = c.cpu_args(device="cuda")
        a[key] = torch.tensor(value, dtype=torch.int32, device="cuda")
        cases.append((ValueError, a))
    for exc, a in cases:
        try:
            c.call(tables.preempt_gangs, a)
        except exc:
            continue
        raise SystemExit("not refused")

print(launches(refuse_all), launches(lambda: c.call(tables.preempt_gangs, c.cpu_args(device="cuda"))))
"""


@pytest.mark.gpu
def test_refusals_launch_nothing():
    import subprocess
    root = os.path.dirname(HERE)
    r = subprocess.run([sys.executable, "-c", LAUNCH_COUNT.format(tests=HERE, root=root)], capture_output=True,
                       text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.split() == ["0", "1"], r.stdout


# (index, bad value): pod_offsets 5, gang_offsets 6, gang_min 7, run_offsets 12, node_offsets 14, run_gang 15,
# run_gang_min 16; G = 4, J = 2, H = 3, N = 3, R = 2
BAD_INDEX = [
    (5, [1, 3, 6, 9, 12]), (5, [0, 3, 3, 9, 12]), (5, [0, 3, 6, 9, 13]),
    (6, [1, 2, 4]), (6, [0, 2, 5]), (6, [0, 0, 4]), (7, [0, 1]), (7, [3, 1]),
    (12, [1, 2, 3, 4]), (12, [0, 2, 2, 4]), (12, [0, -2147483648, 3, 4]),
    (14, [1, 1, 3, 3]), (14, [0, 2, 1, 3]), (14, [0, 1, 3, 2]),
    (15, [0, 2, -1]), (15, [-2, 0, 1]), (16, [1, -1]),
]


@pytest.mark.gpu
def test_bad_index_tensors_during_capture(tables):
    """The raw operator cannot read the index tensors on the host; the kernel refuses them itself: nothing placed or
    evicted, the tables copied, info = [0, 0, 1].  Good tensors in the same graph place as eagerly."""
    fc = np.array([[0, 20], [10, 0], [100, 100]], np.int32)
    fm = np.full((3, 2), 1000, np.int32)
    a = [fc, fm, np.full(3, 2, np.int32), np.full(12, 10, np.int32), np.zeros(12, np.int32),
         np.array([0, 3, 6, 9, 12], np.int32), np.array([0, 2, 4], np.int32), np.array([1, 2], np.int32),
         np.array([5, 9], np.int32), np.array([40, 40, 90, 50], np.int32), np.zeros(4, np.int32),
         np.array([0, 1, 0, 1], np.int8), np.array([0, 2, 3, 4], np.int32), np.array([0, 2, 1], np.int32),
         np.array([0, 1, 3, 3], np.int32), np.array([0, 1, 0], np.int32), np.array([1, 0], np.int32)]
    st = cuda(*a)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.ops.egpu.preempt_gangs(*st)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = torch.ops.egpu.preempt_gangs(*st)
    for i, bad in BAD_INDEX:
        st[i].copy_(torch.tensor(bad, dtype=torch.int32))
        graph.replay()
        torch.cuda.synchronize()
        node, dev, placed, evicted, fco, fmo, info = [t.cpu().numpy() for t in out]
        assert (node == -1).all() and (dev == -1).all() and (placed == 0).all() and (evicted == -1).all(), (i, bad)
        np.testing.assert_array_equal(fco, fc)
        np.testing.assert_array_equal(fmo, fm)
        assert info.tolist() == [0, 0, 1], (i, bad)
        st[i].copy_(torch.from_numpy(a[i]))
    graph.replay()
    torch.cuda.synchronize()
    check(a, [t.cpu().numpy() for t in out])
