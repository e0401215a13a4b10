"""egpu::place_gangs on the GPU (DESIGN.md §2.13): J gangs of pods placed on N capacity tables in gang order, each
kept when at least gang_min of its pods are placed and given back otherwise, in one cooperative launch.

  1. the known answers of tests/golden/place_gangs_kat.json, exactly;
  2. the numpy restatement at the D buckets and their edges, with mixed d_valid, out-of-domain padding, mixed gang
     sizes and gang_min, contended seeds;
  3. bit-identical to the loop of §2.13 written in torch around egpu::place_pods (torch.where keeps or drops each
     gang) at N = 5 000 x D = 8 and N = 512 x D = 64, with at most its round count; J = 1 is place_pods when every
     pod is placed.  Both sides run the same choose, commit and compact phases, so this checks the gang loop (the
     rounds of each gang, keeping and giving back), not the phases: tests/test_gpu_pods_scale.py checks those against
     the restatement past every block, stage, tile and grid threshold;
  4. the invariants (conservation of kept demand per device, rolled-back gangs all -1, placed in {0} or
     [gang_min, size], no -2, no grid wait that gave up);
  5. ragged tiles, empty calls, every pod out of the domain;
  6. inputs unchanged, and two calls bit-identical;
  7. CUDA-graph capture and replay on new inputs, torch.compile(fullgraph=True);
  8. refusals before any launch, and bad index tensors given to the raw operator during capture: nothing placed,
     tables copied, info[2] = 1.
"""
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import place_gangs_np as ref  # noqa: E402
import test_gpu_place_pods as gp  # noqa: E402  (pod builders of the place_pods tests)
import test_gpu_tables as gt  # noqa: E402  (random tables and requests of the bestfit_tables tests)

KAT = json.load(open(os.path.join(HERE, "golden", "place_gangs_kat.json")))["cases"]
KEYS = ("free_core", "free_mem", "d_valid", "req_core", "req_mem", "pod_offsets", "gang_offsets", "gang_min")


@pytest.fixture(scope="module")
def tables():
    from elastic_gpu_agent_b200 import tables as t
    t.load()
    return t


def cuda(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def run(tables, *a):
    out = tables.place_gangs(*cuda(*a))
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


def gangs(g, G, lo=1, hi=8, all_or_nothing=0.5):
    """gang_offsets and gang_min for G pods in gangs of lo to hi pods; a share all or nothing, the rest any min."""
    sizes, total = [], 0
    while total < G:
        s = min(int(g.integers(lo, hi + 1)), G - total)
        sizes.append(s)
        total += s
    sizes = np.array(sizes, np.int64)
    gmin = np.where(g.random(sizes.size) < all_or_nothing, sizes, g.integers(1, sizes + 1))
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32), gmin.astype(np.int32)


def check(a, out, rounds=None, exp=None):
    """Exactly the numpy restatement's placement, placed counts, tables and info (`exp`: its outputs, when already
    computed)."""
    exp = ref.place(*a) if exp is None else exp
    assert out[0].dtype == np.int32 and out[1].dtype == np.int8 and out[2].dtype == np.int32
    for x, y in zip(out[:5], exp[:5]):
        np.testing.assert_array_equal(x, y)
    assert out[5].tolist() == exp[5]
    if rounds is not None:
        rounds.append(int(out[5][0]))


def invariants(a, out):
    """What every answer must satisfy, whatever the reference says."""
    fc, fm, dv, rc, rm, off, goff, gmin = a
    node, dev, placed, fco, fmo, info = [np.asarray(x) for x in out]
    N, D = fc.shape
    assert info[1] == 0 and info[2] == 0 and not (node == -2).any() and not (dev == -2).any()
    size = np.diff(goff)
    assert ((placed == 0) | ((placed >= gmin) & (placed <= size))).all()
    gang_of = np.repeat(np.arange(size.size), size)
    for j in np.flatnonzero(placed == 0):  # a gang given back holds nothing
        assert (node[gang_of == j] == -1).all()
    np.testing.assert_array_equal(np.bincount(gang_of, weights=node >= 0, minlength=size.size), placed)
    pod_of = np.repeat(np.arange(node.size), np.diff(off))
    cnode = node[pod_of]
    assert ((cnode == -1) == (dev == -1)).all()  # all or nothing per pod
    valid = np.arange(D)[None, :] < dv[:, None]
    assert (fco[valid] >= 0).all() and (fmo[valid] >= 0).all()
    np.testing.assert_array_equal(fco[~valid], fc[~valid])
    kept = cnode >= 0
    n, d = cnode[kept].astype(np.int64), dev[kept].astype(np.int64)
    assert (d < dv[n]).all()
    used_c = np.zeros((N, D), np.int64)
    used_m = np.zeros((N, D), np.int64)
    np.add.at(used_c, (n, d), rc[kept])
    np.add.at(used_m, (n, d), rm[kept])
    np.testing.assert_array_equal(fc.astype(np.int64) - fco, used_c)  # free_in - free_out = kept demand, per device
    np.testing.assert_array_equal(fm.astype(np.int64) - fmo, used_m)
    assert (used_c >= 0).all() and (used_m >= 0).all()


def contended(g, N, D, G, hi_pod=4, hi_gang=8):
    fc, fm, dv = gt.random_tables(g, N, D)
    sizes = g.integers(1, hi_pod + 1, G)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    P = int(off[-1])
    rc = g.choice([5, 10, 25, 50, 100], P).astype(np.int32)
    rm = g.choice([0, 1024, 4096, 40_000], P).astype(np.int32)
    bad = g.random(P) < 0.02
    rc[bad] = g.choice([-1, 101, 1 << 30], int(bad.sum()))
    goff, gmin = gangs(g, G, 1, hi_gang)
    return [fc, fm, dv, rc, rm, off, goff, gmin]


def torch_loop(op, args, off_host, goff_host):
    """§2.13's rule written as a torch loop around place_pods (`op`: the raw operator or tables.place_pods): one
    call per gang on its containers and rebased pod offsets, kept or dropped with torch.where.  No host read of device
    data, so it captures into a CUDA graph.  Returns place_gangs' outputs, info = [summed rounds of place_pods, a wait
    gave up, 0]."""
    fc, fm, dv, rc, rm, off, goff, gmin = args
    G, J = off_host.size - 1, goff_host.size - 1
    node = torch.full((G,), -1, dtype=torch.int32, device=fc.device)
    dev = torch.full((rc.shape[0],), -1, dtype=torch.int8, device=fc.device)
    placed = torch.zeros(J, dtype=torch.int32, device=fc.device)
    info = torch.zeros(3, dtype=torch.int32, device=fc.device)
    minus1 = torch.full((), -1, dtype=torch.int32, device=fc.device)  # a fill, not a host copy: capturable
    for j in range(J):
        g0, g1 = int(goff_host[j]), int(goff_host[j + 1])
        c0, c1 = int(off_host[g0]), int(off_host[g1])
        r_node, r_dev, r_fc, r_fm, r_info = op(fc, fm, dv, rc[c0:c1], rm[c0:c1], off[g0:g1 + 1] - c0)
        k = (r_node >= 0).sum(dtype=torch.int32)
        keep = k >= gmin[j]
        node[g0:g1] = torch.where(keep, r_node, minus1)
        dev[c0:c1] = torch.where(keep, r_dev, minus1.to(torch.int8))
        placed[j] = torch.where(keep, k, 0)
        fc = torch.where(keep, r_fc, fc)
        fm = torch.where(keep, r_fm, fm)
        info[:2] += r_info[:2]
    return node, dev, placed, fc, fm, info


# ---- 1. known answers ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(KAT)))
def test_known_answers(case, tables):
    c = KAT[case]
    a = [np.array(c[k], np.int32) for k in KEYS]
    in_domain = all(ref.valid_devices(*a[:3]).any(axis=1))
    # the eager checks refuse a table outside the domain; the raw operator places around it
    out = tables.place_gangs(*cuda(*a)) if in_domain else torch.ops.egpu.place_gangs(*cuda(*a))
    node, dev, placed, fco, fmo, info = [t.cpu().numpy() for t in out]
    assert node.tolist() == c["node"] and dev.tolist() == c["dev"] and placed.tolist() == c["placed"], c["name"]
    assert fco.tolist() == c["free_core_out"] and fmo.tolist() == c["free_mem_out"], c["name"]
    assert info.tolist() == [c["rounds"], 0, 0], c["name"]


# ---- 2. the D buckets, contended -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 5, 8, 9, 16, 17, 32, 33, 64])
def test_restatement_at_the_d_buckets(D, tables):
    rounds, rolled = [], 0
    for k in range(2):
        g = np.random.default_rng(900 + 10 * D + k)
        fc, fm, dv = gt.random_tables(g, 37, D)
        rc, rm = gt.random_requests(g, 600, fc, fm)
        off = gp.pods(g, 600, 4)
        goff, gmin = gangs(g, off.size - 1)
        a = [fc, fm, dv, rc, rm, off, goff, gmin]
        out = run(tables, *a)
        check(a, out, rounds)
        invariants(a, out)
        a = contended(g, 13 + k, D, 200 + 17 * k)
        out = run(tables, *a)
        check(a, out, rounds)
        invariants(a, out)
        rolled += int((out[2] == 0).sum())
    assert rolled >= 1 and max(rounds) >= 10, (rolled, rounds)


# ---- 3./4. the probe's shapes: the torch loop around place_pods -------------------------------------------------
def large(N, D, G, J_lo, J_hi, hi_pod, seed):
    g = np.random.default_rng(seed)
    fc, fm, dv = gt.random_tables(g, N, D, pad=False)
    dv[:] = g.integers(max(1, D // 2), D + 1, N)
    sizes = g.integers(1, hi_pod + 1, G)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    P = int(off[-1])
    rc = g.integers(0, 101, P).astype(np.int32)
    rm = g.integers(0, 81_560, P).astype(np.int32)
    fc[fc == 100] = 99
    fc[: max(1, N // 50), 0] = 100  # few whole free cards ...
    rc[::4] = 100  # ... for a quarter of the containers: gangs that cannot all start are given back
    goff, gmin = gangs(g, G, J_lo, J_hi)
    return [fc, fm, dv, rc, rm, off, goff, gmin]


@pytest.mark.gpu
@pytest.mark.parametrize("N,D,G,hi_pod", [(5000, 8, 1024, 4), (512, 64, 2048, 8)])
def test_large_shapes_equal_the_torch_loop(N, D, G, hi_pod, tables):
    a = large(N, D, G, 1, 16, hi_pod, N + G)
    args = cuda(*a)
    got = tables.place_gangs(*args)
    exp = torch_loop(tables.place_pods, args, a[5], a[6])
    torch.cuda.synchronize()
    for x, y in zip(got[:5], exp[:5]):
        assert torch.equal(x, y)
    assert got[5][1:].tolist() == [0, 0] and 0 < got[5][0] <= exp[5][0]
    out = [t.cpu().numpy() for t in got]
    invariants(a, out)
    assert (out[2] == 0).any() and (out[2] > 0).any()  # some gangs given back, some kept


@pytest.mark.gpu
@pytest.mark.parametrize("N,D,P", [(5000, 8, 4096), (512, 64, 8192)])
def test_one_gang_is_place_pods_when_every_pod_is_placed(N, D, P, tables):
    g = np.random.default_rng(N + 3)
    fc, fm, dv = gt.random_tables(g, N, D, pad=False)
    fc[:] = 100
    fm[:] = 81_559
    off = gp.pods(g, P, 4)
    rc = g.integers(0, 20, P).astype(np.int32)
    rm = g.integers(0, 2000, P).astype(np.int32)
    G = off.size - 1
    args = cuda(fc, fm, dv, rc, rm, off)
    exp = tables.place_pods(*args)
    got = tables.place_gangs(*args, *cuda(np.array([0, G], np.int32), np.array([G], np.int32)))
    torch.cuda.synchronize()
    assert (exp[0] >= 0).all()
    for x, y in zip(got[:2] + got[3:5], exp[:4]):
        assert torch.equal(x, y)
    assert got[2].tolist() == [G] and got[5].tolist() == exp[4].tolist()


# ---- 5. ragged tiles, empty and out-of-domain calls ------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,D,G", [(517, 8, 1100), (523, 8, 257), (61, 64, 300), (67, 33, 700), (9, 16, 260)])
def test_ragged_tiles(N, D, G, tables):
    g = np.random.default_rng(N * 3 + G)
    a = contended(g, N, D, G, hi_gang=40)
    out = run(tables, *a)
    check(a, out)
    invariants(a, out)


@pytest.mark.gpu
@pytest.mark.parametrize("N,P,G,J", [(0, 16, 4, 2), (5, 0, 0, 0), (0, 0, 0, 0)])
def test_empty_calls(N, P, G, J, tables):
    z = dict(dtype=torch.int32, device="cuda")
    fc = torch.full((N, 4), 50, **z)
    fm = torch.full((N, 4), 700, **z)
    off = torch.arange(G + 1, **z) * (P // max(G, 1))
    goff = torch.arange(J + 1, **z) * (G // max(J, 1))
    node, dev, placed, fco, fmo, info = tables.place_gangs(fc, fm, torch.full((N,), 4, **z), torch.zeros(P, **z),
                                                           torch.zeros(P, **z), off, goff, torch.ones(J, **z))
    assert node.shape == (G,) and dev.shape == (P,) and placed.shape == (J,) and fco.shape == fmo.shape == (N, 4)
    assert (node == -1).all() and (dev == -1).all() and (placed == 0).all()
    assert torch.equal(fco, fc) and torch.equal(fmo, fm) and info.tolist() == [0, 0, 0]


@pytest.mark.gpu
def test_every_pod_out_of_the_domain(tables):
    g = np.random.default_rng(3)
    a = contended(g, 20, 8, 120)
    first = a[5][:-1]
    a[3][first] = g.choice([-1, 101, 1 << 30], first.size)  # one bad container per pod
    out = run(tables, *a)
    check(a, out)
    assert (out[0] == -1).all() and (out[1] == -1).all() and (out[2] == 0).all() and out[5].tolist() == [0, 0, 0]
    np.testing.assert_array_equal(out[3], a[0])


# ---- 6. inputs untouched, answers independent of timing --------------------------------------------------------
@pytest.mark.gpu
def test_inputs_unchanged_and_two_calls_bit_identical(tables):
    g = np.random.default_rng(17)
    a = contended(g, 300, 16, 2500, hi_gang=16)
    args = cuda(*a)
    first = tables.place_gangs(*args)
    second = tables.place_gangs(*args)
    torch.cuda.synchronize()
    for t, x in zip(args, a):
        np.testing.assert_array_equal(t.cpu().numpy(), x)
    for x, y in zip(first, second):
        assert torch.equal(x, y)
    assert first[5][0] >= 2 and (first[2] == 0).any()


# ---- 7. CUDA graphs and torch.compile --------------------------------------------------------------------------
@pytest.mark.gpu
def test_cuda_graph_capture_and_replay(tables):
    N, D, G = 40, 16, 300
    st = cuda(*contended(np.random.default_rng(11), N, D, G))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        tables.place_gangs(*st)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = tables.place_gangs(*st)
    P = st[3].shape[0]
    sizes, gsizes = np.diff(st[5].cpu().numpy()), np.diff(st[6].cpu().numpy())
    for seed in (12, 13):  # new inputs in place, pod and gang boundaries too (the same P, G and J), then replay
        ng = np.random.default_rng(seed)
        new = contended(ng, N, D, G)
        new[3] = ng.choice([5, 10, 25, 50, 100], P).astype(np.int32)
        new[4] = ng.choice([0, 1024, 40_000], P).astype(np.int32)
        new[5] = np.concatenate([[0], np.cumsum(ng.permutation(sizes))]).astype(np.int32)
        gs = ng.permutation(gsizes)
        new[6] = np.concatenate([[0], np.cumsum(gs)]).astype(np.int32)
        new[7] = ng.integers(1, gs + 1).astype(np.int32)
        for t, x in zip(st, new):
            t.copy_(torch.from_numpy(x))
        graph.replay()
        torch.cuda.synchronize()
        check(new, [t.cpu().numpy() for t in out])


@pytest.mark.gpu
def test_torch_compile_fullgraph(tables):
    a = contended(np.random.default_rng(21), 19, 9, 90)
    out = torch.compile(tables.place_gangs, fullgraph=True)(*cuda(*a))
    torch.cuda.synchronize()
    check(a, [t.cpu().numpy() for t in out])


# ---- 8. refusals, and bad index tensors during capture ---------------------------------------------------------
def good_args(N=6, D=8, P=12, G=4, J=2):
    z = dict(dtype=torch.int32, device="cuda")
    return dict(fc=torch.full((N, D), 50, **z), fm=torch.full((N, D), 1000, **z), dv=torch.full((N,), D, **z),
                rc=torch.full((P,), 10, **z), rm=torch.full((P,), 10, **z), off=torch.arange(G + 1, **z) * (P // G),
                goff=torch.arange(J + 1, **z) * (G // J), gmin=torch.ones(J, **z))


def refusal_cases():
    """(exception, arguments, refused by the raw operator too): the raw operator reads no data."""

    def with_(**kw):
        a = good_args()
        a.update(kw)
        return a

    def bad(key, at, v):
        a = good_args()
        a[key][at] = v
        return a

    z = dict(dtype=torch.int32, device="cuda")
    return [
        (RuntimeError, with_(fc=good_args()["fc"].to(torch.int64)), True),
        (RuntimeError, with_(dv=good_args()["dv"].cpu()), True),
        (ValueError, with_(fm=torch.full((6, 9), 1000, **z)), True),
        (RuntimeError, with_(off=good_args()["off"].to(torch.int64)), True),
        (ValueError, with_(off=torch.zeros(0, **z)), True),
        (RuntimeError, with_(goff=good_args()["goff"].to(torch.int64)), True),
        (RuntimeError, with_(gmin=good_args()["gmin"].to(torch.int16)), True),
        (RuntimeError, with_(goff=torch.arange(6, **z)[::2]), True),
        (RuntimeError, with_(goff=good_args()["goff"].cpu()), True),
        (RuntimeError, with_(gmin=good_args()["gmin"].cpu()), True),
        (ValueError, with_(goff=torch.zeros(0, **z)), True),
        (ValueError, with_(gmin=torch.ones(3, **z)), True),
        (ValueError, bad("fc", (2, 3), 101), False), (ValueError, bad("off", 4, 11), False),
        (ValueError, bad("goff", 0, 1), False), (ValueError, bad("goff", 2, 3), False),
        (ValueError, bad("goff", 1, 0), False), (ValueError, bad("gmin", 0, 0), False),
        (ValueError, bad("gmin", 1, 3), False),
    ]


def call(fn, a):
    return fn(a["fc"], a["fm"], a["dv"], a["rc"], a["rm"], a["off"], a["goff"], a["gmin"])


@pytest.mark.gpu
def test_refusals(tables):
    for exc, a, raw in refusal_cases():
        with pytest.raises(exc, match="place_gangs"):
            call(tables.place_gangs, a)
        if raw:
            with pytest.raises(exc, match="place_gangs"):
                call(torch.ops.egpu.place_gangs, a)


# Run in a process of its own: a profiler session here would share CUPTI's state with every later profiler
# session of the test process.
LAUNCH_COUNT = r"""
import sys
sys.path[:0] = [{tests!r}, {root!r}]
import torch
from torch.profiler import ProfilerActivity, profile
import test_gpu_place_gangs as t
from elastic_gpu_agent_b200 import tables
tables.load()

def launches(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "place_gangs_kernel" in e.name)

def refuse_all():
    for exc, a, raw in t.refusal_cases():
        for fn in (tables.place_gangs, torch.ops.egpu.place_gangs) if raw else (tables.place_gangs,):
            try:
                t.call(fn, a)
            except exc:
                continue
            raise SystemExit("not refused")

a = t.good_args()
print(launches(refuse_all), launches(lambda: t.call(tables.place_gangs, a)))
"""


@pytest.mark.gpu
def test_refusals_launch_nothing():
    """No place_gangs kernel in a profiler trace of every refusal; the profiler does see an accepted call's."""
    import subprocess
    root = os.path.dirname(HERE)
    r = subprocess.run([sys.executable, "-c", LAUNCH_COUNT.format(tests=HERE, root=root)], capture_output=True,
                       text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.split() == ["0", "1"], r.stdout


BAD_INDEX = [  # (pod_offsets, gang_offsets, gang_min) with one of them bad
    ([1, 3, 6, 9, 12], [0, 2, 4], [1, 1]), ([0, 3, 6, 9, 13], [0, 2, 4], [1, 1]), ([0, 3, 3, 9, 12], [0, 2, 4], [1, 1]),
    ([0, 3, 6, 9, 12], [1, 2, 4], [1, 1]), ([0, 3, 6, 9, 12], [0, 2, 3], [1, 1]), ([0, 3, 6, 9, 12], [0, 2, 5], [1, 1]),
    ([0, 3, 6, 9, 12], [0, 0, 4], [1, 1]), ([0, 3, 6, 9, 12], [0, 3, 1], [1, 1]),
    ([0, 3, 6, 9, 12], [0, -2147483648, 4], [1, 1]), ([0, 3, 6, 9, 12], [0, 2, 4], [0, 1]),
    ([0, 3, 6, 9, 12], [0, 2, 4], [1, 3]), ([0, 3, 6, 9, 12], [0, 2, 4], [-1, 2147483647]),
]


@pytest.mark.gpu
def test_bad_index_tensors_during_capture(tables):
    """The raw operator cannot read the index tensors on the host; the kernel refuses them itself: nothing placed,
    placed all 0, the tables copied, info = [0, 0, 1].  Good index tensors in the same graph place as eagerly."""
    g = np.random.default_rng(41)
    fc, fm, dv = gt.random_tables(g, 12, 8)
    rc, rm = g.choice([10, 25, 50], 12).astype(np.int32), np.zeros(12, np.int32)
    good = [np.array(x, np.int32) for x in ([0, 3, 6, 9, 12], [0, 2, 4], [2, 1])]
    st = cuda(fc, fm, dv, rc, rm, *good)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.ops.egpu.place_gangs(*st)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = torch.ops.egpu.place_gangs(*st)
    for idx in BAD_INDEX:
        for t, x in zip(st[5:], idx):
            t.copy_(torch.tensor(x, dtype=torch.int32))
        graph.replay()
        torch.cuda.synchronize()
        node, dev, placed, fco, fmo, info = [t.cpu().numpy() for t in out]
        assert (node == -1).all() and (dev == -1).all() and (placed == 0).all(), idx
        np.testing.assert_array_equal(fco, fc)
        np.testing.assert_array_equal(fmo, fm)
        assert info.tolist() == [0, 0, 1], idx
    for t, x in zip(st[5:], good):
        t.copy_(torch.from_numpy(x))
    graph.replay()
    torch.cuda.synchronize()
    check([fc, fm, dv, rc, rm, *good], [t.cpu().numpy() for t in out])
