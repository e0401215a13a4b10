"""egpu::place_pods on the GPU (DESIGN.md §2.12): G pods of P containers placed on N capacity tables, every container
of a pod on one node, by best-fit rounds to the fixed point in one cooperative launch.

  1. the known answers of tests/golden/place_pods_kat.json, exactly;
  2. the numpy restatement at the D buckets and their edges, with mixed d_valid, out-of-domain padding, pods of 1 to
     8 containers, and contended seeds, some of which run five rounds or more;
  3. pods of one container: bit-identical to egpu::place_tables at N = 5 000 x D = 8 x P = 4 096 and
     N = 512 x D = 64 x P = 8 192;
  4. at those shapes with pods of 1 to 8 containers: the restatement, and the invariants (all or nothing per pod,
     devices below d_valid, nothing negative, conservation per device, no -2, no grid wait that gave up; for pods
     of one container, where fit is monotone, a -1 pod fits no output table);
  5. ragged tiles, N = 0, P = 0, every pod out of the domain;
  6. inputs unchanged, and two calls bit-identical;
  7. CUDA-graph capture and replay on new inputs, torch.compile(fullgraph=True);
  8. refusals before any launch, and bad offsets given to the raw operator during capture: nothing placed, tables
     copied, info[2] = 1.
"""
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import place_pods_np as ref  # noqa: E402
import test_gpu_tables as gt  # noqa: E402  (random tables and requests of the bestfit_tables tests)

MEM_MAX = (1 << 18) - 1
KAT = json.load(open(os.path.join(HERE, "golden", "place_pods_kat.json")))["cases"]


@pytest.fixture(scope="module")
def tables():
    from elastic_gpu_agent_b200 import tables as t
    t.load()
    return t


def cuda(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def run(tables, fc, fm, dv, rc, rm, off):
    out = tables.place_pods(*cuda(fc, fm, dv, rc, rm, off))
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


def pods(g, P, hi=8):
    """pod_offsets for P containers in pods of 1 to `hi` containers."""
    sizes, total = [], 0
    while total < P:
        s = min(int(g.integers(1, hi + 1)), P - total)
        sizes.append(s)
        total += s
    return np.concatenate([[0], np.cumsum(sizes, dtype=np.int64)]).astype(np.int32)


def check(fc, fm, dv, rc, rm, off, out, rounds=None, exp=None):
    """Exactly the numpy restatement's placement, tables and info (`exp`: its outputs, when already computed)."""
    node, dev, fco, fmo, info = out
    e_node, e_dev, e_fc, e_fm, e_info = ref.place(fc, fm, dv, rc, rm, off) if exp is None else exp
    assert node.dtype == np.int32 and dev.dtype == np.int8
    np.testing.assert_array_equal(node, e_node)
    np.testing.assert_array_equal(dev, e_dev)
    np.testing.assert_array_equal(fco, e_fc)
    np.testing.assert_array_equal(fmo, e_fm)
    assert info.tolist() == e_info
    if rounds is not None:
        rounds.append(int(info[0]))


def invariants(fc, fm, dv, rc, rm, off, out):
    """What every answer must satisfy, whatever the reference says."""
    node, dev, fco, fmo, info = [np.asarray(x) for x in out]
    N, D = fc.shape
    assert info[1] == 0 and info[2] == 0 and not (node == -2).any() and not (dev == -2).any()
    pod_of = np.repeat(np.arange(node.size), np.diff(off))
    cnode = node[pod_of]  # each container's pod's node
    assert ((cnode == -1) == (dev == -1)).all()  # all or nothing per pod
    valid = np.arange(D)[None, :] < dv[:, None]
    assert (fco[valid] >= 0).all() and (fmo[valid] >= 0).all()
    np.testing.assert_array_equal(fco[~valid], fc[~valid])
    np.testing.assert_array_equal(fmo[~valid], fm[~valid])
    placed = cnode >= 0
    n, d = cnode[placed].astype(np.int64), dev[placed].astype(np.int64)
    assert (d < dv[n]).all()
    used_c = np.zeros((N, D), np.int64)
    used_m = np.zeros((N, D), np.int64)
    np.add.at(used_c, (n, d), rc[placed])
    np.add.at(used_m, (n, d), rm[placed])
    np.testing.assert_array_equal(fc.astype(np.int64) - fco, used_c)  # conservation per (n, d)
    np.testing.assert_array_equal(fm.astype(np.int64) - fmo, used_m)
    # fit is monotone for one container: a -1 pod of one container fits no valid device of any output table
    single = np.diff(off) == 1
    for gidx in np.flatnonzero(single & (node == -1)):
        c = off[gidx]
        fits = valid & (fco >= rc[c]) & (fmo >= rm[c]) & (rc[c] >= 0) & (rm[c] >= 0)
        assert not fits.any(), f"pod {gidx} is -1 but fits"


def contended(g, N, D, P, hi=8):
    """Tables of a few distinct values and pods whose containers collide on them: many rounds."""
    fc, fm, dv = gt.random_tables(g, N, D)
    rc = g.choice([5, 10, 25, 50, 100], P).astype(np.int32)
    rm = g.choice([0, 1024, 4096, 40_000], P).astype(np.int32)
    bad = g.random(P) < 0.03
    rc[bad] = g.choice([-1, 101, 1 << 30], int(bad.sum()))
    return fc, fm, dv, rc, rm, pods(g, P, hi)


# ---- 1. known answers ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(KAT)))
def test_known_answers(case, tables):
    c = KAT[case]
    a = [np.array(c[k], np.int32) for k in ("free_core", "free_mem", "d_valid", "req_core", "req_mem", "pod_offsets")]
    in_domain = all(ref.valid_devices(*a[:3]).any(axis=1))
    # the eager checks refuse a table outside the domain; the raw operator places around it
    out = tables.place_pods(*cuda(*a)) if in_domain else torch.ops.egpu.place_pods(*cuda(*a))
    node, dev, fco, fmo, info = [t.cpu().numpy() for t in out]
    assert node.tolist() == c["node"] and dev.tolist() == c["dev"], c["name"]
    assert fco.tolist() == c["free_core_out"] and fmo.tolist() == c["free_mem_out"], c["name"]
    assert info.tolist() == [c["rounds"], 0, 0], c["name"]


# ---- 2. the D buckets, contended -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 5, 8, 9, 16, 17, 32, 33, 64])
def test_restatement_at_the_d_buckets(D, tables):
    rounds = []
    for k in range(3):
        g = np.random.default_rng(500 + 10 * D + k)
        fc, fm, dv = gt.random_tables(g, 37, D)
        rc, rm = gt.random_requests(g, 700, fc, fm)
        off = pods(g, 700)
        out = run(tables, fc, fm, dv, rc, rm, off)
        check(fc, fm, dv, rc, rm, off, out, rounds)
        invariants(fc, fm, dv, rc, rm, off, out)
        a = contended(g, 13 + k, D, 900 + 33 * k)
        out = run(tables, *a)
        check(*a, out, rounds)
        invariants(*a, out)
    assert max(rounds) >= 5, rounds


# ---- 3./4. the probe's shapes: place_tables for one-container pods, the restatement for mixed pods --------------
def large(N, D, P):
    g = np.random.default_rng(N + P)
    fc, fm, dv = gt.random_tables(g, N, D, pad=False)
    dv[:] = g.integers(max(1, D // 2), D + 1, N)
    rc = g.integers(0, 101, P).astype(np.int32)
    rm = g.integers(0, 81_560, P).astype(np.int32)
    rc[::5] = 100  # whole cards: contention for the full devices
    return g, fc, fm, dv, rc, rm


@pytest.mark.gpu
@pytest.mark.parametrize("N,D,P", [(5000, 8, 4096), (512, 64, 8192)])
def test_single_container_pods_are_place_tables(N, D, P, tables):
    _, fc, fm, dv, rc, rm = large(N, D, P)
    args = cuda(fc, fm, dv, rc, rm)
    off = torch.arange(P + 1, dtype=torch.int32, device="cuda")
    got = tables.place_pods(*args, off)
    exp = tables.place_tables(*args)
    torch.cuda.synchronize()
    for x, y in zip(got[:4], exp[:4]):
        assert torch.equal(x, y)
    assert got[4].tolist() == exp[4].tolist() + [0] and got[4][0] >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("N,D,P", [(5000, 8, 4096), (512, 64, 8192)])
def test_large_shapes_with_mixed_pods(N, D, P, tables):
    g, fc, fm, dv, rc, rm = large(N, D, P)
    rc[::5] = 50  # two halves of a card in most pods
    off = pods(g, P)
    out = run(tables, fc, fm, dv, rc, rm, off)
    check(fc, fm, dv, rc, rm, off, out)
    invariants(fc, fm, dv, rc, rm, off, out)
    assert (out[0] >= 0).any() and out[4][0] >= 2


# ---- 5. ragged tiles, empty and out-of-domain calls ------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,D,P,hi", [(517, 8, 4100, 8), (523, 8, 2051, 1), (61, 64, 1032, 3), (67, 33, 3000, 8),
                                      (9, 16, 1025, 2)])
def test_ragged_tiles(N, D, P, hi, tables):
    g = np.random.default_rng(N * 3 + P)
    a = contended(g, N, D, P, hi)
    out = run(tables, *a)
    check(*a, out)
    invariants(*a, out)


@pytest.mark.gpu
@pytest.mark.parametrize("N,P,G", [(0, 16, 4), (5, 0, 0), (0, 0, 0)])
def test_empty_calls(N, P, G, tables):
    fc = torch.full((N, 4), 50, dtype=torch.int32, device="cuda")
    fm = torch.full((N, 4), 700, dtype=torch.int32, device="cuda")
    off = torch.arange(G + 1, dtype=torch.int32, device="cuda") * (P // max(G, 1))
    node, dev, fco, fmo, info = tables.place_pods(fc, fm, torch.full((N,), 4, dtype=torch.int32, device="cuda"),
                                                  torch.zeros(P, dtype=torch.int32, device="cuda"),
                                                  torch.zeros(P, dtype=torch.int32, device="cuda"), off)
    assert node.shape == (G,) and dev.shape == (P,) and fco.shape == fmo.shape == (N, 4)
    assert (node == -1).all() and (dev == -1).all() and torch.equal(fco, fc) and torch.equal(fmo, fm)
    assert info.tolist() == [0, 0, 0]


@pytest.mark.gpu
def test_every_pod_out_of_the_domain(tables):
    g = np.random.default_rng(3)
    fc, fm, dv = gt.random_tables(g, 20, 8)
    rc = g.integers(0, 50, 300).astype(np.int32)
    rm = g.integers(0, 1000, 300).astype(np.int32)
    off = pods(g, 300)
    first = off[:-1]
    rc[first] = g.choice([-1, 101, 1 << 30], first.size)  # one bad container per pod
    out = run(tables, fc, fm, dv, rc, rm, off)
    check(fc, fm, dv, rc, rm, off, out)
    assert (out[0] == -1).all() and (out[1] == -1).all() and out[4].tolist() == [0, 0, 0]


# ---- 6. inputs untouched, answers independent of timing --------------------------------------------------------
@pytest.mark.gpu
def test_inputs_unchanged_and_two_calls_bit_identical(tables):
    g = np.random.default_rng(17)
    a = contended(g, 300, 16, 6000)
    args = cuda(*a)
    first = tables.place_pods(*args)
    second = tables.place_pods(*args)
    torch.cuda.synchronize()
    for t, x in zip(args, a):
        np.testing.assert_array_equal(t.cpu().numpy(), x)
    for x, y in zip(first, second):
        assert torch.equal(x, y)
    assert first[4][0] >= 2


# ---- 7. CUDA graphs and torch.compile --------------------------------------------------------------------------
@pytest.mark.gpu
def test_cuda_graph_capture_and_replay(tables):
    N, D, P = 40, 16, 1024
    g = np.random.default_rng(11)
    st = cuda(*contended(g, N, D, P))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        tables.place_pods(*st)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = tables.place_pods(*st)
    sizes = np.diff(st[5].cpu().numpy())
    for seed in (12, 13):  # new inputs in place, pod boundaries too (the same G), then replay
        ng = np.random.default_rng(seed)
        new = list(contended(ng, N, D, P))
        new[5] = np.concatenate([[0], np.cumsum(ng.permutation(sizes))]).astype(np.int32)
        for t, x in zip(st, new):
            t.copy_(torch.from_numpy(x))
        graph.replay()
        torch.cuda.synchronize()
        check(*new, [t.cpu().numpy() for t in out])


@pytest.mark.gpu
def test_torch_compile_fullgraph(tables):
    g = np.random.default_rng(21)
    a = contended(g, 19, 9, 260)
    out = torch.compile(tables.place_pods, fullgraph=True)(*cuda(*a))
    torch.cuda.synchronize()
    check(*a, [t.cpu().numpy() for t in out])


# ---- 8. refusals, and bad offsets during capture ---------------------------------------------------------------
def good_args(N=6, D=8, P=12, G=4):
    return dict(fc=torch.full((N, D), 50, dtype=torch.int32, device="cuda"),
                fm=torch.full((N, D), 1000, dtype=torch.int32, device="cuda"),
                dv=torch.full((N,), D, dtype=torch.int32, device="cuda"),
                rc=torch.full((P,), 10, dtype=torch.int32, device="cuda"),
                rm=torch.full((P,), 10, dtype=torch.int32, device="cuda"),
                off=torch.arange(G + 1, dtype=torch.int32, device="cuda") * (P // G))


def refusal_cases(N=6, D=8, P=12):
    """(exception, arguments, refused by the raw operator too): the raw operator reads no data."""

    def with_(**kw):
        a = good_args(N, D, P)
        a.update(kw)
        return a

    def bad(key, at, v):
        a = good_args(N, D, P)
        a[key][at] = v
        return a

    z = dict(dtype=torch.int32, device="cuda")
    return [
        (RuntimeError, with_(fc=good_args()["fc"].to(torch.int64)), True),
        (RuntimeError, with_(rm=good_args()["rm"].to(torch.int16)), True),
        (RuntimeError, with_(fc=torch.full((D, N), 50, **z).t()), True),
        (RuntimeError, with_(dv=good_args()["dv"].cpu()), True),
        (ValueError, with_(fm=torch.full((N, D + 1), 1000, **z)), True),
        (ValueError, with_(rm=torch.zeros((P - 1,), **z)), True),
        (RuntimeError, with_(off=good_args()["off"].to(torch.int64)), True),
        (RuntimeError, with_(off=torch.arange(10, **z)[::2]), True),
        (RuntimeError, with_(off=good_args()["off"].cpu()), True),
        (ValueError, with_(off=torch.zeros(0, **z)), True),
        (ValueError, with_(off=torch.zeros((5, 1), **z)), True),
        (ValueError, bad("fc", (2, 3), 101), False), (ValueError, bad("dv", 1, 0), False),
        (ValueError, bad("off", 0, 1), False), (ValueError, bad("off", 4, 11), False),
        (ValueError, bad("off", 2, 3), False), (ValueError, bad("off", 2, 12), False),
    ]


def call(fn, a):
    return fn(a["fc"], a["fm"], a["dv"], a["rc"], a["rm"], a["off"])


@pytest.mark.gpu
def test_refusals(tables):
    for exc, a, raw in refusal_cases():
        with pytest.raises(exc, match="place_pods"):
            call(tables.place_pods, a)
        if raw:
            with pytest.raises(exc, match="place_pods"):
                call(torch.ops.egpu.place_pods, a)


# Run in a process of its own: a profiler session here would share CUPTI's state with every later profiler
# session of the test process.
LAUNCH_COUNT = r"""
import sys
sys.path[:0] = [{tests!r}, {root!r}]
import torch
from torch.profiler import ProfilerActivity, profile
import test_gpu_place_pods as t
from elastic_gpu_agent_b200 import tables
tables.load()

def launches(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "place_pods_kernel" in e.name)

def refuse_all():
    for exc, a, raw in t.refusal_cases():
        for fn in (tables.place_pods, torch.ops.egpu.place_pods) if raw else (tables.place_pods,):
            try:
                t.call(fn, a)
            except exc:
                continue
            raise SystemExit("not refused")

a = t.good_args()
print(launches(refuse_all), launches(lambda: t.call(tables.place_pods, a)))
"""


@pytest.mark.gpu
def test_refusals_launch_nothing():
    """No place_pods kernel in a profiler trace of every refusal; the profiler does see an accepted call's."""
    import subprocess
    root = os.path.dirname(HERE)
    r = subprocess.run([sys.executable, "-c", LAUNCH_COUNT.format(tests=HERE, root=root)], capture_output=True,
                       text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.split() == ["0", "1"], r.stdout


BAD_OFFSETS = [[1, 3, 6, 12], [0, 3, 6, 11], [0, 3, 6, 13], [0, 3, 3, 12], [0, 9, 10, 12], [0, 7, 3, 12],
               [0, -2147483648, 6, 12], [0, 2147483647, 6, 12], [-5, 3, 6, 12], [12, 3, 6, 12]]


@pytest.mark.gpu
def test_bad_offsets_during_capture(tables):
    """The raw operator cannot read the offsets on the host; the kernel refuses them itself: nothing placed, the
    tables copied, info = [0, 0, 1].  A good set of offsets in the same graph places as eagerly."""
    g = np.random.default_rng(41)
    fc, fm, dv, rc, rm = contended(g, 12, 8, 12)[:5]
    st = cuda(fc, fm, dv, rc, rm, np.array([0, 3, 6, 12], np.int32))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.ops.egpu.place_pods(*st)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = torch.ops.egpu.place_pods(*st)
    for off in BAD_OFFSETS:
        st[5].copy_(torch.tensor(off, dtype=torch.int32))
        graph.replay()
        torch.cuda.synchronize()
        node, dev, fco, fmo, info = [t.cpu().numpy() for t in out]
        assert (node == -1).all() and (dev == -1).all(), off
        np.testing.assert_array_equal(fco, fc)
        np.testing.assert_array_equal(fmo, fm)
        assert info.tolist() == [0, 0, 1], off
    good = np.array([0, 3, 6, 12], np.int32)
    st[5].copy_(torch.from_numpy(good))
    graph.replay()
    torch.cuda.synchronize()
    check(fc, fm, dv, rc, rm, good, [t.cpu().numpy() for t in out])
    # one pod of twelve containers is past MAX_POD: refused too
    st[5][:] = torch.tensor([0, 12, 12, 12], dtype=torch.int32)
    graph.replay()
    torch.cuda.synchronize()
    assert out[4].tolist() == [0, 0, 1]
