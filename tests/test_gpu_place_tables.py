"""egpu::place_tables on the GPU (DESIGN.md §2.11): P requests placed on N capacity tables by best-fit rounds to the
fixed point, in one cooperative launch.

  1. the known answers of tests/golden/place_tables_kat.json, exactly;
  2. at most 64 valid devices in all: equal to oracle/bestfit_np.rounds on the concatenated table, and to the
     context's one-launch rounds (egpu_bestfit_batch_dev with EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT | EGPU_F_ROUNDS |
     EGPU_F_DEVICE_ROUNDS) on that table;
  3. the numpy restatement at the D buckets and their edges, with mixed d_valid and out-of-domain padding, which
     comes back unchanged; contended seeds, some of which run five rounds or more;
  4. N = 5 000 x D = 8 x P = 4 096 and N = 512 x D = 64 x P = 8 192: equal to the torch loop around bestfit_tables,
     and the invariants (nothing negative, conservation per device, -1 rows fit nowhere, placements on valid
     devices, no -2, no grid wait that gave up);
  5. ragged tiles, the scalar form (P % 4 != 0, unaligned views), N = 0, P = 0, every request out of the domain;
  6. inputs unchanged, and two calls bit-identical;
  7. CUDA-graph capture and replay on new inputs, torch.compile(fullgraph=True);
  8. refusals before any launch, and the raw operator during capture with a table outside the domain.
"""
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import place_tables_np as ref  # noqa: E402
import test_gpu_tables as gt  # noqa: E402  (random tables and requests of the bestfit_tables tests)

from oracle import bestfit_np  # noqa: E402

MEM_MAX = (1 << 18) - 1
KAT = json.load(open(os.path.join(HERE, "golden", "place_tables_kat.json")))["cases"]


@pytest.fixture(scope="module")
def tables():
    from elastic_gpu_agent_b200 import tables as t
    t.load()
    return t


def cuda(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def run(tables, fc, fm, dv, rc, rm):
    out = tables.place_tables(*cuda(fc, fm, dv, rc, rm))
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


def check(fc, fm, dv, rc, rm, out, rounds=None):
    """Exactly the numpy restatement's placement, tables and rounds; info[1] == 0."""
    node, dev, fco, fmo, info = out
    e_node, e_dev, e_fc, e_fm, e_rounds = ref.place(fc, fm, dv, rc, rm)
    assert node.dtype == np.int32 and dev.dtype == np.int8 and info.tolist()[1] == 0
    np.testing.assert_array_equal(node, e_node)
    np.testing.assert_array_equal(dev, e_dev)
    np.testing.assert_array_equal(fco, e_fc)
    np.testing.assert_array_equal(fmo, e_fm)
    assert info[0] == e_rounds
    if rounds is not None:
        rounds.append(int(info[0]))


def invariants(fc, fm, dv, rc, rm, out):
    """What every answer must satisfy, whatever the reference says."""
    node, dev, fco, fmo, info = [np.asarray(x) for x in out]
    N, D = fc.shape
    assert info[1] == 0 and not (node == -2).any() and not (dev == -2).any()
    assert ((node == -1) == (dev == -1)).all()
    valid = np.arange(D)[None, :] < dv[:, None]
    assert (fco[valid] >= 0).all() and (fmo[valid] >= 0).all()
    np.testing.assert_array_equal(fco[~valid], fc[~valid])
    np.testing.assert_array_equal(fmo[~valid], fm[~valid])
    placed = node >= 0
    n, d = node[placed].astype(np.int64), dev[placed].astype(np.int64)
    assert (d < dv[n]).all()
    used_c = np.zeros((N, D), np.int64)
    used_m = np.zeros((N, D), np.int64)
    np.add.at(used_c, (n, d), rc[placed])
    np.add.at(used_m, (n, d), rm[placed])
    np.testing.assert_array_equal(fc.astype(np.int64) - fco, used_c)  # conservation per (n, d)
    np.testing.assert_array_equal(fm.astype(np.int64) - fmo, used_m)
    # a -1 row fits on no valid device of any output table
    for p in np.flatnonzero(~placed):
        fits = valid & (fco >= rc[p]) & (fmo >= rm[p]) & (rc[p] >= 0) & (rm[p] >= 0)
        assert not fits.any(), f"row {p} is -1 but fits"


# ---- 1. known answers ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(KAT)))
def test_known_answers(case, tables):
    c = KAT[case]
    node, dev, fco, fmo, info = run(tables, *[np.array(c[k], np.int32) for k in
                                              ("free_core", "free_mem", "d_valid", "req_core", "req_mem")])
    assert node.tolist() == c["node"] and dev.tolist() == c["dev"], c["name"]
    assert fco.tolist() == c["free_core_out"] and fmo.tolist() == c["free_mem_out"], c["name"]
    assert info.tolist() == [c["rounds"], 0], c["name"]


# ---- 2. the concatenated table: the rounds oracle and the context's one-launch rounds ---------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(12))
def test_equals_single_table_rounds_on_the_concatenation(seed, tables, alloc):
    g = np.random.default_rng(700 + seed)
    N = int(g.integers(1, 9))
    D = int(g.integers(1, 64 // N + 1))
    fc = g.choice([0, 10, 25, 50, 100], (N, D)).astype(np.int32)
    fm = g.choice([0, 1024, 8192, 81_559], (N, D)).astype(np.int32)
    dv = g.integers(1, D + 1, N).astype(np.int32)
    past = np.arange(D)[None, :] >= dv[:, None]
    fc[past], fm[past] = 101, -1
    P = int(g.integers(1, 3000))
    rc = g.choice([5, 10, 25, 50], P).astype(np.int32)
    rm = g.choice([0, 512, 1024, 4096], P).astype(np.int32)
    out = run(tables, fc, fm, dv, rc, rm)
    check(fc, fm, dv, rc, rm, out)
    node, dev, fco, fmo, info = out
    offset = np.concatenate([[0], np.cumsum(dv)[:-1]])
    cat_c = np.concatenate([fc[n, :dv[n]] for n in range(N)])
    cat_m = np.concatenate([fm[n, :dv[n]] for n in range(N)])
    flat = np.where(node >= 0, offset[np.maximum(node, 0)] + dev, -1)
    o_idx, _, _, o_fc, o_fm, o_rounds, _ = bestfit_np.rounds(cat_c, cat_m, rc, rm)
    np.testing.assert_array_equal(flat, o_idx)
    assert info[0] == o_rounds
    got_c = np.concatenate([fco[n, :dv[n]] for n in range(N)])
    got_m = np.concatenate([fmo[n, :dv[n]] for n in range(N)])
    np.testing.assert_array_equal(got_c, o_fc)
    np.testing.assert_array_equal(got_m, o_fm)
    # the context's rounds in one launch, on the concatenated table
    alloc.set_table(cat_c, cat_m)
    d_rc, d_rm = cuda(rc, rm)
    d_idx = torch.full((P,), -9, dtype=torch.int32, device="cuda")
    d_tab = torch.full((3 * cat_c.size,), -7, dtype=torch.int32, device="cuda")
    alloc.bestfit_rounds_device_dev(d_rc.data_ptr(), d_rm.data_ptr(), P, d_idx.data_ptr(), 0, d_tab.data_ptr(),
                                    torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(d_idx.cpu().numpy(), flat)
    tab = d_tab.cpu().numpy()
    np.testing.assert_array_equal(tab[:cat_c.size], got_c)
    np.testing.assert_array_equal(tab[cat_c.size:2 * cat_c.size], got_m)


# ---- 3. the D buckets, contended -------------------------------------------------------------------------------
def contended(g, N, D, P):
    """Tables of a few distinct values and requests that collide on them: many rounds."""
    fc, fm, dv = gt.random_tables(g, N, D)
    rc = g.choice([5, 10, 25, 50, 100], P).astype(np.int32)
    rm = g.choice([0, 1024, 4096, 40_000], P).astype(np.int32)
    bad = g.random(P) < 0.03
    rc[bad] = g.choice([-1, 101, 1 << 30], int(bad.sum()))
    return fc, fm, dv, rc, rm


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 5, 8, 9, 16, 17, 32, 33, 64])
def test_restatement_at_the_d_buckets(D, tables):
    rounds = []
    for k in range(3):
        g = np.random.default_rng(300 + 10 * D + k)
        fc, fm, dv = gt.random_tables(g, 37, D)
        rc, rm = gt.random_requests(g, 516, fc, fm)
        check(fc, fm, dv, rc, rm, run(tables, fc, fm, dv, rc, rm), rounds)
        fc, fm, dv, rc, rm = contended(g, 13 + k, D, 700 + 33 * k)
        out = run(tables, fc, fm, dv, rc, rm)
        check(fc, fm, dv, rc, rm, out, rounds)
        invariants(fc, fm, dv, rc, rm, out)
    assert max(rounds) >= 5, rounds


# ---- 4. the probe's shapes against the torch loop --------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,D,P", [(5000, 8, 4096), (512, 64, 8192)])
def test_large_shapes_equal_the_torch_loop(N, D, P, tables):
    g = np.random.default_rng(N + P)
    fc, fm, dv = gt.random_tables(g, N, D, pad=False)
    dv[:] = g.integers(max(1, D // 2), D + 1, N)
    rc = g.integers(0, 101, P).astype(np.int32)
    rm = g.integers(0, 81_560, P).astype(np.int32)
    rc[::5] = 100  # whole cards: contention for the full devices
    args = cuda(fc, fm, dv, rc, rm)
    out = tables.place_tables(*args)
    e_node, e_dev, e_fc, e_fm, e_rounds = ref.place_torch(*args)
    torch.cuda.synchronize()
    got = [t.cpu().numpy() for t in out]
    for a, b in zip(got[:4], (e_node, e_dev, e_fc, e_fm)):
        np.testing.assert_array_equal(a, b.cpu().numpy())
    assert got[4][0] == e_rounds
    invariants(fc, fm, dv, rc, rm, got)
    assert (got[0] >= 0).any() and got[4][0] >= 2  # the whole cards collide


# ---- 5. ragged tiles, the scalar form, empty and out-of-domain calls -------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,D,P,offset", [(517, 8, 4100, 0),   # vector form, ragged last tile and chunk
                                          (523, 8, 2051, 0),   # scalar form: P % 4 != 0
                                          (61, 64, 1032, 1),   # scalar form: requests not 16-byte aligned
                                          (67, 33, 3000, 2),   # scalar form, D = 64's bucket
                                          (9, 16, 1025, 0)])   # scalar form, a chunk of one row
def test_ragged_tiles_and_the_scalar_form(N, D, P, offset, tables):
    g = np.random.default_rng(N * 3 + P)
    fc, fm, dv, rc, rm = contended(g, N, D, P)
    cu = cuda(fc, fm, dv)
    rq = []
    for a in (rc, rm):  # a contiguous view that starts `offset` elements into its storage
        buf = torch.zeros(P + offset, dtype=torch.int32, device="cuda")
        buf[offset:] = torch.from_numpy(a).cuda()
        rq.append(buf[offset:])
    out = [t.cpu().numpy() for t in tables.place_tables(*cu, *rq)]
    check(fc, fm, dv, rc, rm, out)
    invariants(fc, fm, dv, rc, rm, out)


@pytest.mark.gpu
@pytest.mark.parametrize("N,P", [(0, 16), (5, 0), (0, 0)])
def test_empty_calls(N, P, tables):
    fc = torch.full((N, 4), 50, dtype=torch.int32, device="cuda")
    fm = torch.full((N, 4), 700, dtype=torch.int32, device="cuda")
    node, dev, fco, fmo, info = tables.place_tables(fc, fm, torch.full((N,), 4, dtype=torch.int32, device="cuda"),
                                                    torch.zeros(P, dtype=torch.int32, device="cuda"),
                                                    torch.zeros(P, dtype=torch.int32, device="cuda"))
    assert node.shape == dev.shape == (P,) and fco.shape == fmo.shape == (N, 4)
    assert (node == -1).all() and (dev == -1).all() and torch.equal(fco, fc) and torch.equal(fmo, fm)
    assert info.tolist() == [0, 0]


@pytest.mark.gpu
def test_every_request_out_of_the_domain(tables):
    g = np.random.default_rng(3)
    fc, fm, dv = gt.random_tables(g, 20, 8)
    rc = g.choice([-1, 101, 1 << 30], 300).astype(np.int32)
    rm = g.choice([-5, 0, MEM_MAX + 1], 300).astype(np.int32)
    out = run(tables, fc, fm, dv, rc, rm)
    check(fc, fm, dv, rc, rm, out)
    assert (out[0] == -1).all() and out[4].tolist() == [0, 0]


# ---- 6. inputs untouched, answers independent of timing --------------------------------------------------------
@pytest.mark.gpu
def test_inputs_unchanged_and_two_calls_bit_identical(tables):
    g = np.random.default_rng(17)
    fc, fm, dv, rc, rm = contended(g, 300, 16, 6000)
    args = cuda(fc, fm, dv, rc, rm)
    first = tables.place_tables(*args)
    second = tables.place_tables(*args)
    torch.cuda.synchronize()
    for t, a in zip(args, (fc, fm, dv, rc, rm)):
        np.testing.assert_array_equal(t.cpu().numpy(), a)
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
        tables.place_tables(*st)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = tables.place_tables(*st)
    for seed in (12, 13):  # new inputs in place, then replay
        new = contended(np.random.default_rng(seed), N, D, P)
        for t, a in zip(st, new):
            t.copy_(torch.from_numpy(a))
        graph.replay()
        torch.cuda.synchronize()
        check(*new, [t.cpu().numpy() for t in out])


@pytest.mark.gpu
def test_torch_compile_fullgraph(tables):
    g = np.random.default_rng(21)
    a = contended(g, 19, 9, 260)
    out = torch.compile(tables.place_tables, fullgraph=True)(*cuda(*a))
    torch.cuda.synchronize()
    check(*a, [t.cpu().numpy() for t in out])


# ---- 8. refusals, and tables outside the domain during capture -------------------------------------------------
def good_args(N=6, D=8, P=12):
    return dict(fc=torch.full((N, D), 50, dtype=torch.int32, device="cuda"),
                fm=torch.full((N, D), 1000, dtype=torch.int32, device="cuda"),
                dv=torch.full((N,), D, dtype=torch.int32, device="cuda"),
                rc=torch.full((P,), 10, dtype=torch.int32, device="cuda"),
                rm=torch.full((P,), 10, dtype=torch.int32, device="cuda"))


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
        (RuntimeError, with_(rc=torch.full((2 * P,), 10, **z)[::2]), True),
        (RuntimeError, with_(dv=good_args()["dv"].cpu()), True),
        (ValueError, with_(fm=torch.full((N, D + 1), 1000, **z)), True),
        (ValueError, with_(fc=torch.zeros((N, 65), **z), fm=torch.zeros((N, 65), **z)), True),
        (ValueError, with_(dv=torch.full((N + 1,), D, **z)), True),
        (ValueError, with_(rm=torch.zeros((P - 1,), **z)), True),
        (ValueError, bad("fc", (2, 3), 101), False), (ValueError, bad("fc", (2, 3), -1), False),
        (ValueError, bad("fm", (4, 0), MEM_MAX + 1), False), (ValueError, bad("dv", 1, 0), False),
        (ValueError, bad("dv", 1, D + 1), False),
    ]


def call(fn, a):
    return fn(a["fc"], a["fm"], a["dv"], a["rc"], a["rm"])


@pytest.mark.gpu
def test_refusals(tables):
    for exc, a, raw in refusal_cases():
        with pytest.raises(exc, match="place_tables"):
            call(tables.place_tables, a)
        if raw:
            with pytest.raises(exc, match="place_tables"):
                call(torch.ops.egpu.place_tables, a)


# Run in a process of its own: a profiler session here would share CUPTI's state with every later profiler
# session of the test process.
LAUNCH_COUNT = r"""
import sys
sys.path[:0] = [{tests!r}, {root!r}]
import torch
from torch.profiler import ProfilerActivity, profile
import test_gpu_place_tables as t
from elastic_gpu_agent_b200 import tables
tables.load()

def launches(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "place_tables_kernel" in e.name)

def refuse_all():
    for exc, a, raw in t.refusal_cases():
        for fn in (tables.place_tables, torch.ops.egpu.place_tables) if raw else (tables.place_tables,):
            try:
                t.call(fn, a)
            except exc:
                continue
            raise SystemExit("not refused")

a = t.good_args()
print(launches(refuse_all), launches(lambda: t.call(tables.place_tables, a)))
"""


@pytest.mark.gpu
def test_refusals_launch_nothing():
    """No place_tables kernel in a profiler trace of every refusal; the profiler does see an accepted call's."""
    import subprocess
    root = os.path.dirname(HERE)
    r = subprocess.run([sys.executable, "-c", LAUNCH_COUNT.format(tests=HERE, root=root)], capture_output=True,
                       text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.split() == ["0", "1"], r.stdout


@pytest.mark.gpu
def test_tables_outside_the_domain_during_capture(tables):
    """When the data checks cannot run, a table outside the domain offers no device and is copied unchanged; the
    other tables are placed on as if it were absent."""
    g = np.random.default_rng(31)
    N, D, P = 12, 16, 600
    fc, fm, dv, rc, rm = contended(g, N, D, P)
    fcb, fmb, dvb = fc.copy(), fm.copy(), dv.copy()
    dvb[:] = np.maximum(dvb, 1)
    fcb[1, 0], fmb[4, 0], fcb[6, 0], dvb[8], dvb[10] = 101, MEM_MAX + 1, -1, 0, D + 1
    bad = [1, 4, 6, 8, 10]
    st = cuda(fcb, fmb, dvb, rc, rm)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.ops.egpu.place_tables(*st)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_g = tables.place_tables(*st)  # the data checks do not run during capture
    graph.replay()
    out_r = torch.ops.egpu.place_tables(*st)
    torch.cuda.synchronize()
    e = ref.place(fcb, fmb, dvb, rc, rm)  # the restatement leaves tables outside the domain out of the concatenation
    for out in (out_g, out_r):
        node, dev, fco, fmo, info = [t.cpu().numpy() for t in out]
        assert not np.isin(node, bad).any()
        np.testing.assert_array_equal(fco[bad], fcb[bad])
        np.testing.assert_array_equal(fmo[bad], fmb[bad])
        for x, y in zip((node, dev, fco, fmo), e[:4]):
            np.testing.assert_array_equal(x, y)
        assert info.tolist() == [e[4], 0]
