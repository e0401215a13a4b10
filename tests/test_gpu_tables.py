"""egpu::bestfit_tables on the GPU (DESIGN.md §2.10): P requests scored against N capacity tables in one launch.

Every case compares exactly with the numpy oracle run on each table alone (oracle/bestfit_np.snapshot for the index,
the Appendix A.3 key as oracle/bestfit_np.pick_grid forms it for the key):

  1. every pair at the D buckets and their edges (D = 1, 5, 8, 9, 16, 17, 32, 33, 64), with mixed d_valid in one call
     and out-of-domain padding past each table's d_valid, which must be ignored;
  2. hand-picked cases: ties, exact fits, full and empty tables, negative and out-of-domain requests;
  3. calls over several CTA tiles with a ragged last tile and a ragged last request chunk, in the vector form
     (P % 4 == 0) and the scalar form (P % 4 != 0, or requests that are not 16-byte aligned); N = 0 and P = 0;
  4. agreement with egpu_bestfit_query per table, with the context's table and launch count unchanged by the op;
  5. CUDA-graph capture and replay, and torch.compile(fullgraph=True);
  6. refusals on the host before any launch (no bestfit_tables kernel in the profile), and the raw operator's answer
     for a table outside the domain during capture: -1 everywhere, without a fault.
"""
import numpy as np
import pytest

import torch

from oracle import bestfit_np

MEM_MAX = (1 << 18) - 1
NO_KEY = 0x7FFFFFFF


@pytest.fixture(scope="module")
def tables():
    from elastic_gpu_agent_b200 import tables as t
    t.load()
    return t


def ref_key(fc, fm, rc, rm):
    """Appendix A.3 as pick_grid forms it: the minimum over the table's devices of (lc << 24) | (lm << 6) | d,
    INT32_MAX where infeasible."""
    fc = np.asarray(fc, np.int64)[None, :]
    fm = np.asarray(fm, np.int64)[None, :]
    rc = np.asarray(rc, np.int64)[:, None]
    rm = np.asarray(rm, np.int64)[:, None]
    lc, lm = fc - rc, fm - rm
    ok = (rc >= 0) & (rm >= 0) & (lc >= 0) & (lm >= 0)
    d = np.arange(fc.shape[1], dtype=np.int64)[None, :]
    return np.where(ok, (lc << 24) | (lm << 6) | d, NO_KEY).min(axis=1)


def check(fc, fm, dv, rc, rm, idx, key):
    """Every (table, request) pair against the oracle run on that table alone."""
    idx, key = idx.cpu().numpy(), key.cpu().numpy()
    assert idx.dtype == np.int8 and key.dtype == np.int32 and idx.shape == key.shape == (fc.shape[0], rc.size)
    for n in range(fc.shape[0]):
        d = int(dv[n])
        o_idx = bestfit_np.snapshot(fc[n, :d], fm[n, :d], rc, rm)[0]
        np.testing.assert_array_equal(idx[n], o_idx, err_msg=f"table {n} (d_valid {d}): indices")
        np.testing.assert_array_equal(key[n], ref_key(fc[n, :d], fm[n, :d], rc, rm), err_msg=f"table {n}: keys")
        np.testing.assert_array_equal(np.where(key[n] == NO_KEY, -1, key[n] & 63), o_idx)


def random_tables(g, N, D, pad=True):
    """N tables of width D with d_valid in [1, D]: random rows, some full, some empty, some with ties; past d_valid
    out-of-domain values that the op must not read as devices."""
    fc = g.integers(0, 101, (N, D)).astype(np.int32)
    fm = g.integers(0, MEM_MAX + 1, (N, D)).astype(np.int32)
    coarse = g.random(N) < 0.5  # few distinct values: ties in core, in memory, and in both
    fc[coarse] = g.choice([0, 25, 50, 100], (int(coarse.sum()), D))
    fm[coarse] = g.choice([0, 1024, 40_000, 81_559], (int(coarse.sum()), D))
    fc[::7], fm[::7] = 100, 81_559  # full
    fc[3::11], fm[3::11] = 0, 0  # empty
    dv = g.integers(1, D + 1, N).astype(np.int32)
    dv[:2] = [1, D]
    if pad:
        past = np.arange(D)[None, :] >= dv[:, None]
        fc[past] = g.choice([-7, 101, 1000], int(past.sum()))
        fm[past] = g.choice([-1, MEM_MAX + 1, 1 << 30], int(past.sum()))
    return fc, fm, dv


def random_requests(g, P, fc, fm):
    """Requests drawn from the tables' own values (exact fits), random ones, and out-of-domain ones."""
    rc = g.integers(0, 101, P).astype(np.int32)
    rm = g.integers(0, 90_000, P).astype(np.int32)
    ok = (fc >= 0) & (fc <= 100) & (fm >= 0) & (fm <= MEM_MAX)
    pick = g.random(P) < 0.3
    vals = np.stack([fc[ok], fm[ok]], 1)
    chosen = vals[g.integers(0, len(vals), int(pick.sum()))]
    rc[pick], rm[pick] = chosen[:, 0], chosen[:, 1]
    rm[g.random(P) < 0.2] = 0
    bad = g.random(P) < 0.05
    rc[bad] = g.choice([-1, 101, 127, 1 << 30, -(1 << 31)], int(bad.sum()))
    bad = g.random(P) < 0.05
    rm[bad] = g.choice([-1, MEM_MAX + 1, 1 << 18, 1 << 30], int(bad.sum()))
    return rc, rm


def run(tables, fc, fm, dv, rc, rm):
    cu = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (fc, fm, dv, rc, rm)]
    return tables.bestfit_tables(*cu)


# ---- 1. every pair at the D buckets ----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 5, 8, 9, 16, 17, 32, 33, 64])
def test_every_pair_matches_the_oracle_per_table(D, tables):
    g = np.random.default_rng(100 + D)
    fc, fm, dv = random_tables(g, 37, D)
    rc, rm = random_requests(g, 516, fc, fm)
    check(fc, fm, dv, rc, rm, *run(tables, fc, fm, dv, rc, rm))


# ---- 2. hand-picked cases --------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_ties_exact_fits_full_empty_and_out_of_domain(tables):
    D = 8
    fc = np.array([[50, 50, 50, 30, 30, 100, 0, 0],     # ties in core, then memory, then index
                   [100] * 8,                           # full
                   [0] * 8,                             # empty
                   [25, 75, 100, 0, 0, 0, 0, 0]], np.int32)
    fm = np.array([[4096, 2048, 2048, 2048, 2048, 81_559, 0, 0],
                   [81_559] * 8,
                   [0] * 8,
                   [1024, 1024, MEM_MAX, 0, 0, 0, 0, 0]], np.int32)
    dv = np.array([8, 8, 8, 3], np.int32)
    rc = np.array([50, 30, 30, 0, 0, 100, 25, 100, 101, -1, 0, 0, 0, 1, 75, 0, 100, 100], np.int32)
    rm = np.array([2048, 2048, 2049, 0, 1, 81_559, 1024, MEM_MAX, 0, 0, -1, MEM_MAX + 1, 1 << 30, 0, 1024, 0, 0, 81_560],
                  np.int32)
    idx, key = run(tables, fc, fm, dv, rc, rm)
    check(fc, fm, dv, rc, rm, idx, key)
    idx, key = idx.cpu().numpy(), key.cpu().numpy()
    assert idx[0, 0] == 1 and key[0, 0] == 1  # (50, 2048) fits devices 0, 1, 2 and 5: exact fits on 1 and 2, lowest index
    assert idx[0, 1] == 3 and key[0, 1] == 3  # exact fit on 3 and 4
    assert idx[0, 3] == 6 and key[0, 3] == 6  # (0, 0): exact fit on the empty devices 6 and 7
    assert idx[1, 5] == 0 and key[1, 5] == 0  # a whole card on a full table: device 0, no leftover
    assert idx[2, 3] == 0 and (idx[2][(rc != 0) | (rm != 0)] == -1).all()  # the empty table fits (0, 0) only
    assert idx[3, 7] == 2 and key[3, 7] == 2  # (100, MEM_MAX) fits device 2 of the 3 valid devices exactly
    assert (idx[:, 8:13] == -1).all() and (key[:, 8:13] == NO_KEY).all()  # out of domain: -1 everywhere
    assert idx[1, 17] == -1 and key[1, 17] == NO_KEY  # mem 81 560 > 81 559


# ---- 3. several tiles, ragged tiles and chunks, both forms -----------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,D,P,offset", [(517, 8, 4100, 0),    # vector form; on 132 SMs 9 chunks, the last of 4 requests
                                          (523, 8, 2051, 0),    # scalar form: P % 4 != 0
                                          (61, 64, 1032, 1),    # scalar form: requests not 16-byte aligned
                                          (67, 33, 8192, 0)])   # vector form at D = 64's bucket
def test_many_tiles_ragged_last_tile_and_chunk(N, D, P, offset, tables):
    g = np.random.default_rng(N * 7 + P)
    fc, fm, dv = random_tables(g, N, D)
    rc, rm = random_requests(g, P, fc, fm)
    cu = [torch.from_numpy(a).cuda() for a in (fc, fm, dv)]
    rq = []
    for a in (rc, rm):  # a contiguous view that starts `offset` elements into its storage
        buf = torch.zeros(P + offset, dtype=torch.int32, device="cuda")
        buf[offset:] = torch.from_numpy(a).cuda()
        rq.append(buf[offset:])
    idx, key = tables.bestfit_tables(*cu, *rq)
    check(fc, fm, dv, rc, rm, idx, key)


@pytest.mark.gpu
@pytest.mark.parametrize("N,P", [(0, 16), (5, 0), (0, 0)])
def test_empty_calls_give_empty_outputs(N, P, tables):
    fc = torch.full((N, 4), 50, dtype=torch.int32, device="cuda")
    idx, key = tables.bestfit_tables(fc, fc.clone(), torch.full((N,), 4, dtype=torch.int32, device="cuda"),
                                     torch.zeros(P, dtype=torch.int32, device="cuda"),
                                     torch.zeros(P, dtype=torch.int32, device="cuda"))
    assert idx.shape == key.shape == (N, P) and idx.dtype == torch.int8 and key.dtype == torch.int32
    assert idx.device.type == key.device.type == "cuda"


# ---- 4. agreement with egpu_bestfit_query on a context ---------------------------------------------------------
@pytest.mark.gpu
def test_agrees_with_query_and_leaves_the_context_alone(alloc, tables):
    g = np.random.default_rng(7)
    fc, fm, dv = random_tables(g, 24, 17)
    rc, rm = random_requests(g, 1000, fc, fm)
    own_c, own_m = fc[5, :int(dv[5])].copy(), fm[5, :int(dv[5])].copy()
    alloc.set_table(own_c, own_m)
    alloc.bestfit(rc, rm, commit=True)  # a table of the context's own, with flags, differs from every table below
    before, launches = alloc.table(), alloc.launch_count
    idx, key = run(tables, fc, fm, dv, rc, rm)
    torch.cuda.synchronize()
    after = alloc.table()
    assert alloc.launch_count == launches
    for a, b in zip(before, after):
        np.testing.assert_array_equal(a, b)
    idx = idx.cpu().numpy()
    for n in range(fc.shape[0]):
        d = int(dv[n])
        np.testing.assert_array_equal(idx[n], alloc.query(fc[n, :d], fm[n, :d], rc, rm), err_msg=f"table {n}")


# ---- 5. CUDA graphs and torch.compile --------------------------------------------------------------------------
@pytest.mark.gpu
def test_cuda_graph_capture_and_replay(tables):
    g = np.random.default_rng(11)
    N, D, P = 40, 16, 1024
    fc, fm, dv = random_tables(g, N, D)
    rc, rm = random_requests(g, P, fc, fm)
    st = [torch.from_numpy(a).cuda() for a in (fc, fm, dv, rc, rm)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        tables.bestfit_tables(*st)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_idx, out_key = tables.bestfit_tables(*st)
    for seed in (12, 13):  # new inputs in place, then replay
        g2 = np.random.default_rng(seed)
        fc2, fm2, dv2 = random_tables(g2, N, D)
        rc2, rm2 = random_requests(g2, P, fc2, fm2)
        for t, a in zip(st, (fc2, fm2, dv2, rc2, rm2)):
            t.copy_(torch.from_numpy(a))
        graph.replay()
        torch.cuda.synchronize()
        check(fc2, fm2, dv2, rc2, rm2, out_idx, out_key)


@pytest.mark.gpu
def test_torch_compile_fullgraph(tables):
    g = np.random.default_rng(21)
    fc, fm, dv = random_tables(g, 19, 9)
    rc, rm = random_requests(g, 260, fc, fm)
    args = [torch.from_numpy(a).cuda() for a in (fc, fm, dv, rc, rm)]

    idx, key = torch.compile(tables.bestfit_tables, fullgraph=True)(*args)
    torch.cuda.synchronize()
    check(fc, fm, dv, rc, rm, idx, key)


# ---- 6. refusals ------------------------------------------------------------------------------------------------
def kernel_launches(fn):
    """Number of bestfit_tables kernels the CUDA profiler sees while fn runs."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "bestfit_tables_kernel" in e.name)


@pytest.mark.gpu
def test_refusals_raise_before_any_launch(tables):
    N, D, P = 6, 8, 12

    def good():
        return dict(fc=torch.full((N, D), 50, dtype=torch.int32, device="cuda"),
                    fm=torch.full((N, D), 1000, dtype=torch.int32, device="cuda"),
                    dv=torch.full((N,), D, dtype=torch.int32, device="cuda"),
                    rc=torch.full((P,), 10, dtype=torch.int32, device="cuda"),
                    rm=torch.full((P,), 10, dtype=torch.int32, device="cuda"))

    def with_(**kw):
        a = good()
        a.update(kw)
        return a

    def bad_fc(v):
        a = good()
        a["fc"][2, 3] = v
        return a

    def bad_fm(v):
        a = good()
        a["fm"][4, 0] = v
        return a

    def bad_dv(v):
        a = good()
        a["dv"][1] = v
        return a

    cases = [
        (RuntimeError, with_(fc=good()["fc"].to(torch.int64))),
        (RuntimeError, with_(rm=good()["rm"].to(torch.int16))),
        (RuntimeError, with_(fc=torch.full((D, N), 50, dtype=torch.int32, device="cuda").t())),
        (RuntimeError, with_(rc=torch.full((2 * P,), 10, dtype=torch.int32, device="cuda")[::2])),
        (RuntimeError, with_(dv=good()["dv"].cpu())),
        (ValueError, with_(fm=torch.full((N, D + 1), 1000, dtype=torch.int32, device="cuda"))),
        (ValueError, with_(fc=torch.full((N,), 50, dtype=torch.int32, device="cuda"),
                           fm=torch.full((N,), 50, dtype=torch.int32, device="cuda"))),
        (ValueError, with_(fc=torch.zeros((N, 0), dtype=torch.int32, device="cuda"),
                           fm=torch.zeros((N, 0), dtype=torch.int32, device="cuda"))),
        (ValueError, with_(fc=torch.zeros((N, 65), dtype=torch.int32, device="cuda"),
                           fm=torch.zeros((N, 65), dtype=torch.int32, device="cuda"))),
        (ValueError, with_(dv=torch.full((N + 1,), D, dtype=torch.int32, device="cuda"))),
        (ValueError, with_(rm=torch.zeros((P - 1,), dtype=torch.int32, device="cuda"))),
        (ValueError, bad_fc(101)), (ValueError, bad_fc(-1)), (ValueError, bad_fm(MEM_MAX + 1)), (ValueError, bad_fm(-5)),
        (ValueError, bad_dv(0)), (ValueError, bad_dv(D + 1)), (ValueError, bad_dv(-3)),
    ]

    def refuse_all():
        for exc, a in cases:
            with pytest.raises(exc, match="bestfit_tables"):
                tables.bestfit_tables(a["fc"], a["fm"], a["dv"], a["rc"], a["rm"])
        for exc, a in cases[:11]:  # the raw operator refuses the same without reading data
            with pytest.raises(exc, match="bestfit_tables"):
                torch.ops.egpu.bestfit_tables(a["fc"], a["fm"], a["dv"], a["rc"], a["rm"])

    assert kernel_launches(refuse_all) == 0
    a = good()  # the profiler does see the kernel
    assert kernel_launches(lambda: tables.bestfit_tables(a["fc"], a["fm"], a["dv"], a["rc"], a["rm"])) == 1


@pytest.mark.gpu
def test_raw_operator_answers_minus_one_for_tables_outside_the_domain(tables):
    """What a caller gets when the data checks cannot run (the raw operator, or the Python function during capture):
    a table outside the domain is infeasible for every request; the other tables are answered as always."""
    g = np.random.default_rng(31)
    N, D, P = 12, 16, 256
    fc, fm, dv = random_tables(g, N, D, pad=False)
    rc, rm = random_requests(g, P, fc, fm)
    fcb, fmb, dvb = fc.copy(), fm.copy(), dv.copy()
    fcb[1, 0], fmb[4, 0], fcb[6, 0], dvb[8], dvb[10] = 101, MEM_MAX + 1, -1, 0, D + 1
    bad = [1, 4, 6, 8, 10]
    st = [torch.from_numpy(a).cuda() for a in (fcb, fmb, dvb, rc, rm)]
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.ops.egpu.bestfit_tables(*st)
    torch.cuda.current_stream().wait_stream(s)
    with torch.cuda.graph(graph):
        idx_g, key_g = tables.bestfit_tables(*st)  # the data checks do not run during capture
    graph.replay()
    idx_r, key_r = torch.ops.egpu.bestfit_tables(*st)
    torch.cuda.synchronize()
    good_rows = [n for n in range(N) if n not in bad]
    for idx, key in ((idx_g, key_g), (idx_r, key_r)):
        i, k = idx.cpu().numpy(), key.cpu().numpy()
        assert (i[bad] == -1).all() and (k[bad] == NO_KEY).all()
        check(fc[good_rows], fm[good_rows], dv[good_rows], rc, rm, idx[good_rows], key[good_rows])
