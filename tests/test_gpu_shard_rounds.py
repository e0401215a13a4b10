"""Rounds to the fixed point over row shards in one launch per rank: egpu_bestfit_batch_shard_prefix_dev with
EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT | EGPU_F_ROUNDS | EGPU_F_DEVICE_ROUNDS [| EGPU_F_PACKED].

The result is egpu_bestfit_batch_rounds (no round limit) on the concatenation of the ranks' shards in rank order,
computed by the persistent shard_rounds_sorted_kernel / shard_rounds_lut_kernel in one cooperative launch per rank:

  1. (CPU) the header documents the flag set; the wrapper passes exactly those flags, and a NULL d_req_mem when
     packed; a numpy restatement of the per-rank algorithm - rank-major base from the uncapped vectors, a cut per
     rank, a compaction per rank, another round iff some device's all-rank uncapped demand exceeds its free
     capacity - equals the C rounds oracle on the concatenation, for 1 to 8 ranks;
  2. world 1 at every D bucket under AUTO, SORTED and LUT, int32 and packed (infeasible rows, out-of-range words):
     bit-exact against the oracle and against egpu_bestfit_batch_dev with EGPU_F_DEVICE_ROUNDS on the same rows;
     one launch per call; sticky oversubscription flags; a CUDA graph replayed before and after egpu_table_set;
  3. a D = 64 case of at least 64 rounds, and 130 calls past the 256-slot exchange ring;
  4. world 2 (two processes on one GPU, started together by the gate): both formats and mixed, a rank with R = 0,
     deferral on one rank only, more CTAs than devices;
  5. refusals: nothing launched, nothing written;
  6. a peer that attaches and never launches: round 1 commits nothing, and the launch ends on its own.
Every GPU test ends with a host-form device-rounds call that reports a grid-barrier timeout of any launch on its
context (the `ctx` fixture of test_gpu_device_rounds), and checks egpu_peer_last_timeout.
"""
import ctypes as C
import os
import re
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_device_rounds as dr  # noqa: E402  (the ctx fixture, the rounds reference, Out, the single-GPU call)
import test_gpu_kernel_matrix as km  # noqa: E402  (cell tables and cases, pack / unpack, packed_words, int32 device arrays)
import test_gpu_packed_multi as pm  # noqa: E402  (words, stream handle, table_is)
import test_gpu_packed_shard as ps  # noqa: E402  (attach)
import test_gpu_peer_exchange as pe  # noqa: E402  (the prefix-commit table and requests, per-rank sums)

ctx = dr.ctx
ROOT = pm.ROOT
MEM_MAX = (1 << 18) - 1
ERR_INVALID, ERR_NO_TABLE, ERR_STATE = -1, -5, -6
AUTO, GRID, SORTED, LUT = 0, 1, 2, 3
F_COMMIT, F_INPUTS_READY, F_PREFIX, F_APPLY, F_PACKED, F_ROUNDS, F_DEVICE_ROUNDS = 1, 2, 4, 8, 16, 32, 128
SR = F_PREFIX | F_COMMIT | F_ROUNDS | F_DEVICE_ROUNDS
D_BUCKETS = (1, 8, 9, 16, 17, 33, 64)
VNAME = ["auto", "grid", "sorted", "lut"]
COUNTS = (0, 1, 513, 4099, 40_003)


def test_shard_rounds_documented():
    src = open(os.path.join(ROOT, "include", "egpu_alloc.h")).read()
    block = src[src.index("Rounds to the fixed point over row shards in one launch"):src.index("int egpu_bestfit_batch_shard_prefix_dev(")]
    assert re.search(r"EGPU_F_PREFIX_COMMIT \| EGPU_F_COMMIT \|\s+\*\s+EGPU_F_ROUNDS \| EGPU_F_DEVICE_ROUNDS \[\| EGPU_F_PACKED\]", block)
    for phrase in ("stays 1011", "step + 2 > 2^47", "R >= 2^31", "`step` and `step + 1`", "about 2 s", "ONE launch",
                   "EGPU_ERR_NOMEM", "EGPU_ERR_NO_TABLE", "d_delta and d_table_out are written at the fixed point only"):
        assert phrase in block, phrase
    head = src[:src.index("/* kernel variants")]
    assert "egpu_bestfit_batch_shard_prefix_dev" in head[head.index("#define EGPU_F_DEVICE_ROUNDS 128"):]


def test_wrapper_flags(egpu):
    """bestfit_shard_rounds_dev passes exactly the flag set and the step, and a NULL d_req_mem when packed"""
    calls = []

    class Lib:
        def __getattr__(self, name):
            return lambda *a: calls.append((name, a)) or 0

    a = object.__new__(egpu.BestFitAllocator)
    a._lib, a._h = Lib(), C.c_void_p(1)
    a.bestfit_shard_rounds_dev(16, 32, 5, 48, 64, 80, 6)
    a.bestfit_shard_rounds_dev(16, 32, 5, 48, 0, 0, 8, packed=True)
    assert [n for n, _ in calls] == ["egpu_bestfit_batch_shard_prefix_dev"] * 2
    assert [c[1][7] for c in calls] == [SR, SR | F_PACKED]
    assert [c[1][8] for c in calls] == [6, 8]
    assert calls[0][1][2].value == 32 and calls[1][1][2] is None
    assert calls[0][1][5].value == 64 and calls[1][1][5].value is None and calls[1][1][6].value is None
    a._lib = None
    a._h = None


# ---- 1. the per-rank algorithm, restated in numpy ------------------------------------------------------------
def sharded_rounds(oracle_c, fc, fm, shards):
    """What each rank of the launch computes, round by round: (per-rank indices, per-rank committed demand [2*D],
    final free_core, free_mem, rounds, per round the ranks that deferred rows).  The scan is the oracle's snapshot
    against the round's table; the cut of rank g starts from the lower ranks' uncapped demand; the decision to run
    another round uses only the all-rank uncapped demand and the table, and is checked against the deferrals."""
    fc, fm = np.asarray(fc, np.int64).copy(), np.asarray(fm, np.int64).copy()
    D, W = fc.size, len(shards)
    rc = [np.asarray(s[0], np.int32) for s in shards]
    rm = [np.asarray(s[1], np.int32) for s in shards]
    out = [np.full(x.size, -3, np.int32) for x in rc]
    pend = [np.arange(x.size) for x in rc]
    total = [np.zeros(2 * D, np.int64) for _ in range(W)]
    rounds, deferring = 0, []
    while True:
        rounds += 1
        cc = [rc[g][pend[g]].astype(np.int64) for g in range(W)]
        cm = [rm[g][pend[g]].astype(np.int64) for g in range(W)]
        choice = [oracle_c.snapshot(fc.astype(np.int32), fm.astype(np.int32), rc[g][pend[g]], rm[g][pend[g]])[0] for g in range(W)]
        unc = np.zeros((W, 2, D), np.int64)  # each rank's uncapped demand vector (exchange step `step`)
        for g in range(W):
            ok = choice[g] >= 0
            np.add.at(unc[g, 0], choice[g][ok], cc[g][ok])
            np.add.at(unc[g, 1], choice[g][ok], cm[g][ok])
        every = unc.sum(axis=0)
        again = bool(((every[0] > fc) | (every[1] > fm)).any())
        committed = np.zeros((2, D), np.int64)  # every rank's committed demand (exchange step `step + 1`)
        nxt, deferred_by = [], []
        for g in range(W):
            base = unc[:g].sum(axis=0)
            res = choice[g].copy()
            for d in np.unique(res[res >= 0]):
                sel = np.flatnonzero(choice[g] == d)
                keep = (base[0, d] + np.cumsum(cc[g][sel]) <= fc[d]) & (base[1, d] + np.cumsum(cm[g][sel]) <= fm[d])
                res[sel[~keep]] = -2
                committed[0, d] += cc[g][sel[keep]].sum()
                committed[1, d] += cm[g][sel[keep]].sum()
                total[g][d] += cc[g][sel[keep]].sum()
                total[g][D + d] += cm[g][sel[keep]].sum()
            out[g][pend[g]] = res
            nxt.append(pend[g][res == -2])
            if (res == -2).any():
                deferred_by.append(g)
        assert again == bool(deferred_by), "the all-rank demand rule disagrees with the deferrals"
        fc, fm = fc - committed[0], fm - committed[1]
        deferring.append(deferred_by)
        pend = nxt
        if not again:
            return out, total, fc.astype(np.int32), fm.astype(np.int32), rounds, deferring


def check_restatement(oracle_c, fc, fm, shards):
    out, total, gfc, gfm, rounds, deferring = sharded_rounds(oracle_c, fc, fm, shards)
    rc = np.concatenate([np.asarray(s[0], np.int32) for s in shards])
    rm = np.concatenate([np.asarray(s[1], np.int32) for s in shards])
    o_idx, o_dc, o_dm, o_fc, o_fm, o_rounds, o_left = oracle_c.rounds(fc, fm, rc, rm)
    assert o_left == 0
    assert np.array_equal(np.concatenate(out), o_idx), "indices"
    assert np.array_equal(sum(total), np.concatenate([o_dc, o_dm])), "demand summed over the ranks"
    lo = 0
    for g, s in enumerate(shards):
        n = len(s[0])
        assert np.array_equal(total[g], pe._rank_partial(o_idx[lo:lo + n], rc[lo:lo + n], rm[lo:lo + n], fc.size)), f"rank {g} sums"
        lo += n
    assert np.array_equal(gfc, o_fc) and np.array_equal(gfm, o_fm), "table"
    assert rounds == max(1, o_rounds), "rounds"
    return deferring


def split(rng, rc, rm, world, empty=True):
    """ragged shards of (rc, rm) in order; with `empty`, some ranks may get none"""
    cuts = np.sort(rng.integers(0, rc.size + 1, world - 1))
    if not empty:
        cuts = np.sort(rng.choice(np.arange(1, rc.size), world - 1, replace=False))
    b = np.concatenate([[0], cuts, [rc.size]])
    return [(rc[b[g]:b[g + 1]], rm[b[g]:b[g + 1]]) for g in range(world)]


def _workload_rows(egpu, name, seed, R, cap_c, cap_m):
    w = egpu.synth.workload(name)
    rc, rm = egpu.synth.requests(3, seed, R)
    return (np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32),
            np.minimum(rc, cap_c).astype(np.int32), np.minimum(rm, cap_m).astype(np.int32))


@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("case", ["ragged", "cfg3", "cfg4", "one-rank-defers"])
def test_restatement_equals_rounds_oracle(case, world, oracle_c, egpu):
    rng = np.random.default_rng([world, len(case)])
    if case == "ragged":
        shards = []
        for g in range(world):
            n = int(rng.choice((0, 1, 3, 5, 511, 513, 1500)))
            shards.append(pe._prefix_requests(100 * world + g, n))
        fc, fm = pe.PREFIX_FC, pe.PREFIX_FM
    elif case in ("cfg3", "cfg4"):
        fc, fm, rc, rm = _workload_rows(egpu, case, 7 + world, 12_000, *((5, 2048) if case == "cfg3" else (2, 1024)))
        shards = split(rng, rc, rm, world)
    else:  # the lower ranks' few zero-core rows all fit; every deferral is the last rank's
        shards = [(np.zeros(3, np.int32), np.ones(3, np.int32)) for _ in range(world - 1)]
        shards.append(pe._prefix_requests(900 + world, 700))
        fc, fm = pe.PREFIX_FC, pe.PREFIX_FM
    deferring = check_restatement(oracle_c, fc, fm, shards)
    if case == "cfg4":
        assert len(deferring) >= 32, len(deferring)
    if case == "one-rank-defers":
        assert len(deferring) > 2 and all(d in ([], [world - 1]) for d in deferring)


# ---- calls ----------------------------------------------------------------------------------------------------
def rows_in(torch, rc, rm, D, packed, oddities=True):
    """(d_req_core, d_req_mem or None, the requests the call stands for): int32 arrays, or packed words with
    out-of-range ones when `oddities`"""
    if packed:
        words = km.packed_words(rc, rm, len(rc), D) if oddities else km.pack(rc, rm)
        return pm.words_dev(torch, words), None, km.unpack(words)
    return km._dev(torch, np.asarray(rc, np.int32)), km._dev(torch, np.asarray(rm, np.int32)), (rc, rm)


def shard_call(alloc, torch, c, m, o, step, stream=None):
    i, dl, t = o.ptrs()
    s = torch.cuda.current_stream().cuda_stream if stream is None else stream
    alloc.bestfit_shard_rounds_dev(c.data_ptr(), m.data_ptr() if m is not None else 0, o.R, i, dl, t, step, packed=o.packed,
                                   stream=s)


def got_of(alloc, o):
    return o.got() + (alloc.table(),)


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a[:3], b[:3])) and all(np.array_equal(x, y) for x, y in zip(a[3], b[3]))


# ---- 2. world 1 ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [AUTO, SORTED, LUT], ids=lambda v: VNAME[v])
@pytest.mark.parametrize("D", D_BUCKETS)
def test_shard_rounds_world1(variant, D, ctx, oracle_c):
    """every table of the cell matrix, both formats, R in COUNTS: the oracle, then the single-GPU one-launch rounds on
    the same rows give the same bytes; one launch per call"""
    import torch
    ctx.set_variant(variant)
    ps.attach(ctx)
    step = 0
    for tname, (fc, fm) in km.cell_tables(D).items():
        for R in COUNTS:
            _, _, rc, rm = km.cell_case(D, tname, R)
            for packed in (False, True):
                where = f"{VNAME[variant]}, D = {D}, table {tname}, R = {R}, {'packed' if packed else 'int32'}"
                c, m, req = rows_in(torch, rc, rm, D, packed)
                exp = dr.ref(oracle_c, fc, fm, *req)
                ctx.set_table(fc, fm)
                o = dr.Out(torch, R, D, packed)
                torch.cuda.synchronize()
                n0 = ctx.launch_count
                shard_call(ctx, torch, c, m, o, step)
                assert ctx.launch_count - n0 == 1, f"{where}: one launch"
                torch.cuda.synchronize()
                got = got_of(ctx, o)
                dr.check(got, exp, where)
                ctx.set_table(fc, fm)
                o1 = dr.Out(torch, R, D, packed)
                torch.cuda.synchronize()
                assert dr.call_dev(ctx, torch, c, m, o1) == 0
                torch.cuda.synchronize()
                assert same(got, got_of(ctx, o1)), f"{where}: differs from egpu_bestfit_batch_dev with EGPU_F_DEVICE_ROUNDS"
                step += 2
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT], ids=lambda v: VNAME[v])
@pytest.mark.parametrize("packed", [False, True])
def test_shard_rounds_keep_oversubscription_flags(variant, packed, ctx, oracle_c):
    """a table with sticky oversubscription flags: the rounds keep them"""
    import torch
    D = 8
    fc, fm = np.full(D, 50, np.int32), np.full(D, 4096, np.int32)
    ctx.set_variant(variant)
    ctx.set_table(fc, fm)
    ctx.bestfit(np.array([30, 30, 30, 30], np.int32), np.array([1, 1, 1, 1], np.int32), commit=True)
    fc1, fm1, ov1 = ctx.table()
    assert ov1.any()
    ps.attach(ctx)
    rng = np.random.default_rng(6)
    rc, rm = rng.integers(0, 12, 20_001).astype(np.int32), rng.integers(0, 300, 20_001).astype(np.int32)
    c, m, req = rows_in(torch, rc, rm, D, packed, oddities=False)
    exp = dr.ref(oracle_c, fc1, fm1, *req, ov=ov1)
    assert exp[4] >= 2
    o = dr.Out(torch, rc.size, D, packed)
    shard_call(ctx, torch, c, m, o, 0)
    torch.cuda.synchronize()
    dr.check(got_of(ctx, o), exp, "sticky flags")
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(SORTED, 8), (LUT, 64), (AUTO, 33)])
@pytest.mark.parametrize("packed", [False, True])
def test_shard_rounds_graph_replay(variant, D, packed, ctx, oracle_c):
    """one call captured in a CUDA graph, replayed with an egpu_table_set before each replay: each replay equals its
    eager run and the oracle on the table it starts from"""
    import torch
    tables = km.cell_tables(D)
    _, _, rc, rm = km.cell_case(D, "dups", 40_003)
    c, m, req = rows_in(torch, rc, rm, D, packed)
    ctx.set_variant(variant)
    ps.attach(ctx)
    o = dr.Out(torch, rc.size, D, packed)
    s = torch.cuda.Stream()
    ctx.set_table(*tables["dups"])
    with torch.cuda.stream(s):
        shard_call(ctx, torch, c, m, o, 0, s.cuda_stream)  # warm-up outside the capture: scratch and occupancy
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        shard_call(ctx, torch, c, m, o, 0, s.cuda_stream)
    for tname in ("dups", "spread"):
        fc, fm = tables[tname]
        exp = dr.ref(oracle_c, fc, fm, *req)
        ctx.set_table(fc, fm)
        o.idx.fill_(-9), o.delta.fill_(-1), o.tab.fill_(-7)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        dr.check(got_of(ctx, o), exp, f"replay, table {tname}")
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


# ---- 3. many rounds, and the exchange ring -------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT], ids=lambda v: VNAME[v])
@pytest.mark.parametrize("packed", [False, True])
def test_shard_rounds_many_rounds_d64(variant, packed, ctx, egpu, oracle_c):
    """the cfg4 table (D = 64) and small requests: every round reuses the same two exchange steps"""
    import torch
    fc, fm, rc, rm = _workload_rows(egpu, "cfg4", 5, 100_003, 2, 1024)
    c, m, req = rows_in(torch, rc, rm, fc.size, packed, oddities=False)
    exp = dr.ref(oracle_c, fc, fm, *req)
    assert exp[4] >= 64, exp[4]
    ctx.set_variant(variant)
    ctx.set_table(fc, fm)
    ps.attach(ctx)
    o = dr.Out(torch, rc.size, fc.size, packed)
    shard_call(ctx, torch, c, m, o, 10)
    torch.cuda.synchronize()
    dr.check(got_of(ctx, o), exp, f"{exp[4]} rounds")
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True])
def test_shard_rounds_past_the_ring(packed, ctx, egpu, oracle_c):
    """130 committing calls at steps 0, 2, ..., 258 on one stream, each on the table the one before left: 260
    exchange steps, more than the 256 slots"""
    import torch
    w = egpu.synth.workload("cfg4")
    fc, fm = np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32)
    D = fc.size
    ps.attach(ctx)
    ctx.set_table(fc, fm)
    rng = np.random.default_rng(17)
    calls, exps, n_rounds = [], [], 0
    cur = (fc, fm)
    for k in range(130):
        R = int(rng.integers(0, 96))
        rc, rm = rng.integers(0, 2, R).astype(np.int32), rng.integers(1, 65, R).astype(np.int32)
        c, m, req = rows_in(torch, rc, rm, D, packed, oddities=False)
        e = dr.ref(oracle_c, *cur, *req)
        cur = e[3][:2]
        n_rounds += e[4]
        calls.append((c, m, dr.Out(torch, R, D, packed)))
        exps.append(e)
    assert n_rounds > 130, n_rounds  # most calls take more than one round
    torch.cuda.synchronize()
    for k, (c, m, o) in enumerate(calls):
        shard_call(ctx, torch, c, m, o, 2 * k)
    torch.cuda.synchronize()
    for k, ((c, m, o), e) in enumerate(zip(calls, exps)):
        idx, delta, tab = o.got()
        assert np.array_equal(idx, e[0]) and np.array_equal(delta, e[1]) and np.array_equal(tab, e[2]), f"call {k}"
    assert pm.table_is(ctx, *cur)
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


# ---- 4. world 2: two processes on one GPU ------------------------------------------------------------------------
def _w2_cases():
    """(name, rank 0's requests, rank 1's requests), each on a fresh PREFIX table"""
    light = (np.zeros(20, np.int32), np.ones(20, np.int32))  # device 3, all fit
    lone = (np.array([75, 101, 120], np.int32), np.ones(3, np.int32))  # device 0 first in the order, then infeasible twice
    return [
        ("rank 0 empty", (np.zeros(0, np.int32), np.zeros(0, np.int32)), pe._prefix_requests(4000, 400)),
        ("rank 1 empty", pe._prefix_requests(4001, 400), (np.zeros(0, np.int32), np.zeros(0, np.int32))),
        ("deferral on rank 1 only", light, pe._prefix_requests(4002, 400)),
        ("deferral on rank 0 only", pe._prefix_requests(4003, 400), lone),
        ("more CTAs than devices", *(lambda r: ((r[0][:40_000], r[1][:40_000]), (r[0][40_000:], r[1][40_000:])))(
            pe._prefix_requests(4004, 70_001))),
    ]


def _rank_main(rank, conn, peer_conn, packed):
    """One rank on cuda:0: every case of _w2_cases from a fresh table, twice: once as a warm-up, then each call
    started together with the other rank through the gate.  The warm-up loads the kernel and allocates the scratch
    first: a kernel's first launch loads its module, which waits for the kernels running on the context - the gate
    among them, which waits for the host - so nothing between gate_dev and gate_open may launch a kernel for the
    first time."""
    sys.path.insert(0, ROOT)
    import torch
    import elastic_gpu_agent_b200 as e
    torch.cuda.set_device(0)
    a = e.BestFitAllocator(0)
    a.set_table(pe.PREFIX_FC, pe.PREFIX_FM)
    mine = a.peer_export()
    peer_conn.send(mine)
    other = peer_conn.recv()
    a.peer_attach(rank, 2, [mine, other] if rank == 0 else [other, mine])
    peer_conn.send("attached")
    assert peer_conn.recv() == "attached"
    D = pe.PREFIX_FC.size
    s = torch.cuda.current_stream().cuda_stream
    ins = []
    for _, *shards in _w2_cases():
        rc, rm = shards[rank]
        c, m, _ = rows_in(torch, rc, rm, D, packed, oddities=False)
        ins.append((c, m, dr.Out(torch, rc.size, D, packed)))
    res = []
    for p, gated in enumerate((False, True)):
        out = []
        for k, (c, m, o) in enumerate(ins):
            a.set_table(pe.PREFIX_FC, pe.PREFIX_FM)
            o.idx.fill_(-9), o.delta.fill_(-1), o.tab.fill_(-7)
            torch.cuda.synchronize()
            if gated:
                a.gate_dev(s)
            shard_call(a, torch, c, m, o, 2 * k + 2 * len(ins) * p, s)
            if gated:
                a.gate_open()
            torch.cuda.synchronize()
            out.append(o.got() + (a.table(),))
        res.append(out)
    timeout, gate_timeouts = a.peer_last_timeout, a.gate_timeouts
    # a host-form device-rounds call reports a grid-barrier timeout of any launch on this context
    one = np.array([1], np.int32)
    idx = np.empty(1, np.int32)
    a.set_table([100], [MEM_MAX])
    rounds_rc = a._lib.egpu_bestfit_batch(a.handle, C.c_void_p(one.ctypes.data), C.c_void_p(one.ctypes.data), 1,
                                          C.c_void_p(idx.ctypes.data), None, None, dr.DR)
    conn.send((rank, res, timeout, gate_timeouts, rounds_rc))
    peer_conn.send("done")
    peer_conn.recv()
    a.peer_detach()
    a.close()


W2_FORMATS = [(False, False), (True, True), (True, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("formats", W2_FORMATS, ids=["int32-int32", "packed-packed", "packed-int32"])
def test_shard_rounds_world2(formats, oracle_c):
    import torch.multiprocessing as mp
    mctx = mp.get_context("spawn")
    a_conn, b_conn = mctx.Pipe()
    res0_r, res0_w = mctx.Pipe(False)
    res1_r, res1_w = mctx.Pipe(False)
    procs = [mctx.Process(target=_rank_main, args=(0, res0_w, a_conn, formats[0])),
             mctx.Process(target=_rank_main, args=(1, res1_w, b_conn, formats[1]))]
    for p in procs:
        p.start()
    try:
        assert res0_r.poll(300) and res1_r.poll(300), "ranks did not finish"
        r0, r1 = res0_r.recv(), res1_r.recv()
        for p in procs:
            p.join(60)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
    assert all(p.exitcode == 0 for p in procs)
    for r in (r0, r1):
        assert r[2] == 0, f"rank {r[0]}: a peer pull timed out at step + 1 = {r[2]}"
        assert r[3] == 0, f"rank {r[0]}: the start gate timed out"
        assert r[4] == 0, f"rank {r[0]}: a grid barrier timed out"
    D = pe.PREFIX_FC.size
    for k, (name, s0, s1) in enumerate(_w2_cases()):
        deferring = check_restatement(oracle_c, pe.PREFIX_FC, pe.PREFIX_FM, [s0, s1])
        if name == "deferral on rank 1 only":
            assert len(deferring) > 2 and all(d in ([], [1]) for d in deferring), deferring
        if name == "deferral on rank 0 only":
            assert len(deferring) > 2 and all(d in ([], [0]) for d in deferring), deferring
        rc, rm = np.concatenate([s0[0], s1[0]]), np.concatenate([s0[1], s1[1]])
        o_idx, _, tab, inst, _ = dr.ref(oracle_c, pe.PREFIX_FC, pe.PREFIX_FM, rc, rm)
        n0 = s0[0].size
        for p, where in enumerate(("warm-up", "gated")):
            (i0, d0, t0, g0), (i1, d1, t1, g1) = r0[1][p][k], r1[1][p][k]
            where = f"{where}, {name}"
            assert np.array_equal(i0, o_idx[:n0]) and np.array_equal(i1, o_idx[n0:]), f"{where}: indices"
            assert np.array_equal(d0, pe._rank_partial(o_idx[:n0], rc[:n0], rm[:n0], D)), f"{where}: rank 0 sums"
            assert np.array_equal(d1, pe._rank_partial(o_idx[n0:], rc[n0:], rm[n0:], D)), f"{where}: rank 1 sums"
            assert np.array_equal(t0, tab) and np.array_equal(t1, tab), f"{where}: table'"
            for g in (g0, g1):
                assert all(np.array_equal(x, y) for x, y in zip(g, inst)), f"{where}: installed table"


# ---- 5. refusals -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_shard_rounds_refusals(ctx):
    import torch
    D = 8
    fc, fm = km.cell_tables(D)["dups"]
    _, _, rc, rm = km.cell_case(D, "dups", 513)
    c32, m32, _ = rows_in(torch, rc, rm, D, False)
    w8, _, _ = rows_in(torch, rc, rm, D, True)
    o32, o8 = dr.Out(torch, 513, D, False), dr.Out(torch, 513, D, True)
    lib, h = ctx._lib, ctx.handle
    s = pm._s(torch)
    vp = C.c_void_p

    def raw(flags, step=0, packed=False, R=513, core=None, mem="given", idx=None):
        """the call on o32 / o8; core, mem and idx replace the arrays (0 = NULL); mem is NULL when packed"""
        o = o8 if packed else o32
        i, dl, t = o.ptrs()
        core = (w8 if packed else c32).data_ptr() if core is None else core
        if mem == "given":
            mem = 0 if packed else m32.data_ptr()
        i = i if idx is None else idx
        return lib.egpu_bestfit_batch_shard_prefix_dev(h, vp(core or None), vp(mem or None), R, vp(i or None), vp(dl), vp(t),
                                                       flags | (F_PACKED if packed else 0), step, s)

    # no table, then unattached
    assert raw(SR) == ERR_NO_TABLE
    ctx.set_table(fc, fm)
    assert raw(SR) == ERR_STATE and raw(SR, packed=True) == ERR_STATE
    ps.attach(ctx)
    before = ctx.table()
    torch.cuda.synchronize()
    n0 = ctx.launch_count
    for f in (F_ROUNDS, F_DEVICE_ROUNDS, F_ROUNDS | F_DEVICE_ROUNDS, F_PREFIX | F_COMMIT | F_ROUNDS, F_PREFIX | F_COMMIT | F_DEVICE_ROUNDS,
              F_COMMIT | F_ROUNDS | F_DEVICE_ROUNDS, F_PREFIX | F_ROUNDS | F_DEVICE_ROUNDS, SR | F_INPUTS_READY, SR | F_APPLY, SR | 64,
              SR | 256, F_PACKED | F_ROUNDS):
        for packed in (False, True):
            assert raw(f, packed=packed) == ERR_INVALID, (f, packed)
    for packed in (False, True):
        fmt = "packed" if packed else "int32"
        base = (w8 if packed else c32).data_ptr()
        ip = (o8 if packed else o32).idx.data_ptr()
        refused = {
            "step + 2 > 2^47": raw(SR, (1 << 47) - 1, packed),
            "step >= 2^47": raw(SR, 1 << 47, packed),
            "R >= 2^31": raw(SR, 0, packed, R=1 << 31),
            "NULL req_core": raw(SR, 0, packed, core=0),
            "NULL indices": raw(SR, 0, packed, idx=0),
            "misaligned req_core": raw(SR, 0, packed, core=base + 4),
            "misaligned indices": raw(SR, 0, packed, idx=ip + (1 if packed else 4)),
        }
        if packed:
            refused["req_mem with EGPU_F_PACKED"] = raw(SR, 0, True, mem=m32.data_ptr())
        else:
            refused["NULL req_mem without EGPU_F_PACKED"] = raw(SR, 0, False, mem=0)
            refused["misaligned req_mem"] = raw(SR, 0, False, mem=m32.data_ptr() + 4)
        for what, code in refused.items():
            assert code == ERR_INVALID, f"{fmt}: {what}"
    ctx.set_variant(GRID)
    assert raw(SR) == ERR_STATE and raw(SR, packed=True) == ERR_STATE
    ctx.set_variant(AUTO)
    torch.cuda.synchronize()
    assert ctx.launch_count == n0, "a refused call launched"
    for o in (o32, o8):
        assert (o.idx.cpu().numpy() == -9).all() and (o.delta.cpu().numpy() == -1).all() and (o.tab.cpu().numpy() == -7).all()
    assert all(np.array_equal(a, b) for a, b in zip(ctx.table(), before))
    # the last accepted step: step + 2 = 2^47
    assert raw(SR, (1 << 47) - 2) == 0
    torch.cuda.synchronize()
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


# ---- 6. a peer that never arrives ------------------------------------------------------------------------------
def _lone_rank_main(rank, conn, peer_conn, R0, packed):
    """rank 0 issues one rounds call; rank 1 attaches and never launches, so rank 0's first pull gives up (~2 s)"""
    sys.path.insert(0, ROOT)
    import torch
    import elastic_gpu_agent_b200 as e
    torch.cuda.set_device(0)
    a = e.BestFitAllocator(0)
    a.set_table(pe.PREFIX_FC, pe.PREFIX_FM)
    mine = a.peer_export()
    peer_conn.send(mine)
    other = peer_conn.recv()
    a.peer_attach(rank, 2, [mine, other] if rank == 0 else [other, mine])
    if rank == 1:
        assert peer_conn.recv() == "done"
        a.peer_detach()
        a.close()
        return
    D = pe.PREFIX_FC.size
    rc, rm = pe._prefix_requests(3000, R0)
    c, m, _ = rows_in(torch, rc, rm, D, packed, oddities=False)
    o = dr.Out(torch, R0, D, packed)
    torch.cuda.synchronize()
    t0 = time.monotonic()
    shard_call(a, torch, c, m, o, 0)
    torch.cuda.synchronize()
    elapsed = time.monotonic() - t0
    idx = o.idx.cpu().numpy().astype(np.int32)
    res = (idx[:R0], o.delta.cpu().numpy(), o.tab.cpu().numpy(), idx[R0:])
    fc, fm, ov = a.table()
    timeout = a.peer_last_timeout
    one = np.array([1], np.int32)
    i1 = np.empty(1, np.int32)
    a.set_table([100], [MEM_MAX])
    rounds_rc = a._lib.egpu_bestfit_batch(a.handle, C.c_void_p(one.ctypes.data), C.c_void_p(one.ctypes.data), 1,
                                          C.c_void_p(i1.ctypes.data), None, None, dr.DR)
    conn.send((res, fc, fm, ov, timeout, rounds_rc, elapsed))
    peer_conn.send("done")
    a.peer_detach()
    a.close()


@pytest.mark.gpu
@pytest.mark.parametrize("R0,packed", [(40_000, False), (40_000, True), (300, False)],
                         ids=["more-ctas-than-devices-int32", "more-ctas-than-devices-packed", "one-cta-per-device-int32"])
def test_shard_rounds_peer_never_arrives(R0, packed, oracle_c):
    """the documented way out of a missing peer: round 1 commits nothing - every row that chose a device in the scan
    ends EGPU_IDX_DEFERRED, the infeasible ones -1 - its sums and table' are left unwritten, the table is unchanged,
    egpu_peer_last_timeout names step 0, and the launch ends on its own within the ~2 s bound"""
    import torch.multiprocessing as mp
    mctx = mp.get_context("spawn")
    a_conn, b_conn = mctx.Pipe()
    res_r, res_w = mctx.Pipe(False)
    procs = [mctx.Process(target=_lone_rank_main, args=(0, res_w, a_conn, R0, packed)),
             mctx.Process(target=_lone_rank_main, args=(1, None, b_conn, R0, packed))]
    for p in procs:
        p.start()
    try:
        assert res_r.poll(240), "rank 0 did not finish"
        res, fc, fm, ov, timeout, rounds_rc, elapsed = res_r.recv()
        for p in procs:
            p.join(60)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
    assert all(p.exitcode == 0 for p in procs)
    rc, rm = pe._prefix_requests(3000, R0)
    snap = oracle_c.snapshot(pe.PREFIX_FC, pe.PREFIX_FM, rc, rm)[0]
    idx, dl, tab, guard = res
    assert (snap >= 0).any()
    assert np.array_equal(idx, np.where(snap >= 0, -2, snap)), "a row kept a device it was never committed to"
    assert (guard == -9).all() and (dl == -1).all() and (tab == -7).all(), "sums or table' written"
    assert np.array_equal(fc, pe.PREFIX_FC) and np.array_equal(fm, pe.PREFIX_FM) and not ov.any(), "the table changed"
    assert timeout == 1, "egpu_peer_last_timeout: step 0 + 1"
    assert rounds_rc in (0, -3)
    assert elapsed < 10, f"the launch took {elapsed:.1f} s to give up"
