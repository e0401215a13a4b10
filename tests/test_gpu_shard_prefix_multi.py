"""K sharded prefix-commits in one launch: egpu_bestfit_batches_shard_dev with EGPU_F_PREFIX_COMMIT
[| EGPU_F_COMMIT] [| EGPU_F_PACKED].

Batch k is one egpu_bestfit_batch_shard_prefix_dev call with step = first_step + 2k, run by the persistent
shard_prefix_multi_sorted_kernel / shard_prefix_multi_lut_kernel in one cooperative launch.  Every GPU case compares
exactly with the C oracle's prefix-commit applied batch after batch (with commit, on the table the batch before left)
and, where it says so, with the K single calls issued in order on one stream:

  1. (CPU) the header documents the flag set; the wrapper passes exactly those flags, and a NULL d_req_mem when packed;
  2. world 1 at every D bucket under AUTO, SORTED and LUT, int32 and packed, with and without commit, ragged batches
     with R = 0 and out-of-range words, K = 1, 2 and 64: indices, per-batch sums and table', the installed table,
     sticky oversubscription flags, one launch;
  3. three K = 64 launches back to back: 384 exchange steps, past the 256-slot ring;
  4. one launch captured in a CUDA graph, replayed before and after egpu_table_set;
  5. world 2 (two processes on one GPU, started together by the gate): both ranks on the new launch, one on it and
     the other on single calls, one rank packed and the other int32, a batch with more CTAs than devices; and a peer
     that attaches but never launches: the batch in progress commits nothing and the later ones are not written;
  6. refusals: nothing launched, nothing written.
Every GPU test ends with a host-form device-rounds call that reports a grid-barrier timeout of any launch on its
context (the `ctx` fixture of test_gpu_device_rounds), and checks egpu_peer_last_timeout.
"""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_device_rounds as dr  # noqa: E402  (the ctx fixture: reports grid-barrier timeouts)
import test_gpu_kernel_matrix as km  # noqa: E402  (cell tables and cases, pack / unpack, packed_words, int32 device arrays)
import test_gpu_packed_multi as pm  # noqa: E402  (words, packed Out, stream handle)
import test_gpu_packed_shard as ps  # noqa: E402  (Out32, attach)
import test_gpu_peer_exchange as pe  # noqa: E402  (rank-major prefix-commit requests and per-rank sums)

ctx = dr.ctx
ROOT = pm.ROOT
MEM_MAX = (1 << 18) - 1
ERR_INVALID, ERR_NO_TABLE, ERR_STATE = -1, -5, -6
AUTO, GRID, SORTED, LUT = 0, 1, 2, 3
F_COMMIT, F_INPUTS_READY, F_PREFIX, F_APPLY, F_PACKED, F_ROUNDS, F_DEVICE_ROUNDS = 1, 2, 4, 8, 16, 32, 128
D_BUCKETS = (1, 8, 9, 16, 17, 33, 64)
VNAME = ["auto", "grid", "sorted", "lut"]
COUNTS = (513, 0, 4099, 1, 40_003, 5)


def test_shard_prefix_multi_documented():
    src = open(os.path.join(ROOT, "include", "egpu_alloc.h")).read()
    block = src[src.index("K sharded prefix-commits in one launch"):src.index("int egpu_bestfit_batches_shard_dev(")]
    assert re.search(r"EGPU_F_PREFIX_COMMIT \[\| EGPU_F_COMMIT\] \[\| EGPU_F_PACKED\]", block)
    assert "stays 1011" in block and "first_step + 2K > 2^47" in block
    assert "EGPU_ERR_ABI" not in src


def test_wrapper_flags(egpu):
    """bestfit_batches_shard_prefix_dev passes exactly the flag set, first_step and, packed, a NULL d_req_mem"""
    calls = []

    class Lib:
        def __getattr__(self, name):
            return lambda *a: calls.append((name, a)) or 0

    a = object.__new__(egpu.BestFitAllocator)
    a._lib, a._h = Lib(), C.c_void_p(1)
    a.bestfit_batches_shard_prefix_dev([(16, 32, 5, 48, 0, 0)], 6)
    a.bestfit_batches_shard_prefix_dev([(16, 32, 5, 48, 0, 0)], 8, commit=True)
    a.bestfit_batches_shard_prefix_dev([(16, 5, 48, 0, 0), (64, 0, 80, 0, 0)], 10, commit=True, packed=True)
    a.bestfit_batches_shard_prefix_dev([(16, 5, 48, 0, 0)], 12, packed=True)
    assert [n for n, _ in calls] == ["egpu_bestfit_batches_shard_dev"] * 4
    assert [c[1][3] for c in calls] == [F_PREFIX, F_PREFIX | F_COMMIT, F_PREFIX | F_COMMIT | F_PACKED, F_PREFIX | F_PACKED]
    assert [c[1][4] for c in calls] == [6, 8, 10, 12]
    assert calls[0][1][1][0].d_req_mem == 32
    for _, args in calls[2:]:
        assert all(b.d_req_mem is None for b in args[1]) and args[2] == len(args[1])
    a._lib = None
    a._h = None


# ---- references and calls ------------------------------------------------------------------------------
def batch_rows(D, tname, counts, packed):
    """per batch the device input (int32 pair, or words with out-of-range ones) and the requests it stands for"""
    rows = []
    for k, R in enumerate(counts):
        _, _, rc, rm = km.cell_case(D, tname, R)
        if k % 2:
            rc, rm = rc[::-1].copy(), rm[::-1].copy()
        if packed:
            words = km.packed_words(rc, rm, R, D)
            rows.append((words, km.unpack(words)))
        else:
            rows.append(((rc, rm), (rc, rm)))
    return rows


def chain_ref(oracle_c, fc, fm, reqs, commit):
    """per batch (idx, dc, dm, table') of the oracle's prefix-commit, batch after batch, and the table left"""
    out = []
    fc, fm = np.asarray(fc, np.int32), np.asarray(fm, np.int32)
    D = fc.size
    for rc, rm in reqs:
        e = oracle_c.prefix_commit(fc, fm, rc, rm)
        out.append(e)
        if commit:
            fc, fm = e[3][:D].astype(np.int32), e[3][D:2 * D].astype(np.int32)
    return out, (fc, fm)


class Call:
    """device inputs and sentinel-filled outputs of a batch list"""

    def __init__(self, torch, rows, D, packed):
        self.packed = packed
        self.inp, self.outs, self.tup = [], [], []
        for x, (rc, _) in rows:
            R = len(rc)
            if packed:
                w = pm.words_dev(torch, x)
                o = pm.Out(torch, R, D)
                self.inp.append(w)
                self.tup.append((w.data_ptr(), R) + o.ptrs())
            else:
                c, m = km._dev(torch, x[0]), km._dev(torch, x[1])
                o = ps.Out32(torch, R, D)
                self.inp.append((c, m))
                self.tup.append((c.data_ptr(), m.data_ptr(), R) + o.ptrs())
            self.outs.append(o)

    def array(self, alloc):
        return alloc.make_packed_batches(self.tup) if self.packed else alloc.make_batches(self.tup)

    def reset(self):
        for o in self.outs:
            o.idx.fill_(-9)
            o.delta.fill_(-1)
            o.tab.fill_(-7)

    def check(self, exp, where):
        for k, (o, e) in enumerate(zip(self.outs, exp)):
            o.check(e, f"{where}, batch {k}")

    def got(self):
        return [(o.idx.cpu().numpy().copy(), o.delta.cpu().numpy().copy(), o.tab.cpu().numpy().copy()) for o in self.outs]


def launch(alloc, torch, call, first_step, commit, stream=None):
    s = torch.cuda.current_stream().cuda_stream if stream is None else stream
    alloc.bestfit_batches_shard_prefix_dev(call.array(alloc), first_step, commit=commit, packed=call.packed, stream=s)


def single_calls(alloc, torch, call, first_step, commit):
    """the K egpu_bestfit_batch_shard_prefix_dev calls the launch stands for, on one stream"""
    s = torch.cuda.current_stream().cuda_stream
    for k, (t, o) in enumerate(zip(call.tup, call.outs)):
        i, dl, tb = o.ptrs()
        if call.packed:
            alloc.bestfit_shard_prefix_packed_dev(t[0], o.R, i, dl, tb, first_step + 2 * k, commit, s)
        else:
            alloc.bestfit_shard_prefix_dev(t[0], t[1], o.R, i, dl, tb, first_step + 2 * k, commit, s)


def installed(alloc, fc, fm, ov=None):
    return pm.table_is(alloc, np.asarray(fc, np.int32), np.asarray(fm, np.int32), ov)


# ---- 2. world 1, every D bucket -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [AUTO, SORTED, LUT], ids=lambda v: VNAME[v])
@pytest.mark.parametrize("D", D_BUCKETS)
def test_shard_prefix_multi_world1(variant, D, ctx, oracle_c):
    """every table of the cell matrix, both formats, with and without commit: the oracle chain, then the single calls
    on the same buffers give the same bytes; one launch per call"""
    import torch
    ctx.set_variant(variant)
    ps.attach(ctx)
    step = 0
    for tname, (fc, fm) in km.cell_tables(D).items():
        for packed in (False, True):
            rows = batch_rows(D, tname, COUNTS, packed)
            call = Call(torch, rows, D, packed)
            for commit in (False, True):
                where = f"{VNAME[variant]}, D = {D}, table {tname}, {'packed' if packed else 'int32'}, commit {commit}"
                exp, left = chain_ref(oracle_c, fc, fm, [r for _, r in rows], commit)
                ctx.set_table(fc, fm)
                call.reset()
                torch.cuda.synchronize()
                n0 = ctx.launch_count
                launch(ctx, torch, call, step, commit)
                assert ctx.launch_count - n0 == 1, f"{where}: one launch"
                torch.cuda.synchronize()
                call.check(exp, where)
                assert installed(ctx, *left), f"{where}: installed table"
                got = call.got()
                ctx.set_table(fc, fm)
                call.reset()
                single_calls(ctx, torch, call, step + 2 * len(rows), commit)
                torch.cuda.synchronize()
                for k, (g, s) in enumerate(zip(got, call.got())):
                    assert all(np.array_equal(x, y) for x, y in zip(g, s)), f"{where}, batch {k}: differs from the single calls"
                assert installed(ctx, *left), f"{where}: installed table after the single calls"
                step += 4 * len(rows)
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(SORTED, 8), (LUT, 64), (AUTO, 17)])
@pytest.mark.parametrize("packed", [False, True])
def test_shard_prefix_multi_batch_counts(variant, D, packed, ctx, oracle_c):
    """K = 1, 2 and 64 (ragged, empty batches among them), committing: the oracle chain"""
    import torch
    ctx.set_variant(variant)
    ps.attach(ctx)
    fc, fm = km.cell_tables(D)["dups"]
    step = 0
    for counts in ((4099,), (0, 513), tuple((0, 1, 3, 5, 511, 513, 4099)[k % 7] for k in range(64))):
        rows = batch_rows(D, "dups", counts, packed)
        exp, left = chain_ref(oracle_c, fc, fm, [r for _, r in rows], True)
        call = Call(torch, rows, D, packed)
        ctx.set_table(fc, fm)
        torch.cuda.synchronize()
        n0 = ctx.launch_count
        launch(ctx, torch, call, step, True)
        assert ctx.launch_count - n0 == 1
        torch.cuda.synchronize()
        call.check(exp, f"K = {len(counts)}")
        assert installed(ctx, *left), f"K = {len(counts)}: installed table"
        step += 2 * len(counts)
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT], ids=lambda v: VNAME[v])
@pytest.mark.parametrize("packed", [False, True])
def test_shard_prefix_multi_keeps_oversubscription_flags(variant, packed, ctx, oracle_c):
    """a table with sticky oversubscription flags: the committing launch keeps them"""
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
    reqs = [(rng.integers(0, 12, R).astype(np.int32), rng.integers(0, 300, R).astype(np.int32)) for R in (5001, 0, 20_001)]
    rows = [((km.pack(rc, rm), (rc, rm)) if packed else ((rc, rm), (rc, rm))) for rc, rm in reqs]
    exp, left = chain_ref(oracle_c, fc1, fm1, reqs, True)
    call = Call(torch, rows, D, packed)
    launch(ctx, torch, call, 0, True)
    torch.cuda.synchronize()
    call.check(exp, "sticky flags")
    assert installed(ctx, *left, ov1)
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


# ---- 3. the exchange ring ------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True])
def test_shard_prefix_multi_wraps_the_ring(packed, ctx, oracle_c, egpu):
    """three K = 64 committing launches back to back: 384 exchange steps, more than the 256 slots"""
    import torch
    w = egpu.synth.workload("cfg3")
    fc, fm = np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32)
    D = fc.size
    ps.attach(ctx)
    ctx.set_table(fc, fm)
    rng = np.random.default_rng(31)
    calls, exps = [], []
    cur = (fc, fm)
    for j in range(3):
        reqs = [tuple(x.astype(np.int32) for x in egpu.synth.requests(3, 300 + 64 * j + k, int(rng.integers(0, 700))))
                for k in range(64)]
        rows = [((km.pack(rc, rm), km.unpack(km.pack(rc, rm))) if packed else ((rc, rm), (rc, rm))) for rc, rm in reqs]
        exp, cur = chain_ref(oracle_c, *cur, [r for _, r in rows], True)
        calls.append(Call(torch, rows, D, packed))
        exps.append(exp)
    torch.cuda.synchronize()
    for j, call in enumerate(calls):
        launch(ctx, torch, call, 128 * j, True)
    torch.cuda.synchronize()
    for j, (call, exp) in enumerate(zip(calls, exps)):
        call.check(exp, f"launch {j}")
    assert installed(ctx, *cur)
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


# ---- 4. CUDA graph -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(SORTED, 8), (LUT, 64), (AUTO, 33)])
@pytest.mark.parametrize("packed", [False, True])
def test_shard_prefix_multi_graph_replay(variant, D, packed, ctx, oracle_c):
    """one committing launch captured in a CUDA graph, replayed twice with an egpu_table_set between: each replay
    equals its eager run and the oracle"""
    import torch
    tables = km.cell_tables(D)
    rows = batch_rows(D, "dups", (4099, 0, 40_003, 513), packed)
    ctx.set_variant(variant)
    ps.attach(ctx)
    call = Call(torch, rows, D, packed)
    s = torch.cuda.Stream()
    ctx.set_table(*tables["dups"])
    with torch.cuda.stream(s):
        launch(ctx, torch, call, 0, True, s.cuda_stream)  # warm-up outside the capture: scratch and occupancy
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        launch(ctx, torch, call, 0, True, s.cuda_stream)
    for tname in ("dups", "spread"):
        fc, fm = tables[tname]
        exp, left = chain_ref(oracle_c, fc, fm, [r for _, r in rows], True)
        ctx.set_table(fc, fm)
        call.reset()
        torch.cuda.synchronize()
        launch(ctx, torch, call, 0, True)
        torch.cuda.synchronize()
        eager = call.got()
        call.check(exp, f"eager, table {tname}")
        ctx.set_table(fc, fm)
        call.reset()
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        for k, (e, r) in enumerate(zip(eager, call.got())):
            assert all(np.array_equal(x, y) for x, y in zip(e, r)), f"replay, table {tname}, batch {k}"
        assert installed(ctx, *left), f"replay, table {tname}: installed table"
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


# ---- 5. world 2: two processes on one GPU --------------------------------------------------------------------------
# (rows of rank 0, rows of rank 1); 40 000 rows at D = 8 give a grid of more CTAs than devices (the CTAs that cut
# nothing wait at barrier 2 while CTAs 0..7 exchange)
W2_STEPS = [(300, 200), (7, 2_001), (0, 64), (40_000, 30_001), (1_000, 1_000), (5, 5), (2_500, 3)]


def _rank_main(rank, conn, peer_conn, how, packed):
    """One rank on cuda:0: the W2_STEPS batches, committing, either as one launch ("multi") or as single calls
    ("single"), twice from a fresh table: once as a warm-up, then started together with the other rank through the
    gate.  The warm-up loads every kernel and allocates the scratch first: a kernel's first launch loads its module,
    which waits for the kernels running on the context - the gate among them, which waits for the host - so nothing
    between gate_dev and gate_open may launch a kernel for the first time."""
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
    rows = []
    for k, (n0, n1) in enumerate(W2_STEPS):
        rc, rm = pe._prefix_requests(2000 + k, n0 + n1)
        rc, rm = (np.ascontiguousarray(x[:n0] if rank == 0 else x[n0:]) for x in (rc, rm))
        rows.append(((km.pack(rc, rm), (rc, rm)) if packed else ((rc, rm), (rc, rm))))
    call = Call(torch, rows, D, packed)
    s = torch.cuda.current_stream().cuda_stream
    res = []
    for first_step, gated in ((0, False), (2 * len(rows), True)):
        a.set_table(pe.PREFIX_FC, pe.PREFIX_FM)
        call.reset()
        torch.cuda.synchronize()
        if gated:
            a.gate_dev(s)
        if how == "multi":
            launch(a, torch, call, first_step, True, s)
        else:
            single_calls(a, torch, call, first_step, True)
        if gated:
            a.gate_open()
        torch.cuda.synchronize()
        res.append([(i[:o.R].astype(np.int32), dl, t) for (i, dl, t), o in zip(call.got(), call.outs)])
    fc, fm, _ = a.table()
    # a host-form device-rounds call reports a grid-barrier timeout of any launch on this context
    one = np.array([1], np.int32)
    idx = np.empty(1, np.int32)
    a.set_table([100], [MEM_MAX])
    rounds_rc = a._lib.egpu_bestfit_batch(a.handle, C.c_void_p(one.ctypes.data), C.c_void_p(one.ctypes.data), 1,
                                          C.c_void_p(idx.ctypes.data), None, None, dr.DR)
    conn.send((rank, res, fc, fm, a.peer_last_timeout, a.gate_timeouts, rounds_rc))
    peer_conn.send("done")
    peer_conn.recv()
    a.peer_detach()
    a.close()


def _run_world2(hows, formats):
    import torch.multiprocessing as mp
    mctx = mp.get_context("spawn")
    a_conn, b_conn = mctx.Pipe()
    res0_r, res0_w = mctx.Pipe(False)
    res1_r, res1_w = mctx.Pipe(False)
    procs = [mctx.Process(target=_rank_main, args=(0, res0_w, a_conn, hows[0], formats[0])),
             mctx.Process(target=_rank_main, args=(1, res1_w, b_conn, hows[1], formats[1]))]
    for p in procs:
        p.start()
    try:
        assert res0_r.poll(240) and res1_r.poll(240), "ranks did not finish"
        r0, r1 = res0_r.recv(), res1_r.recv()
        for p in procs:
            p.join(60)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
    assert all(p.exitcode == 0 for p in procs)
    for r in (r0, r1):
        assert r[4] == 0, f"rank {r[0]}: a peer pull timed out at step + 1 = {r[4]}"
        assert r[5] == 0, f"rank {r[0]}: the start gate timed out"
        assert r[6] == 0, f"rank {r[0]}: a grid barrier timed out"
    return r0, r1


W2_CASES = [(("multi", "multi"), (False, False)), (("multi", "multi"), (True, True)), (("multi", "single"), (False, False)),
            (("single", "multi"), (True, False)), (("multi", "multi"), (True, False))]


@pytest.mark.gpu
@pytest.mark.parametrize("hows,formats", W2_CASES,
                         ids=[f"{h[0]}-{h[1]}-{'-'.join('packed' if f else 'int32' for f in fs)}" for h, fs in W2_CASES])
def test_shard_prefix_multi_world2(hows, formats, oracle_c):
    r0, r1 = _run_world2(hows, formats)
    D = pe.PREFIX_FC.size
    for p, where in enumerate(("warm-up", "gated")):
        cur_c, cur_m = pe.PREFIX_FC, pe.PREFIX_FM
        for k, (n0, n1) in enumerate(W2_STEPS):
            rc, rm = pe._prefix_requests(2000 + k, n0 + n1)
            o_idx, _, _, o_tab = oracle_c.prefix_commit(cur_c, cur_m, rc, rm)
            (i0, d0, t0), (i1, d1, t1) = r0[1][p][k], r1[1][p][k]
            assert np.array_equal(i0, o_idx[:n0]) and np.array_equal(i1, o_idx[n0:]), f"{where}: indices, batch {k}"
            assert np.array_equal(d0, pe._rank_partial(o_idx[:n0], rc[:n0], rm[:n0], D)), f"{where}: rank 0 sums, batch {k}"
            assert np.array_equal(d1, pe._rank_partial(o_idx[n0:], rc[n0:], rm[n0:], D)), f"{where}: rank 1 sums, batch {k}"
            assert np.array_equal(t0, o_tab) and np.array_equal(t1, o_tab), f"{where}: table', batch {k}"
            cur_c, cur_m = o_tab[:D].copy(), o_tab[D:2 * D].copy()
    for r in (r0, r1):
        assert np.array_equal(r[2], cur_c) and np.array_equal(r[3], cur_m), f"rank {r[0]}: installed table"


# ---- 5b. a peer that never arrives -----------------------------------------------------------------------------------
def _lone_rank_main(rank, conn, peer_conn, R0, packed):
    """rank 0 launches three committing batches; rank 1 attaches and never launches, so every wait of rank 0 for it
    gives up (about 2 s) in batch 0"""
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
    rows = []
    for k, n in enumerate((R0, 513, 7)):
        rc, rm = pe._prefix_requests(3000 + k, n)
        rows.append(((km.pack(rc, rm), (rc, rm)) if packed else ((rc, rm), (rc, rm))))
    call = Call(torch, rows, D, packed)
    torch.cuda.synchronize()
    launch(a, torch, call, 0, True)
    torch.cuda.synchronize()
    res = [(i[:o.R].astype(np.int32), dl, t, i[o.R:]) for (i, dl, t), o in zip(call.got(), call.outs)]
    fc, fm, ov = a.table()
    timeout = a.peer_last_timeout
    one = np.array([1], np.int32)
    idx = np.empty(1, np.int32)
    a.set_table([100], [MEM_MAX])
    rounds_rc = a._lib.egpu_bestfit_batch(a.handle, C.c_void_p(one.ctypes.data), C.c_void_p(one.ctypes.data), 1,
                                          C.c_void_p(idx.ctypes.data), None, None, dr.DR)
    conn.send((res, fc, fm, ov, timeout, rounds_rc))
    peer_conn.send("done")
    a.peer_detach()
    a.close()


@pytest.mark.gpu
@pytest.mark.parametrize("R0,packed", [(40_000, False), (40_000, True), (300, False)],
                         ids=["more-ctas-than-devices-int32", "more-ctas-than-devices-packed", "one-cta-per-device-int32"])
def test_shard_prefix_multi_peer_never_arrives(R0, packed, oracle_c):
    """the documented way out of a missing peer: batch 0 commits nothing - every row that chose a device in the scan
    ends EGPU_IDX_DEFERRED, the infeasible ones -1 - its sums and table' and the later batches are left unwritten, the
    table is unchanged and egpu_peer_last_timeout names step 0.  With 40 000 rows the CTAs without a device give up
    at barrier 2 before the pulls do (counted as a grid-barrier timeout); with 300 rows every CTA is pulling."""
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
        res, fc, fm, ov, timeout, rounds_rc = res_r.recv()
        for p in procs:
            p.join(60)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
    assert all(p.exitcode == 0 for p in procs)
    rc, rm = pe._prefix_requests(3000, R0)
    snap = oracle_c.snapshot(pe.PREFIX_FC, pe.PREFIX_FM, rc, rm)[0]
    idx, dl, tab, guard = res[0]
    assert (snap >= 0).any()
    assert np.array_equal(idx, np.where(snap >= 0, -2, snap)), "batch 0: a row kept a device it was never committed to"
    assert (guard == -9).all() and (dl == -1).all() and (tab == -7).all(), "batch 0: sums or table' written"
    for k, (i, d, t, g) in enumerate(res[1:], 1):
        assert (i == -9).all() and (g == -9).all() and (d == -1).all() and (t == -7).all(), f"batch {k} was written"
    assert np.array_equal(fc, pe.PREFIX_FC) and np.array_equal(fm, pe.PREFIX_FM) and not ov.any(), "the table changed"
    assert timeout == 1, "egpu_peer_last_timeout: step 0 + 1"
    if R0 > 2048 * pe.PREFIX_FC.size:
        assert rounds_rc == -3, "the CTAs without a device should have given up at barrier 2 first"


# ---- 6. refusals -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_shard_prefix_multi_refusals(ctx):
    import torch
    from elastic_gpu_agent_b200 import _lib as L
    D = 8
    fc, fm = km.cell_tables(D)["dups"]
    c32 = Call(torch, batch_rows(D, "dups", (513, 4099), False), D, False)
    c8 = Call(torch, batch_rows(D, "dups", (513, 4099), True), D, True)
    lib, h = ctx._lib, ctx.handle
    s = pm._s(torch)

    def raw(batches, flags, first_step=0):
        arr = (L.Batch * max(1, len(batches)))(*[L.Batch(*b) for b in batches])
        return lib.egpu_bestfit_batches_shard_dev(h, arr, len(batches), flags, first_step, s)

    def tup(call, k, **kw):
        b = call.array(ctx)[k]
        t = dict(c=b.d_req_core, m=b.d_req_mem, R=b.R, i=b.d_out_idx, dl=b.d_delta, to=b.d_table_out)
        t.update(kw)
        return (t["c"], t["m"], t["R"], t["i"], t["dl"], t["to"])

    PC = F_PREFIX | F_COMMIT
    # no table, then unattached
    assert raw([tup(c32, 0)], PC) == ERR_NO_TABLE
    ctx.set_table(fc, fm)
    assert raw([tup(c32, 0)], PC) == ERR_STATE and raw([tup(c8, 0)], PC | F_PACKED) == ERR_STATE
    ps.attach(ctx)
    before = ctx.table()
    c32.reset()
    c8.reset()
    torch.cuda.synchronize()
    n0 = ctx.launch_count
    for f in (F_PACKED, F_PACKED | F_COMMIT, PC | F_APPLY, PC | F_INPUTS_READY, F_PREFIX | F_INPUTS_READY, PC | F_ROUNDS,
              PC | F_DEVICE_ROUNDS, PC | F_ROUNDS | F_DEVICE_ROUNDS, PC | 64, PC | 256):
        for call, P in ((c32, 0), (c8, F_PACKED)):
            assert raw([tup(call, 0), tup(call, 1)], f | P) == ERR_INVALID, (f, P)
    for call, P in ((c32, 0), (c8, F_PACKED)):
        fmt = "packed" if P else "int32"
        b0, b1 = tup(call, 0), tup(call, 1)
        refused = {
            "K = 0": ([], 0),
            "K = 65": ([tup(call, 0, R=1, i=b0[3] + 16 * k, dl=None, to=None) for k in range(65)], 0),
            "first_step + 2K > 2^47": ([b0, b1], (1 << 47) - 3),
            "first_step >= 2^47": ([b0], 1 << 47),
            "R >= 2^31": ([b0, tup(call, 1, R=1 << 31)], 0),
            "NULL req_core": ([b0, tup(call, 1, c=None)], 0),
            "NULL indices": ([b0, tup(call, 1, i=None)], 0),
            "misaligned req_core": ([b0, tup(call, 1, c=b1[0] + 4)], 0),
            "misaligned indices": ([b0, tup(call, 1, i=b1[3] + (1 if P else 4))], 0),
            "overlapping indices": ([b0, tup(call, 1, i=b0[3] + 16 * (1 if P else 4))], 0),
            "overlapping demand sums": ([b0, tup(call, 1, dl=b0[4] + 8)], 0),
            "overlapping table'": ([b0, tup(call, 1, to=b0[5])], 0),
            "table' over demand sums": ([b0, tup(call, 1, to=b0[4])], 0),
        }
        if P:
            refused["req_mem with EGPU_F_PACKED"] = ([b0, tup(call, 1, m=c32.array(ctx)[1].d_req_mem)], 0)
        else:
            refused["NULL req_mem without EGPU_F_PACKED"] = ([b0, tup(call, 1, m=None)], 0)
            refused["misaligned req_mem"] = ([b0, tup(call, 1, m=b1[1] + 4)], 0)
        for what, (batches, first) in refused.items():
            assert raw(batches, PC | P, first) == ERR_INVALID, f"{fmt}: {what}"
    ctx.set_variant(GRID)
    assert raw([tup(c32, 0)], PC) == ERR_STATE and raw([tup(c8, 0)], PC | F_PACKED) == ERR_STATE
    ctx.set_variant(AUTO)
    torch.cuda.synchronize()
    assert ctx.launch_count == n0, "a refused call launched"
    for call in (c32, c8):
        for o in call.outs:
            assert (o.idx.cpu().numpy() == -9).all() and (o.delta.cpu().numpy() == -1).all() and (o.tab.cpu().numpy() == -7).all()
    assert all(np.array_equal(a, b) for a, b in zip(ctx.table(), before))
    # the last accepted step: first_step + 2K = 2^47
    assert raw([tup(c32, 0), tup(c32, 1)], PC, (1 << 47) - 4) == 0
    torch.cuda.synchronize()
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()
