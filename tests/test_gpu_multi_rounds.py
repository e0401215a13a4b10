"""Batches placed in order, each to the fixed point, in one launch: egpu_bestfit_batches_dev with
EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT | EGPU_F_ROUNDS | EGPU_F_DEVICE_ROUNDS [| EGPU_F_PACKED].

Batch k runs the rounds of egpu_bestfit_batch_dev with EGPU_F_DEVICE_ROUNDS against the table batches 0..k-1
committed, all K in one launch of the multi-batch rounds kernels (rounds_sorted_multi_kernel /
rounds_lut_multi_kernel).  Every GPU case compares exactly with the C rounds oracle chained batch after batch
(table and sticky oversubscription flags carried over), in both row formats:

  1. the chain at every D bucket under AUTO, SORTED and LUT: indices, per-batch sums and table', the installed
     table, guard elements after every index array, exactly one launch;
  2. agreement with K consecutive single-batch calls (K = 1 included);
  3. the known answer that tells batch after batch from one rounds call on the concatenation;
  4. ragged, empty and 64-batch lists, and a node that fills in batch 1;
  5. 1 Mi-row batches at cfg3 and cfg4;
  6. sticky oversubscription flags;
  7. asynchrony, stream order and CUDA-graph capture;
  8. a seeded sequence of table-changing calls on one context, read back against an int64 model;
  9. refusals: nothing launched, nothing written.
Every GPU test ends with a host-form device-rounds call that would report a grid-barrier timeout of any launch on
its context (the `ctx` fixture of test_gpu_device_rounds).
"""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_context_sequences as cs  # noqa: E402  (the int64 table model, random tables and requests)
import test_gpu_device_rounds as dr  # noqa: E402  (Out, rows_dev, ref, single calls, the ctx fixture)
import test_gpu_kernel_matrix as km  # noqa: E402  (cell tables, pack / unpack, int32 device arrays)
import test_gpu_packed_multi as pm  # noqa: E402  (words, stream handle)

ctx = dr.ctx
MEM_MAX = dr.MEM_MAX
ERR_INVALID, ERR_NO_TABLE, ERR_STATE = dr.ERR_INVALID, dr.ERR_NO_TABLE, dr.ERR_STATE
AUTO, GRID, SORTED, LUT = dr.AUTO, dr.GRID, dr.SORTED, dr.LUT
F_COMMIT, F_INPUTS_READY, F_PREFIX, F_APPLY, F_PACKED, F_ROUNDS = 1, 2, 4, 8, 16, 32
DR = dr.DR
D_BUCKETS = (1, 8, 9, 16, 17, 33, 64)
VNAME = ["auto", "grid", "sorted", "lut"]


def test_multi_rounds_documented_and_versioned():
    src = open(os.path.join(pm.ROOT, "include", "egpu_alloc.h")).read()
    head = src[:src.index("#define EGPU_MAX_BATCHES")]
    block = head[head.rindex("Several batches in ONE launch"):]
    assert re.search(r"EGPU_F_PREFIX_COMMIT \|\s+\*\s+EGPU_F_COMMIT \| EGPU_F_ROUNDS \| EGPU_F_DEVICE_ROUNDS", block)
    assert "a multi-batch launch never commits" not in src
    assert "1.11 EGPU_F_DEVICE_ROUNDS on egpu_bestfit_batches_dev" in src
    from elastic_gpu_agent_b200 import _lib as L
    try:
        lib = L.load()
    except OSError:
        return  # the library is not built here: the header is what can be checked
    assert lib.egpu_abi_version() == 1011


# ---- references and calls ------------------------------------------------------------------------------
def as_requests(rc, rm, packed):
    """the requests the call is compared against: packed words stand for their unpacked requests"""
    return dr.packed_requests(rc, rm) if packed else (rc, rm)


def chain_ref(oracle_c, fc, fm, rows, packed, ov=None):
    """per batch (idx, delta, table'), and the installed (fc, fm, oversub): the C rounds oracle batch after batch"""
    per = []
    ov = np.zeros(len(fc), np.int32) if ov is None else ov
    for rc, rm in rows:
        e = dr.ref(oracle_c, fc, fm, *as_requests(rc, rm, packed), ov)
        per.append(e[:3])
        fc, fm = e[3][0], e[3][1]
    return per, (np.asarray(fc, np.int32), np.asarray(fm, np.int32), ov)


class Call:
    """device rows and sentinel-filled outputs of a batch list, and its egpu_batch array"""

    def __init__(self, torch, rows, D, packed):
        from elastic_gpu_agent_b200 import _lib as L
        self.packed = packed
        self.dev = [dr.rows_dev(torch, rc, rm, packed) for rc, rm in rows]
        self.outs = [dr.Out(torch, len(rc), D, packed) for rc, _ in rows]
        self.arr = (L.Batch * len(rows))()
        for k, ((c, m), o) in enumerate(zip(self.dev, self.outs)):
            i, dl, t = o.ptrs()
            self.arr[k] = L.Batch(c.data_ptr(), m.data_ptr() if m is not None else None, o.R, i, dl, t)

    def reset(self):
        for o in self.outs:
            o.idx.fill_(-9)
            o.delta.fill_(-1)
            o.tab.fill_(-7)

    def got(self):
        return [o.got() for o in self.outs]


def multi(alloc, call, stream=None, flags=0):
    import torch
    s = pm._s(torch) if stream is None else stream
    return alloc._lib.egpu_bestfit_batches_dev(alloc.handle, call.arr, len(call.arr), DR | (F_PACKED if call.packed else 0) | flags, s)


def run_multi(alloc, torch, variant, fc, fm, rows, packed, set_table=True):
    """one call on the list: (per-batch (idx, delta, table'), installed table), checking it added exactly one launch"""
    alloc.set_variant(variant)
    if set_table:
        alloc.set_table(fc, fm)
    call = Call(torch, rows, len(fc), packed)
    torch.cuda.synchronize()
    n0 = alloc.launch_count
    assert multi(alloc, call) == 0, alloc._lib.egpu_last_error(alloc.handle).decode()
    assert alloc.launch_count - n0 == 1, "one launch per call"
    torch.cuda.synchronize()
    return call.got(), alloc.table()


def check_chain(got, exp, where):
    per, inst = got
    e_per, e_inst = exp
    assert len(per) == len(e_per)
    for k, (g, e) in enumerate(zip(per, e_per)):
        assert np.array_equal(g[0], e[0]), f"{where}, batch {k}: indices"
        assert np.array_equal(g[1], e[1]), f"{where}, batch {k}: demand sums"
        assert np.array_equal(g[2], e[2]), f"{where}, batch {k}: table'"
    assert all(np.array_equal(a, b) for a, b in zip(inst, e_inst)), f"{where}: installed table"


def cell_rows(D, tname, counts):
    """batches of the cell matrix's requests: batch k is the cell case of counts[k] rows, reversed for odd k"""
    rows = []
    for k, R in enumerate(counts):
        _, _, rc, rm = km.cell_case(D, tname, R)
        rows.append((rc[::-1].copy(), rm[::-1].copy()) if k % 2 else (rc, rm))
    return rows


CHAIN_COUNTS = (513, 0, 4099, 1, 40_003, 5)


# ---- 1. the oracle chain ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [AUTO, SORTED, LUT], ids=lambda v: VNAME[v])
@pytest.mark.parametrize("D", D_BUCKETS)
def test_multi_rounds_chain(variant, D, ctx, oracle_c):
    import torch
    for tname, (fc, fm) in km.cell_tables(D).items():
        rows = cell_rows(D, tname, CHAIN_COUNTS)
        for packed in (False, True):
            where = f"{VNAME[variant]}, D = {D}, table {tname}, {'packed' if packed else 'int32'}"
            check_chain(run_multi(ctx, torch, variant, fc, fm, rows, packed), chain_ref(oracle_c, fc, fm, rows, packed), where)


# ---- 2. agreement with K single-batch calls ----------------------------------------------------------------
def single_calls(alloc, torch, variant, fc, fm, rows, packed):
    """K consecutive egpu_bestfit_batch_dev calls with the same flags on one stream"""
    alloc.set_variant(variant)
    alloc.set_table(fc, fm)
    outs = []
    keep = []
    for rc, rm in rows:
        c, m = dr.rows_dev(torch, rc, rm, packed)
        o = dr.Out(torch, len(rc), len(fc), packed)
        keep.append((c, m))
        assert dr.call_dev(alloc, torch, c, m, o) == 0
        outs.append(o)
    torch.cuda.synchronize()
    return [o.got() for o in outs], alloc.table()


@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(SORTED, 8), (AUTO, 9), (SORTED, 33), (LUT, 17), (LUT, 64), (AUTO, 64)])
@pytest.mark.parametrize("packed", [False, True])
def test_multi_rounds_match_single_calls(variant, D, packed, ctx):
    import torch
    fc, fm = km.cell_tables(D)["dups"]
    for counts in (CHAIN_COUNTS, (40_003,), (0,)):
        rows = cell_rows(D, "dups", counts)
        single = single_calls(ctx, torch, variant, fc, fm, rows, packed)
        check_chain(run_multi(ctx, torch, variant, fc, fm, rows, packed), single, f"K = {len(counts)}")


# ---- 3. the known answer -------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT], ids=lambda v: VNAME[v])
@pytest.mark.parametrize("packed", [False, True])
def test_multi_rounds_known_answer(variant, packed, ctx, oracle_c):
    """free_core = [60, 100]: batch 1 = [60, 60], batch 2 = [100].  Batch after batch, batch 1's second row is
    deferred in round 1 and takes device 1 in round 2, so batch 2 finds no room; one rounds call on the
    concatenation lets the 100 take device 1 in round 1 instead."""
    import torch
    fc, fm = np.array([60, 100], np.int32), np.array([MEM_MAX, MEM_MAX], np.int32)
    rows = [(np.array([60, 60], np.int32), np.ones(2, np.int32)), (np.array([100], np.int32), np.ones(1, np.int32))]
    got = run_multi(ctx, torch, variant, fc, fm, rows, packed)
    assert [g[0].tolist() for g in got[0]] == [[0, 1], [-1]]
    assert got[0][0][1].tolist() == [60, 60, 1, 1] and got[0][1][1].tolist() == [0, 0, 0, 0]
    check_chain(got, chain_ref(oracle_c, fc, fm, rows, packed), "batch after batch")
    # the other answer: one rounds call on the concatenated rows
    cat = dr.device_rounds(ctx, torch, variant, fc, fm, np.array([60, 60, 100], np.int32), np.ones(3, np.int32), packed)
    assert cat[0].tolist() == [0, -1, 1]
    # the Python entry point gives the first answer
    ctx.set_table(fc, fm)
    call = Call(torch, rows, 2, packed)
    if packed:
        tup = [(c.data_ptr(), o.R) + o.ptrs() for (c, _), o in zip(call.dev, call.outs)]
    else:
        tup = [(c.data_ptr(), m.data_ptr(), o.R) + o.ptrs() for (c, m), o in zip(call.dev, call.outs)]
    ctx.bestfit_batches_rounds_device_dev(tup, packed=packed, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert [g[0].tolist() for g in call.got()] == [[0, 1], [-1]]


# ---- 4. batch lists --------------------------------------------------------------------------------------------
LISTS = {
    "ragged": (1, 40_003, 3, 512, 511, 4),
    "empty first": (0, 4099, 513),
    "empty middle": (4099, 0, 0, 513),
    "empty last": (4099, 513, 0),
    "all empty": (0, 0, 0),
    "one empty": (0,),
    "64": tuple((0, 1, 3, 5, 511, 513, 4099)[k % 7] for k in range(64)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(SORTED, 8), (LUT, 64), (AUTO, 17)])
@pytest.mark.parametrize("packed", [False, True])
def test_multi_rounds_batch_lists(variant, D, packed, ctx, oracle_c):
    import torch
    fc, fm = km.cell_tables(D)["dups"]
    for name, counts in LISTS.items():
        rows = cell_rows(D, "dups", counts)
        got = run_multi(ctx, torch, variant, fc, fm, rows, packed)
        check_chain(got, chain_ref(oracle_c, fc, fm, rows, packed), name)
        for (rc, _), g in zip(rows, got[0]):
            if len(rc) == 0:
                assert not g[1].any(), f"{name}: an empty batch's sums"


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT], ids=lambda v: VNAME[v])
@pytest.mark.parametrize("packed", [False, True])
def test_multi_rounds_node_fills_in_batch_1(variant, packed, ctx, oracle_c):
    """batch 1 takes every core of the node; the 63 batches after it end all -1 with zero sums, and each
    one's table' is the full node"""
    import torch
    D = 4
    fc, fm = np.full(D, 10, np.int32), np.full(D, MEM_MAX, np.int32)
    rows = [(np.full(9, 10, np.int32), np.ones(9, np.int32))]
    rng = np.random.default_rng(4)
    rows += [(rng.integers(1, 60, int(R)).astype(np.int32), rng.integers(0, 100, int(R)).astype(np.int32))
             for R in rng.integers(0, 3000, 63)]
    got = run_multi(ctx, torch, variant, fc, fm, rows, packed)
    check_chain(got, chain_ref(oracle_c, fc, fm, rows, packed), "node full")
    assert sorted(got[0][0][0].tolist()) == [-1] * 5 + [0, 1, 2, 3]
    full = np.concatenate([np.zeros(D, np.int32), np.full(D, MEM_MAX - 1, np.int32), np.zeros(D, np.int32)])
    for g in got[0][1:]:
        assert (g[0] == -1).all() and not g[1].any() and np.array_equal(g[2], full)


# ---- 5. sizes ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("wname,variant", [("cfg3", AUTO), ("cfg4", AUTO)])
@pytest.mark.parametrize("packed", [False, True])
def test_multi_rounds_1mi(wname, variant, packed, ctx, egpu, oracle_c):
    import torch
    w = egpu.synth.workload(wname)
    fc, fm = np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32)
    rows = []
    for seed, R in ((5, 4099), (6, 1 << 20), (7, 20_011)):
        rc, rm = egpu.synth.requests(3, seed, R)
        rows.append((np.minimum(rc, 5).astype(np.int32), np.minimum(rm, 2048).astype(np.int32)))
    check_chain(run_multi(ctx, torch, variant, fc, fm, rows, packed), chain_ref(oracle_c, fc, fm, rows, packed), f"{wname}")


# ---- 6. sticky oversubscription flags -----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT], ids=lambda v: VNAME[v])
@pytest.mark.parametrize("packed", [False, True])
def test_multi_rounds_keep_oversubscription_flags(variant, packed, ctx, oracle_c):
    import torch
    D = 8
    fc, fm = np.full(D, 50, np.int32), np.full(D, 4096, np.int32)
    ctx.set_variant(variant)
    ctx.set_table(fc, fm)
    ctx.bestfit(np.array([30, 30, 30, 30], np.int32), np.array([1, 1, 1, 1], np.int32), commit=True)
    fc1, fm1, ov1 = ctx.table()
    assert ov1.any()
    rng = np.random.default_rng(6)
    rows = [(rng.integers(0, 12, R).astype(np.int32), rng.integers(0, 300, R).astype(np.int32)) for R in (5001, 0, 20_001)]
    got = run_multi(ctx, torch, variant, fc1, fm1, rows, packed, set_table=False)
    check_chain(got, chain_ref(oracle_c, fc1, fm1, rows, packed, ov1), "sticky flags")


# ---- 7. asynchrony, stream order, graph capture ---------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True])
def test_multi_rounds_asynchronous_and_stream_ordered(packed, ctx, egpu, oracle_c):
    """behind a sleeping kernel the call returns while the stream is still busy; a multi-batch snapshot
    enqueued right after it on the same stream scores against the table the last batch committed"""
    import torch
    w = egpu.synth.workload("cfg3")
    fc, fm = np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32)
    D = fc.size
    rows = []
    for seed, R in ((9, 100_001), (10, 0), (11, 50_001)):
        rc, rm = egpu.synth.requests(3, seed, R)
        rows.append((np.minimum(rc, 5).astype(np.int32), np.minimum(rm, 2048).astype(np.int32)))
    exp = chain_ref(oracle_c, fc, fm, rows, packed)
    call = Call(torch, rows, D, packed)
    ctx.set_table(fc, fm)
    assert multi(ctx, call) == 0  # warm-up: scratch and occupancy
    torch.cuda.synchronize()
    ctx.set_table(fc, fm)
    call.reset()
    qc, qm = egpu.synth.requests(3, 12, 10_001)
    d_qc, d_qm = km._dev(torch, qc), km._dev(torch, qm)
    q_idx = torch.full((qc.size + 4,), -9, dtype=torch.int32, device="cuda")
    q_delta = torch.zeros(2 * D, dtype=torch.int64, device="cuda")
    q_tab = torch.zeros(3 * D, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)
    assert multi(ctx, call) == 0
    busy = not torch.cuda.current_stream().query()
    ctx.bestfit_batches_dev([(d_qc.data_ptr(), d_qm.data_ptr(), qc.size, q_idx.data_ptr(), q_delta.data_ptr(), q_tab.data_ptr())],
                            torch.cuda.current_stream().cuda_stream)
    assert busy, "the call waited for its stream"
    torch.cuda.synchronize()
    check_chain((call.got(), ctx.table()), exp, "asynchronous")
    s_idx, s_dc, s_dm, s_tab = oracle_c.snapshot(exp[1][0], exp[1][1], qc, qm)
    assert np.array_equal(q_idx[:qc.size].cpu().numpy(), s_idx), "the next scan did not see the committed table"
    assert np.array_equal(q_delta.cpu().numpy(), np.concatenate([s_dc, s_dm])) and np.array_equal(q_tab.cpu().numpy(), s_tab)


@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(AUTO, 8), (LUT, 64), (SORTED, 33)])
@pytest.mark.parametrize("packed", [False, True])
def test_multi_rounds_graph_replay(variant, D, packed, ctx, oracle_c):
    """the call captured in a CUDA graph and replayed after each egpu_table_set: the eager results"""
    import torch
    tables = km.cell_tables(D)
    rows = cell_rows(D, "dups", (4099, 0, 40_003, 513))
    ctx.set_variant(variant)
    call = Call(torch, rows, D, packed)
    s = torch.cuda.Stream()
    ctx.set_table(*tables["dups"])
    with torch.cuda.stream(s):
        assert multi(ctx, call, stream=C.c_void_p(s.cuda_stream)) == 0  # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        assert multi(ctx, call, stream=C.c_void_p(s.cuda_stream)) == 0
    for tname, (fc, fm) in tables.items():
        exp = chain_ref(oracle_c, fc, fm, rows, packed)
        ctx.set_table(fc, fm)
        call.reset()
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        check_chain((call.got(), ctx.table()), exp, f"replay, table {tname}")
        check_chain(run_multi(ctx, torch, variant, fc, fm, rows, packed), exp, f"eager, table {tname}")


# ---- 8. one context, many calls ----------------------------------------------------------------------------------------
SEQ_OPS = ("set_table", "multi_rounds", "multi_rounds", "multi_rounds_packed", "single_rounds", "commit_snapshot", "replay",
           "multi_snapshot")


@pytest.mark.gpu
@pytest.mark.parametrize("seed", (3, 17))
def test_multi_rounds_context_sequence(seed, ctx, egpu, oracle_c):
    """a seeded sequence mixing this call with egpu_table_set, committing single calls, replay and multi-batch
    snapshots; the table is read back after every operation against the int64 model"""
    import torch
    rng = np.random.default_rng(seed)
    model = cs.Model()
    D = int(rng.choice(D_BUCKETS))
    fc, fm = cs.random_table(rng, D)
    ctx.set_variant(int(rng.choice([AUTO, SORTED, LUT])))
    ctx.set_table(fc, fm)
    model.set_table(fc, fm)
    for step in range(30):
        op = SEQ_OPS[int(rng.integers(0, len(SEQ_OPS)))] if step else "multi_rounds"
        mfc, mfm = model.table32()
        if op == "set_table":
            D = int(rng.choice(D_BUCKETS))
            fc, fm = cs.random_table(rng, D)
            ctx.set_variant(int(rng.choice([AUTO, SORTED, LUT])))
            ctx.set_table(fc, fm)
            model.set_table(fc, fm)
        elif op in ("multi_rounds", "multi_rounds_packed"):
            packed = op.endswith("packed")
            rows = [cs.requests_for(rng, mfc, mfm, int(rng.choice(cs.ROWS))) for _ in range(int(rng.integers(1, 6)))]
            exp = chain_ref(oracle_c, mfc, mfm, rows, packed, model.ov.astype(np.int32))
            call = Call(torch, rows, D, packed)
            assert multi(ctx, call) == 0
            torch.cuda.synchronize()
            for k, (g, e) in enumerate(zip(call.got(), exp[0])):
                assert all(np.array_equal(x, y) for x, y in zip(g, e)), f"step {step}, {op}, batch {k}"
            model.install(exp[1][0], exp[1][1])
        elif op == "single_rounds":
            rc, rm = cs.requests_for(rng, mfc, mfm, int(rng.choice(cs.ROWS)))
            c, m = dr.rows_dev(torch, rc, rm, False)
            o = dr.Out(torch, len(rc), D, False)
            assert dr.call_dev(ctx, torch, c, m, o) == 0
            torch.cuda.synchronize()
            e = dr.ref(oracle_c, mfc, mfm, rc, rm)
            assert np.array_equal(o.got()[0], e[0]), f"step {step}, {op}"
            model.install(e[3][0], e[3][1])
        elif op == "commit_snapshot":
            rc, rm = cs.requests_for(rng, mfc, mfm, int(rng.choice(cs.ROWS)))
            idx, _, _ = ctx.bestfit(rc, rm, commit=True)
            s_idx, _, _, s_tab = oracle_c.snapshot(mfc, mfm, rc, rm)
            assert np.array_equal(idx, s_idx), f"step {step}, {op}"
            model.commit_snapshot(s_tab)
        elif op == "replay":
            kind, a, b = egpu.synth.churn_events(int(rng.integers(0, 1000)), int(rng.choice([1, 257, 4097])))
            got = ctx.replay(kind, a, b)
            exp_idx, efc, efm = oracle_c.replay(mfc, mfm, kind, a, b)
            assert np.array_equal(got, exp_idx), f"step {step}, {op}"
            model.install(efc, efm)
        else:  # multi_snapshot: scores, never commits
            rows = [cs.requests_for(rng, mfc, mfm, int(rng.choice(cs.ROWS))) for _ in range(3)]
            devs = [(km._dev(torch, rc), km._dev(torch, rm)) for rc, rm in rows]
            outs = [dr.Out(torch, len(rc), D, False) for rc, _ in rows]
            ctx.bestfit_batches_dev([(c.data_ptr(), m.data_ptr(), o.R) + o.ptrs() for (c, m), o in zip(devs, outs)],
                                    torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            for (rc, rm), o in zip(rows, outs):
                assert np.array_equal(o.got()[0], oracle_c.snapshot(mfc, mfm, rc, rm)[0]), f"step {step}, {op}"
        g_fc, g_fm, g_ov = ctx.table()
        assert np.array_equal(g_fc, model.fc) and np.array_equal(g_fm, model.fm) and np.array_equal(g_ov, model.ov), \
            f"step {step}: the table after {op}"


# ---- 9. refusals ---------------------------------------------------------------------------------------------------------
REFUSED_FLAGS = dr.REFUSED_FLAGS + [F_COMMIT, F_PREFIX, F_PREFIX | F_COMMIT, F_ROUNDS, F_APPLY, F_PACKED | F_ROUNDS,
                                    F_PACKED | F_PREFIX | F_COMMIT | F_ROUNDS, F_INPUTS_READY | F_COMMIT]


@pytest.mark.gpu
def test_multi_rounds_refusals(ctx):
    import torch
    from elastic_gpu_agent_b200 import _lib as L
    D = 8
    fc, fm = km.cell_tables(D)["dups"]
    rows = cell_rows(D, "dups", (513, 4099))
    lib, h = ctx._lib, ctx.handle
    ctx.set_table(fc, fm)
    before = ctx.table()
    c32, c8 = Call(torch, rows, D, False), Call(torch, rows, D, True)
    s = pm._s(torch)
    torch.cuda.synchronize()
    n0 = ctx.launch_count

    def raw(batches, flags, entry=lib.egpu_bestfit_batches_dev):
        arr = (L.Batch * max(1, len(batches)))(*[L.Batch(*b) for b in batches])
        if entry is lib.egpu_bestfit_batches_shard_dev:
            return entry(h, arr, len(batches), flags, 0, s)
        return entry(h, arr, len(batches), flags, s)

    def tup(call, k, **kw):
        b = call.arr[k]
        t = dict(c=b.d_req_core, m=b.d_req_mem, R=b.R, i=b.d_out_idx, dl=b.d_delta, to=b.d_table_out)
        t.update(kw)
        return (t["c"], t["m"], t["R"], t["i"], t["dl"], t["to"])

    for f in REFUSED_FLAGS:
        assert raw([tup(c32, 0), tup(c32, 1)], f) == ERR_INVALID, f
        assert raw([tup(c8, 0), tup(c8, 1)], f) == ERR_INVALID, f
    for call, P in ((c32, 0), (c8, F_PACKED)):
        fmt = "packed" if P else "int32"
        b0, b1 = tup(call, 0), tup(call, 1)
        refused = {
            "K = 0": ([], DR | P),
            "K = 65": ([tup(call, 0, R=1, i=b0[3] + 16 * k, dl=None, to=None) for k in range(65)], DR | P),
            "R >= 2^31": ([b0, tup(call, 1, R=1 << 31)], DR | P),
            "NULL req_core": ([b0, tup(call, 1, c=None)], DR | P),
            "NULL indices": ([b0, tup(call, 1, i=None)], DR | P),
            "misaligned req_core": ([b0, tup(call, 1, c=b1[0] + 4)], DR | P),
            "misaligned indices": ([b0, tup(call, 1, i=b1[3] + (1 if P else 4))], DR | P),
            "overlapping indices": ([b0, tup(call, 1, i=b0[3] + 16 * (1 if P else 4))], DR | P),
            "overlapping demand sums": ([b0, tup(call, 1, dl=b0[4] + 8)], DR | P),
            "overlapping table'": ([b0, tup(call, 1, to=b0[5])], DR | P),
            "table' over demand sums": ([b0, tup(call, 1, to=b0[4])], DR | P),
        }
        if P:
            refused["req_mem with EGPU_F_PACKED"] = ([b0, tup(call, 1, m=c32.arr[1].d_req_mem)], DR | P)
        else:
            refused["NULL req_mem without EGPU_F_PACKED"] = ([b0, tup(call, 1, m=None)], DR)
            refused["misaligned req_mem"] = ([b0, tup(call, 1, m=b1[1] + 4)], DR)
        for what, (batches, flags) in refused.items():
            assert raw(batches, flags) == ERR_INVALID, f"{fmt}: {what}"
        # the sharded multi-batch entry point keeps refusing the flags
        assert raw([b0, b1], DR | P, lib.egpu_bestfit_batches_shard_dev) == ERR_INVALID, f"{fmt}: sharded"
    ctx.set_variant(GRID)
    assert multi(ctx, c32) == ERR_STATE and multi(ctx, c8) == ERR_STATE
    ctx.set_variant(AUTO)
    torch.cuda.synchronize()
    assert ctx.launch_count == n0, "a refused call launched"
    for call in (c32, c8):
        for o in call.outs:
            assert (o.idx.cpu().numpy() == -9).all() and (o.delta.cpu().numpy() == -1).all() and (o.tab.cpu().numpy() == -7).all()
    assert all(np.array_equal(a, b) for a, b in zip(ctx.table(), before))


@pytest.mark.gpu
def test_multi_rounds_without_table(egpu):
    import torch
    with egpu.BestFitAllocator(0) as a:
        call = Call(torch, [(np.ones(4, np.int32), np.ones(4, np.int32))], 1, False)
        assert multi(a, call) == ERR_NO_TABLE
        assert a.launch_count == 0
