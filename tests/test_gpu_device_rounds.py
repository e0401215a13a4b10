"""Rounds to the fixed point in one launch: egpu_bestfit_batch[_dev] with EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT |
EGPU_F_ROUNDS | EGPU_F_DEVICE_ROUNDS [| EGPU_F_PACKED].

The call runs the rounds of egpu_bestfit_batch_rounds (no round limit) in one persistent cooperative launch
(rounds_sorted_kernel / rounds_lut_kernel).  Every GPU case compares exactly with the C rounds oracle, in both
row formats, and the agreement cases also with egpu_bestfit_batch_rounds_dev and packed EGPU_F_ROUNDS:

  1. the cell matrix: both scans at every D bucket under AUTO, SORTED and LUT, ragged row counts, domain-edge
     rows and words, tables with zeros and duplicates; d_table_out, the installed table, guard bytes, and
     exactly one launch per call;
  2. agreement with the synchronous rounds of both formats;
  3. 1, 2 and many rounds: the cfg1 known answer, a D = 64 table of dozens of rounds, 1 Mi rows;
  4. sticky oversubscription flags;
  5. the host entry point, pageable and pinned, demand sums NULL and not;
  6. asynchrony, stream order and CUDA-graph capture;
  7. refusals: nothing launched, nothing written.
Every GPU test ends with a host-form call that would report a grid-barrier timeout of any launch on its context.
"""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_kernel_matrix as km  # noqa: E402  (cell tables, pack / unpack, int32 device arrays)
import test_gpu_packed_multi as pm  # noqa: E402  (cells, Out, guard bytes, stream handle)

MEM_MAX = (1 << 18) - 1
ERR_INVALID, ERR_NO_TABLE, ERR_STATE = -1, -5, -6
AUTO, GRID, SORTED, LUT = 0, 1, 2, 3
F_COMMIT, F_INPUTS_READY, F_PREFIX, F_APPLY, F_PACKED, F_ROUNDS, F_DEVICE_ROUNDS = 1, 2, 4, 8, 16, 32, 128
DR = F_PREFIX | F_COMMIT | F_ROUNDS | F_DEVICE_ROUNDS
GUARD = pm.GUARD


def test_device_rounds_flag_value():
    import elastic_gpu_agent_b200._lib as L
    src = open(os.path.join(pm.ROOT, "include", "egpu_alloc.h")).read()
    assert "#define EGPU_F_DEVICE_ROUNDS 128" in src and L.F_DEVICE_ROUNDS == F_DEVICE_ROUNDS
    values = [int(v) for v in re.findall(r"^#define EGPU_F_\w+\s+(\d+)", src, re.M)]
    assert 64 not in values and len(values) == len(set(values))  # bit 64 stays unassigned


@pytest.fixture()
def ctx(egpu):
    """an allocator context; on teardown a host-form call reports any grid-barrier timeout of its launches"""
    a = egpu.BestFitAllocator(0)
    yield a
    a.set_variant(AUTO)
    a.set_table([100], [MEM_MAX])
    one = np.array([1], np.int32)
    idx = np.empty(1, np.int32)
    rc = a._lib.egpu_bestfit_batch(a.handle, C.c_void_p(one.ctypes.data), C.c_void_p(one.ctypes.data), 1,
                                   C.c_void_p(idx.ctypes.data), None, None, DR)
    assert rc == 0, a._lib.egpu_last_error(a.handle).decode()
    a.close()


# ---- references and calls --------------------------------------------------------------------------------
def ref(oracle_c, fc, fm, rc, rm, ov=None):
    """(idx, delta, table' of the last round, installed (fc, fm, oversub), rounds) of the C rounds oracle"""
    o_idx, o_dc, o_dm, o_fc, o_fm, o_rounds, o_left = oracle_c.rounds(fc, fm, rc, rm)
    assert o_left == 0 and not (o_idx == -2).any()
    D = len(fc)
    tab = np.concatenate([o_fc, o_fm, np.zeros(D, np.int32)]).astype(np.int32)
    ov = np.zeros(D, np.int32) if ov is None else ov
    return o_idx, np.concatenate([o_dc, o_dm]), tab, (o_fc, o_fm, ov), o_rounds


class Out:
    """outputs of one call, sentinel-filled; int32 or int8 indices with guard elements after them"""

    def __init__(self, torch, R, D, packed):
        self.R, self.packed = R, packed
        self.idx = torch.full((R + GUARD,), -9, dtype=torch.int8 if packed else torch.int32, device="cuda")
        self.delta = torch.full((2 * D,), -1, dtype=torch.int64, device="cuda")
        self.tab = torch.full((3 * D,), -7, dtype=torch.int32, device="cuda")

    def ptrs(self):
        return self.idx.data_ptr(), self.delta.data_ptr(), self.tab.data_ptr()

    def got(self):
        idx = self.idx.cpu().numpy().astype(np.int32)
        assert (idx[self.R:] == -9).all(), "guard elements"
        return idx[:self.R], self.delta.cpu().numpy(), self.tab.cpu().numpy()


def rows_dev(torch, rc, rm, packed):
    """(d_req_core, d_req_mem) device arrays: int32 pair, or the packed words and None"""
    if packed:
        return pm.words_dev(torch, km.pack(rc, rm)), None
    return km._dev(torch, np.asarray(rc, np.int32)), km._dev(torch, np.asarray(rm, np.int32))


def call_dev(alloc, torch, c, m, o, flags=0, stream=None):
    i, dl, t = o.ptrs()
    s = pm._s(torch) if stream is None else stream
    return alloc._lib.egpu_bestfit_batch_dev(alloc.handle, C.c_void_p(c.data_ptr()), C.c_void_p(m.data_ptr()) if m is not None else None,
                                             o.R, C.c_void_p(i), C.c_void_p(dl), C.c_void_p(t),
                                             DR | (F_PACKED if o.packed else 0) | flags, s)


def device_rounds(alloc, torch, variant, fc, fm, rc, rm, packed, set_table=True):
    """one _dev call: (idx, delta, table', installed table), checking it added exactly one launch"""
    D = len(fc)
    alloc.set_variant(variant)
    if set_table:
        alloc.set_table(fc, fm)
    c, m = rows_dev(torch, rc, rm, packed)
    o = Out(torch, len(rc), D, packed)
    torch.cuda.synchronize()
    n0 = alloc.launch_count
    assert call_dev(alloc, torch, c, m, o) == 0, alloc._lib.egpu_last_error(alloc.handle).decode()
    assert alloc.launch_count - n0 == 1, "one launch per call"
    torch.cuda.synchronize()
    return o.got() + (alloc.table(),)


def check(got, exp, where):
    idx, delta, tab, inst = got
    assert np.array_equal(idx, exp[0]), f"{where}: indices"
    assert np.array_equal(delta, exp[1]), f"{where}: demand sums"
    assert np.array_equal(tab, exp[2]), f"{where}: table'"
    assert all(np.array_equal(a, b) for a, b in zip(inst, exp[3])), f"{where}: installed table"


def packed_requests(rc, rm):
    """the requests packed words stand for (what the packed call is compared against)"""
    return km.unpack(km.pack(rc, rm))


# ---- 1. the cell matrix ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", pm.CELLS, ids=[f"{['auto', 'grid', 'sorted', 'lut'][v]}-D{D}" for v, D in pm.CELLS])
def test_device_rounds_cell(variant, D, ctx, oracle_c):
    import torch
    for tname in km.cell_tables(D):
        for R in km.ROW_COUNTS:
            fc, fm, rc, rm = km.cell_case(D, tname, R)
            where = f"variant {variant}, D = {D}, table {tname}, R = {R}"
            check(device_rounds(ctx, torch, variant, fc, fm, rc, rm, False), ref(oracle_c, fc, fm, rc, rm), where + ", int32")
            prc, prm = packed_requests(rc, rm)
            check(device_rounds(ctx, torch, variant, fc, fm, rc, rm, True), ref(oracle_c, fc, fm, prc, prm), where + ", packed")


@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", pm.CELLS, ids=[f"{['auto', 'grid', 'sorted', 'lut'][v]}-D{D}" for v, D in pm.CELLS])
def test_device_rounds_domain_edge_words(variant, D, ctx, oracle_c):
    """words the int32 arrays cannot express: core 101..127, anything >= 2^25, the all-ones word"""
    import torch
    fc, fm, words = pm.cell_words(D, "spread", km.ROW_COUNTS[-1])
    prc, prm = km.unpack(words)
    c = pm.words_dev(torch, words)
    o = Out(torch, words.size, D, True)
    ctx.set_variant(variant)
    ctx.set_table(fc, fm)
    assert call_dev(ctx, torch, c, None, o) == 0
    check(o.got() + (ctx.table(),), ref(oracle_c, fc, fm, prc, prm), f"variant {variant}, D = {D}")


# ---- 2. agreement with the synchronous rounds ------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(SORTED, 8), (SORTED, 33), (LUT, 17), (LUT, 64), (AUTO, 64)])
def test_device_rounds_match_sync_rounds(variant, D, ctx):
    import torch
    fc, fm, rc, rm = km.cell_case(D, "dups", 40_003)
    # int32: egpu_bestfit_batch_rounds_dev, no round limit
    ctx.set_variant(variant)
    ctx.set_table(fc, fm)
    c, m = rows_dev(torch, rc, rm, False)
    idx = torch.full((len(rc) + 4,), -9, dtype=torch.int32, device="cuda")
    delta, rounds, left = ctx.bestfit_rounds_dev(c.data_ptr(), m.data_ptr(), len(rc), idx.data_ptr(),
                                                 stream=torch.cuda.current_stream().cuda_stream)
    assert left == 0 and rounds >= 2
    sync = (idx[:len(rc)].cpu().numpy(), delta, ctx.table())
    got = device_rounds(ctx, torch, variant, fc, fm, rc, rm, False)
    assert np.array_equal(got[0], sync[0]) and np.array_equal(got[1], sync[1])
    assert all(np.array_equal(a, b) for a, b in zip(got[3], sync[2]))
    # packed: EGPU_F_ROUNDS (the synchronous packed rounds)
    ctx.set_table(fc, fm)
    words = km.pack(rc, rm)
    w = pm.words_dev(torch, words)
    o = pm.Out(torch, words.size, D)
    i, dl, t = o.ptrs()
    assert ctx._lib.egpu_bestfit_batch_dev(ctx.handle, C.c_void_p(w.data_ptr()), None, o.R, C.c_void_p(i), C.c_void_p(dl),
                                           C.c_void_p(t), F_PACKED | F_PREFIX | F_COMMIT | F_ROUNDS, pm._s(torch)) == 0
    sync_tab = ctx.table()
    got = device_rounds(ctx, torch, variant, fc, fm, rc, rm, True)
    assert np.array_equal(got[0], o.idx[:o.R].cpu().numpy().astype(np.int32))
    assert np.array_equal(got[1], o.delta.cpu().numpy()) and np.array_equal(got[2], o.tab.cpu().numpy())
    assert all(np.array_equal(a, b) for a, b in zip(got[3], sync_tab))


# ---- 3. one, two and many rounds ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
@pytest.mark.parametrize("packed", [False, True])
def test_device_rounds_cfg1_known_answer(variant, packed, ctx, egpu, oracle_c):
    """five (25, 1024) requests on 8 full devices: four fit device 0, the fifth goes to device 1 in round 2"""
    import torch
    w = egpu.synth.workload("cfg1")
    fc, fm = np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32)
    rc, rm = np.full(5, 25, np.int32), np.full(5, 1024, np.int32)
    exp = ref(oracle_c, fc, fm, rc, rm)
    assert exp[0].tolist() == [0, 0, 0, 0, 1] and exp[4] == 2
    check(device_rounds(ctx, torch, variant, fc, fm, rc, rm, packed), exp, "cfg1")


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [AUTO, SORTED, LUT])
@pytest.mark.parametrize("packed", [False, True])
def test_device_rounds_one_round(variant, packed, ctx, oracle_c):
    """requests that all fit the device they choose: one round, nothing deferred"""
    import torch
    fc, fm = np.full(8, 100, np.int32), np.full(8, MEM_MAX, np.int32)
    rc, rm = np.zeros(1001, np.int32), np.ones(1001, np.int32)
    exp = ref(oracle_c, fc, fm, rc, rm)
    assert exp[4] == 1
    check(device_rounds(ctx, torch, variant, fc, fm, rc, rm, packed), exp, "one round")


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
@pytest.mark.parametrize("packed", [False, True])
def test_device_rounds_many_rounds_d64(variant, packed, ctx, egpu, oracle_c):
    """the cfg4 table (D = 64) and small requests: dozens of rounds"""
    import torch
    w = egpu.synth.workload("cfg4")
    fc, fm = np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32)
    rc, rm = egpu.synth.requests(3, 5, 100_003)
    rc, rm = np.minimum(rc, 5).astype(np.int32), np.minimum(rm, 2048).astype(np.int32)
    exp = ref(oracle_c, fc, fm, rc, rm)
    assert exp[4] >= 24, exp[4]
    check(device_rounds(ctx, torch, variant, fc, fm, rc, rm, packed), exp, f"{exp[4]} rounds")


@pytest.mark.gpu
@pytest.mark.parametrize("wname,variant", [("cfg3", AUTO), ("cfg4", LUT), ("cfg4", SORTED)])
@pytest.mark.parametrize("packed", [False, True])
def test_device_rounds_1mi(wname, variant, packed, ctx, egpu, oracle_c):
    import torch
    w = egpu.synth.workload(wname)
    fc, fm = np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32)
    rc, rm = egpu.synth.requests(3, 5, 1 << 20)
    rc, rm = np.minimum(rc, 5).astype(np.int32), np.minimum(rm, 2048).astype(np.int32)
    check(device_rounds(ctx, torch, variant, fc, fm, rc, rm, packed), ref(oracle_c, fc, fm, rc, rm), f"{wname} 1 Mi")


# ---- 4. sticky oversubscription flags ----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
@pytest.mark.parametrize("packed", [False, True])
def test_device_rounds_keep_oversubscription_flags(variant, packed, ctx, oracle_c):
    """a committing snapshot that oversubscribes devices 0 and 1 sets their flags; the rounds keep them"""
    import torch
    D = 8
    fc, fm = np.full(D, 50, np.int32), np.full(D, 4096, np.int32)
    ctx.set_variant(variant)
    ctx.set_table(fc, fm)
    ctx.bestfit(np.array([30, 30, 30, 30], np.int32), np.array([1, 1, 1, 1], np.int32), commit=True)  # all four on one device
    fc1, fm1, ov1 = ctx.table()
    assert ov1.any()
    rng = np.random.default_rng(5)
    rc, rm = rng.integers(0, 12, 20_001).astype(np.int32), rng.integers(0, 300, 20_001).astype(np.int32)
    exp = ref(oracle_c, fc1, fm1, rc, rm, ov1)
    got = device_rounds(ctx, torch, variant, fc1, fm1, rc, rm, packed, set_table=False)
    check(got, exp, "sticky flags")


# ---- 5. the host entry point ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(AUTO, 8), (LUT, 64), (SORTED, 33)])
def test_device_rounds_host_form(variant, D, ctx, oracle_c):
    fc, fm, rc, rm = km.cell_case(D, "dups", 40_003)
    ctx.set_variant(variant)
    lib, h = ctx._lib, ctx.handle
    for pinned in (False, True):
        # int32: bestfit_rounds(device=True)
        ctx.set_table(fc, fm)
        if pinned:
            pc, pmm = ctx.pinned_array(rc.size, np.int32), ctx.pinned_array(rc.size, np.int32)
            pc[:], pmm[:] = rc, rm
        else:
            pc, pmm = rc, rm
        idx, dc, dm, rounds, left = ctx.bestfit_rounds(pc, pmm, device=True)
        exp = ref(oracle_c, fc, fm, rc, rm)
        assert rounds is None and left == 0
        assert np.array_equal(idx, exp[0]) and np.array_equal(np.concatenate([dc, dm]), exp[1]), f"int32, pinned {pinned}"
        assert all(np.array_equal(a, b) for a, b in zip(ctx.table(), exp[3]))
        # packed: bestfit_packed_prefix(rounds=True, device=True)
        words = km.pack(rc, rm)
        ctx.set_table(fc, fm)
        if pinned:
            pw = ctx.pinned_array(words.size, np.uint32)
            pw[:] = words
        else:
            pw = words
        idx8, dc8, dm8 = ctx.bestfit_packed_prefix(pw, rounds=True, device=True)
        exp8 = ref(oracle_c, fc, fm, *km.unpack(words))
        assert np.array_equal(idx8.astype(np.int32), exp8[0]) and np.array_equal(np.concatenate([dc8, dm8]), exp8[1])
        assert all(np.array_equal(a, b) for a, b in zip(ctx.table(), exp8[3]))
        # demand sums NULL
        ctx.set_table(fc, fm)
        out = np.full(words.size, -9, np.int8)
        assert lib.egpu_bestfit_batch(h, C.c_void_p(pw.ctypes.data), None, words.size, C.c_void_p(out.ctypes.data), None, None,
                                      DR | F_PACKED) == 0
        assert np.array_equal(out.astype(np.int32), exp8[0])
        if pinned:
            for arr in (pc, pmm, pw):
                ctx.host_free(arr.ctypes.data)
    # R = 0: zero sums, nothing changes
    ctx.set_table(fc, fm)
    dc, dm = np.full(D, -1, np.int64), np.full(D, -1, np.int64)
    assert lib.egpu_bestfit_batch(h, None, None, 0, None, C.c_void_p(dc.ctypes.data), C.c_void_p(dm.ctypes.data), DR | F_PACKED) == 0
    assert not dc.any() and not dm.any()
    assert all(np.array_equal(a, b) for a, b in zip(ctx.table(), (fc, fm, np.zeros(D, np.int32))))


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True])
def test_device_rounds_empty_batch(packed, ctx):
    """R = 0 on the _dev form: zero sums, table' = the table, one launch"""
    import torch
    fc, fm, _, _ = km.cell_case(17, "spread", 0)
    got = device_rounds(ctx, torch, LUT, fc, fm, np.zeros(0, np.int32), np.zeros(0, np.int32), packed)
    assert got[0].size == 0 and not got[1].any()
    assert np.array_equal(got[2], np.concatenate([fc, fm, np.zeros(17, np.int32)]))


# ---- 6. asynchrony, stream order, graph capture -------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True])
def test_device_rounds_asynchronous_and_stream_ordered(packed, ctx, egpu, oracle_c):
    """behind a sleeping kernel the call returns while the stream is still busy; a snapshot scan enqueued right
    after it on the same stream scores against the committed table"""
    import torch
    w = egpu.synth.workload("cfg3")
    fc, fm = np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32)
    D = fc.size
    rc, rm = egpu.synth.requests(3, 9, 200_001)
    rc, rm = np.minimum(rc, 5).astype(np.int32), np.minimum(rm, 2048).astype(np.int32)
    exp = ref(oracle_c, fc, fm, rc, rm)
    c, m = rows_dev(torch, rc, rm, packed)
    o = Out(torch, len(rc), D, packed)
    ctx.set_table(fc, fm)
    assert call_dev(ctx, torch, c, m, o) == 0  # warm-up: scratch and occupancy outside the timed call
    torch.cuda.synchronize()
    ctx.set_table(fc, fm)
    o.idx.fill_(-9)
    o.delta.fill_(-1)
    o.tab.fill_(-7)
    qc, qm = egpu.synth.requests(3, 10, 10_001)
    d_qc, d_qm = km._dev(torch, qc), km._dev(torch, qm)
    q_idx = torch.full((qc.size + 4,), -9, dtype=torch.int32, device="cuda")
    q_delta = torch.zeros(2 * D, dtype=torch.int64, device="cuda")
    q_tab = torch.zeros(3 * D, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)  # ~0.1 s of spinning on the current stream
    assert call_dev(ctx, torch, c, m, o) == 0
    busy = not torch.cuda.current_stream().query()
    ctx.bestfit_dev(d_qc.data_ptr(), d_qm.data_ptr(), qc.size, q_idx.data_ptr(), q_delta.data_ptr(), q_tab.data_ptr(),
                    stream=torch.cuda.current_stream().cuda_stream)
    assert busy, "the call waited for its stream"
    torch.cuda.synchronize()
    check(o.got() + (ctx.table(),), exp, "asynchronous")
    s_idx, s_dc, s_dm, s_tab = oracle_c.snapshot(exp[3][0], exp[3][1], qc, qm)
    assert np.array_equal(q_idx[:qc.size].cpu().numpy(), s_idx), "the next scan did not see the committed table"
    assert np.array_equal(q_delta.cpu().numpy(), np.concatenate([s_dc, s_dm]))


@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(AUTO, 8), (LUT, 64), (SORTED, 64)])
@pytest.mark.parametrize("packed", [False, True])
def test_device_rounds_graph_replay(variant, D, packed, ctx, oracle_c):
    """the _dev call captured in a CUDA graph and replayed after each egpu_table_set: the eager results"""
    import torch
    tables = km.cell_tables(D)
    _, _, rc, rm = km.cell_case(D, "dups", 40_003)
    ctx.set_variant(variant)
    c, m = rows_dev(torch, rc, rm, packed)
    o = Out(torch, len(rc), D, packed)
    s = torch.cuda.Stream()
    fc0, fm0 = tables["dups"]
    ctx.set_table(fc0, fm0)
    with torch.cuda.stream(s):
        assert call_dev(ctx, torch, c, m, o) == 0  # warm-up: occupancy query and scratch outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        assert call_dev(ctx, torch, c, m, o) == 0
    for tname, (fc, fm) in tables.items():
        prc, prm = packed_requests(rc, rm) if packed else (rc, rm)
        exp = ref(oracle_c, fc, fm, prc, prm)
        ctx.set_table(fc, fm)
        o.idx.fill_(-9)
        o.delta.fill_(-1)
        o.tab.fill_(-7)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        check(o.got() + (ctx.table(),), exp, f"replay, table {tname}")
        eager = device_rounds(ctx, torch, variant, fc, fm, rc, rm, packed)
        check(eager, exp, f"eager, table {tname}")


# ---- 7. refusals -----------------------------------------------------------------------------------------------
REFUSED_FLAGS = [
    F_DEVICE_ROUNDS, F_ROUNDS | F_DEVICE_ROUNDS, F_PREFIX | F_DEVICE_ROUNDS, F_PREFIX | F_COMMIT | F_DEVICE_ROUNDS,
    F_PREFIX | F_ROUNDS | F_DEVICE_ROUNDS, F_COMMIT | F_ROUNDS | F_DEVICE_ROUNDS, DR | 64, DR | F_APPLY, DR | 256,
    DR | F_PACKED | 64, DR | F_PACKED | F_APPLY, F_COMMIT | F_DEVICE_ROUNDS, F_PACKED | F_DEVICE_ROUNDS,
    F_PREFIX | F_COMMIT | F_ROUNDS,  # int32 rounds exist only with EGPU_F_DEVICE_ROUNDS
]


@pytest.mark.gpu
def test_device_rounds_refusals(ctx):
    import torch
    D = 8
    fc, fm, rc, rm = km.cell_case(D, "dups", 513)
    lib, h = ctx._lib, ctx.handle
    ctx.set_table(fc, fm)
    before = ctx.table()
    c, m = rows_dev(torch, rc, rm, False)
    w, _ = rows_dev(torch, rc, rm, True)
    o32, o8 = Out(torch, len(rc), D, False), Out(torch, len(rc), D, True)
    n0 = ctx.launch_count

    def dev(core, mem, R, o, flags):
        i, dl, t = o.ptrs()
        return lib.egpu_bestfit_batch_dev(h, C.c_void_p(core) if core else None, C.c_void_p(mem) if mem else None, R,
                                          C.c_void_p(i) if i else None, C.c_void_p(dl), C.c_void_p(t), flags, pm._s(torch))

    for f in REFUSED_FLAGS:
        assert dev(c.data_ptr(), m.data_ptr(), o32.R, o32, f) == ERR_INVALID, f
        if f & F_PACKED:
            assert dev(w.data_ptr(), 0, o8.R, o8, f) == ERR_INVALID, f
        hi = np.empty(len(rc), np.int32)
        assert lib.egpu_bestfit_batch(h, C.c_void_p(rc.ctypes.data), C.c_void_p(rm.ctypes.data), len(rc),
                                      C.c_void_p(hi.ctypes.data), None, None, f) == ERR_INVALID, f
    for core, mem, o, f, what in [
        (c.data_ptr(), m.data_ptr(), o32, DR | F_PACKED, "req_mem with EGPU_F_PACKED"),
        (c.data_ptr(), 0, o32, DR, "NULL req_mem without it"),
        (0, m.data_ptr(), o32, DR, "NULL req_core"),
        (c.data_ptr() + 4, m.data_ptr(), o32, DR, "misaligned req_core"),
        (c.data_ptr(), m.data_ptr() + 4, o32, DR, "misaligned req_mem"),
        (w.data_ptr() + 4, 0, o8, DR | F_PACKED, "misaligned words"),
        (0, 0, o8, DR | F_PACKED, "NULL words"),
    ]:
        assert dev(core, mem, o.R, o, f) == ERR_INVALID, what
    i8 = o8.idx.data_ptr()
    assert lib.egpu_bestfit_batch_dev(h, C.c_void_p(w.data_ptr()), None, o8.R, C.c_void_p(i8 + 1), None, None, DR | F_PACKED,
                                      pm._s(torch)) == ERR_INVALID, "misaligned indices"
    assert lib.egpu_bestfit_batch_dev(h, C.c_void_p(c.data_ptr()), C.c_void_p(m.data_ptr()), 1 << 31, C.c_void_p(o32.idx.data_ptr()),
                                      None, None, DR, pm._s(torch)) == ERR_INVALID, "R >= 2^31"
    assert lib.egpu_bestfit_batch(h, C.c_void_p(rc.ctypes.data), C.c_void_p(rm.ctypes.data), 1 << 31, C.c_void_p(rc.ctypes.data),
                                  None, None, DR) == ERR_INVALID, "host form, R >= 2^31"
    ctx.set_variant(GRID)
    assert dev(c.data_ptr(), m.data_ptr(), o32.R, o32, DR) == ERR_STATE
    assert dev(w.data_ptr(), 0, o8.R, o8, DR | F_PACKED) == ERR_STATE
    ctx.set_variant(AUTO)
    torch.cuda.synchronize()
    assert ctx.launch_count == n0, "a refused call launched"
    for o in (o32, o8):
        assert (o.idx.cpu().numpy() == -9).all() and (o.delta.cpu().numpy() == -1).all() and (o.tab.cpu().numpy() == -7).all()
    assert all(np.array_equal(a, b) for a, b in zip(ctx.table(), before))


@pytest.mark.gpu
def test_device_rounds_without_table(egpu):
    import torch
    with egpu.BestFitAllocator(0) as a:
        c, m = rows_dev(torch, np.ones(4, np.int32), np.ones(4, np.int32), False)
        o = Out(torch, 4, 1, False)
        assert call_dev(a, torch, c, m, o) == ERR_NO_TABLE
        one = np.ones(4, np.int32)
        assert a._lib.egpu_bestfit_batch(a.handle, C.c_void_p(one.ctypes.data), C.c_void_p(one.ctypes.data), 4,
                                         C.c_void_p(one.ctypes.data), None, None, DR) == ERR_NO_TABLE
        assert a.launch_count == 0
