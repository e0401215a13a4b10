"""The packed format over row shards: EGPU_F_PACKED on egpu_bestfit_batch_shard_dev, egpu_bestfit_batch_shard_lag_dev
and egpu_bestfit_batch_shard_prefix_dev.

d_req_core holds packed words (EGPU_PACK_REQUEST: core << 18 | mem; a word >= 2^25 is not a request), d_req_mem is
NULL and the indices are int8.  The sharded scans run kKernels<kScanSorted or kScanLut, kRowsPacked>[d_bucket(D)]
(csrc/egpu_alloc.cu), the round-robin packed twins of the single-batch scans with the push and lag epilogue; the sharded prefix-commit
runs the packed CONTIG scans, prefix_cut_packed_shard_kernel and prefix_apply_packed_kernel.  The exchange is the
int32 one.  Every case compares exactly with oracle/bestfit_np.py or the C oracle on the requests the words stand for
(not a request: (-1, -1)), and where it says so with the int32 call on the same requests:

  1. world 1, egpu_bestfit_batch_shard_dev: the cell matrix (both scans, every D bucket, AUTO / SORTED / LUT), ragged
     and empty batches, domain-edge words; a sequence longer than the exchange-slot ring with committing applies and
     one batch above 512 Ki rows;
  2. pipelined chains of packed and int32 sharded scans and packed multi-batch launches on one stream, longer than a
     launch group, with a committing apply that the next packed lookup scan must see;
  3. egpu_bestfit_batch_shard_lag_dev at lag 1, 2 and 16 over more steps than exchange slots, and the int32 call it
     still makes when d_req_mem is given;
  4. world 1, egpu_bestfit_batch_shard_prefix_dev: equal to the single-GPU packed prefix-commit and the oracle;
  5. world 2 (two processes on one GPU): snapshot steps with apply, the lag-2 form, rank-major prefix-commit, and
     worlds where one rank is packed and the other int32;
  6. gate, packed sharded scans and apply launches captured in a CUDA graph and replayed twice;
  7. argument checks: every refusal launches and writes nothing.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_kernel_matrix as km  # noqa: E402  (cell tables, pack / unpack, prefix_case)
import test_gpu_packed_multi as pm  # noqa: E402  (cell words, Out, words_dev, family)
import test_gpu_packed_prefix as pp  # noqa: E402  (cut cases, single-GPU packed prefix-commit)
import test_gpu_peer_exchange as pe  # noqa: E402  (rank-major prefix-commit cases)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEM_MAX = (1 << 18) - 1
ERR_INVALID, ERR_STATE = -1, -6
AUTO, GRID, SORTED, LUT = 0, 1, 2, 3
F_COMMIT, F_INPUTS_READY, F_PREFIX, F_PACKED = 1, 2, 4, 16
XCHG_SLOTS = 256
SHARD_ROWS = (0, 1, 3, 5, 511, 513, 4099)
CELLS = pm.CELLS


def test_packed_snap_twins():
    """the packed twins of the round-robin scans in the kernel table, and a cell for each of their families"""
    twins = pm.packed_twins("snap")
    assert twins == {"kScanSorted": "bestfit_sorted_packed_snap_kernel", "kScanLut": "bestfit_lut_packed_snap_kernel"}
    assert tuple(k.split("_")[1] for k in twins.values()) == pm.PACKED_FAMILIES
    assert {pm.family(v, D) for v, D in CELLS} == {"sorted", "lut"}


def test_wrappers_pass_null_req_mem(egpu):
    """the three packed wrappers never hand a d_req_mem to the library (for the lag call that is what selects packed)"""
    calls = []

    class Lib:
        def __getattr__(self, name):
            return lambda *a: calls.append((name, a)) or 0

    a = object.__new__(egpu.BestFitAllocator)
    a._lib, a._h = Lib(), C.c_void_p(1)
    a.bestfit_shard_packed_dev(16, 5, 32, 0, 7, inputs_ready=True)
    a.bestfit_shard_lag_packed_dev(16, 5, 32, 0, 7, 2)
    a.bestfit_shard_prefix_packed_dev(16, 5, 32, 0, 0, 7, commit=True)
    assert [n for n, _ in calls] == ["egpu_bestfit_batch_shard_dev", "egpu_bestfit_batch_shard_lag_dev",
                                     "egpu_bestfit_batch_shard_prefix_dev"]
    for name, args in calls:
        assert args[2] is None, name
    assert calls[0][1][6] == F_PACKED | F_INPUTS_READY
    assert calls[1][1][6] == F_PACKED
    assert calls[2][1][7] == F_PACKED | F_PREFIX | F_COMMIT
    a._lib = None
    a._h = None


# ---- helpers --------------------------------------------------------------------------------------------
def attach(alloc):
    alloc.peer_attach(0, 1, [alloc.peer_export()])


def stream(torch):
    return torch.cuda.current_stream().cuda_stream


class Out32:
    """the outputs of one int32 batch, sentinel-filled"""

    def __init__(self, torch, R, D):
        self.R = R
        self.idx = torch.full((R + 4,), -9, dtype=torch.int32, device="cuda")
        self.delta = torch.full((2 * D,), -1, dtype=torch.int64, device="cuda")
        self.tab = torch.full((3 * D,), -7, dtype=torch.int32, device="cuda")

    def ptrs(self):
        return self.idx.data_ptr(), self.delta.data_ptr(), self.tab.data_ptr()

    def check(self, exp, where):
        o_idx, o_dc, o_dm, o_tab = exp
        idx = self.idx.cpu().numpy()
        assert np.array_equal(idx[:self.R], o_idx) and (idx[self.R:] == -9).all(), f"{where}: indices"
        assert np.array_equal(self.delta.cpu().numpy(), np.concatenate([o_dc, o_dm])), f"{where}: demand sums"
        assert np.array_equal(self.tab.cpu().numpy(), o_tab), f"{where}: table'"


def words_of(rc, rm):
    return km.pack(rc, rm)


def same_outputs(o8, o32, where):
    assert np.array_equal(o8.idx[:o8.R].cpu().numpy().astype(np.int32), o32.idx[:o32.R].cpu().numpy()), f"{where}: indices vs int32"
    assert bool((o8.delta == o32.delta).all()) and bool((o8.tab == o32.tab).all()), f"{where}: sums / table' vs int32"


# ---- 1. world 1, the sharded snapshot step ---------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", CELLS, ids=[f"{['auto', 'grid', 'sorted', 'lut'][v]}-D{D}" for v, D in CELLS])
def test_packed_shard_cell(variant, D, alloc, egpu):
    """one packed sharded step + a non-committing apply against the oracle, then the int32 sharded step of the same
    requests: same indices, demand sums and table'; the scan is one launch (+ the lookup build), the table stays"""
    import torch
    fam = pm.family(variant, D)
    alloc.set_variant(variant)
    attach(alloc)
    s = stream(torch)
    step = 0
    for tname in km.cell_tables(D):
        for R in SHARD_ROWS:
            where = f"{fam} scan, variant {variant}, D = {D}, table {tname}, R = {R}"
            fc, fm, words = pm.cell_words(D, tname, R)
            exp = pm.ref(fc, fm, words)
            alloc.set_table(fc, fm)
            w = pm.words_dev(torch, words)
            o8 = pm.Out(torch, R, D)
            i, dl, t = o8.ptrs()
            torch.cuda.synchronize()
            n0 = alloc.launch_count
            alloc.bestfit_shard_packed_dev(w.data_ptr(), R, i, dl, step, s)
            assert alloc.launch_count - n0 == 1 + (fam == "lut"), f"{where}: launches"
            alloc.apply_peers_dev(step, t, False, s)
            torch.cuda.synchronize()
            o8.check(exp, where)
            c, m = (km._dev(torch, a) for a in km.unpack(words))
            o32 = Out32(torch, R, D)
            i, dl, t = o32.ptrs()
            alloc.bestfit_shard_dev(c.data_ptr(), m.data_ptr(), R, i, dl, step + 1, s)
            alloc.apply_peers_dev(step + 1, t, False, s)
            torch.cuda.synchronize()
            same_outputs(o8, o32, where)
            assert pm.table_is(alloc, fc, fm), f"{where}: the table changed"
            step += 2
    assert alloc.peer_last_timeout == 0
    alloc.peer_detach()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg3", "cfg4"])
def test_packed_shard_sequence_past_the_slot_ring(name, alloc, oracle_c, egpu):
    """packed and int32 sharded steps in turn, 2 * 140 steps (more than the 256 exchange slots), every fifth int32
    step's apply commits; one packed batch of 600 001 rows (above the 512 Ki-row bound).  After every step both
    agree with the oracle on the table then current, and at the end the context holds the oracle's table."""
    import torch
    w = egpu.synth.workload(name)
    D = int(w["D"])
    alloc.set_table(w["free_core"], w["free_mem"])
    attach(alloc)
    s = stream(torch)
    cur_c, cur_m = w["free_core"].copy(), w["free_mem"].copy()
    N = XCHG_SLOTS // 2 + 12
    for k in range(N):
        R = 600_001 if k == 3 else 20_003 + k
        rc, rm = egpu.synth.requests(w["dist"], 900 + k, R)
        words = words_of(rc, rm)
        exp = oracle_c.snapshot(cur_c, cur_m, *km.unpack(words), 4)
        o8, o32 = pm.Out(torch, R, D), Out32(torch, R, D)
        wd = pm.words_dev(torch, words)
        c, m = km._dev(torch, rc), km._dev(torch, rm)
        i, dl, t = o8.ptrs()
        alloc.bestfit_shard_packed_dev(wd.data_ptr(), R, i, dl, 2 * k, s)
        alloc.apply_peers_dev(2 * k, t, False, s)
        i, dl, t = o32.ptrs()
        alloc.bestfit_shard_dev(c.data_ptr(), m.data_ptr(), R, i, dl, 2 * k + 1, s)
        commit = k % 5 == 4
        alloc.apply_peers_dev(2 * k + 1, t, commit, s)
        torch.cuda.synchronize()
        o8.check(exp, f"step {k}")
        same_outputs(o8, o32, f"step {k}")
        if commit:
            cur_c, cur_m = np.maximum(exp[3][:D], 0), np.maximum(exp[3][D:2 * D], 0)
    assert alloc.peer_last_timeout == 0
    g_c, g_m, _ = alloc.table()
    assert np.array_equal(g_c, cur_c) and np.array_equal(g_m, cur_m)
    alloc.peer_detach()


# ---- 2. pipelining ---------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_packed_shard_pipelined_chain(alloc, egpu):
    """30 EGPU_F_INPUTS_READY launches on one stream - packed sharded scans, int32 sharded scans and packed multi-batch
    launches in turn, more than a launch group (24) - then the applies of the 20 sharded steps, a small packed step
    whose apply commits, and 5 more pipelined packed lookup scans that must see the committed table (the first of them
    rebuilds the lookup table)"""
    import torch
    D = 40
    rng = np.random.default_rng(4040)
    fc = rng.integers(50, 101, D).astype(np.int32)
    fm = rng.choice(np.arange(10_000, MEM_MAX + 1), D, replace=False).astype(np.int32)
    alloc.set_variant(LUT)
    alloc.set_table(fc, fm)
    attach(alloc)
    s = stream(torch)

    def rand_words(R):
        return km.pack(rng.integers(-1, 104, R), rng.integers(-1, 9000, R))

    chain, shard_outs = [], []
    for j in range(30):
        kind = ("packed", "int32", "multi")[j % 3]
        R = int(rng.integers(1, 30_000))
        words = rand_words(R)
        if kind == "multi":
            ws = [words, rand_words(int(rng.integers(0, 5_000)))]
            chain.append((kind, ws, [pm.words_dev(torch, x) for x in ws], [pm.Out(torch, x.size, D) for x in ws]))
        elif kind == "packed":
            chain.append((kind, words, pm.words_dev(torch, words), pm.Out(torch, R, D)))
        else:
            chain.append((kind, words, tuple(km._dev(torch, a) for a in km.unpack(words)), Out32(torch, R, D)))
    commit_words = km.pack(np.ones(7, np.int64), np.full(7, 3))
    cw, co = pm.words_dev(torch, commit_words), pm.Out(torch, 7, D)
    after = [rand_words(int(rng.integers(1000, 40_000))) for _ in range(5)]
    after_dev = [(pm.words_dev(torch, x), pm.Out(torch, x.size, D)) for x in after]
    torch.cuda.synchronize()  # every input is complete before the first launch
    step = 0
    for kind, words, dev, out in chain:
        if kind == "multi":
            pm.packed_multi(alloc, torch, dev, out, inputs_ready=True)
            continue
        i, dl, _ = out.ptrs()
        if kind == "packed":
            alloc.bestfit_shard_packed_dev(dev.data_ptr(), out.R, i, dl, step, s, inputs_ready=True)
        else:
            alloc.bestfit_shard_dev(dev[0].data_ptr(), dev[1].data_ptr(), out.R, i, dl, step, s, inputs_ready=True)
        shard_outs.append(out)
        step += 1
    assert step == 20
    alloc.apply_peers_multi_dev(0, [o.tab.data_ptr() for o in shard_outs], False, s)
    i, dl, t = co.ptrs()
    alloc.bestfit_shard_packed_dev(cw.data_ptr(), 7, i, dl, 20, s, inputs_ready=True)
    alloc.apply_peers_dev(20, t, True, s)
    for k, (wd, o) in enumerate(after_dev):
        i, dl, _ = o.ptrs()
        n0 = alloc.launch_count
        alloc.bestfit_shard_packed_dev(wd.data_ptr(), o.R, i, dl, 21 + k, s, inputs_ready=True)
        assert alloc.launch_count - n0 == (2 if k == 0 else 1), "the lookup table is rebuilt once, after the commit"
    alloc.apply_peers_multi_dev(21, [o.tab.data_ptr() for _, o in after_dev], False, s)
    torch.cuda.synchronize()
    assert alloc.peer_last_timeout == 0
    for j, (kind, words, dev, out) in enumerate(chain):
        if kind == "multi":
            for x, o in zip(words, out):
                o.check(pm.ref(fc, fm, x), f"launch {j} (packed multi-batch)")
        else:
            out.check(pm.ref(fc, fm, words), f"launch {j} ({kind} sharded)")
    c_exp = pm.ref(fc, fm, commit_words)
    co.check(c_exp, "committing step")
    assert not c_exp[3][2 * D:].any()
    new_fc, new_fm = c_exp[3][:D], c_exp[3][D:2 * D]
    assert not (np.array_equal(new_fc, fc) and np.array_equal(new_fm, fm))
    for k, (x, (_, o)) in enumerate(zip(after, after_dev)):
        o.check(pm.ref(new_fc, new_fm, x), f"packed lookup scan {k} after the commit")
    assert pm.table_is(alloc, new_fc, new_fm)
    alloc.peer_detach()


# ---- 3. lag ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg3", "cfg4"])
@pytest.mark.parametrize("lag", [1, 2, 16])
def test_packed_shard_lag(lag, name, alloc, oracle_c, egpu):
    """egpu_bestfit_batch_shard_lag_dev on words over more steps than exchange slots; the tail is flushed by one
    apply_peers_multi_dev.  Then the same call with EGPU_F_PACKED and an int32 d_req_mem: the int32 scan, as before."""
    import torch
    w = egpu.synth.workload(name)
    D = int(w["D"])
    fc, fm = w["free_core"], w["free_mem"]
    alloc.set_table(fc, fm)
    attach(alloc)
    st = torch.cuda.Stream()
    N = XCHG_SLOTS + 14
    bufs = []
    with torch.cuda.stream(st):
        for k in range(N):
            R = 3_001 + (k % 7)
            words = words_of(*egpu.synth.requests(w["dist"], 500 + k, R))
            bufs.append((words, pm.words_dev(torch, words), pm.Out(torch, R, D)))
    torch.cuda.synchronize()
    for k, (_, wd, o) in enumerate(bufs):
        i, dl, _ = o.ptrs()
        lagged = bufs[k - lag][2].tab.data_ptr() if k >= lag else 0
        alloc.bestfit_shard_lag_packed_dev(wd.data_ptr(), o.R, i, dl, k, lag, lagged, st.cuda_stream, inputs_ready=True)
    alloc.apply_peers_multi_dev(N - lag, [bufs[j][2].tab.data_ptr() for j in range(N - lag, N)], False, st.cuda_stream)
    torch.cuda.synchronize()
    assert alloc.peer_last_timeout == 0
    for k, (words, _, o) in enumerate(bufs):
        o.check(oracle_c.snapshot(fc, fm, *km.unpack(words)), f"step {k}")
    # EGPU_F_PACKED with a non-NULL d_req_mem: two int32 arrays and int32 indices, exactly as before this flag existed.
    # A new sequence from step 0 (the previous one is complete): steps 0 .. lag - 1 apply nothing, step `lag` applies
    # step 0 into o32.tab, one apply launch flushes steps 1 .. lag.
    rc, rm = egpu.synth.requests(w["dist"], 77, 5_003)
    c, m = km._dev(torch, rc), km._dev(torch, rm)
    o32 = Out32(torch, 5_003, D)
    i, dl, _ = o32.ptrs()
    for k in range(lag + 1):
        lagged = C.c_void_p(o32.tab.data_ptr()) if k == lag else None
        assert alloc._lib.egpu_bestfit_batch_shard_lag_dev(alloc.handle, C.c_void_p(c.data_ptr()), C.c_void_p(m.data_ptr()), 5_003,
                                                           C.c_void_p(i), C.c_void_p(dl), F_PACKED, k, lag, lagged, pm._s(torch)) == 0
    alloc.apply_peers_multi_dev(1, [0] * lag, False, stream(torch))
    torch.cuda.synchronize()
    o32.check(oracle_c.snapshot(fc, fm, rc, rm), "EGPU_F_PACKED with int32 arrays")
    assert alloc.peer_last_timeout == 0
    alloc.peer_detach()


# ---- 4. world 1, sharded prefix-commit -------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_shard_prefix_world1(variant, alloc, oracle_c, egpu):
    """at world 1 the sharded packed prefix-commit is the single-GPU packed prefix-commit: the device fills inside a
    tile, on a tile boundary, in the ragged tail or never; R = 0; a 1 M-row batch at D = 64; with and without commit"""
    import torch
    alloc.set_variant(variant)
    attach(alloc)
    s = stream(torch)
    R = 3 * 8192 + 3
    tile, _ = pp.tile_rows(R, 256, 8 if variant == SORTED else 32, 1 << 30)
    cases = {f"cut at {what}": pp.cut_case(R, T, 80 + n)
             for n, (what, T) in enumerate({"row 1": 1, "inside a tile": tile + 37, "a tile boundary": 2 * tile,
                                            "the tail": R - 2, "never": None}.items())}
    fc, fm, rc, rm = km.prefix_case(1_000_003)
    cases["1 M rows, D = 64"] = (fc, fm, km.pack(rc, rm))
    cases["R = 0"] = (fc, fm, np.zeros(0, np.uint32))
    step = 0
    for what, (fc, fm, words) in cases.items():
        D, n = fc.size, words.size
        exp = oracle_c.prefix_commit(fc, fm, *km.unpack(words))
        wd = pm.words_dev(torch, words)
        for commit in (False, True):
            where = f"{what}, commit {commit}"
            alloc.set_table(fc, fm)
            o = pm.Out(torch, n, D)
            i, dl, t = o.ptrs()
            alloc.bestfit_shard_prefix_packed_dev(wd.data_ptr(), n, i, dl, t, step, commit, s)
            torch.cuda.synchronize()
            step += 2
            o.check(exp, where)
            assert (o.tab[:2 * D] >= 0).all()
            assert pm.table_is(alloc, *(pp.installed(exp[3], D) if commit else (fc, fm))), where
            alloc.set_table(fc, fm)
            single = pm.Out(torch, n, D)
            pp.prefix_dev(alloc, torch, wd, single, commit)
            assert bool((single.idx == o.idx).all() and (single.delta == o.delta).all() and (single.tab == o.tab).all()), \
                f"{where}: differs from the single-GPU packed prefix-commit"
        if what.startswith("cut at") and what != "cut at never":
            assert (exp[0] == -2).any(), what
    assert alloc.peer_last_timeout == 0
    alloc.peer_detach()


# ---- 5. world 2: two processes on one GPU ----------------------------------------------------------------
W2_STEPS, W2_R = 7, 20_001


def _rank_main(rank, conn, peer_conn, mode, packed):
    """One rank of a world-2 sequence on cuda:0.  mode "snap": sharded step + apply, every third apply commits; "lag":
    the lag-2 form, tail flushed by one apply; "prefix": the rank-major prefix-commit cases of test_gpu_peer_exchange.
    packed: this rank's calls take words and int8 indices, otherwise int32 arrays."""
    sys.path.insert(0, ROOT)
    import torch
    import elastic_gpu_agent_b200 as e
    torch.cuda.set_device(0)
    a = e.BestFitAllocator(0)
    w = e.synth.workload("cfg3")
    a.set_table(*((pe.PREFIX_FC, pe.PREFIX_FM) if mode == "prefix" else (w["free_core"], w["free_mem"])))
    mine = a.peer_export()
    peer_conn.send(mine)
    other = peer_conn.recv()
    a.peer_attach(rank, 2, [mine, other] if rank == 0 else [other, mine])
    peer_conn.send("attached")
    assert peer_conn.recv() == "attached"
    s = torch.cuda.current_stream().cuda_stream
    D = 8
    keep, inputs = [], []  # outputs, and the inputs kept alive until the final synchronisation

    def buffers(rc, rm):
        R = rc.size
        if packed:
            return pm.words_dev(torch, km.pack(rc, rm)), pm.Out(torch, R, D)
        return (km._dev(torch, rc), km._dev(torch, rm)), Out32(torch, R, D)

    if mode == "prefix":
        for k, (n0, n1, fresh) in enumerate(pe.PREFIX_STEPS):
            if fresh:
                torch.cuda.synchronize()
                a.set_table(pe.PREFIX_FC, pe.PREFIX_FM)
            rc, rm = pe._prefix_requests(k, n0 + n1)
            rc, rm = (np.ascontiguousarray(x[:n0] if rank == 0 else x[n0:]) for x in (rc, rm))
            inp, out = buffers(rc, rm)
            i, dl, t = out.ptrs()
            if packed:
                a.bestfit_shard_prefix_packed_dev(inp.data_ptr(), out.R, i, dl, t, 2 * k, True, s)
            else:
                a.bestfit_shard_prefix_dev(inp[0].data_ptr(), inp[1].data_ptr(), out.R, i, dl, t, 2 * k, True, s)
            torch.cuda.synchronize()
            keep.append(out)
    else:
        lag = 2 if mode == "lag" else 0
        for step in range(W2_STEPS):
            rc, rm = e.synth.requests(3, 70 + step, W2_R, first_row=rank * W2_R)
            inp, out = buffers(rc, rm)
            i, dl, t = out.ptrs()
            if lag:
                lagged = keep[step - lag].tab.data_ptr() if step >= lag else 0
                if packed:
                    a.bestfit_shard_lag_packed_dev(inp.data_ptr(), out.R, i, dl, step, lag, lagged, s)
                else:
                    a.bestfit_shard_lag_dev(inp[0].data_ptr(), inp[1].data_ptr(), out.R, i, dl, step, lag, lagged, s)
            else:
                if packed:
                    a.bestfit_shard_packed_dev(inp.data_ptr(), out.R, i, dl, step, s)
                else:
                    a.bestfit_shard_dev(inp[0].data_ptr(), inp[1].data_ptr(), out.R, i, dl, step, s)
                a.apply_peers_dev(step, t, step % 3 == 2, s)
            keep.append(out)
            inputs.append(inp)
        if lag:
            a.apply_peers_multi_dev(W2_STEPS - lag, [keep[j].tab.data_ptr() for j in range(W2_STEPS - lag, W2_STEPS)], False, s)
    torch.cuda.synchronize()
    res = [(o.idx[:o.R].cpu().numpy().astype(np.int32), o.delta.cpu().numpy(), o.tab.cpu().numpy()) for o in keep]
    fc, fm, _ = a.table()
    conn.send((rank, res, fc, fm, a.peer_last_timeout))
    peer_conn.send("done")
    peer_conn.recv()
    a.peer_detach()
    a.close()


def _run_world2(mode, formats):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    a_conn, b_conn = ctx.Pipe()
    res0_r, res0_w = ctx.Pipe(False)
    res1_r, res1_w = ctx.Pipe(False)
    procs = [ctx.Process(target=_rank_main, args=(0, res0_w, a_conn, mode, formats[0])),
             ctx.Process(target=_rank_main, args=(1, res1_w, b_conn, mode, formats[1]))]
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
    assert r0[4] == 0 and r1[4] == 0, "a kernel timed out waiting for its peer"
    return r0, r1


W2_CASES = [("snap", (True, True)), ("lag", (True, True)), ("prefix", (True, True)), ("snap", (True, False)),
            ("lag", (False, True)), ("prefix", (False, True))]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,formats", W2_CASES, ids=[f"{m}-{'-'.join('packed' if f else 'int32' for f in fs)}" for m, fs in W2_CASES])
def test_packed_shard_world2(mode, formats, oracle_c, egpu):
    from elastic_gpu_agent_b200 import sharding
    r0, r1 = _run_world2(mode, formats)
    D = 8
    if mode == "prefix":
        cur_c, cur_m = pe.PREFIX_FC, pe.PREFIX_FM
        for k, (n0, n1, fresh) in enumerate(pe.PREFIX_STEPS):
            if fresh:
                cur_c, cur_m = pe.PREFIX_FC, pe.PREFIX_FM
            rc, rm = pe._prefix_requests(k, n0 + n1)
            o_idx, o_dc, o_dm, o_tab = oracle_c.prefix_commit(cur_c, cur_m, rc, rm)
            (i0, d0, t0), (i1, d1, t1) = r0[1][k], r1[1][k]
            assert np.array_equal(i0, o_idx[:n0]) and np.array_equal(i1, o_idx[n0:]), f"indices, step {k}"
            assert np.array_equal(d0, pe._rank_partial(o_idx[:n0], rc[:n0], rm[:n0], D)), k
            assert np.array_equal(d1, pe._rank_partial(o_idx[n0:], rc[n0:], rm[n0:], D)), k
            assert np.array_equal(t0, o_tab) and np.array_equal(t1, o_tab), k
            cur_c, cur_m = o_tab[:D].copy(), o_tab[D:2 * D].copy()
    else:
        w = egpu.synth.workload("cfg3")
        cur_c, cur_m = w["free_core"].copy(), w["free_mem"].copy()
        for step in range(W2_STEPS):
            tot = np.zeros(2 * D, dtype=np.int64)
            for rank, res in ((0, r0), (1, r1)):
                rc, rm = egpu.synth.requests(3, 70 + step, W2_R, first_row=rank * W2_R)
                o_idx, o_dc, o_dm, _ = oracle_c.snapshot(cur_c, cur_m, rc, rm)
                idx, dl, _ = res[1][step]
                assert np.array_equal(idx, o_idx), f"indices rank {rank} step {step}"
                assert np.array_equal(dl, np.concatenate([o_dc, o_dm])), f"demand rank {rank} step {step}"
                tot += np.concatenate([o_dc, o_dm])
            etab = sharding.combine_demands(cur_c, cur_m, tot[None, :])
            assert np.array_equal(r0[1][step][2], etab) and np.array_equal(r1[1][step][2], etab), f"table' step {step}"
            if step % 3 == 2 and mode == "snap":
                cur_c, cur_m = np.maximum(etab[:D], 0), np.maximum(etab[D:2 * D], 0)
    for res in (r0, r1):
        assert np.array_equal(res[2], cur_c) and np.array_equal(res[3], cur_m)


# ---- 6. CUDA graph ---------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_packed_shard_graph(alloc, oracle_c, egpu):
    """start gate, 6 pipelined packed sharded scans (cfg4: the lookup scan) and one apply launch on a second stream,
    captured once after an eager pass and replayed twice: every replay gives the oracle's outputs"""
    import torch
    w = egpu.synth.workload("cfg4")
    D = 64
    fc, fm = w["free_core"], w["free_mem"]
    alloc.set_table(fc, fm)
    attach(alloc)
    K, R = 6, 30_001
    words = [words_of(*egpu.synth.requests(w["dist"], 40 + k, R)) for k in range(K)]
    exps = [oracle_c.snapshot(fc, fm, *km.unpack(x)) for x in words]
    wds = [pm.words_dev(torch, x) for x in words]
    outs = [pm.Out(torch, R, D) for _ in range(K)]
    st, ap = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()

    def region(scan, gated):
        if gated:
            alloc.gate_dev(scan.cuda_stream)
        for k, (wd, o) in enumerate(zip(wds, outs)):
            i, dl, _ = o.ptrs()
            alloc.bestfit_shard_packed_dev(wd.data_ptr(), R, i, dl, k, scan.cuda_stream, inputs_ready=True)
        alloc.apply_peers_multi_dev(0, [o.tab.data_ptr() for o in outs], False, ap.cuda_stream)

    def check(where):
        for k, (o, e) in enumerate(zip(outs, exps)):
            o.check(e, f"{where}, step {k}")
            o.reset()
        torch.cuda.synchronize()

    ap.wait_stream(st)
    region(st, False)
    st.wait_stream(ap)
    torch.cuda.synchronize()
    check("eager")
    g = torch.cuda.CUDAGraph()
    cap = torch.cuda.Stream()
    cap.wait_stream(st)
    with torch.cuda.stream(cap):
        with torch.cuda.graph(g, stream=cap):
            ap.wait_stream(cap)
            region(cap, True)
            cap.wait_stream(ap)
    torch.cuda.synchronize()
    for rep in range(2):
        g.replay()
        alloc.gate_open()
        torch.cuda.synchronize()
        check(f"replay {rep}")
    assert alloc.gate_timeouts == 0 and alloc.peer_last_timeout == 0
    assert pm.table_is(alloc, fc, fm)
    alloc.peer_detach()


# ---- 7. arguments ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_packed_shard_arguments(alloc, egpu):
    import torch
    D = 6
    fc, fm = np.array([3, 50, 100, 100, 0, 7], np.int32), np.array([10, 500, MEM_MAX, 0, 9, 64], np.int32)
    lib, h, s = alloc._lib, alloc.handle, pm._s(torch)
    words = km.pack(np.arange(200) % 103, (np.arange(200) * 37) % 600)
    w = pm.words_dev(torch, words)
    idx = torch.full((1024,), -9, dtype=torch.int8, device="cuda")
    c32 = torch.zeros(204, dtype=torch.int32, device="cuda")
    tab = torch.full((3 * D,), -7, dtype=torch.int32, device="cuda")
    wp, ip, mp, tp = w.data_ptr(), idx.data_ptr(), c32.data_ptr(), tab.data_ptr()
    vp = C.c_void_p

    def shard(core, mem, R, out, flags, step=0):
        return lib.egpu_bestfit_batch_shard_dev(h, vp(core), vp(mem), R, vp(out), None, flags, step, s)

    def lag(core, mem, R, out, flags, step=0):
        return lib.egpu_bestfit_batch_shard_lag_dev(h, vp(core), vp(mem), R, vp(out), None, flags, step, 2, vp(tp), s)

    def prefix(core, mem, R, out, flags, step=0):
        return lib.egpu_bestfit_batch_shard_prefix_dev(h, vp(core), vp(mem), R, vp(out), None, vp(tp), flags, step, s)

    alloc.set_table(fc, fm)
    # unattached: every packed sharded call is a state error
    assert shard(wp, None, 100, ip, F_PACKED) == ERR_STATE
    assert lag(wp, None, 100, ip, F_PACKED) == ERR_STATE
    assert prefix(wp, None, 100, ip, F_PACKED | F_PREFIX) == ERR_STATE
    attach(alloc)
    torch.cuda.synchronize()
    n0 = alloc.launch_count
    P, PP = F_PACKED, F_PACKED | F_PREFIX
    refused = {
        "shard: req_mem given": shard(wp, mp, 100, ip, P),
        "shard: req_mem given, R = 0": shard(wp, mp, 0, ip, P),
        "shard: NULL words": shard(None, None, 100, ip, P),
        "shard: NULL indices": shard(wp, None, 100, None, P),
        "shard: misaligned words": shard(wp + 4, None, 100, ip, P),
        "shard: misaligned indices": shard(wp, None, 100, ip + 1, P | F_INPUTS_READY),
        "shard: commit": shard(wp, None, 100, ip, P | F_COMMIT),
        "shard: prefix-commit": shard(wp, None, 100, ip, P | F_PREFIX),
        "shard: step >= 2^47": shard(wp, None, 100, ip, P, 1 << 47),
        "lag: NULL words": lag(None, None, 100, ip, P),
        "lag: NULL indices": lag(wp, None, 100, None, P),
        "lag: misaligned words": lag(wp + 4, None, 100, ip, P),
        "lag: misaligned indices": lag(wp, None, 100, ip + 1, P),
        "lag: commit": lag(wp, None, 100, ip, P | F_COMMIT),
        "prefix: req_mem given": prefix(wp, mp, 100, ip, PP),
        "prefix: NULL words": prefix(None, None, 100, ip, PP),
        "prefix: NULL indices": prefix(wp, None, 100, None, PP | F_COMMIT),
        "prefix: misaligned words": prefix(wp + 4, None, 100, ip, PP),
        "prefix: misaligned indices": prefix(wp, None, 100, ip + 1, P),
        "prefix: inputs ready": prefix(wp, None, 100, ip, PP | F_INPUTS_READY),
        "prefix: step >= 2^47": prefix(wp, None, 100, ip, PP, 1 << 47),
    }
    for what, code in refused.items():
        assert code == ERR_INVALID, what
    alloc.set_variant(GRID)
    assert shard(wp, None, 100, ip, P) == ERR_STATE
    assert lag(wp, None, 100, ip, P) == ERR_STATE
    assert prefix(wp, None, 100, ip, PP) == ERR_STATE
    assert prefix(wp, None, 100, ip, P | F_COMMIT) == ERR_STATE
    alloc.set_variant(AUTO)
    torch.cuda.synchronize()
    assert alloc.launch_count == n0, "a refused call launched"
    assert bool((idx == -9).all()) and bool((tab == -7).all()), "a refused call wrote"
    assert pm.table_is(alloc, fc, fm)
    # the accepted forms: the flag alone (no EGPU_F_PREFIX_COMMIT) on the prefix call, and R = 0 everywhere
    exp = pp.ref(fc, fm, words)
    o = pm.Out(torch, 200, D)
    i, dl, t = o.ptrs()
    assert lib.egpu_bestfit_batch_shard_prefix_dev(h, vp(wp), None, 200, vp(i), vp(dl), vp(t), P, 0, s) == 0
    torch.cuda.synchronize()
    o.check(exp, "EGPU_F_PACKED alone on the prefix call")
    e = pm.Out(torch, 0, D)
    i, dl, t = e.ptrs()
    alloc.bestfit_shard_packed_dev(wp, 0, i, dl, 2, stream(torch))
    alloc.apply_peers_dev(2, t, False, stream(torch))
    torch.cuda.synchronize()
    e.check(pm.ref(fc, fm, words[:0]), "R = 0")
    assert alloc.peer_last_timeout == 0
    alloc.peer_detach()
