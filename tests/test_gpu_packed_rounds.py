"""Prefix-commit rounds to the fixed point in the packed format: egpu_bestfit_batch[_dev] with
EGPU_F_PACKED | EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT | EGPU_F_ROUNDS.

The words and int8 indices are those of packed prefix-commit; the call runs committing packed
prefix-commit rounds, re-submitting the deferred words in order (deferred_count_packed_kernel,
deferred_scan_kernel, deferred_scatter_packed_kernel, round_writeback_packed_kernel), until a round
defers nothing.  Every GPU case compares exactly with the C or numpy rounds oracle on the requests the
words stand for (not a request: (-1, -1)), and most also with the int32 egpu_bestfit_batch_rounds_dev:

  1. the cell matrix: both packed scans at every D bucket, under AUTO, SORTED and LUT, ragged row
     counts, domain-edge words and tables; d_table_out, the installed table and the guard bytes;
  2. the number of kernels each round launches;
  3. compaction edges: deferred rows across 1024-row tiles, rounds of n % 4 != 0 rows, a round of one
     row, R = 1 and R = 0, zero-demand rows and words that are not requests, the cfg1 known answer;
  4. 4 Mi + 3 rows at D = 64 under both scans;
  5. the host entry point with pageable and pinned buffers, demand sums NULL and not;
  6. argument checks on both entry points, and that a refused call launches and writes nothing;
  7. agreement with rounds driven by the caller;
  8. what the launches after the call see, behind a pipelined chain of multi-batch launches.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_context_sequences as cs  # noqa: E402  (probe rows)
import test_gpu_kernel_matrix as km  # noqa: E402  (cell tables, pack / unpack, int32 device arrays)
import test_gpu_packed_multi as pm  # noqa: E402  (cells, Out, guard bytes, packed multi-batch launches)

MEM_MAX = (1 << 18) - 1
ERR_INVALID, ERR_NO_TABLE, ERR_STATE = -1, -5, -6
AUTO, GRID, SORTED, LUT = 0, 1, 2, 3
F_COMMIT, F_INPUTS_READY, F_PREFIX, F_APPLY, F_PACKED, F_ROUNDS = 1, 2, 4, 8, 16, 32
PR = F_PACKED | F_PREFIX | F_COMMIT | F_ROUNDS
TILE = 1024  # rows per compaction tile (kCompactTile)


def test_rounds_flag_value():
    import elastic_gpu_agent_b200._lib as L
    src = open(os.path.join(pm.ROOT, "include", "egpu_alloc.h")).read()
    assert "#define EGPU_F_ROUNDS       32" in src and L.F_ROUNDS == F_ROUNDS


# ---- references and calls ------------------------------------------------------------------------------
def ref(oracle_c, fc, fm, words):
    """(idx, delta_core, delta_mem, table' as the last round writes it, rounds) of the C rounds oracle"""
    o_idx, o_dc, o_dm, o_fc, o_fm, o_rounds, o_left = oracle_c.rounds(fc, fm, *km.unpack(words))
    assert o_left == 0 and not (o_idx == -2).any()
    tab = np.concatenate([o_fc, o_fm, np.zeros(len(fc), np.int32)]).astype(np.int32)
    return o_idx, o_dc, o_dm, tab, o_rounds


def round_sizes(oracle_c, fc, fm, words):
    """rows scored in each round, from the oracle stopped after 1, 2, ... rounds"""
    rc, rm = km.unpack(words)
    sizes, n = [words.size], 1
    while True:
        _, _, _, _, _, r, left = oracle_c.rounds(fc, fm, rc, rm, max_rounds=n)
        if left == 0:
            return sizes[:r]
        sizes.append(left)
        n += 1


def launches(n_rounds, lut):
    """kernels run_rounds launches for n rounds: every round the prefix-commit pipeline (scan, cut, apply,
    finalize, and the lookup build after the previous round's commit), then count and scan; every later
    round a scatter before it and a writeback after it"""
    if n_rounds == 0:
        return 4 + lut
    return n_rounds * (4 + lut + 2) + (n_rounds - 1) * 2


def rounds_dev(alloc, torch, w, o, flags=0):
    """the packed rounds on device buffers; returns the launch count it added"""
    torch.cuda.synchronize()
    n0 = alloc.launch_count
    i, dl, t = o.ptrs()
    rc = alloc._lib.egpu_bestfit_batch_dev(alloc.handle, C.c_void_p(w.data_ptr()), None, o.R, C.c_void_p(i), C.c_void_p(dl),
                                           C.c_void_p(t), PR | flags, pm._s(torch))
    assert rc == 0
    return alloc.launch_count - n0


def installed(tab, D):
    return tab[:D], tab[D:2 * D]


def int32_rounds(alloc, torch, variant, fc, fm, words):
    """egpu_bestfit_batch_rounds_dev on the requests the words stand for: (idx, delta, installed table)"""
    rc, rm = km.unpack(words)
    alloc.set_variant(variant)
    alloc.set_table(fc, fm)
    c, m = km._dev(torch, rc), km._dev(torch, rm)
    idx = torch.full((words.size + 4,), -9, dtype=torch.int32, device="cuda")
    delta, _, left = alloc.bestfit_rounds_dev(c.data_ptr(), m.data_ptr(), words.size, idx.data_ptr(),
                                              stream=torch.cuda.current_stream().cuda_stream)
    assert left == 0
    return idx[:words.size].cpu().numpy(), delta, alloc.table()


def run_case(alloc, torch, oracle_c, variant, fc, fm, words, where, exp=None, int32=True):
    """packed rounds against the oracle (indices, sums, table', installed table, guard bytes, launches),
    then the int32 rounds on the same requests"""
    D = fc.size
    exp = ref(oracle_c, fc, fm, words) if exp is None else exp
    alloc.set_variant(variant)
    alloc.set_table(fc, fm)
    o = pm.Out(torch, words.size, D)
    n = rounds_dev(alloc, torch, pm.words_dev(torch, words), o)
    o.check(exp[:4], where)
    lut = pm.family(variant, D) == "lut"
    assert n == launches(exp[4] if words.size else 0, lut), f"{where}: launches for {exp[4]} rounds"
    assert pm.table_is(alloc, *installed(exp[3], D)), f"{where}: installed table"
    if int32:
        idx, delta, tab = int32_rounds(alloc, torch, variant, fc, fm, words)
        got = o.idx[:o.R].cpu().numpy().astype(np.int32)
        assert np.array_equal(got, idx) and np.array_equal(o.delta.cpu().numpy(), delta), f"{where}: differs from int32"
        assert all(np.array_equal(a, b) for a, b in zip(tab, (*installed(exp[3], D), np.zeros(D, np.int32)))), where
    return o


# ---- 1. the cell matrix ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", pm.CELLS, ids=[f"{['auto', 'grid', 'sorted', 'lut'][v]}-D{D}" for v, D in pm.CELLS])
def test_packed_rounds_cell(variant, D, alloc, oracle_c):
    import torch
    for tname in km.cell_tables(D):
        for R in km.ROW_COUNTS:
            fc, fm, words = pm.cell_words(D, tname, R)
            run_case(alloc, torch, oracle_c, variant, fc, fm, words, f"variant {variant}, D = {D}, table {tname}, R = {R}")


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_rounds_against_numpy_oracle(variant, alloc, oracle_c):
    """a random batch of several rounds, also against the numpy rounds (independent of the C loop)"""
    import torch
    from oracle import bestfit_np
    rng = np.random.default_rng(40 + variant)
    D = 12
    fc = rng.integers(20, 101, D).astype(np.int32)
    fm = rng.integers(5000, MEM_MAX + 1, D).astype(np.int32)
    words = km.pack(rng.integers(-1, 40, 9001), rng.integers(-1, 9000, 9001))
    n_idx, n_dc, n_dm, n_fc, n_fm, n_rounds, n_left = bestfit_np.rounds(fc, fm, *km.unpack(words))
    exp = ref(oracle_c, fc, fm, words)
    assert n_left == 0 and n_rounds == exp[4] >= 3
    assert np.array_equal(n_idx, exp[0]) and np.array_equal(n_dc, exp[1]) and np.array_equal(n_dm, exp[2])
    run_case(alloc, torch, oracle_c, variant, fc, fm, words, "random", exp)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_rounds_keep_oversub_flags(variant, alloc, oracle_c):
    """sticky oversubscription flags from a committing snapshot survive the rounds, as in the int32 rounds"""
    import torch
    from oracle import bestfit_np
    D = 5
    fc, fm = np.array([4, 10, 0, 100, 7], np.int32), np.array([50, 9, 0, MEM_MAX, 300], np.int32)
    rc, rm = np.array([4, 4, 10, 0, 99] * 3, np.int32), np.array([50, 1, 9, 0, 70_000] * 3, np.int32)
    _, _, _, o_tab = bestfit_np.snapshot(fc, fm, rc, rm)
    c_fc, c_fm, c_ov = km.committed(o_tab, D)
    assert c_ov.any()
    words = km.pack(np.arange(600) % 12, (np.arange(600) * 7) % 90)
    exp = ref(oracle_c, c_fc, c_fm, words)
    alloc.set_variant(variant)
    alloc.set_table(fc, fm)
    alloc.bestfit(rc, rm, commit=True)
    o = pm.Out(torch, words.size, D)
    rounds_dev(alloc, torch, pm.words_dev(torch, words), o)
    o.check(exp[:4], "packed rounds")
    assert pm.table_is(alloc, *installed(exp[3], D), c_ov)
    alloc.set_table(fc, fm)
    alloc.bestfit(rc, rm, commit=True)
    alloc.bestfit_rounds(*km.unpack(words))
    assert pm.table_is(alloc, *installed(exp[3], D), c_ov)


# ---- 2. + 3. round count and compaction edges -------------------------------------------------------------
def straddle_case(R, T, seed):
    """D = 2.  Device 0 = (0, fm0): rows (0, 1) choose it, fm0 of them fit, and row T is its first deferred
    row, so round 2 holds every (0, 1) row from T on, across several compaction tiles.  Device 1 = (0, 0):
    rows (0, 0) choose it and always commit.  One row in ten is not a request."""
    rng = np.random.default_rng(seed)
    kind = rng.choice(3, R, p=[0.7, 0.2, 0.1])
    kind[T] = 0
    words = np.where(kind == 0, 1, np.where(kind == 1, 0, 0xFFFFFFFF)).astype(np.uint32)
    return np.array([0, 0], np.int32), np.array([int((kind[:T] == 0).sum()), 0], np.int32), words


LADDER = (60, 60, 30, 30, 8, 8, 1, 1, 1)


def ladder_case(R, seed):
    """D = 1, 100 cores.  Zero-demand rows, a few words that are not requests, and the LADDER requests in
    order at random rows.  Round k commits one step of the ladder and defers everything after the next
    one (the zero-demand rows included), which no longer fits in round k + 1: five rounds, each a few
    rows shorter than the one before"""
    rng = np.random.default_rng(seed)
    words = np.zeros(R, np.uint32)
    words[rng.integers(0, R, R // 50)] = 0xFFFFFFFF
    at = np.sort(rng.choice(R, len(LADDER), replace=False))
    words[at] = km.pack(LADDER, [5] * len(LADDER))
    return np.array([100], np.int32), np.array([MEM_MAX], np.int32), words


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_rounds_compaction_edges(variant, alloc, oracle_c):
    import torch
    cases = {}
    # deferred rows across compaction tiles; round 2 of a size that is not a multiple of 4
    R = 5 * TILE + 7
    straddle = {}
    for T in (TILE - 3, TILE, 2 * TILE - 1):
        for seed in range(8):
            fc, fm, words = straddle_case(R, T, seed)
            sizes = round_sizes(oracle_c, fc, fm, words)
            if sizes[1] % 4:
                break
        assert sizes == [R, sizes[1]] and sizes[1] % 4 and sizes[1] > 2 * TILE, (T, sizes)
        cases[f"straddle from row {T}"] = (fc, fm, words)
        straddle[f"straddle from row {T}"] = T
    # many rounds of ragged sizes
    for seed in range(8):
        fc, fm, words = ladder_case(3 * TILE + 1, seed)
        sizes = round_sizes(oracle_c, fc, fm, words)
        if sum(s % 4 != 0 for s in sizes) >= 3:
            break
    assert len(sizes) == 5 and sum(s % 4 != 0 for s in sizes) >= 3, sizes
    cases["ladder"] = (fc, fm, words)
    # a round of exactly one row: device 0 takes fm0 (0, 1) rows, the last one is deferred
    fc, fm = np.array([0, 0], np.int32), np.array([3000, 0], np.int32)
    words = np.where(np.arange(5000) % 3 == 0, 0, 1).astype(np.uint32)
    words[np.flatnonzero(words == 1)[3001:]] = 0xFFFFFFFF
    assert round_sizes(oracle_c, fc, fm, words) == [5000, 1]
    cases["one deferred row"] = (fc, fm, words)
    # R = 1: a row that commits, one that is infeasible, one that is not a request, a zero-demand row
    fc1, fm1 = np.array([10, 3], np.int32), np.array([100, 7], np.int32)
    for w in (km.pack([3], [7]), km.pack([11], [0]), np.array([0xFFFFFFFF], np.uint32), np.array([1 << 25], np.uint32),
              km.pack([0], [0])):
        cases[f"R = 1, word {int(w[0]):#x}"] = (fc1, fm1, w)
    # R = 0: the packed prefix-commit with R = 0
    cases["R = 0"] = (fc1, fm1, np.zeros(0, np.uint32))
    # zero-demand rows and words that are not requests, mixed into rows that defer
    rng = np.random.default_rng(9)
    words = km.pack(rng.integers(0, 4, 4003), rng.integers(0, 5, 4003))
    words[rng.integers(0, 4003, 500)] = 0
    words[rng.integers(0, 4003, 300)] = rng.integers(1 << 25, 1 << 32, 300, dtype=np.uint64).astype(np.uint32)
    words[rng.integers(0, 4003, 300)] = (rng.integers(101, 128, 300).astype(np.uint32) << 18)
    fcz, fmz = np.array([60, 0, 30], np.int32), np.array([900, 0, MEM_MAX], np.int32)
    assert len(round_sizes(oracle_c, fcz, fmz, words)) >= 3
    cases["zero demand and not requests"] = (fcz, fmz, words)
    for what, (fc, fm, words) in cases.items():
        o = run_case(alloc, torch, oracle_c, variant, fc, fm, words, what)
        if what in straddle:  # the (0, 1) rows before T commit in round 1, the rest end infeasible in round 2
            T, got, a = straddle[what], o.idx[:o.R].cpu().numpy(), words == 1
            assert (got[:T][a[:T]] == 0).all() and (got[T:][a[T:]] == -1).all(), what


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_rounds_cfg1_known_answer(variant, alloc, egpu, oracle_c):
    """five (25, 1024) requests on 8 full devices: four fit device 0, the fifth goes to device 1 in round 2"""
    import torch
    w = egpu.synth.workload("cfg1")
    fc, fm = np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32)
    words = km.pack([25] * 5, [1024] * 5)
    exp = ref(oracle_c, fc, fm, words)
    assert exp[0].tolist() == [0, 0, 0, 0, 1] and exp[4] == 2
    run_case(alloc, torch, oracle_c, variant, fc, fm, words, "cfg1")
    alloc.set_variant(variant)
    alloc.set_table(fc, fm)
    idx, dc, dm = alloc.bestfit_packed_prefix(words, rounds=True)
    assert idx.tolist() == [0, 0, 0, 0, 1] and dc[:2].tolist() == [100, 25] and dm[:2].tolist() == [4096, 1024]


# ---- 4. scale --------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_packed_rounds_at_scale(alloc, oracle_c):
    import torch
    R, D = (4 << 20) + 3, 64
    fc, fm, rc, rm = km.prefix_case(R)
    words = km.pack(rc, rm)
    exp = ref(oracle_c, fc, fm, words)
    assert exp[4] >= 3, exp[4]
    for variant in (SORTED, LUT):
        run_case(alloc, torch, oracle_c, variant, fc, fm, words, f"4 Mi + 3 rows, variant {variant}", exp)


# ---- 5. the host entry point ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_rounds_host(variant, alloc, oracle_c):
    import torch
    rng = np.random.default_rng(800 + variant)
    D = 20
    fc = rng.integers(0, 101, D).astype(np.int32)
    fm = rng.integers(0, MEM_MAX + 1, D).astype(np.int32)
    R = 70_001
    words = km.pack(rng.integers(-1, 60, R), rng.integers(-1, 30_000, R))
    exp = ref(oracle_c, fc, fm, words)
    assert exp[4] >= 2
    dev = run_case(alloc, torch, oracle_c, variant, fc, fm, words, "device form", exp, int32=False)
    dev_idx = dev.idx[:R].cpu().numpy()
    alloc.set_variant(variant)
    alloc.set_table(fc, fm)
    idx, dc, dm = alloc.bestfit_packed_prefix(words, rounds=True)
    assert idx.dtype == np.int8 and np.array_equal(idx, dev_idx)
    assert np.array_equal(dc, exp[1]) and np.array_equal(dm, exp[2])
    assert pm.table_is(alloc, *installed(exp[3], D))
    p_words = alloc.pinned_array(R, np.uint32)
    p_idx = alloc.pinned_array(R + 16, np.int8)
    try:
        p_words[:] = words
        for with_delta in (False, True):
            p_idx[:] = -9
            alloc.set_table(fc, fm)
            dc, dm = np.full(D, -1, np.int64), np.full(D, -1, np.int64)
            rc = alloc._lib.egpu_bestfit_batch(alloc.handle, C.c_void_p(p_words.ctypes.data), None, R, C.c_void_p(p_idx.ctypes.data),
                                               C.c_void_p(dc.ctypes.data if with_delta else None),
                                               C.c_void_p(dm.ctypes.data if with_delta else None), PR)
            assert rc == 0
            assert np.array_equal(p_idx[:R], dev_idx) and (p_idx[R:] == -9).all(), with_delta
            if with_delta:
                assert np.array_equal(dc, exp[1]) and np.array_equal(dm, exp[2])
            else:
                assert (dc == -1).all() and (dm == -1).all()
            assert pm.table_is(alloc, *installed(exp[3], D)), with_delta
    finally:
        alloc.host_free(p_words.ctypes.data)
        alloc.host_free(p_idx.ctypes.data)
    # R = 0 through the host form
    alloc.set_table(fc, fm)
    idx, dc, dm = alloc.bestfit_packed_prefix(np.zeros(0, np.uint32), rounds=True)
    assert idx.size == 0 and not dc.any() and not dm.any() and pm.table_is(alloc, fc, fm)


# ---- 6. arguments ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_packed_rounds_arguments(alloc, egpu, oracle_c):
    import torch
    D = 6
    fc, fm = np.array([3, 50, 100, 100, 0, 7], np.int32), np.array([10, 500, MEM_MAX, 0, 9, 64], np.int32)
    alloc.set_table(fc, fm)
    s = pm._s(torch)
    words = km.pack(np.arange(200) % 103, (np.arange(200) * 37) % 600)
    w = pm.words_dev(torch, words)
    idx = torch.full((1024,), -9, dtype=torch.int8, device="cuda")
    c32 = torch.zeros(204, dtype=torch.int32, device="cuda")
    i32 = torch.full((204,), -9, dtype=torch.int32, device="cuda")
    wp, ip, mp = w.data_ptr(), idx.data_ptr(), c32.data_ptr()
    h_words = np.ascontiguousarray(words)
    h_idx = np.full(256, -9, np.int8)
    h_mem = np.zeros(200, np.int32)
    h_i32 = np.full(200, -9, np.int32)
    hw, hi, hm = h_words.ctypes.data, h_idx.ctypes.data, h_mem.ctypes.data
    BIG = 1 << 31

    def dev(core, mem, R, out, flags, a=alloc):
        return a._lib.egpu_bestfit_batch_dev(a.handle, C.c_void_p(core), C.c_void_p(mem), R, C.c_void_p(out), None, None, flags, s)

    def host(core, mem, R, out, flags, a=alloc):
        return a._lib.egpu_bestfit_batch(a.handle, C.c_void_p(core), C.c_void_p(mem), R, C.c_void_p(out), None, None, flags)

    combos = {
        "the flag alone": F_ROUNDS,
        "without packed": PR & ~F_PACKED,
        "without prefix-commit": PR & ~F_PREFIX,
        "without commit": PR & ~F_COMMIT,
        "packed only": F_PACKED | F_ROUNDS,
        "with EGPU_F_APPLY": PR | F_APPLY,
        "with bit 64": PR | 64,
    }
    torch.cuda.synchronize()
    n0 = alloc.launch_count
    refused = {}
    for what, flags in combos.items():
        int32_args = not (flags & F_PACKED)
        refused[f"dev: {what}"] = dev(mp if int32_args else wp, mp if int32_args else None, 100,
                                      i32.data_ptr() if int32_args else ip, flags)
        refused[f"host: {what}"] = host(hm if int32_args else hw, hm if int32_args else None, 100,
                                        h_i32.ctypes.data if int32_args else hi, flags)
    refused.update({
        "dev: req_mem given": dev(wp, mp, 100, ip, PR),
        "dev: req_mem given, R = 0": dev(wp, mp, 0, ip, PR),
        "dev: misaligned words": dev(wp + 4, None, 100, ip, PR),
        "dev: misaligned indices": dev(wp, None, 100, ip + 1, PR),
        "dev: NULL words": dev(None, None, 100, ip, PR),
        "dev: NULL indices": dev(wp, None, 100, None, PR),
        "dev: R = 2^31": dev(wp, None, BIG, ip, PR),
        "host: req_mem given": host(hw, hm, 100, hi, PR),
        "host: NULL words": host(None, None, 100, hi, PR),
        "host: NULL indices": host(hw, None, 100, None, PR),
        "host: R = 2^31": host(hw, None, BIG, hi, PR),
    })
    for what, code in refused.items():
        assert code == ERR_INVALID, what
    alloc.set_variant(GRID)
    assert dev(wp, None, 100, ip, PR) == ERR_STATE
    assert host(hw, None, 100, hi, PR) == ERR_STATE
    assert dev(wp, None, 0, ip, PR) == ERR_STATE
    alloc.set_variant(AUTO)
    torch.cuda.synchronize()
    assert alloc.launch_count == n0, "a refused call launched"
    assert bool((idx == -9).all()) and (h_idx == -9).all() and bool((i32 == -9).all()) and (h_i32 == -9).all(), \
        "a refused call wrote indices"
    assert pm.table_is(alloc, fc, fm)
    fresh = egpu.BestFitAllocator(0)
    try:
        f0 = fresh.launch_count
        assert dev(wp, None, 100, ip, PR, fresh) == ERR_NO_TABLE
        assert host(hw, None, 100, hi, PR, fresh) == ERR_NO_TABLE
        assert fresh.launch_count == f0
    finally:
        fresh.close()
    torch.cuda.synchronize()
    assert bool((idx == -9).all()) and (h_idx == -9).all()
    # EGPU_F_INPUTS_READY is accepted and changes nothing
    o = pm.Out(torch, 200, D)
    rounds_dev(alloc, torch, w, o, F_INPUTS_READY)
    exp = ref(oracle_c, fc, fm, words)
    o.check(exp[:4], "inputs ready")
    assert pm.table_is(alloc, *installed(exp[3], D))


# ---- 7. agreement with the caller-driven loop ---------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_rounds_equal_the_caller_loop(variant, alloc, oracle_c):
    """the loop of test_packed_prefix_rounds_by_the_caller (re-submit the deferred words until none is
    left) and one call with EGPU_F_ROUNDS give the same indices, sums and table"""
    import torch
    rng = np.random.default_rng(700 + variant)
    D = 6
    fc = rng.integers(30, 101, D).astype(np.int32)
    fm = rng.integers(20_000, MEM_MAX + 1, D).astype(np.int32)
    R = 4001
    words = km.pack(rng.integers(0, 12, R), rng.integers(0, 3000, R))
    alloc.set_variant(variant)
    alloc.set_table(fc, fm)
    out = np.full(R, -2, np.int8)
    sum_c, sum_m = np.zeros(D, np.int64), np.zeros(D, np.int64)
    rows = np.arange(R)
    n = 0
    while rows.size:
        idx, dc, dm = alloc.bestfit_packed_prefix(words[rows], commit=True)
        out[rows] = idx
        sum_c += dc
        sum_m += dm
        rows = rows[idx == -2]
        n += 1
    loop_table = alloc.table()
    assert n >= 3
    alloc.set_table(fc, fm)
    idx, dc, dm = alloc.bestfit_packed_prefix(words, rounds=True)
    assert np.array_equal(idx, out) and np.array_equal(dc, sum_c) and np.array_equal(dm, sum_m)
    assert all(np.array_equal(a, b) for a, b in zip(alloc.table(), loop_table))
    exp = ref(oracle_c, fc, fm, words)
    assert exp[4] == n
    o = run_case(alloc, torch, oracle_c, variant, fc, fm, words, "device form", exp, int32=False)
    assert np.array_equal(o.idx[:R].cpu().numpy(), out)


# ---- 8. what follows the call ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_rounds_after_pipelined_chain(variant, alloc, oracle_c):
    """12 pipelined multi-batch launches (packed and int32 in turn), then packed rounds on the same stream:
    the chain's outputs are exact, and packed multi-batch launches (register and lookup scans), an int32
    prefix-commit and table() all read the table the rounds installed"""
    import torch
    from oracle import bestfit_np
    D = 24
    rng = np.random.default_rng(8000 + variant)
    fc = rng.integers(20, 101, D).astype(np.int32)
    fm = rng.choice(np.arange(1000, MEM_MAX + 1), D, replace=False).astype(np.int32)
    alloc.set_variant(variant)
    alloc.set_table(fc, fm)
    s = torch.cuda.current_stream().cuda_stream
    chain = []
    for j in range(12):
        batches = []
        for _ in range(3):
            R = int(rng.integers(1, 20_000))
            words = km.pack(rng.integers(-1, 103, R), rng.integers(-1, 4000, R))
            batches.append((words, pm.ref(fc, fm, words)))
        packed = j % 2 == 0
        if packed:
            dev = [(pm.words_dev(torch, wd), pm.Out(torch, wd.size, D)) for wd, _ in batches]
        else:
            dev = [(km._dev(torch, km.unpack(wd)[0]), km._dev(torch, km.unpack(wd)[1]),
                    torch.full((wd.size + 4,), -9, dtype=torch.int32, device="cuda"),
                    torch.full((2 * D,), -1, dtype=torch.int64, device="cuda"),
                    torch.full((3 * D,), -7, dtype=torch.int32, device="cuda")) for wd, _ in batches]
        chain.append((packed, batches, dev))
    rwords = km.pack(rng.integers(0, 30, 50_000), rng.integers(0, 900, 50_000))
    r_exp = ref(oracle_c, fc, fm, rwords)
    assert r_exp[4] >= 2
    rw, ro = pm.words_dev(torch, rwords), pm.Out(torch, rwords.size, D)
    torch.cuda.synchronize()  # every input is complete before the first launch
    for packed, batches, dev in chain:
        if packed:
            pm.packed_multi(alloc, torch, [w for w, _ in dev], [o for _, o in dev], inputs_ready=True)
        else:
            alloc.bestfit_batches_dev([(c.data_ptr(), m.data_ptr(), wd.size, i.data_ptr(), dl.data_ptr(), t.data_ptr())
                                       for (c, m, i, dl, t), (wd, _) in zip(dev, batches)], s, inputs_ready=True)
    i, dl, t = ro.ptrs()
    alloc.bestfit_packed_prefix_dev(rw.data_ptr(), ro.R, i, dl, t, stream=s, rounds=True)
    new_fc, new_fm = installed(r_exp[3], D)
    pr_c, pr_m = cs.probe_rows(new_fc, new_fm)
    probe = km.pack(pr_c, pr_m)
    probe_outs = []
    for v in (SORTED, LUT):
        alloc.set_variant(v)
        p_out = pm.Out(torch, probe.size, D)
        pm.packed_multi(alloc, torch, [pm.words_dev(torch, probe)], [p_out], inputs_ready=True)
        probe_outs.append((v, p_out))
    q_c, q_m = rng.integers(0, 10, 3000).astype(np.int32), rng.integers(0, 500, 3000).astype(np.int32)
    qc, qm = km._dev(torch, q_c), km._dev(torch, q_m)
    q_idx = torch.full((3004,), -9, dtype=torch.int32, device="cuda")
    alloc.bestfit_dev(qc.data_ptr(), qm.data_ptr(), 3000, q_idx.data_ptr(), 0, 0, False, s, prefix_commit=True)
    torch.cuda.synchronize()
    for j, (packed, batches, dev) in enumerate(chain):
        for k, ((wd, exp), d) in enumerate(zip(batches, dev)):
            where = f"launch {j} ({'packed' if packed else 'int32'}), batch {k}"
            if packed:
                d[1].check(exp, where)
            else:
                _, _, ii, dd, tt = d
                got = ii.cpu().numpy()
                assert np.array_equal(got[:wd.size], exp[0]) and (got[wd.size:] == -9).all(), where
                assert np.array_equal(dd.cpu().numpy(), np.concatenate(exp[1:3])) and np.array_equal(tt.cpu().numpy(), exp[3]), where
    ro.check(r_exp[:4], "packed rounds")
    for v, p_out in probe_outs:
        p_out.check(pm.ref(new_fc, new_fm, probe), f"packed multi-batch launch after the rounds, variant {v}")
    assert np.array_equal(q_idx[:3000].cpu().numpy(), bestfit_np.prefix_commit(new_fc, new_fm, q_c, q_m)[0])
    assert pm.table_is(alloc, new_fc, new_fm)
