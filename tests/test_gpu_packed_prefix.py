"""Prefix-commit in the packed format: egpu_bestfit_batch[_dev] with EGPU_F_PACKED | EGPU_F_PREFIX_COMMIT.

The request array holds packed words (EGPU_PACK_REQUEST: core << 18 | mem; a word >= 2^25 is not a
request), req_mem is NULL and the indices are int8.  The call runs the packed twins of the CONTIG scans
(csrc/egpu_alloc.cu: kKernels<kScanSortedContig or kScanLutContig, kRowsPacked>[d_bucket(D)]), then prefix_cut_packed_kernel,
prefix_apply_packed_kernel and prefix_finalize_kernel.  Every case compares exactly with
oracle/bestfit_np.py or the C oracle on the requests the words stand for (not a request: (-1, -1)), and
most also with the int32 prefix-commit of egpu_bestfit_batch_dev on the same requests:

  1. the cell matrix: both packed scans at every D bucket, under AUTO, SORTED and LUT, with and without
     commit, ragged row counts, domain-edge words and tables;
  2. where the cut falls: the earliest row, the last row, a row of the R % 4 tail, on a CONTIG tile
     boundary and next to it, nowhere; a capped grid whose last tile holds only the tail; zero-demand
     rows that commit on a device of capacity 0;
  3. 16 Mi + 1 rows at D = 64 under both scans;
  4. argument checks on both entry points, and that a refused call launches and writes nothing;
  5. the host entry point with pageable and pinned buffers, demand sums NULL and not;
  6. ordering behind a pipelined chain of multi-batch launches, and what the launches after it see;
  7. rounds driven by the caller, re-submitting the deferred words.
"""
import ctypes as C
import os
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_context_sequences as cs  # noqa: E402  (probe rows)
import test_gpu_kernel_matrix as km  # noqa: E402  (cell tables, prefix_case, int32 prefix-commit)
import test_gpu_packed_multi as pm  # noqa: E402  (cell words, Out, guard bytes)

MEM_MAX = (1 << 18) - 1
ERR_INVALID, ERR_STATE = -1, -6
AUTO, GRID, SORTED, LUT = 0, 1, 2, 3
F_COMMIT, F_INPUTS_READY, F_PREFIX, F_PACKED = 1, 2, 4, 16
PACKED_CONTIG_TWINS = {"kScanSortedContig": "bestfit_sorted_packed_contig_kernel", "kScanLutContig": "bestfit_lut_packed_contig_kernel"}
CELLS = pm.CELLS


def test_packed_contig_twins_cover_every_cell():
    """the packed twins of the CONTIG scans in the kernel table, and a matrix cell for each of their buckets"""
    twins = pm.packed_twins("contig")
    assert twins == PACKED_CONTIG_TWINS and tuple(k.split("_")[1] for k in twins.values()) == pm.PACKED_FAMILIES
    want = {(f, b) for f in pm.PACKED_FAMILIES for b in range(len(km.BUCKET_TOPS))}
    assert {(pm.family(v, D), km.d_bucket(D)) for v, D in CELLS} == want


# ---- references and calls ------------------------------------------------------------------------------
def ref(fc, fm, words):
    from oracle import bestfit_np
    return bestfit_np.prefix_commit(np.asarray(fc, np.int32), np.asarray(fm, np.int32), *km.unpack(words))


def prefix_dev(alloc, torch, w, o, commit, flags=0):
    """the packed prefix-commit on device buffers; returns the launch count it added"""
    torch.cuda.synchronize()
    n0 = alloc.launch_count
    i, dl, t = o.ptrs()
    rc = alloc._lib.egpu_bestfit_batch_dev(alloc.handle, C.c_void_p(w.data_ptr()), None, o.R, C.c_void_p(i), C.c_void_p(dl),
                                           C.c_void_p(t), F_PACKED | F_PREFIX | (F_COMMIT if commit else 0) | flags,
                                           pm._s(torch))
    assert rc == 0
    torch.cuda.synchronize()
    return alloc.launch_count - n0


def installed(o_tab, D, ov=None):
    return o_tab[:D], o_tab[D:2 * D], np.zeros(D, np.int32) if ov is None else ov


def same_as_int32(alloc, torch, variant, fc, fm, words, o, where):
    """the int32 prefix-commit (committing) of the same requests gives the same outputs and table"""
    D = fc.size
    idx, delta, tab = km._prefix_dev(alloc, torch, variant, fc, fm, *km.unpack(words))
    assert np.array_equal(o.idx[:o.R].cpu().numpy().astype(np.int32), idx), f"{where}: indices differ from int32"
    assert np.array_equal(o.delta.cpu().numpy(), delta) and np.array_equal(o.tab.cpu().numpy(), tab), f"{where}: sums / table'"
    return installed(tab, D)


# ---- 1. the cell matrix ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", CELLS, ids=[f"{['auto', 'grid', 'sorted', 'lut'][v]}-D{D}" for v, D in CELLS])
def test_packed_prefix_cell(variant, D, alloc, egpu):
    import torch
    fam = pm.family(variant, D)
    for tname in km.cell_tables(D):
        for R in km.ROW_COUNTS:
            fc, fm, words = pm.cell_words(D, tname, R)
            exp = ref(fc, fm, words)
            w = pm.words_dev(torch, words)
            for commit in (False, True):
                where = f"{fam} scan, variant {variant}, D = {D}, table {tname}, R = {R}, commit {commit}"
                alloc.set_variant(variant)
                alloc.set_table(fc, fm)
                o = pm.Out(torch, R, D)
                n = prefix_dev(alloc, torch, w, o, commit)
                assert n == 4 + (fam == "lut"), f"{where}: launches"  # scan, cut, apply, finalize (+ lookup build)
                o.check(exp, where)
                want = installed(exp[3], D) if commit else (fc, fm, np.zeros(D, np.int32))
                assert pm.table_is(alloc, *want), f"{where}: installed table"
                if commit:
                    e_fc, e_fm, _ = same_as_int32(alloc, torch, 2 if fam == "sorted" else 3, fc, fm, words, o, where)
                    assert np.array_equal(e_fc, want[0]) and np.array_equal(e_fm, want[1]), where


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_prefix_keeps_oversub_flags(variant, alloc, egpu):
    """a committing oversubscribing snapshot sets flags; a packed prefix-commit after it keeps them, as
    the int32 prefix-commit does, and commits against the clamped table"""
    import torch
    from oracle import bestfit_np
    D = 5
    fc, fm = np.array([4, 10, 0, 100, 7], np.int32), np.array([50, 9, 0, MEM_MAX, 300], np.int32)
    rc, rm = np.array([4, 4, 10, 0, 99] * 3, np.int32), np.array([50, 1, 9, 0, 70_000] * 3, np.int32)
    _, _, _, o_tab = bestfit_np.snapshot(fc, fm, rc, rm)
    c_fc, c_fm, c_ov = km.committed(o_tab, D)
    assert c_ov.any()
    words = km.pack(np.arange(600) % 12, (np.arange(600) * 7) % 90)
    exp = ref(c_fc, c_fm, words)
    results = []
    for packed in (True, False):
        alloc.set_variant(variant)
        alloc.set_table(fc, fm)
        alloc.bestfit(rc, rm, commit=True)
        assert pm.table_is(alloc, c_fc, c_fm, c_ov)
        if packed:
            o = pm.Out(torch, words.size, D)
            prefix_dev(alloc, torch, pm.words_dev(torch, words), o, True)
            o.check(exp, "packed")
        else:
            c, m = (km._dev(torch, a) for a in km.unpack(words))
            idx = torch.full((words.size + 4,), -9, dtype=torch.int32, device="cuda")
            alloc.bestfit_dev(c.data_ptr(), m.data_ptr(), words.size, idx.data_ptr(), 0, 0, True,
                              torch.cuda.current_stream().cuda_stream, prefix_commit=True)
            torch.cuda.synchronize()
            assert np.array_equal(idx[:words.size].cpu().numpy(), exp[0])
        results.append(alloc.table())
        assert pm.table_is(alloc, exp[3][:D], exp[3][D:2 * D], c_ov), f"packed {packed}"
    assert all(np.array_equal(a, b) for a, b in zip(*results))


# ---- 2. where the cut falls -------------------------------------------------------------------------------
def cut_case(R, T, seed):
    """D = 2.  Device 0 = (0, fm0): rows (0, 1) choose it, and fm0 is the number of them before row T, so
    row T is its first deferred row (T = None: fm0 = all of them, nothing is deferred).  Device 1 = (0, 0):
    rows (0, 0) choose it and always commit.  One row in ten is not a request."""
    rng = np.random.default_rng(seed)
    kind = rng.choice(3, R, p=[0.7, 0.2, 0.1])
    if T is not None:
        kind[T] = 0
        if T == 1:
            kind[0] = 0
    words = np.where(kind == 0, 1, np.where(kind == 1, 0, 0xFFFFFFFF)).astype(np.uint32)
    fm0 = int((kind[:T] == 0).sum()) if T is not None else int((kind == 0).sum())
    return np.array([0, 0], np.int32), np.array([fm0, 0], np.int32), words


def tile_rows(R, threads, rpt, cap):
    """rows per CONTIG tile of launch_snapshot (every tile but the last)"""
    nvec = R >> 2
    want = min(max(1, -(-nvec // (threads * ((rpt + 3) // 4)))), cap)
    return 4 * -(-nvec // want), want


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_prefix_cut_positions(variant, alloc, egpu):
    import torch
    R = 3 * 8192 + 3  # R % 4 = 3; several tiles in both scans (2048 rows each in SORTED, 8192 in LUT)
    step, n_tiles = tile_rows(R, 256, 8 if variant == SORTED else 32, 1 << 30)
    assert n_tiles >= 3
    cuts = {"earliest": 1, "last row": R - 1, "tail row": R - 2, "tile boundary - 1": 2 * step - 1,
            "tile boundary": 2 * step, "tile boundary + 1": 2 * step + 1, "first tile boundary": step, "never": None}
    for what, T in cuts.items():
        fc, fm, words = cut_case(R, T, zlib.crc32(what.encode()))
        exp = ref(fc, fm, words)
        d0 = np.flatnonzero(exp[0] == -2)
        assert (d0[0] if d0.size else None) == T, what
        assert (exp[0][words == 0] == 1).all(), what  # zero-demand rows commit
        alloc.set_variant(variant)
        alloc.set_table(fc, fm)
        o = pm.Out(torch, R, 2)
        prefix_dev(alloc, torch, pm.words_dev(torch, words), o, True)
        o.check(exp, what)
        assert pm.table_is(alloc, *installed(exp[3], 2)), what
        same_as_int32(alloc, torch, variant, fc, fm, words, o, what)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_prefix_capped_grid_tail_tile(variant, egpu, monkeypatch):
    """EGPU_CTAS_PER_SM=2 and EGPU_ROWS_PER_THREAD=4 cap the grid at 2 * SMs tiles; R is chosen so that ceil(nvec / tiles) vectors per
    tile leave the last tile only the ragged tail, and the cut falls in that tail"""
    import torch
    S = torch.cuda.get_device_properties(0).multi_processor_count
    cap = 2 * S
    p = cap - 4
    nvec = (cap - 1) * p
    R = 4 * nvec + 3
    step, n_tiles = tile_rows(R, 256, 4, cap)
    assert n_tiles == cap and step == 4 * p and step * (cap - 1) == 4 * nvec
    monkeypatch.setenv("EGPU_CTAS_PER_SM", "2")
    monkeypatch.setenv("EGPU_ROWS_PER_THREAD", "4")
    alloc = egpu.BestFitAllocator(0)
    try:
        for what, T in {"tail row": R - 2, "last row": R - 1, "last full tile": R - 5}.items():
            fc, fm, words = cut_case(R, T, 31 + T)
            exp = ref(fc, fm, words)
            alloc.set_variant(variant)
            alloc.set_table(fc, fm)
            o = pm.Out(torch, R, 2)
            prefix_dev(alloc, torch, pm.words_dev(torch, words), o, True)
            o.check(exp, what)
            assert pm.table_is(alloc, *installed(exp[3], 2)), what
            same_as_int32(alloc, torch, variant, fc, fm, words, o, what)
    finally:
        alloc.close()


# ---- 3. size ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_packed_prefix_above_the_two_wave_threshold(alloc, oracle_c):
    import torch
    R, D = (16 << 20) + 1, 64
    fc, fm, rc, rm = km.prefix_case(R)
    words = km.pack(rc, rm)
    o_idx, o_dc, o_dm, o_tab = oracle_c.prefix_commit(fc, fm, *km.unpack(words))
    assert (o_idx[:R // 2] == -2).any() and (o_idx[R // 2:] >= 0).any() and (o_idx[R // 2:] == -2).any()
    w = pm.words_dev(torch, words)
    o = pm.Out(torch, R, D)
    for variant in (SORTED, LUT):
        o.reset()
        alloc.set_variant(variant)
        alloc.set_table(fc, fm)
        prefix_dev(alloc, torch, w, o, True)
        o.check((o_idx, o_dc, o_dm, o_tab), f"variant {variant}")
        assert pm.table_is(alloc, *installed(o_tab, D)), variant


# ---- 4. arguments ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_packed_prefix_arguments(alloc, egpu):
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
    PP = F_PACKED | F_PREFIX
    h_words = np.ascontiguousarray(words)
    h_idx = np.full(256, -9, np.int8)
    h_mem = np.zeros(200, np.int32)
    hw, hi, hm = h_words.ctypes.data, h_idx.ctypes.data, h_mem.ctypes.data

    def dev(core, mem, R, out, flags):
        return alloc._lib.egpu_bestfit_batch_dev(alloc.handle, C.c_void_p(core), C.c_void_p(mem), R, C.c_void_p(out), None, None,
                                                 flags, s)

    def host(core, mem, R, out, flags):
        return alloc._lib.egpu_bestfit_batch(alloc.handle, C.c_void_p(core), C.c_void_p(mem), R, C.c_void_p(out), None, None, flags)

    torch.cuda.synchronize()
    n0 = alloc.launch_count
    refused = {
        "dev: req_mem given with the flag": dev(wp, mp, 100, ip, PP),
        "dev: req_mem given with the flag, R = 0": dev(wp, mp, 0, ip, PP),
        "dev: the flag without prefix-commit": dev(wp, None, 100, ip, F_PACKED),
        "dev: the flag with commit, without prefix-commit": dev(wp, None, 100, ip, F_PACKED | F_COMMIT),
        "dev: misaligned words": dev(wp + 4, None, 100, ip, PP),
        "dev: misaligned indices": dev(wp, None, 100, ip + 1, PP),
        "dev: NULL words": dev(None, None, 100, ip, PP),
        "dev: NULL indices": dev(wp, None, 100, None, PP),
        "dev: packed words without the flag": dev(wp, None, 100, ip, F_PREFIX),
        "host: req_mem given with the flag": host(hw, hm, 100, hi, PP | F_COMMIT),
        "host: the flag without prefix-commit": host(hw, None, 100, hi, F_PACKED | F_COMMIT),
        "host: NULL words": host(None, None, 100, hi, PP),
        "host: NULL indices": host(hw, None, 100, None, PP),
        "host: packed words without the flag": host(hw, None, 100, hi, F_PREFIX | F_COMMIT),
    }
    for what, code in refused.items():
        assert code == ERR_INVALID, what
    alloc.set_variant(GRID)
    assert dev(wp, None, 100, ip, PP) == ERR_STATE
    assert host(hw, None, 100, hi, PP) == ERR_STATE
    alloc.set_variant(AUTO)
    torch.cuda.synchronize()
    assert alloc.launch_count == n0, "a refused call launched"
    assert bool((idx == -9).all()) and (h_idx == -9).all(), "a refused call wrote indices"
    assert pm.table_is(alloc, fc, fm)
    # a NULL req_mem with R = 0 and no flag was always fine: an empty int32 snapshot
    assert dev(mp, None, 0, i32.data_ptr(), 0) == 0
    torch.cuda.synchronize()
    assert alloc.launch_count == n0 + 1 and bool((i32 == -9).all())
    # EGPU_F_INPUTS_READY is accepted and changes nothing; R = 0 runs the whole pipeline
    exp = ref(fc, fm, words)
    o = pm.Out(torch, 200, D)
    assert prefix_dev(alloc, torch, w, o, False, F_INPUTS_READY) == 4
    o.check(exp, "inputs ready")
    e = pm.Out(torch, 0, D)
    assert prefix_dev(alloc, torch, w, e, True) == 4
    e.check(ref(fc, fm, words[:0]), "R = 0")
    assert pm.table_is(alloc, fc, fm)


# ---- 5. the host entry point ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_prefix_host(variant, alloc, egpu):
    rng = np.random.default_rng(500 + variant)
    D = 20
    fc = rng.integers(0, 101, D).astype(np.int32)
    fm = rng.integers(0, MEM_MAX + 1, D).astype(np.int32)
    R = 70_001
    words = km.pack(rng.integers(-1, 110, R), rng.integers(-1, 30_000, R))
    exp = ref(fc, fm, words)
    assert (exp[0] == -2).any() and (exp[0] >= 0).any()
    alloc.set_variant(variant)
    for commit in (False, True):
        alloc.set_table(fc, fm)
        idx, dc, dm = alloc.bestfit_packed_prefix(words, commit=commit)
        assert idx.dtype == np.int8 and np.array_equal(idx.astype(np.int32), exp[0]), commit
        assert np.array_equal(dc, exp[1]) and np.array_equal(dm, exp[2]), commit
        assert pm.table_is(alloc, *(installed(exp[3], D) if commit else (fc, fm))), commit
    # pinned buffers, demand sums NULL and not
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
                                               C.c_void_p(dm.ctypes.data if with_delta else None), F_PACKED | F_PREFIX | F_COMMIT)
            assert rc == 0
            assert np.array_equal(p_idx[:R].astype(np.int32), exp[0]) and (p_idx[R:] == -9).all(), with_delta
            if with_delta:
                assert np.array_equal(dc, exp[1]) and np.array_equal(dm, exp[2])
            assert pm.table_is(alloc, *installed(exp[3], D)), with_delta
    finally:
        alloc.host_free(p_words.ctypes.data)
        alloc.host_free(p_idx.ctypes.data)
    # the same requests through the int32 host prefix-commit
    alloc.set_table(fc, fm)
    idx32, dc32, dm32 = alloc.bestfit(*km.unpack(words), commit=True, prefix_commit=True)
    assert np.array_equal(idx32, exp[0]) and np.array_equal(dc32, exp[1]) and np.array_equal(dm32, exp[2])


# ---- 6. ordering ----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_prefix_after_pipelined_chain(variant, alloc, egpu):
    """12 pipelined multi-batch launches (packed and int32 in turn), then a committing packed prefix-commit
    on the same stream: the chain's outputs are exact, and a packed lookup multi-batch launch, an int32
    prefix-commit and table() all see the table it installed"""
    import torch
    from oracle import bestfit_np
    D = 24
    rng = np.random.default_rng(6000 + variant)
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
    pwords = km.pack(rng.integers(0, 30, 50_000), rng.integers(0, 900, 50_000))
    p_exp = ref(fc, fm, pwords)
    assert (p_exp[0] == -2).any()
    pw, po = pm.words_dev(torch, pwords), pm.Out(torch, pwords.size, D)
    torch.cuda.synchronize()  # every input is complete before the first launch
    for packed, batches, dev in chain:
        if packed:
            pm.packed_multi(alloc, torch, [w for w, _ in dev], [o for _, o in dev], inputs_ready=True)
        else:
            alloc.bestfit_batches_dev([(c.data_ptr(), m.data_ptr(), wd.size, i.data_ptr(), dl.data_ptr(), t.data_ptr())
                                       for (c, m, i, dl, t), (wd, _) in zip(dev, batches)], s, inputs_ready=True)
    i, dl, t = po.ptrs()
    alloc.bestfit_packed_prefix_dev(pw.data_ptr(), po.R, i, dl, t, commit=True, stream=s)
    new_fc, new_fm = p_exp[3][:D], p_exp[3][D:2 * D]
    # a packed lookup launch and an int32 prefix-commit after it, still on the same stream
    alloc.set_variant(LUT)
    pr_c, pr_m = cs.probe_rows(new_fc, new_fm)
    probe = km.pack(pr_c, pr_m)
    p_out = pm.Out(torch, probe.size, D)
    pm.packed_multi(alloc, torch, [pm.words_dev(torch, probe)], [p_out], inputs_ready=True)
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
    po.check(p_exp, "packed prefix-commit")
    p_out.check(pm.ref(new_fc, new_fm, probe), "packed lookup launch after the commit")
    assert np.array_equal(q_idx[:3000].cpu().numpy(), bestfit_np.prefix_commit(new_fc, new_fm, q_c, q_m)[0])
    assert pm.table_is(alloc, new_fc, new_fm)


# ---- 7. rounds by the caller -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_prefix_rounds_by_the_caller(variant, alloc, oracle_c):
    """re-submit the deferred words, in order, until none is left: after every round the indices and the
    table are the rounds reference's with that many rounds, and the table never goes negative"""
    rng = np.random.default_rng(700 + variant)
    D = 6
    fc = rng.integers(30, 101, D).astype(np.int32)
    fm = rng.integers(20_000, MEM_MAX + 1, D).astype(np.int32)
    R = 4001
    words = km.pack(rng.integers(0, 12, R), rng.integers(0, 3000, R))
    alloc.set_variant(variant)
    alloc.set_table(fc, fm)
    out = np.full(R, -2, np.int32)
    rows = np.arange(R)
    n = 0
    while rows.size:
        idx, _, _ = alloc.bestfit_packed_prefix(words[rows], commit=True)
        out[rows] = idx
        rows = rows[idx == -2]
        n += 1
        o_idx, _, _, o_fc, o_fm, o_rounds, o_left = oracle_c.rounds(fc, fm, *km.unpack(words), max_rounds=n)
        assert (o_rounds, o_left) == (n, rows.size), n
        assert np.array_equal(out, o_idx), f"round {n}"
        g_fc, g_fm, g_ov = alloc.table()
        assert np.array_equal(g_fc, o_fc) and np.array_equal(g_fm, o_fm) and not g_ov.any(), f"round {n}"
        assert (g_fc >= 0).all() and (g_fm >= 0).all()
        assert n <= R
    assert n >= 3
