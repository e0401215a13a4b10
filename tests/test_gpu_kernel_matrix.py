"""Every scan kernel the launch table can select, against a plain reference of the same operation.

The snapshot scans are one kernel per (family, D bucket): `kKernels<family, format>[d_bucket(D)]` in
csrc/egpu_alloc.cu (this file: the int32 tables, and kScanPacked's), 8 families x 4 buckets (D <= 8, 16, 32, 64).  This file drives each cell through the
entry point that selects it, at the D values on both sides of every bucket edge, and the grid-sizing
rules of the launchers at their thresholds:

  (a) the cell matrix: tables with ties, all-zero and all-full tables, devices at sorted positions 31,
      32 and 63, lookup tables whose overflow blocks are all in use; requests at the domain edges;
      ragged row counts around the 4-row vectors and the packed scan's 512-row warp chunks;
  (b) the multi-batch size rule around 512 Ki rows, whole waves and the `extra` CTAs of the first batches;
  (c) the multi-batch epilogue switching from the ticket-in-the-top-bits path to the general one
      (>= 2^15 tiles in a batch);
  (d) the two-wave cap of single-batch launches at 16 Mi rows, and prefix-commit, which opts out of it;
  (e) the bound on rows per thread that keeps lane-private sums exact, on both sides.

References: oracle/bestfit_np.py (dense int64 grid) up to about 2^20 rows, the C oracle up to about
32 Mi rows, and above that `torch_snapshot` below, which restates the spec with int64 torch ops on the
GPU.  None of them uses the packed compare word or the lookup tables of the kernels.
"""
import functools
import itertools
import os
import re
import zlib

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "elastic-gpu-agent_b200", "csrc")

INT32_MIN, INT32_MAX = -(2**31), 2**31 - 1
MEM_MAX = (1 << 18) - 1
ERR_INVALID = -1

# ---- the kernel table ---------------------------------------------------------------------------
# Scan families, in the order of enum ScanFamily (csrc/egpu_ctx.h), and the D buckets of d_bucket().
FAMILIES = ("sorted", "sorted_contig", "grid", "lut", "lut_contig", "sorted_multi", "lut_multi", "packed")
ENUM_NAMES = ("kScanSorted", "kScanSortedContig", "kScanGrid", "kScanLut", "kScanLutContig", "kScanSortedMulti",
              "kScanLutMulti", "kScanPacked")
BUCKET_TOPS = (8, 16, 32, 64)

# Every (family, bucket) cell, written out: a family or a bucket added to the launch table without a
# matrix entry here fails test_matrix_covers_every_kernel_cell.
EXPECTED_CELLS = {
    ("sorted", 0), ("sorted", 1), ("sorted", 2), ("sorted", 3),
    ("sorted_contig", 0), ("sorted_contig", 1), ("sorted_contig", 2), ("sorted_contig", 3),
    ("grid", 0), ("grid", 1), ("grid", 2), ("grid", 3),
    ("lut", 0), ("lut", 1), ("lut", 2), ("lut", 3),
    ("lut_contig", 0), ("lut_contig", 1), ("lut_contig", 2), ("lut_contig", 3),
    ("sorted_multi", 0), ("sorted_multi", 1), ("sorted_multi", 2), ("sorted_multi", 3),
    ("lut_multi", 0), ("lut_multi", 1), ("lut_multi", 2), ("lut_multi", 3),
    ("packed", 0), ("packed", 1), ("packed", 2), ("packed", 3),
}

# entry point of the matrix -> the family it selects (variant 1 = grid, 2 = sorted, 3 = lookup)
ENTRIES = {
    "bestfit": "sorted",             # variant 2, host buffers, commit
    "bestfit_dev": "sorted",         # variant 2, device buffers, delta + table_out, commit
    "query": "sorted",               # egpu_bestfit_query always runs the sorted scan
    "grid_dev": "grid",              # variant 1
    "lut_dev": "lut",                # variant 3
    "prefix_sorted": "sorted_contig",  # prefix_commit=True, variant 2
    "rounds_sorted": "sorted_contig",  # bestfit_rounds, variant 2
    "prefix_lut": "lut_contig",
    "rounds_lut": "lut_contig",
    "multi_sorted": "sorted_multi",  # bestfit_batches_dev, variant 2
    "multi_lut": "lut_multi",        # variant 3
    "packed": "packed",              # bestfit_packed
}


def d_bucket(D):
    return next(b for b, top in enumerate(BUCKET_TOPS) if D <= top)


D_EDGES = (1, 8, 9, 16, 17, 32, 33, 64)
_rng_d = np.random.default_rng(20261015)
D_RANDOM = tuple(int(_rng_d.integers(lo, hi + 1)) for lo, hi in ((2, 7), (10, 15), (18, 31), (34, 63)))
D_ALL = D_EDGES + D_RANDOM
ROW_COUNTS = (0, 1, 3, 4, 5, 511, 512, 513, 40_003)
MATRIX = [(entry, D) for entry in ENTRIES for D in D_ALL]

CORE_EDGES = (INT32_MIN, -1, 0, 1, 99, 100, 101, 127, 128, INT32_MAX)
MEM_EDGES = (INT32_MIN, -1, 0, 63, 64, 65, MEM_MAX, MEM_MAX + 1, MEM_MAX + 2, INT32_MAX)
ROUNDS_CAP = 4  # the numpy rounds reference re-scores every deferred row per round


# ---- inputs of the cell matrix ----------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def cell_tables(D):
    """name -> (free_core, free_mem) for D devices"""
    rng = np.random.default_rng(7000 + D)
    out = {}
    # duplicated (fc, fm) pairs: every pair is held by one or more devices; ties go to the lowest d
    k = max(1, (D + 1) // 2)
    pc, pm = rng.integers(0, 101, k), rng.integers(0, MEM_MAX + 1, k)
    pick = np.concatenate([np.arange(k), rng.integers(0, k, D - k)])
    rng.shuffle(pick)
    out["dups"] = (pc[pick], pm[pick])
    out["zeros"] = (np.zeros(D), np.zeros(D))
    out["full"] = (np.full(D, 100), np.full(D, MEM_MAX))
    # distinct pairs in scattered device order: sorted positions 0..D-1 (31, 32 and 63 where D allows, which
    # the scans store mod 32) land on unrelated device numbers; every device gets exact-fit requests below
    out["spread"] = (rng.integers(0, 101, D), rng.choice(MEM_MAX + 1, D, replace=False))
    if D >= 2:
        # D // 2 memory buckets of 64 MiB (32 at D = 64, the most the lookup scan's overflow blocks hold),
        # two distinct free_mem values in each, the first and the last bucket included
        nb = D // 2
        inner = rng.choice(np.arange(1, 4095), max(0, nb - 2), replace=False)
        buckets = [0] + ([4095] if nb >= 2 else []) + [int(b) for b in inner]
        fm = []
        for b in buckets:
            if b == 0:
                fm += [0, 1]
            elif b == 4095:
                fm += [MEM_MAX - 1, MEM_MAX]
            else:
                fm += [int(v) for v in 64 * b + rng.choice(64, 2, replace=False)]
        fm += fm[:D - len(fm)]  # odd D: one value twice
        out["buckets"] = (rng.integers(0, 101, D), rng.permutation(np.array(fm)))
    return {n: (np.asarray(c, np.int32), np.asarray(m, np.int32)) for n, (c, m) in out.items()}


def edge_pairs(fc, fm):
    """the cross product of the edge values: fixed ones, and every device's own capacity -1 / 0 / +1"""
    cores = np.unique(np.concatenate([np.array(CORE_EDGES, np.int64), fc - 1, fc, fc + 1]))
    mems = np.unique(np.concatenate([np.array(MEM_EDGES, np.int64), fm - 1, fm, fm + 1]))
    cc, mm = np.meshgrid(cores, mems, indexing="ij")
    return np.stack([cc.ravel(), mm.ravel()], axis=1)


@functools.lru_cache(maxsize=None)
def cell_case(D, tname, R):
    """(free_core, free_mem, req_core, req_mem): the cross product scattered through seeded random rows;
    every pair appears when R is at least the product's size, a random subset of it otherwise"""
    fc, fm = cell_tables(D)[tname]
    pairs = edge_pairs(fc.astype(np.int64), fm.astype(np.int64))
    rng = np.random.default_rng([D, R, zlib.crc32(tname.encode())])
    pairs = pairs[rng.permutation(len(pairs))]
    if R > len(pairs):
        pairs = np.concatenate([pairs, pairs[rng.integers(0, len(pairs), R - len(pairs))]])
        pairs = pairs[rng.permutation(R)]
    rows = pairs[:R]
    return fc, fm, rows[:, 0].astype(np.int32), rows[:, 1].astype(np.int32)


# packed words the int32 arrays cannot express: core 101..127 (well-formed, infeasible everywhere),
# anything >= 2^25 (not a request) and the all-ones word
def packed_words(rc, rm, R, D):
    words = pack(rc, rm)
    if R:
        rng = np.random.default_rng(91 + D + R)
        n = max(1, R // 16)
        at = rng.integers(0, R, (3, n))
        words[at[0]] = (rng.integers(101, 128, n).astype(np.uint32) << 18) | rng.integers(0, MEM_MAX + 1, n).astype(np.uint32)
        words[at[1]] = rng.integers(1 << 25, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
        words[at[2]] = 0xFFFFFFFF
    return words


def pack(rc, rm):
    c = np.asarray(rc, np.int64)
    m = np.asarray(rm, np.int64)
    ok = (c >= 0) & (c <= 127) & (m >= 0) & (m <= MEM_MAX)
    return np.where(ok, (c << 18) | m, 0xFFFFFFFF).astype(np.uint32)


def unpack(words):
    """packed words -> the int32 request they stand for (not a request: -1, -1)"""
    w = np.asarray(words, np.int64)
    ok = w < (1 << 25)
    return np.where(ok, w >> 18, -1).astype(np.int32), np.where(ok, w & MEM_MAX, -1).astype(np.int32)


# ---- references ---------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def ref_snapshot(D, tname, R):
    from oracle import bestfit_np
    fc, fm, rc, rm = cell_case(D, tname, R)
    return bestfit_np.snapshot(fc, fm, rc, rm)


@functools.lru_cache(maxsize=None)
def ref_packed(D, tname, R):
    from oracle import bestfit_np
    fc, fm, rc, rm = cell_case(D, tname, R)
    words = packed_words(rc, rm, R, D)
    return (words,) + bestfit_np.snapshot(fc, fm, *unpack(words))


@functools.lru_cache(maxsize=None)
def ref_prefix(D, tname, R):
    from oracle import bestfit_np
    return bestfit_np.prefix_commit(*cell_case(D, tname, R))


@functools.lru_cache(maxsize=None)
def ref_rounds(D, tname, R):
    from oracle import bestfit_np
    return bestfit_np.rounds(*cell_case(D, tname, R), max_rounds=ROUNDS_CAP)


def torch_snapshot(free_core, free_mem, c, m, device=None):
    """Spec 2.4 with plain int64 torch ops, chunked over the rows (for batches too large for the host
    references).  Row r is feasible on device d iff 0 <= c <= fc[d] and 0 <= m <= fm[d]; it picks the
    lexicographic minimum of (fc[d] - c, fm[d] - m, d), as one int64 key.  Returns idx int32[R],
    delta int64[2D] and table' int32[3D] (int32 saturation, oversubscription flag)."""
    import torch
    device = device or c.device
    fc = torch.as_tensor(np.asarray(free_core, np.int64), device=device)
    fm = torch.as_tensor(np.asarray(free_mem, np.int64), device=device)
    D = fc.numel()
    dev = torch.arange(D, dtype=torch.int64, device=device)
    none = torch.iinfo(torch.int64).max
    R = c.numel()
    idx = torch.empty(R, dtype=torch.int32, device=device)
    dc = torch.zeros(D, dtype=torch.int64, device=device)
    dm = torch.zeros(D, dtype=torch.int64, device=device)
    step = max(1, (1 << 23) // D)
    for s in range(0, R, step):
        cc = c[s:s + step].to(torch.int64)
        mm = m[s:s + step].to(torch.int64)
        lc = fc[None, :] - cc[:, None]
        lm = fm[None, :] - mm[:, None]
        ok = (cc >= 0)[:, None] & (mm >= 0)[:, None] & (lc >= 0) & (lm >= 0)
        key = torch.where(ok, (lc << 40) | (lm << 8) | dev[None, :], none)
        kmin = key.min(dim=1).values
        pick = torch.where(kmin == none, -1, kmin & 255)
        idx[s:s + step] = pick.to(torch.int32)
        hit = pick >= 0
        dc.index_add_(0, pick[hit], cc[hit])
        dm.index_add_(0, pick[hit], mm[hit])
    left_c, left_m = fc - dc, fm - dm
    over = ((left_c < 0) | (left_m < 0)).to(torch.int64)
    tab = torch.cat([left_c.clamp(INT32_MIN, INT32_MAX), left_m.clamp(INT32_MIN, INT32_MAX), over]).to(torch.int32)
    return idx, torch.cat([dc, dm]), tab


def committed(tab, D):
    """the table a committing snapshot installs: table' clamped to 0, oversubscription as flagged"""
    return np.maximum(tab[:D], 0), np.maximum(tab[D:2 * D], 0), tab[2 * D:]


# ---- tests that need no GPU -------------------------------------------------------------------------
def test_matrix_covers_every_kernel_cell():
    src_ctx = open(os.path.join(CSRC, "egpu_ctx.h")).read()
    enum = re.search(r"enum ScanFamily \{(.*?)\};", src_ctx, re.S).group(1)
    names = [n.strip() for n in enum.split(",") if n.strip()]
    assert names[-1] == "kScanFamilies"
    assert tuple(names[:-1]) == ENUM_NAMES
    src = open(os.path.join(CSRC, "egpu_alloc.cu")).read()
    rule = re.search(r"int d_bucket\(int D\) \{ return D <= (\d+) \? 0 : D <= (\d+) \? 1 : D <= (\d+) \? 2 : 3; \}", src)
    assert rule and tuple(int(x) for x in rule.groups()) + (64,) == BUCKET_TOPS
    assert EXPECTED_CELLS == set(itertools.product(FAMILIES, range(len(BUCKET_TOPS))))
    assert {(ENTRIES[e], d_bucket(D)) for e, D in MATRIX} == EXPECTED_CELLS
    # both edges of every bucket, and one D inside each
    for b, top in enumerate(BUCKET_TOPS):
        lo = 1 if b == 0 else BUCKET_TOPS[b - 1] + 1
        assert lo in D_ALL and top in D_ALL and any(lo < D < top for D in D_RANDOM)


def test_cell_inputs_reach_the_edges():
    for D in D_ALL:
        for tname, (fc, fm) in cell_tables(D).items():
            assert (fc >= 0).all() and (fc <= 100).all() and (fm >= 0).all() and (fm <= MEM_MAX).all()
            _, _, rc, rm = cell_case(D, tname, ROW_COUNTS[-1])
            got = set(zip(rc.tolist(), rm.tolist()))
            assert got == set(map(tuple, edge_pairs(fc.astype(np.int64), fm.astype(np.int64)).tolist()))
        if D >= 2:
            fm = cell_tables(D)["buckets"][1]
            blocks = np.unique(fm >> 6)
            assert len(blocks) == D // 2 and all((fm >> 6 == b).sum() >= 2 for b in blocks)
            assert {0, 1}.issubset(fm.tolist()) and (D < 4 or {MEM_MAX - 1, MEM_MAX}.issubset(fm.tolist()))
    assert len(np.unique(cell_tables(64)["buckets"][1] >> 6)) == 32
    fc, fm = cell_tables(64)["dups"]
    assert len(set(zip(fc.tolist(), fm.tolist()))) < 64


@pytest.mark.parametrize("D", [1, 9, 33, 64])
def test_torch_reference_matches_numpy_oracle(D):
    """the chunked torch reference of the large tests, on the CPU, against oracle/bestfit_np.py"""
    import torch
    for tname in cell_tables(D):
        fc, fm, rc, rm = cell_case(D, tname, ROW_COUNTS[-1])
        idx, delta, tab = torch_snapshot(fc, fm, torch.from_numpy(rc), torch.from_numpy(rm), "cpu")
        o_idx, o_dc, o_dm, o_tab = ref_snapshot(D, tname, ROW_COUNTS[-1])
        assert np.array_equal(idx.numpy(), o_idx)
        assert np.array_equal(delta.numpy(), np.concatenate([o_dc, o_dm]))
        assert np.array_equal(tab.numpy(), o_tab)
    big_c = torch.tensor([100, 0, 1, 100, 100], dtype=torch.int32)  # saturation of table' at int32
    big_m = torch.tensor([MEM_MAX] * 5, dtype=torch.int32)
    _, delta, tab = torch_snapshot([100], [MEM_MAX], big_c.repeat(9000), big_m.repeat(9000), "cpu")
    assert delta.tolist() == [301 * 9000, 5 * MEM_MAX * 9000]
    assert tab.tolist() == [100 - 301 * 9000, INT32_MIN, 1]


# ---- (a) the cell matrix -------------------------------------------------------------------------
def _dev(torch, a, pad=4, fill=None):
    """device copy of a, with `pad` more elements (a non-null, 16-byte aligned array even when a is empty)"""
    t = torch.full((a.size + pad,), fill if fill is not None else 0, dtype=torch.from_numpy(a[:0]).dtype, device="cuda")
    if a.size:
        t[:a.size] = torch.from_numpy(a).cuda()
    return t


def _snapshot_dev(alloc, torch, variant, fc, fm, rc, rm):
    R, D = rc.size, fc.size
    alloc.set_variant(variant)
    alloc.set_table(fc, fm)
    c, m = _dev(torch, rc), _dev(torch, rm)
    idx = torch.full((R + 4,), -9, dtype=torch.int32, device="cuda")
    delta = torch.full((2 * D,), -1, dtype=torch.int64, device="cuda")
    tab = torch.full((3 * D,), -7, dtype=torch.int32, device="cuda")
    alloc.bestfit_dev(c.data_ptr(), m.data_ptr(), R, idx.data_ptr(), delta.data_ptr(), tab.data_ptr(), True,
                      torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    idx = idx.cpu().numpy()
    assert (idx[R:] == -9).all()
    return idx[:R], delta.cpu().numpy(), tab.cpu().numpy()


def _check_committed(alloc, exp_tab, D):
    e_fc, e_fm, e_ov = exp_tab
    fc, fm, ov = alloc.table()
    assert np.array_equal(fc, e_fc) and np.array_equal(fm, e_fm) and np.array_equal(ov, e_ov)


def _run_cell(entry, D, tname, R, alloc, egpu, torch):
    fc, fm, rc, rm = cell_case(D, tname, R)
    last = R == ROW_COUNTS[-1]
    empty = np.zeros(0, np.int32)
    if entry in ("bestfit", "bestfit_dev", "grid_dev", "lut_dev", "query"):
        o_idx, o_dc, o_dm, o_tab = ref_snapshot(D, tname, R)
        if entry == "query":
            assert np.array_equal(alloc.query(fc, fm, rc, rm), o_idx)
            return
        variant = {"bestfit": 2, "bestfit_dev": 2, "grid_dev": 1, "lut_dev": 3}[entry]
        if entry == "bestfit":
            alloc.set_variant(variant)
            alloc.set_table(fc, fm)
            idx, dc, dm = alloc.bestfit(rc, rm, commit=True)
            assert np.array_equal(idx, o_idx) and np.array_equal(dc, o_dc) and np.array_equal(dm, o_dm)
        else:
            idx, delta, tab = _snapshot_dev(alloc, torch, variant, fc, fm, rc, rm)
            assert np.array_equal(idx, o_idx)
            assert np.array_equal(delta, np.concatenate([o_dc, o_dm]))
            assert np.array_equal(tab, o_tab)
        _check_committed(alloc, committed(o_tab, D), D)
        if last:  # the oversubscription flag is sticky: an empty committing batch keeps it
            alloc.bestfit(empty, empty, commit=True)
            _check_committed(alloc, committed(o_tab, D), D)
    elif entry in ("prefix_sorted", "prefix_lut"):
        o_idx, o_dc, o_dm, o_tab = ref_prefix(D, tname, R)
        idx, delta, tab = _prefix_dev(alloc, torch, 2 if entry == "prefix_sorted" else 3, fc, fm, rc, rm)
        assert np.array_equal(idx, o_idx)
        assert np.array_equal(delta, np.concatenate([o_dc, o_dm]))
        assert np.array_equal(tab, o_tab)
        _check_committed(alloc, (o_tab[:D], o_tab[D:2 * D], np.zeros(D, np.int32)), D)
    elif entry in ("rounds_sorted", "rounds_lut"):
        o_idx, o_dc, o_dm, o_fc, o_fm, o_rounds, o_left = ref_rounds(D, tname, R)
        alloc.set_variant(2 if entry == "rounds_sorted" else 3)
        alloc.set_table(fc, fm)
        idx, dc, dm, rounds, left = alloc.bestfit_rounds(rc, rm, ROUNDS_CAP)
        assert (rounds, left) == (o_rounds, o_left)
        assert np.array_equal(idx, o_idx) and np.array_equal(dc, o_dc) and np.array_equal(dm, o_dm)
        _check_committed(alloc, (o_fc, o_fm, np.zeros(D, np.int32)), D)
    elif entry in ("multi_sorted", "multi_lut"):
        o_idx, o_dc, o_dm, o_tab = ref_snapshot(D, tname, R)
        alloc.set_variant(2 if entry == "multi_sorted" else 3)
        alloc.set_table(fc, fm)
        # two batches: the rows, and the same rows reversed (same sums, reversed indices)
        keep, tup = [], []
        for c_h, m_h in ((rc, rm), (rc[::-1].copy(), rm[::-1].copy())):
            t = (_dev(torch, c_h), _dev(torch, m_h), torch.full((R + 4,), -9, dtype=torch.int32, device="cuda"),
                 torch.full((2 * D,), -1, dtype=torch.int64, device="cuda"),
                 torch.full((3 * D,), -7, dtype=torch.int32, device="cuda"))
            keep.append(t)
            tup.append((t[0].data_ptr(), t[1].data_ptr(), R, t[2].data_ptr(), t[3].data_ptr(), t[4].data_ptr()))
        alloc.bestfit_batches_dev(tup, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        for k, (c, m, idx, delta, tab) in enumerate(keep):
            idx = idx.cpu().numpy()
            assert np.array_equal(idx[:R], o_idx if k == 0 else o_idx[::-1]), k
            assert (idx[R:] == -9).all()
            assert np.array_equal(delta.cpu().numpy(), np.concatenate([o_dc, o_dm]))
            assert np.array_equal(tab.cpu().numpy(), o_tab)
        _check_committed(alloc, (fc, fm, np.zeros(D, np.int32)), D)  # a multi-batch launch never commits
    elif entry == "packed":
        words, o_idx, o_dc, o_dm, o_tab = ref_packed(D, tname, R)
        alloc.set_table(fc, fm)
        idx, dc, dm = alloc.bestfit_packed(words, commit=True)
        assert np.array_equal(idx.astype(np.int32), o_idx) and np.array_equal(dc, o_dc) and np.array_equal(dm, o_dm)
        _check_committed(alloc, committed(o_tab, D), D)
        if last:
            alloc.bestfit_packed(np.zeros(0, np.uint32), commit=True)
            _check_committed(alloc, committed(o_tab, D), D)
    else:
        raise AssertionError(entry)


def _prefix_dev(alloc, torch, variant, fc, fm, rc, rm):
    R, D = rc.size, fc.size
    alloc.set_variant(variant)
    alloc.set_table(fc, fm)
    c, m = _dev(torch, rc), _dev(torch, rm)
    idx = torch.full((R + 4,), -9, dtype=torch.int32, device="cuda")
    delta = torch.full((2 * D,), -1, dtype=torch.int64, device="cuda")
    tab = torch.full((3 * D,), -7, dtype=torch.int32, device="cuda")
    alloc.bestfit_dev(c.data_ptr(), m.data_ptr(), R, idx.data_ptr(), delta.data_ptr(), tab.data_ptr(), True,
                      torch.cuda.current_stream().cuda_stream, prefix_commit=True)
    torch.cuda.synchronize()
    idx = idx.cpu().numpy()
    assert (idx[R:] == -9).all()
    return idx[:R], delta.cpu().numpy(), tab.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("entry,D", MATRIX, ids=[f"{e}-D{D}" for e, D in MATRIX])
def test_kernel_cell(entry, D, alloc, egpu):
    import torch
    for tname in cell_tables(D):
        for R in ROW_COUNTS:
            try:
                _run_cell(entry, D, tname, R, alloc, egpu, torch)
            except AssertionError as ex:
                raise AssertionError(f"{entry} ({ENTRIES[entry]}), D = {D}, table {tname}, R = {R}: {ex}") from ex


# ---- (b) the multi-batch size rule -----------------------------------------------------------------
# Below 512 Ki rows (the largest batch of the launch decides) the grid is at most one wave with
# EGPU_MULTI_RPT rows per thread; from 512 Ki rows on, 20 rows per thread (28 in the lookup scan),
# rounded up to whole waves, the first `extra` = (CTAs % K) batches one tile more.  K = 5 and 7 batches
# of 1 Mi rows leave extra > 0 at every D bucket of both scans on an H100.
MULTI_SHAPES = {
    "524287": [524_287],
    "524288": [524_288],
    "524289": [524_289],
    "mixed": [1_000_003, 0, 5, 70_003],
    "5x1Mi": [1 << 20] * 5,
    "7x1Mi": [1 << 20] * 7,
    "64x512Ki": [512 << 10] * 64,
}


def _batch_buffers(torch, alloc, rows, D, dist, seed, s):
    """device requests (synth_requests_dev, rows after each other in one stream of the distribution),
    index arrays with 4 guard words, sentinel-filled delta / table' per batch"""
    out, first = [], 0
    for R in rows:
        c = torch.empty(R + 4, dtype=torch.int32, device="cuda")
        m = torch.empty(R + 4, dtype=torch.int32, device="cuda")
        alloc.synth_requests_dev(dist, seed, first, R, c.data_ptr(), m.data_ptr(), s)
        first += R
        out.append((c, m, torch.empty(R + 4, dtype=torch.int32, device="cuda"),
                    torch.empty(2 * D, dtype=torch.int64, device="cuda"), torch.empty(3 * D, dtype=torch.int32, device="cuda")))
    return out


def _reset(bufs):
    for _, _, idx, delta, tab in bufs:
        idx.fill_(-9)
        delta.fill_(-1)
        tab.fill_(-7)


def _tuples(bufs, rows):
    return [(c.data_ptr(), m.data_ptr(), R, i.data_ptr(), dl.data_ptr(), t.data_ptr()) for (c, m, i, dl, t), R in zip(bufs, rows)]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(MULTI_SHAPES))
@pytest.mark.parametrize("D", [8, 17, 64])
def test_multi_batch_size_rule(D, shape, alloc, oracle_c):
    import torch
    rows = MULTI_SHAPES[shape]
    rng = np.random.default_rng(500 + D)
    fc = rng.integers(0, 101, D).astype(np.int32)
    fm = rng.integers(0, MEM_MAX + 1, D).astype(np.int32)
    s = torch.cuda.current_stream().cuda_stream
    bufs = _batch_buffers(torch, alloc, rows, D, 3, 17 + D, s)
    torch.cuda.synchronize()
    refs = [oracle_c.snapshot(fc, fm, c[:R].cpu().numpy(), m[:R].cpu().numpy(), oracle_c.max_threads())
            for (c, m, _, _, _), R in zip(bufs, rows)]
    alloc.set_table(fc, fm)
    for variant in (2, 3):
        _reset(bufs)
        alloc.set_variant(variant)
        alloc.bestfit_batches_dev(_tuples(bufs, rows), s)
        torch.cuda.synchronize()
        for k, ((_, _, idx, delta, tab), R, (o_idx, o_dc, o_dm, o_tab)) in enumerate(zip(bufs, rows, refs)):
            got = idx.cpu().numpy()
            where = f"variant {variant}, batch {k} of {len(rows)} ({R} rows)"
            assert np.array_equal(got[:R], o_idx), where
            assert (got[R:] == -9).all(), where
            assert np.array_equal(delta.cpu().numpy(), np.concatenate([o_dc, o_dm])), where
            assert np.array_equal(tab.cpu().numpy(), o_tab), where


# ---- (c) a multi-batch batch with >= 2^15 tiles: the general ticket path of the epilogue ----------------
@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 2])
def test_multi_batch_general_ticket_path(K, alloc, egpu):
    """The plain epilogue carries its arrival ticket in bits 49..63 of every running sum, which counts
    to 2^15 - 1; a batch with more tiles takes the general path.  90 M rows at D = 64 are at least
    35 156 tiles of 128 threads x 20 rows, whatever the occupancy (wave rounding only adds tiles)."""
    import torch
    w = egpu.synth.workload("cfg4")
    D = 64
    rows = [90_000_001] if K == 1 else [70_003, 90_000_001]
    s = torch.cuda.current_stream().cuda_stream
    bufs = _batch_buffers(torch, alloc, rows, D, 4, 23, s)
    _reset(bufs)
    alloc.set_variant(2)
    alloc.set_table(w["free_core"], w["free_mem"])
    alloc.bestfit_batches_dev(_tuples(bufs, rows), s)
    torch.cuda.synchronize()
    for k, ((c, m, idx, delta, tab), R) in enumerate(zip(bufs, rows)):
        e_idx, e_delta, e_tab = torch_snapshot(w["free_core"], w["free_mem"], c[:R], m[:R])
        assert torch.equal(idx[:R], e_idx), k
        assert bool((idx[R:] == -9).all()), k
        assert torch.equal(delta, e_delta), (k, delta.tolist()[:4])
        assert torch.equal(tab, e_tab), k
        del e_idx


# ---- (d) the two-wave cap of single-batch launches ------------------------------------------------------
@pytest.mark.gpu
def test_single_batch_two_wave_cap(alloc, oracle_c, egpu):
    """From 16 Mi rows on a single-batch grid may hold two waves of CTAs; exact outputs on both sides,
    for the sorted and the lookup scan, lone (8 / 32 rows per thread) and pipelined (8 / 48)."""
    import torch
    w = egpu.synth.workload("cfg4")
    fc, fm, D = w["free_core"], w["free_mem"], 64
    s = torch.cuda.current_stream().cuda_stream
    r_max = (16 << 20) + 3
    c = torch.empty(r_max + 1, dtype=torch.int32, device="cuda")
    m = torch.empty(r_max + 1, dtype=torch.int32, device="cuda")
    alloc.synth_requests_dev(4, 31, 0, r_max, c.data_ptr(), m.data_ptr(), s)
    idx = torch.empty(r_max + 4, dtype=torch.int32, device="cuda")
    delta = torch.empty(2 * D, dtype=torch.int64, device="cuda")
    tab = torch.empty(3 * D, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    rc, rm = c[:r_max].cpu().numpy(), m[:r_max].cpu().numpy()
    alloc.set_table(fc, fm)
    for R in ((16 << 20) - 4, 16 << 20, r_max):
        o_idx, o_dc, o_dm, o_tab = oracle_c.snapshot(fc, fm, rc[:R], rm[:R], oracle_c.max_threads())
        for variant in (2, 3):
            alloc.set_variant(variant)
            for ready in (False, True):
                idx.fill_(-9)
                delta.fill_(-1)
                tab.fill_(-7)
                alloc.bestfit_dev(c.data_ptr(), m.data_ptr(), R, idx.data_ptr(), delta.data_ptr(), tab.data_ptr(), False, s,
                                  inputs_ready=ready)
                torch.cuda.synchronize()
                got = idx.cpu().numpy()
                where = (R, variant, ready)
                assert np.array_equal(got[:R], o_idx) and (got[R:] == -9).all(), where
                assert np.array_equal(delta.cpu().numpy(), np.concatenate([o_dc, o_dm])), where
                assert np.array_equal(tab.cpu().numpy(), o_tab), where


def prefix_case(R):
    """D = 64; requests whose per-device cuts fall from the first rows to about 70 % of the batch.
    Half the devices have no core left, half all of it; memory differs on every device.  Rows (0, 1..3)
    fill the memory of the fc = 0 device with the least of it, rows (1, 1) the core of the fc = 100
    device with the least memory, and 2000 rows of anything cut the others early."""
    rng = np.random.default_rng(77)
    D = 64
    fc = np.where(np.arange(D) % 2 == 0, 0, 100).astype(np.int32)[rng.permutation(D)]
    fm = rng.choice(np.arange(1 << 17, MEM_MAX + 1), D, replace=False).astype(np.int32)
    rc = np.zeros(R, np.int32)
    rm = np.zeros(R, np.int32)
    u = rng.random(R)
    a = u < 0.6 * (1 << 17) / R
    b = (u >= 0.5) & (u < 0.5 + 150 / R)
    o = (u >= 0.9) & (u < 0.9 + 2000 / R)
    rm[a] = rng.integers(1, 4, a.sum())
    rc[b], rm[b] = 1, 1
    rc[o], rm[o] = rng.integers(-1, 102, o.sum()), rng.integers(-1, MEM_MAX + 2, o.sum())
    return fc, fm, rc, rm


@pytest.mark.gpu
def test_prefix_commit_above_the_two_wave_threshold(alloc, oracle_c):
    """prefix-commit (CONTIG tiles, one wave) is exempt from the two-wave cap: 16 Mi + 1 rows"""
    import torch
    R, D = (16 << 20) + 1, 64
    fc, fm, rc, rm = prefix_case(R)
    o_idx, o_dc, o_dm, o_tab = oracle_c.prefix_commit(fc, fm, rc, rm)
    assert (o_idx[:R // 2] == -2).any() and (o_idx[R // 2:] >= 0).any() and (o_idx[R // 2:] == -2).any()
    s = torch.cuda.current_stream().cuda_stream
    c, m = torch.from_numpy(rc).cuda(), torch.from_numpy(rm).cuda()
    idx = torch.empty(R + 3, dtype=torch.int32, device="cuda")
    delta = torch.empty(2 * D, dtype=torch.int64, device="cuda")
    tab = torch.empty(3 * D, dtype=torch.int32, device="cuda")
    for variant in (2, 3):
        idx.fill_(-9)
        delta.fill_(-1)
        tab.fill_(-7)
        alloc.set_variant(variant)
        alloc.set_table(fc, fm)
        alloc.bestfit_dev(c.data_ptr(), m.data_ptr(), R, idx.data_ptr(), delta.data_ptr(), tab.data_ptr(), True, s,
                          prefix_commit=True)
        torch.cuda.synchronize()
        got = idx.cpu().numpy()
        assert np.array_equal(got[:R], o_idx) and (got[R:] == -9).all(), variant
        assert np.array_equal(delta.cpu().numpy(), np.concatenate([o_dc, o_dm])), variant
        assert np.array_equal(tab.cpu().numpy(), o_tab), variant
        _check_committed(alloc, (o_tab[:D], o_tab[D:2 * D], np.zeros(D, np.int32)), D)


# ---- (e) the bound on rows per thread that keeps lane-private sums exact ---------------------------------
def _max_addend_table(D):
    """device 0 alone takes (100, 2^18 - 1)"""
    fc = np.full(D, 99, np.int32)
    fc[0] = 100
    return fc, np.full(D, MEM_MAX, np.int32)


def _max_addend_expect(D, R):
    dc = np.zeros(D, np.int64)
    dm = np.zeros(D, np.int64)
    dc[0], dm[0] = 100 * R, MEM_MAX * R
    fc, fm = _max_addend_table(D)
    left_c, left_m = fc - dc, fm - dm
    tab = np.concatenate([np.clip(left_c, INT32_MIN, INT32_MAX), np.clip(left_m, INT32_MIN, INT32_MAX),
                          ((left_c < 0) | (left_m < 0)).astype(np.int64)]).astype(np.int32)
    return np.concatenate([dc, dm]), tab


@pytest.mark.gpu
@pytest.mark.parametrize("variant,D,threads", [(2, 8, 256), (2, 64, 128), (3, 64, 256)], ids=["sorted-D8", "sorted-D64", "lut-D64"])
def test_lane_sum_bound(variant, D, threads, egpu, monkeypatch):
    """One CTA (EGPU_ROWS_PER_THREAD=524288), every row the largest request, all on device 0.  The entry
    point accepts R while R / threads + 8 < 2^19: the largest such R gives exact sums, one row more is
    refused before anything is launched or written."""
    import torch
    monkeypatch.setenv("EGPU_ROWS_PER_THREAD", "524288")
    R = threads * ((1 << 19) - 8) - 1
    assert R % 4 == 3
    alloc = egpu.BestFitAllocator(0)
    try:
        s = torch.cuda.current_stream().cuda_stream
        c = torch.full((R + 1,), 100, dtype=torch.int32, device="cuda")
        m = torch.full((R + 1,), MEM_MAX, dtype=torch.int32, device="cuda")
        idx = torch.full((R + 4,), -9, dtype=torch.int32, device="cuda")
        delta = torch.full((2 * D,), -1, dtype=torch.int64, device="cuda")
        tab = torch.full((3 * D,), -7, dtype=torch.int32, device="cuda")
        alloc.set_variant(variant)
        alloc.set_table(*_max_addend_table(D))
        alloc.bestfit_dev(c.data_ptr(), m.data_ptr(), R, idx.data_ptr(), delta.data_ptr(), tab.data_ptr(), False, s)
        torch.cuda.synchronize()
        e_delta, e_tab = _max_addend_expect(D, R)
        assert bool((idx[:R] == 0).all()) and bool((idx[R:] == -9).all())
        assert np.array_equal(delta.cpu().numpy(), e_delta)
        assert np.array_equal(tab.cpu().numpy(), e_tab)
        # one row more: refused, nothing launched (the lookup tables were built by the call above), nothing written
        idx.fill_(-9)
        delta.fill_(-1)
        torch.cuda.synchronize()
        n0 = alloc.launch_count
        with pytest.raises(egpu.EgpuError) as ei:
            alloc.bestfit_dev(c.data_ptr(), m.data_ptr(), R + 1, idx.data_ptr(), delta.data_ptr(), tab.data_ptr(), False, s)
        code = ei.value.code
        del ei  # its traceback holds this frame, and with it 1.6 GB of arrays, until the next garbage collection
        assert code == ERR_INVALID
        torch.cuda.synchronize()
        assert alloc.launch_count == n0
        assert bool((idx == -9).all()) and bool((delta == -1).all())
    finally:
        alloc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(2, 8), (2, 64), (3, 64)])
def test_multi_scan_max_addends(variant, D, egpu, monkeypatch):
    """The multi-batch scans under EGPU_MULTI_RPT=4096: two batches of 524 287 rows, one tile each
    (2048 or 4096 rows per thread), every row the largest request."""
    import torch
    monkeypatch.setenv("EGPU_MULTI_RPT", "4096")
    rows = [524_287, 524_287]
    alloc = egpu.BestFitAllocator(0)
    try:
        s = torch.cuda.current_stream().cuda_stream
        bufs = []
        for R in rows:
            bufs.append((torch.full((R + 4,), 100, dtype=torch.int32, device="cuda"),
                         torch.full((R + 4,), MEM_MAX, dtype=torch.int32, device="cuda"),
                         torch.empty(R + 4, dtype=torch.int32, device="cuda"), torch.empty(2 * D, dtype=torch.int64, device="cuda"),
                         torch.empty(3 * D, dtype=torch.int32, device="cuda")))
        _reset(bufs)
        alloc.set_variant(variant)
        alloc.set_table(*_max_addend_table(D))
        alloc.bestfit_batches_dev(_tuples(bufs, rows), s)
        torch.cuda.synchronize()
        for (_, _, idx, delta, tab), R in zip(bufs, rows):
            e_delta, e_tab = _max_addend_expect(D, R)
            assert bool((idx[:R] == 0).all()) and bool((idx[R:] == -9).all())
            assert np.array_equal(delta.cpu().numpy(), e_delta)
            assert np.array_equal(tab.cpu().numpy(), e_tab)
    finally:
        alloc.close()
