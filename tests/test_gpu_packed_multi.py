"""Multi-batch launches in the packed format: egpu_bestfit_batches_dev with EGPU_F_PACKED.

Every batch's d_req_core holds packed words (EGPU_PACK_REQUEST: core << 18 | mem; a word >= 2^25 is
not a request), d_req_mem is NULL and d_out_idx receives int8 indices.  The launch runs the packed
twins of the multi-batch kernels (csrc/egpu_alloc.cu: kKernels<kScanSortedMulti or kScanLutMulti,
kRowsPacked>[d_bucket(D)], the register scan and the lookup scan).  Each GPU case compares every batch exactly with
oracle/bestfit_np.py or the C oracle on the requests the words stand for, and, where it says so, with a
non-committing egpu_bestfit_batch_packed_dev call on the same words:

  1. the cell matrix: both packed scans at every D bucket edge and one D inside each bucket, under the
     AUTO, SORTED and LUT variants; ragged row counts; domain-edge words and tables;
  2. the grid-size rule around 512 Ki rows, whole waves with `extra` CTAs, and K up to 64;
  3. argument checks: the NULL d_req_mem rule, alignment, K, the grid variant, the sharded entry point,
     int8 output ranges that overlap by one byte or sit back to back;
  4. ordering on one pipelined stream, packed and int32 launches mixed, across group boundaries and
     around the epilogue ring, then a commit that a packed lookup launch must see;
  5. the table after every kind of table change, read by a packed probe batch;
  6. a captured CUDA graph replayed twice;
  7. exact demand sums at the largest rows per thread the launcher allows.
"""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_context_sequences as cs  # noqa: E402  (probe rows, restore cases)
import test_gpu_kernel_matrix as km  # noqa: E402  (cell tables and requests, max-addend tables)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "elastic-gpu-agent_b200", "csrc")
MEM_MAX = (1 << 18) - 1
ERR_INVALID, ERR_STATE = -1, -6
AUTO, GRID, SORTED, LUT = 0, 1, 2, 3
GUARD = 16  # guard bytes after every int8 index array


# ---- the packed kernel table -------------------------------------------------------------------------
PACKED_FAMILIES = ("sorted", "lut")
PACKED_TWINS = {"kScanSortedMulti": "bestfit_sorted_packed_multi_kernel", "kScanLutMulti": "bestfit_lut_packed_multi_kernel"}


def packed_twins(kind):
    """{scan family: its packed twin kernel} of family_kernel() (csrc/egpu_alloc.cu), for the twins named *_packed_<kind>_kernel"""
    src = open(os.path.join(CSRC, "egpu_alloc.cu")).read()
    twins = dict(re.findall(r"F == (kScan\w+)\) return kernel\(P \? (\w+)<", src))
    return {f: k for f, k in twins.items() if k.endswith(f"_packed_{kind}_kernel")}


def family(variant, D):
    """the packed scan a variant selects (AUTO: the register scan up to D = 16)"""
    return "sorted" if variant == SORTED or (variant == AUTO and D <= 16) else "lut"


CELLS = [(v, D) for v in (AUTO, SORTED, LUT) for D in km.D_ALL]


def test_packed_multi_twins_cover_every_cell():
    """the packed twins of the multi-batch scans in the kernel table, and a matrix cell for each of their buckets"""
    twins = packed_twins("multi")
    assert twins == PACKED_TWINS and tuple(k.split("_")[1] for k in twins.values()) == PACKED_FAMILIES
    want = {(f, b) for f in PACKED_FAMILIES for b in range(len(km.BUCKET_TOPS))}
    assert {(family(v, D), km.d_bucket(D)) for v, D in CELLS} == want
    for v in (SORTED, LUT):  # every variant reaches every bucket
        assert {km.d_bucket(D) for vv, D in CELLS if vv == v} == set(range(4))


# ---- inputs and references ---------------------------------------------------------------------------
def cell_words(D, tname, R):
    """the cell matrix's requests as words, with core 101..127 words, feasible words with one bit >= 25
    set, and EGPU_PACKED_INVALID scattered through them"""
    fc, fm, rc, rm = km.cell_case(D, tname, R)
    words = km.pack(rc, rm)
    if R:
        o_idx = km.ref_snapshot(D, tname, R)[0]
        feas = words[(o_idx >= 0) & (words < (1 << 25))]
        rng = np.random.default_rng([D, R, 25])
        n = max(1, R // 16)
        at = rng.integers(0, R, (3, n))
        words[at[0]] = (rng.integers(101, 128, n).astype(np.uint32) << 18) | rng.integers(0, MEM_MAX + 1, n).astype(np.uint32)
        base = feas[rng.integers(0, len(feas), n)] if len(feas) else np.zeros(n, np.uint32)
        words[at[1]] = base | (np.uint32(1) << rng.integers(25, 32, n).astype(np.uint32))
        words[at[2]] = 0xFFFFFFFF
    return fc, fm, words


def ref(fc, fm, words):
    from oracle import bestfit_np
    return bestfit_np.snapshot(np.asarray(fc, np.int32), np.asarray(fm, np.int32), *km.unpack(words))


def _s(torch):
    s = torch.cuda.current_stream().cuda_stream
    return C.c_void_p(1 if s == 0 else s)  # the legacy default stream is cudaStreamLegacy in the C ABI


def words_dev(torch, words):
    """device copy of the words (int32 storage), 4 spare words so an empty batch has a buffer too"""
    t = torch.zeros(words.size + 4, dtype=torch.int32, device="cuda")
    if words.size:
        t[:words.size] = torch.from_numpy(np.ascontiguousarray(words).view(np.int32)).cuda()
    return t


class Out:
    """the outputs of one packed batch, sentinel-filled"""

    def __init__(self, torch, R, D):
        self.R = R
        self.idx = torch.empty(R + GUARD, dtype=torch.int8, device="cuda")
        self.delta = torch.empty(2 * D, dtype=torch.int64, device="cuda")
        self.tab = torch.empty(3 * D, dtype=torch.int32, device="cuda")
        self.reset()

    def reset(self):
        self.idx.fill_(-9)
        self.delta.fill_(-1)
        self.tab.fill_(-7)

    def ptrs(self):
        return self.idx.data_ptr(), self.delta.data_ptr(), self.tab.data_ptr()

    def check(self, exp, where):
        o_idx, o_dc, o_dm, o_tab = exp
        idx = self.idx.cpu().numpy()
        assert np.array_equal(idx[:self.R].astype(np.int32), o_idx), f"{where}: indices"
        assert (idx[self.R:] == -9).all(), f"{where}: guard bytes"
        assert np.array_equal(self.delta.cpu().numpy(), np.concatenate([o_dc, o_dm])), f"{where}: demand sums"
        assert np.array_equal(self.tab.cpu().numpy(), o_tab), f"{where}: table'"


def packed_multi(alloc, torch, ws, outs, inputs_ready=False):
    alloc.bestfit_batches_packed_dev([(w.data_ptr(), o.R) + o.ptrs() for w, o in zip(ws, outs)],
                                     torch.cuda.current_stream().cuda_stream, inputs_ready)


def packed_single(alloc, torch, w, R, D):
    """egpu_bestfit_batch_packed_dev, non-committing, on the same words: (idx int8, delta, table')"""
    o = Out(torch, R, D)
    i, dl, t = o.ptrs()
    rc = alloc._lib.egpu_bestfit_batch_packed_dev(alloc.handle, C.c_void_p(w.data_ptr()), R, C.c_void_p(i), C.c_void_p(dl),
                                                  C.c_void_p(t), 0, _s(torch))
    assert rc == 0
    torch.cuda.synchronize()
    return o


def same_outputs(a, b, where):
    assert torch_equal(a.idx, b.idx) and torch_equal(a.delta, b.delta) and torch_equal(a.tab, b.tab), \
        f"{where}: differs from egpu_bestfit_batch_packed_dev"


def torch_equal(x, y):
    return bool((x == y).all())


def table_is(alloc, fc, fm, ov=None):
    g_fc, g_fm, g_ov = alloc.table()
    ov = np.zeros(len(fc), np.int32) if ov is None else ov
    return np.array_equal(g_fc, fc) and np.array_equal(g_fm, fm) and np.array_equal(g_ov, ov)


# ---- 1. the cell matrix --------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", CELLS, ids=[f"{['auto', 'grid', 'sorted', 'lut'][v]}-D{D}" for v, D in CELLS])
def test_packed_cell(variant, D, alloc, egpu):
    """two batches per launch - the words and the same words reversed - against the oracle and the
    single-batch packed call; the table stays as it was and the launch is one kernel (+ the lookup build)"""
    import torch
    fam = family(variant, D)
    alloc.set_variant(variant)
    for tname in km.cell_tables(D):
        for R in km.ROW_COUNTS:
            where = f"{fam} scan, variant {variant}, D = {D}, table {tname}, R = {R}"
            fc, fm, words = cell_words(D, tname, R)
            exp = ref(fc, fm, words)
            alloc.set_table(fc, fm)
            ws = [words_dev(torch, words), words_dev(torch, words[::-1].copy())]
            outs = [Out(torch, R, D), Out(torch, R, D)]
            torch.cuda.synchronize()
            n0 = alloc.launch_count
            packed_multi(alloc, torch, ws, outs)
            torch.cuda.synchronize()
            assert alloc.launch_count - n0 == (2 if fam == "lut" else 1), f"{where}: launches"
            outs[0].check(exp, f"{where}, batch 0")
            outs[1].check((exp[0][::-1],) + exp[1:], f"{where}, batch 1 (reversed)")
            same_outputs(outs[0], packed_single(alloc, torch, ws[0], R, D), where)
            assert table_is(alloc, fc, fm), f"{where}: the table changed"


# ---- 2. the grid-size rule --------------------------------------------------------------------------------
_rs = np.random.default_rng(2026)
SIZE_SHAPES = {
    "524287": [524_287],
    "524288": [524_288],
    "524289": [524_289],
    "mixed": [1_000_003, 0, 5, 70_003],
    "5x1Mi": [1 << 20] * 5,
    "7x1Mi": [1 << 20] * 7,
    "K1": [77_777],
    "K3": [3, 0, 100_001],
    "K20": [int(x) * (i % 7 != 3) for i, x in enumerate(_rs.integers(1, 60_000, 20))],
    "K64": [int(x) * (i % 9 != 4) for i, x in enumerate(_rs.integers(1, 30_000, 64))],
}


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SIZE_SHAPES))
@pytest.mark.parametrize("D", [8, 17, 64])
def test_packed_size_rule(D, shape, alloc, oracle_c):
    import torch
    rows = SIZE_SHAPES[shape]
    rng = np.random.default_rng(600 + D)
    fc = rng.integers(0, 101, D).astype(np.int32)
    fm = rng.integers(0, MEM_MAX + 1, D).astype(np.int32)
    s = torch.cuda.current_stream().cuda_stream
    ws, refs, first = [], [], 0
    for R in rows:
        c = torch.empty(R + 4, dtype=torch.int32, device="cuda")
        m = torch.empty(R + 4, dtype=torch.int32, device="cuda")
        alloc.synth_requests_dev(3, 41 + D, first, R, c.data_ptr(), m.data_ptr(), s)
        first += R
        ok = (c >= 0) & (c <= 127) & (m >= 0) & (m <= MEM_MAX)
        w = torch.where(ok, (c << 18) | m, torch.full_like(c, -1))
        ws.append(w)
        words = w[:R].cpu().numpy().view(np.uint32)
        refs.append(oracle_c.snapshot(fc, fm, *km.unpack(words), oracle_c.max_threads()))
    alloc.set_table(fc, fm)
    outs = [Out(torch, R, D) for R in rows]
    for variant in (SORTED, LUT):
        alloc.set_variant(variant)
        for o in outs:
            o.reset()
        packed_multi(alloc, torch, ws, outs)
        torch.cuda.synchronize()
        for k, (o, w, exp) in enumerate(zip(outs, ws, refs)):
            where = f"variant {variant}, batch {k} of {len(rows)} ({o.R} rows)"
            o.check(exp, where)
            if k < 4:
                same_outputs(o, packed_single(alloc, torch, w, o.R, D), where)


# ---- 3. arguments ----------------------------------------------------------------------------------------
def _raw(alloc, batches, flags, stream):
    from elastic_gpu_agent_b200 import _lib as L
    arr = (L.Batch * len(batches))(*[L.Batch(*b) for b in batches])
    return alloc._lib.egpu_bestfit_batches_dev(alloc.handle, arr, len(arr), flags, stream)


@pytest.mark.gpu
def test_packed_arguments(alloc, egpu):
    import torch
    from elastic_gpu_agent_b200 import _lib as L
    D = 6
    fc, fm = np.array([3, 50, 100, 100, 0, 7], np.int32), np.array([10, 500, MEM_MAX, 0, 9, 64], np.int32)
    alloc.set_table(fc, fm)
    s = _s(torch)
    P = L.F_PACKED
    words = km.pack(np.arange(200) % 103, (np.arange(200) * 37) % 600)
    w = words_dev(torch, words)
    idx = torch.full((2048,), -9, dtype=torch.int8, device="cuda")
    c32 = torch.zeros(204, dtype=torch.int32, device="cuda")
    i32 = torch.zeros(204, dtype=torch.int32, device="cuda")
    wp, ip = w.data_ptr(), idx.data_ptr()
    torch.cuda.synchronize()
    n0 = alloc.launch_count
    refused = {
        "d_req_mem given with the flag": ([(wp, c32.data_ptr(), 100, ip, None, None)], P, ERR_INVALID),
        "misaligned words": ([(wp + 4, None, 100, ip, None, None)], P, ERR_INVALID),
        "misaligned indices": ([(wp, None, 100, ip + 1, None, None)], P, ERR_INVALID),
        "NULL words": ([(None, None, 100, ip, None, None)], P, ERR_INVALID),
        "K = 65": ([(wp, None, 1, ip + 16 * k, None, None) for k in range(65)], P, ERR_INVALID),
        "a packed batch without the flag": ([(wp, None, 100, ip, None, None)], 0, ERR_INVALID),
        "an unknown flag": ([(wp, None, 100, ip, None, None)], P | 32, ERR_INVALID),
        # int8 outputs overlapping by one byte: [0, 97) and [96, 196)
        "overlapping int8 outputs": ([(wp, None, 97, ip, None, None), (wp, None, 100, ip + 96, None, None)], P, ERR_INVALID),
    }
    for what, (batches, flags, code) in refused.items():
        assert _raw(alloc, batches, flags, s) == code, what
    # a NULL d_req_mem with R = 0 was always fine, and stays fine without the flag
    assert _raw(alloc, [(c32.data_ptr(), None, 0, i32.data_ptr(), None, None)], 0, s) == 0
    # the sharded entry point refuses the flag before it looks at anything else
    arr = (L.Batch * 1)(L.Batch(wp, None, 100, ip, None, None))
    assert alloc._lib.egpu_bestfit_batches_shard_dev(alloc.handle, arr, 1, P, 0, s) == ERR_INVALID
    alloc.set_variant(GRID)
    assert _raw(alloc, [(wp, None, 100, ip, None, None)], P, s) == ERR_STATE
    alloc.set_variant(AUTO)
    torch.cuda.synchronize()
    assert alloc.launch_count == n0 + 1  # only the empty int32 launch
    assert bool((idx == -9).all()), "a refused launch wrote indices"
    # the same two batches back to back, [0, 96) and [96, 196): accepted
    assert _raw(alloc, [(wp, None, 96, ip, None, None), (wp + 4 * 96, None, 100, ip + 96, None, None)], P, s) == 0
    torch.cuda.synchronize()
    exp = ref(fc, fm, words)[0]
    got = idx.cpu().numpy()
    assert np.array_equal(got[:196].astype(np.int32), exp[:196]) and (got[196:] == -9).all()


# ---- 4. ordering on one pipelined stream ------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_pipelined_chain(variant, alloc, egpu):
    """40 launches of 5 batches with EGPU_F_INPUTS_READY, packed and int32 in turn: past the 24-launch
    and half-ring group limits and twice around the 128-slot epilogue ring.  Launch 30 rewrites launch
    10's outputs (both packed) with other words and must land after it.  Then a committing single-batch
    call, and a packed lookup launch that has to see the committed table."""
    import torch
    D = 24
    rng = np.random.default_rng(4000 + variant)
    fc = rng.integers(20, 101, D).astype(np.int32)
    fm = rng.choice(np.arange(1000, MEM_MAX + 1), D, replace=False).astype(np.int32)
    alloc.set_variant(variant)
    alloc.set_table(fc, fm)
    n_launch, K = 40, 5
    plans = []
    for j in range(n_launch):
        sizes = [0 if rng.random() < 0.15 else int(rng.integers(1, 6000)) for _ in range(K)]
        if j == 30:
            sizes = [o.R for o in plans[10][2]]
        batches, outs = [], []
        for R in sizes:
            rc = rng.integers(-2, 103, R).astype(np.int32)
            rm = rng.integers(-2, 4000, R).astype(np.int32)
            words = km.pack(rc, rm)
            batches.append((words, ref(fc, fm, words)))
        packed = j % 2 == 0
        if j == 30:
            outs = plans[10][2]
        else:
            outs = [Out(torch, R, D) if packed else None for R in sizes]
        plans.append((packed, batches, outs))
    dev = []
    for j, (packed, batches, outs) in enumerate(plans):
        if packed:
            dev.append([words_dev(torch, w) for w, _ in batches])
        else:
            arrs = []
            for k, (w, _) in enumerate(batches):
                rc, rm = km.unpack(w)
                R = w.size
                arrs.append((km._dev(torch, rc), km._dev(torch, rm), torch.full((R + 4,), -9, dtype=torch.int32, device="cuda"),
                             torch.full((2 * D,), -1, dtype=torch.int64, device="cuda"),
                             torch.full((3 * D,), -7, dtype=torch.int32, device="cuda")))
            dev.append(arrs)
    rc, rm = rng.integers(0, 30, 5000).astype(np.int32), rng.integers(0, 900, 5000).astype(np.int32)
    from oracle import bestfit_np
    o_idx, o_dc, o_dm, o_tab = bestfit_np.snapshot(fc, fm, rc, rm)
    c_idx = torch.empty(5004, dtype=torch.int32, device="cuda")
    c_rc, c_rm = km._dev(torch, rc), km._dev(torch, rm)
    torch.cuda.synchronize()  # every input is complete before the first launch
    s = torch.cuda.current_stream().cuda_stream
    for j, (packed, batches, outs) in enumerate(plans):
        if packed:
            packed_multi(alloc, torch, dev[j], outs, inputs_ready=True)
        else:
            alloc.bestfit_batches_dev([(c.data_ptr(), m.data_ptr(), w.size, i.data_ptr(), dl.data_ptr(), t.data_ptr())
                                       for (c, m, i, dl, t), (w, _) in zip(dev[j], batches)], s, inputs_ready=True)
    # a committing call (it takes a large share of every device), then a packed lookup launch
    alloc.bestfit_dev(c_rc.data_ptr(), c_rm.data_ptr(), 5000, c_idx.data_ptr(), 0, 0, True, s, inputs_ready=True)
    new_fc, new_fm, new_ov = km.committed(o_tab, D)
    alloc.set_variant(LUT)
    pr_c, pr_m = cs.probe_rows(new_fc, new_fm)
    probe = km.pack(pr_c, pr_m)
    p_out = Out(torch, probe.size, D)
    p_w = words_dev(torch, probe)
    torch.cuda.synchronize()
    packed_multi(alloc, torch, [p_w], [p_out], inputs_ready=True)
    torch.cuda.synchronize()
    for j, (packed, batches, outs) in enumerate(plans):
        if j == 10:
            continue  # its outputs belong to launch 30 now
        for k, (w, exp) in enumerate(batches):
            where = f"launch {j} ({'packed' if packed else 'int32'}), batch {k}"
            if packed:
                outs[k].check(exp, where)
            else:
                _, _, i, dl, t = dev[j][k]
                got = i.cpu().numpy()
                assert np.array_equal(got[:w.size], exp[0]) and (got[w.size:] == -9).all(), where
                assert np.array_equal(dl.cpu().numpy(), np.concatenate(exp[1:3])), where
                assert np.array_equal(t.cpu().numpy(), exp[3]), where
    assert np.array_equal(c_idx[:5000].cpu().numpy(), o_idx)
    assert (new_fc != fc).any()
    p_out.check(ref(new_fc, new_fm, probe), "packed lookup launch after the commit")
    assert table_is(alloc, new_fc, new_fm, new_ov)


# ---- 5. every kind of table change, read by a packed probe batch --------------------------------------------
def _probe(alloc, torch, egpu, where):
    """the probe rows of the context's table, through both packed scans"""
    fc, fm, _ = alloc.table()
    D = fc.size
    pr_c, pr_m = cs.probe_rows(fc, fm)
    words = km.pack(pr_c, pr_m)
    exp = ref(fc, fm, words)
    w = words_dev(torch, words)
    distinct = len(set(zip(fc.tolist(), fm.tolist()))) == D
    for variant in (SORTED, LUT):
        alloc.set_variant(variant)
        o = Out(torch, words.size, D)
        packed_multi(alloc, torch, [w], [o])
        torch.cuda.synchronize()
        o.check(exp, f"{where}, variant {variant}")
        if distinct:  # probe 9 d + 4 is device d's own (free_core, free_mem)
            assert np.array_equal(o.idx[:9 * D].cpu().numpy()[4::9], np.arange(D)), f"{where}: exact fits"
    return distinct


@pytest.mark.gpu
def test_packed_reads_every_table_change(alloc, egpu):
    import torch
    from elastic_gpu_agent_b200 import restore
    rng = np.random.default_rng(5150)
    D = 12
    fc = rng.integers(0, 101, D).astype(np.int32)
    fm = rng.choice(MEM_MAX + 1, D, replace=False).astype(np.int32)
    alloc.set_table(fc, fm)
    # every probe ends under LUT, so the changes below run there too: the lookup tables are built
    # before each change, and a packed launch that did not rebuild them would read stale ones
    assert _probe(alloc, torch, egpu, "set_table")
    rc, rm = rng.integers(0, 40, 3000).astype(np.int32), rng.integers(0, 20_000, 3000).astype(np.int32)
    alloc.bestfit(rc, rm, commit=True)
    _probe(alloc, torch, egpu, "commit")
    alloc.bestfit_rounds(rng.integers(0, 60, 2000).astype(np.int32), rng.integers(0, 30_000, 2000).astype(np.int32))
    _probe(alloc, torch, egpu, "rounds")
    kind, ea, eb = egpu.synth.churn_events(9, 3000)
    alloc.replay(kind, ea, eb)
    _probe(alloc, torch, egpu, "replay")
    case = cs.restore_case(rng, D)
    restore.restore_table(alloc, case["records"], case["links"], case["cap_core"], case["cap_mem"], install=True)
    _probe(alloc, torch, egpu, "restore with install")


# ---- 6. graph capture ----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", [8, 33])  # AUTO: the register scan, the lookup scan
def test_packed_graph_replay(D, alloc, egpu):
    import torch
    fc, fm, words = cell_words(D, "spread", km.ROW_COUNTS[-1])
    exp = ref(fc, fm, words)
    alloc.set_table(fc, fm)
    ws = [words_dev(torch, words), words_dev(torch, words[::-1].copy())]
    outs = [Out(torch, words.size, D) for _ in ws]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        packed_multi(alloc, torch, ws, outs)  # warm-up: occupancy query and lookup tables outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        packed_multi(alloc, torch, ws, outs, inputs_ready=True)
    for rep in range(2):
        for o in outs:
            o.reset()
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        outs[0].check(exp, f"replay {rep}, batch 0")
        outs[1].check((exp[0][::-1],) + exp[1:], f"replay {rep}, batch 1")


# ---- 7. exact sums at the largest rows per thread -------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(SORTED, 8), (SORTED, 64), (LUT, 64)])
def test_packed_max_addends(variant, D, egpu, monkeypatch):
    """EGPU_MULTI_RPT=4096: two batches of 524 287 rows, one tile each, every row the largest request
    (100, 2^18 - 1), all on device 0: exact sums for both scans (the lookup scan folds its 12-bit field
    every kLutFlushTrips trips; each of its warps here runs 256 trips)"""
    import torch
    monkeypatch.setenv("EGPU_MULTI_RPT", "4096")
    rows = [524_287, 524_287]
    alloc = egpu.BestFitAllocator(0)
    try:
        ws = [torch.full((R + 4,), (100 << 18) | MEM_MAX, dtype=torch.int32, device="cuda") for R in rows]
        outs = [Out(torch, R, D) for R in rows]
        alloc.set_variant(variant)
        alloc.set_table(*km._max_addend_table(D))
        packed_multi(alloc, torch, ws, outs)
        torch.cuda.synchronize()
        for k, (o, R) in enumerate(zip(outs, rows)):
            e_delta, e_tab = km._max_addend_expect(D, R)
            assert bool((o.idx[:R] == 0).all()) and bool((o.idx[R:] == -9).all()), k
            assert np.array_equal(o.delta.cpu().numpy(), e_delta), (k, o.delta.cpu().numpy()[[0, D]])
            assert np.array_equal(o.tab.cpu().numpy(), e_tab), k
    finally:
        alloc.close()
