"""egpu_bestfit_batch_packed_dev on the snapshot launch path.

The call scores R packed words (EGPU_PACK_REQUEST: core << 18 | mem; a word >= 2^25 is not a request) into R int8
indices.  Outside the grid variant it runs kKernels<kScanSorted or kScanLut, kRowsPacked>[d_bucket(D)]
(csrc/egpu_alloc.cu), the round-robin packed scans of the sharded calls, in the scan the context's variant selects, and pipelines under
EGPU_F_INPUTS_READY with the other scans of the context; under EGPU_VARIANT_GRID it keeps the warp-chunk scan of
egpu_bestfit_batch_packed.  Every case compares exactly with the C oracle on the requests the words stand for (not a
request: (-1, -1)), and where it says so with the int32 egpu_bestfit_batch_dev on the same requests:

  1. the cell matrix: every D of the kernel matrix under AUTO, SORTED and LUT, its tables and ragged row counts;
  2. kernel selection: the lookup table is built after egpu_table_set and after a commit, and the grid variant
     gives the same results;
  3. a chain of EGPU_F_INPUTS_READY calls mixing packed, int32 and packed multi-batch scans with committing packed
     calls, past the epilogue slot ring, against its fully ordered run, eagerly and replayed from a CUDA graph;
  4. commits: the installed table and sticky oversubscription flags equal the grid variant's, launch counts;
  5. flags other than EGPU_F_COMMIT and EGPU_F_INPUTS_READY are ignored; refusals launch and write nothing.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_kernel_matrix as km  # noqa: E402  (cell tables, D_ALL, ROW_COUNTS, pack / unpack)
import test_gpu_packed_multi as pm  # noqa: E402  (cell words, Out, words_dev, family, table_is)

ERR_INVALID, ERR_NO_TABLE = -1, -5
AUTO, GRID, SORTED, LUT = 0, 1, 2, 3
F_COMMIT, F_INPUTS_READY, F_PREFIX, F_APPLY, F_PACKED, F_ROUNDS, F_DEVICE_ROUNDS = 1, 2, 4, 8, 16, 32, 128
EPI_SLOTS = 32  # kEpiSlots (csrc/egpu_kernels.cuh)
CELLS = pm.CELLS


def test_wrapper_flags(egpu):
    """bestfit_packed_dev hands the library the words, NULL for absent outputs, and only COMMIT / INPUTS_READY"""
    calls = []

    class Lib:
        def __getattr__(self, name):
            return lambda *a: calls.append((name, a)) or 0

    a = object.__new__(egpu.BestFitAllocator)
    a._lib, a._h = Lib(), C.c_void_p(1)
    a.bestfit_packed_dev(16, 5, 32)
    a.bestfit_packed_dev(16, 5, 32, 48, 64, 0, commit=True)
    a.bestfit_packed_dev(16, 5, 32, 48, 0, 7, inputs_ready=True)
    assert {n for n, _ in calls} == {"egpu_bestfit_batch_packed_dev"}
    (_, a0), (_, a1), (_, a2) = calls
    assert (a0[1].value, a0[2], a0[3].value, a0[4].value, a0[5].value, a0[6], a0[7].value) == (16, 5, 32, None, None, 0, None)
    assert (a1[4].value, a1[5].value, a1[6], a1[7].value) == (48, 64, F_COMMIT, 1)  # torch's 0 = cudaStreamLegacy
    assert (a2[5].value, a2[6], a2[7].value) == (None, F_INPUTS_READY, 7)
    a._lib = None
    a._h = None


# ---- helpers --------------------------------------------------------------------------------------------
def stream(torch):
    return torch.cuda.current_stream().cuda_stream


class Out32(pm.Out):
    """the outputs of one int32 batch, sentinel-filled"""

    def __init__(self, torch, R, D):
        self.R = R
        self.idx = torch.empty(R + 4, dtype=torch.int32, device="cuda")
        self.delta = torch.empty(2 * D, dtype=torch.int64, device="cuda")
        self.tab = torch.empty(3 * D, dtype=torch.int32, device="cuda")
        self.reset()


def same_outputs(a, b, where):
    assert np.array_equal(a.idx[:a.R].cpu().numpy().astype(np.int32), b.idx[:b.R].cpu().numpy().astype(np.int32)), f"{where}: indices"
    assert bool((a.delta == b.delta).all()) and bool((a.tab == b.tab).all()), f"{where}: sums / table'"


def int32_of(torch, words):
    return tuple(km._dev(torch, x) for x in km.unpack(words))


def packed_dev(alloc, torch, w, o, commit=False, inputs_ready=False, s=None):
    i, dl, t = o.ptrs()
    alloc.bestfit_packed_dev(w.data_ptr(), o.R, i, dl, t, stream(torch) if s is None else s, commit, inputs_ready)


def int32_dev(alloc, torch, cm, o, commit=False, inputs_ready=False, s=None):
    i, dl, t = o.ptrs()
    alloc.bestfit_dev(cm[0].data_ptr(), cm[1].data_ptr(), o.R, i, dl, t, commit, stream(torch) if s is None else s, inputs_ready)


# ---- 1. the cell matrix ------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", CELLS, ids=[f"{['auto', 'grid', 'sorted', 'lut'][v]}-D{D}" for v, D in CELLS])
def test_packed_dev_cell(variant, D, alloc, oracle_c, egpu):
    """one non-committing call per table and row count against the C oracle, then the int32 call on the same requests:
    same indices, demand sums and table'; one launch (+ the lookup build after egpu_table_set); the table stays"""
    import torch
    fam = pm.family(variant, D)
    alloc.set_variant(variant)
    for tname in km.cell_tables(D):
        for R in km.ROW_COUNTS:
            where = f"{fam} scan, variant {variant}, D = {D}, table {tname}, R = {R}"
            fc, fm, words = pm.cell_words(D, tname, R)
            exp = oracle_c.snapshot(fc, fm, *km.unpack(words))
            alloc.set_table(fc, fm)
            w, o8, o32 = pm.words_dev(torch, words), pm.Out(torch, R, D), Out32(torch, R, D)
            cm = int32_of(torch, words)
            torch.cuda.synchronize()
            n0 = alloc.launch_count
            packed_dev(alloc, torch, w, o8)
            assert alloc.launch_count - n0 == 1 + (fam == "lut"), f"{where}: launches"
            int32_dev(alloc, torch, cm, o32)
            torch.cuda.synchronize()
            o8.check(exp, where)
            same_outputs(o8, o32, where)
            assert pm.table_is(alloc, fc, fm), f"{where}: the table changed"


# ---- 2. kernel selection ----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_packed_dev_lookup_table_after_changes(alloc, oracle_c, egpu):
    """LUT at D = 64: a commit right after egpu_table_set, then a scan, then egpu_table_set and a scan again.  Each call
    after a table change rebuilds the lookup table (two launches), each result is the oracle's on the table then current;
    the int32 lookup scan counts its launches the same way"""
    import torch
    w = egpu.synth.workload("cfg4")
    D = 64
    fc, fm = w["free_core"], w["free_mem"]
    words = [km.pack(*egpu.synth.requests(w["dist"], 70 + k, R)) for k, R in enumerate((3_001, 40_003, 40_003, 40_003))]
    commit_words = km.pack(np.arange(64) % 3 + 1, np.full(64, 200))
    alloc.set_variant(LUT)
    alloc.set_table(fc, fm)
    cw, co = pm.words_dev(torch, commit_words), pm.Out(torch, 64, D)
    torch.cuda.synchronize()
    n0 = alloc.launch_count
    packed_dev(alloc, torch, cw, co, commit=True)
    assert alloc.launch_count - n0 == 2
    c_exp = oracle_c.snapshot(fc, fm, *km.unpack(commit_words))
    new_fc, new_fm, new_ov = km.committed(c_exp[3], D)
    assert not np.array_equal(new_fc, fc)
    wd, o = pm.words_dev(torch, words[1]), pm.Out(torch, 40_003, D)
    n0 = alloc.launch_count
    packed_dev(alloc, torch, wd, o)
    assert alloc.launch_count - n0 == 2, "the scan after the commit rebuilds the lookup table"
    n0 = alloc.launch_count
    wd2, o2 = pm.words_dev(torch, words[2]), pm.Out(torch, 40_003, D)
    packed_dev(alloc, torch, wd2, o2)
    assert alloc.launch_count - n0 == 1, "no table change: no rebuild"
    torch.cuda.synchronize()
    co.check(c_exp, "commit after egpu_table_set")
    o.check(oracle_c.snapshot(new_fc, new_fm, *km.unpack(words[1])), "scan after the commit")
    o2.check(oracle_c.snapshot(new_fc, new_fm, *km.unpack(words[2])), "second scan after the commit")
    assert pm.table_is(alloc, new_fc, new_fm, new_ov)
    alloc.set_table(fc, fm)
    wd3, o3 = pm.words_dev(torch, words[3]), pm.Out(torch, 40_003, D)
    n0 = alloc.launch_count
    packed_dev(alloc, torch, wd3, o3)
    assert alloc.launch_count - n0 == 2, "the scan after egpu_table_set rebuilds the lookup table"
    torch.cuda.synchronize()
    o3.check(oracle_c.snapshot(fc, fm, *km.unpack(words[3])), "scan after egpu_table_set")
    # the int32 lookup scan counts the same
    alloc.set_table(fc, fm)
    cm, o32 = int32_of(torch, words[3]), Out32(torch, 40_003, D)
    n0 = alloc.launch_count
    int32_dev(alloc, torch, cm, o32)
    assert alloc.launch_count - n0 == 2
    torch.cuda.synchronize()
    same_outputs(o3, o32, "int32 lookup scan")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg3", "cfg4"])
def test_packed_dev_grid_variant(name, alloc, oracle_c, egpu):
    """EGPU_VARIANT_GRID keeps the warp-chunk scan (one launch, no lookup build): the same outputs as AUTO, for a
    non-committing and a committing call, a ragged batch and an empty one"""
    import torch
    w = egpu.synth.workload(name)
    D = int(w["D"])
    fc, fm = w["free_core"], w["free_mem"]
    for R in (0, 5, 513, 100_003):
        words = km.packed_words(*egpu.synth.requests(w["dist"], 11 + R, R), R, D)
        wd = pm.words_dev(torch, words)
        outs = {}
        for variant in (AUTO, GRID):
            alloc.set_variant(variant)
            for commit in (False, True):
                alloc.set_table(fc, fm)
                o = pm.Out(torch, R, D)
                torch.cuda.synchronize()
                n0 = alloc.launch_count
                packed_dev(alloc, torch, wd, o, commit=commit)
                if variant == GRID:
                    assert alloc.launch_count - n0 == 1
                torch.cuda.synchronize()
                outs[variant, commit] = (o, alloc.table())
        exp = oracle_c.snapshot(fc, fm, *km.unpack(words))
        for commit in (False, True):
            where = f"{name}, R = {R}, commit {commit}"
            outs[AUTO, commit][0].check(exp, where)
            same_outputs(outs[AUTO, commit][0], outs[GRID, commit][0], where)
            for x, y in zip(outs[AUTO, commit][1], outs[GRID, commit][1]):
                assert np.array_equal(x, y), f"{where}: installed table"


# ---- 3. pipelining and graphs ------------------------------------------------------------------------------
PATTERN = ("packed", "int32", "packed", "multi", "packed", "packed", "int32", "packed", "multi", "packed",
           "commit", "packed", "int32", "multi", "packed", "packed", "int32", "packed", "multi", "packed")
CHAIN = PATTERN * 3  # 48 single-batch scans: past the epilogue slot ring, and past a launch group (24)


class Chain:
    """CHAIN's inputs and outputs: random words (1 .. 30 000 rows), two-batch packed multi-batch launches, and small
    committing packed calls that fit (the table changes, nothing is oversubscribed)"""

    def __init__(self, torch, D, seed):
        rng = np.random.default_rng(seed)
        self.D = D
        self.calls = []
        for kind in CHAIN:
            if kind == "commit":
                words = [km.pack(rng.integers(0, 3, 7), rng.integers(0, 64, 7))]
            elif kind == "multi":
                words = [self.rand(rng, int(rng.integers(1, 30_000))), self.rand(rng, int(rng.integers(0, 5_000)))]
            else:
                words = [self.rand(rng, int(rng.integers(1, 30_000)))]
            outs = [(Out32 if kind == "int32" else pm.Out)(torch, x.size, D) for x in words]
            dev = [int32_of(torch, x) if kind == "int32" else pm.words_dev(torch, x) for x in words]
            self.calls.append((kind, words, dev, outs))
        assert sum(k != "multi" for k in CHAIN) > EPI_SLOTS

    @staticmethod
    def rand(rng, R):
        return km.packed_words(rng.integers(-1, 104, R).astype(np.int32), rng.integers(-1, 9000, R).astype(np.int32), R, 40)

    def run(self, alloc, torch, s, inputs_ready):
        for kind, _, dev, outs in self.calls:
            if kind == "multi":
                alloc.bestfit_batches_packed_dev([(d.data_ptr(), o.R) + o.ptrs() for d, o in zip(dev, outs)], s, inputs_ready)
            elif kind == "int32":
                int32_dev(alloc, torch, dev[0], outs[0], False, inputs_ready, s)
            else:
                packed_dev(alloc, torch, dev[0], outs[0], kind == "commit", inputs_ready, s)

    def reset(self):
        for _, _, _, outs in self.calls:
            for o in outs:
                o.reset()

    def snapshot(self):
        return [[(o.idx.clone(), o.delta.clone(), o.tab.clone()) for o in outs] for _, _, _, outs in self.calls]

    def check_oracle(self, oracle_c, fc, fm):
        """the fully ordered run against the oracle, the table changing at every commit"""
        D = self.D
        for j, (kind, words, _, outs) in enumerate(self.calls):
            for x, o in zip(words, outs):
                exp = oracle_c.snapshot(fc, fm, *km.unpack(x))
                o.check(exp, f"call {j} ({kind}), fully ordered")
                if kind == "commit":
                    assert not exp[3][2 * D:].any()
                    fc, fm = exp[3][:D], exp[3][D:2 * D]
        return fc, fm

    def check_same(self, ref, where):
        for j, ((kind, _, _, outs), r) in enumerate(zip(self.calls, ref)):
            for k, (o, (i, dl, t)) in enumerate(zip(outs, r)):
                assert bool(torch_equal(o.idx, i)) and bool(torch_equal(o.delta, dl)) and bool(torch_equal(o.tab, t)), \
                    f"{where}: call {j} ({kind}) batch {k} differs from the fully ordered run"


def torch_equal(a, b):
    import torch
    return torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(AUTO, 8), (AUTO, 40), (SORTED, 40), (LUT, 8)],
                         ids=["auto-D8", "auto-D40", "sorted-D40", "lut-D8"])
def test_packed_dev_pipelined_chain(variant, D, alloc, oracle_c, egpu):
    """CHAIN fully ordered (checked against the oracle), then with EGPU_F_INPUTS_READY on every call from the same
    table: every output equals the fully ordered run's, and the context ends with the same table"""
    import torch
    rng = np.random.default_rng(5000 + D)
    fc = rng.integers(50, 101, D).astype(np.int32)
    fm = rng.choice(np.arange(10_000, km.MEM_MAX + 1), D, replace=False).astype(np.int32)
    alloc.set_variant(variant)
    ch = Chain(torch, D, 77 + D)
    s = torch.cuda.Stream()
    for inputs_ready in (False, True):
        alloc.set_table(fc, fm)
        ch.reset()
        torch.cuda.synchronize()  # every input is complete before the first launch
        ch.run(alloc, torch, s.cuda_stream, inputs_ready)
        torch.cuda.synchronize()
        if not inputs_ready:
            end_fc, end_fm = ch.check_oracle(oracle_c, fc, fm)
            ref = ch.snapshot()
        else:
            ch.check_same(ref, "pipelined")
        assert pm.table_is(alloc, end_fc, end_fm)


@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(AUTO, 8), (AUTO, 40)], ids=["auto-D8", "auto-D40"])
def test_packed_dev_graph(variant, D, alloc, oracle_c, egpu):
    """CHAIN with EGPU_F_INPUTS_READY captured in a CUDA graph right after egpu_table_set, then replayed twice, each
    time after egpu_table_set of the same table: every replay gives the fully ordered run's outputs and table"""
    import torch
    rng = np.random.default_rng(6000 + D)
    fc = rng.integers(50, 101, D).astype(np.int32)
    fm = rng.choice(np.arange(10_000, km.MEM_MAX + 1), D, replace=False).astype(np.int32)
    alloc.set_variant(variant)
    ch = Chain(torch, D, 99 + D)
    s = torch.cuda.Stream()
    alloc.set_table(fc, fm)
    torch.cuda.synchronize()
    ch.run(alloc, torch, s.cuda_stream, False)  # also the warm-up: occupancy queries outside the capture
    torch.cuda.synchronize()
    end_fc, end_fm = ch.check_oracle(oracle_c, fc, fm)
    ref = ch.snapshot()
    alloc.set_table(fc, fm)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        ch.run(alloc, torch, s.cuda_stream, True)
    for rep in range(2):
        ch.reset()
        alloc.set_table(fc, fm)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        ch.check_same(ref, f"replay {rep}")
        assert pm.table_is(alloc, end_fc, end_fm), f"replay {rep}: table"


# ---- 4. commits -------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(AUTO, 8), (AUTO, 64), (SORTED, 64), (LUT, 8)],
                         ids=["auto-D8", "auto-D64", "sorted-D64", "lut-D8"])
def test_packed_dev_commit(variant, D, alloc, oracle_c, egpu):
    """committing calls in turn - one that oversubscribes, one that fits, an empty one - give the outputs, installed
    tables and sticky oversubscription flags of the same calls under the grid variant (the kernel the call ran before);
    each is one launch, plus the lookup build when the scan is the lookup scan (the table just changed)"""
    import torch
    fc, fm = km.cell_tables(D)["spread"]
    rng = np.random.default_rng(D)
    batches = [km.pack(rng.integers(0, 101, 50_000), rng.integers(0, km.MEM_MAX + 1, 50_000)),
               km.pack(np.zeros(5, np.int64), np.zeros(5, np.int64)), np.zeros(0, np.uint32)]
    lut = pm.family(variant, D) == "lut"
    got = {}
    for v in (variant, GRID):
        alloc.set_variant(v)
        alloc.set_table(fc, fm)
        got[v] = []
        for k, words in enumerate(batches):
            wd, o = pm.words_dev(torch, words), pm.Out(torch, words.size, D)
            torch.cuda.synchronize()
            n0 = alloc.launch_count
            packed_dev(alloc, torch, wd, o, commit=True)
            assert alloc.launch_count - n0 == 1 + (lut and v != GRID), (v, k)
            torch.cuda.synchronize()
            got[v].append((o, alloc.table()))
    cur_fc, cur_fm = fc, fm
    for k, words in enumerate(batches):
        exp = oracle_c.snapshot(cur_fc, cur_fm, *km.unpack(words))
        (o, tab), (og, tab_g) = got[variant][k], got[GRID][k]
        same_outputs(o, og, f"batch {k}")
        assert np.array_equal(o.idx[:o.R].cpu().numpy().astype(np.int32), exp[0]) and \
            np.array_equal(o.delta.cpu().numpy(), np.concatenate(exp[1:3])), f"batch {k}"
        for x, y in zip(tab, tab_g):
            assert np.array_equal(x, y), f"batch {k}: installed table"
        cur_fc, cur_fm = tab[0], tab[1]
    assert got[variant][0][1][2].any(), "the first batch oversubscribes"
    assert np.array_equal(got[variant][2][1][2], got[variant][0][1][2]), "the flags are sticky"


# ---- 5. flags and refusals ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT])
def test_packed_dev_other_flags_ignored(variant, alloc, oracle_c, egpu):
    """EGPU_F_PREFIX_COMMIT, EGPU_F_PACKED, EGPU_F_APPLY, EGPU_F_ROUNDS, EGPU_F_DEVICE_ROUNDS and bit 64, alone or
    together, give the plain snapshot (no EGPU_IDX_DEFERRED, uncapped sums); with EGPU_F_COMMIT the plain commit"""
    import torch
    D = 16
    fc, fm = km.cell_tables(D)["dups"]
    words = km.pack(np.full(4000, 30), np.full(4000, 100))  # far more demand than any device holds
    exp = oracle_c.snapshot(fc, fm, *km.unpack(words))
    wd = pm.words_dev(torch, words)
    lib, h, s = alloc._lib, alloc.handle, pm._s(torch)
    alloc.set_variant(variant)
    for extra in (F_PREFIX, F_PACKED, F_PACKED | F_PREFIX, F_APPLY, 64, F_ROUNDS, F_DEVICE_ROUNDS,
                  F_PREFIX | F_COMMIT | F_ROUNDS | F_DEVICE_ROUNDS | F_PACKED):
        alloc.set_table(fc, fm)
        o = pm.Out(torch, words.size, D)
        i, dl, t = o.ptrs()
        torch.cuda.synchronize()
        n0 = alloc.launch_count
        assert lib.egpu_bestfit_batch_packed_dev(h, C.c_void_p(wd.data_ptr()), words.size, C.c_void_p(i), C.c_void_p(dl),
                                                 C.c_void_p(t), extra, s) == 0, extra
        assert alloc.launch_count - n0 == 1 + (variant == LUT), extra
        torch.cuda.synchronize()
        o.check(exp, f"flags {extra}")
        if extra & F_COMMIT:
            assert pm.table_is(alloc, *km.committed(exp[3], D)), f"flags {extra}: committed table"
        else:
            assert pm.table_is(alloc, fc, fm), f"flags {extra}: the table changed"


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [AUTO, GRID, SORTED, LUT])
def test_packed_dev_refusals(variant, alloc, egpu):
    """NULL or misaligned words or indices with R > 0, R < 0 and (before egpu_table_set) no table: refused before
    anything is launched or written.  R = 0 with NULL arrays is a valid empty batch: zero sums, table' = the table"""
    import torch
    D = 6
    fc, fm = np.array([3, 50, 100, 100, 0, 7], np.int32), np.array([10, 500, km.MEM_MAX, 0, 9, 64], np.int32)
    lib, h, s = alloc._lib, alloc.handle, pm._s(torch)
    words = km.pack(np.arange(200) % 103, (np.arange(200) * 37) % 600)
    w = pm.words_dev(torch, words)
    o = pm.Out(torch, 200, D)
    wp, (ip, dp, tp) = w.data_ptr(), o.ptrs()
    vp = C.c_void_p

    def call(words_p, R, idx_p, flags=0):
        return lib.egpu_bestfit_batch_packed_dev(h, vp(words_p), R, vp(idx_p), vp(dp), vp(tp), flags, s)

    alloc.set_variant(variant)
    assert call(wp, 100, ip) == ERR_NO_TABLE
    alloc.set_table(fc, fm)
    torch.cuda.synchronize()
    n0 = alloc.launch_count
    refused = {
        "NULL words": call(None, 100, ip),
        "NULL indices": call(wp, 100, None, F_COMMIT),
        "misaligned words": call(wp + 4, 100, ip),
        "misaligned indices": call(wp, 100, ip + 1, F_INPUTS_READY),
        "R < 0": call(wp, -1, ip),
    }
    for what, code in refused.items():
        assert code == ERR_INVALID, what
    torch.cuda.synchronize()
    assert alloc.launch_count == n0, "a refused call launched"
    assert bool((o.idx == -9).all()) and bool((o.delta == -1).all()) and bool((o.tab == -7).all()), "a refused call wrote"
    assert pm.table_is(alloc, fc, fm)
    assert call(None, 0, None, F_COMMIT) == 0
    torch.cuda.synchronize()
    assert bool((o.delta == 0).all())
    assert np.array_equal(o.tab.cpu().numpy(), np.concatenate([fc, fm, np.zeros(D, np.int32)]))
    assert pm.table_is(alloc, fc, fm)
