"""Release on the device: egpu_bestfit_batch[_dev] with EGPU_F_RELEASE [| EGPU_F_COMMIT] [| EGPU_F_PACKED] (DESIGN.md 2.8).

Every GPU case compares exactly with the numpy restatement of the rule (tests/release_np.py), in both row formats:

  1. the header text and the flag value;
  2. the hand-derived known answers of tests/golden/release_kat.json;
  3. parity of the sums, table', the installed table and the flags over the D buckets and ragged row counts, dry and
     committing, under every variant setting, with guard elements after the rows and the indices, which are never
     written; 1 Mi + 1 rows;
  4. the host form, pageable and pinned;
  5. the inverse property: rounds in one launch, then release of all rows (at once, or in three chunks) gives the
     table back;
  6. agreement with sequential mode: replay of ALLOCs and FREEs equals replay of the ALLOCs and one release;
  7. refusals: on the device (double release, a flagged device) and on the host (flags, arrays, R, no table);
  8. a churn tick (release of batch t - 2, admission of batch t) in a CUDA graph, replayed 32 times, and a snapshot scan
     after a release (register and lookup scan).
"""
import ctypes as C
import json
import os

import numpy as np
import pytest

import release_np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KATS = json.load(open(os.path.join(ROOT, "tests", "golden", "release_kat.json")))["cases"]
MEM_MAX = (1 << 18) - 1
ERR_INVALID, ERR_NO_TABLE, ERR_STATE = -1, -5, -6
AUTO, GRID, SORTED, LUT = 0, 1, 2, 3
F_COMMIT, F_INPUTS_READY, F_PREFIX, F_APPLY, F_PACKED, F_ROUNDS, F_DEVICE_ROUNDS, F_RELEASE = 1, 2, 4, 8, 16, 32, 128, 256
DR = F_PREFIX | F_COMMIT | F_ROUNDS | F_DEVICE_ROUNDS
GUARD = 16  # guard elements after every row and index array
D_BUCKETS = (1, 8, 16, 17, 32, 64)
ROWS = (0, 1, 3, 4, 513, 4099)


# ---- 1. header ---------------------------------------------------------------------------------------------------
def test_release_header_text_and_flag_value():
    import elastic_gpu_agent_b200._lib as L
    src = open(os.path.join(ROOT, "include", "egpu_alloc.h")).read()
    assert "#define EGPU_F_RELEASE      256" in src and L.F_RELEASE == F_RELEASE
    assert "#define EGPU_REL_FLAGGED     1" in src and "#define EGPU_REL_EXCEEDS     2" in src
    assert (L.REL_FLAGGED, L.REL_EXCEEDS) == (release_np.REL_FLAGGED, release_np.REL_EXCEEDS) == (1, 2)
    block = src[src.index(" * Release (flags EGPU_F_RELEASE"):src.index("int egpu_bestfit_batch_dev(")]
    for text in ("EGPU_F_RELEASE [| EGPU_F_COMMIT] [| EGPU_F_PACKED]", "stays 1011", "EGPU_REL_FLAGGED", "EGPU_REL_EXCEEDS",
                 "EGPU_F_INPUTS_READY", "EGPU_ERR_STATE", "egpu_release_refusals"):
        assert text in block, text
    assert "int64_t egpu_release_refusals(egpu_ctx* ctx);" in src


# ---- cases and calls ---------------------------------------------------------------------------------------------
def placed_rows(seed, D, R, packed):
    """R rows and indices whose release is small enough to fit under a table with head-room: about 20 live rows per
    device, the rest (0, 0) rows or rows that hold nothing, of every skipped kind, with values that would show in
    the sums.  int32: (core, mem, idx); packed: (words, None, idx int8)."""
    g = np.random.default_rng(seed)
    core, mem = np.zeros(R, np.int64), np.zeros(R, np.int64)
    idx = g.integers(0, D, R)
    live = g.permutation(R)[:min(R, 20 * D)]
    core[live] = g.integers(0, 3, live.size)
    mem[live] = g.integers(0, 1001, live.size)
    junk = np.setdiff1d(np.arange(R), live)
    junk = junk[g.random(junk.size) < 0.25]
    kind = g.integers(0, 6, junk.size)
    core[junk], mem[junk] = g.integers(1, 101, junk.size), g.integers(1, MEM_MAX + 1, junk.size)
    idx[junk[kind == 0]] = -1
    idx[junk[kind == 1]] = -2
    idx[junk[kind == 2]] = D + g.integers(0, 127 - D + 1, (kind == 2).sum())
    core[junk[kind == 3]] = 101 + g.integers(0, 27, (kind == 3).sum())
    if not packed:
        idx[junk[kind == 2]] += g.integers(0, 2, (kind == 2).sum()) * 100_000
        core[junk[kind == 4]] = -1 - g.integers(0, 1 << 20, (kind == 4).sum())
        mem[junk[kind == 5]] = MEM_MAX + 1 + g.integers(0, 1 << 12, (kind == 5).sum())
        mem[junk[(kind == 5) & (g.random(junk.size) < 0.3)]] = -3
        return core.astype(np.int32), mem.astype(np.int32), idx.astype(np.int32)
    words = ((core << 18) | mem).astype(np.uint32)
    words[junk[kind == 4]] = 0xFFFFFFFF
    words[junk[kind == 5]] = g.integers(1 << 25, 1 << 32, (kind == 5).sum(), dtype=np.uint64).astype(np.uint32)
    return words, None, idx.astype(np.int8)


def requests_of(core, mem):
    """the int32 requests the rows stand for (packed: mem is None and core holds the words)"""
    return release_np.unpack(core) if mem is None else (core, mem)


def table_with_headroom(seed, core, mem, idx, D):
    """a table that accepts the release of the rows, some devices exactly at the domain bound afterwards"""
    g = np.random.default_rng(seed + 7)
    c, m = requests_of(core, mem)
    u, _, _ = release_np.release(np.zeros(D), np.zeros(D), np.zeros(D), c, m, idx)
    fc = (100 - u[:D]) - g.integers(0, 2, D) * g.integers(0, 100 - u[:D] + 1)
    fm = (MEM_MAX - u[D:]) - g.integers(0, 2, D) * g.integers(0, MEM_MAX - u[D:] + 1)
    return fc.astype(np.int32), fm.astype(np.int32)


class Dev:
    """device copies of one call's rows and indices, each followed by GUARD poisoned elements (a full-capacity row on
    device 0: it would show in the sums), and sentinel-filled outputs"""

    def __init__(self, torch, core, mem, idx, D):
        self.torch, self.R, self.D, self.packed = torch, len(core), D, mem is None
        self.h_idx = np.asarray(idx)
        poison_c = np.full(GUARD, (100 << 18) | MEM_MAX if self.packed else 100, core.dtype)
        self.core = torch.from_numpy(np.concatenate([core, poison_c]).view(np.int32)).cuda()
        self.mem = None if self.packed else torch.from_numpy(np.concatenate([mem, np.full(GUARD, MEM_MAX, np.int32)])).cuda()
        self.idx = torch.from_numpy(np.concatenate([self.h_idx, np.zeros(GUARD, self.h_idx.dtype)])).cuda()
        self.delta = torch.full((2 * D,), -1, dtype=torch.int64, device="cuda")
        self.tab = torch.full((3 * D,), -7, dtype=torch.int32, device="cuda")

    def call(self, a, flags, stream=None, delta=True, tab=True):
        s = self.torch.cuda.current_stream().cuda_stream if stream is None else stream
        return a._lib.egpu_bestfit_batch_dev(
            a.handle, C.c_void_p(self.core.data_ptr()), None if self.packed else C.c_void_p(self.mem.data_ptr()), self.R,
            C.c_void_p(self.idx.data_ptr()), C.c_void_p(self.delta.data_ptr()) if delta else None,
            C.c_void_p(self.tab.data_ptr()) if tab else None, flags | (F_PACKED if self.packed else 0), C.c_void_p(1 if s == 0 else s))

    def got(self):
        self.torch.cuda.synchronize()
        idx = self.idx.cpu().numpy()
        assert np.array_equal(idx[:self.R], self.h_idx) and (idx[self.R:] == 0).all(), "the indices are an input"
        return self.delta.cpu().numpy(), self.tab.cpu().numpy()


def release_dev(a, torch, core, mem, idx, D, commit, where):
    """one _dev release checked against the numpy rule: outputs, installed table and flags, one launch"""
    fc, fm, ov = a.table()
    c, m = requests_of(core, mem)
    u, tab, accepted = release_np.release(fc, fm, ov, c, m, idx)
    d = Dev(torch, core, mem, idx, D)
    torch.cuda.synchronize()
    n0 = a.launch_count
    rc = d.call(a, F_RELEASE | (F_COMMIT if commit else 0))
    assert rc == 0, (where, a._lib.egpu_last_error(a.handle).decode())
    assert a.launch_count - n0 == 1, f"{where}: one launch per call"
    g_u, g_tab = d.got()
    assert np.array_equal(g_u, u), f"{where}: sums"
    assert np.array_equal(g_tab, tab), f"{where}: table' and reasons"
    nfc, nfm, nov = a.table()
    exp = (tab[:D], tab[D:2 * D]) if commit and accepted else (fc, fm)
    assert np.array_equal(nfc, exp[0]) and np.array_equal(nfm, exp[1]) and np.array_equal(nov, ov), f"{where}: installed table"
    return accepted


def install(a, fc, fm, ov):
    """the table (fc, fm) with oversubscription flags ov: a flagged device holds (0, 0) and gets there by an
    oversubscribing snapshot commit of two (1, 1) requests, which choose the smallest device"""
    fc, fm, ov = (np.asarray(x, np.int32) for x in (fc, fm, ov))
    flagged = np.flatnonzero(ov)
    assert (fc[flagged] == 0).all() and (fm[flagged] == 0).all() and (fc[ov == 0] != 1).all()
    t_fc, t_fm = fc.copy(), fm.copy()
    t_fc[flagged], t_fm[flagged] = 1, 1
    a.set_table(t_fc, t_fm)
    for _ in flagged:
        a.bestfit([1, 1], [1, 1], commit=True)
    got = a.table()
    assert np.array_equal(got[0], fc) and np.array_equal(got[1], fm) and np.array_equal(got[2], ov)


# ---- 2. known answers --------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["int32", "packed"])
def test_release_known_answers(packed, alloc):
    import torch
    ran = 0
    for k in KATS:
        core, mem, idx = (np.asarray(k[x], np.int64) for x in ("core", "mem", "idx"))
        if packed and ((core < 0) | (core > 127) | (mem < 0) | (mem > MEM_MAX) | (idx > 127)).any():
            continue  # not expressible in words and int8 indices
        install(alloc, k["free_core"], k["free_mem"], k["oversub"])
        D = len(k["free_core"])
        rows = ((core << 18 | mem).astype(np.uint32), None, idx.astype(np.int8)) if packed else \
            (core.astype(np.int32), mem.astype(np.int32), idx.astype(np.int32))
        for commit in (False, True):
            d = Dev(torch, *rows, D)
            assert d.call(alloc, F_RELEASE | (F_COMMIT if commit else 0)) == 0
            u, tab = d.got()
            assert u.tolist() == k["u_core"] + k["u_mem"] and tab.tolist() == k["table_out"], (k["name"], commit)
        fc, fm, ov = alloc.table()
        assert fc.tolist() + fm.tolist() == k["table_out"][:2 * D] and ov.tolist() == k["oversub"], k["name"]
        ran += 1
    assert ran >= (13 if packed else 17)


# ---- 3. parity ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["int32", "packed"])
@pytest.mark.parametrize("D", D_BUCKETS)
def test_release_parity(D, packed, alloc):
    import torch
    for R in ROWS:
        core, mem, idx = placed_rows(100 * D + R, D, R, packed)
        fc, fm = table_with_headroom(R, core, mem, idx, D)
        alloc.set_table(fc, fm)
        assert release_dev(alloc, torch, core, mem, idx, D, False, f"D={D} R={R} dry")
        assert release_dev(alloc, torch, core, mem, idx, D, True, f"D={D} R={R} commit")
        if R >= 513:  # one unit less room: refused wherever a device was exactly at the bound
            alloc.set_table(np.minimum(fc + 1, 100), fm)
            release_dev(alloc, torch, core, mem, idx, D, True, f"D={D} R={R} again")


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["int32", "packed"])
@pytest.mark.parametrize("variant", [AUTO, GRID, SORTED, LUT], ids=["auto", "grid", "sorted", "lut"])
def test_release_under_every_variant(variant, packed, alloc):
    """the release does not depend on the scan variant: it works under EGPU_VARIANT_GRID too"""
    import torch
    alloc.set_variant(variant)
    for D in (8, 64):
        core, mem, idx = placed_rows(5 + D, D, 4099, packed)
        alloc.set_table(*table_with_headroom(3, core, mem, idx, D))
        assert release_dev(alloc, torch, core, mem, idx, D, True, f"variant {variant} D={D}")


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["int32", "packed"])
@pytest.mark.parametrize("D", [8, 64])
def test_release_1mi_rows(D, packed, alloc):
    import torch
    R = (1 << 20) + 1
    core, mem, idx = placed_rows(77 + D, D, R, packed)
    alloc.set_table(*table_with_headroom(1, core, mem, idx, D))
    assert release_dev(alloc, torch, core, mem, idx, D, True, f"1 Mi + 1 rows, D={D}")


# ---- 4. host form ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["int32", "packed"])
@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
def test_release_host_form(pinned, packed, alloc):
    D, R = 17, 4099
    core, mem, idx = placed_rows(9, D, R, packed)
    fc, fm = table_with_headroom(2, core, mem, idx, D)
    alloc.set_table(fc, fm)
    u, tab, accepted = release_np.release(fc, fm, np.zeros(D), *requests_of(core, mem), idx)
    assert accepted
    arrays = [core, mem, idx]
    if pinned:
        for j, x in enumerate(arrays):
            if x is not None:
                arrays[j] = alloc.pinned_array(R, x.dtype)
                arrays[j][:] = x
    keep = arrays[2].copy()
    n0 = alloc.launch_count
    dc, dm = alloc.release(arrays[0], arrays[1], arrays[2], commit=False, packed=packed)
    assert np.array_equal(np.concatenate([dc, dm]), u) and alloc.launch_count - n0 == 1
    assert np.array_equal(alloc.table()[0], fc) and np.array_equal(alloc.table()[1], fm), "dry run"
    dc, dm = alloc.release(arrays[0], arrays[1], arrays[2], packed=packed)
    assert np.array_equal(np.concatenate([dc, dm]), u) and np.array_equal(arrays[2], keep)
    nfc, nfm, nov = alloc.table()
    assert np.array_equal(nfc, tab[:D]) and np.array_equal(nfm, tab[D:2 * D]) and not nov.any()
    # refused: EGPU_ERR_STATE, the first offending device and the reason in egpu_last_error, the sums still written
    alloc.set_table(np.full(D, 100, np.int32), fm)
    r0 = alloc.release_refusals
    with pytest.raises(Exception) as ei:
        alloc.release(arrays[0], arrays[1], arrays[2], packed=packed)
    first = int(np.flatnonzero(u[:D] > 0)[0])
    assert ei.value.code == ERR_STATE and f"device {first} " in str(ei.value) and "EGPU_REL_EXCEEDS" in str(ei.value)
    assert np.array_equal(np.concatenate(ei.value.released), u)
    assert alloc.release_refusals == r0 + 1 and np.array_equal(alloc.table()[1], fm)
    if pinned:
        for x in arrays:
            if x is not None:
                alloc.host_free(x.ctypes.data)


# ---- 5. inverse of the rounds ------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["int32", "packed"])
@pytest.mark.parametrize("D", [8, 64])
def test_release_gives_back_what_rounds_placed(D, packed, alloc, egpu):
    """egpu_table_set(T), rounds in one launch, release of all rows, unfiltered: the table is T again, flags clear;
    the same when the rows go back in three random chunks"""
    import torch
    w = egpu.synth.workload("cfg3" if D == 8 else "cfg4")
    T = (w["free_core"], w["free_mem"])
    rc, rm = egpu.synth.requests(w["dist"], 11, 4099)
    words = egpu.BestFitAllocator.pack_requests(rc, rm)
    for cuts in ([], sorted(np.random.default_rng(D).integers(0, 4099, 2).tolist())):
        alloc.set_table(*T)
        s = torch.cuda.current_stream().cuda_stream
        if packed:
            c = torch.from_numpy(np.concatenate([words, np.zeros(4, np.uint32)]).view(np.int32)).cuda()
            i = torch.full((4099 + 16,), -9, dtype=torch.int8, device="cuda")
            alloc.bestfit_packed_rounds_device_dev(c.data_ptr(), 4099, i.data_ptr(), stream=s)
        else:
            c, m = torch.from_numpy(rc).cuda(), torch.from_numpy(rm).cuda()
            i = torch.full((4099 + 4,), -9, dtype=torch.int32, device="cuda")
            alloc.bestfit_rounds_device_dev(c.data_ptr(), m.data_ptr(), 4099, i.data_ptr(), stream=s)
        torch.cuda.synchronize()
        idx = i.cpu().numpy()[:4099]
        assert (idx >= 0).any() and not np.array_equal(alloc.table()[0], T[0])
        for lo, hi in zip([0] + cuts, cuts + [4099]):
            rows = (words[lo:hi], None, idx[lo:hi]) if packed else (rc[lo:hi], rm[lo:hi], idx[lo:hi])
            assert release_dev(alloc, torch, *rows, D, True, f"chunk {lo}:{hi}")
        fc, fm, ov = alloc.table()
        assert np.array_equal(fc, T[0]) and np.array_equal(fm, T[1]) and not ov.any()
    assert alloc.release_refusals == 0


# ---- 6. sequential mode ------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_release_agrees_with_replayed_frees(alloc, egpu):
    """replay of E ALLOCs and then FREEs of a random subset == replay of the ALLOCs and one release of the subset"""
    import torch
    g = np.random.default_rng(5)
    E = 300
    core, mem = g.integers(1, 30, E).astype(np.int32), g.integers(1, 20000, E).astype(np.int32)
    sub = np.sort(g.permutation(E)[:120]).astype(np.int32)
    fc, fm = egpu.synth.table_full(8)
    alloc.set_table(fc, fm)
    kind = np.concatenate([np.zeros(E, np.int32), np.ones(sub.size, np.int32)])
    alloc.replay(kind, np.concatenate([core, sub]), np.concatenate([mem, np.zeros(sub.size, np.int32)]))
    want = alloc.table()
    alloc.set_table(fc, fm)
    placed = alloc.replay(np.zeros(E, np.int32), core, mem)
    assert (placed == -1).any() and (placed >= 0).any()
    assert release_dev(alloc, torch, core[sub], mem[sub], placed[sub], 8, True, "subset")
    got = alloc.table()
    assert all(np.array_equal(x, y) for x, y in zip(got, want))


# ---- 7. refusals -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["int32", "packed"])
def test_release_refused_on_the_device(packed, alloc):
    """a double release and a flagged device: the table, the flags and the indices stay, the counter counts"""
    import torch
    D = 8
    core, mem, idx = placed_rows(3, D, 513, packed)
    fc, fm = table_with_headroom(4, core, mem, idx, D)
    fc = np.where(fc == 1, 2, fc)  # install() keeps (1, 1) for the devices it flags
    alloc.set_table(fc, fm)
    r0 = alloc.release_refusals
    assert release_dev(alloc, torch, core, mem, idx, D, True, "first")
    u = release_np.release(fc, fm, np.zeros(D), *requests_of(core, mem), idx)[0]
    alloc.set_table(100 - u[:D] + (u[:D] > 0), fm)  # every touched device is one short of room
    assert not release_dev(alloc, torch, core, mem, idx, D, True, "double release")
    assert not release_dev(alloc, torch, core, mem, idx, D, False, "double release, dry")
    assert alloc.release_refusals == r0 + 2
    # a NULL table' and NULL sums: the counter is how an asynchronous caller finds out
    d = Dev(torch, core, mem, idx, D)
    assert d.call(alloc, F_RELEASE | F_COMMIT, delta=False, tab=False) == 0
    assert alloc.release_refusals == r0 + 3
    assert (d.delta.cpu().numpy() == -1).all() and (d.tab.cpu().numpy() == -7).all()
    # flagged: devices 0 and 1 are flagged and hold rows: refused; once the rows avoid them they block nothing
    ov = np.array([1, 1] + [0] * (D - 2), np.int32)
    install(alloc, np.where(ov, 0, 2), np.where(ov, 0, 5), ov)
    assert not release_dev(alloc, torch, core, mem, idx, D, True, "flagged device")
    away = np.where((idx == 0) | (idx == 1), -1, idx).astype(idx.dtype)
    assert release_dev(alloc, torch, core, mem, away, D, True, "flagged but untouched")
    assert alloc.release_refusals == r0 + 4


BAD_FLAGS = [F_RELEASE | F_INPUTS_READY, F_RELEASE | F_PREFIX, F_RELEASE | F_ROUNDS, F_RELEASE | F_DEVICE_ROUNDS, F_RELEASE | F_APPLY,
             F_RELEASE | 64, F_RELEASE | 512, F_RELEASE | DR, F_RELEASE | F_COMMIT | F_PREFIX, F_RELEASE | F_COMMIT | F_INPUTS_READY,
             F_RELEASE | F_PACKED | F_PREFIX, F_RELEASE | F_PACKED | F_ROUNDS, F_RELEASE | F_ROUNDS | F_DEVICE_ROUNDS]


@pytest.mark.gpu
def test_release_refused_on_the_host(alloc, egpu):
    """EGPU_ERR_INVALID before anything is launched or written; EGPU_ERR_NO_TABLE without a table"""
    import torch
    D, R = 8, 516
    core, mem, idx = placed_rows(1, D, R, False)
    words, _, idx8 = placed_rows(1, D, R, True)
    d, p = Dev(torch, core, mem, idx, D), Dev(torch, words, None, idx8, D)
    lib, h = alloc._lib, alloc.handle
    s = C.c_void_p(1)
    assert d.call(alloc, F_RELEASE) == ERR_NO_TABLE
    assert lib.egpu_bestfit_batch(h, C.c_void_p(core.ctypes.data), C.c_void_p(mem.ctypes.data), R, C.c_void_p(idx.ctypes.data), None,
                                  None, F_RELEASE) == ERR_NO_TABLE
    fc, fm = table_with_headroom(4, core, mem, idx, D)
    alloc.set_table(fc, fm)
    n0 = alloc.launch_count

    def dev(c, m, r, i, flags):
        return lib.egpu_bestfit_batch_dev(h, C.c_void_p(c), C.c_void_p(m) if m else None, r, C.c_void_p(i), C.c_void_p(d.delta.data_ptr()),
                                          C.c_void_p(d.tab.data_ptr()), flags, s)
    pc, pm_, pi = d.core.data_ptr(), d.mem.data_ptr(), d.idx.data_ptr()
    for flags in BAD_FLAGS:
        assert d.call(alloc, flags) == ERR_INVALID, flags
        assert p.call(alloc, flags) == ERR_INVALID, flags
        assert lib.egpu_bestfit_batch(h, C.c_void_p(core.ctypes.data), C.c_void_p(mem.ctypes.data), R, C.c_void_p(idx.ctypes.data),
                                      None, None, flags) == ERR_INVALID, flags
    batch = egpu.BestFitAllocator.make_batches([(pc, pm_, R, pi, 0, 0)])
    for flags in (F_RELEASE, F_RELEASE | F_COMMIT, DR | F_RELEASE, F_RELEASE | F_PACKED):
        assert lib.egpu_bestfit_batches_dev(h, batch, 1, flags, s) == ERR_INVALID
    for c, m, r, i, flags in [(0, pm_, R, pi, F_RELEASE), (pc, 0, R, pi, F_RELEASE), (pc, pm_, R, 0, F_RELEASE),
                              (pc + 4, pm_, R, pi, F_RELEASE), (pc, pm_ + 8, R, pi, F_RELEASE), (pc, pm_, R, pi + 4, F_RELEASE),
                              (pc, pm_, 1 << 31, pi, F_RELEASE), (pc, pm_, -1, pi, F_RELEASE),
                              (p.core.data_ptr(), pm_, R, p.idx.data_ptr(), F_RELEASE | F_PACKED),  # packed with a d_req_mem
                              (p.core.data_ptr(), 0, R, p.idx.data_ptr() + 1, F_RELEASE | F_PACKED),
                              (p.core.data_ptr(), 0, 1 << 31, p.idx.data_ptr(), F_RELEASE | F_PACKED)]:
        assert dev(c, m, r, i, flags) == ERR_INVALID, (c, m, r, i, flags)
    # the sums and table' overlap each other
    assert lib.egpu_bestfit_batch_dev(h, C.c_void_p(pc), C.c_void_p(pm_), R, C.c_void_p(pi), C.c_void_p(d.delta.data_ptr()),
                                      C.c_void_p(d.delta.data_ptr() + 8), F_RELEASE, s) == ERR_INVALID
    torch.cuda.synchronize()
    assert alloc.launch_count == n0 and alloc.release_refusals == 0
    assert (d.delta.cpu().numpy() == -1).all() and (d.tab.cpu().numpy() == -7).all()
    got = alloc.table()
    assert np.array_equal(got[0], fc) and np.array_equal(got[1], fm)
    assert d.call(alloc, F_RELEASE | F_COMMIT) == 0 and p.call(alloc, F_RELEASE) == 0  # and the arguments were fine otherwise
    d.got()


# ---- 8. churn tick in a CUDA graph; scans after a release ---------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["int32", "packed"])
def test_release_churn_tick_graph(packed, alloc, egpu, oracle_c):
    """tick t = release of batch t - 2, then admission of batch t by the rounds in one launch, captured once and
    replayed 32 times against a host model built from the oracles: tables and indices are equal every tick"""
    import torch
    D, R = 8, 96
    fc, fm = egpu.synth.table_full(D)
    alloc.set_table(fc, fm)
    dt = torch.int8 if packed else torch.int32
    rel_c, rel_m, adm_c, adm_m = (torch.zeros(R, dtype=torch.int32, device="cuda") for _ in range(4))
    rel_i, adm_i = torch.full((R,), -1, dtype=dt, device="cuda"), torch.full((R,), -9, dtype=dt, device="cuda")
    s = torch.cuda.Stream()

    def tick():
        alloc.release_dev(rel_c.data_ptr(), rel_m.data_ptr(), R, rel_i.data_ptr(), commit=True, packed=packed, stream=s.cuda_stream)
        if packed:
            alloc.bestfit_packed_rounds_device_dev(adm_c.data_ptr(), R, adm_i.data_ptr(), stream=s.cuda_stream)
        else:
            alloc.bestfit_rounds_device_dev(adm_c.data_ptr(), adm_m.data_ptr(), R, adm_i.data_ptr(), stream=s.cuda_stream)
    with torch.cuda.stream(s):
        tick()  # warm-up: occupancy queries and scratch outside the capture (all-zero rows: nothing placed, nothing released)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        tick()
    alloc.set_table(fc, fm)
    m_fc, m_fm = fc.copy(), fm.copy()
    batches = []
    for t in range(32):
        rc, rm = egpu.synth.requests(2, 100 + t, R)
        rc = np.minimum(rc, 50).astype(np.int32)
        if t >= 2:  # the host model: release of batch t - 2 ...
            o_c, o_m, o_i = batches[t - 2]
            u, tab, accepted = release_np.release(m_fc, m_fm, np.zeros(D), o_c, o_m, o_i)
            assert accepted
            m_fc, m_fm = tab[:D].copy(), tab[D:2 * D].copy()
            rel_c.copy_(torch.from_numpy(egpu.BestFitAllocator.pack_requests(o_c, o_m).view(np.int32) if packed else o_c))
            rel_m.copy_(torch.from_numpy(o_m))
            rel_i.copy_(torch.from_numpy(o_i.astype(np.int8 if packed else np.int32)))
        o_idx, _, _, m_fc, m_fm, _, left = oracle_c.rounds(m_fc, m_fm, rc, rm)  # ... then admission of batch t
        assert left == 0
        batches.append((rc, rm, o_idx))
        adm_c.copy_(torch.from_numpy(egpu.BestFitAllocator.pack_requests(rc, rm).view(np.int32) if packed else rc))
        adm_m.copy_(torch.from_numpy(rm))
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(adm_i.cpu().numpy().astype(np.int32), o_idx), f"tick {t}: indices"
        got = alloc.table()
        assert np.array_equal(got[0], m_fc) and np.array_equal(got[1], m_fm) and not got[2].any(), f"tick {t}: table"
    assert any((b[2] == -1).any() for b in batches) and alloc.release_refusals == 0


@pytest.mark.gpu
@pytest.mark.parametrize("variant,D", [(SORTED, 8), (LUT, 8), (SORTED, 64), (LUT, 64), (AUTO, 64)])
def test_scan_after_release_sees_the_released_table(variant, D, alloc, egpu, oracle_c):
    """a committing release refreshes the sorted view and marks the lookup tables stale: a scan after it scores against
    the released table"""
    import torch
    alloc.set_variant(variant)
    core, mem, idx = placed_rows(21, D, 513, False)
    fc, fm = table_with_headroom(6, core, mem, idx, D)
    alloc.set_table(fc, fm)
    rc, rm = egpu.synth.requests(3, 8, 4099)
    alloc.bestfit(rc, rm)  # builds the lookup tables of the table before the release
    assert release_dev(alloc, torch, core, mem, idx, D, True, "release")
    nfc, nfm, _ = alloc.table()
    assert not (np.array_equal(nfc, fc) and np.array_equal(nfm, fm))
    got, dc, dm = alloc.bestfit(rc, rm)
    o_idx, o_dc, o_dm, _ = oracle_c.snapshot(nfc, nfm, rc, rm)
    assert np.array_equal(got, o_idx) and np.array_equal(dc, o_dc) and np.array_equal(dm, o_dm)
