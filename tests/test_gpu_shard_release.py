"""Release over row shards: egpu_bestfit_batch_shard_prefix_dev with EGPU_F_RELEASE [| EGPU_F_COMMIT] [| EGPU_F_PACKED]
(DESIGN.md 2.8).

The result is, bit for bit, the single-GPU EGPU_F_RELEASE of the concatenation of every rank's rows against the table
the ranks share; d_delta is the rank's own sums, d_table_out the same on every rank.  One exchange step per call:

  1. (CPU) the header documents the flag set, the one step and the ABI number; the wrapper passes exactly the flags and
     the step, and a NULL d_req_mem when packed; summing the per-rank release_np sums and deciding once equals
     release_np on the concatenation, for 1 to 8 ranks, with cases where every rank's own sums fit and the total does
     not;
  2. world 1 at every D bucket, ragged row counts and 1 Mi + 1 rows, int32 and packed, dry and committing, under every
     variant, with guard elements: the single-GPU release and release_np on the same rows; the indices are never
     written; one launch per call;
  3. refusals on the device (double release, flagged device, NULL outputs) and on the host (nothing launched or
     written);
  4. the inverse of the sharded rounds; 150 churn ticks past the 256-slot exchange ring; a churn tick replayed from a
     CUDA graph;
  5. world 2 and world 6 (processes on one GPU, started together by the gate after an ungated first run): formats
     mixed, a rank with R = 0, the sum that exceeds only over the ranks, a flagged device touched by one rank, release
     after sharded rounds;
  6. a peer that attaches and never issues the release: the launch gives up on its own, nothing installed.
Every other GPU test ends with egpu_peer_last_timeout == 0.
"""
import ctypes as C
import os
import re
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import release_np  # noqa: E402
import test_gpu_device_rounds as dr  # noqa: E402  (the ctx fixture, Out)
import test_gpu_packed_shard as ps  # noqa: E402  (attach)
import test_gpu_peer_exchange as pe  # noqa: E402  (the prefix-commit table and requests, per-rank sums)
import test_gpu_release as gr  # noqa: E402  (placed_rows, table_with_headroom, Dev, install)
import test_gpu_shard_rounds as sr  # noqa: E402  (the sharded rounds call)

ctx = dr.ctx
ROOT = gr.ROOT
MEM_MAX = gr.MEM_MAX
ERR_INVALID, ERR_NO_TABLE, ERR_STATE = -1, -5, -6
AUTO, GRID, SORTED, LUT = 0, 1, 2, 3
F_COMMIT, F_INPUTS_READY, F_PREFIX, F_APPLY, F_PACKED, F_ROUNDS, F_DEVICE_ROUNDS, F_RELEASE = 1, 2, 4, 8, 16, 32, 128, 256
SR = F_PREFIX | F_COMMIT | F_ROUNDS | F_DEVICE_ROUNDS


# ---- 1. header, wrapper, the rule over ranks ---------------------------------------------------------------------
def test_shard_release_documented():
    src = open(os.path.join(ROOT, "include", "egpu_alloc.h")).read()
    block = src[src.index(" * Release over row shards"):src.index("int egpu_bestfit_batch_shard_prefix_dev(")]
    for phrase in ("EGPU_F_RELEASE [| EGPU_F_COMMIT] [| EGPU_F_PACKED]", "ONE step, `step`", "advances by 1", "stays 1011",
                   "THIS rank's U_g", "identical on every rank", "about 2 s", "step + 1", "R >= 2^31", "step >= 2^47",
                   "EGPU_ERR_STATE", "EGPU_ERR_NO_TABLE", "egpu_release_refusals", "ONE launch", "EGPU_VARIANT_GRID"):
        assert phrase in block, phrase
    define = src[src.index("#define EGPU_F_RELEASE"):src.index("#define EGPU_REL_FLAGGED")]
    assert "egpu_bestfit_batch_shard_prefix_dev only" in define
    assert re.search(r"egpu_bestfit_batches_shard_dev and egpu_bestfit_batch_shard_dev refuse it", define)


def test_wrapper_flags(egpu):
    """release_shard_dev passes exactly the flag set and the step, and a NULL d_req_mem when packed"""
    calls = []

    class Lib:
        def __getattr__(self, name):
            return lambda *a: calls.append((name, a)) or 0

    a = object.__new__(egpu.BestFitAllocator)
    a._lib, a._h = Lib(), C.c_void_p(1)
    a.release_shard_dev(16, 32, 5, 48, 64, 80, step=6)
    a.release_shard_dev(16, 32, 5, 48, step=9, commit=False, packed=True)
    a.release_shard_dev(16, 32, 5, 48, 0, 0, step=(1 << 47) - 1, commit=False)
    assert [n for n, _ in calls] == ["egpu_bestfit_batch_shard_prefix_dev"] * 3
    assert [c[1][7] for c in calls] == [F_RELEASE | F_COMMIT, F_RELEASE | F_PACKED, F_RELEASE]
    assert [c[1][8] for c in calls] == [6, 9, (1 << 47) - 1]
    assert calls[0][1][2].value == 32 and calls[1][1][2] is None and calls[2][1][2].value == 32
    assert calls[0][1][4].value == 48 and calls[0][1][5].value == 64 and calls[0][1][6].value == 80
    assert calls[1][1][5].value is None and calls[1][1][6].value is None
    with pytest.raises(TypeError):
        a.release_shard_dev(16, 32, 5, 48)  # the step is not optional
    a._lib = None
    a._h = None


def requests_of(rows):
    """the int32 requests and indices one rank's rows stand for (packed: the words unpacked, the int8 indices)"""
    core, mem, idx = rows
    c, m = gr.requests_of(core, mem)
    return np.asarray(c, np.int64), np.asarray(m, np.int64), np.asarray(idx, np.int64)


def sharded_release(fc, fm, ov, shards):
    """what every rank computes: its own sums U_g (release_np's sums of its rows), the total pushed and pulled over one
    exchange step, one decision on the total against the rank's table.  (per-rank U_g, table_out, accepted)"""
    D = len(fc)
    own = [release_np.release(np.zeros(D), np.zeros(D), np.zeros(D), *requests_of(s))[0] for s in shards]
    u = np.sum(own, axis=0) if own else np.zeros(2 * D, np.int64)
    fc, fm, ov = (np.asarray(x, np.int64) for x in (fc, fm, ov))
    touched = (u[:D] > 0) | (u[D:] > 0)
    reason = np.where(touched & (ov != 0), release_np.REL_FLAGGED,
                      np.where(touched & ((fc + u[:D] > release_np.CORE_MAX) | (fm + u[D:] > MEM_MAX)), release_np.REL_EXCEEDS, 0))
    accepted = not reason.any()
    nc, nm = (fc + u[:D], fm + u[D:]) if accepted else (fc, fm)
    return own, np.concatenate([nc, nm, reason]).astype(np.int32), accepted


def concat(shards):
    parts = [requests_of(s) for s in shards]
    return tuple(np.concatenate([p[j] for p in parts]) for j in range(3))


def world_cases(world, formats, D=8):
    """[(name, (fc, fm, ov), rows of every rank, commit, accepted)] of a release over `world` ranks; rank g's rows are
    placed_rows in formats[g % len(formats)] (True = packed), thinned above two ranks so the sum stays in the domain"""
    def rows(seed, counts):
        out = []
        for g, R in enumerate(counts):
            core, mem, idx = gr.placed_rows(seed + g, D, R, formats[g % len(formats)])
            if world > 2:
                idx = np.where(np.random.default_rng(seed + 50 + g).random(R) < 1 - 2 / world, -1, idx).astype(idx.dtype)
            out.append((core, mem, idx))
        return out

    def headroom(seed, shards):
        c, m, i = concat(shards)
        u = release_np.release(np.zeros(D), np.zeros(D), np.zeros(D), c, m, i)[0]
        assert u[:D].max() <= release_np.CORE_MAX and u[D:].max() <= MEM_MAX
        return gr.table_with_headroom(seed, c.astype(np.int32), m.astype(np.int32), i, D)

    zero = np.zeros(D, np.int32)
    cases = []
    ragged = [(513, 4099, 3, 1, 1500, 4, 0, 77)[g % 8] for g in range(world)]
    s = rows(10, ragged)
    cases.append(("ragged", (*headroom(1, s), zero), s, True))
    s = rows(20, ragged[::-1])
    cases.append(("dry", (*headroom(2, s), zero), s, False))
    s = rows(30, [0] + [4099] * (world - 1))
    cases.append(("rank 0 empty", (*headroom(3, s), zero), s, True))
    # every rank's own sums fit, the total exceeds on the devices every rank touches: refused on every rank
    s = rows(40, [4099] * world)
    fc, fm = headroom(4, s)
    own = [release_np.release(zero, zero, zero, *requests_of(x))[0] for x in s]
    tight = np.all([o[:D] > 0 for o in own], axis=0)
    assert tight.any()
    fc = np.where(tight, release_np.CORE_MAX - np.sum(own, axis=0)[:D] + 1, fc).astype(np.int32)
    for x in s if world > 1 else []:
        assert release_np.release(fc, fm, zero, *requests_of(x))[2], "one rank's own sums fit"
    cases.append(("sum exceeds", (fc, fm, zero), s, True))
    # a flagged device touched by the last rank's rows only
    s = rows(50, [513] * world)
    fc, fm = headroom(5, s)
    flag = int(np.flatnonzero(release_np.release(zero, zero, zero, *requests_of(s[-1]))[0][:D] > 0)[0])
    s = [(c, m, np.where(i == flag, -1, i).astype(i.dtype)) if g < world - 1 else (c, m, i) for g, (c, m, i) in enumerate(s)]
    ov = (np.arange(D) == flag).astype(np.int32)
    fc, fm = np.where(ov, 0, np.where(fc == 1, 2, fc)).astype(np.int32), np.where(ov, 0, fm).astype(np.int32)
    cases.append(("flagged, last rank only", (fc, fm, ov), s, True))
    return [(name, t, s, commit, sharded_release(*t, s)[2]) for name, t, s, commit in cases]


@pytest.mark.parametrize("world", range(1, 9))
def test_sum_then_decide_equals_release_of_the_concatenation(world):
    """sums over rows are order-free: the total of the per-rank sums, decided once, is release_np of the concatenation"""
    rng = np.random.default_rng(world)
    formats = [bool(rng.integers(0, 2)) for _ in range(world)]
    outcomes = {}
    for name, (fc, fm, ov), shards, _, accepted in world_cases(world, formats):
        own, tab, acc = sharded_release(fc, fm, ov, shards)
        u, e_tab, e_acc = release_np.release(fc, fm, ov, *concat(shards))
        assert np.array_equal(np.sum(own, axis=0), u) and np.array_equal(tab, e_tab) and acc == e_acc == accepted, name
        outcomes[name] = (accepted, set(tab[2 * len(fc):].tolist()))
    assert outcomes["ragged"][0] and outcomes["dry"][0] and outcomes["rank 0 empty"][0]
    assert not outcomes["sum exceeds"][0] and release_np.REL_EXCEEDS in outcomes["sum exceeds"][1]
    assert outcomes["sum exceeds"][1] <= {0, release_np.REL_EXCEEDS}
    assert outcomes["flagged, last rank only"][0] is False and release_np.REL_FLAGGED in outcomes["flagged, last rank only"][1]


# ---- calls -------------------------------------------------------------------------------------------------------
def shard_call(a, d, flags, step, stream=None, delta=True, tab=True):
    """the sharded release of gr.Dev d's rows (its arrays, guard elements and sentinel outputs)"""
    s = d.torch.cuda.current_stream().cuda_stream if stream is None else stream
    return a._lib.egpu_bestfit_batch_shard_prefix_dev(
        a.handle, C.c_void_p(d.core.data_ptr()), None if d.packed else C.c_void_p(d.mem.data_ptr()), d.R,
        C.c_void_p(d.idx.data_ptr()), C.c_void_p(d.delta.data_ptr()) if delta else None,
        C.c_void_p(d.tab.data_ptr()) if tab else None, flags | (F_PACKED if d.packed else 0), step, C.c_void_p(1 if s == 0 else s))


def release_both(a, torch, core, mem, idx, D, commit, step, where):
    """the single-GPU release, then (same table) the world-1 sharded release on the same rows: the same sums, table',
    installed table, both equal to release_np; one launch each; the indices stay as they were"""
    fc, fm, ov = a.table()
    assert not ov.any()
    u, tab, accepted = release_np.release(fc, fm, ov, *gr.requests_of(core, mem), idx)
    flags = F_RELEASE | (F_COMMIT if commit else 0)
    one, sh = gr.Dev(torch, core, mem, idx, D), gr.Dev(torch, core, mem, idx, D)
    torch.cuda.synchronize()
    assert one.call(a, flags) == 0
    g1 = one.got() + (a.table(),)
    a.set_table(fc, fm)
    torch.cuda.synchronize()
    n0 = a.launch_count
    assert shard_call(a, sh, flags, step) == 0, (where, a._lib.egpu_last_error(a.handle).decode())
    assert a.launch_count - n0 == 1, f"{where}: one launch per call"
    g2 = sh.got() + (a.table(),)
    assert np.array_equal(g2[0], u) and np.array_equal(g2[1], tab), f"{where}: sums and table' against release_np"
    exp = (tab[:D], tab[D:2 * D]) if commit and accepted else (fc, fm)
    assert np.array_equal(g2[2][0], exp[0]) and np.array_equal(g2[2][1], exp[1]) and not g2[2][2].any(), f"{where}: installed"
    assert all(np.array_equal(x, y) for x, y in zip(g1[:2], g2[:2])), f"{where}: differs from the single-GPU release"
    assert all(np.array_equal(x, y) for x, y in zip(g1[2], g2[2])), f"{where}: installed table differs from the single-GPU one"
    return accepted


# ---- 2. world 1 --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["int32", "packed"])
@pytest.mark.parametrize("D", gr.D_BUCKETS)
def test_shard_release_world1_parity(D, packed, ctx):
    import torch
    ps.attach(ctx)
    step = 0
    for R in gr.ROWS:
        core, mem, idx = gr.placed_rows(100 * D + R, D, R, packed)
        fc, fm = gr.table_with_headroom(R, core, mem, idx, D)
        ctx.set_table(fc, fm)
        assert release_both(ctx, torch, core, mem, idx, D, False, step, f"D={D} R={R} dry")
        assert release_both(ctx, torch, core, mem, idx, D, True, step + 1, f"D={D} R={R} commit")
        step += 2
        if R >= 513:  # one unit less room: refused wherever a device was exactly at the bound
            ctx.set_table(np.minimum(fc + 1, 100), fm)
            release_both(ctx, torch, core, mem, idx, D, True, step, f"D={D} R={R} again")
            step += 1
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["int32", "packed"])
@pytest.mark.parametrize("variant", [AUTO, GRID, SORTED, LUT], ids=["auto", "grid", "sorted", "lut"])
def test_shard_release_under_every_variant(variant, packed, ctx):
    """like the single-GPU release, the sharded one does not depend on the scan variant: accepted under GRID too"""
    import torch
    ctx.set_variant(variant)
    ps.attach(ctx)
    for k, D in enumerate((8, 64)):
        core, mem, idx = gr.placed_rows(5 + D, D, 4099, packed)
        ctx.set_table(*gr.table_with_headroom(3, core, mem, idx, D))
        assert release_both(ctx, torch, core, mem, idx, D, True, k, f"variant {variant} D={D}")
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


@pytest.mark.gpu
@pytest.mark.parametrize("D,packed", [(8, False), (64, True)], ids=["d8-int32", "d64-packed"])
def test_shard_release_1mi_rows(D, packed, ctx):
    import torch
    R = (1 << 20) + 1
    core, mem, idx = gr.placed_rows(77 + D, D, R, packed)
    ps.attach(ctx)
    ctx.set_table(*gr.table_with_headroom(1, core, mem, idx, D))
    assert release_both(ctx, torch, core, mem, idx, D, True, 5, f"1 Mi + 1 rows, D={D}")
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


# ---- 3. refusals -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["int32", "packed"])
def test_shard_release_refused_on_the_device(packed, ctx):
    """a double release, a NULL table' and sums, a flagged device: the table, the flags and the indices stay, the
    counter counts"""
    import torch
    D = 8
    core, mem, idx = gr.placed_rows(3, D, 513, packed)
    fc, fm = gr.table_with_headroom(4, core, mem, idx, D)
    fc = np.where(fc == 1, 2, fc)  # install() keeps (1, 1) for the devices it flags
    ps.attach(ctx)
    ctx.set_table(fc, fm)
    r0 = ctx.release_refusals
    assert release_both(ctx, torch, core, mem, idx, D, True, 0, "first")
    u = release_np.release(fc, fm, np.zeros(D), *gr.requests_of(core, mem), idx)[0]
    ctx.set_table(100 - u[:D] + (u[:D] > 0), fm)  # every touched device is one short of room
    assert not release_both(ctx, torch, core, mem, idx, D, True, 1, "double release")
    assert not release_both(ctx, torch, core, mem, idx, D, False, 2, "double release, dry")
    assert ctx.release_refusals == r0 + 4  # each of the two calls: the single-GPU one and the sharded one
    d = gr.Dev(torch, core, mem, idx, D)
    assert shard_call(ctx, d, F_RELEASE | F_COMMIT, 3, delta=False, tab=False) == 0
    assert ctx.release_refusals == r0 + 5
    assert (d.delta.cpu().numpy() == -1).all() and (d.tab.cpu().numpy() == -7).all()
    d.got()
    # flagged: devices 0 and 1 are flagged and hold rows: refused; once the rows avoid them they block nothing
    ov = np.array([1, 1] + [0] * (D - 2), np.int32)
    for step, rows_idx, accepted in ((4, idx, False), (5, np.where((idx == 0) | (idx == 1), -1, idx).astype(idx.dtype), True)):
        gr.install(ctx, np.where(ov, 0, 2), np.where(ov, 0, 5), ov)
        before = ctx.table()
        e_u, e_tab, e_acc = release_np.release(*before, *gr.requests_of(core, mem), rows_idx)
        d = gr.Dev(torch, core, mem, rows_idx, D)
        assert shard_call(ctx, d, F_RELEASE | F_COMMIT, step) == 0
        g_u, g_tab = d.got()
        assert e_acc == accepted and np.array_equal(g_u, e_u) and np.array_equal(g_tab, e_tab), f"flagged, step {step}"
        after = ctx.table()
        assert np.array_equal(after[2], ov)
        assert all(np.array_equal(x, y) for x, y in zip(after[:2], (e_tab[:D], e_tab[D:2 * D]) if accepted else before[:2]))
    assert ctx.release_refusals == r0 + 6
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


BAD_FLAGS = [F_RELEASE | F_INPUTS_READY, F_RELEASE | F_PREFIX, F_RELEASE | F_ROUNDS, F_RELEASE | F_DEVICE_ROUNDS, F_RELEASE | F_APPLY,
             F_RELEASE | 64, F_RELEASE | 512, F_RELEASE | SR, F_RELEASE | F_COMMIT | F_PREFIX, F_RELEASE | F_COMMIT | F_INPUTS_READY,
             F_RELEASE | F_PACKED | F_PREFIX, F_RELEASE | F_PACKED | F_ROUNDS, F_RELEASE | F_ROUNDS | F_DEVICE_ROUNDS]


@pytest.mark.gpu
def test_shard_release_refused_on_the_host(ctx, egpu):
    """EGPU_ERR_INVALID before anything is launched or written; EGPU_ERR_NO_TABLE without a table, EGPU_ERR_STATE
    unattached; the K-batch sharded call keeps refusing the flag"""
    import torch
    D, R = 8, 516
    core, mem, idx = gr.placed_rows(1, D, R, False)
    words, _, idx8 = gr.placed_rows(1, D, R, True)
    d, p = gr.Dev(torch, core, mem, idx, D), gr.Dev(torch, words, None, idx8, D)
    lib, h = ctx._lib, ctx.handle
    s = C.c_void_p(1)
    assert shard_call(ctx, d, F_RELEASE, 0) == ERR_NO_TABLE and shard_call(ctx, p, F_RELEASE, 0) == ERR_NO_TABLE
    fc, fm = gr.table_with_headroom(4, core, mem, idx, D)
    ctx.set_table(fc, fm)
    assert shard_call(ctx, d, F_RELEASE | F_COMMIT, 0) == ERR_STATE and shard_call(ctx, p, F_RELEASE, 0) == ERR_STATE
    ps.attach(ctx)
    torch.cuda.synchronize()
    n0 = ctx.launch_count

    def raw(c, m, r, i, flags, step=0, dl=None, tb=None):
        return lib.egpu_bestfit_batch_shard_prefix_dev(h, C.c_void_p(c), C.c_void_p(m) if m else None, r, C.c_void_p(i),
                                                       C.c_void_p(dl or d.delta.data_ptr()), C.c_void_p(tb or d.tab.data_ptr()),
                                                       flags, step, s)
    for flags in BAD_FLAGS:
        assert shard_call(ctx, d, flags, 0) == ERR_INVALID, flags
        assert shard_call(ctx, p, flags, 0) == ERR_INVALID, flags
    pc, pm_, pi = d.core.data_ptr(), d.mem.data_ptr(), d.idx.data_ptr()
    wc, wi = p.core.data_ptr(), p.idx.data_ptr()
    for c, m, r, i, flags, step in [(0, pm_, R, pi, F_RELEASE, 0), (pc, 0, R, pi, F_RELEASE, 0), (pc, pm_, R, 0, F_RELEASE, 0),
                                    (pc + 4, pm_, R, pi, F_RELEASE, 0), (pc, pm_ + 8, R, pi, F_RELEASE, 0),
                                    (pc, pm_, R, pi + 4, F_RELEASE, 0), (pc, pm_, 1 << 31, pi, F_RELEASE, 0),
                                    (pc, pm_, -1, pi, F_RELEASE, 0), (pc, pm_, R, pi, F_RELEASE, 1 << 47),
                                    (pc, pm_, R, pi, F_RELEASE | F_COMMIT, (1 << 64) - 1),
                                    (wc, pm_, R, wi, F_RELEASE | F_PACKED, 0),  # packed with a d_req_mem
                                    (0, 0, R, wi, F_RELEASE | F_PACKED, 0), (wc, 0, R, 0, F_RELEASE | F_PACKED, 0),
                                    (wc + 4, 0, R, wi, F_RELEASE | F_PACKED, 0), (wc, 0, R, wi + 1, F_RELEASE | F_PACKED, 0),
                                    (wc, 0, 1 << 31, wi, F_RELEASE | F_PACKED, 0), (wc, 0, R, wi, F_RELEASE | F_PACKED, 1 << 47)]:
        assert raw(c, m, r, i, flags, step) == ERR_INVALID, (c, m, r, i, flags, step)
    # the sums and table' overlap each other
    assert raw(pc, pm_, R, pi, F_RELEASE, 0, d.delta.data_ptr(), d.delta.data_ptr() + 8) == ERR_INVALID
    assert raw(wc, 0, R, wi, F_RELEASE | F_PACKED, 0, d.tab.data_ptr() + 4, d.tab.data_ptr()) == ERR_INVALID
    # the K-batch sharded form keeps refusing the flag
    batch = egpu.BestFitAllocator.make_batches([(pc, pm_, R, pi, d.delta.data_ptr(), d.tab.data_ptr())])
    pbatch = egpu.BestFitAllocator.make_batches([(wc, 0, R, wi, d.delta.data_ptr(), d.tab.data_ptr())])
    for flags in (F_RELEASE, F_RELEASE | F_COMMIT):
        assert lib.egpu_bestfit_batches_shard_dev(h, batch, 1, flags, 0, s) == ERR_INVALID, flags
        assert lib.egpu_bestfit_batches_shard_dev(h, pbatch, 1, flags | F_PACKED, 0, s) == ERR_INVALID, flags
    torch.cuda.synchronize()
    assert ctx.launch_count == n0 and ctx.release_refusals == 0
    for x in (d, p):
        assert (x.delta.cpu().numpy() == -1).all() and (x.tab.cpu().numpy() == -7).all()
    got = ctx.table()
    assert np.array_equal(got[0], fc) and np.array_equal(got[1], fm)
    # the arguments were fine otherwise; the last accepted step is 2^47 - 1
    assert shard_call(ctx, d, F_RELEASE | F_COMMIT, (1 << 47) - 1) == 0 and shard_call(ctx, p, F_RELEASE, 0) == 0
    d.got(), p.got()
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


# ---- 4. with the sharded rounds: inverse, past the ring, graph ---------------------------------------------------
def rounds_rows(torch, rc, rm, packed):
    """(d_req_core, d_req_mem or None) of the sharded rounds"""
    c, m, _ = sr.rows_in(torch, rc, rm, 0, packed, oddities=False)
    return c, m


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["int32", "packed"])
@pytest.mark.parametrize("D", [8, 64])
def test_shard_release_gives_back_what_sharded_rounds_placed(D, packed, ctx, egpu):
    """egpu_table_set(T), sharded rounds in one launch, sharded release of all rows, unfiltered: the table is T again,
    flags clear; the same when the rows go back in three random chunks"""
    import torch
    w = egpu.synth.workload("cfg3" if D == 8 else "cfg4")
    T = (np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32))
    rc, rm = egpu.synth.requests(w["dist"], 11, 4099)
    words = egpu.BestFitAllocator.pack_requests(rc, rm)
    ps.attach(ctx)
    step = 0
    for cuts in ([], sorted(np.random.default_rng(D).integers(0, 4099, 2).tolist())):
        ctx.set_table(*T)
        c, m = rounds_rows(torch, rc, rm, packed)
        o = dr.Out(torch, 4099, D, packed)
        sr.shard_call(ctx, torch, c, m, o, step)
        step += 2
        torch.cuda.synchronize()
        idx = o.got()[0]
        assert (idx >= 0).any() and not np.array_equal(ctx.table()[0], T[0])
        for lo, hi in zip([0] + cuts, cuts + [4099]):
            rows = (words[lo:hi], None, idx[lo:hi].astype(np.int8)) if packed else (rc[lo:hi], rm[lo:hi], idx[lo:hi])
            fc, fm, _ = ctx.table()
            u, tab, accepted = release_np.release(fc, fm, np.zeros(D), *gr.requests_of(rows[0], rows[1]), rows[2])
            d = gr.Dev(torch, *rows, D)
            assert shard_call(ctx, d, F_RELEASE | F_COMMIT, step) == 0
            step += 1
            g_u, g_tab = d.got()
            assert accepted and np.array_equal(g_u, u) and np.array_equal(g_tab, tab), f"chunk {lo}:{hi}"
        nfc, nfm, ov = ctx.table()
        assert np.array_equal(nfc, T[0]) and np.array_equal(nfm, T[1]) and not ov.any()
    assert ctx.release_refusals == 0 and ctx.peer_last_timeout == 0
    ctx.peer_detach()


class Tick:
    """the device buffers of one churn tick: the rows released (a batch placed two ticks before) and the rows admitted"""

    def __init__(self, torch, R, D, packed):
        dt = torch.int8 if packed else torch.int32
        self.torch, self.R, self.packed = torch, R, packed
        self.rel_c, self.rel_m, self.adm_c, self.adm_m = (torch.zeros(R, dtype=torch.int32, device="cuda") for _ in range(4))
        self.rel_i, self.adm_i = torch.full((R,), -1, dtype=dt, device="cuda"), torch.full((R,), -9, dtype=dt, device="cuda")
        self.rel_delta, self.adm_delta = (torch.zeros(2 * D, dtype=torch.int64, device="cuda") for _ in range(2))
        self.rel_tab, self.adm_tab = (torch.zeros(3 * D, dtype=torch.int32, device="cuda") for _ in range(2))

    def issue(self, a, step, s):
        """sharded release on `step`, sharded rounds on step + 1 and step + 2: the caller advances by 3"""
        a.release_shard_dev(self.rel_c.data_ptr(), self.rel_m.data_ptr(), self.R, self.rel_i.data_ptr(), self.rel_delta.data_ptr(),
                            self.rel_tab.data_ptr(), step=step, packed=self.packed, stream=s)
        a.bestfit_shard_rounds_dev(self.adm_c.data_ptr(), self.adm_m.data_ptr(), self.R, self.adm_i.data_ptr(),
                                   self.adm_delta.data_ptr(), self.adm_tab.data_ptr(), step + 1, packed=self.packed, stream=s)

    def set_rows(self, egpu, rel, adm):
        torch = self.torch
        pack = egpu.BestFitAllocator.pack_requests
        o_c, o_m, o_i = rel
        self.rel_c.copy_(torch.from_numpy(pack(o_c, o_m).view(np.int32) if self.packed else o_c))
        self.rel_m.copy_(torch.from_numpy(o_m))
        self.rel_i.copy_(torch.from_numpy(o_i.astype(np.int8 if self.packed else np.int32)))
        rc, rm = adm
        self.adm_c.copy_(torch.from_numpy(pack(rc, rm).view(np.int32) if self.packed else rc))
        self.adm_m.copy_(torch.from_numpy(rm))


def churn_model(egpu, oracle_c, fc, fm, n, R, seed):
    """the host model of n churn ticks from the oracles: tick t releases batch t - 2 (release_np) and admits batch t
    (the rounds oracle).  Per tick: (released rows, admitted rows, release sums, table after the release, admitted
    indices, admitted sums, table after the rounds)"""
    D = len(fc)
    m_fc, m_fm = fc.copy(), fm.copy()
    batches, ticks = [], []
    empty = (np.zeros(R, np.int32), np.zeros(R, np.int32), np.full(R, -1, np.int32))
    for t in range(n):
        rc, rm = egpu.synth.requests(2, seed + t, R)
        rc = np.minimum(rc, 50).astype(np.int32)
        rel = batches[t - 2] if t >= 2 else empty
        u, tab, accepted = release_np.release(m_fc, m_fm, np.zeros(D), *rel)
        assert accepted
        m_fc, m_fm = tab[:D].copy(), tab[D:2 * D].copy()
        o_idx, o_dc, o_dm, m_fc, m_fm, _, left = oracle_c.rounds(m_fc, m_fm, rc, rm)
        assert left == 0
        batches.append((rc, rm, o_idx))
        ticks.append((rel, (rc, rm), u, tab, o_idx, np.concatenate([o_dc, o_dm]),
                      np.concatenate([m_fc, m_fm, np.zeros(D, np.int32)]).astype(np.int32)))
    return ticks


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["int32", "packed"])
def test_shard_release_past_the_ring(packed, ctx, egpu, oracle_c):
    """150 churn ticks on one stream, each a sharded release (one step) and sharded rounds (two steps): 450 exchange
    steps, more than the 256 slots; every tick's outputs against the host model"""
    import torch
    D, R, n = 8, 64, 150
    fc, fm = egpu.synth.table_full(D)
    model = churn_model(egpu, oracle_c, fc, fm, n, R, 500)
    ps.attach(ctx)
    ctx.set_table(fc, fm)
    ticks = []
    for rel, adm, *_ in model:
        k = Tick(torch, R, D, packed)
        k.set_rows(egpu, rel, adm)
        ticks.append(k)
    torch.cuda.synchronize()
    s = torch.cuda.current_stream().cuda_stream
    for t, k in enumerate(ticks):
        k.issue(ctx, 3 * t, s)
    torch.cuda.synchronize()
    for t, (k, (_, _, u, tab, o_idx, o_d, o_tab)) in enumerate(zip(ticks, model)):
        assert np.array_equal(k.rel_delta.cpu().numpy(), u) and np.array_equal(k.rel_tab.cpu().numpy(), tab), f"tick {t}: release"
        assert np.array_equal(k.adm_i.cpu().numpy().astype(np.int32), o_idx), f"tick {t}: indices"
        assert np.array_equal(k.adm_delta.cpu().numpy(), o_d) and np.array_equal(k.adm_tab.cpu().numpy(), o_tab), f"tick {t}: rounds"
    got = ctx.table()
    assert np.array_equal(got[0], model[-1][6][:D]) and np.array_equal(got[1], model[-1][6][D:2 * D]) and not got[2].any()
    assert any((m[4] == -1).any() for m in model) and ctx.release_refusals == 0
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True], ids=["int32", "packed"])
def test_shard_release_churn_tick_graph(packed, ctx, egpu, oracle_c):
    """one churn tick (sharded release on step 0, sharded rounds on steps 1 and 2) captured once and replayed 32 times:
    tables and indices equal the host model every tick"""
    import torch
    D, R = 8, 96
    fc, fm = egpu.synth.table_full(D)
    model = churn_model(egpu, oracle_c, fc, fm, 32, R, 100)
    ps.attach(ctx)
    ctx.set_table(fc, fm)
    k = Tick(torch, R, D, packed)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        k.issue(ctx, 0, s.cuda_stream)  # warm-up: occupancy queries and scratch outside the capture (all-zero rows)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        k.issue(ctx, 0, s.cuda_stream)
    ctx.set_table(fc, fm)
    for t, (rel, adm, u, tab, o_idx, o_d, o_tab) in enumerate(model):
        k.set_rows(egpu, rel, adm)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(k.rel_delta.cpu().numpy(), u) and np.array_equal(k.rel_tab.cpu().numpy(), tab), f"tick {t}: release"
        assert np.array_equal(k.adm_i.cpu().numpy().astype(np.int32), o_idx), f"tick {t}: indices"
        got = ctx.table()
        assert np.array_equal(got[0], o_tab[:D]) and np.array_equal(got[1], o_tab[D:2 * D]) and not got[2].any(), f"tick {t}: table"
    assert any((m[4] == -1).any() for m in model) and ctx.release_refusals == 0
    assert ctx.peer_last_timeout == 0
    ctx.peer_detach()


# ---- 5. several processes on one GPU -----------------------------------------------------------------------------
W_FORMATS = [(False, False), (True, True), (True, False)]


def _rank_main(rank, world, conn, formats):
    """One of `world` processes on cuda:0; the parent relays the IPC handles.  Every case of world_cases from its own
    table, twice: once as a warm-up, then each call started together with the other ranks through the gate (nothing
    between gate_dev and gate_open may launch a kernel for the first time: see test_gpu_shard_rounds).  At world 2,
    then the sharded rounds of the prefix-commit requests and the release of what they placed."""
    sys.path.insert(0, ROOT)
    import torch
    import elastic_gpu_agent_b200 as e
    torch.cuda.set_device(0)
    D = 8
    a = e.BestFitAllocator(0)
    a.set_table(np.full(D, 100, np.int32), np.full(D, MEM_MAX, np.int32))
    conn.send(a.peer_export())
    a.peer_attach(rank, world, conn.recv())
    conn.send("attached")
    assert conn.recv() == "go"
    s = torch.cuda.current_stream().cuda_stream
    cases = world_cases(world, formats)
    devs = [gr.Dev(torch, *shards[rank], D) for _, _, shards, _, _ in cases]
    step, res = 0, []
    for gated in (False, True):
        out = []
        for (name, (fc, fm, ov), _, commit, _), d in zip(cases, devs):
            if ov.any():
                gr.install(a, fc, fm, ov)
            else:
                a.set_table(fc, fm)
            d.delta.fill_(-1), d.tab.fill_(-7)
            torch.cuda.synchronize()
            if gated:
                a.gate_dev(s)
            rc = shard_call(a, d, F_RELEASE | (F_COMMIT if commit else 0), step, s)
            if gated:
                a.gate_open()
            step += 1
            out.append((rc,) + d.got() + (a.table(),))
        res.append(out)
    after = None
    if world == 2:  # release after sharded rounds: back to the start table
        rc_all, rm_all = pe._prefix_requests(5000, 800)
        rc, rm = (rc_all[:300], rm_all[:300]) if rank == 0 else (rc_all[300:], rm_all[300:])
        rc, rm = np.ascontiguousarray(rc), np.ascontiguousarray(rm)
        a.set_table(pe.PREFIX_FC, pe.PREFIX_FM)
        c, m = rounds_rows(torch, rc, rm, False)
        o = dr.Out(torch, rc.size, pe.PREFIX_FC.size, False)
        torch.cuda.synchronize()
        sr.shard_call(a, torch, c, m, o, step, s)
        torch.cuda.synchronize()
        idx = o.got()[0]
        placed = a.table()
        packed = formats[rank % len(formats)]
        rows = (e.BestFitAllocator.pack_requests(rc, rm), None, idx.astype(np.int8)) if packed else (rc, rm, idx)
        d = gr.Dev(torch, *rows, pe.PREFIX_FC.size)
        torch.cuda.synchronize()
        a.gate_dev(s)
        assert shard_call(a, d, F_RELEASE | F_COMMIT, step + 2, s) == 0
        a.gate_open()
        after = (idx, placed, d.got(), a.table())
    conn.send((rank, res, after, a.peer_last_timeout, a.gate_timeouts, a.release_refusals))
    assert conn.recv() == "done"
    a.peer_detach()
    a.close()


def run_world(world, formats):
    import torch.multiprocessing as mp
    mctx = mp.get_context("spawn")
    conns, procs = [], []
    for rank in range(world):
        parent, child = mctx.Pipe()
        p = mctx.Process(target=_rank_main, args=(rank, world, child, formats))
        p.start()
        conns.append(parent)
        procs.append(p)
    try:
        assert all(c.poll(240) for c in conns), "ranks did not come up"
        handles = [c.recv() for c in conns]
        for c in conns:
            c.send(handles)
        assert all(c.poll(120) and c.recv() == "attached" for c in conns)
        for c in conns:
            c.send("go")
        assert all(c.poll(300) for c in conns), "ranks did not finish"
        res = sorted((c.recv() for c in conns), key=lambda r: r[0])
        for c in conns:
            c.send("done")
        for p in procs:
            p.join(60)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
    assert all(p.exitcode == 0 for p in procs)
    return res


def check_world(world, formats, res, oracle_c):
    D = 8
    for r in res:
        assert r[3] == 0, f"rank {r[0]}: a peer pull timed out at step + 1 = {r[3]}"
        assert r[4] == 0, f"rank {r[0]}: the start gate timed out"
    cases = world_cases(world, formats)
    refused = 0
    for k, (name, (fc, fm, ov), shards, commit, accepted) in enumerate(cases):
        u, tab, e_acc = release_np.release(fc, fm, ov, *concat(shards))
        own, s_tab, _ = sharded_release(fc, fm, ov, shards)
        assert e_acc == accepted and np.array_equal(s_tab, tab)
        inst = (tab[:D], tab[D:2 * D]) if commit and accepted else (fc, fm)
        refused += 0 if accepted else 1
        for p, where in enumerate(("warm-up", "gated")):
            for g, r in enumerate(res):
                rc, g_u, g_tab, g_table = r[1][p][k]
                at = f"{where}, {name}, rank {g}"
                assert rc == 0, at
                assert np.array_equal(g_u, own[g]), f"{at}: this rank's sums"
                assert np.array_equal(g_tab, tab), f"{at}: table' and reasons"
                assert np.array_equal(g_table[0], inst[0]) and np.array_equal(g_table[1], inst[1]), f"{at}: installed table"
                assert np.array_equal(g_table[2], ov), f"{at}: flags"
        if name == "sum exceeds":
            assert release_np.REL_EXCEEDS in tab[2 * D:] and set(tab[2 * D:].tolist()) <= {0, release_np.REL_EXCEEDS}
        if name.startswith("flagged"):
            assert (tab[2 * D:] == release_np.REL_FLAGGED).sum() == 1
    for r in res:
        assert r[5] == 2 * refused, f"rank {r[0]}: refusals"
    if world == 2:
        rc_all, rm_all = pe._prefix_requests(5000, 800)
        o_idx = dr.ref(oracle_c, pe.PREFIX_FC, pe.PREFIX_FM, rc_all, rm_all)[0]
        for g, r in enumerate(res):
            idx, placed, (g_u, g_tab), table = r[2]
            lo, hi = (0, 300) if g == 0 else (300, 800)
            assert np.array_equal(idx, o_idx[lo:hi]), f"rank {g}: sharded rounds"
            assert np.array_equal(g_u, pe._rank_partial(idx, rc_all[lo:hi], rm_all[lo:hi], D)), f"rank {g}: release sums"
            assert np.array_equal(g_tab, np.concatenate([pe.PREFIX_FC, pe.PREFIX_FM, np.zeros(D, np.int32)]))
            assert np.array_equal(table[0], pe.PREFIX_FC) and np.array_equal(table[1], pe.PREFIX_FM) and not table[2].any()
            assert not np.array_equal(placed[0], pe.PREFIX_FC)


@pytest.mark.gpu
@pytest.mark.parametrize("formats", W_FORMATS, ids=["int32-int32", "packed-packed", "packed-int32"])
def test_shard_release_world2(formats, oracle_c):
    check_world(2, formats, run_world(2, formats), oracle_c)


@pytest.mark.gpu
def test_shard_release_world6(oracle_c):
    """six ranks: the last CTA collects the peers' words four ranks at a time, so ranks 4 and 5 come from the second
    pull group"""
    formats = (False, True, False)
    check_world(6, formats, run_world(6, formats), oracle_c)


# ---- 6. a peer that never arrives --------------------------------------------------------------------------------
def _lone_rank_main(rank, conn, peer_conn):
    """rank 0 issues one release; rank 1 attaches and never issues it, so rank 0's pull gives up (~2 s)"""
    sys.path.insert(0, ROOT)
    import torch
    import elastic_gpu_agent_b200 as e
    torch.cuda.set_device(0)
    D = 8
    core, mem, idx = gr.placed_rows(8, D, 4099, False)
    fc, fm = gr.table_with_headroom(8, core, mem, idx, D)
    a = e.BestFitAllocator(0)
    a.set_table(fc, fm)
    mine = a.peer_export()
    peer_conn.send(mine)
    other = peer_conn.recv()
    a.peer_attach(rank, 2, [mine, other] if rank == 0 else [other, mine])
    if rank == 1:
        assert peer_conn.recv() == "done"
        a.peer_detach()
        a.close()
        return
    d = gr.Dev(torch, core, mem, idx, D)
    torch.cuda.synchronize()
    t0 = time.monotonic()
    rc = shard_call(a, d, F_RELEASE | F_COMMIT, 7)
    torch.cuda.synchronize()
    elapsed = time.monotonic() - t0
    u, tab = d.got()
    conn.send((rc, u, tab, a.table(), a.peer_last_timeout, a.release_refusals, elapsed))
    peer_conn.send("done")
    a.peer_detach()
    a.close()


@pytest.mark.gpu
def test_shard_release_peer_never_arrives():
    """the documented way out of a missing peer, run once: the launch ends on its own within the ~2 s bound, d_delta is
    this rank's sums, d_table_out is left unwritten, the table is unchanged, no refusal is counted, and
    egpu_peer_last_timeout names step 7"""
    import torch.multiprocessing as mp
    mctx = mp.get_context("spawn")
    a_conn, b_conn = mctx.Pipe()
    res_r, res_w = mctx.Pipe(False)
    procs = [mctx.Process(target=_lone_rank_main, args=(0, res_w, a_conn)),
             mctx.Process(target=_lone_rank_main, args=(1, None, b_conn))]
    for p in procs:
        p.start()
    try:
        assert res_r.poll(240), "rank 0 did not finish"
        rc, u, tab, table, timeout, refusals, elapsed = res_r.recv()
        for p in procs:
            p.join(60)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
    assert all(p.exitcode == 0 for p in procs)
    D = 8
    core, mem, idx = gr.placed_rows(8, D, 4099, False)
    fc, fm = gr.table_with_headroom(8, core, mem, idx, D)
    e_u = release_np.release(fc, fm, np.zeros(D), core, mem, idx)[0]
    assert rc == 0
    assert np.array_equal(u, e_u), "d_delta: this rank's sums"
    assert (tab == -7).all(), "table' written"
    assert np.array_equal(table[0], fc) and np.array_equal(table[1], fm) and not table[2].any(), "the table changed"
    assert timeout == 8, "egpu_peer_last_timeout: step 7 + 1"
    assert refusals == 0
    assert elapsed < 10, f"the launch took {elapsed:.1f} s to give up"
