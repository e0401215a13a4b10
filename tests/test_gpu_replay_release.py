"""Release events in sequential replay (EGPU_EV_RELEASE, DESIGN.md 2.6) on the GPU, exact against the restatement
of tests/replay_release_np.py: every replay kernel (selected as in test_gpu_context_sequences.py), the D buckets,
event counts around the 32- and 256-event chunks and both sides of kReplaySmemEvents, GC-style streams, the round
trip through release events (after a replay and after a restore), agreement with a batch EGPU_F_RELEASE, and flagged
devices.  After every call the installed table and flags are read back, and a probe scan reads the re-sorted table
and the lookup tables."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import replay_release_np as rr  # noqa: E402
from replay_release_np import pack  # noqa: E402

MEM_MAX = rr.MEM_MAX
REPLAY_SMEM_EVENTS = 200 * 1024  # kReplaySmemEvents
REPLAY_KERNELS = {"two_warp": ("2", "0"), "one_warp": ("1", "0"), "general": ("1", "1")}
DS = (1, 5, 8, 9, 32, 33, 64)
ES = (1, 31, 32, 33, 255, 256, 257, 1000)


def context(egpu, kernel):
    """a context whose replays run on `kernel` (the two-warp kernel only where it applies: D <= 32 and events that
    fit shared memory; the other two are round 1's one-warp kernels)"""
    variant, general = REPLAY_KERNELS[kernel]
    old = {k: os.environ.get(k) for k in ("EGPU_REPLAY_VARIANT", "EGPU_REPLAY_GENERAL")}
    os.environ["EGPU_REPLAY_VARIANT"], os.environ["EGPU_REPLAY_GENERAL"] = variant, general
    try:
        return egpu.BestFitAllocator(0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def probe(al, fc, fm):
    """a snapshot of each device's (fc, fm) and its neighbours, and edge rows, against the oracle"""
    from oracle import bestfit_np
    fc, fm = np.asarray(fc, np.int64), np.asarray(fm, np.int64)
    rows = [(c + dc, m + dm) for c, m in zip(fc.tolist(), fm.tolist()) for dc in (-1, 0, 1) for dm in (-1, 0, 1)]
    rows += [(0, 0), (100, MEM_MAX), (0, MEM_MAX + 1), (101, 0)]
    r = np.array(rows, np.int64)
    rc, rm = r[:, 0].astype(np.int32), r[:, 1].astype(np.int32)
    idx, _, _ = al.bestfit(rc, rm)
    assert np.array_equal(idx, bestfit_np.snapshot(fc.astype(np.int32), fm.astype(np.int32), rc, rm)[0]), "probe scan"


def replay_checked(al, kind, a, b, what=""):
    """one egpu_replay against the restatement on the context's live table: indices, table, flags, probe scan"""
    fc, fm, ov = al.table()
    want, w_fc, w_fm = rr.replay(fc, fm, ov, kind, a, b)
    got = al.replay(kind, a, b)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{what}: first mismatch at event {bad[0] if bad.size else -1}: got {got[bad[:5]]}, want {want[bad[:5]]}"
    g_fc, g_fm, g_ov = al.table()
    assert np.array_equal(g_fc, w_fc) and np.array_equal(g_fm, w_fm), f"{what}: table"
    assert np.array_equal(g_ov, ov), f"{what}: flags changed"
    probe(al, g_fc, g_fm)
    return got


def flag(al, fc, fm, flagged):
    """installs (fc, fm) with the devices in `flagged` oversubscribed: each is set to (1, 1) and one committing
    snapshot of two (1, 1) rows takes it to (0, 0) with its flag set (fc must avoid 1 elsewhere)"""
    fc, fm = np.asarray(fc, np.int32).copy(), np.asarray(fm, np.int32).copy()
    fc[fc == 1] = 2
    fc[list(flagged)], fm[list(flagged)] = 1, 1
    al.set_table(fc, fm)
    for _ in flagged:
        al.bestfit([1, 1], [1, 1], commit=True)
    g_fc, g_fm, ov = al.table()
    assert sorted(np.flatnonzero(ov).tolist()) == sorted(flagged)
    return g_fc, g_fm, ov


def random_table(rng, D):
    return rng.integers(0, 101, D).astype(np.int32), rng.integers(0, 60_000, D).astype(np.int32)


def allocs(rng, E):
    """E ALLOC events of modest size, a few out of the domain"""
    kind = np.zeros(E, np.int32)
    a = rng.integers(0, 40, E).astype(np.int32)
    b = rng.integers(0, 8000, E).astype(np.int32)
    odd = rng.random(E) < 0.03
    a[odd] = rng.choice([-1, 101, 127], odd.sum())
    return kind, a, b


def gc_stream(rng, E, D, held, frac_release=0.1):
    """a GC-style stream: ALLOCs, FREEs of this stream's earlier events, release events handing back `held`
    (placements of earlier calls, (device, core, mem)) - some twice, some with a bad device or word - and kinds 2
    and 7"""
    kind = rng.choice([0, 0, 0, 1, 1, 2, 7], E, p=[.3, .2, .1, .15, .1, .05, .1]).astype(np.int32)
    a = np.where(kind == 0, rng.integers(0, 30, E), (rng.random(E) * np.arange(E)).astype(np.int64)).astype(np.int32)
    b = rng.integers(0, 6000, E).astype(np.int32)
    rel = np.flatnonzero(rng.random(E) < frac_release)
    for i in rel:
        kind[i] = 3
        r = rng.random()
        if held and r < 0.8:
            d, c, m = held[int(rng.integers(0, len(held)))]
            a[i], b[i] = d, pack(c, m)
        elif r < 0.85:
            a[i], b[i] = rng.choice([-1, D, 64, 1 << 20]), pack(1, 1)
        elif r < 0.9:
            a[i], b[i] = rng.integers(0, D), rng.choice([1 << 25, -1, 101 << 18, (127 << 18) | 3])
        elif r < 0.95:
            a[i], b[i] = rng.integers(0, D), 0
        else:
            a[i], b[i] = rng.integers(0, D), pack(rng.integers(0, 101), rng.integers(0, MEM_MAX + 1))
    return kind, a, b


def placements(kind, a, b, out):
    k, d, w = rr.releases_of(kind, a, b, out)
    return [(int(x), int(y) >> 18, int(y) & MEM_MAX) for x, y in zip(d, w)]


# ---- mixed streams over the kernels, D buckets and chunk edges ---------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", DS)
@pytest.mark.parametrize("kernel", list(REPLAY_KERNELS))
def test_mixed_streams(egpu, kernel, D):
    rng = np.random.default_rng(1000 * D + len(kernel))
    with context(egpu, kernel) as al:
        for E in ES:
            al.set_table(*random_table(rng, D))
            k0, a0, b0 = allocs(rng, 60)
            out0 = al.replay(k0, a0, b0)
            held = placements(k0, a0, b0, out0)
            if rng.random() < 0.5 and D > 1:
                fc, fm, _ = al.table()
                fc, fm, _ = flag(al, fc, fm, [int(rng.integers(0, D))])
            kind, a, b = gc_stream(rng, E, D, held)
            replay_checked(al, kind, a, b, f"{kernel} D={D} E={E}")
            # the same stream again on what it left: double releases, FREEs of the new call's events
            replay_checked(al, kind, a, b, f"{kernel} D={D} E={E}, again")


@pytest.mark.gpu
@pytest.mark.parametrize("E", [REPLAY_SMEM_EVENTS, REPLAY_SMEM_EVENTS + 1])
@pytest.mark.parametrize("D", [8, 33])
@pytest.mark.parametrize("kernel", list(REPLAY_KERNELS))
def test_long_streams_either_side_of_shared_memory(egpu, kernel, D, E):
    """`live` in shared memory up to kReplaySmemEvents events, in HBM past it (and the two-warp kernel hands over)"""
    rng = np.random.default_rng(E + D)
    with context(egpu, kernel) as al:
        al.set_table(np.full(D, 100, np.int32), np.full(D, 200_000, np.int32))
        k0, a0, b0 = allocs(rng, 400)
        held = placements(k0, a0, b0, al.replay(k0, a0, b0))
        kind, a, b = gc_stream(rng, E, D, held)
        replay_checked(al, kind, a, b, f"{kernel} D={D} E={E}")


# ---- round trips --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", DS)
@pytest.mark.parametrize("kernel", list(REPLAY_KERNELS))
def test_round_trip_through_release_events(egpu, kernel, D):
    """ALLOCs (and FREEs) in one call, then release events built from its out_idx in a second call, in any order:
    the starting table comes back exactly"""
    rng = np.random.default_rng(77 + D)
    with context(egpu, kernel) as al:
        for E in (5, 300):
            fc, fm = random_table(rng, D)
            al.set_table(fc, fm)
            kind = rng.choice([0, 0, 0, 1], E).astype(np.int32)
            a = np.where(kind == 0, rng.integers(0, 30, E), rng.integers(0, E, E)).astype(np.int32)
            b = rng.integers(0, 6000, E).astype(np.int32)
            out = replay_checked(al, kind, a, b, "placements")
            rk, ra, rb = rr.releases_of(kind, a, b, out)
            perm = rng.permutation(rk.size)
            back = replay_checked(al, rk[perm], ra[perm], rb[perm], "release events")
            assert np.array_equal(back, ra[perm])
            g_fc, g_fm, _ = al.table()
            assert np.array_equal(g_fc, fc) and np.array_equal(g_fm, fm)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [5, 9, 33])
@pytest.mark.parametrize("kernel", list(REPLAY_KERNELS))
def test_round_trip_after_restore(egpu, kernel, D):
    """a table restored from stored records (EGPU_RESTORE_INSTALL), then one release event per record: the
    capacities come back exactly, and a second hand-back is refused"""
    from restore_util import persisted_state
    from elastic_gpu_agent_b200 import restore
    rng = np.random.default_rng(5 + D)
    mem_cap = 4096
    cap_core, cap_mem = [100] * D, [mem_cap] * D
    used_c, used_m, pl = np.zeros(D, int), np.zeros(D, int), []
    for _ in range(4 * D):
        d, c, m = int(rng.integers(0, D)), int(rng.integers(1, 30)), int(rng.integers(1, 700))
        if used_c[d] + c <= 100 and used_m[d] + m <= mem_cap:
            used_c[d] += c
            used_m[d] += m
            pl.append((d, c, m))
    records, links = persisted_state(pl, D, mem_cap, seed=D)
    with context(egpu, kernel) as al:
        fc, fm, ov, _, _ = restore.restore_table(al, records, links, cap_core, cap_mem, install=True)
        assert fc.tolist() == (100 - used_c).tolist() and fm.tolist() == (mem_cap - used_m).tolist() and not ov.any()
        order = rng.permutation(len(pl))
        kind = np.full(len(pl), rr.EV_RELEASE, np.int32)
        a = np.array([pl[i][0] for i in order], np.int32)
        b = np.array([pack(pl[i][1], pl[i][2]) for i in order], np.int32)
        assert np.array_equal(replay_checked(al, kind, a, b, "release of the records"), a)
        g_fc, g_fm, _ = al.table()
        assert g_fc.tolist() == cap_core and g_fm.tolist() == cap_mem
        again = replay_checked(al, kind, a, b, "second hand-back")
        assert (again == -1).all()


# ---- against a batch release ------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", DS)
@pytest.mark.parametrize("kernel", list(REPLAY_KERNELS))
def test_agrees_with_batch_release(egpu, kernel, D):
    """rows that prefix-commit rounds placed, given back by egpu_bestfit_batch with EGPU_F_RELEASE | EGPU_F_COMMIT on
    one context and as release events on another: the same table whenever the batch is accepted; when it is refused
    (every row, then five of them again) the replay accepts what fits, event by event"""
    rng = np.random.default_rng(300 + D)
    fc, fm = np.full(D, 100, np.int32), np.full(D, MEM_MAX, np.int32)
    rc = rng.integers(0, 12, 40).astype(np.int32)
    rm = rng.integers(1, 3000, 40).astype(np.int32)
    with egpu.BestFitAllocator(0) as batch, context(egpu, kernel) as al:
        batch.set_table(fc, fm)
        idx = batch.bestfit_rounds(rc, rm)[0]
        assert idx[0] >= 0 and (idx >= -1).all()
        placed_fc, placed_fm, _ = batch.table()
        for rows in (np.arange(40), rng.permutation(40)[:17], np.concatenate([np.arange(40), np.arange(5)])):
            batch.set_table(placed_fc, placed_fm)
            al.set_table(placed_fc, placed_fm)
            try:
                batch.release(rc[rows], rm[rows], idx[rows], commit=True)
                accepted = True
            except egpu.EgpuError:
                accepted = False
            a = idx[rows].astype(np.int32)
            b = np.array([pack(c, m) for c, m in zip(rc[rows], rm[rows])], np.int32)
            got = replay_checked(al, np.full(rows.size, rr.EV_RELEASE, np.int32), a, b, f"rows {rows.size}")
            if accepted:
                assert np.array_equal(got, a)
                assert all(np.array_equal(x, y) for x, y in zip(al.table(), batch.table()))
        assert not accepted  # the last row set gives back row 0's memory twice: past EGPU_MEM_MAX
        assert np.array_equal(got[:40], idx.astype(np.int32)) and (got[40:] == -1).all()


# ---- flagged devices --------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", [5, 9, 33])
@pytest.mark.parametrize("kernel", list(REPLAY_KERNELS))
def test_flagged_device(egpu, kernel, D):
    """after an oversubscribing committing snapshot, a release on the flagged device is refused unless it is (0, 0);
    the other devices take theirs, and the flags stay as they are"""
    rng = np.random.default_rng(900 + D)
    with context(egpu, kernel) as al:
        fc, fm = random_table(rng, D)
        fc = np.minimum(fc, 60)
        fc, fm, ov = flag(al, fc, fm, [0, D - 1])
        kind = np.full(6, rr.EV_RELEASE, np.int32)
        a = np.array([0, 0, D - 1, 1, 1, D - 1], np.int32)
        b = np.array([pack(1, 0), 0, pack(0, 1), pack(10, 10), pack(0, 0), pack(0, 0)], np.int32)
        got = replay_checked(al, kind, a, b, "flagged")
        assert got.tolist() == [-1, 0, -1, 1, 1, D - 1]
        # a stream that allocates around them
        kind, a, b = gc_stream(rng, 500, D, [(0, 5, 5), (1, 5, 5), (D - 1, 0, 0)], frac_release=0.3)
        replay_checked(al, kind, a, b, "flagged stream")
