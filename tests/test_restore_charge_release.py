"""Charge and release of stored records against the live table: EGPU_RESTORE_CHARGE and
EGPU_RESTORE_RELEASE on egpu_table_restore[_flat] (include/egpu_restore.h, DESIGN.md §2.7).

The property every test below comes back to: with T(A) the table a full restore of the record set A
installs, CHARGE(B) on T(A) is exactly T(A + B), flags included, and RELEASE(B) for B a part of A is
exactly T(A - B) whenever it is accepted; it is always accepted when no device B touches is
oversubscribed.  The CPU restatement is built on the restore oracle (oracle/restore_py.py: usage, charge,
release): the usage U of a set is what a restore against an unbounded capacity takes away.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest

from oracle import restore_py as R
from oracle.restore_py import Refused, charge, release, usage
from restore_util import persisted_state

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEM_MAX = (1 << 18) - 1
OTHER = "example.com/other-gpu"


def full(records, links, cap_core, cap_mem, verify=True):
    fc, fm, ov, counts, rstat = R.restore(records, links, cap_core, cap_mem, verify=verify)
    return (fc, fm, ov), counts, rstat


# ---- record sets --------------------------------------------------------------------------------------
def rec(name, ids, res, gpus, stored_hash=None):
    """one pod with one container, its record and its symlinks (gpus: the N of every link, in order)"""
    k, v = R.marshal_record("default", name, {"main": (ids, res)})
    h = R.device_hash(sorted(ids))
    if stored_hash is not None:
        v = v.replace(h.encode(), stored_hash.encode())
        h = stored_hash
    return (k, v), [("elastic-gpu-%s-%d" % (h, i), "/dev/nvidia%d" % g) for i, g in enumerate(gpus)]


def core_ids(n, gpu=0, start=0):
    return ["%d-%02d" % (gpu + (start + j) // 100, (start + j) % 100) for j in range(n)]


class Node:
    """A seeded set of stored records, one container each, in both input forms.  Entries: gpu-core
    percent, whole cards, gpu-memory at node scale (4 Ki - 16 Ki IDs), another plugin's resource,
    stale hashes, missing links and links outside the table.  fits=True keeps the counted usage
    (VERIFY or not) inside every device's capacity, so that nothing is oversubscribed."""

    def __init__(self, seed, D=8, n=96, fits=False, mem_cap=183359):
        rng = np.random.default_rng(seed)
        self.D, self.cap_core, self.cap_mem = D, [100] * D, [mem_cap] * D
        self.sets, self.hashes, self.resources, self.gpus, self.records, self.links = [], [], [], [], [], []
        used = np.zeros(D, np.int64)
        for r in range(n):
            kind = rng.integers(0, 20)
            if kind < 9:
                res, cnt = R.MEM, int(rng.choice([4096, 8192, 16384]))
            elif kind < 16:
                res, cnt = R.CORE, int(rng.integers(1, 41))
            elif kind < 19:
                res, cnt = R.CORE, 100 * int(rng.integers(1, 3)) + int(rng.integers(0, 30))
            else:
                res, cnt = OTHER, int(rng.integers(1, 20))
            need = cnt // 100 if (res == R.CORE and cnt > 100) else 1
            gpus = [int(g) for g in rng.choice(D, need, replace=False)]
            if fits and res == R.CORE:
                per = 100 if cnt > 100 else cnt
                if any(used[g] + per > 100 for g in gpus):
                    room = [g for g in range(D) if used[g] + per <= 100]
                    if len(room) < need:
                        res, cnt, need = R.MEM, 4096, 1
                        gpus = [int(rng.integers(0, D))]
                    else:
                        gpus = [int(g) for g in rng.choice(room, need, replace=False)]
            if res == R.MEM:
                ids = ["%d-%02d" % (r % D, j) for j in rng.choice(mem_cap, cnt, replace=False)]
            else:
                ids = ["%d-%02d" % (t // 100, t % 100) for t in rng.choice(D * 100, min(cnt, D * 100), replace=False)]
                cnt = len(ids)
            h = R.device_hash(ids)
            fault = rng.integers(0, 10)
            if fault == 0:
                h = "%08x" % (int(h, 16) ^ 0x10)       # stale hash: counted without VERIFY only
            elif fault == 1:
                gpus = gpus[:-1]                       # a missing link
            elif fault == 2:
                gpus[0] = D + 2                        # a link outside the table
            if fits and res == R.CORE and fault != 1 and fault != 2:
                for g in gpus:
                    used[g] += 100 if cnt > 100 else cnt
            self.sets.append(ids)
            self.hashes.append(h)
            self.resources.append(0 if res == R.CORE else 1 if res == R.MEM else -1)
            self.gpus.append(gpus)
            rv, lk = rec("pod-%d" % r, ids, res, gpus, stored_hash=h)
            self.records.append(rv)
            self.links += lk

    def flat(self, idx):
        return ([self.sets[i] for i in idx], [self.hashes[i] for i in idx], [self.resources[i] for i in idx],
                [self.gpus[i] for i in idx])

    def raw(self, idx):
        """the chosen records, and the node's whole /host/dev listing"""
        return [self.records[i] for i in idx], self.links


def chunks(rng, n, hi=20):
    order = rng.permutation(n).tolist()
    out = []
    while order:
        k = int(rng.integers(1, hi + 1))
        out.append(order[:k])
        order = order[k:]
    return out


# ---- CPU: the restatement against hand-derived cases ------------------------------------------------
CAP2 = ([100, 100], [1000, 1000])


def test_oracle_hand_derived_whole_cards_and_memory():
    (a, la), (b, lb) = rec("a", core_ids(230), R.CORE, [1, 0]), rec("b", ["0-%02d" % j for j in range(300)], R.MEM, [1])
    # 230 IDs of gpu-core: 230 // 100 = 2 whole cards on links 0 and 1; the remainder is not counted
    t, counts, rstat = charge(([100, 100], [1000, 1000], [0, 0]), [a, b], la + lb)
    assert t == ([0, 0], [1000, 700], [0, 0]) and counts == [2, 0, 0, 0, 0] and rstat == [0, 0]
    t2, _, _ = release(t, [a], la + lb, *CAP2)
    assert t2 == ([100, 100], [1000, 700], [0, 0])
    t3, _, _ = release(t2, [b], la + lb, *CAP2)
    assert t3 == ([100, 100], [1000, 1000], [0, 0])


def test_oracle_hand_derived_uncounted_entries_change_nothing():
    t0 = ([60, 100], [900, 1000], [0, 0])
    foreign, lf = rec("f", core_ids(25), OTHER, [0])
    nolink, _ = rec("n", core_ids(25, start=25), R.CORE, [0])     # no symlink listed
    outside, lo = rec("o", core_ids(25, start=50), R.CORE, [7])   # /dev/nvidia7 on a 2-GPU table
    stale, ls = rec("s", core_ids(25, start=75), R.CORE, [0], stored_hash="0badc0de")
    empty, _ = rec("e", [], R.CORE, [])
    links = lf + lo + ls
    for verify in (True, False):
        t, counts, rstat = charge(t0, [foreign, nolink, outside], links, verify)
        assert t == t0 and counts == [0, 0, 1, 2, 0] and rstat == [R.REC_FOREIGN, R.REC_NO_LINK, R.REC_NO_LINK]
        t, counts, rstat = release(t0, [foreign, nolink, outside, empty], links, *CAP2, verify=verify)
        assert t == t0 and counts == [0, 1, 1, 2, 0]
    # a stale hash is a mismatch under VERIFY and counted without it
    t, counts, rstat = charge(t0, [stale], links, verify=True)
    assert t == t0 and rstat == [R.REC_HASH_MISMATCH]
    t, counts, rstat = charge(t0, [stale], links, verify=False)
    assert t == ([35, 100], [900, 1000], [0, 0]) and rstat == [R.REC_OK]


def test_oracle_hand_derived_saturation_and_over_release():
    a, la = rec("a", core_ids(25), R.CORE, [0])
    m, lm = rec("m", ["1-%02d" % j for j in range(50)], R.MEM, [1])
    # saturation: 10 free, 25 charged -> 0 and flagged; the flag is sticky and blocks a release there
    t, _, _ = charge(([10, 100], [1000, 40], [0, 0]), [a, m], la + lm)
    assert t == ([0, 100], [1000, 0], [1, 1])
    with pytest.raises(Refused):
        release(t, [a], la, *CAP2)
    # a flag on a device the release does not touch does not matter
    b, lb = rec("b", core_ids(10), R.CORE, [1])
    assert release(([0, 90], [1000, 1000], [1, 0]), [b], lb, *CAP2)[0] == ([0, 100], [1000, 1000], [1, 0])
    # over-release: the same record released twice on an otherwise empty device
    t, _, _ = charge(([100, 100], [1000, 1000], [0, 0]), [a], la)
    t, _, _ = release(t, [a], la, *CAP2)
    assert t == ([100, 100], [1000, 1000], [0, 0])
    with pytest.raises(Refused):
        release(t, [a], la, *CAP2)


@pytest.mark.parametrize("seed", [3, 17, 29])
@pytest.mark.parametrize("verify", [True, False])
def test_oracle_property_union_and_difference(seed, verify):
    """T(A) charged with B is T(A + B); T(A) released by B, a part of A, is T(A - B) when accepted,
    and it is accepted whenever no device B touches is oversubscribed"""
    rng = np.random.default_rng(seed)
    for fits in (False, True):
        node = Node(seed, D=4, n=24, fits=fits)
        cap = (node.cap_core, node.cap_mem)
        idx = rng.permutation(24).tolist()
        A, B = idx[:12], idx[12:20]
        recs = lambda ix: node.raw(ix)[0]  # noqa: E731
        tA, _, _ = full(recs(A), node.links, *cap, verify=verify)
        got, counts, rstat = charge(tA, recs(B), node.links, verify)
        assert got == full(recs(A + B), node.links, *cap, verify=verify)[0]
        assert rstat == full(recs(B), node.links, *cap, verify=verify)[2]
        sub = A[:5]
        uc, um, _, _ = usage(recs(sub), node.links, 4, verify)
        touched_over = any((uc[d] or um[d]) and tA[2][d] for d in range(4))
        try:
            got, _, _ = release(tA, recs(sub), node.links, *cap, verify=verify)
            assert got == full(recs(A[5:]), node.links, *cap, verify=verify)[0]
        except Refused:
            assert touched_over
        if fits:
            assert not any(tA[2]) and not touched_over


def test_header_documents_both_flags_and_abi():
    text = open(os.path.join(ROOT, "include", "egpu_restore.h")).read()
    assert re.search(r"#define EGPU_RESTORE_CHARGE\s+4\b", text)
    assert re.search(r"#define EGPU_RESTORE_RELEASE\s+8\b", text)
    block = text[text.index("Charge and release"):text.index("#define EGPU_RESTORE_CHARGE")]
    for phrase in ("stays 1011", "EGPU_ERR_STATE", "EGPU_ERR_NO_TABLE", "max(free - U, 0)", "free' = free + U",
                   "All or nothing", "egpu_table_get"):
        assert phrase in block, phrase
    src = open(os.path.join(ROOT, "elastic-gpu-agent_b200", "restore.py")).read()
    assert "RESTORE_CHARGE = 4" in src and "RESTORE_RELEASE = 8" in src


# ---- GPU ----------------------------------------------------------------------------------------------
def gpu_call(alloc, node, idx, form, verify, cap=None, **flags):
    """one call through restore.py; returns (table int32[3D], statuses of the chosen entries)"""
    from elastic_gpu_agent_b200 import restore
    cc, cm = cap or (node.cap_core, node.cap_mem)
    if form == "flat":
        fc, fm, ov, st = restore.restore_table_flat(alloc, *node.flat(idx), cc, cm, verify=verify, **flags)
    else:
        fc, fm, ov, _, st = restore.restore_table(alloc, *node.raw(idx), cc, cm, verify=verify, **flags)
    return np.concatenate([fc, fm, ov]), st


def live(alloc):
    fc, fm, ov = alloc.table()
    return np.concatenate([fc, fm, ov])


def as_table(t):
    return np.asarray(t[0] + t[1] + t[2], np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["flat", "raw"])
@pytest.mark.parametrize("verify", [True, False])
def test_charge_chunks_equal_restore_of_union(alloc, form, verify):
    node = Node(5, fits=False)
    rng = np.random.default_rng(41)
    parts = chunks(rng, len(node.records))
    _, _, _, _, rstat = R.restore(node.records, node.links, node.cap_core, node.cap_mem, verify=verify)
    done = parts[0]
    gpu_call(alloc, node, done, form, verify, install=True)
    for part in parts[1:]:
        got, st = gpu_call(alloc, node, part, form, verify, charge=True)
        done = done + part
        want, _ = gpu_call(alloc, node, done, form, verify)
        assert np.array_equal(got, want) and np.array_equal(live(alloc), want), (form, verify, len(done))
        assert st.tolist() == [rstat[i] for i in part]
    want = full(node.records, node.links, node.cap_core, node.cap_mem, verify)[0]
    assert live(alloc).tolist() == as_table(want).tolist()
    assert want[2].count(1) > 0, "the node set should oversubscribe some device"
    assert len(set(rstat)) >= (4 if verify else 3)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["flat", "raw"])
@pytest.mark.parametrize("verify", [True, False])
def test_release_chunks_equal_restore_of_remainder(alloc, form, verify):
    node = Node(8, fits=True)
    rng = np.random.default_rng(43)
    _, _, _, _, rstat = R.restore(node.records, node.links, node.cap_core, node.cap_mem, verify=verify)
    left = list(range(len(node.records)))
    gpu_call(alloc, node, left, form, verify, install=True)
    assert not live(alloc)[2 * node.D:].any()
    for part in chunks(rng, len(left)):
        got, st = gpu_call(alloc, node, part, form, verify, release=True)
        left = [i for i in left if i not in part]
        want, _ = gpu_call(alloc, node, left, form, verify)
        assert np.array_equal(got, want) and np.array_equal(live(alloc), want), (form, verify, len(left))
        assert st.tolist() == [rstat[i] for i in part]
    assert live(alloc).tolist() == node.cap_core + node.cap_mem + [0] * node.D


@pytest.mark.gpu
@pytest.mark.parametrize("events,mem_cap", [(300, 4096), (400, 183359)])
def test_churn_charge_release_tracks_replay(alloc, egpu, events, mem_cap):
    """every placed ALLOC of a churn charges its record, every FREE that frees releases it: the table
    equals the replay's live table at every checkpoint"""
    from elastic_gpu_agent_b200 import restore
    D = 8
    kind, a, b = egpu.synth.churn_events(7, events)
    b = np.minimum(b, mem_cap // 4).astype(np.int32)
    cap_core, cap_mem = [100] * D, [mem_cap] * D
    with egpu.BestFitAllocator(0) as rep:
        rep.set_table(cap_core, cap_mem)
        out = rep.replay(kind, a, b)
        alloc.set_table(cap_core, cap_mem)
        held, checked = {}, 0
        for i in range(len(kind)):
            if kind[i] == 0 and out[i] >= 0:
                recs, links = persisted_state([(int(out[i]), int(a[i]), int(b[i]))], D, mem_cap, seed=i)
                held[i] = (recs, links)
                restore.restore_table(alloc, recs, links, cap_core, cap_mem, charge=True)
            elif kind[i] == 1 and out[i] >= 0:
                recs, links = held.pop(int(a[i]))
                restore.restore_table(alloc, recs, links, cap_core, cap_mem, release=True)
            if i % 25 == 24 or i == len(kind) - 1:
                rep.set_table(cap_core, cap_mem)
                rep.replay(kind[:i + 1], a[:i + 1], b[:i + 1])
                assert np.array_equal(live(alloc), live(rep)), i
                checked += 1
        assert held and checked >= events // 25


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 8, 9, 17, 33, 64])
def test_scans_read_the_charged_and_released_table(alloc, egpu, D):
    from oracle import bestfit_np
    from elastic_gpu_agent_b200 import restore
    rng = np.random.default_rng(100 + D)
    cap_core = [100] * D
    cap_mem = rng.integers(20000, MEM_MAX + 1, D).tolist()
    entries, used = [], [0] * D
    for r in range(3 * D):
        g, n = int(rng.integers(0, D)), int(rng.integers(1, 30))
        if rng.integers(0, 2) and used[g] + n <= 100:  # nothing oversubscribed: the release below is accepted
            used[g] += n
            entries.append((["%d-%02d" % (r, j) for j in range(n)], 0, [g]))
        else:
            entries.append((["%d-%02d" % (r, j) for j in range(int(rng.integers(1, 300)))], 1, [g]))
    sets = [e[0] for e in entries]
    hashes = [R.device_hash(s) for s in sets]
    res = [e[1] for e in entries]
    links = [e[2] for e in entries]

    def check(fc, fm):
        rows = [(c + dc, m + dm) for c, m in zip(fc, fm) for dc in (-1, 0, 1) for dm in (-1, 0, 1)]
        rc = np.array([r[0] for r in rows], np.int32)
        rm = np.array([r[1] for r in rows], np.int32)
        want = bestfit_np.snapshot(np.asarray(fc, np.int32), np.asarray(fm, np.int32), rc, rm)[0]
        for v in (egpu.VARIANT_LUT, egpu.VARIANT_SORTED, egpu.VARIANT_AUTO):
            alloc.set_variant(v)
            idx, _, _ = alloc.bestfit(rc, rm)
            assert np.array_equal(idx, want), (D, v)

    alloc.set_table(cap_core, cap_mem)
    check(cap_core, cap_mem)  # the lookup tables are built for the capacity table
    fc, fm, ov, _ = restore.restore_table_flat(alloc, sets, hashes, res, links, cap_core, cap_mem, charge=True)
    recs = [rec("p%d" % i, s, R.CORE if r == 0 else R.MEM, l) for i, (s, r, l) in enumerate(zip(sets, res, links))]
    rv, lk = [x[0] for x in recs], [y for x in recs for y in x[1]]
    want, _, _ = charge((cap_core, cap_mem, [0] * D), rv, lk)
    assert (fc.tolist(), fm.tolist(), ov.tolist()) == want
    check(want[0], want[1])
    keep = [i for i in range(len(sets)) if i % 3]
    gone = [i for i in range(len(sets)) if i % 3 == 0]
    fc, fm, ov, _ = restore.restore_table_flat(alloc, [sets[i] for i in gone], [hashes[i] for i in gone],
                                               [res[i] for i in gone], [links[i] for i in gone], cap_core, cap_mem,
                                               release=True)
    want2 = full([rv[i] for i in keep], lk, cap_core, cap_mem)[0]
    assert not any(want[2]) and (fc.tolist(), fm.tolist(), ov.tolist()) == want2
    check(want2[0], want2[1])


# ---- refusals: raw ctypes calls with sentinel outputs ---------------------------------------------------
def call_sentinel(alloc, form, sets, res, gpus, cap_core, cap_mem, flags, D=None):
    """(rc, table, statuses[, counts]) with every output pre-filled with a sentinel"""
    from elastic_gpu_agent_b200 import _lib as L
    from elastic_gpu_agent_b200.devhash import flatten
    D = len(cap_core) if D is None else D
    cc, cm = np.asarray(cap_core, np.int32), np.asarray(cap_mem, np.int32)
    table = np.full(3 * D, -7, np.int32)
    n = len(sets)
    if form == "flat":
        flat, id_off, set_off = flatten(sets)
        h8 = b"".join(R.device_hash(s).encode() for s in sets)
        rs = np.asarray(res or [0], np.int32)
        loff = np.zeros(n + 1, np.int64)
        loff[1:] = np.cumsum([len(g) for g in gpus])
        lg = np.asarray([x for g in gpus for x in g] or [0], np.int32)
        status = np.full(max(1, n), -9, np.int32)
        rc = L.load().egpu_table_restore_flat(alloc.handle, C.c_char_p(flat), C.c_void_p(id_off.ctypes.data), len(id_off) - 1,
                                              C.c_void_p(set_off.ctypes.data), n, C.c_char_p(h8), C.c_void_p(rs.ctypes.data),
                                              C.c_void_p(loff.ctypes.data), C.c_void_p(lg.ctypes.data),
                                              C.c_void_p(cc.ctypes.data), C.c_void_p(cm.ctypes.data), D, flags,
                                              C.c_void_p(table.ctypes.data), C.c_void_p(status.ctypes.data))
        return rc, table, status
    recs, links = [], []
    for i, (s, r, g) in enumerate(zip(sets, res, gpus)):
        rv, lk = rec("p%d" % i, s, R.CORE if r == 0 else R.MEM, g)
        recs.append(rv)
        links += lk
    keys = (C.c_char_p * max(1, n))(*[k for k, _ in recs])
    vals = (C.c_char_p * max(1, n))(*[v for _, v in recs])
    klen = np.asarray([len(k) for k, _ in recs] or [0], np.int64)
    vlen = np.asarray([len(v) for _, v in recs] or [0], np.int64)
    names = (C.c_char_p * max(1, len(links)))(*[x.encode() for x, _ in links])
    targets = (C.c_char_p * max(1, len(links)))(*[y.encode() for _, y in links])
    counts = np.full(5, -5, np.int64)
    rstat = np.full(max(1, n), -9, np.int32)
    rc = L.load().egpu_table_restore(alloc.handle, keys, C.c_void_p(klen.ctypes.data), vals, C.c_void_p(vlen.ctypes.data), n,
                                     names, targets, len(links), C.c_void_p(cc.ctypes.data), C.c_void_p(cm.ctypes.data), D,
                                     flags, C.c_void_p(table.ctypes.data), C.c_void_p(counts.ctypes.data),
                                     C.c_void_p(rstat.ctypes.data))
    return rc, table, np.concatenate([rstat, counts.astype(np.int32)])


def untouched(out):
    _, table, st = out
    return (table == -7).all() and ((st == -9) | (st == -5)).all()


VERIFY, INSTALL, CHARGE, RELEASE = 1, 2, 4, 8


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["flat", "raw"])
def test_refusals(alloc, egpu, form):
    from elastic_gpu_agent_b200 import _lib as L
    cap_c, cap_m = [100, 100], [1000, 1000]
    on0 = ([core_ids(30)], [0], [[0]])
    on1 = ([core_ids(20, start=40)], [0], [[1]])
    # no table: nothing launched
    n0 = alloc.launch_count
    out = call_sentinel(alloc, form, *on0, cap_c, cap_m, CHARGE)
    assert out[0] == L.ERR_NO_TABLE and untouched(out) and alloc.launch_count == n0
    # flag combinations and a D other than the table's: nothing launched, nothing changed
    alloc.set_table(cap_c, cap_m)
    before, n0 = live(alloc), alloc.launch_count
    for flags in (CHARGE | RELEASE, CHARGE | INSTALL, RELEASE | INSTALL, CHARGE | RELEASE | VERIFY, CHARGE | 16, RELEASE | 32):
        out = call_sentinel(alloc, form, *on0, cap_c, cap_m, flags)
        assert out[0] == L.ERR_INVALID and untouched(out), flags
    out = call_sentinel(alloc, form, *on0, cap_c + [100], cap_m + [1000], CHARGE)
    assert out[0] == L.ERR_INVALID and untouched(out)
    out = call_sentinel(alloc, form, *on0, cap_c[:1], cap_m[:1], RELEASE)
    assert out[0] == L.ERR_INVALID and untouched(out)
    assert alloc.launch_count == n0 and np.array_equal(live(alloc), before)
    # over-release: the same record released twice on an otherwise empty device
    assert call_sentinel(alloc, form, *on0, cap_c, cap_m, CHARGE | VERIFY)[0] == L.OK
    assert live(alloc).tolist() == [70, 100, 1000, 1000, 0, 0]
    assert call_sentinel(alloc, form, *on0, cap_c, cap_m, RELEASE | VERIFY)[0] == L.OK
    assert live(alloc).tolist() == [100, 100, 1000, 1000, 0, 0]
    out = call_sentinel(alloc, form, *on0, cap_c, cap_m, RELEASE | VERIFY)
    assert out[0] == L.ERR_STATE and untouched(out) and "device 0" in alloc._lib.egpu_last_error(alloc.handle).decode()
    assert live(alloc).tolist() == [100, 100, 1000, 1000, 0, 0]
    # an oversubscribed device: 30 charged on 20 free saturates and flags it; releasing there is refused
    alloc.set_table([20, 100], cap_m)
    assert call_sentinel(alloc, form, *on0, cap_c, cap_m, CHARGE)[0] == L.OK
    assert live(alloc).tolist() == [0, 100, 1000, 1000, 1, 0]
    out = call_sentinel(alloc, form, *on0, cap_c, cap_m, RELEASE)
    assert out[0] == L.ERR_STATE and untouched(out)
    assert live(alloc).tolist() == [0, 100, 1000, 1000, 1, 0]
    # ... while a release that does not touch it goes through, and the flag stays
    assert call_sentinel(alloc, form, *on1, cap_c, cap_m, CHARGE)[0] == L.OK
    out = call_sentinel(alloc, form, *on1, cap_c, cap_m, RELEASE)
    assert out[0] == L.OK and out[1].tolist() == [0, 100, 1000, 1000, 1, 0]
    assert live(alloc).tolist() == [0, 100, 1000, 1000, 1, 0]


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["flat", "raw"])
@pytest.mark.parametrize("flags", [CHARGE, RELEASE])
def test_nothing_to_apply_reads_the_table(alloc, form, flags):
    """n_sets = 0: the table, flags included, is written out and stays as it was"""
    from elastic_gpu_agent_b200 import _lib as L
    alloc.set_table([20, 100], [1000, 1000])
    assert call_sentinel(alloc, "flat", [core_ids(30)], [0], [[0]], [100, 100], [1000, 1000], CHARGE)[0] == L.OK
    before = live(alloc)
    rc, table, _ = call_sentinel(alloc, form, [], [], [], [100, 100], [1000, 1000], flags)
    assert rc == L.OK and table.tolist() == before.tolist() == [0, 100, 1000, 1000, 1, 0]
    assert np.array_equal(live(alloc), before)
