"""One context across many calls, against an int64 model of the table it keeps.

A context lives as long as the plugin and mixes its calls: commits, replays, prefix-commit rounds,
restores, queries, multi-batch launches.  Besides free_core / free_mem / oversub it carries state from
call to call that the scans read instead of the table itself: the sorted view (sorted_k, sorted_dev,
dev_packed), the lookup tables (rebuilt when ctx->lut_dirty is set), the launch-ordering state and the
epilogue slot rings (seq mod 32, mseq mod 128), the sticky oversubscription flags and grow-only scratch.

Every sequence below is a seeded list of operations on ONE context.  Each operation's own outputs are
compared exactly with the oracles (oracle/oracle_c.py, oracle/bestfit_np.py, oracle/restore_py.py), and
the model table (fc, fm, oversub, D) is advanced by the composition rules of DESIGN.md 2.4-2.7:
  - egpu_table_set installs the table and clears oversub;
  - a committing snapshot (plain, packed, device, apply) installs max(table', 0) and ORs table' < 0 into oversub;
  - prefix-commit, rounds and replay install their table and leave oversub as it was;
  - restore with EGPU_RESTORE_INSTALL installs the restored table with its own oversubscription flags;
  - everything else leaves the table alone.
After every operation the state is read back twice: egpu_table_get against the model, and a probe batch
built from the model's table (every device's own capacity and its +-1 neighbours, so that every row of
the sorted view and of the lookup tables decides some answer) through the next scan family of a fixed
rotation, and after a table change also through the lookup scan: the lookup tables are then rebuilt
before every call, so a later change that does not mark them stale is read back stale.  Each sequence runs once per replay kernel (EGPU_REPLAY_VARIANT / EGPU_REPLAY_GENERAL).

To reproduce a failure alone: run_sequence(seed, replay_kernel, upto=op_index) with the seed, kernel
and operation index the failure message names.
"""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEM_MAX = (1 << 18) - 1
INT32_MIN, INT32_MAX = -(2**31), 2**31 - 1
GRID, SORTED, LUT, AUTO = 1, 2, 3, 0
REPLAY_SMEM_EVENTS = 200 * 1024  # kReplaySmemEvents: larger replays keep their `live` map in HBM

SEEDS = (11, 23, 37, 52)
# (EGPU_REPLAY_VARIANT, EGPU_REPLAY_GENERAL): the two-warp kernel (D <= 32, events in shared memory),
# the one-warp kernels (registers for D <= 8, lane = device above), the lane = device kernel everywhere
REPLAY_KERNELS = {"two_warp": ("2", "0"), "one_warp": ("1", "0"), "general": ("1", "1")}
# set_table walks D across the kernels' buckets (D <= 8, 16, 32, 64) and back down
D_WALK = (1, 5, 8, 9, 16, 17, 33, 64, 33, 17, 16, 9, 8, 5)

# ---- the model ------------------------------------------------------------------------------------
class Model:
    """(fc, fm, oversub, D), int64, advanced by the composition rules of DESIGN.md 2.4-2.7"""

    def __init__(self):
        self.fc = self.fm = self.ov = None

    @property
    def D(self):
        return self.fc.size

    def set_table(self, fc, fm, ov=None):
        self.fc = np.asarray(fc, np.int64).copy()
        self.fm = np.asarray(fm, np.int64).copy()
        self.ov = np.zeros(self.fc.size, np.int64) if ov is None else np.asarray(ov, np.int64).copy()

    def commit_snapshot(self, tab):
        """a committing snapshot's table' (int32[3D]): max(table', 0) installed, oversub sticky"""
        D = self.D
        tab = np.asarray(tab, np.int64)
        self.fc, self.fm = np.maximum(tab[:D], 0), np.maximum(tab[D:2 * D], 0)
        self.ov = self.ov | tab[2 * D:]

    def install(self, fc, fm):
        """prefix-commit, rounds, replay: the table changes, the flags stay"""
        self.fc = np.asarray(fc, np.int64).copy()
        self.fm = np.asarray(fm, np.int64).copy()

    def table32(self):
        return self.fc.astype(np.int32), self.fm.astype(np.int32)


# ---- probe batches ------------------------------------------------------------------------------------
FIXED_PROBES = ((0, 0), (100, MEM_MAX), (0, MEM_MAX + 1), (101, 0), (-1, 0))


def probe_rows(fc, fm):
    """every device's (fc, fm) and its +-1 neighbours in each dimension, and the fixed edge rows"""
    fc, fm = np.asarray(fc, np.int64), np.asarray(fm, np.int64)
    rows = [(c + dc, m + dm) for c, m in zip(fc.tolist(), fm.tolist()) for dc in (-1, 0, 1) for dm in (-1, 0, 1)]
    rows += list(FIXED_PROBES)
    a = np.array(rows, np.int64)
    return a[:, 0].astype(np.int32), a[:, 1].astype(np.int32)


def snapshot_np(fc, fm, rc, rm):
    from oracle import bestfit_np
    return bestfit_np.snapshot(np.asarray(fc, np.int32), np.asarray(fm, np.int32), rc, rm)


# ---- inputs ----------------------------------------------------------------------------------------
CORE_EDGES = (INT32_MIN, -1, 0, 1, 99, 100, 101, 127, 128)
MEM_EDGES = (-1, 0, 1, 64, MEM_MAX, MEM_MAX + 1, INT32_MAX)


def random_table(rng, D):
    kind = rng.integers(0, 5)
    if kind == 0:  # duplicated pairs: ties go to the lowest index
        k = max(1, D // 3)
        pc, pm = rng.integers(0, 101, k), rng.integers(0, MEM_MAX + 1, k)
        pick = rng.integers(0, k, D)
        return pc[pick].astype(np.int32), pm[pick].astype(np.int32)
    if kind == 1:  # mostly full
        fc, fm = np.full(D, 100, np.int32), np.full(D, MEM_MAX, np.int32)
        fc[rng.integers(0, D)] = rng.integers(0, 101)
        return fc, fm
    fc = rng.integers(0, 101, D).astype(np.int32)
    fm = rng.choice(MEM_MAX + 1, D, replace=False).astype(np.int32)
    if kind == 2:  # small memory: requests below oversubscribe it
        fm = rng.choice(4000, D, replace=False).astype(np.int32)
    return fc, fm


def requests_for(rng, fc, fm, R):
    """rows near the devices' own capacities, small and random rows, edge values"""
    fc, fm = np.asarray(fc, np.int64), np.asarray(fm, np.int64)
    D = fc.size
    kind = rng.integers(0, 10, R)
    d = rng.integers(0, D, R)
    c = rng.integers(0, 101, R)
    m = rng.integers(0, MEM_MAX + 1, R)
    near = kind < 4
    c[near] = fc[d[near]] + rng.integers(-2, 2, near.sum())
    m[near] = fm[d[near]] + rng.integers(-2, 2, near.sum())
    small = (kind >= 4) & (kind < 8)
    c[small] = rng.integers(0, 30, small.sum())
    m[small] = rng.integers(0, 5000, small.sum())
    edge = kind == 8
    c[edge] = rng.choice(CORE_EDGES, edge.sum())
    m[edge] = rng.choice(MEM_EDGES, edge.sum())
    return c.astype(np.int32), m.astype(np.int32)


ROWS = (0, 1, 3, 5, 511, 513, 4099, 20_011)


def pack(rc, rm):
    c, m = np.asarray(rc, np.int64), np.asarray(rm, np.int64)
    ok = (c >= 0) & (c <= 127) & (m >= 0) & (m <= MEM_MAX)
    return np.where(ok, (c << 18) | m, 0xFFFFFFFF).astype(np.uint32)


# ---- the operations --------------------------------------------------------------------------------------
# name -> (changes the table, C entry points it calls).  An entry point of include/*.h is either named
# here or in NO_TABLE_CHANGE (test_every_entry_point_has_a_decision).
OPS = {
    "set_table": (True, ("egpu_table_set",)),
    "commit_host": (True, ("egpu_bestfit_batch",)),
    "commit_zero_copy": (True, ("egpu_bestfit_batch", "egpu_host_alloc")),
    "commit_dev": (True, ("egpu_bestfit_batch_dev",)),
    "commit_packed": (True, ("egpu_bestfit_batch_packed",)),
    "commit_packed_dev": (True, ("egpu_bestfit_batch_packed_dev",)),
    "prefix_host": (True, ("egpu_bestfit_batch",)),
    "prefix_dev": (True, ("egpu_bestfit_batch_dev",)),
    "rounds_host": (True, ("egpu_bestfit_batch_rounds",)),
    "rounds_dev": (True, ("egpu_bestfit_batch_rounds_dev",)),
    "replay": (True, ("egpu_replay",)),
    "replay_big": (True, ("egpu_replay",)),
    "apply_deltas": (True, ("egpu_table_apply_deltas_dev",)),
    "shard_apply": (True, ("egpu_bestfit_batch_shard_dev", "egpu_table_apply_peers_dev",
                           "egpu_table_apply_peers_multi_dev")),
    "shard_prefix": (True, ("egpu_bestfit_batch_shard_prefix_dev",)),
    "restore_install": (True, ("egpu_table_restore_flat", "egpu_table_restore")),
    "multi": (False, ("egpu_bestfit_batches_dev",)),
    "multi_big": (False, ("egpu_bestfit_batches_dev", "egpu_synth_requests_dev")),
    "snapshot": (False, ("egpu_bestfit_batch", "egpu_bestfit_batch_dev")),
    "pipelined_chain": (False, ("egpu_bestfit_batch_dev",)),
    "query": (False, ("egpu_bestfit_query",)),
    "preferred": (False, ("egpu_preferred_allocation_batch", "egpu_preferred_allocation")),
    "devhash": (False, ("egpu_device_hash_batch", "egpu_device_hash", "egpu_device_locate")),
    "restore_only": (False, ("egpu_table_restore_flat", "egpu_table_restore")),
    "synth": (False, ("egpu_synth_requests_dev",)),
}

NO_TABLE_CHANGE = {
    "egpu_ctx_create": "creates the context; there is no table yet",
    "egpu_backend": "constant",
    "egpu_abi_version": "constant",
    "egpu_set_variant": "selects the scan kernel; the sequences switch it between calls",
    "egpu_table_get": "the first read-back after every operation",
    "egpu_table_size": "read by every wrapper that sizes its outputs",
    "egpu_host_register": "pins caller memory; no kernel launch",
    "egpu_host_unregister": "unpins caller memory; no kernel launch",
    "egpu_peer_export": "exports the exchange buffer's IPC handle",
    "egpu_peer_attach": "peer configuration only (the part of DevState after the table); each sequence attaches world 1",
    "egpu_peer_detach": "closes the peers' buffers",
    "egpu_peer_gate_dev": "start gate of a sharded sequence; touches gate_epoch only",
    "egpu_peer_gate_open": "host side of the start gate",
    "egpu_bestfit_batches_shard_dev": "never commits: table' goes to d_table_out or comes from an apply call",
    "egpu_bestfit_batch_shard_lag_dev": "never commits (EGPU_F_COMMIT is refused)",
    "egpu_device_id_format": "string formatting, no context",
    "egpu_device_id_parse": "string parsing, no context",
}

ALL_OPS = tuple(OPS)
# every sequence: set_table first, then each operation once (set_table four times, multi-batch six and
# pipelined chains four: both epilogue rings must wrap), then extra draws; multi_big in one sequence only
EXTRA = ("set_table", "commit_host", "commit_dev", "commit_dev", "commit_packed", "prefix_dev", "rounds_host", "replay",
         "replay", "apply_deltas", "shard_apply", "restore_install", "snapshot", "pipelined_chain", "set_table")
READERS = ("sorted", "lut", "grid", "sorted_multi", "lut_multi", "packed", "pipelined")


def plan(seed):
    """the operation names of sequence `seed`, in order"""
    rng = np.random.default_rng(seed)
    body = [n for n in ALL_OPS if n not in ("set_table", "multi_big")] + ["multi"] * 5 + ["set_table"] * 3 + ["pipelined_chain"] * 3
    body += list(rng.choice(EXTRA, 10))
    if seed == SEEDS[0]:
        body.append("multi_big")
    rng.shuffle(body)
    return ["set_table"] + body


def walk_start(seed):
    """where sequence `seed` enters D_WALK: the sequences of SEEDS together cover all of it"""
    return 4 * SEEDS.index(seed) if seed in SEEDS else seed


def d_at(seed, upto):
    """D in force before operation `upto` of sequence `seed` (only set_table changes D)"""
    n = sum(1 for name in plan(seed)[:upto] if name == "set_table")
    return D_WALK[(walk_start(seed) + n - 1) % len(D_WALK)] if n else None


# ---- the sequence runner ------------------------------------------------------------------------------
class Run:
    def __init__(self, alloc, egpu, oracle_c, torch, seed):
        self.a, self.egpu, self.oc, self.torch, self.seed = alloc, egpu, oracle_c, torch, seed
        self.m = Model()
        self.variant = AUTO
        self.n_set = 0
        self.step = 0            # exchange step of the world-1 peer calls
        self.seq_scans = 0       # single-batch scans and packed launches (epilogue slot seq mod 32)
        self.multi_batches = 0   # batches of multi-batch launches (slot mseq mod 128)
        self.lut_built = False
        self.switched_variant_after_lut = self.switched_d_after_lut = False
        self.ts = torch.cuda.Stream()

    # -- helpers --
    def dev(self, a, pad=4):
        t = self.torch
        a = np.ascontiguousarray(a)
        out = t.zeros(a.size + pad, dtype=t.from_numpy(a[:0]).dtype, device="cuda")
        if a.size:
            out[:a.size] = t.from_numpy(a).cuda()
        return out

    def outs(self, R, D):
        t = self.torch
        return (t.full((R + 4,), -9, dtype=t.int32, device="cuda"), t.full((2 * D,), -1, dtype=t.int64, device="cuda"),
                t.full((3 * D,), -7, dtype=t.int32, device="cuda"))

    def stream(self, rng):
        """the context's own stream (None) or a torch stream"""
        return None if rng.integers(0, 2) else self.ts.cuda_stream

    def uses_lut(self, variant=None):
        v = self.variant if variant is None else variant
        return v == LUT or (v == AUTO and self.m.D > 16)

    def set_variant(self, v):
        if v != self.variant and self.lut_built:
            self.switched_variant_after_lut = True
        self.variant = v
        self.a.set_variant(v)

    def pick_variant(self, rng, grid_ok=True):
        self.set_variant(int(rng.choice([AUTO, GRID, SORTED, LUT] if grid_ok else [AUTO, SORTED, LUT])))

    def scanned(self, n=1, variant=None):
        self.seq_scans += n
        if self.uses_lut(variant):
            self.lut_built = True

    def sync(self):
        self.torch.cuda.synchronize()

    def oracle(self, rc, rm, fc=None, fm=None):
        if fc is None:
            fc, fm = self.m.table32()
        return self.oc.snapshot(fc, fm, rc, rm, self.oc.max_threads() if rc.size > 100_000 else 1)

    def rows(self, rng, R=None):
        R = int(rng.choice(ROWS)) if R is None else R
        return requests_for(rng, self.m.fc, self.m.fm, R)

    def dev_call(self, rc, rm, commit, stream, ready=False, prefix=False):
        R, D = rc.size, self.m.D
        c, m = self.dev(rc), self.dev(rm)
        idx, delta, tab = self.outs(R, D)
        self.sync()
        self.a.bestfit_dev(c.data_ptr(), m.data_ptr(), R, idx.data_ptr(), delta.data_ptr(), tab.data_ptr(), commit, stream,
                           inputs_ready=ready, prefix_commit=prefix)
        self.sync()
        idx = idx.cpu().numpy()
        eq(idx[R:], -9, "guard words after idx")
        return idx[:R], delta.cpu().numpy(), tab.cpu().numpy()

    # -- read-back --
    def check_table(self):
        fc, fm, ov = self.a.table()
        eq(fc, self.m.fc, "table() free_core")
        eq(fm, self.m.fm, "table() free_mem")
        eq(ov, self.m.ov, "table() oversub")

    def read(self, reader):
        fc, fm = self.m.table32()
        pc, pm = probe_rows(fc, fm)
        o_idx, o_dc, o_dm, o_tab = snapshot_np(fc, fm, pc, pm)
        o_delta = np.concatenate([o_dc, o_dm])
        keep = self.variant
        if reader in ("sorted", "lut", "grid"):
            v = {"sorted": SORTED, "lut": LUT, "grid": GRID}[reader]
            self.set_variant(v)
            idx, delta, tab = self.dev_call(pc, pm, False, self.ts.cuda_stream)
            self.scanned(variant=v)
            eq(idx, o_idx, "probe idx")
            eq(delta, o_delta, "probe delta")
            eq(tab, o_tab, "probe table'")
        elif reader in ("sorted_multi", "lut_multi"):
            v = SORTED if reader == "sorted_multi" else LUT
            self.set_variant(v)
            got = self.multi_call([(pc, pm), (pc[::-1].copy(), pm[::-1].copy())], self.ts.cuda_stream, False)
            self.multi_batches += 2
            self.lut_built |= v == LUT
            for k, (idx, delta, tab) in enumerate(got):
                eq(idx, o_idx if k == 0 else o_idx[::-1], f"probe batch {k} idx")
                eq(delta, o_delta, f"probe batch {k} delta")
                eq(tab, o_tab, f"probe batch {k} table'")
        elif reader == "packed":
            idx, dc, dm = self.a.bestfit_packed(pack(pc, pm), commit=False)
            self.seq_scans += 1
            eq(idx.astype(np.int32), o_idx, "probe idx")
            eq(np.concatenate([dc, dm]), o_delta, "probe delta")
        elif reader == "pipelined":
            # two launches with EGPU_F_INPUTS_READY on one stream, disjoint outputs: the second pipelines
            # behind the first under the sequence's own variant
            R, D = pc.size, fc.size
            bufs = [(self.dev(pc), self.dev(pm)) + self.outs(R, D),
                    (self.dev(pc[::-1].copy()), self.dev(pm[::-1].copy())) + self.outs(R, D)]
            self.sync()
            for c, m, idx, delta, tab in bufs:
                self.a.bestfit_dev(c.data_ptr(), m.data_ptr(), R, idx.data_ptr(), delta.data_ptr(), tab.data_ptr(), False,
                                   self.ts.cuda_stream, inputs_ready=True)
            self.sync()
            self.scanned(2)
            for k, (c, m, idx, delta, tab) in enumerate(bufs):
                got = idx.cpu().numpy()
                eq(got[:R], o_idx if k == 0 else o_idx[::-1], f"probe launch {k} idx")
                eq(got[R:], -9, "guard words")
                eq(delta.cpu().numpy(), o_delta, f"probe launch {k} delta")
                eq(tab.cpu().numpy(), o_tab, f"probe launch {k} table'")
        else:
            raise AssertionError(reader)
        self.set_variant(keep)

    def multi_call(self, batches, stream, ready):
        """batches: [(rc, rm)] host arrays -> [(idx, delta, table')] of one multi-batch launch"""
        D = self.m.D
        keep, tup = [], []
        for rc, rm in batches:
            R = rc.size
            t = (self.dev(rc), self.dev(rm)) + self.outs(R, D)
            keep.append((R, t))
            tup.append((t[0].data_ptr(), t[1].data_ptr(), R, t[2].data_ptr(), t[3].data_ptr(), t[4].data_ptr()))
        self.sync()
        self.a.bestfit_batches_dev(tup, stream, inputs_ready=ready)
        self.sync()
        out = []
        for R, (_, _, idx, delta, tab) in keep:
            got = idx.cpu().numpy()
            eq(got[R:], -9, "guard words")
            out.append((got[:R], delta.cpu().numpy(), tab.cpu().numpy()))
        return out

    # -- table-changing operations --
    def op_set_table(self, rng):
        D = D_WALK[(walk_start(self.seed) + self.n_set) % len(D_WALK)]
        self.n_set += 1
        if self.m.fc is not None and D != self.m.D and self.lut_built:
            self.switched_d_after_lut = True
        fc, fm = random_table(rng, D)
        self.a.set_table(fc, fm)
        self.m.set_table(fc, fm)

    def _commit_expect(self, rc, rm, idx, dc, dm, tab=None):
        o_idx, o_dc, o_dm, o_tab = self.oracle(rc, rm)
        eq(idx, o_idx, "idx")
        eq(dc, o_dc, "delta_core")
        eq(dm, o_dm, "delta_mem")
        if tab is not None:
            eq(tab, o_tab, "table'")
        self.m.commit_snapshot(o_tab)

    def _oversubscribing(self, rng):
        """rows that overfill one device: the same request (half a device's capacity) many times"""
        rc, rm = self.rows(rng)
        if rc.size >= 5 and rng.integers(0, 2):
            d = int(rng.integers(0, self.m.D))
            rc[: rc.size // 2] = max(1, int(self.m.fc[d]) // 2)
            rm[: rc.size // 2] = int(self.m.fm[d]) // 2
        return rc, rm

    def op_commit_host(self, rng):
        self.pick_variant(rng)
        rc, rm = self._oversubscribing(rng)
        idx, dc, dm = self.a.bestfit(rc, rm, commit=True)
        self.scanned()
        self._commit_expect(rc, rm, idx, dc, dm)

    def op_commit_zero_copy(self, rng):
        self.pick_variant(rng)
        rc, rm = self._oversubscribing(rng)
        R = max(1, rc.size)
        rc, rm = (rc, rm) if rc.size else self.rows(rng, 1)
        bufs = [self.a.pinned_array(R) for _ in range(3)]
        try:
            bufs[0][:] = rc
            bufs[1][:] = rm
            idx, dc, dm = self.a.bestfit(bufs[0], bufs[1], commit=True, out_idx=bufs[2])
            self.scanned()
            self._commit_expect(rc, rm, idx.copy(), dc, dm)
        finally:
            for b in bufs:
                self.a.host_free(b.ctypes.data)

    def op_commit_dev(self, rng):
        self.pick_variant(rng)
        rc, rm = self._oversubscribing(rng)
        idx, delta, tab = self.dev_call(rc, rm, True, self.stream(rng), ready=bool(rng.integers(0, 2)))
        self.scanned()
        D = self.m.D
        self._commit_expect(rc, rm, idx, delta[:D], delta[D:], tab)

    def op_commit_packed(self, rng):
        rc, rm = self._oversubscribing(rng)
        words = pack(rc, rm)
        if words.size:  # words the int32 arrays cannot express: core 101..127, not a request
            words[rng.integers(0, words.size, 2)] = (np.uint32(120) << np.uint32(18)) | np.uint32(5)
            words[rng.integers(0, words.size)] = np.uint32(1 << 26)
        c = np.where(words < (1 << 25), words >> 18, -1).astype(np.int32)
        m = np.where(words < (1 << 25), words & MEM_MAX, -1).astype(np.int32)
        idx, dc, dm = self.a.bestfit_packed(words, commit=True)
        self.seq_scans += 1
        self._commit_expect(c, m, idx.astype(np.int32), dc, dm)

    def op_commit_packed_dev(self, rng):
        t = self.torch
        rc, rm = self._oversubscribing(rng)
        R, D = rc.size, self.m.D
        words = self.dev(pack(rc, rm).view(np.int32))
        idx8 = t.full((R + 16,), -9, dtype=t.int8, device="cuda")
        _, delta, tab = self.outs(0, D)
        self.sync()
        s = self.stream(rng)
        rcode = self.egpu.load().egpu_bestfit_batch_packed_dev(self.a.handle, C.c_void_p(words.data_ptr()), R,
                                                               C.c_void_p(idx8.data_ptr()), C.c_void_p(delta.data_ptr()),
                                                               C.c_void_p(tab.data_ptr()), 1, C.c_void_p(s))
        assert rcode == 0, rcode
        self.sync()
        self.seq_scans += 1
        got = idx8.cpu().numpy().astype(np.int32)
        eq(got[R:], -9, "guard bytes")
        delta = delta.cpu().numpy()
        self._commit_expect(rc, rm, got[:R], delta[:D], delta[D:], tab.cpu().numpy())

    def _prefix_expect(self, rc, rm, idx, delta, tab=None):
        fc, fm = self.m.table32()
        o_idx, o_dc, o_dm, o_tab = self.oc.prefix_commit(fc, fm, rc, rm)
        eq(idx, o_idx, "idx")
        eq(delta, np.concatenate([o_dc, o_dm]), "delta")
        if tab is not None:
            eq(tab, o_tab, "table'")
        D = self.m.D
        self.m.install(o_tab[:D], o_tab[D:2 * D])

    def op_prefix_host(self, rng):
        self.pick_variant(rng, grid_ok=False)
        rc, rm = self._oversubscribing(rng)
        idx, dc, dm = self.a.bestfit(rc, rm, commit=True, prefix_commit=True)
        self.scanned()
        self._prefix_expect(rc, rm, idx, np.concatenate([dc, dm]))

    def op_prefix_dev(self, rng):
        self.pick_variant(rng, grid_ok=False)
        rc, rm = self._oversubscribing(rng)
        idx, delta, tab = self.dev_call(rc, rm, True, self.stream(rng), prefix=True)
        self.scanned()
        self._prefix_expect(rc, rm, idx, delta, tab)

    def _rounds_expect(self, rc, rm, max_rounds, idx, delta, rounds, left):
        fc, fm = self.m.table32()
        o_idx, o_dc, o_dm, o_fc, o_fm, o_rounds, o_left = self.oc.rounds(fc, fm, rc, rm, max_rounds)
        eq(idx, o_idx, "idx")
        eq(delta, np.concatenate([o_dc, o_dm]), "delta")
        assert (rounds, left) == (o_rounds, o_left), f"(rounds, deferred) {(rounds, left)} != {(o_rounds, o_left)}"
        self.m.install(o_fc, o_fm)
        return o_rounds

    def op_rounds_host(self, rng):
        self.pick_variant(rng, grid_ok=False)
        rc, rm = self._oversubscribing(rng)
        max_rounds = int(rng.choice([1, 2, 1 << 20]))
        idx, dc, dm, rounds, left = self.a.bestfit_rounds(rc, rm, max_rounds)
        self.scanned(self._rounds_expect(rc, rm, max_rounds, idx, np.concatenate([dc, dm]), rounds, left))

    def op_rounds_dev(self, rng):
        self.pick_variant(rng, grid_ok=False)
        rc, rm = self._oversubscribing(rng)
        R = rc.size
        max_rounds = int(rng.choice([1, 2, 1 << 20]))
        c, m = self.dev(rc), self.dev(rm)
        idx = self.outs(R, 1)[0]
        self.sync()
        delta, rounds, left = self.a.bestfit_rounds_dev(c.data_ptr(), m.data_ptr(), R, idx.data_ptr(), max_rounds,
                                                        self.stream(rng))
        self.sync()
        got = idx.cpu().numpy()
        eq(got[R:], -9, "guard words")
        self.scanned(self._rounds_expect(rc, rm, max_rounds, got[:R], delta, rounds, left))

    def _replay(self, kind, a, b):
        fc, fm = self.m.table32()
        o_idx, o_fc, o_fm = self.oc.replay(fc, fm, kind, a, b)
        eq(self.a.replay(kind, a, b), o_idx, "replay idx")
        self.m.install(o_fc, o_fm)

    def op_replay(self, rng):
        E = int(rng.choice([1, 255, 256, 257, 1000, 4097]))
        kind, a, b = churn(int(rng.integers(0, 1 << 30)), E)
        self._replay(kind, a, b)

    def op_replay_big(self, rng):
        E = REPLAY_SMEM_EVENTS + int(rng.integers(1, 6000))
        kind, a, b = churn(int(rng.integers(0, 1 << 30)), E)
        self._replay(kind, a, b)

    def op_apply_deltas(self, rng):
        t = self.torch
        D = self.m.D
        G = int(rng.choice([1, 3]))
        dl = np.zeros((G, 2 * D), np.int64)
        dl[:, :D] = rng.integers(0, 20, (G, D))
        dl[:, D:] = rng.integers(0, 3000, (G, D))
        if rng.integers(0, 3):  # non-negative demand that oversubscribes one device
            d = int(rng.integers(0, D))
            dl[0, d] += self.m.fc[d] + 1
            dl[G - 1, D + d] += int(rng.integers(0, 2)) * (self.m.fm[d] + 1)
        deltas = self.dev(dl.ravel())
        tab = self.outs(0, D)[2]
        self.sync()
        self.a.apply_deltas_dev(deltas.data_ptr(), G, tab.data_ptr(), True, self.stream(rng))
        self.sync()
        from oracle import bestfit_np
        o_tab = bestfit_np.apply_delta(self.m.fc, self.m.fm, dl[:, :D].sum(0), dl[:, D:].sum(0))
        eq(tab.cpu().numpy(), o_tab, "table'")
        self.m.commit_snapshot(o_tab)

    def op_shard_apply(self, rng):
        self.pick_variant(rng, grid_ok=False)
        rc, rm = self._oversubscribing(rng)
        R, D = rc.size, self.m.D
        c, m = self.dev(rc), self.dev(rm)
        idx, delta, tab = self.outs(R, D)
        s = self.ts.cuda_stream
        self.sync()
        self.a.bestfit_shard_dev(c.data_ptr(), m.data_ptr(), R, idx.data_ptr(), delta.data_ptr(), self.step, s)
        self.a.apply_peers_dev(self.step, tab.data_ptr(), True, s)
        self.step += 1
        self.sync()
        self.scanned()
        got = idx.cpu().numpy()
        eq(got[R:], -9, "guard words")
        delta = delta.cpu().numpy()
        self._commit_expect(rc, rm, got[:R], delta[:D], delta[D:], tab.cpu().numpy())
        assert self.a.peer_last_timeout == 0

    def op_shard_prefix(self, rng):
        self.pick_variant(rng, grid_ok=False)
        rc, rm = self._oversubscribing(rng)
        R, D = rc.size, self.m.D
        c, m = self.dev(rc), self.dev(rm)
        idx, delta, tab = self.outs(R, D)
        self.sync()
        self.a.bestfit_shard_prefix_dev(c.data_ptr(), m.data_ptr(), R, idx.data_ptr(), delta.data_ptr(), tab.data_ptr(),
                                        self.step, commit=True, stream=self.ts.cuda_stream)
        self.step += 2
        self.sync()
        self.scanned()
        got = idx.cpu().numpy()
        eq(got[R:], -9, "guard words")
        self._prefix_expect(rc, rm, got[:R], delta.cpu().numpy(), tab.cpu().numpy())
        assert self.a.peer_last_timeout == 0

    def _restore(self, rng, install):
        from elastic_gpu_agent_b200 import restore
        from oracle import restore_py
        D = self.m.D
        case = restore_case(rng, D)
        o_fc, o_fm, o_ov, o_counts, o_rstat = restore_py.restore(case["records"], case["links"], case["cap_core"],
                                                                 case["cap_mem"])
        if rng.integers(0, 2):
            fc, fm, ov, status = restore.restore_table_flat(self.a, case["sets"], case["hashes"], case["resources"],
                                                            case["set_links"], case["cap_core"], case["cap_mem"],
                                                            install=install)
            eq(status, o_rstat, "entry status")
        else:
            fc, fm, ov, counts, rstat = restore.restore_table(self.a, case["records"], case["links"], case["cap_core"],
                                                              case["cap_mem"], install=install)
            eq(counts, o_counts, "status counts")
            eq(rstat, o_rstat, "record status")
        eq(fc, o_fc, "restored free_core")
        eq(fm, o_fm, "restored free_mem")
        eq(ov, o_ov, "restored oversub")
        if install:
            self.m.set_table(o_fc, o_fm, o_ov)

    def op_restore_install(self, rng):
        self._restore(rng, True)

    # -- operations that leave the table alone --
    def op_restore_only(self, rng):
        self._restore(rng, False)

    def op_multi(self, rng, big=False):
        self.pick_variant(rng, grid_ok=False)
        K = 4 if big else int(rng.choice([32, 48, 64]))
        sizes = [int(rng.choice((0,) + ROWS[:6])) for _ in range(K)]
        if big:  # the largest batch decides the grid rule: >= 512 Ki rows takes the whole-wave branch
            sizes = [600_011, 0, 5, 70_003]
        batches = [self.rows(rng, R) for R in sizes]
        got = self.multi_call(batches, self.stream(rng), bool(rng.integers(0, 2)))
        self.multi_batches += K
        self.lut_built |= self.uses_lut()
        for k, ((rc, rm), (idx, delta, tab)) in enumerate(zip(batches, got)):
            o_idx, o_dc, o_dm, o_tab = self.oracle(rc, rm)
            eq(idx, o_idx, f"batch {k} idx")
            eq(delta, np.concatenate([o_dc, o_dm]), f"batch {k} delta")
            eq(tab, o_tab, f"batch {k} table'")

    def op_multi_big(self, rng):
        self.op_multi(rng, big=True)

    def op_snapshot(self, rng):
        self.pick_variant(rng)
        rc, rm = self.rows(rng)
        if rng.integers(0, 2):
            idx, dc, dm = self.a.bestfit(rc, rm, commit=False)
            tab = None
        else:
            idx, delta, tab = self.dev_call(rc, rm, False, self.stream(rng), ready=bool(rng.integers(0, 2)))
            dc, dm = delta[:self.m.D], delta[self.m.D:]
        self.scanned()
        o_idx, o_dc, o_dm, o_tab = self.oracle(rc, rm)
        eq(idx, o_idx, "idx")
        eq(np.concatenate([dc, dm]), np.concatenate([o_dc, o_dm]), "delta")
        if tab is not None:
            eq(tab, o_tab, "table'")

    def op_pipelined_chain(self, rng):
        """n non-committing launches with EGPU_F_INPUTS_READY on one stream, disjoint outputs; 26 > the
        24 launches of a pipelined group"""
        self.pick_variant(rng)
        n = int(rng.choice([5, 26]))
        D = self.m.D
        cases = [self.rows(rng, int(rng.choice(ROWS[1:]))) for _ in range(n)]
        bufs = [(self.dev(rc), self.dev(rm)) + self.outs(rc.size, D) for rc, rm in cases]
        self.sync()
        for (rc, _), (c, m, idx, delta, tab) in zip(cases, bufs):
            self.a.bestfit_dev(c.data_ptr(), m.data_ptr(), rc.size, idx.data_ptr(), delta.data_ptr(), tab.data_ptr(), False,
                               self.ts.cuda_stream, inputs_ready=True)
        self.sync()
        self.scanned(n)
        for k, ((rc, rm), (_, _, idx, delta, tab)) in enumerate(zip(cases, bufs)):
            o_idx, o_dc, o_dm, o_tab = self.oracle(rc, rm)
            got = idx.cpu().numpy()
            eq(got[:rc.size], o_idx, f"launch {k} idx")
            eq(got[rc.size:], -9, f"launch {k} guard words")
            eq(delta.cpu().numpy(), np.concatenate([o_dc, o_dm]), f"launch {k} delta")
            eq(tab.cpu().numpy(), o_tab, f"launch {k} table'")

    def op_query(self, rng):
        D = int(rng.choice(D_WALK))
        fc, fm = random_table(rng, D)
        rc, rm = requests_for(rng, fc, fm, int(rng.choice(ROWS[1:])))
        eq(self.a.query(fc, fm, rc, rm), self.oracle(rc, rm, fc, fm)[0], "query idx")

    def op_preferred(self, rng):
        from elastic_gpu_agent_b200 import plugin
        lib = self.egpu.load()
        resource = int(rng.integers(0, 2))
        requests = []
        for _ in range(int(rng.integers(1, 6))):
            avail = ["%d-%02d" % (g, u) for g in rng.choice(8, int(rng.integers(1, 4)), replace=False)
                     for u in sorted(rng.choice(100, int(rng.integers(1, 60)), replace=False))]
            must = list(rng.choice(avail, int(rng.integers(0, 2)), replace=False))
            requests.append((avail, must, int(rng.integers(1, 40))))
        flat, io, so, sz = plugin.flatten_requests(requests)
        pos, gpu, rcs = plugin.preferred_allocation_batch_flat(self.a, resource, flat, io, so, sz)
        off = 0
        for q, (avail, must, n) in enumerate(requests):
            av = (C.c_char_p * len(avail))(*[s.encode() for s in avail])
            mu = (C.c_char_p * max(1, len(must)))(*[s.encode() for s in must])
            out = np.full(n, -1, np.int32)
            g = C.c_int32(-1)
            e_rc = lib.egpu_preferred_allocation(self.a.handle, av, len(avail), mu, len(must), n, resource,
                                                 C.c_void_p(out.ctypes.data), C.byref(g))
            assert rcs[q] == e_rc, (q, rcs[q], e_rc)
            if e_rc == 0:
                assert gpu[q] == g.value and pos[off:off + n].tolist() == out.tolist(), q
            off += n

    def op_devhash(self, rng):
        from elastic_gpu_agent_b200 import devhash
        from oracle import restore_py
        sets = [["%d-%02d" % (int(rng.integers(0, 8)), int(u)) for u in rng.integers(0, 100, int(rng.integers(0, 12)))]
                for _ in range(int(rng.integers(1, 20)))]
        assert devhash.device_hashes(self.a, sets) == [restore_py.device_hash(s) for s in sets]
        request = list(rng.permutation(sets[int(rng.integers(0, len(sets)))]))
        cands = sets if rng.integers(0, 2) else sets[1:]
        exp = next((k for k, s in enumerate(cands) if sorted(s) == sorted(request)), -1)
        assert devhash.locate(self.a, request, cands) == exp

    def op_synth(self, rng):
        t = self.torch
        dist, sd, first = int(rng.choice([2, 3, 4])), int(rng.integers(0, 1000)), int(rng.integers(0, 1 << 20))
        R = int(rng.choice(ROWS[1:]))
        c = t.empty(R, dtype=t.int32, device="cuda")
        m = t.empty(R, dtype=t.int32, device="cuda")
        self.sync()
        self.a.synth_requests_dev(dist, sd, first, R, c.data_ptr(), m.data_ptr(), self.stream(rng))
        self.sync()
        rc, rm = self.egpu.synth.requests(dist, sd, R, first_row=first)
        eq(c.cpu().numpy(), rc, "synth core")
        eq(m.cpu().numpy(), rm, "synth mem")


def eq(got, exp, what):
    got, exp = np.asarray(got), np.asarray(exp)
    if got.shape != exp.shape and exp.ndim:
        raise AssertionError(f"{what}: shape {got.shape} != {exp.shape}")
    bad = np.flatnonzero(np.broadcast_to(got != exp, got.shape))
    if bad.size:
        i = int(bad[0])
        e = exp.ravel()[i] if exp.ndim else exp
        raise AssertionError(f"{what}: {bad.size} entries differ, first at {i}: {got.ravel()[i]} != {e}")


_CHURN = {}


def churn(seed, E):
    """cfg5-style churn with the odd cases (double frees, frees of later events, unknown kinds)"""
    from elastic_gpu_agent_b200 import synth
    if (seed, E) not in _CHURN:
        kind, a, b = (x.copy() for x in synth.churn_events(seed % 1000, E))
        rng = np.random.default_rng(seed)
        for i in rng.integers(0, E, max(1, E // 100)):
            r = rng.integers(0, 3)
            if r == 0:
                kind[i], a[i] = 1, i + 3
            elif r == 1:
                kind[i] = 7
            else:
                kind[i], a[i] = 1, max(0, i - 1)
        _CHURN[(seed, E)] = (kind, a, b)
    return _CHURN[(seed, E)]


def restore_case(rng, D):
    """records / links / flat sets for one restore: partial and whole-card core entries, memory entries,
    entries without a link, with a link outside the table or with a stale hash; small capacities so that
    some devices come back oversubscribed"""
    from oracle import restore_py
    cap_c = rng.integers(0, 101, D).astype(np.int32)
    cap_m = rng.integers(0, MEM_MAX + 1, D).astype(np.int32)
    small = rng.random(D) < 0.4
    cap_c[small] = rng.integers(0, 40, small.sum())
    cap_m[small] = rng.integers(0, 100, small.sum())
    sets, hashes, resources, set_links, records, links = [], [], [], [], [], []
    for e in range(int(rng.integers(1, 8))):
        kind = int(rng.integers(0, 6))
        res = restore_py.MEM if kind == 2 else restore_py.CORE
        cards = int(rng.integers(1, min(3, D) + 1)) if kind == 1 else 0
        n = 100 * cards + int(rng.integers(0, 100)) if kind == 1 else int(rng.integers(1, 120 if kind == 2 else 101))
        ids = sorted("%d-%02d" % (e + 1, j) for j in range(n))
        h = "zzzzzzzz" if kind == 4 else restore_py.device_hash(ids)
        gpus = [int(g) for g in rng.choice(D, max(1, cards), replace=False)]
        if kind == 3:
            gpus[0] = -1  # no link
        elif kind == 5:
            gpus[0] = D   # a link to a GPU outside the table
        sets.append(ids)
        hashes.append(h)
        resources.append(0 if res == restore_py.CORE else 1)
        set_links.append(gpus)
        for i, g in enumerate(gpus):
            if g >= 0:
                links.append((f"elastic-gpu-{h}-{i}", f"/dev/nvidia{g}"))
        body = {"c": {"Hash": h, "List": ids, "ResourceName": res}}
        records.append((f"ns/pod{e}".encode(), json.dumps(body, separators=(",", ":")).encode()))
    return dict(cap_core=cap_c, cap_mem=cap_m, sets=sets, hashes=hashes, resources=resources, set_links=set_links,
                records=records, links=links)


def run_sequence(seed, replay_kernel, upto=None):
    """Runs sequence `seed` on a fresh context under one replay kernel, operations 0..upto (all by
    default), each followed by both read-backs; a failure names the seed, the operation and the reader.
    Returns the Run."""
    import torch

    import elastic_gpu_agent_b200 as egpu
    from oracle import oracle_c
    oracle_c.load()
    variant, general = REPLAY_KERNELS[replay_kernel]
    old = {k: os.environ.get(k) for k in ("EGPU_REPLAY_VARIANT", "EGPU_REPLAY_GENERAL")}
    os.environ["EGPU_REPLAY_VARIANT"], os.environ["EGPU_REPLAY_GENERAL"] = variant, general
    try:
        alloc = egpu.BestFitAllocator(0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    names = plan(seed)
    last = len(names) - 1 if upto is None else upto
    try:
        run = Run(alloc, egpu, oracle_c, torch, seed)
        alloc.peer_attach(0, 1, [alloc.peer_export()])
        for i, name in enumerate(names[:last + 1]):
            where = f"seed {seed}, replay kernel {replay_kernel}, op {i} ({name}, D = {run.m.D if run.m.fc is not None else '-'})"
            rng = np.random.default_rng([seed, i])
            try:
                getattr(run, "op_" + name)(rng)
                run.sync()
            except AssertionError as ex:
                raise AssertionError(f"{where}, the operation's own outputs: {ex}") from ex
            readers = READERS if i == len(names) - 1 else (READERS[i % len(READERS)],)
            if OPS[name][0] and not {"lut", "lut_multi"} & set(readers):
                readers += ("lut",)  # the lookup tables must have been rebuilt before the next call reads them
            for reader in ("table()",) + readers:
                try:
                    run.check_table() if reader == "table()" else run.read(reader)
                except AssertionError as ex:
                    raise AssertionError(f"{where}, reader {reader}: {ex}") from ex
        alloc.peer_detach()
        return run
    finally:
        alloc.close()


# ---- tests that need no GPU ----------------------------------------------------------------------------
def test_model_matches_the_oracles_on_short_chains(oracle_c):
    """commit chains (clamping, sticky flags, set_table clearing them), prefix-commit, rounds and replay,
    composed by the model, against the oracles applied call after call"""
    from oracle import bestfit_np
    rng = np.random.default_rng(5)
    for D in (1, 5, 9, 33, 64):
        fc, fm = random_table(rng, D)
        m = Model()
        m.set_table(fc, fm)
        flags = np.zeros(D, np.int64)
        cur_c, cur_m = fc.astype(np.int64), fm.astype(np.int64)
        for k in range(6):
            rc, rm = requests_for(rng, cur_c, cur_m, 2000)
            o = bestfit_np.snapshot(cur_c.astype(np.int32), cur_m.astype(np.int32), rc, rm)
            assert all(np.array_equal(a, b) for a, b in zip(o, oracle_c.snapshot(cur_c, cur_m, rc, rm)))
            tab = o[3].astype(np.int64)
            m.commit_snapshot(o[3])
            cur_c, cur_m = np.maximum(tab[:D], 0), np.maximum(tab[D:2 * D], 0)
            flags |= (tab[:D] < 0) | (tab[D:2 * D] < 0)
            assert np.array_equal(m.fc, cur_c) and np.array_equal(m.fm, cur_m) and np.array_equal(m.ov, flags)
            assert (m.fc >= 0).all() and (m.fm >= 0).all()
        assert flags.any(), "the chain never oversubscribed"
        # prefix-commit and rounds keep the flags; numpy and C oracles agree
        rc, rm = requests_for(rng, m.fc, m.fm, 3000)
        p_np = bestfit_np.prefix_commit(m.fc, m.fm, rc, rm)
        p_c = oracle_c.prefix_commit(m.fc.astype(np.int32), m.fm.astype(np.int32), rc, rm)
        assert all(np.array_equal(a, b) for a, b in zip(p_np, p_c))
        m.install(p_c[3][:D], p_c[3][D:2 * D])
        assert np.array_equal(m.ov, flags) and not p_c[3][2 * D:].any()
        r_np = bestfit_np.rounds(m.fc, m.fm, rc, rm, 3)
        r_c = oracle_c.rounds(m.fc.astype(np.int32), m.fm.astype(np.int32), rc, rm, 3)
        assert all(np.array_equal(a, b) for a, b in zip(r_np, r_c))
        kind, a, b = churn(D, 3000)
        fc32, fm32 = m.table32()
        assert all(np.array_equal(x, y) for x, y in zip(bestfit_np.replay(fc32, fm32, kind, a, b),
                                                         oracle_c.replay(fc32, fm32, kind, a, b)))
        m.set_table(fc, fm)
        assert not m.ov.any()


def test_probe_rows_decide_every_row_of_the_table():
    """with distinct rows, every device is the answer to its own exact-fit probe, and to no other
    device's; so a stale row of the sorted view or the lookup tables changes some probe answer"""
    from oracle import bestfit_np
    rng = np.random.default_rng(9)
    for D in D_WALK + (2, 31, 32, 63):
        for _ in range(20):
            fc = rng.integers(0, 101, D)
            fm = rng.choice(MEM_MAX + 1, D, replace=False)
            pc, pm = probe_rows(fc, fm)
            idx = bestfit_np.snapshot(fc, fm, pc, pm)[0]
            exact = idx[4::9][:D]  # row (fc[d], fm[d]) of every device
            assert np.array_equal(exact, np.arange(D))
            assert set(idx.tolist()) >= set(range(D))
        # ties: the exact-fit probe of a duplicated row answers the lowest index holding it
        fc, fm = np.array([50] * D), np.array([7] * D)
        assert (bestfit_np.snapshot(fc, fm, *probe_rows(fc, fm))[0][4::9][:D] == 0).all()


def test_sequences_cover_what_the_issue_of_state_needs():
    """every operation in every sequence; replays at D <= 8 and 9..32 (the one-warp and two-warp kernels)
    and one above the shared-memory limit; set_table walks all D buckets; one multi-batch launch takes the
    >= 512 Ki-row branch"""
    seen_d = set()
    for seed in SEEDS:
        names = plan(seed)
        assert names[0] == "set_table" and 30 <= len(names) <= 60
        assert set(names) >= set(ALL_OPS) - {"multi_big"}
        assert names.count("multi") >= 5
        replay_d = [d_at(seed, i) for i, n in enumerate(names) if n.startswith("replay")]
        seen_d |= {d_at(seed, i) for i in range(1, len(names))}
        assert "replay_big" in names and replay_d
    assert sum(plan(s).count("multi_big") for s in SEEDS) == 1
    assert seen_d >= {1, 5, 8, 9, 16, 17, 33, 64}
    replay_d = [d_at(s, i) for s in SEEDS for i, n in enumerate(plan(s)) if n.startswith("replay")]
    assert any(d <= 8 for d in replay_d) and any(8 < d <= 32 for d in replay_d) and any(d > 32 for d in replay_d)


def test_every_entry_point_has_a_decision():
    """every `int egpu_*` of include/*.h is an operation of the sequences or listed as leaving the table
    alone, with its reason: a new entry point needs a decision here"""
    declared = set()
    for f in sorted(os.listdir(os.path.join(ROOT, "include"))):
        if f.endswith(".h"):
            declared |= set(re.findall(r"^int\s+(egpu_\w+)\s*\(", open(os.path.join(ROOT, "include", f)).read(), re.M))
    vocabulary = {e for _, entries in OPS.values() for e in entries}
    assert not vocabulary & set(NO_TABLE_CHANGE)
    assert declared == vocabulary | set(NO_TABLE_CHANGE), (declared ^ (vocabulary | set(NO_TABLE_CHANGE)))
    assert all(NO_TABLE_CHANGE.values())


# ---- GPU ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("replay_kernel", list(REPLAY_KERNELS))
@pytest.mark.parametrize("seed", SEEDS)
def test_context_sequence(seed, replay_kernel):
    run = run_sequence(seed, replay_kernel)
    # the epilogue slot rings wrapped; a lookup table was built and then outlived a variant and a D switch
    assert run.seq_scans > 2 * 32, run.seq_scans
    assert run.multi_batches > 128, run.multi_batches
    assert run.switched_variant_after_lut and run.switched_d_after_lut


@pytest.mark.gpu
def test_restore_install_keeps_the_oversubscription_flag(alloc):
    """an oversubscribed node restored with EGPU_RESTORE_INSTALL stays flagged until egpu_table_set"""
    from elastic_gpu_agent_b200 import restore
    from oracle import restore_py
    ids = ["0-%02d" % u for u in range(60)]
    h = restore_py.device_hash(ids)
    fc, fm, ov, _ = restore.restore_table_flat(alloc, [ids], [h], [restore.RESOURCE_CORE], [[1]], [100, 40], [9, 9],
                                               install=True)
    assert fc.tolist() == [100, 0] and ov.tolist() == [0, 1]
    t_fc, t_fm, t_ov = alloc.table()
    assert t_fc.tolist() == [100, 0] and t_fm.tolist() == [9, 9] and t_ov.tolist() == [0, 1]
    alloc.bestfit(np.zeros(0, np.int32), np.zeros(0, np.int32), commit=True)
    assert alloc.table()[2].tolist() == [0, 1]
    alloc.set_table([100, 40], [9, 9])
    assert alloc.table()[2].tolist() == [0, 0]
