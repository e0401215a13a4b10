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
  - prefix-commit, rounds (host loop, packed, one launch, K batches in order, over row shards) and replay install
    their table and leave oversub as it was;
  - an accepted committing release (EGPU_F_RELEASE) installs free + U and leaves oversub; a refused one changes
    nothing but egpu_release_refusals, which the model counts;
  - restore with EGPU_RESTORE_INSTALL installs the restored table with its own oversubscription flags,
    EGPU_RESTORE_CHARGE installs max(free - U, 0) and ORs the flags, an accepted EGPU_RESTORE_RELEASE free + U;
  - everything else leaves the table alone.
Besides, a place-then-give-back operation checks, whatever the model says, that releasing a committing placement's
rows with its own index array gives back exactly the table it started from; and graph blocks capture one committing
launch on the harness's stream and replay it between eager calls (GraphOp).
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
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import release_np  # noqa: E402

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


def unpack(words):
    """the int32 requests packed words stand for: words >= 2^25 become (-1, -1), infeasible; core 101..127 is
    infeasible as it stands"""
    w = np.asarray(words, np.uint32)
    ok = w < (1 << 25)
    return np.where(ok, w >> 18, -1).astype(np.int32), np.where(ok, w & MEM_MAX, -1).astype(np.int32)


# ---- the operations --------------------------------------------------------------------------------------
# Flag sets: the macro names of include/*.h an operation passes, joined by "|"; "" = no flags, "commit=1" = the
# int commit argument of the apply calls.
C1 = "EGPU_F_COMMIT"
PC = "EGPU_F_PREFIX_COMMIT|EGPU_F_COMMIT"
PPC = "EGPU_F_PACKED|EGPU_F_PREFIX_COMMIT|EGPU_F_COMMIT"
PROUNDS = "EGPU_F_PACKED|EGPU_F_PREFIX_COMMIT|EGPU_F_COMMIT|EGPU_F_ROUNDS"
DROUNDS = "EGPU_F_PREFIX_COMMIT|EGPU_F_COMMIT|EGPU_F_ROUNDS|EGPU_F_DEVICE_ROUNDS"
PDROUNDS = "EGPU_F_PACKED|" + DROUNDS
REL, RELC = "EGPU_F_RELEASE", "EGPU_F_RELEASE|EGPU_F_COMMIT"
PREL, PRELC = "EGPU_F_RELEASE|EGPU_F_PACKED", "EGPU_F_RELEASE|EGPU_F_COMMIT|EGPU_F_PACKED"
RES_INSTALL, RES_CHARGE, RES_RELEASE = ("EGPU_RESTORE_VERIFY|EGPU_RESTORE_" + f for f in ("INSTALL", "CHARGE", "RELEASE"))


def both(entries, *flag_sets):
    return tuple((e, f) for e in entries for f in flag_sets)


BATCH, BATCH_DEV, SHARD_PREFIX = ("egpu_bestfit_batch",), ("egpu_bestfit_batch_dev",), ("egpu_bestfit_batch_shard_prefix_dev",)
BATCHES, BATCHES_SHARD = "egpu_bestfit_batches_dev", "egpu_bestfit_batches_shard_dev"
RESTORES = ("egpu_table_restore_flat", "egpu_table_restore")
# The graph operations: a capture issues one of these launches on the harness's stream, a replay runs it again.
# (kind, packed) -> the (entry point, flag set) it passes.
GRAPH_CALLS = {
    ("commit_dev", False): ("egpu_bestfit_batch_dev", C1),
    ("prefix_dev", False): ("egpu_bestfit_batch_dev", PC), ("prefix_dev", True): ("egpu_bestfit_batch_dev", PPC),
    ("device_rounds_dev", False): ("egpu_bestfit_batch_dev", DROUNDS),
    ("device_rounds_dev", True): ("egpu_bestfit_batch_dev", PDROUNDS),
    ("multi_rounds", False): (BATCHES, DROUNDS), ("multi_rounds", True): (BATCHES, PDROUNDS),
    ("release_dev", False): ("egpu_bestfit_batch_dev", RELC), ("release_dev", True): ("egpu_bestfit_batch_dev", PRELC),
    ("shard_rounds", False): (SHARD_PREFIX[0], DROUNDS), ("shard_rounds", True): (SHARD_PREFIX[0], PDROUNDS),
    ("release_shard", False): (SHARD_PREFIX[0], RELC), ("release_shard", True): (SHARD_PREFIX[0], PRELC),
    ("shard_prefix_multi", False): (BATCHES_SHARD, PC), ("shard_prefix_multi", True): (BATCHES_SHARD, PPC),
}
GRAPH_SPECS = tuple(GRAPH_CALLS)
GRAPH_KINDS = tuple(dict.fromkeys(k for k, _ in GRAPH_SPECS))
# The place-then-give-back operation: (placement, packed) -> the placement's (entry point, flag set); the rows then
# go back through egpu_bestfit_batch_dev with EGPU_F_RELEASE | EGPU_F_COMMIT, int32 or packed.
GIVE_BACK_CALLS = {
    ("prefix", False): ("egpu_bestfit_batch_dev", PC), ("prefix", True): ("egpu_bestfit_batch_dev", PPC),
    ("device_rounds", False): ("egpu_bestfit_batch_dev", DROUNDS), ("device_rounds", True): ("egpu_bestfit_batch_dev", PDROUNDS),
    ("multi_rounds", False): (BATCHES, DROUNDS), ("multi_rounds", True): (BATCHES, PDROUNDS),
    ("shard_rounds", False): (SHARD_PREFIX[0], DROUNDS), ("shard_rounds", True): (SHARD_PREFIX[0], PDROUNDS),
}
GIVE_BACK_SPECS = tuple(GIVE_BACK_CALLS)
# Operations made of the calls of others, which declare what they pass but do not count towards COMMITTING
COMPOSITE = ("give_back", "graph_capture", "graph_replay")
# name -> (changes the table, ((C entry point, flag set), ...) it calls).  An entry point of include/*.h is either
# named here or in NO_TABLE_CHANGE, and an EGPU_F_* / EGPU_RESTORE_* flag either appears here or in
# NO_TABLE_CHANGE_FLAGS; every committing flag set of COMMITTING is passed by an operation that is not COMPOSITE
# (test_every_entry_point_and_flag_set_has_a_decision).
OPS = {
    "set_table": (True, (("egpu_table_set", ""),)),
    "set_table_same": (True, (("egpu_table_set", ""),)),
    "commit_host": (True, both(BATCH, "", C1)),
    "commit_zero_copy": (True, (("egpu_bestfit_batch", C1), ("egpu_host_alloc", ""))),
    "commit_dev": (True, both(BATCH_DEV, C1, C1 + "|EGPU_F_INPUTS_READY")),
    "commit_packed": (True, (("egpu_bestfit_batch_packed", C1),)),
    "commit_packed_dev": (True, (("egpu_bestfit_batch_packed_dev", C1),)),
    "prefix_host": (True, both(BATCH, PC)),
    "prefix_dev": (True, both(BATCH_DEV, PC)),
    "packed_prefix_host": (True, both(BATCH, PPC)),
    "packed_prefix_dev": (True, both(BATCH_DEV, PPC)),
    "rounds_host": (True, (("egpu_bestfit_batch_rounds", ""),)),
    "rounds_dev": (True, (("egpu_bestfit_batch_rounds_dev", ""),)),
    "packed_rounds_host": (True, both(BATCH, PROUNDS)),
    "packed_rounds_dev": (True, both(BATCH_DEV, PROUNDS)),
    "device_rounds_host": (True, both(BATCH, DROUNDS, PDROUNDS)),
    "device_rounds_dev": (True, both(BATCH_DEV, DROUNDS, PDROUNDS)),
    "multi_rounds": (True, both(("egpu_bestfit_batches_dev",), DROUNDS, PDROUNDS)),
    "replay": (True, (("egpu_replay", ""),)),
    "replay_big": (True, (("egpu_replay", ""),)),
    "apply_deltas": (True, (("egpu_table_apply_deltas_dev", "commit=1"),)),
    "shard_apply": (True, (("egpu_bestfit_batch_shard_dev", ""), ("egpu_table_apply_peers_dev", "commit=1"),
                           ("egpu_table_apply_peers_multi_dev", "commit=1"))),
    "shard_prefix": (True, both(SHARD_PREFIX, PC)),
    "shard_prefix_packed": (True, both(SHARD_PREFIX, PPC)),
    "shard_prefix_multi": (True, both(("egpu_bestfit_batches_shard_dev",), "EGPU_F_PREFIX_COMMIT", PC,
                                      "EGPU_F_PACKED|EGPU_F_PREFIX_COMMIT", PPC)),
    "shard_rounds": (True, both(SHARD_PREFIX, DROUNDS, PDROUNDS)),
    "release_host": (True, both(BATCH, REL, RELC, PREL, PRELC)),
    "release_dev": (True, both(BATCH_DEV, REL, RELC, PREL, PRELC)),
    "release_shard": (True, both(SHARD_PREFIX, REL, RELC, PREL, PRELC)),
    "restore_install": (True, both(RESTORES, RES_INSTALL)),
    "restore_charge": (True, both(RESTORES, RES_CHARGE)),
    "restore_release": (True, both(RESTORES, RES_RELEASE)),
    # what the sequences of SEEDS x REPLAY_KERNELS really pass (test_composite_operations_declare_what_they_pass)
    "give_back": (True, tuple(GIVE_BACK_CALLS.values()) + both(BATCH_DEV, RELC, PRELC)),
    "graph_capture": (True, (("egpu_table_set", ""),) + tuple(GRAPH_CALLS.values())),
    "graph_replay": (True, ()),
    "multi": (False, both(("egpu_bestfit_batches_dev",), "", "EGPU_F_INPUTS_READY")),
    "multi_big": (False, (("egpu_bestfit_batches_dev", ""), ("egpu_synth_requests_dev", ""))),
    "snapshot": (False, both(BATCH + BATCH_DEV, "")),
    "pipelined_chain": (False, both(BATCH_DEV, "EGPU_F_INPUTS_READY")),
    "query": (False, (("egpu_bestfit_query", ""),)),
    "preferred": (False, (("egpu_preferred_allocation_batch", ""), ("egpu_preferred_allocation", ""))),
    "devhash": (False, (("egpu_device_hash_batch", ""), ("egpu_device_hash", ""), ("egpu_device_locate", ""))),
    "restore_only": (False, both(RESTORES, "EGPU_RESTORE_VERIFY")),
    "synth": (False, (("egpu_synth_requests_dev", ""),)),
}

# Every flag set an entry point of include/*.h documents as changing the table (with the commit bit where it
# has one): each must be passed by some operation above.
COMMITTING = (
    both(BATCH, C1, PC, PPC, PROUNDS, DROUNDS, PDROUNDS, RELC, PRELC) +
    both(BATCH_DEV, C1, PC, PPC, PROUNDS, DROUNDS, PDROUNDS, RELC, PRELC) +
    both(("egpu_bestfit_batches_dev",), DROUNDS, PDROUNDS) +
    both(("egpu_bestfit_batches_shard_dev",), PC, PPC) +
    both(SHARD_PREFIX, PC, PPC, DROUNDS, PDROUNDS, RELC, PRELC) +
    both(("egpu_bestfit_batch_packed", "egpu_bestfit_batch_packed_dev"), C1) +
    both(RESTORES, RES_INSTALL, RES_CHARGE, RES_RELEASE) +
    both(("egpu_table_apply_deltas_dev", "egpu_table_apply_peers_dev", "egpu_table_apply_peers_multi_dev"), "commit=1") +
    (("egpu_table_set", ""), ("egpu_replay", ""), ("egpu_bestfit_batch_rounds", ""), ("egpu_bestfit_batch_rounds_dev", ""))
)

NO_TABLE_CHANGE_FLAGS = {
    "EGPU_F_APPLY": "the sharded snapshot steps' in-launch apply writes table' to d_table_out and never commits",
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
    "egpu_bestfit_batch_shard_lag_dev": "never commits (EGPU_F_COMMIT is refused)",
    "egpu_device_id_format": "string formatting, no context",
    "egpu_device_id_parse": "string parsing, no context",
}

ALL_OPS = tuple(OPS)
# every sequence: set_table first, then each operation once (set_table four times, multi-batch six and
# pipelined chains four: both epilogue rings must wrap; the three release forms twice, so that every sequence
# sees each outcome), then extra draws, and two graph blocks; multi_big in one sequence only
EXTRA = ("set_table", "commit_host", "commit_dev", "commit_dev", "commit_packed", "prefix_dev", "rounds_host", "replay",
         "replay", "apply_deltas", "shard_apply", "restore_install", "snapshot", "pipelined_chain", "set_table",
         "device_rounds_dev", "multi_rounds", "release_dev", "restore_charge")
GRAPH_OPS = ("graph_capture", "graph_replay", "set_table_same")
# what may sit inside a graph block: anything that keeps D
BLOCK_FILLERS = ("commit_dev", "packed_prefix_dev", "device_rounds_host", "multi_rounds", "release_dev", "restore_charge",
                 "apply_deltas", "replay", "shard_rounds", "pipelined_chain")
RELEASES = ("release_host", "release_dev", "release_shard")
READERS = ("sorted", "lut", "grid", "sorted_multi", "lut_multi", "packed", "pipelined")


def plan(seed):
    """the operation names of sequence `seed`, in order"""
    rng = np.random.default_rng(seed)
    body = [n for n in ALL_OPS if n not in ("set_table", "multi_big") + GRAPH_OPS] + ["multi"] * 5 + ["set_table"] * 3 + \
        ["pipelined_chain"] * 3 + list(RELEASES) + ["restore_release"] * 2 + ["give_back"]
    body += list(rng.choice(EXTRA, 10))
    if seed == SEEDS[0]:
        body.append("multi_big")
    rng.shuffle(body)
    # graph blocks: capture, a table change, egpu_table_set of the same D, replay, another change, replay
    for _ in range(2):
        block = ["graph_capture", str(rng.choice(BLOCK_FILLERS)), "set_table_same", "graph_replay",
                 str(rng.choice(BLOCK_FILLERS)), "graph_replay"]
        at = int(rng.integers(0, len(body) + 1))
        body[at:at] = block
    return ["set_table"] + body


def seed_index(seed):
    return SEEDS.index(seed) if seed in SEEDS else seed


def graph_spec(seed, n, replay_kernel):
    """(kind, packed) of the n-th capture (0 or 1) of sequence `seed` under `replay_kernel`: the 24 captures of
    SEEDS x REPLAY_KERNELS hold every spec"""
    k = list(REPLAY_KERNELS).index(replay_kernel)
    return GRAPH_SPECS[(8 * k + 2 * seed_index(seed) + n) % len(GRAPH_SPECS)]


def give_back_spec(seed, n, replay_kernel):
    """(placement, packed, packed release) of the n-th give-back (0 or 1) of sequence `seed` under `replay_kernel`:
    every placement in both formats under each kernel, each released in both formats over the kernels"""
    k = list(REPLAY_KERNELS).index(replay_kernel)
    s = seed_index(seed)
    return GIVE_BACK_SPECS[(2 * s + n) % len(GIVE_BACK_SPECS)] + ((s + n + k) % 2 == 1,)


def alternate(seed, replay_kernel, count):
    """the format of the count-th instance of a dedicated operation that takes both: int32 and packed alternate, and
    the first instance differs between the replay kernels"""
    return (seed_index(seed) + list(REPLAY_KERNELS).index(replay_kernel) + count) % 2 == 1


def walk_start(seed):
    """where sequence `seed` enters D_WALK: the sequences of SEEDS together cover all of it"""
    return 4 * SEEDS.index(seed) if seed in SEEDS else seed


def d_at(seed, upto):
    """D in force before operation `upto` of sequence `seed` (only set_table changes D)"""
    n = sum(1 for name in plan(seed)[:upto] if name == "set_table")
    return D_WALK[(walk_start(seed) + n - 1) % len(D_WALK)] if n else None


# ---- the sequence runner ------------------------------------------------------------------------------
class Run:
    def __init__(self, alloc, egpu, oracle_c, torch, seed, replay_kernel="two_warp"):
        self.a, self.egpu, self.oc, self.torch, self.seed = alloc, egpu, oracle_c, torch, seed
        self.replay_kernel = replay_kernel
        self.counts = {}             # instances of each dedicated operation that takes both formats
        self.n_give_back = 0
        self.m = Model()
        self.variant = AUTO
        self.n_set = 0
        self.step = 0            # exchange step of the world-1 peer calls
        self.seq_scans = 0       # single-batch scans and packed launches (epilogue slot seq mod 32)
        self.multi_batches = 0   # batches of multi-batch launches (slot mseq mod 128)
        self.lut_built = False
        self.switched_variant_after_lut = self.switched_d_after_lut = False
        self.ts = torch.cuda.Stream()
        self.refusals = 0           # release launches refused on the device (egpu_release_refusals)
        self.n_release = self.n_restore_release = 0
        self.outcomes, self.restore_outcomes = set(), set()  # "accepted", "flagged", "exceeds"
        self.graph = None           # the captured launch (GraphOp) while D stays
        self.n_graph = 0
        self.replays = 0
        self.next_id = 0            # device IDs of the restore records: unique over the sequence

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
        assert self.a.release_refusals == self.refusals, f"egpu_release_refusals {self.a.release_refusals} != {self.refusals}"

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
        if self.graph is not None and D != self.graph.D:
            self.graph = None  # a replay would run against a table of another size

    def op_set_table_same(self, rng):
        fc, fm = random_table(rng, self.m.D)
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

    def _oversubscribing(self, rng, R=None):
        """rows that overfill one device: the same request (half a device's capacity) many times"""
        rc, rm = self.rows(rng, R)
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

    # -- prefix-commit and rounds in the packed format, rounds in one launch, sharded forms at world 1 --
    def packed_next(self, name):
        """the format of this instance of operation `name` (see alternate)"""
        n = self.counts[name] = self.counts.get(name, -1) + 1
        return alternate(self.seed, self.replay_kernel, n)

    def one_launch(self, call):
        """the headers promise ONE launch (egpu_launch_count + 1) for the call"""
        n0 = self.a.launch_count
        call()
        assert self.a.launch_count == n0 + 1, f"{self.a.launch_count - n0} launches, not one"

    def placement_rows(self, rng, packed, R=None):
        """(words or None, c, m): rows that overfill a device; packed: the words, with a few that the int32 arrays
        cannot express, and the requests they stand for"""
        rc, rm = self._oversubscribing(rng, R)
        if not packed:
            return None, rc, rm
        words = pack(rc, rm)
        if words.size:
            words[rng.integers(0, words.size, 2)] = (np.uint32(120) << np.uint32(18)) | np.uint32(5)
            words[rng.integers(0, words.size)] = np.uint32(1 << 26)
        return (words,) + unpack(words)

    def rows_dev(self, words, c, m, R_buf=None):
        """device rows and a -9 filled index array: (core or words, mem or None, idx)"""
        t = self.torch
        R = c.size if R_buf is None else R_buf
        if words is not None:
            return self.dev(words.view(np.int32)), None, t.full((R + 16,), -9, dtype=t.int8, device="cuda")
        return self.dev(c), self.dev(m), t.full((R + 4,), -9, dtype=t.int32, device="cuda")

    def idx_back(self, idx, R):
        got = idx.cpu().numpy().astype(np.int32)
        eq(got[R:], -9, "guard words after idx")
        return got[:R]

    def _rounds_full(self, c, m, idx, delta, tab=None, table=None):
        """rounds with no round limit against `table` (the model's by default); returns the table they leave"""
        fc, fm = self.m.table32() if table is None else table
        o_idx, o_dc, o_dm, o_fc, o_fm, _, left = self.oc.rounds(fc, fm, c, m, 1 << 30)
        assert left == 0
        eq(idx, o_idx, "idx")
        eq(delta, np.concatenate([o_dc, o_dm]), "delta")
        if tab is not None:
            eq(tab, np.concatenate([o_fc, o_fm, np.zeros(fc.size, np.int32)]), "table'")
        return o_fc.astype(np.int32), o_fm.astype(np.int32)

    def _rounds_install(self, *a):
        self.m.install(*self._rounds_full(*a))

    def op_packed_prefix_host(self, rng):
        self.pick_variant(rng, grid_ok=False)
        words, c, m = self.placement_rows(rng, True)
        idx, dc, dm = self.a.bestfit_packed_prefix(words, commit=True)
        self.scanned()
        self._prefix_expect(c, m, idx.astype(np.int32), np.concatenate([dc, dm]))
        return c, m, idx.astype(np.int32)

    def op_packed_prefix_dev(self, rng, packed=True):
        self.pick_variant(rng, grid_ok=False)
        words, c, m = self.placement_rows(rng, packed)
        R, D = c.size, self.m.D
        cw, mm, idx = self.rows_dev(words, c, m)
        _, delta, tab = self.outs(0, D)
        self.sync()
        if packed:
            self.a.bestfit_packed_prefix_dev(cw.data_ptr(), R, idx.data_ptr(), delta.data_ptr(), tab.data_ptr(), commit=True,
                                             stream=self.stream(rng))
        else:
            self.a.bestfit_dev(cw.data_ptr(), mm.data_ptr(), R, idx.data_ptr(), delta.data_ptr(), tab.data_ptr(), True,
                               self.stream(rng), prefix_commit=True)
        self.sync()
        self.scanned()
        got = self.idx_back(idx, R)
        self._prefix_expect(c, m, got, delta.cpu().numpy(), tab.cpu().numpy())
        return c, m, got

    def op_packed_rounds_host(self, rng):
        self.pick_variant(rng, grid_ok=False)
        words, c, m = self.placement_rows(rng, True)
        idx, dc, dm = self.a.bestfit_packed_prefix(words, rounds=True)
        self.scanned()
        self._rounds_install(c, m, idx.astype(np.int32), np.concatenate([dc, dm]))

    def op_packed_rounds_dev(self, rng):
        self.pick_variant(rng, grid_ok=False)
        words, c, m = self.placement_rows(rng, True)
        R, D = c.size, self.m.D
        cw, _, idx = self.rows_dev(words, c, m)
        _, delta, tab = self.outs(0, D)
        self.sync()
        self.a.bestfit_packed_prefix_dev(cw.data_ptr(), R, idx.data_ptr(), delta.data_ptr(), tab.data_ptr(),
                                         stream=self.stream(rng), rounds=True)
        self.sync()
        self.scanned()
        self._rounds_install(c, m, self.idx_back(idx, R), delta.cpu().numpy(), tab.cpu().numpy())

    def op_device_rounds_host(self, rng):
        self.pick_variant(rng, grid_ok=False)
        packed = self.packed_next("device_rounds_host")
        words, c, m = self.placement_rows(rng, packed)
        out = []
        if packed:
            self.one_launch(lambda: out.extend(self.a.bestfit_packed_prefix(words, rounds=True, device=True)))
        else:
            self.one_launch(lambda: out.extend(self.a.bestfit_rounds(c, m, device=True)[:3]))
        self._rounds_install(c, m, out[0].astype(np.int32), np.concatenate(out[1:3]))

    def _device_rounds_dev(self, rng, packed, stream):
        words, c, m = self.placement_rows(rng, packed)
        R, D = c.size, self.m.D
        cw, mm, idx = self.rows_dev(words, c, m)
        _, delta, tab = self.outs(0, D)
        self.sync()
        if packed:
            self.one_launch(lambda: self.a.bestfit_packed_rounds_device_dev(cw.data_ptr(), R, idx.data_ptr(), delta.data_ptr(),
                                                                            tab.data_ptr(), stream))
        else:
            self.one_launch(lambda: self.a.bestfit_rounds_device_dev(cw.data_ptr(), mm.data_ptr(), R, idx.data_ptr(),
                                                                     delta.data_ptr(), tab.data_ptr(), stream))
        self.sync()
        got = self.idx_back(idx, R)
        self._rounds_install(c, m, got, delta.cpu().numpy(), tab.cpu().numpy())
        return c, m, got

    def op_device_rounds_dev(self, rng):
        self.pick_variant(rng, grid_ok=False)
        return self._device_rounds_dev(rng, self.packed_next("device_rounds_dev"), self.stream(rng))

    def _batches(self, rng, packed, sizes):
        """per batch (words, c, m) and device buffers (core or words, mem or None, idx, delta, table'), and the
        tuples of make_batches / make_packed_batches"""
        D = self.m.D
        rows, bufs, tup = [], [], []
        for R in sizes:
            words, c, m = self.placement_rows(rng, packed, R)
            b = self.rows_dev(words, c, m) + self.outs(0, D)[1:]
            rows.append((words, c, m))
            bufs.append(b)
            ptrs = (b[2].data_ptr(), b[3].data_ptr(), b[4].data_ptr())
            tup.append((b[0].data_ptr(), R) + ptrs if packed else (b[0].data_ptr(), b[1].data_ptr(), R) + ptrs)
        return rows, bufs, tup

    def op_multi_rounds(self, rng, packed=None):
        """K batches placed in order, each to its fixed point: ragged, with empty batches"""
        self.pick_variant(rng, grid_ok=False)
        packed = self.packed_next("multi_rounds") if packed is None else packed
        K = int(rng.choice([1, 3, 7]))
        sizes = [0 if k % 3 == 1 else int(rng.choice(ROWS[1:6])) for k in range(K)]
        rows, bufs, tup = self._batches(rng, packed, sizes)
        self.sync()
        self.one_launch(lambda: self.a.bestfit_batches_rounds_device_dev(tup, packed=packed, stream=self.stream(rng)))
        self.sync()
        cs, ms, ids = [], [], []
        for k, ((_, c, m), b) in enumerate(zip(rows, bufs)):
            got = self.idx_back(b[2], c.size)
            try:
                self._rounds_install(c, m, got, b[3].cpu().numpy(), b[4].cpu().numpy())
            except AssertionError as ex:
                raise AssertionError(f"batch {k} (R = {c.size}): {ex}") from ex
            cs.append(c)
            ms.append(m)
            ids.append(got)
        return np.concatenate(cs), np.concatenate(ms), np.concatenate(ids)

    def op_shard_prefix_packed(self, rng):
        self.pick_variant(rng, grid_ok=False)
        words, c, m = self.placement_rows(rng, True)
        R, D = c.size, self.m.D
        cw, _, idx = self.rows_dev(words, c, m)
        _, delta, tab = self.outs(0, D)
        self.sync()
        self.a.bestfit_shard_prefix_packed_dev(cw.data_ptr(), R, idx.data_ptr(), delta.data_ptr(), tab.data_ptr(), self.step,
                                               commit=True, stream=self.ts.cuda_stream)
        self.step += 2
        self.sync()
        self.scanned()
        self._prefix_expect(c, m, self.idx_back(idx, R), delta.cpu().numpy(), tab.cpu().numpy())
        assert self.a.peer_last_timeout == 0

    def op_shard_prefix_multi(self, rng):
        """K sharded prefix-commits in one launch: with EGPU_F_COMMIT each batch sees the table the one before it
        installed, without it every batch sees the current table"""
        self.pick_variant(rng, grid_ok=False)
        packed, commit = self.packed_next("shard_prefix_multi"), bool(rng.integers(0, 3))
        K = int(rng.choice([1, 2, 4]))
        rows, bufs, tup = self._batches(rng, packed, [int(rng.choice(ROWS[:6])) for _ in range(K)])
        self.sync()
        self.one_launch(lambda: self.a.bestfit_batches_shard_prefix_dev(tup, self.step, commit=commit, packed=packed,
                                                                        stream=self.ts.cuda_stream))
        self.step += 2 * K
        self.sync()
        self._shard_prefix_multi_expect(rows, bufs, commit)
        assert self.a.peer_last_timeout == 0

    def _shard_prefix_multi_expect(self, rows, bufs, commit):
        D = self.m.D
        fc, fm = self.m.table32()
        for k, ((_, c, m), b) in enumerate(zip(rows, bufs)):
            o_idx, o_dc, o_dm, o_tab = self.oc.prefix_commit(fc, fm, c, m)
            eq(self.idx_back(b[2], c.size), o_idx, f"batch {k} idx")
            eq(b[3].cpu().numpy(), np.concatenate([o_dc, o_dm]), f"batch {k} delta")
            eq(b[4].cpu().numpy(), o_tab, f"batch {k} table'")
            if commit:
                fc, fm = o_tab[:D].astype(np.int32), o_tab[D:2 * D].astype(np.int32)
        if commit:
            self.m.install(fc, fm)

    def op_shard_rounds(self, rng, packed=None):
        self.pick_variant(rng, grid_ok=False)
        packed = self.packed_next("shard_rounds") if packed is None else packed
        words, c, m = self.placement_rows(rng, packed)
        R, D = c.size, self.m.D
        cw, mm, idx = self.rows_dev(words, c, m)
        _, delta, tab = self.outs(0, D)
        self.sync()
        self.one_launch(lambda: self.a.bestfit_shard_rounds_dev(cw.data_ptr(), 0 if packed else mm.data_ptr(), R, idx.data_ptr(),
                                                                delta.data_ptr(), tab.data_ptr(), self.step, packed=packed,
                                                                stream=self.ts.cuda_stream))
        self.step += 2
        self.sync()
        got = self.idx_back(idx, R)
        self._rounds_install(c, m, got, delta.cpu().numpy(), tab.cpu().numpy())
        assert self.a.peer_last_timeout == 0
        return c, m, got

    # -- release: rows give back what they hold, all or nothing --
    def _flag_a_device(self, rng):
        """charge (EGPU_RESTORE_CHARGE) more than a device has free, so that it is flagged"""
        while not self.m.ov.any():
            g = int(rng.integers(0, self.m.D))
            n = int(self.m.fc[g]) + 1 if self.m.fc[g] < 100 else 50
            self._charge([(self.ids(n), 0, [g])], bool(rng.integers(0, 2)))

    def _unflag_a_device(self):
        """every device flagged leaves nothing to exceed on: egpu_table_set of the same table clears the flags"""
        if self.m.ov.all():
            fc, fm = self.m.table32()
            self.a.set_table(fc, fm)
            self.m.set_table(fc, fm)

    def release_rows(self, rng, target):
        """(c, m, idx) int32 rows aimed at outcome `target` ("accepted", "flagged", "exceeds"): room on unflagged
        devices split over rows, rows that hold nothing (idx -1, -2, D, out-of-domain requests), zero rows, and
        for "flagged" a row on a flagged device, for "exceeds" more than the domain allows on one device"""
        D = self.m.D
        if target == "flagged":
            self._flag_a_device(rng)
        elif target == "exceeds":
            self._unflag_a_device()
        fc, fm, ov = self.m.fc, self.m.fm, self.m.ov
        free = np.flatnonzero(ov == 0)
        rows = []
        for d in rng.permutation(free)[:3].tolist():
            a = int(rng.integers(0, 100 - fc[d] + 1))
            b = int(rng.integers(0, min(MEM_MAX - fm[d], 5000) + 1))
            x, y = int(rng.integers(0, a + 1)), int(rng.integers(0, b + 1))
            rows += [(x, y, d), (a - x, b - y, d)]
        rows += [(5, 5, -1), (5, 5, -2), (3, 3, D), (101, 0, 0), (0, MEM_MAX + 1, 0), (-1, 0, 0)]
        rows += [(0, 0, int(i)) for i in rng.integers(0, D, int(rng.choice([0, 600, 5000])))]
        if target == "flagged":
            rows.append((1, 0, int(rng.choice(np.flatnonzero(ov)))))
        elif target == "exceeds" and free.size:
            d = int(rng.choice(free))
            over = 100 - int(fc[d]) + 1
            rows += [(over // 2, 0, d), (over - over // 2, 0, d)]
        rows = np.array(rows, np.int64)[rng.permutation(len(rows))]
        return rows[:, 0].astype(np.int32), rows[:, 1].astype(np.int32), rows[:, 2].astype(np.int32)

    def next_target(self):
        self.n_release += 1
        return ("accepted", "flagged", "exceeds")[(self.n_release - 1) % 3]

    def _release_expect(self, c, m, idx, packed, u, tab, commit):
        """checks one release's sums and table' (either may be None) against release_np and advances the model"""
        D = self.m.D
        if packed:
            c, m = release_np.unpack(pack(c, m))
        o_u, o_tab, accepted = release_np.release(self.m.fc, self.m.fm, self.m.ov, c, m, idx)
        if u is not None:
            eq(u, o_u, "released sums")
        if tab is not None:
            eq(tab, o_tab, "table' and reason words")
        reasons = set(o_tab[2 * D:].tolist())
        self.outcomes |= ({"accepted"} if accepted else set()) | \
            ({"flagged"} if release_np.REL_FLAGGED in reasons else set()) | \
            ({"exceeds"} if release_np.REL_EXCEEDS in reasons else set())
        if not accepted:
            self.refusals += 1
        elif commit:
            self.m.install(o_tab[:D], o_tab[D:2 * D])
        return accepted

    def op_release_host(self, rng):
        c, m, idx = self.release_rows(rng, self.next_target())
        packed, commit = self.packed_next("release_host"), bool(rng.integers(0, 4))
        from elastic_gpu_agent_b200 import _lib as L
        try:
            u = np.concatenate(self.a.release(pack(c, m) if packed else c, None if packed else m, idx, commit=commit,
                                              packed=packed))
            refused = False
        except L.EgpuError as ex:
            assert ex.code == L.ERR_STATE, ex
            u, refused = np.concatenate(ex.released), True
        assert self._release_expect(c, m, idx, packed, u, None, commit) != refused

    def _release_dev(self, rng, shard):
        c, m, idx = self.release_rows(rng, self.next_target())
        packed, commit = self.packed_next("release_shard" if shard else "release_dev"), bool(rng.integers(0, 4))
        R, D = c.size, self.m.D
        cw, mm, ib = self.rows_dev(pack(c, m) if packed else None, c, m)
        ib[:R] = self.torch.from_numpy(idx.astype(np.int8 if packed else np.int32)).cuda()
        _, delta, tab = self.outs(0, D)
        self.sync()
        if shard:
            self.one_launch(lambda: self.a.release_shard_dev(cw.data_ptr(), 0 if packed else mm.data_ptr(), R, ib.data_ptr(),
                                                             delta.data_ptr(), tab.data_ptr(), step=self.step, commit=commit,
                                                             packed=packed, stream=self.ts.cuda_stream))
            self.step += 1
        else:
            self.one_launch(lambda: self.a.release_dev(cw.data_ptr(), 0 if packed else mm.data_ptr(), R, ib.data_ptr(),
                                                       delta.data_ptr(), tab.data_ptr(), commit=commit, packed=packed,
                                                       stream=self.stream(rng)))
        self.sync()
        got = ib.cpu().numpy()
        eq(got[:R], idx, "the index array (an input)")
        self._release_expect(c, m, idx, packed, delta.cpu().numpy(), tab.cpu().numpy(), commit)

    def op_release_dev(self, rng):
        self._release_dev(rng, False)

    def op_release_shard(self, rng):
        self._release_dev(rng, True)
        assert self.a.peer_last_timeout == 0

    # -- charge and release of stored records --
    def ids(self, n):
        self.next_id += 1
        return ["%d-%02d" % (self.next_id, j) for j in range(n)]

    def _records(self, entries):
        """[(ids, 0 core / 1 mem, gpus)] -> (the flat form's sets, hashes, resources, links), records, links"""
        from oracle import restore_py
        flat, records, links = ([], [], [], []), [], []
        for e, (ids, res, gpus) in enumerate(entries):
            h = restore_py.device_hash(ids)
            for lst, v in zip(flat, (ids, h, res, gpus)):
                lst.append(v)
            records.append(restore_py.marshal_record("ns", "pod%d" % e, {"c": (ids, restore_py.MEM if res else restore_py.CORE)}))
            links += [("elastic-gpu-%s-%d" % (h, i), "/dev/nvidia%d" % g) for i, g in enumerate(gpus)]
        return flat, records, links

    def _restore_call(self, entries, flat_form, cap_core, cap_mem, **flags):
        from elastic_gpu_agent_b200 import restore
        flat, records, links = self._records(entries)
        if flat_form:
            fc, fm, ov, _ = restore.restore_table_flat(self.a, *flat, cap_core, cap_mem, **flags)
        else:
            fc, fm, ov, _, _ = restore.restore_table(self.a, records, links, cap_core, cap_mem, **flags)
        return (fc, fm, ov), records, links

    def _charge(self, entries, flat_form):
        from oracle import restore_py
        D = self.m.D
        got, records, links = self._restore_call(entries, flat_form, [100] * D, [MEM_MAX] * D, charge=True)
        want, _, _ = restore_py.charge((self.m.fc.tolist(), self.m.fm.tolist(), self.m.ov.tolist()), records, links)
        for g, w, what in zip(got, want, ("free_core", "free_mem", "oversub")):
            eq(g, w, "charged " + what)
        self.m.set_table(*want)

    def op_restore_charge(self, rng):
        """partial and whole-card core entries and memory entries, charged to the live table; some oversubscribe"""
        D = self.m.D
        entries = []
        for _ in range(int(rng.integers(1, 5))):
            kind = int(rng.integers(0, 3))
            cards = int(rng.integers(1, min(2, D) + 1))
            n = int(rng.integers(1, 61)) if kind == 0 else 100 * cards + int(rng.integers(0, 30)) if kind == 1 else \
                int(rng.integers(1, 3000))
            gpus = [int(g) for g in rng.choice(D, cards if kind == 1 else 1, replace=False)]
            entries.append((self.ids(n), 1 if kind == 2 else 0, gpus))
        self._charge(entries, bool(rng.integers(0, 2)))

    def op_restore_release(self, rng):
        """release of stored records, aimed in turn at an accepted, an oversubscribed and an over-capacity outcome"""
        from elastic_gpu_agent_b200 import _lib as L
        from oracle import restore_py
        self.n_restore_release += 1
        target = ("accepted", "flagged", "exceeds")[(self.n_restore_release - 1) % 3]
        if target == "flagged":
            self._flag_a_device(rng)
        elif target == "exceeds":
            self._unflag_a_device()
        D = self.m.D
        fc, fm, ov = self.m.fc, self.m.fm, self.m.ov
        cap_core, cap_mem = [100] * D, [MEM_MAX] * D
        free = np.flatnonzero(ov == 0).tolist()
        entries = []
        for g in free[:3]:
            if fc[g] < 100:
                entries.append((self.ids(int(rng.integers(1, 100 - fc[g] + 1))), 0, [g]))
            elif fm[g] < MEM_MAX:
                entries.append((self.ids(int(rng.integers(1, min(MEM_MAX - fm[g], 2000) + 1))), 1, [g]))
        if target == "flagged":
            entries.append((self.ids(1), 0, [int(rng.choice(np.flatnonzero(ov)))]))
        elif target == "exceeds" and free:
            g = free[-1]
            cap_mem[g] = int(fm[g])  # the capacity the caller passes: three more MiB released than it allows
            entries.append((self.ids(3), 1, [g]))
        flat_form = bool(rng.integers(0, 2))
        _, records, links = self._records(entries)
        try:
            want, _, _ = restore_py.release((fc.tolist(), fm.tolist(), ov.tolist()), records, links, cap_core, cap_mem)
        except restore_py.Refused:
            want = None
        try:
            got = self._restore_call(entries, flat_form, cap_core, cap_mem, release=True)[0]
        except L.EgpuError as ex:
            assert ex.code == L.ERR_STATE and want is None, (ex, want)
            uc, um, _, _ = restore_py.usage(records, links, D)
            touched = [d for d in range(D) if uc[d] or um[d]]
            self.restore_outcomes.add("flagged" if any(ov[d] for d in touched) else "exceeds")
            return
        assert want is not None, "EGPU_RESTORE_RELEASE accepted what the release rule refuses"
        for g, w, what in zip(got, want, ("free_core", "free_mem", "oversub")):
            eq(g, w, "released " + what)
        self.m.set_table(*want)
        self.restore_outcomes.add("accepted")

    # -- place, then give the same rows back --
    def op_give_back(self, rng):
        """a committing placement released with its own index array, whole or in two shuffled chunks, in the format
        of give_back_spec, must leave exactly the table it started from"""
        how, packed_place, packed = give_back_spec(self.seed, self.n_give_back, self.replay_kernel)
        self.n_give_back += 1
        if self.m.ov.any():  # rows held on a flagged device are refused: start from an unflagged table
            fc, fm = self.m.table32()
            self.a.set_table(fc, fm)
            self.m.set_table(fc, fm)
        before = (self.m.fc.copy(), self.m.fm.copy(), self.m.ov.copy())
        if how == "prefix":
            c, m, idx = self.op_packed_prefix_dev(rng, packed=packed_place)
        elif how == "device_rounds":
            self.pick_variant(rng, grid_ok=False)
            c, m, idx = self._device_rounds_dev(rng, packed_place, self.ts.cuda_stream)
        else:
            c, m, idx = getattr(self, "op_" + how)(rng, packed=packed_place)
        perm = rng.permutation(c.size)
        cut = int(rng.integers(0, c.size + 1)) if rng.integers(0, 2) else c.size
        for part in (perm[:cut], perm[cut:]) if cut < c.size else (perm,):
            pc, pm, pi = c[part], m[part], idx[part]
            R, D = pc.size, self.m.D
            cw, mm, ib = self.rows_dev(pack(pc, pm) if packed else None, pc, pm)
            if R:
                ib[:R] = self.torch.from_numpy(pi.astype(np.int8 if packed else np.int32)).cuda()
            _, delta, tab = self.outs(0, D)
            self.sync()
            self.a.release_dev(cw.data_ptr(), 0 if packed else mm.data_ptr(), R, ib.data_ptr(), delta.data_ptr(),
                               tab.data_ptr(), commit=True, packed=packed, stream=self.ts.cuda_stream)
            self.sync()
            assert self._release_expect(pc, pm, pi, packed, delta.cpu().numpy(), tab.cpu().numpy(), True), \
                f"the release of the rows placed by {how} was refused"
        fc, fm, ov = self.a.table()
        eq(fc, before[0], f"free_core after {how} and its release")
        eq(fm, before[1], f"free_mem after {how} and its release")
        eq(ov, before[2], f"oversub after {how} and its release")

    # -- CUDA graphs: one launch captured on the harness's stream, replayed later between eager calls --
    def op_graph_capture(self, rng):
        spec = graph_spec(self.seed, self.n_graph, self.replay_kernel)
        self.n_graph += 1
        self.graph = GraphOp(self, rng, *spec)

    def op_graph_replay(self, rng):
        assert self.graph is not None, "graph blocks keep D"
        self.graph.replay(rng)
        self.replays += 1

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


class GraphOp:
    """One launch of `kind` (GRAPH_KINDS: what the headers say replays from a CUDA graph), committing, captured on the
    harness's torch stream with its rows and outputs in fixed device buffers.
    Capture: a warm-up that holds nothing (every row infeasible, or holding nothing), egpu_table_set of a new table
    of the same D (the lookup tables are then stale), and the capture, which must change nothing the readers see.
    Replay: new rows written into the buffers, the graph replayed on the same stream, its outputs checked against
    the oracles applied to the model at replay time, and the model advanced."""

    def __init__(self, run, rng, kind, packed):
        self.run, self.kind, self.D = run, kind, run.m.D
        self.release = kind in ("release_dev", "release_shard")
        self.packed = packed
        run.set_variant(int(rng.choice([LUT, SORTED] if kind == "commit_dev" else [AUTO, SORTED, LUT])))
        if kind == "multi_rounds":
            self.sizes = [int(rng.choice([5, 513, 4099])), 0, int(rng.choice([1, 511]))]
        elif kind == "shard_prefix_multi":
            self.sizes = [int(rng.choice([5, 513])), int(rng.choice([1, 4099]))]
        else:
            self.sizes = [5100 if self.release else int(rng.choice([5, 513, 4099]))]
        self.step = run.step
        run.step += 2 * len(self.sizes)
        self.bufs, self.tup = [], []
        for R in self.sizes:
            z = np.zeros(R, np.int32)
            b = run.rows_dev(z.view(np.uint32) if self.packed else None, z, z) + run.outs(0, self.D)[1:]
            self.bufs.append(b)
            ptrs = (b[2].data_ptr(), b[3].data_ptr(), b[4].data_ptr())
            self.tup.append((b[0].data_ptr(), R) + ptrs if self.packed else (b[0].data_ptr(), b[1].data_ptr(), R) + ptrs)
        # warm-up: occupancy queries, scratch and barrier words outside the capture; the table stays as it was
        for k, R in enumerate(self.sizes):
            none = np.full(R, -1, np.int32)
            self.write(k, none, none, none if self.release else None)
        run.sync()
        self.launch()
        run.sync()
        run.op_set_table_same(rng)
        self.g = run.torch.cuda.CUDAGraph()
        with run.torch.cuda.graph(self.g, stream=run.ts):
            self.launch()
        run.sync()

    def write(self, k, c, m, idx=None, words=None):
        t = self.run.torch
        cw, mm, ib, delta, tab = self.bufs[k]
        R = c.size
        if R:
            if self.packed:
                cw[:R] = t.from_numpy((pack(c, m) if words is None else words).view(np.int32)).cuda()
            else:
                cw[:R] = t.from_numpy(c).cuda()
                mm[:R] = t.from_numpy(m).cuda()
        ib.fill_(-9)
        if idx is not None and R:
            ib[:R] = t.from_numpy(idx.astype(np.int8 if self.packed else np.int32)).cuda()
        delta.fill_(-1)
        tab.fill_(-7)

    def launch(self):
        a, s, k, packed = self.run.a, self.run.ts.cuda_stream, self.kind, self.packed
        if k == "multi_rounds":
            return a.bestfit_batches_rounds_device_dev(self.tup, packed=packed, stream=s)
        if k == "shard_prefix_multi":
            return a.bestfit_batches_shard_prefix_dev(self.tup, self.step, commit=True, packed=packed, stream=s)
        cw, mm, ib, delta, tab = (x.data_ptr() if x is not None else 0 for x in self.bufs[0])
        R = self.sizes[0]
        if k == "commit_dev":
            a.bestfit_dev(cw, mm, R, ib, delta, tab, True, s)
        elif k == "prefix_dev" and packed:
            a.bestfit_packed_prefix_dev(cw, R, ib, delta, tab, commit=True, stream=s)
        elif k == "prefix_dev":
            a.bestfit_dev(cw, mm, R, ib, delta, tab, True, s, prefix_commit=True)
        elif k == "device_rounds_dev" and packed:
            a.bestfit_packed_rounds_device_dev(cw, R, ib, delta, tab, s)
        elif k == "device_rounds_dev":
            a.bestfit_rounds_device_dev(cw, mm, R, ib, delta, tab, s)
        elif k == "release_dev":
            a.release_dev(cw, mm, R, ib, delta, tab, commit=True, packed=packed, stream=s)
        elif k == "release_shard":
            a.release_shard_dev(cw, mm, R, ib, delta, tab, step=self.step, commit=True, packed=packed, stream=s)
        elif k == "shard_rounds":
            a.bestfit_shard_rounds_dev(cw, mm, R, ib, delta, tab, self.step, packed=packed, stream=s)
        else:
            raise AssertionError(k)

    def replay(self, rng):
        run = self.run
        assert run.m.D == self.D
        rows = []
        if self.release:
            c, m, idx = run.release_rows(rng, run.next_target())
            pad = self.sizes[0] - c.size
            c, m = np.concatenate([c, np.zeros(pad, np.int32)]), np.concatenate([m, np.zeros(pad, np.int32)])
            idx = np.concatenate([idx, np.full(pad, -1, np.int32)])
            self.write(0, c, m, idx)
        else:
            for k, R in enumerate(self.sizes):
                words, c, m = run.placement_rows(rng, self.packed, R)
                self.write(k, c, m, words=words)
                rows.append((words, c, m))
        run.sync()
        self.g.replay()
        run.sync()
        b = self.bufs[0]
        D = self.D
        if self.release:
            eq(run.idx_back(b[2], c.size), idx, "the index array (an input)")
            run._release_expect(c, m, idx, self.packed, b[3].cpu().numpy(), b[4].cpu().numpy(), True)
        elif self.kind == "shard_prefix_multi":
            run._shard_prefix_multi_expect(rows, self.bufs, True)
        elif self.kind == "multi_rounds":
            for k, ((_, c, m), bk) in enumerate(zip(rows, self.bufs)):
                try:
                    run._rounds_install(c, m, run.idx_back(bk[2], c.size), bk[3].cpu().numpy(), bk[4].cpu().numpy())
                except AssertionError as ex:
                    raise AssertionError(f"batch {k} (R = {c.size}): {ex}") from ex
        else:
            _, c, m = rows[0]
            idx, delta, tab = run.idx_back(b[2], c.size), b[3].cpu().numpy(), b[4].cpu().numpy()
            if self.kind == "commit_dev":
                run._commit_expect(c, m, idx, delta[:D], delta[D:], tab)
            elif self.kind == "prefix_dev":
                run._prefix_expect(c, m, idx, delta, tab)
            else:
                run._rounds_install(c, m, idx, delta, tab)
        assert run.a.peer_last_timeout == 0


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
        run = Run(alloc, egpu, oracle_c, torch, seed, replay_kernel)
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
            if name.startswith("graph_") and "pipelined" not in readers:
                readers += ("pipelined",)  # an eager pipelined chain on the stream the graph runs on
            for reader in ("table()",) + readers:
                try:
                    run.check_table() if reader == "table()" else run.read(reader)
                except AssertionError as ex:
                    raise AssertionError(f"{where}, reader {reader}: {ex}") from ex
        alloc.peer_detach()
        return run
    finally:
        alloc.close()


class HostArray:
    """a host array standing in for a device buffer the composition helpers of Run read back"""

    def __init__(self, a):
        self.a = np.asarray(a)

    def cpu(self):
        return self

    def numpy(self):
        return self.a


class HostRun(Run):
    """the row and record builders and the composition rules of Run, on the CPU: no context, charges by the
    restatement"""

    def __init__(self, oracle_c=None):
        self.m = Model()
        self.oc = oracle_c
        self.a = type("NoContext", (), {"set_table": staticmethod(lambda fc, fm: None)})()
        self.next_id = 0
        self.outcomes = set()
        self.refusals = 0

    def _charge(self, entries, flat_form):
        from oracle import restore_py
        _, records, links = self._records(entries)
        want, _, _ = restore_py.charge((self.m.fc.tolist(), self.m.fm.tolist(), self.m.ov.tolist()), records, links)
        self.m.set_table(*want)


# ---- tests that need no GPU ----------------------------------------------------------------------------
def test_model_matches_the_oracles_on_short_chains(oracle_c):
    """commit chains (clamping, sticky flags, set_table clearing them), prefix-commit, rounds and replay,
    composed by the model, against the oracles applied call after call; then the rules of K-batch rounds, the K-batch
    sharded prefix-commit, release and charge (check_new_composition_rules)"""
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
        check_new_composition_rules(oracle_c, rng, m)
        m.set_table(fc, fm)
        assert not m.ov.any()


def check_new_composition_rules(oracle_c, rng, m):
    """the rules of the operations added with the release and the one-launch rounds, through Run's own helpers, on a
    model whose flags are set: each must keep or OR them as DESIGN.md says"""
    from oracle import bestfit_np, restore_py
    D = m.D
    h = HostRun(oracle_c)
    h.m = m
    flags = m.ov.copy()
    assert flags.any()
    # K-batch rounds: batch k against the table batches 0..k-1 left (numpy oracle), flags kept
    cur_c, cur_m = m.table32()
    for k, R in enumerate((700, 0, 300)):
        rc, rm = requests_for(rng, cur_c, cur_m, R)
        o = bestfit_np.rounds(cur_c, cur_m, rc, rm, 1 << 30)
        assert o[6] == 0
        h._rounds_install(rc, rm, o[0], np.concatenate([o[1], o[2]]), np.concatenate([o[3], o[4], np.zeros(D)]))
        cur_c, cur_m = np.asarray(o[3], np.int32), np.asarray(o[4], np.int32)
        assert np.array_equal(m.fc, cur_c) and np.array_equal(m.fm, cur_m) and np.array_equal(m.ov, flags), k
    # K-batch sharded prefix-commit: with COMMIT each batch sees the table the one before installed; without it
    # every batch sees the current table and nothing is installed
    for commit in (False, True):
        start = m.table32()
        cur_c, cur_m = start
        rows, bufs = [], []
        for R in (400, 0, 900):
            rc, rm = requests_for(rng, cur_c, cur_m, R)
            o = bestfit_np.prefix_commit(cur_c, cur_m, rc, rm)
            rows.append((None, rc, rm))
            bufs.append((None, None, HostArray(np.concatenate([o[0], [-9] * 4])), HostArray(np.concatenate([o[1], o[2]])),
                         HostArray(o[3])))
            if commit:
                cur_c, cur_m = np.asarray(o[3][:D], np.int32), np.asarray(o[3][D:2 * D], np.int32)
        h._shard_prefix_multi_expect(rows, bufs, commit)
        assert np.array_equal(m.fc, cur_c if commit else start[0]) and np.array_equal(m.fm, cur_m if commit else start[1])
        assert np.array_equal(m.ov, flags)
    # release: accepted installs free + U with the flags kept; refused changes nothing and counts; dry-run installs
    # nothing
    for target, commit in (("accepted", True), ("accepted", False), ("flagged", True), ("exceeds", True)):
        c, mm, idx = h.release_rows(rng, target)
        flags = m.ov.copy()  # "flagged" may have charged a device first
        before = (m.fc.copy(), m.fm.copy(), flags, h.refusals)
        held = (idx >= 0) & (idx < D) & (c >= 0) & (c <= 100) & (mm >= 0) & (mm <= MEM_MAX)
        uc = np.bincount(idx[held], c[held].astype(np.int64), D).astype(np.int64)
        um = np.bincount(idx[held], mm[held].astype(np.int64), D).astype(np.int64)
        accepted = h._release_expect(c, mm, idx, False, None, None, commit)
        assert accepted == (target == "accepted"), target
        if accepted and commit:
            assert np.array_equal(m.fc, before[0] + uc) and np.array_equal(m.fm, before[1] + um)
        else:
            assert np.array_equal(m.fc, before[0]) and np.array_equal(m.fm, before[1])
        assert np.array_equal(m.ov, flags) and h.refusals == before[3] + (not accepted)
    # charge: max(free - U, 0) installed and the flags ORed with free - U < 0
    g = int(rng.integers(0, D))
    entries = [(h.ids(int(m.fc[g]) + 1 if m.fc[g] < 100 else 30), 0, [g]), (h.ids(2000), 1, [int(rng.integers(0, D))])]
    _, records, links = h._records(entries)
    uc, um, _, _ = restore_py.usage(records, links, D)
    c0, m0, ov0 = m.fc.copy(), m.fm.copy(), m.ov.copy()
    h._charge(entries, True)
    left_c, left_m = c0 - np.asarray(uc), m0 - np.asarray(um)
    assert np.array_equal(m.fc, np.maximum(left_c, 0)) and np.array_equal(m.fm, np.maximum(left_m, 0))
    assert np.array_equal(m.ov, ov0 | (left_c < 0) | (left_m < 0))
    assert m.ov[g] or m.fc[g] == c0[g] - uc[g]


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
        assert names[0] == "set_table" and 60 <= len(names) <= 110
        assert set(names) >= set(ALL_OPS) - {"multi_big"}
        assert names.count("multi") >= 5
        # every sequence can see each release outcome: the targets cycle over accepted, flagged, exceeds
        assert sum(names.count(n) for n in RELEASES) >= 3 and names.count("restore_release") >= 3
        # graph blocks: every capture is replayed twice, after an egpu_table_set of the same D and before any
        # egpu_table_set that changes D
        caps = [i for i, n in enumerate(names) if n == "graph_capture"]
        assert len(caps) == 2 and names.count("graph_replay") == 4 and names.count("give_back") == 2
        for i in caps:
            block = names[i:i + 6]
            assert block[2] == "set_table_same" and block[3] == block[5] == "graph_replay", block
            assert "set_table" not in block and len({d_at(seed, j) for j in range(i, i + 7)}) == 1
    assert {graph_spec(s, n, k) for s in SEEDS for n in range(2) for k in REPLAY_KERNELS} == set(GRAPH_SPECS)
    assert {give_back_spec(s, n, k) for s in SEEDS for n in range(2) for k in REPLAY_KERNELS} == \
        {g + (p,) for g in GIVE_BACK_SPECS for p in (False, True)}
    for seed in SEEDS:
        names = plan(seed)
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
    vocabulary = {e for _, calls in OPS.values() for e, _ in calls}
    assert not vocabulary & set(NO_TABLE_CHANGE)
    assert declared == vocabulary | set(NO_TABLE_CHANGE), (declared ^ (vocabulary | set(NO_TABLE_CHANGE)))
    assert all(NO_TABLE_CHANGE.values())


def flag_set(s):
    return frozenset(s.split("|")) - {""}


def test_every_entry_point_and_flag_set_has_a_decision():
    """every EGPU_F_* and EGPU_RESTORE_* flag of include/*.h is passed by an operation of the sequences or listed
    as never changing the table, with its reason; and every flag set an entry point documents as changing the
    table (COMMITTING) is some operation's: a new flag, or a new committing flag set on an existing entry point,
    needs a decision here"""
    macros = set()
    for f in sorted(os.listdir(os.path.join(ROOT, "include"))):
        if f.endswith(".h"):
            text = open(os.path.join(ROOT, "include", f)).read()
            macros |= set(re.findall(r"^#define\s+(EGPU_F_\w+|EGPU_RESTORE_\w+)\s+\d+\b", text, re.M))
    assert {"EGPU_F_COMMIT", "EGPU_F_RELEASE", "EGPU_F_DEVICE_ROUNDS", "EGPU_RESTORE_CHARGE", "EGPU_RESTORE_RELEASE"} <= macros
    passed = {(e, flag_set(f)) for _, calls in OPS.values() for e, f in calls}
    used = set().union(*(fs for _, fs in passed))
    assert used - {"commit=1"} <= macros, used - macros
    assert not used & set(NO_TABLE_CHANGE_FLAGS) and all(NO_TABLE_CHANGE_FLAGS.values())
    assert macros == (used - {"commit=1"}) | set(NO_TABLE_CHANGE_FLAGS), macros ^ ((used - {"commit=1"}) | set(NO_TABLE_CHANGE_FLAGS))
    # the committing flag sets are covered by dedicated operations: the composite ones only reuse their calls
    committing = {(e, flag_set(f)) for e, f in COMMITTING}
    dedicated = {n: calls for n, (_, calls) in OPS.items() if n not in COMPOSITE}
    covered = {(e, flag_set(f)) for calls in dedicated.values() for e, f in calls}
    missing = committing - covered
    assert not missing, sorted((e, "|".join(sorted(fs))) for e, fs in missing)
    # every dedicated operation that changes the table passes a committing flag set
    for name, calls in dedicated.items():
        if OPS[name][0]:
            assert {(e, flag_set(f)) for e, f in calls} & committing, name
    # ... and the composite ones pass nothing the dedicated ones do not
    composite = {(e, flag_set(f)) for n in COMPOSITE for e, f in OPS[n][1]}
    assert composite <= covered, composite - covered
    # an entry point with a committing flag set is never listed as leaving the table alone
    assert not {e for e, _ in COMMITTING} & set(NO_TABLE_CHANGE)


def test_composite_operations_declare_what_they_pass():
    """graph_capture and give_back declare exactly the calls their specs make over SEEDS x REPLAY_KERNELS (two of
    each per sequence), and the dedicated operations that alternate formats pass both formats over the kernels"""
    specs = [(s, n, k) for s in SEEDS for n in range(2) for k in REPLAY_KERNELS]
    captured = {("egpu_table_set", "")} | {GRAPH_CALLS[graph_spec(*x)] for x in specs}
    assert {(e, flag_set(f)) for e, f in OPS["graph_capture"][1]} == {(e, flag_set(f)) for e, f in captured}
    given = set()
    for x in specs:
        how, packed_place, packed = give_back_spec(*x)
        given |= {GIVE_BACK_CALLS[(how, packed_place)], ("egpu_bestfit_batch_dev", PRELC if packed else RELC)}
    assert {(e, flag_set(f)) for e, f in OPS["give_back"][1]} == {(e, flag_set(f)) for e, f in given}
    assert {alternate(s, k, 0) for s in SEEDS for k in REPLAY_KERNELS} == {False, True}
    assert all({alternate(s, k, 0) for k in REPLAY_KERNELS} == {False, True} for s in SEEDS)


def test_release_and_restore_outcomes_are_reachable_on_the_model(oracle_c):
    """the release rows of every target give that outcome under release_np, in both formats, and the charge /
    release restatements compose: charge then release of the same records is the identity when accepted"""
    from oracle import restore_py

    rng = np.random.default_rng(12)
    h = HostRun()
    for D in (1, 5, 9, 33, 64):
        for target in ("accepted", "flagged", "exceeds") * 4:
            h.m.set_table(*random_table(rng, D), ov=rng.integers(0, 2, D) if rng.integers(0, 2) else None)
            c, m, idx = h.release_rows(rng, target)
            for packed in (False, True):
                cc, mm = release_np.unpack(pack(c, m)) if packed else (c, m)
                _, tab, ok = release_np.release(h.m.fc, h.m.fm, h.m.ov, cc, mm, idx)
                reasons = set(tab[2 * D:].tolist())
                want = {"accepted": set(), "flagged": {release_np.REL_FLAGGED}}.get(target, {release_np.REL_EXCEEDS})
                assert (ok == (target == "accepted")) and want <= reasons, (D, target, packed, reasons)
        # charge then release of the same records on an unflagged table gives the table back
        h.m.set_table(*random_table(rng, D))
        fc0, fm0 = h.m.fc.copy(), h.m.fm.copy()
        entries = [(h.ids(int(rng.integers(1, 40))), 0, [int(rng.integers(0, D))]) for _ in range(3)]
        _, records, links = h._records(entries)
        t, _, _ = restore_py.charge((fc0.tolist(), fm0.tolist(), [0] * D), records, links)
        try:
            back, _, _ = restore_py.release(t, records, links, [100] * D, [MEM_MAX] * D)
            assert back == (fc0.tolist(), fm0.tolist(), [0] * D)
        except restore_py.Refused:
            assert any(t[2])


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
    # every release outcome, on the device and from stored records; both captures replayed twice
    assert run.outcomes == {"accepted", "flagged", "exceeds"}, run.outcomes
    assert run.restore_outcomes == {"accepted", "flagged", "exceeds"}, run.restore_outcomes
    assert run.n_graph == 2 and run.replays == 4


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


def _ctx(egpu, D, variant, seed):
    alloc = egpu.BestFitAllocator(0)
    fc, fm = random_table(np.random.default_rng(seed), D)
    alloc.set_table(fc, fm)
    alloc.set_variant(variant)
    return alloc


def _probe_scan(alloc, torch, stream, fc, fm, ready=True):
    """one non-committing scan of the probe rows of (fc, fm) on `stream`; returns (rows, buffers)"""
    pc, pm = probe_rows(fc, fm)
    R, D = pc.size, fc.size
    b = (torch.from_numpy(pc).cuda(), torch.from_numpy(pm).cuda(), torch.full((R + 4,), -9, dtype=torch.int32, device="cuda"),
         torch.full((2 * D,), -1, dtype=torch.int64, device="cuda"), torch.full((3 * D,), -7, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    return (pc, pm), b


def _issue(alloc, b, R, stream, ready=True, commit=False):
    alloc.bestfit_dev(b[0].data_ptr(), b[1].data_ptr(), R, b[2].data_ptr(), b[3].data_ptr(), b[4].data_ptr(), commit, stream,
                      inputs_ready=ready)


def _check_probe(rows, b, fc, fm, what):
    o_idx, o_dc, o_dm, o_tab = snapshot_np(fc, fm, *rows)
    got = b[2].cpu().numpy()
    eq(got[:rows[0].size], o_idx, what + ": idx")
    eq(got[rows[0].size:], -9, what + ": guard words")
    eq(b[3].cpu().numpy(), np.concatenate([o_dc, o_dm]), what + ": delta")
    eq(b[4].cpu().numpy(), o_tab, what + ": table'")


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [SORTED, LUT], ids=["sorted", "lut"])
def test_eager_scan_after_a_capture_waits_for_the_commit_before_it(egpu, variant):
    """A large committing scan C with EGPU_F_INPUTS_READY on a stream, then, with C still running, a capture on the
    same stream of a non-committing scan S (driver API: nothing synchronises), then an eager EGPU_F_INPUTS_READY scan
    E of probe rows.  S never runs at capture, so E's predecessor on the stream is C, which rewrites the table: E
    must be fully ordered behind it and answer from the table C installed.  Then the graph is replayed and another
    eager EGPU_F_INPUTS_READY scan follows the replay without a synchronisation.  Under the lookup scan, C leaves the
    lookup tables stale and the capture of S rebuilds them only inside the graph: E must still rebuild them eagerly."""
    import ctypes as C_
    import torch
    cu = C_.CDLL("libcuda.so.1")
    D = 8 if variant == SORTED else 33
    alloc = _ctx(egpu, D, variant, 3)
    try:
        fc0, fm0, _ = alloc.table()
        ts = torch.cuda.Stream()
        s = ts.cuda_stream
        R = 32 << 20  # ~0.1 ms of scan: E is issued long before C's epilogue installs its table
        big_c = torch.full((R,), 1, dtype=torch.int32, device="cuda")
        big_m = torch.full((R,), 1, dtype=torch.int32, device="cuda")
        big_i = torch.empty(R + 4, dtype=torch.int32, device="cuda")
        rows_s, bs = _probe_scan(alloc, torch, s, fc0, fm0)
        _issue(alloc, bs, rows_s[0].size, s)  # warm-up of S outside the capture
        torch.cuda.synchronize()
        # the committed table: every row (1, 1) on the best fit of the first one
        o_tab = snapshot_np(fc0, fm0, np.ones(1, np.int32), np.ones(1, np.int32))[0]
        d = int(o_tab[0])
        fc1, fm1 = fc0.astype(np.int64).copy(), fm0.astype(np.int64).copy()
        fc1[d], fm1[d] = max(fc1[d] - R, 0), max(fm1[d] - R, 0)
        rows_e, be = _probe_scan(alloc, torch, s, fc1.astype(np.int32), fm1.astype(np.int32))
        graph, exe = C_.c_void_p(), C_.c_void_p()
        alloc.bestfit_dev(big_c.data_ptr(), big_m.data_ptr(), R, big_i.data_ptr(), 0, 0, True, s, inputs_ready=True)
        assert cu.cuStreamBeginCapture_v2(C_.c_void_p(s), 1) == 0  # thread-local capture mode
        _issue(alloc, bs, rows_s[0].size, s)
        assert cu.cuStreamEndCapture(C_.c_void_p(s), C_.byref(graph)) == 0
        _issue(alloc, be, rows_e[0].size, s)
        torch.cuda.synchronize()
        got_fc, got_fm, got_ov = alloc.table()
        eq(got_fc, fc1, "table() free_core after C")
        eq(got_fm, fm1, "table() free_mem after C")
        _check_probe(rows_e, be, fc1, fm1, "eager scan after the capture")
        # replay S, then an eager pipelined scan right behind it
        assert cu.cuGraphInstantiateWithFlags(C_.byref(exe), graph, C_.c_ulonglong(0)) == 0
        for b in (bs, be):
            b[2].fill_(-9)
            b[3].fill_(-1)
            b[4].fill_(-7)
        torch.cuda.synchronize()
        assert cu.cuGraphLaunch(exe, C_.c_void_p(s)) == 0
        _issue(alloc, be, rows_e[0].size, s)
        torch.cuda.synchronize()
        _check_probe(rows_s, bs, fc1, fm1, "replayed S")
        _check_probe(rows_e, be, fc1, fm1, "eager scan after the replay")
        assert cu.cuGraphExecDestroy(exe) == 0 and cu.cuGraphDestroy(graph) == 0
    finally:
        alloc.close()


@pytest.mark.gpu
def test_graph_of_lookup_scans_after_a_table_change_outside_it(egpu):
    """A graph of lookup scans captured while the lookup tables were current holds no rebuild.  After egpu_table_set
    of another table of the same D, the documented remedy - one eager lookup scan before the replay - makes the replay
    answer from the new table; a second table change followed by an eager committing scan, then the remedy, too."""
    import torch
    D = 33
    alloc = _ctx(egpu, D, LUT, 5)
    try:
        rng = np.random.default_rng(6)
        fc0, fm0, _ = alloc.table()
        ts = torch.cuda.Stream()
        s = ts.cuda_stream
        rows = requests_for(rng, fc0, fm0, 4099)
        b = (torch.from_numpy(rows[0]).cuda(), torch.from_numpy(rows[1]).cuda(),
             torch.full((rows[0].size + 4,), -9, dtype=torch.int32, device="cuda"),
             torch.full((2 * D,), -1, dtype=torch.int64, device="cuda"), torch.full((3 * D,), -7, dtype=torch.int32, device="cuda"))
        torch.cuda.synchronize()
        _issue(alloc, b, rows[0].size, s)  # warm-up: the lookup tables are current from here on
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=ts):
            _issue(alloc, b, rows[0].size, s)
        for step in range(2):
            fc, fm = random_table(rng, D)
            alloc.set_table(fc, fm)
            if step == 1:  # an eager commit on top of it
                rc, rm = requests_for(rng, fc, fm, 513)
                alloc.bestfit(rc, rm, commit=True)
                fc, fm, _ = alloc.table()
            pc, pm = probe_rows(fc, fm)
            alloc.bestfit(pc, pm)  # the remedy: one eager lookup scan
            for x in b[2:]:
                x.fill_(-5)
            torch.cuda.synchronize()
            g.replay()
            torch.cuda.synchronize()
            got = b[2].cpu().numpy()
            eq(got[:rows[0].size], snapshot_np(fc, fm, *rows)[0], f"replay {step} idx")
    finally:
        alloc.close()
