"""egpu::place_pods, egpu::place_gangs and egpu::place_tables at scale, without a GPU: the generators of the cases in
tests/test_gpu_pods_scale.py, preconditions that read the restatements' round traces and show that each case crosses
the kernel threshold it is named for, and the known answers of the pod choice word checked against the restatement.

The thresholds of the shared pod phases (DESIGN.md §4.6-§4.8):
  - a round's pending set is compacted in tiles of 256 positions: the commit adds each tile's deferred pods to a
    count, deferred_prefix sums the counts, append_deferred writes each tile's deferred pods in order;
  - the commit phase stages 2 048 pending positions at a time and stages the next 2 048 when a tile's walk passes
    them (`i0 != staged`), so past 2 048 positions every commit CTA re-stages within the round;
  - the grid is min(2 x SMs, ceil(N / 8) x ceil(G / 256)) CTAs, and the commit walks table tiles b, b + grid, ...:
    at N_wave each commit CTA walks 2 or 3 table tiles; N <= 8 is one table tile, committed by CTA 0 alone;
  - place_gangs indexes the deferred counts by the launch's round over all gangs, and a round zeroes the next
    round's counts over ceil(G / 256) tiles: the next round may be the next gang's first, over more positions than
    this one, and must not read counts left from two rounds before;
  - a gang given back returns its pods' demand with give_back_pods, grid-stride over the gang's range.

The cases are cheap for the restatement by construction, whatever their size: every pod has an exact fit of its own.
A unit is one to three pods of the same k containers, container j asking for (c_j, base + 8 j), and one to three groups
of k devices: A holds exactly that demand, B 3 more memory per device and C 6 more.  Each unit has its own base, 64
apart, so a pod's best node is its unit's first free group, and nothing else comes close.  In round 1 every pod of a
unit chooses A; the first in pod order commits, and the others are deferred.  In round 2 they choose B: one commits,
one is deferred.  In round 3 the last one commits on C.  So a call runs 3 rounds, and the deferred pods of each round
sit wherever the shuffled pod order puts them.  A `whole` unit asks for whole cards (100 core per container) and has
no C: its third pod fits nowhere in round 3, and no other pod can use its devices.

Each case's reference is computed once per process (`reference`), and the GPU file reuses it.
"""
import functools
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import place_gangs_np  # noqa: E402
import place_pods_np  # noqa: E402
import test_gpu_place_gangs as gpu_gangs  # noqa: E402  (its invariants hold for the restatement too)
import test_gpu_place_pods as gpu_pods  # noqa: E402
from test_preempt_scale_cpu import SMS, n_wave  # noqa: E402

CORE_MAX, MEM_MAX = 100, (1 << 18) - 1
BLOCK = 256   # positions per compaction tile (kPodBlock, kPlaceBlock)
STAGE = 2048  # positions the commit phase stages at once (kPodStage, kPlaceStage)
SPAN = 64     # memory between two units' bases: a unit's devices hold base + 8 j + {0, 3, 6}, j < 8
GROUPS = {"single": 1, "twin": 2, "triple": 3, "whole": 2}  # device groups (A, B, C) per unit kind


# ---- generators --------------------------------------------------------------------------------------------------
class Cluster:
    """N tables of D devices that the units' device groups are put on, each group on a random table with room, so
    every table holds groups of many units and many gangs.  Devices no group takes are empty (0, 0), and past d_valid
    the tables hold out-of-domain values that must not be read as devices."""

    def __init__(self, g, N, D):
        self.g, self.N, self.D = g, N, D
        self.fc = np.zeros((N, D), np.int32)
        self.fm = np.zeros((N, D), np.int32)
        self.used = np.zeros(N, np.int64)
        self.base = SPAN

    def put(self, cores, mems):
        k = len(cores)
        for _ in range(64):
            n = int(self.g.integers(self.N))
            if self.used[n] + k <= self.D:
                break
        else:
            n = int(self.g.choice(np.flatnonzero(self.used + k <= self.D)))
        d = int(self.used[n])
        self.fc[n, d:d + k] = cores
        self.fm[n, d:d + k] = mems
        self.used[n] += k

    def unit(self, kind, k_hi):
        """The pods of one unit (a list of pods, each a list of (core, memory) containers), its groups put."""
        k = int(self.g.integers(1, k_hi + 1))
        cores = np.full(k, CORE_MAX) if kind == "whole" else self.g.integers(1, CORE_MAX, k)
        mems = self.base + 8 * np.arange(k)
        self.base += SPAN
        assert self.base < MEM_MAX - SPAN
        for extra in (0, 3, 6)[:GROUPS[kind]]:
            self.put(cores, mems + extra)
        pod = list(zip(cores.tolist(), mems.tolist()))
        return [pod] * (3 if kind == "whole" else GROUPS[kind])

    def units(self, kind, count, k_hi):
        return [self.unit(kind, k_hi) for _ in range(count)]

    def odd_pod(self, k_hi, unfit):
        """A pod of small containers but one: in the domain and fitting nowhere (unfit), or outside the domain."""
        k = int(self.g.integers(1, k_hi + 1))
        pod = [(int(self.g.integers(0, 4)), int(self.g.integers(0, SPAN))) for _ in range(k)]
        bad = (CORE_MAX, MEM_MAX) if unfit else [(-1, 0), (CORE_MAX + 1, 0), (0, MEM_MAX + 1), (1 << 30, 5)][
            int(self.g.integers(4))]
        pod[int(self.g.integers(k))] = bad
        return pod

    def args(self, pods):
        """(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets) of the tables and the pods in order."""
        fc, fm = self.fc.copy(), self.fm.copy()
        dv = np.maximum(self.used, self.g.integers(1, self.D + 1, self.N) * (self.used == 0)).astype(np.int32)
        past = np.arange(self.D)[None, :] >= dv[:, None]
        fc[past] = self.g.choice([-7, 101, 1000], int(past.sum()))
        fm[past] = self.g.choice([-1, MEM_MAX + 1, 1 << 30], int(past.sum()))
        rc = np.array([c for pod in pods for c, _ in pod], np.int32)
        rm = np.array([m for pod in pods for _, m in pod], np.int32)
        off = np.concatenate([[0], np.cumsum([len(pod) for pod in pods])]).astype(np.int32)
        return [fc, fm, dv, rc, rm, off]


def shuffled(g, unit_pods):
    """The pods of a list of units (and odd pods, each a list of one pod) in random order."""
    pods = [pod for u in unit_pods for pod in u]
    return [pods[i] for i in g.permutation(len(pods))]


def pods_case(seed, N, D, k_hi, triples, twins, singles=0, unfit=0, bad=0):
    """place_pods' arguments: units and odd pods in one shuffled pod order."""
    g = np.random.default_rng(seed)
    c = Cluster(g, N, D)
    u = c.units("triple", triples, k_hi) + c.units("twin", twins, k_hi) + c.units("single", singles, k_hi)
    u += [[c.odd_pod(k_hi, True)] for _ in range(unfit)] + [[c.odd_pod(k_hi, False)] for _ in range(bad)]
    return c.args(shuffled(g, u))


def gangs_args(c, gangs, gmin):
    """place_gangs' arguments of gangs given as pod lists, in order."""
    a = c.args([pod for gang in gangs for pod in gang])
    goff = np.concatenate([[0], np.cumsum([len(gang) for gang in gangs])]).astype(np.int32)
    return a + [goff, np.array(gmin, np.int32)]


def mixed_units(g, c, k_hi, triples, twins, singles, odd):
    u = c.units("triple", triples, k_hi) + c.units("twin", twins, k_hi) + c.units("single", singles, k_hi)
    u += [[c.odd_pod(k_hi, bool(i % 2))] for i in range(odd)]
    return [u[i] for i in g.permutation(len(u))]


def gang_sequence(seed=5, N=1031, D=8):
    """place_gangs' arguments at N = 1031 x 8, the gangs in this order:
      0 `lead`  103 pods, so the next gang's first pod is not a multiple of 256;
      1 `big`   2 100 pods of units and 45 odd pods (gang_min 2 000): round 2 defers in many tiles;
      2 `stale` 530 single pods, then 15 twins: round 1 defers only positions 530 and up (tile 2), round 2 has 15
                positions (one tile) and ends the gang;
      3 `back`  200 whole units (600 pods, gang_min 600): rounds 1 and 2 commit two pods of each unit, round 3 finds
                no node for the third, and the gang is given back.  Its round 1, the round after `stale`'s last, has
                600 positions and reads tile 2 of the counts `stale`'s round 1 wrote;
      4 `reuse` two pods of each of back's units, which fit only the whole cards back gave back (gang_min 400);
      5...      mixed small gangs, gang_min mixed."""
    g = np.random.default_rng(seed)
    c = Cluster(g, N, D)
    lead = shuffled(g, c.units("triple", 20, 3) + c.units("twin", 15, 3) + c.units("single", 13, 3))
    big = shuffled(g, c.units("triple", 500, 3) + c.units("twin", 300, 3) +
                   [[c.odd_pod(3, i % 2 == 0)] for i in range(45)])
    stale = [pod for u in c.units("single", 530, 1) for pod in u] + shuffled(g, c.units("twin", 15, 3))
    whole = c.units("whole", 200, 3)
    back = shuffled(g, whole)
    reuse = shuffled(g, [u[:2] for u in whole])
    tail = mixed_units(g, c, 3, 10, 10, 10, 6)
    small = [shuffled(g, tail[i::6]) for i in range(6)]
    gangs = [lead, big, stale, back, reuse] + small
    gmin = [1, 2000, len(stale), len(back), len(reuse)] + [len(s) if i % 2 else 1 for i, s in enumerate(small)]
    return gangs_args(c, gangs, gmin)


def mixed_gangs(seed, N, D, k_hi, triples, twins, singles, odd, big=True):
    """Units grouped whole into gangs of 1 to 12 units, gang 3 of a third of the units when `big`; gang_min the
    gang's size (given back unless every pod commits), 1, or in between."""
    g = np.random.default_rng(seed)
    c = Cluster(g, N, D)
    u = mixed_units(g, c, k_hi, triples, twins, singles, odd)
    sizes = []
    while sum(sizes) < len(u):
        sizes.append(len(u) // 3 if big and len(sizes) == 3 else int(g.integers(1, 13)))
    cuts = np.minimum(np.cumsum([0] + sizes), len(u))
    gangs = [shuffled(g, u[cuts[i]:cuts[i + 1]]) for i in range(len(sizes))]
    gmin = []
    for gang in gangs:
        r = g.random()
        gmin.append(len(gang) if r < 0.4 else 1 if r < 0.7 else int(g.integers(1, len(gang) + 1)))
    return gangs_args(c, gangs, gmin)


def given_back_call(nw, seed=7):
    """At N_wave: a lead gang, then gang 1 of 700 whole units (2 100 pods, gang_min 2 100), given back after three
    rounds, then gang 2 (1 400 pods) that fits only the whole cards gang 1 gave back, then small mixed gangs.
    Returns (arguments, j = 1)."""
    g = np.random.default_rng(seed)
    c = Cluster(g, nw, 8)
    lead = shuffled(g, mixed_units(g, c, 3, 40, 40, 40, 10))
    whole = c.units("whole", 700, 3)
    tail = mixed_units(g, c, 8, 20, 20, 20, 10)
    small = [shuffled(g, tail[i::5]) for i in range(5)]
    gangs = [lead, shuffled(g, whole), shuffled(g, [u[:2] for u in whole])] + small
    gmin = [1, 2100, 1400] + [len(s) if i % 2 else 1 for i, s in enumerate(small)]
    return gangs_args(c, gangs, gmin), 1


def without_gang(a, j):
    """place_gangs' arguments with gang j deleted: its pods and containers gone, the later ones re-indexed."""
    fc, fm, dv, rc, rm, off, goff, gmin = a
    g0, g1 = int(goff[j]), int(goff[j + 1])
    c0, c1 = int(off[g0]), int(off[g1])
    return [fc, fm, dv, np.delete(rc, np.s_[c0:c1]), np.delete(rm, np.s_[c0:c1]),
            np.concatenate([off[:g0], off[g1:] - (c1 - c0)]).astype(np.int32),
            np.concatenate([goff[:j], goff[j + 1:] - (g1 - g0)]).astype(np.int32), np.delete(gmin, j)]


def given_back_outputs(a, j, out):
    """The outputs of a call in which gang j was given back, with gang j's entries deleted, for comparison with the
    call without gang j (§2.13: a gang given back leaves the tables as they were).  Asserts that gang j holds
    nothing."""
    node, dev, placed, fco, fmo = [np.asarray(x) for x in out[:5]]
    off, goff = a[5], a[6]
    g0, g1 = int(goff[j]), int(goff[j + 1])
    c0, c1 = int(off[g0]), int(off[g1])
    assert placed[j] == 0 and (node[g0:g1] == -1).all() and (dev[c0:c1] == -1).all()
    return [np.delete(node, np.s_[g0:g1]), np.delete(dev, np.s_[c0:c1]), np.delete(placed, j), fco, fmo]


# ---- the cases and their references -------------------------------------------------------------------------------
NW = n_wave(SMS)  # 4261 on a 132-SM H100
CASES = {  # name -> (operator, builder of the arguments given N_wave)
    # a round 2 of more than 2 048 positions that defers in every stage: N_wave x 8, pods of 1 to 8 containers
    "pods_wave": ("pods", lambda nw: pods_case(11, nw, 8, 8, 1100, 200, 0, 20, 40)),
    # the same at D = 64 and N = 128
    "pods_d64": ("pods", lambda nw: pods_case(12, 128, 64, 3, 900, 400, 0, 10, 20)),
    # N <= 8 and G <= 256: a one-CTA grid, three rounds
    "pods_one_cta": ("pods", lambda nw: pods_case(13, 8, 16, 3, 10, 8, 6, 4, 4)),
    # N <= 8 and G > 2 048: ceil(G / 256) CTAs, one commit tile walking two stages
    "pods_n8_wide": ("pods", lambda nw: pods_case(14, 8, 64, 2, 60, 60, 0, 1000, 1000)),
    # place_tables' rows as pods of one container: a round 2 of more than 2 048 rows at N_wave
    "tables_wave": ("pods", lambda nw: pods_case(15, nw, 2, 1, 2000, 600, 0, 10, 18)),
    "gangs_sequence": ("gangs", lambda nw: gang_sequence()),
    "gangs_257": ("gangs", lambda nw: mixed_gangs(21, 257, 8, 8, 30, 40, 60, 20, big=False)),
    "gangs_1031": ("gangs", lambda nw: mixed_gangs(22, 1031, 8, 8, 150, 150, 200, 40)),
    "gangs_wave": ("gangs", lambda nw: mixed_gangs(23, nw, 8, 8, 350, 250, 350, 60)),
}


def restate(op, a, trace=None):
    return (place_pods_np if op == "pods" else place_gangs_np).place(*a, trace=trace)


@functools.lru_cache(maxsize=None)
def reference(name, nw):
    """(operator, arguments, the restatement's outputs, its round trace) of a named case for N_wave = nw, computed
    once per process and per (name, nw): the GPU file's calls on a 132-SM device hit the entries of these tests.
    Read-only."""
    op, build = CASES[name]
    a = build(nw)
    trace = []
    return op, a, restate(op, a, trace), trace


# ---- what a trace shows --------------------------------------------------------------------------------------------
def ragged(m):
    """The first position of the last compaction tile of m positions when that tile is ragged, else None."""
    return m // BLOCK * BLOCK if m % BLOCK else None


def rounds_of(trace, j):
    return [(len(pos), dfr) for gang, pos, dfr in trace if gang == j]


def stale_tiles(trace):
    """Launch rounds r whose count array holds, without the zeroing over ceil(G / 256) tiles, counts of round r - 2:
    round r - 2 deferred pods in tiles at or past round r - 1's tiles, round r - 1 is the last of that gang, and round
    r (the next gang's first) reads one of those tiles.  Returns [(r, stale tiles round r reads)], r counted from 1."""
    out = []
    for r in range(2, len(trace)):
        (j2, p2, d2), (j1, p1, _), (j0, p0, _) = trace[r - 2], trace[r - 1], trace[r]
        if j2 == j1 and j0 != j1:
            tiles = set((d2 // BLOCK).tolist())
            read = {t for t in tiles if t >= -(-len(p1) // BLOCK) and t < -(-len(p0) // BLOCK)}
            if read:
                out.append((r + 1, sorted(read)))
    return out


# ---- preconditions -------------------------------------------------------------------------------------------------
def test_thresholds_of_the_node_counts():
    assert NW == 4261 and 2 * 8 * 2 * SMS < NW < 3 * 8 * 2 * SMS  # commit CTAs walk two or three table tiles
    assert -(-NW // 8) > 2 * SMS and -(-128 // 8) < 2 * SMS


@pytest.mark.parametrize("name", ["pods_wave", "pods_d64", "tables_wave"])
def test_a_later_round_restages_and_defers_in_every_stage(name):
    """A round >= 2 of more than 2 048 positions: deferred pods in more than one stage and in a ragged last tile.
    The case runs few rounds, and its round 1 has deferred pods past the first tile."""
    op, a, exp, trace = reference(name, NW)
    later = [(len(pos), dfr) for _, pos, dfr in trace[1:] if len(pos) > STAGE]
    assert later, [len(p) for _, p, _ in trace]
    m, dfr = later[0]
    assert len(set((dfr // STAGE).tolist())) >= 2 and ragged(m) is not None and (dfr >= ragged(m)).any(), name
    assert 3 <= exp[4][0] == len(trace) <= 4 and (trace[0][2] >= BLOCK).any(), name
    assert 0 < (exp[0] == -1).sum() <= 60, name  # the odd pods only
    gpu_pods.invariants(*a, exp)
    if name == "tables_wave":
        assert (np.diff(a[5]) == 1).all() and a[3].size % 4 == 0 and a[3].size > 2 * STAGE
    elif name == "pods_wave":  # pods of 1 to 8 containers, and pods outside the domain
        assert set(np.diff(a[5]).tolist()) == set(range(1, 9)) and a[0].shape == (NW, 8)


def test_one_cta_grid_runs_several_rounds():
    op, a, exp, trace = reference("pods_one_cta", NW)
    assert a[0].shape[0] <= 8 and a[5].size - 1 <= BLOCK  # ceil(N / 8) x ceil(G / 256) = 1 CTA
    assert exp[4][0] == len(trace) >= 3 and all(len(d) for _, _, d in trace[:2])


def test_n8_with_more_than_2048_pods_defers_in_two_stages():
    op, a, exp, trace = reference("pods_n8_wide", NW)
    G = a[5].size - 1
    assert a[0].shape[0] <= 8 and G > STAGE  # one table tile, ceil(G / 256) = 16 CTAs
    dfr = trace[0][2]
    assert len(set((dfr // STAGE).tolist())) == 2 and exp[4][0] == len(trace) >= 3
    assert (exp[0] >= 0).sum() == 3 * 60 + 2 * 60  # every unit's pods, no odd pod


def test_gang_sequence_crosses_every_gang_threshold():
    op, a, exp, trace = reference("gangs_sequence", NW)
    node, dev, placed, fco, fmo, info = exp
    goff, gmin = a[6], a[7]
    size = np.diff(goff)
    lead, big, stale, back, reuse = 0, 1, 2, 3, 4
    # big: more than 2 048 pods from a first pod that is not a multiple of 256; defers in round 2 in many tiles
    assert size[big] > STAGE and goff[big] % BLOCK != 0
    r = rounds_of(trace, big)
    assert len(r) == 3 and r[0][0] == size[big] and len(set((r[1][1] // BLOCK).tolist())) >= 4
    assert r[1][0] > 4 * BLOCK and placed[big] >= gmin[big]
    # stale: deferred only past its round 1's first two tiles, then one small round that ends the gang
    r = rounds_of(trace, stale)
    assert len(r) == 2 and r[0][1].min() >= 2 * BLOCK and r[1][0] <= BLOCK and len(r[1][1]) == 0
    assert placed[stale] == size[stale]
    # the round after it is back's first, over 600 positions: it reads the counts of tile 2 stale's round 1 wrote
    first_back = [i for i, (j, _, _) in enumerate(trace) if j == back][0]
    assert (first_back + 1, [2]) in stale_tiles(trace)
    # back: more than 256 pods, not on a tile boundary, defers in rounds 1 and 2, given back after three rounds
    r = rounds_of(trace, back)
    assert size[back] > BLOCK and goff[back] % BLOCK != 0 and len(r) == 3 and len(r[1][1]) > 0
    assert placed[back] == 0 and gmin[back] == size[back]
    # reuse: every pod placed, on the whole cards back gave back; kept gangs before and after back share its nodes
    g0, g1 = goff[reuse], goff[reuse + 1]
    pod_of = np.repeat(np.arange(node.size), np.diff(a[5]))
    mine = (pod_of >= g0) & (pod_of < g1)
    assert placed[reuse] == size[reuse] and (a[0][node[pod_of[mine]], dev[mine]] == CORE_MAX).all()
    before = set(node[goff[stale]:goff[stale + 1]].tolist())
    assert len(before & set(node[g0:g1].tolist())) >= 20
    assert ((placed == 0) | (placed >= gmin)).all() and (placed[5:] > 0).any() and info[0] == len(trace)
    gpu_gangs.invariants(a, exp)


@pytest.mark.parametrize("name", ["gangs_257", "gangs_1031", "gangs_wave"])
def test_mixed_gangs(name):
    """Gangs of mixed sizes (past 256 pods at N = 1031 and N_wave) and gang_min: some kept whole, some kept in part,
    some given back, and gangs that run three rounds."""
    op, a, exp, trace = reference(name, NW)
    placed, goff, gmin = exp[2], a[6], a[7]
    size = np.diff(goff)
    assert ((placed > 0) & (placed == size)).any() and ((placed > 0) & (placed < size)).any(), name
    assert ((placed == 0) & (gmin == size)).sum() >= 2 and (gmin < size).sum() >= 3, name
    assert max(len(rounds_of(trace, j)) for j in range(size.size)) == 3 and exp[5][0] == len(trace), name
    if name != "gangs_257":
        assert size.max() > BLOCK and goff[size.argmax()] % BLOCK != 0, name
    gpu_gangs.invariants(a, exp)


def test_given_back_call_builds():
    """The relation test's call at N_wave: a gang of more than 2 048 pods with gang_min = size, and a later gang that
    fits only the whole cards it holds (shown on the GPU, where the call runs)."""
    a, j = given_back_call(NW)
    size = np.diff(a[6])
    assert size[j] > STAGE and a[7][j] == size[j] and size[j + 1] == 2 * size[j] // 3 and a[0].shape[0] == NW


# ---- the pod choice word: hand-derived known answers ---------------------------------------------------------------
# One pod of five containers (1 core, 0 memory).  Node 0 holds (2, 0) and four (1, 0): the best fit leaves
# sum lc = 1, sum lm = 0.  Node 1 holds five (1, MEM_MAX): sum lc = 0, sum lm = 5 x MEM_MAX = 1 310 715 >= 2^20.  The
# word ~(sum lc << 52 | sum lm << 31 | n) picks node 1; a word with sum lc shifted by 51 bits or less would have
# sum lm carry past it and pick node 0.  A second pod finds node 1 taken and goes to node 0 in round 2.
# The maxima: eight containers of (0, 0) on a device (100, MEM_MAX) leave sum lc = 800 and sum lm = 8 x MEM_MAX =
# 2 097 144; a tie of two such nodes goes to the lower n, and a node with one memory unit less per container wins.
KAT = [
    dict(name="sum lm >= 2^20 against sum lc one larger", free_core=[[2, 1, 1, 1, 1], [1] * 5],
         free_mem=[[0] * 5, [MEM_MAX] * 5], d_valid=[5, 5], req_core=[1] * 5, req_mem=[0] * 5,
         pod_offsets=[0, 5], node=[1], dev=[0, 1, 2, 3, 4], free_core_out=[[2, 1, 1, 1, 1], [0] * 5],
         free_mem_out=[[0] * 5, [MEM_MAX] * 5], rounds=1),
    dict(name="sum lm >= 2^20, a second pod in round 2", free_core=[[2, 1, 1, 1, 1], [1] * 5],
         free_mem=[[0] * 5, [MEM_MAX] * 5], d_valid=[5, 5], req_core=[1] * 10, req_mem=[0] * 10,
         pod_offsets=[0, 5, 10], node=[1, 0], dev=[0, 1, 2, 3, 4, 1, 2, 3, 4, 0],
         free_core_out=[[1, 0, 0, 0, 0], [0] * 5], free_mem_out=[[0] * 5, [MEM_MAX] * 5], rounds=2),
    dict(name="maxima sum lc = 800, sum lm = 2 097 144: a tie goes to the lower n",
         free_core=[[100, 7], [100, 100]], free_mem=[[MEM_MAX, 7], [MEM_MAX, MEM_MAX]], d_valid=[1, 2],
         req_core=[0] * 8, req_mem=[0] * 8, pod_offsets=[0, 8], node=[0], dev=[0] * 8,
         free_core_out=[[100, 7], [100, 100]], free_mem_out=[[MEM_MAX, 7], [MEM_MAX, MEM_MAX]], rounds=1),
    dict(name="maxima: sum lm 8 less wins", free_core=[[100, 7], [100, 100], [100, 100]],
         free_mem=[[MEM_MAX, 7], [MEM_MAX, MEM_MAX], [MEM_MAX, MEM_MAX - 1]], d_valid=[1, 2, 2],
         req_core=[0] * 8, req_mem=[0] * 8, pod_offsets=[0, 8], node=[2], dev=[1] * 8,
         free_core_out=[[100, 7], [100, 100], [100, 100]],
         free_mem_out=[[MEM_MAX, 7], [MEM_MAX, MEM_MAX], [MEM_MAX, MEM_MAX - 1]], rounds=1),
]
KAT_KEYS = ("free_core", "free_mem", "d_valid", "req_core", "req_mem", "pod_offsets")


def kat_args(c):
    return [np.array(c[k], np.int32) for k in KAT_KEYS]


@pytest.mark.parametrize("case", range(len(KAT)))
def test_choice_word_known_answers_are_the_restatement(case):
    c = KAT[case]
    a = kat_args(c)
    assert place_pods_np.valid_devices(*a[:3]).any(axis=1).all()
    node, dev, fco, fmo, info = place_pods_np.place(*a)
    assert node.tolist() == c["node"] and dev.tolist() == c["dev"], c["name"]
    assert fco.tolist() == c["free_core_out"] and fmo.tolist() == c["free_mem_out"], c["name"]
    assert info == [c["rounds"], 0, 0], c["name"]


def test_choice_word_known_answers_decide_at_the_edges():
    """The sums the known answers are about, recomputed with the restatement's replay."""
    sums = []
    for c in KAT[::2] + KAT[3:]:
        a = kat_args(c)
        valid = place_pods_np.valid_devices(*a[:3])
        fits, _, slc, slm = place_pods_np.replay_all(a[0].astype(np.int64), a[1].astype(np.int64), valid,
                                                     a[3][:a[5][1]].astype(np.int64), a[4][:a[5][1]].astype(np.int64))
        assert fits.all()
        sums.append(list(zip(slc.tolist(), slm.tolist())))
    assert sums[0] == [(1, 0), (0, 5 * MEM_MAX)] and 5 * MEM_MAX >= 1 << 20
    assert (1 << 51) < (5 * MEM_MAX) << 31  # shifted by 51, node 1's sum lm would outweigh node 0's sum lc
    assert sums[1] == [(800, 8 * MEM_MAX)] * 2 and 8 * MEM_MAX == 2_097_144 < 1 << 21
    assert sums[2] == [(800, 8 * MEM_MAX)] * 2 + [(800, 8 * MEM_MAX - 8)]
