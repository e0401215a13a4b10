"""egpu::preempt_pods and egpu::preempt_gangs at scale, without a GPU: the generators of the cases in
tests/test_gpu_preempt_scale.py, preconditions showing that each case does what it is there for (it evicts, and it
crosses the kernel threshold it is named after), and the restatements checked against their literal rules in the new
regimes (full-range priorities, saturated clusters).

The kernels' thresholds (DESIGN.md §4.9, §4.10):
  - the choose phases split the N nodes into K = min(32, ceil(N / 8)) chunks, and warp w of a CTA scores nodes
    N k / K + w, + 8, ... of chunk k: past N = 256 a chunk has more than 8 nodes and some warp scores two;
  - the grid is min(SMs x CTAs per SM, K x G) CTAs of 8 warps, and the commit and usable passes walk the nodes with a
    stride of 8 x grid warps: a lone preemptor (G = 1) runs 32 CTAs, so each warp commits about N / 256 nodes;
  - a node's running pods sit in 4 slots of 32 lanes (running pod h0 + lane + 32 i is slot i of the lane);
  - preempt_gangs' budget pass walks a gang's waiting preemptors 32 pods at a time.

Each case's reference is computed once per process (`reference`), so the GPU file reuses what these tests computed.
"""
import functools
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import preempt_gangs_np  # noqa: E402
import preempt_pods_np  # noqa: E402
import test_gpu_preempt_gangs as gpu_gangs  # noqa: E402  (its invariants hold for the restatement too)
import test_preempt_gangs_cpu as gangs  # noqa: E402  (random running jobs and gangs)
import test_preempt_pods_cpu as pods  # noqa: E402  (random tables and running pods)

INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
# full-range priorities: the int32 ends, around 0, and Kubernetes' system classes (2 000 000 000 and 2 000 001 000)
RUN_PRIOS = np.array([INT32_MIN, INT32_MIN + 1, -1, 0, 10**9, 2 * 10**9, 2_000_001_000, INT32_MAX - 1])
PENDING_PRIOS = np.append(RUN_PRIOS, INT32_MAX)  # nothing runs at INT32_MAX, so such a pod may evict anything
BIAS = 1 << 31
SMS = 132  # an H100 SXM's SMs; the GPU tests take the count of the device they run on
CTA_WARPS = 8  # warps per CTA


def chunks(N):
    """The node counts of the choose phases' K chunks."""
    K = min(32, -(-N // CTA_WARPS))
    return [N * (k + 1) // K - N * k // K for k in range(K)]


def n_wave(sms):
    """Nodes for which the commit warps walk two or three nodes each: 37 past two strides of 8 warps x 2 CTAs per SM.
    Assumes 2 CTAs per SM, the occupancy of both kernels on sm_90a (256 threads, at most 128 registers)."""
    return 2 * CTA_WARPS * 2 * sms + 37


# ---- generators --------------------------------------------------------------------------------------------------
# The preempt_pods arguments are [fc, fm, dv, rc, rm, pod_offsets, pod_prio, qc, qm, qd, run_offsets, run_prio,
# node_offsets]; the preempt_gangs ones [fc, fm, dv, rc, rm, pod_offsets, gang_offsets, gang_min, gang_prio, qc, qm,
# qd, run_offsets, run_prio, node_offsets, run_gang, run_gang_min].
def saturate(a, g, share=0.9):
    """Zero `share` of the free core entries after the running pods are placed, so most pending pods only fit by
    evicting.  Free capacity only shrinks, so every node stays consistent."""
    a[0][g.random(a[0].shape) < share] = 0
    return a


def full_range(a, g, gang_args=False):
    """Running priorities drawn from RUN_PRIOS, pending ones (or the gangs') from PENDING_PRIOS."""
    pending, running = (8, 13) if gang_args else (6, 11)
    a[running] = g.choice(RUN_PRIOS, a[running].size).astype(np.int32)
    a[pending] = g.choice(PENDING_PRIOS, a[pending].size).astype(np.int32)
    return a


def dense_nodes(a, g, lo, hi):
    """preempt_pods' arguments in which every node runs lo to hi pods instead of what it ran, each of one container of
    1 core (0 once its device is full) and 0, 100 or 1000 memory on a random device, at priority 0 until full_range
    draws the priorities.  The free tables are what those pods leave of 100 core and 80 000 memory per device
    (consistent by construction)."""
    fc, fm, dv = a[:3]
    N, D = fc.shape
    qc, qm, qd, noff = [], [], [], [0]
    for n in range(N):
        left_c, left_m = np.full(D, 100), np.full(D, 80_000)
        for _ in range(int(g.integers(lo, hi + 1))):
            d = int(g.integers(0, dv[n]))
            c, m = int(min(left_c[d], 1)), int(min(left_m[d], g.choice([0, 100, 1000])))
            left_c[d] -= c
            left_m[d] -= m
            qc.append(c)
            qm.append(m)
            qd.append(d)
        fc[n], fm[n] = left_c, left_m
        noff.append(len(qc))
    H = len(qc)
    a[7:13] = [np.array(qc, np.int32), np.array(qm, np.int32), np.array(qd, np.int8), np.arange(H + 1, dtype=np.int32),
               np.zeros(H, np.int32), np.array(noff, np.int32)]
    return a


def gang_layer(a, g, sizes, gmin, R, below=2):
    """preempt_gangs' arguments from preempt_pods' ones: the pending pods grouped in order into gangs of `sizes` pods
    (summing to G) with minimums gmin, each gang at the priority of its first pod, and the running pods grouped into R
    running jobs (about a third of them in none), each job's minimum its size less 0 to `below`."""
    fc, fm, dv, rc, rm, off, prio, qc, qm, qd, roff, rprio, noff = a
    goff = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    assert goff[-1] == off.size - 1
    H = rprio.size
    rgang = np.where(g.random(H) < 0.35, -1, g.integers(0, R, H)).astype(np.int32)
    size = np.bincount(rgang[rgang >= 0], minlength=R)
    rgmin = np.maximum(size - g.integers(0, below + 1, R), 0).astype(np.int32)
    return [fc, fm, dv, rc, rm, off, goff, np.asarray(gmin, np.int32), prio[goff[:-1]].copy(), qc, qm, qd, roff,
            rprio, noff, rgang, rgmin]


def saturated_pods(seed, N, D, G, share=0.9, **kw):
    g = np.random.default_rng(seed)
    return saturate(pods.random_case(g, N, D, G, **kw), g, share)


def lone_pods(seed, N, G):
    """G preemptors on a cluster with no free core at all: each pod evicts or is -1."""
    g = np.random.default_rng(seed)
    a = saturate(pods.random_case(g, N, 8, G, run_lo=2, run_hi=6), g, 1.0)
    a[6] = g.choice([10, 2_000_001_000, INT32_MAX], G).astype(np.int32)
    return a


def full_range_pods(seed, N, G, share=0.9):
    g = np.random.default_rng(seed)
    return full_range(saturate(pods.random_case(g, N, 8, G), g, share), g)


def full_range_gangs(seed, N, J, share=0.9):
    g = np.random.default_rng(seed)
    return full_range(saturate(gangs.random_case(g, N, 8, J, hi_gang=6), g, share), g, gang_args=True)


def dense_full_range(seed, N, G, J=None):
    """One device per node holding 64 to 128 running pods of 1 core (100 of them at most hold core), full-range
    priorities with 40 % of the pending pods at INT32_MAX: a pod of 100 core evicts up to 100 of them, and the sums
    of their priorities straddle 2^38."""
    g = np.random.default_rng(seed)
    a = pods.random_case(g, N, 1, G, run_hi=0, hi_pod=1)
    a = full_range(saturate(dense_nodes(a, g, 64, 128), g, 1.0), g)
    a[6][g.random(G) < 0.4] = INT32_MAX  # pods that may evict a whole node
    if J is None:
        return a
    sizes = np.diff(np.linspace(0, G, J + 1).astype(np.int64))
    return gang_layer(a, g, sizes, np.ones(J), R=24, below=10**4)


def big_gangs(seed, N, J, R=200):
    """Gangs of 33 to 150 pods with minimums mostly well below their size on a saturated cluster, and about 200
    running jobs whose minimums are at or just below their size."""
    g = np.random.default_rng(seed)
    sizes = g.integers(33, 151, J)
    a = saturate(pods.random_case(g, N, 8, int(sizes.sum()), run_hi=6), g)
    gmin = np.where(g.random(J) < 0.5, 1, g.integers(1, sizes // 4 + 2))
    return gang_layer(a, g, sizes, gmin, R)


def given_back_case(seed=41):
    """Big gangs at N = 257 whose gang 1 has 80 pods, the last of which asks for more memory than any device has, so
    gang 1 starts only with gang_min below 80.  Returns (arguments, j = 1)."""
    g = np.random.default_rng(seed)
    sizes = np.array([40, 80, 60, 50])
    a = saturate(pods.random_case(g, 257, 8, int(sizes.sum()), run_hi=6), g)
    a[6][:] = INT32_MAX
    a = gang_layer(a, g, sizes, [1, 1, 1, 1], R=120, below=3)
    last = a[6][2] - 1  # the last pod of gang 1
    a[4][a[5][last]] = 80_001  # no device has 80 001 memory, evicting everything on it included
    return a, 1


def without_gang(a, j):
    """preempt_gangs' arguments with gang j deleted: its pods and containers gone, the later ones re-indexed."""
    fc, fm, dv, rc, rm, off, goff, gmin, gprio, *run = a
    g0, g1 = int(goff[j]), int(goff[j + 1])
    c0, c1 = int(off[g0]), int(off[g1])
    return [fc, fm, dv, np.delete(rc, np.s_[c0:c1]), np.delete(rm, np.s_[c0:c1]),
            np.concatenate([off[:g0], off[g1:] - (c1 - c0)]).astype(np.int32),
            np.concatenate([goff[:j], goff[j + 1:] - (g1 - g0)]).astype(np.int32), np.delete(gmin, j),
            np.delete(gprio, j), *run]


def given_back_outputs(a, j, out):
    """The outputs of a call in which gang j was given back, with gang j's entries deleted and the later pods
    re-indexed in `evicted`, for comparison with the call without gang j (§2.15: a gang given back changes nothing
    later gangs see).  Asserts that gang j placed and evicted nothing."""
    node, dev, placed, evicted, fco, fmo = [np.asarray(x) for x in out[:6]]
    off, goff = a[5], a[6]
    g0, g1 = int(goff[j]), int(goff[j + 1])
    c0, c1 = int(off[g0]), int(off[g1])
    assert placed[j] == 0 and (node[g0:g1] == -1).all() and (dev[c0:c1] == -1).all()
    assert not ((evicted >= g0) & (evicted < g1)).any()
    evicted = np.where(evicted >= g1, evicted - (g1 - g0), evicted).astype(np.int32)
    return [np.delete(node, np.s_[g0:g1]), np.delete(dev, np.s_[c0:c1]), np.delete(placed, j), evicted, fco, fmo]


def with_gang_min(a, j, m):
    b = list(a)
    b[7] = a[7].copy()
    b[7][j] = m
    return b


# ---- the cases and their references -------------------------------------------------------------------------------
NW = n_wave(SMS)  # 4261 on a 132-SM H100
CASES = {  # name -> (operator, builder of the arguments given N_wave)
    "pods_247": ("pods", lambda nw: saturated_pods(247, 247, 8, 300)),
    "pods_256": ("pods", lambda nw: saturated_pods(256, 256, 8, 300)),
    "pods_257": ("pods", lambda nw: saturated_pods(257, 257, 8, 300)),
    "pods_1031": ("pods", lambda nw: saturated_pods(1031, 1031, 8, 400)),
    "pods_wave": ("pods", lambda nw: saturated_pods(nw, nw, 8, 150, share=1.0)),
    "pods_600x64": ("pods", lambda nw: saturated_pods(600, 600, 64, 200, share=1.0, run_hi=24, hi_pod=8)),
    "lone_1": ("pods", lambda nw: lone_pods(31, 3001, 1)),
    "lone_2": ("pods", lambda nw: lone_pods(32, 3001, 2)),
    "lone_3": ("pods", lambda nw: lone_pods(33, 3001, 3)),
    "full_pods_257": ("pods", lambda nw: full_range_pods(1257, 257, 300)),
    "full_pods_wave": ("pods", lambda nw: full_range_pods(1000 + nw, nw, 150, share=1.0)),
    "full_pods_dense": ("pods", lambda nw: dense_full_range(61, 64, 120)),
    "full_gangs_257": ("gangs", lambda nw: full_range_gangs(2257, 257, 80)),
    "full_gangs_wave": ("gangs", lambda nw: full_range_gangs(2000 + nw, nw, 40, share=1.0)),
    "full_gangs_dense": ("gangs", lambda nw: dense_full_range(61, 64, 120, J=60)),
    "big_gangs_257": ("gangs", lambda nw: big_gangs(3257, 257, 4)),
    "big_gangs_1031": ("gangs", lambda nw: big_gangs(4031, 1031, 6)),
    "big_gangs_wave": ("gangs", lambda nw: big_gangs(3000 + nw, nw, 3)),
}


def restate(op, a):
    return (preempt_pods_np if op == "pods" else preempt_gangs_np).place(*a)


@functools.lru_cache(maxsize=None)
def reference(name, nw):
    """(operator, arguments, the restatement's outputs) of a named case for N_wave = nw, computed once per process
    and per (name, nw): the GPU file's calls on a 132-SM device hit the entries of these tests.  Read-only."""
    op, build = CASES[name]
    a = build(nw)
    return op, a, restate(op, a)


@functools.lru_cache(maxsize=None)
def given_back_reference():
    """(arguments, j, outputs with gang_min = 1, outputs with gang_min = size, outputs without gang j)."""
    a, j = given_back_case()
    size = int(a[6][j + 1] - a[6][j])
    return (a, j, preempt_gangs_np.place(*with_gang_min(a, j, 1)), preempt_gangs_np.place(*with_gang_min(a, j, size)),
            preempt_gangs_np.place(*without_gang(a, j)))


# ---- what the outputs show ---------------------------------------------------------------------------------------
def run_layout(op, a):
    """(run_offsets, run_prio, node_offsets, run_gang or None) of either operator's arguments."""
    return (a[10], a[11], a[12], None) if op == "pods" else (a[12], a[13], a[14], a[15])


def slots(noff):
    """Each running pod's slot on its node."""
    H = int(noff[-1])
    return (np.arange(H) - np.repeat(noff[:-1], np.diff(noff))) >> 5


def victim_sums(rprio, evicted):
    """{evicting pod: sum over its victims of (priority + 2^31)}, exact."""
    out = {}
    for h in np.flatnonzero(evicted >= 0):
        out[int(evicted[h])] = out.get(int(evicted[h]), 0) + int(rprio[h]) + BIAS
    return out


def gang_pos(goff, G):
    """Each pod's gang and its index within the gang."""
    gang_of = np.repeat(np.arange(goff.size - 1), np.diff(goff))
    return gang_of, np.arange(G) - goff[gang_of]


# ---- preconditions -------------------------------------------------------------------------------------------------
def test_thresholds_of_the_node_counts():
    assert len(chunks(247)) == 31 and max(chunks(247)) == 8
    assert chunks(256) == [8] * 32  # one node per warp
    assert len(chunks(257)) == 32 and max(chunks(257)) == 9  # one warp scores two
    assert min(chunks(1031)) == 32 and min(chunks(NW)) >= 133  # every warp scores 4, or 16 and more
    assert NW == 4261 and 2 * 8 * 2 * SMS < NW < 3 * 8 * 2 * SMS  # commit warps walk two or three nodes
    assert 8 * 32 * 11 < 3001 < 8 * 96 * 4  # lone pods: 32 CTAs walk 11 or 12 nodes a warp, 96 CTAs 3 or 4


@pytest.mark.parametrize("name", [n for n, (op, _) in CASES.items() if op == "pods" and not n.startswith("lone")])
def test_pods_cases_evict_many(name):
    op, a, exp = reference(name, NW)
    node, dev, evicted, fco, fmo, info = exp
    evictors = set(evicted[evicted >= 0].tolist())
    assert (node >= 0).sum() >= 30 and len(evictors) >= 20 and (evicted >= 0).sum() >= 40, name
    assert info[0] >= 2, name  # some preemptor waited for a later round
    if name.startswith("full"):  # victims at both ends of the range, and pods placed at INT32_MAX and below 0
        rprio, prio = a[11], a[6]
        assert (rprio[evicted >= 0] == INT32_MIN).any() and (prio[node >= 0] == INT32_MAX).any(), name
        assert (prio[node >= 0] < 0).any(), name
        if name != "full_pods_wave":  # there every preemptor finds a node with a victim at INT32_MIN
            assert (rprio[evicted >= 0] >= 10**9).sum() >= 5 and (rprio[evicted >= 0] >= 2 * 10**9).any(), name


@pytest.mark.parametrize("name", ["full_pods_dense", "full_gangs_dense"])
def test_dense_cases_straddle_2_38(name):
    """On a dense node with 100 pods of 1 core, a pod of 100 core at INT32_MAX evicts all 100, at the same highest
    victim priority (INT32_MAX - 1) on every such node.  Their sums of (priority + 2^31) straddle 2^38 across those
    nodes, so a key that wrapped the shifted sum would choose differently.  Such pods evict, in all four slots."""
    op, a, exp = reference(name, NW)
    roff, rprio, noff, _ = run_layout(op, a)
    qc, rc, off = (a[7], a[3], a[5]) if op == "pods" else (a[9], a[3], a[5])
    evicted = exp[2] if op == "pods" else exp[3]
    N = noff.size - 1
    node_of = np.repeat(np.arange(N), np.diff(noff))
    holds = qc[roff[:-1]] > 0  # one container per running pod
    full = np.bincount(node_of[holds], minlength=N) == 100
    sums = np.zeros(N, object)
    top = np.full(N, INT32_MIN, np.int64)
    for h in np.flatnonzero(holds):
        sums[node_of[h]] += int(rprio[h]) + BIAS
        top[node_of[h]] = max(top[node_of[h]], int(rprio[h]))
    assert (sums[full] >= 2**38).sum() >= 3 and (sums[full] < 2**38).sum() >= 10, name
    assert (top[full] == INT32_MAX - 1).all(), name
    big = [g for g, s in victim_sums(rprio, evicted).items() if (rc[off[g]:off[g + 1]] == 100).any()]
    assert len(big) >= 3, name
    assert set(slots(noff)[evicted >= 0].tolist()) == {0, 1, 2, 3}, name


@pytest.mark.parametrize("G", [1, 2, 3])
def test_lone_pods_all_evict(G):
    op, a, exp = reference(f"lone_{G}", NW)
    node, evicted = exp[0], exp[2]
    assert (node >= 0).all() and set(evicted[evicted >= 0].tolist()) == set(range(G))
    if G == 1:
        pods.equal(exp, preempt_pods_np.single(*a))


@pytest.mark.parametrize("name", [n for n, (op, _) in CASES.items() if op == "gangs"])
def test_gangs_cases_evict_in_jobs(name):
    op, a, exp = reference(name, NW)
    node, dev, placed, evicted, fco, fmo, info = exp
    goff, rgang, noff = a[6], a[15], a[14]
    in_job = (evicted >= 0) & (rgang >= 0)
    assert in_job.sum() >= 10 and (placed > 0).sum() >= 2 and info[0] >= 2 * (goff.size - 1) // 3, name
    if name.startswith("big"):
        # gangs of more than 32 pods evict in jobs, by pods past their first 32 (the budget pass's second step)
        gang_of, pos = gang_pos(goff, node.size)
        by = evicted[in_job]
        assert (np.diff(goff)[gang_of[by]] > 32).all() and (pos[by] >= 32).sum() >= 10, name
        gpu_gangs.invariants(a, exp)


def test_known_answer_counts_a_slot_3_victim_in_the_round_budget():
    """preempt_gangs' known answers include a round in which the earlier preemptor's only job victim is in slot 3 of a
    node with 97 running pods, and that victim alone takes the job's slack, so the later preemptor is deferred."""
    c = next(c for c in gangs.KAT if c["name"].startswith("round budget: a job victim in slot 3"))
    noff, rgang, evicted = np.array(c["node_offsets"]), np.array(c["run_gang"]), np.array(c["evicted"])
    gone = np.flatnonzero(evicted >= 0)
    assert noff[1] - noff[0] >= 97 and gone.tolist() == [96] and slots(noff)[96] == 3 and rgang[96] == 0
    job = np.flatnonzero(rgang == 0)
    assert job.size - c["run_gang_min"][0] == 1 and c["node"][1] == -1 and c["info"][0] == 2


def test_given_back_gang():
    """Gang 1 (80 pods) evicts pods of running jobs with gang_min = 1; with gang_min = 80 it is given back, and the
    call then equals the call without it."""
    a, j, kept, back, without = given_back_reference()
    goff, rgang = a[6], a[15]
    g0, g1 = goff[j], goff[j + 1]
    ev = kept[3]
    mine = (ev >= g0) & (ev < g1)
    assert g1 - g0 >= 64 and kept[2][j] >= 1 and (mine & (rgang >= 0)).sum() >= 10
    assert back[2][j] == 0 and (back[2] > 0).sum() >= 2 and (back[3] >= 0).sum() >= 10
    for x, y in zip(given_back_outputs(a, j, back), without[:6]):
        np.testing.assert_array_equal(x, y)
    assert back[6][1:] == without[6][1:]


# ---- the restatements in the new regimes ---------------------------------------------------------------------------
def test_single_pod_equals_the_literal_rule_at_full_range():
    evictions = top = 0
    for seed in range(300):
        g = np.random.default_rng(7000 + seed)
        a = full_range(pods.random_case(g, int(g.integers(1, 7)), int(g.integers(1, 6)), 1, run_hi=6, full=0.9,
                                        bad_nodes=0.2 if seed % 3 == 0 else 0.0), g)
        got = preempt_pods_np.place(*a)
        pods.equal(got, preempt_pods_np.single(*a))
        evictions += int((got[2] >= 0).any())
        top += int((a[11][got[2] >= 0] >= 2 * 10**9).any())
    assert evictions >= 60 and top >= 10, (evictions, top)


def test_no_running_job_is_the_literal_loop_when_saturated():
    evicted = given_back = 0
    for seed in range(200):
        g = np.random.default_rng(8000 + seed)
        a = saturate(gangs.random_case(g, int(g.integers(1, 9)), int(g.integers(1, 6)), int(g.integers(1, 9)),
                                       R=0, run_hi=6), g, float(g.choice([0.7, 0.9, 1.0])))
        if seed % 2:
            a = full_range(a, g, gang_args=True)
        got, exp = preempt_gangs_np.place(*a), preempt_gangs_np.loop(*a)
        for x, y in zip(got[:6], exp[:6]):
            np.testing.assert_array_equal(x, y)
        assert got[6][0] <= exp[6][0]
        evicted += int((got[3] >= 0).any())
        given_back += int((got[2] == 0).any())
    assert evicted >= 100 and given_back >= 30, (evicted, given_back)
