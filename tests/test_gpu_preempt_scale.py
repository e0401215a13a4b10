"""egpu::preempt_pods and egpu::preempt_gangs on the GPU at the kernels' chunk, grid and slot thresholds: the cases of
tests/test_preempt_scale_cpu.py against the numpy restatements bit for bit (info included), and the invariants.

  1. preempt_pods on saturated clusters at N = 247 (K = 31 chunks), 256 (one node per warp), 257 (one warp scores
     two), 1031, N_wave (commit warps walk two or three nodes) and 600 x 64;
  2. lone preemptors (G = 1, 2, 3: grids of 32, 64 and 96 CTAs) on a saturated cluster of 3001 nodes;
  3. full-range priorities, both operators, at N = 257 and N_wave and on dense nodes whose victim sums pass 2^38;
  4. preempt_gangs with gangs of 33 to 150 pods and about 200 running jobs at N = 257, 1031 and N_wave;
  5. a gang of 80 pods given back: the call equals the call without that gang.

The nodes at every slot edge are in test_gpu_preempt_pods.py and test_gpu_preempt_gangs.py.  Each reference is
computed once per process and shared with the CPU file's preconditions.
"""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import preempt_pods_np  # noqa: E402
import test_gpu_preempt_gangs as gangs  # noqa: E402  (check, invariants of preempt_gangs)
import test_gpu_preempt_pods as pods  # noqa: E402  (check, invariants of preempt_pods)
import test_preempt_scale_cpu as scale  # noqa: E402  (the cases and their references)


@pytest.fixture(scope="module")
def tables():
    from elastic_gpu_agent_b200 import tables as t
    t.load()
    return t


@pytest.fixture(scope="module")
def nw():
    """N_wave of this device, assuming 2 CTAs per SM (both kernels' occupancy on sm_90a): 4261 on a 132-SM H100."""
    return scale.n_wave(torch.cuda.get_device_properties(0).multi_processor_count)


def run_case(tables, name, nw):
    op, a, exp = scale.reference(name, nw)
    m = pods if op == "pods" else gangs
    out = m.run(tables, a)
    m.check(a, out, exp)
    m.invariants(a, out)
    return a, out


# ---- 1. chunk and grid thresholds, preempt_pods ------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["pods_247", "pods_256", "pods_257", "pods_1031", "pods_wave", "pods_600x64"])
def test_preempt_pods_chunk_and_grid_thresholds(name, tables, nw):
    a, out = run_case(tables, name, nw)
    assert (out[2] >= 0).sum() >= 40


# ---- 2. lone preemptors: small grids walking many nodes per warp -----------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 2, 3])
def test_lone_preemptors(G, tables, nw):
    a, out = run_case(tables, f"lone_{G}", nw)
    assert (out[0] >= 0).all() and set(out[2][out[2] >= 0].tolist()) == set(range(G))
    if G == 1:
        single = preempt_pods_np.single(*a)
        for x, y in zip(out[:5], single[:5]):
            np.testing.assert_array_equal(x, y)


# ---- 3. full-range priorities ------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["full_pods_257", "full_pods_wave", "full_pods_dense", "full_gangs_257",
                                  "full_gangs_wave", "full_gangs_dense"])
def test_full_range_priorities(name, tables, nw):
    run_case(tables, name, nw)


# ---- 4. big gangs with running jobs ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["big_gangs_257", "big_gangs_1031", "big_gangs_wave"])
def test_big_gangs_with_running_jobs(name, tables, nw):
    a, out = run_case(tables, name, nw)
    assert ((out[3] >= 0) & (a[15] >= 0)).sum() >= 10


# ---- 5. a gang given back is as if it were not there -------------------------------------------------------------
@pytest.mark.gpu
def test_given_back_gang_is_the_call_without_it(tables):
    """§2.15: a gang given back undoes its placements and evictions, and later gangs see the tables, the alive set and
    the slacks as they were before it.  So with gang_min = size the call equals the call without the gang, pods and
    gangs re-indexed and `evicted` mapped through the shift; only the round count may differ."""
    a, j = scale.given_back_case()
    goff, rgang = a[6], a[15]
    g0, g1 = int(goff[j]), int(goff[j + 1])
    kept = gangs.run(tables, scale.with_gang_min(a, j, 1))
    gangs.invariants(scale.with_gang_min(a, j, 1), kept)
    mine = (kept[3] >= g0) & (kept[3] < g1)
    assert g1 - g0 >= 64 and kept[2][j] >= 1 and (mine & (rgang >= 0)).sum() >= 10  # it evicts in jobs when kept
    back = gangs.run(tables, scale.with_gang_min(a, j, g1 - g0))
    without = gangs.run(tables, scale.without_gang(a, j))
    for x, y in zip(scale.given_back_outputs(a, j, back), without[:6]):
        np.testing.assert_array_equal(x, y)
    assert back[6].tolist()[1:] == without[6].tolist()[1:] == [0, 0]
