"""egpu::place_pods, egpu::place_gangs and egpu::place_tables on the GPU past the shared pod phases' block, stage,
tile and grid thresholds: the cases of tests/test_pods_scale_cpu.py against the numpy restatements bit for bit (info
included), and the invariants.

  1. place_pods: a round 2 of more than 2 048 positions deferring in every stage and in a ragged last tile, at
     N_wave x 8 (pods of 1 to 8 containers) and 128 x 64; a one-CTA grid over three rounds; N = 8 with G > 2 048;
  2. place_tables, vector and scalar form, at N_wave with a round 2 of more than 2 048 rows: the torch loop around
     egpu::bestfit_tables, and the restatement of the same rows as pods of one container;
  3. place_gangs: a gang of more than 2 048 pods deferring in round 2, a round whose counts two rounds before sit in
     tiles the round between did not cover, a gang of 600 pods given back after three rounds followed by a gang that
     uses what it gave back; mixed gang sizes and gang_min at N = 257, 1031 and N_wave;
  4. a gang of 2 100 pods given back at N_wave: the call equals the call without that gang;
  5. the known answers of the pod choice word (sum lm >= 2^20 against sum lc, and the maxima).

Each reference is computed once per process and shared with the CPU file's preconditions.
"""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import place_tables_np  # noqa: E402
import test_gpu_place_gangs as gangs  # noqa: E402  (check, invariants of place_gangs)
import test_gpu_place_pods as pods  # noqa: E402  (check, invariants of place_pods)
import test_pods_scale_cpu as scale  # noqa: E402  (the cases and their references)


@pytest.fixture(scope="module")
def tables():
    from elastic_gpu_agent_b200 import tables as t
    t.load()
    return t


@pytest.fixture(scope="module")
def nw():
    """N_wave of this device, assuming 2 CTAs per SM (the kernels' occupancy on sm_90a): 4261 on a 132-SM H100."""
    return scale.n_wave(torch.cuda.get_device_properties(0).multi_processor_count)


# ---- 1. place_pods ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["pods_wave", "pods_d64", "pods_one_cta", "pods_n8_wide"])
def test_place_pods_past_the_thresholds(name, tables, nw):
    op, a, exp, trace = scale.reference(name, nw)
    out = pods.run(tables, *a)
    pods.check(*a, out, exp=exp)
    pods.invariants(*a, out)


# ---- 2. place_tables -------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0, 1])  # 0: the vector form (P % 4 == 0, 16-byte aligned); 1: the scalar form
def test_place_tables_restages_in_later_rounds(offset, tables, nw):
    op, a, exp, trace = scale.reference("tables_wave", nw)
    fc, fm, dv, rc, rm, _ = a
    cu = pods.cuda(fc, fm, dv)
    rq = []
    for x in (rc, rm):  # a contiguous view that starts `offset` elements into its storage
        buf = torch.zeros(x.size + offset, dtype=torch.int32, device="cuda")
        buf[offset:] = torch.from_numpy(x).cuda()
        rq.append(buf[offset:])
    got = [t.cpu().numpy() for t in tables.place_tables(*cu, *rq)]
    e_node, e_dev, e_fc, e_fm, e_rounds = place_tables_np.place_torch(*cu, *rq)
    for x, y in zip(got[:4], (e_node, e_dev, e_fc, e_fm)):
        np.testing.assert_array_equal(x, y.cpu().numpy())
    assert got[4].tolist() == [e_rounds, 0]
    for x, y in zip(got[:4], exp[:4]):  # the rows as pods of one container: the restatement's rounds
        np.testing.assert_array_equal(x, y)
    assert got[4][0] == exp[4][0] == len(trace)


# ---- 3. place_gangs --------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["gangs_sequence", "gangs_257", "gangs_1031", "gangs_wave"])
def test_place_gangs_past_the_thresholds(name, tables, nw):
    op, a, exp, trace = scale.reference(name, nw)
    out = gangs.run(tables, *a)
    gangs.check(a, out, exp=exp)
    gangs.invariants(a, out)


# ---- 4. a gang given back is as if it were not there -----------------------------------------------------------
@pytest.mark.gpu
def test_given_back_gang_is_the_call_without_it(tables, nw):
    """§2.13: a gang given back leaves the tables as they were.  So with gang_min = size the call equals the call
    without the gang, pods and gangs re-indexed; only the round count differs, by the rounds the gang ran.  With
    gang_min = 1 the gang is kept, and the next gang, which fits only on its whole cards, is given back."""
    a, j = scale.given_back_call(nw)
    size = np.diff(a[6])
    back = gangs.run(tables, *a)
    gangs.invariants(a, back)
    assert back[2][j + 1] == size[j + 1]  # it uses the whole cards gang j gave back
    without = gangs.run(tables, *scale.without_gang(a, j))
    for x, y in zip(scale.given_back_outputs(a, j, back), without[:5]):
        np.testing.assert_array_equal(x, y)
    assert back[5][1:].tolist() == without[5][1:].tolist() == [0, 0] and back[5][0] - without[5][0] == 3
    kept = list(a)
    kept[7] = a[7].copy()
    kept[7][j] = 1
    out = gangs.run(tables, *kept)
    gangs.invariants(kept, out)
    assert out[2][j] == 2 * size[j] // 3 and out[2][j + 1] == 0


# ---- 5. the choice word's known answers ------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(scale.KAT)))
def test_choice_word_known_answers(case, tables):
    c = scale.KAT[case]
    node, dev, fco, fmo, info = pods.run(tables, *scale.kat_args(c))
    assert node.tolist() == c["node"] and dev.tolist() == c["dev"], c["name"]
    assert fco.tolist() == c["free_core_out"] and fmo.tolist() == c["free_mem_out"], c["name"]
    assert info.tolist() == [c["rounds"], 0, 0], c["name"]
