"""CPU tests (no GPU) of the release rule's two restatements (DESIGN.md 2.8): the scalar C loop of
tests/release_oracle.c and the numpy form of tests/release_np.py, against the hand-derived known answers of
tests/golden/release_kat.json and against each other on seeded inputs."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import release_np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "release_oracle.c")
SO = os.path.join(HERE, "_build", "release_oracle.so")  # test artefact, not a product library
KATS = json.load(open(os.path.join(HERE, "golden", "release_kat.json")))["cases"]


@pytest.fixture(scope="module")
def release_c():
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    r = subprocess.run(["/usr/bin/gcc", "-O2", "-fPIC", "-shared", "-std=c11", "-Wall", "-Wextra", "-Werror", "-o", SO, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = C.CDLL(SO)
    vp = C.c_void_p
    lib.oracle_release.restype = C.c_int
    lib.oracle_release.argtypes = [vp, vp, vp, C.c_int32, vp, vp, vp, C.c_int64, vp, vp]

    def release(free_core, free_mem, oversub, core, mem, idx):
        a = [np.ascontiguousarray(x, dtype=np.int32) for x in (free_core, free_mem, oversub, core, mem, idx)]
        D, R = a[0].size, a[3].size
        u = np.full(2 * D, -1, dtype=np.int64)
        tab = np.full(3 * D, -1, dtype=np.int32)
        p = [C.c_void_p(x.ctypes.data) for x in a]
        rc = lib.oracle_release(p[0], p[1], p[2], D, p[3], p[4], p[5], R, C.c_void_p(u.ctypes.data), C.c_void_p(tab.ctypes.data))
        assert rc in (0, 1)
        return u, tab, bool(rc)
    return release


def check_kat(release, k):
    u, tab, ok = release(k["free_core"], k["free_mem"], k["oversub"], k["core"], k["mem"], k["idx"])
    assert u.tolist() == k["u_core"] + k["u_mem"], k["name"]
    assert tab.tolist() == k["table_out"], k["name"]
    assert ok == k["accepted"], k["name"]


def test_kat_file_covers_what_the_rule_names():
    names = {k["name"] for k in KATS}
    assert {"cfg1_release_all", "double_release", "flagged_touched", "flagged_untouched", "empty", "d64", "skip_idx_minus1",
            "skip_idx_deferred", "skip_idx_eq_D", "skip_core_101", "skip_mem_2pow18", "skip_core_negative",
            "skip_mem_negative"} <= names
    for k in KATS:
        D = len(k["free_core"])
        assert len(k["table_out"]) == 3 * D and len(k["u_core"]) == len(k["u_mem"]) == D
        assert k["accepted"] == (not any(k["table_out"][2 * D:]))


@pytest.mark.parametrize("k", KATS, ids=[k["name"] for k in KATS])
def test_numpy_oracle_matches_known_answers(k):
    check_kat(release_np.release, k)


@pytest.mark.parametrize("k", KATS, ids=[k["name"] for k in KATS])
def test_c_oracle_matches_known_answers(release_c, k):
    check_kat(release_c, k)


def seeded_case(seed, D, R, p_junk=0.1):
    """Rows of which most fit under a table with head-room; a share of junk rows of every skipped kind."""
    g = np.random.default_rng(seed)
    core = g.integers(0, 4, R).astype(np.int32)
    mem = g.integers(0, 40, R).astype(np.int32)
    idx = g.integers(0, D, R).astype(np.int32)
    junk = g.random(R) < p_junk
    kind = g.integers(0, 6, R)
    idx = np.where(junk & (kind == 0), -1, idx)
    idx = np.where(junk & (kind == 1), -2, idx)
    idx = np.where(junk & (kind == 2), D + g.integers(0, 100, R), idx).astype(np.int32)
    core = np.where(junk & (kind == 3), 101 + g.integers(0, 27, R), core)
    core = np.where(junk & (kind == 4), -1 - g.integers(0, 5, R), core).astype(np.int32)
    mem = np.where(junk & (kind == 5), (1 << 18) + g.integers(0, 9, R), mem).astype(np.int32)
    return core, mem, idx


@pytest.mark.parametrize("seed", range(12))
def test_oracles_agree_on_seeded_inputs(release_c, seed):
    g = np.random.default_rng(1000 + seed)
    D = [1, 8, 16, 17, 32, 64][seed % 6]
    R = int(g.integers(0, 400))
    core, mem, idx = seeded_case(seed, D, R)
    fc = g.integers(0, 101, D).astype(np.int32)
    fm = g.integers(0, 1 << 18, D).astype(np.int32)
    ov = (g.random(D) < 0.1).astype(np.int32)
    if seed % 2:  # half the cases with head-room, so that acceptance is exercised as well
        fc, fm, ov = np.zeros(D, np.int32), np.zeros(D, np.int32), np.zeros(D, np.int32)
    a, b = release_c(fc, fm, ov, core, mem, idx), release_np.release(fc, fm, ov, core, mem, idx)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]


def test_unpack_is_the_packed_decode():
    w = np.array([(25 << 18) | 1024, (100 << 18) | 262143, (101 << 18) | 5, 1 << 25, 0xFFFFFFFF, 0], dtype=np.uint32)
    c, m = release_np.unpack(w)
    assert c.tolist() == [25, 100, 101, 127, 127, 0] and m.tolist() == [1024, 262143, 5, 0, 0, 0]
