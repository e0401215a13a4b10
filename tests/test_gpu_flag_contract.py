"""The argument contract of every entry point that takes rows or batches and flags, over the whole cross product.

`ACCEPTS` restates in plain Python, one function per entry point, which (flags, arrays, R, step, lag, K) each call
accepts; include/egpu_alloc.h is the source of the rules.  The CPU tests hold the restatement to cases listed from
the header.  The GPU tests call each entry point on a context that has no table, with every combination of flag bits
1 ... 512 (1024 sets) and these argument shapes:

  - int32 arrays, packed words with d_req_mem NULL, packed words with a d_req_mem;
  - R = 0 and R = 8;
  - all arrays fine, the request array misaligned, the index array NULL;
  - the exchange step at both edges of every step rule, the lag at both edges of 1 ... 16;
  - K = 1 and K = 2 batches.

A refused call returns EGPU_ERR_INVALID and an accepted one EGPU_ERR_NO_TABLE: every argument check runs before the
context's state is looked at, and with no table nothing is launched or read, so a wrong check cannot touch a buffer.
"""
import ctypes as C
import itertools
from collections import namedtuple

import pytest

F_COMMIT, F_INPUTS_READY, F_PREFIX, F_APPLY, F_PACKED, F_ROUNDS, F_DEVICE_ROUNDS, F_RELEASE = 1, 2, 4, 8, 16, 32, 128, 256
ERR_INVALID, ERR_NO_TABLE = -1, -5
STEP_END = 1 << 47  # exchange steps travel in 47 bits
ALL_FLAGS = range(1024)  # every set of the bits 1 ... 512
FORMATS = ("int32", "packed", "packed_mem")  # packed_mem: packed words and a non-NULL d_req_mem
BAD = (None, "misaligned", "null")  # the request array misaligned, or the index array NULL
STEPS = (0, STEP_END - 4, STEP_END - 3, STEP_END - 2, STEP_END - 1, STEP_END)
LAGS = (0, 1, 16, 17)

Args = namedtuple("Args", "fmt R bad step lag K", defaults=(None, 0, 1, 1))
ROUNDS_NEEDS = F_PACKED | F_PREFIX | F_COMMIT | F_ROUNDS
DEVICE_ROUNDS_NEEDS = F_PREFIX | F_COMMIT | F_ROUNDS | F_DEVICE_ROUNDS


# ---- the restatement ---------------------------------------------------------------------------------------------
def arrays_ok(packed, a, device=True):
    """rows and indices present when R > 0 and, device arrays, 16-byte aligned; packed rows: d_req_mem NULL"""
    rc = "misaligned" if a.bad == "misaligned" else "ok"
    rm = None if a.fmt == "packed" else "ok"
    idx = None if a.bad == "null" else "ok"

    def ok(p):
        return (a.R == 0 or p is not None) and not (device and p == "misaligned")
    return ok(rc) and ok(idx) and (rm is None if packed else ok(rm))


def only(flags, allowed):
    return (flags & ~allowed) == 0


def release_ok(flags):
    return only(flags, F_RELEASE | F_COMMIT | F_PACKED)


def device_rounds_ok(flags):
    return only(flags, DEVICE_ROUNDS_NEEDS | F_PACKED | F_INPUTS_READY) and (flags & DEVICE_ROUNDS_NEEDS) == DEVICE_ROUNDS_NEEDS


def batch_flags_ok(flags):
    """egpu_bestfit_batch[_dev]: release, device rounds and rounds take fixed sets; otherwise every bit is ignored,
    except that EGPU_F_PACKED needs EGPU_F_PREFIX_COMMIT"""
    if flags & F_RELEASE:
        return release_ok(flags)
    if flags & F_DEVICE_ROUNDS:
        return device_rounds_ok(flags)
    if flags & F_ROUNDS:
        return only(flags, ROUNDS_NEEDS | F_INPUTS_READY) and (flags & ROUNDS_NEEDS) == ROUNDS_NEEDS
    return not flags & F_PACKED or bool(flags & F_PREFIX)


def batch_dev(flags, a):
    return batch_flags_ok(flags) and arrays_ok(flags & F_PACKED, a)


def batch_host(flags, a):
    return batch_flags_ok(flags) and arrays_ok(flags & F_PACKED, a, device=False)


def shard_dev(flags, a):
    return only(flags, F_INPUTS_READY | F_PACKED) and a.step < STEP_END and arrays_ok(flags & F_PACKED, a)


def shard_prefix_dev(flags, a):
    if flags & F_RELEASE:
        ok = release_ok(flags)
    elif flags & (F_ROUNDS | F_DEVICE_ROUNDS):  # INPUTS_READY refused, unlike on one GPU; steps step and step + 1
        ok = (flags & ~F_PACKED) == DEVICE_ROUNDS_NEEDS and a.step + 2 <= STEP_END
    else:
        ok = only(flags, F_COMMIT | F_PREFIX | F_PACKED)
    return ok and a.step < STEP_END and arrays_ok(flags & F_PACKED, a)


def shard_lag_dev(flags, a):
    """refuses EGPU_F_COMMIT only; packed takes the flag AND a NULL d_req_mem, else the call is int32"""
    packed = flags & F_PACKED and a.fmt == "packed"
    return not flags & F_COMMIT and 1 <= a.lag <= 16 and a.step < STEP_END and arrays_ok(packed, a)


def batches_dev(flags, a):
    ok = device_rounds_ok(flags) if flags & F_DEVICE_ROUNDS else only(flags, F_INPUTS_READY | F_PACKED)
    return ok and arrays_ok(flags & F_PACKED, a)


def batches_shard_dev(flags, a):
    if flags & F_PREFIX:  # steps first_step ... first_step + 2K - 1
        ok = only(flags, F_PREFIX | F_COMMIT | F_PACKED) and a.step + 2 * a.K <= STEP_END
    else:
        ok = only(flags, F_INPUTS_READY | F_APPLY)
    return ok and a.step < STEP_END and arrays_ok(flags & F_PACKED, a)


def packed_dev(flags, a):
    """refuses no flag (it masks them to COMMIT | INPUTS_READY); the words and int8 indices as device arrays"""
    return arrays_ok(True, a._replace(fmt="packed"))


def packed_host(flags, a):
    return arrays_ok(True, a._replace(fmt="packed"), device=False)


ACCEPTS = {
    "egpu_bestfit_batch": batch_host, "egpu_bestfit_batch_dev": batch_dev, "egpu_bestfit_batch_shard_dev": shard_dev,
    "egpu_bestfit_batch_shard_prefix_dev": shard_prefix_dev, "egpu_bestfit_batch_shard_lag_dev": shard_lag_dev,
    "egpu_bestfit_batches_dev": batches_dev, "egpu_bestfit_batches_shard_dev": batches_shard_dev,
    "egpu_bestfit_batch_packed_dev": packed_dev, "egpu_bestfit_batch_packed": packed_host,
}


def accepted_sets(fn, a):
    return {f for f in ALL_FLAGS if fn(f, a)}


def subsets(*bits):
    return {sum(c) for n in range(len(bits) + 1) for c in itertools.combinations(bits, n)}


# ---- the restatement against the header's text -------------------------------------------------------------------
INT32, PACKED = Args("int32", 8), Args("packed", 8)


def test_release_sets():
    """EGPU_F_RELEASE [| EGPU_F_COMMIT] [| EGPU_F_PACKED], each in its own row format: exactly four sets"""
    got = {f for f in ALL_FLAGS if f & F_RELEASE and batch_dev(f, PACKED if f & F_PACKED else INT32)}
    assert got == {F_RELEASE | s for s in subsets(F_COMMIT, F_PACKED)}
    assert {f for f in ALL_FLAGS if f & F_RELEASE and shard_prefix_dev(f, PACKED if f & F_PACKED else INT32)} == got
    for fn in (shard_dev, batches_dev, batches_shard_dev):
        assert not {f for f in ALL_FLAGS if f & F_RELEASE and fn(f, PACKED if f & F_PACKED else INT32)}
    assert batch_host(F_RELEASE | F_PACKED, PACKED) and not batch_host(F_RELEASE | F_PACKED, Args("packed_mem", 8))


def test_rounds_sets():
    dr = DEVICE_ROUNDS_NEEDS
    got = {f for f in ALL_FLAGS if f & (F_ROUNDS | F_DEVICE_ROUNDS) and batch_dev(f, PACKED if f & F_PACKED else INT32)}
    assert got == {ROUNDS_NEEDS, ROUNDS_NEEDS | F_INPUTS_READY} | {dr | s for s in subsets(F_PACKED, F_INPUTS_READY)}
    assert not batch_dev(ROUNDS_NEEDS | 64, PACKED) and not batch_dev(ROUNDS_NEEDS & ~F_PACKED, INT32)
    # over row shards only the one-launch set, without EGPU_F_INPUTS_READY, and step + 2 <= 2^47
    got = {f for f in ALL_FLAGS if f & (F_ROUNDS | F_DEVICE_ROUNDS) and shard_prefix_dev(f, PACKED if f & F_PACKED else INT32)}
    assert got == {dr, dr | F_PACKED}
    assert shard_prefix_dev(dr, INT32._replace(step=STEP_END - 2)) and not shard_prefix_dev(dr, INT32._replace(step=STEP_END - 1))
    assert shard_prefix_dev(F_PREFIX, INT32._replace(step=STEP_END - 1))
    # K batches: the single-batch rule with R = 0
    assert accepted_sets(batches_dev, INT32) == subsets(F_INPUTS_READY) | {dr, dr | F_INPUTS_READY}
    assert accepted_sets(batches_dev, PACKED) == {F_PACKED, F_PACKED | F_INPUTS_READY, dr | F_PACKED, dr | F_PACKED | F_INPUTS_READY}


def test_snapshot_and_prefix_ignore_other_bits():
    for f in (0, F_COMMIT, F_INPUTS_READY, F_APPLY, 64, 512, F_APPLY | 64 | 512 | F_COMMIT, F_PREFIX | 64):
        assert batch_dev(f, INT32) and batch_host(f, INT32)
    for f in (F_PACKED, F_PACKED | F_COMMIT, F_PACKED | F_INPUTS_READY):  # EGPU_F_PACKED needs EGPU_F_PREFIX_COMMIT
        assert not batch_dev(f, PACKED) and not batch_host(f, PACKED)
    assert batch_dev(F_PACKED | F_PREFIX | F_COMMIT | 512, PACKED)
    assert not batch_dev(F_PACKED | F_PREFIX, Args("packed_mem", 8)) and not batch_dev(F_PREFIX, PACKED)


def test_sharded_sets():
    assert accepted_sets(shard_dev, INT32) == subsets(F_INPUTS_READY)
    assert accepted_sets(shard_dev, PACKED) == {F_PACKED, F_PACKED | F_INPUTS_READY}
    assert not shard_dev(0, INT32._replace(step=STEP_END)) and shard_dev(0, INT32._replace(step=STEP_END - 1))
    assert accepted_sets(shard_prefix_dev, INT32) - {f for f in ALL_FLAGS if f & (F_RELEASE | F_DEVICE_ROUNDS)} == subsets(F_COMMIT, F_PREFIX)
    # the lag call: every set without EGPU_F_COMMIT; EGPU_F_PACKED with two int32 arrays runs as int32
    lag = Args("int32", 8, lag=1)
    assert accepted_sets(shard_lag_dev, lag) == {f for f in ALL_FLAGS if not f & F_COMMIT}
    assert accepted_sets(shard_lag_dev, lag._replace(fmt="packed")) == {f for f in ALL_FLAGS if not f & F_COMMIT and f & F_PACKED}
    assert accepted_sets(shard_lag_dev, lag._replace(fmt="packed_mem")) == accepted_sets(shard_lag_dev, lag)
    assert not accepted_sets(shard_lag_dev, lag._replace(lag=0)) and not accepted_sets(shard_lag_dev, lag._replace(lag=17))
    assert accepted_sets(shard_lag_dev, lag._replace(lag=16)) == accepted_sets(shard_lag_dev, lag)
    # K sharded batches: prefix-commit within {PREFIX, COMMIT, PACKED} and first_step + 2K <= 2^47, else {INPUTS_READY, APPLY}
    assert accepted_sets(batches_shard_dev, INT32) == {F_PREFIX, F_PREFIX | F_COMMIT} | subsets(F_INPUTS_READY, F_APPLY)
    assert accepted_sets(batches_shard_dev, PACKED) == {F_PREFIX | F_PACKED, F_PREFIX | F_COMMIT | F_PACKED}
    k2 = INT32._replace(K=2)
    assert batches_shard_dev(F_PREFIX, k2._replace(step=STEP_END - 4)) and not batches_shard_dev(F_PREFIX, k2._replace(step=STEP_END - 3))
    assert batches_shard_dev(F_APPLY, k2._replace(step=STEP_END - 1)) and not batches_shard_dev(F_APPLY, k2._replace(step=STEP_END))


def test_arrays():
    for fn in (batch_dev, shard_dev, shard_prefix_dev, batches_dev):
        assert not fn(0 if fn is not shard_prefix_dev else F_PREFIX, INT32._replace(bad="misaligned"))
        assert not fn(F_PREFIX if fn in (batch_dev, shard_prefix_dev) else 0, INT32._replace(bad="null"))
        assert fn(F_PREFIX if fn in (batch_dev, shard_prefix_dev) else 0, Args("int32", 0, "null"))
    # host forms: presence only, no alignment rule
    assert batch_host(0, INT32._replace(bad="misaligned")) and not batch_host(0, INT32._replace(bad="null"))
    assert packed_host(0, INT32._replace(bad="misaligned")) and not packed_dev(0, INT32._replace(bad="misaligned"))
    assert accepted_sets(packed_dev, INT32) == set(ALL_FLAGS) and not accepted_sets(packed_dev, INT32._replace(bad="null"))


# ---- the library against the restatement -------------------------------------------------------------------------
def shapes(name):
    """the argument shapes the matrix crosses with every flag set, for one entry point"""
    fmts = ("int32",) if name.startswith("egpu_bestfit_batch_packed") else FORMATS
    if name == "egpu_bestfit_batch_shard_lag_dev":
        edges = [(st, 1) for st in STEPS] + [(0, lag) for lag in LAGS]
    elif "shard" in name:
        edges = [(st, 1) for st in STEPS]
    else:
        edges = [(0, 1)]
    ks = (1, 2) if name.startswith("egpu_bestfit_batches") else (1,)
    for fmt, R, bad, (step, lag), K in itertools.product(fmts, (0, 8), BAD, edges, ks):
        yield Args(fmt, R, bad, step, lag, K)


class Buffers:
    """a device and a host buffer with room for every array of R = 8 at 256-byte offsets"""

    def __init__(self, torch):
        self.dev = torch.zeros(4096, dtype=torch.uint8, device="cuda")
        self.host = (C.c_uint8 * 4096)()

    def arrays(self, a, device):
        base = self.dev.data_ptr() if device else C.addressof(self.host)
        rc = base + (4 if a.bad == "misaligned" else 0)
        rm = None if a.fmt == "packed" else base + 256
        idx = None if a.bad == "null" else base + 512
        return rc, rm, idx, base + 1024, base + 2048  # rows, mem, indices, sums, table'


def call(lib, h, name, flags, a, buf):
    rc, rm, idx, delta, tab = buf.arrays(a, device=name != "egpu_bestfit_batch" and name != "egpu_bestfit_batch_packed")
    fn = getattr(lib, name)
    if name == "egpu_bestfit_batch":
        return fn(h, rc, rm, a.R, idx, delta, delta + 512, flags)
    if name == "egpu_bestfit_batch_packed":
        return fn(h, rc, a.R, idx, delta, delta + 512, flags)
    if name == "egpu_bestfit_batch_packed_dev":
        return fn(h, rc, a.R, idx, delta, tab, flags, None)
    if name == "egpu_bestfit_batch_dev":
        return fn(h, rc, rm, a.R, idx, delta, tab, flags, None)
    if name == "egpu_bestfit_batch_shard_dev":
        return fn(h, rc, rm, a.R, idx, delta, flags, a.step, None)
    if name == "egpu_bestfit_batch_shard_prefix_dev":
        return fn(h, rc, rm, a.R, idx, delta, tab, flags, a.step, None)
    if name == "egpu_bestfit_batch_shard_lag_dev":
        return fn(h, rc, rm, a.R, idx, delta, flags, a.step, a.lag, tab, None)
    from elastic_gpu_agent_b200 import _lib as L
    good = L.Batch(rc - (4 if a.bad == "misaligned" else 0), rm, a.R, idx or buf.dev.data_ptr() + 512, delta, tab)
    batches = (L.Batch * a.K)(*([good] * (a.K - 1) + [L.Batch(rc, rm, a.R, idx, delta, tab)]))  # the last batch has the shape
    if name == "egpu_bestfit_batches_dev":
        return fn(h, batches, a.K, flags, None)
    return fn(h, batches, a.K, flags, a.step, None)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ACCEPTS))
def test_flag_contract(name, alloc):
    """EGPU_ERR_INVALID where the restatement refuses, EGPU_ERR_NO_TABLE where it accepts, for every flag set and shape"""
    import torch
    lib, h = alloc._lib, alloc.handle
    buf = Buffers(torch)
    accepts = ACCEPTS[name]
    n0 = alloc.launch_count
    wrong, n = [], 0
    for a in shapes(name):
        for flags in ALL_FLAGS:
            want = ERR_NO_TABLE if accepts(flags, a) else ERR_INVALID
            got = call(lib, h, name, flags, a, buf)
            n += 1
            if got != want and len(wrong) < 20:
                wrong.append((flags, a, got, want))
    assert not wrong, wrong
    assert n >= 1024 * 6
    torch.cuda.synchronize()
    assert alloc.launch_count == n0 and not buf.dev.any().item()
