"""egpu_preferred_allocation_batch: every container request of a PreferredAllocationRequest in one call,
from flat ID buffers, with the ID work on the GPU.  Every request's (rc, gpu, positions) must equal what
egpu_preferred_allocation answers for that request alone on the same strings.

CPU: the flattening helper's layout and the call-level argument checks (they run before the context
is touched).  GPU: parity on the fake-kubelet batches, full-card and node-scale gpu-memory requests and a
seeded fuzz batch, hand-written precedence anchors, the context's table, and the launch count."""
import ctypes as C
import random

import numpy as np
import pytest

CORE, MEM = 0, 1
OK, INVALID, PARSE, UNSAT = 0, -1, -7, -8
MALFORMED = ["", "a-01", "1-1", "01-05", "1-005", "1-05x", "-05", "1--05", "1-", "1", "1_05", " 1-05"]


def ids(gpu, units):
    return ["%d-%02d" % (gpu, u) for u in units]


# ---- CPU ------------------------------------------------------------------------------------------

def test_flatten_layout_empty_and_multibyte():
    from elastic_gpu_agent_b200 import plugin
    flat, io, so, sz = plugin.flatten_requests([])
    assert flat == b"" and io.tolist() == [0] and so.tolist() == [0] and sz.size == 0
    flat, io, so, sz = plugin.flatten_requests([([], [], 0), (["0-01", "1-02"], [], 3), ([], ["0-01"], -1)])
    assert flat == b"0-011-020-01" and io.tolist() == [0, 4, 8, 12]
    assert so.tolist() == [0, 0, 0, 2, 2, 2, 3] and sz.tolist() == [0, 3, -1]
    assert io.dtype == np.int64 and so.dtype == np.int64 and sz.dtype == np.int32
    # multi-byte characters: offsets count bytes, not characters
    flat, io, so, sz = plugin.flatten_requests([(["0-00", "é-01", "1-€€"], ["2-05"], 2)])
    assert flat == "0-00é-011-€€2-05".encode()
    assert io.tolist() == [0, 4, 9, 17, 21] and so.tolist() == [0, 3, 4]


def call(lib, ctx, resource, flat, io, so, n_ids, n_req, sizes, pos, gpu, rc):
    p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    return lib.egpu_preferred_allocation_batch(ctx, resource, p(flat), p(io), n_ids, p(so), n_req, p(sizes), p(pos), p(gpu), p(rc))


def test_call_level_argument_errors_need_no_device(egpu):
    from elastic_gpu_agent_b200 import plugin
    lib = egpu.load()
    flat, io, so, sz = plugin.flatten_requests([(["0-00", "0-01"], [], 1), (["1-00"], ["1-00"], 1)])
    flat = np.frombuffer(flat, np.uint8)
    pos, gpu, rc = np.zeros(2, np.int32), np.zeros(2, np.int32), np.zeros(2, np.int32)
    assert call(lib, None, CORE, flat, io, so, 3, 2, sz, pos, gpu, rc) == INVALID           # no context
    # the checks below run before the context is touched: a zeroed stand-in handle is never read
    fake = C.create_string_buffer(1 << 16)
    ctx = C.c_void_p(C.addressof(fake))
    assert call(lib, ctx, 2, flat, io, so, 3, 2, sz, pos, gpu, rc) == INVALID               # bad resource
    assert call(lib, ctx, -1, flat, io, so, 3, 2, sz, pos, gpu, rc) == INVALID
    assert call(lib, ctx, CORE, flat, None, so, 3, 2, sz, pos, gpu, rc) == INVALID          # NULL id offsets
    assert call(lib, ctx, CORE, None, io, so, 3, 2, sz, pos, gpu, rc) == INVALID            # NULL bytes, 12 of them
    assert call(lib, ctx, CORE, flat, io, None, 3, 2, sz, pos, gpu, rc) == INVALID          # NULL set offsets
    assert call(lib, ctx, CORE, flat, io, so, 3, 2, None, pos, gpu, rc) == INVALID          # NULL sizes
    assert call(lib, ctx, CORE, flat, io, so, 3, 2, sz, None, gpu, rc) == INVALID           # NULL positions, 2 slots
    assert call(lib, ctx, CORE, flat, io, so, 3, 2, sz, pos, gpu, None) == INVALID          # NULL return codes
    assert call(lib, ctx, CORE, flat, io, so, -1, 2, sz, pos, gpu, rc) == INVALID           # negative counts
    assert call(lib, ctx, CORE, flat, io, so, 3, -1, sz, pos, gpu, rc) == INVALID
    assert call(lib, ctx, CORE, flat, io, so, 1 << 31, 2, sz, pos, gpu, rc) == INVALID      # n_ids >= 2^31
    assert call(lib, ctx, CORE, flat, io, so, 3, 65537, sz, pos, gpu, rc) == INVALID        # too many requests
    bad = so.copy()
    bad[2] = 3
    bad[3] = 2
    assert call(lib, ctx, CORE, flat, io, bad, 3, 2, sz, pos, gpu, rc) == INVALID           # not monotone
    bad = so.copy()
    bad[-1] = 2
    assert call(lib, ctx, CORE, flat, io, bad, 3, 2, sz, pos, gpu, rc) == INVALID           # does not end at n_ids
    bad = so + 1
    bad[-1] = 3
    assert call(lib, ctx, CORE, flat, io, bad, 3, 2, sz, pos, gpu, rc) == INVALID           # does not start at 0
    neg = io.copy()
    neg[-1] = -4
    assert call(lib, ctx, CORE, flat, neg, so, 3, 2, sz, pos, gpu, rc) == INVALID           # negative buffer length
    z = np.zeros(1, np.int64)
    assert call(lib, ctx, CORE, None, None, z, 0, 0, None, None, None, None) == OK          # nothing asked
    assert call(lib, ctx, CORE, None, None, z, 0, 0, None, None, None, None) == OK
    assert call(lib, ctx, CORE, None, io, z, 3, 0, None, None, None, None) == INVALID       # IDs of no request


# ---- GPU: the reference is egpu_preferred_allocation, one call per request -----------------------

def reference(lib, alloc, available, must, size, resource):
    """(rc, gpu, positions) of egpu_preferred_allocation; IDs as bytes, None = an ID the batch sees as
    malformed (its offsets decrease or leave the buffer)"""
    enc = lambda s: b"x" if s is None else s  # noqa: E731
    av = (C.c_char_p * max(1, len(available)))(*[enc(s) for s in available])
    mu = (C.c_char_p * max(1, len(must)))(*[enc(s) for s in must])
    out = np.full(max(1, size), -1, np.int32)
    gpu = C.c_int32(-1)
    rc = lib.egpu_preferred_allocation(alloc.handle, av, len(available), mu, len(must), int(size), int(resource),
                                       C.c_void_p(out.ctypes.data), C.byref(gpu))
    return rc, gpu.value, out[:max(size, 0)].tolist()


def check_batch(lib, alloc, requests, resource, flat=None, io=None):
    """runs the batch (optionally on given flat bytes / offsets) and compares every request with the reference"""
    from elastic_gpu_agent_b200 import plugin
    f, o, so, sz = plugin.flatten_requests(requests)
    if flat is None:
        flat, io = f, o
        seen = [s.encode() for a, m, _ in requests for s in list(a) + list(m)]
    else:
        # what the device sees for every ID: its bytes, or None when its offsets are not a range of the buffer
        seen = []
        for j in range(len(io) - 1):
            b, e = int(io[j]), int(io[j + 1])
            seen.append(flat[b:e] if 0 <= b <= e <= len(flat) else None)
    pos, gpu, rc = plugin.preferred_allocation_batch_flat(alloc, resource, flat, io, so, sz)
    off, k = 0, 0
    codes = []
    for q, (a, m, n) in enumerate(requests):
        av, mu = seen[k:k + len(a)], seen[k + len(a):k + len(a) + len(m)]
        k += len(a) + len(m)
        e_rc, e_gpu, e_pos = reference(lib, alloc, av, mu, n, resource)
        got = pos[off:off + max(n, 0)].tolist()
        assert rc[q] == e_rc, (q, n, rc[q], e_rc)
        if e_rc == OK:
            assert gpu[q] == e_gpu and got == e_pos, (q, n)
        else:
            assert gpu[q] == -1 and got == [-1] * max(n, 0), (q, n)
        off += max(n, 0)
        codes.append(e_rc)
    return codes


def kubelet_batches():
    available = ids(0, range(40, 100)) + ids(2, range(75, 100))[::-1] + ids(1, range(0, 30))
    six = [(available, must, size) for size, must in ((25, []), (26, []), (31, []), (20, ["0-55", "0-41"]), (61, []), (10, []))]
    whole = ids(0, range(100)) + ids(1, range(60)) + ids(3, range(100))[::-1] + ids(2, range(100))
    seven = [(whole, must, size) for size, must in
             [(200, []), (300, []), (400, []), (250, []), (200, ["2-05"]), (200, ["3-99", "0-00"]), (200, ["1-07"])]]
    return six, seven


@pytest.mark.gpu
def test_kubelet_conversation_batches(alloc, egpu):
    lib = egpu.load()
    six, seven = kubelet_batches()
    assert check_batch(lib, alloc, six, CORE) == [OK, OK, OK, OK, UNSAT, OK]
    codes = check_batch(lib, alloc, seven, CORE)
    assert codes[0] == OK and codes[2] == UNSAT and codes[3] == UNSAT and codes[6] == UNSAT
    from elastic_gpu_agent_b200 import plugin
    got = plugin.preferred_allocation_batch(alloc, six, plugin.RESOURCE_CORE)
    assert got[0] == (ids(2, range(75, 100)), 2, OK) and got[4] == (None, -1, UNSAT)


@pytest.mark.gpu
def test_memory_full_card_two_gpus(alloc, egpu):
    available = ids(0, range(100_000, 183_359)) + ids(1, range(0, 183_359))
    assert check_batch(egpu.load(), alloc, [(available, [], 16_384), (available, [], 90_000)], MEM) == [OK, OK]


@pytest.mark.gpu
def test_memory_node_of_eight_full_cards(alloc, egpu):
    """the gpu-memory plugin of a node of eight 183 359 MiB cards: 1 466 872 IDs per request"""
    node = [s for g in range(8) for s in ids(g, range(183_359))]
    reqs = [(node, [], 16_384), (node, ["5-17", "5-100000"], 50_000), (node, [], 183_359), (node, [], 183_360),
            (node, [], 270_000)]
    assert check_batch(egpu.load(), alloc, reqs, MEM) == [OK, OK, OK, UNSAT, UNSAT]


def fuzz_requests(rng, resource, n_req):
    reqs = []
    for _ in range(n_req):
        D = rng.choice([1, 2, 3, 8, 17, 33, 64])
        av = []
        for g in rng.sample(range(D), rng.randint(1, min(D, 6))) + ([D - 1] if rng.random() < 0.5 else []):
            if resource == CORE:
                units = rng.sample(range(0, 130), rng.randint(1, 110))
            else:
                lo = rng.randint(0, 300)
                units = list(range(lo, lo + rng.randint(1, 1500)))
            av += ids(g, units)
        if rng.random() < 0.3:                                     # duplicated IDs
            av += rng.sample(av, min(len(av), rng.randint(1, 20)))
        if rng.random() < 0.1:                                     # 15-digit units: 17-byte IDs that parse
            av += ["%d-%d" % (rng.randrange(D), 10 ** 14 + rng.randrange(10 ** 14)) for _ in range(3)]
        rng.shuffle(av)
        roll = rng.random()
        if roll < 0.08:
            av.insert(rng.randrange(len(av) + 1), rng.choice(MALFORMED))
        elif roll < 0.12:                                          # 17-26-byte IDs that do not parse, or GPUs >= 64
            av.insert(rng.randrange(len(av) + 1), rng.choice(["1234567890-00", "1-" + "1" * 16, "7-" + "9" * 24,
                                                              "123456789-123456789012345"]))
        elif roll < 0.16:
            av.insert(rng.randrange(len(av) + 1), "%d-%02d" % (rng.randint(64, 70), rng.randrange(100)))
        if rng.random() < 0.05:
            av = []
        must = []
        roll = rng.random()
        valid = [s for s in av if s not in MALFORMED and len(s) < 17 and int(s.split("-")[0]) < 64]
        if valid and roll < 0.35:
            g = int(rng.choice(valid).split("-")[0])
            same = [s for s in valid if s.startswith("%d-" % g)]
            must = rng.sample(same, min(len(same), rng.randint(1, 4)))
            if rng.random() < 0.3:
                must += [must[0]]                                  # listed twice
        elif valid and roll < 0.45:
            must = rng.sample(valid, min(len(valid), rng.randint(2, 4)))  # spanning GPUs
        elif roll < 0.5:
            must = [rng.choice(MALFORMED)] + (rng.sample(valid, 1) if valid else [])
        elif roll < 0.55:
            must = ["%d-%02d" % (rng.randrange(64), 5000 + rng.randrange(100))]  # not available
        rng.shuffle(must)
        n_av = len(av)
        sizes = [0, -1, -rng.randint(2, 1000), rng.randint(1, 100), n_av + rng.randint(1, 50), len(must) - 1,
                 rng.randint(1, max(1, n_av))]
        if resource == CORE:
            sizes += [100 * rng.randint(2, 5), 100 * rng.randint(1, 4) + rng.randint(1, 99)]
        reqs.append((av, must, rng.choice(sizes)))
    return reqs


@pytest.mark.gpu
@pytest.mark.parametrize("resource", [CORE, MEM])
def test_fuzz_batch_matches_per_request_calls(alloc, egpu, resource):
    rng = random.Random(20261015 + resource)
    reqs = fuzz_requests(rng, resource, 300)
    codes = check_batch(egpu.load(), alloc, reqs, resource)
    assert {OK, UNSAT, PARSE, INVALID} <= set(codes), sorted(set(codes))
    # whole-card requests on a core node with full cards: pins, multiples and non-multiples
    if resource == CORE:
        node = [s for g in range(6) for s in ids(g, range(100))] + ids(6, range(70))
        wreqs = [(node, rng.sample(node, rng.randint(0, 3)), rng.choice([100, 200, 300, 600, 700, 250, 0, 50]))
                 for _ in range(64)]
        assert OK in check_batch(egpu.load(), alloc, wreqs, CORE)


@pytest.mark.gpu
def test_offsets_that_decrease_or_leave_the_buffer_are_malformed_ids(alloc, egpu):
    from elastic_gpu_agent_b200 import plugin
    rng = random.Random(7)
    reqs = [(ids(0, range(40)) + ids(1, range(30)), [], 20), (ids(2, range(50)), ["2-07"], 5), (ids(3, range(10)), [], 3),
            (ids(0, range(60)), ["0-01", "0-02"], 10), (ids(5, range(100)), [], 1)]
    flat, io, _, _ = plugin.flatten_requests(reqs)
    io = io.copy()
    io[5] = io[4] - 3                 # request 0: ID 4 decreasing, ID 5 swallows its bytes
    io[73] = len(flat) + 100          # request 1: an available ID leaves the buffer
    io[121] = io[121] + 2             # request 1's must-include ID: two IDs merge/shift
    io[130] = -8                      # request 2: negative start
    for _ in range(3):                # request 4 (IDs 193 ..): decreasing
        j = rng.randrange(195, 260)
        io[j] = io[j - 1] - 1
    codes = check_batch(egpu.load(), alloc, reqs, MEM, flat=flat, io=io)
    assert PARSE in codes and OK in codes


@pytest.mark.gpu
def test_precedence_anchors(alloc, egpu):
    from elastic_gpu_agent_b200 import plugin
    av = ids(0, range(10))
    reqs = [(av[:3] + ["zz"] + av[3:], ids(0, range(3)), 2),     # malformed available ID, n_must > size: UNSAT
            (av[:3] + ["64-00", "zz"] + av[3:], [], 1),          # GPU 64 before a malformed ID: INVALID
            (av[:3] + ["zz", "64-00"] + av[3:], [], 1),          # the reverse: PARSE
            ([], [], 0),                                         # nothing available, nothing asked: OK
            ([], [], 1),
            (av, [], -1),
            (av, ["0-05", "1-00"], 2),                           # not available before malformed: UNSAT
            (av, ["0-05", "zz", "1-00"], 3),                     # malformed first: PARSE
            (av + ids(1, range(5)), ["0-05", "1-00", "zz"], 3),  # spans two GPUs before the malformed one: UNSAT
            (av, ["0-05", "0-05"], 2)]                           # listed twice: given once, then the lowest unit
    got = plugin.preferred_allocation_batch(alloc, reqs, plugin.RESOURCE_CORE)
    assert [g[2] for g in got] == [UNSAT, INVALID, PARSE, OK, UNSAT, INVALID, UNSAT, PARSE, UNSAT, OK]
    assert got[3] == ([], -1, OK) and got[9] == (["0-05", "0-00"], 0, OK)
    check_batch(egpu.load(), alloc, reqs, CORE)


@pytest.mark.gpu
def test_context_table_is_left_alone(alloc, egpu):
    alloc.set_table([100, 40, 75], [183359, 9000, 50000])
    six, seven = kubelet_batches()
    check_batch(egpu.load(), alloc, six + seven, CORE)
    fc, fm, ov = alloc.table()
    assert fc.tolist() == [100, 40, 75] and fm.tolist() == [183359, 9000, 50000] and not ov.any()


@pytest.mark.gpu
def test_launch_count_does_not_depend_on_the_number_of_requests(alloc, egpu):
    from elastic_gpu_agent_b200 import plugin
    six, _ = kubelet_batches()
    deltas = []
    for reqs in ([six[0]], (six * 11)[:64]):
        before = alloc.launch_count
        plugin.preferred_allocation_batch(alloc, reqs, plugin.RESOURCE_CORE)
        deltas.append(alloc.launch_count - before)
    assert deltas[0] == deltas[1] and deltas[0] > 0
