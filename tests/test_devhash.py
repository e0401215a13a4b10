"""Device-set identity (types.NewDevice/hash/Equals, pkg/types/device.go:17-54): parity is
PINNED here — the reference defines this computation.  Golden vectors come from the
reference's formula restated with Python sorted()+hashlib
(tests/golden/make_device_hash_vectors.py); the C oracle and the CUDA path must both match."""
import hashlib
import json
import os
import random

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
G = json.load(open(os.path.join(HERE, "golden", "device_hash.json")))


def ids_of(case):
    if "ids" in case:
        return case["ids"]
    r = case["recipe"]
    units = range(r["count"]) if r["seed"] is None else random.Random(r["seed"]).sample(range(183359), r["count"])
    return ["%d-%02d" % (r["gpu"], j) for j in units]


@pytest.mark.parametrize("f", G["fips180_4"], ids=lambda f: f"len{len(f['msg'])}")
def test_oracle_sha256_fips_vectors(f, oracle_c):
    assert oracle_c.sha256(f["msg"].encode()).hex() == f["sha256"]


def test_oracle_sha256_vs_hashlib_all_lengths(oracle_c):
    rng = random.Random(1)
    for n in list(range(0, 200)) + [1000, 4096, 65537]:
        data = bytes(rng.getrandbits(8) for _ in range(n))
        assert oracle_c.sha256(data) == hashlib.sha256(data).digest(), n


@pytest.mark.parametrize("case", G["cases"], ids=lambda c: c["name"])
def test_oracle_device_hash_golden(case, oracle_c):
    assert oracle_c.device_hash(ids_of(case)) == case["hash"]


@pytest.mark.gpu
def test_cuda_device_hash_golden_batch(alloc, egpu):
    """All golden lists in ONE batch call: hashes and full digests."""
    from elastic_gpu_agent_b200 import devhash
    sets = [ids_of(c) for c in G["cases"]]
    hashes, digests = devhash.device_hashes(alloc, sets, want_digest=True)
    for c, h, d in zip(G["cases"], hashes, digests):
        assert h == c["hash"], c["name"]
        assert d.hex() == c["sha256"], c["name"]


@pytest.mark.gpu
def test_cuda_device_hash_single_call_and_oracle(alloc, egpu, oracle_c):
    from elastic_gpu_agent_b200 import devhash
    for c in G["cases"][:10]:
        ids = ids_of(c)
        assert devhash.device_hash(alloc, ids) == c["hash"] == oracle_c.device_hash(ids)


@pytest.mark.gpu
def test_cuda_device_hash_message_length_sweep(alloc, egpu):
    """Joined-string lengths around the SHA-256 block and padding boundaries (55, 56, 63, 64,
    119, 120 ...): sets of k four-character IDs give length 5k - 1."""
    from elastic_gpu_agent_b200 import devhash
    rng = random.Random(3)
    sets = []
    for k in range(0, 60):
        sets.append(["%d-%02d" % (rng.randrange(8), rng.randrange(100)) for _ in range(k)])
    for k in (1, 2, 3, 11, 12, 13):  # mixed lengths -> other residues
        sets.append(["%d-%02d" % (rng.randrange(8), rng.randrange(183359)) for _ in range(k)])
    got, dig = devhash.device_hashes(alloc, sets, want_digest=True)
    for ids, h, d in zip(sets, got, dig):
        ref = hashlib.sha256(":".join(sorted(ids)).encode()).hexdigest()
        assert d.hex() == ref and h == ref[:8], (len(ids), len(":".join(ids)))


@pytest.mark.gpu
def test_cuda_long_messages_block_count_sweep(alloc, egpu):
    """The one-CTA-per-message SHA-256 (few long sets): list lengths whose padded messages span one to
    sixty-odd groups of 32 blocks (its schedule ring), group counts odd and even, and
    node-scale sizes; full 256-bit digests against hashlib."""
    import random
    from elastic_gpu_agent_b200 import devhash
    rng = random.Random(17)
    sets = []
    for n_ids in [256, 257, 300, 330, 340, 341, 342, 343, 350, 680, 700, 701, 702, 703, 704, 710, 1030, 4096, 16384]:
        sets.append(["%d-%02d" % (rng.randrange(8), j) for j in rng.sample(range(183359), n_ids)])
    assert sum(len(x) for x in sets) // len(sets) >= 256      # the long-message kernel is the one that runs
    got, dig = devhash.device_hashes(alloc, sets, want_digest=True)
    blocks = set()
    for i, ids in enumerate(sets):
        msg = ":".join(sorted(ids)).encode()
        blocks.add((len(msg) + 8) // 64 + 1)
        ref = hashlib.sha256(msg).hexdigest()
        assert (dig[i].hex() if isinstance(dig[i], (bytes, bytearray)) else dig[i]) == ref, (i, len(ids))
        assert got[i] == ref[:8]
    assert {34, 46} <= blocks and max(blocks) > 2048, sorted(blocks)   # spans 1, 2 and 60+ groups of 32 blocks


@pytest.mark.gpu
def test_cuda_many_sets_node_scale(alloc, egpu):
    """A node's worth of candidates: 96 containers x 4096..16384 memory IDs across 8 GPUs."""
    from elastic_gpu_agent_b200 import devhash
    rng = random.Random(11)
    sets = []
    for c in range(96):
        g = c % 8
        n = rng.choice([4096, 8192, 16384])
        sets.append(["%d-%02d" % (g, j) for j in rng.sample(range(183359), n)])
    got = devhash.device_hashes(alloc, sets)
    for ids, h in zip(sets, got):
        assert h == hashlib.sha256(":".join(sorted(ids)).encode()).hexdigest()[:8]


@pytest.mark.gpu
def test_cuda_locate_matches_reference_semantics(alloc, egpu):
    """Locate returns the FIRST candidate whose sorted list equals the request's
    (pkg/kube/locator.go:62-90 walks pods/containers in order and returns on the first
    Equals)."""
    from elastic_gpu_agent_b200 import devhash
    rng = random.Random(5)
    req = ["%d-%02d" % (2, j) for j in rng.sample(range(183359), 2048)]
    same_shuffled = rng.sample(req, len(req))
    other_same_size = ["%d-%02d" % (2, j) for j in rng.sample(range(183359), 2048)]
    one_off = sorted(req)[:-1] + ["2-183358" if "2-183358" not in req else "2-183357"]
    shorter = req[:-1]
    cands = [other_same_size, shorter, one_off, same_shuffled, list(req), []]
    assert devhash.locate(alloc, req, cands) == 3
    assert devhash.locate(alloc, req, cands[:3]) == -1
    assert devhash.locate(alloc, req, []) == -1
    assert devhash.locate(alloc, [], [["1-01"], []]) == 1
    assert devhash.locate(alloc, ["0-05", "0-05"], [["0-05"], ["0-05", "0-05"]]) == 1   # multiset, not set


@pytest.mark.gpu
@pytest.mark.parametrize("bad", [["x-01"], ["0-01", ""], ["0-01", "12345678901234567"], ["0:01"]])
def test_cuda_rejects_foreign_ids(bad, alloc, egpu):
    from elastic_gpu_agent_b200 import devhash
    with pytest.raises(egpu.EgpuError) as ei:
        devhash.device_hashes(alloc, [bad])
    assert ei.value.code == -7


@pytest.mark.gpu
def test_cuda_empty_sets_between_full_ones_and_bad_offsets(alloc, egpu):
    """The set index of every ID comes from a binary search in the set offsets on the device: empty sets
    (equal offsets) at the start, in the middle, doubled and at the end must not shift their neighbours.
    Offsets that run backwards or past the byte buffer are a parse error, not a wild read."""
    import hashlib
    import random
    from elastic_gpu_agent_b200 import devhash
    rng = random.Random(5)
    sets = [[], ["3-07", "3-01"], [], [], ["0-%02d" % j for j in rng.sample(range(5000), 700)], ["12-345"], [], []]
    exp = [hashlib.sha256(":".join(sorted(x)).encode()).hexdigest()[:8] for x in sets]
    assert devhash.device_hashes(alloc, sets) == exp
    assert devhash.locate(alloc, ["3-01", "3-07"], sets) == 1
    assert devhash.locate(alloc, [], sets) == 0
    flat, id_off, set_off = devhash.flatten([["0-01", "0-02", "0-03"]])
    for bad in ([0, 4, 2, 12], [0, 4, 20, 12], [0, -4, 8, 12]):
        off = np.array(bad, dtype=np.int64)
        with pytest.raises(egpu.EgpuError) as ei:
            devhash.device_hashes_flat(alloc, flat, off, set_off)
        assert ei.value.code in (-7, -1), bad
    assert devhash.device_hashes_flat(alloc, flat, id_off, set_off) == [hashlib.sha256(b"0-01:0-02:0-03").hexdigest()[:8]]


@pytest.mark.gpu
def test_cuda_sets_larger_than_shared_memory_take_the_radix_path(alloc, egpu):
    """Sets of up to 16 384 IDs are sorted by one CTA each in shared memory; a batch with a larger set goes
    through the global (set, key) radix sort.  Both must give the reference's hashes, and Locate must agree."""
    import hashlib
    import random
    from elastic_gpu_agent_b200 import devhash
    rng = random.Random(17)
    big = ["%d-%02d" % (rng.randrange(8), j) for j in rng.sample(range(183359), 20_000)]
    small = [["5-07", "5-03", "12-00"], [], ["0-%02d" % j for j in rng.sample(range(9000), 4097)], ["3-100000"]]
    for sets in (small, [big] + small, small + [big[:16_385]], small + [big[:16_384]]):
        exp = [hashlib.sha256(":".join(sorted(x)).encode()).hexdigest()[:8] for x in sets]
        assert devhash.device_hashes(alloc, sets) == exp
        req = list(sets[-1])
        rng.shuffle(req)
        assert devhash.locate(alloc, req, sets) == len(sets) - 1
