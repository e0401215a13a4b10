"""Placement-state restore (include/egpu_restore.h, SURVEY.md §8 row n3).

The stored FORMATS are the reference's (record key/value pkg/types/pod.go:39-58, symlinks
pkg/operator/gpushare.go:31-55) and the identity check is types.NewDevice's hash
(pkg/types/device.go:17-25,49-54): pinned.  The restore RULE is builder-defined (the reference
declares Restore() and never implements it, pkg/manager/manager.go:20): the known answers in
tests/golden/restore_records.json are derived by hand."""
import json
import os

import numpy as np
import pytest

from oracle import restore_py as R
from restore_util import live_placements, persisted_state

HERE = os.path.dirname(os.path.abspath(__file__))
G = json.load(open(os.path.join(HERE, "golden", "restore_records.json")))
RECORDS = [(k.encode(), v.encode()) for k, v in G["records"]]
LINKS = [tuple(l) for l in G["links"]]


def test_marshal_matches_go_json_marshal_layout():
    """json.Marshal(map[string]*Device): keys sorted, fields Hash/List/ResourceName, no spaces,
    List sorted by NewDevice; sha256("0-00:0-01:3-07")[:8] computed independently."""
    k, v = R.marshal_record("default", "pod", {"main": (["0-01", "3-07", "0-00"], R.CORE), "aux": None})
    assert k == b"default/pod"
    assert v == (b'{"aux":null,"main":{"Hash":"e4b78a7c","List":["0-00","0-01","3-07"],'
                 b'"ResourceName":"elasticgpu.io/gpu-core"}}')


@pytest.mark.parametrize("mode", ["verify", "no_verify"])
def test_oracle_known_answers(mode):
    fc, fm, ov, counts, rstat = R.restore(RECORDS, LINKS, G["cap_core"], G["cap_mem"], verify=(mode == "verify"))
    e = G["expect"][mode]
    assert (fc, fm, ov, counts, rstat) == (e["free_core"], e["free_mem"], e["oversub"], e["counts"], e["record_status"])


def test_oracle_rejects_what_newpifromraw_rejects():
    for key, val in G["parse_errors"]:
        with pytest.raises(R.RestoreParseError):
            R.restore([(key.encode(), val.encode())], [], G["cap_core"], G["cap_mem"])


def test_oracle_restore_of_nothing_is_capacity():
    fc, fm, ov, counts, rstat = R.restore([], [], [100, 50], [10, 20])
    assert (fc, fm, ov, counts, rstat) == ([100, 50], [10, 20], [0, 0], [0] * 5, [])


def test_reference_test_record_is_foreign():
    """pkg/storage/storage_test.go:34-38 stores NewDevice({"a","b","c"}) without a resource name."""
    val = b'{"container":{"Hash":"' + R.device_hash(["a", "b", "c"]).encode() + b'","List":["a","b","c"],"ResourceName":""}}'
    fc, fm, ov, counts, rstat = R.restore([(b"default/pod", val)], [], [100], [1000])
    assert counts[R.REC_FOREIGN] == 1 and fc == [100] and rstat == [R.REC_FOREIGN]


# ---------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["verify", "no_verify"])
def test_cuda_known_answers(alloc, mode):
    from elastic_gpu_agent_b200 import restore
    fc, fm, ov, counts, rstat = restore.restore_table(alloc, RECORDS, LINKS, G["cap_core"], G["cap_mem"],
                                                      verify=(mode == "verify"))
    e = G["expect"][mode]
    assert fc.tolist() == e["free_core"] and fm.tolist() == e["free_mem"] and ov.tolist() == e["oversub"]
    assert counts.tolist() == e["counts"] and rstat.tolist() == e["record_status"]


@pytest.mark.gpu
def test_cuda_parse_errors_name_the_record(alloc, egpu):
    from elastic_gpu_agent_b200 import restore
    good = RECORDS[0]
    for key, val in G["parse_errors"]:
        with pytest.raises(egpu.EgpuError) as ei:
            restore.restore_table(alloc, [good, (key.encode(), val.encode())], LINKS, G["cap_core"], G["cap_mem"])
        assert ei.value.code == egpu._lib.ERR_PARSE, str(ei.value)
        assert "record 1" in str(ei.value), str(ei.value)
    # the context is still usable
    fc, *_ = restore.restore_table(alloc, [good], LINKS, G["cap_core"], G["cap_mem"])
    assert fc.tolist() == [100, 75, 100, 100]


@pytest.mark.gpu
def test_cuda_restore_of_nothing_and_install(alloc):
    from elastic_gpu_agent_b200 import restore
    fc, fm, ov, counts, rstat = restore.restore_table(alloc, [], [], [100, 50], [10, 20], install=True)
    assert fc.tolist() == [100, 50] and fm.tolist() == [10, 20] and ov.tolist() == [0, 0] and counts.sum() == 0
    tfc, tfm, _ = alloc.table()
    assert tfc.tolist() == [100, 50] and tfm.tolist() == [10, 20]
    # installed table drives the best-fit scan: (40, 5) fits only GPU 0; (10, 15) only GPU 1
    idx, _, _ = alloc.bestfit(np.array([40, 10], dtype=np.int32), np.array([5, 15], dtype=np.int32))
    assert idx.tolist() == [1, 1]  # (40,5): GPU 1 leaves (10, 15) < GPU 0's (60, 5) in the core-first order


@pytest.mark.gpu
def test_cuda_flat_form_random_vs_oracle(alloc):
    """Random entries through the flat entry point, statuses and table against the oracle."""
    from elastic_gpu_agent_b200 import restore
    rng = np.random.default_rng(7)
    D = 8
    cap_core, cap_mem = [100] * D, [4096] * D
    sets, hashes, resources, links, records, link_rows = [], [], [], [], [], []
    for n in range(300):
        kind = rng.integers(0, 10)
        res = R.CORE if rng.integers(0, 2) == 0 else R.MEM
        count = int(rng.integers(1, 40)) if res == R.CORE else int(rng.integers(1, 600))
        if kind == 0 and res == R.CORE:
            count = int(rng.integers(1, 4)) * 100 + int(rng.integers(0, 50))     # whole cards (+ ignored remainder)
        ids = ["%d-%02d" % (rng.integers(0, D), u) for u in rng.choice(100000, size=count, replace=False)]
        h = R.device_hash(ids)
        need = count // 100 if (res == R.CORE and count > 100) else 1
        gpus = [int(rng.integers(0, D)) for _ in range(need)]
        if kind == 1:
            gpus = gpus[:-1]                       # a link is missing
        if kind == 2:
            h = "%08x" % (int(h, 16) ^ 1)          # stale hash
        if kind == 3:
            gpus[0] = D + 3                        # link outside the table
        sets.append(ids)
        hashes.append(h)
        resources.append(restore.RESOURCE_CORE if res == R.CORE else restore.RESOURCE_MEM)
        links.append(gpus)
        k, v = R.marshal_record("ns", "p%d" % n, {"c": (ids, res)})
        if kind == 2:
            v = v.replace(R.device_hash(ids).encode(), h.encode())
        records.append((k, v))
        link_rows += [("elastic-gpu-%s-%d" % (h, i), "/dev/nvidia%d" % g) for i, g in enumerate(gpus)]
    efc, efm, eov, ecounts, erstat = R.restore(records, link_rows, cap_core, cap_mem)
    fc, fm, ov, status = restore.restore_table_flat(alloc, sets, hashes, resources, links, cap_core, cap_mem)
    assert fc.tolist() == efc and fm.tolist() == efm and ov.tolist() == eov
    assert status.tolist() == erstat
    assert len(set(erstat)) >= 3                   # the case mix really produced several statuses
    # and the raw form agrees with itself
    fc2, fm2, ov2, counts, rstat = restore.restore_table(alloc, records, link_rows, cap_core, cap_mem)
    assert fc2.tolist() == efc and fm2.tolist() == efm and counts.tolist() == ecounts and rstat.tolist() == erstat


@pytest.mark.gpu
@pytest.mark.parametrize("events,mem_cap", [(400, 4096), (3000, 183359)])
def test_cuda_restore_after_churn_equals_live_table(alloc, egpu, events, mem_cap):
    """cfg5-style churn through the sequential replay, then the persisted state of what is still
    placed is restored on a fresh table: it must equal the live table (the 'diff after churn' is
    empty), up to the scale of a 180 GB card (one gpu-memory ID per MiB)."""
    from elastic_gpu_agent_b200 import restore
    D = 8
    kind, a, b = egpu.synth.churn_events(5, events)
    b = np.minimum(b, mem_cap // 4).astype(np.int32)
    cap_core = np.full(D, 100, dtype=np.int32)
    cap_mem = np.full(D, mem_cap, dtype=np.int32)
    alloc.set_table(cap_core, cap_mem)
    out = alloc.replay(kind, a, b)
    live_fc, live_fm, _ = alloc.table()
    placements = live_placements(kind, a, b, out)
    assert placements, "churn left nothing placed"
    records, links = persisted_state(placements, D, mem_cap, seed=events)
    fc, fm, ov, counts, rstat = restore.restore_table(alloc, records, links, cap_core, cap_mem, install=True)
    assert counts[restore.REC_OK] == sum((c > 0) + (m > 0) for _, c, m in placements) and counts[1:].sum() == 0
    assert np.array_equal(fc, live_fc) and np.array_equal(fm, live_fm) and not ov.any()
    tfc, tfm, _ = alloc.table()
    assert np.array_equal(tfc, live_fc) and np.array_equal(tfm, live_fm)
    # oracle agrees
    efc, efm, *_ = R.restore(records, links, cap_core, cap_mem)
    assert fc.tolist() == efc and fm.tolist() == efm
    # drop one symlink (GC removed it, pkg/plugins/base.go:281-300): that entry's capacity comes back
    gone = links[0]
    fc2, fm2, _, counts2, _ = restore.restore_table(alloc, records, links[1:], cap_core, cap_mem)
    assert counts2[restore.REC_NO_LINK] == 1
    assert (fc2.sum() + fm2.sum()) > (fc.sum() + fm.sum()), gone
