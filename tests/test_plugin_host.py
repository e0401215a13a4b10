"""Host logic around the path: device-ID codec (pkg/plugins/gpushare.go:28,163) and
GetPreferredAllocation (pkg/plugins/base.go:94-96 is an empty stub in the reference; the
expected answers below follow the builder-defined best-fit spec, DESIGN.md §2)."""
import pytest


def test_id_codec_matches_reference_format(egpu):
    from elastic_gpu_agent_b200 import plugin
    # fmt.Sprintf("%d-%02d", i, j): pkg/plugins/gpushare.go:28 (core), :163 (memory)
    for gpu, unit in [(0, 0), (3, 7), (7, 99), (0, 100), (7, 183358), (63, 5), (12, 10)]:
        s = plugin.format_device_id(gpu, unit)
        assert s == "%d-%02d" % (gpu, unit)
        assert plugin.parse_device_id(s) == (gpu, unit)


@pytest.mark.parametrize("bad", ["", "a-01", "1-1", "01-05", "1-005", "1-05x", "-05", "1--05", "1-", "1", "1_05", " 1-05"])
def test_id_parse_rejects_malformed(bad, egpu):
    from elastic_gpu_agent_b200 import plugin
    with pytest.raises(egpu.EgpuError) as ei:
        plugin.parse_device_id(bad)
    assert ei.value.code == -7


def test_preferred_allocation_needs_a_context(egpu):
    import ctypes as C
    lib = egpu.load()
    arr = (C.c_char_p * 1)(b"0-00")
    assert lib.egpu_preferred_allocation(None, arr, 1, None, 0, 1, 0, None, None) == -1


def core_ids(gpu, units):
    return ["%d-%02d" % (gpu, u) for u in units]


@pytest.mark.gpu
def test_preferred_allocation_best_fit_and_must_include(alloc, egpu):
    from elastic_gpu_agent_b200 import plugin
    # GPU 0 has 60 free core units, GPU 1 has 30, GPU 2 has 25 (units deliberately shuffled)
    available = core_ids(0, range(40, 100)) + core_ids(2, range(75, 100))[::-1] + core_ids(1, range(0, 30))
    ids, gpu = plugin.preferred_allocation(alloc, available, [], 25, plugin.RESOURCE_CORE)
    assert gpu == 2 and ids == core_ids(2, range(75, 100))          # exact fit on GPU 2, ascending units
    ids, gpu = plugin.preferred_allocation(alloc, available, [], 26, plugin.RESOURCE_CORE)
    assert gpu == 1 and ids == core_ids(1, range(0, 26))            # 2 is too small now; 1 leaves 4, 0 leaves 34
    ids, gpu = plugin.preferred_allocation(alloc, available, [], 31, plugin.RESOURCE_CORE)
    assert gpu == 0 and ids == core_ids(0, range(40, 71))
    with pytest.raises(egpu.EgpuError) as ei:
        plugin.preferred_allocation(alloc, available, [], 61, plugin.RESOURCE_CORE)
    assert ei.value.code == -8
    # must-include pins the GPU even when another one fits tighter
    ids, gpu = plugin.preferred_allocation(alloc, available, ["0-55", "0-41"], 25, plugin.RESOURCE_CORE)
    assert gpu == 0 and ids[:2] == ["0-55", "0-41"] and ids[2:] == [i for i in core_ids(0, range(40, 100)) if i not in ("0-55", "0-41")][:23]
    with pytest.raises(egpu.EgpuError) as ei:                       # must-include spans two GPUs
        plugin.preferred_allocation(alloc, available, ["0-55", "1-03"], 25, plugin.RESOURCE_CORE)
    assert ei.value.code == -8
    with pytest.raises(egpu.EgpuError) as ei:                       # pinned GPU is too small
        plugin.preferred_allocation(alloc, available, ["2-80"], 26, plugin.RESOURCE_CORE)
    assert ei.value.code == -8
    with pytest.raises(egpu.EgpuError) as ei:
        plugin.preferred_allocation(alloc, available + ["zz"], [], 1, plugin.RESOURCE_CORE)
    assert ei.value.code == -7


@pytest.mark.gpu
def test_preferred_allocation_memory_resource_at_full_card_scale(alloc, egpu):
    """gpu-memory advertises one ID per MiB (pkg/plugins/gpushare.go:159-168): a 180 GB card
    contributes 183359 IDs (an H100 80GB 81559).  Two GPUs, one half full."""
    from elastic_gpu_agent_b200 import plugin
    available = ["%d-%02d" % (0, u) for u in range(100_000, 183_359)] + ["%d-%02d" % (1, u) for u in range(0, 183_359)]
    ids, gpu = plugin.preferred_allocation(alloc, available, [], 16_384, plugin.RESOURCE_MEM)
    assert gpu == 0 and ids[0] == "0-100000" and ids[-1] == "0-116383" and len(ids) == 16_384
    ids, gpu = plugin.preferred_allocation(alloc, available, [], 90_000, plugin.RESOURCE_MEM)
    assert gpu == 1 and ids[0] == "1-00" and len(ids) == 90_000
