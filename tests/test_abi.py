"""CPU tests (no GPU): the C-ABI library loads, exports every symbol the headers
declare, and fails loudly — not with a CPU fallback — when there is no device."""
import ctypes as C
import glob
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    names = []
    for h in sorted(glob.glob(os.path.join(ROOT, "include", "*.h"))):
        src = open(h).read()
        src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
        names += re.findall(r"\b(egpu_[a-z0-9_]+)\s*\(", src)
    return sorted(set(names))


def test_headers_declare_something():
    syms = declared_symbols()
    assert "egpu_bestfit_batch" in syms and "egpu_ctx_create" in syms and len(syms) >= 15


def test_library_exports_every_declared_symbol(egpu):
    lib = C.CDLL(egpu.LIB_PATH)
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, f"declared in include/*.h but not exported: {missing}"


def test_header_compiles_as_c():
    r = subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-x", "c"] +
                       sorted(glob.glob(os.path.join(ROOT, "include", "*.h"))),
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_library_is_sm90a_only(egpu):
    out = subprocess.run(["cuobjdump", "-lelf", egpu.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_product_does_not_link_or_import_oracle(egpu):
    out = subprocess.run(["nm", "-D", egpu.LIB_PATH], capture_output=True, text=True).stdout
    assert "oracle_" not in out
    pkg = os.path.join(ROOT, "elastic-gpu-agent_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cc", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
                assert not re.search(r'#include\s+"[^"]*oracle', src), f


def test_strerror_and_version(egpu):
    lib = egpu.load()
    assert lib.egpu_abi_version() >= 1000
    assert egpu.strerror(0) == "ok"
    assert "fallback" in egpu.strerror(-2)


def test_null_arguments_are_rejected_without_a_device(egpu):
    lib = egpu.load()
    assert lib.egpu_ctx_create(0, None) == -1
    assert lib.egpu_table_set(None, None, None, 8) == -1
    assert lib.egpu_bestfit_batch(None, None, None, 0, None, None, None, 0) == -1
    assert lib.egpu_replay(None, None, None, None, 0, None) == -1
    lib.egpu_ctx_destroy(None)  # no-op


def test_no_device_fails_loudly(egpu):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the no-device path cannot be exercised")
    with pytest.raises(egpu.EgpuError) as ei:
        egpu.BestFitAllocator(0)
    assert ei.value.code == -2
