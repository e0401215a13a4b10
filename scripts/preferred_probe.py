"""GetPreferredAllocation latency: egpu_preferred_allocation (one container request per call, ID strings, host
parsing) against egpu_preferred_allocation_batch (every container request of a message in one call, flat ID
buffers, ID work on the GPU).  Prints the GPU's name and power limit, then one JSON line per case with the
median of the timed calls (host wall clock, inputs in and answers out) and whether the answers are equal.

    python scripts/preferred_probe.py [--reps 15]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_name_and_power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, watts = [x.strip() for x in out.split(",")]
        return name, float(watts)
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), None


CSTRINGS_C = r"""
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
/* what cgo's C.CString does for every ID, and the free afterwards */
void make_cstrings(const char* flat, const int64_t* off, int64_t n, char** out) {
    for (int64_t i = 0; i < n; ++i) {
        const size_t l = (size_t)(off[i + 1] - off[i]);
        char* p = (char*)malloc(l + 1);
        memcpy(p, flat + off[i], l);
        p[l] = 0;
        out[i] = p;
    }
}
void free_cstrings(char** s, int64_t n) { for (int64_t i = 0; i < n; ++i) free(s[i]); }
"""


def cstrings_lib(tmp):
    src, so = os.path.join(tmp, "cstrings.c"), os.path.join(tmp, "cstrings.so")
    with open(src, "w") as f:
        f.write(CSTRINGS_C)
    subprocess.run(["cc", "-O2", "-shared", "-fPIC", src, "-o", so], check=True)
    return C.CDLL(so)


def ids(gpu, units):
    return ["%d-%02d" % (gpu, u) for u in units]


def median_ms(fn, reps):
    fn()  # warm-up (the batch call's scratch grows once)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return 1e3 * statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()
    import torch
    import elastic_gpu_agent_b200 as e
    from elastic_gpu_agent_b200 import plugin
    lib = e.load()
    tmp = tempfile.mkdtemp(prefix="preferred_probe_")
    cs = cstrings_lib(tmp)
    cs.make_cstrings.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    cs.free_cstrings.argtypes = [C.c_void_p, C.c_int64]
    name, watts = gpu_name_and_power_limit()
    print(json.dumps({"gpu": name, "power_limit_w": watts, "reps": args.reps}))

    node_mem = [s for g in range(8) for s in ids(g, range(183_359))]
    node_core = [s for g in range(8) for s in ids(g, range(100))]
    pod = [(node_mem, [], size) for size in (16_384, 8_192, 40_000, 1_024, 81_559)]
    cases = [("gpu-core, 800 IDs, size 25", plugin.RESOURCE_CORE, [(node_core, [], 25)]),
             ("gpu-memory, 1 466 872 IDs, size 16 384", plugin.RESOURCE_MEM, [(node_mem, [], 16_384)]),
             ("one pod of 5 gpu-memory containers, one message", plugin.RESOURCE_MEM, pod)]
    with e.BestFitAllocator(0) as alloc:
        for label, res, reqs in cases:
            # the existing function: one call per container request, from an array of char* built beforehand
            arrays = [plugin._strs(av) for av, _, _ in reqs]
            outs = [np.full(max(1, n), -1, np.int32) for _, _, n in reqs]
            gpus = [C.c_int32(-1) for _ in reqs]

            def per_request():
                for (av, _, n), (arr, _k), out, g in zip(reqs, arrays, outs, gpus):
                    rc = lib.egpu_preferred_allocation(alloc.handle, arr, len(av), None, 0, n, res, C.c_void_p(out.ctypes.data),
                                                       C.byref(g))
                    assert rc == 0

            flat, io, so, sz = plugin.flatten_requests(reqs)
            flat_np = np.frombuffer(flat, np.uint8)
            cptrs = (C.c_void_p * int(io.size - 1))()

            def per_request_with_strings():  # what a cgo caller pays: C.CString per ID (in C), the call, the frees
                for q, ((av, _, n), out, g) in enumerate(zip(reqs, outs, gpus)):
                    base = C.c_void_p(C.addressof(cptrs) + 8 * int(so[2 * q]))
                    cs.make_cstrings(C.c_void_p(flat_np.ctypes.data), C.c_void_p(io.ctypes.data + 8 * int(so[2 * q])), len(av), base)
                    rc = lib.egpu_preferred_allocation(alloc.handle, base, len(av), None, 0, n, res, C.c_void_p(out.ctypes.data),
                                                       C.byref(g))
                    cs.free_cstrings(base, len(av))
                    assert rc == 0

            t_single = median_ms(per_request, args.reps)
            t_strings = median_ms(per_request_with_strings, args.reps) if len(reqs[0][0]) > 10_000 else None
            pageable = (np.frombuffer(flat, np.uint8).copy(), io.copy(), so.copy(), sz.copy())
            pinned = tuple(torch.from_numpy(a).pin_memory().numpy() for a in pageable)
            result = {}
            for kind, (f, o, s, z) in (("pinned", pinned), ("pageable", pageable)):
                result[kind] = median_ms(lambda: plugin.preferred_allocation_batch_flat(alloc, res, f, o, s, z), args.reps)
            pos, gpu, rc = plugin.preferred_allocation_batch_flat(alloc, res, *pinned)
            per_request()
            equal, off = bool((rc == 0).all()), 0
            for q, (_, _, n) in enumerate(reqs):
                equal = equal and int(gpu[q]) == gpus[q].value and pos[off:off + n].tolist() == outs[q][:n].tolist()
                off += n
            before = alloc.launch_count
            plugin.preferred_allocation_batch_flat(alloc, res, *pinned)
            row = {"case": label, "requests": len(reqs), "ids": int(io.size - 1),
                   "existing_ms": round(t_single, 3), "batch_pinned_ms": round(result["pinned"], 3),
                   "batch_pageable_ms": round(result["pageable"], 3), "launches_per_batch_call": alloc.launch_count - before,
                   "equal": equal}
            if t_strings is not None:
                row["existing_with_cstrings_ms"] = round(t_strings, 3)
            print(json.dumps(row))
    shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
