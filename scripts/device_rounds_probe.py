"""A/B probe (one GPU): rounds to the fixed point in one launch (EGPU_F_DEVICE_ROUNDS) against the synchronous
rounds (egpu_bestfit_batch_rounds[_dev] on int32 arrays, EGPU_F_ROUNDS on packed words), the two alternating in
one run.  Every repetition checks that indices, demand totals and the installed table are equal.

    python scripts/device_rounds_probe.py [--reps N] [--warmup N] [--json PATH]

Shapes (those of scripts/packed_rounds_probe.py): the cfg3 table (D = 8, AUTO: register scan) and the cfg4 table
(D = 64, lookup scan), 1 Mi requests with core <= 5 and mem <= 2048.  Both row formats; forms: device buffers,
host buffers from pageable memory, host buffers from pinned memory (egpu_host_alloc), and the device form replayed
from a CUDA graph.  Every timed call ends in a synchronise (the device form is asynchronous: the clock stops after
torch.cuda.synchronize()), so a host clock around it measures it; the table is reset outside the timed region.
Medians of --reps calls after --warmup.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import elastic_gpu_agent_b200 as e  # noqa: E402
from elastic_gpu_agent_b200 import _lib as L  # noqa: E402

PR = L.F_PACKED | L.F_PREFIX_COMMIT | L.F_COMMIT | L.F_ROUNDS
DR = L.F_PREFIX_COMMIT | L.F_COMMIT | L.F_ROUNDS | L.F_DEVICE_ROUNDS
SHAPES = {"cfg3_1Mi_D8": ("cfg3", e.VARIANT_AUTO), "cfg4_1Mi_D64_lut": ("cfg4", e.VARIANT_LUT)}


def card():
    """card name and power limit, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def vp(x):
    return C.c_void_p(x)


def run_shape(a, name, reps, warmup):
    wname, variant = SHAPES[name]
    w = e.synth.workload(wname)
    fc, fm = np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32)
    D = fc.size
    rc, rm = e.synth.requests(3, 5, 1 << 20)
    rc, rm = np.minimum(rc, 5).astype(np.int32), np.minimum(rm, 2048).astype(np.int32)
    R = rc.size
    words = a.pack_requests(rc, rm)
    a.set_variant(variant)
    lib, h = a._lib, a.handle
    st = torch.cuda.Stream()
    s = vp(st.cuda_stream)
    dev = {"c": torch.from_numpy(rc).cuda(), "m": torch.from_numpy(rm).cuda(), "w": torch.from_numpy(words.view(np.int32)).cuda(),
           "i32": torch.empty(R, dtype=torch.int32, device="cuda"), "i8": torch.empty(R, dtype=torch.int8, device="cuda"),
           "delta": torch.empty(2 * D, dtype=torch.int64, device="cuda")}
    pg = dict(c=rc.copy(), m=rm.copy(), w=words.copy(), i32=np.empty(R, np.int32), i8=np.empty(R, np.int8))
    pn = dict(c=a.pinned_array(R, np.int32), m=a.pinned_array(R, np.int32), w=a.pinned_array(R, np.uint32),
              i32=a.pinned_array(R, np.int32), i8=a.pinned_array(R, np.int8))
    pn["c"][:], pn["m"][:], pn["w"][:] = rc, rm, words
    torch.cuda.synchronize()
    n_rounds, left = C.c_int32(0), C.c_int64(0)

    def dev_call(packed, device):
        """device buffers: (seconds, return code, indices, totals)"""
        i = dev["i8"] if packed else dev["i32"]
        core, mem = (dev["w"], None) if packed else (dev["c"], dev["m"])
        host_delta = np.empty(2 * D, np.int64)
        t0 = time.perf_counter()
        if device or packed:
            code = lib.egpu_bestfit_batch_dev(h, vp(core.data_ptr()), vp(mem.data_ptr()) if mem is not None else None, R,
                                              vp(i.data_ptr()), vp(dev["delta"].data_ptr()), None,
                                              (DR | (L.F_PACKED if packed else 0)) if device else PR, s)
        else:
            code = lib.egpu_bestfit_batch_rounds_dev(h, vp(core.data_ptr()), vp(mem.data_ptr()), R, vp(i.data_ptr()),
                                                     vp(host_delta.ctypes.data), 1 << 30, C.byref(n_rounds), C.byref(left), s)
        st.synchronize()
        t1 = time.perf_counter()
        delta = host_delta if not (device or packed) else dev["delta"].cpu().numpy()
        return t1 - t0, code, i.cpu().numpy().astype(np.int32), delta

    def host_call(packed, device, b):
        dc, dm = np.empty(D, np.int64), np.empty(D, np.int64)
        i = b["i8"] if packed else b["i32"]
        t0 = time.perf_counter()
        if device or packed:
            code = lib.egpu_bestfit_batch(h, vp(b["w"].ctypes.data if packed else b["c"].ctypes.data),
                                          None if packed else vp(b["m"].ctypes.data), R, vp(i.ctypes.data), vp(dc.ctypes.data),
                                          vp(dm.ctypes.data), (DR | (L.F_PACKED if packed else 0)) if device else PR)
        else:
            code = lib.egpu_bestfit_batch_rounds(h, vp(b["c"].ctypes.data), vp(b["m"].ctypes.data), R, vp(i.ctypes.data),
                                                 vp(dc.ctypes.data), vp(dm.ctypes.data), 1 << 30, C.byref(n_rounds), C.byref(left))
        t1 = time.perf_counter()
        return t1 - t0, code, i.astype(np.int32), np.concatenate([dc, dm])

    # the device form captured in a CUDA graph, one per format (captured after an eager warm-up call)
    graphs = {}
    for packed in (False, True):
        a.set_table(fc, fm)
        with torch.cuda.stream(st):
            assert dev_call(packed, True)[1] == 0
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=st):
                i = dev["i8"] if packed else dev["i32"]
                core, mem = (dev["w"], None) if packed else (dev["c"], dev["m"])
                code = lib.egpu_bestfit_batch_dev(h, vp(core.data_ptr()), vp(mem.data_ptr()) if mem is not None else None, R,
                                                  vp(i.data_ptr()), vp(dev["delta"].data_ptr()), None,
                                                  DR | (L.F_PACKED if packed else 0), s)
                assert code == 0, lib.egpu_last_error(h).decode()
        graphs[packed] = g
    torch.cuda.synchronize()

    def graph_call(packed):
        t0 = time.perf_counter()
        graphs[packed].replay()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        i = dev["i8"] if packed else dev["i32"]
        return t1 - t0, 0, i.cpu().numpy().astype(np.int32), dev["delta"].cpu().numpy()

    res = {}
    try:
        for fmt in ("int32", "packed"):
            packed = fmt == "packed"
            for form in ("dev", "pageable", "pinned", "graph"):
                arms = {"sync": None, "device": None}
                if form == "dev":
                    arms = {"sync": lambda: dev_call(packed, False), "device": lambda: dev_call(packed, True)}
                elif form == "graph":
                    arms = {"sync": lambda: dev_call(packed, False), "device": lambda: graph_call(packed)}
                else:
                    b = pg if form == "pageable" else pn
                    arms = {"sync": lambda b=b: host_call(packed, False, b), "device": lambda b=b: host_call(packed, True, b)}
                times = {"sync": [], "device": []}
                for rep in range(warmup + reps):
                    out = {}
                    for arm, call in arms.items():
                        a.set_table(fc, fm)
                        torch.cuda.synchronize()
                        dt, code, idx, delta = call()
                        assert code == 0, (name, fmt, form, arm, code, lib.egpu_last_error(h).decode())
                        out[arm] = (idx, delta, a.table())
                        if rep >= warmup:
                            times[arm].append(dt)
                    (i_a, d_a, t_a), (i_b, d_b, t_b) = out["sync"], out["device"]
                    assert np.array_equal(i_a, i_b), (name, fmt, form, rep, "indices")
                    assert np.array_equal(d_a, d_b), (name, fmt, form, rep, "totals")
                    assert all(np.array_equal(x, y) for x, y in zip(t_a, t_b)), (name, fmt, form, rep, "table")
                    assert not (i_a == -2).any()
                med = {arm: 1e3 * float(np.median(v)) for arm, v in times.items()}
                res[f"{fmt}_{form}"] = {"sync_ms": round(med["sync"], 3), "device_ms": round(med["device"], 3),
                                        "ratio": round(med["device"] / med["sync"], 3)}
                print(f"{name:18s} {fmt:6s} {form:8s} sync {med['sync']:8.3f} ms  device {med['device']:8.3f} ms  "
                      f"ratio {med['device'] / med['sync']:.3f}  (all {reps + warmup} repetitions equal)", flush=True)
    finally:
        torch.cuda.synchronize()
        for arr in pn.values():
            a.host_free(arr.ctypes.data)
    # rounds of the synchronous path (the int32 call reports them)
    a.set_table(fc, fm)
    assert lib.egpu_bestfit_batch_rounds(h, vp(pg["c"].ctypes.data), vp(pg["m"].ctypes.data), R, vp(pg["i32"].ctypes.data),
                                         None, None, 1 << 30, C.byref(n_rounds), C.byref(left)) == 0
    res["rounds"] = int(n_rounds.value)
    res["D"] = D
    res["R"] = R
    print(f"{name:18s} rounds of the synchronous path: {n_rounds.value}", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert args.reps >= 15
    gpu = card()
    print("card:", gpu, flush=True)
    results = {"card": gpu, "reps": args.reps, "warmup": args.warmup, "shapes": {}}
    with e.BestFitAllocator(0) as a:
        for name in SHAPES:
            results["shapes"][name] = run_shape(a, name, args.reps, args.warmup)
    print(json.dumps(results))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
