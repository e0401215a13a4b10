"""A/B probe (one GPU): prefix-commit rounds to the fixed point on int32 arrays
(egpu_bestfit_batch_rounds[_dev]) against the same requests as packed words (egpu_bestfit_batch[_dev] with
EGPU_F_PACKED | EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT | EGPU_F_ROUNDS), int32 and packed alternating in one
run.  Every repetition checks that the packed indices, demand totals and installed table equal the int32 ones.

    python scripts/packed_rounds_probe.py [--reps N] [--warmup N] [--json PATH]

Shapes: the rounds_probe workload (cfg3 table, D = 8, 1 Mi requests with core <= 5 and mem <= 2048), and the
same requests on the cfg4 table (D = 64) under the lookup scan.  Forms: device buffers, host buffers from
pageable memory, host buffers from pinned memory (egpu_host_alloc).  Every call ends in a synchronise, so a
host clock around it measures it; the table is reset outside the timed region.  Medians of --reps calls after
--warmup.  Across PCIe the int32 call moves 12 B per row, the packed one 5 B.
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
    # device buffers
    d_c, d_m = torch.from_numpy(rc).cuda(), torch.from_numpy(rm).cuda()
    d_i32 = torch.empty(R, dtype=torch.int32, device="cuda")
    d_w = torch.from_numpy(words.view(np.int32)).cuda()
    d_i8 = torch.empty(R, dtype=torch.int8, device="cuda")
    d_delta = torch.empty(2 * D, dtype=torch.int64, device="cuda")
    # pageable and pinned host buffers
    pg = dict(c=rc.copy(), m=rm.copy(), w=words.copy(), i32=np.empty(R, np.int32), i8=np.empty(R, np.int8))
    pn = dict(c=a.pinned_array(R, np.int32), m=a.pinned_array(R, np.int32), w=a.pinned_array(R, np.uint32),
              i32=a.pinned_array(R, np.int32), i8=a.pinned_array(R, np.int8))
    pn["c"][:], pn["m"][:], pn["w"][:] = rc, rm, words
    torch.cuda.synchronize()
    n_rounds, left = C.c_int32(0), C.c_int64(0)

    def int32_call(form):
        dc, dm = np.empty(D, np.int64), np.empty(D, np.int64)
        if form == "dev":
            delta = np.empty(2 * D, np.int64)
            t0 = time.perf_counter()
            rc_ = lib.egpu_bestfit_batch_rounds_dev(h, vp(d_c.data_ptr()), vp(d_m.data_ptr()), R, vp(d_i32.data_ptr()),
                                                    vp(delta.ctypes.data), 1 << 30, C.byref(n_rounds), C.byref(left), s)
            t1 = time.perf_counter()
            return t1 - t0, rc_, d_i32.cpu().numpy(), delta
        b = pg if form == "pageable" else pn
        t0 = time.perf_counter()
        rc_ = lib.egpu_bestfit_batch_rounds(h, vp(b["c"].ctypes.data), vp(b["m"].ctypes.data), R, vp(b["i32"].ctypes.data),
                                            vp(dc.ctypes.data), vp(dm.ctypes.data), 1 << 30, C.byref(n_rounds), C.byref(left))
        t1 = time.perf_counter()
        return t1 - t0, rc_, b["i32"].copy(), np.concatenate([dc, dm])

    def packed_call(form):
        dc, dm = np.empty(D, np.int64), np.empty(D, np.int64)
        if form == "dev":
            t0 = time.perf_counter()
            rc_ = lib.egpu_bestfit_batch_dev(h, vp(d_w.data_ptr()), None, R, vp(d_i8.data_ptr()), vp(d_delta.data_ptr()), None,
                                             PR, s)
            t1 = time.perf_counter()
            return t1 - t0, rc_, d_i8.cpu().numpy().astype(np.int32), d_delta.cpu().numpy()
        b = pg if form == "pageable" else pn
        t0 = time.perf_counter()
        rc_ = lib.egpu_bestfit_batch(h, vp(b["w"].ctypes.data), None, R, vp(b["i8"].ctypes.data), vp(dc.ctypes.data),
                                     vp(dm.ctypes.data), PR)
        t1 = time.perf_counter()
        return t1 - t0, rc_, b["i8"].astype(np.int32), np.concatenate([dc, dm])

    res = {}
    try:
        for form in ("dev", "pageable", "pinned"):
            times = {"int32": [], "packed": []}
            for rep in range(warmup + reps):
                out = {}
                for arm, call in (("int32", int32_call), ("packed", packed_call)):
                    a.set_table(fc, fm)
                    torch.cuda.synchronize()
                    dt, code, idx, delta = call(form)
                    assert code == 0, (name, form, arm, code)
                    out[arm] = (idx, delta, a.table())
                    if rep >= warmup:
                        times[arm].append(dt)
                (i_a, d_a, t_a), (i_b, d_b, t_b) = out["int32"], out["packed"]
                assert np.array_equal(i_a, i_b), (name, form, rep, "indices")
                assert np.array_equal(d_a, d_b), (name, form, rep, "totals")
                assert all(np.array_equal(x, y) for x, y in zip(t_a, t_b)), (name, form, rep, "table")
                assert not (i_a == -2).any()
            med = {arm: 1e3 * float(np.median(v)) for arm, v in times.items()}
            res[form] = {"int32_ms": round(med["int32"], 3), "packed_ms": round(med["packed"], 3),
                         "ratio": round(med["packed"] / med["int32"], 3)}
            print(f"{name:18s} {form:8s} int32 {med['int32']:8.3f} ms  packed {med['packed']:8.3f} ms  "
                  f"ratio {med['packed'] / med['int32']:.3f}  rounds {n_rounds.value}  (all {reps + warmup} repetitions equal)",
                  flush=True)
    finally:
        for arr in pn.values():
            a.host_free(arr.ctypes.data)
    res["rounds"] = int(n_rounds.value)
    res["D"] = D
    res["R"] = R
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
