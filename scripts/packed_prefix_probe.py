"""A/B probe (one GPU): prefix-commit on int32 arrays against the same requests as packed words
(egpu_bestfit_batch[_dev] with EGPU_F_PACKED | EGPU_F_PREFIX_COMMIT), int32 and packed alternating in one
run.  Checks in the same run that the packed indices, demand sums and table' equal the int32 ones.

    python scripts/packed_prefix_probe.py [--reps N] [--host-reps N] [--only NAME] [--json PATH]

Device buffers: non-committing calls (every replay computes the same thing), 20 calls per CUDA graph over
a ring of buffer sets larger than L2, graphs replayed in turn; medians of --reps replays.  A third arm runs
the packed call in a context created with EGPU_ROWS_PER_THREAD set to twice the default CONTIG rule
(16 in the register scan, 64 in the lookup scan): the rows-per-thread question for packed tiles.
Bytes are algorithmic: int32 12 R for the scan + 8 R for the rewrite of the indices, packed 5 R + 2 R, as a
fraction of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s; not a measured peak).

Host buffers: egpu_bestfit_batch with EGPU_F_COMMIT | EGPU_F_PREFIX_COMMIT on pinned and on pageable
arrays, host clock around the synchronous call, the table reset outside the timed region; median of
--host-reps calls.  Across PCIe the int32 call moves 12 B per row, the packed call 5.
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

PEAK_GBS = 3350.0  # H100 SXM data sheet
L2_BYTES = 50 << 20
MEM_MAX = (1 << 18) - 1
CALLS_PER_GRAPH = 20
# name -> (workload, R, variant)
SHAPES = {
    "cfg3_1M_D8": ("cfg3", 1_000_000, e.VARIANT_AUTO),
    "cfg4_1M_D64_lut": ("cfg4", 1_000_000, e.VARIANT_AUTO),
    "100k_D8": ("cfg3", 100_000, e.VARIANT_AUTO),
    "16Mi+1_D64_lut": ("cfg4", (16 << 20) + 1, e.VARIANT_AUTO),
}


def card():
    """card name and power limit, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def fresh_alloc(rpt=None):
    if rpt:
        os.environ["EGPU_ROWS_PER_THREAD"] = str(rpt)
    try:
        return e.BestFitAllocator(0)
    finally:
        os.environ.pop("EGPU_ROWS_PER_THREAD", None)


def run_dev(a, a2, name, reps):
    wname, R, variant = SHAPES[name]
    w = e.synth.workload(wname)
    D = int(w["D"])
    dev = torch.device("cuda", 0)
    sh = torch.cuda.current_stream().cuda_stream
    n_ring = max(2, -(-2 * L2_BYTES // (5 * R)))  # the packed sets alone are twice L2
    sets = []
    for k in range(n_ring):
        c = torch.empty(R + 4, dtype=torch.int32, device=dev)
        m = torch.empty(R + 4, dtype=torch.int32, device=dev)
        a.synth_requests_dev(w["dist"], w["seed"], k * R, R, c.data_ptr(), m.data_ptr(), sh)
        ok = (c >= 0) & (c <= 127) & (m >= 0) & (m <= MEM_MAX)
        words = torch.where(ok, (c << 18) | m, torch.full_like(c, -1))
        out = {tag: (torch.empty(R + 16, dtype=torch.int32 if tag == "int32" else torch.int8, device=dev),
                     torch.zeros(2 * D, dtype=torch.int64, device=dev), torch.zeros(3 * D, dtype=torch.int32, device=dev))
               for tag in ("int32", "packed", "packed_rpt2x")}
        sets.append((c, m, words, out))
    torch.cuda.synchronize()

    def call(tag, k, s):
        c, m, words, out = sets[k % n_ring]
        i, dl, t = (x.data_ptr() for x in out[tag])
        if tag == "int32":
            a.bestfit_dev(c.data_ptr(), m.data_ptr(), R, i, dl, t, False, s, prefix_commit=True)
        else:
            (a if tag == "packed" else a2).bestfit_packed_prefix_dev(words.data_ptr(), R, i, dl, t, False, s)

    graphs = {}
    for tag, al in (("int32", a), ("packed", a), ("packed_rpt2x", a2)):
        al.set_variant(variant)
        al.set_table(w["free_core"], w["free_mem"])
        call(tag, 0, sh)  # warm-up outside the capture: scratch, occupancy, lookup tables
        torch.cuda.synchronize()
        gs = []
        for g0 in range(0, max(n_ring, CALLS_PER_GRAPH), CALLS_PER_GRAPH):
            g = torch.cuda.CUDAGraph()
            cap = torch.cuda.Stream()
            with torch.cuda.stream(cap):
                with torch.cuda.graph(g, stream=cap):
                    for k in range(g0, g0 + CALLS_PER_GRAPH):
                        call(tag, k, cap.cuda_stream)
            g.replay()
            gs.append(g)
        torch.cuda.synchronize()
        graphs[tag] = gs
    st = torch.cuda.current_stream()
    ts = {tag: [] for tag in graphs}
    for rep in range(reps):
        for tag, gs in graphs.items():
            g = gs[rep % len(gs)]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(st)
            g.replay()
            e1.record(st)
            torch.cuda.synchronize()
            ts[tag].append(e0.elapsed_time(e1) * 1e3 / CALLS_PER_GRAPH)
    equal = True
    for c, m, words, out in sets:
        i, dl, t = out["int32"]
        for tag in ("packed", "packed_rpt2x"):
            i8, dl8, t8 = out[tag]
            equal &= bool(torch.equal(i[:R], i8[:R].to(torch.int32))) and bool(torch.equal(dl, dl8)) and bool(torch.equal(t, t8))
    deferred = int((sets[0][3]["int32"][0][:R] == L.IDX_DEFERRED).sum())
    res = {"shape": name, "R": R, "D": D, "variant": variant, "ring_sets": n_ring, "graphs": len(graphs["int32"]),
           "outputs_equal": equal, "deferred_rows_set0": deferred}
    for tag, bpr in (("int32", 20), ("packed", 7), ("packed_rpt2x", 7)):
        x = np.array(ts[tag])
        us = float(np.median(x))
        res[tag] = {"us_per_call_median": us, "min": float(x.min()), "max": float(x.max()),
                    "frac_of_datasheet_hbm": bpr * R / (us * 1e-6) / 1e9 / PEAK_GBS}
    del graphs, sets
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return res


def run_host(a, reps, R=1_000_000):
    w = e.synth.workload("cfg3")
    D = int(w["D"])
    rc, rm = e.synth.requests(w["dist"], w["seed"], R)
    words = a.pack_requests(rc, rm)
    flags = L.F_COMMIT | L.F_PREFIX_COMMIT
    a.set_variant(e.VARIANT_AUTO)
    res = {"R": R, "D": D}
    pin = {"rc": a.pinned_array(R), "rm": a.pinned_array(R), "idx": a.pinned_array(R), "w": a.pinned_array(R, np.uint32),
           "i8": a.pinned_array(R, np.int8)}
    try:
        pin["rc"][:], pin["rm"][:], pin["w"][:] = rc, rm, words
        page = {"rc": rc.copy(), "rm": rm.copy(), "idx": np.empty(R, np.int32), "w": words.copy(), "i8": np.empty(R, np.int8)}
        dc, dm = np.zeros(D, np.int64), np.zeros(D, np.int64)
        pd, pm = C.c_void_p(dc.ctypes.data), C.c_void_p(dm.ctypes.data)
        outs = {}
        for kind, b in (("pinned", pin), ("pageable", page)):
            p = {k: C.c_void_p(v.ctypes.data) for k, v in b.items()}
            arms = {"int32": lambda: a._lib.egpu_bestfit_batch(a.handle, p["rc"], p["rm"], R, p["idx"], pd, pm, flags),
                    "packed": lambda: a._lib.egpu_bestfit_batch(a.handle, p["w"], None, R, p["i8"], pd, pm, flags | L.F_PACKED)}
            ts = {tag: [] for tag in arms}
            for rep in range(reps + 1):  # the first round is the warm-up
                for tag, fn in arms.items():
                    a.set_table(w["free_core"], w["free_mem"])
                    t0 = time.perf_counter()
                    rcode = fn()
                    t1 = time.perf_counter()
                    assert rcode == 0, (kind, tag, rcode)
                    if rep:
                        ts[tag].append((t1 - t0) * 1e6)
                    outs[(kind, tag)] = (b["idx"].copy() if tag == "int32" else b["i8"].astype(np.int32), dc.copy(), dm.copy(),
                                         a.table()[:2])
            res[kind] = {}
            for tag, bpr in (("int32", 12), ("packed", 5)):
                us = float(np.median(ts[tag]))
                res[kind][tag] = {"us_per_call_median": us, "min": float(min(ts[tag])), "max": float(max(ts[tag])),
                                  "pcie_bytes_per_row": bpr, "effective_gbs": bpr * R / (us * 1e-6) / 1e9}
        ref = outs[("pinned", "int32")]
        res["outputs_equal"] = all(all(np.array_equal(x, y) for x, y in zip(ref[:3], o[:3])) and
                                   all(np.array_equal(x, y) for x, y in zip(ref[3], o[3])) for o in outs.values())
    finally:
        for v in pin.values():
            a.host_free(v.ctypes.data)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=101)
    ap.add_argument("--host-reps", type=int, default=15)
    ap.add_argument("--only", action="append")
    ap.add_argument("--no-host", action="store_true")
    ap.add_argument("--json")
    args = ap.parse_args()
    res = {"gpu": card(), "shapes": []}
    a = fresh_alloc()
    try:
        for s in args.only or list(SHAPES):
            a2 = fresh_alloc(64 if SHAPES[s][0] == "cfg4" else 16)
            try:
                r = run_dev(a, a2, s, args.reps)
            finally:
                a2.close()
            res["shapes"].append(r)
            print(f"{s:16s} int32 {r['int32']['us_per_call_median']:9.2f} us ({r['int32']['frac_of_datasheet_hbm']:.2f})  "
                  f"packed {r['packed']['us_per_call_median']:9.2f} us ({r['packed']['frac_of_datasheet_hbm']:.2f})  "
                  f"packed 2x rpt {r['packed_rpt2x']['us_per_call_median']:9.2f} us  equal {r['outputs_equal']}", flush=True)
        if not args.no_host:
            h = run_host(a, args.host_reps)
            res["host"] = h
            for kind in ("pinned", "pageable"):
                print(f"host {kind:8s} 1M D8  int32 {h[kind]['int32']['us_per_call_median']:9.1f} us  "
                      f"packed {h[kind]['packed']['us_per_call_median']:9.1f} us  equal {h['outputs_equal']}", flush=True)
    finally:
        a.close()
    print(f"{res['gpu']}; fractions are algorithmic bytes over the 3.35 TB/s data-sheet bandwidth")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
