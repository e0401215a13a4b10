"""A/B probe (one GPU): multi-batch launches in the int32 format against the same batches in the packed
format (egpu_bestfit_batches_dev with EGPU_F_PACKED), one launch per CUDA graph, the two graphs replayed
in turn, median of 101 replays each.  Checks in the same run that the packed indices equal the int32
indices and that the demand sums and table' are equal.

    python scripts/packed_multi_probe.py [--reps N] [--only NAME] [--json PATH]

Bytes per batch are the algorithmic ones: 12 R + 32 D (int32) and 5 R + 32 D (packed), as a fraction of
the H100 SXM data-sheet HBM bandwidth (3.35 TB/s; not a measured peak).
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import elastic_gpu_agent_b200 as e  # noqa: E402

PEAK_GBS = 3350.0  # H100 SXM data sheet
MEM_MAX = (1 << 18) - 1
# name -> (workload, K, R, variant)
SHAPES = {
    "20x1M_D8": ("cfg3_1m", 20, 1_000_000, e.VARIANT_AUTO),
    "20x1M_D64_lut": ("cfg4", 20, 1_000_000, e.VARIANT_AUTO),
    "20x1M_D64_sorted": ("cfg4", 20, 1_000_000, e.VARIANT_SORTED),
    "64x100k_D8": ("cfg3", 64, 100_000, e.VARIANT_AUTO),
    "64x1k_D8": ("cfg3", 64, 1_000, e.VARIANT_AUTO),
    "1x64Mi_D8": ("cfg3_64mi", 1, 64 << 20, e.VARIANT_AUTO),
}


def card():
    name = torch.cuda.get_device_name(0)
    limit = None
    try:
        import pynvml
        pynvml.nvmlInit()
        limit = pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception:
        try:
            out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                 capture_output=True, text=True, timeout=30).stdout.strip()
            limit = float(out.splitlines()[0])
        except Exception:
            pass
    return name, limit


def run_shape(a, name, reps):
    wname, K, R, variant = SHAPES[name]
    w = e.synth.workload(wname)
    D = int(w["D"])
    a.set_variant(variant)
    a.set_table(w["free_core"], w["free_mem"])
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream()
    sh = st.cuda_stream
    i32, pk = [], []
    for k in range(K):
        c = torch.empty(R, dtype=torch.int32, device=dev)
        m = torch.empty(R, dtype=torch.int32, device=dev)
        a.synth_requests_dev(w["dist"], w["seed"], k * R, R, c.data_ptr(), m.data_ptr(), sh)
        ok = (c >= 0) & (c <= 127) & (m >= 0) & (m <= MEM_MAX)
        words = torch.where(ok, (c << 18) | m, torch.full_like(c, -1))
        i32.append((c, m, torch.empty(R, dtype=torch.int32, device=dev), torch.zeros(2 * D, dtype=torch.int64, device=dev),
                    torch.zeros(3 * D, dtype=torch.int32, device=dev)))
        pk.append((words, torch.empty(R, dtype=torch.int8, device=dev), torch.zeros(2 * D, dtype=torch.int64, device=dev),
                   torch.zeros(3 * D, dtype=torch.int32, device=dev)))
    torch.cuda.synchronize()
    arr32 = a.make_batches([(c.data_ptr(), m.data_ptr(), R, i.data_ptr(), dl.data_ptr(), t.data_ptr()) for c, m, i, dl, t in i32])
    arr8 = a.make_packed_batches([(p.data_ptr(), R, i.data_ptr(), dl.data_ptr(), t.data_ptr()) for p, i, dl, t in pk])

    def graph_of(fn):
        fn(sh)  # warm-up outside the capture: occupancy query, lookup tables
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        cap = torch.cuda.Stream()
        with torch.cuda.stream(cap):
            with torch.cuda.graph(g, stream=cap):
                fn(cap.cuda_stream)
        g.replay()
        torch.cuda.synchronize()
        return g

    g32 = graph_of(lambda s: a.bestfit_batches_dev(arr32, s, inputs_ready=True))
    g8 = graph_of(lambda s: a.bestfit_batches_packed_dev(arr8, s, inputs_ready=True))
    ts = {"int32": [], "packed": []}
    for _ in range(reps):
        for tag, g in (("int32", g32), ("packed", g8)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.gate_dev(sh)  # nothing below starts before the host has enqueued all of it
            e0.record(st)
            g.replay()
            e1.record(st)
            a.gate_open()
            torch.cuda.synchronize()
            ts[tag].append(e0.elapsed_time(e1) * 1e3 / K)
    parity = True
    for (c, m, i, dl, t), (p, i8, dl8, t8) in zip(i32, pk):
        parity &= bool(torch.equal(i, i8.to(torch.int32))) and bool(torch.equal(dl, dl8)) and bool(torch.equal(t, t8))
    out = {"shape": name, "K": K, "R": R, "D": D, "variant": variant, "parity": parity}
    for tag, bpr in (("int32", 12), ("packed", 5)):
        x = np.array(ts[tag])
        us = float(np.median(x))
        out[tag] = {"us_per_batch_median": us, "min": float(x.min()), "max": float(x.max()),
                    "decisions_per_s": R / (us * 1e-6),
                    "frac_of_datasheet_hbm": (bpr * R + 32 * D) / (us * 1e-6) / 1e9 / PEAK_GBS}
    out["packed_over_int32_time"] = out["packed"]["us_per_batch_median"] / out["int32"]["us_per_batch_median"]
    del g32, g8, i32, pk
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=101)
    ap.add_argument("--only", action="append")
    ap.add_argument("--json")
    args = ap.parse_args()
    name, limit = card()
    res = {"gpu": name, "power_limit_w": limit, "env": {k: v for k, v in os.environ.items() if k.startswith("EGPU_")},
           "shapes": []}
    a = e.BestFitAllocator(0)
    try:
        for s in args.only or list(SHAPES):
            r = run_shape(a, s, args.reps)
            res["shapes"].append(r)
            print(f"{s:18s} int32 {r['int32']['us_per_batch_median']:9.3f} us/batch ({r['int32']['frac_of_datasheet_hbm']:.2f})  "
                  f"packed {r['packed']['us_per_batch_median']:9.3f} us/batch ({r['packed']['frac_of_datasheet_hbm']:.2f})  "
                  f"{r['packed']['decisions_per_s'] / 1e9:7.1f} G dec/s  parity {r['parity']}", flush=True)
    finally:
        a.close()
    print(f"{name}, power limit {limit} W; fractions are algorithmic bytes over the 3.35 TB/s data-sheet bandwidth")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
