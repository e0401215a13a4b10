"""A/B probe (one GPU, world 1: the context exchanges with itself): K sharded prefix-commits in ONE launch
(egpu_bestfit_batches_shard_dev with EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT) against K consecutive
egpu_bestfit_batch_shard_prefix_dev calls on one stream.  The two arms alternate in one run; every repetition checks
that per-batch indices, demand sums, table' and the installed table are equal.

    python scripts/shard_prefix_multi_probe.py [--reps N] [--warmup N] [--json PATH]

Shapes, each in the int32 and the packed format:
  queue    64 x 1 Ki cfg2-style requests on the cfg3 table (D = 8): an admission queue;
  small    16 x 64 Ki small requests (core <= 5, mem <= 2048) on the cfg3 table;
  lone     1 x 1 Mi of the same small requests on the cfg3 table;
  cfg4     16 x 64 Ki small requests on the cfg4 table (D = 64, lookup scan).
Forms: eager calls, and each arm captured once in a CUDA graph and replayed.  Every timed call ends in a
synchronise, so the host clock around it measures it; the table is reset by egpu_table_set before every
repetition, outside the timed region.  Medians of --reps (>= 15) repetitions after --warmup.  Multi-GPU is not
measured here.
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

FLAGS = L.F_PREFIX_COMMIT | L.F_COMMIT
# name -> (table, request distribution, clip to small requests, rows per batch)
SHAPES = {
    "queue_64x1Ki_cfg3": ("cfg3", 2, False, [1024] * 64),
    "small_16x64Ki_cfg3": ("cfg3", 3, True, [64 << 10] * 16),
    "lone_1x1Mi_cfg3": ("cfg3", 3, True, [1 << 20]),
    "cfg4_16x64Ki_D64_lut": ("cfg4", 3, True, [64 << 10] * 16),
}


def card():
    """card name and power limit, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def vp(x):
    return C.c_void_p(x)


class Arm:
    """device outputs of one arm: per batch indices, demand sums and table'"""

    def __init__(self, rows, D, packed):
        dt = torch.int8 if packed else torch.int32
        self.idx = [torch.empty(R + 16, dtype=dt, device="cuda") for R in rows]
        self.delta = [torch.empty(2 * D, dtype=torch.int64, device="cuda") for _ in rows]
        self.tab = [torch.empty(3 * D, dtype=torch.int32, device="cuda") for _ in rows]

    def get(self, rows):
        return [(i[:R].cpu().numpy().astype(np.int32), d.cpu().numpy(), t.cpu().numpy())
                for i, d, t, R in zip(self.idx, self.delta, self.tab, rows)]


def run_shape(a, name, reps, warmup):
    wname, dist, clip, rows = SHAPES[name]
    w = e.synth.workload(wname)
    fc, fm = np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32)
    D = fc.size
    a.set_variant(e.VARIANT_AUTO)
    lib, h = a._lib, a.handle
    st = torch.cuda.Stream()
    s = vp(st.cuda_stream)
    res = {"D": D, "K": len(rows), "rows": sum(rows)}
    for fmt in ("int32", "packed"):
        packed = fmt == "packed"
        ins = []
        for k, R in enumerate(rows):
            rc, rm = e.synth.requests(dist, 100 + k, R)
            if clip:
                rc, rm = np.minimum(rc, 5), np.minimum(rm, 2048)
            rc, rm = rc.astype(np.int32), rm.astype(np.int32)
            if packed:
                ins.append((torch.from_numpy(a.pack_requests(rc, rm).view(np.int32)).cuda(), None))
            else:
                ins.append((torch.from_numpy(rc).cuda(), torch.from_numpy(rm).cuda()))
        flags = FLAGS | (L.F_PACKED if packed else 0)
        one, many = Arm(rows, D, packed), Arm(rows, D, packed)
        arr = (L.Batch * len(rows))()
        for k, ((c, m), R) in enumerate(zip(ins, rows)):
            arr[k] = L.Batch(c.data_ptr(), m.data_ptr() if m is not None else None, R, one.idx[k].data_ptr(),
                             one.delta[k].data_ptr(), one.tab[k].data_ptr())

        # world 1: every call consumes its own exchange steps, so each issue may start again from step 0
        def issue_one():
            code = lib.egpu_bestfit_batches_shard_dev(h, arr, len(rows), flags, 0, s)
            assert code == 0, lib.egpu_last_error(h).decode()

        def issue_many():
            for k, ((c, m), R) in enumerate(zip(ins, rows)):
                code = lib.egpu_bestfit_batch_shard_prefix_dev(h, vp(c.data_ptr()), vp(m.data_ptr()) if m is not None else None,
                                                               R, vp(many.idx[k].data_ptr()), vp(many.delta[k].data_ptr()),
                                                               vp(many.tab[k].data_ptr()), flags, 2 * k, s)
                assert code == 0, lib.egpu_last_error(h).decode()

        graphs = {}
        for arm, issue in (("one", issue_one), ("many", issue_many)):
            a.set_table(fc, fm)
            with torch.cuda.stream(st):
                issue()  # eager warm-up: occupancy queries and scratch outside the capture
                st.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=st):
                    issue()
            graphs[arm] = g
        torch.cuda.synchronize()

        def timed(fn):
            t0 = time.perf_counter()
            fn()
            st.synchronize()
            return time.perf_counter() - t0

        for form in ("eager", "graph"):
            arms = {"one": issue_one, "many": issue_many} if form == "eager" else \
                   {"one": graphs["one"].replay, "many": graphs["many"].replay}
            times = {"one": [], "many": []}
            for rep in range(warmup + reps):
                tables = {}
                for arm, fn in arms.items():
                    a.set_table(fc, fm)
                    torch.cuda.synchronize()
                    with torch.cuda.stream(st):
                        dt = timed(fn)
                    tables[arm] = a.table()
                    if rep >= warmup:
                        times[arm].append(dt)
                g_one, g_many = one.get(rows), many.get(rows)
                for k, (x, y) in enumerate(zip(g_one, g_many)):
                    assert all(np.array_equal(p, q) for p, q in zip(x, y)), (name, fmt, form, rep, "batch", k)
                assert all(np.array_equal(p, q) for p, q in zip(tables["one"], tables["many"])), (name, fmt, form, rep, "table")
            assert a.peer_last_timeout == 0
            med = {arm: 1e3 * float(np.median(v)) for arm, v in times.items()}
            res[f"{fmt}_{form}"] = {"one_launch_ms": round(med["one"], 4), "k_calls_ms": round(med["many"], 4),
                                    "ratio": round(med["one"] / med["many"], 3)}
            print(f"{name:22s} {fmt:6s} {form:5s} one launch {med['one']:9.4f} ms  {len(rows)} calls {med['many']:9.4f} ms  "
                  f"ratio {med['one'] / med['many']:.3f}  (all {reps + warmup} repetitions equal)", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    args = ap.parse_args()
    assert args.reps >= 15
    gpu = card()
    print("card:", gpu, flush=True)
    results = {"card": gpu, "gpus": torch.cuda.device_count(), "reps": args.reps, "warmup": args.warmup, "shapes": {}}
    with e.BestFitAllocator(0) as a:
        a.peer_attach(0, 1, [a.peer_export()])
        for name in args.shapes.split(","):
            results["shapes"][name] = run_shape(a, name, args.reps, args.warmup)
        a.peer_detach()
    print(json.dumps(results))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
