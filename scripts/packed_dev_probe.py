"""A/B/C probe (one GPU): egpu_bestfit_batch_packed_dev on the snapshot launch path against the warp-chunk packed scan
it ran before, and against the int32 egpu_bestfit_batch_dev on the same requests, all three alternating in one run.

    python scripts/packed_dev_probe.py [--reps N] [--json PATH]

Arms:
  packed   egpu_bestfit_batch_packed_dev, variant AUTO: the round-robin packed snapshot scan (register scan at D <= 16,
           lookup scan above), pipelined under EGPU_F_INPUTS_READY;
  chunk    the same call in a context set to EGPU_VARIANT_GRID, which keeps the warp-chunk scan of the host call
           (bestfit_sorted_packed_kernel, 512-row warp chunks, always fully ordered): the kernel every variant ran before;
  int32    egpu_bestfit_batch_dev, variant AUTO, on the int32 requests the words stand for.

Shapes: cfg3 (D = 8) and cfg4 (D = 64) at 1 Mi rows, cfg3 at 100 k rows, cfg4 at 16 Mi + 1 rows.  Each shape runs
20 non-committing calls with 20 distinct output sets, "lone" (fully ordered calls) and "pipelined"
(EGPU_F_INPUTS_READY).  The inputs are a ring of seeded request sets (at most 20, at least 160 MB of words where the
shape allows, so the ring does not sit in the 50 MB L2).  Every region is captured once in a CUDA graph after an
eager pass, and the graphs of the arms are replayed in turn --reps times, CUDA events on the launching stream and a
device synchronisation around every replay; the numbers are medians in us per call, with min and max.  Before every
replay the outputs are filled with sentinels; after it every output set of every arm is compared on the device with
the int32 arm's eager result (indices, demand sums, table').
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

MEM_MAX = (1 << 18) - 1
CALLS = 20
SHAPES = (("cfg3", 1 << 20), ("cfg4", 1 << 20), ("cfg3", 100_000), ("cfg4", (16 << 20) + 1))
ARMS = ("packed", "chunk", "int32")
GRID_ARMS = ("half", "double")
# the rows per thread the launcher ships for this call (launch_snapshot_as): a lone register scan 16, a lone lookup
# scan 32, a pipelined scan 48
SHIPPED_RPT = {("cfg3", False): 16, ("cfg4", False): 32, ("cfg3", True): 48, ("cfg4", True): 48}


def card():
    """card name and power limit, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


class Shape:
    """a ring of request sets (int32 arrays and the same requests as words) and CALLS output sets per arm"""

    def __init__(self, a, wname, R):
        w = e.synth.workload(wname)
        self.w, self.R, self.D = w, R, int(w["D"])
        n_in = max(2, min(CALLS, (160 << 20) // (4 * R)))
        dev = torch.device("cuda", 0)
        sh = torch.cuda.current_stream().cuda_stream
        self.inputs = []
        for k in range(n_in):
            c = torch.empty(R + 4, dtype=torch.int32, device=dev)
            m = torch.empty(R + 4, dtype=torch.int32, device=dev)
            a.synth_requests_dev(w["dist"], w["seed"], k * R, R, c.data_ptr(), m.data_ptr(), sh)
            ok = (c >= 0) & (c <= 127) & (m >= 0) & (m <= MEM_MAX)
            self.inputs.append((c, m, torch.where(ok, (c << 18) | m, torch.full_like(c, -1))))
        self.outs = {arm: [(torch.empty(R + 16, dtype=torch.int32 if arm == "int32" else torch.int8, device=dev),
                            torch.empty(2 * self.D, dtype=torch.int64, device=dev),
                            torch.empty(3 * self.D, dtype=torch.int32, device=dev)) for _ in range(CALLS)]
                     for arm in ARMS + GRID_ARMS}
        torch.cuda.synchronize()
        self.expect = None

    def reset(self, arm):
        for i, dl, t in self.outs[arm]:
            i.fill_(-9)
            dl.fill_(-1)
            t.fill_(-7)

    def keep_expect(self):
        """the int32 arm's outputs after its eager pass: what every arm must give"""
        self.expect = [(i[:self.R].clone(), dl.clone(), t.clone()) for i, dl, t in self.outs["int32"]]

    def equal(self, arm):
        ok = True
        for (i, dl, t), (ei, edl, et) in zip(self.outs[arm], self.expect):
            ok &= bool(torch.equal(i[:self.R].to(torch.int32), ei)) and bool(torch.equal(dl, edl)) and bool(torch.equal(t, et))
        return ok


def region(alloc, sh, arm, ready):
    def fn(st):
        for k in range(CALLS):
            c, m, words = sh.inputs[k % len(sh.inputs)]
            i, dl, t = (x.data_ptr() for x in sh.outs[arm][k])
            if arm == "int32":
                alloc.bestfit_dev(c.data_ptr(), m.data_ptr(), sh.R, i, dl, t, False, st.cuda_stream, ready)
            else:
                alloc.bestfit_packed_dev(words.data_ptr(), sh.R, i, dl, t, st.cuda_stream, inputs_ready=ready)
    return fn


def graph_of(fn):
    """fn(stream) run once eagerly (occupancy, lookup tables), then captured"""
    st = torch.cuda.current_stream()
    fn(st)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    cap = torch.cuda.Stream()
    cap.wait_stream(st)
    with torch.cuda.stream(cap):
        with torch.cuda.graph(g, stream=cap):
            fn(cap)
    st.wait_stream(cap)
    torch.cuda.synchronize()
    return g


def timed(sh, graphs, reps):
    st = torch.cuda.current_stream()
    ts = {arm: [] for arm in graphs}
    equal = {arm: True for arm in graphs}
    for _ in range(reps):
        for arm, g in graphs.items():
            sh.reset(arm)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(st)
            g.replay()
            e1.record(st)
            torch.cuda.synchronize()
            ts[arm].append(e0.elapsed_time(e1) * 1e3 / CALLS)
            equal[arm] &= sh.equal(arm)
    out = {arm: {"us_median": float(np.median(x)), "us_min": float(np.min(x)), "us_max": float(np.max(x))} for arm, x in ts.items()}
    out["outputs_equal_every_rep"] = all(equal.values())
    return out


def fresh_alloc(rpt):
    """a context whose scans use `rpt` rows per thread (EGPU_ROWS_PER_THREAD, read when the context is created)"""
    os.environ["EGPU_ROWS_PER_THREAD"] = str(rpt)
    try:
        return e.BestFitAllocator(0)
    finally:
        os.environ.pop("EGPU_ROWS_PER_THREAD", None)


def group_grid(auto, reps):
    """the rows-per-thread rule of the packed snapshot scan: the shipped rule against half and twice it"""
    out = []
    for wname in ("cfg3", "cfg4"):
        sh = Shape(auto, wname, 1 << 20)
        auto.set_table(sh.w["free_core"], sh.w["free_mem"])
        region(auto, sh, "int32", False)(torch.cuda.current_stream())
        torch.cuda.synchronize()
        sh.keep_expect()
        for mode, ready in (("lone", False), ("pipelined", True)):
            rpt = SHIPPED_RPT[wname, ready]
            half, double = fresh_alloc(rpt // 2), fresh_alloc(2 * rpt)
            try:
                for a in (half, double):
                    a.set_table(sh.w["free_core"], sh.w["free_mem"])
                graphs = {"packed": graph_of(region(auto, sh, "packed", ready)),
                          "half": graph_of(region(half, sh, "half", ready)),
                          "double": graph_of(region(double, sh, "double", ready))}
                r = {"shape": f"{wname} D = {sh.D} R = {1 << 20}", "mode": mode, "rpt": {"packed": rpt, "half": rpt // 2, "double": 2 * rpt},
                     **timed(sh, graphs, reps)}
                out.append(r)
                print(f"grid {r['shape']:28s} {mode:9s} rpt {rpt:3d} {r['packed']['us_median']:8.2f} [{r['packed']['us_min']:.2f}, "
                      f"{r['packed']['us_max']:.2f}]  rpt {rpt // 2:3d} {r['half']['us_median']:8.2f} [{r['half']['us_min']:.2f}, "
                      f"{r['half']['us_max']:.2f}]  rpt {2 * rpt:3d} {r['double']['us_median']:8.2f} [{r['double']['us_min']:.2f}, "
                      f"{r['double']['us_max']:.2f}] us/call  equal {r['outputs_equal_every_rep']}", flush=True)
                del graphs
            finally:
                half.close()
                double.close()
        del sh
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=31)
    ap.add_argument("--json")
    args = ap.parse_args()
    res = {"gpu": card(), "reps": args.reps, "calls_per_graph": CALLS, "shapes": []}
    print(f"card, power limit: {res['gpu']}", flush=True)
    auto, grid = e.BestFitAllocator(0), e.BestFitAllocator(0)
    try:
        grid.set_variant(e.VARIANT_GRID)
        res["grid_rule"] = group_grid(auto, args.reps)
        for wname, R in SHAPES:
            sh = Shape(auto, wname, R)
            for alloc in (auto, grid):
                alloc.set_table(sh.w["free_core"], sh.w["free_mem"])
            for mode, ready in (("lone", False), ("pipelined", True)):
                graphs = {arm: graph_of(region(grid if arm == "chunk" else auto, sh, arm, ready)) for arm in ("int32", "packed", "chunk")}
                if sh.expect is None:
                    sh.keep_expect()
                r = {"shape": f"{wname} D = {sh.D} R = {R}", "mode": mode, **timed(sh, graphs, args.reps)}
                res["shapes"].append(r)
                print(f"{r['shape']:28s} {mode:9s} packed {r['packed']['us_median']:9.2f} [{r['packed']['us_min']:.2f}, "
                      f"{r['packed']['us_max']:.2f}]  chunk {r['chunk']['us_median']:9.2f} [{r['chunk']['us_min']:.2f}, "
                      f"{r['chunk']['us_max']:.2f}]  int32 {r['int32']['us_median']:9.2f} [{r['int32']['us_min']:.2f}, "
                      f"{r['int32']['us_max']:.2f}] us/call  equal {r['outputs_equal_every_rep']}", flush=True)
                del graphs
            del sh
            torch.cuda.empty_cache()
    finally:
        auto.close()
        grid.close()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
