"""Probe (one GPU) of egpu::preempt_gangs (DESIGN.md §2.15, §4.10): gangs placed in order on N node tables with
priority preemption that never cuts a running job below its minimum, in one launch, against the numpy restatement's
CPU time, a torch loop of preempt_pods calls and place_gangs.

    python scripts/preempt_gangs_probe.py [--reps N] [--warmup N] [--json PATH] [--only abcd] [--ref DIR]
                                          [--restatement-only]

Workloads (seeded, tests/test_preempt_gangs_cpu.random_case: every node's running pods consistent by construction,
about two thirds of them in running jobs of mixed minimums):
  a  N = 5 000 x D = 8, nearly full, 4 to 16 running pods per node, 128 pending gangs of 1 to 16 pods of mixed
     priority and minimum;
  b  the same at N = 512 x D = 64 with 256 gangs;
  c  a with no running job (R = 0): preempt_gangs against the loop of one raw preempt_pods call per gang
     (tests/test_gpu_preempt_gangs.torch_loop), eager and replayed from one CUDA graph, alternating;
  d  a with nothing evictable: preempt_gangs against place_gangs on the same inputs, alternating.
CUDA events around each call; medians of --reps after --warmup.  Every repetition's outputs are compared with the
restatement's (tests/preempt_gangs_np.py), computed once per workload and timed as CPU time.  The card's name, power
limit and SM clock are read in the same run.  The restatement takes minutes of CPU time per workload: --ref DIR keeps
its outputs and time per workload in DIR (read when present, written otherwise), and --restatement-only fills DIR on
a host without a GPU.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from elastic_gpu_agent_b200 import tables  # noqa: E402
import preempt_gangs_np  # noqa: E402
from test_gpu_preempt_gangs import torch_loop  # noqa: E402
from test_preempt_gangs_cpu import random_case  # noqa: E402


def card():
    """card name, power limit and SM clock, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def workload(name):
    if name == "b":
        return random_case(np.random.default_rng(2), 512, 64, 256, run_lo=4, run_hi=16, hi_gang=16, full=0.9)
    g = np.random.default_rng(1)
    a = random_case(g, 5000, 8, 128, run_lo=4, run_hi=16, hi_gang=16, full=0.9, R=0 if name == "c" else None)
    if name == "d":  # nothing evictable
        a[8][:] = -7
        a[13] = np.maximum(a[13], -7).astype(np.int32)
    return a


def timed(fn, reps, warmup, check):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for _ in range(warmup):
        fn()
    out = []
    for s, e in ev:
        s.record()
        r = fn()
        e.record()
        torch.cuda.synchronize()
        check(r)
        out.append(s.elapsed_time(e))
    return out


def alternate(arms, reps, warmup):
    """arms: {name: (fn, check)}, timed in turn, one call each per repetition"""
    times = {k: [] for k in arms}
    for _ in range(reps):
        for k, (fn, check) in arms.items():
            times[k] += timed(fn, 1, warmup if not times[k] else 0, check)
    return {k: statistics.median(v) for k, v in times.items()}, times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--only", default="abcd")
    ap.add_argument("--ref", default=None)
    ap.add_argument("--restatement-only", action="store_true")
    args = ap.parse_args()
    tables.load()
    result = {"card": "none" if args.restatement_only else card(), "reps": args.reps, "workloads": {}}
    for name in args.only:
        a = workload(name)
        path = os.path.join(args.ref, f"preempt_gangs_{name}.npz") if args.ref else None
        if path and os.path.exists(path):
            z = np.load(path)
            exp = [z[f"o{i}"] for i in range(6)] + [z["info"].tolist()]
            cpu_s = float(z["cpu_s"])
        else:
            t0 = time.perf_counter()
            exp = preempt_gangs_np.place(*a)
            cpu_s = time.perf_counter() - t0
            if path:
                os.makedirs(args.ref, exist_ok=True)
                np.savez(path, cpu_s=cpu_s, info=np.array(exp[6]), **{f"o{i}": exp[i] for i in range(6)})
        if args.restatement_only:
            print(name, "restatement", cpu_s, exp[6], flush=True)
            continue
        st = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in a]

        def check(out, exp=exp, n=7):
            for x, y in zip(out[:6], exp[:6]):
                assert np.array_equal(x.cpu().numpy(), y), "preempt_gangs differs from the restatement"
            if n == 7:
                assert out[6].tolist() == exp[6]

        pg = lambda: torch.ops.egpu.preempt_gangs(*st)  # noqa: E731
        row = {"cpu_restatement_s": cpu_s, "rounds": exp[6][0], "J": int(exp[2].size), "G": int(exp[0].size),
               "H": int(exp[3].size), "R": int(a[16].size), "placed": int((exp[0] >= 0).sum()),
               "evicted": int((exp[3] >= 0).sum()), "gangs_given_back": int((exp[2] == 0).sum())}
        arms = {"preempt_gangs": (pg, check)}
        if name == "c":
            loop_args = st[:6] + st[9:15]
            loop = lambda: torch_loop(loop_args, a[5], a[6], a[7], a[8])  # noqa: E731
            check_loop = lambda out: check(out, n=6)  # noqa: E731
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                loop()
            torch.cuda.current_stream().wait_stream(s)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                g_out = loop()
            arms["loop_eager"] = (loop, check_loop)
            arms["loop_graph"] = (lambda: (graph.replay(), g_out)[1], check_loop)
        if name == "d":
            def check_pg(out, exp=exp):
                for x, y in zip(out[:5], exp[:3] + exp[4:6]):
                    assert np.array_equal(x.cpu().numpy(), y), "place_gangs differs from preempt_gangs"
            arms["place_gangs"] = (lambda: torch.ops.egpu.place_gangs(*st[:8]), check_pg)
        med, times = alternate(arms, args.reps, args.warmup)
        for k, v in med.items():
            row[f"{k}_ms"] = v
        row["preempt_gangs_ms_min_max"] = [min(times["preempt_gangs"]), max(times["preempt_gangs"])]
        result["workloads"][name] = row
        print(name, json.dumps(row), flush=True)
    print(json.dumps(result))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
