"""Probe (one GPU) of egpu::preempt_pods (DESIGN.md §2.14, §4.9): pods placed on N node tables with priority
preemption of running pods, in one launch, against the numpy restatement's CPU time and against place_pods.

    python scripts/preempt_pods_probe.py [--reps N] [--warmup N] [--json PATH]

Workloads (seeded, tests/test_preempt_pods_cpu.random_case: every node's running pods consistent by construction):
  A  N = 5 000 x D = 8, nearly full (most of what the running pods leave is held), 4 to 16 running pods per node of
     1 to 4 containers and mixed priority, 256 pending pods of 1 to 4 containers, all above most running pods;
  B  N = 512 x D = 64, 32 to 128 running pods per node, 1 024 pending pods of mixed priority;
  C  A's tables and pods with nothing evictable (no pending pod above any running pod): preempt_pods against
     place_pods on the same inputs, alternating, the cost of the generality.
CUDA events around each call of the raw operator; medians of --reps after --warmup.  Every repetition's outputs are
compared with the restatement's (tests/preempt_pods_np.py), computed once per workload and timed as CPU time.  The
card's name, power limit and SM clock are read in the same run.
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
import preempt_pods_np  # noqa: E402
from test_preempt_pods_cpu import random_case  # noqa: E402


def card():
    """card name, power limit and SM clock, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def workload(name):
    if name == "A":
        g = np.random.default_rng(1)
        a = random_case(g, 5000, 8, 256, run_lo=4, run_hi=16, full=0.97)
    else:
        g = np.random.default_rng(2)
        a = random_case(g, 512, 64, 1024, run_lo=32, run_hi=128, hi_pod=4, full=0.3)
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    tables.load()
    result = {"card": card(), "reps": args.reps, "workloads": {}}
    for name in ("A", "B", "C"):
        a = workload("A" if name == "C" else name)
        if name == "C":  # nothing evictable
            a[6][:] = -7
            a[11] = np.maximum(a[11], -7).astype(np.int32)
        t0 = time.perf_counter()
        exp = preempt_pods_np.place(*a)
        cpu_s = time.perf_counter() - t0
        args_t = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in a]

        def check(out, exp=exp):
            for x, y in zip(out[:5], exp[:5]):
                assert np.array_equal(x.cpu().numpy(), y), "preempt_pods differs from the restatement"
            assert out[5].tolist() == exp[5]

        pre = lambda: torch.ops.egpu.preempt_pods(*args_t)  # noqa: E731
        row = {"cpu_restatement_s": cpu_s, "rounds": exp[5][0], "placed": int((exp[0] >= 0).sum()),
               "evicted": int((exp[2] >= 0).sum()), "G": int(exp[0].size), "H": int(exp[2].size)}
        if name == "C":
            pp = lambda: torch.ops.egpu.place_pods(*args_t[:6])  # noqa: E731

            def check_pp(out, exp=exp):
                for x, y in zip(out[:4], exp[:2] + exp[3:5]):
                    assert np.array_equal(x.cpu().numpy(), y), "place_pods differs from preempt_pods"

            t_pre, t_pp = [], []
            for _ in range(args.reps):  # the arms alternate
                t_pre += timed(pre, 1, args.warmup if not t_pre else 0, check)
                t_pp += timed(pp, 1, args.warmup if not t_pp else 0, check_pp)
            row["place_pods_ms"] = statistics.median(t_pp)
        else:
            t_pre = timed(pre, args.reps, args.warmup, check)
        row["preempt_pods_ms"] = statistics.median(t_pre)
        row["preempt_pods_ms_min_max"] = [min(t_pre), max(t_pre)]
        result["workloads"][name] = row
        print(name, json.dumps(row), flush=True)
    print(json.dumps(result))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
