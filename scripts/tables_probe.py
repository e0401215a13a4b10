"""Probe (one GPU) of egpu::bestfit_tables (DESIGN.md §2.10): P pending requests scored against N node tables in one
launch, next to what a caller does without it, N egpu_bestfit_query calls, the arms alternating in one run.

    python scripts/tables_probe.py [--reps N] [--warmup N] [--json PATH]

Shapes: N = 5 000 tables x D = 8 x P = 1 024 requests, and N = 512 x D = 64 x P = 8 192 (every table full width,
d_valid = D; seeded random tables and requests; the probe prints the share of feasible pairs).  Arms, per repetition:
  op_x20    20 calls of the raw operator (torch.ops.egpu.bestfit_tables, no data checks) back to back, CUDA events
            around all 20, per call: the rate of a loop that rescores every tick.  20 untimed calls come first: a GPU
            left idle for tens of milliseconds (as the host-bound query arm leaves it) runs its first kernels several
            times slower (about 145 us instead of 17 us for one call at N = 5 000 on an H100 80GB HBM3);
  op_x1     then one call after a 128 MB write that evicts the 50 MB L2, CUDA events around the call on the current
            stream;
  query_xN  N egpu_bestfit_query calls on one context, one per table, host arrays, host clock (the call returns when
            its indices are on the host).
Every repetition checks the operator's indices against the queries' for every table.  Medians of --reps after
--warmup.  "GB/s (algorithmic)" is the bytes the call must move (5 per pair written: int8 index and int32 key; 8 per
table row and 4 per table read; 8 per request read) over the median op_x1 time, beside the H100 SXM data sheet's
3.35 TB/s; it is not an achieved-bandwidth measurement.
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

import torch  # noqa: E402

import elastic_gpu_agent_b200 as e  # noqa: E402
from elastic_gpu_agent_b200 import tables  # noqa: E402

MEM_MAX = (1 << 18) - 1
SHAPES = [("N5000_D8_P1024", 5000, 8, 1024), ("N512_D64_P8192", 512, 64, 8192)]
DATASHEET_GBS = 3350.0


def card():
    """card name and power limit, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def inputs(N, D, P, seed):
    g = np.random.default_rng(seed)
    fc = g.integers(0, 101, (N, D)).astype(np.int32)
    fm = g.integers(0, 81_560, (N, D)).astype(np.int32)
    rc = g.integers(0, 101, P).astype(np.int32)
    rm = g.integers(0, 81_560, P).astype(np.int32)
    return fc, fm, np.full(N, D, np.int32), rc, rm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tables_probe: no CUDA device (timings are only taken on the GPU)")
    tables.load()
    dev = torch.device("cuda", 0)
    flush = torch.empty(128 << 20, dtype=torch.uint8, device=dev)
    result = {"card": card(), "reps": a.reps, "warmup": a.warmup, "shapes": {}}
    print(f"card: {result['card']}  medians of {a.reps} after {a.warmup} warm-up repetitions")
    with e.BestFitAllocator(0) as ctx:
        for name, N, D, P in SHAPES:
            fc, fm, dv, rc, rm = inputs(N, D, P, seed=N + D)
            args = [torch.from_numpy(x).to(dev) for x in (fc, fm, dv, rc, rm)]
            tables.check_tables(*args[:3])
            ctx.set_table(fc[0], fm[0])
            op = torch.ops.egpu.bestfit_tables
            t_x1, t_x20, t_q = [], [], []
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            for rep in range(a.warmup + a.reps):
                for _ in range(20):  # untimed: wakes the GPU the query arm left idle
                    op(*args)
                ev[2].record()
                for _ in range(20):
                    op(*args)
                ev[3].record()
                flush.zero_()
                ev[0].record()
                idx, key = op(*args)
                ev[1].record()
                torch.cuda.synchronize()
                x1, x20 = ev[0].elapsed_time(ev[1]) * 1e3, ev[2].elapsed_time(ev[3]) * 1e3 / 20
                t0 = time.perf_counter()
                q = [ctx.query(fc[n], fm[n], rc, rm) for n in range(N)]
                tq = (time.perf_counter() - t0) * 1e6
                got = idx.cpu().numpy()
                for n in range(N):
                    if not np.array_equal(got[n], q[n]):
                        sys.exit(f"tables_probe: {name}: table {n} differs from egpu_bestfit_query")
                if rep >= a.warmup:
                    t_x1.append(x1)
                    t_x20.append(x20)
                    t_q.append(tq)
            out_bytes = 5 * N * P
            alg_bytes = out_bytes + 8 * N * D + 4 * N + 8 * P
            m1, m20, mq = statistics.median(t_x1), statistics.median(t_x20), statistics.median(t_q)
            gbs = alg_bytes / (m1 * 1e-6) / 1e9
            feas = float((idx >= 0).float().mean())
            r = {"N": N, "D": D, "P": P, "op_x1_us": m1, "op_x20_us_per_call": m20, "query_xN_us": mq,
                 "op_x1_min_max_us": [min(t_x1), max(t_x1)], "query_xN_min_max_us": [min(t_q), max(t_q)],
                 "out_bytes": out_bytes, "alg_bytes": alg_bytes, "alg_gbs": gbs, "of_datasheet": gbs / DATASHEET_GBS,
                 "feasible_pairs": feas, "query_over_op_x1": mq / m1}
            result["shapes"][name] = r
            print(f"{name}: op_x1 {m1:.1f} us (range {min(t_x1):.1f}-{max(t_x1):.1f}), op_x20 {m20:.1f} us/call, "
                  f"{N} queries {mq / 1e3:.1f} ms ({mq / m1:.0f}x); out {out_bytes / 1e6:.1f} MB, "
                  f"{gbs:.0f} GB/s algorithmic = {gbs / DATASHEET_GBS:.2f} of 3.35 TB/s; {feas:.2f} of pairs feasible")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
