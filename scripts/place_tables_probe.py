"""Probe (one GPU) of egpu::place_tables (DESIGN.md §2.11): P pending requests placed on N node tables by best-fit
rounds to the fixed point in one launch, next to what a caller does without it, the arms alternating in one run.

    python scripts/place_tables_probe.py [--reps N] [--warmup N] [--json PATH]

Shapes (seeded):
  N5000_D8_P1024    5 000 tables x D = 8, random free capacity, 1 024 random requests;
  N512_D64_P8192    512 tables x D = 64, random free capacity, 8 192 random requests;
  contended         64 tables x D = 8, every device whole (100 / 81 559), 512 identical whole-card replicas: every
                    replica ranks the same device first, so each round commits one of them and the launch runs
                    one round per device (the rounds rule's worst case, min(P, sum of d_valid) rounds).
Arms, per repetition:
  op_x20      20 calls of the raw operator (torch.ops.egpu.place_tables, no data checks) back to back, CUDA events
              around all 20, per call;
  op_x1       one call after a 128 MB write that evicts the 50 MB L2, CUDA events around the call;
  torch_loop  what a caller does today (tests/place_tables_np.place_torch): a torch loop of the raw
              egpu::bestfit_tables, a min over nodes, a stable sort by device, a segmented cumsum and a
              scatter-subtract, with a host sync per round; host clock around the loop and a final synchronize.
Every repetition checks that the operator's outputs equal the first repetition's and the torch loop's.  Medians of
--reps after --warmup.
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
import place_tables_np  # noqa: E402


def card():
    """card name and power limit, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def inputs(name):
    if name == "contended":
        N, D, P = 64, 8, 512
        return (np.full((N, D), 100, np.int32), np.full((N, D), 81_559, np.int32), np.full(N, D, np.int32),
                np.full(P, 100, np.int32), np.full(P, 81_559, np.int32))
    N, D, P = {"N5000_D8_P1024": (5000, 8, 1024), "N512_D64_P8192": (512, 64, 8192)}[name]
    g = np.random.default_rng(N + D)
    return (g.integers(0, 101, (N, D)).astype(np.int32), g.integers(0, 81_560, (N, D)).astype(np.int32),
            np.full(N, D, np.int32), g.integers(0, 101, P).astype(np.int32), g.integers(0, 81_560, P).astype(np.int32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("place_tables_probe: no CUDA device (timings are only taken on the GPU)")
    tables.load()
    dev = torch.device("cuda", 0)
    flush = torch.empty(128 << 20, dtype=torch.uint8, device=dev)
    result = {"card": card(), "reps": a.reps, "warmup": a.warmup, "shapes": {}}
    print(f"card: {result['card']}  medians of {a.reps} after {a.warmup} warm-up repetitions")
    op = torch.ops.egpu.place_tables
    for name in ("N5000_D8_P1024", "N512_D64_P8192", "contended"):
        host = inputs(name)
        args = [torch.from_numpy(x).to(dev) for x in host]
        tables.check_tables(*args[:3], op="place_tables")
        N, D = host[0].shape
        P = host[3].size
        t_x1, t_x20, t_loop = [], [], []
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        first = None
        for rep in range(a.warmup + a.reps):
            for _ in range(3):  # untimed: wakes a GPU the host-bound loop left idle
                op(*args)
            ev[2].record()
            for _ in range(20):
                op(*args)
            ev[3].record()
            flush.zero_()
            ev[0].record()
            out = op(*args)
            ev[1].record()
            torch.cuda.synchronize()
            x1, x20 = ev[0].elapsed_time(ev[1]) * 1e3, ev[2].elapsed_time(ev[3]) * 1e3 / 20
            t0 = time.perf_counter()
            loop = place_tables_np.place_torch(*args)
            torch.cuda.synchronize()
            tl = (time.perf_counter() - t0) * 1e6
            got = [t.cpu() for t in out]
            if got[4][1] != 0:
                sys.exit(f"place_tables_probe: {name}: a grid wait gave up")
            if first is None:
                first = got
            if not all(torch.equal(x, y) for x, y in zip(got, first)):
                sys.exit(f"place_tables_probe: {name}: repetition {rep} differs from the first")
            if not all(torch.equal(x, y.cpu()) for x, y in zip(got[:4], loop[:4])) or int(got[4][0]) != loop[4]:
                sys.exit(f"place_tables_probe: {name}: differs from the torch loop")
            if rep >= a.warmup:
                t_x1.append(x1)
                t_x20.append(x20)
                t_loop.append(tl)
        m1, m20, ml = statistics.median(t_x1), statistics.median(t_x20), statistics.median(t_loop)
        rounds = int(first[4][0])
        placed = int((first[0] >= 0).sum())
        r = {"N": N, "D": D, "P": P, "rounds": rounds, "placed": placed, "op_x1_us": m1, "op_x20_us_per_call": m20,
             "torch_loop_us": ml, "op_x1_min_max_us": [min(t_x1), max(t_x1)],
             "torch_loop_min_max_us": [min(t_loop), max(t_loop)], "loop_over_op_x1": ml / m1,
             "op_x1_us_per_round": m1 / max(rounds, 1), "torch_loop_us_per_round": ml / max(rounds, 1)}
        result["shapes"][name] = r
        print(f"{name}: {rounds} rounds, {placed} of {P} placed; op_x1 {m1:.1f} us (range {min(t_x1):.1f}-{max(t_x1):.1f}), "
              f"op_x20 {m20:.1f} us/call, torch loop {ml:.1f} us ({ml / m1:.1f}x); per round {m1 / max(rounds, 1):.2f} us "
              f"vs {ml / max(rounds, 1):.1f} us")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
