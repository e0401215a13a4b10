"""Probe (one GPU) of egpu::place_pods (DESIGN.md §2.12, §4.7): G pods placed whole on N node tables by best-fit
rounds to the fixed point in one launch, the arms alternating in one run.

    python scripts/place_pods_probe.py [--reps N] [--warmup N] [--json PATH]

Shapes (seeded):
  N5000_D8_G1024      5 000 tables x D = 8, random free capacity, 1 024 pods of 1 to 4 random containers;
  N512_D64_G4096      512 tables x D = 64, random free capacity, 4 096 pods of 1 to 8 random containers;
  single_N5000_D8     5 000 tables x D = 8, 1 024 pods of one container, next to egpu::place_tables on the same
                      requests: what the generality of the pod replay costs where place_tables answers the same;
  contended           64 tables x D = 8 with two whole free devices each, 256 pods of 2 to 4 whole-device
                      containers (100 core): most pods find a node only after the pods before them commit.
Arms, per repetition:
  op_x20      20 calls of the raw operator back to back, CUDA events around all 20, per call;
  op_x1       one call after a 128 MB write that evicts the 50 MB L2, CUDA events around the call;
  tables_*    the same two arms of egpu::place_tables (single_N5000_D8 only), alternating with place_pods.
Every repetition checks that the outputs equal the first repetition's; the first equals the numpy restatement
(tests/place_pods_np.py) and, for single_N5000_D8, place_tables.  The restatement's run is timed once per shape on
the host CPU: it is the host alternative, a CPU time, not a GPU one.  Medians of --reps after --warmup.
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
import place_pods_np  # noqa: E402


def card():
    """card name, power limit and SM clock, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def offsets(g, G, hi):
    return np.concatenate([[0], np.cumsum(g.integers(1, hi + 1, G))]).astype(np.int32)


def inputs(name):
    if name == "contended":
        N, D, G = 64, 8, 256
        fc = np.zeros((N, D), np.int32)
        fc[:, :2] = 100
        g = np.random.default_rng(7)
        off = offsets(g, G, 4)
        off[1:] = np.cumsum(np.maximum(np.diff(off), 2))  # 2 to 4 containers
        P = int(off[-1])
        return (fc, np.full((N, D), 81_559, np.int32), np.full(N, D, np.int32), np.full(P, 100, np.int32),
                np.full(P, 1024, np.int32), off)
    N, D, G, hi = {"N5000_D8_G1024": (5000, 8, 1024, 4), "N512_D64_G4096": (512, 64, 4096, 8),
                   "single_N5000_D8": (5000, 8, 1024, 1)}[name]
    g = np.random.default_rng(N + D + G)
    off = offsets(g, G, hi)
    P = int(off[-1])
    return (g.integers(0, 101, (N, D)).astype(np.int32), g.integers(0, 81_560, (N, D)).astype(np.int32),
            np.full(N, D, np.int32), g.integers(0, 101, P).astype(np.int32), g.integers(0, 81_560, P).astype(np.int32),
            off)


def timed(op, args, flush, ev):
    """(one call after an L2 flush, per call of 20 back to back) in microseconds, and the single call's outputs"""
    for _ in range(3):  # untimed: wakes a GPU the previous arm may have left idle
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
    return ev[0].elapsed_time(ev[1]) * 1e3, ev[2].elapsed_time(ev[3]) * 1e3 / 20, [t.cpu() for t in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("place_pods_probe: no CUDA device (timings are only taken on the GPU)")
    tables.load()
    dev = torch.device("cuda", 0)
    flush = torch.empty(128 << 20, dtype=torch.uint8, device=dev)
    result = {"card": card(), "reps": a.reps, "warmup": a.warmup, "shapes": {}}
    print(f"card (name, power limit, SM clock, max SM clock): {result['card']}  medians of {a.reps} after {a.warmup} "
          f"warm-up repetitions")
    pods_op, tables_op = torch.ops.egpu.place_pods, torch.ops.egpu.place_tables
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    for name in ("N5000_D8_G1024", "N512_D64_G4096", "single_N5000_D8", "contended"):
        host = inputs(name)
        args = [torch.from_numpy(x).to(dev) for x in host]
        tables.check_tables(*args[:3], op="place_pods")
        tables.check_pods(args[5], host[3].size)
        N, D = host[0].shape
        P, G = host[3].size, host[5].size - 1
        t0 = time.perf_counter()
        exp = place_pods_np.place(*host)
        cpu_s = time.perf_counter() - t0
        single = name.startswith("single")
        times = {"op_x1": [], "op_x20": [], "tables_x1": [], "tables_x20": []}
        first = None
        for rep in range(a.warmup + a.reps):
            x1, x20, got = timed(pods_op, args, flush, ev)
            if single:
                t1, t20, tab = timed(tables_op, args[:5], flush, ev)
                if not all(torch.equal(x, y) for x, y in zip(got[:4], tab[:4])) or got[4][0] != tab[4][0]:
                    sys.exit(f"place_pods_probe: {name}: repetition {rep} differs from place_tables")
            if got[4][1] != 0 or got[4][2] != 0:
                sys.exit(f"place_pods_probe: {name}: info {got[4].tolist()}")
            if first is None:
                first = got
                if not all(np.array_equal(x.numpy(), y) for x, y in zip(got[:4], exp[:4])) or got[4].tolist() != exp[4]:
                    sys.exit(f"place_pods_probe: {name}: differs from the restatement")
            if not all(torch.equal(x, y) for x, y in zip(got, first)):
                sys.exit(f"place_pods_probe: {name}: repetition {rep} differs from the first")
            if rep >= a.warmup:
                times["op_x1"].append(x1)
                times["op_x20"].append(x20)
                if single:
                    times["tables_x1"].append(t1)
                    times["tables_x20"].append(t20)
        med = {k: statistics.median(v) for k, v in times.items() if v}
        rounds, placed = int(first[4][0]), int((first[0] >= 0).sum())
        r = {"N": N, "D": D, "G": G, "P": P, "rounds": rounds, "placed_pods": placed, "cpu_restatement_s": cpu_s,
             **{f"{k}_us": v for k, v in med.items()},
             **{f"{k}_min_max_us": [min(v), max(v)] for k, v in times.items() if v}}
        result["shapes"][name] = r
        line = (f"{name}: N {N} D {D} G {G} P {P}: {rounds} rounds, {placed} of {G} pods placed; op_x1 {med['op_x1']:.1f} us "
                f"(range {min(times['op_x1']):.1f}-{max(times['op_x1']):.1f}), op_x20 {med['op_x20']:.1f} us/call")
        if single:
            line += (f"; place_tables x1 {med['tables_x1']:.1f} us, x20 {med['tables_x20']:.1f} us/call "
                     f"(place_pods / place_tables: {med['op_x1'] / med['tables_x1']:.2f}x, {med['op_x20'] / med['tables_x20']:.2f}x)")
        print(line + f"; numpy restatement on the host CPU {cpu_s * 1e3:.0f} ms")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
