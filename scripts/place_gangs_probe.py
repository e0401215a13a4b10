"""Probe (one GPU) of egpu::place_gangs (DESIGN.md §2.13, §4.8): J gangs of pods placed in gang order on N node
tables, each kept or given back, in one launch, against the same rule as a torch loop of one place_pods call per gang.

    python scripts/place_gangs_probe.py [--reps N] [--warmup N] [--json PATH]

Workloads (seeded):
  A  N = 5 000 x D = 8, random free capacity, 1 024 pods of 1 to 4 random containers in 128 gangs of 1 to 16 pods,
     gang_min = size (a quarter of the containers ask for a whole card, so some gangs are given back);
  B  N = 512 x D = 64, random free capacity, 4 096 pods of 1 to 8 random containers in 256 gangs of 2 to 32 pods,
     half all or nothing and half with gang_min = size / 2;
  C  contended: N = 64 x D = 8 with two whole free devices per table (128 in all), 256 gangs of 2 to 4 pods of one
     whole-device container (core 100), all or nothing: most gangs find the tables full and are given back.
Arms, alternating in every repetition, CUDA events around each call:
  gangs        one call of the raw operator egpu::place_gangs;
  loop_eager   §2.13's rule as a torch loop around the raw egpu::place_pods, one call per gang, torch.where keeping
               or dropping each gang (tests/test_gpu_place_gangs.torch_loop), launched eagerly;
  loop_graph   the same loop captured once into a CUDA graph and replayed.
Every repetition checks that each arm's placement, placed counts and tables equal the first repetition's of the
gangs arm, and the first equals the numpy restatement (tests/place_gangs_np.py).  Medians of --reps after --warmup;
the card's name, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from elastic_gpu_agent_b200 import tables  # noqa: E402
import place_gangs_np  # noqa: E402
from test_gpu_place_gangs import torch_loop  # noqa: E402


def card():
    """card name, power limit and SM clock, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def cut(g, total, parts, lo, hi):
    """`parts` sizes in [lo, hi] summing to `total`"""
    sizes = np.full(parts, lo, np.int64)
    rest = total - lo * parts
    while rest > 0:
        i = int(g.integers(parts))
        if sizes[i] < hi:
            sizes[i] += 1
            rest -= 1
    return sizes


def inputs(name):
    if name == "C":
        N, D, J = 64, 8, 256
        g = np.random.default_rng(11)
        fc = np.zeros((N, D), np.int32)
        fc[:, :2] = 100
        gs = g.integers(2, 5, J)
        G = int(gs.sum())
        off = np.arange(G + 1, dtype=np.int32)
        return (fc, np.full((N, D), 81_559, np.int32), np.full(N, D, np.int32), np.full(G, 100, np.int32),
                np.full(G, 1024, np.int32), off, np.concatenate([[0], np.cumsum(gs)]).astype(np.int32),
                gs.astype(np.int32))
    N, D, G, hi_pod, J, lo_gang, hi_gang = {"A": (5000, 8, 1024, 4, 128, 1, 16),
                                            "B": (512, 64, 4096, 8, 256, 2, 32)}[name]
    g = np.random.default_rng(N + D + G)
    off = np.concatenate([[0], np.cumsum(g.integers(1, hi_pod + 1, G))]).astype(np.int32)
    P = int(off[-1])
    rc = g.integers(0, 101, P).astype(np.int32)
    if name == "A":
        rc[::4] = 100
    gs = cut(g, G, J, lo_gang, hi_gang)
    gmin = gs if name == "A" else np.where(np.arange(J) % 2 == 0, gs, np.maximum(1, gs // 2))
    return (g.integers(0, 101, (N, D)).astype(np.int32), g.integers(0, 81_560, (N, D)).astype(np.int32),
            np.full(N, D, np.int32), rc, g.integers(0, 81_560, P).astype(np.int32), off,
            np.concatenate([[0], np.cumsum(gs)]).astype(np.int32), gmin.astype(np.int32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("place_gangs_probe: no CUDA device (timings are only taken on the GPU)")
    tables.load()
    dev = torch.device("cuda", 0)
    result = {"card": card(), "reps": a.reps, "warmup": a.warmup, "workloads": {}}
    print(f"card (name, power limit, SM clock, max SM clock): {result['card']}  medians of {a.reps} after {a.warmup} "
          f"warm-up repetitions")
    gangs_op, pods_op = torch.ops.egpu.place_gangs, torch.ops.egpu.place_pods
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for name in ("A", "B", "C"):
        host = inputs(name)
        args = [torch.from_numpy(x).to(dev) for x in host]
        tables.check_tables(*args[:3], op="place_gangs")
        tables.check_pods(args[5], host[3].size, op="place_gangs")
        tables.check_gangs(args[6], args[7], host[5].size - 1)
        N, D = host[0].shape
        P, G, J = host[3].size, host[5].size - 1, host[6].size - 1
        exp = place_gangs_np.place(*host)

        def loop():
            return torch_loop(pods_op, args, host[5], host[6])

        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            loop()  # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            graph_out = loop()
        arms = {"gangs": lambda: gangs_op(*args), "loop_eager": loop,
                "loop_graph": lambda: (graph.replay(), graph_out)[1]}
        times = {k: [] for k in arms}
        first = None
        loop_rounds = None
        for rep in range(a.warmup + a.reps):
            for arm, fn in arms.items():
                for _ in range(2):  # untimed: wakes a GPU the previous arm may have left idle
                    fn()
                torch.cuda.synchronize()
                ev[0].record()
                out = fn()
                ev[1].record()
                torch.cuda.synchronize()
                got = [t.cpu() for t in out]
                if arm == "gangs":
                    if got[5][1] != 0 or got[5][2] != 0:
                        sys.exit(f"place_gangs_probe: {name}: info {got[5].tolist()}")
                    if first is None:
                        first = got
                        if not all(np.array_equal(x.numpy(), y) for x, y in zip(got[:5], exp[:5])) or \
                                got[5].tolist() != exp[5]:
                            sys.exit(f"place_gangs_probe: {name}: differs from the restatement")
                else:
                    loop_rounds = int(got[5][0])
                    if got[5][1] != 0:
                        sys.exit(f"place_gangs_probe: {name}: {arm}: a wait gave up")
                if not all(torch.equal(x, y) for x, y in zip(got[:5], first[:5])):
                    sys.exit(f"place_gangs_probe: {name}: {arm}: repetition {rep} differs from the first")
                if rep >= a.warmup:
                    times[arm].append(ev[0].elapsed_time(ev[1]) * 1e3)
        med = {k: statistics.median(v) for k, v in times.items()}
        placed = first[2].numpy()
        r = {"N": N, "D": D, "P": P, "G": G, "J": J, "rounds": int(first[5][0]), "loop_rounds": loop_rounds,
             "gangs_given_back": int((placed == 0).sum()), "pods_placed": int((first[0] >= 0).sum()),
             **{f"{k}_us": v for k, v in med.items()}, **{f"{k}_min_max_us": [min(v), max(v)] for k, v in times.items()}}
        result["workloads"][name] = r
        print(f"{name}: N {N} D {D} P {P} G {G} J {J}: {r['rounds']} rounds (loop {loop_rounds}), "
              f"{r['gangs_given_back']} of {J} gangs given back, {r['pods_placed']} pods placed; "
              + ", ".join(f"{k} {med[k]:.1f} us (range {min(times[k]):.1f}-{max(times[k]):.1f})" for k in arms)
              + f"; loop_graph / gangs {med['loop_graph'] / med['gangs']:.2f}x")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
