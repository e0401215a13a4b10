"""Probe (one GPU) of sequential replay with release events (EGPU_EV_RELEASE): a GC-style stream next to the plain
churn of bench.py's cfg5 row, through the C ABI with host buffers (H2D, kernel, D2H), host clock around each call.

    python scripts/replay_release_probe.py [--reps N] [--warmup N] [--json PATH] [--churn-only]

Streams, 100 k events each, cfg5's table (D = 8, the two-warp kernel):
  cfg5_churn   synth.churn_events(5, 100 000): what bench.py times;
  gc_release   the same churn with about 10 % of its events turned into release events, each naming one of the
               placements a previous call made (device, EGPU_PACK_REQUEST(core, mem)), drawn with repetition: a
               placement's first hand-back is accepted when it fits the device's room, its repeats are refused.  The
               two-warp kernel is branch-free, so an accepted and a refused release cost the same.  The previous call
               is replayed before every repetition, untimed, so every repetition starts from the same table.
Each repetition re-installs the table (egpu_table_set, untimed) and checks the indices and the table against the
restatement of tests/replay_release_np.py once.  --churn-only times cfg5_churn alone, which a library without release
events can also run (EGPU_LIB_PATH selects one).  Medians of --reps after --warmup, and min / max beside them.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import elastic_gpu_agent_b200 as e  # noqa: E402


def card():
    """card name and power limit, read in the same run (read-only query)"""
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
    except OSError:
        out = ""
    return out.splitlines()[0] if out else "unknown"


def gc_stream(seed, E, fc, fm):
    """(placing call, GC-style stream): the churn of cfg5 with ~10 % of its events releasing earlier placements"""
    import replay_release_np as rr
    rng = np.random.default_rng(seed)
    k0, a0, b0 = e.synth.churn_events(seed + 1, 400)
    k0, a0, b0 = k0[k0 == 0], a0[k0 == 0], b0[k0 == 0]  # the placing call: ALLOCs only
    out0 = rr.replay(fc, fm, np.zeros(fc.size), k0, a0, b0)[0]
    _, dev, word = rr.releases_of(k0, a0, b0, out0)
    kind, a, b = (x.copy() for x in e.synth.churn_events(seed, E))
    rel = np.flatnonzero(rng.random(E) < 0.10)
    pick = rng.integers(0, dev.size, rel.size)
    kind[rel], a[rel], b[rel] = 3, dev[pick], word[pick]
    return (k0, a0, b0), (kind, a, b)


def timed(alloc, fc, fm, stream, pre, reps, warmup):
    ms = []
    for r in range(warmup + reps):
        alloc.set_table(fc, fm)
        if pre is not None:
            alloc.replay(*pre)
        t0 = time.perf_counter()
        out = alloc.replay(*stream)
        dt = time.perf_counter() - t0
        if r >= warmup:
            ms.append(1e3 * dt)
    a = np.array(ms)
    return out, {"ms_median": float(np.median(a)), "ms_min": float(a.min()), "ms_max": float(a.max()), "reps": reps,
                 "ns_per_event_median": float(np.median(a)) * 1e6 / len(stream[0])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default="")
    ap.add_argument("--churn-only", action="store_true")
    args = ap.parse_args()
    w = e.synth.workload("cfg5")
    fc, fm, E = np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32), int(w["R"])
    res = {"card": card(), "lib": os.environ.get("EGPU_LIB_PATH", "in-tree"), "D": int(w["D"]), "events": E}
    with e.BestFitAllocator(0) as alloc:
        churn = e.synth.churn_events(w["seed"], E)
        arms = [("cfg5_churn", None, churn)]
        if not args.churn_only:
            pre, gc = gc_stream(w["seed"], E, fc, fm)
            arms.append(("gc_release", pre, gc))
            res["gc_release_events"] = int((gc[0] == 3).sum())
        for name, pre, stream in arms:
            out, t = timed(alloc, fc, fm, stream, pre, args.reps, args.warmup)
            if not args.churn_only:
                import replay_release_np as rr
                f0, m0 = fc, fm
                if pre is not None:
                    _, f0, m0 = rr.replay(fc, fm, np.zeros(fc.size), *pre)
                want, w_fc, w_fm = rr.replay(f0, m0, np.zeros(fc.size), *stream)
                g_fc, g_fm, _ = alloc.table()
                t["exact"] = bool(np.array_equal(out, want) and np.array_equal(g_fc, w_fc) and np.array_equal(g_fm, w_fm))
                t["accepted_releases"] = int(((stream[0] == 3) & (out >= 0)).sum())
            res[name] = t
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
