"""Probe: a GC pass as EGPU_RESTORE_RELEASE against a full restore of the records that remain.

    python scripts/restore_release_probe.py [--reps N] [--warmup N] [--json PATH]

The node-scale record set of bench.py's next_rows: 96 gpu-memory containers of 4 Ki - 16 Ki IDs (934 k IDs,
9.7 MB of JSON) on 8 GPUs, with their symlinks.  A GC that finds k dead pods (k = 1 and 8) brings the table
back in one of two ways:

  release  egpu_table_restore(dead records, the node's links, RELEASE) on the table a full restore of all
           96 records installed (installed outside the timed region);
  restore  egpu_table_restore(the 96 - k remaining records, the node's links, INSTALL).

Both with and without EGPU_RESTORE_VERIFY.  The arms alternate in every repetition (their order swaps
from one repetition to the next), each timed with a host clock around the synchronous call; the dead pods
are drawn afresh every repetition.  Every repetition checks that the two installed tables, flags
included, are equal.  Medians of --reps (>= 15) after --warmup.  The card's name and power limit are read
in the same run.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import elastic_gpu_agent_b200 as e  # noqa: E402
from elastic_gpu_agent_b200 import restore  # noqa: E402
from oracle import restore_py  # noqa: E402


def card():
    """card name and power limit, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def node_set():
    """bench.py's next_rows set: the same seed, sizes and link targets"""
    rng = random.Random(11)
    sets = [["%d-%02d" % (c % 8, j) for j in rng.sample(range(183359), rng.choice([4096, 8192, 16384]))] for c in range(96)]
    recs, links = [], []
    for c, x in enumerate(sets):
        recs.append(restore_py.marshal_record("default", "pod-%d" % c, {"main": (x, restore_py.MEM)}))
        links.append(("elastic-gpu-%s-0" % restore_py.device_hash(x), "/dev/nvidia%d" % (c % 8)))
    return recs, links, sum(len(x) for x in sets)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert args.reps >= 15
    gpu = card()
    print("card:", gpu, flush=True)
    recs, links, n_ids = node_set()
    capc, capm = [100] * 8, [183359] * 8
    results = {"card": gpu, "records": len(recs), "ids": n_ids, "record_bytes": sum(len(v) for _, v in recs),
               "reps": args.reps, "warmup": args.warmup, "cases": {}}
    pick = np.random.default_rng(5)
    with e.BestFitAllocator(0) as a:
        for verify in (True, False):
            for k in (1, 8):
                times = {"release": [], "restore": []}
                for rep in range(args.warmup + args.reps):
                    dead = sorted(pick.choice(len(recs), k, replace=False).tolist())
                    gone = [recs[i] for i in dead]
                    left = [r for i, r in enumerate(recs) if i not in dead]
                    tables = {}
                    order = ("release", "restore") if rep % 2 == 0 else ("restore", "release")
                    for arm in order:
                        if arm == "release":
                            restore.restore_table(a, recs, links, capc, capm, verify=verify, install=True)
                            torch.cuda.synchronize()
                            t0 = time.perf_counter()
                            restore.restore_table(a, gone, links, capc, capm, verify=verify, release=True)
                            dt = time.perf_counter() - t0
                        else:
                            a.set_table(capc, capm)
                            t0 = time.perf_counter()
                            restore.restore_table(a, left, links, capc, capm, verify=verify, install=True)
                            dt = time.perf_counter() - t0
                        tables[arm] = [x.tolist() for x in a.table()]
                        if rep >= args.warmup:
                            times[arm].append(dt)
                    assert tables["release"] == tables["restore"], (verify, k, rep)
                med = {arm: 1e3 * float(np.median(v)) for arm, v in times.items()}
                span = {arm: (1e3 * min(v), 1e3 * max(v)) for arm, v in times.items()}
                name = "gc%d_%s" % (k, "verify" if verify else "no_verify")
                results["cases"][name] = {"dead_pods": k, "verify": verify, "release_ms": round(med["release"], 4),
                                          "restore_ms": round(med["restore"], 4),
                                          "release_ms_min_max": [round(x, 4) for x in span["release"]],
                                          "restore_ms_min_max": [round(x, 4) for x in span["restore"]],
                                          "speedup": round(med["restore"] / med["release"], 2), "tables_equal": True}
                print(f"{name:16s} release {med['release']:8.3f} ms [{span['release'][0]:.3f}, {span['release'][1]:.3f}]   "
                      f"full restore of the rest {med['restore']:8.3f} ms [{span['restore'][0]:.3f}, {span['restore'][1]:.3f}]   "
                      f"(x{med['restore'] / med['release']:.1f}; tables equal in all {args.warmup + args.reps} repetitions)",
                      flush=True)
    print(json.dumps(results))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
