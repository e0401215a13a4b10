"""Probe (one GPU, world 1: the context exchanges with itself): sharded rounds to the fixed point in one launch
(egpu_bestfit_batch_shard_prefix_dev with EGPU_F_PREFIX_COMMIT | EGPU_F_COMMIT | EGPU_F_ROUNDS | EGPU_F_DEVICE_ROUNDS)
against two other ways to the same answer, alternating in one run:

  shard    the new call;
  single   egpu_bestfit_batch_dev with EGPU_F_DEVICE_ROUNDS on the same rows: the one-GPU one-launch rounds, so
           shard - single is the cost of the exchange per round;
  loop     what a multi-GPU caller writes without the new call: egpu_bestfit_batch_shard_prefix_dev committing, then
           synchronise, count the deferred rows, compact them with torch and submit them again, until none is left.

    python scripts/shard_rounds_probe.py [--reps N] [--warmup N] [--json PATH]

Workloads (int32 rows): 1 Mi small requests (core <= 5, mem <= 2048) on the cfg3 table (D = 8, about 10 rounds),
the same on the cfg4 table (D = 64, lookup scan, about 64 rounds), and one 1 Ki batch on the cfg3 table (latency).
Every timed call ends in a synchronise, so the host clock around it measures it; shard and single are also timed
as CUDA-graph replays.  The table is reset by egpu_table_set before every call, outside the timed region; every
repetition checks that the three arms' indices, demand sums, table' and installed tables are equal.  Medians of
--reps (>= 15) repetitions after --warmup.  Multi-GPU is not measured here.
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

DR = L.F_PREFIX_COMMIT | L.F_COMMIT | L.F_ROUNDS | L.F_DEVICE_ROUNDS
# name -> (table, rows)
SHAPES = {
    "1Mi_cfg3_D8": ("cfg3", 1 << 20),
    "1Mi_cfg4_D64_lut": ("cfg4", 1 << 20),
    "1Ki_cfg3_D8": ("cfg3", 1 << 10),
}


def card():
    """card name and power limit, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def vp(x):
    return C.c_void_p(x)


class Outs:
    def __init__(self, R, D):
        self.idx = torch.empty(R + 4, dtype=torch.int32, device="cuda")
        self.delta = torch.empty(2 * D, dtype=torch.int64, device="cuda")
        self.tab = torch.empty(3 * D, dtype=torch.int32, device="cuda")

    def get(self, R):
        return self.idx[:R].cpu().numpy(), self.delta.cpu().numpy(), self.tab.cpu().numpy()


def run_shape(a, name, reps, warmup):
    wname, R = SHAPES[name]
    w = e.synth.workload(wname)
    fc, fm = np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32)
    D = fc.size
    a.set_variant(e.VARIANT_AUTO)
    lib, h = a._lib, a.handle
    st = torch.cuda.Stream()
    s = vp(st.cuda_stream)
    rc, rm = e.synth.requests(3, 5, R)
    rc, rm = np.minimum(rc, 5).astype(np.int32), np.minimum(rm, 2048).astype(np.int32)
    c, m = torch.from_numpy(rc).cuda(), torch.from_numpy(rm).cuda()
    outs = {arm: Outs(R, D) for arm in ("shard", "single", "loop")}
    rnd = Outs(R, D)  # the loop's per-round outputs
    rounds_seen = []

    def issue_shard():
        o = outs["shard"]
        code = lib.egpu_bestfit_batch_shard_prefix_dev(h, vp(c.data_ptr()), vp(m.data_ptr()), R, vp(o.idx.data_ptr()),
                                                       vp(o.delta.data_ptr()), vp(o.tab.data_ptr()), DR, 0, s)
        assert code == 0, lib.egpu_last_error(h).decode()

    def issue_single():
        o = outs["single"]
        code = lib.egpu_bestfit_batch_dev(h, vp(c.data_ptr()), vp(m.data_ptr()), R, vp(o.idx.data_ptr()), vp(o.delta.data_ptr()),
                                          vp(o.tab.data_ptr()), DR, s)
        assert code == 0, lib.egpu_last_error(h).decode()

    def issue_loop():
        o = outs["loop"]
        cur_c, cur_m, rows = c, m, None  # rows: the caller's row of each current row (None: all of them, in order)
        total = torch.zeros(2 * D, dtype=torch.int64, device="cuda")
        n, step, rounds = R, 0, 0
        while True:
            idx = o.idx if rows is None else rnd.idx
            code = lib.egpu_bestfit_batch_shard_prefix_dev(h, vp(cur_c.data_ptr()), vp(cur_m.data_ptr()), n, vp(idx.data_ptr()),
                                                           vp(rnd.delta.data_ptr()), vp(o.tab.data_ptr()),
                                                           L.F_PREFIX_COMMIT | L.F_COMMIT, step, s)
            assert code == 0, lib.egpu_last_error(h).decode()
            rounds += 1
            step += 2
            total += rnd.delta
            got = idx[:n]
            if rows is not None:
                o.idx[rows] = got
            deferred = got == -2
            left = int(deferred.sum().item())  # synchronises
            if left == 0:
                break
            keep = torch.nonzero(deferred).squeeze(1)
            cur_c, cur_m = cur_c[keep].contiguous(), cur_m[keep].contiguous()
            rows = keep if rows is None else rows[keep]
            n = left
        o.delta.copy_(total)
        rounds_seen.append(rounds)

    graphs = {}
    for arm, issue in (("shard", issue_shard), ("single", issue_single)):
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

    res = {"D": D, "rows": R}
    forms = {"eager": {"shard": issue_shard, "single": issue_single, "loop": issue_loop},
             "graph": {"shard": graphs["shard"].replay, "single": graphs["single"].replay}}
    for form, arms in forms.items():
        times = {arm: [] for arm in arms}
        for rep in range(warmup + reps):
            got = {}
            for arm, fn in arms.items():
                a.set_table(fc, fm)
                o = outs[arm]
                o.idx.fill_(-9), o.delta.fill_(-1), o.tab.fill_(-7)
                torch.cuda.synchronize()
                with torch.cuda.stream(st):
                    dt = timed(fn)
                got[arm] = outs[arm].get(R) + a.table()
                if rep >= warmup:
                    times[arm].append(dt)
            ref = got["shard"]
            for arm, g in got.items():
                assert all(np.array_equal(p, q) for p, q in zip(ref, g)), (name, form, rep, arm)
        assert a.peer_last_timeout == 0
        med = {arm: 1e3 * float(np.median(v)) for arm, v in times.items()}
        res[form] = {f"{arm}_ms": round(v, 4) for arm, v in med.items()}
        line = "  ".join(f"{arm} {v:9.4f} ms" for arm, v in med.items())
        print(f"{name:18s} {form:5s} {line}  (all {reps + warmup} repetitions equal)", flush=True)
    res["rounds"] = rounds_seen[-1]
    print(f"{name:18s} rounds {rounds_seen[-1]}", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
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
