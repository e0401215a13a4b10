"""A/B probe (one GPU, world 1: the context attached to itself): the sharded calls on int32 arrays against the same
requests as packed words (EGPU_F_PACKED on egpu_bestfit_batch_shard_dev, _shard_lag_dev and _shard_prefix_dev), int32
and packed alternating in one run.  Checks in the same run that the packed indices, demand sums and table' equal the
int32 ones.

    python scripts/packed_shard_probe.py [--reps N] [--only GROUP] [--json PATH]

Every region is captured once in a CUDA graph and replayed --reps times (graphs of the arms in turn, CUDA events on
the launching stream, a device synchronisation around every replay); the numbers are medians.  Non-committing calls
only, so every replay computes the same thing.  Groups:

  steps   20 sharded steps of 1 M rows (cfg3: D = 8, register scan; cfg4: D = 64, lookup scan) over a ring of 20
          buffer sets (100 MB of packed words, twice the 50 MB L2): EGPU_F_INPUTS_READY scans on one stream and one
          apply launch on a second ("apply"), or the lag-2 form with its tail flush ("lag2").  us per step.
  prefix  one sharded prefix-commit (two exchange steps) of 1 M rows at D = 8 and D = 64, and 16 Mi + 1 rows at D = 64.
  grid    the rows-per-thread rule of the packed sharded scan: the int32 rule (8 rows per thread lone, 32 in the
          lookup scan, 48 pipelined) against twice that, through EGPU_ROWS_PER_THREAD in contexts of their own, and
          the rule the library ships (a context without the override); 20 steps of 1 M rows, "lone" = fully ordered
          scans, "pipelined" = EGPU_F_INPUTS_READY.  us per step.

World 1 measures the scans and the exchange protocol on one card; it says nothing about NVLink traffic between ranks.
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
STEPS = 20
R_STEP = 1 << 20
WORKLOADS = {"D8": "cfg3", "D64_lut": "cfg4"}


def card():
    """card name and power limit, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def fresh_alloc(rpt=None):
    if rpt:
        os.environ["EGPU_ROWS_PER_THREAD"] = str(rpt)
    try:
        a = e.BestFitAllocator(0)
    finally:
        os.environ.pop("EGPU_ROWS_PER_THREAD", None)
    a.peer_attach(0, 1, [a.peer_export()])
    return a


class Ring:
    """n sets of R requests: int32 arrays, the same requests as words, and outputs of both formats"""

    def __init__(self, a, wname, R, n):
        w = e.synth.workload(wname)
        self.w, self.R, self.D = w, R, int(w["D"])
        dev = torch.device("cuda", 0)
        sh = torch.cuda.current_stream().cuda_stream
        self.sets = []
        for k in range(n):
            c = torch.empty(R + 4, dtype=torch.int32, device=dev)
            m = torch.empty(R + 4, dtype=torch.int32, device=dev)
            a.synth_requests_dev(w["dist"], w["seed"], k * R, R, c.data_ptr(), m.data_ptr(), sh)
            ok = (c >= 0) & (c <= 127) & (m >= 0) & (m <= MEM_MAX)
            words = torch.where(ok, (c << 18) | m, torch.full_like(c, -1))
            out = {tag: (torch.full((R + 16,), -9, dtype=torch.int32 if tag == "int32" else torch.int8, device=dev),
                         torch.zeros(2 * self.D, dtype=torch.int64, device=dev), torch.full((3 * self.D,), -7, dtype=torch.int32, device=dev))
                   for tag in ("int32", "packed")}
            self.sets.append((c, m, words, out))
        torch.cuda.synchronize()

    def equal(self):
        ok = True
        for c, m, words, out in self.sets:
            (i, dl, t), (i8, dl8, t8) = out["int32"], out["packed"]
            ok &= bool(torch.equal(i[:self.R], i8[:self.R].to(torch.int32))) and bool(torch.equal(dl, dl8)) and bool(torch.equal(t, t8))
        return ok


def scan(a, ring, tag, k, step, s, inputs_ready=False, lag=0, lagged=0):
    c, m, words, out = ring.sets[k]
    i, dl, _ = (x.data_ptr() for x in out[tag])
    R = ring.R
    if lag:
        if tag == "int32":
            a.bestfit_shard_lag_dev(c.data_ptr(), m.data_ptr(), R, i, dl, step, lag, lagged, s, inputs_ready)
        else:
            a.bestfit_shard_lag_packed_dev(words.data_ptr(), R, i, dl, step, lag, lagged, s, inputs_ready)
    elif tag == "int32":
        a.bestfit_shard_dev(c.data_ptr(), m.data_ptr(), R, i, dl, step, s, inputs_ready)
    else:
        a.bestfit_shard_packed_dev(words.data_ptr(), R, i, dl, step, s, inputs_ready)


def steps_region(a, ring, tag, form, inputs_ready, ap):
    """form "apply": K scans + one apply launch on `ap`; "lag2": K lagged scans + the tail flush"""
    tab = [ring.sets[k][3][tag][2].data_ptr() for k in range(STEPS)]

    def fn(st):
        if form == "apply":
            ap.wait_stream(st)
            for k in range(STEPS):
                scan(a, ring, tag, k, k, st.cuda_stream, inputs_ready)
            a.apply_peers_multi_dev(0, tab, False, ap.cuda_stream)
            st.wait_stream(ap)
        else:
            for k in range(STEPS):
                scan(a, ring, tag, k, k, st.cuda_stream, inputs_ready, 2, tab[k - 2] if k >= 2 else 0)
            a.apply_peers_multi_dev(STEPS - 2, tab[STEPS - 2:], False, st.cuda_stream)
    return fn


def prefix_region(a, ring, tag):
    c, m, words, out = ring.sets[0]
    i, dl, t = (x.data_ptr() for x in out[tag])

    def fn(st):
        if tag == "int32":
            a.bestfit_shard_prefix_dev(c.data_ptr(), m.data_ptr(), ring.R, i, dl, t, 0, False, st.cuda_stream)
        else:
            a.bestfit_shard_prefix_packed_dev(words.data_ptr(), ring.R, i, dl, t, 0, False, st.cuda_stream)
    return fn


def graph_of(fn):
    """fn(stream) run once eagerly (scratch, occupancy, lookup tables), then captured"""
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


def timed(graphs, reps, per):
    """medians (and spread) of reps replays of every graph in turn, in us per `per`"""
    st = torch.cuda.current_stream()
    ts = {tag: [] for tag in graphs}
    for _ in range(reps):
        for tag, g in graphs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(st)
            g.replay()
            e1.record(st)
            torch.cuda.synchronize()
            ts[tag].append(e0.elapsed_time(e1) * 1e3 / per)
    return {tag: {"us_median": float(np.median(x)), "us_min": float(np.min(x)), "us_max": float(np.max(x))} for tag, x in ts.items()}


def set_table(allocs, ring):
    for a in allocs:
        a.set_variant(e.VARIANT_AUTO)
        a.set_table(ring.w["free_core"], ring.w["free_mem"])


def group_steps(a, reps):
    out = []
    ap = torch.cuda.Stream()
    for dname, wname in WORKLOADS.items():
        ring = Ring(a, wname, R_STEP, STEPS)
        for form in ("apply", "lag2"):
            set_table([a], ring)
            graphs = {tag: graph_of(steps_region(a, ring, tag, form, True, ap)) for tag in ("int32", "packed")}
            r = {"shape": f"{wname} {dname} 20 x 1 Mi, {form}", **timed(graphs, reps, STEPS), "outputs_equal": ring.equal()}
            out.append(r)
            print(f"steps  {r['shape']:32s} int32 {r['int32']['us_median']:8.2f} us/step  packed {r['packed']['us_median']:8.2f}  "
                  f"equal {r['outputs_equal']}", flush=True)
            del graphs
        del ring
        torch.cuda.empty_cache()
    return out


def group_prefix(a, reps):
    out = []
    for dname, wname, R in (("D8", "cfg3", 1 << 20), ("D64_lut", "cfg4", 1 << 20), ("D64_lut", "cfg4", (16 << 20) + 1)):
        ring = Ring(a, wname, R, 1)
        set_table([a], ring)
        graphs = {tag: graph_of(prefix_region(a, ring, tag)) for tag in ("int32", "packed")}
        deferred = int((ring.sets[0][3]["int32"][0][:R] == -2).sum())
        r = {"shape": f"{wname} {dname} R = {R}", **timed(graphs, reps, 1), "outputs_equal": ring.equal(), "deferred_rows": deferred}
        out.append(r)
        print(f"prefix {r['shape']:32s} int32 {r['int32']['us_median']:8.2f} us/call  packed {r['packed']['us_median']:8.2f}  "
              f"equal {r['outputs_equal']}  deferred {deferred}", flush=True)
        del graphs, ring
        torch.cuda.empty_cache()
    return out


def group_grid(a, reps):
    """packed at the int32 rule against packed at twice its rows per thread (and int32 at its rule, for reference)"""
    out = []
    ap = torch.cuda.Stream()
    for dname, wname in WORKLOADS.items():
        lut = wname == "cfg4"
        ring = Ring(a, wname, R_STEP, STEPS)
        for mode, ready in (("lone", False), ("pipelined", True)):
            rule = (32 if lut else 8) if not ready else 48
            a1, a2 = fresh_alloc(rule), fresh_alloc(2 * rule)
            try:
                set_table([a, a1, a2], ring)
                graphs = {"int32": graph_of(steps_region(a, ring, "int32", "apply", ready, ap)),
                          "packed": graph_of(steps_region(a, ring, "packed", "apply", ready, ap)),
                          f"packed_rpt{rule}": graph_of(steps_region(a1, ring, "packed", "apply", ready, ap)),
                          f"packed_rpt{2 * rule}": graph_of(steps_region(a2, ring, "packed", "apply", ready, ap))}
                eq = ring.equal()  # the last packed arm wrote the packed outputs
                r = {"shape": f"{wname} {dname} 20 x 1 Mi, {mode}", "rule": rule, **timed(graphs, reps, STEPS), "outputs_equal": eq}
                out.append(r)
                print(f"grid   {r['shape']:32s} int32 {r['int32']['us_median']:8.2f}  packed (shipped rule) {r['packed']['us_median']:8.2f}  "
                      f"packed@{rule} {r[f'packed_rpt{rule}']['us_median']:8.2f}  "
                      f"packed@{2 * rule} {r[f'packed_rpt{2 * rule}']['us_median']:8.2f} us/step  equal {eq}", flush=True)
                del graphs
            finally:
                a1.close()
                a2.close()
        del ring
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=101)
    ap.add_argument("--only", action="append", choices=["steps", "prefix", "grid"])
    ap.add_argument("--json")
    args = ap.parse_args()
    res = {"gpu": card(), "reps": args.reps}
    print(f"card, power limit: {res['gpu']}", flush=True)
    a = fresh_alloc()
    try:
        for name, fn in (("steps", group_steps), ("prefix", group_prefix), ("grid", group_grid)):
            if not args.only or name in args.only:
                res[name] = fn(a, args.reps)
        res["peer_last_timeout"] = a.peer_last_timeout
    finally:
        a.close()
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
