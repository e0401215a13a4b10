"""A/B probe (one GPU): K batches as K pipelined single-batch launches in a CUDA graph vs as
multi-batch launches, median of 31 replays each.  python scripts/multi_probe.py [workload] [K]"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import elastic_gpu_agent_b200 as e  # noqa: E402

args = [x for x in sys.argv[1:] if not x.startswith("--")]
ONLY_MULTI = "--only-multi" in sys.argv  # for ncu: nothing but a few multi-batch launches
name = args[0] if len(args) > 0 else "cfg3_1m"
K = int(args[1]) if len(args) > 1 else 20
w = e.synth.workload(name)
D, R = int(w["D"]), int(w["R"])
dev = torch.device("cuda", 0)
a = e.BestFitAllocator(0)
a.set_table(w["free_core"], w["free_mem"])
st = torch.cuda.Stream()
torch.cuda.set_stream(st)
sh = st.cuda_stream
nb = max(32, K) if R <= (1 << 20) else 2
ring = []
for b in range(nb):
    c = torch.empty(R, dtype=torch.int32, device=dev)
    m = torch.empty(R, dtype=torch.int32, device=dev)
    a.synth_requests_dev(w["dist"], w["seed"], b * R, R, c.data_ptr(), m.data_ptr(), sh)
    ring.append((c, m, torch.empty(R, dtype=torch.int32, device=dev), torch.zeros(2 * D, dtype=torch.int64, device=dev),
                 torch.zeros(3 * D, dtype=torch.int32, device=dev)))
torch.cuda.synchronize()


def tup(k):
    c, m, i, dl, to = ring[k % nb]
    return (c.data_ptr(), m.data_ptr(), R, i.data_ptr(), dl.data_ptr(), to.data_ptr())


def graph_of(fn):
    g = torch.cuda.CUDAGraph()
    cap = torch.cuda.Stream()
    cap.wait_stream(st)
    fn(sh)
    torch.cuda.synchronize()
    with torch.cuda.stream(cap):
        with torch.cuda.graph(g, stream=cap):
            fn(cap.cuda_stream)
    st.wait_stream(cap)
    g.replay()
    torch.cuda.synchronize()
    return g


def timed(g, reps=31):
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.gate_dev(sh)      # nothing below starts before the host has enqueued all of it
        e0.record(st)
        g.replay()
        e1.record(st)
        a.gate_open()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / K)
    ts = np.array(ts)
    return {"us_per_batch_median": float(np.median(ts)), "min": float(ts.min()), "max": float(ts.max())}


def singles(s):
    for k in range(K):
        t = tup(k)
        a.bestfit_dev(t[0], t[1], R, t[3], t[4], t[5], False, s, inputs_ready=True)


def multi(chunk):
    arrs = [a.make_batches([tup(k) for k in range(k0, min(K, k0 + chunk))]) for k0 in range(0, K, chunk)]

    def f(s):
        for arr in arrs:
            a.bestfit_batches_dev(arr, s, inputs_ready=True)
    return f


def timed_eager(fn, reps=31):
    """the same launches without a CUDA graph (a 20-step region is one or two launches)"""
    ts = []
    for _ in range(3):
        fn(sh)
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.gate_dev(sh)
        e0.record(st)
        fn(sh)
        e1.record(st)
        a.gate_open()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / K)
    ts = np.array(ts)
    return {"us_per_batch_median": float(np.median(ts)), "min": float(ts.min()), "max": float(ts.max())}


if ONLY_MULTI:
    f = multi(min(K, 64, nb))
    for _ in range(3):
        f(sh)
    torch.cuda.synchronize()
    a.close()
    sys.exit(0)

peak = 3350.0  # GB/s, H100 SXM data sheet
out = {"workload": name, "K": K, "D": D, "R": R, "env": {k: v for k, v in os.environ.items() if k.startswith("EGPU_")}}
r = timed(graph_of(singles))
out["single_launches"] = r
for chunk in sorted({min(K, 64, nb), min(K, 10, nb), min(K, 32, nb), 1}, reverse=True):
    r = timed(graph_of(multi(chunk)))
    out[f"multi_chunk{chunk}"] = r
out["multi_eager"] = timed_eager(multi(min(K, 64, nb)))
for k, v in out.items():
    if isinstance(v, dict) and "us_per_batch_median" in v:
        v["frac_of_hbm_peak"] = (12 * R + 32 * D) / (v["us_per_batch_median"] * 1e-6) / 1e9 / peak
print(json.dumps(out))
a.close()
