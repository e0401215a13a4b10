"""Probe of the release over row shards (egpu_bestfit_batch_shard_prefix_dev with EGPU_F_RELEASE): what the exchange in
the last CTA adds to a release launch, and a sharded churn tick against the same tick with a host recompute.

    python scripts/shard_release_probe.py [--reps N] [--warmup N] [--json PATH]

World 1 (the context attached to itself), the arms alternating in one run, every shape warmed up first:
  single_x20 / shard_x20
          20 dry release launches (no EGPU_F_COMMIT: every repetition does the same work) replayed from a CUDA graph,
          each over its own copy of the rows, per launch; single = egpu_bestfit_batch_dev with EGPU_F_RELEASE, shard =
          the sharded call on the same rows (one exchange step each).  1 Mi rows, D = 8 and D = 64, int32 and packed.
          The difference is the cost of the push and pull in the last CTA;
  tick / tick_host (1 Mi rows, D = 8)
          a sharded churn tick replayed from a CUDA graph - sharded release of the rows the previous tick placed, then
          sharded rounds placing them again - against the same tick with the rows and indices copied to the host,
          np.bincount and egpu_table_set in place of the release; host clock to the end of a synchronise.
Every repetition checks the outputs: the sums and table' of both release arms against np.bincount, the indices and the
installed table after both ticks.  Medians of --reps after --warmup, with the lowest and highest repetition.  Several
GPUs: only with two GPUs in the machine would a world-2 figure mean anything; two processes on one GPU prove
correctness, not speed, so this probe reports "multi-GPU not measured" and measures world 1 only.
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

import torch  # noqa: E402

import elastic_gpu_agent_b200 as e  # noqa: E402

MEM_MAX = (1 << 18) - 1
R = 1 << 20


def card():
    """card name and power limit, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def rows_for(D, seed):
    """placed rows whose release fits: about 20 live rows per device, every 16th row one that holds nothing"""
    g = np.random.default_rng(seed)
    core, mem = np.zeros(R, np.int32), np.zeros(R, np.int32)
    idx = g.integers(0, D, R).astype(np.int32)
    live = g.permutation(R)[:20 * D]
    core[live], mem[live] = g.integers(0, 3, live.size), g.integers(0, 1001, live.size)
    idx[15::16] = -1
    return core, mem, idx


def host_sums(core, mem, idx, D):
    ok = (idx >= 0) & (idx < D) & (core >= 0) & (core <= 100) & (mem >= 0) & (mem <= MEM_MAX)
    return (np.bincount(idx[ok], weights=core[ok], minlength=D).astype(np.int64),
            np.bincount(idx[ok], weights=mem[ok], minlength=D).astype(np.int64))


def event_us(fn, stream):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    fn()
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b) * 1e3


def stats(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}


def run_launches(a, D, packed, reps, warmup):
    fc, fm = np.full(D, 10, np.int32), np.full(D, 1000, np.int32)
    a.set_table(fc, fm)
    st = torch.cuda.Stream()
    s = st.cuda_stream
    core, mem, idx = rows_for(D, D)
    bufs = []
    for _ in range(20):
        if packed:
            bufs.append((torch.from_numpy(a.pack_requests(core, mem).view(np.int32)).cuda(), None,
                         torch.from_numpy(idx.astype(np.int8)).cuda()))
        else:
            bufs.append((torch.from_numpy(core).cuda(), torch.from_numpy(mem).cuda(), torch.from_numpy(idx).cuda()))
    delta = torch.zeros(2 * D, dtype=torch.int64, device="cuda")
    tab = torch.zeros(3 * D, dtype=torch.int32, device="cuda")
    uc, um = host_sums(core, mem, idx, D)
    want = (np.concatenate([uc, um]), np.concatenate([fc + uc, fm + um, np.zeros(D, np.int64)]).astype(np.int32))

    def single(b):
        a.release_dev(b[0].data_ptr(), 0 if packed else b[1].data_ptr(), R, b[2].data_ptr(), delta.data_ptr(), tab.data_ptr(),
                      commit=False, packed=packed, stream=s)

    def shard(b, step):
        a.release_shard_dev(b[0].data_ptr(), 0 if packed else b[1].data_ptr(), R, b[2].data_ptr(), delta.data_ptr(), tab.data_ptr(),
                            step=step, commit=False, packed=packed, stream=s)

    with torch.cuda.stream(st):
        single(bufs[0])
        shard(bufs[0], 0)
    torch.cuda.synchronize()
    graphs = {}
    for arm in ("single_x20", "shard_x20"):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for k, b in enumerate(bufs):
                single(b) if arm == "single_x20" else shard(b, k)
        graphs[arm] = g
    t = {k: [] for k in graphs}
    for rep in range(warmup + reps):
        for arm in (("single_x20", "shard_x20") if rep % 2 == 0 else ("shard_x20", "single_x20")):
            delta.fill_(-1), tab.fill_(-7)
            us = event_us(graphs[arm].replay, torch.cuda.current_stream())
            assert np.array_equal(delta.cpu().numpy(), want[0]) and np.array_equal(tab.cpu().numpy(), want[1]), arm
            if rep >= warmup:
                t[arm].append(us / 20)
    assert a.release_refusals == 0
    return {k: stats(v) for k, v in t.items()}


def run_tick(a, D, packed, reps, warmup):
    """steady state: every tick releases the rows the previous tick placed and places the same rows again, so the
    indices and the table after a tick are the same every time, whichever arm ran it"""
    st = torch.cuda.Stream()
    s = st.cuda_stream
    w = e.synth.workload("cfg3")
    T = (np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32))
    rc, rm = e.synth.requests(3, 5, R)
    rc, rm = np.minimum(rc, 5).astype(np.int32), np.minimum(rm, 2048).astype(np.int32)
    c = torch.from_numpy(a.pack_requests(rc, rm).view(np.int32) if packed else rc).cuda()
    m = torch.from_numpy(rm).cuda()
    i = torch.empty(R + 16, dtype=torch.int8 if packed else torch.int32, device="cuda")

    def admit(step):
        a.bestfit_shard_rounds_dev(c.data_ptr(), 0 if packed else m.data_ptr(), R, i.data_ptr(), 0, 0, step, packed=packed, stream=s)

    def rel(step):
        a.release_shard_dev(c.data_ptr(), 0 if packed else m.data_ptr(), R, i.data_ptr(), step=step, packed=packed, stream=s)

    a.set_table(*T)
    with torch.cuda.stream(st):
        admit(10)
    torch.cuda.synchronize()
    idx0, full = i.cpu().numpy().copy()[:R], a.table()
    with torch.cuda.stream(st):
        rel(12)
    torch.cuda.synchronize()
    assert np.array_equal(a.table()[0], T[0]) and np.array_equal(a.table()[1], T[1]), "release gives the table back"
    g_tick, g_admit = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(g_tick, stream=st):
        rel(0)
        admit(1)
    with torch.cuda.graph(g_admit, stream=st):
        admit(3)
    with torch.cuda.stream(st):
        admit(5)
    torch.cuda.synchronize()
    t = {"tick": [], "tick_host": []}
    for rep in range(warmup + reps):
        for arm in (("tick", "tick_host") if rep % 2 == 0 else ("tick_host", "tick")):
            t0 = time.perf_counter()
            if arm == "tick":
                g_tick.replay()
            else:
                h = [x.cpu().numpy() for x in ((c, i) if packed else (c, m, i))]
                core, mem = (((h[0].view(np.uint32) >> 18) & 127).astype(np.int32), (h[0].view(np.uint32) & MEM_MAX).astype(np.int32)) \
                    if packed else (h[0], h[1])
                uc, um = host_sums(core[:R], mem[:R], h[-1][:R].astype(np.int32), D)
                cur = a.table()
                a.set_table(cur[0] + uc, cur[1] + um)
                g_admit.replay()
            torch.cuda.synchronize()
            sec = time.perf_counter() - t0
            got = a.table()
            assert np.array_equal(i.cpu().numpy()[:R], idx0) and all(np.array_equal(x, y) for x, y in zip(got, full)), arm
            if rep >= warmup:
                t[arm].append(sec * 1e6)
    assert a.release_refusals == 0 and a.peer_last_timeout == 0
    return {k: stats(v) for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=41)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("shard_release_probe: no CUDA device; this probe measures on the GPU and has no fallback")
    e.load()
    a = e.BestFitAllocator(0)
    a.peer_attach(0, 1, [a.peer_export()])
    out = {"card": card(), "reps": args.reps, "warmup": args.warmup, "gpus": torch.cuda.device_count(), "results": []}
    print(f"card: {out['card']}; medians of {args.reps} after {args.warmup} [min, max]; us per launch / per tick")
    for D in (8, 64):
        for packed in (False, True):
            r = {"D": D, "format": "packed" if packed else "int32", "rows": R, "us": run_launches(a, D, packed, args.reps, args.warmup)}
            if D == 8:
                r["us"].update(run_tick(a, D, packed, args.reps, args.warmup))
            out["results"].append(r)
            print(f"1Mi_D{D} {r['format']}: " + ", ".join(f"{k} {v['median']:.1f} [{v['min']:.1f}, {v['max']:.1f}]"
                                                        for k, v in r["us"].items()), flush=True)
    out["multi_gpu"] = "multi-GPU not measured"
    print(f"multi-GPU not measured ({out['gpus']} GPU(s) visible; two processes on one GPU prove correctness, not speed)")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump(out, open(args.json, "w"), indent=1)
    a.peer_detach()
    a.close()


if __name__ == "__main__":
    main()
