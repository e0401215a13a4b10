"""Probe (one GPU) of the release launch (EGPU_F_RELEASE): what it costs next to the snapshot scan over the same rows
and next to what a caller had to do before it existed, the arms alternating in one run.

    python scripts/release_probe.py [--reps N] [--warmup N] [--json PATH]

Shapes: 1 Mi rows at D = 8 and D = 64, 100 k rows and 16 Mi + 1 rows at D = 8, int32 and packed.  Arms:
  release        one dry release launch (no EGPU_F_COMMIT: the table stays, so every repetition does the same work; the
                 committing form adds D stores and one re-sort by the last CTA), CUDA events around it;
  release_rpt4 / release_rpt16
                 the same launch from contexts created under EGPU_ROWS_PER_THREAD = 4 / 16 (the shipped rule is 8);
  release_x20    20 release launches replayed from a CUDA graph, each over its own buffers of a ring larger than the
                 50 MB L2, per launch (not for 16 Mi + 1 rows: two such batches are already 8 x L2);
  scan / scan_x20
                 the non-committing snapshot scan over the same rows, the traffic yardstick: it loads the requests and
                 stores the indices, the release loads both, so the algorithmic bytes per row are the same;
  host_recompute what a caller did before: rows and indices to the host, np.bincount, egpu_table_set; host clock
                 from the first copy to the end of the call (egpu_table_set synchronises);
  tick / tick_host (1 Mi shapes)
                 a churn tick replayed from a CUDA graph - release of the rows placed by the previous tick, then their
                 admission again by the rounds in one launch - against the same tick with host_recompute in place of
                 the release; host clock to the end of a synchronise.
Every repetition compares the arms' outputs: sums and table' of every release arm with the host recompute, the
indices and installed table of the two ticks.  Medians of --reps after --warmup.  "GB/s (algorithmic)" is the bytes
the algorithm needs (12 per row, 5 packed) over the median time, beside the H100 SXM data sheet's 3.35 TB/s; it is
not an achieved-bandwidth measurement.
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
SHAPES = [("1Mi_D8", 1 << 20, 8), ("1Mi_D64", 1 << 20, 64), ("100k_D8", 100_000, 8), ("16Mi+1_D8", (16 << 20) + 1, 8)]
RING_BYTES = 120 << 20


def card():
    """card name and power limit, read in the same run (read-only query)"""
    out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=60).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def rows_for(R, D, seed):
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


def event_ms(fn, stream):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    fn()
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b)


def run_shape(ctxs, name, R, D, packed, reps, warmup):
    a = ctxs[8]
    fc, fm = np.full(D, 10, np.int32), np.full(D, 1000, np.int32)
    for c in ctxs.values():
        c.set_table(fc, fm)
    row_bytes = 5 if packed else 12
    ring = 2 if R > (1 << 22) else -(-max(20, -(-RING_BYTES // (R * row_bytes))) // 20) * 20
    st = torch.cuda.Stream()
    s = st.cuda_stream
    bufs, ref = [], None
    for k in range(ring):
        core, mem, idx = rows_for(R, D, k if R <= (1 << 20) else 0)
        if k == 0:
            ref = (core, mem, idx)
        if packed:
            bufs.append((torch.from_numpy(a.pack_requests(core, mem).view(np.int32)).cuda(), None, torch.from_numpy(idx.astype(np.int8)).cuda()))
        else:
            bufs.append((torch.from_numpy(core).cuda(), torch.from_numpy(mem).cuda(), torch.from_numpy(idx).cuda()))
    delta = torch.zeros(2 * D, dtype=torch.int64, device="cuda")
    tab = torch.zeros(3 * D, dtype=torch.int32, device="cuda")
    out_idx = torch.empty(R + 16, dtype=torch.int8 if packed else torch.int32, device="cuda")
    uc, um = host_sums(*ref, D)
    want_tab = np.concatenate([fc + uc, fm + um, np.zeros(D, np.int64)]).astype(np.int32)

    def release(ctx, b, commit=False):
        ctx.release_dev(b[0].data_ptr(), 0 if packed else b[1].data_ptr(), R, b[2].data_ptr(), delta.data_ptr(), tab.data_ptr(),
                        commit=commit, packed=packed, stream=s)

    def scan(b):
        if packed:
            a.bestfit_packed_dev(b[0].data_ptr(), R, out_idx.data_ptr(), delta.data_ptr(), 0, stream=s)
        else:
            a.bestfit_dev(b[0].data_ptr(), b[1].data_ptr(), R, out_idx.data_ptr(), delta.data_ptr(), 0, stream=s)

    def graphs_of(fn):
        out = []
        for g0 in range(0, ring if ring >= 20 else 0, 20):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=st):
                for b in bufs[g0:g0 + 20]:
                    fn(b)
            out.append(g)
        return out

    def host_recompute():
        """(seconds, table installed)"""
        t0 = time.perf_counter()
        h = [x.cpu().numpy() for x in bufs[0] if x is not None]
        core, mem = (((h[0].view(np.uint32) >> 18) & 127).astype(np.int32), (h[0].view(np.uint32) & MEM_MAX).astype(np.int32)) if packed \
            else (h[0], h[1])
        c, m = host_sums(core, mem, h[-1].astype(np.int32), D)
        cur = a.table()
        a.set_table(cur[0] + c, cur[1] + m)
        return time.perf_counter() - t0, a.table()

    with torch.cuda.stream(st):
        for c in ctxs.values():
            release(c, bufs[0])
        scan(bufs[0])
    torch.cuda.synchronize()
    g_rel, g_scan = graphs_of(lambda b: release(a, b)), graphs_of(scan)
    t = {k: [] for k in ("release", "release_rpt4", "release_rpt16", "scan", "host_recompute")}
    if g_rel:
        t["release_x20"], t["scan_x20"] = [], []
    for rep in range(warmup + reps):
        keep = rep >= warmup
        for arm, ctx in (("release", a), ("release_rpt4", ctxs[4]), ("release_rpt16", ctxs[16])):
            ms = event_ms(lambda: release(ctx, bufs[0]), st)
            assert np.array_equal(delta.cpu().numpy(), np.concatenate([uc, um])) and np.array_equal(tab.cpu().numpy(), want_tab), arm
            if keep:
                t[arm].append(ms * 1e3)
        ms = event_ms(lambda: scan(bufs[0]), st)
        if keep:
            t["scan"].append(ms * 1e3)
        if g_rel:
            for arm, gs in (("release_x20", g_rel), ("scan_x20", g_scan)):
                g = gs[rep % len(gs)]
                ms = event_ms(g.replay, torch.cuda.current_stream())
                if keep:
                    t[arm].append(ms * 1e3 / 20)
        a.set_table(fc, fm)
        sec, got = host_recompute()
        assert np.array_equal(got[0], want_tab[:D]) and np.array_equal(got[1], want_tab[D:2 * D]), "host recompute"
        a.set_table(fc, fm)
        with torch.cuda.stream(st):
            scan(bufs[0])  # untimed: the lookup scan rebuilds its tables after egpu_table_set
        torch.cuda.synchronize()
        if keep:
            t["host_recompute"].append(sec * 1e6)
    res = {k: float(np.median(v)) for k, v in t.items()}
    if R == 1 << 20:
        res.update(run_tick(a, D, R, packed, reps, warmup, st))
    return {"shape": name, "format": "packed" if packed else "int32", "rows": R, "D": D, "bytes": R * row_bytes, "ring": ring, "us": res}


def run_tick(a, D, R, packed, reps, warmup, st):
    """steady state: every tick releases the rows the previous tick placed and places the same rows again, so the
    indices and the table after a tick are the same every time, whichever arm ran it"""
    s = st.cuda_stream
    w = e.synth.workload("cfg3" if D == 8 else "cfg4")
    T = (np.asarray(w["free_core"], np.int32), np.asarray(w["free_mem"], np.int32))
    rc, rm = e.synth.requests(3, 5, R)
    rc, rm = np.minimum(rc, 5).astype(np.int32), np.minimum(rm, 2048).astype(np.int32)
    c = torch.from_numpy(a.pack_requests(rc, rm).view(np.int32) if packed else rc).cuda()
    m = torch.from_numpy(rm).cuda()
    i = torch.empty(R + 16, dtype=torch.int8 if packed else torch.int32, device="cuda")

    def admit():
        if packed:
            a.bestfit_packed_rounds_device_dev(c.data_ptr(), R, i.data_ptr(), stream=s)
        else:
            a.bestfit_rounds_device_dev(c.data_ptr(), m.data_ptr(), R, i.data_ptr(), stream=s)

    def rel():
        a.release_dev(c.data_ptr(), 0 if packed else m.data_ptr(), R, i.data_ptr(), commit=True, packed=packed, stream=s)

    a.set_table(*T)
    with torch.cuda.stream(st):
        admit()
    torch.cuda.synchronize()
    idx0, full = i.cpu().numpy().copy()[:R], a.table()
    with torch.cuda.stream(st):
        rel()
    torch.cuda.synchronize()
    assert np.array_equal(a.table()[0], T[0]) and np.array_equal(a.table()[1], T[1]), "release gives the table back"
    g_tick, g_admit = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(g_tick, stream=st):
        rel()
        admit()
    with torch.cuda.graph(g_admit, stream=st):
        admit()
    with torch.cuda.stream(st):
        admit()
    torch.cuda.synchronize()
    t = {"tick": [], "tick_host": []}
    for rep in range(warmup + reps):
        for arm in ("tick", "tick_host"):
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
    assert a.release_refusals == 0
    return {k: float(np.median(v)) for k, v in t.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=41)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("release_probe: no CUDA device; this probe measures on the GPU and has no fallback")
    e.load()
    ctxs = {}
    for rpt in (8, 4, 16):  # EGPU_ROWS_PER_THREAD is read when a context is created
        os.environ.pop("EGPU_ROWS_PER_THREAD", None)
        if rpt != 8:
            os.environ["EGPU_ROWS_PER_THREAD"] = str(rpt)
        ctxs[rpt] = e.BestFitAllocator(0)
    os.environ.pop("EGPU_ROWS_PER_THREAD", None)
    out = {"card": card(), "reps": args.reps, "warmup": args.warmup, "data_sheet_TBps": 3.35, "results": []}
    print(f"card: {out['card']}; medians of {args.reps} after {args.warmup}; us (GB/s algorithmic, data sheet 3350)")
    for name, R, D in SHAPES:
        for packed in (False, True):
            r = run_shape(ctxs, name, R, D, packed, args.reps, args.warmup)
            out["results"].append(r)
            cells = []
            for k, v in r["us"].items():
                gbps = f" ({r['bytes'] / v / 1e3:.0f})" if k.startswith(("release", "scan")) else ""
                cells.append(f"{k} {v:.1f}{gbps}")
            print(f"{name} {r['format']}: " + ", ".join(cells), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump(out, open(args.json, "w"), indent=1)
    for c in ctxs.values():
        c.close()


if __name__ == "__main__":
    main()
