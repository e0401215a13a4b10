"""Best fit of many pending requests against many capacity tables in one launch: the PyTorch operators
`egpu::bestfit_tables` (DESIGN.md §2.10), `egpu::place_tables` (§2.11), `egpu::place_pods` (§2.12),
`egpu::place_gangs` (§2.13), `egpu::preempt_pods` (§2.14) and `egpu::preempt_gangs` (§2.15).

A scheduler scores every pending pod against every node's device table; `bestfit_tables` does all N x P
pairs in one CUDA launch on the current stream instead of N `egpu_bestfit_query` calls.  `place_tables`
places the pods: best-fit rounds of prefix-commit to the fixed point over every node's devices, in one
launch, so that no device is oversubscribed.  `place_pods` does the same for pods of several containers, every
container of a pod on one node.  `place_gangs` places jobs (gangs of pods) in queue order, each kept only when at
least its `minAvailable` pods are placed and given back otherwise, so that no job holds capacity it cannot start
with.  `preempt_pods` places pods as `place_pods` does, and where a pod fits no node as it is, evicts the fewest,
lowest-priority running pods of one node that make it fit.  `preempt_gangs` places gangs as `place_gangs` does,
each at its priority with `preempt_pods`' evictions, keeps a gang's evictions only when the gang is kept, and never
evicts a running job below its `minAvailable`.  The kernels live in csrc/egpu_tables.cu and are built by
__graft_entry__.build() as lib/libegpu_tables.so; it is separate from libegpu_alloc.so and its C ABI,
reads no context and writes no table of a context.  Importing this module does not load the library; the
first call (or `load()`) does, and a missing library raises: there is no fallback.
"""
from __future__ import annotations

import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libegpu_tables.so")

MAX_DEVICES = 64
MAX_POD = 8  # containers per pod (place_pods)
MAX_RUN = 128  # running pods per node (preempt_pods)
CORE_MAX = 100
MEM_MAX = (1 << 18) - 1
NO_KEY = 0x7FFFFFFF  # key of a pair with no feasible device

_loaded = False


def load() -> None:
    """Load lib/libegpu_tables.so (it registers egpu::bestfit_tables, egpu::place_tables, egpu::place_pods,
    egpu::place_gangs, egpu::preempt_pods and egpu::preempt_gangs) and the operators' fake implementations."""
    global _loaded
    if _loaded:
        return
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc -gencode arch=compute_90a,code=sm_90a). There is no CPU fallback.")
    torch.ops.load_library(LIB_PATH)
    torch.library.register_fake("egpu::bestfit_tables")(_fake)
    torch.library.register_fake("egpu::place_tables")(_fake_place)
    torch.library.register_fake("egpu::place_pods")(_fake_pods)
    torch.library.register_fake("egpu::place_gangs")(_fake_gangs)
    torch.library.register_fake("egpu::preempt_pods")(_fake_preempt)
    torch.library.register_fake("egpu::preempt_gangs")(_fake_preempt_gangs)
    _loaded = True


def check_args(free_core, free_mem, d_valid, req_core, req_mem, op: str = "bestfit_tables") -> None:
    """The operators' checks on dtypes, contiguity, shapes and device (no data is read), in the operators' order:
    RuntimeError for a dtype, layout or device, ValueError for a shape.  `op` names the operator in the messages."""
    names = ("free_core", "free_mem", "d_valid", "req_core", "req_mem")
    ts = (free_core, free_mem, d_valid, req_core, req_mem)
    for name, t in zip(names, ts):
        if t.dtype != torch.int32:
            raise RuntimeError(f"{op}: {name} must be int32, got {t.dtype}")
        if not t.is_contiguous():
            raise RuntimeError(f"{op}: {name} must be contiguous")
    if free_core.dim() != 2 or free_mem.shape != free_core.shape:
        raise ValueError(f"{op}: free_core and free_mem must both be [N, D], got {tuple(free_core.shape)} "
                         f"and {tuple(free_mem.shape)}")
    N, D = free_core.shape
    if not 1 <= D <= MAX_DEVICES:
        raise ValueError(f"{op}: D must be in [1, 64], got {D}")
    if d_valid.dim() != 1 or d_valid.shape[0] != N:
        raise ValueError(f"{op}: d_valid must be [N] = [{N}], got {tuple(d_valid.shape)}")
    if req_core.dim() != 1 or req_mem.shape != req_core.shape:
        raise ValueError(f"{op}: req_core and req_mem must both be [P], got {tuple(req_core.shape)} "
                         f"and {tuple(req_mem.shape)}")
    if N >= 2**31 or req_core.shape[0] >= 2**31:
        raise ValueError(f"{op}: N and P must be below 2^31, got {N} and {req_core.shape[0]}")
    dev = free_core.device
    for t in ts:
        if t.device.type != "cuda" or t.device != dev:
            raise RuntimeError(f"{op}: every tensor must be on one CUDA device, got {t.device} and {dev}")


def check_tables(free_core, free_mem, d_valid, op: str = "bestfit_tables") -> None:
    """ValueError unless every table is in §2.1's domain: 1 <= d_valid[n] <= D, and the first d_valid[n] devices of
    table n have free_core in [0, 100] and free_mem in [0, 2^18 - 1].  Reads the data: one host round trip."""
    D = free_core.shape[1]
    dv = d_valid.to(torch.int64)
    live = torch.arange(D, device=free_core.device)[None, :] < dv[:, None]
    out = (free_core < 0) | (free_core > CORE_MAX) | (free_mem < 0) | (free_mem > MEM_MAX)
    bad_dv = int(((dv < 1) | (dv > D)).sum())
    bad_rows = int((live & out).any(dim=1).sum())
    if bad_dv:
        raise ValueError(f"{op}: {bad_dv} table(s) with d_valid outside [1, {D}]")
    if bad_rows:
        raise ValueError(f"{op}: {bad_rows} table(s) outside the domain (free_core in [0, 100], "
                         f"free_mem in [0, 2^18 - 1] on the first d_valid devices)")


def _fake(free_core, free_mem, d_valid, req_core, req_mem):
    check_args(free_core, free_mem, d_valid, req_core, req_mem)
    N, P = free_core.shape[0], req_core.shape[0]
    return (free_core.new_empty((N, P), dtype=torch.int8), free_core.new_empty((N, P), dtype=torch.int32))


def bestfit_tables(free_core: torch.Tensor, free_mem: torch.Tensor, d_valid: torch.Tensor,
                   req_core: torch.Tensor, req_mem: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """Score P requests against N capacity tables in one launch (DESIGN.md §2.10).

    free_core, free_mem: int32[N, D], 1 <= D <= 64; table n holds its first d_valid[n] devices (int32[N],
    1 <= d_valid[n] <= D), each with free_core in [0, 100] (percent) and free_mem in [0, 2^18 - 1] (MiB).
    req_core, req_mem: int32[P].  All contiguous, on one CUDA device.

    Returns (idx int8[N, P], key int32[N, P]).  idx[n, p] is the device egpu_bestfit_query would choose for
    request p against table n alone: the feasible device (core <= free_core, mem <= free_mem, both >= 0) with
    the smallest (free_core - core, free_mem - mem, d), or -1.  key[n, p] is that order packed as
    (lc << 24) | (lm << 6) | d, the leftovers of the chosen device, so nodes can be ranked by it directly;
    it is 0x7fffffff when idx is -1.  A request outside the domain (negative, core > 100, mem >= 2^18) is
    -1 everywhere.  N = 0 or P = 0 gives empty outputs.

    Stateless: no context is read and no table written; no demand sums.  Asynchronous on the current stream.
    Shapes, dtypes, layout and device are checked before any launch (ValueError for a shape, RuntimeError
    otherwise).  Eagerly, this function also checks the tables' domain and d_valid (ValueError), which
    reads them back; during CUDA-graph capture or torch.compile tracing it cannot, and the operator
    answers -1 (key 0x7fffffff) for every request against a table outside the domain.
    """
    load()
    check_args(free_core, free_mem, d_valid, req_core, req_mem)
    if not torch.compiler.is_compiling() and not torch.cuda.is_current_stream_capturing():
        check_tables(free_core, free_mem, d_valid)
    return torch.ops.egpu.bestfit_tables(free_core, free_mem, d_valid, req_core, req_mem)


def _fake_place(free_core, free_mem, d_valid, req_core, req_mem):
    check_args(free_core, free_mem, d_valid, req_core, req_mem, op="place_tables")
    P = req_core.shape[0]
    return (req_core.new_empty((P,), dtype=torch.int32), req_core.new_empty((P,), dtype=torch.int8),
            torch.empty_like(free_core), torch.empty_like(free_mem), free_core.new_empty((2,), dtype=torch.int32))


def place_tables(free_core: torch.Tensor, free_mem: torch.Tensor, d_valid: torch.Tensor,
                 req_core: torch.Tensor, req_mem: torch.Tensor):
    """Place P requests on N capacity tables in one launch, without oversubscribing a device (DESIGN.md §2.11).

    Inputs as bestfit_tables.  A request takes the feasible device (n, d), d < d_valid[n], with the smallest
    (free_core - core, free_mem - mem, n, d): best fit over every table's valid devices, node-major.  Rounds of
    prefix-commit run to the fixed point: per device, in request order, a request commits while the running demand
    of the requests that chose the device fits; the deferred ones are scored again against the tables the round
    left, until a round defers nothing.  A request that fits nowhere when scored is -1.

    Returns (node int32[P], dev int8[P], free_core_out int32[N, D], free_mem_out int32[N, D], info int32[2]):
    the placement (-1, -1 when none), the tables after every commit (columns at or past d_valid copied unchanged),
    and info = [rounds run (0 when no request is in the domain), 1 if a grid wait gave up after ~2 s, else 0].
    When a wait gives up, unfinished requests stay -2 and the tables are those of the last committed round.
    The inputs are not written.  N = 0 or P = 0 gives -1 placements, copied tables and info [0, 0].

    Stateless and asynchronous on the current stream; it captures into a CUDA graph and traces under
    torch.compile(fullgraph=True).  Refusals are those of bestfit_tables, with "place_tables" in the messages;
    during capture or tracing a table outside the domain offers no device and is copied unchanged.
    """
    load()
    check_args(free_core, free_mem, d_valid, req_core, req_mem, op="place_tables")
    if not torch.compiler.is_compiling() and not torch.cuda.is_current_stream_capturing():
        check_tables(free_core, free_mem, d_valid, op="place_tables")
    return torch.ops.egpu.place_tables(free_core, free_mem, d_valid, req_core, req_mem)


def check_pod_args(free_core, pod_offsets, op: str = "place_pods") -> None:
    """place_pods' checks on pod_offsets' dtype, layout, shape and device (no data is read), after check_args and in
    the operator's order: RuntimeError for a dtype, layout or device, ValueError for a shape.  `op` names the
    operator in the messages."""
    if pod_offsets.dtype != torch.int32:
        raise RuntimeError(f"{op}: pod_offsets must be int32, got {pod_offsets.dtype}")
    if not pod_offsets.is_contiguous():
        raise RuntimeError(f"{op}: pod_offsets must be contiguous")
    if pod_offsets.dim() != 1 or pod_offsets.shape[0] < 1:
        raise ValueError(f"{op}: pod_offsets must be [G + 1], got {tuple(pod_offsets.shape)}")
    if pod_offsets.shape[0] >= 2**31:
        raise ValueError(f"{op}: G + 1 must be below 2^31, got {pod_offsets.shape[0]}")
    if pod_offsets.device.type != "cuda" or pod_offsets.device != free_core.device:
        raise RuntimeError(f"{op}: every tensor must be on one CUDA device, got {pod_offsets.device} and "
                           f"{free_core.device}")


def check_pods(pod_offsets, P: int, op: str = "place_pods") -> None:
    """ValueError unless pod_offsets lists pods of 1 to MAX_POD containers each, covering all P containers: first 0,
    last P, every step in [1, MAX_POD].  Reads the data: one host round trip."""
    o = pod_offsets.to(torch.int64)
    if int(o[0]) != 0:
        raise ValueError(f"{op}: pod_offsets must start at 0, got {int(o[0])}")
    if int(o[-1]) != P:
        raise ValueError(f"{op}: pod_offsets must end at P = {P}, got {int(o[-1])}")
    step = o[1:] - o[:-1]
    bad = int(((step < 1) | (step > MAX_POD)).sum())
    if bad:
        raise ValueError(f"{op}: {bad} pod(s) with a container count outside [1, {MAX_POD}]")


def _fake_pods(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets):
    check_args(free_core, free_mem, d_valid, req_core, req_mem, op="place_pods")
    check_pod_args(free_core, pod_offsets)
    G, P = pod_offsets.shape[0] - 1, req_core.shape[0]
    return (pod_offsets.new_empty((G,), dtype=torch.int32), req_core.new_empty((P,), dtype=torch.int8),
            torch.empty_like(free_core), torch.empty_like(free_mem), free_core.new_empty((3,), dtype=torch.int32))


def place_pods(free_core: torch.Tensor, free_mem: torch.Tensor, d_valid: torch.Tensor, req_core: torch.Tensor,
               req_mem: torch.Tensor, pod_offsets: torch.Tensor):
    """Place G pods on N capacity tables in one launch, every container of a pod on one node, without
    oversubscribing a device (DESIGN.md §2.12).

    Tables as bestfit_tables.  req_core, req_mem: int32[P], the containers listed pod by pod; pod g holds
    containers pod_offsets[g] .. pod_offsets[g + 1] - 1 (pod_offsets int32[G + 1], first 0, last P, 1 to MAX_POD
    containers per pod).  A pod with a container outside the domain is -1.

    A pod's fit on node n is the in-node replay: its containers placed in order on table n, each by best fit
    (smallest (free_core - core, free_mem - mem, d), d < d_valid[n]) against the table as the pod's earlier
    containers left it.  The pod fits n when every container finds a device, and scores (sum of core leftovers,
    sum of memory leftovers, n); it takes the node with the smallest score.  Per node, in pod order, a pod commits
    when none of the devices it chose is closed and, on each of them, the demand committed so far plus its own fits;
    a pod that does not commit is deferred and closes every device it chose.  Deferred pods are scored again against
    the tables the round left, until a round defers nothing.  A pod that fits no node when scored is -1.  A pod's
    fit is not monotone in the table (a container can take the device a later one needed), so -1 means "fit no node
    when last scored", not "fits no output table".

    Returns (node int32[G], dev int8[P], free_core_out int32[N, D], free_mem_out int32[N, D], info int32[3]): each
    pod's node and each container's device on it (all of a pod's containers are placed or none is; -1 when none),
    the tables after every commit (columns at or past d_valid, and tables outside the domain, copied unchanged), and
    info = [rounds run (0 when no pod is in the domain), 1 if a grid wait gave up after ~2 s else 0, 1 if the kernel
    refused pod_offsets else 0].  When a wait gives up, unfinished pods stay -2.  The inputs are not written.  N = 0
    or P = 0 gives -1 placements, copied tables and info [0, 0, 0].

    Stateless and asynchronous on the current stream; it captures into a CUDA graph and traces under
    torch.compile(fullgraph=True).  Refusals are those of bestfit_tables with "place_pods" in the messages, then
    pod_offsets' dtype, layout, shape and device.  Eagerly this function also checks the tables and the offsets'
    values (ValueError), which reads them back; during capture or tracing the kernel checks the offsets itself and,
    if one is bad, places nothing: all -1, tables copied, info[2] = 1.
    """
    load()
    check_args(free_core, free_mem, d_valid, req_core, req_mem, op="place_pods")
    check_pod_args(free_core, pod_offsets)
    if not torch.compiler.is_compiling() and not torch.cuda.is_current_stream_capturing():
        check_tables(free_core, free_mem, d_valid, op="place_pods")
        check_pods(pod_offsets, req_core.shape[0])
    return torch.ops.egpu.place_pods(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets)


def check_gang_args(free_core, gang_offsets, gang_min, op: str = "place_gangs") -> None:
    """place_gangs' checks on gang_offsets' and gang_min's dtype, layout, shapes and device (no data is read), after
    check_args and check_pod_args and in the operator's order: RuntimeError for a dtype, layout or device,
    ValueError for a shape.  `op` names the operator in the messages."""
    for name, t in (("gang_offsets", gang_offsets), ("gang_min", gang_min)):
        if t.dtype != torch.int32:
            raise RuntimeError(f"{op}: {name} must be int32, got {t.dtype}")
        if not t.is_contiguous():
            raise RuntimeError(f"{op}: {name} must be contiguous")
    if gang_offsets.dim() != 1 or gang_offsets.shape[0] < 1:
        raise ValueError(f"{op}: gang_offsets must be [J + 1], got {tuple(gang_offsets.shape)}")
    if gang_offsets.shape[0] >= 2**31:
        raise ValueError(f"{op}: J + 1 must be below 2^31, got {gang_offsets.shape[0]}")
    J = gang_offsets.shape[0] - 1
    if gang_min.dim() != 1 or gang_min.shape[0] != J:
        raise ValueError(f"{op}: gang_min must be [J] = [{J}], got {tuple(gang_min.shape)}")
    for t in (gang_offsets, gang_min):
        if t.device.type != "cuda" or t.device != free_core.device:
            raise RuntimeError(f"{op}: every tensor must be on one CUDA device, got {t.device} and "
                               f"{free_core.device}")


def check_gangs(gang_offsets, gang_min, G: int, op: str = "place_gangs") -> None:
    """ValueError unless gang_offsets lists gangs of at least one pod each, covering all G pods (first 0, last G,
    every step >= 1), and every gang_min[j] is in [1, size of gang j].  Reads the data: one host round trip."""
    o, m = torch.cat([gang_offsets.to(torch.int64), gang_min.to(torch.int64)]).cpu().split(
        [gang_offsets.shape[0], gang_min.shape[0]])
    if int(o[0]) != 0:
        raise ValueError(f"{op}: gang_offsets must start at 0, got {int(o[0])}")
    if int(o[-1]) != G:
        raise ValueError(f"{op}: gang_offsets must end at G = {G}, got {int(o[-1])}")
    size = o[1:] - o[:-1]
    bad = int((size < 1).sum())
    if bad:
        raise ValueError(f"{op}: {bad} gang(s) with no pod")
    bad = int(((m < 1) | (m > size)).sum())
    if bad:
        raise ValueError(f"{op}: {bad} gang(s) with gang_min outside [1, gang size]")


def _fake_gangs(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets, gang_offsets, gang_min):
    check_args(free_core, free_mem, d_valid, req_core, req_mem, op="place_gangs")
    check_pod_args(free_core, pod_offsets, op="place_gangs")
    check_gang_args(free_core, gang_offsets, gang_min)
    G, P, J = pod_offsets.shape[0] - 1, req_core.shape[0], gang_offsets.shape[0] - 1
    return (pod_offsets.new_empty((G,), dtype=torch.int32), req_core.new_empty((P,), dtype=torch.int8),
            gang_offsets.new_empty((J,), dtype=torch.int32), torch.empty_like(free_core), torch.empty_like(free_mem),
            free_core.new_empty((3,), dtype=torch.int32))


def place_gangs(free_core: torch.Tensor, free_mem: torch.Tensor, d_valid: torch.Tensor, req_core: torch.Tensor,
                req_mem: torch.Tensor, pod_offsets: torch.Tensor, gang_offsets: torch.Tensor, gang_min: torch.Tensor):
    """Place J gangs (jobs) of pods on N capacity tables in one launch, in gang order, each gang kept only when at
    least gang_min of its pods are placed, and given back otherwise (DESIGN.md §2.13).

    Tables, containers and pod_offsets as place_pods.  The pods are listed gang by gang: gang j holds pods
    gang_offsets[j] .. gang_offsets[j + 1] - 1 (gang_offsets int32[J + 1], first 0, last G, at least one pod per
    gang).  gang_min int32[J] is each gang's minAvailable, in [1, size of the gang]; gang_min = size is all or nothing.

    The rule is a loop over place_pods: for j = 0 .. J - 1, gang j's pods are placed by place_pods against the tables
    the gangs before it left; if at least gang_min[j] of them are placed, their placement and tables are kept, and
    otherwise every pod of the gang is -1 and the tables are as before it, so later gangs see the capacity it gave
    back.  A gang's rounds stop as soon as its placed plus pending pods fall below gang_min[j] (before round 1, its
    pods in the domain are pending): it can no longer be kept.

    Returns (node int32[G], dev int8[P], placed int32[J], free_core_out int32[N, D], free_mem_out int32[N, D],
    info int32[3]): node and dev as place_pods; placed[j] is 0 for a gang given back and its placed pods (in
    [gang_min[j], size]) for a gang kept; the tables after every kept gang (columns at or past d_valid, and tables
    outside the domain, copied unchanged); info = [rounds run, summed over gangs, 1 if a grid wait gave up after ~2 s
    else 0, 1 if the kernel refused pod_offsets, gang_offsets or gang_min else 0].  When a wait gives up the outputs
    are not a placement and the caller must discard them.  The inputs are not written.  N = 0 or P = 0 gives -1
    placements, placed all 0, copied tables and info [0, 0, 0].

    Stateless and asynchronous on the current stream; it captures into a CUDA graph and traces under
    torch.compile(fullgraph=True).  Refusals are place_pods' with "place_gangs" in the messages, then gang_offsets'
    and gang_min's dtype, layout, shapes and device.  Eagerly this function also checks the tables and the values of
    pod_offsets, gang_offsets and gang_min (ValueError), which reads them back; during capture or tracing the kernel
    checks the three index tensors itself and, if one is bad, places nothing: all -1, placed all 0, tables copied,
    info = [0, 0, 1].
    """
    load()
    check_args(free_core, free_mem, d_valid, req_core, req_mem, op="place_gangs")
    check_pod_args(free_core, pod_offsets, op="place_gangs")
    check_gang_args(free_core, gang_offsets, gang_min)
    if not torch.compiler.is_compiling() and not torch.cuda.is_current_stream_capturing():
        check_tables(free_core, free_mem, d_valid, op="place_gangs")
        check_pods(pod_offsets, req_core.shape[0], op="place_gangs")
        check_gangs(gang_offsets, gang_min, pod_offsets.shape[0] - 1)
    return torch.ops.egpu.place_gangs(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets, gang_offsets,
                                      gang_min)


def check_preempt_args(free_core, pod_offsets, pod_prio, run_core, run_mem, run_dev, run_offsets, run_prio,
                       node_offsets, op: str = "preempt_pods") -> None:
    """preempt_pods' checks on the six new tensors' dtype, layout, shapes and device (no data is read), after
    check_args and check_pod_args and in the operator's order: RuntimeError for a dtype, layout or device,
    ValueError for a shape.  `op` names the operator in the messages; preempt_gangs, whose priority is per gang,
    passes pod_prio=None and its checks are skipped."""
    for name, t, dt in (("pod_prio", pod_prio, torch.int32), ("run_core", run_core, torch.int32),
                        ("run_mem", run_mem, torch.int32), ("run_dev", run_dev, torch.int8),
                        ("run_offsets", run_offsets, torch.int32), ("run_prio", run_prio, torch.int32),
                        ("node_offsets", node_offsets, torch.int32)):
        if t is None:
            continue
        if t.dtype != dt:
            raise RuntimeError(f"{op}: {name} must be {str(dt).replace('torch.', '')}, got {t.dtype}")
        if not t.is_contiguous():
            raise RuntimeError(f"{op}: {name} must be contiguous")
    N, G = free_core.shape[0], pod_offsets.shape[0] - 1
    if pod_prio is not None and (pod_prio.dim() != 1 or pod_prio.shape[0] != G):
        raise ValueError(f"{op}: pod_prio must be [G] = [{G}], got {tuple(pod_prio.shape)}")
    if run_core.dim() != 1 or run_mem.shape != run_core.shape or run_dev.shape != run_core.shape:
        raise ValueError(f"{op}: run_core, run_mem and run_dev must all be [Q], got {tuple(run_core.shape)}, "
                         f"{tuple(run_mem.shape)} and {tuple(run_dev.shape)}")
    if run_offsets.dim() != 1 or run_offsets.shape[0] < 1:
        raise ValueError(f"{op}: run_offsets must be [H + 1], got {tuple(run_offsets.shape)}")
    Q, H = run_core.shape[0], run_offsets.shape[0] - 1
    if Q >= 2**31 - 1 or H >= 2**31 - 1:
        raise ValueError(f"{op}: Q and H + 1 must be below 2^31, got {Q} and {H + 1}")
    if run_prio.dim() != 1 or run_prio.shape[0] != H:
        raise ValueError(f"{op}: run_prio must be [H] = [{H}], got {tuple(run_prio.shape)}")
    if node_offsets.dim() != 1 or node_offsets.shape[0] != N + 1:
        raise ValueError(f"{op}: node_offsets must be [N + 1] = [{N + 1}], got {tuple(node_offsets.shape)}")
    for t in (pod_prio, run_core, run_mem, run_dev, run_offsets, run_prio, node_offsets):
        if t is not None and (t.device.type != "cuda" or t.device != free_core.device):
            raise RuntimeError(f"{op}: every tensor must be on one CUDA device, got {t.device} and {free_core.device}")


def check_running(free_core, free_mem, d_valid, run_core, run_mem, run_dev, run_offsets, node_offsets,
                  op: str = "preempt_pods") -> None:
    """ValueError unless run_offsets lists running pods of 1 to MAX_POD containers covering all Q containers (first
    0, last Q, every step in [1, MAX_POD]), node_offsets lists 0 to MAX_RUN running pods per node covering all H
    (first 0, last H, every step in [0, MAX_RUN]), and every node's running data is consistent: each run_dev in
    [0, d_valid[n]), each running container in the request domain, and on each device free plus the demand of its
    running containers within the table domain.  Reads the data: one host round trip."""
    ro, no = run_offsets.to(torch.int64).cpu(), node_offsets.to(torch.int64).cpu()
    Q, H = run_core.shape[0], ro.shape[0] - 1
    if int(ro[0]) != 0:
        raise ValueError(f"{op}: run_offsets must start at 0, got {int(ro[0])}")
    if int(ro[-1]) != Q:
        raise ValueError(f"{op}: run_offsets must end at Q = {Q}, got {int(ro[-1])}")
    step = ro[1:] - ro[:-1]
    bad = int(((step < 1) | (step > MAX_POD)).sum())
    if bad:
        raise ValueError(f"{op}: {bad} running pod(s) with a container count outside [1, {MAX_POD}]")
    if int(no[0]) != 0:
        raise ValueError(f"{op}: node_offsets must start at 0, got {int(no[0])}")
    if int(no[-1]) != H:
        raise ValueError(f"{op}: node_offsets must end at H = {H}, got {int(no[-1])}")
    step = no[1:] - no[:-1]
    bad = int(((step < 0) | (step > MAX_RUN)).sum())
    if bad:
        raise ValueError(f"{op}: {bad} node(s) with a running pod count outside [0, {MAX_RUN}]")
    if Q == 0:
        return
    N, D = free_core.shape
    dev = free_core.device
    pod_of = torch.repeat_interleave(torch.arange(H), ro[1:] - ro[:-1])
    node_of = torch.repeat_interleave(torch.arange(N), no[1:] - no[:-1])[pod_of].to(dev)
    d = run_dev.to(torch.int64)
    bad_c = (d < 0) | (d >= d_valid.to(torch.int64)[node_of]) | (run_core < 0) | (run_core > CORE_MAX) | \
        (run_mem < 0) | (run_mem > MEM_MAX)
    flat = node_of * D + d.clamp(0, D - 1)
    tot_c = free_core.to(torch.int64).flatten().index_add(0, flat, run_core.to(torch.int64))
    tot_m = free_mem.to(torch.int64).flatten().index_add(0, flat, run_mem.to(torch.int64))
    over = ((tot_c > CORE_MAX) | (tot_m > MEM_MAX)).view(N, D)
    live = torch.arange(D, device=dev)[None, :] < d_valid.to(torch.int64)[:, None]
    bad_n = torch.zeros(N, dtype=torch.int64, device=dev).index_add(0, node_of, bad_c.to(torch.int64)) > 0
    bad = int((bad_n | (over & live).any(dim=1)).sum())
    if bad:
        raise ValueError(f"{op}: {bad} node(s) with inconsistent running data (run_dev outside [0, d_valid), a "
                         f"running container outside the domain, or free plus running demand outside the domain)")


def _fake_preempt(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets, pod_prio, run_core, run_mem, run_dev,
                  run_offsets, run_prio, node_offsets):
    check_args(free_core, free_mem, d_valid, req_core, req_mem, op="preempt_pods")
    check_pod_args(free_core, pod_offsets, op="preempt_pods")
    check_preempt_args(free_core, pod_offsets, pod_prio, run_core, run_mem, run_dev, run_offsets, run_prio,
                       node_offsets)
    G, P, H = pod_offsets.shape[0] - 1, req_core.shape[0], run_offsets.shape[0] - 1
    return (pod_offsets.new_empty((G,), dtype=torch.int32), req_core.new_empty((P,), dtype=torch.int8),
            run_offsets.new_empty((H,), dtype=torch.int32), torch.empty_like(free_core), torch.empty_like(free_mem),
            free_core.new_empty((3,), dtype=torch.int32))


def preempt_pods(free_core: torch.Tensor, free_mem: torch.Tensor, d_valid: torch.Tensor, req_core: torch.Tensor,
                 req_mem: torch.Tensor, pod_offsets: torch.Tensor, pod_prio: torch.Tensor, run_core: torch.Tensor,
                 run_mem: torch.Tensor, run_dev: torch.Tensor, run_offsets: torch.Tensor, run_prio: torch.Tensor,
                 node_offsets: torch.Tensor):
    """Place G pods on N capacity tables in one launch as place_pods does, evicting the fewest, lowest-priority
    running pods of one node where a pod fits no node as it is (DESIGN.md §2.14).

    Tables, containers and pod_offsets as place_pods; pod_prio int32[G] is each pod's priority.  The running pods:
    running pod h holds containers run_offsets[h] .. run_offsets[h + 1] - 1 (run_core, run_mem int32[Q], run_dev
    int8[Q] the device on its node; 1 to MAX_POD containers per pod) and has priority run_prio[h]; node n holds
    running pods node_offsets[n] .. node_offsets[n + 1] - 1 (0 to MAX_RUN), oldest first.  The tables are what is
    free with the running pods in place.

    Pod g's victims on node n: none when its in-node replay fits table n as it is; otherwise C, the alive running
    pods of n below pod_prio[g], if the replay fits table n plus C's demand (else n is no candidate), less each member
    of C, walked by (priority descending, h ascending), without which the replay still fits.  The pod takes the
    candidate with the smallest (highest victim priority, sum of (priority + 2^31), victims, sum lc, sum lm, n); no
    victim ranks below every victim.  Per node, in pod order: a pod without victims commits as in place_pods; a pod
    with victims commits only when it is the first of the round to choose the node, evicts them and takes its demand,
    and closes the node for the round either way.  Deferred pods are scored again against the tables and running pods
    the round left, until a round defers nothing.  With no pod above any running pod the outputs are place_pods'.

    Returns (node int32[G], dev int8[P], evicted int32[H], free_core_out int32[N, D], free_mem_out int32[N, D],
    info int32[3]): node and dev as place_pods; evicted[h] the pod that evicted running pod h, or -1; the tables
    after every eviction and placement, assuming the evicted pods are gone; info = [rounds run (0 when no pod is in
    the domain), 1 if a grid wait gave up after ~2 s else 0, 1 if the kernel refused an index tensor else 0].  When a
    wait gives up the outputs are not a placement and the caller must discard them.  The inputs are not written.
    N = 0 or P = 0 gives -1 placements, evicted all -1, copied tables and info [0, 0, 0].

    Stateless and asynchronous on the current stream; it captures into a CUDA graph and traces under
    torch.compile(fullgraph=True).  Refusals are place_pods' with "preempt_pods" in the messages, then the six new
    tensors' dtype, layout, shapes and device.  Eagerly this function also checks the tables, pod_offsets, and the
    running pods (check_running; ValueError), which reads them back; during capture or tracing the kernel checks the
    three offset tensors itself and, if one is bad, places and evicts nothing: all -1, tables copied, info = [0, 0, 1];
    a node whose table is outside the domain or whose running data is inconsistent offers no candidate and is copied.
    """
    load()
    check_args(free_core, free_mem, d_valid, req_core, req_mem, op="preempt_pods")
    check_pod_args(free_core, pod_offsets, op="preempt_pods")
    check_preempt_args(free_core, pod_offsets, pod_prio, run_core, run_mem, run_dev, run_offsets, run_prio,
                       node_offsets)
    if not torch.compiler.is_compiling() and not torch.cuda.is_current_stream_capturing():
        check_tables(free_core, free_mem, d_valid, op="preempt_pods")
        check_pods(pod_offsets, req_core.shape[0], op="preempt_pods")
        check_running(free_core, free_mem, d_valid, run_core, run_mem, run_dev, run_offsets, node_offsets)
    return torch.ops.egpu.preempt_pods(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets, pod_prio, run_core,
                                       run_mem, run_dev, run_offsets, run_prio, node_offsets)


def check_preempt_gang_args(free_core, gang_offsets, run_offsets, gang_prio, run_gang, run_gang_min) -> None:
    """preempt_gangs' checks on gang_prio's, run_gang's and run_gang_min's dtype, layout, shapes and device (no data is
    read), after those of place_gangs and preempt_pods and in the operator's order: RuntimeError for a dtype, layout
    or device, ValueError for a shape."""
    op = "preempt_gangs"
    for name, t in (("gang_prio", gang_prio), ("run_gang", run_gang), ("run_gang_min", run_gang_min)):
        if t.dtype != torch.int32:
            raise RuntimeError(f"{op}: {name} must be int32, got {t.dtype}")
        if not t.is_contiguous():
            raise RuntimeError(f"{op}: {name} must be contiguous")
    J, H = gang_offsets.shape[0] - 1, run_offsets.shape[0] - 1
    if gang_prio.dim() != 1 or gang_prio.shape[0] != J:
        raise ValueError(f"{op}: gang_prio must be [J] = [{J}], got {tuple(gang_prio.shape)}")
    if run_gang.dim() != 1 or run_gang.shape[0] != H:
        raise ValueError(f"{op}: run_gang must be [H] = [{H}], got {tuple(run_gang.shape)}")
    if run_gang_min.dim() != 1:
        raise ValueError(f"{op}: run_gang_min must be [R], got {tuple(run_gang_min.shape)}")
    if run_gang_min.shape[0] >= 2**31 - 1:
        raise ValueError(f"{op}: R must be below 2^31 - 1, got {run_gang_min.shape[0]}")
    for t in (gang_prio, run_gang, run_gang_min):
        if t.device.type != "cuda" or t.device != free_core.device:
            raise RuntimeError(f"{op}: every tensor must be on one CUDA device, got {t.device} and {free_core.device}")


def check_running_gangs(run_gang, run_gang_min) -> None:
    """ValueError unless every run_gang[h] is in [-1, R) (R = run_gang_min's length) and every run_gang_min[r] is at
    least 0.  Reads the data: one host round trip."""
    op = "preempt_gangs"
    R = run_gang_min.shape[0]
    bad = int(((run_gang < -1) | (run_gang >= R)).sum())
    if bad:
        raise ValueError(f"{op}: {bad} running pod(s) with run_gang outside [-1, {R})")
    bad = int((run_gang_min < 0).sum())
    if bad:
        raise ValueError(f"{op}: {bad} running job(s) with run_gang_min below 0")


def _fake_preempt_gangs(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets, gang_offsets, gang_min,
                        gang_prio, run_core, run_mem, run_dev, run_offsets, run_prio, node_offsets, run_gang,
                        run_gang_min):
    op = "preempt_gangs"
    check_args(free_core, free_mem, d_valid, req_core, req_mem, op=op)
    check_pod_args(free_core, pod_offsets, op=op)
    check_gang_args(free_core, gang_offsets, gang_min, op=op)
    check_preempt_args(free_core, pod_offsets, None, run_core, run_mem, run_dev, run_offsets, run_prio, node_offsets,
                       op=op)
    check_preempt_gang_args(free_core, gang_offsets, run_offsets, gang_prio, run_gang, run_gang_min)
    G, P, J, H = pod_offsets.shape[0] - 1, req_core.shape[0], gang_offsets.shape[0] - 1, run_offsets.shape[0] - 1
    return (pod_offsets.new_empty((G,), dtype=torch.int32), req_core.new_empty((P,), dtype=torch.int8),
            gang_offsets.new_empty((J,), dtype=torch.int32), run_offsets.new_empty((H,), dtype=torch.int32),
            torch.empty_like(free_core), torch.empty_like(free_mem), free_core.new_empty((3,), dtype=torch.int32))


def preempt_gangs(free_core: torch.Tensor, free_mem: torch.Tensor, d_valid: torch.Tensor, req_core: torch.Tensor,
                  req_mem: torch.Tensor, pod_offsets: torch.Tensor, gang_offsets: torch.Tensor, gang_min: torch.Tensor,
                  gang_prio: torch.Tensor, run_core: torch.Tensor, run_mem: torch.Tensor, run_dev: torch.Tensor,
                  run_offsets: torch.Tensor, run_prio: torch.Tensor, node_offsets: torch.Tensor,
                  run_gang: torch.Tensor, run_gang_min: torch.Tensor):
    """Place J gangs (jobs) of pods on N capacity tables in one launch, in gang order, each gang's pods placed as
    preempt_pods places them at the gang's priority, kept only when at least gang_min of them are placed, and never
    evicting a running job below its minAvailable (DESIGN.md §2.15).

    Tables, containers, pod_offsets, gang_offsets and gang_min as place_gangs; gang_prio int32[J] is each gang's
    priority (one PodGroup, one priority class).  The running pods as preempt_pods; run_gang int32[H] in [-1, R) names
    the running job (gang) each running pod belongs to (-1: none), and run_gang_min int32[R] >= 0 is each running
    job's minAvailable.  A running job's slack is its listed running pods not evicted, on any node, less its
    minAvailable (0 when that is negative).

    The rule is place_gangs' loop over gangs, each gang's pods placed by preempt_pods' rounds, with two changes.  On
    each node, C keeps of each running job only the slack pods of that job that come last in the walk order (priority
    descending, h ascending), the slack read at the start of the round.  And a round's first-on-node preemptors with
    a victim in a running job commit, in pod order, only while every such job's victims of this pod and of the
    preemptors before it stay within the job's slack; the others are deferred.  A gang that ends with fewer than
    gang_min pods placed is given back: placements and evictions are undone, and later gangs see the tables, the
    running pods and the slacks as they were before it.

    Returns (node int32[G], dev int8[P], placed int32[J], evicted int32[H], free_core_out int32[N, D], free_mem_out
    int32[N, D], info int32[3]): node and dev as place_pods; placed as place_gangs; evicted[h] the pod that evicted
    running pod h, or -1 (only pods of kept gangs evict); the tables after every kept gang, assuming the evicted pods
    are gone; info = [rounds run, summed over gangs, 1 if a grid wait gave up after ~2 s else 0, 1 if the kernel
    refused an index tensor or run_gang_min else 0].  When a wait gives up the outputs are not a placement and the
    caller must discard them.  The inputs are not written.  N = 0 or P = 0 gives -1 placements, placed all 0, evicted
    all -1, copied tables and info [0, 0, 0].

    Stateless and asynchronous on the current stream; it captures into a CUDA graph and traces under
    torch.compile(fullgraph=True).  Refusals are place_gangs' and preempt_pods' (without pod_prio) with
    "preempt_gangs" in the messages, then gang_prio's, run_gang's and run_gang_min's dtype, layout, shapes and device.
    Eagerly this function also checks the tables, the index tensors, the running pods and the running jobs
    (ValueError), which reads them back; during capture or tracing the kernel checks the five index tensors and
    run_gang_min itself and, if one is bad, places and evicts nothing: all -1, placed all 0, tables copied,
    info = [0, 0, 1]; a node whose table is outside the domain or whose running data is inconsistent offers no
    candidate and is copied.
    """
    load()
    op = "preempt_gangs"
    check_args(free_core, free_mem, d_valid, req_core, req_mem, op=op)
    check_pod_args(free_core, pod_offsets, op=op)
    check_gang_args(free_core, gang_offsets, gang_min, op=op)
    check_preempt_args(free_core, pod_offsets, None, run_core, run_mem, run_dev, run_offsets, run_prio, node_offsets,
                       op=op)
    check_preempt_gang_args(free_core, gang_offsets, run_offsets, gang_prio, run_gang, run_gang_min)
    if not torch.compiler.is_compiling() and not torch.cuda.is_current_stream_capturing():
        check_tables(free_core, free_mem, d_valid, op=op)
        check_pods(pod_offsets, req_core.shape[0], op=op)
        check_gangs(gang_offsets, gang_min, pod_offsets.shape[0] - 1, op=op)
        check_running(free_core, free_mem, d_valid, run_core, run_mem, run_dev, run_offsets, node_offsets, op=op)
        check_running_gangs(run_gang, run_gang_min)
    return torch.ops.egpu.preempt_gangs(free_core, free_mem, d_valid, req_core, req_mem, pod_offsets, gang_offsets,
                                        gang_min, gang_prio, run_core, run_mem, run_dev, run_offsets, run_prio,
                                        node_offsets, run_gang, run_gang_min)
