"""egpu::bestfit_tables without a GPU (DESIGN.md §2.10): the fake implementation's shapes and dtypes, which
torch.compile and CUDA-graph tracing see, and every argument check the operator and its Python interface make before
a launch.  The same cases run through the fake, the compiled operator (its CPU registration refuses with the same
messages) and the Python checks, so the three cannot drift apart."""
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

MEM_MAX = (1 << 18) - 1


@pytest.fixture(scope="module")
def tables():
    from elastic_gpu_agent_b200 import tables as t
    t.load()
    return t


def args(N=6, D=8, P=12, device="cpu", **kw):
    a = dict(fc=torch.full((N, D), 50, dtype=torch.int32, device=device),
             fm=torch.full((N, D), 1000, dtype=torch.int32, device=device),
             dv=torch.full((N,), D, dtype=torch.int32, device=device),
             rc=torch.full((P,), 10, dtype=torch.int32, device=device),
             rm=torch.full((P,), 10, dtype=torch.int32, device=device))
    a.update(kw)
    return a["fc"], a["fm"], a["dv"], a["rc"], a["rm"]


def refusals(device):
    z = dict(dtype=torch.int32, device=device)
    return [
        (RuntimeError, "free_core must be int32", dict(fc=torch.full((6, 8), 50, dtype=torch.int64, device=device))),
        (RuntimeError, "req_mem must be int32", dict(rm=torch.zeros(12, dtype=torch.int16, device=device))),
        (RuntimeError, "d_valid must be int32", dict(dv=torch.full((6,), 8.0, device=device))),
        (RuntimeError, "free_core must be contiguous", dict(fc=torch.zeros((8, 6), **z).t())),
        (RuntimeError, "req_core must be contiguous", dict(rc=torch.zeros(24, **z)[::2])),
        (ValueError, "must both be \\[N, D\\]", dict(fm=torch.zeros((6, 9), **z))),
        (ValueError, "must both be \\[N, D\\]", dict(fc=torch.zeros(6, **z), fm=torch.zeros(6, **z))),
        (ValueError, "D must be in \\[1, 64\\], got 0", dict(fc=torch.zeros((6, 0), **z), fm=torch.zeros((6, 0), **z))),
        (ValueError, "D must be in \\[1, 64\\], got 65", dict(fc=torch.zeros((6, 65), **z), fm=torch.zeros((6, 65), **z))),
        (ValueError, "d_valid must be \\[N\\]", dict(dv=torch.zeros(7, **z))),
        (ValueError, "d_valid must be \\[N\\]", dict(dv=torch.zeros((6, 1), **z))),
        (ValueError, "must both be \\[P\\]", dict(rm=torch.zeros(11, **z))),
        (ValueError, "must both be \\[P\\]", dict(rc=torch.zeros((12, 1), **z), rm=torch.zeros((12, 1), **z))),
    ]


@pytest.mark.parametrize("N,D,P", [(6, 8, 12), (5000, 8, 1024), (512, 64, 8192), (0, 3, 7), (4, 1, 0)])
def test_fake_gives_shapes_and_dtypes(N, D, P, tables):
    with FakeTensorMode():
        idx, key = torch.ops.egpu.bestfit_tables(*args(N, D, P, device="cuda"))
    assert idx.shape == key.shape == (N, P)
    assert idx.dtype == torch.int8 and key.dtype == torch.int32
    assert idx.device.type == key.device.type == "cuda"


@pytest.mark.parametrize("case", range(13))
def test_fake_operator_and_python_checks_refuse_alike(case, tables):
    exc, msg, kw = refusals("cpu")[case]
    with pytest.raises(exc, match=msg):
        torch.ops.egpu.bestfit_tables(*args(**kw))  # the compiled operator, CPU tensors: refused before the device check
    with pytest.raises(exc, match=msg):
        tables.check_args(*args(**kw))
    with pytest.raises(exc, match=msg):
        tables.bestfit_tables(*args(**kw))
    with FakeTensorMode():
        exc_f, msg_f, kw_f = refusals("cuda")[case]
        with pytest.raises(exc_f, match=msg_f):
            torch.ops.egpu.bestfit_tables(*args(device="cuda", **kw_f))


def test_tensors_off_the_gpu_are_refused(tables):
    for call in (torch.ops.egpu.bestfit_tables, tables.check_args, tables.bestfit_tables):
        with pytest.raises(RuntimeError, match="one CUDA device"):
            call(*args())
    with FakeTensorMode():
        fc, fm, dv, rc, rm = args(device="cuda")
        with pytest.raises(RuntimeError, match="one CUDA device"):
            torch.ops.egpu.bestfit_tables(fc, fm, dv, torch.zeros(12, dtype=torch.int32), rm)


def test_table_domain_and_d_valid_checks(tables):
    fc, fm, dv, _, _ = args(N=4, D=8)
    dv[:] = torch.tensor([1, 3, 8, 5], dtype=torch.int32)
    past = torch.arange(8)[None, :] >= dv[:, None]
    fc[past], fm[past] = 1000, -1  # padding past d_valid is not a device
    tables.check_tables(fc, fm, dv)
    for col, c, m in ((0, 101, 0), (2, -1, 0), (4, 50, MEM_MAX + 1), (3, 50, -5)):
        f2, m2 = fc.clone(), fm.clone()
        f2[3, col], m2[3, col] = c, (m if m else m2[3, col])
        with pytest.raises(ValueError, match="outside the domain"):
            tables.check_tables(f2, m2, dv)
    for bad in (0, 9, -1):
        d2 = dv.clone()
        d2[2] = bad
        with pytest.raises(ValueError, match="d_valid outside \\[1, 8\\]"):
            tables.check_tables(fc, fm, d2)
    f2 = fc.clone()
    f2[1, :3] = torch.tensor([0, 100, 100], dtype=torch.int32)
    fm[1, :3] = torch.tensor([0, MEM_MAX, 81_559], dtype=torch.int32)
    tables.check_tables(f2, fm, dv)  # the domain's edges are in it
