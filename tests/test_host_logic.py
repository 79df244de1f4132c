"""CPU tests of the host side: partition bookkeeping (bit-exact vs the oracle),
exchange plans, the C-ABI library's symbol table, and the communicator shim on
a world_size-2 gloo group.  No compute kernels are called."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import pylops_mpi_oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_abi_library_loads_and_exports_every_declared_symbol():
    import importlib.util
    spec = importlib.util.spec_from_file_location("_b200_build", os.path.join(ROOT, "pylops_mpi_b200", "build.py"))
    build = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build)  # not via the package: importing it needs the built library
    path = build.build()            # builds on first use (nvcc cross-compiles without a GPU)
    lib = ctypes.CDLL(path)
    header = open(os.path.join(ROOT, "include", "b200lops.h")).read()
    declared = set(re.findall(r"\b(b2_[a-z0-9_]+)\s*\(", header))
    assert len(declared) >= 30
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/b200lops.h but not exported"
    assert lib.b2_version() == 100
    lib.b2_strerror.restype = ctypes.c_char_p
    assert b"halo" in lib.b2_strerror(2003)


def test_python_binding_covers_header():
    import pylops_mpi_b200._lib as L
    header = open(os.path.join(ROOT, "include", "b200lops.h")).read()
    declared = set(re.findall(r"\b(b2_[a-z0-9_]+)\s*\(", header))
    assert declared == set(L.EXPORTS)


def test_product_fails_loudly_without_gpu():
    import torch
    import pylops_mpi_b200 as pm
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(pm._lib.B200Error):
        pm.DistributedArray(global_shape=10)


@pytest.mark.parametrize("n", [0, 1, 7, 231, 600, 1000003])
@pytest.mark.parametrize("P", [1, 2, 3, 4, 8, 9])
def test_local_split_sizes_bit_exact(n, P):
    from pylops_mpi_b200.utils.partition import local_split_sizes
    assert local_split_sizes(n, P) == [o.local_split((n,), P, r)[0] for r in range(P)]


@pytest.mark.parametrize("dims", [(11, 21), (600,), (100, 151), (101, 51, 100), (79, 101, 50)])
@pytest.mark.parametrize("P", [1, 2, 3, 4, 8])
def test_repartition_plan_moves_every_element_once(dims, P):
    from pylops_mpi_b200.utils.partition import local_split_sizes, repartition_plan, reshaped_ghost_cells
    n = int(np.prod(dims))
    src = local_split_sizes(n, P)
    dst = [e * int(np.prod(dims[1:])) for e in local_split_sizes(dims[0], P)]
    x = np.arange(n)
    xs = np.split(x, np.cumsum(src)[:-1])
    out = [np.full(d, -1) for d in dst]
    for r in range(P):
        sends, _ = repartition_plan(src, dst, r)
        for peer, off, cnt in sends:
            _, recvs = repartition_plan(src, dst, peer)
            doff = [q for q in recvs if q[0] == r][0]
            assert doff[2] == cnt
            out[peer][doff[1]:doff[1] + cnt] = xs[r][off:off + cnt]
    assert np.array_equal(np.concatenate(out), x)
    # and it agrees with the reference's neighbour-only plan whenever that plan is legal
    try:
        ref = o.reshaped_in([a.copy() for a in xs], [(e,) + tuple(dims[1:]) for e in local_split_sizes(dims[0], P)])
    except ValueError:
        return
    for r in range(P):
        assert np.array_equal(ref[r].ravel(), out[r])
        cf, cb, idx = reshaped_ghost_cells(dst, src, r)
        assert cf >= 0 and cb >= 0 and idx >= 0


def test_halo_plan_matches_oracle_ghost_cells():
    from pylops_mpi_b200.utils.partition import halo_plan, local_split_sizes
    rows = local_split_sizes(101, 4)
    for r in range(4):
        p = halo_plan(rows, r, 2, 2)
        assert p["recv_lo"] == (0 if r == 0 else 2) and p["recv_hi"] == (0 if r == 3 else 2)
        assert p["send_lo"] == (0 if r == 0 else 2) and p["send_hi"] == (0 if r == 3 else 2)
    with pytest.raises(ValueError):
        halo_plan([3, 1, 3], 0, 2, 2)


def test_single_process_comm_shim():
    from pylops_mpi_b200.comm import Comm
    c = Comm(0, 1)
    assert c.Get_rank() == 0 and c.Get_size() == 1
    assert c.allgather((3, 4)) == [(3, 4)]
    assert c.allreduce(5) == 5 and c.bcast("a") == "a"
    s = c.Split(0, 0)
    assert s.Get_size() == 1 and c.nccl is None
    c.Barrier()


_WORKER = r'''
import os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "oracle"))
import numpy as np
import pylops_mpi_oracle as o
from pylops_mpi_b200.comm import get_comm_world
from pylops_mpi_b200.utils.partition import local_split_sizes, halo_plan
from pylops_mpi_b200.DistributedArray import local_split, Partition
comm = get_comm_world()
rank, size = comm.Get_rank(), comm.Get_size()
assert size == 2
assert comm.allgather(rank * 10) == [0, 10]
assert comm.allreduce(rank + 1) == 3
assert comm.allreduce(rank + 1, "max") == 2
assert comm.bcast({"a": rank}, root=1) == {"a": 1}
# local_split through the communicator == oracle == closed formula
for shape, axis in [((11, 21), 0), ((500, 501), 1), ((7,), 0)]:
    mine = local_split(shape, comm, Partition.SCATTER, axis)
    assert mine == o.local_split(shape, size, rank, o.SCATTER, axis)
    assert comm.allgather(mine[axis]) == local_split_sizes(shape[axis], size)
# Split: each rank alone, then everybody together with reversed keys
solo = comm.Split(color=rank, key=0)
assert solo.Get_size() == 1 and solo.Get_rank() == 0
rev = comm.Split(color=0, key=size - rank)
assert rev.Get_size() == 2 and rev.Get_rank() == 1 - rank
assert rev.allgather(rank) == [1, 0]
m = comm.split_by_mask([0, 0]); assert m.Get_size() == 2
assert comm.split_by_mask([0, 0]) is m            # cached
# halo plan is symmetric between neighbours
rows = local_split_sizes(11, size)
p = halo_plan(rows, rank, 1, 1)
q = comm.allgather(p)
assert q[0]["send_hi"] == q[1]["recv_lo"] and q[1]["send_lo"] == q[0]["recv_hi"]
comm.Barrier()
print("WORKER_OK", rank)
'''


def test_comm_shim_world_size_2_gloo(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    from op_checks import run_on_ranks
    out = run_on_ranks(str(script), 2, args=(ROOT,), env=dict(CUDA_VISIBLE_DEVICES=""), timeout=300)
    assert out.count("WORKER_OK") == 2


# ---- the boundary is a C ABI: a plain-C99 client must compile against the header and link the library ------------
def _build_c_client(tmp_path):
    import shutil
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "pylops_mpi_b200")
    exe = str(tmp_path / "abi_smoke")
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(root, "include"),
                    os.path.join(root, "tests", "abi", "abi_smoke.c"), "-o", exe, "-L", libdir, "-lb200lops", "-lm",
                    f"-Wl,-rpath,{libdir}"], check=True, timeout=120)
    return exe


def test_c99_client_compiles_and_fails_loudly_without_gpu(tmp_path):
    import subprocess
    import torch
    exe = _build_c_client(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    res = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert res.returncode == 2 and "b2_ctx_create" in res.stderr     # no CPU fallback: the product path needs the GPU


def test_reference_import_paths_and_names():
    """a pylops-mpi user switching packages finds the same module paths / public names (reference
    pylops_mpi/__init__.py, basicoperators/__init__.py:22-47, optimization/, signalprocessing/, waveeqprocessing/)"""
    import importlib
    pm = importlib.import_module("pylops_mpi_b200")
    for name in ("DistributedArray", "Partition", "StackedDistributedArray", "MPILinearOperator", "asmpilinearoperator",
                 "MPIStackedLinearOperator", "MPIMatrixMult", "MPIBlockDiag", "MPIStackedBlockDiag", "MPIVStack",
                 "MPIStackedVStack", "MPIHStack", "MPIFirstDerivative", "MPISecondDerivative", "MPILaplacian",
                 "MPIGradient", "MPIFredholm1", "MPIMDC", "cg", "cgls", "ista", "fista", "dottest"):
        assert hasattr(pm, name), name
    for mod, names in (("basicoperators", ("MPIMatrixMult", "MPIBlockDiag", "MPIStackedBlockDiag", "MPIVStack",
                                           "MPIStackedVStack", "MPIHStack", "MPIFirstDerivative", "MPISecondDerivative",
                                           "MPILaplacian", "MPIGradient")),
                       ("basicoperators.Gradient", ("MPIGradient",)),
                       ("basicoperators.MatrixMult", ("MPIMatrixMult", "active_grid_comm", "local_block_split", "block_gather")),
                       ("StackedLinearOperator", ("MPIStackedLinearOperator",)),
                       ("LinearOperator", ("MPILinearOperator", "asmpilinearoperator")),
                       ("DistributedArray", ("DistributedArray", "Partition", "local_split", "StackedDistributedArray")),
                       ("signalprocessing", ("MPIFredholm1",)), ("signalprocessing.Fredholm1", ("MPIFredholm1",)),
                       ("waveeqprocessing", ("MPIMDC",)), ("waveeqprocessing.MDC", ("MPIMDC",)),
                       ("optimization.basic", ("cg", "cgls")), ("optimization.cls_basic", ("CG", "CGLS")),
                       ("optimization.sparsity", ("ista", "fista")), ("optimization.cls_sparsity", ("ISTA", "FISTA")),
                       ("optimization.eigs", ("power_iteration",)), ("utils.dottest", ("dottest",)),
                       ("utils.decorators", ("reshaped",))):
        m = importlib.import_module("pylops_mpi_b200." + mod)
        for n in names:
            assert hasattr(m, n), f"{mod}.{n}"


# ---- property tests of the integer bookkeeping (bit-exact rows a1 / a8) -----------------------------------------
from hypothesis import given, settings, strategies as st  # noqa: E402


@settings(max_examples=200, deadline=None)
@given(st.lists(st.integers(0, 50), min_size=1, max_size=9), st.data())
def test_repartition_plan_property(src, data):
    """any source partition -> any destination partition of the same total: every element moves exactly once,
    sends and receives pair up, nothing is sent to oneself twice"""
    from pylops_mpi_b200.utils.partition import repartition_plan
    P, n = len(src), sum(src)
    cuts = sorted(data.draw(st.lists(st.integers(0, n), min_size=P - 1, max_size=P - 1)))
    dst = [b - a for a, b in zip([0] + cuts, cuts + [n])]
    x = np.arange(n)
    xs = np.split(x, np.cumsum(src)[:-1])
    out = [np.full(d, -1) for d in dst]
    for r in range(P):
        sends, recvs = repartition_plan(src, dst, r)
        assert sum(c for _, _, c in sends) == src[r] and sum(c for _, _, c in recvs) == dst[r]
        assert len({p for p, _, _ in sends}) == len(sends) and len({p for p, _, _ in recvs}) == len(recvs)
        for peer, off, cnt in sends:
            assert cnt > 0
            back = [q for q in repartition_plan(src, dst, peer)[1] if q[0] == r]
            assert len(back) == 1 and back[0][2] == cnt
            out[peer][back[0][1]:back[0][1] + cnt] = xs[r][off:off + cnt]
    assert np.array_equal(np.concatenate(out) if n else np.zeros(0, int), x)


@settings(max_examples=200, deadline=None)
@given(st.integers(0, 10 ** 7), st.integers(1, 64))
def test_local_split_sizes_property(n, P):
    from pylops_mpi_b200.utils.partition import local_split_sizes, offsets
    s = local_split_sizes(n, P)
    assert len(s) == P and sum(s) == n and max(s) - min(s) <= 1 and s == sorted(s, reverse=True)
    off = offsets(s)
    assert off[0] == 0 and off[-1] == n and len(off) == P + 1


@pytest.mark.parametrize("dims", [(11, 21), (600,), (100, 7), (101, 5, 3), (79, 4, 5)])
@pytest.mark.parametrize("P", [2, 3, 4, 8])
def test_strict_parity_mode_raises_exactly_where_the_reference_does(dims, P):
    """B2_STRICT_REFERENCE / decorators.STRICT_PARITY: the native re-partition handles any overlap; the strict
    check must raise iff the reference's neighbour-only add_ghost_cells plan does (DistributedArray.py:918-923),
    i.e. iff the oracle's restatement of @reshaped raises for the same split (e.g. (11, 21) at P = 8)."""
    from types import SimpleNamespace
    from pylops_mpi_b200.utils import decorators as D
    from pylops_mpi_b200.utils.partition import local_split_sizes
    n = int(np.prod(dims))
    src = local_split_sizes(n, P)
    ext = local_split_sizes(dims[0], P)
    dst = [e * int(np.prod(dims[1:])) for e in ext]
    x = SimpleNamespace(_local_shapes=[(s,) for s in src], size=P, global_shape=(n,))
    try:
        o.reshaped_in(o.to_dist(np.arange(float(n)), P), [(e,) + tuple(dims[1:]) for e in ext])
        ref_raises = False
    except ValueError:
        ref_raises = True
    if ref_raises:
        with pytest.raises(ValueError, match="Local Shape at rank="):
            D._strict_check(x, dst)
    else:
        D._strict_check(x, dst)


def test_cgls_graph_safety_is_conservative_and_typed():
    """CGLS replays its iteration as a CUDA graph only for operator trees made of the package's rank-local kernel
    operators (recognised by type) and whitelisted MPI classes; anything unknown (user operators, including one that
    merely shares a kernel operator's class name, MPIFredholm1's host-toggled fused mode, MDC's FFT wrappers) keeps the
    eager path"""
    from pylops_mpi_b200 import local
    from pylops_mpi_b200.optimization.cls_basic import _graph_safe

    def make(name, **attrs):
        return type(name, (), {"shape": (4, 4), **attrs})()
    blk = object.__new__(local.MatrixMult)                                   # a kernel operator, no device needed
    assert _graph_safe(make("MPIBlockDiag", ops=[blk]))
    assert not _graph_safe(make("MPIBlockDiag", ops=[make("MatrixMult")]))  # safe by type, not by class name
    assert _graph_safe(make("_ProductLinearOperator", args=(make("MPIBlockDiag", ops=[blk]), make("MPIFirstDerivative"))))
    assert _graph_safe(make("_ScaledLinearOperator", args=(make("MPIVStack", ops=[blk]), 2.0)))
    assert not _graph_safe(make("MPIFredholm1"))
    assert not _graph_safe(make("MPILinearOperator"))                       # wrapper of an arbitrary local operator
    assert not _graph_safe(make("MPIBlockDiag", ops=[make("SomeUserOperator")]))
    assert not _graph_safe(make("_SumLinearOperator", args=(make("MPIBlockDiag", ops=[blk]), make("MPIFredholm1"))))


def test_stacked_operator_algebra_without_a_device():
    """shape / type bookkeeping and the error behaviour of the MPIStackedLinearOperator algebra
    (StackedLinearOperator.py:117-228, 268-293) need no device: checked with shape-only stand-in operators"""
    import pylops_mpi_b200 as pm

    class Shape:
        def __init__(self, m, n):
            self.shape, self.dtype = (m, n), np.dtype(np.float64)

    V1, V2 = (pm.MPIStackedVStack([Shape(4, 3), Shape(5, 3)]) for _ in range(2))
    B1, B2 = pm.MPIStackedBlockDiag([Shape(4, 3), Shape(5, 3)]), pm.MPIStackedBlockDiag([Shape(3, 3)])
    assert V1.shape == (9, 3) and B1.shape == (9, 6)
    with pytest.raises(ValueError, match="both operands cannot be MPIStackedVStack"):
        V1 * V2
    with pytest.raises(ValueError, match="different number of ops"):
        B1 * B2
    with pytest.raises(ValueError, match="different number of columns"):
        pm.MPIStackedVStack([Shape(4, 3), Shape(5, 2)])
    assert (B1.H * B1).shape == (6, 6) and (B1 + B1).shape == (9, 6) and (2 * B1).shape == (9, 6)
    assert B1.H.shape == (6, 9) and (-B1).shape == (9, 6) and (B1.H * V1.H.H).shape == (6, 3)
    # the classes live where the reference keeps them; the old module path still resolves
    import pylops_mpi_b200.StackedArray as sa
    assert sa.MPIGradient is pm.MPIGradient and sa.MPIStackedLinearOperator is pm.MPIStackedLinearOperator
    assert pm.MPIGradient.__module__.endswith("basicoperators.Gradient")
    assert pm.MPIStackedLinearOperator.__module__.endswith("StackedLinearOperator")


def test_stacked_operator_dispatch_on_host_buffers():
    """matvec / rmatvec / adjoint / product dispatch of MPIStackedVStack and MPIStackedBlockDiag
    (VStack.py:152-201, BlockDiag.py:146-204, StackedLinearOperator.py:230-293) with stand-in operators working on
    host buffers: the composition glue itself never touches the device"""
    import torch
    import pylops_mpi_b200 as pm
    from pylops_mpi_b200.DistributedArray import DistributedArray
    comm = pm.get_comm_world()

    def da(v):
        t = torch.as_tensor(np.asarray(v, dtype=np.float64))
        return DistributedArray._internal((t.numel(),), [(t.numel(),)], comm, torch.float64, buffer=t)

    class Dense:
        def __init__(self, A):
            self.A, self.shape, self.dtype = np.asarray(A, float), np.shape(A), np.dtype(float)

        def matvec(self, x):
            return da(self.A @ x.local_array.numpy())

        def rmatvec(self, x):
            return da(self.A.T @ x.local_array.numpy())

    rng = np.random.default_rng(0)
    A1, A2 = rng.standard_normal((4, 3)), rng.standard_normal((5, 3))
    x = da(rng.standard_normal(3))
    y = pm.MPIStackedVStack([Dense(A1), Dense(A2)]).matvec(x)
    assert isinstance(y, pm.StackedDistributedArray) and y.narrays == 2
    np.testing.assert_allclose(y[0].local_array.numpy(), A1 @ x.local_array.numpy())
    np.testing.assert_allclose(y[1].local_array.numpy(), A2 @ x.local_array.numpy())
    B = pm.MPIStackedBlockDiag([Dense(A1), Dense(A2)])
    xs = pm.StackedDistributedArray([da(rng.standard_normal(3)), da(rng.standard_normal(3))])
    yb = B.matvec(xs)
    zb = B.H.matvec(yb)
    np.testing.assert_allclose(zb[1].local_array.numpy(), A2.T @ (A2 @ xs[1].local_array.numpy()))
    zp = (B.H * B).matvec(xs)
    np.testing.assert_allclose(zp[0].local_array.numpy(), A1.T @ (A1 @ xs[0].local_array.numpy()))
    with pytest.raises(ValueError):
        B.matvec(x)          # a plain 3-vector is not the 6-element stacked model


def test_gradient_constructor_bookkeeping(monkeypatch):
    """MPIGradient (Gradient.py:21-119) = distributed first derivative along axis 0 + one rank-local BlockDiag per
    other axis: shapes, sampling broadcast and operator types (constructor only; the device context is stubbed)"""
    import pylops_mpi_b200 as pm
    from pylops_mpi_b200 import _lib
    monkeypatch.setattr(_lib, "ctx", lambda device=None: None)
    G = pm.MPIGradient((8, 5, 3), sampling=(1.0, 0.5, 2.0), kind="centered", dtype="float64")
    assert G.shape == (3 * 120, 120) and G.dtype == np.float64
    assert [type(op).__name__ for op in G.ops] == ["MPIFirstDerivative", "MPIBlockDiag", "MPIBlockDiag"]
    G1 = pm.MPIGradient((8, 5), sampling=2.0, kind="forward", edge=True)
    assert G1.shape == (80, 40) and G1.sampling == (2.0, 2.0) and G1.edge and G1.kind == "forward"
    assert isinstance(G1, pm.MPIStackedVStack) and isinstance(G1, pm.MPIStackedLinearOperator)
