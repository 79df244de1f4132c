"""The shared apply of the rank-local kernel operators (``local._KernelOperator``): the result dtype for every data
dtype, ``out=`` in every form against ``out=None`` bit for bit, complex data equal to its real and imaginary parts,
length errors, no allocation on the direct path, and CUDA-graph safety by type."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

F32, F64, C64, C128 = torch.float32, torch.float64, torch.complex64, torch.complex128
XDTYPES = (F32, F64, C64, C128)

# result dtype of an apply to data of dtype float32, float64, complex64, complex128
RESULT = {
    "MatrixMult": (F32, F32, C64, C128),                # float32 A; complex data: each part a float32 GEMV
    "MatrixMult-complex": (C64, C64, C64, C64),         # complex64 A
    "FirstDerivative": (F32, F32, C64, C128),           # float32; complex data: one launch over (re, im) pairs
    "SecondDerivative": (F64, F64, C128, C128),         # float64
    "Convolve1D": (F32, F32, C64, C128),                # float32
    "PoststackLinearModelling": (F64, F64, C128, C128),  # float64 wavelet
    "Kirchhoff": (F32, F64, C64, C128),                 # float32; float64 data run in float64; complex part by part
    "NonStationaryConvolve1D": (F32, F32, C64, C128),   # float32 real taps; complex data: one launch, promoted
    "NonStationaryConvolve2D": (F32, F32, C64, C128),   # float32
    "NonStationaryConvolve2D-float64": (F64, F64, C128, C128),
    "NonStationaryConvolve3D": (F32, F32, C64, C128),   # float32
    "NonStationaryConvolve3D-float64": (F64, F64, C128, C128),
    "NonStationaryFilters1D": (F64, F64, C128, C128),   # float64; complex data part by part
    "NonStationaryFilters2D": (F32, F32, C64, C128),    # float32
    "NonStationaryFilters2D-float64": (F64, F64, C128, C128),
    "Radon2D": (F64, F64, C128, C128),                  # float64 real taps
    "Radon3D": (F32, F32, C64, C128),                   # float32
}
SQUARE = ("MatrixMult", "FirstDerivative", "SecondDerivative", "Convolve1D", "PoststackLinearModelling",
          "NonStationaryConvolve1D", "NonStationaryConvolve2D", "NonStationaryConvolve2D-float64",
          "NonStationaryConvolve3D", "NonStationaryConvolve3D-float64")
REAL_OF = {C64: F32, C128: F64}


@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def make(pm, name):
    rng = np.random.default_rng(5)
    L = pm.local
    if name == "MatrixMult":
        return L.MatrixMult(rng.standard_normal((6, 6)).astype(np.float32))
    if name == "MatrixMult-complex":
        return L.MatrixMult((rng.standard_normal((7, 5)) + 1j * rng.standard_normal((7, 5))).astype(np.complex64))
    if name == "FirstDerivative":
        return L.FirstDerivative((6, 7), axis=1, sampling=0.5, dtype=np.float32)
    if name == "SecondDerivative":
        return L.SecondDerivative((5, 4, 3), axis=1, edge=True, dtype=np.float64)
    if name == "Convolve1D":
        return L.Convolve1D((9, 4), rng.standard_normal(5), offset=2, axis=0, dtype="float32")
    if name == "PoststackLinearModelling":
        return L.PoststackLinearModelling(rng.standard_normal(7), nt0=12, spatdims=3)
    if name == "Kirchhoff":
        srcs = np.array([[0.0, 20.0], [0.0, 0.0]])
        recs = np.array([[10.0, 30.0, 40.0], [0.0, 0.0, 0.0]])
        return L.Kirchhoff(np.arange(4) * 10.0, np.arange(5) * 10.0, np.arange(32) * 0.004, srcs, recs, 1000.0,
                           np.array([1.0, -2.0, 4.0, -1.0, 0.5]), 2, mode="analytic", dtype="float32")
    name, _, dt = name.partition("-")
    dt = dt or "float32"
    if name == "NonStationaryConvolve1D":
        return L.NonStationaryConvolve1D((9, 4), rng.standard_normal((3, 5)), [1, 4, 7], axis=0, dtype=dt)
    if name == "NonStationaryConvolve2D":
        return L.NonStationaryConvolve2D((6, 5), rng.standard_normal((2, 2, 3, 3)), [1, 4], [1, 3], dtype=dt)
    if name == "NonStationaryConvolve3D":
        return L.NonStationaryConvolve3D((5, 4, 6), rng.standard_normal((2, 2, 2, 3, 3, 3)), [1, 3], [1, 2], [1, 4],
                                         dtype=dt)
    if name == "NonStationaryFilters1D":
        return L.NonStationaryFilters1D(rng.standard_normal(12), 5, [3, 8], dtype="float64")
    if name == "NonStationaryFilters2D":
        return L.NonStationaryFilters2D(rng.standard_normal((10, 9)), (3, 5), [2, 6], [1, 4], dtype=dt)
    t = np.arange(16) * 0.004
    if name == "Radon2D":
        return L.Radon2D(t, np.arange(5) * 10.0, np.linspace(-1e-3, 1e-3, 4), dtype="float64")
    if name == "Radon3D":
        return L.Radon3D(t, np.arange(3) * 20.0, np.arange(4) * 10.0, np.linspace(-1e-3, 1e-3, 2),
                         np.linspace(-2e-3, 2e-3, 3), dtype="float32")
    raise KeyError(name)


def sizes(op, adjoint):
    """(n_in, n_out) of the apply"""
    return (op.shape[0], op.shape[1]) if adjoint else (op.shape[1], op.shape[0])


def data(n, dt, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, dtype=torch.float64, generator=g)
    if dt.is_complex:
        x = torch.complex(x, torch.randn(n, dtype=torch.float64, generator=g))
    return x.to(dt).cuda()


def other(dt):
    return {F32: F64, F64: F32, C64: C128, C128: C64}[dt]


@pytest.mark.parametrize("adjoint", [False, True])
@pytest.mark.parametrize("name", list(RESULT))
def test_result_dtype(pm, name, adjoint):
    op = make(pm, name)
    f = op.rmatvec if adjoint else op.matvec
    nin, nout = sizes(op, adjoint)
    for xdt, want in zip(XDTYPES, RESULT[name]):
        y = f(data(nin, xdt))
        assert y.dtype == want and y.shape == (nout,), (xdt, y.dtype)


@pytest.mark.parametrize("xdt", [F32, C128])
@pytest.mark.parametrize("adjoint", [False, True])
@pytest.mark.parametrize("name", list(RESULT))
def test_out_equals_out_none(pm, name, adjoint, xdt):
    """out= of the result dtype, of another dtype and non-contiguous: the out=None result, bit for bit"""
    op = make(pm, name)
    f = op.rmatvec if adjoint else op.matvec
    nin, nout = sizes(op, adjoint)
    x = data(nin, xdt)
    ref = f(x)
    out = torch.full((nout,), 7.0, dtype=ref.dtype, device="cuda")
    assert f(x, out=out) is out and torch.equal(out, ref)
    out = torch.full((nout,), 7.0, dtype=other(ref.dtype), device="cuda")
    f(x, out=out)
    assert torch.equal(out, ref.to(out.dtype))
    buf = torch.full((nout, 2), 7.0, dtype=ref.dtype, device="cuda")
    f(x, out=buf[:, 0])
    assert torch.equal(buf[:, 0], ref) and bool((buf[:, 1] == 7.0).all())
    assert torch.equal(f(x), ref)                                  # repeated applies: the same bits


@pytest.mark.parametrize("kind", ["real", "complex"])
@pytest.mark.parametrize("adjoint", [False, True])
@pytest.mark.parametrize("name", SQUARE)
def test_out_aliasing_x(pm, name, adjoint, kind):
    """out= that is x itself, x already of the result dtype: the out=None result on a copy of x"""
    op = make(pm, name)
    f = op.rmatvec if adjoint else op.matvec
    x = data(op.shape[0], RESULT[name][0] if kind == "real" else C128)
    ref = f(x.clone())
    assert ref.dtype == x.dtype
    assert f(x, out=x) is x and torch.equal(x, ref)


@pytest.mark.parametrize("adjoint", [False, True])
@pytest.mark.parametrize("name", list(RESULT))
def test_complex_data_equals_its_parts(pm, name, adjoint):
    """complex data: torch.complex(f(re), f(im)) bit for bit, re and im the parts the apply computes on: the parts
    themselves when it applies them one after the other, the parts in the real dtype of its launch on (re, im) pairs
    otherwise -- except where no real apply computes in that dtype (complex128 data of a float32 operator with real
    taps, computed in float64)"""
    op = make(pm, name)
    f = op.rmatvec if adjoint else op.matvec
    compared = 0
    for xdt in (C64, C128):
        x = data(sizes(op, adjoint)[0], xdt)
        ref = f(x)
        cdt = op._compute_dtype(xdt)
        pdt = REAL_OF[cdt] if cdt.is_complex else REAL_OF[xdt]
        re, im = f(x.real.to(pdt)), f(x.imag.to(pdt))
        if not cdt.is_complex or re.dtype == pdt:
            assert torch.equal(ref, torch.complex(re, im).to(ref.dtype)), xdt
            compared += 1
    assert compared or name == "MatrixMult-complex"


@pytest.mark.parametrize("name", list(RESULT))
def test_complex_into_real_out_warns_and_keeps_the_real_part(pm, name):
    op = make(pm, name)
    for adjoint in (False, True):
        f = op.rmatvec if adjoint else op.matvec
        nin, nout = sizes(op, adjoint)
        x = data(nin, C128)
        ref = f(x)
        out = torch.zeros(nout, dtype=F64, device="cuda")
        with pytest.warns(np.exceptions.ComplexWarning):
            f(x, out=out)
        assert torch.equal(out, ref.real.to(F64))


@pytest.mark.parametrize("adjoint", [False, True])
@pytest.mark.parametrize("name", list(RESULT))
def test_wrong_length_raises(pm, name, adjoint):
    op = make(pm, name)
    f = op.rmatvec if adjoint else op.matvec
    nin, nout = sizes(op, adjoint)
    dt = RESULT[name][0]
    for n in (nin - 1, nin + 1):
        with pytest.raises(ValueError, match="dimension mismatch"):
            f(torch.zeros(n, dtype=dt, device="cuda"))
    for n in (nout - 1, nout + 1):
        with pytest.raises(ValueError, match="dimension mismatch"):
            f(torch.zeros(nin, dtype=dt, device="cuda"), out=torch.zeros(n, dtype=dt, device="cuda"))


@pytest.mark.parametrize("name", list(RESULT))
def test_direct_out_allocates_nothing(pm, name):
    """after one warm-up apply, an apply into an out= of the compute dtype allocates nothing; so does the same
    apply through ``apply_into`` on the operator's ``.H``"""
    op = make(pm, name)
    dt = RESULT[name][0]
    for adjoint in (False, True):
        f = op.rmatvec if adjoint else op.matvec
        nin, nout = sizes(op, adjoint)
        x = data(nin, dt)
        out = torch.empty(nout, dtype=dt, device="cuda")
        f(x, out=out)
        torch.cuda.synchronize()
        before = torch.cuda.memory_stats()["allocation.all.allocated"]
        f(x, out=out)
        pm.local.apply_into(op.H, x, out, not adjoint)
        torch.cuda.synchronize()
        assert torch.cuda.memory_stats()["allocation.all.allocated"] - before == 0


@pytest.mark.parametrize("name", list(RESULT))
def test_graph_safe_by_type(pm, name):
    from pylops_mpi_b200.optimization.cls_basic import _graph_safe
    op = make(pm, name)

    class Plain(pm.local.LocalOperator):
        shape, dtype = op.shape, op.dtype

        def _matvec(self, x):
            return x

    assert _graph_safe(pm.MPIBlockDiag([op]))
    assert not _graph_safe(pm.MPIBlockDiag([pm.local.Transpose((2, 3), (1, 0))]))
    assert not _graph_safe(pm.MPIBlockDiag([op.H @ op]))           # a product applied one factor at a time
    assert not _graph_safe(pm.MPIBlockDiag([op.H]))
    assert not _graph_safe(pm.MPIBlockDiag([Plain()]))
