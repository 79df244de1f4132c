"""The apply frames of the dense distributed operators at one GPU.

MPIMatrixMult (SUMMA): every mode, in both directions, has the right output dtype and local shape, matches a float64
dense product within the bounds of tests/parity_checks.py, and repeats its bits on a second apply.  At one rank the
output tile is never padded; padded (ragged) tiles need a grid of several ranks and are checked by
tests/parity_checks.py and tests/multi_worker.py through tests/test_gpu_multi.py.

MPIFredholm1: at one rank an apply is exactly one product call of the library, on the tensor-core plan or the SIMT
kernel, with the data side broadcast or scattered."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


MODES = {"summa": {}, "replicated": {"replicate": True}, "stationary": {"stationary": True}}


@pytest.mark.parametrize("adjoint", [False, True])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("N,K,M,dtype", [(64, 48, 40, "float64"), (37, 29, 23, "float64"), (64, 48, 1, "float64"),
                                         (64, 128, 64, "bfloat16"), (96, 64, 1, "bfloat16")])
def test_summa_apply(pm, N, K, M, dtype, mode, adjoint):
    bf16 = dtype == "bfloat16"
    if mode == "stationary" and not (bf16 and M % 32 == 0):
        pytest.skip("stationary=True serves bf16 tiles with M % 32 == 0")
    rng = np.random.default_rng(7)
    A = torch.as_tensor(rng.standard_normal((N, K)) / 16)
    A = A.float().to(torch.bfloat16) if bf16 else A
    Op = pm.MPIMatrixMult(A, M, kind="summa", dtype=dtype, **MODES[mode])
    rows_in, rows_out = (N, K) if adjoint else (K, N)
    xv = rng.standard_normal((rows_in, M)).astype(np.float32 if bf16 else np.float64)
    x = pm.DistributedArray(global_shape=rows_in * M, dtype=xv.dtype)
    x.local_array.copy_(torch.as_tensor(xv.ravel()))
    apply = Op.rmatvec if adjoint else Op.matvec
    y = apply(x)
    assert y.local_array.dtype is (torch.float32 if bf16 else torch.float64)
    assert y.local_shape == (rows_out * M,)
    assert torch.equal(apply(x).local_array, y.local_array)
    opA = A.double().numpy().T if adjoint else A.double().numpy()
    got = y.local_array.cpu().numpy().reshape(rows_out, M)
    if bf16:
        # a single column goes through the bf16 x fp32 gemv; wider tiles round the operand to bf16 first
        xr = torch.as_tensor(xv).to(torch.bfloat16).double().numpy() if M > 1 else xv.astype(np.float64)
        bound = (np.abs(opA) @ np.abs(xr)) * rows_in * 6e-8 + (1e-4 if adjoint else 1e-6)
        assert np.all(np.abs(got - opA @ xr) <= bound)
    else:
        tol = 1e-10 if adjoint else 1e-11
        np.testing.assert_allclose(got, opA @ xv, rtol=tol, atol=tol)


@pytest.mark.parametrize("scatter_data", [False, True])
@pytest.mark.parametrize("dtype,plan", [(np.float32, True), (np.complex64, True), (np.float32, False),
                                        (np.complex64, False), (np.float64, False), (np.complex128, False)])
def test_fredholm1_single_rank_apply_is_one_product(pm, monkeypatch, dtype, plan, scatter_data):
    import pylops_mpi_b200._lib as L
    monkeypatch.setattr(pm.signalprocessing.Fredholm1, "TC_MIN_PRODUCTS", 0 if plan else 1 << 62)
    nsl, nx, ny, nz = 6, 40, 24, 9
    rng = np.random.default_rng(5)
    G = rng.standard_normal((nsl, nx, ny))
    xv = rng.standard_normal(nsl * ny * nz)
    if np.issubdtype(dtype, np.complexfloating):
        G = G + 1j * rng.standard_normal(G.shape)
        xv = xv + 1j * rng.standard_normal(xv.shape)
    Fr = pm.MPIFredholm1(G.astype(dtype), nz=nz, dtype=dtype, fused=False, scatter_data=scatter_data)
    assert (Fr._plan is not None) == plan

    def product(src, nout, adjoint):
        out = torch.empty(nout, dtype=src.dtype, device="cuda")
        if plan:
            L.check(L.lib.b2_fredholm_apply(Fr._plan, src.data_ptr(), out.data_ptr(), None, 0, int(adjoint),
                                            L.stream()), "b2_fredholm_apply")
        else:
            L.check(L.lib.b2_batched_gemm(L.ctx(), Fr.G.data_ptr(), src.data_ptr(), out.data_ptr(), nsl, nx, ny, nz,
                                          int(adjoint), L.code(src.dtype), L.stream()), "b2_batched_gemm")
        return out

    x = pm.DistributedArray.to_dist(xv.astype(dtype), partition=pm.Partition.BROADCAST)
    y = Fr @ x
    assert y.partition is (pm.Partition.SCATTER if scatter_data else pm.Partition.BROADCAST)
    assert torch.equal(y.local_array, product(x.local_array, nsl * nx * nz, False))
    xa = Fr.H @ y
    assert xa.partition is pm.Partition.BROADCAST
    assert torch.equal(xa.local_array, product(y.local_array, nsl * ny * nz, True))
    with pytest.raises(ValueError):
        Fr @ pm.DistributedArray.to_dist(xv.astype(dtype))                     # the model is broadcast
    if scatter_data:
        with pytest.raises(ValueError):
            Fr.H @ pm.DistributedArray.to_dist(y.local_array.cpu().numpy(), partition=pm.Partition.BROADCAST)
