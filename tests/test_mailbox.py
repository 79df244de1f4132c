"""The peer-memory mailbox on one GPU: one ``b2_mailbox`` handle serves the scalar all-reduce, the vector all-reduce,
the all-gather and the halo exchange of ``b2_derivative_peer``, each at least twice so that both parities of its region
are used, with results equal to torch's.  Its argument checks return B2_ERR_ARG without an allocation or a launch."""
import ctypes as C

import numpy as np
import pytest
import torch

B2_OK, B2_ERR_ARG = 0, 2002
F64, SUM, MAX, MIN, CENTERED = 1, 0, 1, 2, 2
# box layout of csrc/peer.cuh: [scalar Slots | vector region | halo region], each region 256-byte aligned.  The scalar
# flags follow the 2 x 8 x 8 float64 values of Slots; the vector flags open their region.
SLOTS_BYTES = 2 * 8 * 8 * 8 + 2 * 8 * 8
VEC_OFF = -(-SLOTS_BYTES // 256) * 256
SCALAR_FLAG = 2 * 8 * 8 * 8


@pytest.fixture(scope="module")
def L():
    import pylops_mpi_b200._lib as L
    return L


def flags(box, off):
    """flag[0][0], flag[1][0] (parity 0 / 1 of rank 0) of the region header at byte offset off"""
    f = box[off:off + 2 * 8 * 8].view(torch.int64).view(2, 8)
    return int(f[0, 0]), int(f[1, 0])


def centered_ref(x, adjoint):
    """y = D x or D^T x for the centered 3-point first derivative without edge rows, sampling 1"""
    if adjoint:
        d = torch.nn.functional.pad(x[1:-1], (0, 0, 2, 2))
        return (d[:-2] - d[2:]) * 0.5
    y = torch.zeros_like(x)
    y[1:-1] = (x[2:] - x[:-2]) * 0.5
    return y


@pytest.mark.gpu
def test_one_rank_mailbox_serves_every_use(L):
    cap = 4096
    nbytes = L.lib.b2_mailbox_bytes(cap)
    halo_off = nbytes - 256 - 4 * cap
    box = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")
    boxes = (C.c_void_p * 1)(box.data_ptr())
    h = C.c_void_p()
    cases = {"null out": (0, 1, boxes, cap, None), "null boxes": (0, 1, None, cap, C.byref(h)),
             "size 0": (0, 0, boxes, cap, C.byref(h)), "size 9": (0, 9, boxes, cap, C.byref(h)),
             "rank -1": (-1, 1, boxes, cap, C.byref(h)), "rank = size": (1, 1, boxes, cap, C.byref(h)),
             "cap 0": (0, 1, boxes, 0, C.byref(h)), "cap 8": (0, 1, boxes, 8, C.byref(h))}
    got = {name: L.lib.b2_mailbox_create(*a) for name, a in cases.items()}
    assert all(rc == B2_ERR_ARG for rc in got.values()) and h.value is None, got
    assert L.lib.b2_mailbox_destroy(None) == B2_OK
    L.check(L.lib.b2_mailbox_create(0, 1, boxes, cap, C.byref(h)), "b2_mailbox_create")
    st, ctx = L.stream(), L.ctx()
    g = torch.Generator(device="cuda").manual_seed(7)
    try:
        for lo, hi in ((0, SLOTS_BYTES), (VEC_OFF, VEC_OFF + 256), (halo_off, halo_off + 256)):
            assert not box[lo:hi].any(), f"header [{lo}, {hi}) not zeroed by b2_mailbox_create"

        # scalar all-reduce: four calls, both parities; one rank's reduction is its own values
        for op, k in ((SUM, 8), (MAX, 3), (MIN, 1), (SUM, 5)):
            v = torch.randn(k, dtype=torch.float64, device="cuda", generator=g)
            want = v.clone()
            L.check(L.lib.b2_peer_allreduce(h, v.data_ptr(), k, op, st), "b2_peer_allreduce")
            torch.cuda.synchronize()
            assert torch.equal(v, want), f"op {op}, k {k}"

        # the halo exchange inside the stencil kernel: forward, then adjoint
        for adjoint in (0, 1):
            x = torch.randn(16, 64, dtype=torch.float64, device="cuda", generator=g)
            y = torch.full_like(x, np.nan)
            L.check(L.lib.b2_derivative_peer(ctx, h, x.data_ptr(), y.data_ptr(), 16, 64, 0, 16, 1, CENTERED, 3, 0,
                                             1.0, adjoint, F64, st), "b2_derivative_peer")
            torch.cuda.synchronize()
            assert torch.equal(y, centered_ref(x, adjoint)), f"adjoint {adjoint}"

        # vector all-reduce (a tail past the 16-byte words) and all-gather (16- and 4-byte copy words)
        for dt, n in ((torch.float32, 1001), (torch.float64, 777)):
            v = torch.randn(n, dtype=dt, device="cuda", generator=g)
            want = v.clone()
            L.check(L.lib.b2_peer_vec_allreduce(h, v.data_ptr(), n, L.code(dt), st), "b2_peer_vec_allreduce")
            torch.cuda.synchronize()
            assert torch.equal(v, want), f"{dt}, n {n}"
        for dt, n, off in ((torch.float64, 5000, 0), (torch.float32, 333, 1)):
            send = torch.randn(n + off, dtype=dt, device="cuda", generator=g)[off:]
            recv = torch.full((n + off,), np.nan, dtype=dt, device="cuda")[off:]
            counts = (C.c_size_t * 1)(n)
            L.check(L.lib.b2_peer_vec_allgatherv(h, send.data_ptr(), recv.data_ptr(), counts, L.code(dt), st),
                    "b2_peer_vec_allgatherv")
            torch.cuda.synchronize()
            assert torch.equal(recv, send), f"{dt}, n {n}, offset {off}"

        # every use kept its own sequence counter and alternated parities: 4 scalar calls, 4 vector calls
        assert flags(box, SCALAR_FLAG) == (4, 3)
        assert flags(box, VEC_OFF) == (4, 3)

        # null handles and out-of-range sizes are refused before any launch
        v = torch.ones(16, dtype=torch.float64, device="cuda")
        counts = (C.c_size_t * 1)(L.lib.b2_peer_vec_max_bytes() // 8 + 1)
        bad = {
            "allreduce null": L.lib.b2_peer_allreduce(None, v.data_ptr(), 1, SUM, st),
            "allreduce k 0": L.lib.b2_peer_allreduce(h, v.data_ptr(), 0, SUM, st),
            "allreduce k 9": L.lib.b2_peer_allreduce(h, v.data_ptr(), 9, SUM, st),
            "allreduce op 3": L.lib.b2_peer_allreduce(h, v.data_ptr(), 1, 3, st),
            "vec null": L.lib.b2_peer_vec_allreduce(None, v.data_ptr(), 16, F64, st),
            "vec too long": L.lib.b2_peer_vec_allreduce(h, v.data_ptr(), L.lib.b2_peer_vec_max_bytes() // 8 + 1,
                                                        F64, st),
            "gather null": L.lib.b2_peer_vec_allgatherv(None, v.data_ptr(), v.data_ptr(), counts, F64, st),
            "gather too long": L.lib.b2_peer_vec_allgatherv(h, v.data_ptr(), v.data_ptr(), counts, F64, st),
            "derivative null": L.lib.b2_derivative_peer(ctx, None, v.data_ptr(), v.data_ptr(), 2, 8, 0, 2, 1,
                                                        CENTERED, 3, 0, 1.0, 0, F64, st),
        }
        torch.cuda.synchronize()
        assert all(rc == B2_ERR_ARG for rc in bad.values()), bad
        assert torch.equal(v, torch.ones_like(v))
        assert flags(box, SCALAR_FLAG) == (4, 3) and flags(box, VEC_OFF) == (4, 3)
    finally:
        L.check(L.lib.b2_mailbox_destroy(h), "b2_mailbox_destroy")

