"""Measure the fused post-stack modelling kernel (b2_poststack_axis, csrc/convolve.cu) on one GPU and print JSON.

    python bench_poststack.py [--iters 20] [--warmup 3]

Workloads, on the per-GPU block (128, 1024, 1024) with nh = 41 (offset 20), float32 and float64, forward and adjoint:
  - time along axis -1 (n_inner == 1 path): the layout tutorials/poststack.py reaches once Top.H @ PPop @ Top is folded;
  - time along axis 0 of the (1024, 131072) view (middle-axis path): pylops' native layout.
On each: the fused operator (one launch), the two-launch chain FirstDerivative + Convolve1D (b2_derivative_axis and
b2_convolve_axis, the adjoint in reverse) and Convolve1D alone.  Per line: CUDA-event time, algorithmic bytes
2 N sizeof(T) over that time, and the fraction of the HBM bound (bytes / 3.35 TB/s, the data-sheet peak of an H100 SXM
at 700 W).  Also ms per iteration of cgls on MPIBlockDiag([Top.H @ PPop @ Top]) in float32.  The card name and power
limit are read in the same run.
"""
import argparse
import json

import numpy as np
import torch

import pylops_mpi_b200 as pm
from bench_convolve import HBM, SHAPE, card, time_ms

NH, OFF = 41, 20


def line(name, ms, n, dt):
    nbytes = 2 * n * torch.tensor([], dtype=dt).element_size()
    return {"name": name, "dtype": str(dt).replace("torch.", ""), "nh": NH, "ms": round(ms, 4),
            "GB_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1), "fraction_of_hbm_bound": round(nbytes / HBM / (ms * 1e-3), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    res = {"device": card(), "shape": SHAPE, "results": []}
    out = res["results"]
    n = int(np.prod(SHAPE))
    L = pm._lib
    ctx, st = L.ctx(), L.stream()
    gen = torch.Generator(device="cuda").manual_seed(0)
    for dt in (torch.float32, torch.float64):
        code = L.code(dt)
        x = torch.randn(n, device="cuda", dtype=dt, generator=gen)
        y, t = torch.empty_like(x), torch.empty_like(x)
        h = torch.randn(NH, device="cuda", dtype=dt, generator=gen)

        def fused(shp, adj):
            return lambda: L.check(L.lib.b2_poststack_axis(ctx, x.data_ptr(), y.data_ptr(), *shp, h.data_ptr(), NH,
                                                           OFF, L.FD_CENTERED, adj, code, st), "b2_poststack_axis")

        def conv(shp, adj, src, dst):
            return lambda: L.check(L.lib.b2_convolve_axis(ctx, src.data_ptr(), dst.data_ptr(), *shp, h.data_ptr(), NH,
                                                          OFF, adj, code, st), "b2_convolve_axis")

        def deriv(shp, adj, src, dst):
            return lambda: L.check(L.lib.b2_derivative_axis(ctx, src.data_ptr(), dst.data_ptr(), *shp, 1, L.FD_CENTERED,
                                                            3, 0, 1.0, adj, code, st), "b2_derivative_axis")

        for lay, shp in (("axis-1", (SHAPE[0] * SHAPE[1], SHAPE[2], 1)), ("axis0 of (1024,131072)", (1, 1024, n // 1024))):
            for adj in (0, 1):
                if adj:
                    c, d = conv(shp, 1, x, t), deriv(shp, 1, t, y)
                    chain = lambda: (c(), d())       # noqa: E731
                else:
                    d, c = deriv(shp, 0, x, t), conv(shp, 0, t, y)
                    chain = lambda: (d(), c())       # noqa: E731
                tag = f"{lay} {'adj' if adj else 'fwd'}"
                # alternate the three so that clock and neighbour noise hit each alike
                ms = {"fused": [], "chain": [], "conv": []}
                for _ in range(3):
                    ms["fused"].append(time_ms(fused(shp, adj), a.iters, a.warmup))
                    ms["chain"].append(time_ms(chain, a.iters, a.warmup))
                    ms["conv"].append(time_ms(conv(shp, adj, x, y), a.iters, a.warmup))
                for k, name in (("fused", "poststack fused"), ("chain", "FirstDerivative + Convolve1D"),
                                ("conv", "Convolve1D alone")):
                    out.append(line(f"{tag} {name}", min(ms[k]), n, dt))
        del x, y, t
        torch.cuda.empty_cache()

    # cgls on the folded tutorial operator, float32: ms per iteration, end to end
    t0 = (np.arange(NH // 2 + 1)) * 0.004
    w = (1 - 2 * (np.pi * 15 * t0) ** 2) * np.exp(-(np.pi * 15 * t0) ** 2)
    wav = np.concatenate((w[:0:-1], w)).astype(np.float32)
    ny, nx, nz = SHAPE
    PPop = pm.local.PoststackLinearModelling(wav, nt0=nz, spatdims=(ny, nx))
    Top = pm.local.Transpose((ny, nx, nz), (2, 0, 1))
    BDiag = pm.MPIBlockDiag([Top.H @ PPop @ Top])
    d = BDiag @ pm.DistributedArray.to_dist(torch.randn(n, device="cuda", dtype=torch.float32, generator=gen))
    x0 = pm.DistributedArray.to_dist(torch.zeros(n, device="cuda", dtype=torch.float32))
    pm.cgls(BDiag, d, x0=x0, niter=2, tol=0.0)
    niter = max(a.iters, 5)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _, _, iiter, _, _, _ = pm.cgls(BDiag, d, x0=x0, niter=niter, tol=0.0)
    e1.record()
    torch.cuda.synchronize()
    res["poststack_cgls"] = {"dtype": "float32", "nh": NH, "folded_operator": type(BDiag.ops[0]).__name__,
                             "iterations": int(iiter), "ms_per_iteration": round(e0.elapsed_time(e1) / max(int(iiter), 1), 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
