"""Measure the time-space patch operators (b2_radon_patches, csrc/radon.cu; b2_patch, csrc/sliding.cu) on one GPU and
print JSON, one line per case.

    python bench_patch.py [--iters 10] [--warmup 2]

Cases:
  - Patch2D over Radon2D (linear, hyperbolic) on a section of 1024 traces x 1024 samples, nwin (64, 128), nover
    (32, 64) (31 x 15 patches), np 64: float32 / float64, forward and adjoint, three routes timed in alternating rounds
    (best of 3): the fused launch, the per-patch route (b2_radon per patch, then b2_patch: the operator with its fused
    path switched off) and a hand-built MPIBlockDiag of the 465 Radon2D (the patches' Radon only: no taper, no
    overlap-add); the largest difference between the fused and per-patch outputs (relative to max |y|) on the same
    seeded input;
  - Patch3D over Radon3D (linear, float32) on a 128 x 128-trace volume of 256 samples, nwin (32, 32, 64), nover
    (16, 16, 32) (7 x 7 x 7 patches), np 16 x 16, fused and per-patch;
  - Patch2D over MatrixMult (float32, a 64 x 128-sample patch from 512 model values), the generic path;
  - ms per fista iteration on MPIBlockDiag of 4 Patch2D(Radon2D linear, float32) sections.
The card name and power limit are read in the same run; nothing is set.
"""
import argparse
import json

import numpy as np
import torch

import pylops_mpi_b200 as pm
from bench_convolve import card, time_ms
from bench_sliding import DH, DT, P_RANGE, rounds, unfused

L = pm.local
NWIN, NOVER = (64, 128), (32, 64)


def patch2d(kind, dt, n=1024, nt=1024, npp=64):
    R = L.Radon2D(np.arange(NWIN[1]) * DT, np.arange(NWIN[0]) * DH, np.linspace(*P_RANGE[kind], npp), kind=kind,
                  dtype=dt)
    nwins, dims, _, _ = L.patch2d_design((n, nt), NWIN, NOVER, (npp, NWIN[1]))
    return R, L.Patch2D(R, dims, (n, nt), NWIN, NOVER, (npp, NWIN[1])), nwins


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    print(json.dumps({"card": card()}), flush=True)
    gen = torch.Generator(device="cuda").manual_seed(0)
    tdt = {"float32": torch.float32, "float64": torch.float64}

    for kind in ("linear", "hyperbolic"):
        for dt in ("float32", "float64"):
            R, S, nwins = patch2d(kind, dt)
            U = unfused(S)
            B = pm.MPIBlockDiag([R] * (nwins[0] * nwins[1]))
            for adjoint in (False, True):
                nin = S.shape[0] if adjoint else S.shape[1]
                x = torch.randn(nin, device="cuda", dtype=tdt[dt], generator=gen)
                yf = torch.empty(S.shape[1] if adjoint else S.shape[0], device="cuda", dtype=tdt[dt])
                yu = torch.empty_like(yf)
                f = (lambda: S.rmatvec(x, out=yf)) if adjoint else (lambda: S.matvec(x, out=yf))
                u = (lambda: U.rmatvec(x, out=yu)) if adjoint else (lambda: U.matvec(x, out=yu))
                xb = pm.DistributedArray.to_dist(torch.randn(B.shape[0] if adjoint else B.shape[1], device="cuda",
                                                             dtype=tdt[dt], generator=gen))
                b = (lambda: B.H @ xb) if adjoint else (lambda: B @ xb)
                ms = rounds({"fused": f, "per_patch": u, "blockdiag_radon_only": b}, a.iters, a.warmup)
                f(), u()
                torch.cuda.synchronize()
                diff = float((yf - yu).abs().max() / yf.abs().max().clamp_min(1e-300))
                print(json.dumps({"name": f"Patch2D(Radon2D {kind}) n1024 nt1024 nwin64x128 nover32x64 np64",
                                  "dtype": dt, "direction": "adjoint" if adjoint else "forward",
                                  "patches": nwins[0] * nwins[1], "ms": {k: round(v, 4) for k, v in ms.items()},
                                  "fused_vs_per_patch_max_rel_diff": diff}), flush=True)

    # Patch3D over Radon3D
    nwin, nover, npp = (32, 32, 64), (16, 16, 32), (16, 16)
    R3 = L.Radon3D(np.arange(nwin[2]) * DT, np.arange(nwin[0]) * DH, np.arange(nwin[1]) * DH,
                   np.linspace(-1e-3, 1e-3, npp[0]), np.linspace(-1e-3, 1e-3, npp[1]), dtype="float32")
    nw, dims, _, _ = L.patch3d_design((128, 128, 256), nwin, nover, (*npp, nwin[2]))
    S3 = L.Patch3D(R3, dims, (128, 128, 256), nwin, nover, (*npp, nwin[2]))
    U3 = unfused(S3)
    for adjoint in (False, True):
        x = torch.randn(S3.shape[0] if adjoint else S3.shape[1], device="cuda", generator=gen)
        yf = torch.empty(S3.shape[1] if adjoint else S3.shape[0], device="cuda")
        yu = torch.empty_like(yf)
        f = (lambda: S3.rmatvec(x, out=yf)) if adjoint else (lambda: S3.matvec(x, out=yf))
        u = (lambda: U3.rmatvec(x, out=yu)) if adjoint else (lambda: U3.matvec(x, out=yu))
        ms = rounds({"fused": f, "per_patch": u}, max(2, a.iters // 3), 1)
        f(), u()
        torch.cuda.synchronize()
        print(json.dumps({"name": "Patch3D(Radon3D linear) 128x128 traces nt256 nwin32x32x64 nover16x16x32 np16x16",
                          "dtype": "float32", "direction": "adjoint" if adjoint else "forward",
                          "patches": nw[0] * nw[1] * nw[2], "ms": {k: round(v, 4) for k, v in ms.items()},
                          "fused_vs_per_patch_max_rel_diff": float((yf - yu).abs().max() / yf.abs().max())}),
              flush=True)

    # Patch2D over MatrixMult: the generic path
    A = torch.randn(NWIN[0] * NWIN[1], 512, device="cuda", generator=gen)
    nwm, dims, _, _ = L.patch2d_design((1024, 1024), NWIN, NOVER, (512, 1))
    SM = L.Patch2D(L.MatrixMult(A), dims, (1024, 1024), NWIN, NOVER, (512, 1))
    for adjoint in (False, True):
        x = torch.randn(SM.shape[0] if adjoint else SM.shape[1], device="cuda", generator=gen)
        y = torch.empty(SM.shape[1] if adjoint else SM.shape[0], device="cuda")
        f = (lambda: SM.rmatvec(x, out=y)) if adjoint else (lambda: SM.matvec(x, out=y))
        print(json.dumps({"name": "Patch2D(MatrixMult 8192x512) n1024 nt1024 nwin64x128 nover32x64",
                          "dtype": "float32", "direction": "adjoint" if adjoint else "forward",
                          "patches": nwm[0] * nwm[1],
                          "ms": round(min(time_ms(f, a.iters, a.warmup) for _ in range(3)), 4)}), flush=True)

    # fista on 4 sections (linear, float32): ms per iteration, end to end
    _, S, _ = patch2d("linear", "float32")
    B = pm.MPIBlockDiag([S] * 4)
    m = torch.zeros(B.shape[1], device="cuda")
    m[torch.randint(0, B.shape[1], (4 * 400,), device="cuda", generator=gen)] = 1.0
    d = B @ pm.DistributedArray.to_dist(m)
    x0 = pm.DistributedArray.to_dist(torch.zeros(B.shape[1], device="cuda"))
    alpha = 1.0 / (64 * 4 * 128)            # 1 / (||S||_1 ||S||_inf) bounds: columns <= nwin0, rows <= 4 patches x 2 np
    pm.fista(B, d, x0, niter=2, eps=0.1, alpha=alpha, tol=0.0)
    niter = max(a.iters, 5)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _, iiter, _ = pm.fista(B, d, x0, niter=niter, eps=0.1, alpha=alpha, tol=0.0)
    e1.record()
    torch.cuda.synchronize()
    print(json.dumps({"name": "fista MPIBlockDiag 4 x Patch2D(Radon2D linear) n1024 nt1024 nwin64x128 nover32x64 np64",
                      "dtype": "float32", "iterations": int(iiter),
                      "ms_per_iteration": round(e0.elapsed_time(e1) / max(int(iiter), 1), 3)}), flush=True)


if __name__ == "__main__":
    main()
