"""Measure the sliding-window operators (b2_radon_windows, csrc/radon.cu; b2_sliding, csrc/sliding.cu) on one GPU and
print JSON, one line per case.

    python bench_sliding.py [--iters 10] [--warmup 2]

Cases:
  - Sliding2D over Radon2D (linear, hyperbolic) on a section of 1024 traces x 1024 samples, nwin 64, nover 32
    (31 windows), np 64: float32 / float64, forward and adjoint, three routes timed in alternating rounds (best of 3):
    the fused launch, the per-window route (b2_radon per window, then b2_sliding: the operator with its fused path
    switched off) and a hand-built MPIBlockDiag of the 31 Radon2D (the windows' Radon only: no taper, no overlap-add);
    the largest difference between the fused and per-window outputs (relative to max |y|) on the same seeded input;
  - Sliding3D over Radon3D (linear, float32) on a 128 x 128-trace volume of 256 samples, nwin (32, 32), nover (16, 16)
    (7 x 7 windows), np 16 x 16, fused and per-window;
  - Sliding2D over MatrixMult (float32, a 64 x 256-sample window from 512 model values), the generic path;
  - ms per fista iteration on MPIBlockDiag of 4 Sliding2D(Radon2D linear, float32) sections.
The card name and power limit are read in the same run; nothing is set.
"""
import argparse
import json

import numpy as np
import torch

import pylops_mpi_b200 as pm
from bench_convolve import card, time_ms

DT, DH = 0.004, 12.5
P_RANGE = {"linear": (-1.2e-3, 1.2e-3), "hyperbolic": (1500.0, 4500.0)}
L = pm.local


def sliding2d(kind, dt, n=1024, nt=1024, nwin=64, nover=32, npp=64):
    R = L.Radon2D(np.arange(nt) * DT, np.arange(nwin) * DH, np.linspace(*P_RANGE[kind], npp), kind=kind, dtype=dt)
    nwins, dims, _, _ = L.sliding2d_design((n, nt), nwin, nover, (npp, nt))
    return R, L.Sliding2D(R, dims, (n, nt), nwin, nover), nwins


def unfused(S):
    """the same operator on the per-window route"""
    import copy
    T = copy.copy(S)
    T._fused, T._work = None, {}
    return T


def rounds(routes, iters, warmup):
    """best of 3 alternating rounds of every route, ms"""
    best = {k: float("inf") for k in routes}
    for _ in range(3):
        for k, fn in routes.items():
            best[k] = min(best[k], time_ms(fn, iters, warmup))
    return best


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
            R, S, nwins = sliding2d(kind, dt)
            U = unfused(S)
            B = pm.MPIBlockDiag([R] * nwins)
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
                ms = rounds({"fused": f, "per_window": u, "blockdiag_radon_only": b}, a.iters, a.warmup)
                f(), u()
                torch.cuda.synchronize()
                diff = float((yf - yu).abs().max() / yf.abs().max().clamp_min(1e-300))
                print(json.dumps({"name": f"Sliding2D(Radon2D {kind}) n1024 nt1024 nwin64 nover32 np64",
                                  "dtype": dt, "direction": "adjoint" if adjoint else "forward", "windows": nwins,
                                  "ms": {k: round(v, 4) for k, v in ms.items()},
                                  "fused_vs_per_window_max_rel_diff": diff}), flush=True)

    # Sliding3D over Radon3D
    nt, nwin, nover, npp = 256, (32, 32), (16, 16), (16, 16)
    R3 = L.Radon3D(np.arange(nt) * DT, np.arange(nwin[0]) * DH, np.arange(nwin[1]) * DH,
                   np.linspace(-1e-3, 1e-3, npp[0]), np.linspace(-1e-3, 1e-3, npp[1]), dtype="float32")
    nw, dims, _, _ = L.sliding3d_design((128, 128, nt), nwin, nover, (*npp, nt))
    S3 = L.Sliding3D(R3, dims, (128, 128, nt), nwin, nover, (*npp, nt))
    U3 = unfused(S3)
    for adjoint in (False, True):
        x = torch.randn(S3.shape[0] if adjoint else S3.shape[1], device="cuda", generator=gen)
        yf = torch.empty(S3.shape[1] if adjoint else S3.shape[0], device="cuda")
        yu = torch.empty_like(yf)
        f = (lambda: S3.rmatvec(x, out=yf)) if adjoint else (lambda: S3.matvec(x, out=yf))
        u = (lambda: U3.rmatvec(x, out=yu)) if adjoint else (lambda: U3.matvec(x, out=yu))
        ms = rounds({"fused": f, "per_window": u}, max(2, a.iters // 3), 1)
        f(), u()
        torch.cuda.synchronize()
        print(json.dumps({"name": "Sliding3D(Radon3D linear) 128x128 traces nt256 nwin32x32 nover16x16 np16x16",
                          "dtype": "float32", "direction": "adjoint" if adjoint else "forward",
                          "windows": nw[0] * nw[1], "ms": {k: round(v, 4) for k, v in ms.items()},
                          "fused_vs_per_window_max_rel_diff": float((yf - yu).abs().max() / yf.abs().max())}),
              flush=True)

    # Sliding2D over MatrixMult: the generic path
    A = torch.randn(64 * 256, 512, device="cuda", generator=gen)
    nwm, dims, _, _ = L.sliding2d_design((1024, 256), 64, 32, (512, 1))
    SM = L.Sliding2D(L.MatrixMult(A), dims, (1024, 256), 64, 32)
    for adjoint in (False, True):
        x = torch.randn(SM.shape[0] if adjoint else SM.shape[1], device="cuda", generator=gen)
        y = torch.empty(SM.shape[1] if adjoint else SM.shape[0], device="cuda")
        f = (lambda: SM.rmatvec(x, out=y)) if adjoint else (lambda: SM.matvec(x, out=y))
        print(json.dumps({"name": "Sliding2D(MatrixMult 16384x512) n1024 nt256 nwin64 nover32", "dtype": "float32",
                          "direction": "adjoint" if adjoint else "forward", "windows": nwm,
                          "ms": round(min(time_ms(f, a.iters, a.warmup) for _ in range(3)), 4)}), flush=True)

    # fista on 4 sections (linear, float32): ms per iteration, end to end
    _, S, _ = sliding2d("linear", "float32")
    B = pm.MPIBlockDiag([S] * 4)
    m = torch.zeros(B.shape[1], device="cuda")
    m[torch.randint(0, B.shape[1], (4 * 400,), device="cuda", generator=gen)] = 1.0
    d = B @ pm.DistributedArray.to_dist(m)
    x0 = pm.DistributedArray.to_dist(torch.zeros(B.shape[1], device="cuda"))
    alpha = 1.0 / (64 * 2 * 128)            # 1 / (||S||_1 ||S||_inf) bounds: columns <= nwin, rows <= 2 windows x 2 np
    pm.fista(B, d, x0, niter=2, eps=0.1, alpha=alpha, tol=0.0)
    niter = max(a.iters, 5)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _, iiter, _ = pm.fista(B, d, x0, niter=niter, eps=0.1, alpha=alpha, tol=0.0)
    e1.record()
    torch.cuda.synchronize()
    print(json.dumps({"name": "fista MPIBlockDiag 4 x Sliding2D(Radon2D linear) n1024 nt1024 nwin64 nover32 np64",
                      "dtype": "float32", "iterations": int(iiter),
                      "ms_per_iteration": round(e0.elapsed_time(e1) / max(int(iiter), 1), 3)}), flush=True)


if __name__ == "__main__":
    main()
