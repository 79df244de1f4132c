"""Measure the non-stationary convolution kernels (b2_nsconvolve_axis / b2_nspoststack_axis, csrc/nsconvolve.cu) on
one GPU and print JSON.

    python bench_nsconvolve.py [--iters 20] [--warmup 3]

Workloads, on the per-GPU block (128, 1024, 1024) with nh = 41 (centre 20), float32 and float64, forward and adjoint,
along axis -1 (n_inner == 1 path: the layout Top.H @ PPop @ Top folds to) and along axis 0 of the (1024, 131072) view
(middle-axis path: pylops' native layout):
  - NonStationaryConvolve1D with 9 filters at samples 0, 128, ..., 1024, against the stationary b2_convolve_axis;
  - PoststackLinearModelling with one wavelet per time sample, against the stationary b2_poststack_axis and against
    pylops' own route for a 2-D wavelet: the dense nonstationary_convmtx (nt0 x nt0) through torch.matmul with TF32
    off, plus the derivative (b2_derivative_axis).
Per line: CUDA-event time (best of 3 alternating rounds), algorithmic bytes 2 N sizeof(T) over that time, the fraction
of the HBM bound (bytes / 3.35 TB/s, the data-sheet peak of an H100 SXM at 700 W), and the ratio to the stationary
kernel on the same line.  Also ms per iteration of cgls on MPIBlockDiag([Top.H @ PPop @ Top]) in float32, with the
2-D and with a 1-D wavelet.  The card name and power limit are read in the same run; nothing is set.
"""
import argparse
import json

import numpy as np
import torch

import pylops_mpi_b200 as pm
from bench_convolve import HBM, SHAPE, card, time_ms

NH, HC, NFILT, DH = 41, 20, 9, 128


def line(name, ms, n, dt, floor_ms=None):
    nbytes = 2 * n * torch.tensor([], dtype=dt).element_size()
    out = {"name": name, "dtype": str(dt).replace("torch.", ""), "nh": NH, "ms": round(ms, 4),
           "GB_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1),
           "fraction_of_hbm_bound": round(nbytes / HBM / (ms * 1e-3), 3)}
    if floor_ms is not None:
        out["x_stationary"] = round(ms / floor_ms, 3)
    return out


def convmtx(wav, n, hc):
    """pylops' nonstationary_convmtx(wav, n, hc, pad=(n, n)): C[i, j] = wav[j, hc + i - j]"""
    nw = wav.shape[1]
    i = torch.arange(n, device=wav.device)[:, None]
    j = torch.arange(n, device=wav.device)[None, :]
    k = hc + i - j
    ok = (k >= 0) & (k < nw)
    return torch.where(ok, wav[j.expand(n, n), k.clamp(0, nw - 1)], torch.zeros((), dtype=wav.dtype, device=wav.device))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    res = {"device": card(), "shape": SHAPE, "nfilt": NFILT, "dh": DH, "results": []}
    out = res["results"]
    n = int(np.prod(SHAPE))
    nt = SHAPE[2]
    L = pm._lib
    ctx, st = L.ctx(), L.stream()
    gen = torch.Generator(device="cuda").manual_seed(0)
    for dt in (torch.float32, torch.float64):
        code = L.code(dt)
        x = torch.randn(n, device="cuda", dtype=dt, generator=gen)
        y, t = torch.empty_like(x), torch.empty_like(x)
        h = torch.randn(NH, device="cuda", dtype=dt, generator=gen)
        hs = torch.randn(NFILT, NH, device="cuda", dtype=dt, generator=gen)
        wav = torch.randn(nt, NH, device="cuda", dtype=dt, generator=gen)
        C = convmtx(wav, nt, HC)

        def run(fn, *args):
            return lambda: L.check(fn(ctx, x.data_ptr(), y.data_ptr(), *args, code, st), fn.__name__)

        def deriv(shp, adj, src, dst):
            L.check(L.lib.b2_derivative_axis(ctx, src.data_ptr(), dst.data_ptr(), *shp, 1, L.FD_CENTERED, 3, 0, 1.0,
                                             adj, code, st), "b2_derivative_axis")

        for lay, shp in (("axis-1", (SHAPE[0] * SHAPE[1], nt, 1)), ("axis0 of (1024,131072)", (1, nt, n // nt))):
            X, Y, Tt = (v.view(-1, nt) if lay == "axis-1" else v.view(nt, -1) for v in (x, y, t))

            def dense(adj):
                # pylops' route: MatrixMult(nonstationary_convmtx) * FirstDerivative (adjoint: D^T C^T)
                def fn():
                    if lay == "axis-1":
                        if adj:
                            torch.matmul(X, C, out=Tt)
                            deriv(shp, 1, t, y)
                        else:
                            deriv(shp, 0, x, t)
                            torch.matmul(Tt, C.T, out=Y)
                    elif adj:
                        torch.matmul(C.T, X, out=Tt)
                        deriv(shp, 1, t, y)
                    else:
                        deriv(shp, 0, x, t)
                        torch.matmul(C, Tt, out=Y)
                return fn

            for adj in (0, 1):
                tag = f"{lay} {'adj' if adj else 'fwd'}"
                fns = {
                    "ns": run(L.lib.b2_nsconvolve_axis, *shp, hs.data_ptr(), NFILT, NH, HC, 0, DH, adj),
                    "conv": run(L.lib.b2_convolve_axis, *shp, h.data_ptr(), NH, HC, adj),
                    "nspost": run(L.lib.b2_nspoststack_axis, *shp, wav.data_ptr(), nt, NH, HC, 0, 1, L.FD_CENTERED,
                                  adj),
                    "post": run(L.lib.b2_poststack_axis, *shp, h.data_ptr(), NH, HC, L.FD_CENTERED, adj),
                    "dense": dense(adj),
                }
                ms = {k: [] for k in fns}
                for _ in range(3):                     # alternate, so that clock and neighbour noise hit each alike
                    for k, fn in fns.items():
                        ms[k].append(time_ms(fn, a.iters if k != "dense" else max(2, a.iters // 4), a.warmup))
                best = {k: min(v) for k, v in ms.items()}
                out.append(line(f"{tag} NonStationaryConvolve1D", best["ns"], n, dt, best["conv"]))
                out.append(line(f"{tag} Convolve1D (stationary)", best["conv"], n, dt))
                out.append(line(f"{tag} PoststackLinearModelling 2-D wavelet", best["nspost"], n, dt, best["post"]))
                out.append(line(f"{tag} PoststackLinearModelling (stationary)", best["post"], n, dt))
                out.append(line(f"{tag} dense convmtx matmul + derivative", best["dense"], n, dt, best["post"]))
        del x, y, t, X, Y, Tt
        torch.cuda.empty_cache()

    # cgls on the folded tutorial operator, float32: ms per iteration, end to end
    t0 = np.arange(NH // 2 + 1) * 0.004

    def rick(f):
        w = (1 - 2 * (np.pi * f * t0) ** 2) * np.exp(-(np.pi * f * t0) ** 2)
        return np.concatenate((w[:0:-1], w))

    ny, nx, nz = SHAPE
    wavs = {"2-D": np.stack([rick(f) for f in np.linspace(25.0, 10.0, nz)]).astype(np.float32),
            "1-D": rick(15.0).astype(np.float32)}
    res["poststack_cgls"] = {}
    xg = torch.randn(n, device="cuda", dtype=torch.float32, generator=gen)
    for name, w in wavs.items():
        PPop = pm.local.PoststackLinearModelling(w, nt0=nz, spatdims=(ny, nx))
        Top = pm.local.Transpose((ny, nx, nz), (2, 0, 1))
        BDiag = pm.MPIBlockDiag([Top.H @ PPop @ Top])
        d = BDiag @ pm.DistributedArray.to_dist(xg)
        x0 = pm.DistributedArray.to_dist(torch.zeros(n, device="cuda", dtype=torch.float32))
        pm.cgls(BDiag, d, x0=x0, niter=2, tol=0.0)
        niter = max(a.iters, 5)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _, _, iiter, _, _, _ = pm.cgls(BDiag, d, x0=x0, niter=niter, tol=0.0)
        e1.record()
        torch.cuda.synchronize()
        res["poststack_cgls"][name] = {"dtype": "float32", "nh": NH, "folded_operator": type(BDiag.ops[0]).__name__,
                                       "iterations": int(iiter),
                                       "ms_per_iteration": round(e0.elapsed_time(e1) / max(int(iiter), 1), 3)}
        del d, x0, BDiag, PPop
    print(json.dumps(res))


if __name__ == "__main__":
    main()
