"""Measure the non-stationary 3-D convolution kernel (b2_nsconvolve3d, csrc/nsconvolve3d.cu) on one GPU and print
JSON.

    python bench_nsconvolve3d.py [--iters 5] [--warmup 1] [--cgls 20]

Workload: one 160^3 volume per GPU, a 5 x 5 x 5 bank of filters at the points 16 + 32 a along every axis (every
interior point between eight filters, both edges extrapolated), filters of 15^3 and 31^3 taps (PSF windows), float32
and float64, forward and adjoint.  Per line:
  - CUDA-event time of b2_nsconvolve3d (best of 3 alternating rounds);
  - the algorithmic rate 2 n nhx nhy nhz flop over that time, and its fraction of the data-sheet FP32 (67 TF/s) or
    FP64 vector (34 TF/s) rate of an H100 SXM;
  - the ratio to a stationary floor: cuDNN conv3d of the volume with ONE filter of the same size (TF32 off);
  - the ratio to the torch route for the same non-stationary map: the trilinear decomposition from library calls
    (``Tensor.unfold`` on three axes cuts every filter's weighted support patch, one grouped cuDNN ``conv3d`` runs all
    filters, the overlapping patch outputs are summed), and the largest difference between the two results relative
    to max |y|.
Then ms per iteration of cgls on MPIBlockDiag([NonStationaryConvolve3D]) in bench_kirchhoff3d.py's image
(96 x 96 x 64, (ny, nx, nz)) with a 3 x 3 x 2 bank of 15^3 and 21^3 PSFs, against cgls on that bench's 3-D Kirchhoff
(MPIVStack([Kirchhoff]), resident tables) in the same dtype, float32 and float64.  The card name and power limit are
read in the same run; nothing is set.
"""
import argparse
import json

import numpy as np
import torch
import torch.nn.functional as F

import bench_kirchhoff3d as bk
import pylops_mpi_b200 as pm
from bench_convolve import FLOPS, card, time_ms
from bench_nsconvolve2d import axis_weights

N, NF, DH, OH = 160, 5, 32, 16
NHS = (15, 31)
CGLS_NHS = (15, 21)


def timer(fn, iters, warmup):
    """time_ms, with a single timed call when one call takes more than half a second (the slow torch routes)"""
    t = time_ms(fn, 1, 0)
    return t if t > 500 else time_ms(fn, iters, warmup)


class TorchRoute:
    """the non-stationary map from torch library calls: filter (a, b, e) acts on the patch [oh + (a - 1) dh,
    oh + (a + 1) dh) x [...] x [...] that holds its support, weighted by W_abe = (wz_e wy_b) wx_a (forward: before a
    grouped convolution; adjoint: after a grouped correlation over the patch and a halo of hc)"""

    def __init__(self, hs, dt):
        self.nh = hs.shape[-1]
        self.hc = self.nh // 2
        P = 2 * DH
        # every support fits its patch when OH <= DH and N <= OH + NF DH; a patch output fits three blocks of DH
        assert OH <= DH and N <= OH + NF * DH and P + self.nh - 1 <= 3 * DH
        w = torch.as_tensor(axis_weights(N, NF, OH, DH))
        pad = torch.zeros(NF, 2 * DH, dtype=w.dtype)
        wp = torch.cat([pad[:, :DH], w, pad], 1)                      # sample s at index s + DH
        wpatch = torch.stack([wp[a, OH + a * DH:OH + (a + 2) * DH] for a in range(NF)])   # (NF, P)
        W = (wpatch[None, None, :, None, None, :] * wpatch[None, :, None, None, :, None]) * \
            wpatch[:, None, None, :, None, None]                      # (wz wy) wx
        self.W = W.to(dt).reshape(1, NF ** 3, P, P, P).cuda()
        self.h = hs.reshape(NF ** 3, 1, self.nh, self.nh, self.nh).contiguous()
        self.hflip = torch.flip(self.h, (2, 3, 4)).contiguous()

    @staticmethod
    def overlap_sum(o, nb):
        """(NF^3, nb DH, nb DH, nb DH) patch outputs at stride DH summed into one ((NF + nb - 1) DH)^3 volume"""
        o = o.reshape(NF, NF, NF, nb, DH, nb, DH, nb, DH)
        M = NF + nb - 1
        Y = o.new_zeros(M, M, M, DH, DH, DH)
        for ka in range(nb):
            for kb in range(nb):
                for ke in range(nb):
                    Y[ka:ka + NF, kb:kb + NF, ke:ke + NF] += o[:, :, :, ka, :, kb, :, ke, :]
        return Y.permute(0, 3, 1, 4, 2, 5).reshape(M * DH, M * DH, M * DH)

    def forward(self, x):
        P, K, hc = 2 * DH, self.nh, self.hc
        xp = F.pad(x.view(1, 1, N, N, N), (DH, 2 * DH) * 3)[0, 0]
        u = xp[OH:, OH:, OH:].unfold(0, P, DH).unfold(1, P, DH).unfold(2, P, DH)[:NF, :NF, :NF]
        u = u.reshape(1, NF ** 3, P, P, P) * self.W
        o = F.conv3d(u, self.hflip, padding=K - 1, groups=NF ** 3)[0]              # (NF^3, q, q, q)
        q = P + K - 1
        o = F.pad(o, (0, 3 * DH - q) * 3)
        y = self.overlap_sum(o, 3)
        r0 = DH - OH + hc                            # patch 0 starts at sample OH - DH, its output hc before that
        return y[r0:r0 + N, r0:r0 + N, r0:r0 + N]

    def adjoint(self, y):
        P, K, hc = 2 * DH, self.nh, self.hc
        q = P + K - 1
        lo = DH + hc                                 # padding before sample 0: patch 0's window starts at OH - DH - hc
        yp = F.pad(y.view(1, 1, N, N, N), (lo, lo + DH + K) * 3)[0, 0]
        s0 = OH - DH - hc + lo
        v = yp[s0:, s0:, s0:].unfold(0, q, DH).unfold(1, q, DH).unfold(2, q, DH)[:NF, :NF, :NF]
        o = F.conv3d(v.reshape(1, NF ** 3, q, q, q), self.h, groups=NF ** 3) * self.W          # (1, NF^3, P, P, P)
        x = self.overlap_sum(o[0], 2)
        r0 = DH - OH
        return x[r0:r0 + N, r0:r0 + N, r0:r0 + N]


def kernel_lines(a, out, gen):
    ihs = OH + DH * np.arange(NF)
    n = N ** 3
    for nh in NHS:
        for dt in (torch.float32, torch.float64):
            hs = torch.randn(NF, NF, NF, nh, nh, nh, device="cuda", dtype=dt, generator=gen)
            op = pm.local.NonStationaryConvolve3D((N, N, N), hs, ihs, ihs, ihs, dtype=str(dt).replace("torch.", ""))
            x = torch.randn(n, device="cuda", dtype=dt, generator=gen)
            y = torch.empty_like(x)
            h1 = hs[NF // 2, NF // 2, NF // 2].reshape(1, 1, nh, nh, nh).contiguous()
            route = TorchRoute(hs, dt)
            for adj in (0, 1):
                kern = (lambda: op.rmatvec(x, out=y)) if adj else (lambda: op.matvec(x, out=y))
                floor = lambda: F.conv3d(x.view(1, 1, N, N, N), h1, padding=nh // 2)        # noqa: E731
                tr = (lambda: route.adjoint(x.view(N, N, N))) if adj else (lambda: route.forward(x.view(N, N, N)))
                fns = {"ns": kern, "floor": floor, "torch": tr}
                ms = {k: [] for k in fns}
                for _ in range(3):                     # alternate, so that clock and neighbour noise hit each alike
                    for k, fn in fns.items():
                        ms[k].append(timer(fn, a.iters, a.warmup))
                best = {k: min(v) for k, v in ms.items()}
                kern()
                ref = tr().reshape(-1)
                flop = 2 * n * nh ** 3
                out.append({"name": f"{'adj' if adj else 'fwd'} NonStationaryConvolve3D", "dtype": str(dt)[6:],
                            "nh": [nh] * 3, "ms": round(best["ns"], 3), "runs_ms": [round(v, 3) for v in ms["ns"]],
                            "TFLOP_per_s": round(flop / (best["ns"] * 1e-3) / 1e12, 2),
                            "fraction_of_fp_peak": round(flop / FLOPS[dt] / (best["ns"] * 1e-3), 3),
                            "stationary_cudnn_ms": round(best["floor"], 3),
                            "x_stationary_cudnn": round(best["ns"] / best["floor"], 3),
                            "torch_route_ms": round(best["torch"], 3),
                            "x_torch_route": round(best["ns"] / best["torch"], 3),
                            "torch_route_max_rel_diff": float((y - ref).abs().max() / ref.abs().max())})
                del ref
            del op, x, y, route
            torch.cuda.empty_cache()


def cgls_ms(Op, d, x0, niter):
    pm.cgls(Op, d, x0=x0, niter=2, tol=0.0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _, _, iiter, _, _, _ = pm.cgls(Op, d, x0=x0, niter=niter, tol=0.0)
    e1.record()
    torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) / max(int(iiter), 1), 3), int(iiter)


def cgls_lines(a, res, gen):
    dims = (bk.NY, bk.NX, bk.NZ)
    ni = bk.NY * bk.NX * bk.NZ
    ih = [16 + 32 * np.arange((n - 16 - 1) // 32 + 1) for n in dims]
    z, x, t, srcs, recs, y = bk.geometry()
    wav = bk.ricker(np.arange(21) * bk.DT, 20.0)
    refl = np.zeros(dims)
    refl[:, :, bk.NZ // 3], refl[:, :, 2 * bk.NZ // 3] = -1.0, 0.5
    res["cgls"] = {"image": list(dims), "nfilt": [len(i) for i in ih], "iterations": a.cgls, "results": []}
    for name, dt in (("float32", torch.float32), ("float64", torch.float64)):
        line = {"dtype": name}
        for nh in CGLS_NHS:
            hs = torch.randn(*(len(i) for i in ih), nh, nh, nh, device="cuda", dtype=dt, generator=gen)
            BDiag = pm.MPIBlockDiag([pm.local.NonStationaryConvolve3D(dims, hs, *ih, dtype=name)])
            d = BDiag @ pm.DistributedArray.to_dist(torch.randn(ni, device="cuda", dtype=dt, generator=gen))
            x0 = pm.DistributedArray.to_dist(torch.zeros(ni, device="cuda", dtype=dt))
            line[f"nsconvolve3d_{nh}^3_ms_per_iteration"] = cgls_ms(BDiag, d, x0, a.cgls)[0]
            del BDiag, d, x0
        V = pm.MPIVStack([pm.local.Kirchhoff(z, x, t, srcs, recs, bk.VEL, wav, len(wav) // 2, y=y, mode="analytic",
                                             dtype=name)])
        dd = V @ pm.DistributedArray.to_dist(refl.ravel().astype(name), partition=pm.Partition.BROADCAST)
        x0 = pm.DistributedArray.to_dist(np.zeros(ni, dtype=name), partition=pm.Partition.BROADCAST)
        line["kirchhoff_ms_per_iteration"] = cgls_ms(V, dd, x0, a.cgls)[0]
        for nh in CGLS_NHS:
            line[f"kirchhoff_over_nsconvolve3d_{nh}^3"] = round(
                line["kirchhoff_ms_per_iteration"] / line[f"nsconvolve3d_{nh}^3_ms_per_iteration"], 2)
        res["cgls"]["results"].append(line)
        del V, dd, x0
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--cgls", type=int, default=20)
    a = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    res = {"device": card(), "volume": [N, N, N], "nfilt": [NF] * 3, "ih": f"{OH} + {DH} a", "results": []}
    gen = torch.Generator(device="cuda").manual_seed(0)
    kernel_lines(a, res["results"], gen)
    cgls_lines(a, res, gen)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
