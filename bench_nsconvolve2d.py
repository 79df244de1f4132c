"""Measure the non-stationary 2-D convolution kernel (b2_nsconvolve2d, csrc/nsconvolve2d.cu) on one GPU and print
JSON.

    python bench_nsconvolve2d.py [--iters 10] [--warmup 2]

Workload: one (2048, 2048) image per GPU, a 32 x 32 bank of filters at the points 32 + 64 a along both axes (every
image point between four filters, both edges extrapolated), filters of 31 x 31 and 61 x 61 taps (PSF windows),
float32 and float64, forward and adjoint.  Per line:
  - CUDA-event time of b2_nsconvolve2d (best of 3 alternating rounds);
  - the algorithmic rate 2 nx nz nhx nhz flop over that time, and its fraction of the data-sheet FP32 (67 TF/s) or
    FP64 vector (34 TF/s) rate of an H100 SXM;
  - the ratio to a stationary floor: cuDNN conv2d of the image with ONE filter of the same size (TF32 off);
  - the ratio to the torch route for the same non-stationary map: the bilinear decomposition from library calls
    (``unfold`` cuts every filter's weighted support patch, one depthwise cuDNN ``conv2d`` runs all filters, ``fold``
    sums the overlapping outputs), and the largest difference between the two results relative to max |y|.
Also ms per iteration of cgls on MPIBlockDiag([NonStationaryConvolve2D]) in float32.  The card name and power limit
are read in the same run; nothing is set.
"""
import argparse
import json

import numpy as np
import torch
import torch.nn.functional as F

import pylops_mpi_b200 as pm
from bench_convolve import FLOPS, card, time_ms

N, NF, DH, OH = 2048, 32, 64, 32
NHS = (31, 61)


def axis_weights(n, nf, oh, dh):
    """(nf, n) float64 weights of every filter at every sample (the operator's per-axis interpolation)"""
    j = np.arange(n)
    v = (j - oh) / dh
    lo = np.floor(v)
    W = np.zeros((nf, n))
    left = lo < 0
    right = lo >= nf - 1
    mid = ~(left | right)
    W[0, left] = 1.0
    W[nf - 1, right] = 1.0
    l, w = lo[mid].astype(int), (v - lo)[mid]
    W[l, j[mid]] += 1.0 - w
    W[l + 1, j[mid]] += w
    return W


class TorchRoute:
    """the non-stationary map from torch library calls: filter (a, b) acts on the patch [oh + (a - 1) dh, oh + (a + 1)
    dh) x [...] that holds its support, weighted by W_ab = wx_a wz_b (forward: before a depthwise convolution;
    adjoint: after a depthwise correlation over the patch and a halo of hc)"""

    def __init__(self, hs, dt):
        self.nh = hs.shape[-1]
        self.hc = self.nh // 2
        # every support fits its patch when OH <= DH and N <= OH + NF DH
        assert OH <= DH and N <= OH + NF * DH
        wx = torch.as_tensor(axis_weights(N, NF, OH, DH))
        pad = torch.zeros(NF, 2 * DH, dtype=wx.dtype)
        wxp = torch.cat([pad[:, :DH], wx, pad], 1)                   # sample s at index s + DH
        # filter a's patch starts at sample OH + (a - 1) DH, index OH + a DH
        wpatch = torch.stack([wxp[a, OH + a * DH:OH + (a + 2) * DH] for a in range(NF)])   # (NF, 2 DH)
        self.W = (wpatch[:, None, :, None] * wpatch[None, :, None, :]).to(dt).reshape(NF * NF, 2 * DH, 2 * DH).cuda()
        self.h = hs.reshape(NF * NF, 1, self.nh, self.nh).contiguous()
        self.hflip = torch.flip(self.h, (2, 3)).contiguous()

    def forward(self, x):
        P, K, hc = 2 * DH, self.nh, self.hc
        xp = F.pad(x.view(1, 1, N, N), (DH, DH + DH, DH, DH + DH))
        u = xp[0, 0, OH:, OH:].unfold(0, P, DH).unfold(1, P, DH)[:NF, :NF]       # (NF, NF, P, P)
        u = u.reshape(1, NF * NF, P, P) * self.W
        o = F.conv2d(u, self.hflip, padding=K - 1, groups=NF * NF)                # (1, NF^2, P + K - 1, ...)
        q = P + K - 1
        o = o.reshape(1, NF * NF, q * q).view(1, NF, NF, q * q).permute(0, 3, 1, 2).reshape(1, q * q, NF * NF)
        size = (DH * (NF - 1) + q, DH * (NF - 1) + q)
        y = F.fold(o, size, q, stride=DH)                                        # sums the overlapping patches
        r0 = DH - OH + hc                            # patch 0 starts at sample OH - DH, its output hc before that
        return y[0, 0, r0:r0 + N, r0:r0 + N]

    def adjoint(self, y):
        P, K, hc = 2 * DH, self.nh, self.hc
        q = P + K - 1
        lo = DH + hc                                 # padding before sample 0: patch 0's window starts at OH - DH - hc
        yp = F.pad(y.view(1, 1, N, N), (lo, lo + DH + K, lo, lo + DH + K))
        s0 = OH - DH - hc + lo
        v = yp[0, 0, s0:, s0:].unfold(0, q, DH).unfold(1, q, DH)[:NF, :NF].reshape(1, NF * NF, q, q)
        o = F.conv2d(v, self.h, groups=NF * NF) * self.W                          # (1, NF^2, P, P)
        o = o.reshape(1, NF, NF, P * P).permute(0, 3, 1, 2).reshape(1, P * P, NF * NF)
        x = F.fold(o, (DH * (NF - 1) + P, DH * (NF - 1) + P), P, stride=DH)
        r0 = DH - OH
        return x[0, 0, r0:r0 + N, r0:r0 + N]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    ihs = OH + DH * np.arange(NF)
    res = {"device": card(), "image": [N, N], "nfilt": [NF, NF], "ih": f"{OH} + {DH} a", "results": []}
    out = res["results"]
    gen = torch.Generator(device="cuda").manual_seed(0)
    for nh in NHS:
        for dt in (torch.float32, torch.float64):
            hs = torch.randn(NF, NF, nh, nh, device="cuda", dtype=dt, generator=gen)
            op = pm.local.NonStationaryConvolve2D((N, N), hs, ihs, ihs, dtype=str(dt).replace("torch.", ""))
            x = torch.randn(N * N, device="cuda", dtype=dt, generator=gen)
            y = torch.empty_like(x)
            h1 = hs[NF // 2, NF // 2].reshape(1, 1, nh, nh).contiguous()
            route = TorchRoute(hs, dt)
            for adj in (0, 1):
                kern = (lambda: op.rmatvec(x, out=y)) if adj else (lambda: op.matvec(x, out=y))
                floor = lambda: F.conv2d(x.view(1, 1, N, N), h1, padding=nh // 2)        # noqa: E731
                tr = (lambda: route.adjoint(x.view(N, N))) if adj else (lambda: route.forward(x.view(N, N)))
                fns = {"ns": kern, "floor": floor, "torch": tr}
                ms = {k: [] for k in fns}
                for _ in range(3):                     # alternate, so that clock and neighbour noise hit each alike
                    for k, fn in fns.items():
                        ms[k].append(time_ms(fn, a.iters, a.warmup))
                best = {k: min(v) for k, v in ms.items()}
                kern()
                ref = tr().reshape(-1)
                flop = 2 * N * N * nh * nh
                out.append({"name": f"{'adj' if adj else 'fwd'} NonStationaryConvolve2D", "dtype": str(dt)[6:],
                            "nh": [nh, nh], "ms": round(best["ns"], 3),
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

    # cgls on MPIBlockDiag([NonStationaryConvolve2D]), float32: ms per iteration, end to end
    res["cgls"] = []
    for nh in NHS:
        hs = torch.randn(NF, NF, nh, nh, device="cuda", dtype=torch.float32, generator=gen)
        BDiag = pm.MPIBlockDiag([pm.local.NonStationaryConvolve2D((N, N), hs, ihs, ihs, dtype="float32")])
        d = BDiag @ pm.DistributedArray.to_dist(torch.randn(N * N, device="cuda", dtype=torch.float32, generator=gen))
        x0 = pm.DistributedArray.to_dist(torch.zeros(N * N, device="cuda", dtype=torch.float32))
        pm.cgls(BDiag, d, x0=x0, niter=2, tol=0.0)
        niter = max(a.iters, 5)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _, _, iiter, _, _, _ = pm.cgls(BDiag, d, x0=x0, niter=niter, tol=0.0)
        e1.record()
        torch.cuda.synchronize()
        res["cgls"].append({"dtype": "float32", "nh": [nh, nh], "iterations": int(iiter),
                            "ms_per_iteration": round(e0.elapsed_time(e1) / max(int(iiter), 1), 3)})
        del BDiag, d, x0
    print(json.dumps(res))


if __name__ == "__main__":
    main()
