"""Measure the non-stationary filter-estimation adjoint (b2_nsfilters2d_adjoint, csrc/nsfilters.cu) on one GPU and
print JSON.

    python bench_nsfilters.py [--iters 10] [--warmup 2]

Workload: the shapes of bench_nsconvolve2d.py -- one (2048, 2048) image, a 32 x 32 bank at the points 32 + 64 a along
both axes, filters of 31 x 31 and 61 x 61 taps, float32 and float64 -- where each filter's support is about 127 x 127
(many small supports, one part per filter), plus a 2 x 3 bank at (512 + 1024 a, 1023 b) with supports up to 1536 x
2048 (few huge supports, split into parts and folded).  Per line:
  - CUDA-event time of NonStationaryFilters2D's adjoint (best of 3 alternating rounds);
  - the algorithmic rate 2 nx nz nhx nhz flop over that time;
  - the ratio to NonStationaryConvolve2D's adjoint on the same image and bank, which has the same count of work;
  - the ratio to a torch route for the same map, and the largest difference between the two relative to max |g|:
    for the 32 x 32 bank ``unfold`` cuts every filter's weighted input patch and its data window and one grouped
    cuDNN ``conv2d`` correlates them all; for the 2 x 3 bank one cuDNN ``conv2d`` per filter on its support.
Also ms per iteration of cgls on MPIVStack([NonStationaryFilters2D] * 3) with 31 x 31 filters on the 32 x 32 bank, in
float32.  The card name and power limit are read in the same run; nothing is set.
"""
import argparse
import json

import numpy as np
import torch
import torch.nn.functional as F

import pylops_mpi_b200 as pm
from bench_convolve import card, time_ms
from bench_nsconvolve2d import DH, NF, NHS, OH, N, TorchRoute, axis_weights

HUGE_IHX, HUGE_IHZ = (512, 1536), (0, 1023, 2046)


class GroupedRoute(TorchRoute):
    """g_c = the correlation of d's window around filter c's patch with u_c = W_c . inp over the patch, for every
    filter in one grouped cuDNN conv2d (the patch geometry of bench_nsconvolve2d.TorchRoute)"""

    def __init__(self, inp, nh, dt):
        super().__init__(torch.zeros(NF, NF, nh, nh, dtype=dt, device="cuda"), dt)
        P = 2 * DH
        xp = F.pad(inp.view(1, 1, N, N), (DH, 2 * DH, DH, 2 * DH))
        u = xp[0, 0, OH:, OH:].unfold(0, P, DH).unfold(1, P, DH)[:NF, :NF].reshape(NF * NF, P, P) * self.W
        self.u = u.reshape(NF * NF, 1, P, P).contiguous()

    def adjoint(self, d):
        P, K, hc = 2 * DH, self.nh, self.hc
        q = P + K - 1
        lo = DH + hc
        dp = F.pad(d.view(1, 1, N, N), (lo, lo + DH + K, lo, lo + DH + K))
        s0 = OH - DH - hc + lo
        v = dp[0, 0, s0:, s0:].unfold(0, q, DH).unfold(1, q, DH)[:NF, :NF].reshape(1, NF * NF, q, q)
        return F.conv2d(v, self.u, groups=NF * NF).reshape(-1)


class PerFilterRoute:
    """g_c = conv2d(d's window around S_c, W_c . inp on S_c), one cuDNN call per filter"""

    def __init__(self, inp, nh, ihx, ihz, dt):
        self.nh, self.hc = nh, nh // 2
        wx = torch.as_tensor(axis_weights(N, len(ihx), ihx[0], ihx[1] - ihx[0])).cuda()
        wz = torch.as_tensor(axis_weights(N, len(ihz), ihz[0], ihz[1] - ihz[0])).cuda()
        self.parts = []
        for a in range(len(ihx)):
            for b in range(len(ihz)):
                sx, sz = torch.nonzero(wx[a]).ravel(), torch.nonzero(wz[b]).ravel()
                x0, x1, z0, z1 = int(sx[0]), int(sx[-1]) + 1, int(sz[0]), int(sz[-1]) + 1
                W = (wx[a, x0:x1, None] * wz[b, None, z0:z1]).to(dt)
                u = (W * inp.view(N, N)[x0:x1, z0:z1]).reshape(1, 1, x1 - x0, z1 - z0).contiguous()
                self.parts.append((x0, x1, z0, z1, u))

    def adjoint(self, d):
        hc, nh = self.hc, self.nh
        dp = F.pad(d.view(1, 1, N, N), (hc, hc, hc, hc))
        return torch.cat([F.conv2d(dp[:, :, x0:x1 + nh - 1, z0:z1 + nh - 1], u).reshape(-1)
                          for x0, x1, z0, z1, u in self.parts])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    ihs = OH + DH * np.arange(NF)
    res = {"device": card(), "image": [N, N], "results": []}
    gen = torch.Generator(device="cuda").manual_seed(0)
    lines = [(nh, dt, "32x32") for nh in NHS for dt in (torch.float32, torch.float64)]
    lines += [(31, dt, "2x3") for dt in (torch.float32, torch.float64)]
    for nh, dt, bank in lines:
        name = str(dt).replace("torch.", "")
        ihx, ihz = (ihs, ihs) if bank == "32x32" else (HUGE_IHX, HUGE_IHZ)
        inp = torch.randn(N * N, device="cuda", dtype=dt, generator=gen)
        d = torch.randn(N * N, device="cuda", dtype=dt, generator=gen)
        hs = torch.randn(len(ihx), len(ihz), nh, nh, device="cuda", dtype=dt, generator=gen)
        nsf = pm.local.NonStationaryFilters2D(inp.view(N, N), (nh, nh), ihx, ihz, dtype=name)
        nsc = pm.local.NonStationaryConvolve2D((N, N), hs, ihx, ihz, dtype=name)
        g = torch.empty(hs.numel(), device="cuda", dtype=dt)
        xa = torch.empty_like(d)
        route = GroupedRoute(inp, nh, dt) if bank == "32x32" else PerFilterRoute(inp, nh, ihx, ihz, dt)
        fns = {"nsf": lambda: nsf.rmatvec(d, out=g), "nsc": lambda: nsc.rmatvec(d, out=xa),
               "torch": lambda: route.adjoint(d)}
        ms = {k: [] for k in fns}
        for _ in range(3):                             # alternate, so that clock and neighbour noise hit each alike
            for k, fn in fns.items():
                ms[k].append(time_ms(fn, a.iters, a.warmup))
        best = {k: min(v) for k, v in ms.items()}
        fns["nsf"]()
        ref = route.adjoint(d)
        flop = 2 * N * N * nh * nh
        res["results"].append({
            "name": "adj NonStationaryFilters2D", "dtype": name, "bank": bank, "nh": [nh, nh],
            "parts_workspace_bytes": 0 if nsf._work is None else nsf._work.numel(),
            "ms": round(best["nsf"], 3), "TFLOP_per_s": round(flop / (best["nsf"] * 1e-3) / 1e12, 2),
            "nsc2d_adjoint_ms": round(best["nsc"], 3), "x_nsc2d_adjoint": round(best["nsf"] / best["nsc"], 3),
            "torch_route_ms": round(best["torch"], 3), "x_torch_route": round(best["nsf"] / best["torch"], 3),
            "torch_route_max_rel_diff": float((g - ref).abs().max() / ref.abs().max())})
        del nsf, nsc, route, ref, inp, d, hs, g, xa
        torch.cuda.empty_cache()

    # cgls on MPIVStack([NonStationaryFilters2D] * 3), float32: ms per iteration, end to end
    ops = [pm.local.NonStationaryFilters2D(torch.randn(N, N, device="cuda", generator=gen), (31, 31), ihs, ihs,
                                           dtype="float32") for _ in range(3)]
    V = pm.MPIVStack(ops)
    x = pm.DistributedArray.to_dist(torch.randn(V.shape[1], device="cuda", generator=gen),
                                    partition=pm.Partition.BROADCAST)
    y = V @ x
    x0 = pm.DistributedArray.to_dist(torch.zeros(V.shape[1], device="cuda"), partition=pm.Partition.BROADCAST)
    pm.cgls(V, y, x0=x0, niter=2, tol=0.0)
    niter = max(a.iters, 5)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _, _, iiter, _, _, _ = pm.cgls(V, y, x0=x0, niter=niter, tol=0.0)
    e1.record()
    torch.cuda.synchronize()
    res["cgls"] = {"dtype": "float32", "images": 3, "bank": [NF, NF], "nh": [31, 31], "iterations": int(iiter),
                   "ms_per_iteration": round(e0.elapsed_time(e1) / max(int(iiter), 1), 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
