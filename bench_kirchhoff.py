"""Measure Kirchhoff demigration (b2_kirchhoff, csrc/kirchhoff.cu, and local.Kirchhoff) on one GPU and print JSON.

    python bench_kirchhoff.py [--iters 10] [--warmup 2] [--no-numba]

Per-GPU shape: a 512 x 256 image (ni = 131072), ns = 32 sources, nr = 256 receivers (8192 traces), nt = 1024, an
81-tap Ricker wavelet, constant velocity; float32 and float64.  Per line, forward and adjoint:
  - "kernel": the spreading / stacking stage alone (one b2_kirchhoff launch); "operator": the whole local.Kirchhoff
    apply (kernel + wavelet convolution);
  - CUDA-event time and (image point, trace) pairs per second;
  - for the kernel stage, two lower bounds on its time: the bytes it must move (both tables once, the image, the
    traces) over HBM bandwidth, and FP64_PER_PAIR float64 instructions per pair over the FP64 instruction rate; the
    larger one is the binding bound;
  - the same map composed from torch ops on the device (chunks of traces: index math, gather / index_add_).
Also the numba CPU loops of pylops' engine="numba" (prange over sources forward, over image points adjoint, float64,
on this host's cores, one run each), and the tutorials/lsm.py flow (81 x 60, 10 sources, 11 receivers, nt = 651):
cgls in ms per iteration.  The card name and power limit are read in the same run.
"""
import argparse
import json
import os

import numpy as np
import torch

import pylops_mpi_b200 as pm
from bench_convolve import card, time_ms

NX, NZ, NS, NR, NT, DT, VEL, DX = 512, 256, 32, 256, 1024, 0.002, 2000.0, 5.0
HBM = 3.35e12                       # B/s, H100 SXM data-sheet peak
FP64_RATE = 132 * 64 * 1.98e9       # float64 instructions / s: 132 SMs x 64 FP64 lanes x 1.98 GHz (H100 SXM boost)
# float64 instructions per pair in the inner loops' SASS (sm_90a, -O3): the IEEE divide's fast path (1 MUFU.RCP64H,
# 8 DFMA, 1 DSETP), the traveltime add, the range test (2 DSETP), trunc and its conversion back (F2I.F64, I2F.F64),
# q - it, 1 - d, two products and two adds
FP64_PER_PAIR = 21


def ricker(t, f0):
    w = (1 - 2 * (np.pi * f0 * t) ** 2) * np.exp(-(np.pi * f0 * t) ** 2)
    return np.concatenate((np.flipud(w[1:]), w), axis=0)


def geometry(nx=NX, nz=NZ, ns=NS, nr=NR, nt=NT, dx=DX):
    x, z = np.arange(nx) * dx, np.arange(nz) * dx
    srcs = np.vstack((np.linspace(0, x[-1], ns), np.zeros(ns)))
    recs = np.vstack((np.linspace(0, x[-1], nr), np.zeros(nr)))
    return z, x, np.arange(nt) * DT, srcs, recs


class TorchKirchhoff:
    """the same spreading / stacking map from torch ops, a chunk of traces at a time"""

    def __init__(self, ts, tr, nt, dt, chunk=16):
        self.ts, self.tr, self.nt, self.dt, self.chunk = ts, tr, nt, dt, chunk
        self.ns, self.ni = ts.shape
        self.nr = tr.shape[0]

    def _pairs(self, g0, g1):
        g = torch.arange(g0, g1, device="cuda")
        s, r = g // self.nr, g % self.nr
        q = (self.ts[s] + self.tr[r]) / self.dt
        it = torch.trunc(q)
        ok = (it >= 0) & (it < self.nt - 1)
        d = q - it
        it = torch.where(ok, it, torch.zeros_like(it)).long()
        return g, it, d, ok

    def forward(self, x, y):
        y.zero_()
        ntr = self.ns * self.nr
        for g0 in range(0, ntr, self.chunk):
            g, it, d, ok = self._pairs(g0, min(g0 + self.chunk, ntr))
            xv = x.to(torch.float64)[None, :] * ok
            base = (g[:, None] * self.nt + it).reshape(-1)
            y.index_add_(0, base, (xv * (1 - d)).reshape(-1).to(y.dtype))
            y.index_add_(0, base + 1, (xv * d).reshape(-1).to(y.dtype))

    def adjoint(self, x, y):
        acc = torch.zeros(self.ni, dtype=torch.float64, device="cuda")
        ntr = self.ns * self.nr
        for g0 in range(0, ntr, self.chunk):
            g, it, d, ok = self._pairs(g0, min(g0 + self.chunk, ntr))
            base = g[:, None] * self.nt + it
            a, b = x[base].to(torch.float64), x[base + 1].to(torch.float64)
            acc += ((a * (1 - d) + b * d) * ok).sum(0)
        y.copy_(acc)


def numba_loops():
    from numba import njit, prange

    @njit(parallel=True, cache=False)
    def fwd(x, y, ts, tr, dt, nt):
        ns, ni = ts.shape
        nr = tr.shape[0]
        for isrc in prange(ns):
            for irec in range(nr):
                for ii in range(ni):
                    trav = ts[isrc, ii] + tr[irec, ii]
                    it = int(trav / dt)
                    d = trav / dt - it
                    if 0 <= it < nt - 1:
                        y[isrc * nr + irec, it] += x[ii] * (1 - d)
                        y[isrc * nr + irec, it + 1] += x[ii] * d

    @njit(parallel=True, cache=False)
    def adj(x, y, ts, tr, dt, nt):
        ns, ni = ts.shape
        nr = tr.shape[0]
        for ii in prange(ni):
            for isrc in range(ns):
                for irec in range(nr):
                    trav = ts[isrc, ii] + tr[irec, ii]
                    it = int(trav / dt)
                    d = trav / dt - it
                    if 0 <= it < nt - 1:
                        y[ii] += x[isrc * nr + irec, it] * (1 - d) + x[isrc * nr + irec, it + 1] * d

    return fwd, adj


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-numba", action="store_true")
    a = ap.parse_args()
    z, x, t, srcs, recs = geometry()
    ni, ntr = NX * NZ, NS * NR
    pairs = ni * ntr
    wav = ricker(np.arange(41) * DT, 15.0)
    res = {"device": card(), "shape": {"nx": NX, "nz": NZ, "ns": NS, "nr": NR, "nt": NT, "nh": wav.size},
           "pairs": pairs, "results": []}
    out = res["results"]
    L = pm._lib
    ctx, st = L.ctx(), L.stream()
    gen = torch.Generator(device="cuda").manual_seed(0)
    for dt in (torch.float32, torch.float64):
        K = pm.local.Kirchhoff(z, x, t, srcs, recs, VEL, wav, len(wav) // 2, mode="analytic",
                               dtype="float32" if dt == torch.float32 else "float64")
        m = torch.randn(ni, device="cuda", dtype=dt, generator=gen)
        d = torch.randn(ntr * NT, device="cuda", dtype=dt, generator=gen)
        dm, md = torch.empty_like(d), torch.empty_like(m)
        esz = m.element_size()
        bound_bytes = (NS + NR) * ni * 8 + (ni + ntr * NT) * esz
        hbm_ms, fp64_ms = bound_bytes / HBM * 1e3, pairs * FP64_PER_PAIR / FP64_RATE * 1e3
        tk = TorchKirchhoff(K._ts, K._tr, NT, K.dt)

        def kern(src, dst, adj):
            return lambda: L.check(L.lib.b2_kirchhoff(ctx, src.data_ptr(), dst.data_ptr(), K._ts.data_ptr(),
                                                      K._tr.data_ptr(), ni, NS, NR, NT, K.dt, adj, L.code(dt), st),
                                   "b2_kirchhoff")

        for adj, name in ((0, "forward"), (1, "adjoint")):
            runs = {
                "kernel": kern(d, md, 1) if adj else kern(m, dm, 0),
                "operator": (lambda: K.rmatvec(d, out=md)) if adj else (lambda: K.matvec(m, out=dm)),
                "torch ops": (lambda: tk.adjoint(d, md)) if adj else (lambda: tk.forward(m, dm)),
            }
            ms = {k: [] for k in runs}
            for _ in range(2):                   # alternate, so that clock and neighbour noise hit each alike
                for k, fn in runs.items():
                    ms[k].append(time_ms(fn, a.iters if k != "torch ops" else max(a.iters // 5, 1), a.warmup))
            for k in runs:
                t_ms = min(ms[k])
                row = {"name": f"{name} {k}", "dtype": str(dt).replace("torch.", ""), "ms": round(t_ms, 3),
                       "Gpairs_per_s": round(pairs / (t_ms * 1e-3) / 1e9, 2)}
                if k == "kernel":
                    row.update({"hbm_bound_ms": round(hbm_ms, 3), "fp64_bound_ms": round(fp64_ms, 3),
                                "binding": "fp64" if fp64_ms > hbm_ms else "hbm",
                                "fraction_of_bound": round(max(fp64_ms, hbm_ms) / t_ms, 3)})
                out.append(row)
        del K, m, d, dm, md, tk
        torch.cuda.empty_cache()

    if not a.no_numba:
        try:
            import time
            fwd, adj = numba_loops()
            from pylops_mpi_b200.local import _traveltime_tables
            tsh, trh = (np.ascontiguousarray(v.T) for v in _traveltime_tables(z, x, srcs, recs, VEL))
            rng = np.random.default_rng(0)
            mh, dh = rng.standard_normal(ni), rng.standard_normal((ntr, NT))
            small = (tsh[:, :256].copy(), trh[:, :256].copy())
            fwd(mh[:256], np.zeros((ntr, NT)), *small, DT, NT)          # compile
            adj(dh, np.zeros(256), *small, DT, NT)
            t0 = time.perf_counter()
            fwd(mh, np.zeros((ntr, NT)), tsh, trh, DT, NT)
            t1 = time.perf_counter()
            adj(dh, np.zeros(ni), tsh, trh, DT, NT)
            t2 = time.perf_counter()
            res["numba_cpu"] = {"cores": os.cpu_count(), "dtype": "float64", "forward_ms": round((t1 - t0) * 1e3, 1),
                                "adjoint_ms": round((t2 - t1) * 1e3, 1)}
        except ImportError as exc:
            res["numba_cpu"] = {"skipped": str(exc)}

    # tutorials/lsm.py: cgls on MPIVStack([LSM(...).Demop]), float64, ms per iteration
    z, x, t, srcs, recs = geometry(81, 60, 10, 11, 651, 4.0)
    srcs = np.vstack((np.linspace(40, 284, 10), 10 * np.ones(10)))
    recs = np.vstack((np.linspace(40, 284, 11), 20 * np.ones(11)))
    t = np.arange(651) * 0.004
    w = ricker(t[:41], 20)
    V = pm.MPIVStack([pm.local.LSM(z, x, t, srcs, recs, 1000, w, 40, mode="analytic").Demop])
    refl = np.zeros((81, 60))
    refl[:, 30], refl[:, 50] = -1, 0.5
    dd = V @ pm.DistributedArray.to_dist(refl.ravel(), partition=pm.Partition.BROADCAST)
    x0 = pm.DistributedArray.to_dist(np.zeros(81 * 60), partition=pm.Partition.BROADCAST)
    pm.cgls(V, dd, x0=x0, niter=2, tol=0.0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _, _, iiter, _, _, _ = pm.cgls(V, dd, x0=x0, niter=100, tol=0.0)
    e1.record()
    torch.cuda.synchronize()
    res["lsm_cgls"] = {"dtype": "float64", "iterations": int(iiter),
                       "ms_per_iteration": round(e0.elapsed_time(e1) / max(int(iiter), 1), 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
