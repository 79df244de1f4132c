"""Measure the eikonal traveltime solver (b2_eikonal_tables) and Kirchhoff(mode="eikonal") on one GPU and print JSON.

    python bench_eikonal.py [--iters 3] [--warmup 1]

Two geometries, each with a velocity of a vertical gradient times a slow lens (``velocity``):
  - "2d": tutorials/lsm.py's 81 x 60 image (h = 4 m), 10 sources, 11 receivers, nt = 651;
  - "3d": bench_kirchhoff3d.py's 96 x 96 x 64 image (h = 5 m), 8 sources, 16 x 16 receivers, nt = 1024.
Lines per geometry:
  - the table build (all ns + nr fields, one call each for sources and receivers) in ms, with the Jacobi steps, the
    passes, the share of (tile, field) blocks computed, and the table bytes one global Jacobi step would move (read
    and write every table once) over the HBM data-sheet bound; plain global Jacobi needs one such step per Jacobi
    iteration;
  - b2_kirchhoff_tables (analytic, constant velocity) at the same size, for scale;
  - 2-D only: the NumPy restatement on the host (one run), and whether the device tables equal it bit for bit;
  - the operator's float64 forward and adjoint with the eikonal tables and with analytic ones (same kernels).
The card name and power limit are read in the same run.
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np
import torch

import pylops_mpi_b200 as pm
from bench_convolve import card, time_ms

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests", "golden", "refshim"))


def ricker(t, f0):
    w = (1 - 2 * (np.pi * f0 * t) ** 2) * np.exp(-(np.pi * f0 * t) ** 2)
    return np.concatenate((np.flipud(w[1:]), w), axis=0)


def velocity(axes):
    """(1500 + 0.8 z) m/s times a lens 30 % slower at the image centre"""
    grids = np.meshgrid(*axes, indexing="ij")
    r2 = sum((g - 0.5 * (a[0] + a[-1])) ** 2 for g, a in zip(grids, axes))
    return (1500.0 + 0.8 * grids[-1]) * (1.0 - 0.3 * np.exp(-r2 / (0.2 * (axes[-2][-1] - axes[-2][0])) ** 2))


def geometry(kind):
    if kind == "2d":
        nx, nz, h, nt, dt = 81, 60, 4.0, 651, 0.004
        x, z = np.arange(nx) * h, np.arange(nz) * h
        srcs = np.vstack((np.linspace(10 * h, (nx - 10) * h, 10), np.full(10, 10.0)))
        recs = np.vstack((np.linspace(10 * h, (nx - 10) * h, 11), np.full(11, 20.0)))
        return z, x, np.arange(nt) * dt, srcs, recs, None
    ny, nx, nz, h, nt, dt = 96, 96, 64, 5.0, 1024, 0.002
    y, x, z = np.arange(ny) * h, np.arange(nx) * h, np.arange(nz) * h
    SY, SX = np.meshgrid(np.linspace(0, y[-1], 2), np.linspace(0, x[-1], 4), indexing="ij")
    srcs = np.vstack((SY.ravel(), SX.ravel(), np.zeros(8)))
    RY, RX = np.meshgrid(np.linspace(0, y[-1], 16), np.linspace(0, x[-1], 16), indexing="ij")
    recs = np.vstack((RY.ravel(), RX.ravel(), np.zeros(256)))
    return z, x, np.arange(nt) * dt, srcs, recs, y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    from pylops.waveeqprocessing import eikonal
    res = {"device": card(), "results": []}
    for kind in ("2d", "3d"):
        z, x, t, srcs, recs, y = geometry(kind)
        axes = (x, z) if y is None else (y, x, z)
        vel = velocity(axes)
        wav = ricker(np.arange(21) * (t[1] - t[0]), 20.0)
        K = pm.local.Kirchhoff(z, x, t, srcs, recs, vel, wav, len(wav) // 2, y=y, mode="eikonal")
        ni, ns, nr = K.ni, K.ns, K.nr
        full = (K.ny, K.nx, K.nz)
        h = eikonal.spacings(axes)
        nodes = {"srcs": eikonal.snap(srcs, axes), "recs": eikonal.snap(recs, axes)}
        dvel = torch.as_tensor(vel).cuda()
        L = pm._lib
        work = torch.empty(L.lib.b2_eikonal_work_bytes(*full, max(ns, nr)), dtype=torch.uint8, device="cuda")
        infos = {}

        def build():
            for key, tab in (("srcs", K._ts), ("recs", K._tr)):
                nd = np.ascontiguousarray(nodes[key], dtype=np.int64)
                info = (ctypes.c_longlong * 4)()
                L.check(L.lib.b2_eikonal_tables(L.ctx(), dvel.data_ptr(), *full, *h, nd.ctypes.data, len(nd), ni,
                                                tab.data_ptr(), work.data_ptr(), info, L.stream()), "eikonal")
                infos[key] = list(info)

        build_ms = time_ms(build, a.iters, a.warmup)
        step_bytes = 2 * (ns + nr) * ni * 8
        line = {"geometry": kind, "shape": list(full), "ns": ns, "nr": nr, "nt": t.size,
                "table_bytes": (ns + nr) * ni * 8, "eikonal_build_ms": round(build_ms, 3),
                "jacobi_steps": {k: v[0] for k, v in infos.items()}, "passes": {k: v[1] for k, v in infos.items()},
                "active_block_share": {k: round(v[2] / v[3], 4) for k, v in infos.items()},
                "global_step_bytes": step_bytes,
                "global_step_hbm_bound_ms": round(step_bytes / HBM_BYTES_PER_S * 1e3, 4),
                "plain_jacobi_hbm_bound_ms": round(max(infos["srcs"][0], infos["recs"][0]) * step_bytes
                                                   / HBM_BYTES_PER_S * 1e3, 2)}
        A = pm.local.Kirchhoff(z, x, t, srcs, recs, 1500.0, wav, len(wav) // 2, y=y, mode="analytic")
        line["analytic_tables_ms"] = round(time_ms(lambda: A._tables(0, ni), a.iters, a.warmup), 3)
        if kind == "2d":
            t0 = time.perf_counter()
            hs = eikonal.traveltime_table(vel, axes, srcs)
            hr = eikonal.traveltime_table(vel, axes, recs)
            line["host_numpy_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            line["bit_equal_to_numpy"] = bool(np.array_equal(K.trav_srcs.cpu().numpy(), hs)
                                              and np.array_equal(K.trav_recs.cpu().numpy(), hr))
        gen = torch.Generator(device="cuda").manual_seed(0)
        m = torch.randn(ni, device="cuda", dtype=torch.float64, generator=gen)
        d = torch.randn(ns * nr * t.size, device="cuda", dtype=torch.float64, generator=gen)
        dm, md = torch.empty_like(d), torch.empty_like(m)
        for name, op in (("eikonal", K), ("analytic", A)):
            line[f"{name}_forward_ms"] = round(time_ms(lambda o=op: o.matvec(m, out=dm), a.iters, a.warmup), 3)
            line[f"{name}_adjoint_ms"] = round(time_ms(lambda o=op: o.rmatvec(d, out=md), a.iters, a.warmup), 3)
        res["results"].append(line)
        del K, A, work, m, d, dm, md
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
