"""Measure 3-D Kirchhoff demigration (local.Kirchhoff with a y axis) on one GPU and print JSON.

    python bench_kirchhoff3d.py [--iters 5] [--warmup 1] [--chunks 8] [--cgls 20]

Per-GPU shape: a 96 x 96 x 64 image (ni = 589,824), 8 sources, a 16 x 16 receiver grid (2,048 traces), nt = 1024
(1.21e9 point-trace pairs per apply), a 41-tap Ricker wavelet, constant velocity.  Lines:
  - traveltime tables, (ns + nr) * ni float64 (1.25 GB): pylops' NumPy expressions on the host (one run) against
    b2_kirchhoff_tables on the device;
  - the operator's forward and adjoint, float32 and float64, with resident tables and with the table budget lowered
    to give ``--chunks`` chunks (the tables are rebuilt on every apply), runs alternated; and whether the two give the
    same bits;
  - cgls on MPIVStack([Kirchhoff]) in ms per iteration, float64, resident and chunked.
Expected extra cost of chunking, an estimate to check: rebuilding (ns + nr) table entries per image point against
ns * nr pairs per image point, i.e. about (ns + nr) / (ns * nr) = 13 % more work per pair if a table entry costs what
a pair does.  The card name and power limit are read in the same run.
"""
import argparse
import json
import time

import numpy as np
import torch

import pylops_mpi_b200 as pm
from bench_convolve import card, time_ms

NY, NX, NZ, NS, NRY, NRX, NT, DT, VEL, DX = 96, 96, 64, 8, 16, 16, 1024, 0.002, 2000.0, 5.0


def ricker(t, f0):
    w = (1 - 2 * (np.pi * f0 * t) ** 2) * np.exp(-(np.pi * f0 * t) ** 2)
    return np.concatenate((np.flipud(w[1:]), w), axis=0)


def geometry():
    y, x, z = np.arange(NY) * DX, np.arange(NX) * DX, np.arange(NZ) * DX
    SY, SX = np.meshgrid(np.linspace(0, y[-1], 2), np.linspace(0, x[-1], NS // 2), indexing="ij")
    srcs = np.vstack((SY.ravel(), SX.ravel(), np.zeros(NS)))
    RY, RX = np.meshgrid(np.linspace(0, y[-1], NRY), np.linspace(0, x[-1], NRX), indexing="ij")
    recs = np.vstack((RY.ravel(), RX.ravel(), np.zeros(NRY * NRX)))
    return z, x, np.arange(NT) * DT, srcs, recs, y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--chunks", type=int, default=8)
    ap.add_argument("--cgls", type=int, default=20)
    a = ap.parse_args()
    z, x, t, srcs, recs, y = geometry()
    ni, nr = NY * NX * NZ, NRY * NRX
    pairs = ni * NS * nr
    wav = ricker(np.arange(21) * DT, 20.0)
    budget = pm.local.KIRCHHOFF_TABLE_BYTES
    chunk_budget = (NS + nr) * 8 * (-(-ni // a.chunks))
    res = {"device": card(), "shape": {"ny": NY, "nx": NX, "nz": NZ, "ns": NS, "nr": nr, "nt": NT, "nh": wav.size},
           "pairs": pairs, "table_bytes": (NS + nr) * ni * 8, "results": []}
    out = res["results"]

    # tables: host NumPy (one run) against the device builder
    from pylops_mpi_b200.local import _traveltime_tables
    t0 = time.perf_counter()
    hts, htr = _traveltime_tables(z, x, srcs, recs, VEL, y=y)
    host_ms = (time.perf_counter() - t0) * 1e3
    K = pm.local.Kirchhoff(z, x, t, srcs, recs, VEL, wav, len(wav) // 2, y=y, mode="analytic")
    dev_ms = time_ms(lambda: K._tables(0, ni), a.iters, a.warmup)
    same = bool(np.array_equal(K._ts.cpu().numpy(), hts.T) and np.array_equal(K._tr.cpu().numpy(), htr.T))
    res["tables"] = {"host_numpy_ms": round(host_ms, 1), "device_ms": round(dev_ms, 3),
                     "device_GB_per_s": round((NS + nr) * ni * 8 / (dev_ms * 1e-3) / 1e9, 1), "bit_equal": same}
    del hts, htr, K
    torch.cuda.empty_cache()

    gen = torch.Generator(device="cuda").manual_seed(0)
    for dt, name in ((torch.float32, "float32"), (torch.float64, "float64")):
        pm.local.KIRCHHOFF_TABLE_BYTES = budget
        R = pm.local.Kirchhoff(z, x, t, srcs, recs, VEL, wav, len(wav) // 2, y=y, mode="analytic", dtype=name)
        pm.local.KIRCHHOFF_TABLE_BYTES = chunk_budget
        C = pm.local.Kirchhoff(z, x, t, srcs, recs, VEL, wav, len(wav) // 2, y=y, mode="analytic", dtype=name)
        pm.local.KIRCHHOFF_TABLE_BYTES = budget
        assert not R.chunked and C.chunked
        m = torch.randn(ni, device="cuda", dtype=dt, generator=gen)
        d = torch.randn(NS * nr * NT, device="cuda", dtype=dt, generator=gen)
        dm, md = torch.empty_like(d), torch.empty_like(m)
        for adj, which in ((0, "forward"), (1, "adjoint")):
            runs = {"resident": (lambda o=R: o.rmatvec(d, out=md)) if adj else (lambda o=R: o.matvec(m, out=dm)),
                    "chunked": (lambda o=C: o.rmatvec(d, out=md)) if adj else (lambda o=C: o.matvec(m, out=dm))}
            ms = {k: [] for k in runs}
            for _ in range(2):                   # alternate, so that clock and neighbour noise hit each alike
                for k, fn in runs.items():
                    ms[k].append(time_ms(fn, a.iters, a.warmup))
            eq = bool(torch.equal(R.rmatvec(d), C.rmatvec(d)) if adj else torch.equal(R.matvec(m), C.matvec(m)))
            for k in runs:
                t_ms = min(ms[k])
                out.append({"name": f"{which} {k}", "dtype": name, "ms": round(t_ms, 3), "runs_ms": [round(v, 3) for v
                            in ms[k]], "Gpairs_per_s": round(pairs / (t_ms * 1e-3) / 1e9, 2),
                            **({"chunks": -(-ni // C._nc), "bit_equal_to_resident": eq} if k == "chunked" else {})})
        del R, C, m, d, dm, md
        torch.cuda.empty_cache()

    # cgls, float64, ms per iteration
    refl = np.zeros((NY, NX, NZ))
    refl[:, :, NZ // 3], refl[:, :, 2 * NZ // 3] = -1.0, 0.5
    res["cgls"] = {"dtype": "float64", "iterations": a.cgls}
    for k, b in (("resident", budget), ("chunked", chunk_budget)):
        pm.local.KIRCHHOFF_TABLE_BYTES = b
        V = pm.MPIVStack([pm.local.LSM(z, x, t, srcs, recs, VEL, wav, len(wav) // 2, y=y, mode="analytic").Demop])
        pm.local.KIRCHHOFF_TABLE_BYTES = budget
        dd = V @ pm.DistributedArray.to_dist(refl.ravel(), partition=pm.Partition.BROADCAST)
        x0 = pm.DistributedArray.to_dist(np.zeros(ni), partition=pm.Partition.BROADCAST)
        pm.cgls(V, dd, x0=x0, niter=2, tol=0.0)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _, _, iiter, _, _, _ = pm.cgls(V, dd, x0=x0, niter=a.cgls, tol=0.0)
        e1.record()
        torch.cuda.synchronize()
        res["cgls"][f"{k}_ms_per_iteration"] = round(e0.elapsed_time(e1) / max(int(iiter), 1), 3)
        del V, dd, x0
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
