"""LSQR against CGLS on one GPU, ms per iteration, and print JSON.

    python bench_lsqr.py [--rounds 5] [--short 10] [--long 30]

Two workloads, each solved by lsqr and cgls alternately in the same process (``--rounds`` rounds; medians and ranges):
  - blockdiag: bench.py's block, MPIBlockDiag of one 4096 x 4096 float32 MatrixMult (randn / 128 + 2 I), from
    x0 = 0 with the user stopping tests off (lsqr atol = btol = 0, conlim = 0; cgls tol = 0).  LSQR keeps its
    machine-precision tests (istop 4-6), which this block meets at iteration 33, so both iteration counts stay below;
  - lsm: tutorials/lsm.py's flow (81 x 60 image, 10 sources, 11 receivers, nt = 651, analytic Kirchhoff in
    MPIVStack), float64, the same settings.
Both solvers do one matvec and one rmatvec per iteration.  Time is host clock around a whole solve (setup, eager
first iteration and graph capture included) that ends in a device synchronise.  The steady-state cost of one
replayed iteration is the slope between a --short and a --long solve, which removes the fixed costs; the whole-solve
time per iteration of the long solve is reported too.  The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

import pylops_mpi_b200 as pm
from bench_convolve import card

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests", "golden"))


def blockdiag():
    nb = 4096
    A = torch.randn(nb, nb, device="cuda", generator=torch.Generator(device="cuda").manual_seed(100)) / 128
    A += 2 * torch.eye(nb, device="cuda")
    Op = pm.MPIBlockDiag([pm.MatrixMult(A)])
    xt = pm.DistributedArray(global_shape=nb, dtype=np.float32)
    xt.local_array.normal_()
    return Op, Op.matvec(xt), xt.zeros_like()


def lsm():
    import make_golden_kirchhoff as mgk
    z, x, t, srcs, recs, v0, wav, wavc, refl = mgk.flow_setup(1)
    Op = pm.MPIVStack([pm.local.LSM(z, x, t, srcs, recs, v0, wav, wavc, mode="analytic").Demop])
    m = pm.DistributedArray.to_dist(refl.ravel(), partition=pm.Partition.BROADCAST)
    x0 = pm.DistributedArray.to_dist(np.zeros(Op.shape[1]), partition=pm.Partition.BROADCAST)
    return Op, Op.matvec(m), x0


def solve(name, Op, y, x0, niter):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if name == "lsqr":
        out = pm.lsqr(Op, y, x0=x0, niter=niter, atol=0.0, btol=0.0, conlim=0.0)
        it = out[2]
    else:
        out = pm.cgls(Op, y, x0=x0, niter=niter, tol=0.0)
        it = out[2]
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / it, it


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--short", type=int, default=10)
    ap.add_argument("--long", type=int, default=30)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    res = {"card": card(), "niter": [args.short, args.long]}
    for wname, make in (("blockdiag_4096_f32", blockdiag), ("lsm_tutorial_f64", lsm)):
        Op, y, x0 = make()
        for name in ("lsqr", "cgls"):                      # warm-up: modules, workspaces, graph pool
            solve(name, Op, y, x0, 5)
        slope, whole = {"lsqr": [], "cgls": []}, {"lsqr": [], "cgls": []}
        for _ in range(args.rounds):
            for name in ("lsqr", "cgls"):
                ms_s, it_s = solve(name, Op, y, x0, args.short)
                ms_l, it_l = solve(name, Op, y, x0, args.long)
                assert (it_s, it_l) == (args.short, args.long), (name, it_s, it_l)
                slope[name].append((ms_l * it_l - ms_s * it_s) / (it_l - it_s))
                whole[name].append(ms_l)
        res[wname] = {k: {"steady_ms_per_iter_median": float(np.median(slope[k])), "steady_min": min(slope[k]),
                          "steady_max": max(slope[k]), f"whole_solve_ms_per_iter_{args.long}": float(np.median(whole[k]))}
                      for k in slope}
        res[wname]["lsqr_over_cgls_steady"] = res[wname]["lsqr"]["steady_ms_per_iter_median"] / \
            res[wname]["cgls"]["steady_ms_per_iter_median"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
