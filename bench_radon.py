"""Measure the Radon kernels (b2_radon, csrc/radon.cu) on one GPU and print JSON, one line per case.

    python bench_radon.py [--iters 10] [--warmup 2]

Cases:
  - Radon2D on one gather, nt = 1024, nh = 256, np = 256: each kind, float32 / float64, forward and adjoint;
  - 64 such gathers (linear) in MPIBlockDiag, float32 / float64, forward and adjoint;
  - Radon3D at nt = 512, nhy = nhx = npy = npx = 64: each kind in float32, linear in float64, forward and adjoint.
Per line: CUDA-event time (best of 3 alternating rounds), curve evaluations per second (one per (model sample, trace)
pair: npy npx nhy nhx nt per gather), and the ratio to a torch route for the same map with the largest difference
between the two relative to max |y|.  The torch route computes pylops' index and weight tables on the fly in float64
(a survey-size 3-D table holds 10^10 pairs and does not fit in memory), one model-y slice at a time, and applies them
with ``gather`` and ``index_add_``.  Last line: ms per fista iteration on MPIBlockDiag of the 64 gathers (linear,
float32).  The card name and power limit are read in the same run; nothing is set.
"""
import argparse
import json

import numpy as np
import torch

import pylops_mpi_b200 as pm
from bench_convolve import card, time_ms

DT, DH = 0.004, 12.5
P_RANGE = {"linear": (-1.2e-3, 1.2e-3), "parabolic": (-1e-5, 1e-5), "hyperbolic": (1500.0, 4500.0)}


def geometry(kind, nt, nh, npp):
    return np.arange(nt) * DT, np.arange(nh) * DH, np.linspace(*P_RANGE[kind], npp)


class TorchRoute:
    """the map of a Radon operator in torch, from the operator's unitless device axes"""

    def __init__(self, op):
        self.op, self.nt = op, op.dims[-1]
        ax = op._axes
        self.hy, self.hx, self.py, self.px = (None, ax[0], None, ax[1]) if len(ax) == 2 else ax
        self.nh = op.shape[0] // self.nt

    def _pairs(self, ipy):
        """(rows of the first tap, model column, d, used) for the model traces of one py, all traces"""
        nt, kind = self.nt, self.op.kind
        t0 = torch.arange(nt, device="cuda", dtype=torch.float64)
        hx, px = self.hx.view(1, 1, -1, 1), self.px.view(-1, 1, 1, 1)
        hy = None if self.hy is None else self.hy.view(1, -1, 1, 1)
        py = None if self.py is None else self.py[ipy]
        if kind == "hyperbolic":
            v = t0 * t0 + (hx / px) ** 2
            if hy is not None:
                v = v + (hy / py) ** 2
            v = torch.sqrt(v)
        else:
            v = t0 + px * (hx if kind == "linear" else hx * hx)
            if hy is not None:
                v = v + py * (hy if kind == "linear" else hy * hy)
        it = torch.nan_to_num(v, nan=-1.0, posinf=-1.0, neginf=-1.0).floor()
        ok = (v >= 0) & (v < nt - 1) if self.op.interp else (v >= 0) & (v < nt)
        npx, nhy, nhx = px.shape[0], 1 if hy is None else hy.shape[1], hx.shape[2]
        trace = torch.arange(nhy * nhx, device="cuda").view(1, nhy, nhx, 1)
        row = (trace * nt + it.long().clamp(0, nt - 1))
        col = ((ipy * npx + torch.arange(npx, device="cuda")).view(-1, 1, 1, 1) * nt
               + torch.arange(nt, device="cuda").view(1, 1, 1, -1)).expand_as(row)
        return row[ok], col[ok], (v - it)[ok]

    def forward(self, x):
        y = torch.zeros(self.nh * self.nt, dtype=x.dtype, device="cuda")
        for ipy in range(1 if self.py is None else self.py.numel()):
            row, col, d = self._pairs(ipy)
            xv = x.gather(0, col)
            if self.op.interp:
                y.index_add_(0, row, (xv * (1 - d)).to(x.dtype))
                y.index_add_(0, row + 1, (xv * d).to(x.dtype))
            else:
                y.index_add_(0, row, xv)
        return y

    def adjoint(self, x):
        y = torch.zeros(self.op.shape[1], dtype=x.dtype, device="cuda")
        for ipy in range(1 if self.py is None else self.py.numel()):
            row, col, d = self._pairs(ipy)
            v = x.gather(0, row) * (1 - d) + x.gather(0, row + 1) * d if self.op.interp else x.gather(0, row)
            y.index_add_(0, col, v.to(x.dtype))
        return y


def measure(name, op, route, ngathers, dt, adjoint, iters, warmup, gen):
    n_in = op.shape[0] if adjoint else op.shape[1]
    x = torch.randn(n_in, device="cuda", dtype=dt, generator=gen)
    out = torch.empty(op.shape[1] if adjoint else op.shape[0], device="cuda", dtype=dt)
    ours = (lambda: op.rmatvec(x, out=out)) if adjoint else (lambda: op.matvec(x, out=out))
    theirs = route.adjoint if adjoint else route.forward
    ms = {"ours": [], "torch": []}
    for _ in range(3):                                  # alternate, so that clock and neighbour noise hit both alike
        ms["ours"].append(time_ms(ours, iters, warmup))
        ms["torch"].append(time_ms(lambda: theirs(x), max(1, iters // 5), 1))
    best = {k: min(v) for k, v in ms.items()}
    ours()
    ref = theirs(x)
    nt = op.dims[-1]
    evals = (op.shape[1] // nt // ngathers) * (op.shape[0] // nt // ngathers) * nt * ngathers
    line = {"name": name, "dtype": str(dt).replace("torch.", ""), "direction": "adjoint" if adjoint else "forward",
            "gathers": ngathers, "ms": round(best["ours"], 3),
            "curve_evals_per_s": float(f"{evals / (best['ours'] * 1e-3):.4g}"),
            "torch_route_ms": round(best["torch"], 3), "x_torch_route": round(best["ours"] / best["torch"], 4),
            "torch_route_max_rel_diff": float((out.double() - ref.double()).abs().max() / ref.double().abs().max())}
    print(json.dumps(line), flush=True)


class Gathers:
    """``n`` copies of one gather operator applied as MPIBlockDiag, and the torch route gather by gather"""

    def __init__(self, op, n):
        self.B = pm.MPIBlockDiag([op] * n)
        self.op, self.n = op, n
        self.shape, self.dims = self.B.shape, op.dims
        self.route = TorchRoute(op)

    def matvec(self, x, out=None):
        out.copy_((self.B @ pm.DistributedArray.to_dist(x)).local_array)

    def rmatvec(self, x, out=None):
        out.copy_((self.B.H @ pm.DistributedArray.to_dist(x)).local_array)

    def forward(self, x):
        m = self.op.shape[1]
        return torch.cat([self.route.forward(x[g * m:(g + 1) * m]) for g in range(self.n)])

    def adjoint(self, x):
        m = self.op.shape[0]
        return torch.cat([self.route.adjoint(x[g * m:(g + 1) * m]) for g in range(self.n)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    print(json.dumps({"device": card()}), flush=True)
    gen = torch.Generator(device="cuda").manual_seed(0)
    f32, f64 = torch.float32, torch.float64
    for kind in ("linear", "parabolic", "hyperbolic"):
        for dt in (f32, f64):
            op = pm.local.Radon2D(*geometry(kind, 1024, 256, 256), kind=kind, dtype=str(dt).replace("torch.", ""))
            for adjoint in (False, True):
                measure(f"Radon2D {kind} nt1024 nh256 np256", op, TorchRoute(op), 1, dt, adjoint, a.iters, a.warmup,
                        gen)
    for dt in (f32, f64):
        op = pm.local.Radon2D(*geometry("linear", 1024, 256, 256), dtype=str(dt).replace("torch.", ""))
        G = Gathers(op, 64)
        for adjoint in (False, True):
            measure("MPIBlockDiag 64 x Radon2D linear nt1024 nh256 np256", G, G, 64, dt, adjoint, max(2, a.iters // 5),
                    1, gen)
    for kind, dt in (("linear", f32), ("parabolic", f32), ("hyperbolic", f32), ("linear", f64)):
        t, h, p = geometry(kind, 512, 64, 64)
        op = pm.local.Radon3D(t, h, h, p, p, kind=kind, dtype=str(dt).replace("torch.", ""))
        for adjoint in (False, True):
            measure(f"Radon3D {kind} nt512 nh64x64 np64x64", op, TorchRoute(op), 1, dt, adjoint, max(2, a.iters // 3),
                    1, gen)

    # fista on the 64 gathers (linear, float32): ms per iteration, end to end
    op = pm.local.Radon2D(*geometry("linear", 1024, 256, 256), dtype="float32")
    B = pm.MPIBlockDiag([op] * 64)
    m = torch.zeros(B.shape[1], device="cuda")
    m[torch.randint(0, B.shape[1], (64 * 40,), device="cuda", generator=gen)] = 1.0
    d = B @ pm.DistributedArray.to_dist(m)
    x0 = pm.DistributedArray.to_dist(torch.zeros(B.shape[1], device="cuda"))
    alpha = 1.0 / (256 * 512)               # 1 / (||R||_1 ||R||_inf): columns sum to <= nh, rows to <= 2 np
    pm.fista(B, d, x0, niter=2, eps=0.1, alpha=alpha, tol=0.0)
    niter = max(a.iters, 5)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _, iiter, _ = pm.fista(B, d, x0, niter=niter, eps=0.1, alpha=alpha, tol=0.0)
    e1.record()
    torch.cuda.synchronize()
    print(json.dumps({"name": "fista MPIBlockDiag 64 x Radon2D linear nt1024 nh256 np256", "dtype": "float32",
                      "iterations": int(iiter), "ms_per_iteration": round(e0.elapsed_time(e1) / max(int(iiter), 1),
                                                                          3)}), flush=True)


if __name__ == "__main__":
    main()
