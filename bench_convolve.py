"""Measure the rank-local Convolve1D kernel (csrc/convolve.cu) on one GPU and print the results as JSON.

    python bench_convolve.py [--iters 20] [--warmup 3]

Workloads, on the per-GPU block (128, 1024, 1024) with nh = 41, offset = 20 unless stated:
  - axis -1 (innermost, n_inner == 1 path), forward and adjoint, float32 and float64;
  - axis 0 of the (1024, 131072) view (middle-axis path), forward, float32 and float64;
  - an nh sweep over {5, 41, 127, 301} on axis -1;
  - torch.nn.functional.conv1d (cuDNN) on the same axis -1 map, the baseline a user would otherwise reach for;
  - the reflectivity ISTA iteration (MPIBlockDiag([Convolve1D]) forward + adjoint + thresholded update), float32.
Per line: CUDA-event kernel time, algorithmic bytes 2 N sizeof(T) and 2 nh N flop over that time, and the fraction
of the larger of the two bounds (bytes / 3.35 TB/s, or flop / 67 TF/s in float32, 34 TF/s in float64), naming it.
Data-sheet peaks are for an H100 SXM at 700 W; the card name and power limit are read in the same run.
"""
import argparse
import json
import subprocess

import numpy as np
import torch

import pylops_mpi_b200 as pm

HBM = 3.35e12
FLOPS = {torch.float32: 67e12, torch.float64: 34e12}
SHAPE = (128, 1024, 1024)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:                       # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unknown ({exc})"}


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def line(name, ms, n, nh, dt):
    t = ms * 1e-3
    size = torch.tensor([], dtype=dt).element_size()
    nbytes, flop = 2 * n * size, 2 * nh * n
    tb, tf = nbytes / HBM, flop / FLOPS[dt]
    return {"name": name, "dtype": str(dt).replace("torch.", ""), "nh": nh, "ms": round(ms, 4),
            "GB_per_s": round(nbytes / t / 1e9, 1), "TFLOP_per_s": round(flop / t / 1e12, 2),
            "bound": "hbm" if tb >= tf else "fp", "fraction_of_bound": round(max(tb, tf) / t, 3)}


def conv_launch(x, y, h, shape, off, adjoint):
    L = pm._lib
    code = L.code(x.dtype)
    ctx, st = L.ctx(), L.stream()

    def run():
        L.check(L.lib.b2_convolve_axis(ctx, x.data_ptr(), y.data_ptr(), shape[0], shape[1], shape[2], h.data_ptr(),
                                       h.numel(), off, adjoint, code, st), "b2_convolve_axis")
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    res = {"device": card(), "shape": SHAPE, "results": []}
    out = res["results"]
    n = int(np.prod(SHAPE))
    gen = torch.Generator(device="cuda").manual_seed(0)
    for dt in (torch.float32, torch.float64):
        x = torch.randn(n, device="cuda", dtype=dt, generator=gen)
        y = torch.empty_like(x)
        for nh in (5, 41, 127, 301):
            off = nh // 2
            h = torch.randn(nh, device="cuda", dtype=dt, generator=gen)
            lines = (("axis-1 fwd", (SHAPE[0] * SHAPE[1], SHAPE[2], 1), 0),)
            if nh == 41:
                lines += (("axis-1 adj", (SHAPE[0] * SHAPE[1], SHAPE[2], 1), 1),
                          ("axis0 of (1024,131072) fwd", (1, 1024, n // 1024), 0))
            for name, shp, adj in lines:
                out.append(line(name, time_ms(conv_launch(x, y, h, shp, off, adj), a.iters, a.warmup), n, nh, dt))
            # cuDNN: y[i] = sum_k h[k] x[i + off - k] is conv1d (cross-correlation) with flipped taps, padding nh // 2
            w = h.flip(0).reshape(1, 1, nh)
            xin = x.reshape(-1, 1, SHAPE[2])
            ms = time_ms(lambda: torch.nn.functional.conv1d(xin, w, padding=off), a.iters, a.warmup)
            out.append(line("axis-1 fwd torch conv1d (cuDNN)", ms, n, nh, dt))
        del x, y
        torch.cuda.empty_cache()

    # reflectivity ISTA iteration on the same block (float32): ms per iteration, end to end
    t = (np.arange(41) - 20) * 0.004
    wav = (1 - 2 * (np.pi * 20 * t) ** 2) * np.exp(-(np.pi * 20 * t) ** 2)
    Cop = pm.MPIBlockDiag([pm.local.Convolve1D(SHAPE, wav, offset=20, axis=-1, dtype="float32")])
    d = Cop @ pm.DistributedArray.to_dist(torch.randn(n, device="cuda", dtype=torch.float32, generator=gen))
    x0 = pm.DistributedArray.to_dist(torch.zeros(n, device="cuda", dtype=torch.float32))
    alpha = 1.0 / float(np.abs(wav).sum() ** 2)
    pm.ista(Cop, d, x0, niter=2, eps=0.1, alpha=alpha, tol=0.0)
    niter = max(a.iters, 5)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _, iiter, _ = pm.ista(Cop, d, x0, niter=niter, eps=0.1, alpha=alpha, tol=0.0)
    e1.record()
    torch.cuda.synchronize()
    res["reflectivity_ista"] = {"dtype": "float32", "nh": 41, "iterations": int(iiter),
                                "ms_per_iteration": round(e0.elapsed_time(e1) / max(int(iiter), 1), 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
