"""Generate the non-stationary filter-estimation fixtures by running the REAL reference's MPIVStack (a pylops-mpi
checkout named by PYLOPS_MPI_REFERENCE, imported unmodified through make_golden.load_reference) over refshim's
restated ``pylops.signalprocessing.NonStationaryFilters1D`` / ``NonStationaryFilters2D``
(refshim/pylops/signalprocessing/nonstatfilters.py).

    PYLOPS_MPI_REFERENCE=<checkout> python tests/golden/make_golden_nsfilters.py   # writes nsfilters_golden.npz

A stack of NI fixed inputs (1-D traces of N1 samples, or NX x NZ images) split over P in {1, 2, 3} ranks: rank r
holds MPIVStack([NonStationaryFilters(inp_k, ...) for its inputs k]), several operators per rank.  The model, one
filter bank, is broadcast; the forward of x gives the stacked data and the adjoint of v (stacked data) the bank, which
the reference all-reduces over the ranks.  1-D filter sizes ``HSIZES`` with banks ``BANKS1``; 2-D filter sizes
``NHS2`` (41 x 41 is larger than the image) with the banks of make_golden_nsconvolve2d.py; ih = 1 + dh * arange(nf)
per axis, so both ends of both axes are extrapolated.  Inputs are exactly representable: inp and v have entries in
{-1, 0, 1}, the taps of x are drawn from {-1, -1/2, 1/2, 1} and the steps are 1 or 4, so every weight is a multiple
of 1/16 and every output a multiple of 1/32, the SAME in float64, float32 and complex128 and at every P (all checked
here).  Each output is stored once, losslessly, as int32 of ENC * y.

  f1/h{hsize}/nf{nf}/dh{dh}/{y,ya}            gathered forward of x / adjoint of v
  f2/nh{nhx}x{nhz}/nf{nfx}x{nfz}/dh{dhx}x{dhz}/{y,ya}
  .../{yi,yai}   imaginary parts of the complex128 runs, for the cases of ``complex_case``

Flow 1, time-varying wavelet estimation.  FLOW1_NTR seeded sparse reflectivity traces of FLOW1_N samples, split over
the ranks; data from the restated NonStationaryConvolve1D with a bank of Ricker wavelets (make_golden_nsconvolve.py's
``ricker``, FLOW_NWAV taps, FLOW_DT) at the samples FLOW1_IH, whose peak frequency falls from 25 to 10 Hz.  Then
cgls(MPIVStack([NonStationaryFilters1D(r_k, FLOW_NWAV, FLOW1_IH) ...]), d, x0 = 0) for FLOW1_NITER iterations.

Flow 2, a deblurring filter for image-domain least-squares migration.  The layered reflectivities m_k and their
migrations K^H K m_k of make_golden_nsconvolve2d.py's flow (refshim's analytic Kirchhoff); the first FLOW2_NTRAIN
pairs, split over the ranks, train a FLOW2_NH bank at the nodes (FLOW_IHX, FLOW_IHZ) of that flow:
cgls(MPIVStack([NonStationaryFilters2D(K^H K m_k, FLOW2_NH, FLOW_IHX, FLOW_IHZ) ...]), m, x0 = 0) for FLOW2_NITER
iterations, and the estimated filter F is applied to the held-out migration: NonStationaryConvolve2D(F) K^H K m_last.

For each flow, ``cond`` is the 2-norm condition number of the stacked operator (its dense float64 matrix) and
``spread`` how far rounding alone moves the reference's own run: the largest change of x (relative to max |x|) and
of the cost history (relative) when every apply of the restated operators is jittered by 4 ulps, over the seeds
FLOW_JITTER_SEEDS at P = 1.  The tests take their tolerance from both.  The wavelet problem is well conditioned
(cond 3.8): 12 iterations cut the cost 3000-fold with a spread of 4e-15.  The deblurring problem is not (cond 2.2e4:
neighbouring filters of a smooth migrated image are nearly collinear): at 8 iterations the spread is 4e-14, at 20 it
is 6 % of max |x| while the cost falls only from 10.3 to 9.8, because cgls then fits directions whose components
rounding alone decides, which no other summation order would reproduce.  So the 2-D flow stops at 8.

  flow1/refl, flow1/d, flow1/cond, flow1/spread, flow1/P{P}/{x,iiter,cost}
  flow2/mmig, flow2/m, flow2/cond, flow2/spread, flow2/P{P}/{x,iiter,cost,heldout}
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from fixture_codec import encode, rows_of  # noqa: E402
import make_golden_nsconvolve as mgn  # noqa: E402
import make_golden_nsconvolve2d as mg2  # noqa: E402
from make_golden_nsconvolve2d import BANKS as BANKS2, NX, NZ, nodes  # noqa: E402

NI = 4
N1 = 30
HSIZES = (1, 5, 41)
BANKS1 = ((1, 1), (2, 1), (2, 4), (5, 1), (5, 4))
NHS2 = ((1, 1), (3, 5), (7, 3), (41, 41))
DTYPES = ("float64", "float32", "complex128")
ENC = 32         # stored value = ENC * y, exact in int32

FLOW1_NTR, FLOW1_N, FLOW1_IH, FLOW1_NITER = 6, 160, (10, 45, 80, 115, 150), 12
FLOW2_NTRAIN, FLOW2_NH, FLOW2_NITER = 3, (9, 9), 8
FLOW_JITTER_SEEDS = (1, 2, 3)


def complex_case(kind, nh, bank):
    return (kind == 1 and nh == 5 and bank == (5, 4)) or (kind == 2 and nh == (3, 5) and bank[0] == (2, 3))


def cases():
    """(kind, nh, bank, dtype): kind 1 with (hsize, (nf, dh)), kind 2 with ((nhx, nhz), ((nfx, nfz), (dhx, dhz)))"""
    out = [(1, h, b) for h in HSIZES for b in BANKS1] + [(2, nh, b) for nh in NHS2 for b in BANKS2]
    return [(k, nh, b, dt) for k, nh, b in out for dt in DTYPES if dt != "complex128" or complex_case(k, nh, b)]


def key(kind, nh, bank):
    if kind == 1:
        return f"f1/h{nh}/nf{bank[0]}/dh{bank[1]}"
    (nfx, nfz), (dhx, dhz) = bank
    return f"f2/nh{nh[0]}x{nh[1]}/nf{nfx}x{nfz}/dh{dhx}x{dhz}"


def case_inputs(kind, nh, bank, dt):
    """NI inputs (the real dtype of dt, shape (NI, N1) or (NI, NX, NZ)), the node indices (a tuple of arrays), the
    bank shape, the model x (dtype dt) and the global data v (dtype dt)"""
    if kind == 1:
        ih = (1 + bank[1] * np.arange(bank[0]),)
        dims, bshape = (N1,), (bank[0], nh)
    else:
        ih = nodes(bank)
        dims, bshape = (NX, NZ), bank[0] + nh
    rdt = np.real(np.ones(1, dt)).dtype
    rng = np.random.default_rng(700 + 31 * kind + 97 * int(np.sum(nh)) + 7 * int(np.sum(bank)))
    inp = rng.integers(-1, 2, (NI,) + dims).astype(rdt)
    x, xi = (rng.choice([-1.0, -0.5, 0.5, 1.0], bshape).ravel() for _ in range(2))
    v, vi = (rng.integers(-1, 2, NI * int(np.prod(dims))).astype(np.float64) for _ in range(2))
    if dt == "complex128":
        x, v = x + 1j * xi, v + 1j * vi
    return inp, ih, bshape, x.astype(dt), v.astype(dt)


def restated(name):
    """refshim's pylops.signalprocessing.<name>"""
    import importlib
    added = mg2.REFSHIM not in sys.path
    if added:
        sys.path.insert(0, mg2.REFSHIM)
    try:
        return importlib.import_module(f"pylops.signalprocessing.{name}")
    finally:
        if added:
            sys.path.remove(mg2.REFSHIM)


def flow1_inputs():
    """(Ricker bank (len(FLOW1_IH), FLOW_NWAV), reflectivities (FLOW1_NTR, FLOW1_N), data (FLOW1_NTR * FLOW1_N,))"""
    t = np.arange(mgn.FLOW_NWAV // 2 + 1) * mgn.FLOW_DT
    wav = np.stack([mgn.ricker(t, f) for f in np.linspace(mgn.FLOW_F0[0], mgn.FLOW_F0[1], len(FLOW1_IH))])
    rng = np.random.default_rng(41)
    refl = np.where(rng.random((FLOW1_NTR, FLOW1_N)) < 0.1, rng.standard_normal((FLOW1_NTR, FLOW1_N)), 0.0)
    C = restated("nonstatconvolve1d").NonStationaryConvolve1D(FLOW1_N, wav, FLOW1_IH)
    return wav, refl, np.concatenate([C.matvec(r) for r in refl])


def flow2_inputs():
    """(migrated images K^H K m (FLOW_NY, FLOW_NX, FLOW_NZ), reflectivities m (the same shape))"""
    kirchhoff, _ = mg2.refshim_kirchhoff()
    z, x, t, srcs, recs, vel, wav, wavc = mg2.flow_geometry()
    K = kirchhoff.Kirchhoff(z, x, t, srcs, recs, vel, wav, wavc, mode="analytic")
    _, m_true = mg2.flow_models()
    mmig = np.stack([K.rmatvec(K.matvec(m.ravel())).reshape(mg2.FLOW_NX, mg2.FLOW_NZ) for m in m_true])
    return mmig, m_true


def main():
    from make_golden import load_reference          # puts refshim/ (mpi4py, pylops) on the path
    from mpi4py import MPI
    from pylops.signalprocessing.nonstatfilters import NonStationaryFilters1D, NonStationaryFilters2D
    pkg, mods = load_reference()
    DA, Partition = pkg.DistributedArray, pkg.Partition
    VS = mods["VStack"].MPIVStack
    out = {}

    def t_op(rank, P, kind, nh, bank, dt):
        inp, ih, bshape, x, v = case_inputs(kind, nh, bank, dt)
        ny = rows_of(P, NI)
        k0 = sum(ny[:rank])
        plane = int(np.prod(inp.shape[1:]))
        if kind == 1:
            ops = [NonStationaryFilters1D(inp[k], nh, ih[0], dtype=dt) for k in range(k0, k0 + ny[rank])]
        else:
            ops = [NonStationaryFilters2D(inp[k], nh, ih[0], ih[1], dtype=dt) for k in range(k0, k0 + ny[rank])]
        Op = VS(ops, dtype=dt)
        xd = DA(global_shape=x.size, partition=Partition.BROADCAST, dtype=dt)
        xd[:] = x
        return {"y": (Op @ xd).asarray(),
                "ya": (Op.H @ DA.to_dist(v, local_shapes=[(r * plane,) for r in ny])).asarray()}

    for kind, nh, bank, _ in cases():
        k = key(kind, nh, bank)
        if f"{k}/y" in out:
            continue
        runs = {}
        for dt in DTYPES:
            if dt == "complex128" and not complex_case(kind, nh, bank):
                continue
            for P in (1, 2, 3):
                res = MPI.run_world(P, t_op, P, kind, nh, bank, dt)[0]
                if P == 1:
                    runs[dt] = res
                for n in ("y", "ya"):                      # exact values: the result does not depend on P
                    assert np.array_equal(res[n], runs[dt][n])
        for n in ("y", "ya"):
            assert np.array_equal(runs["float32"][n], runs["float64"][n])
            out[f"{k}/{n}"] = encode(runs["float64"][n], ENC, np.int32)
            if "complex128" in runs:
                assert np.array_equal(runs["complex128"][n].real, runs["float64"][n])
                out[f"{k}/{n}i"] = encode(runs["complex128"][n].imag, ENC, np.int32)

    # flows, in float64
    import importlib
    basic = importlib.import_module("pylops_mpi.optimization.basic")
    NSC2D = restated("nonstatconvolve2d").NonStationaryConvolve2D
    wav, refl, d1 = flow1_inputs()
    mmig, m_true = flow2_inputs()
    out["flow1/refl"], out["flow1/d"] = refl, d1
    out["flow2/mmig"], out["flow2/m"] = mmig, m_true
    flows = {1: (FLOW1_NITER, refl, d1, (len(FLOW1_IH), mgn.FLOW_NWAV)),
             2: (FLOW2_NITER, mmig[:FLOW2_NTRAIN], m_true[:FLOW2_NTRAIN].ravel(),
                 (len(mg2.FLOW_IHX), len(mg2.FLOW_IHZ)) + FLOW2_NH)}

    def make_op(kind, inp, seed=None):
        cls = NonStationaryFilters1D if kind == 1 else NonStationaryFilters2D
        args = (inp, mgn.FLOW_NWAV, FLOW1_IH) if kind == 1 else (inp, FLOW2_NH, mg2.FLOW_IHX, mg2.FLOW_IHZ)
        if seed is None:
            return cls(*args)

        class Jittered(cls):
            """the restated operator with every output scaled by 1 + 4 u g, g standard normal, seeded"""
            rng = np.random.default_rng(seed)

            def _matvec(self, x):
                y = super()._matvec(x)
                return y * (1 + 4 * 2.0 ** -53 * self.rng.standard_normal(y.shape))

            def _rmatvec(self, x):
                y = super()._rmatvec(x)
                return y * (1 + 4 * 2.0 ** -53 * self.rng.standard_normal(y.shape))
        return Jittered(*args)

    def t_flow(rank, P, kind, seed=None):
        niter, inps, d, bshape = flows[kind]
        ny = rows_of(P, len(inps))
        k0 = sum(ny[:rank])
        plane = int(np.prod(inps.shape[1:]))
        Op = VS([make_op(kind, inps[k], seed) for k in range(k0, k0 + ny[rank])])
        dd = DA.to_dist(d, local_shapes=[(r * plane,) for r in ny])
        x0 = DA(global_shape=int(np.prod(bshape)), partition=Partition.BROADCAST)
        x0[:] = 0
        xinv, istop, iiter, r1, r2, cost = basic.cgls(Op, dd, x0=x0, niter=niter, tol=0.0)
        return {"x": xinv.asarray(), "iiter": iiter, "cost": np.asarray(cost)}

    for kind, (niter, inps, d, bshape) in flows.items():
        f = f"flow{kind}"
        nb = int(np.prod(bshape))
        ops = [make_op(kind, i) for i in inps]
        A = np.concatenate([np.stack([op.matvec(e) for e in np.eye(nb)], 1) for op in ops])
        out[f"{f}/cond"] = np.asarray(np.linalg.cond(A))
        for P in (1, 2, 3):
            res = MPI.run_world(P, t_flow, P, kind)[0]
            for k in ("x", "iiter", "cost"):
                out[f"{f}/P{P}/{k}"] = np.asarray(res[k])
            if kind == 2:
                out[f"{f}/P{P}/heldout"] = NSC2D((mg2.FLOW_NX, mg2.FLOW_NZ), res["x"].reshape(bshape), mg2.FLOW_IHX,
                                                 mg2.FLOW_IHZ).matvec(mmig[-1].ravel())
        spread = np.zeros(2)
        x1, c1 = out[f"{f}/P1/x"], out[f"{f}/P1/cost"]
        for seed in FLOW_JITTER_SEEDS:
            res = MPI.run_world(1, t_flow, 1, kind, seed)[0]
            spread = np.maximum(spread, [np.abs(res["x"] - x1).max() / np.abs(x1).max(),
                                         (np.abs(res["cost"] - c1) / c1).max()])
        out[f"{f}/spread"] = spread
        print(f"{f}: cond {float(out[f + '/cond']):.3e}, spread {spread}, cost {c1[0]:.3e} -> {c1[-1]:.3e}")

    path = os.path.join(HERE, os.environ.get("GOLDEN_OUT", "nsfilters_golden.npz"))
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays, {os.path.getsize(path) / 1e3:.0f} KB")


if __name__ == "__main__":
    main()
