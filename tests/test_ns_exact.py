"""Exact checks of the non-stationary convolution kernels at production geometry: b2_nsconvolve2d, b2_nsconvolve3d
and b2_nsfilters2d_adjoint (which also serves as the adjoint of NonStationaryFilters1D), all built on the correlation
core of csrc/ns_core.cuh.

The references evaluate the definition (ns_reference.py) directly at chosen outputs, so they need no dense matrix:
``point_ref`` sums one output's footprint, ``spike_ref`` builds the whole output of an input that is zero except on
a lattice of spikes, and ``nsfilters_ref`` takes one tap of the filter-estimation adjoint as a dot product over its
filter's support.  ``seam_outputs`` picks the outputs where tiling goes wrong: both sides of every tile seam, the
nodes and support edges, the first and last samples.

Exact inputs.  With node spacings dh = 2^p every weight (j - oh) / dh is a multiple of 2^-p, and a product of d
weights is a multiple of the quantum q = 2^-(p_1 + .. + p_d).  With taps and data small integers, |v| <= 4, every
term W h x is a multiple of q, and so is every partial sum.  A sum is exact in a dtype of m significand bits while
(sum of |terms|) / q < 2^m, whatever the order of its fma.  Then the kernel must equal the float64 reference bit
for bit.  In 2-D at dh = 64 (q = 2^-12) with 61 x 61 taps, one output has at most 4 * 61^2 terms of at most 16, so
it stays below 4 * 61^2 * 16 < 2^18: 30 bits for dense float64 inputs.  Spikes placed so that no two share a
footprint put one spike in each: at most 4 terms below 2^6, 18 bits, which float32 holds too.  ``exact_bits`` computes
these counts for each case and the tests assert them; a tap of the filter-estimation adjoint sums its filter's whole
support, and ``nsf_exact_bits`` counts that.  The spike runs of a case (``spike_rounds``) together put spikes on
every residue of the tile sizes along each axis, on every node and its neighbours and on the first and last samples,
which a CPU test asserts.

The adjoint identity <A x, y> = <x, A^T y> over whole arrays is checked in integers: the kernel's float64 outputs
divided by q are integers (asserted), and the products are summed in int64, where a float64 sum would round (at
2048^2 it needs about 54 bits).

Random inputs at any spacing, dyadic or not, must fall within gamma_n (sum |terms|) of the float64 definition at the
seam outputs, repeat bit for bit and leave the guard cells around the output intact.  Each such case prints its
worst error / bound ratio.  Past 2^31 elements the spike inputs are built on the device and only the seam outputs
come back; those cases run one at a time and skip when the device has too little free memory."""
import itertools
import math
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ns_reference import (Geometry, assert_within, axis_specials, c_ns, filter_window, gamma,  # noqa: E402
                          nsfilters_ref, ns_matrix, nterms, point_ref, run_kernel, seam_outputs, spike_ref, tile_sizes)
from op_checks import host  # noqa: E402
from test_nsfilters import adjoint_ref, run_adjoint, work_bytes  # noqa: E402

F32, F64 = np.float32, np.float64
MANT = {F32: 24, F64: 53}
DTS = pytest.mark.parametrize("dt", [F32, F64], ids=["f32", "f64"])

# the bench geometries: bench_nsconvolve2d.py / bench_nsfilters.py, bench_nsconvolve3d.py (volume and CGLS image)
BENCH2 = {nh: Geometry((2048, 2048), (32, 32), (nh, nh), (32, 32), (64, 64)) for nh in (31, 61)}
BENCH3 = {nh: Geometry((160, 160, 160), (5, 5, 5), (nh,) * 3, (16,) * 3, (32,) * 3) for nh in (15, 31)}
CGLS3 = {nh: Geometry((96, 96, 64), (3, 3, 2), (nh,) * 3, (16,) * 3, (32,) * 3) for nh in (15, 21)}

# 2-D geometries with dyadic spacings (exact checks)
EXACT2 = {
    "bench31": BENCH2[31],
    "bench61": BENCH2[61],
    **{f"nh{n}": Geometry((300, 520), (4, 5), (n, n), (20, 5), (64, 128)) for n in (31, 33, 63, 65, 97)},
    "nh65x1": Geometry((300, 520), (4, 5), (65, 1), (20, 5), (64, 128)),
    "nh1x97": Geometry((300, 520), (4, 5), (1, 97), (20, 5), (64, 128)),
    "dh1": Geometry((256, 300), (256, 3), (5, 5), (0, 40), (1, 128)),
    "end-extrapolated": Geometry((2048, 2048), (8, 8), (31, 31), (0, 0), (64, 64)),
    "filters-past-image": Geometry((40, 600), (2, 5), (97, 33), (8, 40), (16, 128)),
    "70000x3": Geometry((70000, 3), (5, 2), (9, 3), (1000, 0), (16384, 2)),
    "3x70000": Geometry((3, 70000), (2, 5), (3, 9), (0, 1000), (2, 16384)),
}
# 2-D geometries at any spacing (bound checks)
RANDOM2 = {
    "bench61": BENCH2[61],
    "bench61-dh65": Geometry((2048, 2048), (32, 32), (61, 61), (32, 32), (65, 65)),
    **{f"nh{n}-dh65x127": Geometry((300, 520), (4, 5), (n, n), (20, 5), (65, 127)) for n in (31, 33, 63, 65, 97)},
    "nh65x1-dh13x31": Geometry((300, 520), (4, 5), (65, 1), (20, 5), (13, 31)),
    "nh1x97-dh31x13": Geometry((300, 520), (4, 5), (1, 97), (20, 5), (31, 13)),
    "dh1": Geometry((256, 300), (256, 3), (5, 5), (0, 40), (1, 127)),
    "end-extrapolated": Geometry((2048, 2048), (8, 8), (31, 31), (0, 0), (65, 127)),
    "filters-past-image": Geometry((40, 600), (3, 5), (97, 33), (1, 3), (13, 127)),
    "70000x3": Geometry((70000, 3), (5, 2), (9, 3), (1000, 0), (16383, 2)),
    "3x70000": Geometry((3, 70000), (2, 5), (3, 9), (0, 1000), (2, 16383)),
}
EXACT3 = {
    "bench15": BENCH3[15], "bench31": BENCH3[31], "cgls15": CGLS3[15], "cgls21": CGLS3[21],
    **{f"nx{n}": Geometry((n, 70, 150), (2, 3, 3), (5, 7, 9), (3, 5, 7), (16, 32, 64)) for n in (33, 34, 35)},
    **{f"nh{'x'.join(map(str, nh))}": Geometry((40, 80, 150), (2, 2, 3), nh, (4, 10, 20), (32, 64, 64))
       for nh in ((33, 17, 15), (15, 33, 17), (17, 15, 33))},
    "yz-tiles": Geometry((9, 96, 200), (2, 3, 4), (5, 33, 33), (1, 16, 5), (4, 32, 64)),
}
RANDOM3 = {                     # 31^3 taps at 160^3: test_dense_f64_bitwise_and_adjoint_identity and the spikes
    "bench15-dh31": Geometry((160, 160, 160), (5, 5, 5), (15,) * 3, (16,) * 3, (31,) * 3),
    "cgls21-dh13": Geometry((96, 96, 64), (3, 3, 2), (21,) * 3, (16,) * 3, (13, 31, 13)),
    **{f"nx{n}": Geometry((n, 70, 150), (2, 3, 3), (5, 7, 9), (3, 5, 7), (13, 31, 65)) for n in (33, 34, 35)},
    **{f"nh{'x'.join(map(str, nh))}": Geometry((40, 80, 150), (2, 2, 3), nh, (4, 10, 20), (31, 65, 64))
       for nh in ((33, 17, 15), (15, 33, 17), (17, 15, 33))},
    "yz-tiles": Geometry((9, 96, 200), (2, 3, 4), (5, 33, 33), (1, 16, 5), (4, 31, 65)),
}
# NonStationaryFilters2D: the 32 x 32 bank of the bench, the split-and-fold 2 x 3 bank of bench_nsfilters.py, and a
# bank whose short supports leave some of the parts of the longest one empty
NSF = {
    "bench31": BENCH2[31],
    "split2x3": Geometry((2048, 2048), (2, 3), (31, 31), (512, 0), (1024, 1023)),
    "empty-parts": Geometry((1100, 900), (3, 2), (5, 5), (900, 0), (64, 850)),
}
NSF1D = Geometry((1, 4000), (1, 31), (1, 81), (0, 40), (1, 128))


# ---------------------------------------------------------------------------------------------------------------
# inputs and the exactness argument
# ---------------------------------------------------------------------------------------------------------------
def small_ints(rng, shape, dt=np.float64, zero=True):
    """integers in [-4, 4] (without 0 unless ``zero``)"""
    v = rng.integers(-4, 5, shape)
    if not zero:
        v = np.where(v == 0, 4, v)
    return v.astype(dt)


def quantum(g):
    """the weight quantum 2^-(sum p) of a geometry with dyadic spacings dh = 2^p (a single filter: weight 1)"""
    p = 0
    for nf, dh in zip(g.nf, g.dh):
        if nf > 1:
            assert dh & (dh - 1) == 0, f"spacing {dh} is not a power of two"
            p += dh.bit_length() - 1
    return 2.0 ** -p


def exact_bits(g, dense, vmax=4):
    """the significand bits an output of integer taps and data (|v| <= vmax) needs at quantum(g): each output has at
    most 2^d filters times (dense) every tap of its footprint, or (a spike lattice spaced at least nh apart) one"""
    terms = 2 ** g.nd * (int(np.prod(g.nh)) if dense else 1)
    return math.ceil(math.log2(terms * vmax * vmax / quantum(g)))


def assert_exact(g, dt, dense, *arrays):
    for a in arrays:
        assert np.all(a == np.round(a)) and np.abs(a).max() <= 4
    assert exact_bits(g, dense) <= MANT[dt], (g, exact_bits(g, dense))


def nsf_exact_bits(g, vmax=4):
    """the significand bits a tap of the filter-estimation adjoint needs at quantum(g) with integer image and data
    (|v| <= vmax): one term per sample of its filter's support, the largest of which is bounded by filter_window"""
    most = max(int(np.prod([hi - lo for lo, hi in w]))
               for w in itertools.product(*[[filter_window(n, o, h, f, a) for a in range(f)]
                                            for n, o, h, f in zip(g.dims, g.oh, g.dh, g.nf)]))
    return math.ceil(math.log2(most * vmax * vmax / quantum(g)))


def assert_exact_nsf(g, dt, *arrays):
    """both directions of NonStationaryFilters exact: the convolution's dense count and the adjoint's support count"""
    assert_exact(g, dt, True, *arrays)
    assert nsf_exact_bits(g) <= MANT[dt], (g, nsf_exact_bits(g))


SPIKE_TILES = {2: (32, 64), 3: (4, 32, 64)}   # the largest tile per axis (3-D x: the float32 forward's TX = 4)


def spike_targets(g):
    """per axis, the coordinates some spike must take: ("mod", r) a coordinate of residue r modulo the axis's largest
    tile size (which covers the residues of the smaller ones, TX = 2 and 1), ("at", j) the sample j itself for every
    node and its neighbours (a support's edges) and the first and last samples"""
    out = []
    for n, T, oh, dh, nf in zip(g.dims, SPIKE_TILES[g.nd], g.oh, g.dh, g.nf):
        t = [("mod", r) for r in range(min(n, T))]
        at = {oh + a * dh + e for a in range(nf) for e in (-1, 0, 1)} | {0, n - 1}
        out.append(t + [("at", j) for j in sorted(at) if 0 <= j < n])
    return out


def spike_rounds(g, seed, min_rounds=2):
    """the spike positions of each run, (P, nd) per run: in each, no two spikes share a footprint (they differ by at
    least nh along some axis), so every output sees one spike.  Each run first places the targets of spike_targets
    still open (the k-th spike takes the k-th open target of every axis, its other coordinates random), then fills
    the free room with a lattice of odd spacing s_d >= nh_d from its own origin; until every target is met and at
    least ``min_rounds`` runs"""
    rng = np.random.default_rng(seed)
    nh = np.array(g.nh)
    s = [max(n, 3) | 1 for n in g.nh]
    origins = [(0,) * g.nd, tuple(o + 1 for o in g.oh), tuple(o + d + 1 for o, d in zip(g.oh, g.dh))]
    todo = spike_targets(g)
    rounds = []
    while any(todo) or len(rounds) < min_rounds:
        cells, pts = {}, []

        def place(p):
            c = tuple(v // h for v, h in zip(p, g.nh))
            for dc in itertools.product((-1, 0, 1), repeat=g.nd):
                for q in cells.get(tuple(a + b for a, b in zip(c, dc)), ()):
                    if np.all(np.abs(np.subtract(p, q)) < nh):
                        return False
            cells.setdefault(c, []).append(tuple(p))
            pts.append(tuple(p))
            return True

        def coord(t, d):
            n, T = g.dims[d], SPIKE_TILES[g.nd][d]
            if t is None:
                return int(rng.integers(n))
            return t[1] if t[0] == "at" else t[1] + T * int(rng.integers((n - 1 - t[1]) // T + 1))

        left = [[] for _ in range(g.nd)]
        for k in range(max(len(t) for t in todo)):
            want = [todo[d][k] if k < len(todo[d]) else None for d in range(g.nd)]
            if not any(place([coord(want[d], d) for d in range(g.nd)]) for _ in range(16)):
                for d in range(g.nd):
                    if want[d] is not None:
                        left[d].append(want[d])
        todo = left
        origin = origins[len(rounds) % len(origins)]
        ax = [np.arange(o % sd, n, sd) for o, sd, n in zip(origin, s, g.dims)]
        for p in np.stack(np.meshgrid(*ax, indexing="ij"), -1).reshape(-1, g.nd).tolist():
            place(p)
        rounds.append(np.array(sorted(pts), np.int64))
        assert len(rounds) <= 64, "spike targets that never fit"
    return rounds


def shares_footprint(g, pos):
    """whether two spikes of pos lie closer than nh along every axis"""
    nh = np.array(g.nh)
    for i in range(0, len(pos), 256):
        close = np.all(np.abs(pos[i:i + 256, None, :] - pos[None, :, :]) < nh, -1)
        close[np.arange(len(close)), np.arange(i, i + len(close))] = False
        if close.any():
            return True
    return False


def dense_array(pos, val, dims):
    x = np.zeros(tuple(dims) + (val.shape[1],))
    x[tuple(pos.T)] = val
    return x


# ---------------------------------------------------------------------------------------------------------------
# CPU: the references
# ---------------------------------------------------------------------------------------------------------------
SMALL = [Geometry((11, 13), (2, 3), (3, 5), (1, 2), (3, 2)), Geometry((17, 12), (3, 2), (7, 3), (2, 0), (5, 7)),
         Geometry((9, 40), (2, 4), (11, 33), (0, 3), (8, 10)),
         Geometry((6, 9, 5), (2, 2, 1), (3, 5, 3), (1, 2, 0), (4, 3, 1)),
         Geometry((5, 7, 11), (2, 2, 3), (5, 3, 3), (0, 1, 2), (3, 5, 4))]


@pytest.mark.parametrize("dt", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("g", SMALL, ids=lambda g: "x".join(map(str, g.dims)))
def test_point_and_spike_refs_equal_the_matrix(g, dt):
    rng = np.random.default_rng(sum(g.dims))
    hs = rng.standard_normal(g.nf + g.nh).astype(dt)
    M, B = ns_matrix(hs, g.dims, g.oh, g.dh), ns_matrix(hs, g.dims, g.oh, g.dh, absolute=True)
    x = rng.standard_normal(g.dims + (2,))
    every = np.stack(np.unravel_index(np.arange(int(np.prod(g.dims))), g.dims), 1)
    for adjoint in (False, True):
        MM, BB = (M.T, B.T) if adjoint else (M, B)
        v, b = point_ref(g, hs, x, every, adjoint, dt)
        np.testing.assert_allclose(v, MM @ x.reshape(-1, 2), rtol=0, atol=1e-13)
        np.testing.assert_allclose(b, BB @ np.abs(x.reshape(-1, 2)), rtol=1e-14, atol=0)
        # a callable input gives the same values
        v2, _ = point_ref(g, hs, lambda *c: x[c], every[::3], adjoint, dt)
        np.testing.assert_array_equal(v2, v[::3])
        # spikes: every third sample, the rest zero
        pos, val = every[::3], x.reshape(-1, 2)[::3]
        s = spike_ref(g, hs, pos, val, adjoint, dt, n_inner=2)
        np.testing.assert_allclose(s.reshape(-1, 2), MM @ dense_array(pos, val, g.dims).reshape(-1, 2), rtol=0,
                                   atol=1e-13)


@pytest.mark.parametrize("dt", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("case", [((20, 24), (2, 3), (3, 5), (1, 1), (1, 4)),
                                  ((20, 24), (4, 5), (41, 41), (1, 1), (4, 4)),
                                  ((1, 37), (1, 3), (1, 5), (0, 4), (1, 12)),
                                  ((70, 130), (3, 4), (33, 65), (5, 7), (30, 40))],
                         ids=["small", "big-filters", "x1", "partial"])
def test_nsfilters_ref_equals_the_adjoint_ref(case, dt):
    g = Geometry(*case)
    rng = np.random.default_rng(sum(g.dims))
    d, inp = rng.standard_normal(g.dims), rng.standard_normal(g.dims)
    ref, bnd = adjoint_ref(d, inp, g.nf, g.nh, g.oh, g.dh, dt)
    taps = np.stack(np.unravel_index(np.arange(ref.size), ref.shape), 1)
    v, b, _ = nsfilters_ref(g, d, inp, taps, dt)
    np.testing.assert_allclose(v, ref.ravel(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(b, bnd.ravel(), rtol=1e-13, atol=0)
    v2, _, _ = nsfilters_ref(g, lambda jx, jz: d[jx, jz][..., None], lambda jx, jz: inp[jx, jz][..., None], taps, dt)
    np.testing.assert_array_equal(v2, v)


@pytest.mark.parametrize("nd,dt,adjoint", [(2, F32, False), (2, F64, True), (3, F32, False), (3, F32, True),
                                           (3, F64, False)])
def test_seam_outputs_hold_every_seam(nd, dt, adjoint):
    g = BENCH2[61] if nd == 2 else Geometry((160, 200, 300), (5, 6, 4), (15, 15, 15), (16, 3, 40), (32, 33, 70))
    outs = seam_outputs(g, dt, adjoint)
    assert len(outs) >= 2048 and len(np.unique(outs, axis=0)) == len(outs)
    assert np.all(outs >= 0) and np.all(outs < np.array(g.dims))
    T = tile_sizes(nd, dt, adjoint)
    assert T == ((32, 64) if nd == 2 else ({F32: 2 if adjoint else 4, F64: 1}[dt], 32, 64))
    for d in range(nd):
        have = set(outs[:, d].tolist())
        for m in range(T[d], g.dims[d], T[d]):
            assert {m - 1, m} <= have, (d, m)
        for a in range(g.nf[d]):
            node = g.oh[d] + a * g.dh[d]
            assert {node - 1, node, node + 1} & set(range(g.dims[d])) <= have
        assert {0, 1, g.dims[d] - 2, g.dims[d] - 1} <= have
    assert set(axis_specials(70000, 32, 1000, 16384, 5).tolist()) >= {31, 32, 69983, 69984, 999, 1000, 1001, 69999}


@pytest.mark.parametrize("name", [f"2d-{k}" for k in EXACT2] + [f"3d-{k}" for k in EXACT3])
def test_spike_rounds_cover_every_residue_node_and_edge(name):
    """the spike runs of every exact case: no two spikes of a run share a footprint, and together the runs put a
    spike on every residue of each tile size the kernels use along each axis, on every node and its neighbours (the
    supports' edges), and on the first and last samples"""
    kind, key = name.split("-", 1)
    g = (EXACT2 if kind == "2d" else EXACT3)[key]
    rounds = spike_rounds(g, len(key))
    assert len(rounds) >= 2
    for pos in rounds:
        assert len(pos) and np.all(pos >= 0) and np.all(pos < np.array(g.dims))
        assert not shares_footprint(g, pos)
    every = np.concatenate(rounds)
    for d, n in enumerate(g.dims):
        have = set(every[:, d].tolist())
        for dt, adjoint in itertools.product((F32, F64), (False, True)):
            T = tile_sizes(g.nd, dt, adjoint)[d]
            assert {v % T for v in have} == set(range(min(n, T))), (d, T)
        nodes = {g.oh[d] + a * g.dh[d] + e for a in range(g.nf[d]) for e in (-1, 0, 1)}
        assert nodes & set(range(n)) <= have, d
        assert {0, n - 1} <= have


def test_magnitude_sketch():
    """dh = 64 in 2-D: quantum 2^-12; a dense output of 61^2 taps stays below 4 * 61^2 * 16 < 2^18, so it needs 30
    bits, and a spike lattice's at most 18; every exact case fits its dtype"""
    g = BENCH2[61]
    assert quantum(g) == 2.0 ** -12 and 4 * 61 ** 2 * 16 < 2 ** 18
    assert exact_bits(g, True) == 30 and exact_bits(g, False) <= 18
    for g in list(EXACT2.values()) + list(EXACT3.values()):
        assert exact_bits(g, True) <= 53 and exact_bits(g, False) <= 24, g
    assert exact_bits(NSF1D, True) <= 53
    # a tap of the filter-estimation adjoint sums its filter's support: 129^2 samples at most at the bench bank,
    # 31 bits at q = 2^-12
    assert nsf_exact_bits(BENCH2[31]) == 31 and nsf_exact_bits(NSF1D) <= 53


# ---------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pm():
    import pylops_mpi_b200 as pm
    return pm


def report(what, ratio):
    print(f"\nNS_EXACT_RATIO {what} {ratio:.3e}")


def check_bound(got, ref, bnd, n, dt, what):
    """|got - ref| <= gamma_n bnd componentwise; reports the worst ratio"""
    tol = gamma(n, dt) * bnd
    err = np.abs(got.astype(np.float64) - ref)
    assert_within(got, ref, tol)
    report(what, float(np.max(np.where(tol > 0, err / np.where(tol > 0, tol, 1), 0.0))))


def at(y, outs):
    return y[tuple(np.asarray(outs).T)]


def int_inner(a, b):
    return int(np.dot(a.ravel().astype(np.int64), b.ravel().astype(np.int64)))


def to_ints(v, q):
    s = v.astype(np.float64) / q
    assert np.all(s == np.round(s)), "an exact output is not a multiple of the weight quantum"
    return s.astype(np.int64)


def nsf_geom(g):
    return (g.dims[0], g.dims[1], g.nf[0], g.nf[1], g.nh[0], g.nh[1], g.oh[0], g.dh[0], g.oh[1], g.dh[1])


# ---------------------------------------------------------------------------------------------------------------
# GPU: dense integer inputs, float64, bitwise at the seam outputs, and the adjoint identity in integers
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["2d-bench31", "2d-bench61", "3d-bench15", "3d-bench31", "3d-cgls15", "3d-cgls21"])
def test_dense_f64_bitwise_and_adjoint_identity(pm, name):
    kind, key = name.split("-")
    g = (BENCH2 if kind == "2d" else BENCH3 if "bench" in key else CGLS3)[int(key[-2:])]
    rng = np.random.default_rng(len(name))
    hs, x, v = small_ints(rng, g.nf + g.nh), small_ints(rng, g.dims + (1,)), small_ints(rng, g.dims + (1,))
    assert_exact(g, F64, True, hs, x, v)
    y, ok1, same1 = run_kernel(pm, x, hs, g.oh, g.dh, False, F64)
    xa, ok2, same2 = run_kernel(pm, v, hs, g.oh, g.dh, True, F64)
    assert ok1 and ok2 and same1 and same2
    for adjoint, got, inp in ((False, y, x), (True, xa, v)):
        outs = seam_outputs(g, F64, adjoint)
        ref, _ = point_ref(g, hs, inp, outs, adjoint, F64, bound=False)
        np.testing.assert_array_equal(at(got, outs), ref, err_msg=f"{name} adjoint={adjoint}")
    q = quantum(g)
    assert int_inner(to_ints(y, q), v) == int_inner(x, to_ints(xa, q))


@pytest.mark.gpu
@pytest.mark.parametrize("nh", [31, 61])
def test_nsfilters2d_dense_f64_bitwise_and_adjoint_identity(pm, nh):
    """forward b2_nsconvolve2d of the image by the model bank against adjoint b2_nsfilters2d_adjoint"""
    import torch
    g = BENCH2[nh]
    rng = np.random.default_rng(nh)
    inp, m, d = small_ints(rng, g.dims), small_ints(rng, g.nf + g.nh), small_ints(rng, g.dims)
    assert_exact_nsf(g, F64, inp, m, d)
    y, ok, same = run_kernel(pm, inp[..., None], m, g.oh, g.dh, False, F64)
    assert ok and same
    gk, ok, same, nw = run_adjoint(pm, d, inp, g.nf, g.nh, g.oh, g.dh, F64)
    assert ok and same and nw == 0
    taps = nsf_taps(g, rng)
    ref, _, _ = nsfilters_ref(g, d, inp, taps, F64)
    np.testing.assert_array_equal(gk[tuple(taps.T)], ref)
    q = quantum(g)
    assert int_inner(to_ints(y[..., 0], q), d) == int_inner(m, to_ints(gk, q))
    torch.cuda.empty_cache()


def nsf_taps(g, rng, need=2048):
    """bank entries (a, b, kx, kz) worth checking: every tap of the first and last filters along each axis and of
    one filter in the middle, both sides of every 32 x 64 tap-tile seam, then random fill"""
    nf, nh = g.nf, g.nh
    filt = {(a, b) for a in {0, nf[0] // 2, nf[0] - 1} for b in {0, nf[1] // 2, nf[1] - 1}}
    out = set()
    for a, b in filt:
        for kx in range(nh[0]):
            for kz in range(nh[1]):
                out.add((a, b, kx, kz))
    for kx in [k for m in range(32, nh[0], 32) for k in (m - 1, m)] or [nh[0] - 1]:
        for kz in range(nh[1]):
            out.add((int(rng.integers(nf[0])), int(rng.integers(nf[1])), kx, kz))
    for kz in [k for m in range(64, nh[1], 64) for k in (m - 1, m)] or [nh[1] - 1]:
        for kx in range(nh[0]):
            out.add((int(rng.integers(nf[0])), int(rng.integers(nf[1])), kx, kz))
    total = int(np.prod(nf + nh))
    while len(out) < min(need, total):
        out.add(tuple(int(rng.integers(n)) for n in nf + nh))
    return np.array(sorted(out), np.int64)


@pytest.mark.gpu
def test_nsfilters1d_forward_against_adjoint_exact(pm):
    """NonStationaryFilters1D: forward b2_nsconvolve_axis against adjoint b2_nsfilters2d_adjoint with a singleton x
    axis, both bit for bit against the definition, and the adjoint identity in integers"""
    import torch
    g = NSF1D
    L = pm._lib
    rng = np.random.default_rng(1)
    inp, m, d = small_ints(rng, g.dims), small_ints(rng, g.nf + g.nh), small_ints(rng, g.dims)
    assert_exact_nsf(g, F64, inp, m, d)
    n, nf, nh = g.dims[1], g.nf[1], g.nh[1]
    xi, hm = torch.as_tensor(inp.ravel()).cuda(), torch.as_tensor(m.ravel()).cuda()
    y = torch.full((n,), 7.25, dtype=torch.float64, device="cuda")
    assert L.lib.b2_nsconvolve_axis(L.ctx(), xi.data_ptr(), y.data_ptr(), 1, n, 1, hm.data_ptr(), nf, nh, nh // 2,
                                    g.oh[1], g.dh[1], 0, L.F64, L.stream()) == 0
    y = host(y).reshape(g.dims)
    every = np.stack(np.unravel_index(np.arange(n), g.dims), 1)
    ref, _ = point_ref(g, m, inp, every, False, F64, bound=False)
    np.testing.assert_array_equal(y.ravel(), ref[:, 0])
    gk, ok, same, nw = run_adjoint(pm, d, inp, g.nf, g.nh, g.oh, g.dh, F64)
    assert ok and same
    taps = np.stack(np.unravel_index(np.arange(gk.size), gk.shape), 1)
    gref, _, _ = nsfilters_ref(g, d, inp, taps, F64)
    np.testing.assert_array_equal(gk.ravel(), gref)
    q = quantum(g)
    assert int_inner(to_ints(y, q), d) == int_inner(m, to_ints(gk, q))


# ---------------------------------------------------------------------------------------------------------------
# GPU: spike lattices, whole output bitwise
# ---------------------------------------------------------------------------------------------------------------
def run_spikes(pm, g, dt, adjoint, seed):
    rng = np.random.default_rng(seed)
    hs = small_ints(rng, g.nf + g.nh, dt)
    for i, pos in enumerate(spike_rounds(g, seed)):
        ni = 1 + i % 2
        val = small_ints(rng, (len(pos), ni), zero=False)
        assert_exact(g, dt, False, hs, val)
        x = dense_array(pos, val, g.dims).astype(dt)
        y, ok, same = run_kernel(pm, x, hs, g.oh, g.dh, adjoint, dt)
        assert ok and same
        want = spike_ref(g, hs, pos, val, adjoint, dt, ni)
        np.testing.assert_array_equal(y, want, err_msg=f"run {i} n_inner {ni}")


@pytest.mark.gpu
@pytest.mark.parametrize("adjoint", [False, True], ids=["fwd", "adj"])
@DTS
@pytest.mark.parametrize("name", list(EXACT2))
def test_spikes_2d_bitwise(pm, name, dt, adjoint):
    run_spikes(pm, EXACT2[name], dt, adjoint, len(name))


@pytest.mark.gpu
@pytest.mark.parametrize("adjoint", [False, True], ids=["fwd", "adj"])
@DTS
@pytest.mark.parametrize("name", list(EXACT3))
def test_spikes_3d_bitwise(pm, name, dt, adjoint):
    run_spikes(pm, EXACT3[name], dt, adjoint, len(name))


# ---------------------------------------------------------------------------------------------------------------
# GPU: random inputs at any spacing, within gamma_n of the definition at the seam outputs
# ---------------------------------------------------------------------------------------------------------------
def run_random(pm, g, dt, adjoint, name):
    rng = np.random.default_rng(len(name) + 7 * adjoint)
    hs = rng.standard_normal(g.nf + g.nh).astype(dt)
    x = rng.standard_normal(g.dims + (1,)).astype(dt)
    y, ok, same = run_kernel(pm, x, hs, g.oh, g.dh, adjoint, dt)
    assert ok and same
    outs = seam_outputs(g, dt, adjoint)
    ref, bnd = point_ref(g, hs, x.astype(np.float64), outs, adjoint, dt)
    check_bound(at(y, outs), ref, bnd, nterms(g), dt, f"{g.nd}d/{name}/{dt.__name__}/{'adj' if adjoint else 'fwd'}")


@pytest.mark.gpu
@pytest.mark.parametrize("adjoint", [False, True], ids=["fwd", "adj"])
@DTS
@pytest.mark.parametrize("name", list(RANDOM2))
def test_random_2d_within_bound(pm, name, dt, adjoint):
    run_random(pm, RANDOM2[name], dt, adjoint, name)


@pytest.mark.gpu
@pytest.mark.parametrize("adjoint", [False, True], ids=["fwd", "adj"])
@DTS
@pytest.mark.parametrize("name", list(RANDOM3))
def test_random_3d_within_bound(pm, name, dt, adjoint):
    run_random(pm, RANDOM3[name], dt, adjoint, name)


@pytest.mark.gpu
@DTS
@pytest.mark.parametrize("name", list(NSF))
def test_nsfilters_within_bound(pm, name, dt):
    """the adjoint within gamma_K (sum |terms|) at chosen taps (K the support's samples + 3, as in
    test_nsfilters.py), and the forward, b2_nsconvolve2d with the image as its input, at the seam outputs.  The
    split bank's image is a spike lattice spaced 11, so that its reference stays cheap over supports of millions of
    samples"""
    g = NSF[name]
    rng = np.random.default_rng(len(name))
    d = rng.standard_normal(g.dims).astype(dt)
    inp = rng.standard_normal(g.dims).astype(dt)
    if name == "split2x3":
        lat = np.zeros(g.dims, dt)
        lat[::11, 3::11] = inp[::11, 3::11]
        inp = lat
    gk, ok, same, nw = run_adjoint(pm, d, inp, g.nf, g.nh, g.oh, g.dh, dt)
    assert ok and same
    assert (nw > 0) == (name != "bench31"), nw
    taps = nsf_taps(g, rng)
    ref, bnd, K = nsfilters_ref(g, d.astype(np.float64), inp.astype(np.float64), taps, dt)
    check_bound(gk[tuple(taps.T)], ref, bnd, K + 3, dt, f"nsf/{name}/{dt.__name__}/adj")
    m = rng.standard_normal(g.nf + g.nh).astype(dt)
    y, ok, same = run_kernel(pm, inp[..., None], m, g.oh, g.dh, False, dt)
    assert ok and same
    outs = seam_outputs(g, dt, False)
    ref, bnd = point_ref(g, m, inp[..., None].astype(np.float64), outs, False, dt)
    check_bound(at(y, outs), ref, bnd, nterms(g), dt, f"nsf/{name}/{dt.__name__}/fwd")


# ---------------------------------------------------------------------------------------------------------------
# GPU: past 2^31 elements, float32 spikes built on the device, checked at the seam outputs
# ---------------------------------------------------------------------------------------------------------------
def need_memory(nbytes):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + (1 << 30):
        pytest.skip(f"needs {nbytes / 2 ** 30:.1f} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")


def device_spikes(n, pos_flat, val, dt):
    import torch
    x = torch.zeros(n, dtype=getattr(torch, np.dtype(dt).name), device="cuda")
    x[torch.as_tensor(pos_flat).cuda()] = torch.as_tensor(val.astype(dt)).cuda()
    return x


def run_big(call, n, outs_flat, dt, guard=5):
    """call(y) twice into n elements between guard cells of 7.25; returns the first run's values at outs_flat and
    checks the guards and that the second run repeats them"""
    import torch
    yb = torch.full((n + 2 * guard,), 7.25, dtype=getattr(torch, np.dtype(dt).name), device="cuda")
    y = yb[guard:guard + n]
    idx = torch.as_tensor(outs_flat).cuda()
    assert call(y.data_ptr()) == 0
    first = host(y[idx])
    assert call(y.data_ptr()) == 0
    torch.cuda.synchronize()
    assert np.array_equal(host(y[idx]), first)
    assert bool((yb[:guard] == 7.25).all()) and bool((yb[guard + n:] == 7.25).all())
    return first


def spike_value(pos):
    """the value of the spike at flat position(s) pos: an integer in [-4, 4] \\ {0}"""
    v = (pos * 7 + 3) % 8 - 4
    return np.where(v == 0, 4, v)


def lattice_flat(g, s, n_inner=1):
    """the flat positions (spikes spaced s along every axis, offset 1 along the last) of a spike lattice"""
    ax = [np.arange(0, n, s) if d < g.nd - 1 else np.arange(1, n, s) for d, n in enumerate(g.dims)]
    pos = np.stack(np.meshgrid(*ax, indexing="ij"), -1).reshape(-1, g.nd)
    flat = np.ravel_multi_index(tuple(pos.T), g.dims).astype(np.int64)
    return pos, flat


def big_outputs(g, adjoint, pos, dt):
    """seam outputs plus the outputs around the last spikes (whose flat index is past 2^31)"""
    outs = seam_outputs(g, dt, adjoint)
    steps = np.stack(np.meshgrid(*[np.arange(-h, h + 1) for h in g.hc], indexing="ij"), -1).reshape(-1, g.nd)
    near = (pos[-64:, None, :] + steps[None]).reshape(-1, g.nd)
    near = near[np.all((near >= 0) & (near < np.array(g.dims)), 1)]
    return np.unique(np.concatenate([outs, near]), axis=0)


def check_big_conv(pm, g, n_inner, adjoint):
    import torch
    dt = F32
    L = pm._lib
    total = int(np.prod(g.dims)) * n_inner
    assert total > 2 ** 31
    need_memory(2 * total * 4)
    torch.cuda.reset_peak_memory_stats()
    rng = np.random.default_rng(3)
    hs = small_ints(rng, g.nf + g.nh, dt)
    s = 61
    pos, flat = lattice_flat(g, s)
    vals = np.stack([spike_value(flat * n_inner + c) for c in range(n_inner)], 1).astype(np.float64)
    assert_exact(g, dt, False, hs, vals)
    xfl = (flat[:, None] * n_inner + np.arange(n_inner)[None]).ravel()
    assert xfl.max() >= 2 ** 31
    x = device_spikes(total, xfl, vals.ravel(), dt)
    del xfl
    hd = torch.as_tensor(hs).cuda()
    outs = big_outputs(g, adjoint, pos, dt)
    oflat = (np.ravel_multi_index(tuple(outs.T), g.dims).astype(np.int64)[:, None] * n_inner
             + np.arange(n_inner)[None]).ravel()
    got = run_big(lambda yp: c_ns(pm, x.data_ptr(), yp, g.dims, n_inner, hd.data_ptr(), g.nf, g.nh, g.oh, g.dh,
                                  int(adjoint), L.F32), total, oflat, dt)

    def xs(*c):
        """the spike input at coordinates c: spike_value on the lattice, 0 elsewhere"""
        on = (c[-1] % s == 1)
        for cd in c[:-1]:
            on = on & (cd % s == 0)
        f = np.ravel_multi_index(c, g.dims).astype(np.int64)
        return np.stack([np.where(on, spike_value(f * n_inner + ch), 0) for ch in range(n_inner)], -1)

    ref, _ = point_ref(g, hs, xs, outs, adjoint, dt, bound=False)
    np.testing.assert_array_equal(got.reshape(-1, n_inner), ref)
    peak = torch.cuda.max_memory_allocated()
    print(f"\nNS_EXACT_PEAK {g.nd}d {'x'.join(map(str, g.dims))}x{n_inner} {'adj' if adjoint else 'fwd'} "
          f"{peak / 2 ** 30:.2f} GiB")
    del x, hd
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("adjoint", [False, True], ids=["fwd", "adj"])
def test_past_2_31_conv2d(pm, adjoint):
    check_big_conv(pm, Geometry((46400, 46400), (725, 725), (5, 5), (32, 32), (64, 64)), 1, adjoint)


@pytest.mark.gpu
@pytest.mark.parametrize("adjoint", [False, True], ids=["fwd", "adj"])
def test_past_2_31_conv3d_complex(pm, adjoint):
    """complex 1040 x 1024^2: its addresses pass 2^31 through the n_inner factor only (the sample index stays below
    2^30); test_past_2_31_conv3d has the sample index itself past 2^31"""
    check_big_conv(pm, Geometry((1040, 1024, 1024), (32, 32, 32), (5, 5, 5), (16, 16, 16), (32, 32, 32)), 2, adjoint)


@pytest.mark.gpu
@pytest.mark.parametrize("adjoint", [False, True], ids=["fwd", "adj"])
def test_past_2_31_conv3d(pm, adjoint):
    """1300^3 real: (x ny + y) nz itself passes 2^31, so a 32-bit sample index would wrap"""
    check_big_conv(pm, Geometry((1300, 1300, 1300), (41, 41, 41), (5, 5, 5), (16, 16, 16), (32, 32, 32)), 1, adjoint)


@pytest.mark.gpu
def test_past_2_31_nsfilters(pm):
    """an image of 46400^2 with 3 x 3 taps: inp a spike lattice spaced 9 (at most 15^2 spikes per support of 128^2,
    so every sum is exact in float32), d a pattern computed on the device"""
    import torch
    dt = F32
    L = pm._lib
    g = Geometry((46400, 46400), (725, 725), (3, 3), (32, 32), (64, 64))
    nx, nz = g.dims
    total = nx * nz
    need_memory(2 * total * 4)
    torch.cuda.reset_peak_memory_stats()
    s = 9
    assert ((nx - 1) // s * s) * nz >= 2 ** 31                 # the last rows of spikes lie past 2^31
    assert 15 * 15 * 16 / quantum(g) < 2 ** 24
    inp = torch.zeros(total, dtype=torch.float32, device="cuda")
    d = torch.empty(total, dtype=torch.float32, device="cuda")
    cols = torch.arange(nz, device="cuda", dtype=torch.int64)
    lx, lz = torch.arange(0, nx, s, device="cuda"), torch.arange(1, nz, s, device="cuda")
    for r0 in range(0, len(lx), 256):
        f = lx[r0:r0 + 256, None] * nz + lz[None]
        v = (f * 7 + 3) % 8 - 4
        inp[f.ravel()] = torch.where(v == 0, 4, v).float().ravel()
    for r0 in range(0, nx, 2048):
        rows = torch.arange(r0, min(nx, r0 + 2048), device="cuda", dtype=torch.int64)
        d.view(nx, nz)[r0:r0 + len(rows)] = ((rows[:, None] * 5 + cols[None] * 3) % 9 - 4).float()

    def dval(jx, jz):
        return ((jx * 5 + jz * 3) % 9 - 4)[..., None].astype(np.float64)

    def ival(jx, jz):
        on = (jx % s == 0) & (jz % s == 1)
        return np.where(on, spike_value(jx.astype(np.int64) * nz + jz), 0)[..., None].astype(np.float64)

    gm = nsf_geom(g)
    code = L.F32
    nw = work_bytes(pm, gm, code)
    work = torch.empty(max(nw, 1), dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(0)
    taps = nsf_taps(g, rng)
    nb = int(np.prod(g.nf + g.nh))
    tflat = np.ravel_multi_index(tuple(taps.T), g.nf + g.nh).astype(np.int64)
    got = run_big(lambda gp: L.lib.b2_nsfilters2d_adjoint(L.ctx(), d.data_ptr(), inp.data_ptr(), gp, *gm,
                                                          work.data_ptr(), nw, code, L.stream()), nb, tflat, dt)
    ref, _, _ = nsfilters_ref(g, dval, ival, taps, dt)
    np.testing.assert_array_equal(got, ref)
    print(f"\nNS_EXACT_PEAK nsf 46400x46400 {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    del inp, d, work
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
# GPU: argument limits of the 32-bit 3-D kernel
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_conv3d_axis_limit(pm):
    """an axis, filter size or node position of 2^29 samples is refused and y is left untouched; an axis of 2^29 - 1
    runs and is right at its seams and around its spikes, along x and along z.  The refused calls get buffers as
    large as their shapes, so that a launch they should not make would stay inside them and fail the test cleanly"""
    import torch
    L = pm._lib
    LIM = 2 ** 29
    need_memory(3 * LIM * 4)
    x = torch.zeros(LIM, dtype=torch.float32, device="cuda")
    y = torch.full((LIM,), 7.25, dtype=torch.float32, device="cuda")
    hs = torch.ones(LIM, dtype=torch.float32, device="cuda")
    base = dict(dims=(1, 1, 1), nf=(1, 1, 1), nh=(1, 1, 1), oh=(0, 0, 0), dh=(1, 1, 1))
    for kw in (dict(dims=(LIM, 1, 1)), dict(dims=(1, LIM, 1)), dict(dims=(1, 1, LIM)), dict(nh=(1, 1, LIM)),
               dict(nf=(1, 1, 2), oh=(0, 0, LIM - 1), dh=(1, 1, 1)), dict(nf=(1, 1, 2), dh=(1, 1, LIM))):
        a = dict(base, **kw)
        for adjoint in (0, 1):
            assert c_ns(pm, x.data_ptr(), y.data_ptr(), a["dims"], 1, hs.data_ptr(), a["nf"], a["nh"], a["oh"],
                        a["dh"], adjoint, L.F32) == 2002, kw
    torch.cuda.synchronize()
    assert bool((y == 7.25).all())
    del x, y, hs
    torch.cuda.empty_cache()
    rng = np.random.default_rng(5)
    for axis in (0, 2):
        dims = [1, 1, 1]
        dims[axis] = LIM - 1
        nf, nh, oh, dh = [1, 1, 1], [1, 1, 1], [0, 0, 0], [1, 1, 1]
        nf[axis], nh[axis], oh[axis], dh[axis] = 3, 5, 2 ** 26, 2 ** 27
        g = Geometry(dims, nf, nh, oh, dh)
        hs = small_ints(rng, g.nf + g.nh, F32)
        # spikes at both ends, on and between the nodes and past the last one
        p = np.array(sorted({0, 5, 2 ** 26, 2 ** 26 + 2 ** 25 + 3, 2 ** 27 + 2 ** 26, 2 ** 28 + 2 ** 26,
                             2 ** 28 + 2 ** 26 + 7, LIM - 3, LIM - 2}), np.int64)
        val = spike_value(p).astype(np.float64)
        xd = device_spikes(LIM - 1, p, val, F32)
        hd = torch.as_tensor(hs).cuda()
        for adjoint in (False, True):
            # the seams of the first and last 64 tiles, the nodes +- 1, and the spikes' footprints
            T = tile_sizes(3, F32, adjoint)[axis]
            last = (LIM - 2) // T * T
            js = [np.arange(0, 64 * T), np.arange(last - 64 * T, LIM - 1), p[:, None] + np.arange(-2, 3),
                  g.oh[axis] + g.dh[axis] * np.arange(3)[:, None] + np.arange(-1, 2)[None]]
            j = np.unique(np.clip(np.concatenate([np.ravel(v) for v in js]), 0, LIM - 2))
            outs = np.zeros((len(j), 3), np.int64)
            outs[:, axis] = j
            oflat = outs[:, axis].astype(np.int64)
            got = run_big(lambda yp: c_ns(pm, xd.data_ptr(), yp, g.dims, 1, hd.data_ptr(), g.nf, g.nh, g.oh, g.dh,
                                          int(adjoint), L.F32), LIM - 1, oflat, F32)
            pset = dict(zip(p.tolist(), val.tolist()))

            def xs(*c):
                j = c[axis]
                return np.vectorize(lambda t: pset.get(int(t), 0.0))(j)[..., None]

            ref, bnd = point_ref(g, hs, xs, outs, adjoint, F32)     # weights of 2^-27: within the bound
            assert np.count_nonzero(ref) >= 2 * len(p)
            assert_within(got, ref[:, 0], gamma(nterms(g), F32) * bnd[:, 0])
        del xd, hd
        torch.cuda.empty_cache()
