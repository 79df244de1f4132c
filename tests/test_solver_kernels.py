"""GPU tests, kernel level, of the kernels under the solvers: the ISTA / FISTA update (b2_sparse_update), the CGLS
vector updates (b2_lincomb_dev, b2_lincomb_dev_norm2), the reductions (b2_dot_multi, b2_norm_partial, b2_norm_axis)
and the device-scalar helpers (b2_scalar_div, b2_history_push), called through the C ABI and compared with plain
float64 (or long double) NumPy references.

Conventions:
- every output buffer has GUARD sentinel elements before and after it, checked after each call;
- edge sizes come from the device's SM count: V = scalars per 16-byte vector, the unrolled loop of the vector path
  engages when nvec > 3 * 256 * grid, the grid is capped at sm_count * 8 (reductions, sparse update) and
  sm_count * 16 (b2_norm_axis);
- every tolerance is a bound written in units of the unit roundoff 2^-p of the array's precision (p = 24 or 53) or of
  float64 (2^-53), derived where it is used.
Complex infinities are out of scope: the threshold of a complex +-inf is not tested.
"""
import ctypes as C
import importlib.util
import math
import os
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
_SHIM = os.path.join(HERE, "golden", "refshim", "pylops", "optimization", "cls_sparsity.py")
_spec = importlib.util.spec_from_file_location("_refshim_cls_sparsity", _SHIM)
ref_sparsity = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(ref_sparsity)

GUARD = 16         # sentinel scalars each side of an output (64 / 128 bytes: the payload keeps its 16-byte alignment)
SENT = -1234.5     # exact in float32 and float64
U64 = 2.0 ** -53   # float64 unit roundoff

# name: (numpy dtype, real numpy dtype, real torch dtype, ABI code, complex, precision bits p)
DT = {"f32": (np.float32, np.float32, torch.float32, 0, False, 24),
      "f64": (np.float64, np.float64, torch.float64, 1, False, 53),
      "c64": (np.complex64, np.float32, torch.float32, 2, True, 24),
      "c128": (np.complex128, np.float64, torch.float64, 3, True, 53)}
NONE, SOFT, HARD, HALF = 0, 1, 2, 3
KINDS = {"none": NONE, "soft": SOFT, "hard": HARD, "half": HALF}
RESTATE = {SOFT: ref_sparsity._softthreshold, HARD: ref_sparsity._hardthreshold, HALF: ref_sparsity._halfthreshold}
NRM_COUNT, NRM_ABS, NRM_SQ, NRM_MAX, NRM_MIN, NRM_POW = range(6)


@pytest.fixture(scope="module")
def L():
    import pylops_mpi_b200._lib as L
    return L


@pytest.fixture(scope="module")
def sms(L):
    n = C.c_int()
    L.check(L.lib.b2_ctx_sm_count(L.ctx(), C.byref(n)))
    return n.value


def red_cap(sms):
    """the grid cap of the fused reductions, restating b2_red_grid in csrc/common.cuh"""
    return min(sms * 8, 2048)


def shift_of(dt):
    """real scalars a pointer is moved by to leave 16-byte alignment: one element, except complex128, whose
    elements are 16 bytes (8 bytes is its natural float64 alignment)"""
    return {"f32": 1, "f64": 1, "c64": 2, "c128": 1}[dt]


class Buf:
    """device copy of a host array (as real scalars) between two runs of GUARD sentinels, `shift` scalars in"""

    def __init__(self, host, dt, shift=0):
        npdt, rdt, tdt, _, cx, _ = DT[dt]
        self.dt, self.cx = dt, cx
        real = np.ascontiguousarray(np.asarray(host, dtype=npdt)).view(rdt).ravel()
        self.n = real.size
        self.off = GUARD + shift
        self.t = torch.full((2 * GUARD + shift + max(self.n, 1),), SENT, dtype=tdt, device="cuda")
        if self.n:
            self.t[self.off:self.off + self.n] = torch.from_numpy(real.copy()).cuda()

    @property
    def ptr(self):
        return self.t.data_ptr() + self.off * self.t.element_size()

    def get(self):
        npdt, rdt = DT[self.dt][:2]
        return self.t[self.off:self.off + self.n].cpu().numpy().astype(rdt).view(npdt)

    def check_guards(self):
        a = self.t.cpu().numpy()
        assert np.all(a[:self.off] == SENT), "write before the buffer"
        assert np.all(a[self.off + self.n:] == SENT), "write after the buffer"


def dbuf(n, fill=SENT):
    """float64 device scalars (outputs of the reductions), sentinel-filled, with guards"""
    return Buf(np.full(n, fill), "f64")


def rnd(rng, n, dt, scale=1.0):
    npdt, _, _, _, cx, _ = DT[dt]
    a = rng.standard_normal(n) * scale
    if cx:
        a = a + 1j * rng.standard_normal(n) * scale
    return a.astype(npdt)


def bits_equal(a, b):
    """bit equality of two float arrays (complex compared per component)"""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if np.iscomplexobj(a):
        a, b = a.view(a.real.dtype), b.view(b.real.dtype)
    ui = np.uint32 if a.dtype == np.float32 else np.uint64
    return np.array_equal(a.view(ui), b.view(ui))


def ld(a):
    """exact widening to long double (complex: a pair of long double arrays)"""
    if np.iscomplexobj(a):
        return a.real.astype(np.longdouble), a.imag.astype(np.longdouble)
    return a.astype(np.longdouble)


def vec_sizes(dt, sms):
    """element counts at the edges of the 16-byte vector path of the streaming kernels (grid 1 below 1024 vectors)"""
    _, rdt, _, _, cx, _ = DT[dt]
    V = 16 // np.dtype(rdt).itemsize           # real scalars per vector
    per = 2 if cx else 1
    Ve = max(V // per, 1)                       # elements per vector
    tail = (V - per) // per                     # most elements a vector tail can hold
    s = {1, Ve, Ve + 1, 768 * Ve, 768 * Ve + tail, 769 * Ve, 769 * Ve + tail}   # unrolled group: nvec > 3 * 256
    if Ve > 1:
        s.add(Ve - 1)
    if dt == "c64":
        s |= {3, 769 * Ve + 1}                   # odd complex64 counts: one trailing pair
    return sorted(x for x in s if x >= 1)


def big_size(dt, sms):
    """capped grid, unrolled loop striding twice, then the remainder loop and a vector tail"""
    _, rdt, _, _, cx, _ = DT[dt]
    V = 16 // np.dtype(rdt).itemsize
    per = 2 if cx else 1
    nvec = 9 * 256 * red_cap(sms) + 5
    return (nvec * V + (V - per)) // per


# ======================================================================================================================
# b2_sparse_update
# ======================================================================================================================
# roles -> buffer names; the aliasing patterns the solvers use plus fully distinct ones
CONFIGS = {
    "thresh": dict(base="A", xnew="A"),                                   # thresholding only
    "ista": dict(base="A", g="G", xold="A", xnew="A"),                     # fused ISTA step, in place
    "fista": dict(base="Z", g="G", xold="X", xnew="X", znew="Z"),         # fused FISTA step: z and x in place
    "distinct": dict(base="A", g="G", xold="B", xnew="D", znew="E"),
    "g_no_xold": dict(base="A", g="G", xnew="D"),
    "xold_no_g": dict(base="A", xold="B", xnew="D", znew="E"),
}


def sparse_call(L, roles, bufs, alpha, thresh, kind, c, sums, n, code):
    p = {r: (bufs[b].ptr if b else None) for r, b in ((r, roles.get(r)) for r in ("base", "g", "xold", "xnew", "znew"))}
    return L.lib.b2_sparse_update(L.ctx(), p["base"], p["g"], alpha, p["xold"], thresh, kind, p["xnew"], p["znew"], c,
                                  sums.ptr if sums is not None else None, n, code, L.stream())


def run_sparse(L, dt, kind, cfg, n, rng, alpha, thresh, c, align="aligned", nan_at=()):
    roles = CONFIGS[cfg]
    code = DT[dt][3]
    names = sorted(set(roles.values()))
    host = {b: rnd(rng, n, dt) for b in names}
    for i in nan_at:                              # NaN in the base of u and, one element on, in the gradient
        host[roles["base"]][i] = np.nan
        if "g" in roles and i + 1 < n:
            host[roles["g"]][i + 1] = np.nan
    sh = shift_of(dt)
    shifts = {b: 0 for b in names}
    if align == "shifted":
        shifts = {b: sh for b in names}
    elif align == "mixed":
        shifts[names[-1]] = sh
    bufs = {b: Buf(host[b], dt, shifts[b]) for b in names}
    sums = dbuf(2)
    L.check(sparse_call(L, roles, bufs, alpha, thresh, kind, c, sums, n, code), "b2_sparse_update")
    torch.cuda.synchronize()
    for b in bufs.values():
        b.check_guards()
    sums.check_guards()
    out = dict(v=bufs[roles["xnew"]].get(), sums=sums.get(),
               base=host[roles["base"]], g=host.get(roles.get("g")), xold=host.get(roles.get("xold")))
    out["z"] = bufs[roles["znew"]].get() if "znew" in roles else None
    return out


def u_of(r, dt, alpha):
    """u = base + alpha*g in the array's precision.  alpha is a power of two: alpha*g is exact, so NumPy's two
    operations round once, like the kernel's fma"""
    _, rdt, _, _, cx, _ = DT[dt]
    if r["g"] is None:
        return r["base"].copy()
    b, g = r["base"].view(rdt), r["g"].view(rdt)
    return (b + rdt(alpha) * g).view(r["base"].dtype)


def restate(u, kind, thresh):
    return u.copy() if kind == NONE else RESTATE[kind](u, thresh)


# half threshold, relative error bound of the kernel against the exact function, in units of 2^-p.  CUDA's ulp table:
# rsqrt 2 ulp (float; 1 in double), acos 2 ulp, cos 2 ulp, one ulp <= 2 * 2^-p relative.  r = rsqrt(a * 1/3):
# 2 roundings + 4 = 6; r^3: 3*6 + 2 = 20; arg = (t/8) r^3: 20 + 2 = 22.  Past the cut arg <= 1/sqrt(2), where acos is
# conditioned by arg / sqrt(1 - arg^2) <= 1: 22 abs, + 4 * pi/2 for acos itself = 29; phi = 2/3 acos: ~20 + 2;
# 2pi/3 - phi: +2 + 2 (constant and subtraction); cos has slope <= 1 and value in [0, 1/2]: +2; 1 + cos >= 1, so the
# absolute error is a relative one: ~27; times 2/3 and u: +3 = 30.  40 leaves room; the float64 reference's own
# rounding (a few 2^-53) is covered in the double case by the same margin plus 16.
HALF_ULPS = 56


def check_threshold(r, dt, kind, thresh, alpha):
    """xnew against the restatement applied to u (the exact u: alpha is dyadic)"""
    npdt, rdt, _, _, cx, p = DT[dt]
    u = u_of(r, dt, alpha)
    v = r["v"]
    up = 2.0 ** -p
    if not cx and kind in (NONE, SOFT, HARD):
        # the restatement in the array's precision does exactly what the kernel does: bit equality
        ref = restate(u, kind, thresh)
        assert bits_equal(v, ref), (dt, kind, np.flatnonzero(v != ref)[:8])
        return
    if not cx:                                    # half
        ref = ref_sparsity._halfthreshold(u.astype(np.float64), thresh)
        # which elements are cut: decided by the restatement in the array's precision (its cut is a Python float)
        zero = restate(u, HALF, thresh) == 0
        assert np.all(v[zero] == 0), np.flatnonzero(v[zero] != 0)[:8]
        cut = (54 ** (1.0 / 3.0) / 4.0) * thresh ** (2.0 / 3.0)
        amb = ~zero & (ref == 0)                  # float64 cut, float32 |u|: only within an ulp of the cut
        assert np.all(np.abs(np.abs(u[amb].astype(np.float64)) - cut) <= 2.0 ** (1 - p) * cut)
        kept = ~zero & ~amb
        err = np.abs(v[kept].astype(np.float64) - ref[kept])
        bound = HALF_ULPS * up * np.abs(u[kept].astype(np.float64))
        assert np.all(err <= bound), (dt, float(np.max(err / np.maximum(bound, 1e-300))))
        return
    u128 = u.astype(np.complex128)
    if kind == NONE:
        assert bits_equal(v, u)
        return
    ref = restate(u128, kind, thresh)
    if kind == HARD:
        # kept values are u itself, cut ones 0 (the kernel scales by 0, so a zero may carry u's sign); the kernel's |u|
        # is a hypot (<= 3 ulp) compared with the cut rounded to the precision: both outcomes are right within
        # 8 * 2^-p of the cut
        cut = math.sqrt(2 * thresh)
        band = np.abs(np.abs(u128) - cut) <= 8 * up * cut
        ok = np.where(band, (v == 0) | (v == u), v == ref.astype(npdt))
        assert np.all(ok), np.flatnonzero(~ok)[:8]
        return
    # complex soft: s = max(a - t, 0) / a with a = hypot (<= 3 ulp: 6 * 2^-p), subtraction and division 1 each, the
    # error of a again through the denominator 6, the product with u 1: <= 15 * 2^-p * |u| per component
    bound = 16 * up * np.abs(u128)
    assert np.all(np.abs(v.real - ref.real) <= bound) and np.all(np.abs(v.imag - ref.imag) <= bound)


def check_sums(r, dt, n):
    """sums against long double sums of the STORED xnew and the original xold"""
    _, _, _, _, cx, p = DT[dt]
    v, xo, s = r["v"], r["xold"], r["sums"]
    nr = 2 * n if cx else n
    if xo is None:
        assert s[0] == 0.0
    else:
        if cx:
            (vr, vi), (orr, oi) = ld(v), ld(xo)
            terms = (vr - orr) ** 2 + (vi - oi) ** 2
        else:
            terms = (ld(v) - ld(xo)) ** 2
        ref = float(np.sum(terms))
        # d = v - xold rounds once (relative 2^-p, 3 * 2^-p on d^2), the per-vector partial in the precision adds up
        # to 4 terms (4 * 2^-p), the float64 running sums (n + 64) * 2^-53
        assert abs(s[0] - ref) <= (8 * 2.0 ** -p + (nr + 64) * U64) * ref, (s[0], ref)
    if cx:
        vr, vi = ld(v)
        terms = np.sqrt(vr * vr + vi * vi)
    else:
        terms = np.abs(ld(v))
    ref = float(np.sum(terms))
    # real: |v| is exact, the per-vector partial adds up to 4 terms.  complex: |v| is a*s (hypot 6, product 1), the
    # stored components rounded once (1), 2-term partial (2): 10.  Then the float64 running sums.
    assert abs(s[1] - ref) <= (16 * 2.0 ** -p + (nr + 64) * U64) * ref, (s[1], ref)


def check_znew(r, dt, c):
    """znew = v + c (v - xold): fma(c, d, v) with d = v - xold in the precision.  Rounding c to the precision and d
    each cost 2^-p |c d|, the fma 2^-p |z|: |err| <= 2^-p (|z| + 2 |c d|), majorised by 2 * 2^-p (|z| + |c d|)"""
    if r["z"] is None:
        return
    _, _, _, _, cx, p = DT[dt]
    v, xo, z = r["v"], r["xold"], r["z"]
    if cx:
        pairs = [(ld(v)[0], ld(xo)[0], ld(z)[0]), (ld(v)[1], ld(xo)[1], ld(z)[1])]
    else:
        pairs = [(ld(v), ld(xo), ld(z))]
    for vv, oo, zz in pairs:
        cd = np.longdouble(c) * (vv - oo)
        ref = vv + cd
        assert np.all(np.abs(zz - ref) <= 2 * 2.0 ** -p * (np.abs(ref) + np.abs(cd)))


KIND_DT = [(k, d) for k in KINDS for d in DT if not (k == "half" and DT[d][4])]


@pytest.mark.parametrize("align", ["aligned", "shifted", "mixed"])
@pytest.mark.parametrize("cfg", list(CONFIGS))
@pytest.mark.parametrize("kind,dt", KIND_DT)
def test_sparse_update_edges(L, sms, kind, dt, cfg, align):
    rng = np.random.default_rng(zlib.crc32(f"{kind}{dt}{cfg}{align}".encode()))
    alpha, thresh, c = -0.25, 0.3, 0.375
    for n in vec_sizes(dt, sms):
        r = run_sparse(L, dt, KINDS[kind], cfg, n, rng, alpha, thresh, c, align)
        check_threshold(r, dt, KINDS[kind], thresh, alpha)
        check_sums(r, dt, n)
        check_znew(r, dt, c)


@pytest.mark.parametrize("align", ["aligned", "shifted"])
@pytest.mark.parametrize("kind,dt", KIND_DT)
def test_sparse_update_capped_grid(L, sms, kind, dt, align):
    rng = np.random.default_rng(7)
    n = big_size(dt, sms)
    alpha, thresh, c = 0.5, 0.3, -0.625
    r = run_sparse(L, dt, KINDS[kind], "distinct", n, rng, alpha, thresh, c, align)
    check_threshold(r, dt, KINDS[kind], thresh, alpha)
    check_sums(r, dt, n)
    check_znew(r, dt, c)


@pytest.mark.parametrize("dt", list(DT))
@pytest.mark.parametrize("kind", ["none", "soft"])
def test_sparse_update_general_alpha(L, sms, kind, dt):
    """alpha = 0.3 is not exact: the kernel's u is fma(alpha_p, g, base), the exact u rounded ONCE (alpha_p = alpha in
    the precision), so |u_kernel - u| <= 2^-p |u|.  NONE returns u; soft is 1-Lipschitz and rounds a - t once more
    (2^-p |v|): |v_kernel - soft(u)| <= 2^-p (|u| + |v|)."""
    npdt, rdt, _, _, cx, p = DT[dt]
    rng = np.random.default_rng(11)
    alpha, thresh = 0.3, 0.3
    for n in (769 * max(16 // np.dtype(rdt).itemsize // (2 if cx else 1), 1) + 1, big_size(dt, sms)):
        r = run_sparse(L, dt, KINDS[kind], "g_no_xold", n, rng, alpha, thresh, 0.0)
        b, g = r["base"].view(rdt), r["g"].view(rdt)
        ag = np.longdouble(float(rdt(alpha))) * ld(g)    # exact for float32 data, rounded at 2^-64 for float64
        u = ld(b) + ag
        v = ld(r["v"].view(rdt))
        if kind == "none":
            ref = u
        elif not cx:
            ref = np.sign(u) * np.maximum(np.abs(u) - np.longdouble(float(rdt(thresh))), 0)
        else:
            ur, ui = u[0::2], u[1::2]
            a = np.sqrt(ur * ur + ui * ui)
            s = np.maximum(a - np.longdouble(float(rdt(thresh))), 0) / np.where(a > 0, a, 1)
            ref = np.empty_like(u)
            ref[0::2], ref[1::2] = ur * s, ui * s
            u = np.repeat(a, 2)                   # complex soft: bound against |u| as in test_sparse_update_edges
        # complex soft: 15 * 2^-p |u| of test_sparse_update_edges plus 2^-p |u| from rounding u; (1 + 2^-20) takes
        # the second-order terms of using |ref| for |v|
        # the long double reference itself: alpha * g and the sum round at 2^-64, which matters where b + alpha g
        # cancels: 2^-62 |alpha g| covers both
        k = 1 if not cx or kind == "none" else 17
        bound = k * 2.0 ** -p * (np.abs(u) + np.abs(ref)) * (1 + 2.0 ** -20) + 2.0 ** -62 * np.abs(ag)
        assert np.all(np.abs(v - ref) <= bound), (dt, kind)
        check_sums(r, dt, n)


@pytest.mark.parametrize("kind,dt", KIND_DT)
@pytest.mark.parametrize("cfg", ["thresh", "ista", "distinct"])
def test_sparse_update_nan_propagates(L, sms, kind, dt, cfg):
    """a NaN in u gives NaN in xnew under every kind, as NumPy's thresholds do, and NaN sums"""
    rng = np.random.default_rng(3)
    _, rdt, _, _, cx, _ = DT[dt]
    for n in (vec_sizes(dt, sms)[-1], 5):
        at = sorted({0, n // 2, n - 2 if n > 2 else 0})
        r = run_sparse(L, dt, KINDS[kind], cfg, n, rng, -0.25, 0.3, 0.0, "aligned", nan_at=at)
        u = u_of(r, dt, -0.25)
        ref = restate(u, KINDS[kind], 0.3)
        got_nan = np.isnan(r["v"].view(rdt))
        ref_nan = np.isnan(ref.view(rdt)) if not cx else np.isnan(ref.astype(np.complex128).view(np.float64))
        assert ref_nan.any()
        assert np.array_equal(got_nan, ref_nan), (np.flatnonzero(got_nan != ref_nan)[:8])
        assert np.isnan(r["sums"][1])
        if r["xold"] is not None:
            assert np.isnan(r["sums"][0])


def _cut_points(x):
    """x and one ulp either side, at the precision of x"""
    return [np.nextafter(x, -np.inf), x, np.nextafter(x, np.inf)]


def _run_values(L, dt, kind, thresh, vals):
    vals = np.asarray(vals, dtype=DT[dt][0])
    b = Buf(vals, dt)
    sums = dbuf(2)
    L.check(L.lib.b2_sparse_update(L.ctx(), b.ptr, None, 0.0, None, thresh, kind, b.ptr, None, 0.0, sums.ptr,
                                   vals.size, DT[dt][3], L.stream()))
    torch.cuda.synchronize()
    b.check_guards()
    return vals, b.get()


THRESHOLDS = [0.3, 0.5, 1e-3, 2.7, 7e-5, 1.7]


def test_sparse_update_cut_boundaries_f64(L):
    """|u| at the soft, hard and half cuts and one ulp either side: zeroed exactly when the restatement zeros it.
    The half cut is pylops' (54 ** (1/3) / 4) t^(2/3); cbrt(54) is one ulp above 54 ** (1/3), so the points around
    the cbrt-based cut are included too."""
    for t in THRESHOLDS:
        half = (54 ** (1.0 / 3.0) / 4.0) * t ** (2.0 / 3.0)
        half_cbrt = (math.cbrt(54.0) / 4.0) * t ** (2.0 / 3.0)
        pts = {SOFT: _cut_points(np.float64(t)), HARD: _cut_points(np.sqrt(2 * np.float64(t))),
               HALF: _cut_points(np.float64(half)) + _cut_points(np.float64(half_cbrt))}
        for kind, p in pts.items():
            vals = np.array(p + [-x for x in p])
            vals, got = _run_values(L, "f64", kind, t, vals)
            ref = restate(vals, kind, t)
            assert np.array_equal(got == 0, ref == 0), (t, kind, vals[(got == 0) != (ref == 0)])
            if kind != HALF:
                assert bits_equal(got, ref)


def test_sparse_update_cut_boundaries_f32(L):
    """float32: the soft cut (|u| - t in float32, as NumPy with a Python-float t) and the hard cut (NumPy compares
    |u| with np.sqrt(2 t), a float64 scalar, so in float64) at the float32 neighbours of the cut.  For the half
    threshold NumPy's comparison depends on how t arrives: a Python float keeps it in float32, a NumPy float64 moves
    it to float64.  Within an ulp of the cut the reference has no single answer, so |u| is kept 2 and 3 ulp away."""
    rounded_up = 0
    for t in THRESHOLDS:
        hard = np.sqrt(2 * np.float64(t))
        rounded_up += float(np.float32(hard)) > hard
        half = np.float32((54 ** (1.0 / 3.0) / 4.0) * t ** (2.0 / 3.0))
        away = []
        for k in (2, 3):
            lo = hi = half
            for _ in range(k):
                lo, hi = np.nextafter(lo, np.float32(0)), np.nextafter(hi, np.float32(np.inf))
            away += [lo, hi]
        pts = {SOFT: _cut_points(np.float32(t)), HARD: _cut_points(np.float32(hard)), HALF: away}
        for kind, p in pts.items():
            vals = np.array(p + [-x for x in p], dtype=np.float32)
            vals, got = _run_values(L, "f32", kind, t, vals)
            ref = restate(vals, kind, t)
            assert np.array_equal(got == 0, ref == 0), (t, kind, vals[(got == 0) != (ref == 0)])
            if kind != HALF:
                assert bits_equal(got, ref)
    assert rounded_up, "no threshold whose float32 hard cut rounds up: the float64 comparison is not exercised"


def test_sparse_update_errors(L):
    x = torch.zeros(64, dtype=torch.float64, device="cuda")
    p = x.data_ptr()
    sums = dbuf(2)

    def call(kind=SOFT, thresh=0.1, dtype=1, xold=None, znew=None, n=8, base=p, xnew=p, s=sums.ptr):
        return L.lib.b2_sparse_update(L.ctx(), base, None, 1.0, xold, thresh, kind, xnew, znew, 0.5, s, n, dtype,
                                      L.stream())
    assert call(kind=4) == 2002
    assert call(kind=-1) == 2002
    assert call(thresh=-1e-300) == 2002
    assert call(znew=p) == 2002                       # znew needs xold
    assert call(kind=HALF, dtype=2) == 2005
    assert call(kind=HALF, dtype=3) == 2005
    assert call(dtype=4) == 2001
    assert call(dtype=5) == 2001
    assert L.lib.b2_sparse_update(None, p, None, 1.0, None, 0.1, SOFT, p, None, 0.0, None, 8, 1, L.stream()) == 2002
    torch.cuda.synchronize()
    assert np.all(sums.get() == SENT)                 # nothing written on an error
    # a rank owning no elements: sums zeroed, array pointers may be null
    assert call(n=0, base=None, xnew=None) == 0
    assert call(n=0, base=None, xnew=None, s=None) == 0
    torch.cuda.synchronize()
    assert np.array_equal(sums.get(), [0.0, 0.0])
    sums.check_guards()


# ======================================================================================================================
# b2_lincomb_dev / b2_lincomb_dev_norm2
# ======================================================================================================================
def lincomb_case(L, dt, n, a, a_scale, b, b_scale, alias, align, fused, rng):
    """out = (a_scale a) x + (b_scale b) y with device scalars a, b (None -> 1); alias in (None, 'x', 'y')"""
    code = DT[dt][3]
    x, y, o = rnd(rng, n, dt), rnd(rng, n, dt), rnd(rng, n, dt)
    sh = shift_of(dt) if align != "aligned" else 0
    bx = Buf(x, dt, sh)
    by = Buf(y, dt, sh if align == "shifted" else 0)
    bo = Buf(o, dt, sh if align == "shifted" else 0)
    out = {None: bo, "x": bx, "y": by}[alias]
    sc = Buf(np.array([SENT if a is None else a, SENT if b is None else b]), "f64")
    ap = sc.ptr if a is not None else None
    bp = sc.ptr + 8 if b is not None else None
    nrm = dbuf(2)
    if fused:
        rc = L.lib.b2_lincomb_dev_norm2(L.ctx(), out.ptr, ap, a_scale, bx.ptr, bp, b_scale, by.ptr, n, code, nrm.ptr,
                                        L.stream())
    else:
        rc = L.lib.b2_lincomb_dev(L.ctx(), out.ptr, ap, a_scale, bx.ptr, bp, b_scale, by.ptr, n, code, L.stream())
    L.check(rc, "lincomb")
    torch.cuda.synchronize()
    for bb in (bx, by, bo, nrm):
        bb.check_guards()
    return x, y, out.get(), nrm.get()


LC_SCALARS = [(None, 1.0, None, -1.0), (0.75, 2.0, None, 1.0), (None, -0.5, 1.5, 0.25), (-3.0, 0.125, 0.625, -2.0)]


@pytest.mark.parametrize("align", ["aligned", "shifted", "mixed"])
@pytest.mark.parametrize("alias", [None, "x", "y"])
@pytest.mark.parametrize("dt", list(DT))
def test_lincomb_dev_and_norm2(L, sms, dt, alias, align):
    """coefficients exact in every precision: with an fma, a x rounds once and b y twice; without, each twice:
    |err| <= 2 * 2^-p (|a x| + |b y|) either way.  norm2[0] is the float64 sum of squares of the STORED output
    ((n + 1) * 2^-53 relative: fma per term, n additions); norm2[1] is 0 for complex dtypes and untouched for real"""
    _, rdt, _, _, cx, p = DT[dt]
    rng = np.random.default_rng(5)
    sizes = vec_sizes(dt, sms) + [big_size(dt, sms) // 3]
    for n in sizes:
        for a, asc, b, bsc in (LC_SCALARS if n < sizes[-1] else LC_SCALARS[-1:]):
            outs = []
            for fused in (False, True):
                x, y, got, nrm = lincomb_case(L, dt, n, a, asc, b, bsc, alias, align, fused, np.random.default_rng(n))
                ca = asc * (1.0 if a is None else a)
                cb = bsc * (1.0 if b is None else b)
                xr, yr, gr = ld(x.view(rdt)), ld(y.view(rdt)), ld(got.view(rdt))
                ax, by = np.longdouble(ca) * xr, np.longdouble(cb) * yr
                assert np.all(np.abs(gr - (ax + by)) <= 2 * 2.0 ** -p * (np.abs(ax) + np.abs(by))), (n, a, b, fused)
                if fused:
                    ref = float(np.sum(gr * gr))
                    assert abs(nrm[0] - ref) <= (gr.size + 1) * U64 * ref
                    assert nrm[1] == (0.0 if cx else SENT)
                else:
                    assert np.all(nrm == SENT)
                outs.append(got)
            assert bits_equal(outs[0], outs[1]), (n, a, b)


@pytest.mark.parametrize("dt", ["f32", "c64"])
def test_lincomb_dev_scale_rounds_once(L, sms, dt):
    """a = a_scale * (*a_dev) in float64, rounded to the precision once (the header's contract): with b = 0 the
    output is fl(a) * x exactly.  a_scale = 0.1 is not a float32, so rounding a_scale first gives other bits; both
    entry points must write the same ones"""
    _, rdt, _, _, _, _ = DT[dt]
    n = vec_sizes(dt, sms)[-1]
    for adev in (0.3, -1.2, 2.4):       # values where rounding a_scale first changes fl(a)
        outs = []
        for fused in (False, True):
            x, y, got, _ = lincomb_case(L, dt, n, adev, 0.1, None, 0.0, None, "aligned", fused,
                                        np.random.default_rng(1))
            a32 = rdt(np.float64(0.1) * np.float64(adev))
            assert bits_equal(got.view(rdt), a32 * x.view(rdt)), (adev, fused)
            outs.append(got)
        assert bits_equal(outs[0], outs[1])
        # with b y in play as well (CGLS's c = r + b c): the same bits from both entry points
        outs = [lincomb_case(L, dt, n, adev, 0.1, 0.3, -0.7, "y", "aligned", f, np.random.default_rng(2))[2]
                for f in (False, True)]
        assert bits_equal(outs[0], outs[1])


def test_lincomb_dev_zero_and_errors(L):
    nrm = dbuf(2)
    x = torch.zeros(8, dtype=torch.float64, device="cuda")
    for code, expect in ((0, [0.0, SENT]), (2, [0.0, 0.0])):
        nrm = dbuf(2)
        assert L.lib.b2_lincomb_dev_norm2(L.ctx(), None, None, 1.0, None, None, 1.0, None, 0, code, nrm.ptr,
                                          L.stream()) == 0
        torch.cuda.synchronize()
        assert np.array_equal(nrm.get(), expect)
        nrm.check_guards()
    p = x.data_ptr()
    assert L.lib.b2_lincomb_dev(L.ctx(), p, None, 1.0, p, None, 1.0, p, 8, 4, L.stream()) == 2001
    assert L.lib.b2_lincomb_dev_norm2(L.ctx(), p, None, 1.0, p, None, 1.0, p, 8, 4, nrm.ptr, L.stream()) == 2001
    assert L.lib.b2_lincomb_dev_norm2(L.ctx(), p, None, 1.0, p, None, 1.0, None, 8, 1, nrm.ptr, L.stream()) == 2002
    assert L.lib.b2_lincomb_dev_norm2(L.ctx(), p, None, 1.0, p, None, 1.0, p, 8, 1, None, L.stream()) == 2002


# ======================================================================================================================
# reductions
# ======================================================================================================================
def dot_ref(x, y, conj):
    """long double (re, im) and the sums of |terms| the bounds scale with"""
    if np.iscomplexobj(x):
        (xr, xi), (yr, yi) = ld(x), ld(y)
        if conj:
            xi = -xi
        re = np.sum(xr * yr) - np.sum(xi * yi)
        im = np.sum(xr * yi) + np.sum(xi * yr)
        return (float(re), float(im)), (float(np.sum(np.abs(xr * yr)) + np.sum(np.abs(xi * yi))),
                                         float(np.sum(np.abs(xr * yi)) + np.sum(np.abs(xi * yr))))
    p = ld(x) * ld(y)
    return (float(np.sum(p)), 0.0), (float(np.sum(np.abs(p))), 0.0)


@pytest.mark.parametrize("conj", [0, 1])
@pytest.mark.parametrize("dt", list(DT))
def test_dot_multi(L, sms, dt, conj):
    """k = 1..4 distinct (x_j, y_j) pairs.  Products and sums in float64: a real term is one fma, a complex one
    a*c - b*d (2 roundings); (n + 4) * 2^-53 * sum|terms| bounds the float64 accumulation of either"""
    _, rdt, _, code, cx, _ = DT[dt]
    rng = np.random.default_rng(17)
    per = 2 if cx else 1
    for n in (1, 3, 1025, 3 * 256 * red_cap(sms) + 7):
        for k in (1, 2, 3, 4):
            xs = [rnd(rng, n, dt) for _ in range(k)]
            ys = [rnd(rng, n, dt) for _ in range(k)]
            bx = [Buf(a, dt) for a in xs]
            by = [Buf(a, dt, shift_of(dt) if j % 2 else 0) for j, a in enumerate(ys)]
            out = dbuf(2 * k)
            px = (C.c_void_p * k)(*[b.ptr for b in bx])
            py = (C.c_void_p * k)(*[b.ptr for b in by])
            L.check(L.lib.b2_dot_multi(L.ctx(), k, px, py, n, code, conj, out.ptr, L.stream()))
            torch.cuda.synchronize()
            out.check_guards()
            got = out.get()
            for j in range(k):
                (re, im), (sre, sim) = dot_ref(xs[j], ys[j], conj)
                g = got[per * j:per * j + per]
                assert abs(g[0] - re) <= (n + 4) * U64 * sre, (n, k, j)
                if cx:
                    assert abs(g[1] - im) <= (n + 4) * U64 * sim, (n, k, j)
            if not cx:
                assert np.all(got[k:] == SENT)      # real dtypes: k doubles, nothing behind them


def test_dot_multi_empty_and_errors(L):
    for code, cx in ((0, False), (1, False), (2, True), (3, True)):
        for k in (1, 2, 3, 4):
            out = dbuf(8)
            nulls = (C.c_void_p * k)()
            assert L.lib.b2_dot_multi(L.ctx(), k, nulls, nulls, 0, code, 1, out.ptr, L.stream()) == 0
            torch.cuda.synchronize()
            got = out.get()
            m = 2 * k if cx else k
            assert np.all(got[:m] == 0.0) and np.all(got[m:] == SENT), (code, k)
            out.check_guards()
    x = torch.zeros(8, dtype=torch.float64, device="cuda")
    ptrs = (C.c_void_p * 5)(*([x.data_ptr()] * 5))
    out = dbuf(10)
    for k in (0, 5, -1):
        assert L.lib.b2_dot_multi(L.ctx(), k, ptrs, ptrs, 8, 1, 0, out.ptr, L.stream()) == 2002
    torch.cuda.synchronize()
    assert np.all(out.get() == SENT)


def norm_ref(a, kind, p):
    """long double reference of the local norm partial over |x| (float64 magnitudes); returns (value, scale)"""
    if kind == NRM_COUNT:
        return float(np.count_nonzero(a)), 0.0
    if kind == NRM_MAX:
        return (float(np.max(a)) if a.size else 0.0), 0.0
    if kind == NRM_MIN:
        return (float(np.min(a)) if a.size else np.inf), 0.0
    t = {NRM_ABS: ld(a), NRM_SQ: ld(a) ** 2, NRM_POW: ld(a) ** np.longdouble(p)}[kind]
    return float(np.sum(t)), float(np.sum(np.abs(t)))


def abs64(x):
    return np.abs(x.astype(np.complex128 if np.iscomplexobj(x) else np.float64))


def check_norm(got, ref, scale, kind, n, p, cx):
    """sums: (n + 8 + 8p) * 2^-53 * sum|terms| -- n float64 additions, pow <= 2 ulp, hypot <= 2 ulp raised to p;
    max / min: exact for real data, hypot's 4 * 2^-53 for complex"""
    if np.isnan(ref):
        assert np.isnan(got), (kind, got)
    elif kind == NRM_COUNT:
        assert got == ref
    elif kind in (NRM_MAX, NRM_MIN):
        assert (got == ref) if not cx or not np.isfinite(ref) else abs(got - ref) <= 4 * U64 * ref, (kind, got, ref)
    else:
        assert abs(got - ref) <= (n + 8 + 8 * p) * U64 * scale, (kind, p, got, ref)


NORM_KINDS = [(NRM_COUNT, 0.0), (NRM_ABS, 0.0), (NRM_SQ, 0.0), (NRM_MAX, 0.0), (NRM_MIN, 0.0),
              (NRM_POW, 0.5), (NRM_POW, 1.5), (NRM_POW, 3.0)]


@pytest.mark.parametrize("nan", [False, True])
@pytest.mark.parametrize("dt", list(DT))
def test_norm_partial(L, sms, dt, nan):
    """every kind, vector-path edges and a capped grid; a NaN anywhere gives NaN, as np.linalg.norm and np.max do,
    and is counted by count_nonzero"""
    cx = DT[dt][4]
    rng = np.random.default_rng(23)
    for n in vec_sizes(dt, sms) + [big_size(dt, sms) // 2]:
        x = rnd(rng, n, dt, scale=0.5)
        if nan:
            x[rng.integers(0, n)] = np.nan
            x[n - 1] = np.nan * (1 + 1j) if cx else np.nan
        for shift in (0, shift_of(dt)):
            b = Buf(x, dt, shift)
            a = abs64(x)
            for kind, p in NORM_KINDS:
                out = dbuf(1)
                L.check(L.lib.b2_norm_partial(L.ctx(), b.ptr, n, DT[dt][3], kind, p, out.ptr, L.stream()))
                torch.cuda.synchronize()
                out.check_guards()
                ref, scale = norm_ref(a, kind, p)
                check_norm(out.get()[0], ref, scale, kind, n, p, cx)


def axis_ref(x, shape, kind, p):
    a = abs64(x).reshape(shape)
    if kind == NRM_COUNT:
        return np.count_nonzero(a, axis=1).astype(np.float64), None
    if kind == NRM_MAX:
        return (np.max(a, axis=1) if shape[1] else np.zeros((shape[0], shape[2]))), None
    if kind == NRM_MIN:
        return (np.min(a, axis=1) if shape[1] else np.full((shape[0], shape[2]), np.inf)), None
    t = {NRM_ABS: ld(a), NRM_SQ: ld(a) ** 2, NRM_POW: ld(a) ** np.longdouble(p)}[kind]
    return np.sum(t, axis=1).astype(np.float64), np.sum(np.abs(t), axis=1).astype(np.float64)


def axis_shapes(sms):
    cap16 = sms * 16
    return [(5, 63, 1), (5, 64, 1), (3, 200, 1), (4, 17, 2), (3, 9, 3), (2, 70, 33), (1, 1, 1),
            (cap16 * 8 + 3, 64, 1),            # warp-per-row kernel past its grid cap (8 warps per block)
            (cap16 * 256 * 2 // 3 + 5, 3, 3),  # thread-per-output kernel past its grid cap
            (7, 0, 5), (3, 0, 1)]              # an empty axis: the identity of each kind


@pytest.mark.parametrize("nan", [False, True])
@pytest.mark.parametrize("dt", list(DT))
def test_norm_axis(L, sms, dt, nan):
    cx = DT[dt][4]
    rng = np.random.default_rng(29)
    for shape in axis_shapes(sms):
        n = int(np.prod(shape))
        x = rnd(rng, n, dt, scale=0.5)
        if nan and n:
            x[rng.integers(0, n, size=3)] = np.nan
        b = Buf(x, dt)
        nout = shape[0] * shape[2]
        for kind, p in NORM_KINDS:
            out = dbuf(nout)
            L.check(L.lib.b2_norm_axis(L.ctx(), b.ptr if n else None, *shape, DT[dt][3], kind, p, out.ptr,
                                       L.stream()))
            torch.cuda.synchronize()
            out.check_guards()
            got = out.get()
            ref, scale = axis_ref(x, shape, kind, p)
            ref = ref.ravel()
            if scale is None and np.isinf(ref).any():   # MIN over an empty axis: +inf, compared exactly
                ok = got == ref
            elif scale is None:
                if kind == NRM_COUNT or not cx:
                    ok = (got == ref) | (np.isnan(got) & np.isnan(ref))
                else:
                    ok = (np.abs(got - ref) <= 4 * U64 * ref) | (got == ref) | (np.isnan(got) & np.isnan(ref))
            else:
                # n_axis float64 additions, pow / hypot <= 2 ulp each (raised to p): (n_axis + 8 + 8p) * 2^-53
                bound = (shape[1] + 8 + 8 * p) * U64 * scale.ravel()
                ok = (np.abs(got - ref) <= bound) | (np.isnan(got) & np.isnan(ref))
            assert np.all(ok), (shape, kind, p, np.flatnonzero(~ok)[:5], got[~ok][:5], ref[~ok][:5])


def test_norm_axis_errors(L):
    out = dbuf(4)
    x = torch.zeros(8, dtype=torch.float64, device="cuda")
    assert L.lib.b2_norm_axis(L.ctx(), x.data_ptr(), 2, 2, 2, 1, 6, 0.0, out.ptr, L.stream()) == 2002
    assert L.lib.b2_norm_axis(L.ctx(), x.data_ptr(), 2, 2, 2, 1, -1, 0.0, out.ptr, L.stream()) == 2002
    assert L.lib.b2_norm_axis(L.ctx(), None, 2, 2, 2, 1, 2, 0.0, out.ptr, L.stream()) == 2002
    assert L.lib.b2_norm_axis(L.ctx(), x.data_ptr(), 2, 2, 2, 4, 2, 0.0, out.ptr, L.stream()) == 2001
    assert L.lib.b2_norm_axis(L.ctx(), x.data_ptr(), 0, 2, 2, 1, 2, 0.0, out.ptr, L.stream()) == 0
    torch.cuda.synchronize()
    assert np.all(out.get() == SENT)


def test_reductions_share_workspace_deterministically(L, sms):
    """calls with different grids back to back on one b2_ctx return the bits each returns alone, and a repeated
    call the same bits: the last-CTA ticket is reset by every call, b2_sparse_update without sums and
    b2_lsqr_update included"""
    rng = np.random.default_rng(31)
    big = 9 * 256 * red_cap(sms) * 2 + 3
    xb = Buf(rnd(rng, big, "f64"), "f64")
    xs = Buf(rnd(rng, 1000, "f32"), "f32")
    ys = Buf(rnd(rng, 1000, "f32"), "f32")
    xm = Buf(rnd(rng, 300_001, "c64"), "c64")
    ym = Buf(rnd(rng, 300_001, "c64"), "c64")
    xu = Buf(rnd(rng, 700_003, "f32"), "f32")
    ou = Buf(np.zeros(700_003, np.float32), "f32")
    xc = Buf(rnd(rng, 50_001, "c128"), "c128")
    # the LSQR update with t1 = t2 = 0 and inv_alfa = 1 keeps x and sets w = v; w starts equal to v, so every call
    # returns the same ||dk||^2
    lv = rnd(rng, 200_003, "c64")
    lx, lw, lvv, lvar = (Buf(a, "c64") for a in (rnd(rng, 200_003, "c64"), lv, lv, rnd(rng, 200_003, "c64")))
    coef = Buf(np.array([0.0, 0.0, 0.75, 1.0]), "f64")
    outs = [dbuf(2) for _ in range(8)]
    s = L.stream()
    calls = [
        lambda: L.lib.b2_norm_partial(L.ctx(), xb.ptr, big, 1, NRM_SQ, 0.0, outs[0].ptr, s),
        lambda: L.lib.b2_dot_multi(L.ctx(), 1, (C.c_void_p * 1)(xs.ptr), (C.c_void_p * 1)(ys.ptr), 1000, 0, 0,
                                   outs[1].ptr, s),
        lambda: L.lib.b2_sparse_update(L.ctx(), xu.ptr, None, 0.0, None, 0.1, SOFT, ou.ptr, None, 0.0, None,
                                       700_003, 0, s),
        lambda: L.lib.b2_dot(L.ctx(), xm.ptr, ym.ptr, 300_001, 2, 1, outs[2].ptr, s),
        lambda: L.lib.b2_sparse_update(L.ctx(), xu.ptr, None, 0.0, xu.ptr, 0.2, HARD, ou.ptr, None, 0.0,
                                       outs[3].ptr, 700_003, 0, s),
        lambda: L.lib.b2_lincomb_dev_norm2(L.ctx(), ou.ptr, None, 0.5, xu.ptr, None, 0.25, xu.ptr, 700_003, 0,
                                           outs[4].ptr, s),
        lambda: L.lib.b2_lsqr_update(L.ctx(), lx.ptr, lw.ptr, lvv.ptr, lvar.ptr, 200_003, 2, coef.ptr, None,
                                     outs[7].ptr, s),
        lambda: L.lib.b2_norm_partial(L.ctx(), xc.ptr, 50_001, 3, NRM_MAX, 0.0, outs[5].ptr, s),
        lambda: L.lib.b2_norm_partial(L.ctx(), xm.ptr, 300_001, 2, NRM_POW, 1.5, outs[6].ptr, s),
    ]
    alone = []
    for f in calls:
        got = []
        for _ in range(2):
            L.check(f())
            torch.cuda.synchronize()
            got.append(np.concatenate([o.get() for o in outs]))
        assert bits_equal(got[0], got[1])
        alone.append(got[0])
    for o in outs:
        o.t.fill_(SENT)
    for f in calls:
        L.check(f())
    torch.cuda.synchronize()
    seq = np.concatenate([o.get() for o in outs])
    assert bits_equal(seq, alone[-1])
    for o in outs:
        o.check_guards()


# ======================================================================================================================
# b2_scalar_div / b2_history_push
# ======================================================================================================================
def test_scalar_div(L):
    """out = |num / (den1 + alpha den2)|.  Dyadic operands keep the denominator exact, so the correctly rounded
    division gives NumPy's bits; zero and 0/0 denominators give inf and nan, as the NumPy scalars do"""
    cases = [(3.0, 0.75, None, 0.0), (-5.0, 0.5, 0.25, 2.0), (1.0, 3.0, 1.5, -2.0), (1.0, 0.0, None, 0.0),
             (-1.0, -0.0, None, 0.0), (2.0, 1.0, 0.5, -2.0), (0.0, 0.0, None, 0.0), (0.0, 1.0, 0.5, -2.0),
             (0.1, 0.3, 0.7, 1e-3)]
    with np.errstate(divide="ignore", invalid="ignore"):
        for num, d1, d2, alpha in cases:
            for alias in (False, True):
                v = Buf(np.array([num, d1, SENT if d2 is None else d2, SENT]), "f64")
                optr = v.ptr if alias else v.ptr + 24
                L.check(L.lib.b2_scalar_div(optr, v.ptr, v.ptr + 8, v.ptr + 16 if d2 is not None else None, alpha,
                                            L.stream()))
                torch.cuda.synchronize()
                v.check_guards()
                got = v.get()[0 if alias else 3]
                den = np.float64(d1) + (np.float64(alpha) * np.float64(d2) if d2 is not None else 0.0)
                ref = np.abs(np.float64(num) / den)
                if num == 0.1:                    # general operands: den rounds (or fuses) once more
                    assert abs(got - ref) <= 4 * U64 * ref
                else:
                    assert bits_equal(np.array([got]), np.array([ref])) or (np.isnan(got) and np.isnan(ref)), \
                        (num, d1, d2, alpha, got, ref)


def push(L, src, nvals, stride, hist, it, cap, cdst=None, csrc=None):
    return L.lib.b2_history_push(src, nvals, stride, hist, it, cap, cdst, csrc, L.stream())


@pytest.mark.parametrize("nvals,stride", [(1, 1), (3, 2), (16, 1), (16, 3)])
def test_history_push(L, nvals, stride):
    cap = 4
    srcv = np.arange(1, nvals * stride + 1, dtype=np.float64) * (-1.0) ** np.arange(nvals * stride)
    src = Buf(srcv, "f64")
    hist = dbuf(cap * nvals)
    scal = Buf(np.array([SENT, 42.5]), "f64")              # [copy_dst, copy_src]
    for start in (0, cap - 1, cap, cap + 5, 2 ** 32 + 1):
        hist.t.fill_(SENT)
        scal.t[scal.off] = SENT
        it = torch.tensor([start], dtype=torch.int64, device="cuda")
        L.check(push(L, src.ptr, nvals, stride, hist.ptr, it.data_ptr(), cap, scal.ptr, scal.ptr + 8))
        torch.cuda.synchronize()
        hist.check_guards()
        h = hist.get().reshape(cap, nvals)
        expect = np.full((cap, nvals), SENT)
        if start < cap:                                    # a 32-bit counter would wrap 2^32 + 1 to 1 and write
            expect[start] = np.abs(srcv[::stride][:nvals])
        assert np.array_equal(h, expect), start
        assert it.item() == start + 1                     # the counter keeps counting past cap, in 64 bits
        assert scal.get()[0] == 42.5                      # and the copy still happens


def test_history_push_rejects(L):
    src = Buf(np.ones(32), "f64")
    hist = dbuf(64)
    it = torch.zeros(1, dtype=torch.int64, device="cuda")
    s, h, i = src.ptr, hist.ptr, it.data_ptr()
    assert push(L, None, 1, 1, h, i, 4) == 2002
    assert push(L, s, 1, 1, None, i, 4) == 2002
    assert push(L, s, 1, 1, h, None, 4) == 2002
    assert push(L, s, 0, 1, h, i, 4) == 2002
    assert push(L, s, 17, 1, h, i, 4) == 2002
    assert push(L, s, 1, 0, h, i, 4) == 2002
    assert push(L, s, 1, 1, h, i, 4, cdst=s) == 2002
    assert push(L, s, 1, 1, h, i, 4, csrc=s) == 2002
    torch.cuda.synchronize()
    assert it.item() == 0 and np.all(hist.get() == SENT)
