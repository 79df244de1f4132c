"""LSQR's scalar recurrence on the host, in float64 NumPy: the statement of ``b2_lsqr_scalars`` (csrc/lsqr.cu) on the
same state layout.  The definition is ``scipy.sparse.linalg.lsqr`` (Paige & Saunders 1982): given the same reductions,
this module follows scipy's loop operation for operation.  NumPy only, so the fixture generator and the CPU tests load
it without the CUDA library; LSQR's generic (stacked-array) path runs it."""
import numpy as np

# offsets in the device state of b2_lsqr_scalars / b2_lsqr_update (include/b200lops.h, B2_LSQR_*)
(_BB, _DD, _AA, _ALFA, _BETA, _RHOBAR, _PHIBAR, _ANORM, _DDNORM, _RES2, _XXNORM, _Z, _CS2, _SN2, _ITN, _ISTOP,
 _PENDING, _STOPPED) = (0, 2, 4) + tuple(range(8, 23))
_DAMP, _DAMPSQ, _ATOL, _BTOL, _CTOL, _BNORM, _ITER_LIM = range(24, 31)
_R1NORM, _R2NORM, _ACOND, _ARNORM, _XNORM, _TEST1, _TEST2, _TT1, _RTOL = range(32, 41)
_CUB, _CVA, _CVB = 42, 43, 44
_T1, _T2, _INV_RHO, _INV_ALFA = 48, 49, 50, 51
_SCRATCH, _NSTATE, _NHIST = 52, 56, 9
_EPS = float(np.finfo(np.float64).eps)


def _sym_ortho(a: float, b: float):
    """scipy.sparse.linalg._isolve.lsqr._sym_ortho"""
    sign = lambda t: float(np.sign(t))                               # noqa: E731
    if b == 0:
        return sign(a), 0.0, abs(a)
    if a == 0:
        return 0.0, sign(b), abs(b)
    if abs(b) > abs(a):
        tau = a / b
        s = sign(b) / np.sqrt(1 + tau * tau)
        return s * tau, s, b / s
    tau = b / a
    c = sign(a) / np.sqrt(1 + tau * tau)
    return c, c * tau, a / c


def lsqr_scalars_host(s: np.ndarray, phase: int):
    """float64 NumPy statement of ``b2_lsqr_scalars`` on the same state layout (csrc/lsqr.cu writes out the
    sequence): scipy's lsqr loop body, operation for operation.  Returns the history row a finished iteration
    writes, else None.  The generic (stacked-array) path runs it, and the kernel is tested against it bit for bit."""
    s = s.view(np.float64)
    f = lambda i: float(s[i])                                        # noqa: E731
    if f(_STOPPED) != 0.0:
        return None
    if phase != 1:
        row = None
        if f(_PENDING) != 0.0:
            s[_DDNORM] = f(_DDNORM) + f(_DD)
            s[_DD] = 0.0
            anorm = f(_ANORM)
            acond = anorm * np.sqrt(f(_DDNORM))
            test1, test2, tt1 = f(_TEST1), f(_TEST2), f(_TT1)
            test3 = 1 / (acond + _EPS)
            istop = 0.0
            if f(_ITN) >= f(_ITER_LIM):
                istop = 7.0
            if 1 + test3 <= 1:
                istop = 6.0
            if 1 + test2 <= 1:
                istop = 5.0
            if 1 + tt1 <= 1:
                istop = 4.0
            if test3 <= f(_CTOL):
                istop = 3.0
            if test2 <= f(_ATOL):
                istop = 2.0
            if test1 <= f(_RTOL):
                istop = 1.0
            s[_ACOND], s[_ISTOP], s[_PENDING] = acond, istop, 0.0
            if istop != 0.0:
                s[_STOPPED] = 1.0
            row = np.array([f(_R1NORM), f(_R2NORM), anorm, acond, f(_ARNORM), f(_XNORM), test1, test2, istop])
        if phase == 2 or f(_STOPPED) != 0.0:
            return row
        beta = float(np.sqrt(f(_BB)))
        s[_BETA] = beta
        if beta > 0:
            s[_CVA], s[_CVB] = 1 / beta, beta * f(_INV_ALFA)
        else:
            s[_CVA], s[_CVB] = 0.0, -1.0
        return row
    damp, dampsq, beta = f(_DAMP), f(_DAMPSQ), f(_BETA)
    s[_ITN] = f(_ITN) + 1
    alfa, anorm = f(_ALFA), f(_ANORM)
    if beta > 0:
        anorm = float(np.sqrt(anorm * anorm + alfa * alfa + beta * beta + dampsq))
        alfa = float(np.sqrt(f(_AA)))
        s[_INV_ALFA] = 1 / alfa if alfa > 0 else 1.0
    rhobar, phibar = f(_RHOBAR), f(_PHIBAR)
    if damp > 0:
        rhobar1 = float(np.sqrt(rhobar * rhobar + dampsq))
        cs1, sn1 = rhobar / rhobar1, damp / rhobar1
        psi = sn1 * phibar
        phibar = cs1 * phibar
    else:
        rhobar1, psi = rhobar, 0.0
    cs, sn, rho = _sym_ortho(rhobar1, beta)
    theta = sn * alfa
    rhobar = -cs * alfa
    phi = cs * phibar
    phibar = sn * phibar
    tau = sn * phi
    s[_T1], s[_T2], s[_INV_RHO] = phi / rho, -theta / rho, 1 / rho
    delta, gambar = f(_SN2) * rho, -f(_CS2) * rho
    rhs = phi - delta * f(_Z)
    zbar = rhs / gambar
    xxnorm = f(_XXNORM)
    xnorm = float(np.sqrt(xxnorm + zbar * zbar))
    gamma = float(np.sqrt(gambar * gambar + theta * theta))
    s[_CS2], s[_SN2] = gambar / gamma, theta / gamma
    z = rhs / gamma
    xxnorm = xxnorm + z * z
    s[_Z], s[_XXNORM] = z, xxnorm
    res1 = phibar * phibar
    res2 = f(_RES2) + psi * psi
    rnorm = float(np.sqrt(res1 + res2))
    arnorm = alfa * abs(tau)
    r1norm = rnorm
    if damp > 0:
        r1sq = rnorm * rnorm - dampsq * xxnorm
        r1norm = float(np.sqrt(abs(r1sq)))
        if r1sq < 0:
            r1norm = -r1norm
    bnorm = f(_BNORM)
    test1 = rnorm / bnorm
    s[_TEST1] = test1
    s[_TEST2] = arnorm / (anorm * rnorm + _EPS)
    s[_TT1] = test1 / (1 + anorm * xnorm / bnorm)
    s[_RTOL] = f(_BTOL) + f(_ATOL) * anorm * xnorm / bnorm
    s[_ALFA], s[_ANORM], s[_RHOBAR], s[_PHIBAR] = alfa, anorm, rhobar, phibar
    s[_RES2], s[_XNORM], s[_ARNORM], s[_R1NORM], s[_R2NORM] = res2, xnorm, arnorm, r1norm, rnorm
    s[_PENDING] = 1.0
    s[_CUB] = alfa * (1 / beta if beta > 0 else 1.0)
    return None
