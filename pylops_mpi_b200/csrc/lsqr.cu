// LSQR on the device (optimization/cls_basic.py LSQR): the scalar recurrence of scipy.sparse.linalg.lsqr
// (Paige & Saunders 1982, scipy 1.x _isolve/lsqr.py) in one thread, and the fused model-side update.
//
// The iteration keeps u and v UNNORMALISED: U = u' (norm beta) and V = v' (norm alfa), scipy's vectors before its
// `u = (1/beta) u` / `v = (1/alfa) v` passes.  The normalisations are folded into the coefficients of the next
// combination, so one iteration is
//   U <- inv_alfa A V - (alfa inv_beta) U          b2_lincomb_dev_norm2 -> BB = |U|^2    (all-reduced with DD)
//   phase 0: finish the previous iteration (DD), beta = sqrt(BB), v-step coefficients
//   V <- inv_beta A^H U - (beta inv_alfa) V        b2_lincomb_dev_norm2 -> AA = |V|^2    (all-reduced)
//   phase 1: alfa = sqrt(AA) and the rest of scipy's loop body up to its stopping tests
//   x += t1 w;  dk = inv_rho w;  var += dk^2;  DD = |dk|^2;  w = inv_alfa V + t2 w         b2_lsqr_update
// acond (and so test3 and istop) needs ddnorm after the update, so the tests of iteration k are finished by phase 0
// of iteration k + 1 (or phase 2 after the last one): DD rides in the all-reduce of BB and an iteration costs two
// scalar collectives, as CGLS.  Once an iteration stops, `stopped` is set and every later phase and update is a
// no-op: the iterations that follow in a replayed block change neither x, w, var nor the scalars.
//
// Scalar arithmetic: scipy's operations in scipy's order, each an explicit round-to-nearest intrinsic (no
// contraction), `a**2` as a * a (CPython's pow(a, 2.0) is correctly rounded, so it is the same double).  Given the
// same BB / AA / DD inputs the state equals a float64 NumPy transcription of the loop bit for bit
// (tests/test_lsqr.py).  Per iteration, with the names of lsqr.py:
//   phase 1:  itn += 1
//             if beta > 0:  anorm = sqrt(anorm*anorm + alfa*alfa + beta*beta + dampsq);  alfa = sqrt(AA)
//             if damp > 0:  rhobar1 = sqrt(rhobar*rhobar + dampsq); cs1 = rhobar/rhobar1; sn1 = damp/rhobar1
//                           psi = sn1*phibar; phibar = cs1*phibar
//             else:         rhobar1 = rhobar; psi = 0
//             cs, sn, rho = _sym_ortho(rhobar1, beta)
//             theta = sn*alfa; rhobar = -cs*alfa; phi = cs*phibar; phibar = sn*phibar; tau = sn*phi
//             t1 = phi/rho; t2 = -theta/rho; inv_rho = 1/rho
//             delta = sn2*rho; gambar = -cs2*rho; rhs = phi - delta*z; zbar = rhs/gambar
//             xnorm = sqrt(xxnorm + zbar*zbar); gamma = sqrt(gambar*gambar + theta*theta)
//             cs2 = gambar/gamma; sn2 = theta/gamma; z = rhs/gamma; xxnorm = xxnorm + z*z
//             res1 = phibar*phibar; res2 = res2 + psi*psi; rnorm = sqrt(res1 + res2); arnorm = alfa*|tau|
//             damp > 0: r1sq = rnorm*rnorm - dampsq*xxnorm; r1norm = +-sqrt(|r1sq|) (sign of r1sq); else rnorm
//             r2norm = rnorm; test1 = rnorm/bnorm; test2 = arnorm/(anorm*rnorm + eps)
//             tt1 = test1/(1 + anorm*xnorm/bnorm); rtol = btol + atol*anorm*xnorm/bnorm    (left to right)
//   finish:   ddnorm = ddnorm + DD; acond = anorm*sqrt(ddnorm); test3 = 1/(acond + eps)
//             istop: 7 (itn >= iter_lim), 6 (1 + test3 <= 1), 5 (1 + test2 <= 1), 4 (1 + tt1 <= 1),
//                    3 (test3 <= ctol), 2 (test2 <= atol), 1 (test1 <= rtol), the last that holds
// The update is HBM-bound: per model element it reads x, w, V (and var) and writes x, w (and var).
#include <math.h>
#include "common.cuh"

namespace {

constexpr double EPS = 2.220446049250313e-16;   // np.finfo(np.float64).eps
constexpr int UPD_THREADS = B2_RED_THREADS;

__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dvd(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double rt(double a) { return __dsqrt_rn(a); }
__device__ __forceinline__ double sgn(double a) { return a > 0.0 ? 1.0 : (a < 0.0 ? -1.0 : a); }  // np.sign (0, nan kept)

// scipy's _sym_ortho(a, b) -> (c, s, r)
__device__ void sym_ortho(double a, double b, double& c, double& s, double& r) {
  if (b == 0.0) {
    c = sgn(a); s = 0.0; r = fabs(a);
  } else if (a == 0.0) {
    c = 0.0; s = sgn(b); r = fabs(b);
  } else if (fabs(b) > fabs(a)) {
    const double tau = dvd(a, b);
    s = dvd(sgn(b), rt(add(1.0, mul(tau, tau))));
    c = mul(s, tau);
    r = dvd(b, s);
  } else {
    const double tau = dvd(b, a);
    c = dvd(sgn(a), rt(add(1.0, mul(tau, tau))));
    s = mul(c, tau);
    r = dvd(a, c);
  }
}

// tests of the pending iteration, now that its ||dk||^2 (DD) is reduced; writes its history row
__device__ void finish(double* s, double* hist, size_t cap) {
  s[B2_LSQR_DDNORM] = add(s[B2_LSQR_DDNORM], s[B2_LSQR_DD]);
  s[B2_LSQR_DD] = 0.0;
  const double anorm = s[B2_LSQR_ANORM];
  const double acond = mul(anorm, rt(s[B2_LSQR_DDNORM]));
  const double test1 = s[B2_LSQR_TEST1], test2 = s[B2_LSQR_TEST2], tt1 = s[B2_LSQR_TT1];
  const double test3 = dvd(1.0, add(acond, EPS));
  const double itn = s[B2_LSQR_ITN];
  double istop = 0.0;
  if (itn >= s[B2_LSQR_ITER_LIM]) istop = 7.0;
  if (add(1.0, test3) <= 1.0) istop = 6.0;
  if (add(1.0, test2) <= 1.0) istop = 5.0;
  if (add(1.0, tt1) <= 1.0) istop = 4.0;
  if (test3 <= s[B2_LSQR_CTOL]) istop = 3.0;
  if (test2 <= s[B2_LSQR_ATOL]) istop = 2.0;
  if (test1 <= s[B2_LSQR_RTOL]) istop = 1.0;
  s[B2_LSQR_ACOND] = acond;
  s[B2_LSQR_ISTOP] = istop;
  s[B2_LSQR_PENDING] = 0.0;
  if (istop != 0.0) s[B2_LSQR_STOPPED] = 1.0;
  const size_t row = (size_t)itn - 1;
  if (hist && row < cap) {
    double* h = hist + row * B2_LSQR_HIST;
    h[0] = s[B2_LSQR_R1NORM]; h[1] = s[B2_LSQR_R2NORM]; h[2] = anorm; h[3] = acond; h[4] = s[B2_LSQR_ARNORM];
    h[5] = s[B2_LSQR_XNORM]; h[6] = test1; h[7] = test2; h[8] = istop;
  }
}

__global__ void lsqr_scalars_kernel(double* s, int phase, double* hist, size_t cap) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (s[B2_LSQR_STOPPED] != 0.0) return;
  if (phase != 1) {
    if (s[B2_LSQR_PENDING] != 0.0) finish(s, hist, cap);
    if (phase == 2 || s[B2_LSQR_STOPPED] != 0.0) return;
    // beta of this iteration and the coefficients of V <- cvA A^H U - cvB V (scipy: v = A^H (U / beta) - beta v);
    // beta == 0 leaves v as it is (scipy skips the v-step)
    const double beta = rt(s[B2_LSQR_BB]);
    s[B2_LSQR_BETA] = beta;
    if (beta > 0.0) {
      s[B2_LSQR_CVA] = dvd(1.0, beta);
      s[B2_LSQR_CVB] = mul(beta, s[B2_LSQR_INV_ALFA]);
    } else {
      s[B2_LSQR_CVA] = 0.0;
      s[B2_LSQR_CVB] = -1.0;
    }
    return;
  }
  const double damp = s[B2_LSQR_DAMP], dampsq = s[B2_LSQR_DAMPSQ], beta = s[B2_LSQR_BETA];
  s[B2_LSQR_ITN] = add(s[B2_LSQR_ITN], 1.0);
  double alfa = s[B2_LSQR_ALFA], anorm = s[B2_LSQR_ANORM];
  if (beta > 0.0) {
    anorm = rt(add(add(add(mul(anorm, anorm), mul(alfa, alfa)), mul(beta, beta)), dampsq));
    alfa = rt(s[B2_LSQR_AA]);
    s[B2_LSQR_INV_ALFA] = alfa > 0.0 ? dvd(1.0, alfa) : 1.0;
  }
  double rhobar = s[B2_LSQR_RHOBAR], phibar = s[B2_LSQR_PHIBAR], rhobar1, psi;
  if (damp > 0.0) {
    rhobar1 = rt(add(mul(rhobar, rhobar), dampsq));
    const double cs1 = dvd(rhobar, rhobar1), sn1 = dvd(damp, rhobar1);
    psi = mul(sn1, phibar);
    phibar = mul(cs1, phibar);
  } else {
    rhobar1 = rhobar;
    psi = 0.0;
  }
  double cs, sn, rho;
  sym_ortho(rhobar1, beta, cs, sn, rho);
  const double theta = mul(sn, alfa);
  rhobar = mul(-cs, alfa);
  const double phi = mul(cs, phibar);
  phibar = mul(sn, phibar);
  const double tau = mul(sn, phi);
  s[B2_LSQR_T1] = dvd(phi, rho);
  s[B2_LSQR_T2] = dvd(-theta, rho);
  s[B2_LSQR_INV_RHO] = dvd(1.0, rho);
  // plane rotation on the right: the xnorm estimate
  const double delta = mul(s[B2_LSQR_SN2], rho), gambar = mul(-s[B2_LSQR_CS2], rho);
  const double rhs = sub(phi, mul(delta, s[B2_LSQR_Z]));
  const double zbar = dvd(rhs, gambar);
  double xxnorm = s[B2_LSQR_XXNORM];
  const double xnorm = rt(add(xxnorm, mul(zbar, zbar)));
  const double gamma = rt(add(mul(gambar, gambar), mul(theta, theta)));
  s[B2_LSQR_CS2] = dvd(gambar, gamma);
  s[B2_LSQR_SN2] = dvd(theta, gamma);
  const double z = dvd(rhs, gamma);
  xxnorm = add(xxnorm, mul(z, z));
  s[B2_LSQR_Z] = z;
  s[B2_LSQR_XXNORM] = xxnorm;
  // residual norms and the tests that do not need ddnorm
  const double res1 = mul(phibar, phibar);
  const double res2 = add(s[B2_LSQR_RES2], mul(psi, psi));
  const double rnorm = rt(add(res1, res2));
  const double arnorm = mul(alfa, fabs(tau));
  double r1norm = rnorm;
  if (damp > 0.0) {
    const double r1sq = sub(mul(rnorm, rnorm), mul(dampsq, xxnorm));
    r1norm = rt(fabs(r1sq));
    if (r1sq < 0.0) r1norm = -r1norm;
  }
  const double bnorm = s[B2_LSQR_BNORM];
  const double test1 = dvd(rnorm, bnorm);
  s[B2_LSQR_TEST1] = test1;
  s[B2_LSQR_TEST2] = dvd(arnorm, add(mul(anorm, rnorm), EPS));
  s[B2_LSQR_TT1] = dvd(test1, add(1.0, dvd(mul(anorm, xnorm), bnorm)));
  s[B2_LSQR_RTOL] = add(s[B2_LSQR_BTOL], dvd(mul(mul(s[B2_LSQR_ATOL], anorm), xnorm), bnorm));
  s[B2_LSQR_ALFA] = alfa; s[B2_LSQR_ANORM] = anorm; s[B2_LSQR_RHOBAR] = rhobar; s[B2_LSQR_PHIBAR] = phibar;
  s[B2_LSQR_RES2] = res2; s[B2_LSQR_XNORM] = xnorm; s[B2_LSQR_ARNORM] = arnorm;
  s[B2_LSQR_R1NORM] = r1norm; s[B2_LSQR_R2NORM] = rnorm;
  s[B2_LSQR_PENDING] = 1.0;
  // next u-step: U <- inv_alfa A V - cub U  (scipy: u = A (V / alfa) - alfa (U / beta))
  s[B2_LSQR_CUB] = mul(alfa, beta > 0.0 ? dvd(1.0, beta) : 1.0);
}

// ---- model-side update ------------------------------------------------------------------------------------------
__device__ __forceinline__ float rmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float radd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float rsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double rmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double radd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double rsub(double a, double b) { return __dsub_rn(a, b); }

struct UpdCoef {
  double t1, t2, inv_rho, inv_alfa;
};

// one real element (x, w, v); returns dk
template <typename T>
__device__ __forceinline__ T upd1(T& x, T& w, T v, T t1, T t2, T ir, T ia) {
  const T wo = w;
  const T dk = rmul(ir, wo);
  x = radd(x, rmul(t1, wo));
  w = radd(rmul(ia, v), rmul(t2, wo));
  return dk;
}
// var += dk^2 for one real element, or for one complex element (dr, di) as NumPy's complex square
template <typename T>
__device__ __forceinline__ void var_real(T& var, T dk) { var = radd(var, rmul(dk, dk)); }
template <typename T>
__device__ __forceinline__ void var_cx(T& vr, T& vi, T dr, T di) {
  vr = radd(vr, rsub(rmul(dr, dr), rmul(di, di)));
  vi = radd(vi, radd(rmul(dr, di), rmul(di, dr)));
}

template <typename T, bool CX, bool VAR, bool VEC>
__global__ void __launch_bounds__(UPD_THREADS)
lsqr_update_kernel(T* __restrict__ x, T* __restrict__ w, const T* __restrict__ v, T* __restrict__ var,
                   size_t n_real, const double* __restrict__ coef, const double* __restrict__ stop,
                   double* __restrict__ partials, unsigned int* __restrict__ ticket, double* __restrict__ dd) {
  if (stop && *stop != 0.0) return;                       // uniform across the grid: no CTA takes a ticket
  const UpdCoef c = *reinterpret_cast<const UpdCoef*>(coef);
  const T t1 = (T)c.t1, t2 = (T)c.t2, ir = (T)c.inv_rho, ia = (T)c.inv_alfa;
  double acc = 0.0;
  const size_t stride = (size_t)gridDim.x * UPD_THREADS;
  size_t i = (size_t)blockIdx.x * UPD_THREADS + threadIdx.x;
  constexpr int V = Vec16<T>::N;
  size_t done = 0;
  if (VEC) {
    const size_t nvec = n_real / V;
    for (; i < nvec; i += stride) {
      Vec16<T> vx = load_vec_coherent(x + i * V), vw = load_vec_coherent(w + i * V);
      const Vec16<T> vv = load_vec(v + i * V);
      Vec16<T> dk;
#pragma unroll
      for (int k = 0; k < V; ++k) {
        dk.v[k] = upd1(vx.v[k], vw.v[k], vv.v[k], t1, t2, ir, ia);
        acc = fma((double)dk.v[k], (double)dk.v[k], acc);
      }
      store_vec(x + i * V, vx);
      store_vec(w + i * V, vw);
      if (VAR) {
        Vec16<T> vr = load_vec_coherent(var + i * V);
        if (CX) {
#pragma unroll
          for (int k = 0; k < V; k += 2) var_cx(vr.v[k], vr.v[k + 1], dk.v[k], dk.v[k + 1]);
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) var_real(vr.v[k], dk.v[k]);
        }
        store_vec(var + i * V, vr);
      }
    }
    done = nvec * V;
    i = done + ((size_t)blockIdx.x * UPD_THREADS + threadIdx.x) * (CX ? 2 : 1);   // tail: at most V - 1 reals
  } else {
    i *= (CX ? 2 : 1);
  }
  // scalar path (whole array when unaligned, else the tail): one real, or one complex pair, per step
  const size_t step = stride * (CX ? 2 : 1);
  for (; i < n_real; i += step) {
    if (CX) {
      const T dr = upd1(x[i], w[i], v[i], t1, t2, ir, ia);
      const T di = upd1(x[i + 1], w[i + 1], v[i + 1], t1, t2, ir, ia);
      acc = fma((double)dr, (double)dr, acc);
      acc = fma((double)di, (double)di, acc);
      if (VAR) var_cx(var[i], var[i + 1], dr, di);
    } else {
      const T dk = upd1(x[i], w[i], v[i], t1, t2, ir, ia);
      acc = fma((double)dk, (double)dk, acc);
      if (VAR) var_real(var[i], dk);
    }
  }
  b2_grid_fold<1, RED_SUM>(&acc, partials, ticket, dd);
}

template <typename T, bool CX, bool VAR>
int launch_update(b2_ctx* ctx, void* x, void* w, const void* v, void* var, size_t n_real, const double* coef,
                  const double* stop, double* dd, cudaStream_t st) {
  constexpr int V = Vec16<T>::N;
  const bool vec = b2_aligned16(x) && b2_aligned16(w) && b2_aligned16(v) && (!VAR || b2_aligned16(var)) &&
                   n_real >= (size_t)V;
  const size_t items = vec ? n_real / V : (CX ? n_real / 2 : n_real);
  const int grid = b2_red_grid(ctx, items, UPD_THREADS);   // one item per thread: no unrolled loop
  if (vec)
    lsqr_update_kernel<T, CX, VAR, true><<<grid, UPD_THREADS, 0, st>>>(
        (T*)x, (T*)w, (const T*)v, (T*)var, n_real, coef, stop, ctx->red_partials, ctx->tickets, dd);
  else
    lsqr_update_kernel<T, CX, VAR, false><<<grid, UPD_THREADS, 0, st>>>(
        (T*)x, (T*)w, (const T*)v, (T*)var, n_real, coef, stop, ctx->red_partials, ctx->tickets, dd);
  B2_LAUNCH_CHECK();
  return B2_OK;
}

template <typename T, bool CX>
int launch_update_var(b2_ctx* ctx, void* x, void* w, const void* v, void* var, size_t n_real, const double* coef,
                      const double* stop, double* dd, cudaStream_t st) {
  if (var) return launch_update<T, CX, true>(ctx, x, w, v, var, n_real, coef, stop, dd, st);
  return launch_update<T, CX, false>(ctx, x, w, v, var, n_real, coef, stop, dd, st);
}

}  // namespace

extern "C" int b2_lsqr_scalars(double* state_dev, int phase, double* hist_dev, size_t cap, void* stream) {
  if (!state_dev || phase < 0 || phase > 2 || (!hist_dev && cap)) return B2_ERR_ARG;
  lsqr_scalars_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(state_dev, phase, hist_dev, cap);
  B2_LAUNCH_CHECK();
  return B2_OK;
}

extern "C" int b2_lsqr_update(b2_ctx* ctx, void* x, void* w, const void* v, void* var, size_t n, int dtype,
                              const double* coef_dev, const double* stop_dev, double* dd_dev, void* stream) {
  if (!ctx || !coef_dev || !dd_dev) return B2_ERR_ARG;
  const bool cx = (dtype == B2_C64 || dtype == B2_C128);
  if (!cx && dtype != B2_F32 && dtype != B2_F64) return B2_ERR_DTYPE;
  cudaStream_t st = (cudaStream_t)stream;
  // a rank may own no model elements (n == 0, null arrays allowed): one CTA writes its ||dk||^2 = 0 unless stopped,
  // and it is still all-reduced
  if (n && (!x || !w || !v || x == w || x == v || w == v || (var && (var == x || var == w || var == v))))
    return B2_ERR_ARG;
  const size_t n_real = cx ? 2 * n : n;
  return b2_dispatch(dtype, [&](auto t) {
    return launch_update_var<b2_real_t<decltype(t)>, b2_is_cx_v<decltype(t)>>(ctx, x, w, v, var, n_real, coef_dev,
                                                                              stop_dev, dd_dev, st);
  });
}
