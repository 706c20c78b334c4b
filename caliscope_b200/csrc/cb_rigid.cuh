// Robust pose of a rigid body seen by a calibrated rig (cb_rigid_pose_robust, DESIGN.md section 4.14): per group (the
// rows of one body at one moment, every camera's), Horn poses of triples of triangulated model points scored by MSAC
// over all rows, the consensus rows, then Levenberg-Marquardt over the body pose (r, t) with X_w = R(r) M + t and its
// first-order covariance with the rig's camera term.  oracle/rigid_pose_robust.py states the rule and
// oracle/rigid_pose_gp3p.py its gP3P hypotheses.
//
// The point hypotheses come from tri_consensus_kernel run unchanged on the (group, model point) sub-groups; the kernels
// here take the qualified points of each group (qX, qM: ascending model index) and follow the short shape of
// cb_resect_robust: LANES (8 or 32) lanes per group, the camera table staged in shared memory when it fits.
// No floating-point atomics: every sum has a fixed order, so repeated calls give bit-identical outputs.
#pragma once
#include <cstdint>

#include "cb_device.cuh"
#include "cb_kernels.cuh"
#include "cb_resect.cuh"
#include "cb_triangulate.cuh"

namespace cb {

constexpr double RIG_DEGENERATE = 1e-9;  // |u x v| <= this |u| |v|: a model triangle without a rotation
constexpr int RIG_AMBIGUOUS = 6;  // status: a gP3P winner whose consensus rows hold fewer than four model points

// Horn's closed-form absolute orientation (JOSA A 4(4), 1987) without scale of three model points M against their
// world points X: q the eigenvector of the largest eigenvalue of Horn's N (sym4_min_eigvec of -N), R = R(q),
// t = mean(X) - R mean(M).  False when the model triangle is degenerate or R, t are not finite.
__device__ __forceinline__ bool rig_horn(const double M[3][3], const double X[3][3], double* R, double* t) {
  double u[3], v[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    u[a] = M[1][a] - M[0][a];
    v[a] = M[2][a] - M[0][a];
  }
  const double c0 = u[1] * v[2] - u[2] * v[1], c1 = u[2] * v[0] - u[0] * v[2], c2 = u[0] * v[1] - u[1] * v[0];
  const double nc = sqrt(c0 * c0 + c1 * c1 + c2 * c2);
  const double nu = sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]), nv = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (!(nc > RIG_DEGENERATE * nu * nv)) return false;
  double mb[3], xb[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    mb[a] = (M[0][a] + M[1][a] + M[2][a]) / 3.0;
    xb[a] = (X[0][a] + X[1][a] + X[2][a]) / 3.0;
  }
  double S[3][3];  // sum_i (M_i - mean M)(X_i - mean X)^T
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      double s = 0.0;
#pragma unroll
      for (int i = 0; i < 3; ++i) s += (M[i][a] - mb[a]) * (X[i][b] - xb[b]);
      S[a][b] = s;
    }
  // -N
  double A[4][4];
  A[0][0] = -(S[0][0] + S[1][1] + S[2][2]);
  A[0][1] = A[1][0] = -(S[1][2] - S[2][1]);
  A[0][2] = A[2][0] = -(S[2][0] - S[0][2]);
  A[0][3] = A[3][0] = -(S[0][1] - S[1][0]);
  A[1][1] = -(S[0][0] - S[1][1] - S[2][2]);
  A[1][2] = A[2][1] = -(S[0][1] + S[1][0]);
  A[1][3] = A[3][1] = -(S[2][0] + S[0][2]);
  A[2][2] = -(-S[0][0] + S[1][1] - S[2][2]);
  A[2][3] = A[3][2] = -(S[1][2] + S[2][1]);
  A[3][3] = -(-S[0][0] - S[1][1] + S[2][2]);
  double q[4];
  sym4_min_eigvec(A, q);
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  R[0] = w * w + x * x - y * y - z * z; R[1] = 2.0 * (x * y - w * z);         R[2] = 2.0 * (x * z + w * y);
  R[3] = 2.0 * (x * y + w * z);         R[4] = w * w - x * x + y * y - z * z; R[5] = 2.0 * (y * z - w * x);
  R[6] = 2.0 * (x * z - w * y);         R[7] = 2.0 * (y * z + w * x);         R[8] = w * w - x * x - y * y + z * z;
  bool ok = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    t[a] = xb[a] - (R[3 * a] * mb[0] + R[3 * a + 1] * mb[1] + R[3 * a + 2] * mb[2]);
    ok = ok && isfinite(t[a]);
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) ok = ok && isfinite(R[k]);
  return ok;
}

// squared pixel error of caller row r at body pose (R, t) in its own camera, and whether it is in front of it
__device__ __forceinline__ double rig_row_err2(const double* cams, int stride, const double* R, const double* t, int r,
                                               const int* __restrict__ obs_cam, const int* __restrict__ obs_pt,
                                               const double* __restrict__ obs_px, const double* __restrict__ model,
                                               bool& front) {
  const double* M = model + 3 * (size_t)obs_pt[r];
  double X[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) X[a] = fma(R[3 * a], M[0], fma(R[3 * a + 1], M[1], fma(R[3 * a + 2], M[2], t[a])));
  return tri_row_err2(cams + (size_t)stride * obs_cam[r], X, reinterpret_cast<const double2*>(obs_px)[r], front);
}

// ---- generalized three-point pose (gP3P) -------------------------------------------------------------------------------
// The body poses that put three model points M_i on three rays X_i = c_i + lambda_i d_i from different cameras (one
// camera: P3P).  oracle/gp3p.py states the rule; the constants are its own.
constexpr double GP3P_PARALLEL = 1e-12;  // det(sum (I - d d^T)) at or below this: the rays are parallel
constexpr double GP3P_CLAMP = 1e-8;      // Delta_j >= -GP3P_CLAMP (1 + p_j^2) is clamped to 0, below it: no hypothesis
constexpr double GP3P_UMAX = 1e9;        // roots beyond |u_1| = GP3P_UMAX are not sought
constexpr int GP3P_NEWTON = 3;           // Newton steps of the polish at most
constexpr int GP3P_MAX = 8;              // roots of the octic, so hypotheses of one sample: slot 1 + 8 m + c
constexpr int GP3P_ITERS = 100;          // safeguarded Newton steps per root at most

// the normalised system of one sample (oracle/gp3p.py steps 1-2): lh the depths of the feet of X^ on the lines, cp the
// feet relative to X^ over s, D2 the squared model sides over s^2 (12, 13, 23), p_j and Delta_j (j = 2, 3) in u_1, and
// the octic F, lowest degree first
struct GP3PSys {
  double Xh[3], lh[3], cp[3][3], s, D2[3];
  double p[2][2], dl[2][3];
  double f[9];
};

template <int NA, int NB>
__device__ __forceinline__ void gp_mul(const double (&a)[NA], const double (&b)[NB], double (&o)[NA + NB - 1]) {
#pragma unroll
  for (int i = 0; i < NA + NB - 1; ++i) o[i] = 0.0;
#pragma unroll
  for (int i = 0; i < NA; ++i)
#pragma unroll
    for (int j = 0; j < NB; ++j) o[i + j] = fma(a[i], b[j], o[i + j]);
}

__device__ __forceinline__ double gp_dot(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// Steps 0-2 on camera centres c, unit rays d and model points M: false for a degenerate model triangle or parallel rays
__device__ __forceinline__ bool rig_gp3p_system(const double c[3][3], const double d[3][3], const double M[3][3],
                                                GP3PSys& S) {
  double u[3], v[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    u[a] = M[1][a] - M[0][a];
    v[a] = M[2][a] - M[0][a];
  }
  const double x0 = u[1] * v[2] - u[2] * v[1], x1 = u[2] * v[0] - u[0] * v[2], x2 = u[0] * v[1] - u[1] * v[0];
  const double nu2 = gp_dot(u, u), nv2 = gp_dot(v, v);
  if (!(sqrt(x0 * x0 + x1 * x1 + x2 * x2) > RIG_DEGENERATE * sqrt(nu2) * sqrt(nv2))) return false;
  // A = sum (I - d d^T), b = sum (I - d d^T) c, X^ = A^-1 b by the adjugate
  double A[3][3], bb[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    bb[a] = 0.0;
#pragma unroll
    for (int e = 0; e < 3; ++e) A[a][e] = 0.0;
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double dc = gp_dot(d[i], c[i]);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      bb[a] += c[i][a] - d[i][a] * dc;
#pragma unroll
      for (int e = 0; e < 3; ++e) A[a][e] += (a == e ? 1.0 : 0.0) - d[i][a] * d[i][e];
    }
  }
  const double C00 = A[1][1] * A[2][2] - A[1][2] * A[2][1], C01 = A[1][2] * A[2][0] - A[1][0] * A[2][2],
               C02 = A[1][0] * A[2][1] - A[1][1] * A[2][0];
  const double det = A[0][0] * C00 + A[0][1] * C01 + A[0][2] * C02;
  if (!(det > GP3P_PARALLEL)) return false;
  const double C11 = A[0][0] * A[2][2] - A[0][2] * A[2][0], C12 = A[0][1] * A[2][0] - A[0][0] * A[2][1],
               C22 = A[0][0] * A[1][1] - A[0][1] * A[1][0];
  const double id = 1.0 / det;
  double* Xh = S.Xh;  // A is symmetric: its adjugate is the cofactor matrix
  Xh[0] = (C00 * bb[0] + C01 * bb[1] + C02 * bb[2]) * id;
  Xh[1] = (C01 * bb[0] + C11 * bb[1] + C12 * bb[2]) * id;
  Xh[2] = (C02 * bb[0] + C12 * bb[1] + C22 * bb[2]) * id;
  const double D01 = sqrt(nu2), D02 = sqrt(nv2);
  double w[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) w[a] = M[2][a] - M[1][a];
  const double D12 = sqrt(gp_dot(w, w));
  S.s = fmax(fmax(D01, D02), D12);
  const double is = 1.0 / S.s;
  S.D2[0] = (D01 * is) * (D01 * is);
  S.D2[1] = (D02 * is) * (D02 * is);
  S.D2[2] = (D12 * is) * (D12 * is);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    double xc[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) xc[a] = Xh[a] - c[i][a];
    S.lh[i] = gp_dot(d[i], xc);
#pragma unroll
    for (int a = 0; a < 3; ++a) S.cp[i][a] = (c[i][a] + S.lh[i] * d[i][a] - Xh[a]) / S.s;
  }
  // p_j, Delta_j for j = 2, 3 (index 0, 1 here)
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    double wj[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) wj[a] = S.cp[0][a] - S.cp[1 + j][a];
    const double dw = gp_dot(d[1 + j], wj), a1 = gp_dot(d[0], d[1 + j]);
    S.p[j][0] = dw;
    S.p[j][1] = a1;
    S.dl[j][0] = dw * dw - (gp_dot(wj, wj) - S.D2[j]);
    S.dl[j][1] = 2.0 * dw * a1 - 2.0 * gp_dot(d[0], wj);
    S.dl[j][2] = a1 * a1 - 1.0;
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) w[a] = S.cp[1][a] - S.cp[2][a];
  const double a23 = gp_dot(d[1], d[2]), e2 = gp_dot(d[1], w), e3 = gp_dot(d[2], w);
  const double(&p2)[2] = S.p[0];
  const double(&p3)[2] = S.p[1];
  double p22[3], p33[3], p23[3];
  gp_mul(p2, p2, p22);
  gp_mul(p3, p3, p33);
  gp_mul(p2, p3, p23);
  double P0[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) P0[i] = p22[i] + S.dl[0][i] + p33[i] + S.dl[1][i] - 2.0 * a23 * p23[i];
#pragma unroll
  for (int i = 0; i < 2; ++i) P0[i] += 2.0 * e2 * p2[i] - 2.0 * e3 * p3[i];
  P0[0] += gp_dot(w, w) - S.D2[2];
  double P2[2], P3[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    P2[i] = 2.0 * p2[i] - 2.0 * a23 * p3[i];
    P3[i] = 2.0 * p3[i] - 2.0 * a23 * p2[i];
  }
  P2[0] += 2.0 * e2;
  P3[0] -= 2.0 * e3;
  const double P23 = -2.0 * a23;
  double d23[5], P00[5], P22[3], P33[3], P22d[5], P33d[5], P2P3[3];
  gp_mul(S.dl[0], S.dl[1], d23);
  gp_mul(P0, P0, P00);
  gp_mul(P2, P2, P22);
  gp_mul(P3, P3, P33);
  gp_mul(P22, S.dl[0], P22d);
  gp_mul(P33, S.dl[1], P33d);
  gp_mul(P2, P3, P2P3);
  double Q0[5], Q1[3];
#pragma unroll
  for (int i = 0; i < 5; ++i) Q0[i] = P00[i] + P23 * P23 * d23[i] - (P22d[i] + P33d[i]);
#pragma unroll
  for (int i = 0; i < 3; ++i) Q1[i] = 2.0 * (P23 * P0[i] - P2P3[i]);
  double Q00[9], Q11[5], Q11d[9];
  gp_mul(Q0, Q0, Q00);
  gp_mul(Q1, Q1, Q11);
  gp_mul(Q11, d23, Q11d);
#pragma unroll
  for (int i = 0; i < 9; ++i) S.f[i] = Q00[i] - Q11d[i];
  return true;
}

// G_J = F^(J) (degree 8 - J) at x and its derivative
template <int J>
__device__ __forceinline__ void gp_deriv_eval(const double (&f)[9], double x, double& g, double& dg) {
  constexpr int N = 8 - J;
  double c[N + 1];
#pragma unroll
  for (int i = 0; i <= N; ++i) {
    double k = 1.0;
#pragma unroll
    for (int q = 1; q <= J; ++q) k *= (double)(i + q);  // (i + J)! / i!
    c[i] = f[i + J] * k;
  }
  g = c[N];
  dg = 0.0;
#pragma unroll
  for (int i = N - 1; i >= 0; --i) {
    dg = fma(dg, x, g);
    g = fma(g, x, c[i]);
  }
}

// The root of G_J in (lo, hi] where G_J is monotone (glo = G_J(lo), ghi = G_J(hi)), NaN without a sign change there:
// Newton steps safeguarded by the bracket, bisection when a step leaves it
template <int J>
__device__ __forceinline__ double gp_bracket(const double (&f)[9], double lo, double hi, double glo, double ghi) {
  if (!((glo < 0.0 && ghi >= 0.0) || (glo > 0.0 && ghi <= 0.0))) return res_nan();
  if (ghi == 0.0) return hi;
  double a = glo < 0.0 ? lo : hi, b = glo < 0.0 ? hi : lo;  // G(a) < 0 < G(b)
  double x = 0.5 * (lo + hi);
#pragma unroll 1
  for (int it = 0; it < GP3P_ITERS; ++it) {
    double g, dg;
    gp_deriv_eval<J>(f, x, g, dg);
    if (g == 0.0) break;
    if (g < 0.0) a = x;
    else b = x;
    double xn = x - g / dg;
    if (!(xn > fmin(a, b) && xn < fmax(a, b))) xn = 0.5 * (a + b);
    const bool done = fabs(xn - x) <= 1e-15 * fmax(1.0, fabs(x));
    x = xn;
    if (done) break;
  }
  return x;
}

// The roots of G_J, ascending in slots 0..7-J (NaN: none in that slot), from those of G_{J+1} (slots 0..6-J): G_J is
// monotone between consecutive real roots of its derivative, so each such interval of [-B, B] holds at most one root
template <int J>
__device__ __forceinline__ void gp_level(const double (&f)[9], double B, double (&r)[GP3P_MAX]) {
  double lo = -B, g, dg;
  gp_deriv_eval<J>(f, lo, g, dg);
  double glo = g;
#pragma unroll
  for (int i = 0; i < 8 - J; ++i) {
    const double hi = i < 7 - J ? r[i] : B;  // r[i] is G_{J+1}'s slot i and becomes G_J's
    if (i < 7 - J && isnan(hi)) continue;
    gp_deriv_eval<J>(f, hi, g, dg);
    r[i] = gp_bracket<J>(f, lo, hi, glo, g);
    lo = hi;
    glo = g;
  }
}

// The real roots of the octic F in [-B, B], B = Fujiwara's bound 2 max |f_{8-i} / f_8|^(1/i) clamped to [1, GP3P_UMAX],
// ascending in r (NaN: none), through the derivative chain F^(7), ..., F (Gauss-Lucas: the derivatives' real roots lie
// within F's bound too).  Only the coefficients and the eight slots stay in registers.
__device__ __forceinline__ void rig_gp3p_roots(const double (&f)[9], double (&r)[GP3P_MAX]) {
  double B = 0.0;
#pragma unroll
  for (int i = 1; i <= 8; ++i) B = fmax(B, pow(fabs(f[8 - i] / f[8]), 1.0 / i));
  B = 2.0 * B;
  B = isnan(B) ? GP3P_UMAX : fmin(fmax(B, 1.0), GP3P_UMAX);
#pragma unroll
  for (int i = 0; i < GP3P_MAX; ++i) r[i] = res_nan();
  // F^(8) is a constant: F^(7) has its one slot in [-B, B]
  gp_level<7>(f, B, r);
  gp_level<6>(f, B, r);
  gp_level<5>(f, B, r);
  gp_level<4>(f, B, r);
  gp_level<3>(f, B, r);
  gp_level<2>(f, B, r);
  gp_level<1>(f, B, r);
  gp_level<0>(f, B, r);
}

// f_12, f_13, f_23 at u and the points Y_i = c'_i + u_i d_i
__device__ __forceinline__ void gp_resid(const GP3PSys& S, const double d[3][3], const double* u, double* fr,
                                         double Y[3][3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int a = 0; a < 3; ++a) Y[i][a] = fma(u[i], d[i][a], S.cp[i][a]);
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const int i = q == 2 ? 1 : 0, j = q == 0 ? 1 : 2;
    double e[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) e[a] = Y[i][a] - Y[j][a];
    fr[q] = gp_dot(e, e) - S.D2[q];
  }
}

// Step 3 for root u1: the world points X_i = X^ + s (c'_i + u_i d_i) = c_i + lambda_i d_i (false: no hypothesis).
// Not inlined: the system S then stays in the lane's local memory, which keeps rig_consensus_kernel<LANES, true> free
// of spills (inlined, the root loop needs more than 255 registers).
__device__ __noinline__ bool rig_gp3p_points(const GP3PSys& S, const double d[3][3], double u1, double X[3][3]) {
  double pv[2], sq[2];
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    pv[j] = fma(S.p[j][1], u1, S.p[j][0]);
    const double dv = fma(fma(S.dl[j][2], u1, S.dl[j][1]), u1, S.dl[j][0]);
    ok = ok && !(dv < -GP3P_CLAMP * (1.0 + pv[j] * pv[j]));
    sq[j] = sqrt(fmax(dv, 0.0));
  }
  if (!ok) return false;
  double u[3] = {u1, 0.0, 0.0}, best = __longlong_as_double(0x7ff0000000000000LL);
  bool any = false;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const double t[3] = {u1, pv[0] + (q < 2 ? sq[0] : -sq[0]), pv[1] + ((q & 1) == 0 ? sq[1] : -sq[1])};
    double fr[3], Y[3][3];
    gp_resid(S, d, t, fr, Y);
    if (fabs(fr[2]) < best) {
      best = fabs(fr[2]);
      u[1] = t[1];
      u[2] = t[2];
      any = true;
    }
  }
  if (!any) return false;
  double fr[3], Y[3][3];
  gp_resid(S, d, u, fr, Y);
  double ss = fr[0] * fr[0] + fr[1] * fr[1] + fr[2] * fr[2];
#pragma unroll 1
  for (int it = 0; it < GP3P_NEWTON; ++it) {
    // J rows (f_12, f_13, f_23): d f_ij / d u_i = 2 e . d_i, d f_ij / d u_j = -2 e . d_j, e = Y_i - Y_j
    double e[3][3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      e[0][a] = Y[0][a] - Y[1][a];
      e[1][a] = Y[0][a] - Y[2][a];
      e[2][a] = Y[1][a] - Y[2][a];
    }
    const double J00 = 2.0 * gp_dot(e[0], d[0]), J01 = -2.0 * gp_dot(e[0], d[1]);
    const double J10 = 2.0 * gp_dot(e[1], d[0]), J12 = -2.0 * gp_dot(e[1], d[2]);
    const double J21 = 2.0 * gp_dot(e[2], d[1]), J22 = -2.0 * gp_dot(e[2], d[2]);
    // [[J00 J01 0] [J10 0 J12] [0 J21 J22]] x = f by Cramer
    const double det = J00 * (-J12 * J21) - J01 * (J10 * J22);
    const double x0 = (fr[0] * (-J12 * J21) - J01 * (fr[1] * J22 - J12 * fr[2])) / det;
    const double x1 = (J00 * (fr[1] * J22 - J12 * fr[2]) - fr[0] * (J10 * J22)) / det;
    const double x2 = (fr[0] * (J10 * J21) - J00 * (J21 * fr[1]) - J01 * (J10 * fr[2])) / det;
    const double un[3] = {u[0] - x0, u[1] - x1, u[2] - x2};
    double fn[3], Yn[3][3];
    gp_resid(S, d, un, fn, Yn);
    const double sn = fn[0] * fn[0] + fn[1] * fn[1] + fn[2] * fn[2];
    if (!(sn < ss)) break;
    ss = sn;
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      u[q] = un[q];
      fr[q] = fn[q];
#pragma unroll
      for (int a = 0; a < 3; ++a) Y[q][a] = Yn[q][a];
    }
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double lam = fma(S.s, u[i], S.lh[i]);
    ok = ok && isfinite(lam) && lam > 0.0;
#pragma unroll
    for (int a = 0; a < 3; ++a) X[i][a] = fma(S.s, Y[i][a], S.Xh[a]);
  }
  return ok;
}

// Per group, the first qualified point qstart[g] (qG: the group of each qualified point, ascending; qstart[n_groups] =
// n_q) and the prior row of the group's key (-1: none) by binary searches
__global__ void rig_group_kernel(const int* __restrict__ start, const int* __restrict__ rows,
                                 const long long* __restrict__ obs_key, int n_groups, const int* __restrict__ qG, int n_q,
                                 const long long* __restrict__ prior_key, int n_prior, int* __restrict__ qstart,
                                 int* __restrict__ prior_idx) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g > n_groups) return;
  int lo = 0, hi = n_q;  // first qualified point of a group >= g
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (qG[mid] < g) lo = mid + 1;
    else hi = mid;
  }
  qstart[g] = lo;
  if (g == n_groups) return;
  const long long key = obs_key[rows[start[g]]];
  lo = 0;
  hi = n_prior;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (prior_key[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  prior_idx[g] = (lo < n_prior && prior_key[lo] == key) ? lo : -1;
}

// 1 for a sub-group with a point hypothesis (consensus status 0), and a zero past the end for the scan
__global__ void rig_qual_flag_kernel(const int* __restrict__ cstatus, int n_sub, int* __restrict__ flag) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n_sub) flag[s] = cstatus[s] == TRI_OK ? 1 : 0;
  if (s == n_sub) flag[s] = 0;
}

// The qualified points in (group, model point) order: qX the point hypothesis, qM the model point, qG the group, at
// position qpos[s] (exclusive scan of the flags) of sub-group s; the sub-group's (group, point) comes from its sorted key
__global__ void rig_qual_kernel(const int* __restrict__ sstart, const unsigned long long* __restrict__ skey,
                                const int* __restrict__ cstatus, const double* __restrict__ xyz0, int n_sub, int pt_bits,
                                const int* __restrict__ qpos, double* __restrict__ qX, int* __restrict__ qM,
                                int* __restrict__ qG) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_sub || cstatus[s] != TRI_OK) return;
  const int j = qpos[s];
  const unsigned long long k = skey[sstart[s]];
#pragma unroll
  for (int a = 0; a < 3; ++a) qX[3 * (size_t)j + a] = xyz0[3 * (size_t)s + a];
  qM[j] = (int)(k & ((1ULL << pt_bits) - 1));
  qG[j] = (int)(k >> pt_bits);
}

// The gP3P hypotheses of sample m (row positions p of the group starting at b) scored over the group's rows [b, e):
// the best of them replaces (best, best_s, bR, bt) when its score is lower, at slot 1 + GP3P_MAX m + c
__device__ __forceinline__ void rig_gp3p_task(const double* cams, int stride, const int* __restrict__ rows,
                                              const int* __restrict__ obs_cam, const int* __restrict__ obs_pt,
                                              const double* __restrict__ obs_px, const double* __restrict__ obs_xy,
                                              const double* __restrict__ model, int b, int e, const int (&p)[3],
                                              long long m, double tau2, double& best, long long& best_s, double* bR,
                                              double* bt) {
  double c[3][3], d[3][3], M[3][3];
  int pt[3];
  bool ok = true;
#pragma unroll
  for (int s = 0; s < 3; ++s) {
    const int r = rows[b + p[s]];
    pt[s] = obs_pt[r];
    const double* cam = cams + (size_t)stride * obs_cam[r];
    const double* mp = model + 3 * (size_t)pt[s];
    const double2 n = reinterpret_cast<const double2*>(obs_xy)[r];
    const bool fish = (((int)cam[CT_FLAGS]) & 2) != 0;
    ok = ok && isfinite(n.x) && isfinite(n.y) && !(fish && n.x == -1000000.0 && n.y == -1000000.0);
    const double in = 1.0 / sqrt(n.x * n.x + n.y * n.y + 1.0);
    const double y[3] = {n.x * in, n.y * in, in};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      M[s][a] = mp[a];
      ok = ok && isfinite(mp[a]);
      // c = -R^T t, d = R^T y
      c[s][a] = -(cam[CT_R + a] * cam[CT_T] + cam[CT_R + 3 + a] * cam[CT_T + 1] + cam[CT_R + 6 + a] * cam[CT_T + 2]);
      d[s][a] = cam[CT_R + a] * y[0] + cam[CT_R + 3 + a] * y[1] + cam[CT_R + 6 + a] * y[2];
    }
  }
  ok = ok && pt[0] != pt[1] && pt[0] != pt[2] && pt[1] != pt[2];
  GP3PSys S;
  if (!ok || !rig_gp3p_system(c, d, M, S)) return;
  double roots[GP3P_MAX];
  rig_gp3p_roots(S.f, roots);
  int h = 0;
#pragma unroll 1
  for (int q = 0; q < GP3P_MAX; ++q) {
    double u1 = roots[0];
#pragma unroll
    for (int j = 1; j < GP3P_MAX; ++j) u1 = q == j ? roots[j] : u1;  // selects, so the slots stay in registers
    double X[3][3], R[9], t[3];
    if (isnan(u1) || !rig_gp3p_points(S, d, u1, X)) continue;
    double Mq[3][3];  // the model points again from memory: fewer registers live across the root loop
#pragma unroll
    for (int s = 0; s < 3; ++s)
#pragma unroll
      for (int a = 0; a < 3; ++a) Mq[s][a] = model[3 * (size_t)pt[s] + a];
    if (!rig_horn(Mq, X, R, t)) continue;
    double sc = 0.0;
    for (int i = b; i < e; ++i) {
      bool front;
      const double e2 = rig_row_err2(cams, stride, R, t, rows[i], obs_cam, obs_pt, obs_px, model, front);
      sc += msac_term(front, e2, tau2);
    }
    if (sc < best) {
      best = sc;
      best_s = 1 + GP3P_MAX * m + h;
#pragma unroll
      for (int a = 0; a < 9; ++a) bR[a] = R[a];
#pragma unroll
      for (int a = 0; a < 3; ++a) bt[a] = t[a];
    }
    ++h;
  }
}

// One group per LANES lanes.  Task 0 is the group's prior pose (prior_idx >= 0), task 1 + m sample m of the group's
// n_q qualified points (res_sample<3>); the lanes stride over the tasks, each builds its task's Horn pose and scores it
// over all k rows (slots increase along a lane's tasks, so the first of equal scores stays).  group_argmin picks the
// winner, which reaches the group's lanes from the lane that owns its task; then consensus_classify.  Writes hyp
// (R row-major, t; NaN without consensus), count, rep_row, n_inliers, n_points (n_q), status (1, 5 or 0) and the flags.
// GP3P (launched when gp3p_samples > 0): in a group with k >= 4 rows and n_q < 3, task 1 + m is instead gP3P sample m
// of the group's k rows (res_sample<3> with gp3p_samples, rig_gp3p_task on the undistorted coordinates obs_xy), whose
// hypotheses take slots 1 + 8 m + c; the slot's task, not the slot, names the owning lane.  Every other group runs the
// Horn path as it is.  GP3P also writes ambiguous[g] = 1 for a group with consensus whose winner is a gP3P hypothesis
// and whose consensus rows hold fewer than four distinct model points (lane 0 scans the flags in order and stops at the
// fourth), else 0; rig_ambiguous_kernel turns it into status 6 after the refinement.  GP3P = false ignores obs_xy,
// gp3p_samples and ambiguous.
template <int LANES, bool GP3P>
__global__ void __launch_bounds__(TRI_THREADS)
rig_consensus_kernel(const double* __restrict__ camtab, int n_cams, int cam_in_smem, const int* __restrict__ start,
                     const int* __restrict__ rows, const int* __restrict__ obs_cam, const int* __restrict__ obs_pt,
                     const double* __restrict__ obs_px, const double* __restrict__ model, const int* __restrict__ qstart,
                     const double* __restrict__ qX, const int* __restrict__ qM, const int* __restrict__ prior_idx,
                     const double* __restrict__ prior_pose, int n_groups, double tau, int min_inliers, int max_samples,
                     double* __restrict__ hyp, int* __restrict__ count, int* __restrict__ rep_row,
                     int* __restrict__ n_inliers, int* __restrict__ n_points, int* __restrict__ status,
                     unsigned char* __restrict__ pos_flag, unsigned char* __restrict__ inlier,
                     const double* __restrict__ obs_xy, int gp3p_samples, unsigned char* __restrict__ ambiguous) {
  extern __shared__ double s_cam[];
  int stride;
  const double* cams = tri_stage_camtab(camtab, n_cams, cam_in_smem, s_cam, stride);
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  const bool live = g < n_groups;
  const int b = live ? start[g] : 0, e = live ? start[g + 1] : 0, k = e - b;
  const int q0 = live ? qstart[g] : 0, nq = live ? qstart[g + 1] - q0 : 0;
  const int pi = live ? prior_idx[g] : -1;
  const int st = k < 4 ? TRI_FEW_ROWS : TRI_OK;
  const double tau2 = tau * tau;
  const double inf = __longlong_as_double(0x7ff0000000000000LL);
  const bool gp = GP3P && nq < 3;  // this group's samples are gP3P samples of its rows
  const long long T = gp ? res_triples(k) : res_triples(nq);
  const int cap = gp ? gp3p_samples : max_samples;
  const long long ntask = (live && st == TRI_OK) ? 1 + (T < cap ? T : (long long)cap) : 0;
  double best = inf, bR[9], bt[3];
#pragma unroll
  for (int a = 0; a < 9; ++a) bR[a] = 0.0;
#pragma unroll
  for (int a = 0; a < 3; ++a) bt[a] = 0.0;
  long long best_s = 0x7fffffffffffffffLL;
  for (long long task = lane; task < ntask; task += LANES) {
    if constexpr (GP3P) {
      if (gp && task > 0) {
        int p[3];
        if (res_sample<3>(task - 1, T, cap, k, p))
          rig_gp3p_task(cams, stride, rows, obs_cam, obs_pt, obs_px, obs_xy, model, b, e, p, task - 1, tau2, best,
                        best_s, bR, bt);
        continue;
      }
    }
    double R[9], t[3];
    if (task == 0) {
      if (pi < 0) continue;
      const double* p = prior_pose + 6 * (size_t)pi;
      double E[CT_JR + 9];
      cam_prep_rot(p[0], p[1], p[2], E);
#pragma unroll
      for (int a = 0; a < 9; ++a) R[a] = E[CT_R + a];
#pragma unroll
      for (int a = 0; a < 3; ++a) t[a] = p[3 + a];
    } else {
      int p[3];
      if (!res_sample<3>(task - 1, T, max_samples, nq, p)) continue;
      double M[3][3], X[3][3];
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int j = q0 + p[s];
        const double* m = model + 3 * (size_t)qM[j];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          M[s][a] = m[a];
          X[s][a] = qX[3 * (size_t)j + a];
        }
      }
      if (!rig_horn(M, X, R, t)) continue;
    }
    double sc = 0.0;
    for (int i = b; i < e; ++i) {
      bool front;
      const double e2 = rig_row_err2(cams, stride, R, t, rows[i], obs_cam, obs_pt, obs_px, model, front);
      sc += msac_term(front, e2, tau2);
    }
    if (sc < best) {
      best = sc;
      best_s = task;
#pragma unroll
      for (int a = 0; a < 9; ++a) bR[a] = R[a];
#pragma unroll
      for (int a = 0; a < 3; ++a) bt[a] = t[a];
    }
  }
  group_argmin<LANES>(best, best_s);
  const bool found = best < inf;
  const long long wtask = gp && best_s > 0 ? 1 + (best_s - 1) / GP3P_MAX : best_s;  // the winner's task
  const int owner = found ? (int)(wtask % LANES) : 0;
  group_bcast<LANES>(bR, owner);
  group_bcast<LANES>(bt, owner);
  int nin;
  const bool ok = consensus_classify<LANES>(
      found && st == TRI_OK, rows, b, e, lane, tau2, min_inliers,
      [&](int r, bool& front) { return rig_row_err2(cams, stride, bR, bt, r, obs_cam, obs_pt, obs_px, model, front); },
      pos_flag, inlier, nin);
  if constexpr (GP3P) __syncwarp();  // every lane's pos_flag from consensus_classify is visible to lane 0
  if (!live || lane != 0) return;
  if constexpr (GP3P) {
    int ns = 0;  // distinct model points of the consensus rows, up to 4
    if (ok && gp && best_s > 0) {
      int p0 = -1, p1 = -1, p2 = -1;
      for (int i = b; i < e && ns < 4; ++i) {
        if (!pos_flag[i]) continue;
        const int pt = obs_pt[rows[i]];
        if (pt == p0 || pt == p1 || pt == p2) continue;
        p2 = ns == 2 ? pt : p2;
        p1 = ns == 1 ? pt : p1;
        p0 = ns == 0 ? pt : p0;
        ++ns;
      }
    }
    ambiguous[g] = ns > 0 && ns < 4 ? 1 : 0;
  }
  count[g] = k;
  rep_row[g] = rows[b];
  n_inliers[g] = ok ? nin : 0;
  n_points[g] = nq;
  status[g] = st != TRI_OK ? st : ok ? TRI_OK : TRI_NO_CONSENSUS;
#pragma unroll
  for (int a = 0; a < 9; ++a) hyp[RES_HYP * g + a] = ok ? bR[a] : res_nan();
#pragma unroll
  for (int a = 0; a < 3; ++a) hyp[RES_HYP * g + 9 + a] = ok ? bt[a] : res_nan();
}

// Status 6 for the groups rig_consensus_kernel<LANES, true> flagged ambiguous: it comes before 2, 3 and 4, so it replaces
// whatever the refinement wrote (every flagged group had consensus).  The covariance kernels then leave cov NaN.
__global__ void rig_ambiguous_kernel(const unsigned char* __restrict__ ambiguous, int n_groups, int* __restrict__ status) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n_groups && ambiguous[g]) status[g] = RIG_AMBIGUOUS;
}

// J = d pi / d (r, t) of the body pose (2 x 6, pixels) from the row's J_X (normalised, 2 x 3) at B (R(r) and its right
// Jacobian, cam_prep_rot's layout): X_w = R M + t, d X_w / d r = -R [M]x Jr, so row i of J_r is -((J_X,i R) x M) Jr
__device__ __forceinline__ void rig_jq(const double* B, const double* M, const double* JX, double fx0, double* J) {
  const double* R = B + CT_R;
  const double* Jr = B + CT_JR;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    double w[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) w[a] = (JX[3 * i] * R[a] + JX[3 * i + 1] * R[3 + a] + JX[3 * i + 2] * R[6 + a]) * fx0;
    const double c0 = w[1] * M[2] - w[2] * M[1], c1 = w[2] * M[0] - w[0] * M[2], c2 = w[0] * M[1] - w[1] * M[0];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      J[6 * i + a] = -(c0 * Jr[a] + c1 * Jr[3 + a] + c2 * Jr[6 + a]);
      J[6 * i + 3 + a] = JX[3 * i + a] * fx0;
    }
  }
}

// X_w = R M + t at B (cam_prep_rot's layout)
__device__ __forceinline__ void rig_world(const double* B, const double* t, const double* M, double* X) {
  const double* R = B + CT_R;
#pragma unroll
  for (int a = 0; a < 3; ++a) X[a] = fma(R[3 * a], M[0], fma(R[3 * a + 1], M[1], fma(R[3 * a + 2], M[2], t[a])));
}

// one row's pixel residual rr (2) and J (rig_jq) at body pose B, t
__device__ __forceinline__ void rig_row_jac(const double* cam, const double* B, const double* t, const double* M,
                                            double2 px, double* rr, double* J) {
  double X[3], f[2], JX[6];
  rig_world(B, t, M, X);
  obs_res_jx(cam, X[0], X[1], X[2], px.x, px.y, 0, 1.0, f, JX);
  const double fx0 = cam[CT_FX0];
  rr[0] = f[0] * fx0;
  rr[1] = f[1] * fx0;
  rig_jq(B, M, JX, fx0, J);
}

// Cost, H = J^T J (packed, 21) and g = J^T r (6) of a group's rows [b, e) at body pose q, summed over the LANES lanes
template <int LANES>
__device__ __forceinline__ void rig_normal_eq(const double* cams, int stride, const double* q,
                                              const int* __restrict__ rows, const int* __restrict__ obs_cam,
                                              const int* __restrict__ obs_pt, const double* __restrict__ obs_px,
                                              const double* __restrict__ model, int b, int e, int lane, bool on,
                                              double (&acc)[28]) {
#pragma unroll
  for (int k = 0; k < 28; ++k) acc[k] = 0.0;
  if (on) {
    double B[CT_JR + 9];
    cam_prep_rot(q[0], q[1], q[2], B);
    for (int i = b + lane; i < e; i += LANES) {
      const int r = rows[i];
      double rr[2], J[12];
      rig_row_jac(cams + (size_t)stride * obs_cam[r], B, q + 3, model + 3 * (size_t)obs_pt[r],
                  reinterpret_cast<const double2*>(obs_px)[r], rr, J);
#pragma unroll
      for (int a = 0; a < 6; ++a) {
#pragma unroll
        for (int c = a; c < 6; ++c) acc[ut<6>(a, c)] = fma(J[a], J[c], fma(J[6 + a], J[6 + c], acc[ut<6>(a, c)]));
        acc[21 + a] = fma(J[a], rr[0], fma(J[6 + a], rr[1], acc[21 + a]));
      }
      acc[27] = fma(rr[0], rr[0], fma(rr[1], rr[1], acc[27]));
    }
  }
  group_sum<LANES>(acc);
}

// Per group with consensus (status 0 from the consensus stage), Levenberg-Marquardt (lm_iterate) over q = (r, t) on the
// consensus rows (start, rows) from the winner hyp (R to a rotation vector by res_rot_log): res_refine_kernel's loop
// with every row in its own camera.  Writes pose (the hypothesis for status 2, NaN without consensus), rmse over the
// consensus rows and status (the consensus stage's 1 and 5, else 2, 3, 4 or 0).
template <int LANES>
__global__ void __launch_bounds__(TRI_THREADS)
rig_refine_kernel(const double* __restrict__ camtab, int n_cams, int cam_in_smem, const int* __restrict__ start,
                  const int* __restrict__ rows, const int* __restrict__ obs_cam, const int* __restrict__ obs_pt,
                  const double* __restrict__ obs_px, const double* __restrict__ model, int n_groups,
                  const int* __restrict__ cstatus, const double* __restrict__ hyp, int max_iter, double xtol,
                  double* __restrict__ pose, double* __restrict__ rmse, int* __restrict__ status) {
  extern __shared__ double s_cam[];
  int stride;
  const double* cams = tri_stage_camtab(camtab, n_cams, cam_in_smem, s_cam, stride);
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  const bool live = g < n_groups;
  int st = live ? cstatus[g] : TRI_FEW_ROWS;
  const bool on = st == TRI_OK;
  const int b = on ? start[g] : 0, e = on ? start[g + 1] : 0, n = e - b;
  double q0[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (on) {
    res_rot_log(hyp + RES_HYP * g, q0);
#pragma unroll
    for (int k = 0; k < 3; ++k) q0[3 + k] = hyp[RES_HYP * g + 9 + k];
  }
  double q[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) q[k] = q0[k];
  // the sums at the current q live in shared memory, one copy per group, as in res_refine_kernel
  __shared__ double s_acc[TRI_THREADS / LANES][28];
  double* sa = s_acc[threadIdx.x / LANES];
  double cost;
  {
    double acc[28];
    rig_normal_eq<LANES>(cams, stride, q, rows, obs_cam, obs_pt, obs_px, model, b, e, lane, on, acc);
    if (on && !res_pd<6>(acc)) st = TRI_NOT_PD;
    if (lane == 0)
#pragma unroll
      for (int k = 0; k < 28; ++k) sa[k] = acc[k];
    cost = acc[27];
  }
  const double cost0 = cost;
  double tr[28];
  st = lm_iterate<6>(
      q, on && st == TRI_OK, st, max_iter, xtol,
      [&](double lam, bool on_, double* d) {
        __syncwarp();  // lane 0's last write of sa is visible
        if (!on_) return;
        double A[21], L[6][6];
#pragma unroll
        for (int k = 0; k < 21; ++k) A[k] = sa[k];
#pragma unroll
        for (int k = 0; k < 6; ++k) {
          A[ut<6>(k, k)] = sa[ut<6>(k, k)] * (1.0 + lam);
          d[k] = -sa[21 + k];
        }
        res_chol<6>(A, 0.0, L);
        res_chol_solve<6>(L, d);
      },
      [&](const double* qt, bool on_) {
        rig_normal_eq<LANES>(cams, stride, qt, rows, obs_cam, obs_pt, obs_px, model, b, e, lane, on_, tr);
        __syncwarp();  // every lane has read sa
        return tr[27] < cost;
      },
      [&] {
        if (lane == 0)
#pragma unroll
          for (int k = 0; k < 28; ++k) sa[k] = tr[k];
        cost = tr[27];
      },
      [](const double* v) {
        double s2 = 0.0;
#pragma unroll
        for (int k = 0; k < 6; ++k) s2 += v[k] * v[k];
        return sqrt(s2);
      });
  __syncwarp();  // lane 0's last write of sa is visible
  if (st == TRI_OK || st == TRI_MAX_ITER) {
    double h[21];
#pragma unroll
    for (int k = 0; k < 21; ++k) h[k] = sa[k];
    if (!res_pd<6>(h)) st = TRI_NOT_PD;
  }
  double B[CT_JR + 9];
  if (live && st == TRI_OK) cam_prep_rot(q[0], q[1], q[2], B);
  st = status_behind<LANES>(st, live, b, e, lane, [&](int i) {
    const int r = rows[i];
    bool front;
    rig_row_err2(cams, stride, B + CT_R, q + 3, r, obs_cam, obs_pt, obs_px, model, front);
    return front ? 1.0 : 0.0;
  });
  if (!live || lane != 0) return;
  const double nan = res_nan();
  const bool at_start = st == TRI_NOT_PD;
#pragma unroll
  for (int k = 0; k < 6; ++k) pose[6 * g + k] = !on ? nan : at_start ? q0[k] : q[k];
  rmse[g] = !on ? nan : sqrt((at_start ? cost0 : cost) / n);
  status[g] = st;
}

// The body pose of group g for the covariance kernels: q = pose[g] and B = cam_prep_rot(q) when `on`, zeros otherwise
__device__ __forceinline__ void rig_cov_pose(const double* __restrict__ pose, long long g, bool on, double* q,
                                             double* B) {
#pragma unroll
  for (int a = 0; a < 6; ++a) q[a] = on ? pose[6 * g + a] : 0.0;
  cam_prep_rot(q[0], q[1], q[2], B);
}

// The camera term of the covariance, per group with status 0, 3 or 4 at the refined pose q* (zero otherwise):
//   M = sum_{c,d} B_c Sigma_cd B_d^T (packed, 21 per group),  B_c = sum over the consensus rows of camera c of J_q^T J_c
//   (6 x P, pixels),  Sigma = the camera covariance at a uniform stride P.
// `rows` are the group's consensus rows sorted by camera within the group (stable), so each camera's rows are adjacent:
// the lane holding the first row of a run sums the run's B_c into Bs at that position (first = 1), three rows of it at a
// time (tri_cov_kernel's register budget); the run heads are compacted (hpos), and the lanes gather the unordered pairs
// of runs with cov_pair_gather over the 3-row halves of each B.
template <int P, int LANES>
__global__ void __launch_bounds__(TRI_THREADS)
rig_camterm_kernel(const double* __restrict__ camtab, int n_cams, int cam_in_smem, const int* __restrict__ start,
                   const int* __restrict__ rows, const int* __restrict__ obs_cam, const int* __restrict__ obs_pt,
                   const double* __restrict__ obs_px, const double* __restrict__ model, int n_groups,
                   const double* __restrict__ pose, const int* __restrict__ status, const double* __restrict__ Sig,
                   double* __restrict__ Bs, int* __restrict__ first, int* __restrict__ hpos,
                   double* __restrict__ Mout) {
  extern __shared__ double s_cam[];
  int stride;
  const double* cams = tri_stage_camtab(camtab, n_cams, cam_in_smem, s_cam, stride);
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  const bool live = g < n_groups;
  const int st = live ? status[g] : TRI_FEW_ROWS;
  const bool on = st == TRI_OK || st == TRI_MAX_ITER || st == TRI_BEHIND;
  const int b = on ? start[g] : 0, e = on ? start[g + 1] : 0;
  const int nP = n_cams * P;
  double q[6], B[CT_JR + 9];
  rig_cov_pose(pose, g, on, q, B);
  for (int i = b + lane; i < e; i += LANES) {
    const int c = obs_cam[rows[i]];
    const bool head = i == b || obs_cam[rows[i - 1]] != c;
    first[i] = head ? 1 : 0;
    if (!head) continue;
    const double* cam = cams + (size_t)stride * c;
    const double fx0 = cam[CT_FX0];
#pragma unroll 1
    for (int hh = 0; hh < 2; ++hh) {
      double Bc[3][P];
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int p = 0; p < P; ++p) Bc[a][p] = 0.0;
      for (int j = i; j < e && (j == i || obs_cam[rows[j]] == c); ++j) {
        const int rj = rows[j];
        const double* M = model + 3 * (size_t)obs_pt[rj];
        const double2 px = reinterpret_cast<const double2*>(obs_px)[rj];
        double X[3], f[2], JX[6], Jc[2 * P], J[12];
        rig_world(B, q + 3, M, X);
        obs_jac<P>(cam, X[0], X[1], X[2], px.x, px.y, 0, 1.0, f, JX, Jc);
        rig_jq(B, M, JX, fx0, J);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          const double j0 = hh ? J[3 + a] : J[a], j1 = hh ? J[9 + a] : J[6 + a];
#pragma unroll
          for (int p = 0; p < P; ++p) Bc[a][p] = fma(j0, Jc[p] * fx0, fma(j1, Jc[P + p] * fx0, Bc[a][p]));
        }
      }
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int p = 0; p < P; ++p) Bs[(size_t)i * 6 * P + (3 * hh + a) * P + p] = Bc[a][p];
    }
  }
  __syncwarp();
  // the positions of the runs' first rows, compacted per group into hpos[b ..], nh of them (the same on every lane)
  const int wl = threadIdx.x & 31;
  const unsigned gmask = LANES == 32 ? 0xffffffffu : ((1u << LANES) - 1) << (wl & ~(LANES - 1));
  int nh = 0;
  for (int base = b; __any_sync(0xffffffffu, base < e); base += LANES) {
    const int i = base + lane;
    const bool hd = i < e && first[i];
    const unsigned hm = __ballot_sync(0xffffffffu, hd) & gmask;
    if (hd) hpos[b + nh + __popc(hm & ((1u << wl) - 1))] = i;
    nh += __popc(hm);
  }
  __syncwarp();
  // M in 3 x 3 blocks: m00, m01 (m10 = m01^T), m11
  double m00[3][3], m01[3][3], m11[3][3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int c = 0; c < 3; ++c) m00[a][c] = m01[a][c] = m11[a][c] = 0.0;
  // x = B_a Sig_ab B_b^T of a pair of runs by 3 x 3 blocks hh (00, 11, 01, 10), one block per iteration; the unordered
  // pair adds its transpose too
  for (int idx = lane; idx < 4 * nh * nh; idx += LANES) {
    const int pr = idx >> 2, hh = idx & 3, ia = pr / nh, ib = pr % nh;
    const bool same = ia == ib;
    if (ib < ia || (same && hh == 3)) continue;
    const int pa = hpos[b + ia], pb = hpos[b + ib];
    const int ha = hh == 1 || hh == 3 ? 1 : 0, hb = hh == 1 || hh == 2 ? 1 : 0;
    double x[3][3];
    cov_pair_gather<P>(Bs + ((size_t)pa * 6 + 3 * ha) * P, Bs + ((size_t)pb * 6 + 3 * hb) * P, P, Sig, nP,
                       obs_cam[rows[pa]], obs_cam[rows[pb]], x);
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double d = same ? x[a][c] : x[a][c] + x[c][a];
        m00[a][c] += hh == 0 ? d : 0.0;
        m11[a][c] += hh == 1 ? d : 0.0;
        m01[a][c] += hh == 2 ? x[a][c] : hh == 3 ? x[c][a] : 0.0;
      }
  }
  double m[21];
#pragma unroll
  for (int a = 0; a < 6; ++a)
#pragma unroll
    for (int c = a; c < 6; ++c)
      m[ut<6>(a, c)] = a < 3 ? (c < 3 ? m00[a][c] : m01[a][c - 3]) : m11[a - 3][c - 3];
  group_sum<LANES>(m);
  if (!live || lane != 0) return;
#pragma unroll
  for (int a = 0; a < 21; ++a) Mout[21 * (size_t)g + a] = m[a];
}

// Per group with status 0, 3 or 4 (NaN otherwise), at the refined pose q*:
//   Sigma_q = s2 H^-1 + H^-1 M H^-1,  H = sum over the consensus rows of J_q^T J_q,  M = rig_camterm_kernel's camera term
//   (nullptr: M = 0).
template <int LANES>
__global__ void __launch_bounds__(TRI_THREADS)
rig_cov_kernel(const double* __restrict__ camtab, int n_cams, int cam_in_smem, const int* __restrict__ start,
               const int* __restrict__ rows, const int* __restrict__ obs_cam, const int* __restrict__ obs_pt,
               const double* __restrict__ obs_px, const double* __restrict__ model, int n_groups,
               const double* __restrict__ pose, const int* __restrict__ status, const double* __restrict__ Mg,
               double s2, double* __restrict__ cov) {
  extern __shared__ double s_cam[];
  int stride;
  const double* cams = tri_stage_camtab(camtab, n_cams, cam_in_smem, s_cam, stride);
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  const bool live = g < n_groups;
  const int st = live ? status[g] : TRI_FEW_ROWS;
  const bool on = st == TRI_OK || st == TRI_MAX_ITER || st == TRI_BEHIND;
  const int b = on ? start[g] : 0, e = on ? start[g + 1] : 0;
  double q[6], B[CT_JR + 9];
  rig_cov_pose(pose, g, on, q, B);
  double h[21];
#pragma unroll
  for (int a = 0; a < 21; ++a) h[a] = 0.0;
  for (int i = b + lane; i < e; i += LANES) {
    const int r = rows[i];
    double J[12], rr[2];
    rig_row_jac(cams + (size_t)stride * obs_cam[r], B, q + 3, model + 3 * (size_t)obs_pt[r],
                reinterpret_cast<const double2*>(obs_px)[r], rr, J);
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
      for (int c = a; c < 6; ++c) h[ut<6>(a, c)] = fma(J[a], J[c], fma(J[6 + a], J[6 + c], h[ut<6>(a, c)]));
  }
  group_sum<LANES>(h);
  if (!live || lane != 0) return;
  double* out = cov + 36 * (size_t)g;
  if (!on) {
    for (int a = 0; a < 36; ++a) out[a] = res_nan();
    return;
  }
  double m[21];
#pragma unroll
  for (int a = 0; a < 21; ++a) m[a] = Mg ? Mg[21 * (size_t)g + a] : 0.0;
  // H^-1 column by column, then out = s2 H^-1 + H^-1 M H^-1 (symmetrised), res_cov_kernel's tail
  double L[6][6], Hi[6][6];
  res_chol<6>(h, 0.0, L);
#pragma unroll
  for (int c = 0; c < 6; ++c) {
    double v[6];
#pragma unroll
    for (int a = 0; a < 6; ++a) v[a] = a == c ? 1.0 : 0.0;
    res_chol_solve<6>(L, v);
#pragma unroll
    for (int a = 0; a < 6; ++a) Hi[a][c] = v[a];
  }
  double T[6][6];  // M H^-1
#pragma unroll
  for (int a = 0; a < 6; ++a)
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      double v = 0.0;
#pragma unroll
      for (int j = 0; j < 6; ++j) v += m[a <= j ? ut<6>(a, j) : ut<6>(j, a)] * Hi[j][c];
      T[a][c] = v;
    }
#pragma unroll
  for (int a = 0; a < 6; ++a)
#pragma unroll
    for (int c = a; c < 6; ++c) {
      double v1 = s2 * Hi[a][c], v2 = s2 * Hi[c][a];
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        v1 += Hi[a][j] * T[j][c];
        v2 += Hi[c][j] * T[j][a];
      }
      out[6 * a + c] = out[6 * c + a] = 0.5 * (v1 + v2);
    }
}

}  // namespace cb
