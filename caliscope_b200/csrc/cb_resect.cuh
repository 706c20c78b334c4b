// Robust resection of cameras against known world points (cb_resect_robust, DESIGN.md section 4.9): per group (the rows
// of one pose of one camera), P3P hypotheses from row triples scored by MSAC over all rows, the consensus rows, then
// Levenberg-Marquardt over the pose (r, t) and its first-order covariance.  oracle/resection_robust.py states the rule.
//
// Two shapes, chosen from the rows per group:
//   * short groups (a marker cluster per frame): LANES (8 or 32) lanes per group, res_consensus_kernel builds and scores
//     every hypothesis of its group in registers and classifies the rows (tri_consensus_kernel's structure);
//   * long groups (a whole camera over a session): res_hyp_kernel writes every hypothesis to a table, res_score_kernel
//     scores (row chunk, hypothesis block) tiles with the chunk's rows in shared memory and writes one partial score per
//     (chunk, hypothesis), res_select_kernel sums the partials in chunk order and picks the winner, res_classify_kernel
//     classifies the rows.
// No floating-point atomics: every sum has a fixed order, so repeated calls give bit-identical outputs.
#pragma once
#include <cstdint>

#include "cb_device.cuh"
#include "cb_kernels.cuh"
#include "cb_triangulate.cuh"

namespace cb {

enum { RES_MULTI_CAM = 6 };
constexpr int RES_SLOTS_PER_SAMPLE = 4;  // P3P solutions per sample; slot 0 is the prior, 1 + 4 m + c sample m's c-th
constexpr int RES_DRAWS = 16;            // hashed draws of one sample before it gives up
constexpr int RES_HYP = 12;              // a hypothesis in a table: R (row-major, 9), t (3); R[0] NaN = no hypothesis
constexpr int RES_SCORE_THREADS = 128;   // hypotheses per res_score_kernel block
constexpr int RES_CHUNK = 512;           // rows per res_score_kernel block (5 doubles each in shared memory)

__device__ __forceinline__ double res_nan() { return __longlong_as_double(0x7ff8000000000000LL); }

// C(k, 3), saturated far above any max_samples
__device__ __forceinline__ long long res_triples(int k) {
  return k >= (1 << 20) ? (1LL << 62) : (long long)k * (k - 1) * (k - 2) / 6;
}

// Positions p[0] < ... < p[S-1] of candidate sample m of a group of k rows, T = C(k, S): the lexicographic rank m when
// T <= max_samples, else the first S distinct of splitmix64(m 2^32 + t) mod k, t = 0, 1, ..., sorted (false after
// RES_DRAWS draws without S).  splitmix64(x) = mix(x + 0x9e3779b97f4a7c15), tri_mix's finaliser.  Resection samples
// S = 3 rows, the relative pose S = 5 correspondences.
template <int S>
__device__ __forceinline__ bool res_sample(long long m, long long T, int max_samples, int k, int (&p)[S]) {
  if (T <= max_samples) {
    long long r = m;
    int i = -1;
#pragma unroll
    for (int s = 0; s < S; ++s) {
      for (i = i + 1;; ++i) {
        long long c = 1;  // C(k - 1 - i, S - 1 - s): the subsets with p[s] = i
#pragma unroll
        for (int q = 0; q < S - 1 - s; ++q) c = c * (k - 1 - i - q) / (q + 1);
        if (r < c) break;
        r -= c;
      }
      p[s] = i;
    }
    return true;
  }
  int got = 0;
#pragma unroll 1
  for (int t = 0; t < RES_DRAWS && got < S; ++t) {
    const int v = (int)(tri_mix(((unsigned long long)m << 32) + (unsigned long long)t, 0x9e3779b97f4a7c15ULL) %
                        (unsigned long long)k);
    bool dup = false;
#pragma unroll
    for (int q = 0; q < S; ++q) dup = dup || (q < got && p[q] == v);
    if (!dup) {
#pragma unroll
      for (int q = 0; q < S; ++q)
        if (q == got) p[q] = v;
      ++got;
    }
  }
  if (got < S) return false;
#pragma unroll
  for (int a = 1; a < S; ++a)
#pragma unroll
    for (int q = a; q > 0; --q)
      if (p[q - 1] > p[q]) {
        const int tmp = p[q];
        p[q] = p[q - 1];
        p[q - 1] = tmp;
      }
  return true;
}

// the two real roots of x^2 + b x + c (false when there are none): the larger-magnitude root first formed without
// cancellation, the other as c / it
__device__ __forceinline__ bool res_root2(double b, double c, double& r1, double& r2) {
  const double v = b * b - 4.0 * c;
  if (!(v >= 0.0)) return false;
  const double y = sqrt(v);
  const double q = b < 0.0 ? 0.5 * (-b + y) : 0.5 * (-b - y);
  r1 = q;
  r2 = c / q;
  return true;
}

// a real root of x^3 + b x^2 + c x + d (Lambda Twist's cubic): start beyond a stationary point, 50 Newton steps at most
__device__ __forceinline__ double res_cubic_root(double b, double c, double d) {
  double r0;
  if (b * b >= 3.0 * c) {
    const double v = sqrt(b * b - 3.0 * c);
    const double t1 = (-b - v) / 3.0;
    double k = ((t1 + b) * t1 + c) * t1 + d;
    if (k > 0.0) {
      r0 = t1 - sqrt(-k / (3.0 * t1 + b));
    } else {
      const double t2 = (-b + v) / 3.0;
      k = ((t2 + b) * t2 + c) * t2 + d;
      r0 = t2 + sqrt(-k / (3.0 * t2 + b));
    }
  } else {
    r0 = -b / 3.0;
    if (fabs((3.0 * r0 + 2.0 * b) * r0 + c) < 1e-4) r0 += 1.0;
  }
#pragma unroll 1
  for (int it = 0; it < 50; ++it) {
    const double fx = ((r0 + b) * r0 + c) * r0 + d;
    if (it >= 7 && !(fabs(fx) > 2.220446049250313e-16)) break;
    const double fpx = (3.0 * r0 + 2.0 * b) * r0 + c;
    r0 -= fx / fpx;
  }
  return r0;
}

// Lambda Twist P3P (Persson & Nordberg, ECCV 2018) up to the depths.  y: unit bearings (rows), x: world points (rows).
// Candidate c of 4 (the +v / -v eigen-combination times the two roots tau of its quadratic) is a solution when ok[c];
// L[c] are its depths after Gauss-Newton polishing.  The coefficients a_ij = |x_i - x_j|^2, b_ij = -2 y_i . y_j.
struct P3PDepths {
  double L[4][3];
  bool ok[4];
  double a12, a13, a23, b12, b13, b23;
};

__device__ __forceinline__ void res_p3p_depths(const double y[3][3], const double x[3][3], P3PDepths& o) {
  const double b12 = -2.0 * (y[0][0] * y[1][0] + y[0][1] * y[1][1] + y[0][2] * y[1][2]);
  const double b13 = -2.0 * (y[0][0] * y[2][0] + y[0][1] * y[2][1] + y[0][2] * y[2][2]);
  const double b23 = -2.0 * (y[1][0] * y[2][0] + y[1][1] * y[2][1] + y[1][2] * y[2][2]);
  double d12[3], d13[3], d23[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    d12[q] = x[0][q] - x[1][q];
    d13[q] = x[0][q] - x[2][q];
    d23[q] = x[1][q] - x[2][q];
  }
  const double a12 = d12[0] * d12[0] + d12[1] * d12[1] + d12[2] * d12[2];
  const double a13 = d13[0] * d13[0] + d13[1] * d13[1] + d13[2] * d13[2];
  const double a23 = d23[0] * d23[0] + d23[1] * d23[1] + d23[2] * d23[2];
  o.a12 = a12; o.a13 = a13; o.a23 = a23; o.b12 = b12; o.b13 = b13; o.b23 = b23;
  const double c31 = -0.5 * b13, c23 = -0.5 * b23, c12 = -0.5 * b12;
  const double blob = c12 * c23 * c31 - 1.0;
  const double s31 = 1.0 - c31 * c31, s23 = 1.0 - c23 * c23, s12 = 1.0 - c12 * c12;
  double p3 = a13 * (a23 * s31 - a13 * s23);
  double p2 = 2.0 * blob * a23 * a13 + a13 * (2.0 * a12 + a13) * s23 + a23 * (a23 - a12) * s31;
  double p1 = a23 * (a13 - a23) * s12 - a12 * a12 * s23 - 2.0 * a12 * (blob * a23 + a13 * s23);
  double p0 = a12 * (a12 * s23 - a23 * s12);
  p3 = 1.0 / p3;
  p2 *= p3; p1 *= p3; p0 *= p3;
  const double g = res_cubic_root(p2, p1, p0);
  // the 3x3 A(g) (rank 2) and its two non-zero eigenpairs, larger magnitude first
  const double A00 = a23 * (1.0 - g), A01 = (a23 * b12) * 0.5, A02 = (a23 * b13 * g) * (-0.5);
  const double A11 = a23 - a12 + a13 * g, A12 = b23 * (a13 * g - a12) * 0.5, A22 = g * (a13 - a23) - a12;
  const double eb = -A00 - A11 - A22;
  const double ec = -A01 * A01 - A02 * A02 - A12 * A12 + A00 * (A11 + A22) + A11 * A22;
  double e1 = 0.0, e2 = 0.0;
  const bool eig_ok = res_root2(eb, ec, e1, e2);
  if (fabs(e1) < fabs(e2)) {
    const double tmp = e1;
    e1 = e2;
    e2 = tmp;
  }
  const double mx0011 = -A00 * A11;
  const double prec0 = A01 * A12 - A02 * A11, prec1 = A01 * A02 - A00 * A12;
  double V[3][2];
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const double e = q ? e2 : e1;
    const double tmp = 1.0 / (e * (A00 + A11) + mx0011 - e * e + A01 * A01);
    double v0 = -(e * A02 + prec0) * tmp, v1 = -(e * A12 + prec1) * tmp;
    const double rn = 1.0 / sqrt(v0 * v0 + v1 * v1 + 1.0);
    V[0][q] = v0 * rn;
    V[1][q] = v1 * rn;
    V[2][q] = rn;
  }
  const double v = sqrt(fmax(0.0, -e2 / e1));
#pragma unroll
  for (int sgn = 0; sgn < 2; ++sgn) {
    const double s = sgn ? -v : v;
    const double w2 = 1.0 / (s * V[0][1] - V[0][0]);
    const double w0 = (V[1][0] - s * V[1][1]) * w2;
    const double w1 = (V[2][0] - s * V[2][1]) * w2;
    const double a = 1.0 / ((a13 - a12) * w1 * w1 - a12 * b13 * w1 - a12);
    const double bq = (a13 * b12 * w1 - a12 * b13 * w0 - 2.0 * w0 * w1 * (a12 - a13)) * a;
    const double cq = ((a13 - a12) * w0 * w0 + a13 * b12 * w0 + a13) * a;
    double tau[2] = {0.0, 0.0};
    const bool real = eig_ok && res_root2(bq, cq, tau[0], tau[1]);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int c = 2 * sgn + r;
      const double tq = tau[r];
      const double d = a23 / (tq * (b23 + tq) + 1.0);
      const double l2 = sqrt(d), l3 = tq * l2, l1 = w0 * l2 + w1 * l3;
      o.ok[c] = real && tq > 0.0 && d > 0.0 && l1 >= 0.0;
      o.L[c][0] = l1; o.L[c][1] = l2; o.L[c][2] = l3;
    }
  }
  // Gauss-Newton on the three distance equations l_i^2 + l_j^2 + b_ij l_i l_j = a_ij, 5 steps at most, a step kept only
  // when it does not raise the sum of absolute residuals
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    if (!o.ok[c]) continue;
    double l1 = o.L[c][0], l2 = o.L[c][1], l3 = o.L[c][2];
#pragma unroll 1
    for (int it = 0; it < 5; ++it) {
      const double r1 = l1 * l1 + l2 * l2 + b12 * l1 * l2 - a12;
      const double r2 = l1 * l1 + l3 * l3 + b13 * l1 * l3 - a13;
      const double r3 = l2 * l2 + l3 * l3 + b23 * l2 * l3 - a23;
      const double rs = fabs(r1) + fabs(r2) + fabs(r3);
      if (rs < 1e-10) break;
      const double v0 = 2.0 * l1 + b12 * l2, v1 = 2.0 * l2 + b12 * l1;
      const double v3 = 2.0 * l1 + b13 * l3, v5 = 2.0 * l3 + b13 * l1;
      const double v7 = 2.0 * l2 + b23 * l3, v8 = 2.0 * l3 + b23 * l2;
      const double det = 1.0 / (-v0 * v5 * v7 - v1 * v3 * v8);
      const double n1 = l1 - det * (-v5 * v7 * r1 - v1 * v8 * r2 + v1 * v5 * r3);
      const double n2 = l2 - det * (-v3 * v8 * r1 + v0 * v8 * r2 - v0 * v5 * r3);
      const double n3 = l3 - det * (v3 * v7 * r1 - v0 * v7 * r2 - v1 * v3 * r3);
      const double q1 = n1 * n1 + n2 * n2 + b12 * n1 * n2 - a12;
      const double q2 = n1 * n1 + n3 * n3 + b13 * n1 * n3 - a13;
      const double q3 = n2 * n2 + n3 * n3 + b23 * n2 * n3 - a23;
      if (fabs(q1) + fabs(q2) + fabs(q3) > rs) break;
      l1 = n1; l2 = n2; l3 = n3;
    }
    o.L[c][0] = l1; o.L[c][1] = l2; o.L[c][2] = l3;
  }
}

// the pose of depths l: R = Y X^-1 with X = [x1-x2, x1-x3, (x1-x2) x (x1-x3)] and Y the same of the camera-frame points
// l_i y_i; t = l_1 y_1 - R x_1.  Xi = X^-1 (row-major).  Returns whether R, t are finite and the three points have
// Xc.z > 0.
__device__ __forceinline__ bool res_p3p_pose(const double y[3][3], const double x[3][3], const double Xi[9],
                                             const double* l, double* R, double* t) {
  double p[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int q = 0; q < 3; ++q) p[i][q] = y[i][q] * l[i];
  double u[3], w[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    u[q] = p[0][q] - p[1][q];
    w[q] = p[0][q] - p[2][q];
  }
  const double uw[3] = {u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0]};
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) R[3 * i + j] = u[i] * Xi[j] + w[i] * Xi[3 + j] + uw[i] * Xi[6 + j];
  bool ok = true;
#pragma unroll
  for (int i = 0; i < 3; ++i) t[i] = p[0][i] - (R[3 * i] * x[0][0] + R[3 * i + 1] * x[0][1] + R[3 * i + 2] * x[0][2]);
#pragma unroll
  for (int i = 0; i < 9; ++i) ok = ok && isfinite(R[i]);
#pragma unroll
  for (int i = 0; i < 3; ++i) ok = ok && isfinite(t[i]);
#pragma unroll
  for (int i = 0; i < 3; ++i) ok = ok && (R[6] * x[i][0] + R[7] * x[i][1] + R[8] * x[i][2] + t[2]) > 0.0;
  return ok;
}

// inverse of the world-side matrix X of res_p3p_pose (row-major)
__device__ __forceinline__ void res_p3p_xinv(const double x[3][3], double Xi[9]) {
  double a[3], b[3];
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    a[q] = x[0][q] - x[1][q];
    b[q] = x[0][q] - x[2][q];
  }
  const double c[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
  // X columns a, b, c: X = [[a0 b0 c0], [a1 b1 c1], [a2 b2 c2]]; X^-1 rows = (b x c, c x a, a x b) / det
  const double det = a[0] * (b[1] * c[2] - b[2] * c[1]) - b[0] * (a[1] * c[2] - a[2] * c[1]) + c[0] * (a[1] * b[2] - a[2] * b[1]);
  const double id = 1.0 / det;
  Xi[0] = (b[1] * c[2] - b[2] * c[1]) * id; Xi[1] = (b[2] * c[0] - b[0] * c[2]) * id; Xi[2] = (b[0] * c[1] - b[1] * c[0]) * id;
  Xi[3] = (c[1] * a[2] - c[2] * a[1]) * id; Xi[4] = (c[2] * a[0] - c[0] * a[2]) * id; Xi[5] = (c[0] * a[1] - c[1] * a[0]) * id;
  Xi[6] = (a[1] * b[2] - a[2] * b[1]) * id; Xi[7] = (a[2] * b[0] - a[0] * b[2]) * id; Xi[8] = (a[0] * b[1] - a[1] * b[0]) * id;
}

// The inputs of one sample of a group: bearings of the float32-rounded undistorted coordinates and the world points of
// rows (rows[b + i], rows[b + j], rows[b + l]).  False when a point is not finite (an unusable row).
__device__ __forceinline__ bool res_sample_inputs(const int* __restrict__ rows, const int* __restrict__ obs_pt,
                                                  const double* __restrict__ obs_xy, const double* __restrict__ pts,
                                                  int b, int i, int j, int l, double y[3][3], double x[3][3]) {
  bool ok = true;
#pragma unroll
  for (int s = 0; s < 3; ++s) {
    const int r = rows[b + (s == 0 ? i : s == 1 ? j : l)];
    const double2 n = reinterpret_cast<const double2*>(obs_xy)[r];
    const double in = 1.0 / sqrt(n.x * n.x + n.y * n.y + 1.0);
    y[s][0] = n.x * in; y[s][1] = n.y * in; y[s][2] = in;
    const double* X = pts + 3 * (size_t)obs_pt[r];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      x[s][q] = X[q];
      ok = ok && isfinite(X[q]);
    }
  }
  return ok;
}

// squared pixel error of a row at pose (R, t) with the intrinsics of the camera table entry `cam` (the engine's
// projection; project_obs reads R and t from the entry, so they replace the entry's own in registers); front: Xc.z > 0
__device__ __forceinline__ double res_row_err2(const double* cam, const double* R, const double* t, double X0, double X1,
                                               double X2, double2 px, bool& front) {
  double E[CT_SIZE];
#pragma unroll
  for (int q = 0; q < CT_SIZE; ++q) E[q] = cam[q];
#pragma unroll
  for (int q = 0; q < 9; ++q) E[CT_R + q] = R[q];
#pragma unroll
  for (int q = 0; q < 3; ++q) E[CT_T + q] = t[q];
  ProjOut o;
  project_obs<false>(E, (((int)cam[CT_FLAGS]) & 2) != 0, X0, X1, X2, o);
  front = o.Xc[2] > 0.0;
  const double du = o.u - px.x, dv = o.v - px.y;
  return du * du + dv * dv;
}

// MSAC score of pose (R, t) over rows [b, e): sum of min(e_r^2, tau^2), tau^2 for a row behind the camera, with a
// non-finite error or an unusable point
__device__ __forceinline__ double res_score_rows(const double* cam, const double* R, const double* t,
                                                 const int* __restrict__ rows, const int* __restrict__ obs_pt,
                                                 const double* __restrict__ obs_px, const double* __restrict__ pts, int b,
                                                 int e, double tau2) {
  double score = 0.0;
  for (int p = b; p < e; ++p) {
    const int r = rows[p];
    const double* X = pts + 3 * (size_t)obs_pt[r];
    bool front;
    const double e2 = res_row_err2(cam, R, t, X[0], X[1], X[2], reinterpret_cast<const double2*>(obs_px)[r], front);
    score += msac_term(front, e2, tau2);
  }
  return score;
}

// The camera of a group (its first row's) and whether another camera appears in it, the same on every lane
template <int LANES>
__device__ __forceinline__ int res_group_cam(const int* __restrict__ rows, const int* __restrict__ obs_cam, int b, int e,
                                             int lane, bool live, bool& multi) {
  const int c0 = live && e > b ? obs_cam[rows[b]] : 0;
  int m = 0;
  for (int i = b + lane; i < e; i += LANES) m |= obs_cam[rows[i]] != c0;
  m = group_or<LANES>(m);
  multi = m != 0;
  return c0;
}

// consensus_classify at the winner (R, t) (found: there is one), then the group's outputs: lane 0 writes cam, count,
// rep_row, n_inliers, status (6, 1, 5 or 0) and the winner (NaN without consensus).
template <int LANES>
__device__ __forceinline__ void res_classify(const double* cam, const double* R, const double* t, bool found, int st,
                                             int c0, const int* __restrict__ rows, const int* __restrict__ obs_pt,
                                             const double* __restrict__ obs_px, const double* __restrict__ pts, int b,
                                             int e, int lane, bool live, long long g, double tau2, int min_inliers,
                                             double* __restrict__ hyp, int* __restrict__ cam_out, int* __restrict__ count,
                                             int* __restrict__ rep_row, int* __restrict__ n_inliers,
                                             int* __restrict__ status, unsigned char* __restrict__ pos_flag,
                                             unsigned char* __restrict__ inlier) {
  int nin;
  const bool ok = consensus_classify<LANES>(
      found, rows, b, e, lane, tau2, min_inliers,
      [&](int r, bool& front) {
        const double* X = pts + 3 * (size_t)obs_pt[r];
        return res_row_err2(cam, R, t, X[0], X[1], X[2], reinterpret_cast<const double2*>(obs_px)[r], front);
      },
      pos_flag, inlier, nin);
  if (!live || lane != 0) return;
  cam_out[g] = c0;
  count[g] = e - b;
  rep_row[g] = rows[b];
  n_inliers[g] = ok ? nin : 0;
  status[g] = st != TRI_OK ? st : ok ? TRI_OK : TRI_NO_CONSENSUS;
#pragma unroll
  for (int q = 0; q < 9; ++q) hyp[RES_HYP * g + q] = ok ? R[q] : res_nan();
#pragma unroll
  for (int q = 0; q < 3; ++q) hyp[RES_HYP * g + 9 + q] = ok ? t[q] : res_nan();
}

// status before any hypothesis: 6 several cameras, 1 fewer than 4 rows, else 0
__device__ __forceinline__ int res_pre_status(bool multi, int k) {
  return multi ? RES_MULTI_CAM : k < 4 ? TRI_FEW_ROWS : TRI_OK;
}

// ---- short groups ---------------------------------------------------------------------------------------------------
// One group per LANES lanes.  Task 0 is the prior (the camera's pose in the table, when use_prior), task 1 + m sample m;
// the lanes stride over the tasks, each scores its task's hypotheses over all k rows and keeps the lowest score (slots
// increase along a lane's tasks, so the first of equal scores stays).  An xor butterfly over (score, slot) picks the
// winner (group_argmin), which reaches the group's lanes by shuffle from the lane that owns its task; then res_classify.
template <int LANES>
__global__ void __launch_bounds__(TRI_THREADS)
res_consensus_kernel(const double* __restrict__ camtab, const int* __restrict__ start, const int* __restrict__ rows,
                     const int* __restrict__ obs_cam, const int* __restrict__ obs_pt, const double* __restrict__ obs_xy,
                     const double* __restrict__ obs_px, const double* __restrict__ pts, int n_groups, double tau,
                     int min_inliers, int max_samples, int use_prior, double* __restrict__ hyp, int* __restrict__ cam_out,
                     int* __restrict__ count, int* __restrict__ rep_row, int* __restrict__ n_inliers,
                     int* __restrict__ status, unsigned char* __restrict__ pos_flag, unsigned char* __restrict__ inlier) {
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  const bool live = g < n_groups;
  const int b = live ? start[g] : 0, e = live ? start[g + 1] : 0, k = e - b;
  bool multi;
  const int c0 = res_group_cam<LANES>(rows, obs_cam, b, e, lane, live, multi);
  const int st = res_pre_status(multi, k);
  const double* cam = camtab + (size_t)CT_SIZE * c0;
  const double tau2 = tau * tau;
  const double inf = __longlong_as_double(0x7ff0000000000000LL);
  const long long T = res_triples(k);
  const long long ntask = (live && st == TRI_OK) ? 1 + (T < max_samples ? T : (long long)max_samples) : 0;
  double best = inf, bR[9], bt[3];
#pragma unroll
  for (int q = 0; q < 9; ++q) bR[q] = 0.0;
#pragma unroll
  for (int q = 0; q < 3; ++q) bt[q] = 0.0;
  long long best_s = 0x7fffffffffffffffLL;
  for (long long task = lane; task < ntask; task += LANES) {
    if (task == 0) {
      if (!use_prior) continue;
      double R[9], t[3];
#pragma unroll
      for (int q = 0; q < 9; ++q) R[q] = cam[CT_R + q];
#pragma unroll
      for (int q = 0; q < 3; ++q) t[q] = cam[CT_T + q];
      const double sc = res_score_rows(cam, R, t, rows, obs_pt, obs_px, pts, b, e, tau2);
      if (sc < best) {
        best = sc;
        best_s = 0;
#pragma unroll
        for (int q = 0; q < 9; ++q) bR[q] = R[q];
#pragma unroll
        for (int q = 0; q < 3; ++q) bt[q] = t[q];
      }
      continue;
    }
    const long long m = task - 1;
    int p[3];
    if (!res_sample<3>(m, T, max_samples, k, p)) continue;
    double y[3][3], x[3][3];
    if (!res_sample_inputs(rows, obs_pt, obs_xy, pts, b, p[0], p[1], p[2], y, x)) continue;
    P3PDepths d;
    res_p3p_depths(y, x, d);
    double Xi[9];
    res_p3p_xinv(x, Xi);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if (!d.ok[c]) continue;
      double R[9], t[3];
      if (!res_p3p_pose(y, x, Xi, d.L[c], R, t)) continue;
      const double sc = res_score_rows(cam, R, t, rows, obs_pt, obs_px, pts, b, e, tau2);
      if (sc < best) {
        best = sc;
        best_s = 1 + RES_SLOTS_PER_SAMPLE * m + c;
#pragma unroll
        for (int q = 0; q < 9; ++q) bR[q] = R[q];
#pragma unroll
        for (int q = 0; q < 3; ++q) bt[q] = t[q];
      }
    }
  }
  group_argmin<LANES>(best, best_s);
  const bool found = best < inf;
  const long long task = found ? (best_s == 0 ? 0 : 1 + (best_s - 1) / RES_SLOTS_PER_SAMPLE) : 0;
  const int owner = (int)(task % LANES);
  group_bcast<LANES>(bR, owner);
  group_bcast<LANES>(bt, owner);
  res_classify<LANES>(cam, bR, bt, found, st, c0, rows, obs_pt, obs_px, pts, b, e, lane, live, g, tau2, min_inliers, hyp,
                      cam_out, count, rep_row, n_inliers, status, pos_flag, inlier);
}

// ---- long groups ----------------------------------------------------------------------------------------------------
// Thread (group, task) of a flat index over n_groups x (1 + max_samples): writes the hypothesis table tab[g][slot][12]
// (S = 1 + 4 max_samples slots per group) for its task's slots, R[0] = NaN where there is no hypothesis.
__global__ void res_hyp_kernel(const double* __restrict__ camtab, const int* __restrict__ start,
                               const int* __restrict__ rows, const int* __restrict__ obs_cam,
                               const int* __restrict__ obs_pt, const double* __restrict__ obs_xy,
                               const double* __restrict__ pts, int n_groups, int max_samples, int use_prior,
                               double* __restrict__ tab) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long ntask = 1 + (long long)max_samples;
  if (idx >= (long long)n_groups * ntask) return;
  const long long g = idx / ntask, task = idx % ntask;
  const int b = start[g], e = start[g + 1], k = e - b;
  const long long S = 1 + (long long)RES_SLOTS_PER_SAMPLE * max_samples;
  const double nan = res_nan();
  if (task == 0) {
    double* o = tab + (size_t)RES_HYP * (size_t)(g * S);
    const double* cam = camtab + (size_t)CT_SIZE * obs_cam[rows[b]];
    const bool on = use_prior && k >= 4;
#pragma unroll
    for (int q = 0; q < 9; ++q) o[q] = on ? cam[CT_R + q] : nan;
#pragma unroll
    for (int q = 0; q < 3; ++q) o[9 + q] = on ? cam[CT_T + q] : nan;
    return;
  }
  const long long m = task - 1;
  double* o = tab + (size_t)RES_HYP * (size_t)(g * S + 1 + RES_SLOTS_PER_SAMPLE * m);
  const long long T = res_triples(k);
  bool any = false;
  int p[3];
  double y[3][3], x[3][3];
  if (k >= 4 && m < T && res_sample<3>(m, T, max_samples, k, p) &&
      res_sample_inputs(rows, obs_pt, obs_xy, pts, b, p[0], p[1], p[2], y, x)) {
    any = true;
    P3PDepths d;
    res_p3p_depths(y, x, d);
    double Xi[9];
    res_p3p_xinv(x, Xi);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      double R[9], t[3];
      const bool ok = d.ok[c] && res_p3p_pose(y, x, Xi, d.L[c], R, t);
#pragma unroll
      for (int q = 0; q < 9; ++q) o[RES_HYP * c + q] = ok ? R[q] : nan;
#pragma unroll
      for (int q = 0; q < 3; ++q) o[RES_HYP * c + 9 + q] = ok ? t[q] : nan;
    }
  }
  if (!any)
    for (int c = 0; c < 4; ++c) o[RES_HYP * c] = nan;
}

// One block per (row chunk, block of RES_SCORE_THREADS slots): the chunk's points and pixels go to shared memory, each
// thread scores its slot's hypothesis over them in row order and writes part[chunk][slot] (+inf: no hypothesis).  The
// chunks of group g are chunk_off[g] .. chunk_off[g + 1] - 1, RES_CHUNK rows each from the group's start.
__global__ void __launch_bounds__(RES_SCORE_THREADS)
res_score_kernel(const double* __restrict__ camtab, const int* __restrict__ start, const int* __restrict__ chunk_off,
                 const int* __restrict__ rows, const int* __restrict__ obs_cam, const int* __restrict__ obs_pt,
                 const double* __restrict__ obs_px, const double* __restrict__ pts, int n_groups, int S,
                 const double* __restrict__ tab, double tau, double* __restrict__ part) {
  __shared__ double s_row[RES_CHUNK * 5];
  const int chunk = blockIdx.x;
  int lo = 0, hi = n_groups;  // the group of the chunk: the last g with chunk_off[g] <= chunk
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (chunk_off[mid] <= chunk) lo = mid;
    else hi = mid;
  }
  const int g = lo;
  const int b = start[g] + (chunk - chunk_off[g]) * RES_CHUNK, e = min(start[g + 1], b + RES_CHUNK), n = e - b;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int r = rows[b + i];
    const double* X = pts + 3 * (size_t)obs_pt[r];
    const double2 px = reinterpret_cast<const double2*>(obs_px)[r];
    s_row[5 * i + 0] = X[0]; s_row[5 * i + 1] = X[1]; s_row[5 * i + 2] = X[2];
    s_row[5 * i + 3] = px.x; s_row[5 * i + 4] = px.y;
  }
  __syncthreads();
  const int s = blockIdx.y * RES_SCORE_THREADS + threadIdx.x;
  if (s >= S) return;
  const double* h = tab + (size_t)RES_HYP * ((size_t)g * S + s);
  const double tau2 = tau * tau;
  double score = __longlong_as_double(0x7ff0000000000000LL);
  if (!isnan(h[0])) {
    const double* cam = camtab + (size_t)CT_SIZE * obs_cam[rows[start[g]]];
    double R[9], t[3];
#pragma unroll
    for (int q = 0; q < 9; ++q) R[q] = h[q];
#pragma unroll
    for (int q = 0; q < 3; ++q) t[q] = h[9 + q];
    score = 0.0;
    for (int i = 0; i < n; ++i) {
      bool front;
      const double* v = s_row + 5 * i;
      const double e2 = res_row_err2(cam, R, t, v[0], v[1], v[2], make_double2(v[3], v[4]), front);
      score += msac_term(front, e2, tau2);
    }
  }
  part[(size_t)chunk * S + s] = score;
}

// One block per group: the score of each slot is the sum of its partials in chunk order; the lowest wins, the lowest
// slot on a tie.  best[g] = the winning slot, -1 when no slot has a hypothesis.
__global__ void __launch_bounds__(RES_SCORE_THREADS)
res_select_kernel(const int* __restrict__ chunk_off, int S, const double* __restrict__ part, int* __restrict__ best) {
  __shared__ double s_sc[RES_SCORE_THREADS];
  __shared__ int s_sl[RES_SCORE_THREADS];
  const int g = blockIdx.x;
  const int c0 = chunk_off[g], c1 = chunk_off[g + 1];
  const double inf = __longlong_as_double(0x7ff0000000000000LL);
  double bs = inf;
  int bsl = 0x7fffffff;
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    double sc = 0.0;
    for (int c = c0; c < c1; ++c) sc += part[(size_t)c * S + s];
    if (sc < bs) {
      bs = sc;
      bsl = s;
    }
  }
  s_sc[threadIdx.x] = bs;
  s_sl[threadIdx.x] = bsl;
  __syncthreads();
  for (int w = RES_SCORE_THREADS / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) {
      const double o = s_sc[threadIdx.x + w];
      const int os = s_sl[threadIdx.x + w];
      if (o < s_sc[threadIdx.x] || (o == s_sc[threadIdx.x] && os < s_sl[threadIdx.x])) {
        s_sc[threadIdx.x] = o;
        s_sl[threadIdx.x] = os;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) best[g] = s_sc[0] < inf ? s_sl[0] : -1;
}

// The classification of the long shape: one group per 32 lanes, the winner read from the hypothesis table
__global__ void __launch_bounds__(TRI_THREADS)
res_classify_kernel(const double* __restrict__ camtab, const int* __restrict__ start, const int* __restrict__ rows,
                    const int* __restrict__ obs_cam, const int* __restrict__ obs_pt, const double* __restrict__ obs_px,
                    const double* __restrict__ pts, int n_groups, int S, const double* __restrict__ tab,
                    const int* __restrict__ best, double tau, int min_inliers, double* __restrict__ hyp,
                    int* __restrict__ cam_out, int* __restrict__ count, int* __restrict__ rep_row,
                    int* __restrict__ n_inliers, int* __restrict__ status, unsigned char* __restrict__ pos_flag,
                    unsigned char* __restrict__ inlier) {
  constexpr int LANES = 32;
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  const bool live = g < n_groups;
  const int b = live ? start[g] : 0, e = live ? start[g + 1] : 0;
  bool multi;
  const int c0 = res_group_cam<LANES>(rows, obs_cam, b, e, lane, live, multi);
  const int st = res_pre_status(multi, e - b);
  const int w = live ? best[g] : -1;
  const bool found = st == TRI_OK && w >= 0;
  double R[9], t[3];
  const double* h = tab + (size_t)RES_HYP * ((size_t)g * S + (found ? w : 0));
#pragma unroll
  for (int q = 0; q < 9; ++q) R[q] = found ? h[q] : 0.0;
#pragma unroll
  for (int q = 0; q < 3; ++q) t[q] = found ? h[9 + q] : 0.0;
  res_classify<LANES>(camtab + (size_t)CT_SIZE * c0, R, t, found, st, c0, rows, obs_pt, obs_px, pts, b, e, lane, live, g,
                      tau * tau, min_inliers, hyp, cam_out, count, rep_row, n_inliers, status, pos_flag, inlier);
}

// chunks of every group (res_score_kernel), n_groups + 1 entries with a zero past the end for the scan
__global__ void res_chunks_kernel(const int* __restrict__ start, int n_groups, int* __restrict__ nchunk) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n_groups) nchunk[g] = max(1, (start[g + 1] - start[g] + RES_CHUNK - 1) / RES_CHUNK);
  if (g == n_groups) nchunk[g] = 0;
}

// ---- refinement and covariance ----------------------------------------------------------------------------------------
// rotation vector of R with theta in [0, pi] (cv2.Rodrigues' matrix-to-vector branch, without its SVD
// re-orthonormalisation)
__device__ __forceinline__ void res_rot_log(const double* R, double* r) {
  double rx = R[7] - R[5], ry = R[2] - R[6], rz = R[3] - R[1];
  const double s = sqrt((rx * rx + ry * ry + rz * rz) * 0.25);
  double c = (R[0] + R[4] + R[8] - 1.0) * 0.5;
  c = c > 1.0 ? 1.0 : c < -1.0 ? -1.0 : c;
  const double th = acos(c);
  if (s < 1e-5) {
    if (c > 0.0) {
      rx = ry = rz = 0.0;
    } else {
      rx = sqrt(fmax((R[0] + 1.0) * 0.5, 0.0));
      ry = sqrt(fmax((R[4] + 1.0) * 0.5, 0.0)) * (R[1] < 0.0 ? -1.0 : 1.0);
      rz = sqrt(fmax((R[8] + 1.0) * 0.5, 0.0)) * (R[2] < 0.0 ? -1.0 : 1.0);
      if (fabs(rx) < fabs(ry) && fabs(rx) < fabs(rz) && ((R[5] > 0.0) != (ry * rz > 0.0))) rz = -rz;
      const double sc = th / sqrt(rx * rx + ry * ry + rz * rz);
      rx *= sc; ry *= sc; rz *= sc;
    }
  } else {
    const double v = th / (2.0 * s);
    rx *= v; ry *= v; rz *= v;
  }
  r[0] = rx; r[1] = ry; r[2] = rz;
}

// camera table entry of pose q = (r, t) with the intrinsics of entry `cam`
__device__ __forceinline__ void res_entry(const double* cam, const double* q, double* E) {
#pragma unroll
  for (int i = 0; i < CT_SIZE; ++i) E[i] = cam[i];
  cam_prep_rot(q[0], q[1], q[2], E);
  E[CT_T + 0] = q[3]; E[CT_T + 1] = q[4]; E[CT_T + 2] = q[5];
}

// one row's pixel residual r (2) and derivative J = d pi / d (r, t) (2 x 6) at entry E
__device__ __forceinline__ void res_row_jac(const double* E, const double* X, double2 px, double* rr, double* J,
                                            double* JX) {
  double f[2], Jc[12];
  obs_jac<6>(E, X[0], X[1], X[2], px.x, px.y, 0, 1.0, f, JX, Jc);
  const double fx0 = E[CT_FX0];
  rr[0] = f[0] * fx0;
  rr[1] = f[1] * fx0;
#pragma unroll
  for (int q = 0; q < 12; ++q) J[q] = Jc[q] * fx0;
#pragma unroll
  for (int q = 0; q < 6; ++q) JX[q] *= fx0;
}

// Cost, H = J^T J (packed, 21) and g = J^T r (6) of a group's rows [b, e) of `rows` at pose q, summed over the LANES lanes
template <int LANES>
__device__ __forceinline__ void res_normal_eq(const double* cam, const double* q, const int* __restrict__ rows,
                                              const int* __restrict__ obs_pt, const double* __restrict__ obs_px,
                                              const double* __restrict__ pts, int b, int e, int lane, bool on,
                                              double (&acc)[28]) {
#pragma unroll
  for (int k = 0; k < 28; ++k) acc[k] = 0.0;
  if (on) {
    double E[CT_SIZE];
    res_entry(cam, q, E);
    for (int i = b + lane; i < e; i += LANES) {
      const int r = rows[i];
      double rr[2], J[12], JX[6];
      res_row_jac(E, pts + 3 * (size_t)obs_pt[r], reinterpret_cast<const double2*>(obs_px)[r], rr, J, JX);
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

// Cholesky factor L (row-major lower, N x N) of packed symmetric h; returns whether every pivot exceeds `thr`
template <int N>
__device__ __forceinline__ bool res_chol(const double* h, double thr, double L[N][N]) {
  bool ok = true;
#pragma unroll
  for (int j = 0; j < N; ++j) {
    double d = h[ut<N>(j, j)];
#pragma unroll
    for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k];
    ok = ok && d > thr;
    L[j][j] = sqrt(d);
    const double il = 1.0 / L[j][j];
#pragma unroll
    for (int i = j + 1; i < N; ++i) {
      double v = h[ut<N>(j, i)];
#pragma unroll
      for (int k = 0; k < j; ++k) v -= L[i][k] * L[j][k];
      L[i][j] = v * il;
    }
#pragma unroll
    for (int i = 0; i < j; ++i) L[i][j] = 0.0;
  }
  return ok;
}

// H positive definite: every Cholesky pivot of the Jacobi-scaled D^-1/2 H D^-1/2 above TRI_PD_RTOL (radians and metres
// mix in H, so the raw pivots have no common scale)
template <int N>
__device__ __forceinline__ bool res_pd(const double* h) {
  double s[N], hs[N * (N + 1) / 2], L[N][N];
#pragma unroll
  for (int i = 0; i < N; ++i) s[i] = 1.0 / sqrt(h[ut<N>(i, i)]);
#pragma unroll
  for (int i = 0; i < N; ++i)
#pragma unroll
    for (int j = i; j < N; ++j) hs[ut<N>(i, j)] = h[ut<N>(i, j)] * s[i] * s[j];
  return res_chol<N>(hs, TRI_PD_RTOL, L);
}

// (L L^T) x = v in place
template <int N>
__device__ __forceinline__ void res_chol_solve(const double L[N][N], double* v) {
#pragma unroll
  for (int i = 0; i < N; ++i) {
    double a = v[i];
#pragma unroll
    for (int k = 0; k < i; ++k) a -= L[i][k] * v[k];
    v[i] = a / L[i][i];
  }
#pragma unroll
  for (int i = N - 1; i >= 0; --i) {
    double a = v[i];
#pragma unroll
    for (int k = i + 1; k < N; ++k) a -= L[k][i] * v[k];
    v[i] = a / L[i][i];
  }
}

// Per group with consensus (status 0 from the consensus stage), Levenberg-Marquardt (lm_iterate) over q = (r, t) on the
// consensus rows (start, rows) from the winner hyp (R to a rotation vector by res_rot_log).  Writes pose (the hypothesis for status 2, NaN
// without consensus), rmse over the consensus rows and status (the consensus stage's 1, 5, 6, else 2, 3, 4 or 0).
template <int LANES>
__global__ void __launch_bounds__(TRI_THREADS)
res_refine_kernel(const double* __restrict__ camtab, const int* __restrict__ start, const int* __restrict__ rows,
                  const int* __restrict__ obs_pt, const double* __restrict__ obs_px, const double* __restrict__ pts,
                  int n_groups, const int* __restrict__ cam, const int* __restrict__ cstatus,
                  const double* __restrict__ hyp, int max_iter, double xtol, double* __restrict__ pose,
                  double* __restrict__ rmse, int* __restrict__ status) {
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  const bool live = g < n_groups;
  int st = live ? cstatus[g] : TRI_FEW_ROWS;
  const bool on = st == TRI_OK;
  const int b = on ? start[g] : 0, e = on ? start[g + 1] : 0, n = e - b;
  const double* ce = camtab + (size_t)CT_SIZE * (on ? cam[g] : 0);
  double q0[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (on) {
    res_rot_log(hyp + RES_HYP * g, q0);
#pragma unroll
    for (int k = 0; k < 3; ++k) q0[3 + k] = hyp[RES_HYP * g + 9 + k];
  }
  double q[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) q[k] = q0[k];
  // the sums at the current q live in shared memory, one copy per group (every lane holds the same values), which keeps
  // the trial's sums and the row loop in registers
  __shared__ double s_acc[TRI_THREADS / LANES][28];
  double* sa = s_acc[threadIdx.x / LANES];
  double cost;
  {
    double acc[28];
    res_normal_eq<LANES>(ce, q, rows, obs_pt, obs_px, pts, b, e, lane, on, acc);
    if (on && !res_pd<6>(acc)) st = TRI_NOT_PD;
    if (lane == 0)
#pragma unroll
      for (int k = 0; k < 28; ++k) sa[k] = acc[k];
    cost = acc[27];
  }
  const double cost0 = cost;
  double tr[28];  // the sums at the trial pose
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
        res_normal_eq<LANES>(ce, qt, rows, obs_pt, obs_px, pts, b, e, lane, on_, tr);
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
  if ((st == TRI_OK || st == TRI_MAX_ITER)) {
    double h[21];
#pragma unroll
    for (int k = 0; k < 21; ++k) h[k] = sa[k];
    if (!res_pd<6>(h)) st = TRI_NOT_PD;
  }
  double E[CT_SIZE];
  if (live && st == TRI_OK) res_entry(ce, q, E);
  st = status_behind<LANES>(st, live, b, e, lane, [&](int i) {
    const double* X = pts + 3 * (size_t)obs_pt[rows[i]];
    return fma(E[CT_R + 6], X[0], fma(E[CT_R + 7], X[1], fma(E[CT_R + 8], X[2], E[CT_T + 2])));
  });
  if (!live || lane != 0) return;
  const double nan = res_nan();
  const bool at_start = st == TRI_NOT_PD;
#pragma unroll
  for (int k = 0; k < 6; ++k) pose[6 * g + k] = !on ? nan : at_start ? q0[k] : q[k];
  rmse[g] = !on ? nan : sqrt((at_start ? cost0 : cost) / n);
  status[g] = st;
}

// Per group with status 0, 3 or 4 (NaN otherwise), at the refined pose q*:
//   Sigma_q = s2 H^-1 + H^-1 M H^-1,  M = sum_p G_p Sigma_p G_p^T,  G_p = sum over the consensus rows of point p of
//   J_q^T J_X (6 x 3, pixels),  Sigma_p = pts_cov[p]  (pts_cov nullptr: M = 0).
// `rows` are the group's consensus rows sorted by point within the group (stable), so each point's rows are adjacent:
// the lane holding the first row of a run sums the run's G_p before the quadratic form.
template <int LANES>
__global__ void __launch_bounds__(TRI_THREADS)
res_cov_kernel(const double* __restrict__ camtab, const int* __restrict__ start, const int* __restrict__ rows,
               const int* __restrict__ obs_pt, const double* __restrict__ obs_px, const double* __restrict__ pts,
               const double* __restrict__ pts_cov, int n_groups, const int* __restrict__ cam,
               const int* __restrict__ status, const double* __restrict__ pose, double s2, double* __restrict__ cov) {
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  const bool live = g < n_groups;
  const int st = live ? status[g] : TRI_FEW_ROWS;
  const bool on = st == TRI_OK || st == TRI_MAX_ITER || st == TRI_BEHIND;
  const int b = on ? start[g] : 0, e = on ? start[g + 1] : 0;
  double h[21], m[21];
#pragma unroll
  for (int k = 0; k < 21; ++k) h[k] = m[k] = 0.0;
  if (on) {
    double q[6], E[CT_SIZE];
#pragma unroll
    for (int k = 0; k < 6; ++k) q[k] = pose[6 * g + k];
    res_entry(camtab + (size_t)CT_SIZE * cam[g], q, E);
    for (int i = b + lane; i < e; i += LANES) {
      const int p = obs_pt[rows[i]];
      const bool head = pts_cov && (i == b || obs_pt[rows[i - 1]] != p);
      double G[6][3];
#pragma unroll
      for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int c = 0; c < 3; ++c) G[a][c] = 0.0;
      // row i, then (first row of its point's run only) the rest of the run
      for (int j = i; j < e; ++j) {
        const int r = rows[j];
        if (j > i && (!head || obs_pt[r] != p)) break;
        double rr[2], J[12], JX[6];
        res_row_jac(E, pts + 3 * (size_t)p, reinterpret_cast<const double2*>(obs_px)[r], rr, J, JX);
        if (j == i)
#pragma unroll
          for (int a = 0; a < 6; ++a)
#pragma unroll
            for (int c = a; c < 6; ++c) h[ut<6>(a, c)] = fma(J[a], J[c], fma(J[6 + a], J[6 + c], h[ut<6>(a, c)]));
        if (head)
#pragma unroll
          for (int a = 0; a < 6; ++a)
#pragma unroll
            for (int c = 0; c < 3; ++c) G[a][c] = fma(J[a], JX[c], fma(J[6 + a], JX[3 + c], G[a][c]));
      }
      if (head) {
        const double* Sp = pts_cov + 9 * (size_t)p;
        double GS[6][3];
#pragma unroll
        for (int a = 0; a < 6; ++a)
#pragma unroll
          for (int c = 0; c < 3; ++c) GS[a][c] = G[a][0] * Sp[c] + G[a][1] * Sp[3 + c] + G[a][2] * Sp[6 + c];
#pragma unroll
        for (int a = 0; a < 6; ++a)
#pragma unroll
          for (int c = a; c < 6; ++c) m[ut<6>(a, c)] += GS[a][0] * G[c][0] + GS[a][1] * G[c][1] + GS[a][2] * G[c][2];
      }
    }
  }
#pragma unroll
  for (int s = LANES / 2; s > 0; s >>= 1)
#pragma unroll
    for (int k = 0; k < 21; ++k) {
      h[k] += __shfl_xor_sync(0xffffffffu, h[k], s);
      m[k] += __shfl_xor_sync(0xffffffffu, m[k], s);
    }
  if (!live || lane != 0) return;
  double* out = cov + 36 * (size_t)g;
  if (!on) {
    for (int k = 0; k < 36; ++k) out[k] = res_nan();
    return;
  }
  // H^-1 column by column, then out = s2 H^-1 + H^-1 M H^-1 (symmetrised)
  double L[6][6], Hi[6][6];
  res_chol<6>(h, 0.0, L);
#pragma unroll
  for (int c = 0; c < 6; ++c) {
    double v[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) v[k] = k == c ? 1.0 : 0.0;
    res_chol_solve<6>(L, v);
#pragma unroll
    for (int k = 0; k < 6; ++k) Hi[k][c] = v[k];
  }
  double T[6][6];  // M H^-1
#pragma unroll
  for (int a = 0; a < 6; ++a)
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      double v = 0.0;
#pragma unroll
      for (int k = 0; k < 6; ++k) v += m[a <= k ? ut<6>(a, k) : ut<6>(k, a)] * Hi[k][c];
      T[a][c] = v;
    }
#pragma unroll
  for (int a = 0; a < 6; ++a)
#pragma unroll
    for (int c = a; c < 6; ++c) {
      double v1 = s2 * Hi[a][c], v2 = s2 * Hi[c][a];
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        v1 += Hi[a][k] * T[k][c];
        v2 += Hi[c][k] * T[k][a];
      }
      out[6 * a + c] = out[6 * c + a] = 0.5 * (v1 + v2);
    }
}

// the key (group, point) of every consensus row, for the stable sort that makes each point's rows adjacent
template <int LANES>
__global__ void __launch_bounds__(TRI_THREADS)
res_pt_key_kernel(const int* __restrict__ start, const int* __restrict__ rows, const int* __restrict__ obs_pt,
                  int n_groups, int pt_bits, unsigned long long* __restrict__ key) {
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  if (g >= n_groups) return;
  for (int i = start[g] + lane; i < start[g + 1]; i += LANES)
    key[i] = ((unsigned long long)g << pt_bits) | (unsigned long long)obs_pt[rows[i]];
}

}  // namespace cb
