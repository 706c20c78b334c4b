// Robust relative pose of every camera pair from 2-D correspondences alone (cb_relative_pose_robust, DESIGN.md section
// 4.11): per pair (its correspondences: two rows of one key from the pair's cameras), Nister five-point hypotheses from
// 5-samples scored by MSAC on the Sampson distance, the consensus set, then Levenberg-Marquardt over (r, alpha, beta)
// and the first-order covariance.  oracle/relative_pose.py states the rule.
//   rp_slots_kernel     the correspondence slots of every key (stereo_slot, cb_stereo_rmse's enumeration): pair key,
//                       oriented rows
//   rp_gather_kernel    the pair-sorted slots' undistorted coordinates (xa, ya, xb, yb), NaN when a row is unusable
//   rp_hyp_kernel       one thread per (pair, sample): the five-point solver with its 10 x 20 elimination and Sturm
//                       chain in shared memory, the decomposition and cheirality, up to 10 table slots per sample
//   rp_score_kernel     (correspondence chunk, hypothesis block) tiles, res_score_kernel's layout; res_select_kernel
//                       picks the winner
//   rp_classify_kernel  the consensus set at the winner (consensus_classify), 32 lanes per pair
//   rp_refine_kernel / rp_cov_kernel   8 or 32 lanes per pair (res_refine_kernel's layout)
// No floating-point atomics: every sum has a fixed order, so repeated calls give bit-identical outputs.
#pragma once
#include <cstdint>

#include "cb_bootstrap.cuh"
#include "cb_resect.cuh"

namespace cb {

constexpr int RP_SLOTS_PER_SAMPLE = 10;  // essential matrices per sample at most; slot 10 m + c
constexpr int RP_HYP = 12;               // R (row-major, 9), t (3); R[0] NaN = no hypothesis
constexpr int RP_HYP_THREADS = 32;       // samples per rp_hyp_kernel block (a full warp)
constexpr int RP_CAM = 4;                // per camera: 1 / fx^2, 1 / fy^2, fisheye, unused
constexpr int RP_ROOT_STEPS = 200;       // bisection steps per root at most
// rp_hyp_kernel's per-thread shared workspace (doubles): null basis N [0, 36), E E^T's 6 distinct entries [36, 96) and
// later B(z) [36, 81), the 10 x 20 constraint matrix [96, 296) (the QR of the 5 x 9 system before it: A^T [96, 141),
// reflectors [141, 186)), later the Sturm chain 11 x 11 [96, 217), det B(z) [217, 228), chain degrees [228, 239) and
// the polish's Jacobian columns [240, 270)
constexpr int RP_WS = 296;
enum { RP_N = 0, RP_EET = 36, RP_BZ = 36, RP_M = 96, RP_A = 96, RP_V = 141, RP_CH = 96, RP_P = 217, RP_DEG = 228,
       RP_J = 240 };
constexpr int RP_HYP_SMEM = (int)sizeof(double) * RP_WS * RP_HYP_THREADS;  // 75.8 KB, above the 48 KB static limit
static_assert(RP_M + 200 <= RP_WS && RP_DEG + 11 <= RP_J && RP_J + 30 <= RP_WS, "rp_hyp_kernel's workspace layout");

__constant__ const int rp_ll_q[4][4] = {{0, 3, 4, 6}, {3, 1, 5, 7}, {4, 5, 2, 8}, {6, 7, 8, 9}};
__constant__ const int rp_ql_c[10][4] = {{0, 2, 4, 5},   {3, 1, 6, 7},    {10, 13, 16, 17}, {2, 3, 8, 9},
                                         {4, 8, 10, 11}, {8, 6, 13, 14},  {5, 9, 11, 12},   {9, 7, 14, 15},
                                         {11, 14, 17, 18}, {12, 15, 18, 19}};

// C(k, 5), saturated far above any max_samples
__device__ __forceinline__ long long rp_quintuples(int k) {
  if (k < 5) return 0;
  if (k >= 6000) return 1LL << 62;
  const long long c4 = (long long)k * (k - 1) / 2 * (k - 2) / 3 * (k - 3) / 4;
  return c4 * (k - 4) / 5;
}

// ---- correspondences ------------------------------------------------------------------------------------------------
// Every slot of every key (stereo_slots_kernel's counts, exclusive scan slot_start): key = a n_cams + b for rows of
// cameras a < b (n_cams^2 for two rows of one camera), val = (row of a) << 32 | (row of b)
template <int LANES>
__global__ void __launch_bounds__(BS_THREADS)
rp_slots_kernel(const int* __restrict__ start, const int* __restrict__ rows, const int* __restrict__ obs_cam, int n_groups,
                const long long* __restrict__ slot_start, int n_cams, unsigned int* __restrict__ key_out,
                unsigned long long* __restrict__ val_out) {
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  if (g >= n_groups) return;
  const int b = start[g], n = start[g + 1] - b;
  const long long s0 = slot_start[g], np = (long long)n * (n - 1) / 2;
  for (long long k = lane; k < np; k += LANES) {
    int ra, rb, ca, cb;
    stereo_slot(k, n, b, rows, obs_cam, ra, rb, ca, cb);
    key_out[s0 + k] = ca != cb ? (unsigned int)(ca * n_cams + cb) : (unsigned int)(n_cams * n_cams);
    val_out[s0 + k] = ((unsigned long long)(unsigned int)ra << 32) | (unsigned int)rb;
  }
}

// xy4[s] = (xa, ya, xb, yb) of the pair-sorted slot s, NaN when a row's coordinates are not finite or are a fisheye
// camera's (-1e6, -1e6) failure sentinel
__global__ void rp_gather_kernel(const unsigned long long* __restrict__ val, const int* __restrict__ obs_cam,
                                 const double* __restrict__ xy, const double* __restrict__ cams, long long n,
                                 double* __restrict__ xy4) {
  const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (s >= n) return;
  const unsigned long long v = val[s];
  const int r[2] = {(int)(v >> 32), (int)(v & 0xffffffffULL)};
  double o[4];
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const double2 p = reinterpret_cast<const double2*>(xy)[r[q]];
    const bool fish = cams[RP_CAM * obs_cam[r[q]] + 2] != 0.0;
    const bool ok = isfinite(p.x) && isfinite(p.y) && !(fish && p.x == -1000000.0 && p.y == -1000000.0);
    o[2 * q] = ok ? p.x : res_nan();
    o[2 * q + 1] = ok ? p.y : res_nan();
  }
  reinterpret_cast<double4*>(xy4)[s] = make_double4(o[0], o[1], o[2], o[3]);
}

// ---- geometry ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void rp_cross(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// E = [t]x R (row-major)
__device__ __forceinline__ void rp_essential(const double* R, const double* t, double* E) {
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    E[j] = -t[2] * R[3 + j] + t[1] * R[6 + j];
    E[3 + j] = t[2] * R[j] - t[0] * R[6 + j];
    E[6 + j] = -t[1] * R[j] + t[0] * R[3 + j];
  }
}

// depths (la, lb): least squares of [R x_a, -x_b] (la, lb)^T = -t, x = (x, y, 1); true when both are > 0
__device__ __forceinline__ bool rp_depths_ok(const double* R, const double* t, double xa, double ya, double xb,
                                             double yb) {
  const double u0 = R[0] * xa + R[1] * ya + R[2], u1 = R[3] * xa + R[4] * ya + R[5], u2 = R[6] * xa + R[7] * ya + R[8];
  const double uu = u0 * u0 + u1 * u1 + u2 * u2, vv = xb * xb + yb * yb + 1.0, uv = u0 * xb + u1 * yb + u2;
  const double ut = u0 * t[0] + u1 * t[1] + u2 * t[2], vt = xb * t[0] + yb * t[1] + t[2];
  const double det = uu * vv - uv * uv;
  const double la = (uv * vt - ut * vv) / det, lb = (uu * vt - uv * ut) / det;
  return la > 0.0 && lb > 0.0;
}

// (x_b^T E x_a, Sampson denominator) with fi = (1/fx_a^2, 1/fy_a^2, 1/fx_b^2, 1/fy_b^2); Ex = E x_a, Etx = E^T x_b
__device__ __forceinline__ void rp_sampson(const double* E, const double* fi, double xa, double ya, double xb, double yb,
                                           double& num, double& den, double* Ex, double* Etx) {
#pragma unroll
  for (int i = 0; i < 3; ++i) Ex[i] = E[3 * i] * xa + E[3 * i + 1] * ya + E[3 * i + 2];
#pragma unroll
  for (int j = 0; j < 3; ++j) Etx[j] = E[j] * xb + E[3 + j] * yb + E[6 + j];
  num = xb * Ex[0] + yb * Ex[1] + Ex[2];
  den = Ex[0] * Ex[0] * fi[2] + Ex[1] * Ex[1] * fi[3] + Etx[0] * Etx[0] * fi[0] + Etx[1] * Etx[1] * fi[1];
}

// the pair's fi from the per-camera table
__device__ __forceinline__ void rp_focal(const double* __restrict__ cams, int a, int b, double* fi) {
  fi[0] = cams[RP_CAM * a];
  fi[1] = cams[RP_CAM * a + 1];
  fi[2] = cams[RP_CAM * b];
  fi[3] = cams[RP_CAM * b + 1];
}

// ---- the five-point solver (Nister), one thread's workspace w (stride RP_HYP_THREADS) -----------------------------
#define RPW(e) w[(e) * RP_HYP_THREADS]

// Horner on ascending coefficients w[off .. off + deg]
__device__ __forceinline__ double rp_peval(const double* w, int off, int deg, double x) {
  double v = 0.0;
#pragma unroll 1
  for (int i = deg; i >= 0; --i) v = v * x + RPW(off + i);
  return v;
}

// sign changes of the Sturm chain (n polynomials at RP_CH + 11 i, degrees at RP_DEG + i) at x
__device__ __forceinline__ int rp_sign_changes(const double* w, int n, double x) {
  int c = 0;
  double last = 0.0;
#pragma unroll 1
  for (int i = 0; i < n; ++i) {
    const double v = rp_peval(w, RP_CH + 11 * i, (int)RPW(RP_DEG + i), x);
    if (v != 0.0) {
      if (last != 0.0 && ((v < 0.0) != (last < 0.0))) ++c;
      last = v;
    }
  }
  return c;
}

// scale w[off .. off + deg] by 1 / max |coefficient|; false when all are zero
__device__ __forceinline__ bool rp_pnormalize(double* w, int off, int deg) {
  double m = 0.0;
#pragma unroll 1
  for (int i = 0; i <= deg; ++i) m = fmax(m, fabs(RPW(off + i)));
  if (!(m > 0.0)) return false;
#pragma unroll 1
  for (int i = 0; i <= deg; ++i) RPW(off + i) = RPW(off + i) / m;
  return true;
}

// null basis of the 5 x 9 epipolar system (rows of the five correspondences c) into N: columns 5..8 of the orthogonal
// factor of the Householder QR of its transpose A (9 x 5).  False when a reflector's column is zero.
__device__ __forceinline__ bool rp_null_basis(double* w, const double (&c)[5][4]) {
#pragma unroll
  for (int s = 0; s < 5; ++s) {
    const double xa = c[s][0], ya = c[s][1], xb = c[s][2], yb = c[s][3];
    const double q[9] = {xb * xa, xb * ya, xb, yb * xa, yb * ya, yb, xa, ya, 1.0};
#pragma unroll
    for (int r = 0; r < 9; ++r) RPW(RP_A + 5 * r + s) = q[r];
  }
#pragma unroll 1
  for (int k = 0; k < 5; ++k) {
    double nx = 0.0;
#pragma unroll 1
    for (int r = k; r < 9; ++r) nx += RPW(RP_A + 5 * r + k) * RPW(RP_A + 5 * r + k);
    nx = sqrt(nx);
    if (!(nx > 0.0)) return false;
    double vv = 0.0;
#pragma unroll 1
    for (int r = 0; r < 9; ++r) {
      double v = r < k ? 0.0 : RPW(RP_A + 5 * r + k);
      if (r == k) v += RPW(RP_A + 5 * r + k) >= 0.0 ? nx : -nx;
      RPW(RP_V + 9 * k + r) = v;
      vv += v * v;
    }
    const double s2 = 2.0 / vv;
#pragma unroll 1
    for (int col = k; col < 5; ++col) {
      double d = 0.0;
#pragma unroll 1
      for (int r = k; r < 9; ++r) d += RPW(RP_V + 9 * k + r) * RPW(RP_A + 5 * r + col);
      const double f = s2 * d;
#pragma unroll 1
      for (int r = k; r < 9; ++r) RPW(RP_A + 5 * r + col) -= RPW(RP_V + 9 * k + r) * f;
    }
  }
#pragma unroll 1
  for (int f = 0; f < 4; ++f) {
    double x[9];
#pragma unroll
    for (int r = 0; r < 9; ++r) x[r] = r == 5 + f ? 1.0 : 0.0;
#pragma unroll 1
    for (int k = 4; k >= 0; --k) {
      double vx = 0.0, vv = 0.0;
#pragma unroll
      for (int r = 0; r < 9; ++r) {
        vx += RPW(RP_V + 9 * k + r) * x[r];
        vv += RPW(RP_V + 9 * k + r) * RPW(RP_V + 9 * k + r);
      }
      const double s = 2.0 * vx / vv;
#pragma unroll
      for (int r = 0; r < 9; ++r) x[r] -= RPW(RP_V + 9 * k + r) * s;
    }
#pragma unroll
    for (int r = 0; r < 9; ++r) RPW(RP_N + 9 * f + r) = x[r];
  }
  return true;
}

// the linear polynomial (x, y, z, 1) of entry e of E = x N0 + y N1 + z N2 + N3
__device__ __forceinline__ void rp_lin(const double* w, int e, double (&l)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) l[i] = RPW(RP_N + 9 * i + e);
}

__device__ __forceinline__ void rp_mul_ll(const double (&a)[4], const double (&b)[4], double (&o)[10], double sgn) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[rp_ll_q[i][j]] += sgn * (a[i] * b[j]);
}

// o += sgn * (a b), a quadratic, b linear
__device__ __forceinline__ void rp_mul_ql(const double (&a)[10], const double (&b)[4], double (&o)[20], double sgn) {
#pragma unroll
  for (int i = 0; i < 10; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[rp_ql_c[i][j]] += sgn * (a[i] * b[j]);
}

__device__ __forceinline__ int rp_sym(int i, int j) { return i <= j ? 3 * i + j - i * (i + 1) / 2 : 3 * j + i - j * (j + 1) / 2; }

// the 10 x 20 constraint matrix (det E, then 2 E E^T E - tr(E E^T) E row-major) into M
__device__ __forceinline__ void rp_constraints(double* w) {
  {
    double o[20];
#pragma unroll
    for (int k = 0; k < 20; ++k) o[k] = 0.0;
    const int cof[3][4] = {{4, 8, 5, 7}, {3, 8, 5, 6}, {3, 7, 4, 6}};  // minors of E00, E01, E02
#pragma unroll 1
    for (int j = 0; j < 3; ++j) {
      double a[4], b[4], c[4], d[4], q[10], e0[4];
      rp_lin(w, cof[j][0], a);
      rp_lin(w, cof[j][1], b);
      rp_lin(w, cof[j][2], c);
      rp_lin(w, cof[j][3], d);
      rp_lin(w, j, e0);
#pragma unroll
      for (int k = 0; k < 10; ++k) q[k] = 0.0;
      rp_mul_ll(a, b, q, 1.0);
      rp_mul_ll(c, d, q, -1.0);
      rp_mul_ql(q, e0, o, j == 1 ? -1.0 : 1.0);
    }
#pragma unroll
    for (int k = 0; k < 20; ++k) RPW(RP_M + k) = o[k];
  }
#pragma unroll 1
  for (int i = 0; i < 3; ++i)
#pragma unroll 1
    for (int j = i; j < 3; ++j) {
      double q[10];
#pragma unroll
      for (int k = 0; k < 10; ++k) q[k] = 0.0;
#pragma unroll 1
      for (int k = 0; k < 3; ++k) {
        double a[4], b[4];
        rp_lin(w, 3 * i + k, a);
        rp_lin(w, 3 * j + k, b);
        rp_mul_ll(a, b, q, 1.0);
      }
#pragma unroll
      for (int k = 0; k < 10; ++k) RPW(RP_EET + 10 * rp_sym(i, j) + k) = q[k];
    }
  double tr[10];
#pragma unroll
  for (int k = 0; k < 10; ++k) tr[k] = RPW(RP_EET + 10 * rp_sym(0, 0) + k) + RPW(RP_EET + 10 * rp_sym(1, 1) + k) +
                                       RPW(RP_EET + 10 * rp_sym(2, 2) + k);
#pragma unroll 1
  for (int i = 0; i < 3; ++i)
#pragma unroll 1
    for (int j = 0; j < 3; ++j) {
      double o[20], s[20];
#pragma unroll
      for (int k = 0; k < 20; ++k) o[k] = s[k] = 0.0;
#pragma unroll 1
      for (int k = 0; k < 3; ++k) {
        double q[10], l[4];
#pragma unroll
        for (int m = 0; m < 10; ++m) q[m] = RPW(RP_EET + 10 * rp_sym(i, k) + m);
        rp_lin(w, 3 * k + j, l);
        rp_mul_ql(q, l, o, 1.0);
      }
      double l[4];
      rp_lin(w, 3 * i + j, l);
      rp_mul_ql(tr, l, s, 1.0);
#pragma unroll
      for (int k = 0; k < 20; ++k) RPW(RP_M + 20 * (1 + 3 * i + j) + k) = 2.0 * o[k] - s[k];
    }
}

// Gauss-Jordan with partial pivoting on M's first ten columns (the first row of a largest |pivot|); false when a pivot
// is zero
__device__ __forceinline__ bool rp_gauss_jordan(double* w) {
#pragma unroll 1
  for (int c = 0; c < 10; ++c) {
    int p = c;
    double best = fabs(RPW(RP_M + 20 * c + c));
#pragma unroll 1
    for (int r = c + 1; r < 10; ++r) {
      const double v = fabs(RPW(RP_M + 20 * r + c));
      if (v > best) {
        best = v;
        p = r;
      }
    }
    if (!(best > 0.0)) return false;
    if (p != c)
#pragma unroll 1
      for (int k = 0; k < 20; ++k) {
        const double t = RPW(RP_M + 20 * c + k);
        RPW(RP_M + 20 * c + k) = RPW(RP_M + 20 * p + k);
        RPW(RP_M + 20 * p + k) = t;
      }
    const double piv = RPW(RP_M + 20 * c + c);
#pragma unroll 1
    for (int k = 0; k < 20; ++k) RPW(RP_M + 20 * c + k) = RPW(RP_M + 20 * c + k) / piv;
#pragma unroll 1
    for (int r = 0; r < 10; ++r) {
      if (r == c) continue;
      const double f = RPW(RP_M + 20 * r + c);
#pragma unroll 1
      for (int k = 0; k < 20; ++k) RPW(RP_M + 20 * r + k) -= f * RPW(RP_M + 20 * c + k);
    }
  }
  return true;
}

// B(z) (3 x 3 polynomials, 5 ascending coefficients) from the reduced M: rows x^2 z - z x^2, y^2 z - z y^2, xyz - z xy
// over (x, y, 1); then det B(z) (11 coefficients) into P
__device__ __forceinline__ void rp_hidden(double* w) {
  const int src[3][4] = {{12, 11, 10, -1}, {15, 14, 13, -1}, {19, 18, 17, 16}};
#pragma unroll 1
  for (int r = 0; r < 3; ++r) {
    const int e = 4 + 2 * r, f = 5 + 2 * r;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      double o[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
      const int n = c == 2 ? 4 : 3;
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (i < n) {
          o[i] += RPW(RP_M + 20 * e + src[c][i]);
          o[i + 1] -= RPW(RP_M + 20 * f + src[c][i]);
        }
#pragma unroll
      for (int i = 0; i < 5; ++i) RPW(RP_BZ + 15 * r + 5 * c + i) = o[i];
    }
  }
  double p[11];
#pragma unroll
  for (int i = 0; i < 11; ++i) p[i] = 0.0;
#pragma unroll 1
  for (int c = 0; c < 3; ++c) {
    const int c1 = c == 0 ? 1 : 0, c2 = c == 2 ? 1 : 2;  // the minor's columns
    double m9[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) m9[i] = 0.0;
#pragma unroll
    for (int i = 0; i < 5; ++i)
#pragma unroll
      for (int j = 0; j < 5; ++j)
        m9[i + j] += RPW(RP_BZ + 15 * 1 + 5 * c1 + i) * RPW(RP_BZ + 15 * 2 + 5 * c2 + j) -
                     RPW(RP_BZ + 15 * 1 + 5 * c2 + i) * RPW(RP_BZ + 15 * 2 + 5 * c1 + j);
    const double sg = c == 1 ? -1.0 : 1.0;
#pragma unroll
    for (int i = 0; i < 5; ++i)
#pragma unroll
      for (int j = 0; j < 9; ++j)
        if (i + j < 11) p[i + j] += sg * (RPW(RP_BZ + 5 * c + i) * m9[j]);
  }
#pragma unroll
  for (int i = 0; i < 11; ++i) RPW(RP_P + i) = p[i];
}

// Sturm chain of P into RP_CH / RP_DEG; returns its length (0: P constant or not finite) and P's degree in deg
__device__ __forceinline__ int rp_sturm(double* w, int& deg) {
  deg = 10;
  while (deg > 0 && RPW(RP_P + deg) == 0.0) --deg;
  bool fin = true;
#pragma unroll 1
  for (int i = 0; i <= 10; ++i) fin = fin && isfinite(RPW(RP_P + i));
  if (deg < 1 || !fin) return 0;
#pragma unroll 1
  for (int i = 0; i <= deg; ++i) RPW(RP_CH + i) = RPW(RP_P + i);
  rp_pnormalize(w, RP_CH, deg);
  RPW(RP_DEG) = deg;
#pragma unroll 1
  for (int i = 0; i < deg; ++i) RPW(RP_CH + 11 + i) = (i + 1) * RPW(RP_P + i + 1);
  rp_pnormalize(w, RP_CH + 11, deg - 1);
  RPW(RP_DEG + 1) = deg - 1;
  int n = 2;
#pragma unroll 1
  while (n < 11 && RPW(RP_DEG + n - 1) > 0) {
    const int a = RP_CH + 11 * (n - 2), b = RP_CH + 11 * (n - 1), o = RP_CH + 11 * n;
    const int da = (int)RPW(RP_DEG + n - 2), db = (int)RPW(RP_DEG + n - 1);
#pragma unroll 1
    for (int i = 0; i <= da; ++i) RPW(o + i) = RPW(a + i);
#pragma unroll 1
    for (int d = da; d >= db; --d) {
      const double q = RPW(o + d) / RPW(b + db);
#pragma unroll 1
      for (int i = 0; i <= db; ++i) RPW(o + d - db + i) -= q * RPW(b + i);
      RPW(o + d) = 0.0;
    }
    int dr = db - 1;
    while (dr > 0 && RPW(o + dr) == 0.0) --dr;
#pragma unroll 1
    for (int i = 0; i <= dr; ++i) RPW(o + i) = -RPW(o + i);
    if (!rp_pnormalize(w, o, dr)) break;
    RPW(RP_DEG + n) = dr;
    ++n;
  }
  return n;
}

constexpr int RP_POLISH_STEPS = 3;

// E = x N0 + y N1 + z N2 + N3 (p = (x, y, z)) and its ten cubic constraints f: det E, then 2 E E^T E - tr(E E^T) E
__device__ __forceinline__ void rp_cubic(const double* w, const double* p, double* E, double* f) {
#pragma unroll
  for (int e = 0; e < 9; ++e)
    E[e] = p[0] * RPW(RP_N + e) + p[1] * RPW(RP_N + 9 + e) + p[2] * RPW(RP_N + 18 + e) + RPW(RP_N + 27 + e);
  double c0[3];
  rp_cross(E + 3, E + 6, c0);
  f[0] = E[0] * c0[0] + E[1] * c0[1] + E[2] * c0[2];
  double EEt[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) EEt[3 * i + j] = E[3 * i] * E[3 * j] + E[3 * i + 1] * E[3 * j + 1] + E[3 * i + 2] * E[3 * j + 2];
  const double tr = EEt[0] + EEt[4] + EEt[8];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      f[1 + 3 * i + j] = 2.0 * (EEt[3 * i] * E[j] + EEt[3 * i + 1] * E[3 + j] + EEt[3 * i + 2] * E[6 + j]) - tr * E[3 * i + j];
}

// Up to RP_POLISH_STEPS Gauss-Newton steps on p = (x, y, z) over the ten cubic constraints, each kept only when it lowers
// their sum of squares (oracle/relative_pose.py polish): B(z)'s null vector loses accuracy where B(z) is nearly rank one,
// the constraints themselves stay well conditioned there
__device__ __forceinline__ void rp_polish(double* w, double* p) {
  double E[9], f[10];
  rp_cubic(w, p, E, f);
  double ff = 0.0;
#pragma unroll
  for (int i = 0; i < 10; ++i) ff += f[i] * f[i];
#pragma unroll 1
  for (int it = 0; it < RP_POLISH_STEPS; ++it) {
    double EEt[9], EtE[9], cof[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        EEt[3 * i + j] = E[3 * i] * E[3 * j] + E[3 * i + 1] * E[3 * j + 1] + E[3 * i + 2] * E[3 * j + 2];
        EtE[3 * i + j] = E[i] * E[j] + E[3 + i] * E[3 + j] + E[6 + i] * E[6 + j];
      }
    const double tr = EEt[0] + EEt[4] + EEt[8];
    rp_cross(E + 3, E + 6, cof);
    rp_cross(E + 6, E, cof + 3);
    rp_cross(E, E + 3, cof + 6);
    double A[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, g[3] = {0.0, 0.0, 0.0};  // J^T J (packed), J^T f
#pragma unroll 1
    for (int k = 0; k < 3; ++k) {
      double D[9], J[10];
#pragma unroll
      for (int e = 0; e < 9; ++e) D[e] = RPW(RP_N + 9 * k + e);
      double de = 0.0, cd = 0.0;
#pragma unroll
      for (int e = 0; e < 9; ++e) {
        de += D[e] * E[e];
        cd += cof[e] * D[e];
      }
      J[0] = cd;
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          double v = 0.0;
#pragma unroll
          for (int m = 0; m < 3; ++m) {
            double edte = 0.0;  // (E D^T E)_ij = sum_m (E D^T)_im E_mj
#pragma unroll
            for (int l = 0; l < 3; ++l) edte += E[3 * i + l] * D[3 * m + l];
            v += D[3 * i + m] * EtE[3 * m + j] + edte * E[3 * m + j] + EEt[3 * i + m] * D[3 * m + j];
          }
          J[1 + 3 * i + j] = 2.0 * v - 2.0 * de * E[3 * i + j] - tr * D[3 * i + j];
        }
#pragma unroll
      for (int r = 0; r < 10; ++r) RPW(RP_J + 10 * k + r) = J[r];  // column k of J
    }
#pragma unroll
    for (int r = 0; r < 10; ++r) {
      const double j0 = RPW(RP_J + r), j1 = RPW(RP_J + 10 + r), j2 = RPW(RP_J + 20 + r);
      A[0] += j0 * j0; A[1] += j0 * j1; A[2] += j0 * j2; A[3] += j1 * j1; A[4] += j1 * j2; A[5] += j2 * j2;
      g[0] += j0 * f[r]; g[1] += j1 * f[r]; g[2] += j2 * f[r];
    }
    // Cramer on the symmetric 3 x 3 system A d = -g
    const double c00 = A[3] * A[5] - A[4] * A[4], c01 = A[2] * A[4] - A[1] * A[5], c02 = A[1] * A[4] - A[2] * A[3];
    const double c11 = A[0] * A[5] - A[2] * A[2], c12 = A[1] * A[2] - A[0] * A[4], c22 = A[0] * A[3] - A[1] * A[1];
    const double det = A[0] * c00 + A[1] * c01 + A[2] * c02;
    if (!(det != 0.0) || !isfinite(det)) break;
    const double pn[3] = {p[0] - (c00 * g[0] + c01 * g[1] + c02 * g[2]) / det,
                          p[1] - (c01 * g[0] + c11 * g[1] + c12 * g[2]) / det,
                          p[2] - (c02 * g[0] + c12 * g[1] + c22 * g[2]) / det};
    double En[9], fn[10];
    rp_cubic(w, pn, En, fn);
    double ffn = 0.0;
#pragma unroll
    for (int i = 0; i < 10; ++i) ffn += fn[i] * fn[i];
    if (!(ffn < ff)) break;
    p[0] = pn[0]; p[1] = pn[1]; p[2] = pn[2];
#pragma unroll
    for (int e = 0; e < 9; ++e) E[e] = En[e];
#pragma unroll
    for (int i = 0; i < 10; ++i) f[i] = fn[i];
    ff = ffn;
  }
}

// The essential matrices of one sample and their hypotheses: for each real root z of det B(z) in ascending order, (x, y)
// from B(z)'s null vector (the cross product of two of its rows with the largest |third component|), E = x N0 + y N1 +
// z N2 + N3, its decomposition (R1, t), (R1, -t), (R2, t), (R2, -t) and the first that puts the five points in front of
// both cameras; written to o[RP_HYP c], c counting the finite E.  Returns the number of E.
__device__ __forceinline__ int rp_solve(double* w, const double (&cs)[5][4], double* __restrict__ o) {
  int ne = 0;
  if (!rp_null_basis(w, cs)) return 0;
  rp_constraints(w);
  if (!rp_gauss_jordan(w)) return 0;
  rp_hidden(w);
  int deg;
  const int nch = rp_sturm(w, deg);
  if (nch == 0) return 0;
  double bound = 0.0;
#pragma unroll 1
  for (int i = 0; i < deg; ++i) bound = fmax(bound, fabs(RPW(RP_P + i) / RPW(RP_P + deg)));
  bound += 1.0;
  if (!isfinite(bound)) return 0;
  const int v0 = rp_sign_changes(w, nch, -bound);
  const int nroot = v0 - rp_sign_changes(w, nch, bound);
#pragma unroll 1
  for (int r = 0; r < nroot && ne < RP_SLOTS_PER_SAMPLE; ++r) {
    double lo = -bound, hi = bound;
    int clo = 0, chi = nroot, steps = 0;
    double flo = rp_peval(w, RP_P, deg, lo), fhi = rp_peval(w, RP_P, deg, hi);
#pragma unroll 1
    while (steps < RP_ROOT_STEPS &&
           !(chi - clo == 1 && ((flo < 0.0) != (fhi < 0.0)) && flo != 0.0 && fhi != 0.0)) {
      const double mid = 0.5 * (lo + hi);
      const int cm = v0 - rp_sign_changes(w, nch, mid);
      if (cm > r) {
        hi = mid; chi = cm; fhi = rp_peval(w, RP_P, deg, mid);
      } else {
        lo = mid; clo = cm; flo = rp_peval(w, RP_P, deg, mid);
      }
      ++steps;
    }
#pragma unroll 1
    while (steps < RP_ROOT_STEPS) {
      const double mid = 0.5 * (lo + hi);
      if (!(lo < mid && mid < hi)) break;
      const double fm = rp_peval(w, RP_P, deg, mid);
      if (fm == 0.0) {
        lo = hi = mid;
        break;
      }
      if ((fm < 0.0) == (flo < 0.0)) {
        lo = mid; flo = fm;
      } else {
        hi = mid; fhi = fm;
      }
      ++steps;
    }
    double z = 0.5 * (lo + hi), fz = rp_peval(w, RP_P, deg, z);
#pragma unroll 1
    for (int it = 0; it < 3; ++it) {
      double dz = 0.0;
#pragma unroll 1
      for (int i = deg; i >= 1; --i) dz = dz * z + i * RPW(RP_P + i);
      if (!(dz != 0.0)) break;
      const double zn = z - fz / dz, fn = rp_peval(w, RP_P, deg, zn);
      if (!(fabs(fn) <= fabs(fz))) break;
      z = zn;
      fz = fn;
    }
    // (x, y, 1) from B(z)
    double B[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) B[i][j] = rp_peval(w, RP_BZ + 15 * i + 5 * j, 4, z);
    double c0[3], c1[3], c2[3];
    rp_cross(B[0], B[1], c0);
    rp_cross(B[0], B[2], c1);
    rp_cross(B[1], B[2], c2);
    double v[3] = {c0[0], c0[1], c0[2]};
    if (fabs(c1[2]) > fabs(v[2])) { v[0] = c1[0]; v[1] = c1[1]; v[2] = c1[2]; }
    if (fabs(c2[2]) > fabs(v[2])) { v[0] = c2[0]; v[1] = c2[1]; v[2] = c2[2]; }
    if (!(fabs(v[2]) > 0.0)) continue;
    double pz[3] = {v[0] / v[2], v[1] / v[2], z};
    rp_polish(w, pz);
    double E[9];
    bool fin = true;
#pragma unroll
    for (int e = 0; e < 9; ++e) {
      E[e] = pz[0] * RPW(RP_N + e) + pz[1] * RPW(RP_N + 9 + e) + pz[2] * RPW(RP_N + 18 + e) + RPW(RP_N + 27 + e);
      fin = fin && isfinite(E[e]);
    }
    if (!fin) continue;
    // decomposition: |E|_F^2 = 2, t the largest cross product of two columns, R1,2 = cof(E) -+ [t]x E
    double nE = 0.0;
#pragma unroll
    for (int e = 0; e < 9; ++e) nE += E[e] * E[e];
    const double sc = sqrt(2.0) / sqrt(nE);
#pragma unroll
    for (int e = 0; e < 9; ++e) E[e] *= sc;
    const double col[3][3] = {{E[0], E[3], E[6]}, {E[1], E[4], E[7]}, {E[2], E[5], E[8]}};
    double t[3], tc[3];
    rp_cross(col[0], col[1], t);
    double tn = t[0] * t[0] + t[1] * t[1] + t[2] * t[2];
    rp_cross(col[0], col[2], tc);
    double tcn = tc[0] * tc[0] + tc[1] * tc[1] + tc[2] * tc[2];
    if (tcn > tn) { t[0] = tc[0]; t[1] = tc[1]; t[2] = tc[2]; tn = tcn; }
    rp_cross(col[1], col[2], tc);
    tcn = tc[0] * tc[0] + tc[1] * tc[1] + tc[2] * tc[2];
    if (tcn > tn) { t[0] = tc[0]; t[1] = tc[1]; t[2] = tc[2]; tn = tcn; }
    const double itn = 1.0 / sqrt(tn);
#pragma unroll
    for (int i = 0; i < 3; ++i) t[i] *= itn;
    double cof[9], tE[9];
    rp_cross(E + 3, E + 6, cof);
    rp_cross(E + 6, E, cof + 3);
    rp_cross(E, E + 3, cof + 6);
    rp_essential(E, t, tE);  // [t]x E: the same product with E in place of R
    double* h = o + RP_HYP * ne;
    h[0] = res_nan();
#pragma unroll 1
    for (int d = 0; d < 4; ++d) {
      const double sr = d < 2 ? -1.0 : 1.0, st = (d & 1) ? -1.0 : 1.0;
      double R[9], tt[3];
#pragma unroll
      for (int e = 0; e < 9; ++e) R[e] = cof[e] + sr * tE[e];
#pragma unroll
      for (int i = 0; i < 3; ++i) tt[i] = st * t[i];
      bool ok = true;
#pragma unroll
      for (int s = 0; s < 5; ++s) ok = ok && rp_depths_ok(R, tt, cs[s][0], cs[s][1], cs[s][2], cs[s][3]);
      if (ok) {
#pragma unroll
        for (int e = 0; e < 9; ++e) h[e] = R[e];
#pragma unroll
        for (int i = 0; i < 3; ++i) h[9 + i] = tt[i];
        break;
      }
    }
    ++ne;
  }
  return ne;
}
#undef RPW

// Thread (pair, sample m) of a flat index over n_pairs x max_samples: the table slots 10 m .. 10 m + 9 of its pair
// (S = 10 max_samples per pair), R[0] = NaN where there is no hypothesis (also for every slot of a pair with fewer than
// min_inliers correspondences)
__global__ void __launch_bounds__(RP_HYP_THREADS)
rp_hyp_kernel(const int* __restrict__ start, const double* __restrict__ xy4, int n_pairs, int max_samples,
              int min_inliers, double* __restrict__ tab) {
  extern __shared__ double s_ws[];  // RP_HYP_SMEM bytes
  double* w = s_ws + threadIdx.x;
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)n_pairs * max_samples) return;
  const long long g = idx / max_samples, m = idx % max_samples;
  const int b = start[g], k = start[g + 1] - b;
  const long long S = (long long)RP_SLOTS_PER_SAMPLE * max_samples;
  double* o = tab + (size_t)RP_HYP * (size_t)(g * S + RP_SLOTS_PER_SAMPLE * m);
  int ne = 0;
  const long long T = rp_quintuples(k);
  int p[5];
  if (k >= min_inliers && m < T && res_sample<5>(m, T, max_samples, k, p)) {
    double cs[5][4];
    bool ok = true;
#pragma unroll
    for (int s = 0; s < 5; ++s) {
      const double4 v = reinterpret_cast<const double4*>(xy4)[b + p[s]];
      cs[s][0] = v.x; cs[s][1] = v.y; cs[s][2] = v.z; cs[s][3] = v.w;
      ok = ok && isfinite(v.x) && isfinite(v.z);  // unusable rows are NaN in both coordinates
    }
    if (ok) ne = rp_solve(w, cs, o);
  }
  for (int c = ne; c < RP_SLOTS_PER_SAMPLE; ++c) o[RP_HYP * c] = res_nan();
}

// One block per (correspondence chunk, block of RES_SCORE_THREADS slots), res_score_kernel's tiles: the chunk's
// coordinates go to shared memory, each thread scores its slot's E = [t]x R over them in order (min(e^2, tau^2), tau^2
// for a non-finite e) and writes part[chunk][slot] (+inf: no hypothesis)
__global__ void __launch_bounds__(RES_SCORE_THREADS)
rp_score_kernel(const int* __restrict__ start, const int* __restrict__ chunk_off, const double* __restrict__ xy4,
                const int* __restrict__ cam_a, const int* __restrict__ cam_b, const double* __restrict__ cams,
                int n_pairs, int S, const double* __restrict__ tab, double tau, double* __restrict__ part) {
  __shared__ double4 s_c[RES_CHUNK];
  const int chunk = blockIdx.x;
  int lo = 0, hi = n_pairs;  // the pair of the chunk: the last g with chunk_off[g] <= chunk
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (chunk_off[mid] <= chunk) lo = mid;
    else hi = mid;
  }
  const int g = lo;
  const int b = start[g] + (chunk - chunk_off[g]) * RES_CHUNK, e = min(start[g + 1], b + RES_CHUNK), n = e - b;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s_c[i] = reinterpret_cast<const double4*>(xy4)[b + i];
  __syncthreads();
  const int s = blockIdx.y * RES_SCORE_THREADS + threadIdx.x;
  if (s >= S) return;
  const double* h = tab + (size_t)RP_HYP * ((size_t)g * S + s);
  const double tau2 = tau * tau;
  double score = __longlong_as_double(0x7ff0000000000000LL);
  if (!isnan(h[0])) {
    double E[9], fi[4];
    rp_essential(h, h + 9, E);
    rp_focal(cams, cam_a[g], cam_b[g], fi);
    score = 0.0;
    for (int i = 0; i < n; ++i) {
      const double4 c = s_c[i];
      double num, den, Ex[3], Etx[3];
      rp_sampson(E, fi, c.x, c.y, c.z, c.w, num, den, Ex, Etx);
      score += msac_term(true, num * num / den, tau2);
    }
  }
  part[(size_t)chunk * S + s] = score;
}

// The consensus set at the winner, one pair per 32 lanes (positions `pos` = 0, 1, ... of the pair-sorted
// correspondences): lane 0 writes count, n_inliers, status (1, 5 or 0) and the winner (NaN without consensus)
__global__ void __launch_bounds__(TRI_THREADS)
rp_classify_kernel(const int* __restrict__ start, const int* __restrict__ pos, const double* __restrict__ xy4,
                   const int* __restrict__ cam_a, const int* __restrict__ cam_b, const double* __restrict__ cams,
                   int n_pairs, int S, const double* __restrict__ tab, const int* __restrict__ best, double tau,
                   int min_inliers, double* __restrict__ hyp, int* __restrict__ count, int* __restrict__ n_inliers,
                   int* __restrict__ status, unsigned char* __restrict__ pos_flag, unsigned char* __restrict__ inlier) {
  constexpr int LANES = 32;
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  const bool live = g < n_pairs;
  const int b = live ? start[g] : 0, e = live ? start[g + 1] : 0, k = e - b;
  const bool few = k < min_inliers;
  const int wslot = live ? best[g] : -1;
  const bool found = live && !few && wslot >= 0;
  double R[9], t[3], E[9], fi[4];
  const double* h = tab + (size_t)RP_HYP * ((size_t)g * S + (found ? wslot : 0));
#pragma unroll
  for (int q = 0; q < 9; ++q) R[q] = found ? h[q] : 0.0;
#pragma unroll
  for (int q = 0; q < 3; ++q) t[q] = found ? h[9 + q] : 0.0;
  rp_essential(R, t, E);
  rp_focal(cams, live ? cam_a[g] : 0, live ? cam_b[g] : 0, fi);
  int nin;
  const bool ok = consensus_classify<LANES>(
      found, pos, b, e, lane, tau * tau, min_inliers,
      [&](int r, bool& front) {
        const double4 c = reinterpret_cast<const double4*>(xy4)[r];
        double num, den, Ex[3], Etx[3];
        rp_sampson(E, fi, c.x, c.y, c.z, c.w, num, den, Ex, Etx);
        front = rp_depths_ok(R, t, c.x, c.y, c.z, c.w);
        return num * num / den;
      },
      pos_flag, inlier, nin);
  if (!live || lane != 0) return;
  count[g] = k;
  n_inliers[g] = ok ? nin : 0;
  status[g] = few ? TRI_FEW_ROWS : ok ? TRI_OK : TRI_NO_CONSENSUS;
#pragma unroll
  for (int q = 0; q < 9; ++q) hyp[RP_HYP * g + q] = ok ? R[q] : res_nan();
#pragma unroll
  for (int q = 0; q < 3; ++q) hyp[RP_HYP * g + 9 + q] = ok ? t[q] : res_nan();
}

// ---- refinement and covariance ----------------------------------------------------------------------------------------
// columns 1 and 2 of the Householder reflector I - 2 v v^T / v^T v, v = t0 + sign(t0_z) |t0| e3, which takes t0 to -+e3
__device__ __forceinline__ void rp_chart(const double* t0, double* u1, double* u2) {
  const double n = sqrt(t0[0] * t0[0] + t0[1] * t0[1] + t0[2] * t0[2]);
  const double v[3] = {t0[0], t0[1], t0[2] + (t0[2] >= 0.0 ? n : -n)};
  const double s = 2.0 / (v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    u1[i] = (i == 0 ? 1.0 : 0.0) - s * v[i] * v[0];
    u2[i] = (i == 1 ? 1.0 : 0.0) - s * v[i] * v[1];
  }
}

// R and t at q = (r, alpha, beta) in the chart (t0, u1, u2): R = Rodrigues(r) (I + [r]x below theta^2 = 1e-30),
// t = normalize(t0 + alpha u1 + beta u2); with ed: E = [t]x R (ed[0..8]) and dE/dq (ed[9 + 5 e + k]).  Not inlined: the
// refinement's LM loop keeps its sums in registers, and this body's temporaries would push them to local memory.
__device__ __noinline__ void rp_pose(const double* q, const double* t0, const double* u1, const double* u2,
                                        double* R, double* t, double* ed) {
  const double r[3] = {q[0], q[1], q[2]};
  const double th2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
  const double K[9] = {0.0, -r[2], r[1], r[2], 0.0, -r[0], -r[1], r[0], 0.0};
  const bool small = th2 < 1e-30;
  double a = 1.0, bq = 0.0;
  if (!small) {
    const double th = sqrt(th2);
    a = sin(th) / th;
    bq = (1.0 - cos(th)) / th2;
  }
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double kk = K[3 * i] * K[j] + K[3 * i + 1] * K[3 + j] + K[3 * i + 2] * K[6 + j];
      R[3 * i + j] = (i == j ? 1.0 : 0.0) + a * K[3 * i + j] + bq * kk;
    }
  double wv[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) wv[i] = t0[i] + q[3] * u1[i] + q[4] * u2[i];
  const double nw = sqrt(wv[0] * wv[0] + wv[1] * wv[1] + wv[2] * wv[2]);
#pragma unroll
  for (int i = 0; i < 3; ++i) t[i] = wv[i] / nw;
  if (!ed) return;
  rp_essential(R, t, ed);
  // dR/dr_i = (r_i [r]x + [r x ((I - R) e_i)]x) R / theta^2, or [e_i]x at theta^2 < 1e-30
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    double D[9];
    if (small) {
      const double ei[3] = {i == 0 ? 1.0 : 0.0, i == 1 ? 1.0 : 0.0, i == 2 ? 1.0 : 0.0};
      const double S[9] = {0.0, -ei[2], ei[1], ei[2], 0.0, -ei[0], -ei[1], ei[0], 0.0};
#pragma unroll
      for (int e = 0; e < 9; ++e) D[e] = S[e];
    } else {
      const double c[3] = {(i == 0 ? 1.0 : 0.0) - R[i], (i == 1 ? 1.0 : 0.0) - R[3 + i], (i == 2 ? 1.0 : 0.0) - R[6 + i]};
      double x[3];
      rp_cross(r, c, x);
      const double M[9] = {0.0, -(r[i] * r[2] + x[2]), r[i] * r[1] + x[1], r[i] * r[2] + x[2], 0.0,
                           -(r[i] * r[0] + x[0]), -(r[i] * r[1] + x[1]), r[i] * r[0] + x[0], 0.0};
#pragma unroll
      for (int u = 0; u < 3; ++u)
#pragma unroll
        for (int v = 0; v < 3; ++v)
          D[3 * u + v] = (M[3 * u] * R[v] + M[3 * u + 1] * R[3 + v] + M[3 * u + 2] * R[6 + v]) / th2;
    }
    double dE[9];
    rp_essential(D, t, dE);
#pragma unroll
    for (int e = 0; e < 9; ++e) ed[9 + 5 * e + i] = dE[e];
  }
  // dt/dalpha = (u1 - t (t . u1)) / |w|, the same for beta with u2
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const double* u = k ? u2 : u1;
    const double tu = t[0] * u[0] + t[1] * u[1] + t[2] * u[2];
    const double dt[3] = {(u[0] - t[0] * tu) / nw, (u[1] - t[1] * tu) / nw, (u[2] - t[2] * tu) / nw};
    double dE[9];
    rp_essential(R, dt, dE);
#pragma unroll
    for (int e = 0; e < 9; ++e) ed[9 + 5 * e + 3 + k] = dE[e];
  }
}

// Cost, H = J^T J (packed, 15) and g = J^T r (5) of the signed Sampson residuals of positions [b, e) of `pos`, at the E
// and dE/dq in ed (shared, the group's), summed over the LANES lanes
template <int LANES>
__device__ __forceinline__ void rp_normal_eq(const double* ed, const double* fi, const double* __restrict__ xy4,
                                             const int* __restrict__ pos, int b, int e, int lane, bool on,
                                             double (&acc)[21]) {
#pragma unroll
  for (int k = 0; k < 21; ++k) acc[k] = 0.0;
  if (on) {
    double E[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) E[q] = ed[q];
    // dE/dq is read from shared memory at every row: held in registers across the row loop it would spill the sums
    const volatile double* dE = ed + 9;
    for (int i = b + lane; i < e; i += LANES) {
      const double4 c = reinterpret_cast<const double4*>(xy4)[pos[i]];
      double num, den, Ex[3], Etx[3];
      rp_sampson(E, fi, c.x, c.y, c.z, c.w, num, den, Ex, Etx);
      const double sd = sqrt(den), r = num / sd, hr = r / (2.0 * den), isd = 1.0 / sd;
      const double ha[3] = {c.x, c.y, 1.0}, hb[3] = {c.z, c.w, 1.0};
      const double fb[3] = {2.0 * fi[2] * Ex[0], 2.0 * fi[3] * Ex[1], 0.0};
      const double fa[3] = {2.0 * fi[0] * Etx[0], 2.0 * fi[1] * Etx[1], 0.0};
      double J[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int u = 0; u < 3; ++u)
#pragma unroll
        for (int v = 0; v < 3; ++v) {
          const double dr = hb[u] * ha[v] * isd - hr * (fb[u] * ha[v] + fa[v] * hb[u]);
#pragma unroll
          for (int k = 0; k < 5; ++k) J[k] = fma(dr, dE[5 * (3 * u + v) + k], J[k]);
        }
#pragma unroll
      for (int a = 0; a < 5; ++a) {
#pragma unroll
        for (int cc = a; cc < 5; ++cc) acc[ut<5>(a, cc)] = fma(J[a], J[cc], acc[ut<5>(a, cc)]);
        acc[15 + a] = fma(J[a], r, acc[15 + a]);
      }
      acc[20] = fma(r, r, acc[20]);
    }
  }
  group_sum<LANES>(acc);
}

// Per pair with consensus, Levenberg-Marquardt (lm_iterate) over q = (r, alpha, beta) on the consensus positions
// (start, pos) from the winner hyp (R by res_rot_log, the chart at its t).  Writes pose (r, t) (the hypothesis for
// status 2, NaN without consensus), the Sampson rmse and the mean parallax over the consensus set, and the status (the
// consensus stage's 1 or 5, else 2, 3, 4 or 0).
template <int LANES>
__global__ void __launch_bounds__(TRI_THREADS)
rp_refine_kernel(const int* __restrict__ start, const int* __restrict__ pos, const double* __restrict__ xy4,
                 const int* __restrict__ cam_a, const int* __restrict__ cam_b, const double* __restrict__ cams,
                 int n_pairs, const int* __restrict__ cstatus, const double* __restrict__ hyp, int max_iter, double xtol,
                 double* __restrict__ pose, double* __restrict__ rmse, double* __restrict__ parallax,
                 int* __restrict__ status) {
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  const bool live = g < n_pairs;
  int st = live ? cstatus[g] : TRI_FEW_ROWS;
  const bool on = st == TRI_OK;
  const int b = on ? start[g] : 0, e = on ? start[g + 1] : 0, n = e - b;
  double fi[4], t0[3] = {0.0, 0.0, 1.0}, u1[3], u2[3];
  rp_focal(cams, on ? cam_a[g] : 0, on ? cam_b[g] : 0, fi);
  double q0[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  if (on) {
    res_rot_log(hyp + RP_HYP * g, q0);
#pragma unroll
    for (int k = 0; k < 3; ++k) t0[k] = hyp[RP_HYP * g + 9 + k];
  }
  rp_chart(t0, u1, u2);
  double q[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) q[k] = q0[k];
  // per group in shared memory: the sums at the current q and the E, dE/dq of the pose being evaluated
  __shared__ double s_acc[TRI_THREADS / LANES][21];
  __shared__ double s_ed[TRI_THREADS / LANES][54];
  double* sa = s_acc[threadIdx.x / LANES];
  double* se = s_ed[threadIdx.x / LANES];
  auto sums = [&](const double* qq, bool on_, double (&acc)[21]) {
    __syncwarp();  // every lane has read se
    if (on_ && lane == 0) {
      double R[9], t[3];
      rp_pose(qq, t0, u1, u2, R, t, se);
    }
    __syncwarp();
    rp_normal_eq<LANES>(se, fi, xy4, pos, b, e, lane, on_, acc);
  };
  double cost;
  {
    double acc[21];
    sums(q, on, acc);
    if (on && !res_pd<5>(acc)) st = TRI_NOT_PD;
    if (lane == 0)
#pragma unroll
      for (int k = 0; k < 21; ++k) sa[k] = acc[k];
    cost = acc[20];
  }
  const double cost0 = cost;
  double tr[21];
  st = lm_iterate<5>(
      q, on && st == TRI_OK, st, max_iter, xtol,
      [&](double lam, bool on_, double* d) {
        __syncwarp();  // lane 0's last write of sa is visible
        if (!on_) return;
        double A[15], L[5][5];
#pragma unroll
        for (int k = 0; k < 15; ++k) A[k] = sa[k];
#pragma unroll
        for (int k = 0; k < 5; ++k) {
          A[ut<5>(k, k)] = sa[ut<5>(k, k)] * (1.0 + lam);
          d[k] = -sa[15 + k];
        }
        res_chol<5>(A, 0.0, L);
        res_chol_solve<5>(L, d);
      },
      [&](const double* qt, bool on_) {
        sums(qt, on_, tr);
        __syncwarp();  // every lane has read sa
        return tr[20] < cost;
      },
      [&] {
        if (lane == 0)
#pragma unroll
          for (int k = 0; k < 21; ++k) sa[k] = tr[k];
        cost = tr[20];
      },
      [](const double* v) {
        double s2 = 0.0;
#pragma unroll
        for (int k = 0; k < 5; ++k) s2 += v[k] * v[k];
        return sqrt(s2);
      });
  __syncwarp();  // lane 0's last write of sa is visible
  if (st == TRI_OK || st == TRI_MAX_ITER) {
    double h[15];
#pragma unroll
    for (int k = 0; k < 15; ++k) h[k] = sa[k];
    if (!res_pd<5>(h)) st = TRI_NOT_PD;
  }
  const bool at_start = st == TRI_NOT_PD;
  double qf[5], R[9], t[3];
#pragma unroll
  for (int k = 0; k < 5; ++k) qf[k] = at_start ? q0[k] : q[k];
  rp_pose(qf, t0, u1, u2, R, t, nullptr);
  st = status_behind<LANES>(st, on, b, e, lane, [&](int i) {
    const double4 c = reinterpret_cast<const double4*>(xy4)[pos[i]];
    return rp_depths_ok(R, t, c.x, c.y, c.z, c.w) ? 1.0 : -1.0;
  });
  // the mean angle between R x_a and x_b over the consensus set, at the reported pose
  double ang = 0.0;
  if (on)
    for (int i = b + lane; i < e; i += LANES) {
      const double4 c = reinterpret_cast<const double4*>(xy4)[pos[i]];
      const double u[3] = {R[0] * c.x + R[1] * c.y + R[2], R[3] * c.x + R[4] * c.y + R[5], R[6] * c.x + R[7] * c.y + R[8]};
      const double co = (u[0] * c.z + u[1] * c.w + u[2]) /
                        (sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]) * sqrt(c.z * c.z + c.w * c.w + 1.0));
      ang += acos(fmin(1.0, fmax(-1.0, co)));
    }
  ang = group_sum<LANES>(ang);
  if (!live || lane != 0) return;
  const double nan = res_nan();
#pragma unroll
  for (int k = 0; k < 3; ++k) pose[6 * g + k] = on ? qf[k] : nan;
#pragma unroll
  for (int k = 0; k < 3; ++k) pose[6 * g + 3 + k] = on ? t[k] : nan;
  rmse[g] = on ? sqrt((at_start ? cost0 : cost) / n) : nan;
  parallax[g] = on ? ang * (180.0 / 3.141592653589793) / n : nan;
  status[g] = st;
}

// Per pair with status 0, 3 or 4 (NaN otherwise), at the refined pose (r, t*): the chart re-based at t*,
// cov5 = s2 H^-1 over (r, du), written as J cov5 J^T with J = diag(I3, [u1 u2](t*)) (6 x 6, rank 5)
template <int LANES>
__global__ void __launch_bounds__(TRI_THREADS)
rp_cov_kernel(const int* __restrict__ start, const int* __restrict__ pos, const double* __restrict__ xy4,
              const int* __restrict__ cam_a, const int* __restrict__ cam_b, const double* __restrict__ cams,
              int n_pairs, const int* __restrict__ status, const double* __restrict__ pose, double s2,
              double* __restrict__ cov) {
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  const bool live = g < n_pairs;
  const int st = live ? status[g] : TRI_FEW_ROWS;
  const bool on = st == TRI_OK || st == TRI_MAX_ITER || st == TRI_BEHIND;
  const int b = on ? start[g] : 0, e = on ? start[g + 1] : 0;
  __shared__ double s_ed[TRI_THREADS / LANES][54];
  double* se = s_ed[threadIdx.x / LANES];
  double fi[4], t0[3] = {0.0, 0.0, 1.0}, u1[3], u2[3], q[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  rp_focal(cams, on ? cam_a[g] : 0, on ? cam_b[g] : 0, fi);
  if (on) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      q[k] = pose[6 * g + k];
      t0[k] = pose[6 * g + 3 + k];
    }
  }
  rp_chart(t0, u1, u2);
  if (on && lane == 0) {
    double R[9], t[3];
    rp_pose(q, t0, u1, u2, R, t, se);
  }
  __syncwarp();
  double acc[21];
  rp_normal_eq<LANES>(se, fi, xy4, pos, b, e, lane, on, acc);
  if (!live || lane != 0) return;
  double* out = cov + 36 * (size_t)g;
  if (!on) {
    for (int k = 0; k < 36; ++k) out[k] = res_nan();
    return;
  }
  double L[5][5], Hi[5][5];
  res_chol<5>(acc, 0.0, L);
#pragma unroll
  for (int c = 0; c < 5; ++c) {
    double v[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) v[k] = k == c ? s2 : 0.0;
    res_chol_solve<5>(L, v);
#pragma unroll
    for (int k = 0; k < 5; ++k) Hi[k][c] = v[k];
  }
  double Jt[6][5];
#pragma unroll
  for (int a = 0; a < 6; ++a)
#pragma unroll
    for (int c = 0; c < 5; ++c) Jt[a][c] = a < 3 ? (a == c ? 1.0 : 0.0) : c == 3 ? u1[a - 3] : c == 4 ? u2[a - 3] : 0.0;
  double T[6][5];  // Jt cov5
#pragma unroll
  for (int a = 0; a < 6; ++a)
#pragma unroll
    for (int c = 0; c < 5; ++c) {
      double v = 0.0;
#pragma unroll
      for (int k = 0; k < 5; ++k) v += Jt[a][k] * Hi[k][c];
      T[a][c] = v;
    }
#pragma unroll
  for (int a = 0; a < 6; ++a)
#pragma unroll
    for (int c = a; c < 6; ++c) {
      double v1 = 0.0, v2 = 0.0;
#pragma unroll
      for (int k = 0; k < 5; ++k) {
        v1 += T[a][k] * Jt[c][k];
        v2 += T[c][k] * Jt[a][k];
      }
      out[6 * a + c] = out[6 * c + a] = 0.5 * (v1 + v2);
    }
}

}  // namespace cb
