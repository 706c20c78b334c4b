// Kernels of the extrinsic bootstrap (SURVEY.md section 8(f) rank 1): what produces the start vector of bundle adjustment.
//
//   pnp_ippe_kernel     == compute_camera_to_object_poses_pnp
//                          (reference core/bootstrap_pose/pose_network_builder.py:211-330): one planar PnP per
//                          (camera, sync_index, object) group with cv2.solvePnP(..., SOLVEPNP_IPPE) on undistorted
//                          normalised points (:301-306), reprojection RMSE in the normalised plane (:314-318).
//                          OpenCV is an un-vendored dependency; the published algorithms are restated: IPPE (Collins &
//                          Bartoli, IJCV 2014) on the Harker-O'Leary homography (BMVC 2005), see oracle/ippe.py which is
//                          pinned against cv2 to 1e-13.
//   stereo_pairs_kernel == calculate_stereo_rmse_for_pair (:638-685) for ALL camera pairs at once: every pair of
//                          observations of the same (sync, object, keypoint) from two cameras that have an aggregated
//                          relative pose is triangulated from the two views (cv2.triangulatePoints: DLT, :668),
//                          projected back into both (:672-676) and its squared residuals are emitted under the pair's id;
//                          a stable sort + segmented sum gives sqrt(mean) per pair (:678-679).
//
// Both are latency / fp64-pipe bound (a few dependent 3x3 / 4x4 eigen-solves per group), not HBM bound: 28-36 algorithmic
// bytes per observation against hundreds of dependent flops.
#pragma once
#include "cb_triangulate.cuh"

namespace cb {

constexpr int BS_THREADS = 256;

// Eigenvector of the smallest eigenvalue of a symmetric 3x3 (cyclic Jacobi).
__device__ __forceinline__ void sym3_min_eigvec(double a[3][3], double out[3]) {
  double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
#pragma unroll 1
  for (int sweep = 0; sweep < 16; ++sweep) {
    const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
    const double dg = a[0][0] * a[0][0] + a[1][1] * a[1][1] + a[2][2] * a[2][2];
    if (off <= 1e-36 * dg) break;
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
      for (int q = p + 1; q < 3; ++q) {
        const double apq = a[p][q];
        if (apq != 0.0) {
          const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
          const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
          const double c = rsqrt(t * t + 1.0), s = t * c;
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const double akp = a[k][p], akq = a[k][q];
            a[k][p] = c * akp - s * akq;
            a[k][q] = s * akp + c * akq;
          }
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const double apk = a[p][k], aqk = a[q][k];
            a[p][k] = c * apk - s * aqk;
            a[q][k] = s * apk + c * aqk;
          }
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const double vkp = V[k][p], vkq = V[k][q];
            V[k][p] = c * vkp - s * vkq;
            V[k][q] = s * vkp + c * vkq;
          }
        }
      }
  }
  int m = 0;
  if (a[1][1] < a[m][m]) m = 1;
  if (a[2][2] < a[m][m]) m = 2;
#pragma unroll
  for (int k = 0; k < 3; ++k) out[k] = (m == 0) ? V[k][0] : (m == 1) ? V[k][1] : V[k][2];
}

__device__ __forceinline__ void mat3_mul(const double* A, const double* B, double* C) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}

// The two IPPE rotations from the 2x2 Jacobian J of the model-to-image map at the model centroid and the image (p, q) of
// the centroid; returns gamma, the first-order scale (<= 0 / NaN: degenerate).
__device__ __forceinline__ double ippe_rotations(double j00, double j01, double j10, double j11, double p, double q,
                                                 double Rs[2][9]) {
  double Rv[9];
  {
    const double nrm = sqrt(p * p + q * q + 1.0), ax = p / nrm, ay = q / nrm, az = 1.0 / nrm;
    const double d = 1.0 / (1.0 + az);  // az > 0
    // rotation taking (p, q, 1) onto +z, transposed
    Rv[0] = 1.0 - ax * ax * d; Rv[1] = -ax * ay * d;      Rv[2] = ax;
    Rv[3] = -ax * ay * d;      Rv[4] = 1.0 - ay * ay * d; Rv[5] = ay;
    Rv[6] = -ax;               Rv[7] = -ay;               Rv[8] = 1.0 - (ax * ax + ay * ay) * d;
  }
  const double b00 = Rv[0] - p * Rv[6], b01 = Rv[1] - p * Rv[7], b10 = Rv[3] - q * Rv[6], b11 = Rv[4] - q * Rv[7];
  const double dti = 1.0 / (b00 * b11 - b01 * b10);
  const double bi00 = dti * b11, bi01 = -dti * b01, bi10 = -dti * b10, bi11 = dti * b00;
  const double A00 = bi00 * j00 + bi01 * j10, A01 = bi00 * j01 + bi01 * j11, A10 = bi10 * j00 + bi11 * j10,
               A11 = bi10 * j01 + bi11 * j11;
  const double ata00 = A00 * A00 + A01 * A01, ata01 = A00 * A10 + A01 * A11, ata11 = A10 * A10 + A11 * A11;
  const double gamma = sqrt(0.5 * (ata00 + ata11 + sqrt((ata00 - ata11) * (ata00 - ata11) + 4.0 * ata01 * ata01)));
  const double r00 = A00 / gamma, r01 = A01 / gamma, r10 = A10 / gamma, r11 = A11 / gamma;
  const double bb0 = sqrt(fmax(0.0, 1.0 - r00 * r00 - r10 * r10));
  double bb1 = sqrt(fmax(0.0, 1.0 - r01 * r01 - r11 * r11));
  if (-r00 * r01 - r10 * r11 < 0) bb1 = -bb1;
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const double sg = s == 0 ? 1.0 : -1.0;
    const double c0[3] = {r00, r10, sg * bb0}, c1v[3] = {r01, r11, sg * bb1};
    const double c2v[3] = {c0[1] * c1v[2] - c0[2] * c1v[1], c0[2] * c1v[0] - c0[0] * c1v[2], c0[0] * c1v[1] - c0[1] * c1v[0]};
    const double Rt[9] = {c0[0], c1v[0], c2v[0], c0[1], c1v[1], c2v[1], c0[2], c1v[2], c2v[2]};
    mat3_mul(Rv, Rt, Rs[s]);
  }
  return gamma;
}

// exp([w]x) (Rodrigues)
__device__ __forceinline__ void rot_exp(const double* w, double* R) {
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], th = sqrt(th2);
  double a, b;  // R = I + a K + b K^2, K = [w]x
  if (th < 1e-8) { a = 1.0; b = 0.5; }
  else { a = sin(th) / th; b = (1.0 - cos(th)) / th2; }
  const double K[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
  double K2[9];
  mat3_mul(K, K, K2);
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = ((i % 4 == 0) ? 1.0 : 0.0) + a * K[i] + b * K2[i];
}

// solve the SPD 6x6 system H d = -g in place (Cholesky); H packed upper (21), returns false if not positive definite
__device__ __forceinline__ bool solve6(const double* Hp, const double* g, double* d) {
  double L[6][6];
  int t = 0;
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j) { L[j][i] = Hp[t]; ++t; }
  double tr = 0.0;
  for (int i = 0; i < 6; ++i) tr += L[i][i];
  for (int i = 0; i < 6; ++i) L[i][i] += 1e-12 * tr;
  for (int j = 0; j < 6; ++j) {
    double v = L[j][j];
    for (int k = 0; k < j; ++k) v -= L[j][k] * L[j][k];
    if (!(v > 0.0)) return false;
    v = sqrt(v);
    L[j][j] = v;
    for (int i = j + 1; i < 6; ++i) {
      double s = L[i][j];
      for (int k = 0; k < j; ++k) s -= L[i][k] * L[j][k];
      L[i][j] = s / v;
    }
  }
  double y[6];
  for (int i = 0; i < 6; ++i) {
    double s = -g[i];
    for (int k = 0; k < i; ++k) s -= L[i][k] * y[k];
    y[i] = s / L[i][i];
  }
  for (int i = 5; i >= 0; --i) {
    double s = y[i];
    for (int k = i + 1; k < 6; ++k) s -= L[k][i] * d[k];
    d[i] = s / L[i][i];
  }
  return true;
}

// Harker-O'Leary homography (BMVC 2005) of the rows [b, e) of `rows`, one warp: img ~ H (x - mx, y - my, 1) with the
// model points x = ax(r, 0..1) centred on their mean (mx, my) and the image points img(r, 0..1) (mean (mu, mv)).
// Returns false when the points have no spread or the model points' 2x2 moment matrix is singular; det, a00 and a11
// come back with H so that a caller can reject (nearly) collinear model points.  pnp_ippe_kernel (float32 model points)
// and intr_view_kernel (full precision) both fit with it.
struct HoFit {
  double betaA, betaB, c1, c2, c3, c4, a00, a11, det, i00, i01, i11;
  double H[9];
};

template <typename AX, typename IMG>
__device__ __forceinline__ bool ho_fit(const int* __restrict__ rows, int b, int e, int lane, int n, double mx, double my,
                                       double mu, double mv, AX ax, IMG img, HoFit& f) {
  // ---- pass 1: isotropic scales
  double ka = 0, kb = 0;
  for (int i = b + lane; i < e; i += 32) {
    const int r = rows[i];
    const double ax0 = ax(r, 0) - mx, ay0 = ax(r, 1) - my, bu = img(r, 0) - mu, bv = img(r, 1) - mv;
    ka += ax0 * ax0 + ay0 * ay0;
    kb += bu * bu + bv * bv;
  }
  ka = warp_sum(ka); kb = warp_sum(kb);
  if (!(ka > 0.0) || !(kb > 0.0)) return false;
  const double betaA = sqrt(2.0 * n / ka), betaB = sqrt(2.0 * n / kb);
  // normalised source A = betaA (obj - mean), target B = betaB (img - mean)
#define HO_LOAD(r)                                                                                     \
  const double A0 = betaA * (ax(r, 0) - mx), A1 = betaA * (ax(r, 1) - my);                             \
  const double B0 = betaB * (img(r, 0) - mu), B1 = betaB * (img(r, 1) - mv)
  // ---- pass 2: means of C1..C4, A A^T
  double c1 = 0, c2 = 0, c3 = 0, c4 = 0, a00 = 0, a01 = 0, a11 = 0;
  for (int i = b + lane; i < e; i += 32) {
    const int r = rows[i];
    HO_LOAD(r);
    c1 += -B0 * A0; c2 += -B0 * A1; c3 += -B1 * A0; c4 += -B1 * A1;
    a00 += A0 * A0; a01 += A0 * A1; a11 += A1 * A1;
  }
  c1 = warp_sum(c1) / n; c2 = warp_sum(c2) / n; c3 = warp_sum(c3) / n; c4 = warp_sum(c4) / n;
  a00 = warp_sum(a00); a01 = warp_sum(a01); a11 = warp_sum(a11);
  const double det = a00 * a11 - a01 * a01;
  if (!(fabs(det) > 0.0)) return false;
  const double i00 = a11 / det, i01 = -a01 / det, i11 = a00 / det;
  // ---- pass 3: A Mx, A My (2x3 each)
  double amx[6] = {0, 0, 0, 0, 0, 0}, amy[6] = {0, 0, 0, 0, 0, 0};
  for (int i = b + lane; i < e; i += 32) {
    const int r = rows[i];
    HO_LOAD(r);
    const double mxr[3] = {-B0 * A0 - c1, -B0 * A1 - c2, -B0}, myr[3] = {-B1 * A0 - c3, -B1 * A1 - c4, -B1};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      amx[k] += A0 * mxr[k]; amx[3 + k] += A1 * mxr[k];
      amy[k] += A0 * myr[k]; amy[3 + k] += A1 * myr[k];
    }
  }
  double Bx[6], By[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) { amx[k] = warp_sum(amx[k]); amy[k] = warp_sum(amy[k]); }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    Bx[k] = i00 * amx[k] + i01 * amx[3 + k]; Bx[3 + k] = i01 * amx[k] + i11 * amx[3 + k];
    By[k] = i00 * amy[k] + i01 * amy[3 + k]; By[3 + k] = i01 * amy[k] + i11 * amy[3 + k];
  }
  // ---- pass 4: D^T D with D rows = Mx_i - A_i^T Bx ; My_i - A_i^T By
  double dd[6] = {0, 0, 0, 0, 0, 0};
  for (int i = b + lane; i < e; i += 32) {
    const int r = rows[i];
    HO_LOAD(r);
    double d1[3], d2[3];
    const double mxr[3] = {-B0 * A0 - c1, -B0 * A1 - c2, -B0}, myr[3] = {-B1 * A0 - c3, -B1 * A1 - c4, -B1};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      d1[k] = mxr[k] - (A0 * Bx[k] + A1 * Bx[3 + k]);
      d2[k] = myr[k] - (A0 * By[k] + A1 * By[3 + k]);
    }
    dd[0] += d1[0] * d1[0] + d2[0] * d2[0]; dd[1] += d1[0] * d1[1] + d2[0] * d2[1]; dd[2] += d1[0] * d1[2] + d2[0] * d2[2];
    dd[3] += d1[1] * d1[1] + d2[1] * d2[1]; dd[4] += d1[1] * d1[2] + d2[1] * d2[2]; dd[5] += d1[2] * d1[2] + d2[2] * d2[2];
  }
#pragma unroll
  for (int k = 0; k < 6; ++k) dd[k] = warp_sum(dd[k]);
  double M[3][3] = {{dd[0], dd[1], dd[2]}, {dd[1], dd[3], dd[4]}, {dd[2], dd[4], dd[5]}};
  double h789[3];
  sym3_min_eigvec(M, h789);
  // normalised-frame homography, then H = TB^-1 Hn TA
  double Hn[9];
  Hn[0] = -(Bx[0] * h789[0] + Bx[1] * h789[1] + Bx[2] * h789[2]);
  Hn[1] = -(Bx[3] * h789[0] + Bx[4] * h789[1] + Bx[5] * h789[2]);
  Hn[2] = -(c1 * h789[0] + c2 * h789[1]);
  Hn[3] = -(By[0] * h789[0] + By[1] * h789[1] + By[2] * h789[2]);
  Hn[4] = -(By[3] * h789[0] + By[4] * h789[1] + By[5] * h789[2]);
  Hn[5] = -(c3 * h789[0] + c4 * h789[1]);
  Hn[6] = h789[0]; Hn[7] = h789[1]; Hn[8] = h789[2];
  // canonical source frame = centred object points (mean removed), so TA = diag(betaA, betaA, 1) there
  const double TA[9] = {betaA, 0, 0, 0, betaA, 0, 0, 0, 1};
  const double TBi[9] = {1.0 / betaB, 0, mu, 0, 1.0 / betaB, mv, 0, 0, 1};
  double T1[9];
  mat3_mul(Hn, TA, T1);
  mat3_mul(TBi, T1, f.H);
#undef HO_LOAD
  f.betaA = betaA; f.betaB = betaB; f.c1 = c1; f.c2 = c2; f.c3 = c3; f.c4 = c4;
  f.a00 = a00; f.a11 = a11; f.det = det; f.i00 = i00; f.i01 = i01; f.i11 = i11;
  return true;
}

// status codes of a PnP group
constexpr int PNP_OK = 0, PNP_TOO_FEW = 1, PNP_NON_PLANAR = 2, PNP_DEGENERATE = 3, PNP_OK_FALLBACK = 4;
constexpr double IPPE_GAMMA_MIN = 1e-7;

// One warp per (camera, sync, object) group; rows[start[g] .. start[g+1]) index the caller's observation arrays.
// obj: (n_obs, 3) object-frame coordinates (NaN z counts as 0, as the reference's nan_to_num), img: (n_obs, 2) undistorted
// normalised coordinates already rounded to float32 (the undistortion kernel does that).  Outputs per group:
// R (9, row-major), t (3), rmse, status, count, representative row.
__global__ void __launch_bounds__(BS_THREADS)
pnp_ippe_kernel(const int* __restrict__ start, const int* __restrict__ rows, const double* __restrict__ obj,
                const double* __restrict__ img, int n_groups, int min_points, double* __restrict__ R_out,
                double* __restrict__ t_out, double* __restrict__ rmse_out, int* __restrict__ status_out,
                int* __restrict__ count_out, int* __restrict__ rep_out) {
  const int lane = threadIdx.x & 31;
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  if (g >= n_groups) return;
  const int b = start[g], e = start[g + 1], n = e - b;
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  auto fail = [&](int code) {
    if (lane == 0) {
      for (int k = 0; k < 9; ++k) R_out[9 * g + k] = nan;
      for (int k = 0; k < 3; ++k) t_out[3 * g + k] = nan;
      rmse_out[g] = nan;
      status_out[g] = code;
      count_out[g] = n;
      rep_out[g] = rows[b];
    }
  };
  // float32 object coordinates (the reference casts obj_points to float32 before the call, :296)
  auto ox = [&](int r, int k) {
    double v = obj[3 * (size_t)r + k];
    if (k == 2 && v != v) v = 0.0;
    return (double)(float)v;
  };
  // ---- pass 0: means, z spread
  double sx = 0, sy = 0, sz = 0, su = 0, sv = 0, zmin = 1e300, zmax = -1e300;
  for (int i = b + lane; i < e; i += 32) {
    const int r = rows[i];
    double zraw = obj[3 * (size_t)r + 2];
    if (zraw != zraw) zraw = 0.0;
    sx += ox(r, 0); sy += ox(r, 1); sz += ox(r, 2);
    su += img[2 * (size_t)r]; sv += img[2 * (size_t)r + 1];
    zmin = fmin(zmin, zraw); zmax = fmax(zmax, zraw);
  }
  sx = warp_sum(sx); sy = warp_sum(sy); sz = warp_sum(sz); su = warp_sum(su); sv = warp_sum(sv);
  zmax = warp_max(zmax); zmin = -warp_max(-zmin);
  if (!(zmax - zmin < 1e-6)) { fail(PNP_NON_PLANAR); return; }  // np.ptp(z) < 1e-6 (:279)
  if (n < min_points) { fail(PNP_TOO_FEW); return; }
  const double mx = sx / n, my = sy / n, mz = sz / n, mu = su / n, mv = sv / n;
  // ---- passes 1-4: the homography of the centred model plane
  HoFit f;
  if (!ho_fit(rows, b, e, lane, n, mx, my, mu, mv, ox, [&](int r, int k) { return img[2 * (size_t)r + k]; }, f)) {
    fail(PNP_DEGENERATE);
    return;
  }
  double* H = f.H;
  // all model points on one line: no pose (cv2 reports success with a NaN pose; the reference keeps the group and its
  // NaN filter drops it later, pose_network_builder.py:364-367)
  if (!(fabs(f.det) > 1e-12 * (f.a00 + f.a11) * (f.a00 + f.a11))) { fail(PNP_DEGENERATE); return; }
  double Rs[2][9], ts[2][3], err[2];
  double gamma = -1.0;
  if (fabs(H[8]) > 0.0) {
#pragma unroll
    for (int k = 0; k < 8; ++k) H[k] /= H[8];
    H[8] = 1.0;
    // ---- the two IPPE rotations from the first-order behaviour of H at the origin
    const double p = H[2], q = H[5];
    gamma = ippe_rotations(H[0] - H[6] * p, H[1] - H[7] * p, H[3] - H[6] * q, H[4] - H[7] * q, p, q, Rs);
  }
  // OpenCV's IPPE gives up when the homography is degenerate (three of four points collinear, ...): gamma collapses to
  // ~1e-10 and the reference falls back to SOLVEPNP_ITERATIVE (:308-311).  Restated (oracle/ippe.py): the two IPPE poses of
  // the AFFINE fit, each refined by Gauss-Newton on the reprojection error, the better one kept.
  const bool fallback = !(gamma >= IPPE_GAMMA_MIN);
  if (fallback) {
    // affine fit in normalised coordinates: B ~ Mn A, Mn = (sum B A^T)(sum A A^T)^-1, sum B A^T = -n [c1 c2; c3 c4]
    const double s00 = -n * f.c1, s01 = -n * f.c2, s10 = -n * f.c3, s11 = -n * f.c4, sc = f.betaA / f.betaB;
    const double m00 = sc * (s00 * f.i00 + s01 * f.i01), m01 = sc * (s00 * f.i01 + s01 * f.i11);
    const double m10 = sc * (s10 * f.i00 + s11 * f.i01), m11 = sc * (s10 * f.i01 + s11 * f.i11);
    gamma = ippe_rotations(m00, m01, m10, m11, mu, mv, Rs);
    if (!(gamma > 0.0)) { fail(PNP_DEGENERATE); return; }
  }
  // ---- pass 5: translations (least squares), both candidates
  {
    double acc[2][3] = {{0, 0, 0}, {0, 0, 0}}, suu = 0, su1 = 0, sv1 = 0;
    for (int i = b + lane; i < e; i += 32) {
      const int r = rows[i];
      const double X = ox(r, 0) - mx, Y = ox(r, 1) - my, u = img[2 * (size_t)r], v = img[2 * (size_t)r + 1];
      su1 += u; sv1 += v; suu += u * u + v * v;
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const double* R = Rs[s];
        const double rx = R[0] * X + R[1] * Y, ry = R[3] * X + R[4] * Y, rz = R[6] * X + R[7] * Y;
        const double bx = u * rz - rx, by = v * rz - ry;
        acc[s][0] += bx; acc[s][1] += by; acc[s][2] -= u * bx + v * by;
      }
    }
    su1 = warp_sum(su1); sv1 = warp_sum(sv1); suu = warp_sum(suu);
#pragma unroll
    for (int s = 0; s < 2; ++s) {
#pragma unroll
      for (int k = 0; k < 3; ++k) acc[s][k] = warp_sum(acc[s][k]);
      // A^T A = [n 0 -su; 0 n -sv; -su -sv suu]: eliminate tx, ty
      const double nn = (double)n;
      const double den = suu - (su1 * su1 + sv1 * sv1) / nn;
      const double tz = (acc[s][2] + (su1 * acc[s][0] + sv1 * acc[s][1]) / nn) / den;
      ts[s][0] = (acc[s][0] + su1 * tz) / nn;
      ts[s][1] = (acc[s][1] + sv1 * tz) / nn;
      ts[s][2] = tz;
    }
  }
  // ---- fallback only: Gauss-Newton on the reprojection error, both candidates (rotation increment on the left)
  if (fallback) {
#pragma unroll 1
    for (int s2 = 0; s2 < 2; ++s2) {
#pragma unroll 1
      for (int it = 0; it < 30; ++it) {
        double Hp[21], gv[6];
#pragma unroll
        for (int k = 0; k < 21; ++k) Hp[k] = 0.0;
#pragma unroll
        for (int k = 0; k < 6; ++k) gv[k] = 0.0;
        const double* R = Rs[s2];
        for (int i = b + lane; i < e; i += 32) {
          const int r = rows[i];
          const double X = ox(r, 0) - mx, Y = ox(r, 1) - my, u0 = img[2 * (size_t)r], v0 = img[2 * (size_t)r + 1];
          const double xr = R[0] * X + R[1] * Y, yr = R[3] * X + R[4] * Y, zr = R[6] * X + R[7] * Y;
          const double zc = zr + ts[s2][2], iz = 1.0 / zc, u = (xr + ts[s2][0]) * iz, v = (yr + ts[s2][1]) * iz;
          // d(u, v)/d(Xc) rows, then Xc = exp(w) (R X) + t: dXc/dw = -[R X]x, dXc/dt = I
          const double du[3] = {iz, 0.0, -u * iz}, dv[3] = {0.0, iz, -v * iz};
          double Ju[6], Jv[6];
          Ju[0] = du[1] * (-zr) + du[2] * yr;  Ju[1] = du[0] * zr + du[2] * (-xr);  Ju[2] = du[0] * (-yr) + du[1] * xr;
          Jv[0] = dv[1] * (-zr) + dv[2] * yr;  Jv[1] = dv[0] * zr + dv[2] * (-xr);  Jv[2] = dv[0] * (-yr) + dv[1] * xr;
#pragma unroll
          for (int k = 0; k < 3; ++k) { Ju[3 + k] = du[k]; Jv[3 + k] = dv[k]; }
          const double ru = u - u0, rv = v - v0;
          int t2 = 0;
#pragma unroll
          for (int a2 = 0; a2 < 6; ++a2) {
            gv[a2] += Ju[a2] * ru + Jv[a2] * rv;
#pragma unroll
            for (int b2 = a2; b2 < 6; ++b2) { Hp[t2] += Ju[a2] * Ju[b2] + Jv[a2] * Jv[b2]; ++t2; }
          }
        }
#pragma unroll
        for (int k = 0; k < 21; ++k) Hp[k] = warp_sum(Hp[k]);
#pragma unroll
        for (int k = 0; k < 6; ++k) gv[k] = warp_sum(gv[k]);
        double d6[6];
        if (!solve6(Hp, gv, d6)) break;
        double dR[9], Rn[9];
        rot_exp(d6, dR);
        mat3_mul(dR, Rs[s2], Rn);
#pragma unroll
        for (int k = 0; k < 9; ++k) Rs[s2][k] = Rn[k];
        ts[s2][0] += d6[0 + 3]; ts[s2][1] += d6[1 + 3]; ts[s2][2] += d6[2 + 3];
        const double dn = d6[0] * d6[0] + d6[1] * d6[1] + d6[2] * d6[2] + d6[3] * d6[3] + d6[4] * d6[4] + d6[5] * d6[5];
        if (dn < 1e-28) break;
      }
    }
  }
  // ---- pass 6: reprojection error of both, best first
  {
    double e0 = 0, e1 = 0;
    for (int i = b + lane; i < e; i += 32) {
      const int r = rows[i];
      const double X = ox(r, 0) - mx, Y = ox(r, 1) - my, u = img[2 * (size_t)r], v = img[2 * (size_t)r + 1];
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const double* R = Rs[s];
        const double xc = R[0] * X + R[1] * Y + ts[s][0], yc = R[3] * X + R[4] * Y + ts[s][1], zc = R[6] * X + R[7] * Y + ts[s][2];
        const double du = u - xc / zc, dv = v - yc / zc;
        if (s == 0) e0 += du * du + dv * dv; else e1 += du * du + dv * dv;
      }
    }
    err[0] = warp_sum(e0); err[1] = warp_sum(e1);
  }
  const int best = (err[1] < err[0]) ? 1 : 0;
  if (lane == 0) {
    const double* R = Rs[best];
    // canonical (centred, z = mean z) frame -> the caller's object frame: t - R mean
    const double tx = ts[best][0] - (R[0] * mx + R[1] * my + R[2] * mz);
    const double ty = ts[best][1] - (R[3] * mx + R[4] * my + R[5] * mz);
    const double tz = ts[best][2] - (R[6] * mx + R[7] * my + R[8] * mz);
#pragma unroll
    for (int k = 0; k < 9; ++k) R_out[9 * g + k] = R[k];
    t_out[3 * g] = tx; t_out[3 * g + 1] = ty; t_out[3 * g + 2] = tz;
    rmse_out[g] = sqrt(err[best] / n);
    status_out[g] = (R[0] == R[0] && tz == tz) ? (fallback ? PNP_OK_FALLBACK : PNP_OK) : PNP_DEGENERATE;
    count_out[g] = n;
    rep_out[g] = rows[b];
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Stereo RMSE of every camera pair.  Groups = rows sharing (sync, object, keypoint); pair_of[a * n_cams + b] (a < b) =
// index of the pair's pose [R | t] (camera a at the origin, camera b = R X + t) or -1.  Each group emits one slot per
// unordered pair of its rows (slot_start from an exclusive scan of n (n - 1) / 2): key = pair index (n_pairs = none),
// value = squared residuals of the two views.
// ------------------------------------------------------------------------------------------------------------------
__global__ void stereo_slots_kernel(const int* __restrict__ start, int n_groups, long long* __restrict__ nslots) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_groups) return;
  const long long n = start[g + 1] - start[g];
  nslots[g] = n * (n - 1) / 2;
}

// Slot k of a group of n rows from key-sorted position b: k -> (i, j), i < j, row-major over the strict upper triangle;
// rows (ra, rb) and their cameras (ca, cb) swapped so that ca <= cb
__device__ __forceinline__ void stereo_slot(long long k, int n, int b, const int* __restrict__ rows,
                                            const int* __restrict__ obs_cam, int& ra, int& rb, int& ca, int& cb) {
  int i = (int)((2.0 * n - 1.0 - sqrt((2.0 * n - 1.0) * (2.0 * n - 1.0) - 8.0 * (double)k)) * 0.5);
  while ((long long)i * (2 * n - i - 1) / 2 > k) --i;
  while ((long long)(i + 1) * (2 * n - i - 2) / 2 <= k) ++i;
  const int j = (int)(k - (long long)i * (2 * n - i - 1) / 2) + i + 1;
  ra = rows[b + i];
  rb = rows[b + j];
  ca = obs_cam[ra];
  cb = obs_cam[rb];
  if (ca > cb) { int t = ca; ca = cb; cb = t; t = ra; ra = rb; rb = t; }
}

__device__ __forceinline__ double sq_res_f32(double nx, double ny, double px, double py) {
  // the reference subtracts float32 projections from float32 points and squares in float32 (:678-679)
  const float ex = (float)nx - (float)px, ey = (float)ny - (float)py;
  return (double)(ex * ex) + (double)(ey * ey);
}

template <int LANES>
__global__ void __launch_bounds__(BS_THREADS)
stereo_pairs_kernel(const int* __restrict__ start, const int* __restrict__ rows, const int* __restrict__ obs_cam,
                    const double* __restrict__ xy, int n_groups, const long long* __restrict__ slot_start, int n_cams,
                    const int* __restrict__ pair_of, const double* __restrict__ pair_Rt, int n_pairs,
                    int* __restrict__ key_out, double* __restrict__ val_out) {
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  if (g >= n_groups) return;
  const int b = start[g], n = start[g + 1] - b;
  const long long s0 = slot_start[g], np = (long long)n * (n - 1) / 2;
  for (long long k = lane; k < np; k += LANES) {
    int ra, rb, ca, cb;
    stereo_slot(k, n, b, rows, obs_cam, ra, rb, ca, cb);
    int pid = (ca != cb) ? pair_of[(size_t)ca * n_cams + cb] : -1;
    double val = 0.0;
    if (pid >= 0) {
      const double* Rt = pair_Rt + 12 * (size_t)pid;  // [R (9) | t (3)]
      const double ax = xy[2 * (size_t)ra], ay = xy[2 * (size_t)ra + 1], bx = xy[2 * (size_t)rb], by = xy[2 * (size_t)rb + 1];
      // DLT rows: x P[2] - P[0], y P[2] - P[1] for P1 = [I | 0], P2 = [R | t]
      double r[4][4];
      r[0][0] = -1; r[0][1] = 0; r[0][2] = ax; r[0][3] = 0;
      r[1][0] = 0; r[1][1] = -1; r[1][2] = ay; r[1][3] = 0;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        r[2][c] = bx * Rt[6 + c] - Rt[c];
        r[3][c] = by * Rt[6 + c] - Rt[3 + c];
      }
      r[2][3] = bx * Rt[11] - Rt[9];
      r[3][3] = by * Rt[11] - Rt[10];
      double M[4][4];
#pragma unroll
      for (int p2 = 0; p2 < 4; ++p2)
#pragma unroll
        for (int q2 = 0; q2 < 4; ++q2) M[p2][q2] = r[0][p2] * r[0][q2] + r[1][p2] * r[1][q2] + r[2][p2] * r[2][q2] + r[3][p2] * r[3][q2];
      double w[4];
      sym4_min_eigvec(M, w);
      // cv2.triangulatePoints returns float32 for float32 inputs; the reference divides in float32 (:669)
      const float w3 = (float)w[3];
      const double X = (double)((float)w[0] / w3), Y = (double)((float)w[1] / w3), Z = (double)((float)w[2] / w3);
      const double pax = X / Z, pay = Y / Z;
      const double xb = Rt[0] * X + Rt[1] * Y + Rt[2] * Z + Rt[9], yb = Rt[3] * X + Rt[4] * Y + Rt[5] * Z + Rt[10],
                   zb = Rt[6] * X + Rt[7] * Y + Rt[8] * Z + Rt[11];
      val = sq_res_f32(ax, ay, pax, pay) + sq_res_f32(bx, by, xb / zb, yb / zb);
    } else {
      pid = n_pairs;
    }
    key_out[s0 + k] = pid;
    val_out[s0 + k] = val;
  }
}


// ---------------------------------------------------------------------------------------------------------------------
// Relative-pose network (pose_network_builder.py): compute_relative_poses (:486-560) -> reject_outliers (:340-412) ->
// aggregate_poses (:520-560, quaternion_average :414-437) for EVERY camera pair in one pass over device arrays.
//   rel_pose_kernel       one thread per (frame group, camera a, camera b) combination: T_B_A = T_B_obj inv(T_A_obj),
//                         unit quaternion (Shepperd), |t|, sort key = a * span + b
//   (radix sort by pair, run-length encode -> one segment per camera pair, segmented sorts for the quartiles)
//   quat_average_kernel   block per pair: sum of q q^T over (masked) rows, largest eigenvector (Jacobi), sum of t, row count
//   rel_angle_kernel      angle between each sample and its pair's mean rotation
//   seg_quartile_kernel   np.percentile(.., [25, 75]) of a sorted segment, NumPy's 'linear' rule and its lerp
//   rel_flag_kernel       the IQR rule (pairs with >= 5 samples)
// ---------------------------------------------------------------------------------------------------------------------
constexpr int REL_THREADS = 128;

__device__ __forceinline__ void quat_from_matrix(const double* r, double* q) {
  const double m00 = r[0], m11 = r[4], m22 = r[8];
  const double tr = m00 + m11 + m22;
  int c = 0;
  double best = tr;
  if (m00 > best) { best = m00; c = 1; }
  if (m11 > best) { best = m11; c = 2; }
  if (m22 > best) { best = m22; c = 3; }
  if (c == 0) {
    const double w = sqrt(fmax(1.0 + m00 + m11 + m22, 0.0)) / 2.0;
    q[0] = w; q[1] = (r[7] - r[5]) / (4.0 * w); q[2] = (r[2] - r[6]) / (4.0 * w); q[3] = (r[3] - r[1]) / (4.0 * w);
  } else if (c == 1) {
    const double x = sqrt(fmax(1.0 + m00 - m11 - m22, 0.0)) / 2.0;
    q[0] = (r[7] - r[5]) / (4.0 * x); q[1] = x; q[2] = (r[1] + r[3]) / (4.0 * x); q[3] = (r[2] + r[6]) / (4.0 * x);
  } else if (c == 2) {
    const double y = sqrt(fmax(1.0 - m00 + m11 - m22, 0.0)) / 2.0;
    q[0] = (r[2] - r[6]) / (4.0 * y); q[1] = (r[1] + r[3]) / (4.0 * y); q[2] = y; q[3] = (r[5] + r[7]) / (4.0 * y);
  } else {
    const double z = sqrt(fmax(1.0 - m00 - m11 + m22, 0.0)) / 2.0;
    q[0] = (r[3] - r[1]) / (4.0 * z); q[1] = (r[2] + r[6]) / (4.0 * z); q[2] = (r[5] + r[7]) / (4.0 * z); q[3] = z;
  }
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}

__device__ __forceinline__ void quat_to_matrix(const double* qin, double* R) {
  const double n = sqrt(qin[0] * qin[0] + qin[1] * qin[1] + qin[2] * qin[2] + qin[3] * qin[3]);
  const double w = qin[0] / n, x = qin[1] / n, y = qin[2] / n, z = qin[3] / n;
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w); R[2] = 2 * (x * z + y * w);
  R[3] = 2 * (x * y + z * w); R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
  R[6] = 2 * (x * z - y * w); R[7] = 2 * (y * z + x * w); R[8] = 1 - 2 * (x * x + y * y);
}

// frame groups: rows frame_start[f] .. frame_start[f+1] of the (sync, object, camera id)-sorted PnP poses; pair_off[f] =
// number of combinations in earlier groups.  Combination m of group f is the l-th entry of np.triu_indices(s, 1).
__global__ void rel_pose_kernel(const long long* __restrict__ pair_off, const int* __restrict__ frame_start, int n_frames,
                                long long M, const int* __restrict__ cam_id, const int* __restrict__ cam_pos,
                                const double* __restrict__ R, const double* __restrict__ t, unsigned span,
                                unsigned* __restrict__ key, unsigned* __restrict__ idx, double* __restrict__ Rr,
                                double* __restrict__ tr, double* __restrict__ q, double* __restrict__ tmag,
                                unsigned char* __restrict__ valid_out) {
  const long long m = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (m >= M) return;
  int lo = 0, hi = n_frames;  // largest f with pair_off[f] <= m
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (pair_off[mid] <= m) lo = mid; else hi = mid;
  }
  const int f = lo, b0 = frame_start[f], n = frame_start[f + 1] - b0;
  const long long k = m - pair_off[f];
  int i = (int)((2.0 * n - 1.0 - sqrt((2.0 * n - 1.0) * (2.0 * n - 1.0) - 8.0 * (double)k)) * 0.5);
  if (i < 0) i = 0;
  while ((long long)i * (2 * n - i - 1) / 2 > k) --i;
  while ((long long)(i + 1) * (2 * n - i - 2) / 2 <= k) ++i;
  const int j = (int)(k - (long long)i * (2 * n - i - 1) / 2) + i + 1;
  const int ga = b0 + i, gb = b0 + j;
  idx[m] = (unsigned)m;
  const unsigned invalid = span * span;
  const bool formed = cam_pos[ga] < cam_pos[gb];  // the reference forms (first, second) in dict order and keeps first < second
  if (valid_out) valid_out[m] = formed ? 1 : 0;
  if (!formed) { key[m] = invalid; return; }
  const double* Ra = R + 9 * (size_t)ga;
  const double* Rb = R + 9 * (size_t)gb;
  const double* ta = t + 3 * (size_t)ga;
  const double* tb = t + 3 * (size_t)gb;
  double rr[9], tt[3], tai[3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int c = 0; c < 3; ++c) rr[3 * a + c] = Rb[3 * a] * Ra[3 * c] + Rb[3 * a + 1] * Ra[3 * c + 1] + Rb[3 * a + 2] * Ra[3 * c + 2];
#pragma unroll
  for (int c = 0; c < 3; ++c) tai[c] = -(Ra[c] * ta[0] + Ra[3 + c] * ta[1] + Ra[6 + c] * ta[2]);
#pragma unroll
  for (int a = 0; a < 3; ++a) tt[a] = Rb[3 * a] * tai[0] + Rb[3 * a + 1] * tai[1] + Rb[3 * a + 2] * tai[2] + tb[a];
  bool fin = true;
#pragma unroll
  for (int a = 0; a < 9; ++a) fin = fin && isfinite(rr[a]);
#pragma unroll
  for (int a = 0; a < 3; ++a) fin = fin && isfinite(tt[a]);
  if (!fin) { key[m] = invalid; return; }  // the reference's NaN filter (:364-367)
  key[m] = (unsigned)cam_id[ga] * span + (unsigned)cam_id[gb];
  double qq[4];
  quat_from_matrix(rr, qq);
#pragma unroll
  for (int a = 0; a < 9; ++a) Rr[9 * (size_t)m + a] = rr[a];
#pragma unroll
  for (int a = 0; a < 3; ++a) tr[3 * (size_t)m + a] = tt[a];
#pragma unroll
  for (int a = 0; a < 4; ++a) q[4 * (size_t)m + a] = qq[a];
  tmag[m] = sqrt(tt[0] * tt[0] + tt[1] * tt[1] + tt[2] * tt[2]);
}

// rows into pair-sorted order (perm = values of the radix sort), plus the segment id of each sorted row
__global__ void rel_gather_kernel(const unsigned* __restrict__ perm, long long Mv, const double* __restrict__ Rr,
                                  const double* __restrict__ tr, const double* __restrict__ q,
                                  const double* __restrict__ tmag, double* __restrict__ Rs, double* __restrict__ ts,
                                  double* __restrict__ qs, double* __restrict__ tmag_s) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= Mv) return;
  const size_t m = perm[i];
#pragma unroll
  for (int a = 0; a < 9; ++a) Rs[9 * (size_t)i + a] = Rr[9 * m + a];
#pragma unroll
  for (int a = 0; a < 3; ++a) ts[3 * (size_t)i + a] = tr[3 * m + a];
#pragma unroll
  for (int a = 0; a < 4; ++a) qs[4 * (size_t)i + a] = q[4 * m + a];
  tmag_s[i] = tmag[m];
}
__global__ void seg_fill_kernel(const int* __restrict__ seg_off, int n_seg, int* __restrict__ seg) {
  const int s = blockIdx.x;
  if (s >= n_seg) return;
  for (int i = seg_off[s] + threadIdx.x; i < seg_off[s + 1]; i += blockDim.x) seg[i] = s;
}

// numpy.percentile(v, [25, 75]) of every sorted segment ('linear' method, numpy's _lerp)
__device__ __forceinline__ double np_percentile_sorted(const double* v, int cnt, double q01) {
  const double vi = (double)(cnt - 1) * q01;
  const double fl = floor(fmax(vi, 0.0));
  const int lo = (int)fl;
  const int hi = min(lo + 1, max(cnt - 1, 0));
  const double a = v[lo], b = v[hi], tt = vi - floor(vi);
  const double d = __dsub_rn(b, a);
  if (d == 0.0) return a;
  if (tt >= 0.5) return __dsub_rn(b, __dmul_rn(d, __dsub_rn(1.0, tt)));
  return __dadd_rn(a, __dmul_rn(d, tt));
}
__global__ void seg_quartile_kernel(const double* __restrict__ sorted, const int* __restrict__ seg_off, int n_seg,
                                    double* __restrict__ q1, double* __restrict__ q3) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_seg) return;
  const int b = seg_off[s], cnt = seg_off[s + 1] - b;
  if (cnt <= 0) { q1[s] = 0.0; q3[s] = 0.0; return; }
  q1[s] = np_percentile_sorted(sorted + b, cnt, 25.0 / 100.0);
  q3[s] = np_percentile_sorted(sorted + b, cnt, 75.0 / 100.0);
}

// block per camera pair: eigenvector of sum q q^T (largest eigenvalue, w >= 0) over the rows with mask != 0 (all rows when
// mask == nullptr), sum of t, row count, first such row.  Outputs the mean rotation as a matrix; a single row is passed
// through untouched (the reference returns the lone sample itself, :551-553).
__global__ void __launch_bounds__(REL_THREADS)
quat_average_kernel(const int* __restrict__ seg_off, int n_seg, const double* __restrict__ qs,
                    const double* __restrict__ ts, const double* __restrict__ Rs, const unsigned char* __restrict__ mask,
                    double* __restrict__ R_out, double* __restrict__ t_out, long long* __restrict__ cnt_out) {
  __shared__ double sh[REL_THREADS / 32][14];
  __shared__ int sh_first[REL_THREADS / 32];
  const int s = blockIdx.x;
  if (s >= n_seg) return;
  const int b = seg_off[s], e = seg_off[s + 1];
  double acc[14];
#pragma unroll
  for (int k = 0; k < 14; ++k) acc[k] = 0.0;
  int first = 0x7fffffff;
  for (int i = b + threadIdx.x; i < e; i += REL_THREADS) {
    if (mask && !mask[i]) continue;
    const double q0 = qs[4 * (size_t)i], q1 = qs[4 * (size_t)i + 1], q2 = qs[4 * (size_t)i + 2], q3 = qs[4 * (size_t)i + 3];
    acc[0] += q0 * q0; acc[1] += q0 * q1; acc[2] += q0 * q2; acc[3] += q0 * q3;
    acc[4] += q1 * q1; acc[5] += q1 * q2; acc[6] += q1 * q3;
    acc[7] += q2 * q2; acc[8] += q2 * q3; acc[9] += q3 * q3;
    acc[10] += ts[3 * (size_t)i]; acc[11] += ts[3 * (size_t)i + 1]; acc[12] += ts[3 * (size_t)i + 2];
    acc[13] += 1.0;
    first = min(first, i);
  }
#pragma unroll
  for (int k = 0; k < 14; ++k)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 14; ++k) sh[wid][k] = acc[k];
    sh_first[wid] = first;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
#pragma unroll
  for (int k = 0; k < 14; ++k) {
    double v = 0.0;
    for (int w = 0; w < REL_THREADS / 32; ++w) v += sh[w][k];
    acc[k] = v;
  }
  for (int w = 0; w < REL_THREADS / 32; ++w) first = min(first, sh_first[w]);
  const long long cnt = (long long)(acc[13] + 0.5);
  cnt_out[s] = cnt;
  double* Ro = R_out + 9 * (size_t)s;
  double* to = t_out + 3 * (size_t)s;
  if (cnt == 0) {
#pragma unroll
    for (int k = 0; k < 9; ++k) Ro[k] = 0.0;
    to[0] = to[1] = to[2] = 0.0;
    return;
  }
  if (cnt == 1) {
#pragma unroll
    for (int k = 0; k < 9; ++k) Ro[k] = Rs[9 * (size_t)first + k];
#pragma unroll
    for (int k = 0; k < 3; ++k) to[k] = ts[3 * (size_t)first + k];
    return;
  }
  double A[4][4];  // -sum q q^T: its smallest eigenvalue is the largest of the sum
  A[0][0] = -acc[0]; A[0][1] = A[1][0] = -acc[1]; A[0][2] = A[2][0] = -acc[2]; A[0][3] = A[3][0] = -acc[3];
  A[1][1] = -acc[4]; A[1][2] = A[2][1] = -acc[5]; A[1][3] = A[3][1] = -acc[6];
  A[2][2] = -acc[7]; A[2][3] = A[3][2] = -acc[8]; A[3][3] = -acc[9];
  double q[4];
  sym4_min_eigvec(A, q);
  if (q[0] < 0.0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
  quat_to_matrix(q, Ro);
  const double c = (double)cnt;
  to[0] = acc[10] / c; to[1] = acc[11] / c; to[2] = acc[12] / c;
}

// angle (degrees) between each sample and the mean rotation of its pair: acos((trace(R Rm^T) - 1) / 2), trace clipped to [-1, 3]
__global__ void rel_angle_kernel(const double* __restrict__ Rs, const int* __restrict__ seg, const double* __restrict__ Rm,
                                 long long Mv, double* __restrict__ ang) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= Mv) return;
  const double* r = Rs + 9 * (size_t)i;
  const double* m = Rm + 9 * (size_t)seg[i];
  double tr = 0.0;
#pragma unroll
  for (int k = 0; k < 9; ++k) tr += r[k] * m[k];
  tr = fmin(fmax(tr, -1.0), 3.0);
  ang[i] = acos((tr - 1.0) / 2.0) * (180.0 / 3.14159265358979323846);
}

// IQR rule (reject_outliers :369-400): applied to pairs with at least 5 samples; comparisons with NaN are false (kept), as in NumPy
__global__ void rel_flag_kernel(const int* __restrict__ seg, const int* __restrict__ seg_off, long long Mv,
                                const double* __restrict__ tmag, const double* __restrict__ ang,
                                const double* __restrict__ tq1, const double* __restrict__ tq3,
                                const double* __restrict__ rq1, const double* __restrict__ rq3, double rot_m, double tr_m,
                                const unsigned* __restrict__ perm, unsigned char* __restrict__ ok,
                                unsigned char* __restrict__ keep_out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= Mv) return;
  const int s = seg[i];
  const bool big = seg_off[s + 1] - seg_off[s] >= 5;
  const double ti = __dsub_rn(tq3[s], tq1[s]), ri = __dsub_rn(rq3[s], rq1[s]);
  const double t_lo = __dsub_rn(tq1[s], __dmul_rn(tr_m, ti)), t_hi = __dadd_rn(tq3[s], __dmul_rn(tr_m, ti));
  const double r_hi = __dadd_rn(rq3[s], __dmul_rn(rot_m, ri));
  const bool bad = (tmag[i] < t_lo) || (tmag[i] > t_hi) || (ang[i] > r_hi);
  const unsigned char k = (bad && big) ? 0 : 1;
  ok[i] = k;
  if (keep_out) keep_out[perm[i]] = k;
}

}  // namespace cb
