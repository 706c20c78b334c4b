// Parameter covariance at a bundle-adjustment solution (cb_ba_covariance, DESIGN.md section 4.6).
//
//   pt_pass_kernel<..., COV = true>  (cb_lm.cuh) the point pass at lambda = 0 with the pseudo-inverse root R of V_j
//                                    (V_j^+ = R^T R, pinv_root3) instead of the damped Cholesky: Z_j = W_j R^T into Zt
//   schur_syrk / schur_finalize      unchanged: S = U - Z Z^T, the undamped reduced camera system
//   cov_prep / cov_sweep_* / cov_finish   dense SPD inverse of S with the fixed and masked rows and columns replaced by
//                                    unit vectors: block sweep (Gauss-Jordan) with 32 x 32 pivots, Cholesky-checked
//   cov_point_kernel                 per unconstrained point R^T (I + Z_j^T S^-1 Z_j) R, gathered over the point's own
//                                    cameras (the P x P blocks of S^-1 between every pair of them)
#pragma once
#include "cb_constraints.cuh"

namespace cb {

constexpr double COV_EIG_RTOL = 1e-12;  // eigenvalues of V_j at or below this times the largest count as zero
constexpr int CV_B = 32;                // pivot block edge of the sweep

// Pseudo-inverse root of a symmetric PSD 3x3 (packed 00,01,02,11,12,22): R (row-major) with R^T R = V^+, and rank(V).
// Cyclic Jacobi; row i of R is the i-th eigenvector over the square root of its eigenvalue, zero for a null eigenvalue.
__device__ __forceinline__ void pinv_root3(const double* v, double* R, int& rank) {
  double a[3][3] = {{v[0], v[1], v[2]}, {v[1], v[3], v[4]}, {v[2], v[4], v[5]}};
  double q[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
  for (int sweep = 0; sweep < 8; ++sweep) {
#pragma unroll
    for (int pr = 0; pr < 3; ++pr) {
      const int p = pr == 2 ? 1 : 0, r = pr == 0 ? 1 : 2, o = 3 - p - r;
      const double apr = a[p][r];
      if (!(fabs(apr) > 1e-20 * (fabs(a[p][p]) + fabs(a[r][r])))) { a[p][r] = a[r][p] = 0.0; continue; }
      const double th = (a[r][r] - a[p][p]) / (2.0 * apr);
      const double t = copysign(1.0, th) / (fabs(th) + sqrt(th * th + 1.0));
      const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
      a[p][p] -= t * apr;
      a[r][r] += t * apr;
      a[p][r] = a[r][p] = 0.0;
      const double aop = a[o][p], aor = a[o][r];
      a[o][p] = a[p][o] = c * aop - s * aor;
      a[o][r] = a[r][o] = s * aop + c * aor;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double qp = q[k][p], qr = q[k][r];
        q[k][p] = c * qp - s * qr;
        q[k][r] = s * qp + c * qr;
      }
    }
  }
  const double wmax = fmax(fmax(a[0][0], a[1][1]), fmax(a[2][2], 0.0));
  rank = 0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const bool nz = wmax > 0.0 && a[i][i] > COV_EIG_RTOL * wmax;
    rank += nz ? 1 : 0;
    const double sc = nz ? 1.0 / sqrt(a[i][i]) : 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) R[3 * i + k] = sc * q[k][i];
  }
}

// A (n x n, n a multiple of CV_B) = S on the free parameters, unit rows / columns elsewhere; diag0 = diag(A)
__global__ void cov_prep_kernel(const double* __restrict__ S, int nP, const unsigned char* __restrict__ free_, int n,
                                double* __restrict__ A, double* __restrict__ diag0) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)n * n) return;
  const int i = (int)(idx / n), j = (int)(idx % n);
  const bool f = i < nP && j < nP && free_[i] && free_[j];
  const double v = f ? S[(size_t)i * nP + j] : (i == j ? 1.0 : 0.0);
  A[idx] = v;
  if (i == j) diag0[i] = v;
}

// Pivot block kb of the sweep (one CTA): D = A_kk^-1 through its Cholesky factor, and a copy of the column panel
// C = A[:, kb:kb+32] taken before the update overwrites it.  A pivot at or below rtol times the parameter's own diagonal
// of S marks the matrix as singular: the smallest such global index goes to *fail.
__global__ void __launch_bounds__(CV_B * CV_B)
cov_sweep_pivot_kernel(const double* __restrict__ A, int n, int kb, const double* __restrict__ diag0, double rtol,
                       double* __restrict__ D, double* __restrict__ C, int* __restrict__ fail) {
  __shared__ double L[CV_B][CV_B + 1], Li[CV_B][CV_B + 1];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  L[ty][tx] = A[(size_t)(kb + ty) * n + kb + tx];
  for (int i = threadIdx.x; i < n * CV_B; i += blockDim.x) C[i] = A[(size_t)(i / CV_B) * n + kb + i % CV_B];
  __syncthreads();
  for (int k = 0; k < CV_B; ++k) {
    if (threadIdx.x == 0) {
      double d = L[k][k];
      const double d0 = diag0[kb + k];
      if (!(d > rtol * d0)) {
        atomicMin(fail, kb + k);
        d = d0 > 0.0 ? d0 : 1.0;  // keep the numbers finite; the call reports the failure
      }
      L[k][k] = sqrt(d);
    }
    __syncthreads();
    if (ty == 0 && tx > k) L[tx][k] /= L[k][k];
    __syncthreads();
    if (ty > k && tx > k && tx <= ty) L[ty][tx] -= L[ty][k] * L[tx][k];
    __syncthreads();
  }
  if (ty == 0) {  // Li = L^-1, one lane per column, row by row
    for (int i = 0; i < CV_B; ++i) {
      double s = (i == tx) ? 1.0 : 0.0;
      for (int k = tx; k < i; ++k) s -= L[i][k] * Li[k][tx];
      Li[i][tx] = (tx <= i) ? s / L[i][i] : 0.0;
      __syncwarp();
    }
  }
  __syncthreads();
  double s = 0.0;
  for (int k = max(tx, ty); k < CV_B; ++k) s = fma(Li[k][ty], Li[k][tx], s);
  D[ty * CV_B + tx] = s;
}

// One 32 x 32 tile (I, J) of the sweep on pivot block k (D = A_kk^-1, C = old column panel, A symmetric):
//   A_kk = -D,  A_Ik = C_I D,  A_kJ = D C_J^T,  A_IJ -= C_I D C_J^T.
// After every block has been swept, A = -A0^-1.
__global__ void __launch_bounds__(CV_B * CV_B)
cov_sweep_update_kernel(double* __restrict__ A, int n, int kb, const double* __restrict__ D, const double* __restrict__ C) {
  __shared__ double Ci[CV_B][CV_B + 1], Cj[CV_B][CV_B + 1], Ds[CV_B][CV_B + 1], T[CV_B][CV_B + 1];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int I = blockIdx.y * CV_B, J = blockIdx.x * CV_B;
  Ci[ty][tx] = C[(size_t)(I + ty) * CV_B + tx];
  Cj[ty][tx] = C[(size_t)(J + ty) * CV_B + tx];
  Ds[ty][tx] = D[ty * CV_B + tx];
  __syncthreads();
  double t = 0.0;
#pragma unroll 8
  for (int m = 0; m < CV_B; ++m) t = fma(Ci[ty][m], Ds[m][tx], t);
  T[ty][tx] = t;
  __syncthreads();
  double* a = A + (size_t)(I + ty) * n + J + tx;
  const bool rk = I == kb, ck = J == kb;
  if (rk && ck) {
    *a = -Ds[ty][tx];
  } else if (ck) {
    *a = T[ty][tx];
  } else if (rk) {
    double s = 0.0;
#pragma unroll 8
    for (int m = 0; m < CV_B; ++m) s = fma(Ds[ty][m], Cj[tx][m], s);
    *a = s;
  } else {
    double s = 0.0;
#pragma unroll 8
    for (int m = 0; m < CV_B; ++m) s = fma(T[ty][m], Cj[tx][m], s);
    *a -= s;
  }
}

// Sigma_hat (nP x nP, internal slot order) = S_F^-1 on the free parameters (symmetrised), zero elsewhere
__global__ void cov_finish_kernel(const double* __restrict__ A, int n, int nP, const unsigned char* __restrict__ free_,
                                  double* __restrict__ out) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)nP * nP) return;
  const int i = (int)(idx / nP), j = (int)(idx % nP);
  out[idx] = (free_[i] && free_[j]) ? -0.5 * (A[(size_t)i * n + j] + A[(size_t)j * n + i]) : 0.0;
}

// Smallest component whose factor comp_build_kernel froze (its E was not positive definite: diagonal 1e150)
__global__ void comp_failed_kernel(ConstraintTables T, const double* __restrict__ compL, int* __restrict__ fail) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < T.n_comp && compL[T.comp_L_off[c]] == 1e150) atomicMin(fail, c);
}

// Per-point marginal covariance, one warp per point:  s2 * R^T (I + sum_{c,d} Z_c^T Sigma_hat_cd Z_d) R  over the unique
// cameras c, d of the point (Z_c: the point's three Zt rows in camera c's P columns).  Points whose V_j is rank
// deficient, and points of constraint components (rank -1), get NaN.
template <int P>
__global__ void __launch_bounds__(256)
cov_point_kernel(const int* __restrict__ pt_start, const int* __restrict__ pm_cam, int n_pts, const double* __restrict__ Zt,
                 size_t LD, const double* __restrict__ Sig, int nP, const double* __restrict__ R9,
                 const int* __restrict__ rank, double s2, double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  for (int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); j < n_pts; j += nwarps) {
    if (rank[j] != 3) {
      if (lane < 9) out[9 * (size_t)j + lane] = __longlong_as_double(0x7ff8000000000000ll);
      continue;
    }
    const int s = pt_start[j], k = pt_start[j + 1] - s;
    const double* zrow = Zt + 3 * (size_t)j * LD;
    double m[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
    for (int idx = lane; idx < k * k; idx += 32) {
      const int pa = s + idx / k, pb = s + idx % k;
      if (pb < pa) continue;  // X_dc = X_cd^T: each unordered pair once
      const int ca = pm_cam[pa], cb = pm_cam[pb];
      if ((pa > s && pm_cam[pa - 1] == ca) || (pb > s && pm_cam[pb - 1] == cb)) continue;  // repeated rows of one camera
      double x[3][3];
      cov_pair_gather<P>(zrow + (size_t)ca * P, zrow + (size_t)cb * P, LD, Sig, nP, ca, cb, x);
      const bool same = pa == pb;
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) m[a][b] += same ? x[a][b] : x[a][b] + x[b][a];
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) m[a][b] = warp_sum(m[a][b]);
    if (lane == 0) {
      const double* R = R9 + 9 * (size_t)j;
      double t[3][3];  // (I + m) R
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b)
          t[a][b] = R[3 * a + b] + m[a][0] * R[b] + m[a][1] * R[3 + b] + m[a][2] * R[6 + b];
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b)
          out[9 * (size_t)j + 3 * a + b] = s2 * (R[a] * t[0][b] + R[3 + a] * t[1][b] + R[6 + a] * t[2][b]);
    }
  }
}

}  // namespace cb
