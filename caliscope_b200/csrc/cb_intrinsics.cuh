// Intrinsic calibration of every camera from its planar-board views (cb_calibrate_intrinsics, DESIGN.md section 4.10):
// pinhole + Brown-Conrady (k1 k2 p1 p2 k3), the model and optimum of cv2.calibrateCamera.
//
//   intr_view_kernel   one warp per view (rows of one key): view status and the Harker-O'Leary homography from the
//                      board plane to the pixels (ho_fit, shared with pnp_ippe_kernel, on full-precision inputs)
//   intr_zhang_kernel  one thread per camera: the guess, or Zhang's closed form from the homographies in view order
//   intr_pose_kernel   one thread per view: the IPPE pose of pnp_ippe_kernel as (r, t), or status 5
//   intr_lm_kernel     one thread-block cluster per camera: Levenberg-Marquardt over the free intrinsics and every view
//                      pose with the views eliminated (Schur form), no host round trip per iteration
//   intr_cov_kernel    one cluster per camera: the covariance at the solution
//
// The two cluster kernels share one layout.  Warps take the camera's views round-robin (view j of the camera's list to
// warp j mod (cluster warps)); per view, a warp forms the packed 16 x 16 Gram matrix of [J_theta J_q | r] over the
// view's rows (the 136 entries are U (9x9), W (9x6), V (6x6), g and the cost), staging 32 rows' Jacobians in shared
// memory and giving each lane a fixed set of entries, so every sum over rows runs in row order.  Sums over views run
// in a fixed split: each CTA sums a contiguous range of the view list, the CTAs' partials are added in rank order by
// rank 0 through distributed shared memory.  No floating-point atomics: repeated calls are bit-identical.
#pragma once
#include <cooperative_groups.h>

#include "cb_bootstrap.cuh"
#include "cb_resect.cuh"

namespace cb {

namespace cg = cooperative_groups;

constexpr int INTR_THREADS = 256, INTR_WARPS = INTR_THREADS / 32, INTR_MAX_CLUSTER = 8;
constexpr int INTR_USE_GUESS = 1 << 9;
constexpr int IV_OK = 0, IV_TOO_FEW = 1, IV_NON_PLANAR = 2, IV_DEGENERATE = 5, IV_MULTI_CAM = 6;
constexpr int IC_OK = 0, IC_TOO_FEW_VIEWS = 1, IC_NO_START = 2, IC_NOT_PD = 3, IC_MAX_ITER = 4;
constexpr int INTR_G = 136;    // packed upper 16 x 16 Gram of [J_theta (9) J_q (6) | r] per view
constexpr int INTR_CON = 64;   // per view: S_v (45), diag U_v (9), rhs_v (9), cost_v (1)
constexpr int INTR_TRIAL = 9;  // per view: q + dq (6), trial cost, |dq|^2, |q|^2
constexpr int INTR_STAGE = 32 * 32;  // doubles of one warp's staging buffer: 32 rows x ([J_u r_u] [J_v r_v])
constexpr size_t INTR_SMEM = sizeof(double) * INTR_WARPS * INTR_STAGE;

// ---- views ---------------------------------------------------------------------------------------------------------
// Per view (rows start[v] .. start[v+1] of rows): camera (of the first row), count, rep_row, status (6, 1, 2, else 0)
// and, for status 0, the homography pixels ~ H (X, Y, 1) with H[8] = 1 (status 5 when it is degenerate).
__global__ void __launch_bounds__(BS_THREADS)
intr_view_kernel(const int* __restrict__ start, const int* __restrict__ rows, const int* __restrict__ obs_cam,
                 const double* __restrict__ obj, const double* __restrict__ px, int n_views, int min_points,
                 int* __restrict__ vcam, int* __restrict__ vcount, int* __restrict__ vrep, int* __restrict__ vstatus,
                 double* __restrict__ vH) {
  const int lane = threadIdx.x & 31;
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  if (g >= n_views) return;
  const int b = start[g], e = start[g + 1], n = e - b;
  const int c0 = obs_cam[rows[b]];
  int multi = 0;
  double sx = 0, sy = 0, su = 0, sv = 0, zmin = 1e300, zmax = -1e300;
  for (int i = b + lane; i < e; i += 32) {
    const int r = rows[i];
    multi |= obs_cam[r] != c0;
    const double z = obj[3 * (size_t)r + 2];
    sx += obj[3 * (size_t)r]; sy += obj[3 * (size_t)r + 1];
    su += px[2 * (size_t)r]; sv += px[2 * (size_t)r + 1];
    zmin = fmin(zmin, z); zmax = fmax(zmax, z);
    if (z != z) zmax = z;
  }
  multi = __any_sync(0xffffffffu, multi);
  const bool znan = __any_sync(0xffffffffu, zmax != zmax);
  sx = warp_sum(sx); sy = warp_sum(sy); su = warp_sum(su); sv = warp_sum(sv);
  zmax = warp_max(zmax); zmin = -warp_max(-zmin);
  int st = multi ? IV_MULTI_CAM : n < min_points ? IV_TOO_FEW : (znan || !(zmax - zmin < 1e-6)) ? IV_NON_PLANAR : IV_OK;
  double H[9];
  if (st == IV_OK) {
    const double mx = sx / n, my = sy / n, mu = su / n, mv = sv / n;
    HoFit f;
    const bool fit = ho_fit(rows, b, e, lane, n, mx, my, mu, mv, [&](int r, int k) { return obj[3 * (size_t)r + k]; },
                            [&](int r, int k) { return px[2 * (size_t)r + k]; }, f);
    // collinear model points: pnp_ippe_kernel's test
    if (!fit || !(fabs(f.det) > 1e-12 * (f.a00 + f.a11) * (f.a00 + f.a11))) {
      st = IV_DEGENERATE;
    } else {
      // from the centred board frame to (X, Y, 1): H [I | -m]
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        H[3 * k] = f.H[3 * k];
        H[3 * k + 1] = f.H[3 * k + 1];
        H[3 * k + 2] = f.H[3 * k + 2] - f.H[3 * k] * mx - f.H[3 * k + 1] * my;
      }
      const double h8 = H[8];
      bool fin = h8 != 0.0;
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        H[k] /= h8;
        fin = fin && isfinite(H[k]);
      }
      if (!fin) st = IV_DEGENERATE;
    }
  }
  if (lane == 0) {
    vcam[g] = c0;
    vcount[g] = n;
    vrep[g] = rows[b];
    vstatus[g] = st;
#pragma unroll
    for (int k = 0; k < 9; ++k) vH[9 * g + k] = st == IV_OK ? H[k] : __longlong_as_double(0x7ff8000000000000LL);
  }
}

// ---- start ---------------------------------------------------------------------------------------------------------
// theta[c] = the guess (bit INTR_USE_GUESS) or Zhang's closed form over the views hv_list[hv_start[c] .. hv_start[c+1])
// (the camera's views with a homography, key order): cv2.initIntrinsicParams2D without an aspect ratio; status 2 when
// 1/fx^2 or 1/fy^2 comes out <= 0 or not finite (theta NaN).
__global__ void intr_zhang_kernel(const int* __restrict__ cflags, const double* __restrict__ guess,
                                  const int* __restrict__ isize, const int* __restrict__ hv_start,
                                  const int* __restrict__ hv_list, const double* __restrict__ vH, int n_cams,
                                  double* __restrict__ theta, int* __restrict__ cstatus) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cams) return;
  double* th = theta + 9 * (size_t)c;
  if (cflags[c] & INTR_USE_GUESS) {
    for (int k = 0; k < 9; ++k) th[k] = guess[9 * (size_t)c + k];
    cstatus[c] = IC_OK;
    return;
  }
  const double cx = (isize[2 * c] - 1) * 0.5, cy = (isize[2 * c + 1] - 1) * 0.5;
  double m00 = 0, m01 = 0, m11 = 0, r0 = 0, r1 = 0;
  for (int j = hv_start[c]; j < hv_start[c + 1]; ++j) {
    const double* H = vH + 9 * (size_t)hv_list[j];
    double h[3], v[3], d1[3], d2[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double s = k == 0 ? cx : k == 1 ? cy : 0.0;
      h[k] = H[3 * k] - H[6] * s;
      v[k] = H[3 * k + 1] - H[7] * s;
      d1[k] = (h[k] + v[k]) * 0.5;
      d2[k] = (h[k] - v[k]) * 0.5;
    }
    const double nh = 1.0 / sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2]);
    const double nv = 1.0 / sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    const double n1 = 1.0 / sqrt(d1[0] * d1[0] + d1[1] * d1[1] + d1[2] * d1[2]);
    const double n2 = 1.0 / sqrt(d2[0] * d2[0] + d2[1] * d2[1] + d2[2] * d2[2]);
    const double s1 = nh * nv, s2 = n1 * n2;
    const double A00 = h[0] * v[0] * s1, A01 = h[1] * v[1] * s1, b0 = -h[2] * v[2] * s1;
    const double A10 = d1[0] * d2[0] * s2, A11 = d1[1] * d2[1] * s2, b1 = -d1[2] * d2[2] * s2;
    m00 += A00 * A00 + A10 * A10; m01 += A00 * A01 + A10 * A11; m11 += A01 * A01 + A11 * A11;
    r0 += A00 * b0 + A10 * b1; r1 += A01 * b0 + A11 * b1;
  }
  const double det = m00 * m11 - m01 * m01;
  const double fa = (m11 * r0 - m01 * r1) / det, fb = (m00 * r1 - m01 * r0) / det;
  if (isfinite(fa) && isfinite(fb) && fa > 0.0 && fb > 0.0) {
    const double t[9] = {sqrt(1.0 / fa), sqrt(1.0 / fb), cx, cy, 0, 0, 0, 0, 0};
    for (int k = 0; k < 9; ++k) th[k] = t[k];
    cstatus[c] = IC_OK;
  } else {
    for (int k = 0; k < 9; ++k) th[k] = __longlong_as_double(0x7ff8000000000000LL);
    cstatus[c] = IC_NO_START;
  }
}

// q[v] = (rotation vector of R, t) of pnp_ippe_kernel's pose for every status-0 view of a camera with a start; status 5
// when that pose failed or is not finite.
__global__ void intr_pose_kernel(const int* __restrict__ vcam, const int* __restrict__ cstatus,
                                 const double* __restrict__ R, const double* __restrict__ t,
                                 const int* __restrict__ pnp_status, int n_views, int* __restrict__ vstatus,
                                 double* __restrict__ q) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_views) return;
  double qv[6];
  res_rot_log(R + 9 * (size_t)v, qv);
  bool ok = pnp_status[v] == PNP_OK || pnp_status[v] == PNP_OK_FALLBACK;
#pragma unroll
  for (int k = 0; k < 3; ++k) qv[3 + k] = t[3 * (size_t)v + k];
#pragma unroll
  for (int k = 0; k < 6; ++k) ok = ok && isfinite(qv[k]);
  const bool live = vstatus[v] == IV_OK && cstatus[vcam[v]] == IC_OK;
  if (live && !ok) vstatus[v] = IV_DEGENERATE;
#pragma unroll
  for (int k = 0; k < 6; ++k) q[6 * (size_t)v + k] = (live && ok) ? qv[k] : __longlong_as_double(0x7ff8000000000000LL);
}

// ---- Levenberg-Marquardt and covariance ---------------------------------------------------------------------------
struct IntrArgs {
  const int* start;     // view v's rows: rows[start[v] .. start[v+1])
  const int* rows;
  const double* obj;    // (n, 3) board coordinates
  const double* px;     // (n, 2) pixels
  const int* cams;      // the cameras to solve, one cluster each
  const int* uv_start;  // used views of camera c: uv_list[uv_start[c] .. uv_start[c+1]) (view indices, key order)
  const int* uv_list;
  const int* cflags;
  const int* crows;     // rows over the camera's used views
  double* theta;        // (n_cams, 9), in / out
  double* q;            // (n_views, 6), in / out
  double* gram;         // (used views, INTR_G), slot = position in uv_list
  double* con;          // (used views, INTR_CON)
  double* trial;        // (used views, INTR_TRIAL)
  int* cstatus;
  int* iters;
  double* sse;          // (n_cams) SSE at the solution
  double* std_out;      // (n_cams, 9)
  double* cov_out;      // (n_cams, 81), nullable
  double* sigma2;
  double* vstd;         // (n_views, 6)
  double* vrmse;        // (n_views)
  int max_iter;
  double xtol;
};

// camera table entry (project_obs' layout) of pose q with intrinsics th
__device__ __forceinline__ void intr_entry(const double* th, const double* q, double* E) {
  cam_prep_rot(q[0], q[1], q[2], E);
  E[CT_T + 0] = q[3]; E[CT_T + 1] = q[4]; E[CT_T + 2] = q[5];
  E[CT_FX] = th[0]; E[CT_FY] = th[1]; E[CT_CX] = th[2]; E[CT_CY] = th[3];
#pragma unroll
  for (int k = 0; k < 5; ++k) E[CT_D + k] = th[4 + k];
}

// one row's [J_theta J_q | r] for u (ju) and v (jv), pixels
__device__ __forceinline__ void intr_row(const double* E, const double* X, double2 p, double* ju, double* jv) {
  ProjOut o;
  project_obs<true>(E, false, X[0], X[1], X[2], o);
  const double fx = E[CT_FX], fy = E[CT_FY], a = o.a, b = o.b, r2 = o.r2;
  ju[0] = o.xd; ju[1] = 0.0; ju[2] = 1.0; ju[3] = 0.0;
  jv[0] = 0.0; jv[1] = o.yd; jv[2] = 0.0; jv[3] = 1.0;
  ju[4] = fx * a * r2; ju[5] = ju[4] * r2; ju[8] = ju[5] * r2;
  jv[4] = fy * b * r2; jv[5] = jv[4] * r2; jv[8] = jv[5] * r2;
  ju[6] = fx * 2.0 * a * b; ju[7] = fx * (r2 + 2.0 * a * a);
  jv[6] = fy * (r2 + 2.0 * b * b); jv[7] = fy * 2.0 * a * b;
  const double sx = fx * o.iz, sy = fy * o.iz;
  double Jt[6];
  Jt[0] = sx * o.xa; Jt[1] = sx * o.xb; Jt[2] = -(Jt[0] * a + Jt[1] * b);
  Jt[3] = sy * o.ya; Jt[4] = sy * o.yb; Jt[5] = -(Jt[3] * a + Jt[4] * b);
  const double* R = E + CT_R;
  const double* Jr = E + CT_JR;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    double* J = i == 0 ? ju : jv;
    double JX[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) JX[k] = Jt[3 * i] * R[k] + Jt[3 * i + 1] * R[3 + k] + Jt[3 * i + 2] * R[6 + k];
    const double c0 = JX[1] * X[2] - JX[2] * X[1], c1 = JX[2] * X[0] - JX[0] * X[2], c2 = JX[0] * X[1] - JX[1] * X[0];
#pragma unroll
    for (int k = 0; k < 3; ++k) J[9 + k] = -(c0 * Jr[k] + c1 * Jr[3 + k] + c2 * Jr[6 + k]);
#pragma unroll
    for (int k = 0; k < 3; ++k) J[12 + k] = Jt[3 * i + k];
  }
  ju[15] = o.u - p.x;
  jv[15] = o.v - p.y;
}

// The view's packed Gram matrix of [J | r] at (th, q) into g (global), one warp; lane l owns entries l, l+32, ...
__device__ __forceinline__ void intr_gram(const IntrArgs& A, const double* th, const double* q, int v, double* g,
                                          double* stage, int lane) {
  double E[CT_SIZE];
  intr_entry(th, q, E);
  int ep[5], eq[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    int e = lane + 32 * k, p = 0;
    while (e >= 16 - p && p < 16) { e -= 16 - p; ++p; }
    ep[k] = p; eq[k] = p + e;
  }
  double acc[5] = {0, 0, 0, 0, 0};
  const int b = A.start[v], e = A.start[v + 1];
  for (int base = b; base < e; base += 32) {
    const int i = base + lane;
    if (i < e) {
      const int r = A.rows[i];
      intr_row(E, A.obj + 3 * (size_t)r, reinterpret_cast<const double2*>(A.px)[r], stage + 32 * lane,
               stage + 32 * lane + 16);
    }
    __syncwarp();
    const int nr = min(32, e - base);
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      if (lane + 32 * k < INTR_G) {
        const int p = ep[k], c = eq[k];
        double s = acc[k];
        for (int rr = 0; rr < nr; ++rr) {
          const double* row = stage + 32 * rr;
          s = fma(row[p], row[c], fma(row[16 + p], row[16 + c], s));
        }
        acc[k] = s;
      }
    }
    __syncwarp();
  }
#pragma unroll
  for (int k = 0; k < 5; ++k)
    if (lane + 32 * k < INTR_G) g[lane + 32 * k] = acc[k];
  __syncwarp();
}

// Cholesky of the view block V + lam diag V
__device__ __forceinline__ bool intr_chol_v(const double* g, double lam, double L[6][6]) {
  double h[21];
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = i; j < 6; ++j) h[ut<6>(i, j)] = g[ut<16>(9 + i, 9 + j)] * (i == j ? 1.0 + lam : 1.0);
  return res_chol<6>(h, 0.0, L);
}

// The view's Schur contribution at damping lam into con: row i of S_v = U_v - W_v V_lam^-1 W_v^T on lane i < 9, diag
// U_v, rhs_v = g_theta - W_v V_lam^-1 g_q, cost (NaN in S_v when V_lam is not positive definite)
__device__ __forceinline__ void intr_schur(const double* g, double lam, double* con, int lane) {
  if (lane < 9) {
    const int i = lane;
    double L[6][6];
    const bool ok = intr_chol_v(g, lam, L);
    double y[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) y[k] = g[ut<16>(i, 9 + k)];
    res_chol_solve<6>(L, y);
    for (int j = i; j < 9; ++j) {
      double s = g[ut<16>(i <= j ? i : j, j)];
#pragma unroll
      for (int k = 0; k < 6; ++k) s -= y[k] * g[ut<16>(j, 9 + k)];
      con[ut<9>(i, j)] = ok ? s : __longlong_as_double(0x7ff8000000000000LL);
    }
    double rh = g[ut<16>(i, 15)];
#pragma unroll
    for (int k = 0; k < 6; ++k) rh -= y[k] * g[ut<16>(9 + k, 15)];
    con[45 + i] = g[ut<16>(i, i)];
    con[54 + i] = rh;
  }
  if (lane == 0) con[63] = g[ut<16>(15, 15)];
  __syncwarp();
}

// Fixed-order sum over the camera's n view slots of columns [0, ncols) of src (row stride ld) into `out` of rank 0:
// each CTA sums a contiguous range (split in two halves over its threads), rank 0 adds the CTAs' partials in rank order.
// Every thread of the cluster calls it after writing its rows of src; on return rank 0's `out` holds the sums.
__device__ __forceinline__ void intr_reduce(cg::cluster_group& cl, const double* src, int ld, int n, int ncols,
                                            double* part, double* cta, double* out) {
  const int tid = threadIdx.x, rank = (int)cl.block_rank(), cs = (int)cl.num_blocks();
  const int lo = (int)((long long)n * rank / cs), hi = (int)((long long)n * (rank + 1) / cs);
  const int nsub = INTR_THREADS / 64, col = tid % 64, sub = tid / 64;
  __threadfence();
  cl.sync();  // every warp of the cluster has written its views' rows of src
  if (col < ncols) {
    const int a = lo + (int)((long long)(hi - lo) * sub / nsub), z = lo + (int)((long long)(hi - lo) * (sub + 1) / nsub);
    double s = 0.0;
    for (int j = a; j < z; ++j) s += src[(size_t)j * ld + col];
    part[tid] = s;
  }
  __syncthreads();
  if (tid < ncols) {
    double s = 0.0;
    for (int k = 0; k < nsub; ++k) s += part[64 * k + tid];
    cta[tid] = s;
  }
  __threadfence();
  cl.sync();
  if (rank == 0 && tid < ncols) {
    double s = 0.0;
    for (int r = 0; r < cs; ++r) s += cl.map_shared_rank(cta, r)[tid];
    out[tid] = s;
  }
  __syncthreads();
}

// 9 x 9 S (packed ut<9>) restricted to the free parameters (fixed rows / columns become the identity); Cholesky factor
// L (lower, row-major); pivots must exceed thr (of the Jacobi-scaled matrix when scaled)
__device__ __forceinline__ bool intr_chol9(const double* Sp, int fixed, bool scaled, double thr, double L[9][9],
                                           double* d) {
#pragma unroll 1
  for (int i = 0; i < 9; ++i) d[i] = ((fixed >> i) & 1) ? 1.0 : (scaled ? 1.0 / sqrt(Sp[ut<9>(i, i)]) : 1.0);
  bool ok = true;
#pragma unroll 1
  for (int j = 0; j < 9; ++j) {
    for (int i = j; i < 9; ++i) {
      const bool fx = ((fixed >> i) & 1) || ((fixed >> j) & 1);
      double v = fx ? (i == j ? 1.0 : 0.0) : Sp[ut<9>(j, i)] * d[i] * d[j];
      for (int k = 0; k < j; ++k) v -= L[i][k] * L[j][k];
      if (i == j) {
        ok = ok && v > thr;
        L[j][j] = sqrt(v);
      } else {
        L[i][j] = v / L[j][j];
      }
    }
  }
  return ok;
}

__device__ __forceinline__ void intr_chol9_solve(const double L[9][9], double* x) {
#pragma unroll 1
  for (int i = 0; i < 9; ++i) {
    double a = x[i];
    for (int k = 0; k < i; ++k) a -= L[i][k] * x[k];
    x[i] = a / L[i][i];
  }
#pragma unroll 1
  for (int i = 8; i >= 0; --i) {
    double a = x[i];
    for (int k = i + 1; k < 9; ++k) a -= L[k][i] * x[k];
    x[i] = a / L[i][i];
  }
}

struct IntrShared {
  double part[INTR_THREADS];
  double cta[INTR_CON];
  double tot[INTR_CON];
  double bc[16];  // rank 0's broadcast: 9 values, flag, done
  double th[9];
  double dth[9];
};

// One cluster per camera cams[blockIdx.x / cluster size]: Levenberg-Marquardt (DESIGN.md section 4.10, lm_iterate's
// acceptance and stopping rules) from theta and q, writing theta, q, the SSE, the iterations and status 0 / 4.
__global__ void __launch_bounds__(INTR_THREADS)
intr_lm_kernel(IntrArgs A) {
  cg::cluster_group cl = cg::this_cluster();
  extern __shared__ double stage_all[];
  __shared__ IntrShared sh;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rank = (int)cl.block_rank(), cs = (int)cl.num_blocks();
  const int c = A.cams[blockIdx.x / cs];
  const int fixed = A.cflags[c] & 511;
  const int v0 = A.uv_start[c], nv = A.uv_start[c + 1] - v0;
  const int gw = rank * INTR_WARPS + warp, nw = cs * INTR_WARPS;
  double* stage = stage_all + warp * INTR_STAGE;
  if (tid < 9) sh.th[tid] = A.theta[9 * (size_t)c + tid];
  __syncthreads();
  double lam = TRI_LAMBDA0, cost = 0.0;  // rank 0 thread 0's
  int it = 0, st = IC_OK;
  bool relin = true;
  while (true) {
    for (int j = gw; j < nv; j += nw) {
      const int v = A.uv_list[v0 + j];
      double* g = A.gram + (size_t)(v0 + j) * INTR_G;
      if (relin) intr_gram(A, sh.th, A.q + 6 * (size_t)v, v, g, stage, lane);
      intr_schur(g, lam, A.con + (size_t)(v0 + j) * INTR_CON, lane);
    }
    intr_reduce(cl, A.con + (size_t)v0 * INTR_CON, INTR_CON, nv, INTR_CON, sh.part, sh.cta, sh.tot);
    if (rank == 0 && tid == 0) {
      cost = sh.tot[63];
      double Sp[45], L[9][9], dsc[9], x[9];
      for (int k = 0; k < 45; ++k) Sp[k] = sh.tot[k];
      for (int i = 0; i < 9; ++i) Sp[ut<9>(i, i)] += lam * sh.tot[45 + i];
      const bool ok = intr_chol9(Sp, fixed, false, 0.0, L, dsc);
      for (int i = 0; i < 9; ++i) x[i] = ((fixed >> i) & 1) ? 0.0 : -sh.tot[54 + i];
      if (ok) intr_chol9_solve(L, x);
      for (int i = 0; i < 9; ++i) sh.bc[i] = ((fixed >> i) & 1) ? 0.0 : x[i];
      sh.bc[9] = ok ? 1.0 : 0.0;
      sh.bc[10] = 0.0;
      if (!ok) {  // a damped block not positive definite: a rejected step without the stopping test
        ++it;
        if (it == A.max_iter) { st = IC_MAX_ITER; sh.bc[10] = 1.0; }
      }
    }
    __threadfence();
    cl.sync();
    const double* bc0 = cl.map_shared_rank(sh.bc, 0);
    double bcl[11];
#pragma unroll
    for (int k = 0; k < 11; ++k) bcl[k] = bc0[k];
    if (tid < 9) sh.dth[tid] = bcl[tid];
    __syncthreads();
    if (bcl[9] == 0.0) {
      lam *= 10.0;
      relin = false;
      if (bcl[10] != 0.0) break;
      continue;
    }
    // back-substitution, trial point and its cost
    double tt[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) tt[k] = sh.th[k] + sh.dth[k];
    for (int j = gw; j < nv; j += nw) {
      const int v = A.uv_list[v0 + j];
      const double* g = A.gram + (size_t)(v0 + j) * INTR_G;
      const double* qv = A.q + 6 * (size_t)v;
      double L[6][6], dq[6], qt[6];
      intr_chol_v(g, lam, L);
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        double s = g[ut<16>(9 + k, 15)];
#pragma unroll
        for (int i = 0; i < 9; ++i) s += g[ut<16>(i, 9 + k)] * sh.dth[i];
        dq[k] = s;
      }
      res_chol_solve<6>(L, dq);
      double dq2 = 0.0, q2 = 0.0;
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        dq[k] = -dq[k];
        qt[k] = qv[k] + dq[k];
        dq2 += dq[k] * dq[k];
        q2 += qv[k] * qv[k];
      }
      double E[CT_SIZE];
      intr_entry(tt, qt, E);
      double ct = 0.0;
      for (int i = A.start[v] + lane; i < A.start[v + 1]; i += 32) {
        const int r = A.rows[i];
        ProjOut o;
        project_obs<false>(E, false, A.obj[3 * (size_t)r], A.obj[3 * (size_t)r + 1], A.obj[3 * (size_t)r + 2], o);
        const double eu = o.u - A.px[2 * (size_t)r], ev = o.v - A.px[2 * (size_t)r + 1];
        ct = fma(eu, eu, fma(ev, ev, ct));
      }
      ct = warp_sum(ct);
      double* tr = A.trial + (size_t)(v0 + j) * INTR_TRIAL;
      if (lane < 6) tr[lane] = qt[lane];
      if (lane == 6) tr[6] = ct;
      if (lane == 7) tr[7] = dq2;
      if (lane == 8) tr[8] = q2;
      __syncwarp();
    }
    intr_reduce(cl, A.trial + (size_t)v0 * INTR_TRIAL + 6, INTR_TRIAL, nv, 3, sh.part, sh.cta, sh.tot);
    if (rank == 0 && tid == 0) {
      ++it;
      double dn = sh.tot[1], xn = sh.tot[2];
      for (int i = 0; i < 9; ++i)
        if (!((fixed >> i) & 1)) { dn += sh.dth[i] * sh.dth[i]; xn += sh.th[i] * sh.th[i]; }
      dn = sqrt(dn);
      xn = sqrt(xn);
      const bool lower = sh.tot[0] < cost;
      bool done = dn <= A.xtol * (xn + A.xtol);
      if (!done && it == A.max_iter) { st = IC_MAX_ITER; done = true; }
      sh.bc[9] = lower ? 1.0 : 0.0;
      sh.bc[10] = done ? 1.0 : 0.0;
    }
    __threadfence();
    cl.sync();
    const bool lower = bc0[9] != 0.0, done = bc0[10] != 0.0;
    lam = lower ? lam * 0.1 : lam * 10.0;
    __syncthreads();
    if (lower) {
      if (tid < 9) sh.th[tid] += sh.dth[tid];
      for (int j = gw; j < nv; j += nw)
        if (lane < 6) A.q[6 * (size_t)A.uv_list[v0 + j] + lane] = A.trial[(size_t)(v0 + j) * INTR_TRIAL + lane];
    }
    relin = lower;
    __syncthreads();
    // every CTA has read rank 0's broadcast before rank 0 writes it again (after the next reduction's cluster barrier)
    if (done) break;
  }
  if (relin) {  // the Gram blocks at the final point for the covariance kernel's cost and rmse
    for (int j = gw; j < nv; j += nw)
      intr_gram(A, sh.th, A.q + 6 * (size_t)A.uv_list[v0 + j], A.uv_list[v0 + j], A.gram + (size_t)(v0 + j) * INTR_G,
                stage, lane);
  }
  if (rank == 0 && tid < 9) A.theta[9 * (size_t)c + tid] = sh.th[tid];
  if (rank == 0 && tid == 0) {
    A.cstatus[c] = st;
    A.iters[c] = it;
  }
  cl.sync();  // no CTA leaves while another may still read its shared memory
}

// One cluster per camera: the covariance at the solution (lambda = 0) from the Gram blocks intr_lm_kernel left at the
// final point.  sigma^2 = SSE / (2N - p); status 3 (std NaN) when S is not positive definite.
__global__ void __launch_bounds__(INTR_THREADS)
intr_cov_kernel(IntrArgs A) {
  cg::cluster_group cl = cg::this_cluster();
  __shared__ IntrShared sh;
  __shared__ double sinv[81];
  __shared__ double wbuf[INTR_WARPS][6 * 6 + 6 * 9];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rank = (int)cl.block_rank(), cs = (int)cl.num_blocks();
  const int c = A.cams[blockIdx.x / cs];
  const int fixed = A.cflags[c] & 511;
  const int v0 = A.uv_start[c], nv = A.uv_start[c + 1] - v0;
  const int gw = rank * INTR_WARPS + warp, nw = cs * INTR_WARPS;
  for (int j = gw; j < nv; j += nw)
    intr_schur(A.gram + (size_t)(v0 + j) * INTR_G, 0.0, A.con + (size_t)(v0 + j) * INTR_CON, lane);
  intr_reduce(cl, A.con + (size_t)v0 * INTR_CON, INTR_CON, nv, INTR_CON, sh.part, sh.cta, sh.tot);
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  if (rank == 0 && tid == 0) {
    const double sse = sh.tot[63];
    int nfree = 0;
    for (int i = 0; i < 9; ++i) nfree += !((fixed >> i) & 1);
    const long long N = A.crows[c], p = nfree + 6LL * nv;
    const double s2 = 2 * N > p ? sse / (double)(2 * N - p) : nan;
    double L[9][9], dsc[9];
    bool ok = intr_chol9(sh.tot, fixed, true, TRI_PD_RTOL, L, dsc);
    if (ok) ok = intr_chol9(sh.tot, fixed, false, 0.0, L, dsc);
    for (int j = 0; j < 9; ++j) {
      double x[9];
      for (int i = 0; i < 9; ++i) x[i] = i == j ? 1.0 : 0.0;
      if (ok) intr_chol9_solve(L, x);
      for (int i = 0; i < 9; ++i) sinv[9 * i + j] = !ok ? nan : (((fixed >> i) | (fixed >> j)) & 1) ? 0.0 : x[i];
    }
    if (!ok) A.cstatus[c] = IC_NOT_PD;
    A.sse[c] = sse;
    A.sigma2[c] = s2;
    for (int i = 0; i < 9; ++i) A.std_out[9 * (size_t)c + i] = sqrt(s2 * sinv[10 * i]);
    if (A.cov_out)
      for (int k = 0; k < 81; ++k) A.cov_out[81 * (size_t)c + k] = s2 * sinv[k];
    sh.bc[0] = s2;
  }
  __threadfence();
  cl.sync();
  const double s2 = cl.map_shared_rank(sh.bc, 0)[0];
  const double* si0 = cl.map_shared_rank(sinv, 0);
  if (rank != 0 && tid < 81) sinv[tid] = si0[tid];
  __syncthreads();
  double* vi = wbuf[warp];       // V^-1 (6 x 6)
  double* M = wbuf[warp] + 36;   // V^-1 W^T (6 x 9)
  for (int j = gw; j < nv; j += nw) {
    const int v = A.uv_list[v0 + j];
    const double* g = A.gram + (size_t)(v0 + j) * INTR_G;
    double L[6][6];
    intr_chol_v(g, 0.0, L);
    if (lane < 15) {
      double y[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) y[k] = lane < 6 ? (k == lane ? 1.0 : 0.0) : g[ut<16>(lane - 6, 9 + k)];
      res_chol_solve<6>(L, y);
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        if (lane < 6) vi[6 * k + lane] = y[k];
        else M[9 * k + lane - 6] = y[k];
      }
    }
    __syncwarp();
    if (lane < 6) {
      double s = 0.0;
      for (int a = 0; a < 9; ++a) {
        double t = 0.0;
        for (int b2 = 0; b2 < 9; ++b2) t += sinv[9 * a + b2] * M[9 * lane + b2];
        s += M[9 * lane + a] * t;
      }
      A.vstd[6 * (size_t)v + lane] = sqrt(s2 * (vi[7 * lane] + s));
    }
    if (lane == 0) A.vrmse[v] = sqrt(g[ut<16>(15, 15)] / (A.start[v + 1] - A.start[v]));
    __syncwarp();
  }
  cl.sync();
}

}  // namespace cb
