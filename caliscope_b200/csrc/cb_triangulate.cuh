// Kernels for the step in front of bundle adjustment (SURVEY.md §8(f) rank 3):
//   * undistort_kernel     == CameraData.undistort_points  (reference cameras/camera_array.py:135-174, which calls
//                             cv2.undistortPoints / cv2.fisheye.undistortPoints on float32 copies of the points)
//   * tri_* kernels        == triangulate_image_points     (reference core/point_data.py:122-229): group observations
//                             by a 64-bit composite key, DLT system per group, smallest right singular vector.
// Algorithmic traffic is 36 B (undistort) / 24 B (DLT, gathered) per observation; the arithmetic per byte
// (iterative inverse distortion; 4x4 eigen-solve) is high enough that the fp64 pipe, not HBM, is expected to bound both.
#pragma once
#include <cstdint>

#include "cb_device.cuh"

namespace cb {

struct UndistCam {
  double fx, fy, cx, cy, skew;
  double d[12];  // pinhole: k1 k2 p1 p2 k3 k4 k5 k6 s1 s2 s3 s4 ; fisheye: k1..k4
  int fisheye;
  int pad;
};

__device__ __forceinline__ float2 load_px(const double* p, long long i) {
  const double2 v = reinterpret_cast<const double2*>(p)[i];
  return make_float2((float)v.x, (float)v.y);
}
__device__ __forceinline__ float2 load_px(const float* p, long long i) { return reinterpret_cast<const float2*>(p)[i]; }

// Unfused fp64 arithmetic for the undistortion.  OpenCV's x86 build rounds every product and every sum; nvcc would
// contract a * b + c into one fma, which moves the double by up to an ulp, and the float32 result shows that wherever
// the sum cancels (a pixel near 0, x0 - dx near 0).  These three are never contracted.
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }

// float32 in -> double arithmetic -> float32 out, exactly the precision contract of the reference call.  OpenCV's
// expressions in OpenCV's evaluation order, so the only operation that is not bit-exact is the fisheye model's tan().
// TIN = double (caller's array, rounded to float32 here) or float (already rounded on the host while staging).
// Edges as OpenCV has them: a fisheye point whose Newton iteration fails or flips theta's sign is (-1e6, -1e6) in
// both outputs; a NaN theta_d clamps to -pi/2 and iterates (std::max keeps its first argument on NaN); pixel output
// is the homography P [x y 1]^T over its third row, which is NaN in both coordinates when x or y is not finite.
template <typename TIN>
__global__ void undistort_kernel(const UndistCam* __restrict__ cams, const int* __restrict__ obs_cam,
                                 const TIN* __restrict__ xy_in, double* __restrict__ xy_out, long long n,
                                 int to_pixels) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const UndistCam& c = cams[obs_cam ? obs_cam[i] : 0];
  const float2 in = load_px(xy_in, i);
  const double u = (double)in.x, v = (double)in.y;
  double x, y;
  bool sentinel = false;
  if (c.fisheye) {
    const double pwx = sub_rn(u, c.cx) / c.fx, pwy = sub_rn(v, c.cy) / c.fy;
    double theta_d = sqrt(add_rn(mul_rn(pwx, pwx), mul_rn(pwy, pwy)));
    const double half_pi = 1.5707963267948966;
    theta_d = (-half_pi < theta_d) ? theta_d : -half_pi;  // std::min(std::max(-pi/2, theta_d), pi/2)
    theta_d = (half_pi < theta_d) ? half_pi : theta_d;
    bool converged = false;
    double th = theta_d, scale = 0.0;
    if (fabs(theta_d) > 1e-8) {
      for (int j = 0; j < 10; ++j) {
        const double t2 = mul_rn(th, th), t4 = mul_rn(t2, t2), t6 = mul_rn(t4, t2), t8 = mul_rn(t6, t2);
        const double k0 = mul_rn(c.d[0], t2), k1 = mul_rn(c.d[1], t4), k2 = mul_rn(c.d[2], t6), k3 = mul_rn(c.d[3], t8);
        const double num = sub_rn(mul_rn(th, add_rn(add_rn(add_rn(add_rn(1.0, k0), k1), k2), k3)), theta_d);
        const double den = add_rn(add_rn(add_rn(add_rn(1.0, mul_rn(3.0, k0)), mul_rn(5.0, k1)), mul_rn(7.0, k2)),
                                  mul_rn(9.0, k3));
        const double fix = num / den;
        th = sub_rn(th, fix);
        if (fabs(fix) < 1e-8) {
          converged = true;
          break;
        }
      }
      scale = tan(th) / theta_d;
    } else {
      converged = true;
    }
    const bool flipped = (theta_d < 0 && th > 0) || (theta_d > 0 && th < 0);
    if (converged && !flipped) {
      x = mul_rn(pwx, scale);
      y = mul_rn(pwy, scale);
    } else {
      x = -1000000.0;
      y = -1000000.0;
      sentinel = true;
    }
  } else {
    // the reciprocals, as OpenCV scales by them (the fisheye model above divides)
    const double ifx = 1.0 / c.fx, ify = 1.0 / c.fy;
    const double x0 = mul_rn(sub_rn(u, c.cx), ifx), y0 = mul_rn(sub_rn(v, c.cy), ify);
    const double* k = c.d;
    x = x0;
    y = y0;
#pragma unroll 1
    for (int j = 0; j < 5; ++j) {
      const double r2 = add_rn(mul_rn(x, x), mul_rn(y, y));
      // (1 + ((k6 r2 + k5) r2 + k4) r2) / (1 + ((k3 r2 + k2) r2 + k1) r2)
      const double icdist = add_rn(1.0, mul_rn(add_rn(mul_rn(add_rn(mul_rn(k[7], r2), k[6]), r2), k[5]), r2)) /
                            add_rn(1.0, mul_rn(add_rn(mul_rn(add_rn(mul_rn(k[4], r2), k[1]), r2), k[0]), r2));
      if (icdist < 0) {
        x = x0;
        y = y0;
        break;
      }
      // dx = 2 p1 x y + p2 (r2 + 2 x x) + s1 r2 + s2 r2 r2,  dy = p1 (r2 + 2 y y) + 2 p2 x y + s3 r2 + s4 r2 r2
      const double dx = add_rn(add_rn(add_rn(mul_rn(mul_rn(2 * k[2], x), y), mul_rn(k[3], add_rn(r2, mul_rn(2 * x, x)))),
                                      mul_rn(k[8], r2)),
                               mul_rn(mul_rn(k[9], r2), r2));
      const double dy = add_rn(add_rn(add_rn(mul_rn(k[2], add_rn(r2, mul_rn(2 * y, y))), mul_rn(mul_rn(2 * k[3], x), y)),
                                      mul_rn(k[10], r2)),
                               mul_rn(mul_rn(k[11], r2), r2));
      x = mul_rn(sub_rn(x0, dx), icdist);
      y = mul_rn(sub_rn(y0, dy), icdist);
    }
  }
  if (to_pixels && !sentinel) {
    if (isfinite(x) && isfinite(y)) {
      const double px = add_rn(add_rn(mul_rn(c.fx, x), mul_rn(c.skew, y)), c.cx), py = add_rn(mul_rn(c.fy, y), c.cy);
      x = px;
      y = py;
    } else {
      x = y = __longlong_as_double(0x7ff8000000000000LL);
    }
  }
  reinterpret_cast<double2*>(xy_out)[i] = make_double2((double)(float)x, (double)(float)y);
}

// ---- grouping --------------------------------------------------------------------------------------------------
__global__ void tri_iota_kernel(int* __restrict__ v, long long n) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) v[i] = (int)i;
}

// counts rows whose camera index is outside [0, n_cams) or whose key is negative
__global__ void tri_validate_kernel(const int* __restrict__ cam, const long long* __restrict__ key, long long n,
                                    int n_cams, int* __restrict__ bad) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool b = cam[i] < 0 || cam[i] >= n_cams || (key && key[i] < 0);
  if (b) atomicAdd(bad, 1);
}

__global__ void tri_heads_kernel(const unsigned long long* __restrict__ k, long long n, int* __restrict__ head) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) head[i] = (i == 0 || k[i] != k[i - 1]) ? 1 : 0;
}

// gid = inclusive scan of head; start[gid-1] = i at heads; start[n_groups] = n
__global__ void tri_starts_kernel(const int* __restrict__ head, const int* __restrict__ gid, long long n,
                                  int* __restrict__ start) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (head[i]) start[gid[i] - 1] = (int)i;
  if (i == n - 1) start[gid[i]] = (int)n;
}

// ---- DLT ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long tri_mix(unsigned long long x, unsigned long long salt) {
  x += salt;
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ULL;
  x ^= x >> 27; x *= 0x94d049bb133111ebULL;
  x ^= x >> 31;
  return x;
}

// Eigenvector of the smallest eigenvalue of a symmetric 4x4 (cyclic Jacobi; quadratic convergence, <= 12 sweeps).
__device__ __forceinline__ void sym4_min_eigvec(double a[4][4], double out[4]) {
  double V[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) V[i][j] = (i == j) ? 1.0 : 0.0;
#pragma unroll 1
  for (int sweep = 0; sweep < 12; ++sweep) {
    double off = 0.0, dg = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      dg += a[i][i] * a[i][i];
#pragma unroll
      for (int j = i + 1; j < 4; ++j) off += a[i][j] * a[i][j];
    }
    if (off <= 1e-34 * dg) break;
#pragma unroll
    for (int p = 0; p < 3; ++p)
#pragma unroll
      for (int q = p + 1; q < 4; ++q) {
        const double apq = a[p][q];
        if (apq != 0.0) {
          const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
          const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
          const double c = rsqrt(t * t + 1.0), s = t * c;
#pragma unroll
          for (int k = 0; k < 4; ++k) {  // A <- A J
            const double akp = a[k][p], akq = a[k][q];
            a[k][p] = c * akp - s * akq;
            a[k][q] = s * akp + c * akq;
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {  // A <- J^T A
            const double apk = a[p][k], aqk = a[q][k];
            a[p][k] = c * apk - s * aqk;
            a[q][k] = s * apk + c * aqk;
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const double vkp = V[k][p], vkq = V[k][q];
            V[k][p] = c * vkp - s * vkq;
            V[k][q] = s * vkp + c * vkq;
          }
        }
      }
  }
  int m = 0;
  double best = a[0][0];
#pragma unroll
  for (int i = 1; i < 4; ++i)
    if (a[i][i] < best) {
      best = a[i][i];
      m = i;
    }
#pragma unroll
  for (int k = 0; k < 4; ++k) out[k] = (m == 0) ? V[k][0] : (m == 1) ? V[k][1] : (m == 2) ? V[k][2] : V[k][3];
}

// Adds the two DLT rows of the undistorted point xy under the 3x4 projection Pc (row-major) to the packed normal matrix
// m (00 01 02 03 11 12 13 22 23 33):  M += (x P2 - P0)(x P2 - P0)^T + (y P2 - P1)(y P2 - P1)^T.
__device__ __forceinline__ void dlt_accumulate(const double* Pc, double2 xy, double m[10]) {
  double a[4], bb[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double p2 = Pc[8 + k];
    a[k] = xy.x * p2 - Pc[k];
    bb[k] = xy.y * p2 - Pc[4 + k];
  }
  int t = 0;
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = p; q < 4; ++q) {
      m[t] = fma(a[p], a[q], fma(bb[p], bb[q], m[t]));
      ++t;
    }
}

// The DLT point X (3) of packed normal matrix m: its smallest eigenvector, de-homogenised
__device__ __forceinline__ void dlt_solve(const double m[10], double* X) {
  double A[4][4];
  int t = 0;
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = p; q < 4; ++q) {
      A[p][q] = m[t];
      A[q][p] = m[t];
      ++t;
    }
  double w[4];
  sym4_min_eigvec(A, w);
#pragma unroll
  for (int k = 0; k < 3; ++k) X[k] = w[k] / w[3];
}

constexpr int TRI_THREADS = 256;

// One group of observations (same (sync, object, keypoint) key) per TRI_LANES lanes (8 for the 2-6 views of a
// charuco corner, 32 when groups average more than 16 rows).  Each lane accumulates the normal matrix
// M = sum_rows (x P2 - P0)(x P2 - P0)^T + (y P2 - P1)(y P2 - P1)^T  of the DLT system over its rows, an
// xor-butterfly leaves the identical sum on all lanes, the smallest eigenvector is de-homogenised.
// `proj` is the [n_cams][3][4] table (shared-memory copy when it fits).
template <int TRI_LANES>
__global__ void __launch_bounds__(TRI_THREADS)
tri_dlt_kernel(const double* __restrict__ proj, int n_cams, int proj_in_smem, const int* __restrict__ start,
               const int* __restrict__ rows, const int* __restrict__ obs_cam, const double* __restrict__ obs_xy,
               int n_groups, double* __restrict__ xyz, int* __restrict__ count, int* __restrict__ rep_row,
               unsigned long long* __restrict__ sig) {
  extern __shared__ double s_proj[];
  // shared-memory copy with a stride of 13 doubles per camera: lanes read DIFFERENT cameras' rows, and a stride of 12 puts
  // the same entry of consecutive cameras into 4 of the 16 eight-byte banks (round 1: 4.1 M bank conflicts per launch)
  constexpr int PSTRIDE_SM = 13;
  if (proj_in_smem) {
    for (int i = threadIdx.x; i < n_cams * 12; i += blockDim.x) s_proj[(i / 12) * PSTRIDE_SM + i % 12] = proj[i];
    __syncthreads();
  }
  const double* P = proj_in_smem ? s_proj : proj;
  const int pstride = proj_in_smem ? PSTRIDE_SM : 12;
  const int lane = threadIdx.x & (TRI_LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / TRI_LANES;
  const bool live = g < n_groups;
  const int b = live ? start[g] : 0, e = live ? start[g + 1] : 0;
  double m[10];
#pragma unroll
  for (int k = 0; k < 10; ++k) m[k] = 0.0;
  unsigned long long h[2] = {0, 0};
  for (int i = b + lane; i < e; i += TRI_LANES) {
    const int r = rows[i];
    const int c = obs_cam[r];
    dlt_accumulate(P + (size_t)pstride * (size_t)c, reinterpret_cast<const double2*>(obs_xy)[r], m);
    h[0] += tri_mix((unsigned long long)(unsigned)c, 0x9e3779b97f4a7c15ULL);
    h[1] += tri_mix((unsigned long long)(unsigned)c, 0xd1b54a32d192ed03ULL);
  }
  group_sum<TRI_LANES>(m);
  group_sum<TRI_LANES>(h);
  if (!live || lane != 0) return;
  const int n = e - b;
  count[g] = n;
  rep_row[g] = rows[b];
  sig[2 * g] = h[0];
  sig[2 * g + 1] = h[1];
  if (n < 2) {
    xyz[3 * g] = xyz[3 * g + 1] = xyz[3 * g + 2] = __longlong_as_double(0x7ff8000000000000LL);
    return;
  }
  dlt_solve(m, xyz + 3 * g);
}

// ---- refinement to the reprojection optimum and point covariance (cb_triangulate_refine, DESIGN.md section 4.7) -------
// Group status codes, first match wins.
enum { TRI_OK = 0, TRI_FEW_ROWS = 1, TRI_NOT_PD = 2, TRI_MAX_ITER = 3, TRI_BEHIND = 4, TRI_NO_CONSENSUS = 5 };
constexpr double TRI_LAMBDA0 = 1e-3;  // initial Levenberg-Marquardt damping
constexpr double TRI_PD_RTOL = 1e-12;

// Cholesky factor (packed 00 10 20 11 21 22) of a symmetric 3x3 h (packed 00 01 02 11 12 22).  Returns false when a pivot
// is at or below rtol times the largest diagonal entry of h (or is not a number): the depth of a point seen along
// near-parallel rays is such a direction, although no single coordinate axis need be.
__device__ __forceinline__ bool chol3(const double* h, double rtol, double* L) {
  const double thr = rtol * fmax(h[0], fmax(h[3], h[5]));
  const double p0 = h[0];
  L[0] = sqrt(p0);
  L[1] = h[1] / L[0];
  L[2] = h[2] / L[0];
  const double p1 = h[3] - L[1] * L[1];
  L[3] = sqrt(p1);
  L[4] = (h[4] - L[2] * L[1]) / L[3];
  const double p2 = h[5] - L[2] * L[2] - L[4] * L[4];
  L[5] = sqrt(p2);
  return p0 > thr && p1 > thr && p2 > thr;
}

// (L L^T) d = -g
__device__ __forceinline__ void chol3_solve_neg(const double* L, const double* g, double* d) {
  const double y0 = -g[0] / L[0];
  const double y1 = (-g[1] - L[1] * y0) / L[3];
  const double y2 = (-g[2] - L[2] * y0 - L[4] * y1) / L[5];
  d[2] = y2 / L[5];
  d[1] = (y1 - L[4] * d[2]) / L[3];
  d[0] = (y0 - L[1] * d[1] - L[2] * d[2]) / L[0];
}

// camera-table staging shared by the two kernels below: an odd stride in shared memory (CT_SMEM, lanes of a warp read
// different cameras), the global table as it is otherwise
__device__ __forceinline__ const double* tri_stage_camtab(const double* __restrict__ camtab, int n_cams, int in_smem,
                                                          double* s_cam, int& stride) {
  if (in_smem) {
    for (int i = threadIdx.x; i < n_cams * CT_SIZE; i += blockDim.x) s_cam[(i / CT_SIZE) * CT_SMEM + i % CT_SIZE] = camtab[i];
    __syncthreads();
    stride = CT_SMEM;
    return s_cam;
  }
  stride = CT_SIZE;
  return camtab;
}

// Cost (squared pixels), J^T J and J^T r (pixels) of one group's rows at X, summed over the LANES lanes of the group: an
// xor butterfly leaves the identical sums on every lane.  Lanes with `on` false contribute zero but still shuffle.
template <int LANES>
__device__ __forceinline__ void tri_normal_eq(const double* cams, int stride, const int* __restrict__ rows,
                                              const int* __restrict__ obs_cam, const double* __restrict__ obs_px, int b,
                                              int e, int lane, bool on, const double* X, double (&acc)[10]) {
#pragma unroll
  for (int k = 0; k < 10; ++k) acc[k] = 0.0;
  if (on)
    for (int i = b + lane; i < e; i += LANES) {
      const int r = rows[i];
      const double* cam = cams + (size_t)stride * obs_cam[r];
      const double2 px = reinterpret_cast<const double2*>(obs_px)[r];
      double f[2], J[6];
      obs_res_jx(cam, X[0], X[1], X[2], px.x, px.y, 0, 1.0, f, J);
      const double fx0 = cam[CT_FX0];
      const double r0 = f[0] * fx0, r1 = f[1] * fx0;
#pragma unroll
      for (int k = 0; k < 6; ++k) J[k] *= fx0;
      acc[0] = fma(J[0], J[0], fma(J[3], J[3], acc[0]));
      acc[1] = fma(J[0], J[1], fma(J[3], J[4], acc[1]));
      acc[2] = fma(J[0], J[2], fma(J[3], J[5], acc[2]));
      acc[3] = fma(J[1], J[1], fma(J[4], J[4], acc[3]));
      acc[4] = fma(J[1], J[2], fma(J[4], J[5], acc[4]));
      acc[5] = fma(J[2], J[2], fma(J[5], J[5], acc[5]));
      acc[6] = fma(J[0], r0, fma(J[3], r1, acc[6]));
      acc[7] = fma(J[1], r0, fma(J[4], r1, acc[7]));
      acc[8] = fma(J[2], r0, fma(J[5], r1, acc[8]));
      acc[9] = fma(r0, r0, fma(r1, r1, acc[9]));
    }
  group_sum<LANES>(acc);
}

// Levenberg-Marquardt over the N parameters x of one group, from sums at x that the caller has formed and found positive
// definite (active: the group takes steps):  solve (H + lam diag H) d = -g;  accept when the cost drops (lam /= 10),
// else lam *= 10;  stop when |d| <= xtol (|x| + xtol) (st stays) or after max_iter steps (st = TRI_MAX_ITER).  Every lane
// of a group holds the same reduced sums, so every lane takes the same decision; the loop runs until no group of the
// warp is active, because the reductions need the whole warp.  The caller owns the sums, where they live and how the
// damped system is solved, through
//   step(lam, on, d)   d = the damped step at x when on (called on every lane);
//   trial(xt, on)      forms the sums at xt (every lane; the rows' terms only when on) and returns whether their cost
//                      is below x's;
//   keep()             the trial's sums become x's (the group's accepting lanes);
//   norm(v)            |v| of a parameter vector, in the caller's own arithmetic.
template <int N, typename Step, typename Trial, typename Keep, typename Norm>
__device__ __forceinline__ int lm_iterate(double* x, bool active, int st, int max_iter, double xtol, Step step,
                                          Trial trial, Keep keep, Norm norm) {
  double lam = TRI_LAMBDA0;
  int it = 0;
  while (__any_sync(0xffffffffu, active)) {
    if (active && it == max_iter) {
      st = TRI_MAX_ITER;
      active = false;
    }
    double d[N], xt[N];
#pragma unroll
    for (int k = 0; k < N; ++k) d[k] = 0.0;
    step(lam, active, d);
#pragma unroll
    for (int k = 0; k < N; ++k) xt[k] = x[k] + d[k];
    const bool lower = trial(xt, active);
    if (active) {
      ++it;
      const double dn = norm(d), xn = norm(x);
      if (lower) {
#pragma unroll
        for (int k = 0; k < N; ++k) x[k] = xt[k];
        keep();
        lam *= 0.1;
      } else {
        lam *= 10.0;
      }
      if (dn <= xtol * (xn + xtol)) active = false;
    }
  }
  return st;
}

// TRI_BEHIND when st is TRI_OK and depth(i) > 0 fails for a row position i in [b, e) of the group (on: a live group),
// else st; the same on every lane
template <int LANES, typename Depth>
__device__ __forceinline__ int status_behind(int st, bool on, int b, int e, int lane, Depth depth) {
  int behind = 0;
  if (on && st == TRI_OK)
    for (int i = b + lane; i < e; i += LANES) behind |= !(depth(i) > 0.0);
  behind = group_or<LANES>(behind);
  return st == TRI_OK && behind ? TRI_BEHIND : st;
}

// Per group, Levenberg-Marquardt (lm_iterate) on the pixel reprojection cost from the DLT point xyz0
// (oracle/triangulation_refine.py refine_points states the same rule), the sums in registers and the damped 3x3 system
// solved by chol3.  Writes xyz (the DLT point when H is not positive definite),
// the pixel RMSE and the status code.
template <int LANES>
__global__ void __launch_bounds__(TRI_THREADS)
tri_refine_kernel(const double* __restrict__ camtab, int n_cams, int cam_in_smem, const int* __restrict__ start,
                  const int* __restrict__ rows, const int* __restrict__ obs_cam, const double* __restrict__ obs_px,
                  int n_groups, const double* __restrict__ xyz0, int max_iter, double xtol, double* __restrict__ xyz,
                  double* __restrict__ rmse, int* __restrict__ status) {
  extern __shared__ double s_cam[];
  int stride;
  const double* cams = tri_stage_camtab(camtab, n_cams, cam_in_smem, s_cam, stride);
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  const bool live = g < n_groups;
  const int b = live ? start[g] : 0, e = live ? start[g + 1] : 0, n = e - b;
  double X[3] = {0.0, 0.0, 0.0};
  if (live)
#pragma unroll
    for (int k = 0; k < 3; ++k) X[k] = xyz0[3 * g + k];
  int st = n < 2 ? TRI_FEW_ROWS : TRI_OK;
  double acc[10], L[6];
  tri_normal_eq<LANES>(cams, stride, rows, obs_cam, obs_px, b, e, lane, live && st == TRI_OK, X, acc);
  const double cost0 = acc[9];
  if (st == TRI_OK && !chol3(acc, TRI_PD_RTOL, L)) st = TRI_NOT_PD;
  double tr[10];  // the sums at the trial point
  st = lm_iterate<3>(
      X, live && st == TRI_OK, st, max_iter, xtol,
      [&](double lam, bool on, double* d) {
        if (!on) return;
        double A[6] = {acc[0] * (1.0 + lam), acc[1], acc[2], acc[3] * (1.0 + lam), acc[4], acc[5] * (1.0 + lam)};
        chol3(A, 0.0, L);
        chol3_solve_neg(L, acc + 6, d);
      },
      [&](const double* xt, bool on) {
        tri_normal_eq<LANES>(cams, stride, rows, obs_cam, obs_px, b, e, lane, on, xt, tr);
        return tr[9] < acc[9];
      },
      [&] {
#pragma unroll
        for (int k = 0; k < 10; ++k) acc[k] = tr[k];
      },
      [](const double* v) { return sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); });
  if ((st == TRI_OK || st == TRI_MAX_ITER) && !chol3(acc, TRI_PD_RTOL, L)) st = TRI_NOT_PD;
  st = status_behind<LANES>(st, live, b, e, lane, [&](int i) {
    const double* cam = cams + (size_t)stride * obs_cam[rows[i]];
    return fma(cam[CT_R + 6], X[0], fma(cam[CT_R + 7], X[1], fma(cam[CT_R + 8], X[2], cam[CT_T + 2])));
  });
  if (!live || lane != 0) return;
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  const bool at_start = st == TRI_FEW_ROWS || st == TRI_NOT_PD;
#pragma unroll
  for (int k = 0; k < 3; ++k) xyz[3 * g + k] = at_start ? xyz0[3 * g + k] : X[k];
  rmse[g] = st == TRI_FEW_ROWS ? nan : sqrt((at_start ? cost0 : acc[9]) / n);
  status[g] = st;
}

// Per group at the refined point X (status 0, 3 or 4; NaN otherwise), the first-order covariance
//   Sigma_X = s2 H^-1 + H^-1 M H^-1,   M = sum_{c,d} B_c Sigma_cd B_d^T,   B_c = sum over the rows of camera c of J_X^T J_c
// (pixels).  Sig (n_cams*P square, uniform stride P, nullptr: no camera term) is read from L2.  The lanes of a group write
// each camera's B_c once (at the position of its first row in the group, scratch `Bs` / `first`), then gather the
// unordered camera pairs with cov_pair_gather, the gather of cov_point_kernel.
template <int P, int LANES>
__global__ void __launch_bounds__(TRI_THREADS)
tri_cov_kernel(const double* __restrict__ camtab, int n_cams, int cam_in_smem, const int* __restrict__ start,
               const int* __restrict__ rows, const int* __restrict__ obs_cam, const double* __restrict__ obs_px,
               int n_groups, const double* __restrict__ xyz, const int* __restrict__ status,
               const double* __restrict__ Sig, double s2, double* __restrict__ Bs, int* __restrict__ first,
               double* __restrict__ cov) {
  extern __shared__ double s_cam[];
  int stride;
  const double* cams = tri_stage_camtab(camtab, n_cams, cam_in_smem, s_cam, stride);
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  const bool live = g < n_groups;
  const int st = live ? status[g] : TRI_FEW_ROWS;
  const bool on = st == TRI_OK || st == TRI_MAX_ITER || st == TRI_BEHIND;
  const int b = on ? start[g] : 0, e = on ? start[g + 1] : 0, k = e - b;
  const int nP = n_cams * P;
  double X[3] = {0.0, 0.0, 0.0};
  if (on)
#pragma unroll
    for (int q = 0; q < 3; ++q) X[q] = xyz[3 * g + q];
  double h[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int i = b + lane; i < e; i += LANES) {
    const int c = obs_cam[rows[i]];
    bool is_first = true;
    if (Sig)
      for (int j = b; j < i && is_first; ++j) is_first = obs_cam[rows[j]] != c;
    double Bc[3][P];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int q = 0; q < P; ++q) Bc[a][q] = 0.0;
    // row i, then (first row of its camera only) the later rows of the same camera
    for (int j = i; j < e; ++j) {
      const int r = rows[j];
      if (j > i && (!Sig || !is_first)) break;
      if (obs_cam[r] != c) continue;
      const double* cam = cams + (size_t)stride * c;
      const double2 px = reinterpret_cast<const double2*>(obs_px)[r];
      double f[2], J[6], Jc[2 * P];
      obs_jac<P>(cam, X[0], X[1], X[2], px.x, px.y, 0, 1.0, f, J, Jc);
      const double fx0 = cam[CT_FX0];
#pragma unroll
      for (int q = 0; q < 6; ++q) J[q] *= fx0;
      if (j == i) {
        h[0] = fma(J[0], J[0], fma(J[3], J[3], h[0]));
        h[1] = fma(J[0], J[1], fma(J[3], J[4], h[1]));
        h[2] = fma(J[0], J[2], fma(J[3], J[5], h[2]));
        h[3] = fma(J[1], J[1], fma(J[4], J[4], h[3]));
        h[4] = fma(J[1], J[2], fma(J[4], J[5], h[4]));
        h[5] = fma(J[2], J[2], fma(J[5], J[5], h[5]));
      }
      if (Sig && is_first)
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
          for (int q = 0; q < P; ++q) Bc[a][q] = fma(J[a], Jc[q] * fx0, fma(J[3 + a], Jc[P + q] * fx0, Bc[a][q]));
    }
    if (Sig) {
      first[i] = is_first ? 1 : 0;
      if (is_first)
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
          for (int q = 0; q < P; ++q) Bs[(size_t)i * 3 * P + a * P + q] = Bc[a][q];
    }
  }
  double m[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
  if (Sig) {
    __syncwarp();
    for (int idx = lane; idx < k * k; idx += LANES) {
      const int pa = b + idx / k, pb = b + idx % k;
      if (pb < pa || !first[pa] || !first[pb]) continue;
      double x[3][3];
      cov_pair_gather<P>(Bs + (size_t)pa * 3 * P, Bs + (size_t)pb * 3 * P, P, Sig, nP, obs_cam[rows[pa]],
                         obs_cam[rows[pb]], x);
      const bool same = pa == pb;
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int c = 0; c < 3; ++c) m[a][c] += same ? x[a][c] : x[a][c] + x[c][a];
    }
  }
  group_sum<LANES>(h);
#pragma unroll
  for (int a = 0; a < 3; ++a) group_sum<LANES>(m[a]);
  if (!live || lane != 0) return;
  double* out = cov + 9 * (size_t)g;
  if (!on) {
    for (int q = 0; q < 9; ++q) out[q] = __longlong_as_double(0x7ff8000000000000LL);
    return;
  }
  // H^-1 = L^-T L^-1
  double L[6];
  chol3(h, 0.0, L);
  const double i0 = 1.0 / L[0], i3 = 1.0 / L[3], i5 = 1.0 / L[5];
  const double li[3][3] = {{i0, 0.0, 0.0},
                           {-L[1] * i0 * i3, i3, 0.0},
                           {(L[1] * L[4] * i3 - L[2]) * i0 * i5, -L[4] * i3 * i5, i5}};
  double Hi[3][3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int c = 0; c < 3; ++c) Hi[a][c] = li[0][a] * li[0][c] + li[1][a] * li[1][c] + li[2][a] * li[2][c];
  double t[3][3];  // M H^-1
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int c = 0; c < 3; ++c) t[a][c] = m[a][0] * Hi[0][c] + m[a][1] * Hi[1][c] + m[a][2] * Hi[2][c];
  double o[3][3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int c = 0; c < 3; ++c) o[a][c] = s2 * Hi[a][c] + Hi[a][0] * t[0][c] + Hi[a][1] * t[1][c] + Hi[a][2] * t[2][c];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int c = 0; c < 3; ++c) out[3 * a + c] = 0.5 * (o[a][c] + o[c][a]);
}

// ---- consensus over view pairs (cb_triangulate_robust, DESIGN.md section 4.8) ------------------------------------------
// Positions (i, j), i < j, of the m-th candidate pair of a group of k rows with T = k (k - 1) / 2 pairs: lexicographic rank
// m when T <= max_pairs, else floor(m T / max_pairs), computed exactly as m q + floor(m rem / max_pairs) with
// T = q max_pairs + rem (m rem < max_pairs^2 < 2^62).  rank(i, j) = i k - i (i + 1) / 2 + (j - i - 1).
__device__ __forceinline__ long long tri_pair_base(long long i, long long k) { return i * k - i * (i + 1) / 2; }

__device__ __forceinline__ void tri_candidate_pair(long long m, long long T, int max_pairs, int k, int& i, int& j) {
  long long r = m;
  if (T > max_pairs) r = m * (T / max_pairs) + (m * (T % max_pairs)) / max_pairs;
  const double kk = 2.0 * k - 1.0;
  long long a = (long long)(0.5 * (kk - sqrt(kk * kk - 8.0 * (double)r)));  // largest a with base(a) <= r, up to rounding
  a = max(0LL, min(a, (long long)k - 2));
  while (a > 0 && tri_pair_base(a, k) > r) --a;
  while (a < k - 2 && tri_pair_base(a + 1, k) <= r) ++a;
  i = (int)a;
  j = (int)(r - tri_pair_base(a, k) + a + 1);
}

// squared pixel error of one row at X and whether the row is in front of its camera
__device__ __forceinline__ double tri_row_err2(const double* cam, const double* X, double2 px, bool& front) {
  ProjOut o;
  project_obs<false>(cam, (((int)cam[CT_FLAGS]) & 2) != 0, X[0], X[1], X[2], o);
  front = o.Xc[2] > 0.0;
  const double du = o.u - px.x, dv = o.v - px.y;
  return du * du + dv * dv;
}

// a row's MSAC cost: its squared error within tau in front of the camera, else tau^2 (also for a non-finite error)
__device__ __forceinline__ double msac_term(bool front, double e2, double tau2) { return (front && e2 <= tau2) ? e2 : tau2; }

// Classification at the winner of a group's consensus (found: there is one).  Each lane flags its rows in front of the
// camera with e_r^2 <= tau^2 (err2(r, front): the squared pixel error of caller row r) into `pos_flag` (key-sorted
// position) and `inlier` (caller row); both are cleared when fewer than min_inliers rows agree.  Returns whether the
// group has consensus; nin is the count of agreeing rows, the same on every lane.
template <int LANES, typename RowErr2>
__device__ __forceinline__ bool consensus_classify(bool found, const int* __restrict__ rows, int b, int e, int lane,
                                                   double tau2, int min_inliers, RowErr2 err2,
                                                   unsigned char* __restrict__ pos_flag,
                                                   unsigned char* __restrict__ inlier, int& nin) {
  nin = 0;
  for (int i = b + lane; i < e; i += LANES) {
    const int r = rows[i];
    bool in = false;
    if (found) {
      bool front;
      const double e2 = err2(r, front);
      in = front && e2 <= tau2;
    }
    pos_flag[i] = in ? 1 : 0;
    inlier[r] = in ? 1 : 0;
    nin += in ? 1 : 0;
  }
  nin = group_sum<LANES>(nin);
  const bool ok = found && nin >= min_inliers;
  if (!ok && nin > 0)
    for (int i = b + lane; i < e; i += LANES) {
      pos_flag[i] = 0;
      inlier[rows[i]] = 0;
    }
  return ok;
}

// One group per LANES lanes (the lane choice of tri_dlt_kernel).  The lanes stride over the group's candidate pairs; each
// builds its pair's DLT point (tri_dlt_kernel's normal matrix on the undistorted float32-rounded coordinates `obs_xy`,
// then sym4_min_eigvec) and scores it by MSAC over all k rows, sum min(e_r^2, tau^2) in raw pixels (a row behind its camera
// or with a non-finite error costs tau^2).  A pair of rows from one camera, a non-finite point or one not in front of both
// of the pair's cameras is no hypothesis.  An xor butterfly over (score, candidate index) picks the lowest score, the
// lowest rank on a tie (rank grows with the index); the winner's point reaches the group's lanes by shuffle.  Each lane
// then classifies its rows (in front and e_r^2 <= tau^2) into `pos_flag` (key-sorted position) and `inlier` (caller row);
// both are cleared when the group has no hypothesis or fewer than min_inliers consensus rows (status 5).  Writes count,
// rep_row, n_inliers, status (0, 1 or 5) and xyz0 = the selected hypothesis (NaN for status 1 and 5).
// `camtab` and `proj` are staged in shared memory independently (camera table first) when their flags say so.
template <int LANES>
__global__ void __launch_bounds__(TRI_THREADS)
tri_consensus_kernel(const double* __restrict__ camtab, int cam_in_smem, const double* __restrict__ proj, int proj_in_smem,
                     int n_cams, const int* __restrict__ start, const int* __restrict__ rows,
                     const int* __restrict__ obs_cam, const double* __restrict__ obs_xy, const double* __restrict__ obs_px,
                     int n_groups, double tau, int min_inliers, int max_pairs, double* __restrict__ xyz0,
                     int* __restrict__ count, int* __restrict__ rep_row, int* __restrict__ n_inliers,
                     int* __restrict__ status, unsigned char* __restrict__ pos_flag, unsigned char* __restrict__ inlier) {
  extern __shared__ double s_cam[];
  int stride;
  const double* cams = tri_stage_camtab(camtab, n_cams, cam_in_smem, s_cam, stride);
  constexpr int PSTRIDE_SM = 13;  // odd stride, see tri_dlt_kernel
  double* s_proj = s_cam + (cam_in_smem ? (size_t)CT_SMEM * n_cams : 0);
  if (proj_in_smem) {
    for (int i = threadIdx.x; i < n_cams * 12; i += blockDim.x) s_proj[(i / 12) * PSTRIDE_SM + i % 12] = proj[i];
    __syncthreads();
  }
  const double* Pt = proj_in_smem ? s_proj : proj;
  const int pstride = proj_in_smem ? PSTRIDE_SM : 12;
  const int lane = threadIdx.x & (LANES - 1);
  const long long g = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / LANES;
  const bool live = g < n_groups;
  const int b = live ? start[g] : 0, e = live ? start[g + 1] : 0, k = e - b;
  const double tau2 = tau * tau;
  const double inf = __longlong_as_double(0x7ff0000000000000LL);
  const long long T = (long long)k * (k - 1) / 2;
  const long long nh = T < max_pairs ? T : (long long)max_pairs;
  double best = inf, X[3] = {0.0, 0.0, 0.0};
  long long best_m = 0x7fffffffffffffffLL;
  for (long long m = lane; m < nh; m += LANES) {
    int i, j;
    tri_candidate_pair(m, T, max_pairs, k, i, j);
    const int ri = rows[b + i], rj = rows[b + j];
    const int ci = obs_cam[ri], cj = obs_cam[rj];
    if (ci == cj) continue;
    double mm[10], h[3];
#pragma unroll
    for (int t = 0; t < 10; ++t) mm[t] = 0.0;
    dlt_accumulate(Pt + (size_t)pstride * (size_t)ci, reinterpret_cast<const double2*>(obs_xy)[ri], mm);
    dlt_accumulate(Pt + (size_t)pstride * (size_t)cj, reinterpret_cast<const double2*>(obs_xy)[rj], mm);
    dlt_solve(mm, h);
    if (!isfinite(h[0]) || !isfinite(h[1]) || !isfinite(h[2])) continue;
    const double* Ci = cams + (size_t)stride * ci;
    const double* Cj = cams + (size_t)stride * cj;
    const double zi = fma(Ci[CT_R + 6], h[0], fma(Ci[CT_R + 7], h[1], fma(Ci[CT_R + 8], h[2], Ci[CT_T + 2])));
    const double zj = fma(Cj[CT_R + 6], h[0], fma(Cj[CT_R + 7], h[1], fma(Cj[CT_R + 8], h[2], Cj[CT_T + 2])));
    if (!(zi > 0.0) || !(zj > 0.0)) continue;
    double score = 0.0;
    for (int p = b; p < e; ++p) {
      const int r = rows[p];
      bool front;
      const double e2 = tri_row_err2(cams + (size_t)stride * obs_cam[r], h, reinterpret_cast<const double2*>(obs_px)[r], front);
      score += msac_term(front, e2, tau2);
    }
    if (score < best) {  // candidates of a lane come in increasing rank: the first of equal scores stays
      best = score;
      best_m = m;
#pragma unroll
      for (int q = 0; q < 3; ++q) X[q] = h[q];
    }
  }
  group_argmin<LANES>(best, best_m);
  const bool found = best < inf;
  group_bcast<LANES>(X, found ? (int)(best_m % LANES) : 0);
  int nin;
  const bool ok = consensus_classify<LANES>(
      found, rows, b, e, lane, tau2, min_inliers,
      [&](int r, bool& front) {
        return tri_row_err2(cams + (size_t)stride * obs_cam[r], X, reinterpret_cast<const double2*>(obs_px)[r], front);
      },
      pos_flag, inlier, nin);
  if (!live || lane != 0) return;
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  count[g] = k;
  rep_row[g] = rows[b];
  n_inliers[g] = ok ? nin : 0;
  status[g] = k < 2 ? TRI_FEW_ROWS : ok ? TRI_OK : TRI_NO_CONSENSUS;
#pragma unroll
  for (int q = 0; q < 3; ++q) xyz0[3 * g + q] = ok ? X[q] : nan;
}

}  // namespace cb
