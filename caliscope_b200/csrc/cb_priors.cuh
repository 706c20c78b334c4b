// Gaussian priors on chosen cameras and points (DESIGN.md §4.13).  A prior adds
//   1/2 (x_c - m_c)^T L_c (x_c - m_c)   or   1/2 (X_j - m_j)^T L_j (X_j - m_j)
// to the objective, always quadratic whatever the loss: the rows W (x - m) with W^T W = L of the augmented least-squares
// problem.  Each term enters where its parameter's blocks are already formed:
//   camera priors   add_cam_priors, called by reduced_prep_body (HELD, after the (all-)reduce, before the fixed mask)
//                   and by prior_cam_kernel on the covariance path: L_c into the camera's diagonal block of S,
//                   L_c (x_c - m_c) into b and the g_c slot, diag L_c into the diag-U slot that feeds the scaling Dc2;
//   point priors    pt_pass_kernel (HELD): L_j into V_j, L_j (X_j - m_j) into g_j, before D, the damping and the
//                   factor (the covariance variant: before the pseudo-inverse);
//   prior cost      prior_cost_kernel, one partial per CTA into the extra cost slots trial_reduce_kernel sums.
#pragma once
#include "cb_kernels.cuh"

namespace cb {

constexpr int PRIOR_THREADS = 128;

// n camera priors by internal camera slot; width: the camera's parameter count (6 or 9, <= P); mean n x 9 and info n x 81
// (row-major 9 x 9) in the camera's own parameter order; xc: the camera buffers (stride P), current / trial.
struct CamPriors {
  const int* slot;
  const int* width;
  const double* mean;
  const double* info;
  int n;
  CPtr2 xc;
};

// n point priors: pt the point of each, mean n x 3, info n x 9 (row-major 3 x 3); idx[j]: the prior of point j or -1
// (read only by the HELD point-pass variants).
struct PointPriors {
  const int* idx;
  const int* pt;
  const double* mean;
  const double* info;
  int n;
};

// The camera priors at camera buffer xc, added into red = [S (nP x nP) | b | g_c | diag U | ...] by the calling CTA.  No
// two priors share a camera, so every entry is written by one thread; the caller synchronises before reading red.
template <int P>
__device__ __forceinline__ void add_cam_priors(double* __restrict__ red, int nP, const double* __restrict__ xc,
                                               const CamPriors& cp) {
  const size_t nn = (size_t)nP * nP;
  for (int t = threadIdx.x; t < cp.n * P * P; t += blockDim.x) {
    const int k = t / (P * P), a = (t / P) % P, b = t % P, w = cp.width[k], s = cp.slot[k];
    if (a < w && b < w) red[(size_t)(s * P + a) * nP + s * P + b] += cp.info[81 * (size_t)k + 9 * a + b];
  }
  for (int t = threadIdx.x; t < cp.n * P; t += blockDim.x) {
    const int k = t / P, a = t % P, w = cp.width[k], s = cp.slot[k];
    if (a >= w) continue;  // the padding slots of a 6-parameter camera under P = 9
    const double* L = cp.info + 81 * (size_t)k + 9 * a;
    const double* m = cp.mean + 9 * (size_t)k;
    const double* x = xc + (size_t)s * P;
    double g = 0.0;
#pragma unroll
    for (int b = 0; b < P; ++b)  // unrolled: the loads issue together instead of one dependent round trip per b
      if (b < w) g = fma(L[b], x[b] - m[b], g);
    const size_t i = (size_t)s * P + a;
    red[nn + i] += g;
    red[nn + nP + i] += g;
    red[nn + 2 * (size_t)nP + i] += L[a];
  }
}

// Covariance path: the camera priors into the undamped reduced system at buffer 0.  One CTA.
template <int P>
__global__ void __launch_bounds__(256) prior_cam_kernel(double* __restrict__ red, int nP, CamPriors cp) {
  add_cam_priors<P>(red, nP, cp.xc.p[0], cp);
}

// Prior cost at buffer cur ^ flip (st == nullptr: buffer 0): thread t takes camera prior t, or point prior t - cp.n; one
// partial per CTA into cost_part[blockIdx.x] (fixed grid and order: deterministic).
__global__ void __launch_bounds__(PRIOR_THREADS)
prior_cost_kernel(const LmState* __restrict__ st, int flip, int P, CamPriors cp, PointPriors pp, CPtr2 xp2,
                  double* __restrict__ cost_part) {
  __shared__ double sh[PRIOR_THREADS / 32];
  int sel = 0;
  if (st != nullptr) {
    if (st->done) return;
    sel = st->cur ^ flip;
  }
  const int t = blockIdx.x * PRIOR_THREADS + threadIdx.x;
  double q = 0.0;
  if (t < cp.n) {
    const int w = cp.width[t];
    const double* x = cp.xc.p[sel] + (size_t)cp.slot[t] * P;
    const double* m = cp.mean + 9 * (size_t)t;
    const double* L = cp.info + 81 * (size_t)t;
    double d[9];  // unrolled with constant indices: registers, and L is zero outside the camera's w x w block
#pragma unroll
    for (int a = 0; a < 9; ++a) d[a] = a < w ? x[a] - m[a] : 0.0;
#pragma unroll
    for (int a = 0; a < 9; ++a) {
      double r = 0.0;
#pragma unroll
      for (int b = 0; b < 9; ++b) r = fma(L[9 * a + b], d[b], r);
      q = fma(d[a], r, q);
    }
  } else if (t < cp.n + pp.n) {
    const int k = t - cp.n;
    const double* X = xp2.p[sel] + 4 * (size_t)pp.pt[k];
    const double* m = pp.mean + 3 * (size_t)k;
    const double* L = pp.info + 9 * (size_t)k;
    const double d[3] = {X[0] - m[0], X[1] - m[1], X[2] - m[2]};
#pragma unroll
    for (int a = 0; a < 3; ++a) q = fma(d[a], fma(L[3 * a], d[0], fma(L[3 * a + 1], d[1], L[3 * a + 2] * d[2])), q);
  }
  q = warp_sum(0.5 * q);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = q;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < PRIOR_THREADS / 32; ++w) s += sh[w];
    cost_part[blockIdx.x] = s;
  }
}

}  // namespace cb
