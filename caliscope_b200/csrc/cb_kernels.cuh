// CUDA kernels of the caliscope_b200 bundle-adjustment engine (sm_90a, fp64 throughout).
//
// Per LM linearisation (reference analogues in brackets, paths relative to /root/reference):
//   cam_prep_kernel     Rodrigues + SO(3) right Jacobian + intrinsics per camera
//                       [bundle_parameterization.py:166-186 trial_projection_inputs]
//   resjac_kernel       camera-major pass: residual + analytic 2x(P+3) Jacobian block per observation kept in
//                       registers, fused per-camera U = Jc^T Jc, g = Jc^T r and cost accumulation
//                       [src/caliscope/core/reprojection.py:75-119 and :128-234]
//   pt_pass_kernel      (cb_lm.cuh) point-major pass: V, g, 3x3 damped Cholesky, Z = (Jc^T Jp) L^-T -> k-major Zt
//   schur_syrk_kernel   Z Z^T (+ Z t) with bulk-async (TMA) staged shared-memory tiles, split-K
//   schur_finalize_kernel  S = U - Z Z^T, b = g_c - Z t into the all-reduce buffer
//   reduced_prep_kernel (cb_lm.cuh) Marquardt scaling (running max of diag U, scipy x_scale='jac' analogue,
//                       site-packages/scipy/optimize/_lsq/common.py:598-610), damping, block-Jacobi inverses
//   pcg_cluster_kernel  block-Jacobi PCG on the dense reduced system (small rigs: small_rig_step_kernel, cb_lm.cuh,
//                       runs damping, a direct LDL^T solve and the camera step in one CTA instead)
//   cam_step_kernel / pt_backsub_kernel (cb_lm.cuh)   step, bounds clamp, predicted reduction
#pragma once
#include <cooperative_groups.h>

#include "cb_device.cuh"

namespace cb {
namespace cg = cooperative_groups;

constexpr int RJ_THREADS = 128;   // resjac / cost block size
constexpr int RJ_CHUNK = 2048;    // observations per block (all of one camera)
constexpr int PT_WARPS = 8;       // warps (points) per block in the point-centric kernels
constexpr int SY_TILE = 96;       // Schur tile edge
constexpr int SY_KC = 32;         // k rows per pipeline stage
constexpr int SY_STAGES = 4;
constexpr int SY_CONSUMER_WARPS = 8;
constexpr int SY_THREADS = 32 * (SY_CONSUMER_WARPS + 1);  // + one producer warp
constexpr int PCG_THREADS = 512;

template <int P>
struct RowT {
  static constexpr int NU = P * (P + 1) / 2;
  static constexpr int NACC = NU + P + 1;                 // U packed, g, cost
};

// scalar slots (device double array `sc`)
enum {
  SC_COST = 0, SC_GNORM_C, SC_COST_NEW, SC_PRED_C, SC_STEP2_C, SC_X2_C, SC_PRED_P, SC_STEP2_P, SC_X2_P,
  SC_PCG_ITS, SC_PCG_REL, SC_PCG_FLAG, SC_GNORM_P, SC_PCG_T0 = 16, SC_COUNT = 24
};

// ---------------------------------------------------------------------------------------------
// x (BundleParameterization.pack layout, caller's camera order) <-> engine buffers.  Internal camera slot i holds the
// caller's camera whose block starts at cam_xoff[i] (the engine may reorder cameras so that cameras that see the same
// points share Schur tiles); its width is 9 with free intrinsics, else 6.
__global__ void unpack_x_kernel(const double* __restrict__ x, const int* __restrict__ cam_xoff,
                                const int* __restrict__ cam_flags, const double* __restrict__ cam_const,
                                int n_cams, int P, int n_pts, int ncp, double* __restrict__ xc, double* __restrict__ xp4) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_cams * P) {
    int c = i / P, p = i % P;
    int w = (cam_flags[c] & 1) ? 9 : 6;
    double v;
    if (p < w) v = x[cam_xoff[c] + p];
    else v = (p == 6) ? 1.0 : cam_const[c * 9 + 4 + (p - 7)];  // s = 1, k1_initial, k2_initial
    xc[i] = v;
  }
  if (i < n_pts) {
    xp4[4 * (size_t)i + 0] = x[ncp + 3 * (size_t)i + 0];
    xp4[4 * (size_t)i + 1] = x[ncp + 3 * (size_t)i + 1];
    xp4[4 * (size_t)i + 2] = x[ncp + 3 * (size_t)i + 2];
    xp4[4 * (size_t)i + 3] = 0.0;
  }
}

__global__ void pack_x_kernel(double* __restrict__ x, const int* __restrict__ cam_xoff, const int* __restrict__ cam_flags,
                              int n_cams, int P, int n_pts, int ncp, const double* __restrict__ xc,
                              const double* __restrict__ xp4) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_cams * P) {
    int c = i / P, p = i % P;
    if (p < ((cam_flags[c] & 1) ? 9 : 6)) x[cam_xoff[c] + p] = xc[i];
  }
  if (i < n_pts) {
    x[ncp + 3 * (size_t)i + 0] = xp4[4 * (size_t)i + 0];
    x[ncp + 3 * (size_t)i + 1] = xp4[4 * (size_t)i + 1];
    x[ncp + 3 * (size_t)i + 2] = xp4[4 * (size_t)i + 2];
  }
}

// ---------------------------------------------------------------------------------------------
// Levenberg-Marquardt state, resident in device memory for the whole solve (cb_lm.cuh holds the kernels that
// advance it).  Every per-trial kernel returns at once when `done` is set, picks its input buffers by `cur`
// and reads the damping from `lam`, so a trial is the same launch sequence every time (one CUDA graph).
// ---------------------------------------------------------------------------------------------
struct LmState {
  double lam, nu, cost, gnorm, initial_cost;
  double ftol, xtol, gtol;
  long long nfev, njev, nit, max_nfev, pcg_total;
  unsigned long long epoch_big, epoch_small;
  double fscale, pcg_tol2;  // robust-loss scale, squared PCG tolerance (read by the kernels, not baked into the launches)
  int cur, done, status, new_lin, err, bad_streak, n_log, log_cap;
  int loss, pcg_max_iter;
};
struct Ptr2 {
  double* p[2];
};
struct CPtr2 {
  const double* p[2];
};

// camera table entry: Rodrigues, SO(3) right Jacobian, intrinsics  [bundle_parameterization.py:166-186]
__device__ __forceinline__ void cam_prep_one(const double* __restrict__ q, const double* __restrict__ k, int flags,
                                             double* __restrict__ o) {
  const bool free_i = (flags & 1) != 0;
  const double r0 = q[0], r1 = q[1], r2 = q[2];
  const double th2 = r0 * r0 + r1 * r1 + r2 * r2, th = sqrt(th2);
  double R[9];
  double s = 0.0, co = 1.0;
  if (th >= 1e-12) sincos(th, &s, &co);
  if (th < 1e-12) {
    R[0] = 1; R[1] = -r2; R[2] = r1; R[3] = r2; R[4] = 1; R[5] = -r0; R[6] = -r1; R[7] = r0; R[8] = 1;
  } else {
    const double it = 1.0 / th, kx = r0 * it, ky = r1 * it, kz = r2 * it, c1 = 1.0 - co;
    R[0] = co + c1 * kx * kx;      R[1] = c1 * kx * ky - s * kz; R[2] = c1 * kx * kz + s * ky;
    R[3] = c1 * ky * kx + s * kz;  R[4] = co + c1 * ky * ky;     R[5] = c1 * ky * kz - s * kx;
    R[6] = c1 * kz * kx - s * ky;  R[7] = c1 * kz * ky + s * kx; R[8] = co + c1 * kz * kz;
  }
  double B, C;
  if (th < 1e-4) {
    B = 0.5 - th2 / 24.0 + th2 * th2 / 720.0;
    C = 1.0 / 6.0 - th2 / 120.0 + th2 * th2 / 5040.0;
  } else {
    B = (1.0 - co) / th2;
    C = (th - s) / (th2 * th);
  }
  // K = [r]x ; K^2 = r r^T - |r|^2 I ; Jr = I - B K + C K^2
  const double K2[9] = {r0 * r0 - th2, r0 * r1, r0 * r2, r1 * r0, r1 * r1 - th2, r1 * r2, r2 * r0, r2 * r1, r2 * r2 - th2};
  const double Km[9] = {0, -r2, r1, r2, 0, -r0, -r1, r0, 0};
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    o[CT_R + i] = R[i];
    o[CT_JR + i] = ((i % 4 == 0) ? 1.0 : 0.0) - B * Km[i] + C * K2[i];
  }
  o[CT_T + 0] = q[3]; o[CT_T + 1] = q[4]; o[CT_T + 2] = q[5];
  double sc = 1.0, k1 = k[4], k2 = k[5];
  if (free_i) { sc = q[6]; k1 = q[7]; k2 = q[8]; }
  const double fx = sc * k[0], fy = sc * k[1];
  o[CT_FX] = fx; o[CT_FY] = fy; o[CT_CX] = k[2]; o[CT_CY] = k[3];
  o[CT_D + 0] = k1; o[CT_D + 1] = k2; o[CT_D + 2] = k[6]; o[CT_D + 3] = k[7]; o[CT_D + 4] = k[8];
  o[CT_IFX0] = 1.0 / k[0];
  o[CT_SX] = fx / k[0];
  o[CT_SY] = fy / k[0];
  o[CT_FYR] = k[1] / k[0];
  o[CT_FLAGS] = (double)flags;
  o[35] = k[0];
}

__global__ void cam_prep_kernel(const double* __restrict__ xc, const int* __restrict__ cam_flags,
                                const double* __restrict__ cam_const, int n_cams, int P,
                                double* __restrict__ camtab) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cams) return;
  cam_prep_one(xc + (size_t)c * P, cam_const + (size_t)c * 9, cam_flags[c], camtab + (size_t)c * CT_SIZE);
}

// ---------------------------------------------------------------------------------------------
// Camera-major pass.  One block = one chunk of <= RJ_CHUNK observations of ONE camera: the camera table
// entry is block-uniform (shared memory broadcast) and the per-camera normal-equation blocks reduce in
// registers -> warp shuffles -> one partial per chunk.  No Jacobian row is written: the point-major pass
// (cb_lm.cuh pt_pass_kernel) recomputes the blocks it needs from the same 24 B / observation.
//
// MODE 0: linearisation: residual + Jacobian blocks in registers, accumulate U_c, g_c, cost.
// MODE 1: cost only.
// MODE 2: raw residuals to out2[orig*2]      (== joint_residuals order)
// MODE 3: pixel errors to out2[orig*2]       (== reprojection_errors)
// MODE 4: euclidean pixel error to out2[q]   (camera-major, for the percentile filter)
// With `st` the kernel is one step of the LM trial: it returns when st->done and evaluates at buffer
// (st->cur ^ flip) of camtab2 / xp2 (flip = 1: the trial point).
// ---------------------------------------------------------------------------------------------
template <int P, int MODE>
__global__ void __launch_bounds__(RJ_THREADS, (MODE == 0 && P == 6) ? 3 : 1)
resjac_kernel(const LmState* __restrict__ st, int flip, const int* __restrict__ chunk_cam,
              const int* __restrict__ chunk_begin, const int* __restrict__ chunk_end,
              const double2* __restrict__ cm_xy, const int* __restrict__ cm_pt, const int* __restrict__ cm_orig,
              CPtr2 camtab2, CPtr2 xp2, int loss, double fscale, double* __restrict__ partial,
              double* __restrict__ out2) {
  using RT = RowT<P>;
  __shared__ double cam[CT_SIZE];
  __shared__ double red[(MODE == 0 ? RT::NACC : 1) * (RJ_THREADS / 32)];
  int sel = 0;
  if (st != nullptr) {
    if (st->done) return;
    sel = st->cur ^ flip;
    loss = st->loss;
    fscale = st->fscale;
  }
  const double* __restrict__ camtab = camtab2.p[sel];
  const double* __restrict__ xp4 = xp2.p[sel];
  const int chunk = blockIdx.x;
  const int c = chunk_cam[chunk];
  const int begin = chunk_begin[chunk], end = chunk_end[chunk];
  if (threadIdx.x < CT_SIZE) cam[threadIdx.x] = camtab[(size_t)c * CT_SIZE + threadIdx.x];
  __syncthreads();
  const int flags = (int)cam[CT_FLAGS];
  const bool fish = (flags & 2) != 0;

  double acc[(MODE == 0) ? RT::NACC : 1];
#pragma unroll
  for (int k = 0; k < ((MODE == 0) ? RT::NACC : 1); ++k) acc[k] = 0.0;

  // Two-deep software pipeline over this thread's observations: the index pair of iteration i+2 and the
  // point gather of iteration i+1 are in flight while iteration i computes (the loads are a dependent
  // chain cm_pt -> xp4[pt], ~2 DRAM/L2 latencies, so the latency has to be hidden inside the thread).
  int q = begin + threadIdx.x;
  double2 xy_a = make_double2(0.0, 0.0), xy_b = xy_a;
  int pt_a = 0, org_a = 0, pt_b = 0, org_b = 0;
  double Xn0 = 0.0, Xn1 = 0.0, Xn2 = 0.0, Xn3 = 0.0;
  auto load_idx = [&](int qq, double2& xy, int& pt, int& org) {
    if (qq < end) {
      xy = cm_xy[qq];
      pt = cm_pt[qq];
      if constexpr (MODE == 2 || MODE == 3) org = cm_orig[qq];
    }
  };
  load_idx(q, xy_a, pt_a, org_a);
  load_idx(q + RJ_THREADS, xy_b, pt_b, org_b);
  if (q < end) ld256nc(xp4 + 4 * (size_t)pt_a, Xn0, Xn1, Xn2, Xn3);
  for (; q < end; q += RJ_THREADS) {
    const double2 xy = xy_a;
    const int org = org_a;
    const double X0 = Xn0, X1 = Xn1, X2 = Xn2;
    (void)org;
    // rotate the pipeline
    xy_a = xy_b; pt_a = pt_b; org_a = org_b;
    if (q + RJ_THREADS < end) ld256nc(xp4 + 4 * (size_t)pt_a, Xn0, Xn1, Xn2, Xn3);
    load_idx(q + 2 * RJ_THREADS, xy_b, pt_b, org_b);
    if constexpr (MODE == 0) {
      double f[2], JX[6], Jc[2 * P];
      acc[RT::NACC - 1] += obs_jac<P>(cam, X0, X1, X2, xy.x, xy.y, loss, fscale, f, JX, Jc);
      // U (packed upper), g
      int u = 0;
#pragma unroll
      for (int a = 0; a < P; ++a)
#pragma unroll
        for (int b = a; b < P; ++b) {
          acc[u] = fma(Jc[a], Jc[b], fma(Jc[P + a], Jc[P + b], acc[u]));
          ++u;
        }
#pragma unroll
      for (int a = 0; a < P; ++a) acc[RT::NU + a] = fma(Jc[a], f[0], fma(Jc[P + a], f[1], acc[RT::NU + a]));
    } else {
      ProjOut o;
      project_obs<false>(cam, fish, X0, X1, X2, o);
      const double ex = o.u - xy.x, ey = o.v - xy.y;
      if constexpr (MODE == 3) {
        const size_t i = (size_t)org;
        out2[2 * i] = ex; out2[2 * i + 1] = ey;
      } else if constexpr (MODE == 4) {
        // explicit round-to-nearest products and sums (no FMA contraction): the value is compared with thresholds
        // computed on the host with NumPy from the MODE 3 errors and must agree to the last bit
        out2[q] = sqrt(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)));
      } else {
        const double f0 = ex * cam[CT_IFX0], f1 = ey * cam[CT_IFX0];
        if constexpr (MODE == 2) {
          const size_t i = (size_t)org;
          out2[2 * i] = f0; out2[2 * i + 1] = f1;
        } else {
          acc[0] += robust_cost_only(loss, fscale, f0) + robust_cost_only(loss, fscale, f1);
        }
      }
    }
  }
  if constexpr (MODE == 0 || MODE == 1) {
    constexpr int NA = (MODE == 0) ? RT::NACC : 1;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < NA; ++k) {
      double v = warp_sum(acc[k]);
      if (lane == 0) red[wid * NA + k] = v;
    }
    __syncthreads();
    if (threadIdx.x < NA) {
      double v = 0.0;
#pragma unroll
      for (int w = 0; w < RJ_THREADS / 32; ++w) v += red[w * NA + threadIdx.x];
      partial[(size_t)chunk * NA + threadIdx.x] = v;
    }
  }
}

// deterministic single-block sum of n doubles -> out[0]
__global__ void sum_kernel(const double* __restrict__ in, int n, double* __restrict__ out) {
  __shared__ double sh[32];
  double v = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) v += in[i];
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.0;
    v = warp_sum(v);
    if (threadIdx.x == 0) out[0] = v;
  }
}

// Jacobian blocks in caller order for the test / diagnostic entry point cb_ba_jacobian_blocks:
// Jc (n_obs, 2, 9) with zeros beyond the camera's width, Jp (n_obs, 2, 3)   [== joint_jacobian's non-zeros]
template <int P>
__global__ void jac_blocks_kernel(const int* __restrict__ obs_cam, const int* __restrict__ cam_slot,
                                  const int* __restrict__ obs_pt,
                                  const double2* __restrict__ obs_xy, int n, const double* __restrict__ camtab,
                                  const double* __restrict__ xp4, double* __restrict__ Jc_out,
                                  double* __restrict__ Jp_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* X = xp4 + 4 * (size_t)obs_pt[i];
  const double2 xy = obs_xy[i];
  double f[2], JX[6], Jc[2 * P];
  obs_jac<P>(camtab + (size_t)cam_slot[obs_cam[i]] * CT_SIZE, X[0], X[1], X[2], xy.x, xy.y, 0, 1.0, f, JX, Jc);
  for (int k = 0; k < 6; ++k) Jp_out[(size_t)i * 6 + k] = JX[k];
  for (int r = 0; r < 2; ++r)
    for (int p = 0; p < 9; ++p) Jc_out[(size_t)i * 18 + r * 9 + p] = (p < P) ? Jc[r * P + p] : 0.0;
}

// 3x3 SPD: E = V + lam * D ; L = chol(E) ; returns Linv (lower, packed 00,10,11,20,21,22); zero if not PD
__device__ __forceinline__ void chol3_inv(const double* V6, const double* D2, double lam, double* Li) {
  const double d0 = D2[0] > 0.0 ? D2[0] : 1.0, d1 = D2[1] > 0.0 ? D2[1] : 1.0, d2 = D2[2] > 0.0 ? D2[2] : 1.0;
  const double e00 = V6[0] + lam * d0, e01 = V6[1], e02 = V6[2], e11 = V6[3] + lam * d1, e12 = V6[4],
               e22 = V6[5] + lam * d2;
  // reciprocal square roots instead of sqrt + divide (fp64 div/sqrt expand to long instruction sequences)
  bool ok = e00 > 0.0;
  const double i00 = rsqrt(ok ? e00 : 1.0);
  const double l10 = e01 * i00, l20 = e02 * i00;
  const double t11 = e11 - l10 * l10;
  ok = ok && t11 > 0.0;
  const double i11 = rsqrt(ok ? t11 : 1.0);
  const double l21 = (e12 - l20 * l10) * i11;
  const double t22 = e22 - l20 * l20 - l21 * l21;
  ok = ok && t22 > 0.0;
  const double i22 = rsqrt(ok ? t22 : 1.0);
  const double i10 = -l10 * i00 * i11;
  const double i21 = -l21 * i11 * i22;
  const double i20 = -(l20 * i00 + l21 * i10) * i22;
  if (ok) {
    Li[0] = i00; Li[1] = i10; Li[2] = i11; Li[3] = i20; Li[4] = i21; Li[5] = i22;
  } else {
    Li[0] = Li[1] = Li[2] = Li[3] = Li[4] = Li[5] = 0.0;
  }
}

// ---------------------------------------------------------------------------------------------
// Schur product  part[split][tile] = A_I^T A_J  over a slab of k rows (k = 3*point + axis), where
// Zt is k-major: Zt[k][col], col = camera*P + p.  Tiles are staged through shared memory with
// 1-D bulk async copies (TMA engine, mbarrier completion), SY_STAGES deep; each thread owns a
// 6x6 register tile.  Diagonal tiles also accumulate Z t (the reduced right-hand side).
// ---------------------------------------------------------------------------------------------
constexpr int SY_LDS = SY_TILE + 4;  // padded smem row stride (doubles): conflict-free DMMA fragment loads

struct SyrkSmem {
  double A[SY_STAGES][SY_KC * SY_LDS];
  double B[SY_STAGES][SY_KC * SY_LDS];
  double t[SY_STAGES][SY_KC];
  unsigned long long full[SY_STAGES];
  unsigned long long empty[SY_STAGES];
};

// D(8x8) += A(8x4) * B(4x8), fp64 tensor path (SASS: DMMA.8x8x4)
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// D(16x8) += A(16x16) * B(16x8), fp64 tensor path (SASS: DMMA.16x8x16).  Fragments (PTX m16n8k16.f64), g = lane>>2,
// t = lane&3:  a[i] = A[g + 8*(i&1)][t + 4*(i>>1)],  b[j] = B[t + 4*j][g],
//              c = {D[g][2t], D[g][2t+1], D[g+8][2t], D[g+8][2t+1]}
__device__ __forceinline__ void dmma16816(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
      "{%0,%1,%2,%3};"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// One CTA of the Schur product: either an off-diagonal 96x96 tile (I < J) or a PAIR of diagonal tiles
// (I, I) and (I2, I2) whose upper triangles together are one tile's worth of work, over k chunks [c0, c1).
struct SyItem {
  int kind;    // 0: off-diagonal tile, 1: diagonal pair (I2 < 0: single diagonal tile)
  int I, J;    // kind 0: tile (I, J); kind 1: tiles (I, I) and (J, J) with J = I2
  int c0, c1;  // k-chunk range (chunks of SY_KC rows; of the item's k-list when koff >= 0, of 0..K_pad otherwise)
  int slotA, slotB;  // partial-output slots (kind 0 uses slotA only)
  int koff;    // >= 0: offset of this item's compacted row list in `klist` (only the rows k = 3*point + axis of points
               // seen by cameras of BOTH column tiles; padded with the index of an all-zero row); -1: all rows
};

// Diagonal blocks (24 x 24, not a multiple of 16 rows) stay on m8n8k4.
// Fragment ownership (PTX m8n8k4.f64): A[row = lane>>2][k = lane&3], B[k = lane&3][col = lane>>2],
// C[row = lane>>2][col = 2*(lane&3) + {0,1}];  A[i][k] = Zt[k][I*96 + i], B[k][j] = Zt[k][J*96 + j].
//
// kind 0: 8 consumer warps as 2 (row groups of 48) x 4 (column groups of 24): 3 x 3 m16n8k16 tiles per warp
//         (A[i][k] sits in shared memory at As[k*SY_LDS + i], B[k][j] likewise).
// kind 1: only the 10 upper-triangular 24x24 blocks of each diagonal tile are formed; the 20 blocks of the
//         pair are dealt 3/3/3/3/2/2/2/2 to warps 0..7 so every SM sub-partition (warps w and w+4) carries 5.
__constant__ signed char SY_DIAG_BLOCKS[8][3][3] = {
    // {tile select, block row, block col}; select -1 = no block
    {{0, 0, 0}, {0, 0, 1}, {0, 0, 2}}, {{0, 0, 3}, {0, 1, 3}, {0, 2, 3}}, {{0, 1, 1}, {0, 1, 2}, {0, 2, 2}},
    {{0, 3, 3}, {1, 3, 3}, {1, 2, 2}}, {{1, 0, 0}, {1, 0, 1}, {-1, 0, 0}}, {{1, 0, 2}, {1, 0, 3}, {-1, 0, 0}},
    {{1, 1, 1}, {1, 1, 2}, {-1, 0, 0}}, {{1, 1, 3}, {1, 2, 3}, {-1, 0, 0}}};

__global__ void __launch_bounds__(SY_THREADS, 1)
schur_syrk_kernel(const LmState* __restrict__ st, const double* __restrict__ Zt, size_t LD,
                  const double* __restrict__ tvec, const SyItem* __restrict__ items, const int* __restrict__ klist,
                  double* __restrict__ part, double* __restrict__ tpart) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  SyrkSmem& sm = *reinterpret_cast<SyrkSmem*>(smem_raw);
  if (st->done) return;
  const SyItem item = items[blockIdx.x];
  const bool diag = item.kind == 1;
  const bool two = diag ? (item.J >= 0) : true;  // second smem tile in use
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int fr = lane >> 2, fk = lane & 3;

  if (tid == 0) {
    for (int s = 0; s < SY_STAGES; ++s) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], SY_CONSUMER_WARPS);
    }
    mbar_fence_init();
  }
  __syncthreads();

  const uint32_t row_bytes = SY_TILE * 8;
  const uint32_t stage_bytes = SY_KC * row_bytes * (two ? 2u : 1u);
  const int n_it = item.c1 - item.c0;

  if (wid == SY_CONSUMER_WARPS) {
    // ---- producer warp: runs ahead, one k row per lane per tile, stage recycled on `empty` ----
    for (int it = 0; it < n_it; ++it) {
      const int stage = it % SY_STAGES, round = it / SY_STAGES;
      if (round > 0) mbar_wait(&sm.empty[stage], (uint32_t)((round - 1) & 1));
      // row of this lane: straight through k, or through the item's compacted list (rows of points that both
      // column tiles see; everything else would multiply structural zeros)
      const size_t k = item.koff >= 0 ? (size_t)klist[(size_t)item.koff + (size_t)(item.c0 + it) * SY_KC + lane]
                                      : (size_t)(item.c0 + it) * SY_KC + lane;
      // t rides along as a plain shared-memory store: ordered before lane 0's arrive (release) by the warp barrier,
      // visible to the consumers after their acquire on `full`
      if (diag) sm.t[stage][lane] = tvec[k];
      __syncwarp();
      if (lane == 0) mbar_expect_tx(&sm.full[stage], stage_bytes);
      __syncwarp();
      bulk_g2s(&sm.A[stage][lane * SY_LDS], Zt + k * LD + (size_t)item.I * SY_TILE, row_bytes, &sm.full[stage]);
      if (two)
        bulk_g2s(&sm.B[stage][lane * SY_LDS], Zt + k * LD + (size_t)item.J * SY_TILE, row_bytes, &sm.full[stage]);
    }
    return;
  }

  if (!diag) {
    // ---------------- off-diagonal tile ----------------
    const int wr = wid >> 2, wc = wid & 3;
    double acc[3][3][4];
#pragma unroll
    for (int u = 0; u < 3; ++u)
#pragma unroll
      for (int v = 0; v < 3; ++v)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[u][v][e] = 0.0;
    for (int it = 0; it < n_it; ++it) {
      const int stage = it % SY_STAGES;
      mbar_wait(&sm.full[stage], (uint32_t)((it / SY_STAGES) & 1));
      const double* As = sm.A[stage] + fk * SY_LDS + wr * 48 + fr;
      const double* Bs = sm.B[stage] + fk * SY_LDS + wc * 24 + fr;
#pragma unroll
      for (int ks = 0; ks < SY_KC / 16; ++ks) {
        double a[3][8], b[3][4];
#pragma unroll
        for (int u = 0; u < 3; ++u)
#pragma unroll
          for (int i = 0; i < 8; ++i) a[u][i] = As[(ks * 16 + 4 * (i >> 1)) * SY_LDS + u * 16 + 8 * (i & 1)];
#pragma unroll
        for (int v = 0; v < 3; ++v)
#pragma unroll
          for (int j = 0; j < 4; ++j) b[v][j] = Bs[(ks * 16 + 4 * j) * SY_LDS + v * 8];
#pragma unroll
        for (int u = 0; u < 3; ++u)
#pragma unroll
          for (int v = 0; v < 3; ++v) dmma16816(acc[u][v], a[u], b[v]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.empty[stage]);
    }
    double* out = part + (size_t)item.slotA * (SY_TILE * SY_TILE);
#pragma unroll
    for (int u = 0; u < 3; ++u)
#pragma unroll
      for (int v = 0; v < 3; ++v)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = wr * 48 + u * 16 + 8 * h + fr, cc = wc * 24 + v * 8 + 2 * fk;
          *reinterpret_cast<double2*>(out + r * SY_TILE + cc) = make_double2(acc[u][v][2 * h], acc[u][v][2 * h + 1]);
        }
    return;
  }

  // ---------------- diagonal pair ----------------
  int bsel[3], brow[3], bcol[3];
  const int wmap = wid;
#pragma unroll
  for (int b = 0; b < 3; ++b) {
    bsel[b] = SY_DIAG_BLOCKS[wmap][b][0];
    brow[b] = SY_DIAG_BLOCKS[wmap][b][1];
    bcol[b] = SY_DIAG_BLOCKS[wmap][b][2];
    if (bsel[b] == 1 && !two) bsel[b] = -1;
  }
  double acc[3][3][3][2];
#pragma unroll
  for (int b = 0; b < 3; ++b)
#pragma unroll
    for (int u = 0; u < 3; ++u)
#pragma unroll
      for (int v = 0; v < 3; ++v) acc[b][u][v][0] = acc[b][u][v][1] = 0.0;
  double tacc = 0.0;
  const int trow = tid % SY_TILE, tsel = tid / SY_TILE;  // threads 0..191: one row of Z t each
  const bool tact = tid < 2 * SY_TILE && (tsel == 0 || two);
  for (int it = 0; it < n_it; ++it) {
    const int stage = it % SY_STAGES;
    mbar_wait(&sm.full[stage], (uint32_t)((it / SY_STAGES) & 1));
#pragma unroll
    for (int ks = 0; ks < SY_KC / 4; ++ks) {
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        if (bsel[b] < 0) continue;  // warp-uniform
        const double* T = (bsel[b] == 0 ? sm.A[stage] : sm.B[stage]) + (ks * 4 + fk) * SY_LDS + fr;
        double a[3], bb[3];
#pragma unroll
        for (int u = 0; u < 3; ++u) a[u] = T[brow[b] * 24 + u * 8];
#pragma unroll
        for (int v = 0; v < 3; ++v) bb[v] = T[bcol[b] * 24 + v * 8];
#pragma unroll
        for (int u = 0; u < 3; ++u)
#pragma unroll
          for (int v = 0; v < 3; ++v) dmma884(acc[b][u][v][0], acc[b][u][v][1], a[u], bb[v]);
      }
    }
    if (tact) {
      const double* Ad = (tsel == 0 ? sm.A[stage] : sm.B[stage]);
#pragma unroll 8
      for (int k = 0; k < SY_KC; ++k) tacc = fma(Ad[k * SY_LDS + trow], sm.t[stage][k], tacc);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.empty[stage]);
  }
#pragma unroll
  for (int b = 0; b < 3; ++b) {
    if (bsel[b] < 0) continue;
    double* out = part + (size_t)(bsel[b] == 0 ? item.slotA : item.slotB) * (SY_TILE * SY_TILE);
#pragma unroll
    for (int u = 0; u < 3; ++u)
#pragma unroll
      for (int v = 0; v < 3; ++v) {
        const int r = brow[b] * 24 + u * 8 + fr, cc = bcol[b] * 24 + v * 8 + 2 * fk;
        *reinterpret_cast<double2*>(out + r * SY_TILE + cc) = make_double2(acc[b][u][v][0], acc[b][u][v][1]);
      }
  }
  if (tact) tpart[(size_t)(tsel == 0 ? item.slotA : item.slotB) * SY_TILE + trow] = tacc;
}

// red = [ S (nP*nP) | b (nP) | gc (nP) | diagU (nP) | cost | gpmax slots ... ]   (local partials)
// one output element of S = U - Z Z^T, b = g_c - Z t (+ g_c, diag U, cost) from the split-K partial tiles;
// diagonal tiles hold only their upper-triangular 24x24 blocks
template <int P>
__device__ __forceinline__ void finalize_elem(size_t idx, int nP, int n_blk, const int* __restrict__ tile_of,
                                              const int* __restrict__ tile_slot_start,
                                              const int* __restrict__ tile_slots, const double* __restrict__ part,
                                              const double* __restrict__ tpart, const double* __restrict__ Upk,
                                              const double* __restrict__ gc, const double* __restrict__ cam_cost_sum,
                                              double* __restrict__ red) {
  using RT = RowT<P>;
  const size_t nn = (size_t)nP * nP;
  if (idx < nn) {
    const int i = (int)(idx / nP), j = (int)(idx % nP);
    int I = i / SY_TILE, J = j / SY_TILE, li = i % SY_TILE, lj = j % SY_TILE;
    if (I > J) { int t = I; I = J; J = t; t = li; li = lj; lj = t; }
    if (I == J && li / 24 > lj / 24) { int t = li; li = lj; lj = t; }
    const int tile = tile_of[I * n_blk + J];
    double s = 0.0;
    const int q1 = tile_slot_start[tile + 1];
#pragma unroll 8
    for (int q = tile_slot_start[tile]; q < q1; ++q)  // fixed slot order: the sum is reproducible run to run
      s += part[(size_t)tile_slots[q] * (SY_TILE * SY_TILE) + li * SY_TILE + lj];
    double u = 0.0;
    const int ci = i / P, cj = j / P;
    if (ci == cj) {
      int a = i % P, b = j % P;
      if (a > b) { int t = a; a = b; b = t; }
      u = Upk[(size_t)ci * RT::NU + (a * P - a * (a - 1) / 2 + (b - a))];
    }
    red[idx] = u - s;
  } else if (idx < nn + (size_t)nP) {
    const int i = (int)(idx - nn);
    const int I = i / SY_TILE, li = i % SY_TILE;
    const int tile = tile_of[I * n_blk + I];
    double s = 0.0;
    const int q1 = tile_slot_start[tile + 1];
#pragma unroll 8
    for (int q = tile_slot_start[tile]; q < q1; ++q)
      s += tpart[(size_t)tile_slots[q] * SY_TILE + li];
    red[nn + i] = gc[i] - s;
    red[nn + nP + i] = gc[i];
    const int c = i / P, a = i % P;
    red[nn + 2 * (size_t)nP + i] = Upk[(size_t)c * RT::NU + (a * P - a * (a - 1) / 2)];
  } else if (idx == nn + (size_t)nP) {
    red[nn + 3 * (size_t)nP] = cam_cost_sum[0];
  }
}

// single-rank / NCCL / callback transports: this rank's partial reduced system into `red`, the point-gradient
// inf-norm into this rank's slot (so that a SUM all-reduce carries the max)
template <int P>
__global__ void schur_finalize_kernel(const LmState* __restrict__ st, int nP, int n_blk,
                                      const int* __restrict__ tile_of, const int* __restrict__ tile_slot_start,
                                      const int* __restrict__ tile_slots, const double* __restrict__ part,
                                      const double* __restrict__ tpart, CPtr2 Upk2, CPtr2 gc2, CPtr2 costsum2,
                                      const double* __restrict__ gmax, int red_slots, int rank_slot,
                                      double* __restrict__ red) {
  if (st->done) return;
  const int cur = st->cur;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  finalize_elem<P>(idx, nP, n_blk, tile_of, tile_slot_start, tile_slots, part, tpart, Upk2.p[cur], gc2.p[cur],
                   costsum2.p[cur], red);
  const size_t slot0 = (size_t)nP * nP + 3 * (size_t)nP + 1;
  if (idx < (size_t)red_slots) red[slot0 + idx] = ((int)idx == rank_slot) ? gmax[0] : 0.0;
}

// ---------------------------------------------------------------------------------------------
// PCG on the dense reduced camera system S x = -b, one thread-block cluster.  Each CTA owns a slab
// of rows of S, computes its slice of w = S u and writes
// it into every CTA's w buffer through distributed shared memory; all vector updates and dot
// products are replicated in every CTA, so the only cluster-wide exchange is that slice.
// Chronopoulos-Gear single-reduction recurrence: one fused (r.u, w.u) reduction and one cluster
// barrier per iteration:
//   u = M^-1 r, w = S u, g = r.u, d = w.u, beta = g/g_old, alpha = g / (d - beta g / alpha_old)
//   p = u + beta p, q = w + beta q (= S p), x += alpha p, r -= alpha q
// ---------------------------------------------------------------------------------------------
// MODE 1: slab streamed from global/L2 (any size), 2: slab in REGISTERS (3 rows x CL columns-per-lane
// per warp; n_camera_params <= 32*CL, rows_per <= 48) -- the matvec then touches shared memory only for
// the vector u.
//
// Per iteration: [A] replicated vector update + block-Jacobi solve (each thread recomputes the P residual
// entries of its camera block, so no barrier is needed between the two), __syncthreads, [B] slab matvec,
// rows of w and this warp's share of d = w.u written into every CTA through DSMEM, cluster barrier,
// [C] every warp sums the d slots (and the CTA-local g = r.u slots): one block barrier and one cluster
// barrier per iteration, all loop buffers double-buffered by iteration parity.
template <int MODE, int P, int CL>
__global__ void __launch_bounds__(PCG_THREADS, 1)
pcg_cluster_kernel(const LmState* __restrict__ st, const double* __restrict__ S, const double* __restrict__ bvec,
                   const double* __restrict__ Minv, int nP, int nPa, int rows_per, double tol2, int max_iter,
                   double* __restrict__ xout, double* __restrict__ sc) {
  if (st != nullptr) {
    if (st->done) return;  // uniform over the cluster, before any cluster operation
    tol2 = st->pcg_tol2;
    max_iter = st->pcg_max_iter;
  }
  constexpr int NW = PCG_THREADS / 32;
  constexpr int MAXC = 16;  // largest cluster
  extern __shared__ __align__(16) double psm[];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank(), csize = (int)cluster.num_blocks();
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  // layout: x u p | r[2] q[2] w[2] (nPa each) | gslot[2][NW] | dslot[2][MAXC*NW] | Minv
  double* vx = psm;
  double* vu = vx + nPa;
  double* vp = vu + nPa;
  double* vr = vp + nPa;      // two buffers
  double* vq = vr + 2 * nPa;  // two buffers
  double* vw = vq + 2 * nPa;  // two buffers
  double* gslot = vw + 2 * nPa;
  double* dslot = gslot + 2 * NW;
  double* Mi = dslot + 2 * MAXC * NW;
  const int row0 = rank * rows_per;
  const int nrows = max(0, min(rows_per, nP - row0));
  const int n_cams = nP / P;

  for (int i = tid; i < n_cams * P * P; i += PCG_THREADS) Mi[i] = Minv[i];
  double sreg[MODE == 2 ? 3 : 1][MODE == 2 ? CL : 1];
  if constexpr (MODE == 2) {
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < CL; ++c) {
        const int row = wid * 3 + r, col = lane + 32 * c;
        sreg[r][c] = (row < nrows && col < nP) ? S[(size_t)(row0 + row) * nP + col] : 0.0;
      }
  }
  for (int i = tid; i < nPa; i += PCG_THREADS) {
    vx[i] = 0.0; vp[i] = 0.0; vu[i] = 0.0;
    vq[i] = 0.0; vq[nPa + i] = 0.0;
    vr[i] = (i < nP) ? -bvec[i] : 0.0;  // buffer 0 = r_0
    vr[nPa + i] = 0.0;
  }
  for (int i = tid; i < 2 * MAXC * NW; i += PCG_THREADS) dslot[i] = 0.0;
  __syncthreads();

  // [A] for iteration `it` (it = 0: only u = M^-1 r and g = r.u):  reads r/q buffer (it+1)&1 ... see below
  auto phase_a = [&](int it, double alpha, double beta) {
    // buffers: current r, q live in parity `it & 1`; the updated ones go to parity `(it + 1) & 1`
    const double* rc = vr + (it & 1) * nPa;
    double* rn = vr + ((it + 1) & 1) * nPa;
    const double* qc = vq + (it & 1) * nPa;
    double* qn = vq + ((it + 1) & 1) * nPa;
    const double* wc = vw + (it & 1) * nPa;
    double pg = 0.0;
    for (int i = tid; i < nP; i += PCG_THREADS) {
      const int c = i / P, a = i - c * P;
      const double* m = Mi + (size_t)c * P * P + a * P;
      double s = 0.0, r_own = 0.0;
      if (it == 0) {
#pragma unroll
        for (int b = 0; b < P; ++b) {
          const double rb = rc[c * P + b];
          s = fma(m[b], rb, s);
          if (b == a) r_own = rb;
        }
        rn[i] = r_own;
        qn[i] = 0.0;
      } else {
        const double ui = vu[i];
        const double pi = fma(beta, vp[i], ui);
        vp[i] = pi;
        vx[i] = fma(alpha, pi, vx[i]);
#pragma unroll
        for (int b = 0; b < P; ++b) {
          const int k = c * P + b;
          const double qb = fma(beta, qc[k], wc[k]);   // q_new of the neighbour, recomputed
          const double rb = fma(-alpha, qb, rc[k]);    // r_new of the neighbour, recomputed
          s = fma(m[b], rb, s);
          if (b == a) { r_own = rb; qn[i] = qb; }
        }
        rn[i] = r_own;
      }
      vu[i] = s;  // only its owner reads vu[i] in this phase
      pg = fma(r_own, s, pg);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) pg += __shfl_xor_sync(0xffffffffu, pg, o);
    if (lane == 0) gslot[(it & 1) * NW + wid] = pg;
  };

  // [B] w[row0 + r] = S_row . u for this CTA's rows and this warp's share of d = w.u -> every CTA
  auto phase_b = [&](int it) {
    double* wbuf = vw + ((it + 1) & 1) * nPa;
    double* dbuf = dslot + ((it + 1) & 1) * (MAXC * NW);
    double dpart = 0.0;
    for (int r0 = wid * 3; r0 < nrows; r0 += NW * 3) {
      const bool h1 = r0 + 1 < nrows, h2 = r0 + 2 < nrows;
      double s0, s1, s2;
      if constexpr (MODE == 2) {
        double e0 = 0, e1 = 0, e2 = 0, o0 = 0, o1 = 0, o2 = 0;
#pragma unroll
        for (int c = 0; c < CL; ++c) {
          const double uk = vu[lane + 32 * c];
          if (c & 1) { o0 = fma(sreg[0][c], uk, o0); o1 = fma(sreg[1][c], uk, o1); o2 = fma(sreg[2][c], uk, o2); }
          else { e0 = fma(sreg[0][c], uk, e0); e1 = fma(sreg[1][c], uk, e1); e2 = fma(sreg[2][c], uk, e2); }
        }
        s0 = e0 + o0; s1 = e1 + o1; s2 = e2 + o2;
      } else {
        const double* a0 = S + (size_t)(row0 + r0) * nP;
        const double* a1 = a0 + (h1 ? nP : 0);
        const double* a2 = a0 + (h2 ? 2 * nP : 0);
        double t0[4] = {0, 0, 0, 0}, t1[4] = {0, 0, 0, 0}, t2[4] = {0, 0, 0, 0};
        int k = lane;
        for (; k + 96 < nP; k += 128) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const double uk = vu[k + 32 * j];
            t0[j] = fma(__ldg(a0 + k + 32 * j), uk, t0[j]);
            t1[j] = fma(__ldg(a1 + k + 32 * j), uk, t1[j]);
            t2[j] = fma(__ldg(a2 + k + 32 * j), uk, t2[j]);
          }
        }
        for (; k < nP; k += 32) {
          const double uk = vu[k];
          t0[0] = fma(__ldg(a0 + k), uk, t0[0]);
          t1[0] = fma(__ldg(a1 + k), uk, t1[0]);
          t2[0] = fma(__ldg(a2 + k), uk, t2[0]);
        }
        s0 = (t0[0] + t0[1]) + (t0[2] + t0[3]);
        s1 = (t1[0] + t1[1]) + (t1[2] + t1[3]);
        s2 = (t2[0] + t2[1]) + (t2[2] + t2[3]);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
      }
      dpart = fma(s0, vu[row0 + r0], dpart);
      if (h1) dpart = fma(s1, vu[row0 + r0 + 1], dpart);
      if (h2) dpart = fma(s2, vu[row0 + r0 + 2], dpart);
      if (lane < csize) {
        double* dst = cluster.map_shared_rank(wbuf, lane) + row0 + r0;
        dst[0] = s0;
        if (h1) dst[1] = s1;
        if (h2) dst[2] = s2;
      }
    }
    if (lane < csize) cluster.map_shared_rank(dbuf, lane)[rank * NW + wid] = dpart;
  };

  // [C] g (CTA-local slots of phase A) and d (cluster-wide slots of phase B), identical in every thread
  auto phase_c = [&](int it, double& g, double& d) {
    const double* gs = gslot + (it & 1) * NW;
    const double* ds = dslot + ((it + 1) & 1) * (MAXC * NW);
    double pg = (lane < NW) ? gs[lane] : 0.0;
    double pd = 0.0;
    for (int k = lane; k < csize * NW; k += 32) pd += ds[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      pg += __shfl_xor_sync(0xffffffffu, pg, o);
      pd += __shfl_xor_sync(0xffffffffu, pd, o);
    }
    g = pg; d = pd;
  };

  double g = 0.0, d = 0.0;
  phase_a(0, 0.0, 0.0);
  __syncthreads();
  cluster.sync();  // every CTA of the cluster is running before the first remote write
  phase_b(0);
  cluster.sync();
  phase_c(0, g, d);
  const double g0 = g;
  double alpha = (d > 0.0) ? g / d : 0.0, beta = 0.0;
  int it = 0, flag = 0;
  long long tprof[5] = {0, 0, 0, 0, 0};  // cycles: A, block barrier, B, cluster barrier, C (thread 0)
  if (g0 > 0.0 && !(d > 0.0)) flag = 1;
  if (g0 > 0.0 && flag == 0) {
    for (it = 1; it <= max_iter; ++it) {
      const long long c0 = clock64();
      phase_a(it, alpha, beta);
      const long long c1 = clock64();
      __syncthreads();
      const long long c2 = clock64();
      phase_b(it);
      const long long c3 = clock64();
      cluster.sync();
      const long long c4 = clock64();
      double gn, dn;
      phase_c(it, gn, dn);
      const long long c5 = clock64();
      tprof[0] += c1 - c0; tprof[1] += c2 - c1; tprof[2] += c3 - c2; tprof[3] += c4 - c3; tprof[4] += c5 - c4;
      if (!(gn == gn) || !(dn == dn)) { flag = 2; break; }
      if (gn <= tol2 * g0) { g = gn; break; }
      beta = gn / g;
      const double den = dn - beta * gn / alpha;
      if (!(den > 0.0)) { flag = 1; g = gn; break; }
      alpha = gn / den;
      g = gn;
    }
  }
  cluster.sync();  // nobody exits while peers may still write into its buffers
  if (rank == 0) {
    for (int i = tid; i < nP; i += PCG_THREADS) xout[i] = vx[i];  // x and r were advanced together in phase A
    if (tid == 0) {
      sc[SC_PCG_ITS] = (double)it;
      sc[SC_PCG_REL] = (g0 > 0.0) ? sqrt(fabs(g) / g0) : 0.0;
      sc[SC_PCG_FLAG] = (double)flag;
      for (int k = 0; k < 5; ++k) sc[SC_PCG_T0 + k] = (double)tprof[k];
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Direct solve of the reduced camera system for SMALL rigs (n = n_camera_params <= DIRECT_MAX_N: up to 16 cameras with
// extrinsics only -- every rig Caliscope ships fixtures for).  One CTA, the lower triangle of S in shared memory with the
// right-hand side as an extra row n, LDL^T without pivoting (S is SPD: U + damping minus a Schur term):
//   step k: every thread reads column k (final since step k-1) and updates trailing entries
//           a_ij -= a_ik a_jk / d_k  (k < j <= i <= n): one block barrier per step; row n comes out as z = L^-1 (-b)
//   back substitution L^T x = D^-1 z by warp 0 alone (register-resident, shuffles, no block barrier).
// Same contract as pcg_cluster_kernel: x solves S x = -b; SC_PCG_FLAG = 1 on a non-positive pivot, 2 on NaN.
// A small PCG needs ~20 cluster-synchronised iterations per trial; this is one pass of one CTA, run inside
// small_rig_step_kernel (cb_lm.cuh).
// ---------------------------------------------------------------------------------------------
constexpr int DIRECT_MAX_N = 96;
constexpr int DIRECT_THREADS = 256;
__device__ __forceinline__ void dense_ldlt_body(double* __restrict__ dsm, const double* __restrict__ S,
                                                const double* __restrict__ bvec, int n, double* __restrict__ xout,
                                                double* __restrict__ sc) {
  const int ld = n | 1;  // odd row stride: a warp touching two rows spreads over all banks
  double* A = dsm;                  // (n + 1) x ld, lower triangle used
  double* dinv = dsm + (size_t)(n + 1) * ld;
  const int tid = threadIdx.x;
  for (int idx = tid; idx < n * n; idx += DIRECT_THREADS) {
    const int i = idx / n, j = idx - i * n;
    if (j <= i) A[i * ld + j] = S[(size_t)i * n + j];
  }
  for (int j = tid; j < n; j += DIRECT_THREADS) A[n * ld + j] = -bvec[j];
  const int tx = tid & 15, ty = tid >> 4;
  int flag = 0;
  for (int k = 0; k < n; ++k) {
    __syncthreads();
    const double dk = A[k * ld + k];
    if (!(dk > 0.0)) { flag = (dk == dk) ? 1 : 2; break; }  // uniform: every thread reads the same pivot
    const double inv = 1.0 / dk;
    if (tid == 0) dinv[k] = inv;
    for (int i = k + 1 + ty; i <= n; i += 16) {
      const double lik = A[i * ld + k] * inv;
      for (int j = k + 1 + tx; j <= i && j < n; j += 16) A[i * ld + j] = fma(-lik, A[j * ld + k], A[i * ld + j]);
    }
  }
  __syncthreads();
  if (flag == 0 && tid < 32) {
    // l_k = z_k / d_k held by lane k % 32; x_i known for i > current k
    constexpr int PER = (DIRECT_MAX_N + 31) / 32;
    double l[PER], di[PER];
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      const int k = tid + 32 * q;
      di[q] = k < n ? dinv[k] : 0.0;
      l[q] = k < n ? A[n * ld + k] * di[q] : 0.0;
    }
    for (int i = n - 1; i >= 0; --i) {
      double own = 0.0;
#pragma unroll
      for (int q = 0; q < PER; ++q)
        if (q == (i >> 5)) own = l[q];
      const double xi = __shfl_sync(0xffffffffu, own, i & 31);
#pragma unroll
      for (int q = 0; q < PER; ++q) {
        const int k = tid + 32 * q;
        if (k < i) l[q] = fma(-A[i * ld + k] * di[q], xi, l[q]);
      }
    }
    bool bad = false;
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      const int k = tid + 32 * q;
      if (k < n) { xout[k] = l[q]; bad |= !(l[q] == l[q]); }
    }
    if (__any_sync(0xffffffffu, bad)) flag = 2;
  }
  if (tid == 0) {
    sc[SC_PCG_ITS] = 1.0;
    sc[SC_PCG_REL] = 0.0;
    sc[SC_PCG_FLAG] = (double)flag;
  }
}

// ---------------------------------------------------------------------------------------------
// index building helpers (setup)
// ---------------------------------------------------------------------------------------------
__global__ void make_keys_kernel(const int* __restrict__ a, const int* __restrict__ b, long long nb, int n,
                                 unsigned long long* __restrict__ keys, int* __restrict__ vals) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    keys[i] = (unsigned long long)a[i] * (unsigned long long)nb + (unsigned long long)b[i];
    vals[i] = i;
  }
}
// sorted keys = major*nb + minor -> major/minor arrays
__global__ void split_keys_kernel(const unsigned long long* __restrict__ keys, long long nb, int n,
                                  int* __restrict__ major, int* __restrict__ minor) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    major[i] = (int)(keys[i] / (unsigned long long)nb);
    minor[i] = (int)(keys[i] % (unsigned long long)nb);
  }
}
// start[j] = first index i with sorted_major[i] >= j, j in [0, nbins]
__global__ void lower_bound_kernel(const int* __restrict__ sorted_major, int n, int nbins, int* __restrict__ start) {
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j > nbins) return;
  int lo = 0, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (sorted_major[mid] < j) lo = mid + 1; else hi = mid;
  }
  start[j] = lo;
}
// camera-major gather: q -> point-major position -> (point, original observation, xy)
__global__ void cm_gather_kernel(const int* __restrict__ cm_pos, const int* __restrict__ pm_orig,
                                 const int* __restrict__ pm_pt, const double2* __restrict__ obs_xy, int n,
                                 int* __restrict__ cm_pt, int* __restrict__ cm_orig, double2* __restrict__ cm_xy) {
  int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q < n) {
    const int pos = cm_pos[q];
    const int o = pm_orig[pos];
    cm_pt[q] = pm_pt[pos];
    cm_orig[q] = o;
    cm_xy[q] = obs_xy[o];
  }
}
__global__ void widen_i16_kernel(const short* __restrict__ in, int n, int* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (int)in[i];
}
// caller's camera id -> internal slot, in place
__global__ void remap_kernel(int* __restrict__ a, const int* __restrict__ map, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = map[a[i]];
}
// co-visibility counts over a sample of points (one warp per sampled point): W[a][b] += 1 for every pair of cameras
// that see it.  Only used to choose the internal camera order of sparse rigs.
__global__ void covis_kernel(const int* __restrict__ pt_start, const int* __restrict__ pm_cam, int n_pts, int stride,
                             int n_cams, unsigned int* __restrict__ W) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const long long j = (long long)w * stride;
  if (j >= n_pts) return;
  const int s = pt_start[j], e = min(pt_start[j + 1], s + 256);
  for (int a = s + lane; a < e; a += 32) {
    const int ca = pm_cam[a];
    if (a > s && pm_cam[a - 1] == ca) continue;
    for (int b = s; b < e; ++b) {
      const int cb = pm_cam[b];
      if (b > s && pm_cam[b - 1] == cb) continue;
      atomicAdd(&W[(size_t)ca * n_cams + cb], 1u);
    }
  }
}
// per point: bit I set iff some camera that sees the point owns a column of Schur tile I (pm_cam holds internal slots)
__global__ void pt_tile_mask_kernel(const int* __restrict__ pt_start, const int* __restrict__ pm_cam, int n_pts, int P,
                                    unsigned long long* __restrict__ mask) {
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_pts) return;
  unsigned long long m = 0ull;
  for (int pos = pt_start[j]; pos < pt_start[j + 1]; ++pos) {
    const int c0 = pm_cam[pos] * P;
    m |= 1ull << (c0 / SY_TILE);
    m |= 1ull << ((c0 + P - 1) / SY_TILE);
  }
  mask[j] = m;
}
// per rigid-constraint component: every point gets the union of its component's tile masks.  comp_build_kernel writes a
// component point's Zt rows in the columns of every camera that sees ANY point of the component, so a point seen only
// from tile A still has non-zero rows in tile B when another point of its component is seen from B.  Components are
// disjoint, so one thread per component reads and writes its own points only.
__global__ void comp_tile_mask_kernel(const int* __restrict__ comp_pt_start, const int* __restrict__ comp_pts, int n_comp,
                                      unsigned long long* __restrict__ mask) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_comp) return;
  unsigned long long m = 0ull;
  for (int i = comp_pt_start[c]; i < comp_pt_start[c + 1]; ++i) m |= mask[comp_pts[i]];
  for (int i = comp_pt_start[c]; i < comp_pt_start[c + 1]; ++i) mask[comp_pts[i]] = m;
}
// cnt[tile(I,J)] = number of points whose mask has bits I and J (I <= J; tile(I,J) = I*nb - I(I-1)/2 + J-I): what the host
// needs to choose between the dense and the k-list Schur product, without downloading the masks.  Lanes holding the same
// mask (the usual case: neighbouring points are seen by the same cameras) are counted once per warp.
__global__ void tile_pair_count_kernel(const unsigned long long* __restrict__ mask, int n_pts, int nb,
                                       unsigned long long* __restrict__ cnt) {
  extern __shared__ unsigned int tp_cnt[];
  const int nt = nb * (nb + 1) / 2;
  for (int i = threadIdx.x; i < nt; i += blockDim.x) tp_cnt[i] = 0u;
  __syncthreads();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long m = j < n_pts ? mask[j] : 0ull;
  const unsigned peers = __match_any_sync(0xffffffffu, m);
  if (m && (threadIdx.x & 31) == __ffs(peers) - 1) {
    const unsigned k = __popc(peers);
    for (unsigned long long a = m; a; a &= a - 1) {
      const int I = __ffsll((long long)a) - 1;
      for (unsigned long long b = a; b; b &= b - 1) {
        const int J = __ffsll((long long)b) - 1;
        atomicAdd(&tp_cnt[I * nb - I * (I - 1) / 2 + (J - I)], k);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nt; i += blockDim.x)
    if (tp_cnt[i]) atomicAdd(&cnt[i], (unsigned long long)tp_cnt[i]);
}
// Compacted row lists of the sparse Schur product, built on the device.  Every (tile pair, point) incidence becomes one
// 64-bit key  tile(I,J) * n_pts + point  (inc_count / exclusive scan / inc_emit: no atomics, fixed positions); a radix sort
// leaves each tile pair's points contiguous and ascending; klist_expand writes rows 3j..3j+2 at the pair's offset.  Padding
// entries (to a multiple of SY_KC per pair) keep the fill value = the index of an all-zero row.
__global__ void inc_count_kernel(const unsigned long long* __restrict__ mask, int n_pts, int* __restrict__ n_inc) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_pts) return;
  const int b = __popcll(mask[j]);
  n_inc[j] = b * (b + 1) / 2;
}
__global__ void inc_emit_kernel(const unsigned long long* __restrict__ mask, const int* __restrict__ inc_off, int n_pts,
                                int nb, unsigned long long* __restrict__ keys) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_pts) return;
  int o = inc_off[j];
  for (unsigned long long a = mask[j]; a; a &= a - 1) {
    const int I = __ffsll((long long)a) - 1;
    for (unsigned long long b = a; b; b &= b - 1) {
      const int J = __ffsll((long long)b) - 1;
      keys[o++] = (unsigned long long)(I * nb - I * (I - 1) / 2 + (J - I)) * (unsigned long long)n_pts + (unsigned long long)j;
    }
  }
}
__global__ void fill_int_kernel(int* __restrict__ a, long long n, int v) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) a[i] = v;
}
__global__ void klist_expand_kernel(const unsigned long long* __restrict__ keys_sorted, long long n_inc, int n_pts,
                                    const long long* __restrict__ pair_start, const long long* __restrict__ koff,
                                    int* __restrict__ klist) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n_inc) return;
  const unsigned long long key = keys_sorted[i];
  const int t = (int)(key / (unsigned long long)n_pts);
  const int j = (int)(key - (unsigned long long)t * (unsigned long long)n_pts);
  const long long base = koff[t] + 3 * (i - pair_start[t]);
  klist[base] = 3 * j;
  klist[base + 1] = 3 * j + 1;
  klist[base + 2] = 3 * j + 2;
}
// point-major pixel list
__global__ void pm_gather_kernel(const int* __restrict__ pm_orig, const double2* __restrict__ obs_xy, int n,
                                 double2* __restrict__ pm_xy) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) pm_xy[i] = obs_xy[pm_orig[i]];
}
__global__ void count_dups_kernel(const int* __restrict__ pm_pt, const int* __restrict__ pm_cam, int n,
                                  int* __restrict__ count) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > 0 && i < n && pm_pt[i] == pm_pt[i - 1] && pm_cam[i] == pm_cam[i - 1]) atomicAdd(count, 1);
}
__global__ void validate_kernel(const int* __restrict__ cam, const int* __restrict__ pt, int n, int n_cams, int n_pts,
                                int* __restrict__ bad) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && (cam[i] < 0 || cam[i] >= n_cams || pt[i] < 0 || pt[i] >= n_pts)) atomicAdd(bad, 1);
}

// ---------------------------------------------------------------------------------------------
// per-camera order statistics of non-negative doubles (camera-major, contiguous per camera):
// 8-bit radix select on the IEEE bit pattern, one block per camera, two ranks per call
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
order_stats_kernel(const double* __restrict__ err_cm, const int* __restrict__ cam_start, double qfrac,
                   double* __restrict__ lo_out, double* __restrict__ hi_out, long long* __restrict__ cnt_out) {
  __shared__ unsigned int hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ long long s_k;
  const int c = blockIdx.x;
  const int s = cam_start[c], e = cam_start[c + 1];
  const long long n = e - s;
  if (threadIdx.x == 0) cnt_out[c] = n;
  if (n == 0) {
    if (threadIdx.x == 0) { lo_out[c] = 0.0; hi_out[c] = 0.0; }
    return;
  }
  const double vidx = (double)(n - 1) * qfrac;
  long long klo = (long long)floor(vidx);
  if (klo < 0) klo = 0;
  if (klo > n - 1) klo = n - 1;
  long long khi = klo + 1 < n ? klo + 1 : n - 1;
  for (int which = 0; which < 2; ++which) {
    if (threadIdx.x == 0) { s_prefix = 0ull; s_k = which ? khi : klo; }
    __syncthreads();
    for (int pass = 7; pass >= 0; --pass) {
      hist[threadIdx.x] = 0u;
      __syncthreads();
      const unsigned long long prefix = s_prefix;
      const int shift = 8 * pass;
      for (int i = s + threadIdx.x; i < e; i += 256) {
        const unsigned long long key = (unsigned long long)__double_as_longlong(err_cm[i]);
        const bool match = (pass == 7) || ((key >> (shift + 8)) == prefix);
        if (match) atomicAdd(&hist[(unsigned)((key >> shift) & 0xffull)], 1u);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        long long k = s_k;
        int b = 0;
        for (; b < 256; ++b) {
          if (k < (long long)hist[b]) break;
          k -= hist[b];
        }
        s_k = k;
        s_prefix = (prefix << 8) | (unsigned long long)b;
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      const double v = __longlong_as_double((long long)s_prefix);
      if (which) hi_out[c] = v; else lo_out[c] = v;
    }
    __syncthreads();
  }
}

// per camera: number of observations with error <= threshold, and sum of squared errors (block per camera)
__global__ void __launch_bounds__(256)
cam_err_stats_kernel(const double* __restrict__ err_cm, const int* __restrict__ cam_start,
                     const double* __restrict__ thr, long long* __restrict__ kept, double* __restrict__ sumsq) {
  __shared__ double sh[8];
  __shared__ long long shk[8];
  const int c = blockIdx.x;
  const double t = thr ? thr[c] : 0.0;
  long long k = 0;
  double s = 0.0;
  for (int i = cam_start[c] + threadIdx.x; i < cam_start[c + 1]; i += 256) {
    const double e = err_cm[i];
    k += (thr && e <= t) ? 1 : 0;
    s = fma(e, e, s);
  }
  s = warp_sum(s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) k += __shfl_xor_sync(0xffffffffu, k, o);
  if ((threadIdx.x & 31) == 0) { sh[threadIdx.x >> 5] = s; shk[threadIdx.x >> 5] = k; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    long long b = 0;
    for (int w = 0; w < 8; ++w) { a += sh[w]; b += shk[w]; }
    sumsq[c] = a;
    if (kept) kept[c] = b;
  }
}

// keep flag per observation in CALLER order: error <= threshold of its camera (camera found from cam_start)
__global__ void keep_flag_kernel(const double* __restrict__ err_cm, const int* __restrict__ cm_orig,
                                 const int* __restrict__ cam_start, int n_cams, const double* __restrict__ thr, int n,
                                 unsigned char* __restrict__ flag) {
  int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  int lo = 0, hi = n_cams;  // largest c with cam_start[c] <= q
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (cam_start[mid] <= q) lo = mid; else hi = mid;
  }
  flag[cm_orig[q]] = err_cm[q] <= thr[lo] ? 1 : 0;
}

// gather the kept observations (indices `sel` into the caller-order arrays) into compact arrays
__global__ void gather_obs_kernel(const int* __restrict__ sel, int n_sel, const int* __restrict__ cam,
                                  const int* __restrict__ pt, const double2* __restrict__ xy, int* __restrict__ cam_o,
                                  int* __restrict__ pt_o, double2* __restrict__ xy_o) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_sel) {
    const int o = sel[i];
    cam_o[i] = cam[o];
    pt_o[i] = pt[o];
    xy_o[i] = xy[o];
  }
}
__global__ void iota_kernel(int* __restrict__ a, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = i;
}

__global__ void cm_to_orig_kernel(const double* __restrict__ in_cm, const int* __restrict__ cm_orig, int n,
                                  double* __restrict__ out) {
  int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q < n) out[cm_orig[q]] = in_cm[q];
}

}  // namespace cb
