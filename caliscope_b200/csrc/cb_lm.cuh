// Device-resident Levenberg-Marquardt state machine and the Jacobian-free point kernels.
//
// Round-2 structure of one LM trial (every kernel reads the damping, the current-buffer index and the
// stop flag from LmState in device memory, so the host never has to look at a number between launches and
// the whole trial replays as one CUDA graph):
//
//   pt_pass_kernel        per point: recompute r, Jp, Jc of its observations from (pixel, camera table, point),
//                         V = sum Jp^T Jp, g = sum Jp^T r, Marquardt scale, 3x3 damped Cholesky, t = L^-1 g and
//                         Z = (Jc^T Jp) L^-T into the k-major Schur factor, as whole 64-byte granules   [reprojection.py:171-205]
//   schur_syrk_kernel     Z Z^T (+ Z t), split-K                                               (cb_kernels.cuh)
//   schur_finalize(_peer) S = U - Z Z^T, b = g_c - Z t (+ the all-reduce over NVLink peers)
//   reduced_prep_kernel   damping, gradient norm, gtol / max_nfev tests, block-Jacobi inverses
//   pcg_cluster_kernel    reduced camera solve
//   cam_step_kernel       camera step, bounds clamp, predicted reduction, camera table of the trial point
//                         (n_camera_params <= 96: these three are small_rig_step_kernel, with a direct LDL^T solve)
//   pt_backsub_kernel     dX = -L^-T (t + L sum Jp^T (Jc dc)), again recomputed from the observation list
//   resjac_kernel<P,5>    camera-major pass at the TRIAL point: cost, U_c, g_c (these are the next linearisation's
//                         camera blocks if the step is accepted)
//   trial_reduce_kernel   chunk partials -> per-camera blocks, trial sums, and (single GPU) the accept/reject decision
//   lm_decide_kernel      (multi GPU) 4-double all-reduce over peer memory + the decision
//
// The decision follows scipy's TRF bookkeeping (site-packages/scipy/optimize/_lsq/trf.py:465-560,
// common.py:705-717): nfev / njev / nit count the same events, termination statuses 0..4 are scipy's.
//
// Held parameters -- fixed sets (DESIGN.md §4.12) and Gaussian priors (§4.13, cb_priors.cuh) -- enter behind one template
// flag per side, chosen at creation: HELD in reduced_prep_body (camera priors into S and b, then unit rows / columns of S
// and zero b for fixed camera parameters, before the damping) and HELD in pt_pass_kernel (point priors into V and g, and
// V^-1 := 0 for a fixed point, flagged in the pad slot of xp4).  pt_backsub_kernel's FIXP gives a fixed point a zero step.
#pragma once
#include "cb_covariance.cuh"
#include "cb_priors.cuh"

namespace cb {

constexpr int LM_ERR_NONFINITE_X0 = 1;   // scipy: "Residuals are not finite in the initial point."
constexpr int LM_ERR_STUCK_NONFINITE = 2;  // damping saturated and every trial non-finite: stop instead of spinning

struct LmLogRow {
  double nit, nfev, cost, cost_new, ratio, lam, step, gnorm, pcg;
};

// ---------------------------------------------------------------------------------------------
// Point pass.  LANES lanes per point (32 / LANES points per warp), persistent grid-stride over points so the camera
// table is staged into shared memory once per CTA.  DUPS: repeated (camera, point) rows exist (static objects seen
// in many frames); they are adjacent in the point-major list and the first lane of a run sums the run.
// Points tied by rigid-distance constraints (pt_comp >= 0) only get V, g and the untransformed W = Jc^T Jp written to
// their Zt rows; comp_build_kernel eliminates the component.
// ---------------------------------------------------------------------------------------------
// CAMSM: the camera table is staged in shared memory (it fits: <= 64 KB).  A template parameter, not a run-time pointer
// select: with a pointer that may be shared or global the compiler emits GENERIC loads (LD.E) for the ~36 table reads per
// observation, which wait on the long scoreboard like global loads (ncu: 55 % of the stalls of the first version).
//
// COV: the covariance linearisation (cb_covariance.cuh).  The damping is ignored and the factor is the pseudo-inverse root R
// of V (V^+ = R^T R, 9 values per point into Linv6, rank(V) into pt_rank, -1 for component points); Z = (Jc^T Jp) R^T,
// t = 0, and neither Dp2 nor the gradient norm is touched.
//
// HELD: the problem holds some points fixed (DESIGN §4.12) or near a prior (§4.13).  A fixed point carries 1.0 in the pad
// slot of xp4 (0.0 otherwise) and is a constant: its factor is zero (V^-1 := 0, so Z = 0 and t = 0), its gradient is left
// out of the gradient norm, and the covariance variant reports rank -2 for it.  The prior of point j (pp.idx[j] >= 0;
// every entry is -1 in a problem with fixed points only) adds L_j to V_j and L_j (X_j - m_j) to g_j before D, the damping
// and the factor are formed.
template <bool COV>
__device__ __forceinline__ void pt_factor_rows(const double* JX, const double* Li, double& q00, double& q01, double& q02,
                                               double& q10, double& q11, double& q12) {
  if constexpr (COV) {
    q00 = JX[0] * Li[0] + JX[1] * Li[1] + JX[2] * Li[2];
    q01 = JX[0] * Li[3] + JX[1] * Li[4] + JX[2] * Li[5];
    q02 = JX[0] * Li[6] + JX[1] * Li[7] + JX[2] * Li[8];
    q10 = JX[3] * Li[0] + JX[4] * Li[1] + JX[5] * Li[2];
    q11 = JX[3] * Li[3] + JX[4] * Li[4] + JX[5] * Li[5];
    q12 = JX[3] * Li[6] + JX[4] * Li[7] + JX[5] * Li[8];
  } else {
    q00 = JX[0] * Li[0]; q01 = JX[0] * Li[1] + JX[1] * Li[2]; q02 = JX[0] * Li[3] + JX[1] * Li[4] + JX[2] * Li[5];
    q10 = JX[3] * Li[0]; q11 = JX[3] * Li[1] + JX[4] * Li[2]; q12 = JX[3] * Li[3] + JX[4] * Li[4] + JX[5] * Li[5];
  }
}

// Zt staging of one point group (dynamic shared memory after the camera table): the Z pieces of one round of LANES rows
// (lane l's in slot l + 1; slot 0 keeps the last piece of the previous round), their cameras, and the 64-byte granules
// the round writes as (granule << 12 | slot of the previous piece << 6 | owning slot).  A P-double piece touches at most
// two granules of a row.
template <int P, int LANES>
struct PtStage {
  double z[LANES + 1][3][P];
  int cam[LANES + 1];
  int list[2 * LANES];
};
template <int P, int LANES>
constexpr size_t pt_stage_bytes() { return sizeof(PtStage<P, LANES>) * PT_WARPS * (32 / LANES); }

template <int P, int LANES, bool DUPS, bool CAMSM, bool COV = false, bool HELD = false>
__global__ void __launch_bounds__(PT_WARPS * 32, 2)
pt_pass_kernel(const LmState* __restrict__ st, const int* __restrict__ pt_start, const int* __restrict__ pm_cam,
               const double2* __restrict__ pm_xy, const int* __restrict__ pt_comp, int n_pts, int n_cams,
               CPtr2 camtab2, CPtr2 xp2, double* __restrict__ V6, double* __restrict__ gp,
               double* __restrict__ Dp2, double* __restrict__ Linv6, double* __restrict__ tvec,
               double* __restrict__ Zt, size_t LD, unsigned long long* __restrict__ gmax_bits,
               int* __restrict__ pt_rank, PointPriors pp) {
  extern __shared__ __align__(16) double pt_sm[];
  __shared__ double wmax[PT_WARPS];
  if (st->done) return;
  const int cur = st->cur;
  const double lam = st->lam;
  const int loss = st->loss;
  const double fscale = st->fscale;
  const double* __restrict__ gtab = camtab2.p[cur];
  const double* xp4 = xp2.p[cur];
  constexpr int cstride = CAMSM ? CT_SMEM : CT_SIZE;
  if constexpr (CAMSM) {
    for (int i = threadIdx.x; i < n_cams * CT_SIZE; i += blockDim.x) pt_sm[(i / CT_SIZE) * CT_SMEM + i % CT_SIZE] = gtab[i];
    __syncthreads();
  }
  // camera table entry of camera c: shared (LDS) or global (LDG), decided at compile time
  auto cam_entry = [&](int c) -> const double* {
    if constexpr (CAMSM) return pt_sm + (size_t)c * cstride;
    else return gtab + (size_t)c * cstride;
  };
  constexpr int GPW = 32 / LANES;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int gl = lane % LANES, grp = lane / LANES;
  constexpr unsigned LMASK = LANES == 32 ? 0xffffffffu : (1u << LANES) - 1u;
  const unsigned gmask = LMASK << (grp * LANES);
  double gm = 0.0;
  for (int j0 = (blockIdx.x * PT_WARPS + wid) * GPW; j0 < n_pts; j0 += gridDim.x * PT_WARPS * GPW) {
    const int j = j0 + grp;
    const bool valid = j < n_pts;
    int s = 0, e = 0;
    double X0 = 0.0, X1 = 0.0, X2 = 0.0, X3;
    if (valid) {
      s = pt_start[j]; e = pt_start[j + 1];
      ld256nc(xp4 + 4 * (size_t)j, X0, X1, X2, X3);
    }
    (void)X3;
    const bool in_comp = valid && pt_comp != nullptr && pt_comp[j] >= 0;
    // ---- phase 1: V, g over the point's observations (residual and d f / d X only)
    double v[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) v[k] = 0.0;
    // (index / pixel of the next row are requested before the current one is evaluated: the kernel is latency bound --
    // 16 warps per SM, long_scoreboard 60 % of the stalls in the first version)
    int cam_n = 0;
    double2 xy_n = make_double2(0.0, 0.0);
    bool unsorted = false;  // the point's rows are not in camera-slot order (the engine reordered the cameras)
    if (s + gl < e) { cam_n = pm_cam[s + gl]; xy_n = pm_xy[s + gl]; }
    for (int pos = s + gl; pos < e; pos += LANES) {
      const int cam = cam_n;
      const double2 xy = xy_n;
      if (pos + LANES < e) { cam_n = pm_cam[pos + LANES]; xy_n = pm_xy[pos + LANES]; }
      if (!DUPS && pos + 1 < e && pm_cam[pos + 1] < cam) unsorted = true;
      double f[2], JX[6];
      obs_res_jx(cam_entry(cam), X0, X1, X2, xy.x, xy.y, loss, fscale, f, JX);
      v[0] += JX[0] * JX[0] + JX[3] * JX[3]; v[1] += JX[0] * JX[1] + JX[3] * JX[4]; v[2] += JX[0] * JX[2] + JX[3] * JX[5];
      v[3] += JX[1] * JX[1] + JX[4] * JX[4]; v[4] += JX[1] * JX[2] + JX[4] * JX[5]; v[5] += JX[2] * JX[2] + JX[5] * JX[5];
      v[6] += JX[0] * f[0] + JX[3] * f[1]; v[7] += JX[1] * f[0] + JX[4] * f[1]; v[8] += JX[2] * f[0] + JX[5] * f[1];
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) v[k] = group_sum<LANES>(v[k]);
    if constexpr (HELD) {
      const int q = valid ? pp.idx[j] : -1;
      if (q >= 0) {
        const double* L = pp.info + 9 * (size_t)q;
        const double* m = pp.mean + 3 * (size_t)q;
        const double d0 = X0 - m[0], d1 = X1 - m[1], d2 = X2 - m[2];
        v[0] += L[0]; v[1] += L[1]; v[2] += L[2]; v[3] += L[4]; v[4] += L[5]; v[5] += L[8];
        v[6] += fma(L[0], d0, fma(L[1], d1, L[2] * d2));
        v[7] += fma(L[3], d0, fma(L[4], d1, L[5] * d2));
        v[8] += fma(L[6], d0, fma(L[7], d1, L[8] * d2));
      }
    }
    bool pieces_only = false;
    if constexpr (!DUPS) pieces_only = ((__ballot_sync(0xffffffffu, unsorted) >> (grp * LANES)) & LMASK) != 0;
    double D[3] = {1.0, 1.0, 1.0};
    if (valid) {
      const double* d = Dp2 + (size_t)j * 3;
      D[0] = fmax(d[0], v[0]); D[1] = fmax(d[1], v[3]); D[2] = fmax(d[2], v[5]);
    }
    constexpr int NL = COV ? 9 : 6;
    double Li[NL];
    int rank = -1;
    // the flag is read again here rather than kept from the load above: live across the observation loop it costs spills
    const bool fixed = HELD && valid && xp4[4 * (size_t)j + 3] != 0.0;
    if (in_comp) {
#pragma unroll
      for (int k = 0; k < NL; ++k) Li[k] = 0.0;
      if constexpr (COV) Li[0] = Li[4] = Li[8] = 1.0;
      else Li[0] = Li[2] = Li[5] = 1.0;
    } else if (fixed) {
#pragma unroll
      for (int k = 0; k < NL; ++k) Li[k] = 0.0;
      rank = -2;
    } else {
      if constexpr (COV) pinv_root3(v, Li, rank);
      else chol3_inv(v, D, lam, Li);
    }
    if constexpr (COV) {
      if (valid && gl == 0) {
#pragma unroll
        for (int k = 0; k < 6; ++k) V6[(size_t)j * 6 + k] = v[k];
#pragma unroll
        for (int k = 0; k < 9; ++k) Linv6[(size_t)j * 9 + k] = Li[k];
#pragma unroll
        for (int k = 0; k < 3; ++k) gp[(size_t)j * 3 + k] = v[6 + k];
        if (!in_comp)
#pragma unroll
          for (int k = 0; k < 3; ++k) tvec[3 * (size_t)j + k] = 0.0;
        pt_rank[j] = rank;
      }
    } else if (valid && gl == 0) {
#pragma unroll
      for (int k = 0; k < 6; ++k) V6[(size_t)j * 6 + k] = v[k];
#pragma unroll
      for (int k = 0; k < 3; ++k) { gp[(size_t)j * 3 + k] = v[6 + k]; Dp2[(size_t)j * 3 + k] = D[k]; }
      if (!in_comp) {
#pragma unroll
        for (int k = 0; k < 6; ++k) Linv6[(size_t)j * 6 + k] = Li[k];
        tvec[3 * (size_t)j + 0] = Li[0] * v[6];
        tvec[3 * (size_t)j + 1] = Li[1] * v[6] + Li[2] * v[7];
        tvec[3 * (size_t)j + 2] = Li[3] * v[6] + Li[4] * v[7] + Li[5] * v[8];
        if (!fixed) gm = fmax(gm, fmax(fabs(v[6]), fmax(fabs(v[7]), fabs(v[8]))));
      }
    }
    // ---- phase 2: Z = (Jc^T Jp) Linv^T per (camera, point) pair, rows 3j..3j+2 of the k-major factor.
    if constexpr (DUPS) {
      // Run-summed pieces (rigs with few cameras whose points repeat rows) are stored as they are: staging does not pay
      // on those shapes (cfg2, cfg3; DESIGN §7), and this loop is the one the kernel had before staging.
      for (int pos = s + gl; pos < e; pos += LANES) {
        const int cam = pm_cam[pos];
        if (pos > s && pm_cam[pos - 1] == cam) continue;  // not the first row of its (point, camera) run
        double f[2], JX[6], Jc[2 * P];
        double z[3][P];
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
          for (int p = 0; p < P; ++p) z[a][p] = 0.0;
        int r = pos;
        do {
          const double2 xy = pm_xy[r];
          obs_jac<P>(cam_entry(cam), X0, X1, X2, xy.x, xy.y, loss, fscale, f, JX, Jc);
          double q00, q01, q02, q10, q11, q12;
          pt_factor_rows<COV>(JX, Li, q00, q01, q02, q10, q11, q12);
#pragma unroll
          for (int p = 0; p < P; ++p) {
            z[0][p] = fma(Jc[p], q00, fma(Jc[P + p], q10, z[0][p]));
            z[1][p] = fma(Jc[p], q01, fma(Jc[P + p], q11, z[1][p]));
            z[2][p] = fma(Jc[p], q02, fma(Jc[P + p], q12, z[2][p]));
          }
          ++r;
        } while (r < e && pm_cam[r] == cam);
        (void)f;
        double* z0 = Zt + (3 * (size_t)j) * LD + (size_t)cam * P;
        if constexpr (P == 6) {
#pragma unroll
          for (int a = 0; a < 3; ++a) {
            double2* dst = reinterpret_cast<double2*>(z0 + a * LD);  // cam*48 B and LD*8 B are 16-byte multiples
            dst[0] = make_double2(z[a][0], z[a][1]);
            dst[1] = make_double2(z[a][2], z[a][3]);
            dst[2] = make_double2(z[a][4], z[a][5]);
          }
        } else {
#pragma unroll
          for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int p = 0; p < P; ++p) z0[a * LD + p] = z[a][p];
        }
      }
    } else {
      // Written as whole 64-byte granules, four lanes per granule, from pieces staged in shared memory: stored piece by
      // piece, most granules of a row reach L2 as partial pieces in many requests, and the store stream ran at a third
      // of the rate of whole granules (profiles/microbench/zt_store.cu, DESIGN §7).  Each round of LANES rows writes the
      // granules its pieces touch, zeros included where a granule covers a camera the point does not see (a structural
      // zero), except a last granule the next camera's piece shares: the next round writes that one, reading this
      // round's last piece from slot 0.
      PtStage<P, LANES>& sg =
          reinterpret_cast<PtStage<P, LANES>*>(pt_sm + (CAMSM ? (size_t)n_cams * CT_SMEM : 0))[wid * GPW + grp];
      if (gl == 0) sg.cam[0] = -1;
      if (s + gl < e) { cam_n = pm_cam[s + gl]; xy_n = pm_xy[s + gl]; }
      for (int base = s; base < e; base += LANES) {
        const int pos = base + gl;
        int cam = -1, next = -1;
        bool has = false;
        double* zs = &sg.z[gl + 1][0][0];  // this lane's piece
        if (pos < e) {
          double f[2], JX[6], Jc[2 * P];
          cam = cam_n;
          const double2 xy = xy_n;
          if (pos + LANES < e) { cam_n = pm_cam[pos + LANES]; xy_n = pm_xy[pos + LANES]; }
          obs_jac<P>(cam_entry(cam), X0, X1, X2, xy.x, xy.y, loss, fscale, f, JX, Jc);
          (void)f;
          double q00, q01, q02, q10, q11, q12;
          pt_factor_rows<COV>(JX, Li, q00, q01, q02, q10, q11, q12);
#pragma unroll
          for (int p = 0; p < P; ++p) {
            zs[p] = fma(Jc[p], q00, Jc[P + p] * q10);
            zs[P + p] = fma(Jc[p], q01, Jc[P + p] * q11);
            zs[2 * P + p] = fma(Jc[p], q02, Jc[P + p] * q12);
          }
          has = true;
        }
        // camera of row pos + 1: the next lane's, or for the last lane the one lane 0 has just prefetched
        const int nx = __shfl_sync(gmask, gl == 0 ? cam_n : cam, (gl + 1) % LANES, LANES);
        if (pos + 1 < e) next = nx;
        if (pieces_only) {  // the granule ownership below needs rows in slot order: store each piece as it is
          if (has) {
            double* z0 = Zt + (3 * (size_t)j) * LD + (size_t)cam * P;
#pragma unroll
            for (int a = 0; a < 3; ++a)
#pragma unroll
              for (int p = 0; p < P; p += (P == 6 ? 2 : 1)) {
                if constexpr (P == 6)  // cam*48 B and LD*8 B are 16-byte multiples
                  *reinterpret_cast<double2*>(z0 + a * LD + p) = make_double2(zs[a * P + p], zs[a * P + p + 1]);
                else z0[a * LD + p] = zs[a * P + p];
              }
          }
          continue;
        }
        // lanes with a piece, in camera order; the previous camera the point sees is the piece of the next lower such
        // lane, or of slot 0 for the lowest
        const unsigned bal = (__ballot_sync(gmask, has) >> (grp * LANES)) & LMASK;
        const unsigned below = bal & ((1u << gl) - 1u);
        const int prev = below ? 32 - __clz(below) : 0;  // slot of the previous piece
        int g0 = 0, ng = 0;
        if (has) {
          sg.cam[gl + 1] = cam;
          g0 = (cam * P) >> 3;
          const int g1 = (cam * P + P - 1) >> 3;
          ng = g1 - g0 + 1;
          if (next == cam + 1 && ((cam + 1) * P) >> 3 == g1) --ng;  // shared with the next piece: written with it
        }
        int off = ng;  // inclusive scan of the granule counts over the group
#pragma unroll
        for (int o = 1; o < LANES; o <<= 1) {
          const int t = __shfl_up_sync(gmask, off, o, LANES);
          if (gl >= o) off += t;
        }
        const int total = __shfl_sync(gmask, off, LANES - 1, LANES);
        for (int q = 0; q < ng; ++q) sg.list[off - ng + q] = ((g0 + q) << 12) | (prev << 6) | (gl + 1);
        __syncwarp(gmask);
        double* zrow = Zt + (3 * (size_t)j) * LD;
        for (int it = gl; it < total * 12; it += LANES) {  // (granule, row, 16-byte quarter)
          const int ent = sg.list[it / 12], a = (it >> 2) % 3, col0 = 8 * (ent >> 12) + 2 * (it & 3);
          const int sl = ent & 63, ps = (ent >> 6) & 63;
          const int oc = sg.cam[sl] * P, pc = sg.cam[ps] * P;
          double v[2];
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int col = col0 + u;
            if (col >= oc) v[u] = col < oc + P ? sg.z[sl][a][col - oc] : 0.0;
            else v[u] = pc == oc - P ? sg.z[ps][a][col - pc] : 0.0;
          }
          *reinterpret_cast<double2*>(zrow + a * LD + col0) = make_double2(v[0], v[1]);  // LD*8 B is a multiple of 64
        }
        __syncwarp(gmask);
        if (bal) {  // the round's last piece becomes slot 0 of the next
          const int last = 32 - __clz(bal);
          for (int i = gl; i < 3 * P; i += LANES) sg.z[0][i / P][i % P] = sg.z[last][i / P][i % P];
          if (gl == 0) sg.cam[0] = sg.cam[last];
        }
        __syncwarp(gmask);
      }
    }
  }
  gm = warp_max(gm);
  if (lane == 0) wmax[wid] = gm;
  __syncthreads();
  if (threadIdx.x == 0) {
    double m = 0.0;
    for (int w = 0; w < PT_WARPS; ++w) m = fmax(m, wmax[w]);
    if (m > 0.0) atomicMax(gmax_bits, (unsigned long long)__double_as_longlong(m));
  }
}

// ---------------------------------------------------------------------------------------------
// Point back-substitution, Jacobian-free:  Z_j^T dc = L^-1 sum_obs Jp^T (Jc dc_cam), so
//   dX_j = -L^-T (t_j + L^-1 u),  u = sum_obs Jp^T (Jc dc)
// recomputed from the observation list (24 B / observation) instead of streaming the dense factor.
// Per-CTA partial sums of the predicted reduction / step / x norms (fixed grid => deterministic).
// FIXP: a fixed point (pad slot of xp4 non-zero) is copied to the trial buffer as it is, flag included, and adds nothing
// to the three sums.
// ---------------------------------------------------------------------------------------------
template <int P, int LANES, bool CAMSM, bool FIXP = false>
__global__ void __launch_bounds__(PT_WARPS * 32, 2)
pt_backsub_kernel(const LmState* __restrict__ st, const int* __restrict__ pt_start, const int* __restrict__ pm_cam,
                  const double2* __restrict__ pm_xy, const int* __restrict__ pt_comp, int n_pts, int n_cams, int nP,
                  CPtr2 camtab2, Ptr2 xp2, const double* __restrict__ dc,
                  const double* __restrict__ Linv6, const double* __restrict__ tvec, const double* __restrict__ gp,
                  const double* __restrict__ Dp2, double* __restrict__ dp_out, double* __restrict__ bpart,
                  int bpart_stride) {
  extern __shared__ __align__(16) double bs_sm[];
  __shared__ double wsum[3][PT_WARPS];
  if (st->done) return;
  const int cur = st->cur;
  const double lam = st->lam;
  const int loss = st->loss;
  const double fscale = st->fscale;
  double* dcs = bs_sm;
  const double* __restrict__ gtab = camtab2.p[cur];
  const double* xp4 = xp2.p[cur];
  double* xp4_new = xp2.p[cur ^ 1];
  for (int i = threadIdx.x; i < nP; i += blockDim.x) dcs[i] = dc[i];
  constexpr int cstride = CAMSM ? CT_SMEM : CT_SIZE;
  double* cs = bs_sm + ((nP + 3) & ~3);
  if constexpr (CAMSM)
    for (int i = threadIdx.x; i < n_cams * CT_SIZE; i += blockDim.x) cs[(i / CT_SIZE) * CT_SMEM + i % CT_SIZE] = gtab[i];
  __syncthreads();
  auto cam_entry = [&](int c) -> const double* {
    if constexpr (CAMSM) return cs + (size_t)c * cstride;
    else return gtab + (size_t)c * cstride;
  };
  constexpr int GPW = 32 / LANES;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int gl = lane % LANES, grp = lane / LANES;
  double pred = 0.0, st2 = 0.0, x2 = 0.0;
  for (int j0 = (blockIdx.x * PT_WARPS + wid) * GPW; j0 < n_pts; j0 += gridDim.x * PT_WARPS * GPW) {
    const int j = j0 + grp;
    const bool valid = j < n_pts && !(pt_comp != nullptr && pt_comp[j] >= 0);
    int s = 0, e = 0;
    double X0 = 0.0, X1 = 0.0, X2 = 0.0, X3;
    if (valid) {
      s = pt_start[j]; e = pt_start[j + 1];
      ld256nc(xp4 + 4 * (size_t)j, X0, X1, X2, X3);
    }
    (void)X3;
    const bool fixed = FIXP && valid && X3 != 0.0;
    if (fixed) e = s;  // no observation to visit: the step is zero
    double u0 = 0.0, u1 = 0.0, u2 = 0.0;
    int cam_n = 0;
    double2 xy_n = make_double2(0.0, 0.0);
    if (s + gl < e) { cam_n = pm_cam[s + gl]; xy_n = pm_xy[s + gl]; }
    for (int pos = s + gl; pos < e; pos += LANES) {
      const int cam = cam_n;
      const double2 xy = xy_n;
      if (pos + LANES < e) { cam_n = pm_cam[pos + LANES]; xy_n = pm_xy[pos + LANES]; }
      double f[2], JX[6], Jc[2 * P];
      obs_jac<P>(cam_entry(cam), X0, X1, X2, xy.x, xy.y, loss, fscale, f, JX, Jc);
      const double* d = dcs + cam * P;
      double s0 = 0.0, s1 = 0.0;
#pragma unroll
      for (int p = 0; p < P; ++p) { s0 = fma(Jc[p], d[p], s0); s1 = fma(Jc[P + p], d[p], s1); }
      u0 = fma(JX[0], s0, fma(JX[3], s1, u0));
      u1 = fma(JX[1], s0, fma(JX[4], s1, u1));
      u2 = fma(JX[2], s0, fma(JX[5], s1, u2));
    }
    u0 = group_sum<LANES>(u0); u1 = group_sum<LANES>(u1); u2 = group_sum<LANES>(u2);
    if (fixed && gl == 0) {
      double* xn = xp4_new + 4 * (size_t)j;
      xn[0] = X0; xn[1] = X1; xn[2] = X2; xn[3] = X3;
      if (dp_out) { dp_out[3 * (size_t)j] = 0.0; dp_out[3 * (size_t)j + 1] = 0.0; dp_out[3 * (size_t)j + 2] = 0.0; }
    } else if (valid && gl == 0) {
      const double* Li = Linv6 + (size_t)j * 6;
      const double w0 = Li[0] * u0, w1 = Li[1] * u0 + Li[2] * u1, w2 = Li[3] * u0 + Li[4] * u1 + Li[5] * u2;
      const double v0 = tvec[3 * (size_t)j] + w0, v1 = tvec[3 * (size_t)j + 1] + w1, v2 = tvec[3 * (size_t)j + 2] + w2;
      const double d0 = -(Li[0] * v0 + Li[1] * v1 + Li[3] * v2);
      const double d1 = -(Li[2] * v1 + Li[4] * v2);
      const double d2 = -(Li[5] * v2);
      double* xn = xp4_new + 4 * (size_t)j;
      xn[0] = X0 + d0; xn[1] = X1 + d1; xn[2] = X2 + d2; xn[3] = 0.0;
      if (dp_out) { dp_out[3 * (size_t)j] = d0; dp_out[3 * (size_t)j + 1] = d1; dp_out[3 * (size_t)j + 2] = d2; }
      const double* D = Dp2 + 3 * (size_t)j;
      const double* g = gp + 3 * (size_t)j;
      const double e0 = D[0] > 0.0 ? D[0] : 1.0, e1 = D[1] > 0.0 ? D[1] : 1.0, e2 = D[2] > 0.0 ? D[2] : 1.0;
      pred += 0.5 * (d0 * (lam * e0 * d0 - g[0]) + d1 * (lam * e1 * d1 - g[1]) + d2 * (lam * e2 * d2 - g[2]));
      st2 += d0 * d0 + d1 * d1 + d2 * d2;
      x2 += X0 * X0 + X1 * X1 + X2 * X2;
    }
  }
  pred = warp_sum(pred); st2 = warp_sum(st2); x2 = warp_sum(x2);
  if (lane == 0) { wsum[0][wid] = pred; wsum[1][wid] = st2; wsum[2][wid] = x2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, b = 0, c = 0;
    for (int w = 0; w < PT_WARPS; ++w) { a += wsum[0][w]; b += wsum[1][w]; c += wsum[2][w]; }
    bpart[blockIdx.x] = a;
    bpart[bpart_stride + blockIdx.x] = b;
    bpart[2 * (size_t)bpart_stride + blockIdx.x] = c;
  }
}

// ---------------------------------------------------------------------------------------------
// After the (all-)reduce of [S | b | g_c | diag U | cost | per-rank point-gradient slots]: Marquardt scaling and
// damping of the reduced system, gradient norm, the start-of-iteration tests, block-Jacobi inverses.  One CTA.
// ---------------------------------------------------------------------------------------------
template <int P>
__device__ __forceinline__ void block_inverse_one(const double* __restrict__ S, int nP, int c, double* __restrict__ out) {
  double A[P][P], Li[P][P];
  for (int i = 0; i < P; ++i)
    for (int j = 0; j < P; ++j) A[i][j] = S[(size_t)(c * P + i) * nP + c * P + j];
  bool ok = true;
  for (int j = 0; j < P; ++j) {
    double d = A[j][j];
    for (int k = 0; k < j; ++k) d -= A[j][k] * A[j][k];
    if (!(d > 0.0)) { ok = false; d = 1.0; }
    d = sqrt(d);
    A[j][j] = d;
    for (int i = j + 1; i < P; ++i) {
      double s = A[i][j];
      for (int k = 0; k < j; ++k) s -= A[i][k] * A[j][k];
      A[i][j] = s / d;
    }
  }
  for (int j = 0; j < P; ++j) {
    Li[j][j] = 1.0 / A[j][j];
    for (int i = j + 1; i < P; ++i) {
      double s = 0.0;
      for (int k = j; k < i; ++k) s -= A[i][k] * Li[k][j];
      Li[i][j] = s / A[i][i];
    }
  }
  for (int i = 0; i < P; ++i)
    for (int j = 0; j < P; ++j) {
      double s = 0.0;
      if (ok) {
        for (int k = (i > j ? i : j); k < P; ++k) s += Li[k][i] * Li[k][j];
      } else {
        const double d = S[(size_t)(c * P + i) * nP + c * P + i];
        s = (i == j) ? (d > 0.0 ? 1.0 / d : 1.0) : 0.0;
      }
      out[i * P + j] = s;
    }
}

// HELD: the problem holds camera parameters fixed (DESIGN §4.12) or near a prior (§4.13).  The camera priors *cpp
// (cb_priors.cuh; a device pointer rather than a by-value parameter, which leaves the kernels without held parameters
// their own SASS; cpp->n = 0 with fixed parameters only) at the current cameras enter S, b, the g_c slot and the diag-U
// slot first.  Then fixc[0..n_fixc), the fixed camera parameters (internal slot indices), get unit rows and columns of S
// and zero entries of b before the damping, so every solver returns a zero step for them, while their diagonal prior
// information still reaches Dc2; their active bytes are clear, so the gradient norm, the step and the predicted
// reduction leave them out.
template <int P, bool WANT_MINV, bool HELD = false>
__device__ __forceinline__ void reduced_prep_body(LmState* __restrict__ st, int nP, int n_cams, int red_slots,
                                                  double* __restrict__ red, double* __restrict__ Dc2,
                                                  const unsigned char* __restrict__ active, double* __restrict__ Minv,
                                                  unsigned long long* __restrict__ gmax_bits, double* __restrict__ sc,
                                                  const int* __restrict__ fixc, int n_fixc, const CamPriors* __restrict__ cpp) {
  __shared__ double sh[32];
  const size_t nn = (size_t)nP * nP;
  const double lam = st->lam;
  if constexpr (HELD) {
    const CamPriors cp = *cpp;
    add_cam_priors<P>(red, nP, cp.xc.p[st->cur], cp);
    __syncthreads();
    for (int t = threadIdx.x; t < n_fixc * nP; t += blockDim.x) {
      const int f = fixc[t / nP], i = t % nP;
      const double v = i == f ? 1.0 : 0.0;
      red[(size_t)f * nP + i] = v;
      red[(size_t)i * nP + f] = v;
    }
    for (int t = threadIdx.x; t < n_fixc; t += blockDim.x) red[nn + fixc[t]] = 0.0;
    __syncthreads();
  }
  double gm = 0.0;
  for (int i = threadIdx.x; i < nP; i += blockDim.x) {
    double d = fmax(Dc2[i], red[nn + 2 * (size_t)nP + i]);  // running max; idempotent when the point is unchanged
    Dc2[i] = d;
    red[(size_t)i * nP + i] += lam * (d > 0.0 ? d : 1.0);
    if (active[i]) gm = fmax(gm, fabs(red[nn + nP + i]));
  }
  const size_t slot0 = nn + 3 * (size_t)nP + 1;
  for (int s = threadIdx.x; s < red_slots; s += blockDim.x) gm = fmax(gm, red[slot0 + s]);
  gm = warp_max(gm);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = gm;
  __syncthreads();
  if (threadIdx.x == 0) {
    double m = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m = fmax(m, sh[w]);
    sc[SC_GNORM_C] = m;
    const double cost = red[nn + 3 * (size_t)nP];
    sc[SC_COST] = cost;
    *gmax_bits = 0ull;  // consumed by the finalize kernel; the next point pass accumulates afresh
    st->epoch_big += 1;
    int done = 0;
    if (st->new_lin) {
      st->cost = cost;
      st->gnorm = m;
      if (st->njev == 1) {
        st->initial_cost = cost;
        if (!isfinite(cost)) { st->err = LM_ERR_NONFINITE_X0; done = 1; }
      }
      if (!done && m < st->gtol) { st->status = 1; done = 1; }
      if (!done) st->nit += 1;
    }
    if (!done && st->nfev >= st->max_nfev) { st->status = 0; done = 1; }
    if (done) st->done = 1;
  }
  __syncthreads();
  if constexpr (WANT_MINV)
    for (int c = threadIdx.x; c < n_cams; c += blockDim.x) block_inverse_one<P>(red, nP, c, Minv + (size_t)c * P * P);
}
template <int P, bool HELD = false>
__global__ void __launch_bounds__(256)
reduced_prep_kernel(LmState* __restrict__ st, int nP, int n_cams, int red_slots, double* __restrict__ red,
                    double* __restrict__ Dc2, const unsigned char* __restrict__ active, double* __restrict__ Minv,
                    unsigned long long* __restrict__ gmax_bits, double* __restrict__ sc, const int* __restrict__ fixc,
                    int n_fixc, const CamPriors* __restrict__ cp) {
  if (st->done) return;
  reduced_prep_body<P, true, HELD>(st, nP, n_cams, red_slots, red, Dc2, active, Minv, gmax_bits, sc, fixc, n_fixc, cp);
}

// ---------------------------------------------------------------------------------------------
// camera step: bounds clamp, effective step back into dc, predicted reduction (camera part), then the camera
// table of the trial point.  One CTA.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void cam_step_body(const LmState* __restrict__ st, int nP, int n_cams, int P, Ptr2 xc2,
                                              double* __restrict__ dc, const double* __restrict__ lo,
                                              const double* __restrict__ hi, const double* __restrict__ gc_total,
                                              const double* __restrict__ Dc2, const unsigned char* __restrict__ active,
                                              const int* __restrict__ cam_flags, const double* __restrict__ cam_const,
                                              Ptr2 camtab2, double* __restrict__ sc) {
  __shared__ double sh[3][32];
  const int cur = st->cur;
  const double lam = st->lam;
  const double* xc = xc2.p[cur];
  double* xc_new = xc2.p[cur ^ 1];
  double pred = 0.0, st2 = 0.0, x2 = 0.0;
  for (int i = threadIdx.x; i < nP; i += blockDim.x) {
    const double x = xc[i];
    double xn = x + dc[i];
    xn = fmin(fmax(xn, lo[i]), hi[i]);
    if (!active[i]) xn = x;
    const double de = xn - x;
    dc[i] = de;
    xc_new[i] = xn;
    if (active[i]) {
      const double d = Dc2[i] > 0.0 ? Dc2[i] : 1.0;
      pred += 0.5 * de * (lam * d * de - gc_total[i]);
      st2 += de * de;
      x2 += x * x;
    }
  }
  pred = warp_sum(pred); st2 = warp_sum(st2); x2 = warp_sum(x2);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { sh[0][wid] = pred; sh[1][wid] = st2; sh[2][wid] = x2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, b = 0, c = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { a += sh[0][w]; b += sh[1][w]; c += sh[2][w]; }
    sc[SC_PRED_C] = a; sc[SC_STEP2_C] = b; sc[SC_X2_C] = c;
  }
  for (int c = threadIdx.x; c < n_cams; c += blockDim.x)
    cam_prep_one(xc_new + (size_t)c * P, cam_const + (size_t)c * 9, cam_flags[c], camtab2.p[cur ^ 1] + (size_t)c * CT_SIZE);
}
__global__ void __launch_bounds__(256)
cam_step_kernel(const LmState* __restrict__ st, int nP, int n_cams, int P, Ptr2 xc2, double* __restrict__ dc,
                const double* __restrict__ lo, const double* __restrict__ hi, const double* __restrict__ gc_total,
                const double* __restrict__ Dc2, const unsigned char* __restrict__ active,
                const int* __restrict__ cam_flags, const double* __restrict__ cam_const, Ptr2 camtab2,
                double* __restrict__ sc) {
  if (st->done) return;
  cam_step_body(st, nP, n_cams, P, xc2, dc, lo, hi, gc_total, Dc2, active, cam_flags, cam_const, camtab2, sc);
}

// Small rigs (n_camera_params <= DIRECT_MAX_N): damping + head-of-iteration tests, the direct reduced solve and the camera
// step in ONE single-CTA kernel -- three launches and two kernel boundaries become one.
template <int P, bool HELD = false>
__global__ void __launch_bounds__(DIRECT_THREADS, 1)
small_rig_step_kernel(LmState* __restrict__ st, int nP, int n_cams, int red_slots, double* __restrict__ red,
                      double* __restrict__ Dc2, const unsigned char* __restrict__ active,
                      unsigned long long* __restrict__ gmax_bits, double* __restrict__ sc, Ptr2 xc2,
                      double* __restrict__ dc, const double* __restrict__ lo, const double* __restrict__ hi,
                      const int* __restrict__ cam_flags, const double* __restrict__ cam_const, Ptr2 camtab2,
                      const int* __restrict__ fixc, int n_fixc, const CamPriors* __restrict__ cp) {
  extern __shared__ __align__(16) double dsm[];
  if (st->done) return;
  reduced_prep_body<P, false, HELD>(st, nP, n_cams, red_slots, red, Dc2, active, nullptr, gmax_bits, sc, fixc, n_fixc,
                                    cp);
  __syncthreads();
  if (st->done) return;  // set by thread 0 before the barrier: gtol / max_nfev / non-finite start (uniform)
  const size_t nn = (size_t)nP * nP;
  dense_ldlt_body(dsm, red, red + nn, nP, dc, sc);
  __syncthreads();
  cam_step_body(st, nP, n_cams, P, xc2, dc, lo, hi, red + nn + nP, Dc2, active, cam_flags, cam_const, camtab2, sc);
}

// ---------------------------------------------------------------------------------------------
// The accept / reject decision of one trial (scipy trf.py:465-560 bookkeeping, Marquardt/Nielsen damping update).
// red2 = [cost_new, predicted reduction (points), |dX|^2 (points), |X|^2 (points)] summed over ranks.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void lm_decide(LmState* __restrict__ st, const double* __restrict__ sc,
                                          const double* __restrict__ red2, LmLogRow* __restrict__ log) {
  st->nfev += 1;
  st->pcg_total += (long long)sc[SC_PCG_ITS];
  const double cost = st->cost;
  const double cost_new = red2[0];
  const double pred = sc[SC_PRED_C] + red2[1];
  const double step2 = sc[SC_STEP2_C] + red2[2];
  const double x2 = sc[SC_X2_C] + red2[3];
  const bool pcg_bad = sc[SC_PCG_FLAG] != 0.0;
  const bool finite = isfinite(cost_new) && isfinite(pred) && !pcg_bad;
  const double actual = finite ? cost - cost_new : -1.0;
  const double ratio = (finite && pred > 0) ? actual / pred : -1.0;
  const double step_norm = sqrt(step2), x_norm = sqrt(x2);
  const bool ft = finite && actual < st->ftol * cost && ratio > 0.25;
  const bool xt = finite && step_norm < st->xtol * (st->xtol + x_norm);
  const int term = (ft && xt) ? 4 : ft ? 2 : xt ? 3 : 0;
  if (log != nullptr && st->n_log < st->log_cap) {
    LmLogRow& r = log[st->n_log];
    r.nit = (double)st->nit; r.nfev = (double)st->nfev; r.cost = cost; r.cost_new = cost_new; r.ratio = ratio;
    r.lam = st->lam; r.step = step_norm; r.gnorm = st->gnorm; r.pcg = sc[SC_PCG_ITS];
    st->n_log += 1;
  }
  double lam = st->lam;
  if (finite && actual > 0) {
    st->cur ^= 1;
    const double t = 2.0 * ratio - 1.0;
    lam = fmax(lam * fmax(1.0 / 3.0, 1.0 - t * t * t), 1e-15);
    st->nu = 2.0;
    st->cost = cost_new;
    st->new_lin = 1;
    st->bad_streak = 0;
    if (term) { st->status = term; st->done = 1; }
    else st->njev += 1;
  } else {
    lam = fmin(lam * st->nu, 1e12);
    st->nu *= 2.0;
    st->new_lin = 0;
    if (term) { st->status = term; st->done = 1; }
    if (!finite) {
      // every trial non-finite with the damping at its cap: nothing can change any more (scipy would raise or stop
      // on max_nfev = 100 n; stop now with status 0 instead of spinning for millions of evaluations)
      if (++st->bad_streak >= 6 && lam >= 1e12 && !st->done) { st->status = 0; st->err = LM_ERR_STUCK_NONFINITE; st->done = 1; }
    } else {
      st->bad_streak = 0;
    }
  }
  st->lam = lam;
}

// ---------------------------------------------------------------------------------------------
// Chunk partials of the camera pass -> per-camera packed U, g and the cost; block n_cams sums the point-step
// partials.  The last block to finish adds up the cost in fixed order and (MODE 1) takes the decision.
//   MODE 0: initial linearisation (writes slot cur, no decision)
//   MODE 1: trial point, single GPU: decision fused
//   MODE 2: trial point, several GPUs: red2 goes through the all-reduce, lm_decide_kernel follows
// ---------------------------------------------------------------------------------------------
template <int P>
__global__ void __launch_bounds__(64)
trial_reduce_kernel(LmState* __restrict__ st, int mode, int n_cams, const int* __restrict__ cam_chunk_start,
                    const double* __restrict__ partial, Ptr2 Upk2, Ptr2 gc2, Ptr2 costsum2,
                    double* __restrict__ cam_cost, int n_extra_cost, const double* __restrict__ bpart, int bpart_n,
                    int bpart_stride, double* __restrict__ red2, unsigned int* __restrict__ counter,
                    const double* __restrict__ sc, LmLogRow* __restrict__ log) {
  using RT = RowT<P>;
  __shared__ double sh[2];
  __shared__ int s_last;
  if (st->done) return;
  const int sel = (mode == 0) ? st->cur : (st->cur ^ 1);
  const int c = blockIdx.x, k = threadIdx.x;
  if (c < n_cams) {
    if (k < RT::NACC) {
      double v = 0.0;
      for (int ch = cam_chunk_start[c]; ch < cam_chunk_start[c + 1]; ++ch) v += partial[(size_t)ch * RT::NACC + k];
      if (k < RT::NU) Upk2.p[sel][(size_t)c * RT::NU + k] = v;
      else if (k < RT::NU + P) gc2.p[sel][(size_t)c * P + (k - RT::NU)] = v;
      else cam_cost[c] = v;
    }
  } else if (mode != 0) {
    // three deterministic sums of bpart_n values each
    for (int q = 0; q < 3; ++q) {
      const double* src = bpart + (size_t)q * bpart_stride;
      double v = 0.0;
      for (int i = k; i < bpart_n; i += 64) v += src[i];
      v = warp_sum(v);
      if ((k & 31) == 0) sh[k >> 5] = v;
      __syncthreads();
      if (k == 0) red2[1 + q] = sh[0] + sh[1];
      __syncthreads();
    }
  }
  __syncthreads();
  if (k == 0) {
    __threadfence();
    const unsigned prev = atomicAdd(counter, 1u);
    s_last = (prev == gridDim.x - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  double v = 0.0;
  for (int i = k; i < n_cams + n_extra_cost; i += 64) v += __ldcg(cam_cost + i);
  v = warp_sum(v);
  if ((k & 31) == 0) sh[k >> 5] = v;
  __syncthreads();
  if (k == 0) {
    const double cost = sh[0] + sh[1];
    costsum2.p[sel][0] = cost;
    *counter = 0u;
    if (mode != 0) {
      red2[0] = cost;
      if (mode == 1) {
        __threadfence();
        const double r2[4] = {cost, __ldcg(red2 + 1), __ldcg(red2 + 2), __ldcg(red2 + 3)};
        lm_decide(st, sc, r2, log);
      }
    }
  }
}

// Last node of the WHILE-loop body (device-loop mode): keep looping until the state machine says done.
__global__ void lm_loop_cond_kernel(const LmState* __restrict__ st, cudaGraphConditionalHandle h) {
  cudaGraphSetConditional(h, st->done ? 0u : 1u);
}

}  // namespace cb
