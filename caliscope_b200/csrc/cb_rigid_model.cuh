// Refinement of a rigid body's marker layout from tracked frames (cb_rigid_model_refine, DESIGN.md section 4.15): one
// Levenberg-Marquardt over the layout M (3K, K <= 32 markers) and every frame pose q_f = (r, t), X_w = R(r) M_k + t,
// with the frames eliminated (Schur form) and the gauge held by inner constraints on the start layout, then the
// layout's covariance.  oracle/rigid_model.py states the rule.
//
//   rmod_frame_kernel  one thread per frame (rows of one key): its body, marker mask, start pose and whether it is used
//   rmod_lm_kernel     one thread-block cluster per body: the whole loop on the device, as intr_lm_kernel
//   rmod_cov_kernel    one cluster per body: status 2 / 4, rmse and the covariance at the solution
//
// Warps take the body's used frames round-robin.  Per frame, lane l owns the frame's l-th marker and sums its rows'
// blocks (A_k = J_M^T J_M, W_k = J_M^T J_q, g_k = J_M^T r) in row order, and its share of the frame blocks
// (V = J_q^T J_q, g_f, cost), which a butterfly adds over the lanes; these 27 m + 28 doubles are the frame's slot of
// `gram`.  The frame's Schur contribution blockdiag(A_k) - Z Z^T, Z = W L^-T with V_lam = L L^T, goes to the warp's
// shared scratch; the CTA adds its warps' contributions to its partial S and b in warp order, and rank 0 adds the CTAs'
// partials in rank order over distributed shared memory.  Rank 0 forms N^T S_lam N (N: an orthonormal basis of the
// gauge constraints' null space, from the host), factors it with all its threads and solves.  No floating-point atomics:
// repeated calls are bit-identical.
#pragma once
#include <cooperative_groups.h>

#include "cb_intrinsics.cuh"
#include "cb_rigid.cuh"

namespace cb {

constexpr int RMOD_THREADS = 256, RMOD_WARPS = RMOD_THREADS / 32, RMOD_KMAX = 32, RMOD_NMAX = 3 * RMOD_KMAX;
constexpr int RMOD_SP = RMOD_NMAX * (RMOD_NMAX + 1) / 2;  // packed S of the largest body
constexpr int RM_OK = 0, RM_UNUSED = 1, RM_NOT_PD = 2, RM_MAX_ITER = 3, RM_BEHIND = 4;
constexpr int RMOD_FRAME = 28, RMOD_MARK = 27;  // gram doubles per frame and per marker of the frame

__device__ __forceinline__ int rmod_pk(int i, int j, int n) {  // packed upper index, i <= j
  return i * n - i * (i - 1) / 2 + (j - i);
}

// Per frame f (rows start[f] .. start[f+1] of rows): fbody (the body of its first row; bad[0] counts frames whose rows
// span two bodies), fmask (its markers, bit k = marker body_start[b] + k), fpose (the start pose of its key, NaN when
// none) and fused (a finite start pose, >= 4 rows, >= 3 markers).
__global__ void rmod_frame_kernel(const int* __restrict__ start, const int* __restrict__ rows,
                                  const int* __restrict__ obs_pt, const long long* __restrict__ obs_key,
                                  const int* __restrict__ body_start, int n_bodies, const long long* __restrict__ skey,
                                  const double* __restrict__ spose, int n_start, int n_frames, int* __restrict__ fbody,
                                  unsigned* __restrict__ fmask, int* __restrict__ fused, double* __restrict__ fpose,
                                  int* __restrict__ bad) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_frames) return;
  const int b0 = start[f], e0 = start[f + 1];
  auto body_of = [&](int pt) {
    int lo = 0, hi = n_bodies;  // last b with body_start[b] <= pt
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (body_start[mid] <= pt) lo = mid;
      else hi = mid;
    }
    return lo;
  };
  const int b = body_of(obs_pt[rows[b0]]);
  unsigned mask = 0;
  bool span = false;
  for (int i = b0; i < e0; ++i) {
    const int pt = obs_pt[rows[i]];
    span = span || pt < body_start[b] || pt >= body_start[b + 1];
    if (!span) mask |= 1u << (pt - body_start[b]);
  }
  if (span) atomicAdd(bad, 1);
  const long long key = obs_key[rows[b0]];
  int lo = 0, hi = n_start;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (skey[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  const bool has = lo < n_start && skey[lo] == key;
  bool fin = has;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const double v = has ? spose[6 * (size_t)lo + k] : res_nan();
    fin = fin && isfinite(v);
    fpose[6 * (size_t)f + k] = v;
  }
  fbody[f] = b;
  fmask[f] = mask;
  fused[f] = fin && e0 - b0 >= 4 && __popc(mask) >= 3 ? 1 : 0;
}

struct RmodArgs {
  const double* camtab;
  int stride;              // camera table stride (CT_SIZE)
  const int* start;        // frame f's rows: rows[start[f] .. start[f+1])
  const int* rows;
  const int* obs_cam;
  const int* obs_pt;
  const double* obs_px;
  const int* bodies;       // the bodies to solve, one cluster each
  const int* body_start;   // model range of each body
  const int* uf_start;     // used frames of body b: uf_list[uf_start[b] .. uf_start[b+1]) (frame indices, key order)
  const int* uf_list;
  const long long* goff;   // gram offset of each used-frame slot (position in uf_list)
  const unsigned* fmask;
  const double* N;         // per body, (3K x (3K - 6)) row-major at noff[b]
  const long long* noff;
  double* model;           // (n_model, 3), in / out
  double* pose;            // (n_frames, 6), in / out
  double* gram;
  double* trial;           // per used-frame slot: q + dq (6)
  double* tot;             // per body at toff[b]: scratch (2 x 3K (3K - 6)), then S (packed), b, diag H_MM, cost
  const long long* toff;
  int* status;
  int* iters;
  double* fcost;           // per frame, the cost at the solution
  double* cov;             // per body (3K)^2 at coff[b], nullable
  double* pmat;            // per body N (N^T S N)^-1 N^T at coff[b], nullable (the camera term's)
  const long long* coff;
  double s2;
  int max_iter;
  double xtol;
};

// The shared memory of the two cluster kernels (dynamic): the CTA's partial S, b, diag H_MM and cost, the layout and
// its step, the warps' scratch, and rank 0's reduced matrix
struct RmodWarp {
  double Z[RMOD_NMAX * 6];
  double A[RMOD_KMAX * 6];
  double bc[RMOD_NMAX];
  double cost, dq2, q2, behind;
  int loc[RMOD_KMAX];  // marker of the body -> its row block in Z (-1: not in the frame)
};
struct RmodShared {
  double S[RMOD_SP];
  double b[RMOD_NMAX], hd[RMOD_NMAX], M[RMOD_NMAX], dM[RMOD_NMAX];
  double R[(RMOD_NMAX - 6) * (RMOD_NMAX - 6)];
  double bc[RMOD_NMAX + 8];  // rank 0's broadcast: dM, flags
  double part[8];
  RmodWarp w[RMOD_WARPS];
};
constexpr size_t RMOD_SMEM = sizeof(RmodShared);

// One row's pixel residual rr (2), J_q (2 x 6, rig_jq) and J_M (2 x 3) = J_X R at body pose B, t and marker Mk;
// out of line so the accumulating loops keep their registers
__device__ __noinline__ void rmod_row(const RmodArgs& A, const double* B, const double* t, const double* Mk, int r,
                                      double* rr, double* J, double* JM) {
  const double* cam = A.camtab + (size_t)A.stride * A.obs_cam[r];
  const double2 px = reinterpret_cast<const double2*>(A.obs_px)[r];
  double X[3], fr[2], JX[6];
  rig_world(B, t, Mk, X);
  obs_res_jx(cam, X[0], X[1], X[2], px.x, px.y, 0, 1.0, fr, JX);
  const double fx0 = cam[CT_FX0];
  rr[0] = fr[0] * fx0;
  rr[1] = fr[1] * fx0;
  rig_jq(B, Mk, JX, fx0, J);
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int c = 0; c < 3; ++c)
      JM[3 * s + c] = (JX[3 * s] * B[CT_R + c] + JX[3 * s + 1] * B[CT_R + 3 + c] + JX[3 * s + 2] * B[CT_R + 6 + c]) * fx0;
}

// The frame's gram slot at layout M (shared) and pose q, one warp: lane l owns the frame's l-th marker and sums, in
// row order, first its marker blocks, then its share of the frame blocks (added over the lanes by a butterfly)
__device__ __noinline__ void rmod_gram(const RmodArgs& A, int f, int lo, unsigned mask, const double* M,
                                       const double* q, double* g, int lane) {
  double B[CT_JR + 9];
  cam_prep_rot(q[0], q[1], q[2], B);
  const int m = __popc(mask);
  int kk = -1;  // lane's marker (body index)
  {
    unsigned mm = mask;
    for (int l = 0; l < lane && mm; ++l) mm &= mm - 1;
    if (lane < m) kk = __ffs(mm) - 1;
  }
  const double* Mk = M + 3 * (kk < 0 ? 0 : kk);
  if (kk >= 0) {
    double a[6] = {}, w[18] = {}, gm[3] = {};
    for (int i = A.start[f]; i < A.start[f + 1]; ++i) {
      const int r = A.rows[i];
      if (A.obs_pt[r] - lo != kk) continue;
      double rr[2], J[12], JM[6];
      rmod_row(A, B, q + 3, Mk, r, rr, J, JM);
#pragma unroll
      for (int x = 0; x < 3; ++x) {
#pragma unroll
        for (int y = x; y < 3; ++y) a[ut<3>(x, y)] = fma(JM[x], JM[y], fma(JM[3 + x], JM[3 + y], a[ut<3>(x, y)]));
#pragma unroll
        for (int y = 0; y < 6; ++y) w[6 * x + y] = fma(JM[x], J[y], fma(JM[3 + x], J[6 + y], w[6 * x + y]));
        gm[x] = fma(JM[x], rr[0], fma(JM[3 + x], rr[1], gm[x]));
      }
    }
    double* gk = g + RMOD_FRAME + RMOD_MARK * lane;
#pragma unroll
    for (int x = 0; x < 6; ++x) gk[x] = a[x];
#pragma unroll
    for (int x = 0; x < 18; ++x) gk[6 + x] = w[x];
#pragma unroll
    for (int x = 0; x < 3; ++x) gk[24 + x] = gm[x];
  }
  double v[21] = {}, gf[6] = {}, cost = 0.0;
  if (kk >= 0) {
    for (int i = A.start[f]; i < A.start[f + 1]; ++i) {
      const int r = A.rows[i];
      if (A.obs_pt[r] - lo != kk) continue;
      double rr[2], J[12], JM[6];
      rmod_row(A, B, q + 3, Mk, r, rr, J, JM);
#pragma unroll
      for (int x = 0; x < 6; ++x) {
#pragma unroll
        for (int y = x; y < 6; ++y) v[ut<6>(x, y)] = fma(J[x], J[y], fma(J[6 + x], J[6 + y], v[ut<6>(x, y)]));
        gf[x] = fma(J[x], rr[0], fma(J[6 + x], rr[1], gf[x]));
      }
      cost = fma(rr[0], rr[0], fma(rr[1], rr[1], cost));
    }
  }
#pragma unroll
  for (int x = 0; x < 21; ++x) v[x] = warp_sum(v[x]);
#pragma unroll
  for (int x = 0; x < 6; ++x) gf[x] = warp_sum(gf[x]);
  cost = warp_sum(cost);
  if (lane == 0) {
#pragma unroll
    for (int x = 0; x < 21; ++x) g[x] = v[x];
#pragma unroll
    for (int x = 0; x < 6; ++x) g[21 + x] = gf[x];
    g[27] = cost;
  }
  __syncwarp();
}

// v = L^-1 v (the forward half of res_chol_solve<6>)
__device__ __forceinline__ void rmod_fwd6(const double L[6][6], double* v) {
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    double a = v[i];
#pragma unroll
    for (int k = 0; k < i; ++k) a -= L[i][k] * v[k];
    v[i] = a / L[i][i];
  }
}

// Cholesky of the frame block V + lam diag V from the gram slot
__device__ __forceinline__ bool rmod_chol_v(const double* g, double lam, double L[6][6]) {
  double h[21];
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = i; j < 6; ++j) h[ut<6>(i, j)] = g[ut<6>(i, j)] * (i == j ? 1.0 + lam : 1.0);
  return res_chol<6>(h, 0.0, L);
}

// The frame's Schur contribution at lam into the warp's scratch: Z rows of the lane's marker, A, bc = g_k - Z_k y,
// loc, cost (NaN in Z when V_lam is not positive definite)
__device__ __forceinline__ void rmod_schur(const double* g, unsigned mask, int K, double lam, RmodWarp& W, int lane) {
  double L[6][6];
  const bool ok = rmod_chol_v(g, lam, L);
  double y[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) y[k] = g[21 + k];
  rmod_fwd6(L, y);
  const int m = __popc(mask);
  if (lane < K) W.loc[lane] = ((mask >> lane) & 1) ? __popc(mask & ((1u << lane) - 1)) : -1;
  if (lane < m) {
    const double* gk = g + RMOD_FRAME + RMOD_MARK * lane;
#pragma unroll
    for (int x = 0; x < 6; ++x) W.A[6 * lane + x] = gk[x];
#pragma unroll
    for (int x = 0; x < 3; ++x) {
      double z[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) z[k] = gk[6 + 6 * x + k];
      rmod_fwd6(L, z);
      double s = gk[24 + x];
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        W.Z[6 * (3 * lane + x) + k] = ok ? z[k] : res_nan();
        s -= z[k] * y[k];
      }
      W.bc[3 * lane + x] = s;
    }
  }
  if (lane == 0) W.cost = g[27];
  __syncwarp();
}

// Adds the warps' scratch (warps with `active` set) to the CTA's partials in warp order; every thread of the CTA
__device__ __forceinline__ void rmod_accumulate(RmodShared& sh, int K, const int* active) {
  const int n3 = 3 * K, tid = threadIdx.x;
  for (int e = tid; e < n3 * n3; e += RMOD_THREADS) {
    const int i = e / n3, j = e % n3;
    if (j < i) continue;
    const int ki = i / 3, kj = j / 3, ai = i % 3, aj = j % 3;
    double s = sh.S[rmod_pk(i, j, n3)];
    for (int w = 0; w < RMOD_WARPS; ++w) {
      if (!active[w]) continue;
      const int li = sh.w[w].loc[ki], lj = sh.w[w].loc[kj];
      if (li < 0 || lj < 0) continue;
      const double* zi = sh.w[w].Z + 6 * (3 * li + ai);
      const double* zj = sh.w[w].Z + 6 * (3 * lj + aj);
      double v = ki == kj ? sh.w[w].A[6 * li + ut<3>(ai, aj)] : 0.0;
#pragma unroll
      for (int k = 0; k < 6; ++k) v -= zi[k] * zj[k];
      s += v;
    }
    sh.S[rmod_pk(i, j, n3)] = s;
  }
  if (tid < n3) {
    const int k = tid / 3, a = tid % 3;
    double sb = sh.b[tid], sd = sh.hd[tid];
    for (int w = 0; w < RMOD_WARPS; ++w) {
      if (!active[w] || sh.w[w].loc[k] < 0) continue;
      const int l = sh.w[w].loc[k];
      sb += sh.w[w].bc[3 * l + a];
      sd += sh.w[w].A[6 * l + ut<3>(a, a)];
    }
    sh.b[tid] = sb;
    sh.hd[tid] = sd;
  }
  if (tid == RMOD_THREADS - 1) {
    double c = sh.part[0];
    for (int w = 0; w < RMOD_WARPS; ++w)
      if (active[w]) c += sh.w[w].cost;
    sh.part[0] = c;
  }
}

// One pass over the body's used frames at lam (relin: the gram slots first, at the current layout and poses), the
// CTAs' partials added in rank order into tot (S packed, b, diag H_MM, cost) by rank 0.  Every thread of the cluster.
__device__ __noinline__ void rmod_pass(cg::cluster_group& cl, RmodShared& sh, const RmodArgs& A, int bi, int K, int lo, double lam,
                          bool relin, double* tot) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rank = (int)cl.block_rank(), cs = (int)cl.num_blocks();
  const int n3 = 3 * K, np = n3 * (n3 + 1) / 2;
  const int f0 = A.uf_start[bi], nf = A.uf_start[bi + 1] - f0, nw = cs * RMOD_WARPS;
  for (int e = tid; e < np; e += RMOD_THREADS) sh.S[e] = 0.0;
  if (tid < n3) sh.b[tid] = sh.hd[tid] = 0.0;
  if (tid == 0) sh.part[0] = 0.0;
  __shared__ int active[RMOD_WARPS];
  const int rounds = (nf + nw - 1) / nw;
  for (int rd = 0; rd < rounds; ++rd) {
    const int j = rd * nw + rank * RMOD_WARPS + warp;
    if (lane == 0) active[warp] = j < nf;
    if (j < nf) {
      const int f = A.uf_list[f0 + j];
      double* g = A.gram + A.goff[f0 + j];
      if (relin) rmod_gram(A, f, lo, A.fmask[f], sh.M, A.pose + 6 * (size_t)f, g, lane);
      rmod_schur(g, A.fmask[f], K, lam, sh.w[warp], lane);
    }
    __syncthreads();
    rmod_accumulate(sh, K, active);
    __syncthreads();
  }
  __threadfence();
  cl.sync();
  if (rank == 0) {
    double* ts = tot;
    for (int e = tid; e < np + 2 * n3 + 1; e += RMOD_THREADS) {
      double s = 0.0;
      for (int r = 0; r < cs; ++r) {
        const RmodShared* o = cl.map_shared_rank(&sh, r);
        s += e < np ? o->S[e] : e < np + n3 ? o->b[e - np] : e < np + 2 * n3 ? o->hd[e - np - n3] : o->part[0];
      }
      ts[e] = s;
    }
  }
  __threadfence();
  cl.sync();
}

// Rank 0, every thread: R = N^T (S + lam diag H_MM) N into sh.R and its Cholesky factor in place (scaled: of the
// Jacobi-scaled R, whose scales stay in sh.dM[0 .. nr)); pivots must exceed thr.  T (3K x nr) is global scratch.
__device__ __noinline__ bool rmod_factor(RmodShared& sh, const double* tot, double* T, const double* N, int K, double lam,
                            bool scaled, double thr) {
  const int n3 = 3 * K, nr = n3 - 6, np = n3 * (n3 + 1) / 2, tid = threadIdx.x;
  const double* S = tot;
  const double* hd = tot + np + n3;
  for (int e = tid; e < n3 * nr; e += RMOD_THREADS) {
    const int i = e / nr, a = e % nr;
    double s = 0.0;
    for (int j = 0; j < n3; ++j)
      s = fma(S[i <= j ? rmod_pk(i, j, n3) : rmod_pk(j, i, n3)] + (i == j ? lam * hd[i] : 0.0), N[(size_t)j * nr + a], s);
    T[e] = s;
  }
  __syncthreads();
  for (int e = tid; e < nr * nr; e += RMOD_THREADS) {
    const int a = e / nr, c = e % nr;
    if (c < a) continue;
    double s = 0.0;
    for (int i = 0; i < n3; ++i) s = fma(N[(size_t)i * nr + a], T[(size_t)i * nr + c], s);
    sh.R[a * nr + c] = sh.R[c * nr + a] = s;
  }
  __syncthreads();
  if (scaled) {
    if (tid < nr) sh.dM[tid] = 1.0 / sqrt(sh.R[tid * nr + tid]);
    __syncthreads();
    for (int e = tid; e < nr * nr; e += RMOD_THREADS) sh.R[e] *= sh.dM[e / nr] * sh.dM[e % nr];
  }
  __shared__ int ok;
  if (tid == 0) ok = 1;
  for (int j = 0; j < nr; ++j) {
    __syncthreads();
    if (tid == 0) {
      const double d = sh.R[j * nr + j];
      if (!(d > thr)) ok = 0;
      sh.R[j * nr + j] = sqrt(d);
    }
    __syncthreads();
    for (int i = j + 1 + tid; i < nr; i += RMOD_THREADS) sh.R[i * nr + j] /= sh.R[j * nr + j];
    __syncthreads();
    const int w = nr - j - 1;
    for (int e = tid; e < w * w; e += RMOD_THREADS) {
      const int i = j + 1 + e / w, k = j + 1 + e % w;
      if (k <= i) sh.R[i * nr + k] -= sh.R[i * nr + j] * sh.R[k * nr + j];
    }
  }
  __syncthreads();
  return ok != 0;
}

// Rank 0, warp 0: x = R^-1 x (forward and back substitution on sh.R's factor), lane-parallel dot products
__device__ __forceinline__ void rmod_solve(const RmodShared& sh, int nr, double* x, int lane) {
  for (int i = 0; i < nr; ++i) {
    double s = 0.0;
    for (int k = lane; k < i; k += 32) s += sh.R[i * nr + k] * x[k];
    s = warp_sum(s);
    if (lane == 0) x[i] = (x[i] - s) / sh.R[i * nr + i];
    __syncwarp();
  }
  for (int i = nr - 1; i >= 0; --i) {
    double s = 0.0;
    for (int k = i + 1 + lane; k < nr; k += 32) s += sh.R[k * nr + i] * x[k];
    s = warp_sum(s);
    if (lane == 0) x[i] = (x[i] - s) / sh.R[i * nr + i];
    __syncwarp();
  }
}

// Frame f (used-frame slot j) at damping lam, one warp: its step by back-substitution, the trial pose q + dq into
// trial[j] and the trial cost at M + dM over its rows (ct), |dq|^2 and |q|^2
__device__ __noinline__ void rmod_trial(const RmodArgs& A, const RmodShared& sh, int f, int slot, int lo, double lam,
                                        int lane, double& ct_out, double& dq2_out, double& q2_out) {
    const unsigned mask = A.fmask[f];
    const double* g = A.gram + A.goff[slot];
    const double* qv = A.pose + 6 * (size_t)f;
    double h[6] = {0, 0, 0, 0, 0, 0};  // W^T dM over the frame's markers
    if (lane < __popc(mask)) {
      unsigned mm = mask;
      for (int l = 0; l < lane; ++l) mm &= mm - 1;
      const int kk = __ffs(mm) - 1;
      const double* gk = g + RMOD_FRAME + RMOD_MARK * lane;
#pragma unroll
      for (int y = 0; y < 6; ++y)
#pragma unroll
        for (int x = 0; x < 3; ++x) h[y] = fma(gk[6 + 6 * x + y], sh.dM[3 * kk + x], h[y]);
    }
    double L[6][6], dq[6], qt[6];
#pragma unroll
    for (int y = 0; y < 6; ++y) dq[y] = g[21 + y] + warp_sum(h[y]);
    rmod_chol_v(g, lam, L);
    res_chol_solve<6>(L, dq);
    double dq2 = 0.0, q2 = 0.0;
#pragma unroll
    for (int y = 0; y < 6; ++y) {
      dq[y] = -dq[y];
      qt[y] = qv[y] + dq[y];
      dq2 += dq[y] * dq[y];
      q2 += qv[y] * qv[y];
    }
    double B[CT_JR + 9];
    cam_prep_rot(qt[0], qt[1], qt[2], B);
    double ct = 0.0;
    for (int i = A.start[f] + lane; i < A.start[f + 1]; i += 32) {
      const int r = A.rows[i];
      const int k = A.obs_pt[r] - lo;
      const double Mk[3] = {sh.M[3 * k] + sh.dM[3 * k], sh.M[3 * k + 1] + sh.dM[3 * k + 1],
                            sh.M[3 * k + 2] + sh.dM[3 * k + 2]};
      double rr[2], J[12], JM[6];
      rmod_row(A, B, qt + 3, Mk, r, rr, J, JM);
      ct = fma(rr[0], rr[0], fma(rr[1], rr[1], ct));
    }
    ct = warp_sum(ct);
    double* tr = A.trial + 6 * (size_t)slot;
    if (lane < 6) tr[lane] = qt[lane];
  __syncwarp();
  ct_out = ct;
  dq2_out = dq2;
  q2_out = q2;
}

__device__ __forceinline__ void rmod_setup(const RmodArgs& A, cg::cluster_group& cl, int& bi, int& K, int& lo,
                                           const double*& N, double*& tot, double*& T) {
  bi = A.bodies[blockIdx.x / cl.num_blocks()];
  lo = A.body_start[bi];
  K = A.body_start[bi + 1] - lo;
  N = A.N + A.noff[bi];
  T = A.tot + A.toff[bi];
  tot = T + 2 * (size_t)(3 * K) * (3 * K - 6);
}

// One cluster per body: Levenberg-Marquardt (DESIGN.md section 4.15, intr_lm_kernel's acceptance and stopping) from
// the start layout and poses; status 2 when N^T S N fails the scaled test at the start.  Writes model, pose, status,
// iterations.
__global__ void __launch_bounds__(RMOD_THREADS)
rmod_lm_kernel(RmodArgs A) {
  cg::cluster_group cl = cg::this_cluster();
  extern __shared__ __align__(16) unsigned char rmod_smem[];
  RmodShared& sh = *reinterpret_cast<RmodShared*>(rmod_smem);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rank = (int)cl.block_rank(), cs = (int)cl.num_blocks();
  int bi, K, lo;
  const double* N;
  double *tot, *T;
  rmod_setup(A, cl, bi, K, lo, N, tot, T);
  const int n3 = 3 * K, nr = n3 - 6, np = n3 * (n3 + 1) / 2;
  const int f0 = A.uf_start[bi], nf = A.uf_start[bi + 1] - f0;
  const int gw = rank * RMOD_WARPS + warp, nw = cs * RMOD_WARPS;
  if (tid < n3) sh.M[tid] = A.model[3 * (size_t)lo + tid];
  __syncthreads();
  const double* bc0 = cl.map_shared_rank(sh.bc, 0);
  // the start: N^T S N at lambda = 0
  rmod_pass(cl, sh, A, bi, K, lo, 0.0, true, tot);
  if (rank == 0) {
    const bool ok = rmod_factor(sh, tot, T, N, K, 0.0, true, TRI_PD_RTOL);
    if (tid == 0) sh.bc[n3] = ok ? 1.0 : 0.0;
  }
  __threadfence();
  cl.sync();
  if (bc0[n3] == 0.0) {
    if (rank == 0 && tid == 0) {
      A.status[bi] = RM_NOT_PD;
      A.iters[bi] = 0;
    }
    cl.sync();
    return;
  }
  double lam = TRI_LAMBDA0, cost = 0.0;  // rank 0 thread 0's cost
  int it = 0, st = RM_OK;
  bool relin = false;
  while (true) {
    rmod_pass(cl, sh, A, bi, K, lo, lam, relin, tot);
    if (rank == 0) {
      const bool ok = rmod_factor(sh, tot, T, N, K, lam, false, 0.0);
      double* x = sh.bc;  // x = -N^T b, then N x
      if (tid < nr) {
        double s = 0.0;
        for (int i = 0; i < n3; ++i) s = fma(N[(size_t)i * nr + tid], tot[np + i], s);
        sh.dM[tid] = -s;
      }
      __syncthreads();
      if (ok && warp == 0) rmod_solve(sh, nr, sh.dM, lane);
      __syncthreads();
      if (tid < n3) {
        double s = 0.0;
        for (int a = 0; a < nr; ++a) s = fma(N[(size_t)tid * nr + a], sh.dM[a], s);
        x[tid] = ok ? s : 0.0;
      }
      if (tid == 0) {
        cost = tot[np + 2 * n3];
        x[n3] = ok ? 1.0 : 0.0;
        x[n3 + 1] = 0.0;
        if (!ok) {  // a damped block not positive definite: a rejected step without the stopping test
          ++it;
          if (it == A.max_iter) { st = RM_MAX_ITER; x[n3 + 1] = 1.0; }
        }
      }
    }
    __threadfence();
    cl.sync();
    if (tid < n3) sh.dM[tid] = bc0[tid];
    const bool step_ok = bc0[n3] != 0.0, stop = bc0[n3 + 1] != 0.0;
    __syncthreads();
    if (!step_ok) {
      lam *= 10.0;
      relin = false;
      cl.sync();  // every CTA has read the broadcast before rank 0 writes it again
      if (stop) break;
      continue;
    }
    // back-substitution, trial poses and the trial cost at M + dM
    double wsum[3] = {0.0, 0.0, 0.0};  // lane 0: trial cost, |dq|^2, |q|^2 over the warp's frames, in order
    for (int j = gw; j < nf; j += nw) {
      double ct, dq2, q2;
      rmod_trial(A, sh, A.uf_list[f0 + j], f0 + j, lo, lam, lane, ct, dq2, q2);
      wsum[0] += ct;
      wsum[1] += dq2;
      wsum[2] += q2;
      __syncwarp();
    }
    if (lane == 0) {
      sh.w[warp].cost = wsum[0];
      sh.w[warp].dq2 = wsum[1];
      sh.w[warp].q2 = wsum[2];
    }
    __syncthreads();
    if (tid < 3) {
      double s = 0.0;
      for (int w = 0; w < RMOD_WARPS; ++w) s += tid == 0 ? sh.w[w].cost : tid == 1 ? sh.w[w].dq2 : sh.w[w].q2;
      sh.part[1 + tid] = s;
    }
    __threadfence();
    cl.sync();
    if (rank == 0 && tid == 0) {
      double tc = 0.0, dn = 0.0, xn = 0.0;
      for (int r = 0; r < cs; ++r) {
        const double* p = cl.map_shared_rank(sh.part, r);
        tc += p[1];
        dn += p[2];
        xn += p[3];
      }
      ++it;
      for (int i = 0; i < n3; ++i) {
        dn += sh.dM[i] * sh.dM[i];
        xn += sh.M[i] * sh.M[i];
      }
      dn = sqrt(dn);
      xn = sqrt(xn);
      const bool lower = tc < cost;
      bool done = dn <= A.xtol * (xn + A.xtol);
      if (!done && it == A.max_iter) { st = RM_MAX_ITER; done = true; }
      sh.bc[n3 + 2] = lower ? 1.0 : 0.0;
      sh.bc[n3 + 3] = done ? 1.0 : 0.0;
    }
    __threadfence();
    cl.sync();
    const bool lower = bc0[n3 + 2] != 0.0, done = bc0[n3 + 3] != 0.0;
    lam = lower ? lam * 0.1 : lam * 10.0;
    if (lower) {
      if (tid < n3) sh.M[tid] += sh.dM[tid];
      for (int j = gw; j < nf; j += nw)
        if (lane < 6) A.pose[6 * (size_t)A.uf_list[f0 + j] + lane] = A.trial[6 * (size_t)(f0 + j) + lane];
    }
    relin = lower;
    __threadfence();
    cl.sync();  // every CTA has read rank 0's broadcast and partials before they are written again
    if (done) break;
  }
  if (rank == 0 && tid < n3) A.model[3 * (size_t)lo + tid] = sh.M[tid];
  if (rank == 0 && tid == 0) {
    A.status[bi] = st;
    A.iters[bi] = it;
  }
  cl.sync();
}

// Rank 0, every thread, after rmod_factor's scaled factor of N^T S N: cov = s2 P, P = N (N^T S N)^-1 N^T (and P itself
// into pmat for the camera term)
__device__ __noinline__ void rmod_cov_out(const RmodArgs& A, const RmodShared& sh, double* T, const double* N, int K,
                                          int bi) {
  const int n3 = 3 * K, nr = n3 - 6, tid = threadIdx.x;
      // (R~)^-1 column by column into T's first nr rows, then R^-1 = D R~^-1 D, U = N R^-1 and cov = s2 U N^T
  double* Ri = T;
  double* U = T + (size_t)nr * nr;
  for (int c = tid; c < nr; c += RMOD_THREADS) {
    double* x = Ri + (size_t)c * nr;  // column c (R^-1 is symmetric: row c)
    for (int i = 0; i < nr; ++i) {
      double s = i == c ? 1.0 : 0.0;
      for (int k = 0; k < i; ++k) s -= sh.R[i * nr + k] * x[k];
      x[i] = s / sh.R[i * nr + i];
    }
    for (int i = nr - 1; i >= 0; --i) {
      double s = x[i];
      for (int k = i + 1; k < nr; ++k) s -= sh.R[k * nr + i] * x[k];
      x[i] = s / sh.R[i * nr + i];
    }
  }
  __syncthreads();
  for (int e = tid; e < n3 * nr; e += RMOD_THREADS) {
    const int i = e / nr, a = e % nr;
    double s = 0.0;
    for (int c = 0; c < nr; ++c) s = fma(N[(size_t)i * nr + c], Ri[(size_t)c * nr + a] * sh.dM[c] * sh.dM[a], s);
    U[e] = s;
  }
  __syncthreads();
  double* cov = A.cov + A.coff[bi];
  for (int e = tid; e < n3 * n3; e += RMOD_THREADS) {
    const int i = e / n3, k = e % n3;
    if (k < i) continue;
    double s1 = 0.0, s2 = 0.0;
    for (int a = 0; a < nr; ++a) {
      s1 = fma(U[(size_t)i * nr + a], N[(size_t)k * nr + a], s1);
      s2 = fma(U[(size_t)k * nr + a], N[(size_t)i * nr + a], s2);
    }
    const double v = 0.5 * (s1 + s2);
    cov[(size_t)i * n3 + k] = cov[(size_t)k * n3 + i] = A.s2 * v;
    if (A.pmat) A.pmat[A.coff[bi] + (size_t)i * n3 + k] = A.pmat[A.coff[bi] + (size_t)k * n3 + i] = v;
  }
}

// One cluster per body of status 0 or 3 after rmod_lm_kernel: the gram slots at the solution, status 2 when N^T S N
// fails the scaled test, status 4 when a row is behind its camera, each frame's cost, and cov = s2 N (N^T S N)^-1 N^T.
__global__ void __launch_bounds__(RMOD_THREADS)
rmod_cov_kernel(RmodArgs A) {
  cg::cluster_group cl = cg::this_cluster();
  extern __shared__ __align__(16) unsigned char rmod_smem[];
  RmodShared& sh = *reinterpret_cast<RmodShared*>(rmod_smem);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rank = (int)cl.block_rank(), cs = (int)cl.num_blocks();
  int bi, K, lo;
  const double* N;
  double *tot, *T;
  rmod_setup(A, cl, bi, K, lo, N, tot, T);
  if (A.status[bi] == RM_NOT_PD) return;  // the whole cluster: the status is the same for every CTA
  const int n3 = 3 * K, nr = n3 - 6;
  const int f0 = A.uf_start[bi], nf = A.uf_start[bi + 1] - f0;
  const int gw = rank * RMOD_WARPS + warp, nw = cs * RMOD_WARPS;
  if (tid < n3) sh.M[tid] = A.model[3 * (size_t)lo + tid];
  __syncthreads();
  rmod_pass(cl, sh, A, bi, K, lo, 0.0, true, tot);
  // rows behind their camera, and each frame's cost
  int behind = 0;
  for (int j = gw; j < nf; j += nw) {
    const int f = A.uf_list[f0 + j];
    const double* q = A.pose + 6 * (size_t)f;
    double B[CT_JR + 9];
    cam_prep_rot(q[0], q[1], q[2], B);
    for (int i = A.start[f] + lane; i < A.start[f + 1]; i += 32) {
      const int r = A.rows[i];
      double X[3];
      bool front;
      rig_world(B, q + 3, sh.M + 3 * (A.obs_pt[r] - lo), X);
      tri_row_err2(A.camtab + (size_t)A.stride * A.obs_cam[r], X, reinterpret_cast<const double2*>(A.obs_px)[r], front);
      behind |= !front;
    }
    if (lane == 0) A.fcost[f] = A.gram[A.goff[f0 + j] + 27];
  }
  behind = __any_sync(0xffffffffu, behind);
  if (lane == 0) sh.w[warp].behind = behind;
  __syncthreads();
  if (tid == 0) {
    double bh = 0.0;
    for (int w = 0; w < RMOD_WARPS; ++w) bh += sh.w[w].behind;
    sh.part[1] = bh;
  }
  __threadfence();
  cl.sync();
  if (rank == 0) {
    const bool ok = rmod_factor(sh, tot, T, N, K, 0.0, true, TRI_PD_RTOL);
    double bh = 0.0;
    for (int r = 0; r < cs; ++r) bh += cl.map_shared_rank(sh.part, r)[1];
    if (tid == 0) {
      const int st = A.status[bi];
      A.status[bi] = !ok ? RM_NOT_PD : (st == RM_OK && bh > 0.0) ? RM_BEHIND : st;
    }
    if (ok && A.cov) rmod_cov_out(A, sh, T, N, K, bi);
  }
  cl.sync();
}

// ---- the camera term (cam_cov given) ---------------------------------------------------------------------------------
// The used rows sorted by (frame, camera) form runs.  Per run (frame f, camera c) rmod_run_kernel writes
//   D = E - X F  (3 m_f x P, the frame's markers in mask order),  E_k = sum over the run's rows of marker k of J_M^T J_c,
//   F = sum over the run's rows of J_q^T J_c (6 x P),  X_k = W_k V^-1 at the solution (lambda = 0),
// so that the body's Schur-reduced cross term is G^_c = sum over its frames (in key order) of their camera-c runs' D,
// which rmod_gsum_kernel adds entry by entry; rmod_camterm_kernel then adds P G^ Sigma_c G^^T P to cov.

// Per run r (rows rstart[r] .. rstart[r+1] of the (frame, camera)-sorted keys skey): its frame and camera, its D size
// 3 m P (0 when its frame is unused or its body is not solved) and, at frame heads, each frame's run range
__global__ void rmod_runs_kernel(const int* __restrict__ rstart, const unsigned long long* __restrict__ skey,
                                 int cam_bits, int n_runs, const int* __restrict__ fslot,
                                 const unsigned* __restrict__ fmask, const int* __restrict__ fbody,
                                 const int* __restrict__ status, int P, int* __restrict__ rframe, int* __restrict__ rcam,
                                 long long* __restrict__ rsize, int* __restrict__ frun0, int* __restrict__ frun1) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > n_runs) return;
  if (r == n_runs) {
    rsize[r] = 0;
    return;
  }
  const unsigned long long k = skey[rstart[r]];
  const int f = (int)(k >> cam_bits), c = (int)(k & ((1ULL << cam_bits) - 1));
  rframe[r] = f;
  rcam[r] = c;
  const int st = status[fbody[f]];
  const bool on = fslot[f] >= 0 && (st == RM_OK || st == RM_MAX_ITER || st == RM_BEHIND);
  rsize[r] = on ? 3LL * __popc(fmask[f]) * P : 0;
  if (r == 0 || (int)(skey[rstart[r - 1]] >> cam_bits) != f) frun0[f] = r;
  if (r == n_runs - 1 || (int)(skey[rstart[r + 1]] >> cam_bits) != f) frun1[f] = r + 1;
}

constexpr int RMOD_RUN_WARPS = 4;
template <int P>
struct RmodRunWarp {
  double J[32][6 + 12 + 2 * P];  // staged rows: J_M, J_q, J_c (pixels)
  double F[6 * P];
  double E[RMOD_NMAX * P];
  double X[RMOD_NMAX * 6];
  int lr[32];  // the staged row's marker position in the frame
};

// One run row's J_M (3 per pixel axis), J_q (12) and J_c (2 P), pixels, into Jr (out of line: rmod_run_kernel's loops
// keep their registers)
template <int P>
__device__ __noinline__ void rmod_run_row(const RmodArgs& A, const double* B, const double* q, const double* Mk, int row,
                                          double* Jr) {
  const double* cam = A.camtab + (size_t)A.stride * A.obs_cam[row];
  const double2 px = reinterpret_cast<const double2*>(A.obs_px)[row];
  double X[3], fr[2], JX[6], Jc[2 * P];
  rig_world(B, q + 3, Mk, X);
  obs_jac<P>(cam, X[0], X[1], X[2], px.x, px.y, 0, 1.0, fr, JX, Jc);
  const double fx0 = cam[CT_FX0];
  rig_jq(B, Mk, JX, fx0, Jr + 6);
#pragma unroll
  for (int s2 = 0; s2 < 2; ++s2)
#pragma unroll
    for (int c = 0; c < 3; ++c)
      Jr[3 * s2 + c] = (JX[3 * s2] * B[CT_R + c] + JX[3 * s2 + 1] * B[CT_R + 3 + c] + JX[3 * s2 + 2] * B[CT_R + 6 + c]) * fx0;
#pragma unroll
  for (int p = 0; p < 2 * P; ++p) Jr[18 + p] = Jc[p] * fx0;
}

// One warp per run: D = E - X F (see above) into D + roff[r]
template <int P>
__global__ void __launch_bounds__(32 * RMOD_RUN_WARPS, 1)
rmod_run_kernel(RmodArgs A, const int* __restrict__ rstart, const int* __restrict__ crow, const int* __restrict__ rframe,
                const long long* __restrict__ roff, const int* __restrict__ fslot, const int* __restrict__ fbody,
                int n_runs, double* __restrict__ D) {
  extern __shared__ __align__(16) unsigned char rmod_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  RmodRunWarp<P>& W = reinterpret_cast<RmodRunWarp<P>*>(rmod_smem)[warp];
  const long long r = (long long)blockIdx.x * RMOD_RUN_WARPS + warp;
  if (r >= n_runs || roff[r + 1] == roff[r]) return;
  const int f = rframe[r], slot = fslot[f], lo = A.body_start[fbody[f]];
  const unsigned mask = A.fmask[f];
  const int m = __popc(mask);
  const double* g = A.gram + A.goff[slot];
  if (lane < m) {  // X_l = W_l V^-1
    double L[6][6];
    rmod_chol_v(g, 0.0, L);
#pragma unroll 1
    for (int x = 0; x < 3; ++x) {
      double z[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) z[k] = g[RMOD_FRAME + RMOD_MARK * lane + 6 + 6 * x + k];
      res_chol_solve<6>(L, z);
#pragma unroll
      for (int k = 0; k < 6; ++k) W.X[6 * (3 * lane + x) + k] = z[k];
    }
  }
  for (int e = lane; e < 6 * P; e += 32) W.F[e] = 0.0;
  for (int e = lane; e < 3 * m * P; e += 32) W.E[e] = 0.0;
  const double* q = A.pose + 6 * (size_t)f;
  double B[CT_JR + 9];
  cam_prep_rot(q[0], q[1], q[2], B);
  const int b = rstart[r], e = rstart[r + 1];
  for (int base = b; base < e; base += 32) {
    const int i = base + lane, nr = min(32, e - base);
    if (i < e) {
      const int row = crow[i];
      const int k = A.obs_pt[row] - lo;
      const int lrow = __popc(mask & ((1u << k) - 1));
      W.lr[lane] = lrow;
      rmod_run_row<P>(A, B, q, A.model + 3 * (size_t)(lo + k), row, W.J[lane]);
    }
    __syncwarp();
    for (int x = lane; x < 6 * P; x += 32) {  // F, row order
      const int a = x / P, p = x % P;
      double sum = W.F[x];
      for (int rr = 0; rr < nr; ++rr) sum = fma(W.J[rr][6 + a], W.J[rr][18 + p], fma(W.J[rr][12 + a], W.J[rr][18 + P + p], sum));
      W.F[x] = sum;
    }
    for (int x = lane; x < 3 * m * P; x += 32) {  // E, row order, rows of the entry's marker
      const int l = x / (3 * P), a = (x / P) % 3, p = x % P;
      double sum = W.E[x];
      for (int rr = 0; rr < nr; ++rr) {
        if (W.lr[rr] != l) continue;
        sum = fma(W.J[rr][a], W.J[rr][18 + p], fma(W.J[rr][3 + a], W.J[rr][18 + P + p], sum));
      }
      W.E[x] = sum;
    }
    __syncwarp();
  }
  double* out = D + roff[r];
  for (int x = lane; x < 3 * m * P; x += 32) {
    const int row = x / P, p = x % P;
    double sum = W.E[x];
#pragma unroll
    for (int k = 0; k < 6; ++k) sum -= W.X[6 * row + k] * W.F[k * P + p];
    out[x] = sum;
  }
}

// One thread per entry (i, c, p) of a solved body's G^ (3K x n_cams P, at goff2[b]): the sum over the body's used
// frames in key order of the frame's camera-c run's D row of marker i / 3 (none when the frame lacks the camera or the
// marker)
__global__ void rmod_gsum_kernel(RmodArgs A, int n_active, int n_cams, int P, const long long* __restrict__ gofs,
                                 const int* __restrict__ frun0, const int* __restrict__ frun1,
                                 const int* __restrict__ rcam, const long long* __restrict__ roff,
                                 const double* __restrict__ D, double* __restrict__ G) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  int j = 0;  // the active body of entry t
  while (j < n_active && t >= gofs[j + 1]) ++j;
  if (j >= n_active) return;
  const int bi = A.bodies[j], st = A.status[bi];
  const long long e = t - gofs[j];
  const int nP = n_cams * P, i = (int)(e / nP), c = (int)((e % nP) / P), p = (int)(e % P), k = i / 3, a = i % 3;
  double sum = 0.0;
  if (st == RM_OK || st == RM_MAX_ITER || st == RM_BEHIND) {
    for (int s = A.uf_start[bi]; s < A.uf_start[bi + 1]; ++s) {
      const int f = A.uf_list[s];
      const unsigned mask = A.fmask[f];
      if (!((mask >> k) & 1)) continue;
      for (int r = frun0[f]; r < frun1[f]; ++r) {
        if (rcam[r] != c) continue;
        const int l = __popc(mask & ((1u << k) - 1));
        sum += D[roff[r] + (3 * l + a) * P + p];
        break;
      }
    }
  }
  G[t] = sum;
}

// One block per solved body: cov += P Y P, Y = G^ Sigma G^^T (Sigma at the uniform stride P, nP = n_cams P), with
// global scratch GS (3K x nP) and Y, T2 (3K x 3K) at the body's offsets
__global__ void __launch_bounds__(256)
rmod_camterm_kernel(RmodArgs A, int nP, const long long* __restrict__ gofs, const double* __restrict__ G,
                    const double* __restrict__ Sig, double* __restrict__ GS, double* __restrict__ Y,
                    double* __restrict__ T2) {
  const int j = blockIdx.x, bi = A.bodies[j], st = A.status[bi], tid = threadIdx.x;
  if (!(st == RM_OK || st == RM_MAX_ITER || st == RM_BEHIND)) return;
  const int n3 = 3 * (A.body_start[bi + 1] - A.body_start[bi]);
  const double* g = G + gofs[j];
  double* gs = GS + gofs[j];
  double* y = Y + A.coff[bi];
  double* t2 = T2 + A.coff[bi];
  const double* P = A.pmat + A.coff[bi];
  double* cov = A.cov + A.coff[bi];
  for (long long e = tid; e < (long long)n3 * nP; e += blockDim.x) {
    const int i = (int)(e / nP), c = (int)(e % nP);
    double s = 0.0;
    for (int x = 0; x < nP; ++x) s = fma(g[(size_t)i * nP + x], Sig[(size_t)x * nP + c], s);
    gs[e] = s;
  }
  __syncthreads();
  for (int e = tid; e < n3 * n3; e += blockDim.x) {
    const int i = e / n3, k = e % n3;
    double s = 0.0;
    for (int x = 0; x < nP; ++x) s = fma(gs[(size_t)i * nP + x], g[(size_t)k * nP + x], s);
    y[e] = s;
  }
  __syncthreads();
  for (int e = tid; e < n3 * n3; e += blockDim.x) {
    const int i = e / n3, k = e % n3;
    double s = 0.0;
    for (int x = 0; x < n3; ++x) s = fma(y[(size_t)i * n3 + x], P[(size_t)x * n3 + k], s);
    t2[e] = s;
  }
  __syncthreads();
  for (int e = tid; e < n3 * n3; e += blockDim.x) {
    const int i = e / n3, k = e % n3;
    if (k < i) continue;
    double s1 = 0.0, s2 = 0.0;
    for (int x = 0; x < n3; ++x) {
      s1 = fma(P[(size_t)i * n3 + x], t2[(size_t)x * n3 + k], s1);
      s2 = fma(P[(size_t)k * n3 + x], t2[(size_t)x * n3 + i], s2);
    }
    const double v = cov[(size_t)i * n3 + k] + 0.5 * (s1 + s2);
    cov[(size_t)i * n3 + k] = cov[(size_t)k * n3 + i] = v;
  }
}

}  // namespace cb
