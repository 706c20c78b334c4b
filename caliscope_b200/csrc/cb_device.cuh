// Device-side helpers for the caliscope_b200 bundle-adjustment engine (sm_90a).
#pragma once
#include <cuda.h>  // CUtensorMap (type only: the encoder is reached through cudaGetDriverEntryPoint)
#include <cuda_runtime.h>
#include <stdint.h>

namespace cb {

// ---------------------------------------------------------------------------------------------
// camera table (one entry per camera, rebuilt by cam_prep_kernel for every evaluation point)
// ---------------------------------------------------------------------------------------------
constexpr int CT_R = 0;      // 9  rotation, row-major
constexpr int CT_T = 9;      // 3  translation
constexpr int CT_JR = 12;    // 9  SO(3) right Jacobian: d(R X)/dr = -R [X]x Jr
constexpr int CT_FX = 21;    // fx = s * fx0
constexpr int CT_FY = 22;
constexpr int CT_CX = 23;
constexpr int CT_CY = 24;
constexpr int CT_D = 25;     // 5  Brown-Conrady k1 k2 p1 p2 k3 | fisheye k1 k2 k3 k4 -
constexpr int CT_IFX0 = 30;  // 1 / fx0
constexpr int CT_SX = 31;    // fx / fx0
constexpr int CT_SY = 32;    // fy / fx0
constexpr int CT_FYR = 33;   // fy0 / fx0
constexpr int CT_FLAGS = 34; // flags as double
constexpr int CT_FX0 = 35;   // fx0
constexpr int CT_SIZE = 36;
// stride of a camera-table entry in SHARED memory when lanes of a warp read DIFFERENT cameras (point-major kernels): an odd
// number of doubles, so that the same field of 16 consecutive cameras falls into 16 different 8-byte banks (stride 36 puts
// them into 4: an 8-way conflict on every one of the ~36 table reads per observation)
constexpr int CT_SMEM = 37;

constexpr double CB_EPS = 2.220446049250313e-16;

// index of entry (i, j), i <= j, of a symmetric N x N matrix packed as its upper triangle row by row
template <int N>
__host__ __device__ constexpr int ut(int i, int j) { return i * N - i * (i - 1) / 2 + (j - i); }

// ---------------------------------------------------------------------------------------------
// one full 32-byte sector per thread (32-byte aligned): sm_90 has no 256-bit global access, so two 128-bit
// accesses (LDG.E.128 / STG.E.128) to the two halves of the same sector
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void st256(double* p, double a, double b, double c, double d) {
  asm volatile("st.global.v2.f64 [%0], {%1,%2};\n\tst.global.v2.f64 [%0+16], {%3,%4};" ::"l"(p), "d"(a), "d"(b), "d"(c),
               "d"(d)
               : "memory");
}
__device__ __forceinline__ void ld256(const double* p, double& a, double& b, double& c, double& d) {
  asm volatile("ld.global.v2.f64 {%0,%1}, [%4];\n\tld.global.v2.f64 {%2,%3}, [%4+16];"
               : "=d"(a), "=d"(b), "=d"(c), "=d"(d)
               : "l"(p));
}
__device__ __forceinline__ void ld256nc(const double* p, double& a, double& b, double& c, double& d) {
  asm volatile("ld.global.nc.v2.f64 {%0,%1}, [%4];\n\tld.global.nc.v2.f64 {%2,%3}, [%4+16];"
               : "=d"(a), "=d"(b), "=d"(c), "=d"(d)
               : "l"(p));
}

// ---------------------------------------------------------------------------------------------
// mbarrier + 1-D bulk async copy (TMA engine; SASS: UBLKCP)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t phase) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(phase)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// global -> shared bulk copy, completion signalled on `bar` (bytes % 16 == 0, 16-byte aligned)
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// global -> shared 2-D tensor copy of one box of `map` at element coordinates (c0 innermost, c1), completion signalled
// on `bar` with the whole box's bytes (out-of-bounds elements arrive as zeros); dst 128-byte aligned (SASS: UTMALDG)
__device__ __forceinline__ void tma_load_2d(void* dst_smem, const CUtensorMap* map, int c0, int c1, unsigned long long* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(dst_smem)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}

// ---------------------------------------------------------------------------------------------
// reductions
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---------------------------------------------------------------------------------------------
// robust loss: rho(z), rho'(z), rho''(z), z = (f / f_scale)^2   (scipy least_squares.py loss table)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void loss_eval(int loss, double z, double& r0, double& r1, double& r2) {
  switch (loss) {
    case 1: {  // soft_l1
      double t = 1.0 + z, s = sqrt(t);
      r0 = 2.0 * (s - 1.0);
      r1 = 1.0 / s;
      r2 = -0.5 / (t * s);
    } break;
    case 2: {  // huber
      if (z <= 1.0) {
        r0 = z; r1 = 1.0; r2 = 0.0;
      } else {
        double s = sqrt(z);
        r0 = 2.0 * s - 1.0; r1 = 1.0 / s; r2 = -0.5 / (z * s);
      }
    } break;
    case 3: {  // cauchy
      double t = 1.0 + z;
      r0 = log1p(z); r1 = 1.0 / t; r2 = -1.0 / (t * t);
    } break;
    case 4: {  // arctan
      double t = 1.0 + z * z;
      r0 = atan(z); r1 = 1.0 / t; r2 = -2.0 * z / (t * t);
    } break;
    default:
      r0 = z; r1 = 1.0; r2 = 0.0;
  }
}

// Per scalar residual row: returns the cost contribution 0.5 * fs^2 * rho(z) and rescales
// (f, jacobian-row weight) as scipy's scale_for_robust_loss_function (common.py:720-731):
//   w = max(rho' + 2 rho'' z, EPS);  J_row *= sqrt(w);  f <- f * rho' / sqrt(w)
__device__ __forceinline__ double robust_row(int loss, double fs, double& f, double& jscale) {
  if (loss == 0) {
    jscale = 1.0;
    return 0.5 * f * f;
  }
  double q = f / fs, z = q * q, r0, r1, r2;
  loss_eval(loss, z, r0, r1, r2);
  double w = fmax(r1 + 2.0 * r2 * z, CB_EPS);
  jscale = sqrt(w);
  f = f * r1 / jscale;
  return 0.5 * fs * fs * r0;
}
__device__ __forceinline__ double robust_cost_only(int loss, double fs, double f) {
  if (loss == 0) return 0.5 * f * f;
  double q = f / fs, z = q * q, r0, r1, r2;
  loss_eval(loss, z, r0, r1, r2);
  return 0.5 * fs * fs * r0;
}

// ---------------------------------------------------------------------------------------------
// projection of one observation (cv2.projectPoints / cv2.fisheye.projectPoints closed forms)
// ---------------------------------------------------------------------------------------------
struct ProjOut {
  double u, v;         // pixels
  double a, b, r2;     // normalised coordinates and a^2 + b^2
  double xd, yd;       // distorted normalised coordinates
  double xa, xb, ya, yb;  // d(xd,yd)/d(a,b)
  double iz;
  double Xc[3];
};

template <bool JAC>
__device__ __forceinline__ void project_obs(const double* __restrict__ cam, bool fisheye, double X0, double X1,
                                            double X2, ProjOut& o) {
  const double* R = cam + CT_R;
  o.Xc[0] = fma(R[0], X0, fma(R[1], X1, fma(R[2], X2, cam[CT_T + 0])));
  o.Xc[1] = fma(R[3], X0, fma(R[4], X1, fma(R[5], X2, cam[CT_T + 1])));
  o.Xc[2] = fma(R[6], X0, fma(R[7], X1, fma(R[8], X2, cam[CT_T + 2])));
  double iz = (o.Xc[2] != 0.0) ? 1.0 / o.Xc[2] : 1.0;  // OpenCV: z == 0 -> 1
  double a = o.Xc[0] * iz, b = o.Xc[1] * iz;
  double r2 = a * a + b * b;
  o.iz = iz; o.a = a; o.b = b; o.r2 = r2;
  const double* d = cam + CT_D;
  if (!fisheye) {
    double k1 = d[0], k2 = d[1], p1 = d[2], p2 = d[3], k3 = d[4];
    double cd = 1.0 + r2 * (k1 + r2 * (k2 + r2 * k3));
    o.xd = a * cd + 2.0 * p1 * a * b + p2 * (r2 + 2.0 * a * a);
    o.yd = b * cd + p1 * (r2 + 2.0 * b * b) + 2.0 * p2 * a * b;
    if (JAC) {
      double dcd = k1 + r2 * (2.0 * k2 + 3.0 * k3 * r2);
      o.xa = cd + 2.0 * a * a * dcd + 2.0 * p1 * b + 6.0 * p2 * a;
      o.xb = 2.0 * a * b * dcd + 2.0 * p1 * a + 2.0 * p2 * b;
      o.ya = o.xb;
      o.yb = cd + 2.0 * b * b * dcd + 6.0 * p1 * b + 2.0 * p2 * a;
    }
  } else {
    double rr = sqrt(r2);
    double th = atan(rr), th2 = th * th;
    double thd = th * (1.0 + th2 * (d[0] + th2 * (d[1] + th2 * (d[2] + th2 * d[3]))));
    bool big = rr > 1e-8;
    double inv_r = big ? 1.0 / rr : 1.0;
    double cdist = big ? thd * inv_r : 1.0;
    o.xd = a * cdist;
    o.yd = b * cdist;
    if (JAC) {
      double dthd = 1.0 + th2 * (3.0 * d[0] + th2 * (5.0 * d[1] + th2 * (7.0 * d[2] + th2 * 9.0 * d[3])));
      double dcdr = big ? (dthd / (1.0 + r2) - cdist) * inv_r : 0.0;
      double fa = big ? a * inv_r : 0.0, fb = big ? b * inv_r : 0.0;
      o.xa = cdist + a * dcdr * fa;
      o.xb = a * dcdr * fb;
      o.ya = b * dcdr * fa;
      o.yb = cdist + b * dcdr * fb;
    }
  }
  o.u = fma(cam[CT_FX], o.xd, cam[CT_CX]);
  o.v = fma(cam[CT_FY], o.yd, cam[CT_CY]);
}

// ---------------------------------------------------------------------------------------------
// One observation's scaled residual and analytic Jacobian blocks, recomputed from (camera table entry,
// point, pixel) wherever they are needed (camera pass, point pass, back-substitution): no Jacobian row
// is ever written to HBM.  Reference: src/caliscope/core/reprojection.py:96-110 (residual / fx0),
// :171-205 (camera block [J_r, J_t (, J_s, J_k1, J_k2)] / fx0, point block J_t R / fx0); robust rescaling
// as scipy common.py:720-731.
//   f[2]      residuals (after robust rescale)
//   JX[6]     d f / d X      (2 x 3, row-major)
//   Jc[2*P]   d f / d camera (2 x P, row-major); P = 9 slots are zero for a locked camera
// returns the cost contribution 0.5 * fs^2 * (rho(z0) + rho(z1)).
// ---------------------------------------------------------------------------------------------
// light form for the V / g reduction of the point pass: residuals and d f / d X only (no camera block)
__device__ __forceinline__ void obs_res_jx(const double* __restrict__ cam, double X0, double X1, double X2, double ox,
                                           double oy, int loss, double fscale, double* __restrict__ f,
                                           double* __restrict__ JX) {
  const int flags = (int)cam[CT_FLAGS];
  ProjOut o;
  project_obs<true>(cam, (flags & 2) != 0, X0, X1, X2, o);
  double f0 = (o.u - ox) * cam[CT_IFX0], f1 = (o.v - oy) * cam[CT_IFX0];
  double w0, w1;
  robust_row(loss, fscale, f0, w0);
  robust_row(loss, fscale, f1, w1);
  f[0] = f0; f[1] = f1;
  const double sx = cam[CT_SX] * o.iz * w0, sy = cam[CT_SY] * o.iz * w1;
  const double t0 = sx * o.xa, t1 = sx * o.xb, t2 = -(t0 * o.a + t1 * o.b);
  const double t3 = sy * o.ya, t4 = sy * o.yb, t5 = -(t3 * o.a + t4 * o.b);
  const double* R = cam + CT_R;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    JX[k] = t0 * R[k] + t1 * R[3 + k] + t2 * R[6 + k];
    JX[3 + k] = t3 * R[k] + t4 * R[3 + k] + t5 * R[6 + k];
  }
}

// ---------------------------------------------------------------------------------------------
// One camera pair of a point covariance gather: x = Z_a Sig_ab Z_b^T for the 3 x P blocks Z_a, Z_b (row stride ld) and
// the P x P block (ca, cb) of Sig (row stride nP).  cov_point_kernel (Z = the point's Zt rows) and tri_cov_kernel
// (Z = the per-camera blocks J_X^T J_c of a triangulated point) both sum these over the unordered camera pairs.
// ---------------------------------------------------------------------------------------------
template <int P>
__device__ __forceinline__ void cov_pair_gather(const double* __restrict__ za, const double* __restrict__ zb, size_t ld,
                                                const double* __restrict__ Sig, int nP, int ca, int cb, double x[3][3]) {
  double zr[3][P];
#pragma unroll
  for (int b = 0; b < 3; ++b)
#pragma unroll
    for (int q = 0; q < P; ++q) zr[b][q] = zb[(size_t)b * ld + q];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) x[a][b] = 0.0;
#pragma unroll
  for (int p = 0; p < P; ++p) {
    const double* srow = Sig + (size_t)(ca * P + p) * nP + (size_t)cb * P;
    double y0 = 0.0, y1 = 0.0, y2 = 0.0;
#pragma unroll
    for (int q = 0; q < P; ++q) {
      const double sv = srow[q];
      y0 = fma(sv, zr[0][q], y0); y1 = fma(sv, zr[1][q], y1); y2 = fma(sv, zr[2][q], y2);
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double v = za[(size_t)a * ld + p];
      x[a][0] = fma(v, y0, x[a][0]); x[a][1] = fma(v, y1, x[a][1]); x[a][2] = fma(v, y2, x[a][2]);
    }
  }
}

template <int P>
__device__ __forceinline__ double obs_jac(const double* __restrict__ cam, double X0, double X1, double X2,
                                          double ox, double oy, int loss, double fscale, double* __restrict__ f,
                                          double* __restrict__ JX, double* __restrict__ Jc) {
  const int flags = (int)cam[CT_FLAGS];
  const bool fish = (flags & 2) != 0;
  const bool free_i = (P == 9) && (flags & 1) != 0;
  ProjOut o;
  project_obs<true>(cam, fish, X0, X1, X2, o);
  double f0 = (o.u - ox) * cam[CT_IFX0], f1 = (o.v - oy) * cam[CT_IFX0];
  double w0, w1;
  const double cost = robust_row(loss, fscale, f0, w0) + robust_row(loss, fscale, f1, w1);
  f[0] = f0; f[1] = f1;
  const double sx = cam[CT_SX] * o.iz * w0, sy = cam[CT_SY] * o.iz * w1;
  double Jt[6];
  Jt[0] = sx * o.xa; Jt[1] = sx * o.xb; Jt[2] = -(Jt[0] * o.a + Jt[1] * o.b);
  Jt[3] = sy * o.ya; Jt[4] = sy * o.yb; Jt[5] = -(Jt[3] * o.a + Jt[4] * o.b);
  const double* R = cam + CT_R;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int k = 0; k < 3; ++k) JX[3 * i + k] = Jt[3 * i] * R[k] + Jt[3 * i + 1] * R[3 + k] + Jt[3 * i + 2] * R[6 + k];
  const double* Jr = cam + CT_JR;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    // (J_X,i x X) Jr, negated
    const double a0 = JX[3 * i], a1 = JX[3 * i + 1], a2 = JX[3 * i + 2];
    const double c0 = a1 * X2 - a2 * X1, c1 = a2 * X0 - a0 * X2, c2 = a0 * X1 - a1 * X0;
#pragma unroll
    for (int k = 0; k < 3; ++k) Jc[P * i + k] = -(c0 * Jr[k] + c1 * Jr[3 + k] + c2 * Jr[6 + k]);
    Jc[P * i + 3] = Jt[3 * i]; Jc[P * i + 4] = Jt[3 * i + 1]; Jc[P * i + 5] = Jt[3 * i + 2];
  }
  if constexpr (P == 9) {
    if (free_i) {
      const double ar2 = cam[CT_SX] * o.a * o.r2 * w0, br2 = cam[CT_SY] * o.b * o.r2 * w1;
      Jc[6] = o.xd * w0;  Jc[P + 6] = cam[CT_FYR] * o.yd * w1;
      Jc[7] = ar2;        Jc[P + 7] = br2;
      Jc[8] = ar2 * o.r2; Jc[P + 8] = br2 * o.r2;
    } else {
      Jc[6] = Jc[7] = Jc[8] = 0.0;
      Jc[P + 6] = Jc[P + 7] = Jc[P + 8] = 0.0;
    }
  }
  return cost;
}

// ---- the lanes of one group ----------------------------------------------------------------------------------------
// A group owns LANES consecutive, aligned lanes of a warp, so xor offsets below LANES stay inside it.  The reductions
// are xor butterflies over s = LANES/2 ... 1: every lane of the group ends with the identical result, summed in one
// fixed order.  Every lane of the warp must take part, live group or not.

// the group's sum of a scalar
template <int LANES, typename T>
[[nodiscard]] __device__ __forceinline__ T group_sum(T v) {
#pragma unroll
  for (int s = LANES / 2; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
  return v;
}

// the group's sums of an array, in place
template <int LANES, typename T, int N>
__device__ __forceinline__ void group_sum(T (&v)[N]) {
#pragma unroll
  for (int s = LANES / 2; s > 0; s >>= 1)
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] += __shfl_xor_sync(0xffffffffu, v[k], s);
}

template <int LANES>
[[nodiscard]] __device__ __forceinline__ int group_or(int v) {
#pragma unroll
  for (int s = LANES / 2; s > 0; s >>= 1) v |= __shfl_xor_sync(0xffffffffu, v, s);
  return v;
}

// the lowest score of the group, the lowest index on a tie, in place
template <int LANES>
__device__ __forceinline__ void group_argmin(double& score, long long& index) {
#pragma unroll
  for (int s = LANES / 2; s > 0; s >>= 1) {
    const double os = __shfl_xor_sync(0xffffffffu, score, s);
    const long long oi = __shfl_xor_sync(0xffffffffu, index, s);
    if (os < score || (os == score && oi < index)) {
      score = os;
      index = oi;
    }
  }
}

// v from lane `owner` of the group to all its lanes
template <int LANES, int N>
__device__ __forceinline__ void group_bcast(double (&v)[N], int owner) {
#pragma unroll
  for (int q = 0; q < N; ++q) v[q] = __shfl_sync(0xffffffffu, v[q], owner, LANES);
}

}  // namespace cb
