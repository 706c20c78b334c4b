// Microbenchmark: what the point pass's Zt stores cost on cfg4's shape, and whether writing whole 64-byte granules
// instead of 48-byte pieces changes it.  Zt is (3 n_pts + 32) x LD doubles with its structural zeros pre-written; a
// seeded visibility (a random 40 of 64 cameras per point, or 8 adjacent cameras per point like sparse64); a 256 MB L2
// flush before every launch; CUDA events around each of 24 launches.  The stored values are a cheap function of
// (point, camera, row, column), so the variants are checked bit for bit against (a) after each run.
//   (a) today's pattern: 8 lanes per point, each writes its camera's three P-double pieces (16-byte stores at P = 6)
//   (b) the group stages its eight pieces in shared memory, then writes every granule they touch whole, four lanes
//       per granule (coalesced 16-byte stores), zeros where a granule covers a camera the point does not see
//   (c) the granules of (b) assembled in shared memory and written by cp.async.bulk (64 B each)
//   (d) whole rows: all LD doubles of each of the point's three rows
//   (f) the stores of (a) plus zeros over the rest of each boundary granule whose neighbour camera is unseen (no
//       shared memory: every granule a point touches ends up fully written in L2, by the lanes that own it)
//   (e) a frozen copy of the point pass as it was before its stores were staged, the same copy with the Zt stores
//       replaced by a sum written once per thread (what the rest of the kernel costs), and the engine's pt_pass_kernel
//       (cb_lm.cuh) with its staged whole-granule stores, checked bit for bit against the copy's Zt
// Prints us per launch and GB/s of Zt payload (the pieces only).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o zt_store zt_store.cu && ./zt_store
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <random>
#include <vector>

#include "../../caliscope_b200/csrc/cb_lm.cuh"

constexpr int LANES = 8, THREADS = cb::PT_WARPS * 32;

__device__ __forceinline__ double zval(int j, int cam, int a, int p) {
  return (double)((j * 131 + cam * 7 + a * 3) & 1023) + 0.125 * p + 1.0;
}

__device__ __forceinline__ void bulk_s2g(void* gdst, const void* ssrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
               "r"((uint32_t)__cvta_generic_to_shared(ssrc)), "r"(bytes) : "memory");
}

// per-group staging of (b) / (c): the round's pieces (slot 0: the last piece of the previous round), the granules they
// own as (granule << 4 | slot), and (c)'s assembled granules
template <int P, bool BULK>
struct Stage {
  static constexpr int NSLOT = LANES + 1, GMAX = 2 * LANES;
  double z[NSLOT][3][P];
  int cam[NSLOT];
  int list[GMAX];
  __align__(16) double g[BULK ? 3 * GMAX : 1][8];
};

// MODE 0: (a), 1: (b), 2: (c), 3: (d), 5: (f)
template <int P, int MODE>
__global__ void __launch_bounds__(THREADS, 2)
store_kernel(const int* __restrict__ pt_start, const int* __restrict__ pm_cam, int n_pts, int n_cams,
             double* __restrict__ Zt, size_t LD) {
  extern __shared__ __align__(16) unsigned char raw[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, gl = lane % LANES, grp = lane / LANES;
  Stage<P, MODE == 2>& sg = reinterpret_cast<Stage<P, MODE == 2>*>(raw)[wid * (32 / LANES) + grp];
  const unsigned gmask = (LANES == 32) ? 0xffffffffu : (((1u << LANES) - 1u) << (grp * LANES));
  for (int j0 = (blockIdx.x * cb::PT_WARPS + wid) * (32 / LANES); j0 < n_pts; j0 += gridDim.x * cb::PT_WARPS * (32 / LANES)) {
    const int j = j0 + grp;
    int s = 0, e = 0;
    if (j < n_pts) { s = pt_start[j]; e = pt_start[j + 1]; }
    double* row = Zt + 3 * (size_t)j * LD;
    if constexpr (MODE == 0 || MODE == 5) {
      for (int pos = s + gl; pos < e; pos += LANES) {
        const int cam = pm_cam[pos];
        double* z0 = row + (size_t)cam * P;
        for (int a = 0; a < 3; ++a)
          for (int p = 0; p < P; p += (P == 6 ? 2 : 1)) {
            if constexpr (P == 6) *reinterpret_cast<double2*>(z0 + a * LD + p) = make_double2(zval(j, cam, a, p), zval(j, cam, a, p + 1));
            else z0[a * LD + p] = zval(j, cam, a, p);
          }
        if constexpr (MODE == 5) {
          const int c0 = cam * P, c1 = c0 + P;
          const bool prev_seen = pos > s && pm_cam[pos - 1] == cam - 1, next_seen = pos + 1 < e && pm_cam[pos + 1] == cam + 1;
          for (int a = 0; a < 3; ++a) {
            double* r = row + a * LD;
            if (!prev_seen)
              for (int c = c0 & ~7; c < c0; c += (P == 6 ? 2 : 1)) {
                if constexpr (P == 6) *reinterpret_cast<double2*>(r + c) = make_double2(0.0, 0.0);
                else r[c] = 0.0;
              }
            if (!next_seen)
              for (int c = c1; c < ((c1 + 7) & ~7); c += (P == 6 ? 2 : 1)) {
                if constexpr (P == 6) *reinterpret_cast<double2*>(r + c) = make_double2(0.0, 0.0);
                else r[c] = 0.0;
              }
          }
        }
      }
    } else if constexpr (MODE == 3) {
      unsigned long long seen = 0ull;
      for (int pos = s + gl; pos < e; pos += LANES) seen |= 1ull << pm_cam[pos];
      for (int o = LANES / 2; o > 0; o >>= 1) seen |= __shfl_xor_sync(gmask, seen, o);
      if (j < n_pts)
        for (int a = 0; a < 3; ++a)
          for (int c = 2 * gl; c < (int)LD; c += 2 * LANES) {
            double v[2];
            for (int u = 0; u < 2; ++u) {
              const int cam = (c + u) / P;
              v[u] = (cam < n_cams && ((seen >> cam) & 1)) ? zval(j, cam, a, (c + u) - cam * P) : 0.0;
            }
            *reinterpret_cast<double2*>(row + a * LD + c) = make_double2(v[0], v[1]);
          }
    } else {
      if (gl == 0) sg.cam[0] = -1;
      __syncwarp(gmask);
      for (int base = s; base < e; base += LANES) {
        const int pos = base + gl;
        const bool act = pos < e;
        const int cam = act ? pm_cam[pos] : -1;
        const int next = (pos + 1 < e) ? pm_cam[pos + 1] : -1;
        if (act)
          for (int a = 0; a < 3; ++a)
            for (int p = 0; p < P; ++p) sg.z[gl + 1][a][p] = zval(j, cam, a, p);
        sg.cam[gl + 1] = cam;
        // granules this lane's piece owns: all it touches, except a last one the next camera's piece shares
        int g0 = 0, ng = 0;
        if (act) {
          g0 = (cam * P) >> 3;
          const int g1 = (cam * P + P - 1) >> 3;
          ng = g1 - g0 + 1;
          if (next == cam + 1 && ((cam + 1) * P) >> 3 == g1) --ng;
        }
        int off = ng;  // inclusive scan over the group
        for (int o = 1; o < LANES; o <<= 1) {
          const int t = __shfl_up_sync(gmask, off, o, LANES);
          if (gl >= o) off += t;
        }
        const int total = __shfl_sync(gmask, off, LANES - 1, LANES);
        for (int q = 0; q < ng; ++q) sg.list[off - ng + q] = ((g0 + q) << 4) | (gl + 1);
        __syncwarp(gmask);
        // item = (granule, row, quarter); four consecutive lanes fill one granule
        for (int it = gl; it < total * 12; it += LANES) {
          const int gi = it / 12, a = (it / 4) % 3, qtr = it & 3;
          const int ent = sg.list[gi], G = ent >> 4, sl = ent & 15;
          const int oc = sg.cam[sl], pc = sg.cam[sl - 1];
          double v[2];
          for (int u = 0; u < 2; ++u) {
            const int col = 8 * G + 2 * qtr + u;
            if (col >= oc * P) v[u] = col < oc * P + P ? sg.z[sl][a][col - oc * P] : 0.0;
            else v[u] = pc == oc - 1 ? sg.z[sl - 1][a][col - pc * P] : 0.0;
          }
          if constexpr (MODE == 1) {
            *reinterpret_cast<double2*>(row + a * LD + 8 * G + 2 * qtr) = make_double2(v[0], v[1]);
          } else {
            sg.g[gi * 3 + a][2 * qtr] = v[0];
            sg.g[gi * 3 + a][2 * qtr + 1] = v[1];
          }
        }
        if constexpr (MODE == 2) {
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          __syncwarp(gmask);
          for (int it = gl; it < total * 3; it += LANES) {
            const int gi = it / 3, a = it % 3, G = sg.list[gi] >> 4;
            bulk_s2g(row + a * LD + 8 * G, sg.g[gi * 3 + a], 64);
          }
          asm volatile("cp.async.bulk.commit_group;" ::: "memory");
          asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        }
        __syncwarp(gmask);
        // carry the last piece of this round into slot 0
        const int last = min(e - base, LANES);
        for (int i = gl; i < 3 * P; i += LANES) sg.z[0][i / P][i % P] = sg.z[last][i / P][i % P];
        if (gl == 0) sg.cam[0] = sg.cam[last];
        __syncwarp(gmask);
      }
    }
  }
}

// (e): a frozen copy of cb::pt_pass_kernel<P, 8, false, true> (no repeated rows, camera table in shared memory) as it was
// before its Zt stores were staged: STORE writes each observation's pieces straight to Zt (16-byte stores at P = 6);
// without STORE the pieces go into a running sum written once per thread
template <int P, bool STORE>
__global__ void __launch_bounds__(THREADS, 2)
pt_pass_copy(const cb::LmState* __restrict__ st, const int* __restrict__ pt_start, const int* __restrict__ pm_cam,
             const double2* __restrict__ pm_xy, int n_pts, int n_cams, cb::CPtr2 camtab2, cb::CPtr2 xp2,
             double* __restrict__ V6, double* __restrict__ gp, double* __restrict__ Dp2, double* __restrict__ Linv6,
             double* __restrict__ tvec, double* __restrict__ Zt, size_t LD, double* __restrict__ sink) {
  using namespace cb;
  extern __shared__ __align__(16) double pt_sm[];
  const double lam = st->lam;
  const int loss = st->loss;
  const double fscale = st->fscale;
  const double* __restrict__ gtab = camtab2.p[0];
  const double* xp4 = xp2.p[0];
  for (int i = threadIdx.x; i < n_cams * CT_SIZE; i += blockDim.x) pt_sm[(i / CT_SIZE) * CT_SMEM + i % CT_SIZE] = gtab[i];
  __syncthreads();
  constexpr int GPW = 32 / LANES;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, gl = lane % LANES, grp = lane / LANES;
  double acc = 0.0;
  for (int j0 = (blockIdx.x * PT_WARPS + wid) * GPW; j0 < n_pts; j0 += gridDim.x * PT_WARPS * GPW) {
    const int j = j0 + grp;
    const bool valid = j < n_pts;
    int s = 0, e = 0;
    double X0 = 0.0, X1 = 0.0, X2 = 0.0, X3;
    if (valid) { s = pt_start[j]; e = pt_start[j + 1]; ld256nc(xp4 + 4 * (size_t)j, X0, X1, X2, X3); }
    (void)X3;
    double v[9];
    for (int k = 0; k < 9; ++k) v[k] = 0.0;
    int cam_n = 0;
    double2 xy_n = make_double2(0.0, 0.0);
    if (s + gl < e) { cam_n = pm_cam[s + gl]; xy_n = pm_xy[s + gl]; }
    for (int pos = s + gl; pos < e; pos += LANES) {
      const int cam = cam_n;
      const double2 xy = xy_n;
      if (pos + LANES < e) { cam_n = pm_cam[pos + LANES]; xy_n = pm_xy[pos + LANES]; }
      double f[2], JX[6];
      obs_res_jx(pt_sm + cam * CT_SMEM, X0, X1, X2, xy.x, xy.y, loss, fscale, f, JX);
      v[0] += JX[0] * JX[0] + JX[3] * JX[3]; v[1] += JX[0] * JX[1] + JX[3] * JX[4]; v[2] += JX[0] * JX[2] + JX[3] * JX[5];
      v[3] += JX[1] * JX[1] + JX[4] * JX[4]; v[4] += JX[1] * JX[2] + JX[4] * JX[5]; v[5] += JX[2] * JX[2] + JX[5] * JX[5];
      v[6] += JX[0] * f[0] + JX[3] * f[1]; v[7] += JX[1] * f[0] + JX[4] * f[1]; v[8] += JX[2] * f[0] + JX[5] * f[1];
    }
    for (int k = 0; k < 9; ++k) v[k] = group_sum<LANES>(v[k]);
    double D[3] = {1.0, 1.0, 1.0};
    if (valid) { const double* d = Dp2 + (size_t)j * 3; D[0] = fmax(d[0], v[0]); D[1] = fmax(d[1], v[3]); D[2] = fmax(d[2], v[5]); }
    double Li[6];
    chol3_inv(v, D, lam, Li);
    if (valid && gl == 0) {
      for (int k = 0; k < 6; ++k) V6[(size_t)j * 6 + k] = v[k];
      for (int k = 0; k < 3; ++k) { gp[(size_t)j * 3 + k] = v[6 + k]; Dp2[(size_t)j * 3 + k] = D[k]; }
      for (int k = 0; k < 6; ++k) Linv6[(size_t)j * 6 + k] = Li[k];
      tvec[3 * (size_t)j + 0] = Li[0] * v[6];
      tvec[3 * (size_t)j + 1] = Li[1] * v[6] + Li[2] * v[7];
      tvec[3 * (size_t)j + 2] = Li[3] * v[6] + Li[4] * v[7] + Li[5] * v[8];
    }
    if (s + gl < e) { cam_n = pm_cam[s + gl]; xy_n = pm_xy[s + gl]; }
    for (int pos = s + gl; pos < e; pos += LANES) {
      const int cam = cam_n;
      const double2 xy = xy_n;
      if (pos + LANES < e) { cam_n = pm_cam[pos + LANES]; xy_n = pm_xy[pos + LANES]; }
      double f[2], JX[6], Jc[2 * P];
      obs_jac<P>(pt_sm + cam * CT_SMEM, X0, X1, X2, xy.x, xy.y, loss, fscale, f, JX, Jc);
      double q00, q01, q02, q10, q11, q12;
      pt_factor_rows<false>(JX, Li, q00, q01, q02, q10, q11, q12);
      double z[3][P];
      for (int p = 0; p < P; ++p) {
        z[0][p] = fma(Jc[p], q00, Jc[P + p] * q10);
        z[1][p] = fma(Jc[p], q01, Jc[P + p] * q11);
        z[2][p] = fma(Jc[p], q02, Jc[P + p] * q12);
      }
      if constexpr (STORE) {
        double* z0 = Zt + (3 * (size_t)j) * LD + (size_t)cam * P;
        for (int a = 0; a < 3; ++a) {
          if constexpr (P == 6) {
            double2* dst = reinterpret_cast<double2*>(z0 + a * LD);
            dst[0] = make_double2(z[a][0], z[a][1]);
            dst[1] = make_double2(z[a][2], z[a][3]);
            dst[2] = make_double2(z[a][4], z[a][5]);
          } else {
            for (int p = 0; p < P; ++p) z0[a * LD + p] = z[a][p];
          }
        }
      } else {
        for (int p = 0; p < P; ++p) acc += z[0][p] + z[1][p] + z[2][p];
      }
    }
  }
  sink[blockIdx.x * (size_t)blockDim.x + threadIdx.x] = acc;
}

__global__ void count_diff(const double* __restrict__ a, const double* __restrict__ b, size_t n,
                           unsigned long long* __restrict__ out) {
  unsigned long long d = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    d += __double_as_longlong(a[i]) != __double_as_longlong(b[i]);
  if (d) atomicAdd(out, d);
}

struct Case { const char* name; int P, n_pts, per_pt; bool adjacent; };

static void run_case(const Case& cs, int sms, double* flush, size_t flush_bytes) {
  const int n_cams = 64, P = cs.P, n_pts = cs.n_pts;
  const size_t LD = (size_t)(n_cams * P + 95) / 96 * 96;
  std::mt19937_64 rng(20261015ull + P * 7 + cs.adjacent);
  std::vector<int> start(n_pts + 1, 0), cams;
  std::vector<double> xy;
  std::vector<int> perm(n_cams);
  for (int j = 0; j < n_pts; ++j) {
    std::vector<int> c;
    if (cs.adjacent) {
      const int c0 = (int)(rng() % (n_cams - cs.per_pt + 1));
      for (int i = 0; i < cs.per_pt; ++i) c.push_back(c0 + i);
    } else {
      for (int i = 0; i < n_cams; ++i) perm[i] = i;
      for (int i = 0; i < cs.per_pt; ++i) std::swap(perm[i], perm[i + rng() % (n_cams - i)]);
      c.assign(perm.begin(), perm.begin() + cs.per_pt);
      std::sort(c.begin(), c.end());
    }
    cams.insert(cams.end(), c.begin(), c.end());
    start[j + 1] = (int)cams.size();
  }
  const size_t n_obs = cams.size();
  std::uniform_real_distribution<double> U(-1.0, 1.0);
  for (size_t i = 0; i < n_obs; ++i) { xy.push_back(640.0 + 300.0 * U(rng)); xy.push_back(480.0 + 300.0 * U(rng)); }
  // payload: the pieces; granule and sector counts of the rows (what reaches L2 as partial lines)
  double granules = 0, partial = 0;
  for (int j = 0; j < n_pts; ++j) {
    std::vector<int> cov(LD / 8, 0);
    for (int i = start[j]; i < start[j + 1]; ++i)
      for (int col = cams[i] * P; col < cams[i] * P + P; ++col) cov[col / 8]++;
    for (int v : cov) { granules += v > 0; partial += v > 0 && v < 8; }
  }
  const double payload = 24.0 * P * n_obs;
  printf("\n== %s: P = %d, LD = %zu, %d points, %zu observations, payload %.1f MB; per row %.1f granules touched, "
         "%.1f partly\n", cs.name, P, LD, n_pts, n_obs, payload * 1e-6, granules / n_pts, partial / n_pts);

  int *d_start, *d_cam;
  double2* d_xy;
  const size_t zn = (3 * (size_t)n_pts + 32) * LD;
  double *Zt, *Zref;
  cudaMalloc(&d_start, (n_pts + 1) * sizeof(int));
  cudaMalloc(&d_cam, n_obs * sizeof(int));
  cudaMalloc(&d_xy, n_obs * sizeof(double2));
  cudaMalloc(&Zt, zn * sizeof(double));
  cudaMalloc(&Zref, zn * sizeof(double));
  cudaMemcpy(d_start, start.data(), start.size() * sizeof(int), cudaMemcpyHostToDevice);
  cudaMemcpy(d_cam, cams.data(), n_obs * sizeof(int), cudaMemcpyHostToDevice);
  cudaMemcpy(d_xy, xy.data(), n_obs * sizeof(double2), cudaMemcpyHostToDevice);
  unsigned long long* d_diff;
  cudaMalloc(&d_diff, sizeof(unsigned long long));
  const int grid = std::min((n_pts + cb::PT_WARPS * 4 - 1) / (cb::PT_WARPS * 4), 2 * sms);
  const int reps = 24;

  auto timed = [&](auto launch) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    float tot = 0.f;
    for (int r = 0; r < reps + 2; ++r) {
      cudaMemsetAsync(flush, r & 0xff, flush_bytes);
      cudaEventRecord(e0);
      launch();
      cudaEventRecord(e1);
      cudaEventSynchronize(e1);
      float ms = 0.f;
      cudaEventElapsedTime(&ms, e0, e1);
      if (r >= 2) tot += ms;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    const cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) { printf("CUDA error: %s\n", cudaGetErrorString(err)); return NAN; }
    return tot / reps;
  };
  auto report = [&](const char* name, float ms, bool check) {
    printf("  %-58s %8.1f us  %7.0f GB/s payload", name, ms * 1e3, payload / (ms * 1e-3) * 1e-9);
    if (check) {
      cudaMemset(d_diff, 0, sizeof(unsigned long long));
      count_diff<<<1024, 256>>>(Zt, Zref, zn, d_diff);
      unsigned long long h = 0;
      cudaMemcpy(&h, d_diff, sizeof(h), cudaMemcpyDeviceToHost);
      printf("  %s (%llu words differ from the reference)", h ? "MISMATCH" : "identical", h);
    }
    printf("\n");
  };
  auto variant = [&](auto kern, const char* name, int smem, bool check) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaMemset(Zt, 0, zn * sizeof(double));
    const float ms = timed([&] { kern<<<grid, THREADS, smem>>>(d_start, d_cam, n_pts, n_cams, Zt, LD); });
    if (!check) cudaMemcpy(Zref, Zt, zn * sizeof(double), cudaMemcpyDeviceToDevice);
    report(name, ms, check);
  };
  const int groups = cb::PT_WARPS * (32 / LANES);
  if (P == 6) {
    const int sm = (int)sizeof(Stage<6, false>) * groups, smb = (int)sizeof(Stage<6, true>) * groups;
    variant(store_kernel<6, 0>, "(a) 48-byte pieces, 16-byte stores", 0, false);
    variant(store_kernel<6, 1>, "(b) staged, whole granules, 4 lanes per granule", sm, true);
    variant(store_kernel<6, 2>, "(c) staged, whole granules by cp.async.bulk", smb, true);
    variant(store_kernel<6, 3>, "(d) whole rows", 0, true);
    variant(store_kernel<6, 5>, "(f) pieces + zeros completing the boundary granules", 0, true);
  } else {
    const int sm = (int)sizeof(Stage<9, false>) * groups, smb = (int)sizeof(Stage<9, true>) * groups;
    variant(store_kernel<9, 0>, "(a) 72-byte pieces, 8-byte stores", 0, false);
    variant(store_kernel<9, 1>, "(b) staged, whole granules, 4 lanes per granule", sm, true);
    variant(store_kernel<9, 2>, "(c) staged, whole granules by cp.async.bulk", smb, true);
    variant(store_kernel<9, 3>, "(d) whole rows", 0, true);
    variant(store_kernel<9, 5>, "(f) pieces + zeros completing the boundary granules", 0, true);
  }

  // (e) the engine kernel and its copy without Zt stores
  {
    std::vector<double> xc((size_t)n_cams * P), kc((size_t)n_cams * 9, 0.0), xp(4 * (size_t)n_pts, 0.0);
    std::vector<int> flags(n_cams, P == 9 ? 1 : 0);
    for (int c = 0; c < n_cams; ++c) {
      double* q = &xc[(size_t)c * P];
      q[0] = 0.05 * U(rng); q[1] = 0.05 * U(rng); q[2] = 0.05 * U(rng);
      q[3] = 0.1 * U(rng); q[4] = 0.1 * U(rng); q[5] = 5.0 + 0.1 * U(rng);
      if (P == 9) { q[6] = 1.0; q[7] = 0.0; q[8] = 0.0; }
      double* k = &kc[(size_t)c * 9];
      k[0] = 1000.0; k[1] = 1000.0; k[2] = 640.0; k[3] = 480.0;
    }
    for (int j = 0; j < n_pts; ++j)
      for (int a = 0; a < 3; ++a) xp[4 * (size_t)j + a] = U(rng);
    double *d_xc, *d_kc, *d_tab, *d_xp, *V6, *gp, *Dp2, *Li, *tv, *sink;
    int* d_flags;
    unsigned long long* gmax;
    cudaMalloc(&d_xc, xc.size() * 8); cudaMalloc(&d_kc, kc.size() * 8); cudaMalloc(&d_xp, xp.size() * 8);
    cudaMalloc(&d_tab, (size_t)n_cams * cb::CT_SIZE * 8); cudaMalloc(&d_flags, n_cams * 4);
    cudaMalloc(&V6, (size_t)n_pts * 48); cudaMalloc(&gp, (size_t)n_pts * 24); cudaMalloc(&Dp2, (size_t)n_pts * 24);
    cudaMalloc(&Li, (size_t)n_pts * 48); cudaMalloc(&tv, (size_t)n_pts * 24);
    cudaMalloc(&sink, (size_t)grid * THREADS * 8); cudaMalloc(&gmax, 8);
    cudaMemset(Dp2, 0, (size_t)n_pts * 24);
    cudaMemcpy(d_xc, xc.data(), xc.size() * 8, cudaMemcpyHostToDevice);
    cudaMemcpy(d_kc, kc.data(), kc.size() * 8, cudaMemcpyHostToDevice);
    cudaMemcpy(d_xp, xp.data(), xp.size() * 8, cudaMemcpyHostToDevice);
    cudaMemcpy(d_flags, flags.data(), n_cams * 4, cudaMemcpyHostToDevice);
    cb::cam_prep_kernel<<<1, 64>>>(d_xc, d_flags, d_kc, n_cams, P, d_tab);
    cb::LmState h{};
    h.lam = 1e-3; h.fscale = 1.0;
    cb::LmState* d_st;
    cudaMalloc(&d_st, sizeof(h));
    cudaMemcpy(d_st, &h, sizeof(h), cudaMemcpyHostToDevice);
    const cb::CPtr2 tab2{{d_tab, d_tab}}, xp2{{d_xp, d_xp}};
    const int smem = cb::CT_SMEM * n_cams * 8;
    auto engine_and_copies = [&](auto engine, auto copy_store, auto copy_sum, int stage_bytes, const char* name) {
      cudaMemset(Zt, 0, zn * sizeof(double));
      report("(e) copy of pt_pass_kernel before staging, piece stores", timed([&] {
        copy_store<<<grid, THREADS, smem>>>(d_st, d_start, d_cam, d_xy, n_pts, n_cams, tab2, xp2, V6, gp, Dp2, Li, tv, Zt, LD, sink);
      }), false);
      cudaMemcpy(Zref, Zt, zn * sizeof(double), cudaMemcpyDeviceToDevice);
      report("(e) the same without its Zt stores", timed([&] {
        copy_sum<<<grid, THREADS, smem>>>(d_st, d_start, d_cam, d_xy, n_pts, n_cams, tab2, xp2, V6, gp, Dp2, Li, tv, Zt, LD, sink);
      }), false);
      // the engine kernel stages its Zt granules after the camera table
      const int esmem = smem + stage_bytes;
      cudaFuncSetAttribute(engine, cudaFuncAttributeMaxDynamicSharedMemorySize, esmem);
      cudaMemset(Zt, 0, zn * sizeof(double));
      report(name, timed([&] {
        engine<<<grid, THREADS, esmem>>>(d_st, d_start, d_cam, d_xy, nullptr, n_pts, n_cams, tab2, xp2, V6, gp, Dp2, Li, tv,
                                         Zt, LD, gmax, nullptr);
      }), true);
    };
    if (P == 6)
      engine_and_copies(cb::pt_pass_kernel<6, 8, false, true>, pt_pass_copy<6, true>, pt_pass_copy<6, false>,
                        (int)cb::pt_stage_bytes<6, 8>(), "(e) engine pt_pass_kernel<6,8,false,true>, whole granules");
    else
      engine_and_copies(cb::pt_pass_kernel<9, 8, false, true>, pt_pass_copy<9, true>, pt_pass_copy<9, false>,
                        (int)cb::pt_stage_bytes<9, 8>(), "(e) engine pt_pass_kernel<9,8,false,true>, whole granules");
    for (void* p : {(void*)d_xc, (void*)d_kc, (void*)d_tab, (void*)d_xp, (void*)V6, (void*)gp, (void*)Dp2, (void*)Li,
                    (void*)tv, (void*)sink, (void*)d_flags, (void*)gmax, (void*)d_st})
      cudaFree(p);
  }
  cudaFree(d_start); cudaFree(d_cam); cudaFree(d_xy); cudaFree(Zt); cudaFree(Zref); cudaFree(d_diff);
}

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  printf("%s, %d SMs, %.0f MB L2\n", prop.name, sms, prop.l2CacheSize / 1048576.0);
  const size_t flush_bytes = 256ull << 20;
  double* flush;
  cudaMalloc(&flush, flush_bytes);
  run_case({"cfg4: a random 40 of 64 cameras per point", 6, 50000, 40, false}, sms, flush, flush_bytes);
  run_case({"cfg4 with free intrinsics: 40 of 64", 9, 50000, 40, false}, sms, flush, flush_bytes);
  run_case({"sparse64-like: 8 adjacent cameras per point", 6, 250000, 8, true}, sms, flush, flush_bytes);
  cudaFree(flush);
  return 0;
}
