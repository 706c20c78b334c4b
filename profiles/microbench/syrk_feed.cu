// Microbenchmark: what limits the dense Schur product S = Zt^T Zt on the cfg4 shape (64 cameras x P = 6 -> 4 column
// tiles of 96, 150 016 k rows; Zt is 461 MB).  A seeded random Zt and the dense item schedule of the engine
// (6 off-diagonal tiles + 2 diagonal pairs, each split over k to fill one CTA per SM), timed with CUDA events:
//   (a) per-item feed: each CTA bulk-copies its two 96-column tiles
//   (b) the same loads, consumers only wait and arrive (no MMA)
//   (c) the MMAs on shared-memory-resident stages (no loads)
// (a)-(c) run a copy of the product as it was with diagonal tiles on m8n8k4; if (c) is about as slow as (a), the MMAs,
// not the feed, set the time, and fetching each column tile once per cluster would not help.  Then
//   (e) the engine's schur_syrk_kernel (cb_kernels.cuh) per item kind, which gives the split weights of
//       build_schur_items, and on the cfg4 schedule built with them;
//   (d) the engine's per-stage math (diagonal tiles on m16n8k16) in the modes of (a)-(c) at that schedule: the same
//       stop test on the kernel as it is now.  The feed alone (loads only) in four variants: (i) one 768-byte row copy
//       per lane per tile, (ii) one 2-D tensor box per tile per stage (what the engine's dense path does), (iii) the row
//       copies of (i) in lock-step chunk order (CTA s of a group of n takes chunks s, s + n, ...: every group sweeps k at
//       the same pace, so a row's readers meet in L2), and (ii) in that order.  Last, the MMAs alone on a schedule
//       weighted by MMA-only costs: the product's MMA bound.
// Prints us per launch, GB/s of global -> shared feed and TFLOP/s of issued MMA work.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o syrk_feed syrk_feed.cu && ./syrk_feed
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <vector>

#include "../../caliscope_b200/csrc/cb_kernels.cuh"

using cb::bulk_g2s;
using cb::mbar_arrive;
using cb::mbar_expect_tx;
using cb::mbar_fence_init;
using cb::mbar_init;
using cb::mbar_wait;

constexpr int TILE = 96, LDS = TILE + 4, NB = 4, LD = NB * TILE, N_PTS = 50000;
constexpr int STAGES = 4, CWARPS = 8, THREADS = 32 * (CWARPS + 1);

__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__device__ __forceinline__ void dmma16816(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
               "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]),
                 "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

struct Item { int kind, I, J, c0, c1; };

// ---------------------------------------------------------------------------------------------
// (a)-(c): the per-item feed (k chunks of 32 rows, two 96-column tiles per stage)
// MODE 0: loads + MMA, 1: loads only, 2: MMA only
// ---------------------------------------------------------------------------------------------
constexpr int KC_OLD = 32;
struct OldSmem {
  double A[STAGES][KC_OLD * LDS];
  double B[STAGES][KC_OLD * LDS];
  unsigned long long full[STAGES], empty[STAGES];
};
__constant__ signed char DIAG_BLOCKS[8][3][3] = {
    {{0, 0, 0}, {0, 0, 1}, {0, 0, 2}}, {{0, 0, 3}, {0, 1, 3}, {0, 2, 3}}, {{0, 1, 1}, {0, 1, 2}, {0, 2, 2}},
    {{0, 3, 3}, {1, 3, 3}, {1, 2, 2}}, {{1, 0, 0}, {1, 0, 1}, {-1, 0, 0}}, {{1, 0, 2}, {1, 0, 3}, {-1, 0, 0}},
    {{1, 1, 1}, {1, 1, 2}, {-1, 0, 0}}, {{1, 1, 3}, {1, 2, 3}, {-1, 0, 0}}};

template <int MODE>
__global__ void __launch_bounds__(THREADS, 1) old_feed(const double* __restrict__ Zt, const Item* __restrict__ items,
                                                       double* __restrict__ out) {
  extern __shared__ __align__(128) unsigned char raw[];
  OldSmem& sm = *reinterpret_cast<OldSmem*>(raw);
  const Item item = items[blockIdx.x];
  const bool diag = item.kind == 1;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, fr = lane >> 2, fk = lane & 3;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], CWARPS); }
    mbar_fence_init();
  }
  __syncthreads();
  const int n_it = item.c1 - item.c0;
  const uint32_t row_bytes = TILE * 8;
  if (wid == CWARPS) {
    if constexpr (MODE != 2) {
      for (int it = 0; it < n_it; ++it) {
        const int stage = it % STAGES, round = it / STAGES;
        if (round > 0) mbar_wait(&sm.empty[stage], (uint32_t)((round - 1) & 1));
        const size_t k = (size_t)(item.c0 + it) * KC_OLD + lane;
        if (lane == 0) mbar_expect_tx(&sm.full[stage], 2 * KC_OLD * row_bytes);
        __syncwarp();
        bulk_g2s(&sm.A[stage][lane * LDS], Zt + k * LD + (size_t)item.I * TILE, row_bytes, &sm.full[stage]);
        bulk_g2s(&sm.B[stage][lane * LDS], Zt + k * LD + (size_t)item.J * TILE, row_bytes, &sm.full[stage]);
      }
    }
    return;
  }
  double sum = 0.0;
  if (!diag) {
    const int wr = wid >> 2, wc = wid & 3;
    double acc[3][3][4] = {};
    for (int it = 0; it < n_it; ++it) {
      const int stage = it % STAGES;
      if (MODE != 2) mbar_wait(&sm.full[stage], (uint32_t)((it / STAGES) & 1));
      if (MODE != 1) {
        const double* As = sm.A[stage] + fk * LDS + wr * 48 + fr;
        const double* Bs = sm.B[stage] + fk * LDS + wc * 24 + fr;
#pragma unroll
        for (int ks = 0; ks < KC_OLD / 16; ++ks) {
          double a[3][8], b[3][4];
#pragma unroll
          for (int u = 0; u < 3; ++u)
#pragma unroll
            for (int i = 0; i < 8; ++i) a[u][i] = As[(ks * 16 + 4 * (i >> 1)) * LDS + u * 16 + 8 * (i & 1)];
#pragma unroll
          for (int v = 0; v < 3; ++v)
#pragma unroll
            for (int j = 0; j < 4; ++j) b[v][j] = Bs[(ks * 16 + 4 * j) * LDS + v * 8];
#pragma unroll
          for (int u = 0; u < 3; ++u)
#pragma unroll
            for (int v = 0; v < 3; ++v) dmma16816(acc[u][v], a[u], b[v]);
        }
      }
      __syncwarp();
      if (MODE != 2 && lane == 0) mbar_arrive(&sm.empty[stage]);
    }
#pragma unroll
    for (int u = 0; u < 3; ++u)
#pragma unroll
      for (int v = 0; v < 3; ++v) sum += acc[u][v][0] + acc[u][v][1] + acc[u][v][2] + acc[u][v][3];
  } else {
    double acc[3][3][3][2] = {};
    for (int it = 0; it < n_it; ++it) {
      const int stage = it % STAGES;
      if (MODE != 2) mbar_wait(&sm.full[stage], (uint32_t)((it / STAGES) & 1));
      if (MODE != 1) {
#pragma unroll
        for (int ks = 0; ks < KC_OLD / 4; ++ks)
#pragma unroll
          for (int b = 0; b < 3; ++b) {
            const int sel = DIAG_BLOCKS[wid][b][0], br = DIAG_BLOCKS[wid][b][1], bc = DIAG_BLOCKS[wid][b][2];
            if (sel < 0) continue;
            const double* T = (sel == 0 ? sm.A[stage] : sm.B[stage]) + (ks * 4 + fk) * LDS + fr;
            double a[3], bb[3];
#pragma unroll
            for (int u = 0; u < 3; ++u) a[u] = T[br * 24 + u * 8];
#pragma unroll
            for (int v = 0; v < 3; ++v) bb[v] = T[bc * 24 + v * 8];
#pragma unroll
            for (int u = 0; u < 3; ++u)
#pragma unroll
              for (int v = 0; v < 3; ++v) dmma884(acc[b][u][v][0], acc[b][u][v][1], a[u], bb[v]);
          }
      }
      __syncwarp();
      if (MODE != 2 && lane == 0) mbar_arrive(&sm.empty[stage]);
    }
#pragma unroll
    for (int b = 0; b < 3; ++b)
#pragma unroll
      for (int u = 0; u < 3; ++u)
#pragma unroll
        for (int v = 0; v < 3; ++v) sum += acc[b][u][v][0] + acc[b][u][v][1];
  }
  out[(size_t)blockIdx.x * THREADS + tid] = sum;
}

// ---------------------------------------------------------------------------------------------
// (d): the engine's product (cb::schur_syrk_kernel: same shared-memory ring, same producer, the per-stage MMAs of
// cb::syrk_offdiag_stage / cb::syrk_diag_stage, diagonal tiles on m16n8k16) with the same three modes as (a)-(c):
// MODE 0: loads + MMA, 1: loads only, 2: MMA only.  Z t and the output stores are left out (one store per thread).
// ---------------------------------------------------------------------------------------------
// BOX: the producer loads a stage with one 2-D tensor box per tile (as the engine's dense path does) instead of one
// 768-byte row copy per lane per tile.  CTA b walks chunks c0, c0 + cstep[b], ... below c1.
template <int MODE, bool BOX = false>
__global__ void __launch_bounds__(cb::SY_THREADS, 1) engine_feed(const __grid_constant__ CUtensorMap zt_map,
                                                                const double* __restrict__ Zt,
                                                                const cb::SyItem* __restrict__ items,
                                                                const int* __restrict__ cstep,
                                                                double* __restrict__ out) {
  extern __shared__ __align__(128) unsigned char raw[];
  cb::SyrkSmem& sm = *reinterpret_cast<cb::SyrkSmem*>(raw);
  const cb::SyItem item = items[blockIdx.x];
  const bool diag = item.kind == 1, two = diag ? item.J >= 0 : true;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, fr = lane >> 2, fk = lane & 3;
  if (tid == 0) {
    for (int s = 0; s < cb::SY_STAGES; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], cb::SY_CONSUMER_WARPS); }
    mbar_fence_init();
  }
  __syncthreads();
  const int step = cstep[blockIdx.x], n_it = (item.c1 - item.c0 + step - 1) / step;
  const uint32_t row_bytes = TILE * 8;
  if (wid == cb::SY_CONSUMER_WARPS) {
    if constexpr (MODE != 2) {
      for (int it = 0; it < n_it; ++it) {
        const int stage = it % cb::SY_STAGES, round = it / cb::SY_STAGES, chunk = item.c0 + it * step;
        if (round > 0) mbar_wait(&sm.empty[stage], (uint32_t)((round - 1) & 1));
        if constexpr (BOX) {
          if (lane == 0) {
            mbar_expect_tx(&sm.full[stage], cb::SY_KC * LDS * 8 * (two ? 2u : 1u));
            cb::tma_load_2d(sm.A[stage], &zt_map, item.I * TILE, chunk * cb::SY_KC, &sm.full[stage]);
            if (two) cb::tma_load_2d(sm.B[stage], &zt_map, item.J * TILE, chunk * cb::SY_KC, &sm.full[stage]);
          }
        } else {
          const size_t k = (size_t)chunk * cb::SY_KC + lane;
          if (lane == 0) mbar_expect_tx(&sm.full[stage], cb::SY_KC * row_bytes * (two ? 2u : 1u));
          __syncwarp();
          bulk_g2s(&sm.A[stage][lane * LDS], Zt + k * LD + (size_t)item.I * TILE, row_bytes, &sm.full[stage]);
          if (two) bulk_g2s(&sm.B[stage][lane * LDS], Zt + k * LD + (size_t)item.J * TILE, row_bytes, &sm.full[stage]);
        }
      }
    }
    return;
  }
  double sum = 0.0;
  if (!diag) {
    double acc[3][3][4] = {};
    for (int it = 0; it < n_it; ++it) {
      const int stage = it % cb::SY_STAGES;
      if (MODE != 2) mbar_wait(&sm.full[stage], (uint32_t)((it / cb::SY_STAGES) & 1));
      if (MODE != 1) cb::syrk_offdiag_stage(acc, sm.A[stage], sm.B[stage], wid >> 2, wid & 3, fr, fk);
      __syncwarp();
      if (MODE != 2 && lane == 0) mbar_arrive(&sm.empty[stage]);
    }
    for (int u = 0; u < 3; ++u)
      for (int v = 0; v < 3; ++v) sum += acc[u][v][0] + acc[u][v][1] + acc[u][v][2] + acc[u][v][3];
  } else {
    const cb::SyDiagRuns run = cb::SY_DIAG_RUNS[two ? 0 : 1][wid];
    double acc[cb::SY_DIAG_MAX][4] = {};
    for (int it = 0; it < n_it; ++it) {
      const int stage = it % cb::SY_STAGES;
      if (MODE != 2) mbar_wait(&sm.full[stage], (uint32_t)((it / cb::SY_STAGES) & 1));
      if (MODE != 1) cb::syrk_diag_stage(acc, run.sel == 0 ? sm.A[stage] : sm.B[stage], run, fr, fk);
      __syncwarp();
      if (MODE != 2 && lane == 0) mbar_arrive(&sm.empty[stage]);
    }
    for (int j = 0; j < cb::SY_DIAG_MAX; ++j) sum += acc[j][0] + acc[j][1] + acc[j][2] + acc[j][3];
  }
  out[(size_t)blockIdx.x * THREADS + tid] = sum;
}

// ---------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------
__global__ void fill_kernel(double* z, size_t n, unsigned long long seed) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    unsigned long long x = (i + 1) * 0x9E3779B97F4A7C15ull ^ seed;
    x ^= x >> 31; x *= 0xBF58476D1CE4E5B9ull; x ^= x >> 27;
    z[i] = (double)(x >> 11) * 0x1.0p-53 - 0.5;
  }
}

// dense cfg4 schedule of the per-item feed: CTAs per group in proportion to its weight, leftovers to the heaviest
static std::vector<Item> old_items(int sms, int k_chunks, double w_pair) {
  struct G { int kind, I, J; double w; };
  std::vector<G> g;
  for (int I = 0; I < NB; ++I)
    for (int J = I + 1; J < NB; ++J) g.push_back({0, I, J, 1.0});
  for (int I = 0; I < NB; I += 2) g.push_back({1, I, I + 1, w_pair});
  double W = 0.0;
  for (auto& x : g) W += x.w;
  std::vector<int> n(g.size());
  int used = 0;
  for (size_t i = 0; i < g.size(); ++i) used += n[i] = std::max(1, (int)std::floor(sms * g[i].w / W));
  while (used < sms) {
    size_t best = 0;
    for (size_t i = 1; i < g.size(); ++i)
      if (g[i].w / n[i] > g[best].w / n[best]) best = i;
    ++n[best]; ++used;
  }
  std::vector<Item> items;
  for (size_t i = 0; i < g.size(); ++i)
    for (int s = 0; s < n[i]; ++s)
      items.push_back({g[i].kind, g[i].I, g[i].J, (int)((long long)k_chunks * s / n[i]),
                       (int)((long long)k_chunks * (s + 1) / n[i])});
  return items;
}

template <typename F>
static float time_ms(F f, int reps) {
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  f(); f();
  cudaDeviceSynchronize();
  cudaEventRecord(e0);
  for (int r = 0; r < reps; ++r) f();
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) { printf("CUDA error: %s\n", cudaGetErrorString(err)); return NAN; }
  return ms / reps;
}

static void report(const char* name, float ms, double bytes, double flop) {
  printf("%-52s %8.1f us  %7.0f GB/s feed  %6.2f TFLOP/s\n", name, ms * 1e3, bytes / (ms * 1e-3) * 1e-9,
         flop / (ms * 1e-3) * 1e-12);
}

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  printf("%s, %d SMs, %.0f MB L2\n", prop.name, sms, prop.l2CacheSize / 1048576.0);
  const int K_pad = (3 * N_PTS + KC_OLD - 1) / KC_OLD * KC_OLD;
  const size_t zn = ((size_t)K_pad + KC_OLD) * LD;
  double *Zt, *out;
  cudaMalloc(&Zt, zn * sizeof(double));
  cudaMalloc(&out, (size_t)sms * 16 * THREADS * sizeof(double));
  fill_kernel<<<1024, 256>>>(Zt, zn, 12345);
  printf("Zt: %d x %d doubles = %.1f MB\n", K_pad, LD, (double)K_pad * LD * 8 * 1e-6);
  const int reps = 20;

  {
    const std::vector<Item> items = old_items(sms, K_pad / KC_OLD, 1.55);
    Item* d_items;
    cudaMalloc(&d_items, items.size() * sizeof(Item));
    cudaMemcpy(d_items, items.data(), items.size() * sizeof(Item), cudaMemcpyHostToDevice);
    double bytes = 0.0, flop = 0.0;
    for (auto& it : items) {
      bytes += 2.0 * (it.c1 - it.c0) * KC_OLD * TILE * 8;
      flop += 2.0 * (it.kind == 0 ? 96.0 * 96.0 : 20.0 * 24 * 24) * (it.c1 - it.c0) * KC_OLD;
    }
    const int smem = sizeof(OldSmem);
    cudaFuncSetAttribute(old_feed<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(old_feed<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(old_feed<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    const int grid = (int)items.size();
    report("(a) per-item feed, loads + MMA", time_ms([&] { old_feed<0><<<grid, THREADS, smem>>>(Zt, d_items, out); }, reps),
           bytes, flop);
    report("(b) per-item feed, loads only", time_ms([&] { old_feed<1><<<grid, THREADS, smem>>>(Zt, d_items, out); }, reps),
           bytes, 0.0);
    report("(c) MMA on resident stages, no loads", time_ms([&] { old_feed<2><<<grid, THREADS, smem>>>(Zt, d_items, out); }, reps),
           0.0, flop);
    // relative cost per k chunk of a diagonal-pair CTA vs an off-diagonal one (MMA only): the split weight
    std::vector<Item> off(sms, Item{0, 0, 1, 0, 256}), pair(sms, Item{1, 0, 1, 0, 256});
    Item* d_w;
    cudaMalloc(&d_w, sms * sizeof(Item));
    cudaMemcpy(d_w, off.data(), sms * sizeof(Item), cudaMemcpyHostToDevice);
    const float t_off = time_ms([&] { old_feed<2><<<sms, THREADS, smem>>>(Zt, d_w, out); }, reps);
    cudaMemcpy(d_w, pair.data(), sms * sizeof(Item), cudaMemcpyHostToDevice);
    const float t_pair = time_ms([&] { old_feed<2><<<sms, THREADS, smem>>>(Zt, d_w, out); }, reps);
    printf("per-item feed: diagonal pair / off-diagonal CTA cost (MMA only) = %.3f\n", t_pair / t_off);
    printf("feed bytes per launch: %.3f GB\n", bytes * 1e-9);
    cudaFree(d_w);
    cudaFree(d_items);
  }
  {
    // (e) the engine's schur_syrk_kernel (diagonal tiles on m16n8k16, dense items fed by tensor boxes): cost per k chunk
    // of each item kind, one CTA per SM, which sets build_schur_items' split weights; then the cfg4 schedule built with
    // those weights
    cb::LmState h_st{};
    cb::LmState* d_st;
    cudaMalloc(&d_st, sizeof(cb::LmState));
    cudaMemcpy(d_st, &h_st, sizeof(cb::LmState), cudaMemcpyHostToDevice);
    double *part, *tpart;
    cudaMalloc(&part, (size_t)2 * sms * TILE * TILE * sizeof(double));
    cudaMalloc(&tpart, (size_t)2 * sms * TILE * sizeof(double));
    CUtensorMap zmap;
    if (cb::make_zt_tensor_map(&zmap, Zt, LD, (size_t)K_pad + KC_OLD) != cudaSuccess) {
      printf("tensor map encoding failed\n");
      return 1;
    }
    const int smem = sizeof(cb::SyrkSmem);
    cudaFuncSetAttribute(cb::schur_syrk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cb::SyItem* d_it;
    cudaMalloc(&d_it, 2 * sms * sizeof(cb::SyItem));
    auto run = [&](const std::vector<cb::SyItem>& v) {
      cudaMemcpy(d_it, v.data(), v.size() * sizeof(cb::SyItem), cudaMemcpyHostToDevice);
      return time_ms([&] {
        cb::schur_syrk_kernel<<<(int)v.size(), cb::SY_THREADS, smem>>>(zmap, d_st, Zt, LD, Zt, d_it, nullptr, part, tpart);
      }, reps);
    };
    auto mk = [&](int kind, int I, int J, int c0, int c1, int s) { return cb::SyItem{kind, I, J, c0, c1, s, s + sms, -1}; };
    const int ch = 256;
    std::vector<cb::SyItem> off, pair, single;
    for (int s = 0; s < sms; ++s) {
      off.push_back(mk(0, 0, 1, 0, ch, s));
      pair.push_back(mk(1, 0, 1, 0, ch, s));
      single.push_back(mk(1, 0, -1, 0, ch, s));
    }
    const float t_off = run(off), t_pair = run(pair), t_single = run(single);
    const double fl_off = 2.0 * 96 * 96 * ch * KC_OLD * sms;
    report("(e) engine kernel, off-diagonal CTAs only", t_off, 2.0 * ch * KC_OLD * TILE * 8 * sms, fl_off);
    report("(e) engine kernel, diagonal-pair CTAs only", t_pair, 2.0 * ch * KC_OLD * TILE * 8 * sms, fl_off * 84 / 72);
    report("(e) engine kernel, single-diagonal CTAs only", t_single, 1.0 * ch * KC_OLD * TILE * 8 * sms, fl_off * 42 / 72);
    printf("engine kernel: diagonal pair / off-diagonal = %.3f, single diagonal / off-diagonal = %.3f\n", t_pair / t_off,
           t_single / t_off);
    // cfg4 schedule at pair weight w: contiguous k slabs per CTA, or lock-step (CTA s of a group of n takes chunks s,
    // s + n, s + 2n, ...: every group sweeps k at the same pace, so a row's readers meet in L2)
    double bytes = 0.0, flop = 0.0;
    std::vector<int> steps;  // cstep of engine_feed, per CTA, for the schedule sched() built last
    auto sched = [&](double w, bool lockstep) {
      const std::vector<Item> g = old_items(sms, K_pad / KC_OLD, w);
      std::vector<cb::SyItem> v;
      steps.clear();
      bytes = flop = 0.0;
      for (size_t i = 0; i < g.size();) {
        size_t e = i;
        while (e < g.size() && g[e].kind == g[i].kind && g[e].I == g[i].I && g[e].J == g[i].J) ++e;
        const int n = (int)(e - i);
        for (size_t q = i; q < e; ++q) {
          const Item& x = g[q];
          v.push_back(lockstep ? mk(x.kind, x.I, x.J, (int)(q - i), K_pad / KC_OLD, (int)q)
                               : mk(x.kind, x.I, x.J, x.c0, x.c1, (int)q));
          steps.push_back(lockstep ? n : 1);
          bytes += 2.0 * (x.c1 - x.c0) * KC_OLD * TILE * 8;
          flop += 2.0 * (x.kind == 0 ? 96.0 * 96.0 : 84.0 * 16 * 8) * (x.c1 - x.c0) * KC_OLD;
        }
        i = e;
      }
      return v;
    };
    report("(e) engine kernel, cfg4 schedule at w_pair 1.31", run(sched(1.31, false)), bytes, flop);
    const std::vector<cb::SyItem> vl = sched(t_pair / t_off, true);
    const std::vector<int> steps_l = steps;
    const std::vector<cb::SyItem> v = sched(t_pair / t_off, false);
    report("(e) engine kernel, cfg4 schedule at the measured weight", run(v), bytes, flop);
    // (d) the stop test of (a)-(c) repeated on the engine's math at that schedule, and the feed alone (loads only):
    //   (i) row copies, (ii) one tensor box per tile per stage, (iii) row copies in lock-step order, and boxes in lock-step
    cudaFuncSetAttribute(engine_feed<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(engine_feed<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(engine_feed<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(engine_feed<0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(engine_feed<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    int* d_step;
    cudaMalloc(&d_step, 2 * sms * sizeof(int));
    auto run_mode = [&](int mode, const std::vector<cb::SyItem>& items, const std::vector<int>* st = nullptr) {
      const std::vector<int> ones(items.size(), 1);
      cudaMemcpy(d_it, items.data(), items.size() * sizeof(cb::SyItem), cudaMemcpyHostToDevice);
      cudaMemcpy(d_step, (st ? *st : ones).data(), items.size() * sizeof(int), cudaMemcpyHostToDevice);
      const int g = (int)items.size();
      return time_ms([&] {
        if (mode == 0) engine_feed<0><<<g, cb::SY_THREADS, smem>>>(zmap, Zt, d_it, d_step, out);
        else if (mode == 1) engine_feed<1><<<g, cb::SY_THREADS, smem>>>(zmap, Zt, d_it, d_step, out);
        else if (mode == 2) engine_feed<2><<<g, cb::SY_THREADS, smem>>>(zmap, Zt, d_it, d_step, out);
        else if (mode == 3) engine_feed<0, true><<<g, cb::SY_THREADS, smem>>>(zmap, Zt, d_it, d_step, out);
        else engine_feed<1, true><<<g, cb::SY_THREADS, smem>>>(zmap, Zt, d_it, d_step, out);
      }, reps);
    };
    report("(d) engine math, cfg4 schedule, loads + MMA (row copies)", run_mode(0, v), bytes, flop);
    report("(d) engine math, cfg4 schedule, loads + MMA (boxes)", run_mode(3, v), bytes, flop);
    report("(d) engine math, lock-step schedule, loads + MMA (row copies)", run_mode(0, vl, &steps_l), bytes, flop);
    report("(d) engine math, lock-step schedule, loads + MMA (boxes)", run_mode(3, vl, &steps_l), bytes, flop);
    report("(d)(i) loads only, row copies", run_mode(1, v), bytes, 0.0);
    report("(d)(ii) loads only, tensor boxes", run_mode(4, v), bytes, 0.0);
    report("(d)(iii) loads only, row copies, lock-step", run_mode(1, vl, &steps_l), bytes, 0.0);
    report("(d)(ii+iii) loads only, tensor boxes, lock-step", run_mode(4, vl, &steps_l), bytes, 0.0);
    report("(d) engine math, cfg4 schedule, MMA only", run_mode(2, v), 0.0, flop);
    const float m_off = run_mode(2, off), m_pair = run_mode(2, pair), m_single = run_mode(2, single);
    report("(d) engine math, off-diagonal CTAs only, MMA only", m_off, 0.0, fl_off);
    report("(d) engine math, diagonal-pair CTAs only, MMA only", m_pair, 0.0, fl_off * 84 / 72);
    report("(d) engine math, single-diagonal CTAs only, MMA only", m_single, 0.0, fl_off * 42 / 72);
    printf("engine math, MMA only: diagonal pair / off-diagonal = %.3f, single diagonal / off-diagonal = %.3f\n",
           m_pair / m_off, m_single / m_off);
    // the MMA bound of the product: MMA only on a schedule weighted by MMA-only costs
    const std::vector<cb::SyItem> vm = sched(m_pair / m_off, false);
    report("(d) engine math, schedule at the MMA-only weight, MMA only", run_mode(2, vm), 0.0, flop);
    cudaFree(d_step); cudaFree(d_it); cudaFree(part); cudaFree(tpart); cudaFree(d_st);
  }
  cudaFree(Zt);
  cudaFree(out);
  return 0;
}
