// Stand-alone harness for the K1 tensor-core leapfrog kernel (mici_b200/csrc/leapfrog_dmma.cuh):
// C1-shaped synthetic input (8192 chains x 128, funnel target, SPD metric), CUDA-event timing of
// 50- and 200-step launches, a checksum to compare variants, and (with -DK1_TRACE) a per-warp
// phase timeline of CTA 0 (clock64 at the phase boundaries marked MB200_K1_TRACE in the kernel).
// With -DK1_AB the binary also holds the previous generation of the kernel
// (profiles/experiments/leapfrog_dmma4.cuh, `leapfrog_dmma4_kernel`) and compares the two in one
// process: alternating launches at 50 and 200 steps, median per launch and per-step slope of
// each, and the largest ulp difference of q, p and h between them (with -DK1_TRACE as well, the
// phase tables of both).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -fmad=false -lineinfo \
//        [-DK1_TRACE] [-DK1_AB] -o k1_bench k1_bench.cu
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <vector>
#include <cuda_runtime.h>

#ifdef K1_TRACE
#include <algorithm>
// phases: 0 drift start, 1 drift issued, 6 first accumulator value read (the DMMAs have drained),
// 2 partials written, 3 reduce barrier passed, 4 kick done, 5 publish barrier passed
constexpr int TR_STEPS = 8, TR_PHASES = 7, TR_WARPS = 32;
__device__ long long g_trace[TR_WARPS][TR_STEPS][TR_PHASES];
#define MB200_K1_TRACE(phase)                                                          \
  do {                                                                                 \
    if (blockIdx.x == 0 && (threadIdx.x & 31) == 0 && s >= 20 && s < 20 + TR_STEPS)    \
      g_trace[threadIdx.x >> 5][s - 20][phase] = clock64();                            \
  } while (0)
// the empty asm makes x an operand that must exist before the clock is read, so the timestamp
// follows the instruction that computes x
// the same for step s - 1 (the barrier that closes a step's update phase, passed in the next
// step's drift)
#define MB200_K1_TRACE_PREV(phase)                                                     \
  do {                                                                                 \
    if (blockIdx.x == 0 && (threadIdx.x & 31) == 0 && s >= 21 && s < 21 + TR_STEPS)    \
      g_trace[threadIdx.x >> 5][s - 21][phase] = clock64();                            \
  } while (0)
#define MB200_K1_TRACE_AFTER(phase, x)                                                 \
  do {                                                                                 \
    asm volatile("" ::"d"(x));                                                         \
    MB200_K1_TRACE(phase);                                                             \
  } while (0)
__device__ long long g_mark[2][8];
__device__ unsigned long long g_gt[2][8];
#define MB200_K1_MARK(id)                                                              \
  do {                                                                                 \
    if ((blockIdx.x == 0 || blockIdx.x == 100) && threadIdx.x == 0) {                  \
      unsigned long long gt;                                                           \
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));                           \
      g_mark[blockIdx.x == 100][id] = clock64();                                       \
      g_gt[blockIdx.x == 100][id] = gt;                                                \
    }                                                                                  \
  } while (0)
#endif
// K1's host launcher (k1_launch) and its kernel, as the library builds them
#include "../../mici_b200/csrc/api_dmma.cu"
#ifdef K1_AB
#include <algorithm>
#include <cstring>
#include "../experiments/leapfrog_dmma4.cuh"
#endif

using namespace mb200;

#ifdef K1_AB
// k1_run of api_dmma.cu with the previous generation's kernel (shared step size)
template <class Target, int DP>
static int k1_run_dmma4(const EuclidArgs& a) {
  const int sms = num_sms();
  const int64_t total_tiles = (a.n + 7) / 8;
  int64_t tpc = (total_tiles + sms - 1) / sms;
  if (tpc > DMMA_TILES_PER_CTA) tpc = DMMA_TILES_PER_CTA;
  auto al16 = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
  const int even = (a.dim & 1) == 0;
  const int vec2 = even && al16(a.q_in) && al16(a.p_in) && al16(a.q_out) && al16(a.p_out);
  const int tma_rows = even && al16(a.minv);
  return eu_launch(leapfrog_dmma4_kernel<Target, DP, false>, "leapfrog_dmma4_kernel",
                   (total_tiles + tpc - 1) / tpc, 1, DMMA_THREADS, sizeof(DmmaSmem<DP>), a.st,
                   a.q_in, a.p_in, a.q_out, a.p_out, a.dir, a.sched.step_sizes, a.n, a.dim, a.eps,
                   a.n_steps, a.minv, a.m, a.h_out, a.status, a.n_done, (int)tpc, vec2, tma_rows);
}
template <class Target>
static int k1_launch_dmma4(const EuclidArgs& a) {
  if (a.dim <= 32) return k1_run_dmma4<Target, 32>(a);
  if (a.dim <= 64) return k1_run_dmma4<Target, 64>(a);
  if (a.dim <= 96) return k1_run_dmma4<Target, 96>(a);
  return k1_run_dmma4<Target, 128>(a);
}
// distance in units in the last place between two doubles (0 for equal values, also +0 / -0)
static int64_t ulp_diff(double a, double b) {
  auto key = [](double x) {
    int64_t i;
    std::memcpy(&i, &x, 8);
    return i < 0 ? INT64_MIN - i : i;  // monotonic in x
  };
  const int64_t ka = key(a), kb = key(b);
  return ka > kb ? ka - kb : kb - ka;
}
#endif

#ifdef K1_TRACE
// marks and phase timeline of the last launch (200 steps)
static void print_trace(const char* kernel) {
  printf("==== trace of %s\n", kernel);
  {
    long long mk[2][8];
    unsigned long long gt[2][8];
    cudaMemcpyFromSymbol(mk, g_mark, sizeof(mk));
    cudaMemcpyFromSymbol(gt, g_gt, sizeof(gt));
    printf("marks of the last launch (200 steps), thread 0 of CTA 0 / CTA 100: 0 kernel start, 1 smem zeroed, "
           "2 A landed, 3 A scaled, 4 state loaded, 5 first kick done, 6 steps done, 7 stored\n");
    for (int b = 0; b < 2; ++b) {
      printf("CTA %3d cycles:", b ? 100 : 0);
      for (int i = 0; i < 8; ++i) printf(" %9lld", mk[b][i] - mk[b][0]);
      printf("\n        ns    :");
      for (int i = 0; i < 8; ++i) printf(" %9lld", (long long)(gt[b][i] - gt[0][0]));
      printf("\n");
    }
  }
  {
    static long long tr[TR_WARPS][TR_STEPS][TR_PHASES];
    cudaMemcpyFromSymbol(tr, g_trace, sizeof(tr));
    long long t0 = tr[0][0][0];
    for (int w = 0; w < DMMA_THREADS / 32; ++w)
      for (int s = 0; s < TR_STEPS; ++s)
        if (tr[w][s][0] < t0 && tr[w][s][0] > 0) t0 = tr[w][s][0];
    printf("trace (CTA 0, cycles relative to first event; phases: 0 drift start, 1 drift issued, "
           "2 partials written, 3 reduce barrier passed, 4 kick done, 5 publish barrier passed, "
           "6 first accumulator value read)\n");
    for (int w = 0; w < DMMA_THREADS / 32; ++w)
      for (int s = 0; s < TR_STEPS; ++s) {
        printf("w%02d sp%d g%d s%d:", w, w & 3, w >> 2, s);
        for (int ph = 0; ph < TR_PHASES; ++ph) printf(" %7lld", tr[w][s][ph] - t0);
        printf("\n");
      }
    // median cycles of each sub-phase, by group and by the warp that holds coordinate 0 (the
    // kernel's w == 0) versus the other three
    auto median = [](std::vector<long long> v) {
      if (v.empty()) return 0.0;
      std::sort(v.begin(), v.end());
      const size_t n = v.size();
      return n & 1 ? (double)v[n / 2] : 0.5 * (v[n / 2 - 1] + v[n / 2]);
    };
    // {from, to} phase pairs; step = drift start to the next step's drift start
    const int sub[][2] = {{0, 1}, {1, 6}, {6, 2}, {2, 3}, {3, 4}, {4, 5}, {6, 5}, {0, 6}};
    const char* names[] = {"drift issue", "DMMA drain", "partials", "wait bar1",
                           "kick", "wait bar2", "update", "drift+drain"};
    const int n_sub = 8;
    const int groups = DMMA_THREADS / 128;
    printf("update sub-phases (median cycles over steps 20-%d):\n%-14s", 20 + TR_STEPS - 2, "");
    for (int i = 0; i < n_sub; ++i) printf(" %11s", names[i]);
    printf(" %11s\n", "step");
    for (int g = -1; g < groups; ++g)
      for (int kind = 0; kind < 3; ++kind) {
        if ((g < 0) != (kind == 2)) continue;  // per group: w0 / others; overall: all warps
        std::vector<long long> d[n_sub + 1];
        for (int wp = 0; wp < DMMA_THREADS / 32; ++wp) {
          const int grp = wp >> 2, w = ((wp & 3) + grp) & 3;  // the kernel's quarter rotation
          if (g >= 0 && (grp != g || (w == 0) != (kind == 0))) continue;
          for (int s = 0; s + 1 < TR_STEPS; ++s) {
            for (int i = 0; i < n_sub; ++i)
              d[i].push_back(tr[wp][s][sub[i][1]] - tr[wp][s][sub[i][0]]);
            d[n_sub].push_back(tr[wp][s + 1][0] - tr[wp][s][0]);
          }
        }
        char label[32];
        if (g < 0) snprintf(label, sizeof(label), "all warps");
        else snprintf(label, sizeof(label), "g%d %s", g, kind == 0 ? "w0" : "others");
        printf("%-14s", label);
        for (int i = 0; i <= n_sub; ++i) printf(" %11.0f", median(d[i]));
        printf("\n");
      }
    // how far apart the groups are: the spread (latest - earliest) over the groups of the group's
    // drift start (earliest warp), its last arrival at each barrier and its release.  A group may
    // run a whole step ahead of the others, so each group's event is the one nearest in time to
    // group 0's, not the one with the same step index.
    const int ev[][2] = {{0, 0}, {2, 1}, {3, 0}, {4, 1}, {5, 0}};  // {phase, 1: latest warp}
    const char* ev_names[] = {"drift start", "bar1 arrival", "bar1 release", "bar2 arrival",
                              "bar2 release"};
    auto group_event = [&](int g, int s, int e) {
      long long t = ev[e][1] ? -(1LL << 62) : (1LL << 62);
      for (int k = 0; k < 4; ++k) {
        const long long x = tr[4 * g + k][s][ev[e][0]];
        t = ev[e][1] ? std::max(t, x) : std::min(t, x);
      }
      return t;
    };
    printf("group skew (median over steps of max - min over the groups, cycles):");
    for (int e = 0; e < 5; ++e) {
      std::vector<long long> spread;
      for (int s = 1; s + 1 < TR_STEPS; ++s) {
        const long long ref = group_event(0, s, e);
        long long lo = ref, hi = ref;
        for (int g = 1; g < groups; ++g) {
          long long best = group_event(g, 0, e);
          for (int s2 = 1; s2 < TR_STEPS; ++s2) {
            const long long t = group_event(g, s2, e);
            if (std::llabs(t - ref) < std::llabs(best - ref)) best = t;
          }
          lo = std::min(lo, best), hi = std::max(hi, best);
        }
        spread.push_back(hi - lo);
      }
      printf("  %s %.0f", ev_names[e], median(spread));
    }
    printf("\n");
  }
}
#endif

int main(int argc, char** argv) {
  const int64_t n = argc > 1 ? atoll(argv[1]) : 8192;
  const int dim = argc > 2 ? atoi(argv[2]) : 128;
  std::vector<double> q(n * dim), p(n * dim), minv(dim * dim);
  srand(1234);
  auto rnd = [] { return (rand() / (double)RAND_MAX - 0.5) * 2.0; };
  for (auto& v : q) v = 0.1 * rnd();
  for (auto& v : p) v = rnd();
  // SPD "M^-1": I + G G^T / dim
  std::vector<double> g(dim * dim);
  for (auto& v : g) v = rnd();
  for (int i = 0; i < dim; ++i)
    for (int j = 0; j < dim; ++j) {
      double s = (i == j) ? 1.0 : 0.0;
      for (int k = 0; k < dim; ++k) s += g[i * dim + k] * g[j * dim + k] / dim;
      minv[i * dim + j] = s;
    }
  for (int i = 0; i < dim; ++i)
    for (int j = 0; j < i; ++j) minv[i * dim + j] = minv[j * dim + i];
  double *dq, *dp, *dqo, *dpo, *dm, *dh;
  int32_t *dst, *dnd;
  cudaMalloc(&dq, n * dim * 8), cudaMalloc(&dp, n * dim * 8), cudaMalloc(&dqo, n * dim * 8);
  cudaMalloc(&dpo, n * dim * 8), cudaMalloc(&dm, dim * dim * 8), cudaMalloc(&dh, n * 8);
  cudaMalloc(&dst, n * 4), cudaMalloc(&dnd, n * 4);
  cudaMemcpy(dq, q.data(), n * dim * 8, cudaMemcpyHostToDevice);
  cudaMemcpy(dp, p.data(), n * dim * 8, cudaMemcpyHostToDevice);
  cudaMemcpy(dm, minv.data(), dim * dim * 8, cudaMemcpyHostToDevice);
  ModelArgs m;
  memset(&m, 0, sizeof(m));
  m.target_id = MB200_TARGET_NEAL_FUNNEL;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0), cudaEventCreate(&e1);
  const bool with_h = argc > 3 ? atoi(argv[3]) != 0 : true;
  for (int steps : {1, 2, 10, 50, 200}) {
    float best = 1e30f;
    for (int rep = 0; rep < 6; ++rep) {
      cudaEventRecord(e0);
      EuclidArgs a{};
      a.q_in = dq, a.p_in = dp, a.q_out = dqo, a.p_out = dpo, a.n = n, a.dim = dim, a.eps = 0.01;
      a.n_steps = steps, a.minv = dm, a.m = m, a.h_out = with_h ? dh : nullptr, a.status = dst;
      a.n_done = dnd;
      int rc = k1_launch<NealFunnelTarget>(a);
      cudaEventRecord(e1);
      cudaEventSynchronize(e1);
      if (rc != 0) { printf("k1_launch rc=%d: %s\n", rc, g_err); return 1; }
      float ms;
      cudaEventElapsedTime(&ms, e0, e1);
      if (rep > 0 && ms < best) best = ms;
    }
    std::vector<double> qo(n * dim), ho(n);
    cudaMemcpy(qo.data(), dqo, n * dim * 8, cudaMemcpyDeviceToHost);
    cudaMemcpy(ho.data(), dh, n * 8, cudaMemcpyDeviceToHost);
    double cs = 0, hs = 0;
    for (auto v : qo) cs += v;
    for (auto v : ho) hs += v;
    const double rate = (double)n * steps / (best * 1e-3);
    // peaks of the H100 SXM data sheet (700 W): FP64 tensor 67 TFLOP/s, HBM3 3.35 TB/s
    printf("steps %3d: %.4f ms  %.4f G steps/s  DMMA %.1f%% of 67 TF  HBM-roofline %.3f  "
           "checksum q %.15e h %.15e  (%s)\n",
           steps, best, rate * 1e-9, rate * 2.0 * dim * dim / 67.0e12 * 100,
           rate * 32.0 * dim / 3350.0e9, cs, hs, cudaGetErrorString(cudaGetLastError()));
  }
#ifndef K1_AB
#ifdef K1_TRACE
  print_trace("leapfrog_dmma_kernel");
#endif
#else
  // ---- A/B: the previous generation against the current kernel, alternating in one process
  auto launch = [&](bool old, int steps) {
    EuclidArgs a{};
    a.q_in = dq, a.p_in = dp, a.q_out = dqo, a.p_out = dpo, a.n = n, a.dim = dim, a.eps = 0.01;
    a.n_steps = steps, a.minv = dm, a.m = m, a.h_out = with_h ? dh : nullptr, a.status = dst;
    a.n_done = dnd;
    cudaEventRecord(e0);
    const int rc = old ? k1_launch_dmma4<NealFunnelTarget>(a) : k1_launch<NealFunnelTarget>(a);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    if (rc != 0) { printf("launch rc=%d: %s\n", rc, g_err); exit(1); }
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    return ms;
  };
  const char* kname[2] = {"leapfrog_dmma_kernel (new)", "leapfrog_dmma4_kernel (old)"};
  const int step_counts[2] = {50, 200};
  const int reps = argc > 4 ? atoi(argv[4]) : 21;
  for (int k = 0; k < 2; ++k)
    for (int si = 0; si < 2; ++si) launch(k == 1, step_counts[si]);  // warm-up
  std::vector<float> t[2][2];
  for (int rep = 0; rep < reps; ++rep)
    for (int si = 0; si < 2; ++si)
      for (int o = 0; o < 2; ++o) {
        const int k = (rep + o) & 1;  // alternate which kernel goes first
        t[k][si].push_back(launch(k == 1, step_counts[si]));
      }
  auto med = [](std::vector<float> v) {
    std::sort(v.begin(), v.end());
    const size_t h = v.size() / 2;
    return v.size() & 1 ? (double)v[h] : 0.5 * (v[h - 1] + v[h]);
  };
  printf("A/B, %d alternating launches of each kernel and step count (%lld chains x %d, funnel)\n",
         reps, (long long)n, dim);
  double m50[2], m200[2];
  for (int k = 0; k < 2; ++k) {
    for (int si = 0; si < 2; ++si) {
      const auto mm = std::minmax_element(t[k][si].begin(), t[k][si].end());
      const double md = med(t[k][si]);
      (si ? m200 : m50)[k] = md;
      printf("  %-28s %3d steps: median %.4f ms  min %.4f  max %.4f  (max-min %.4f ms)\n", kname[k],
             step_counts[si], md, *mm.first, *mm.second, *mm.second - *mm.first);
    }
    const double slope = (m200[k] - m50[k]) / 150.0;
    printf("  %-28s per-step slope (T200 - T50) / 150 = %.3f us = %.4f G steps/s\n", kname[k],
           slope * 1e3, n / (slope * 1e-3) * 1e-9);
  }
  printf("  new / old: 50 steps %.4f, 200 steps %.4f, slope %.4f\n", m50[0] / m50[1],
         m200[0] / m200[1], (m200[0] - m50[0]) / (m200[1] - m50[1]));
  // the two kernels on the same input: largest ulp distance of q, p, h
  for (int si = 0; si < 2; ++si) {
    std::vector<double> out[2][3];
    for (int k = 0; k < 2; ++k) {
      launch(k == 1, step_counts[si]);
      out[k][0].resize(n * dim), out[k][1].resize(n * dim), out[k][2].resize(n);
      cudaMemcpy(out[k][0].data(), dqo, n * dim * 8, cudaMemcpyDeviceToHost);
      cudaMemcpy(out[k][1].data(), dpo, n * dim * 8, cudaMemcpyDeviceToHost);
      cudaMemcpy(out[k][2].data(), dh, n * 8, cudaMemcpyDeviceToHost);
    }
    const char* names[3] = {"q", "p", "h"};
    printf("  new vs old, %3d steps:", step_counts[si]);
    for (int v = 0; v < 3; ++v) {
      // ulp distance of each value, and the difference relative to the largest |value| of its
      // chain in units of 2^-52 (a coordinate near zero can be many ulp off after a last-bit
      // difference elsewhere in its chain)
      const int len = v < 2 ? dim : 1;
      int64_t worst = 0, differ = 0;
      double worst_rel = 0.0;
      for (size_t ch = 0; ch * len < out[0][v].size(); ++ch) {
        double scale = 0.0;
        for (int i = 0; i < len; ++i) scale = std::max(scale, std::fabs(out[1][v][ch * len + i]));
        for (int i = 0; i < len; ++i) {
          const double a = out[0][v][ch * len + i], b = out[1][v][ch * len + i];
          const int64_t d = ulp_diff(a, b);
          worst = std::max(worst, d);
          differ += d != 0;
          if (scale > 0.0) worst_rel = std::max(worst_rel, std::fabs(a - b) / scale / 0x1p-52);
        }
      }
      printf("  %s max %lld ulp, %.1f x 2^-52 of the chain's largest (%lld of %zu differ)",
             names[v], (long long)worst, worst_rel, (long long)differ, out[0][v].size());
    }
    printf("\n");
  }
#ifdef K1_TRACE
  for (int k = 1; k >= 0; --k) {
    launch(k == 1, 200);
    print_trace(kname[k]);
  }
#endif
#endif
  return 0;
}
