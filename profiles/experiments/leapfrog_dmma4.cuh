// K1, fourth generation: the headline kernel as it was before each warp kept its own momenta in
// registers (mici_b200/csrc/leapfrog_dmma.cuh has the current one).  Every step the update phase
// reloads the warp's own momentum slots from the shared-memory tile, kicks them and stores them
// back, and the drift reads all of its A fragments from the tile, in k order 0, 1, ..., DP/16 - 1
// for every warp, after the second group barrier.  The drift keeps two stages of A / B fragments
// in flight (`#pragma unroll 2` over k-blocks).  Kept for A/B comparison
// (profiles/tools/k1_bench.cu -DK1_AB); not compiled into the library.
#pragma once
#include "../../mici_b200/csrc/leapfrog_dmma.cuh"

namespace mb200 {

// A operand as a[tile][k-pair], in the order the previous layout loads it
__device__ __forceinline__ void dmma_m16n8k16(double& c0, double& c1, double& c2, double& c3,
                                              const double2 (&a)[2][2], const double2 (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, "
      "{%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
      : "+d"(c0), "+d"(c1), "+d"(c2), "+d"(c3)
      : "d"(a[0][0].x), "d"(a[1][0].x), "d"(a[0][0].y), "d"(a[1][0].y),
        "d"(a[0][1].x), "d"(a[1][1].x), "d"(a[0][1].y), "d"(a[1][1].y),
        "d"(b[0].x), "d"(b[0].y), "d"(b[1].x), "d"(b[1].y));
}

// One group's work: MT (1 or 2) row tiles starting at CTA-local row `row0`.
//
// Formulation used inside the kernel (exact re-parametrisation of integrators.py:170-173):
//   s = dir * p   (signed momentum; the sign flip is exact)
//   kick:  s -= (eps/2) * grad l(q)          == dir * (p - (dir*eps/2) * grad)
//   drift: q += s . (eps * A)                == q + (dir*eps) * (A p)
// so the per-chain direction only appears in the load and the store, sm.A holds eps*A (scaled
// once after the TMA lands), and the drift is a DMMA whose accumulator operand IS q: positions
// never leave the accumulator registers.
//
// Scheduling facts this is written around (profiles/tools fp64_arb / fp64_mix / k1_bench -DK1_TRACE):
// a warp whose next instruction is a scalar FP64 operation makes almost NO progress while other
// warps of its SM sub-partition stream DMMAs (two or more streaming DMMA.8x8x4; a single one
// streaming DMMA.16x8x16 already holds it to ~390 cycles per instruction), so the per-step
// update phase of every group ends up running after the drifts of the whole sub-partition (the
// groups lock-step) and the step time is  drift (DMMA-pipe bound) + update phase (issue /
// latency bound).  The update phase is therefore kept as short as possible: no bounds logic
// (phantom coordinates are zero and stay zero under every registry target's kick), one FMA chain
// for the reduction, the chains of all tiles issued before any shuffle, the per-chain scalar
// (funnel: exp(-v)) evaluated for all the group's chains in one pass of the coordinate-0 warp and
// published instead of being summed, own momenta pre-loaded before the group barrier, two
// barriers per step.
//
// PC = true: per-chain step sizes (adaptive warm-up, adapters.py:40-235 per chain).  sm.A then holds
// A unscaled (step_size = 1) and the momentum tile holds  s = eps_c * dir * p:
//   kick:  s -= (eps_c^2 / 2) * grad l(q)      drift: q += s . A
// -- the same two flows, with eps_c applied on the momentum side instead of the matrix side.
template <class Target, int DP, int MT, bool PC>
__device__ __forceinline__ void leapfrog_dmma4_group(
    DmmaSmem<DP>& sm, const Target& target, const double* q_in, const double* p_in,
    double* q_out, double* p_out, const int32_t* __restrict__ dir,
    const double* __restrict__ step_sizes, int64_t n_chains, int dim,
    double step_size, int n_steps, double* __restrict__ h_out, int32_t* __restrict__ status,
    int32_t* __restrict__ n_done, int64_t chain0, int row0, int w, int lane, int bar_id,
    int cta_threads, bool vec2, int32_t* __restrict__ counters) {
  constexpr int LDA = DmmaSmem<DP>::LDA;
  constexpr int NT = DP / 32;  // 8-column tiles per warp
  constexpr int KS = DP / 4;   // k steps
  const int r = lane >> 2, c = lane & 3;
  const int col0 = w * (DP / 4);  // first column of this warp's slice
  const double mh = -0.5 * step_size;
  // the lane that holds coordinate 0 of its rows (in q[mt][0][0])
  const bool owner = (w == 0) && (c == 0);

  // registers: positions of the slice in C-fragment layout (row 8mt + r, columns
  // col0 + 8nt + 2c + {0,1}); signed momenta live in sm.P with the same ownership
  double q[MT][NT][2], mhr[PC ? MT : 1];
  bool live[MT];
  int row[MT];
  // momentum scale of a live chain: dir (+-1), times eps_c with per-chain step sizes; read again
  // for the store rather than held in registers through the launch
  auto load_scale = [&](int64_t ch) {
    const double d = (dir != nullptr && dir[ch] < 0) ? -1.0 : 1.0;
    return PC ? d * step_sizes[ch] : d;
  };
  // own momentum slots &sm.P[row[mt]][col0 + 8nt + 2c], addressed from one 32-bit offset (the
  // MT x NT slots fold into load / store immediates; pointers would hold 2 registers per tile)
  const uint32_t pofs = (uint32_t)((row0 + r) * LDA + col0 + 2 * c);
  auto pslot = [&](int mt, int nt) -> double2& {
    return *reinterpret_cast<double2*>(&sm.P[pofs + mt * 8 * LDA + 8 * nt]);
  };

#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
    row[mt] = row0 + 8 * mt + r;
    const int64_t ch = chain0 + row[mt];
    live[mt] = ch < n_chains;
    const double sgn = live[mt] ? load_scale(ch) : (PC ? 0.0 : 1.0);
    if (PC) mhr[mt] = -0.5 * (sgn * sgn);
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const int i = col0 + 8 * nt + 2 * c;
      double2 a = make_double2(0.0, 0.0), b = make_double2(0.0, 0.0);
      if (live[mt] && i < dim) {
        if (vec2) {  // even dim, 16-byte aligned state arrays
          a = *reinterpret_cast<const double2*>(q_in + (size_t)ch * dim + i);
          b = *reinterpret_cast<const double2*>(p_in + (size_t)ch * dim + i);
        } else {
          a.x = q_in[(size_t)ch * dim + i], b.x = p_in[(size_t)ch * dim + i];
          if (i + 1 < dim) a.y = q_in[(size_t)ch * dim + i + 1], b.y = p_in[(size_t)ch * dim + i + 1];
        }
      }
      q[mt][nt][0] = a.x, q[mt][nt][1] = a.y;
      pslot(mt, nt) = make_double2(sgn * b.x, sgn * b.y);
    }
  }

  int s = -1;  // current step (read by the profiling hook only)

  // ---- update phase, part 1 (before the group barrier): this warp's share of the per-chain
  // reduction and, on the coordinate-0 warp, the per-chain scalar
  auto tile_sums = [&]() {
    if (!Target::TILE_SUM) return;
    // sum of squares over the slice: two FMA chains per row, the chains of all tiles issued
    // before the shuffles of any
    double v[MT];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      double t0 = q[mt][0][0] * q[mt][0][0];
      if (Target::COORD0) t0 = owner ? 0.0 : t0;
      t0 = fma(q[mt][0][1], q[mt][0][1], t0);
      if (mt == 0) MB200_K1_TRACE_AFTER(6, t0);
      double t1 = 0.0;
#pragma unroll
      for (int nt = 1; nt < NT; ++nt) {
        double& t = (nt & 1) ? t1 : t0;
        t = fma(q[mt][nt][0], q[mt][nt][0], t);
        t = fma(q[mt][nt][1], q[mt][nt][1], t);
      }
      v[mt] = t0 + t1;
    }
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) v[mt] += __shfl_xor_sync(FULL_MASK, v[mt], 1);
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) v[mt] += __shfl_xor_sync(FULL_MASK, v[mt], 2);
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
      if (c == 0) sm.psum[row[mt]][w] = v[mt];
  };
  auto publish_partials = [&]() {
    if (Target::ROW_SCALAR && w == 0) {  // warp-uniform
      // one pass for all the group's chains: lane 4r + mt evaluates row 8mt + r, whose
      // coordinate 0 lane 4r holds in q[mt][0][0]; lanes with c >= MT evaluate a dummy
      double v0 = (c == 0) ? q[0][0][0] : 0.0;
#pragma unroll
      for (int mt = 1; mt < MT; ++mt) {
        const double vm = __shfl_sync(FULL_MASK, q[mt][0][0], lane & ~3);
        v0 = (c == mt) ? vm : v0;
      }
      // the sums and the scalar are independent: in one basic block the scheduler interleaves them
      tile_sums();
      const double rs = target.row_scalar(v0);
      if (c < MT) sm.rscal[row0 + 8 * c + r] = rs;
    } else {
      tile_sums();
    }
  };

  // ---- the update phase: part 1, the group barrier, then part 2: s -= (eps/2) * grad l(q),
  // KICKS times (1 or 2: the two half-steps either side of a step boundary stay two separately
  // rounded updates, systems.py:152), one FMA per coordinate and kick; then make the new momenta
  // visible to the group.  The first barrier also orders "all A-fragment reads of sm.P done"
  // before the in-place update.
  //
  // The phase moves every momentum through shared memory twice (load own slots, store them
  // back): 2 x 64 KB per CTA and step at 64 chains x 128, 1024 cycles at 128 B/clk -- more than
  // its FP64 work.  So the own-slot loads are issued before part 1, where they overlap the DMMA
  // drain and the partial sums, and the per-chain scalars of all tiles are loaded before the
  // first tile's stores, which they would otherwise queue behind.
  auto update_phase = [&](auto kicks_tag) {
    constexpr int KICKS = decltype(kicks_tag)::value;
    double2 pv[MT][NT];
    if (KICKS > 0) {
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) pv[mt][nt] = pslot(mt, nt);  // own slots: no hazard
    }
    publish_partials();
    MB200_K1_TRACE(2);
    named_barrier_sync(bar_id, 128);
    MB200_K1_TRACE(3);
    if (KICKS == 0) return;
    double rs[MT];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) rs[mt] = Target::ROW_SCALAR ? sm.rscal[row[mt]] : 1.0;
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      const double mhm = PC ? mhr[PC ? mt : 0] : mh;
      const double coef = target.kick_coef(mhm, rs[mt]);
      double c00 = coef, a00 = q[mt][0][0];
      if (Target::COORD0 && w == 0) {  // warp-uniform; only the owner lanes differ
        const double4 ps = *reinterpret_cast<const double4*>(&sm.psum[row[mt]][0]);
        const double g0 = target.grad0(q[mt][0][0], ((ps.x + ps.y) + ps.z) + ps.w, rs[mt]);
        c00 = owner ? mhm : coef;
        a00 = owner ? g0 : a00;
      }
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        double2 v = pv[mt][nt];
        if (Target::LINEAR) {
#pragma unroll
          for (int k = 0; k < KICKS; ++k) {
            v.x = (nt == 0) ? fma(c00, a00, v.x) : fma(coef, q[mt][nt][0], v.x);
            v.y = fma(coef, q[mt][nt][1], v.y);
          }
        } else {
#pragma unroll
          for (int k = 0; k < KICKS; ++k)
            target.kick_pair_nl(mhm, q[mt][nt][0], q[mt][nt][1], v.x, v.y);
        }
        pslot(mt, nt) = v;
      }
    }
    MB200_K1_TRACE(4);
    named_barrier_sync(bar_id, 128);
    MB200_K1_TRACE(5);
  };
  using K0 = std::integral_constant<int, 0>;
  using K1 = std::integral_constant<int, 1>;
  using K2 = std::integral_constant<int, 2>;

  // acc += S * (eps A) on the tensor pipe (acc = q for the drift, acc = 0 for the energy).
  // Fragments are fetched with 128-bit loads: lane c of a row holds k = 8J + 2c and 8J + 2c + 1.
  // The pairing of lanes with k is free as long as the A and B fragments agree.
  auto drift = [&](double (&acc)[MT][NT][2]) {
    const double2* a_base = reinterpret_cast<const double2*>(&sm.P[(row0 + r) * LDA + 2 * c]);
    const double2* b_base = reinterpret_cast<const double2*>(&sm.A[(col0 + r) * LDA + 2 * c]);
    if constexpr (MT == 2) {
      // The group's two row tiles are the 16 rows of DMMA.16x8x16 (twice the FP64 rate of
      // DMMA.8x8x4 on sm_90): rows r / r + 8 are the C fragment's c0,c1 / c2,c3, i.e. q[0][nt]
      // and q[1][nt].  Fragment slot i (logical k = c + 4i) of lane c holds physical k
      // 16J + {2c, 2c + 1, 8 + 2c, 9 + 2c}[i]: the two 128-bit loads of k-pairs 2J and 2J + 1.
#pragma unroll 2
      for (int j = 0; j < KS / 4; ++j) {
        double2 a[2][2], b[NT][2];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int h = 0; h < 2; ++h) a[mt][h] = a_base[mt * 4 * LDA + 4 * (2 * j + h)];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
          for (int h = 0; h < 2; ++h) b[nt][h] = b_base[nt * 4 * LDA + 4 * (2 * j + h)];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
          dmma_m16n8k16(acc[0][nt][0], acc[0][nt][1], acc[1][nt][0], acc[1][nt][1], a, b[nt]);
      }
    } else {
      // DMMA.8x8x4 per row tile: the two DMMAs of a k-pair contract {8J, 8J+2, 8J+4, 8J+6} and
      // {8J+1, ..., 8J+7}.  A single row tile gives a warp only NT independent accumulator
      // chains (DMMA latency ~ 10 issue slots): the two halves of every k-pair then go to
      // separate accumulator sets that are added at the end (same products, summed in a
      // different order)
      constexpr bool KSPLIT = (MT == 1);
      double acc2[KSPLIT ? NT : 1][2];
      if (KSPLIT) {
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) acc2[nt][0] = 0.0, acc2[nt][1] = 0.0;
      }
#pragma unroll 4
      for (int j = 0; j < KS / 2; ++j) {
        double2 a[MT], b[NT];
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) a[mt] = a_base[mt * 4 * LDA + 4 * j];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) b[nt] = b_base[nt * 4 * LDA + 4 * j];
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
          for (int nt = 0; nt < NT; ++nt)
            dmma_m8n8k4(acc[mt][nt][0], acc[mt][nt][1], a[mt].x, b[nt].x);
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            if (KSPLIT) dmma_m8n8k4(acc2[nt][0], acc2[nt][1], a[mt].y, b[nt].y);
            else dmma_m8n8k4(acc[mt][nt][0], acc[mt][nt][1], a[mt].y, b[nt].y);
          }
      }
      if (KSPLIT) {
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) acc[0][nt][0] += acc2[nt][0], acc[0][nt][1] += acc2[nt][1];
      }
    }
  };

  MB200_K1_MARK(4);
  if (n_steps > 0) update_phase(K1{});
  else update_phase(K0{});
  MB200_K1_MARK(5);
  for (s = 0; s < n_steps - 1; ++s) {
    MB200_K1_TRACE(0);
    drift(q);  // h2_flow (systems.py:363): q += dir*eps * (A p)
    MB200_K1_TRACE(1);
    update_phase(K2{});  // closes step s and (cached gradient) opens step s+1
  }
  if (n_steps > 0) {
    drift(q);
    update_phase(K1{});
  }

  MB200_K1_MARK(6);
  // ---- store (p = dir * s)
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
    const int64_t ch = chain0 + row[mt];
    if (!live[mt]) continue;
    const double sgn = load_scale(ch);
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const int i = col0 + 8 * nt + 2 * c;
      if (i < dim) {
        const double2 sv = pslot(mt, nt);
        double2 pv = make_double2(sgn * sv.x, sgn * sv.y);  // dir = +-1: exact
        if (PC) {
          // s = (dir eps_c) p  ->  p = s / (dir eps_c); a chain with eps_c = 0 has not moved
          if (sgn != 0.0) {
            pv = make_double2(sv.x / sgn, sv.y / sgn);
          } else {
            pv.x = p_in[(size_t)ch * dim + i];
            pv.y = (i + 1 < dim) ? p_in[(size_t)ch * dim + i + 1] : 0.0;
          }
          // eps_c^2 zero or subnormal: the energy epilogue contracts the stored p itself
          if (h_out != nullptr && !(sgn * sgn >= DBL_MIN)) pslot(mt, nt) = pv;
        }
        if (vec2) {
          *reinterpret_cast<double2*>(q_out + (size_t)ch * dim + i) =
              make_double2(q[mt][nt][0], q[mt][nt][1]);
          *reinterpret_cast<double2*>(p_out + (size_t)ch * dim + i) = pv;
        } else {
          q_out[(size_t)ch * dim + i] = q[mt][nt][0], p_out[(size_t)ch * dim + i] = pv.x;
          if (i + 1 < dim)
            q_out[(size_t)ch * dim + i + 1] = q[mt][nt][1], p_out[(size_t)ch * dim + i + 1] = pv.y;
        }
      }
    }
    if (w == 0 && c == 0) {
      if (status != nullptr) status[ch] = MB200_STATUS_OK;
      if (n_done != nullptr) n_done[ch] = n_steps;
      if (counters != nullptr) counters[ch * MB200_N_COUNTERS + MB200_COUNT_GRAD] += n_steps + 1;
    }
  }

  MB200_K1_MARK(7);
  // ---- Hamiltonian of the final state: l(q) + p . (A p) / 2   (systems.py:187-196, 348-350)
  // sm.psum / sm.rscal hold the reduction of the final positions (last update phase).  Without
  // per-chain step sizes sm.P holds s = dir p against eps A, and s . (eps A) s / eps = p . A p.
  // With them A is unscaled and a row of sm.P holds s = eps_c dir p, and s . A s / eps_c^2 = p . A p
  // -- except where eps_c^2 is zero or subnormal (0/0 for eps_c = 0, few significant bits below
  // |eps_c| = 2^-511): those rows were overwritten with the stored p above, and their kinetic
  // term is p . A p directly.  (Rows are independent in the contraction.)
  if (h_out != nullptr) {
    if (PC) named_barrier_sync(bar_id, 128);  // every warp's rows are in sm.P before drift(u)
    double l[MT], kin[MT], u[MT][NT][2];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      double red[2] = {0.0, 1.0};
      if (Target::TILE_SUM) {
        const double4 ps = *reinterpret_cast<const double4*>(&sm.psum[row[mt]][0]);
        red[0] = ((ps.x + ps.y) + ps.z) + ps.w;
      }
      if (Target::ROW_SCALAR) red[1] = sm.rscal[row[mt]];
      l[mt] = 0.0;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const int i = col0 + 8 * nt + 2 * c;
        if (i < dim) l[mt] += target.nld_pair(i, q[mt][nt][0], q[mt][nt][1], red);
        u[mt][nt][0] = 0.0, u[mt][nt][1] = 0.0;
      }
    }
    drift(u);  // u = s . (eps A)
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      kin[mt] = 0.0;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const double2 sv = pslot(mt, nt);
        kin[mt] = fma(sv.x, u[mt][nt][0], kin[mt]);
        kin[mt] = fma(sv.y, u[mt][nt][1], kin[mt]);
      }
      kin[mt] += __shfl_xor_sync(FULL_MASK, kin[mt], 1);
      kin[mt] += __shfl_xor_sync(FULL_MASK, kin[mt], 2);
      l[mt] += __shfl_xor_sync(FULL_MASK, l[mt], 1);
      l[mt] += __shfl_xor_sync(FULL_MASK, l[mt], 2);
      if (c == 0) {
        sm.ex[0][row[mt]][w] = kin[mt];
        sm.ex[1][row[mt]][w] = l[mt];
      }
    }
    named_barrier_sync(bar_id, 128);
    if (w == 0 && c == 0) {
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        if (!live[mt]) continue;
        const double4 k4 = *reinterpret_cast<const double4*>(&sm.ex[0][row[mt]][0]);
        const double4 l4 = *reinterpret_cast<const double4*>(&sm.ex[1][row[mt]][0]);
        const double ks = ((k4.x + k4.y) + k4.z) + k4.w;
        const double ls = ((l4.x + l4.y) + l4.z) + l4.w;
        if (PC) {  // ks = eps_c^2 p.A p, or p.A p where eps_c^2 is zero or subnormal
          const double e = step_sizes[chain0 + row[mt]];
          h_out[chain0 + row[mt]] = ls + 0.5 * (e * e >= DBL_MIN ? ks / (e * e) : ks);
        } else {
          h_out[chain0 + row[mt]] = ls + 0.5 * (ks / step_size);
        }
      }
    }
  }
}

template <class Target, int DP, bool PC>
__global__ void __launch_bounds__(DMMA_THREADS, 1)
    leapfrog_dmma4_kernel(const double* q_in, const double* p_in, double* q_out, double* p_out,
                         const int32_t* __restrict__ dir, const double* __restrict__ step_sizes,
                         int64_t n_chains, int dim,
                         double step_size, int n_steps, const double* __restrict__ minv,
                         ModelArgs model, double* __restrict__ h_out,
                         int32_t* __restrict__ status, int32_t* __restrict__ n_done,
                         int tiles_per_cta, int vec2, int tma_rows) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  DmmaSmem<DP>& sm = *reinterpret_cast<DmmaSmem<DP>*>(smem_raw);
  constexpr int LDA = DmmaSmem<DP>::LDA;
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const int group = warp >> 2;  // 4 groups: tiles {0,1}, {2,3}, {4,5}, {6,7}
  // Column quarter owned by this warp.  warp & 3 is its SM sub-partition; rotating the quarters by
  // the group index puts each group's "coordinate 0" warp (which carries the target's per-chain
  // special work, e.g. exp(-v) of the funnel) on a different sub-partition -- otherwise one
  // sub-partition is systematically slower and the other three idle at the group barriers.
  const int w = ((warp & 3) + group) & 3;
  const Target target(model, dim);
  MB200_K1_MARK(0);

  // ---- stage A = M^-1 into shared memory: one TMA bulk copy per row, one mbarrier.  Issued
  // first; everything below until the wait overlaps the copies.
  const uint32_t mbar = smem_u32(&sm.mbar);
  if (tma_rows && warp == 0) {
    if (lane == 0) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mbar));
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    const uint32_t row_bytes = (uint32_t)dim * 8u;
    if (lane == 0)
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar),
                   "r"(row_bytes * (uint32_t)dim)
                   : "memory");
    __syncwarp();
#pragma unroll 1
    for (int row = lane; row < dim; row += 32) {  // the 32 lanes issue the row copies
      const unsigned long long src =
          reinterpret_cast<unsigned long long>(minv) + (unsigned long long)row * row_bytes;
      asm volatile(
          "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
          ::"r"(smem_u32(&sm.A[row * LDA])),
          "l"(src), "r"(row_bytes), "r"(mbar)
          : "memory");
    }
  }
  // pull this CTA's first block of state rows towards L2 while A is in flight
  {
    const int64_t chain0 = (int64_t)blockIdx.x * (8 * tiles_per_cta);
    const int64_t left = n_chains - chain0;
    const int64_t rows = left < 8 * tiles_per_cta ? left : 8 * tiles_per_cta;
    const int64_t lines = (rows * dim * 8 + 127) / 128;
    for (int64_t i = tid; i < 2 * lines; i += blockDim.x) {
      const double* base = (i < lines ? q_in : p_in) + (size_t)chain0 * dim;
      const char* ptr = reinterpret_cast<const char*>(base) + (i < lines ? i : i - lines) * 128;
      asm volatile("prefetch.global.L2 [%0];" ::"l"(ptr));
    }
  }
  if (!tma_rows) {  // odd dim / unaligned matrix: rows are not 16-byte multiples, plain copies
    for (int idx = tid; idx < dim * dim; idx += blockDim.x) {
      const int row = idx / dim, col = idx - row * dim;
      sm.A[row * LDA + col] = minv[idx];
    }
  }
  // zero the part of the padding that the fragment loads read (rows / columns in [dim, DP)) --
  // disjoint from the TMA destinations; sm.P needs none (every slot that is read is written by
  // the state load, phantom coordinates as zeros)
  if (dim < DP) {
    for (int idx = tid; idx < DP * DP; idx += blockDim.x) {
      const int row = idx / DP, col = idx - row * DP;
      if (row >= dim || col >= dim) sm.A[row * LDA + col] = 0.0;
    }
  }
  MB200_K1_MARK(1);
  // every thread polls the mbarrier below: its initialisation by warp 0 (and the zero-fill
  // above) must be visible first
  __syncthreads();
  // wait for the bytes to land (phase 0), then scale the staged metric: sm.A = eps * A
  if (tma_rows) {
    uint32_t done = 0;
    while (!done) {
      asm volatile(
          "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n"
          " selp.u32 %0, 1, 0, p;\n}"
          : "=r"(done)
          : "r"(mbar)
          : "memory");
    }
  }
  MB200_K1_MARK(2);
  if (!PC)  // per-chain step sizes: the matrix stays unscaled
#pragma unroll 4
  for (int idx = tid; idx < DP * (DP / 2); idx += blockDim.x) {
    const int row = idx / (DP / 2), c2 = idx - row * (DP / 2);
    double2* ptr = reinterpret_cast<double2*>(&sm.A[row * LDA]) + c2;
    double2 v = *ptr;
    v.x *= step_size, v.y *= step_size;
    *ptr = v;
  }
  __syncthreads();
  MB200_K1_MARK(3);

  // A CTA owns `tiles_per_cta` (<= 8) row tiles of 8 chains per pass -- 8 when the batch fills
  // the GPU (64 chains per SM), fewer for small batches so that the tiles spread over all SMs
  // (strong scaling: 1024 chains -> 128 CTAs of one tile instead of 16 CTAs of eight).  The
  // tiles of a pass are dealt to the 4 groups as evenly as possible (7 -> 2,2,2,1; 4 -> 1,1,1,1).
  const int rows_per_cta = 8 * tiles_per_cta;
  for (int64_t blk = blockIdx.x; blk * rows_per_cta < n_chains; blk += gridDim.x) {
    const int64_t chain0 = blk * rows_per_cta;
    const int64_t left = n_chains - chain0;
    const int tiles = (int)((left >= rows_per_cta) ? tiles_per_cta : (left + 7) / 8);
    const int base = tiles / DMMA_GROUPS, rem = tiles % DMMA_GROUPS;
    const int mt = base + (group < rem ? 1 : 0);
    const int row0 = 8 * (group * base + (group < rem ? group : rem));
    const int cta_threads = 128 * (tiles < DMMA_GROUPS ? tiles : DMMA_GROUPS);
#define MB200_GROUP(MT)                                                                       \
  leapfrog_dmma4_group<Target, DP, MT, PC>(sm, target, q_in, p_in, q_out, p_out, dir,          \
                                          step_sizes, n_chains, dim, step_size, n_steps,      \
                                          h_out, status, n_done, chain0, row0, w, lane,       \
                                          1 + group, cta_threads, vec2 != 0, model.counters)
    if (DMMA_MAX_MT >= 4 && mt == 4) MB200_GROUP(4);
    else if (DMMA_MAX_MT >= 3 && mt == 3) MB200_GROUP(3);
    else if (mt == 2) MB200_GROUP(2);
    else if (mt == 1) MB200_GROUP(1);
#undef MB200_GROUP
    __syncthreads();  // next block of chains reuses sm.P / sm.part
  }
}

}  // namespace mb200
