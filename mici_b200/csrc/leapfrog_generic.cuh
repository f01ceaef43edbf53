// K1g / K7: explicit leapfrog on a Euclidean-metric system -- general-dimension kernel.
//
// Replaces, per chain (reference paths):
//   LeapfrogIntegrator._step          integrators.py:170-173
//   System.h1_flow                    systems.py:143-152     p -= dt * grad l(q)
//   EuclideanMetricSystem.h2_flow     systems.py:362-363     q += dt * M^-1 p
//   EuclideanMetricSystem.h2 / h      systems.py:348-350, 187-196
//
// Layout: one warp owns CPW chains.  A chain's vectors live in registers, lane `l` owning the
// coordinate pairs (2l + 64k, 2l + 64k + 1), k < KP, so global loads/stores are coalesced
// 128-bit accesses of the row-major [n_chains x dim] arrays.  The dense metric inverse A = M^-1
// (explicit, symmetric: matrices.py:1183-1188) is read through L1/L2 one row at a time and
// shared by the CPW chains of the warp; momenta are staged in shared memory for the broadcast.
// This kernel handles every (dim, metric kind); the tensor-core kernel in leapfrog_dmma.cuh
// takes over for dense metrics with dim <= 128.
#pragma once
#include "metric_ops.cuh"
#include "targets.cuh"

namespace mb200 {

// Whole-vector targets (user-written models, user_target.cuh) set `WHOLE_VECTOR = true`: they see
// a chain's whole position vector in shared memory instead of the pair interface of targets.cuh.
template <class T, class = void>
struct IsWholeVector {
  static constexpr bool value = false;
};
template <class T>
struct IsWholeVector<T, decltype(void(T::WHOLE_VECTOR))> {
  static constexpr bool value = T::WHOLE_VECTOR;
};

template <class Target, int KP, int CPW>
struct LeapfrogGeneric {
  static constexpr int NV = 2 * KP;  // coordinates per lane per chain
  static constexpr bool WHOLE = IsWholeVector<Target>::value;

  // Staging area of a whole-vector target: q then g, 64 KP doubles each, per warp, after the
  // CPW * 64 KP doubles per warp of inv_metric_apply (launch_generic / launch_eval size both).
  // The warp's chains call the target one after the other, so one area per warp suffices.
  static __device__ __forceinline__ double* whole_stage() {
    extern __shared__ double smem[];
    return smem + (size_t)(blockDim.x >> 5) * CPW * 64 * KP + (size_t)(threadIdx.x >> 5) * 128 * KP;
  }
  static __device__ __forceinline__ void whole_put_q(int lane, const double (&q)[NV], double* qs) {
    __syncwarp();
#pragma unroll
    for (int k = 0; k < KP; ++k) {
      const int i = 2 * lane + 64 * k;
      qs[i] = q[2 * k];
      qs[i + 1] = q[2 * k + 1];
    }
    __syncwarp();
  }
  static __device__ __forceinline__ void whole_grad(const Target& t, int dim, int lane,
                                                    const double (&q)[NV], double (&g)[NV]) {
    double* qs = whole_stage();
    double* gs = qs + 64 * KP;
    whole_put_q(lane, q, qs);
    t.grad(qs, dim, lane, gs);
    __syncwarp();
#pragma unroll
    for (int k = 0; k < KP; ++k) {
      const int i = 2 * lane + 64 * k;
      g[2 * k] = (i < dim) ? gs[i] : 0.0;
      g[2 * k + 1] = (i + 1 < dim) ? gs[i + 1] : 0.0;
    }
  }
  static __device__ __forceinline__ double whole_nld(const Target& t, int dim, int lane,
                                                     const double (&q)[NV]) {
    double* qs = whole_stage();
    whole_put_q(lane, q, qs);
    const double l = t.nld(qs, dim, lane);
    __syncwarp();
    return l;
  }

  // gradient of l at q (pair layout); all lanes of the warp participate
  static __device__ __forceinline__ void grad(const Target& t, int dim, int lane,
                                              const double (&q)[NV], double (&g)[NV]) {
    if constexpr (WHOLE) whole_grad(t, dim, lane, q, g);
    else pair_grad(t, dim, lane, q, g);
  }
  // the same gradient, also handing out the target's reduced sums at q (red[NRED + 1]) so that a
  // caller which needs l(q) at the same position next (a NUTS leaf) does not reduce them again;
  // a whole-vector target has none
  static __device__ __forceinline__ void grad_keep(const Target& t, int dim, int lane,
                                                   const double (&q)[NV], double (&g)[NV],
                                                   double (&red)[Target::NRED + 1]) {
    if constexpr (WHOLE) whole_grad(t, dim, lane, q, g);
    else pair_grad_keep(t, dim, lane, q, g, red);
  }
  // l(q) from sums already reduced at this q (grad_keep)
  static __device__ __forceinline__ double neg_log_dens_with(const Target& t, int dim, int lane,
                                                             const double (&q)[NV],
                                                             const double (&red)[Target::NRED + 1]) {
    if constexpr (WHOLE) return whole_nld(t, dim, lane, q);
    else return pair_neg_log_dens_with(t, dim, lane, q, red);
  }
  static __device__ __forceinline__ double neg_log_dens(const Target& t, int dim, int lane,
                                                        const double (&q)[NV]) {
    if constexpr (WHOLE) return whole_nld(t, dim, lane, q);
    else return pair_neg_log_dens(t, dim, lane, q);
  }

  // ---- pair interface (targets.cuh)
  static __device__ __forceinline__ void pair_grad(const Target& t, int dim, int lane,
                                                   const double (&q)[NV], double (&g)[NV]) {
    double red[Target::NRED + 1];
#pragma unroll
    for (int r = 0; r < Target::NRED; ++r) red[r] = 0.0;
    if (Target::NRED > 0) {
#pragma unroll
      for (int k = 0; k < KP; ++k) {
        const int i = 2 * lane + 64 * k;
        if (i < dim) t.accumulate(i, q[2 * k], q[2 * k + 1], red);
      }
#pragma unroll
      for (int r = 0; r < Target::NRED; ++r) red[r] = warp_sum(red[r]);
    }
#pragma unroll
    for (int k = 0; k < KP; ++k) {
      const int i = 2 * lane + 64 * k;
      t.grad_pair(i, q[2 * k], q[2 * k + 1], red, g[2 * k], g[2 * k + 1]);
      if (i >= dim) g[2 * k] = 0.0;
      if (i + 1 >= dim) g[2 * k + 1] = 0.0;
    }
  }

  static __device__ __forceinline__ void pair_grad_keep(const Target& t, int dim, int lane,
                                                        const double (&q)[NV], double (&g)[NV],
                                                        double (&red)[Target::NRED + 1]) {
#pragma unroll
    for (int r = 0; r < Target::NRED + 1; ++r) red[r] = 0.0;
    if (Target::NRED > 0) {
#pragma unroll
      for (int k = 0; k < KP; ++k) {
        const int i = 2 * lane + 64 * k;
        if (i < dim) t.accumulate(i, q[2 * k], q[2 * k + 1], red);
      }
#pragma unroll
      for (int r = 0; r < Target::NRED; ++r) red[r] = warp_sum(red[r]);
    }
#pragma unroll
    for (int k = 0; k < KP; ++k) {
      const int i = 2 * lane + 64 * k;
      t.grad_pair(i, q[2 * k], q[2 * k + 1], red, g[2 * k], g[2 * k + 1]);
      if (i >= dim) g[2 * k] = 0.0;
      if (i + 1 >= dim) g[2 * k + 1] = 0.0;
    }
  }
  static __device__ __forceinline__ double pair_neg_log_dens_with(
      const Target& t, int dim, int lane, const double (&q)[NV],
      const double (&red)[Target::NRED + 1]) {
    double l = 0.0;
#pragma unroll
    for (int k = 0; k < KP; ++k) {
      const int i = 2 * lane + 64 * k;
      if (i < dim) l += t.nld_pair(i, q[2 * k], q[2 * k + 1], red);
    }
    return warp_sum(l);
  }

  static __device__ __forceinline__ double pair_neg_log_dens(const Target& t, int dim, int lane,
                                                             const double (&q)[NV]) {
    double red[Target::NRED + 1];
#pragma unroll
    for (int r = 0; r < Target::NRED; ++r) red[r] = 0.0;
    if (Target::NRED > 0) {
#pragma unroll
      for (int k = 0; k < KP; ++k) {
        const int i = 2 * lane + 64 * k;
        if (i < dim) t.accumulate(i, q[2 * k], q[2 * k + 1], red);
      }
#pragma unroll
      for (int r = 0; r < Target::NRED; ++r) red[r] = warp_sum(red[r]);
    }
    double l = 0.0;
#pragma unroll
    for (int k = 0; k < KP; ++k) {
      const int i = 2 * lane + 64 * k;
      if (i < dim) l += t.nld_pair(i, q[2 * k], q[2 * k + 1], red);
    }
    return warp_sum(l);
  }

};

template <class Target, int KP, int CPW, bool GAUSS = false>
__global__ void __launch_bounds__(128)
    leapfrog_generic_kernel(const double* q_in, const double* p_in,
                            double* q_out, double* p_out,
                            const int32_t* __restrict__ dir, int64_t n_chains, int dim,
                            double step_size, int n_steps, FlowSchedule sched, int metric_kind,
                            const double* __restrict__ minv,
                            ModelArgs model, double* __restrict__ h_out,
                            int32_t* __restrict__ status, int32_t* __restrict__ n_done) {
  using K = LeapfrogGeneric<Target, KP, CPW>;
  constexpr int NV = K::NV;
  extern __shared__ double smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int warps_per_block = blockDim.x >> 5;
  double* psm = smem + (size_t)warp * CPW * 64 * KP;
  const Target target(model, dim);
  const bool even = (dim & 1) == 0;

  const int64_t n_groups = (n_chains + CPW - 1) / CPW;
  for (int64_t grp = (int64_t)blockIdx.x * warps_per_block + warp; grp < n_groups;
       grp += (int64_t)gridDim.x * warps_per_block) {
    double q[CPW][NV], p[CPW][NV], g[CPW][NV], v[CPW][NV];
    double dt[CPW];
    int ns[CPW];
    int ns_max = 0;
#pragma unroll
    for (int c = 0; c < CPW; ++c) {
      const int64_t ch = grp * CPW + c;
      const bool live = ch < n_chains;
      const double eps = (live && sched.step_sizes != nullptr) ? sched.step_sizes[ch] : step_size;
      dt[c] = (live && dir != nullptr) ? (double)dir[ch] * eps : eps;
      ns[c] = !live ? 0 : (sched.n_steps != nullptr ? min(sched.n_steps[ch], n_steps) : n_steps);
      ns_max = max(ns_max, ns[c]);
#pragma unroll
      for (int k = 0; k < KP; ++k) {
        const int i = 2 * lane + 64 * k;
        double q0 = 0, q1 = 0, p0 = 0, p1 = 0;
        if (live && i < dim) {
          const size_t o = (size_t)ch * dim + i;
          if (even) {
            const double2 a = *reinterpret_cast<const double2*>(q_in + o);
            const double2 b = *reinterpret_cast<const double2*>(p_in + o);
            q0 = a.x, q1 = a.y, p0 = b.x, p1 = b.y;
          } else {
            q0 = q_in[o], p0 = p_in[o];
            if (i + 1 < dim) q1 = q_in[o + 1], p1 = p_in[o + 1];
          }
        }
        q[c][2 * k] = q0, q[c][2 * k + 1] = q1, p[c][2 * k] = p0, p[c][2 * k + 1] = p1;
      }
      K::grad(target, dim, lane, q[c], g[c]);
    }
    for (int s = 0; s < ns_max; ++s) {
      // chains whose own trajectory length is reached stop moving (updates predicated off)
      for (int f = 0; f < sched.n; ++f) {
        if (GAUSS && ((sched.drift_mask >> f) & 1u)) {
          // GaussianEuclideanMetricSystem.h2_flow (systems.py:464-474): exact flow of
          // h2 = q.q/2 + p.M^-1 p/2 in the eigenbasis of M, w = 1/sqrt(eigval):
          //   q' = U (cos(w dt) U^T q + (sin(w dt) w) U^T p)
          //   p' = U (cos(w dt) U^T p - (sin(w dt) / w) U^T q)
          if (metric_kind == MB200_METRIC_DENSE) {
            int drift_idx = 0;
            for (int ff = 0; ff < f; ++ff) drift_idx += (sched.drift_mask >> ff) & 1u;
            const double* cqq = sched.rot + (size_t)drift_idx * 3 * dim * dim;
            const double* cqp = cqq + (size_t)dim * dim;
            const double* cpq = cqp + (size_t)dim * dim;
            double w1[CPW][NV], w2[CPW][NV];
            inv_metric_apply<KP, CPW>(metric_kind, cqq, dim, lane, psm, q, v);
            inv_metric_apply<KP, CPW>(metric_kind, cqp, dim, lane, psm, p, w1);
            inv_metric_apply<KP, CPW>(metric_kind, cpq, dim, lane, psm, q, w2);
#pragma unroll
            for (int c = 0; c < CPW; ++c) {
              const double sgn = dt[c] < 0.0 ? -1.0 : 1.0;  // sin is odd in dt
#pragma unroll
              for (int e = 0; e < NV; ++e)
                if (s < ns[c]) q[c][e] = __dadd_rn(v[c][e], __dmul_rn(sgn, w1[c][e]));
            }
            inv_metric_apply<KP, CPW>(metric_kind, cqq, dim, lane, psm, p, v);
#pragma unroll
            for (int c = 0; c < CPW; ++c) {
              if (s >= ns[c]) continue;
              const double sgn = dt[c] < 0.0 ? -1.0 : 1.0;
#pragma unroll
              for (int e = 0; e < NV; ++e) p[c][e] = __dadd_rn(v[c][e], __dmul_rn(sgn, w2[c][e]));
              K::grad(target, dim, lane, q[c], g[c]);
            }
          } else {
#pragma unroll
            for (int c = 0; c < CPW; ++c) {
              if (s >= ns[c]) continue;
              const double dtf = sched.coef[f] * dt[c];
#pragma unroll
              for (int k = 0; k < KP; ++k) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const int i = 2 * lane + 64 * k + h;
                  const int e = 2 * k + h;
                  double om = 1.0;
                  if (metric_kind == MB200_METRIC_DIAGONAL)
                    om = (i < dim) ? 1.0 / sqrt(sched.rot[i]) : 1.0;
                  double sn, cs;
                  sincos(__dmul_rn(om, dtf), &sn, &cs);
                  const double qe = q[c][e], pe = p[c][e];
                  q[c][e] = __dadd_rn(__dmul_rn(cs, qe), __dmul_rn(__dmul_rn(sn, om), pe));
                  p[c][e] = __dsub_rn(__dmul_rn(cs, pe), __dmul_rn(__ddiv_rn(sn, om), qe));
                }
              }
              K::grad(target, dim, lane, q[c], g[c]);
            }
          }
        } else if ((sched.drift_mask >> f) & 1u) {
          // h2_flow: q += (c*dt) * M^-1 p (systems.py:362-363); gradient re-evaluated at the new q
          // (the reference's cache on `pos` is invalidated: states.py:248-258)
          inv_metric_apply<KP, CPW>(metric_kind, minv, dim, lane, psm, p, v);
#pragma unroll
          for (int c = 0; c < CPW; ++c) {
            if (s >= ns[c]) continue;
            const double dtf = sched.coef[f] * dt[c];
#pragma unroll
            for (int e = 0; e < NV; ++e) q[c][e] = __dadd_rn(q[c][e], __dmul_rn(dtf, v[c][e]));
            K::grad(target, dim, lane, q[c], g[c]);
          }
        } else {
          // h1_flow: p -= (c*dt) * grad -- product and difference rounded separately, exactly
          // as NumPy evaluates `state.mom -= dt * self.dh1_dpos(state)` (systems.py:152)
#pragma unroll
          for (int c = 0; c < CPW; ++c) {
            if (s >= ns[c]) continue;
            const double dtf = sched.coef[f] * dt[c];
#pragma unroll
            for (int e = 0; e < NV; ++e) p[c][e] = __dsub_rn(p[c][e], __dmul_rn(dtf, g[c][e]));
          }
        }
      }
    }
    if (h_out != nullptr) inv_metric_apply<KP, CPW>(metric_kind, minv, dim, lane, psm, p, v);
#pragma unroll
    for (int c = 0; c < CPW; ++c) {
      const int64_t ch = grp * CPW + c;
      if (ch >= n_chains) continue;
#pragma unroll
      for (int k = 0; k < KP; ++k) {
        const int i = 2 * lane + 64 * k;
        if (i < dim) {
          const size_t o = (size_t)ch * dim + i;
          if (even) {
            *reinterpret_cast<double2*>(q_out + o) = make_double2(q[c][2 * k], q[c][2 * k + 1]);
            *reinterpret_cast<double2*>(p_out + o) = make_double2(p[c][2 * k], p[c][2 * k + 1]);
          } else {
            q_out[o] = q[c][2 * k], p_out[o] = p[c][2 * k];
            if (i + 1 < dim) q_out[o + 1] = q[c][2 * k + 1], p_out[o + 1] = p[c][2 * k + 1];
          }
        }
      }
      if (h_out != nullptr) {
        double kin = 0.0;
#pragma unroll
        for (int e = 0; e < NV; ++e) kin = fma(p[c][e], v[c][e], kin);
        kin = warp_sum(kin);
        double l = K::neg_log_dens(target, dim, lane, q[c]);
        if (GAUSS) {  // h2 = q.q/2 + p.M^-1 p/2 (systems.py:450-453)
          double qq = 0.0;
#pragma unroll
          for (int e = 0; e < NV; ++e) qq = fma(q[c][e], q[c][e], qq);
          l += 0.5 * warp_sum(qq);
        }
        if (lane == 0) h_out[ch] = l + 0.5 * kin;
      }
      if (lane == 0) {
        if (status != nullptr) status[ch] = MB200_STATUS_OK;
        if (n_done != nullptr) n_done[ch] = ns[c];
        if (model.counters != nullptr)  // one gradient per position update + the initial one
          model.counters[ch * MB200_N_COUNTERS + MB200_COUNT_GRAD] +=
              1 + ns[c] * __popc(sched.drift_mask & ((1u << sched.n) - 1u));
      }
    }
  }
}

// Individual pieces of the Euclidean system for callers outside `Integrator.step`
// (System.neg_log_dens / grad_neg_log_dens / dh2_dmom / h2: systems.py:97-119, 348-354).
// Any of the four outputs may be NULL.
template <class Target, int KP>
__global__ void __launch_bounds__(128)
    euclidean_eval_kernel(const double* __restrict__ q_in, const double* __restrict__ p_in,
                          int64_t n_chains, int dim, int metric_kind,
                          const double* __restrict__ minv, ModelArgs model,
                          double* __restrict__ nld_out, double* __restrict__ grad_out,
                          double* __restrict__ vel_out, double* __restrict__ kin_out) {
  using K = LeapfrogGeneric<Target, KP, 1>;
  constexpr int NV = 2 * KP;
  extern __shared__ double smem[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  double* psm = smem + (size_t)warp * 64 * KP;
  const Target target(model, dim);
  for (int64_t ch = (int64_t)blockIdx.x * wpb + warp; ch < n_chains;
       ch += (int64_t)gridDim.x * wpb) {
    double q[NV], p[1][NV], v[1][NV], g[NV];
#pragma unroll
    for (int e = 0; e < NV; ++e) {
      const int i = 2 * lane + 64 * (e >> 1) + (e & 1);
      q[e] = (i < dim) ? q_in[(size_t)ch * dim + i] : 0.0;
      p[0][e] = (i < dim) ? p_in[(size_t)ch * dim + i] : 0.0;
    }
    if (nld_out != nullptr) {
      const double l = K::neg_log_dens(target, dim, lane, q);
      if (lane == 0) nld_out[ch] = l;
    }
    if (grad_out != nullptr) {
      K::grad(target, dim, lane, q, g);
#pragma unroll
      for (int e = 0; e < NV; ++e) {
        const int i = 2 * lane + 64 * (e >> 1) + (e & 1);
        if (i < dim) grad_out[(size_t)ch * dim + i] = g[e];
      }
    }
    if (vel_out != nullptr || kin_out != nullptr) {
      inv_metric_apply<KP, 1>(metric_kind, minv, dim, lane, psm, p, v);
      if (vel_out != nullptr) {
#pragma unroll
        for (int e = 0; e < NV; ++e) {
          const int i = 2 * lane + 64 * (e >> 1) + (e & 1);
          if (i < dim) vel_out[(size_t)ch * dim + i] = v[0][e];
        }
      }
      if (kin_out != nullptr) {
        double kin = 0.0;
#pragma unroll
        for (int e = 0; e < NV; ++e) kin = fma(p[0][e], v[0][e], kin);
        kin = warp_sum(kin);
        if (lane == 0) kin_out[ch] = 0.5 * kin;
      }
    }
  }
}

}  // namespace mb200
