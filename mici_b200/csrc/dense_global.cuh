// K2g: per-chain DENSE position-dependent metric for dimensions whose D x D matrices do not fit in
// shared memory (config C4: D = 512) -- blocked Cholesky, triangular solves, explicit inverse and
// the two gradient matrices on the FP64 tensor pipe (DMMA m8n8k4), matrices in a per-CTA global
// workspace (L2 / HBM), panels staged in shared memory.
//
// Replaces, per chain (reference paths):
//   DensePositiveDefiniteMatrix.factor   matrices.py:1161-1173   L = chol(M)
//   .inv / InverseTriangularMatrix       matrices.py:1183-1188, 897-912   M^-1 = L^-T L^-1
//   .log_abs_det                         matrices.py:982-984     2 sum log L_ii
//   .grad_log_abs_det                    matrices.py:1175-1177   M^-1 (dense, explicit)
//   .grad_quadratic_form_inv             matrices.py:1179-1181   -(M^-1 p)(M^-1 p)^T
//   DenseRiemannianMetricSystem          systems.py:1710-1760, 1381-1399 (vjp_metric_func on both)
//
// One CTA (8 warps) per chain.  Right-looking blocked Cholesky with 32-column panels:
//   diagonal block   one warp, one row per lane in registers (warp_chol32), its inverse W = L_kk^-1
//                    by the same warp (columns of W per lane)
//   panel            L_ik = A_ik W^T as 32x32x32 DMMA products, staged in shared memory
//   trailing update  A_ij -= L_ik L_jk^T for all block pairs i >= j > k: one 32x32 tile per warp,
//                    A / B fragments from the shared-memory panel (B through the "col" operand =
//                    rows of L), C tiles streamed from / to the workspace
// The triangular solves use the stored W_kk (blocked substitution, one 32-wide block per step);
// the explicit inverse is X = L^-1 by block rows followed by M^-1 = X^T X, both on DMMA tiles.
// A metric MODEL supplies the matrix and its vector-Jacobian products (systems.py:1335-1358):
//   fill(q, M)            M(q) into the workspace matrix
//   vjp_dense(q, V, out)  out_k = sum_ij V_ij dM_ij/dq_k for a dense symmetric V (here V = M^-1)
//   vjp_rank1(q, w, out)  the same for V = -w w^T without forming it (the generic route that
//                         forms -w w^T in the workspace and calls vjp_dense is kept: mp[3] != 0)
// A registry model fills through entry(q, i, j), lower triangle only.  A model with its own
// fill(k, q, M, ld) (the user model of user_riemannian.cuh) writes the whole n x n matrix; the
// policy then checks every entry for finiteness and writes the identity padding itself.  A model
// without vjp_rank1 always takes the generic route, and mp[3] is never read for it.
#pragma once
#include "riemannian.cuh"

namespace mb200 {

constexpr int DG_THREADS = 256;
constexpr int DG_NB = 32;
constexpr int DG_LDP = 36;  // shared-memory row stride (doubles): rows shift by 32 B mod 128 B

__device__ __forceinline__ void dg_dmma(double& c0, double& c1, double a, double b) {
  asm volatile(
      "mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
      : "+d"(c0), "+d"(c1)
      : "d"(a), "d"(b));
}

struct DgWork {
  int n, np, nblk;
  double *L, *X, *Minv, *W;      // global: [np*np] x 3, [nblk*32*32]
  double *panel, *dblk, *wblk;   // shared
};

__host__ __device__ inline size_t dg_workspace_doubles(int dim) {
  const size_t np = (size_t)dg_padded_dim(dim);
  return 3 * np * np + (np / DG_NB) * DG_NB * DG_NB;
}

// a chain's layout under this policy
__host__ __device__ inline RmLayout dg_layout(int dim) {
  return RmLayout{dim, RM_DENSE_GLOBAL, 0, 0, false};
}

__device__ inline void dg_attach(DgWork& g, const RmWork& w, const ModelArgs& m) {
  g.n = w.dim;
  g.np = dg_padded_dim(w.dim);
  g.nblk = g.np / DG_NB;
  double* base = m.workspace + (size_t)blockIdx.x * m.ws_stride;
  const size_t sq = (size_t)g.np * g.np;
  g.L = base;
  g.X = base + sq;
  g.Minv = base + 2 * sq;
  g.W = base + 3 * sq;
  g.panel = w.extra;
  g.dblk = w.extra + (size_t)(g.np > 32 ? g.np - 32 : 32) * DG_LDP;
  g.wblk = g.dblk + 32 * DG_LDP;
}

// Cholesky factor of a 32 x 32 SPD block held one row per lane (rowv[c] valid for c <= lane);
// entries above the diagonal end up undefined.  Returns false on a non-positive / non-finite pivot.
__device__ __forceinline__ bool warp_chol32(double (&rowv)[32], double (&rdiag)[32], int lane) {
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const double d = __shfl_sync(FULL_MASK, rowv[j], j);
    if (!(d > 0.0) || isinf(d)) ok = false;  // warp-uniform
    // this warp is the critical path of every panel step: one reciprocal square root (and two
    // multiplications) per column instead of a square root and a division
    const double rs = rsqrt(d);
    const double l = d * rs;
    rdiag[j] = rs;  // 1 / L[j][j], reused by the inversion below
    const double x = (lane == j) ? l : rowv[j] * rs;
    rowv[j] = x;
#pragma unroll
    for (int c = j + 1; c < 32; ++c) {
      const double xc = __shfl_sync(FULL_MASK, x, c);  // L[c][j]
      rowv[c] -= x * xc;                                // used for lane >= c only
    }
  }
  return ok;
}

// Inverse of the lower-triangular 32 x 32 factor held one row per lane: lane c returns column c of
// W = L^-1 in w[i] (zero for i < c).  rdiag[i] = 1 / L[i][i].
__device__ __forceinline__ void warp_trinv32(const double (&rowv)[32], const double (&rdiag)[32],
                                             double (&w)[32], int lane) {
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    // two partial sums: halves the dependent chain of row i
    double s0 = (lane == i) ? 1.0 : 0.0, s1 = 0.0;
#pragma unroll
    for (int k = 0; k < i; ++k) {
      const double lik = __shfl_sync(FULL_MASK, rowv[k], i);
      if (k & 1) s1 -= lik * w[k];
      else s0 -= lik * w[k];
    }
    w[i] = (s0 + s1) * rdiag[i];
  }
}

// acc[4][4][2] += A(32 x 4K) * B^T(32 x 4K)^T with both operands given by ROWS (row stride lda / ldb
// doubles): A fragment lane (r, c) = A[8 mt + r][4 ks + c], B fragment = B[8 nt + r][4 ks + c].
__device__ __forceinline__ void dg_tile_abt(double (&acc)[4][4][2], const double* A, int lda,
                                            const double* B, int ldb, int ksteps, int r, int c) {
  for (int ks = 0; ks < ksteps; ++ks) {
    double a[4], b[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      a[t] = A[(size_t)(8 * t + r) * lda + 4 * ks + c];
      b[t] = B[(size_t)(8 * t + r) * ldb + 4 * ks + c];
    }
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) dg_dmma(acc[mt][nt][0], acc[mt][nt][1], a[mt], b[nt]);
  }
}

// acc += A(32 x 4K, by rows) * B(4K x 32, by rows: B fragment lane (r, c) = B[4 ks + c][8 nt + r])
__device__ __forceinline__ void dg_tile_ab(double (&acc)[4][4][2], const double* A, int lda,
                                           const double* B, int ldb, int ksteps, int r, int c) {
  for (int ks = 0; ks < ksteps; ++ks) {
    double a[4], b[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      a[t] = A[(size_t)(8 * t + r) * lda + 4 * ks + c];
      b[t] = B[(size_t)(4 * ks + c) * ldb + 8 * t + r];
    }
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) dg_dmma(acc[mt][nt][0], acc[mt][nt][1], a[mt], b[nt]);
  }
}

// acc += A^T * B with A (4K x 32) and B (4K x 32) both by rows: A fragment lane (r, c) =
// A[4 ks + c][8 mt + r]
__device__ __forceinline__ void dg_tile_atb(double (&acc)[4][4][2], const double* A, int lda,
                                            const double* B, int ldb, int ksteps, int r, int c) {
  for (int ks = 0; ks < ksteps; ++ks) {
    double a[4], b[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      a[t] = A[(size_t)(4 * ks + c) * lda + 8 * t + r];
      b[t] = B[(size_t)(4 * ks + c) * ldb + 8 * t + r];
    }
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) dg_dmma(acc[mt][nt][0], acc[mt][nt][1], a[mt], b[nt]);
  }
}

__device__ __forceinline__ void dg_zero(double (&acc)[4][4][2]) {
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) acc[mt][nt][0] = 0.0, acc[mt][nt][1] = 0.0;
}

// Factor the 32 x 32 diagonal block at `Akk` (row stride np) and invert the factor: one warp, one
// row per lane.  Publishes L_kk to the workspace (strict upper part zeroed) and W_kk = L_kk^-1 to
// g.wblk (shared, for the panel product) and g.W (workspace, for the triangular solves).
__device__ __forceinline__ int dg_factor_diag(DgWork& g, int kb, int lane) {
  const int np = g.np;
  double* Akk = g.L + (size_t)(kb * DG_NB) * np + kb * DG_NB;
  double rowv[32], w[32], rdiag[32];
#pragma unroll
  for (int j = 0; j < 32; j += 2) {
    const double2 v = *reinterpret_cast<const double2*>(&Akk[(size_t)lane * np + j]);
    rowv[j] = v.x, rowv[j + 1] = v.y;
  }
  const int ok = warp_chol32(rowv, rdiag, lane) ? 1 : 0;
#pragma unroll
  for (int j = 0; j < 32; ++j) w[j] = 0.0;
  warp_trinv32(rowv, rdiag, w, lane);
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    Akk[(size_t)lane * np + j] = j <= lane ? rowv[j] : 0.0;
    g.wblk[j * DG_LDP + lane] = w[j];  // W[j][lane]
    g.W[(size_t)kb * DG_NB * DG_NB + j * DG_NB + lane] = w[j];
  }
  return ok;
}

// tile index t of the lower-triangular enumeration (0,0), (1,0), (1,1), (2,0), ... -> (bi, bj)
__device__ __forceinline__ void dg_tile_decode(int t, int& bi, int& bj) {
  bi = (int)((sqrtf(8.0f * (float)t + 1.0f) - 1.0f) * 0.5f);
  while (bi * (bi + 1) / 2 > t) --bi;
  while ((bi + 1) * (bi + 2) / 2 <= t) ++bi;
  bj = t - bi * (bi + 1) / 2;
}

// In-place blocked Cholesky of the SPD matrix in g.L (lower triangle referenced; on return the
// lower triangle holds L, the strict upper triangle of the diagonal blocks is zero, blocks above
// the diagonal are untouched) and W_kk = L_kk^-1 in g.W.  Returns false on a failed pivot
// (-> LinAlgError "Cholesky factorisation failed", matrices.py:1170-1172).
//
// Per 32-column panel: [panel product L_ik = A_ik W^T] -> barrier -> [trailing update, tiles
// handed out through a shared counter; warp 0 takes the tile of the NEXT diagonal block first and
// factors / inverts it while the other warps finish the update (look-ahead: the serial 32 x 32
// factorisation leaves the critical path)] -> barrier.  8 warps with 255 registers: 16 warps
// under a 128-register budget, and a register-prefetched next C tile, both measured slower
// (the diagonal-block code spills).
// The routines below are not inlined: DgWork reaches them through memory, where the compiler
// cannot see which of its pointers are shared and which global and would emit generic LD / ST for
// all of them (riemannian.cuh: RM_SHARED / RM_GLOBAL).  They work on a local copy with the address
// spaces stated.
#define DG_LOCAL(g, g_in)                                        \
  DgWork g = g_in;                                               \
  RM_SHARED(g.panel), RM_SHARED(g.dblk), RM_SHARED(g.wblk);      \
  RM_GLOBAL(g.L), RM_GLOBAL(g.X), RM_GLOBAL(g.Minv), RM_GLOBAL(g.W)

__device__ __noinline__ bool dg_cholesky(const Blk& k, DgWork& g_in) {
  DG_LOCAL(g, g_in);
  const int np = g.np, lane = k.lane, r = lane >> 2, c = lane & 3;
  int* counter = reinterpret_cast<int*>(g.dblk);  // shared work counter (+ failure flag)
  if (k.tid == 0) counter[0] = 0, counter[1] = 1;
  __syncthreads();
  if (k.warp == 0) {
    const int ok = dg_factor_diag(g, 0, lane);
    if (lane == 0) counter[1] = ok;
  }
  __syncthreads();
  for (int kb = 0; kb < g.nblk; ++kb) {
    if (counter[1] == 0) return false;  // uniform: written before the last barrier
    const int d0 = kb * DG_NB;
    const int m = np - d0 - DG_NB;  // rows below the diagonal block
    if (m == 0) break;
    // ---- panel: raw A[d0+32 .., d0 .. d0+32) into shared memory
    const double* Ap = g.L + (size_t)(d0 + DG_NB) * np + d0;
    for (int idx0 = k.tid; idx0 < m * 16; idx0 += 4 * k.nthr) {  // four loads in flight
      double2 v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int idx = idx0 + e * k.nthr;
        if (idx < m * 16)
          v[e] = *reinterpret_cast<const double2*>(Ap + (size_t)(idx >> 4) * np + 2 * (idx & 15));
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int idx = idx0 + e * k.nthr;
        if (idx < m * 16)
          *reinterpret_cast<double2*>(&g.panel[(idx >> 4) * DG_LDP + 2 * (idx & 15)]) = v[e];
      }
    }
    if (k.tid == 0) counter[0] = 1;  // tile 0 is reserved for warp 0
    __syncthreads();
    // L_ik = A_ik W^T, one 32-row block per warp, in place (a warp touches only its own rows)
    for (int ib = k.warp; ib < m / DG_NB; ib += k.nwarp) {
      double acc[4][4][2];
      dg_zero(acc);
      double* Pi = g.panel + (size_t)ib * DG_NB * DG_LDP;
      dg_tile_abt(acc, Pi, DG_LDP, g.wblk, DG_LDP, 8, r, c);
      __syncwarp();
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const double2 v = make_double2(acc[mt][nt][0], acc[mt][nt][1]);
          *reinterpret_cast<double2*>(&Pi[(8 * mt + r) * DG_LDP + 8 * nt + 2 * c]) = v;
          *reinterpret_cast<double2*>(
              &g.L[(size_t)(d0 + DG_NB + ib * DG_NB + 8 * mt + r) * np + d0 + 8 * nt + 2 * c]) = v;
        }
    }
    __syncthreads();
    // ---- trailing update: A_ij -= L_ik L_jk^T over the block pairs i >= j
    const int rb = m / DG_NB, ntiles = rb * (rb + 1) / 2;
    double* C0 = g.L + (size_t)(d0 + DG_NB) * np + d0 + DG_NB;
    auto tile_ptr = [&](int t, int& bi, int& bj) {
      dg_tile_decode(t, bi, bj);
      return C0 + (size_t)(bi * DG_NB) * np + bj * DG_NB;
    };
    auto next_tile = [&]() {
      int t = 0;
      if (lane == 0) t = atomicAdd(&counter[0], 1);
      return __shfl_sync(FULL_MASK, t, 0);
    };
    double cur[4][4][2];
    int t = (k.warp == 0) ? 0 : next_tile();
    while (t < ntiles) {
      int bi, bj;
      double* Cij = tile_ptr(t, bi, bj);
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const double2 v =
              *reinterpret_cast<const double2*>(&Cij[(size_t)(8 * mt + r) * np + 8 * nt + 2 * c]);
          cur[mt][nt][0] = v.x, cur[mt][nt][1] = v.y;
        }
      // cur -= L_i L_j^T: the A fragments enter negated
      {
        const double* A = g.panel + (size_t)bi * DG_NB * DG_LDP;
        const double* B = g.panel + (size_t)bj * DG_NB * DG_LDP;
        for (int ks = 0; ks < 8; ++ks) {
          double a[4], b[4];
#pragma unroll
          for (int tt = 0; tt < 4; ++tt) {
            a[tt] = -A[(8 * tt + r) * DG_LDP + 4 * ks + c];
            b[tt] = B[(8 * tt + r) * DG_LDP + 4 * ks + c];
          }
#pragma unroll
          for (int mt = 0; mt < 4; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) dg_dmma(cur[mt][nt][0], cur[mt][nt][1], a[mt], b[nt]);
        }
      }
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
          *reinterpret_cast<double2*>(&Cij[(size_t)(8 * mt + r) * np + 8 * nt + 2 * c]) =
              make_double2(cur[mt][nt][0], cur[mt][nt][1]);
      if (k.warp == 0 && t == 0) {
        // look-ahead: the tile just written is the next diagonal block
        __syncwarp();
        const int ok = dg_factor_diag(g, kb + 1, lane);
        if (lane == 0 && !ok) counter[1] = 0;
        __syncwarp();
      }
      t = next_tile();
    }
    __syncthreads();
  }
  return counter[1] != 0;
}

// x = L^-1 b (forward) then x = L^-T x (backward) with the stored diagonal-block inverses; b, x in
// shared memory (x may alias b), `tmp` a shared scratch vector of np doubles is NOT needed: the
// right-hand side is updated in place.  Only entries < g.n are meaningful (padding rows are the
// identity).
__device__ __noinline__ void dg_solve(const Blk& k, const DgWork& g_in, const double* b, double* x,
                                bool forward, bool backward) {
  DG_LOCAL(g, g_in);
  RM_SHARED(b), RM_SHARED(x);  // every caller passes per-chain vectors of the shared workspace
  const int np = g.np, n = g.n;
  for (int i = k.tid; i < n; i += k.nthr) x[i] = b[i];
  __syncthreads();
  double* y = g.dblk;  // 32-vector scratch (the block solution of the current step)
  if (forward) {
    for (int kb = 0; kb < g.nblk; ++kb) {
      const int d0 = kb * DG_NB;
      // y = W_kk x_kb: 8 threads per row (4 columns each), reduced with shuffles
      {
        const int row = k.tid >> 3, part = k.tid & 7;
        const double* Wk = g.W + (size_t)kb * DG_NB * DG_NB + (size_t)row * DG_NB + 4 * part;
        double s = 0.0;
        if (k.tid < 8 * DG_NB) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int gj = d0 + 4 * part + j;
            s = fma(Wk[j], gj < n ? x[gj] : 0.0, s);
          }
        }
        s += __shfl_xor_sync(FULL_MASK, s, 1);
        s += __shfl_xor_sync(FULL_MASK, s, 2);
        s += __shfl_xor_sync(FULL_MASK, s, 4);
        if (k.tid < 8 * DG_NB && part == 0) y[row] = s;
      }
      __syncthreads();
      if (k.tid < DG_NB && d0 + k.tid < n) x[d0 + k.tid] = y[k.tid];
      // x_i -= L[i, kb-block] y for the rows below: 8 threads per row (4 columns each: a row's 32
      // entries are one 256-byte piece read by 8 neighbouring lanes), reduced with shuffles; the
      // passes over row groups are independent loads (a thread per row was a chain of 32 loads)
      {
        const int part = k.tid & 7, rows_per_pass = k.nthr >> 3;
        const double y0 = y[4 * part], y1 = y[4 * part + 1], y2 = y[4 * part + 2],
                     y3 = y[4 * part + 3];
#pragma unroll 4
        for (int base = d0 + DG_NB; base < n; base += rows_per_pass) {
          const int i = base + (k.tid >> 3);
          double s = 0.0;
          if (i < n) {
            const double* Li = g.L + (size_t)i * np + d0 + 4 * part;
            s = fma(Li[3], y3, fma(Li[2], y2, fma(Li[1], y1, Li[0] * y0)));
          }
          s += __shfl_xor_sync(FULL_MASK, s, 1);
          s += __shfl_xor_sync(FULL_MASK, s, 2);
          s += __shfl_xor_sync(FULL_MASK, s, 4);
          if (i < n && part == 0) x[i] -= s;
        }
      }
      __syncthreads();
    }
  }
  if (backward) {
    for (int kb = g.nblk - 1; kb >= 0; --kb) {
      const int d0 = kb * DG_NB;
      // y = W_kk^T x_kb: 8 threads per output entry (4 rows of W each), reduced with shuffles
      {
        const int col = k.tid >> 3, part = k.tid & 7;
        const double* Wk = g.W + (size_t)kb * DG_NB * DG_NB + col;
        double s = 0.0;
        if (k.tid < 8 * DG_NB) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int jj = 4 * part + j, gj = d0 + jj;
            s = fma(Wk[(size_t)jj * DG_NB], gj < n ? x[gj] : 0.0, s);
          }
        }
        s += __shfl_xor_sync(FULL_MASK, s, 1);
        s += __shfl_xor_sync(FULL_MASK, s, 2);
        s += __shfl_xor_sync(FULL_MASK, s, 4);
        if (k.tid < 8 * DG_NB && part == 0) y[col] = s;
      }
      __syncthreads();
      if (k.tid < DG_NB && d0 + k.tid < n) x[d0 + k.tid] = y[k.tid];
      // x_col -= sum_j L[d0 + j][col] y_j for the columns to the left (coalesced along rows of L)
      for (int col = k.tid; col < d0; col += k.nthr) {
        double s = 0.0;
#pragma unroll 8
        for (int j = 0; j < DG_NB; ++j) s = fma(g.L[(size_t)(d0 + j) * np + col], y[j], s);
        x[col] -= s;
      }
      __syncthreads();
    }
  }
}

// Explicit inverse: X = L^-1 (block rows, X_ic = -W_ii sum_{c<=k<i} L_ik X_kc) then
// M^-1 = X^T X; both matrices in the workspace, M^-1 stored full (symmetric).
__device__ __noinline__ void dg_explicit_inverse(const Blk& k, DgWork& g_in) {
  DG_LOCAL(g, g_in);
  const int np = g.np, nb = g.nblk, lane = k.lane, r = lane >> 2, c = lane & 3;
  // ---- X = L^-1
  for (int i = 0; i < nb; ++i) {
    const double* Wi = g.W + (size_t)i * DG_NB * DG_NB;
    // stage W_ii (A operand of the first product) in shared memory
    for (int idx = k.tid; idx < DG_NB * DG_NB; idx += k.nthr)
      g.wblk[(idx >> 5) * DG_LDP + (idx & 31)] = Wi[idx];
    __syncthreads();
    // pass 1: Lt_ik = W_ii L_ik (k < i) into the shared panel, laid out [32 x 32 i], stride ldt
    const int ldt = DG_NB * i + 4;
    for (int kb = k.warp; kb < i; kb += k.nwarp) {
      double acc[4][4][2];
      dg_zero(acc);
      dg_tile_ab(acc, g.wblk, DG_LDP, g.L + (size_t)(i * DG_NB) * np + kb * DG_NB, np, 8, r, c);
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
          *reinterpret_cast<double2*>(&g.panel[(8 * mt + r) * ldt + kb * DG_NB + 8 * nt + 2 * c]) =
              make_double2(acc[mt][nt][0], acc[mt][nt][1]);
    }
    __syncthreads();
    // pass 2: X_ic = -sum_{k=c}^{i-1} Lt_ik X_kc ; X_ii = W_ii ; blocks right of the diagonal zero
    for (int cb = k.warp; cb <= i; cb += k.nwarp) {
      double* Xic = g.X + (size_t)(i * DG_NB) * np + cb * DG_NB;
      if (cb == i) {
#pragma unroll
        for (int mt = 0; mt < 4; ++mt)
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) {
            const int row = 8 * mt + r, col = 8 * nt + 2 * c;
            *reinterpret_cast<double2*>(&Xic[(size_t)row * np + col]) =
                make_double2(g.wblk[row * DG_LDP + col], g.wblk[row * DG_LDP + col + 1]);
          }
        continue;
      }
      double acc[4][4][2];
      dg_zero(acc);
      for (int kb = cb; kb < i; ++kb)
        dg_tile_ab(acc, g.panel + kb * DG_NB, ldt, g.X + (size_t)(kb * DG_NB) * np + cb * DG_NB, np,
                   8, r, c);
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
          *reinterpret_cast<double2*>(&Xic[(size_t)(8 * mt + r) * np + 8 * nt + 2 * c]) =
              make_double2(-acc[mt][nt][0], -acc[mt][nt][1]);
    }
    __syncthreads();
  }
  // ---- M^-1 = X^T X: tile (a, b), a >= b: sum over block rows kb >= a of X_ka^T X_kb
  int cnt = 0;
  for (int a = 0; a < nb; ++a)
    for (int b = 0; b <= a; ++b, ++cnt) {
      if (cnt % k.nwarp != k.warp) continue;
      double acc[4][4][2];
      dg_zero(acc);
      for (int kb = a; kb < nb; ++kb)
        dg_tile_atb(acc, g.X + (size_t)(kb * DG_NB) * np + a * DG_NB, np,
                    g.X + (size_t)(kb * DG_NB) * np + b * DG_NB, np, 8, r, c);
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int row = a * DG_NB + 8 * mt + r, col = b * DG_NB + 8 * nt + 2 * c;
          *reinterpret_cast<double2*>(&g.Minv[(size_t)row * np + col]) =
              make_double2(acc[mt][nt][0], acc[mt][nt][1]);
          if (a != b) {
            g.Minv[(size_t)col * np + row] = acc[mt][nt][0];
            g.Minv[(size_t)(col + 1) * np + row] = acc[mt][nt][1];
          }
        }
    }
  __syncthreads();
  // diagonal tiles were written from the (a, a) product in full: already symmetric up to rounding;
  // make them exactly symmetric (lower -> upper)
  for (int idx = k.tid; idx < nb * DG_NB * DG_NB; idx += k.nthr) {
    const int a = idx / (DG_NB * DG_NB), rem = idx % (DG_NB * DG_NB);
    const int i = rem / DG_NB, j = rem % DG_NB;
    if (j > i)
      g.Minv[(size_t)(a * DG_NB + i) * np + a * DG_NB + j] =
          g.Minv[(size_t)(a * DG_NB + j) * np + a * DG_NB + i];
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// Metric models (device side of mici_b200.targets metric registry)
// ---------------------------------------------------------------------------------------------

// M(q) = B + c q q^T ; vjp(V) = c (V + V^T) q
struct Rank1Model {
  const double* B;
  double c;
  int n;
  __device__ Rank1Model(const ModelArgs& m, int dim) : B(m.maux), c(m.mp[0]), n(dim) {}
  __device__ __forceinline__ double entry(const double* q, int i, int j) const {
    const double* const Bg = B;
    RM_GLOBAL(Bg);
    return Bg[(size_t)i * n + j] + c * (q[i] * q[j]);
  }
  // out = c (V + V^T) q for the symmetric V stored full with stride ld
  __device__ void vjp_dense(const Blk& k, const double* q, const double* V, int ld, double* out) const {
    for (int i = k.warp; i < n; i += k.nwarp) {
      double s = 0.0;
      for (int j = k.lane; j < n; j += 32) s = fma(V[(size_t)i * ld + j], q[j], s);
      s = warp_sum(s);
      if (k.lane == 0) out[i] = c * (s + s);
    }
    __syncthreads();
  }
  // V = -w w^T: V q = -w (w.q)
  __device__ void vjp_rank1(const Blk& k, const double* q, const double* w, double* out) const {
    double s = 0.0;
    for (int i = k.tid; i < n; i += k.nthr) s = fma(w[i], q[i], s);
    const double wq = block_sum(k, s);
    for (int i = k.tid; i < n; i += k.nthr) {
      const double vq = -(w[i] * wq);
      out[i] = c * (vq + vq);
    }
    __syncthreads();
  }
};

// M(q) = B + c (q q^T) o S, S symmetric positive definite (Schur product theorem: M is SPD and in
// general of full rank: no low-rank shortcut exists); dM_ij/dq_k = c S_ij (d_ik q_j + d_jk q_i),
// vjp(V)_k = c sum_j (V_kj + V_jk) S_kj q_j.  aux = [B | S], params: c.
struct HadamardModel {
  const double *B, *S;
  double c;
  int n;
  __device__ HadamardModel(const ModelArgs& m, int dim)
      : B(m.maux), S(m.maux + (size_t)dim * dim), c(m.mp[0]), n(dim) {}
  __device__ __forceinline__ double entry(const double* q, int i, int j) const {
    const double* const Bg = B;
    const double* const Sg = S;
    RM_GLOBAL(Bg), RM_GLOBAL(Sg);
    return Bg[(size_t)i * n + j] + c * ((q[i] * q[j]) * Sg[(size_t)i * n + j]);
  }
  __device__ void vjp_dense(const Blk& k, const double* q, const double* V, int ld, double* out) const {
    for (int i = k.warp; i < n; i += k.nwarp) {
      double s = 0.0;
      for (int j = k.lane; j < n; j += 32)
        s = fma(V[(size_t)i * ld + j] * S[(size_t)i * n + j], q[j], s);
      s = warp_sum(s);
      if (k.lane == 0) out[i] = c * (s + s);
    }
    __syncthreads();
  }
  // V = -w w^T: out_k = -2 c w_k sum_j S_kj w_j q_j
  __device__ void vjp_rank1(const Blk& k, const double* q, const double* w, double* out) const {
    for (int i = k.warp; i < n; i += k.nwarp) {
      double s = 0.0;
      for (int j = k.lane; j < n; j += 32) s = fma(S[(size_t)i * n + j], w[j] * q[j], s);
      s = warp_sum(s);
      if (k.lane == 0) {
        const double vq = -(w[i] * s);
        out[i] = c * (vq + vq);
      }
    }
    __syncthreads();
  }
};

// ---------------------------------------------------------------------------------------------
// Metric policy (same interface as the shared-memory policies of riemannian.cuh)
// ---------------------------------------------------------------------------------------------

// true for models that fill the whole matrix themselves (`fill`) instead of entry by entry
template <class M, class = void>
struct dg_model_fills {
  static constexpr bool value = false;
};
template <class M>
struct dg_model_fills<M, decltype(void(&M::fill))> {
  static constexpr bool value = true;
};
// true for models with a rank-one VJP (`vjp_rank1`); the others take the generic route
template <class M, class = void>
struct dg_model_rank1 {
  static constexpr bool value = false;
};
template <class M>
struct dg_model_rank1<M, decltype(void(&M::vjp_rank1))> {
  static constexpr bool value = true;
};

template <class Target, class Model>
struct GlobalDenseMetricT {
  static constexpr bool SOFTABS = false;
  static constexpr RmPlace PLACE = RM_DENSE_GLOBAL;
  static constexpr int MIN_BLOCKS = 1;  // ~200 KB of shared memory per CTA: one CTA per SM
  static constexpr int THREADS = DG_THREADS;
  const Target& t;
  Model model;
  DgWork g;
  bool attached, have_inv, generic_rank1;
  const ModelArgs& margs;

  __device__ GlobalDenseMetricT(const Target& tt, const ModelArgs& m)
      : t(tt), model(m, tt.dim), attached(false), have_inv(false),
        generic_rank1(!dg_model_rank1<Model>::value || m.mp[3] != 0.0), margs(m) {}
  __device__ void reset() {}

  __device__ int build(const Blk& k, RmWork& w, const double* q) {
    if (!attached) {
      dg_attach(g, w, margs);
      attached = true;
    }
    have_inv = false;
    if constexpr (dg_model_fills<Model>::value) return build_filled(k, q);
    else return build_entries(k, q);
  }
  __device__ __forceinline__ int build_entries(const Blk& k, const double* q) {
    const int n = g.n, np = g.np;
    bool bad = false;
    // lower triangle only (the factorisation never reads above the diagonal blocks): one row
    // per warp, lanes along the row
    // (four entries per lane and pass: their loads of the model's matrices are independent
    // round trips to L2 -- one at a time this fill was 12 % of a C4 step)
    double* const Lg = g.L;
    RM_GLOBAL(Lg);
    for (int i = k.warp; i < np; i += k.nwarp) {
      const int jmax = (i | 31) + 1;  // through the end of the row's diagonal block
      for (int j0 = k.lane; j0 < jmax; j0 += 128) {
        double v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int j = j0 + 32 * e;
          v[e] = (i == j) ? 1.0 : 0.0;  // identity padding
          if (j < jmax && i < n && j < n) v[e] = model.entry(q, i, j);
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int j = j0 + 32 * e;
          if (j < jmax) {
            if (i < n && j < n && !isfinite(v[e])) bad = true;
            Lg[(size_t)i * np + j] = v[e];
          }
        }
      }
    }
    if (block_any(k, bad)) return MB200_STATUS_LINALG;  // "Array is not finite" (:211-215)
    if (!dg_cholesky(k, g)) return MB200_STATUS_LINALG;
    return 0;
  }
  // the model writes M(q) into rows / columns [0, n) of g.L; every one of those n x n entries is
  // checked (both triangles: "Array is not finite", :211-215), then the rows and columns from n
  // to np are reset to the identity and the lower triangle is factored
  __device__ int build_filled(const Blk& k, const double* q) {
    const int n = g.n, np = g.np;
    double* const Lg = g.L;
    RM_GLOBAL(Lg);
    model.fill(k, q, Lg, np);
    bool bad = false;
    // one row per warp, lanes along the row
    for (int i = k.warp; i < np; i += k.nwarp) {
#pragma unroll 4
      for (int j = k.lane; j < np; j += 32) {
        if (i < n && j < n) {
          if (!isfinite(Lg[(size_t)i * np + j])) bad = true;
        } else {
          Lg[(size_t)i * np + j] = (i == j) ? 1.0 : 0.0;
        }
      }
    }
    if (block_any(k, bad)) return MB200_STATUS_LINALG;
    if (!dg_cholesky(k, g)) return MB200_STATUS_LINALG;
    return 0;
  }
  __device__ double log_abs_det(const Blk& k, RmWork&) const {
    double s = 0.0;
    for (int i = k.tid; i < g.n; i += k.nthr) s += log(fabs(g.L[(size_t)i * g.np + i]));
    return 2.0 * block_sum(k, s);  // matrices.py:982-984
  }
  __device__ void inv_matvec(const Blk& k, RmWork&, const double* v, double* out) const {
    dg_solve(k, g, v, out, true, true);
  }
  // out = L v (sqrt of a DensePositiveDefiniteMatrix is its Cholesky factor, matrices.py:1212-1216)
  __device__ bool sqrt_matvec(const Blk& k, RmWork&, const double* v, double* out) const {
    for (int i = k.warp; i < g.n; i += k.nwarp) {
      double s = 0.0;
      for (int j = k.lane; j <= i; j += 32) s = fma(g.L[(size_t)i * g.np + j], v[j], s);
      s = warp_sum(s);
      if (k.lane == 0) out[i] = s;
    }
    __syncthreads();
    return true;
  }
  // vjp(grad_log_abs_det) with grad_log_abs_det = M^-1 explicit (matrices.py:1175-1177)
  __device__ void vjp_grad_log_abs_det(const Blk& k, RmWork&, const double* q, double* out) {
    if (!have_inv) {
      dg_explicit_inverse(k, g);
      have_inv = true;
    }
    model.vjp_dense(k, q, g.Minv, g.np, out);
  }
  // vjp(grad_quadratic_form_inv(p)), grad = -(M^-1 p)(M^-1 p)^T (matrices.py:1179-1181)
  __device__ void vjp_grad_quad_inv(const Blk& k, RmWork& w, const double* q, const double* p,
                                    double* out) {
    dg_solve(k, g, p, w.ev, true, true);  // w = M^-1 p
    if constexpr (dg_model_rank1<Model>::value) {
      if (!generic_rank1) {
        model.vjp_rank1(k, q, w.ev, out);
        return;
      }
    }
    // generic route: materialise V = -w w^T in the workspace (X is free between inverses)
    const int n = g.n, np = g.np;
    for (int idx = k.tid; idx < n * n; idx += k.nthr) {
      const int i = idx / n, j = idx - i * n;
      g.X[(size_t)i * np + j] = -(w.ev[i] * w.ev[j]);
    }
    __syncthreads();
    model.vjp_dense(k, q, g.X, np, out);
  }
};

template <class Target>
using GlobalDenseRank1 = GlobalDenseMetricT<Target, Rank1Model>;
template <class Target>
using GlobalDenseHadamard = GlobalDenseMetricT<Target, HadamardModel>;

#ifndef __CUDACC_RTC__  // library self-test: kept out of the run-time compiled user images
// Diagnostic kernel: factor / solve / invert arbitrary SPD matrices (one CTA per matrix) so that
// the blocked routines can be checked against numpy.linalg directly (tests/test_parity_gpu.py).
static __global__ void __launch_bounds__(DG_THREADS)
    dense_global_selftest_kernel(const double* __restrict__ mats, const double* __restrict__ rhs,
                                 int64_t n_mats, int dim, ModelArgs margs,
                                 double* __restrict__ chol_out, double* __restrict__ inv_out,
                                 double* __restrict__ sol_out, double* __restrict__ logdet_out,
                                 int32_t* __restrict__ status) {
  Blk k;
  RmWork w;
  rm_begin<false>(dg_layout(dim), margs, k, w);
  DgWork g;
  dg_attach(g, w, margs);
  const int n = dim, np = g.np;
  for (int64_t mi = blockIdx.x; mi < n_mats; mi += gridDim.x) {
    __syncthreads();
    const double* src = mats + (size_t)mi * n * n;
    for (int idx = k.tid; idx < np * np; idx += k.nthr) {
      const int i = idx / np, j = idx - i * np;
      g.L[idx] = (i < n && j < n) ? src[(size_t)i * n + j] : (i == j ? 1.0 : 0.0);
    }
    for (int i = k.tid; i < n; i += k.nthr) w.v1[i] = rhs[(size_t)mi * n + i];
    __syncthreads();
    const bool ok = dg_cholesky(k, g);
    if (ok) {
      dg_solve(k, g, w.v1, w.v2, true, true);
      dg_explicit_inverse(k, g);
      double s = 0.0;
      for (int i = k.tid; i < n; i += k.nthr) s += log(fabs(g.L[(size_t)i * np + i]));
      const double ld = 2.0 * block_sum(k, s);
      for (int idx = k.tid; idx < n * n; idx += k.nthr) {
        const int i = idx / n, j = idx - i * n;
        chol_out[(size_t)mi * n * n + idx] = j <= i ? g.L[(size_t)i * np + j] : 0.0;
        inv_out[(size_t)mi * n * n + idx] = g.Minv[(size_t)i * np + j];
      }
      for (int i = k.tid; i < n; i += k.nthr) sol_out[(size_t)mi * n + i] = w.v2[i];
      if (k.tid == 0) logdet_out[mi] = ld;
    }
    if (k.tid == 0) status[mi] = ok ? 0 : MB200_STATUS_LINALG;
  }
}
#endif

}  // namespace mb200
