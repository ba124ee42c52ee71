// Batched dense QP: primal-dual interior point (Mehrotra predictor-corrector), one warp per problem.
// Replaces the qpOASES active-set call of legged::WeightedWbc::update (legged_wbc/src/WeightedWbc.cpp:44-55):
//     min 1/2 x'(H + rho I)x + g'x   s.t.  lbA <= A x <= ubA
// rows with lbA == ubA are equalities, |bound| >= 1e19 means "no bound" (qpOASES::INFTY = 1e20), all-zero rows are
// dropped (the reference appends 3 zero rows per swing contact, WbcBase.cpp:212). rho is the Tikhonov weight that
// selects the least-norm point of the optimal face, as qpOASES' setToMPC() regularisation does (SURVEY App. C.6).
//
// Linear algebra per iteration, all in shared memory, float64:
//   K = H + rho I + D' diag(z/s) D      (span-aware rank-1 updates; WBC inequality rows touch 1..3 columns)
//   K = L L' (left-looking Cholesky, lanes over rows), Li = L^-1 (lane per column), V = Li Aeq', S = V'V = Ls Ls', Si = Ls^-1
//   every Newton solve is then a chain of mat-vecs (no sequential triangular solve on the critical path).
// The iteration around these Newton steps is qp_mehrotra_warp, which level 0 of the hierarchical WBC (hb_hoqp.cuh) runs too.
#pragma once
#include "hb_common.cuh"

namespace hb {

constexpr int QP_MAX_N = 80;    // variables (38 for the WBC; 78 for a lifted HoQP level: 38 decision + 40 slack variables)
constexpr int QP_MAX_EQ = 32;   // equality rows
constexpr int QP_MAX_IN = 96;   // one-sided inequality entries (two-sided rows count twice)
constexpr int QP_MAX_M = 160;   // rows of A

struct QpWorkspace {
  double *H, *Aeq, *K, *V, *S;
  double *kdi, *sdi;
  double *g, *x, *rd, *dx, *t1, *t2;
  double *beq, *y, *rp, *dy, *t3;
  double *f, *s, *z, *rs, *ds, *dz, *rc, *sgn, *wt;   // wt: per-entry weight / coefficient scratch (two-sided rows merged on their first entry)
  int *in_row, *in_c0, *in_c1, *in_pair, *ord, *eq_row;   // ord: entries in processing order, wide rows first, merged partners left out   // in_pair: partner entry of a two-sided row (-1 none, -2 merged into its partner)
  int ldn, ldv, lds;
  int me_cap, mi_cap;   // capacity of the equality / one-sided inequality lists
};

__host__ __device__ constexpr int qp_ld(int n) { return n | 1; }

// Lower triangle of a symmetric n x n matrix, row by row: entry (i, c), c <= i, at tri_row(i) + c
__host__ __device__ constexpr int tri_row(int i) { return i * (i + 1) / 2; }

// doubles needed by one warp for problems with n variables, <= me_cap equalities and <= mi_cap one-sided inequality entries;
// packed_h: H is kept as its packed lower triangle (see qp_solve_warp)
__host__ __device__ constexpr size_t qp_workspace_doubles(int n, int me_cap = QP_MAX_EQ, int mi_cap = QP_MAX_IN, bool packed_h = false) {
  const int ldn = qp_ld(n), lde = me_cap | 1;
  size_t d = 0;
  d += packed_h ? (size_t)tri_row(n) : (size_t)n * ldn;   // H
  d += (size_t)me_cap * ldn;       // Aeq
  d += (size_t)n * ldn;            // K
  d += (size_t)n * lde;            // V
  d += (size_t)me_cap * lde;       // S
  d += n + me_cap;                 // kdi, sdi
  d += 6 * (size_t)n;              // g x rd dx t1 t2
  d += 5 * (size_t)me_cap;         // beq y rp dy t3
  d += 9 * (size_t)mi_cap;         // f s z rs ds dz rc sgn wt
  d += (5 * (size_t)mi_cap + me_cap + 1) / 2 + 1;  // int arrays
  return d;
}

__device__ inline void qp_carve(double* base, int n, QpWorkspace& w, int me_cap = QP_MAX_EQ, int mi_cap = QP_MAX_IN, bool packed_h = false) {
  const int ldn = qp_ld(n), lde = me_cap | 1;
  w.ldn = ldn; w.ldv = lde; w.lds = lde; w.me_cap = me_cap; w.mi_cap = mi_cap;
  double* p = base;
  w.H = p; p += packed_h ? tri_row(n) : n * ldn;
  w.Aeq = p; p += me_cap * ldn;
  w.K = p; p += n * ldn;
  w.V = p; p += n * lde;
  w.S = p; p += me_cap * lde;
  w.kdi = p; p += n;
  w.sdi = p; p += me_cap;
  w.g = p; p += n; w.x = p; p += n; w.rd = p; p += n; w.dx = p; p += n; w.t1 = p; p += n; w.t2 = p; p += n;
  w.beq = p; p += me_cap; w.y = p; p += me_cap; w.rp = p; p += me_cap; w.dy = p; p += me_cap; w.t3 = p; p += me_cap;
  w.f = p; p += mi_cap; w.s = p; p += mi_cap; w.z = p; p += mi_cap; w.rs = p; p += mi_cap;
  w.ds = p; p += mi_cap; w.dz = p; p += mi_cap; w.rc = p; p += mi_cap; w.sgn = p; p += mi_cap; w.wt = p; p += mi_cap;
  int* ip = reinterpret_cast<int*>(p);
  w.in_row = ip; ip += mi_cap; w.in_c0 = ip; ip += mi_cap; w.in_c1 = ip; ip += mi_cap; w.in_pair = ip; ip += mi_cap; w.ord = ip; ip += mi_cap; w.eq_row = ip;
}

// In-place Cholesky M = L L' (lower triangle) followed by Li = L^-1, stored transposed in the strict upper triangle
// (Li[i][k] at M[k*ld + i], i > k) with diag(Li) = invdiag. Returns false when a pivot is not positive.
__device__ inline bool warp_chol_inv(double* M, int n, int ld, double* invdiag, int lane, double piv_floor = 0.0) {
  bool ok = true;
  for (int j = 0; j < n; ++j) {
    for (int i = j + lane; i < n; i += 32) {
      const double* ri = M + i * ld;
      const double* rj = M + j * ld;
      double a0 = ri[j], a1 = 0.0, a2 = 0.0, a3 = 0.0;
      int k = 0;
      for (; k + 3 < j; k += 4) {
        a0 -= ri[k] * rj[k]; a1 -= ri[k + 1] * rj[k + 1]; a2 -= ri[k + 2] * rj[k + 2]; a3 -= ri[k + 3] * rj[k + 3];
      }
      for (; k < j; ++k) a0 -= ri[k] * rj[k];
      M[i * ld + j] = (a0 + a1) + (a2 + a3);
    }
    __syncwarp();
    double d = M[j * ld + j];
    if (!(d > piv_floor)) {
      // piv_floor > 0: regularised factorisation (the interior-point residuals are exact, so a floored pivot only perturbs the
      // search direction); piv_floor == 0: strict, report failure
      if (piv_floor > 0.0 && d == d) d = piv_floor; else { ok = false; d = 1.0; }
    }
    const double r = 1.0 / sqrt(d);
    __syncwarp();
    for (int i = j + lane; i < n; i += 32) M[i * ld + j] *= r;
    if (lane == 0) invdiag[j] = r;
    __syncwarp();
  }
  // Li by forward substitution on the identity, lane c owns column c (rows are swept uniformly so L reads broadcast)
  for (int c0 = 0; c0 < n; c0 += 32) {
    const int c = c0 + lane;
    const bool act = c < n;
    for (int i = c0 + 1; i < n; ++i) {
      if (act && i > c) {
        const double* Li_row = M + i * ld;   // L[i][k], k < i  (lower)
        double* col = M + c * ld;            // Li[k][c] at M[c*ld + k], k > c (upper)
        double a0 = Li_row[c] * invdiag[c], a1 = 0.0;
        int k = c + 1;
        for (; k + 1 < i; k += 2) { a0 += Li_row[k] * col[k]; a1 += Li_row[k + 1] * col[k + 1]; }
        if (k < i) a0 += Li_row[k] * col[k];
        col[i] = -(a0 + a1) * invdiag[i];
      }
    }
  }
  __syncwarp();
  return ok;
}

// Row-in-registers form of warp_chol_inv for n <= WMAX <= 32 and a compile-time leading dimension. The shared-memory version was the
// largest instruction cost of the fused WBC kernel: two shared loads per multiply-add plus the
// index arithmetic of a triangular loop nest. Here lane i keeps row i of the trailing matrix in registers as a SLIDING window: a[0] is
// always the pivot column, and the rank-1 update writes a[k] from a[k+1], so the window advances without a move and the loop over the
// pivots stays ROLLED (register arrays only ever see compile-time indices). The pivot column goes through shared memory once (it is
// L, which the inverse needs anyway) and comes back as warp-uniform loads at immediate offsets: one LDS + one DFMA per term.
// The window narrows in stages of seven columns (28 -> 21 -> 14 -> 7), so the code is four short loops rather than one unrolled
// triangle -- a fully unrolled variant (~2.6k straight-line instructions per call) was faster for one in-phase wave of warps and 25-40 %
// SLOWER once several waves ran out of phase and every warp streamed that code through the instruction cache on its own.
// The inverse uses the same window on the residual of L y = e_c (lane c owns column c of Li).
// A stage reads up to 6 + (W - rem) rows past row n-1 of M; those values only ever reach window slots of columns >= n, which are never
// pivots, and the bytes lie inside the warp's workspace (K is followed by V, S by the vectors).
template <int LD, int W, int WMAX>
__device__ __forceinline__ void chol_window_factor(double (&a)[WMAX], double* M, int& j, int jend, int n, double* invdiag, int lane,
                                                   double piv_floor, bool& ok) {
  for (; j < jend; ++j) {
    double d = __shfl_sync(HB_FULL_MASK, a[0], j);
    if (!(d > piv_floor)) { if (piv_floor > 0.0 && d == d) d = piv_floor; else { ok = false; d = 1.0; } }
    const double r = rsqrt(d);
    const double l = a[0] * r;                       // L[i][j] on lane i > j
    if (lane < n) M[lane * LD + j] = l;              // rows above the diagonal hold scratch; the inverse overwrites them
    if (lane == j) invdiag[j] = r;
    __syncwarp();
    const double* col = M + (j + 1) * LD + j;        // L[j+1+k][j]
#pragma unroll
    for (int k = 0; k < W - 1; ++k) a[k] = fma(-l, col[k * LD], a[k + 1]);
  }
}

template <int LD, int W, int WMAX>
__device__ __forceinline__ void chol_window_inverse(double (&res)[WMAX], double* M, int& j, int jend, const double* invdiag, int lane) {
  for (; j < jend; ++j) {
    const double y = res[0] * invdiag[j];            // Li[j][lane]; zero while j < lane
    if (lane < j) M[lane * LD + j] = y;
    const double* col = M + (j + 1) * LD + j;
#pragma unroll
    for (int k = 0; k < W - 1; ++k) res[k] = fma(-col[k * LD], y, res[k + 1]);
  }
}

template <int LD, int WMAX>
__device__ __noinline__ bool warp_chol_inv_window(double* M, int n, double* invdiag, int lane, double piv_floor) {
  static_assert(WMAX <= 32 && WMAX % 7 == 0, "one lane per row, stages of seven columns");
  bool ok = true;
  double a[WMAX];
#pragma unroll
  for (int c = 0; c < WMAX; ++c) a[c] = (lane < n && c <= lane) ? M[lane * LD + c] : 0.0;
  __syncwarp();
  int j = 0;
  if constexpr (WMAX >= 28) chol_window_factor<LD, 28, WMAX>(a, M, j, n - 21, n, invdiag, lane, piv_floor, ok);
  if constexpr (WMAX >= 21) chol_window_factor<LD, 21, WMAX>(a, M, j, n - 14, n, invdiag, lane, piv_floor, ok);
  if constexpr (WMAX >= 14) chol_window_factor<LD, 14, WMAX>(a, M, j, n - 7, n, invdiag, lane, piv_floor, ok);
  chol_window_factor<LD, 7, WMAX>(a, M, j, n, n, invdiag, lane, piv_floor, ok);
  __syncwarp();
#pragma unroll
  for (int c = 0; c < WMAX; ++c) a[c] = (c == lane) ? 1.0 : 0.0;
  j = 0;
  if constexpr (WMAX >= 28) chol_window_inverse<LD, 28, WMAX>(a, M, j, n - 21, invdiag, lane);
  if constexpr (WMAX >= 21) chol_window_inverse<LD, 21, WMAX>(a, M, j, n - 14, invdiag, lane);
  if constexpr (WMAX >= 14) chol_window_inverse<LD, 14, WMAX>(a, M, j, n - 7, invdiag, lane);
  chol_window_inverse<LD, 7, WMAX>(a, M, j, n, invdiag, lane);
  __syncwarp();
  return ok;
}

// dispatch on the layout: the window form for the fused WBC problem (16 + 3 n_stance <= 28 variables at ld 29, <= 6 equalities at ld 7),
// the shared-memory form for everything else
__device__ inline bool warp_chol_inv_any(double* M, int n, int ld, double* invdiag, int lane, double piv_floor) {
  if (ld == 29 && n <= 28) return warp_chol_inv_window<29, 28>(M, n, invdiag, lane, piv_floor);
  if (ld == 7 && n <= 7) return warp_chol_inv_window<7, 7>(M, n, invdiag, lane, piv_floor);
  return warp_chol_inv(M, n, ld, invdiag, lane, piv_floor);
}

// y = Li v  (lower-triangular inverse stored as described above); lanes over rows
__device__ inline void warp_li_mv(const double* M, int n, int ld, const double* invdiag, const double* v, double* y, int lane) {
  for (int i = lane; i < n; i += 32) {
    double a0 = invdiag[i] * v[i], a1 = 0.0;
    int k = 0;
    for (; k + 1 < i; k += 2) { a0 += M[k * ld + i] * v[k]; a1 += M[(k + 1) * ld + i] * v[k + 1]; }
    if (k < i) a0 += M[k * ld + i] * v[k];
    y[i] = a0 + a1;
  }
  __syncwarp();
}
// y = Li' v
__device__ inline void warp_lit_mv(const double* M, int n, int ld, const double* invdiag, const double* v, double* y, int lane) {
  for (int i = lane; i < n; i += 32) {
    const double* row = M + i * ld;
    double a0 = invdiag[i] * v[i], a1 = 0.0;
    int k = i + 1;
    for (; k + 1 < n; k += 2) { a0 += row[k] * v[k]; a1 += row[k + 1] * v[k + 1]; }
    if (k < n) a0 += row[k] * v[k];
    y[i] = a0 + a1;
  }
  __syncwarp();
}

struct QpResult { int status; int iters; };

// The Mehrotra predictor-corrector iteration of qp_solve_warp and of level 0 of the hierarchical WBC (hwbc_level0_warp), which supply only
// their Newton systems. It owns the slacks s and multipliers z of the mi one-sided inequality entries (row_j x + s_j = bound(j), s_j >= 0),
// the start point, the tests and status codes (0 converged, 1 iteration limit, 2 Newton matrix not factored, 3 non-finite or diverging),
// the predictor, the centring, the corrector and the step. The problem supplies bound(j); residuals(rdn, rpn): its residuals, rs among
// them, raising the lane-partial max norms rdn (dual) and rpn (primal) and returning the lane partial of sum s z; factor(): build and
// factor its Newton matrix, false on failure; newton(): the solve for the complementarity target rc, its own direction and ds, dz;
// step(alpha): its own variables += alpha * direction. gs, bs, fsum are the lane partials of max(1, 1 + |gradient|), max(1, 1 + |right-hand
// side or bound|) and sum |bound|: each caller sums over its own lanes in its own order, and only the warp reductions happen here.
template <class Bound, class Residuals, class Factor, class Newton, class Step>
__device__ __forceinline__ QpResult qp_mehrotra_warp(int mi, int max_iter, double gs, double bs, double fsum, double* s, double* z, double* ds,
                                                     double* dz, double* rc, Bound bound, Residuals residuals, Factor factor, Newton newton,
                                                     Step step) {
  const int lane = lane_id();
  // starting point: slacks s = max(theta, bound), multipliers z = theta / s (uniform complementarity s z = theta) with theta the mean
  // magnitude of the bounds -- about 30 % fewer iterations than s = max(1, bound), z = 1 on the WBC problems
  fsum = warp_sum(fsum);
  const double theta = fmax(1.0, mi > 0 ? fsum / mi : 1.0);
  for (int j = lane; j < mi; j += 32) { const double sj = fmax(theta, bound(j)); s[j] = sj; z[j] = theta / sj; }
  gs = warp_max(gs); bs = warp_max(bs);
  __syncwarp();
  auto max_step = [&]() {
    double a = 1.0;
    for (int j = lane; j < mi; j += 32) {
      if (ds[j] < 0.0) a = fmin(a, -s[j] / ds[j]);
      if (dz[j] < 0.0) a = fmin(a, -z[j] / dz[j]);
    }
    return warp_min(a);
  };
  QpResult res{1, 0};
  int it = 0;
  for (; it < max_iter; ++it) {
    double rdn = 0.0, rpn = 0.0;
    const double sz = residuals(rdn, rpn);
    rdn = warp_max(rdn); rpn = warp_max(rpn);
    const double mu = mi > 0 ? warp_sum(sz) / mi : 0.0;
    if (!(rdn == rdn) || !(rpn == rpn) || !(mu == mu) || rdn > 1e300 || rpn > 1e300) { res.status = 3; break; }
    if (rdn < 1e-10 * gs && rpn < 1e-10 * bs && mu < 1e-12) { res.status = 0; break; }
    if (!factor()) { res.status = 2; break; }
    // predictor (affine step), centring sigma = (mu_aff / mu)^3, corrector
    for (int j = lane; j < mi; j += 32) rc[j] = s[j] * z[j];
    __syncwarp();
    newton();
    if (mi > 0) {
      const double a_aff = max_step();
      double ma = 0.0;
      for (int j = lane; j < mi; j += 32) ma += (s[j] + a_aff * ds[j]) * (z[j] + a_aff * dz[j]);
      ma = warp_sum(ma) / mi;
      const double r = ma / mu;
      const double sigma = r * r * r;
      for (int j = lane; j < mi; j += 32) rc[j] = s[j] * z[j] + ds[j] * dz[j] - sigma * mu;
      __syncwarp();
      newton();
    }
    const double alpha = fmin(1.0, 0.995 * max_step());
    step(alpha);
    for (int j = lane; j < mi; j += 32) { s[j] += alpha * ds[j]; z[j] += alpha * dz[j]; }
    __syncwarp();
  }
  res.iters = it;
  return res;
}

// A, lbA, ubA, H, g may live in global or shared memory (generic pointers). x_out: n doubles (generic).
// PACKED_H: the caller assembled H in w.H as its packed lower triangle (tri_row) and passes H == nullptr; H must be exactly symmetric.
// The products read the same values in the same order as with the full matrix, so the iterates are bit-identical.
template <bool PACKED_H = false>
__device__ inline QpResult qp_solve_warp(int n, int m, const double* __restrict__ H, const double* __restrict__ g,
                                         const double* __restrict__ A, const double* __restrict__ lbA,
                                         const double* __restrict__ ubA, double rho, int max_iter, double* x_out,
                                         QpWorkspace& w) {
  const int lane = lane_id();
  const int ldn = w.ldn, ldv = w.ldv, lds = w.lds;
  // ---------------- classify rows
  int me = 0, mi = 0;
  bool infeasible = false;
  for (int r0 = 0; r0 < m; r0 += 32) {
    const int r = r0 + lane;
    int c0 = n, c1 = 0;
    double lo = 0.0, hi = 0.0;
    if (r < m) {
      const double* a = A + (size_t)r * n;
      for (int c = 0; c < n; ++c) if (a[c] != 0.0) { if (c < c0) c0 = c; c1 = c + 1; }
      lo = lbA[r]; hi = ubA[r];
    }
    const bool valid = r < m;
    const bool zero_row = valid && c1 == 0;
    const bool has_lo = valid && lo > -1e19, has_hi = valid && hi < 1e19;
    if (zero_row && ((has_lo && lo > 1e-12) || (has_hi && hi < -1e-12))) infeasible = true;
    const bool is_eq = valid && !zero_row && has_lo && has_hi && lo == hi;
    const bool up = valid && !zero_row && !is_eq && has_hi;
    const bool dn = valid && !zero_row && !is_eq && has_lo;
    const unsigned beq = __ballot_sync(HB_FULL_MASK, is_eq);
    const unsigned bup = __ballot_sync(HB_FULL_MASK, up);
    const unsigned bdn = __ballot_sync(HB_FULL_MASK, dn);
    const unsigned below = (1u << lane) - 1u;
    if (is_eq) { const int e = me + __popc(beq & below); if (e < w.me_cap) { w.eq_row[e] = r; w.beq[e] = hi; } }
    const int mi2 = mi + __popc(bup);
    const int e_up = mi + __popc(bup & below), e_dn = mi2 + __popc(bdn & below);
    if (up && e_up < w.mi_cap) { w.in_row[e_up] = r; w.in_c0[e_up] = c0; w.in_c1[e_up] = c1; w.sgn[e_up] = 1.0; w.f[e_up] = hi; w.in_pair[e_up] = (dn && e_dn < w.mi_cap) ? e_dn : -1; }
    if (dn && e_dn < w.mi_cap) { w.in_row[e_dn] = r; w.in_c0[e_dn] = c0; w.in_c1[e_dn] = c1; w.sgn[e_dn] = -1.0; w.f[e_dn] = -lo; w.in_pair[e_dn] = up ? -2 : -1; }
    me += __popc(beq);
    mi = mi2 + __popc(bdn);
  }
  infeasible = __any_sync(HB_FULL_MASK, infeasible);
  QpResult res{1, 0};
  // status 2: an all-zero row whose bounds exclude 0; status 4: more rows than the workspace holds (the problem itself may be feasible)
  if (infeasible) res.status = 2;
  else if (me > w.me_cap || mi > w.mi_cap || n > QP_MAX_N) res.status = 4;
  if (res.status != 1) {
    for (int i = lane; i < n; i += 32) x_out[i] = 0.0;
    return res;
  }
  __syncwarp();
  // processing order of the inequality entries: "wide" rows (span > 8 columns, e.g. the dense torque rows of the WBC) first, then
  // the narrow ones (friction pyramid rows: 3 columns); the second entry of a two-sided row is merged into the first
  int nwide = 0, nact = 0;
  for (int pass = 0; pass < 2; ++pass) {
    for (int j0 = 0; j0 < mi; j0 += 32) {
      const int j = j0 + lane;
      const bool sel = j < mi && w.in_pair[j] != -2 && ((w.in_c1[j] - w.in_c0[j] > 8) == (pass == 0));
      const unsigned msk = __ballot_sync(HB_FULL_MASK, sel);
      if (sel) w.ord[nact + __popc(msk & ((1u << lane) - 1u))] = j;
      nact += __popc(msk);
    }
    if (pass == 0) nwide = nact;
  }
  __syncwarp();
  // n <= 32: lane = column. Which narrow entries touch this lane's column is fixed for the whole solve: one bit per narrow entry (in
  // processing order), so the loops below visit the 5 friction rows of a force column instead of testing the span of all 20.
  const bool colmask = n <= 32 && nact - nwide <= 32;
  unsigned nmask = 0u;
  if (colmask && lane < n)
    for (int q = nwide; q < nact; ++q) { const int j = w.ord[q]; if (lane >= w.in_c0[j] && lane < w.in_c1[j]) nmask |= 1u << (q - nwide); }
  // a = base + sum_j wt[j] A[row_j][i] over the ordered entries (A' times the merged coefficient vector), lane i
  auto at_mul = [&](int i, double a) {
    for (int q = 0; q < nwide; ++q) { const int j = w.ord[q]; a = fma(w.wt[j], A[(size_t)w.in_row[j] * n + i], a); }
    if (colmask) {          // i == lane; same entries in the same order as the span test below
      for (unsigned mk = nmask; mk; mk &= mk - 1u) { const int j = w.ord[nwide + __ffs(mk) - 1]; a = fma(w.wt[j], A[(size_t)w.in_row[j] * n + i], a); }
      return a;
    }
    for (int q = nwide; q < nact; ++q) {
      const int j = w.ord[q];
      if (i >= w.in_c0[j] && i < w.in_c1[j]) a = fma(w.wt[j], A[(size_t)w.in_row[j] * n + i], a);
    }
    return a;
  };
  // ---------------- stage H, Aeq, g; initial point
  // H == nullptr: the caller assembled the Hessian directly in w.H (leading dimension ldn)
  if (H != nullptr) for (int idx = lane; idx < n * n; idx += 32) { const int i = idx / n, c = idx - i * n; w.H[i * ldn + c] = H[idx]; }
  for (int e = 0; e < me; ++e) {
    const double* a = A + (size_t)w.eq_row[e] * n;
    for (int c = lane; c < n; c += 32) w.Aeq[e * ldn + c] = a[c];
  }
  double gs = 1.0, bs = 1.0;
  for (int i = lane; i < n; i += 32) { const double gi = g[i]; w.g[i] = gi; w.x[i] = 0.0; gs = fmax(gs, 1.0 + fabs(gi)); }
  for (int e = lane; e < me; e += 32) { w.y[e] = 0.0; bs = fmax(bs, 1.0 + fabs(w.beq[e])); }
  // starting point: x = 0, y = 0; the slacks and multipliers are qp_mehrotra_warp's
  double fsum = 0.0;
  for (int j = lane; j < mi; j += 32) { fsum += fabs(w.f[j]); bs = fmax(bs, 1.0 + fabs(w.f[j])); }
  // ---------------- the Newton system qp_mehrotra_warp iterates on: residuals, K and S factorised, the solve, the step of x and y
  auto residuals = [&](double& rdn, double& rpn) {
    for (int j = lane; j < mi; j += 32) {
      const int pr = w.in_pair[j];
      double cj = w.sgn[j] * w.z[j];
      if (pr >= 0) cj += w.sgn[pr] * w.z[pr];
      w.wt[j] = cj;
    }
    __syncwarp();
    for (int i = lane; i < n; i += 32) {
      double a = w.g[i] + rho * w.x[i];
      if (PACKED_H) {
        const double* hr = w.H + tri_row(i);
        for (int c = 0; c <= i; ++c) a += hr[c] * w.x[c];
        for (int c = i + 1; c < n; ++c) a += w.H[tri_row(c) + i] * w.x[c];
      } else {
        const double* hr = w.H + i * ldn;
        for (int c = 0; c < n; ++c) a += hr[c] * w.x[c];
      }
      for (int e = 0; e < me; ++e) a += w.Aeq[e * ldn + i] * w.y[e];
      w.rd[i] = at_mul(i, a);
    }
    for (int e = lane; e < me; e += 32) {
      double a = -w.beq[e];
      for (int c = 0; c < n; ++c) a += w.Aeq[e * ldn + c] * w.x[c];
      w.rp[e] = a;
    }
    double sz = 0.0;
    for (int j = lane; j < mi; j += 32) {
      const double* a = A + (size_t)w.in_row[j] * n;
      double d = 0.0;
      for (int c = w.in_c0[j]; c < w.in_c1[j]; ++c) d += a[c] * w.x[c];
      w.rs[j] = w.sgn[j] * d + w.s[j] - w.f[j];
      sz += w.s[j] * w.z[j];
    }
    __syncwarp();
    for (int i = lane; i < n; i += 32) rdn = fmax(rdn, fabs(w.rd[i]));
    for (int e = lane; e < me; e += 32) rpn = fmax(rpn, fabs(w.rp[e]));
    for (int j = lane; j < mi; j += 32) rpn = fmax(rpn, fabs(w.rs[j]));
    return sz;
  };
  auto factor = [&]() {
    // ---------------- K = H + rho I + D' W D
    // (only the lower triangle of K is read before the factorisation overwrites the upper one with L^-1)
    if (PACKED_H) {
      for (int idx = lane; idx < n * ldn; idx += 32) { const int i = idx / ldn, c = idx - i * ldn; if (c <= i) w.K[idx] = w.H[tri_row(i) + c] + ((i == c) ? rho : 0.0); }
    } else {
      for (int idx = lane; idx < n * ldn; idx += 32) { const int i = idx / ldn, c = idx - i * ldn; w.K[idx] = w.H[idx] + ((i == c) ? rho : 0.0); }
    }
    __syncwarp();
    // lower triangle only; a two-sided row contributes once with the sum of its two weights
    for (int j = lane; j < mi; j += 32) {
      const int pr = w.in_pair[j];
      double wj = w.z[j] / w.s[j];
      if (pr >= 0) wj += w.z[pr] / w.s[pr];
      w.wt[j] = wj;
    }
    __syncwarp();
    // wide rows as a product: lane c owns column c of the lower triangle, K[i][c] += sum_j (wt_j a_j[c]) a_j[i]; the per-row
    // factors wt_j a_j[c] stay in registers and a_j[i] is a broadcast load
    {
      constexpr int WCH = 10;
      for (int cb = 0; cb < n; cb += 32) {
        const int c = cb + lane;
        const bool act = c < n;
        for (int q0 = 0; q0 < nwide; q0 += WCH) {
          double t[WCH]; int roff[WCH];
#pragma unroll
          for (int q = 0; q < WCH; ++q) {
            const bool on = q0 + q < nwide;
            const int j = on ? w.ord[q0 + q] : 0;
            roff[q] = on ? w.in_row[j] * n : 0;
            t[q] = (on && act) ? w.wt[j] * A[(size_t)roff[q] + c] : 0.0;
          }
          for (int i = cb; i < n; ++i) {
            double acc = 0.0;
#pragma unroll
            for (int q = 0; q < WCH; ++q) acc = fma(t[q], A[(size_t)roff[q] + i], acc);
            if (act && i >= c) w.K[i * ldn + c] += acc;
          }
        }
      }
    }
    __syncwarp();
    // narrow rows: rank-1 update inside the span. n <= 32: lane c owns column c of the lower triangle and walks only the entries that
    // touch it (no two lanes write the same element, no barrier between entries); otherwise entry by entry, lanes over the columns c <= i
    if (colmask) {
      for (unsigned mk = nmask; mk; mk &= mk - 1u) {
        const int j = w.ord[nwide + __ffs(mk) - 1];
        const int c1 = w.in_c1[j];
        const double wj = w.wt[j];
        const double* a = A + (size_t)w.in_row[j] * n;
        const double ac = a[lane];
        for (int i = lane; i < c1; ++i) w.K[i * ldn + lane] += (wj * a[i]) * ac;
      }
      __syncwarp();
    } else
    for (int q = nwide; q < nact; ++q) {
      const int j = w.ord[q];
      const int c0 = w.in_c0[j], c1 = w.in_c1[j];
      const double wj = w.wt[j];
      const double* a = A + (size_t)w.in_row[j] * n;
      for (int i = c0; i < c1; ++i) {
        const double ai = wj * a[i];
        for (int c = c0 + lane; c <= i; c += 32) w.K[i * ldn + c] += ai * a[c];
      }
      __syncwarp();
    }
    // directions that only the Tikhonov term rho controls have pivots ~1e-8 next to barrier weights ~1e10 late in the solve:
    // floor the pivots instead of failing
    bool ok = warp_chol_inv_any(w.K, n, ldn, w.kdi, lane, 1e-10);
    // ---------------- V = Li Aeq'  (n x me), lane per equality row
    if (me > 0) {
      // entries (i, e) spread over all lanes (a lane per equality row would leave most of the warp idle: me is 6 for the WBC)
      for (int idx = lane; idx < n * me; idx += 32) {
        const int i = idx / me, e = idx - i * me;
        const double* ar = w.Aeq + e * ldn;
        double a0 = w.kdi[i] * ar[i], a1 = 0.0;
        int k = 0;
        for (; k + 1 < i; k += 2) { a0 += w.K[k * ldn + i] * ar[k]; a1 += w.K[(k + 1) * ldn + i] * ar[k + 1]; }
        if (k < i) a0 += w.K[k * ldn + i] * ar[k];
        w.V[i * ldv + e] = a0 + a1;
      }
      __syncwarp();
      // S = V'V (lower), then Cholesky + inverse
      for (int idx = lane; idx < me * me; idx += 32) {
        const int a = idx / me, b = idx - a * me;
        if (b <= a) {
          double s0 = 0.0, s1 = 0.0;
          int i = 0;
          for (; i + 1 < n; i += 2) { s0 += w.V[i * ldv + a] * w.V[i * ldv + b]; s1 += w.V[(i + 1) * ldv + a] * w.V[(i + 1) * ldv + b]; }
          if (i < n) s0 += w.V[i * ldv + a] * w.V[i * ldv + b];
          w.S[a * lds + b] = s0 + s1;
        }
      }
      __syncwarp();
      ok = warp_chol_inv_any(w.S, me, lds, w.sdi, lane, 1e-14) && ok;
    }
    return ok;
  };
  // Newton solve for the complementarity target in w.rc; results in dx, dy, ds, dz
  auto newton = [&]() {
    for (int j = lane; j < mi; j += 32) {
      const int pr = w.in_pair[j];
      double cj = w.sgn[j] * ((w.rc[j] - w.z[j] * w.rs[j]) / w.s[j]);
      if (pr >= 0) cj += w.sgn[pr] * ((w.rc[pr] - w.z[pr] * w.rs[pr]) / w.s[pr]);
      w.wt[j] = cj;
    }
    __syncwarp();
    for (int i = lane; i < n; i += 32) w.t2[i] = at_mul(i, -w.rd[i]);
    __syncwarp();
    warp_li_mv(w.K, n, ldn, w.kdi, w.t2, w.t1, lane);  // t1 = Li r1
    if (me > 0) {
      for (int e = lane; e < me; e += 32) {
        double a = w.rp[e];
        for (int i = 0; i < n; ++i) a += w.V[i * ldv + e] * w.t1[i];
        w.t3[e] = a;
      }
      __syncwarp();
      warp_li_mv(w.S, me, lds, w.sdi, w.t3, w.dy, lane);
      for (int e = lane; e < me; e += 32) w.t3[e] = w.dy[e];
      __syncwarp();
      warp_lit_mv(w.S, me, lds, w.sdi, w.t3, w.dy, lane);
      for (int i = lane; i < n; i += 32) {
        double a = w.t1[i];
        for (int e = 0; e < me; ++e) a -= w.V[i * ldv + e] * w.dy[e];
        w.t2[i] = a;
      }
      __syncwarp();
    } else {
      for (int i = lane; i < n; i += 32) w.t2[i] = w.t1[i];
      __syncwarp();
    }
    warp_lit_mv(w.K, n, ldn, w.kdi, w.t2, w.dx, lane);
    for (int j = lane; j < mi; j += 32) {
      const double* a = A + (size_t)w.in_row[j] * n;
      double d = 0.0;
      for (int c = w.in_c0[j]; c < w.in_c1[j]; ++c) d += a[c] * w.dx[c];
      const double dsj = -w.rs[j] - w.sgn[j] * d;
      w.ds[j] = dsj;
      w.dz[j] = -(w.rc[j] + w.z[j] * dsj) / w.s[j];
    }
    __syncwarp();
  };
  auto step = [&](double alpha) {
    for (int i = lane; i < n; i += 32) w.x[i] += alpha * w.dx[i];
    for (int e = lane; e < me; e += 32) w.y[e] += alpha * w.dy[e];
  };
  res = qp_mehrotra_warp(mi, max_iter, gs, bs, fsum, w.s, w.z, w.ds, w.dz, w.rc, [&](int j) { return w.f[j]; }, residuals, factor, newton, step);
  for (int i = lane; i < n; i += 32) x_out[i] = w.x[i];
  return res;
}

}  // namespace hb

namespace {  // the kernels: internal linkage, the library exports only the hb_* entry points
using namespace hb;
__global__ void qp_batch_kernel(int B, int n, int m, const double* H, const double* g, const double* A, const double* lbA, const double* ubA,
                                size_t strideH, size_t strideA, size_t strideB, const int32_t* m_per, double rho, int max_iter, double* x,
                                int32_t* status, int32_t* iters) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int inst = blockIdx.x * wpb + warp;
  if (inst >= B) return;
  double* base = reinterpret_cast<double*>(smem_raw) + (size_t)warp * qp_workspace_doubles(n);
  QpWorkspace w;
  qp_carve(base, n, w);
  const int mi = m_per ? m_per[inst] : m;
  QpResult r = qp_solve_warp(n, mi, H + inst * strideH, g + (size_t)inst * n, A + inst * strideA, lbA + inst * strideB, ubA + inst * strideB,
                             rho, max_iter, x + (size_t)inst * n, w);
  if (lane_id() == 0) { if (status) status[inst] = r.status; if (iters) iters[inst] = r.iters; }
}
}  // namespace
