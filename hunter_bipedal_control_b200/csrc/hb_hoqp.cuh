// Hierarchical QP (HoQP) on the device, one warp per instance: legged::HoQp (legged_wbc/src/HoQp.cpp:21-198) and the three-level cascade of
// legged::HierarchicalWbc::update (legged_wbc/src/HierarchicalWbc.cpp:18-31). SURVEY 8f row N4.
//
// Level k (task: A_k x = b_k in the least-squares sense, D_k x <= f_k softened by slacks v >= 0) is solved in the null space Z of all
// higher-priority equality tasks, x = x_prev + Z z:
//     min 1/2 ||A_k (x_prev + Z z) - b_k||^2 + 1/2 ||v||^2
//     s.t. -v <= 0,   D_prev (x_prev + Z z) <= f_prev + v_prev*  (stacked higher levels, their slack solutions frozen),   D_k (x_prev + Z z) - v <= f_k
// exactly the (H, c, D, f) of HoQp::buildHMatrix / buildCVector / buildDMatrix / buildFVector, handed to the batched interior point
// (qp_solve_warp replaces qpOASES as in the weighted WBC). Then Z <- Z kernel(A_k Z) (HoQp::buildZMatrix: Eigen FullPivLU::kernel; here a
// Gauss-Jordan elimination with complete pivoting -- any basis of the same null space gives the same x).
//
// hwbc_fused_kernel runs HierarchicalWbc::update in one launch without materialising an hb_hoqp_problem: the tasks are built in shared
// memory from the WBC terms and every level is solved at its real shape (hwbc_level0_warp for level 0, qp_solve_warp at <= 28 variables
// for levels 1 and 2; both are qp_mehrotra_warp with their own Newton systems). Both cascades take a level through the same steps: the task
// residual (hoqp_task_residual), the normal equations of its objective (hoqp_normal_eq), the update x += Z z (hoqp_update_x) and the
// null-space step (hoqp_null_space_step).
#pragma once
#include "hb_common.cuh"
#include "hb_qp.cuh"
#include "hb_wbc.cuh"
#include "../../include/hunter_b200.h"

namespace hb {

constexpr int HQ_N = HB_HOQP_N, HQ_MA = HB_HOQP_MAX_EQ, HQ_MD = HB_HOQP_MAX_IN, HQ_STK = HB_HOQP_MAX_STACKED;
constexpr int HQ_NQ = HQ_N + HQ_MD;                // variables of a lifted level problem (z, v)
constexpr int HQ_ROWS = 2 * HQ_MD + HQ_STK;         // rows of a lifted level problem
constexpr int HQ_LDZ = HQ_N + 1, HQ_LDA = HQ_N + 1;
static_assert(HQ_N <= 64, "hoqp_update_x: two entries of x per lane");
// global scratch per instance (doubles): the lifted inequality rows and their bounds, which qp_solve_warp reads as a dense row-major A
constexpr size_t HQ_SCRATCH = (size_t)HQ_ROWS * HQ_NQ + 2 * HQ_ROWS;

struct HoqpShared {
  double Z[HQ_N * HQ_LDZ];       // current null-space basis (n x nx)
  double AZ[HQ_MA * HQ_LDA];     // A_k Z (ma x nx), then its reduced row echelon form
  double Zn[HQ_N * HQ_LDZ];      // next basis while it is formed
  double x[HQ_N], r[HQ_MA];
  double c[HQ_NQ], z[HQ_NQ];     // gradient and solution of the lifted level problem
  double slk[HQ_STK];            // slack solutions of the levels so far, stacked in level order
  int pcol[HQ_MA], prow[HQ_MA], isp[HQ_N], freec[HQ_N];
};
__host__ __device__ constexpr size_t hoqp_smem_bytes() { return sizeof(HoqpShared) + qp_workspace_doubles(HQ_NQ, 1, HQ_ROWS) * sizeof(double); }
static_assert(hoqp_smem_bytes() <= 227 * 1024, "hoqp_kernel must fit the 227 KB opt-in shared memory of a block");

// Z <- Z kernel(A Z) (HoQp::buildZMatrix) for ma > 0, nx > 0: reduced row echelon form of AZ (ma x nx, leading dimension HQ_LDA, overwritten)
// with complete pivoting, the new basis formed in Zn and copied back to Z (n x nfree, leading dimension HQ_LDZ). Returns nfree.
__device__ inline int hoqp_null_space_step(double* Z, double* AZ, double* Zn, int* pcol, int* prow, int* isp, int* freec, int n, int ma, int nx) {
  const int lane = lane_id();
  double amax = 0.0;
  for (int idx = lane; idx < ma * nx; idx += 32) amax = fmax(amax, fabs(AZ[(idx / nx) * HQ_LDA + idx % nx]));
  amax = warp_max(amax);
  const double tol = 1e-9 * fmax(amax, 1e-300);
  for (int j = lane; j < nx; j += 32) isp[j] = 0;
  __syncwarp();
  int rank = 0;
  unsigned long long rowused = 0ull;
  for (int step = 0; step < min(ma, nx); ++step) {
    double best = -1.0; int bi = 0, bj = 0;
    for (int idx = lane; idx < ma * nx; idx += 32) {
      const int i = idx / nx, j = idx - i * nx;
      if (((rowused >> i) & 1ull) || isp[j]) continue;
      const double a = fabs(AZ[i * HQ_LDA + j]);
      if (a > best) { best = a; bi = i; bj = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ob = __shfl_xor_sync(HB_FULL_MASK, best, o);
      const int oi = __shfl_xor_sync(HB_FULL_MASK, bi, o), oj = __shfl_xor_sync(HB_FULL_MASK, bj, o);
      if (ob > best || (ob == best && (oi < bi || (oi == bi && oj < bj)))) { best = ob; bi = oi; bj = oj; }
    }
    if (!(best > tol)) break;
    const double inv = 1.0 / AZ[bi * HQ_LDA + bj];
    __syncwarp();
    for (int j = lane; j < nx; j += 32) AZ[bi * HQ_LDA + j] *= inv;
    __syncwarp();
    for (int idx = lane; idx < ma * nx; idx += 32) {
      const int i = idx / nx, j = idx - i * nx;
      if (i == bi || j == bj) continue;
      AZ[i * HQ_LDA + j] -= AZ[i * HQ_LDA + bj] * AZ[bi * HQ_LDA + j];
    }
    __syncwarp();
    for (int i = lane; i < ma; i += 32) if (i != bi) AZ[i * HQ_LDA + bj] = 0.0;
    if (lane == 0) { pcol[rank] = bj; prow[rank] = bi; isp[bj] = 1; }
    rowused |= 1ull << bi;
    ++rank;
    __syncwarp();
  }
  int nfree = 0;
  for (int j = 0; j < nx; ++j) if (!isp[j]) { if (lane == 0) freec[nfree] = j; ++nfree; }
  __syncwarp();
  // column c of the new basis: Z[:, f] - sum_i Z[:, pcol_i] R[prow_i][f]
  for (int idx = lane; idx < n * nfree; idx += 32) {
    const int k = idx / nfree, c = idx - k * nfree, fcol = freec[c];
    double s = Z[k * HQ_LDZ + fcol];
    for (int i = 0; i < rank; ++i) s = fma(-Z[k * HQ_LDZ + pcol[i]], AZ[prow[i] * HQ_LDA + fcol], s);
    Zn[k * HQ_LDZ + c] = s;
  }
  __syncwarp();
  for (int idx = lane; idx < n * nfree; idx += 32) { const int k = idx / nfree, c = idx - k * nfree; Z[k * HQ_LDZ + c] = Zn[k * HQ_LDZ + c]; }
  __syncwarp();
  return nfree;
}

// ---- the level steps both cascades share (Z, AZ at leading dimensions HQ_LDZ, HQ_LDA)

// task residual of a level: AZ = A Z (ma x nx), r = A x - b, for task rows A (ma x n, leading dimension lda)
__device__ inline void hoqp_task_residual(const double* A, int lda, const double* b, const double* Z, const double* x, int n, int ma, int nx,
                                          double* AZ, double* r) {
  const int lane = lane_id();
  for (int idx = lane; idx < ma * nx; idx += 32) {
    const int i = idx / nx, j = idx - i * nx;
    double s = 0.0;
    for (int k = 0; k < n; ++k) s = fma(A[i * lda + k], Z[k * HQ_LDZ + j], s);
    AZ[i * HQ_LDA + j] = s;
  }
  for (int i = lane; i < ma; i += 32) { double s = -b[i]; for (int k = 0; k < n; ++k) s = fma(A[i * lda + k], x[k], s); r[i] = s; }
  __syncwarp();
}

// normal equations of a level's objective 1/2 ||AZ z + r||^2: H = (AZ)'AZ + 1e-12 I (nx x nx; PACKED: its lower triangle at tri_row,
// otherwise at leading dimension ldh) and c = (AZ)'r
template <bool PACKED = false>
__device__ inline void hoqp_normal_eq(const double* AZ, const double* r, int ma, int nx, double* H, int ldh, double* c) {
  const int lane = lane_id();
  for (int idx = lane; idx < nx * nx; idx += 32) {
    const int i = idx / nx, j = idx - i * nx;
    if (PACKED && j > i) continue;
    double s = 0.0;
    for (int k = 0; k < ma; ++k) s = fma(AZ[k * HQ_LDA + i], AZ[k * HQ_LDA + j], s);
    if (i == j) s += 1e-12;
    H[PACKED ? tri_row(i) + j : i * ldh + j] = s;
  }
  for (int i = lane; i < nx; i += 32) { double s = 0.0; for (int k = 0; k < ma; ++k) s = fma(AZ[k * HQ_LDA + i], r[k], s); c[i] = s; }
}

// x <- x + Z z (x of n entries, z of nx)
__device__ inline void hoqp_update_x(double* x, const double* Z, const double* z, int n, int nx) {
  const int lane = lane_id();
  double xn = 0.0, xn2 = 0.0;
  if (lane < n) { xn = x[lane]; for (int j = 0; j < nx; ++j) xn = fma(Z[lane * HQ_LDZ + j], z[j], xn); }
  if (lane + 32 < n) { xn2 = x[lane + 32]; for (int j = 0; j < nx; ++j) xn2 = fma(Z[(lane + 32) * HQ_LDZ + j], z[j], xn2); }
  __syncwarp();
  if (lane < n) x[lane] = xn;
  if (lane + 32 < n) x[lane + 32] = xn2;
  __syncwarp();
}

// Solve one hierarchy. Returns 0, or the first failing level's QP status * 10 + level.
__device__ inline int hoqp_solve_warp(const hb_hoqp_problem& pb, HoqpShared& sh, QpWorkspace& w, double* scratch, int max_iter, double* x_out,
                                      double* slack_out) {
  const int lane = lane_id();
  const int n = min(max(pb.n, 1), HQ_N), L = min(max(pb.levels, 0), HB_HOQP_MAX_LEVELS);
  auto md_of = [&](int l) { return min(max(pb.md[l], 0), HQ_MD); };
  // row s of the stacked inequalities (Task::operator+, Task.h:46-58: the higher levels' rows in level order) and its bound f
  auto stacked = [&](int s, double& f) { int l = 0; while (s >= md_of(l)) s -= md_of(l++); f = pb.f[l][s]; return pb.d[l][s]; };
  double* Dq = scratch; double* lbq = Dq + (size_t)HQ_ROWS * HQ_NQ; double* ubq = lbq + HQ_ROWS;
  for (int idx = lane; idx < n * HQ_LDZ; idx += 32) { const int i = idx / HQ_LDZ, j = idx - i * HQ_LDZ; sh.Z[idx] = (i == j) ? 1.0 : 0.0; }
  for (int i = lane; i < n; i += 32) sh.x[i] = 0.0;
  __syncwarp();
  int nx = n, nstk = 0, status = 0;
  for (int lvl = 0; lvl < L; ++lvl) {
    const int ma = min(max(pb.ma[lvl], 0), HQ_MA), md = md_of(lvl);
    const double* D = &pb.d[lvl][0][0]; const double* fvec = pb.f[lvl];
    if (nstk + md > HQ_STK) { status = 20 + lvl; break; }
    double* slk = sh.slk + nstk;                   // slack solution of this level goes to the end of the stack
    if (nx > 0) {
      hoqp_task_residual(&pb.a[lvl][0][0], HQ_N, pb.b[lvl], sh.Z, sh.x, n, ma, nx, sh.AZ, sh.r);
      const int nq = nx + md, nr = 2 * md + nstk;
      // lifted Hessian and gradient (HoQp::buildHMatrix / buildCVector), assembled in the QP workspace: the identity on the slacks
      hoqp_normal_eq(sh.AZ, sh.r, ma, nx, w.H, w.ldn, sh.c);
      for (int idx = lane; idx < nq * nq; idx += 32) { const int i = idx / nq, j = idx - i * nq; if (i >= nx || j >= nx) w.H[i * w.ldn + j] = (i == j) ? 1.0 : 0.0; }
      for (int i = nx + lane; i < nq; i += 32) sh.c[i] = 0.0;
      // lifted inequality rows (HoQp::buildDMatrix / buildFVector)
      for (int idx = lane; idx < nr * nq; idx += 32) {
        const int i = idx / nq, j = idx - i * nq;
        double s = 0.0;
        if (i < md) s = (j == nx + i) ? -1.0 : 0.0;
        else if (i < md + nstk) { if (j < nx) { double f; const double* dr = stacked(i - md, f); for (int k = 0; k < n; ++k) s = fma(dr[k], sh.Z[k * HQ_LDZ + j], s); } }
        else { const int ii = i - md - nstk; if (j < nx) { for (int k = 0; k < n; ++k) s = fma(D[ii * HQ_N + k], sh.Z[k * HQ_LDZ + j], s); } else s = (j == nx + ii) ? -1.0 : 0.0; }
        Dq[idx] = s;
      }
      for (int i = lane; i < nr; i += 32) {
        double u = 0.0;
        if (i >= md && i < md + nstk) { double f; const double* dr = stacked(i - md, f); double s = 0.0; for (int k = 0; k < n; ++k) s = fma(dr[k], sh.x[k], s); u = f - s + sh.slk[i - md]; }
        else if (i >= md + nstk) { const int ii = i - md - nstk; double s = 0.0; for (int k = 0; k < n; ++k) s = fma(D[ii * HQ_N + k], sh.x[k], s); u = fvec[ii] - s; }
        lbq[i] = -1e20; ubq[i] = u;
      }
      __syncwarp();
      const QpResult qr = qp_solve_warp(nq, nr, nullptr, sh.c, Dq, lbq, ubq, 1e-10, max_iter, sh.z, w);
      __syncwarp();
      if (qr.status != 0 && status == 0) status = 10 * qr.status + lvl;
      hoqp_update_x(sh.x, sh.Z, sh.z, n, nx);
      for (int i = lane; i < md; i += 32) slk[i] = sh.z[nx + i];
    } else {
      // nothing left to decide: the slacks absorb whatever the higher priorities leave
      for (int i = lane; i < md; i += 32) { double s = -fvec[i]; for (int k = 0; k < n; ++k) s = fma(D[i * HQ_N + k], sh.x[k], s); slk[i] = s > 0.0 ? s : 0.0; }
    }
    nstk += md;                                    // this level's inequalities join the stack
    __syncwarp();
    // Z <- Z kernel(A Z): reduced row echelon form of AZ with complete pivoting
    if (ma > 0 && nx > 0) nx = hoqp_null_space_step(sh.Z, sh.AZ, sh.Zn, sh.pcol, sh.prow, sh.isp, sh.freec, n, ma, nx);
  }
  for (int i = lane; i < n; i += 32) x_out[i] = sh.x[i];
  if (slack_out) for (int i = lane; i < HQ_STK; i += 32) slack_out[i] = i < nstk ? sh.slk[i] : 0.0;
  return status;
}

// ---- the fused hierarchical WBC (hwbc_fused_kernel): one warp per instance, everything in shared memory
// hwbc_fused_kernel calls level 0 and the null-space steps out of line: inlined into the kernel next to the WBC assembly, whose peak sits
// at the 255-register ceiling, they made ptxas spill; hoqp_kernel keeps hoqp_null_space_step inline.
__device__ __noinline__ int hwbc_null_space_step(double* Z, double* AZ, double* Zn, int* pcol, int* prow, int* isp, int* freec, int n, int ma, int nx) {
  return hoqp_null_space_step(Z, AZ, Zn, pcol, prow, isp, freec, n, ma, nx);
}
constexpr int HW_NX = 28;   // free variables a level 1 / 2 QP holds (leading dimension 29: the register-window factorisation)
constexpr int HW_LD0 = NWBC + 1;
struct HwbcShared {
  double Z[HQ_N * HQ_LDZ];        // null-space basis of the levels solved so far
  double AZ[WBC_MA0 * HQ_LDA];    // the level's task rows times Z, then their reduced row echelon form
  double x[HQ_N], r[WBC_MA0];     // solution so far; task residual A x - b
  double dco[HQ_MD * 3], f0[HQ_MD], v0[HQ_MD];   // task0 inequality rows (nonzeros from column dc0), bounds, level-0 slack solution
  double At[18 * 16], bt[18];     // the unit-weight motion rows of WbcShared that tasks 1 and 2 are built from
  int pcol[WBC_MA0], prow[WBC_MA0], isp[HQ_N], freec[HQ_N], dc0[HQ_MD], dlen[HQ_MD];
};
// scratch shared by the phases: the assembly (WbcShared), level 0 (hwbc_level0_warp), a level-1/2 task and its QP, the next basis Zn
__host__ __device__ constexpr size_t hw_level0_doubles() { return (size_t)tri_row(NWBC) + NWBC * HW_LD0 + 6 * NWBC + 6 * HQ_MD + 7 * 2 * HQ_MD; }
__host__ __device__ constexpr size_t hw_level12_doubles() { return qp_workspace_doubles(HW_NX, 1, HQ_MD) + (size_t)HQ_MD * HW_NX + 2 * HQ_MD + 2 * HW_NX; }
__host__ __device__ constexpr size_t hw_max(size_t a, size_t b) { return a > b ? a : b; }
__host__ __device__ constexpr size_t hwbc_scratch_doubles() {
  return hw_max(hw_max(hw_level0_doubles(), hw_level12_doubles()),
                hw_max(hw_max(sizeof(WbcStaged) / sizeof(double), (size_t)HQ_N * HQ_LDZ), (size_t)WBC_MA0 * NWBC + WBC_MA0));
}
__host__ __device__ constexpr size_t hwbc_fused_bytes() { return sizeof(HwbcShared) + hwbc_scratch_doubles() * sizeof(double); }
// one warp per block: 4 blocks per SM put a 1024-instance batch in two waves on 132 SMs (the runtime reserves 1 KB per block)
static_assert(4 * (hwbc_fused_bytes() + 1024) <= 228 * 1024, "hwbc_fused_kernel must fit 4 blocks per SM");

// Level 0 of the cascade (Z = I, x_prev = 0) at its real shape. The lifted problem hoqp_solve_warp hands qp_solve_warp is, in x (38) and
// one slack v_j per inequality row D_j of task0,
//     min 1/2 x'G x + c'x + 1/2 v'v   s.t.  -v <= 0,  D x - v <= f,      G = A'A + 1e-12 I,  c = A'r  (r = -b)
// qp_mehrotra_warp solves it with this Newton system, which never forms the (38 + md)-square matrix: its slack block is diagonal,
// d = 1 + rho + w_b + w_d (w = z / s of the two rows that hold v_j), so the Newton step is the 38 x 38 Schur complement
// S = G + rho I + D' diag(w_d (1 + rho + w_b) / d) D, and D has at most 3 nonzeros per row. x -> sh.x, v -> sh.v0.
__device__ __noinline__ QpResult hwbc_level0_warp(HwbcShared& sh, int md, double rho, int max_iter, double* work) {
  const int lane = lane_id();
  constexpr int n = NWBC, ld = HW_LD0;
  const int mi = 2 * md;                    // entries: 0 .. md-1 the bounds -v <= 0, md .. 2md-1 the rows D x - v <= f
  double* G = work; double* K = G + tri_row(n); double* kdi = K + n * ld;
  double* c = kdi + n; double* rdx = c + n; double* dx = rdx + n; double* t1 = dx + n; double* t2 = t1 + n;
  double* v = t2 + n; double* dv = v + HQ_MD; double* rdv = dv + HQ_MD; double* dd = rdv + HQ_MD; double* wd = dd + HQ_MD; double* qv = wd + HQ_MD;
  double* s = qv + HQ_MD; double* z = s + 2 * HQ_MD; double* ds = z + 2 * HQ_MD; double* dz = ds + 2 * HQ_MD; double* rs = dz + 2 * HQ_MD;
  double* rc = rs + 2 * HQ_MD; double* cw = rc + 2 * HQ_MD;
  // row j of D times a vector
  auto drow = [&](int j, const double* y) { double a = 0.0; for (int k = 0; k < sh.dlen[j]; ++k) a = fma(sh.dco[3 * j + k], y[sh.dc0[j] + k], a); return a; };
  // sum_j q_j D_j[i] over the rows that touch column i
  auto dtmul = [&](int i, const double* q, double a) {
    for (int j = 0; j < md; ++j) { const int k = i - sh.dc0[j]; if (k >= 0 && k < sh.dlen[j]) a = fma(q[j], sh.dco[3 * j + k], a); }
    return a;
  };
  hoqp_normal_eq<true>(sh.AZ, sh.r, WBC_MA0, n, G, 0, c);
  // start point x = 0, v = 0; the bound sums run over f0 in row order (the bounds of -v <= 0 are 0 and add nothing)
  double gs = 1.0, bs = 1.0, fsum = 0.0;
  for (int i = lane; i < n; i += 32) { sh.x[i] = 0.0; gs = fmax(gs, 1.0 + fabs(c[i])); }
  for (int j = lane; j < md; j += 32) { v[j] = 0.0; fsum += fabs(sh.f0[j]); bs = fmax(bs, 1.0 + fabs(sh.f0[j])); }
  auto residuals = [&](double& rdn, double& rpn) {
    for (int i = lane; i < n; i += 32) {
      double a = c[i] + rho * sh.x[i];
      for (int k = 0; k <= i; ++k) a += G[tri_row(i) + k] * sh.x[k];
      for (int k = i + 1; k < n; ++k) a += G[tri_row(k) + i] * sh.x[k];
      rdx[i] = dtmul(i, z + md, a);
    }
    double sz = 0.0;
    for (int j = lane; j < md; j += 32) {
      rdv[j] = rho * v[j] + v[j] - z[j] - z[md + j];
      rs[j] = -v[j] + s[j];
      rs[md + j] = drow(j, sh.x) - v[j] + s[md + j] - sh.f0[j];
      sz += s[j] * z[j] + s[md + j] * z[md + j];
      rdn = fmax(rdn, fabs(rdv[j])); rpn = fmax(rpn, fmax(fabs(rs[j]), fabs(rs[md + j])));
    }
    __syncwarp();
    for (int i = lane; i < n; i += 32) rdn = fmax(rdn, fabs(rdx[i]));
    return sz;
  };
  auto factor = [&]() {
    // ---- Schur complement S (lower triangle): lane c owns column c, so the rows sharing a column block never collide
    for (int j = lane; j < md; j += 32) {
      const double wb = z[j] / s[j], w = z[md + j] / s[md + j], d = 1.0 + rho + wb + w;
      dd[j] = d; wd[j] = w; cw[j] = w * (1.0 + rho + wb) / d;
    }
    for (int idx = lane; idx < n * ld; idx += 32) { const int i = idx / ld, k = idx - i * ld; if (k <= i && i < n) K[idx] = G[tri_row(i) + k] + (i == k ? rho : 0.0); }
    __syncwarp();
    for (int col = lane; col < n; col += 32)
      for (int j = 0; j < md; ++j) {
        const int k = col - sh.dc0[j];
        if (k < 0 || k >= sh.dlen[j]) continue;
        const double a = cw[j] * sh.dco[3 * j + k];
        for (int m = k; m < sh.dlen[j]; ++m) K[(sh.dc0[j] + m) * ld + col] += a * sh.dco[3 * j + m];
      }
    __syncwarp();
    return warp_chol_inv(K, n, ld, kdi, lane, 1e-10);
  };
  // ---- Newton step for the complementarity target rc: dx, dv, ds, dz
  auto newton = [&]() {
    for (int e = lane; e < mi; e += 32) cw[e] = (rc[e] - z[e] * rs[e]) / s[e];
    __syncwarp();
    for (int j = lane; j < md; j += 32) { const double rv = -rdv[j] - cw[j] - cw[md + j]; dv[j] = rv; qv[j] = cw[md + j] + wd[j] * rv / dd[j]; }
    __syncwarp();
    for (int i = lane; i < n; i += 32) t2[i] = dtmul(i, qv, -rdx[i]);
    __syncwarp();
    warp_li_mv(K, n, ld, kdi, t2, t1, lane);
    warp_lit_mv(K, n, ld, kdi, t1, dx, lane);
    for (int j = lane; j < md; j += 32) {
      const double ddx = drow(j, dx), dvj = (dv[j] + wd[j] * ddx) / dd[j];
      dv[j] = dvj;
      ds[j] = -rs[j] + dvj;
      ds[md + j] = -rs[md + j] - (ddx - dvj);
      dz[j] = -(rc[j] + z[j] * ds[j]) / s[j];
      dz[md + j] = -(rc[md + j] + z[md + j] * ds[md + j]) / s[md + j];
    }
    __syncwarp();
  };
  auto step = [&](double alpha) {
    for (int i = lane; i < n; i += 32) sh.x[i] += alpha * dx[i];
    for (int j = lane; j < md; j += 32) v[j] += alpha * dv[j];
  };
  const QpResult res = qp_mehrotra_warp(mi, max_iter, gs, bs, fsum, s, z, ds, dz, rc, [&](int e) { return e < md ? 0.0 : sh.f0[e - md]; },
                                        residuals, factor, newton, step);
  for (int j = lane; j < md; j += 32) sh.v0[j] = v[j];
  __syncwarp();
  return res;
}

}  // namespace hb

namespace {  // the kernels: internal linkage, the library exports only the hb_* entry points
using namespace hb;
__global__ void __launch_bounds__(32) hoqp_kernel(int B, const hb_hoqp_problem* problems, double* scratch, int max_iter, double* x, double* slack, int32_t* status) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int inst = blockIdx.x;
  if (inst >= B) return;
  HoqpShared& sh = *reinterpret_cast<HoqpShared*>(smem_raw);
  QpWorkspace w;
  qp_carve(reinterpret_cast<double*>(smem_raw + sizeof(HoqpShared)), HQ_NQ, w, 1, HQ_ROWS);
  const int st = hoqp_solve_warp(problems[inst], sh, w, scratch + (size_t)inst * HQ_SCRATCH, max_iter, x + (size_t)inst * HQ_N, slack ? slack + (size_t)inst * HQ_STK : nullptr);
  if (status && threadIdx.x == 0) status[inst] = st;
}

// The three tasks of HierarchicalWbc::update from the WBC terms of one instance (decision vector [qdd(16), F(12), tau(10)]):
//   task0 = formulateFloatingBaseEomTask + formulateTorqueLimitsTask + formulateFrictionConeTask + formulateNoContactMotionTask
//   task1 = formulateBaseAccelTask          task2 = formulateContactForceTask * 0.1 + formulateSwingLegTask * 1     (WbcBase.cpp:138-338)
__global__ void __launch_bounds__(32) hwbc_tasks_kernel(int B, hb_wbc_settings ws, const __grid_constant__ InstanceView<hb_terrain> maps,
                                                        const double* x_des, const double* u_des, const double* rbd, const int32_t* mode,
                                                        hb_hoqp_problem* problems) {
  __shared__ WbcShared sh;
  const int inst = blockIdx.x, lane = threadIdx.x;
  if (inst >= B) return;
  const int md_ = mode[inst];
  wbc_terms_warp(x_des + (size_t)inst * NX, u_des + (size_t)inst * NU, rbd + (size_t)inst * 32, md_, false, ws, maps, inst, sh);
  const WbcRows n = wbc_rows(md_, false);
  hb_hoqp_problem& pb = problems[inst];
  if (lane == 0) { pb.n = NWBC; pb.levels = 3; pb.ma[0] = WBC_MA0; pb.md[0] = n.md0; pb.ma[1] = 6; pb.md[1] = 0; pb.ma[2] = n.ma2; pb.md[2] = 0; }
  for (int idx = lane; idx < HB_HOQP_MAX_EQ * NWBC; idx += 32) { (&pb.a[0][0][0])[idx] = 0.0; (&pb.a[1][0][0])[idx] = 0.0; (&pb.a[2][0][0])[idx] = 0.0; }
  for (int idx = lane; idx < HB_HOQP_MAX_IN * NWBC; idx += 32) (&pb.d[0][0][0])[idx] = 0.0;
  __syncwarp();
  wbc_task0_eq(sh, md_, n, WBC_MA0, &pb.a[0][0][0], NWBC, pb.b[0]);
  for (int q = lane; q < n.md0; q += 32) {
    int c0, len; double coef[3];
    pb.f[0][q] = wbc_task0_ineq(ws, md_, q, c0, len, coef, wbc_frames(maps, inst, sh));
    for (int k = 0; k < len; ++k) pb.d[0][q][c0 + k] = coef[k];
  }
  wbc_task12_rows(1, sh.At, sh.bt, n, u_des + (size_t)inst * NU, &pb.a[1][0][0], NWBC, pb.b[1]);
  wbc_task12_rows(2, sh.At, sh.bt, n, u_des + (size_t)inst * NU, &pb.a[2][0][0], NWBC, pb.b[2]);
}

// HierarchicalWbc::update in one launch, one warp per instance (block): WBC terms (wbc_terms_warp), the three tasks in shared memory,
// level 0 by hwbc_level0_warp, levels 1 and 2 by qp_solve_warp at their real shape (n = the free variables level 0 leaves, rows = the
// stacked task0 inequalities), the null-space steps of hoqp_solve_warp in between. sol = x (38), status as hoqp_kernel: 0,
// 10 * (QP status) + level of the first failing level, or 20 + level when a level leaves more than HW_NX free variables.
__global__ void __launch_bounds__(32, 4) hwbc_fused_kernel(int B, hb_wbc_settings ws_ctx, InstanceView<hb_controller_setting> cs,
                                                           const __grid_constant__ InstanceView<hb_terrain> maps, const double* x_des,
                                                           const double* u_des, const double* rbd, const int32_t* mode, int max_iter, double* sol,
                                                           int32_t* status) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int inst = blockIdx.x, lane = threadIdx.x;
  if (inst >= B) return;
  HwbcShared& sh = *reinterpret_cast<HwbcShared*>(smem_raw);
  double* U = reinterpret_cast<double*>(smem_raw + sizeof(HwbcShared));     // scratch of the current phase
  WbcStaged& stg = *reinterpret_cast<WbcStaged*>(U);
  WbcShared& wsh = stg.sh;
  const hb_wbc_settings& ws = wbc_select_settings(ws_ctx, cs, inst, stg.ws);   // read until level 0 takes over U
  const int md_ = mode[inst];
  const double* ud = u_des + (size_t)inst * NU;
  wbc_terms_warp(x_des + (size_t)inst * NX, ud, rbd + (size_t)inst * 32, md_, false, ws, maps, inst, wsh);
  const WbcRows n = wbc_rows(md_, false);
  // task0 (Z = I: AZ = A, r = -b), its inequality rows (the frames are read here, before level 0 takes over U), the motion rows tasks 1
  // and 2 are built from
  wbc_task0_eq(wsh, md_, n, WBC_MA0, sh.AZ, HQ_LDA, sh.r);
  for (int q = lane; q < n.md0; q += 32) sh.f0[q] = wbc_task0_ineq(ws, md_, q, sh.dc0[q], sh.dlen[q], &sh.dco[3 * q], wbc_frames(maps, inst, wsh));
  for (int i = lane; i < 18 * 16; i += 32) sh.At[i] = wsh.At[i];
  if (lane < 18) sh.bt[lane] = wsh.bt[lane];
  for (int idx = lane; idx < HQ_N * HQ_LDZ; idx += 32) { const int i = idx / HQ_LDZ, j = idx - i * HQ_LDZ; sh.Z[idx] = (i == j) ? 1.0 : 0.0; }
  __syncwarp();
  for (int i = lane; i < WBC_MA0; i += 32) sh.r[i] = -sh.r[i];
  __syncwarp();
  const QpResult r0 = hwbc_level0_warp(sh, n.md0, 1e-10, max_iter, U);
  int status_ = r0.status != 0 ? 10 * r0.status : 0;
  int nx = hwbc_null_space_step(sh.Z, sh.AZ, U, sh.pcol, sh.prow, sh.isp, sh.freec, HQ_N, WBC_MA0, HQ_N);
  for (int lvl = 1; lvl < 3; ++lvl) {
    if (nx > HW_NX) { status_ = 20 + lvl; break; }
    double* Ak = U; double* bk = U + WBC_MA0 * NWBC;
    const int ma = wbc_task12_rows(lvl, sh.At, sh.bt, n, ud, Ak, NWBC, bk);
    __syncwarp();
    if (nx == 0) continue;
    hoqp_task_residual(Ak, NWBC, bk, sh.Z, sh.x, HQ_N, ma, nx, sh.AZ, sh.r);
    // the level's QP: H = (AZ)'AZ + 1e-12 I, c = (AZ)'r, rows D0 Z <= f0 - D0 x + v0 (no slack of its own: tasks 1 and 2 have no inequalities)
    QpWorkspace w;
    qp_carve(U, HW_NX, w, 1, HQ_MD);               // over the task rows, which the residual has consumed
    double* Dq = U + qp_workspace_doubles(HW_NX, 1, HQ_MD); double* lbq = Dq + HQ_MD * HW_NX; double* ubq = lbq + HQ_MD;
    double* cq = ubq + HQ_MD; double* zq = cq + HW_NX;
    hoqp_normal_eq(sh.AZ, sh.r, ma, nx, w.H, w.ldn, cq);
    for (int idx = lane; idx < n.md0 * nx; idx += 32) {
      const int i = idx / nx, j = idx - i * nx;
      double s = 0.0;
      for (int k = 0; k < sh.dlen[i]; ++k) s = fma(sh.dco[3 * i + k], sh.Z[(sh.dc0[i] + k) * HQ_LDZ + j], s);
      Dq[idx] = s;
    }
    for (int i = lane; i < n.md0; i += 32) {
      double s = 0.0;
      for (int k = 0; k < sh.dlen[i]; ++k) s = fma(sh.dco[3 * i + k], sh.x[sh.dc0[i] + k], s);
      lbq[i] = -1e20; ubq[i] = sh.f0[i] - s + sh.v0[i];
    }
    __syncwarp();
    const QpResult qr = qp_solve_warp(nx, n.md0, nullptr, cq, Dq, lbq, ubq, 1e-10, max_iter, zq, w);
    __syncwarp();
    if (qr.status != 0 && status_ == 0) status_ = 10 * qr.status + lvl;
    hoqp_update_x(sh.x, sh.Z, zq, HQ_N, nx);
    if (ma > 0) nx = hwbc_null_space_step(sh.Z, sh.AZ, U, sh.pcol, sh.prow, sh.isp, sh.freec, HQ_N, ma, nx);
  }
  double* out = sol + (size_t)inst * NWBC;
  for (int i = lane; i < NWBC; i += 32) out[i] = sh.x[i];
  if (status && lane == 0) status[inst] = status_;
}
}  // namespace
