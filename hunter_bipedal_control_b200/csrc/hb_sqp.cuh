// SQP iteration: the per-node work is split from the sequential recursion so that every SM runs many warps.
//
//   K0 lin_kernel      one warp = TWO horizon nodes (half-warp each). Lane-parallel unit / dual sweeps of the kinematic tree
//                      give, per node and RK2 stage, the non-trivial rows of d f/dx, d f/du and the contact kinematics with
//                      their Jacobians. Output: a compact "linearisation record" per node (LIN_STRIDE doubles).
//   K1 lq_kernel       one warp = one node. RK2 sensitivities using the row sparsity of the flow-map Jacobian, cost and soft
//                      constraints, equality constraints, least-squares projection of the contact-velocity rows (10x10 normal
//                      equations), projected LQ model. Output: "projected record" (PROJ_STRIDE doubles).
//   K2 riccati_kernel  one warp = one instance, sequential in k, only the value-function recursion: S, s, K, k.
//   K3 forward_ls      one warp = one instance: forward pass through the projected model, then the filter line search with
//                      lanes = nodes (flow_map_lane / node_values_lane in hb_mpc.cuh).
//
// Block structure used throughout (x = [hbar(6) | p(3) | theta(3) | qj(10)], u = [F(12) | vj(10)]):
//   d f/dx has non-zero rows 3..11 only; d f/dF is (1/m) I in rows 0..2, (r_c - com)x / m in rows 3..5;
//   d f/dvj is -A_b^-1 A_j in rows 6..11 and I in rows 12..21;
//   the state-input equalities split into "swing force = 0" (selector rows) and contact-velocity rows that involve vj only,
//   so the projection is a 10-dimensional problem; free inputs are the stance forces and the null space of the velocity rows.
#pragma once
#include "hb_common.cuh"
#include "hb_mpc.cuh"
#include "hb_planner.h"
#include "hb_rbd.cuh"

namespace hb {

// ---------------------------------------------------------------- record layouts (doubles)
constexpr int LIN_F1 = 0, LIN_F2 = 22, LIN_A1 = 44, LIN_A2 = 242, LIN_BF1 = 440, LIN_BF2 = 476, LIN_BV1 = 512, LIN_BV2 = 572,
              LIN_EPOS = 632, LIN_EVEL = 644, LIN_DPQ = 656, LIN_DVX = 812, LIN_DVV = 1076, LIN_STRIDE = 1200;
constexpr int NTMAX = 16;   // free inputs after projection: 3 n_stance + (10 - rank of the velocity rows); 12 / 9 / 6 in regular poses
constexpr int NVMAX = 8;    // null-space columns kept for the velocity rows
// Projected record: only the entries that carry data. Each reader stages one contiguous span of it:
//   [B~ rows 3..11 (9 x NTMAX) | A~ rows 3..11 (9 x 22) | P_xv (10 x 22) | N_v (10 x NVMAX) | b~ | q~ | r~ | META]  K2 (one bulk copy)
//   ... followed by p_ev                                                                                           K3 (one bulk copy)
//   Q~ (22 x 22, full: its two halves are not bitwise symmetric)                                                   K2
//   P~ null-space rows (nv x 22 of NVMAX x 22; the stance-force rows of P~ are zero)                               K2
//   R~ packed: one 3x3 block per stance contact (force columns 3b..3b+2), then the nv x nv null block (ld NVMAX)   K2
// The closed-form parts are not stored: A~ rows 0..2 = [I 0], A~ rows 12..21 = [0 I] + dt P_xv, B~ rows 0..2 = dt/m at row c % 3 of
// the force columns c < NF, B~ rows 12..21 = dt N_v on the null-space columns, R~ = I on the padded diagonal and 0 between the blocks.
// Columns of B~, entries of r~ and N_v beyond nt / nv, R~ blocks of swing contacts and P~ / R~ null rows beyond nv are not written.
// The bulk copies still stage those bytes (uninitialised); every reader gates them out by nf / nt / nv, so no value depends on them.
constexpr int PJ_BT = 0, PJ_AT = 144, PJ_PXV = 342, PJ_NV = 562, PJ_BTV = 642, PJ_QV = 664, PJ_RV = 686, PJ_META = 702, PJ_PEV = 710,
              PJ_QT = 720, PJ_PT = 1204, PJ_RF = 1380, PJ_RN = 1416, PJ_STRIDE = 1480;
constexpr int PJ_RT_PACKED = PJ_STRIDE - PJ_RF;   // 4 force blocks (36) + the null block (NVMAX x NVMAX)
static_assert(PJ_AT + 9 * NX == PJ_PXV && PJ_RN + NVMAX * NVMAX == PJ_STRIDE && PJ_PEV + NJ == PJ_QT, "projected record blocks are contiguous");
static_assert(PJ_QT % 2 == 0 && PJ_PT % 2 == 0 && PJ_RF % 2 == 0 && PJ_STRIDE % 2 == 0, "bulk-copied blocks start on 16 bytes");
// META: [0] nt, [1] n_stance_force_dims, [2] nv, [3] dt cost, [4] dt defect^2, [5] dt eq^2, [6] overflow flag, [7] dt
constexpr int RK_STRIDE = NTMAX * NX + NTMAX;  // K (nt x 22, ld 22) + kff

// ---------------------------------------------------------------- K0
struct LinHalf {
  double x[NX], u[NU], x2[NX], f[NX];
  double Acm[6 * 16], Jc[12 * 16], dp[12 * NDIR], dv[12 * NDIR];
  double Abinv[36], AbinvAj[6 * NJ], vgen[16], epos[12], evel[12], com[3];
  double sn[NDIR], cs[NDIR];   // sines / cosines of yaw, pitch, roll and the ten joint angles, shared by all sweeps of a stage
  // dh (6 x 13), dcom (3 x 13), dvb (6 x 13) are contiguous: the per-lane partial sums of a chain-split sweep (`part`: 16 lanes x {P(3), Lo(3),
  // mc(3)}) live in the same storage -- they are consumed (into registers) before dh / dcom / dvb are written
  double dh[6 * NDIR], dcom[3 * NDIR], dvb[6 * NDIR];
  double vals[2 * 6];          // values from the two base-seeded lanes 0 (base + left chain) and 3 (right chain): P(3), mc(3)
};
static_assert(16 * 9 <= 6 * NDIR + 3 * NDIR + 6 * NDIR, "partial sums must fit in the dh | dcom | dvb storage");

// Linearise the flow map of one node at state xs (half-warp cooperative; `hl` = lane within the half, `act` = node exists).
// Writes f, compact A rows 3..11 (9x22), Bf rows 3..5 (3x12), Bv rows 6..11 (6x10); with want_ee the contact kinematics record.
__device__ __noinline__ void lin_half(LinHalf& sh, const ChainModel& cm, const double* xs, int hl, bool act, double* rec_f, double* rec_A, double* rec_Bf,
                                      double* rec_Bv, bool want_ee, double* rec) {
  const double m = c_model.total_mass, im = 1.0 / m;   // products with im instead of divisions on the dependent chains
  double* part = sh.dh;       // aliased storage, see LinHalf
  if (hl < NDIR) { double s, c; sincos(xs[9 + hl], &s, &c); sh.sn[hl] = s; sh.cs[hl] = c; }
  __syncwarp();
  // Lane tasks of the two chain-split sweeps (16 lanes, all busy):
  //   hl 0..2  : Euler coordinate hl,     base body + left chain        hl 3..5  : Euler coordinate hl-3, right chain
  //   hl 6..10 : left joint hl-6, left chain                            hl 11..15: right joint hl-11, right chain
  // `gen` is the generalised coordinate the lane seeds (for joints it equals the lane index). A joint coordinate only moves its own
  // chain; the three translation coordinates have closed-form columns.
  const bool euler = hl < 6;
  const int leg = (hl < 3 || (hl >= 6 && hl < 11)) ? 0 : 1;
  const int gen = euler ? 3 + (hl % 3) : hl;
  const bool with_base = hl < 3;
  const bool vlane = (hl == 0 || hl == 3);   // lanes whose VALUES (not seeds) are used: base + left chain, right chain
  {
    // sweep 1: unit generalised velocity e_gen -> column gen of the centroidal momentum matrix and of the contact Jacobians
    ChainOut<double> co;
    kin_chain_f<double>(cm, leg, with_base, [&](int i) { return xs[6 + i]; }, [&](int i) { return (i == gen) ? 1.0 : 0.0; },
                        [&](int k, double& s, double& c) { s = sh.sn[k]; c = sh.cs[k]; }, co);
#pragma unroll
    for (int i = 0; i < 3; ++i) { part[hl * 9 + i] = co.P[i]; part[hl * 9 + 3 + i] = co.Lo[i]; }
    if (vlane) {
#pragma unroll
      for (int i = 0; i < 3; ++i) sh.vals[(hl / 3) * 6 + 3 + i] = co.mc[i];
    }
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const int c = leg + 2 * t;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        sh.Jc[(3 * c + i) * 16 + gen] = co.cvel[3 * t + i];
        if (!euler) sh.Jc[(3 * (c ^ 1) + i) * 16 + gen] = 0.0;      // the other leg's contacts do not move
        if (vlane) sh.epos[3 * c + i] = co.cpos[3 * t + i];
      }
    }
    if (hl < 3) {   // translation columns: h = [m e; 0], every contact moves with e
#pragma unroll
      for (int r = 0; r < 6; ++r) sh.Acm[r * 16 + hl] = (r == hl) ? m : 0.0;
#pragma unroll
      for (int r = 0; r < 12; ++r) sh.Jc[r * 16 + hl] = ((r % 3) == hl) ? 1.0 : 0.0;
    }
  }
  __syncwarp();
  if (hl < NDIR) {
    // column g = 3 + hl: sum the chain parts, then refer the angular momentum to the centre of mass
    const int g = 3 + hl, la = (hl < 3) ? hl : g;
    double P[3], Lo[3], com[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      P[i] = part[la * 9 + i]; Lo[i] = part[la * 9 + 3 + i];
      if (hl < 3) { P[i] += part[(3 + hl) * 9 + i]; Lo[i] += part[(3 + hl) * 9 + 3 + i]; }
      com[i] = (sh.vals[3 + i] + sh.vals[9 + i]) * im;
    }
    sh.Acm[0 * 16 + g] = P[0]; sh.Acm[1 * 16 + g] = P[1]; sh.Acm[2 * 16 + g] = P[2];
    sh.Acm[3 * 16 + g] = Lo[0] - (com[1] * P[2] - com[2] * P[1]);
    sh.Acm[4 * 16 + g] = Lo[1] - (com[2] * P[0] - com[0] * P[2]);
    sh.Acm[5 * 16 + g] = Lo[2] - (com[0] * P[1] - com[1] * P[0]);
    if (hl == 0) { sh.com[0] = com[0]; sh.com[1] = com[1]; sh.com[2] = com[2]; }
  }
  __syncwarp();
  if (hl < 7) {
    double Ab[36], rhs[6], y[6];
#pragma unroll
    for (int r = 0; r < 6; ++r)
#pragma unroll
      for (int c = 0; c < 6; ++c) Ab[6 * r + c] = sh.Acm[r * 16 + c];
    if (hl < 6) {
#pragma unroll
      for (int r = 0; r < 6; ++r) rhs[r] = (r == hl) ? 1.0 : 0.0;
    } else {
#pragma unroll
      for (int r = 0; r < 6; ++r) { double s = m * xs[r]; for (int j = 0; j < NJ; ++j) s -= sh.Acm[r * 16 + 6 + j] * sh.u[12 + j]; rhs[r] = s; }
    }
    solve6_cmm(Ab, rhs, y);
    if (hl < 6) {
#pragma unroll
      for (int r = 0; r < 6; ++r) sh.Abinv[6 * r + hl] = y[r];
    } else {
#pragma unroll
      for (int r = 0; r < 6; ++r) sh.vgen[r] = y[r];
    }
  }
  if (hl >= 6) sh.vgen[hl] = sh.u[6 + hl];   // vgen[6..15] = joint velocities u[12..21]
  __syncwarp();
  if (hl < NJ) {
#pragma unroll
    for (int r = 0; r < 6; ++r) { double s = 0.0; for (int c = 0; c < 6; ++c) s += sh.Abinv[6 * r + c] * sh.Acm[c * 16 + 6 + hl]; sh.AbinvAj[r * NJ + hl] = s; }
  }
  {
    // sweep 2: dual numbers seeded along configuration coordinate gen (direction gen - 3), generalised velocity held fixed
    const int dir = gen - 3;
    ChainOut<D1> co;
    kin_chain_f<D1>(cm, leg, with_base, [&](int i) { return D1(xs[6 + i], (i == gen) ? 1.0 : 0.0); }, [&](int i) { return D1(sh.vgen[i], 0.0); },
                    [&](int k, D1& s, D1& c) { const double sv = sh.sn[k], cv = sh.cs[k]; const double on = (k == dir) ? 1.0 : 0.0; s = D1(sv, cv * on); c = D1(cv, -sv * on); },
                    co);
#pragma unroll
    for (int i = 0; i < 3; ++i) { part[hl * 9 + i] = co.P[i].d; part[hl * 9 + 3 + i] = co.Lo[i].d; part[hl * 9 + 6 + i] = co.mc[i].d; }
    if (vlane) {
#pragma unroll
      for (int i = 0; i < 3; ++i) { sh.vals[(hl / 3) * 6 + i] = co.P[i].v; sh.vals[(hl / 3) * 6 + 3 + i] = co.mc[i].v; }
    }
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const int c = leg + 2 * t;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const int row = 3 * c + i;
        sh.dp[row * NDIR + dir] = co.cpos[3 * t + i].d;
        sh.dv[row * NDIR + dir] = co.cvel[3 * t + i].d;
        if (!euler) { sh.dp[(3 * (c ^ 1) + i) * NDIR + dir] = 0.0; sh.dv[(3 * (c ^ 1) + i) * NDIR + dir] = 0.0; }
        if (vlane) sh.evel[row] = co.cvel[3 * t + i].v;
      }
    }
  }
  __syncwarp();
  double Pd[3], Ld[3], dc[3], Pv[3], cv[3];
  if (hl < NDIR) {
    const int la = (hl < 3) ? hl : 3 + hl;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      Pd[i] = part[la * 9 + i]; Ld[i] = part[la * 9 + 3 + i]; dc[i] = part[la * 9 + 6 + i];
      if (hl < 3) { Pd[i] += part[(3 + hl) * 9 + i]; Ld[i] += part[(3 + hl) * 9 + 3 + i]; dc[i] += part[(3 + hl) * 9 + 6 + i]; }
      dc[i] *= im;
      Pv[i] = sh.vals[i] + sh.vals[6 + i];
      cv[i] = (sh.vals[3 + i] + sh.vals[9 + i]) * im;
    }
  }
  __syncwarp();     // every partial sum is in registers before dh / dcom overwrite the storage they share
  if (hl < NDIR) {
    // d/dq of h = [P ; Lo - com x P]
    sh.dh[0 * NDIR + hl] = Pd[0]; sh.dh[1 * NDIR + hl] = Pd[1]; sh.dh[2 * NDIR + hl] = Pd[2];
    sh.dh[3 * NDIR + hl] = Ld[0] - ((dc[1] * Pv[2] - dc[2] * Pv[1]) + (cv[1] * Pd[2] - cv[2] * Pd[1]));
    sh.dh[4 * NDIR + hl] = Ld[1] - ((dc[2] * Pv[0] - dc[0] * Pv[2]) + (cv[2] * Pd[0] - cv[0] * Pd[2]));
    sh.dh[5 * NDIR + hl] = Ld[2] - ((dc[0] * Pv[1] - dc[1] * Pv[0]) + (cv[0] * Pd[1] - cv[1] * Pd[0]));
    sh.dcom[0 * NDIR + hl] = dc[0]; sh.dcom[1 * NDIR + hl] = dc[1]; sh.dcom[2 * NDIR + hl] = dc[2];
  }
  __syncwarp();
  if (hl < NDIR) {
#pragma unroll
    for (int r = 0; r < 6; ++r) { double s = 0.0; for (int c = 0; c < 6; ++c) s += sh.Abinv[6 * r + c] * sh.dh[c * NDIR + hl]; sh.dvb[r * NDIR + hl] = -s; }
  }
  // flow map value (all 16 lanes of the half take part; entries 16..21 by lanes 0..5 in a second round)
  for (int i = hl; i < NX; i += 16) {
    double val;
    if (i < 3) {
      double s = 0.0;
      for (int c = 0; c < NC; ++c) s += sh.u[3 * c + i];
      val = s * im - (i == 2 ? HB_GRAVITY : 0.0);
    } else if (i < 6) {
      const int a = i - 3, a1 = (a + 1) % 3, a2 = (a + 2) % 3;
      double s = 0.0;
      for (int c = 0; c < NC; ++c) s += (sh.epos[3 * c + a1] - sh.com[a1]) * sh.u[3 * c + a2] - (sh.epos[3 * c + a2] - sh.com[a2]) * sh.u[3 * c + a1];
      val = s * im;
    } else if (i < 12) val = sh.vgen[i - 6];
    else val = sh.u[i];
    sh.f[i] = val;
    if (act) rec_f[i] = val;
  }
  __syncwarp();
  if (!act) return;
  // compact Jacobian blocks; column j of the 9x22 block by lane (two rounds for 22 columns)
  for (int j = hl; j < NX; j += 16) {
    double ca[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) ca[i] = 0.0;
    if (j < 6) {
#pragma unroll
      for (int r = 0; r < 6; ++r) ca[3 + r] = m * sh.Abinv[6 * r + j];
    } else if (j >= 9) {
      const int k = j - 9;
      double t0 = 0.0, t1 = 0.0, t2 = 0.0;
      for (int c = 0; c < NC; ++c) {
        const double d0 = sh.dp[(3 * c) * NDIR + k] - sh.dcom[k], d1 = sh.dp[(3 * c + 1) * NDIR + k] - sh.dcom[NDIR + k], d2 = sh.dp[(3 * c + 2) * NDIR + k] - sh.dcom[2 * NDIR + k];
        const double* F = sh.u + 3 * c;
        t0 += d1 * F[2] - d2 * F[1]; t1 += d2 * F[0] - d0 * F[2]; t2 += d0 * F[1] - d1 * F[0];
      }
      ca[0] = t0 * im; ca[1] = t1 * im; ca[2] = t2 * im;
#pragma unroll
      for (int r = 0; r < 6; ++r) ca[3 + r] = sh.dvb[r * NDIR + k];
    }
#pragma unroll
    for (int i = 0; i < 9; ++i) rec_A[i * NX + j] = ca[i];
  }
  if (hl < 12) {
    const int c = hl / 3, a = hl - 3 * c;
    const double r0 = (sh.epos[3 * c] - sh.com[0]) * im, r1 = (sh.epos[3 * c + 1] - sh.com[1]) * im, r2 = (sh.epos[3 * c + 2] - sh.com[2]) * im;
    double b0 = 0.0, b1 = 0.0, b2 = 0.0;   // (r - com) x e_a / m
    if (a == 0) { b1 = r2; b2 = -r1; } else if (a == 1) { b0 = -r2; b2 = r0; } else { b0 = r1; b1 = -r0; }
    rec_Bf[0 * 12 + hl] = b0; rec_Bf[1 * 12 + hl] = b1; rec_Bf[2 * 12 + hl] = b2;
  }
  if (hl < NJ) {
#pragma unroll
    for (int r = 0; r < 6; ++r) rec_Bv[r * NJ + hl] = -sh.AbinvAj[r * NJ + hl];
  }
  if (want_ee) {
    if (hl < 12) { rec[LIN_EPOS + hl] = sh.epos[hl]; rec[LIN_EVEL + hl] = sh.evel[hl]; }
    // 29 equal work items (12 rows x one 6-term product each) over the 16 lanes of the node: state columns 0..5 (momentum), 9..21
    // (orientation + joints; the position columns 6..8 are zero) and the ten joint-velocity columns; two rounds, every lane busy in both
    for (int t = hl; t < 29; t += 16) {
      if (t < 6) {
        for (int r = 0; r < 12; ++r) {
          double vx = 0.0;
          for (int c = 0; c < 6; ++c) vx += sh.Jc[r * 16 + c] * sh.Abinv[6 * c + t];
          rec[LIN_DVX + r * NX + t] = vx * m;
        }
      } else if (t < 19) {
        const int k = t - 6, j = 9 + k;
        for (int r = 0; r < 12; ++r) {
          double vx = sh.dv[r * NDIR + k];
          for (int c = 0; c < 6; ++c) vx += sh.Jc[r * 16 + c] * sh.dvb[c * NDIR + k];
          rec[LIN_DPQ + r * NDIR + k] = sh.dp[r * NDIR + k];
          rec[LIN_DVX + r * NX + j] = vx;
        }
      } else {
        const int jj = t - 19;
        for (int r = 0; r < 12; ++r) {
          double vu = sh.Jc[r * 16 + 6 + jj];
          for (int c = 0; c < 6; ++c) vu -= sh.Jc[r * 16 + c] * sh.AbinvAj[c * NJ + jj];
          rec[LIN_DVV + r * NJ + jj] = vu;
        }
      }
    }
    if (hl < 12) { rec[LIN_DVX + hl * NX + 6] = 0.0; rec[LIN_DVX + hl * NX + 7] = 0.0; rec[LIN_DVX + hl * NX + 8] = 0.0; }
  }
}

struct SqpArgs {
  int B, N;
  double dt;
  const double* x_ref; const double* swing; const int32_t* mode;
  double* xt; double* ut;
  double* lin;     // B x N x LIN_STRIDE
  double* proj;    // B x N x PROJ_STRIDE
  double* rk;      // B x N x RK_STRIDE
  double* dxt; double* dut; double* perf; int32_t* flags;
  const double* x0;
  // time discretisation (row S1): node times tk (B x (N+1)) and active interval counts nn (B) of a grid with event nodes; both null =
  // uniform grid of N intervals of length dt. N stays the capacity (stride) of every per-node array.
  const double* tk; const int32_t* nn;
  // MPC maps (hb_mpc_set_maps): each instance's map, and sth, B x (N+1) x 4 ground heights under the stance contacts of each node. K1
  // looks the heights up (stance_height_lane) and writes them for K3; both stance z rows subtract them. sth is null while no map is set,
  // and then no kernel reads either.
  InstanceView<hb_terrain> maps;
  double* sth;
  // MPC cone maps (hb_mpc_set_cone_maps): each instance's map, and cgr, B x (N+1) x 4 x 2 ground gradients (gx, gy) under the stance
  // contacts of each node. K1 looks them up (cone_gradient) and writes them for K3; both friction cones are about the surface frame
  // hbplan::surface_frame builds from them. cgr is null while no cone map is set, and then no kernel reads either.
  InstanceView<hb_terrain> cone_maps;
  double* cgr;
};

// The ground under stance contact `lane` (< 4) of node k on the instance's MPC map: hbplan::map_height at the swing reference's (x, y);
// +0 for a swing contact or an instance without a map (a +0 height leaves the stance z row's bits as they are without one). Stored to
// sth for K3's stance z rows; lanes >= 4 return 0 and store nothing. Read only while a.sth is set.
__device__ __forceinline__ double stance_height_lane(const SqpArgs& a, int inst, int k, int lane, unsigned flm, const double* swing) {
  double h = 0.0;
  if (lane < 4) {
    const hb_terrain* m = a.maps.of(inst);
    if (m && ((flm >> lane) & 1u)) h = hbplan::map_height(m, swing[6 * lane], swing[6 * lane + 1]);
    a.sth[((size_t)inst * (a.N + 1) + k) * 4 + lane] = h;
  }
  return h;
}

// The ground's gradient under stance contact c of node k on the instance's MPC cone map, at the swing reference's (x, y) as for
// stance_height_lane; (+0, +0), flat, for a swing contact or an instance without a cone map. Stored to cgr for K3's cones.
__device__ __forceinline__ void cone_gradient(const SqpArgs& a, int inst, int k, int c, unsigned flm, const double* swing, double& gx, double& gy) {
  gx = 0.0; gy = 0.0;
  const hb_terrain* m = a.cone_maps.of(inst);
  if (m && ((flm >> c) & 1u)) hbplan::terrain_height<true>(*m, swing[6 * c], swing[6 * c + 1], &gx, &gy);
  double* g = a.cgr + (((size_t)inst * (a.N + 1) + k) * 4 + c) * 2;
  g[0] = gx; g[1] = gy;
}
__device__ __forceinline__ int sqp_nn(const SqpArgs& a, int inst) { return a.nn ? a.nn[inst] : a.N; }
__device__ __forceinline__ double sqp_dt(const SqpArgs& a, int inst, int k) {
  if (!a.tk) return a.dt;
  const double* t = a.tk + (size_t)inst * (a.N + 1) + k;
  return t[1] - t[0];
}

#ifndef HB_LIN_MINB
#define HB_LIN_MINB 6
#endif
__global__ void __launch_bounds__(64, HB_LIN_MINB) lin_kernel(SqpArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp_in_block = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31, half = lane >> 4, hl = lane & 15;
  LinHalf& sh = reinterpret_cast<LinHalf*>(smem_raw)[warp_in_block * 2 + half];
  ChainModel& cm = *reinterpret_cast<ChainModel*>(smem_raw + 4 * sizeof(LinHalf));
  chain_model_load(cm, threadIdx.x, blockDim.x);
  __syncthreads();
  const int N = a.N, NP = (N + 1) >> 1;
  const long long w = (long long)blockIdx.x * (blockDim.x >> 5) + warp_in_block;
  if (w >= (long long)a.B * NP) return;
  const int inst = (int)(w / NP), pr = (int)(w - (long long)inst * NP);
  const int nn = sqp_nn(a, inst);
  if (2 * pr >= nn) return;              // both nodes of the pair lie beyond this instance's grid (warp-uniform)
  const int k = 2 * pr + half;
  const bool act = k < nn;
  const int kk = act ? k : nn - 1;
  const double* xk = (kk == 0) ? a.x0 + (size_t)inst * NX : a.xt + ((size_t)inst * (N + 1) + kk) * NX;   // node 0 is pinned to the measured state
  const double* uk = a.ut + ((size_t)inst * N + kk) * NU;
  for (int i = hl; i < NX; i += 16) { sh.x[i] = xk[i]; sh.u[i] = uk[i]; }
  __syncwarp();
  double* rec = a.lin + ((size_t)inst * N + kk) * LIN_STRIDE;
  lin_half(sh, cm, sh.x, hl, act, rec + LIN_F1, rec + LIN_A1, rec + LIN_BF1, rec + LIN_BV1, true, rec);
  const double dtk = sqp_dt(a, inst, kk);
  for (int i = hl; i < NX; i += 16) sh.x2[i] = sh.x[i] + dtk * sh.f[i];
  __syncwarp();
  lin_half(sh, cm, sh.x2, hl, act, rec + LIN_F2, rec + LIN_A2, rec + LIN_BF2, rec + LIN_BV2, false, rec);
}

}  // namespace hb

namespace {  // internal linkage: the library exports only the hb_* entry points
using namespace hb;
// parity probe of the SHIPPING linearisation (lin_half of K0): flow map value, the full Jacobian tiles rebuilt from the compact
// record (rows 3..11 of df/dx, the force / joint-velocity blocks of df/du) and the contact kinematics with their Jacobians.
struct ProbeShared { LinHalf h[2]; ChainModel cm; double rec[LIN_STRIDE]; double dummy[LIN_STRIDE]; };
__global__ void __launch_bounds__(32) probe_flow_map_kernel(int B, const double* x, const double* u, double* f, double* A, double* Bm, double* ee) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  ProbeShared& ps = *reinterpret_cast<ProbeShared*>(smem_raw);
  const int inst = blockIdx.x, lane = threadIdx.x, half = lane >> 4, hl = lane & 15;
  chain_model_load(ps.cm, threadIdx.x, blockDim.x);
  LinHalf& sh = ps.h[half];
  for (int i = hl; i < NX; i += 16) { sh.x[i] = x[(size_t)inst * NX + i]; sh.u[i] = u[(size_t)inst * NU + i]; }
  __syncwarp();
  // both halves linearise the same node; only half 0 writes the record (half 1 runs with act = false into a dummy record)
  double* rec = half == 0 ? ps.rec : ps.dummy;
  lin_half(sh, ps.cm, sh.x, hl, half == 0, rec + LIN_F1, rec + LIN_A1, rec + LIN_BF1, rec + LIN_BV1, true, rec);
  __syncwarp();
  const double im = 1.0 / c_model.total_mass;
  if (lane < NX) f[(size_t)inst * NX + lane] = ps.rec[LIN_F1 + lane];
  for (int idx = lane; idx < TS; idx += 32) {
    const int i = idx / NX, j = idx - i * NX;
    double a = 0.0, b = 0.0;
    if (i >= 3 && i < 12) a = ps.rec[LIN_A1 + (i - 3) * NX + j];
    if (j < 12) {
      if (i < 3) b = (j % 3 == i) ? im : 0.0;
      else if (i < 6) b = ps.rec[LIN_BF1 + (i - 3) * 12 + j];
    } else {
      if (i >= 6 && i < 12) b = ps.rec[LIN_BV1 + (i - 6) * NJ + j - 12];
      else if (i >= 12) b = (i == j) ? 1.0 : 0.0;
    }
    A[(size_t)inst * TS + idx] = a; Bm[(size_t)inst * TS + idx] = b;
  }
  if (ee) {
    double* o = ee + (size_t)inst * (24 + 3 * 12 * NX);
    if (lane < 12) { o[lane] = ps.rec[LIN_EPOS + lane]; o[12 + lane] = ps.rec[LIN_EVEL + lane]; }
    for (int idx = lane; idx < 12 * NX; idx += 32) {
      const int r = idx / NX, j = idx - r * NX;
      double dp = 0.0;
      if (j >= 6 && j < 9) dp = (j - 6 == r % 3) ? 1.0 : 0.0;
      else if (j >= 9) dp = ps.rec[LIN_DPQ + r * NDIR + j - 9];
      o[24 + idx] = dp;
      o[24 + 12 * NX + idx] = ps.rec[LIN_DVX + idx];
      o[24 + 24 * NX + idx] = (j >= 12) ? ps.rec[LIN_DVV + r * NJ + j - 12] : 0.0;
    }
  }
}
}  // namespace

namespace hb {

// ---------------------------------------------------------------- K1
// TMA bulk copies (1-D, cp.async.bulk) completing on an mbarrier: one elected lane arms the barrier with the byte count and issues the
// copies, every lane waits on the phase bit. Addresses and sizes must be multiples of 16 bytes (the node records are).
__device__ __forceinline__ unsigned smem_u32(const void* p) { return static_cast<unsigned>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes),
               "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }   // generic-proxy accesses before, async-proxy (TMA) writes after
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned phase) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(phase)
      : "memory");
}

// Shared memory of the node LQ kernel (14 312 B: 15 CTAs per SM with the 1 KB per-block reserve). `rec` receives the linearisation record by one TMA bulk
// copy; its regions are re-used as soon as they are dead:
//   A1 (9x22)            -> Ad  : rows 3..11 of the discrete A                     (after the RK2 sensitivities)
//   A2 (9x22)            -> BdF (9x12), Bdv (9x10): rows 3..11 of the discrete B
//   EPOS .. DVX (632..)  -> T = [Pxv | Nv | pev | 0] (10 x 32): the joint-velocity part of the input as an affine map of (dx, w, 1)
// `G` holds the 10 x 33 tableau of the least-squares projection, then YZ (8 x 32: reduced gradients of the soft swing rows) + gv (8 x 10).
struct LqShared {
  double rec[LIN_STRIDE];
  double G[NJ * 34];
  double x[NX], u[NU], swing[24];
  double q[NX], Qd[NX], r[NU], b[NX];
  double ev[12], rowg[12], dvd[NJ], RFF[36];
  unsigned long long bar;
  int rowi[12], rowa[12], piv[NJ], freev[NJ];
};
constexpr int LQ_AD = LIN_A1, LQ_BDF = LIN_A2, LQ_BDV = LIN_A2 + 108, LQ_T = LIN_EPOS, LQ_TL = 32, LQ_GL = 34, LQ_YZ = 0, LQ_GV = 256;
static_assert(LQ_BDV + 9 * NJ <= LIN_BF1, "discrete B must fit in the A2 region");
static_assert(LQ_T + NJ * LQ_TL <= LIN_STRIDE && LQ_GV + 8 * NJ <= NJ * LQ_GL, "aliased areas overflow");
static_assert((LQ_T % 2) == 0 && (sizeof(double) * LIN_STRIDE) % 16 == 0, "T is read with 128-bit loads");

// RK2 sensitivities (S2) and the stage cost (M2, M6, M8) of one node: the part of the LQ approximation that does not depend on the number
// of swing contacts, so one copy of its code serves every lq_node<NSW>. Leaves the discrete A / B rows 3..11 in the record and q, Qd, r,
// b, RFF, dvd in shared memory; returns this lane's share of the cost and the warp's squared dynamics defect.
__device__ __forceinline__ void lq_model(LqShared& sh, const SqpArgs& a, int inst, int k, int lane, unsigned flm, int nsw, double dt, double xn_l,
                                         double xref_l, double& cost_l, double& d2_w) {
  const Model& md = c_model;
  const double im = 1.0 / md.total_mass;
  const double* A1c = sh.rec + LIN_A1; const double* A2c = sh.rec + LIN_A2;
  const double* Bf1 = sh.rec + LIN_BF1; const double* Bf2 = sh.rec + LIN_BF2;
  const double* Bv1 = sh.rec + LIN_BV1; const double* Bv2 = sh.rec + LIN_BV2;
  const double* f1 = sh.rec + LIN_F1; const double* f2 = sh.rec + LIN_F2;
  double* Ad = sh.rec + LQ_AD; double* BdF = sh.rec + LQ_BDF; double* Bdv = sh.rec + LQ_BDV;
  // ---- RK2 sensitivities (S2) on the non-trivial rows 3..11, lane = column. Column j of A1 is read by lane j alone, so Ad replaces it
  // at once; B stays in registers until every lane has read A2.
  double bd[9];
  double d2 = 0.0;
  if (lane < NX) {
    const int j = lane;
    double c1[9];
#pragma unroll
    for (int kk = 0; kk < 9; ++kk) c1[kk] = A1c[kk * NX + j];
#pragma unroll 1
    for (int i = 0; i < 9; ++i) {
      double s = 0.0;
#pragma unroll
      for (int kk = 0; kk < 9; ++kk) s = fma(A2c[i * NX + 3 + kk], c1[kk], s);
      Ad[i * NX + j] = 0.5 * dt * (A1c[i * NX + j] + A2c[i * NX + j] + dt * s) + ((3 + i == j) ? 1.0 : 0.0);
    }
    if (j < 12) {
      // B1 force column j = [e_a / m ; Bf1[:, j] ; 0]: (A2 B1)[i][j] = A2c[i][a] / m + A2c[i][3:6] Bf1[:, j]
      const double b0 = Bf1[j], b1 = Bf1[12 + j], b2 = Bf1[24 + j];
      const int ja = j % 3;
#pragma unroll
      for (int i = 0; i < 9; ++i) {
        const double s = A2c[i * NX + 3] * b0 + A2c[i * NX + 4] * b1 + A2c[i * NX + 5] * b2 + A2c[i * NX + ja] * im;
        const double base = (i < 3) ? (Bf1[i * 12 + j] + Bf2[i * 12 + j]) : 0.0;
        bd[i] = 0.5 * dt * (base + dt * s);
      }
    } else {
      const int jj = j - 12;
      double cb[6];
#pragma unroll
      for (int kk = 0; kk < 6; ++kk) cb[kk] = Bv1[kk * NJ + jj];
#pragma unroll
      for (int i = 0; i < 9; ++i) {
        double s = A2c[i * NX + 12 + jj];
#pragma unroll
        for (int kk = 0; kk < 6; ++kk) s = fma(A2c[i * NX + 6 + kk], cb[kk], s);
        const double base = (i >= 3) ? (Bv1[(i - 3) * NJ + jj] + Bv2[(i - 3) * NJ + jj]) : 0.0;
        bd[i] = 0.5 * dt * (base + dt * s);
      }
    }
    const double bb = sh.x[lane] + 0.5 * dt * (f1[lane] + f2[lane]) - xn_l;
    sh.b[lane] = bb; d2 = bb * bb;
  }
  d2 = warp_sum(d2);
  __syncwarp();          // every lane has read A2: its storage takes the discrete B
  if (lane < NX) {
    const int j = lane;
    if (j < 12) {
#pragma unroll
      for (int i = 0; i < 9; ++i) BdF[i * 12 + j] = bd[i];
    } else {
#pragma unroll
      for (int i = 0; i < 9; ++i) Bdv[i * NJ + j - 12] = bd[i];
    }
  }
  // ---- cost (M2, M6, M8), scaled by dt at the end
  const double* __restrict__ ltab = g_lq_lane + lane * LQ_LANE_TAB;     // this lane's constants (global memory: see hb_common.cuh)
  const double fz = (nsw < 4) ? md.total_mass * HB_GRAVITY / (4 - nsw) : 0.0;
  double cost = 0.0;
  if (lane < NX) {
    const double d = sh.x[lane] - xref_l;
    const double Ql = ltab[0];
    sh.q[lane] = Ql * d;
    sh.Qd[lane] = Ql;
    cost += 0.5 * Ql * d * d;
    double s = 0.0;
    if (lane < 12) { double dul = sh.u[lane]; if ((lane % 3) == 2 && ((flm >> (lane / 3)) & 1u)) dul -= fz; s = ltab[1] * dul; cost += 0.5 * dul * s; }
    else {
#pragma unroll
      for (int j = 0; j < NJ; ++j) s = fma(ltab[2 + j], sh.u[12 + j], s);
      cost += 0.5 * sh.u[lane] * s;
    }
    sh.r[lane] = s;
  }
  if (lane < 12) {      // RFF: one 3x3 block per contact (the friction-cone Hessian couples the axes of one contact only)
    const int c = lane / 3, ax = lane - 3 * c;
    sh.RFF[c * 9 + ax * 3] = 0.0; sh.RFF[c * 9 + ax * 3 + 1] = 0.0; sh.RFF[c * 9 + ax * 3 + 2] = 0.0;
  }
  __syncwarp();
  if (lane < 12) { const int c = lane / 3, ax = lane - 3 * c; sh.RFF[c * 9 + ax * 4] = ltab[1]; }
  // all scalar penalties in ONE pass: lanes 0-9 joint position limits, 10-19 joint velocity limits, 20-23 normal-force limits
  // (double sided), 24-27 friction cones of stance contacts (one sided); on sloped ground of an MPC cone map the cone bounds the local
  // force in the surface frame fr (tilt)
  double shiftsum = 0.0;
  {
    double h = 1.0, lo = 0.0, hi = 2.0, pmu = 0.0, pdl = 1.0;
    bool two = true, on = false, tilt = false;
    double Fx = 0.0, Fy = 0.0, Fz = 0.0, tn = 1.0, t2 = 1.0, fr[9];
    if (lane < 10) { h = sh.x[12 + lane]; lo = ltab[12]; hi = ltab[13]; pmu = HB_LIMIT_POS_MU; pdl = HB_LIMIT_POS_DELTA; on = true; }
    else if (lane < 20) { const int j = lane - 10; h = sh.u[12 + j]; lo = ltab[12]; hi = ltab[13]; pmu = HB_LIMIT_VEL_MU; pdl = HB_LIMIT_VEL_DELTA; on = true; }
    else if (lane < 24) { const int c = lane - 20; h = sh.u[3 * c + 2]; lo = 0.0; hi = HB_LIMIT_FORCE_MAX; pmu = HB_LIMIT_FORCE_MU; pdl = HB_LIMIT_FORCE_DELTA; on = true; }
    else if (lane < 28) {
      const int c = lane - 24;
      if (a.cgr) { double gx, gy; cone_gradient(a, inst, k, c, flm, sh.swing, gx, gy); tilt = hbplan::surface_frame(gx, gy, fr); }
      if ((flm >> c) & 1u) {
        Fx = sh.u[3 * c]; Fy = sh.u[3 * c + 1]; Fz = sh.u[3 * c + 2];
        if (tilt) cone_local_force(fr, Fx, Fy, Fz);
        t2 = Fx * Fx + Fy * Fy + HB_FRICTION_REGULARIZATION; tn = sqrt(t2);
        h = HB_FRICTION_MU * Fz - tn; lo = 0.0; pmu = HB_FRICTION_BARRIER_MU; pdl = HB_FRICTION_BARRIER_DELTA; two = false; on = true;
      }
    }
    const Pen pa = relaxed_barrier(h - lo, pmu, pdl);
    const Pen pb = relaxed_barrier(two ? hi - h : 1.0, two ? pmu : 0.0, pdl);
    const double pv = pa.v + pb.v, p1 = pa.d1 - pb.d1, p2 = pa.d2 + pb.d2;
    __syncwarp();
    if (on) {
      cost += pv;
      if (lane < 10) { sh.q[12 + lane] += p1; sh.Qd[12 + lane] += p2; }
      else if (lane < 20) { const int j = lane - 10; sh.r[12 + j] += p1; sh.dvd[j] = p2; }
      else if (lane < 24) { const int c = lane - 20; sh.r[3 * c + 2] += p1; sh.RFF[c * 9 + 8] += p2; }
    }
    __syncwarp();
    if (on && lane >= 24) {
      const int c = lane - 24;
      const double it = 1.0 / tn, it32 = 1.0 / (tn * t2);
      const double g0 = -Fx * it, g1 = -Fy * it, g2 = HB_FRICTION_MU;
      const double h00 = -(Fy * Fy + HB_FRICTION_REGULARIZATION) * it32, h01 = Fx * Fy * it32, h11 = -(Fx * Fx + HB_FRICTION_REGULARIZATION) * it32;
      double* Rc = sh.RFF + c * 9;
      if (tilt) {
        // chained through dF_du = t_R_w, whose rows are t1, t2, n (FrictionConeConstraint.cpp:185-196): g = t_R_w' g_l and
        // H = t_R_w' H_l t_R_w = t1 (h00 t1 + h01 t2)' + t2 (h01 t1 + h11 t2)', H_l having no n row or column
        double gw[3], m1[3], m2[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          gw[i] = g0 * fr[3 + i] + g1 * fr[6 + i] + g2 * fr[i];
          m1[i] = h00 * fr[3 + i] + h01 * fr[6 + i]; m2[i] = h01 * fr[3 + i] + h11 * fr[6 + i];
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          sh.r[3 * c + i] += p1 * gw[i];
#pragma unroll
          for (int j = 0; j < 3; ++j) Rc[3 * i + j] += p2 * gw[i] * gw[j] + p1 * (fr[3 + i] * m1[j] + fr[6 + i] * m2[j]);
        }
      } else {
        sh.r[3 * c] += p1 * g0; sh.r[3 * c + 1] += p1 * g1; sh.r[3 * c + 2] += p1 * g2;
        Rc[0] += p2 * g0 * g0 + p1 * h00; Rc[1] += p2 * g0 * g1 + p1 * h01; Rc[2] += p2 * g0 * g2;
        Rc[3] += p2 * g1 * g0 + p1 * h01; Rc[4] += p2 * g1 * g1 + p1 * h11; Rc[5] += p2 * g1 * g2;
        Rc[6] += p2 * g2 * g0;            Rc[7] += p2 * g2 * g1;            Rc[8] += p2 * g2 * g2;
      }
      shiftsum = -p1 * HB_FRICTION_HESSIAN_SHIFT;
    }
  }
  shiftsum = warp_sum(shiftsum);
  __syncwarp();
  if (lane < NX) sh.Qd[lane] += shiftsum;
  if (lane < 12) sh.RFF[(lane / 3) * 9 + (lane % 3) * 4] += shiftsum;
  else if (lane >= 16 && lane < 16 + NJ) sh.dvd[lane - 16] += shiftsum;
  cost_l = cost; d2_w = d2;
}

// One node of the LQ approximation. NSW = number of swing contacts (0 stance, 2 single support, 4 flight): 3 (4 - NSW) stance-force inputs,
// 12 - 2 NSW contact-velocity rows, 2 NSW soft swing rows.
//
// Every quadratic term in the joint velocities v is reduced through the affine map v = T (dx, w, 1) of the projection:
//   stage cost  1/2 v' Rb v + r_v' v        ->  T' Rb T  (blocks: Qt, Pt, Rt_nn and the vectors qt, rt_n)
//   soft swing  1/2 w_s (h + gx' dx + gv' v)^2  ->  rank one in YZ_p = [gx_p | 0 | h_p] + gv_p' T
// so the projected model is M = T' Rb T + w_s YZ' YZ evaluated once, lane = column, rows streamed from shared memory.
template <int NSW>
__device__ __forceinline__ void lq_node(LqShared& sh, const SqpArgs& a, int inst, int k, int lane, unsigned flm, double dt, double cost, double d2) {
  constexpr int MR = 12 - 2 * NSW, NP = 2 * NSW, NF = 3 * (4 - NSW), GL = LQ_GL, TL = LQ_TL;
  const int N = a.N;
  const Model& md = c_model;
  const double im = 1.0 / md.total_mass;
  double* out = a.proj + ((size_t)inst * N + k) * PJ_STRIDE;
  const double* epos = sh.rec + LIN_EPOS; const double* evel = sh.rec + LIN_EVEL;
  const double* dpq = sh.rec + LIN_DPQ; const double* dvx = sh.rec + LIN_DVX; const double* dvv = sh.rec + LIN_DVV;
  double* Ad = sh.rec + LQ_AD; double* BdF = sh.rec + LQ_BDF; double* Bdv = sh.rec + LQ_BDV; double* T = sh.rec + LQ_T;
  double* G = sh.G; double* YZ = sh.G + LQ_YZ; double* GV = sh.G + LQ_GV;
  // ---- contact-velocity equality rows (M4, M5); swing forces handled separately (M3). Row r -> contact-kinematics row rowi[r] = 3c + axis.
  if (lane == 0) {
    int mr = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if ((flm >> c) & 1u) {
#pragma unroll
        for (int ax = 0; ax < 3; ++ax) { sh.rowi[mr] = 3 * c + ax; sh.rowa[mr] = ax; sh.rowg[mr] = (ax == 2) ? (double)HB_ZEROVEL_Z_GAIN : 0.0; ++mr; }
      } else { sh.rowi[mr] = 3 * c + 2; sh.rowa[mr] = 2; sh.rowg[mr] = (double)HB_POSITION_ERROR_GAIN; ++mr; }
    }
  }
  __syncwarp();
  double hrow = 0.0;      // on an MPC map: the ground under the contact of this lane's row (lane < MR)
  if (a.sth) hrow = __shfl_sync(HB_FULL_MASK, stance_height_lane(a, inst, k, lane, flm, sh.swing), lane < MR ? sh.rowi[lane] / 3 : 0);
  double e2 = 0.0;
  if (lane < MR) {
    const int row = sh.rowi[lane], c = row / 3, ax = row - 3 * c;
    double evv;
    if ((flm >> c) & 1u) {
      evv = evel[row] + (ax == 2 ? HB_ZEROVEL_Z_GAIN * epos[row] + HB_ZEROVEL_Z_OFFSET : 0.0);
      if (ax == 2 && a.sth) evv -= HB_ZEROVEL_Z_GAIN * hrow;       // held at 0.02 + h on a map
    } else evv = evel[row] - sh.swing[6 * c + 5] + HB_POSITION_ERROR_GAIN * (epos[row] - sh.swing[6 * c + 2]);
    sh.ev[lane] = evv;
    e2 = evv * evv;
  }
  if (lane >= 16 && lane < 28) { const int j = lane - 16; if (!((flm >> (j / 3)) & 1u)) e2 += sh.u[j] * sh.u[j]; }
  e2 = warp_sum(e2);
  // ---- least-squares projection on vj: tableau G = Dv' [Dv | -Cv | -ev] (10 x 33, ld 34) built straight from the record. Lane j owns column
  // j: its right operand X[r][j] (Dv for j < 10, -Cv for the 22 state columns) stays in registers, Dv[r][i] is a broadcast load.
  {
    double xr[MR];
#pragma unroll
    for (int r = 0; r < MR; ++r) {
      const int row = sh.rowi[r];
      double v;
      if (lane < NJ) v = dvv[row * NJ + lane];
      else {
        const int jj = lane - NJ;
        double px = 0.0;
        if (jj >= 6 && jj < 9) px = (jj - 6 == sh.rowa[r]) ? 1.0 : 0.0;
        else if (jj >= 9) px = dpq[row * NDIR + jj - 9];
        v = -(dvx[row * NX + jj] + sh.rowg[r] * px);
      }
      xr[r] = v;
    }
#pragma unroll 1
    for (int i = 0; i < NJ; ++i) {
      double s = 0.0;
#pragma unroll
      for (int r = 0; r < MR; ++r) s = fma(dvv[sh.rowi[r] * NJ + i], xr[r], s);
      G[i * GL + lane] = s;
    }
    if (lane < NJ) {
      double s = 0.0;
#pragma unroll
      for (int r = 0; r < MR; ++r) s = fma(-xr[r], sh.ev[r], s);
      G[lane * GL + NJ + NX] = s;
      sh.piv[lane] = 0;
    }
  }
  __syncwarp();
  double dmax = lane < NJ ? G[lane * GL + lane] : 0.0;
  if (NSW > 0) dmax = fmax(dmax, 1.0);     // the swing-force selector rows of D have unit diagonal in D'D
  dmax = warp_max(dmax);
  const double tol = 1e-9 * fmax(dmax, 1e-300);
  for (int step = 0; step < NJ; ++step) {
    double dv = (lane < NJ && !sh.piv[lane]) ? G[lane * GL + lane] : -1.0;
    int pi = lane;
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {      // candidates live in lanes 0..9: a 16-lane butterfly suffices
      const double ov = __shfl_xor_sync(HB_FULL_MASK, dv, o);
      const int oi = __shfl_xor_sync(HB_FULL_MASK, pi, o);
      if (ov > dv || (ov == dv && oi < pi)) { dv = ov; pi = oi; }
    }
    dv = __shfl_sync(HB_FULL_MASK, dv, 0); pi = __shfl_sync(HB_FULL_MASK, pi, 0);
    if (!(dv > tol)) break;
    const int p = pi;
    const double inv = 1.0 / dv;
    // lane j owns column j (j < 32) of the 10 x 33 tableau; the last column (index 32) is updated by lane i for row i
    const double pj = G[p * GL + lane] * inv;                   // scaled pivot-row entry of this lane's column
    const double p32 = G[p * GL + 32] * inv;
    const double colv = (lane < NJ) ? G[lane * GL + p] : 0.0;   // column p before elimination, one entry per lane
    __syncwarp();
    G[p * GL + lane] = pj;
    if (lane == 0) { G[p * GL + 32] = p32; sh.piv[p] = 1; }
#pragma unroll
    for (int i = 0; i < NJ; ++i) {
      const double ci = __shfl_sync(HB_FULL_MASK, colv, i);
      if (i != p) G[i * GL + lane] -= ci * pj;
    }
    if (lane < NJ && lane != p) G[lane * GL + 32] -= colv * p32;
    __syncwarp();
  }
  int nv = 0;
#pragma unroll
  for (int i = 0; i < NJ; ++i) if (!sh.piv[i]) { if (lane == 0) sh.freev[nv] = i; ++nv; }
  bool overflow = false;
  if (nv > NVMAX) { nv = NVMAX; overflow = true; }       // degenerate pose (velocity rows lost rank): flagged, instance reported as failed
  if (NF + nv > NTMAX) { nv = NTMAX - NF; overflow = true; }
  const int nt = NF + nv;
  __syncwarp();
  // ---- column `lane` of T = [Pxv (22) | Nv (8) | pev | 0] in registers
  const int cc = lane - NX;                               // null-space column of lanes 22..29
  const bool nlane = cc >= 0 && cc < nv;                  // lane owns an active null-space column
  double tc[NJ];
  {
    const int fc = (cc >= 0 && cc < NVMAX && cc < nv) ? sh.freev[cc] : -1;
#pragma unroll
    for (int i = 0; i < NJ; ++i) {
      const bool pv = sh.piv[i] != 0;
      double v = 0.0;
      if (lane < NX) v = pv ? G[i * GL + NJ + lane] : 0.0;
      else if (fc >= 0) v = pv ? -G[i * GL + fc] : ((i == fc) ? 1.0 : 0.0);
      else if (lane == 30) v = pv ? G[i * GL + NJ + NX] : 0.0;
      tc[i] = v;
    }
  }
  __syncwarp();       // the tableau is dead: its storage takes YZ and gv
  // ---- xy swing soft constraint (M7): row p = [gx_p (22) | 0 (8) | h_p | 0], gv_p (10)
  if (NP > 0) {
    int p = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if ((flm >> c) & 1u) continue;
#pragma unroll
      for (int ax = 0; ax < 2; ++ax) {
        const int row = 3 * c + ax;
        double v = 0.0;
        if (lane < NX) {
          double px = 0.0;
          if (lane >= 6 && lane < 9) px = (lane - 6 == ax) ? 1.0 : 0.0;
          else if (lane >= 9) px = dpq[row * NDIR + lane - 9];
          v = dvx[row * NX + lane] + HB_XY_POSITION_GAIN * px;
        } else if (lane == 30) v = evel[row] - sh.swing[6 * c + 3 + ax] + HB_XY_POSITION_GAIN * (epos[row] - sh.swing[6 * c + ax]);
        if (p < NP) {
          YZ[p * TL + lane] = v;
          if (lane < NJ) GV[p * NJ + lane] = dvv[row * NJ + lane];
        }
        ++p;
      }
    }
  }
  __syncwarp();       // every read of the contact-kinematics part of the record is done: T takes its place
#pragma unroll
  for (int i = 0; i < NJ; ++i) T[i * TL + lane] = tc[i];
  const double* tl = T + lane;      // column `lane` of T from here on: read back where it is used rather than held in registers
  double wyz[NP > 0 ? NP : 1];
  if (NP > 0) {
    if (lane < NP) { const double g = YZ[lane * TL + 30]; cost += 0.5 * HB_SOFT_SWING_WEIGHT * g * g; }
    __syncwarp();       // the unreduced h_p are read before lane 30 replaces them
    double yz[NP > 0 ? NP : 1];
#pragma unroll
    for (int p = 0; p < NP; ++p) yz[p] = YZ[p * TL + lane];
#pragma unroll 1
    for (int kk = 0; kk < NJ; ++kk) {
      const double t = tl[kk * TL];
#pragma unroll
      for (int p = 0; p < NP; ++p) yz[p] = fma(GV[p * NJ + kk], t, yz[p]);
    }
#pragma unroll
    for (int p = 0; p < NP; ++p) {
      wyz[p] = HB_SOFT_SWING_WEIGHT * yz[p];
      YZ[p * TL + lane] = yz[p];
    }
  }
  cost = warp_sum(cost);
  // ---- Rb T (column `lane`): Rb = R_vv (constant) + diag(velocity-limit curvature + shift); linear term r_v' T
  double rb[NJ];
  double lin = 0.0;
#pragma unroll
  for (int i = 0; i < NJ; ++i) rb[i] = sh.dvd[i] * tl[i * TL];
#pragma unroll 1
  for (int kk = 0; kk < NJ; ++kk) {
    const double t = tl[kk * TL];
#pragma unroll
    for (int i = 0; i < NJ; ++i) rb[i] = fma(md.R[(12 + i) * NU + 12 + kk], t, rb[i]);
    lin = fma(sh.r[12 + kk], t, lin);
  }
  __syncwarp();
  // ---- M = T' Rb T + YZ' (w YZ), row by row (rows come in pairs with 128-bit broadcast loads); lane = column:
  //   lanes 0..21 : rows 0..21 -> Qt, row 30 -> qt          lanes 22..29 : rows 0..21 -> Pt (stored input-major, NTMAX x 22), rows 22..29 -> Rt (null block), row 30 -> rt
  const double Qd_l = (lane < NX) ? sh.Qd[lane] : 0.0;
  auto m_store = [&](int i, double s) {
    if (i < NX) {
      if (lane < NX) out[PJ_QT + i * NX + lane] = dt * (s + ((i == lane) ? Qd_l : 0.0));
      else if (nlane) out[PJ_PT + cc * NX + i] = dt * s;
    } else if (i < NX + NVMAX) {
      if (nlane && i - NX < nv) out[PJ_RN + (i - NX) * NVMAX + cc] = dt * s;
    } else {
      if (lane < NX) out[PJ_QV + lane] = dt * (sh.q[lane] + s + lin);
      else if (nlane) out[PJ_RV + NF + cc] = dt * (s + lin);
    }
  };
#pragma unroll 1
  for (int i = 0; i < 30; i += 2) {
    double s0 = 0.0, s1 = 0.0;
#pragma unroll
    for (int kk = 0; kk < NJ; ++kk) {
      const double2 t = *reinterpret_cast<const double2*>(T + kk * TL + i);
      s0 = fma(t.x, rb[kk], s0); s1 = fma(t.y, rb[kk], s1);
    }
#pragma unroll
    for (int p = 0; p < NP; ++p) {
      const double2 y = *reinterpret_cast<const double2*>(YZ + p * TL + i);
      s0 = fma(y.x, wyz[p], s0); s1 = fma(y.y, wyz[p], s1);
    }
    m_store(i, s0); m_store(i + 1, s1);
  }
  {
    double s = 0.0;
#pragma unroll
    for (int kk = 0; kk < NJ; ++kk) s = fma(T[kk * TL + 30], rb[kk], s);
#pragma unroll
    for (int p = 0; p < NP; ++p) s = fma(YZ[p * TL + 30], wyz[p], s);
    m_store(30, s);
  }
  // ---- dynamics through T: Bdv T (rows 3..11) -> At (lanes 0..21, + Ad), Bt null columns (lanes 22..29), bt (lane 30); rows 12..21 are dt T
  double at9[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) at9[i] = (lane < NX) ? Ad[i * NX + lane] : 0.0;
#pragma unroll 1
  for (int kk = 0; kk < NJ; ++kk) {
    const double t = tl[kk * TL];
#pragma unroll
    for (int i = 0; i < 9; ++i) at9[i] = fma(Bdv[i * NJ + kk], t, at9[i]);
  }
  if (lane == 30) {
#pragma unroll
    for (int i = 0; i < 9; ++i) sh.b[3 + i] += at9[i];
#pragma unroll
    for (int kk = 0; kk < NJ; ++kk) sh.b[12 + kk] += dt * tl[kk * TL];
  }
  // role of the lane in the input-column writes: lanes 0..NF-1 own the stance-force columns, lanes 22..29 the null-space columns NF + cc
  const bool fcol = lane < NF;
  const int col = nlane ? NF + cc : lane;
  int sj = 0;           // input index of stance-force column `lane`
  if (fcol) {
    int cnt = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) if ((flm >> c) & 1u) { if (lane >= cnt && lane < cnt + 3) sj = 3 * c + lane - cnt; cnt += 3; }
  }
  if (lane < NX) {
#pragma unroll
    for (int i = 0; i < 9; ++i) out[PJ_AT + i * NX + lane] = at9[i];
#pragma unroll
    for (int i = 0; i < NJ; ++i) out[PJ_PXV + i * NX + lane] = tl[i * TL];
  } else if (nlane) {
#pragma unroll
    for (int i = 0; i < NJ; ++i) out[PJ_NV + i * NVMAX + cc] = tl[i * TL];
  } else if (lane == 30) {
#pragma unroll
    for (int i = 0; i < NJ; ++i) out[PJ_PEV + i] = tl[i * TL];
  }
  if (fcol || nlane) {
#pragma unroll
    for (int i = 0; i < 9; ++i) out[PJ_BT + i * NTMAX + col] = fcol ? BdF[i * 12 + sj] : at9[i];
  }
  if (fcol) {
    // column sa of the 3x3 R~ block of this lane's contact, stored as block lane / 3 (the contact's rank among the stance contacts)
    const int sa = sj % 3;
    out[PJ_RV + col] = dt * sh.r[sj];
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) out[PJ_RF + 9 * (lane / 3) + ax * 3 + sa] = dt * sh.RFF[(sj / 3) * 9 + ax * 3 + sa];
  }
  __syncwarp();
  // bt = b + Bd_v pev + dt pev - Bd_F[:, swing] F_swing
  if (lane < NX) {
    const int i = lane;
    double s = sh.b[i];
    if (NSW > 0) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if ((flm >> c) & 1u) continue;
        if (i < 3) s -= dt * im * sh.u[3 * c + i];
        else if (i < 12) s -= BdF[(i - 3) * 12 + 3 * c] * sh.u[3 * c] + BdF[(i - 3) * 12 + 3 * c + 1] * sh.u[3 * c + 1] + BdF[(i - 3) * 12 + 3 * c + 2] * sh.u[3 * c + 2];
      }
    }
    out[PJ_BTV + lane] = s;
  }
  if (lane == 0) { out[PJ_META] = nt; out[PJ_META + 1] = NF; out[PJ_META + 2] = nv; out[PJ_META + 3] = dt * cost; out[PJ_META + 4] = dt * d2; out[PJ_META + 5] = dt * e2; out[PJ_META + 6] = overflow ? 1.0 : 0.0; out[PJ_META + 7] = dt; }
}

// Minimum resident warps per SM: 15 is what shared memory allows, with the full carveout hb_create requests. A warp lives on one of the
// SM's four 16 K-register sub-partitions, so 13..16 warps cap a thread at 128 registers; the kernel fits in that without spills because
// Ad and the column of T go to shared memory instead of waiting in registers. The extra warps pay only with compact code, since warps
// out of phase each stream it through the instruction cache: hence lq_model as one copy and the rolled inner-product loops. On H100
// (configs[1]) K1 takes 1.74 ms per step, against 2.88 ms at 8 warps and 3.04 ms at 15 warps with every loop unrolled.
#ifndef HB_LQ_MINB
#define HB_LQ_MINB 15
#endif
static_assert(HB_LQ_MINB * (sizeof(LqShared) + 1024) <= 228 * 1024, "lq_kernel must fit HB_LQ_MINB blocks per SM");
__global__ void __launch_bounds__(32, HB_LQ_MINB) lq_kernel(SqpArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  LqShared& sh = *reinterpret_cast<LqShared*>(smem_raw);
  const int lane = threadIdx.x;
  const int N = a.N;
  const long long w = blockIdx.x;
  const int inst = (int)(w / N), k = (int)(w - (long long)inst * N);
  if (k >= sqp_nn(a, inst)) return;      // node beyond this instance's grid (event-node grids have per-instance interval counts)
  const double* grec = a.lin + ((size_t)inst * N + k) * LIN_STRIDE;
  const double* xk = (k == 0) ? a.x0 + (size_t)inst * NX : a.xt + ((size_t)inst * (N + 1) + k) * NX;
  // ---- one TMA bulk copy for the record (9568 B) and one each for x, u, the swing references; a single mbarrier collects the bytes
  if (lane == 0) {
    constexpr unsigned REC_BYTES = (LIN_DVV + 12 * NJ) * sizeof(double), V_BYTES = NX * sizeof(double), SW_BYTES = 24 * sizeof(double);
    mbar_init(&sh.bar, 1);
    mbar_expect_tx(&sh.bar, REC_BYTES + 2 * V_BYTES + SW_BYTES);
    bulk_g2s(sh.rec, grec, REC_BYTES, &sh.bar);
    bulk_g2s(sh.x, xk, V_BYTES, &sh.bar);
    bulk_g2s(sh.u, a.ut + ((size_t)inst * N + k) * NU, V_BYTES, &sh.bar);
    bulk_g2s(sh.swing, a.swing + ((size_t)inst * (N + 1) + k) * 24, SW_BYTES, &sh.bar);
  }
  __syncwarp();
  const int mode = a.mode[(size_t)inst * (N + 1) + k];
  double xn_l = 0.0, xref_l = 0.0;
  if (lane < NX) { xn_l = a.xt[((size_t)inst * (N + 1) + k + 1) * NX + lane]; xref_l = a.x_ref[((size_t)inst * (N + 1) + k) * NX + lane]; }
  int nsw = 0;
#pragma unroll
  for (int c = 0; c < 4; ++c) nsw += contact_flag(mode, c) ? 0 : 1;
  mbar_wait(&sh.bar, 0);
  const double dt = sqp_dt(a, inst, k);
  const unsigned flm = (contact_flag(mode, 0) ? 1u : 0u) | (contact_flag(mode, 1) ? 2u : 0u) | (contact_flag(mode, 2) ? 4u : 0u) | (contact_flag(mode, 3) ? 8u : 0u);
  double cost, d2;
  lq_model(sh, a, inst, k, lane, flm, nsw, dt, xn_l, xref_l, cost, d2);
  if (nsw == 2) lq_node<2>(sh, a, inst, k, lane, flm, dt, cost, d2);
  else if (nsw == 0) lq_node<0>(sh, a, inst, k, lane, flm, dt, cost, d2);
  else lq_node<4>(sh, a, inst, k, lane, flm, dt, cost, d2);
}

// ---------------------------------------------------------------- K2: value-function recursion
// Row-owner products: lane i owns row i of the result, the right operand is streamed from shared memory with 128-bit
// broadcast loads (two doubles per load), N accumulators stay in registers. NTP = number of free inputs padded to an even
// compile-time size (6 flight, 10 single support, 12 stance, 16 degenerate); the padded rows/columns of the projected model
// are zero (identity on the diagonal of R~), so the padded gains are zero.
// TC: the result is stored transposed (C[j * ldc + i]): lanes then touch consecutive addresses -- the layout of choice whenever the
// row-major leading dimension would be a multiple of 16 doubles (every lane in the same bank).

// acc_rows: c[j] = fma(a(k), B[k * ldb + j], c[j]) for k = 0 .. kn-1 in ascending order; a(k) is the lane's entry of the left operand.
template <int N, class AF>
__device__ __forceinline__ void acc_rows(double (&c)[N], AF a, const double* __restrict__ B, int ldb, int kn) {
#pragma unroll 2
  for (int k = 0; k < kn; ++k) {
    const double ak = a(k);
    const double* br = B + k * ldb;
#pragma unroll
    for (int j = 0; j < N; j += 2) {
      const double2 b2 = *reinterpret_cast<const double2*>(br + j);
      c[j] = fma(ak, b2.x, c[j]);
      c[j + 1] = fma(ak, b2.y, c[j + 1]);
    }
  }
}

// Row-owner shell: lane i < m owns row i of C (N columns): c starts at 0 (MODE 0) or at C (MODE 1), body(c, i) accumulates, c is stored.
template <int N, int MODE, bool TC = false, class Body>
__device__ __forceinline__ void rowmm_by(double* __restrict__ C, int ldc, int m, Body body) {
  const int i = lane_id();
  if (i < m) {
    double c[N];
#pragma unroll
    for (int j = 0; j < N; ++j) c[j] = (MODE == 1) ? (TC ? C[j * ldc + i] : C[i * ldc + j]) : 0.0;
    body(c, i);
#pragma unroll
    for (int j = 0; j < N; ++j) { if (TC) C[j * ldc + i] = c[j]; else C[i * ldc + j] = c[j]; }
  }
  __syncwarp();
}

// Tile products, for the 22 x 22 results of the node: the lanes form a grid of 32 / GJ x GJ, and lane (li, lj) owns the TI x TJ block
// of the result at row li * TI, column lj * TJ. Both operands are k-major (L[k * ldl + i], R[k * ldr + j]), so per k a lane loads the
// TI and TJ consecutive entries under its block (the right span with 128-bit loads when TJ is even) and issues TI * TJ DFMAs: 5 loads
// for 12 DFMAs with 3 x 4 blocks, on every lane, where the row-owner form issues 12 loads for 22 DFMAs on 22 of 32 lanes. Each
// accumulator still sees its operands in ascending k, so the values are the row-owner ones. Entries beyond the m x n result are loaded
// as zeros and never stored.

// acc_tile: c[r][j] = fma(L[k * ldl + r], R[k * ldr + j], c[r][j]) for k = 0 .. kn-1 in ascending order; L and R point at the lane's first
// row and column, mi and nj are the rows and columns of its block that lie inside the result.
template <int TI, int TJ>
__device__ __forceinline__ void acc_tile(double (&c)[TI][TJ], const double* __restrict__ L, int ldl, int mi, const double* __restrict__ R, int ldr, int nj, int kn) {
#pragma unroll 2
  for (int k = 0; k < kn; ++k) {
    double a[TI], b[TJ];
#pragma unroll
    for (int r = 0; r < TI; ++r) a[r] = (r < mi) ? L[k * ldl + r] : 0.0;
    if constexpr (TJ % 2 == 0) {
#pragma unroll
      for (int j = 0; j < TJ; j += 2) {
        const double2 b2 = (j < nj) ? *reinterpret_cast<const double2*>(R + k * ldr + j) : make_double2(0.0, 0.0);
        b[j] = b2.x; b[j + 1] = b2.y;
      }
    } else {
#pragma unroll
      for (int j = 0; j < TJ; ++j) b[j] = (j < nj) ? R[k * ldr + j] : 0.0;
    }
#pragma unroll
    for (int r = 0; r < TI; ++r) {
#pragma unroll
      for (int j = 0; j < TJ; ++j) c[r][j] = fma(a[r], b[j], c[r][j]);
    }
  }
}

// Tile shell: c starts at 0, body(c, i0, j0, mi, nj) accumulates, the block is stored to C (row-major, m x n). An even TJ needs n, ldc
// and C's offset even: its column pairs are then whole and 16-byte aligned.
template <int TI, int TJ, int GJ, class Body>
__device__ __forceinline__ void tilemm_by(double* __restrict__ C, int ldc, int m, int n, Body body) {
  const int lane = lane_id(), i0 = (lane / GJ) * TI, j0 = (lane % GJ) * TJ;
  const int mi = m - i0, nj = n - j0;
  double c[TI][TJ];
#pragma unroll
  for (int r = 0; r < TI; ++r) {
#pragma unroll
    for (int j = 0; j < TJ; ++j) c[r][j] = 0.0;
  }
  body(c, i0, j0, mi, nj);
#pragma unroll
  for (int r = 0; r < TI; ++r) {
    if (r < mi) {
      double* cr = C + (i0 + r) * ldc + j0;
      if constexpr (TJ % 2 == 0) {
#pragma unroll
        for (int j = 0; j < TJ; j += 2) if (j < nj) *reinterpret_cast<double2*>(cr + j) = make_double2(c[r][j], c[r][j + 1]);
      } else {
#pragma unroll
        for (int j = 0; j < TJ; ++j) if (j < nj) cr[j] = c[r][j];
      }
    }
  }
  __syncwarp();
}

// Tile shell for the lower triangle of a symmetric NX x NX result: the TI x TJ blocks that hold an entry on or below the diagonal are
// numbered row of blocks by row of blocks, and thread t takes block t (30 blocks of 3 x 4, 55 of 3 x 2). c starts at init(i, j),
// body(c, i0, j0, mi, nj) accumulates, store(i, j, v) takes every entry with j <= i; the entries of a diagonal block above the diagonal
// are computed and dropped.
template <int TI, int TJ, class Init, class Body, class Store>
__device__ __forceinline__ void tri_tile(int t, Init init, Body body, Store store) {
  constexpr int NBI = (NX + TI - 1) / TI, NBJ = (NX + TJ - 1) / TJ;
  int bi = 0;
  for (; bi < NBI; ++bi) {
    const int nb = min(NBJ, (TI * bi + TI - 1) / TJ + 1);      // blocks of block row bi that reach the diagonal
    if (t < nb) break;
    t -= nb;
  }
  const int i0 = bi * TI, j0 = t * TJ;
  const int mi = bi < NBI ? NX - i0 : 0, nj = NX - j0;
  double c[TI][TJ];
#pragma unroll
  for (int r = 0; r < TI; ++r) {
#pragma unroll
    for (int j = 0; j < TJ; ++j) c[r][j] = (r < mi && j0 + j <= i0 + r) ? init(i0 + r, j0 + j) : 0.0;
  }
  body(c, i0, j0, mi, nj);
#pragma unroll
  for (int r = 0; r < TI; ++r) {
#pragma unroll
    for (int j = 0; j < TJ; ++j) if (r < mi && j0 + j <= i0 + r) store(i0 + r, j0 + j, c[r][j]);
  }
  __syncwarp();
}

constexpr int SB_LD = 18;
// Node inputs as staged in shared memory: the leading span of the projected record, one bulk copy. The rows of A~ and B~ that the record
// does not store are closed-form values; the recursion multiplies only the support of each row and column of A~ and B~:
//   A~ rows 0..2    the identity rows: adds (fma(a, 1.0, c) rounds as a + c)
//   A~ rows 12..21  [0 I] + dt P_xv, regenerated in place of the staged P_xv with the fma lq_node used for them
//   B~ rows 0..2    dt/m (dt * (1/m)) at row c % 3 of each stance-force column c < nf
//   B~ rows 12..21  dt N_v on the null-space columns nf .. nt-1
//   padded columns  nt .. NTP-1 of B~ are zero: no rows at all
// Skipping fma(a, 0.0, c) leaves c as it was, and the remaining terms keep their order, so every value is the one the full products
// give (the sign of an exact zero aside).
struct RicNodeIn { double Bt9[9 * NTMAX], At3[19 * NX], Nv[NJ * NVMAX], bt[NX], qt[NX], rt[NTMAX], meta[8]; };
static_assert(offsetof(RicNodeIn, At3) == PJ_AT * sizeof(double) && offsetof(RicNodeIn, Nv) == PJ_NV * sizeof(double) &&
              offsetof(RicNodeIn, meta) == PJ_META * sizeof(double) && sizeof(RicNodeIn) == PJ_PEV * sizeof(double), "RicNodeIn mirrors the record");
// Column classes of a node: nf stance-force columns, then the null-space columns up to nt, then padding up to NTP. NF >= 0: the regular
// class of a stance (12), single-support (6) or flight (0) node, with NF and NT known at compile time; NF < 0: any other node (rank
// loss of the contact-velocity rows), classes read from META.
__host__ __device__ constexpr int nt_regular(int nf) { return nf == 12 ? 12 : (nf == 6 ? 9 : 6); }
template <int NF>
struct NodeCols {
  double dt, dtim; int nf, nt;
  __device__ explicit NodeCols(const double* meta)
      : dt(meta[7]), dtim(meta[7] * (1.0 / c_model.total_mass)), nf(NF >= 0 ? NF : (int)meta[1]), nt(NF >= 0 ? nt_regular(NF) : (int)meta[1] + (int)meta[2]) {}
  __device__ bool force(int c) const { return c < nf; }
  __device__ bool null(int c) const { return c >= nf && c < nt; }
  __device__ bool data(int c) const { return c < nt; }
};
// c[j] += sum_k a(k) B~[k][j] (B~ as the right operand), k = 0..21 in order, over the support of each column j
template <int NTP, int NF, class AF>
__device__ __forceinline__ void acc_bt(double (&c)[NTP], const RicNodeIn& in, const NodeCols<NF>& g, AF a) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double ak = a(k);
#pragma unroll
    for (int j = k; j < NTP; j += 3) if (g.force(j)) c[j] = fma(ak, g.dtim, c[j]);
  }
#pragma unroll 2
  for (int k = 0; k < 9; ++k) {
    const double ak = a(k + 3);
    const double* br = in.Bt9 + k * NTMAX;
#pragma unroll
    for (int j = 0; j < NTP; j += 2) {
      if (g.data(j)) {
        const double2 b2 = *reinterpret_cast<const double2*>(br + j);
        c[j] = fma(ak, b2.x, c[j]);
        if (g.data(j + 1)) c[j + 1] = fma(ak, b2.y, c[j + 1]);
      }
    }
  }
#pragma unroll 2
  for (int k = 0; k < NJ; ++k) {
    const double ak = a(k + 12);
#pragma unroll
    for (int j = 0; j < NTP; ++j) if (g.null(j)) c[j] = fma(ak, g.dt * in.Nv[k * NVMAX + j - g.nf], c[j]);
  }
}

struct RicShared {
  double S[TS], SA[TS];
  RicNodeIn in[2];                                   // node data, staged one node ahead by TMA
  double SBK[NX * SB_LD];                            // SB (22 x NTP, leading dimension 18: 2-way instead of 16-way bank conflicts on the row-owner stores), later K (NTMAX x 22)
  double Hux[NTMAX * NX], Huu[NTMAX * 18];           // Hux input-major (NTMAX x 22): lanes = state index touch consecutive addresses
  double sv[NX], sb[NX], hu[NTMAX], kff[NTMAX];
  unsigned long long bar[4];                         // mbarriers of the TMA staging: node inputs (two buffers), P~ / R~, Q~
};
// The packed R~ lands at the end of Huu and is expanded from there (every entry read before any is written)
constexpr int HUU_RP = NTMAX * 18 - PJ_RT_PACKED;
constexpr int SA_SPLIT = 14;                         // phase A: columns 0..13 of SA on warp 0, 14..21 (with SB, sb) on warp 1
static_assert(sizeof(RicNodeIn) % 16 == 0 && (TS * sizeof(double)) % 16 == 0 && (NX * sizeof(double)) % 16 == 0 && HUU_RP % 2 == 0 &&
              (PJ_RT_PACKED * sizeof(double)) % 16 == 0 && SA_SPLIT % 2 == 0, "bulk copies and 128-bit loads need 16-byte multiples");
// One block per instance: 8 blocks per SM put a 1024-instance batch in one wave on 132 SMs (8 x 132 >= 1024; at 7 a tail wave of 100
// blocks costs almost as much as the full one). The runtime reserves 1 KB of shared memory per block.
static_assert(8 * (sizeof(RicShared) + 1024) <= 228 * 1024, "riccati_kernel must fit 8 blocks per SM");

// node inputs by TMA: one elected lane arms the buffer's mbarrier with the byte count and issues the bulk copies
__device__ __forceinline__ void ric_prefetch_tma(RicNodeIn& n, const double* __restrict__ rec, unsigned long long* bar) {
  fence_proxy_async();
  mbar_expect_tx(bar, (unsigned)sizeof(RicNodeIn));
  bulk_g2s(&n, rec, sizeof(RicNodeIn), bar);
}

// One node of the recursion, executed by the TWO warps of the block. The products that do not depend on each other are split
// between the warps by result columns; the 22 x 22 results (SA, Qt + At' SA, S += Hux' K) are tile products over all 32 lanes, the
// products with B~ (SB, Hux, Huu), which skip the zeros of its columns, are row-owner products. The Cholesky of Huu and the gain
// solve (one warp, latency bound) overlap with the largest product At' S At of the other warp.
template <int NTP, int NF>
__device__ __noinline__ void riccati_node(RicShared& sh, RicNodeIn& in, const double* __restrict__ rec, double* __restrict__ rk, bool& fail,
                                          int warp_arg, unsigned ph) {
  // the role as a value the compiler knows to be the same on every lane: taken as it arrives, it brackets each shuffle of the
  // role's branch in a WARPSYNC / ENDCOLLECTIVE pair
  const int warp = __shfl_sync(HB_FULL_MASK, warp_arg, 0);
  const int lane = lane_id();
  const NodeCols<NF> g(in.meta);
  double* SB = sh.SBK; double* K = sh.SBK;
  {
    // A~ rows 12..21 over this warp's phase-A columns, in place of the staged P_xv: fma(P_xv, dt, 1 or 0) as lq_node formed them
    const int c0 = warp == 0 ? 0 : SA_SPLIT, w = warp == 0 ? SA_SPLIT : NX - SA_SPLIT;
    for (int idx = lane; idx < NJ * w; idx += 32) {
      const int r = idx / w, j = c0 + idx - r * w;
      double& v = in.At3[(9 + r) * NX + j];
      v = __fma_rn(v, g.dt, (12 + r == j) ? 1.0 : 0.0);
    }
    __syncwarp();
  }
  // ---- phase A: [SA | SB | sb] = S [At | Bt | bt] (+ s): 22 + NTP + 1 result columns, split SA_SPLIT / rest. S is exactly symmetric (phase D
  // writes both halves with the same value), so lane i reads its row as column i: consecutive addresses, no
  // bank conflicts (S^T: lane i reads S[k][i])
  if (warp == 0) {
    tilemm_by<3, 4, 4>(sh.SA, NX, NX, SA_SPLIT, [&](double (&c)[3][4], int i0, int j0, int mi, int nj) {
      if (j0 == 0) {                          // columns 0..2: the identity rows of A~
#pragma unroll
        for (int r = 0; r < 3; ++r) {
#pragma unroll
          for (int j = 0; j < 3; ++j) if (r < mi) c[r][j] = c[r][j] + sh.S[j * NX + i0 + r];
        }
      }
      acc_tile(c, sh.S + 3 * NX + i0, NX, mi, in.At3 + j0, NX, nj, 19);
    });
    mbar_wait(&sh.bar[2], ph);                // P~ / R~ staged by this warp at the top of the node
  } else {
    tilemm_by<3, 2, 4>(sh.SA + SA_SPLIT, NX, NX, NX - SA_SPLIT, [&](double (&c)[3][2], int i0, int j0, int mi, int nj) {
      acc_tile(c, sh.S + 3 * NX + i0, NX, mi, in.At3 + SA_SPLIT + j0, NX, nj, 19);
    });
    rowmm_by<NTP, 0>(SB, SB_LD, NX, [&](double (&c)[NTP], int i) { acc_bt(c, in, g, [&](int k) { return sh.S[k * NX + i]; }); });
    if (lane < NX) {
      double s0 = sh.sv[lane], s1 = 0.0;
#pragma unroll
      for (int k = 0; k < NX; k += 2) { s0 = fma(sh.S[k * NX + lane], in.bt[k], s0); s1 = fma(sh.S[(k + 1) * NX + lane], in.bt[k + 1], s1); }
      sh.sb[lane] = s0 + s1;
    }
  }
  __syncthreads();
  // ---- phase B: Hux (NTP x 22, stored input-major) = Pt + Bt^T SA (warp 0: row-owner over the state index, transposed store) ; Huu = Rt + Bt^T SB, hu = rt + Bt^T sb (warp 1)
  if (warp == 0) {
    rowmm_by<NTP, 0, true>(sh.Hux, NX, NX, [&](double (&c)[NTP], int i) {     // P~ is zero outside the null-space rows
#pragma unroll
      for (int j = 0; j < NTP; ++j) if (g.null(j)) c[j] = sh.Hux[j * NX + i];
      acc_bt(c, in, g, [&](int k) { return sh.SA[k * NX + i]; });
    });
  } else {
    // S is dead until phase C: stage Qt into it now (arrives while Huu is formed)
    if (lane == 0) { fence_proxy_async(); mbar_expect_tx(&sh.bar[3], TS * sizeof(double)); bulk_g2s(sh.S, rec + PJ_QT, TS * sizeof(double), &sh.bar[3]); }
    rowmm_by<NTP, 0>(sh.Huu, 18, NTP, [&](double (&c)[NTP], int i) {      // Bt^T: lane i owns column i of Bt
      // row i of R~ from its packed blocks at Huu + HUU_RP: 3x3 force blocks, the null block, I on the padded diagonal. Every lane
      // reads its row before any lane stores one over the packed blocks.
      const double* rp = sh.Huu + HUU_RP;
#pragma unroll
      for (int j = 0; j < NTP; ++j) {
        if (g.force(i) && g.force(j) && i / 3 == j / 3) c[j] = rp[9 * (i / 3) + (i % 3) * 3 + j % 3];
        else if (g.null(i) && g.null(j)) c[j] = rp[PJ_RN - PJ_RF + (i - g.nf) * NVMAX + j - g.nf];
        else if (i == j && !g.data(i)) c[j] = 1.0;
      }
      __syncwarp((1u << NTP) - 1u);
      if (g.force(i)) acc_rows(c, [&](int) { return g.dtim; }, SB + (i % 3) * SB_LD, SB_LD, 1);
      if (g.data(i)) acc_rows(c, [&](int k) { return in.Bt9[k * NTMAX + i]; }, SB + 3 * SB_LD, SB_LD, 9);
      if (g.null(i)) acc_rows(c, [&](int k) { return g.dt * in.Nv[k * NVMAX + i - g.nf]; }, SB + 12 * SB_LD, SB_LD, NJ);
    });
    if (lane < NTP) {
      double s0 = g.data(lane) ? in.rt[lane] : 0.0;
      if (g.force(lane)) s0 = fma(g.dtim, sh.sb[lane % 3], s0);
      if (g.data(lane)) {
#pragma unroll
        for (int k = 0; k < 9; ++k) s0 = fma(in.Bt9[k * NTMAX + lane], sh.sb[3 + k], s0);
      }
      if (g.null(lane)) {
#pragma unroll
        for (int k = 0; k < NJ; ++k) s0 = fma(g.dt * in.Nv[k * NVMAX + lane - g.nf], sh.sb[12 + k], s0);
      }
      sh.hu[lane] = s0;
    }
  }
  __syncthreads();
  // ---- phase C: gains (warp 0) || S = Qt + At' SA (warp 1)
  // (Measured and rejected: factorising Huu in warp 1's phase-B slack and keeping the factor in registers across the barrier -- the
  // kernel needs 255 registers then, and capped for occupancy the factor lives in local memory, which is slower. 8 blocks/SM, which
  // puts 1024 instances in one wave, leave 128 registers per thread.)
  // The identity rows of A~ are adds on the result rows 0..2 (result row i takes row i of SA; the other rows skip fma(0.0, SA, c) = c).
  if (warp == 0) {
    // Cholesky of the symmetrised Huu entirely in registers: lane i owns row i (right-looking, column by column, the pivot column is
    // broadcast with shuffles), then forward / backward substitution of the 22 + 1 right-hand sides, one per lane, with the factor
    // entries fetched from their owner lanes. No shared-memory round trips on this latency-bound stretch.
    {
      // 1 / L[j][j] stays on lane j alone and is broadcast where a substitution divides by it (off the dependent chain): as a per-lane
      // array of NTP equal values it would not leave room for 8 blocks per SM
      double a[NTP], rinv = 0.0;
#pragma unroll
      for (int c = 0; c < NTP; ++c) a[c] = (lane < NTP && c <= lane) ? 0.5 * (sh.Huu[lane * 18 + c] + sh.Huu[c * 18 + lane]) : 0.0;
#pragma unroll
      for (int j = 0; j < NTP; ++j) {
        double d = __shfl_sync(HB_FULL_MASK, a[j], j);
        if (!(d > 0.0)) { fail = true; d = 1.0; }
        const double r = rsqrt(d);
        if (lane == j) rinv = r;
        const double l = a[j] * r;              // L[i][j] on lane i >= j
        a[j] = l;
#pragma unroll
        for (int k = j + 1; k < NTP; ++k) a[k] = fma(-l, __shfl_sync(HB_FULL_MASK, l, k), a[k]);
      }
      double col[NTP], y[NTP];
#pragma unroll
      for (int c = 0; c < NTP; ++c) {
        double sacc = (lane < NX) ? sh.Hux[c * NX + lane] : ((lane == NX) ? sh.hu[c] : 0.0);
#pragma unroll
        for (int kk = 0; kk < c; ++kk) sacc = fma(-__shfl_sync(HB_FULL_MASK, a[kk], c), y[kk], sacc);
        y[c] = sacc * __shfl_sync(HB_FULL_MASK, rinv, c);
      }
#pragma unroll
      for (int c = NTP - 1; c >= 0; --c) {
        double sacc = y[c];
#pragma unroll
        for (int kk = c + 1; kk < NTP; ++kk) sacc = fma(-__shfl_sync(HB_FULL_MASK, a[c], kk), col[kk], sacc);
        col[c] = sacc * __shfl_sync(HB_FULL_MASK, rinv, c);     // solution of Huu x = rhs; the gain is its negative
      }
      if (lane < NX) {
#pragma unroll
        for (int c = 0; c < NTP; ++c) { K[c * NX + lane] = -col[c]; rk[c * NX + lane] = -col[c]; }     // SB is dead: K takes its place
      } else if (lane == NX) {
#pragma unroll
        for (int c = 0; c < NTP; ++c) { sh.kff[c] = -col[c]; rk[NTMAX * NX + c] = -col[c]; }
      }
    }
    __syncwarp();
    // s <- qt + At' sb + Hux' kff
    if (lane < NX) {
      double s0 = in.qt[lane], s1 = 0.0;
      if (lane == 1) s1 = s1 + sh.sb[1];                    // rows 0..2 of A~ (identity), even rows on s0 and odd rows on s1
      else if (lane < 3) s0 = s0 + sh.sb[lane];
#pragma unroll
      for (int k = 3; k < NX; ++k) {
        if (k & 1) s1 = fma(in.At3[(k - 3) * NX + lane], sh.sb[k], s1);
        else s0 = fma(in.At3[(k - 3) * NX + lane], sh.sb[k], s0);
      }
#pragma unroll
      for (int c = 0; c < NTP; ++c) s0 = fma(sh.Hux[c * NX + lane], sh.kff[c], s0);
      sh.sv[lane] = s0 + s1;
    }
  } else {
    mbar_wait(&sh.bar[3], ph);   // Qt has landed in S
    __syncwarp();
    // lower triangle only, started from the symmetric part of Qt (the record's halves differ in the last bits); the entries above the
    // diagonal are read here and never written, so no lane reads what another stores
    tri_tile<3, 4>(lane, [&](int i, int j) { return 0.5 * (sh.S[i * NX + j] + sh.S[j * NX + i]); },
                   [&](double (&c)[3][4], int i0, int j0, int mi, int nj) {   // At^T: row i of the result takes column i of At
#pragma unroll
      for (int r = 0; r < 3; ++r) {             // rows 0..2 of A~ (identity): result row i < 3 takes row i of SA
#pragma unroll
        for (int j = 0; j < 4; ++j) if (i0 + r < 3 && j < nj) c[r][j] = c[r][j] + sh.SA[(i0 + r) * NX + j0 + j];
      }
      acc_tile(c, in.At3 + i0, NX, mi, sh.SA + 3 * NX + j0, NX, nj, 19);
    }, [&](int i, int j, double v) { sh.S[i * NX + j] = v; });
  }
  __syncthreads();
  // ---- phase D: S += Hux' K on the lower triangle, its 55 blocks of 3 x 2 over the 64 threads; every value goes to both halves, so S is
  // exactly symmetric with no averaging pass. The init reads entries on or below the diagonal only, the mirror stores go above it.
  tri_tile<3, 2>((int)threadIdx.x, [&](int i, int j) { return sh.S[i * NX + j]; },
                 [&](double (&c)[3][2], int i0, int j0, int mi, int nj) { acc_tile(c, sh.Hux + i0, NX, mi, K + j0, NX, nj, NTP); },
                 [&](int i, int j, double v) { sh.S[i * NX + j] = v; if (j < i) sh.S[j * NX + i] = v; });
  __syncthreads();
}

// 128 registers x 64 threads also allow 8 blocks per SM, and the bound says so: with the warp-uniform role ptxas schedules the node
// more freely and takes 138 registers when left alone (6 blocks per SM, two waves at 1024 instances); bounded it uses 126 with the same
// 8 B stack frame and no spills.
__global__ void __launch_bounds__(64, 8) riccati_kernel(SqpArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  RicShared& sh = *reinterpret_cast<RicShared*>(smem_raw);
  const int inst = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double* proj = a.proj + (size_t)inst * a.N * PJ_STRIDE;
  const int N = sqp_nn(a, inst);         // active intervals of this instance; a.N is the stride
  // warp 1 owns the node-input prefetch (and the Qt staging), warp 0 the Pt / Rt staging
  if (threadIdx.x == 0) { for (int b = 0; b < 4; ++b) mbar_init(&sh.bar[b], 1); }
  __syncthreads();
  if (warp == 1 && lane == 0) ric_prefetch_tma(sh.in[(N - 1) & 1], proj + (size_t)(N - 1) * PJ_STRIDE, &sh.bar[(N - 1) & 1]);
  unsigned ph_in0 = 0u, ph_in1 = 0u;
  for (int idx = threadIdx.x; idx < TS; idx += 64) sh.S[idx] = 0.0;   // no terminal cost (SURVEY App. B)
  if (threadIdx.x < NX) sh.sv[threadIdx.x] = 0.0;
  bool fail = false;
  double merit = 0.0, dyn = 0.0, eqs = 0.0;
  __syncthreads();
  for (int k = N - 1; k >= 0; --k) {
    const double* rec = proj + (size_t)k * PJ_STRIDE;
    double* rk = a.rk + ((size_t)inst * a.N + k) * RK_STRIDE;
    const unsigned ph = (unsigned)(N - 1 - k) & 1u;      // phase of the once-per-node barriers
    // every thread waits for the inputs of node k (prefetched one node ahead); the block barrier that ends the previous node (after
    // phase D, the last reader of Hux and K; the other input buffer was last read in phase C) already orders the re-use of Hux / Huu / that
    // buffer, so no barrier is needed here
    if (k & 1) { mbar_wait(&sh.bar[1], ph_in1); ph_in1 ^= 1u; } else { mbar_wait(&sh.bar[0], ph_in0); ph_in0 ^= 1u; }
    RicNodeIn& in = sh.in[k & 1];
    const int nt = (int)in.meta[0], nf = (int)in.meta[1], nv = (int)in.meta[2];
    if (warp == 0) {
      if (lane == 0) {
        // P~ null rows -> rows nf .. nt-1 of Hux (input-major, contiguous) and the packed R~ -> the end of Huu: 2 bulk copies on one mbarrier
        fence_proxy_async();
        mbar_expect_tx(&sh.bar[2], (unsigned)((nv * NX + PJ_RT_PACKED) * sizeof(double)));
        if (nv > 0) bulk_g2s(sh.Hux + nf * NX, rec + PJ_PT, nv * NX * sizeof(double), &sh.bar[2]);
        bulk_g2s(sh.Huu + HUU_RP, rec + PJ_RF, PJ_RT_PACKED * sizeof(double), &sh.bar[2]);
      }
    } else if (k > 0 && lane == 0) {
      ric_prefetch_tma(sh.in[(k - 1) & 1], proj + (size_t)(k - 1) * PJ_STRIDE, &sh.bar[(k - 1) & 1]);
    }
    merit += in.meta[3]; dyn += in.meta[4]; eqs += in.meta[5];
    if (in.meta[6] != 0.0) fail = true;
    if (nf == 12 && nt == nt_regular(12)) riccati_node<12, 12>(sh, in, rec, rk, fail, warp, ph);
    else if (nf == 6 && nt == nt_regular(6)) riccati_node<10, 6>(sh, in, rec, rk, fail, warp, ph);
    else if (nf == 0 && nt == nt_regular(0)) riccati_node<6, 0>(sh, in, rec, rk, fail, warp, ph);
    else riccati_node<NTMAX, -1>(sh, in, rec, rk, fail, warp, ph);
  }
  if (threadIdx.x == 0) {
    double* pf = a.perf + (size_t)inst * 4;
    pf[0] = merit; pf[1] = dyn; pf[2] = eqs; pf[3] = 0.0;
    a.flags[inst] = fail ? 1 : 0;
  }
}

// ---------------------------------------------------------------- K3: forward pass + filter line search
// per-node data of the forward pass, double-buffered and filled with cp.async (16-byte LDGSTS) one node ahead
// The record stores rows 3..11 of A~ and B~ only: rows 0..2 are the identity plus dt/m on the stance-force coordinates, rows 12..21 are
// I + dt P_xv and dt N_v, and P_xv / N_v are loaded anyway for the input step. Three bulk copies: the leading span of the projected
// record, the gains (K then kff) and the input.
struct FwNode {
  double Bt9[9 * NTMAX], At9[9 * NX], Pxv[NJ * NX], Nv[NJ * NVMAX], bt[NX], qt[NX], rt[NTMAX], meta[8], pev[NJ];
  double K[NTMAX * NX], kff[NTMAX], u[NU];
};
static_assert(offsetof(FwNode, At9) == PJ_AT * sizeof(double) && offsetof(FwNode, pev) == PJ_PEV * sizeof(double) &&
              offsetof(FwNode, K) == PJ_QT * sizeof(double) && offsetof(FwNode, u) == offsetof(FwNode, K) + RK_STRIDE * sizeof(double),
              "FwNode mirrors the record and the gains");
struct Fw2Shared {
  FwNode nd[2];
  double dx[NX], dxn[NX], w[NTMAX];
  unsigned long long bar[2];
};
static_assert(sizeof(FwNode) % 16 == 0 && (NJ * sizeof(double)) % 16 == 0 && (NJ * NX * sizeof(double)) % 16 == 0, "bulk copies need 16-byte multiples");

__device__ __forceinline__ void fw_prefetch_tma(FwNode& n, const double* __restrict__ rec, const double* __restrict__ rk, const double* __restrict__ uk,
                                                unsigned long long* bar) {
  fence_proxy_async();
  mbar_expect_tx(bar, (unsigned)sizeof(FwNode));
  bulk_g2s(n.Bt9, rec, PJ_QT * sizeof(double), bar);
  bulk_g2s(n.K, rk, RK_STRIDE * sizeof(double), bar);
  bulk_g2s(n.u, uk, sizeof(n.u), bar);
}

__global__ void __launch_bounds__(32) forward_linesearch2_kernel(SqpArgs a, int max_trials, void* info_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fw2Shared& sh = *reinterpret_cast<Fw2Shared*>(smem_raw);
  const int inst = blockIdx.x, lane = threadIdx.x, NS = a.N;     // NS: stride (capacity); N: active intervals of this instance
  const int N = sqp_nn(a, inst);
  double* xt = a.xt + (size_t)inst * (NS + 1) * NX;
  double* ut = a.ut + (size_t)inst * NS * NU;
  double* dxt = a.dxt + (size_t)inst * (NS + 1) * NX;
  double* dut = a.dut + (size_t)inst * NS * NU;
  const double* xref = a.x_ref + (size_t)inst * (NS + 1) * NX;
  const double* swing = a.swing + (size_t)inst * (NS + 1) * 24;
  const int32_t* mode = a.mode + (size_t)inst * (NS + 1);
  const double* proj = a.proj + (size_t)inst * NS * PJ_STRIDE;
  const double* rkb = a.rk + (size_t)inst * NS * RK_STRIDE;
  if (lane == 0) { mbar_init(&sh.bar[0], 1); mbar_init(&sh.bar[1], 1); }
  __syncwarp();
  if (lane == 0) fw_prefetch_tma(sh.nd[0], proj, rkb, ut, &sh.bar[0]);
  unsigned fph0 = 0u, fph1 = 0u;
  if (lane < NX) { xt[lane] = a.x0[(size_t)inst * NX + lane]; sh.dx[lane] = 0.0; dxt[lane] = 0.0; }
  double armijo = 0.0;
  bool finite = (a.flags[inst] == 0);
  const double im_mass = 1.0 / c_model.total_mass;
  for (int k = 0; k < N; ++k) {
    // the other buffer was last read at node k - 1 (the __syncwarp that ends every node orders those reads before the new copies)
    if (k + 1 < N && lane == 0) fw_prefetch_tma(sh.nd[(k + 1) & 1], proj + (size_t)(k + 1) * PJ_STRIDE, rkb + (size_t)(k + 1) * RK_STRIDE, ut + (k + 1) * NU, &sh.bar[(k + 1) & 1]);
    if (k & 1) { mbar_wait(&sh.bar[1], fph1); fph1 ^= 1u; } else { mbar_wait(&sh.bar[0], fph0); fph0 ^= 1u; }
    const FwNode& nd = sh.nd[k & 1];
    const int nt = (int)nd.meta[0], nf = (int)nd.meta[1], nv = (int)nd.meta[2];
    const int md_k = mode[k];
    const double dtk = sqp_dt(a, inst, k);
    unsigned fmask = 0u;      // stance force coordinates of the node (three bits per stance contact)
#pragma unroll
    for (int c = 0; c < 4; ++c) if (contact_flag(md_k, c)) fmask |= 7u << (3 * c);
    double arm = 0.0;
    if (lane < nt) {
      double s = nd.kff[lane];
#pragma unroll
      for (int j = 0; j < NX; ++j) s = fma(nd.K[lane * NX + j], sh.dx[j], s);
      sh.w[lane] = s;
      arm = nd.rt[lane] * s;
    }
    __syncwarp();
    if (lane < NX) {
      // du: stance forces are free variables, swing forces go to zero, vj from the projection
      double du;
      if (lane < 12) {
        if (contact_flag(md_k, lane / 3)) du = sh.w[__popc(fmask & ((1u << lane) - 1u))];      // index among the stance force coordinates
        else du = -nd.u[lane];
      } else {
        const int i = lane - 12;
        du = nd.pev[i];
#pragma unroll
        for (int j = 0; j < NX; ++j) du = fma(nd.Pxv[i * NX + j], sh.dx[j], du);
        for (int c = 0; c < nv; ++c) du = fma(nd.Nv[i * NVMAX + c], sh.w[nf + c], du);
      }
      // dx' = A~ dx + B~ w + b~ by row class
      double s = nd.bt[lane];
      if (lane >= 3 && lane < 12) {
        const double* ar = nd.At9 + (lane - 3) * NX;
        const double* br = nd.Bt9 + (lane - 3) * NTMAX;
        double s1 = 0.0;
#pragma unroll
        for (int j = 0; j < NX; j += 2) { s = fma(ar[j], sh.dx[j], s); s1 = fma(ar[j + 1], sh.dx[j + 1], s1); }
        s += s1;
        for (int c = 0; c < nt; ++c) s = fma(br[c], sh.w[c], s);
      } else if (lane < 3) {
        double fsum = 0.0;      // linear momentum rate: sum of the stance-force steps along this axis
#pragma unroll
        for (int c = 0; c < 4; ++c) if (contact_flag(md_k, c)) fsum += sh.w[__popc(fmask & ((1u << (3 * c + lane)) - 1u))];
        s += sh.dx[lane] + (dtk * im_mass) * fsum;
      } else {
        s += sh.dx[lane] + dtk * (du - nd.pev[lane - 12]);      // rows I + dt P_xv | dt N_v: dt times the joint-velocity step without its affine part
      }
      sh.dxn[lane] = s;
      dxt[(k + 1) * NX + lane] = s;
      arm += nd.qt[lane] * sh.dx[lane];
      dut[k * NU + lane] = du;
      if (!isfinite(s) || !isfinite(du)) finite = false;
    }
    armijo += warp_sum(arm);
    __syncwarp();
    if (lane < NX) sh.dx[lane] = sh.dxn[lane];
    __syncwarp();
  }
  finite = __all_sync(HB_FULL_MASK, finite);
  const double* pf = a.perf + (size_t)inst * 4;
  const double merit0 = pf[0], v0 = sqrt(pf[1] + pf[2]);
  const double gamma_c = 1e-6, armijoFactor = 1e-4, alpha_decay = 0.5, alpha_min = 1e-4;
  double alpha = 1.0, merit1 = merit0, v1 = v0;
  bool accepted = false;
  int trials = 0;
  if (finite) {
    while (alpha >= alpha_min && trials < max_trials) {
      double ms = 0.0, ds = 0.0, es = 0.0;
      for (int k = lane; k < N; k += 32) {
        const double dt = sqp_dt(a, inst, k);
        double x[NX], u[NU], xn[NX], f1[NX], f2[NX], x2[NX], ep[12], ev[12], xr[NX], sw[24];
        for (int i = 0; i < NX; ++i) { x[i] = xt[k * NX + i] + alpha * dxt[k * NX + i]; xn[i] = xt[(k + 1) * NX + i] + alpha * dxt[(k + 1) * NX + i]; xr[i] = xref[k * NX + i]; }
        for (int i = 0; i < NU; ++i) u[i] = ut[k * NU + i] + alpha * dut[k * NU + i];
        for (int i = 0; i < 24; ++i) sw[i] = swing[k * 24 + i];
        flow_map_lane(x, u, f1, ep, ev);
        for (int i = 0; i < NX; ++i) x2[i] = x[i] + dt * f1[i];
        flow_map_lane(x2, u, f2, nullptr, nullptr);
        double d2 = 0.0;
        for (int i = 0; i < NX; ++i) { const double d = x[i] + 0.5 * dt * (f1[i] + f2[i]) - xn[i]; d2 += d * d; }
        double cost, e2;
        node_values_lane(x, u, xr, sw, mode[k], ep, ev, a.sth ? a.sth + ((size_t)inst * (NS + 1) + k) * 4 : nullptr,
                         a.cgr ? a.cgr + ((size_t)inst * (NS + 1) + k) * 8 : nullptr, cost, e2);
        ms += dt * cost; ds += dt * d2; es += dt * e2;
      }
      ms = warp_sum(ms); ds = warp_sum(ds); es = warp_sum(es);
      ++trials;
      const double vn = sqrt(ds + es);
      const double am = alpha * armijo;
      bool acc;
      if (vn > HB_SQP_G_MAX) acc = vn < (1.0 - gamma_c) * v0;
      else if (vn < HB_SQP_G_MIN && v0 < HB_SQP_G_MIN && am < 0.0) acc = ms < merit0 + armijoFactor * am;
      else acc = ms < (merit0 - gamma_c * v0) || vn < (1.0 - gamma_c) * v0;
      if (isfinite(ms) && isfinite(vn) && acc) { accepted = true; merit1 = ms; v1 = vn; break; }
      alpha *= alpha_decay;
    }
  }
  if (accepted) {
    // accepted step: x += alpha dx, u += alpha du; four independent loads in flight per lane (one warp streams 70 KB here)
    auto axpy = [&](double* y, const double* d, int n) {
      int idx = lane;
      for (; idx + 96 < n; idx += 128) {
        const double y0 = y[idx], y1 = y[idx + 32], y2 = y[idx + 64], y3 = y[idx + 96];
        const double d0 = d[idx], d1 = d[idx + 32], d2 = d[idx + 64], d3 = d[idx + 96];
        y[idx] = fma(alpha, d0, y0); y[idx + 32] = fma(alpha, d1, y1); y[idx + 64] = fma(alpha, d2, y2); y[idx + 96] = fma(alpha, d3, y3);
      }
      for (; idx < n; idx += 32) y[idx] = fma(alpha, d[idx], y[idx]);
    };
    axpy(xt, dxt, (N + 1) * NX);
    axpy(ut, dut, N * NU);
  }
  if (lane == 0 && info_out) {
    struct Info { double alpha, merit0, merit1, viol0, viol1, armijo; int32_t status, n_trials; };
    Info* io = reinterpret_cast<Info*>(info_out) + inst;
    io->alpha = accepted ? alpha : 0.0; io->merit0 = merit0; io->merit1 = merit1; io->viol0 = v0; io->viol1 = v1;
    io->armijo = armijo; io->status = finite ? 0 : 3; io->n_trials = trials;
  }
}

}  // namespace hb
