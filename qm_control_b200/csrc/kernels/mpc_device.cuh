// Warp-per-node pieces of the LQ projection kernel (K2b of mpc_kernels.cu): the state reference of a lane and the quadratic model of the node's cost
//   LeggedRobotStateInputQuadraticCost (include/qm_interface/cost/LeggedRobotQuadraticTrackingCost.h:34-40),
//   EndEffectorConstraint soft cost (src/constraint/EndEffectorConstraint.cpp:36-113, QMInterface.cpp:147-172),
//   arm joint soft box (QMInterface.cpp:177-259), friction-cone soft constraint (QMInterface.cpp:344-358).
// The kinematics, the flow map with its analytic Jacobian blocks, the foot-velocity rows (ZeroVelocity / NormalVelocity, QMInterface.cpp:116-131) and the
// end-effector error with its Jacobian come from the thread-per-node flow kernel (node_eval.cuh); the reference differentiates all of these with CppAD tapes.
#pragma once
#include "dev_common.cuh"
#include "mpc_scalar.cuh"

namespace qmb {

// state reference of this lane at time t (TargetTrajectories::getDesiredState().head(30), linear interpolation between the knots)
__device__ __forceinline__ double target_xnom(const double* tt, const double* ts /*[K][37]*/, int nk, double t, int lane) {
  int idx; double a; time_segment(tt, nk, t, idx, a);
  const double* l = ts + (size_t)idx * 37; const double* rr = ts + (size_t)((nk > 1) ? idx + 1 : idx) * 37;
  if (nk <= 1) a = 1.0;
  return (lane < NX) ? a * l[lane] + (1.0 - a) * rr[lane] : 0.0;
}

// Intermediate (or terminal) cost value and its quadratic model in the compact form of QuadWs (NOT scaled by dt).  ws: {x[30], u[30]} of the node; cw: end-effector
// error e[6] and its Jacobian Je[6][12] (flow kernel); sc: the robot's SRBD constants (srbd_of); tn: the robot's end-effector weights and friction coefficient (tuning_of);
// xnom: this lane's state reference; `flagmask` = contact flags (bit i = foot i).  Returns the value (lane-uniform).
template <class WS, class CW>
__device__ __forceinline__ double stage_cost_quad(const DevModel* __restrict__ mdl, const SrbdConst* sc, const Tuning* tn, const WS* ws, const CW* cw, QuadWs* qw, double xnom, int flagmask, bool terminal, int lane) {
  double value = 0.0;
  for (int e = lane; e < 144; e += 32) qw->E[e] = 0.0; for (int e = lane; e < 36; e += 32) qw->fric[e] = 0.0; if (lane < NX) { qw->qdiag[lane] = 0.0; qw->rdiag[lane] = 0.0; qw->qf[lane] = 0.0; qw->rf[lane] = 0.0; } __syncwarp();
  int nst = 0; for (int i = 0; i < 4; ++i) nst += (flagmask >> i) & 1;
  if (!terminal) {
    // tracking cost: 1/2 dx'Q dx + 1/2 du'R du, u_nom = weightCompensatingInput(contact flags)
    double dx = 0.0, du = 0.0;
    if (lane < NX) { dx = ws->x[lane] - xnom; double un = 0.0; if (lane < 12 && (lane % 3) == 2 && ((flagmask >> (lane / 3)) & 1)) un = sc->m * 9.81 / nst; du = ws->u[lane] - un; }
    double qd = 0.0, rd = 0.0;
    if (mdl->q_is_diag) { if (lane < NX) qd = mdl->Qdiag[lane] * dx; }
    else { const double* Qr = mdl->Q + (lane < NX ? lane : 0) * NX;
#pragma unroll 6
      for (int j = 0; j < NX; ++j) qd = fma(Qr[j], __shfl_sync(FULL, dx, j), qd); }
    { // R is block diagonal (checked at create): 3x3 blocks over the 8 force / leg-joint triples, diagonal over the arm
      const int blk = lane < 24 ? lane / 3 : 0, row = lane - 3 * blk; const double* Rb = mdl->Rblk[blk] + 3 * (lane < 24 ? row : 0);
      const double d0 = __shfl_sync(FULL, du, 3 * blk), d1 = __shfl_sync(FULL, du, 3 * blk + 1), d2 = __shfl_sync(FULL, du, 3 * blk + 2);
      if (lane < 24) rd = fma(Rb[0], d0, fma(Rb[1], d1, Rb[2] * d2)); else if (lane < NU) rd = mdl->Rarm[lane - 24] * du; }
    value += 0.5 * warp_sum(lane < NX ? dx * qd + du * rd : 0.0);
    if (lane < NX) { qw->qf[lane] = qd; qw->rf[lane] = rd; }
    __syncwarp();
  }
  // end-effector soft constraint (quadratic penalty, Gauss-Newton)
  {
    const double mup = terminal ? tn->mu_final_ee_pos : tn->mu_ee_pos, muo = terminal ? tn->mu_final_ee_ori : tn->mu_ee_ori;
    double v = 0.0; for (int r = 0; r < 6; ++r) v += 0.5 * (r < 3 ? mup : muo) * cw->e[r] * cw->e[r]; value += v;
    {
      for (int e = lane; e < 144; e += 32) { const int i = e / 12, j = e % 12; double s = 0.0; for (int r = 0; r < 6; ++r) s += (r < 3 ? mup : muo) * cw->Je[r * 12 + i] * cw->Je[r * 12 + j]; qw->E[e] = s; }
      if (lane < 12) { double s = 0.0; for (int r = 0; r < 6; ++r) s += (r < 3 ? mup : muo) * cw->e[r] * cw->Je[r * 12 + lane]; qw->qf[ee_col(lane)] += s; }
      __syncwarp();
    }
  }
  if (!terminal) {
    // arm joint position (state 24:30) and velocity (input 24:30) soft box, relaxed log barrier
    double bv = 0.0;
    if (lane < 12) {
      const int i = lane % 6; const bool pos = lane < 6; const double val = pos ? ws->x[24 + i] : ws->u[24 + i];
      const double lo = pos ? mdl->arm_pos_lower[i] : mdl->arm_vel_lower[i], hi = pos ? mdl->arm_pos_upper[i] : mdl->arm_vel_upper[i];
      const double mu = pos ? mdl->pos_limit_mu : mdl->vel_limit_mu, de = pos ? mdl->pos_limit_delta : mdl->vel_limit_delta;
      double a0, a1, a2, b0, b1, b2; relaxed_barrier(mu, de, val - lo, a0, a1, a2); relaxed_barrier(mu, de, hi - val, b0, b1, b2);
      bv = a0 + b0;
      if (pos) { qw->qf[24 + i] += a1 - b1; qw->qdiag[24 + i] += a2 + b2; } else { qw->rf[24 + i] += a1 - b1; qw->rdiag[24 + i] += a2 + b2; }
    }
    // friction cone soft constraints of the stance feet; hessianDiagonalShift acts on every state and input diagonal [upstream FrictionConeConstraint]
    double shift = 0.0;
    if (lane >= 12 && lane < 16) {
      const int i = lane - 12;
      if ((flagmask >> i) & 1) {
        const double Fx = ws->u[3 * i], Fy = ws->u[3 * i + 1], Fz = ws->u[3 * i + 2]; const double n2 = Fx * Fx + Fy * Fy + mdl->friction_reg, n = sqrt(n2), in = 1.0 / n, in32 = in * in * in;
        const double h = tn->friction_mu * Fz - n; double p0, p1, p2; relaxed_barrier(mdl->friction_barrier_mu, mdl->friction_barrier_delta, h, p0, p1, p2); bv = p0;
        {
          const double g[3] = {-Fx * in, -Fy * in, tn->friction_mu}; const double H2[9] = {-(Fy * Fy + mdl->friction_reg) * in32, Fx * Fy * in32, 0, Fx * Fy * in32, -(Fx * Fx + mdl->friction_reg) * in32, 0, 0, 0, 0};
          for (int a = 0; a < 3; ++a) { qw->rf[3 * i + a] += p1 * g[a]; for (int b = 0; b < 3; ++b) qw->fric[i * 9 + 3 * a + b] = p2 * g[a] * g[b] + p1 * H2[3 * a + b]; }
          shift = -p1 * mdl->friction_hess_shift;
        }
      }
    }
    value += warp_sum(bv);
    shift = warp_sum(shift); __syncwarp(); if (lane < NX) { qw->qdiag[lane] += shift; qw->rdiag[lane] += shift; }
  }
  __syncwarp();
  return value;
}

}  // namespace qmb
