// Scalar helpers of the MPC path shared by the warp-per-node kernels (mpc_device.cuh) and the thread-per-node evaluator (node_eval.cuh); host + device so
// that the evaluator can be checked on the CPU against the oracle (tests/nodeeval_host.cpp).
#pragma once
#include "dev_common.cuh"

namespace qmb {

constexpr int MU = 18;      // max projected input dimension (30 - 12 equality rows in stance)
constexpr int MAXDEP = 16;  // max dependent inputs (fly: 4 x (3 forces + 1 joint))
constexpr double WEAK_EPS = 1e-6;   // ocs2 numeric_traits::weakEpsilon: interval start/end shift at event nodes [upstream]
// leg (joint order LF, LH, RF, RH) → foot (contact order) map packed two bits per leg: loaded once per kernel, every lookup is then pure ALU
// (the map sits in front of shared-memory indexing in the flat stage-record sweeps, so a global load per lookup is a dependent chain)
QMB_HD int pack_leg_foot(const DevModel* __restrict__ mdl) { return mdl->leg_foot[0] | (mdl->leg_foot[1] << 2) | (mdl->leg_foot[2] << 4) | (mdl->leg_foot[3] << 6); }
QMB_HD int foot_of_leg_joint(int lfp, int j) { return (lfp >> (2 * (j / 3))) & 3; }
// ---- reference signals -------------------------------------------------------------------------------
// ocs2::lookup::findIndexInTimeArray (std::lower_bound)
QMB_HD int lower_bound_idx(const double* a, int n, double t) { int lo = 0, hi = n; while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] < t) lo = mid + 1; else hi = mid; } return lo; }
template <class MT> QMB_HD int mode_at_time(const double* ev, const MT* modes, int ne, double t) { return modes[lower_bound_idx(ev, ne, t)]; }
// ocs2::LinearInterpolation::timeSegment
QMB_HD void time_segment(const double* times, int n, double t, int& index, double& alpha) {
  if (n <= 1) { index = 0; alpha = 1.0; return; }
  const int part = lower_bound_idx(times, n, t); int idx = (part != 0 || t != times[0]) ? part - 1 : 0; const int last = n - 1;
  if (idx >= 0) {
    if (idx < last) { const double len = times[idx + 1] - times[idx], till = times[idx + 1] - t; index = idx; alpha = (len > 2.0 * 2.220446049250313e-16) ? till / len : (till > 0.5 * len ? 1.0 : 0.0); return; }
    index = (last - 1 > 0) ? last - 1 : 0; alpha = 0.0; return;
  }
  index = 0; alpha = 1.0;
}
// SwingTrajectoryPlanner::getZvelocityConstraint / getZpositionConstraint [upstream]: status=false when the swing phase is not enclosed
template <class MT> QMB_HD bool swing_reference(const DevModel* __restrict__ mdl, const double* ev, const MT* modes, int ne, int leg, double t, double& zp, double& zv) {
  const int np = ne + 1; const int p = lower_bound_idx(ev, ne, t); zp = 0.0; zv = 0.0;
  if (contact_flag(modes[p], leg)) return true;
  int start = -1; for (int ip = p - 1; ip >= 0; --ip) if (contact_flag(modes[ip], leg)) { start = ip; break; }
  int fin = np - 1; for (int ip = p + 1; ip < np; ++ip) if (contact_flag(modes[ip], leg)) { fin = ip - 1; break; }
  if (start < 0 || fin >= np - 1) return false;
  const double t0 = ev[start], t1 = ev[fin]; const double scaling = fmin(1.0, (t1 - t0) / mdl->swing_time_scale); const double tm = 0.5 * (t0 + t1), zm = scaling * mdl->swing_height;
  double ta, pa, va, tb, pb, vb;
  if (t < tm) { ta = t0; pa = 0.0; va = scaling * mdl->lift_off_velocity; tb = tm; pb = zm; vb = 0.0; } else { ta = tm; pa = zm; va = 0.0; tb = t1; pb = 0.0; vb = scaling * mdl->touch_down_velocity; }
  const double dtt = tb - ta, dp = pb - pa, dv = vb - va; const double c0 = pa, c1 = va * dtt, c2 = -(3.0 * va + dv) * dtt + 3.0 * dp, c3 = (2.0 * va + dv) * dtt - 2.0 * dp; const double idt = 1.0 / dtt, tn = (t - ta) * idt;
  zp = ((c3 * tn + c2) * tn + c1) * tn + c0; zv = ((3.0 * c3 * tn + 2.0 * c2) * tn + c1) * idt; return true;
}
// ocs2 RelaxedBarrierPenalty [upstream]
// (one logarithm of the selected argument: lanes of a warp that fall on different sides of delta do not evaluate it twice)
QMB_HD void relaxed_barrier(double mu, double delta, double h, double& p0, double& p1, double& p2) {
  const bool inside = h > delta; const double lg = log(inside ? h : delta);
  if (inside) { const double ih = 1.0 / h; p0 = -mu * lg; p1 = -mu * ih; p2 = mu * ih * ih; }
  else { const double t = (h - 2.0 * delta) / delta; p0 = mu * (-lg + 0.5 * t * t - 0.5); p1 = mu * (h - 2.0 * delta) / (delta * delta); p2 = mu / (delta * delta); }
}

QMB_HD int ee_pos(int c) { return (c >= 6 && c < 12) ? c - 6 : (c >= 24 ? c - 18 : -1); }
QMB_HD int ee_col(int i) { return i < 6 ? 6 + i : 18 + i; }   // 12 state columns the EE pose depends on: p(6:9), theta(9:12), arm(24:30)
// state column of support position `pos` (0..11) for the leg whose first joint is `first`
QMB_HD int sup_col(int pos, int first) { return pos < 6 ? pos : (pos < 9 ? pos + 3 : 12 + first + pos - 9); }

// Quadratic model of the intermediate cost (unscaled by dt) in COMPACT form: the constant weights stay in DevModel (L1/L2 resident),
// only what depends on (x,u) is stored:  Qf = Q + diag(qdiag) + scatter(E on the 12 end-effector columns),
// Rf = R + diag(rdiag) + blockdiag(fric[foot]) on the 12 force inputs.
struct QuadWs { double E[144], fric[36], qdiag[NX], rdiag[NU], qf[NX], rf[NU]; };
QMB_HD double quad_R(const DevModel* __restrict__ mdl, const QuadWs* q, int i, int j) {
  if (i >= 24 || j >= 24) return (i == j) ? mdl->Rarm[i - 24] + q->rdiag[i] : 0.0;
  const int bi = i / 3; if (bi != j / 3) return 0.0;
  double v = mdl->Rblk[bi][(i - 3 * bi) * 3 + (j - 3 * bi)]; if (i == j) v += q->rdiag[i]; if (i < 12) v += q->fric[bi * 9 + (i - 3 * bi) * 3 + (j - 3 * bi)]; return v; }
// per-leg blocks of the structured projection (K2): the velocity constraint of a foot touches 12 state columns (h, euler angles, own leg joints) and its own 3
// joint-velocity inputs, the input weight couples joint velocities only inside a leg
struct LegWs {
  double Px[3][12];     // rows of P_x of the dependent joint-velocity inputs of this leg on the support columns (stance: 3 rows; swing: pivot row only)
  double G[9];          // elimination matrix: P_x row j = sum_a G[3j+a] C[a], P_e[j] = sum_a G[3j+a] e[a] (stance: minus the inverse of the foot's joint-velocity Jacobian; swing: -1 / pivot entry at (pivot, z), zero elsewhere)
  double Pu2[2];        // swing: coupling of the pivot joint to the two free joints
  int dep[3];           // is joint j of this leg dependent
  int pivot, stance, first, free_col[3];   // projected-input column of each free joint (-1 if dependent)
};

}  // namespace qmb
