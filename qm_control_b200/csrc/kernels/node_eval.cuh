// One THREAD = one node: scalar restatement of the per-node evaluation of the MPC path - forward kinematics of the five serial chains, the SRBD flow map of
//   PinocchioCentroidalDynamicsAD behind QMDynamicsAD (qm_interface/src/dynamics/QMDynamicsAD.cpp:22-33) with its analytic Jacobian blocks,
//   the foot-velocity rows of ZeroVelocity / NormalVelocity (QMInterface.cpp:116-131, NormalVelocityConstraintCppAd.cpp:37-66),
//   the end-effector error of EndEffectorConstraint (src/constraint/EndEffectorConstraint.cpp:36-113) with its Jacobian,
//   the intermediate / terminal cost value (LeggedRobotQuadraticTrackingCost.h:34-40, QMInterface.cpp:147-259, 344-358).
// Why a second formulation next to the warp-per-node one of mpc_device.cuh: the kinematics are chains of 3x3 products with at most five bodies per tree level,
// so a warp spends 3..9 active lanes on them; one thread per node keeps every lane busy (32 nodes per warp), the chain state lives in registers, and nothing
// needs shared memory.  K2a (mpc_flow_kernel) and K4 (mpc_linesearch_kernel) run on it; the matrix work of K2 stays warp-per-node.
// Host + device: tests/nodeeval_host.cpp compiles this header with g++ and checks every output against the oracle on the CPU.
// Assumes what the warp formulation assumes (leg i = joints foot_leg[i]..+2, arm = joints 12..17) plus: every chain is serial from the base
// (parent[j] is the base or body j) - checked on the host when the model is built (qm_config.cpp).
#pragma once
#include "mpc_scalar.cuh"

namespace qmb {
namespace ne {

// ---- the record K2a hands to K2b per node, in the order the flow kernel produces it (one flush of its transposition tile per block) ----
struct FootBlk { double d[3], pf[3], Jl[9], JxF[9], e[3], C[3][12]; };   // foot - com, foot position, leg Jacobian Jl[3 * j + a], (J_j x F_i) / m, foot velocity residual and its rows on the 12 support columns
struct FlowBlk {                      // rows 3:12 of df/dx are [d hdot_ang; d pdot; d thetadot] and only these blocks (+ the feet's JxF, d) are non-trivial (mpc_device.cuh point_eval)
  double f[12];                       // rows 0:12 of the flow map (rows 12:30 are the joint-velocity inputs)
  double Mpc[9], Mtw[9];              // d pdot / d h_ang ; d thetadot / d h_ang
  double hth[3][3], vp[3][3], vt[3][3];   // columns theta_k of hdot_ang, pdot, thetadot  ([k][a])
};
struct EeRec { double Je[6 * 12]; double e[6]; };
struct Foot2Blk { double d[3], JxF[9]; };                                // second RK2 stage: what the flow Jacobian needs from a foot
struct NodeRec { FootBlk foot[4]; FlowBlk s1; EeRec ee; Foot2Blk foot2[4]; FlowBlk s2; };
constexpr int FOOT_DBL = 63, FLOW_DBL = 57, EE_DBL = 78, FOOT2_DBL = 12;
constexpr int NODE_REC_DBL = 4 * FOOT_DBL + FLOW_DBL + EE_DBL + 4 * FOOT2_DBL + FLOW_DBL;   // 492
static_assert(sizeof(FootBlk) == FOOT_DBL * 8 && sizeof(FlowBlk) == FLOW_DBL * 8 && sizeof(EeRec) == EE_DBL * 8 && sizeof(Foot2Blk) == FOOT2_DBL * 8 && sizeof(NodeRec) == NODE_REC_DBL * 8, "the record is a flat array of doubles");
static_assert(sizeof(NodeRec) % 16 == 0, "records stay 16-byte aligned");

// base-frame quantities shared by the pieces below
struct BaseKin { double tr[6], R0[9], T[9], Tinv[9], W[9], c[3], rcom[3], omega[3], thd[3], dom[3][3]; };
// sums over the feet that the flow map needs
struct FlowAcc { double fsum[3], hang[3], hth[3][3]; };

// a[3 * s + c] for a block s in 0..3 known only at run time (a foot's forces, a leg's joints): a chain of selects with static register indices.  Indexing the
// thread's array with s directly would place the whole array in local memory.
QMB_HD double pick3(const double* a, int s, int c) { return s == 0 ? a[c] : (s == 1 ? a[3 + c] : (s == 2 ? a[6 + c] : a[9 + c])); }

// The SRBD constants the flow map and the cost use (base_eval, foot_eval, flow_finish, cost_value take the robot's as `sc`): the model's when sc is null.
QMB_HD const SrbdConst& srbd_or_nominal(const DevModel* __restrict__ mdl, const SrbdConst* sc) { return sc ? *sc : *srbd_of(mdl, nullptr, 0); }

// one serial chain from the base: joints first .. first + NJC - 1 at angles q[0 .. NJC - 1]; returns the last body's frame, every joint's origin and axis (world)
template <int NJC>
QMB_HD void chain_fk(const DevModel* __restrict__ mdl, const double* R0, const double* p0, const double* q, int first, double* Rl, double* pl, double (*org)[3], double (*axs)[3]) {
  double Rp[9], pp[3];
#pragma unroll
  for (int i = 0; i < 9; ++i) Rp[i] = R0[i];
  pp[0] = p0[0]; pp[1] = p0[1]; pp[2] = p0[2];
#pragma unroll
  for (int jj = 0; jj < NJC; ++jj) {
    const int j = first + jj; double s, c; sincos(q[jj], &s, &c);
    const int ax = mdl->axis[j]; const double* Rj = mdl->Rj[j]; double Rlq[9];
#pragma unroll
    for (int i = 0; i < 3; ++i) { const double r0 = Rj[3 * i], r1 = Rj[3 * i + 1], r2 = Rj[3 * i + 2];   // Rj * Rq(axis, q): Rq mixes the two columns after the axis
      if (ax == 0) { Rlq[3 * i] = r0; Rlq[3 * i + 1] = c * r1 + s * r2; Rlq[3 * i + 2] = -s * r1 + c * r2; }
      else if (ax == 1) { Rlq[3 * i] = c * r0 - s * r2; Rlq[3 * i + 1] = r1; Rlq[3 * i + 2] = s * r0 + c * r2; }
      else { Rlq[3 * i] = c * r0 + s * r1; Rlq[3 * i + 1] = -s * r0 + c * r1; Rlq[3 * i + 2] = r2; } }
    double Rw[9], pw[3]; matmul3(Rp, Rlq, Rw); const double pj[3] = {mdl->pj[j][0], mdl->pj[j][1], mdl->pj[j][2]}; matvec3(Rp, pj, pw);
    pw[0] += pp[0]; pw[1] += pp[1]; pw[2] += pp[2];
    org[jj][0] = pw[0]; org[jj][1] = pw[1]; org[jj][2] = pw[2];
    axs[jj][0] = ax == 0 ? Rw[0] : (ax == 1 ? Rw[1] : Rw[2]); axs[jj][1] = ax == 0 ? Rw[3] : (ax == 1 ? Rw[4] : Rw[5]); axs[jj][2] = ax == 0 ? Rw[6] : (ax == 1 ? Rw[7] : Rw[8]);
#pragma unroll
    for (int i = 0; i < 9; ++i) Rp[i] = Rw[i];
    pp[0] = pw[0]; pp[1] = pw[1]; pp[2] = pw[2];
  }
#pragma unroll
  for (int i = 0; i < 9; ++i) Rl[i] = Rp[i];
  pl[0] = pp[0]; pl[1] = pp[1]; pl[2] = pp[2];
}

template <bool JAC>
QMB_HD void base_eval(const DevModel* __restrict__ mdl, const double* x, BaseKin& bk, const SrbdConst* sc = nullptr) {
  sincos(x[9], &bk.tr[0], &bk.tr[1]); sincos(x[10], &bk.tr[2], &bk.tr[3]); sincos(x[11], &bk.tr[4], &bk.tr[5]);
  rot_zyx_sc(bk.tr, bk.R0); euler_rate_map_sc(bk.tr, bk.T); inv3(bk.T, bk.Tinv);
  const SrbdConst& S = srbd_or_nominal(mdl, sc); const double m = S.m; const double* R = bk.R0; const double* Ii = S.I_nom_inv; const double* ha = x + 3;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int jj = 0; jj < 3; ++jj) { double acc = 0.0;
#pragma unroll
      for (int bq = 0; bq < 3; ++bq) { const double rib = R[3 * i] * Ii[bq] + R[3 * i + 1] * Ii[3 + bq] + R[3 * i + 2] * Ii[6 + bq]; acc = fma(rib, R[3 * jj + bq], acc); }
      bk.W[3 * i + jj] = m * acc; }
  matvec3(R, S.c_nom, bk.c);
  for (int a = 0; a < 3; ++a) bk.rcom[a] = x[6 + a] - bk.c[a];
  matvec3(bk.W, ha, bk.omega); matvec3(bk.Tinv, bk.omega, bk.thd);
  if (JAC) { for (int k = 0; k < 3; ++k) { const double Tk[3] = {bk.T[k], bk.T[3 + k], bk.T[6 + k]}; double t1[3], t2[3], t3[3];
      cross3(Tk, bk.omega, t1); cross3(Tk, ha, t2); matvec3(bk.W, t2, t3); for (int a = 0; a < 3; ++a) bk.dom[k][a] = t1[a] - t3[a]; } }   // d omega / d theta_k
}

QMB_HD void flow_acc_init(FlowAcc& acc) { for (int a = 0; a < 3; ++a) { acc.fsum[a] = 0.0; acc.hang[a] = 0.0; for (int k = 0; k < 3; ++k) acc.hth[k][a] = 0.0; } }

// One foot (contact order i; its leg's joints foot_leg[i] .. + 2): chain kinematics, foot - com, leg Jacobian columns Jl[3 * j + a] (+ joint axes al, same layout),
// the foot's share of the flow map (accumulated in acc) and, with JAC, (J_j x F_i) / m.  Jl / al / pf / JxF may be null.
template <bool JAC>
QMB_HD void foot_eval(const DevModel* __restrict__ mdl, const double* x, const double* u, const BaseKin& bk, int i, FlowAcc& acc, double* d, double* pf, double* Jl, double* al, double* JxF,
                      const SrbdConst* sc = nullptr) {
  const int first = mdl->foot_leg[i]; double Rl[9], pl[3], org[3][3], axs[3][3];
  const double q[3] = {pick3(x + 12, first / 3, 0), pick3(x + 12, first / 3, 1), pick3(x + 12, first / 3, 2)};
  chain_fk<3>(mdl, bk.R0, x + 6, q, first, Rl, pl, org, axs);
  double pw[3]; matvec3(Rl, mdl->foot_p[i], pw);
  for (int a = 0; a < 3; ++a) { pw[a] += pl[a]; d[a] = pw[a] - bk.rcom[a]; if (pf) pf[a] = pw[a]; }
  const double F[3] = {pick3(u, i, 0), pick3(u, i, 1), pick3(u, i, 2)}; const double im = 1.0 / srbd_or_nominal(mdl, sc).m;
  for (int a = 0; a < 3; ++a) acc.fsum[a] += F[a];
  cross3_add(d, F, acc.hang);
  for (int j = 0; j < 3; ++j) { const double r[3] = {pw[0] - org[j][0], pw[1] - org[j][1], pw[2] - org[j][2]}; double col[3]; cross3(axs[j], r, col);
    if (Jl) for (int a = 0; a < 3; ++a) Jl[3 * j + a] = col[a];
    if (al) for (int a = 0; a < 3; ++a) al[3 * j + a] = axs[j][a];
    if (JAC) { double jf[3]; cross3(col, F, jf); for (int a = 0; a < 3; ++a) JxF[3 * j + a] = jf[a] * im; } }
  if (JAC) for (int k = 0; k < 3; ++k) { const double Tk[3] = {bk.T[k], bk.T[3 + k], bk.T[6 + k]}; double t[3]; cross3(Tk, d, t); cross3_add(t, F, acc.hth[k]); }
}

// rows 0:12 of the flow map from the accumulated foot terms (+ the base-frame Jacobian blocks)
template <bool JAC>
QMB_HD void flow_finish(const DevModel* __restrict__ mdl, const double* x, const BaseKin& bk, const FlowAcc& acc, double* f, FlowBlk* fb, const SrbdConst* sc = nullptr) {
  const double im = 1.0 / srbd_or_nominal(mdl, sc).m; const double* om = bk.omega; const double* c = bk.c;
  for (int a = 0; a < 3; ++a) { f[a] = acc.fsum[a] * im + (a == 2 ? -9.81 : 0.0); f[3 + a] = acc.hang[a] * im; f[9 + a] = bk.thd[a]; }
  { double oc[3]; cross3(om, c, oc); for (int a = 0; a < 3; ++a) f[6 + a] = x[a] + oc[a]; }
  if (JAC) {
    const double* tr = bk.tr; const double sz = tr[0], cz = tr[1], sy = tr[2], cy = tr[3]; const double th1 = bk.thd[1], th2 = bk.thd[2];
    for (int k = 0; k < 3; ++k) {
      double dT[3];
      if (k == 0) { dT[0] = -cz * th1 - cy * sz * th2; dT[1] = -sz * th1 + cy * cz * th2; dT[2] = 0.0; }
      else if (k == 1) { dT[0] = -sy * cz * th2; dT[1] = -sy * sz * th2; dT[2] = -cy * th2; }
      else { dT[0] = 0.0; dT[1] = 0.0; dT[2] = 0.0; }
      const double Tk[3] = {bk.T[k], bk.T[3 + k], bk.T[6 + k]}; const double* domk = bk.dom[k];
      double tc[3], vpk[3]; cross3(Tk, c, tc); cross3(domk, c, vpk); cross3_add(om, tc, vpk);           // d(omega x c)/d theta_k
      for (int a = 0; a < 3; ++a) { fb->vp[k][a] = vpk[a]; fb->hth[k][a] = acc.hth[k][a] * im; }
      const double tmp[3] = {domk[0] - dT[0], domk[1] - dT[1], domk[2] - dT[2]}; matvec3(bk.Tinv, tmp, fb->vt[k]);
    }
    const double* W = bk.W;
    for (int i = 0; i < 3; ++i) for (int jj = 0; jj < 3; ++jj) {   // Mpc = -S(c) W ; Mtw = Tinv W
      const double s0 = (i == 0) ? 0.0 : (i == 1 ? c[2] : -c[1]), s1 = (i == 0) ? -c[2] : (i == 1 ? 0.0 : c[0]), s2 = (i == 0) ? c[1] : (i == 1 ? -c[0] : 0.0);
      fb->Mpc[3 * i + jj] = -(s0 * W[jj] + s1 * W[3 + jj] + s2 * W[6 + jj]);
      fb->Mtw[3 * i + jj] = bk.Tinv[3 * i] * W[jj] + bk.Tinv[3 * i + 1] * W[3 + jj] + bk.Tinv[3 * i + 2] * W[6 + jj]; }
  }
}

// foot velocity v_i = h_lin + omega x d_i + sum_j Jl_j qd_j (+ its state Jacobian on the 12 support columns), foot_velocity<> of mpc_device.cuh for one foot
template <bool JAC>
QMB_HD void foot_velocity_1(const DevModel* __restrict__ mdl, const double* x, const double* u, const BaseKin& bk, int i, const double* d, const double* Jli, const double* ali, double* e, double (*C)[12]) {
  const int leg = mdl->foot_leg[i] / 3; const double* om = bk.omega; const double qd[3] = {pick3(u + 12, leg, 0), pick3(u + 12, leg, 1), pick3(u + 12, leg, 2)};
  double w[3] = {0, 0, 0}; for (int j = 0; j < 3; ++j) for (int a = 0; a < 3; ++a) w[a] += Jli[3 * j + a] * qd[j];
  double v[3]; cross3(om, d, v); for (int a = 0; a < 3; ++a) e[a] = v[a] + x[a] + w[a];
  if (JAC) {
    for (int a = 0; a < 3; ++a) for (int cc = 0; cc < 12; ++cc) C[a][cc] = (cc == a) ? 1.0 : 0.0;
    const double Sd[9] = {0, -d[2], d[1], d[2], 0, -d[0], -d[1], d[0], 0}; double SW[9]; matmul3(Sd, bk.W, SW);
    for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) C[a][3 + b] = -SW[3 * a + b];
    for (int k = 0; k < 3; ++k) { const double Tk[3] = {bk.T[k], bk.T[3 + k], bk.T[6 + k]}; double t[3], col[3]; cross3(bk.dom[k], d, col); cross3(Tk, d, t); cross3_add(om, t, col); cross3_add(Tk, w, col); for (int a = 0; a < 3; ++a) C[a][6 + k] = col[a]; }
    for (int j = 0; j < 3; ++j) {
      const double* Jj = Jli + 3 * j; const double* aj = ali + 3 * j; double above[3] = {0, 0, 0}, below[3] = {0, 0, 0};
      for (int l = j + 1; l < 3; ++l) for (int a = 0; a < 3; ++a) above[a] += Jli[3 * l + a] * qd[l];
      for (int l = 0; l <= j; ++l) for (int a = 0; a < 3; ++a) below[a] += ali[3 * l + a] * qd[l];
      double col[3]; cross3(om, Jj, col); cross3_add(aj, above, col); cross3_add(below, Jj, col);
      for (int a = 0; a < 3; ++a) C[a][9 + j] = col[a];
    }
  }
}

// Target trajectory references at time t (target_reference of mpc_device.cuh): the two knots and the interpolation weight of the state reference
// (xnom_i = a * l[i] + (1 - a) * rr[i]) and the end-effector pose reference (EndEffectorConstraint::interpolateEndEffectorPose, Eigen slerp semantics)
struct TargetSeg { const double* l; const double* rr; double a; };
QMB_HD TargetSeg target_segment(const double* tt, const double* ts /*[K][37]*/, int nk, double t) {
  int idx; double a; time_segment(tt, nk, t, idx, a); TargetSeg sg; sg.l = ts + (size_t)idx * 37; sg.rr = ts + (size_t)((nk > 1) ? idx + 1 : idx) * 37; sg.a = (nk <= 1) ? 1.0 : a; return sg;
}
// The slerp's sines take angles in [0, pi/2]; Sin lets a caller that must stay off the stack pass a sine without the huge-argument slow path
// (metrics_api.cuh's BoundedSin).
struct StdSin { QMB_HD double operator()(double x) const { return sin(x); } };
template <class Sin = StdSin>
QMB_HD void target_pose(const TargetSeg& sg, int nk, double* pref, double* qref, Sin sine = Sin()) {
  const double* l = sg.l; const double* rr = sg.rr; const double a = sg.a;
  for (int i = 0; i < 3; ++i) pref[i] = a * l[30 + i] + (1.0 - a) * rr[30 + i];
  if (nk > 1) {
    const double* ql = l + 33; const double* qr = rr + 33; const double tq = 1.0 - a; double d = 0.0; for (int i = 0; i < 4; ++i) d += ql[i] * qr[i];
    const double ad = fabs(d); double s0, s1;
    if (ad >= 1.0 - 2.220446049250313e-16) { s0 = 1.0 - tq; s1 = tq; } else { const double th = acos(ad), st = sine(th); const double ist = 1.0 / st; s0 = sine((1.0 - tq) * th) * ist; s1 = sine(tq * th) * ist; }
    if (d < 0.0) s1 = -s1;
    for (int i = 0; i < 4; ++i) qref[i] = s0 * ql[i] + s1 * qr[i];
  } else { for (int i = 0; i < 4; ++i) qref[i] = l[33 + i]; }
}

// End-effector error e = [p_ee - p_ref; quaternionDistance(q_ee, q_ref)] (+ Jacobian on the 12 columns p, theta, arm): ee_error<> of mpc_device.cuh
template <bool JAC>
QMB_HD void ee_eval(const DevModel* __restrict__ mdl, const double* x, const BaseKin& bk, const double* pref, const double* qref, double* e, double* Je /*[6][12]*/) {
  double Rl[9], pl[3], org[6][3], axs[6][3];
  chain_fk<6>(mdl, bk.R0, x + 6, x + 24, 12, Rl, pl, org, axs);
  double R[9]; matmul3(Rl, mdl->ee_R, R); double pw[3]; matvec3(Rl, mdl->ee_p, pw);
  for (int a = 0; a < 3; ++a) { pw[a] += pl[a]; e[a] = pw[a] - pref[a]; }
  double q[4]; const double tr = R[0] + R[4] + R[8];   // rotation -> quaternion (w,x,y,z); sign free (quadratic penalty), same q used for e and its Jacobian
  if (tr > 0.0) { const double s = sqrt(tr + 1.0) * 2.0, is = 1.0 / s; q[0] = 0.25 * s; q[1] = (R[7] - R[5]) * is; q[2] = (R[2] - R[6]) * is; q[3] = (R[3] - R[1]) * is; }
  else if (R[0] > R[4] && R[0] > R[8]) { const double s = sqrt(1.0 + R[0] - R[4] - R[8]) * 2.0, is = 1.0 / s; q[0] = (R[7] - R[5]) * is; q[1] = 0.25 * s; q[2] = (R[1] + R[3]) * is; q[3] = (R[2] + R[6]) * is; }
  else if (R[4] > R[8]) { const double s = sqrt(1.0 + R[4] - R[0] - R[8]) * 2.0, is = 1.0 / s; q[0] = (R[2] - R[6]) * is; q[1] = (R[1] + R[3]) * is; q[2] = 0.25 * s; q[3] = (R[5] + R[7]) * is; }
  else { const double s = sqrt(1.0 + R[8] - R[0] - R[4]) * 2.0, is = 1.0 / s; q[0] = (R[3] - R[1]) * is; q[1] = (R[2] + R[6]) * is; q[2] = (R[5] + R[7]) * is; q[3] = 0.25 * s; }
  const double* rv = qref; const double rw = qref[3]; const double* qv = q + 1; double cr[3]; cross3(qv, rv, cr);
  for (int a = 0; a < 3; ++a) e[3 + a] = q[0] * rv[a] - rw * qv[a] + cr[a];   // ocs2 quaternionDistance(q, qRef) [upstream]
  if (JAC) {
    for (int cidx = 0; cidx < 12; ++cidx) {   // column: angular direction n and linear velocity of the EE point for a unit rate of the coordinate
      double n[3] = {0, 0, 0}, lin[3] = {0, 0, 0};
      if (cidx < 3) lin[cidx] = 1.0;
      else if (cidx < 6) { const int k = cidx - 3; n[0] = bk.T[k]; n[1] = bk.T[3 + k]; n[2] = bk.T[6 + k]; const double r[3] = {pw[0] - x[6], pw[1] - x[7], pw[2] - x[8]}; cross3(n, r, lin); }
      else { const int j = cidx - 6; n[0] = axs[j][0]; n[1] = axs[j][1]; n[2] = axs[j][2]; const double r[3] = {pw[0] - org[j][0], pw[1] - org[j][1], pw[2] - org[j][2]}; cross3(n, r, lin); }
      const double dw = -0.5 * dot3(n, qv); double dv[3]; cross3(n, qv, dv); for (int a = 0; a < 3; ++a) dv[a] = 0.5 * (q[0] * n[a] + dv[a]);
      double cr2[3]; cross3(dv, rv, cr2);
      for (int a = 0; a < 3; ++a) { Je[a * 12 + cidx] = lin[a]; Je[(3 + a) * 12 + cidx] = dw * rv[a] - rw * dv[a] + cr2[a]; }
    }
  }
}

// Intermediate (or terminal) cost VALUE at (x, u) given the end-effector error (stage_cost<false> of mpc_device.cuh; unscaled by dt).  tn: the robot's tuning row
// (tuning_of), NULL for the model's values.
QMB_HD double cost_value(const DevModel* __restrict__ mdl, const double* x, const double* u, const TargetSeg& sg, const double* ee, int flagmask, bool terminal, const SrbdConst* sc = nullptr,
                         const Tuning* tn = nullptr) {
  if (!tn) tn = tuning_of(mdl, nullptr, 0);
  double value = 0.0;
  if (!terminal) {
    int nst = 0; for (int i = 0; i < 4; ++i) nst += (flagmask >> i) & 1;
    // deviations from the references element by element where they are used: whole dx[30] / du[30] arrays would not fit in registers next to (x, u)
    auto dx = [&](int i) { return x[i] - (sg.a * sg.l[i] + (1.0 - sg.a) * sg.rr[i]); };
    const double un = srbd_or_nominal(mdl, sc).m * 9.81 / nst;
    double acc = 0.0;
    if (mdl->q_is_diag) { for (int i = 0; i < NX; ++i) { const double d = dx(i); acc = fma(d * mdl->Qdiag[i], d, acc); } }
    else { for (int i = 0; i < NX; ++i) { double qd = 0.0; for (int j = 0; j < NX; ++j) qd = fma(mdl->Q[i * NX + j], dx(j), qd); acc = fma(dx(i), qd, acc); } }
#pragma unroll
    for (int blk = 0; blk < 8; ++blk) { const double* Rb = mdl->Rblk[blk];   // blocks 0..3: the feet's forces (weight compensation on the z force of a stance foot)
      const double d3[3] = {u[3 * blk], u[3 * blk + 1], u[3 * blk + 2] - ((blk < 4 && ((flagmask >> blk) & 1)) ? un : 0.0)};
      for (int r = 0; r < 3; ++r) acc = fma(d3[r], fma(Rb[3 * r], d3[0], fma(Rb[3 * r + 1], d3[1], Rb[3 * r + 2] * d3[2])), acc); }
    for (int i = 0; i < 6; ++i) acc = fma(u[24 + i] * mdl->Rarm[i], u[24 + i], acc);
    value += 0.5 * acc;
  }
  { const double mup = terminal ? tn->mu_final_ee_pos : tn->mu_ee_pos, muo = terminal ? tn->mu_final_ee_ori : tn->mu_ee_ori;
    double v = 0.0; for (int r = 0; r < 6; ++r) v += 0.5 * (r < 3 ? mup : muo) * ee[r] * ee[r]; value += v; }
  if (!terminal) {
    // relaxed log barriers: sum_i -mu log(h_i) = -mu log(prod_i h_i) over the entries in the logarithmic branch (24 + 4 fp64 logarithms become 3); the
    // quadratic extension (h <= delta) is summed as it is
    double bv = 0.0;
    for (int grp = 0; grp < 2; ++grp) {   // arm joint position (state 24:30) and velocity (input 24:30) soft box
      const bool pos = grp == 0; const double mu = pos ? mdl->pos_limit_mu : mdl->vel_limit_mu, de = pos ? mdl->pos_limit_delta : mdl->vel_limit_delta; double prod = 1.0;
      for (int i = 0; i < 6; ++i) { const double val = pos ? x[24 + i] : u[24 + i]; const double lo = pos ? mdl->arm_pos_lower[i] : mdl->arm_vel_lower[i], hi = pos ? mdl->arm_pos_upper[i] : mdl->arm_vel_upper[i];
        const double h2[2] = {val - lo, hi - val};
        for (int sd = 0; sd < 2; ++sd) { const double h = h2[sd]; if (h > de) prod *= h; else { const double tq = (h - 2.0 * de) / de; bv += mu * (-log(de) + 0.5 * tq * tq - 0.5); } } }
      bv -= mu * log(prod); }
    { double prod = 1.0; const double mu = mdl->friction_barrier_mu, de = mdl->friction_barrier_delta;   // friction cone soft constraints of the stance feet
      for (int i = 0; i < 4; ++i) if ((flagmask >> i) & 1) { const double Fx = u[3 * i], Fy = u[3 * i + 1], Fz = u[3 * i + 2]; const double h = tn->friction_mu * Fz - sqrt(Fx * Fx + Fy * Fy + mdl->friction_reg);
        if (h > de) prod *= h; else { const double tq = (h - 2.0 * de) / de; bv += mu * (-log(de) + 0.5 * tq * tq - 0.5); } }
      bv -= mu * log(prod); }
    value += bv;
  }
  return value;
}

// foot i's terms of equality_ss added to es (feet in contact order, so a caller can add them foot by foot without keeping every foot's e and pf)
template <class MT>
QMB_HD void equality_add(const DevModel* __restrict__ mdl, const double* u, const double* e, const double* pf, int flagmask, const double* ev, const MT* modes, int ne, double t, int i, double& es, bool& ok) {
  if ((flagmask >> i) & 1) { for (int a = 0; a < 3; ++a) es += e[a] * e[a]; }
  else { double zp, zv; ok &= swing_reference(mdl, ev, modes, ne, i, t, zp, zv); double ez = e[2] - zv; if (mdl->position_error_gain != 0.0) ez += mdl->position_error_gain * (pf[2] - zp);
    es += ez * ez; for (int a = 0; a < 3; ++a) { const double F = pick3(u, i, a); es += F * F; } }
}
// squared equality-constraint residual of a node (ZeroVelocity on stance feet; ZeroForce + NormalVelocity on swing feet); swing_ok reports an unenclosed swing phase
template <class MT>
QMB_HD double equality_ss(const DevModel* __restrict__ mdl, const double* u, const double (*e)[3], const double (*pf)[3], int flagmask, const double* ev, const MT* modes, int ne, double t, bool* swing_ok) {
  double es = 0.0; bool ok = true;
  for (int i = 0; i < 4; ++i) equality_add(mdl, u, e[i], pf[i], flagmask, ev, modes, ne, t, i, es, ok);
  if (swing_ok) *swing_ok = ok;
  return es;
}

}  // namespace ne
}  // namespace qmb
