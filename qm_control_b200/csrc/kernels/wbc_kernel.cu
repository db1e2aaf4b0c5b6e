// Batched whole-body controller: one warp per robot.
//
// Path replaced (reference, CPU, one robot per call):
//   WbcBase::update            qm_wbc/src/WbcBase.cpp:118-132   (mode → contact flags)
//   WbcBase::updateMeasured    WbcBase.cpp:134-191               (Pinocchio FK/Jacobians/crba/nle)
//   WbcBase::updateDesired     WbcBase.cpp:193-226               (centroidal desired base acceleration, incl. the
//                                                                 SRBD/full-model evaluation-order quirk, SURVEY §8a-W3)
//   formulate*Task             WbcBase.cpp:228-546
//   HierarchicalWbc::update    qm_wbc/src/HierarchicalWbc.cpp:18-44, HierarchicalMpcWbc.cpp:18-34
//   HoQp (3 levels)            qm_wbc/src/HoQp.cpp:12-159        (qpOASES dense active set per level)
//   WbcBase::updateCmd         WbcBase.cpp:548-563
//
// GPU-first restatement of HoQp: the cascade "min ||A_p x - b_p||^2 + ||v_p||^2 over the optimal set of the
// higher levels, D x <= f + v" is solved directly in the 36-dim decision space with an ORTHONORMAL null-space
// basis Z (Householder complete orthogonal decomposition) instead of Eigen's fullPivLu kernel + a 92-variable
// QP with explicit slack variables: level 0's slack is eliminated analytically (v = max(0, D x - f)), the torque
// and friction rows are never materialised (they are read out of M and J), and inequalities are handled by a
// primal active set on the step.  The cascade optimum is basis independent, so the result equals the
// reference's wherever that optimum is unique (DESIGN.md §WBC).
#include "dev_common.cuh"
#include "payload.cuh"
#include "wlinalg.cuh"

namespace qmb {

constexpr int LDM = 25;   // leading dimension of 24-column matrices (odd → conflict-free column walks)
constexpr int LDZ = 37;   // leading dimension of 36-column / 36-row matrices
constexpr int LZ = 19;    // leading dimension of matrices in null-space coordinates (at most 18 columns: level 0 always has 18 independent rows)
constexpr int MAXR = 24;  // max rows of one level's equality task (22 in flight mode)
constexpr int MAXR0 = 32; // max rows of level 0's least squares: its 18 task rows + up to 14 violated inequalities (w_qrcp factors at most 32 columns)
constexpr int KG0 = 27;   // max rank of a rank-deficient level-0 pass of more than MAXR rows that forms its Gram (behind the rows); above it the pass solves on its independent rows
constexpr int LJC = 9;    // pitch of a compact foot-Jacobian row
constexpr int MAXW = 20;  // max size of the inequality working set
#ifndef QMB_WBC_WARPS
#define QMB_WBC_WARPS 8
#endif
constexpr int WBC_WARPS = QMB_WBC_WARPS;   // robots (= warps) per CTA, one CTA per SM: the kernel is latency bound, its speed is the number of warps an SM holds

enum { ST_OK = 0, ST_ITER_CAP = 1, ST_TOO_MANY_ROWS = 2, ST_NAN = 4 };

// end-effector quantities: produced by the rigid-body passes, consumed when the level-1 rows are built - they live where the projected rows go afterwards
struct EeWs { double Jee[6 * LDM], djv_ee[6], ee_m_pos[3], ee_m_vel[3], ee_m_rot[9], ee_m_w[3], ee_d_pos[3], ee_d_vel[3], ee_d_rot[9]; };
// QP workspace, 20 KB per robot (round 1: 44 KB, which capped the SM at four warps; the whole per-robot block is now 28 KB = eight warps per SM):
//   * the null-space basis is kept in null-space width (36 x <= 18) instead of 36 x 36,
//   * the level-0 factorisation runs in place on the task rows (row i of the task IS column i of the column-major QR workspace),
//   * levels >= 1 iterate in null-space coordinates on the projected rows A_p Z (<= 22 x 18), so the 36-wide rows are only a build area that the
//     factorisation workspaces of the level reuse; working-set rows are regenerated from M / J instead of being cached.
struct QpWs {
  union ZA { struct Q { double Z[36 * LZ];        // orthonormal basis of the current null space, active columns [off, nzc).  Level 0, a pass with more than MAXR
                                                  //   rows: its rows (up to MAXR0, reaching into AR) and the Gram scratch behind row MAXR0
                        double AR[MAXR * LDZ];    // level 0: task rows / their in-place QR.  levels >= 1: raw task rows while they are built, then the
                      } q;                        //   step workspace W1 (LZ x MAXR, at AR) and the working-set factorisation Wc (LZ x MAXW, behind it)
             RbdWs rbd;                           // rigid-body passes (before the hierarchy starts)
             __device__ ZA() {} } za;
  union AH { double Ah[MAXR * LZ];                // projected task rows A_p Z (rows x nz, pitch LZ) = column-major nz x rows for the null-space QR of the level
             EeWs ee; __device__ AH() {} } ah;
  union GL { double G[18 * 19 / 2 + 1];           // normal equations (packed lower triangle) of an overdetermined / rank-deficient step (k <= 18 at levels >= 1)
             struct L0 { double b[MAXR0], tau[MAXR0], t18[MAXR0]; int perm[MAXR0]; } l0;   // level 0: right-hand side and QR scratch of its MAXR0 rows
             __device__ GL() {} } gl;
  double tau[MAXR], tauc[MAXW];
  double xbar[36], dx[36], g[36], y[36], s[36], zac[LZ + 1], rhs[MAXR], bp[MAXR], bh[MAXR], lam[MAXW], t18[MAXR];
  int perm[MAXR], permc[MAXW], wset[MAXW];
};
static_assert(LZ * MAXR + LZ * MAXW <= MAXR * LDZ, "W1 and Wc share the row build area");
static_assert(sizeof(RbdWs) <= sizeof(double) * (36 * LZ + MAXR * LDZ), "rigid-body workspace overlays Z + AR only");
static_assert(MAXR0 * LDZ + KG0 * (KG0 + 1) / 2 <= 36 * LZ + MAXR * LDZ, "level 0's rows and the Gram of a rank-deficient pass fit in Z + AR");
static_assert(MAXR0 <= 32, "w_qrcp factors at most 32 columns");

struct WbcSmem {
  double q[NQ], v[NQ], qd[NQ], vd[NQ];
  double M[NQ * LDM], nle[NQ];
  // foot Jacobians in their sparsity: row 3 f + a = [6 base columns | the 3 columns of the foot's own leg] (the other 15 of the 24 columns are structurally zero)
  double Jc[12 * LJC], djv_f[12], fpos_m[12], fvel_m[12], fpos_d[12], fvel_d[12];
  double Tm[9], wdot_base[3], base_acc[6], fdes[12], lim[NJ], vstar[56];   // fdes: the MPC's contact forces (the rest of x_des / u_des is read from HBM once)
  QpWs qp;
  Tuning tun;   // the robot's gains and friction pyramid (tuning_of), staged here so that no pointer to them stays live in registers
};

// ---------------------------------------------------------------------------------------------------------
// Inequality rows of task0 (never stored): i in [0,18): +tau_i <= lim_i ; [18,36): -tau_i <= lim_i ;
// [36, 36+5*nc): friction pyramid of the stance feet (WbcBase.cpp:360-383, 407-437).  The trailing all-zero
// rows the reference appends (WbcBase.cpp:426-427) can never be active and are skipped.
// value(i, x) = D_i x - f_i
struct IneqCtx { const WbcSmem* sm; int mode; int nc; double mu; int lfp, ffp; };   // lfp: leg -> foot, two bits per leg; ffp: foot -> first joint of its leg, four bits per foot
__device__ __forceinline__ int foot_first(int ffp, int f) { return (ffp >> (4 * f)) & 15; }
// (J_f^T F)[6 + jn]: the only contact forces that load joint jn are those of the joint's own foot
__device__ __forceinline__ double jt_force(const WbcSmem* sm, int lfp, int jn, const double* F) {
  if (jn >= 12) return 0.0;
  const int lg = jn / 3, f = (lfp >> (2 * lg)) & 3, d = jn - 3 * lg; const double* J = sm->Jc + 3 * f * LJC + 6 + d;
  return J[0] * F[3 * f] + J[LJC] * F[3 * f + 1] + J[2 * LJC] * F[3 * f + 2];
}

__device__ __forceinline__ int stance_foot_by_rank(int mode, int rank) { int k = 0; for (int f = 0; f < 4; ++f) if (contact_flag(mode, f)) { if (k == rank) return f; ++k; } return -1; }

__device__ __forceinline__ double ineq_row_dot(const IneqCtx& c, int i, const double* x) {  // D_i . x
  if (i < 36) {
    const int jn = i < 18 ? i : i - 18; const double* Mr = c.sm->M + (6 + jn) * LDM; double s = 0.0;
    for (int k = 0; k < NQ; ++k) s += Mr[k] * x[k];
    s -= jt_force(c.sm, c.lfp, jn, x + NQ);
    return i < 18 ? s : -s;
  }
  const int r = i - 36; const int foot = stance_foot_by_rank(c.mode, r / 5); const int t = r % 5; const double* F = x + NQ + 3 * foot;
  if (t == 0) return -F[2];
  if (t == 1) return F[0] - c.mu * F[2];
  if (t == 2) return -F[0] - c.mu * F[2];
  if (t == 3) return F[1] - c.mu * F[2];
  return -F[1] - c.mu * F[2];
}
__device__ __forceinline__ double ineq_rhs(const IneqCtx& c, int i) {   // f_i + v*_i
  double f = 0.0;
  if (i < 18) f = c.sm->lim[i] - c.sm->nle[6 + i]; else if (i < 36) f = c.sm->lim[i - 18] + c.sm->nle[6 + i - 18];
  return f + c.sm->vstar[i];
}
__device__ __forceinline__ double ineq_row_elem(const IneqCtx& c, int i, int k) {   // D_i[k]
  if (i < 36) { const int jn = i < 18 ? i : i - 18; const double sgn = i < 18 ? 1.0 : -1.0; if (k < NQ) return sgn * c.sm->M[(6 + jn) * LDM + k];
    const int r = k - NQ, d = jn - foot_first(c.ffp, r / 3); return (d >= 0 && d < 3) ? -sgn * c.sm->Jc[r * LJC + 6 + d] : 0.0; }
  const int r = i - 36; const int foot = stance_foot_by_rank(c.mode, r / 5); const int t = r % 5; const int kk = k - NQ - 3 * foot;
  if (kk < 0 || kk > 2) return 0.0;
  if (kk == 2) return t == 0 ? -1.0 : -c.mu;
  if (kk == 0) return t == 1 ? 1.0 : (t == 2 ? -1.0 : 0.0);
  return t == 3 ? 1.0 : (t == 4 ? -1.0 : 0.0);
}

// ---------------------------------------------------------------------------------------------------------
// Minimum-norm least squares  min || Abar y - rhs ||  with Abar^T stored column-wise in W (n x r, leading dimension ldw): COD.
// On exit y[0..n) holds the solution in the coordinates of W's rows; returns rank.  Rank-deficient rows of a rank above kg (no room for their Gram) are solved on
// their k independent rows, which is the same solution when the dependent rows are consistent with them; otherwise y holds that solution and returns -1.
// Scratch: tau / perm (r entries), t (k) and G (k(k+1)/2 doubles, k <= kg).
__device__ int cod_lstsq(double* W, int n, int r, int ldw, const double* rhs, double* y, double* G, int kg, double* tau, int* perm, double* t, int lane) {
  const int k = w_qrcp(W, n, r, ldw, tau, perm, 1e-11, lane);
  // Abar = P R^T Q^T  →  residual_c = sum_{i<=min(c,k-1)} R[i][c] y_i - rhs[perm[c]]
  for (int i = lane; i < n; i += 32) y[i] = 0.0;
  __syncwarp();
  if (k == 0) return 0;
  if (k == r || k > kg) {   // square lower-triangular system R11^T y1 = P^T rhs
    for (int c = 0; c < k; ++c) {
      double part = 0.0; if (lane < c) part = W[lane + c * ldw] * y[lane];
      const double s = warp_sum(part);
      if (lane == 0) y[c] = (rhs[perm[c]] - s) / W[c + c * ldw];
      __syncwarp();
    }
    if (k < r) {   // the dependent rows must hold at that solution (lane = row, r <= 32)
      bool off = false;
      if (lane >= k && lane < r) { double s = 0.0; for (int i = 0; i < k; ++i) s += W[i + lane * ldw] * y[i]; const double b = rhs[perm[lane]]; off = fabs(s - b) > 1e-9 * (1.0 + fabs(b)); }
      if (__any_sync(FULL, off)) { w_apply_q(W, n, k, ldw, tau, y, lane); return -1; }   // y: the solution on the independent rows, in x coordinates
    }
  } else {        // overdetermined / rank deficient: normal equations on the k x k triangular factor, G = R R^T as a packed lower triangle
    { int a = 0, b = lane; while (b > a) { b -= a + 1; ++a; }   // entry number `lane` of the packed triangle; the lane then strides by 32 entries
      while (a < k) { double s = 0.0; for (int c = a; c < r; ++c) s += W[a + c * ldw] * W[b + c * ldw]; G[tri(a) + b] = s;
        b += 32; while (b > a) { b -= a + 1; ++a; } } }
    if (lane < k) { double s = 0.0; for (int c = lane; c < r; ++c) s += W[lane + c * ldw] * rhs[perm[c]]; t[lane] = s; }
    __syncwarp();
    w_cholesky(G, k, lane);
    w_chol_solve(G, k, t, lane);
    if (lane < k) y[lane] = t[lane];
    __syncwarp();
  }
  w_apply_q(W, n, k, ldw, tau, y, lane);
  return k;
}

// Build the task rows of one hierarchy level into the row build area qp.za.q.AR (pitch LDZ) / qp.bp (level 0: qp.gl.l0.b).  Returns the row count.
//   level 0: floating-base EoM + no-contact-motion + swing zero-force           (WbcBase.cpp:338-356, 386-401, 407-415)
//   level 1: HierarchicalWbc: height, base angular, EE linear, EE angular, 100*swing (t>=10) | arm joint tracking (t<10)
//            HierarchicalMpcWbc: height, base angular, base linear, 100*swing
//   level 2: contact force + base linear | contact force
__device__ int build_level(WbcSmem& sm, const Tuning* __restrict__ tn, int level, int mode, int variant, bool init_phase, int ffp, int lane) {
  QpWs& qp = sm.qp; double* Ap = qp.za.q.AR; const EeWs& ee = qp.ah.ee; int nc = 0; for (int f = 0; f < 4; ++f) nc += contact_flag(mode, f);
  double* b0 = qp.gl.l0.b; int rows = 0;
  if (level == 0) rows = 18;
  else if (level == 1) rows = (variant == 0) ? (init_phase ? 6 : 10 + 3 * (4 - nc)) : (6 + 3 * (4 - nc));
  else rows = (variant == 0) ? 14 : 12;
  for (int e = lane; e < rows * LDZ; e += 32) Ap[e] = 0.0;
  __syncwarp();
  if (level == 0) {
    for (int e = lane; e < 6 * 36; e += 32) { const int r = e / 36, k = e % 36; Ap[r * LDZ + k] = (k < NQ) ? sm.M[r * LDM + k] : -sm.Jc[(k - NQ) * LJC + r]; }
    if (lane < 6) b0[lane] = -sm.nle[lane];
    int row = 6;
    for (int f = 0; f < 4; ++f) if (contact_flag(mode, f)) { if (lane < 27) { const int a = lane / 9, c = lane - 9 * a; Ap[(row + a) * LDZ + (c < 6 ? c : foot_first(ffp, f) + c)] = sm.Jc[(3 * f + a) * LJC + c]; } if (lane < 3) b0[row + lane] = -sm.djv_f[3 * f + lane]; row += 3; }
    for (int f = 0; f < 4; ++f) if (!contact_flag(mode, f)) { if (lane < 3) { Ap[(row + lane) * LDZ + NQ + 3 * f + lane] = 1.0; b0[row + lane] = 0.0; } row += 3; }
  } else if (level == 1) {
    int row = 0;
    if (variant == 0 && init_phase) {   // formulateArmJointNomalTrackingTask (WbcBase.cpp:439-465)
      if (lane < 6) { const int k = NQ - 6 + lane; Ap[lane * LDZ + k] = 1.0; qp.bp[lane] = tn->arm_joint_kp[lane] * (sm.qd[k] - sm.q[k]) + tn->arm_joint_kd[lane] * (sm.vd[k] - sm.v[k]); }
      row = 6;
    } else {
      // formulateBaseHeightMotionTask (WbcBase.cpp:296-308)
      if (lane == 0) { Ap[2] = 1.0; qp.bp[0] = sm.base_acc[2] + tn->base_height_kp * (sm.qd[2] - sm.q[2]) + tn->base_height_kd * (sm.vd[2] - sm.v[2]); }
      // formulateBaseAngularMotionTask (WbcBase.cpp:258-293): base_j angular rows are [0 | T | 0]
      if (lane < 3) {
        const int r = lane; for (int k = 0; k < 3; ++k) Ap[(1 + r) * LDZ + 3 + k] = sm.Tm[3 * r + k];
        double wM[3], wD[3]; matvec3(sm.Tm, sm.v + 3, wM); matvec3(sm.Tm, sm.vd + 3, wD);
        double Rm[9], Rr[9], err[3]; rot_zyx(sm.q[3], sm.q[4], sm.q[5], Rm); rot_zyx(sm.qd[3], sm.qd[4], sm.qd[5], Rr); rotation_error_world(Rr, Rm, err);
        // getGlobalAngularAccelerationFromEulerAnglesZyxDerivatives(eulerMeasured, eulerRatesDesired, eulerAccDesired) = T edd + Tdot(ed) ed
        double tdd[3], tde[3]; matvec3(sm.Tm, sm.base_acc + 3, tdd); euler_rate_map_dot_times(sm.q[3], sm.q[4], sm.vd + 3, tde);
        qp.bp[1 + r] = tdd[r] + tde[r] + tn->base_angular_kp * err[r] + tn->base_angular_kd * (wD[r] - wM[r]) - sm.wdot_base[r];
      }
      row = 4;
      if (variant == 0) {
        // formulateEeLinearMotionTrackingTask (WbcBase.cpp:467-492) and formulateEeAngularMotionTrackingTask (:494-531)
        for (int e = lane; e < 6 * NQ; e += 32) { const int a = e / NQ, k = e % NQ; const bool zero = (a >= 3 && k >= 3 && k < 6); Ap[(row + a) * LDZ + k] = zero ? 0.0 : ee.Jee[a * LDM + k]; }
        if (lane < 3) qp.bp[row + lane] = tn->ee_linear_kp[lane] * (ee.ee_d_pos[lane] - ee.ee_m_pos[lane]) + tn->ee_linear_kd[lane] * (ee.ee_d_vel[lane] - ee.ee_m_vel[lane]) - ee.djv_ee[lane];
        if (lane == 3) { double err[3]; rotation_error_world(ee.ee_d_rot, ee.ee_m_rot, err);
          // arm_dj_tmp zeroes columns 3:6 of the angular rows: Jdot_w v minus the base euler part (= Tdot ed = base angular bias acc)
          for (int a = 0; a < 3; ++a) qp.bp[row + 3 + a] = tn->ee_angular_kp[a] * err[a] - tn->ee_angular_kd[a] * ee.ee_m_w[a] - (ee.djv_ee[3 + a] - sm.wdot_base[a]); }
        row += 6;
      } else {
        // formulateBaseLinearMotionTask (WbcBase.cpp:228-240)
        if (lane < 2) { Ap[(row + lane) * LDZ + lane] = 1.0; qp.bp[row + lane] = sm.base_acc[lane] + tn->base_linear_kp * (sm.qd[lane] - sm.q[lane]) + tn->base_linear_kd * (sm.vd[lane] - sm.v[lane]); }
        row += 2;
      }
      // formulateSwingLegTask * 100 (WbcBase.cpp:311-334, HierarchicalWbc.cpp:29)
      for (int f = 0; f < 4; ++f) if (!contact_flag(mode, f)) {
        if (lane < 27) { const int a = lane / 9, c = lane - 9 * a; Ap[(row + a) * LDZ + (c < 6 ? c : foot_first(ffp, f) + c)] = 100.0 * sm.Jc[(3 * f + a) * LJC + c]; }
        if (lane < 3) { const int i = 3 * f + lane; qp.bp[row + lane] = 100.0 * (tn->kp_swing * (sm.fpos_d[i] - sm.fpos_m[i]) + tn->kd_swing * (sm.fvel_d[i] - sm.fvel_m[i]) - sm.djv_f[i]); }
        row += 3;
      }
    }
  } else {
    // formulateContactForceTask (WbcBase.cpp:534-546)
    if (lane < 12) { Ap[lane * LDZ + NQ + lane] = 1.0; qp.bp[lane] = sm.fdes[lane]; }
    if (variant == 0 && lane < 2) { Ap[(12 + lane) * LDZ + lane] = 1.0; qp.bp[12 + lane] = sm.base_acc[lane] + tn->base_linear_kp * (sm.qd[lane] - sm.q[lane]) + tn->base_linear_kd * (sm.vd[lane] - sm.v[lane]); }
  }
  __syncwarp();
  return rows;
}

// Projected task of a level >= 1:  Ah = A_p Z[:, off:nzc] (rows x nz, pitch LZ),  bh = b_p - A_p xbar.  The 36-wide rows are dead afterwards.
__device__ __forceinline__ void project_task(QpWs& qp, int rows, int off, int nz, int lane) {
  const double* Ap = qp.za.q.AR; const double* Z = qp.za.q.Z;
  for (int e = lane; e < rows * nz; e += 32) { const int i = e / nz, c = e - i * nz; const double* a = Ap + i * LDZ; double s0 = 0.0, s1 = 0.0;
#pragma unroll 6
    for (int k = 0; k < 36; k += 2) { s0 = fma(a[k], Z[k * LZ + off + c], s0); s1 = fma(a[k + 1], Z[(k + 1) * LZ + off + c], s1); }
    qp.ah.Ah[i * LZ + c] = s0 + s1; }
  if (lane < rows) { const double* a = Ap + lane * LDZ; double s = 0.0; for (int k = 0; k < 36; ++k) s = fma(a[k], qp.xbar[k], s); qp.bh[lane] = qp.bp[lane] - s; }
  __syncwarp();
}

// One hierarchy level >= 1 in null-space coordinates: primal active set over the hard inequalities, equality residual |Ah z - bh| minimised in the window.
__device__ int solve_level(WbcSmem& sm, const IneqCtx& ic, int rows, int off, int nzc, int& nw, int lane, int& iters_out, int iter_cap) {
  QpWs& qp = sm.qp; const int nz = nzc - off; const int nineq = 36 + 5 * ic.nc; int status = 0;
  if (nz <= 0) return 0;
  const double* Z = qp.za.q.Z; const double* Ah = qp.ah.Ah; double* W1 = qp.za.q.AR; double* Wc = qp.za.q.AR + LZ * MAXR;
  if (lane < LZ + 1) qp.zac[lane] = 0.0;   // accumulated step of this level in window coordinates
  __syncwarp();
  bool converged = false;
  for (int iter = 0; iter < iter_cap; ++iter) {
    iters_out = iter + 1;
    // (1) working-set constraints in window coordinates: Wc[c + k*LZ] = D_{w_k} . Z[:, off+c]  (the row is regenerated from M / J, never stored)
    int kc = 0;
    if (nw > 0) {
      for (int k = 0; k < nw; ++k) {
        const int wi = qp.wset[k]; qp.y[lane] = ineq_row_elem(ic, wi, lane); if (lane < 4) qp.y[32 + lane] = ineq_row_elem(ic, wi, 32 + lane);
        __syncwarp();
        if (lane < nz) { double s0 = 0.0, s1 = 0.0;
#pragma unroll 6
          for (int j = 0; j < 36; j += 2) { s0 = fma(qp.y[j], Z[j * LZ + off + lane], s0); s1 = fma(qp.y[j + 1], Z[(j + 1) * LZ + off + lane], s1); }
          Wc[lane + k * LZ] = s0 + s1; }
        __syncwarp();
      }
      kc = w_qrcp(Wc, nz, nw, LZ, qp.tauc, qp.permc, 1e-10, lane);
      if (kc < nw) {   // dependent rows in this window: keep an independent subset and refactor
        int keep = (lane < kc) ? qp.wset[qp.permc[lane]] : -1; __syncwarp(); if (lane < kc) qp.wset[lane] = keep; nw = kc; __syncwarp();
        continue;
      }
    }
    // (2) least squares for the step in the free directions
    for (int e = lane; e < rows * LZ; e += 32) W1[e] = Ah[e];   // W1 (nz x rows, column-major) has the memory layout of Ah (rows x nz, row-major)
    if (lane < rows) { const double* a = Ah + lane * LZ; double s = 0.0; for (int c = 0; c < nz; ++c) s = fma(a[c], qp.zac[c], s); qp.rhs[lane] = qp.bh[lane] - s; }
    __syncwarp();
    if (kc > 0) w_apply_qt_cols(Wc, nz, kc, LZ, qp.tauc, W1, rows, LZ, lane);
    const int nfree = nz - kc;
    for (int i = lane; i < nz; i += 32) qp.s[i] = 0.0;
    __syncwarp();
    if (nfree > 0) cod_lstsq(W1 + kc, nfree, rows, LZ, qp.rhs, qp.s + kc, qp.gl.G, 18, qp.tau, qp.perm, qp.t18, lane);
    if (kc > 0) w_apply_q(Wc, nz, kc, LZ, qp.tauc, qp.s, lane);
    for (int i = lane; i < 36; i += 32) { double d = 0.0; for (int c = 0; c < nz; ++c) d = fma(Z[i * LZ + off + c], qp.s[c], d); qp.dx[i] = d; }
    __syncwarp();
    double dmax = 0.0, xmax = 0.0; for (int i = lane; i < 36; i += 32) { dmax = fmax(dmax, fabs(qp.dx[i])); xmax = fmax(xmax, fabs(qp.xbar[i])); }
    dmax = warp_max(dmax); xmax = warp_max(xmax);
    bool full_step = true;
    if (dmax > 1e-12 * (1.0 + xmax)) {
      // (3) ratio test over the inequalities outside the working set
      double alpha = 1.0; int blk = -1;
      for (int i = lane; i < nineq; i += 32) {
        bool inw = false; for (int k = 0; k < nw; ++k) inw |= (qp.wset[k] == i);
        if (inw) continue;
        const double ad = ineq_row_dot(ic, i, qp.dx);
        if (ad > 1e-12 * (1.0 + dmax)) { double r = (ineq_rhs(ic, i) - ineq_row_dot(ic, i, qp.xbar)) / ad; if (r < 0.0) r = 0.0; if (r < alpha) { alpha = r; blk = i; } }
      }
      { double a = alpha; int b = (blk < 0) ? 0x7fffffff : blk; warp_argmin(a, b); alpha = a; blk = (alpha < 1.0) ? b : -1; }
      for (int i = lane; i < 36; i += 32) qp.xbar[i] += alpha * qp.dx[i];
      if (lane < nz) qp.zac[lane] += alpha * qp.s[lane];
      __syncwarp();
      if (blk >= 0) { if (nw >= MAXW) { status |= ST_TOO_MANY_ROWS; break; } if (lane == 0) qp.wset[nw] = blk; nw += 1; __syncwarp(); full_step = false; }
    }
    if (!full_step) continue;
    if (nw == 0) { converged = true; break; }
    // (4) multipliers of the working set at the face minimiser:  C^T lam = -g,  g = Ah^T (Ah z - bh)
    if (lane < rows) { const double* a = Ah + lane * LZ; double s = 0.0; for (int c = 0; c < nz; ++c) s = fma(a[c], qp.zac[c], s); qp.rhs[lane] = s - qp.bh[lane]; }
    __syncwarp();
    for (int c = lane; c < nz; c += 32) { double s = 0.0; for (int r = 0; r < rows; ++r) s = fma(Ah[r * LZ + c], qp.rhs[r], s); qp.g[c] = s; }
    __syncwarp();
    w_apply_qt(Wc, nz, kc, LZ, qp.tauc, qp.g, lane);
    double gmax = 0.0; for (int i = lane; i < nz; i += 32) gmax = fmax(gmax, fabs(qp.g[i])); gmax = warp_max(gmax);
    for (int c = kc - 1; c >= 0; --c) {   // back substitution R lam_p = -g[0:kc]
      double part = 0.0; if (lane > c && lane < kc) part = Wc[c + lane * LZ] * qp.lam[lane];
      const double s = warp_sum(part);
      if (lane == 0) qp.lam[c] = (-qp.g[c] - s) / Wc[c + c * LZ];
      __syncwarp();
    }
    double lmin = (lane < kc) ? qp.lam[lane] : 1e300; int li = lane; warp_argmin(lmin, li);
    if (lmin >= -1e-9 * (1.0 + gmax)) { converged = true; break; }
    // drop the constraint with the most negative multiplier (position li in pivoted order)
    { const int drop = qp.permc[li]; int keep = -1; if (lane < nw) { int src = lane < drop ? lane : lane + 1; keep = (src < nw) ? qp.wset[src] : -1; } __syncwarp(); if (lane < nw - 1) qp.wset[lane] = keep;
      nw -= 1; __syncwarp(); }
  }
  if (!converged) status |= ST_ITER_CAP;
  return status;
}

// TUNED: the batch has robot tuning rows.  Without them the kernel reads the gains at their fixed place in DevModel, as it did before rows existed.
template <bool TUNED>
__global__ void __launch_bounds__(32 * WBC_WARPS) wbc_update_kernel(const DevModel* __restrict__ mdl, int b0, int B, const double* __restrict__ x_des, const double* __restrict__ u_des,
                                                                   const double* __restrict__ rbd_meas, const int32_t* __restrict__ mode_in, const double* __restrict__ period_in,
                                                                   const double* __restrict__ time_in, double* __restrict__ input_last, int variant,
                                                                   double* __restrict__ cmd_out, int32_t* __restrict__ status_out, int32_t* __restrict__ diag_out,
                                                                   const double* __restrict__ srbd, const double* __restrict__ payload, const double* __restrict__ tuning) {
  // srbd [B][SRBD_DBL] / payload [B][8]: the robot's model payload (qmb200_set_model_payload) - its SRBD constants and the point masses the rigid-body passes add
  // (payload.cuh); both NULL without one (the same for the whole grid).  tuning [B][TUNING_DBL]: the robot's gains and friction pyramid (qmb200_set_robot_tuning), NULL for the
  // handle's (WbcBase::dynamicCallback, WbcBase.cpp:69-117; frictionConeTask.frictionCoefficient, task.info:346-348)
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = b0 + blockIdx.x * (int)(blockDim.x >> 5) + warp;   // robots per CTA = warps per CTA, chosen at launch (the warps of a CTA never synchronise with each other)
  if (b >= B) return;
  WbcSmem& sm = reinterpret_cast<WbcSmem*>(smem_raw)[warp];
  const int mode = mode_in[b]; const double period = period_in[b]; const double time = time_in[b];
  int nc = 0; for (int f = 0; f < 4; ++f) nc += contact_flag(mode, f);

  // ---- load the robot's inputs (coalesced, one 240-B / 440-B record each) ----
  const double* xdes = x_des + (size_t)b * NX; const double* udes = u_des + (size_t)b * NU;
  if (lane < 12) sm.fdes[lane] = udes[lane];
  const int lfp = mdl->leg_foot[0] | (mdl->leg_foot[1] << 2) | (mdl->leg_foot[2] << 4) | (mdl->leg_foot[3] << 6);
  const int ffp = mdl->foot_leg[0] | (mdl->foot_leg[1] << 4) | (mdl->foot_leg[2] << 8) | (mdl->foot_leg[3] << 12);
  // updateMeasured (WbcBase.cpp:138-144)
  if (lane < NJ) sm.lim[lane] = (lane < 12) ? mdl->effort[lane % 3] : mdl->effort[lane];
  for (int i = lane; i < 56; i += 32) sm.vstar[i] = 0.0;
  rbd_read(rbd_meas + (size_t)b * 55, sm.q, sm.v, sm.Tm, lane);
  if (lane < NQ) sm.qd[lane] = xdes[6 + lane];
  __syncwarp();

  // ---- measured side: M, nle, foot/EE Jacobians and bias accelerations ----
  RbdWs* ws = &sm.qp.za.rbd; EeWs& ee = sm.qp.ah.ee;   // the end-effector block sits outside the rigid-body overlay
  rbd_kinematics<true>(mdl, sm.q, sm.v, ws, lane);
  rbd_inertias(mdl, ws, lane, 1);
  if (payload) { if (lane < 2) payload_load(mdl, ws, lane, payload + (size_t)b * 8 + 4 * lane, true); __syncwarp(); }   // lane 0: [m_ee, o_ee], lane 1: [m_base, o_base]
  rbd_accumulate(mdl, ws, lane, true);
  rbd_mass_matrix_nle(mdl, ws, sm.M, LDM, sm.nle, lane);
  for (int f = 0; f < 4; ++f) {
    const int body = mdl->foot_body[f]; double pw[3]; foot_point(mdl, ws, f, pw);
    if (lane < 9) { const double* S = ws->S[lane < 6 ? lane : foot_first(ffp, f) + lane]; double col[3]; point_vel(S, pw, col);   // = point_jacobian restricted to the non-zero columns
      for (int a = 0; a < 3; ++a) sm.Jc[(3 * f + a) * LJC + lane] = col[a]; }
    if (lane == 0) { double vel[3], acc[3]; point_vel_acc(ws->V[body], ws->A[body], pw, vel, acc); for (int a = 0; a < 3; ++a) { sm.fpos_m[3 * f + a] = pw[a]; sm.fvel_m[3 * f + a] = vel[a]; sm.djv_f[3 * f + a] = acc[a]; } }
  }
  {
    const int body = mdl->ee_body; double pw[3]; ee_pose(mdl, ws, pw, lane == 0 ? ee.ee_m_rot : nullptr);
    point_jacobian(ws, pw, 12, 17, ee.Jee, LDM, lane);
    if (lane < NQ) { const bool on = (lane < 6) || (lane >= 18); for (int a = 0; a < 3; ++a) ee.Jee[(3 + a) * LDM + lane] = on ? ws->S[lane][a] : 0.0; }
    if (lane == 0) { double vel[3], acc[3]; point_vel_acc(ws->V[body], ws->A[body], pw, vel, acc); for (int a = 0; a < 3; ++a) { ee.ee_m_pos[a] = pw[a]; ee.ee_m_vel[a] = vel[a]; ee.djv_ee[a] = acc[a]; ee.djv_ee[3 + a] = ws->A[body][a]; ee.ee_m_w[a] = ws->V[body][a]; sm.wdot_base[a] = ws->A[0][a]; } }
  }
  __syncwarp();

  // ---- desired side (WbcBase.cpp:193-226) ----
  // vDesired = [A_b^{-1}(qD) m h ; u joints]  (SRBD mapping); jointAccel = (u - inputLast)/period; inputLast <- u
  double jacc = 0.0;
  if (lane < NJ) { const double uj = udes[12 + lane]; jacc = (uj - input_last[(size_t)b * NU + 12 + lane]) / period; sm.vd[6 + lane] = uj; }
  __syncwarp();
  if (lane < NU) input_last[(size_t)b * NU + lane] = udes[lane];
  double A22inv[9], A12[9];   // SRBD blocks at qDesired (kept in lane 0's registers; bound BEFORE dccrba in the reference)
  if (lane == 0) {
    const SrbdConst* sc = srbd_of(mdl, srbd, b);
    double R[9], T[9]; rot_zyx(sm.qd[3], sm.qd[4], sm.qd[5], R); euler_rate_map(sm.qd[3], sm.qd[4], T);
    double c[3]; matvec3(R, sc->c_nom, c);
    double RI[9], RIRt[9], A22[9]; matmul3(R, sc->I_nom, RI); matmul3_nt(RI, R, RIRt); matmul3(RIRt, T, A22); inv3(A22, A22inv);
    const double Sx[9] = {0, -c[2], c[1], c[2], 0, -c[0], -c[1], c[0], 0}; double ST[9]; matmul3(Sx, T, ST); for (int i = 0; i < 9; ++i) A12[i] = sc->m * ST[i];
    double ha[3] = {sc->m * xdes[3], sc->m * xdes[4], sc->m * xdes[5]}, ed[3]; matvec3(A22inv, ha, ed);
    double t[3]; matvec3(A12, ed, t);
    for (int a = 0; a < 3; ++a) { sm.vd[a] = xdes[a] - t[a] / sc->m; sm.vd[3 + a] = ed[a]; }
  }
  __syncwarp();
  rbd_kinematics<true>(mdl, sm.qd, sm.vd, ws, lane);
  rbd_inertias(mdl, ws, lane, 2);            // bias forces WITHOUT gravity: sum = dAg * v about the origin
  if (payload) { if (lane < 2) payload_load(mdl, ws, lane, payload + (size_t)b * 8 + 4 * lane, false); __syncwarp(); }
  rbd_accumulate(mdl, ws, lane, true);
  // Aj * jointAccel: sum_j (Ic_{j+1} S_j) qdd_j  (full-model centroidal momentum matrix columns, after dccrba)
  double Phi[6] = {0, 0, 0, 0, 0, 0};
  if (lane < NJ) { inertia_apply(ws->Ic[lane + 1], ws->S[6 + lane], Phi); for (int i = 0; i < 6; ++i) Phi[i] *= jacc; }
  for (int i = 0; i < 6; ++i) Phi[i] = warp_sum(Phi[i]);
  for (int f = 0; f < 4; ++f) {
    double pw[3]; foot_point(mdl, ws, f, pw);
    if (lane == 0) { double vel[3]; point_vel(ws->V[mdl->foot_body[f]], pw, vel); for (int a = 0; a < 3; ++a) { sm.fpos_d[3 * f + a] = pw[a]; sm.fvel_d[3 * f + a] = vel[a]; } }
  }
  if (lane == 0) {
    double pw[3], vel[3]; ee_pose(mdl, ws, pw, ee.ee_d_rot); point_vel(ws->V[mdl->ee_body], pw, vel);
    for (int a = 0; a < 3; ++a) { ee.ee_d_pos[a] = pw[a]; ee.ee_d_vel[a] = vel[a]; }
    // centroidalMomentumRate = m*getNormalizedCentroidalMomentumRate(u) [true COM] - dAg v - Aj qdd_j ; baseAcc = AbInv(SRBD) * that
    const SrbdConst* sc = srbd_of(mdl, srbd, b);
    const double mt = ws->Ic[0][0]; const double com[3] = {ws->Ic[0][1] / mt, ws->Ic[0][2] / mt, ws->Ic[0][3] / mt};
    double lin[3] = {0, 0, -9.81 * sc->m}, ang[3] = {0, 0, 0};
    for (int f = 0; f < 4; ++f) { const double* F = sm.fdes + 3 * f; const double r[3] = {sm.fpos_d[3 * f] - com[0], sm.fpos_d[3 * f + 1] - com[1], sm.fpos_d[3 * f + 2] - com[2]}; lin[0] += F[0]; lin[1] += F[1]; lin[2] += F[2]; cross3_add(r, F, ang); }
    // spatial force about the origin → about the COM: n_com = nO - com x f
    const double* Fb = ws->F[0]; double cf[3]; cross3(com, Fb + 3, cf);
    double cp[3]; cross3(com, Phi + 3, cp);
    for (int a = 0; a < 3; ++a) { lin[a] -= Fb[3 + a] + Phi[3 + a]; ang[a] -= (Fb[a] - cf[a]) + (Phi[a] - cp[a]); }
    double ed[3]; matvec3(A22inv, ang, ed); double t[3]; matvec3(A12, ed, t);
    for (int a = 0; a < 3; ++a) { sm.base_acc[a] = (lin[a] - t[a]) / sc->m; sm.base_acc[3 + a] = ed[a]; }
  }
  __syncwarp();

  // ---- hierarchy ----
  // with rows, every level reads the robot's row staged in shared memory (visible after the __syncwarp below): a pointer to it held in registers across the
  // hierarchy costs spills
  if (TUNED) { const double* tr = tuning + (size_t)b * TUNING_DBL; for (int i = lane; i < TUNING_MODEL; i += 32) reinterpret_cast<double*>(&sm.tun)[i] = tr[i]; }
  const Tuning* tn = TUNED ? &sm.tun : tuning_of(mdl, nullptr, 0);
  QpWs& qp = sm.qp; IneqCtx ic{&sm, mode, nc, TUNED ? tuning[(size_t)b * TUNING_DBL + 1] : mdl->wbc_friction, lfp, ffp}; int status = 0;
  const bool init_phase = time < 10.0;   // HierarchicalWbc.cpp:32
  double* AR = qp.za.q.AR; double* Z = qp.za.q.Z; QpWs::GL::L0& l0 = qp.gl.l0;
  for (int i = lane; i < 36; i += 32) qp.xbar[i] = 0.0;
  __syncwarp();
  // level 0: min ||A0 x - b0||^2 + ||(D0 x - f0)_+||^2  — semismooth iteration on the violated set V.  The rows are factorised IN PLACE (row i of the task is
  // column i of the column-major QR workspace), so every pass rebuilds them from M / J (a few hundred element writes; the generic case takes one pass + one check)
  const int nineq = 36 + 5 * nc; const int cap0 = mdl->wbc_iter_cap0, cap = mdl->wbc_iter_cap; int it0 = 0;
  unsigned vmask0 = 0, vmask1 = 0;   // violated set, bit per inequality (lane-uniform)
  int k0 = 0;
  for (int it = 0; it < cap0; ++it) {
    int r = build_level(sm, tn, 0, mode, variant, init_phase, ffp, lane); it0 = it + 1;
    // a pass with more than MAXR rows moves the task rows to the start of Z (not in use before level 0 ends) and lets the violated rows run on into AR;
    // every other pass works in AR and keeps Z as the scratch of the rank-deficient branch, so the last pass of a robot whose set stays empty leaves the QR of A0 in AR
    const bool big = r + __popc(vmask0) + __popc(vmask1) > MAXR; double* W = big ? Z : AR;
    if (big) { for (int e = lane; e < r * LDZ; e += 32) W[e] = AR[e]; __syncwarp(); }
    // append violated rows
    for (int i = 0; i < nineq; ++i) { const bool in = (i < 32) ? ((vmask0 >> i) & 1u) : ((vmask1 >> (i - 32)) & 1u); if (in) { if (r >= MAXR0) { status |= ST_TOO_MANY_ROWS; break; }
        for (int k = lane; k < 36; k += 32) W[r * LDZ + k] = ineq_row_elem(ic, i, k); if (lane == 0) l0.b[r] = ineq_rhs(ic, i); ++r; } }
    __syncwarp();
    k0 = cod_lstsq(W, 36, r, LDZ, l0.b, qp.xbar, big ? Z + MAXR0 * LDZ : Z, big ? KG0 : 36, l0.tau, l0.perm, l0.t18, lane);
    if (k0 < 0) { status |= ST_TOO_MANY_ROWS; break; }
    __syncwarp();
    unsigned n0 = 0, n1 = 0;   // next violated set: strictly violated rows, plus rows of V sitting on their boundary
    for (int i = lane; i < nineq; i += 32) { const double val = ineq_row_dot(ic, i, qp.xbar) - ineq_rhs(ic, i); const double sc = 1e-9 * (1.0 + fabs(ineq_rhs(ic, i)));
      const bool inV = (i < 32) ? ((vmask0 >> i) & 1u) : ((vmask1 >> (i - 32)) & 1u);
      if (val > sc || (inV && val >= -sc)) { if (i < 32) n0 |= 1u << i; else n1 |= 1u << (i - 32); } }
    for (int o = 16; o > 0; o >>= 1) { n0 |= __shfl_xor_sync(FULL, n0, o); n1 |= __shfl_xor_sync(FULL, n1, o); }
    if (n0 == vmask0 && n1 == vmask1) break;
    vmask0 = n0; vmask1 = n1;
    if (it == cap0 - 1) status |= ST_ITER_CAP;
  }
  // optimal slack of level 0 and the null space of A0 (HoQp::buildZMatrix, HoQp.cpp:126-133)
  for (int i = lane; i < nineq; i += 32) { const double val = ineq_row_dot(ic, i, qp.xbar) - ineq_rhs(ic, i); sm.vstar[i] = val > 0.0 ? val : 0.0; }
  __syncwarp();
  int off = 0, nzc = 0, nw = 0, it1 = 0, it2 = 0;
  {
    if (vmask0 | vmask1) {   // the last factorisation contains violated rows: factor A0 alone (otherwise the one in AR already is the QR of A0')
      const int rows0 = build_level(sm, tn, 0, mode, variant, init_phase, ffp, lane);
      k0 = w_qrcp(AR, 36, rows0, LDZ, l0.tau, l0.perm, 1e-11, lane);
    }
    nzc = 36 - k0;
    if (nzc > LZ - 1) { status |= ST_TOO_MANY_ROWS; nzc = 0; }   // (A0 has 18 independent rows for every physical model: the mass matrix and a contact Jacobian)
    else w_form_q_tail(AR, 36, k0, LDZ, l0.tau, Z, LZ, lane);
  }
  // levels 1 and 2
  for (int level = 1; level <= 2 && nzc > 0; ++level) {
    const int rows = build_level(sm, tn, level, mode, variant, init_phase, ffp, lane);
    const int nz = nzc - off;
    if (nz <= 0) break;                                   // trivial kernel (the reference keeps one zero column, HoQp.cpp:129)
    project_task(qp, rows, off, nz, lane);
    status |= solve_level(sm, ic, rows, off, nzc, nw, lane, level == 1 ? it1 : it2, cap);
    if (level == 1) {                                    // Z <- Z * kernel(A_1 Z): QR of (A_1 Z)' in place on the projected rows
      const int k = w_qrcp(qp.ah.Ah, nz, rows, LZ, qp.tau, qp.perm, 1e-11, lane);
      w_apply_q_right(qp.ah.Ah, nz, k, LZ, qp.tau, Z, 36, LZ, off, lane);
      off += k;
    }
  }
  // ---- updateCmd (WbcBase.cpp:548-563): tau = [M_j, -J_j^T] x + h_j ; cmd = [x; tau] ----
  double* out = cmd_out + (size_t)b * 54;
  for (int i = lane; i < 36; i += 32) out[i] = qp.xbar[i];
  bool bad = false;
  if (lane < NJ) { const double* Mr = sm.M + (6 + lane) * LDM; double s = sm.nle[6 + lane]; for (int k = 0; k < NQ; ++k) s += Mr[k] * qp.xbar[k]; s -= jt_force(&sm, lfp, lane, qp.xbar + NQ); out[36 + lane] = s; bad = !isfinite(s); }
  if (__any_sync(FULL, bad)) status |= ST_NAN;
  // status word: WBC flags only, in the low byte (bits 8..15 carry the MPC flags after qmb200_tick's merge, bit 16 = QMB200_ST_SAFETY: include/qmb200.h);
  // iteration counts / working-set size go to the separate diagnostics word: it0 | it1 << 8 | it2 << 16 | nw << 24
  if (lane == 0) { status_out[b] = status; if (diag_out) diag_out[b] = (it0 & 0xff) | ((it1 & 0xff) << 8) | ((it2 & 0xff) << 16) | ((nw & 0xff) << 24); }
}

static_assert(sizeof(WbcSmem) * WBC_WARPS <= 227 * 1024, "WBC shared-memory budget exceeded");
size_t wbc_smem_bytes() { return sizeof(WbcSmem) * WBC_WARPS; }

void launch_wbc_update(const DevModel* mdl, int B, const double* x_des, const double* u_des, const double* rbd, const int32_t* mode, const double* period, const double* time,
                       double* input_last, int variant, double* cmd, int32_t* status, cudaStream_t stream, int b0, int b1, int32_t* diag, const double* srbd, const double* payload, const double* tuning) {
  if (b1 < 0) b1 = B; if (b1 <= b0) return;
  // Eight robots per CTA, one CTA per SM (8 x 28 KB of shared memory: the same 227 KB budget per block on H100).  Smaller CTAs would even out the per-CTA tail, but
  // the kernel is ~24 k SASS instructions (sm_90a build) and the warps of one CTA run in phase and share the instruction cache; a batch of one wave takes the time of its slowest
  // robot whatever the CTA shape.
  const int nb = b1 - b0; const int wpc = WBC_WARPS;
  const int grid = (nb + wpc - 1) / wpc;
  (tuning ? wbc_update_kernel<true> : wbc_update_kernel<false>)<<<grid, 32 * wpc, sizeof(WbcSmem) * wpc, stream>>>(mdl, b0, b1, x_des, u_des, rbd, mode, period, time, input_last, variant, cmd, status, diag, srbd, payload, tuning);
}

// cudaFuncSetAttribute is per device: called from qmb200_create after cudaSetDevice (one handle per GPU, several handles / devices per process allowed)
int wbc_configure_device() {
  cudaError_t e = cudaFuncSetAttribute(wbc_update_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wbc_smem_bytes());
  if (e == cudaSuccess) e = cudaFuncSetAttribute(wbc_update_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wbc_smem_bytes());
  return (int)e;
}

}  // namespace qmb
