// Device-side common definitions for the batched MPC+WBC kernels (sm_90a, fp64).
// One warp owns one robot; lanes cooperate over bodies / matrix rows; all per-robot state lives in
// shared memory or registers, HBM is touched only for the batch I/O buffers.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include <cmath>
#include <string>

// Scalar helpers are host + device: tests/nodeeval_host.cpp compiles the one-thread-per-node evaluator (node_eval.cuh) with g++ and checks it against the
// oracle on the CPU.  Everything that needs warp intrinsics stays inside #ifdef __CUDACC__.
#ifdef __CUDACC__
#define QMB_HD __host__ __device__ __forceinline__
#else
#define QMB_HD inline
#endif

namespace qmb {

constexpr int NQ = 24;   // generalized coordinates (WbcBase.cpp:36, task.info:150-189)
constexpr int NJ = 18;   // actuated joints
constexpr int NB = 19;   // bodies (base + one per joint)
constexpr int NX = 30;   // centroidal state
constexpr int NU = 30;   // input: 12 contact forces (LF,RF,LH,RH) + 18 joint velocities
constexpr int NDEC = 36; // WBC decision vector [vdot(24); F(12)]
constexpr unsigned FULL = 0xffffffffu;
// The measured state rbd[55] (include/qmb200.h): euler ZYX, base position, joint positions, world angular velocity, base linear velocity, joint velocities,
// end-effector position and orientation quaternion xyzw
constexpr int RBD_ZYX = 0, RBD_POS = 3, RBD_JPOS = 6, RBD_W = 24, RBD_V = 27, RBD_JVEL = 30, RBD_EE_POS = 48, RBD_EE_QUAT = 51;

// Model + settings constants, replicated per GPU (read-only, L1/L2 resident).
struct DevModel {
  // kinematic tree: joint j moves body j+1
  int parent[NJ];          // parent body index
  int axis[NJ];            // 0/1/2 = x/y/z in the joint frame
  int depth[NB];           // base 0
  int chain_start[NJ];     // first joint of the serial chain joint j belongs to
  double Rj[NJ][9];        // joint frame in parent body frame (row-major)
  double pj[NJ][3];
  double mass[NB];
  double com[NB][3];       // body frame
  double Ib[NB][9];        // about com, body frame
  int foot_body[4];        // contact order LF, RF, LH, RH
  int foot_leg[4];         // index of the leg's first joint (joint order LF, LH, RF, RH)
  int leg_foot[4];         // inverse map: leg (first joint / 3) → foot index
  double foot_p[4][3];
  int ee_body; double ee_R[9]; double ee_p[3];
  double ee_body_R0[9], ee_body_p0[3];       // world pose of ee_body at defaultJointState (base at the origin, level): where srbd_payload_fold places o_ee
  double total_mass;
  double I_nom[9], I_nom_inv[9], c_nom[3];   // SRBD centroidalInertiaNominal, its inverse, comToBasePositionNominal
  double effort[NJ];
  double arm_pos_lower[6], arm_pos_upper[6];
  // MPC settings (task.info:75-92,138-147,192-343)
  double Q[NX * NX], R[NU * NU];
  double Qdiag[NX]; int q_is_diag;   // Q of task.info:192-233 is diagonal: fast path when the loaded matrix really is (checked at create), dense fallback otherwise
  double Rblk[8][9], Rarm[6];   // R is block diagonal (QMInterface.cpp:274-299): 3x3 blocks per foot force / per leg, diagonal for the arm; checked at create
  // what the projection kernel reads per node stays on adjacent cache lines, from Qdiag to the end-effector weights of the tuned block
  double pos_limit_mu, pos_limit_delta, vel_limit_mu, vel_limit_delta;
  double arm_vel_lower[6], arm_vel_upper[6];
  double friction_barrier_mu, friction_barrier_delta, friction_reg, friction_hess_shift;
  // The tuned block, in Tuning's order (a robot with a tuning row reads its own copy, qmb200_set_robot_tuning): the MPC friction-cone coefficient
  // (task.info:290-292), the WBC friction pyramid (task.info:346-348), the end-effector soft-constraint weights (task.info:235-246) and the WBC gains
  // (wbcWigeht.cfg:7-47)
  double friction_mu, wbc_friction;
  double mu_ee_pos, mu_ee_ori, mu_final_ee_pos, mu_final_ee_ori;
  double kp_swing, kd_swing, base_height_kp, base_height_kd, base_linear_kp, base_linear_kd, base_angular_kp, base_angular_kd;
  double arm_joint_kp[6], arm_joint_kd[6], ee_linear_kp[3], ee_linear_kd[3], ee_angular_kp[3], ee_angular_kd[3];
  double lift_off_velocity, touch_down_velocity, swing_height, swing_time_scale, position_error_gain;
  double dt, time_horizon, delta_tol, g_max, g_min, alpha_decay, alpha_min, gamma_c, armijo_factor;
  double rk_c, rk_w1, rk_w2;
  // solver variant (qmb200_mpc_set_solver): 0 = multiple-shooting SQP (sqp{}, what QMController runs), 1 = multiple-shooting IPM (ipm{}: this OCP has no
  // inequality rows, so the interior-point step IS the equality-constrained Newton step; only the tolerances differ), 2 = DDP (ddp{}: single-shooting rollouts,
  // discrete Riccati backward pass, rollout line search on the merit cost + penalty * sqrt(equality SSE))
  int solver; double ddp_penalty, ddp_min_step, ddp_max_step, ddp_armijo, ddp_contraction;
  int wbc_iter_cap0, wbc_iter_cap;   // WBC iteration caps: level-0 semismooth passes (30) and active-set iterations per level (80); qmb200_wbc_set_iteration_caps (diagnostics / tests)
  double cost_tol; int sqp_iterations;   // sqp.sqpIteration (task.info:28) and costTol [upstream ocs2_sqp default 1e-4]: SqpSolver::runImpl loop + checkConvergence
};

// The SRBD constants of one robot (createCentroidalModelInfo [upstream]): robotMass, centroidalInertiaNominal, its inverse, comToBasePositionNominal, in the order
// DevModel keeps the nominal robot's.  A robot with a model payload (qmb200_set_model_payload) has its own block of SRBD_DBL doubles in this order, so the kernels
// read either through one pointer: srbd_of(mdl, srbd, b) with srbd = the per-robot blocks, or NULL for the nominal model.
struct SrbdConst { double m, I_nom[9], I_nom_inv[9], c_nom[3]; };
constexpr int SRBD_DBL = 24;   // SrbdConst padded to 16-byte rows
static_assert(offsetof(DevModel, I_nom) == offsetof(DevModel, total_mass) + offsetof(SrbdConst, I_nom) && offsetof(DevModel, I_nom_inv) == offsetof(DevModel, total_mass) + offsetof(SrbdConst, I_nom_inv) &&
              offsetof(DevModel, c_nom) == offsetof(DevModel, total_mass) + offsetof(SrbdConst, c_nom) && sizeof(SrbdConst) <= SRBD_DBL * 8, "DevModel's SRBD fields have SrbdConst's layout");
QMB_HD const SrbdConst* srbd_of(const DevModel* mdl, const double* srbd, int b) {
  return srbd ? reinterpret_cast<const SrbdConst*>(srbd + (size_t)SRBD_DBL * b) : reinterpret_cast<const SrbdConst*>(&mdl->total_mass);
}

// The controller parameters one robot may override (qmb200_set_robot_tuning), in the order DevModel keeps the handle's: the first TUNING_MODEL doubles of a
// tuning row.  The row's last two doubles are the control law's arm gains (ControlLawParams arm_kp / arm_kd), read by the control law alone.  As with
// SrbdConst, every consumer reads through one pointer: tuning_of(mdl, rows, b) with rows = the per-robot rows, or NULL for the handle's values.
struct Tuning {
  double friction_mu, wbc_friction, mu_ee_pos, mu_ee_ori, mu_final_ee_pos, mu_final_ee_ori;
  double kp_swing, kd_swing, base_height_kp, base_height_kd, base_linear_kp, base_linear_kd, base_angular_kp, base_angular_kd;
  double arm_joint_kp[6], arm_joint_kd[6], ee_linear_kp[3], ee_linear_kd[3], ee_angular_kp[3], ee_angular_kd[3];
};
constexpr int TUNING_MODEL = 38, TUNING_DBL = 40, TUNING_ARM_KP = 38, TUNING_ARM_KD = 39;
static_assert(sizeof(Tuning) == TUNING_MODEL * 8 && offsetof(DevModel, ee_angular_kd) + 3 * 8 - offsetof(DevModel, friction_mu) == sizeof(Tuning) &&
              offsetof(DevModel, wbc_friction) == offsetof(DevModel, friction_mu) + offsetof(Tuning, wbc_friction) &&
              offsetof(DevModel, mu_ee_pos) == offsetof(DevModel, friction_mu) + offsetof(Tuning, mu_ee_pos) &&
              offsetof(DevModel, kp_swing) == offsetof(DevModel, friction_mu) + offsetof(Tuning, kp_swing) &&
              offsetof(DevModel, arm_joint_kp) == offsetof(DevModel, friction_mu) + offsetof(Tuning, arm_joint_kp) &&
              offsetof(DevModel, ee_angular_kd) == offsetof(DevModel, friction_mu) + offsetof(Tuning, ee_angular_kd), "DevModel's tuned fields have Tuning's layout");
QMB_HD const Tuning* tuning_of(const DevModel* mdl, const double* rows, int b) {
  return rows ? reinterpret_cast<const Tuning*>(rows + (size_t)TUNING_DBL * b) : reinterpret_cast<const Tuning*>(&mdl->friction_mu);
}

#ifdef __CUDACC__
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(FULL, v, o));
  return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(FULL, v, o));
  return v;
}
// argmax over lanes: returns (value, index) of the maximum; ties → lowest index
__device__ __forceinline__ void warp_argmax(double& v, int& idx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double ov = __shfl_xor_sync(FULL, v, o); int oi = __shfl_xor_sync(FULL, idx, o);
    if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
}
// argmax over the ACTIVE lanes of non-negative values (ties -> lowest lane; v = -1 when no lane is active): a non-negative double orders like its bit
// pattern, so two 32-bit REDUX maxima (high word, then low word among the lanes holding the high maximum) and a ballot replace five shuffle rounds
__device__ __forceinline__ void warp_argmax_nonneg(double& v, int& idx, bool active) {
  const unsigned long long b = active ? (unsigned long long)__double_as_longlong(v) : 0ull;
  const unsigned hi = (unsigned)(b >> 32), lo = (unsigned)b;
  const unsigned mh = __reduce_max_sync(FULL, hi);
  const unsigned ml = __reduce_max_sync(FULL, hi == mh ? lo : 0u);
  const unsigned m = __ballot_sync(FULL, active && hi == mh && lo == ml);
  if (m == 0u) { v = -1.0; idx = 0; return; }
  idx = __ffs(m) - 1; v = __longlong_as_double((long long)(((unsigned long long)mh << 32) | ml));
}
__device__ __forceinline__ void warp_argmin(double& v, int& idx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double ov = __shfl_xor_sync(FULL, v, o); int oi = __shfl_xor_sync(FULL, idx, o);
    if (ov < v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
}

#endif  // __CUDACC__

// ---- tiny 3-vector / 3x3 helpers on plain arrays ----
QMB_HD void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1]; c[1] = a[2] * b[0] - a[0] * b[2]; c[2] = a[0] * b[1] - a[1] * b[0];
}
QMB_HD void cross3_add(const double* a, const double* b, double* c) {
  c[0] += a[1] * b[2] - a[2] * b[1]; c[1] += a[2] * b[0] - a[0] * b[2]; c[2] += a[0] * b[1] - a[1] * b[0];
}
QMB_HD double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
QMB_HD void matvec3(const double* M, const double* v, double* o) {
  o[0] = M[0] * v[0] + M[1] * v[1] + M[2] * v[2]; o[1] = M[3] * v[0] + M[4] * v[1] + M[5] * v[2]; o[2] = M[6] * v[0] + M[7] * v[1] + M[8] * v[2];
}
QMB_HD void matTvec3(const double* M, const double* v, double* o) {
  o[0] = M[0] * v[0] + M[3] * v[1] + M[6] * v[2]; o[1] = M[1] * v[0] + M[4] * v[1] + M[7] * v[2]; o[2] = M[2] * v[0] + M[5] * v[1] + M[8] * v[2];
}
QMB_HD void matmul3(const double* A, const double* B, double* C) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
// C = A * B^T
QMB_HD void matmul3_nt(const double* A, const double* B, double* C) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[3 * j] + A[3 * i + 1] * B[3 * j + 1] + A[3 * i + 2] * B[3 * j + 2];
}
// R = Rz(z) Ry(y) Rx(x)   (ocs2 getRotationMatrixFromZyxEulerAngles).  The formula of rot_zyx_sc, written out: computed through rot_zyx_sc, nvcc
// contracts the WBC's desired-side rotation into different FMAs and its commands move in the last bits.
QMB_HD void rot_zyx(double z, double y, double x, double* R) {
  double sz, cz, sy, cy, sx, cx; sincos(z, &sz, &cz); sincos(y, &sy, &cy); sincos(x, &sx, &cx);
  R[0] = cz * cy; R[1] = cz * sy * sx - sz * cx; R[2] = cz * sy * cx + sz * sx;
  R[3] = sz * cy; R[4] = sz * sy * sx + cz * cx; R[5] = sz * sy * cx - cz * sx;
  R[6] = -sy;     R[7] = cy * sx;                R[8] = cy * cx;
}
// T: euler-ZYX rates → world angular velocity (ocs2 getMappingFromEulerAnglesZyxDerivativeToGlobalAngularVelocity)
QMB_HD void euler_rate_map(double z, double y, double* T) {
  double sz, cz, sy, cy; sincos(z, &sz, &cz); sincos(y, &sy, &cy);
  T[0] = 0; T[1] = -sz; T[2] = cy * cz; T[3] = 0; T[4] = cz; T[5] = cy * sz; T[6] = 1; T[7] = 0; T[8] = -sy;
}
// Tdot * ed  (time derivative of T along euler rates ed=(zd,yd,xd), applied to ed)
QMB_HD void euler_rate_map_dot_times(double z, double y, const double* ed, double* o) {
  double sz, cz, sy, cy; sincos(z, &sz, &cz); sincos(y, &sy, &cy);
  const double zd = ed[0], yd = ed[1];
  // d/dt of columns: col1 = (-sz, cz, 0) → (-cz zd, -sz zd, 0); col2 = (cy cz, cy sz, -sy) → (-sy yd cz - cy sz zd, -sy yd sz + cy cz zd, -cy yd)
  o[0] = (-cz * zd) * ed[1] + (-sy * yd * cz - cy * sz * zd) * ed[2];
  o[1] = (-sz * zd) * ed[1] + (-sy * yd * sz + cy * cz * zd) * ed[2];
  o[2] = (-cy * yd) * ed[2];
}
// Variants taking precomputed trig values tr = {sin z, cos z, sin y, cos y, sin x, cos x} (one warp-wide sincos pass serves all users)
QMB_HD void rot_zyx_sc(const double* tr, double* R) {
  const double sz = tr[0], cz = tr[1], sy = tr[2], cy = tr[3], sx = tr[4], cx = tr[5];
  R[0] = cz * cy; R[1] = cz * sy * sx - sz * cx; R[2] = cz * sy * cx + sz * sx;
  R[3] = sz * cy; R[4] = sz * sy * sx + cz * cx; R[5] = sz * sy * cx - cz * sx;
  R[6] = -sy;     R[7] = cy * sx;                R[8] = cy * cx;
}
QMB_HD void euler_rate_map_sc(const double* tr, double* T) {
  const double sz = tr[0], cz = tr[1], sy = tr[2], cy = tr[3];
  T[0] = 0; T[1] = -sz; T[2] = cy * cz; T[3] = 0; T[4] = cz; T[5] = cy * sz; T[6] = 1; T[7] = 0; T[8] = -sy;
}
QMB_HD void euler_rate_map_dot_times_sc(const double* tr, const double* ed, double* o) {
  const double sz = tr[0], cz = tr[1], sy = tr[2], cy = tr[3]; const double zd = ed[0], yd = ed[1];
  o[0] = (-cz * zd) * ed[1] + (-sy * yd * cz - cy * sz * zd) * ed[2];
  o[1] = (-sz * zd) * ed[1] + (-sy * yd * sz + cy * cz * zd) * ed[2];
  o[2] = (-cy * yd) * ed[2];
}
// Eigen::Quaterniond(const Matrix3d&) (Shepperd's method, largest diagonal pivot); out = x, y, z, w
QMB_HD void rot_to_quat_xyzw(const double* m, double* o) {
  const double t = m[0] + m[4] + m[8];
  if (t > 0.0) {
    double s = sqrt(t + 1.0); o[3] = 0.5 * s; s = 0.5 / s;
    o[0] = (m[7] - m[5]) * s; o[1] = (m[2] - m[6]) * s; o[2] = (m[3] - m[1]) * s;
  } else if (m[8] > (m[4] > m[0] ? m[4] : m[0])) {   // pivot z (the three pivots written out: no run-time register indices)
    double s = sqrt(m[8] - m[0] - m[4] + 1.0); o[2] = 0.5 * s; s = 0.5 / s;
    o[3] = (m[3] - m[1]) * s; o[0] = (m[2] + m[6]) * s; o[1] = (m[5] + m[7]) * s;
  } else if (m[4] > m[0]) {                           // pivot y
    double s = sqrt(m[4] - m[8] - m[0] + 1.0); o[1] = 0.5 * s; s = 0.5 / s;
    o[3] = (m[2] - m[6]) * s; o[2] = (m[7] + m[5]) * s; o[0] = (m[1] + m[3]) * s;
  } else {                                            // pivot x
    double s = sqrt(m[0] - m[4] - m[8] + 1.0); o[0] = 0.5 * s; s = 0.5 / s;
    o[3] = (m[7] - m[5]) * s; o[1] = (m[3] + m[1]) * s; o[2] = (m[6] + m[2]) * s;
  }
}
QMB_HD void inv3(const double* m, double* o) {
  const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
  const double id = 1.0 / (m[0] * c00 + m[1] * c01 + m[2] * c02);
  o[0] = c00 * id; o[1] = (m[2] * m[7] - m[1] * m[8]) * id; o[2] = (m[1] * m[5] - m[2] * m[4]) * id;
  o[3] = c01 * id; o[4] = (m[0] * m[8] - m[2] * m[6]) * id; o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
  o[6] = c02 * id; o[7] = (m[1] * m[6] - m[0] * m[7]) * id; o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
}
// rotation vector of E = L * R^T  (ocs2 rotationErrorInWorld)
QMB_HD void rotation_error_world(const double* L, const double* Rr, double* e) {
  double E[9]; matmul3_nt(L, Rr, E);
  const double w[3] = {E[7] - E[5], E[2] - E[6], E[3] - E[1]};
  const double c = 0.5 * (E[0] + E[4] + E[8] - 1.0), s = 0.5 * sqrt(dot3(w, w));
  if (s < 1e-12) { e[0] = 0.5 * w[0]; e[1] = 0.5 * w[1]; e[2] = 0.5 * w[2]; return; }
  const double k = atan2(s, c) / (2.0 * s); e[0] = k * w[0]; e[1] = k * w[1]; e[2] = k * w[2];
}
// A composite rigid body being folded: mass, COM and inertia about the COM, all in one frame.  lump_add adds a body (mass m, COM c, inertia I about c) to it.
struct SrbdLump { double m = 0.0, c[3] = {0, 0, 0}, I[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}; };
QMB_HD void lump_shift(double mm, const double* cc, const double* II, const double* cn, double* out) {   // II about cc → about cn (parallel axis)
  const double d[3] = {cc[0] - cn[0], cc[1] - cn[1], cc[2] - cn[2]}; const double dd = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) out[3 * i + j] = II[3 * i + j] + mm * ((i == j ? dd : 0.0) - d[i] * d[j]);
}
QMB_HD void lump_add(SrbdLump& a, double m, const double* c, const double* I) {
  if (m == 0.0) { for (int i = 0; i < 9; ++i) a.I[i] += I[i]; return; }
  const double mt = a.m + m; double cn[3]; for (int i = 0; i < 3; ++i) cn[i] = (a.m * a.c[i] + m * c[i]) / mt;
  double I1[9], I2[9]; lump_shift(a.m, a.c, a.I, cn, I1); lump_shift(m, c, I, cn, I2);
  for (int i = 0; i < 9; ++i) a.I[i] = I1[i] + I2[i];
  a.m = mt; for (int i = 0; i < 3; ++i) a.c[i] = cn[i];
}

// rbd row s[55] → centroidal state x[30] = [h_lin / m, h_ang / m, base position, euler ZYX, joints] by the SRBD mapping of robot constants sc
// (CentroidalModelRbdConversions::computeCentroidalStateFromRbdModel [upstream, recalled]): h_lin / m = v_lin + (R c_nom) x w, h_ang = R I_nom R^T w.
// The yaw is copied as measured; the controller's observation unwraps it.
QMB_HD void centroidal_from_rbd(const SrbdConst& sc, const double* s, double* x) {
  double R[9]; rot_zyx(s[RBD_ZYX], s[RBD_ZYX + 1], s[RBD_ZYX + 2], R);
  const double w[3] = {s[RBD_W], s[RBD_W + 1], s[RBD_W + 2]};
  double c[3]; matvec3(R, sc.c_nom, c);
  double cw[3]; cross3(c, w, cw);
  double Rtw[3], IRtw[3], L[3]; matTvec3(R, w, Rtw); matvec3(sc.I_nom, Rtw, IRtw); matvec3(R, IRtw, L);
  const double inv_m = 1.0 / sc.m;
#pragma unroll
  for (int i = 0; i < 3; ++i) { x[i] = s[RBD_V + i] + cw[i]; x[3 + i] = L[i] * inv_m; x[6 + i] = s[RBD_POS + i]; x[9 + i] = s[RBD_ZYX + i]; }
#pragma unroll
  for (int j = 0; j < NJ; ++j) x[12 + j] = s[RBD_JPOS + j];
}

// The SRBD constants of one robot with model payload pl = [m_ee, o_ee(3), m_base, o_base(3)] (or NULL) → out[SRBD_DBL]: DevModel's nominal block (the fold of the
// bodies at defaultJointState: total_mass, I_nom about the composite COM, -c_nom) with each point mass added at its position in the default joint state, o_ee
// in the end-effector frame (ee_body at ee_body_R0 / ee_body_p0) and o_base in the base frame (at the origin, level), then the cofactor inverse of the inertia.
// A zero mass is skipped, and with both skipped out is the nominal block bit for bit.  The host's srbd_constants and the payload estimator's commit kernel
// both call this function.
QMB_HD void srbd_payload_fold(const DevModel& d, const double* pl, double* out) {
  const SrbdConst& nom = *reinterpret_cast<const SrbdConst*>(&d.total_mass);
  SrbdLump whole; whole.m = nom.m; for (int i = 0; i < 3; ++i) whole.c[i] = -nom.c_nom[i]; for (int i = 0; i < 9; ++i) whole.I[i] = nom.I_nom[i];
  double mass = nom.m; bool added = false;
  for (int k = 0; pl && k < 2; ++k) {
    const double m = pl[4 * k]; if (m == 0.0) continue;
    double cb[3] = {pl[4 * k + 1], pl[4 * k + 2], pl[4 * k + 3]};
    const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, z3[3] = {0, 0, 0};
    const double* R = k == 0 ? d.ee_body_R0 : I3; const double* p = k == 0 ? d.ee_body_p0 : z3;
    if (k == 0) { double o[3]; matvec3(d.ee_R, cb, o); for (int i = 0; i < 3; ++i) cb[i] = o[i] + d.ee_p[i]; }
    double c[3]; matvec3(R, cb, c); for (int i = 0; i < 3; ++i) c[i] += p[i];
    const double I0[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}; lump_add(whole, m, c, I0); mass += m; added = true;
  }
  double* o = out; o[0] = mass;
  for (int i = 0; i < 9; ++i) o[1 + i] = whole.I[i];
  if (added) inv3(whole.I, o + 10); else for (int i = 0; i < 9; ++i) o[10 + i] = nom.I_nom_inv[i];
  for (int i = 0; i < 3; ++i) o[19 + i] = -whole.c[i];
  for (int i = 22; i < SRBD_DBL; ++i) o[i] = 0.0;
}

// splitmix64's finaliser: a bijection of 64-bit words whose output bits each depend on every input bit.  The counter-based draws hash their keys with
// it: the sensor noise (state_est_api.cuh), the per-episode plant rows (episode_api.cuh) and spawns (spawn_api.cuh).
QMB_HD uint64_t mix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull; z = (z ^ (z >> 27)) * 0x94d049bb133111ebull; return z ^ (z >> 31);
}
// The key of one counter-based draw: (seed ^ domain, robot, index, column) hashed in turn.  Each consumer xors its own domain constant into the seed, so
// that its draws and another's of the same words are unrelated.  No generator state, so a draw does not depend on the batch or the launch.
QMB_HD uint64_t keyed_hash(uint64_t seed, uint64_t domain, uint64_t robot, uint64_t index, int column) {
  return mix64(mix64(mix64(mix64(seed ^ domain) ^ robot) ^ index) ^ (uint64_t)column);
}
// u in (0, 1) of a key h: the 53 high bits of one more hash, plus a half
QMB_HD double hash_uniform(uint64_t h) { return ((double)(mix64(h) >> 11) + 0.5) * 1.1102230246251565e-16; }
QMB_HD double keyed_uniform(uint64_t seed, uint64_t domain, uint64_t robot, uint64_t index, int column) {
  return hash_uniform(keyed_hash(seed, domain, robot, index, column));
}

// The check of a per-episode draw's ranges lo, hi [B][width] (qmb200_episode_set_ranges, qmb200_spawn_set_ranges; who names the entry point): "" when
// valid, else the first offence naming the field and the robot.  Every column needs finite bounds, lo <= hi and a finite hi - lo; extra(c, lo, hi)
// returns column c's own offence, or "".
template <class Extra>
std::string ranges_error(const char* who, const char* const* names, int width, const double* lo, const double* hi, size_t B, Extra extra) {
  for (size_t b = 0; b < B; ++b) for (int c = 0; c < width; ++c) {
    const double l = lo[b * width + c], u = hi[b * width + c];
    const std::string why = !(std::isfinite(l) && std::isfinite(u)) ? "bounds must be finite" : !(l <= u) ? "lo must be <= hi"
                          : !std::isfinite(u - l) ? "hi - lo must be finite" : extra(c, l, u);
    if (!why.empty()) return std::string(who) + ": " + names[c] + " of robot " + std::to_string(b) + ": " + why;
  }
  return "";
}

// modeNumber2StanceLeg: bit3 LF, bit2 RF, bit1 LH, bit0 RH (contact order LF,RF,LH,RH)
QMB_HD bool contact_flag(int mode, int foot) { return (mode >> (3 - foot)) & 1; }

}  // namespace qmb
