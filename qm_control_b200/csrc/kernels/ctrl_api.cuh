// Host-visible interface of the controller-side kernels (observation, target front-end, control law, hybrid-joint plant law).  The target front-end's
// per-robot body (target_robot) is host + device: ctrl_target_kernel runs it, and tests/ee_frame_host.cpp compiles it with g++ for the CPU suite.
#pragma once
#include <cuda_runtime.h>

#include "dev_common.cuh"
#include "mpc_api.cuh"
#include "sim_api.cuh"

namespace qmb {

constexpr int HW_DEPTH = 32;   // command-delay ring entries per robot (delay 0.009 s at a 1 kHz loop needs 10; gazebo/config/default.yaml:2)

// constants of the target publisher node (QmTargetTrajectoriesPublisher_node.cpp:225-229)
struct TargetParams {
  double com_height;                     // reference.info comHeight
  double target_displacement_velocity;   // reference.info targetDisplacementVelocity
  double target_rotation_velocity;       // reference.info targetRotationVelocity
  double time_to_target;                 // task.info mpc.timeHorizon
  double default_joint_state[NJ];        // reference.info defaultJointState
};

// The frame a robot's end-effector targets are stated in (qmb200_set_ee_frame; DESIGN.md §4.19)
constexpr int EE_FRAME_WORLD = 0, EE_FRAME_HEADING = 1;
// The check of qmb200_set_ee_frame on rows frame [B]: "" when every row is EE_FRAME_WORLD or EE_FRAME_HEADING, else the message naming the first robot
inline std::string ee_frame_error(const int32_t* frame, size_t B) {
  for (size_t b = 0; b < B; ++b)
    if (frame[b] != EE_FRAME_WORLD && frame[b] != EE_FRAME_HEADING)
      return "qmb200_set_ee_frame: frame of robot " + std::to_string(b) + " is " + std::to_string(frame[b]) +
             ", not QMB200_EE_FRAME_WORLD (0) or QMB200_EE_FRAME_HEADING (1)";
  return "";
}

// The heading frame H of a base at (x, y, yaw): origin (x, y, 0), rotation Rz(yaw), z the world's.  s, c: sine and cosine of yaw; sh, ch: of yaw / 2,
// from spawn_sincos, whose device path needs no stack for an unwrapped yaw of many turns.  A position maps as p_w = Rz p_H + (x, y, 0), a quaternion
// (xyzw) as q_w = q_z(yaw) q_H: the product spawn_stand applies to a world-frame hold.  At (0, 0, 0) both maps return their input bit for bit.
struct Heading { double x, y, s, c, sh, ch; };
QMB_HD Heading heading_at(double x, double y, double yaw) {
  Heading h{x, y, 0.0, 1.0, 0.0, 1.0}; spawn_sincos(yaw, h.s, h.c); spawn_sincos(0.5 * yaw, h.sh, h.ch); return h;
}
// pose p [7] (position, quaternion xyzw) in H → o [7] in the world; o may not alias p
QMB_HD void heading_to_world(const Heading& h, const double* p, double* o) {
  o[0] = (h.c * p[0] - h.s * p[1]) + h.x; o[1] = (h.s * p[0] + h.c * p[1]) + h.y; o[2] = p[2];
  o[3] = h.ch * p[3] - h.sh * p[4]; o[4] = h.ch * p[4] + h.sh * p[3]; o[5] = h.ch * p[5] + h.sh * p[6]; o[6] = h.ch * p[6] - h.sh * p[5];
}
// position p [3] in the world → o [3] in H
QMB_HD void heading_pos_from_world(const Heading& h, const double* p, double* o) {
  const double dx = p[0] - h.x, dy = p[1] - h.y;
  o[0] = h.c * dx + h.s * dy; o[1] = h.c * dy - h.s * dx; o[2] = p[2];
}
// quaternion q [4] (xyzw) in the world → o [4] in H: q_z(-yaw) q
QMB_HD void heading_quat_from_world(const Heading& h, const double* q, double* o) {
  o[0] = h.ch * q[0] + h.sh * q[1]; o[1] = h.ch * q[1] - h.sh * q[0]; o[2] = h.ch * q[2] - h.sh * q[3]; o[3] = h.ch * q[3] + h.sh * q[2];
}

// Eigen::Quaterniond(w, x, y, z).toRotationMatrix()
QMB_HD void quat_to_rot(double w, double x, double y, double z, double* R) {
  const double tx = 2.0 * x, ty = 2.0 * y, tz = 2.0 * z, twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1.0 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = 1.0 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1.0 - (txx + tyy);
}

// One robot of the target front-end (ctrl_target_kernel): kind 0 /cmd_vel (c = vx, vy, vz, yaw rate), 1 /ee_cmd_vel (c = vx, vy, vz), 2 goal pose
// (c = pos(3), quat xyzw(4)); t, x: the observation time and state [NX], ee [7]: the measured hand, le [7]: the held end-effector target (in-out).
// Writes the 2-knot TargetTrajectories [time; 37-dim state = (0_6 | v, base pose, defaultJointState, EE pose)]: tt [KMAX], ts [KMAX][TARGET_DIM].
// heading false: upstream's world-frame arithmetic.  heading true (DESIGN.md §4.19): le is the hold in the robot's heading frame H(cur) of the
// observed base (x[6], x[7], x[9]), a goal c is a pose in H(cur), and the base offset of kinds 1 and 2 turns with the yaw.
QMB_HD void target_robot(const TargetParams& prm, int kind, bool heading, const double* c, double t, const double* x, const double* ee, double* le,
                         int32_t* n_target, double* tt, double* ts) {
  double base_cur[6]; for (int i = 0; i < 6; ++i) base_cur[i] = x[6 + i];
  double base_tgt[6], ee_cur[7], ee_tgt[7], vel[3] = {0.0, 0.0, 0.0}, t_reach;
  const Heading hc = heading ? heading_at(base_cur[0], base_cur[1], base_cur[3]) : Heading{0.0, 0.0, 0.0, 1.0, 0.0, 1.0};
  if (kind == 0) {            // cmdVelToTargetTrajectories (:73-113)
    double R[9]; rot_zyx(base_cur[3], base_cur[4], base_cur[5], R); matvec3(R, c, vel);
    base_tgt[0] = base_cur[0] + vel[0] * prm.time_to_target; base_tgt[1] = base_cur[1] + vel[1] * prm.time_to_target; base_tgt[2] = prm.com_height;
    base_tgt[3] = base_cur[3] + c[3] * prm.time_to_target; base_tgt[4] = 0.0; base_tgt[5] = 0.0;
    if (!heading) {
      const double d0 = le[0] - ee[0], d1 = le[1] - ee[1], d2 = le[2] - ee[2];
      if (sqrt(d0 * d0 + d1 * d1 + d2 * d2) > 0.1) { le[0] = ee[0]; le[1] = ee[1]; le[2] = ee[2]; }
      for (int i = 0; i < 7; ++i) { ee_tgt[i] = le[i]; ee_cur[i] = le[i]; }   // eeStateLast.state = EeTargetPose (:104-105)
    } else {                  // the hold rides on the base: H(cur) le now, H(tgt) le at the base target
      heading_to_world(hc, le, ee_cur);
      const double d0 = ee_cur[0] - ee[0], d1 = ee_cur[1] - ee[1], d2 = ee_cur[2] - ee[2];
      if (sqrt(d0 * d0 + d1 * d1 + d2 * d2) > 0.1) { heading_pos_from_world(hc, ee, le); heading_to_world(hc, le, ee_cur); }
      heading_to_world(heading_at(base_tgt[0], base_tgt[1], base_tgt[3]), le, ee_tgt);
    }
    t_reach = t + prm.time_to_target;
  } else if (kind == 1) {     // EeCmdVelToTargetTrajectories (:118-165)
    double Rq[9], Ri[9], M[9]; quat_to_rot(ee[6], ee[3], ee[4], ee[5], Rq); quat_to_rot(-0.5, 0.5, -0.5, 0.5, Ri); matmul3_nt(Rq, Ri, M);
    double v[3]; matvec3(M, c, v);
    for (int i = 0; i < 7; ++i) ee_cur[i] = ee[i];
    ee_tgt[0] = ee[0] + v[0] * prm.time_to_target; ee_tgt[1] = ee[1] + v[1] * prm.time_to_target;
    if (!heading) for (int i = 2; i < 7; ++i) ee_tgt[i] = le[i];
    else { double hw[7]; heading_to_world(hc, le, hw); for (int i = 2; i < 7; ++i) ee_tgt[i] = hw[i]; }
    for (int i = 0; i < 6; ++i) base_tgt[i] = base_cur[i];
    if (!heading) { base_tgt[0] = ee_tgt[0] - 0.52; base_tgt[1] = ee_tgt[1] - 0.09; }
    else { base_tgt[0] = ee_tgt[0] - (hc.c * 0.52 - hc.s * 0.09); base_tgt[1] = ee_tgt[1] - (hc.s * 0.52 + hc.c * 0.09); }
    base_tgt[2] = prm.com_height; base_tgt[4] = 0.0; base_tgt[5] = 0.0;
    t_reach = t + prm.time_to_target;
  } else {                    // EEgoalPoseToTargetTrajectories (:172-208) + processFeedback's lastEeTarget_ update
    double g[7];              // the goal in the world: c itself, or H(cur) c
    if (!heading) for (int i = 0; i < 7; ++i) g[i] = c[i];
    else heading_to_world(hc, c, g);
    for (int i = 0; i < 7; ++i) { ee_cur[i] = ee[i]; ee_tgt[i] = g[i]; }
    for (int i = 0; i < 6; ++i) base_tgt[i] = base_cur[i];
    if (!heading) { base_tgt[0] = g[0] - 0.52; base_tgt[1] = g[1] - 0.09; }
    else { base_tgt[0] = g[0] - (hc.c * 0.52 - hc.s * 0.09); base_tgt[1] = g[1] - (hc.s * 0.52 + hc.c * 0.09); }
    base_tgt[2] = prm.com_height; base_tgt[4] = 0.0; base_tgt[5] = 0.0;
    // quaternionDistance(q_current, q_target) = w_c v_t - w_t v_c + v_c x v_t [upstream ocs2_robotic_tools, recalled]
    const double wc = ee[6], wt = g[6]; const double vc[3] = {ee[3], ee[4], ee[5]}, vt[3] = {g[3], g[4], g[5]}; double cr[3]; cross3(vc, vt, cr);
    double dl = 0.0, dr = 0.0;
    for (int i = 0; i < 3; ++i) { const double dp = g[i] - ee[i], dq = wc * vt[i] - wt * vc[i] + cr[i]; dl += dp * dp; dr += dq * dq; }
    t_reach = t + fmax(sqrt(dr) / prm.target_rotation_velocity, sqrt(dl) / prm.target_displacement_velocity);   // estimateTimeToTarget (:24-41)
    if (!heading) for (int i = 0; i < 7; ++i) le[i] = g[i];
    else {                    // the goal in H(tgt): the base target keeps the current yaw, so H(tgt) turns as H(cur) does
      const Heading ht{base_tgt[0], base_tgt[1], hc.s, hc.c, hc.sh, hc.ch};
      heading_pos_from_world(ht, g, le); heading_quat_from_world(ht, g + 3, le + 3);
    }
  }
  base_cur[2] = prm.com_height; base_cur[4] = 0.0; base_cur[5] = 0.0;   // targetPoseToTargetTrajectories (:44-68)
  *n_target = 2; tt[0] = t; tt[1] = t_reach; for (int k = 2; k < KMAX; ++k) tt[k] = 0.0;
  for (int k = 0; k < 2; ++k) {
    double* s = ts + k * TARGET_DIM;
    for (int i = 0; i < 3; ++i) { s[i] = vel[i]; s[3 + i] = 0.0; }
    for (int i = 0; i < 6; ++i) s[6 + i] = k == 0 ? base_cur[i] : base_tgt[i];
    for (int j = 0; j < NJ; ++j) s[12 + j] = prm.default_joint_state[j];
    for (int i = 0; i < 7; ++i) s[30 + i] = k == 0 ? ee_cur[i] : ee_tgt[i];
  }
  for (int i = 2 * TARGET_DIM; i < KMAX * TARGET_DIM; ++i) ts[i] = 0.0;
}

// End-effector paths (qmb200_set_ee_paths, qmb200_target_trajectories_path; DESIGN.md §4.20).  A waypoint is (tau, position 3, quaternion xyzw 4); a
// path row of the table is EE_PATH_MAX waypoints.  A robot's path state row: index, t0, the heading at the start (x0, y0, yaw0), the hand's start pose [7].
constexpr int TARGET_EE_PATH = 3, TARGET_EE_PATH_FOLLOW = 4;
constexpr int EE_PATH_MAX = 32, EE_PATH_WAY = 8, EE_PATH_STATE = 12;
// The check of qmb200_set_ee_paths on n_paths paths (n_way [n_paths], way [n_paths][EE_PATH_MAX][EE_PATH_WAY]) for a handle of time horizon T: "" when
// accepted, else the message naming the path and the waypoint
inline std::string ee_paths_error(int n_paths, const int32_t* n_way, const double* way, double T) {
  const std::string who = "qmb200_set_ee_paths: ";
  if (n_paths < 0) return who + "n_paths must be >= 0";
  for (int p = 0; p < n_paths; ++p) {
    const std::string path = "path " + std::to_string(p);
    if (n_way[p] < 1 || n_way[p] > EE_PATH_MAX) return who + path + " has " + std::to_string(n_way[p]) + " waypoints, not 1 to QMB200_EE_PATH_MAX (32)";
    for (int i = 0; i < n_way[p]; ++i) {
      const double* w = way + ((size_t)p * EE_PATH_MAX + i) * EE_PATH_WAY; const std::string at = who + path + ", waypoint " + std::to_string(i) + ": ";
      for (int k = 0; k < EE_PATH_WAY; ++k) if (!std::isfinite(w[k])) return at + "value " + std::to_string(k) + " is not finite";
      if (i == 0 && !(w[0] > 0.0)) return at + "its time must be > 0 (seconds after the path starts)";
      if (i > 0 && !(w[0] > w[-EE_PATH_WAY])) return at + "its time is not after waypoint " + std::to_string(i - 1) + "'s";
      if (i > 0 && w[0] - w[-EE_PATH_WAY] < 0.5 * T) return at + "its gap to waypoint " + std::to_string(i - 1) + " is under T/2 = " + std::to_string(0.5 * T) + " s";
      const double qn = std::sqrt(w[4] * w[4] + w[5] * w[5] + w[6] * w[6] + w[7] * w[7]);
      if (!(std::fabs(qn - 1.0) <= 1e-9)) return at + "its quaternion must have unit norm (within 1e-9)";
    }
  }
  return "";
}

// o [7] = the pose at weight a between poses l and r [7] as target_pose interpolates two knots (a l + (1 - a) r, Eigen slerp semantics); a == 1 gives l
// itself.  The slerp's sines take angles in [0, pi/2]: spawn_sincos, whose device path needs no stack.
QMB_HD void path_pose(const double* l, const double* r, double a, double* o) {
  if (a == 1.0) { for (int i = 0; i < 7; ++i) o[i] = l[i]; return; }
  for (int i = 0; i < 3; ++i) o[i] = a * l[i] + (1.0 - a) * r[i];
  const double* ql = l + 3; const double* qr = r + 3; const double tq = 1.0 - a; double d = 0.0; for (int i = 0; i < 4; ++i) d += ql[i] * qr[i];
  const double ad = fabs(d); double s0, s1, cs;
  if (ad >= 1.0 - 2.220446049250313e-16) { s0 = 1.0 - tq; s1 = tq; }
  else { const double th = acos(ad); double st; spawn_sincos(th, st, cs); const double ist = 1.0 / st; spawn_sincos((1.0 - tq) * th, s0, cs); spawn_sincos(tq * th, s1, cs); s0 *= ist; s1 *= ist; }
  if (d < 0.0) s1 = -s1;
  for (int i = 0; i < 4; ++i) o[3 + i] = s0 * ql[i] + s1 * qr[i];
}

// waypoint w [EE_PATH_WAY] of a path → its pose o [7] in the world: itself, or h0 (the heading frame at the path's start) applied to it
QMB_HD void path_way_world(const Heading& h0, bool heading, const double* w, double* o) {
  if (!heading) for (int i = 0; i < 7; ++i) o[i] = w[1 + i];
  else heading_to_world(h0, w + 1, o);
}

// One robot of the target front-end on a path (DESIGN.md §4.20): start (kind TARGET_EE_PATH: path index c[0]) or follow (TARGET_EE_PATH_FOLLOW) with
// the path state row ps [EE_PATH_STATE] (in-out) on the table (n_paths paths, n_way [n_paths], way [n_paths][EE_PATH_MAX][EE_PATH_WAY]).  Arguments
// otherwise as target_robot's.  A path index outside [0, n_paths) leaves everything untouched; so does a path with no waypoint after t, after a start's
// writes.  Knot 0 is the path's own pose p(t) (not the measured hand), so that between knots the MPC's reference is the path itself.
QMB_HD void target_path(const TargetParams& prm, bool start, bool heading, const double* c, double t, const double* x, const double* ee, double* le, double* ps,
                        int n_paths, const int32_t* n_way, const double* way, int32_t* n_target, double* tt, double* ts) {
  const double fi = start ? c[0] : ps[0];
  if (!(fi >= 0.0 && fi < (double)n_paths && floor(fi) == fi)) return;
  const int p = (int)fi, n = n_way[p]; const double* wp = way + (size_t)p * EE_PATH_MAX * EE_PATH_WAY;
  const Heading hc = heading ? heading_at(x[6], x[7], x[9]) : Heading{0.0, 0.0, 0.0, 1.0, 0.0, 1.0};
  const double ox = heading ? hc.c * 0.52 - hc.s * 0.09 : 0.52, oy = heading ? hc.s * 0.52 + hc.c * 0.09 : 0.09;   // the base offset, as the goal's
  if (start) {
    ps[0] = fi; ps[1] = t; ps[2] = x[6]; ps[3] = x[7]; ps[4] = x[9]; for (int i = 0; i < 7; ++i) ps[5 + i] = ee[i];
    double g[7]; path_way_world(hc, heading, wp + (size_t)(n - 1) * EE_PATH_WAY, g);   // H(start) is H(cur) on the start tick
    if (!heading) for (int i = 0; i < 7; ++i) le[i] = g[i];   // the final waypoint as a goal published now leaves the hold
    else { const Heading ht{g[0] - ox, g[1] - oy, hc.s, hc.c, hc.sh, hc.ch}; heading_pos_from_world(ht, g, le); heading_quat_from_world(ht, g + 3, le + 3); }
  }
  const double t0 = ps[1];
  int j = 0; while (j < n && !(t0 + wp[(size_t)j * EE_PATH_WAY] > t)) ++j;   // the first waypoint after t (n <= EE_PATH_MAX)
  if (j == n) return;
  const Heading h0 = heading ? heading_at(ps[2], ps[3], ps[4]) : hc;
  double e[7], r[7];
  path_way_world(h0, heading, wp + (size_t)j * EE_PATH_WAY, r);
  const double tr = t0 + wp[(size_t)j * EE_PATH_WAY];
  if (j == 0) path_pose(ps + 5, r, fmin((tr - t) / (tr - t0), 1.0), e);   // before its start the path is its start pose
  else { double l[7]; path_way_world(h0, heading, wp + (size_t)(j - 1) * EE_PATH_WAY, l); const double tl = t0 + wp[(size_t)(j - 1) * EE_PATH_WAY]; path_pose(l, r, (tr - t) / (tr - tl), e); }
  const int m = n - j < KMAX - 1 ? n - j : KMAX - 1;   // waypoint knots
  *n_target = 1 + m; tt[0] = t;
  for (int k = 0; k < KMAX; ++k) {
    double* s = ts + k * TARGET_DIM;
    if (k > m) { tt[k] = 0.0; for (int i = 0; i < TARGET_DIM; ++i) s[i] = 0.0; continue; }
    if (k > 0) { const double* w = wp + (size_t)(j + k - 1) * EE_PATH_WAY; tt[k] = t0 + w[0]; path_way_world(h0, heading, w, e); }
    for (int i = 0; i < 6; ++i) s[i] = 0.0;
    s[6] = k == 0 ? x[6] : e[0] - ox; s[7] = k == 0 ? x[7] : e[1] - oy; s[8] = prm.com_height; s[9] = x[9]; s[10] = 0.0; s[11] = 0.0;
    for (int jj = 0; jj < NJ; ++jj) s[12 + jj] = prm.default_joint_state[jj];
    for (int i = 0; i < 7; ++i) s[30 + i] = e[i];
  }
}

struct ControlLawParams {
  static constexpr int ROBOTS = 7, THREADS = 128;   // 7 robots x 18 joints = 126 threads of a 128-thread CTA
  int variant;                // 0 QMController, 1 QMMpcController
  double arm_kp, arm_kd;      // dynamic_reconfigure kp_arm_wbc / kd_arm_wbc (qm_controllers/cfg/weight.cfg:7-8: 0.0, 0.5)
};

int launch_observation(const DevModel* mdl, int B, const double* rbd, const double* period, double* t_obs, double* x_obs, cudaStream_t s, const double* srbd /*[B][SRBD_DBL] or NULL*/);
// kinds [B] (device, or NULL: every robot `kind`): per-robot kind; robots outside [0, 2] (and the path kinds when paths.state is set) are left
// untouched.  frame [B] (device, or NULL: every robot EE_FRAME_WORLD): per-robot end-effector frame
// paths: the path rows of qmb200_target_trajectories_path (state NULL: none; robots of the path kinds are then left untouched)
struct TargetPaths { double* state; int n; const int32_t* n_way; const double* way; };
int launch_target(const TargetParams& prm, int kind, const int32_t* kinds, int B, const double* cmd, const double* t_obs, const double* x_obs, const double* ee_state,
                  double* last_ee_target, int32_t* n_target, double* target_times, double* target_states, cudaStream_t s, const int32_t* frame,
                  const TargetPaths& paths = TargetPaths{nullptr, 0, nullptr, nullptr});
int launch_control_law(const ControlLawParams& prm, int B, const double* x_des, const double* u_des, const double* wbc_cmd, const double* t_obs, const double* x_obs,
                       double* joint_cmd, double* arm_pos_cmd, double* last_time, int32_t* status, cudaStream_t s,
                       const double* tuning /*[B][TUNING_DBL] or NULL: the robots' arm gains in place of prm's*/);
int launch_hw_write(int B, double delay, const double* time, const double* period, const double* joint_cmd, const double* joint_pos, const double* joint_vel,
                    double* ring_cmd, double* ring_stamp, int32_t* ring_state, double* effort, int32_t* status, cudaStream_t s);

}  // namespace qmb
