// Batched kernels for the steps either side of the MPC+WBC path (SURVEY.md §8f rows 1, 2 and 4):
//   ctrl_observation_kernel   QMController::updateStateEstimation tail (qm_controllers/src/QMController.cpp:236-243):
//                             currentObservation_.time += period; state = computeCentroidalStateFromRbdModel(rbd); yaw unwrap
//   ctrl_target_kernel        cmdVelToTargetTrajectories / EeCmdVelToTargetTrajectories / EEgoalPoseToTargetTrajectories
//                             (qm_controllers/src/QmTargetTrajectoriesPublisher_node.cpp:44-208) incl. the lastEeTarget_ bookkeeping
//                             (QmTargetTrajectoriesPublisher.h:55-57, QmTargetTrajectoriesPublisher.cpp:107-108)
//   ctrl_control_law_kernel   SafetyChecker::check (SafetyChecker.h:22-35) + QMController::updateControlLaw (QMController.cpp:177-190)
//                             / QMMpcController::updateControlLaw (QMController.cpp:427-445)
//   ctrl_hw_write_kernel      QMHWSim::writeSim (qm_gazebo/src/QMHWSim.cpp:98-116): command delay buffer + hybrid joint law
//                             tau = kp (posDes - q) + kd (velDes - qd) + ff (HybridJointInterface.h:55-61)
// All of them are maps over robots with O(100) flops and O(1 KB) of I/O per robot: HBM/latency bound.  One thread owns one robot
// (or one joint of a robot); rows are staged through shared memory so that every global access is a coalesced row-major sweep.
#include "ctrl_api.cuh"

namespace qmb {

namespace {
constexpr int OBS_ROBOTS = 64;    // robots per CTA of the row-staged kernels
constexpr double PI = 3.14159265358979323846;

// coalesced copy of `rows` consecutive rows of width W between global memory and a shared tile with leading dimension LD (odd → the
// thread-per-row accesses that follow are bank-conflict free)
template <int W, int LD> __device__ __forceinline__ void tile_load(double* tile, const double* __restrict__ g, int rows) {
  for (int i = threadIdx.x; i < rows * W; i += blockDim.x) tile[(i / W) * LD + (i % W)] = g[i];
}
template <int W, int LD> __device__ __forceinline__ void tile_store(double* __restrict__ g, const double* tile, int rows) {
  for (int i = threadIdx.x; i < rows * W; i += blockDim.x) g[i] = tile[(i / W) * LD + (i % W)];
}

// angles::shortest_angular_distance(from, to) = normalize_angle(to - from), normalize_angle(a) = fmod(fmod(a, 2pi) + 2pi, 2pi), shifted into (-pi, pi]
__device__ __forceinline__ double shortest_angular_distance(double from, double to) {
  double a = fmod(fmod(to - from, 2.0 * PI) + 2.0 * PI, 2.0 * PI);
  if (a > PI) a -= 2.0 * PI;
  return a;
}

}  // namespace

// -----------------------------------------------------------------------------------------------------------------
// Observation: rbd[55] → centroidal state (centroidal_from_rbd, as qmb200_centroidal_state_from_rbd) with the controller's yaw unwrap.  srbd: per-robot SRBD
// constants [B][SRBD_DBL] of a model payload, or NULL for the model's.
__global__ void __launch_bounds__(OBS_ROBOTS) ctrl_observation_kernel(const DevModel* __restrict__ mdl, int B, const double* __restrict__ rbd, const double* __restrict__ period,
                                                                       double* __restrict__ t_obs, double* __restrict__ x_obs, const double* __restrict__ srbd) {
  __shared__ double s_rbd[OBS_ROBOTS * 55];   // leading dimension 55 (odd)
  __shared__ double s_x[OBS_ROBOTS * 31];
  const int b0 = blockIdx.x * OBS_ROBOTS, rows = min(OBS_ROBOTS, B - b0), r = threadIdx.x;
  tile_load<55, 55>(s_rbd, rbd + (size_t)b0 * 55, rows);
  __syncthreads();
  if (r < rows) {
    double* o = s_x + r * 31;
    centroidal_from_rbd(*srbd_of(mdl, srbd, b0 + r), s_rbd + r * 55, o);
    const double yaw_last = x_obs[(size_t)(b0 + r) * NX + 9];           // currentObservation_.state(9) of the previous update
    o[9] = yaw_last + shortest_angular_distance(yaw_last, o[9]);
    t_obs[b0 + r] += period[b0 + r];
  }
  __syncthreads();
  tile_store<NX, 31>(x_obs + (size_t)b0 * NX, s_x, rows);
}

// -----------------------------------------------------------------------------------------------------------------
// Target front-end.  kind 0: /cmd_vel (cmd = vx, vy, vz, yaw rate), 1: /ee_cmd_vel (cmd = vx, vy, vz), 2: goal pose (cmd = pos(3), quat xyzw(4)).
// kinds [B] (or NULL: every robot `kind`): robot b's kind; a robot whose kind lies outside [0, 2] (-1: its goal is held) is left untouched.
// frame [B] (or NULL: every robot in the world frame): robot b's end-effector frame, EE_FRAME_WORLD or EE_FRAME_HEADING (target_robot).
// paths.state set: robots of kind TARGET_EE_PATH / _FOLLOW run target_path on their path state row and the path table (2 to KMAX knots).
// Output: the 2-knot TargetTrajectories [time; 37-dim state = (0_6 | v, base pose, defaultJointState, EE pose)] in the solver's layout.
__global__ void __launch_bounds__(128) ctrl_target_kernel(TargetParams prm, int kind_all, const int32_t* __restrict__ kinds, int B, const double* __restrict__ cmd /*[B][7]*/,
                                                           const double* __restrict__ t_obs, const double* __restrict__ x_obs, const double* __restrict__ ee_state /*[B][7]*/,
                                                           double* __restrict__ last_ee_target /*[B][7]*/, int32_t* __restrict__ n_target, double* __restrict__ target_times /*[B][KMAX]*/,
                                                           double* __restrict__ target_states /*[B][KMAX][37]*/, const int32_t* __restrict__ frame, TargetPaths paths) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x; if (b >= B) return;
  const int kind = kinds ? kinds[b] : kind_all;
  if (kind >= 0 && kind <= 2)
    target_robot(prm, kind, frame && frame[b] == EE_FRAME_HEADING, cmd + (size_t)b * 7, t_obs[b], x_obs + (size_t)b * NX, ee_state + (size_t)b * 7,
                 last_ee_target + (size_t)b * 7, n_target + b, target_times + (size_t)b * KMAX, target_states + (size_t)b * KMAX * TARGET_DIM);
  else if (paths.state && (kind == TARGET_EE_PATH || kind == TARGET_EE_PATH_FOLLOW))
    target_path(prm, kind == TARGET_EE_PATH, frame && frame[b] == EE_FRAME_HEADING, cmd + (size_t)b * 7, t_obs[b], x_obs + (size_t)b * NX, ee_state + (size_t)b * 7,
                last_ee_target + (size_t)b * 7, paths.state + (size_t)b * EE_PATH_STATE, paths.n, paths.n_way, paths.way, n_target + b,
                target_times + (size_t)b * KMAX, target_states + (size_t)b * KMAX * TARGET_DIM);
}

// -----------------------------------------------------------------------------------------------------------------
// Control law: one thread per (robot, joint).  joint_cmd[b][j] = (posDes, velDes, kp, kd, ff) as HybridJointHandle::setCommand receives them.
// variant 0 (QMController): legs only once time > 10 (before that the handle keeps its previous command: the entry is left untouched);
//   arm joints (posDes, 0, arm_kp, arm_kd, torque), with the robot's own arm gains when it has a tuning row (tuning [B][TUNING_DBL], NULL: none).
// variant 1 (QMMpcController): legs always; the arm is position controlled at 100 Hz: arm_pos_cmd[b][j] = state(24+j) + velDes(12+j)/100
//   whenever time - last_time > 1/100 (last_time is then advanced); its hybrid entries are left untouched.
// status: bit 0 = SafetyChecker orientation check failed (|roll| > pi/2 → the reference calls stopRequest).
__global__ void __launch_bounds__(ControlLawParams::THREADS) ctrl_control_law_kernel(ControlLawParams prm, int B, const double* __restrict__ x_des, const double* __restrict__ u_des, const double* __restrict__ wbc_cmd,
                                                                                      const double* __restrict__ t_obs, const double* __restrict__ x_obs, double* __restrict__ joint_cmd /*[B][18][5]*/,
                                                                                      double* __restrict__ arm_pos_cmd /*[B][6]*/, double* __restrict__ last_time /*[B]*/, int32_t* __restrict__ status,
                                                                                      const double* __restrict__ tuning) {
  const int b = blockIdx.x * ControlLawParams::ROBOTS + threadIdx.x / NJ, j = threadIdx.x % NJ;
  const bool live = threadIdx.x < ControlLawParams::ROBOTS * NJ && b < B;
  double t = 0.0, lt = 0.0;
  if (live) {
    t = t_obs[b];
    const double pos_des = x_des[(size_t)b * NX + 12 + j], vel_des = u_des[(size_t)b * NU + 12 + j], tau = wbc_cmd[(size_t)b * 54 + 36 + j];
    double* jc = joint_cmd + ((size_t)b * NJ + j) * 5;
    if (j < 12) {
      if (prm.variant == 1 || t > 10.0) { jc[0] = pos_des; jc[1] = vel_des; jc[2] = 0.0; jc[3] = 3.0; jc[4] = tau; }
    } else if (prm.variant == 0) {
      double kp = prm.arm_kp, kd = prm.arm_kd;
      if (tuning) { const double* tr = tuning + (size_t)b * TUNING_DBL; kp = tr[TUNING_ARM_KP]; kd = tr[TUNING_ARM_KD]; }
      jc[0] = pos_des; jc[1] = 0.0; jc[2] = kp; jc[3] = kd; jc[4] = tau;
    } else {
      lt = last_time[b];
      if (t - lt > 1.0 / 100.0) arm_pos_cmd[(size_t)b * 6 + j - 12] = x_obs[(size_t)b * NX + 12 + j] + vel_des * 1.0 / 100.0;
    }
    if (j == 0) { const double roll = x_obs[(size_t)b * NX + 11]; status[b] = (roll > 0.5 * PI || roll < -0.5 * PI) ? 1 : 0; }
  }
  __syncthreads();   // every arm thread has read last_time before it moves
  if (live && prm.variant == 1 && j == 12 && t - lt > 1.0 / 100.0) last_time[b] = t;
}

// -----------------------------------------------------------------------------------------------------------------
// QMHWSim::writeSim: per robot a FIFO of stamped commands (ring of HW_DEPTH entries, oldest at `tail`); the command applied is the oldest
// one that is not older than `delay`.  One thread per (robot, joint); all joints of a robot share the stamps.
__global__ void __launch_bounds__(ControlLawParams::THREADS) ctrl_hw_write_kernel(int B, double delay, const double* __restrict__ time, const double* __restrict__ period,
                                                                                   const double* __restrict__ joint_cmd /*[B][18][5]*/, const double* __restrict__ joint_pos /*[B][18]*/,
                                                                                   const double* __restrict__ joint_vel, double* __restrict__ ring_cmd /*[B][HW_DEPTH][18][5]*/,
                                                                                   double* __restrict__ ring_stamp /*[B][HW_DEPTH]*/, int32_t* __restrict__ ring_state /*[B][2] tail, count*/,
                                                                                   double* __restrict__ effort /*[B][18]*/, int32_t* __restrict__ status) {
  const int b = blockIdx.x * ControlLawParams::ROBOTS + threadIdx.x / NJ, j = threadIdx.x % NJ;
  const bool live = threadIdx.x < ControlLawParams::ROBOTS * NJ && b < B;
  int tail = 0, count = 0, st = 0; double t = 0.0;
  if (live) {
    t = time[b]; tail = ring_state[2 * b]; count = ring_state[2 * b + 1];
    const double* stamp = ring_stamp + (size_t)b * HW_DEPTH;
    if (t == period[b]) count = 0;                                                             // simulation reset (:101-103)
    while (count > 0 && stamp[tail] + delay < t) { tail = (tail + 1) % HW_DEPTH; --count; }    // pop_back of expired commands (:105-107)
    if (count == HW_DEPTH) { tail = (tail + 1) % HW_DEPTH; --count; st = 2; }                  // ring full (the reference deque is unbounded): drop the oldest, flag it
    const int head = (tail + count) % HW_DEPTH;
    const double* jc = joint_cmd + ((size_t)b * NJ + j) * 5; double* slot = ring_cmd + (((size_t)b * HW_DEPTH + head) * NJ + j) * 5;
    double c5[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) { c5[i] = jc[i]; slot[i] = c5[i]; }                            // push_front (:108-109)
    if (count > 0) { const double* old = ring_cmd + (((size_t)b * HW_DEPTH + tail) * NJ + j) * 5;
#pragma unroll
      for (int i = 0; i < 5; ++i) c5[i] = old[i]; }                                            // buffer.back() (:111)
    effort[(size_t)b * NJ + j] = c5[2] * (c5[0] - joint_pos[(size_t)b * NJ + j]) + c5[3] * (c5[1] - joint_vel[(size_t)b * NJ + j]) + c5[4];
  }
  __syncthreads();   // every joint thread has read the stamps / ring state of its robot
  if (live && j == 0) { ring_stamp[(size_t)b * HW_DEPTH + (tail + count) % HW_DEPTH] = t; ring_state[2 * b] = tail; ring_state[2 * b + 1] = count + 1; status[b] = st; }
}

// -----------------------------------------------------------------------------------------------------------------
int launch_observation(const DevModel* mdl, int B, const double* rbd, const double* period, double* t_obs, double* x_obs, cudaStream_t s, const double* srbd) {
  ctrl_observation_kernel<<<(B + OBS_ROBOTS - 1) / OBS_ROBOTS, OBS_ROBOTS, 0, s>>>(mdl, B, rbd, period, t_obs, x_obs, srbd); return 1;
}
int launch_target(const TargetParams& prm, int kind, const int32_t* kinds, int B, const double* cmd, const double* t_obs, const double* x_obs, const double* ee_state,
                  double* last_ee_target, int32_t* n_target, double* target_times, double* target_states, cudaStream_t s, const int32_t* frame,
                  const TargetPaths& paths) {
  ctrl_target_kernel<<<(B + 127) / 128, 128, 0, s>>>(prm, kind, kinds, B, cmd, t_obs, x_obs, ee_state, last_ee_target, n_target, target_times, target_states, frame,
                                                     paths); return 1;
}
int launch_control_law(const ControlLawParams& prm, int B, const double* x_des, const double* u_des, const double* wbc_cmd, const double* t_obs, const double* x_obs,
                       double* joint_cmd, double* arm_pos_cmd, double* last_time, int32_t* status, cudaStream_t s, const double* tuning) {
  ctrl_control_law_kernel<<<(B + ControlLawParams::ROBOTS - 1) / ControlLawParams::ROBOTS, ControlLawParams::THREADS, 0, s>>>(prm, B, x_des, u_des, wbc_cmd, t_obs, x_obs, joint_cmd, arm_pos_cmd, last_time, status, tuning); return 1;
}
int launch_hw_write(int B, double delay, const double* time, const double* period, const double* joint_cmd, const double* joint_pos, const double* joint_vel,
                    double* ring_cmd, double* ring_stamp, int32_t* ring_state, double* effort, int32_t* status, cudaStream_t s) {
  ctrl_hw_write_kernel<<<(B + ControlLawParams::ROBOTS - 1) / ControlLawParams::ROBOTS, ControlLawParams::THREADS, 0, s>>>(B, delay, time, period, joint_cmd, joint_pos, joint_vel, ring_cmd, ring_stamp, ring_state, effort, status); return 1;
}

}  // namespace qmb
